"""-m gpu: StreamRunner's frames mode -- raw uint8 camera frames of per-stream sizes warped, normalised and packed on the
device (ct_pack_stem_frames on the bf16 engine, ct_warp_affine_normalize per stream on the others), tracks in each
stream's source pixels.  Against the unfused kernels byte for byte, against a runner fed the fp32 images of
pre_process_device bit for bit, and closed-loop against the host pipeline."""
import ctypes as C

import numpy as np
import pytest
import torch

from centertrack_b200 import _lib as L
from centertrack_b200 import synthetic as wt
from helpers import make_model, make_opt

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')
EXACT = ('tracking_id', 'age', 'active', 'class')


def _host_detector(opt):
  from centertrack_b200.dataset_info import get_dataset
  from centertrack_b200.detector import Detector
  from centertrack_b200.tracker import Tracker
  det = object.__new__(Detector)
  ds = get_dataset(opt.dataset)
  det.opt, det.cnt, det.pre_images, det.tracker = opt, 0, None, Tracker(opt)
  det.mean = np.array(ds.mean, dtype=np.float32).reshape(1, 1, 3)
  det.std = np.array(ds.std, dtype=np.float32).reshape(1, 1, 3)
  det.rest_focal_length = opt.test_focal_length if opt.test_focal_length >= 0 else ds.rest_focal_length
  det.flip_idx = ds.flip_idx
  return det


def _frame(h, w, seed):
  """A uint8 BGR camera-like frame: the synthetic band-limited scene brought back to pixel values."""
  x = wt.synthetic_inputs(1, h, w, seed=seed, n_blobs=0)[0][0].permute(1, 2, 0).numpy()
  return np.ascontiguousarray(np.clip(x * 70.0 + 115.0, 0, 255).astype(np.uint8))


# ------------------------------------------------------------------------------------------------ kernel bytes
def _ragged(opt, streams, seed):
  """streams: (h, w, row pitch) -> (cur, prev device buffers, ct_frame array, minv [B,6] on the device)."""
  from centertrack_b200.detector import frame_geometry
  rng = np.random.RandomState(seed)
  frames = (L.Frame * len(streams))()
  bufs = [bytearray(), bytearray()]
  minv = []
  for b, (h, w, pitch) in enumerate(streams):
    off = len(bufs[0])
    for i, buf in enumerate(bufs):       # the pitch padding is noise: never read
      img = rng.randint(0, 256, size=(h, pitch), dtype=np.uint8)
      img[:, :3 * w] = _frame(h, w, seed + 7 * b + i).reshape(h, 3 * w)
      buf += img.tobytes() + bytes((-(h * pitch)) % 16)
    _, m = frame_geometry(opt, h, w)
    f = frames[b]
    f.offset, f.h, f.w, f.step = off, h, w, pitch
    f.minv[:] = m.tolist()
    minv.append(m)
  dev = [torch.frombuffer(bytearray(bb), dtype=torch.uint8).to(DEV) for bb in bufs]
  return dev[0], dev[1], frames, torch.from_numpy(np.stack(minv)).to(DEV)


@pytest.mark.parametrize('out_hw', [(544, 960), (384, 1280)])
def test_pack_stem_frames_equals_warp_then_pack_byte_for_byte(out_hw):
  """Ragged streams in one call -- 1080x1920, 480x640, KITTI's 375x1242 (zero border), 544x960 (the identity map at
  544x960), an odd width with a padded row pitch -- against ct_warp_affine_normalize per stream + ct_pack_stem_input,
  for the first frame (prev = cur), no previous frame, no pre_hm, and both present."""
  H, W = out_hw
  opt = make_opt('mot', ['--input_h', str(H), '--input_w', str(W)])
  from centertrack_b200.dataset_info import get_dataset
  ds = get_dataset(opt.dataset)
  mean = np.ascontiguousarray(ds.mean, np.float32).reshape(3)
  std = np.ascontiguousarray(ds.std, np.float32).reshape(3)
  ms = C.c_void_p(mean.ctypes.data), C.c_void_p(std.ctypes.data)
  streams = [(1080, 1920, 5760), (480, 640, 1920), (375, 1242, 3726), (544, 960, 2880), (301, 457, 1392)]
  B = len(streams)
  cur, prev, frames, minv = _ragged(opt, streams, 11)
  hm = torch.rand((B, 1, H, W), device=DEV)
  lib, st = L.lib(), L.stream_ptr()

  def warped(buf):
    img = torch.empty((B, 3, H, W), device=DEV)
    for b, f in enumerate(frames):
      L.check(lib.ct_warp_affine_normalize(C.c_void_p(buf.data_ptr() + f.offset), 1, f.h, f.w, f.step, L.ptr(minv[b]),
                                           *ms, L.ptr(img[b]), H, W, st))
    return img

  img_cur, img_prev = warped(cur), warped(prev)
  for name, pv, pre_img, h in (('first', cur, img_cur, hm), ('no_prev', None, None, hm),
                               ('no_hm', prev, img_prev, None), ('both', prev, img_prev, hm)):
    ref = torch.full((B, H, W, 8), 7.0, dtype=torch.bfloat16, device=DEV)
    got = torch.full((B, H, W, 8), -7.0, dtype=torch.bfloat16, device=DEV)
    L.check(lib.ct_pack_stem_input(L.ptr(img_cur), L.ptr(pre_img), L.ptr(h), L.ptr(ref), B, H, W, st))
    L.check(lib.ct_pack_stem_frames(L.ptr(cur), L.ptr(pv), frames, B, *ms, L.ptr(h), L.ptr(got), H, W, st))
    torch.cuda.synchronize()
    eq = got.view(torch.int16) == ref.view(torch.int16)
    assert bool(eq.all()), (name, int((~eq).sum()), [int((~eq[b]).sum()) for b in range(B)])
  if out_hw == (544, 960):   # the identity stream is the frame itself, normalised
    x = torch.from_numpy(np.frombuffer(cur.cpu().numpy().tobytes()[frames[3].offset:][:544 * 2880], np.uint8).copy())
    want = ((x.view(544, 960, 3).double() / 255 - torch.from_numpy(mean).double()) / torch.from_numpy(std).double())
    assert torch.equal(img_cur[3].permute(1, 2, 0).cpu(), want.float())


# ------------------------------------------------------------------------------------------ records vs fp32 images
SIZES = [(120, 200), (97, 131), (160, 128)]


def _coco(extra=()):
  return make_model('coco_tracking', extra=['--track_thresh', '0.1', '--new_thresh', '0.1', '--pre_thresh', '0.1',
                                            '--input_h', '128', '--input_w', '160'] + list(extra))


@pytest.mark.parametrize('precision', ['bf16', 'bf16x3'])
@pytest.mark.parametrize('graph', [True, False], ids=['graph', 'eager'])
def test_frames_mode_records_equal_the_fp32_image_runner(precision, graph):
  """device_tracking=False, 5 steps: step_frames on uint8 frames of three sizes vs step_host on the stacked
  pre_process_device images of the same frames -- the same records, bit for bit."""
  from centertrack_b200.runner import StreamRunner
  opt, model, _ = _coco()
  model = model.cuda()
  opt.device = DEV
  det = _host_detector(opt)
  B, H, W = len(SIZES), 128, 160
  kw = dict(K=40, precision=precision, device='cuda', opt=opt, use_graph=graph)
  fr = StreamRunner(model, B, H, W, frame_sizes=SIZES, **kw)
  ref = StreamRunner(model, B, H, W, **kw)
  for r in (fr, ref):
    r.warm()
  want_launches = ref.launches_per_step + (0 if precision == 'bf16' else B)
  assert fr.launches_per_step == want_launches
  assert fr.h2d_bytes_per_step == sum((h * w * 3 + 15) // 16 * 16 for h, w in SIZES) + B * H * W * 4
  for t in range(5):
    frames = [_frame(h, w, 100 * t + b) for b, (h, w) in enumerate(SIZES)]
    fr.step_frames(frames)
    a = fr.fetch()                      # one runner at a time: the two share the engine's activation buffers
    imgs = torch.cat([det.pre_process_device(f, 1.0)[0] for f in frames], 0).cpu()
    ref.step_host(imgs)
    b = ref.fetch()
    assert np.array_equal(a, b), (precision, graph, t)
    for k in range(B):
      assert fr.meta(k)['width'] == SIZES[k][1]


def test_frame_buffers_are_written_in_place():
  """Frames written through frame_buffers() (then step_frames(None)) give the records of passing the arrays, step
  after step: the views always point at the staging of the step about to be submitted."""
  from centertrack_b200.runner import StreamRunner
  opt, model, _ = _coco()
  model = model.cuda()
  B, H, W = len(SIZES), 128, 160
  runners = [StreamRunner(model, B, H, W, K=40, precision='bf16', device='cuda', opt=opt, frame_sizes=SIZES)
             for _ in range(2)]
  for r in runners:
    r.warm()
  outs = [[], []]
  for t in range(7):
    frames = [_frame(h, w, 300 + 10 * t + b) for b, (h, w) in enumerate(SIZES)]
    runners[0].step_frames(frames)
    outs[0].append(runners[0].fetch())
    views = runners[1].frame_buffers()
    assert [v.shape for v in views] == [(h, w, 3) for h, w in SIZES]
    for v, f in zip(views, frames):
      v[...] = f
    runners[1].step_frames(None)
    outs[1].append(runners[1].fetch())
  for t, (a, b) in enumerate(zip(*outs)):
    assert np.array_equal(a, b), t


def test_frames_mode_argument_checks():
  from centertrack_b200.runner import StreamRunner
  opt, model, _ = _coco()
  model = model.cuda()
  B, H, W = len(SIZES), 128, 160
  r = StreamRunner(model, B, H, W, K=40, precision='bf16', device='cuda', opt=opt, frame_sizes=SIZES)
  good = [_frame(h, w, b) for b, (h, w) in enumerate(SIZES)]
  with pytest.raises(ValueError, match='expected 3 arrays'):
    r.step_frames(good[:2])
  with pytest.raises(ValueError, match='uint8'):
    r.step_frames([good[0].astype(np.float32)] + good[1:])
  with pytest.raises(ValueError, match='uint8'):
    r.step_frames([torch.from_numpy(good[0])] + good[1:])
  with pytest.raises(ValueError, match='expected shape'):
    r.step_frames(good[:2] + [good[2][:, :-1]])
  with pytest.raises(ValueError, match='expected shape'):
    r.step_frames(good[:2] + [good[2][..., 0]])
  assert r.t == 0                       # nothing was submitted
  plain = StreamRunner(model, B, H, W, K=40, precision='bf16', device='cuda', opt=opt)
  with pytest.raises(ValueError, match='frame_sizes'):
    plain.step_frames(good)
  with pytest.raises(ValueError, match='frame_sizes'):
    plain.frame_buffers()
  with pytest.raises(ValueError, match='network input'):
    StreamRunner(model, B, 256, 320, K=40, precision='bf16', device='cuda', opt=opt, frame_sizes=SIZES)


# --------------------------------------------------------------------------------------------------- closed loop
def _public_points(rng, dets, h, w):
  """Public detections in source pixels: near some of the frame's detections, and a few anywhere."""
  pts = [np.asarray(d['ct'], np.float32) + rng.normal(0, 1.0, 2).astype(np.float32) for d in dets[::2][:8]]
  pts += [np.float32([rng.uniform(0, w), rng.uniform(0, h)]) for _ in range(3)]
  return np.stack(pts).astype(np.float32)


@pytest.mark.parametrize('cfg,precision,extra', [
    ('coco_tracking', 'fp32', []),
    ('coco_tracking', 'bf16', []),
    ('coco_tracking', 'fp32', ['--public_det', '--hungarian']),
    ('nuscenes_ddd', 'fp32', [])], ids=['fp32', 'bf16', 'public_hungarian', 'nuscenes_ddd'])
def test_frames_mode_closes_the_loop_like_the_host_pipeline(cfg, precision, extra):
  """device_tracking=True, B = 3 streams of different source sizes, --max_age 2: fetch_results() against the host loop
  pre_process_device -> eng.forward -> generic_decode -> generic_post_process (each stream's own meta and default
  calib) -> Tracker, with the host pre_hm render -- tracks, public detections and 3D payload in source pixels."""
  from centertrack_b200.decode import generic_decode
  from centertrack_b200.post_process import generic_post_process
  from centertrack_b200.runner import StreamRunner
  from centertrack_b200.tracker import Tracker
  H, W, K = 128, 160, 30
  opt, model, _ = make_model(cfg, extra=['--track_thresh', '0.1', '--new_thresh', '0.1', '--pre_thresh', '0.1',
                                         '--input_h', str(H), '--input_w', str(W), '--max_age', '2'] + extra)
  if cfg == 'nuscenes_ddd':
    with torch.no_grad():           # boxes of a few pixels (the synthetic weights give ~0 wh)
      model.state_dict()['wh.2.bias'].fill_(3.0)
  model = model.cuda()
  sizes = [(120, 200), (97, 131), (240, 320)]
  B = len(sizes)
  runner = StreamRunner(model, B, H, W, K=K, precision=precision, device='cuda', opt=opt, device_tracking=True,
                        frame_sizes=sizes)
  runner.warm()
  eng = model.engine_for(B, H, W, DEV, precision)
  det = _host_detector(opt)
  metas = [runner.meta(b) for b in range(B)]
  for b, (h, w) in enumerate(sizes):
    assert np.array_equal(metas[b]['calib'], det._get_default_calib(w, h))
  hosts = [Tracker(opt) for _ in range(B)]
  for t in hosts:
    t.init_track([])
  rng = np.random.RandomState(5)
  pre = None
  total = 0
  for t in range(5):
    frames = [_frame(h, w, 500 + 10 * t + b) for b, (h, w) in enumerate(sizes)]
    # host loop
    opt.device = DEV
    x = torch.cat([det.pre_process_device(f, 1.0)[0] for f in frames], 0)
    opt.device = torch.device('cpu')
    hms = [det._get_additional_inputs(hosts[b].tracks, metas[b], with_hm=True)[0] for b in range(B)]
    out = dict(eng.forward(x, x if pre is None else pre, torch.cat(hms, 0).cuda()))
    views = {k: v.cpu().numpy() for k, v in generic_decode(out, K=K).items()}
    dets = []
    for b in range(B):
      m = metas[b]
      one = {k: v[b:b + 1] for k, v in views.items()}
      r = generic_post_process(opt, one, [m['c']], [m['s']], m['out_height'], m['out_width'], opt.num_classes,
                               [m['calib']])[0]
      dets.append([q for q in r if q['score'] > opt.out_thresh])
    pub = [_public_points(rng, dets[b], h, w) for b, (h, w) in enumerate(sizes)] if opt.public_det else None
    runner.step_frames(frames, public_dets=pub)
    got = runner.fetch_results()
    for b in range(B):
      want = hosts[b].step(dets[b], [{'ct': p} for p in pub[b]] if pub is not None else None)
      assert len(got[b]) == len(want), (t, b, len(got[b]), len(want))
      for a, w in zip(got[b], want):
        assert tuple(a[k] for k in EXACT) == tuple(int(w[k]) for k in EXACT), (t, b, a, w)
        for k in ('ct', 'tracking', 'bbox') + tuple(runner.tracker.payload_layout):
          assert np.allclose(np.asarray(a[k], np.float64), np.asarray(w[k], np.float64).reshape(np.shape(a[k])),
                             rtol=1e-4, atol=1e-3), (t, b, k)
        assert abs(a['score'] - float(w['score'])) < 1e-6
      total += len(want)
    pre = x
  assert total > 0 and max(h.id_count for h in hosts) > 0
