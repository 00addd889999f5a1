"""-m gpu: --flip_test in StreamRunner -- each stream's frame and its mirror in one batched step of 2B images, merged on
the device.  The kernels against their one-pair / unfused forms bit for bit (ct_flip_merge_heads, ct_mirror_x,
ct_pack_stem_frames_flip_dev); each stream of a flip runner against Detector.process with --flip_test, bit for bit; the
closed loop against the host pipeline; video starts against a fresh flip runner."""
import ctypes as C

import numpy as np
import pytest
import torch

from centertrack_b200 import _lib as L
from centertrack_b200 import synthetic as wt
from helpers import make_model, make_opt
from test_gpu_frames import _frame, _ragged

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')
EXACT = ('tracking_id', 'age', 'active', 'class')
H, W, B, K = 64, 96, 3, 30
SIZES = [(120, 200), (97, 131), (64, 96)]


def _bits(t):
  return t.contiguous().view(torch.int32) if t.dtype == torch.float32 else t.contiguous().view(torch.int16)


def _detector(opt, model, precision):
  """A Detector on `model` (the runner's weights) at `precision`, without the checkpoint loading of __init__."""
  from centertrack_b200.dataset_info import get_dataset
  from centertrack_b200.detector import Detector
  from centertrack_b200.tracker import Tracker
  det = object.__new__(Detector)
  ds = get_dataset(opt.dataset)
  det.opt, det.model, det.cnt, det.pre_images, det.tracker = opt, model, 0, None, Tracker(opt)
  det.mean = np.array(ds.mean, dtype=np.float32).reshape(1, 1, 3)
  det.std = np.array(ds.std, dtype=np.float32).reshape(1, 1, 3)
  det.rest_focal_length = opt.test_focal_length if opt.test_focal_length >= 0 else ds.rest_focal_length
  det.flip_idx = ds.flip_idx
  det._graphs = {}
  model.precision = precision
  return det


def _pair(x):
  """[1,c,h,w] -> the (frame, mirror) pair [2,c,h,w] of detector.py:225-226,285-286."""
  return torch.cat((x, x.flip(3)), 0).contiguous()


# ------------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize('cfg', ['coco_pose', 'nuscenes_ddd'])
@pytest.mark.parametrize('nb', [1, 3])
def test_batched_merge_equals_per_head_per_pair_merge(cfg, nb):
  """ct_flip_merge_heads over every averaged head and nb pairs == ct_flip_merge per head and per pair, bit for bit
  (coco_pose: perm + sign on hps, perm on hm_hp; nuscenes_ddd: sign on amodel_offset)."""
  from centertrack_b200.dataset_info import get_dataset
  from centertrack_b200.detector import flip_output, flip_plan
  opt = make_opt(cfg)
  oh, ow = 13, 17
  g = torch.Generator(device='cuda').manual_seed(5)
  out = {h: torch.randn((2 * nb, c, oh, ow), device=DEV, generator=g) for h, c in opt.heads.items()}
  plan = flip_plan(out, get_dataset(opt.dataset).flip_idx, DEV)
  if cfg == 'coco_pose':
    assert plan['hps'][0] is not None and plan['hps'][1] is not None and plan['hm_hp'][0] is not None
  else:
    assert plan['amodel_offset'][1] is not None
  merged = {h: torch.full((nb,) + tuple(out[h].shape[1:]), 7.0, device=DEV) for h in plan}
  lib = L.lib()
  n0 = lib.ct_launch_count()
  res = flip_output(out, plan, merged)
  assert lib.ct_launch_count() - n0 == 1                     # one launch for every head of every pair
  torch.cuda.synchronize()
  for h, t in out.items():
    if h not in plan:
      assert res[h].data_ptr() == t.data_ptr() and res[h].shape[0] == nb
      continue
    perm, sign = plan[h]
    for b in range(nb):
      in2 = torch.stack((t[b], t[nb + b])).contiguous()
      one = torch.empty((1,) + tuple(t.shape[1:]), device=DEV)
      L.check(lib.ct_flip_merge(L.ptr(in2), L.ptr(one), t.shape[1], oh, ow, L.ptr(perm), L.ptr(sign), L.stream_ptr()))
      torch.cuda.synchronize()
      assert torch.equal(_bits(one[0]), _bits(merged[h][b])), (h, b)


@pytest.mark.parametrize('n', [1, 3])
def test_mirror_x_equals_torch_flip(n):
  """ct_mirror_x into the second half of a 2B buffer (odd W) == torch.flip(x, [3]); nothing else is written."""
  Bn, c, h, w = 3, 3, 11, 37
  x = torch.randn((2 * Bn, c, h, w), device=DEV)
  before = x.clone()
  b = 1 if n == 1 else 0
  L.check(L.lib().ct_mirror_x(L.ptr(x[b]), L.ptr(x[Bn + b]), n, c, h, w, L.stream_ptr()))
  torch.cuda.synchronize()
  assert torch.equal(_bits(x[Bn + b:Bn + b + n]), _bits(torch.flip(before[b:b + n], [3])))
  keep = torch.ones(2 * Bn, dtype=torch.bool)
  keep[Bn + b:Bn + b + n] = False
  assert torch.equal(_bits(x[keep]), _bits(before[keep]))


def _pack_flip_check(opt, cur, prev, frames, nb, hh, ww, hm):
  from centertrack_b200.dataset_info import get_dataset
  ds = get_dataset(opt.dataset)
  mean = np.ascontiguousarray(ds.mean, np.float32).reshape(3)
  std = np.ascontiguousarray(ds.std, np.float32).reshape(3)
  ms = C.c_void_p(mean.ctypes.data), C.c_void_p(std.ctypes.data)
  lib, st = L.lib(), L.stream_ptr()
  fdev = torch.frombuffer(bytearray(bytes(frames)), dtype=torch.uint8).to(DEV)
  args = L.ptr(fdev), nb, cur.numel()
  for name, pv, h in (('first', cur, hm), ('no_prev', None, hm), ('no_hm', prev, None), ('both', prev, hm)):
    ref = torch.full((nb, hh, ww, 8), 7.0, dtype=torch.bfloat16, device=DEV)
    got = torch.full((2 * nb, hh, ww, 8), -7.0, dtype=torch.bfloat16, device=DEV)
    L.check(lib.ct_pack_stem_frames_dev(L.ptr(cur), L.ptr(pv), *args, *ms, L.ptr(h), L.ptr(ref), hh, ww, st))
    L.check(lib.ct_pack_stem_frames_flip_dev(L.ptr(cur), L.ptr(pv), *args, *ms, L.ptr(h), L.ptr(got), hh, ww, st))
    torch.cuda.synchronize()
    want = torch.cat((ref, ref.flip(2)), 0)
    eq = _bits(got) == _bits(want)
    assert bool(eq.all()), (name, int((~eq).sum()), [int((~eq[b]).sum()) for b in range(2 * nb)])


@pytest.mark.parametrize('out_hw', [(544, 960), (384, 1280)])
def test_dev_flip_pack_equals_dev_pack_then_mirror_byte_for_byte(out_hw):
  """ct_pack_stem_frames_flip_dev == ct_pack_stem_frames_dev followed by a flip of each packed [H, W, 8] image along
  W, on the ragged streams of the unfused-pack test (odd width, padded pitch), with and without prev / pre_hm."""
  hh, ww = out_hw
  opt = make_opt('mot', ['--input_h', str(hh), '--input_w', str(ww)])
  streams = [(1080, 1920, 5760), (480, 640, 1920), (375, 1242, 3726), (544, 960, 2880), (301, 457, 1392)]
  cur, prev, frames, _ = _ragged(opt, streams, 11)
  hm = torch.rand((len(streams), 1, hh, ww), device=DEV)
  _pack_flip_check(opt, cur, prev, frames, len(streams), hh, ww, hm)


def test_flip_pack_of_many_streams():
  """B = 53 streams of small ragged frames, odd output width."""
  hh, ww = 48, 77
  opt = make_opt('mot', ['--input_h', str(hh), '--input_w', str(ww)])
  nb = 53
  streams = [((40, 66, 198), (31, 57, 176), (48, 77, 231))[b % 3] for b in range(nb)]
  cur, prev, frames, _ = _ragged(opt, streams, 23)
  hm = torch.rand((nb, 1, hh, ww), device=DEV)
  _pack_flip_check(opt, cur, prev, frames, nb, hh, ww, hm)


# ------------------------------------------------------------------------------------- runner == Detector
def _model(cfg, extra=()):
  opt, model, _ = make_model(cfg, extra=['--track_thresh', '0.1', '--new_thresh', '0.1', '--pre_thresh', '0.1',
                                         '--input_h', str(H), '--input_w', str(W), '--max_age', '2', '--K', str(K),
                                         '--flip_test'] + list(extra))
  if cfg == 'nuscenes_ddd':
    with torch.no_grad():            # boxes of a few pixels (the synthetic weights give ~0 wh)
      model.state_dict()['wh.2.bias'].fill_(3.0)
  opt.device = DEV
  return opt, model.cuda()


RUNNER_CASES = [('coco_tracking', p, m, True) for p in ('fp32', 'bf16x3', 'bf16') for m in ('images', 'frames')] + \
    [('coco_tracking', 'bf16', 'frames', False), ('coco_tracking', 'fp32', 'images', False),
     ('coco_tracking', 'bf16x3', 'frames', False),
     ('coco_pose', 'bf16', 'frames', True), ('coco_pose', 'fp32', 'images', True),
     ('nuscenes_ddd', 'bf16', 'frames', True), ('nuscenes_ddd', 'bf16x3', 'images', False)]


@pytest.mark.parametrize('cfg,precision,mode,graph', RUNNER_CASES,
                         ids=['%s-%s-%s-%s' % (c, p, m, 'graph' if g else 'eager') for c, p, m, g in RUNNER_CASES])
def test_flip_runner_equals_detector_per_stream_bit_for_bit(cfg, precision, mode, graph):
  """B = 3 streams on different inputs, 3 steps, caller-given pre_hm: each stream's records and merged head maps equal
  Detector.process with --flip_test on that stream's (image, pre_image, pre_hm), bit for bit.  In frames mode the
  Detector takes pre_process_device's images of the stream's frame."""
  from centertrack_b200.runner import StreamRunner
  frames_mode = mode == 'frames'
  opt, model = _model(cfg)
  r = StreamRunner(model, B, H, W, K=K, precision=precision, device='cuda', opt=opt, use_graph=graph,
                   frame_sizes=SIZES if frames_mode else None)
  r.warm()
  assert r.flip and r.eng.B == 2 * B and sorted(r.merged) == sorted(r.flip_plan)
  plain_bytes = (sum((h * w * 3 + 15) // 16 * 16 for h, w in SIZES) if frames_mode else B * 3 * H * W * 4) + B * H * W * 4
  assert r.h2d_bytes_per_step == plain_bytes                 # only the B frames (and pre_hm) are uploaded
  det = _detector(opt, model, precision)
  prev = None
  for t in range(3):
    if frames_mode:
      frames = [_frame(h, w, 100 * t + 7 * b) for b, (h, w) in enumerate(SIZES)]
      imgs = [det.pre_process_device(f, 1.0)[0] for f in frames]          # already (frame, mirror) pairs
    else:
      x = torch.stack([wt.synthetic_inputs(1, H, W, seed=40 * t + b)[0][0] for b in range(B)])
      imgs = [_pair(x[b:b + 1].to(DEV)) for b in range(B)]
    hm = torch.stack([wt.synthetic_inputs(1, H, W, seed=900 + 40 * t + b, n_blobs=8)[2][0] for b in range(B)])
    if frames_mode:
      r.step_frames(frames, pre_hms=hm)
    else:
      r.step_host(x, pre_hms=hm)
    rec = r.fetch()
    merged = {h: v.clone() for h, v in r.merged.items()}
    for b in range(B):
      pre = imgs[b] if prev is None else prev[b]
      output, _ = det.process(imgs[b], pre, _pair(hm[b:b + 1].to(DEV)), None)
      (p,) = det._graphs.values()                           # one input signature: one plan
      want = p['rec'].cpu()
      assert torch.equal(_bits(want[0]), _bits(torch.from_numpy(rec[b]))), (t, b)
      for h in merged:
        assert torch.equal(_bits(output[h][0]), _bits(merged[h][b])), (t, b, h)
    prev = imgs


# ------------------------------------------------------------------------------------------------ closed loop
@pytest.mark.parametrize('cfg,extra', [('coco_tracking', []), ('coco_tracking', ['--public_det', '--hungarian']),
                                       ('nuscenes_ddd', [])], ids=['greedy', 'public_hungarian', 'nuscenes_ddd'])
def test_flip_closed_loop_matches_the_host_pipeline(cfg, extra):
  """device_tracking=True, --flip_test, 7 steps, B = 3 crowded synthetic streams (fp32 engine): fetch_results() per
  stream against Detector.process (flip pair, host-rendered flipped pre_hm) -> generic_post_process -> Tracker."""
  from centertrack_b200.image import get_affine_transform
  from centertrack_b200.post_process import generic_post_process
  from centertrack_b200.runner import StreamRunner
  from centertrack_b200.tracker import Tracker
  opt, model = _model(cfg, extra)
  if opt.public_det:
    with torch.no_grad():            # boxes of a few pixels, so that a public detection can claim a detection
      model.state_dict()['wh.2.bias'].fill_(3.0)
  runner = StreamRunner(model, B, H, W, K=K, precision='fp32', device='cuda', opt=opt, device_tracking=True)
  runner.warm()
  det = _detector(opt, model, 'fp32')
  c = np.array([W / 2., H / 2.], np.float32)
  s = max(H, W) * 1.0
  meta = {'c': c, 's': s, 'inp_width': W, 'inp_height': H, 'out_width': W // 4, 'out_height': H // 4,
          'trans_input': get_affine_transform(c, s, 0, [W, H]),
          'trans_output': get_affine_transform(c, s, 0, [W // 4, H // 4]),
          'calib': runner.tracker.calib[0].cpu().numpy() if runner.tracker.calib is not None else None}
  hosts = [Tracker(opt) for _ in range(B)]
  for h in hosts:
    h.init_track([])
  rng = np.random.RandomState(9)
  prev = None
  total = 0
  for t in range(7):
    x = torch.stack([wt.synthetic_inputs(1, H, W, seed=700 + 13 * t + b, n_blobs=40)[0][0] for b in range(B)])
    dets = []
    for b in range(B):
      img = _pair(x[b:b + 1].to(DEV))
      hm, _ = det._get_additional_inputs(hosts[b].tracks, meta, with_hm=True)      # [2,1,H,W]: flipped by the host
      _, d = det.process(img, img if prev is None else prev[b], hm, None)
      kw = {'calibs': [meta['calib']]} if meta['calib'] is not None else {}
      res = generic_post_process(opt, d, [c], [s], H // 4, W // 4, opt.num_classes, **kw)[0]
      dets.append([q for q in res if q['score'] > opt.out_thresh])
    pub = None
    if opt.public_det:
      pub = []
      for b in range(B):
        pts = [np.asarray(q['ct'], np.float32) + np.asarray(q['tracking'], np.float32) +    # near the predicted centre
               rng.normal(0, 0.2, 2).astype(np.float32) for q in dets[b][::2][:8]]
        pts += [np.float32([rng.uniform(0, W), rng.uniform(0, H)]) for _ in range(3)]
        pub.append(np.stack(pts).astype(np.float32))
    runner.step_host(x, public_dets=pub)
    got = runner.fetch_results()
    for b in range(B):
      want = hosts[b].step(dets[b], [{'ct': q} for q in pub[b]] if pub is not None else None)
      assert len(got[b]) == len(want), (t, b, len(got[b]), len(want))
      for a, w in zip(got[b], want):
        assert tuple(a[k] for k in EXACT) == tuple(int(w[k]) for k in EXACT), (t, b, a, w)
        for k in ('ct', 'tracking', 'bbox'):
          assert np.allclose(np.asarray(a[k], np.float64), np.asarray(w[k], np.float64), rtol=1e-4, atol=1e-4), (t, b, k)
        for k in runner.tracker.payload_layout:
          assert np.allclose(np.asarray(a[k], np.float64), np.asarray(w[k], np.float64).reshape(np.shape(a[k])),
                             rtol=1e-4, atol=1e-3), (t, b, k)
        assert abs(a['score'] - float(w['score'])) < 1e-6
      total += len(want)
    prev = [_pair(x[b:b + 1].to(DEV)) for b in range(B)]
  assert total > 0 and max(h.id_count for h in hosts) > 0


# ------------------------------------------------------------------------------------------------ video starts
@pytest.mark.parametrize('precision,mode', [('fp32', 'images'), ('bf16', 'frames'), ('bf16x3', 'frames')])
def test_flip_started_stream_equals_a_fresh_flip_runner(precision, mode):
  """With --flip_test, each started video's records, track table and counts equal a fresh flip runner playing it from
  t = 0, bit for bit, the unstarted streams equal a runner without starts, and no slot's graph is recaptured."""
  import test_gpu_stream_starts as ss
  frames_mode = mode == 'frames'
  opt, model = ss._model('coco_tracking', ['--flip_test'])
  keys, feed, videos = ss._schedule(frames_mode, True)
  r = ss._runner(model, opt, precision, frames_mode)
  assert r.flip
  got = ss._play(r, feed, frames_mode, [id(g) for g in r.graphs])
  del r
  plain = ss._runner(model, opt, precision, frames_mode)
  base = ss._play(plain, [(x, None, None) for x, _, _ in feed], frames_mode)
  del plain
  first = {b: min([t for t, s in ss.STARTS.items() if b in s]) for b in range(ss.B)}
  for t in range(ss.STEPS):
    for b in range(ss.B):
      if t < first[b]:
        ss._same(got[t], base[t], b, b, ('unstarted', t, b))
  assert sum(int(got[t]['cnt'][b, 0]) for t in range(ss.STEPS) for b in range(ss.B)) > 0
  for b, t0, n in videos:
    fresh = ss._runner(model, opt, precision, frames_mode)
    pre = feed[t0][2]
    pre = {b: pre[b]} if pre and b in pre else None
    vfeed = []
    for i in range(n):
      xs = [ss._inputs(frames_mode, q, keys[t0 + i][q]) for q in range(ss.B)]
      vfeed.append((ss._stack(frames_mode, xs), [b] if (i == 0 and pre) else None, pre if i == 0 else None))
    want = ss._play(fresh, vfeed, frames_mode)
    del fresh
    for i in range(n):
      ss._same(got[t0 + i], want[i], b, b, ('video', b, t0, i))
