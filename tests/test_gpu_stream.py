"""-m gpu: the per-stream device state of SURVEY 8f (device tracker + prior heat-map render, --flip_test, device
pre_process), the graph-captured Detector.process, and --dla_node conv|gcn -- each against the host implementation
that is itself pinned to the reference's goldens, or against the reference goldens directly."""
import copy
import os

import numpy as np
import pytest
import torch

import ct_oracle as co
from centertrack_b200 import _lib as L
from centertrack_b200 import synthetic as wt
from helpers import HOST_CASES, decode_inputs, flip_inputs, host_case_inputs, make_model, make_opt

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')


def _host_detector(opt):
  from centertrack_b200.detector import Detector
  from centertrack_b200.dataset_info import get_dataset
  from centertrack_b200.tracker import Tracker
  det = object.__new__(Detector)
  ds = get_dataset(opt.dataset)
  det.opt, det.cnt, det.pre_images, det.tracker = opt, 0, None, Tracker(opt)
  det.mean = np.array(ds.mean, dtype=np.float32).reshape(1, 1, 3)
  det.std = np.array(ds.std, dtype=np.float32).reshape(1, 1, 3)
  det.rest_focal_length = ds.rest_focal_length
  det.flip_idx = ds.flip_idx
  return det


def _records_from_maps(maps, K):
  from centertrack_b200.decode import generic_decode
  out = {k: torch.from_numpy(v).to(DEV) for k, v in maps.items()}
  return generic_decode(out, K=K)


def _check_tracks(got, want, ctx):
  assert len(got) == len(want), (ctx, len(got), len(want))
  for a, b in zip(got, want):
    assert (a['tracking_id'], a['age'], a['active'], a['class']) == \
        (int(b['tracking_id']), int(b['age']), int(b['active']), int(b['class'])), (ctx, a, b)
    for k in ('ct', 'tracking', 'bbox'):
      assert np.allclose(np.asarray(a[k], np.float64), np.asarray(b[k], np.float64), rtol=1e-4, atol=1e-3), (ctx, k)
    assert abs(a['score'] - float(b['score'])) < 1e-6


def test_device_tracker_matches_reference_golden_three_frames(golden_dir):
  """The 3-frame post_process + Tracker golden of the UNMODIFIED reference (tests/golden/post_track.npz): the device
  tracker must produce the same rows in the same order -- ids, age, active, class exact; ct / tracking / bbox to 1e-4."""
  from centertrack_b200.device_tracker import DeviceTracker
  g = np.load(os.path.join(golden_dir, 'post_track.npz'))
  cfg, kind, C_, H, W = 'coco_tracking', 'coco', 80, 128, 128
  opt = make_opt(cfg, ['--track_thresh', '0.05', '--new_thresh', '0.05'])
  height, width = 480, 640
  c = np.array([width / 2., height / 2.], dtype=np.float32)
  s = max(height, width) * 1.0
  base = decode_inputs(kind, 1, C_, H, W, 100)
  trk = None
  for frame in range(3):
    inp = {k: v.copy() for k, v in base.items()}
    inp['tracking'] = (np.random.RandomState(1000 + frame).randn(*inp['tracking'].shape) * 0.5).astype(np.float32)
    res = _records_from_maps(inp, 100)
    if trk is None:
      trk = DeviceTracker(opt, 1, 100, res.records.shape[2], res.layout, H * 4, W * 4, DEV, centers=[c], scales=[s])
    trk.step(res.records)
    torch.cuda.synchronize()
    got = trk.results(trk.tracks.cpu().numpy(), trk.counts.cpu().numpy())[0]
    n, id_count = g['%s.f%d.n' % (cfg, frame)]
    assert len(got) == n and int(trk.counts[0, 1]) == id_count
    want = [{k: g['%s.f%d.%s' % (cfg, frame, k)][i] for k in ('score', 'class', 'ct', 'tracking', 'bbox', 'tracking_id',
                                                               'age', 'active')} for i in range(n)]
    _check_tracks(got, want, frame)


@pytest.mark.parametrize('seed', range(4))
def test_device_tracker_equals_host_tracker_on_random_streams(seed):
  """Crowded random streams with coasting tracks (--max_age 2 on odd seeds), B = 3 streams at once: device tracker vs
  the host pipeline (views of the same records -> generic_post_process -> Tracker.step), and the prior heat-map the
  device splats for the next frame vs Detector._get_additional_inputs on the host tracker's tracks."""
  from centertrack_b200.decode import views_from_records
  from centertrack_b200.device_tracker import DeviceTracker
  from centertrack_b200.image import get_affine_transform
  from centertrack_b200.post_process import generic_post_process
  from centertrack_b200.tracker import Tracker
  rng = np.random.RandomState(seed)
  max_age = [-1, 2][seed % 2]
  B, K, F = 3, 64, 13
  inp_h, inp_w = 256, 320
  out_h, out_w = inp_h // 4, inp_w // 4
  opt = make_opt('coco_tracking', ['--track_thresh', '0.2', '--new_thresh', '0.3', '--pre_thresh', '0.25', '--max_age',
                                   str(max_age), '--input_h', str(inp_h), '--input_w', str(inp_w)])
  layout = {'wh': (9, 2), 'tracking': (11, 2)}
  img_hw = [(240, 320), (300, 260), (256, 320)]
  centers = [np.array([w / 2., h / 2.], np.float32) for h, w in img_hw]
  scales = [max(h, w) * 1.0 for h, w in img_hw]
  dev_trk = DeviceTracker(opt, B, K, F, layout, inp_h, inp_w, DEV, centers=centers, scales=scales)
  hosts = [Tracker(opt) for _ in range(B)]
  det = _host_detector(opt)
  for t in hosts:
    t.init_track([])
  pre_hm = torch.zeros((B, 1, inp_h, inp_w), device=DEV)
  for frame in range(6):
    rec = np.zeros((B, K, F), np.float32)
    for b in range(B):
      n = 0 if (seed == 3 and frame == 2 and b == 0) else int(rng.randint(1, K))
      sc = np.sort(rng.uniform(0.21, 1.0, n).astype(np.float32))[::-1]
      rec[b, :n, 0] = sc
      rec[b, n:, 0] = np.sort(rng.uniform(0.0, 0.19, K - n).astype(np.float32))[::-1]
      rec[b, :, 1] = rng.randint(0, 3, K)
      rec[b, :, 2] = rng.randint(0, out_w, K)
      rec[b, :, 3] = rng.randint(0, out_h, K)
      wh = rng.uniform(1, 20, (K, 2))
      cx, cy = rec[b, :, 2] + rng.rand(K), rec[b, :, 3] + rng.rand(K)
      rec[b, :, 4], rec[b, :, 5], rec[b, :, 6], rec[b, :, 7] = cx - wh[:, 0] / 2, cy - wh[:, 1] / 2, cx + wh[:, 0] / 2, cy + wh[:, 1] / 2
      rec[b, :, 9:11] = wh
      rec[b, :, 11:13] = rng.normal(0, 2, (K, 2))
    rec_t = torch.from_numpy(rec).to(DEV)
    dev_trk.step(rec_t)
    dev_trk.render(pre_hm)
    torch.cuda.synchronize()
    got = dev_trk.results(dev_trk.tracks.cpu().numpy(), dev_trk.counts.cpu().numpy())
    views = {k: v.numpy() for k, v in views_from_records(torch.from_numpy(rec), layout).items()}
    for b in range(B):
      one = {k: v[b:b + 1] for k, v in views.items()}
      res = generic_post_process(opt, one, [centers[b]], [scales[b]], out_h, out_w, opt.num_classes)[0]
      res = [r for r in res if r['score'] > opt.out_thresh]
      want = hosts[b].step(copy.deepcopy(res))
      _check_tracks(got[b], want, (seed, frame, b))
      assert int(dev_trk.counts[b, 1]) == hosts[b].id_count
      meta = {'inp_width': inp_w, 'inp_height': inp_h, 'out_width': out_w, 'out_height': out_h,
              'trans_input': get_affine_transform(centers[b], scales[b], 0, [inp_w, inp_h]),
              'trans_output': get_affine_transform(centers[b], scales[b], 0, [out_w, out_h])}
      opt.device = torch.device('cpu')
      hm_host, _ = det._get_additional_inputs(hosts[b].tracks, meta, with_hm=True)
      diff = np.abs(pre_hm[b].cpu().numpy() - hm_host.numpy()[0])
      # a box edge that lands within an ulp of an integer may move a radius / centre by one on one of the two sides
      assert (diff > 1e-6).mean() < 2e-3, (seed, frame, b, float(diff.max()), float((diff > 1e-6).mean()))


def test_stream_runner_device_tracking_closes_the_loop_like_the_host_pipeline():
  """StreamRunner(device_tracking=True): pre_hm(t) = splat(tracks(t-1)) -> network + decode -> Tracker.step, all
  inside one CUDA graph per step, against the same loop run step by step through the host tracker and the host
  pre_hm render (fp32 engine, B = 2 streams, 5 frames).  First frame: pre_images = images, empty pre_hm."""
  from centertrack_b200.decode import generic_decode
  from centertrack_b200.image import get_affine_transform
  from centertrack_b200.post_process import generic_post_process
  from centertrack_b200.runner import StreamRunner
  from centertrack_b200.tracker import Tracker
  B, H, W, K = 2, 64, 96, 30
  opt, model, sd = make_model('coco_tracking', extra=['--track_thresh', '0.1', '--new_thresh', '0.1', '--pre_thresh', '0.1',
                                                       '--input_h', str(H), '--input_w', str(W), '--max_age', '2'])
  model = model.cuda()
  runner = StreamRunner(model, B, H, W, K=K, precision='fp32', device='cuda', opt=opt, device_tracking=True)
  runner.warm()
  eng = model.engine_for(B, H, W, DEV, 'fp32')
  det = _host_detector(opt)
  hosts = [Tracker(opt) for _ in range(B)]
  for t in hosts:
    t.init_track([])
  c = np.array([W / 2., H / 2.], np.float32)
  s = max(H, W) * 1.0
  meta = {'inp_width': W, 'inp_height': H, 'out_width': W // 4, 'out_height': H // 4,
          'trans_input': get_affine_transform(c, s, 0, [W, H]), 'trans_output': get_affine_transform(c, s, 0, [W // 4, H // 4])}
  opt.device = torch.device('cpu')
  frames = [wt.synthetic_inputs(B, H, W, seed=60 + t)[0] for t in range(5)]
  pre = None
  for t, img in enumerate(frames):
    runner.step_host(img.pin_memory())
    tracks_np, counts_np = runner.fetch_tracks()
    got = runner.tracker.results(tracks_np, counts_np)
    # host loop
    hms = [det._get_additional_inputs(hosts[b].tracks, meta, with_hm=True)[0] for b in range(B)]
    hm = torch.cat(hms, 0).cuda()
    x = img.cuda()
    out = dict(eng.forward(x, x if pre is None else pre, hm))
    res = generic_decode(out, K=K)
    views = {k: v.cpu().numpy() for k, v in res.items()}
    total = 0
    for b in range(B):
      one = {k: v[b:b + 1] for k, v in views.items()}
      r = generic_post_process(opt, one, [c], [s], H // 4, W // 4, opt.num_classes)[0]
      want = hosts[b].step([q for q in r if q['score'] > opt.out_thresh])
      _check_tracks(got[b], want, (t, b))
      total += len(want)
    assert total > 0
    pre = x
  assert max(h.id_count for h in hosts) > 0


@pytest.mark.parametrize('cfg', ['coco_pose', 'nuscenes_ddd'])
def test_flip_test_process_matches_reference_golden(cfg, golden_dir):
  """--flip_test through Detector.process (batch of frame + mirrored frame, ct_flip_merge, fused decode) against the
  reference's model + _sigmoid_output + _flip_output + generic_decode (fp32 engine, 1e-3 x scale)."""
  from centertrack_b200.detector import Detector
  g = np.load(os.path.join(golden_dir, 'flip_cases.npz'))
  opt, model, sd = make_model(cfg, extra=['--b200_precision', 'fp32', '--flip_test', '--K', '50'])
  det = Detector.__new__(Detector)
  det.opt, det.model = opt, model.cuda()
  img, pre, hm = flip_inputs()
  output, dets = det.process(img.cuda(), pre.cuda(), hm.cuda(), None)
  for h in opt.heads:
    ref = g['%s.head.%s' % (cfg, h)]
    got = output[h].cpu().numpy()
    assert got.shape == ref.shape, (h, got.shape, ref.shape)
    tol = 1e-3 if h != 'dep' else 2e-2
    assert np.abs(got - ref).max() <= tol * max(1.0, np.abs(ref).max()), (h, float(np.abs(got - ref).max()))
  host = {k: v.cpu().numpy() for k, v in output.items() if k != 'pre_inds' and v is not None}
  od = co.generic_decode(host, 50)
  assert np.array_equal((dets['ys'] * 24 + dets['xs']).astype(np.int64), od['_inds'])
  assert np.array_equal(dets['scores'], od['scores']) and np.array_equal(dets['bboxes'], od['bboxes'])
  # the merge itself, bit for bit, on the device's own un-merged maps
  eng = next(iter(det._graphs.values()))['eng']
  raw = {k: v.cpu().numpy() for k, v in eng.outputs.items()}
  from centertrack_b200.dataset_info import get_dataset
  merged = co.flip_output(raw, get_dataset(opt.dataset).flip_idx)
  for h in opt.heads:
    assert np.array_equal(merged[h], output[h].cpu().numpy()), h


@pytest.mark.parametrize('i', range(len(HOST_CASES)), ids=[c[0] for c in HOST_CASES])
def test_device_pre_process_matches_cv2_pre_process(i):
  """ct_warp_affine_normalize (cv2's fixed-point bilinear restated) vs Detector.pre_process (cv2.warpAffine on the
  host, itself pinned to the reference by host_pre.npz): same meta, the same fp32 image bit for bit."""
  name, extra, hw, with_calib = HOST_CASES[i]
  opt = make_opt('coco_tracking', ['--pre_thresh', '0.3'] + extra)
  opt.device = DEV
  det = _host_detector(opt)
  image, tracks, calib = host_case_inputs(i, hw)
  ref_img, ref_meta = det.pre_process(image, 1.0, {'calib': calib} if with_calib else {})
  img, meta = det.pre_process_device(image, 1.0, {'calib': calib} if with_calib else {})
  assert img.is_cuda and img.dtype == torch.float32 and tuple(img.shape) == tuple(ref_img.shape)
  for k in ref_meta:
    assert np.array_equal(np.asarray(meta[k]), np.asarray(ref_meta[k])), k
  bad = img.cpu().numpy().view(np.int32) != ref_img.numpy().view(np.int32)
  assert not bad.any(), (name, int(bad.sum()), np.argwhere(bad)[:4].tolist())


def test_detector_process_graph_replay_equals_eager(monkeypatch):
  """Detector.process as ONE graph replay (the per-image latency path) returns exactly what the eager launches do,
  call after call, including the first-frame (no pre_hm) signature."""
  from centertrack_b200.detector import Detector
  opt, model, sd = make_model('coco_tracking')
  model = model.cuda()
  res = {}
  for mode in ('graph', 'eager'):
    monkeypatch.setenv('CTB_NO_GRAPH', '1' if mode == 'eager' else '0')
    det = Detector.__new__(Detector)
    det.opt, det.model = opt, model
    outs = []
    for seed, with_hm in ((1, True), (2, True), (3, False), (1, True)):
      img, pre, hm = wt.synthetic_inputs(1, 64, 96, seed=seed)
      _, dets = det.process(img.cuda(), pre.cuda(), hm.cuda() if with_hm else None, None)
      outs.append({k: v.copy() for k, v in dets.items()})
    res[mode] = outs
    assert all(np.array_equal(outs[0][k], outs[3][k]) for k in outs[0])
  for a, b in zip(res['graph'], res['eager']):
    assert a.keys() == b.keys() and all(np.array_equal(a[k], b[k]) for k in a)


@pytest.mark.parametrize('node', ['conv', 'gcn'])
def test_dla_node_conv_and_gcn_match_reference_golden(node, golden_dir):
  """--dla_node conv | gcn (dla.py:466-503,588-592): fp32 engine vs the reference golden (1e-3 x scale); bf16 engine vs
  the oracle run with the engine's rounding points."""
  g = np.load(os.path.join(golden_dir, 'net_coco_tracking_%s_64x96.npz' % node))
  opt, model, sd = make_model('coco_tracking', extra=['--dla_node', node])
  model = model.cuda()
  img, pre, hm = wt.synthetic_inputs(1, 64, 96)
  eng = model.engine_for(1, 64, 96, DEV, 'fp32')
  out = eng.forward(img.cuda(), pre.cuda(), hm.cuda())
  torch.cuda.synchronize()
  for h in opt.heads:
    ref = g['head.' + h]
    err = np.abs(out[h].cpu().numpy() - ref)
    assert err.max() <= 1e-3 * max(1.0, np.abs(ref).max()), (h, float(err.max()))
  for k in [x for x in g.files if x.startswith('stage.')]:
    name = k[len('stage.'):]
    ref = g[k]
    got = eng.stage('feat' if name == 'ida_up.node_2' else name).cpu().numpy()
    assert np.abs(got - ref).max() <= 1e-3 * max(1.0, np.abs(ref).max()), name
  emu = co.DLA34Oracle(sd, opt.heads, emulate_bf16=True, dla_node=node).forward(img, pre, hm)
  e16 = model.engine_for(1, 64, 96, DEV, 'bf16')
  o16 = e16.forward(img.cuda(), pre.cuda(), hm.cuda())
  for h in opt.heads:
    r = emu[h].numpy()
    err = np.abs(o16[h].cpu().numpy() - r)
    assert err.mean() <= 5e-2 * max(float(r.std()), 1e-6), (h, float(err.mean()), float(r.std()))
