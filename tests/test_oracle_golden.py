"""The oracle (oracle/ct_oracle.py) is pinned against outputs of the UNMODIFIED reference run in the
build container (fixtures in tests/golden/, generator oracle/gen_golden.py).  CPU only.

Tolerances: network = 1e-3 absolute (north_star's fp32 bar; observed ~3e-4, two fp32 summation
orders); decode / top-K indices = bit-exact; post-process / tracker = 1e-4 relative (float32 affine
arithmetic evaluated in a different association order)."""
import os

import numpy as np
import pytest
import torch

import ct_oracle as co
from centertrack_b200 import synthetic as wt
from helpers import DECODE_CASES, HOST_CASES, decode_inputs, host_case_inputs, load_generic_golden, make_opt, make_model


@pytest.mark.parametrize('cfg', ['coco_tracking', 'mot', 'nuscenes_ddd', 'coco_pose', 'coco_tracking_conv',
                                 'coco_tracking_gcn'])
def test_oracle_network_matches_reference_golden(cfg, golden_dir):
  g = np.load(os.path.join(golden_dir, 'net_%s_64x96.npz' % cfg))
  node = cfg.rsplit('_', 1)[1] if cfg.endswith(('_conv', '_gcn')) else 'dcn'       # --dla_node (dla.py:588-592)
  opt, model, sd = make_model(cfg[:-len(node) - 1] if node != 'dcn' else cfg, extra=['--dla_node', node])
  assert sorted(sd.keys()) == list(g['keys'])          # state-dict key compatibility
  img, pre, hm = wt.synthetic_inputs(1, 64, 96)
  trace = {}
  out = co.DLA34Oracle(sd, opt.heads, dla_node=node).forward(img, pre, hm, trace=trace)
  for k in out:
    ref = g['head.' + k]
    assert out[k].shape == ref.shape
    assert np.abs(out[k].numpy() - ref).max() < 1e-3, k
  for k in [x for x in g.files if x.startswith('stage.')]:
    name = k[len('stage.'):]
    key = 'feat' if name == 'ida_up.node_2' else name
    assert np.abs(trace[key].numpy() - g[k]).max() < 1e-3 * max(1.0, np.abs(g[k]).max()), name


@pytest.mark.parametrize('case', range(len(DECODE_CASES)))
def test_oracle_decode_matches_reference_golden(case, golden_dir):
  g = np.load(os.path.join(golden_dir, 'decode_cases.npz'))
  kind, B, C, H, W, K, seed = DECODE_CASES[case]
  inp = decode_inputs(kind, B, C, H, W, seed)
  out = co.generic_decode(inp, K)
  keys = [k.split('.', 1)[1] for k in g.files if k.startswith('%d.' % case)]
  assert sorted(keys) == sorted(k for k in out if not k.startswith('_'))
  for k in keys:
    ref = g['%d.%s' % (case, k)]
    got = out[k].reshape(ref.shape)
    if k in ('hps', 'kps_score'):
      assert np.abs(got - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max()), k
    else:
      assert np.array_equal(got, ref), k          # bit-exact (tie-free seeded inputs)
  # the flat indices are consistent with xs/ys
  assert np.array_equal(out['_inds'], (out['ys'] * W + out['xs']).astype(np.int64))


def _run_post_track(cfg, kind, C, H, W, ci, post_fn, tracker):
  height, width = 480, 640
  c = np.array([width / 2., height / 2.], dtype=np.float32)
  s = max(height, width) * 1.0
  calib = np.array([[1200, 0, width / 2, 0], [0, 1200, height / 2, 0], [0, 0, 1, 0]], dtype=np.float32)
  base = decode_inputs(kind, 1, C, H, W, 100 + ci)
  frames = []
  for frame in range(3):
    inp = {k: v.copy() for k, v in base.items()}
    rng = np.random.RandomState(1000 + frame)
    inp['tracking'] = (rng.randn(*inp['tracking'].shape) * 0.5).astype(np.float32)
    if 'dep' in inp:
      inp['dep'] = (1. / (1. / (1 + np.exp(-inp['dep'] / 30 + 1)) + 1e-6) - 1.).astype(np.float32)
    dets = co.generic_decode(inp, 100)
    dets = {k: v for k, v in dets.items() if not k.startswith('_')}
    res = post_fn(dets, c, s, H, W, calib, height, width)
    res = [r for r in res if r['score'] > 0.05]
    if frame == 0:
      tracker.init_track([])
    frames.append((tracker.step(res), tracker.id_count))
  return frames


CASES = [('coco_tracking', 'coco', 80, 128, 128), ('nuscenes_ddd', 'ddd', 10, 112, 200),
         ('coco_pose', 'pose', 1, 128, 128)]


def _check_frames(cfg, frames, g):
  for f, (out, id_count) in enumerate(frames):
    n = g['%s.f%d.n' % (cfg, f)]
    assert [len(out), id_count] == list(n)
    for key in out[0].keys():
      ref = g['%s.f%d.%s' % (cfg, f, key)]
      got = np.array([np.asarray(o[key], dtype=np.float64) for o in out])
      if key in ('tracking_id', 'age', 'active', 'class'):
        assert np.array_equal(got, ref), (cfg, f, key)
      else:
        assert np.allclose(got, ref, rtol=1e-4, atol=1e-3), (cfg, f, key, np.abs(got - ref).max())


@pytest.mark.parametrize('ci', range(3))
def test_oracle_post_process_and_tracker_match_reference_golden(ci, golden_dir):
  g = np.load(os.path.join(golden_dir, 'post_track.npz'))
  cfg, kind, C, H, W = CASES[ci]
  post = lambda d, c, s, h, w, calib, height, width: co.generic_post_process(d, [c], [s], h, w, 0.05, [calib])[0]
  frames = _run_post_track(cfg, kind, C, H, W, ci, post, co.TrackerOracle(0.05))
  _check_frames(cfg, frames, g)


@pytest.mark.parametrize('ci', range(3))
def test_product_host_post_process_and_tracker_match_reference_golden(ci, golden_dir):
  """centertrack_b200.post_process / tracker are host (numpy) code of the product path."""
  from centertrack_b200.post_process import generic_post_process
  from centertrack_b200.tracker import Tracker
  g = np.load(os.path.join(golden_dir, 'post_track.npz'))
  cfg, kind, C, H, W = CASES[ci]
  opt = make_opt(cfg, ['--track_thresh', '0.05', '--new_thresh', '0.05'])
  post = lambda d, c, s, h, w, calib, height, width: generic_post_process(
      opt, d, [c], [s], h, w, opt.num_classes, [calib], height, width)[0]
  frames = _run_post_track(cfg, kind, C, H, W, ci, post, Tracker(opt))
  _check_frames(cfg, frames, g)


def test_oracle_dcn_matches_torchvision():
  """Second, independent anchor for the un-vendored DCNv2 arithmetic (SURVEY Appendix B)."""
  tv = pytest.importorskip('torchvision.ops')
  g = torch.Generator().manual_seed(5)
  x = torch.randn(2, 16, 9, 11, generator=g)
  w = torch.randn(8, 16, 3, 3, generator=g) * 0.1
  b = torch.randn(8, generator=g)
  wo = torch.randn(27, 16, 3, 3, generator=g) * 0.05      # offsets up to a few pixels, some out of image
  bo = torch.randn(27, generator=g) * 1.5
  got = co.dcn_v2_forward(x, w, b, wo, bo)
  om = torch.nn.functional.conv2d(x, wo, bo, 1, 1)
  ref = tv.deform_conv2d(x, om[:, :18], w, b, 1, 1, 1, torch.sigmoid(om[:, 18:]))
  assert (got - ref).abs().max() < 1e-4


@pytest.mark.parametrize('cfg', ['coco_pose', 'nuscenes_ddd'])
def test_oracle_flip_test_matches_reference_golden(cfg, golden_dir):
  """--flip_test: oracle network on the (frame, mirrored frame) pair + sigmoid_output + flip_output + decode vs the
  reference's model + _sigmoid_output + _flip_output + generic_decode (detector.py:311-332)."""
  from helpers import flip_inputs
  from centertrack_b200.dataset_info import get_dataset
  g = np.load(os.path.join(golden_dir, 'flip_cases.npz'))
  opt, model, sd = make_model(cfg)
  img, pre, hm = flip_inputs()
  out = co.sigmoid_output(co.DLA34Oracle(sd, opt.heads).forward(img, pre, hm))
  merged = co.flip_output(out, get_dataset(opt.dataset).flip_idx)
  for h in opt.heads:
    ref = g['%s.head.%s' % (cfg, h)]
    assert merged[h].shape == ref.shape
    tol = 1e-3 if h != 'dep' else 2e-2
    assert np.abs(merged[h] - ref).max() <= tol * max(1.0, np.abs(ref).max()), h
  # decode of the reference's own merged maps: bit-exact indices
  od = co.generic_decode({h: g['%s.head.%s' % (cfg, h)] for h in opt.heads}, 50)
  pos = g[cfg + '.det.scores'][0] > 0          # fewer than K positive peaks on this tiny map: zero-score ties (hazard H1)
  assert pos.sum() >= 10
  assert np.array_equal(od['_inds'][0][pos], (g[cfg + '.det.ys'] * 24 + g[cfg + '.det.xs']).astype(np.int64)[0][pos])
  assert np.array_equal(od['scores'], g[cfg + '.det.scores'])


def test_oracle_topk_tie_rule():
  v = np.array([[0.5, 0.0, 0.5, 0.7, 0.0, 0.0]], dtype=np.float32)
  s, i = co.topk_desc(v, 4)
  assert list(i[0]) == [3, 0, 2, 1] and list(s[0]) == [0.7, 0.5, 0.5, 0.0]


@pytest.mark.parametrize('i', range(len(HOST_CASES)), ids=[c[0] for c in HOST_CASES])
def test_product_host_pre_process_and_pre_hm_match_reference_golden(i, golden_dir):
  """Detector.pre_process / _transform_scale / _get_additional_inputs (host numpy + cv2; rows a17, a18) against the
  unmodified reference's outputs: every resolution mode (fix_res, keep_res, fix_short), calib given or default,
  tracks that are inactive / below pre_thresh / degenerate / partly outside the image."""
  from centertrack_b200.detector import Detector
  from centertrack_b200.dataset_info import get_dataset
  g = np.load(os.path.join(golden_dir, 'host_pre.npz'))
  name, extra, hw, with_calib = HOST_CASES[i]
  opt = make_opt('coco_tracking', ['--pre_thresh', '0.3'] + extra)
  opt.device = torch.device('cpu')
  det = object.__new__(Detector)              # host methods only: no model, no device
  ds = get_dataset(opt.dataset)
  det.opt = opt
  det.mean = np.array(ds.mean, dtype=np.float32).reshape(1, 1, 3)
  det.std = np.array(ds.std, dtype=np.float32).reshape(1, 1, 3)
  det.rest_focal_length = ds.rest_focal_length
  image, tracks, calib = host_case_inputs(i, hw)
  images, meta = det.pre_process(image, 1.0, {'calib': calib} if with_calib else {})
  # the affine matrices come from a closed-form solve here and from cv2.getAffineTransform in the reference:
  # equal to ~1e-16; the warped image may differ by an interpolation rounding on isolated pixels
  assert images.dtype == torch.float32 and images.shape == g[name + '.images'].shape
  err = np.abs(images.numpy() - g[name + '.images'])
  assert err.max() <= 2e-2 and (err > 1e-5).mean() < 1e-3, (err.max(), (err > 1e-5).mean())
  for k in ('c', 's', 'calib', 'trans_input', 'trans_output'):
    assert np.allclose(np.asarray(meta[k], dtype=np.float64), g[name + '.meta.' + k], rtol=0, atol=1e-9), k
  ints = [meta[k] for k in ('height', 'width', 'out_height', 'out_width', 'inp_height', 'inp_width')]
  assert np.array_equal(np.array(ints, dtype=np.int64), g[name + '.meta.ints'])
  hm, inds = det._get_additional_inputs(tracks, meta, with_hm=True)
  assert tuple(hm.shape) == g[name + '.pre_hm'].shape and np.array_equal(hm.numpy(), g[name + '.pre_hm'])
  assert inds.dtype == torch.int64 and np.array_equal(inds.numpy(), g[name + '.pre_inds'])


def test_detector_run_host_control_flow_with_stubbed_device_path(monkeypatch):
  """Detector.run's host orchestration (input kinds, first-frame tracker initialisation, pre_hm render, post_process,
  tracker step, the reference's return dict) with `process` -- the only method that touches the GPU -- replaced by a
  stub that decodes synthetic maps with the oracle.  Compared step by step with the same pipeline assembled by hand."""
  import time
  from centertrack_b200.detector import Detector
  from centertrack_b200.dataset_info import get_dataset
  from centertrack_b200.tracker import Tracker
  opt = make_opt('coco_tracking', ['--input_h', '128', '--input_w', '160', '--track_thresh', '0.05',
                                   '--new_thresh', '0.05', '--pre_thresh', '0.05'])
  opt.device = torch.device('cpu')
  det = object.__new__(Detector)
  ds = get_dataset(opt.dataset)
  det.opt, det.cnt, det.pre_images, det.tracker = opt, 0, None, Tracker(opt)
  det.mean = np.array(ds.mean, dtype=np.float32).reshape(1, 1, 3)
  det.std = np.array(ds.std, dtype=np.float32).reshape(1, 1, 3)
  det.rest_focal_length = ds.rest_focal_length
  monkeypatch.setattr(torch.cuda, 'synchronize', lambda *a, **k: None)
  seen = []

  def fake_process(images, pre_images=None, pre_hms=None, pre_inds=None, return_time=False):
    seen.append((tuple(images.shape), pre_images is not None, None if pre_hms is None else float(pre_hms.max()),
                 None if pre_inds is None else int(pre_inds.numel())))
    maps = decode_inputs('coco', 1, 80, 32, 40, 500 + len(seen))
    dets = {k: v for k, v in co.generic_decode(maps, 100).items() if not k.startswith('_')}
    return {}, dets, time.time()

  det.process = fake_process
  rng = np.random.RandomState(5)
  ref_tracker = Tracker(opt)
  ref_tracker.init_track([])
  for f in range(3):
    frame = rng.randint(0, 255, (120, 160, 3)).astype(np.uint8)
    ret = det.run(frame)
    assert set(ret) == {'results', 'tot', 'load', 'pre', 'net', 'dec', 'post', 'merge', 'track', 'display'}
    assert all(ret[k] >= 0 for k in ret if k != 'results') and ret['tot'] >= ret['net']
    # the same step by hand
    _, meta = det.pre_process(frame, 1.0)
    maps = decode_inputs('coco', 1, 80, 32, 40, 500 + f + 1)
    dets = {k: v for k, v in co.generic_decode(maps, 100).items() if not k.startswith('_')}
    want = ref_tracker.step(det.merge_outputs([det.post_process(dets, meta, 1.0)]))
    got = ret['results']
    assert len(got) == len(want) > 0
    for a, b in zip(got, want):
      assert a['tracking_id'] == b['tracking_id'] and a['class'] == b['class'] and a['active'] == b['active']
      assert np.array_equal(np.asarray(a['bbox']), np.asarray(b['bbox']))
    # device-path arguments: first frame is its own pre_image; pre_hm is empty until tracks exist
    shape, has_pre, hm_max, n_inds = seen[f]
    assert shape == (1, 3, 128, 160) and has_pre
    assert (hm_max == 0.0 and n_inds == 0) if f == 0 else (hm_max > 0.5 and n_inds > 0)
  assert det.cnt == 3 and det.tracker.id_count == ref_tracker.id_count


def test_product_opts_derive_the_same_fields_as_the_reference(golden_dir):
  """centertrack_b200.opts vs the reference's opts().init() on seven command lines (tests/golden/opts_cases.json):
  heads (names, channels AND order), head_conv, resolutions, thresholds, tracking switches."""
  import json
  from centertrack_b200.opts import opts
  g = json.load(open(os.path.join(golden_dir, 'opts_cases.json')))
  for argv, want in zip(g['cases'], g['fields']):
    opt = opts().init(argv + ['--gpus', '-1'])
    for k, v in want.items():
      got = getattr(opt, k)
      if isinstance(got, dict):
        got = [[n, c] for n, c in got.items()]
      assert got == v, (argv, k, got, v)


@pytest.mark.parametrize('seed', range(8))
def test_product_tracker_equals_oracle_on_random_streams(seed):
  """Randomised streams (crowded scenes, class changes, empty frames, tracks that coast with --max_age) through
  centertrack_b200.tracker.Tracker and the oracle restatement (itself pinned to the reference by post_track.npz)."""
  import copy
  from centertrack_b200.tracker import Tracker
  rng = np.random.RandomState(seed)
  max_age = [-1, 2][seed % 2]
  opt = make_opt('coco_tracking', ['--track_thresh', '0.2', '--new_thresh', '0.3', '--max_age', str(max_age)])
  prod, orc = Tracker(opt), co.TrackerOracle(opt.new_thresh, max_age)
  first = True
  for frame in range(6):
    n = 0 if (seed == 3 and frame == 2) else int(rng.randint(1, 40))
    dets = []
    for _ in range(n):
      ct = rng.uniform(0, 200, 2)
      wh = rng.uniform(2, 60, 2)
      dets.append({'score': float(rng.uniform(0.2, 1.0)), 'class': int(rng.randint(1, 4)),
                   'ct': ct.astype(np.float32), 'tracking': rng.normal(0, 6, 2).astype(np.float32),
                   'bbox': np.array([ct[0] - wh[0] / 2, ct[1] - wh[1] / 2, ct[0] + wh[0] / 2, ct[1] + wh[1] / 2],
                                    np.float32)})
    dets.sort(key=lambda d: -d['score'])
    a, b = copy.deepcopy(dets), copy.deepcopy(dets)
    if first:
      prod.init_track([]); orc.init_track([])
      first = False
    ra, rb = prod.step(a), orc.step(b)
    assert len(ra) == len(rb) and prod.id_count == orc.id_count
    for x, y in zip(ra, rb):
      assert (x['tracking_id'], x['age'], x['active'], x['class']) == (y['tracking_id'], y['age'], y['active'], y['class'])
      assert np.array_equal(x['bbox'], y['bbox'])


TRACK_MODES = [('greedy_age2', ['--max_age', '2']), ('hungarian', ['--hungarian']),
               ('hungarian_age2', ['--hungarian', '--max_age', '2']), ('public', ['--public_det']),
               ('public_hungarian_age2', ['--public_det', '--hungarian', '--max_age', '2'])]


def _track_rows(out):
  return np.array([[o['tracking_id'], o['age'], o['active'], o['class'], o['score']] + list(map(float, o['bbox']))
                   for o in out], np.float64).reshape(-1, 9)


@pytest.mark.parametrize('mode', range(len(TRACK_MODES)))
@pytest.mark.parametrize('which', ['oracle', 'product'])
def test_tracker_modes_match_reference_golden(mode, which, golden_dir):
  """--hungarian, --public_det and --max_age coasting (tracker.py:52-72,83-103,105-120) on crowded seeded streams:
  every returned row (id, age, active, class, score, bbox -- in the reference's output order) equals what the
  reference's Tracker produced (tests/golden/track_modes.npz, oracle/gen_golden.py::gen_track_modes; sklearn's removed
  linear_assignment is stood in for by scipy there and here)."""
  import copy
  from centertrack_b200.tracker import Tracker
  g = np.load(os.path.join(golden_dir, 'track_modes.npz'))
  name, extra = TRACK_MODES[mode]
  seen = {'rejected': 0, 'coast': 0, 'born': 0}
  for seed in range(4):
    opt = make_opt('coco_tracking', ['--track_thresh', '0.2', '--new_thresh', '0.3'] + extra)
    trk = Tracker(opt) if which == 'product' else \
        co.TrackerOracle(opt.new_thresh, opt.max_age, opt.hungarian, opt.public_det)
    for f, (dets, pub) in enumerate(wt.synthetic_track_stream(seed)):
      if f == 0:
        trk.init_track([])
      before = trk.id_count
      out = trk.step(copy.deepcopy(dets), pub)
      ref = g['%s.s%d.f%d' % (name, seed, f)]
      assert [len(out), trk.id_count] == list(g['%s.s%d.f%d.n' % (name, seed, f)]), (name, seed, f)
      assert np.array_equal(_track_rows(out), ref), (name, seed, f)
      seen['coast'] += int((ref[:, 2] == 0).sum())
      seen['born'] += trk.id_count - before
  assert seen['born'] > 0
  if 'age2' in name:
    assert seen['coast'] > 0            # the streams do exercise coasting tracks


def test_hungarian_rejects_forced_pairs_and_orders_births_like_the_reference():
  """The solver must pair min(N, M) rows even through blocked cells; such pairs come back as unmatched AFTER the
  naturally unmatched ones (tracker.py:63-70), which decides the ids new tracks get."""
  from centertrack_b200.tracker import Tracker
  opt = make_opt('coco_tracking', ['--track_thresh', '0.1', '--new_thresh', '0.1', '--hungarian'])
  mk = lambda x, y, cls, score: {'score': score, 'class': cls, 'ct': np.array([x, y], np.float32),
                                'tracking': np.zeros(2, np.float32),
                                'bbox': np.array([x - 5, y - 5, x + 5, y + 5], np.float32)}
  prod, orc = Tracker(opt), co.TrackerOracle(0.1, -1, True, False)
  for t in (prod, orc):
    t.init_track([mk(10, 10, 1, 0.9), mk(100, 100, 1, 0.8)])
    # det 0 is far from everything (forced, rejected), det 1 continues track 1, det 2 has no column left
    out = t.step([mk(200, 200, 1, 0.9), mk(11, 10, 1, 0.8), mk(50, 50, 2, 0.7)])
    assert [(o['tracking_id'], o['active']) for o in out] == [(1, 2), (3, 1), (4, 1)]
    assert [float(o['ct'][0]) for o in out] == [11.0, 50.0, 200.0]    # natural unmatched (det 2) before the rejected det 0


@pytest.mark.parametrize('tag,extra', [('hc64', []), ('hc256', ['--head_conv', '256'])])
def test_generic_arch_oracle_and_product_keys_match_reference_golden(tag, extra, golden_dir):
  """--arch generic --backbone dla34 --neck dlaup (generic_network.py:29-107): state-dict keys of the product module
  equal the reference GenericNetwork's, the head width follows opts.py:295 (64 unless --head_conv), and the oracle
  restatement reproduces the reference's outputs and stages."""
  g = load_generic_golden(golden_dir)
  opt, model, sd = make_model('coco_tracking', extra=['--arch', 'generic'] + extra)
  assert sorted(sd.keys()) == list(g[tag + '.keys'])
  assert [opt.head_conv[h][0] for h in opt.heads] == list(g[tag + '.head_conv'])
  img, pre, hm = wt.synthetic_inputs(1, 64, 96)
  trace = {}
  out = co.GenericDLA34Oracle(sd, opt.heads).forward(img, pre, hm, trace=trace)
  for k in out:
    assert np.abs(out[k].numpy() - g['%s.head.%s' % (tag, k)]).max() < 1e-3, k
  for k in [x for x in g.files if x.startswith(tag + '.stage.')]:
    name = k[len(tag + '.stage.'):]
    key = 'feat' if name == 'ida_up.node_2' else name
    assert np.abs(trace[key].numpy() - g[k]).max() < 1e-3 * max(1.0, np.abs(g[k]).max()), name


def test_generic_arch_is_the_dla34_graph_under_other_names(golden_dir):
  """With --head_conv 256 the reference's GenericNetwork and DLASeg(34) agree exactly on the same tensors (recorded by
  the generator), the generic golden equals the dla_34 golden, and the product hands its engine the very state dict
  the dla_34 module does -- so the device plan that runs is the one the dla_34 GPU tests cover."""
  g = load_generic_golden(golden_dir)
  d = np.load(os.path.join(golden_dir, 'net_coco_tracking_64x96.npz'))
  assert np.all(g['hc256.max_abs_diff_vs_dla_34'] == 0)
  for h in ('hm', 'reg', 'wh', 'tracking'):
    assert np.array_equal(g['hc256.head.' + h], d['head.' + h])
  _, gen, _ = make_model('coco_tracking', extra=['--arch', 'generic', '--head_conv', '256'])
  _, dla, sd = make_model('coco_tracking')
  esd = gen._engine_state_dict()
  assert list(esd) == list(sd)                       # same names, same registration order
  assert all(torch.equal(esd[k], sd[k]) for k in sd)


def test_unsupported_archs_raise_not_implemented():
  from centertrack_b200.model import create_model
  opt = make_opt('coco_tracking', ['--arch', 'generic', '--backbone', 'resnet'])
  with pytest.raises(NotImplementedError):
    create_model(opt.arch, opt.heads, opt.head_conv, opt=opt)
  opt = make_opt('coco_tracking', ['--arch', 'generic', '--neck', 'msraup'])
  with pytest.raises(NotImplementedError):
    create_model(opt.arch, opt.heads, opt.head_conv, opt=opt)
  for arch in ('resdcn_18', 'res_18', 'dlav0_34'):
    opt = make_opt('coco_tracking', ['--arch', arch])
    with pytest.raises(NotImplementedError):
      create_model(opt.arch, opt.heads, opt.head_conv, opt=opt)


def test_dataset_constants_match_the_reference_classes(golden_dir):
  """dataset_info.py against the class attributes of the reference's dataset classes (generic_dataset.py:21-52,
  datasets/*.py; fixture written by oracle/gen_golden.py::gen_dataset_info).  `null` = the reference class leaves the
  attribute unset (crowdhuman's num_categories), where the product may be more helpful."""
  import json
  from centertrack_b200.dataset_info import dataset_factory
  g = json.load(open(os.path.join(golden_dir, 'dataset_info.json')))
  assert sorted(g) == sorted(dataset_factory)
  for name, ref in g.items():
    d = dataset_factory[name]
    for k in ('default_resolution', 'num_categories', 'rest_focal_length', 'num_joints', 'flip_idx'):
      if ref[k] is not None:
        got = getattr(d, k)
        assert (list(got) if isinstance(got, (list, tuple)) else got) == ref[k], (name, k, got, ref[k])
    assert np.allclose(np.ravel(d.mean), ref['mean'], atol=1e-7) and np.allclose(np.ravel(d.std), ref['std'], atol=1e-7)


def test_product_flag_defaults_equal_the_reference_parser(golden_dir):
  """Every flag the product parser shares with the reference's (opts.py:11-254, 134 flags dumped by
  oracle/gen_golden.py::gen_opts into opts_defaults.json) has the same default; the only product-specific flags are
  the --b200_* ones."""
  import json
  from centertrack_b200.opts import opts
  ref = json.load(open(os.path.join(golden_dir, 'opts_defaults.json')))
  mine = {a.dest: a.default for a in opts().parser._actions if a.dest != 'help'}
  assert sorted(k for k in mine if k not in ref) == ['b200_device_pre', 'b200_precision']
  assert {k: v for k, v in mine.items() if k in ref and ref[k] != v} == {}


@pytest.mark.parametrize('extra', [['--hungarian'], ['--public_det'], ['--public_det', '--hungarian', '--max_age', '3'],
                                   ['--max_age', '1']], ids=lambda e: '_'.join(x.strip('-') for x in e))
def test_product_tracker_modes_equal_oracle_on_many_streams(extra):
  """Beyond the golden's four streams: 24 more seeded crowded streams per mode, product tracker against the oracle
  restatement (itself pinned to the reference by track_modes.npz) -- ids, age, active, class, order, boxes exact."""
  import copy
  from centertrack_b200.tracker import Tracker
  for seed in range(10, 34):
    opt = make_opt('coco_tracking', ['--track_thresh', '0.2', '--new_thresh', '0.3'] + extra)
    prod = Tracker(opt)
    orc = co.TrackerOracle(opt.new_thresh, opt.max_age, opt.hungarian, opt.public_det)
    for f, (dets, pub) in enumerate(wt.synthetic_track_stream(seed, frames=5, crowd=30 + seed)):
      if f == 0:
        prod.init_track([]); orc.init_track([])
      a, b = prod.step(copy.deepcopy(dets), pub), orc.step(copy.deepcopy(dets), pub)
      assert prod.id_count == orc.id_count and np.array_equal(_track_rows(a), _track_rows(b)), (extra, seed, f)


@pytest.mark.parametrize('seed', range(6))
def test_product_pre_hm_render_equals_oracle_on_random_tracks(seed):
  """Detector._get_additional_inputs against the oracle restatement (pinned to the reference by host_pre.npz) on random
  track sets: boxes partly / fully outside the frame, degenerate boxes, inactive and low-score tracks, every
  resolution policy -- heat-maps and output-grid indices exact."""
  from centertrack_b200.detector import Detector
  from centertrack_b200.dataset_info import get_dataset
  rng = np.random.RandomState(50 + seed)
  name, extra, hw, _ = HOST_CASES[seed % len(HOST_CASES)]
  opt = make_opt('coco_tracking', ['--pre_thresh', '0.3'] + extra)
  opt.device = torch.device('cpu')
  det = object.__new__(Detector)
  ds = get_dataset(opt.dataset)
  det.opt, det.rest_focal_length = opt, ds.rest_focal_length
  det.mean = np.array(ds.mean, dtype=np.float32).reshape(1, 1, 3)
  det.std = np.array(ds.std, dtype=np.float32).reshape(1, 1, 3)
  h, w = int(rng.randint(60, 400)), int(rng.randint(60, 400))
  image = rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8)
  _, meta = det.pre_process(image, 1.0, {})
  tracks = []
  for _ in range(int(rng.randint(0, 60))):
    x0, y0 = rng.uniform(-0.3 * w, 1.1 * w), rng.uniform(-0.3 * h, 1.1 * h)
    bw, bh = rng.choice([0.0, 1.0]) * rng.uniform(0, 0.6 * w), rng.uniform(0, 0.6 * h)
    tracks.append({'score': float(rng.uniform(0.0, 1.0)), 'active': int(rng.randint(0, 3)),
                   'bbox': [float(x0), float(y0), float(x0 + bw), float(y0 + bh)]})
  hm, inds = det._get_additional_inputs(tracks, meta, with_hm=True)
  ref_hm, ref_inds = co.render_pre_hm(tracks, meta['trans_input'], meta['trans_output'], meta['inp_width'],
                                      meta['inp_height'], meta['out_width'], meta['out_height'], opt.pre_thresh)
  assert np.array_equal(hm.numpy(), ref_hm) and np.array_equal(inds.numpy(), ref_inds)


@pytest.mark.parametrize('ci', range(3))
@pytest.mark.parametrize('seed', range(3))
def test_product_post_process_equals_oracle_on_random_geometry(ci, seed):
  """generic_post_process (post_process.py:21-91, ddd_utils.py:91-136) against the oracle restatement (pinned to the
  reference by post_track.npz) for random source rectangles (c, s), image sizes and calibrations, on the coco / ddd /
  pose head sets: every field of every kept detection to 1e-5 relative."""
  from centertrack_b200.post_process import generic_post_process
  cfg, kind, C, H, W = CASES[ci]
  rng = np.random.RandomState(300 + 10 * ci + seed)
  opt = make_opt(cfg, ['--track_thresh', '0.05', '--new_thresh', '0.05'])
  inp = decode_inputs(kind, 1, C, H, W, 400 + 10 * ci + seed)
  if 'dep' in inp:
    inp['dep'] = (1. / (1. / (1 + np.exp(-inp['dep'] / 30 + 1)) + 1e-6) - 1.).astype(np.float32)
  dets = {k: v for k, v in co.generic_decode(inp, 100).items() if not k.startswith('_')}
  height, width = int(rng.randint(200, 900)), int(rng.randint(200, 1400))
  c = np.array([width * rng.uniform(0.3, 0.7), height * rng.uniform(0.3, 0.7)], dtype=np.float32)
  s = float(max(height, width) * rng.uniform(0.7, 1.4))
  f = float(rng.uniform(500, 1500))
  calib = np.array([[f, 0, width / 2, rng.uniform(-50, 50)], [0, f, height / 2, rng.uniform(-5, 5)],
                    [0, 0, 1, rng.uniform(-0.01, 0.01)]], dtype=np.float32)
  got = generic_post_process(opt, dets, [c], [s], H, W, opt.num_classes, [calib], height, width)[0]
  ref = co.generic_post_process(dets, [c], [s], H, W, opt.out_thresh, [calib])[0]
  got = [r for r in got if r['score'] > opt.out_thresh]
  ref = [r for r in ref if r['score'] > opt.out_thresh]
  assert len(got) == len(ref) > 0
  for a, b in zip(got, ref):
    assert set(a) == set(b)
    for k in a:
      x, y = np.asarray(a[k], np.float64), np.asarray(b[k], np.float64)
      assert np.allclose(x, y, rtol=1e-5, atol=1e-4), (k, x, y)
