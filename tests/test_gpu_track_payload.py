"""Pose and 3D task fields on the device tracker (ct_track_step_payload): the payload table beside the track table and
the amodal centre 3D head sets associate on.  Against the reference's post_process + Tracker golden (post_track.npz),
against generic_post_process + the host Tracker on crowded random streams, and closed-loop in StreamRunner.  The
layout, results() and descriptor checks at the end need no GPU."""
import copy
import ctypes as C
import os

import numpy as np
import pytest
import torch

from centertrack_b200 import _lib as L
from centertrack_b200 import synthetic as wt
from helpers import decode_inputs, make_model, make_opt

gpu = pytest.mark.gpu
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


def _fetch(trk):
  torch.cuda.synchronize()
  pay = trk.payload.cpu().numpy() if trk.payload is not None else None
  return trk.tracks.cpu().numpy(), trk.counts.cpu().numpy(), pay


# ------------------------------------------------------------------------------------------------ reference golden
@gpu
@pytest.mark.parametrize('ci', [1, 2], ids=['nuscenes_ddd', 'coco_pose'])
def test_device_tracker_payload_matches_reference_golden_three_frames(ci, golden_dir):
  """The 3-frame golden of the unmodified reference's generic_post_process + Tracker, built like
  test_device_tracker_matches_reference_golden_three_frames (640x480 source, its calib): rows, ids and id_count exact,
  every other key the golden has (ct -- the amodal centre on nuscenes_ddd --, tracking, bbox, hps, dep, dim, alpha,
  loc, rot_y) within the golden check's tolerance."""
  from centertrack_b200.decode import generic_decode
  from centertrack_b200.device_tracker import DeviceTracker
  g = np.load(os.path.join(golden_dir, 'post_track.npz'))
  cfg, kind, C_, H, W = [None, ('nuscenes_ddd', 'ddd', 10, 112, 200), ('coco_pose', 'pose', 1, 128, 128)][ci]
  opt = make_opt(cfg, ['--track_thresh', '0.05', '--new_thresh', '0.05'])
  height, width = 480, 640
  c = np.array([width / 2., height / 2.], dtype=np.float32)
  s = max(height, width) * 1.0
  calib = np.array([[1200, 0, width / 2, 0], [0, 1200, height / 2, 0], [0, 0, 1, 0]], dtype=np.float32)
  base = decode_inputs(kind, 1, C_, H, W, 100 + ci)
  trk = None
  for frame in range(3):
    inp = {k: v.copy() for k, v in base.items()}
    inp['tracking'] = (np.random.RandomState(1000 + frame).randn(*inp['tracking'].shape) * 0.5).astype(np.float32)
    if 'dep' in inp:
      inp['dep'] = (1. / (1. / (1 + np.exp(-inp['dep'] / 30 + 1)) + 1e-6) - 1.).astype(np.float32)
    res = generic_decode({k: torch.from_numpy(v).to(DEV) for k, v in inp.items()}, K=100)
    if trk is None:
      trk = DeviceTracker(opt, 1, 100, res.records.shape[2], res.layout, H * 4, W * 4, DEV, centers=[c], scales=[s],
                          calibs=[calib])
      assert trk.payload is not None
    trk.step(res.records)
    got = trk.results(*_fetch(trk))[0]
    n, id_count = g['%s.f%d.n' % (cfg, frame)]
    assert len(got) == n and int(trk.counts[0, 1]) == id_count
    keys = [k.split('.', 2)[2] for k in g.files if k.startswith('%s.f%d.' % (cfg, frame)) and not k.endswith('.n')]
    assert set(keys) <= set(got[0]), (set(keys) - set(got[0]))
    for key in keys:
      ref = g['%s.f%d.%s' % (cfg, frame, key)]
      arr = np.array([np.asarray(o[key], dtype=np.float64) for o in got]).reshape(ref.shape)
      if key in EXACT:
        assert np.array_equal(arr, ref), (cfg, frame, key)
      else:
        assert np.allclose(arr, ref, rtol=1e-4, atol=1e-3), (cfg, frame, key, np.abs(arr - ref).max())


# ------------------------------------------------------------------------------------- device vs host, random streams
def _ddd(extra=()):
  lay = {'reg': (9, 2), 'wh': (11, 2), 'tracking': (13, 2), 'dep': (15, 1), 'rot': (16, 8), 'dim': (24, 3)}
  off = 27
  for name, w in extra:
    lay[name] = (off, w)
    off += w
  return lay, off


def _pose(refined):
  lay = {'reg': (9, 2), 'wh': (11, 2), 'tracking': (13, 2), 'hps': (15, 34)}
  if refined:
    lay.update({'hps_refined': (49, 34), 'kps_score': (83, 1)})
  return lay, 84 if refined else 49


LAYOUTS = {'ddd_amodel_offset': _ddd([('amodel_offset', 2)]), 'ddd_box_centre': _ddd(),
           'ddd_velocity_att': _ddd([('amodel_offset', 2), ('nuscenes_att', 8), ('velocity', 3)]),
           'pose_refined': _pose(True), 'pose_raw': _pose(False)}
MODES = {'greedy_age3': ['--max_age', '3'], 'hungarian_age3': ['--hungarian', '--max_age', '3'],
         'public_age3': ['--public_det', '--max_age', '3'],
         'public_hungarian_age3': ['--public_det', '--hungarian', '--max_age', '3'], 'greedy_age2': ['--max_age', '2']}


def _random_records(rng, objs, layout, F, K, out_hw):
  """One frame of one stream: a crowded cluster of small objects (1.5-4 output cells) whose heat-map peak sits up to
  a cell off the box centre and whose amodel_offset reaches ~2.5 cells, a few below-threshold records, score-sorted."""
  out_h, out_w = out_hw
  move = rng.normal(0, 0.6, objs['pos'].shape)
  objs['pos'] = np.clip(objs['pos'] + move, 2, [out_w - 3, out_h - 3])
  vis = np.nonzero(rng.uniform(size=len(objs['pos'])) < 0.8)[0][:K - 4]
  rec = np.zeros((K, F), np.float32)
  n = len(vis)
  rec[:n, 0] = np.sort(rng.uniform(0.3, 1.0, n))[::-1]
  rec[n:, 0] = np.sort(rng.uniform(0.0, 0.09, K - n))[::-1]
  rec[:, 1] = rng.randint(0, 2, K)
  rec[:n, 1] = objs['cls'][vis]
  pos = np.concatenate([objs['pos'][vis], rng.uniform([2, 2], [out_w - 2, out_h - 2], (K - n, 2))])
  half = np.concatenate([objs['half'][vis], rng.uniform(0.7, 2.0, (K - n, 2))])
  rec[:, 2:4] = pos
  skew = rng.uniform(-1.0, 1.0, (K, 2))                     # box centre - peak, output cells
  rec[:, 4:6] = pos - half + skew
  rec[:, 6:8] = pos + half + skew
  rec[:, 9:11] = rng.rand(K, 2)
  rec[:, 11:13] = 2 * half
  rec[:n, 13:15] = -move[vis] + rng.normal(0, 0.2, (n, 2))
  if 'dep' in layout:
    rec[:, layout['dep'][0]] = rng.uniform(5, 60, K)
    rec[:, layout['rot'][0]:layout['rot'][0] + 8] = rng.randn(K, 8)
    rec[:, layout['dim'][0]:layout['dim'][0] + 3] = rng.uniform(0.3, 4, (K, 3))
  if 'amodel_offset' in layout:
    ao = np.concatenate([objs['ao'][vis], rng.normal(0, 1, (K - n, 2))]) + rng.normal(0, 0.1, (K, 2))
    rec[:, layout['amodel_offset'][0]:layout['amodel_offset'][0] + 2] = ao
  for h in ('velocity', 'nuscenes_att', 'hps', 'hps_refined', 'kps_score'):
    if h in layout:
      o, w = layout[h]
      rec[:, o:o + w] = rng.randn(K, w) * (3 if h.startswith('hps') else 1)
      if h.startswith('hps'):
        rec[:, o:o + w] += np.tile(pos, w // 2)
  return rec


def _new_objects(rng, K, out_hw):
  n = K - 6
  out_h, out_w = out_hw
  ctr = np.array([out_w / 2., out_h / 2.])
  return {'pos': ctr + rng.uniform(-14, 14, (n, 2)), 'half': rng.uniform(0.75, 2.0, (n, 2)),
          'cls': rng.randint(0, 2, n), 'ao': np.clip(rng.normal(0, 1.2, (n, 2)), -2.5, 2.5)}


def _public_near(res, rng):
  p = [np.asarray(r['ct'], np.float32) + np.asarray(r['tracking'], np.float32) + rng.uniform(-1, 1, 2)
       for r in res if rng.uniform() < 0.7]
  p += [rng.uniform([0, 0], [320, 300]) for _ in range(2)]
  return np.array(p, np.float32).reshape(-1, 2)


def _core_row(o):
  return np.array([o['score'], o['class'], *o['ct'], *o['tracking'], *o['bbox'], o['tracking_id'], o['age'],
                   o['active']], np.float32)


@gpu
@pytest.mark.parametrize('mode', list(MODES))
@pytest.mark.parametrize('lay', list(LAYOUTS))
def test_device_tracker_payload_equals_host_pipeline_on_crowded_streams(lay, mode):
  """B = 3 seeded crowded streams, 6 frames, with coasting: the device track table's 13 columns equal the host
  pipeline's (views of the same records -> generic_post_process -> Tracker.step) bit for bit, the amodal `ct`
  included; payload fields agree to 1e-5 relative (1e-6 absolute for angles near 0: atan2f is within 3 ulp of
  numpy's); a coasting row's payload is bit-equal to the row it came from.  On the 3D layouts the streams must
  contain detections that associate differently on the amodal centre than on the heat-map peak."""
  from centertrack_b200.decode import views_from_records
  from centertrack_b200.device_tracker import DeviceTracker
  from centertrack_b200.image import get_affine_transform, transform_preds_with_trans
  from centertrack_b200.post_process import generic_post_process
  from centertrack_b200.tracker import Tracker, greedy_assignment, hungarian_assignment
  layout, F = LAYOUTS[lay]
  B, K, inp_h, inp_w = 3, 48, 256, 320
  out_hw = (inp_h // 4, inp_w // 4)
  opt = make_opt('nuscenes_ddd' if 'dep' in layout else 'coco_pose',
                 ['--track_thresh', '0.2', '--new_thresh', '0.4', '--input_h', str(inp_h), '--input_w', str(inp_w)] +
                 MODES[mode])
  img_hw = [(240, 320), (300, 260), (256, 320)]
  centers = [np.array([w / 2., h / 2.], np.float32) for h, w in img_hw]
  scales = [max(h, w) * 1.0 for h, w in img_hw]
  calibs = [np.array([[f, 0, cx, 0], [0, f, cy, 0.5], [0, 0, 1, 0.25]], np.float32)
            for f, cx, cy in ((1200, 160, 120), (1000, 131.5, 149), (800, 170, 128.25))]
  trans = [get_affine_transform(centers[b], scales[b], 0, (out_hw[1], out_hw[0]), inv=1).astype(np.float32)
           for b in range(B)]
  trk = DeviceTracker(opt, B, K, F, layout, inp_h, inp_w, DEV, centers=centers, scales=scales, calibs=calibs,
                      max_public_dets=64)
  assert trk.payload is not None
  hosts = [Tracker(opt) for _ in range(B)]
  for h in hosts:
    h.init_track([])
  seed = 7 * list(LAYOUTS).index(lay) + list(MODES).index(mode)
  rng = np.random.RandomState(4000 + seed)
  objs = [_new_objects(rng, K, out_hw) for _ in range(B)]
  prev = [dict() for _ in range(B)]
  seen = dict.fromkeys(['amodal_differs', 'coast', 'born', 'matched'], 0)
  for frame in range(6):
    rec = np.stack([_random_records(rng, objs[b], layout, F, K, out_hw) for b in range(B)])
    views = {k: v.numpy() for k, v in views_from_records(torch.from_numpy(rec), layout).items()}
    results, pubs = [], []
    for b in range(B):
      one = {k: v[b:b + 1] for k, v in views.items()}
      res = generic_post_process(opt, one, [centers[b]], [scales[b]], out_hw[0], out_hw[1], opt.num_classes,
                                 [calibs[b]])[0]
      results.append([r for r in res if r['score'] > opt.out_thresh])
      pubs.append(_public_near(results[b], rng))
    pub_ct = np.zeros((B, 64, 2), np.float32)
    for b, p in enumerate(pubs):
      pub_ct[b, :len(p)] = p
    pub = (torch.from_numpy(pub_ct).to(DEV), torch.tensor([len(p) for p in pubs], dtype=torch.int32, device=DEV))
    trk.step(torch.from_numpy(rec).to(DEV), *(pub if trk.public_det else ()))
    tab, cnt, pay = _fetch(trk)
    got = trk.results(tab, cnt, pay)
    for b in range(B):
      res = results[b]
      if 'loc' in trk.payload_layout and res and hosts[b].tracks:   # does the amodal centre change the association?
        peak = transform_preds_with_trans(views['cts'][b, :len(res)].reshape(-1, 2), trans[b])
        at_peak = [dict(r, ct=peak[i]) for i, r in enumerate(res)]
        assign = (lambda c: hungarian_assignment(c)[0]) if trk.hungarian else greedy_assignment
        a = assign(hosts[b]._gated_cost(res))
        p = assign(hosts[b]._gated_cost(at_peak))
        seen['amodal_differs'] += sorted(map(tuple, a)) != sorted(map(tuple, p))
      before = hosts[b].id_count
      want = hosts[b].step(copy.deepcopy(res), [{'ct': q} for q in pubs[b]])
      seen['born'] += hosts[b].id_count - before
      ctx = (lay, mode, frame, b)
      assert int(cnt[b, 0]) == len(want) and int(cnt[b, 1]) == hosts[b].id_count, ctx
      assert np.array_equal(tab[b, :len(want)], np.array([_core_row(w) for w in want]).reshape(-1, L.CT_TRK_FLOATS)), ctx
      for r, (g, w) in enumerate(zip(got[b], want)):
        for k in trk.payload_layout:
          assert np.allclose(np.asarray(g[k], np.float64), np.asarray(w[k], np.float64).reshape(np.shape(g[k])),
                             rtol=1e-5, atol=1e-6), (ctx, k, g[k], w[k])
        if g['active'] == 0:
          seen['coast'] += 1
          assert np.array_equal(pay[b, r], prev[b][g['tracking_id']]), ctx
        elif g['active'] > 1:
          seen['matched'] += 1
      prev[b] = {g['tracking_id']: pay[b, r].copy() for r, g in enumerate(got[b])}
  assert seen['coast'] > 0 and seen['born'] > 0 and seen['matched'] > 0, seen
  if 'loc' in trk.payload_layout:
    assert seen['amodal_differs'] > 0, seen


# --------------------------------------------------------------------------------------------------- closed loop
@gpu
@pytest.mark.parametrize('cfg', ['nuscenes_ddd', 'coco_pose'])
def test_stream_runner_payload_closes_the_loop_like_the_host_pipeline(cfg):
  """StreamRunner(device_tracking=True) on the 3D and pose head sets (fp32 engine, B = 2, 5 frames): fetch_results()
  against the same loop run through the host pre_hm render, generic_post_process (the default calib) and the host
  Tracker; graph replays give the same track and payload tables as an eager runner."""
  from centertrack_b200.decode import generic_decode
  from centertrack_b200.image import get_affine_transform
  from centertrack_b200.post_process import generic_post_process
  from centertrack_b200.runner import StreamRunner
  from centertrack_b200.tracker import Tracker
  B, H, W, K = 2, 64, 96, 30
  opt, model, sd = make_model(cfg, extra=['--track_thresh', '0.1', '--new_thresh', '0.1', '--pre_thresh', '0.1',
                                          '--input_h', str(H), '--input_w', str(W), '--max_age', '2'])
  with torch.no_grad():           # boxes of a few pixels (the synthetic weights give ~0 wh)
    model.state_dict()['wh.2.bias'].fill_(3.0)
  model = model.cuda()
  runners = {g: StreamRunner(model, B, H, W, K=K, precision='fp32', device='cuda', opt=opt, device_tracking=True,
                             use_graph=g) for g in (True, False)}
  for r in runners.values():
    r.warm()
  runner = runners[True]
  assert runner.tracker.payload is not None
  assert runner.d2h_bytes_per_step == (runner.rec.numel() + runner.tracker.tracks.numel() + B * 2 +
                                       runner.tracker.payload.numel()) * 4
  eng = model.engine_for(B, H, W, DEV, 'fp32')
  det = _host_detector(opt)
  calib = det._get_default_calib(W, H)
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
  total = 0
  for t, img in enumerate(frames):
    for r in runners.values():
      r.step_host(img.pin_memory())
      r.fetch()                   # one runner at a time: the two share the engine's activation buffers
    got = runner.fetch_results()
    tabs = [r.fetch_tracks() + (r.h_pay[(r.t - 1) & 1].numpy(),) for r in runners.values()]
    assert all(np.array_equal(a, b) for a, b in zip(*tabs)), t
    hms = [det._get_additional_inputs(hosts[b].tracks, meta, with_hm=True)[0] for b in range(B)]
    x = img.cuda()
    out = dict(eng.forward(x, x if pre is None else pre, torch.cat(hms, 0).cuda()))
    views = {k: v.cpu().numpy() for k, v in generic_decode(out, K=K).items()}
    for b in range(B):
      one = {k: v[b:b + 1] for k, v in views.items()}
      r = generic_post_process(opt, one, [c], [s], H // 4, W // 4, opt.num_classes, [calib])[0]
      want = hosts[b].step([q for q in r if q['score'] > opt.out_thresh])
      assert len(got[b]) == len(want), (t, b)
      for a, w in zip(got[b], want):
        assert tuple(a[k] for k in EXACT) == tuple(int(w[k]) for k in EXACT), (t, b, a, w)
        for k in ('ct', 'tracking', 'bbox') + tuple(runner.tracker.payload_layout):
          assert np.allclose(np.asarray(a[k], np.float64), np.asarray(w[k], np.float64).reshape(np.shape(a[k])),
                             rtol=1e-4, atol=1e-3), (t, b, k)
        assert abs(a['score'] - float(w['score'])) < 1e-6
      assert int(runner.fetch_tracks()[1][b, 1]) == hosts[b].id_count
      total += len(want)
    pre = x
  assert total > 0 and max(h.id_count for h in hosts) > 0


# ------------------------------------------------------------------------------------------------------- CPU only
def test_payload_layout_follows_the_decode_heads():
  from centertrack_b200.device_tracker import payload_layout
  assert payload_layout({'wh': (9, 2), 'tracking': (11, 2)}) == {}
  assert payload_layout(LAYOUTS['pose_refined'][0]) == {'hps': (0, 34)}
  assert payload_layout(LAYOUTS['ddd_box_centre'][0]) == {'dep': (0, 1), 'dim': (1, 3), 'alpha': (4, 1),
                                                          'loc': (5, 3), 'rot_y': (8, 1)}
  assert payload_layout(LAYOUTS['ddd_velocity_att'][0]) == {
      'dep': (0, 1), 'dim': (1, 3), 'alpha': (4, 1), 'loc': (5, 3), 'rot_y': (8, 1), 'velocity': (9, 3),
      'nuscenes_att': (12, 8)}
  assert payload_layout({'rot': (9, 8), 'velocity': (17, 3)}) == {'alpha': (0, 1), 'velocity': (1, 3)}
  with pytest.raises(ValueError, match='dim head with 2 channels'):
    payload_layout({'dim': (9, 2)})


def test_device_tracker_results_carry_the_payload_fields(built_lib):
  from centertrack_b200.device_tracker import DeviceTracker
  layout, F = LAYOUTS['ddd_velocity_att']
  opt = make_opt('nuscenes_ddd')
  trk = DeviceTracker(opt, 2, 4, F, layout, 64, 96, 'cpu')
  assert trk.Wp == 20 and tuple(trk.payload.shape) == (2, trk.T, 20)
  from centertrack_b200.dataset_info import get_dataset
  f = opt.test_focal_length if opt.test_focal_length >= 0 else get_dataset(opt.dataset).rest_focal_length
  assert np.array_equal(trk.calib.numpy()[1], np.array([[f, 0, 48, 0], [0, f, 32, 0], [0, 0, 1, 0]], np.float32))
  tracks = np.zeros((2, trk.T, L.CT_TRK_FLOATS), np.float32)
  tracks[0, :2, L.CT_TRK_ID] = [3, 5]
  counts = np.array([[2, 5], [0, 0]], np.int32)
  pay = np.arange(2 * trk.T * 20, dtype=np.float32).reshape(2, trk.T, 20)
  got = trk.results(tracks, counts, pay)
  assert [len(g) for g in got] == [2, 0]
  row = got[0][1]
  assert row['tracking_id'] == 5
  assert {k: np.shape(row[k]) for k in trk.payload_layout} == {'dep': (1,), 'dim': (3,), 'alpha': (), 'loc': (3,),
                                                                'rot_y': (), 'velocity': (3,), 'nuscenes_att': (8,)}
  assert isinstance(row['alpha'], float) and row['alpha'] == pay[0, 1, 4] and row['rot_y'] == pay[0, 1, 8]
  assert np.array_equal(row['nuscenes_att'], pay[0, 1, 12:20])
  with pytest.raises(ValueError, match='payload_np'):
    trk.results(tracks, counts)
  with pytest.raises(ValueError, match='calibs'):
    DeviceTracker(opt, 2, 4, F, layout, 64, 96, 'cpu', calibs=[np.eye(3, 4)])
  plain = DeviceTracker(make_opt('coco_tracking'), 1, 4, 13, {'wh': (9, 2), 'tracking': (11, 2)}, 64, 96, 'cpu')
  assert plain.payload is None and plain.Wp == 0
  assert set(plain.results(tracks[:1], counts[:1])[0][0]) == {'score', 'class', 'ct', 'tracking', 'bbox', 'tracking_id',
                                                             'age', 'active'}


def test_track_step_payload_rejects_bad_descriptors_before_launch(built_lib):
  """Each case fails validation and returns -1 with a message; none reaches a launch."""
  lib = L.lib()
  d, a, p = L.TrackDesc(), L.TrackAssoc(), L.TrackPayload()
  d.B, d.K, d.F, d.rec_tracking, d.max_tracks = 2, 100, 40, 13, 100
  d.records = d.trans_out_inv = d.tracks = d.counts = 64          # never dereferenced: validation fails first

  def ddd():
    q = L.TrackPayload()
    q.width, q.payload, q.calib = 20, 64, 64
    q.rec_hps, q.rec_dep, q.rec_rot, q.rec_dim, q.rec_amodel_offset = -1, 15, 16, 24, 27
    q.rec_nuscenes_att, q.att_floats, q.rec_velocity, q.velocity_floats = 29, 8, 37, 3
    return q

  def fails(q, msg):
    assert lib.ct_track_step_payload(C.byref(d), C.byref(a), C.byref(q), None) == -1
    assert msg in lib.ct_last_error(), lib.ct_last_error()

  p = ddd()
  p.payload = None
  fails(p, b'null payload')
  for field, value in (('rec_velocity', 38), ('rec_dep', 3), ('rec_dim', 38), ('rec_hps', 30)):
    p = ddd()
    setattr(p, field, value)                  # outside [CT_REC_HEADS, F), or rec_hps with hps_floats = 0
    fails(p, b'outside the record')
  p = ddd()
  p.width = 19
  fails(p, b'payload width')
  p = ddd()
  p.rec_rot, p.width = -1, 16                 # without rot there is no alpha, loc or rot_y: 15 floats
  fails(p, b'payload width')
  p = ddd()
  p.calib = None
  fails(p, b'calib')
  p = ddd()
  d.max_tracks = 2000                         # the table fits in shared memory, its payload rows do not
  assert lib.ct_track_smem_bytes(100, 2000) <= 200 * 1024 < lib.ct_track_payload_smem_bytes(100, 2000, 20, 0)
  fails(p, b'shared memory')
  assert lib.ct_track_payload_smem_bytes(100, 400, 34, 1) == lib.ct_track_assoc_smem_bytes(100, 400) + 400 * 34 * 4
