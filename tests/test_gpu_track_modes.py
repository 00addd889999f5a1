"""--hungarian and --public_det association on the device tracker (ct_track_step_assoc): against the reference's
Tracker golden (track_modes.npz), against the host Tracker on tie-heavy streams, and closed-loop in StreamRunner.
The argument checks at the end need no GPU."""
import copy
import ctypes as C
import os

import numpy as np
import pytest
import torch

from centertrack_b200 import _lib as L
from centertrack_b200 import synthetic as wt
from helpers import make_model, make_opt

gpu = pytest.mark.gpu

TRACK_MODES = [('greedy_age2', ['--max_age', '2']), ('hungarian', ['--hungarian']),
               ('hungarian_age2', ['--hungarian', '--max_age', '2']), ('public', ['--public_det']),
               ('public_hungarian_age2', ['--public_det', '--hungarian', '--max_age', '2'])]
LAYOUT = {'tracking': (9, 2)}            # records: score, cls, xs, ys, bbox[4], ind, tracking[2]
F = 11
IDENTITY = [1., 0., 0., 0., 1., 0.]


def _track_rows(out):
  return np.array([[o['tracking_id'], o['age'], o['active'], o['class'], o['score']] + list(map(float, o['bbox']))
                   for o in out], np.float64).reshape(-1, 9)


def _records(streams, K):
  """Post-processed detections (image coordinates, score-sorted) of B streams -> decode records [B,K,F] that the
  device tracker maps back with an identity output affine; unused slots score 0 (below out_thresh)."""
  rec = np.zeros((len(streams), K, F), np.float32)
  for b, dets in enumerate(streams):
    assert len(dets) <= K
    for i, d in enumerate(dets):
      rec[b, i, 0], rec[b, i, 1] = d['score'], d['class'] - 1
      rec[b, i, 2:4], rec[b, i, 4:8], rec[b, i, 9:11] = d['ct'], d['bbox'], d['tracking']
  return rec


def _public(pubs, P):
  ct = np.zeros((len(pubs), P, 2), np.float32)
  n = np.zeros(len(pubs), np.int32)
  for b, p in enumerate(pubs):
    a = np.array([q['ct'] for q in p], np.float32).reshape(-1, 2)
    ct[b, :len(a)], n[b] = a, len(a)
  return torch.from_numpy(ct).cuda(), torch.from_numpy(n).cuda()


def _device_tracker(opt, B, K, inp=256, max_public=128):
  """Records in image coordinates: identity output affine, and out_thresh below every score (the streams' detections
  are already the kept ones)."""
  from centertrack_b200.device_tracker import DeviceTracker
  opt.out_thresh = 0.1
  trk = DeviceTracker(opt, B, K, F, LAYOUT, inp, inp, 'cuda', max_public_dets=max_public)
  trk.trans_out_inv.copy_(torch.tensor([IDENTITY] * B))
  return trk


def _check_predictions(rec, streams, K):
  """Precondition of an exact comparison: the device's fp32 ct + tracking of every detection equals the host's.  A
  fresh greedy tracker that gives every detection a track lists all of them, in order."""
  opt = make_opt('coco_tracking')
  opt.new_thresh = -1.0
  trk = _device_tracker(opt, len(streams), K)
  trk.step(torch.from_numpy(rec).cuda())
  tab, cnt = trk.tracks.cpu().numpy(), trk.counts.cpu().numpy()
  for b, dets in enumerate(streams):
    assert int(cnt[b, 0]) == len(dets)
    got = tab[b, :len(dets), L.CT_TRK_CT:L.CT_TRK_CT + 2] + tab[b, :len(dets), L.CT_TRK_TRACKING:L.CT_TRK_TRACKING + 2]
    want = np.array([np.asarray(d['ct']) + np.asarray(d['tracking']) for d in dets], np.float32).reshape(-1, 2)
    assert np.array_equal(got, want), b


@gpu
@pytest.mark.parametrize('mode', range(len(TRACK_MODES)), ids=[m[0] for m in TRACK_MODES])
def test_device_tracker_modes_match_reference_golden(mode, golden_dir):
  """The reference Tracker's rows of track_modes.npz (4 seeded crowded streams x 6 frames per mode), all four streams
  in one batch: id, age, active, class, score, bbox, in order, and id_count exactly."""
  g = np.load(os.path.join(golden_dir, 'track_modes.npz'))
  name, extra = TRACK_MODES[mode]
  K, seeds = 64, range(4)
  opt = make_opt('coco_tracking', ['--track_thresh', '0.2', '--new_thresh', '0.3'] + extra)
  trk = _device_tracker(opt, len(seeds), K)
  streams = [wt.synthetic_track_stream(s) for s in seeds]
  for f in range(len(streams[0])):
    dets = [st[f][0] for st in streams]
    rec = _records(dets, K)
    _check_predictions(rec, dets, K)
    pub = _public([st[f][1] for st in streams], trk.max_public) if trk.public_det else (None, None)
    trk.step(torch.from_numpy(rec).cuda(), *pub)
    got = trk.results(trk.tracks.cpu().numpy(), trk.counts.cpu().numpy())
    for b, s in enumerate(seeds):
      assert [len(got[b]), int(trk.counts[b, 1])] == list(g['%s.s%d.f%d.n' % (name, s, f)]), (name, s, f)
      assert np.array_equal(_track_rows(got[b]), g['%s.s%d.f%d' % (name, s, f)]), (name, s, f)


def _tie_stream(seed, K, frames=6):
  """Seeded streams built for exact ties: objects on an integer grid in a small crowded area moving by whole pixels
  with exact `tracking`, a few box sizes, a handful of score values, exact duplicate detections, single-class crowds
  (every third seed), clutter far from the objects, an empty frame, frames with every record slot used and frames
  with a few detections.  Public detections sit on the predicted centres with integer
  jitter and are duplicated too."""
  rng = np.random.RandomState(9100 + seed)
  n_obj = int(rng.randint(K // 2, K))
  ct = rng.randint(20, 70, (n_obj, 2)).astype(np.float64)
  wh = np.array([6., 10., 16.])[rng.randint(0, 3, (n_obj, 2))]
  cls = np.ones(n_obj, int) if seed % 3 == 0 else rng.randint(1, 3, n_obj)
  scores = np.array([0.25, 0.4, 0.4, 0.6, 0.9], np.float32)
  empty = 2 + seed % 3
  out = []
  for f in range(frames):
    move = rng.randint(-2, 3, (n_obj, 2)).astype(np.float64)
    ct = ct + move
    kind = 'empty' if f == empty else ['full', 'few', 'some'][(f + seed) % 3]
    n_vis = {'empty': 0, 'full': n_obj, 'few': int(rng.randint(1, 5)), 'some': int(rng.randint(n_obj // 3, n_obj))}[kind]
    dets = []
    for i in rng.permutation(n_obj)[:n_vis]:
      c = ct[i].astype(np.float32)
      w, h = wh[i]
      dets.append({'score': float(scores[rng.randint(0, len(scores))]), 'class': int(cls[i]), 'ct': c,
                   'tracking': (-move[i]).astype(np.float32),
                   'bbox': np.array([c[0] - w / 2, c[1] - h / 2, c[0] + w / 2, c[1] + h / 2], np.float32)})
    if dets:
      for _ in range(int(rng.randint(0, 4))):                       # exact duplicates
        dets.append(copy.deepcopy(dets[rng.randint(0, len(dets))]))
      # clutter far from the objects (rows with every cell blocked); in a full frame it takes every free record slot,
      # and the new tracks it starts coast later, so that the table grows towards its max_age bound
      for _ in range(K - len(dets) if kind == 'full' else int(rng.randint(0, 3))):
        c = rng.randint(100, 250, 2).astype(np.float32)
        dets.append({'score': float(scores[rng.randint(0, len(scores))]), 'class': int(rng.randint(1, 3)), 'ct': c,
                     'tracking': np.zeros(2, np.float32), 'bbox': np.array([c[0] - 3, c[1] - 3, c[0] + 3, c[1] + 3],
                                                                           np.float32)})
    order = np.argsort([-d['score'] for d in dets], kind='stable')
    dets = [dets[i] for i in order][:K]
    pub = []
    for d in dets:
      if rng.uniform() < 0.7:
        q = {'ct': (d['ct'] + d['tracking'] + rng.randint(-1, 2, 2)).astype(np.float32)}
        pub.append(q)
        if rng.uniform() < 0.2:
          pub.append(copy.deepcopy(q))
    if dets:
      pub.append({'ct': np.array([500., 500.], np.float32)})        # claims nothing
    out.append((dets, pub))
  return out


def _host_detector(opt):
  from centertrack_b200.dataset_info import get_dataset
  from centertrack_b200.detector import Detector
  from centertrack_b200.tracker import Tracker
  det = object.__new__(Detector)
  ds = get_dataset(opt.dataset)
  det.opt, det.cnt, det.pre_images, det.tracker = opt, 0, None, Tracker(opt)
  det.mean = np.array(ds.mean, dtype=np.float32).reshape(1, 1, 3)
  det.std = np.array(ds.std, dtype=np.float32).reshape(1, 1, 3)
  det.rest_focal_length = ds.rest_focal_length
  det.flip_idx = ds.flip_idx
  return det


MANY_MODES = [['--hungarian'], ['--hungarian', '--max_age', '2'], ['--public_det'], ['--public_det', '--max_age', '2'],
              ['--public_det', '--hungarian', '--max_age', '3']]


@gpu
@pytest.mark.parametrize('extra', MANY_MODES, ids=lambda e: '_'.join(x.strip('-') for x in e))
def test_device_tracker_modes_equal_host_tracker_on_tie_heavy_streams(extra):
  """24 seeded tie-heavy streams per mode, 3 streams per batch: the device rows (id, age, active, class, score, bbox,
  order) and id_count equal the host Tracker's exactly, and the prior heat-map splatted for the next frame matches
  Detector._get_additional_inputs on the host tracks.  The streams must cover N > M, N < M, N = 0, M = 0, fully
  blocked rows, and (Hungarian) pairs forced through a blocked cell."""
  from centertrack_b200.image import get_affine_transform
  from centertrack_b200.tracker import Tracker, hungarian_assignment
  K, B, inp = 32, 3, 256
  opt = make_opt('coco_tracking', ['--track_thresh', '0.2', '--new_thresh', '0.3',
                                   '--pre_thresh', '0.3', '--input_h', str(inp), '--input_w', str(inp)] + extra)
  det = _host_detector(opt)
  c, s = np.array([inp / 2., inp / 2.], np.float32), float(inp)
  meta = {'inp_width': inp, 'inp_height': inp, 'out_width': inp // 4, 'out_height': inp // 4,
          'trans_input': get_affine_transform(c, s, 0, [inp, inp]),
          'trans_output': get_affine_transform(c, s, 0, [inp // 4, inp // 4])}
  seen = dict.fromkeys(['N>M', 'N<M', 'N=0', 'M=0', 'blocked_row', 'rejected', 'born', 'coast'], 0)
  for first in range(0, 24, B):
    seeds = range(first, first + B)
    trk = _device_tracker(opt, B, K, inp=inp)
    hosts = [Tracker(opt) for _ in seeds]
    for h in hosts:
      h.init_track([])
    streams = [_tie_stream(sd, K) for sd in seeds]
    pre_hm = torch.zeros((B, 1, inp, inp), device='cuda')
    for f in range(len(streams[0])):
      dets = [st[f][0] for st in streams]
      pubs = [st[f][1] for st in streams]
      rec = _records(dets, K)
      _check_predictions(rec, dets, K)
      trk.step(torch.from_numpy(rec).cuda(), *(_public(pubs, trk.max_public) if trk.public_det else ()))
      trk.render(pre_hm)
      got = trk.results(trk.tracks.cpu().numpy(), trk.counts.cpu().numpy())
      for b in range(B):
        n, m = len(dets[b]), len(hosts[b].tracks)
        seen['N>M'] += n > m; seen['N<M'] += n < m; seen['N=0'] += n == 0; seen['M=0'] += m == 0
        if n and m:
          cost = hosts[b]._gated_cost(dets[b])
          seen['blocked_row'] += int((cost >= 1e18).all(axis=1).sum())
          if trk.hungarian:
            seen['rejected'] += len(hungarian_assignment(cost.copy())[1])
        before = hosts[b].id_count
        want = hosts[b].step(copy.deepcopy(dets[b]), pubs[b])
        seen['born'] += hosts[b].id_count - before
        seen['coast'] += sum(1 for w in want if w['active'] == 0)
        ctx = (extra, seeds[b], f)
        assert int(trk.counts[b, 1]) == hosts[b].id_count, ctx
        assert np.array_equal(_track_rows(got[b]), _track_rows(want)), ctx
        opt.device = torch.device('cpu')
        hm_host, _ = det._get_additional_inputs(hosts[b].tracks, meta, with_hm=True)
        diff = np.abs(pre_hm[b].cpu().numpy() - hm_host.numpy()[0])
        assert (diff > 1e-6).mean() < 2e-3, (ctx, float(diff.max()), float((diff > 1e-6).mean()))
  assert all(seen[k] > 0 for k in ('N>M', 'N<M', 'N=0', 'M=0', 'blocked_row', 'born')), seen
  if '--hungarian' in extra:
    assert seen['rejected'] > 0, seen
  if '--max_age' in extra:
    assert seen['coast'] > 0, seen


@gpu
def test_device_tracker_reports_hungarian_search_steps():
  """The optional per-stream step counter: at least one Dijkstra step per assigned row, 0 in a greedy call."""
  K = 32
  opt = make_opt('coco_tracking', ['--new_thresh', '0.3', '--hungarian'])
  trk = _device_tracker(opt, 1, K)
  stream = _tie_stream(1, K)
  steps = torch.full((1,), -1, dtype=torch.int32, device='cuda')
  for f in range(2):
    m = int(trk.counts[0, 0])
    dets = stream[f][0]
    trk.step(torch.from_numpy(_records([dets], K)).cuda(), steps=steps)
    assert int(steps[0]) >= min(len(dets), m)
  gopt = make_opt('coco_tracking', ['--new_thresh', '0.3'])
  g = _device_tracker(gopt, 1, K)
  g.step(torch.from_numpy(_records([stream[0][0]], K)).cuda(), steps=steps)
  assert int(steps[0]) == 0


CLOSED_LOOP = [['--hungarian'], ['--public_det'], ['--public_det', '--hungarian', '--max_age', '2']]


def _public_near(dets, H, W, t):
  """Public detections of one frame: near the predicted centres of about 70 % of the frame's detections (jittered),
  plus a few anywhere in the image."""
  rng = np.random.RandomState(500 + t)
  out = []
  for ds in dets:
    p = [np.asarray(d['ct'], np.float32) + np.asarray(d['tracking'], np.float32) + rng.uniform(-0.5, 0.5, 2)
         for d in ds if rng.uniform() < 0.7]
    p += [rng.uniform([0, 0], [W, H]) for _ in range(3)]
    out.append(np.array(p, np.float32).reshape(-1, 2))
  return out


@gpu
@pytest.mark.parametrize('extra', CLOSED_LOOP, ids=lambda e: '_'.join(x.strip('-') for x in e))
def test_stream_runner_modes_close_the_loop_like_the_host_pipeline(extra):
  """StreamRunner(device_tracking=True) with --hungarian / --public_det: pre_hm(t) = splat(tracks(t-1)) -> network +
  decode -> association, one CUDA graph per step with the public detections staged per input slot, against the same
  loop run through the host tracker and the host pre_hm render (fp32 engine, B = 2 streams, 5 frames).  An eager
  runner gives the same track tables as the graph replays."""
  from centertrack_b200.decode import generic_decode
  from centertrack_b200.image import get_affine_transform
  from centertrack_b200.post_process import generic_post_process
  from centertrack_b200.runner import StreamRunner
  from centertrack_b200.tracker import Tracker
  B, H, W, K = 2, 64, 96, 30
  opt, model, sd = make_model('coco_tracking', extra=['--track_thresh', '0.1', '--new_thresh', '0.1', '--pre_thresh', '0.1',
                                                       '--input_h', str(H), '--input_w', str(W)] + extra)
  with torch.no_grad():           # boxes of a few pixels (the synthetic weights give ~0 wh): gating and claims can pass
    model.state_dict()['wh.2.bias'].fill_(3.0)
  model = model.cuda()
  runners = {g: StreamRunner(model, B, H, W, K=K, precision='fp32', device='cuda', opt=opt, device_tracking=True,
                             use_graph=g) for g in (True, False)}
  for r in runners.values():
    r.warm()
  runner = runners[True]
  public = '--public_det' in extra
  if public:
    frame = wt.synthetic_inputs(B, H, W, seed=60)[0].pin_memory()
    with pytest.raises(ValueError, match='public'):
      runner.step_host(frame)
    with pytest.raises(ValueError, match='max_public_dets'):
      runner.step_host(frame, public_dets=[np.zeros((513, 2), np.float32)] * B)
    assert runner.t == 0
    assert runner.h2d_bytes_per_step == B * 3 * H * W * 4 + B * (512 * 2 + 1) * 4
  eng = model.engine_for(B, H, W, torch.device('cuda'), 'fp32')
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
  born = 0
  for t, img in enumerate(frames):
    # host loop first: its detections place the frame's public detections
    hms = [det._get_additional_inputs(hosts[b].tracks, meta, with_hm=True)[0] for b in range(B)]
    hm = torch.cat(hms, 0).cuda()
    x = img.cuda()
    out = dict(eng.forward(x, x if pre is None else pre, hm))
    res = generic_decode(out, K=K)
    views = {k: v.cpu().numpy() for k, v in res.items()}
    dets = []
    for b in range(B):
      one = {k: v[b:b + 1] for k, v in views.items()}
      r = generic_post_process(opt, one, [c], [s], H // 4, W // 4, opt.num_classes)[0]
      dets.append([q for q in r if q['score'] > opt.out_thresh])
    pub = _public_near(dets, H, W, t) if public else None
    for r in runners.values():
      r.step_host(img.pin_memory(), public_dets=pub)
      r.fetch()                   # one runner at a time: the two share the engine's activation buffers
    tracks_np, counts_np = runner.fetch_tracks()
    eager = runners[False].fetch_tracks()
    assert np.array_equal(counts_np, eager[1]) and np.array_equal(tracks_np, eager[0]), t
    got = runner.tracker.results(tracks_np, counts_np)
    total = 0
    for b in range(B):
      before = hosts[b].id_count
      want = hosts[b].step(dets[b], [{'ct': p} for p in pub[b]] if public else None)
      born += hosts[b].id_count - before
      assert len(got[b]) == len(want), (t, b)
      for a, w in zip(got[b], want):
        assert (a['tracking_id'], a['age'], a['active'], a['class']) == \
            (int(w['tracking_id']), int(w['age']), int(w['active']), int(w['class'])), (t, b, a, w)
        for k in ('ct', 'tracking', 'bbox'):
          assert np.allclose(np.asarray(a[k], np.float64), np.asarray(w[k], np.float64), rtol=1e-4, atol=1e-3), (t, b, k)
        assert abs(a['score'] - float(w['score'])) < 1e-6
      assert int(counts_np[b, 1]) == hosts[b].id_count
      total += len(want)
    assert total > 0
    pre = x
  assert born > 0


# ---------------------------------------------------------------------------------------------- argument checks (CPU)
def test_track_step_assoc_rejects_bad_descriptors_before_launch(built_lib):
  """Every case below fails validation and returns -1 with a message; none reaches a launch."""
  lib = L.lib()
  d = L.TrackDesc()
  a = L.TrackAssoc()
  assert lib.ct_track_step_assoc(None, C.byref(a), None) == -1 and b'null pointer' in lib.ct_last_error()
  d.B, d.K, d.F, d.rec_tracking, d.max_tracks = 2, 100, F, 9, 100
  d.records = d.trans_out_inv = d.tracks = d.counts = 64          # never dereferenced: validation fails first
  assert lib.ct_track_step_assoc(C.byref(d), None, None) == -1 and b'null pointer' in lib.ct_last_error()
  a.public_det, a.max_public = 1, 16
  assert lib.ct_track_step_assoc(C.byref(d), C.byref(a), None) == -1
  assert b'public_det needs public_ct' in lib.ct_last_error()
  a.public_ct, a.public_n, a.max_public = 64, 64, 0
  assert lib.ct_track_step_assoc(C.byref(d), C.byref(a), None) == -1 and b'max_public' in lib.ct_last_error()
  a = L.TrackAssoc()
  a.hungarian = 1
  d.max_tracks = 2500          # the greedy table fits in shared memory, the solver's scratch does not
  assert lib.ct_track_smem_bytes(100, 2500) <= 200 * 1024 < lib.ct_track_assoc_smem_bytes(100, 2500)
  assert lib.ct_track_step_assoc(C.byref(d), C.byref(a), None) == -1 and b'shared memory' in lib.ct_last_error()


def test_device_tracker_and_runner_refuse_missing_or_too_many_public_detections(built_lib):
  from centertrack_b200.device_tracker import DeviceTracker
  from centertrack_b200.runner import StreamRunner
  opt = make_opt('coco_tracking', ['--public_det', '--hungarian'])
  trk = DeviceTracker(opt, 2, 16, F, LAYOUT, 64, 64, 'cpu', max_public_dets=8)
  with pytest.raises(ValueError, match='public'):
    trk.step(torch.zeros((2, 16, F)))
  with pytest.raises(ValueError):
    DeviceTracker(opt, 2, 16, F, LAYOUT, 64, 64, 'cpu', max_public_dets=0)
  with pytest.raises(ValueError, match='shared memory'):
    DeviceTracker(opt, 2, 100, F, LAYOUT, 64, 64, 'cpu', max_tracks=2500)
  r = object.__new__(StreamRunner)                # the checks step_host / load_device_inputs run before any copy
  r.B, r.public, r.tracker = 2, True, trk
  with pytest.raises(ValueError, match='public'):
    r._check_public(None)
  with pytest.raises(ValueError, match='one per stream'):
    r._check_public([np.zeros((1, 2))])
  with pytest.raises(ValueError, match='max_public_dets'):
    r._check_public([np.zeros((9, 2)), np.zeros((0, 2))])
  with pytest.raises(ValueError, match=r'\[P, 2\]'):
    r._check_public([np.zeros((3, 3)), np.zeros((0, 2))])
  got = r._check_public([np.ones((8, 2)), []])
  assert [a.shape for a in got] == [(8, 2), (0, 2)] and got[0].dtype == np.float32
  r.public = False
  with pytest.raises(ValueError, match='only read'):
    r._check_public([np.zeros((1, 2))] * 2)
