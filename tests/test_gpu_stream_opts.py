"""-m gpu: per-stream tracker settings (stream_opts, options=).  The _opts kernels against the existing entry points
launched with each stream's own scalars (track step plain / mapped / payload, start boxes, post-process prefixes), and
StreamRunner streams against runners built with each stream's opt_b and fed the same frames.  Everything bit for bit."""
import copy

import numpy as np
import pytest
import torch

from centertrack_b200 import _lib as L
from centertrack_b200.device_tracker import DeviceTracker, resolve_options
from helpers import make_opt
from test_gpu_track_modes import IDENTITY, _public, _records, _tie_stream, _track_rows

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')
K = 32


def _flags(rng):
  """Random per-stream flags: thresholds below and above track_thresh, greedy / Hungarian, private / public births."""
  f = {}
  for k in ('track_thresh', 'out_thresh', 'pre_thresh', 'new_thresh'):
    if rng.uniform() < 0.6:
      f[k] = float(rng.choice([0.2, 0.3, 0.35, 0.45, 0.5, 0.65]))
  if rng.uniform() < 0.7:
    f['max_age'] = int(rng.choice([-1, 1, 2, 3]))
  f['hungarian'] = bool(rng.uniform() < 0.4)
  f['public_det'] = bool(rng.uniform() < 0.4)
  return f


def _opt_b(opt, flags):
  """A copy of opt with a stream's resolved settings: what a runner built with opt_b runs."""
  o = copy.deepcopy(opt)
  for k, v in resolve_options(opt, flags).items():
    setattr(o, k, v)
  return o


def _tracker(opt, B, layout, F, stream_opts=None):
  trk = DeviceTracker(opt, B, K, F, layout, 256, 256, 'cuda', max_public_dets=128, stream_opts=stream_opts)
  trk.trans_out_inv.copy_(torch.tensor([IDENTITY] * B))
  return trk


def _bits(t):
  return t.detach().contiguous().view(torch.int32).cpu()


def _payload_stream(rng, lay, K, frames):
    """Per frame: records [K, F] of a crowded payload stream (test_gpu_track_payload's) and public centres on some of
    its detections (the predicted previous centre, so that they claim)."""
    from test_gpu_track_payload import LAYOUTS as PL, _new_objects, _random_records
    layout, F = PL[lay]
    objs = _new_objects(rng, K, (64, 64))
    out = []
    for _ in range(frames):
      rec = _random_records(rng, objs, layout, F, K, (64, 64))
      t = layout['tracking'][0]
      pub = [{'ct': (rec[i, 2:4] + rec[i, t:t + 2]).astype(np.float32)} for i in range(0, K, 3) if rec[i, 0] > 0.3]
      out.append((rec, pub))
    return out


KERNEL_LAYOUTS = {'plain': ('coco_tracking', None), 'pose': ('coco_pose', 'pose_refined'),
                  'nuscenes': ('nuscenes_ddd', 'ddd_velocity_att')}


@pytest.mark.parametrize('B', [1, 32, 97])
@pytest.mark.parametrize('mapped', [False, True])
@pytest.mark.parametrize('lay', sorted(KERNEL_LAYOUTS))
def test_opts_kernels_equal_each_stream_launched_with_its_own_scalars(B, mapped, lay):
  """ct_track_step_opts, ct_track_restore_opts and ct_track_start_opts on B streams with mixed settings == a
  one-stream tracker per stream built with its opt_b (ct_track_step / _assoc / _payload, ct_track_restore /
  ct_track_start), over closed-loop frames of crowded, tie-heavy records (plain), or of the pose and nuScenes payload
  record layouts: rows, counts, boxes and payload.  On the plain layout also the host Tracker(opt_b), row for row."""
  from centertrack_b200.tracker import Tracker
  from test_gpu_track_payload import LAYOUTS as PL
  cfg, pl = KERNEL_LAYOUTS[lay]
  layout, F = ({'tracking': (9, 2)}, 11) if pl is None else PL[pl]
  rng = np.random.RandomState(4400 + B + 7 * mapped + 31 * len(lay))
  opt = make_opt(cfg, ['--track_thresh', '0.3'])
  flags = [_flags(rng) for _ in range(B)]
  flags[0] = None if B > 1 else flags[0]
  trk = _tracker(opt, B, layout, F, flags)
  refs = [_tracker(_opt_b(opt, f or {}), 1, layout, F) for f in flags]
  hosts = [Tracker(_opt_b(opt, f or {})) for f in flags] if pl is None else None
  for h in hosts or ():
    h.init_track([])
  started = set()
  if pl is None:
    streams = [_tie_stream(b % 12, K, frames=5) for b in range(B)]
  else:
    streams = [_payload_stream(np.random.RandomState(b), pl, K, 5) for b in range(B)]
  for f in range(5):
    if pl is None:
      dets = [st[f][0] for st in streams]
      rec = _records(dets, K)
    else:
      rec = np.stack([st[f][0] for st in streams])
    rec_d = torch.from_numpy(rec).to(DEV)
    pubs = [st[f][1] for st in streams]
    pub = _public(pubs, 128)
    live = sorted(rng.choice(B, max(1, B - B // 3), replace=False).tolist()) if mapped else list(range(B))
    if mapped:
      smap = torch.tensor(live + [-1] * (B - len(live)), dtype=torch.int32, device=DEV)
      trk.step_mapped(rec_d[live].contiguous(), smap, *pub)
    else:
      trk.step(rec_d, *pub)
    for b in live:
      r = refs[b]
      rp = _public([pubs[b]], 128) if r.public_det else ()
      r.step(rec_d[b:b + 1].contiguous(), *rp)
      if hosts is not None and b not in started:
        o = refs[b].opt
        kept = [copy.deepcopy(d) for d in dets[b] if np.float32(d['score']) > np.float32(o.out_thresh)]
        want = hosts[b].step(kept, pubs[b])
        got = r.results(trk.tracks[b:b + 1].cpu().numpy(), trk.counts[b:b + 1].cpu().numpy())[0]
        assert int(trk.counts[b, 1]) == hosts[b].id_count, (f, b)
        assert np.array_equal(_track_rows(got), _track_rows(want)), (f, b)
    if f == 2:                           # restores: each listed stream's own rows back, boxes with its pre_thresh
      back = live[1::4]
      cnt = trk.counts.cpu().numpy()
      ent = torch.tensor([[b, cnt[b, 0], cnt[b, 1]] for b in back], dtype=torch.int32).reshape(-1, 3).to(DEV)
      rows = [trk.tracks[b, :cnt[b, 0]].clone() for b in back]
      pay = [trk.payload[b, :cnt[b, 0]].clone() for b in back] if trk.payload is not None else []
      if back:
        trk.restore_device(ent, len(back), torch.cat(rows), torch.cat(pay) if pay else None)
      for i, b in enumerate(back):
        e = torch.tensor([[0, cnt[b, 0], cnt[b, 1]]], dtype=torch.int32, device=DEV)
        refs[b].restore_device(e, 1, rows[i], pay[i] if pay else None)
    if f == 3:                           # video starts (seeded on 2-D layouts): the boxes use each stream's pre_thresh
      starts = live[::3]
      seeds = {b: [{'score': float(s), 'class': 1, 'bbox': [20. + b % 7, 30., 60., 80. + 3 * i]}
                   for i, s in enumerate((0.25, 0.4, 0.55, 0.7))] for b in starts} if trk.payload is None else None
      trk.start(starts, seeds)
      for b in starts:
        refs[b].start([0], {0: seeds[b]} if seeds else None)
      started |= set(starts)
    torch.cuda.synchronize()
    for b in range(B):
      r = refs[b]
      n = int(r.counts[0, 0])
      assert torch.equal(trk.counts[b].cpu(), r.counts[0].cpu()), (f, b)
      assert torch.equal(_bits(trk.tracks[b, :n]), _bits(r.tracks[0, :n])), (f, b)
      tb, rb = trk.boxes[b, :r.T], r.boxes[0]
      assert torch.equal(_bits(tb[:, 1:]), _bits(rb[:, 1:])), (f, b)
      assert bool((trk.boxes[b, r.T:, 3] < 0).all()), (f, b)
      if trk.payload is not None:
        assert torch.equal(_bits(trk.payload[b, :n]), _bits(r.payload[0, :n])), (f, b)


def test_post_process_opts_keeps_each_streams_prefix():
  """ct_post_process_opts == ct_post_process launched per stream with that stream's out_thresh, mapped and not."""
  from centertrack_b200.device_detections import DeviceDetections
  rng = np.random.RandomState(5)
  opt = make_opt('coco_tracking')
  B, layout, F = 33, {'tracking': (9, 2)}, 11
  outs = [None if b % 4 == 0 else {'out_thresh': float(rng.uniform(0.0, 0.9))} for b in range(B)]
  rec = np.zeros((B, K, F), np.float32)
  rec[:, :, 0] = -np.sort(-rng.uniform(0, 1, (B, K)), axis=1)
  rec[:, :, 2:8] = rng.uniform(0, 60, (B, K, 6))
  rec_d = torch.from_numpy(rec).to(DEV)
  for mapped in (False, True):
    det = DeviceDetections(opt, B, K, F, layout, 64, 64, 'cuda', stream_opts=outs)
    if mapped:
      live = list(range(1, B, 2))
      det.step_mapped(rec_d[live].contiguous(), torch.tensor(live, dtype=torch.int32, device=DEV))
    else:
      live = list(range(B))
      det.step(rec_d)
    for b in live:
      o = copy.deepcopy(opt)
      o.out_thresh = resolve_options(opt, outs[b], ('out_thresh',))['out_thresh']
      ref = DeviceDetections(o, 1, K, F, layout, 64, 64, 'cuda')
      ref.step(rec_d[b:b + 1].contiguous())
      n = int(ref.counts[0])
      assert int(det.counts[b]) == n and n == int((rec[b, :, 0] > np.float32(o.out_thresh)).sum())
      assert torch.equal(_bits(det.dets[b, :n]), _bits(ref.dets[0, :n])), b


# ------------------------------------------------------------------------------------------------ runner
RUN_OPTS = [None, {'hungarian': True, 'max_age': 3}, {'track_thresh': 0.3, 'public_det': True},
            {'pre_thresh': 0.5, 'new_thresh': 0.4, 'max_age': 1}]
CHANGE = (3, 1, {'max_age': 2, 'track_thresh': 0.2})          # (step, stream, options) of a video start


def _runner(opt, model, precision, graph, **kw):
  from centertrack_b200.runner import StreamRunner
  from test_gpu_stream_starts import H, W
  r = StreamRunner(model, len(RUN_OPTS), H, W, K=K, precision=precision, device='cuda', opt=opt, use_graph=graph,
                   device_tracking=True, **kw)
  r.warm()
  return r


def _pub_of(step, b):
  rng = np.random.RandomState(100 * step + b)
  return rng.uniform(0, 96, (int(rng.randint(0, 6)), 2)).astype(np.float32)


@pytest.mark.parametrize('precision', ['bf16', 'bf16x3'])
@pytest.mark.parametrize('graph', [True, False])
def test_runner_streams_equal_runners_built_with_their_opt(precision, graph):
  """A runner with mixed stream_opts (greedy, Hungarian, public births, other thresholds and max_age; a start that
  changes stream 1's settings) against one runner per distinct opt_b fed the same frames and starts: each stream's
  records, track rows, counts and results, after every step."""
  from test_gpu_stream_starts import _image, _model
  opt, model = _model('coco_tracking')
  B = len(RUN_OPTS)
  mixed = _runner(opt, model, precision, graph, stream_opts=RUN_OPTS)
  sets = {b: RUN_OPTS[b] or {} for b in range(B)}
  keys = [repr(sorted(f.items())) for f in list(sets.values()) + [CHANGE[2]]]
  flags = dict(zip(keys, list(sets.values()) + [CHANGE[2]]))
  refs = {k: _runner(_opt_b(opt, f), model, precision, graph) for k, f in flags.items()}
  cur = {b: repr(sorted(sets[b].items())) for b in range(B)}
  for step in range(7):
    img = torch.stack([_image(1000 * step + b) for b in range(B)]).pin_memory()
    kw = {}
    if step == CHANGE[0]:
      kw = dict(starts=[CHANGE[1]])
    pub_all = [_pub_of(step, b) for b in range(B)]
    now = dict(sets)
    if step >= CHANGE[0]:
      now[CHANGE[1]] = CHANGE[2]
    mixed.step_host(img, public_dets=[p if resolve_options(opt, now[b])['public_det'] else None
                                      for b, p in enumerate(pub_all)],
                    options={CHANGE[1]: CHANGE[2]} if step == CHANGE[0] else None, **kw)
    torch.cuda.synchronize()           # the runners share the model's engine: one runner's step at a time
    if step == CHANGE[0]:
      cur[CHANGE[1]] = repr(sorted(CHANGE[2].items()))
    for k, r in refs.items():
      r.step_host(img, public_dets=pub_all if r.public else None, **kw)
      torch.cuda.synchronize()
    rec = mixed.fetch()
    trk, cnt = mixed.fetch_tracks()
    res = mixed.fetch_results()
    for b in range(B):
      r = refs[cur[b]]
      rrec = r.fetch()
      rtrk, rcnt = r.fetch_tracks()
      n = int(rcnt[b, 0])
      assert np.array_equal(rec[b].view(np.int32), rrec[b].view(np.int32)), (step, b)
      assert np.array_equal(cnt[b], rcnt[b]), (step, b)
      assert np.array_equal(trk[b, :n].view(np.int32), rtrk[b, :n].view(np.int32)), (step, b)
      assert len(res[b]) == n and [d['tracking_id'] for d in res[b]] == \
          [d['tracking_id'] for d in r.fetch_results()[b]], (step, b)


def test_default_runner_launches_and_results_unchanged_by_equal_stream_opts():
  """A runner without stream_opts issues as many launches per step as one whose stream_opts all equal opt, and both
  compute the same records and tracks."""
  from test_gpu_stream_starts import _image, _model
  opt, model = _model('coco_tracking', ['--hungarian'])
  from centertrack_b200.runner import StreamRunner
  from test_gpu_stream_starts import H, W
  B = 4
  mk = lambda **kw: StreamRunner(model, B, H, W, K=K, precision='bf16', device='cuda', opt=opt, device_tracking=True,
                                 **kw)
  plain, equal = mk(), mk(stream_opts=[{}] * B)
  plain.warm()
  equal.warm()
  assert plain.launches_per_step == equal.launches_per_step
  for step in range(4):
    img = torch.stack([_image(77 * step + b) for b in range(B)]).pin_memory()
    counts = []
    for r in (plain, equal):
      torch.cuda.synchronize()
      L.lib().ct_reset_launch_count()
      r.step_host(img)
      counts.append(L.lib().ct_launch_count())
      torch.cuda.synchronize()         # the runners share the model's engine: one runner's step at a time
    if step > 0:                                           # replays: one graph launch each
      assert counts[0] == counts[1]
    assert np.array_equal(plain.fetch(), equal.fetch())
    a, b = plain.fetch_tracks(), equal.fetch_tracks()
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[0], b[0])


def test_post_process_runner_with_per_stream_out_thresh():
  """A device_post_process ctdet runner with per-stream out_thresh: each stream's detections equal those of a runner
  built with that out_thresh."""
  from centertrack_b200.runner import StreamRunner
  from test_gpu_post_process import H, W
  from test_gpu_post_process import _model as post_model
  from centertrack_b200 import synthetic as wt
  opt, model = post_model('ctdet')
  outs = [None, {'out_thresh': 0.05}, {'out_thresh': 0.2}]
  B = len(outs)
  mk = lambda o, **kw: StreamRunner(model, B, H, W, K=K, precision='bf16', device='cuda', opt=o,
                                    device_post_process=True, **kw)
  mixed = mk(opt, stream_opts=outs)
  refs = []
  for f in outs:
    o = copy.deepcopy(opt)
    o.out_thresh = resolve_options(opt, f, ('out_thresh',))['out_thresh']
    refs.append(mk(o))
  for step in range(3):
    img = wt.synthetic_inputs(B, H, W, seed=step)[0].contiguous()
    mixed.step_host(img)
    torch.cuda.synchronize()           # the runners share the model's engine: one runner's step at a time
    for r in refs:
      r.step_host(img)
      torch.cuda.synchronize()
    d, c, _ = mixed.fetch_detections()
    for b, r in enumerate(refs):
      rd, rc, _ = r.fetch_detections()
      assert c[b] == rc[b]
      assert np.array_equal(d[b, :c[b]].view(np.int32), rd[b, :rc[b]].view(np.int32)), (step, b)
      assert len(mixed.fetch_results()[b]) == rc[b]


# ------------------------------------------------------------------------------------------------ frames-mode runners
FR_OPTS = [None, {'hungarian': True, 'max_age': 3}, {'public_det': True, 'track_thresh': 0.3},
           {'pre_thresh': 0.5, 'new_thresh': 0.4, 'max_age': 1}]
# per step: (idle, resume, starts with their options)
SCHEDULE = [((), (), {}), ((1,), (), {}), ((1, 3), (), {}), ((), (1, 3), {}), ((0,), (), {}),
            ((), (0,), {2: {'max_age': 1, 'track_thresh': 0.2}}), ((3,), (), {}), ((), (3,), {})]


def _frames_runner(model, o, cfg, stream_opts=None, idle=True):
  from centertrack_b200.runner import StreamRunner
  from test_gpu_stream_resume import MAXF, SIZE
  r = StreamRunner(model, 4, o.input_h, o.input_w, K=K, precision='bf16', device='cuda', opt=o, device_tracking=True,
                   frame_sizes=[SIZE[b] for b in range(4)], max_frame_size=MAXF, idle_streams=True if idle else None,
                   stream_opts=stream_opts)
  r.warm()
  return r


def _tables(r):
  """The last submitted step's (records, tracks, counts, payload) per stream, numpy copies."""
  rec = r.fetch()
  i = (r.t - 1) & 1
  pay = r.h_pay[i].numpy().copy() if r.tracker.payload is not None else None
  return rec, r.h_trk[i].numpy().copy(), r.h_cnt[i].numpy().copy(), pay


def _same_stream(a, w, b, ctx):
  rec, trk, cnt, pay = a
  wrec, wtrk, wcnt, wpay = w
  n = int(wcnt[b, 0])
  assert np.array_equal(rec[b].view(np.int32), wrec[b].view(np.int32)), ctx
  assert np.array_equal(cnt[b], wcnt[b]), ctx
  assert np.array_equal(trk[b, :n].view(np.int32), wtrk[b, :n].view(np.int32)), ctx
  if pay is not None:
    assert np.array_equal(pay[b, :n].view(np.int32), wpay[b, :n].view(np.int32)), ctx


@pytest.mark.parametrize('cfg', ['mot', 'nuscenes_ddd'])
def test_frames_runner_with_idle_resume_start_and_restore_equals_runners_of_each_opt(cfg):
  """step_frames on a capacity idle-streams runner with mixed stream_opts (greedy, Hungarian, public births, other
  thresholds and max_age): idle steps, resumes, and a start that changes a stream's settings, against one runner per
  distinct opt_b fed the same frames, idle lists, resumes and starts -- each live stream's records, tracks, counts and
  payload after every step.  Then stream 1's StreamState is restored, with its options, into stream 2 of another mixed
  runner, and continues there as it does on a runner built with its opt_b."""
  from test_gpu_frames import _frame
  from test_gpu_stream_resume import SIZE, _model
  opt, model = _model(cfg)
  mixed = _frames_runner(model, opt, cfg, FR_OPTS)
  refs = {}

  def ref(o):
    key = repr(sorted(o.items()))
    if key not in refs:
      refs[key] = _frames_runner(model, _opt_b(opt, o), cfg)
    return key

  cur = {b: ref(FR_OPTS[b] or {}) for b in range(4)}
  for _, _, st in SCHEDULE:
    for o in st.values():
      ref(o)
  for k, (idle, resume, starts) in enumerate(SCHEDULE):
    for b, o in starts.items():
      cur[b] = ref(o)
    xs = [None if b in idle else _frame(*SIZE[b], seed=1000 * b + k) for b in range(4)]
    pubs = [np.random.RandomState(100 * k + b).uniform(0, 100, (3, 2)).astype(np.float32) for b in range(4)]
    now = [resolve_options(opt, FR_OPTS[b]) for b in range(4)]
    for s in range(k + 1):
      for b, o in SCHEDULE[s][2].items():
        now[b] = resolve_options(opt, o)
    kw = dict(idle=list(idle), resume=list(resume), starts=sorted(starts) or None)
    mixed.step_frames(xs, public_dets=[p if now[b]['public_det'] and b not in idle else None
                                       for b, p in enumerate(pubs)], options=starts or None, **kw)
    torch.cuda.synchronize()           # the runners share the model's engine: one runner's step at a time
    for r in refs.values():
      r.step_frames(xs, public_dets=[None if b in idle else p for b, p in enumerate(pubs)] if r.public else None, **kw)
      torch.cuda.synchronize()
    got = _tables(mixed)
    for b in range(4):
      if b not in idle:
        _same_stream(got, _tables(refs[cur[b]]), b, (cfg, k, b))
  # stream 1's video moves, with its settings, to stream 2 of a runner whose own entry for stream 2 differs
  st_m, st_r = mixed.stream_state(1), refs[cur[1]].stream_state(1)
  assert st_m.options == st_r.options == resolve_options(opt, FR_OPTS[1])
  C = _frames_runner(model, opt, cfg, [None, None, {'max_age': 3, 'track_thresh': 0.5}, None], idle=False)
  RC = _frames_runner(model, _opt_b(opt, FR_OPTS[1]), cfg, idle=False)
  for k in range(3):
    xs = [_frame(*SIZE[b], seed=7000 + 10 * k + b) for b in range(4)]
    xs[2] = _frame(*SIZE[1], seed=1000 + len(SCHEDULE) + k)
    for r, st in ((C, st_m), (RC, st_r)):
      r.step_frames(xs, restore={2: st} if k == 0 else None)
      torch.cuda.synchronize()
    _same_stream(_tables(C), _tables(RC), 2, (cfg, 'restore', k))
  assert C.tracker.options[2] == st_m.options


def test_track_videos_with_per_video_options_equals_runners_of_each_opt():
  """track_videos on a mot capacity runner whose videos bring options: --public_det --hungarian on some videos only,
  the others the runner's opt.  Every frame's results equal those of track_videos of the same videos on a runner
  built with that video's opt."""
  from centertrack_b200.videos import Video, track_videos
  from test_gpu_frames import _frame
  from test_gpu_stream_resume import SIZE, _model
  opt, model = _model('mot')
  pub_opts = {'public_det': True, 'hungarian': True}
  spec = [(SIZE[0], 3, False), (SIZE[1], 2, True), (SIZE[2], 4, False), (SIZE[3], 2, True), (SIZE[0], 3, True),
          (SIZE[1], 3, False)]

  def vids(which):
    out = []
    for v, (s, n, public) in enumerate(spec):
      if which is not None and public != which:
        continue
      rng = np.random.RandomState(v)
      pd = [rng.uniform(0, 100, (4, 2)).astype(np.float32) for _ in range(n)] if public else None
      out.append(Video(v, [_frame(s[0], s[1], 50 * v + i) for i in range(n)], public_dets=pd,
                       options=pub_opts if public else None))
    return out

  mixed = _frames_runner(model, opt, 'mot', [pub_opts] + [None] * 3, idle=False)
  got = {(v, i): res for v, i, res in track_videos(mixed, vids(None))}
  assert sorted(got) == sorted((v, i) for v, (_, n, _) in enumerate(spec) for i in range(n))
  for public in (False, True):
    r = _frames_runner(model, _opt_b(opt, pub_opts) if public else opt, 'mot', idle=False)
    vs = vids(public)
    for v in vs:                 # a runner built with the video's opt, without stream_opts
      v.options = None
    want = {(v, i): res for v, i, res in track_videos(r, vs)}
    for key, w in want.items():
      a = got[key]
      assert len(a) == len(w), key
      for x, y in zip(a, w):
        for k in x:
          assert np.array_equal(np.asarray(x[k]), np.asarray(y[k])), (key, k)
