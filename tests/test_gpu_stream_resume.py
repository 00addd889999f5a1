"""-m gpu: idle StreamRunner streams that resume their video, and videos moved between streams and runners
(stream_state, restore).  ct_track_restore against the track step and ct_track_start; a resuming idle-streams runner
against a plain capacity runner fed each stream's delivered frames one after the other; a restored stream against the
stream that ran the whole video; launches and uploads of later steps unchanged.  Everything bit for bit."""
import copy

import numpy as np
import pytest
import torch

from centertrack_b200 import _lib as L
from helpers import make_opt
from test_gpu_camera_switch import _model, _pub
from test_gpu_frames import _frame
from test_gpu_idle_streams import _seed
from test_gpu_track_payload import LAYOUTS, _new_objects, _random_records
from yuv_oracle import bgr_to_yuv420

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')
K = 40
MAXF = (160, 200)
SIZE = {0: (120, 200), 1: (96, 130), 2: (160, 128), 3: (120, 200)}   # even: every format takes them
B = 4
# per stream: whether it has a frame in each step.  Idle runs of 1-4 steps; step 3 resumes 0 and 3 (1, 2 idle), step 4
# resumes 1 and 2, step 7 resumes 0 and 3 while 2 starts a video and 1 is idle
MASK = np.array([[1, 1, 0, 1, 1, 0, 0, 1, 1, 1, 1, 1],
                 [1, 0, 0, 0, 1, 1, 1, 0, 0, 0, 0, 1],
                 [1, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1, 1],
                 [1, 1, 0, 1, 1, 1, 0, 1, 0, 1, 1, 0]], bool)
STARTS = {(7, 2)}                                            # (step, stream)


def _bits(a):
  return np.ascontiguousarray(a).view(np.uint32)


def _tbits(t):
  return t.contiguous().view(torch.int32)


# ------------------------------------------------------------------------------------------------ ct_track_restore
def _tracker(opt, layout, F, n_streams, inp, geo):
  from centertrack_b200.device_tracker import DeviceTracker
  centers, scales = geo
  return DeviceTracker(opt, n_streams, K, F, layout, inp[0], inp[1], DEV, centers=centers, scales=scales)


@pytest.mark.parametrize('lay', ['plain_2d', 'ddd_amodel_offset', 'pose_refined'])
def test_track_restore_writes_the_rows_the_track_step_wrote(lay):
  if lay == 'plain_2d':
    layout, F = {'reg': (9, 2), 'wh': (11, 2), 'tracking': (13, 2)}, 15
  else:
    layout, F = LAYOUTS[lay]
  cfg = 'nuscenes_ddd' if 'dep' in layout else ('coco_pose' if 'hps' in layout else 'mot')
  inp = (256, 320)
  out_hw = (inp[0] // 4, inp[1] // 4)
  opt = make_opt(cfg, ['--track_thresh', '0.2', '--new_thresh', '0.4', '--pre_thresh', '0.2', '--max_age', '3',
                       '--input_h', str(inp[0]), '--input_w', str(inp[1])])
  Bn = 5
  img_hw = [(240, 320)] * Bn                                 # one camera: the boxes depend on the stream index only
  geo = ([np.array([w / 2., h / 2.], np.float32) for h, w in img_hw], [max(h, w) * 1.0 for h, w in img_hw])
  rng = np.random.RandomState(7 + len(lay))
  src = _tracker(opt, layout, F, Bn, inp, geo)
  objs = [_new_objects(rng, K, out_hw) for _ in range(Bn)]
  for _ in range(4):
    src.step(torch.from_numpy(np.stack([_random_records(rng, objs[b], layout, F, K, out_hw) for b in range(Bn)])).to(DEV))
  torch.cuda.synchronize()
  s = 3
  n, ids = (int(v) for v in src.counts[s].cpu())
  assert n > 0 and ids >= n
  dst = _tracker(opt, layout, F, Bn, inp, geo)
  for _ in range(2):                                         # other contents to overwrite and to keep
    dst.step(torch.from_numpy(np.stack([_random_records(rng, objs[b], layout, F, K, out_hw) for b in range(Bn)])).to(DEV))
  tables = lambda t: [t.tracks, t.counts, t.boxes] + ([t.payload] if t.payload is not None else [])
  for target in (s, 1):
    before = [x.clone() for x in tables(dst)]
    ent = torch.tensor([[-1, n, ids], [target, n, ids], [Bn, n, ids]], dtype=torch.int32, device=DEV)
    rows = torch.cat([src.tracks[s, :n]] * 3)                # out-of-range entries (-1, B) write nothing
    pay = torch.cat([src.payload[s, :n]] * 3) if src.payload is not None else None
    dst.restore_device(ent, 3, rows, pay)
    torch.cuda.synchronize()
    for name, a, b_, old in zip(('tracks', 'counts', 'boxes', 'payload'), tables(dst), tables(src), before):
      want = b_[s].clone()
      if name == 'boxes':
        want[:, 0] = float(target)                           # column 0: the stream index
      assert torch.equal(_tbits(a[target]), _tbits(want)), (lay, target, name)
      for o in range(Bn):
        if o != target:
          assert torch.equal(_tbits(a[o]), _tbits(old[o])), (lay, target, name, o)
    assert bool((dst.boxes[target, :n, 3] >= 0).any())


def test_track_restore_of_fresh_ids_equals_track_start():
  """Rows with ids 1..n, age 1 and active 1 restored with id_count n: the tables ct_track_start writes from them."""
  from centertrack_b200.device_tracker import seed_rows
  layout, F = {'reg': (9, 2), 'wh': (11, 2), 'tracking': (13, 2)}, 15
  inp = (256, 320)
  opt = make_opt('mot', ['--new_thresh', '0.4', '--pre_thresh', '0.2', '--input_h', str(inp[0]), '--input_w',
                         str(inp[1])])
  geo = ([np.array([160., 120.], np.float32)] * 3, [320.] * 3)
  items = [{'score': 0.9 - 0.1 * i, 'class': 1, 'bbox': [10. + 20 * i, 12., 60. + 20 * i, 70. + 5 * i]}
           for i in range(5)]
  rows = seed_rows(items, opt.new_thresh)
  n = len(rows)
  a, b = _tracker(opt, layout, F, 3, inp, geo), _tracker(opt, layout, F, 3, inp, geo)
  a.start([1], {1: items})
  b.restore_device(torch.tensor([[1, n, n]], dtype=torch.int32, device=DEV), 1, torch.from_numpy(rows).to(DEV))
  torch.cuda.synchronize()
  for x, y in zip((a.tracks, a.counts, a.boxes), (b.tracks, b.counts, b.boxes)):
    assert torch.equal(_tbits(x), _tbits(y))


# ------------------------------------------------------------------------------------------------ resume
def _src(fmt, b, k):
  x = _frame(*SIZE[b], seed=1000 * b + k)
  return x if fmt == 'bgr' else bgr_to_yuv420(x, fmt)


def _make(cfg, mode, precision, graph, flip, fmt, idle):
  extra = (['--flip_test'] if flip else []) + {'': [], 'hungarian': ['--hungarian'], 'public': ['--public_det']}[mode]
  if cfg == 'ctdet':
    from test_gpu_post_process import _model as post_model
    opt, model = post_model('ctdet', extra)
  else:
    opt, model = _model(cfg, extra)
  from centertrack_b200.runner import StreamRunner
  r = StreamRunner(model, B, opt.input_h, opt.input_w, K=K, precision=precision, device='cuda', opt=opt,
                   device_tracking=cfg != 'ctdet', device_post_process=cfg == 'ctdet', use_graph=graph,
                   frame_sizes=[SIZE[b] for b in range(B)], max_frame_size=MAXF, frame_format=fmt,
                   idle_streams=True if idle else None)
  r.warm()
  return r


def _snap(r):
  """The last submitted step's tables, per stream."""
  rec = r.fetch()
  if r.post is not None:
    dets, cnt, pay = r.fetch_detections()
    return [(rec[b], dets[b], cnt[b], pay[b] if pay is not None else None) for b in range(B)]
  i = (r.t - 1) & 1
  trk, cnt = r.h_trk[i].numpy(), r.h_cnt[i].numpy()
  pay = r.h_pay[i].numpy() if r.tracker.payload is not None else None
  return [(rec[b], trk[b].copy(), cnt[b].copy(), pay[b].copy() if pay is not None else None) for b in range(B)]


def _feed(r, xs, form, **kw):
  if form == 'buffers':
    views = r.frame_buffers()
    for v, x in zip(views, xs):
      if x is not None:
        v[...] = x
    return r.step_frames(None, **kw)
  if form == 'device':
    xs = [torch.from_numpy(x).to(DEV) if x is not None else None for x in xs]
  return r.step_frames(xs, **kw)


def _seeds(r, k):
  """pre_dets of every stream's first frame on 2-D head sets: tracks exist from the start (public births are rare)."""
  if k or r.tracker is None or r.tracker.payload is not None:
    return {}
  return dict(starts=list(range(B)), pre_dets={b: _seed(b) for b in range(B)})


def _play_idle(r, fmt, form, public):
  """-> {(stream, k): its tables after its k-th delivered frame}."""
  out, count = {}, [0] * B
  for step in range(MASK.shape[1]):
    live = [b for b in range(B) if MASK[b, step]]
    idle = [b for b in range(B) if b not in live]
    starts = [b for b in live if (step, b) in STARTS]
    resume = [b for b in live if step and not MASK[b, step - 1]]
    xs = [_src(fmt, b, count[b]) if b in live else None for b in range(B)]
    pub = [_pub(1000 * b + count[b], SIZE[b]) if b in live else None for b in range(B)]
    kw = _seeds(r, step) or dict(starts=starts or None)
    _feed(r, xs, form, idle=idle, resume=resume or None, public_dets=pub if public else None, **kw)
    snap = _snap(r)
    for b in live:
      out[(b, count[b])] = snap[b]
      count[b] += 1
  return out


def _play_plain(r, fmt, public):
  """Each stream's delivered frames one after the other, its start at the same frame of its video."""
  n = int(MASK.sum(1).max())
  starts = {(int(MASK[b, :s].sum()), b) for s, b in STARTS}
  out = {}
  for k in range(n):
    xs = [_src(fmt, b, k) for b in range(B)]
    pub = [_pub(1000 * b + k, SIZE[b]) for b in range(B)]
    st = [b for b in range(B) if (k, b) in starts]
    kw = _seeds(r, k) or dict(starts=st or None)
    r.step_frames(xs, public_dets=pub if public else None, **kw)
    for b, s in enumerate(_snap(r)):
      out[(b, k)] = s
  return out


CASES = [('mot', '', 'bf16', True, False, 'bgr', 'array'), ('mot', 'hungarian', 'bf16', False, True, 'nv12', 'buffers'),
         ('mot', 'public', 'bf16x3', True, True, 'i420', 'device'), ('mot', '', 'fp32', True, False, 'bgr', 'device'),
         ('mot', 'public', 'fp32', False, True, 'nv12', 'array'),
         ('mot', 'hungarian', 'bf16x3', False, False, 'i420', 'array'),
         ('nuscenes_ddd', '', 'bf16', True, False, 'bgr', 'array'), ('coco_pose', '', 'bf16x3', True, True, 'i420', 'buffers'),
         ('ctdet', '', 'bf16', True, False, 'nv12', 'device')]


@pytest.mark.parametrize('cfg,mode,precision,graph,flip,fmt,form', CASES, ids=['-'.join(map(str, c)) for c in CASES])
def test_resumed_streams_equal_streams_fed_only_their_frames(cfg, mode, precision, graph, flip, fmt, form):
  plain = _make(cfg, mode, precision, graph, flip, fmt, idle=False)
  want = _play_plain(plain, fmt, mode == 'public')
  del plain
  got = _play_idle(_make(cfg, mode, precision, graph, flip, fmt, idle=True), fmt, form, mode == 'public')
  seen = 0
  for key, g in sorted(got.items()):
    for i, (a, w) in enumerate(zip(g, want[key])):
      if a is not None:
        assert np.array_equal(_bits(a), _bits(w)), (key, ('rec', 'tables', 'counts', 'payload')[i])
    seen += int(np.asarray(g[2]).ravel()[0])
  assert seen > 0
  if cfg != 'ctdet' and mode != 'public':                    # track ids carry over from frame to frame
    ids = lambda b, k: set(got[(b, k)][1][:int(got[(b, k)][2][0]), L.CT_TRK_ID].astype(int))
    assert sum(len(ids(b, k - 1) & ids(b, k)) for b, k in got if k) > 0


def test_later_steps_launch_and_upload_what_they_would_without_resume_or_restore():
  """Two idle-streams runners take the same steps but for step 2, where one resumes stream 1 and restores stream 3 (from
  stream 0's state) and the other starts both.  Every later step makes the same launches and uploads the same bytes."""
  opt, model = _model('mot')
  from centertrack_b200.runner import StreamRunner
  lib = L.lib()

  def run(r, moved):
    xs = lambda k, s3=SIZE[3]: [_frame(*(SIZE[b] if b != 3 else s3), seed=10 * k + b) for b in range(B)]
    r.step_frames(xs(0))
    r.step_frames([x if b != 1 else None for b, x in enumerate(xs(1))], idle=[1])
    kw = dict(resume=[1], restore={3: r.stream_state(0)}) if moved else dict(starts=[1, 3])
    r.step_frames(xs(2, SIZE[0]), **kw)
    seen = []
    for k in range(3, 7):
      n0 = lib.ct_launch_count()
      r.step_frames(xs(k, SIZE[0]), idle=[2] if k == 5 else None, resume=[2] if k == 6 and moved else None,
                    starts=[2] if k == 6 and not moved else None)
      seen.append((lib.ct_launch_count() - n0, r.h2d_bytes_per_step))
    r.fetch()
    return seen[:-1]                                         # the last step differs by design (resume against start)

  mk = lambda: StreamRunner(model, B, opt.input_h, opt.input_w, K=K, precision='bf16', device='cuda', opt=opt,
                            device_tracking=True, frame_sizes=[SIZE[b] for b in range(B)], max_frame_size=MAXF,
                            idle_streams=True)
  a, b = mk(), mk()
  a.warm()
  b.warm()
  assert run(a, True) == run(b, False)


# ------------------------------------------------------------------------------------------------ restore
V_LEN, T_EXPORT = 9, 4


def _video(k):
  return _frame(*SIZE[1], seed=500 + k)


@pytest.mark.parametrize('precision', ['bf16', 'fp32'])
def test_restored_stream_equals_the_stream_that_ran_the_whole_video(precision):
  """Stream 5 of runner A (B = 8) plays a video and exports after frame T_EXPORT; from the next frame on the video
  continues on stream 5, on A's stream 1, on stream 2 of a B = 4 runner (restored in its third step) and on stream 2 of
  a B = 4 idle-streams runner (restored in its first step, idle in a later one), and on another GPU when there is one.
  Every copy's records, tracks (ids, ages, active) and counts equal stream 5's."""
  from centertrack_b200.runner import StreamRunner
  opt, model = _model('mot')
  kw = dict(K=K, precision=precision, device='cuda', opt=opt, device_tracking=True, max_frame_size=MAXF)
  sizes8 = [SIZE[b % 4] for b in range(8)]
  sizes8[5] = SIZE[1]
  A = StreamRunner(model, 8, opt.input_h, opt.input_w, frame_sizes=sizes8, **kw)
  Bp = StreamRunner(model, B, opt.input_h, opt.input_w, frame_sizes=[SIZE[b] for b in range(B)], **kw)
  Bi = StreamRunner(model, B, opt.input_h, opt.input_w, frame_sizes=[SIZE[b] for b in range(B)], idle_streams=True,
                    **kw)
  others = [(Bp, 2, 2, None), (Bi, 2, 0, 3)]                # (runner, stream, steps before the restore, an idle step)
  if torch.cuda.device_count() > 1:
    m1 = copy.deepcopy(model).to('cuda:1')
    kw1 = dict(kw, device='cuda:1')
    with torch.cuda.device(1):
      others.append((StreamRunner(m1, B, opt.input_h, opt.input_w, frame_sizes=[SIZE[b] for b in range(B)], **kw1), 1, 1,
                     None))
  for r in [A] + [o[0] for o in others]:
    r.warm()
  want, state = {}, None
  for k in range(V_LEN):
    xs = [_frame(*sizes8[b], seed=10 * k + b) for b in range(8)]
    xs[5] = _video(k)
    extra = {}
    if k > T_EXPORT:
      xs[1] = _video(k)
      if k == T_EXPORT + 1:
        extra = dict(restore={1: state})
    A.step_frames(xs, **extra)
    snap = _snap_n(A, 8)
    want[k] = snap[5]
    if k > T_EXPORT:
      _same(snap[1], snap[5], ('A', 1, k))
    if k == T_EXPORT:
      state = A.stream_state(5)
      assert state.counts[0] > 0 and state.frame.shape == SIZE[1] + (3,)
  for r, s, pre, idle_at in others:
    dev = r.u8[0].device
    with torch.cuda.device(dev):
      for j in range(pre):
        r.step_frames([_frame(*SIZE[b], seed=77 * j + b) for b in range(B)])
      for k in range(T_EXPORT + 1, V_LEN):
        xs = [_frame(*SIZE[b], seed=33 * k + b) for b in range(B)]
        xs[s] = _video(k)
        extra = dict(restore={s: state}) if k == T_EXPORT + 1 else {}
        if idle_at is not None and k == T_EXPORT + 1 + idle_at:
          xs[0], extra = None, dict(idle=[0])
        r.step_frames(xs, **extra)
        _same(_snap_n(r, B)[s], want[k], (r.B, s, k))


def _snap_n(r, n):
  """Per stream: records, its counts[0] track rows (the rows past them hold whatever the table held before), counts."""
  rec = r.fetch()
  i = (r.t - 1) & 1
  trk, cnt = r.h_trk[i].numpy(), r.h_cnt[i].numpy()
  return [(rec[b], trk[b, :cnt[b, 0]].copy(), cnt[b].copy()) for b in range(n)]


def _same(a, w, ctx):
  for i, (x, y) in enumerate(zip(a, w)):
    assert np.array_equal(_bits(x), _bits(y)), (ctx, ('rec', 'tracks', 'counts')[i])
