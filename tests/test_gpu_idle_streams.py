"""-m gpu: StreamRunner idle streams.  The mapped track step and render against the identity ones, the engine at a batch
n against the B-image run, and an idle-streams runner against a plain capacity runner fed the same frames (its idle
streams re-fed), bit for bit on every live stream."""
import numpy as np
import pytest
import torch

from centertrack_b200 import _lib as L
from helpers import make_model, make_opt
from test_gpu_camera_switch import _model, _pub
from test_gpu_frames import _frame
from test_gpu_track_payload import LAYOUTS, MODES, _new_objects, _random_records

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')


# ------------------------------------------------------------------------------------------------ kernels
def _state(trk):
  return [t.clone() for t in (trk.tracks, trk.counts, trk.boxes) + ((trk.payload,) if trk.payload is not None else ())]


def _bits(t):
  return t.contiguous().view(torch.int32)


@pytest.mark.parametrize('mode', ['greedy_age3', 'hungarian_age3', 'public_age3', 'public_hungarian_age3'])
@pytest.mark.parametrize('lay', ['plain_2d', 'ddd_amodel_offset', 'pose_refined'])
def test_mapped_track_step_equals_identity_step_on_the_same_streams(lay, mode):
  """B = 6 crowded streams, 7 frames; each frame a random subset of them in a random order (n = 1 and n = B
  included) runs through ct_track_step_mapped with padding (-1) and out-of-range entries; a second tracker runs the
  identity step on all B and has its other streams put back.  Every table is equal bit for bit after every frame, and
  the streams that were not listed are byte-identical to before."""
  from centertrack_b200.device_tracker import DeviceTracker
  if lay == 'plain_2d':
    layout, F = {'reg': (9, 2), 'wh': (11, 2), 'tracking': (13, 2)}, 15
  else:
    layout, F = LAYOUTS[lay]
  B, K, inp_h, inp_w, P = 6, 48, 256, 320, 64
  out_hw = (inp_h // 4, inp_w // 4)
  cfg = 'nuscenes_ddd' if 'dep' in layout else ('coco_pose' if 'hps' in layout else 'mot')
  opt = make_opt(cfg, ['--track_thresh', '0.2', '--new_thresh', '0.4', '--input_h', str(inp_h), '--input_w',
                       str(inp_w)] + MODES[mode])
  rng = np.random.RandomState(17 + 5 * ['plain_2d', 'ddd_amodel_offset', 'pose_refined'].index(lay) + len(mode))
  img_hw = [(240, 320), (300, 260), (256, 320), (200, 300), (320, 320), (256, 256)]
  centers = [np.array([w / 2., h / 2.], np.float32) for h, w in img_hw]
  scales = [max(h, w) * 1.0 for h, w in img_hw]
  calibs = [np.array([[900 + 50 * b, 0, 150 + b, 0], [0, 900 + 50 * b, 120 - b, 0.5], [0, 0, 1, 0.25]], np.float32)
            for b in range(B)]
  mk = lambda: DeviceTracker(opt, B, K, F, layout, inp_h, inp_w, DEV, centers=centers, scales=scales, calibs=calibs,
                             max_public_dets=P)
  ref, got = mk(), mk()
  objs = [_new_objects(rng, K, out_hw) for _ in range(B)]
  subsets = [list(range(B)), [3], None, None, list(range(B)), None, None]
  for frame, sub in enumerate(subsets):
    if sub is None:
      sub = sorted(rng.choice(B, rng.randint(1, B), replace=False).tolist())
    order = rng.permutation(sub).tolist()
    rec = np.stack([_random_records(rng, objs[b], layout, F, K, out_hw) for b in range(B)])
    pub_ct = rng.uniform(0, 320, (B, P, 2)).astype(np.float32)
    pub_n = rng.randint(0, 12, B).astype(np.int32)
    pub = (torch.from_numpy(pub_ct).to(DEV), torch.from_numpy(pub_n).to(DEV)) if ref.public_det else ()
    before = _state(ref)
    ref.step(torch.from_numpy(rec).to(DEV), *pub)      # the identity step, then the unlisted streams put back
    now = [ref.tracks, ref.counts, ref.boxes] + ([ref.payload] if ref.payload is not None else [])
    for t, v in zip(now, before):
      for b in range(B):
        if b not in sub:
          t[b].copy_(v[b])
    n_pad = min(len(order) + 2, B)                     # padding images: -1 and an out-of-range stream
    streams = (order + [-1, 7 if frame % 2 else -5])[:n_pad]
    recs = np.concatenate([rec[order], rng.uniform(0, 1, (n_pad - len(order), K, F)).astype(np.float32)])
    recs[len(order):, :, 0] = np.sort(recs[len(order):, :, 0], axis=1)[:, ::-1]
    g_before = _state(got)
    got.step_mapped(torch.from_numpy(np.ascontiguousarray(recs)).to(DEV),
                    torch.tensor(streams + [-1] * (B - n_pad), dtype=torch.int32, device=DEV), *pub)
    torch.cuda.synchronize()
    for name, a, b_ in zip(('tracks', 'counts', 'boxes', 'payload'), _state(got), _state(ref)):
      assert torch.equal(_bits(a), _bits(b_)), (lay, mode, frame, name)
    for a, v in zip(_state(got), g_before):
      for b in range(B):
        if b not in sub:
          assert torch.equal(_bits(a[b]), _bits(v[b])), (lay, mode, frame, b)
  assert int(ref.counts[:, 0].sum()) > 0


def test_mapped_render_equals_render_of_the_gathered_boxes():
  from centertrack_b200.device_tracker import DeviceTracker
  layout, F = {'reg': (9, 2), 'wh': (11, 2), 'tracking': (13, 2)}, 15
  B, K, inp_h, inp_w = 5, 48, 256, 320
  out_hw = (inp_h // 4, inp_w // 4)
  opt = make_opt('mot', ['--track_thresh', '0.2', '--new_thresh', '0.4', '--pre_thresh', '0.2', '--input_h',
                         str(inp_h), '--input_w', str(inp_w)])
  rng = np.random.RandomState(3)
  trk = DeviceTracker(opt, B, K, F, layout, inp_h, inp_w, DEV)
  objs = [_new_objects(rng, K, out_hw) for _ in range(B)]
  for _ in range(3):
    trk.step(torch.from_numpy(np.stack([_random_records(rng, objs[b], layout, F, K, out_hw) for b in range(B)])).to(DEV))
  lib, T = L.lib(), trk.T
  for live, n_img in (([4, 0, 2], 4), ([1], 1), ([0, 1, 2, 3, 4], 5), ([3, 1], 2)):
    image_of = np.full(B, -1, np.int32)
    image_of[live] = np.arange(len(live))
    got = torch.full((n_img, 1, inp_h, inp_w), 5.0, device=DEV)
    trk.render_mapped(got, torch.from_numpy(image_of).to(DEV))
    gathered = trk.boxes[live].clone()                # rows of stream live[i], relabelled as image i
    gathered[:, :, 0] = torch.arange(len(live), device=DEV, dtype=torch.float32).view(-1, 1)
    want = torch.full((n_img, 1, inp_h, inp_w), -5.0, device=DEV)
    L.check(lib.ct_render_tracks(L.ptr(gathered), len(live) * T, L.ptr(want), n_img, inp_h, inp_w, L.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.equal(_bits(got), _bits(want)), live
    assert float(got[:len(live)].sum()) > 0
    assert not bool(got[len(live):].any())           # padded images come out zero


# ------------------------------------------------------------------------------------------------ engine
@pytest.mark.parametrize('precision', ['bf16', 'bf16x3', 'fp32'])
def test_engine_at_batch_n_equals_the_b_image_run(precision):
  _, model, _ = make_model('coco_tracking')
  model = model.cuda()
  Bn, Hn, Wn = 5, 64, 96
  eng = model.engine_for(Bn, Hn, Wn, DEV, precision)
  g = torch.Generator().manual_seed(11)
  img = torch.randn((Bn, 3, Hn, Wn), generator=g).to(DEV)
  pre = torch.randn((Bn, 3, Hn, Wn), generator=g).to(DEV)
  hm = torch.rand((Bn, 1, Hn, Wn), generator=g).to(DEV)
  full = {h: t.clone() for h, t in eng.forward(img, pre, hm).items()}
  for n in (1, 2, 4):
    out = eng.forward(img[:n].contiguous(), pre[:n].contiguous(), hm[:n].contiguous(), n=n)
    torch.cuda.synchronize()
    for h, t in out.items():
      assert t.shape[0] == n
      assert torch.equal(_bits(t), _bits(full[h][:n])), (precision, n, h)
  with pytest.raises(ValueError, match='batch'):
    eng.forward(img, pre, hm, n=Bn + 1)


# ------------------------------------------------------------------------------------------------ runner
H, W, K, B = 128, 160, 40, 4
S0, S1, S2 = (120, 200), (97, 131), (160, 128)
MAXF = (160, 200)
SIZE = {0: S0, 1: S1, 2: S2, 3: S0}
# per step: (idle streams, starts, seeded starts): n = B, 2, 1, back with starts, n = B, ...
SCHEDULE = [([], [], []), ([1, 3], [], []), ([1, 2, 3], [], []), ([2], [1, 3], [3]), ([], [2], []), ([0], [], []),
            ([3], [0], [0]), ([], [3], [])]


def _idle_runner(model, opt, precision, graph, g):
  from centertrack_b200.runner import StreamRunner
  r = StreamRunner(model, B, H, W, K=K, precision=precision, device='cuda', opt=opt, device_tracking=True,
                   use_graph=graph, frame_sizes=[SIZE[b] for b in range(B)], max_frame_size=MAXF,
                   idle_streams=g)
  r.warm()
  return r


def _seed(b):
  return [{'score': 0.9, 'class': 1, 'bbox': [10. + b, 12., 60., 70. + b]}, {'score': 0.8, 'class': 1,
                                                                               'bbox': [70., 30., 110., 90.]}]


def _grab(r, i, rec):
  return dict(rec=rec, trk=r.h_trk[i].numpy().copy(), cnt=r.h_cnt[i].numpy().copy(),
              pay=r.h_pay[i].numpy().copy() if r.tracker.payload is not None else None)


def _run_schedule(r, public, idle_mode):
  """-> per step {rec, trk, cnt, pay}.  idle_mode: idle streams marked idle (frames None); otherwise re-fed."""
  out, last = [], {}
  for k, (idle, starts, seeded) in enumerate(SCHEDULE):
    xs, pub = [], []
    for b in range(B):
      if b in idle and idle_mode:
        xs.append(None)
        pub.append(None)
        continue
      if b in idle:
        x, p = last[b]
      else:
        x, p = _frame(*SIZE[b], seed=100 * k + b), _pub(100 * k + b, SIZE[b])
        last[b] = (x, p)
      xs.append(x)
      pub.append(p)
    kw = dict(starts=starts or None, pre_dets={b: _seed(b) for b in seeded} or None,
              public_dets=pub if public else None)
    if idle_mode:
      kw['idle'] = idle
    rec = r.step_frames(xs, **kw)
    if k:
      out.append(_grab(r, (k - 1) & 1, rec))
  out.append(_grab(r, (len(SCHEDULE) - 1) & 1, r.fetch()))
  return out


CASES = [('bf16', False, '', 1, True), ('bf16', True, 'public_hungarian', 4, True), ('bf16', False, '', 4, False),
         ('bf16x3', False, 'public_hungarian', 1, True), ('bf16x3', True, '', 4, True),
         ('fp32', True, 'public_hungarian', 1, True), ('fp32', False, '', 4, False)]


@pytest.mark.parametrize('precision,flip,mode,g,graph', CASES,
                         ids=['-'.join(map(str, c)) for c in CASES])
def test_idle_streams_runner_equals_plain_runner_on_live_streams(precision, flip, mode, g, graph):
  extra = (['--flip_test'] if flip else []) + (['--public_det', '--hungarian'] if mode else [])
  opt, model = _model('mot', extra)
  from centertrack_b200.runner import StreamRunner
  plain = StreamRunner(model, B, H, W, K=K, precision=precision, device='cuda', opt=opt, device_tracking=True,
                       use_graph=graph, frame_sizes=[SIZE[b] for b in range(B)], max_frame_size=MAXF)
  plain.warm()
  want = _run_schedule(plain, bool(mode), False)
  del plain
  r = _idle_runner(model, opt, precision, graph, g)
  if graph:
    assert len(r.idle_graphs) == 3 * len(r.batches())
  got = _run_schedule(r, bool(mode), True)
  _compare(got, want)


def _compare(got, want):
  live_seen = 0
  for k, (idle, _, _) in enumerate(SCHEDULE):
    for b in range(B):
      if b in idle:
        assert not got[k]['rec'][b].any(), (k, b)
        prev = got[k - 1]
        for key in ('trk', 'cnt', 'pay'):        # an idle stream's tables stay byte for byte
          if got[k][key] is not None:
            assert np.array_equal(got[k][key][b].view(np.uint32), prev[key][b].view(np.uint32)), (k, b, key)
        continue
      live_seen += int(got[k]['cnt'][b, 0])
      for key in ('rec', 'trk', 'cnt', 'pay'):
        if got[k][key] is not None:
          assert np.array_equal(np.ascontiguousarray(got[k][key][b]).view(np.uint32),
                                np.ascontiguousarray(want[k][key][b]).view(np.uint32)), (k, b, key)
  assert live_seen > 0


def test_idle_streams_runner_payload_equals_plain_runner():
  opt, model = _model('nuscenes_ddd')
  from centertrack_b200.runner import StreamRunner
  plain = StreamRunner(model, B, H, W, K=K, precision='bf16', device='cuda', opt=opt, device_tracking=True,
                       frame_sizes=[SIZE[b] for b in range(B)], max_frame_size=MAXF)
  plain.warm()
  global SCHEDULE
  saved = SCHEDULE
  SCHEDULE = [(i, s, []) for i, s, _ in saved]             # payload head sets take no seeds
  try:
    want = _run_schedule(plain, False, False)
    del plain
    got = _run_schedule(_idle_runner(model, opt, 'bf16', True, 2), False, True)
    assert got[0]['pay'] is not None
    _compare(got, want)
  finally:
    SCHEDULE = saved


def test_track_videos_on_an_idle_streams_runner_yields_the_same_and_computes_less():
  from centertrack_b200.runner import StreamRunner
  from centertrack_b200.videos import Video, track_videos
  opt, model = _model('mot')
  sizes = [S0, S1, S2, S0, S1, S2, S0]
  lengths = [5, 2, 7, 3, 1, 4, 2]

  def videos():
    return [Video(v, [_frame(*sizes[v], seed=1000 * v + i) for i in range(lengths[v])],
                  pre_dets=_seed(v) if v == 3 else None) for v in range(len(sizes))]

  def play(r):
    images = []
    step = r.step_frames

    def counted(*a, **kw):
      out = step(*a, **kw)
      images.append(r._n)
      return out
    r.step_frames = counted
    return list(track_videos(r, videos())), sum(images)

  plain = StreamRunner(model, B, H, W, K=K, precision='bf16', device='cuda', opt=opt, device_tracking=True,
                       frame_sizes=[S0] * B, max_frame_size=MAXF)
  plain.warm()
  want, n_plain = play(plain)
  del plain
  r = StreamRunner(model, B, H, W, K=K, precision='bf16', device='cuda', opt=opt, device_tracking=True,
                   frame_sizes=[S0] * B, max_frame_size=MAXF, idle_streams=1)
  r.warm()
  got, n_idle = play(r)
  assert [(v, f) for v, f, _ in got] == [(v, f) for v, f, _ in want]
  assert len(got) == sum(lengths)
  for (v, f, a), (_, _, b) in zip(got, want):
    assert len(a) == len(b), (v, f)
    for x, y in zip(a, b):
      assert sorted(x) == sorted(y)
      for key in x:
        assert np.array_equal(np.asarray(x[key]), np.asarray(y[key])), (v, f, key)
  assert n_idle < n_plain, (n_idle, n_plain)


def test_idle_streams_runner_past_64_streams_equals_plain_runner():
  """B = 72, g = 8: steps alternate between padded batches <= 64 and 72.  ct_decode's workspace keeps one counter per
  image at its start and its candidates after align256(4 n), so a decode at n <= 64 must not write where the decode
  at 72 keeps the counters of images 64..71: every live stream's records and tables equal the plain runner's."""
  from centertrack_b200.runner import StreamRunner
  opt, model = _model('mot')
  Bx = 72
  # per step: idle streams, starts (every stream idle in the step before starts again)
  sched = [([], []), (list(range(32, 72)), []), ([], list(range(32, 72))), (list(range(0, 72, 7)), []),
           ([5], list(range(0, 72, 7))), (list(range(10, 72)), [5]), ([], list(range(10, 72))),
           (list(range(60, 72)), [])]
  kw = dict(K=K, precision='bf16', device='cuda', opt=opt, device_tracking=True, frame_sizes=[S0] * Bx,
            max_frame_size=MAXF)

  def play(r, idle_mode):
    out, last = [], {}
    for k, (idle, starts) in enumerate(sched):
      xs = []
      for b in range(Bx):
        if b in idle:
          xs.append(None if idle_mode else last[b])
          continue
        last[b] = _frame(*S0, seed=1000 * k + b)
        xs.append(last[b])
      extra = dict(idle=idle) if idle_mode else {}
      rec = r.step_frames(xs, starts=starts or None, **extra)
      if k:
        out.append(_grab(r, (k - 1) & 1, rec))
    out.append(_grab(r, (len(sched) - 1) & 1, r.fetch()))
    return out

  plain = StreamRunner(model, Bx, H, W, **kw)
  plain.warm()
  want = play(plain, False)
  del plain
  r = StreamRunner(model, Bx, H, W, idle_streams=8, **kw)
  r.warm()
  got = play(r, True)
  assert [r.padded_batch(Bx - len(i)) for i, _ in sched] == [72, 32, 72, 64, 72, 16, 72, 64]
  seen = 0
  for k, (idle, _) in enumerate(sched):
    for b in range(Bx):
      if b in idle:
        assert not got[k]['rec'][b].any(), (k, b)
        continue
      seen += int(got[k]['cnt'][b, 0])
      for key in ('rec', 'trk', 'cnt'):
        assert np.array_equal(np.ascontiguousarray(got[k][key][b]).view(np.uint32),
                              np.ascontiguousarray(want[k][key][b]).view(np.uint32)), (k, b, key)
  assert seen > 0
