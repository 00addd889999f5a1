"""-m gpu: StreamRunner streams that change their source frame size and camera at a video start (max_frame_size):
the batched frame warp against the per-stream one bit for bit, invalid descriptors, and a capacity runner's tracks
against a fresh fixed-size runner playing each video alone."""
import ctypes as C

import numpy as np
import pytest
import torch

from centertrack_b200 import _lib as L
from helpers import make_model, make_opt
from test_gpu_frames import _frame, _ragged

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')
STREAMS = [(1080, 1920, 5760), (480, 640, 1920), (375, 1242, 3726), (544, 960, 2880), (301, 457, 1392)]


def _mean_std(opt):
  from centertrack_b200.dataset_info import get_dataset
  ds = get_dataset(opt.dataset)
  mean = np.ascontiguousarray(ds.mean, np.float32).reshape(3)
  std = np.ascontiguousarray(ds.std, np.float32).reshape(3)
  return mean, std


def _dev_frames(frames):
  return torch.from_numpy(np.frombuffer(bytes(frames), np.uint8).copy()).to(DEV)


def test_warp_frames_normalize_equals_per_stream_warp_bit_for_bit():
  H, W = 544, 960
  opt = make_opt('mot')
  mean, std = _mean_std(opt)
  ms = C.c_void_p(mean.ctypes.data), C.c_void_p(std.ctypes.data)
  B = len(STREAMS)
  cur, _, frames, minv = _ragged(opt, STREAMS, 5)
  lib, st = L.lib(), L.stream_ptr()
  ref = torch.full((B, 3, H, W), 3.0, device=DEV)
  got = torch.full((B, 3, H, W), -3.0, device=DEV)
  for b, f in enumerate(frames):
    L.check(lib.ct_warp_affine_normalize(C.c_void_p(cur.data_ptr() + f.offset), 1, f.h, f.w, f.step, L.ptr(minv[b]),
                                         *ms, L.ptr(ref[b]), H, W, st))
  L.check(lib.ct_warp_frames_normalize(L.ptr(cur), L.ptr(_dev_frames(frames)), B, cur.numel(), *ms, L.ptr(got), H, W,
                                       st))
  torch.cuda.synchronize()
  assert torch.equal(got.view(torch.int32), ref.view(torch.int32))


def test_invalid_descriptors_give_zeros_and_read_nothing():
  """buf_bytes is smaller than the allocation, so a faulty bound shows as wrong bytes rather than a bad access."""
  H, W = 64, 96
  opt = make_opt('mot', ['--input_h', str(H), '--input_w', str(W)])
  mean, std = _mean_std(opt)
  ms = C.c_void_p(mean.ctypes.data), C.c_void_p(std.ctypes.data)
  streams = [(40, 60, 180), (40, 60, 180), (40, 60, 180), (40, 60, 180), (40, 60, 180), (40, 60, 180), (40, 60, 180)]
  cur, prev, frames, _ = _ragged(opt, streams, 9)
  limit = frames[4].offset + 39 * 180 + 180          # stream 4 ends exactly at the bound: valid
  frames[1].h = 0
  frames[2].w = -3
  frames[3].step = 179                                # < 3 w
  frames[5].offset = limit - 39 * 180 - 179           # one byte past the bound
  frames[6].offset = -16
  bad = [1, 2, 3, 5, 6]
  dfr = _dev_frames(frames)
  B, lib, st = len(streams), L.lib(), L.stream_ptr()
  hm = torch.rand((B, 1, H, W), device=DEV)
  for fn, n in ((lib.ct_pack_stem_frames_dev, B), (lib.ct_pack_stem_frames_flip_dev, 2 * B)):
    got = torch.full((n, H, W, 8), -7.0, dtype=torch.bfloat16, device=DEV)
    L.check(fn(L.ptr(cur), L.ptr(prev), L.ptr(dfr), B, limit, *ms, L.ptr(hm), L.ptr(got), H, W, st))
    torch.cuda.synchronize()
    for b in range(B):
      zero = not bool(got[b].view(torch.int16).any())
      assert zero == (b in bad), b
      if n > B:
        assert bool(torch.equal(got[B + b], got[b].flip(1)))
  img = torch.full((B, 3, H, W), -3.0, device=DEV)
  L.check(lib.ct_warp_frames_normalize(L.ptr(cur), L.ptr(dfr), B, limit, *ms, L.ptr(img), H, W, st))
  torch.cuda.synchronize()
  for b in range(B):
    assert (not bool(img[b].view(torch.int32).any())) == (b in bad), b


# ------------------------------------------------------------------------------------------------ the runner
H, W, K, B = 128, 160, 40, 2
S0, S1, S2 = (120, 200), (97, 131), (160, 128)
MAXF = (160, 200)
# per stream: videos (size, first step, length); stream 0 goes S0 -> S1, stream 1 S2 -> S0 -> S1
VIDEOS = {0: [(S0, 0, 3), (S1, 3, 4)], 1: [(S2, 0, 2), (S0, 2, 2), (S1, 4, 3)]}
STEPS = 7


def _model(cfg, extra=()):
  opt, model, _ = make_model(cfg, extra=['--track_thresh', '0.1', '--new_thresh', '0.1', '--pre_thresh', '0.1',
                                         '--input_h', str(H), '--input_w', str(W), '--max_age', '2'] + list(extra))
  if cfg == 'nuscenes_ddd':
    with torch.no_grad():
      model.state_dict()['wh.2.bias'].fill_(3.0)
  return opt, model.cuda()


def _runner(model, opt, precision, sizes, graph, max_frame_size=None, calibs=None):
  from centertrack_b200.runner import StreamRunner
  r = StreamRunner(model, B, H, W, K=K, precision=precision, device='cuda', opt=opt, device_tracking=True,
                   use_graph=graph, frame_sizes=sizes, max_frame_size=max_frame_size, calibs=calibs)
  r.warm()
  return r


def _pub(key, size):
  """Public detection centres over the whole frame (a 10-pixel grid, jittered per frame): tracks can be born anywhere."""
  rng = np.random.RandomState(key)
  ys, xs = np.mgrid[0:size[0]:10, 0:size[1]:10]
  ct = np.stack([xs.ravel(), ys.ravel()], 1).astype(np.float32)
  return ct + rng.uniform(0, 5, ct.shape).astype(np.float32)


def _play(r, feed, graphs=None, launches=None):
  """feed: per step (frames, starts, public, calibs) -> per step {rec, trk, cnt, pay} of each stream.  launches: a list
  that receives the library launches (ct_launch_count) each step_frames call made on this thread."""
  out = []
  lib = L.lib()

  def grab(i, rec):
    return dict(rec=rec, trk=r.h_trk[i].numpy().copy(), cnt=r.h_cnt[i].numpy().copy(),
                pay=r.h_pay[i].numpy().copy() if r.tracker.payload is not None else None)

  for k, (x, starts, pub, cal) in enumerate(feed):
    n0 = lib.ct_launch_count()
    rec = r.step_frames(x, starts=starts, public_dets=pub, calibs=cal)
    if launches is not None:
      launches.append(lib.ct_launch_count() - n0)
    if graphs is not None:
      assert [id(g) for g in r.graphs] == graphs, k
    if k:
      out.append(grab((k - 1) & 1, rec))
  out.append(grab((len(feed) - 1) & 1, r.fetch()))
  return out


def _same(a, b, s, ctx):
  for k in ('rec', 'trk', 'cnt', 'pay'):
    if a[k] is not None:
      assert np.array_equal(np.ascontiguousarray(a[k][s]).view(np.uint32),
                            np.ascontiguousarray(b[k][s]).view(np.uint32)), (ctx, k)


def _switch_feed(public, calib_of=None):
  feed = []
  for t in range(STEPS):
    xs, starts, pub, cal = [], [], [], {}
    for b, vids in VIDEOS.items():
      for v, (size, t0, n) in enumerate(vids):
        if t0 <= t < t0 + n:
          xs.append(_frame(size[0], size[1], 1000 * b + 100 * v + t - t0))
          pub.append(_pub(1000 * b + 100 * v + t - t0, size))
          if t == t0 and t > 0:
            starts.append(b)
            if calib_of is not None:
              cal[b] = calib_of(b, v)
    feed.append((xs, starts or None, pub if public else None, cal or None))
  return feed


CASES = [('bf16', True, False, False), ('bf16', False, True, False), ('bf16x3', True, True, True),
         ('bf16x3', False, False, False), ('bf16', True, False, True)]


@pytest.mark.parametrize('precision,graph,flip,public', CASES,
                         ids=['%s-%s-%s-%s' % (p, 'graph' if g else 'eager', 'flip' if f else 'noflip',
                                               'public' if u else 'greedy') for p, g, f, u in CASES])
def test_size_switches_equal_a_fresh_fixed_runner(precision, graph, flip, public):
  extra = (['--flip_test'] if flip else []) + (['--public_det', '--hungarian'] if public else [])
  opt, model = _model('coco_tracking', extra)
  feed = _switch_feed(public)
  r = _runner(model, opt, precision, [S0, S2], graph, MAXF)
  graphs, counted = [id(g) for g in r.graphs], []
  got = _play(r, feed, graphs if graph else None, counted)
  assert [r.meta(b)['width'] for b in range(B)] == [S1[1], S1[1]]
  if graph:                                    # after the first (eager) step: one replay of a slot's graph
    assert all(n == 0 for t, n in enumerate(counted) if t and not feed[t][1]), counted
  else:                                        # eager: the launches of a step without starts, before and after switches
    plain = {n for t, n in enumerate(counted) if not feed[t][1]}
    assert len(plain) == 1, counted
  cap_launches = r.launches_per_step
  del r
  if not public:      # --public_det births tracks only at public centres: the records below carry that case
    assert sum(int(got[t]['cnt'][b, 0]) for t in range(STEPS) for b in range(B)) > 0
  for b, vids in VIDEOS.items():
    for v, (size, t0, n) in enumerate(vids):
      fresh = _runner(model, opt, precision, [size, size], graph)
      vfeed = []
      for i in range(n):
        x = _frame(size[0], size[1], 1000 * b + 100 * v + i)
        p = _pub(1000 * b + 100 * v + i, size)
        vfeed.append(([x, x], None, [p, p] if public else None, None))
      fixed_counted = []
      want = _play(fresh, vfeed, launches=fixed_counted)
      if not graph:                            # launches_per_step: the capacity runner's count equals the fixed one's
        assert len(set(fixed_counted)) == 1, fixed_counted
        assert list(plain)[0] == fixed_counted[0] and cap_launches == fresh.launches_per_step, (plain, fixed_counted)
      del fresh
      for i in range(n):
        _same(got[t0 + i], want[i], b, (b, v, i))


def test_camera_follows_the_video_on_3d_head_sets():
  opt, model = _model('nuscenes_ddd')
  rng = np.random.RandomState(4)
  cams = {(b, v): np.float32([[rng.uniform(500, 1500), 0, rng.uniform(50, 150), 0],
                              [0, rng.uniform(500, 1500), rng.uniform(40, 100), 0], [0, 0, 1, 0]])
          for b, vids in VIDEOS.items() for v in range(len(vids))}
  feed = _switch_feed(False, lambda b, v: cams[(b, v)])
  first = [cams[(0, 0)], cams[(1, 0)]]
  r = _runner(model, opt, 'bf16', [S0, S2], True, MAXF, calibs=first)
  got = _play(r, feed)
  del r
  for b, vids in VIDEOS.items():
    for v, (size, t0, n) in enumerate(vids):
      fresh = _runner(model, opt, 'bf16', [size, size], True, calibs=[cams[(b, v)]] * 2)
      want = _play(fresh, [([_frame(size[0], size[1], 1000 * b + 100 * v + i)] * 2, None, None, None)
                           for i in range(n)])
      del fresh
      for i in range(n):
        _same(got[t0 + i], want[i], b, (b, v, i))


@pytest.mark.parametrize('precision', ['bf16', 'bf16x3'])
def test_capacity_runner_at_capacity_equals_the_fixed_runner(precision):
  opt, model = _model('coco_tracking')
  feed = [([_frame(S0[0], S0[1], 10 * t + b) for b in range(B)], None, None, None) for t in range(4)]
  cap = _runner(model, opt, precision, [S0, S0], True, S0)
  a = _play(cap, feed)
  h2d = cap.h2d_bytes_per_step
  del cap
  fixed = _runner(model, opt, precision, [S0, S0], True)
  want = _play(fixed, feed)
  assert h2d == fixed.h2d_bytes_per_step
  for t in range(4):
    for b in range(B):
      _same(a[t], want[t], b, (t, b))


def test_track_videos_on_a_capacity_runner_equals_fresh_runners():
  from centertrack_b200.videos import Video, track_videos
  opt, model = _model('coco_tracking')
  spec = [(S0, 3), (S2, 2), (S1, 4), (S0, 2), (S2, 3)]
  vids = lambda: [Video(v, [_frame(s[0], s[1], 50 * v + i) for i in range(n)]) for v, (s, n) in enumerate(spec)]
  r = _runner(model, opt, 'bf16', [S0, S0], True, MAXF)
  got = {(v, i): res for v, i, res in track_videos(r, vids())}
  del r
  assert sorted(got) == sorted((v, i) for v, (_, n) in enumerate(spec) for i in range(n))
  for v, (s, n) in enumerate(spec):
    fresh = _runner(model, opt, 'bf16', [s, s], True)
    want = {(v2, i): res for v2, i, res in track_videos(fresh, [vids()[v]])}
    del fresh
    for i in range(n):
      a, w = got[(v, i)], want[(v, i)]
      assert len(a) == len(w), (v, i)
      for x, y in zip(a, w):
        for k in x:
          assert np.array_equal(np.asarray(x[k]), np.asarray(y[k])), (v, i, k)
