"""Video starts on one StreamRunner stream, on the host (no GPU): the argument checks that run before anything is
enqueued, the seed rows against Tracker.init_track, ct_track_start's own checks, and the video scheduler's placement
against a runner stand-in."""
import ctypes as C
import copy
from types import SimpleNamespace

import numpy as np
import pytest

from centertrack_b200 import _lib as L
from centertrack_b200.device_tracker import plan_starts, seed_rows
from helpers import make_opt


def _runner(B=3, T=8, payload=False, tracking=True, opt=None):
  """A StreamRunner with nothing but what _check_starts reads."""
  from centertrack_b200.runner import StreamRunner
  r = object.__new__(StreamRunner)
  r.B, r.opt = B, opt or make_opt('coco_tracking', ['--new_thresh', '0.3'])
  r.tracker = SimpleNamespace(T=T, payload=object() if payload else None) if tracking else None
  return r


def _dets(rng, n, lists=True):
  out = []
  for i in range(n):
    x0, y0 = rng.uniform(0, 300, 2)
    w, h = rng.uniform(1, 60, 2)
    box = [float(x0), float(y0), float(x0 + w), float(y0 + h)]
    d = {'score': float(rng.uniform(0, 1)), 'class': int(rng.randint(1, 4)), 'bbox': box if lists else np.float32(box)}
    if i % 3 == 0:
      d['ct'] = [float(x0 + 1.5), float(y0 + 2.5)]
    if i % 2 == 0:
      d['tracking'] = [float(v) for v in rng.normal(0, 2, 2)]
    out.append(d)
  return out


def test_start_argument_errors():
  r = _runner()
  good = [{'score': 0.9, 'class': 1, 'bbox': [0., 0., 4., 4.]}]
  for starts, pre_dets, msg in (([3], None, 'out of range'), ([-1], None, 'out of range'), ([1, 1], None, 'twice'),
                                ([0], {1: good}, 'does not start'), (None, {0: good}, 'do not start'),
                                ([], {0: good}, 'do not start'), ([0.0], None, 'integers'), ([True], None, 'integers'),
                                ([0], {0: good * 9}, 'more than the 8 rows'),
                                ([0], {0: [{'score': 0.9, 'bbox': [0., 0., 1., 1.]}]}, 'class')):
    with pytest.raises(ValueError, match=msg):
      r._check_starts(starts, pre_dets)
  # nine items of which only eight are kept fit the table
  ok = good * 8 + [{'score': 0.3, 'class': 1, 'bbox': [0., 0., 1., 1.]}]
  streams, seeds = r._check_starts(np.array([2, 0]), {0: ok})
  assert streams == [2, 0] and [len(s) for s in seeds] == [0, 8]
  assert r._check_starts(None, None) is None and r._check_starts([], {}) is None
  with pytest.raises(ValueError, match='payload'):
    _runner(payload=True)._check_starts([0], {0: good})
  with pytest.raises(ValueError, match='payload'):
    _runner(payload=True)._check_starts([0], {0: []})
  assert _runner(payload=True)._check_starts([0, 2], None)[0] == [0, 2]       # a reset without seeds is fine
  plain = _runner(tracking=False)                                             # no device tracking: pre_images only
  assert plain._check_starts([1], None)[0] == [1]
  with pytest.raises(ValueError, match='device_tracking'):
    plain._check_starts([1], {1: good})
  with pytest.raises(ValueError, match='out of range'):
    plain._check_starts([5], None)


@pytest.mark.parametrize('seed', range(4))
def test_seed_rows_equal_tracker_init_track(seed):
  """The rows ct_track_start writes are Tracker.init_track's tracks: the score > new_thresh filter, the input order,
  ids 1..n, age = active = 1, ct from the bbox in float64 when missing, then stored as fp32."""
  from centertrack_b200.device_tracker import DeviceTracker
  from centertrack_b200.tracker import Tracker
  rng = np.random.RandomState(seed)
  opt = make_opt('coco_tracking', ['--new_thresh', '0.4'])
  items = _dets(rng, 25)
  rows = seed_rows(copy.deepcopy(items), opt.new_thresh)
  host = Tracker(opt)
  host.init_track(copy.deepcopy(items))
  assert len(rows) == len(host.tracks) == host.id_count > 0
  for r, t in zip(rows, host.tracks):
    assert r[L.CT_TRK_SCORE] == np.float32(t['score']) and r[L.CT_TRK_CLASS] == t['class']
    assert (r[L.CT_TRK_ID], r[L.CT_TRK_AGE], r[L.CT_TRK_ACTIVE]) == (t['tracking_id'], t['age'], t['active'])
    assert np.array_equal(r[L.CT_TRK_CT:L.CT_TRK_CT + 2], np.float32(t['ct']))
    assert np.array_equal(r[L.CT_TRK_BBOX:L.CT_TRK_BBOX + 4], np.float32(t['bbox']))
    assert np.array_equal(r[L.CT_TRK_TRACKING:L.CT_TRK_TRACKING + 2], np.float32(t.get('tracking', [0., 0.])))
  # the rows read back through DeviceTracker.results are the host tracks
  trk = object.__new__(DeviceTracker)
  trk.Wp = 0
  got = trk.results(rows[None], np.array([[len(rows), len(rows)]], np.int32))[0]
  for a, t in zip(got, host.tracks):
    assert (a['tracking_id'], a['class'], a['age'], a['active']) == (t['tracking_id'], t['class'], 1, 1)
  # the centre is computed in float64 and rounded once
  box = [0.1, 0.2, 0.30000001, 16777217.0]
  r = seed_rows([{'score': 1.0, 'class': 1, 'bbox': box}], 0.5)[0]
  assert r[L.CT_TRK_CT] == np.float32((0.1 + 0.30000001) / 2) and r[L.CT_TRK_CT + 1] == np.float32((0.2 + 16777217.0) / 2)
  assert seed_rows([], 0.5).shape == (0, L.CT_TRK_FLOATS)
  assert plan_starts(4, 100, 0.4, False, [3], {3: items})[1][0].tobytes() == rows.tobytes()


def test_track_start_rejects_bad_arguments_without_a_gpu(built_lib):
  lib = L.lib()
  p = C.c_void_p(256)
  d = L.TrackDesc()
  d.B, d.K, d.F, d.max_tracks = 3, 4, 13, 8
  d.tracks, d.counts = 256, 512
  pay = L.TrackPayload()
  pay.width, pay.payload = 5, 1024

  def call(desc=d, payload=None, starts=p, n=1, seeds=None):
    return lib.ct_track_start(C.byref(desc) if desc is not None else None, C.byref(payload) if payload else None,
                              starts, n, seeds, None)

  def expect(msg, **kw):
    assert call(**kw) == L.CT_ERR_INVALID and msg in lib.ct_last_error(), (kw, lib.ct_last_error())

  expect(b'null pointer', desc=None)
  for f in ('tracks', 'counts'):
    bad = L.TrackDesc.from_buffer_copy(d)
    setattr(bad, f, None)
    expect(b'null pointer', desc=bad)
  for f, v in (('B', 0), ('max_tracks', 0), ('B', -2)):
    bad = L.TrackDesc.from_buffer_copy(d)
    setattr(bad, f, v)
    expect(b'bad shape', desc=bad)
  bad = L.TrackDesc.from_buffer_copy(d)
  bad.boxes = 2048
  expect(b'boxes need trans_input', desc=bad)
  expect(b'n_starts outside', n=4)
  expect(b'n_starts outside', n=-1)
  expect(b'null start list', starts=None)
  pay0 = L.TrackPayload.from_buffer_copy(pay)
  pay0.payload = None
  expect(b'payload table', payload=pay0)
  pay0 = L.TrackPayload.from_buffer_copy(pay)
  pay0.width = 0
  expect(b'payload table', payload=pay0)
  assert call(n=0, starts=None) == L.CT_OK          # nothing to start: no launch, no device needed


# ------------------------------------------------------------------------------------------------- the scheduler
class _FakeRunner(object):
  """What track_videos calls on a StreamRunner: every step's frames, starts and seeds are recorded, and a stream's
  results are the frames it was fed, so that each yielded result can be traced to its step and stream."""

  def __init__(self, sizes, public=False):
    self.B, self.frames_mode, self.frame_sizes, self.public = len(sizes), True, sizes, public
    self.tracker = object()
    self.steps = []

  def step_frames(self, frames, public_dets=None, starts=None, pre_dets=None):
    assert len(frames) == self.B and all(f.shape == s + (3,) for f, s in zip(frames, self.frame_sizes))
    assert (public_dets is not None) == self.public
    self.steps.append(dict(frames=[int(f[0, 0, 0]) for f in frames], starts=list(starts), pre_dets=pre_dets,
                           public=public_dets))

  def _res(self, i):
    return [[('step', i, b, v)] for b, v in enumerate(self.steps[i]['frames'])]

  def previous_results(self):
    return self._res(len(self.steps) - 2)

  def fetch_results(self):
    return self._res(len(self.steps) - 1)


def _video(vid, n, size, code, **kw):
  """n frames of `size` whose pixel (0, 0, 0) encodes (video, frame)."""
  frames = [np.full(size + (3,), code * 10 + i, np.uint8) for i in range(n)]
  return dict(id=vid, frames=iter(frames), **kw)


def test_scheduler_places_every_frame_once_on_a_stream_of_its_size():
  from centertrack_b200.videos import track_videos
  A, Bs = (12, 20), (9, 13)
  sizes = [A, Bs, A]
  lengths = [1, 2, 3, 4, 5, 6, 8]
  vsize = [A, Bs, A, Bs, A, A, Bs]
  seeds = {2: [{'score': 0.9, 'class': 1, 'bbox': [1., 1., 3., 3.]}]}
  r = _FakeRunner(sizes, public=True)
  vids = [_video(v, n, s, v, pre_dets=seeds.get(v),
                 public_dets=[np.full((1, 2), 10 * v + i, np.float32) for i in range(n)])
          for v, (n, s) in enumerate(zip(lengths, vsize))]
  vids.insert(3, dict(id='empty', frames=[]))
  out = list(track_videos(r, vids))
  keys = [(v, i) for v, i, _ in out]
  assert sorted(keys) == sorted((v, i) for v, n in enumerate(lengths) for i in range(n))   # each frame exactly once
  stream_of = {}
  for v, i, res in out:
    (_, step, b, fed), = res
    assert fed == 10 * v + i                              # the result is that frame's stream at that step
    assert r.frame_sizes[b] == vsize[v]
    assert stream_of.setdefault(v, b) == b                # a video stays on one stream
    pub = r.steps[step]['public'][b]
    assert pub.shape == (1, 2) and pub[0, 0] == 10 * v + i
    assert (b in r.steps[step]['starts']) == (i == 0)    # its first frame, and only that one, starts the stream
    if i == 0:
      pd = r.steps[step]['pre_dets'] or {}
      assert (pd.get(b) is not None) == (v in seeds)
  # a video goes to the first free stream of its size: 0 -> stream 0, 1 -> stream 1, 2 -> stream 2
  assert [stream_of[v] for v in range(3)] == [0, 1, 2]
  # idle streams re-feed their last frame
  for s in r.steps:
    assert all(p is not None for p in s['public'])
  with pytest.raises(ValueError, match='size'):
    list(track_videos(_FakeRunner(sizes), [_video('odd', 2, (7, 7), 0)]))
  with pytest.raises(ValueError, match='device_tracking'):
    fr = _FakeRunner(sizes)
    fr.tracker = None
    list(track_videos(fr, []))
