"""A StreamRunner stream changing its source frame size and camera at a video start, on the host (no GPU): the argument
checks that run before anything is enqueued, the capacity slot layout and its upload runs, the descriptor uploads, the
metas, the scheduler's placement on a capacity runner, and the new entry points' own checks."""
import ctypes as C

import numpy as np
import pytest

from centertrack_b200 import _lib as L
from helpers import make_opt

MOT = [(1080, 1920), (480, 640)]


def _runner(sizes, H=544, W=960, max_frame_size=(1080, 1920), cfg='mot'):
  """A StreamRunner with nothing but the frames-mode geometry and host state (what the checks and the planning read)."""
  from centertrack_b200.runner import StreamRunner
  r = object.__new__(StreamRunner)
  r.B, r.H, r.W, r.opt = len(sizes), H, W, make_opt(cfg)
  r.frames_mode, r.tracker, r.t = True, None, 0
  r._frame_geometry(sizes, None, max_frame_size)
  r._desc_mirror = [bytes(r.frames)] * 3
  return r


def _pre_process_meta(opt, h, w):
  from centertrack_b200.dataset_info import get_dataset
  from centertrack_b200.detector import Detector
  det = object.__new__(Detector)
  ds = get_dataset(opt.dataset)
  det.opt = opt
  det.mean = np.array(ds.mean, dtype=np.float32).reshape(1, 1, 3)
  det.std = np.array(ds.std, dtype=np.float32).reshape(1, 1, 3)
  det.rest_focal_length = ds.rest_focal_length
  return det.pre_process(np.zeros((h, w, 3), np.uint8), 1.0, {})[1]


def _same_meta(got, ref):
  assert sorted(got) == sorted(ref)
  for k in ref:
    assert np.array_equal(np.asarray(got[k]), np.asarray(ref[k])), k


def _frames(sizes):
  return [np.zeros((h, w, 3), np.uint8) for h, w in sizes]


def test_size_changes_are_checked_before_anything_is_enqueued():
  r = _runner(MOT)
  started = [1]
  with pytest.raises(ValueError, match='more than the 6220800 of max_frame_size'):
    r._check_sizes(r._frame_sizes_of(_frames([(1080, 1920), (1081, 1920)])), started)
  with pytest.raises(ValueError, match='network input'):     # --keep_res-like sizes are refused via another opt
    kr = _runner(MOT, max_frame_size=(1080, 1920))
    kr.opt = make_opt('mot', ['--keep_res'])
    kr._check_sizes([(1080, 1920), (480, 640 + 32)], started)
  with pytest.raises(ValueError, match='only when it starts a video'):
    r._check_sizes([(480, 640), (480, 640)], started)
  with pytest.raises(ValueError, match=r'expected shape \[h, w, 3\]'):
    r._frame_sizes_of([np.zeros((4, 4), np.uint8)] * 2)
  changed = r._check_sizes([(1080, 1920), (375, 1242)], started)
  assert list(changed) == [1] and changed[1][0]['height'] == 375
  # frame_buffers(sizes=) must be followed by a start of those streams
  with pytest.raises(ValueError, match='out of range'):
    _pending(r, {2: (480, 640)})
  with pytest.raises(ValueError, match='max_frame_size'):
    _pending(r, {0: (1081, 1920)})
  _pending(r, {0: (480, 640)})
  assert r._frame_sizes_of(None) == [(480, 640), (480, 640)]
  with pytest.raises(ValueError, match='only when it starts a video'):
    r._check_sizes(r._frame_sizes_of(None), [1])
  assert list(r._check_sizes(r._frame_sizes_of(None), [0])) == [0]
  # a fixed runner refuses any other shape with today's wording
  fixed = _runner(MOT, max_frame_size=None)
  with pytest.raises(ValueError, match='expected shape'):
    fixed._frame_sizes_of(_frames([(1080, 1920), (375, 1242)]))
  with pytest.raises(ValueError, match='fixed'):
    _pending(fixed, {1: (375, 1242)})


def _pending(r, sizes):
  """frame_buffers(sizes) without the pinned views."""
  r._views = lambda slot, s: s
  r.h_u8 = [None] * 3
  return r.frame_buffers(sizes)


def test_calibs_only_for_started_streams_and_of_shape_3x4():
  r = _runner(MOT)
  k = np.arange(12, dtype=np.float32).reshape(3, 4)
  with pytest.raises(ValueError, match='does not start'):
    r._check_calibs({0: k}, [1])
  with pytest.raises(ValueError, match=r'\[3, 4\]'):
    r._check_calibs({1: np.zeros((3, 3))}, [1])
  assert r._check_calibs(None, [1]) == {} and r._check_calibs({1: k.tolist()}, [1])[1].dtype == np.float32


def test_slot_layout_and_upload_runs():
  r = _runner([(1080, 1920), (480, 640), (1080, 1920), (1080, 1920)])
  cap = 1080 * 1920 * 3
  assert r.cap == cap and r.slot_bytes == 4 * cap and [f.offset for f in r.frames] == [0, cap, 2 * cap, 3 * cap]
  assert r._upload_runs() == [(0, 480 * 640 * 3 + cap), (2 * cap, 4 * cap)]
  full = _runner([(1080, 1920)] * 4)
  fixed = _runner([(1080, 1920)] * 4, max_frame_size=None)
  assert full._upload_runs() == [(0, fixed.slot_bytes)]     # at capacity: the fixed runner's one copy
  odd = _runner([(301, 457), (301, 457)], max_frame_size=(301, 457))   # padded to 16 bytes: still one run
  assert odd.cap % 16 == 0 and odd._upload_runs() == [(0, 2 * odd.cap)]
  ragged = _runner([(1080, 1920), (301, 457), (480, 640)], max_frame_size=None)   # fixed: contiguous ragged frames
  assert [f.offset for f in ragged.frames] == [0, cap, cap + (301 * 457 * 3 + 15) // 16 * 16]
  assert ragged._upload_runs() == [(0, ragged.slot_bytes)]


def test_descriptors_upload_only_when_a_slot_changes():
  r = _runner(MOT)
  uploads = []
  for t, sizes in enumerate([MOT, MOT, [(1080, 1920), (375, 1242)], [(1080, 1920), (375, 1242)],
                             [(1080, 1920), (375, 1242)], [(1080, 1920), (375, 1242)], [(375, 1242), (375, 1242)]]):
    changed = r._check_sizes(sizes, [0, 1])
    desc, _ = r._plan_geometry(t % 3, changed, {})
    uploads.append(desc is not None)
  # the change at step 2 reaches slots 2, 0, 1 once each; steady state uploads nothing; step 6 changes slot 0 again
  assert uploads == [False, False, True, True, True, False, True]
  fixed = _runner(MOT, max_frame_size=None)                 # its descriptors never change: never uploaded
  assert all(fixed._plan_geometry(t % 3, {}, {})[0] is None for t in range(6))


def test_meta_and_previous_meta_follow_each_frame():
  from centertrack_b200.detector import default_calib
  opt = make_opt('mot')
  r = _runner(MOT)
  k = np.arange(12, dtype=np.float32).reshape(3, 4)
  # (sizes, calibs) per step; the camera each stream must have then: a changed size without a calib takes the default
  # calib of that size, an unchanged size without one keeps its camera
  steps = [(MOT, {}, ['default', 'default']), ([(1080, 1920), (375, 1242)], {}, ['default', 'default']),
           ([(480, 640), (375, 1242)], {0: k}, [k, 'default']), ([(480, 640), (375, 1242)], {1: k}, [k, k]),
           ([(1080, 1920), (375, 1242)], {}, ['default', k])]
  last = (MOT, ['default', 'default'])
  for sizes, cal, want in steps:
    r._plan_geometry(0, r._check_sizes(sizes, [0, 1]), cal)
    for b in range(2):
      for got, (hw, w) in ((r.meta(b), (sizes[b], want[b])), (r.previous_meta(b), (last[0][b], last[1][b]))):
        ref = _pre_process_meta(opt, *hw)
        if not isinstance(w, str):
          ref['calib'] = w
        _same_meta(got, ref)
    last = (sizes, want)
  assert np.array_equal(r.meta(0)['calib'], default_calib(r.focal, 1920, 1080))


# ------------------------------------------------------------------------------------------------- the scheduler
class _FakeCapacityRunner(object):
  """track_videos' view of a capacity runner: streams take any size that fits and maps to (H, W); every step's frames,
  starts and calibs are recorded and a stream's results are the frame it was fed."""

  def __init__(self, sizes, max_bytes, refuse=()):
    self.B, self.frames_mode, self.frame_sizes, self.public = len(sizes), True, list(sizes), False
    self.max_frame_bytes, self.refuse = max_bytes, set(refuse)
    self.tracker = object()
    self.steps = []

  def check_frame_size(self, size):
    if size[0] * size[1] * 3 > self.max_frame_bytes or tuple(size) in self.refuse:
      raise ValueError('frame size %s refused' % (size,))

  def step_frames(self, frames, public_dets=None, starts=None, pre_dets=None, calibs=None):
    for b, f in enumerate(frames):
      if f.shape[:2] != self.frame_sizes[b]:
        assert b in starts, 'a size change without a start'
        self.frame_sizes[b] = f.shape[:2]
    self.steps.append(dict(frames=[int(f[0, 0, 0]) for f in frames], starts=list(starts), calibs=calibs))

  def _res(self, i):
    return [[('step', i, b, v)] for b, v in enumerate(self.steps[i]['frames'])]

  def previous_results(self):
    return self._res(len(self.steps) - 2)

  def fetch_results(self):
    return self._res(len(self.steps) - 1)


def _video(vid, n, size, code, **kw):
  frames = [np.full(size + (3,), (code * 10 + i) % 256, np.uint8) for i in range(n)]
  return dict(id=vid, frames=iter(frames), **kw)


def test_scheduler_on_a_capacity_runner():
  from centertrack_b200.videos import track_videos
  A, Bs = (12, 20), (9, 13)
  lengths = [3, 5, 2, 4, 6, 1, 3]
  vsize = [A, A, Bs, A, Bs, Bs, A]
  calib = {3: np.eye(3, 4, dtype=np.float32)}
  r = _FakeCapacityRunner([A, A], 12 * 20 * 3)
  vids = [_video(v, n, s, v, calib=calib.get(v)) for v, (n, s) in enumerate(zip(lengths, vsize))]
  out = list(track_videos(r, vids))
  assert sorted((v, i) for v, i, _ in out) == sorted((v, i) for v, n in enumerate(lengths) for i in range(n))
  stream_of = {}
  for v, i, res in out:
    (_, step, b, fed), = res
    assert fed == 10 * v + i
    assert stream_of.setdefault(v, b) == b
    assert (b in r.steps[step]['starts']) == (i == 0)
    if i == 0:
      cal = r.steps[step]['calibs'] or {}
      assert (b in cal) == (v in calib) and (v not in calib or cal[b] is calib[v])
  # every stream is busy until the videos run out (no stream waits for a video of its own size): only the tail of the
  # last video runs beside an idle stream
  last_start = max(i for i, s in enumerate(r.steps) if s['starts'])
  assert 2 * len(r.steps) - sum(lengths) <= len(r.steps) - 1 - last_start
  with pytest.raises(ValueError, match='refused'):
    list(track_videos(_FakeCapacityRunner([A, A], 12 * 20 * 3), [_video('big', 2, (13, 20), 0)]))
  with pytest.raises(ValueError, match='refused'):
    list(track_videos(_FakeCapacityRunner([A, A], 10 ** 6, refuse=[(9, 13)]), [_video('other', 2, Bs, 0)]))


def test_mot_like_mix_needs_fewer_steps_than_streams_split_by_size():
  """A quarter of the videos at 640x480: a fixed runner with the same B split 3:1 by size idles the streams of the
  size whose videos ran out; a capacity runner keeps all of them busy."""
  from centertrack_b200.videos import track_videos
  from test_stream_starts_host import _FakeRunner
  rng = np.random.RandomState(3)
  big, small = (12, 20), (6, 8)
  spec = [(int(rng.randint(3, 12)), big) for v in range(18)] + [(int(rng.randint(3, 12)), small) for v in range(6)]
  vids = lambda: [_video(v, n, s, v) for v, (n, s) in enumerate(spec)]
  cap = _FakeCapacityRunner([big] * 4, 12 * 20 * 3)
  fixed = _FakeRunner([big, big, big, small])
  n_cap = len(list(track_videos(cap, vids())))
  n_fixed = len(list(track_videos(fixed, vids())))
  assert n_cap == n_fixed == sum(n for n, _ in spec)
  assert len(cap.steps) < len(fixed.steps), (len(cap.steps), len(fixed.steps))


# ------------------------------------------------------------------------------------------ entry point checks
def test_device_descriptor_entry_points_reject_bad_arguments_without_a_gpu(built_lib):
  lib = L.lib()
  p = C.c_void_p(256)
  mean = np.zeros(3, np.float32)
  std = np.ones(3, np.float32)
  m, s = C.c_void_p(mean.ctypes.data), C.c_void_p(std.ctypes.data)

  def expect(msg, rc):
    assert rc == L.CT_ERR_INVALID and msg in lib.ct_last_error(), lib.ct_last_error()

  for fn in (lib.ct_pack_stem_frames_dev, lib.ct_pack_stem_frames_flip_dev):
    def call(cur=p, fr=p, B=2, nb=1024, ms=m, out=p, H=8, W=8):
      return fn(cur, None, fr, B, nb, ms, s, None, out, H, W, None)
    for kw in (dict(cur=None), dict(fr=None), dict(ms=None), dict(out=None)):
      expect(b'null pointer', call(**kw))
    for kw in (dict(B=0), dict(B=65536), dict(H=0), dict(W=-1)):
      expect(b'bad shape', call(**kw))
    expect(b'buf_bytes', call(nb=-1))

  def warp(src=p, fr=p, B=2, nb=1024, ms=m, dst=p, H=8, W=8):
    return lib.ct_warp_frames_normalize(src, fr, B, nb, ms, s, dst, H, W, None)
  for kw in (dict(src=None), dict(fr=None), dict(ms=None), dict(dst=None)):
    expect(b'null pointer', warp(**kw))
  for kw in (dict(B=0), dict(H=0), dict(W=0)):
    expect(b'bad shape', warp(**kw))
  expect(b'buf_bytes', warp(nb=-5))
