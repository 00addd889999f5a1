"""Resuming idle streams and moving a stream's video between runners, on the host (no GPU): the refusals that run
before anything is enqueued, the last_slot bookkeeping and the resume copy plan, the StreamState layout checks, and
ct_track_restore in the header and the binding."""
import numpy as np
import pytest

from centertrack_b200 import _lib as L
from helpers import make_opt

MOT = [(1080, 1920), (480, 640), (1080, 1920), (480, 640), (1080, 1920)]
LAYOUT = {'reg': (9, 2), 'wh': (11, 2), 'tracking': (13, 2)}


def _runner(sizes=MOT, g=1, fmt='bgr', max_frame_size=(1080, 1920)):
  """A StreamRunner with nothing but the frames-mode geometry and the idle-streams / resume host state."""
  from centertrack_b200.runner import StreamRunner
  r = object.__new__(StreamRunner)
  r.B, r.H, r.W, r.opt = len(sizes), 544, 960, make_opt('mot')
  r.frames_mode, r.tracker, r.t, r.frame_format = True, None, 0, fmt
  r._frame_geometry(sizes, None, max_frame_size)
  r.idle_g, r._was_idle, r._live = g, set(), [None, None]
  r.last_slot, r._restores, r.layout = [None] * r.B, [None] * 3, dict(LAYOUT)
  return r


def _state(r, b=0, **kw):
  """A StreamState with r's layout facts (no device tensors: the checks read shapes and facts only)."""
  from centertrack_b200.runner import StreamState
  f = dict(frame=None, size=MOT[b], calib=np.eye(3, 4, dtype=np.float32), tracks=None, counts=None, payload=None,
           input_size=(r.H, r.W), record_layout=dict(LAYOUT), payload_layout=None, max_tracks=None,
           frame_format=r.frame_format)
  f.update(kw)
  return StreamState(**f)


def _step(r, live, resumed=()):
  """The host bookkeeping of one step_frames call: -> its resume copies."""
  slot = r.t % 3
  copies = r._plan_resume(slot, live, list(resumed))
  r._was_idle = set(range(r.B)) - set(live)
  r.t += 1
  return copies


def test_resume_refusals_run_before_anything_is_enqueued():
  r = _runner()
  _step(r, [0, 1, 2, 3, 4])
  _step(r, [0, 2, 4])                                        # 1 and 3 idle
  with pytest.raises(ValueError, match=r'\[0\] were live in the last step'):
    r._check_resume([0], (), None, {})
  with pytest.raises(ValueError, match=r'\[1\] also start a video'):
    r._check_resume([1], [1], None, {})
  with pytest.raises(ValueError, match=r'\[3\] also are idle'):
    r._check_resume([3], (), [3], {})
  with pytest.raises(ValueError, match=r'\[1\] also are restored'):
    r._check_resume([1], (), None, {1: None})
  with pytest.raises(ValueError, match='out of range'):
    r._check_resume([5], (), None, {})
  with pytest.raises(ValueError, match='twice'):
    r._check_resume([1, 1], (), None, {})
  with pytest.raises(ValueError, match='integers'):
    r._check_resume([True], (), None, {})
  assert r._check_resume([3, 1], (), None, {}) == [1, 3]
  assert r._check_resume(None, (), None, {}) == []
  # the existing refusal stays: back without starts or resume
  with pytest.raises(ValueError, match=r'\[3\] were idle in the last step: an idle stream comes back only'):
    r._check_idle([], [1], None)
  assert r._check_idle([], [1, 3], None) == [0, 1, 2, 3, 4]
  # a frame of another size than the stream's last one is refused as any size change without a start
  sizes = list(MOT)
  sizes[1] = (1080, 1920)
  with pytest.raises(ValueError, match='differs from'):
    r._check_sizes(sizes, [])
  # idle in the very first step: no frame to continue from
  r2 = _runner()
  _step(r2, [0, 2, 3, 4])
  with pytest.raises(ValueError, match='no frame since'):
    r2._check_resume([1], (), None, {})
  plain = _runner()
  plain.idle_g = None
  with pytest.raises(ValueError, match='without idle_streams'):
    plain._check_resume([1], (), None, {})


@pytest.mark.parametrize('fmt', ['bgr', 'nv12', 'i420'])
@pytest.mark.parametrize('run', [1, 2, 3, 4])
def test_last_slot_and_the_resume_copy_plan(fmt, run):
  """Stream 1 is idle for `run` steps from step 2 and resumes; stream 3 stays live.  The copy goes from the slot of
  stream 1's last frame to the previous slot at its region with its frame's bytes, and only when those slots differ."""
  r = _runner(fmt=fmt)
  nbytes = {'bgr': 480 * 640 * 3, 'nv12': 480 * 640 * 3 // 2, 'i420': 480 * 640 * 3 // 2}[fmt]
  assert _step(r, range(5)) == [] and _step(r, range(5)) == []
  assert r.last_slot == [1] * 5
  for k in range(run):
    assert _step(r, [0, 2, 3, 4]) == []
    assert r.last_slot[1] == 1 and r.last_slot[3] == (2 + k) % 3
  t = r.t
  assert r._check_resume([1], (), None, {}) == [1]
  copies = _step(r, range(5), [1])
  prev = (t - 1) % 3
  if run == 3:                                               # its last slot is the previous slot: nothing to copy
    assert prev == 1 and copies == []
  else:
    assert copies == [(1, 1, prev, r.cap, nbytes)]
    assert copies[0][1] == {1: (t + 1) % 3, 2: t % 3, 4: (t + 1) % 3}[run]   # run 2: the slot this step writes
  assert r.last_slot == [t % 3] * 5


def test_several_resumes_in_one_step_with_a_start_and_an_idle_stream():
  r = _runner()
  _step(r, range(5))
  _step(r, [0, 4])                                           # t = 1: 1, 2, 3 idle
  _step(r, [0, 2, 4])                                        # t = 2: 2 live again (a start), 1 and 3 idle
  assert r._check_resume([1, 3], [0], [4], {}) == [1, 3]
  copies = _step(r, [0, 1, 3], [1, 3])                       # t = 3: 1 and 3 resume, 0 starts, 2 and 4 idle
  assert copies == [(1, 0, 2, r.cap, 480 * 640 * 3), (3, 0, 2, 3 * r.cap, 480 * 640 * 3)]
  assert r.last_slot == [0, 0, 2, 0, 2]


def test_restore_refusals_and_state_layout_checks():
  from centertrack_b200.runner import StreamState
  r = _runner()
  _step(r, range(5))
  ok = _state(r, 1)
  assert r._check_restore({2: ok}, (), None) == {2: ok}
  assert r._check_restore(None, (), None) == {}
  with pytest.raises(ValueError, match=r'\[2\] also start a video'):
    r._check_restore({2: ok}, [2], None)
  with pytest.raises(ValueError, match=r'\[2\] also are idle'):
    r._check_restore({2: ok}, (), [2])
  with pytest.raises(ValueError, match='out of range'):
    r._check_restore({7: ok}, (), None)
  with pytest.raises(ValueError, match='StreamState'):
    r._check_restore({2: 'state'}, (), None)
  bad = [(dict(input_size=(512, 512)), 'network input'), (dict(record_layout={'reg': (9, 2)}), 'record layout'),
         (dict(frame_format='nv12'), 'frame_format'), (dict(payload_layout={'dep': (0, 1)}), 'payload layout'),
         (dict(tracks=object(), counts=(1, 1)), 'track table'), (dict(size=(2160, 3840)), 'more than the')]
  for kw, msg in bad:
    with pytest.raises(ValueError, match=msg):
      r._check_restore({2: _state(r, 1, **kw)}, (), None)
  kr = _runner()                                             # --keep_res: a size that maps to another network input
  kr.opt = make_opt('mot', ['--keep_res'])
  with pytest.raises(ValueError, match='network input'):
    kr._check_restore({2: _state(kr, 1, size=(480, 672))}, (), None)
  # a tracking runner: rows within the table, the same payload layout
  trk = type('T', (), {'T': 8, 'payload_layout': {}})()
  r.tracker = trk
  rows = dict(tracks=object(), payload_layout={}, max_tracks=8)
  assert r._check_restore({2: _state(r, 1, counts=(8, 30), **rows)}, (), None)
  with pytest.raises(ValueError, match='9 track rows, more than the 8'):
    r._check_restore({2: _state(r, 1, counts=(9, 30), **rows)}, (), None)
  with pytest.raises(ValueError, match='track table'):
    r._check_restore({2: ok}, (), None)
  # resume and restore of one stream
  r._was_idle = {2}
  with pytest.raises(ValueError, match='also are restored'):
    r._check_resume([2], (), None, {2: ok})
  fixed = _runner()
  fixed.cap = None
  with pytest.raises(ValueError, match='capacity frames runner'):
    fixed._check_restore({0: ok}, (), None)
  with pytest.raises(ValueError, match='capacity frames runner'):
    fixed.stream_state(0)
  r.tracker = None
  with pytest.raises(ValueError, match='no frame since'):
    _runner().stream_state(0)
  assert isinstance(ok, StreamState) and ok.size == (480, 640) and ok.input_size == (544, 960)


def test_binding_lists_ct_track_restore():
  import os
  import re
  from conftest import ROOT
  src = re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'ctb200.h')).read(), flags=re.S)
  declared = sorted(set(re.findall(r'\b(ct_[a-z0-9_]+)\s*\(', src)))
  assert 'ct_track_restore' in declared and 'ct_track_restore' in L.EXPORTS
  assert sorted(L.EXPORTS) == declared


def test_ct_track_restore_validates_without_touching_the_gpu(built_lib):
  import ctypes as C
  lib = L.lib()
  d = L.TrackDesc()
  assert lib.ct_track_restore(C.byref(d), None, None, 0, None, None, None) == -1
  assert b'null pointer' in lib.ct_last_error()
  p = C.c_void_p(16)
  d.tracks, d.counts, d.B, d.max_tracks = p, p, 4, 8
  assert lib.ct_track_restore(C.byref(d), None, None, 1, None, None, None) == -1
  assert b'null entry list' in lib.ct_last_error()
  assert lib.ct_track_restore(C.byref(d), None, p, 5, None, None, None) == -1
  assert b'n_entries' in lib.ct_last_error()
  assert lib.ct_track_restore(C.byref(d), None, p, 0, None, None, None) == 0    # nothing to launch
