"""Idle streams on a StreamRunner, on the host (no GPU): the refusals that run before anything is enqueued, the stream
maps and padded batches, the upload runs of the live streams, the image-ordered descriptors, the expansion of the
compacted records, None results for idle streams, and the new entry points in the header and the binding."""
import numpy as np
import pytest

from centertrack_b200 import _lib as L
from helpers import make_opt

MOT = [(1080, 1920), (480, 640), (1080, 1920), (480, 640), (1080, 1920)]


def _runner(sizes=MOT, g=1, max_frame_size=(1080, 1920)):
  """A StreamRunner with nothing but the frames-mode geometry and the idle-streams host state."""
  from centertrack_b200.runner import StreamRunner
  r = object.__new__(StreamRunner)
  r.B, r.H, r.W, r.opt = len(sizes), 544, 960, make_opt('mot')
  r.frames_mode, r.tracker, r.t = True, None, 0
  r._frame_geometry(sizes, None, max_frame_size)
  r.idle_g, r._was_idle, r._live = g, set(), [None, None]
  return r


def test_constructor_refuses_idle_streams_without_a_capacity_frames_runner():
  from centertrack_b200.runner import StreamRunner
  for kw in (dict(), dict(frame_sizes=[(480, 640)])):       # images mode, fixed-size frames
    with pytest.raises(ValueError, match='capacity frames runner'):
      StreamRunner(None, 1, 544, 960, opt=make_opt('mot'), idle_streams=1, **kw)
  for g in (0, -1, 1.5, np.True_):
    with pytest.raises(ValueError, match='idle_streams'):
      StreamRunner(None, 1, 544, 960, opt=make_opt('mot'), frame_sizes=[(480, 640)], max_frame_size=(480, 640),
                   idle_streams=g)
  with pytest.raises(ValueError, match='capacity frames runner'):    # True: on, with the default granule
    StreamRunner(None, 1, 544, 960, opt=make_opt('mot'), idle_streams=True)


@pytest.mark.parametrize('B', [4, 64, 65, 72, 200])
def test_decode_workspace_keeps_the_candidates_where_the_b_layout_has_them(B):
  """ct_decode's counters are [0, 4 n) of its workspace and its candidates start at align256(4 n).  At every batch n
  the runner's view must keep the counters inside the B layout's counter area and start the candidates at
  align256(4 B), or a decode at one batch overwrites the counters another batch relies on being zero."""
  import torch
  from centertrack_b200.runner import StreamRunner
  a = lambda x: (x + 255) // 256 * 256
  r = object.__new__(StreamRunner)
  r.B = B
  C, J, K = 3, 0, 10
  r.ws = torch.zeros(a(4 * B) + 8 * B * (C + J) * K, dtype=torch.uint8)
  base = r.ws.data_ptr()
  for n in range(1, B + 1):
    v = r._decode_ws(n)
    off = v.data_ptr() - base
    assert off + 4 * n <= a(4 * B)                  # counters in the counter area
    assert off + a(4 * n) == a(4 * B)               # candidates where the B layout's begin
    assert v.numel() >= a(4 * n) + 8 * n * (C + J) * K
  assert r._decode_ws(B) is r.ws


def test_idle_checks_run_before_anything_is_enqueued():
  r = _runner()
  with pytest.raises(ValueError, match='pre_hms'):
    r._check_idle([1], (), np.zeros(1))
  with pytest.raises(ValueError, match='out of range'):
    r._check_idle([5], (), None)
  with pytest.raises(ValueError, match='twice'):
    r._check_idle([1, 1], (), None)
  with pytest.raises(ValueError, match='integers'):
    r._check_idle([True], (), None)
  with pytest.raises(ValueError, match='every stream is idle'):
    r._check_idle(range(5), (), None)
  with pytest.raises(ValueError, match='also start a video'):
    r._check_idle([1, 3], [3], None)
  assert r._check_idle([1, 3], [0], None) == [0, 2, 4]
  assert r._check_idle(None, (), None) == [0, 1, 2, 3, 4]
  r._was_idle = {1, 3}                                       # idle in the last step: back only with a start
  with pytest.raises(ValueError, match=r'\[3\] were idle'):
    r._check_idle([], [1], None)
  assert r._check_idle([3], [1], None) == [0, 1, 2, 4]
  plain = _runner()
  plain.idle_g = None
  with pytest.raises(ValueError, match='without idle_streams'):
    plain._check_idle([1], (), None)
  assert plain._check_idle(None, (), np.zeros(1)) is None


def test_step_host_is_refused_on_an_idle_streams_runner():
  r = _runner()
  with pytest.raises(ValueError, match='step_frames'):
    r.step_host(None)


@pytest.mark.parametrize('B,g', [(5, 1), (5, 2), (5, 4), (32, 4), (32, 1), (7, 3)])
def test_maps_and_padded_batches(B, g):
  r = _runner([(480, 640)] * B, g=g)
  rng = np.random.RandomState(B * 10 + g)
  for n in [1, B] + list(rng.randint(1, B + 1, size=6)):
    live = sorted(rng.choice(B, n, replace=False).tolist())
    m = r._maps(live)
    streams, image_of = m[:B], m[B:]
    n_pad = r.padded_batch(n)
    assert n <= n_pad <= B and (n_pad % g == 0 or n_pad == B) and n_pad - n < g
    assert streams[:n].tolist() == live and (streams[n:] == -1).all()
    for b in range(B):
      assert image_of[b] == (live.index(b) if b in live else -1)
    assert m.dtype == np.int32
  assert r.batches() == sorted({min(-(-n // g) * g, B) for n in range(1, B + 1)})
  assert r.batches()[-1] == B


def test_upload_runs_cover_exactly_the_live_streams():
  r = _runner()
  cap = r.cap
  f = lambda h, w: (h * w * 3 + 15) // 16 * 16
  assert r._upload_runs() == [(0, cap + f(480, 640)), (2 * cap, 3 * cap + f(480, 640)), (4 * cap, 5 * cap)]
  assert r._upload_runs([0, 2, 4]) == [(0, cap), (2 * cap, 3 * cap), (4 * cap, 5 * cap)]
  assert r._upload_runs([0, 1]) == [(0, cap + f(480, 640))]
  assert r._upload_runs([1, 2]) == [(cap, cap + f(480, 640)), (2 * cap, 3 * cap)]
  assert r._upload_runs([3]) == [(3 * cap, 3 * cap + f(480, 640))]


def test_descriptors_in_image_order_and_zero_padding():
  r = _runner()
  r._desc_mirror = [bytes(r.frames)] * 3
  live = [1, 4]
  arr = r._image_frames(live)
  for i, b in enumerate(live):
    assert bytes(arr[i]) == bytes(r.frames[b]) and arr[i].offset == b * r.cap
  for i in range(len(live), r.B):
    assert arr[i].h == 0 and arr[i].w == 0                 # invalid: a zero input on the device
  desc, _ = r._plan_geometry(0, {}, {}, live)
  assert desc == bytes(arr)
  assert r._plan_geometry(0, {}, {}, live)[0] is None        # unchanged: nothing to upload
  assert r._plan_geometry(0, {}, {}, None)[0] == bytes(r.frames)


def test_frames_and_public_entries_of_idle_streams_are_ignored():
  r = _runner()
  frames = [np.zeros((h, w, 3), np.uint8) for h, w in MOT]
  frames[1] = frames[3] = None
  assert r._frame_sizes_of(frames, {1, 3}) == [tuple(s) for s in MOT]
  with pytest.raises(ValueError, match='uint8'):
    r._frame_sizes_of(frames, {1})
  r.public = True

  class _T:
    max_public = 4
  r.tracker = _T()
  pub = r._check_public([np.zeros((2, 2)), None, np.zeros((0, 2)), None, np.ones((1, 2))], {1, 3})
  assert [len(p) for p in pub] == [2, 0, 0, 0, 1]


def test_records_are_expanded_and_idle_results_are_none():
  from centertrack_b200.device_tracker import DeviceTracker
  r = _runner([(480, 640)] * 4)
  K, F, T = 3, 12, 6
  r.compute = type('S', (), {'synchronize': lambda self: None})()
  import torch
  rec = torch.zeros((4, K, F))
  rec[0] = 1.
  rec[1] = 2.
  r.h_rec = [rec.clone(), rec.clone()]
  r._live = [None, [0, 3]]
  r.t = 2                                                     # the last submitted step is t = 1
  out = r.fetch()
  assert out.shape == (4, K, F)
  assert (out[0] == 1).all() and (out[3] == 2).all() and (out[1] == 0).all() and (out[2] == 0).all()
  r._live[1] = [0, 1, 2, 3]                                   # every stream live: the buffer as it is
  assert np.array_equal(r.fetch(), rec.numpy())
  trk = object.__new__(DeviceTracker)
  trk.Wp, trk.payload_layout = 0, {}
  r.tracker = trk
  trk.payload = None
  r.h_trk = [torch.zeros((4, T, L.CT_TRK_FLOATS))] * 2
  cnt = torch.zeros((4, 2), dtype=torch.int32)
  cnt[:, 0] = 1
  r.h_cnt = [cnt] * 2
  r._live = [[1, 2], [0, 3]]
  res = r.fetch_results()
  assert res[1] is None and res[2] is None and len(res[0]) == 1 and len(res[3]) == 1
  prev = r.previous_results()                                 # step t = 0
  assert prev[0] is None and prev[3] is None and len(prev[1]) == 1 and len(prev[2]) == 1


def test_binding_lists_the_mapped_entry_points():
  import os
  import re
  from conftest import ROOT
  src = re.sub(r'/\*.*?\*/', '', open(os.path.join(ROOT, 'include', 'ctb200.h')).read(), flags=re.S)
  declared = sorted(set(re.findall(r'\b(ct_[a-z0-9_]+)\s*\(', src)))
  assert sorted(L.EXPORTS) == declared
  for name in ('ct_track_step_mapped', 'ct_render_tracks_mapped'):
    assert name in declared


def test_mapped_entry_points_validate_without_touching_the_gpu(built_lib):
  import ctypes as C
  lib = L.lib()
  d = L.TrackDesc()
  assert lib.ct_track_step_mapped(C.byref(d), None, None, None, 4, None) == -1
  assert b'null stream map' in lib.ct_last_error()
  p = C.c_void_p(16)
  assert lib.ct_track_step_mapped(C.byref(d), None, None, p, 0, None) == -1
  assert lib.ct_render_tracks_mapped(p, 8, None, 4, p, 2, 8, 8, None) == -1
  assert b'null pointer' in lib.ct_last_error()
  assert lib.ct_render_tracks_mapped(p, 8, p, 4, p, 0, 8, 8, None) == -1
  assert b'bad shape' in lib.ct_last_error()
