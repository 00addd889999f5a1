"""NV12 / I420 camera frames in StreamRunner, on the host (no GPU): the YUV reference against cv2.cvtColor byte for
byte, a 4:2:0 runner's frame shapes, slot layout, upload runs and staging views, and its argument checks."""
import ctypes as C

import cv2
import numpy as np
import pytest

from centertrack_b200 import _lib as L
from helpers import make_opt
from yuv_oracle import random_yuv420, yuv420_to_bgr

CODES = {'nv12': cv2.COLOR_YUV2BGR_NV12, 'i420': cv2.COLOR_YUV2BGR_I420}
SIZES = [(2, 2), (480, 640), (376, 1242), (1080, 1920), (6, 18)]


@pytest.mark.parametrize('fmt', ['nv12', 'i420'])
@pytest.mark.parametrize('hw', SIZES, ids=['%dx%d' % s for s in SIZES])
def test_reference_equals_cv2_on_random_frames(fmt, hw):
  h, w = hw
  f = random_yuv420(h, w, h * 7 + w)
  assert np.array_equal(yuv420_to_bgr(f, h, w, fmt), cv2.cvtColor(f, CODES[fmt]))


@pytest.mark.parametrize('fmt', ['nv12', 'i420'])
def test_reference_equals_cv2_at_the_range_ends(fmt):
  """Y in 0..16 (clamped to 16) and 235..255, U and V at 0 and 255 (every channel saturates at 0 or 255 somewhere)."""
  h, w = 64, 96
  rng = np.random.RandomState(5)
  f = np.empty((h * 3 // 2, w), np.uint8)
  f[:h // 2] = rng.randint(0, 17, (h // 2, w))
  f[h // 2:h] = rng.randint(235, 256, (h // 2, w))
  f[h:] = rng.choice(np.uint8([0, 1, 127, 128, 254, 255]), (h // 2, w))
  ref = cv2.cvtColor(f, CODES[fmt])
  assert np.array_equal(yuv420_to_bgr(f, h, w, fmt), ref)
  assert (ref == 0).any() and (ref == 255).any()


@pytest.mark.parametrize('fmt', ['nv12', 'i420'])
@pytest.mark.parametrize('hw', [(480, 640), (6, 18), (1082, 1922)], ids=['480x640', '6x18', '1082x1922'])
def test_reference_equals_cv2_with_a_padded_pitch(fmt, hw):
  """A frame that is a view into wider rows (a decoder's pitched surface): cv2 reads the luma and the chroma rows at
  that pitch, and so does the reference."""
  h, w = hw
  buf = random_yuv420(h, w, 11, pitch=w + 70)
  view = buf[:, :w]
  assert not view.flags['C_CONTIGUOUS']
  assert np.array_equal(yuv420_to_bgr(view, h, w, fmt), cv2.cvtColor(view, CODES[fmt]))


# ------------------------------------------------------------------------------------------------- the runner
def _runner(sizes, fmt, H=544, W=960, max_frame_size=(1080, 1920), cfg='mot'):
  """A StreamRunner with nothing but the frames-mode geometry and host state (what the checks and the planning read)."""
  from centertrack_b200.runner import StreamRunner
  r = object.__new__(StreamRunner)
  r.B, r.H, r.W, r.opt = len(sizes), H, W, make_opt(cfg)
  r.frames_mode, r.tracker, r.t, r.frame_format = True, None, 0, fmt
  r._frame_geometry(sizes, None, max_frame_size)
  r._desc_mirror = [bytes(r.frames)] * 3
  return r


def test_frame_layout_and_shape_inference():
  from centertrack_b200.runner import frame_layout, frame_size_of
  assert frame_layout('bgr', 1080, 1920) == ((1080, 1920, 3), 6220800, 5760)
  for fmt in ('nv12', 'i420'):
    assert frame_layout(fmt, 1080, 1920) == ((1620, 1920), 3110400, 1920)
    assert frame_layout(fmt, 480, 640)[1] == 460800
    assert frame_size_of(fmt, (1620, 1920)) == (1080, 1920)
    assert frame_size_of(fmt, (3, 2)) == (2, 2)
    for bad in [(1621, 1920), (1620, 1921), (1080, 1920, 3), (1620,), (1620, 1920, 1)]:
      assert frame_size_of(fmt, bad) is None, bad
  assert frame_size_of('bgr', (1080, 1920, 3)) == (1080, 1920) and frame_size_of('bgr', (1620, 1920)) is None


@pytest.mark.parametrize('fmt', ['nv12', 'i420'])
def test_frame_shapes_are_inferred_and_checked(fmt):
  r = _runner([(1080, 1920), (480, 640)], fmt)
  frames = [np.zeros((1620, 1920), np.uint8), np.zeros((720, 640), np.uint8)]
  assert r._frame_sizes_of(frames) == [(1080, 1920), (480, 640)]
  up = fmt.upper()
  for bad in (np.zeros((1621, 1920), np.uint8), np.zeros((1620, 1919), np.uint8), np.zeros((1080, 1920, 3), np.uint8)):
    with pytest.raises(ValueError, match=r'frames\[1\]: expected a %s frame of shape \[3h/2, w\]' % up):
      r._frame_sizes_of([frames[0], bad])
  with pytest.raises(ValueError, match='uint8'):
    r._frame_sizes_of([frames[0], frames[1].astype(np.int16)])
  # a size is refused when odd, past the region (half the bytes of BGR), or mapping to another input
  with pytest.raises(ValueError, match='even height and width'):
    r._check_sizes([(1080, 1920), (482, 642 + 1)], [1])
  assert r._size_geometry('s', 1080, 1920)[0]['height'] == 1080
  with pytest.raises(ValueError, match='3116160 bytes, more than the 3110400 of max_frame_size'):
    r._size_geometry('s', 1082, 1920)
  with pytest.raises(ValueError, match='frame size'):
    r.check_frame_size((375, 1243))
  changed = r._check_sizes([(1080, 1920), (376, 1242)], [1])
  assert list(changed) == [1]
  r._plan_geometry(0, changed, {})
  f = r.frames[1]
  assert (f.h, f.w, f.step, f.format) == (376, 1242, 1242, L.CT_FRAME_NV12 if fmt == 'nv12' else L.CT_FRAME_I420)


@pytest.mark.parametrize('fmt', ['nv12', 'i420'])
def test_slot_layout_and_upload_runs_of_mixed_streams(fmt):
  """1080p and 480p 4:2:0 streams: regions of 1080 * 1920 * 3 / 2 bytes, uploads of each frame's own bytes."""
  r = _runner([(1080, 1920), (480, 640), (1080, 1920), (1080, 1920)], fmt)
  cap = 1080 * 1920 * 3 // 2
  assert r.max_frame_bytes == cap and r.cap == cap and r.slot_bytes == 4 * cap
  assert [f.offset for f in r.frames] == [0, cap, 2 * cap, 3 * cap]
  assert [f.step for f in r.frames] == [1920, 640, 1920, 1920]
  assert r._upload_runs() == [(0, 480 * 640 * 3 // 2 + cap), (2 * cap, 4 * cap)]
  assert r._upload_runs(live=[1, 3]) == [(cap, cap + 460800), (3 * cap, 4 * cap)]
  bgr = _runner([(1080, 1920), (480, 640), (1080, 1920), (1080, 1920)], 'bgr')
  assert sum(e - a for a, e in bgr._upload_runs()) == 2 * sum(e - a for a, e in r._upload_runs())


@pytest.mark.parametrize('fmt', ['nv12', 'i420'])
def test_frame_buffers_are_views_of_the_4_2_0_shape(fmt):
  import torch
  r = _runner([(1080, 1920), (480, 640)], fmt)
  r.h_u8 = [torch.zeros(r.slot_bytes, dtype=torch.uint8) for _ in range(3)]
  views = r.frame_buffers()
  assert [v.shape for v in views] == [(1620, 1920), (720, 640)]
  views[1][:] = 7
  assert r.h_u8[0].numpy()[r.cap:r.cap + 460800].min() == 7 and not r.h_u8[0].numpy()[:r.cap].any()
  views = r.frame_buffers({1: (376, 1242)})
  assert views[1].shape == (564, 1242) and r._frame_sizes_of(None) == [(1080, 1920), (376, 1242)]


def test_frame_format_needs_a_capacity_runner():
  from centertrack_b200.runner import StreamRunner
  for kw in (dict(frame_sizes=[(480, 640)]), dict()):
    with pytest.raises(ValueError, match='needs frame_sizes and max_frame_size'):
      StreamRunner(None, 1, 512, 512, opt=make_opt('coco_tracking'), frame_format='nv12', **kw)
  with pytest.raises(ValueError, match='frame_format: expected one of'):
    StreamRunner(None, 1, 512, 512, opt=make_opt('coco_tracking'), frame_sizes=[(480, 640)],
                 max_frame_size=(480, 640), frame_format='yuyv')


def test_track_videos_sizes_4_2_0_frames():
  """The scheduler reads a 4:2:0 frame's (h, w) from its [3h/2, w] shape and refuses other shapes."""
  from centertrack_b200.videos import track_videos
  from test_camera_switch_host import _FakeCapacityRunner

  seen = []

  class Fake(_FakeCapacityRunner):
    frame_format = 'nv12'

    def check_frame_size(self, size):
      seen.append(tuple(size))
      if size[0] * size[1] * 3 // 2 > self.max_frame_bytes:
        raise ValueError('frame size %s refused' % (size,))

    def step_frames(self, frames, public_dets=None, starts=None, pre_dets=None, calibs=None):
      for b, f in enumerate(frames):
        hw = (f.shape[0] // 3 * 2, f.shape[1])
        if hw != self.frame_sizes[b]:
          assert b in starts
          self.frame_sizes[b] = hw
      self.steps.append(dict(frames=[int(f[0, 0]) for f in frames], starts=list(starts), calibs=calibs))

  A, Bs = (12, 20), (8, 14)
  vids = [dict(id=v, frames=[np.full((s[0] * 3 // 2, s[1]), 10 * v + i, np.uint8) for i in range(n)])
          for v, (s, n) in enumerate([(A, 3), (Bs, 2), (A, 2)])]
  r = Fake([A, A], 12 * 20 * 3 // 2)
  out = list(track_videos(r, vids))
  assert sorted((v, i) for v, i, _ in out) == [(0, 0), (0, 1), (0, 2), (1, 0), (1, 1), (2, 0), (2, 1)]
  assert set(seen) == {A, Bs}
  with pytest.raises(ValueError, match='not a NV12 frame'):
    list(track_videos(Fake([A, A], 10 ** 6), [dict(id='bgr', frames=[np.zeros((12, 20, 3), np.uint8)])]))
