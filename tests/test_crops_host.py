"""Track crops without a GPU: the ct_crop_desc ABI, the crop oracle (documented map + warp_affine_u8) against
cv2.warpAffine(INTER_LINEAR | WARP_INVERSE_MAP) byte for byte, the active-prefix property of the host Tracker's rows
that the kernel relies on, and the refusals of ct_crop_boxes and of StreamRunner(crop_size=)."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import cv2
import numpy as np
import pytest

from conftest import ROOT
from centertrack_b200 import _lib as L
from crop_oracle import MAX_COORD, crop, crop_map
from helpers import make_opt
from yuv_oracle import random_yuv420, yuv420_to_bgr


def test_crop_desc_layout_matches_the_header():
  offs = [getattr(L.CropDesc, f).offset for f in ('buf', 'buf_bytes', 'frames', 'rows', 'row_floats', 'rows_per_stream',
                                                  'counts', 'counts_stride', 'active_col', 'K', 'out_h', 'out_w', 'out',
                                                  'out_counts')]
  assert [C.sizeof(L.CropDesc)] + offs == [88, 0, 8, 16, 24, 32, 36, 40, 48, 52, 56, 60, 64, 72, 80]
  assert 'ct_crop_boxes' in L.EXPORTS
  cc = shutil.which('cc') or shutil.which('gcc')
  if cc is None:
    pytest.skip('no C compiler to read the header')
  fields = ['buf', 'buf_bytes', 'frames', 'rows', 'row_floats', 'rows_per_stream', 'counts', 'counts_stride',
            'active_col', 'K', 'out_h', 'out_w', 'out', 'out_counts']
  prog = '#include <stddef.h>\n#include <stdio.h>\n#include "ctb200.h"\nint main(void) {\n  printf("%zu", ' \
      'sizeof(ct_crop_desc));\n' + ''.join('  printf(" %%zu", offsetof(ct_crop_desc, %s));\n' % f for f in fields) + \
      '  printf("\\n");\n  return 0;\n}\n'
  with tempfile.TemporaryDirectory() as tmp:
    with open(os.path.join(tmp, 'p.c'), 'w') as f:
      f.write(prog)
    exe = os.path.join(tmp, 'p')
    subprocess.run([cc, '-I', os.path.join(ROOT, 'include'), os.path.join(tmp, 'p.c'), '-o', exe], check=True)
    got = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()
  assert [int(v) for v in got] == [88] + offs


# ------------------------------------------------------------------------------------------------ the oracle vs cv2
def _cv2_crop(bgr, box, oh, ow):
  m = crop_map(box, oh, ow).reshape(2, 3)
  return cv2.warpAffine(bgr, m, (ow, oh), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP,
                        borderMode=cv2.BORDER_CONSTANT, borderValue=0)


def _boxes(h, w, rng):
  """Inside, partly and wholly outside, sub-pixel, inverted, whole-frame and +-16384 px boxes of an h x w frame."""
  out = [(0, 0, w, h), (w * .25, h * .2, w * .75, h * .9), (-w * .3, -h * .4, w * .5, h * .6),
         (w * .6, h * .5, w * 1.7, h * 1.3), (w + 5, h + 3, w + 40, h + 90), (-80, -50, -10, -2),
         (w * .4, h * .4, w * .4 + .3, h * .4 + .7), (3.3, 2.1, 3.35, 2.12), (w * .8, h * .9, w * .1, h * .2),
         (w * .2, h * .7, w * .6, h * .1), (-MAX_COORD, -MAX_COORD, MAX_COORD, MAX_COORD),
         (MAX_COORD, MAX_COORD, -MAX_COORD, -MAX_COORD), (-MAX_COORD, 0, w, MAX_COORD), (0, -MAX_COORD, MAX_COORD, h)]
  for _ in range(10):
    x = rng.uniform(-0.5 * w, 1.5 * w, 2)
    y = rng.uniform(-0.5 * h, 1.5 * h, 2)
    out.append((x[0], y[0], x[1], y[1]))
  return [np.float32(b) for b in out]


FRAMES = [('bgr', (48, 64)), ('bgr', (1, 1)), ('bgr', (1, 37)), ('bgr', (29, 1)), ('bgr', (375, 1242)),
          ('nv12', (60, 80)), ('i420', (34, 126)), ('nv12', (2, 2))]


@pytest.mark.parametrize('fmt,hw', FRAMES, ids=['%s_%dx%d' % (f, h, w) for f, (h, w) in FRAMES])
def test_crop_oracle_equals_cv2(fmt, hw):
  h, w = hw
  rng = np.random.RandomState(h * 1000 + w)
  if fmt == 'bgr':
    bgr = rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8)
  else:
    bgr = yuv420_to_bgr(random_yuv420(h, w, h + w), h, w, fmt)
  for oh, ow in ((37, 23), (256, 128), (1, 1), (8, 16)):
    for box in _boxes(h, w, rng):
      got = crop(bgr, box, oh, ow)
      want = _cv2_crop(bgr, box, oh, ow)
      assert got.shape == (oh, ow, 3)
      assert np.array_equal(got, want), (fmt, hw, (oh, ow), box.tolist(), int((got != want).sum()))


def test_crop_map_is_evaluated_in_the_documented_order():
  box = np.float32([10.1, 20.7, 210.3, 95.9])
  x0, y0, x1, y1 = (float(v) for v in box)
  sx, sy = (x1 - x0) / 23, (y1 - y0) / 37
  assert crop_map(box, 37, 23).tolist() == [sx, 0.0, (x0 - 0.5) + 0.5 * sx, 0.0, sy, (y0 - 0.5) + 0.5 * sy]


def test_zero_rule_beyond_the_bound_and_for_non_finite_boxes():
  bgr = np.full((40, 50, 3), 200, np.uint8)
  assert crop(bgr, (-MAX_COORD, -MAX_COORD, MAX_COORD, MAX_COORD), 9, 7).any()
  big = np.nextafter(np.float32(MAX_COORD), np.float32(np.inf))
  for box in ((0, 0, big, 30), (-big, 0, 20, 30), (0, 0, 20, -big), (0, big, 20, 30), (0, 0, np.nan, 30),
              (np.inf, 0, 20, 30), (0, -np.inf, 20, 30), (0, 0, 20, 1e30)):
    assert not crop(bgr, box, 9, 7).any(), box


# ------------------------------------------------------------------------------------------------ the active prefix
MODES = {'greedy': [], 'hungarian': ['--hungarian'], 'public_det': ['--public_det'],
         'max_age': ['--max_age', '3'], 'hungarian_public_max_age': ['--hungarian', '--public_det', '--max_age', '2']}


@pytest.mark.parametrize('mode', list(MODES))
def test_active_tracks_are_a_prefix_of_the_tracker_rows(mode):
  """Crowded seeded streams: many overlapping boxes of few classes jittering and vanishing, so that every step has
  matches, births and coasting tracks; after every step the rows with active != 0 come first."""
  from centertrack_b200.tracker import Tracker
  opt = make_opt('coco_tracking', ['--new_thresh', '0.3'] + MODES[mode])
  seen = {'active': 0, 'coasting': 0}
  for seed in range(4):
    rng = np.random.RandomState(seed)
    trk = Tracker(opt)
    ct = rng.uniform(0, 200, (60, 2))
    for step in range(12):
      ct += rng.normal(0, 4, ct.shape)
      keep = rng.rand(len(ct)) < 0.7
      results = []
      for c in ct[keep]:
        s = rng.uniform(4, 30)
        results.append({'score': float(rng.uniform(0.05, 1.0)), 'class': int(rng.randint(1, 3)),
                        'ct': np.float32(c), 'tracking': np.float32(rng.normal(0, 3, 2)),
                        'bbox': np.float32([c[0] - s, c[1] - s, c[0] + s, c[1] + s])})
      results.sort(key=lambda r: -r['score'])
      pub = [{'ct': np.float32(c + rng.normal(0, 2, 2))} for c in ct[rng.rand(len(ct)) < 0.5]]
      rows = trk.step(results, public_det=pub if opt.public_det else None)
      act = [r['active'] != 0 for r in rows]
      n = sum(act)
      assert act == [True] * n + [False] * (len(act) - n), (mode, seed, step)
      seen['active'] += n
      seen['coasting'] += len(act) - n
  assert seen['active'] > 0
  assert seen['coasting'] > 0 or opt.max_age <= 1, seen


# ------------------------------------------------------------------------------------------------ refusals
def test_crop_boxes_refuses_before_launching(built_lib):
  """Each invalid argument returns -1 with a message from the host checks and launches nothing (no GPU here)."""
  lib = L.lib()

  def desc():
    d = L.CropDesc()
    d.buf = d.frames = d.rows = d.counts = d.out = d.out_counts = 64   # never dereferenced: validation fails first
    d.buf_bytes, d.row_floats, d.rows_per_stream, d.counts_stride, d.active_col = 1 << 20, 13, 300, 2, 12
    d.K, d.out_h, d.out_w = 100, 256, 128
    return d

  def fails(msg, d=None, streams=None, n=2, n_streams=2):
    lib.ct_reset_launch_count()
    d = d if d is not None else desc()
    assert lib.ct_crop_boxes(C.byref(d), streams, n, n_streams, None) == -1
    assert msg in lib.ct_last_error(), lib.ct_last_error()
    assert lib.ct_launch_count() == 0

  assert lib.ct_crop_boxes(None, None, 2, 2, None) == -1
  for field in ('buf', 'frames', 'rows', 'counts', 'out', 'out_counts'):
    d = desc()
    setattr(d, field, None)
    fails(b'null pointer', d)
  fails(b'bad batch', n=0)
  fails(b'bad batch', n_streams=0)
  fails(b'bad batch', n=-3)
  for field, value in (('K', 0), ('out_h', 0), ('out_w', -1), ('K', 65536)):
    d = desc()
    setattr(d, field, value)
    fails(b'bad shape', d)
  for field, value in (('rows_per_stream', 0), ('counts_stride', 0), ('buf_bytes', -1)):
    d = desc()
    setattr(d, field, value)
    fails(b'bad table', d)
  for rf, col in ((9, -1), (12, 12), (13, 13), (13, -2)):
    d = desc()
    d.row_floats, d.active_col = rf, col
    fails(b'bbox or active column', d)
  fails(b'n <= n_streams', n=3, n_streams=2)


def test_runner_refuses_crop_size_without_frames_tables_or_a_good_size():
  """Raised before anything else is looked at: no model, no device, no CUDA work."""
  from centertrack_b200.runner import StreamRunner
  opt = make_opt('mot')
  frames = dict(frame_sizes=[(1080, 1920)])
  with pytest.raises(ValueError, match='frames mode'):
    StreamRunner(None, 1, 544, 960, opt=opt, device_tracking=True, crop_size=(64, 32))
  with pytest.raises(ValueError, match='device_tracking or device_post_process'):
    StreamRunner(None, 1, 544, 960, opt=opt, crop_size=(64, 32), **frames)
  for bad in ((0, 32), (64, -1), (64,), (64, 32, 3), 64, (64.0, 32), (True, 32), 'ab'):
    with pytest.raises(ValueError, match='crop_size'):
      StreamRunner(None, 1, 544, 960, opt=opt, device_tracking=True, crop_size=bad, **frames)


def test_track_videos_refuses_crops_without_crop_size():
  from centertrack_b200.videos import track_videos

  class R(object):
    tracker, post, crop = object(), None, None
  with pytest.raises(ValueError, match='crop_size'):
    next(track_videos(R(), [], crops=True))
