"""The packed, normalised crop batch without a GPU: the oracle (torchvision's Normalize(ToTensor()) on the CPU, then
.to(dtype)) against the documented formula in numpy, the ct_crop_tensor ABI, the refusals of ct_crop_boxes_tensor
(no launch), and those of StreamRunner(crop_format=) and track_videos."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from conftest import ROOT
from centertrack_b200 import _lib as L
from crop_tensor_oracle import IMAGENET, bits, normalize, pack
from helpers import make_opt

DTYPES = [torch.float32, torch.float16, torch.bfloat16]
FORMATS = {'imagenet': IMAGENET, 'identity': {'mean': (0., 0., 0.), 'std': (1., 1., 1.)},
           'degenerate': {'mean': (1e30, -0.5, 1.0), 'std': (1e-40, -3e-8, 7.0)},
           'tiny_std': {'mean': (0.5, 0.5, 0.5), 'std': (1e-6, 1e-3, -1e5)}}


def _round(x, dtype):
  """fp32 numpy -> the bits of dtype, round to nearest even (numpy's float16 cast is; bf16 restated)."""
  if dtype == torch.float32:
    return x.view(np.int32)
  if dtype == torch.float16:
    return x.astype(np.float16).view(np.int16)
  u = x.view(np.uint32).astype(np.uint64)
  r = (u + 0x7FFF + ((u >> 16) & 1)) >> 16
  return r.astype(np.uint16).view(np.int16)


@pytest.mark.parametrize('fmt', list(FORMATS))
@pytest.mark.parametrize('channels', ['rgb', 'bgr'])
@pytest.mark.parametrize('dtype', DTYPES, ids=['f32', 'f16', 'bf16'])
def test_oracle_equals_the_documented_formula(dtype, channels, fmt):
  """Every byte value in every channel: the crop [3, 256, 3] has byte v at (y, v) in channel (c + y) % 3."""
  mean, std = FORMATS[fmt]['mean'], FORMATS[fmt]['std']
  v = np.arange(256, dtype=np.uint8)
  crop = np.zeros((3, 256, 3), np.uint8)
  for y in range(3):
    for c in range(3):
      crop[y, :, c] = np.roll(v, 37 * y + 11 * c)
  got = bits(normalize(crop[None], dtype, channels, mean, std))[0].numpy()
  src = crop[..., ::-1] if channels == 'rgb' else crop
  with np.errstate(over='ignore', divide='ignore', invalid='ignore'):
    for c in range(3):
      x = src[..., c].astype(np.float32) / np.float32(255)
      want = (x - np.float32(mean[c])) / np.float32(std[c])
      assert want.dtype == np.float32
      assert np.array_equal(got[c], _round(want, dtype)), (dtype, channels, fmt, c)


def test_pack_rule():
  u8 = np.arange(4 * 3 * 2 * 2 * 3, dtype=np.uint8).reshape(4, 3, 2, 2, 3)
  batch, off = pack(u8, [2, 3, 1, 0], {0, 2, 3}, torch.float32, 'bgr', (0, 0, 0), (1, 1, 1))
  assert off.tolist() == [0, 2, 2, 3, 3]
  want = np.concatenate([u8[0, :2], u8[2, :1]]).transpose(0, 3, 1, 2).astype(np.float32) / np.float32(255)
  assert np.array_equal(batch.numpy(), want)


def test_crop_tensor_layout_matches_the_header():
  fields = ['type', 'order', 'mean', 'std', 'rows_cap', 'out', 'out_offsets']
  offs = [getattr(L.CropTensor, f).offset for f in fields]
  assert [C.sizeof(L.CropTensor)] + offs == [56, 0, 4, 8, 20, 32, 40, 48]
  assert (L.CT_CROP_F32, L.CT_CROP_F16, L.CT_CROP_BF16, L.CT_CROP_RGB, L.CT_CROP_BGR) == (0, 1, 2, 0, 1)
  assert 'ct_crop_boxes_tensor' in L.EXPORTS
  cc = shutil.which('cc') or shutil.which('gcc')
  if cc is None:
    pytest.skip('no C compiler to read the header')
  prog = '#include <stddef.h>\n#include <stdio.h>\n#include "ctb200.h"\nint main(void) {\n  printf("%zu", ' \
      'sizeof(ct_crop_tensor));\n' + ''.join('  printf(" %%zu", offsetof(ct_crop_tensor, %s));\n' % f for f in fields) + \
      '  printf(" %d %d %d %d %d\\n", CT_CROP_F32, CT_CROP_F16, CT_CROP_BF16, CT_CROP_RGB, CT_CROP_BGR);\n' \
      '  return 0;\n}\n'
  with tempfile.TemporaryDirectory() as tmp:
    with open(os.path.join(tmp, 'p.c'), 'w') as f:
      f.write(prog)
    exe = os.path.join(tmp, 'p')
    subprocess.run([cc, '-I', os.path.join(ROOT, 'include'), os.path.join(tmp, 'p.c'), '-o', exe], check=True)
    got = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()
  assert [int(v) for v in got] == [56] + offs + [0, 1, 2, 0, 1]


def test_crop_boxes_tensor_refuses_before_launching(built_lib):
  """Each invalid argument returns -1 with a message from the host checks and launches nothing (no GPU here)."""
  lib = L.lib()

  def desc():
    d = L.CropDesc()
    d.buf = d.frames = d.rows = d.counts = d.out_counts = 64   # never dereferenced: validation fails first
    d.buf_bytes, d.row_floats, d.rows_per_stream, d.counts_stride, d.active_col = 1 << 20, 13, 300, 2, 12
    d.K, d.out_h, d.out_w = 100, 256, 128
    return d

  def tensor():
    t = L.CropTensor()
    t.type, t.order, t.rows_cap, t.out, t.out_offsets = L.CT_CROP_F16, L.CT_CROP_RGB, 200, 256, 64
    t.mean[:], t.std[:] = IMAGENET['mean'], IMAGENET['std']
    return t

  def fails(msg, d=None, t=None, streams=None, n=2, n_streams=2):
    lib.ct_reset_launch_count()
    d = d if d is not None else desc()
    t = t if t is not None else tensor()
    assert lib.ct_crop_boxes_tensor(C.byref(d), C.byref(t), streams, n, n_streams, None) == -1
    assert msg in lib.ct_last_error(), lib.ct_last_error()
    assert lib.ct_launch_count() == 0

  lib.ct_reset_launch_count()
  assert lib.ct_crop_boxes_tensor(None, C.byref(tensor()), None, 2, 2, None) == -1
  assert lib.ct_crop_boxes_tensor(C.byref(desc()), None, None, 2, 2, None) == -1
  assert lib.ct_launch_count() == 0
  # what ct_crop_boxes refuses (its uint8 out aside: not read here)
  for field in ('buf', 'frames', 'rows', 'counts', 'out_counts'):
    d = desc()
    setattr(d, field, None)
    fails(b'null pointer', d)
  fails(b'bad batch', n=0)
  fails(b'bad batch', n_streams=0)
  fails(b'bad batch', n=65536, n_streams=65536)
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
  # the tensor's own
  for field in ('out', 'out_offsets'):
    t = tensor()
    setattr(t, field, None)
    fails(b'null pointer', t=t)
  for value in (3, -1):
    t = tensor()
    t.type = value
    fails(b'unknown element type', t=t)
    t = tensor()
    t.order = 2 if value == 3 else -1
    fails(b'unknown channel order', t=t)
  for key, c, value in (('mean', 0, np.nan), ('mean', 2, np.inf), ('std', 1, -np.inf), ('std', 0, np.nan),
                        ('std', 2, 0.0), ('std', 1, -0.0)):
    t = tensor()
    getattr(t, key)[c] = value
    fails(b'finite, std != 0', t=t)
  t = tensor()
  t.rows_cap = 199
  fails(b'rows_cap < n * K', t=t)
  d, t = desc(), tensor()
  d.K, t.rows_cap = 65535, 1 << 40
  fails(b'n * K above', d, t, n=40000, n_streams=40000)
  for typ, addr in ((L.CT_CROP_F16, 257), (L.CT_CROP_BF16, 259), (L.CT_CROP_F32, 258)):
    t = tensor()
    t.type, t.out = typ, addr
    fails(b'aligned', t=t)


BAD_FORMATS = [
    ('dict', ('float16', 'rgb')),
    ('exactly', {'dtype': torch.float16, 'channels': 'rgb', 'mean': (0, 0, 0)}),
    ('exactly', dict(IMAGENET, dtype=torch.float16, channels='rgb', scale=1)),
    ('dtype', dict(IMAGENET, dtype=torch.float64, channels='rgb')),
    ('dtype', dict(IMAGENET, dtype='float16', channels='rgb')),
    ('dtype', dict(IMAGENET, dtype=np.float16, channels='rgb')),
    ('dtype', dict(IMAGENET, dtype=torch.uint8, channels='rgb')),
    ('channels', dict(IMAGENET, dtype=torch.float16, channels='RGB')),
    ('channels', dict(IMAGENET, dtype=torch.float16, channels=0)),
    ('mean', {'dtype': torch.float16, 'channels': 'rgb', 'mean': (0.5, 0.5), 'std': (1, 1, 1)}),
    ('mean', {'dtype': torch.float16, 'channels': 'rgb', 'mean': 0.5, 'std': (1, 1, 1)}),
    ('mean', {'dtype': torch.float16, 'channels': 'rgb', 'mean': (0.5, '0.5', 0.5), 'std': (1, 1, 1)}),
    ('mean', {'dtype': torch.float16, 'channels': 'rgb', 'mean': (0.5, True, 0.5), 'std': (1, 1, 1)}),
    ('mean', {'dtype': torch.float16, 'channels': 'rgb', 'mean': (0.5, np.nan, 0.5), 'std': (1, 1, 1)}),
    ('mean', {'dtype': torch.float16, 'channels': 'rgb', 'mean': (0.5, 1e39, 0.5), 'std': (1, 1, 1)}),
    ('std', {'dtype': torch.float16, 'channels': 'rgb', 'mean': (0, 0, 0), 'std': (1, 0, 1)}),
    ('std', {'dtype': torch.float16, 'channels': 'rgb', 'mean': (0, 0, 0), 'std': (1, 1, 1e-50)}),
    ('std', {'dtype': torch.float16, 'channels': 'rgb', 'mean': (0, 0, 0), 'std': (1, -np.inf, 1)}),
    ('std', {'dtype': torch.float16, 'channels': 'rgb', 'mean': (0, 0, 0), 'std': (1, 1, 1, 1)}),
]


def test_runner_refuses_bad_crop_format():
  """Raised at construction before anything else is looked at: no model, no device, no CUDA work."""
  from centertrack_b200.runner import StreamRunner, check_crop_format
  opt = make_opt('mot')
  kw = dict(opt=opt, device_tracking=True, frame_sizes=[(1080, 1920)])
  good = dict(IMAGENET, dtype=torch.bfloat16, channels='bgr')
  with pytest.raises(ValueError, match='crop_format.*crop_size'):
    StreamRunner(None, 1, 544, 960, crop_format=good, **kw)
  for match, bad in BAD_FORMATS:
    with pytest.raises(ValueError, match='crop_format.*' + match):
      StreamRunner(None, 1, 544, 960, crop_size=(64, 32), crop_format=bad, **kw)
  got = check_crop_format(dict(good, mean=np.array([0, 1, 2]), std=[1e-40, -2, 3]), (64, 32))
  assert got['dtype'] is torch.bfloat16 and got['channels'] == 'bgr'
  assert got['mean'] == (0.0, 1.0, 2.0) and got['std'] == tuple(float(np.float32(v)) for v in (1e-40, -2, 3))
  assert check_crop_format(None, (64, 32)) is None and check_crop_format(None, None) is None


def test_track_videos_refuses_a_crop_format_in_place_of_crops():
  from centertrack_b200.videos import track_videos

  class R(object):
    tracker, post, crop, crop_format = object(), None, (8, 8), None
  for bad in ('rgb', dict(IMAGENET, dtype=torch.float16, channels='rgb'), torch.float16, 2):
    with pytest.raises(ValueError, match='crops must be True or False'):
      next(track_videos(R(), [], crops=bad))
