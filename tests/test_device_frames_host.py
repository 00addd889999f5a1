"""Device frames without a GPU: device_frame_source (step_frames' parsing of CUDA tensors into ct_frame_src) on CPU
tensors and views, every refusal, the numpy staging oracle against cv2, and the ct_frame_src ABI."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import cv2
import numpy as np
import pytest
import torch

from conftest import ROOT
from centertrack_b200 import _lib as L
from centertrack_b200.runner import device_frame_source, is_device_frame
from device_frames_oracle import stage_oracle
from yuv_oracle import random_yuv420, yuv420_planes, yuv420_to_bgr

CPU = torch.device('cpu')


def _rand(shape, seed):
  return torch.from_numpy(np.random.RandomState(seed).randint(0, 256, size=shape).astype(np.uint8))


def _src(x, fmt, layout='bgr'):
  return device_frame_source(x, fmt, layout, CPU, 'frames[3]')


# ------------------------------------------------------------------------------------------------ parsing

@pytest.mark.parametrize('layout', ['bgr', 'rgb'])
def test_interleaved_contiguous_padded_and_offset_views(layout):
  code = L.CT_SRC_BGR if layout == 'bgr' else L.CT_SRC_RGB
  x = _rand((5, 7, 3), 0)
  hw, s = _src(x, 'bgr', layout)
  assert hw == (5, 7) and s.layout == code and s.plane[0] == x.data_ptr() and s.pitch[0] == 21
  surf = _rand((9, 12, 3), 1)                              # a wider, taller surface; the frame its top-left corner
  v = surf[:5, :7]
  hw, s = _src(v, 'bgr', layout)
  assert hw == (5, 7) and s.plane[0] == surf.data_ptr() and s.pitch[0] == 36
  v = surf[2:7, 3:10]                                      # an offset view
  hw, s = _src(v, 'bgr', layout)
  assert hw == (5, 7) and s.plane[0] == surf.data_ptr() + 2 * 36 + 3 * 3 and s.pitch[0] == 36
  hw, s = _src(_rand((1, 1, 3), 2), 'bgr', layout)        # a single pixel: its pitch is its row
  assert hw == (1, 1) and s.pitch[0] == 3


def test_planar_rgb_views():
  x = _rand((3, 4, 6), 0)
  hw, s = _src(x, 'bgr', 'rgb_planar')
  assert hw == (4, 6) and s.layout == L.CT_SRC_RGB_PLANAR
  assert [s.plane[c] for c in range(3)] == [x.data_ptr() + 24 * c for c in range(3)] and list(s.pitch) == [6] * 3
  surf = _rand((3, 8, 16), 1)
  v = surf[:, 1:5, 2:8]
  hw, s = _src(v, 'bgr', 'rgb_planar')
  assert hw == (4, 6) and [s.plane[c] for c in range(3)] == [surf.data_ptr() + 128 * c + 16 + 2 for c in range(3)]
  assert list(s.pitch) == [16] * 3


def test_nv12_one_tensor_and_planes_with_chroma_at_an_aligned_height():
  h, w = 1080, 1920
  x = _rand((h * 3 // 2, w), 0)
  hw, s = _src(x, 'nv12')
  assert hw == (h, w) and s.layout == L.CT_SRC_NV12
  assert (s.plane[0], s.plane[1], s.pitch[0], s.pitch[1]) == (x.data_ptr(), x.data_ptr() + h * w, w, w)
  surf = torch.zeros((1088 + 544, 2048), dtype=torch.uint8)    # a decoder surface: chroma at the aligned height 1088
  Y, UV = surf[:h, :w], surf[1088:1088 + h // 2, :w]
  hw, s = _src((Y, UV), 'nv12')
  assert hw == (h, w) and s.plane[0] == surf.data_ptr() and s.plane[1] == surf.data_ptr() + 1088 * 2048
  assert (s.pitch[0], s.pitch[1]) == (2048, 2048)
  v = torch.zeros((h * 3 // 2, 2048), dtype=torch.uint8)[:, :w]   # one pitched tensor
  hw, s = _src(v, 'nv12')
  assert hw == (h, w) and s.plane[1] == v.data_ptr() + h * 2048 and s.pitch[1] == 2048


def test_i420_one_tensor_and_triples():
  h, w = 6, 10
  x = _rand((9, 10), 0)
  hw, s = _src(x, 'i420')
  assert hw == (h, w) and s.layout == L.CT_SRC_I420
  assert [s.plane[i] for i in range(3)] == [x.data_ptr(), x.data_ptr() + 60, x.data_ptr() + 75]
  assert list(s.pitch) == [10, 5, 5]
  Y, U, V = _rand((8, 16), 1)[:h, :w], _rand((4, 8), 2)[1:4, 2:7], _rand((3, 5), 3)
  hw, s = _src((Y, U, V), 'i420')
  assert hw == (h, w) and list(s.pitch) == [16, 8, 5]
  assert [s.plane[i] for i in range(3)] == [Y.data_ptr(), U.data_ptr(), V.data_ptr()]


def test_is_device_frame():
  t = torch.zeros(2, 2, 3, dtype=torch.uint8)
  assert is_device_frame(t) and is_device_frame((t, t))
  assert not is_device_frame(np.zeros((2, 2, 3), np.uint8)) and not is_device_frame(None)
  assert not is_device_frame(()) and not is_device_frame((t, np.zeros(2)))


def _refuse(x, fmt, layout, match, device=CPU):
  with pytest.raises(ValueError, match=match) as e:
    device_frame_source(x, fmt, layout, device, 'frames[3]')
  assert 'frames[3]' in str(e.value) or 'layout' in str(e.value)


def test_refusals():
  u8 = lambda *s: torch.zeros(s, dtype=torch.uint8)
  _refuse(torch.zeros((4, 4, 3)), 'bgr', 'bgr', r'frames\[3\]: expected a uint8 tensor, got torch.float32')
  _refuse(u8(4, 4, 3), 'bgr', 'bgr', r"frames\[3\]: on cpu, not on the runner's device cuda:0",
          device=torch.device('cuda', 0))
  _refuse((u8(4, 4), u8(2, 4).float()), 'nv12', 'bgr', r'frames\[3\]\[1\]: expected a uint8 tensor')
  # innermost strides
  _refuse(u8(4, 4, 4)[..., :3], 'bgr', 'bgr', r'frames\[3\]: the innermost stride must be 1 and the pixel stride 3')
  _refuse(u8(3, 5, 4).permute(1, 2, 0), 'bgr', 'rgb', r'innermost stride')     # a CHW tensor viewed as HWC
  _refuse(u8(3, 6, 4).transpose(1, 2), 'bgr', 'rgb_planar', r'frames\[3\]: the innermost stride must be 1')
  _refuse(u8(8, 6).t(), 'nv12', 'bgr', r'frames\[3\]: the innermost stride must be 1')
  _refuse((u8(4, 8), u8(8, 2).t()), 'nv12', 'bgr', r'frames\[3\]\[1\]: the innermost stride must be 1')
  # pitch shorter than a row
  _refuse(torch.as_strided(u8(64), (4, 5, 3), (12, 3, 1)), 'bgr', 'bgr', r'row pitch of 12 bytes is shorter than a '
                                                                          r'row of 15')
  _refuse(torch.as_strided(u8(96), (3, 4, 6), (24, 5, 1)), 'bgr', 'rgb_planar', r'row pitch of 5 bytes')
  _refuse(torch.as_strided(u8(64), (6, 4), (3, 1)), 'nv12', 'bgr', r'row pitch of 3 bytes is shorter than a row of 4')
  _refuse((u8(4, 8), torch.as_strided(u8(64), (2, 4), (2, 1)), u8(2, 4)), 'i420', 'bgr', r'frames\[3\]\[1\]: row pitch')
  # plane shapes that disagree
  _refuse((u8(4, 8), u8(2, 6)), 'nv12', 'bgr', r'frames\[3\]\[1\]: expected shape \(2, 8\) for a Y plane of \(4, 8\)')
  _refuse((u8(4, 8), u8(2, 4), u8(3, 4)), 'i420', 'bgr', r'frames\[3\]\[2\]: expected shape \(2, 4\)')
  _refuse((u8(4, 8), u8(2, 8), u8(2, 8)), 'nv12', 'bgr', r'expected NV12 planes \(Y, UV\), got 3 tensors')
  _refuse((u8(4, 8), u8(2, 4)), 'i420', 'bgr', r'expected I420 planes \(Y, U, V\), got 2 tensors')
  _refuse(u8(4, 3, 4), 'bgr', 'bgr', r"layout 'bgr' expects shape \[h, w, 3\]")
  _refuse(u8(4, 4, 3), 'bgr', 'rgb_planar', r"layout 'rgb_planar' expects shape \[3, h, w\]")
  # odd 4:2:0 sizes
  _refuse((u8(5, 8), u8(2, 8)), 'nv12', 'bgr', r'frames\[3\]\[0\]: Y plane of shape \(5, 8\); NV12 frames have an even')
  _refuse((u8(4, 7), u8(2, 3), u8(2, 3)), 'i420', 'bgr', r'I420 frames have an even')
  _refuse(u8(9, 7), 'nv12', 'bgr', r'expected a NV12 frame of shape \[3h/2, w\]')
  _refuse(u8(8, 8), 'i420', 'bgr', r'rows a multiple of 3')
  # an I420 tensor of pitched rows; layouts
  _refuse(u8(6, 16)[:, :8], 'i420', 'bgr', r'needs rows of exactly w = 8 bytes')
  _refuse(u8(6, 8), 'nv12', 'rgb', r"layout='rgb': a NV12 runner takes its own format only")
  _refuse(u8(4, 4, 3), 'bgr', 'bgra', r"layout: expected one of \['bgr', 'rgb', 'rgb_planar'\]")


def test_one_tensor_tuple_on_bgr_and_two_refused():
  t = torch.zeros((4, 4, 3), dtype=torch.uint8)
  with pytest.raises(ValueError, match=r'a BGR runner takes one tensor per frame, got 2'):
    device_frame_source((t, t), 'bgr', 'bgr', CPU, 'frames[0]')


# ------------------------------------------------------------------------------------------------ the oracle

SIZES = [(1, 1), (2, 2), (3, 5), (17, 31), (480, 640), (1080, 1920)]


@pytest.mark.parametrize('h,w', SIZES)
def test_oracle_equals_cv2_on_rgb_and_planar(h, w):
  rgb = np.random.RandomState(h * 7 + w).randint(0, 256, size=(h, w, 3)).astype(np.uint8)
  want = cv2.cvtColor(rgb, cv2.COLOR_RGB2BGR)
  assert np.array_equal(stage_oracle(torch.from_numpy(rgb), 'bgr', 'rgb'), want)
  assert np.array_equal(stage_oracle(torch.from_numpy(np.ascontiguousarray(rgb.transpose(2, 0, 1))), 'bgr',
                                     'rgb_planar'), want)
  assert np.array_equal(stage_oracle(torch.from_numpy(want), 'bgr', 'bgr'), want)
  wide = torch.from_numpy(np.pad(rgb, ((0, 3), (0, 5), (0, 0))))[:h, :w]          # a pitched view
  assert np.array_equal(stage_oracle(wide, 'bgr', 'rgb'), want)


@pytest.mark.parametrize('fmt', ['nv12', 'i420'])
@pytest.mark.parametrize('h,w', [(2, 2), (6, 10), (480, 640), (1080, 1920)])
def test_oracle_4_2_0_from_planes_converts_as_cv2(fmt, h, w):
  buf = random_yuv420(h, w, h + w)
  Y, U, V = yuv420_planes(buf, h, w, fmt)
  if fmt == 'nv12':
    planes = (torch.from_numpy(np.ascontiguousarray(Y)), torch.from_numpy(np.ascontiguousarray(buf[h:])))
  else:
    planes = tuple(torch.from_numpy(np.ascontiguousarray(p)) for p in (Y, U, V))
  got = stage_oracle(planes, fmt)
  assert np.array_equal(got, buf)
  code = cv2.COLOR_YUV2BGR_NV12 if fmt == 'nv12' else cv2.COLOR_YUV2BGR_I420
  assert np.array_equal(yuv420_to_bgr(got, h, w, fmt), cv2.cvtColor(buf, code))
  assert np.array_equal(stage_oracle(torch.from_numpy(buf), fmt), buf)


# ------------------------------------------------------------------------------------------------ the ABI

def test_frame_src_layout_matches_the_header():
  assert C.sizeof(L.FrameSrc) == 56
  assert (L.FrameSrc.plane.offset, L.FrameSrc.pitch.offset, L.FrameSrc.layout.offset) == (0, 24, 48)
  assert (L.CT_SRC_BGR, L.CT_SRC_RGB, L.CT_SRC_RGB_PLANAR, L.CT_SRC_NV12, L.CT_SRC_I420) == (0, 1, 2, 3, 4)
  assert 'ct_stage_frames' in L.EXPORTS
  cc = shutil.which('cc') or shutil.which('gcc')
  if cc is None:
    pytest.skip('no C compiler to read the header')
  prog = r'''#include <stddef.h>
#include <stdio.h>
#include "ctb200.h"
int main(void) {
  printf("%zu %zu %zu %zu %d %d %d %d %d\n", sizeof(ct_frame_src), offsetof(ct_frame_src, plane),
         offsetof(ct_frame_src, pitch), offsetof(ct_frame_src, layout), CT_SRC_BGR, CT_SRC_RGB, CT_SRC_RGB_PLANAR,
         CT_SRC_NV12, CT_SRC_I420);
  return 0;
}
'''
  with tempfile.TemporaryDirectory() as tmp:
    with open(os.path.join(tmp, 'p.c'), 'w') as f:
      f.write(prog)
    exe = os.path.join(tmp, 'p')
    subprocess.run([cc, '-I', os.path.join(ROOT, 'include'), os.path.join(tmp, 'p.c'), '-o', exe], check=True)
    got = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()
  assert [int(v) for v in got] == [56, 0, 24, 48, 0, 1, 2, 3, 4]


def test_stage_frames_refuses_before_launching(built_lib):
  """Every invalid argument is CT_ERR_INVALID from the host checks, with no GPU on this machine."""
  lib = L.lib()
  buf, nbytes = C.c_void_p(256), 1 << 20

  def one(layout, fmt, h, w, pitch=(4096,) * 3, step=None, planes=(4096, 8192, 12288), offset=0, limit=nbytes, n=1):
    s = L.FrameSrc()
    for i in range(3):
      s.plane[i], s.pitch[i] = planes[i], pitch[i]
    s.layout = layout
    f = L.Frame()
    f.offset, f.h, f.w, f.format = offset, h, w, fmt
    f.step = step if step is not None else (w if fmt != L.CT_FRAME_BGR else 3 * w)
    return lib.ct_stage_frames(C.byref(s), C.byref(f), n, buf, limit, None)

  B, N, I = L.CT_FRAME_BGR, L.CT_FRAME_NV12, L.CT_FRAME_I420
  assert one(L.CT_SRC_RGB, B, 4, 4, n=0) == L.CT_ERR_INVALID
  assert one(7, B, 4, 4) == L.CT_ERR_INVALID and b'unknown source layout' in lib.ct_last_error()
  for layout, fmt in ((L.CT_SRC_NV12, B), (L.CT_SRC_RGB, N), (L.CT_SRC_I420, N), (L.CT_SRC_NV12, I)):
    assert one(layout, fmt, 4, 4) == L.CT_ERR_INVALID and b'destination format' in lib.ct_last_error()
  assert one(L.CT_SRC_BGR, B, 0, 4) == L.CT_ERR_INVALID
  assert one(L.CT_SRC_NV12, N, 5, 4) == L.CT_ERR_INVALID and b'even' in lib.ct_last_error()
  assert one(L.CT_SRC_I420, I, 4, 6 + 1) == L.CT_ERR_INVALID
  assert one(L.CT_SRC_RGB_PLANAR, B, 4, 4, planes=(4096, 0, 8192)) == L.CT_ERR_INVALID
  assert b'null source plane' in lib.ct_last_error()
  assert one(L.CT_SRC_I420, I, 4, 8, planes=(4096, 8192, 0)) == L.CT_ERR_INVALID
  assert one(L.CT_SRC_RGB, B, 4, 8, pitch=(23, 0, 0)) == L.CT_ERR_INVALID
  assert b'source pitch' in lib.ct_last_error()
  assert one(L.CT_SRC_I420, I, 4, 8, pitch=(8, 4, 3)) == L.CT_ERR_INVALID
  assert one(L.CT_SRC_BGR, B, 4, 8, step=23) == L.CT_ERR_INVALID and b'destination step' in lib.ct_last_error()
  assert one(L.CT_SRC_NV12, N, 4, 8, limit=47) == L.CT_ERR_INVALID and b'past buf_bytes' in lib.ct_last_error()
  assert one(L.CT_SRC_BGR, B, 4, 8, offset=16, limit=16 + 95) == L.CT_ERR_INVALID
  s, f = L.FrameSrc(), L.Frame()
  assert lib.ct_stage_frames(None, C.byref(f), 1, buf, nbytes, None) == L.CT_ERR_INVALID
  assert lib.ct_stage_frames(C.byref(s), C.byref(f), 1, None, nbytes, None) == L.CT_ERR_INVALID
