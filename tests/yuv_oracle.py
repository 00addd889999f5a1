"""The reference of StreamRunner's NV12 / I420 frames: cv2.cvtColor(COLOR_YUV2BGR_NV12 / _I420) restated in int64 numpy
(equal to cv2 byte for byte: tests/test_yuv_frames_host.py).  Its BGR output feeds ct_oracle.warp_affine_u8 /
normalize_chw / stem_pixels like any camera frame."""
import numpy as np

# cv2's BT.601 limited-range coefficients in 20-bit fixed point (color_yuv.simd.hpp ITUR_BT_601_*)
CY, CUB, CUG, CVG, CVR, SHIFT = 1220542, 2116026, -409993, -852492, 1673527, 20


def yuv420_planes(buf, h, w, fmt):
  """buf: uint8 [3h/2, w] (any row stride) in cv2's NV12 or I420 layout -> (Y [h, w], U [h/2, w/2], V [h/2, w/2]).
  I420's chroma planes are read as cv2 reads them from a strided image: half-width rows, two to a row of buf."""
  buf = np.asarray(buf)
  assert buf.dtype == np.uint8 and buf.shape == (h * 3 // 2, w) and h % 2 == 0 and w % 2 == 0, (buf.shape, h, w)
  if fmt == 'nv12':
    uv = buf[h:]
    return buf[:h], uv[:, 0::2], uv[:, 1::2]
  if fmt == 'i420':
    half = buf[h:].reshape(h, w // 2)
    return buf[:h], half[:h // 2], half[h // 2:]
  raise ValueError('fmt: %r' % (fmt,))


def yuv420_to_bgr(buf, h, w, fmt):
  """cv2.cvtColor(buf, COLOR_YUV2BGR_NV12 or _I420) -> uint8 [h, w, 3]: per pixel, with the U, V of its 2x2 block,
  y = max(Y - 16, 0) CY, B = sat((y + 2^19 + CUB u) >> 20), G = sat((y + 2^19 + CVG v + CUG u) >> 20),
  R = sat((y + 2^19 + CVR v) >> 20), u = U - 128, v = V - 128."""
  Y, U, V = yuv420_planes(buf, h, w, fmt)
  up = lambda p: np.repeat(np.repeat(p.astype(np.int64) - 128, 2, 0), 2, 1)
  u, v = up(U), up(V)
  y = np.maximum(Y.astype(np.int64) - 16, 0) * CY + (1 << (SHIFT - 1))
  b = (y + CUB * u) >> SHIFT
  g = (y + CVG * v + CUG * u) >> SHIFT
  r = (y + CVR * v) >> SHIFT
  return np.clip(np.stack([b, g, r], -1), 0, 255).astype(np.uint8)


def random_yuv420(h, w, seed, pitch=None, fill=0xA5):
  """A random 4:2:0 frame as a uint8 [3h/2, pitch] array (pitch >= w, the padding columns `fill`, never read); the
  frame itself is the view [:, :w]."""
  pitch = w if pitch is None else pitch
  buf = np.full((h * 3 // 2, pitch), fill, np.uint8)
  buf[:, :w] = np.random.RandomState(seed).randint(0, 256, size=(h * 3 // 2, w)).astype(np.uint8)
  return buf


def bgr_to_yuv420(bgr, fmt):
  """A 4:2:0 frame of fmt whose conversion is close to bgr (cv2.cvtColor COLOR_BGR2YUV_I420, re-laid as NV12 when asked):
  test content with image structure rather than noise."""
  import cv2
  h, w = bgr.shape[:2]
  i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
  if fmt == 'i420':
    return i420
  _, U, V = yuv420_planes(i420, h, w, 'i420')
  out = np.empty_like(i420)
  out[:h] = i420[:h]
  out[h:, 0::2], out[h:, 1::2] = U, V
  return out
