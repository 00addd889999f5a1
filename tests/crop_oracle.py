"""The reference of ct_crop_boxes: the documented crop map in numpy fp64 and ct_oracle.warp_affine_u8 (equal to
cv2.warpAffine with WARP_INVERSE_MAP byte for byte: tests/test_crops_host.py)."""
import numpy as np

import ct_oracle as co

MAX_COORD = 16384.0


def crop_map(box, out_h, out_w):
  """The dst -> src map of box (x0, y0, x1, y1), read as fp32 and widened to fp64: sx = (x1 - x0) / out_w,
  sy = (y1 - y0) / out_h, M = [sx, 0, (x0 - 0.5) + 0.5 sx, 0, sy, (y0 - 0.5) + 0.5 sy], left to right (numpy rounds
  every operation on its own)."""
  x0, y0, x1, y1 = (np.float64(v) for v in np.asarray(box, np.float32)[:4])
  sx = (x1 - x0) / np.float64(out_w)
  sy = (y1 - y0) / np.float64(out_h)
  return np.array([sx, 0.0, (x0 - 0.5) + 0.5 * sx, 0.0, sy, (y0 - 0.5) + 0.5 * sy], np.float64)


def crop(bgr, box, out_h, out_w):
  """uint8 [out_h, out_w, 3] crop of the BGR image bgr at box; zeros for a box with a non-finite coordinate or one of
  magnitude above MAX_COORD."""
  b = np.asarray(box, np.float32)[:4]
  if not np.all(np.abs(b) <= MAX_COORD):
    return np.zeros((out_h, out_w, 3), np.uint8)
  return co.warp_affine_u8(bgr, crop_map(b, out_h, out_w), out_h, out_w)
