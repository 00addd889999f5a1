"""The reference of ct_stage_frames: what StreamRunner's frame slot holds after a device frame is staged, in numpy.
A frame given as a tensor (or a tuple of plane tensors) on any device -> the dense bytes of its slot layout: BGR rows of
3w bytes, or cv2's [3h/2, w] NV12 / I420 layout."""
import numpy as np


def _np(t):
  return t.cpu().numpy() if hasattr(t, 'cpu') else np.asarray(t)


def stage_oracle(x, fmt, layout='bgr'):
  """x: a device frame as step_frames takes it (fmt: the runner's frame_format) -> uint8 [h, w, 3] BGR or [3h/2, w]."""
  if fmt == 'bgr':
    a = _np(x)
    if layout == 'bgr':
      return a.copy()
    if layout == 'rgb':
      return np.ascontiguousarray(a[..., ::-1])
    if layout == 'rgb_planar':
      return np.ascontiguousarray(a.transpose(1, 2, 0)[..., ::-1])
    raise ValueError(layout)
  if not isinstance(x, tuple):
    return _np(x).copy()
  planes = [_np(t) for t in x]
  h, w = planes[0].shape
  if fmt == 'nv12':
    return np.concatenate(planes, 0)
  return np.concatenate([p.reshape(-1) for p in planes]).reshape(h * 3 // 2, w)
