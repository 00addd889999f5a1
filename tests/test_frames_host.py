"""StreamRunner's frames mode on the host (no GPU): each stream's geometry is Detector.pre_process's meta for its source
size, the warp map is the one pre_process_device samples with, and ct_pack_stem_frames validates its arguments before
it touches the device."""
import ctypes as C

import numpy as np
import pytest

from centertrack_b200 import _lib as L
from helpers import HOST_CASES, host_case_inputs, make_opt


def _host_detector(opt):
  from centertrack_b200.dataset_info import get_dataset
  from centertrack_b200.detector import Detector
  det = object.__new__(Detector)
  ds = get_dataset(opt.dataset)
  det.opt = opt
  det.mean = np.array(ds.mean, dtype=np.float32).reshape(1, 1, 3)
  det.std = np.array(ds.std, dtype=np.float32).reshape(1, 1, 3)
  det.rest_focal_length = opt.test_focal_length if opt.test_focal_length >= 0 else ds.rest_focal_length
  det.flip_idx = ds.flip_idx
  return det


def _geometry_only_runner(opt, sizes, H, W):
  """A StreamRunner with nothing but the frames-mode geometry (what its constructor computes before any allocation)."""
  from centertrack_b200.runner import StreamRunner
  r = object.__new__(StreamRunner)
  r.B, r.H, r.W, r.opt = len(sizes), H, W, opt
  r.frames_mode = True
  calibs = r._frame_geometry(sizes, None)
  return r, calibs


@pytest.mark.parametrize('i', range(len(HOST_CASES)), ids=[c[0] for c in HOST_CASES])
def test_frames_geometry_is_the_pre_process_meta(i, monkeypatch):
  import cv2
  import torch
  name, extra, hw, _ = HOST_CASES[i]
  opt = make_opt('coco_tracking', extra)
  det = _host_detector(opt)
  image, _, _ = host_case_inputs(i, hw)
  _, ref = det.pre_process(image, 1.0, {})
  r, calibs = _geometry_only_runner(opt, [hw, hw], ref['inp_height'], ref['inp_width'])
  for b in range(2):
    got = r.meta(b)
    assert sorted(got) == sorted(ref), (name, sorted(got), sorted(ref))
    for k in ref:
      assert np.asarray(got[k]).dtype == np.asarray(ref[k]).dtype, (name, k)
      assert np.array_equal(np.asarray(got[k]), np.asarray(ref[k])), (name, k)
    assert np.array_equal(calibs[b], ref['calib'].astype(np.float32))
  # the dst -> src map: cv2's own inversion, and what pre_process_device hands ct_warp_affine_normalize
  minv = np.frombuffer(bytes(r.frames[0].minv), np.float64)
  assert np.array_equal(minv, cv2.invertAffineTransform(ref['trans_input']).reshape(6)), name
  seen = {}

  class _Lib(object):
    def ct_warp_affine_normalize(self, src, B, h, w, step, minv_ptr, *rest):
      seen['minv'] = np.array((C.c_double * 6).from_address(minv_ptr.value))
      seen['shape'] = (B, h, w, step)
      return 0

  monkeypatch.setattr(L, 'lib', lambda: _Lib())
  monkeypatch.setattr(L, 'stream_ptr', lambda: None)
  opt.device = torch.device('cpu')
  _, meta = det.pre_process_device(image, 1.0, {})
  assert np.array_equal(seen['minv'], minv) and seen['shape'] == (1, hw[0], hw[1], 3 * hw[1])
  for k in ref:
    assert np.array_equal(np.asarray(meta[k]), np.asarray(ref[k])), (name, k)
  f = r.frames[1]
  assert (f.h, f.w, f.step) == (hw[0], hw[1], 3 * hw[1]) and f.offset % 16 == 0 and f.offset >= hw[0] * hw[1] * 3


def test_ragged_slots_and_calibs_follow_each_source():
  opt = make_opt('mot')
  sizes = [(1080, 1920), (544, 960), (480, 854), (1081, 1921)]
  r, calibs = _geometry_only_runner(opt, sizes, 544, 960)
  ends = [f.offset + f.h * f.w * 3 for f in r.frames]
  assert [f.offset for f in r.frames] == [0] + [(e + 15) // 16 * 16 for e in ends[:-1]]
  assert r.slot_bytes == (ends[-1] + 15) // 16 * 16
  for b, (h, w) in enumerate(sizes):
    assert np.array_equal(calibs[b][:2, 2], np.float32([w / 2., h / 2.]))   # the source's centre, odd sizes too
  assert np.array_equal(np.frombuffer(bytes(r.frames[1].minv), np.float64), [1, 0, 0, 0, 1, 0])   # identity


@pytest.mark.parametrize('extra,size,HW', [([], (480, 640), (512, 512)),
                                           (['--keep_res'], (480, 640), (544, 960)),
                                           (['--fix_short', '96'], (150, 400), (96, 192))])
def test_frame_size_with_another_input_size_is_refused(extra, size, HW):
  opt = make_opt('mot', extra)
  with pytest.raises(ValueError, match='network input'):
    _geometry_only_runner(opt, [(544, 960), size], *HW)


def test_pack_stem_frames_rejects_bad_arguments_without_a_gpu(built_lib):
  lib = L.lib()
  frames = (L.Frame * 2)()
  for f in frames:
    f.h, f.w, f.step = 4, 5, 15
  frames[1].offset = 64
  p = C.c_void_p(16)
  mean = np.zeros(3, np.float32)
  std = np.ones(3, np.float32)
  m, s = C.c_void_p(mean.ctypes.data), C.c_void_p(std.ctypes.data)

  def call(cur=p, fr=frames, B=2, out=p, H=8, W=8, ms=m):
    return lib.ct_pack_stem_frames(cur, None, fr, B, ms, s, None, out, H, W, None)

  for kwargs in (dict(cur=None), dict(fr=None), dict(out=None), dict(ms=None)):
    assert call(**kwargs) == L.CT_ERR_INVALID and b'null pointer' in lib.ct_last_error(), kwargs
  for kwargs in (dict(B=0), dict(B=-1), dict(H=0), dict(W=-8)):
    assert call(**kwargs) == L.CT_ERR_INVALID and b'bad shape' in lib.ct_last_error(), kwargs
  frames[1].step = 14                                       # row pitch below 3 w
  assert call() == L.CT_ERR_INVALID and b'step >= 3 w' in lib.ct_last_error()
  frames[1].step, frames[1].offset = 15, -16
  assert call() == L.CT_ERR_INVALID and b'frame descriptor' in lib.ct_last_error()
  frames[1].offset, frames[0].h = 64, 0
  assert call() == L.CT_ERR_INVALID and b'frame descriptor' in lib.ct_last_error()
