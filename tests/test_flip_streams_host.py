"""--flip_test entry points on the host (no GPU): ct_flip_merge_heads, ct_mirror_x and ct_pack_stem_frames_flip_dev
reject null pointers, bad shapes and too many heads per launch before they launch anything; StreamRunner's flip plan is
Detector's."""
import ctypes as C

import numpy as np
import pytest

from centertrack_b200 import _lib as L


def _heads(n, C_=4):
  heads = (L.FlipHead * max(n, 1))()
  for i in range(n):
    heads[i].input, heads[i].out, heads[i].C = 16, 32, C_
  return heads


def test_flip_merge_heads_rejects_bad_arguments_without_a_gpu(built_lib):
  lib = L.lib()

  def call(heads, n, B=2, H=8, W=8):
    return lib.ct_flip_merge_heads(heads, n, B, H, W, None)

  assert call(None, 1) == L.CT_ERR_INVALID and b'null pointer' in lib.ct_last_error()
  for n in (0, -1, L.CT_FLIP_MAX_HEADS + 1):
    assert call(_heads(max(n, 1)), n) == L.CT_ERR_INVALID and b'n_heads' in lib.ct_last_error(), n
  for kw in (dict(B=0), dict(B=-3), dict(H=0), dict(W=-1)):
    assert call(_heads(2), 2, **kw) == L.CT_ERR_INVALID and b'bad shape' in lib.ct_last_error(), kw
  h = _heads(3)
  h[2].input = None
  assert call(h, 3) == L.CT_ERR_INVALID and b'null pointer' in lib.ct_last_error()
  h = _heads(3)
  h[1].out = None
  assert call(h, 3) == L.CT_ERR_INVALID and b'null pointer' in lib.ct_last_error()
  h = _heads(3)
  h[0].C = 0
  assert call(h, 3) == L.CT_ERR_INVALID and b'bad shape' in lib.ct_last_error()
  # the one-pair, one-head form keeps its checks
  p = C.c_void_p(16)
  assert lib.ct_flip_merge(None, p, 4, 8, 8, None, None, None) == L.CT_ERR_INVALID
  assert b'null pointer' in lib.ct_last_error()
  assert lib.ct_flip_merge(p, p, 0, 8, 8, None, None, None) == L.CT_ERR_INVALID
  assert b'bad shape' in lib.ct_last_error()


def test_mirror_x_rejects_bad_arguments_without_a_gpu(built_lib):
  lib = L.lib()
  p = C.c_void_p(16)

  def call(src=p, dst=p, n=2, C_=3, H=8, W=7):
    return lib.ct_mirror_x(src, dst, n, C_, H, W, None)

  for kw in (dict(src=None), dict(dst=None)):
    assert call(**kw) == L.CT_ERR_INVALID and b'null pointer' in lib.ct_last_error(), kw
  for kw in (dict(n=0), dict(C_=0), dict(H=-1), dict(W=0)):
    assert call(**kw) == L.CT_ERR_INVALID and b'bad shape' in lib.ct_last_error(), kw


def test_pack_stem_frames_flip_dev_rejects_bad_arguments_without_a_gpu(built_lib):
  """The host checks run before any launch; the descriptors live in device memory, where the kernel checks each one
  (test_invalid_descriptors_give_zeros_and_read_nothing)."""
  lib = L.lib()
  p = C.c_void_p(16)
  mean = np.zeros(3, np.float32)
  std = np.ones(3, np.float32)
  m, s = C.c_void_p(mean.ctypes.data), C.c_void_p(std.ctypes.data)

  def call(cur=p, fr=p, B=2, out=p, H=8, W=8, ms=m):
    return lib.ct_pack_stem_frames_flip_dev(cur, None, fr, B, 1024, ms, s, None, out, H, W, None)

  for kwargs in (dict(cur=None), dict(fr=None), dict(out=None), dict(ms=None)):
    assert call(**kwargs) == L.CT_ERR_INVALID and b'null pointer' in lib.ct_last_error(), kwargs
  for kwargs in (dict(B=0), dict(B=-1), dict(H=0), dict(W=-8)):
    assert call(**kwargs) == L.CT_ERR_INVALID and b'bad shape' in lib.ct_last_error(), kwargs


def test_flip_head_descriptor_matches_the_header():
  """ct_flip_head: two pointers, C, reserved, two pointers -- 40 bytes on x86-64, as the C struct lays it out."""
  assert C.sizeof(L.FlipHead) == 40
  assert [L.FlipHead.input.offset, L.FlipHead.out.offset, L.FlipHead.C.offset, L.FlipHead.perm.offset,
          L.FlipHead.sign.offset] == [0, 8, 16, 24, 32]


@pytest.mark.parametrize('cfg', ['coco_pose', 'nuscenes_ddd', 'coco_tracking'])
def test_flip_plan_is_the_detectors(cfg):
  """detector.flip_plan (what StreamRunner builds) is Detector._flip_plan's plan: same heads, perms and signs."""
  import torch
  from centertrack_b200.dataset_info import get_dataset
  from centertrack_b200.detector import Detector, flip_plan
  from helpers import make_opt
  opt = make_opt(cfg, ['--flip_test'])
  outputs = {h: torch.zeros((2, c, 4, 6)) for h, c in opt.heads.items()}

  class _Eng(object):
    pass

  eng = _Eng()
  eng.outputs, eng.device = outputs, torch.device('cpu')
  det = object.__new__(Detector)
  det.opt, det.flip_idx = opt, get_dataset(opt.dataset).flip_idx
  want = det._flip_plan(eng)
  got = flip_plan(outputs, get_dataset(opt.dataset).flip_idx, torch.device('cpu'))
  assert sorted(got) == sorted(want) and sorted(got) == sorted(h for h in opt.heads if h in (
      'hm', 'wh', 'dep', 'dim', 'amodel_offset', 'hps', 'hm_hp'))
  for h in got:
    for a, b in zip(got[h], want[h]):
      assert (a is None and b is None) or torch.equal(a, b), h
  if cfg == 'coco_pose':
    perm, sign = got['hps']
    assert perm[2:4].tolist() == [4, 5] and sign[:4].tolist() == [-1., 1., -1., 1.]
    assert got['hm_hp'][0][1:3].tolist() == [2, 1] and got['hm_hp'][1] is None
  if cfg == 'nuscenes_ddd':
    assert got['amodel_offset'][0] is None and got['amodel_offset'][1].tolist() == [-1., 1.]
