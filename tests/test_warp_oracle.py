"""The pre_process warp oracle (ct_oracle.warp_affine_u8) against cv2.warpAffine byte for byte: every resolution policy
over camera frame sizes, and inverse maps given with WARP_INVERSE_MAP -- the fused-multiply-add tie maps, rotation,
shear, translations, maps outside the frame, a frame with a padded row pitch.  The device tests hold ct_warp_*,
ct_pack_stem_frames* to this oracle; this file holds the oracle to cv2."""
import cv2
import numpy as np
import pytest

import ct_oracle as co
from helpers import WARP_GEOMETRIES, warp_geometry, warp_maps

MAPS = warp_maps()


def _image(h, w, seed):
  return np.random.RandomState(seed).randint(0, 256, size=(h, w, 3)).astype(np.uint8)


def _same(got, want, name):
  diff = got != want
  assert not diff.any(), (name, int(diff.sum()), np.argwhere(diff)[:5].tolist())


@pytest.mark.parametrize('i', range(len(WARP_GEOMETRIES)), ids=[g[0] for g in WARP_GEOMETRIES])
def test_oracle_warp_equals_cv2_on_every_resolution_policy(i):
  """cv2.warpAffine(img, trans_input, INTER_LINEAR) -- Detector.pre_process's call -- and the oracle given
  frame_geometry's inverted map."""
  (h, w), (oh, ow), minv, fwd = warp_geometry(i)
  img = _image(h, w, i)
  want = cv2.warpAffine(img, fwd, (ow, oh), flags=cv2.INTER_LINEAR)
  _same(co.warp_affine_u8(img, minv, oh, ow), want, WARP_GEOMETRIES[i][0])


@pytest.mark.parametrize('i', range(len(MAPS)), ids=[m[0] for m in MAPS])
def test_oracle_warp_equals_cv2_on_inverse_maps(i):
  name, minv, (h, w), (oh, ow) = MAPS[i]
  img = _image(h, w, 100 + i)
  want = cv2.warpAffine(img, minv.reshape(2, 3), (ow, oh), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP)
  _same(co.warp_affine_u8(img, minv, oh, ow), want, name)
  if name == 'wholly_outside':
    assert not want.any()


def test_tie_maps_move_a_whole_row_when_the_row_term_is_fused():
  """The tie maps do what they are for: the oracle with the row term computed as one fused multiply-add (exact, then
  one rounding) differs from cv2 on the tie row and nowhere else."""
  from fractions import Fraction
  ties = [m for m in MAPS if m[0].startswith('tie_')]
  assert len(ties) == 6
  for name, minv, (h, w), (oh, ow) in ties:
    y0 = int(name.split('row')[1])
    img = _image(h, w, 7)
    want = cv2.warpAffine(img, minv.reshape(2, 3), (ow, oh), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP)
    fused = minv.copy()        # the fused row term at y0, restated as M[2] (or M[5]) of a map with no y slope
    s, o = (1, 2) if name.startswith('tie_x') else (4, 5)
    fused[o], fused[s] = float(Fraction(minv[s]) * y0 + Fraction(minv[o])), 0.
    row = co.warp_affine_u8(img, fused, oh, ow)[y0]
    assert (row != want[y0]).any(), name
    assert np.array_equal(co.warp_affine_u8(img, minv, oh, ow)[y0], want[y0]), name


def test_oracle_warp_reads_a_frame_with_a_padded_row_pitch():
  """A frame given as a view into wider rows (the pitch of a ct_frame) warps as the contiguous frame does."""
  wide = _image(375, 1250, 5)
  img = wide[:, 3:1245]
  assert not img.flags['C_CONTIGUOUS']
  for name, minv, _, (oh, ow) in MAPS[6:9]:
    want = cv2.warpAffine(np.ascontiguousarray(img), minv.reshape(2, 3), (ow, oh),
                          flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP)
    _same(co.warp_affine_u8(img, minv, oh, ow), want, name)
    _same(cv2.warpAffine(img, minv.reshape(2, 3), (ow, oh), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP), want, name)


def test_normalize_and_stem_pixels():
  """normalize_chw is pre_process's fp64 expression rounded once; stem_pixels rounds each channel to bf16 ties to even
  (torch's fp32 -> bf16) and mirrors all eight channels under flip."""
  import torch
  img = _image(6, 9, 3)
  mean, std = np.float32([0.408, 0.447, 0.47]), np.float32([0.289, 0.274, 0.278])
  chw = co.normalize_chw(img, mean, std)
  want = ((img / 255. - mean.reshape(1, 1, 3)) / std.reshape(1, 1, 3)).astype(np.float32).transpose(2, 0, 1)
  assert chw.dtype == np.float32 and np.array_equal(chw.view(np.int32), want.view(np.int32))
  prev = co.normalize_chw(_image(6, 9, 4), mean, std)
  hm = np.random.RandomState(0).rand(6, 9).astype(np.float32)
  bits = co.stem_pixels(chw, prev, hm, flip=True)
  v = torch.from_numpy(np.concatenate([chw, prev, hm[None], np.zeros((1, 6, 9), np.float32)]).transpose(1, 2, 0).copy())
  ref = v.to(torch.bfloat16).view(torch.int16).numpy()
  assert np.array_equal(bits[0], ref) and np.array_equal(bits[1], ref[:, ::-1])
  ties = np.float32([1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8)])        # exact bf16 ties: to even
  assert co.bf16_bits(ties).tolist() == torch.from_numpy(ties).to(torch.bfloat16).view(torch.int16).tolist()
  alone = co.stem_pixels(chw, None, None)
  assert not alone[..., 3:].any() and np.array_equal(alone[..., :3], ref[..., :3])
