"""-m gpu: the halo kernel's pixel-major flavour (n_tile == C_out == 64: weights on wgmma M, the item's 128 pixels on N,
one warpgroup per item) on what the plan audits do not reach: CTAs with an odd number of work items (the warpgroups'
turn-taking ends on either one), a batch prefix of a launch built for more images, and channel slices of wider
buffers for the input, the residual and the output -- every walk it instantiates, against fp64 bounds."""
import ctypes as C

import pytest
import torch

import bounds as bd
from centertrack_b200 import _lib as L

pytestmark = pytest.mark.gpu

SENTINEL = -7.0          # exact in bf16: every channel outside the output slice must keep it

# (name, B, C_in, H, W, k, residual): one per compile-time walk (conv_halo.cu PX_WALKS).  At 3 x 120 x 124 a persistent
# grid of 132 CTAs gets 2 or 3 of the 384 tiles (8 x 16 tiles, ragged at the right and bottom edges).
CASES = [
    ('3x3 64->64 +res', 3, 64, 120, 124, 3, True),
    ('2x2 128->64', 3, 128, 120, 124, 2, False),
    ('1x1 32->64', 3, 32, 120, 124, 1, False),
    ('1x1 128->64 +res', 3, 128, 120, 124, 1, True),
    ('3x3 64->64 one tile per CTA', 1, 64, 40, 24, 3, True),
]


def _launch(case, seed, B=None, pad_in=16, off_in=8, pad_out=32, off_out=16, pad_res=24, off_res=8):
  """The case's launch reading channels [off_in, off_in + C_in) of a wider input, adding channels [off_res, +64) of a
  wider residual and writing channels [off_out, +64) of a wider output, on its first B images.
  -> (output buffer [B, H, W, 64 + pad_out], inputs (x, w, b, r) fp32 NCHW, ct_conv_config)."""
  from gpu_helpers import conv_desc
  name, B0, Cin, H, W, k, res = case
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(B0, Cin, H, W, generator=g)
  w = torch.randn(64, Cin, k, k, generator=g) * (2.0 / (Cin * k * k)) ** 0.5
  b = torch.randn(64, generator=g) * 0.1
  r = torch.randn(B0, 64, H, W, generator=g) if res else None
  d, _, keep = conv_desc(L.CT_ENGINE_TCGEN05_HALO, L.CT_BF16, x.cuda(), w, b, 1, True, None, n_tile=64,
                         ld_pad=pad_in, ch_off=off_in)
  if res:
    rb = torch.full((B0, H, W, 64 + pad_res), SENTINEL, dtype=torch.bfloat16, device='cuda')
    rb[..., off_res:off_res + 64] = r.permute(0, 2, 3, 1).to('cuda', torch.bfloat16)
    d.residual, d.ld_res = rb.data_ptr() + 2 * off_res, 64 + pad_res
    keep = keep + (rb,)
  out = torch.full((B0, H, W, 64 + pad_out), SENTINEL, dtype=torch.bfloat16, device='cuda')
  d.out, d.ld_out = out.data_ptr() + 2 * off_out, 64 + pad_out
  if B is not None:
    d.B = B
  cfg = L.conv_config(d)
  L.check(L.lib().ct_conv_forward(C.byref(d), L.stream_ptr()), 'conv')
  torch.cuda.synchronize()
  del keep
  return out, (x, w, b, r), cfg


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_pixel_major_slices_against_fp64(case):
  name, B, Cin, H, W, k, res = case
  out, (x, w, b, r), cfg = _launch(case, 900)
  assert cfg.pixel_major == 1 and cfg.tile_w == 8 and cfg.tile_h == 16, name
  o = out.float()
  assert (o[..., :16] == SENTINEL).all() and (o[..., 80:] == SENTINEL).all(), name + ': wrote outside its slice'
  q = lambda t: t.bfloat16().double().cuda() if t is not None else None
  p = (1, 0, 1, 0) if k == 2 else (k // 2,) * 4
  ref, mag = bd.conv_ref(q(x), q(w.float()), b, q(r), 1, p)
  bd.assert_bound(o[..., 16:80].permute(0, 3, 1, 2), ref, mag, bd.ALPHA_BF16, True, name, 'relu')


@pytest.mark.parametrize('case', CASES[:2], ids=[c[0] for c in CASES[:2]])
def test_pixel_major_batch_prefix_is_bit_identical(case):
  """The same buffers launched for their first image only: that image bit for bit, the others untouched."""
  full, _, _ = _launch(case, 901)
  one, _, cfg = _launch(case, 901, B=1)
  assert cfg.pixel_major == 1
  assert torch.equal(one[:1], full[:1]), case[0]
  assert (one[1:].float() == SENTINEL).all(), case[0]
