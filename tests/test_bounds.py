"""The per-element error bound of tests/bounds.py on the CPU: it accepts exactly what a correct kernel produces and
rejects wrong rounding and a single missing product."""
import pytest
import torch

import bounds as bd
import ct_oracle as co


def _case(seed=0):
  g = torch.Generator().manual_seed(seed)
  x = bd.round_bf16(torch.randn(2, 64, 10, 12, generator=g, dtype=torch.float64))
  w = bd.round_bf16(torch.randn(32, 64, 3, 3, generator=g, dtype=torch.float64) * (2.0 / 576) ** 0.5)
  sh = torch.randn(32, generator=g, dtype=torch.float64).float() * 0.1
  ref, mag = bd.conv_ref(x, w, sh, pad=(1, 1, 1, 1))
  return x, w, ref, mag


def test_round_bf16_single_rounding():
  t = torch.tensor([1 + 2 ** -8 + 2 ** -30, 1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8 + 2 ** -30), 0.0, 3.0],
                   dtype=torch.float64)
  want = torch.tensor([1 + 2 ** -7, 1.0, 1 + 2 ** -6, -(1 + 2 ** -7), 0.0, 3.0], dtype=torch.float64)
  assert torch.equal(bd.round_bf16(t), want)
  r = torch.randn(10000, dtype=torch.float32)
  assert torch.equal(bd.round_bf16(r.double()), r.bfloat16().double())      # fp32 -> bf16 is a single rounding
  assert torch.equal(bd.ulp_bf16(torch.tensor([1.0, 1.5, 2.0, 0.75], dtype=torch.float64)),
                     torch.tensor([2 ** -7, 2 ** -7, 2 ** -6, 2 ** -8], dtype=torch.float64))


@pytest.mark.parametrize('act', ['none', 'relu'])
def test_round_to_nearest_passes_truncation_fails(act):
  _, _, ref, mag = _case()
  if act == 'relu':
    ref_out = ref.clamp_min(0)
  else:
    ref_out = ref
  got = bd.round_bf16(ref_out)
  assert bd.ratio(got, ref, mag, bd.ALPHA_BF16, True, act).max() <= 1.0
  u = bd.ulp_bf16(ref_out.abs())
  tz = torch.sign(ref_out) * torch.floor(ref_out.abs() / u) * u      # bf16 rounding toward zero
  r = bd.ratio(tz, ref, mag, bd.ALPHA_BF16, True, act)
  assert r.max() > 1.0
  assert (r > 1.0).double().mean() > 0.05      # about a third of the elements are more than half an ulp off


@pytest.mark.parametrize('bf16_out', [True, False])
def test_one_missing_product_fails(bf16_out):
  x, w, ref, mag = _case(1)
  b, o, y, xx = 1, 17, 4, 0                       # a border pixel: the left column of taps reads padding
  xp = torch.nn.functional.pad(x, (1, 1, 1, 1))
  prods = xp[b, :, y:y + 3, xx:xx + 3] * w[o]
  c, ky, kx = [int(i) for i in torch.nonzero(prods.abs() == prods.abs().max())[0]]
  assert kx > 0 and prods[c, ky, kx] != 0
  wrong = ref.clone()
  wrong[b, o, y, xx] -= prods[c, ky, kx]
  got = bd.round_bf16(wrong) if bf16_out else wrong
  coef = bd.ALPHA_BF16 if bf16_out else bd.BETA_X3
  r = bd.ratio(got, ref, mag, coef, bf16_out)
  assert r[b, o, y, xx] > 1.0
  r[b, o, y, xx] = 0
  assert r.max() <= 1.0                           # every other element still passes
  with pytest.raises(AssertionError, match="'c': 17"):
    bd.assert_bound(got, ref, mag, coef, bf16_out, 'one product dropped')


def test_fp32_bounds_accept_accumulation_noise():
  _, _, ref, mag = _case(2)
  g = torch.Generator().manual_seed(5)
  for coef in (bd.BETA_X3, bd.GAMMA_SIMT, bd.ALPHA_BF16):
    noisy = ref + (torch.rand(ref.shape, generator=g, dtype=torch.float64) * 2 - 1) * 0.9 * coef * mag
    assert bd.ratio(noisy, ref, mag, coef, False).max() <= 1.0
    assert bd.ratio(ref + 1.1 * coef * mag, ref, mag, coef, False).min() > 1.0


def test_monotone_epilogue_intervals():
  ref = torch.linspace(-30, 30, 601, dtype=torch.float64)
  mag = ref.abs() + 1.0
  e = bd.ALPHA_BF16 * mag
  for act in ('sigmoid', 'depth'):
    f = torch.sigmoid(ref) if act == 'sigmoid' else 1.0 / (torch.sigmoid(ref) + 1e-6) - 1.0
    assert bd.ratio(f.float(), ref, mag, bd.ALPHA_BF16, False, act).max() <= 1.0
    lo, hi = bd.interval(ref, e, act)
    assert (lo <= f).all() and (f <= hi).all()
    shifted = torch.sigmoid(ref + 0.01) if act == 'sigmoid' else 1.0 / (torch.sigmoid(ref + 0.01) + 1e-6) - 1.0
    assert bd.ratio(shifted, ref, mag, bd.ALPHA_BF16, False, act).max() > 1.0


def test_exact_bf16_dcn_blend_rounds_once():
  """fp64 columns with bf16_blend: every fma step rounds the exact sum once (the kernels' fma.rn.bf16x2); the
  fp32 emulation rounds fp32(acc + g w) to bf16 and can differ by one bf16 ulp."""
  g = torch.Generator().manual_seed(3)
  B, C, H, W = 1, 8, 6, 7
  x = torch.randn(B, C, H, W, generator=g).bfloat16().float()
  off = torch.randn(B, 18, H, W, generator=g) * 2
  mask = torch.rand(B, 9, H, W, generator=g)
  cols = co.dcn_sample_columns(x.double(), off, mask, bf16_blend=True)
  assert cols.dtype == torch.float64
  assert torch.equal(bd.round_bf16(cols), cols)           # every column is a bf16 value
  # direct per-element emulation of channel c: weights as the kernels compute them (fp32, then bf16)
  b, c = 0, 5
  for k in range(9):
    for y in range(H):
      for xx in range(W):
        py = torch.tensor(y - 1 + k // 3, dtype=torch.float32) + off[b, 2 * k, y, xx]
        px = torch.tensor(xx - 1 + k % 3, dtype=torch.float32) + off[b, 2 * k + 1, y, xx]
        y0, x0 = torch.floor(py), torch.floor(px)
        ly, lx = py - y0, px - x0
        hy, hx = 1 - ly, 1 - lx
        acc = 0.0
        if -1 < float(py) < H and -1 < float(px) < W:
          for yy, xc, wgt in ((y0, x0, hy * hx), (y0, x0 + 1, hy * lx), (y0 + 1, x0, ly * hx), (y0 + 1, x0 + 1, ly * lx)):
            yi, xi = int(yy), int(xc)
            if 0 <= yi < H and 0 <= xi < W:
              wq = float((wgt * mask[b, k, y, xx]).bfloat16())
              acc = float(bd.round_bf16(torch.tensor(acc + float(x[b, c, yi, xi]) * wq, dtype=torch.float64)))
        assert float(cols[b, c, k, y, xx]) == acc, (k, y, xx)
  # the fp32-input path is unchanged (fp32 columns, as the goldens were made)
  assert co.dcn_sample_columns(x, off, mask, bf16_blend=True).dtype == torch.float32
