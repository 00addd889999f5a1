"""Per-element error bounds for the convolution engines, against an fp64 reference computed from the exact operands a
kernel read (test infrastructure; importable without a GPU).

For an output element with exact value `ref` (fp64 sum over the operands the kernel saw) and
`mag` = conv(|x|, |w|) + |shift| + |residual| (the sum of the magnitudes of every term):

  bf16 output   |got - ref| <= alpha mag + 1/2 ulp_bf16(|ref| + alpha mag)
                got is the round-to-nearest of something within alpha mag of ref.  alpha covers the fp32 accumulation of
                the wgmma engines.  One dropped product is ~ mag / K >= 2e-4 mag (K <= 4608 in DLA-34), far above alpha,
                so a missing tap, channel group or K block fails on the element where it happens.
  fp32 output   |got - ref| <= c mag, c = ALPHA_BF16 (bf16 engines: operands exact, accumulation only), BETA_X3 or
                GAMMA_SIMT.
  monotone epilogues (ReLU, sigmoid, the depth transform) map the interval [ref - e, ref + e] through the activation,
  widened by the error of the fast sigmoid / division of the tensor-core epilogues.

The ratio |got - centre| / half-width of the allowed interval is reported; <= 1 passes.
"""
import torch

from ct_oracle import round_bf16  # noqa: F401  (fp64 -> bf16 with one rounding)

# Accumulation coefficients, calibrated on an H100 80GB HBM3 (400 W power limit) from the plan audit
# (tests/test_gpu_plan_layers.py: every launch of nine product plans, B up to 32), as the largest observed
# (|got - ref| - rounding of the output) / mag; the constant sits 2-4x above it.
# wgmma fp32 accumulation (bf16 engines, gather and halo): observed 5.1e-7 (gather, fp32-output offset conv of
# dla_up.ida_0.proj_1, nuscenes_ddd 448x800), 2.7e-7 (halo): 2^-19 = 1.9e-6 is 3.8x above.  A dropped product
# (>= 2e-4 mag) is 100x above it.
ALPHA_BF16 = 2.0 ** -19
# bf16x3: a = hi + lo + ea with |a - hi| <= 2^-9 |a| and |ea| <= 2^-9 |a - hi| <= 2^-18 |a| (lo is rounded too); the
# engine computes hi_a hi_b + hi_a lo_b + lo_a hi_b, so per product the missing part is lo_a lo_b + ea b + a eb
# <= 3 * 2^-18 |ab| (+ higher order) = 1.1e-5 |ab|, plus the fp32 accumulation of three MMAs per product (~ALPHA_BF16).
# Observed 7.3e-6 (the 7x7 stem, B = 32): 2^-16 = 1.5e-5 is 2.1x above and just above the derived worst case.
BETA_X3 = 2.0 ** -16
# SIMT fp32: one fp32 fma per product, sequential over K per output (and the fp32 fma chain of the up-sampling):
# observed 4.1e-7 (dla_up.ida_2.proj_2, 512x512): 2^-20 = 9.5e-7 is 2.3x above.
GAMMA_SIMT = 2.0 ** -20
# sigmoidf_fast = __fdividef(1, 1 + __expf(-x)) (ex2.approx / rcp.approx, a few ulp) and the depth transform's
# __fdividef: absolute + relative slack on the activation's value.
ACT_ABS = 2.0 ** -21
ACT_REL = 2.0 ** -18


def ulp_bf16(a):
  """Spacing of bf16 values at magnitude a >= 0 (fp64): 2^(exponent - 7) for a in [2^exponent, 2^(exponent+1))."""
  _, e = torch.frexp(a.clamp_min(2.0 ** -126))
  return torch.ldexp(torch.ones_like(a), e - 8)


def conv_ref(x, w, shift=None, residual=None, stride=1, pad=(0, 0, 0, 0)):
  """fp64 NCHW conv + shift + residual and its magnitude.  x [B,C,H,W], w [O,C,kh,kw] (the values the kernel read);
  pad = (left, right, top, bottom) zero padding.  Returns (ref, mag) fp64 on x's device."""
  x = x.double()
  w = w.double().to(x.device)
  xp = torch.nn.functional.pad(x, pad)
  ref = torch.nn.functional.conv2d(xp, w, None, stride)
  mag = torch.nn.functional.conv2d(xp.abs(), w.abs(), None, stride)
  if shift is not None:
    s = shift.double().to(x.device).view(1, -1, 1, 1)
    ref = ref + s
    mag = mag + s.abs()
  if residual is not None:
    r = residual.double()
    ref = ref + r
    mag = mag + r.abs()
  return ref, mag


def _sigmoid(t):
  return torch.sigmoid(t)


def interval(ref, e, act='none', depth_scale=1.0, relu=False):
  """[lo, hi] of act(v) over |v - ref| <= e (act monotone, after an optional ReLU), widened by the fast-math slack of
  the fused sigmoid / depth epilogues.  act: 'none' | 'relu' | 'sigmoid' | 'depth'."""
  a, b = ref - e, ref + e
  if relu or act == 'relu':
    a, b = a.clamp_min(0), b.clamp_min(0)
  if act in ('none', 'relu'):
    return a, b
  if act == 'sigmoid':
    lo, hi = _sigmoid(a), _sigmoid(b)
    return lo - ACT_ABS - ACT_REL * lo, hi + ACT_ABS + ACT_REL * hi
  if act == 'depth':               # decreasing in v; the sigmoid's slack goes through 1 / s
    s_lo = (_sigmoid(a) - ACT_ABS - ACT_REL * _sigmoid(a)).clamp_min(0)
    s_hi = _sigmoid(b) + ACT_ABS + ACT_REL * _sigmoid(b)
    lo, hi = (1.0 / (s_hi + 1e-6) - 1.0) * depth_scale, (1.0 / (s_lo + 1e-6) - 1.0) * depth_scale
    return lo - ACT_REL * (lo.abs() + abs(depth_scale)), hi + ACT_REL * (hi.abs() + abs(depth_scale))
  raise ValueError(act)


def stem_interval(ref, mag, coef, mask):
  """The stem epilogue sum_g relu(group g) over the present groups (bit g of mask) of a 48-channel result
  [B, 48, H, W] -> (lo, hi) of the 16-channel sum."""
  lo = hi = 0
  for g in range(3):
    if (mask >> g) & 1:
      a, b = interval(ref[:, 16 * g:16 * g + 16], coef * mag[:, 16 * g:16 * g + 16], relu=True)
      lo, hi = lo + a, hi + b
  return lo, hi


def ratio(got, ref, mag, coef, bf16_out, act='none', depth_scale=1.0):
  """Per-element |got - centre| / half-width of the allowed interval (<= 1 passes); fp64, same shape as ref."""
  lo, hi = interval(ref, coef * mag, act, depth_scale)
  return ratio_interval(got, lo, hi, bf16_out)


def ratio_interval(got, lo, hi, bf16_out):
  """Like ratio(), for an interval [lo, hi] the exact-arithmetic value may lie in."""
  got = got.to(lo.device).double()
  if bf16_out:                     # the stored value is the round-to-nearest of a value in [lo, hi]
    half = 0.5 * ulp_bf16(torch.maximum(lo.abs(), hi.abs()))
    lo, hi = lo - half, hi + half
  mid, rad = 0.5 * (lo + hi), 0.5 * (hi - lo)
  d = (got - mid).abs()
  r = torch.where(rad > 0, d / torch.where(rad > 0, rad, torch.ones_like(rad)), torch.where(d > 0, float('inf'), 0.0))
  r = torch.where((got >= lo) & (got <= hi), r.clamp_max(1.0), r)     # an endpoint is inside, whatever mid rounds to
  return torch.where(torch.isnan(got), torch.full_like(r, float('inf')), r)


def accum_use(got, ref, mag, bf16_out):
  """Smallest accumulation coefficient c that would explain each element (what the constants are calibrated from):
  (|got - ref| - 1/2 ulp(|ref|)) / mag for bf16 outputs, |got - ref| / mag for fp32 outputs; 0 where mag == 0."""
  err = (got.to(ref.device).double() - ref).abs()
  if bf16_out:
    err = (err - 0.5 * ulp_bf16(ref.abs())).clamp_min(0)
  return torch.where(mag > 0, err / torch.where(mag > 0, mag, torch.ones_like(mag)), torch.zeros_like(mag))


def worst(r, names='bchw'):
  """(max ratio, index tuple of the worst element as a dict)."""
  flat = torch.nan_to_num(r, nan=float('inf')).reshape(-1)
  i = int(torch.argmax(flat))
  idx = []
  for s in reversed(r.shape):
    idx.append(i % s)
    i //= s
  return float(flat.max()), dict(zip(names, reversed(idx)))


def assert_bound(got, ref, mag, coef, bf16_out, what='', act='none', depth_scale=1.0):
  """Assert every element within its bound; returns the worst ratio (for calibration reports)."""
  r = ratio(got, ref, mag, coef, bf16_out, act, depth_scale)
  m, at = worst(r)
  if not m <= 1.0:
    key = tuple(at.values())
    raise AssertionError('%s: worst element %s |got - bound centre| / bound = %.3g (got %.8g, ref %.8g, mag %.4g)' % (
        what, at, m, float(got.reshape(r.shape)[key]), float(ref[key]), float(mag[key])))
  return m
