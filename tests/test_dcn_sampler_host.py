"""The DCNv2 sampler checks' own footing (host code, no GPU): the oracle's exact fp32 fma, the power and spread of the
offset / mask catalogue of tests/test_gpu_dcn_sampler.py, and ct_conv_config / ct_conv_forward's refusal of offset maps
the tensor-core samplers cannot read (16-byte vector loads of each pixel's offset / mask row)."""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest
import torch

import ct_oracle as co
import dcn_catalogue as dc
from centertrack_b200 import _lib as L


# ---- fma_f32 against exact rational arithmetic ------------------------------------------------------------------------
def _round_f32(q):
  """Fraction -> nearest fp32 (ties to even)."""
  r = np.float32(float(q))
  cands = [r, np.nextafter(r, np.float32(np.inf)), np.nextafter(r, np.float32(-np.inf))]
  best = min(abs(Fraction(float(c)) - q) for c in cands)
  near = [c for c in cands if abs(Fraction(float(c)) - q) == best]
  return float(min(near, key=lambda c: int(np.array(c).view(np.uint32)) & 1))


def _triples():
  f = lambda v: float(np.float32(v))
  out = []
  rng = np.random.default_rng(3)
  for _ in range(300):                                   # ordinary triples
    a, b, c = (f(rng.normal() * 2.0 ** rng.integers(-20, 20)) for _ in range(3))
    out.append((a, b, c))
  for _ in range(100):                                   # large exponent gaps: a b far below c and far above
    a, b = f(rng.normal() * 2.0 ** -40), f(rng.normal() * 2.0 ** -30)
    c = f(rng.normal())
    out += [(a, b, c), (f(rng.normal() * 2 ** 30), f(rng.normal() * 2 ** 20), f(rng.normal() * 2.0 ** -40))]
  for e in range(-10, 10):                               # a b + c a hair (2^-46 relative to half an ulp) off an fp32 tie
    for mant in (1.0, 1 + 2.0 ** -23, 1.5, 1.75 + 2.0 ** -23):
      c = f(mant * 2.0 ** e)
      h = 2.0 ** (e - 24)                                # half an ulp of c
      a, b = f(h * (1 + 2.0 ** -23)), f(1 - 2.0 ** -23)   # a b = h (1 - 2^-46)
      out += [(a, b, c), (-a, b, c), (a, b, -c), (-a, b, -c)]
  return out


def test_fma_f32_is_the_correctly_rounded_fp32_fma():
  t = np.array(_triples(), np.float64)
  got = co.fma_f32(torch.from_numpy(t[:, 0]), torch.from_numpy(t[:, 1]), torch.from_numpy(t[:, 2])).numpy()
  ref = np.array([_round_f32(Fraction(a) * Fraction(b) + Fraction(c)) for a, b, c in t])
  assert np.array_equal(got, ref), t[got != ref][:5]
  naive = (t[:, 0] * t[:, 1] + t[:, 2]).astype(np.float32).astype(np.float64)   # fp64 sum, then fp32: double rounding
  assert int((naive != ref).sum()) >= 40            # the tie triples need the TwoSum correction


# ---- the catalogue's power: wrong samplers must differ from the oracle on it ------------------------------------------
def _to_bf16(t, mode):
  """fp32 -> bf16 value (as fp32) by round-to-nearest-even, toward zero or half away from zero."""
  if mode == 'rn':
    return t.to(torch.bfloat16).float()
  u = t.contiguous().view(torch.int32)
  if mode == 'away':
    u = u + 0x8000
  return (u & -65536).view(torch.float32)


def _bf16_columns(x, off, mask, mut=None):
  """The bf16 chain of dcn_sample_columns(bf16_blend=True), restated with one deliberate mistake `mut`:
  'rz' / 'away' weight conversion, 'swap_corners' (01 and 10 read each other's pixel), 'mask_after' (the mask scales
  the blended value instead of the weights), 'swap_dydx', 'ge' (py >= -1 and px >= -1 count as inside)."""
  B, Cn, H, W = x.shape
  xf = x.reshape(B, Cn, H * W)
  ys = torch.arange(H, dtype=torch.float32).view(1, H, 1)
  xs = torch.arange(W, dtype=torch.float32).view(1, 1, W)
  qw = lambda t: _to_bf16(t, mut if mut in ('rz', 'away') else 'rn').double()
  cols = torch.zeros(B, Cn, 9, H, W, dtype=torch.float64)
  for k in range(9):
    dy, dx = off[:, 2 * k], off[:, 2 * k + 1]
    if mut == 'swap_dydx':
      dy, dx = dx, dy
    py, px = ys - 1 + k // 3 + dy, xs - 1 + k % 3 + dx
    lo_y, lo_x = (py >= -1, px >= -1) if mut == 'ge' else (py > -1, px > -1)
    valid = lo_y & (py < H) & lo_x & (px < W)
    y0, x0 = torch.floor(py), torch.floor(px)
    ly, lx = py - y0, px - x0
    hy, hx = 1 - ly, 1 - lx
    corners = [(y0, x0, hy * hx), (y0, x0 + 1, hy * lx), (y0 + 1, x0, ly * hx), (y0 + 1, x0 + 1, ly * lx)]
    acc = torch.zeros(B, Cn, H, W, dtype=torch.float64)
    for n, (yy, xx, wgt) in enumerate(corners):
      inb = (yy >= 0) & (yy <= H - 1) & (xx >= 0) & (xx <= W - 1) & valid
      if mut == 'swap_corners' and n in (1, 2):
        yy, xx = corners[3 - n][:2]
      idx = (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).long()
      g = torch.gather(xf, 2, idx.view(B, 1, H * W).expand(B, Cn, H * W)).view(B, Cn, H, W)
      m = 1.0 if mut == 'mask_after' else mask[:, k]
      acc = co.round_bf16(acc + g * qw(wgt * m * inb.float()).unsqueeze(1))
    if mut == 'mask_after':
      acc = co.round_bf16(acc * qw(mask[:, k]).unsqueeze(1))
    cols[:, :, k] = acc
  return cols


MUTANTS = ['rz', 'away', 'swap_corners', 'mask_after', 'swap_dydx', 'ge']
POWER_SHAPES = [(2, 7, 5), (3, 9, 17), (2, 33, 61), (1, 64, 96)]


def _catalogue_inputs(B, H, W, seed):
  om, cat = dc.catalogue(B, H, W, 2, seed)
  g = torch.Generator().manual_seed(seed)
  x = ((torch.randint(0, 2, (B, 4, H, W), generator=g) * 2 - 1) *
       torch.exp2(torch.rand(B, 4, H, W, generator=g) * 6 - 3)).bfloat16().double()
  o = torch.from_numpy(om).permute(0, 3, 1, 2).contiguous()
  return x, o[:, :18].contiguous(), o[:, 18:27].contiguous(), cat


def test_catalogue_catches_wrong_samplers():
  diff = {m: np.zeros(len(dc.CATEGORIES), np.int64) for m in MUTANTS}
  total = np.zeros(len(dc.CATEGORIES), np.int64)
  for B, H, W in POWER_SHAPES:
    x, off, mask, cat = _catalogue_inputs(B, H, W, H * W)
    errs = []
    ref = co.dcn_sample_columns(x, off, mask, bf16_blend=True, errors=errs)
    assert all(int((e != 0).sum()) == 0 for e in errs)
    assert torch.equal(_bf16_columns(x, off, mask), ref)              # the restatement is the oracle
    total += np.bincount(cat.ravel(), minlength=len(dc.CATEGORIES))
    for m in MUTANTS:
      d = (_bf16_columns(x, off, mask, m) != ref).any(1).permute(0, 2, 3, 1).numpy()   # [B, H, W, 9] per entry
      diff[m] += np.bincount(cat[d], minlength=len(dc.CATEGORIES))
  print('\nentries per category: ' + ', '.join('%s %d' % kv for kv in zip(dc.CATEGORIES, total)))
  for m in MUTANTS:
    print('%-12s differs on: %s' % (m, ', '.join('%s %d' % kv for kv in zip(dc.CATEGORIES, diff[m]) if kv[1])))
  at = lambda m, name: int(diff[m][dc.CATEGORIES.index(name)])
  # every deliberate mistake but 'ge' is seen on many entries, and in the categories built for it
  for m in ('rz', 'swap_corners', 'mask_after', 'swap_dydx'):
    assert diff[m].sum() >= 1000, (m, diff[m])
  for name in ('y_low', 'x_low', 'y_high', 'x_high', 'frac', 'win_y', 'win_x', 'normal'):
    assert at('swap_dydx', name) >= 50 and at('swap_corners', name) >= 50, name
  # the mask moves only where two corners blend (one-corner samples and masks exact in bf16 round alike)
  for name in ('y_low', 'x_low', 'y_high', 'x_high', 'frac', 'win_y', 'win_x', 'normal'):
    assert at('mask_after', name) >= 50, name
  assert at('rz', 'tie') >= 100 and at('rz', 'normal') >= 100
  # round-half-away differs from round-half-even only on ties: the tie entries catch it, N(0, 3) offsets never do
  assert at('away', 'tie') >= 100 and at('away', 'normal') == 0, diff['away']
  # py = -1 (or px = -1) samples nothing either way: row -1 lies outside and row 0 has weight ly = 0, so the strict
  # bound is not observable in values -- the mutant must agree everywhere
  assert diff['ge'].sum() == 0, diff['ge']


def test_catalogue_spread():
  """Over the shapes of the GPU probe, every category meets corners, edges, the interior, ragged patches and every tap."""
  seen = set()
  for B, H, W in dc.PROBE_SHAPES:
    cat = dc.categories(B, H, W)
    reg, ragged = dc.regions(B, H, W)
    tap = np.broadcast_to(np.arange(9), cat.shape)
    seen |= {('region', int(c), int(r)) for c, r in zip(cat.ravel(), reg.ravel())}
    seen |= {('tap', int(c), int(t)) for c, t in zip(cat.ravel(), tap.ravel())}
    seen |= {('ragged', int(c), 1) for c in cat[ragged]}
  for c in range(len(dc.CATEGORIES)):
    for r in range(3):
      assert ('region', c, r) in seen, (dc.CATEGORIES[c], ('interior', 'edge', 'corner')[r])
    for t in range(9):
      assert ('tap', c, t) in seen, (dc.CATEGORIES[c], t)
    assert ('ragged', c, 1) in seen, dc.CATEGORIES[c]


def test_catalogue_reaches_both_sides_of_the_window():
  for margin in (0, 2, 6):
    om, _ = dc.catalogue(2, 33, 61, margin, 1)
    split = np.bincount(dc.window_split(om, margin).ravel(), minlength=3)
    assert split.min() >= 1000, (margin, split)


# ---- refusals of offset maps the tensor-core samplers cannot read ------------------------------------------------------
DCN_PATHS = [('gather', L.CT_ENGINE_TCGEN05, L.CT_BF16, L.CT_A_DCN, 64),
             ('window', L.CT_ENGINE_TCGEN05, L.CT_BF16, L.CT_A_DCN_WIN, 64),
             ('x3', L.CT_ENGINE_TCGEN05_X3, L.CT_F32, L.CT_A_DCN, 64),
             ('simt', L.CT_ENGINE_SIMT, L.CT_F32, L.CT_A_DCN, 0)]


def _dcn_desc(engine, dtype, a_mode, n_tile, ld_om):
  d = L.ConvDesc()
  d.engine, d.dtype, d.a_mode = engine, dtype, a_mode
  d.B, d.H, d.W, d.C_in, d.ld_in, d.C_out = 1, 16, 24, 64, 64, 64
  d.KH = d.KW = 3
  d.stride, d.pad, d.OH, d.OW = 1, 1, 16, 24
  d.out_mode, d.ld_out, d.n_tile, d.ld_om = L.CT_OUT_NHWC, 64, n_tile, ld_om
  return d


def _config(d):
  lib = L.lib()
  c = L.ConvConfig()
  return lib.ct_conv_config(C.byref(d), C.byref(c)), lib.ct_last_error()


@pytest.mark.parametrize('path', DCN_PATHS, ids=[p[0] for p in DCN_PATHS])
def test_ld_om_the_sampler_can_read(built_lib, path):
  _, engine, dtype, a_mode, n_tile = path
  for ld_om in (27, 28, 29, 30, 31, 32, 36):
    rc, msg = _config(_dcn_desc(engine, dtype, a_mode, n_tile, ld_om))
    if engine == L.CT_ENGINE_SIMT or ld_om % 4 == 0:        # SIMT reads om element by element
      assert rc == L.CT_OK, (ld_om, msg)
    else:
      assert rc == L.CT_ERR_INVALID and b'ld_om % 4 == 0' in msg, (ld_om, msg)
  rc, msg = _config(_dcn_desc(engine, dtype, a_mode, n_tile, 26))
  assert rc == L.CT_ERR_INVALID and b'ld_om >= 27' in msg, msg


# ct_conv_forward on stand-in pointers for descriptors ct_conv_config ACCEPTS: only the om pointer check stands between
# the call and a launch, so the calls run in a child process that sees no CUDA device.  Without the check (an older
# build, or the check moved after the tensor-map encode) the child's launch fails cleanly with no device instead of
# reading addresses that do not exist.
_REFUSALS = r"""
import ctypes as C, json, sys
from centertrack_b200 import _lib as L
engine, dtype, a_mode, n_tile, skew = map(int, sys.argv[1:6])
lib = L.lib()
res = []
for ld_om in (28, 32, 30):
  d = L.ConvDesc()
  d.engine, d.dtype, d.a_mode = engine, dtype, a_mode
  d.B, d.H, d.W, d.C_in, d.ld_in, d.C_out = 1, 16, 24, 64, 64, 64
  d.KH = d.KW = 3
  d.stride, d.pad, d.OH, d.OW = 1, 1, 16, 24
  d.out_mode, d.ld_out, d.n_tile, d.ld_om = L.CT_OUT_NHWC, 64, n_tile, ld_om
  d.x = d.w = d.out = 1 << 20
  d.om = (1 << 21) + skew
  rc = lib.ct_conv_forward(C.byref(d), None)
  res.append((ld_om, rc, lib.ct_last_error().decode()))
print(json.dumps(res))
"""


@pytest.mark.parametrize('path', DCN_PATHS[:3], ids=[p[0] for p in DCN_PATHS[:3]])
@pytest.mark.parametrize('skew', [4, 8])
def test_misaligned_om_is_refused_before_any_cuda_call(built_lib, path, skew):
  """The refusal comes from the pointer check, which runs before the tensor-map encode and launch: the call returns
  CT_ERR_INVALID with its message, not a CUDA error (the child process has no device to report one from)."""
  import json
  import os
  import subprocess
  import sys
  _, engine, dtype, a_mode, n_tile = path
  for ld_om in (28, 32):                                # accepted by the configuration step: only the pointer is wrong
    assert _config(_dcn_desc(engine, dtype, a_mode, n_tile, ld_om))[0] == L.CT_OK
  repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
  r = subprocess.run([sys.executable, '-c', _REFUSALS] + [str(v) for v in (engine, dtype, a_mode, n_tile, skew)],
                     cwd=repo, env=env, capture_output=True, text=True, timeout=300)
  assert r.returncode == 0, r.stderr[-2000:]
  res = json.loads(r.stdout.strip().splitlines()[-1])
  for ld_om, rc, msg in res:
    assert rc == L.CT_ERR_INVALID, (ld_om, rc, msg)
    # ld_om 30: the configuration step refuses first, with its own message
    assert ('ld_om % 4 == 0' if ld_om == 30 else '16-byte aligned om') in msg, (ld_om, msg)
