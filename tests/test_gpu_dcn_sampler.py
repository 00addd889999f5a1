"""-m gpu: every DCNv2 sampler, sample by sample, against the oracle -- no tolerance.

Probe launches: one-hot weights (C_out = 9 C_in, W[tap C_in + c, c, tap] = 1, no shift, ReLU or residual) make output
channel tap C_in + c exactly sample (c, tap): it is the only non-zero product of its row, the fp32 accumulation adds
exact zeros (wgmma and SIMT alike) and a bf16 sample survives the bf16 store.  A swapped tap or channel, a dy / dx swap
or a wrong chunk-major K order of CT_A_DCN_WIN moves a sample to another channel.  Expected values, compared as values
(-0 == +0):

  gather bf16 (CT_A_DCN, CT_A_DCN_WIN)  the oracle's bf16 chain (dcn_sample_columns(bf16_blend=True)), bit for bit
  SIMT fp32                             the fp32 chain (dcn_sample_columns(fp32_chain=True))
  SIMT bf16                             bf16 round-to-nearest of the fp32 chain
  bf16x3                                hi + lo of the fp32 chain: hi = bf16(v), lo = bf16(v - hi) (split8)

(the SIMT gather accumulates `av += w v`, which nvcc contracts into FFMA; the first corner is an FFMA onto the zero
register, i.e. a plain multiply.)

Offsets and masks come from tests/dcn_catalogue.py.  Buffers are poisoned: x sits in a NaN-filled [B + 2, H, W,
C_in + 64] buffer (channels 32 .. 32 + C_in of images 1 .. B), om rows carry NaN from channel 27 on, and out is
NaN-filled with ld_out = C_out + 16 and a NaN guard after it.  A read outside the slice turns the pixel's whole output
row NaN (0 x NaN in the sampler or the MMA), and a store outside C_out or past the map shows in the padding or the
guard."""
import ctypes as C
import os
import subprocess
import sys
from collections import defaultdict

import numpy as np
import pytest
import torch

import bounds as bd
import ct_oracle as co
import dcn_catalogue as dc
from centertrack_b200 import _lib as L

pytestmark = pytest.mark.gpu

# (name, engine, dtype, a_mode)
PATHS = [('simt_f32', L.CT_ENGINE_SIMT, L.CT_F32, L.CT_A_DCN), ('simt_bf16', L.CT_ENGINE_SIMT, L.CT_BF16, L.CT_A_DCN),
         ('gather_bf16', L.CT_ENGINE_TCGEN05, L.CT_BF16, L.CT_A_DCN),
         ('window_bf16', L.CT_ENGINE_TCGEN05, L.CT_BF16, L.CT_A_DCN_WIN),
         ('x3', L.CT_ENGINE_TCGEN05_X3, L.CT_F32, L.CT_A_DCN)]
SHAPES = dc.PROBE_SHAPES
C_INS = {'simt_f32': [16, 32, 64, 128, 256, 512], 'simt_bf16': [16, 32, 64, 128, 256, 512],
         'gather_bf16': [16, 24, 32, 64, 128, 256, 512], 'window_bf16': [64, 128, 256, 512],
         'x3': [16, 24, 32, 64, 128, 256, 512]}


def _cases(path):
  """Every shape, each with a C_in of the engine (cycling), the largest maps at the smaller widths."""
  cins = C_INS[path]
  out = []
  for i, (B, H, W) in enumerate(SHAPES):
    cin = cins[i % len(cins)]
    if H * W >= 2000:
      cin = min(cin, 128)
    out.append((B, H, W, cin))
  out.append((2, 9, 17, cins[-1]))            # the widest C_in on a ragged map
  return out


CASES = [(p[0], c) for p in PATHS for c in _cases(p[0])]
MARGIN = int(os.environ.get('CTB_TC_DCN_MARGIN', '2'))     # what conv_tc reads (clamped to [0, 6])
MARGIN = max(0, min(6, MARGIN))
COUNTS = defaultdict(lambda: defaultdict(int))


def _path(name):
  return next(p for p in PATHS if p[0] == name)


def _nan_bits(t):
  return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _pack(engine, a_mode, w, n_tile):
  """ct_pack_weights as gpu_helpers.conv_desc packs them (chunk-major K order for CT_A_DCN_WIN)."""
  lib = L.lib()
  w32 = w.float().contiguous()
  O, Cin = w32.shape[:2]
  pc, pkh, pkw = Cin, 3, 3
  if a_mode == L.CT_A_DCN_WIN:
    nch = Cin // 64
    w32 = w32.reshape(O, nch, 64, 3, 3).permute(0, 2, 1, 3, 4).reshape(O, 64, nch * 3, 3).contiguous()
    pc, pkh, pkw = 64, nch * 3, 3
  wp = torch.empty(lib.ct_packed_weight_bytes(engine, O, pc, pkh, pkw, n_tile), dtype=torch.uint8)
  L.check(lib.ct_pack_weights(engine, C.c_void_p(w32.data_ptr()), O, pc, pkh, pkw, n_tile, C.c_void_p(wp.data_ptr())))
  return wp.cuda()


def _one_hot(Cin):
  """[9 C_in rounded up to 16 (the tensor-core engines' C_out granule), C_in, 3, 3]: the extra channels stay 0."""
  w = torch.zeros((9 * Cin + 15) // 16 * 16, Cin, 3, 3)
  c = torch.arange(Cin)
  for tap in range(9):
    w[tap * Cin + c, c, tap // 3, tap % 3] = 1.0
  return w


def _x_values(B, Cin, H, W, seed):
  """Sign x 2^U(-3, 3): magnitudes in [1/8, 8), so every fp64 step of the bf16 chain stays exact on the catalogue."""
  g = torch.Generator().manual_seed(seed)
  return (torch.randint(0, 2, (B, Cin, H, W), generator=g) * 2 - 1) * torch.exp2(torch.rand(B, Cin, H, W, generator=g) * 6 - 3)


def launch(path, B, H, W, Cin, w=None, n_tile=0, ld_om=None, tight=False, seed=0, margin=MARGIN):
  """One DCN launch of `path` on poisoned buffers over the catalogue.  -> dict of the sampled inputs (x fp64 NCHW,
  offsets, masks, om, categories), the output [B, H, W, C_out] and the checks of the buffers around it."""
  name, engine, dtype, a_mode = _path(path)
  act = torch.bfloat16 if dtype == L.CT_BF16 else torch.float32
  x = _x_values(B, Cin, H, W, seed).to(act)
  om_np, cat = dc.catalogue(B, H, W, margin, seed)
  w = _one_hot(Cin) if w is None else w
  Cout = w.shape[0]
  if n_tile == 0 and engine != L.CT_ENGINE_SIMT:
    n_tile = 64 if engine == L.CT_ENGINE_TCGEN05 else 128
  wp = _pack(engine, a_mode, w, n_tile)
  off = 0 if tight else 32
  ld_in = Cin if tight else Cin + 64
  xb = torch.full((B + 2, H, W, ld_in), float('nan'), dtype=act, device='cuda')
  xb[1:B + 1, :, :, off:off + Cin] = x.permute(0, 2, 3, 1).cuda()
  if ld_om is None:
    ld_om = 27 if engine == L.CT_ENGINE_SIMT else 28
  P = B * H * W
  omb = torch.full((P, ld_om), float('nan'), dtype=torch.float32, device='cuda')
  omb[:, :27] = torch.from_numpy(om_np).reshape(P, 27).cuda()
  ld_out, guard = Cout + 16, 4096
  outb = torch.full((P * ld_out + guard,), float('nan'), dtype=act, device='cuda')
  d = L.ConvDesc()
  d.engine, d.dtype, d.a_mode = engine, dtype, a_mode
  d.B, d.H, d.W, d.C_in, d.ld_in, d.C_out = B, H, W, Cin, ld_in, Cout
  d.KH = d.KW = 3
  d.stride, d.pad, d.OH, d.OW = 1, 1, H, W
  d.out_mode, d.relu, d.sig_from, d.depth_scale, d.n_tile = L.CT_OUT_NHWC, 0, 1 << 30, 1.0, n_tile
  d.x = xb.data_ptr() + (H * W * ld_in + off) * xb.element_size()
  d.w, d.shift, d.om, d.ld_om = wp.data_ptr(), None, omb.data_ptr(), ld_om
  d.out, d.ld_out = outb.data_ptr(), ld_out
  L.check(L.lib().ct_conv_forward(C.byref(d), L.stream_ptr()), '%s launch' % name)
  torch.cuda.synchronize()
  out = outb[:P * ld_out].view(P, ld_out)
  fill = _nan_bits(torch.full((1,), float('nan'), dtype=act, device='cuda'))
  assert torch.equal(_nan_bits(out[:, Cout:].contiguous()), fill.expand(P, 16)), '%s: a store landed in ld_out padding' % name
  assert torch.equal(_nan_bits(outb[P * ld_out:]), fill.expand(guard)), '%s: a store landed after the map' % name
  om_t = torch.from_numpy(om_np).permute(0, 3, 1, 2).contiguous().cuda()
  return dict(x=x.double().cuda(), off=om_t[:, :18].contiguous(), mask=om_t[:, 18:27].contiguous(), om=om_np, cat=cat,
              out=out[:, :Cout].reshape(B, H, W, Cout), C_in=Cin)


def expected(path, s):
  """[B, H, W, 9, C_in] fp64: what each path must produce for sample (c, tap) (module docstring)."""
  x, off, mask = s['x'], s['off'], s['mask']
  if path in ('gather_bf16', 'window_bf16'):
    errs = []
    cols = co.dcn_sample_columns(x, off, mask, bf16_blend=True, errors=errs)
    assert all(int((e != 0).sum()) == 0 for e in errs), 'an fp64 step of the bf16 chain is inexact on this catalogue'
  else:
    cols = co.dcn_sample_columns(x, off, mask, fp32_chain=True)
    if path == 'simt_bf16':
      cols = co.round_bf16(cols)
    elif path == 'x3':
      hi = co.round_bf16(cols)
      cols = hi + co.round_bf16(cols - hi)
  return cols.permute(0, 3, 4, 2, 1)            # [B, C, 9, H, W] -> [B, H, W, 9, C]


def check(path, s, label):
  B, H, W, Cout = s['out'].shape
  Cin = s['C_in']
  pad = s['out'][..., 9 * Cin:]
  assert bool((pad == 0).all()), '%s: an all-zero weight column produced a non-zero output' % label
  got = s['out'][..., :9 * Cin].double().reshape(B, H, W, 9, Cin)
  exp = expected(path, s)
  nan_rows = torch.isnan(got).reshape(B * H * W, -1).any(1)
  assert not bool(nan_rows.any()), '%s: %d output rows hold NaN (a read outside the slice), first pixel %d' % (
      label, int(nan_rows.sum()), int(nan_rows.nonzero()[0]))
  bad = got != exp
  if bool(bad.any()):
    b, y, x_, tap, c = [int(v) for v in bad.nonzero()[0]]
    cat = dc.CATEGORIES[s['cat'][b, y, x_, tap]]
    raise AssertionError('%s: %d of %d samples differ; first (b %d, y %d, x %d, tap %d, c %d, %s): got %r, expected %r, '
                         'om dy %r dx %r m %r' % (label, int(bad.sum()), bad.numel(), b, y, x_, tap, c, cat,
                                                  float(got[b, y, x_, tap, c]), float(exp[b, y, x_, tap, c]),
                                                  float(s['om'][b, y, x_, 2 * tap]), float(s['om'][b, y, x_, 2 * tap + 1]),
                                                  float(s['om'][b, y, x_, 18 + tap])))
  counts = np.bincount(s['cat'].ravel(), minlength=len(dc.CATEGORIES)) * Cin
  for i, n in enumerate(counts):
    COUNTS[path][dc.CATEGORIES[i]] += int(n)
  COUNTS[path]['(launches)'] += 1
  line = '[%s] %s: %d samples equal' % (path, label, got.numel())
  if path == 'window_bf16':
    split = np.bincount(dc.window_split(s['om'], MARGIN).ravel(), minlength=3) * Cin
    COUNTS[path]['(window)'] += int(split[1])
    COUNTS[path]['(global)'] += int(split[2])
    line += '; margin %d: window %d, global fall-back %d, outside %d' % (MARGIN, split[1], split[2], split[0])
  print(line)


@pytest.mark.parametrize('path,case', CASES, ids=['%s-%dx%dx%d-c%d' % ((p,) + c) for p, c in CASES])
def test_probe_samples_equal_oracle(path, case):
  B, H, W, Cin = case
  engine = _path(path)[1]
  ld_om = None if engine == L.CT_ENGINE_SIMT else (28 if (H * W) % 2 else 36)
  s = launch(path, B, H, W, Cin, ld_om=ld_om, seed=B * 1000 + H * W + Cin)
  check(path, s, '%dx%dx%d C_in %d ld_om %d' % (B, H, W, Cin, ld_om or 27))


@pytest.mark.parametrize('path', ['simt_bf16', 'gather_bf16', 'window_bf16', 'x3'])
def test_probe_tight_ld_in(path):
  """x with ld_in = C_in: the neighbouring images are NaN, nothing else is."""
  cin = 64
  s = launch(path, 2, 9, 17, cin, tight=True, seed=77)
  check(path, s, 'tight ld_in 2x9x17 C_in %d' % cin)


def _n_tiles(path, cin):
  """The N tiles ct_conv_config accepts for this DCN path at C_out = 9 C_in."""
  _, engine, dtype, a_mode = _path(path)
  ok = []
  for n in range(16, 257, 16):
    d = L.ConvDesc()
    d.engine, d.dtype, d.a_mode = engine, dtype, a_mode
    d.B, d.H, d.W, d.C_in, d.ld_in, d.C_out = 1, 7, 5, cin, cin + 64, 9 * cin
    d.KH = d.KW = 3
    d.stride, d.pad, d.OH, d.OW = 1, 1, 7, 5
    d.out_mode, d.ld_out, d.n_tile, d.ld_om = L.CT_OUT_NHWC, 9 * cin + 16, n, 28
    if L.conv_config(d) is not None:
      ok.append(n)
  return ok


@pytest.mark.parametrize('path', ['gather_bf16', 'window_bf16', 'x3'])
def test_probe_every_n_tile(path):
  cin = 16 if path != 'window_bf16' else 64
  tiles = _n_tiles(path, cin)
  assert tiles[:8] == list(range(16, 129, 16)), tiles
  if path != 'x3':
    assert tiles == list(range(16, 257, 16)), tiles
  for n in tiles:
    s = launch(path, 2, 7, 5, cin, n_tile=n, ld_om=36, seed=n)
    check(path, s, 'n_tile %d, 2x7x5 C_in %d' % (n, cin))


@pytest.mark.parametrize('margin', [0, 6])
def test_probe_window_margins(margin):
  """CT_A_DCN_WIN at the smallest and largest offset margin (CTB_TC_DCN_MARGIN, read once per process) in a process of
  its own; the default margin 2 runs above."""
  here = os.path.dirname(os.path.abspath(__file__))
  ids = ['%s::test_probe_samples_equal_oracle[%s]' % (os.path.join(here, 'test_gpu_dcn_sampler.py'),
                                                      '%s-%dx%dx%d-c%d' % ((p,) + c)) for p, c in CASES if p == 'window_bf16']
  env = dict(os.environ, CTB_TC_DCN_MARGIN=str(margin))
  r = subprocess.run([sys.executable, '-m', 'pytest', '-q', '-s', '-p', 'no:cacheprovider'] + ids,
                     cwd=os.path.dirname(here), env=env, capture_output=True, text=True)
  print('\n'.join(l for l in r.stdout.splitlines() if '[window_bf16]' in l))
  assert r.returncode == 0 and '%d passed' % len(ids) in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]


@pytest.mark.parametrize('path', [p[0] for p in PATHS])
def test_random_weights_over_the_catalogue(path):
  """The probe tied to ordinary use: random weights over the same catalogue and poisoned buffers, against the fp64
  GEMM of the path's exact columns with the per-element bound of tests/bounds.py."""
  _, engine, dtype, a_mode = _path(path)
  B, H, W, cin, cout = 2, 33, 61, 64, 96
  g = torch.Generator().manual_seed(5)
  w = torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (cin * 9)) ** 0.5
  s = launch(path, B, H, W, cin, w=w, ld_om=36 if engine != L.CT_ENGINE_SIMT else 27, seed=9)
  cols = expected(path, s)                                    # [B, H, W, 9, C]
  if path in ('simt_bf16', 'x3'):                             # these GEMMs read the fp32 sample itself (x3: split)
    cols = co.dcn_sample_columns(s['x'], s['off'], s['mask'], fp32_chain=True).permute(0, 3, 4, 2, 1)
  wq = w.bfloat16().double() if engine == L.CT_ENGINE_TCGEN05 else w.double()
  wm = wq.permute(0, 2, 3, 1).reshape(cout, 9 * cin).cuda()     # k = tap C_in + c
  cm = cols.reshape(B, H, W, 9 * cin)
  ref = torch.einsum('ok,bhwk->bohw', wm, cm)
  mag = torch.einsum('ok,bhwk->bohw', wm.abs(), cm.abs())
  coef = {L.CT_ENGINE_SIMT: bd.GAMMA_SIMT, L.CT_ENGINE_TCGEN05: bd.ALPHA_BF16, L.CT_ENGINE_TCGEN05_X3: bd.BETA_X3}[engine]
  got = s['out'].permute(0, 3, 1, 2).float()
  m = bd.assert_bound(got, ref, mag, coef, dtype == L.CT_BF16, '%s random weights' % path)
  print('[%s] random weights 2x33x61 64 -> 96: worst |err| / bound %.3f' % (path, m))


def test_zz_report_counts():
  """Per path: the samples checked in each catalogue category (and the window / global split) by the probe launches
  THIS process ran before this test -- a -k selection, another order or a distributed run reports fewer launches (or
  none), and the margin 0 / 6 launches of their child processes are not counted here."""
  print('\nprobe launches checked in this process: %s' % (
      ', '.join('%s %d' % (p, COUNTS[p]['(launches)']) for p in sorted(COUNTS)) or 'none'))
  for path in sorted(COUNTS):
    print('[%s] %s' % (path, ', '.join('%s %d' % kv for kv in sorted(COUNTS[path].items()))))
