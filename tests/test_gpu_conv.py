"""-m gpu: the conv / DCN engines through ct_conv_forward (C ABI) against an fp64 reference computed from the operands
each kernel read (activations in the engine's dtype, weights rounded as ct_pack_weights rounds them), with the
per-element bounds of tests/bounds.py: bf16 outputs must be the round-to-nearest of a value within ALPHA_BF16 x mag of
the exact result, fp32 outputs within BETA_X3 (bf16x3) / GAMMA_SIMT (SIMT) / ALPHA_BF16 (bf16 engines) x mag, where mag
is the sum of the magnitudes of every term of the output."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import bounds as bd
import ct_oracle as co
from centertrack_b200 import _lib as L

pytestmark = pytest.mark.gpu

ENGINES = [('simt_f32', L.CT_ENGINE_SIMT, L.CT_F32), ('simt_bf16', L.CT_ENGINE_SIMT, L.CT_BF16),
           ('tcgen05', L.CT_ENGINE_TCGEN05, L.CT_BF16),
           # bf16 hi/lo split operands on fp32 activations, three MMAs per term
           ('tcgen05_x3', L.CT_ENGINE_TCGEN05_X3, L.CT_F32)]
COEF = {L.CT_ENGINE_SIMT: bd.GAMMA_SIMT, L.CT_ENGINE_TCGEN05: bd.ALPHA_BF16, L.CT_ENGINE_TCGEN05_HALO: bd.ALPHA_BF16,
        L.CT_ENGINE_TCGEN05_X3: bd.BETA_X3}
N_TILES = list(range(16, 257, 16))      # every instantiation of conv_tc_kernel / conv_halo_kernel


def _operands(engine, dtype, x, w, r=None):
  """fp64 CUDA copies of what the kernel reads: activations in its dtype, weights as packed (bf16 engines round
  the fp32 weight to bf16, x3 and SIMT keep fp32)."""
  act = torch.bfloat16 if dtype == L.CT_BF16 else torch.float32
  wq = w.float()
  if engine in (L.CT_ENGINE_TCGEN05, L.CT_ENGINE_TCGEN05_HALO):
    wq = wq.bfloat16()
  q = lambda t: t.to(act).double().cuda() if t is not None else None
  return q(x), wq.double().cuda(), q(r)


def _check(got, ref, mag, engine, dtype, what, act='none', out_f32=False, depth_scale=1.0):
  bf16_out = dtype == L.CT_BF16 and not out_f32
  return bd.assert_bound(got, ref, mag, COEF[engine], bf16_out, what, act, depth_scale)


def _conv_case(engine, dtype, B, Cin, Cout, H, W, k, s, res, seed, ld_pad=0, ch_off=0, n_tile=0, relu=True,
               out_mode=L.CT_OUT_NHWC):
  from gpu_helpers import run_conv
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(B, Cin, H, W, generator=g)
  w = torch.randn(Cout, Cin, k, k, generator=g) * (2.0 / (Cin * k * k)) ** 0.5
  b = torch.randn(Cout, generator=g) * 0.1
  OH, OW = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
  r = torch.randn(B, Cout, OH, OW, generator=g) if res else None
  xq, wq, rq = _operands(engine, dtype, x, w, r)
  p = k // 2
  ref, mag = bd.conv_ref(xq, wq, b, rq, s, (p, p, p, p))
  got = run_conv(engine, dtype, x.cuda(), w, b, s, relu, r.cuda() if res else None, ld_pad=ld_pad, ch_off=ch_off,
                 n_tile=n_tile, out_mode=out_mode)
  return got, ref, mag


def _case_list():
  from gpu_helpers import conv_cases
  return conv_cases()


N_CASES = 9
assert N_CASES == len(_case_list())


@pytest.mark.parametrize('eng', ENGINES, ids=[e[0] for e in ENGINES])
@pytest.mark.parametrize('case', range(N_CASES))
def test_conv_bn_residual_relu(eng, case):
  name, engine, dtype = eng
  cname, B, Cin, Cout, H, W, k, s, res, ld_pad, ch_off = _case_list()[case]
  got, ref, mag = _conv_case(engine, dtype, B, Cin, Cout, H, W, k, s, res, case, ld_pad, ch_off)
  _check(got, ref, mag, engine, dtype, '%s %s' % (name, cname), 'relu')


def test_conv_2d_pixel_patches():
  """The gather engine's 8 x 16 pixel-patch M tiles (CTB_TC_TILE2D=1, read once per process): the two conv_cases named
  after them, in a process of their own."""
  here = os.path.dirname(os.path.abspath(__file__))
  env = dict(os.environ, CTB_TC_TILE2D='1')
  ids = ['%s::test_conv_bn_residual_relu[%d-%s]' % (os.path.join(here, 'test_gpu_conv.py'), case, e[0])
         for case in (7, 8) for e in ENGINES]
  r = subprocess.run([sys.executable, '-m', 'pytest', '-q', '-p', 'no:cacheprovider'] + ids, cwd=os.path.dirname(here),
                     env=env, capture_output=True, text=True)
  assert r.returncode == 0 and '8 passed' in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]


@pytest.mark.parametrize('x3', [False, True], ids=['bf16', 'x3'])
@pytest.mark.parametrize('n_tile', N_TILES)
def test_gather_n_tile_sweep(x3, n_tile):
  """Every N instantiation of the gather kernel: a 3x3 64 -> N + 16 conv (K = 576, nine full K slices; a ragged second
  n-tile of 16 channels; 480 pixels = 3.75 M tiles, one straddling the two images), with a residual for odd N / 16,
  then a 1x1 head writing N + 3 fp32 NCHW channels."""
  engine, dtype = (L.CT_ENGINE_TCGEN05_X3, L.CT_F32) if x3 else (L.CT_ENGINE_TCGEN05, L.CT_BF16)
  res = (n_tile // 16) % 2 == 1
  got, ref, mag = _conv_case(engine, dtype, 2, 64, n_tile + 16, 12, 20, 3, 1, res, 1000 + n_tile, n_tile=n_tile)
  _check(got, ref, mag, engine, dtype, 'gather N=%d 3x3' % n_tile, 'relu')
  got, ref, mag = _conv_case(engine, dtype, 2, 64, n_tile + 3, 8, 40, 1, 1, False, 2000 + n_tile, n_tile=n_tile,
                             relu=False, out_mode=L.CT_OUT_NCHW_F32)
  _check(got, ref, mag, engine, dtype, 'gather N=%d head' % n_tile, out_f32=True)


@pytest.mark.parametrize('eng', ENGINES, ids=[e[0] for e in ENGINES])
@pytest.mark.parametrize('cout_act', [(2, 0), (80, 1), (1, 2), (17, 1)])
def test_head_1x1_writes_reference_layout_with_fused_activation(eng, cout_act):
  from gpu_helpers import run_conv
  _, engine, dtype = eng
  Cout, act = cout_act
  g = torch.Generator().manual_seed(Cout)
  x = torch.randn(2, 256, 16, 24, generator=g)
  w = torch.randn(Cout, 256, 1, 1, generator=g) * 0.05
  b = torch.randn(Cout, generator=g)
  xq, wq, _ = _operands(engine, dtype, x, w)
  ref, mag = bd.conv_ref(xq, wq, b)
  got = run_conv(engine, dtype, x.cuda(), w, b, 1, False, out_mode=L.CT_OUT_NCHW_F32, head_act=act)
  _check(got, ref, mag, engine, dtype, 'head', ('none', 'sigmoid', 'depth')[act], out_f32=True)


DCN_ENGINES = [ENGINES[0], ENGINES[2], ENGINES[2] + ('win',), ENGINES[3]]


@pytest.mark.parametrize('eng', DCN_ENGINES, ids=['simt_f32', 'tcgen05', 'tcgen05_window', 'tcgen05_x3'])
@pytest.mark.parametrize('shape', [(1, 64, 64, 24, 40), (2, 128, 64, 16, 16), (1, 256, 256, 8, 12),
                                   (1, 512, 256, 4, 6), (1, 64, 64, 5, 7), (2, 64, 64, 24, 32), (3, 64, 128, 40, 56),
                                   (4, 64, 64, 64, 96), (4, 128, 64, 64, 96)])     # > 148 patches: several tiles per persistent CTA
def test_dcn_v2(eng, shape):
  """Offset/mask conv + modulated deformable conv; large offsets push samples across and beyond the
  border (zero padding, partial bilinear weights) and, for the shared-memory-window variant (CT_A_DCN_WIN), beyond
  the staged window (global fall-back path) -- ragged 8x16 patches included.  The bf16 samplers' columns are
  emulated exactly (fp64 blend, one bf16 rounding per fma step), so the GEMM gets the plain bf16 bound."""
  from gpu_helpers import run_conv
  _, engine, dtype = eng[:3]
  dcn_mode = L.CT_A_DCN_WIN if len(eng) > 3 else L.CT_A_DCN
  B, Cin, Cout, H, W = shape
  g = torch.Generator().manual_seed(H * W)
  x = torch.randn(B, Cin, H, W, generator=g)
  w = torch.randn(Cout, Cin, 3, 3, generator=g) * (2.0 / (Cin * 9)) ** 0.5
  b = torch.randn(Cout, generator=g) * 0.1
  wo = torch.randn(27, Cin, 3, 3, generator=g) * (0.6 / (Cin * 9) ** 0.5)
  bo = torch.randn(27, generator=g) * 1.5
  tc = engine == L.CT_ENGINE_TCGEN05
  xq, woq, _ = _operands(engine, dtype, x, wo)
  om_ref, om_mag = bd.conv_ref(xq, woq, bo, pad=(1, 1, 1, 1))
  om = run_conv(engine, dtype, x.cuda(), wo, bo, 1, relu=False, out_mode=L.CT_OUT_NHWC_F32, sig_from=18, n_tile=32)
  _check(om[:, :18], om_ref[:, :18], om_mag[:, :18], engine, dtype, 'offsets', out_f32=True)
  _check(om[:, 18:27], om_ref[:, 18:27], om_mag[:, 18:27], engine, dtype, 'mask', 'sigmoid', out_f32=True)
  # feed the DEVICE offsets to both sides so the sampling positions are identical
  om_dev = om.permute(0, 2, 3, 1).contiguous()
  assert float(om[:, :18].abs().max()) > 2.0          # the case really leaves the 3x3 window
  cols = co.dcn_sample_columns(xq, om[:, :18].contiguous(), om[:, 18:27].contiguous(), bf16_blend=tc)
  _, wq, _ = _operands(engine, dtype, x, w)
  wm, cols = wq.reshape(Cout, Cin * 9), cols.reshape(B, Cin * 9, H * W)
  ref = torch.matmul(wm, cols).view(B, Cout, H, W) + b.double().cuda().view(1, -1, 1, 1)
  mag = torch.matmul(wm.abs(), cols.abs()).view(B, Cout, H, W) + b.double().cuda().abs().view(1, -1, 1, 1)
  got = run_conv(engine, dtype, x.cuda(), w, b, 1, relu=True, a_mode=dcn_mode, om=om_dev)
  _check(got, ref, mag, engine, dtype, 'dcn', 'relu')


HALO_CASES = [('3x3 64->64 +res', 2, 64, 64, 24, 40, 3, True, 0), ('3x3 16->16', 1, 16, 16, 40, 56, 3, False, 0),
              ('3x3 32->64 ragged tile', 1, 32, 64, 20, 28, 3, False, 0), ('1x1 64->32', 1, 64, 32, 16, 24, 1, False, 0),
              ('3x3 64->1024 8 n-tiles', 1, 64, 1024, 16, 24, 3, False, 128), ('3x3 48->16 odd size', 1, 48, 16, 33, 17, 3, False, 0),
              ('3x3 64->64 many tiles per CTA', 4, 64, 64, 128, 128, 3, True, 0),
              ('3x3 128->128 two 64-ch chunks', 2, 128, 128, 24, 40, 3, True, 32),
              ('1x1 256->128 four chunks', 1, 256, 128, 16, 24, 1, False, 128), ('3x3 128->64', 1, 128, 64, 20, 28, 3, False, 32)] + \
    [('3x3 32->%d N=%d' % (n + 16, n), 2, 32, n + 16, 20, 28, 3, (n // 16) % 2 == 1, n) for n in N_TILES]
    # the sweep: every N instantiation, a ragged second n-tile of 16 channels, ragged 8 x 16 tiles, residual for odd N / 16


@pytest.mark.parametrize('case', range(len(HALO_CASES)), ids=[c[0] for c in HALO_CASES])
def test_halo_engine_conv(case):
  """CT_ENGINE_TCGEN05_HALO (TMA halo tile, taps by descriptor shift, persistent CTAs): multi-tile persistence,
  n-tiling, image borders and ragged tiles."""
  from gpu_helpers import run_conv
  name, B, Cin, Cout, H, W, k, res, nt = HALO_CASES[case]
  g = torch.Generator().manual_seed(100 + case)
  x = torch.randn(B, Cin, H, W, generator=g)
  w = torch.randn(Cout, Cin, k, k, generator=g) * (2.0 / (Cin * k * k)) ** 0.5
  b = torch.randn(Cout, generator=g) * 0.1
  r = torch.randn(B, Cout, H, W, generator=g) if res else None
  xq, wq, rq = _operands(L.CT_ENGINE_TCGEN05_HALO, L.CT_BF16, x, w, r)
  p = k // 2
  ref, mag = bd.conv_ref(xq, wq, b, rq, 1, (p, p, p, p))
  got = run_conv(L.CT_ENGINE_TCGEN05_HALO, L.CT_BF16, x.cuda(), w, b, 1, True, r.cuda() if res else None, n_tile=nt)
  _check(got, ref, mag, L.CT_ENGINE_TCGEN05_HALO, L.CT_BF16, name, 'relu')


@pytest.mark.parametrize('n_tile', N_TILES)
def test_halo_head_n_tile_sweep(n_tile):
  """Every N instantiation of the halo kernel writing fp32 NCHW head planes (N + 3 channels: a ragged second n-tile)
  through the 32 x 4 wide tile, with the fused sigmoid for odd N / 16."""
  from gpu_helpers import run_conv
  g = torch.Generator().manual_seed(3000 + n_tile)
  x = torch.randn(2, 64, 8, 64, generator=g)
  w = torch.randn(n_tile + 3, 64, 1, 1, generator=g) * 0.1
  b = torch.randn(n_tile + 3, generator=g)
  act = (n_tile // 16) % 2
  xq, wq, _ = _operands(L.CT_ENGINE_TCGEN05_HALO, L.CT_BF16, x, w)
  ref, mag = bd.conv_ref(xq, wq, b)
  got = run_conv(L.CT_ENGINE_TCGEN05_HALO, L.CT_BF16, x.cuda(), w, b, 1, relu=False, out_mode=L.CT_OUT_NCHW_F32,
                 head_act=act, n_tile=n_tile)
  _check(got, ref, mag, L.CT_ENGINE_TCGEN05_HALO, L.CT_BF16, 'halo head N=%d' % n_tile, ('none', 'sigmoid')[act],
         out_f32=True)


def test_halo_engine_fp32_outputs():
  from gpu_helpers import run_conv
  H_ = L.CT_ENGINE_TCGEN05_HALO
  g = torch.Generator().manual_seed(21)
  x = torch.randn(1, 64, 24, 40, generator=g)
  w = torch.randn(27, 64, 3, 3, generator=g) * 0.03
  b = torch.randn(27, generator=g)
  xq, wq, _ = _operands(H_, L.CT_BF16, x, w)
  ref, mag = bd.conv_ref(xq, wq, b, pad=(1, 1, 1, 1))
  got = run_conv(H_, L.CT_BF16, x.cuda(), w, b, 1, relu=False, out_mode=L.CT_OUT_NHWC_F32, sig_from=18, n_tile=32)
  _check(got[:, :18], ref[:, :18], mag[:, :18], H_, L.CT_BF16, 'offsets', out_f32=True)
  _check(got[:, 18:27], ref[:, 18:], mag[:, 18:], H_, L.CT_BF16, 'mask', 'sigmoid', out_f32=True)
  x = torch.randn(2, 64, 16, 24, generator=g)
  w = torch.randn(80, 64, 1, 1, generator=g) * 0.1
  b = torch.randn(80, generator=g)
  xq, wq, _ = _operands(H_, L.CT_BF16, x, w)
  ref, mag = bd.conv_ref(xq, wq, b)
  got = run_conv(H_, L.CT_BF16, x.cuda(), w, b, 1, relu=False, out_mode=L.CT_OUT_NCHW_F32, head_act=1, n_tile=80)
  _check(got, ref, mag, H_, L.CT_BF16, 'hm 8x16 tile', 'sigmoid', out_f32=True)
  # 32 x 4 pixel tiles (W % 32 == 0): the 1x1 heads at full resolution, 256 input channels in four chunks
  x = torch.randn(2, 256, 8, 64, generator=g)
  w = torch.randn(80, 256, 1, 1, generator=g) * 0.05
  xq, wq, _ = _operands(H_, L.CT_BF16, x, w)
  ref, mag = bd.conv_ref(xq, wq, b)
  got = run_conv(H_, L.CT_BF16, x.cuda(), w, b, 1, relu=False, out_mode=L.CT_OUT_NCHW_F32, head_act=1, n_tile=80)
  _check(got, ref, mag, H_, L.CT_BF16, 'hm 32x4 tile', 'sigmoid', out_f32=True)
  w2 = torch.randn(2, 256, 1, 1, generator=g) * 0.05
  xq, wq, _ = _operands(H_, L.CT_BF16, x, w2)
  ref, mag = bd.conv_ref(xq, wq, b[:2])
  got = run_conv(H_, L.CT_BF16, x.cuda(), w2, b[:2], 1, relu=False, out_mode=L.CT_OUT_NCHW_F32, n_tile=16)
  _check(got, ref, mag, H_, L.CT_BF16, 'reg 32x4 tile', out_f32=True)


@pytest.mark.parametrize('mask', [7, 1, 3])
def test_halo_engine_tensor_core_stem(mask):
  """7x7, C_in = 8 = (img3, pre3, hm1, 0), two taps per K=16 MMA, block-diagonal 48 outputs; the epilogue
  applies ReLU per stem and sums the PRESENT stems (mask bit g) -- dla.py:305-311."""
  from gpu_helpers import run_conv
  g = torch.Generator().manual_seed(mask)
  img, pre, hm = torch.randn(2, 3, 40, 56, generator=g), torch.randn(2, 3, 40, 56, generator=g), torch.rand(2, 1, 40, 56, generator=g)
  ws = [torch.randn(16, c, 7, 7, generator=g) * 0.1 for c in (3, 3, 1)]
  sh = torch.randn(48, generator=g) * 0.2
  w48 = torch.zeros(48, 8, 7, 7)
  w48[0:16, 0:3], w48[16:32, 3:6], w48[32:48, 6:7] = ws[0], ws[1], ws[2]
  x8 = torch.cat([img, pre, hm, torch.zeros(2, 1, 40, 56)], 1)
  xq, wq, _ = _operands(L.CT_ENGINE_TCGEN05_HALO, L.CT_BF16, x8, w48)
  ref, mag = bd.conv_ref(xq, wq, sh, pad=(3, 3, 3, 3))
  lo, hi = bd.stem_interval(ref, mag, bd.ALPHA_BF16, mask)
  got = run_conv(L.CT_ENGINE_TCGEN05_HALO, L.CT_BF16, x8.cuda(), w48, sh, 1, relu=False, n_tile=48, sum3=mask)
  r = bd.ratio_interval(got, lo, hi, True)
  assert float(r.max()) <= 1.0, 'stem: worst element %s, ratio %.3g' % bd.worst(r)[::-1]


def test_pack_stem_input():
  import ctypes as C
  g = torch.Generator().manual_seed(4)
  img, pre, hm = torch.randn(2, 3, 9, 13, generator=g).cuda(), torch.randn(2, 3, 9, 13, generator=g).cuda(), torch.rand(2, 1, 9, 13, generator=g).cuda()
  out = torch.empty(2, 9, 13, 8, dtype=torch.bfloat16, device='cuda')
  L.check(L.lib().ct_pack_stem_input(L.ptr(img), L.ptr(pre), L.ptr(None), L.ptr(out), 2, 9, 13, L.stream_ptr()))
  ref = torch.cat([img, pre, torch.zeros_like(hm), torch.zeros_like(hm)], 1).permute(0, 2, 3, 1).bfloat16()
  assert torch.equal(out, ref)


def test_halo_even_kernel_and_space_to_depth_output():
  """The two pieces of level1-as-a-2x2-convolution (engine.py): a 2x2 stride-1 conv padded on the top / left only, and a
  3x3 conv whose NHWC output is written space-to-depth; then the composition against the 3x3 stride-2 conv itself."""
  from gpu_helpers import run_conv
  H_, BF = L.CT_ENGINE_TCGEN05_HALO, L.CT_BF16
  g = torch.Generator().manual_seed(21)
  B, H, W = 2, 48, 80
  x = torch.randn(B, 64, H, W, generator=g)
  w = torch.randn(32, 64, 2, 2, generator=g) * 0.08
  b = torch.randn(32, generator=g) * 0.1
  got = run_conv(H_, BF, x.cuda(), w, b, 1, True, n_tile=32)
  xq, wq, _ = _operands(H_, BF, x, w)
  ref, mag = bd.conv_ref(xq, wq, b, pad=(1, 0, 1, 0))
  assert got.shape == ref.shape
  _check(got, ref, mag, H_, BF, '2x2 top/left padded', 'relu')

  x0 = torch.randn(B, 16, H, W, generator=g)
  w0 = torch.randn(16, 16, 3, 3, generator=g) * 0.15
  b0 = torch.randn(16, generator=g) * 0.1
  plain = run_conv(H_, BF, x0.cuda(), w0, b0, 1, True, n_tile=16).cpu()
  s2d = run_conv(H_, BF, x0.cuda(), w0, b0, 1, True, n_tile=16, out_mode=L.CT_OUT_NHWC_S2D).cpu()
  assert torch.equal(plain, s2d)                      # same values, only the layout differs

  # the stem's sum-of-three epilogue writing space-to-depth (what level0-on-the-s2d-grid reads)
  x8 = torch.randn(B, 8, H, W, generator=g)
  w48 = torch.randn(48, 8, 7, 7, generator=g) * 0.05
  b48 = torch.randn(48, generator=g) * 0.1
  st_plain = run_conv(H_, BF, x8.cuda(), w48, b48, 1, False, n_tile=48, sum3=7).cpu()
  st_s2d = run_conv(H_, BF, x8.cuda(), w48, b48, 1, False, n_tile=48, sum3=7, out_mode=L.CT_OUT_NHWC_S2D).cpu()
  assert st_plain.shape == (B, 16, H, W) and torch.equal(st_plain, st_s2d)

  # level2's inputs: 2x2 max-pool of a space-to-depth tensor, and the 3x3 stride-2 32 -> 64 conv as a 2x2 over 128 channels
  import ctypes as C
  y = torch.randn(B, 32, H, W, generator=g).bfloat16()
  ys = y.reshape(B, 32, H // 2, 2, W // 2, 2).permute(0, 2, 4, 3, 5, 1).reshape(B, H // 2, W // 2, 128).contiguous().cuda()
  po = torch.empty(B, H // 2, W // 2, 32, dtype=torch.bfloat16, device='cuda')
  L.check(L.lib().ct_maxpool2_s2d(L.ptr(ys), L.ptr(po), L.CT_BF16, B, H // 2, W // 2, 32, 128, 32, L.stream_ptr()))
  assert torch.equal(po.permute(0, 3, 1, 2).float().cpu(), F.max_pool2d(y.float(), 2, 2))
  from centertrack_b200.engine import s2d_weights_3x3_s2
  w2 = torch.randn(64, 32, 3, 3, generator=g) * 0.08
  b2 = torch.randn(64, generator=g) * 0.1
  via2 = run_conv(H_, BF, ys.permute(0, 3, 1, 2).float(), s2d_weights_3x3_s2(w2), b2, 1, True, n_tile=64)
  yq, w2q, _ = _operands(H_, BF, y.float(), w2)
  ref2, mag2 = bd.conv_ref(yq, w2q, b2, None, 2, (1, 1, 1, 1))     # the regrouping moves weights, it rounds none
  _check(via2, ref2, mag2, H_, BF, '3x3 s2 as 2x2 over space-to-depth', 'relu')

  # composition: 3x3 stride-2 16 -> 32 == 2x2 stride-1 over the space-to-depth view with the regrouped weights
  w1 = torch.randn(32, 16, 3, 3, generator=g) * 0.1
  b1 = torch.randn(32, generator=g) * 0.1
  w1s = torch.zeros(32, 64, 2, 2)
  tap = ((0, 1), (1, 0), (1, 1))
  for ky in range(3):
    for kx in range(3):
      (ty, sy), (tx, sx) = tap[ky], tap[kx]
      w1s[:, (sy * 2 + sx) * 16:(sy * 2 + sx) * 16 + 16, ty, tx] = w1[:, :, ky, kx]
  xs = plain.reshape(B, 16, H // 2, 2, W // 2, 2).permute(0, 3, 5, 1, 2, 4).reshape(B, 64, H // 2, W // 2)
  via = run_conv(H_, BF, xs.cuda(), w1s, b1, 1, True, n_tile=32)
  direct = run_conv(L.CT_ENGINE_TCGEN05, BF, plain.cuda(), w1, b1, 2, True)
  pq, w1q, _ = _operands(H_, BF, plain, w1)
  ref1, mag1 = bd.conv_ref(pq, w1q, b1, None, 2, (1, 1, 1, 1))
  _check(via, ref1, mag1, H_, BF, '3x3 s2 16->32 via space-to-depth', 'relu')
  _check(direct, ref1, mag1, L.CT_ENGINE_TCGEN05, BF, '3x3 s2 16->32 gather', 'relu')


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_maxpool_and_upsample_add(dtype):
  lib = L.lib()
  import ctypes as C
  ct = L.CT_F32 if dtype == torch.float32 else L.CT_BF16
  g = torch.Generator().manual_seed(3)
  x = torch.randn(2, 32, 12, 20, generator=g).to(dtype)
  xn = x.permute(0, 2, 3, 1).contiguous().cuda()
  out = torch.zeros(2, 6, 10, 48, dtype=dtype, device='cuda')          # write into a slice of a wider buffer
  L.check(lib.ct_maxpool2(L.ptr(xn), C.c_void_p(out.data_ptr() + 8 * out.element_size()), ct, 2, 12, 20, 32, 32, 48,
                          L.stream_ptr()))
  ref = F.max_pool2d(x.float(), 2, 2)
  assert torch.equal(out[..., 8:40].permute(0, 3, 1, 2).float().cpu(), ref)
  assert float(out[..., :8].abs().max()) == 0 and float(out[..., 40:].abs().max()) == 0
  for f in (2, 4, 8):
    w = torch.rand(32, 1, 2 * f, 2 * f, generator=g)
    skip = torch.randn(2, 32, 12 * f, 20 * f, generator=g).to(dtype)
    o = torch.empty(2, 12 * f, 20 * f, 32, dtype=dtype, device='cuda')
    wd = w.reshape(32, 2 * f, 2 * f).permute(1, 2, 0).contiguous().cuda()     # channel-last
    sk = skip.permute(0, 2, 3, 1).contiguous().cuda()
    L.check(lib.ct_upsample_add(L.ptr(xn), L.ptr(sk), L.ptr(wd), L.ptr(o), ct, 2, 12, 20, 32, f, 32, 32, 32,
                                L.stream_ptr()))
    ref = F.conv_transpose2d(x.float(), w, None, stride=f, padding=f // 2, groups=32) + skip.float()
    tol = 1e-5 if dtype == torch.float32 else 2e-2
    assert (o.permute(0, 3, 1, 2).float().cpu() - ref).abs().max() < tol


def test_stem_three_inputs_relu_before_sum():
  lib = L.lib()
  g = torch.Generator().manual_seed(9)
  B, H, W = 2, 40, 56
  img, pre, hm = torch.randn(B, 3, H, W, generator=g), torch.randn(B, 3, H, W, generator=g), torch.rand(B, 1, H, W, generator=g)
  ws = [torch.randn(16, c, 7, 7, generator=g) * 0.1 for c in (3, 3, 1)]
  sh = torch.randn(3, 16, generator=g) * 0.2
  wst = torch.zeros(49, 7, 16)
  for w, c0 in zip(ws, (0, 3, 6)):
    wst[:, c0:c0 + w.shape[1]] = w.permute(2, 3, 1, 0).reshape(49, w.shape[1], 16)
  w48 = torch.zeros(48, 8, 7, 7)
  w48[0:16, 0:3], w48[16:32, 3:6], w48[32:48, 6:7] = ws[0], ws[1], ws[2]
  x8 = torch.cat([img, pre, hm, torch.zeros(B, 1, H, W)], 1).double().cuda()
  ref, mag = bd.conv_ref(x8, w48.double(), sh.reshape(48), pad=(3, 3, 3, 3))
  out = torch.empty(B, H, W, 16, device='cuda')
  wd, sd_, di, dp, dh = wst.cuda(), sh.cuda(), img.cuda(), pre.cuda(), hm.cuda()     # keep alive
  args = (L.ptr(wd), L.ptr(sd_), L.ptr(out), L.CT_F32, B, H, W, 16, L.stream_ptr())
  for mask, ptrs in ((7, (di, dp, dh)), (1, (di, None, None))):       # mask 1: first frame of a plain detector
    L.check(lib.ct_stem_forward(*[L.ptr(t) for t in ptrs], *args))
    r = bd.ratio_interval(out.permute(0, 3, 1, 2), *bd.stem_interval(ref, mag, bd.GAMMA_SIMT, mask), False)
    assert float(r.max()) <= 1.0, 'stem mask %d: worst element %s, ratio %.3g' % ((mask,) + bd.worst(r)[::-1])


def test_conv_argument_validation():
  import ctypes as C
  lib = L.lib()
  d = L.ConvDesc()
  assert lib.ct_conv_forward(C.byref(d), None) == -1
  assert b'null pointer' in lib.ct_last_error()
