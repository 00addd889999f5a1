"""-m gpu: the TMA-fed plain convolution of the bf16 gather engine (conv_tma_kernel: C_in % 64 == 0, 8 x 16 patches that
pad the map by at most 15 %; the other shapes below check the register gather that takes them) against the fp64
per-element bounds of tests/bounds.py, and bit for bit against itself wherever the sum order of an output element is
fixed: at every N tile, at B = n inside a larger allocation, and in a CUDA graph replay."""
import ctypes as C

import pytest
import torch

import bounds as bd
from centertrack_b200 import _lib as L
from gpu_helpers import conv_desc

pytestmark = pytest.mark.gpu

BF16 = (L.CT_ENGINE_TCGEN05, L.CT_BF16)


def _operands(B, Cin, Cout, H, W, k, seed, res=False):
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(B, Cin, H, W, generator=g)
  w = torch.randn(Cout, Cin, k, k, generator=g) * (2.0 / (Cin * k * k)) ** 0.5
  b = torch.randn(Cout, generator=g) * 0.1
  return x, w, b


def _launch(d):
  L.check(L.lib().ct_conv_forward(C.byref(d), L.stream_ptr()), 'conv')


def _run(x, w, b, s, n_tile=0, res=None, ld_pad=0, ch_off=0, out_pad=0, out_off=0, out_mode=L.CT_OUT_NHWC, relu=True):
  """One launch; out_pad / out_off: the output is channels out_off .. out_off + C_out of a wider NHWC buffer (a concat
  slice) whose other channels must stay NaN.  -> (output NCHW fp32, descriptor, buffers)."""
  d, out, keep = conv_desc(*BF16, x.cuda(), w, b, s, relu, res.cuda() if res is not None else None, n_tile=n_tile,
                           ld_pad=ld_pad, ch_off=ch_off, out_mode=out_mode)
  if out_pad:
    B, OH, OW, O = out.shape
    wide = torch.full((B, OH, OW, O + out_pad), float('nan'), dtype=out.dtype, device=out.device)
    d.out, d.ld_out = wide.data_ptr() + out_off * wide.element_size(), O + out_pad
    _launch(d)
    torch.cuda.synchronize()
    rest = torch.cat([wide[..., :out_off], wide[..., out_off + O:]], -1)
    assert torch.isnan(rest.float()).all(), 'store outside the output slice'
    return wide[..., out_off:out_off + O].permute(0, 3, 1, 2).float(), d, keep + (wide,)
  _launch(d)
  torch.cuda.synchronize()
  if out_mode == L.CT_OUT_NHWC_F32:
    return out[..., :w.shape[0]].permute(0, 3, 1, 2), d, keep + (out,)
  return out.permute(0, 3, 1, 2).float(), d, keep + (out,)


def _check(got, x, w, b, s, res=None, bf16_out=True, what=''):
  p = w.shape[-1] // 2
  wq = w.float().bfloat16().double().cuda()
  xq = x.bfloat16().double().cuda()
  rq = res.bfloat16().double().cuda() if res is not None else None
  ref, mag = bd.conv_ref(xq, wq, b, rq, s, (p, p, p, p))
  bd.assert_bound(got, ref, mag, bd.ALPHA_BF16, bf16_out, what, act='relu')


# (B, C_in, C_out, H, W, k, stride, residual, ld_pad, ch_off, out_pad, out_off)
CASES = [
    ('3x3 s1 level4', 32, 256, 256, 32, 32, 3, 1, True, 0, 0, 0, 0),
    ('3x3 s2 level5', 32, 256, 512, 32, 32, 3, 2, False, 0, 0, 0, 0),
    ('3x3 s2 odd input', 3, 128, 256, 35, 61, 3, 2, False, 0, 0, 0, 0),
    ('1x1 root slice in, concat out', 4, 448, 128, 64, 64, 1, 1, True, 64, 64, 128, 64),
    ('3x3 slice in (ld_in > C_in)', 2, 128, 128, 64, 64, 3, 1, False, 320, 192, 0, 0),
    ('3x3 mot level5 17x30', 3, 512, 512, 17, 30, 3, 1, True, 768, 0, 0, 0),
    ('3x3 nuscenes level5 14x25', 2, 512, 512, 14, 25, 3, 1, False, 0, 0, 768, 0),
    ('3x3 partial patches 60x120', 2, 128, 128, 60, 120, 3, 1, True, 0, 0, 0, 0),
    ('3x3 OH < 8', 5, 64, 64, 7, 32, 3, 1, False, 0, 0, 0, 0),
    ('B 1, fewer tiles than SMs', 1, 256, 256, 16, 16, 3, 1, True, 0, 0, 0, 0),
    ('B 97, more items than CTAs', 97, 128, 128, 32, 32, 3, 1, False, 0, 0, 0, 0),
    ('C_out 80 at N 64', 2, 64, 80, 40, 24, 3, 1, True, 0, 0, 0, 0),
]


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_tma_conv_within_bounds(built_lib, case):
  _, B, Cin, Cout, H, W, k, s, res, ld_pad, ch_off, out_pad, out_off = case
  x, w, b = _operands(B, Cin, Cout, H, W, k, seed=B * 7 + Cin + k)
  OH, OW = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
  r = torch.randn(B, Cout, OH, OW, generator=torch.Generator().manual_seed(5)) if res else None
  n_tile = 64 if Cout == 80 else 0
  got, d, _ = _run(x, w, b, s, n_tile=n_tile, res=r, ld_pad=ld_pad, ch_off=ch_off, out_pad=out_pad, out_off=out_off)
  util = OH * OW / (((OW + 15) // 16) * ((OH + 7) // 8) * 128.0)
  assert (L.conv_config(d).tile_w == 16) == (util >= 0.85)      # mot / nuScenes level5: the register gather
  _check(got, x, w, b, s, r, what=case[0])


def test_tma_conv_offset_map_fp32_out(built_lib):
  # the DCN offset convs: C_out 27 into a 32-wide fp32 map, sigmoid from channel 18, N = 32 (C_out not a multiple of N)
  x, w, b = _operands(2, 256, 27, 32, 32, 3, seed=11)
  d, out, keep = conv_desc(*BF16, x.cuda(), w, b, 1, False, None, n_tile=32, out_mode=L.CT_OUT_NHWC_F32, sig_from=18)
  _launch(d)
  torch.cuda.synchronize()
  got = out[..., :27].permute(0, 3, 1, 2)
  wq, xq = w.float().bfloat16().double().cuda(), x.bfloat16().double().cuda()
  ref, mag = bd.conv_ref(xq, wq, b, None, 1, (1, 1, 1, 1))
  bd.assert_bound(got[:, :18], ref[:, :18], mag[:, :18], bd.ALPHA_BF16, False, 'offsets')
  bd.assert_bound(got[:, 18:], ref[:, 18:], mag[:, 18:], bd.ALPHA_BF16, False, 'masks', act='sigmoid')


@pytest.mark.parametrize('shape', [(32, 256, 256, 32, 32, 1), (3, 512, 512, 17, 30, 1), (4, 128, 256, 64, 64, 2)],
                         ids=['level4', 'mot_level5', 'stride2'])
def test_every_n_tile_is_bit_identical(built_lib, shape):
  B, Cin, Cout, H, W, s = shape
  x, w, b = _operands(B, Cin, Cout, H, W, 3, seed=3)
  ref = None
  for n in range(16, 257, 16):
    got, _, _ = _run(x, w, b, s, n_tile=n)
    if ref is None:
      ref = got
    assert torch.equal(got, ref), 'N = %d differs from N = 16' % n


def test_batch_prefix_of_a_larger_allocation_is_bit_identical(built_lib):
  # B = n < B_alloc as the idle-streams runner issues it: the first n images of a 32-image buffer
  x, w, b = _operands(32, 256, 256, 32, 32, 3, seed=4)
  full, d, keep = _run(x, w, b, 1)
  for n in (1, 5, 31):
    d.B = n
    out = keep[-1]
    out.zero_()
    _launch(d)
    torch.cuda.synchronize()
    assert torch.equal(out[:n].permute(0, 3, 1, 2).float(), full[:n]), n
    assert (out[n:] == 0).all(), 'store past image %d' % n
    alone, _, _ = _run(x[:n], w, b, 1)
    assert torch.equal(alone, full[:n]), n


def test_graph_replay_is_bit_identical(built_lib):
  x, w, b = _operands(8, 512, 512, 16, 16, 3, seed=6)
  eager, d, keep = _run(x, w, b, 1)
  out = keep[-1]
  out.zero_()
  s = torch.cuda.Stream()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.stream(s):
    with torch.cuda.graph(g, stream=s):
      _launch(d)
  g.replay()
  g.replay()
  torch.cuda.synchronize()
  assert torch.equal(out.permute(0, 3, 1, 2).float(), eager)
