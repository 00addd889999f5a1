"""-m gpu: conv_tma_kernel at patch counts the bench shapes do not reach -- one 8 x 16 patch, odd counts, stride 2, a
concat-slice input and output -- against the fp64 per-element bounds of tests/bounds.py, bit for bit across every N tile
(each N has its own stage count and the epilogue passes 16 columns at a time), and in a CUDA graph replay of the fp32
offset-map output."""
import pytest
import torch

from centertrack_b200 import _lib as L
from gpu_helpers import conv_desc
from test_gpu_conv_tma import BF16, _check, _launch, _operands, _run

pytestmark = pytest.mark.gpu

# (B, C_in, C_out, H, W, k, stride, residual, ld_pad, ch_off, out_pad, out_off)
CASES = [
    ('one patch', 1, 128, 128, 8, 16, 3, 1, True, 0, 0, 0, 0),
    ('3 patches', 3, 256, 256, 8, 16, 3, 1, False, 0, 0, 0, 0),
    ('5 patches, stride 2', 5, 128, 256, 16, 32, 3, 2, False, 0, 0, 0, 0),
    ('97 patches', 97, 128, 128, 8, 16, 3, 1, True, 0, 0, 0, 0),
    ('3 patches, slice in, concat out', 3, 448, 128, 8, 16, 1, 1, True, 64, 64, 128, 64),
    ('C_out 80 at N 64, 3 patches', 3, 64, 80, 8, 16, 3, 1, True, 0, 0, 0, 0),
]


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_tma_conv_within_bounds(built_lib, case):
  _, B, Cin, Cout, H, W, k, s, res, ld_pad, ch_off, out_pad, out_off = case
  x, w, b = _operands(B, Cin, Cout, H, W, k, seed=B * 7 + Cin + k)
  OH, OW = (H + 2 * (k // 2) - k) // s + 1, (W + 2 * (k // 2) - k) // s + 1
  r = torch.randn(B, Cout, OH, OW, generator=torch.Generator().manual_seed(5)) if res else None
  got, d, _ = _run(x, w, b, s, n_tile=64 if Cout == 80 else 0, res=r, ld_pad=ld_pad, ch_off=ch_off, out_pad=out_pad,
                   out_off=out_off)
  assert L.conv_config(d).tile_w == 16
  _check(got, x, w, b, s, r, what=case[0])


@pytest.mark.parametrize('shape', [(1, 128, 128, 8, 16, 1), (3, 256, 256, 8, 16, 1), (5, 128, 256, 16, 32, 2)],
                         ids=['one_patch', '3_patches', '5_patches_stride2'])
def test_every_n_tile_is_bit_identical(built_lib, shape):
  B, Cin, Cout, H, W, s = shape
  x, w, b = _operands(B, Cin, Cout, H, W, 3, seed=3)
  ref = None
  for n in range(16, 257, 16):
    got, _, _ = _run(x, w, b, s, n_tile=n)
    if ref is None:
      ref = got
    assert torch.equal(got, ref), 'N = %d differs from N = 16' % n


def test_graph_replay_of_the_offset_map_is_bit_identical(built_lib):
  # C_out 27 into a 32-wide fp32 map at N = 32 over 3 patches
  x, w, b = _operands(3, 256, 27, 8, 16, 3, seed=12)
  d, out, keep = conv_desc(*BF16, x.cuda(), w, b, 1, False, None, n_tile=32, out_mode=L.CT_OUT_NHWC_F32, sig_from=18)
  _launch(d)
  torch.cuda.synchronize()
  eager = out.clone()
  out.zero_()
  s = torch.cuda.Stream()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.stream(s):
    with torch.cuda.graph(g, stream=s):
      _launch(d)
  g.replay()
  g.replay()
  torch.cuda.synchronize()
  assert torch.equal(out, eager)
