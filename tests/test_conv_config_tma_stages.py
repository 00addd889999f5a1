"""ct_conv_config (host code, no GPU) of conv_tma_kernel at every batch a runner is built at: with the epilogue staged
16 columns at a time, each TMA launch of the four bench plans holds as many stages (up to 4) as fit in its CTA's share
of the SM -- 3 at N = 128, 4 at N <= 64 -- and odd numbers of 8 x 16 patches are accepted."""
import pytest

from centertrack_b200 import _lib as L
from plan_rows import BATCHES, BENCH_SHAPES, cpu_plan

A_STAGE, STAGING = 16384, 2 * 64 * 20 * 4        # one A box; both warpgroups' 64 x 16 fp32 staging tiles (pitch 20)


def _smem(n_tile, stages):
  return stages * (A_STAGE + n_tile * 128) + STAGING + 16 * stages + 1024


def _stages_that_fit(n_tile):
  limit = (113 if n_tile <= 128 else 227) << 10
  s = 4
  while s > 2 and _smem(n_tile, s) > limit:
    s -= 1
  return s


@pytest.mark.parametrize('cfg', sorted(BENCH_SHAPES))
@pytest.mark.parametrize('B', BATCHES)
def test_every_tma_launch_holds_the_stages_that_fit(built_lib, cfg, B):
  eng = cpu_plan(cfg, BENCH_SHAPES[cfg], B, 'bf16')
  tma = [(name, d, L.conv_config(d)) for kind, d, name in eng.ops
         if kind == 'conv' and d.engine == L.CT_ENGINE_TCGEN05 and d.a_mode == L.CT_A_CONV]
  tma = [(name, d, c) for name, d, c in tma if (c.tile_w, c.tile_h) == (16, 8)]
  assert tma, cfg
  for name, d, c in tma:
    assert c.stages == _stages_that_fit(d.n_tile), (name, d.n_tile, c.stages)
    assert c.smem_bytes == _smem(d.n_tile, c.stages), (name, c.smem_bytes)
    assert c.smem_bytes <= (113 if d.n_tile <= 128 else 227) << 10, (name, c.smem_bytes)


@pytest.mark.parametrize('n_tile,stages', [(16, 4), (32, 4), (64, 4), (96, 3), (128, 3), (256, 4)])
def test_stage_counts(built_lib, n_tile, stages):
  assert _stages_that_fit(n_tile) == stages


@pytest.mark.parametrize('B,H,W', [(1, 8, 16), (3, 8, 16), (5, 16, 32), (97, 8, 16)])
def test_odd_patch_counts_are_accepted(built_lib, B, H, W):
  d = L.ConvDesc()
  d.engine, d.dtype, d.a_mode = L.CT_ENGINE_TCGEN05, L.CT_BF16, L.CT_A_CONV
  d.B, d.H, d.W, d.C_in, d.ld_in, d.C_out = B, H, W, 128, 128, 128
  d.KH = d.KW = 3
  d.stride, d.pad, d.OH, d.OW = 1, 1, H, W
  d.out_mode, d.ld_out, d.n_tile = L.CT_OUT_NHWC, 128, 128
  c = L.conv_config(d)
  assert c is not None and (c.tile_w, c.tile_h) == (16, 8) and c.stages == 3
