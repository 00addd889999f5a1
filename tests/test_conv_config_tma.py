"""ct_conv_config (host code, no GPU) of the TMA-fed plain convolutions of the bf16 gather engine: every such launch of
the four bench plans gets 16 x 8 patches and stages that fit in its CTA's share of the SM, and a refused shape returns
the status and message of ct_conv_forward."""
import ctypes as C

import pytest

from centertrack_b200 import _lib as L

PLANS = {'coco_tracking': (512, 512), 'mot': (544, 960), 'nuscenes_ddd': (448, 800), 'coco_pose': (512, 512)}


@pytest.mark.parametrize('cfg', sorted(PLANS))
def test_plain_gather_launches_take_the_tma_path_and_fit(built_lib, cfg):
  from helpers import make_model
  from centertrack_b200.engine import DLA34Engine
  opt, model, _ = make_model(cfg)
  H, W = PLANS[cfg]
  eng = DLA34Engine(model._engine_state_dict(), model.heads, 32, H, W, precision='bf16', device='cpu',
                    depth_scale=getattr(opt, 'depth_scale', 1.0))
  plain = [(name, d, L.conv_config(d)) for kind, d, name in eng.ops
           if kind == 'conv' and d.engine == L.CT_ENGINE_TCGEN05 and d.a_mode == L.CT_A_CONV]
  tma = [(name, d, c) for name, d, c in plain if (c.tile_w, c.tile_h) == (16, 8)]
  for name, d, c in plain:
    assert d.C_in % 64 == 0, name
    # 8 x 16 patches wherever they pad the map by at most 15 %
    util = d.OH * d.OW / (((d.OW + 15) // 16) * ((d.OH + 7) // 8) * 128.0)
    assert ((c.tile_w, c.tile_h) == (16, 8)) == (util >= 0.85), (name, util)
  for name, d, c in tma:
    assert d.n_tile <= 128 and 2 <= c.stages <= 4, name
    assert c.smem_bytes <= 113 << 10, (name, c.smem_bytes)        # two CTAs per SM at N <= 128
  if cfg in ('coco_tracking', 'coco_pose'):
    assert len(tma) == len(plain) == 29
  # level3's 3x3 128 -> 128 run on this path, not on the halo engine at N = 32
  lv3 = [d for name, d, c in tma if name.startswith('base.level3') and d.KH == 3 and d.stride == 1]
  assert len(lv3) == 7 and all(d.C_in == 128 and d.C_out == 128 for d in lv3)


def _desc(C_in=256, C_out=256, n_tile=256, k=3, stride=1):
  d = L.ConvDesc()
  d.engine, d.dtype, d.a_mode = L.CT_ENGINE_TCGEN05, L.CT_BF16, L.CT_A_CONV
  d.B, d.H, d.W, d.C_in, d.ld_in, d.C_out = 2, 60, 120, C_in, C_in, C_out
  d.KH = d.KW = k
  d.stride, d.pad = stride, k // 2
  d.OH, d.OW = (60 + 2 * (k // 2) - k) // stride + 1, (120 + 2 * (k // 2) - k) // stride + 1
  d.out_mode, d.ld_out, d.n_tile = L.CT_OUT_NHWC, C_out, n_tile
  return d


@pytest.mark.parametrize('n_tile', list(range(16, 257, 16)))
def test_every_n_tile_fits(built_lib, n_tile):
  c = L.conv_config(_desc(n_tile=n_tile))
  assert c is not None and (c.tile_w, c.tile_h) == (16, 8) and c.stages >= 2
  assert c.smem_bytes <= (113 if n_tile <= 128 else 227) << 10


def test_refusal_returns_the_forward_status(built_lib):
  lib = L.lib()
  d = _desc(C_out=40, n_tile=64)
  c = L.ConvConfig()
  rc, msg = lib.ct_conv_config(C.byref(d), C.byref(c)), lib.ct_last_error()
  assert rc == L.CT_ERR_INVALID and b'C_out % 16' in msg, msg
  d.x = d.w = d.out = 1 << 20
  assert (lib.ct_conv_forward(C.byref(d), None), lib.ct_last_error()) == (rc, msg)
