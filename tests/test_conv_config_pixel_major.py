"""ct_conv_config (host code, no GPU): which halo launches take the pixel-major flavour (weights on wgmma M, the item's
128 pixels on N).  Exactly the 64 -> 64-channel layers at n_tile 64 with NHWC bf16 output: level0, level2's four
convolutions, its project and its root, in every benchmarked plan; every other launch reports 0."""
import pytest

from centertrack_b200 import _lib as L

PLANS = {'coco_tracking': (512, 512), 'mot': (544, 960), 'nuscenes_ddd': (448, 800), 'coco_pose': (512, 512)}
LEVEL2 = ['base.level2.project', 'base.level2.tree1.conv1', 'base.level2.tree1', 'base.level2.tree2.conv1',
          'base.level2.tree2', 'base.level2']


@pytest.mark.parametrize('B', [1, 32])
@pytest.mark.parametrize('cfg', sorted(PLANS))
def test_pixel_major_is_the_64_channel_halo_layers(built_lib, cfg, B):
  from helpers import make_model
  from centertrack_b200.engine import DLA34Engine
  opt, model, _ = make_model(cfg)
  H, W = PLANS[cfg]
  eng = DLA34Engine(model._engine_state_dict(), model.heads, B, H, W, precision='bf16', device='cpu',
                    depth_scale=getattr(opt, 'depth_scale', 1.0))
  got = set()
  for kind, d, name in eng.ops:
    if kind != 'conv':
      continue
    c = L.conv_config(d)
    want = d.engine == L.CT_ENGINE_TCGEN05_HALO and d.n_heads == 0 and d.n_tile == 64 and d.C_out == 64
    assert c.pixel_major == int(want), name
    if c.pixel_major:
      got.add(name)
      # level0 and level2's 3x3 / 2x2 layers run one CTA per SM, whose two warpgroups take turns on the tensor cores
      assert (c.ctas_per_sm, c.overlap) == ((2, 0) if d.KH == 1 else (1, 1)), name
  assert got == set(['base.level0'] + LEVEL2)


def test_pixel_major_needs_a_compiled_walk(built_lib):
  from test_conv_config import _desc
  assert L.conv_config(_desc(C_in=64, C_out=64, n_tile=64)).pixel_major == 1
  assert L.conv_config(_desc(C_in=16, C_out=64, n_tile=64)).pixel_major == 0      # no walk for 3x3 16 -> 64
  assert L.conv_config(_desc(C_in=64, C_out=128, n_tile=64)).pixel_major == 0     # two n tiles
  assert L.conv_config(_desc(C_in=64, C_out=64, n_tile=32)).pixel_major == 0
