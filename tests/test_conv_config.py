"""ct_conv_config (host code, no GPU): the launch configuration of every conv of the shipped plans, its refusals, and
the halo engine's choice of the overlapped one-CTA-per-SM flavour."""
import ctypes as C

import pytest

from centertrack_b200 import _lib as L

SMEM_PER_CTA = 227 << 10          # the dynamic shared memory one CTA can opt in to on an H100 (sm_90)

PLANS = {'coco_tracking': (512, 512), 'mot': (544, 960), 'nuscenes_ddd': (448, 800), 'coco_pose': (512, 512)}


@pytest.mark.parametrize('B', [1, 32])
@pytest.mark.parametrize('precision', ['bf16', 'bf16x3', 'fp32'])
@pytest.mark.parametrize('cfg', sorted(PLANS))
def test_shipped_plan_convs_have_a_configuration(built_lib, cfg, precision, B):
  from helpers import make_model
  from centertrack_b200.engine import DLA34Engine
  opt, model, _ = make_model(cfg)
  H, W = PLANS[cfg]
  eng = DLA34Engine(model._engine_state_dict(), model.heads, B, H, W, precision=precision, device='cpu',
                    depth_scale=getattr(opt, 'depth_scale', 1.0))
  convs = [(name, d) for kind, d, name in eng.ops if kind == 'conv']
  assert convs
  for name, d in convs:
    c = L.conv_config(d)
    assert c is not None, name
    assert 0 <= c.smem_bytes <= SMEM_PER_CTA, (name, c.smem_bytes)
    if d.engine == L.CT_ENGINE_SIMT:
      assert (c.smem_bytes, c.stages, c.tile_w, c.tile_h, c.ctas_per_sm, c.overlap) == (0, 0, 0, 0, 0, 0), name
    elif d.engine == L.CT_ENGINE_TCGEN05_HALO:
      assert c.stages >= 2 and (c.tile_w, c.tile_h) in ((8, 16), (32, 4)) and c.ctas_per_sm in (1, 2), name
    else:
      assert c.smem_bytes > 0 and c.stages >= 1 and (c.tile_w, c.tile_h) in ((128, 1), (16, 8)), name
      assert c.ctas_per_sm == 0 and c.overlap == 0, name


def _desc(engine=L.CT_ENGINE_TCGEN05_HALO, C_in=64, C_out=64, k=3, n_tile=64, stride=1, H=64, W=64):
  """A plain convolution with NHWC output and no pointers (fp32 activations on the SIMT and x3 engines)."""
  d = L.ConvDesc()
  d.engine, d.dtype, d.a_mode = engine, L.CT_F32 if engine in (L.CT_ENGINE_SIMT, L.CT_ENGINE_TCGEN05_X3) else L.CT_BF16, 0
  d.B, d.H, d.W, d.C_in, d.ld_in, d.C_out = 1, H, W, C_in, C_in, C_out
  d.KH = d.KW = k
  d.stride, d.pad = stride, k // 2
  d.OH, d.OW = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
  d.out_mode, d.ld_out, d.n_tile = L.CT_OUT_NHWC, C_out, n_tile
  return d


def _config(d):
  lib = L.lib()
  c = L.ConvConfig()
  return lib.ct_conv_config(C.byref(d), C.byref(c)), lib.ct_last_error(), c


def _forward(d):
  """ct_conv_forward on 16-byte aligned stand-in pointers: only for descriptors it refuses before any CUDA call."""
  lib = L.lib()
  d.x = d.w = d.out = 1 << 20
  return lib.ct_conv_forward(C.byref(d), None), lib.ct_last_error()


def test_oversized_halo_tile_is_unsupported(built_lib):
  # 3x3 256 -> 256 at N = 128: 144 K blocks of weights (576 KB) per CTA
  rc, msg, _ = _config(_desc(C_in=256, C_out=256, n_tile=128))
  assert rc == L.CT_ERR_UNSUPPORTED and b'shared memory' in msg, msg
  assert _forward(_desc(C_in=256, C_out=256, n_tile=128)) == (rc, msg)
  assert L.conv_config(_desc(C_in=256, C_out=256, n_tile=128)) is None


BAD = [
    ('halo stride 2', dict(stride=2), b"stride-1 'same'"),
    ('halo C_in 40', dict(C_in=40), b'C_in must be'),
    ('halo n_tile 0', dict(n_tile=0), b'bad n_tile'),
    ('halo n_tile 24', dict(n_tile=24), b'bad n_tile'),
    ('gather C_in 12', dict(engine=L.CT_ENGINE_TCGEN05, C_in=12), b'multiples of 8'),
    ('gather n_tile 0', dict(engine=L.CT_ENGINE_TCGEN05, n_tile=0), b'n_tile must be'),
    ('gather C_out 40', dict(engine=L.CT_ENGINE_TCGEN05, C_out=40), b'C_out % 16'),
    ('x3 C_in 12', dict(engine=L.CT_ENGINE_TCGEN05_X3, C_in=12), b'multiples of 8'),
    ('simt C_in 8', dict(engine=L.CT_ENGINE_SIMT, C_in=8), b'multiple of 16'),
    ('unknown engine', dict(engine=7), b'unknown engine'),
]


@pytest.mark.parametrize('case', BAD, ids=[b[0] for b in BAD])
def test_bad_shapes_get_the_status_and_message_of_ct_conv_forward(built_lib, case):
  _, kw, what = case
  rc, msg, _ = _config(_desc(**kw))
  assert rc == L.CT_ERR_INVALID and what in msg, msg
  assert _forward(_desc(**kw)) == (rc, msg)


def test_inconsistent_output_size_is_invalid(built_lib):
  d = _desc(engine=L.CT_ENGINE_TCGEN05)
  d.OH += 1
  rc, msg, _ = _config(d)
  assert rc == L.CT_ERR_INVALID and b'OH inconsistent' in msg, msg
  assert _forward(d) == (rc, msg)


OVERLAP = [
    # (C_in, N, CTAs per SM, overlap): 3x3 halo convolutions
    (128, 32, 1, 0),     # one CTA per SM, but one m64n32 chain alone leaves the tensor pipe half idle
    (64, 64, 1, 1),      # one CTA per SM: the two warpgroups take turns
    (32, 64, 2, 0),      # two CTAs per SM: the other CTA's MMAs fill this one's epilogue
]


@pytest.mark.parametrize('case', OVERLAP, ids=['C_in%d_N%d' % c[:2] for c in OVERLAP])
def test_halo_overlap_rule(built_lib, case):
  C_in, n, ctas, overlap = case
  c = L.conv_config(_desc(C_in=C_in, C_out=n, n_tile=n))
  assert (c.ctas_per_sm, c.overlap) == (ctas, overlap)
