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


# The gather engines' 32-bit element offsets: B H W ld_in < 2^31.  2^31 - 8 = 120 x 1247 x 113 x 127, the largest
# input a multiple of 8 channels wide can have (tests/test_gpu_conv.py runs a launch of that size).
EDGE_ACCEPTED = dict(B=1247, H=113, W=127, ld_in=120)
EDGE_REFUSED = dict(B=4096, H=64, W=64, ld_in=128)


@pytest.mark.parametrize('engine', [L.CT_ENGINE_TCGEN05, L.CT_ENGINE_TCGEN05_X3], ids=['bf16', 'x3'])
@pytest.mark.parametrize('k', [1, 3])
def test_gather_input_size_limit(built_lib, engine, k):
  for shape, n in ((EDGE_ACCEPTED, (1 << 31) - 8), (EDGE_REFUSED, 1 << 31)):
    d = _desc(engine=engine, C_in=40, C_out=16, k=k, n_tile=16, H=shape['H'], W=shape['W'])
    d.B, d.ld_in = shape['B'], shape['ld_in']
    assert d.B * d.H * d.W * d.ld_in == n
    rc, msg, _ = _config(d)
    if n < 1 << 31:
      assert rc == L.CT_OK, msg
    else:
      assert rc == L.CT_ERR_INVALID and b'input tensor exceeds 2^31 elements' in msg, msg
      assert _forward(d) == (rc, msg)


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


# ---- the fused head launch (csrc/conv_heads.cu): a halo descriptor with a head table ----------------------------------
def _heads_desc(mid=256, n_heads=4, nh=None, n2=80, c_outs=None):
  """heads.0 (3x3 64 -> n_heads x mid at n_tile nh) with a table of n_heads heads at the common 1x1 n_tile n2, no
  pointers but the table (which the descriptor keeps alive)."""
  d = _desc(C_in=64, C_out=n_heads * mid, n_tile=nh or (128 if mid == 256 else 64))
  d.out_mode, d.ld_out, d.relu = L.CT_OUT_NCHW_F32, 0, 1
  c_outs = c_outs or [n2] * n_heads
  table = (L.Head * max(1, len(c_outs)))()
  for t, c in zip(table, c_outs):
    t.C_out, t.n_tile = c, n2
  d.n_heads, d.heads = n_heads, C.cast(table, C.POINTER(L.Head))
  d._table = table
  return d


@pytest.mark.parametrize('n2', [16, 32, 48, 64, 80])
@pytest.mark.parametrize('mid', [64, 256])
def test_fused_heads_configuration_on_every_instantiation(built_lib, mid, n2):
  for n_heads in (1, 12):
    c = L.conv_config(_heads_desc(mid, n_heads, n2=n2, c_outs=[1, n2, n2 - 7, 2][:n_heads] + [n2] * (n_heads - 4)))
    assert c is not None and c.smem_bytes <= SMEM_PER_CTA and c.stages >= 3, (mid, n2, n_heads)
    assert (c.tile_w, c.tile_h, c.ctas_per_sm, c.overlap) == (8, 16, 1, 0), (mid, n2, n_heads)


def _set(**kw):
  def f(d):
    for k, v in kw.items():
      setattr(d, k, v)
  return f


def _head(i, **kw):
  def f(d):
    for k, v in kw.items():
      setattr(d.heads[i], k, v)
  return f


HEADS_BAD = [
    ('n_heads -1', _set(n_heads=-1), b'1 .. 12 heads'),
    ('n_heads 13', lambda d: setattr(d, 'n_heads', 13) or setattr(d, 'C_out', 13 * 256), b'1 .. 12 heads'),
    ('null table', _set(heads=C.POINTER(L.Head)()), b'1 .. 12 heads'),
    ('mid 128', _set(C_out=4 * 128), b'64 or 256 mid channels'),
    ('C_out not a multiple of n_heads', _set(C_out=4 * 256 + 2), b'64 or 256 mid channels'),
    ('n_tile 64 for mid 256', _set(n_tile=64), b'n_tile must be 128'),
    ('n_tile 128 for mid 64', lambda d: setattr(d, 'C_out', 4 * 64), b'n_tile must be 128'),
    ('different 1x1 n_tiles', _head(2, n_tile=64), b'one n_tile for every head'),
    ('C_out > n_tile', _head(1, C_out=81), b'one n_tile for every head'),
    ('C_out 0', _head(3, C_out=0), b'one n_tile for every head'),
    ('n_tile 96', lambda d: [setattr(d.heads[i], 'n_tile', 96) for i in range(4)], b'one n_tile for every head'),
    ('n_tile 40', lambda d: [setattr(d.heads[i], 'n_tile', 40) or setattr(d.heads[i], 'C_out', 40) for i in range(4)],
     b'one n_tile for every head'),
    ('NHWC output', _set(out_mode=L.CT_OUT_NHWC, ld_out=1024), b'fp32 NCHW outputs'),
    ('no ReLU', _set(relu=0), b'fp32 NCHW outputs'),
    ('residual', _set(residual=1 << 20, ld_res=1024), b'fp32 NCHW outputs'),
    ('epilogue_sum3', _set(epilogue_sum3=1), b'fp32 NCHW outputs'),
    ('C_in 32', _set(C_in=32, ld_in=32), b'C_in must be 64'),
    ('1x1 kernel', _set(KH=1, KW=1, pad=0), b"3x3 stride-1 'same'"),
    ('stride 2', _set(stride=2, OH=32, OW=32), b"3x3 stride-1 'same'"),
]


@pytest.mark.parametrize('case', HEADS_BAD, ids=[b[0] for b in HEADS_BAD])
def test_fused_heads_refusals_get_the_status_and_message_of_ct_conv_forward(built_lib, case):
  _, edit, what = case
  d = _heads_desc()
  edit(d)
  rc, msg, _ = _config(d)
  assert rc == L.CT_ERR_INVALID and what in msg, msg
  assert _forward(d) == (rc, msg)


def _forward_heads(d, **ptrs):
  """ct_conv_forward of a valid head descriptor on stand-in pointers (16-byte aligned unless given): it must refuse
  before any CUDA call."""
  lib = L.lib()
  d.x = d.w = d.shift = 1 << 20
  for i in range(d.n_heads):
    d.heads[i].w = d.heads[i].bias = d.heads[i].out = 1 << 20
  for k, v in ptrs.items():
    if k.startswith('head_'):
      setattr(d.heads[1], k[5:], v)
    else:
      setattr(d, k, v)
  return lib.ct_conv_forward(C.byref(d), None), lib.ct_last_error()


@pytest.mark.parametrize('ptrs,what', [
    (dict(head_w=(1 << 20) + 8), b'every head needs 16-byte aligned w'),
    (dict(head_w=0), b'every head needs 16-byte aligned w'),
    (dict(head_bias=0), b'every head needs 16-byte aligned w'),
    (dict(head_out=0), b'every head needs 16-byte aligned w'),
    (dict(x=(1 << 20) + 2), b'x / w must be 16-byte aligned'),
    (dict(w=(1 << 20) + 4), b'x / w must be 16-byte aligned'),
    (dict(shift=0), b'x / w must be 16-byte aligned'),
], ids=['misaligned_head_w', 'null_head_w', 'null_head_bias', 'null_head_out', 'misaligned_x', 'misaligned_w',
        'null_shift'])
def test_fused_heads_pointer_checks_refuse_before_any_cuda_call(built_lib, ptrs, what):
  rc, msg = _forward_heads(_heads_desc(), **ptrs)
  assert rc == L.CT_ERR_INVALID and what in msg, msg
  if next(iter(ptrs)).startswith('head_'):
    assert b'(head 1)' in msg, msg


def test_fused_heads_need_n_heads_to_route_to_the_head_launch(built_lib):
  """n_heads = 0 is a plain halo convolution: with the head table but no output it is refused as a null pointer."""
  d = _heads_desc()
  d.n_heads = 0
  lib = L.lib()
  d.x = d.w = d.shift = 1 << 20
  assert lib.ct_conv_forward(C.byref(d), None) == L.CT_ERR_INVALID and b'null pointer' in lib.ct_last_error()
