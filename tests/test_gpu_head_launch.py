"""-m gpu: the fused head launch (csrc/conv_heads.cu) on every instantiation, through ct_conv_forward on descriptors
and head tables built by hand (gpu_helpers.heads_desc packs them as engine._fused_heads does).

Per case: (a) every head map equals, bit for bit, the two-pass launches on the same operands (halo 3x3 64 ->
n_heads x mid at n_tile NH with ReLU and bf16 NHWC output, then one halo 1x1 per head at its own n_tile with fp32
NCHW output and the same activation); (b) that intermediate is within the bf16 bound (tests/bounds.py) of the fp64
3x3 of the bf16-rounded operands; (c) each head is within ALPHA_BF16 x mag of the fp64 1x1 over that intermediate,
through its activation.  The head maps share one NaN-filled buffer whose guard bands must come back untouched."""
import pytest
import torch

import bounds as bd
from centertrack_b200 import _lib as L

pytestmark = pytest.mark.gpu

ACTS = [L.CT_HEAD_NONE, L.CT_HEAD_SIGMOID, L.CT_HEAD_DEPTH]
ACT_NAME = {L.CT_HEAD_NONE: 'none', L.CT_HEAD_SIGMOID: 'sigmoid', L.CT_HEAD_DEPTH: 'depth'}
DEPTH_SCALE = 2.5

# (NH, N2, n_heads, B, OH, OW, input as channels 64..127 of a 128-channel NHWC buffer)
#   16 x 24 at B = 1: 3 tiles, fewer than SMs;  128 x 128 at B = 4: 512 tiles, several per CTA (ring and halo stages
#   wrap with changing parity);  40 x 44: last tile row half outside (OH % 16 == 8) and a ragged last column;
#   8 x 40: OH < 16
CASES = [
    (128, 16, 12, 1, 16, 24, False),
    (128, 32, 5, 2, 40, 44, True),
    (128, 48, 2, 4, 128, 128, False),
    (128, 64, 1, 2, 8, 40, False),
    (128, 80, 5, 2, 40, 44, False),
    (128, 80, 12, 2, 8, 40, True),
    (64, 16, 5, 4, 128, 128, False),
    (64, 32, 12, 2, 40, 44, False),
    (64, 48, 1, 1, 16, 24, True),
    (64, 64, 2, 2, 8, 40, True),
    (64, 80, 12, 4, 128, 128, False),
    (64, 16, 2, 2, 40, 44, True),
]
RAN = {}


def _case_id(c):
  return 'NH%d_N%d_%dheads_b%d_%dx%d%s' % (c[:6] + ('_slice' if c[6] else '',))


def _c_outs(n2, n):
  """Ragged head widths within one launch: a partly used 16-column group, and at N2 = 48 / 80 a staging chunk whose
  upper half is never stored."""
  return [[n2, 1, min(17, n2 - 7), 2][i % 4] for i in range(n)]


def _two_pass(x, w1, b1, heads, ld_pad, ch_off):
  """heads.0 (bf16 NHWC) and one 1x1 per head, as separate halo launches -> (mid [B, H, W, n_heads x mid], outs)."""
  from gpu_helpers import conv_desc
  keep = []
  d0, mid, bufs = conv_desc(L.CT_ENGINE_TCGEN05_HALO, L.CT_BF16, x, w1, b1, 1, relu=True,
                            n_tile=128 if w1.shape[0] // len(heads) == 256 else 64, ld_pad=ld_pad, ch_off=ch_off)
  keep.append(bufs)
  L.check(L.lib().ct_conv_forward(d0, L.stream_ptr()), 'heads.0')
  mc = w1.shape[0] // len(heads)
  outs = []
  for i, (w2, b2, act) in enumerate(heads):
    d, o, bufs = conv_desc(L.CT_ENGINE_TCGEN05_HALO, L.CT_BF16, mid[..., i * mc:(i + 1) * mc].permute(0, 3, 1, 2), w2,
                           b2, 1, relu=False, out_mode=L.CT_OUT_NCHW_F32, head_act=act)
    d.depth_scale = DEPTH_SCALE
    keep.append(bufs)
    L.check(L.lib().ct_conv_forward(d, L.stream_ptr()), 'head %d' % i)
    outs.append(o)
  torch.cuda.synchronize()
  return mid, outs


@pytest.mark.parametrize('case', CASES, ids=[_case_id(c) for c in CASES])
def test_fused_head_launch(case):
  from gpu_helpers import heads_desc
  nh, n2, n, B, H, W, sliced = case
  mc = 256 if nh == 128 else 64
  g = torch.Generator().manual_seed(1000 + 7 * n2 + n)
  x = torch.randn(B, 64, H, W, generator=g)
  w1 = torch.randn(n * mc, 64, 3, 3, generator=g) * (2.0 / 576) ** 0.5
  b1 = torch.randn(n * mc, generator=g) * 0.1
  heads = [(torch.randn(c, mc, 1, 1, generator=g) * mc ** -0.5, torch.randn(c, generator=g), ACTS[i % 3])
           for i, c in enumerate(_c_outs(n2, n))]
  ld_pad, ch_off = (64, 64) if sliced else (0, 0)
  d, outs, buf, guards, _keep = heads_desc(x, w1, b1, heads, n2, ld_pad, ch_off, DEPTH_SCALE)
  cfg = L.conv_config(d)
  assert cfg is not None and cfg.ctas_per_sm == 1 and cfg.stages >= 3
  L.check(L.lib().ct_conv_forward(d, L.stream_ptr()), 'fused heads')
  torch.cuda.synchronize()
  for i, gs in enumerate(guards):
    assert bool(torch.isnan(buf[gs]).all()), 'guard band %d written (after head %d)' % (i, i - 1)
  mid, two = _two_pass(x, w1, b1, heads, ld_pad, ch_off)
  # (a) bit-identical to the two-pass plan
  for i, (o, t) in enumerate(zip(outs, two)):
    assert torch.equal(o, t), 'head %d (C_out %d, %s): fused != two-pass, %d elements differ' % (
        i, o.shape[1], ACT_NAME[heads[i][2]], int((o != t).sum()))
  # (b) the intermediate against the fp64 3x3 of the bf16-rounded operands
  xq = x.bfloat16().double().cuda()
  w1q = w1.bfloat16().double()
  midd = mid.permute(0, 3, 1, 2).double()
  for i in range(n):                                 # per head: bounds the fp64 temporaries
    ref, mag = bd.conv_ref(xq, w1q[i * mc:(i + 1) * mc], b1[i * mc:(i + 1) * mc], pad=(1, 1, 1, 1))
    bd.assert_bound(midd[:, i * mc:(i + 1) * mc], ref, mag, bd.ALPHA_BF16, True, 'head %d intermediate' % i, 'relu')
  # (c) each head against the fp64 1x1 over that intermediate
  for i, ((w2, b2, act), o) in enumerate(zip(heads, outs)):
    ref, mag = bd.conv_ref(midd[:, i * mc:(i + 1) * mc], w2.bfloat16().double(), b2.float())
    bd.assert_bound(o.double(), ref, mag, bd.ALPHA_BF16, False, 'head %d (C_out %d)' % (i, w2.shape[0]),
                    ACT_NAME[act], DEPTH_SCALE)
  RAN[case] = tuple(sorted(set(w2.shape[0] for w2, _, _ in heads)))


def test_zz_head_launch_coverage():
  """Print which (NH, N2) instantiations and head counts ran; all of them when every case above ran."""
  if not RAN:
    pytest.skip('no fused head launch ran in this session')
  print('\n NH  N2  heads  B  OHxOW    slice  C_out')
  for c in sorted(RAN):
    print('%3d %3d %5d %3d %4dx%-4d %5s  %s' % (c[:6] + (c[6], ','.join(map(str, RAN[c])))))
  if len(RAN) == len(CASES):
    assert {(c[0], c[1]) for c in RAN} == {(nh, n2) for nh in (64, 128) for n2 in (16, 32, 48, 64, 80)}
    assert {1, 12} <= {c[2] for c in RAN}
