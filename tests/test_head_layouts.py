"""The head plan DLA34Engine builds for every output-head layout of tests/helpers.py::HEAD_LAYOUTS (host code, no GPU):
the fused head launch where the eligibility rule allows it (every head = 3x3 64 -> 64 or 256 + ReLU -> 1x1 with at
most 80 channels, at most 12 heads), else heads.0, the hidden 1x1 layers and one 1x1 per head in opt.heads order."""
import pytest

from centertrack_b200 import _lib as L
from helpers import HEAD_LAYOUTS, make_model

SMEM_PER_CTA = 227 << 10


def _engine(cfg, extra, B=32, hw=(512, 512)):
  from centertrack_b200.engine import DLA34Engine
  opt, model, _ = make_model(cfg, extra=extra)
  return opt, DLA34Engine(model._engine_state_dict(), model.heads, B, hw[0], hw[1], precision='bf16', device='cpu',
                          depth_scale=getattr(opt, 'depth_scale', 1.0))


@pytest.mark.parametrize('layout', HEAD_LAYOUTS, ids=[r[0] for r in HEAD_LAYOUTS])
def test_head_layout_builds_its_plan(built_lib, layout):
  _, cfg, extra, plan = layout
  opt, eng = _engine(cfg, extra)
  heads = list(opt.heads)
  head_ops = [(name, d) for kind, d, name in eng.ops if name in ('heads', 'heads.0') or name.split('.')[0] in heads]
  mc = opt.head_conv[heads[0]][0]
  if plan[0] == 'fused':
    _, nh, n2, n_heads = plan
    assert [n for n, _ in head_ops] == ['heads']
    d = head_ops[0][1]
    assert (d.engine, d.KH, d.C_in, d.C_out, d.n_tile, d.n_heads) == (L.CT_ENGINE_TCGEN05_HALO, 3, 64, n_heads * mc, nh,
                                                                      n_heads)
    assert eng.head_names == heads and len(heads) == n_heads
    assert [(d.heads[i].C_out, d.heads[i].n_tile) for i in range(n_heads)] == [(opt.heads[h], n2) for h in heads]
    c = L.conv_config(d)
    assert c is not None and c.smem_bytes <= SMEM_PER_CTA and c.stages >= 3 and c.ctas_per_sm == 1
  else:
    _, k, hidden = plan
    want = ['heads.0']
    for h in heads:
      want += ['%s.%d' % (h, 2 + 2 * j) for j in range(0 if h == 'reg' else hidden)] + [h]
    assert [n for n, _ in head_ops] == want
    descs = dict(head_ops)
    d0 = descs['heads.0']
    assert (d0.KH, d0.KW, d0.C_in, d0.C_out) == (k, k, 64, mc * len(heads))
    for h in heads:
      for j in range(0 if h == 'reg' else hidden):
        d = descs['%s.%d' % (h, 2 + 2 * j)]
        assert (d.KH, d.C_in, d.C_out, d.relu, d.out_mode) == (1, mc, mc, 1, L.CT_OUT_NHWC)
      d = descs[h]
      assert (d.KH, d.C_in, d.C_out, d.relu, d.out_mode) == (1, mc, opt.heads[h], 0, L.CT_OUT_NCHW_F32)
  for name, d in [(n, d) for kind, d, n in eng.ops if kind == 'conv']:
    assert L.conv_config(d) is not None, name


@pytest.mark.parametrize('k', [2, 4])
def test_even_head_kernel_is_refused_at_engine_construction(built_lib, k):
  """padding k // 2 makes an even kernel's head maps one row and column larger than the output grid: no plan."""
  with pytest.raises(ValueError, match='head_kernel must be odd'):
    _engine('coco_tracking', ['--head_kernel', str(k)], B=1, hw=(64, 96))
