"""The fused head launch (csrc/conv_heads.cu): all heads' 3x3 + ReLU + 1x1 in one launch whose 3x3 result never leaves
the chip.  Its K order and MMA shapes are those of the two-pass plan (CTB_HEAD_FUSE=0: heads.0, then one 1x1 per head),
so the head maps must be bit-identical to it; and the kernel alone against a torch reference of one head."""
import pytest
import torch
import torch.nn.functional as F

from centertrack_b200 import _lib as L

SMEM_PER_CTA = 227 << 10


def _engine(cfg, extra, hw, B, fuse, monkeypatch, device):
  from helpers import make_model
  from centertrack_b200.engine import DLA34Engine
  monkeypatch.setenv('CTB_HEAD_FUSE', '1' if fuse else '0')
  opt, model, _ = make_model(cfg, extra=extra)
  return DLA34Engine(model._engine_state_dict(), model.heads, B, hw[0], hw[1], precision='bf16', device=device,
                     depth_scale=getattr(opt, 'depth_scale', 1.0))


@pytest.mark.parametrize('cfg', ['coco_tracking', 'nuscenes_ddd', 'coco_pose'])
def test_fused_plan_has_one_head_launch(built_lib, cfg, monkeypatch):
  """One 'heads' conv op on the halo engine in place of heads.0 + one 1x1 per head, counted at its exact flops, with a
  launch configuration that fits one CTA per SM."""
  eng = _engine(cfg, [], (512, 512), 32, True, monkeypatch, 'cpu')
  names = [name for _, _, name in eng.ops]
  assert 'heads' in names and 'heads.0' not in names and not set(eng.heads) & set(names)
  (d,) = [d for kind, d, name in eng.ops if name == 'heads']
  assert d.engine == L.CT_ENGINE_TCGEN05_HALO and d.n_heads == len(eng.heads)
  mc = d.C_out // d.n_heads
  assert eng.algo_flops['heads'] == 2.0 * 32 * 128 * 128 * (9 * 64 * d.C_out + mc * sum(eng.heads.values()))
  c = L.conv_config(d)
  assert c is not None and c.smem_bytes <= SMEM_PER_CTA and c.ctas_per_sm == 1 and (c.tile_w, c.tile_h) == (8, 16)
  assert c.stages >= 3
  # the records of the unfused layers it computes (the per-layer audit) come with it
  assert [sp['name'] for sp in eng.specs[-1 - len(eng.heads):]] == ['heads.0'] + list(eng.heads)
  unfused = _engine(cfg, [], (512, 512), 32, False, monkeypatch, 'cpu')
  assert 'heads.0' in [name for _, _, name in unfused.ops]


CASES = [
    ('coco_tracking', [], (64, 96)),
    ('mot', [], (64, 96)),
    ('nuscenes_ddd', [], (64, 96)),
    ('coco_pose', [], (64, 96)),
    ('generic_hc64', ['--arch', 'generic'], (64, 96)),
    ('coco_tracking_partial_tiles', [], (96, 128)),       # 24 x 32 output: the last tile row is half outside
]


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_fused_heads_bit_identical_to_two_pass_plan(case, monkeypatch):
  from centertrack_b200 import synthetic as syn
  name, extra, hw = case
  cfg = 'coco_tracking' if name.startswith(('generic', 'coco_tracking')) else name
  dev = torch.device('cuda')
  fused = _engine(cfg, extra, hw, 2, True, monkeypatch, dev)
  two_pass = _engine(cfg, extra, hw, 2, False, monkeypatch, dev)
  assert 'heads' in [n for _, _, n in fused.ops] and 'heads.0' in [n for _, _, n in two_pass.ops]
  img, pre, hm = (t.to(dev) for t in syn.synthetic_inputs(2, hw[0], hw[1], seed=11))
  for act in (False, True):
    fused.set_fused_activations(act)
    two_pass.set_fused_activations(act)
    a = {k: v.clone() for k, v in fused.forward(img, pre, hm).items()}
    b = two_pass.forward(img, pre, hm)
    torch.cuda.synchronize()
    for h in fused.heads:
      assert torch.equal(a[h], b[h]), '%s: head %s (fused activations %s) differs from the two-pass plan' % (name, h, act)
    fused.in_img.copy_(img); fused.in_pre.copy_(pre); fused.in_hm.copy_(hm)
    g = fused.replay()                                   # the CUDA-graph replay runs the same launch
    torch.cuda.synchronize()
    for h in fused.heads:
      assert torch.equal(g[h], b[h]), '%s: replayed head %s differs' % (name, h)


@pytest.mark.gpu
def test_fused_head_against_torch_reference(monkeypatch):
  """One head (hm, 80 classes) of the fused launch against relu(conv3x3) -> conv1x1 in fp64 on the bf16-rounded
  operands the kernel reads, with the intermediate rounded to bf16 as the kernel rounds it."""
  from centertrack_b200 import synthetic as syn
  dev = torch.device('cuda')
  eng = _engine('coco_tracking', [], (64, 96), 2, True, monkeypatch, dev)
  img, pre, hm = (t.to(dev) for t in syn.synthetic_inputs(2, 64, 96, seed=3))
  out = eng.forward(img, pre, hm)['hm'].double()
  torch.cuda.synchronize()
  feat = eng.named['feat'].tensor().permute(0, 3, 1, 2).double()
  bf = lambda t: t.to(dev).float().bfloat16().double()
  w1, b1 = bf(eng.sd['hm.0.weight']), eng.sd['hm.0.bias'].float().double().to(dev)
  w2, b2 = bf(eng.sd['hm.2.weight']), eng.sd['hm.2.bias'].float().double().to(dev)
  mid = F.relu(F.conv2d(feat, w1, b1, padding=1)).float().bfloat16().double()
  ref = F.conv2d(mid, w2, b2)
  mag = F.conv2d(mid.abs(), w2.abs(), b2.abs())
  err = (out - ref).abs()
  # fp32 accumulation of the 1x1, plus one bf16 step of mid where the fp32 and fp64 3x3 sums round differently
  assert bool((err <= 1e-2 * mag + 1e-4).all()), float((err / (mag + 1e-6)).max())
