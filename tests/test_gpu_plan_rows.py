"""-m gpu: the launch configurations of the product plans that no test_gpu_plan_layers.CASES plan runs, audited op by op,
and the batch-prefix runs (engine.forward(..., n)) of the benchmarked mot plan against its full-batch run.

plan_rows.TARGETED names, per product plan, the ops that run a configuration nothing else audits (tests/plan_rows.py);
each plan is built as the product builds it, replayed once on synthetic_inputs, and only those ops are recomputed in fp64
and held to the bounds of tests/bounds.py, as test_gpu_plan_layers does for whole plans."""
import pytest
import torch

import bounds as bd
import plan_rows as pr
import test_gpu_plan_layers as tpl
from centertrack_b200.engine import DeferredTV

pytestmark = pytest.mark.gpu

PLANS = {pid: (cfg, hw, B, p) for pid, cfg, hw, B, p in pr.PRODUCT_PLANS}


@pytest.mark.parametrize('pid', sorted(pr.TARGETED))
def test_targeted_ops_within_bounds(pid, monkeypatch):
  cfg, hw, B, precision = PLANS[pid]
  eng = tpl._build(cfg, hw, B, precision, [], {}, monkeypatch, {})
  tpl._assert_no_overlapping_writes(eng)
  specs = {sp['name']: sp for sp in eng.specs}
  failures, report = [], []
  for name in pr.TARGETED[pid]:
    sp = specs[name]
    row = pr.format_row(pr.launch_row(eng, sp))
    worst, where, use = 0.0, None, 0.0
    for b0 in range(0, eng.B, tpl.CHUNK):
      bs = slice(b0, min(eng.B, b0 + tpl.CHUNK))
      res = tpl._check_conv(eng, sp, bs) if sp['kind'] == 'conv' else tpl._check_other(eng, sp, bs)
      if res is None:
        continue
      m, at = bd.worst(res[0])
      if where is None or m > worst:
        worst, where = m, dict(at, b=at['b'] + b0)
      if res[1] is not None:
        use = max(use, float(res[1].max()))
      del res
    coef = tpl.COEF[tpl.KERNEL[sp['engine']]] if sp['kind'] == 'conv' else bd.ALPHA_BF16 if precision == 'bf16' \
        else bd.GAMMA_SIMT
    report.append('  %-34s %.3f  %.3f  %s' % (name, worst, use / coef, row))
    if not worst <= 1.0:
      failures.append('%s: op %s (row %s): worst element %s, |err| / bound = %.3g' % (pid, name, row, where, worst))
  print('\n[%s] per audited op: worst |err| / bound, largest |err| / mag beyond the output rounding as a multiple of '
        'its constant, row\n%s' % (pid, '\n'.join(report)))
  assert not failures, '\n'.join(failures)


def _written_buffers(eng):
  """{data_ptr: (buffer, [op names writing it])} of every buffer a launch of the plan writes (channel slices by their
  whole buffer; the fused head launch's intermediate never exists and is left out)."""
  bufs = {}
  for sp in eng.specs:
    o = sp['out']
    if isinstance(o, DeferredTV):
      continue
    t = o.buf if hasattr(o, 'buf') else o
    bufs.setdefault(t.data_ptr(), (t, []))[1].append(sp['name'])
  return bufs


def test_batch_prefix_matches_full_batch_at_bench_shape():
  """mot 544x960 bf16 at B = 32 replayed once; then forward(n) on the first n images: every op's output on those images
  equals the full-batch run bit for bit (fused heads and space-to-depth buffers included), and not one byte of the other
  images changes -- they are filled with 0xff (a NaN in bf16 and fp32) before the run, inputs included, so a launch that
  read them would also spoil the first n."""
  from helpers import make_model
  from centertrack_b200 import synthetic as syn
  B, (H, W) = 32, pr.BENCH_SHAPES['mot']
  _, model, _ = make_model('mot')
  dev = torch.device('cuda')
  eng = model.to(dev).engine_for(B, H, W, dev, 'bf16')
  img, pre, hm = syn.synthetic_inputs(B, H, W)
  eng.in_img.copy_(img)
  eng.in_pre.copy_(pre)
  eng.in_hm.copy_(hm)
  eng.set_fused_activations(True)
  eng.replay()
  torch.cuda.synchronize()
  bufs = _written_buffers(eng)
  assert any(n == 'heads' for _, _, n in eng.ops) and eng.s2d_named, 'the plan has fused heads and s2d buffers'
  full = {p: t.clone() for p, (t, _) in bufs.items()}
  inputs = (eng.in_img, eng.in_pre, eng.in_hm)
  for n in (1, 13, 31):
    for p, (t, _) in bufs.items():
      t.copy_(full[p])
      t[n:].view(torch.uint8).fill_(0xff)
    for t, src in zip(inputs, (img, pre, hm)):
      t.copy_(src)
      t[n:].view(torch.uint8).fill_(0xff)
    eng.forward(eng.in_img[:n], eng.in_pre[:n], eng.in_hm[:n], n=n)
    torch.cuda.synchronize()
    bad = []
    for p, (t, names) in bufs.items():
      if not torch.equal(t[:n].view(torch.uint8), full[p][:n].view(torch.uint8)):
        diff = (t[:n].view(torch.uint8) != full[p][:n].view(torch.uint8)).reshape(n, -1).any(1)
        bad.append('%s: images %s differ from the B = %d run' % (','.join(names), diff.nonzero().flatten().tolist()[:8], B))
      if not bool((t[n:].view(torch.uint8) == 0xff).all()):
        hit = (t[n:].view(torch.uint8) != 0xff).reshape(B - n, -1).any(1)
        bad.append('%s: bytes of images %s written' % (','.join(names), (hit.nonzero().flatten() + n).tolist()[:8]))
    assert not bad, 'forward(n=%d) on the B = %d plan:\n  %s' % (n, B, '\n  '.join(bad))
