"""The launch configurations of the product plans (tests/plan_rows.py) are all audited on the GPU (no GPU needed here).

Every row of every PRODUCT_PLANS plan -- bench.py's configs at their resolutions, bf16 / bf16x3 / fp32, B = 1 ... 64,
built on the CPU with the H100 SXM's 132 SMs -- must be run by a plan of test_gpu_plan_layers.CASES or by an op that
plan_rows.TARGETED names (audited by tests/test_gpu_plan_rows.py).  A planner or library change that makes a product
plan pick a configuration nothing audits fails here, listing the rows and the ops that run them."""
import pytest

import plan_rows as pr


@pytest.fixture(scope='module')
def audit(built_lib):
  from test_gpu_plan_layers import CASES
  return pr.unaudited(CASES, pr.TARGETED)


def test_product_plans_cover_every_bench_config():
  import bench
  assert set(pr.BENCH_SHAPES) == set(bench.CONFIGS)
  for cfg, (H, W) in pr.BENCH_SHAPES.items():
    assert bench.CONFIGS[cfg][:2] == (H, W), cfg
  got = {(cfg, hw, B, p) for _, cfg, hw, B, p in pr.PRODUCT_PLANS}
  assert got == {(cfg, pr.BENCH_SHAPES[cfg], B, p) for cfg in bench.CONFIGS for B in (1, 2, 4, 8, 16, 32, 64)
                 for p in ('bf16', 'bf16x3', 'fp32')}


def test_bench_plans_are_audited_whole():
  """Rows shared by two plans are audited once; the benchmarked plans are audited whole regardless."""
  from test_gpu_plan_layers import CASES
  whole = {pr.plan_id(cfg, hw, B, p) for _, cfg, hw, B, p, extra, kw, env in CASES if not (extra or kw or env)}
  missing = [pid for pid in pr.WHOLE_PLANS if pid not in whole]
  assert not missing, 'no test_gpu_plan_layers.CASES entry audits these product plans whole: %s' % missing


def test_every_product_row_is_audited(audit):
  missing, _ = audit
  assert not missing, '%d launch configurations of the product plans are audited by no CASES plan and no TARGETED ' \
      'op (plan, ops that run it, row):\n  %s' % (len(missing), '\n  '.join(
          '%s  %s  %s' % (pid, ','.join(names), pr.format_row(r)) for pid, r, names in missing))


def test_targeted_ops_exist_and_have_a_checker(audit):
  from test_gpu_plan_layers import OTHER_KINDS
  _, plans = audit
  for pid, names in pr.TARGETED.items():
    assert pid in plans, '%s is not a product plan' % pid
    ran = {n: r for r, ns in plans[pid].items() for n in ns}
    for n in names:
      assert n in ran, '%s: no op %s runs a launch of the plan' % (pid, n)
  for pid, cfg, hw, B, p in pr.PRODUCT_PLANS:
    if pid in pr.TARGETED:
      eng = pr.cpu_plan(cfg, hw, B, p)
      kinds = {sp['name']: sp['kind'] for sp in eng.specs}
      for n in pr.TARGETED[pid]:
        assert kinds[n] == 'conv' or kinds[n] in OTHER_KINDS, (pid, n, kinds[n])


def test_refused_product_plans_say_why(built_lib):
  for pid, cfg, hw, B, p in pr.PRODUCT_PLANS:
    if pid in pr.REFUSED:
      with pytest.raises(RuntimeError, match=pr.REFUSED[pid].replace('^', r'\^')):
        pr.cpu_plan(cfg, hw, B, p)
