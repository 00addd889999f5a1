"""The launch configurations of the product plans (tests/plan_rows.py) are all audited on the GPU (no GPU needed here).

Every row of every PRODUCT_PLANS plan -- bench.py's configs at their resolutions and the product's other input sizes
(plan_rows.PRODUCT_SHAPES), bf16 / bf16x3 / fp32, B = 1 ... 64, built on the CPU with the H100 SXM's 132 SMs -- must be run by a plan of test_gpu_plan_layers.CASES or by an op that
plan_rows.TARGETED names (audited by tests/test_gpu_plan_rows.py).  A planner or library change that makes a product
plan pick a configuration nothing audits fails here, listing the rows and the ops that run them.  Likewise every row
with an operand of >= 2^31 bytes must have its largest launch named in plan_rows.EXTENT_TARGETED, which
tests/test_gpu_plan_rows.py runs at full size."""
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
  got = {(cfg, hw, B, p) for _, cfg, hw, B, p, extra in pr.PRODUCT_PLANS if hw == pr.BENCH_SHAPES[cfg] and not extra}
  assert got == {(cfg, pr.BENCH_SHAPES[cfg], B, p) for cfg in bench.CONFIGS for B in (1, 2, 4, 8, 16, 32, 64)
                 for p in ('bf16', 'bf16x3', 'fp32')}
  assert len({pid for pid, _, _, _, _, _ in pr.PRODUCT_PLANS}) == len(pr.PRODUCT_PLANS)


def test_product_plans_cover_the_product_shapes():
  """The sizes beyond the bench: the large cameras under --keep_res, KITTI's default and --keep_res sizes, VGA, a wide
  strip and the smallest input, each at every precision and at least at the batches up to 16."""
  got = {(cfg, hw, tuple(extra), B, p) for _, cfg, hw, B, p, extra in pr.PRODUCT_PLANS}
  want = {('mot', (1088, 1920), ()), ('nuscenes_ddd', (928, 1632), ()),
          ('coco_tracking', (384, 1280), ('--num_classes', '3')), ('coco_tracking', (384, 1248), ('--num_classes', '3')),
          ('coco_tracking', (480, 640), ()), ('coco_tracking', (64, 1024), ()), ('coco_tracking', (32, 64), ())}
  assert {(cfg, hw, tuple(extra)) for _, cfg, hw, extra, _ in pr.PRODUCT_SHAPES} == want
  for cfg, hw, extra in want:
    for B in (1, 2, 4, 8, 16):
      for p in ('bf16', 'bf16x3', 'fp32'):
        assert (cfg, hw, extra, B, p) in got, (cfg, hw, extra, B, p)


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


@pytest.fixture(scope='module')
def large(built_lib):
  return pr.large_launches()


def test_every_large_launch_is_audited_at_its_size(large):
  """The op with the largest operand of every row that reaches 2^31 bytes runs, at its plan's batch, in
  tests/test_gpu_plan_rows.py: a planner change that makes a bigger launch fails here until EXTENT_TARGETED names it."""
  missing = pr.extent_unaudited(pr.EXTENT_TARGETED, large)
  assert not missing, '%d launches with an operand of >= 2^31 bytes are audited at no batch that large; add to ' \
      'plan_rows.EXTENT_TARGETED (plan, op, its largest operand, row):\n  %s' % (len(missing), '\n  '.join(
          '%s  %s  %s %d elements, %.2f GB  %s' % (pid, name, k, n, nbytes / 1e9, pr.format_row(r))
          for r, (pid, name, nbytes, n, k) in missing))


def test_extent_targeted_ops_are_the_largest_conv_launches(large):
  """No stale entry: each EXTENT_TARGETED op is the largest launch of its row, and a convolution (which the GPU test
  slices by images)."""
  want = {(pid, name) for pid, name, _, _, _ in large.values()}
  for pid, names in pr.EXTENT_TARGETED.items():
    for n in names:
      assert (pid, n) in want, '%s: %s is not the largest launch of a row with an operand of >= 2^31 bytes' % (pid, n)
  for r in large:
    assert r[0] in ('simt', 'gather', 'gather_x3', 'halo'), r


def test_extent_bench_ops_are_large_bench_launches(large):
  """Each EXTENT_BENCH op is a convolution of a benchmarked config's plan with an operand of >= 2^31 bytes, in a row
  whose largest launch EXTENT_TARGETED names in another plan."""
  plans = {pid: (cfg, hw, B, p, extra) for pid, cfg, hw, B, p, extra in pr.PRODUCT_PLANS}
  assert not set(pr.EXTENT_BENCH) & set(pr.EXTENT_TARGETED)
  for pid, names in pr.EXTENT_BENCH.items():
    cfg, hw, B, p, extra = plans[pid]
    assert hw == pr.BENCH_SHAPES[cfg] and not extra, pid
    eng = pr.cpu_plan(cfg, hw, B, p, extra)
    rows = {sp['name']: pr.launch_row(eng, sp) for sp in eng.specs}
    ext = pr.op_extents(eng)
    for n in names:
      assert pr.largest_operand(ext[n])[0] >= pr.LARGE, (pid, n)
      assert rows[n] in large and large[rows[n]][0] != pid, (pid, n, pr.format_row(rows[n]))
    del eng


def test_op_extents_count_whole_buffers(built_lib):
  """A channel slice counts its whole NHWC buffer (ld, not C); the fp32 head planes B C_out OH OW; the fused head
  launch's records are left out."""
  eng = pr.cpu_plan('mot', pr.BENCH_SHAPES['mot'], 2, 'bf16x3')
  ext = pr.op_extents(eng)
  H, W = pr.BENCH_SHAPES['mot']
  px4, px8 = (H // 4) * (W // 4), (H // 8) * (W // 8)
  mid = 256 * len(eng.heads)                            # the heads' fp32 intermediate; hm reads channels 0 .. 255
  assert ext['hm']['x'] == (2 * px4 * mid, 2 * px4 * mid * 4)
  assert ext['hm']['out'] == (2 * eng.heads['hm'] * px4, 2 * eng.heads['hm'] * px4 * 4)
  assert ext['base.level3.tree1']['x'] == (2 * px8 * 256, 2 * px8 * 256 * 4)      # level3.tree1's [x2 | x1] buffer
  assert ext['base.level3.tree1']['out'][0] == 2 * px8 * (3 * 128 + 64)           # a slice of level3's root input
  fused = pr.op_extents(pr.cpu_plan('mot', pr.BENCH_SHAPES['mot'], 2, 'bf16'))
  assert 'heads.0' not in fused and 'hm' not in fused and 'base.level0' in fused


def test_targeted_ops_exist_and_have_a_checker(audit):
  from test_gpu_plan_layers import OTHER_KINDS
  _, plans = audit
  for pid, names in pr.TARGETED.items():
    assert pid in plans, '%s is not a product plan' % pid
    ran = {n: r for r, ns in plans[pid].items() for n in ns}
    for n in names:
      assert n in ran, '%s: no op %s runs a launch of the plan' % (pid, n)
  for pid, cfg, hw, B, p, extra in pr.PRODUCT_PLANS:
    if pid in pr.TARGETED:
      eng = pr.cpu_plan(cfg, hw, B, p, extra)
      kinds = {sp['name']: sp['kind'] for sp in eng.specs}
      for n in pr.TARGETED[pid]:
        assert kinds[n] == 'conv' or kinds[n] in OTHER_KINDS, (pid, n, kinds[n])


def test_refused_product_plans_say_why(built_lib):
  for pid, cfg, hw, B, p, extra in pr.PRODUCT_PLANS:
    if pid in pr.REFUSED:
      with pytest.raises(RuntimeError, match=pr.REFUSED[pid].replace('^', r'\^')):
        pr.cpu_plan(cfg, hw, B, p, extra)
