"""Launch configuration rows of the shipped plans (test infrastructure; builds plans on the CPU, needs no GPU).

A row is what decides which kernel instantiation runs an op and how its work is laid out:
  * conv launches: (kernel, N tile, C_in, k, stride, a_mode, out_mode, residual, s2d, sum3, tile, stages, overlap, work),
    where `work` says whether a CTA of a persistent kernel (the gather engine's TMA path, the halo engine) takes one work
    item ('one') or strides over several ('several'), computed from ct_conv_config and the grid rule of its forward;
    '-' for the grid-per-tile kernels;
  * the fused head launch (csrc/conv_heads.cu): ('heads', mid channels per pass, 1x1 n_tile, heads, C_in, tile, stages,
    work), run by the 1x1 records of its heads;
  * up (ct_upsample_add): ('up', dtype, C, f), which picks the variant;
  * the other ops: (kind, dtype).
The row depends on the batch and the SM count (n_sm = 132 on the CPU, the H100 SXM's count), so one layer runs other
kernels at other batches.  tests/test_plan_rows.py checks that every row of every PRODUCT_PLANS plan is audited by a
test_gpu_plan_layers.CASES plan or by an op named in TARGETED; tests/test_gpu_plan_rows.py audits the TARGETED ops.

A row says nothing about the size of the tensors, and the engines index memory with 32-bit offsets, guarded by host
checks (the gather engines refuse an input of 2^31 elements).  So for every row that has an operand of at least 2^31
bytes in some product plan, the op with the largest operand in that row (op_extents) must be named in EXTENT_TARGETED;
tests/test_gpu_plan_rows.py runs those at their full batch and compares every image with the same launch on 4-image
slices.

`python tests/plan_rows.py` prints the rows no audit reaches and the TARGETED entries that would cover them, then the
same for the large launches and EXTENT_TARGETED.
"""
import contextlib
import os
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (os.path.dirname(_HERE), os.path.join(os.path.dirname(_HERE), 'oracle'), _HERE):
  if _p not in sys.path:
    sys.path.insert(0, _p)

from centertrack_b200 import _lib as L   # noqa: E402

KERNEL = {L.CT_ENGINE_SIMT: 'simt', L.CT_ENGINE_TCGEN05: 'gather', L.CT_ENGINE_TCGEN05_X3: 'gather_x3',
          L.CT_ENGINE_TCGEN05_HALO: 'halo'}
A_MODE = {L.CT_A_CONV: 'conv', L.CT_A_DCN: 'dcn', L.CT_A_DCN_WIN: 'dcn_win'}
OUT_MODE = {L.CT_OUT_NHWC: 'nhwc', L.CT_OUT_NHWC_F32: 'nhwc_f32', L.CT_OUT_NCHW_F32: 'nchw_f32',
            L.CT_OUT_NHWC_S2D: 'nhwc_s2d'}

# bench.py's --config resolutions, every precision it takes, and the batches a StreamRunner is commonly built at
BENCH_SHAPES = {'coco_tracking': (512, 512), 'mot': (544, 960), 'nuscenes_ddd': (448, 800), 'coco_pose': (512, 512)}
PRECISIONS = ('bf16', 'bf16x3', 'fp32')
BATCHES = (1, 2, 4, 8, 16, 32, 64)
# the --keep_res sizes of the large cameras stop at B = 16: from B = 32 on, bf16x3 is refused (an input past 2^31
# elements) and the fp32 plans alone hold 60 GB (928 x 1632) and 65 GB (1088 x 1920) of buffers at B = 32, 120 and
# 131 GB at B = 64, so that neither they nor the full-size audit of their largest launches (tests/test_gpu_plan_rows.py)
# fit an 80 GB H100
KEEP_BATCHES = (1, 2, 4, 8, 16)

# input sizes the product builds plans at beyond the bench: (name, config, (H, W), extra options, batches).  --keep_res
# pads each camera's frame up to a multiple of 32 (detector.frame_geometry), a StreamRunner stream can switch to such a
# camera at a video start, and --input_h / --input_w / --input_res / --fix_short take any multiple of 32.  The name
# starts the plan id: the config's, or the dataset's where the options change the model.  Map-size-dependent choices
# (TMA or register gather, N tile, halo stages, work items per persistent CTA) differ from the bench sizes', and the
# partial edge patches, TMA boxes overhanging the map and the upsample's grid-stride carries depend on H and W.
PRODUCT_SHAPES = [
    ('mot', 'mot', (1088, 1920), [], KEEP_BATCHES),                   # a 1080p camera under --keep_res
    ('nuscenes_ddd', 'nuscenes_ddd', (928, 1632), [], KEEP_BATCHES),  # nuScenes' 900 x 1600 under --keep_res
    ('kitti_tracking', 'coco_tracking', (384, 1280), ['--num_classes', '3'], BATCHES),  # kitti(_tracking)'s default
    ('kitti_tracking', 'coco_tracking', (384, 1248), ['--num_classes', '3'], BATCHES),  # KITTI's 375 x 1242, --keep_res
    ('coco_tracking', 'coco_tracking', (480, 640), [], BATCHES),      # a VGA camera under --keep_res
    ('coco_tracking', 'coco_tracking', (64, 1024), [], BATCHES),      # a wide strip: level 5 is 2 x 32
    ('coco_tracking', 'coco_tracking', (32, 64), [], BATCHES),        # the smallest input: level 5 is 1 x 2
]


def plan_id(cfg, hw, B, precision):
  return '%s_%dx%d_b%d_%s' % (cfg, hw[0], hw[1], B, precision)


# (id, config, (H, W), B, precision, extra options), in the order TARGETED was filled: bench.py's shapes by batch, then
# config, then precision; then PRODUCT_SHAPES by batch, then shape, then precision
PRODUCT_PLANS = [(plan_id(cfg, BENCH_SHAPES[cfg], B, p), cfg, BENCH_SHAPES[cfg], B, p, [])
                 for B in BATCHES for cfg in sorted(BENCH_SHAPES) for p in PRECISIONS] + \
    [(plan_id(name, hw, B, p), cfg, hw, B, p, extra)
     for B in BATCHES for name, cfg, hw, extra, batches in PRODUCT_SHAPES if B in batches for p in PRECISIONS]

# product plans test_gpu_plan_layers.CASES audits whole, every op: bench.py's default batch in bf16 for every config,
# and in bf16x3 for the three whose deep maps differ (coco_pose shares coco_tracking's backbone and neck)
WHOLE_PLANS = [plan_id(cfg, BENCH_SHAPES[cfg], 32, p) for cfg in sorted(BENCH_SHAPES) for p in ('bf16', 'bf16x3')
               if not (cfg == 'coco_pose' and p == 'bf16x3')]

# product plans the library refuses to build, -> what the refusal says.  nuScenes' two-pass heads at B = 64 in bf16x3:
# the 1x1 heads read a 2048-channel intermediate of 2.9e9 elements, beyond the gather engine's 32-bit offsets; under
# --keep_res at 928 x 1632 the same from B = 16 (3.1e9 elements).  (At B = 32, which KEEP_BATCHES leaves out, mot at
# 1088 x 1920 is refused too: its 1024-channel head intermediate has 4.3e9 elements.)
REFUSED = {plan_id(cfg, hw, B, 'bf16x3'): 'input tensor exceeds 2^31 elements'
           for cfg, hw, B in (('nuscenes_ddd', BENCH_SHAPES['nuscenes_ddd'], 64), ('nuscenes_ddd', (928, 1632), 16))}

# product plan id -> the ops tests/test_gpu_plan_rows.py audits in it: for each row that no test_gpu_plan_layers.CASES
# plan and no earlier entry runs, the first op of the plan that runs it (see `python tests/plan_rows.py`)
TARGETED = {
    'coco_pose_512x512_b1_bf16': ['hm'],
    'mot_544x960_b1_bf16': ['base.level3.tree1.tree1.conv1', 'base.level3.tree1.tree1', 'base.level3.tree1.tree2.conv1',
                            'base.level3', 'base.level4.tree1.tree1.conv1', 'base.level4.tree1.tree1',
                            'base.level4.tree1.tree2.conv1', 'base.level4.tree1', 'base.level4'],
    'mot_544x960_b2_bf16x3': ['base.level4.tree1.tree1.conv1', 'base.level4.tree1.tree1', 'base.level4.tree1.tree2.conv1',
                              'base.level4.tree1', 'base.level4', 'base.level5.tree1.conv1', 'base.level5.tree1',
                              'base.level5.tree2.conv1', 'base.level5', 'dla_up.ida_0.node_1',
                              'dla_up.ida_1.node_1.offset'],
    'coco_pose_512x512_b4_bf16': ['base.level4.tree1.tree1.conv1', 'base.level4.tree1.tree1',
                                  'base.level4.tree1.tree2.conv1', 'base.level4.tree1', 'base.level4',
                                  'base.level5.tree1.conv1', 'base.level5.tree1', 'base.level5.tree2.conv1', 'base.level5'],
    'mot_544x960_b4_bf16': ['base.level5.tree1.conv1', 'base.level5.tree1', 'base.level5.tree2.conv1', 'base.level5',
                            'dla_up.ida_0.proj_1'],
    'mot_544x960_b4_bf16x3': ['base.level5.tree1.conv1', 'base.level5.tree1', 'base.level5.tree2.conv1', 'base.level5',
                              'dla_up.ida_0.proj_1'],
    'nuscenes_ddd_448x800_b4_bf16': ['base.level3.tree1.tree1.conv1', 'base.level3.tree1.tree1',
                                     'base.level3.tree1.tree2.conv1', 'base.level3'],
    'coco_pose_512x512_b8_bf16': ['base.level5.tree1.conv1', 'base.level5.tree1', 'base.level5.tree2.conv1', 'base.level5'],
    'mot_544x960_b8_bf16': ['base.level4.tree1.tree1.conv1', 'base.level4.tree1.tree1', 'base.level4.tree1.tree2.conv1',
                            'base.level4.tree1', 'base.level4', 'dla_up.ida_0.proj_1', 'dla_up.ida_0.node_1.offset'],
    'mot_544x960_b8_bf16x3': ['base.level4.tree1.project', 'base.level4.tree1.tree1.conv1', 'base.level4.tree1.tree1',
                              'base.level4.tree1.tree2.conv1', 'base.level4.tree1', 'base.level4', 'dla_up.ida_0.proj_1',
                              'dla_up.ida_0.node_1.offset'],
    'coco_pose_512x512_b16_bf16': ['base.level4.tree1.tree1.conv1', 'base.level4.tree1.tree1',
                                   'base.level4.tree1.tree2.conv1', 'base.level4.tree1', 'base.level4',
                                   'dla_up.ida_0.node_1.offset'],
    'mot_544x960_b16_bf16': ['base.level5.tree1.conv1', 'base.level5.tree1', 'base.level5.tree2.conv1', 'base.level5'],
    'coco_pose_512x512_b64_bf16': ['base.level5.tree1.conv1', 'base.level5.tree1', 'base.level5.tree2.conv1',
                                   'base.level5', 'dla_up.ida_0.proj_1.offset', 'dla_up.ida_0.node_1.offset'],
    'mot_544x960_b64_bf16': ['dla_up.ida_0.proj_1'],
    # PRODUCT_SHAPES: the rows test_gpu_plan_layers' cases at those sizes do not run
    'coco_tracking_64x1024_b1_bf16x3': ['base.level1', 'heads.0'],
    'mot_1088x1920_b2_bf16': ['dla_up.ida_0.node_1.offset'],
    'coco_tracking_32x64_b4_bf16x3': ['stem48'],
    'coco_tracking_32x64_b64_bf16': ['base.level3.tree1.tree1', 'base.level3.tree1.tree2.conv1'],
}


# product plan id -> the ops tests/test_gpu_plan_rows.py runs at their full size, image by image: for each row with an
# operand of at least LARGE bytes in some product plan, the op of the largest extent in that row (op_extents,
# `python tests/plan_rows.py`)
EXTENT_TARGETED = {
    # bf16x3: the stem's 48-channel fp32 output, and the 1x1 heads reading 256-channel slices of the 1024- / 1792-channel
    # fp32 head intermediate (mot's is 99.6 % of the gather engine's 2^31-element limit; coco_tracking's largest is
    # at 480 x 640)
    'coco_pose_512x512_b64_bf16x3': ['hm_hp', 'hps'],
    'mot_544x960_b64_bf16x3': ['stem48', 'base.level0', 'heads.0', 'hm'],
    'coco_tracking_480x640_b64_bf16x3': ['hm'],
    # the SIMT engine: eight heads' 2048-channel intermediate, 3.1e9 elements under nuScenes' --keep_res at B = 16
    'nuscenes_ddd_928x1632_b16_fp32': ['heads.0', 'hm'],
}

# bench.py's own launches of rows whose largest launch EXTENT_TARGETED names at a PRODUCT_SHAPES size: also run at full
# size by tests/test_gpu_plan_rows.py, being what the benchmarked configs run at B = 64 (each must still have an operand
# of at least LARGE bytes, in a row of large_launches())
EXTENT_BENCH = {
    'coco_tracking_512x512_b64_bf16x3': ['hm'],
    'nuscenes_ddd_448x800_b64_fp32': ['heads.0', 'hm'],
}

LARGE =1 << 31          # bytes: an operand this large has elements (or bytes) past a 32-bit signed offset


def _conv_work(eng, d, kern, cfg):
  """'one' / 'several' work items per CTA of the persistent kernels, '-' for the others (conv_tc.cu / conv_halo.cu)."""
  if kern == 'gather' and d.a_mode == L.CT_A_CONV and (cfg.tile_w, cfg.tile_h) == (16, 8):   # tc_uses_tma
    items = d.B * ((d.OW + 15) // 16) * ((d.OH + 7) // 8) * ((d.C_out + d.n_tile - 1) // d.n_tile)
    grid = min(items, eng.n_sm * (2 if d.n_tile <= 128 else 1))
    return 'one' if items <= grid else 'several'
  if kern == 'halo':
    n_tiles_n = (d.C_out + d.n_tile - 1) // d.n_tile
    tiles = d.B * ((d.OW + cfg.tile_w - 1) // cfg.tile_w) * ((d.OH + cfg.tile_h - 1) // cfg.tile_h)
    groups = min(max(1, eng.n_sm * cfg.ctas_per_sm // n_tiles_n), tiles)
    return 'one' if tiles <= groups else 'several'
  return '-'


def _heads_row(eng):
  d = [pl for kind, pl, name in eng.ops if name == 'heads'][0]
  cfg = L.conv_config(d)
  assert cfg is not None
  tiles = d.B * ((d.OW + cfg.tile_w - 1) // cfg.tile_w) * ((d.OH + cfg.tile_h - 1) // cfg.tile_h)
  return ('heads', d.n_tile, d.heads[0].n_tile, d.n_heads, d.C_in, '%dx%d' % (cfg.tile_w, cfg.tile_h), cfg.stages,
          'one' if tiles <= min(eng.n_sm, tiles) else 'several')


def launch_row(eng, sp):
  """The row of spec sp of engine eng, or None for a record no launch of the plan computes (the fused head launch's
  intermediate, heads.0)."""
  kind = sp['kind']
  dtype = 'bf16' if eng.precision == 'bf16' else 'f32'
  if kind == 'up':
    return ('up', dtype, sp['x'].C, sp['f'])
  if kind != 'conv':
    return (kind, dtype)
  if eng.head_table is not None and sp['name'] not in {name for _, _, name in eng.ops}:
    return None if sp['name'] == 'heads.0' else _heads_row(eng)
  d = sp['desc']
  kern = KERNEL[sp['engine']]
  kh, kw = sp['k']
  cfg = L.conv_config(d)             # the launch configuration the library picks for this op
  assert cfg is not None, sp['name']
  launch = ('%dx%d' % (cfg.tile_w, cfg.tile_h), cfg.stages, cfg.overlap) if kern != 'simt' else ('-', '-', '-')
  return (kern, sp['n_tile'], d.C_in, '%dx%d' % (kh, kw), sp['stride'], A_MODE[sp['a_mode']],
          OUT_MODE[sp['out_mode']], int(sp['residual'] is not None),
          int(sp['out_mode'] == L.CT_OUT_NHWC_S2D or sp['name'] in eng.s2d_named), int(bool(sp['sum3']))) + \
      launch + (_conv_work(eng, d, kern, cfg),)


def plan_rows(eng):
  """{row: [names of the ops that run it, in plan order]}."""
  rows = {}
  for sp in eng.specs:
    r = launch_row(eng, sp)
    if r is not None:
      rows.setdefault(r, []).append(sp['name'])
  return rows


OPERANDS = ('x', 'residual', 'om', 'skip', 'out')


def op_extents(eng):
  """{op name: {operand: (elements, bytes)}} of every op a launch of the plan computes, for each operand it reads or
  writes: a channel slice by the whole NHWC buffer it lies in (B H W ld), a tensor (the offset / mask map, the fp32 NCHW
  head planes B C_out OH OW) by itself.  Leaves out the fused head launch's records (heads.0 and the 1x1s that read its
  intermediate, which never exists); its outputs are the same planes those 1x1 records describe."""
  from centertrack_b200.engine import DeferredTV, TV
  res = {}
  for sp in eng.specs:
    if isinstance(sp.get('x'), DeferredTV) or launch_row(eng, sp) is None:
      continue
    ext = {}
    for k in OPERANDS:
      t = sp.get(k)
      if t is None:
        continue
      b = t.buf if isinstance(t, TV) else t
      ext[k] = (b.numel(), b.numel() * b.element_size())
    d = sp['desc']
    if d is not None:                # what the gather engine's guard counts: the whole buffer x lies in
      assert ext['x'][0] == d.B * d.H * d.W * d.ld_in, sp['name']
      if d.out_mode == L.CT_OUT_NCHW_F32:
        assert ext['out'][0] == d.B * d.C_out * d.OH * d.OW, sp['name']
    res[sp['name']] = ext
  return res


def largest_operand(ext):
  """(bytes, elements, operand) of the largest operand of an op_extents entry."""
  return max((b, n, k) for k, (n, b) in ext.items())


def large_launches():
  """{row: (plan id, op, bytes, elements, operand)}: for every row with an operand of at least LARGE bytes in a
  (buildable) PRODUCT_PLANS plan, the op with the largest operand in that row, at the first plan that has it."""
  big = {}
  for pid, cfg, hw, B, precision, extra in PRODUCT_PLANS:
    if pid in REFUSED:
      continue
    eng = cpu_plan(cfg, hw, B, precision, extra)
    rows = {sp['name']: launch_row(eng, sp) for sp in eng.specs}
    for name, ext in op_extents(eng).items():
      nbytes, n, k = largest_operand(ext)
      row = rows[name]
      if row not in big or nbytes > big[row][2]:
        big[row] = (pid, name, nbytes, n, k)
    del eng
  return {r: v for r, v in big.items() if v[2] >= LARGE}


def extent_unaudited(targeted, large=None):
  """[(row, (plan id, op, bytes, elements, operand))] of the large launches (large_launches(), or `large`) whose op
  targeted does not name in its plan."""
  large = large_launches() if large is None else large
  return [(r, v) for r, v in large.items() if v[1] not in targeted.get(v[0], ())]


def format_row(row):
  return ' '.join('%s' % v for v in row)


_MODELS = {}


@contextlib.contextmanager
def _env(env):
  old = {k: os.environ.get(k) for k in env}
  os.environ.update(env)
  try:
    yield
  finally:
    for k, v in old.items():
      if v is None:
        os.environ.pop(k, None)
      else:
        os.environ[k] = v


def cpu_plan(cfg, hw, B, precision, extra=(), kw=None, env=None):
  """The plan the product builds for (cfg, hw, B, precision), on the CPU (ct_conv_config needs no GPU; n_sm = 132)."""
  from helpers import make_model
  from centertrack_b200.engine import DLA34Engine
  key = (cfg, tuple(extra))
  if key not in _MODELS:
    _MODELS[key] = make_model(cfg, extra=list(extra))[:2]
  opt, model = _MODELS[key]
  with _env(env or {}):
    return DLA34Engine(model._engine_state_dict(), model.heads, B, hw[0], hw[1], precision=precision, device='cpu',
                       depth_scale=getattr(opt, 'depth_scale', 1.0), dla_node=getattr(opt, 'dla_node', 'dcn'),
                       **(kw or {}))


def case_rows(cases):
  """{row: set of case ids} of test_gpu_plan_layers.CASES-style tuples."""
  cov = {}
  for cid, cfg, hw, B, precision, extra, kw, env in cases:
    for r in plan_rows(cpu_plan(cfg, hw, B, precision, extra, kw, env)):
      cov.setdefault(r, set()).add(cid)
  return cov


def unaudited(cases, targeted):
  """Rows of the product plans that neither a case nor a targeted op runs: [(plan id, row, [ops that run it])], each
  row once, at the first plan (PRODUCT_PLANS order) that runs it.  Also returns the product plans' rows."""
  audited = set(case_rows(cases))
  plans = {}
  for pid, cfg, hw, B, precision, extra in PRODUCT_PLANS:
    if pid in REFUSED:
      continue
    rows = plan_rows(cpu_plan(cfg, hw, B, precision, extra))
    plans[pid] = rows
    for r, names in rows.items():
      if set(names) & set(targeted.get(pid, ())):
        audited.add(r)
  missing, seen = [], set()
  for pid in plans:
    for r, names in plans[pid].items():
      if r not in audited and r not in seen:
        seen.add(r)
        missing.append((pid, r, names))
  return missing, plans


if __name__ == '__main__':
  from test_gpu_plan_layers import CASES
  missing, _ = unaudited(CASES, TARGETED)
  add = {}
  for pid, r, names in missing:
    print('%-36s %-12s %s' % (pid, names[0], format_row(r)))
    add.setdefault(pid, []).append(names[0])
  print('\n%d rows unaudited; TARGETED entries that cover them:' % len(missing))
  for pid, _, _, _, _, _ in PRODUCT_PLANS:
    if pid in add:
      print('    %r: %r,' % (pid, add[pid]))
  big = extent_unaudited(EXTENT_TARGETED)
  add = {}
  print()
  for r, (pid, name, nbytes, n, k) in big:
    print('%-36s %-12s %-8s %13d elements %6.2f GB  %s' % (pid, name, k, n, nbytes / 1e9, format_row(r)))
    add.setdefault(pid, []).append(name)
  print('\n%d launches with an operand of >= 2^31 bytes unaudited; EXTENT_TARGETED entries that cover them:' % len(big))
  for pid, _, _, _, _, _ in PRODUCT_PLANS:
    if pid in add:
      print('    %r: %r,' % (pid, add[pid]))
