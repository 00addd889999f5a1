"""-m gpu: every launch of the shipped plans against an fp64 reference with per-element error bounds (tests/bounds.py).

The engine is built as the product builds it (synthetic calibrated checkpoint, realistic inputs), one CUDA-graph
replay runs with the fused activations, and then every op's output is recomputed in fp64 from the buffers as they are
after the replay.  That is valid because the plan never writes in place: every buffer still holds what its consumer
read -- which the test asserts first by checking that no two ops write overlapping bytes.  Each layer therefore runs at
the (engine, N tile, stages, tile shape, ld / offset) its plan selects for that batch and resolution.
"""
import pytest
import torch
import torch.nn.functional as F

import bounds as bd
import ct_oracle as co
from centertrack_b200 import _lib as L
from helpers import HEAD_LAYOUTS
from plan_rows import format_row, launch_row

pytestmark = pytest.mark.gpu

KERNEL = {L.CT_ENGINE_SIMT: 'simt', L.CT_ENGINE_TCGEN05: 'gather', L.CT_ENGINE_TCGEN05_X3: 'gather_x3',
          L.CT_ENGINE_TCGEN05_HALO: 'halo'}
COEF = {'simt': bd.GAMMA_SIMT, 'gather': bd.ALPHA_BF16, 'gather_x3': bd.BETA_X3, 'halo': bd.ALPHA_BF16}
HEAD_ACT = {L.CT_HEAD_NONE: 'none', L.CT_HEAD_SIGMOID: 'sigmoid', L.CT_HEAD_DEPTH: 'depth'}

# (id, config, (H, W), B, precision, extra options, engine keyword arguments, environment)
CASES = [
    ('coco_tracking_512_b32_bf16', 'coco_tracking', (512, 512), 32, 'bf16', [], {}, {}),
    ('coco_tracking_512_b32_bf16x3', 'coco_tracking', (512, 512), 32, 'bf16x3', [], {}, {}),
    ('coco_tracking_512_b1_bf16', 'coco_tracking', (512, 512), 1, 'bf16', [], {}, {}),
    ('coco_tracking_512_b1_bf16x3', 'coco_tracking', (512, 512), 1, 'bf16x3', [], {}, {}),
    ('coco_tracking_512_b1_fp32', 'coco_tracking', (512, 512), 1, 'fp32', [], {}, {}),
    ('mot_544x960_b2_bf16', 'mot', (544, 960), 2, 'bf16', [], {}, {}),
    ('nuscenes_ddd_448x800_b2_bf16', 'nuscenes_ddd', (448, 800), 2, 'bf16', [], {}, {}),
    ('coco_pose_512_b2_bf16', 'coco_pose', (512, 512), 2, 'bf16', [], {}, {}),
    ('coco_pose_512_b2_bf16x3', 'coco_pose', (512, 512), 2, 'bf16x3', [], {}, {}),
    # bench.py's batch: the 34 x 60 / 28 x 50 maps on the register gather at N = 256, the window DCN at N = 128 over 512
    # channels, and in bf16x3 level5 and the global DCN at N = 128
    ('mot_544x960_b32_bf16', 'mot', (544, 960), 32, 'bf16', [], {}, {}),
    ('mot_544x960_b32_bf16x3', 'mot', (544, 960), 32, 'bf16x3', [], {}, {}),
    ('nuscenes_ddd_448x800_b32_bf16', 'nuscenes_ddd', (448, 800), 32, 'bf16', [], {}, {}),
    ('nuscenes_ddd_448x800_b32_bf16x3', 'nuscenes_ddd', (448, 800), 32, 'bf16x3', [], {}, {}),
    ('coco_pose_512_b32_bf16', 'coco_pose', (512, 512), 32, 'bf16', [], {}, {}),
    ('dla_node_conv_64x96_b2_bf16', 'coco_tracking', (64, 96), 2, 'bf16', ['--dla_node', 'conv'], {}, {}),
    ('dla_node_gcn_64x96_b2_bf16', 'coco_tracking', (64, 96), 2, 'bf16', ['--dla_node', 'gcn'], {}, {}),
    ('coco_tracking_256_b2_bf16_no_halo', 'coco_tracking', (256, 256), 2, 'bf16', [], {'use_halo': False}, {}),
    ('coco_tracking_256_b2_bf16_dcn_global', 'coco_tracking', (256, 256), 2, 'bf16', [], {}, {'CTB_DCN_WINDOW': '0'}),
    # input sizes beyond the bench (plan_rows.PRODUCT_SHAPES): kitti(_tracking)'s default, whose level 5 is 12 x 40 ...
    ('kitti_tracking_384x1280_b2_bf16', 'coco_tracking', (384, 1280), 2, 'bf16', ['--num_classes', '3'], {}, {}),
    ('kitti_tracking_384x1280_b2_bf16x3', 'coco_tracking', (384, 1280), 2, 'bf16x3', ['--num_classes', '3'], {}, {}),
    # ... a 1080p camera under --keep_res: level 4's convs on the plain gather at N = 64 with several work items per CTA
    ('mot_keep_1088x1920_b1_bf16', 'mot', (1088, 1920), 1, 'bf16', [], {}, {}),
    # ... a 64 x 1024 strip: the bf16x3 gather at N = 16 on level 2 and the global DCN
    ('wide_64x1024_b2_bf16x3', 'coco_tracking', (64, 1024), 2, 'bf16x3', [], {}, {}),
    # ... and a VGA camera under --keep_res (level 5 is 15 x 20)
    ('coco_keep_480x640_b2_bf16', 'coco_tracking', (480, 640), 2, 'bf16', [], {}, {}),
] + [  # the other output-head layouts (tests/helpers.py::HEAD_LAYOUTS); bf16x3 plans them all in two passes
    ('heads_%s_64x96_b2_%s' % (tag, precision), cfg, (64, 96), 2, precision, extra, {}, {})
    for tag, cfg, extra, plan in HEAD_LAYOUTS for precision in ('bf16', 'bf16x3')
    if precision == 'bf16' or plan[0] == 'two_pass']

CHUNK = 4      # images per fp64 reference pass (bounds the memory of the fp64 DCN columns)


def _nchw(t):
  return t.permute(0, 3, 1, 2).double()


def _unshuffle(t):
  """[B, h, w, (sy, sx, c)] space-to-depth -> [B, c, 2h, 2w] fp64."""
  B, h, w, c4 = t.shape
  c = c4 // 4
  return t.reshape(B, h, w, 2, 2, c).permute(0, 5, 1, 3, 2, 4).reshape(B, c, 2 * h, 2 * w).double()


def _out_ranges(eng):
  """(op name, base address, bytes, first channel, end channel) of what every op writes."""
  res = []
  for sp in eng.specs:
    o = sp['out']
    if hasattr(o, 'buf'):           # TV: a channel slice of an NHWC buffer
      res.append((sp['name'], o.buf.data_ptr(), o.buf.numel() * o.buf.element_size(), o.off, o.off + o.C))
    else:
      res.append((sp['name'], o.data_ptr(), o.numel() * o.element_size(), 0, o.shape[-1]))
  return res


def _assert_no_overlapping_writes(eng):
  rs = _out_ranges(eng)
  for i in range(len(rs)):
    for j in range(i):
      (na, pa, sa, ca0, ca1), (nb, pb, sb, cb0, cb1) = rs[i], rs[j]
      if pa == pb and sa == sb:
        assert ca1 <= cb0 or cb1 <= ca0, 'ops %s and %s write overlapping channels of one buffer' % (na, nb)
      else:
        assert pa + sa <= pb or pb + sb <= pa, 'ops %s and %s write overlapping memory' % (na, nb)


def _conv_chunk(eng, sp, bs):
  """fp64 (ref, mag) of a conv op for images bs, from the operands as the kernel read them."""
  kern = KERNEL[sp['engine']]
  w = sp['w'].float()
  w = (w.bfloat16() if kern in ('gather', 'halo') else w).double().cuda()   # ct_pack_weights: fp32, then bf16 RNE
  shift = sp['shift'].float().double().cuda()
  if sp['name'] == 'stem48':
    d = sp['desc']
    assert d.shift == eng.stem48_shift[1 | 2 * eng.has_pre_img | 4 * eng.has_pre_hm].data_ptr()
    shift = eng.stem48_shift[1 | 2 * eng.has_pre_img | 4 * eng.has_pre_hm].double()
  x = _nchw(sp['x'].tensor()[bs])
  kh, kw = sp['k']
  ph, pw = sp['pad']
  OH, OW = sp['out_hw']
  if sp['a_mode'] == L.CT_A_CONV:
    xp = F.pad(x, (pw, pw, ph, ph))
    ref = F.conv2d(xp, w, None, sp['stride'])[..., :OH, :OW]
    mag = F.conv2d(xp.abs(), w.abs(), None, sp['stride'])[..., :OH, :OW]
  else:
    om = sp['om'][bs].permute(0, 3, 1, 2)
    cols = co.dcn_sample_columns(x, om[:, :18].contiguous(), om[:, 18:27].contiguous(), bf16_blend=kern == 'gather')
    n, C = x.shape[0], x.shape[1]
    wm = w.reshape(w.shape[0], C * 9)
    cols = cols.reshape(n, C * 9, OH * OW)
    ref = torch.matmul(wm, cols).view(n, -1, OH, OW)
    mag = torch.matmul(wm.abs(), cols.abs()).view(n, -1, OH, OW)
    del cols
  C_out = w.shape[0]
  ref = ref + shift[:C_out].view(1, -1, 1, 1)
  mag = mag + shift[:C_out].abs().view(1, -1, 1, 1)
  if sp['residual'] is not None:
    r = _nchw(sp['residual'].tensor()[bs])
    ref, mag = ref + r, mag + r.abs()
  return ref, mag


def _check_conv(eng, sp, bs):
  """-> (per-element ratio to the bound, per-element accumulation use or None) for images bs."""
  kern = KERNEL[sp['engine']]
  coef = COEF[kern]
  ref, mag = _conv_chunk(eng, sp, bs)
  om = sp['out_mode']
  bf16_out = om in (L.CT_OUT_NHWC, L.CT_OUT_NHWC_S2D) and eng.precision == 'bf16'
  d = sp['desc']
  if sp['sum3']:                   # stem: sum over the present stems of relu(group + shift)
    lo, hi = bd.stem_interval(ref, mag, coef, d.epilogue_sum3)
    got = sp['out'].tensor()[bs]
    got = _unshuffle(got) if om == L.CT_OUT_NHWC_S2D else _nchw(got)
    return bd.ratio_interval(got, lo, hi, bf16_out), None
  if om == L.CT_OUT_NCHW_F32:
    got = sp['out'][bs].double()
    act = HEAD_ACT[d.head_act]
    r = bd.ratio(got, ref, mag, coef, False, act, eng.depth_scale) if not sp['relu'] else \
        bd.ratio_interval(got, *bd.interval(ref, coef * mag, act, eng.depth_scale, relu=True), False)
    use = bd.accum_use(got, ref, mag, False) if act == 'none' and not sp['relu'] else None
    return r, use
  if om == L.CT_OUT_NHWC_F32:
    got = _nchw(sp['out'][bs])[:, :ref.shape[1]]
    sig = torch.arange(ref.shape[1], device=ref.device).view(1, -1, 1, 1) >= sp['sig_from']
    lo_i, hi_i = bd.interval(ref, coef * mag, 'none', relu=sp['relu'])
    lo_s, hi_s = bd.interval(ref, coef * mag, 'sigmoid', relu=sp['relu'])
    r = bd.ratio_interval(got, torch.where(sig, lo_s, lo_i), torch.where(sig, hi_s, hi_i), False)
    use = bd.accum_use(got, ref, mag, False)
    use = torch.where(sig, torch.zeros_like(use), use)
    return r, use
  got = sp['out'].tensor()[bs]
  got = _unshuffle(got) if om == L.CT_OUT_NHWC_S2D else _nchw(got)
  r = bd.ratio(got, ref, mag, coef, bf16_out, 'relu' if sp['relu'] else 'none')
  use = bd.accum_use(got, ref.clamp_min(0) if sp['relu'] else ref, mag, bf16_out)
  if sp['relu']:                   # only where the ReLU did not clip
    use = torch.where(ref > coef * mag, use, torch.zeros_like(use))
  return r, use


OTHER_KINDS = ('pack', 'pack32', 'pool', 'pool_s2d', 'up', 'stem')     # the kinds _check_other checks


def _check_other(eng, sp, bs):
  """Non-conv ops: pack / pool exact, up (depthwise ConvT + skip) and the SIMT stem by the bound."""
  k = sp['kind']
  bf16 = eng.precision == 'bf16'
  if k in ('pack', 'pack32'):
    parts = [eng.in_img[bs], eng.in_pre[bs] if eng.has_pre_img else torch.zeros_like(eng.in_img[bs]),
             eng.in_hm[bs] if eng.has_pre_hm else torch.zeros_like(eng.in_hm[bs]), torch.zeros_like(eng.in_hm[bs])]
    want = torch.cat(parts, 1).permute(0, 2, 3, 1).to(torch.bfloat16 if k == 'pack' else torch.float32)
    assert torch.equal(sp['out'].tensor()[bs], want), '%s: packed stem input differs' % sp['name']
    return None
  if k == 'pool':
    want = F.max_pool2d(_nchw(sp['x'].tensor()[bs]), 2, 2)
    assert torch.equal(_nchw(sp['out'].tensor()[bs]), want), 'maxpool differs'
    return None
  if k == 'pool_s2d':
    x = sp['x'].tensor()[bs]
    want = x.reshape(*x.shape[:3], 4, x.shape[-1] // 4).amax(3)
    assert torch.equal(sp['out'].tensor()[bs], want), 'space-to-depth maxpool differs'
    return None
  coef = bd.ALPHA_BF16 if bf16 else bd.GAMMA_SIMT
  if k == 'stem':
    coef = bd.GAMMA_SIMT
  if k == 'up':
    x, f = _nchw(sp['x'].tensor()[bs]), sp['f']
    w = sp['w'].double().cuda()
    C = x.shape[1]
    ref = F.conv_transpose2d(x, w, None, stride=f, padding=f // 2, groups=C)
    mag = F.conv_transpose2d(x.abs(), w.abs(), None, stride=f, padding=f // 2, groups=C)
    s = _nchw(sp['skip'].tensor()[bs])
    ref, mag = ref + s, mag + s.abs()
    got = _nchw(sp['out'].tensor()[bs])
    return bd.ratio(got, ref, mag, coef, bf16), bd.accum_use(got, ref, mag, bf16)
  assert k == 'stem'                # SIMT stem: three 7x7 convs 3/3/1 -> 16 in fp32, ReLU each, summed, stored
  wst, sh = sp['w'], sp['shift']
  x8 = torch.cat([eng.in_img[bs], eng.in_pre[bs], eng.in_hm[bs]], 1).double()
  lo = hi = 0
  for g, (c0, cn) in enumerate(((0, 3), (3, 3), (6, 1))):
    if g == 1 and not eng.has_pre_img or g == 2 and not eng.has_pre_hm:
      continue
    w = wst[:, c0:c0 + cn, :].reshape(7, 7, cn, 16).permute(3, 2, 0, 1).cuda()
    ref, mag = bd.conv_ref(x8[:, c0:c0 + cn], w, sh[g], pad=(3, 3, 3, 3))
    a, b = bd.interval(ref, coef * mag, relu=True)
    lo, hi = lo + a, hi + b
  return bd.ratio_interval(_nchw(sp['out'].tensor()[bs]), lo, hi, bf16), None


def _build(cfg, hw, B, precision, extra, kw, monkeypatch, env):
  from helpers import make_model
  from centertrack_b200 import synthetic as syn
  from centertrack_b200.engine import DLA34Engine
  for k, v in env.items():
    monkeypatch.setenv(k, v)
  opt, model, _ = make_model(cfg, extra=extra)
  dev = torch.device('cuda')
  model = model.to(dev)
  if kw:
    eng = DLA34Engine(model._engine_state_dict(), model.heads, B, hw[0], hw[1], precision=precision, device=dev,
                      depth_scale=getattr(opt, 'depth_scale', 1.0), dla_node=getattr(opt, 'dla_node', 'dcn'), **kw)
  else:
    eng = model.engine_for(B, hw[0], hw[1], dev, precision)
  img, pre, hm = syn.synthetic_inputs(B, hw[0], hw[1])
  eng.in_img.copy_(img)
  eng.in_pre.copy_(pre)
  eng.in_hm.copy_(hm)
  eng.set_fused_activations(True)
  eng.replay()
  torch.cuda.synchronize()
  return eng


COVERAGE = {}


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_plan_layers_within_bounds(case, monkeypatch):
  cid, cfg, hw, B, precision, extra, kw, env = case
  eng = _build(cfg, hw, B, precision, extra, kw, monkeypatch, env)
  _assert_no_overlapping_writes(eng)
  failures, worst_ratio, worst_use = [], (0.0, ''), {}
  for sp in eng.specs:
    is_conv = sp['kind'] == 'conv'
    kern = KERNEL[sp['engine']] if is_conv else sp['kind']
    layer_worst, layer_at, layer_use = 0.0, None, 0.0
    for b0 in range(0, eng.B, CHUNK):
      bs = slice(b0, min(eng.B, b0 + CHUNK))
      res = _check_conv(eng, sp, bs) if is_conv else _check_other(eng, sp, bs)
      if res is None:
        continue
      r, use = res[0], res[1]
      m, at = bd.worst(r)
      if m > layer_worst or layer_at is None:
        layer_worst, layer_at = m, dict(at, b=at['b'] + b0)
      if use is not None:
        layer_use = max(layer_use, float(use.max()))
      del res, r, use
    row = launch_row(eng, sp)
    if row is not None:
      COVERAGE.setdefault(row, set()).add(cid)
    if layer_at is None:
      continue
    if is_conv:
      key = (kern, 'fp32 out' if sp['out_mode'] in (L.CT_OUT_NHWC_F32, L.CT_OUT_NCHW_F32) or precision != 'bf16'
             else 'bf16 out')
    else:
      key = (kern, precision)
    if layer_use > worst_use.get(key, (0.0, ''))[0]:
      worst_use[key] = (layer_use, sp['name'])
    if layer_worst > worst_ratio[0]:
      worst_ratio = (layer_worst, sp['name'])
    if not layer_worst <= 1.0:
      failures.append('%s (%s, N=%s): worst element %s, |err| / bound = %.3g' % (
          sp['name'], kern, sp.get('n_tile', '-'), layer_at, layer_worst))
  print('\n[%s] %d ops; worst |err| / bound %.3f (%s)' % (cid, len(eng.specs), worst_ratio[0], worst_ratio[1]))
  for key, (u, name) in sorted(worst_use.items()):
    c = COEF.get(key[0], bd.ALPHA_BF16 if precision == 'bf16' else bd.GAMMA_SIMT)
    print('  %-10s %-8s largest |err| / mag beyond the output rounding %.3g = %.3f x its constant (%s)' % (
        key[0], key[1], u, u / c, name))
  assert not failures, '%s: %d ops out of bounds:\n  %s' % (cid, len(failures), '\n  '.join(failures))


def test_zz_plan_coverage_table():
  """Print the launch configuration rows (tests/plan_rows.py) the plans above ran (runs after them in file order):
  conv rows are (kernel, N, C_in, k, stride, a_mode, out_mode, residual, s2d, sum3, tile, stages, overlap, work per
  CTA)."""
  if not COVERAGE:
    pytest.skip('no plan audited in this session')
  for row in sorted(COVERAGE, key=lambda r: tuple(str(v) for v in r)):
    print('%-62s  %s' % (format_row(row), ','.join(sorted(COVERAGE[row]))))
