"""-m gpu: the launch configurations of the product plans that no test_gpu_plan_layers.CASES plan runs, audited op by op,
the product's largest launches at their full size, and the batch-prefix runs (engine.forward(..., n)) of the
benchmarked mot plan against its full-batch run.

plan_rows.TARGETED names, per product plan, the ops that run a configuration nothing else audits (tests/plan_rows.py);
each plan is built as the product builds it, replayed once on synthetic_inputs, and only those ops are recomputed in fp64
and held to the bounds of tests/bounds.py, as test_gpu_plan_layers does for whole plans.

plan_rows.EXTENT_TARGETED and EXTENT_BENCH name the launches with operands of >= 2^31 bytes (B = 64, or 16 under
nuScenes' --keep_res): they are checked in fp64 on their first and last four images, and bit for bit on every image
against the same launch on 4-image slices, so an offset that wraps past 32 bits anywhere in the batch fails."""
import ctypes as C
import gc
import time

import pytest
import torch

import bounds as bd
import plan_rows as pr
import test_gpu_plan_layers as tpl
from centertrack_b200 import _lib as L
from centertrack_b200.engine import DeferredTV

pytestmark = pytest.mark.gpu

PLANS = {pid: (cfg, hw, B, p, extra) for pid, cfg, hw, B, p, extra in pr.PRODUCT_PLANS}


def _ops_within_bounds(eng, pid, names, chunks):
  """fp64 bounds of ops `names` of eng on the image slices `chunks` -> (failures, report lines); a report line gives the
  op's worst |err| / bound, then that of each chunk, the largest |err| / mag beyond the output rounding as a multiple of
  its constant, and the row."""
  specs = {sp['name']: sp for sp in eng.specs}
  failures, report = [], []
  for name in names:
    sp = specs[name]
    row = pr.format_row(pr.launch_row(eng, sp))
    worst, where, use, per_chunk = 0.0, None, 0.0, []
    for bs in chunks:
      res = tpl._check_conv(eng, sp, bs) if sp['kind'] == 'conv' else tpl._check_other(eng, sp, bs)
      if res is None:
        continue
      m, at = bd.worst(res[0])
      per_chunk.append('%d-%d: %.3f' % (bs.start, bs.stop - 1, m))
      if where is None or m > worst:
        worst, where = m, dict(at, b=at['b'] + bs.start)
      if res[1] is not None:
        use = max(use, float(res[1].max()))
      del res
    coef = tpl.COEF[tpl.KERNEL[sp['engine']]] if sp['kind'] == 'conv' else bd.ALPHA_BF16 if eng.precision == 'bf16' \
        else bd.GAMMA_SIMT
    report.append('  %-34s %.3f%s  %.3f  %s' % (name, worst, ' (images %s)' % ', '.join(per_chunk)
                                                if len(chunks) <= 2 else '', use / coef, row))
    if not worst <= 1.0:
      failures.append('%s: op %s (row %s): worst element %s, |err| / bound = %.3g' % (pid, name, row, where, worst))
  return failures, report


def _chunks(B):
  return [slice(b0, min(B, b0 + tpl.CHUNK)) for b0 in range(0, B, tpl.CHUNK)]


@pytest.mark.parametrize('pid', sorted(pr.TARGETED))
def test_targeted_ops_within_bounds(pid, monkeypatch):
  cfg, hw, B, precision, extra = PLANS[pid]
  eng = tpl._build(cfg, hw, B, precision, extra, {}, monkeypatch, {})
  tpl._assert_no_overlapping_writes(eng)
  failures, report = _ops_within_bounds(eng, pid, pr.TARGETED[pid], _chunks(eng.B))
  print('\n[%s] per audited op: worst |err| / bound, largest |err| / mag beyond the output rounding as a multiple of '
        'its constant, row\n%s' % (pid, '\n'.join(report)))
  assert not failures, '\n'.join(failures)


# ---- the largest launches of the product plans (plan_rows.EXTENT_TARGETED), at their full size ------------------------
def _image_stride(t):
  """Bytes from one image to the next of an operand (a channel slice of an NHWC buffer, or a tensor)."""
  b = t.buf if hasattr(t, 'buf') else t
  return b.stride(0) * b.element_size()


def _int_view(t):
  return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _sliced_matches(eng, sp, n=tpl.CHUNK):
  """Re-issue conv op sp's launch on n-image slices (its descriptor with B = n and x / residual / om / out advanced by
  the slice's first image) into a NaN-filled copy of its output buffer -> [problems].  Every image's output must equal
  the full-batch launch's bit for bit, and no byte of the copy outside the op's channels may change.

  Valid because each engine accumulates an output element over K in an order that does not depend on its pixel's
  position in the batch: the SIMT kernel's fma chain over k, the gather / x3 kernels' K slices in order through the same
  wgmma chain for every GEMM row (one row per pixel, whatever M tile it lands in).  A launch at B = n reaches only
  offsets below n images, so a wrapped 32-bit offset in the full-batch launch shows up as a difference."""
  d0 = sp['desc']
  o = sp['out']
  full = o.buf if hasattr(o, 'buf') else o
  off, nc = (o.off, o.C) if hasattr(o, 'buf') else (0, full.shape[-1])
  fresh = torch.full_like(full, float('nan'))
  step = {k: _image_stride(sp[k]) for k in ('x', 'residual', 'om', 'out') if sp[k] is not None}
  lib, st = L.lib(), L.stream_ptr()
  for b0 in range(0, eng.B, n):
    d = L.ConvDesc.from_buffer_copy(d0)
    d.B = min(n, eng.B - b0)
    d.x = d0.x + b0 * step['x']
    if 'residual' in step:
      d.residual = d0.residual + b0 * step['residual']
    if 'om' in step:
      d.om = d0.om + b0 * step['om']
    d.out = fresh.data_ptr() + (d0.out - full.data_ptr()) + b0 * step['out']
    L.check(lib.ct_conv_forward(C.byref(d), st), '%s on images %d..' % (sp['name'], b0))
  torch.cuda.synchronize()
  bad = []
  nan = _int_view(torch.full((1,), float('nan'), dtype=full.dtype, device=full.device))
  for b0 in range(0, eng.B, n):
    got, want = _int_view(fresh[b0:b0 + n]), _int_view(full[b0:b0 + n])
    if hasattr(o, 'buf'):
      diff = (got[..., off:off + nc] != want[..., off:off + nc]).reshape(got.shape[0], -1).any(1)
      stray = torch.cat([got[..., :off], got[..., off + nc:]], -1) != nan
      stray = stray.reshape(got.shape[0], -1).any(1)
    else:
      diff = (got != want).reshape(got.shape[0], -1).any(1)
      stray = torch.zeros_like(diff)
    if bool(diff.any()):
      bad.append('%s: images %s differ from the B = %d launch' % (sp['name'], (diff.nonzero().flatten() + b0).tolist(),
                                                                   eng.B))
    if bool(stray.any()):
      bad.append('%s: the sliced launch wrote outside its channels in images %s' % (
          sp['name'], (stray.nonzero().flatten() + b0).tolist()))
  del fresh
  return bad


def _plan_need(cfg, hw, B, precision, extra, names):
  """Device bytes the extent test needs for a plan: its buffers at batch B (the B = 1 plan's activations times B, plus
  weights), and twice the largest operand of the audited ops (the NaN-filled output copy, or the fp64 reference of
  4 images)."""
  eng = pr.cpu_plan(cfg, hw, 1, precision, extra)
  seen = {}
  for t in eng.keep + [eng.in_img, eng.in_pre, eng.in_hm] + list(eng.outputs.values()):
    seen[t.data_ptr()] = t.numel() * t.element_size() * (B if t.dim() == 4 else 1)
  ext = pr.op_extents(eng)
  return sum(seen.values()) + 2 * B * max(pr.largest_operand(ext[n])[0] for n in names)


EXTENT_RUN = dict(pr.EXTENT_TARGETED, **pr.EXTENT_BENCH)


@pytest.mark.parametrize('pid', sorted(EXTENT_RUN))
def test_largest_launches_at_full_size(pid, monkeypatch):
  """The product's launches with operands of >= 2^31 bytes, at their plan's batch (plan_rows.EXTENT_TARGETED, and the
  benchmarked configs' own such launches, plan_rows.EXTENT_BENCH): each audited op within the fp64 bounds on its first
  and last 4-image chunk (the last holds the largest offsets), and bit-identical on every image to the same launch
  issued on 4-image slices."""
  cfg, hw, B, precision, extra = PLANS[pid]
  names = EXTENT_RUN[pid]
  need = _plan_need(cfg, hw, B, precision, extra, names)
  gc.collect()
  torch.cuda.empty_cache()
  free, total = torch.cuda.mem_get_info()
  if free < need:
    pytest.skip('%s needs about %.1f GB of device memory, %.1f GB of %.1f GB free' % (pid, need / 1e9, free / 1e9,
                                                                                      total / 1e9))
  torch.cuda.reset_peak_memory_stats()
  t0 = time.time()
  eng = specs = None
  try:
    eng = tpl._build(cfg, hw, B, precision, extra, {}, monkeypatch, {})
    tpl._assert_no_overlapping_writes(eng)
    specs = {sp['name']: sp for sp in eng.specs}
    ext = pr.op_extents(eng)
    # the first and last CHUNK images, in passes as small as the fp64 reference needs: up to about twenty fp64 tensors
    # the size of the largest operand's images are alive at once (nuScenes' 2048-channel head intermediate is 1.6 GB an
    # image at 928 x 1632)
    per_image = max(pr.largest_operand(ext[n])[1] for n in names) // B * 8
    step = int(max(1, min(tpl.CHUNK, torch.cuda.mem_get_info()[0] // (24 * per_image))))
    chunks = [slice(b, min(b + step, e)) for s, e in ((0, tpl.CHUNK), (B - tpl.CHUNK, B)) for b in range(s, e, step)]
    failures, report = _ops_within_bounds(eng, pid, names, chunks)
    for name in names:
      failures += _sliced_matches(eng, specs[name])
      nbytes, n, k = pr.largest_operand(ext[name])
      report.append('  %-34s bit-identical on %d images (4-image slices); largest operand %s, %d elements, %.2f GB' % (
          name, B, k, n, nbytes / 1e9) if not any(f.startswith(name + ':') for f in failures) else
          '  %-34s DIFFERS from its 4-image slices' % name)
    print('\n[%s] per audited op: worst |err| / bound (first and last chunk), largest |err| / mag beyond the output '
          'rounding as a multiple of its constant, row\n%s\n  peak device memory %.1f GB (estimated need %.1f GB), '
          '%.0f s' % (pid, '\n'.join(report), torch.cuda.max_memory_allocated() / 1e9, need / 1e9, time.time() - t0))
    assert not failures, '\n'.join(failures)
  finally:                            # free the plan's buffers before the next case, even if a frame still holds eng
    if eng is not None:
      eng.__dict__.clear()
    eng = specs = None
    gc.collect()
    torch.cuda.empty_cache()


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
  read them would also spoil the first n.  Images < n are restored to the full-batch result before each run, so an
  element of them that forward(n) leaves unwritten still passes: test_gpu_plan_fresh_state.py's
  test_graph_eager_and_prefix_agree_from_poisoned_buffers poisons every image and restores nothing."""
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
