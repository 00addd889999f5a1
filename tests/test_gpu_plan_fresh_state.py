"""-m gpu: every launch of the shipped plans audited from poisoned buffers on a second input set.

test_gpu_plan_layers and test_gpu_plan_rows audit a plan on buffers that already hold the right answer: the graph
capture runs the op list twice eagerly on the same inputs before the replay that is checked, so an element a launch
fails to write still holds the correct value, and a read that overtakes its producer under programmatic dependent
launch (PDL) still finds it.  Here every byte of an op's result is first filled with 0xff (a NaN in bf16 and fp32),
every channel of a written buffer that holds no op's result with a large finite sentinel, and the plan then runs once
on a second input set:

  1. the graph replay, every op against fp64 within its bound (tests/bounds.py), and every op's output changed;
  2. the graph replay = an eager forward = forward(n) on the first n images, bit for bit, each from poisoned buffers,
     with the images at and after n left as they were poisoned;
  3. the plan with PDL on = the plan with PDL off (CTB_PDL=0, in a process of its own), op by op;
  4. a StreamRunner whose engine and records are overwritten before every step = one that is not, bit for bit;
  5. that the old protocol passes a plan with a launch left out, and this one names it.
"""
import gc
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import test_gpu_plan_layers as tpl
from centertrack_b200 import _lib as L
from centertrack_b200.engine import DeferredTV
from test_gpu_plan_layers import CASES, CHUNK, _build, _check_conv, _check_other
from test_gpu_plan_rows import _int_view, _written_buffers

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BY_ID = {c[0]: c for c in CASES}
SEED_A, SEED_B = 317, 4242    # input sets A (synthetic_inputs' default, which _build loads) and B
SENTINEL = 16384.0            # exact in bf16 and fp32: 2^14
A_MODE = {L.CT_A_CONV: '', L.CT_A_DCN: ' dcn', L.CT_A_DCN_WIN: ' dcn_win'}

# part 1: every kernel family and launch path the benchmarked plans select
FRESH_CASES = ['coco_tracking_512_b32_bf16', 'coco_tracking_512_b32_bf16x3',
               'mot_544x960_b32_bf16',                  # register gather at N = 256, window DCN at N = 128
               'nuscenes_ddd_448x800_b32_bf16',
               'coco_pose_512_b2_bf16x3',               # two-pass heads
               'coco_tracking_512_b1_fp32',             # SIMT convs, ct_stem_forward, fp32 upsample
               'coco_tracking_256_b2_bf16_dcn_global', 'coco_tracking_256_b2_bf16_no_halo',
               'kitti_tracking_384x1280_b2_bf16']       # a non-bench size: level 5's 12 x 40 ends in partial patches
PREFIX_CASES = ['mot_544x960_b32_bf16', 'coco_tracking_512_b32_bf16x3']
PDL_CASES = ['coco_tracking_512_b32_bf16', 'mot_544x960_b32_bf16x3']


# ---- what the plan writes --------------------------------------------------------------------------------------------
def _label(sp, seen):
  """The op's name, numbered from its second occurrence on (the plan has several ops named 'maxpool')."""
  n = seen[sp['name']] = seen.get(sp['name'], 0) + 1
  return sp['name'] if n == 1 else '%s#%d' % (sp['name'], n)


def _op_views(eng):
  """[(op label, view of the op's result)]; the fused head launch's intermediate, which no launch writes, is left
  out."""
  res, seen = [], {}
  for sp in eng.specs:
    o = sp['out']
    if isinstance(o, DeferredTV):
      continue
    if hasattr(o, 'buf'):                                  # a channel slice of an NHWC buffer
      res.append((_label(sp, seen), o.tensor()))
    elif sp.get('out_mode') == L.CT_OUT_NHWC_F32:         # the DCN offset / mask map: C_out of its 32 channels
      res.append((_label(sp, seen), o[..., :sp['desc'].C_out]))
    else:                                                 # fp32 NCHW head planes
      res.append((_label(sp, seen), o))
  return res


def _audited_views(eng):
  """_op_views, plus the fused head launch's intermediate as its record computes it from the current feature."""
  return _op_views(eng) + [(sp['name'], sp['out'].tensor()) for sp in eng.specs if isinstance(sp['out'], DeferredTV)]


def _unwritten_views(eng):
  """[(op names writing the buffer, view of a channel range of that NHWC buffer that holds no op's result)] -- the ld
  padding, the offset / mask map's channels 27..31.  The tensor-core engines store the offset / mask map's padded
  32-channel row whole (wgmma.cuh, store_f32_nhwc16), so its channels 27..31 are overwritten on the images those
  launches cover; the SIMT engine stores only the 27."""
  spans = {}
  for sp in eng.specs:
    o = sp['out']
    if isinstance(o, DeferredTV) or sp.get('out_mode') == L.CT_OUT_NCHW_F32:
      continue
    t, c0, c1 = (o.buf, o.off, o.off + o.C) if hasattr(o, 'buf') else (o, 0, sp['desc'].C_out)
    spans.setdefault(t.data_ptr(), (t, [], []))
    spans[t.data_ptr()][1].append((c0, c1))
    spans[t.data_ptr()][2].append(sp['name'])
  res = []
  for t, written, names in spans.values():
    c = 0
    for c0, c1 in sorted(written) + [(t.shape[-1], t.shape[-1])]:
      if c0 > c:
        res.append((','.join(names), t[..., c:c0]))
      c = max(c, c1)
  assert set(_written_buffers(eng)) == {p for p in spans} | {t.data_ptr() for t in eng.outputs.values()}
  return res


def poison(eng, images=slice(None), fill=None):
  """Overwrite images `images` of every buffer a launch of the plan writes: each op's output bytes with 0xff (a NaN in
  bf16 and fp32), or with the finite value `fill`; the channels of those buffers that hold no op's result with SENTINEL,
  which a launch reading them with a zero weight leaves exact and one mixing them into a result does not.  The
  fused-head planes (eng.outputs), the packed stem input and the DCN offset / mask maps are op outputs.  Engine inputs,
  weights and shifts are left alone."""
  for _, v in _op_views(eng):
    if fill is None:
      _int_view(v[images]).fill_(-1)
    else:
      v[images].fill_(fill)
  for _, v in _unwritten_views(eng):
    v[images].fill_(SENTINEL)


def _still_poisoned(v):
  """Elements of an op's output view that still hold the 0xff poison."""
  return _int_view(v) == -1


def _load(eng, seed):
  from centertrack_b200 import synthetic as syn
  img, pre, hm = syn.synthetic_inputs(eng.B, eng.H, eng.W, seed=seed)
  eng.in_img.copy_(img)
  eng.in_pre.copy_(pre)
  eng.in_hm.copy_(hm)


def _forget_deferred(eng):
  """The fused head launch's records read an intermediate that their audit computes on first use: drop it, so that
  the next audit recomputes it from the current 64-channel feature."""
  for sp in eng.specs:
    for k in ('out', 'x'):
      if isinstance(sp.get(k), DeferredTV):
        sp[k].holder['t'] = None


def _build_case(cid, monkeypatch):
  _, cfg, hw, B, precision, extra, kw, env = BY_ID[cid]
  return _build(cfg, hw, B, precision, extra, kw, monkeypatch, env)


def _release(eng):
  if eng is not None:
    eng.__dict__.clear()
  gc.collect()
  torch.cuda.empty_cache()


# ---- the per-op fp64 audit -------------------------------------------------------------------------------------------
def _family(eng, sp):
  if sp['kind'] != 'conv':
    return '%s %s' % (sp['kind'], eng.precision)
  out = ' fp32 out' if sp['out_mode'] in (L.CT_OUT_NHWC_F32, L.CT_OUT_NCHW_F32) else ''
  return tpl.KERNEL[sp['engine']] + A_MODE[sp['a_mode']] + out


def _audit(eng):
  """Every op of eng on every CHUNK of images against fp64, as test_plan_layers_within_bounds audits it ->
  (failure lines, names of the failing ops, {kernel family: (worst |err| / bound, op)})."""
  failures, failed, worst = [], set(), {}
  for sp in eng.specs:
    is_conv = sp['kind'] == 'conv'
    kern = tpl.KERNEL[sp['engine']] if is_conv else sp['kind']
    layer_worst, layer_at = 0.0, None
    for b0 in range(0, eng.B, CHUNK):
      bs = slice(b0, min(eng.B, b0 + CHUNK))
      if is_conv and sp['a_mode'] != L.CT_A_CONV and not bool(torch.isfinite(sp['om'][bs, ..., :27]).all()):
        # the fp64 sampler turns offsets into gather indices: a NaN one has no reference (the kernel samples zero)
        failures.append('%s (%s): the offset / mask map it read is not finite' % (sp['name'], kern))
        failed.add(sp['name'])
        break
      try:
        res = _check_conv(eng, sp, bs) if is_conv else _check_other(eng, sp, bs)
      except AssertionError as e:                         # the exact kinds (pack, pool) assert
        failures.append('%s (%s): %s' % (sp['name'], kern, str(e).split('\n')[0]))
        failed.add(sp['name'])
        break
      if res is None:
        continue
      m, at = tpl.bd.worst(res[0])
      if m > layer_worst or layer_at is None:
        layer_worst, layer_at = m, dict(at, b=at['b'] + b0)
      del res
    fam = _family(eng, sp)
    if layer_at is None:
      if sp['name'] not in failed:                       # pack / pool: checked exactly
        worst.setdefault(fam + ' (exact)', (0.0, sp['name']))
      continue
    if layer_worst > worst.get(fam, (-1.0, ''))[0]:
      worst[fam] = (layer_worst, sp['name'])
    if not layer_worst <= 1.0:
      failures.append('%s (%s, N=%s): worst element %s, |err| / bound = %.3g' % (
          sp['name'], kern, sp.get('n_tile', '-'), layer_at, layer_worst))
      failed.add(sp['name'])
  return failures, failed, worst


# ---- 1. per-op fp64 audit on a second input set from poisoned buffers ------------------------------------------------
@pytest.mark.parametrize('cid', FRESH_CASES)
def test_plan_on_new_inputs_from_poisoned_buffers(cid, monkeypatch):
  """Build on input set A (one captured graph), keep the first CHUNK images of every op's output, poison, load input set
  B and replay the graph once: no output byte may still hold the poison, every op must lie within its fp64 bound, and
  every op's output must have changed from set A on most of its non-zero elements (it really computed on new data)."""
  eng = None
  try:
    eng = _build_case(cid, monkeypatch)
    tpl._assert_no_overlapping_writes(eng)
    n0 = min(CHUNK, eng.B)
    before = {name: v[:n0].clone() for name, v in _audited_views(eng)}
    poison(eng)
    _forget_deferred(eng)
    _load(eng, SEED_B)
    eng.replay()
    torch.cuda.synchronize()
    unwritten = []
    for name, v in _op_views(eng):
      n = int(_still_poisoned(v).sum())
      if n:
        unwritten.append('%s: %d of %d elements still hold the poison' % (name, n, v.numel()))
    assert not unwritten, '%s: the replay left bytes unwritten:\n  %s' % (cid, '\n  '.join(unwritten))
    failures, _, worst = _audit(eng)
    print('\n[%s] %d ops from poisoned buffers on input set B; worst |err| / bound per kernel family:' % (
        cid, len(eng.specs)))
    for fam, (w, name) in sorted(worst.items()):
      print('  %-28s %.3f (%s)' % (fam, w, name))
    assert not failures, '%s: %d ops out of bounds:\n  %s' % (cid, len(failures), '\n  '.join(failures))
    after = dict(_audited_views(eng))
    stale, fracs = [], []
    for name, old in before.items():
      new = after[name][:n0]
      nz = old != 0
      frac = float(((new != old) & nz).sum()) / max(1, int(nz.sum()))
      fracs.append('%s %.3f' % (name, frac))
      if not frac > 0.5:
        stale.append('%s: %.3f of its non-zero elements changed' % (name, frac))
    print('  fraction of non-zero elements changed from input set A, per op (images 0-%d):\n    %s' % (
        n0 - 1, '\n    '.join(fracs)))
    assert not stale, '%s: ops whose output did not follow the new inputs:\n  %s' % (cid, '\n  '.join(stale))
  finally:
    _release(eng)


# ---- 2. graph = eager = batch prefix, each from poisoned buffers -----------------------------------------------------
def _sentinel_intact(eng, images):
  """Problems where the channels that hold no op's result no longer hold SENTINEL on images `images`."""
  return ['%s: channels outside every op\'s result changed' % names for names, v in _unwritten_views(eng)
          if not bool((v[images] == SENTINEL).all())]


@pytest.mark.parametrize('cid', PREFIX_CASES)
def test_graph_eager_and_prefix_agree_from_poisoned_buffers(cid, monkeypatch):
  """Input set B: one graph replay; then from poisoned buffers an eager forward, which must equal the replay bit for
  bit on every byte a launch writes; then for n = 1, 13 and B - 1, every image poisoned and nothing restored,
  forward(n): images < n equal the replay bit for bit, images >= n keep the poison (and the sentinel) byte for byte."""
  eng = None
  try:
    eng = _build_case(cid, monkeypatch)
    B = eng.B
    _load(eng, SEED_B)
    eng.replay()
    torch.cuda.synchronize()
    full = {name: v.clone() for name, v in _op_views(eng)}
    poison(eng)
    eng.forward(eng.in_img, eng.in_pre, eng.in_hm)
    torch.cuda.synchronize()
    bad = ['%s differs from the graph replay' % name for name, v in _op_views(eng)
           if not torch.equal(_int_view(v), _int_view(full[name]))]
    assert not bad, '%s: eager forward from poisoned buffers:\n  %s' % (cid, '\n  '.join(bad))
    for n in (1, 13, B - 1):
      poison(eng)
      eng.forward(eng.in_img[:n], eng.in_pre[:n], eng.in_hm[:n], n=n)
      torch.cuda.synchronize()
      bad = []
      for name, v in _op_views(eng):
        if not torch.equal(_int_view(v[:n]), _int_view(full[name][:n])):
          diff = (_int_view(v[:n]) != _int_view(full[name][:n])).reshape(n, -1).any(1)
          left = int(_still_poisoned(v[:n]).sum())
          bad.append('%s: images %s differ from the B = %d replay (%d elements still poisoned)' % (
              name, diff.nonzero().flatten().tolist()[:8], B, left))
        if not bool(_still_poisoned(v[n:]).all()):
          hit = (~_still_poisoned(v[n:])).reshape(B - n, -1).any(1)
          bad.append('%s: images %s written' % (name, (hit.nonzero().flatten() + n).tolist()[:8]))
      bad += _sentinel_intact(eng, slice(n, None))
      assert not bad, '%s: forward(n=%d) from poisoned buffers:\n  %s' % (cid, n, '\n  '.join(bad))
    print('\n[%s] graph replay = eager forward = forward(n) for n = 1, 13, %d, from poisoned buffers' % (cid, B - 1))
  finally:
    _release(eng)


# ---- 3. PDL on and off give the same bytes ---------------------------------------------------------------------------
def _digests(cid, monkeypatch):
  """{op name: SHA-256 of every byte its launch writes} after one graph replay on input set B from poisoned buffers."""
  eng = None
  try:
    eng = _build_case(cid, monkeypatch)
    poison(eng)
    _load(eng, SEED_B)
    eng.replay()
    torch.cuda.synchronize()
    return {name: hashlib.sha256(_int_view(v).contiguous().cpu().numpy().tobytes()).hexdigest()
            for name, v in _op_views(eng)}
  finally:
    _release(eng)


DIGESTS = 'op digests: '


def _digest_child(cid):
  """Entry point of the other-PDL process (test_pdl_off_equals_pdl_on)."""
  with pytest.MonkeyPatch.context() as mp:
    print(DIGESTS + json.dumps(_digests(cid, mp)))


@pytest.mark.parametrize('cid', PDL_CASES)
def test_pdl_off_equals_pdl_on(cid, monkeypatch):
  """The plan's launches with PDL (this process, unless CTB_PDL=0) and stream-serialised (a child process with the
  other setting: the library reads CTB_PDL once per process): every op's output bytes equal.  The kernels are
  deterministic, so a difference is a read that overtook its producer."""
  pdl_here = int(os.environ.get('CTB_PDL', '1')) != 0
  mine = _digests(cid, monkeypatch)
  env = dict(os.environ, CTB_PDL='0' if pdl_here else '1')
  paths = [ROOT, os.path.join(ROOT, 'oracle'), os.path.join(ROOT, 'tests')]
  code = 'import sys; sys.path[:0] = %r; import test_gpu_plan_fresh_state as t; t._digest_child(%r)' % (paths, cid)
  r = subprocess.run([sys.executable] + (['-s'] if sys.flags.no_user_site else []) + ['-c', code], cwd=ROOT, env=env,
                     capture_output=True, text=True)
  assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
  theirs = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith(DIGESTS)][-1][len(DIGESTS):])
  assert sorted(theirs) == sorted(mine)
  differ = [name for name in mine if mine[name] != theirs[name]]
  print('\n[%s] %d ops, PDL %s here and %s in the child: %d op digests equal%s' % (
      cid, len(mine), 'on' if pdl_here else 'off', 'off' if pdl_here else 'on', len(mine) - len(differ),
      '; differ: ' + ', '.join(differ) if differ else ''))
  assert not differ, '%s: ops whose output depends on PDL: %s' % (cid, ', '.join(differ))


# ---- 4. a StreamRunner step depends only on its declared state -------------------------------------------------------
RH, RW, RK, RB = 128, 160, 40, 4
SIZES = [(120, 200), (97, 131), (160, 128), (120, 200)]
MAXF = (160, 200)
# per step: (idle streams, resumed streams); step 2 runs the network at n = 3 (forward(n) under the runner)
SCHEDULE = [([], []), ([], []), ([1], []), ([], [1]), ([], [])]


@pytest.mark.parametrize('precision', ['bf16', 'bf16x3'])
def test_stream_step_ignores_poisoned_activations(precision):
  """Two frames-mode device-tracking runners of two models built from the same seeded state dict (no engine buffer in
  common), over the same 5-frame B = 4 video with one idle step: before every step the second runner's engine outputs
  and decode records are overwritten with -3.0 (what the runner carries between frames -- frame slots, pre_hm, track
  tables -- is left alone).  Records and tracks must be bit-identical after every step."""
  from helpers import make_model
  from test_gpu_frames import _frame
  from centertrack_b200.runner import StreamRunner
  runners = []
  for _ in range(2):
    opt, model, _ = make_model('mot', extra=['--track_thresh', '0.1', '--new_thresh', '0.1', '--pre_thresh', '0.1',
                                             '--input_h', str(RH), '--input_w', str(RW), '--max_age', '2'])
    r = StreamRunner(model.cuda(), RB, RH, RW, K=RK, precision=precision, device='cuda', opt=opt, device_tracking=True,
                     frame_sizes=SIZES, max_frame_size=MAXF, idle_streams=1)
    r.warm()
    runners.append(r)
  ref, got = runners
  assert ref.eng is not got.eng and ref.eng.outputs['hm'].data_ptr() != got.eng.outputs['hm'].data_ptr()
  u32 = lambda a: np.ascontiguousarray(a).view(np.uint32)
  tracks = 0
  for k, (idle, resume) in enumerate(SCHEDULE):
    frames = [None if b in idle else _frame(*SIZES[b], seed=100 * k + b) for b in range(RB)]
    poison(got.eng, fill=-3.0)
    got.rec.fill_(-3.0)
    torch.cuda.synchronize()
    prev = [r.step_frames(frames, idle=idle, resume=resume or None) for r in runners]
    assert got._n == RB - len(idle)
    if k:
      assert np.array_equal(u32(prev[0]), u32(prev[1])), 'step %d: records of the step before differ' % k
    assert np.array_equal(u32(ref.fetch()), u32(got.fetch())), 'step %d: records differ' % k
    (ta, ca), (tb, cb) = ref.fetch_tracks(), got.fetch_tracks()
    assert np.array_equal(u32(ta), u32(tb)) and np.array_equal(u32(ca), u32(cb)), 'step %d: tracks differ' % k
    tracks += int(ca[:, 0].sum())
  assert tracks > 0
  print('\n[%s] %d steps, %d track rows, the poisoned runner bit-identical to the clean one' % (
      precision, len(SCHEDULE), tracks))


# ---- 5. the old protocol misses a skipped launch, the new one names it -----------------------------------------------
def _region(t):
  """(buffer identity, first channel, end channel) of an operand or output; a plain tensor as a whole."""
  if isinstance(t, DeferredTV):
    return (id(t.holder), t.off, t.off + t.C)
  if hasattr(t, 'buf'):
    return (t.buf.data_ptr(), t.off, t.off + t.C)
  return (t.data_ptr(), 0, 1 << 30)


def _downstream(eng, names):
  """Names of the ops that read, directly or through other ops, what ops `names` write."""
  tainted, out = [_region(sp['out']) for sp in eng.specs if sp['name'] in names], set()
  for sp in eng.specs:
    reads = [_region(sp[k]) for k in ('x', 'residual', 'om', 'skip') if sp.get(k) is not None]
    if any(p == q and a0 < b1 and b0 < a1 for p, a0, a1 in reads for q, b0, b1 in tainted):
      out.add(sp['name'])
      tainted.append(_region(sp['out']))
  return out


def test_fresh_state_catches_a_skipped_launch(monkeypatch):
  """coco_tracking 256 x 256 bf16, B = 2, with one launch left out of the op list: a window DCN conv, then the fused
  head launch.  The old protocol (warm up on inputs A, run the short op list on the same inputs) passes the audit; from
  poisoned buffers on inputs B the audit fails the skipped op (for the head launch: its planes), and nothing but it and
  the ops downstream of it."""
  eng = _build('coco_tracking', (256, 256), 2, 'bf16', [], {}, monkeypatch, {})
  all_ops = list(eng.ops)
  assert any(name == 'heads' for _, _, name in all_ops), 'the plan runs the fused head launch'
  dcn = [sp['name'] for sp in eng.specs if sp['kind'] == 'conv' and sp['a_mode'] == L.CT_A_DCN_WIN]
  assert dcn, 'the plan runs window DCN convs'
  for skip in (dcn[len(dcn) // 2], 'heads'):
    records = set(eng.head_names) if skip == 'heads' else {skip}    # the fused launch's records: the 1x1 head planes
    _load(eng, SEED_A)
    monkeypatch.setattr(eng, 'ops', all_ops)
    eng.forward(eng.in_img, eng.in_pre, eng.in_hm)                   # warm-up on inputs A
    monkeypatch.setattr(eng, 'ops', [op for op in all_ops if op[2] != skip])
    eng.forward(eng.in_img, eng.in_pre, eng.in_hm)                   # old protocol: the same inputs, no poison
    torch.cuda.synchronize()
    _forget_deferred(eng)
    failures, failed, _ = _audit(eng)
    assert not failures, 'old protocol, %s skipped: the audit was expected to pass:\n  %s' % (skip,
                                                                                            '\n  '.join(failures))
    poison(eng)
    _load(eng, SEED_B)
    eng.forward(eng.in_img, eng.in_pre, eng.in_hm)                   # new protocol: poisoned buffers, inputs B
    torch.cuda.synchronize()
    _forget_deferred(eng)
    failures, failed, _ = _audit(eng)
    down = _downstream(eng, records)
    print('\n[%s skipped] old protocol: audit passes; from poisoned buffers on inputs B it fails %d ops: %s'
          '\n  downstream ops that still pass: %s' % (skip, len(failed), ', '.join(sorted(failed)),
                                                      ', '.join(sorted(down - failed)) or 'none'))
    assert records <= failed, '%s skipped: the audit does not report %s' % (skip, sorted(records - failed))
    assert failed <= records | down, '%s skipped: the audit reports ops not downstream of it: %s' % (
        skip, sorted(failed - records - down))
    if skip == 'heads':
      assert failed == records
    else:
      assert failed - records, '%s skipped: no op downstream of it fails' % skip
