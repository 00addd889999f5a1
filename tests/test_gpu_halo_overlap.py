"""-m gpu: the halo kernel's one-CTA-per-SM flavour (the two warpgroups' MMA chains take turns, so one warpgroup's epilogue
overlaps the other's MMAs) computes bit-for-bit what the serial schedule computes (CTB_HALO_OVERLAP=0).  The switch is
read once per process, so each schedule runs in a process of its own and writes its outputs to a file."""
import os
import subprocess
import sys

import pytest
import torch

import bounds as bd
from centertrack_b200 import _lib as L

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

# (name, B, C_in, C_out, H, W, k, residual, n_tile, output).  Every shape takes the overlapped path (asserted below from
# the library's configuration); the sizes give the persistent CTAs (132 on an H100 SXM) a mix of 1 and 2 work items,
# and 8-9 (heads.0) or 3-4 (3x3 64 -> 160) items.
CASES = [
    ('heads.0 3x3 64->1024 nt128', 1, 64, 1024, 176, 104, 3, False, 128, 'nhwc'),
    ('3x3 64->160 +res nt80', 8, 64, 160, 64, 64, 3, True, 80, 'nhwc'),
    ('level2 3x3 64->64 +res nt64', 1, 64, 64, 176, 104, 3, True, 64, 'nhwc'),
    ('3x3 64->64 nt64 space-to-depth output', 1, 64, 64, 176, 104, 3, False, 64, 's2d'),
    ('tree1.conv1 2x2 128->64 nt64', 3, 128, 64, 80, 120, 2, False, 64, 'nhwc'),
    ('3x3 64->27 nt64 fp32 NHWC sigmoid (offset map)', 3, 64, 27, 96, 88, 3, False, 64, 'f32_nhwc'),
    ('hm 1x1 256->80 nt80 fp32 NCHW sigmoid, 32x4 tiles', 2, 256, 80, 100, 96, 1, False, 80, 'nchw_sigmoid'),
    ('hm 1x1 256->80 nt80 fp32 NCHW sigmoid, 8x16 tiles', 2, 256, 80, 48, 40, 1, False, 80, 'nchw_sigmoid'),
    ('1x1 256->98 nt112 fp32 NCHW', 2, 256, 98, 100, 96, 1, False, 112, 'nchw'),
    ('1x1 256->128 nt128', 1, 256, 128, 176, 104, 1, False, 128, 'nhwc'),
    ('3x3 64->176 +res nt96 (ragged second n-tile)', 1, 64, 176, 120, 72, 3, True, 96, 'nhwc'),
]


def _inputs(case, seed):
  name, B, Cin, Cout, H, W, k, res, nt, out = case
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(B, Cin, H, W, generator=g)
  w = torch.randn(Cout, Cin, k, k, generator=g) * (2.0 / (Cin * k * k)) ** 0.5
  b = torch.randn(Cout, generator=g) * 0.1
  r = torch.randn(B, Cout, H, W, generator=g) if res else None
  return x, w, b, r


def _conv_args(case, seed):
  """(args, keyword args) of gpu_helpers.run_conv / conv_desc for this case."""
  name, B, Cin, Cout, H, W, k, res, nt, out = case
  x, w, b, r = _inputs(case, seed)
  kw = {'nhwc': {}, 's2d': dict(out_mode=L.CT_OUT_NHWC_S2D),
        'f32_nhwc': dict(out_mode=L.CT_OUT_NHWC_F32, sig_from=18),
        'nchw_sigmoid': dict(out_mode=L.CT_OUT_NCHW_F32, head_act=1), 'nchw': dict(out_mode=L.CT_OUT_NCHW_F32)}[out]
  relu = out in ('nhwc', 's2d')
  return (L.CT_ENGINE_TCGEN05_HALO, L.CT_BF16, x.cuda(), w, b, 1, relu, r.cuda() if res else None), dict(kw, n_tile=nt)


def _run(case, seed):
  from gpu_helpers import run_conv
  args, kw = _conv_args(case, seed)
  return run_conv(*args, **kw)


def dump_cases(path):
  torch.save({c[0]: _run(c, 500 + i).cpu() for i, c in enumerate(CASES)}, path)


def dump_plan(path):
  """coco_tracking 512x512 at B = 32, one graph replay with the fused activations: head maps and decode records."""
  from helpers import make_model
  from centertrack_b200 import synthetic as syn
  from centertrack_b200.decode import generic_decode
  opt, model, _ = make_model('coco_tracking')
  dev = torch.device('cuda')
  model = model.to(dev)
  B, H, W = 32, 512, 512
  eng = model.engine_for(B, H, W, dev, 'bf16')
  img, pre, hm = syn.synthetic_inputs(B, H, W)
  eng.in_img.copy_(img)
  eng.in_pre.copy_(pre)
  eng.in_hm.copy_(hm)
  eng.set_fused_activations(True)
  eng.replay()
  out = {k: v.clone() for k, v in eng.outputs.items()}
  dets = generic_decode(out, K=100)
  torch.cuda.synchronize()
  res = {'head_' + k: v.cpu() for k, v in out.items()}
  res['records'] = dets.records.cpu()
  torch.save(res, path)


def _in_process(fn, path, overlap):
  code = ('import sys; sys.path[:0] = %r; import test_gpu_halo_overlap as t; t.%s(%r)' %
          ([ROOT, HERE, os.path.join(ROOT, 'oracle')], fn, str(path)))
  r = subprocess.run([sys.executable, '-c', code], cwd=ROOT, env=dict(os.environ, CTB_HALO_OVERLAP=overlap),
                     capture_output=True, text=True)
  assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
  return torch.load(path)


def test_one_cta_halo_shapes_bit_identical_to_serial(tmp_path):
  from gpu_helpers import conv_desc
  for i, c in enumerate(CASES):
    args, kw = _conv_args(c, 500 + i)
    cfg = L.conv_config(conv_desc(*args, **kw)[0])
    assert cfg.ctas_per_sm == 1 and cfg.overlap == 1, c[0]
  got = _in_process('dump_cases', tmp_path / 'overlap.pt', '1')
  serial = _in_process('dump_cases', tmp_path / 'serial.pt', '0')
  for i, c in enumerate(CASES):
    name, B, Cin, Cout, H, W, k, res, nt, out = c
    assert torch.equal(got[name], serial[name]), name
    x, w, b, r = _inputs(c, 500 + i)
    q = lambda t: t.bfloat16().double().cuda() if t is not None else None
    p = (1, 0, 1, 0) if k == 2 else (k // 2,) * 4
    ref, mag = bd.conv_ref(q(x), q(w.float()), b, q(r), 1, p)
    o = got[name]
    if out == 'f32_nhwc':
      bd.assert_bound(o[:, :18], ref[:, :18], mag[:, :18], bd.ALPHA_BF16, False, name + ' offsets')
      bd.assert_bound(o[:, 18:27], ref[:, 18:], mag[:, 18:], bd.ALPHA_BF16, False, name + ' mask', 'sigmoid')
    elif out.startswith('nchw'):
      bd.assert_bound(o, ref, mag, bd.ALPHA_BF16, False, name, 'sigmoid' if out == 'nchw_sigmoid' else 'none')
    else:
      bd.assert_bound(o, ref, mag, bd.ALPHA_BF16, True, name, 'relu')


def test_coco_tracking_plan_bit_identical_to_serial(tmp_path):
  got = _in_process('dump_plan', tmp_path / 'overlap.pt', '1')
  serial = _in_process('dump_plan', tmp_path / 'serial.pt', '0')
  assert sorted(got) == sorted(serial) and 'records' in got and 'head_hm' in got
  for k in got:
    assert torch.equal(got[k], serial[k]), k
