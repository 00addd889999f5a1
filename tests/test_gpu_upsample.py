"""-m gpu: ct_upsample_add -- IDAUp's depthwise ConvTranspose2d(2f, stride f, pad f/2) + skip -- at irregular map shapes.

Three kernels compute it (csrc/elementwise.cu):
  * the warp kernel, which every plan runs: all f*f phases of an input pixel in one CTA, a grid-stride walk over the
    input pixels whose (b, m, n) advance by the stride with carries over rows and images;
  * the phase kernel, selected by CTB_UP_MODE=0, which the library reads once per process: run in a child process;
  * the plain kernel, for channel counts whose 16-byte vectors do not divide 256 (bf16 C = 48, fp32 C = 24).
Each result is held to an fp64 conv_transpose2d + skip with the GAMMA_SIMT bound (fp32 accumulation of four taps and
the skip), at every (dtype, C, f) the plans run, on maps of one row, one column, odd sizes, and B H W several times the
warp kernel's grid; with and without a skip; on channel slices of wider buffers whose other channels hold NaN, which
must stay untouched.  The kernels accumulate in the same order, so the phase kernel must equal the warp kernel bit for
bit, and the plain kernel must equal the warp kernel on the same channels padded to a width the warp kernel takes.
"""
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import bounds as bd
from centertrack_b200 import _lib as L

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DT = {'bf16': (torch.bfloat16, L.CT_BF16, 8), 'f32': (torch.float32, L.CT_F32, 4)}   # dtype, code, 16-byte vector

# (dtype, C, f): the 'up' rows of the plans (tests/plan_rows.py), and the two plain-kernel widths
PLAN_ROWS = [('bf16', 64, 2), ('bf16', 64, 4), ('bf16', 128, 2), ('bf16', 256, 2),
             ('f32', 64, 2), ('f32', 64, 4), ('f32', 128, 2), ('f32', 256, 2)]
PLAIN_ROWS = [('bf16', 48, 2), ('bf16', 48, 4), ('f32', 24, 2), ('f32', 24, 4)]
# (B, H, W): one pixel, one row, one column, odd sizes, and B H W = 29391: 3.5 to 28 times the input pixels one pass of
# the warp kernel's grid covers (1056 CTAs on 132 SMs, of 1 to 8 input pixels each), with a stride that is no multiple
# of W or H, so that the walk carries over rows and images at every step
SHAPES = [(1, 1, 1), (3, 1, 7), (2, 5, 1), (2, 7, 13), (3, 97, 101)]
# (skip, channel slices): a plain tensor with a skip, one without, and slices of wider NaN-filled buffers
LAYOUTS = ['skip', 'no_skip', 'sliced']


def _case_ids():
  return ['%s_c%d_f%d' % r for r in PLAN_ROWS + PLAIN_ROWS]


def _buffer(B, H, W, C, ld, off, dt, gen, scale=1.0):
  """A [B, H, W, ld] NaN-filled buffer whose channels off .. off + C hold N(0, scale) values (exact in dt)."""
  buf = torch.full((B, H, W, ld), float('nan'), dtype=dt)
  buf[..., off:off + C] = (torch.randn(B, H, W, C, generator=gen, dtype=torch.float64) * scale).to(dt)
  return buf.cuda()


def _inputs(row, shape, layout, seed=7):
  """(x, skip, w, out buffers with their channel offsets and ld) of one case."""
  dtype, C_, f = row
  dt, _, V = DT[dtype]
  B, H, W = shape
  gen = torch.Generator().manual_seed(seed + 1000 * C_ + 100 * f + H * 7 + W)
  sliced = layout == 'sliced'
  lx, ls, lo = (C_ + 2 * V, C_ + 3 * V, C_ + V) if sliced else (C_, C_, C_)
  ox, os_, oo = (V, 2 * V, 0) if sliced else (0, 0, 0)
  x = _buffer(B, H, W, C_, lx, ox, dt, gen)
  skip = _buffer(B, H * f, W * f, C_, ls, os_, dt, gen) if layout != 'no_skip' else None
  w = (torch.randn(C_, 1, 2 * f, 2 * f, generator=gen, dtype=torch.float64) * 0.5).float()
  out = torch.full((B, H * f, W * f, lo), float('nan'), dtype=dt).cuda()
  return (x, ox, lx), (skip, os_, ls), w, (out, oo, lo)


def _launch(row, B, H, W, xs, ss, w, os_):
  dtype, C_, f = row
  (x, ox, lx), (skip, osk, ls), (out, oo, lo) = xs, ss, os_
  e = x.element_size()
  wk = w.reshape(C_, 2 * f, 2 * f).permute(1, 2, 0).contiguous().cuda()          # channel-last [2f][2f][C]
  rc = L.lib().ct_upsample_add(C.c_void_p(x.data_ptr() + ox * e),
                               C.c_void_p(skip.data_ptr() + osk * e) if skip is not None else None,
                               C.c_void_p(wk.data_ptr()), C.c_void_p(out.data_ptr() + oo * e), DT[dtype][1],
                               B, H, W, C_, f, lx, ls, lo, L.stream_ptr())
  L.check(rc, 'ct_upsample_add %s' % (row,))
  torch.cuda.synchronize()


def _run(row, shape, layout):
  """The case's output buffer after one launch."""
  xs, ss, w, os_ = _inputs(row, shape, layout)
  _launch(row, *shape, xs, ss, w, os_)
  return xs, ss, w, os_


def _check(row, shape, layout, xs, ss, w, os_):
  """-> [problems]: the result within the fp64 bound, the channels around the slice still NaN."""
  dtype, C_, f = row
  (x, ox, _), (skip, osk, _), (out, oo, _) = xs, ss, os_
  xd = x[..., ox:ox + C_].permute(0, 3, 1, 2).double()
  wd = w.double().cuda()
  ref = F.conv_transpose2d(xd, wd, None, stride=f, padding=f // 2, groups=C_)
  mag = F.conv_transpose2d(xd.abs(), wd.abs(), None, stride=f, padding=f // 2, groups=C_)
  if skip is not None:
    s = skip[..., osk:osk + C_].permute(0, 3, 1, 2).double()
    ref, mag = ref + s, mag + s.abs()
  got = out[..., oo:oo + C_].permute(0, 3, 1, 2)
  m, at = bd.worst(bd.ratio(got, ref, mag, bd.GAMMA_SIMT, dtype == 'bf16'))
  bad = []
  if not m <= 1.0:
    bad.append('%s %s %s: worst element %s, |err| / bound = %.3g' % (row, shape, layout, at, m))
  rest = torch.cat([out[..., :oo], out[..., oo + C_:]], -1)
  if not bool(torch.isnan(rest).all()):
    bad.append('%s %s %s: channels outside the slice written' % (row, shape, layout))
  return bad, m


@pytest.mark.parametrize('row', PLAN_ROWS + PLAIN_ROWS, ids=_case_ids())
def test_upsample_add_within_bounds(row):
  bad, worst = [], 0.0
  for shape in SHAPES:
    for layout in LAYOUTS:
      b, m = _check(row, shape, layout, *_run(row, shape, layout))
      bad += b
      worst = max(worst, m)
  print('\n[%s C=%d f=%d] %d shapes x %d layouts: worst |err| / bound %.3f' % (row + (len(SHAPES), len(LAYOUTS), worst)))
  assert not bad, '\n'.join(bad)


def _bits(t):
  return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


@pytest.mark.parametrize('row', PLAIN_ROWS, ids=['%s_c%d_f%d' % r for r in PLAIN_ROWS])
def test_plain_kernel_equals_warp_kernel(row):
  """The plain kernel (C = 48 bf16 / 24 fp32) = the warp kernel on the same channels padded to 64 / 32 with zeros,
  bit for bit on those channels: depthwise, so the padding changes no other channel."""
  dtype, C_, f = row
  wide = (dtype, C_ + DT[dtype][2] * 2, f)
  for shape in SHAPES:
    xs, ss, w, os_ = _run(row, shape, 'skip')
    pad = lambda t: F.pad(t, (0, wide[1] - C_))
    x2, s2 = pad(xs[0]).contiguous(), pad(ss[0]).contiguous()
    w2 = torch.cat([w, torch.zeros(wide[1] - C_, *w.shape[1:])], 0)
    o2 = torch.full((*os_[0].shape[:3], wide[1]), float('nan'), dtype=os_[0].dtype, device='cuda')
    _launch(wide, *shape, (x2, 0, wide[1]), (s2, 0, wide[1]), w2, (o2, 0, wide[1]))
    assert torch.equal(_bits(o2[..., :C_]), _bits(os_[0])), '%s %s: plain and warp kernels differ' % (row, shape)


# ---- the phase kernel (CTB_UP_MODE=0) --------------------------------------------------------------------------------
DIGESTS = 'upsample digests: '


def _digests():
  """{case: SHA-256 of its output buffer} over every plan row, shape and layout."""
  res = {}
  for row in PLAN_ROWS:
    for shape in SHAPES:
      for layout in LAYOUTS:
        out = _run(row, shape, layout)[3][0]
        res['%s %s %s' % (row, shape, layout)] = hashlib.sha256(_bits(out).cpu().numpy().tobytes()).hexdigest()
  return res


def _digest_child():
  print(DIGESTS + json.dumps(_digests()))


def test_phase_kernel_equals_warp_kernel():
  """The same cases with the other CTB_UP_MODE in a child process: every output byte equal, the NaN around the slices
  included."""
  mode_here = int(os.environ.get('CTB_UP_MODE', '1'))
  mine = _digests()
  env = dict(os.environ, CTB_UP_MODE='0' if mode_here == 1 else '1')
  paths = [ROOT, os.path.join(ROOT, 'oracle'), os.path.join(ROOT, 'tests')]
  code = 'import sys; sys.path[:0] = %r; import test_gpu_upsample as t; t._digest_child()' % (paths,)
  r = subprocess.run([sys.executable] + (['-s'] if sys.flags.no_user_site else []) + ['-c', code], cwd=ROOT, env=env,
                     capture_output=True, text=True)
  assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
  theirs = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith(DIGESTS)][-1][len(DIGESTS):])
  assert sorted(theirs) == sorted(mine)
  differ = [k for k in mine if mine[k] != theirs[k]]
  print('\n%d cases, CTB_UP_MODE %d here and %s in the child: %d equal' % (len(mine), mode_here, env['CTB_UP_MODE'],
                                                                           len(mine) - len(differ)))
  assert not differ, 'phase and warp kernels differ on: %s' % ', '.join(differ[:10])
