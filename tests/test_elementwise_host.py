"""Host checks of the pooling and up-sampling entry points (no GPU): ct_upsample_add, ct_maxpool2 and ct_maxpool2_s2d
refuse empty or negative shapes and row strides narrower than the channels they cover.  With B < 0 the kernels'
(size_t)B * ... element count wraps to an enormous grid-stride range, and a stride below C makes pixels overlap.

The calls run in a child process that sees no CUDA device, on stand-in pointers: the refusals must come back as
CT_ERR_INVALID with their messages before any CUDA call.  An accepted call there fails at the launch with
CT_ERR_CUDA instead, which the control call of each entry point shows."""
import json
import os
import subprocess
import sys

import pytest

from centertrack_b200 import _lib as L

_CALLS = r"""
import ctypes as C, json
from centertrack_b200 import _lib as L
lib = L.lib()
p = C.c_void_p(1 << 20)
w = C.c_void_p(1 << 21)
BF, F32 = L.CT_BF16, L.CT_F32
res = []
def up(B, H, W, Cn, ld_in, ld_skip, ld_out, skip=True, dtype=BF, f=2):
  return lib.ct_upsample_add(p, p if skip else None, w, p, dtype, B, H, W, Cn, f, ld_in, ld_skip, ld_out, None)
def pool(B, H, W, Cn, ld_in, ld_out, dtype=BF):
  return lib.ct_maxpool2(p, p, dtype, B, H, W, Cn, ld_in, ld_out, None)
def s2d(B, H2, W2, Cn, ld_in, ld_out, dtype=BF):
  return lib.ct_maxpool2_s2d(p, p, dtype, B, H2, W2, Cn, ld_in, ld_out, None)
CASES = [
  ('up', 'control', lambda: up(2, 4, 6, 64, 64, 64, 64)),
  ('up', 'B = 0', lambda: up(0, 4, 6, 64, 64, 64, 64)),
  ('up', 'B < 0', lambda: up(-2, 4, 6, 64, 64, 64, 64)),
  ('up', 'H = 0', lambda: up(2, 0, 6, 64, 64, 64, 64)),
  ('up', 'W < 0', lambda: up(2, 4, -6, 64, 64, 64, 64)),
  ('up', 'C = 0', lambda: up(2, 4, 6, 0, 64, 64, 64)),
  ('up', 'ld_in < C', lambda: up(2, 4, 6, 64, 56, 64, 64)),
  ('up', 'ld_skip < C', lambda: up(2, 4, 6, 64, 64, 56, 64)),
  ('up', 'ld_out < C', lambda: up(2, 4, 6, 64, 64, 64, 56)),
  ('up', 'ld_out < C fp32', lambda: up(2, 4, 6, 32, 32, 32, 28, dtype=F32)),
  ('up', 'control, no skip, ld_skip 0', lambda: up(2, 4, 6, 64, 64, 0, 64, skip=False)),
  ('pool', 'control', lambda: pool(2, 4, 6, 64, 64, 64)),
  ('pool', 'B = 0', lambda: pool(0, 4, 6, 64, 64, 64)),
  ('pool', 'B < 0', lambda: pool(-2, 4, 6, 64, 64, 64)),
  ('pool', 'H < 0', lambda: pool(2, -4, 6, 64, 64, 64)),
  ('pool', 'ld_in < C', lambda: pool(2, 4, 6, 64, 56, 64)),
  ('pool', 'ld_out < C', lambda: pool(2, 4, 6, 64, 64, 56)),
  ('pool', 'ld_out < C fp32', lambda: pool(2, 4, 6, 32, 32, 28, dtype=F32)),
  ('s2d', 'control', lambda: s2d(2, 4, 6, 16, 64, 16)),
  ('s2d', 'B = 0', lambda: s2d(0, 4, 6, 16, 64, 16)),
  ('s2d', 'B < 0', lambda: s2d(-2, 4, 6, 16, 64, 16)),
  ('s2d', 'W2 = 0', lambda: s2d(2, 4, 0, 16, 64, 16)),
  ('s2d', 'ld_out < C', lambda: s2d(2, 4, 6, 16, 64, 8)),
]
for op, what, call in CASES:
  rc = call()
  res.append((op, what, rc, lib.ct_last_error().decode()))
print(json.dumps(res))
"""

MESSAGE = {'B': 'bad shape', 'H': 'bad shape', 'W': 'bad shape', 'W2': 'bad shape', 'C': 'bad shape', 'ld_in': 'ld_in',
           'ld_skip': 'ld_skip', 'ld_out': 'ld_out'}


@pytest.fixture(scope='module')
def results(built_lib):
  repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
  r = subprocess.run([sys.executable] + (['-s'] if sys.flags.no_user_site else []) + ['-c', _CALLS], cwd=repo, env=env,
                     capture_output=True, text=True, timeout=300)
  assert r.returncode == 0, r.stderr[-2000:]
  return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize('op', ['up', 'pool', 's2d'])
def test_bad_shapes_and_strides_are_refused_before_any_cuda_call(results, op):
  seen = 0
  for o, what, rc, msg in results:
    if o != op:
      continue
    seen += 1
    if what.startswith('control'):          # accepted: the launch itself fails, there being no device
      assert rc == L.CT_ERR_CUDA, (what, rc, msg)
      continue
    assert rc == L.CT_ERR_INVALID, (what, rc, msg)
    assert MESSAGE[what.split()[0]] in msg, (what, msg)
  assert seen >= 5
