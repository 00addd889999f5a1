"""Timeline of CTA 0 of the halo conv kernel for a few layer shapes (B=16): python tools/halo_trace.py"""
import ctypes as C
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from centertrack_b200 import _lib as L       # noqa
from gpu_helpers import run_conv             # noqa

lib = L.lib()
import os as _os
cases = [('stem 7x7 8->48 sum3 512x512', 16, 8, 48, 512, 512, 7, False, 48),
         ('level0 16->16 512x512', 16, 16, 16, 512, 512, 3, False, 16),
         ('level0 64->64 256x256 (space-to-depth grid)', 16, 64, 64, 256, 256, 3, False, 64),
         ('heads.0 64->1024 nt128 128x128', 16, 64, 1024, 128, 128, 3, False, 128),
         ('level2 64->64 +res 128x128', 16, 64, 64, 128, 128, 3, True, 64),
         ('level3 128->128 +res nt32 64x64', 16, 128, 128, 64, 64, 3, True, 32),
         ('offset 64->27 nt32 128x128', 16, 64, 32, 128, 128, 3, False, 32),
         ('level0 16->16 512x512', 16, 16, 16, 512, 512, 3, False, 16),
         ('1x1 64->64 (canonical SBO=1024) 128x128', 16, 64, 64, 128, 128, 1, False, 64),
         ('1x1 64->128 128x128', 16, 64, 128, 128, 128, 1, False, 128),
         ('1x1 256->128 4 chunks 128x128', 16, 256, 128, 128, 128, 1, False, 128),
         ('5x5 64->64 (100 MMAs/item) 128x128', 16, 64, 64, 128, 128, 5, False, 64),
         ('5x5 64->16 128x128', 16, 64, 16, 128, 128, 5, False, 16)]
HEADS = [('head hm 1x1 256->80 NCHW f32 sigmoid', 16, 256, 80, 128, 128, 1, False, 80),
         ('head wh 1x1 256->2 NCHW f32', 16, 256, 2, 128, 128, 1, False, 16),
         ('offset 64->27 nt32 128x128 f32 NHWC', 16, 64, 27, 128, 128, 3, False, 32)]
if _os.environ.get('TRACE_SET') == 'heads':
  cases = HEADS
g = torch.Generator().manual_seed(0)
for (name, B, Cin, Cout, H, W, k, res, nt) in cases:
  x = torch.randn(B, Cin, H, W, generator=g)
  w = torch.randn(Cout, Cin, k, k, generator=g) * 0.05
  b = torch.zeros(Cout)
  r = torch.randn(B, Cout, H, W, generator=g).cuda() if res else None
  tr = torch.zeros(256 * 8, dtype=torch.int64, device='cuda')
  kw = dict(n_tile=nt, sum3=7) if Cin == 8 else dict(n_tile=nt)
  relu = Cin != 8
  if name.startswith('head'):
    kw.update(out_mode=L.CT_OUT_NCHW_F32, head_act=1 if 'sigmoid' in name else 0)
    relu = False
  if 'f32 NHWC' in name:
    kw.update(out_mode=L.CT_OUT_NHWC_F32, sig_from=18)
    relu = False
  run_conv(L.CT_ENGINE_TCGEN05_HALO, L.CT_BF16, x.cuda(), w, b, 1, relu, r, **kw)     # warm
  L.check(lib.ct_debug_trace(C.c_void_p(tr.data_ptr())))
  run_conv(L.CT_ENGINE_TCGEN05_HALO, L.CT_BF16, x.cuda(), w, b, 1, relu, r, **kw)
  torch.cuda.synchronize()
  L.check(lib.ct_debug_trace(None))
  t = tr.cpu().numpy().reshape(256, 8).astype(np.int64)
  n = int((t[:, 4] > 0).sum())
  t0 = t[0, 0]
  print('==== %s : %d items in CTA 0' % (name, n))
  # stamps (conv_halo.cu h_stamp): 0 producer acquired the stage, 1 TMA issued, 2 MMA saw the halo, 4 MMAs complete,
  # 5 epilogue started, 6 epilogue done
  print('  it   prod_acq  tma_iss | mma_halo mma_done | epi_start epi_done   (cycles since start; item period)')
  for i in list(range(min(n, 8))) + list(range(max(8, n - 2), n)):
    row = t[i] - t0
    per = (t[i, 4] - t[i - 1, 4]) if i > 0 else 0
    print('  %3d %9d %8d | %8d %8d | %8d %8d   period %d' % (i, row[0], row[1], row[2], row[4], row[5], row[6], per))
  nblk = (k * k * (Cin // 16)) if Cin != 8 else k * ((k + 1) // 2)
  if n > 4:
    d = t[2:n]
    print('  MMA phase per K16 block: %.0f cycles (nblk %d); period per block %.0f' % (
        np.mean(d[:, 4] - d[:, 2]) / nblk, nblk, np.mean(np.diff(t[1:n, 4])) / nblk))
    print('  mean over items 2..: MMA phase %.0f | epilogue %.0f | tma_latency(iss->mma_halo of same item) %.0f  period %.0f' % (
        np.mean(d[:, 4] - d[:, 2]), np.mean(d[:, 6] - d[:, 5]), np.mean(d[:, 2] - d[:, 1]), np.mean(np.diff(t[1:n, 4]))))
