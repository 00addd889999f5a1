"""Build the launch plan of every engine on the CPU (nothing is launched by the constructor): catches Python-side
errors in engine.py before a GPU run is spent on them.    python tools/plan_dryrun.py"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import helpers as th                                   # noqa
from centertrack_b200 import _lib as L                 # noqa
from centertrack_b200 import engine as E               # noqa

for cfg, (H, W) in (('coco_tracking', (64, 96)), ('coco_pose', (64, 64))):
  opt, m, sd = th.make_model(cfg)
  for prec in ('bf16', 'bf16x3', 'fp32'):
    e = E.DLA34Engine(sd, opt.heads, 2, H, W, precision=prec, device='cpu')
    print(cfg, prec, len(e.ops), 'ops')
    for kind, d, name in e.ops:
      if name in ('base.level0', 'base.level1') and kind == 'conv':
        c = L.conv_config(d)
        print('   %-12s engine %d  k %dx%d s%d pad %d  C %d -> %d  %dx%d -> %dx%d  out_mode %d ld_out %d n_tile %d  '
              'smem %d stages %d tile %dx%d ctas/SM %d overlap %d'
              % (name, d.engine, d.KH, d.KW, d.stride, d.pad, d.C_in, d.C_out, d.H, d.W, d.OH, d.OW, d.out_mode, d.ld_out,
                 d.n_tile, c.smem_bytes, c.stages, c.tile_w, c.tile_h, c.ctas_per_sm, c.overlap))
