"""Shared helpers for the parity tests (test infrastructure; may import oracle/)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'oracle')):
  if p not in sys.path:
    sys.path.insert(0, p)

from centertrack_b200 import synthetic as wt   # noqa: E402

TASKS = {'coco_tracking': ['tracking'], 'mot': ['tracking', '--num_classes', '1', '--input_h', '544',
                                                 '--input_w', '960'],
         'nuscenes_ddd': ['tracking,ddd'], 'coco_pose': ['tracking,multi_pose']}


def make_opt(cfg, extra=()):
  from centertrack_b200.opts import opts
  return opts().init(TASKS[cfg] + ['--pre_hm'] + list(extra))


def make_model(cfg, seed=317, extra=()):
  """Product model with the deterministic synthetic weights (same tensors the goldens were made with)."""
  from centertrack_b200.model import create_model
  opt = make_opt(cfg, extra)
  m = create_model(opt.arch, opt.heads, opt.head_conv, opt=opt)
  sd = wt.make_state_dict(m.state_dict(), seed, rename=getattr(m, 'RENAME', ()))
  m.load_state_dict(sd)
  return opt, m, sd


def load_generic_golden(golden_dir):
  """The --arch generic goldens (oracle/gen_golden.py::gen_generic): the hc256 and hc64 tags are stored in two files
  so that each stays under 1 MB."""
  g = _NpzDict()
  for f in ('net_generic_coco_tracking_64x96.npz', 'net_generic_coco_tracking_64x96_hc64.npz'):
    z = np.load(os.path.join(golden_dir, f))
    g.update({k: z[k] for k in z.files})
  return g


class _NpzDict(dict):
  """A dict of arrays with np.load's `.files`."""
  @property
  def files(self):
    return list(self.keys())


def decode_inputs(kind, B, C, H, W, seed):
  """Must stay identical to oracle/gen_golden.py::decode_inputs."""
  rng = np.random.RandomState(seed)
  out = {'hm': (1. / (1. + np.exp(-(2 * rng.randn(B, C, H, W) - 4.6)))).astype(np.float32),
         'reg': rng.rand(B, 2, H, W).astype(np.float32),
         'wh': (rng.randn(B, 2, H, W) * 6).astype(np.float32),
         'tracking': (rng.randn(B, 2, H, W) * 3).astype(np.float32)}
  if kind == 'ddd':
    out.update({'dep': (rng.rand(B, 1, H, W) * 60).astype(np.float32),
                'rot': rng.randn(B, 8, H, W).astype(np.float32),
                'dim': (rng.rand(B, 3, H, W) * 4).astype(np.float32),
                'amodel_offset': rng.randn(B, 2, H, W).astype(np.float32)})
  if kind == 'pose':
    out.update({'hps': (rng.randn(B, 34, H, W) * 6).astype(np.float32),
                'hm_hp': (1. / (1. + np.exp(-(2 * rng.randn(B, 17, H, W) - 3.0)))).astype(np.float32),
                'hp_offset': rng.rand(B, 2, H, W).astype(np.float32)})
  if kind == 'mot':
    out['ltrb_amodal'] = (rng.randn(B, 4, H, W) * 8).astype(np.float32)
  return out


DECODE_CASES = [('coco', 1, 80, 128, 128, 100, 11), ('mot', 1, 1, 136, 240, 100, 12),
                ('ddd', 1, 10, 112, 200, 100, 13), ('pose', 1, 1, 128, 128, 100, 14),
                ('coco', 2, 80, 32, 32, 50, 15)]


# Must stay identical to oracle/gen_golden.py::HOST_CASES / host_case_inputs (Detector.pre_process goldens).
HOST_CASES = [('fix_res', ['--input_h', '128', '--input_w', '160'], (120, 200), False),
              ('fix_res_tall', ['--input_h', '160', '--input_w', '128'], (333, 210), True),
              ('keep_res', ['--keep_res'], (97, 131), False),
              ('fix_short', ['--fix_short', '96'], (150, 260), False),
              ('fix_short_tall', ['--fix_short', '64'], (300, 170), True)]


def host_case_inputs(i, hw):
  rng = np.random.RandomState(900 + i)
  image = rng.randint(0, 256, size=(hw[0], hw[1], 3)).astype(np.uint8)
  n = 6
  x0 = rng.uniform(-10, hw[1] * 0.8, n); y0 = rng.uniform(-10, hw[0] * 0.8, n)
  w = rng.uniform(0, hw[1] * 0.5, n); h = rng.uniform(0, hw[0] * 0.5, n)
  w[0] = 0.0
  tracks = [{'score': float(sc), 'active': int(ac), 'bbox': [float(a), float(b), float(a + c), float(b + d)]}
            for sc, ac, a, b, c, d in zip(rng.uniform(0.1, 1.0, n), [1, 1, 0, 1, 1, 1], x0, y0, w, h)]
  tracks[3]['score'] = 0.05
  calib = np.array([[700., 0, hw[1] / 2., 40.], [0, 700., hw[0] / 2., 1.], [0, 0, 1, 0.01]], dtype=np.float32)
  return image, tracks, calib


def flip_inputs(hw=(64, 96)):
  """Must stay identical to oracle/gen_golden.py::flip_inputs (--flip_test goldens)."""
  img, pre, hm = wt.synthetic_inputs(1, hw[0], hw[1], seed=77)
  cat = lambda t: torch.cat((t, t.flip(3)), 0).contiguous()
  return cat(img), cat(pre), cat(hm)


def e2e_frame(hw, batch, frame, seed):
  """Must stay identical to oracle/gen_golden.py::e2e_frame (full-size goldens)."""
  img, pre, hm = wt.synthetic_inputs(batch, hw[0], hw[1], seed=seed)
  return img[frame:frame + 1].clone(), pre[frame:frame + 1].clone(), hm[frame:frame + 1].clone()


E2E_CASES = {  # file stem -> (cfg, (H, W), batch, frame, seed); mirrors oracle/gen_golden.py::E2E_CASES
    'e2e_coco_tracking_512': ('coco_tracking', (512, 512), 1, 0, 317),
    'e2e_coco_tracking_512_b32f0': ('coco_tracking', (512, 512), 32, 0, 4242),
    'e2e_coco_tracking_512_b32f31': ('coco_tracking', (512, 512), 32, 31, 4242),
    'e2e_mot_544x960': ('mot', (544, 960), 1, 0, 317),
    'e2e_coco_pose_512': ('coco_pose', (512, 512), 1, 0, 317)}
