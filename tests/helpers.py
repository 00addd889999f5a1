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


# Output-head layouts beyond the shipped tables, one option each (opts.py --num_classes / --head_conv /
# --num_head_conv / --head_kernel and the optional heads), with the head plan DLA34Engine builds for each on the bf16
# tensor-core path:
#   ('fused', NH, N2, n_heads): one launch of csrc/conv_heads.cu, NH mid channels per pass, a common 1x1 n_tile N2;
#   ('two_pass', k, hidden): heads.0 (k x k, every head's first conv), `hidden` extra 1x1 convs for each head but reg
#   (opts.py: reg keeps one hidden conv), then one 1x1 per head.
# oracle/gen_golden.py::gen_head_layouts runs the reference on the same rows (tests/golden/net_head_layouts_64x96.npz).
HEAD_LAYOUTS = [
    ('classes20', 'coco_tracking', ['--num_classes', '20'], ('fused', 128, 32, 4)),
    ('classes60', 'coco_tracking', ['--num_classes', '60'], ('fused', 128, 64, 4)),
    ('hc64', 'coco_tracking', ['--head_conv', '64'], ('fused', 64, 80, 4)),
    ('classes1_hc64', 'coco_tracking', ['--num_classes', '1', '--head_conv', '64'], ('fused', 64, 16, 4)),
    ('pose_hc64', 'coco_pose', ['--head_conv', '64'], ('fused', 64, 48, 7)),
    ('ddd_12_heads', 'nuscenes_ddd', ['--ltrb', '--ltrb_amodal', '--velocity', '--nuscenes_att'], ('fused', 128, 16, 12)),
    ('classes90', 'coco_tracking', ['--num_classes', '90'], ('two_pass', 3, 0)),
    ('hc128', 'coco_tracking', ['--head_conv', '128'], ('two_pass', 3, 0)),
    ('num_head_conv2', 'coco_tracking', ['--num_head_conv', '2'], ('two_pass', 3, 1)),
    ('head_kernel1', 'coco_tracking', ['--head_kernel', '1'], ('two_pass', 1, 0)),
    ('head_kernel5', 'coco_tracking', ['--head_kernel', '5'], ('two_pass', 5, 0)),
]


def load_generic_golden(golden_dir):
  """The --arch generic goldens (oracle/gen_golden.py::gen_generic): the hc256 and hc64 tags are stored in two files
  so that each stays under 1 MB."""
  g = _NpzDict()
  for f in ('net_generic_coco_tracking_64x96.npz', 'net_generic_coco_tracking_64x96_hc64.npz'):
    z = np.load(os.path.join(golden_dir, f))
    g.update({k: z[k] for k in z.files})
  return g


def load_head_layout_golden(golden_dir):
  """The HEAD_LAYOUTS goldens (oracle/gen_golden.py::gen_head_layouts), stored as two files (fused and two-pass
  layouts) so that each stays under 1 MB."""
  g = _NpzDict()
  for f in ('net_head_layouts_64x96.npz', 'net_head_layouts_two_pass_64x96.npz'):
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


# pre_process's warp (cv2.warpAffine, INTER_LINEAR) on every resolution policy of detector.py:175-204 -- fixed input
# size, --keep_res with the DLA's pad 31 and the hourglass's 127, --fix_short in both orientations -- over camera
# frame sizes (1080p, KITTI, nuScenes, VGA, 4K), tiny upscales and 1 x 1, 1 x N, N x 1 frames:
# (name, cfg, extra argv, pad or None = the option's, source (h, w)).
WARP_GEOMETRIES = [
    ('coco_vga', 'coco_tracking', [], None, (480, 640)),
    ('mot_1080p', 'mot', [], None, (1080, 1920)),
    ('mot_portrait', 'mot', [], None, (1920, 1080)),
    ('kitti', 'coco_tracking', ['--input_h', '384', '--input_w', '1280'], None, (375, 1242)),
    ('nuscenes', 'coco_tracking', ['--input_h', '448', '--input_w', '800'], None, (900, 1600)),
    ('down_4k', 'coco_tracking', [], None, (2160, 3840)),
    ('up_100x60', 'coco_tracking', [], None, (60, 100)),
    ('up_7x5', 'coco_tracking', ['--input_h', '64', '--input_w', '96'], None, (5, 7)),
    ('odd_203x121', 'coco_tracking', ['--input_h', '128', '--input_w', '160'], None, (121, 203)),
    ('px_1x1', 'coco_tracking', ['--input_h', '64', '--input_w', '96'], None, (1, 1)),
    ('row_1x37', 'coco_tracking', ['--input_h', '64', '--input_w', '96'], None, (1, 37)),
    ('col_29x1', 'coco_tracking', ['--input_h', '64', '--input_w', '96'], None, (29, 1)),
    ('keep_res_kitti', 'coco_tracking', ['--keep_res'], None, (375, 1242)),
    ('keep_res_odd', 'coco_tracking', ['--keep_res'], None, (97, 131)),
    ('keep_res_1x1', 'coco_tracking', ['--keep_res'], None, (1, 1)),
    ('keep_res127_vga', 'coco_tracking', ['--keep_res'], 127, (480, 640)),
    ('keep_res127_nuscenes', 'coco_tracking', ['--keep_res'], 127, (900, 1600)),
    ('fix_short_wide', 'coco_tracking', ['--fix_short', '384'], None, (1080, 1920)),
    ('fix_short_tall', 'coco_tracking', ['--fix_short', '256'], None, (1920, 1080)),
    ('fix_short_kitti', 'coco_tracking', ['--fix_short', '128'], None, (375, 1242)),
]


def warp_geometry(i):
  """WARP_GEOMETRIES[i] -> (source (h, w), network input (oh, ow), minv fp64 [6], forward map fp64 [2, 3])."""
  from centertrack_b200.detector import frame_geometry
  _, cfg, extra, pad, hw = WARP_GEOMETRIES[i]
  opt = make_opt(cfg, extra)
  if pad is not None:
    opt.pad = pad
  meta, minv = frame_geometry(opt, *hw)
  return hw, (meta['inp_height'], meta['inp_width']), minv, np.asarray(meta['trans_input'], np.float64)


def _tie_maps(rng, n, term):
  """n inverse maps on which a fused multiply-add changes a whole output row: for one row y0 the row term M[1] y0 + M[2]
  (term 'x') or M[4] y0 + M[5] (term 'y'), rounded after the product and after the sum as cv2 rounds it, lands exactly on
  (32 m + 15 + 1/2) / 1024 px.  cvRound takes that tie to the even 32 m + 16, the next 1/32 px step, while the exact
  value -- what one rounding of a fused multiply-add keeps -- lies on one side of it and rounds to the other step."""
  from fractions import Fraction
  maps = []
  while len(maps) < n:
    a, c = float(rng.uniform(0.3, 1.5)), float(rng.uniform(0.05, 0.4))
    y0 = int(rng.randint(1, 300))
    tie = (32 * int(rng.randint(0, 100 * 1024 // 32)) + 15.5) / 1024
    slope = c if term == 'x' else a
    off = tie - slope * y0
    if slope * y0 + off != tie or np.rint((slope * y0 + off) * 1024) == \
        np.rint(float(Fraction(slope) * y0 + Fraction(off)) * 1024):
      continue
    m = [a, c, off, 0., 1.0, 0.5] if term == 'x' else [a, 0., 0.25, 0., a, off]
    maps.append(('tie_%s_row%d' % (term, y0), np.array(m, np.float64), (400, 500), (320, 200)))
  return maps


def warp_maps():
  """Inverse (dst -> src) maps beyond the resolution policies: (name, minv fp64 [6], source (h, w), output (oh, ow)).
  The fused-multiply-add tie maps, rotation and shear (M[1], M[3] != 0), a mirror, negative and fractional
  translations, and maps that land partly or wholly outside the frame.  Source coordinates stay within +-32767."""
  rng = np.random.RandomState(2024)
  maps = _tie_maps(rng, 3, 'y') + _tie_maps(rng, 3, 'x')
  ang, sc = np.deg2rad(17.0), 1.3
  maps += [
      ('rotate', np.array([sc * np.cos(ang), -sc * np.sin(ang), 120.25, sc * np.sin(ang), sc * np.cos(ang), -40.5]),
       (400, 500), (320, 200)),
      ('shear', np.array([1.0, 0.37, -20.5, 0.21, 0.9, 3.25]), (400, 500), (320, 200)),
      ('mirror', np.array([-1.0, 0.0, 499.0, 0.0, 1.0, 0.0]), (400, 500), (320, 200)),
      ('negative_fractional', np.array([0.75, 0.0, -13.37, 0.0, 1.25, -7.0625]), (400, 500), (320, 200)),
      ('partly_outside', np.array([2.5, 0.0, -100.3, 0.0, 2.5, -50.7]), (400, 500), (320, 200)),
      ('wholly_outside', np.array([1.0, 0.0, 5000.0, 0.0, 1.0, -3000.0]), (400, 500), (320, 200)),
      ('down_3_7x', np.array([3.7, 0.0, 0.4, 0.0, 3.7, 0.9]), (1080, 1920), (288, 512)),
  ]
  return maps


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
