"""Deterministic, reference-free synthetic weights and inputs for benchmarks, smoke and tests.

The reference's default init collapses the 64-channel feature to ~1e-5 (SURVEY hazard H3), and no
pretrained checkpoint is available offline, so goldens and benchmarks use a variance-preserving
He-fan-in init that is a pure function of (state-dict key, shape, seed): the SAME tensors can be
materialised for the reference model (in the build container, to generate goldens) and for the H100
model (on the GPU machine, where no reference checkout exists).

BatchNorm running statistics come from data/bn_calib_seed<seed>.npz -- the batch statistics each BN
saw on one synthetic frame pair, recorded once by oracle/calibrate.py (what training-mode BN would have
accumulated).  With them activations stay O(1) through the 50-layer trunk and DCN offsets are O(1 px)
like in a trained network; without them the residual stream grows to |x|~250 and offsets to tens of
pixels, an ill-conditioned network on which no reduced-precision implementation can be judged.

Conditioning (round 2).  A randomly initialised conv-BN-ReLU stack is NOT a neutral instrument for judging a
reduced-precision engine: BatchNorm's mean subtraction removes signal energy but not perturbation energy, so
every conv-BN-ReLU layer multiplies the relative size of ANY perturbation by sqrt(pi/(pi-1)) = 1.21 (the
"gradient explosion at initialisation" of BN networks); the round-1 weights amplified a 1e-4 input perturbation
x85 by the 64-channel feature and decorrelated a bf16 run from the fp32 one (relative error 0.46).  Trained
networks sit near unit gain.  The synthetic checkpoint is therefore conditioned the way trained DLA/ResNet
checkpoints look: BN shifts of the plain conv-BN-ReLU layers ~ N(1.25, 0.2) (most units active), residual
branches down-weighted (bn2 gamma ~ 0.5 x U(0.8,1.2)), DCN offsets dominated by their static part (offset-conv
bias ~ N(0, 0.7) px, weights N(0, 0.01): |offset| ~ 0.8 px mean, 2-3 px max), heat-map logits with std ~1.2.
Measured end-to-end gain of a relative input perturbation at the 64-channel feature: x3 (oracle, 128x160).
"""
import os
import math
import zlib

import torch


def _gen(key, seed):
  g = torch.Generator()
  g.manual_seed((zlib.crc32(key.encode()) ^ (seed * 2654435761)) & 0x7FFFFFFF)
  return g


_cache = {}
_DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'data')


def calib_path(seed):
  return os.path.join(_DATA, 'bn_calib_seed%d.npz' % seed)


def make_state_dict(template, seed=317, hm_scale=1.0, calibrated=True, rename=()):
  """template: {key: tensor} (only shapes/dtypes are read).  Returns a new state_dict.
  rename: ((prefix, dla_prefix), ...) for modules that hold the DLASeg graph under other names (--arch generic:
  `backbone.` = `base.`, `neck.dla_up.` = `dla_up.`, ...): tensors are generated (and BN statistics looked up) under
  the DLASeg name, so both archs get the SAME weights, and returned under the template's own keys."""
  if rename:
    def canon(k):
      for a, b in rename:
        if k.startswith(a):
          return b + k[len(a):]
      return k
    names = {k: canon(k) for k in template}
    sd = make_state_dict({names[k]: v for k, v in template.items()}, seed, hm_scale, calibrated)
    return {k: sd[names[k]] for k in template}
  ck = (tuple(sorted((k, tuple(v.shape)) for k, v in template.items())), seed, hm_scale, calibrated)
  if ck in _cache:
    return {k: v.clone() for k, v in _cache[ck].items()}
  out = _raw_state_dict(template, seed, hm_scale)
  if calibrated:
    import numpy as np
    path = calib_path(seed)
    if not os.path.exists(path):
      raise RuntimeError('%s missing: run `python oracle/calibrate.py %d`' % (path, seed))
    stats = np.load(path)
    for k in out:
      if (k.endswith('running_mean') or k.endswith('running_var')) and k in stats.files:
        out[k] = torch.from_numpy(stats[k]).to(out[k].dtype)
  _cache[ck] = {k: v.clone() for k, v in out.items()}
  return out


def _raw_state_dict(template, seed, hm_scale):
  out = {}
  bn_prefixes = {k[:-len('.running_mean')] for k in template if k.endswith('.running_mean')}
  for k, t in template.items():
    g = _gen(k, seed)
    shape = tuple(t.shape)
    if k.endswith('num_batches_tracked'):
      out[k] = torch.zeros(shape, dtype=t.dtype)
    elif k.endswith('running_var'):
      out[k] = torch.empty(shape).uniform_(0.8, 1.2, generator=g)
    elif k.endswith('running_mean'):
      out[k] = torch.empty(shape).normal_(0, 0.05, generator=g)
    elif k.rsplit('.', 1)[0] in bn_prefixes:
      # BatchNorm affine.  bn2 = the BN that closes a BasicBlock's residual branch (dla.py:57-63)
      res_branch = '.bn2.' in k
      if k.endswith('weight'):
        out[k] = (0.5 if res_branch else 1.0) * torch.empty(shape).uniform_(0.8, 1.2, generator=g)
      else:
        out[k] = torch.empty(shape).normal_(0.0, 0.1, generator=g) if res_branch else \
            torch.empty(shape).normal_(1.25, 0.2, generator=g)
    elif 'conv_offset_mask' in k:
      if k.endswith('weight'):
        out[k] = torch.empty(shape).normal_(0, 0.01, generator=g)
      else:
        b = torch.empty(shape).normal_(0, 0.7, generator=g)       # static offsets, O(1 px)
        b[18:] = torch.empty(shape[0] - 18).normal_(0, 0.5, generator=g)   # mask logits
        out[k] = b
    elif '.up_' in k and k.endswith('weight'):
      # learnable depthwise upsampling kernel: bilinear +- 10 % so learnability is exercised
      kk = shape[2]
      f = (kk + 1) // 2
      c = (2 * f - 1 - f % 2) / (2. * f)
      i = torch.arange(kk, dtype=torch.float32)
      b = 1 - (i / f - c).abs()
      base = (b[:, None] * b[None, :]).expand(shape)
      out[k] = base * torch.empty(shape).uniform_(0.9, 1.1, generator=g)
    elif len(shape) == 4:
      fan_in = shape[1] * shape[2] * shape[3]
      w = torch.empty(shape).normal_(0, math.sqrt(2.0 / fan_in), generator=g)
      head = k.split('.')[0]
      if 'hm' in head and k.endswith('.2.weight'):
        w = w * hm_scale
      out[k] = w
    elif len(shape) == 1:
      head = k.split('.')[0]
      if 'hm' in head and (k.endswith('.2.bias') or k == head + '.bias'):
        out[k] = torch.full(shape, -4.6)
      elif k.endswith('.conv.bias'):          # DCN bias
        out[k] = torch.empty(shape).normal_(0, 0.05, generator=g)
      else:
        out[k] = torch.empty(shape).normal_(0, 0.1, generator=g)
    else:
      out[k] = torch.zeros(shape, dtype=t.dtype)
    out[k] = out[k].to(t.dtype) if t.dtype.is_floating_point else out[k]
  return out


def synthetic_inputs(B, H, W, seed=317, n_blobs=20):
  """images: band-limited noise (octaves of bicubic-upsampled N(0,1) + 30 % white noise, unit variance -- the
  1/f-like spectrum of a normalised photograph); pre_images: the same scene shifted by (2, 3) px plus 10 % fresh
  noise (a video pair); pre_hm = max-splat of gaussians (SURVEY 8d)."""
  import torch.nn.functional as F
  g = torch.Generator().manual_seed(seed)
  white = torch.randn(B, 3, H, W, generator=g)
  fresh = torch.randn(B, 3, H, W, generator=g)
  low = torch.zeros(B, 3, H, W)
  for s in (4, 8, 16, 32):
    n = torch.randn(B, 3, max(2, H // s + 1), max(2, W // s + 1), generator=g)
    low = low + F.interpolate(n, size=(H, W), mode='bicubic', align_corners=False)
  low = low / low.std()
  img = (0.7 * low + 0.3 * white).contiguous()
  pre = (torch.roll(img, shifts=(2, 3), dims=(2, 3)) + 0.1 * fresh).contiguous()
  hm = torch.zeros(B, 1, H, W)
  ys = torch.arange(H, dtype=torch.float32).view(H, 1)
  xs = torch.arange(W, dtype=torch.float32).view(1, W)
  for b in range(B):
    for _ in range(n_blobs):
      cx = float(torch.rand(1, generator=g)) * W
      cy = float(torch.rand(1, generator=g)) * H
      r = 3 + float(torch.rand(1, generator=g)) * 12
      sig = (2 * r + 1) / 6
      blob = torch.exp(-((xs - cx) ** 2 + (ys - cy) ** 2) / (2 * sig * sig))
      hm[b, 0] = torch.maximum(hm[b, 0], blob)
  return img, pre, hm


def synthetic_track_stream(seed, frames=6, crowd=40):
  """Seeded post-processed detections of a crowded stream for the association tests and goldens (no network involved):
  per frame a score-sorted list of {score, class, ct, tracking, bbox} in image coordinates plus a list of public
  detections ({ct}) jittered around a subset of them (the MOT public-detection protocol, tracker.py:83-103).
  One frame of every stream is empty, objects persist with small motion so that matches, births, rejected
  assignments and coasting tracks all occur."""
  import numpy as np
  rng = np.random.RandomState(7000 + seed)
  n_obj = int(rng.randint(crowd // 2, crowd))
  ct = rng.uniform(10, 300, (n_obj, 2))
  wh = rng.uniform(4, 50, (n_obj, 2))
  cls = rng.randint(1, 4, n_obj)
  out = []
  for f in range(frames):
    move = rng.normal(0, 4, (n_obj, 2))
    ct = ct + move
    seen = rng.uniform(size=n_obj) < (0.0 if f == 3 and seed % 2 == 0 else 0.8)
    dets = []
    for i in np.nonzero(seen)[0]:
      c = (ct[i] + rng.normal(0, 0.5, 2)).astype(np.float32)
      w, h = wh[i] * rng.uniform(0.9, 1.1, 2)
      dets.append({'score': float(np.float32(rng.uniform(0.15, 1.0))), 'class': int(cls[i]),
                   'ct': c, 'tracking': (-move[i] + rng.normal(0, 1.5, 2)).astype(np.float32),
                   'bbox': np.array([c[0] - w / 2, c[1] - h / 2, c[0] + w / 2, c[1] + h / 2], np.float32)})
    for _ in range(int(rng.randint(0, 6))):        # clutter: detections that belong to no object
      c = rng.uniform(0, 310, 2).astype(np.float32)
      w, h = rng.uniform(3, 30, 2)
      dets.append({'score': float(np.float32(rng.uniform(0.15, 0.6))), 'class': int(rng.randint(1, 4)),
                   'ct': c, 'tracking': rng.normal(0, 3, 2).astype(np.float32),
                   'bbox': np.array([c[0] - w / 2, c[1] - h / 2, c[0] + w / 2, c[1] + h / 2], np.float32)})
    dets.sort(key=lambda d: -d['score'])
    pub = [{'ct': (d['ct'] + d['tracking'] + rng.normal(0, 2.0, 2)).astype(np.float32)}
           for d in dets if rng.uniform() < 0.6]
    out.append((dets, pub))
  return out
