"""Cost of --flip_test in StreamRunner (each stream's frame and its mirror in one step of 2B images):
    python tools/flip_time.py [--config coco_tracking kitti mot] [--B 32] [--steps 30] [--rounds 3]

Per config (coco_tracking: 640x480 sources into 512x512; kitti: KITTI's 1242x375 sources into 384x1280, 3 classes;
mot: 1920x1080 sources into 544x960), bf16 engine, device tracking, frames written in place through frame_buffers():
1. end-to-end frames/s of a flip runner (2B images per step) against a runner without the flip, timed alternately,
   `rounds` rounds of `steps` steps each (host clock around steps that end in a sync).  B is --B, or the largest
   halving of it whose runners fit in device memory;
2. device time per call of ct_pack_stem_frames_flip_dev against ct_pack_stem_frames_dev on the same slot data, and of one
   ct_flip_merge_heads launch against the per-head, per-pair ct_flip_merge launches it replaces, CUDA events around
   50 calls, alternating rounds.
Prints the card and its power limit with the numbers, and one JSON line.  Needs a GPU."""
import argparse
import copy
import ctypes as C
import gc
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from centertrack_b200 import _lib as L                 # noqa
from centertrack_b200 import synthetic as wt          # noqa
from helpers import make_model                         # noqa

# config -> (helpers task, extra options, source (h, w))
CONFIGS = {'coco_tracking': ('coco_tracking', [], (480, 640)),
           'kitti': ('coco_tracking', ['--dataset', 'kitti_tracking', '--num_classes', '3', '--input_h', '384',
                                       '--input_w', '1280'], (375, 1242)),
           'mot': ('mot', [], (1080, 1920))}


def card():
  name = torch.cuda.get_device_name()
  try:
    pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i',
                         str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    pl = 'unknown'
  return '%s, power limit %s' % (name, pl or 'unknown')


def frame(h, w, seed):
  x = wt.synthetic_inputs(1, h, w, seed=seed, n_blobs=0)[0][0].permute(1, 2, 0).numpy()
  return np.ascontiguousarray(np.clip(x * 70.0 + 115.0, 0, 255).astype(np.uint8))


def time_steps(runner, steps):
  if runner.t:
    runner.fetch()
  t0 = time.perf_counter()
  for _ in range(steps):
    runner.step_frames(None)
  runner.fetch()
  return (time.perf_counter() - t0) / steps


def events(fns, rounds, n=50):
  """ms per call of each fn: CUDA events around n calls, the fns alternating, median over rounds."""
  for fn in fns.values():
    fn()
  torch.cuda.synchronize()
  out = {k: [] for k in fns}
  for _ in range(rounds):
    for k, fn in fns.items():
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(n):
        fn()
      e1.record()
      torch.cuda.synchronize()
      out[k].append(e0.elapsed_time(e1) / n)
  return {k: float(np.median(v)) for k, v in out.items()}


def kernel_times(fl, rounds):
  """The flip pack vs the plain pack (same slot data, into the flip engine's stem input), and the batched merge vs one
  ct_flip_merge per head and pair (each pair's maps staged contiguously, as ct_flip_merge reads them)."""
  lib, B, H, W = L.lib(), fl.B, fl.H, fl.W
  ms = C.c_void_p(fl.mean.ctypes.data), C.c_void_p(fl.std.ctypes.data)
  cur, prev, hm, stem = fl.u8[1], fl.u8[0], fl.hm[1], fl.eng.stem_input
  from centertrack_b200.detector import flip_output
  outs = dict(fl.eng.outputs)
  pairs = {h: torch.stack((outs[h][:B], outs[h][B:]), 1).contiguous() for h in fl.flip_plan}   # [B,2,C,h,w]
  one = {h: torch.empty_like(fl.merged[h][0:1]) for h in fl.flip_plan}

  def per_head():
    for h, (perm, sign) in fl.flip_plan.items():
      t = pairs[h]
      for b in range(B):
        L.check(lib.ct_flip_merge(L.ptr(t[b]), L.ptr(one[h]), t.shape[2], t.shape[3], t.shape[4], L.ptr(perm),
                                  L.ptr(sign), L.stream_ptr()))

  desc = L.ptr(fl.d_frames[1]), B, fl.slot_bytes
  fns = {'ct_pack_stem_frames_flip_dev': lambda: L.check(lib.ct_pack_stem_frames_flip_dev(
             L.ptr(cur), L.ptr(prev), *desc, *ms, L.ptr(hm), L.ptr(stem), H, W, L.stream_ptr())),
         'ct_pack_stem_frames_dev': lambda: L.check(lib.ct_pack_stem_frames_dev(
             L.ptr(cur), L.ptr(prev), *desc, *ms, L.ptr(hm), L.ptr(stem), H, W, L.stream_ptr())),
         'ct_flip_merge_heads (1 launch)': lambda: flip_output(outs, fl.flip_plan, fl.merged),
         'ct_flip_merge (%d launches)' % (len(fl.flip_plan) * B): per_head}
  return events(fns, rounds)


def build(cfg, B):
  from centertrack_b200.runner import StreamRunner
  task, extra, (h, w) = CONFIGS[cfg]
  opt, model, _ = make_model(task, extra=extra)
  model = model.cuda()
  H, W = opt.input_h, opt.input_w
  kw = dict(K=100, precision='bf16', device='cuda', opt=opt, device_tracking=True, frame_sizes=[(h, w)] * B)
  plain = StreamRunner(model, B, H, W, **kw)
  opt_f = copy.copy(opt)
  opt_f.flip_test = True
  fl = StreamRunner(model, B, H, W, **dict(kw, opt=opt_f))
  for r in (plain, fl):
    r.warm()
  return model, plain, fl


def run_config(cfg, B, steps, rounds):
  _, _, (h, w) = CONFIGS[cfg]
  while True:
    try:
      model, plain, fl = build(cfg, B)
      break
    except torch.cuda.OutOfMemoryError:
      gc.collect()
      torch.cuda.empty_cache()
      if B == 1:
        raise
      B //= 2
  frames = [frame(h, w, 10 + b) for b in range(B)]
  for r in (plain, fl):      # every staging slot holds the frames once: a decoder wrote them there in place
    for buf in r.h_u8:
      for f, q in zip(frames, r.frames):
        buf.numpy()[q.offset:q.offset + q.h * q.w * 3] = f.reshape(-1)
  arms = {'no flip': plain, 'flip_test': fl}
  for r in arms.values():
    time_steps(r, 3)
  times = {k: [] for k in arms}
  for _ in range(rounds):
    for k, r in arms.items():
      times[k].append(time_steps(r, steps))
  fps = {k: B / float(np.median(v)) for k, v in times.items()}
  fps_all = {k: [B / v for v in vs] for k, vs in times.items()}
  kern = kernel_times(fl, rounds)
  res = {'config': cfg, 'B': B, 'source': [h, w], 'input': [fl.H, fl.W], 'frames_per_s': fps,
         'frames_per_s_rounds': fps_all, 'kernel_ms': kern,
         'launches_per_step': {'no flip': plain.launches_per_step, 'flip_test': fl.launches_per_step},
         'h2d_bytes_per_step': {'no flip': plain.h2d_bytes_per_step, 'flip_test': fl.h2d_bytes_per_step},
         'max_memory_allocated_gb': torch.cuda.max_memory_allocated() / 1e9}
  del model, plain, fl
  gc.collect()
  torch.cuda.empty_cache()
  torch.cuda.reset_peak_memory_stats()
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--config', nargs='+', default=['coco_tracking', 'kitti', 'mot'], choices=sorted(CONFIGS))
  ap.add_argument('--B', type=int, default=32)
  ap.add_argument('--steps', type=int, default=30)
  ap.add_argument('--rounds', type=int, default=3)
  a = ap.parse_args()
  assert torch.cuda.is_available(), 'flip_time.py needs a GPU'
  dev = card()
  print('card:', dev)
  out = []
  for cfg in a.config:
    r = run_config(cfg, a.B, a.steps, a.rounds)
    out.append(r)
    print('%s: B=%d, %dx%d sources -> %dx%d input (flip: %d images per step)' % (
        cfg, r['B'], r['source'][0], r['source'][1], r['input'][0], r['input'][1], 2 * r['B']))
    for k, v in r['frames_per_s'].items():
      print('  %-12s %8.1f frames/s  (rounds: %s)' % (k, v, ', '.join('%.1f' % x for x in r['frames_per_s_rounds'][k])))
    for k, v in r['kernel_ms'].items():
      print('  %-32s %8.4f ms per call' % (k, v))
    print('  peak device memory %.1f GB' % r['max_memory_allocated_gb'])
  print(json.dumps({'card': dev, 'results': out}))


if __name__ == '__main__':
  main()
