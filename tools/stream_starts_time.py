"""Cost of starting videos on StreamRunner streams (starts= / pre_dets=):
    python tools/stream_starts_time.py [--config mot] [--B 32] [--seeds 100] [--steps 40] [--rounds 3] [--steady-only]

bf16 engine, device tracking, frames mode (1920x1080 sources into 544x960 at mot, 640x480 into 512x512 at
coco_tracking), frames written in place through frame_buffers(), one graph replay per step:
1. the start prologue alone (first-frame pre_images copy per started stream + one ct_track_start launch), for 1 and for
   B streams starting with `seeds` seeds each: CUDA events around 50 prologues on staged start lists, per round;
2. end-to-end frames/s with no starts (--steady-only prints only this; run it from a checkout of another commit to
   compare against it, alternating);
3. end-to-end frames/s with one stream restarting every step with `seeds` seeds (the worst case), alternated with 2.
Host clock around `steps` steps that end in a sync.  Prints the card and its power limit and one JSON line.  Needs a
GPU."""
import argparse
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
from centertrack_b200 import synthetic as wt          # noqa
from helpers import make_model                         # noqa

SOURCES = {'mot': (1080, 1920), 'coco_tracking': (480, 640)}


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


def seeds(rng, n, h, w, thresh):
  """n seeds above new_thresh, in source pixels."""
  out = []
  for _ in range(n):
    bw, bh = rng.uniform(20, 120, 2)
    x0, y0 = rng.uniform(0, w - bw), rng.uniform(0, h - bh)
    out.append({'score': float(rng.uniform(thresh + 0.05, 1.0)), 'class': 1,
                'bbox': [float(x0), float(y0), float(x0 + bw), float(y0 + bh)]})
  return out


def time_steps(fn, steps, runner):
  if runner.t:
    runner.fetch()
  t0 = time.perf_counter()
  for i in range(steps):
    fn(i)
  runner.fetch()
  return (time.perf_counter() - t0) / steps


def prologue_ms(runner, streams, pre_dets, rounds, n=50):
  """ms per start prologue of `streams` (staged once in slot 1, as a step with t > 0 runs it)."""
  slot = 1
  plan = runner._check_starts(streams, pre_dets)
  runner._upload_starts(slot, plan, non_blocking=False)
  runner._starts[slot] = None                 # staged for the timing only: no step consumes it
  torch.cuda.synchronize()
  out = []
  for _ in range(rounds):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
      runner._start_prologue(slot, plan[0])
    e1.record()
    torch.cuda.synchronize()
    out.append(e0.elapsed_time(e1) / n)
  return float(np.median(out))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--config', default='mot', choices=sorted(SOURCES))
  ap.add_argument('--B', type=int, default=32)
  ap.add_argument('--seeds', type=int, default=100)
  ap.add_argument('--steps', type=int, default=40)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--steady-only', action='store_true')
  a = ap.parse_args()
  assert torch.cuda.is_available(), 'stream_starts_time.py needs a GPU'
  from centertrack_b200.runner import StreamRunner
  dev = card()
  print('card:', dev)
  h, w = SOURCES[a.config]
  opt, model, _ = make_model(a.config)
  model = model.cuda()
  B, H, W = a.B, opt.input_h, opt.input_w
  r = StreamRunner(model, B, H, W, K=100, precision='bf16', device='cuda', opt=opt, device_tracking=True,
                   frame_sizes=[(h, w)] * B)
  r.warm()
  frames = [frame(h, w, 10 + b) for b in range(B)]
  for buf in r.h_u8:                          # every staging slot holds the frames: a decoder wrote them in place
    for f, q in zip(frames, r.frames):
      buf.numpy()[q.offset:q.offset + q.h * q.w * 3] = f.reshape(-1)
  arms = {'no starts': lambda i: r.step_frames(None)}
  res = {'config': a.config, 'B': B, 'source': [h, w], 'input': [H, W], 'card': dev}
  if not a.steady_only:
    rng = np.random.RandomState(0)
    pre = {b: seeds(rng, a.seeds, h, w, opt.new_thresh) for b in range(B)}
    arms['one stream restarts every step'] = lambda i: r.step_frames(None, starts=[i % B],
                                                                     pre_dets={i % B: pre[i % B]})
  for fn in arms.values():                    # warm-up steps of every arm
    time_steps(fn, 3, r)
  times = {k: [] for k in arms}
  for _ in range(a.rounds):
    for k, fn in arms.items():
      times[k].append(time_steps(fn, a.steps, r))
  res['frames_per_s'] = {k: [B / t for t in v] for k, v in times.items()}
  res['launches_per_step'] = r.launches_per_step
  print('%s: B=%d, %dx%d sources -> %dx%d input, bf16, device tracking, frames in place' % (a.config, B, h, w, H, W))
  for k, v in res['frames_per_s'].items():
    print('  %-32s %s frames/s (median %.1f)' % (k, ' '.join('%.1f' % x for x in v), float(np.median(v))))
  if not a.steady_only:
    r.fetch()
    res['prologue_ms'] = {}
    for n in (1, B):
      streams = list(range(n))
      res['prologue_ms'][n] = prologue_ms(r, streams, {b: pre[b] for b in streams}, a.rounds)
      print('  start prologue, %2d stream(s) x %d seeds: %.4f ms' % (n, a.seeds, res['prologue_ms'][n]))
    plan = r._check_starts([0], {0: pre[0]})
    res['start_h2d_bytes'] = r._upload_starts(1, plan, non_blocking=False)
    r._starts[1] = None
    print('  start upload: %d bytes per started stream with %d seeds' % (res['start_h2d_bytes'], a.seeds))
  print(json.dumps(res))


if __name__ == '__main__':
  main()
