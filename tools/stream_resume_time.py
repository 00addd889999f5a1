"""What resuming idle streams buys on a StreamRunner:
    python tools/stream_resume_time.py [--config mot] [--B 32] [--steps 60] [--rounds 3] [--p_miss 0.2]

1. --config mot (1920x1080 NV12 frames -> 544x960), B streams, bf16, device tracking, idle_streams, graphs, frames
   written in place through frame_buffers(); every stream misses each step with probability p_miss (seeded).  Frames/s of
   delivered frames when a stream that missed steps comes back with resume= against the same schedule where it comes
   back with a video start (starts=), in alternating rounds, medians; and the number of track-id restarts of each (a
   start restarts a stream's ids; checked on the device tables in an untimed pass);
2. the resume copy alone (one ct_stage_frames of n streams' last frames into the previous slot, on the copy stream):
   CUDA events around `calls` calls, for n = 1 and for the schedule's mean number of copies per step;
3. stream_state of one stream plus a step that restores it, against a plain step (host clock around work that ends in a
   synchronise), medians.
Prints the card and its power limit with the numbers, and one JSON line.  Needs a GPU."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from frames_time import card, frame                    # noqa  (also puts the repository and tests/ on sys.path)
from helpers import make_model                         # noqa
from yuv_oracle import bgr_to_yuv420                   # noqa

SIZE = (1080, 1920)


def schedule(B, steps, p, seed=5):
  """bool [steps, B]: whether stream b has a frame in each step (the first step: every stream; never all missing)."""
  rng = np.random.RandomState(seed)
  m = rng.uniform(size=(steps, B)) >= p
  m[0] = True
  for s in range(steps):
    if not m[s].any():
      m[s, rng.randint(B)] = True
  return m


def play(r, mask, pool, arm, check=False):
  """One pass of the schedule; -> (seconds from step 2 to the end, delivered frames timed, id restarts).  check: also
  read the tables each step and count the streams whose id counter went back (ids restarted)."""
  B = r.B
  r.reset_tracking()
  restarts, last_ids, t0, frames = 0, np.zeros(B, np.int64), None, 0
  for s in range(mask.shape[0]):
    if s == 2:
      r.fetch()
      t0 = time.perf_counter()
    live = np.nonzero(mask[s])[0].tolist()
    back = [b for b in live if s and not mask[s - 1, b]]
    views = r.frame_buffers()
    for b in live:
      np.copyto(views[b], pool[(s + b) % len(pool)])
    kw = dict(resume=back or None) if arm == 'resume' else dict(starts=back or None)
    r.step_frames(None, idle=[b for b in range(B) if b not in live], **kw)
    if s >= 2:
      frames += len(live)
    if check:
      _, cnt = r.fetch_tracks()
      restarts += int((cnt[:, 1] < last_ids).sum())
      last_ids = cnt[:, 1].astype(np.int64)
  r.fetch()
  return time.perf_counter() - t0, frames, restarts


def copy_time(r, n, calls):
  """ms per ct_stage_frames of n streams' frames from slot 0 to slot 1 (the resume copy), on the copy stream."""
  copies = [(b, 0, 1, r.frames[b].offset, r._upload_runs([b])[0][1] - r._upload_runs([b])[0][0]) for b in range(n)]
  with torch.cuda.stream(r.copy):
    for _ in range(5):
      r._copy_resumed(copies)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
      r._copy_resumed(copies)
    e1.record()
  e1.synchronize()
  return e0.elapsed_time(e1) / calls


def move_time(r, pool, rounds):
  """(stream_state ms, restore step ms, plain step ms) of stream 0, medians; each step ends in a synchronise."""
  st_ms, rest_ms, plain_ms = [], [], []
  r.reset_tracking()
  for _ in range(rounds * 5):
    r.fetch()
    t0 = time.perf_counter()
    for v in r.frame_buffers():
      np.copyto(v, pool[0])
    r.step_frames(None)
    r.fetch()
    plain_ms.append(1e3 * (time.perf_counter() - t0))
    t0 = time.perf_counter()
    st = r.stream_state(0)
    st_ms.append(1e3 * (time.perf_counter() - t0))
    t0 = time.perf_counter()
    for v in r.frame_buffers():
      np.copyto(v, pool[0])
    r.step_frames(None, restore={0: st})
    r.fetch()
    rest_ms.append(1e3 * (time.perf_counter() - t0))
  return float(np.median(st_ms)), float(np.median(rest_ms)), float(np.median(plain_ms))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--config', default='mot', choices=['mot'])
  ap.add_argument('--B', type=int, default=32)
  ap.add_argument('--steps', type=int, default=60)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--p_miss', type=float, default=0.2)
  ap.add_argument('--calls', type=int, default=200)
  a = ap.parse_args()
  assert torch.cuda.is_available(), 'stream_resume_time.py needs a GPU'
  dev = card()
  print('card:', dev)
  from centertrack_b200.runner import StreamRunner
  opt, model, _ = make_model(a.config)
  model = model.cuda()
  r = StreamRunner(model, a.B, opt.input_h, opt.input_w, K=100, precision='bf16', device='cuda', opt=opt,
                   device_tracking=True, frame_sizes=[SIZE] * a.B, max_frame_size=SIZE, frame_format='nv12',
                   idle_streams=True)
  r.warm()
  pool = [bgr_to_yuv420(frame(SIZE[0], SIZE[1], 11 + i), 'nv12') for i in range(4)]
  mask = schedule(a.B, a.steps, a.p_miss)
  backs = int(sum(((~mask[s - 1]) & mask[s]).sum() for s in range(1, a.steps)))
  restarts = {arm: play(r, mask, pool, arm, check=True)[2] for arm in ('resume', 'start')}
  fps = {'resume': [], 'start': []}
  for _ in range(a.rounds):
    for arm in fps:
      dt, n, _ = play(r, mask, pool, arm)
      fps[arm].append(n / dt)
  fps = {k: float(np.median(v)) for k, v in fps.items()}
  n_mean = max(1, int(round(backs / (a.steps - 1))))
  copy_ms = {n: copy_time(r, n, a.calls) for n in sorted({1, n_mean})}
  st_ms, rest_ms, plain_ms = move_time(r, pool, a.rounds)
  print('%s 1920x1080 NV12 -> %dx%d, B=%d, bf16, p_miss %.2f, %d steps, %d returns after a miss' %
        (a.config, opt.input_h, opt.input_w, a.B, a.p_miss, a.steps, backs))
  for arm in fps:
    print('  %-6s %8.1f delivered frames/s (median of %d rounds), %d track-id restarts' % (arm, fps[arm], a.rounds,
                                                                                          restarts[arm]))
  for n, ms in copy_ms.items():
    print('  resume copy of %d stream(s): %.4f ms per call' % (n, ms))
  print('  stream_state %.3f ms; a step restoring one stream %.3f ms against %.3f ms for a plain step' %
        (st_ms, rest_ms, plain_ms))
  print(json.dumps({'card': dev, 'config': a.config, 'B': a.B, 'p_miss': a.p_miss, 'steps': a.steps, 'returns': backs,
                    'frames_per_s': fps, 'id_restarts': restarts, 'resume_copy_ms': copy_ms,
                    'stream_state_ms': st_ms, 'restore_step_ms': rest_ms, 'plain_step_ms': plain_ms}))


if __name__ == '__main__':
  main()
