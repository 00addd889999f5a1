"""What idle streams save on a StreamRunner (idle_streams=g):
    python tools/idle_streams_time.py [--B 32] [--steps 20] [--rounds 3] [--videos 64] [--min_len 100] [--max_len 400]

1. step time against the number of live streams n, at B streams, for the plain capacity runner and idle-streams runners
   with g = 1 and g = 4: coco_tracking (640x480 -> 512x512) and mot (1920x1080 -> 544x960), bf16, device tracking,
   graphs, frames written in place through frame_buffers(); alternating rounds of `steps` steps, medians;
2. the MOT17-style schedule of camera_switch_time.py (`videos` videos of min_len..max_len frames, every fourth at
   640x480) through track_videos: steps, images computed, real frames/s, plain against idle;
3. a 7-video schedule (as a MOT17 half-validation split) on the same runners.
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

CASES = {'coco_tracking': (480, 640), 'mot': (1080, 1920)}
NS = (1, 2, 4, 8, 16, 24, 32)


def _runners(model, opt, B, size, gs):
  from centertrack_b200.runner import StreamRunner
  kw = dict(K=100, precision='bf16', device='cuda', opt=opt, device_tracking=True, frame_sizes=[size] * B,
            max_frame_size=size)
  out = {'plain': StreamRunner(model, B, opt.input_h, opt.input_w, **kw)}
  for g in gs:
    out['idle g=%d' % g] = StreamRunner(model, B, opt.input_h, opt.input_w, idle_streams=g, **kw)
  for r in out.values():
    r.warm()
  return out


def n_curve(cfg, B, steps, rounds, gs=(1, 4)):
  opt, model, _ = make_model(cfg)
  model = model.cuda()
  size = CASES[cfg]
  runners = _runners(model, opt, B, size, gs)
  img = frame(size[0], size[1], 5)
  for r in runners.values():                    # every slot's staging holds a frame: later steps write nothing
    for _ in range(3):
      for v in r.frame_buffers():
        np.copyto(v, img)
      r.step_frames(None)
    r.fetch()

  def run(r, n, k):
    idle = list(range(n, B)) if r.idle_g is not None else None
    r.reset_tracking()
    t0 = None
    for i in range(k + 2):                      # two untimed steps: the first is eager (pre_images = images)
      if i == 2:
        r.fetch()
        t0 = time.perf_counter()
      r.frame_buffers()
      r.step_frames(None, idle=idle)
    r.fetch()
    return (time.perf_counter() - t0) / k

  res = {}
  for n in [x for x in NS if x <= B]:
    t = {k: [] for k in runners}
    for _ in range(rounds):
      for k, r in runners.items():
        t[k].append(run(r, n, steps))
    res[n] = {k: 1e3 * float(np.median(v)) for k, v in t.items()}
    print('%s %s -> %dx%d, B=%d, n=%2d live: ' % (cfg, size, opt.input_h, opt.input_w, B, n) +
          ', '.join('%s %.2f ms' % (k, v) for k, v in res[n].items()) + ' per step (median of %d rounds)' % rounds)
  del runners
  return {'source': list(size), 'input': [opt.input_h, opt.input_w], 'ms_per_step': res}


def schedules(B, n_videos, min_len, max_len, g):
  from centertrack_b200.videos import Video, track_videos
  opt, model, _ = make_model('mot')
  model = model.cuda()
  big, small = (1080, 1920), (480, 640)
  pool = {sz: [frame(sz[0], sz[1], 100 * i + sz[0]) for i in range(4)] for sz in (big, small)}
  rng = np.random.RandomState(17)
  mot64 = [(small if v % 4 == 3 else big, int(rng.randint(min_len, max_len + 1))) for v in range(n_videos)]
  rng = np.random.RandomState(7)
  seven = [(big, int(rng.randint(400, 1100) // 2)) for _ in range(7)]
  runners = _runners(model, opt, B, big, (g,))
  out = {}
  for name, spec in (('%d videos' % n_videos, mot64), ('7 videos', seven)):
    total = sum(n for _, n in spec)
    out[name] = {'frames': total}
    for k, r in runners.items():
      images = []
      step = r.step_frames

      def counted(*a, **kw):
        res = step(*a, **kw)
        images.append(r._n)
        return res
      r.step_frames = counted
      r.reset_tracking()
      vids = [Video(v, (pool[sz][(v + i) % 4] for i in range(n))) for v, (sz, n) in enumerate(spec)]
      t0 = time.perf_counter()
      got = sum(1 for _ in track_videos(r, vids))
      dt = time.perf_counter() - t0
      del r.step_frames
      assert got == total, (got, total)
      out[name][k] = {'steps': len(images), 'images': int(sum(images)), 'real_frames_per_s': total / dt}
      print('%s on B=%d (%d frames): %-9s %5d steps, %7d images computed, %8.1f real frames/s' %
            (name, B, total, k, len(images), sum(images), total / dt))
  del runners
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--B', type=int, default=32)
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--videos', type=int, default=64)
  ap.add_argument('--min_len', type=int, default=100)
  ap.add_argument('--max_len', type=int, default=400)
  ap.add_argument('--g', type=int, default=1, help='idle_streams of the schedule runs')
  a = ap.parse_args()
  assert torch.cuda.is_available(), 'idle_streams_time.py needs a GPU'
  dev = card()
  print('card:', dev)
  res = {'card': dev, 'B': a.B, 'n_curve': {cfg: n_curve(cfg, a.B, a.steps, a.rounds) for cfg in CASES}}
  res['schedules'] = schedules(a.B, a.videos, a.min_len, a.max_len, a.g)
  print(json.dumps(res))


if __name__ == '__main__':
  main()
