"""Cost of per-stream tracker settings (StreamRunner stream_opts):
    python tools/stream_opts_time.py [--steps 60] [--rounds 3]

1. The track step alone at B = 32 streams, K = 100, --max_age 3, on the crowded synthetic records of
   tools/track_modes_time.py: ct_track_step (every stream greedy, no stream_opts), ct_track_step_opts with 32 equal
   greedy records, ct_track_step_opts with 8 Hungarian streams among 24 greedy ones, and ct_track_step_assoc with every
   stream Hungarian; microseconds per launch (CUDA events, median), the four timed in alternating rounds.
2. --config mot StreamRunner (960x544, bf16, B = 32, device tracking, one graph replay per step) frames/s without
   stream_opts, with stream_opts all equal to opt, and with a mixed set (8 streams --hungarian, 8 --track_thresh 0.5,
   the rest opt), the three runners timed alternately.
Prints the card and its power limit with the numbers.  Needs a GPU."""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from centertrack_b200 import synthetic as wt          # noqa
from centertrack_b200.device_tracker import DeviceTracker   # noqa
from helpers import make_model, make_opt               # noqa
from track_modes_time import B, F, K, card, track_inputs   # noqa

MIXED = [{'hungarian': True} if b % 4 == 1 else None for b in range(B)]
MOT_MIXED = [{'hungarian': True} if b % 4 == 1 else {'track_thresh': 0.5} if b % 4 == 2 else None for b in range(B)]


def time_track_step(passes=20):
  frames = track_inputs()
  base = ['--track_thresh', '0.2', '--new_thresh', '0.3', '--max_age', '3']
  cases = {'greedy (ct_track_step)': (base, None), 'equal opts (ct_track_step_opts)': (base, [None] * B),
           'mixed 8 hungarian (ct_track_step_opts)': (base, MIXED),
           'all hungarian (ct_track_step_assoc)': (base + ['--hungarian'], None)}
  trackers = {}
  for name, (args, so) in cases.items():
    opt = make_opt('coco_tracking', args)
    opt.out_thresh = 0.1
    trk = DeviceTracker(opt, B, K, F, {'tracking': (9, 2)}, 544, 960, 'cuda', stream_opts=so)
    trk.trans_out_inv.copy_(torch.tensor([[1., 0., 0., 0., 1., 0.]] * B))
    trackers[name] = trk
  us = {k: [] for k in trackers}
  for p in range(passes + 1):
    for name, trk in trackers.items():
      trk.reset()
      for rec, _, _ in frames:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        trk.step(rec)
        e1.record()
        torch.cuda.synchronize()
        if p > 0:                                     # pass 0 warms up
          us[name].append(e0.elapsed_time(e1) * 1000)
  return {k: sorted(v)[len(v) // 2] for k, v in us.items()}


def time_mot(steps, rounds):
  H, W = 544, 960
  from centertrack_b200.runner import NS, StreamRunner
  img, _, _ = wt.synthetic_inputs(2, H, W, seed=317)
  g = torch.Generator().manual_seed(0)
  host_img = [(img[s:s + 1] + 0.05 * torch.randn(B, 3, H, W, generator=g)) for s in range(2)]
  _, model, _ = make_model('mot')
  model = model.cuda()                                # one network (and engine) shared by the runners, run in turn
  opt = make_opt('mot')
  runners = {}
  for name, so in (('no stream_opts', None), ('equal stream_opts', [None] * B), ('mixed stream_opts', MOT_MIXED)):
    r = StreamRunner(model, B, H, W, K=K, precision='bf16', device='cuda', opt=opt, device_tracking=True,
                     stream_opts=so)
    for s in range(NS):
      r.load_device_inputs(host_img[s & 1].cuda(), None, s)
    r.warm()
    runners[name] = r
  fps = {k: [] for k in runners}
  for _ in range(rounds):
    for name, r in runners.items():
      for _ in range(5):
        r.step_device()
      torch.cuda.synchronize()
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(steps):
        r.step_device()
      e1.record()
      torch.cuda.synchronize()
      fps[name].append(B * steps / (e0.elapsed_time(e1) / 1000))
  return fps


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=60)
  ap.add_argument('--rounds', type=int, default=3)
  args = ap.parse_args()
  assert torch.cuda.is_available(), 'needs a GPU'
  print('card:', card())
  print('track step, B=%d K=%d, --max_age 3 (T = %d), crowded synthetic records, alternating passes:' % (B, K, 4 * K))
  for name, med in time_track_step().items():
    print('  %-40s median %7.1f us/launch' % (name, med))
  print('--config mot StreamRunner, bf16, B=%d, %d steps per sample, %d alternating rounds:' % (B, args.steps, args.rounds))
  for name, v in time_mot(args.steps, args.rounds).items():
    print('  %-20s %s frames/s (median %.1f)' % (name, ' '.join('%.1f' % x for x in v), sorted(v)[len(v) // 2]))


if __name__ == '__main__':
  main()
