"""Cost of the association modes on the device tracker:
    python tools/track_modes_time.py [--steps 60] [--rounds 3] [--config nuscenes_ddd | coco_pose]

1. ct_track_step / ct_track_step_assoc alone at B = 32 streams, K = 100, on crowded synthetic records
   (synthetic.synthetic_track_stream with up to K detections per frame, identity output affine): microseconds per
   launch (CUDA events around each launch, median over the frames of several passes) and the largest number of
   Dijkstra search steps one stream's Hungarian solve took in a frame.
2. --config mot StreamRunner (960x544, bf16, B = 32, device tracking, one graph replay per step) frames/s with greedy,
   --hungarian and --public_det --hungarian association, the three runners timed alternately.
With --config nuscenes_ddd | coco_pose: step 1 only, on the same records widened by the head set's payload columns
(dep, rot, dim, amodel_offset / raw and refined keypoints), timed with the payload table (ct_track_step_payload) and
without it (the same records read as a 2-D layout).
Prints the card and its power limit with the numbers.  Needs a GPU."""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from centertrack_b200 import synthetic as wt          # noqa
from centertrack_b200.device_tracker import DeviceTracker   # noqa
from helpers import make_model, make_opt               # noqa

MODES = [('greedy', []), ('hungarian', ['--hungarian']), ('public', ['--public_det']),
         ('public_hungarian', ['--public_det', '--hungarian'])]
B, K, F = 32, 100, 11
# record heads after tracking (9, 2) of the payload configs
PAYLOAD_HEADS = {'nuscenes_ddd': [('dep', 1), ('rot', 8), ('dim', 3), ('amodel_offset', 2)],
                 'coco_pose': [('hps', 34), ('hps_refined', 34), ('kps_score', 1)]}


def payload_layout(config):
  """(decode layout, F) of the crowded records with the config's payload heads appended."""
  layout, off = {'tracking': (9, 2)}, F
  for name, w in PAYLOAD_HEADS.get(config, ()):
    layout[name] = (off, w)
    off += w
  return layout, off


def card():
  name = torch.cuda.get_device_name()
  try:
    pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i',
                         str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    pl = 'unknown'
  return '%s, power limit %s' % (name, pl or 'unknown')


def track_inputs(frames=6, Fr=F):
  """Per frame: records [B,K,Fr] on the device and the public detections (public_ct [B,P,2], public_n [B]); columns
  past F are seeded random head outputs."""
  streams = [wt.synthetic_track_stream(100 + b, frames=frames, crowd=2 * K) for b in range(B)]
  rng = np.random.RandomState(7)
  out = []
  for f in range(frames):
    rec = np.zeros((B, K, Fr), np.float32)
    rec[:, :, F:] = rng.uniform(0.1, 1.0, (B, K, Fr - F))
    pub = np.zeros((B, 512, 2), np.float32)
    n = np.zeros(B, np.int32)
    for b, st in enumerate(streams):
      dets, pubs = st[f]
      for i, d in enumerate(dets[:K]):
        rec[b, i, 0], rec[b, i, 1] = d['score'], d['class'] - 1
        rec[b, i, 2:4], rec[b, i, 4:8], rec[b, i, 9:11] = d['ct'], d['bbox'], d['tracking']
      p = np.array([q['ct'] for q in pubs], np.float32).reshape(-1, 2)[:512]
      pub[b, :len(p)], n[b] = p, len(p)
    out.append((torch.from_numpy(rec).cuda(), torch.from_numpy(pub).cuda(), torch.from_numpy(n).cuda()))
  return out


def time_track_step(passes=20, config=None, payload=False):
  layout, Fr = payload_layout(config)
  frames = track_inputs(Fr=Fr)
  res = {}
  for name, extra in MODES:
    opt = make_opt(config or 'coco_tracking', ['--track_thresh', '0.2', '--new_thresh', '0.3', '--max_age', '3'] + extra)
    opt.out_thresh = 0.1
    trk = DeviceTracker(opt, B, K, Fr, layout if payload else {'tracking': (9, 2)}, 544, 960, 'cuda')
    assert (trk.payload is not None) == payload
    trk.trans_out_inv.copy_(torch.tensor([[1., 0., 0., 0., 1., 0.]] * B))
    steps = torch.zeros(B, dtype=torch.int32, device='cuda')
    us, max_steps, max_tracks = [], 0, 0
    for p in range(passes + 1):
      trk.reset()
      for rec, pub, n in frames:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        trk.step(rec, pub, n, steps=steps)
        e1.record()
        torch.cuda.synchronize()
        if p > 0:                                     # pass 0 warms up
          us.append(e0.elapsed_time(e1) * 1000)
        max_steps = max(max_steps, int(steps.max()))
        max_tracks = max(max_tracks, int(trk.counts[:, 0].max()))
    us.sort()
    res[name] = (us[len(us) // 2], us[0], max_steps, max_tracks)
  return res


def time_mot(steps, rounds):
  H, W = 544, 960
  from centertrack_b200.runner import NS, StreamRunner
  img, pre, hm = wt.synthetic_inputs(2, H, W, seed=317)
  g = torch.Generator().manual_seed(0)
  host_img = [(img[s:s + 1] + 0.05 * torch.randn(B, 3, H, W, generator=g)) for s in range(2)]
  rng = np.random.RandomState(0)
  public = [[rng.uniform([0, 0], [W, H], (200, 2)).astype(np.float32) for _ in range(B)] for _ in range(NS)]
  _, model, _ = make_model('mot')
  model = model.cuda()                                # one network (and engine) shared by the runners, run in turn
  runners = {}
  for name, extra in (('greedy', []), ('hungarian', ['--hungarian']), ('public_hungarian', ['--public_det', '--hungarian'])):
    opt = make_opt('mot', extra)
    r = StreamRunner(model, B, H, W, K=K, precision='bf16', device='cuda', opt=opt, device_tracking=True)
    for s in range(NS):
      r.load_device_inputs(host_img[s & 1].cuda(), None, s, public[s] if r.public else None)
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
  ap.add_argument('--config', choices=sorted(PAYLOAD_HEADS), default=None)
  args = ap.parse_args()
  assert torch.cuda.is_available(), 'needs a GPU'
  print('card:', card())
  if args.config:
    print('track step, --config %s, B=%d K=%d, --max_age 3 (T = %d), crowded synthetic records:' % (args.config, B, K, 4 * K))
    for payload in (False, True):
      print(' %s payload:' % ('with' if payload else 'without'))
      for name, (med, lo, st, mt) in time_track_step(config=args.config, payload=payload).items():
        print('  %-17s median %7.1f us/launch (min %7.1f), max tracks %d' % (name, med, lo, mt))
    return
  print('track step, B=%d K=%d, --max_age 3 (T = %d), crowded synthetic records:' % (B, K, 4 * K))
  for name, (med, lo, st, mt) in time_track_step().items():
    print('  %-17s median %7.1f us/launch (min %7.1f), max Dijkstra steps in a frame %4d, max tracks %d' %
          (name, med, lo, st, mt))
  print('--config mot StreamRunner, bf16, B=%d, %d steps per sample, %d alternating rounds:' % (B, args.steps, args.rounds))
  for name, v in time_mot(args.steps, args.rounds).items():
    print('  %-17s %s frames/s (median %.1f)' % (name, ' '.join('%.1f' % x for x in v), sorted(v)[len(v) // 2]))


if __name__ == '__main__':
  main()
