"""A/B of the halo kernel's one-CTA overlap: bench.py with CTB_HALO_OVERLAP=0 (serial schedule) and =1, alternating.

  python tools/halo_overlap_ab.py [--pairs 4] [--steps 200] [--config coco_tracking]

Prints the card's name and power limit, one line per run and the median gain in frames/s.  Only the device-resident
frames/s leg of bench.py runs (the baselines, parity and latency legs are skipped)."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bench(overlap, steps, warmup, config):
  cmd = [sys.executable, os.path.join(ROOT, 'bench.py'), '--gpus', '1', '--steps', str(steps), '--warmup', str(warmup),
         '--config', config, '--no-cpu-baseline', '--no-gpu-baseline', '--no-accurate', '--no-latency', '--no-parity']
  r = subprocess.run(cmd, cwd=ROOT, env=dict(os.environ, CTB_HALO_OVERLAP=str(overlap)), capture_output=True, text=True)
  if r.returncode != 0:
    raise RuntimeError('bench.py failed (CTB_HALO_OVERLAP=%d):\n%s' % (overlap, r.stderr[-3000:]))
  return json.loads(r.stdout.strip().splitlines()[-1])['value']


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--pairs', type=int, default=4)
  ap.add_argument('--steps', type=int, default=200)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--config', default='coco_tracking')
  args = ap.parse_args()
  smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip()
  print('card: %s' % smi)
  runs = {0: [], 1: []}
  for i in range(args.pairs):
    for ov in (0, 1):
      v = bench(ov, args.steps, args.warmup, args.config)
      runs[ov].append(v)
      print('pair %d  CTB_HALO_OVERLAP=%d  %.1f frames/s' % (i, ov, v), flush=True)
  old, new = runs[0], runs[1]
  gain = statistics.median(new) / statistics.median(old) - 1
  print('serial  %.1f .. %.1f frames/s (spread %.2f %%)' % (min(old), max(old), 100 * (max(old) / min(old) - 1)))
  print('overlap %.1f .. %.1f frames/s (spread %.2f %%)' % (min(new), max(new), 100 * (max(new) / min(new) - 1)))
  print('median gain %+.2f %%; every overlap run faster than every serial run: %s' % (100 * gain, min(new) > max(old)))


if __name__ == '__main__':
  main()
