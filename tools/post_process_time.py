"""Cost and gain of StreamRunner(device_post_process=True) on detection models:
    python tools/post_process_time.py [--B 32] [--steps 30] [--rounds 3] [--calls 50]

1. ct_post_process per launch, CUDA events around `calls` launches after a warm-up, `rounds` rounds alternating over
   the cases, medians; B streams of K = 100 records from seeded heads, out_thresh = -1 (every record kept, the default
   without tracking): ctdet (80 classes, 512x512 input), ddd (448x800 input) and multi_pose (512x512 input).
2. End to end, bf16 engine, B streams, frames written in place through frame_buffers(), one graph replay per step,
   `rounds` rounds of `steps` steps with the arms alternating, medians of frames/s and of host CPU time per step
   (process time, every thread): ddd with 1600x900 frames and ctdet with 640x480 frames into 512x512, each with three
   arms -- (a) device_post_process + previous_results() (the dicts fetch_results() gives), (b) the same runner without
   the option + generic_post_process of the returned records with previous_meta(b) on the host, (c) device_post_process
   + previous_detections() (the tables).
Prints the card, its power limit and SM clock with the numbers, and one JSON line.  Needs a GPU.  The synthetic
weights stand in for trained ones: the work per step does not depend on the weights' values."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))

# kernel cases: (name, task, classes, decode_inputs kind, output grid (h, w))
KERNEL_CASES = [('ctdet', 'ctdet', 80, 'coco', (128, 128)), ('ddd', 'ddd', 10, 'ddd', (112, 200)),
                ('multi_pose', 'multi_pose', 1, 'pose', (128, 128))]
# end-to-end cases: (name, task, source frame (h, w))
E2E_CASES = [('ddd', 'ddd', (900, 1600)), ('ctdet', 'ctdet', (480, 640))]


def model_of(task):
  from centertrack_b200 import synthetic as wt
  from centertrack_b200.model import create_model
  from centertrack_b200.opts import opts
  opt = opts().init([task])
  m = create_model(opt.arch, opt.heads, opt.head_conv, opt=opt)
  m.load_state_dict(wt.make_state_dict(m.state_dict(), 317, rename=getattr(m, 'RENAME', ())))
  return opt, m.cuda()


def kernel_cases(B, K, rounds, calls):
  import torch
  from centertrack_b200.decode import generic_decode
  from centertrack_b200.device_detections import DeviceDetections
  from centertrack_b200.opts import opts
  from helpers import decode_inputs
  arms = {}
  for name, task, C_, kind, (h, w) in KERNEL_CASES:
    maps = decode_inputs(kind, B, C_, h, w, 31)
    maps.pop('tracking')                  # detection models: no tracking head
    res = generic_decode({k: torch.from_numpy(v).cuda() for k, v in maps.items()}, K=K)
    opt = opts().init([task])
    det = DeviceDetections(opt, B, K, res.records.shape[2], res.layout, 4 * h, 4 * w, 'cuda')
    rec = res.records
    arms[name] = (lambda det=det, rec=rec: det.step(rec))
  for fn in arms.values():
    fn()
  torch.cuda.synchronize()
  times = {k: [] for k in arms}
  for _ in range(rounds):
    for k, fn in arms.items():
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(calls):
        fn()
      e1.record()
      torch.cuda.synchronize()
      times[k].append(e0.elapsed_time(e1) / calls)
  return {k: float(np.median(v)) for k, v in times.items()}


def host_post_process(opt, runner, rec):
  """Detector.post_process + merge_outputs of every stream's records, as a caller of a runner without the option."""
  import torch
  from centertrack_b200.decode import views_from_records
  from centertrack_b200.post_process import generic_post_process
  views = {k: v.numpy() for k, v in views_from_records(torch.from_numpy(rec), runner.layout).items()}
  out = []
  for b in range(runner.B):
    m = runner.previous_meta(b)
    one = {k: v[b:b + 1] for k, v in views.items()}
    res = generic_post_process(opt, one, [m['c']], [m['s']], m['out_height'], m['out_width'], opt.num_classes,
                               [m['calib']])[0]
    out.append([r for r in res if r['score'] > opt.out_thresh])
  return out


def e2e(task, size, B, steps, rounds):
  import torch
  from centertrack_b200.runner import StreamRunner
  from frames_time import frame
  opt, model = model_of(task)
  H, W = opt.input_h, opt.input_w
  frames = [frame(size[0], size[1], 10 + b) for b in range(B)]
  kw = dict(K=100, precision='bf16', device='cuda', opt=opt, frame_sizes=[size] * B)
  post = StreamRunner(model, B, H, W, device_post_process=True, **kw)
  plain = StreamRunner(model, B, H, W, **kw)
  for r in (post, plain):
    r.warm()
    for s in range(3):            # the decoder wrote every staging slot once
      for v, f in zip(r._views(s, r.frame_sizes), frames):
        v[...] = f
  sink = []

  def arm_a():
    post.step_frames(None)
    if post.t >= 2:
      sink.append(post.previous_results())

  def arm_b():
    rec = plain.step_frames(None)
    if rec is not None:
      sink.append(host_post_process(opt, plain, rec))

  def arm_c():
    post.step_frames(None)
    if post.t >= 2:
      sink.append(post.previous_detections())

  arms = {'(a) device_post_process + fetch_results dicts': (arm_a, post),
          '(b) host generic_post_process': (arm_b, plain),
          '(c) device_post_process + fetch_detections tables': (arm_c, post)}

  def time_arm(fn, runner, n):
    runner.fetch()
    t0, c0 = time.perf_counter(), time.process_time()
    for _ in range(n):
      fn()
      sink.clear()
    runner.fetch()
    return (time.perf_counter() - t0) / n, (time.process_time() - c0) / n

  for fn, r in arms.values():
    fn()
    fn()
    time_arm(fn, r, 3)
  times = {k: [] for k in arms}
  for _ in range(rounds):
    for k, (fn, r) in arms.items():
      times[k].append(time_arm(fn, r, steps))
  torch.cuda.synchronize()
  return {k: {'frames_per_s': B / float(np.median([t[0] for t in v])),
              'host_cpu_ms_per_step': 1e3 * float(np.median([t[1] for t in v]))} for k, v in times.items()}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--B', type=int, default=32)
  ap.add_argument('--steps', type=int, default=30)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--calls', type=int, default=50, help='launches per timed window (>= 50)')
  a = ap.parse_args()
  if a.calls < 50:
    ap.error('--calls: at least 50')
  import torch
  assert torch.cuda.is_available(), 'post_process_time.py needs a GPU'
  from device_frames_time import card
  dev = card()
  print('card:', dev)
  kern = kernel_cases(a.B, 100, a.rounds, a.calls)
  print('ct_post_process, B=%d, K=100, out_thresh=-1:' % a.B)
  for k, v in kern.items():
    print('  %-12s %8.4f ms per launch' % (k, v))
  out = {'card': dev, 'B': a.B, 'kernel_ms': kern, 'end_to_end': {}}
  for name, task, size in E2E_CASES:
    res = e2e(task, size, a.B, a.steps, a.rounds)
    out['end_to_end'][name] = res
    print('%s, %dx%d frames, B=%d, bf16:' % (name, size[1], size[0], a.B))
    for k, v in res.items():
      print('  %-50s %8.1f frames/s, host CPU %.2f ms per step' % (k, v['frames_per_s'], v['host_cpu_ms_per_step']))
  print(json.dumps(out))


if __name__ == '__main__':
  main()
