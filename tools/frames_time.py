"""Cost of StreamRunner's frames mode (raw uint8 camera frames in, the warp + normalise + stem packing on the device):
    python tools/frames_time.py [--config mot coco_tracking] [--B 32] [--steps 40] [--rounds 3]

Per config (mot: 1920x1080 sources into the 544x960 input; coco_tracking: 640x480 sources into 512x512), bf16 engine,
device tracking, B streams, one graph replay per step:
1. end-to-end frames/s of step_frames -- with the frames passed as arrays (copied into the pinned staging) and written
   in place through frame_buffers() -- against step_host fed the already pre-processed fp32 frames (pinned), the
   runners timed alternately, `rounds` rounds of `steps` steps each (host clock around steps that end in a sync);
2. host CPU time (process time, every thread) of Detector.pre_process (cv2.warpAffine + normalise + HWC->CHW) per
   source frame, for context;
3. device time per call of ct_pack_stem_frames against B x ct_warp_affine_normalize + ct_pack_stem_input (the unfused
   path of the fp32-image runner, whose previous image is already warped), CUDA events around 50 calls, alternating
   rounds.
Prints the card and its power limit with the numbers, and one JSON line.  Needs a GPU."""
import argparse
import ctypes as C
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


def host_detector(opt):
  from centertrack_b200.dataset_info import get_dataset
  from centertrack_b200.detector import Detector
  det = object.__new__(Detector)
  ds = get_dataset(opt.dataset)
  det.opt = opt
  det.mean = np.array(ds.mean, dtype=np.float32).reshape(1, 1, 3)
  det.std = np.array(ds.std, dtype=np.float32).reshape(1, 1, 3)
  det.rest_focal_length = ds.rest_focal_length
  return det


def time_steps(fn, steps, runner):
  if runner.t:
    runner.fetch()
  t0 = time.perf_counter()
  for _ in range(steps):
    fn()
  runner.fetch()
  return (time.perf_counter() - t0) / steps


def kernel_times(runner, rounds, n=50):
  """ms per call: fused ct_pack_stem_frames vs B x ct_warp_affine_normalize + ct_pack_stem_input, same slot data."""
  lib, eng, B, H, W = L.lib(), runner.eng, runner.B, runner.H, runner.W
  ms = C.c_void_p(runner.mean.ctypes.data), C.c_void_p(runner.std.ctypes.data)
  cur, prev, hm = runner.u8[1], runner.u8[0], runner.hm[1]
  img, pre = runner.img[1], runner.img[0]

  def fused():
    L.check(lib.ct_pack_stem_frames(L.ptr(cur), L.ptr(prev), runner.frames, B, *ms, L.ptr(hm), L.ptr(eng.stem_input),
                                    H, W, L.stream_ptr()))

  def unfused():
    runner._warp_frames(1)
    L.check(lib.ct_pack_stem_input(L.ptr(img), L.ptr(pre), L.ptr(hm), L.ptr(eng.stem_input), B, H, W, L.stream_ptr()))

  out = {'fused': [], 'unfused': []}
  for fn in (fused, unfused):
    fn()
  torch.cuda.synchronize()
  for _ in range(rounds):
    for name, fn in (('fused', fused), ('unfused', unfused)):
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(n):
        fn()
      e1.record()
      torch.cuda.synchronize()
      out[name].append(e0.elapsed_time(e1) / n)
  return {k: float(np.median(v)) for k, v in out.items()}


def run_config(cfg, B, steps, rounds):
  from centertrack_b200.runner import StreamRunner
  h, w = SOURCES[cfg]
  opt, model, _ = make_model(cfg)
  model = model.cuda()
  H, W = opt.input_h, opt.input_w
  sizes = [(h, w)] * B
  frames = [frame(h, w, 10 + b) for b in range(B)]
  kw = dict(K=100, precision='bf16', device='cuda', opt=opt, device_tracking=True)
  fr = StreamRunner(model, B, H, W, frame_sizes=sizes, **kw)
  hr = StreamRunner(model, B, H, W, **kw)
  for r in (fr, hr):
    r.warm()
  det = host_detector(opt)
  det.pre_process(frames[0], 1.0)                          # first call imports cv2
  t0 = time.process_time()
  n_pre = 8
  for i in range(n_pre):
    det.pre_process(frames[i % B], 1.0)
  pre_ms = (time.process_time() - t0) / n_pre * 1e3
  imgs = torch.cat([det.pre_process(f, 1.0)[0] for f in frames], 0).pin_memory()

  arms = {'step_frames(arrays)': (lambda: fr.step_frames(frames), fr),
          'step_frames(frame_buffers)': (lambda: fr.step_frames(None), fr),
          'step_host(fp32 pinned)': (lambda: hr.step_host(imgs), hr)}
  for buf in fr.h_u8:        # every staging slot holds the frames once: the in-place arm's decoder wrote them there
    for f, (o, n) in zip(frames, [(q.offset, q.h * q.w * 3) for q in fr.frames]):
      buf.numpy()[o:o + n] = f.reshape(-1)
  for fn, r in arms.values():                              # warm-up steps of every arm
    time_steps(fn, 3, r)
  times = {k: [] for k in arms}
  for _ in range(rounds):
    for k, (fn, r) in arms.items():
      times[k].append(time_steps(fn, steps, r))
  fps = {k: B / float(np.median(v)) for k, v in times.items()}
  kern = kernel_times(fr, rounds)
  src_mb = h * w * 3 / 1e6
  img_mb = 3 * H * W * 4 / 1e6
  res = {'config': cfg, 'B': B, 'source': [h, w], 'input': [H, W], 'frames_per_s': fps,
         'pre_process_host_cpu_ms_per_frame': pre_ms, 'kernel_ms': kern,
         'h2d_mb_per_frame': {'uint8 source': src_mb, 'fp32 image': img_mb},
         'h2d_bytes_per_step': {'frames': fr.h2d_bytes_per_step, 'fp32 images': hr.h2d_bytes_per_step},
         'launches_per_step': {'frames': fr.launches_per_step, 'fp32 images': hr.launches_per_step}}
  return res


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--config', nargs='+', default=['mot', 'coco_tracking'], choices=sorted(SOURCES))
  ap.add_argument('--B', type=int, default=32)
  ap.add_argument('--steps', type=int, default=40)
  ap.add_argument('--rounds', type=int, default=3)
  a = ap.parse_args()
  assert torch.cuda.is_available(), 'frames_time.py needs a GPU'
  dev = card()
  print('card:', dev)
  out = []
  for cfg in a.config:
    r = run_config(cfg, a.B, a.steps, a.rounds)
    out.append(r)
    print('%s: B=%d, %dx%d sources -> %dx%d input' % (cfg, a.B, r['source'][0], r['source'][1], r['input'][0],
                                                       r['input'][1]))
    for k, v in r['frames_per_s'].items():
      print('  %-28s %8.1f frames/s' % (k, v))
    print('  Detector.pre_process host CPU  %8.2f ms per frame' % r['pre_process_host_cpu_ms_per_frame'])
    print('  ct_pack_stem_frames            %8.3f ms per call' % r['kernel_ms']['fused'])
    print('  B x warp + ct_pack_stem_input  %8.3f ms per call' % r['kernel_ms']['unfused'])
    print('  H2D per frame: uint8 %.2f MB, fp32 %.2f MB' % (r['h2d_mb_per_frame']['uint8 source'],
                                                           r['h2d_mb_per_frame']['fp32 image']))
  print(json.dumps({'card': dev, 'results': out}))


if __name__ == '__main__':
  main()
