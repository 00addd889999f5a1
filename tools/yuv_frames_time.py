"""Cost and gain of NV12 / I420 frames in StreamRunner (the 4:2:0 -> BGR conversion fused into the device warp):
    python tools/yuv_frames_time.py [--config mot coco_tracking] [--B 32] [--steps 40] [--rounds 3]
                                    [--baseline_lib PATH]

Per config (mot: 1920x1080 sources into the 544x960 input; coco_tracking: 640x480 sources into 512x512), B streams:
1. device time per call of ct_pack_stem_frames_dev on BGR, NV12 and I420 frames of the same scenes (previous frame and
   pre_hm read), CUDA events around 50 calls, the formats alternating, `rounds` rounds, medians.  --baseline_lib: also
   the BGR call of another build of the library (e.g. the parent commit's), alternating with this one's;
2. end-to-end frames/s of step_frames on capacity runners (max_frame_size = the source size), bf16 engine, device
   tracking, one graph replay per step, BGR against NV12 -- frames passed as arrays (copied into the pinned staging)
   and written in place through frame_buffers() -- the four arms alternating, `rounds` rounds of `steps` steps;
3. host time of cv2.cvtColor(COLOR_YUV2BGR_NV12) per source frame, CPU (process time, every thread) and wall clock:
   the conversion a BGR runner's caller runs and a 4:2:0 runner does not.
Prints the card and its power limit with the numbers, and one JSON line.  Needs a GPU."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from centertrack_b200 import _lib as L                 # noqa
from frames_time import SOURCES, card, frame, time_steps   # noqa
from helpers import make_model                         # noqa
from yuv_oracle import bgr_to_yuv420 as yuv            # noqa

FORMATS = ('bgr', 'nv12', 'i420')


def slot(frames, fmt, minv):
  """B frames of one format -> (device buffer at b * cap, device ct_frame [B], buffer bytes)."""
  from centertrack_b200.runner import FRAME_FORMATS, frame_layout
  h, w = frames[0].shape[:2] if fmt == 'bgr' else (frames[0].shape[0] * 2 // 3, frames[0].shape[1])
  _, n, step = frame_layout(fmt, h, w)
  cap = (n + 15) // 16 * 16
  buf = np.zeros(len(frames) * cap, np.uint8)
  desc = (L.Frame * len(frames))()
  for b, f in enumerate(frames):
    buf[b * cap:b * cap + n] = f.reshape(-1)
    d = desc[b]
    d.offset, d.h, d.w, d.step, d.format = b * cap, h, w, step, FRAME_FORMATS[fmt]
    d.minv[:] = minv.tolist()
  dev = torch.from_numpy(buf).cuda()
  return dev, torch.from_numpy(np.frombuffer(bytes(desc), np.uint8).copy()).cuda(), buf.size


def kernel_times(opt, bgr, rounds, baseline=None, n=50):
  """ms per call of ct_pack_stem_frames_dev per format (and of the baseline library's BGR call), same scenes."""
  from centertrack_b200.dataset_info import get_dataset
  from centertrack_b200.detector import frame_geometry
  B, H, W = len(bgr), opt.input_h, opt.input_w
  ds = get_dataset(opt.dataset)
  mean = np.ascontiguousarray(ds.mean, np.float32).reshape(3)
  std = np.ascontiguousarray(ds.std, np.float32).reshape(3)
  ms = C.c_void_p(mean.ctypes.data), C.c_void_p(std.ctypes.data)
  minv = frame_geometry(opt, *bgr[0].shape[:2])[1]
  hm = torch.rand((B, 1, H, W), device='cuda')
  out = torch.empty((B, H, W, 8), dtype=torch.bfloat16, device='cuda')
  data = {}
  for fmt in FORMATS:
    cur = bgr if fmt == 'bgr' else [yuv(f, fmt) for f in bgr]
    prev = cur[1:] + cur[:1]
    data[fmt] = slot(cur, fmt, minv), slot(prev, fmt, minv)
  libs = {'this': L.lib()}
  if baseline is not None:
    libs['baseline'] = baseline
  arms = {}
  for fmt in FORMATS:
    for name, lib in libs.items():
      if name != 'this' and fmt != 'bgr':
        continue
      (cur, dfr, nb), (prev, _, _) = data[fmt]
      arms['%s %s' % (fmt, name) if len(libs) > 1 and fmt == 'bgr' else fmt] = (
          lambda lib=lib, cur=cur, prev=prev, dfr=dfr, nb=nb: L.check(lib.ct_pack_stem_frames_dev(
              L.ptr(cur), L.ptr(prev), L.ptr(dfr), B, nb, *ms, L.ptr(hm), L.ptr(out), H, W, L.stream_ptr())))
  for fn in arms.values():
    fn()
  torch.cuda.synchronize()
  times = {k: [] for k in arms}
  for _ in range(rounds):
    for k, fn in arms.items():
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(n):
        fn()
      e1.record()
      torch.cuda.synchronize()
      times[k].append(e0.elapsed_time(e1) / n)
  return {k: float(np.median(v)) for k, v in times.items()}


def load_baseline(path):
  """Another build of libctb200.so, with this build's signature of ct_pack_stem_frames_dev."""
  lib = C.CDLL(os.path.abspath(path))
  lib.ct_pack_stem_frames_dev.argtypes = L.lib().ct_pack_stem_frames_dev.argtypes
  lib.ct_last_error.restype = C.c_char_p
  return lib


def run_config(cfg, B, steps, rounds, baseline):
  from centertrack_b200.runner import StreamRunner
  h, w = SOURCES[cfg]
  opt, model, _ = make_model(cfg)
  model = model.cuda()
  H, W = opt.input_h, opt.input_w
  bgr = [frame(h, w, 10 + b) for b in range(B)]
  nv12 = [yuv(f, 'nv12') for f in bgr]
  kern = kernel_times(opt, bgr, rounds, baseline)

  cv2.cvtColor(nv12[0], cv2.COLOR_YUV2BGR_NV12)
  n_cvt = 100
  t0, w0 = time.process_time(), time.perf_counter()
  for i in range(n_cvt):
    cv2.cvtColor(nv12[i % B], cv2.COLOR_YUV2BGR_NV12)
  cvt_ms = (time.process_time() - t0) / n_cvt * 1e3
  cvt_wall_ms = (time.perf_counter() - w0) / n_cvt * 1e3

  kw = dict(K=100, precision='bf16', device='cuda', opt=opt, device_tracking=True, frame_sizes=[(h, w)] * B,
            max_frame_size=(h, w))
  runners = {fmt: StreamRunner(model, B, H, W, frame_format=fmt, **kw) for fmt in ('bgr', 'nv12')}
  inputs = {'bgr': [cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12) for f in nv12], 'nv12': nv12}
  for fmt, r in runners.items():
    r.warm()
    for s in range(3):      # every staging slot holds the frames once: the in-place arm's decoder wrote them there
      for v, f in zip(r._views(s, r.frame_sizes), inputs[fmt]):
        v[...] = f
  arms = {}
  for fmt, r in runners.items():
    arms['%s step_frames(arrays)' % fmt] = (lambda r=r, x=inputs[fmt]: r.step_frames(x), r)
    arms['%s step_frames(frame_buffers)' % fmt] = (lambda r=r: r.step_frames(None), r)
  for fn, r in arms.values():
    time_steps(fn, 3, r)
  times = {k: [] for k in arms}
  for _ in range(rounds):
    for k, (fn, r) in arms.items():
      times[k].append(time_steps(fn, steps, r))
  fps = {k: B / float(np.median(v)) for k, v in times.items()}
  return {'config': cfg, 'B': B, 'source': [h, w], 'input': [H, W], 'frames_per_s': fps, 'kernel_ms': kern,
          'cvtColor_nv12_host_cpu_ms_per_frame': cvt_ms, 'cvtColor_nv12_wall_ms_per_frame': cvt_wall_ms,
          'h2d_bytes_per_step': {fmt: r.h2d_bytes_per_step for fmt, r in runners.items()}}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--config', nargs='+', default=['mot', 'coco_tracking'], choices=sorted(SOURCES))
  ap.add_argument('--B', type=int, default=32)
  ap.add_argument('--steps', type=int, default=40)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--baseline_lib', default=None, help='another libctb200.so whose BGR _dev pack is timed alongside')
  a = ap.parse_args()
  assert torch.cuda.is_available(), 'yuv_frames_time.py needs a GPU'
  dev = card()
  print('card:', dev)
  baseline = load_baseline(a.baseline_lib) if a.baseline_lib else None
  out = []
  for cfg in a.config:
    r = run_config(cfg, a.B, a.steps, a.rounds, baseline)
    out.append(r)
    print('%s: B=%d, %dx%d sources -> %dx%d input' % (cfg, a.B, r['source'][0], r['source'][1], r['input'][0],
                                                       r['input'][1]))
    for k, v in r['kernel_ms'].items():
      print('  ct_pack_stem_frames_dev %-14s %8.3f ms per call' % (k, v))
    for k, v in r['frames_per_s'].items():
      print('  %-34s %8.1f frames/s' % (k, v))
    print('  cv2.cvtColor NV12 -> BGR           %8.3f ms CPU, %.3f ms wall per frame' %
          (r['cvtColor_nv12_host_cpu_ms_per_frame'], r['cvtColor_nv12_wall_ms_per_frame']))
    print('  H2D per step: %s' % r['h2d_bytes_per_step'])
  print(json.dumps({'card': dev, 'results': out}))


if __name__ == '__main__':
  main()
