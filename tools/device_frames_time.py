"""Cost and gain of device frames in StreamRunner (decoder frames already in device memory, staged into the frame slot
by ct_stage_frames instead of being uploaded from the host):
    python tools/device_frames_time.py [--B 32] [--steps 40] [--rounds 3] [--calls 50] [--dry_run]

1. ct_stage_frames per call, CUDA events around `calls` calls after a warm-up, `rounds` rounds, medians, B streams:
   mot's 1080p NV12 as two planes of a decoder surface (chroma at the aligned height 1088, 2048-byte pitch), and
   coco_tracking's 640x480 planar RGB ([3, h, w], what nvJPEG / torchvision decode to).  Achieved bandwidth = (bytes
   read + bytes written) / time, against the H100 SXM data sheet's 3.35 TB/s.  For NV12 also the alternative: B x two
   torch copies of the plane views into the slot (strided device-to-device copies), alternating with the kernel.
2. End to end, bf16 engine, device tracking, one graph replay per step, the arms alternating, `rounds` rounds of
   `steps` steps, medians of frames/s and of host CPU time per step (process time, every thread):
   mot 1080p on an NV12 capacity runner: device tensors, host arrays (copied into the pinned staging), written in place
   through frame_buffers(); coco_tracking 640x480 on a BGR capacity runner: planar RGB device tensors against BGR arrays.
Prints the card, its power limit and SM clock with the numbers, and one JSON line.  Needs a GPU, except --dry_run, which
prints the byte accounting of the kernel cases and exits."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))

HBM_TBPS = 3.35           # H100 SXM data sheet
# (config, source (h, w), source layout of the kernel case)
CASES = [('mot', (1080, 1920), 'nv12_planes'), ('coco_tracking', (480, 640), 'rgb_planar')]


def stage_bytes(layout, h, w):
  """(bytes read, bytes written) of staging one h x w frame of this source layout: a pure copy, each byte once."""
  n = h * w * 3 // 2 if layout.startswith('nv12') or layout.startswith('i420') else h * w * 3
  return n, n


def card():
  import torch
  name = torch.cuda.get_device_name()
  try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader', '-i',
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    q = ''
  parts = [p.strip() for p in q.split(',')] if q else []
  pl, sm, smax = (parts + ['unknown'] * 3)[:3]
  return '%s, power limit %s, SM clock %s (max %s)' % (name, pl, sm, smax)


def nv12_surfaces(frames, pitch=2048, align=16):
  """NV12 [3h/2, w] arrays -> (Y, UV) device views of decoder-style surfaces: chroma at h rounded up to `align` rows."""
  import torch
  out = []
  for f in frames:
    h, w = f.shape[0] * 2 // 3, f.shape[1]
    ha = (h + align - 1) // align * align
    surf = torch.zeros((ha + h // 2, pitch), dtype=torch.uint8, device='cuda')
    Y, UV = surf[:h, :w], surf[ha:ha + h // 2, :w]
    Y.copy_(torch.from_numpy(f[:h]))
    UV.copy_(torch.from_numpy(f[h:]))
    out.append((Y, UV))
  return out


def planar_rgb(frames):
  import torch
  return [torch.from_numpy(np.ascontiguousarray(f[..., ::-1].transpose(2, 0, 1))).cuda() for f in frames]


def events_ms(arms, rounds, calls):
  """ms per call of each arm: CUDA events around `calls` calls, arms alternating, medians over rounds."""
  import torch
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


def kernel_case(cfg, size, layout, B, rounds, calls, frames):
  """ct_stage_frames (and, for NV12, B x two plane copies) into a capacity slot of B streams."""
  import torch
  from centertrack_b200 import _lib as L
  from centertrack_b200.runner import FRAME_FORMATS, device_frame_source, frame_layout
  h, w = size
  fmt = 'nv12' if layout.startswith('nv12') else 'bgr'
  srcs_t = nv12_surfaces(frames) if fmt == 'nv12' else planar_rgb(frames)
  _, n, step = frame_layout(fmt, h, w)
  cap = (n + 15) // 16 * 16
  slot = torch.zeros(B * cap, dtype=torch.uint8, device='cuda')
  srcs, dsts = (L.FrameSrc * B)(), (L.Frame * B)()
  for b, x in enumerate(srcs_t):
    _, srcs[b] = device_frame_source(x, fmt, 'rgb_planar' if fmt == 'bgr' else 'bgr', slot.device)
    d = dsts[b]
    d.offset, d.h, d.w, d.step, d.format = b * cap, h, w, step, FRAME_FORMATS[fmt]
  lib = L.lib()
  arms = {'ct_stage_frames': lambda: L.check(lib.ct_stage_frames(srcs, dsts, B, L.ptr(slot), slot.numel(),
                                                                  L.stream_ptr()), 'ct_stage_frames')}
  if fmt == 'nv12':
    views = [(slot[b * cap:b * cap + h * w].view(h, w), slot[b * cap + h * w:b * cap + n].view(h // 2, w))
             for b in range(B)]

    def plane_copies():
      for (dy, duv), (sy, suv) in zip(views, srcs_t):
        dy.copy_(sy)
        duv.copy_(suv)
    arms['2B plane copies'] = plane_copies
  ms = events_ms(arms, rounds, calls)
  rd, wr = stage_bytes(layout, h, w)
  moved = B * (rd + wr)
  if fmt == 'nv12':             # the two copies give the same slot bytes
    plane_copies()
    want = slot.clone()
    arms['ct_stage_frames']()
    torch.cuda.synchronize()
    assert torch.equal(slot, want), 'ct_stage_frames and the plane copies disagree'
  return {k: {'ms': v, 'GB_per_s': moved / v / 1e6, 'share_of_3.35TB_s': moved / v / 1e9 / HBM_TBPS}
          for k, v in ms.items()}, moved


def time_arm(fn, steps, runner):
  """(wall s, process CPU s) per step over `steps` steps, ending in a device synchronise."""
  if runner.t:
    runner.fetch()
  t0, c0 = time.perf_counter(), time.process_time()
  for _ in range(steps):
    fn()
  runner.fetch()
  return (time.perf_counter() - t0) / steps, (time.process_time() - c0) / steps


def e2e(cfg, size, B, steps, rounds, frames):
  from centertrack_b200.runner import StreamRunner
  from helpers import make_model
  from yuv_oracle import bgr_to_yuv420
  opt, model, _ = make_model(cfg)
  model = model.cuda()
  H, W = opt.input_h, opt.input_w
  h, w = size
  kw = dict(K=100, precision='bf16', device='cuda', opt=opt, device_tracking=True, frame_sizes=[size] * B,
            max_frame_size=size)
  arms = {}
  if cfg == 'mot':
    nv12 = [bgr_to_yuv420(f, 'nv12') for f in frames]
    r = StreamRunner(model, B, H, W, frame_format='nv12', **kw)
    dev = nv12_surfaces(nv12)
    arms['nv12 device tensors'] = (lambda: r.step_frames(dev), r)
    arms['nv12 host arrays'] = (lambda: r.step_frames(nv12), r)
    arms['nv12 written in place'] = (lambda: r.step_frames(None), r)
    fill = nv12
  else:
    r = StreamRunner(model, B, H, W, **kw)
    dev = planar_rgb(frames)
    arms['rgb_planar device tensors'] = (lambda: r.step_frames(dev, layout='rgb_planar'), r)
    arms['bgr host arrays'] = (lambda: r.step_frames(frames), r)
    fill = frames
  r.warm()
  for s in range(3):            # the in-place arm's decoder wrote every staging slot once
    for v, f in zip(r._views(s, r.frame_sizes), fill):
      v[...] = f
  for fn, rr in arms.values():
    time_arm(fn, 3, rr)
  times = {k: [] for k in arms}
  for _ in range(rounds):
    for k, (fn, rr) in arms.items():
      times[k].append(time_arm(fn, steps, rr))
  h2d = {}
  for k, (fn, rr) in arms.items():
    fn()
    h2d[k] = rr.h2d_bytes_per_step
  rr.fetch()
  return {k: {'frames_per_s': B / float(np.median([t[0] for t in v])),
              'host_cpu_ms_per_step': 1e3 * float(np.median([t[1] for t in v])),
              'h2d_bytes_per_step': h2d[k]} for k, v in times.items()}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--B', type=int, default=32)
  ap.add_argument('--steps', type=int, default=40)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--calls', type=int, default=50, help='ct_stage_frames calls per timed window (>= 50)')
  ap.add_argument('--dry_run', action='store_true', help='print the byte accounting and exit (no GPU needed)')
  a = ap.parse_args()
  if a.calls < 50:
    ap.error('--calls: at least 50')
  if a.dry_run:
    for cfg, (h, w), layout in CASES:
      rd, wr = stage_bytes(layout, h, w)
      print('%s %dx%d %s: B=%d, %d bytes read + %d written per call; at %.2f TB/s >= %.3f ms' %
            (cfg, h, w, layout, a.B, a.B * rd, a.B * wr, HBM_TBPS, a.B * (rd + wr) / HBM_TBPS / 1e9))
    return
  import torch
  assert torch.cuda.is_available(), 'device_frames_time.py needs a GPU'
  from frames_time import frame
  dev = card()
  print('card:', dev)
  out = []
  for cfg, size, layout in CASES:
    frames = [frame(size[0], size[1], 10 + b) for b in range(a.B)]
    from yuv_oracle import bgr_to_yuv420
    kframes = [bgr_to_yuv420(f, 'nv12') for f in frames] if layout.startswith('nv12') else frames
    kern, moved = kernel_case(cfg, size, layout, a.B, a.rounds, a.calls, kframes)
    res = e2e(cfg, size, a.B, a.steps, a.rounds, frames)
    out.append({'config': cfg, 'source': list(size), 'layout': layout, 'B': a.B, 'bytes_per_call': moved,
                'kernel': kern, 'end_to_end': res})
    print('%s: B=%d, %dx%d %s' % (cfg, a.B, size[0], size[1], layout))
    for k, v in kern.items():
      print('  %-18s %8.3f ms per call, %7.1f GB/s (%.0f%% of 3.35 TB/s)' % (k, v['ms'], v['GB_per_s'],
                                                                           100 * v['share_of_3.35TB_s']))
    for k, v in res.items():
      print('  %-28s %8.1f frames/s, host CPU %.2f ms per step, H2D %d bytes per step' %
            (k, v['frames_per_s'], v['host_cpu_ms_per_step'], v['h2d_bytes_per_step']))
  print(json.dumps({'card': dev, 'results': out}))


if __name__ == '__main__':
  main()
