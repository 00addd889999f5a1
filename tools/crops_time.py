"""Cost of track crops in StreamRunner (crop_size: ct_crop_boxes, the last launch of every step):
    python tools/crops_time.py [--B 32] [--K 100] [--crop 256 128] [--steps 40] [--rounds 3] [--calls 200] [--dry_run]

1. ct_crop_boxes alone, CUDA events around `calls` launches after a warm-up, medians over `rounds` rounds: B streams,
   every one with K active tracks (the most a step can crop), boxes of 20 to 400 px inside the frame: mot's 1080p NV12
   frames (the 544x960 runner's) and coco_tracking's 640x480 BGR frames (512x512).  Achieved bandwidth = crop bytes
   written / time, against the H100 SXM data sheet's 3.35 TB/s (the frame reads are not counted).
2. End to end, bf16 engine, device tracking, one graph replay per step: runners with and without crop_size on the same
   frames, the arms alternating, `rounds` rounds of `steps` steps, medians of frames/s; the crops per stream the model
   (synthetic weights) gives are printed beside them.
Prints the card, its power limit and SM clock with the numbers, and one JSON line.  Needs a GPU, except --dry_run, which
prints the byte accounting and exits."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from device_frames_time import HBM_TBPS, card, events_ms, time_arm   # noqa: E402

CASES = [('mot', (1080, 1920), 'nv12'), ('coco_tracking', (480, 640), 'bgr')]


def crop_bytes(B, K, crop):
  return B * K * crop[0] * crop[1] * 3


def kernel_case(size, fmt, B, K, crop, rounds, calls, frames):
  """ct_crop_boxes of B streams x K active tracks from a capacity slot of the frames."""
  import torch
  from centertrack_b200 import _lib as L
  from centertrack_b200.runner import FRAME_FORMATS, frame_layout
  h, w = size
  _, n, step = frame_layout(fmt, h, w)
  cap = (n + 15) // 16 * 16
  slot = torch.zeros(B * cap, dtype=torch.uint8, device='cuda')
  desc = (L.Frame * B)()
  for b, f in enumerate(frames):
    slot[b * cap:b * cap + n].copy_(torch.from_numpy(np.ascontiguousarray(f).reshape(-1)))
    d = desc[b]
    d.offset, d.h, d.w, d.step, d.format = b * cap, h, w, step, FRAME_FORMATS[fmt]
  rng = np.random.RandomState(3)
  rows = np.zeros((B, K, L.CT_TRK_FLOATS), np.float32)
  sz = rng.uniform(20, 400, (B, K, 2))
  x0, y0 = rng.uniform(0, w - sz[..., 0]), rng.uniform(0, h - np.minimum(sz[..., 1], h - 1))
  rows[..., L.CT_TRK_BBOX:L.CT_TRK_BBOX + 4] = np.stack([x0, y0, x0 + sz[..., 0], y0 + sz[..., 1]], -1)
  rows[..., L.CT_TRK_ACTIVE] = 1
  d_rows = torch.from_numpy(rows).cuda()
  d_counts = torch.full((B, 2), K, dtype=torch.int32, device='cuda')
  d_frames = torch.frombuffer(bytearray(bytes(desc)), dtype=torch.uint8).cuda()
  out = torch.zeros((B, K) + tuple(crop) + (3,), dtype=torch.uint8, device='cuda')
  out_counts = torch.zeros((B,), dtype=torch.int32, device='cuda')
  cd = L.CropDesc()
  cd.buf, cd.buf_bytes, cd.frames = slot.data_ptr(), slot.numel(), d_frames.data_ptr()
  cd.rows, cd.row_floats, cd.rows_per_stream = d_rows.data_ptr(), L.CT_TRK_FLOATS, K
  cd.counts, cd.counts_stride, cd.active_col = d_counts.data_ptr(), 2, L.CT_TRK_ACTIVE
  cd.K, cd.out_h, cd.out_w, cd.out, cd.out_counts = K, crop[0], crop[1], out.data_ptr(), out_counts.data_ptr()
  lib = L.lib()
  ms = events_ms({'ct_crop_boxes': lambda: L.check(lib.ct_crop_boxes(C.byref(cd), None, B, B, L.stream_ptr()),
                                                   'ct_crop_boxes')}, rounds, calls)['ct_crop_boxes']
  assert int(out_counts.sum()) == B * K
  moved = crop_bytes(B, K, crop)
  return {'ms': ms, 'GB_per_s': moved / ms / 1e6, 'share_of_3.35TB_s': moved / ms / 1e9 / HBM_TBPS}


def e2e(cfg, size, fmt, B, K, crop, steps, rounds, frames):
  from centertrack_b200.runner import StreamRunner
  from helpers import make_model
  opt, model, _ = make_model(cfg)
  model = model.cuda()
  kw = dict(K=K, precision='bf16', device='cuda', opt=opt, device_tracking=True, frame_sizes=[size] * B,
            max_frame_size=size, frame_format=fmt)
  runners = {'without crop_size': StreamRunner(model, B, opt.input_h, opt.input_w, **kw),
             'crop_size=%dx%d' % tuple(crop): StreamRunner(model, B, opt.input_h, opt.input_w, crop_size=tuple(crop),
                                                           **kw)}
  for r in runners.values():
    r.warm()
    time_arm(lambda r=r: r.step_frames(frames), 3, r)
  times = {k: [] for k in runners}
  for _ in range(rounds):
    for k, r in runners.items():
      times[k].append(time_arm(lambda r=r: r.step_frames(frames), steps, r)[0])
  out = {k: {'frames_per_s': B / float(np.median(v)), 'ms_per_step': 1e3 * float(np.median(v)),
             'launches_per_step': runners[k].launches_per_step, 'd2h_bytes_per_step': runners[k].d2h_bytes_per_step}
         for k, v in times.items()}
  cut = runners['crop_size=%dx%d' % tuple(crop)]
  out['crops_per_stream'] = float(cut.fetch_crops()[1].mean())
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--B', type=int, default=32)
  ap.add_argument('--K', type=int, default=100)
  ap.add_argument('--crop', type=int, nargs=2, default=[256, 128])
  ap.add_argument('--steps', type=int, default=40)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--calls', type=int, default=200, help='ct_crop_boxes launches per timed window (>= 50)')
  ap.add_argument('--dry_run', action='store_true', help='print the byte accounting and exit (no GPU needed)')
  a = ap.parse_args()
  if a.calls < 50:
    ap.error('--calls: at least 50')
  moved = crop_bytes(a.B, a.K, a.crop)
  if a.dry_run:
    print('B=%d, K=%d, %dx%d crops: %d bytes written per launch; at %.2f TB/s >= %.3f ms' %
          (a.B, a.K, a.crop[0], a.crop[1], moved, HBM_TBPS, moved / HBM_TBPS / 1e9))
    return
  import torch
  assert torch.cuda.is_available(), 'crops_time.py needs a GPU'
  from frames_time import frame
  from yuv_oracle import bgr_to_yuv420
  dev = card()
  print('card:', dev)
  out = []
  for cfg, size, fmt in CASES:
    frames = [frame(size[0], size[1], 10 + b) for b in range(a.B)]
    if fmt == 'nv12':
      frames = [bgr_to_yuv420(f, 'nv12') for f in frames]
    kern = kernel_case(size, fmt, a.B, a.K, a.crop, a.rounds, a.calls, frames)
    res = e2e(cfg, size, fmt, a.B, a.K, a.crop, a.steps, a.rounds, frames)
    out.append({'config': cfg, 'source': list(size), 'format': fmt, 'B': a.B, 'K': a.K, 'crop': a.crop,
                'bytes_per_launch': moved, 'kernel': kern, 'end_to_end': res})
    print('%s: B=%d, %dx%d %s, K=%d crops of %dx%d per stream' % (cfg, a.B, size[0], size[1], fmt, a.K, *a.crop))
    print('  ct_crop_boxes %8.3f ms per launch, %7.1f GB/s written (%.0f%% of 3.35 TB/s)' %
          (kern['ms'], kern['GB_per_s'], 100 * kern['share_of_3.35TB_s']))
    for k, v in res.items():
      if isinstance(v, dict):
        print('  %-22s %8.1f frames/s, %.3f ms per step, %d launches, D2H %d bytes per step' %
              (k, v['frames_per_s'], v['ms_per_step'], v['launches_per_step'], v['d2h_bytes_per_step']))
    print('  crops per stream in the last step: %.1f' % res['crops_per_stream'])
  print(json.dumps({'card': dev, 'results': out}))


if __name__ == '__main__':
  main()
