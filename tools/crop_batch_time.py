"""Cost of StreamRunner's crops as one packed, normalised fp16 batch (crop_format), against ct_crop_boxes' uint8 crops
plus the torch chain a consumer would otherwise run on them:
    python tools/crop_batch_time.py [--B 32] [--K 100] [--crop 256 128] [--steps 40] [--rounds 3] [--calls 50]
                                    [--dry_run]

The chain, per stream b: crops[b, :counts[b]].permute(0, 3, 1, 2).flip(1).float() / 255, torchvision's
Normalize(ImageNet mean, std), .half(); then torch.cat of the B slices: one RGB fp16 NCHW batch, what
crop_format={'dtype': torch.float16, 'channels': 'rgb', ImageNet mean / std} writes in the crop launch.

1. The launches alone, CUDA events around `calls` calls after a warm-up, the arms alternating, medians over `rounds`
   rounds: ct_crop_boxes_tensor (offsets + crop pass) against ct_crop_boxes + the chain, and ct_crop_boxes alone.  B
   streams of K active tracks each, boxes of 20 to 400 px inside the frame: mot's 1080p NV12 frames (the 544x960
   runner's) and coco_tracking's 640x480 BGR frames (512x512), as tools/crops_time.py.
2. End to end, bf16 engine, device tracking, one graph replay per step, frames/s of runners on the same frames, the
   arms alternating, `rounds` rounds of `steps` steps, medians: without crops (the baseline), crop_size alone, crop_size
   + the chain on each step's crops (previous_crops), and crop_format (previous_crops gives the batch).
Prints the card, its power limit and SM clock with the numbers, and one JSON line.  Needs a GPU, except --dry_run, which
prints the byte accounting and exits."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from crops_time import CASES, crop_bytes   # noqa: E402
from device_frames_time import card, events_ms   # noqa: E402

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
FORMAT = None   # crop_format, set in main (needs torch)


def chain(crops, counts):
  """The consumer's torch chain on uint8 BGR crops [B, K, h, w, 3] and host counts: one RGB fp16 NCHW batch."""
  import torch
  from torchvision.transforms import functional as TF
  return torch.cat([TF.normalize(crops[b, :counts[b]].permute(0, 3, 1, 2).flip(1).float() / 255, MEAN, STD).half()
                    for b in range(len(counts))])


def kernel_case(size, fmt, B, K, crop, rounds, calls, frames):
  """ct_crop_boxes_tensor against ct_crop_boxes + chain (and alone) on B streams x K active tracks of the frames."""
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
  u8 = torch.zeros((B, K) + tuple(crop) + (3,), dtype=torch.uint8, device='cuda')
  batch = torch.zeros((B * K, 3) + tuple(crop), dtype=torch.float16, device='cuda')
  offsets = torch.zeros((B + 1,), dtype=torch.int32, device='cuda')
  out_counts = torch.zeros((B,), dtype=torch.int32, device='cuda')
  cd = L.CropDesc()
  cd.buf, cd.buf_bytes, cd.frames = slot.data_ptr(), slot.numel(), d_frames.data_ptr()
  cd.rows, cd.row_floats, cd.rows_per_stream = d_rows.data_ptr(), L.CT_TRK_FLOATS, K
  cd.counts, cd.counts_stride, cd.active_col = d_counts.data_ptr(), 2, L.CT_TRK_ACTIVE
  cd.K, cd.out_h, cd.out_w, cd.out, cd.out_counts = K, crop[0], crop[1], u8.data_ptr(), out_counts.data_ptr()
  ct = L.CropTensor()
  ct.type, ct.order, ct.rows_cap = L.CT_CROP_F16, L.CT_CROP_RGB, B * K
  ct.mean[:], ct.std[:] = MEAN, STD
  ct.out, ct.out_offsets = batch.data_ptr(), offsets.data_ptr()
  lib = L.lib()
  host_counts = np.full((B,), K, np.int32)           # what fetch_crops() hands the consumer
  res = {}

  def boxes():
    L.check(lib.ct_crop_boxes(C.byref(cd), None, B, B, L.stream_ptr()), 'ct_crop_boxes')

  def boxes_chain():
    boxes()
    res['chain'] = chain(u8, host_counts)

  def fused():
    L.check(lib.ct_crop_boxes_tensor(C.byref(cd), C.byref(ct), None, B, B, L.stream_ptr()), 'ct_crop_boxes_tensor')

  ms = events_ms({'ct_crop_boxes_tensor': fused, 'ct_crop_boxes + chain': boxes_chain, 'ct_crop_boxes': boxes},
                 rounds, calls)
  torch.cuda.synchronize()
  assert int(offsets[-1]) == B * K and int(out_counts.sum()) == B * K
  # the chain on the GPU may divide by multiplying with a reciprocal: count the elements it rounds differently
  diff = res['chain'] != batch
  ulp = (res['chain'].view(torch.int16).int() - batch.view(torch.int16).int()).abs().max()
  return {'ms': ms, 'speedup_vs_chain': ms['ct_crop_boxes + chain'] / ms['ct_crop_boxes_tensor'],
          'fp16_bytes_written': batch.numel() * 2, 'u8_bytes_written': crop_bytes(B, K, crop),
          'fused_GB_per_s': batch.numel() * 2 / ms['ct_crop_boxes_tensor'] / 1e6,
          'chain_elements_differing': int(diff.sum()), 'chain_max_ulp': int(ulp)}


def e2e(cfg, size, fmt, B, K, crop, steps, rounds, frames):
  import torch
  from centertrack_b200.runner import StreamRunner
  from helpers import make_model
  opt, model, _ = make_model(cfg)
  model = model.cuda()
  kw = dict(K=K, precision='bf16', device='cuda', opt=opt, device_tracking=True, frame_sizes=[size] * B,
            max_frame_size=size, frame_format=fmt)
  crop = tuple(crop)
  runners = {'without crops': StreamRunner(model, B, opt.input_h, opt.input_w, **kw),
             'crop_size': StreamRunner(model, B, opt.input_h, opt.input_w, crop_size=crop, **kw),
             'crop_size + torch chain': StreamRunner(model, B, opt.input_h, opt.input_w, crop_size=crop, **kw),
             'crop_format fp16': StreamRunner(model, B, opt.input_h, opt.input_w, crop_size=crop,
                                              crop_format=FORMAT, **kw)}
  out_batches = {}

  def step(k, r):
    r.step_frames(frames)
    if k == 'crop_size + torch chain' and r.t >= 2:
      crops, counts = r.previous_crops()
      out_batches[k] = chain(crops, counts)
    elif k == 'crop_format fp16' and r.t >= 2:
      out_batches[k] = r.previous_crops()[0]

  def arm(k, r, n):
    """Seconds per step over n steps, ending when the step and the chain queued on torch's stream are done."""
    if r.t:
      r.fetch()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
      step(k, r)
    r.fetch()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n

  for k, r in runners.items():
    r.warm()
    arm(k, r, 3)
  times = {k: [] for k in runners}
  for _ in range(rounds):
    for k, r in runners.items():
      times[k].append(arm(k, r, steps))
  out = {k: {'frames_per_s': B / float(np.median(v)), 'ms_per_step': 1e3 * float(np.median(v)),
             'launches_per_step': runners[k].launches_per_step, 'd2h_bytes_per_step': runners[k].d2h_bytes_per_step}
         for k, v in times.items()}
  out['crops_per_stream'] = float(runners['crop_format fp16'].fetch_crops()[1].mean())
  out['batch_rows'] = {k: int(v.shape[0]) for k, v in out_batches.items()}
  return out


def main():
  global FORMAT
  ap = argparse.ArgumentParser()
  ap.add_argument('--B', type=int, default=32)
  ap.add_argument('--K', type=int, default=100)
  ap.add_argument('--crop', type=int, nargs=2, default=[256, 128])
  ap.add_argument('--steps', type=int, default=40)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--calls', type=int, default=50, help='launches per timed window (>= 50)')
  ap.add_argument('--dry_run', action='store_true', help='print the byte accounting and exit (no GPU needed)')
  a = ap.parse_args()
  if a.calls < 50:
    ap.error('--calls: at least 50')
  u8 = crop_bytes(a.B, a.K, a.crop)
  if a.dry_run:
    print('B=%d, K=%d, %dx%d crops: uint8 %d bytes, fp16 batch %d bytes, fp32 intermediate %d bytes' %
          (a.B, a.K, a.crop[0], a.crop[1], u8, 2 * u8, 4 * u8))
    return
  import torch
  assert torch.cuda.is_available(), 'crop_batch_time.py needs a GPU'
  from frames_time import frame
  from yuv_oracle import bgr_to_yuv420
  FORMAT = {'dtype': torch.float16, 'channels': 'rgb', 'mean': MEAN, 'std': STD}
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
                'kernel': kern, 'end_to_end': res})
    print('%s: B=%d, %dx%d %s, K=%d crops of %dx%d per stream' % (cfg, a.B, size[0], size[1], fmt, a.K, *a.crop))
    for k, v in kern['ms'].items():
      print('  %-24s %8.3f ms per call' % (k, v))
    print('  fused / (boxes + chain): %.2fx faster; fp16 batch written at %.1f GB/s; chain elements rounded '
          'differently: %d (max %d ulp)' % (kern['speedup_vs_chain'], kern['fused_GB_per_s'],
                                            kern['chain_elements_differing'], kern['chain_max_ulp']))
    for k, v in res.items():
      if isinstance(v, dict) and 'frames_per_s' in v:
        print('  %-24s %8.1f frames/s, %.3f ms per step, %d launches, D2H %d bytes per step' %
              (k, v['frames_per_s'], v['ms_per_step'], v['launches_per_step'], v['d2h_bytes_per_step']))
    print('  crops per stream in the last step: %.1f; batch rows %s' % (res['crops_per_stream'], res['batch_rows']))
  print(json.dumps({'card': dev, 'results': out}))


if __name__ == '__main__':
  main()
