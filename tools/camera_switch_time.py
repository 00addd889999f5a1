"""Cost and benefit of StreamRunner streams that change frame size at a video start (max_frame_size):
    python tools/camera_switch_time.py [--B 32] [--steps 40] [--rounds 7] [--videos 64] [--min_len 100] [--max_len 400]

1. device time per call of ct_pack_stem_frames_dev, B streams, mot 1920x1080 -> 544x960 and KITTI 1242x375 ->
   384x1280, CUDA events around 50 calls, medians over rounds;
2. steady-state frames/s of a capacity runner (max_frame_size = 1080x1920) against a fixed runner, B uniform 1920x1080
   streams, --config mot, bf16, device tracking, graphs; alternating rounds of `steps` steps, medians and the spread;
3. a MOT17-style schedule through track_videos: `videos` synthetic videos of min_len..max_len frames, a quarter of them
   640x480 and the rest 1920x1080 (seeded frames cycled per video), on a capacity runner against a fixed runner whose
   streams are split by size (3/4 at 1920x1080); frames/s of real frames and idle stream-steps, for the 640x480 videos
   interleaved with the others and for them listed together; then the same with half of the videos at 640x480, a mix
   the fixed runner's split was not provisioned for.
Prints the card and its power limit with the numbers, and one JSON line.  Needs a GPU."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from frames_time import card, frame                    # noqa  (also puts the repository and tests/ on sys.path)
from centertrack_b200 import _lib as L                 # noqa
from helpers import make_model, make_opt               # noqa

# (source size, input size): mot's and kitti_tracking's default inputs
KERNEL_CASES = {'mot': ((1080, 1920), (544, 960)), 'kitti': ((375, 1242), (384, 1280))}


def pack_times(cfg, B, rounds, n=50):
  from centertrack_b200.dataset_info import get_dataset
  from centertrack_b200.detector import frame_geometry
  (h, w), (ih, iw) = KERNEL_CASES[cfg]
  opt = make_opt('mot', ['--input_h', str(ih), '--input_w', str(iw)])
  meta, minv = frame_geometry(opt, h, w)
  H, W = meta['inp_height'], meta['inp_width']
  cap = (h * w * 3 + 15) // 16 * 16
  frames = (L.Frame * B)()
  for b, f in enumerate(frames):
    f.offset, f.h, f.w, f.step = b * cap, h, w, 3 * w
    f.minv[:] = minv.tolist()
  dfr = torch.from_numpy(np.frombuffer(bytes(frames), np.uint8).copy()).cuda()
  g = torch.Generator(device='cuda').manual_seed(1)
  cur = torch.randint(0, 256, (B * cap,), dtype=torch.uint8, device='cuda', generator=g)
  prev = torch.randint(0, 256, (B * cap,), dtype=torch.uint8, device='cuda', generator=g)
  hm = torch.rand((B, 1, H, W), device='cuda')
  out = torch.empty((B, H, W, 8), dtype=torch.bfloat16, device='cuda')
  ds = get_dataset(opt.dataset)
  mean = np.ascontiguousarray(ds.mean, np.float32).reshape(3)
  std = np.ascontiguousarray(ds.std, np.float32).reshape(3)
  ms = C.c_void_p(mean.ctypes.data), C.c_void_p(std.ctypes.data)
  lib = L.lib()

  def pack():
    L.check(lib.ct_pack_stem_frames_dev(L.ptr(cur), L.ptr(prev), L.ptr(dfr), B, cur.numel(), *ms, L.ptr(hm),
                                        L.ptr(out), H, W, L.stream_ptr()))

  pack()
  torch.cuda.synchronize()
  t = []
  for _ in range(rounds):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
      pack()
    e1.record()
    torch.cuda.synchronize()
    t.append(e0.elapsed_time(e1) / n)
  return {'source': [h, w], 'input': [H, W], 'ms_per_call': float(np.median(t))}


def steady_state(model, opt, B, steps, rounds):
  from centertrack_b200.runner import StreamRunner
  H, W = opt.input_h, opt.input_w
  frames = [frame(1080, 1920, 10 + b) for b in range(B)]
  kw = dict(K=100, precision='bf16', device='cuda', opt=opt, device_tracking=True, frame_sizes=[(1080, 1920)] * B)
  runners = {'fixed': StreamRunner(model, B, H, W, **kw),
             'capacity': StreamRunner(model, B, H, W, max_frame_size=(1080, 1920), **kw)}

  def run(r, n):
    if r.t:
      r.fetch()
    t0 = time.perf_counter()
    for _ in range(n):
      r.step_frames(frames)
    r.fetch()
    return (time.perf_counter() - t0) / n

  for r in runners.values():
    r.warm()
    run(r, 3)
  t = {k: [] for k in runners}
  for _ in range(rounds):
    for k, r in runners.items():
      t[k].append(run(r, steps))
  res = {'frames_per_s': {k: B / float(np.median(v)) for k, v in t.items()},
         'frames_per_s_rounds': {k: sorted(B / x for x in v) for k, v in t.items()},
         'h2d_bytes_per_step': {k: r.h2d_bytes_per_step for k, r in runners.items()},
         'launches_per_step': {k: r.launches_per_step for k, r in runners.items()}}
  del runners
  return res


def schedule(model, opt, B, n_videos, min_len, max_len, order, small_every=4):
  """order 'interleaved': every `small_every`-th video is 640x480; 'grouped': the same videos, the 640x480 ones listed together
  after the first half of the 1920x1080 ones (as a dataset listing its sequences camera by camera)."""
  from centertrack_b200.runner import StreamRunner
  from centertrack_b200.videos import Video, track_videos
  H, W = opt.input_h, opt.input_w
  big, small = (1080, 1920), (480, 640)
  rng = np.random.RandomState(17)
  spec = [(small if v % small_every == small_every - 1 else big, int(rng.randint(min_len, max_len + 1))) for v in range(n_videos)]
  if order == 'grouped':
    bigs, smalls = [x for x in spec if x[0] == big], [x for x in spec if x[0] == small]
    spec = bigs[:len(bigs) // 2] + smalls + bigs[len(bigs) // 2:]
  pool = {sz: [frame(sz[0], sz[1], 100 * i + sz[0]) for i in range(4)] for sz in (big, small)}
  fed = {}

  def frames_of(size, v, n):          # one video's frames, bound per video
    fed[size] = fed.get(size, 0) + 1
    for i in range(n):
      yield pool[size][(v + i) % 4]

  def videos():
    return [Video(v, frames_of(size, v, n)) for v, (size, n) in enumerate(spec)]

  n_small = B // 4
  kw = dict(K=100, precision='bf16', device='cuda', opt=opt, device_tracking=True)
  arms = {'capacity': dict(frame_sizes=[big] * B, max_frame_size=big),
          'fixed split by size': dict(frame_sizes=[big] * (B - n_small) + [small] * n_small)}
  total = sum(n for _, n in spec)
  want = {big: sum(1 for x in spec if x[0] == big), small: sum(1 for x in spec if x[0] == small)}
  out = {}
  for k, a in arms.items():
    r = StreamRunner(model, B, H, W, **dict(kw, **a))
    r.warm()
    fed.clear()
    t0 = time.perf_counter()
    n = sum(1 for _ in track_videos(r, videos()))
    dt = time.perf_counter() - t0
    assert n == total and fed == want, (n, total, fed, want)     # the size mix that was actually fed
    steps = r.t
    out[k] = {'steps': steps, 'real_frames_per_s': total / dt, 'idle_stream_steps': steps * B - total,
              'seconds': dt}
    del r
  return {'order': order, 'small_every': small_every, 'videos': n_videos, 'frames': total, 'small_videos': want[small], 'arms': out}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--B', type=int, default=32)
  ap.add_argument('--steps', type=int, default=40)
  ap.add_argument('--rounds', type=int, default=7)
  ap.add_argument('--videos', type=int, default=64)
  ap.add_argument('--min_len', type=int, default=100)
  ap.add_argument('--max_len', type=int, default=400)
  a = ap.parse_args()
  assert torch.cuda.is_available(), 'camera_switch_time.py needs a GPU'
  dev = card()
  print('card:', dev)
  res = {'card': dev, 'B': a.B, 'pack': {cfg: pack_times(cfg, a.B, a.rounds) for cfg in KERNEL_CASES}}
  for cfg, r in res['pack'].items():
    print('%s %s -> %s, B=%d: ct_pack_stem_frames_dev %.3f ms per call' % (cfg, r['source'], r['input'], a.B,
                                                                          r['ms_per_call']))
  opt, model, _ = make_model('mot')
  model = model.cuda()
  res['steady'] = steady_state(model, opt, a.B, a.steps, a.rounds)
  for k, v in res['steady']['frames_per_s'].items():
    r = res['steady']['frames_per_s_rounds'][k]
    print('steady 1920x1080, B=%d: %-9s %8.1f frames/s (median of %d rounds; min %.1f, max %.1f)' %
          (a.B, k, v, len(r), r[0], r[-1]))
  # a quarter of the videos at 640x480 (the mix the fixed runner's 3:1 split is provisioned for), interleaved and
  # grouped; then half of them (a mix the split was not provisioned for)
  res['schedule'] = [schedule(model, opt, a.B, a.videos, a.min_len, a.max_len, o, e)
                     for o, e in (('interleaved', 4), ('grouped', 4), ('interleaved', 2))]
  for sc in res['schedule']:
    for k, v in sc['arms'].items():
      print('MOT17-style schedule, %s (%d videos, %d at 640x480, %d frames): %-20s %6d steps, %8.1f real frames/s, '
            '%6d idle stream-steps' % (sc['order'], sc['videos'], sc['small_videos'], sc['frames'], k, v['steps'],
                                       v['real_frames_per_s'], v['idle_stream_steps']))
  print(json.dumps(res))


if __name__ == '__main__':
  main()
