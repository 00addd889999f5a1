"""-m gpu: NV12 / I420 camera frames.  The device-descriptor entry points (ct_warp_frames_normalize,
ct_pack_stem_frames_dev, ct_pack_stem_frames_flip_dev) against the oracle chain yuv420_to_bgr -> warp_affine_u8 ->
normalize_chw / stem_pixels with no tolerance, formats mixed in one launch; and a 4:2:0 StreamRunner against a BGR
capacity runner fed cv2.cvtColor of the same frames, records and tracks bit for bit."""
import ctypes as C

import cv2
import numpy as np
import pytest
import torch

import ct_oracle as co
from centertrack_b200 import _lib as L
from helpers import make_opt, warp_maps
from test_gpu_camera_switch import _model, _pub
from test_gpu_frames import _frame
from yuv_oracle import bgr_to_yuv420, random_yuv420, yuv420_to_bgr

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')
MEAN = np.float32([0.408, 0.447, 0.470])
STD = np.float32([0.289, 0.274, 0.278])
MS = (C.c_void_p(MEAN.ctypes.data), C.c_void_p(STD.ctypes.data))
FMT = {'bgr': L.CT_FRAME_BGR, 'nv12': L.CT_FRAME_NV12, 'i420': L.CT_FRAME_I420}
CODES = {'nv12': cv2.COLOR_YUV2BGR_NV12, 'i420': cv2.COLOR_YUV2BGR_I420}


def _bits(got, want, ctx):
  g = got.cpu()
  g = g.view(torch.int16).numpy() if g.dtype == torch.bfloat16 else g.numpy().view(np.int32)
  w = want.view(np.int32) if want.dtype == np.float32 else want
  assert g.shape == w.shape, (ctx, g.shape, w.shape)
  bad = g != w
  assert not bad.any(), '%s: %d values differ, first at %s' % (ctx, int(bad.sum()), np.argwhere(bad)[:4].tolist())


def _source(fmt, h, w, pitch, seed):
  """-> (the frame's bytes at a row pitch of `pitch`, its BGR image as the oracle sees it)."""
  if fmt == 'bgr':
    img = np.random.RandomState(seed).randint(0, 256, size=(h, w, 3)).astype(np.uint8)
    buf = np.full((h, pitch), 0xA5, np.uint8)
    buf[:, :3 * w] = img.reshape(h, 3 * w)
    return buf, img
  buf = random_yuv420(h, w, seed, pitch)
  return buf, yuv420_to_bgr(buf[:, :w], h, w, fmt)


def _ragged(streams, seed):
  """streams: [(fmt, (h, w), pitch, minv)] -> (cur, prev device buffers, device ct_frame array, bytes, [cur BGR],
  [prev BGR])."""
  frames = (L.Frame * len(streams))()
  bufs, imgs = [bytearray(), bytearray()], [[], []]
  for b, (fmt, (h, w), pitch, minv) in enumerate(streams):
    off = len(bufs[0])
    for k in range(2):
      raw, bgr = _source(fmt, h, w, pitch, seed + 2 * b + k)
      imgs[k].append(bgr)
      bufs[k] += raw.tobytes() + bytes((-raw.size) % 16)
    f = frames[b]
    f.offset, f.h, f.w, f.step, f.format = off, h, w, pitch, FMT[fmt]
    f.minv[:] = [float(v) for v in minv]
  dev = [torch.frombuffer(bytearray(bb), dtype=torch.uint8).to(DEV) for bb in bufs]
  fdev = torch.frombuffer(bytearray(bytes(frames)), dtype=torch.uint8).to(DEV)
  return dev[0], dev[1], fdev, len(bufs[0]), imgs[0], imgs[1]


def _policy_streams(opt):
  from centertrack_b200.detector import frame_geometry
  spec = [('nv12', (1080, 1920), 1984), ('i420', (376, 1242), 1248), ('bgr', (900, 1600), 4800),
          ('i420', (480, 640), 640), ('nv12', (302, 458), 467), ('i420', (1920, 1080), 1080), ('nv12', (2, 38), 38),
          ('i420', (30, 2), 2), ('bgr', (375, 1242), 3729), ('nv12', (720, 1280), 1280)]
  return [(fmt, hw, pitch, frame_geometry(opt, *hw)[1]) for fmt, hw, pitch in spec]


GROUPS = ['mot_544x960', 'kitti_384x1280', 'keep_res', 'maps_320x200']


def _group(name):
  if name == 'maps_320x200':               # the adversarial inverse maps (ties, rotation, shear, mirror, outside)
    sel = [m for m in warp_maps() if m[2] == (400, 500) and m[3] == (320, 200)]
    fmts = ['nv12', 'i420', 'bgr']
    return [(fmts[k % 3], hw, (500 if k % 3 < 2 else 1500) + 2 * k, m) for k, (_, m, hw, _) in enumerate(sel)], \
        (320, 200)
  if name == 'keep_res':                   # --keep_res: a 1080p source into its own padded input
    opt = make_opt('mot', ['--keep_res'])
    from centertrack_b200.detector import frame_geometry
    meta, m = frame_geometry(opt, 1080, 1920)
    streams = [('nv12', (1080, 1920), 1920, m), ('i420', (1080, 1920), 1952, m), ('bgr', (1080, 1920), 5760, m)]
    return streams, (meta['inp_height'], meta['inp_width'])
  H, W = (544, 960) if name.startswith('mot') else (384, 1280)
  return _policy_streams(make_opt('mot', ['--input_h', str(H), '--input_w', str(W)])), (H, W)


def _check_entry_points(streams, H, W, seed, ctx):
  B = len(streams)
  cur, prev, fdev, nbytes, cur_bgr, prev_bgr = _ragged(streams, seed)
  want_cur = [co.normalize_chw(co.warp_affine_u8(im, s[3], H, W), MEAN, STD) for im, s in zip(cur_bgr, streams)]
  want_prev = [co.normalize_chw(co.warp_affine_u8(im, s[3], H, W), MEAN, STD) for im, s in zip(prev_bgr, streams)]
  hm = torch.rand((B, 1, H, W), device=DEV)
  hm_np = hm.cpu().numpy()
  lib, st = L.lib(), L.stream_ptr()
  img = torch.full((B, 3, H, W), 7.0, device=DEV)
  L.check(lib.ct_warp_frames_normalize(L.ptr(cur), L.ptr(fdev), B, nbytes, *MS, L.ptr(img), H, W, st))
  for b in range(B):
    _bits(img[b], want_cur[b], (ctx, 'warp_frames', streams[b][0], b))
  for fname, flip in (('ct_pack_stem_frames_dev', False), ('ct_pack_stem_frames_flip_dev', True)):
    for pv, h in ((prev, hm), (None, None)):
      out = torch.full(((2 if flip else 1) * B, H, W, 8), -7.0, dtype=torch.bfloat16, device=DEV)
      L.check(getattr(lib, fname)(L.ptr(cur), L.ptr(pv), L.ptr(fdev), B, nbytes, *MS, L.ptr(h), L.ptr(out), H, W, st))
      for b in range(B):
        want = co.stem_pixels(want_cur[b], want_prev[b] if pv is not None else None,
                              hm_np[b, 0] if h is not None else None, flip=flip)
        _bits(out[b], want[0] if flip else want, (ctx, fname, streams[b][0], b, pv is None))
        if flip:
          _bits(out[B + b], want[1], (ctx, fname, 'mirror', streams[b][0], b))


@pytest.mark.parametrize('group', GROUPS)
def test_device_entry_points_equal_the_oracle_on_mixed_formats(group):
  """BGR, NV12 and I420 streams in one launch (padded and odd pitches, 2 x N and N x 2 frames), on the resolution
  policies and the adversarial maps: ct_warp_frames_normalize, and both _dev packs with and without the previous frame
  and pre_hm, both halves of the flip."""
  streams, (H, W) = _group(group)
  _check_entry_points(streams, H, W, 700, group)


def test_device_entry_points_at_49_streams():
  from centertrack_b200.detector import frame_geometry
  opt = make_opt('coco_tracking', ['--input_h', '32', '--input_w', '48'])
  sizes = [(6, 8), (18, 24), (32, 40), (2, 2), (2, 10), (12, 2), (40, 64), (34, 48), (20, 30), (48, 32), (10, 62)]
  fmts = ['nv12', 'i420', 'bgr']
  streams = []
  for b in range(49):
    fmt, hw = fmts[b % 3], sizes[b % len(sizes)]
    pitch = (3 if fmt == 'bgr' else 1) * hw[1] + (b % 4) * 5
    streams.append((fmt, hw, pitch, frame_geometry(opt, *hw)[1]))
  _check_entry_points(streams, 32, 48, 900, 'B49')


def test_invalid_yuv_descriptors_give_zeros_and_read_nothing():
  """Odd sizes, an unknown format, a pitch below w, a frame one byte past buf_bytes (the bound is smaller than the
  allocation, so a faulty bound shows as wrong bytes) give zeros; a frame ending exactly at the bound is read."""
  H, W = 64, 96
  opt = make_opt('mot', ['--input_h', str(H), '--input_w', str(W)])
  from centertrack_b200.detector import frame_geometry
  m = frame_geometry(opt, 40, 60)[1]
  fmts = ['nv12', 'i420', 'nv12', 'i420', 'nv12', 'i420', 'nv12', 'nv12']
  streams = [(f, (40, 60), 64, m) for f in fmts]
  cur, prev, _, _, _, _ = _ragged(streams, 3)
  frames = (L.Frame * len(streams))()
  for b, f in enumerate(frames):
    f.offset, f.h, f.w, f.step, f.format = b * 3840, 40, 60, 64, FMT[fmts[b]]
    f.minv[:] = m.tolist()
  limit = frames[4].offset + 59 * 64 + 60            # stream 4's last chroma row ends exactly at the bound: valid
  frames[0].h = 39
  frames[1].w = 61
  frames[2].format = 3
  frames[3].step = 59                                 # < w
  frames[5].offset = limit - 59 * 64 - 59             # one byte past the bound
  frames[6].offset = -16
  frames[7].format = -1
  bad = [0, 1, 2, 3, 5, 6, 7]
  fdev = torch.frombuffer(bytearray(bytes(frames)), dtype=torch.uint8).to(DEV)
  B, lib, st = len(streams), L.lib(), L.stream_ptr()
  hm = torch.rand((B, 1, H, W), device=DEV)
  for fn, n in ((lib.ct_pack_stem_frames_dev, B), (lib.ct_pack_stem_frames_flip_dev, 2 * B)):
    got = torch.full((n, H, W, 8), -7.0, dtype=torch.bfloat16, device=DEV)
    L.check(fn(L.ptr(cur), L.ptr(prev), L.ptr(fdev), B, limit, *MS, L.ptr(hm), L.ptr(got), H, W, st))
    for b in range(B):
      assert (not bool(got[b].view(torch.int16).any())) == (b in bad), (fn, b)
  img = torch.full((B, 3, H, W), -3.0, device=DEV)
  L.check(lib.ct_warp_frames_normalize(L.ptr(cur), L.ptr(fdev), B, limit, *MS, L.ptr(img), H, W, st))
  for b in range(B):
    assert (not bool(img[b].view(torch.int32).any())) == (b in bad), b


# ------------------------------------------------------------------------------------------------ the runner
H, W, K, B = 128, 160, 40, 3
S0, S1, S2 = (120, 200), (96, 130), (160, 128)
MAXF = (160, 200)
# per step: (sizes, starts, idle); stream 1 starts a video at another size (and camera) at step 2, stream 2 is idle at
# step 3 (on idle runners) and comes back with a video start at step 4 at another size
SCHEDULE = [([S0, S2, S0], [], []), ([S0, S2, S0], [], []), ([S0, S1, S0], [1], []), ([S0, S1, S0], [], [2]),
            ([S0, S1, S2], [2], []), ([S0, S1, S2], [], [])]


def _yuv(fmt, size, seed):
  return bgr_to_yuv420(_frame(size[0], size[1], seed), fmt)


def _make(model, opt, precision, graph, fmt, idle):
  from centertrack_b200.runner import StreamRunner
  r = StreamRunner(model, B, H, W, K=K, precision=precision, device='cuda', opt=opt, device_tracking=True,
                   use_graph=graph, frame_sizes=SCHEDULE[0][0], max_frame_size=MAXF, idle_streams=idle or None,
                   frame_format=fmt)
  r.warm()
  return r


def _play(r, src, idle, public):
  """-> per step (records, tracks, counts, fetch_results()) of the schedule's 4:2:0 frames of format src, fed as they
  are or, to a BGR runner, as cv2.cvtColor converts them."""
  out = []
  for k, (sizes, starts, gone) in enumerate(SCHEDULE):
    xs, pub = [], []
    for b, s in enumerate(sizes):
      if idle and b in gone:
        xs.append(None)
        pub.append(None)
        continue
      y = _yuv(src, s, 100 * k + b)
      xs.append(y if r.frame_format == src else cv2.cvtColor(y, CODES[src]))
      pub.append(_pub(100 * k + b, s))
    kw = dict(starts=starts or None, public_dets=pub if public else None)
    if 1 in starts:
      kw['calibs'] = {1: np.float32([[900, 0, 60, 0], [0, 900, 50, 0], [0, 0, 1, 0]])}
    if idle:
      kw['idle'] = gone
    r.step_frames(xs, **kw)
    out.append((r.fetch(), *r.fetch_tracks(), r.fetch_results()))
  return out


def _same(got, want):
  seen = 0
  for k, (a, w) in enumerate(zip(got, want)):
    for i in range(3):
      assert np.array_equal(np.ascontiguousarray(a[i]).view(np.uint32), np.ascontiguousarray(w[i]).view(np.uint32)), \
          (k, i)
    seen += int(a[2][:, 0].sum())
    for b, (x, y) in enumerate(zip(a[3], w[3])):
      assert (x is None) == (y is None), (k, b)
      for p, q in zip(x or [], y or []):
        for key in q:
          assert np.array_equal(np.asarray(p[key]), np.asarray(q[key])), (k, b, key)
  assert seen > 0


CASES = [('bf16', True, False, False, 'nv12'), ('bf16', False, True, True, 'i420'),
         ('bf16x3', True, True, False, 'i420'), ('bf16x3', False, False, True, 'nv12'),
         ('fp32', True, False, True, 'nv12'), ('fp32', False, True, False, 'i420')]


@pytest.mark.parametrize('precision,graph,flip,idle,fmt', CASES,
                         ids=['%s-%s-%s-%s-%s' % (p, 'graph' if g else 'eager', 'flip' if f else 'noflip',
                                                  'idle' if i else 'busy', fm) for p, g, f, i, fm in CASES])
def test_yuv_runner_equals_bgr_runner_on_converted_frames(precision, graph, flip, idle, fmt):
  opt, model = _model('coco_tracking', ['--flip_test'] if flip else [])
  results = {}
  for f in ('bgr', fmt):
    r = _make(model, opt, precision, graph, f, idle)
    results[f] = _play(r, fmt, idle, False)
    del r
  _same(results[fmt], results['bgr'])


def test_track_videos_mot_public_hungarian_yuv_equals_bgr():
  """Videos seeded with pre_dets (--public_det births no track from this model's scores), their tracks coasting and
  matched by --hungarian."""
  from centertrack_b200.runner import StreamRunner
  from centertrack_b200.videos import Video, track_videos
  opt, model = _model('mot', ['--public_det', '--hungarian'])
  spec = [(S0, 3), (S2, 2), (S1, 4), (S0, 2), (S2, 3)]

  def videos(fmt):
    out = []
    for v, (s, n) in enumerate(spec):
      ys = [_yuv('nv12', s, 50 * v + i) for i in range(n)]
      frames = ys if fmt == 'nv12' else [cv2.cvtColor(y, cv2.COLOR_YUV2BGR_NV12) for y in ys]
      seeds = [{'score': 0.9, 'class': 1, 'bbox': [10. + v, 12., 60., 70. + v]},
               {'score': 0.8, 'class': 1, 'bbox': [70., 30., 110., 90.]}]
      out.append(Video(v, frames, pre_dets=seeds, public_dets=[_pub(50 * v + i, s) for i in range(n)]))
    return out

  got = {}
  for fmt in ('bgr', 'nv12'):
    r = StreamRunner(model, 2, H, W, K=K, precision='bf16', device='cuda', opt=opt, device_tracking=True,
                     frame_sizes=[S0, S0], max_frame_size=MAXF, frame_format=fmt)
    r.warm()
    got[fmt] = {(v, i): res for v, i, res in track_videos(r, videos(fmt))}
    del r
  assert sorted(got['nv12']) == sorted(got['bgr']) == sorted((v, i) for v, (_, n) in enumerate(spec) for i in range(n))
  n = 0
  for key, want in got['bgr'].items():
    a = got['nv12'][key]
    assert len(a) == len(want), key
    n += len(a)
    for x, y in zip(a, want):
      for k in y:
        assert np.array_equal(np.asarray(x[k]), np.asarray(y[k])), (key, k)
  assert n > 0
