"""-m gpu: the device pre_process and prior heat-map against the CPU oracle with no tolerance.

Every entry point of the one warp (`warp_bilinear_u8`) -- ct_warp_affine_normalize, ct_warp_frames_normalize,
ct_pack_stem_frames_dev and ct_pack_stem_frames_flip_dev -- on every resolution policy over camera frame sizes
and on adversarial inverse maps, against ct_oracle.warp_affine_u8 (itself equal to cv2.warpAffine byte for byte:
tests/test_warp_oracle.py): fp32 compared as int32 bits, bf16 as int16 bits.  Both splats, ct_render_pre_hm and
ct_render_tracks, against draw_umich_gaussian into an fp32 map; the render boxes ct_track_start and ct_track_step write
against _get_additional_inputs's box arithmetic."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import ct_oracle as co
from centertrack_b200 import _lib as L
from helpers import WARP_GEOMETRIES, make_opt, warp_geometry, warp_maps

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')
MEAN = np.float32([0.408, 0.447, 0.470])
STD = np.float32([0.289, 0.274, 0.278])
MS = (C.c_void_p(MEAN.ctypes.data), C.c_void_p(STD.ctypes.data))
MAPS = warp_maps()


def _image(h, w, seed):
  return np.random.RandomState(seed).randint(0, 256, size=(h, w, 3)).astype(np.uint8)


def _want_chw(img, minv, oh, ow):
  return co.normalize_chw(co.warp_affine_u8(img, minv, oh, ow), MEAN, STD)


def _check_bits(got, want, ctx):
  """got: device or host fp32 / bf16 tensor, want: numpy fp32 (compared as int32) or int16 bf16 bits."""
  g = got.cpu()
  g = g.view(torch.int16).numpy() if g.dtype == torch.bfloat16 else g.numpy().view(np.int32)
  w = want.view(np.int32) if want.dtype == np.float32 else want
  assert g.shape == w.shape, (ctx, g.shape, w.shape)
  bad = g != w
  if bad.any():
    where = np.argwhere(bad)
    raise AssertionError('%s: %d values differ, first at %s' % (ctx, int(bad.sum()), where[:4].tolist()))


def _pitched(img, pitch, fill=0xA5):
  """img uint8 [h, w, 3] -> bytes with a row pitch of `pitch` bytes; the padding is never read."""
  h, w = img.shape[:2]
  buf = np.full((h, pitch), fill, np.uint8)
  buf[:, :3 * w] = img.reshape(h, 3 * w)
  return buf


# ------------------------------------------------------------------------------------ ct_warp_affine_normalize
CASES = [('geometry', i, g[0]) for i, g in enumerate(WARP_GEOMETRIES)] + [('map', i, m[0]) for i, m in enumerate(MAPS)]


def _case(kind, i):
  """-> (source (h, w), output (oh, ow), minv)"""
  if kind == 'geometry':
    hw, ohw, minv, _ = warp_geometry(i)
    return hw, ohw, minv
  _, minv, hw, ohw = MAPS[i]
  return hw, ohw, minv


@pytest.mark.parametrize('kind,i', [c[:2] for c in CASES], ids=[c[2] for c in CASES])
def test_warp_affine_normalize_equals_the_oracle(kind, i):
  """B = 1 per case, the frame once contiguous and once with an odd padded row pitch."""
  (h, w), (oh, ow), minv = _case(kind, i)
  img = _image(h, w, 31 + i)
  want = _want_chw(img, minv, oh, ow)
  m = torch.from_numpy(minv.reshape(1, 6)).to(DEV)
  for pitch in (3 * w, 3 * w + 7):
    src = torch.from_numpy(_pitched(img, pitch)).to(DEV)
    out = torch.full((1, 3, oh, ow), 7.0, device=DEV)
    L.check(L.lib().ct_warp_affine_normalize(L.ptr(src), 1, h, w, pitch, L.ptr(m), *MS, L.ptr(out), oh, ow,
                                             L.stream_ptr()))
    _check_bits(out[0], want, (CASES[i if kind == 'geometry' else len(WARP_GEOMETRIES) + i][2], pitch))


def test_warp_affine_normalize_batch_with_a_map_per_image():
  """B = 12 frames of one size in one call, each with its own inverse map (the tie, rotation, shear, mirror,
  translation and outside maps), padded pitch."""
  sel = [m for m in MAPS if m[2] == (400, 500) and m[3] == (320, 200)]
  assert len(sel) == 12
  h, w, pitch, oh, ow = 400, 500, 1503, 320, 200
  imgs = [_image(h, w, 70 + k) for k in range(len(sel))]
  src = torch.from_numpy(np.stack([_pitched(im, pitch) for im in imgs])).to(DEV)
  minv = torch.from_numpy(np.stack([m[1] for m in sel])).to(DEV)
  out = torch.full((len(sel), 3, oh, ow), 7.0, device=DEV)
  L.check(L.lib().ct_warp_affine_normalize(L.ptr(src), len(sel), h, w, pitch, L.ptr(minv), *MS, L.ptr(out), oh, ow,
                                           L.stream_ptr()))
  for k, (name, m, _, _) in enumerate(sel):
    _check_bits(out[k], _want_chw(imgs[k], m, oh, ow), name)


# ------------------------------------------------------------------- ragged frames: the pack and frames entry points
def _ragged(streams, seed):
  """streams: [(image (h, w), row pitch, minv)] -> (cur, prev device buffers, device ct_frame array, buffer bytes,
  [cur image], [prev image])."""
  frames = (L.Frame * len(streams))()
  bufs, cur, prev = [bytearray(), bytearray()], [], []
  for b, ((h, w), pitch, minv) in enumerate(streams):
    off = len(bufs[0])
    for k, (buf, imgs) in enumerate(zip(bufs, (cur, prev))):
      imgs.append(_image(h, w, seed + 2 * b + k))
      buf += _pitched(imgs[-1], pitch).tobytes() + bytes((-(h * pitch)) % 16)
    f = frames[b]
    f.offset, f.h, f.w, f.step = off, h, w, pitch
    f.minv[:] = [float(v) for v in minv]
  dev = [torch.frombuffer(bytearray(bb), dtype=torch.uint8).to(DEV) for bb in bufs]
  fdev = torch.frombuffer(bytearray(bytes(frames)), dtype=torch.uint8).to(DEV)
  return dev[0], dev[1], fdev, len(bufs[0]), cur, prev


def _mot_streams(opt):
  from centertrack_b200.detector import frame_geometry
  sizes = [((1080, 1920), 5760), ((375, 1242), 3729), ((900, 1600), 4800), ((480, 640), 1936), ((301, 457), 1375),
           ((1920, 1080), 3240), ((1, 37), 111), ((29, 1), 5)]
  return [(hw, pitch, frame_geometry(opt, *hw)[1]) for hw, pitch in sizes]


GROUPS = ['mot_544x960', 'kitti_384x1280', 'maps_320x200']


def _group(name):
  if name == 'maps_320x200':
    sel = [m for m in MAPS if m[2] == (400, 500) and m[3] == (320, 200)]
    return [(hw, 1500 + 3 * k, m) for k, (_, m, hw, _) in enumerate(sel)], (320, 200)
  H, W = (544, 960) if name.startswith('mot') else (384, 1280)
  return _mot_streams(make_opt('mot', ['--input_h', str(H), '--input_w', str(W)])), (H, W)


@pytest.mark.parametrize('group', GROUPS)
def test_device_descriptor_entry_points_equal_the_oracle(group):
  """Ragged buffers mixing camera sizes (odd and padded pitches, 1 x N and N x 1 frames) or the adversarial maps given
  through ct_frame.minv, one descriptor per stream: ct_warp_frames_normalize, ct_pack_stem_frames_dev (with and
  without the previous frame and pre_hm) and ct_pack_stem_frames_flip_dev (both halves)."""
  streams, (H, W) = _group(group)
  B = len(streams)
  cur, prev, fdev, nbytes, cur_imgs, prev_imgs = _ragged(streams, 500)
  want_cur = [_want_chw(im, s[2], H, W) for im, s in zip(cur_imgs, streams)]
  want_prev = [_want_chw(im, s[2], H, W) for im, s in zip(prev_imgs, streams)]
  hm = torch.rand((B, 1, H, W), device=DEV)
  hm_np = hm.cpu().numpy()
  lib, st = L.lib(), L.stream_ptr()

  img = torch.full((B, 3, H, W), 7.0, device=DEV)
  L.check(lib.ct_warp_frames_normalize(L.ptr(cur), L.ptr(fdev), B, nbytes, *MS, L.ptr(img), H, W, st))
  for b in range(B):
    _check_bits(img[b], want_cur[b], (group, 'warp_frames', b))

  def packed(fn, flip, pv, h):
    out = torch.full(((2 if flip else 1) * B, H, W, 8), -7.0, dtype=torch.bfloat16, device=DEV)
    L.check(fn(L.ptr(cur), L.ptr(pv), L.ptr(fdev), B, nbytes, *MS, L.ptr(h), L.ptr(out), H, W, st))
    return out

  for fname, flip in (('ct_pack_stem_frames_dev', False), ('ct_pack_stem_frames_flip_dev', True)):
    out = packed(getattr(lib, fname), flip, prev, hm)
    for b in range(B):
      want = co.stem_pixels(want_cur[b], want_prev[b], hm_np[b, 0], flip=flip)
      _check_bits(out[b], want[0] if flip else want, (group, fname, b))
      if flip:
        _check_bits(out[B + b], want[1], (group, fname, 'mirror', b))
  out = packed(lib.ct_pack_stem_frames_dev, False, None, None)
  for b in range(B):
    _check_bits(out[b], co.stem_pixels(want_cur[b], None, None), (group, 'no prev, no pre_hm', b))


@pytest.mark.parametrize('B', [49, 97])
def test_dev_packs_of_many_ragged_streams(B):
  """Many streams of small ragged frames in one launch of each _dev pack: every stream, 32 x 48 output."""
  from centertrack_b200.detector import frame_geometry
  opt = make_opt('coco_tracking', ['--input_h', '32', '--input_w', '48'])
  sizes = [(5, 7), (17, 23), (31, 40), (1, 1), (1, 9), (12, 1), (40, 64), (33, 47), (20, 30), (48, 32), (9, 61)]
  streams = [(hw, 3 * hw[1] + (b % 3) * 5, frame_geometry(opt, *hw)[1])
             for b, hw in ((b, sizes[b % len(sizes)]) for b in range(B))]
  cur, prev, fdev, nbytes, cur_imgs, prev_imgs = _ragged(streams, 900 + B)
  H, W = 32, 48
  hm = torch.rand((B, 1, H, W), device=DEV)
  hm_np = hm.cpu().numpy()
  lib, st = L.lib(), L.stream_ptr()
  for fname, flip in (('ct_pack_stem_frames_dev', False), ('ct_pack_stem_frames_flip_dev', True)):
    out = torch.full(((2 if flip else 1) * B, H, W, 8), -7.0, dtype=torch.bfloat16, device=DEV)
    L.check(getattr(lib, fname)(L.ptr(cur), L.ptr(prev), L.ptr(fdev), B, nbytes, *MS, L.ptr(hm), L.ptr(out), H, W,
                                st))
    for b, (_, _, minv) in enumerate(streams):
      want = co.stem_pixels(_want_chw(cur_imgs[b], minv, H, W), _want_chw(prev_imgs[b], minv, H, W), hm_np[b, 0],
                            flip=flip)
      _check_bits(out[b], want[0] if flip else want, (fname, b))
      if flip:
        _check_bits(out[B + b], want[1], (fname, 'mirror', b))


# ---------------------------------------------------------------------------------------------------- the splats
def _splat_bounds(boxes, B, H, W, skip_negative):
  """draw_umich_gaussian of the valid rows into fp32 maps, as the pair (lo, hi): equal except at the named pixels,
  where the winning gaussian's fp64 value lies within 1e-15 (relative) of an fp32 rounding midpoint, so that a last-bit
  difference between two fp64 exp implementations may round it either way; there lo and hi are the two roundings."""
  lo = np.zeros((B, H, W), np.float32)
  hi = np.zeros((B, H, W), np.float32)
  ref = np.zeros((B, H, W), np.float32)
  for b, cx, cy, r, _ in boxes:
    b, cx, cy = int(b), int(cx), int(cy)
    if (skip_negative and r < 0) or not 0 <= b < B:
      continue
    r = int(r)
    co.draw_umich_gaussian(ref[b], (cx, cy), r)
    d = 2 * r + 1
    sigma = d / 6
    y, x = np.ogrid[-r:r + 1, -r:r + 1]
    g = np.exp(-(x * x + y * y) / (2 * sigma * sigma))
    g[g < np.finfo(g.dtype).eps * g.max()] = 0
    g32 = g.astype(np.float32)
    nb = np.nextafter(g32, np.where(g > g32, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
    mid = (g32.astype(np.float64) + nb.astype(np.float64)) / 2
    near = (g != g32) & (np.abs(g - mid) <= 1e-15 * np.abs(mid))
    glo, ghi = np.where(near, np.minimum(g32, nb), g32), np.where(near, np.maximum(g32, nb), g32)
    left, right, top, bottom = min(cx, r), min(W - cx, r + 1), min(cy, r), min(H - cy, r + 1)
    if left + right <= 0 or top + bottom <= 0:
      continue
    sl = (b, slice(cy - top, cy + bottom), slice(cx - left, cx + right))
    gs = (slice(r - top, r + bottom), slice(r - left, r + right))
    lo[sl] = np.maximum(lo[sl], glo[gs])
    hi[sl] = np.maximum(hi[sl], ghi[gs])
  assert np.all(lo <= ref) and np.all(ref <= hi)
  return ref, lo, hi


def _splat_rows(B, H, W, rng):
  rows = []
  edges = [(0, 0), (W - 1, 0), (0, H - 1), (W - 1, H - 1), (W // 2, 0), (W // 2, H - 1), (0, H // 2), (W - 1, H // 2)]
  for b, r in ((1, 0), (2, 1), (3, 7), (4, max(H, W) + 50)):     # radius 0, 1, small, larger than the map
    rows += [(b, x, y, r, 0) for x, y in edges]
  rows.append((4, W // 3, H // 3, max(H, W) + 50, 0))
  cx, cy = rng.randint(W // 4, 3 * W // 4, 600), rng.randint(H // 4, 3 * H // 4, 600)
  rows += [(0, x, y, int(r), 0) for x, y, r in zip(cx, cy, rng.randint(0, 41, 600))]        # 600 overlapping blobs
  for b in range(5, B):
    if b % 3 == 0:
      continue                                                    # images without boxes stay zero
    for _ in range(int(rng.randint(1, 6))):
      rows.append((b, int(rng.randint(0, W)), int(rng.randint(0, H)), int(rng.randint(0, 60)), 0))
  rows += [(6, W // 2, H // 2, -1, 0), (9, 10, 10, -3, 0), (-1, 5, 5, 4, 0), (B, 5, 5, 4, 0), (B + 900, 5, 5, 4, 0)]
  perm = rng.permutation(len(rows))
  return [rows[k] for k in perm]


@pytest.mark.parametrize('hw', [(544, 960), (384, 1280)], ids=['544x960', '384x1280'])
@pytest.mark.parametrize('fn', ['ct_render_pre_hm', 'ct_render_tracks'])
def test_splats_equal_draw_umich_gaussian(fn, hw):
  """B = 64 maps: radius 0, 1 and larger than the map at every corner and edge, 600 overlapping blobs on one image,
  images without boxes, rows with radius < 0 or b outside [0, B) (which write nothing).  Equal to draw_umich_gaussian
  into an fp32 map except at named fp64 exp midpoints."""
  H, W = hw
  B = 64
  rows = _splat_rows(B, H, W, np.random.RandomState(H))
  if fn == 'ct_render_tracks':
    rows.append((11, 20, 20, -0.5, 0))            # its rows are skipped on radius < 0, fractional ones included
  boxes = torch.tensor(rows, dtype=torch.float32, device=DEV)
  out = torch.full((B, 1, H, W), 7.0, device=DEV)
  L.check(getattr(L.lib(), fn)(L.ptr(boxes), len(rows), L.ptr(out), B, H, W, L.stream_ptr()))
  got = out.cpu().numpy()[:, 0]
  ref, lo, hi = _splat_bounds(rows, B, H, W, skip_negative=True)
  named = np.argwhere(lo != hi)
  assert len(named) < 64, len(named)
  outside = ~((lo <= got) & (got <= hi))
  assert not outside.any(), (fn, int(outside.sum()), np.argwhere(outside)[:4].tolist())
  exact = lo == hi
  assert np.array_equal(got[exact].view(np.int32), ref[exact].view(np.int32))
  empty = [b for b in range(B) if not any(int(r[0]) == b and r[3] >= 0 for r in rows)]
  assert len(empty) > 15 and not got[empty].any()
  assert got[0].max() == 1.0 and (got[0] > 0).sum() > 0.1 * H * W


# ------------------------------------------------------------------------------------------------ the render boxes
def _host_boxes(rows, t_in, inp_w, inp_h, pre_thresh, b):
  """_get_additional_inputs's boxes (detector.py:254-290) from track rows, in numpy: each corner through trans_input
  left to right in fp64 (t0 x + t1 y, then + t2, as the reference's np.dot of three terms; not np.dot here, whose BLAS
  may fuse), to fp32, clipped to [0, inp - 1]; gaussian_radius of the ceiled fp32 extent; centre (x0 + x1) / 2 in fp32
  truncated.  -> [T, 5] rows (b, cx, cy, radius or -1, 0)."""
  out = np.zeros((len(rows), 5), np.float32)
  out[:, 0], out[:, 3] = b, -1
  t = np.asarray(t_in, np.float64).reshape(6)
  for k, r in enumerate(rows):
    if r[L.CT_TRK_ACTIVE] == 0 or r[L.CT_TRK_SCORE] < np.float32(pre_thresh):
      continue
    x0, y0, x1, y1 = (np.float64(v) for v in r[L.CT_TRK_BBOX:L.CT_TRK_BBOX + 4])
    px = [np.float32(t[0] * x + t[1] * y + t[2]) for x, y in ((x0, y0), (x1, y1))]
    py = [np.float32(t[3] * x + t[4] * y + t[5]) for x, y in ((x0, y0), (x1, y1))]
    bx0, bx1 = (np.clip(v, np.float32(0), np.float32(inp_w - 1)) for v in px)
    by0, by1 = (np.clip(v, np.float32(0), np.float32(inp_h - 1)) for v in py)
    h, w = np.float32(by1 - by0), np.float32(bx1 - bx0)
    if not (h > 0 and w > 0):
      continue
    out[k, 3] = max(0, int(co.gaussian_radius((math.ceil(h), math.ceil(w)))))
    out[k, 1] = np.float32(np.float32(bx0 + bx1) / np.float32(2)).astype(np.int32)
    out[k, 2] = np.float32(np.float32(by0 + by1) / np.float32(2)).astype(np.int32)
  return out


def _near(t, fixed, target, axis):
  """fp32 source coordinates c (with the other coordinate `fixed`) whose input coordinate, t's row `axis` in fp64 then
  fp32, is exactly `target` or one ulp either side of it -> {offset in ulps of target: c}."""
  r0, r1, r2 = (float(v) for v in t[3 * axis:3 * axis + 3])
  ideal = (target - r2 - (r1 if axis == 0 else r0) * fixed) / (r0 if axis == 0 else r1)
  cands = [np.float32(ideal)]
  for direction in (np.float32(np.inf), np.float32(-np.inf)):
    v = cands[0]
    for _ in range(64):
      v = np.nextafter(v, direction)
      cands.append(v)
  found = {}
  for v in cands:
    x, y = (np.float64(v), np.float64(fixed)) if axis == 0 else (np.float64(fixed), np.float64(v))
    m = np.float32(r0 * x + r1 * y + r2)
    for k in (-1, 0, 1):
      want = np.float32(target) if k == 0 else np.nextafter(np.float32(target), np.float32(k * np.inf))
      if m == want:
        found.setdefault(k, v)
  return found


def test_render_boxes_equal_the_host_box_arithmetic():
  """ct_track_start's boxes from DeviceTracker.start seeds on two camera geometries (KITTI 1242 x 375 and 1080p into a
  384 x 1280 input): corners that land on an input integer and one ulp either side of it, clipping at 0 and at
  inp - 1, zero-width boxes, score == pre_thresh and one ulp below it; then a ct_track_step without detections under
  --max_age, which keeps the tracks inactive: every row's radius is -1."""
  from centertrack_b200.device_tracker import DeviceTracker, seed_rows
  inp_h, inp_w = 384, 1280
  opt = make_opt('coco_tracking', ['--input_h', str(inp_h), '--input_w', str(inp_w), '--pre_thresh', '0.25',
                                   '--new_thresh', '0.2', '--track_thresh', '0.2', '--max_age', '3'])
  assert (opt.pre_thresh, opt.new_thresh) == (0.25, 0.2)      # opts raises both to at least track_thresh
  img_hw = [(375, 1242), (1080, 1920)]
  centers = [np.array([w / 2., h / 2.], np.float32) for h, w in img_hw]
  scales = [max(h, w) * 1.0 for h, w in img_hw]
  K, F = 16, 11
  trk = DeviceTracker(opt, 2, K, F, {'tracking': (9, 2)}, inp_h, inp_w, DEV, centers=centers, scales=scales,
                      max_tracks=64)
  t_in = trk.trans_input.cpu().numpy()
  rng = np.random.RandomState(3)
  items = {}
  for b, (h, w) in enumerate(img_hw):
    t = t_in[b]
    its = []
    add = lambda bbox, score=0.9: its.append({'score': float(score), 'class': 1, 'bbox': [float(v) for v in bbox]})
    def corner(X, Y, kx, ky):
      # KITTI's map magnifies (1.03): every target is reachable.  1080p's shrinks (2/3), so one source ulp moves the
      # input coordinate by more than one ulp; there the exact integer stands in for a target it cannot reach.
      fx = _near(t, 0.0, X, 0)             # t[1] == 0: the input x does not depend on the source y
      fy = _near(t, float(fx.get(kx, fx[0])), Y, 1)
      assert t[1] == 0 and (b == 1 or set(fx) == set(fy) == {-1, 0, 1}), (b, X, Y, fx, fy)
      return fx.get(kx, fx[0]), fy.get(ky, fy[0])
    for kx in (-1, 0, 1):
      for ky in (-1, 0, 1):
        # odd x0 + x1 and y0 + y1 about an integer: the truncated centre; then the ceiled extent
        add(list(corner(101.0, 50.0, kx, ky)) + list(corner(358.0, 81.0, -kx, ky)))
        add(list(corner(102.0, 50.0, kx, -ky)) + list(corner(357.0, 120.0, kx, ky)))
    add([-50.0, -20.0, 60.0, 40.0])                                          # clipped at 0
    add([w - 40.0, h - 30.0, w + 80.0, h + 90.0])                            # clipped at inp - 1
    add([w + 10.0, 5.0, w + 90.0, 40.0])                                     # wholly right: zero width after clip
    add([30.0, 30.0, 30.0, 90.0])                                            # zero width
    add([30.0, 60.0, 90.0, 60.0])                                            # zero height
    add([200.0, 100.0, 260.0, 170.0], score=0.25)                            # score == pre_thresh: splatted
    add([200.0, 100.0, 260.0, 170.0], score=np.nextafter(np.float32(0.25), np.float32(0)))   # just below: not
    for _ in range(12):
      x0, y0 = rng.uniform(-30, w), rng.uniform(-30, h)
      add([x0, y0, x0 + rng.uniform(0, 300), y0 + rng.uniform(0, 200)], score=rng.uniform(0.21, 1.0))
    items[b] = its
  trk.start([0, 1], items)
  boxes = trk.boxes.cpu().numpy()
  for b in range(2):
    rows = np.zeros((trk.T, L.CT_TRK_FLOATS), np.float32)
    seeds = seed_rows(items[b], opt.new_thresh)
    rows[:len(seeds)] = seeds
    want = _host_boxes(rows, t_in[b], inp_w, inp_h, opt.pre_thresh, b)
    bad = np.nonzero((boxes[b].view(np.int32) != want.view(np.int32)).any(1))[0]
    assert len(bad) == 0, (b, bad[:4].tolist(), boxes[b][bad[:4]].tolist(), want[bad[:4]].tolist())
    assert (want[:, 3] >= 0).sum() > 20 and (want[:len(seeds), 3] < 0).sum() >= 4
  records = torch.zeros((2, K, F), device=DEV)           # no detection scores above out_thresh: every track coasts
  trk.step(records)
  tracks, boxes = trk.tracks.cpu().numpy(), trk.boxes.cpu().numpy()
  counts = trk.counts.cpu().numpy()
  for b in range(2):
    n = counts[b, 0]
    assert n == len(seed_rows(items[b], opt.new_thresh)) and not tracks[b, :n, L.CT_TRK_ACTIVE].any()
    assert np.array_equal(boxes[b].view(np.int32), _host_boxes(tracks[b], t_in[b], inp_w, inp_h, opt.pre_thresh,
                                                               b).view(np.int32))
    assert (boxes[b, :, 3] == -1).all()
