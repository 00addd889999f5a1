"""-m gpu: crops of every active track (or kept detection) out of each stream's frame.  ct_crop_boxes against the
oracle (crop_oracle: the documented map + warp_affine_u8, cv2-exact) bit for bit with exact counts and untouched slots
past them, on mixed formats, track and detection tables, invalid descriptors and the mapped form; and
StreamRunner(crop_size=) against the oracle on the frames it was fed and the boxes fetch_results() gives, on every
engine and runner kind, with the same records and tables as a runner without crops."""
import ctypes as C

import numpy as np
import pytest
import torch

from centertrack_b200 import _lib as L
from crop_oracle import crop
from helpers import make_model
from test_gpu_frames import _frame
from test_gpu_yuv_frames import FMT, _source
from yuv_oracle import bgr_to_yuv420, yuv420_to_bgr

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')
SENTINEL = 0x5A


# ------------------------------------------------------------------------------------------------ kernel
def _slot(spec, seed):
  """spec [(fmt, (h, w), pitch)] -> (device buffer, host ct_frame array, bytes, [BGR image the oracle sees])."""
  frames = (L.Frame * len(spec))()
  buf, imgs = bytearray(), []
  for i, (fmt, (h, w), pitch) in enumerate(spec):
    off = len(buf)
    raw, bgr = _source(fmt, h, w, pitch, seed + i)
    buf += raw.tobytes() + bytes((-raw.size) % 16)
    imgs.append(bgr)
    f = frames[i]
    f.offset, f.h, f.w, f.step, f.format = off, h, w, pitch, FMT[fmt]
  return torch.frombuffer(bytearray(buf), dtype=torch.uint8).to(DEV), frames, len(buf), imgs


def _box(rng, h, w):
  kind = rng.randint(8)
  if kind == 0:                                            # the guard: non-finite or beyond 16384 px
    return np.float32([rng.choice([np.nan, np.inf, 2e4, -16385.]), 0, w, h])
  if kind == 1:                                            # inverted
    return np.float32([w * .9, h * .8, w * .1, h * .3])
  if kind == 2:                                            # sub-pixel
    x, y = rng.uniform(0, w), rng.uniform(0, h)
    return np.float32([x, y, x + .4, y + .3])
  x, y = rng.uniform(-.3 * w, 1.1 * w, 2), rng.uniform(-.3 * h, 1.1 * h, 2)
  return np.float32([min(x), min(y), max(x) + 1, max(y) + 1])


def _table(rng, imgs_of, n_streams, K, track):
  """A random table: track rows [n_streams, T, 13] with an active prefix of 0..K rows, coasting rows, then rows active
  again past the first coasting one; or detection rows [n_streams, K, 10] with counts beyond K and below 0."""
  RF, T = (L.CT_TRK_FLOATS, 2 * K + 3) if track else (L.CT_DET_FLOATS, K)
  rows = rng.uniform(-5, 5, (n_streams, T, RF)).astype(np.float32)
  counts = np.zeros((n_streams, 2) if track else (n_streams,), np.int32)
  for b in range(n_streams):
    h, w = imgs_of(b).shape[:2] if imgs_of(b) is not None else (16, 16)
    for r in range(T):
      rows[b, r, L.CT_TRK_BBOX:L.CT_TRK_BBOX + 4] = _box(rng, h, w)
    if track:
      a, c = rng.randint(0, K + 1), rng.randint(0, 3)
      rows[b, :, L.CT_TRK_ACTIVE] = rng.randint(1, 9, T)
      rows[b, a:a + c, L.CT_TRK_ACTIVE] = 0
      counts[b] = (min(a + c + rng.randint(0, 4), T), 77)
    else:
      counts[b] = rng.randint(-2, K + 3)
  return rows, counts


def _want_count(rows, counts, b, K, track):
  n = max(0, min(int(counts[b, 0] if track else counts[b]), K, rows.shape[1]))
  if track:
    inactive = np.nonzero(rows[b, :n, L.CT_TRK_ACTIVE] == 0)[0]
    n = int(inactive[0]) if len(inactive) else n
  return n


def _run(spec, n_streams, K, oh, ow, track, seed, streams=None, bad=()):
  """One ct_crop_boxes launch; image i has frame spec[i] (streams[i]'s, or stream i's without a map); `bad` images get
  invalid descriptors.  Checks every stream's count, crops and untouched slots."""
  rng = np.random.RandomState(seed)
  buf, frames, nbytes, imgs = _slot(spec, seed)
  for i, how in bad:
    if how == 'format':
      frames[i].format = 7
    elif how == 'offset':
      frames[i].offset = nbytes
    else:
      frames[i].step = 1
  n = len(spec)
  img_of_stream = {}
  for i in range(n):
    s = i if streams is None else streams[i]
    if 0 <= s < n_streams:
      img_of_stream[s] = i
  rows, counts = _table(rng, lambda b: imgs[img_of_stream[b]] if b in img_of_stream else None, n_streams, K, track)
  d = L.CropDesc()
  d_rows, d_counts = torch.from_numpy(rows).to(DEV), torch.from_numpy(counts).to(DEV)
  d_frames = torch.frombuffer(bytearray(bytes(frames)), dtype=torch.uint8).to(DEV)
  out = torch.full((n_streams, K, oh, ow, 3), SENTINEL, dtype=torch.uint8, device=DEV)
  out_counts = torch.full((n_streams,), -7, dtype=torch.int32, device=DEV)
  d.buf, d.buf_bytes, d.frames = buf.data_ptr(), nbytes, d_frames.data_ptr()
  d.rows, d.row_floats, d.rows_per_stream = d_rows.data_ptr(), rows.shape[2], rows.shape[1]
  d.counts, d.counts_stride, d.active_col = d_counts.data_ptr(), 2 if track else 1, L.CT_TRK_ACTIVE if track else -1
  d.K, d.out_h, d.out_w, d.out, d.out_counts = K, oh, ow, out.data_ptr(), out_counts.data_ptr()
  d_map = torch.tensor(streams, dtype=torch.int32, device=DEV) if streams is not None else None
  L.check(L.lib().ct_crop_boxes(C.byref(d), L.ptr(d_map), n, n_streams, L.stream_ptr()), 'ct_crop_boxes')
  got, got_n = out.cpu().numpy(), out_counts.cpu().numpy()
  bad_imgs = {i for i, _ in bad}
  total = 0
  for b in range(n_streams):
    if b not in img_of_stream:                           # no image: untouched
      assert got_n[b] == -7 and (got[b] == SENTINEL).all(), b
      continue
    i = img_of_stream[b]
    want_n = 0 if i in bad_imgs else _want_count(rows, counts, b, K, track)
    assert got_n[b] == want_n, (b, got_n[b], want_n)
    for k in range(want_n):
      want = crop(imgs[i], rows[b, k, L.CT_TRK_BBOX:L.CT_TRK_BBOX + 4], oh, ow)
      bad_px = got[b, k] != want
      assert not bad_px.any(), (b, k, spec[i], rows[b, k, L.CT_TRK_BBOX:L.CT_TRK_BBOX + 4].tolist(),
                                np.argwhere(bad_px)[:3].tolist())
    assert (got[b, want_n:] == SENTINEL).all(), b
    total += want_n
  assert total > 0
  return total


MIXED = [('nv12', (60, 80), 96), ('bgr', (48, 64), 200), ('i420', (34, 126), 126), ('bgr', (1, 1), 16),
         ('bgr', (1, 37), 111), ('nv12', (2, 2), 2), ('i420', (90, 120), 136), ('bgr', (29, 3), 13)]


@pytest.mark.parametrize('oh,ow', [(37, 23), (16, 32), (1, 1), (256, 128)])
@pytest.mark.parametrize('track', [True, False], ids=['tracks', 'detections'])
def test_kernel_equals_the_oracle_on_mixed_frames(oh, ow, track):
  K = 4 if (oh, ow) == (256, 128) else 9
  _run(MIXED, len(MIXED), K, oh, ow, track, 11 + oh)


def test_invalid_descriptors_give_count_zero_and_write_nothing():
  _run(MIXED, len(MIXED), 6, 16, 32, True, 5, bad=[(0, 'format'), (2, 'offset'), (6, 'step')])
  _run(MIXED, len(MIXED), 6, 16, 32, False, 6, bad=[(1, 'format'), (4, 'step')])


@pytest.mark.parametrize('track', [True, False], ids=['tracks', 'detections'])
def test_mapped_form_with_idle_and_out_of_range_entries(track):
  n_streams = 11
  streams = [3, -1, 0, 99, 7, 10, 11, 5]                  # idle: 1, 2, 4, 6, 8, 9
  _run(MIXED, n_streams, 7, 37, 23, track, 21, streams=streams, bad=[(5, 'offset')])


@pytest.mark.parametrize('B', [49, 97])
def test_many_streams(B):
  fmts = ['nv12', 'i420', 'bgr']
  sizes = [(6, 8), (18, 24), (32, 40), (2, 2), (2, 10), (40, 64), (20, 30), (48, 32)]
  spec = []
  for b in range(B):
    fmt, hw = fmts[b % 3], sizes[b % len(sizes)]
    spec.append((fmt, hw, (3 if fmt == 'bgr' else 1) * hw[1] + (b % 4) * 2))
  _run(spec, B, 5, 16, 32, True, B)
  _run(spec, B + 3, 5, 8, 8, False, B + 1, streams=list(range(B + 2, 2, -1))[:B])


# ------------------------------------------------------------------------------------------------ runner
H, W, K, B = 128, 160, 40, 2
S0, S1, S2 = (120, 200), (97, 131), (160, 128)
MAXF = (160, 200)
CROP = (24, 16)


def _model(extra=()):
  opt, model, _ = make_model('coco_tracking', extra=['--track_thresh', '0.1', '--new_thresh', '0.1', '--pre_thresh',
                                                     '0.1', '--input_h', str(H), '--input_w', str(W), '--max_age', '2'] +
                             list(extra))
  with torch.no_grad():                 # boxes of some pixels (the synthetic weights give ~0 wh)
    model.state_dict()['wh.2.bias'].fill_(3.0)
  return opt, model.cuda()


def _check(r, fed, ctx):
  """fetch_crops() of the last step against the oracle of the BGR frames fed and fetch_results()' boxes; -> crops."""
  crops, counts = r.fetch_crops()
  res = r.fetch_results()
  assert crops.shape == (r.B, r.K) + r.crop_size + (3,) and crops.dtype == torch.uint8 and crops.is_cuda
  assert counts.dtype == np.int32 and counts.shape == (r.B,)
  got = crops.cpu().numpy()
  n = 0
  for b in range(r.B):
    if res[b] is None:
      assert counts[b] == 0, (ctx, b)
      continue
    act = [d.get('active', 1) != 0 for d in res[b]]
    assert counts[b] == sum(act) and all(act[:counts[b]]), (ctx, b, counts[b], act)
    for k in range(counts[b]):
      want = crop(fed[b], res[b][k]['bbox'], *r.crop_size)
      assert np.array_equal(got[b, k], want), (ctx, b, k, res[b][k]['bbox'])
    n += int(counts[b])
  return n


def _bgr(fmt, frame):
  if fmt == 'bgr':
    return frame
  h = frame.shape[0] // 3 * 2
  return yuv420_to_bgr(frame, h, frame.shape[1], fmt)


RUNNERS = {
    'bf16_graph_fixed': ('bf16', True, 'fixed', []),
    'bf16_eager_fixed': ('bf16', False, 'fixed', []),
    'bf16x3_graph_capacity': ('bf16x3', True, 'capacity', []),
    'fp32_eager_capacity': ('fp32', False, 'capacity', []),
    'fp32_graph_fixed': ('fp32', True, 'fixed', []),
    'bf16_graph_nv12_device': ('bf16', True, 'nv12_device', []),
    'bf16_graph_idle': ('bf16', True, 'idle', []),
    'fp32_graph_idle': ('fp32', True, 'idle', []),
    'bf16_graph_flip': ('bf16', True, 'fixed', ['--flip_test']),
    'bf16x3_eager_flip_capacity': ('bf16x3', False, 'capacity', ['--flip_test']),
}


@pytest.mark.parametrize('name', list(RUNNERS))
def test_runner_crops_equal_the_oracle(name):
  from centertrack_b200.runner import StreamRunner
  precision, graph, mode, extra = RUNNERS[name]
  opt, model = _model(extra)
  fmt = 'nv12' if mode == 'nv12_device' else 'bgr'
  sizes = [S0, S1 if fmt == 'bgr' else (96, 130)]       # 4:2:0 frames have even sizes
  kw = dict(K=K, precision=precision, opt=opt, device_tracking=True, use_graph=graph, frame_sizes=list(sizes),
            crop_size=CROP)
  if mode != 'fixed':
    kw.update(max_frame_size=MAXF, frame_format=fmt)
  if mode == 'idle':
    kw['idle_streams'] = True
  r = StreamRunner(model, B, H, W, **kw)
  r.warm()
  n = 0
  for t in range(6):
    step_kw = {}
    if mode != 'fixed' and t == 3:                         # a new video at another size and camera on stream 1
      sizes[1] = S2
      step_kw = dict(starts=[1], calibs={1: np.array([[300., 0, 60, 0], [0, 310, 75, 0], [0, 0, 1, 0]], np.float32)})
    if mode == 'idle' and t == 1:
      step_kw = dict(idle=[0])
    if mode == 'idle' and t == 2:
      step_kw = dict(starts=[0])
    frames = [_frame(h, w, 100 * t + b) for b, (h, w) in enumerate(sizes)]
    if fmt != 'bgr':
      frames = [bgr_to_yuv420(f, fmt) for f in frames]
    fed = [_bgr(fmt, f) for f in frames]
    if mode == 'nv12_device':
      frames = [torch.from_numpy(f).to(DEV) for f in frames]
    if 'idle' in step_kw:
      frames[0] = None
    r.step_frames(frames, **step_kw)
    n += _check(r, fed, (name, t))
  assert n > 0, name


def test_post_process_runner_crops_equal_the_oracle():
  """device_post_process on a ctdet model: crop k of stream b is detection k."""
  from centertrack_b200.runner import StreamRunner
  from test_gpu_post_process import H as PH, W as PW, _model as pp_model
  opt, model = pp_model('ctdet', ['--out_thresh', '0.05'])
  sizes = [(120, 200), (90, 140), (64, 96)]
  r = StreamRunner(model, 3, PH, PW, K=K, opt=opt, device_post_process=True, frame_sizes=sizes, crop_size=(37, 23))
  r.warm()
  n = 0
  for t in range(4):
    frames = [_frame(h, w, 50 * t + b) for b, (h, w) in enumerate(sizes)]
    r.step_frames(frames)
    n += _check(r, frames, ('ctdet', t))
  assert n > 0


def test_track_videos_crops_equal_the_oracle():
  from centertrack_b200.runner import StreamRunner
  from centertrack_b200.videos import Video, track_videos
  opt, model = _model()
  r = StreamRunner(model, B, H, W, K=K, opt=opt, device_tracking=True, frame_sizes=[S0, S1], max_frame_size=MAXF,
                   idle_streams=True, crop_size=CROP)
  r.warm()
  vids = {'a': [_frame(*S0, 300 + i) for i in range(4)], 'b': [_frame(*S2, 400 + i) for i in range(2)],
          'c': [_frame(*S1, 500 + i) for i in range(3)]}
  n, seen = 0, 0
  for vid, i, res, cut in track_videos(r, [Video(k, v) for k, v in vids.items()], crops=True):
    act = [d for d in res if d['active'] != 0]
    assert cut.shape == (len(act),) + CROP + (3,) and cut.is_cuda
    got = cut.cpu().numpy()
    for k, d in enumerate(act):
      assert np.array_equal(got[k], crop(vids[vid][i], d['bbox'], *CROP)), (vid, i, k)
    n += len(act)
    seen += 1
  assert seen == 9 and n > 0


@pytest.mark.parametrize('graph', [True, False], ids=['graph', 'eager'])
def test_crops_change_no_record_or_table(graph):
  """The same frames through runners with and without crop_size: records and track tables byte-identical every step,
  one more launch per step, B * 4 more bytes down."""
  from centertrack_b200.runner import StreamRunner
  opt, model = _model()
  kw = dict(K=K, opt=opt, device_tracking=True, use_graph=graph, frame_sizes=[S0, S1], max_frame_size=MAXF)
  plain, cut = StreamRunner(model, B, H, W, **kw), StreamRunner(model, B, H, W, crop_size=CROP, **kw)
  for r in (plain, cut):
    r.warm()
  assert cut.launches_per_step == plain.launches_per_step + 1
  assert cut.d2h_bytes_per_step == plain.d2h_bytes_per_step + B * 4
  lib = L.lib()
  for t in range(5):
    frames = [_frame(*S0, 700 + t), _frame(*S1, 800 + t)]
    launches = []
    for r in (plain, cut):
      n0 = lib.ct_launch_count()
      r.step_frames(frames)
      launches.append(lib.ct_launch_count() - n0)
    if not graph and t > 0:
      assert launches[1] == launches[0] + 1, launches
    a, b = plain.fetch(), cut.fetch()
    assert a.tobytes() == b.tobytes(), t
    for x, y in zip(plain.fetch_tracks(), cut.fetch_tracks()):
      assert x.tobytes() == y.tobytes(), t


def test_a_steps_crops_stay_until_its_slot_is_reused():
  from centertrack_b200.runner import StreamRunner
  opt, model = _model()
  r = StreamRunner(model, B, H, W, K=K, opt=opt, device_tracking=True, frame_sizes=[S0, S1], crop_size=CROP)
  r.warm()
  r.step_frames([_frame(*S0, 1), _frame(*S1, 2)])
  crops, counts = r.fetch_crops()
  keep = crops.clone()
  assert counts.sum() > 0
  for t in range(2):
    r.step_frames([_frame(*S0, 10 + t), _frame(*S1, 20 + t)])
    prev, _ = r.previous_crops()
  torch.cuda.synchronize()
  assert torch.equal(crops, keep)
  assert prev.data_ptr() != crops.data_ptr()
