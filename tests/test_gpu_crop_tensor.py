"""-m gpu: track crops as one packed, normalised NCHW batch.  ct_crop_boxes_tensor against ct_crop_boxes on the same
slot and tables, converted by the CPU oracle (torchvision's Normalize(ToTensor()).to(dtype)) and packed by the
documented rule, bit for bit, with NaN-filled rows past N untouched; and StreamRunner(crop_format=) against the uint8
crops of an otherwise identical runner the same way, on every engine and runner kind, with the records, tables and
counts of runners without it, a batch that outlives the next two steps and rows that do not depend on what the buffer
held."""
import ctypes as C

import numpy as np
import pytest
import torch

from centertrack_b200 import _lib as L
from crop_oracle import crop
from crop_tensor_oracle import IMAGENET, bits, normalize, pack
from test_gpu_crops import B, CROP, H, K, MAXF, MIXED, RUNNERS, S0, S1, S2, W, _bgr, _model, _slot, _table
from test_gpu_frames import _frame
from yuv_oracle import bgr_to_yuv420

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')
DEGENERATE = {'mean': (1e30, -0.5, 1.0), 'std': (1e-40, -3e-8, 7.0)}
# (dtype, channels, mean / std): every dtype and order, ImageNet's statistics and values that overflow or vanish
FORMATS = [(torch.float16, 'rgb', IMAGENET), (torch.bfloat16, 'bgr', IMAGENET), (torch.float32, 'rgb', DEGENERATE),
           (torch.float16, 'bgr', DEGENERATE), (torch.bfloat16, 'rgb', DEGENERATE), (torch.float32, 'bgr', IMAGENET)]
TYPES = {torch.float32: L.CT_CROP_F32, torch.float16: L.CT_CROP_F16, torch.bfloat16: L.CT_CROP_BF16}


def _fmt(i):
  dtype, channels, ms = FORMATS[i % len(FORMATS)]
  return dict(dtype=dtype, channels=channels, mean=ms['mean'], std=ms['std'])


# ------------------------------------------------------------------------------------------------ kernel
def _run(spec, n_streams, K_, oh, ow, track, seed, streams=None, bad=(), formats=range(len(FORMATS))):
  """ct_crop_boxes, then ct_crop_boxes_tensor in each of `formats` on the same slot and tables; the batch must equal
  the uint8 crops converted and packed by the oracle, the offsets and counts theirs, the rows past N their NaN fill."""
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
  rows, counts = _table(rng, lambda b: imgs[img_of_stream[b]] if b in img_of_stream else None, n_streams, K_, track)
  d = L.CropDesc()
  d_rows, d_counts = torch.from_numpy(rows).to(DEV), torch.from_numpy(counts).to(DEV)
  d_frames = torch.frombuffer(bytearray(bytes(frames)), dtype=torch.uint8).to(DEV)
  u8 = torch.zeros((n_streams, K_, oh, ow, 3), dtype=torch.uint8, device=DEV)
  u8_counts = torch.full((n_streams,), -7, dtype=torch.int32, device=DEV)
  d.buf, d.buf_bytes, d.frames = buf.data_ptr(), nbytes, d_frames.data_ptr()
  d.rows, d.row_floats, d.rows_per_stream = d_rows.data_ptr(), rows.shape[2], rows.shape[1]
  d.counts, d.counts_stride, d.active_col = d_counts.data_ptr(), 2 if track else 1, L.CT_TRK_ACTIVE if track else -1
  d.K, d.out_h, d.out_w, d.out, d.out_counts = K_, oh, ow, u8.data_ptr(), u8_counts.data_ptr()
  d_map = torch.tensor(streams, dtype=torch.int32, device=DEV) if streams is not None else None
  lib = L.lib()
  L.check(lib.ct_crop_boxes(C.byref(d), L.ptr(d_map), n, n_streams, L.stream_ptr()), 'ct_crop_boxes')
  want_counts = u8_counts.cpu().numpy()
  got_u8 = u8.cpu().numpy()
  N = 0
  for j in formats:
    f = _fmt(j)
    out = torch.full((n * K_, 3, oh, ow), float('nan'), dtype=f['dtype'], device=DEV)
    fill = bits(out[:1].cpu())[0]
    offsets = torch.full((n_streams + 1,), -9, dtype=torch.int32, device=DEV)
    t_counts = torch.full((n_streams,), -7, dtype=torch.int32, device=DEV)
    t = L.CropTensor()
    t.type, t.order = TYPES[f['dtype']], L.CT_CROP_RGB if f['channels'] == 'rgb' else L.CT_CROP_BGR
    t.mean[:], t.std[:] = f['mean'], f['std']
    t.rows_cap, t.out, t.out_offsets = out.shape[0], out.data_ptr(), offsets.data_ptr()
    d.out, d.out_counts = None, t_counts.data_ptr()
    lib.ct_reset_launch_count()
    L.check(lib.ct_crop_boxes_tensor(C.byref(d), C.byref(t), L.ptr(d_map), n, n_streams, L.stream_ptr()),
            'ct_crop_boxes_tensor')
    assert lib.ct_launch_count() == 2
    assert np.array_equal(t_counts.cpu().numpy(), want_counts), (j, t_counts.cpu().numpy(), want_counts)
    want, want_off = pack(got_u8, want_counts, set(img_of_stream), f['dtype'], f['channels'], f['mean'], f['std'])
    got_off = offsets.cpu().numpy()
    assert np.array_equal(got_off, want_off), (j, got_off, want_off)
    N = int(want_off[-1])
    got = bits(out.cpu())
    bad_px = got[:N] != bits(want)
    assert not bad_px.any(), (j, np.argwhere(bad_px.numpy())[:3].tolist())
    assert (got[N:] == fill).all(), j                      # rows past N are not written
  return N


@pytest.mark.parametrize('oh,ow', [(1, 1), (255, 127), (256, 128)])
@pytest.mark.parametrize('track', [True, False], ids=['tracks', 'detections'])
def test_kernel_equals_the_converted_uint8_crops_on_mixed_frames(oh, ow, track):
  assert _run(MIXED, len(MIXED), 4 if oh > 1 else 9, oh, ow, track, 31 + oh) > 0


def test_invalid_descriptors_give_no_rows():
  _run(MIXED, len(MIXED), 6, 16, 32, True, 5, bad=[(0, 'format'), (2, 'offset'), (6, 'step')])
  _run(MIXED, len(MIXED), 6, 17, 31, False, 6, bad=[(1, 'format'), (4, 'step')])


@pytest.mark.parametrize('track', [True, False], ids=['tracks', 'detections'])
def test_mapped_form_with_idle_and_out_of_range_entries(track):
  _run(MIXED, 11, 7, 37, 23, track, 21, streams=[3, -1, 0, 99, 7, 10, 11, 5], bad=[(5, 'offset')])


@pytest.mark.parametrize('B_', [49, 97])
def test_many_streams(B_):
  fmts = ['nv12', 'i420', 'bgr']
  sizes = [(6, 8), (18, 24), (32, 40), (2, 2), (2, 10), (40, 64), (20, 30), (48, 32)]
  spec = []
  for b in range(B_):
    fmt, hw = fmts[b % 3], sizes[b % len(sizes)]
    spec.append((fmt, hw, (3 if fmt == 'bgr' else 1) * hw[1] + (b % 4) * 2))
  _run(spec, B_, 5, 16, 32, True, B_, formats=[0, 2])
  _run(spec, B_ + 3, 5, 8, 8, False, B_ + 1, streams=list(range(B_ + 2, 2, -1))[:B_], formats=[1, 3])


# ------------------------------------------------------------------------------------------------ runner
def _same_outputs(a, b, ctx):
  """Records, tables and counts of two runners' last steps are byte-identical."""
  assert a.fetch().tobytes() == b.fetch().tobytes(), ctx
  if a.tracker is not None:
    for x, y in zip(a.fetch_tracks(), b.fetch_tracks()):
      assert x.tobytes() == y.tobytes(), ctx
  else:
    for x, y in zip(a.fetch_detections()[:2], b.fetch_detections()[:2]):
      assert x.tobytes() == y.tobytes(), ctx


def _check(u8r, tr, ctx):
  """fetch_crops() of the crop_format runner tr against the uint8 crops of u8r, converted and packed; -> N."""
  crops, counts = u8r.fetch_crops()
  batch, got_counts = tr.fetch_crops()
  f = tr.crop_format
  assert np.array_equal(got_counts, counts) and got_counts.dtype == np.int32, (ctx, got_counts, counts)
  assert batch.is_cuda and batch.dtype == f['dtype'] and batch.shape == (int(counts.sum()), 3) + tr.crop_size, ctx
  want, _ = pack(crops.cpu().numpy(), counts, set(range(tr.B)), f['dtype'], f['channels'], f['mean'], f['std'])
  assert torch.equal(bits(batch.cpu()), bits(want)), ctx
  _same_outputs(u8r, tr, ctx)
  return int(counts.sum())


@pytest.mark.parametrize('name', list(RUNNERS))
def test_runner_batch_equals_the_converted_uint8_crops(name):
  from centertrack_b200.runner import StreamRunner
  precision, graph, mode, extra = RUNNERS[name]
  opt, model = _model(extra)
  fmt = 'nv12' if mode == 'nv12_device' else 'bgr'
  sizes = [S0, S1 if fmt == 'bgr' else (96, 130)]
  kw = dict(K=K, precision=precision, opt=opt, device_tracking=True, use_graph=graph, frame_sizes=list(sizes),
            crop_size=CROP)
  if mode != 'fixed':
    kw.update(max_frame_size=MAXF, frame_format=fmt)
  if mode == 'idle':
    kw['idle_streams'] = True
  u8r = StreamRunner(model, B, H, W, **kw)
  tr = StreamRunner(model, B, H, W, crop_format=_fmt(list(RUNNERS).index(name)), **kw)
  for r in (u8r, tr):
    r.warm()
  assert tr.launches_per_step == u8r.launches_per_step + 1
  assert tr.d2h_bytes_per_step == u8r.d2h_bytes_per_step and tr.h2d_bytes_per_step == u8r.h2d_bytes_per_step
  n = 0
  for t in range(6):
    step_kw = {}
    if mode != 'fixed' and t == 3:
      sizes[1] = S2
      step_kw = dict(starts=[1], calibs={1: np.array([[300., 0, 60, 0], [0, 310, 75, 0], [0, 0, 1, 0]], np.float32)})
    if mode == 'idle' and t == 1:
      step_kw = dict(idle=[0])
    if mode == 'idle' and t == 2:
      step_kw = dict(starts=[0])
    frames = [_frame(h, w, 100 * t + b) for b, (h, w) in enumerate(sizes)]
    if fmt != 'bgr':
      frames = [bgr_to_yuv420(f, fmt) for f in frames]
    if mode == 'nv12_device':
      frames = [torch.from_numpy(f).to(DEV) for f in frames]
    if 'idle' in step_kw:
      frames[0] = None
    for r in (u8r, tr):
      r.step_frames(list(frames), **step_kw)
    n += _check(u8r, tr, (name, t))
    if 'idle' in step_kw:
      assert tr.fetch_crops()[1][0] == 0
  assert n > 0, name


def test_post_process_runner_batch_equals_the_converted_uint8_crops():
  from centertrack_b200.runner import StreamRunner
  from test_gpu_post_process import H as PH, W as PW, _model as pp_model
  opt, model = pp_model('ctdet', ['--out_thresh', '0.05'])
  sizes = [(120, 200), (90, 140), (64, 96)]
  kw = dict(K=K, opt=opt, device_post_process=True, frame_sizes=sizes, crop_size=(37, 23))
  u8r, tr = StreamRunner(model, 3, PH, PW, **kw), StreamRunner(model, 3, PH, PW, crop_format=_fmt(2), **kw)
  for r in (u8r, tr):
    r.warm()
  n = 0
  for t in range(4):
    frames = [_frame(h, w, 50 * t + b) for b, (h, w) in enumerate(sizes)]
    for r in (u8r, tr):
      r.step_frames(frames)
    n += _check(u8r, tr, ('ctdet', t))
  assert n > 0


def test_track_videos_yields_each_frames_rows_of_the_batch():
  from centertrack_b200.runner import StreamRunner
  from centertrack_b200.videos import Video, track_videos
  opt, model = _model()
  f = _fmt(0)
  r = StreamRunner(model, B, H, W, K=K, opt=opt, device_tracking=True, frame_sizes=[S0, S1], max_frame_size=MAXF,
                   idle_streams=True, crop_size=CROP, crop_format=f)
  r.warm()
  vids = {'a': [_frame(*S0, 300 + i) for i in range(4)], 'b': [_frame(*S2, 400 + i) for i in range(2)],
          'c': [_frame(*S1, 500 + i) for i in range(3)]}
  n, seen = 0, 0
  for vid, i, res, cut in track_videos(r, [Video(k, v) for k, v in vids.items()], crops=True):
    act = [d for d in res if d['active'] != 0]
    assert cut.shape == (len(act), 3) + CROP and cut.dtype == f['dtype'] and cut.is_cuda
    if act:
      want = normalize(np.stack([crop(vids[vid][i], d['bbox'], *CROP) for d in act]), f['dtype'], f['channels'],
                       f['mean'], f['std'])
      assert torch.equal(bits(cut.cpu()), bits(want)), (vid, i)
    n += len(act)
    seen += 1
  assert seen == 9 and n > 0


@pytest.mark.parametrize('graph', [True, False], ids=['graph', 'eager'])
def test_crop_format_changes_no_record_table_or_count(graph):
  """The same frames through runners without crops, with uint8 crops and with the batch: records, tables and counts
  byte-identical every step; the batch runner launches one more kernel per step than the uint8 one and moves the same
  bytes."""
  from centertrack_b200.runner import StreamRunner
  opt, model = _model()
  kw = dict(K=K, opt=opt, device_tracking=True, use_graph=graph, frame_sizes=[S0, S1], max_frame_size=MAXF)
  plain = StreamRunner(model, B, H, W, **kw)
  u8r = StreamRunner(model, B, H, W, crop_size=CROP, **kw)
  tr = StreamRunner(model, B, H, W, crop_size=CROP, crop_format=_fmt(1), **kw)
  for r in (plain, u8r, tr):
    r.warm()
  assert tr.launches_per_step == plain.launches_per_step + 2
  assert tr.d2h_bytes_per_step == u8r.d2h_bytes_per_step == plain.d2h_bytes_per_step + B * 4
  lib = L.lib()
  for t in range(5):
    frames = [_frame(*S0, 700 + t), _frame(*S1, 800 + t)]
    launches = []
    for r in (plain, u8r, tr):
      n0 = lib.ct_launch_count()
      r.step_frames(frames)
      launches.append(lib.ct_launch_count() - n0)
    if not graph and t > 0:
      assert launches[2] == launches[0] + 2 == launches[1] + 1, launches
    _same_outputs(plain, tr, t)
    _check(u8r, tr, t)


def test_a_steps_batch_stays_while_the_next_two_steps_are_submitted():
  from centertrack_b200.runner import StreamRunner
  opt, model = _model()
  r = StreamRunner(model, B, H, W, K=K, opt=opt, device_tracking=True, frame_sizes=[S0, S1], crop_size=CROP,
                   crop_format=_fmt(0))
  r.warm()
  r.step_frames([_frame(*S0, 1), _frame(*S1, 2)])
  batch, counts = r.fetch_crops()
  keep = batch.clone()
  assert counts.sum() > 0
  for t in range(2):
    r.step_frames([_frame(*S0, 10 + t), _frame(*S1, 20 + t)])
    prev, _ = r.previous_crops()
  torch.cuda.synchronize()
  assert torch.equal(bits(batch), bits(keep))
  assert prev.data_ptr() != batch.data_ptr()


@pytest.mark.parametrize('graph', [True, False], ids=['graph', 'eager'])
def test_a_poisoned_buffer_gives_the_same_rows(graph):
  """Each step's batch buffer NaN-filled before the step: rows < N equal those of a runner whose buffer was not, and
  rows >= N keep the fill."""
  from centertrack_b200.runner import NS, StreamRunner
  opt, model = _model()
  kw = dict(K=K, opt=opt, device_tracking=True, use_graph=graph, frame_sizes=[S0, S1], max_frame_size=MAXF,
            idle_streams=True, crop_size=CROP, crop_format=_fmt(4))
  clean, poisoned = StreamRunner(model, B, H, W, **kw), StreamRunner(model, B, H, W, **kw)
  for r in (clean, poisoned):
    r.warm()
  n = 0
  for t in range(5):
    frames = [_frame(*S0, 900 + t), _frame(*S1, 950 + t)]
    step_kw = dict(idle=[1]) if t == 2 else dict(starts=[1]) if t == 3 else {}
    if t == 2:
      frames[1] = None
    torch.cuda.synchronize()
    buf = poisoned.crops[poisoned.t % NS]
    buf.fill_(float('nan'))
    fill = bits(buf[:1].cpu())[0]
    torch.cuda.synchronize()
    for r in (clean, poisoned):
      r.step_frames(list(frames), **step_kw)
    a, ca = clean.fetch_crops()
    b, cb = poisoned.fetch_crops()
    assert np.array_equal(ca, cb) and torch.equal(bits(a.cpu()), bits(b.cpu())), t
    assert (bits(buf[len(b):].cpu()) == fill).all(), t
    n += len(b)
  assert n > 0
