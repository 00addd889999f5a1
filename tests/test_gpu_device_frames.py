"""-m gpu: device frames.  ct_stage_frames against the numpy staging oracle byte for byte (every layout, pitched and
misaligned sources, padded destinations, B across launches, a sentinel around the regions, refusals that write
nothing); StreamRunner fed CUDA tensors against the same runner fed the equivalent arrays, records, tracks and results
bit for bit; ordering against the caller's stream, source lifetime, upload bytes and launch counts."""
import numpy as np
import pytest
import torch

from centertrack_b200 import _lib as L
from centertrack_b200.runner import device_frame_source
from device_frames_oracle import stage_oracle
from test_gpu_camera_switch import _model, _pub
from test_gpu_frames import _frame
from test_gpu_yuv_frames import B, H, K, MAXF, S0, S1, S2, SCHEDULE, W, _same, _yuv

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')
SENTINEL = 0x5A
FMT_OF = {'bgr': 'bgr', 'rgb': 'bgr', 'rgb_planar': 'bgr', 'nv12': 'nv12', 'nv12_planes': 'nv12', 'i420': 'i420',
          'i420_planes': 'i420'}
CT_FMT = {'bgr': L.CT_FRAME_BGR, 'nv12': L.CT_FRAME_NV12, 'i420': L.CT_FRAME_I420}


class _Pool(object):
  """Random device bytes; views into it at a chosen misalignment (the source surfaces of one test)."""

  def __init__(self, nbytes, seed):
    g = torch.Generator(device='cpu').manual_seed(seed)
    self.buf = torch.randint(0, 256, (nbytes + 4096,), dtype=torch.uint8, generator=g).to(DEV)
    self.at = 0

  def view(self, shape, strides, mis):
    """A view of this shape and strides whose first byte is `mis` bytes past a 16-byte boundary."""
    self.at = (self.at + 15) // 16 * 16 + mis
    extent = 1 + sum((n - 1) * s for n, s in zip(shape, strides))
    v = torch.as_strided(self.buf, shape, strides, self.at)
    self.at += extent
    assert self.at <= self.buf.numel()
    return v


def _source(pool, kind, h, w, extra, mis):
  """A device frame of `kind` (a key of FMT_OF) at a row pitch `extra` bytes longer than its row."""
  if kind in ('bgr', 'rgb'):
    return pool.view((h, w, 3), (3 * w + extra, 3, 1), mis)
  if kind == 'rgb_planar':
    p = w + extra
    return pool.view((3, h, w), (h * p + 7, p, 1), mis)
  if kind == 'nv12':
    return pool.view((h * 3 // 2, w), (w + extra, 1), mis)
  if kind == 'i420':                                       # one tensor: rows of exactly w bytes
    return pool.view((h * 3 // 2, w), (w, 1), mis)
  if kind == 'nv12_planes':                               # chroma at an aligned height of the same surface
    p, ha = w + extra, (h + 15) // 16 * 16
    surf = pool.view((ha + h // 2, p), (p, 1), mis)
    return surf[:h, :w], surf[ha:ha + h // 2, :w]
  return (pool.view((h, w), (w + extra, 1), mis), pool.view((h // 2, w // 2), (w // 2 + extra, 1), (mis + 3) % 16),
          pool.view((h // 2, w // 2), (w // 2 + 2 * extra, 1), (mis + 7) % 16))


def _place(exp, f, dense):
  """The expected slot bytes of one staged frame: the oracle's dense frame laid at f.offset with row pitch f.step."""
  o, h, w, step = f.offset, f.h, f.w, f.step
  if f.format == L.CT_FRAME_BGR:
    rows = dense.reshape(h, 3 * w)
  elif f.format == L.CT_FRAME_NV12:
    rows = dense
  else:
    for r in range(h):
      exp[o + r * step:o + r * step + w] = dense[r]
    half = dense[h:].reshape(h, w // 2)                  # U half-rows, then V; two to a destination row
    for q in range(h):
      a = o + (h + q // 2) * step + (q % 2) * (w // 2)
      exp[a:a + w // 2] = half[q]
    return
  for r in range(rows.shape[0]):
    exp[o + r * step:o + r * step + rows.shape[1]] = rows[r]


def _run(streams, seed, pad_step=False):
  """streams: [(kind, (h, w), pitch extra, misalignment)] -> stages them all in one call and checks the whole buffer."""
  total = sum(3 * (h + 16) * (w + 64) + 4096 for _, (h, w), _, _ in streams)
  pool = _Pool(total, seed)
  srcs, dsts, want = (L.FrameSrc * len(streams))(), (L.Frame * len(streams))(), []
  off = 0
  for i, (kind, (h, w), extra, mis) in enumerate(streams):
    fmt = FMT_OF[kind]
    layout = kind if fmt == 'bgr' else 'bgr'
    x = _source(pool, kind, h, w, extra, mis)
    hw, srcs[i] = device_frame_source(x, fmt, layout, DEV, 'stream %d' % i)
    assert hw == (h, w)
    want.append(stage_oracle(x, fmt, layout))
    f = dsts[i]
    row = 3 * w if fmt == 'bgr' else w
    f.h, f.w, f.format = h, w, CT_FMT[fmt]
    f.step = row + (i % 5 if pad_step and fmt != 'i420' else 0)
    f.offset = off + 16 * (i % 3)                           # gaps of sentinel bytes between the regions
    nrows = h if fmt == 'bgr' else h * 3 // 2
    off = (f.offset + (nrows - 1) * f.step + row + 15) // 16 * 16
  nbytes = off + 32
  slot = torch.full((nbytes,), SENTINEL, dtype=torch.uint8, device=DEV)
  lib = L.lib()
  n0 = lib.ct_launch_count()
  L.check(lib.ct_stage_frames(srcs, dsts, len(streams), L.ptr(slot), nbytes, L.stream_ptr()), 'ct_stage_frames')
  assert lib.ct_launch_count() - n0 == -(-len(streams) // L.CT_FRAMES_PER_LAUNCH)
  exp = np.full(nbytes, SENTINEL, np.uint8)
  for f, dense in zip(dsts, want):
    _place(exp, f, dense)
  got = slot.cpu().numpy()
  bad = np.flatnonzero(got != exp)
  assert bad.size == 0, 'bytes differ at %s' % bad[:8].tolist()
  return slot, srcs, dsts, nbytes


KINDS = ['bgr', 'rgb', 'rgb_planar', 'nv12', 'nv12_planes', 'i420', 'i420_planes']


def _mixed(n, seed, sizes):
  rng = np.random.RandomState(seed)
  out = []
  for i in range(n):
    kind = KINDS[i % len(KINDS)]
    h, w = sizes[rng.randint(len(sizes))]
    if FMT_OF[kind] != 'bgr':
      h, w = h + h % 2, w + w % 2
    out.append((kind, (h, w), int(rng.randint(0, 40)), i % 16))
  return out


@pytest.mark.parametrize('kind', KINDS)
def test_every_layout_on_pitched_and_misaligned_surfaces(kind):
  """One layout per call: dense and pitched sources, 16-byte aligned and offset by 1-15 bytes, odd widths on the BGR
  family, 1x1 and 2x2 frames, 1080p, and padded destination rows."""
  sizes = [(1, 1), (2, 2), (2, 2), (3, 17), (37, 53), (64, 96), (480, 640), (1080, 1920)]
  if FMT_OF[kind] != 'bgr':
    sizes = [(h + h % 2, w + w % 2) for h, w in sizes]
  streams = [(kind, hw, extra, mis) for hw in sizes for extra, mis in ((0, 0), (13, 5))]
  streams += [(kind, (36, 48), 32, m) for m in range(1, 16)]
  _run(streams, 11)
  _run(streams, 12, pad_step=True)


@pytest.mark.parametrize('n', [49, 97])
def test_mixed_layouts_across_launches(n):
  _run(_mixed(n, n, [(1, 1), (2, 2), (5, 7), (30, 41), (64, 80), (120, 200)]), 300 + n)


def test_decoder_surfaces_at_full_hd():
  """mot's 1080p NV12 as planes with chroma at 1088 on a 2048-byte pitch, and 1080p RGB / planar RGB."""
  _run([('nv12_planes', (1080, 1920), 128, 0)] * 3 + [('rgb', (1080, 1920), 0, 0), ('rgb_planar', (1080, 1920), 0, 0),
                                                       ('i420_planes', (1080, 1920), 64, 0)], 5)


def test_invalid_arguments_return_invalid_and_write_nothing():
  slot, srcs, dsts, nbytes = _run([('rgb', (6, 10), 0, 0), ('nv12', (4, 8), 0, 0), ('i420_planes', (4, 8), 0, 0)], 9)
  before = slot.clone()
  lib = L.lib()

  def call(mutate, n=3, limit=nbytes, buf=slot):
    s = (L.FrameSrc * 3)(*srcs)
    d = (L.Frame * 3)(*dsts)
    mutate(s, d)
    rc = lib.ct_stage_frames(s, d, n, L.ptr(buf), limit, L.stream_ptr())
    torch.cuda.synchronize()
    assert rc == L.CT_ERR_INVALID, lib.ct_last_error()
    assert torch.equal(slot, before)

  def setp(**kw):
    def m(s, d):
      for k, v in kw.items():
        target, i, field = k.split('_', 2)
        setattr((s if target == 's' else d)[int(i)], field, v)
    return m

  call(lambda s, d: None, n=0)
  last = dsts[2]                                                  # I420 4 x 8: 6 rows of 8 bytes
  call(lambda s, d: None, limit=last.offset + 5 * last.step + 8 - 1)   # one byte past the bound
  call(setp(d_2_offset=nbytes))
  call(setp(d_1_h=5))                                       # odd 4:2:0
  call(setp(d_2_w=7))
  call(setp(d_0_w=0))
  call(setp(d_0_step=29))                                   # < 3 w
  call(setp(d_1_format=L.CT_FRAME_BGR))                     # NV12 source into a BGR frame
  call(setp(d_0_format=L.CT_FRAME_I420))
  call(setp(s_1_layout=9))
  call(lambda s, d: s[0].pitch.__setitem__(0, 29))                # < 3 w
  call(lambda s, d: s[2].pitch.__setitem__(2, 3))                 # V pitch < w / 2
  call(lambda s, d: s[2].plane.__setitem__(1, None))
  call(lambda s, d: None, buf=None)


# ------------------------------------------------------------------------------------------------ the runner

def _device(x, fmt, layout, form, seed):
  """A host frame as the runner takes it -> the same frame as a device tensor (or planes) on a pitched surface."""
  rng = np.random.RandomState(seed)
  if fmt == 'bgr':
    h, w = x.shape[:2]
    if layout == 'rgb_planar':
      surf = torch.randint(0, 256, (3, h + 2, w + 9), dtype=torch.uint8, device=DEV)
      v = surf[:, 1:h + 1, 3:w + 3]
      v.copy_(torch.from_numpy(np.ascontiguousarray(x[..., ::-1].transpose(2, 0, 1))))
      return v
    surf = torch.randint(0, 256, (h + 3, w + 5, 3), dtype=torch.uint8, device=DEV)
    v = surf[:h, 2:w + 2]
    v.copy_(torch.from_numpy(np.ascontiguousarray(x if layout == 'bgr' else x[..., ::-1])))
    return v
  h, w = x.shape[0] // 3 * 2, x.shape[1]
  if form == 'one':
    if fmt == 'i420':
      return torch.from_numpy(x).to(DEV)
    surf = torch.randint(0, 256, (x.shape[0], w + 32), dtype=torch.uint8, device=DEV)
    surf[:, :w] = torch.from_numpy(x)
    return surf[:, :w]
  ha = (h + 15) // 16 * 16
  p = w + int(rng.randint(1, 64))
  if fmt == 'nv12':
    surf = torch.randint(0, 256, (ha + h // 2, p), dtype=torch.uint8, device=DEV)
    Y, UV = surf[:h, :w], surf[ha:ha + h // 2, :w]
    Y.copy_(torch.from_numpy(x[:h]))
    UV.copy_(torch.from_numpy(x[h:]))
    return Y, UV
  half = x[h:].reshape(h, w // 2)
  planes = []
  for a in (x[:h], half[:h // 2], half[h // 2:]):
    s = torch.randint(0, 256, (a.shape[0] + 1, a.shape[1] + 11), dtype=torch.uint8, device=DEV)
    v = s[1:, 5:5 + a.shape[1]]
    v.copy_(torch.from_numpy(np.ascontiguousarray(a)))
    planes.append(v)
  return tuple(planes)


def _host(fmt, size, seed):
  return _frame(size[0], size[1], seed) if fmt == 'bgr' else _yuv(fmt, size, seed)


def _make(model, opt, precision, graph, fmt, idle, capacity):
  from centertrack_b200.runner import StreamRunner
  sizes = SCHEDULE[0][0]
  r = StreamRunner(model, B, H, W, K=K, precision=precision, device='cuda', opt=opt, device_tracking=True,
                   use_graph=graph, frame_sizes=sizes, max_frame_size=MAXF if capacity else None,
                   idle_streams=idle or None, frame_format=fmt)
  r.warm()
  return r


def _play(r, fmt, idle, capacity, device=None, public=False):
  """The schedule's frames (device=(layout, form): as device frames) -> per step (records, tracks, counts, results).
  A fixed-size runner keeps each stream's first size and starts stream 1 without a size change."""
  out = []
  for k, (sizes, starts, gone) in enumerate(SCHEDULE):
    if not capacity:
      sizes = SCHEDULE[0][0]
    xs, pub = [], []
    for b, s in enumerate(sizes):
      if idle and b in gone:
        xs.append(None)
        pub.append(None)
        continue
      x = _host(fmt, s, 100 * k + b)
      xs.append(x if device is None else _device(x, fmt, device[0], device[1], 100 * k + b))
      pub.append(_pub(100 * k + b, s))
    kw = dict(starts=starts or None, public_dets=pub if public else None)
    if 1 in starts:
      kw['calibs'] = {1: np.float32([[900, 0, 60, 0], [0, 900, 50, 0], [0, 0, 1, 0]])}
    if idle:
      kw['idle'] = gone
    if device is not None:
      kw['layout'] = device[0]
    r.step_frames(xs, **kw)
    out.append((r.fetch(), *r.fetch_tracks(), r.fetch_results()))
  return out


# (precision, graph, flip, idle, capacity, frame_format, layout, form)
CASES = [('bf16', True, False, False, True, 'bgr', 'bgr', None),
         ('bf16', False, True, True, True, 'bgr', 'rgb', None),
         ('bf16x3', True, False, True, True, 'bgr', 'rgb_planar', None),
         ('fp32', False, True, False, True, 'nv12', 'bgr', 'one'),
         ('bf16', True, True, True, True, 'nv12', 'bgr', 'planes'),
         ('fp32', True, False, True, True, 'i420', 'bgr', 'one'),
         ('bf16x3', False, True, False, True, 'i420', 'bgr', 'planes'),
         ('bf16', True, False, False, False, 'bgr', 'rgb', None),
         ('fp32', False, True, False, False, 'bgr', 'rgb_planar', None),
         ('bf16x3', True, True, False, False, 'bgr', 'bgr', None)]


@pytest.mark.parametrize('precision,graph,flip,idle,capacity,fmt,layout,form', CASES,
                         ids=['%s-%s-%s-%s-%s-%s-%s' % (p, 'graph' if g else 'eager', 'flip' if f else 'noflip',
                                                        'idle' if i else 'busy', 'cap' if c else 'fixed',
                                                        fm if fm != 'bgr' else la, fo or '')
                              for p, g, f, i, c, fm, la, fo in CASES])
def test_device_fed_runner_equals_array_fed_runner(precision, graph, flip, idle, capacity, fmt, layout, form):
  """Sizes change at starts (capacity runners), calibs, idle streams, --flip_test: the same records, tracks, counts and
  fetch_results() whether the frames come as arrays or as device tensors."""
  opt, model = _model('coco_tracking', ['--flip_test'] if flip else [])
  got = {}
  for feed in ('host', 'device'):
    r = _make(model, opt, precision, graph, fmt, idle, capacity)
    got[feed] = _play(r, fmt, idle, capacity, None if feed == 'host' else (layout, form))
    if feed == 'device':
      assert r.frames_read() is not None and r.frames_read().query() in (True, False)
    del r
  _same(got['device'], got['host'])


def test_track_videos_mot_public_hungarian_device_tensors():
  from centertrack_b200.runner import StreamRunner
  from centertrack_b200.videos import Video, track_videos
  opt, model = _model('mot', ['--public_det', '--hungarian'])
  spec = [(S0, 3), (S2, 2), (S1, 4), (S0, 2), (S2, 3)]

  def videos(device):
    out = []
    for v, (s, n) in enumerate(spec):
      fs = [_yuv('nv12', s, 50 * v + i) for i in range(n)]
      if device:
        fs = [_device(y, 'nv12', 'bgr', 'planes' if v % 2 else 'one', 50 * v + i) for i, y in enumerate(fs)]
      seeds = [{'score': 0.9, 'class': 1, 'bbox': [10. + v, 12., 60., 70. + v]},
               {'score': 0.8, 'class': 1, 'bbox': [70., 30., 110., 90.]}]
      out.append(Video(v, fs, pre_dets=seeds, public_dets=[_pub(50 * v + i, s) for i in range(n)]))
    return out

  got = {}
  for device in (False, True):
    # six streams for five videos: stream 5 never plays one and is fed the filler frame of the videos' kind
    r = StreamRunner(model, 6, H, W, K=K, precision='bf16', device='cuda', opt=opt, device_tracking=True,
                     frame_sizes=[S0] * 6, max_frame_size=MAXF, frame_format='nv12')
    r.warm()
    got[device] = {(v, i): res for v, i, res in track_videos(r, videos(device))}
    del r
  assert sorted(got[True]) == sorted(got[False]) == sorted((v, i) for v, (_, n) in enumerate(spec) for i in range(n))
  n = 0
  for key, want in got[False].items():
    a = got[True][key]
    assert len(a) == len(want), key
    n += len(a)
    for x, y in zip(a, want):
      for k in y:
        assert np.array_equal(np.asarray(x[k]), np.asarray(y[k])), (key, k)
  assert n > 0


def test_track_videos_refuses_mixed_kinds():
  from centertrack_b200.runner import StreamRunner
  from centertrack_b200.videos import Video, track_videos
  opt, model = _model('coco_tracking')
  r = StreamRunner(model, 2, H, W, K=K, precision='bf16', device='cuda', opt=opt, device_tracking=True,
                   frame_sizes=[S0, S0], max_frame_size=MAXF)
  x = _frame(S0[0], S0[1], 1)
  vids = [Video('a', [x]), Video('b', [torch.from_numpy(x).to(DEV)]), Video('c', [x])]
  with pytest.raises(ValueError, match="video 'b' brings device frames; the videos before it bring arrays"):
    list(track_videos(r, vids))


# ------------------------------------------------------------------------------------------------ ordering, lifetime

def test_ordering_lifetime_upload_bytes_and_launches():
  """Frames written by torch ops on a non-default stream made current before step_frames, and sources deleted right
  after it whose memory is reallocated and overwritten on the caller's stream (while the copy stream is held back) give
  the array-fed records.  A device-fed step uploads no frame bytes and runs launches_per_step + the staging launches."""
  opt, model = _model('coco_tracking')
  lib = L.lib()
  want = None
  res = {}
  for feed in ('host', 'device'):
    r = _make(model, opt, 'bf16', False, 'bgr', False, True)
    side = torch.cuda.Stream()
    out, counts, h2d = [], [], []
    for k in range(5):
      xs = [_frame(s[0], s[1], 100 * k + b) for b, s in enumerate(SCHEDULE[0][0])]
      if feed == 'host':
        n0 = lib.ct_launch_count()
        r.step_frames(xs)
        counts.append(lib.ct_launch_count() - n0)
      else:
        pinned = [torch.from_numpy(x).pin_memory() for x in xs]
        with torch.cuda.stream(side):
          torch.cuda._sleep(20000000)                         # the writes land well after step_frames returns
          dev = [torch.zeros(x.shape, dtype=torch.uint8, device=DEV) for x in xs]
          for d, p in zip(dev, pinned):
            d.copy_(p, non_blocking=True)
            d.add_(1).sub_(1)
          with torch.cuda.stream(r.copy):                     # hold the copy stream back behind the caller's reuse
            torch.cuda._sleep(20000000)
          n0 = lib.ct_launch_count()
          r.step_frames(dev)
          counts.append(lib.ct_launch_count() - n0)
          del dev, d
          junk = [torch.empty(x.shape, dtype=torch.uint8, device=DEV).fill_(77) for x in xs]
          del junk
      h2d.append(r.h2d_bytes_per_step)
      out.append((r.fetch(), *r.fetch_tracks(), r.fetch_results()))
    res[feed] = (out, counts, h2d, r.launches_per_step)
    del r
  _same(res['device'][0], res['host'][0])
  out, counts, h2d, per_step = res['device']
  assert all(b == 0 for b in h2d), h2d
  assert all(b > 0 for b in res['host'][2]), res['host'][2]
  # B = 3 streams: one staging launch on top of the step's
  assert [c - 1 for c in counts[1:]] == res['host'][1][1:], (counts, res['host'][1])
  assert all(c == per_step + 1 for c in counts[1:]), (counts, per_step)


def test_step_refuses_mixed_kinds_and_layouts_on_arrays():
  opt, model = _model('coco_tracking')
  r = _make(model, opt, 'bf16', False, 'bgr', False, True)
  xs = [_frame(s[0], s[1], b) for b, s in enumerate(SCHEDULE[0][0])]
  mixed = [xs[0], torch.from_numpy(xs[1]).to(DEV), xs[2]]
  with pytest.raises(ValueError, match=r'stream\(s\) \[1\] bring device tensors and stream\(s\) \[0, 2\] host arrays'):
    r.step_frames(mixed)
  with pytest.raises(ValueError, match="layout='rgb': applies to device frames"):
    r.step_frames(xs, layout='rgb')
  with pytest.raises(ValueError, match=r"frames\[1\]: on cpu, not on the runner's device"):
    r.step_frames([torch.from_numpy(x) if b == 1 else torch.from_numpy(x).to(DEV) for b, x in enumerate(xs)])
  assert r.t == 0 and r.frames_read() is None
