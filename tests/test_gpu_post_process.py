"""Detections post-processed on the device (ct_post_process, StreamRunner(device_post_process=True)): the kernel against
the host generic_post_process + merge_outputs on records decoded from seeded heads, its mapped form against the
identity launch, runners of detection and tracking models against host post-processing of their own records, the
records and launches of runners without the option, and track_videos."""
import numpy as np
import pytest
import torch

from centertrack_b200 import _lib as L
from centertrack_b200 import synthetic as wt
from helpers import decode_inputs

gpu = pytest.mark.gpu
DEV = torch.device('cuda')
EXACT_PAY = ('dep', 'dim', 'velocity', 'nuscenes_att')          # copied fields: bit for bit against the host
ANGLES = ('alpha', 'loc', 'rot_y')          # atan2f: within 1e-5 relative, 1e-6 absolute of numpy's
SENTINEL = 12345.0


def _opt(task, extra=()):
  from centertrack_b200.opts import opts
  return opts().init([task] + list(extra))


def _host(opt, rec, layout, metas):
  """generic_post_process of each stream's records with its meta, then merge_outputs' score > out_thresh."""
  from centertrack_b200.decode import views_from_records
  from centertrack_b200.post_process import generic_post_process
  views = {k: v.numpy() for k, v in views_from_records(torch.from_numpy(rec), layout).items()}
  out = []
  for b, m in enumerate(metas):
    if m is None:
      out.append(None)
      continue
    one = {k: v[b:b + 1] for k, v in views.items()}
    res = generic_post_process(opt, one, [m['c']], [m['s']], m['out_height'], m['out_width'], opt.num_classes,
                               [m['calib']])[0]
    out.append([r for r in res if r['score'] > opt.out_thresh])
  return out


def _row(item):
  """The CT_DET_FLOATS columns of a host result dict (tracking 0 when the head set has none)."""
  return np.array([item['score'], item['class'], *np.asarray(item['ct'], np.float32),
                   *np.asarray(item.get('tracking', (0., 0.)), np.float32), *item['bbox']], np.float32)


def _restate(rec, layout, trans):
  """generic_post_process's affine as the kernel computes it, in numpy's elementwise fp32 (x t0 + y t1 + t2, each
  product and sum rounded once): the 10 columns and the keypoints of records [n, F] through trans [2, 3].  The host
  path's transform_preds_with_trans is an fp32 np.dot, whose BLAS may fuse a multiply-add (1 ulp apart on some CPUs)."""
  t = np.asarray(trans, np.float32)
  aff = lambda x, y, r: (t[r, 0] * x + t[r, 1] * y) + t[r, 2]
  cx, cy = rec[:, L.CT_REC_XS], rec[:, L.CT_REC_YS]
  ctx, cty = aff(cx, cy, 0), aff(cx, cy, 1)
  tx = ty = np.zeros_like(cx)
  if 'tracking' in layout:
    o = layout['tracking'][0]
    px, py = rec[:, o] + cx, rec[:, o + 1] + cy
    tx, ty = aff(px, py, 0) - ctx, aff(px, py, 1) - cty
  bl, bt, br, bb = (rec[:, L.CT_REC_BBOX + i] for i in range(4))
  x0, y0, x1, y1 = aff(bl, bt, 0), aff(bl, bt, 1), aff(br, bb, 0), aff(br, bb, 1)
  if all(k in layout for k in ('rot', 'dep', 'dim')):      # the amodal centre
    if 'amodel_offset' in layout:
      o = layout['amodel_offset'][0]
      mx, my = (bl + br) * np.float32(0.5) + rec[:, o], (bt + bb) * np.float32(0.5) + rec[:, o + 1]
      ctx, cty = aff(mx, my, 0), aff(mx, my, 1)
    else:
      ctx, cty = (x0 + x1) * np.float32(0.5), (y0 + y1) * np.float32(0.5)
  rows = np.stack([rec[:, L.CT_REC_SCORE], rec[:, L.CT_REC_CLS] + np.float32(1), ctx, cty, tx, ty, x0, y0, x1, y1], 1)
  hps = None
  if 'hps' in layout:
    o, w = layout['hps_refined' if 'hps_refined' in layout else 'hps']
    q = rec[:, o:o + w]
    hps = np.stack([aff(q[:, 2 * (k // 2)], q[:, 2 * (k // 2) + 1], k % 2) for k in range(w)], 1)
  return rows.astype(np.float32), hps


def _close(a, b):
  """Coordinates of the device and of the host path: equal up to the host np.dot's fused multiply-adds."""
  return np.allclose(np.asarray(a, np.float64), np.asarray(b, np.float64), rtol=1e-6, atol=5e-4)


def _check_stream(ctx, want, dets, count, pay, pay_layout, rec, layout, trans):
  """One stream's device rows: the count, score and class, and the copied payload fields (dep, dim, velocity,
  nuscenes_att) bit for bit against the host dicts; the 10 columns and the keypoints bit for bit against the kernel's
  fp32 arithmetic restated (_restate) and within np.dot's rounding of the host's; alpha, loc and rot_y within the
  atan2f bound; the sentinel past the count untouched."""
  assert count == len(want), (ctx, count, len(want))
  assert np.all(dets[count:] == SENTINEL), ctx
  if pay is not None:
    assert np.all(pay[count:] == SENTINEL), ctx
  if not want:
    return
  host = np.stack([_row(w) for w in want])
  rows, hps = _restate(rec[:count], layout, trans)
  assert np.array_equal(dets[:count], rows), (ctx, np.argwhere(dets[:count] != rows)[:4])
  assert np.array_equal(dets[:count, :2], host[:, :2]) and _close(dets[:count], host), ctx
  for k, (o, w) in pay_layout.items():
    got = pay[:count, o:o + w]
    ref = np.array([np.asarray(x[k], np.float64).reshape(w) for x in want]).reshape(-1, w)
    if k in EXACT_PAY:
      assert np.array_equal(got, ref.astype(np.float32)), (ctx, k)
    elif k == 'hps':
      assert np.array_equal(got, hps) and _close(got, ref), (ctx, k)
    else:
      assert np.allclose(got.astype(np.float64), ref, rtol=1e-5, atol=1e-6), (ctx, k, np.abs(got - ref).max())


# ------------------------------------------------------------------------------------------------ kernel vs host
def _heads(kind, B, C_, H, W, seed):
  """Seeded head maps of one head set -> (task for opts, maps)."""
  base = decode_inputs('ddd' if kind.startswith('ddd') or kind == 'nuscenes' else
                       ('pose' if kind == 'pose' else ('mot' if kind == 'ltrb_amodal' else 'coco')), B, C_, H, W, seed)
  rng = np.random.RandomState(seed + 1)
  base['dep'] = base['dep'] + 1.0 if 'dep' in base else None
  keep = {'2d': ('hm', 'reg', 'wh'), 'tracking': ('hm', 'reg', 'wh', 'tracking'),
          'ltrb_amodal': ('hm', 'reg', 'wh', 'tracking', 'ltrb_amodal'),
          'ddd_offset': ('hm', 'reg', 'wh', 'dep', 'rot', 'dim', 'amodel_offset'),
          'ddd_box': ('hm', 'reg', 'wh', 'dep', 'rot', 'dim'),
          'nuscenes': ('hm', 'reg', 'wh', 'tracking', 'dep', 'rot', 'dim', 'amodel_offset'),
          'pose': ('hm', 'reg', 'wh', 'hps', 'hm_hp', 'hp_offset')}[kind]
  maps = {k: base[k] for k in keep}
  if kind == 'nuscenes':
    maps['velocity'] = rng.randn(B, 3, H, W).astype(np.float32)
    maps['nuscenes_att'] = rng.rand(B, 8, H, W).astype(np.float32)
  task = {'pose': 'multi_pose', 'nuscenes': 'tracking,ddd'}.get(kind, 'ddd' if kind.startswith('ddd') else 'ctdet')
  return task, maps


def _streams_geometry(B, seed):
  """Each stream its own source size, (c, s) and calib, and the metas of generic_post_process."""
  rng = np.random.RandomState(seed)
  metas = []
  for _ in range(B):
    h, w = int(rng.randint(200, 1000)), int(rng.randint(200, 1700))
    c = np.array([w / 2. + rng.uniform(-9, 9), h / 2. + rng.uniform(-9, 9)], np.float32)
    calib = np.array([[rng.uniform(600, 1300), 0, w / 2. + rng.uniform(-20, 20), rng.uniform(-1, 1)],
                      [0, rng.uniform(600, 1300), h / 2. + rng.uniform(-20, 20), rng.uniform(-1, 1)],
                      [0, 0, 1, rng.uniform(-0.1, 0.1)]], np.float32)
    metas.append(dict(c=c, s=max(h, w) * float(rng.uniform(0.9, 1.2)), calib=calib))
  return metas


def _decoded(kind, B, K, seed, H=24, W=40):
  from centertrack_b200.decode import generic_decode
  task, maps = _heads(kind, B, 10 if kind != 'pose' else 1, H, W, seed)
  res = generic_decode({k: torch.from_numpy(v).to(DEV) for k, v in maps.items()}, K=K)
  return task, res.records.contiguous(), res.layout


def _tables(opt, B, K, layout, F, metas, H, W):
  from centertrack_b200.device_detections import DeviceDetections
  det = DeviceDetections(opt, B, K, F, layout, 4 * H, 4 * W, DEV, centers=[m['c'] for m in metas],
                         scales=[m['s'] for m in metas], calibs=np.stack([m['calib'] for m in metas]))
  det.dets.fill_(SENTINEL)
  if det.payload is not None:
    det.payload.fill_(SENTINEL)
  return det


KINDS = ['2d', 'tracking', 'ltrb_amodal', 'ddd_offset', 'ddd_box', 'nuscenes', 'pose']
SHAPES = [(1, 1), (32, 100), (97, 512)]


@gpu
@pytest.mark.parametrize('thresh', ['-1', '0.3', 'record'])
@pytest.mark.parametrize('B,K', SHAPES, ids=['B1K1', 'B32K100', 'B97K512'])
@pytest.mark.parametrize('kind', KINDS)
def test_kernel_equals_host_post_process(kind, B, K, thresh):
  H, W = 24, 40
  task, rec, layout = _decoded(kind, B, K, 700 + KINDS.index(kind))
  opt = _opt(task)
  rec_np = rec.cpu().numpy()
  if thresh == 'record':          # exactly one record's score: that record and every one after it are excluded
    opt.out_thresh = float(rec_np[B // 2, K // 2, L.CT_REC_SCORE])
  else:
    opt.out_thresh = float(thresh)
  metas = [dict(m, out_height=H, out_width=W) for m in _streams_geometry(B, 11 + K)]
  det = _tables(opt, B, K, layout, rec.shape[2], metas, H, W)
  det.step(rec)
  torch.cuda.synchronize()
  dets, counts = det.dets.cpu().numpy(), det.counts.cpu().numpy()
  pay = det.payload.cpu().numpy() if det.payload is not None else None
  want = _host(opt, rec_np, layout, metas)
  if thresh == 'record':
    assert counts[B // 2] == (rec_np[B // 2, :, 0] > opt.out_thresh).sum() < K
  from centertrack_b200.image import get_affine_transform
  for b in range(B):
    trans = get_affine_transform(metas[b]['c'], metas[b]['s'], 0, (W, H), inv=1).astype(np.float32)
    _check_stream((kind, B, K, thresh, b), want[b], dets[b], int(counts[b]), None if pay is None else pay[b],
                  det.payload_layout, rec_np[b], layout, trans)
  assert counts.sum() > 0 or (thresh == 'record' and B * K == 1)


@gpu
@pytest.mark.parametrize('kind', ['tracking', 'nuscenes', 'pose'])
def test_mapped_form_equals_the_identity_launch_on_permuted_records(kind):
  """Images [n] with a permuted map and -1 padding: each listed stream's rows equal the identity launch's on the
  records permuted into stream order; streams no image maps to keep their bytes."""
  B, K, n = 12, 64, 9
  task, rec, layout = _decoded(kind, B, K, 810)
  opt = _opt(task, ['--out_thresh', '0.2'])
  metas = _streams_geometry(B, 99)
  full = _tables(opt, B, K, layout, rec.shape[2], metas, 24, 40)
  full.step(rec)
  rng = np.random.RandomState(3)
  streams = rng.permutation(B)[:n - 2].tolist() + [-1, -1]        # 7 live images, 2 padding
  imgs = torch.zeros((n, K, rec.shape[2]), dtype=torch.float32, device=DEV)
  for i, s in enumerate(streams):
    if s >= 0:
      imgs[i] = rec[s]
  mapped = _tables(opt, B, K, layout, rec.shape[2], metas, 24, 40)
  garbage = torch.from_numpy(np.random.RandomState(4).randn(B, K, L.CT_DET_FLOATS).astype(np.float32)).to(DEV)
  mapped.dets.copy_(garbage)
  mapped.counts.fill_(-7)
  mapped.step_mapped(imgs, torch.tensor(streams, dtype=torch.int32, device=DEV))
  torch.cuda.synchronize()
  for b in range(B):
    if b in streams:
      c = int(full.counts[b])
      assert int(mapped.counts[b]) == c
      assert torch.equal(mapped.dets[b, :c], full.dets[b, :c]), b
      assert torch.equal(mapped.dets[b, c:], garbage[b, c:]), b
      if full.payload is not None:
        assert torch.equal(mapped.payload[b, :c], full.payload[b, :c]), b
    else:
      assert int(mapped.counts[b]) == -7 and torch.equal(mapped.dets[b], garbage[b]), b
      if full.payload is not None:
        assert torch.all(mapped.payload[b] == SENTINEL)


# ------------------------------------------------------------------------------------------------ runners
H, W = 64, 96


def _model(task, extra=()):
  from centertrack_b200.model import create_model
  opt = _opt(task, ['--input_h', str(H), '--input_w', str(W)] + list(extra))
  m = create_model(opt.arch, opt.heads, opt.head_conv, opt=opt)
  m.load_state_dict(wt.make_state_dict(m.state_dict(), 317, rename=getattr(m, 'RENAME', ())))
  with torch.no_grad():           # boxes of a few pixels (the synthetic weights give ~0 wh)
    m.state_dict()['wh.2.bias'].fill_(3.0)
  return opt, m.cuda()


def _images_meta(opt):
  """The default geometry of images mode: a source image of exactly the network input size, its default calib."""
  from centertrack_b200.dataset_info import get_dataset
  from centertrack_b200.detector import default_calib
  c, s = np.array([W / 2., H / 2.], np.float32), max(H, W) * 1.0
  f = opt.test_focal_length if opt.test_focal_length >= 0 else get_dataset(opt.dataset).rest_focal_length
  return dict(c=c, s=s, out_height=H // 4, out_width=W // 4, calib=default_calib(f, W, H))


def _frames(rng, sizes, fmt='bgr'):
  from centertrack_b200.runner import frame_layout
  return [rng.randint(0, 256, frame_layout(fmt, h, w)[0]).astype(np.uint8) for h, w in sizes]


def _trans(m):
  from centertrack_b200.image import get_affine_transform
  return get_affine_transform(m['c'], m['s'], 0, (m['out_width'], m['out_height']), inv=1).astype(np.float32)


def _same(ctx, g, w, rec_row, layout, trans):
  """A device result dict against the host's for the same record: the keys, score and class, the copied fields bit
  for bit; the 10 columns and the keypoints bit for bit against _restate and within np.dot's rounding of the host's;
  the angles within the atan2f bound."""
  assert set(g) == set(w), (ctx, set(g) ^ set(w))
  rows, hps = _restate(rec_row[None], layout, trans)
  assert np.array_equal(_row(g), rows[0]) and np.array_equal(_row(g)[:2], _row(w)[:2]) and _close(_row(g), _row(w)), ctx
  for k in set(g) - {'score', 'class', 'ct', 'tracking', 'bbox'}:
    a, e = np.asarray(g[k], np.float64), np.asarray(w[k], np.float64).reshape(np.shape(g[k]))
    if k in ANGLES:
      assert np.allclose(a, e, rtol=1e-5, atol=1e-6), (ctx, k)
    elif k == 'hps':
      assert np.array_equal(np.asarray(g[k], np.float32), hps[0]) and _close(a, e), (ctx, k)
    else:
      assert np.array_equal(a, e), (ctx, k)


def _compare(runner, opt, rec, metas, ctx):
  """previous_results() (the step whose records `rec` are) against host post-processing of those records."""
  got = runner.previous_results()
  want = _host(opt, rec, runner.layout, metas)
  for b in range(runner.B):
    if want[b] is None:
      assert got[b] is None, (ctx, b)
      continue
    assert len(got[b]) == len(want[b]), (ctx, b)
    for j, (g, w) in enumerate(zip(got[b], want[b])):
      _same((ctx, b, j), g, w, rec[b, j], runner.layout, _trans(metas[b]))
  return sum(len(w) for w in want if w)


RUNNERS = {
    # name: (task, extra opts, precision, graph, mode)
    'ctdet_bf16_graph_images': ('ctdet', [], 'bf16', True, 'images'),
    'ctdet_fp32_eager_fixed': ('ctdet', ['--out_thresh', '0.05'], 'fp32', False, 'fixed'),
    'ctdet_bf16_graph_idle': ('ctdet', [], 'bf16', True, 'idle'),
    'ctdet_bf16_graph_device': ('ctdet', [], 'bf16', True, 'device'),
    'ddd_bf16x3_graph_capacity': ('ddd', [], 'bf16x3', True, 'capacity'),
    'ddd_fp32_graph_idle_flip': ('ddd', ['--flip_test'], 'fp32', True, 'idle'),
    'ddd_bf16_eager_nv12': ('ddd', [], 'bf16', False, 'nv12'),
    'pose_bf16_graph_fixed_flip': ('multi_pose', ['--flip_test'], 'bf16', True, 'fixed'),
    'pose_fp32_graph_images': ('multi_pose', [], 'fp32', True, 'images'),
    'tracking_bf16_graph_capacity': ('tracking', ['--pre_hm'], 'bf16', True, 'capacity'),
    'tracking_bf16x3_eager_images_flip': ('tracking', ['--flip_test'], 'bf16x3', False, 'images'),
}


@gpu
@pytest.mark.parametrize('name', list(RUNNERS))
def test_runner_results_equal_host_post_process_of_its_records(name):
  """fetch_results() / previous_results() / fetch_detections() of a device_post_process runner against
  generic_post_process + merge_outputs of the records the same runner returns, with meta(b) (frames mode) or the
  default geometry (images mode).  Capacity runners start streams with a new size and calib mid-run."""
  from centertrack_b200.runner import StreamRunner
  task, extra, precision, graph, mode = RUNNERS[name]
  opt, model = _model(task, extra)
  B, K, steps = 3, 40, 5
  rng = np.random.RandomState(sum(map(ord, name)))
  sizes = [(120, 200), (90, 140), (64, 96)]
  calibs = [np.array([[700. + 50 * b, 0, 100 - b, 0.5], [0, 720., 60 + b, -0.2], [0, 0, 1, 0.01]], np.float32)
            for b in range(B)]
  kw = dict(K=K, precision=precision, opt=opt, use_graph=graph, device_post_process=True)
  fmt = 'nv12' if mode == 'nv12' else 'bgr'
  if mode != 'images':
    kw.update(frame_sizes=sizes, calibs=calibs)
  if mode in ('capacity', 'idle', 'nv12', 'device'):
    kw.update(max_frame_size=(240, 320), frame_format=fmt)
  if mode == 'idle':
    kw['idle_streams'] = True
  runner = StreamRunner(model, B, H, W, **kw)
  runner.warm()
  assert runner.post is not None and runner.tracker is None
  checked = 0
  metas = None
  for t in range(steps):
    step_kw = {}
    if mode in ('capacity', 'nv12', 'device') and t == 2:     # a new camera on stream 1: size and calib change
      sizes[1] = (200, 150)
      step_kw = dict(starts=[1], calibs={1: np.array([[900., 0, 70, 0], [0, 880, 95, 0], [0, 0, 1, 0]], np.float32)})
    idle = []
    if mode == 'idle' and t in (1, 2):
      idle = [2]
      step_kw['idle'] = idle
    if mode == 'idle' and t == 3:
      step_kw['starts'] = [2]
    if mode == 'images':
      rec = runner.step_host(wt.synthetic_inputs(B, H, W, seed=40 + t)[0].pin_memory(), **step_kw)
      now = [_images_meta(opt)] * B
    else:
      frames = _frames(rng, sizes, fmt)
      if mode == 'device':
        frames = [torch.from_numpy(f).to(DEV) for f in frames]
      for b in idle:
        frames[b] = None
      rec = runner.step_frames(frames, **step_kw)
      now = [None if b in idle else runner.meta(b) for b in range(B)]
    if rec is not None:
      checked += _compare(runner, opt, rec, metas, (name, t))
    metas = now
  got = runner.fetch_results()
  dets, counts, pay = runner.fetch_detections()
  rec = runner.fetch()
  want = _host(opt, rec, runner.layout, metas)
  for b in range(B):
    assert len(got[b]) == len(want[b]) == counts[b]
    for j, (g, w) in enumerate(zip(got[b], want[b])):
      _same((name, b, j), g, w, rec[b, j], runner.layout, _trans(metas[b]))
      assert np.array_equal(dets[b, j], _row(g)), (name, b, j)
      for k, (o, n) in runner.post.payload_layout.items():
        assert np.array_equal(np.asarray(g[k], np.float32).reshape(n), pay[b, j, o:o + n]), (name, b, k)
  assert (pay is None) == (runner.post.payload is None)
  assert 'tracking' in got[0][0] if task == 'tracking' else 'tracking' not in got[0][0]
  assert checked > 0


@gpu
@pytest.mark.parametrize('task,extra,precision,mode', [('ctdet', [], 'bf16', 'fixed'), ('ddd', [], 'fp32', 'images'),
                                                       ('multi_pose', ['--flip_test'], 'bf16', 'idle')])
def test_option_changes_no_records_and_adds_one_launch_and_the_table(task, extra, precision, mode):
  """The same model and frames through a runner with and without device_post_process: byte-identical records every
  step; launches_per_step one more (and that many launches counted in an eager step), d2h_bytes_per_step the table,
  counts and payload more."""
  from centertrack_b200.runner import StreamRunner
  opt, model = _model(task, extra)
  B, K = 3, 30
  sizes = [(120, 200), (90, 140), (64, 96)]
  kw = dict(K=K, precision=precision, opt=opt)
  if mode != 'images':
    kw['frame_sizes'] = sizes
  if mode == 'idle':
    kw.update(max_frame_size=(240, 320), idle_streams=True)
  runners = [StreamRunner(model, B, H, W, device_post_process=p, **kw) for p in (False, True)]
  eager = [StreamRunner(model, B, H, W, device_post_process=p, use_graph=False, **kw) for p in (False, True)]
  for r in runners + eager:
    r.warm()
  plain, post = runners
  assert post.launches_per_step == plain.launches_per_step + 1
  table = post.post.dets.numel() * 4 + B * 4 + (post.post.payload.numel() * 4 if post.post.payload is not None else 0)
  assert post.d2h_bytes_per_step == plain.d2h_bytes_per_step + table
  rng = np.random.RandomState(8)
  for t in range(4):
    if mode == 'images':
      x = wt.synthetic_inputs(B, H, W, seed=70 + t)[0].pin_memory()
      step = lambda r: r.step_host(x)
    else:
      frames = _frames(rng, sizes)
      idle = [0] if (mode == 'idle' and t == 2) else None
      step = lambda r: r.step_frames([None if idle and b in idle else f for b, f in enumerate(frames)],
                                     idle=idle, starts=[0] if (mode == 'idle' and t == 3) else None)
    outs = []
    for r in runners + eager:
      step(r)
      outs.append(r.fetch())          # one runner at a time: they share the engine's activation buffers
    assert all(np.array_equal(outs[0].view(np.uint8), o.view(np.uint8)) for o in outs[1:]), t
  for r in eager:                     # launches of one eager step, counted by the library
    r._n = r.B
    L.lib().ct_reset_launch_count()
    r._eager(r.t % 3)
    torch.cuda.synchronize()
    r.counted = L.lib().ct_launch_count()
  assert eager[1].counted == eager[0].counted + 1


@gpu
def test_track_videos_on_a_post_process_runner_equals_per_frame_host_post_processing():
  """Videos of different lengths, sizes and calibs through a capacity ddd runner with idle streams: every frame is
  yielded once, with the detections host post-processing gives for that frame's records -- the same runner fed that
  frame alone (a stateless network: records depend on the frame alone) and meta(0).  pre_dets are refused."""
  from centertrack_b200.runner import StreamRunner
  from centertrack_b200.videos import Video, track_videos
  opt, model = _model('ddd')
  B, K = 2, 30
  runner = StreamRunner(model, B, H, W, K=K, precision='fp32', opt=opt, frame_sizes=[(120, 200)] * B,
                        max_frame_size=(240, 320), device_post_process=True, idle_streams=True)
  runner.warm()
  rng = np.random.RandomState(21)
  vids = [Video('v%d' % i, _frames(rng, [hw] * n), calib=np.array([[800. + i, 0, hw[1] / 2, 0], [0, 800., hw[0] / 2, 0],
                                                                   [0, 0, 1, 0]], np.float32))
          for i, (hw, n) in enumerate([((120, 200), 3), ((90, 140), 2), ((200, 150), 4)])]
  got = {(v, i): res for v, i, res in track_videos(runner, vids)}
  assert sorted(got) == sorted((v.id, i) for v in vids for i in range(len(v.frames)))
  for v in vids:
    for i, f in enumerate(v.frames):
      runner.step_frames([f, None], idle=[1], starts=[0], calibs={0: v.calib})
      rec = runner.fetch()
      want = _host(opt, rec, runner.layout, [runner.meta(0), None])[0]
      res = got[(v.id, i)]
      assert len(res) == len(want) > 0, (v.id, i)
      for j, (g, q) in enumerate(zip(res, want)):
        _same((v.id, i, j), g, q, rec[0, j], runner.layout, _trans(runner.meta(0)))
  with pytest.raises(ValueError, match='pre_dets'):
    list(track_videos(runner, [Video('p', _frames(rng, [(120, 200)]), pre_dets=[])]))
