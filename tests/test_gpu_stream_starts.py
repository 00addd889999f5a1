"""-m gpu: a StreamRunner stream starts a new video at any step (starts= / pre_dets=), the others unaffected: a started
video equals the same video played from t = 0 by a fresh runner, bit for bit, on every engine, with fp32 images and
raw frames; graph equals eager and nothing is recaptured; closed loop against the host pipeline with seeds
(reset_tracking + init_track(pre_dets)); payload head sets; the video scheduler; and ct_track_start directly."""
import copy

import numpy as np
import pytest
import torch

from centertrack_b200 import _lib as L
from centertrack_b200 import synthetic as wt
from helpers import make_model, make_opt

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')
EXACT = ('tracking_id', 'age', 'active', 'class')
H, W, B, K = 64, 96, 3, 30
SIZES = [(120, 200), (97, 131), (64, 96)]
STEPS = 8
# stream 1 starts a video at step 3 and again at step 4 (a one-frame video); streams 0 and 2 start at step 5
STARTS = {3: [1], 4: [1], 5: [0, 2]}


def _host_detector(opt):
  from centertrack_b200.dataset_info import get_dataset
  from centertrack_b200.detector import Detector
  from centertrack_b200.tracker import Tracker
  det = object.__new__(Detector)
  ds = get_dataset(opt.dataset)
  det.opt, det.cnt, det.pre_images, det.tracker = opt, 0, None, Tracker(opt)
  det.mean = np.array(ds.mean, dtype=np.float32).reshape(1, 1, 3)
  det.std = np.array(ds.std, dtype=np.float32).reshape(1, 1, 3)
  det.rest_focal_length = opt.test_focal_length if opt.test_focal_length >= 0 else ds.rest_focal_length
  det.flip_idx = ds.flip_idx
  return det


def _frame(h, w, seed):
  x = wt.synthetic_inputs(1, h, w, seed=seed, n_blobs=0)[0][0].permute(1, 2, 0).numpy()
  return np.ascontiguousarray(np.clip(x * 70.0 + 115.0, 0, 255).astype(np.uint8))


def _image(seed):
  return wt.synthetic_inputs(1, H, W, seed=seed)[0][0]


def _seeds(rng, n, h, w, classes=1):
  """pre_dets in source pixels: boxes of 8-30 px, scores on both sides of new_thresh, some without ct / tracking."""
  out = []
  for i in range(n):
    bw, bh = rng.uniform(8, 30, 2)
    x0, y0 = rng.uniform(0, w - bw), rng.uniform(0, h - bh)
    d = {'score': float(rng.uniform(0.05, 1.0)), 'class': int(rng.randint(1, classes + 1)),
         'bbox': [float(x0), float(y0), float(x0 + bw), float(y0 + bh)]}
    if i % 3 == 1:
      d['ct'] = [float(x0 + bw / 2 + 0.25), float(y0 + bh / 2 - 0.5)]
    d['tracking'] = [float(v) for v in rng.normal(0, 1, 2)]
    out.append(d)
  return out


def _model(cfg, extra=()):
  opt, model, _ = make_model(cfg, extra=['--track_thresh', '0.1', '--new_thresh', '0.1', '--pre_thresh', '0.1',
                                         '--input_h', str(H), '--input_w', str(W), '--max_age', '2'] + list(extra))
  if cfg == 'nuscenes_ddd':
    with torch.no_grad():            # boxes of a few pixels (the synthetic weights give ~0 wh)
      model.state_dict()['wh.2.bias'].fill_(3.0)
  return opt, model.cuda()


def _runner(model, opt, precision, frames, graph=True):
  from centertrack_b200.runner import StreamRunner
  r = StreamRunner(model, B, H, W, K=K, precision=precision, device='cuda', opt=opt, device_tracking=True,
                   use_graph=graph, frame_sizes=SIZES if frames else None)
  r.warm()
  return r


def _play(r, feed, frames_mode, graphs=None):
  """feed: per step (inputs, starts, pre_dets).  Pipelined like a user would run it: step t's outputs are read after
  step t+1 is submitted.  -> per step {rec, trk, cnt, pay} (host copies)."""
  out = []

  def grab(i, rec):
    d = dict(rec=rec, trk=r.h_trk[i].numpy().copy(), cnt=r.h_cnt[i].numpy().copy())
    d['pay'] = r.h_pay[i].numpy().copy() if r.tracker.payload is not None else None
    return d

  for k, (x, starts, pre) in enumerate(feed):
    if frames_mode:
      rec = r.step_frames(x, starts=starts, pre_dets=pre)
    else:
      rec = r.step_host(x, starts=starts, pre_dets=pre)
    if graphs is not None:
      assert [id(g) for g in r.graphs] == graphs, k          # a start step replays the captured graph
    if k:
      out.append(grab((k - 1) & 1, rec))
  rec = r.fetch()
  out.append(grab((len(feed) - 1) & 1, rec))
  return out


def _inputs(frames_mode, b, key):
  """Stream b's input for a frame identified by key."""
  if frames_mode:
    h, w = SIZES[b]
    return _frame(h, w, 1000 + 37 * key)
  return _image(1000 + 37 * key)


def _stack(frames_mode, xs):
  return xs if frames_mode else torch.stack(xs)


def _bits(a):
  return None if a is None else np.ascontiguousarray(a).view(np.uint32)


def _same(a, b, b_a, b_b, ctx):
  for k in ('rec', 'trk', 'cnt', 'pay'):
    if a[k] is None:
      continue
    assert np.array_equal(_bits(a[k][b_a]), _bits(b[k][b_b])), (ctx, k)


def _schedule(frames_mode, seeded):
  """The frame key each stream gets at each step (a new video starts at STARTS), the pre_dets of the starts, and the
  started videos as (stream, first step, length)."""
  keys = [[10 * b + t for b in range(B)] for t in range(STEPS)]
  feed, videos = [], []
  rng = np.random.RandomState(7)
  for t in range(STEPS):
    st = STARTS.get(t)
    pre = None
    if st and seeded and t in (4, 5):                        # seeds on stream 1's second start and on stream 0's
      b = st[0] if t == 4 else 0
      h, w = SIZES[b] if frames_mode else (H, W)
      pre = {b: _seeds(rng, 12, h, w)}
    feed.append((_stack(frames_mode, [_inputs(frames_mode, b, keys[t][b]) for b in range(B)]), st, pre))
  for t, st in sorted(STARTS.items()):
    for b in st:
      end = min([u for u, s in STARTS.items() if u > t and b in s] + [STEPS])
      videos.append((b, t, end - t))
  return keys, feed, videos


CASES = [('coco_tracking', p, m) for p in ('bf16', 'bf16x3', 'fp32') for m in ('images', 'frames')] + \
        [('nuscenes_ddd', 'bf16', 'images'), ('coco_pose', 'bf16', 'frames')]


@pytest.mark.parametrize('cfg,precision,mode', CASES, ids=['%s-%s-%s' % c for c in CASES])
def test_started_stream_equals_a_fresh_runner_bit_for_bit(cfg, precision, mode):
  """Each started video's records, track table, counts and payload equal those of a fresh runner playing the same video
  in the same stream from t = 0 (with the same pre_dets), and the streams that have not started equal a runner given
  the same frames without starts.  Payload head sets restart without seeds: the payload is cleared."""
  frames_mode = mode == 'frames'
  opt, model = _model(cfg)
  seeded = cfg == 'coco_tracking'
  keys, feed, videos = _schedule(frames_mode, seeded)
  r = _runner(model, opt, precision, frames_mode)
  graphs = [id(g) for g in r.graphs]
  got = _play(r, feed, frames_mode, graphs)
  del r
  plain = _runner(model, opt, precision, frames_mode)
  base = _play(plain, [(x, None, None) for x, _, _ in feed], frames_mode)
  del plain
  first = {b: min([t for t, s in STARTS.items() if b in s]) for b in range(B)}
  for t in range(STEPS):
    for b in range(B):
      if t < first[b]:
        _same(got[t], base[t], b, b, ('unstarted', t, b))
  assert sum(int(got[t]['cnt'][b, 0]) for t in range(STEPS) for b in range(B)) > 0
  for b, t0, n in videos:
    fresh = _runner(model, opt, precision, frames_mode)
    pre = feed[t0][2]
    pre = {b: pre[b]} if pre and b in pre else None
    vfeed = []
    for i in range(n):
      xs = [_inputs(frames_mode, q, keys[t0 + i][q]) for q in range(B)]
      vfeed.append((_stack(frames_mode, xs), [b] if (i == 0 and pre) else None, pre if i == 0 else None))
    want = _play(fresh, vfeed, frames_mode)
    del fresh
    for i in range(n):
      _same(got[t0 + i], want[i], b, b, ('video', b, t0, i))
    n_rows = int(got[t0]['cnt'][b, 0])                     # the start cleared the rows the previous video left
    assert not got[t0]['trk'][b, n_rows:].any(), (b, t0)
    if got[t0]['pay'] is not None:
      assert not got[t0]['pay'][b, n_rows:].any(), (b, t0)
  if seeded:                                               # the seeded starts keep their seeds' ids
    assert int(got[4]['cnt'][1, 1]) >= sum(1 for d in feed[4][2][1] if d['score'] > opt.new_thresh)


@pytest.mark.parametrize('precision,mode', [('bf16', 'frames'), ('fp32', 'images')])
def test_start_steps_graph_equals_eager(precision, mode):
  """The same schedule without CUDA graphs gives identical outputs; with graphs, no slot's graph is recaptured."""
  frames_mode = mode == 'frames'
  opt, model = _model('coco_tracking')
  _, feed, _ = _schedule(frames_mode, True)
  r = _runner(model, opt, precision, frames_mode)
  g = _play(r, feed, frames_mode, [id(x) for x in r.graphs])
  del r
  e = _runner(model, opt, precision, frames_mode, graph=False)
  assert e.graphs == [None] * 3
  ea = _play(e, feed, frames_mode)
  assert e.graphs == [None] * 3
  for t in range(STEPS):
    for k in ('rec', 'trk', 'cnt'):
      assert np.array_equal(_bits(g[t][k]), _bits(ea[t][k])), (t, k)


def _check_tracks(got, want, ctx):
  assert len(got) == len(want), (ctx, len(got), len(want))
  for a, w in zip(got, want):
    assert tuple(a[k] for k in EXACT) == tuple(int(w[k]) for k in EXACT), (ctx, a, w)
    for k in ('ct', 'tracking', 'bbox'):
      assert np.allclose(np.asarray(a[k], np.float64), np.asarray(w[k], np.float64), rtol=1e-4, atol=1e-3), (ctx, k)
    assert abs(a['score'] - float(w['score'])) < 1e-6


@pytest.mark.parametrize('cfg,extra', [
    ('coco_tracking', []), ('coco_tracking', ['--hungarian']),
    ('mot', ['--public_det', '--ltrb_amodal', '--track_thresh', '0.4', '--pre_thresh', '0.5'])],
    ids=['greedy', 'hungarian', 'mot17_public_det'])
def test_starts_with_seeds_close_the_loop_like_the_host_pipeline(cfg, extra):
  """fp32 engine, B = 3: every stream starts at t = 0, stream 1 again at step 2 and streams 0 and 2 at step 3, each
  with pre_dets.  Host reference per video: reset_tracking + init_track(pre_dets) + _get_additional_inputs +
  generic_post_process + Tracker.step.  Tracks match, and each start's device-rendered pre_hm is the host's."""
  from centertrack_b200.decode import generic_decode
  from centertrack_b200.image import get_affine_transform
  from centertrack_b200.post_process import generic_post_process
  from centertrack_b200.runner import StreamRunner
  from centertrack_b200.tracker import Tracker
  args = ['--input_h', str(H), '--input_w', str(W), '--max_age', '2'] + extra
  if cfg == 'coco_tracking':
    args = ['--track_thresh', '0.1', '--new_thresh', '0.1', '--pre_thresh', '0.1'] + args
  opt, model, _ = make_model(cfg, extra=args)
  model = model.cuda()
  runner = StreamRunner(model, B, H, W, K=K, precision='fp32', device='cuda', opt=opt, device_tracking=True)
  runner.warm()
  eng = model.engine_for(B, H, W, DEV, 'fp32')
  det = _host_detector(opt)
  hosts = [Tracker(opt) for _ in range(B)]
  c = np.array([W / 2., H / 2.], np.float32)
  s = max(H, W) * 1.0
  meta = {'inp_width': W, 'inp_height': H, 'out_width': W // 4, 'out_height': H // 4,
          'trans_input': get_affine_transform(c, s, 0, [W, H]), 'trans_output': get_affine_transform(c, s, 0, [W // 4, H // 4])}
  starts = {0: [0, 1, 2], 2: [1], 3: [0, 2]}
  rng = np.random.RandomState(11)
  pre = None
  total = seeded = 0
  for t in range(5):
    x = torch.stack([_image(300 + 10 * t + b) for b in range(B)]).cuda()
    st = starts.get(t, [])
    pre_dets = {b: _seeds(rng, 10, H, W, classes=min(3, opt.num_classes)) for b in st}
    for b in st:                                           # reset_tracking + init_track(pre_dets)
      hosts[b].reset()
      hosts[b].init_track(copy.deepcopy(pre_dets[b]))
      seeded += len(hosts[b].tracks)
    opt.device = torch.device('cpu')
    hms = [det._get_additional_inputs(hosts[b].tracks, meta, with_hm=True)[0] for b in range(B)]
    p = x.clone() if pre is None else pre.clone()
    for b in st:
      p[b] = x[b]
    out = dict(eng.forward(x, p, torch.cat(hms, 0).cuda()))
    views = {k: v.cpu().numpy() for k, v in generic_decode(out, K=K).items()}
    dets = []
    for b in range(B):
      one = {k: v[b:b + 1] for k, v in views.items()}
      r = generic_post_process(opt, one, [c], [s], H // 4, W // 4, opt.num_classes)[0]
      dets.append([q for q in r if q['score'] > opt.out_thresh])
    pub = None
    if opt.public_det:
      pub = []
      for b in range(B):
        pts = [np.asarray(d['ct'], np.float32) + rng.normal(0, 1.0, 2).astype(np.float32) for d in dets[b][::2][:6]]
        pts += [np.float32([rng.uniform(0, W), rng.uniform(0, H)]) for _ in range(2)]
        pub.append(np.stack(pts).astype(np.float32))
    runner.step_host(x.cpu(), public_dets=pub, starts=st, pre_dets=pre_dets)
    got = runner.fetch_results()
    for b in st:                                           # the first frame's prior heat-map, rendered from the seeds
      diff = np.abs(runner.hm[t % 3][b].cpu().numpy() - hms[b].numpy()[0])
      assert (diff > 1e-6).mean() < 2e-3, (t, b, float(diff.max()), float((diff > 1e-6).mean()))
      if hosts[b].tracks:
        assert float(hms[b].max()) > 0
    for b in range(B):
      want = hosts[b].step(dets[b], [{'ct': q} for q in pub[b]] if pub is not None else None)
      _check_tracks(got[b], want, (t, b))
      assert int(runner.tracker.counts[b, 1]) == hosts[b].id_count
      total += len(want)
    pre = x
  assert total > 0 and seeded > 0


def test_scheduler_yields_every_frame_once_with_a_fresh_runners_tracks():
  """track_videos: 7 videos of 1, 2, 3, 4, 5, 6 and 8 frames, two source sizes across B = 3 streams (frames mode, bf16),
  one video seeded.  Every (video, frame) is yielded once, and its tracks equal those of the video played alone from
  t = 0 (reset_tracking) in a runner whose streams have its size."""
  from centertrack_b200.runner import StreamRunner
  from centertrack_b200.videos import Video, track_videos
  opt, model = _model('coco_tracking')
  A, Bs = (120, 200), (97, 131)
  lengths = [1, 2, 3, 4, 5, 6, 8]
  vsize = [A, Bs, Bs, A, A, Bs, A]
  rng = np.random.RandomState(3)
  vids = []
  for v, (n, (h, w)) in enumerate(zip(lengths, vsize)):
    frames = [_frame(h, w, 5000 + 100 * v + i) for i in range(n)]
    vids.append(Video('v%d' % v, frames, pre_dets=_seeds(rng, 8, h, w) if v == 4 else None))
  kw = dict(K=K, precision='bf16', device='cuda', opt=opt, device_tracking=True)
  runner = StreamRunner(model, B, H, W, frame_sizes=[A, Bs, A], **kw)
  runner.warm()
  out = list(track_videos(runner, vids))
  assert sorted((v, i) for v, i, _ in out) == sorted(('v%d' % v, i) for v, n in enumerate(lengths) for i in range(n))
  got = {(v, i): res for v, i, res in out}
  del runner
  refs = {}
  for size in (A, Bs):
    refs[size] = StreamRunner(model, B, H, W, frame_sizes=[size] * B, **kw)
    refs[size].warm()
  n_tracks = 0
  for v, video in enumerate(vids):
    ref = refs[vsize[v]]
    ref.reset_tracking()
    for i, f in enumerate(video.frames):
      pre = {0: video.pre_dets} if (i == 0 and video.pre_dets is not None) else None
      ref.step_frames([f] * B, starts=[0] if pre else None, pre_dets=pre)
      want = ref.fetch_results()[0]
      have = got[('v%d' % v, i)]
      assert len(have) == len(want), (v, i)
      for a, w in zip(have, want):
        for k in a:
          assert np.array_equal(np.asarray(a[k]), np.asarray(w[k])), (v, i, k)
      n_tracks += len(want)
  assert n_tracks > 0


def test_track_start_directly_on_random_tables():
  """ct_track_start on random tables (payload head set, B = 5, T = 40): the started streams hold exactly the seed rows,
  counts (n, n) and a zeroed payload; every byte of the other streams' tables, counts, payloads and boxes is unchanged;
  and ct_render_tracks of the written boxes is _get_additional_inputs on the host tracker after init_track."""
  from centertrack_b200.device_tracker import DeviceTracker, seed_rows
  from centertrack_b200.image import get_affine_transform
  from centertrack_b200.tracker import Tracker
  inp_h, inp_w = 128, 160
  opt = make_opt('coco_pose', ['--new_thresh', '0.3', '--pre_thresh', '0.25', '--input_h', str(inp_h), '--input_w',
                               str(inp_w)])
  Bn, Kn, T = 5, 20, 40
  layout = {'tracking': (9, 2), 'hps': (11, 34)}
  img_hw = [(240, 320), (300, 260), (128, 160), (500, 700), (90, 120)]
  centers = [np.array([w / 2., h / 2.], np.float32) for h, w in img_hw]
  scales = [max(h, w) * 1.0 for h, w in img_hw]
  trk = DeviceTracker(opt, Bn, Kn, 45, layout, inp_h, inp_w, DEV, centers=centers, scales=scales, max_tracks=T)
  assert trk.payload is not None and trk.T == T
  g = torch.Generator(device='cuda').manual_seed(1)
  for t in (trk.tracks, trk.boxes, trk.payload):
    t.copy_(torch.rand(t.shape, device=DEV, generator=g) * 100)
  trk.counts.copy_(torch.randint(0, T, trk.counts.shape, device=DEV, generator=g, dtype=torch.int32))
  before = [t.clone() for t in (trk.tracks, trk.counts, trk.payload, trk.boxes)]
  rng = np.random.RandomState(2)
  items = {3: _seeds(rng, 30, *img_hw[3], classes=1), 0: [], 1: _seeds(rng, 6, *img_hw[1], classes=1)}
  streams = [3, 0, 1]
  rows = [seed_rows(items[b], opt.new_thresh) for b in streams]
  assert len(rows[0]) > 5
  lst = torch.tensor([[b, len(r)] for b, r in zip(streams, rows)], dtype=torch.int32, device=DEV)
  seeds = torch.from_numpy(np.concatenate(rows)).to(DEV)
  trk.start_device(lst, len(streams), seeds)
  torch.cuda.synchronize()
  after = [t.clone() for t in (trk.tracks, trk.counts, trk.payload, trk.boxes)]
  for b in range(Bn):
    if b in streams:
      r = rows[streams.index(b)]
      n = len(r)
      assert np.array_equal(after[0][b, :n].cpu().numpy().view(np.uint32), r.view(np.uint32))
      assert not after[0][b, n:].any()
      assert after[1][b].tolist() == [n, n]
      assert not after[2][b].any()
    else:
      for x, y in zip(before, after):
        assert torch.equal(x[b].view(torch.int32) if x.dtype == torch.float32 else x[b],
                           y[b].view(torch.int32) if y.dtype == torch.float32 else y[b]), b
  # the render: the other streams' random boxes are switched off so that they cannot splat into the started streams
  for b in range(Bn):
    if b not in streams:
      trk.boxes[b, :, 3] = -1.0
  pre_hm = torch.full((Bn, 1, inp_h, inp_w), 5.0, device=DEV)
  trk.render(pre_hm)
  torch.cuda.synchronize()
  det = _host_detector(opt)
  opt.device = torch.device('cpu')
  for b in streams:
    host = Tracker(opt)
    host.init_track(copy.deepcopy(items[b]))
    h, w = img_hw[b]
    meta = {'inp_width': inp_w, 'inp_height': inp_h, 'out_width': inp_w // 4, 'out_height': inp_h // 4,
            'trans_input': get_affine_transform(centers[b], scales[b], 0, [inp_w, inp_h]),
            'trans_output': get_affine_transform(centers[b], scales[b], 0, [inp_w // 4, inp_h // 4])}
    hm, _ = det._get_additional_inputs(host.tracks, meta, with_hm=True)
    diff = np.abs(pre_hm[b].cpu().numpy() - hm.numpy()[0])
    assert (diff > 1e-6).mean() < 2e-3, (b, float(diff.max()), float((diff > 1e-6).mean()))
    assert (float(hm.max()) > 0) == bool(host.tracks)
  # DeviceTracker.start: the dict-level call does the same on a 2-D head set, and refuses seeds with a payload
  with pytest.raises(ValueError, match='payload'):
    trk.start([3], {3: items[3]})
  trk.start([2, 4])
  torch.cuda.synchronize()
  assert trk.counts[2].tolist() == [0, 0] and trk.counts[4].tolist() == [0, 0] and not trk.payload[2].any()
