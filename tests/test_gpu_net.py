"""-m gpu: whole hot path on the H100 vs the reference goldens (tests/golden, produced by the
unmodified reference) and vs the oracle.

Tolerances
  fp32 engine : |err| <= 1e-3 x max(1, |ref|max) per tensor  (north_star's fp32 bar; DCN bilinear
                sampling amplifies fp32 summation-order noise to ~3e-4, the same gap the reference's
                CPU path shows against the oracle)
  bf16 engine : checked against the oracle evaluated with the engine's own rounding points
                (DLA34Oracle(emulate_bf16=True): BN folded into bf16 weights, bf16 activation storage, fp32
                accumulation).  Where rounding noise has not been amplified yet the agreement is essentially
                exact (measured mean |err| / std: stem 7e-8, level0 1e-6, level1 3e-6, level2 2e-4 -- isolated
                bf16 rounding flips from fp32 summation order).  This randomly initialised, BN-calibrated
                network is chaotic: it multiplies ANY perturbation by ~5 per DLA level (level3 6e-3, level5
                3e-2, heads 6e-2..8e-2 against the emulation; 0.2..0.25 against the fp32 reference, and the
                CPU emulation deviates from fp32 by exactly as much), so deeper stages get stage-specific
                bounds and the fp32 comparison asserts correlation >= 0.9 and mean |err| <= 0.4 x std.
                Every launch of the shipped plans, individually, is checked per element against an fp64
                reference of its own operands in tests/test_gpu_plan_layers.py."""
import os

import numpy as np
import pytest
import torch

import ct_oracle as co
from centertrack_b200 import synthetic as wt
from helpers import make_model

pytestmark = pytest.mark.gpu
TOL = {'fp32': (1e-3, 2e-4), 'bf16x3': (1e-3, 2e-4)}
# mean |err| / std bounds of the bf16 engine against the bf16-emulating oracle, per stage (x ~3 of measured)
EMU_STAGE_TOL = {'stem': 2e-6, 'base.level0': 2e-5, 'base.level1': 1e-4, 'base.level2': 2e-3, 'base.level3': 3e-2,
                 'base.level4': 8e-2, 'base.level5': 1.2e-1}
EMU_TOL = 0.2          # DCN stages and heads


def _check(got, ref, precision, name):
  tol_max, tol_mean = TOL[precision]
  got = got.detach().float().cpu().numpy()
  scale = max(1.0, float(np.abs(ref).max()))
  err = np.abs(got - ref)
  assert err.max() <= tol_max * scale, '%s: max err %.3e (scale %.2f)' % (name, err.max(), scale)
  assert err.mean() <= tol_mean * scale, '%s: mean err %.3e' % (name, err.mean())


def _check_stat(got, ref, name, mean_tol, corr_min=None):
  got = got.detach().float().cpu().numpy().ravel()
  ref = np.asarray(ref, dtype=np.float32).ravel()
  std = max(float(ref.std()), 1e-6)
  err = np.abs(got - ref).mean()
  assert err <= mean_tol * std, '%s: mean err %.3e vs std %.3e' % (name, err, std)
  if corr_min is not None:
    c = np.corrcoef(got, ref)[0, 1]
    assert c >= corr_min, '%s: correlation %.3f' % (name, c)


@pytest.mark.parametrize('cfg', ['coco_tracking', 'mot', 'nuscenes_ddd', 'coco_pose'])
def test_bf16_network_matches_bf16_emulating_oracle_and_tracks_fp32_golden(cfg, golden_dir):
  g = np.load(os.path.join(golden_dir, 'net_%s_64x96.npz' % cfg))
  opt, model, sd = make_model(cfg)
  model = model.cuda()
  img, pre, hm = wt.synthetic_inputs(1, 64, 96)
  eng = model.engine_for(1, 64, 96, torch.device('cuda'), 'bf16')
  out = eng.forward(img.cuda(), pre.cuda(), hm.cuda())
  torch.cuda.synchronize()
  trace = {}
  emu = co.DLA34Oracle(sd, opt.heads, emulate_bf16=True).forward(img, pre, hm, trace=trace)
  for name in ['stem', 'base.level0', 'base.level1', 'base.level2', 'base.level3', 'base.level4', 'base.level5',
               'dla_up.ida_0.node_1', 'dla_up.ida_2.node_3', 'feat']:
    _check_stat(eng.stage(name), trace[name].numpy(), name, EMU_STAGE_TOL.get(name, EMU_TOL))
  for h in opt.heads:
    _check_stat(out[h], emu[h].numpy(), h, EMU_TOL)
    _check_stat(out[h], g['head.' + h], h + ' vs fp32 reference', 0.4, corr_min=0.9)


@pytest.mark.parametrize('precision', ['fp32', 'bf16x3'])
@pytest.mark.parametrize('cfg', ['coco_tracking', 'mot', 'nuscenes_ddd', 'coco_pose'])
def test_network_matches_reference_golden(cfg, precision, golden_dir):
  g = np.load(os.path.join(golden_dir, 'net_%s_64x96.npz' % cfg))
  opt, model, sd = make_model(cfg)
  model = model.cuda()
  img, pre, hm = wt.synthetic_inputs(1, 64, 96)
  eng = model.engine_for(1, 64, 96, torch.device('cuda'), precision)
  out = eng.forward(img.cuda(), pre.cuda(), hm.cuda())
  torch.cuda.synchronize()
  for h in opt.heads:
    _check(out[h], g['head.' + h], precision, h)
  for k in [x for x in g.files if x.startswith('stage.')]:
    name = k[len('stage.'):]
    _check(eng.stage('feat' if name == 'ida_up.node_2' else name), g[k], precision, name)
  # CUDA-graph replay must be bit-identical to the eager launches
  eager = {h: out[h].clone() for h in out}
  eng.in_img.copy_(img); eng.in_pre.copy_(pre); eng.in_hm.copy_(hm)
  rep = eng.replay()
  torch.cuda.synchronize()
  assert all(torch.equal(eager[h], rep[h]) for h in eager)


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_batched_frames_are_independent(precision):
  """B frames per launch (stream sharding unit): each frame's result equals its B=1 result."""
  opt, model, sd = make_model('coco_tracking')
  model = model.cuda()
  dev = torch.device('cuda')
  img, pre, hm = wt.synthetic_inputs(3, 64, 96, seed=5)
  e3 = model.engine_for(3, 64, 96, dev, precision)
  o3 = {k: v.clone() for k, v in e3.forward(img.cuda(), pre.cuda(), hm.cuda()).items()}
  e1 = model.engine_for(1, 64, 96, dev, precision)
  for b in range(3):
    o1 = e1.forward(img[b:b + 1].cuda().contiguous(), pre[b:b + 1].cuda().contiguous(), hm[b:b + 1].cuda().contiguous())
    for h in o1:
      assert torch.equal(o1[h][0], o3[h][b]), (h, b)


def test_first_frame_and_no_pre_hm_variants():
  """pre_hm=None (dla.py:310) and detection-only (no pre_img either) against the oracle."""
  opt, model, sd = make_model('coco_tracking')
  model = model.cuda()
  img, pre, hm = wt.synthetic_inputs(1, 64, 96, seed=8)
  orc = co.DLA34Oracle(sd, opt.heads)
  eng = model.engine_for(1, 64, 96, torch.device('cuda'), 'fp32')
  for p, h in ((pre, None), (None, None)):
    ref = orc.forward(img, p, h)
    out = eng.forward(img.cuda(), None if p is None else p.cuda(), None if h is None else h.cuda())
    for k in ref:
      _check(out[k], ref[k].numpy(), 'fp32', k)


def test_module_surface_and_dcn_module():
  """create_model(...)(x, pre_img, pre_hm)[-1] (raw, un-sigmoided dict) and the drop-in DCN module."""
  from centertrack_b200.dcn import DCN
  opt, model, sd = make_model('coco_tracking', extra=['--b200_precision', 'fp32'])
  model = model.cuda().eval()
  img, pre, hm = wt.synthetic_inputs(1, 64, 96)
  with torch.no_grad():
    out = model(img.cuda(), pre.cuda(), hm.cuda())
  assert isinstance(out, list) and len(out) == 1 and set(out[0]) == set(opt.heads)
  ref = co.DLA34Oracle(sd, opt.heads).forward(img, pre, hm)
  for k in ref:
    _check(out[0][k], ref[k].numpy(), 'fp32', k)
  opt.model_output_list = True
  lst = model(img.cuda(), pre.cuda(), hm.cuda())[0]
  assert isinstance(lst, list) and len(lst) == len(opt.heads)
  # DCN module: same parameter names as upstream, forward == oracle restatement
  d = DCN(64, 128).cuda()
  assert sorted(k for k, _ in d.named_parameters()) == ['bias', 'conv_offset_mask.bias', 'conv_offset_mask.weight', 'weight']
  g = torch.Generator().manual_seed(2)
  with torch.no_grad():
    d.conv_offset_mask.weight.copy_(torch.randn(27, 64, 3, 3, generator=g) * 0.02)
    d.conv_offset_mask.bias.copy_(torch.randn(27, generator=g))
    d.bias.copy_(torch.randn(128, generator=g))
  x = torch.randn(2, 64, 12, 20, generator=g)
  ref = co.dcn_v2_forward(x, d.weight.detach().cpu(), d.bias.detach().cpu(), d.conv_offset_mask.weight.detach().cpu(),
                          d.conv_offset_mask.bias.detach().cpu())
  d.precision = 'fp32'
  assert (d(x.cuda()).cpu() - ref).abs().max() < 1e-4
  d.precision = 'bf16'
  assert (d(x.cuda()).cpu() - ref).abs().max() < 5e-2
  with pytest.raises(RuntimeError, match='no CPU fallback'):
    d(x)


def test_checkpoint_roundtrip_and_module_prefix(tmp_path):
  from centertrack_b200.model import create_model, load_model, save_model
  opt, model, sd = make_model('coco_tracking')
  path = str(tmp_path / 'model.pth')
  torch.save({'epoch': 3, 'state_dict': {'module.' + k: v for k, v in sd.items()}}, path)   # DataParallel-style keys
  m2 = load_model(create_model(opt.arch, opt.heads, opt.head_conv, opt=opt), path, opt)
  assert all(torch.equal(m2.state_dict()[k], sd[k]) for k in sd)
  save_model(path, 4, m2)
  assert set(torch.load(path)['state_dict']) == set(sd)


@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_e2e_512_process_matches_reference_golden(precision, golden_dir):
  """Config 2: coco_tracking 512x512 through Detector.process (network + fused sigmoid + fused decode)
  against the reference's outputs: sampled head values, and the decoded detections."""
  from centertrack_b200.detector import Detector
  g = np.load(os.path.join(golden_dir, 'e2e_coco_tracking_512.npz'))
  opt, model, sd = make_model('coco_tracking', extra=['--b200_precision', precision])
  opt.load_model = ''
  det = Detector.__new__(Detector)
  det.opt, det.model = opt, model.cuda()
  img, pre, hm = wt.synthetic_inputs(1, 512, 512)
  output, dets = det.process(img.cuda(), pre.cuda(), hm.cuda(), None)
  pos = g['pos']
  for k in ('hm', 'reg', 'wh', 'tracking'):
    v = output[k].cpu().numpy().reshape(output[k].shape[1], -1)[:, pos]
    if precision == 'fp32':
      _check(torch.from_numpy(v), g['sample.' + k], precision, k)
    else:
      _check_stat(torch.from_numpy(v), g['sample.' + k], k, 0.5, corr_min=0.8)   # chaotic random-weight net, see module docstring
  ref_inds = (g['det.ys'] * 128 + g['det.xs']).astype(np.int64) + g['det.clses'].astype(np.int64) * 128 * 128
  got_inds = (dets['ys'] * 128 + dets['xs']).astype(np.int64) + dets['clses'].astype(np.int64) * 128 * 128
  if precision == 'fp32':
    # the top-100 scores of this random-weight model sit on the saturated end of the sigmoid (0.99..0.999995),
    # closer to each other than fp32 summation noise, so rank ORDER is not comparable; the SET of peaks and the
    # values decoded at common peaks are
    common = sorted(set(ref_inds[0].tolist()) & set(got_inds[0].tolist()))
    assert len(common) >= 90, len(common)
    ri = {v: i for i, v in enumerate(ref_inds[0].tolist())}
    gi = {v: i for i, v in enumerate(got_inds[0].tolist())}
    r_idx = np.array([ri[v] for v in common]); g_idx = np.array([gi[v] for v in common])
    assert np.abs(dets['scores'][0][g_idx] - g['det.scores'][0][r_idx]).max() < 1e-3
    # regression maps of this model reach |v| ~ 8: 1e-3 x scale
    assert np.abs(dets['bboxes'][0][g_idx] - g['det.bboxes'][0][r_idx]).max() < 1e-2
    assert np.abs(dets['tracking'][0][g_idx] - g['det.tracking'][0][r_idx]).max() < 1e-2
  else:
    # the top-100 scores of this model are saturated (0.99..0.999995) and closer together than the bf16 path's
    # deviation, so WHICH peaks make the top-100 is not comparable with the fp32 reference; what must hold is that
    # the fused decode of the bf16 maps is exactly the oracle's decode of those same maps
    host = {k: v.cpu().numpy() for k, v in output.items() if k != 'pre_inds' and v is not None}
    od = co.generic_decode(host, 100)
    assert np.array_equal((dets['ys'] * 128 + dets['xs']).astype(np.int64), od['_inds'])
    assert np.array_equal(dets['scores'], od['scores']) and np.array_equal(dets['bboxes'], od['bboxes'])


def test_detector_run_three_frames_matches_oracle_pipeline():
  """Detector.run() on a synthetic BGR video: pre_process -> process -> post_process -> tracker, fp32
  engine, against the same pipeline assembled from the oracle (network, decode, post-process, tracker)."""
  from centertrack_b200.detector import Detector
  opt, model, sd = make_model('coco_tracking', extra=['--b200_precision', 'fp32', '--track_thresh', '0.02',
                                                       '--new_thresh', '0.02', '--input_h', '128', '--input_w', '160'])
  opt.load_model = ''
  from centertrack_b200 import detector as D
  saved = D.create_model
  D.create_model = lambda *a, **k: model
  try:
    det = Detector(opt)
  finally:
    D.create_model = saved
  rng = np.random.RandomState(0)
  frames = [rng.randint(0, 255, (120, 160, 3)).astype(np.uint8) for _ in range(3)]
  orc = co.DLA34Oracle(sd, opt.heads)
  trk = co.TrackerOracle(opt.new_thresh)
  pre_img_t = None
  for fi, f in enumerate(frames):
    ret = det.run(f)
    assert set(ret) == {'results', 'tot', 'load', 'pre', 'net', 'dec', 'post', 'merge', 'track', 'display'}
    images, meta = det.pre_process(f, 1.0)
    if pre_img_t is None:
      pre_img_t = images
      trk.init_track([])
    phm, _ = co.render_pre_hm(trk.tracks, meta['trans_input'], meta['trans_output'], meta['inp_width'],
                              meta['inp_height'], meta['out_width'], meta['out_height'], opt.pre_thresh)
    out = co.sigmoid_output(orc.forward(images, pre_img_t, torch.from_numpy(phm)))
    dets = co.generic_decode({k: v for k, v in out.items()}, opt.K)
    dets = {k: v for k, v in dets.items() if not k.startswith('_')}
    res = co.generic_post_process(dets, [meta['c']], [meta['s']], meta['out_height'], meta['out_width'],
                                  opt.out_thresh, [meta['calib']])[0]
    res = [r for r in res if r['score'] > opt.out_thresh]
    ref = trk.step(res)
    pre_img_t = images
    got = ret['results']
    assert len(got) > 0
    # the two lists are matched by box (the random-weight network produces many near-equal scores, so list
    # order and greedy association are not stable under 1e-6 differences); a few near-threshold detections may differ
    assert abs(len(got) - len(ref)) <= max(2, len(ref) // 20)
    gb = np.asarray([r['bbox'] for r in got], np.float32)
    matched, same_id, miss = 0, 0, []
    for b in ref:
      d = np.abs(gb - np.asarray(b['bbox'], np.float32)[None]).max(1)
      # boxes are in image pixels (tens of px wide): 1e-3 x |wh| head tolerance -> a fraction of a pixel; several
      # classes can peak at the same cell and share one box, so the class takes part in the match
      cand = [j for j in np.nonzero(d < 0.5)[0]
              if got[j]['class'] == b['class'] and abs(got[j]['score'] - b['score']) < 1e-3]
      if cand:
        matched += 1
        same_id += got[cand[0]]['tracking_id'] == b['tracking_id']
      else:
        miss.append((float(d.min()), b['class'], float(b['score'])))
    assert matched >= 0.9 * len(ref), (fi, matched, len(ref), miss)
    assert same_id >= 0.9 * matched, (fi, same_id, matched)


@pytest.mark.parametrize('cfg,hw', [('mot', (544, 960)), ('nuscenes_ddd', (448, 800)), ('coco_pose', (512, 512))])
def test_full_size_configs_fp32_engine_vs_oracle(cfg, hw):
  """BASELINE configs 3-5 at their real resolutions (ragged 8x16 tiles at 136x240 / 112x200 outputs):
  fp32 engine vs the oracle, and the fused decode of the device's own maps vs the oracle decode."""
  from centertrack_b200.decode import generic_decode
  opt, model, sd = make_model(cfg)
  model = model.cuda()
  H, W = hw
  img, pre, hm = wt.synthetic_inputs(1, H, W, seed=11)
  ref = co.DLA34Oracle(sd, opt.heads).forward(img, pre, hm)
  eng = model.engine_for(1, H, W, torch.device('cuda'), 'fp32')
  eng.set_fused_activations(True)
  out = dict(eng.forward(img.cuda(), pre.cuda(), hm.cuda()))
  refs = co.sigmoid_output(ref)
  for k in refs:
    tol = 1e-3 if k != 'dep' else 2e-2          # dep = 1/(sigmoid+1e-6)-1 stretches small logit differences
    r = refs[k].numpy()
    err = np.abs(out[k].cpu().numpy() - r)
    assert err.max() <= tol * max(1.0, np.abs(r).max()), (k, err.max())
  dets = generic_decode(out, K=100)
  host = {k: v.cpu().numpy() for k, v in out.items()}
  od = co.generic_decode(host, 100)
  assert np.array_equal(dets.inds.cpu().numpy(), od['_inds'].astype(np.int32))
  for k in ('bboxes', 'tracking', 'scores'):
    assert np.array_equal(dets[k].cpu().numpy().reshape(od[k].shape), od[k]), k


@pytest.mark.parametrize('cfg,hw', [('mot', (544, 960)), ('nuscenes_ddd', (448, 800))])
def test_full_size_configs_bf16_engine_vs_emulating_oracle(cfg, hw):
  opt, model, sd = make_model(cfg)
  model = model.cuda()
  H, W = hw
  img, pre, hm = wt.synthetic_inputs(1, H, W, seed=12)
  emu = co.DLA34Oracle(sd, opt.heads, emulate_bf16=True).forward(img, pre, hm)
  eng = model.engine_for(1, H, W, torch.device('cuda'), 'bf16')
  out = eng.forward(img.cuda(), pre.cuda(), hm.cuda())
  for h in opt.heads:
    _check_stat(out[h], emu[h].numpy(), h, EMU_TOL)


# ---- what bf16 costs, as hard bounds against the REFERENCE's fp32 outputs (tests/golden/e2e_*.npz) ----------------
# Errors are |d| / max(1, |ref|max) per tensor (tests/parity.py).  The bounds are ~1.5x what was measured on an H100
# (coco_tracking, mot, coco_pose and the two b32 frames: head max 0.074-0.099, stage max 0.070-0.106, |d score| at
# reference peaks 0.011-0.082, |d bbox| 0.25-0.43 output px, |d tracking| 0.22-0.31 px, top-100 overlap 0.75-0.85) -- which is what the oracle predicts for this
# engine's rounding points (bf16 operands and activation storage, fp32 accumulate: 50 layers x ~3e-3 each on a network
# of unit perturbation gain -> ~3e-2 rms at the heads).  The fp32 engine measures 1.2e-5 on the same files.
BF16_BOUNDS = {'head_max': 0.15, 'stage_max': 0.15, 'bbox_max': 0.7, 'tracking_max': 0.55, 'topk_overlap': 0.65}
BF16_SCORE_MAX = {'coco_tracking': 0.05, 'mot': 0.15, 'coco_pose': 0.1}


def _dump(name, obj):
  out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'gpurun_out')
  if os.path.isdir(out):
    import json
    with open(os.path.join(out, 'parity_%s.json' % name), 'w') as f:
      json.dump(obj, f, indent=1, sort_keys=True)


def _full_size_parity(stem, precision, golden_dir, batch_engine=False):
  import parity as P
  from helpers import E2E_CASES
  from centertrack_b200.decode import generic_decode
  cfg, hw, batch, frame, seed = E2E_CASES[stem]
  g = np.load(os.path.join(golden_dir, stem + '.npz'))
  opt, model, sd = make_model(cfg)
  model = model.cuda()
  img, pre, hm = wt.synthetic_inputs(batch, hw[0], hw[1], seed=seed)
  if not batch_engine:
    img, pre, hm = img[frame:frame + 1], pre[frame:frame + 1], hm[frame:frame + 1]
    frame = 0
  B = img.shape[0]
  eng = model.engine_for(B, hw[0], hw[1], torch.device('cuda'), precision)
  eng.set_fused_activations(True)
  out = dict(eng.forward(img.cuda().contiguous(), pre.cuda().contiguous(), hm.cuda().contiguous()))
  dets = generic_decode(out, K=100)
  torch.cuda.synchronize()
  d = {k: dets[k].cpu().numpy() for k in ('clses', 'xs', 'ys')}
  m = P.summarize(P.head_metrics(out, g, frame), P.peak_metrics(out, d, g, frame), P.stage_metrics(eng.stage, g, frame))
  _dump('%s_%s%s' % (stem, precision, '_batched' if batch_engine else ''), m)
  return cfg, m


@pytest.mark.parametrize('precision', ['fp32', 'bf16x3'])
@pytest.mark.parametrize('stem', ['e2e_coco_tracking_512', 'e2e_mot_544x960', 'e2e_coco_pose_512'])
def test_fp32_and_bf16x3_engines_full_size_meet_1e3_against_reference(stem, precision, golden_dir):
  """north_star's bar (fp32 heat-maps / offsets within 1e-3 of the reference) at BASELINE configs 2, 3 and 5: met by
  the SIMT fp32 engine and by the TENSOR-CORE bf16x3 engine (bf16 hi/lo split operands, fp32 accumulate)."""
  cfg, m = _full_size_parity(stem, precision, golden_dir)
  assert max(m['head_max'].values()) <= 1e-3 and max(m['stage_max'].values()) <= 1e-3, m
  assert m['score_max'] <= 1e-3 and m['topk_overlap'] >= 0.97, m
  assert m['bbox_max'] <= 1e-2 and m['tracking_max'] <= 1e-2, m          # output-grid pixels


@pytest.mark.parametrize('stem', ['e2e_coco_tracking_512', 'e2e_mot_544x960', 'e2e_coco_pose_512'])
def test_bf16_engine_full_size_hard_bounds_against_reference(stem, golden_dir):
  """The benchmarked engine against the reference's fp32 outputs at BASELINE configs 2, 3 and 5: per-head and
  per-stage MAX error, errors at the reference's own top-100 peaks, and the overlap of the two top-100 sets."""
  cfg, m = _full_size_parity(stem, 'bf16', golden_dir)
  assert max(m['head_max'].values()) <= BF16_BOUNDS['head_max'], m
  assert max(m['stage_max'].values()) <= BF16_BOUNDS['stage_max'], m
  assert m['score_max'] <= BF16_SCORE_MAX[cfg], m
  assert m['bbox_max'] <= BF16_BOUNDS['bbox_max'] and m['tracking_max'] <= BF16_BOUNDS['tracking_max'], m
  assert m['topk_overlap'] >= BF16_BOUNDS['topk_overlap'], m


@pytest.mark.parametrize('stem', ['e2e_coco_tracking_512_b32f0', 'e2e_coco_tracking_512_b32f31'])
def test_bf16_engine_at_the_benchmarked_shape_b32(stem, golden_dir):
  """The exact shape bench.py runs (32 frames x 512x512 per launch: its own n_tile choices, grids and persistent-CTA
  striding): first and last frame of the batch against the reference run on that frame alone."""
  cfg, m = _full_size_parity(stem, 'bf16', golden_dir, batch_engine=True)
  assert max(m['head_max'].values()) <= BF16_BOUNDS['head_max'], m
  assert max(m['stage_max'].values()) <= BF16_BOUNDS['stage_max'], m
  assert m['score_max'] <= BF16_SCORE_MAX[cfg] and m['topk_overlap'] >= BF16_BOUNDS['topk_overlap'], m
  assert m['bbox_max'] <= BF16_BOUNDS['bbox_max'] and m['tracking_max'] <= BF16_BOUNDS['tracking_max'], m


def test_render_pre_hm_matches_draw_umich_gaussian():
  """ct_render_pre_hm (device max-splat) vs the oracle's draw_umich_gaussian, including gaussians clipped
  by the image border and overlapping blobs."""
  import ctypes as C
  from centertrack_b200 import _lib as L
  H, W = 96, 128
  rng = np.random.RandomState(0)
  boxes = []
  ref = np.zeros((2, 1, H, W), np.float32)
  for b in range(2):
    for _ in range(12):
      cx, cy, r = int(rng.randint(0, W)), int(rng.randint(0, H)), int(rng.randint(0, 20))
      boxes.append([b, cx, cy, r, 0])
      co.draw_umich_gaussian(ref[b, 0], (cx, cy), r)
  bt = torch.tensor(boxes, dtype=torch.float32, device='cuda')
  out = torch.full((2, 1, H, W), 7.0, device='cuda')
  L.check(L.lib().ct_render_pre_hm(L.ptr(bt), len(boxes), L.ptr(out), 2, H, W, L.stream_ptr()))
  assert np.abs(out.cpu().numpy() - ref).max() < 1e-6
  L.check(L.lib().ct_render_pre_hm(L.ptr(None), 0, L.ptr(out), 2, H, W, L.stream_ptr()))
  assert float(out.abs().max()) == 0.0


def test_stream_runner_host_pipeline_matches_device_path():
  """StreamRunner.step_host (pinned H2D on a copy stream, CUDA-graph replay, D2H of the packed records,
  one-step software pipeline) returns exactly what the eager device path computes, step after step."""
  from centertrack_b200.decode import generic_decode
  from centertrack_b200.runner import StreamRunner
  opt, model, sd = make_model('coco_tracking')
  model = model.cuda()
  B, H, W = 2, 64, 96
  runner = StreamRunner(model, B, H, W, K=20, precision='bf16', device='cuda')
  runner.warm()
  eng = model.engine_for(B, H, W, torch.device('cuda'), 'bf16')
  frames = [wt.synthetic_inputs(B, H, W, seed=40 + t) for t in range(4)]
  got = []
  for t, (img, _, hm) in enumerate(frames):
    prev = runner.step_host(img.pin_memory(), hm.pin_memory())
    if prev is not None:
      got.append(prev.copy())
  got.append(runner.fetch().copy())
  # reference: same sequence eagerly; pre_images = previous step's images (first step: the frame itself, detector.py:99-103)
  pre = None
  for t, (img, _, hm) in enumerate(frames):
    out = dict(eng.forward(img.cuda(), img.cuda() if pre is None else pre, hm.cuda()))
    rec = generic_decode(out, K=20).records.cpu().numpy()
    assert np.array_equal(rec, got[t]), t
    pre = img.cuda()


def test_bf16_network_is_deterministic_under_repetition():
  """Race detector for the warp-specialised pipelines (TMA producer / MMA issuers / epilogue): 40 replays of the
  512x512 step at B=4 must be bit-identical."""
  opt, model, sd = make_model('coco_tracking')
  model = model.cuda()
  B = 4
  img, pre, hm = wt.synthetic_inputs(B, 512, 512, seed=21)
  eng = model.engine_for(B, 512, 512, torch.device('cuda'), 'bf16')
  x, p, h = img.cuda(), pre.cuda(), hm.cuda()
  ref = {k: v.clone() for k, v in eng.forward(x, p, h).items()}
  for it in range(40):
    out = eng.forward(x, p, h)
    torch.cuda.synchronize()
    for k in ref:
      assert torch.equal(out[k], ref[k]), (it, k)
