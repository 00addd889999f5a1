"""The fused decode (csrc/decode.cu) on every path its one launch can take, each checked against the oracle
(ct_oracle.generic_decode, pinned to the reference by decode_cases.npz).

ct_decode picks among these paths, by shape and by data:
  plane source   bulk: each class plane is staged in shared memory by cp.async.bulk copies (H*W*4 <= PLANE_CAP and
                 W % 4 == 0, unless CTB_DEC_BULK=0); register: the plane streams through registers
  per-plane      list: radix select over the compacted kept positive peaks (16-byte loads, K <= npk <= PEAK_CAP);
  select         full: radix select over all H*W keys (fewer than K peaks, a list that overflows, W % 4 != 0, an hm
                 base that is not 16-byte aligned)
  merge keys     smem: the C*K merge keys staged in shared memory (C*K <= key_cap); l2: read from L2 on every pass
  pose           hm_hp given: joint planes sorted per joint, keypoint refinement, a pose scratch that can set the
                 shared-memory size

Bar: top-K indices and every gathered value bit-exact, the refined keypoints and kps_score included (the kernel
rounds them with __f*_rn in the oracle's order of operations).  Two tests need no GPU: the path table covers every
cell, and ct_decode's argument checks return before any CUDA call.
"""
import collections
import ctypes as C
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

import ct_oracle as co
from centertrack_b200 import _lib as L

gpu = pytest.mark.gpu

# ---------------------------------------------------------------------------------------------------------------------
# The host dispatch of ct_decode, restated from decode.cu (constants: lines 20-22; dispatch: lines 515-523; the merge
# keys' location is then decided at line 340, the per-plane select by the data at line 267).  This is documentation of
# the path each case below is meant to reach; the GPU tests check results, not this helper.
# ---------------------------------------------------------------------------------------------------------------------
MAXK, PEAK_CAP, PLANE_CAP = 512, 4096, 65536
SMEM_LIMIT = 200 * 1024


def decode_path(C_, H, W, K, J=0):
  """-> (plane source 'bulk' | 'register', merge keys 'smem' | 'l2'), or None where the pose scratch is refused."""
  bulk = H * W * 4 <= PLANE_CAP and W % 4 == 0
  smem = max(PEAK_CAP * 8 + (PLANE_CAP if bulk else 0), (7 * K + 4 * J * K) * 4)
  if smem > SMEM_LIMIT:
    return None
  return ('bulk' if bulk else 'register', 'smem' if C_ * K <= smem // 8 else 'l2')


HEAD_CH = {'reg': 2, 'wh': 2, 'ltrb': 4, 'tracking': 2, 'dep': 1, 'rot': 8, 'dim': 3, 'amodel_offset': 2,
           'nuscenes_att': 8, 'velocity': 3, 'ltrb_amodal': 4, 'hps': 34, 'hp_offset': 2}
COCO = ('reg', 'wh', 'tracking')
NUSCENES = ('reg', 'wh', 'tracking', 'dep', 'rot', 'dim', 'amodel_offset', 'nuscenes_att', 'velocity')
POSE = ('reg', 'wh', 'hps', 'hp_offset')
POSE_REG = ('reg', 'wh', 'hps')                   # no hp_offset: the refinement offsets joint peaks by reg
ALL_HEADS = ('reg', 'wh', 'ltrb', 'tracking', 'dep', 'rot', 'dim', 'amodel_offset', 'nuscenes_att', 'velocity',
             'ltrb_amodal', 'hps')                # CT_DECODE_MAX_HEADS of them
BOUNDARY = lambda K: (K - 1, K, PEAK_CAP, PEAK_CAP + 1)
PLANE_KINDS = ('lattice', 'lattice_q', 'flat')     # see _peak_plane
FEW = (20, 45, 7)                                  # kept peaks of class planes 0, 1, 2 of a 'few' case
FILLER = 300                                       # kept peaks of a 'boundary' case's filler planes

# data: None = sigmoid-noise heat-maps, whose every plane takes the per-plane select `select`; otherwise the class
# planes are built with known kept-peak counts (_plane_spec), so that the data-chosen select is chosen on purpose:
#   boundary: image b features one class plane with npk in BOUNDARY(K) x PLANE_KINDS (12 images), above low filler
#             planes, so the image's top K is that plane's own top K;
#   few:      fewer positive peaks than K in every plane and in all of them together, so the merge ranks zeros too.
Case = collections.namedtuple('Case', 'name B C H W K J heads data path select')
CASES = [
    Case('coco_136x240_k100', 2, 80, 136, 240, 100, 0, COCO, None, ('register', 'l2'), 'list'),
    Case('coco_136x240_k256', 2, 80, 136, 240, 256, 0, COCO, None, ('register', 'l2'), 'list'),
    Case('coco_128_k200', 1, 80, 128, 128, 200, 0, COCO, None, ('bulk', 'l2'), 'list'),
    Case('nuscenes_112x200_k450', 1, 10, 112, 200, 450, 0, NUSCENES, None, ('register', 'l2'), 'list'),
    Case('k512_128', 1, 20, 128, 128, 512, 0, COCO, None, ('bulk', 'smem'), 'list'),
    Case('k512_136x240', 1, 20, 136, 240, 512, 0, COCO, None, ('register', 'l2'), 'list'),
    Case('pose_128_k512', 1, 1, 128, 128, 512, 17, POSE, None, ('bulk', 'smem'), 'list'),
    Case('pose_128_k512_reg', 1, 1, 128, 128, 512, 17, POSE_REG, None, ('bulk', 'smem'), 'list'),
    Case('pose_136x240_k512', 1, 1, 136, 240, 512, 17, POSE, None, ('register', 'smem'), 'list'),
    Case('pose_136x240_k512_reg', 1, 1, 136, 240, 512, 17, POSE_REG, None, ('register', 'smem'), 'list'),
    Case('pose80_128_k256', 1, 80, 128, 128, 256, 17, POSE, None, ('bulk', 'l2'), 'list'),
    Case('pose80_136x240_k256', 1, 80, 136, 240, 256, 17, POSE, None, ('register', 'l2'), 'list'),
    Case('k_eq_hw_16x32', 2, 3, 16, 32, 512, 0, COCO, None, ('bulk', 'smem'), 'full'),
    Case('h1_w128', 2, 4, 1, 128, 32, 0, COCO, None, ('bulk', 'smem'), 'list'),   # bulk copies of 1, 2, 3 and 3
    Case('h2_w128', 2, 4, 2, 128, 32, 0, COCO, None, ('bulk', 'smem'), 'list'),   # chunks, and the list select
    Case('h3_w128', 2, 4, 3, 128, 32, 0, COCO, None, ('bulk', 'smem'), 'list'),   # reads only what they staged
    Case('h5_w128', 2, 4, 5, 128, 32, 0, COCO, None, ('bulk', 'smem'), 'list'),
    Case('ragged_64x132', 2, 8, 64, 132, 100, 0, COCO, None, ('bulk', 'smem'), 'list'),
    Case('ragged_128x132', 1, 8, 128, 132, 100, 0, COCO, None, ('register', 'smem'), 'list'),
    Case('w6', 2, 6, 40, 6, 50, 0, COCO, None, ('register', 'smem'), 'full'),
    Case('w30', 2, 6, 40, 30, 50, 0, COCO, None, ('register', 'smem'), 'full'),
    Case('all_heads', 2, 3, 64, 96, 100, 0, ALL_HEADS, None, ('bulk', 'smem'), 'list'),
    Case('all_heads_pose', 2, 3, 64, 96, 100, 17, ALL_HEADS, None, ('bulk', 'smem'), 'list'),
    Case('boundary_128', 12, 4, 128, 128, 100, 0, COCO, 'boundary', ('bulk', 'smem'), None),
    Case('boundary_128_l2', 12, 64, 128, 128, 200, 0, COCO, 'boundary', ('bulk', 'l2'), None),
    Case('boundary_136x240', 12, 4, 136, 240, 100, 0, COCO, 'boundary', ('register', 'smem'), None),
    Case('boundary_136x240_l2', 12, 48, 136, 240, 100, 0, COCO, 'boundary', ('register', 'l2'), None),
    Case('few_peaks_128', 2, 3, 128, 128, 100, 0, COCO, 'few', ('bulk', 'smem'), None),
    Case('few_peaks_136x240', 2, 3, 136, 240, 100, 0, COCO, 'few', ('register', 'smem'), None),
]
CASE = {c.name: c for c in CASES}
BENCH = Case('bench', 32, 80, 128, 128, 100, 0, COCO, None, ('bulk', 'smem'), 'list')
GRAPH = Case('graph', 2, 80, 136, 240, 100, 0, COCO, None, ('register', 'l2'), 'list')
REUSE = Case('reuse', 3, 80, 128, 128, 100, 0, COCO, None, ('bulk', 'smem'), 'list')
RECORDS_ENV = 'CTB_TEST_DECODE_RECORDS'            # directory test_decode_case writes its records to, when set


def _featured(case, b):
  """Class of the boundary plane image b of a 'boundary' case features (spread from the first class to the last)."""
  return b * (case.C - 1) // (case.B - 1)


def _plane_spec(case):
  """[B][C] (kept-peak count, kind) of the class planes of a data-chosen case."""
  if case.data == 'few':
    return [[(FEW[c % 3], PLANE_KINDS[c % 3]) for c in range(case.C)] for _ in range(case.B)]
  combos = [(n, kind) for n in BOUNDARY(case.K) for kind in PLANE_KINDS]
  assert case.B == len(combos), case.name
  spec = [[(FILLER, 'filler')] * case.C for _ in range(case.B)]
  for b, nk in enumerate(combos):
    spec[b][_featured(case, b)] = nk
  return spec


def test_path_table_covers_every_cell():
  """Every (plane source x merge-key location) cell with and without pose has a case, each case is on the path the
  table says, each plane source has cases whose planes all take the list select and cases whose planes all take the
  full-plane one, and on each cell without pose a boundary case puts npk = K - 1, K, PEAK_CAP and PEAK_CAP + 1."""
  cells = set()
  for c in CASES + [BENCH, GRAPH, REUSE]:
    assert decode_path(c.C, c.H, c.W, c.K, c.J) == c.path, c.name
    assert c.K <= min(MAXK, c.H * c.W), c.name
    cells.add(c.path + (c.J > 0,))
  assert cells == {(p, k, pose) for p in ('bulk', 'register') for k in ('smem', 'l2') for pose in (False, True)}
  assert {(c.path[0], c.select) for c in CASES if c.data is None} == \
      {(p, s) for p in ('bulk', 'register') for s in ('list', 'full')}
  boundary = {c.path for c in CASES if c.data == 'boundary'}
  assert boundary == {(p, k) for p in ('bulk', 'register') for k in ('smem', 'l2')}
  assert {c.path[0] for c in CASES if c.data == 'few'} == {'bulk', 'register'}
  assert any(c.J and c.heads == ALL_HEADS for c in CASES) and any(not c.J and c.heads == ALL_HEADS for c in CASES)
  assert len(ALL_HEADS) == L.CT_DECODE_MAX_HEADS


def _kept(planes):
  return (co.nms_keep(planes) & (planes > 0)).sum((2, 3))


@pytest.mark.parametrize('name', [c.name for c in CASES] + [BENCH.name])
def test_case_planes_take_the_intended_select(name):
  """The per-plane select is chosen by the data (decode.cu:174,267: list when 16-byte loads can read the plane and
  K <= npk <= PEAK_CAP, else full), so it is asserted here on each case's inputs, with the oracle's NMS:
  sigmoid-noise cases, class and joint planes alike, all take the select the table names; data-chosen planes keep
  exactly the npk they were built with; in a boundary case every image's top K holds min(npk, K) records of the
  featured plane; in a few case every positive peak is a record and zeros fill the rest."""
  case = CASE.get(name, BENCH)
  inp = _inputs(case)
  if case.data is None:
    planes = np.concatenate([inp['hm'], inp['hm_hp']], 1) if case.J else inp['hm']
    kept = _kept(planes)
    listed = (case.W % 4 == 0) & (kept >= case.K) & (kept <= PEAK_CAP)
    assert (listed if case.select == 'list' else ~listed).all(), (kept.min(), kept.max())
    return
  spec = _plane_spec(case)
  _same(_kept(inp['hm']), np.array([[n for n, _ in row] for row in spec]), name + ' kept peaks')
  ref = co.generic_decode(inp, case.K)
  if case.data == 'boundary':
    for b, row in enumerate(spec):
      f = _featured(case, b)
      assert (ref['clses'][b] == f).sum() == min(row[f][0], case.K), (name, b, row[f])
  else:
    _same((ref['scores'] > 0).sum(1), np.full(case.B, sum(FEW)), name + ' positive records')


# ---------------------------------------------------------------------------------------------------------------------
# argument checks (no GPU)
# ---------------------------------------------------------------------------------------------------------------------
def _desc(**fields):
  """A descriptor that passes every check, with non-null dummy pointers (nothing may dereference them), then `fields`."""
  d = L.DecodeDesc()
  d.B, d.C, d.H, d.W, d.K = 1, 1, 64, 64, 100
  d.hm = d.records = d.workspace = 16
  d.n_heads, d.rec_floats, d.rec_hps, d.rec_kps_score = 0, L.CT_REC_HEADS, -1, -1
  for k, v in fields.items():
    setattr(d, k, v)
  return d


@pytest.mark.parametrize('fields, status, msg', [
    (dict(K=0), L.CT_ERR_INVALID, b'K out of range'),
    (dict(K=513), L.CT_ERR_INVALID, b'K out of range'),
    (dict(H=4, W=4, K=17), L.CT_ERR_INVALID, b'K out of range'),
    (dict(n_heads=13), L.CT_ERR_INVALID, b'too many heads'),
    (dict(hm_hp=16, J=0), L.CT_ERR_INVALID, b'hm_hp without J'),
    (dict(rec_floats=L.CT_REC_HEADS - 1), L.CT_ERR_INVALID, b'record too small'),
    (dict(C=32768, H=256, W=256), L.CT_ERR_INVALID, b'C*H*W must stay below 2^31'),
    (dict(hm_hp=16, J=24, K=512), L.CT_ERR_UNSUPPORTED, b'shared-memory scratch of the pose refinement'),
], ids=['K0', 'K513', 'K_gt_HW', 'heads13', 'hm_hp_J0', 'rec_floats8', 'CHW_2e31', 'pose_scratch_J24_K512'])
def test_decode_argument_checks_return_before_any_cuda_call(built_lib, fields, status, msg):
  lib = L.lib()
  launches = lib.ct_launch_count()
  assert lib.ct_decode(C.byref(_desc(**fields)), None) == status
  assert msg in lib.ct_last_error(), lib.ct_last_error()
  assert lib.ct_launch_count() == launches


# ---------------------------------------------------------------------------------------------------------------------
# inputs, runs and the comparison
# ---------------------------------------------------------------------------------------------------------------------
def _sigmoid_noise(rng, shape, bias):
  return (1. / (1. + np.exp(-(2 * rng.randn(*shape) - bias)))).astype(np.float32)


def _peak_plane(rng, H, W, n, kind):
  """An H x W plane whose 3x3 max-equals NMS keeps exactly n positive peaks; the rest of it is exact zeros, which are
  never kept.
    lattice:   strict maxima in [0.3, 1) at the first n (even y, even x) points in raster order, each over its own
               2 x 2 block of lower positive background (every background pixel then has a higher lattice neighbour).
               A full lattice holds ceil(H/2) * ceil(W/2) peaks; e more are made by raising row 0's first 2e + 1 pixels
               to one ridge value (equal neighbours are all kept), so that 128 x 128 gets PEAK_CAP + 1 distinct-valued
               peaks as well.
    lattice_q: the same with peaks quantised to 1/20 in [0.3, 0.95] (many equal scores in one plane).
    flat:      the first n pixels in raster order at 0.95 (a plateau keeps every pixel).
    filler:    a lattice with peaks quantised to 0.1 .. 0.25, below every other kind's peaks (equal scores across
               classes), over a background of 0.05."""
  p = np.zeros((H, W), np.float32)
  if kind == 'flat':
    p.reshape(-1)[:n] = 0.95
    return p
  lw = (W + 1) // 2
  lattice = min(n, (H + 1) // 2 * lw)
  ridge = n - lattice
  assert 2 * ridge < W, (H, W, n)
  ys, xs = 2 * (np.arange(lattice) // lw), 2 * (np.arange(lattice) % lw)
  for dy, dx in ((0, 1), (1, 0), (1, 1)):
    yy, xx = ys + dy, xs + dx
    ok = (yy < H) & (xx < W)
    m = int(ok.sum())
    p[yy[ok], xx[ok]] = {'lattice': lambda: rng.uniform(0.02, 0.25, m), 'lattice_q': lambda: rng.randint(1, 6, m) / 20.,
                         'filler': lambda: 0.05}[kind]()
  p[ys, xs] = {'lattice': lambda: rng.uniform(0.3, 1.0, lattice), 'lattice_q': lambda: rng.randint(6, 20, lattice) / 20.,
               'filler': lambda: rng.randint(2, 6, lattice) / 20.}[kind]()
  if ridge:
    p[0, :2 * ridge + 1] = p[ys, xs].max()
  return p


def _inputs(case, seed=None):
  rng = np.random.RandomState(zlib.crc32(case.name.encode()) if seed is None else seed)
  B, C_, H, W = case.B, case.C, case.H, case.W
  if case.data is None:
    hm = _sigmoid_noise(rng, (B, C_, H, W), 4.6)
  else:
    hm = np.stack([np.stack([_peak_plane(rng, H, W, n, kind) for n, kind in row]) for row in _plane_spec(case)])
  out = {'hm': hm}
  for name in case.heads:
    shape = (B, HEAD_CH[name], H, W)
    if name in ('reg', 'hp_offset'):
      out[name] = rng.rand(*shape).astype(np.float32)
    else:                                       # wh: negative widths are clamped to 0 by the decode
      out[name] = (rng.randn(*shape) * (6 if name in ('wh', 'hps') else 8 if 'ltrb' in name else 3)).astype(np.float32)
  if case.J:
    out['hm_hp'] = _sigmoid_noise(rng, (B, case.J, H, W), 3.0)
  return out


def _gpu_records(inp, K, **kw):
  from centertrack_b200.decode import generic_decode
  res = generic_decode({k: torch.from_numpy(v).cuda() for k, v in inp.items()}, K=K, **kw)
  return res.records.cpu().numpy(), res.layout


def _same(got, want, what):
  """Bit-identical: float32 arrays are compared as their bit patterns (so -0.0 is not 0.0), others by value."""
  got = np.asarray(got).reshape(want.shape)
  if want.dtype.kind == 'f':
    assert got.dtype == want.dtype == np.float32, (what, got.dtype, want.dtype)
    bad = got.view(np.uint32) != want.view(np.uint32)
  else:
    bad = got != want
  if bad.any():
    i = tuple(int(v) for v in np.argwhere(bad)[0])
    rel = np.abs(got.astype(np.float64) - want).max() / max(1.0, np.abs(want).max())
    raise AssertionError('%s: %d of %d differ, first at %s: got %r, want %r (max rel diff %.3g)'
                         % (what, int(bad.sum()), bad.size, i, got[i], want[i], rel))


def _check(rec, layout, inp, K, tag=''):
  """Records [B,K,F] of one launch against the oracle: the reference's dict bit-exact, key set included, and the raw
  record slices of reg, wh (clamped), ltrb, ltrb_amodal and hps (plus the center, before the refinement), which that
  dict does not expose, bit-exact as well."""
  from centertrack_b200.decode import views_from_records
  ref = co.generic_decode(inp, K)
  got = views_from_records(torch.from_numpy(rec), layout)
  inds = ref['_inds']
  _same(got.inds.numpy(), inds.astype(np.int32), tag + ' top-K indices')
  assert set(got) == set(ref) - {'_inds'}, (tag, sorted(got), sorted(ref))
  for k, r in ref.items():
    if not k.startswith('_'):
      _same(got[k].numpy(), r, '%s %s' % (tag, k))
  for name in ('reg', 'wh', 'ltrb', 'ltrb_amodal', 'hps'):
    if name in layout:
      o, w = layout[name]
      want = co.gather_feat(inp[name], inds)
      if name == 'wh':
        want = np.where(want < 0, np.float32(0), want)
      if name == 'hps':
        want = want.copy()
        want[..., ::2] += ref['xs'][..., None]
        want[..., 1::2] += ref['ys'][..., None]
      _same(rec[:, :, o:o + w], want, '%s %s record slice' % (tag, name))


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the case table
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('name', [c.name for c in CASES])
def test_decode_case(name):
  """One case of the table against the oracle (test_case_planes_take_the_intended_select checks the same inputs reach
  the per-plane select the table intends)."""
  case = CASE[name]
  inp = _inputs(case)
  rec, layout = _gpu_records(inp, case.K)
  if os.environ.get(RECORDS_ENV):
    np.save(os.path.join(os.environ[RECORDS_ENV], name + '.npy'), rec)
  if case.heads == ALL_HEADS:
    assert len(set(layout) - {'hps_refined', 'kps_score'}) == L.CT_DECODE_MAX_HEADS
  _check(rec, layout, inp, case.K, name)


@gpu
def test_register_streaming_gives_the_bulk_records(tmp_path):
  """CTB_DEC_BULK=0 (read once per process) streams every plane through registers: the bulk-eligible cases run again in
  a process of their own, pass against the oracle there, and write records bit-identical to the bulk-staged ones."""
  if os.environ.get('CTB_DEC_BULK', '1').strip() == '0':
    pytest.skip('this process already streams every plane through registers')
  names = [c.name for c in CASES if c.path[0] == 'bulk']
  here = os.path.abspath(__file__)
  env = dict(os.environ, CTB_DEC_BULK='0')
  env[RECORDS_ENV] = str(tmp_path)
  r = subprocess.run([sys.executable, '-m', 'pytest', '-q', '-p', 'no:cacheprovider'] +
                     ['%s::test_decode_case[%s]' % (here, n) for n in names],
                     cwd=os.path.dirname(os.path.dirname(here)), env=env, capture_output=True, text=True)
  assert r.returncode == 0 and '%d passed' % len(names) in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
  for n in names:
    rec, _ = _gpu_records(_inputs(CASE[n]), CASE[n].K)
    reg = np.load(os.path.join(str(tmp_path), n + '.npy'))
    assert np.array_equal(rec.view(np.uint32), reg.view(np.uint32)), n


@gpu
@pytest.mark.parametrize('offset', [1, 2], ids=['4B', '8B'])
@pytest.mark.parametrize('shape', [(2, 3, 64, 96, 50), (1, 80, 136, 240, 100)], ids=['bulk', 'register'])
def test_decode_misaligned_hm(shape, offset):
  """hm (and reg, wh) one or two floats past a 16-byte boundary of a larger allocation: the 16-byte loads cannot read
  it, so every class plane takes the full-plane select.  The descriptor is built here as decode.py builds it, so the
  view's pointer reaches the kernel as it is."""
  B, C_, H, W, K = shape
  inp = _inputs(Case('misaligned', B, C_, H, W, K, 0, ('reg', 'wh'), None, None, 'full'), seed=offset)
  dev = {}
  for k, v in inp.items():
    buf = torch.zeros(v.size + 4, dtype=torch.float32, device='cuda')
    dev[k] = buf[offset:offset + v.size].view(v.shape)
    dev[k].copy_(torch.from_numpy(v))
    assert dev[k].data_ptr() % 16 == 4 * offset
  d = L.DecodeDesc()
  d.B, d.C, d.H, d.W, d.K = B, C_, H, W, K
  d.hm = dev['hm'].data_ptr()
  layout, off = {}, L.CT_REC_HEADS
  for n, (name, role) in enumerate((('reg', L.CT_ROLE_REG), ('wh', L.CT_ROLE_WH))):
    d.heads[n].map, d.heads[n].channels, d.heads[n].role, d.heads[n].rec_offset = dev[name].data_ptr(), 2, role, off
    layout[name] = (off, 2)
    off += 2
  d.n_heads, d.has_bbox, d.rec_hps, d.rec_kps_score, d.rec_floats = 2, 1, -1, -1, off
  rec = torch.empty((B, K, off), dtype=torch.float32, device='cuda')
  ws = torch.zeros(L.lib().ct_decode_workspace_bytes(B, C_, 0, K), dtype=torch.uint8, device='cuda')
  d.records, d.workspace = rec.data_ptr(), ws.data_ptr()
  L.check(L.lib().ct_decode(C.byref(d), L.stream_ptr()), 'ct_decode')
  _check(rec.cpu().numpy(), layout, inp, K, 'misaligned')


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the bench shape, CUDA-graph replay, and reuse of the arrival counters
# ---------------------------------------------------------------------------------------------------------------------
@gpu
def test_bench_shape_every_image():
  """B = 32, 80 x 128 x 128, K = 100: 2560 CTAs, the last to arrive for each image merges it.  Every image is checked,
  one oracle call per image."""
  case = BENCH
  inp = _inputs(case)
  rec, layout = _gpu_records(inp, case.K)
  for b in range(case.B):
    _check(rec[b:b + 1], layout, {k: v[b:b + 1] for k, v in inp.items()}, case.K, 'image %d' % b)


@gpu
def test_graph_replays_with_new_maps():
  """generic_decode captured in a CUDA graph with a caller-owned workspace (as Detector and StreamRunner capture it),
  replayed three times with different maps copied into the captured inputs: every replay matches the oracle."""
  from centertrack_b200.decode import generic_decode
  case = GRAPH
  maps = [_inputs(case, seed=s) for s in range(4)]
  static = {k: torch.from_numpy(v).cuda() for k, v in maps[0].items()}
  ws = torch.zeros(L.lib().ct_decode_workspace_bytes(case.B, case.C, 0, case.K), dtype=torch.uint8, device='cuda')
  first = generic_decode(static, K=case.K, workspace=ws)
  rec, layout = torch.empty_like(first.records), first.layout
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    generic_decode(static, K=case.K, records_out=rec, workspace=ws)
  torch.cuda.current_stream().wait_stream(side)
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    generic_decode(static, K=case.K, records_out=rec, workspace=ws)
  for i, inp in enumerate(maps[1:]):
    for k, v in inp.items():
      static[k].copy_(torch.from_numpy(v))
    g.replay()
    _check(rec.cpu().numpy(), layout, inp, case.K, 'replay %d' % i)


@gpu
def test_back_to_back_launches_on_one_workspace():
  """Two eager launches on the same workspace with different data, the second enqueued right behind the first: each
  one's last CTA resets the arrival counters the next one counts on."""
  from centertrack_b200.decode import generic_decode
  case = REUSE
  maps = [_inputs(case, seed=s) for s in (10, 11)]
  ws = torch.zeros(L.lib().ct_decode_workspace_bytes(case.B, case.C, 0, case.K), dtype=torch.uint8, device='cuda')
  dev = [{k: torch.from_numpy(v).cuda() for k, v in m.items()} for m in maps]
  res = [generic_decode(d, K=case.K, workspace=ws) for d in dev]
  for i, (r, inp) in enumerate(zip(res, maps)):
    _check(r.records.cpu().numpy(), r.layout, inp, case.K, 'launch %d' % i)
