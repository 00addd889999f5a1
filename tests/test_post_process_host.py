"""Device post-processing without a GPU: the ct_det_desc ABI, ct_post_process's host refusals, the runner's refusal
of a tracker together with device_post_process, and DeviceDetections.results (the dicts fetch_results() builds from
column copies) against a plain per-item builder."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT
from centertrack_b200 import _lib as L
from helpers import make_opt


def test_det_desc_layout_matches_the_header():
  assert C.sizeof(L.DetDesc) == 56
  assert (L.DetDesc.n.offset, L.DetDesc.rec_tracking.offset, L.DetDesc.out_thresh.offset, L.DetDesc.records.offset,
          L.DetDesc.trans_out_inv.offset, L.DetDesc.dets.offset, L.DetDesc.counts.offset) == (0, 12, 16, 24, 32, 40, 48)
  assert L.CT_DET_FLOATS == 10 == L.CT_TRK_BBOX + 4
  assert 'ct_post_process' in L.EXPORTS
  cc = shutil.which('cc') or shutil.which('gcc')
  if cc is None:
    pytest.skip('no C compiler to read the header')
  prog = r'''#include <stddef.h>
#include <stdio.h>
#include "ctb200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %d\n", sizeof(ct_det_desc), offsetof(ct_det_desc, n),
         offsetof(ct_det_desc, rec_tracking), offsetof(ct_det_desc, out_thresh), offsetof(ct_det_desc, records),
         offsetof(ct_det_desc, trans_out_inv), offsetof(ct_det_desc, dets), offsetof(ct_det_desc, counts),
         CT_DET_FLOATS);
  return 0;
}
'''
  with tempfile.TemporaryDirectory() as tmp:
    with open(os.path.join(tmp, 'p.c'), 'w') as f:
      f.write(prog)
    exe = os.path.join(tmp, 'p')
    subprocess.run([cc, '-I', os.path.join(ROOT, 'include'), os.path.join(tmp, 'p.c'), '-o', exe], check=True)
    got = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()
  assert [int(v) for v in got] == [56, 0, 12, 16, 24, 32, 40, 48, 10]


def test_post_process_refuses_before_launching(built_lib):
  """Each invalid argument returns -1 with a message from the host checks and launches nothing (no GPU here)."""
  lib = L.lib()

  def desc():
    d = L.DetDesc()
    d.n, d.K, d.F, d.rec_tracking, d.out_thresh = 2, 100, 40, 13, 0.3
    d.records = d.trans_out_inv = d.dets = d.counts = 64          # never dereferenced: validation fails first
    return d

  def ddd():
    q = L.TrackPayload()
    q.width, q.payload, q.calib = 20, 64, 64
    q.rec_hps, q.rec_dep, q.rec_rot, q.rec_dim, q.rec_amodel_offset = -1, 15, 16, 24, 27
    q.rec_nuscenes_att, q.att_floats, q.rec_velocity, q.velocity_floats = 29, 8, 37, 3
    return q

  def fails(msg, d=None, p=None, streams=None, n_streams=2):
    lib.ct_reset_launch_count()
    d = d if d is not None else desc()
    rc = lib.ct_post_process(C.byref(d), C.byref(p) if p is not None else None, streams, n_streams, None)
    assert rc == -1
    assert msg in lib.ct_last_error(), lib.ct_last_error()
    assert lib.ct_launch_count() == 0

  assert lib.ct_post_process(None, None, None, 2, None) == -1
  for field in ('records', 'trans_out_inv', 'dets', 'counts'):
    d = desc()
    setattr(d, field, None)
    fails(b'null pointer', d)
  for field, value in (('n', 0), ('K', 0), ('F', 8)):
    d = desc()
    setattr(d, field, value)
    fails(b'bad shape', d)
  for value in (39, 3):                        # past the record's end, inside its fixed columns
    d = desc()
    d.rec_tracking = value
    fails(b'tracking offset outside the record', d)
  fails(b'n_streams <= 0', n_streams=0)
  d = desc()
  d.n = 3
  fails(b'n <= n_streams', d)                  # identity map: image 2 has no stream
  p = ddd()
  p.payload = None
  fails(b'null payload', p=p)
  for field, value in (('rec_velocity', 38), ('rec_dep', 3), ('rec_dim', 38), ('rec_hps', 30)):
    p = ddd()
    setattr(p, field, value)
    fails(b'outside the record', p=p)
  p = ddd()
  p.width = 19
  fails(b'payload width', p=p)
  p = ddd()
  p.calib = None
  fails(b'calib', p=p)


def test_runner_refuses_a_tracker_with_device_post_process():
  """Raised before anything else is looked at: no model, no device, no CUDA work."""
  from centertrack_b200.runner import StreamRunner
  with pytest.raises(ValueError, match='device_post_process is for runners without a tracker'):
    StreamRunner(None, 2, 64, 96, device='cuda', device_tracking=True, device_post_process=True)


def test_track_videos_refuses_a_runner_without_tracker_or_post_process():
  from centertrack_b200.videos import track_videos

  class R(object):
    tracker = post = None
  with pytest.raises(ValueError, match='device_tracking=True or device_post_process=True'):
    next(track_videos(R(), []))


# ------------------------------------------------------------------------------------------------ the dict builder
def _layouts():
  ddd = {'reg': (9, 2), 'wh': (11, 2), 'dep': (13, 1), 'rot': (14, 8), 'dim': (22, 3), 'amodel_offset': (25, 2),
         'nuscenes_att': (27, 8), 'velocity': (35, 3)}
  return {'ctdet': ('ctdet', {'reg': (9, 2), 'wh': (11, 2)}, 13),
          'tracking': ('tracking', {'reg': (9, 2), 'wh': (11, 2), 'tracking': (13, 2)}, 15),
          'ddd': ('ddd', ddd, 38),
          'pose': ('multi_pose', {'reg': (9, 2), 'wh': (11, 2), 'hps': (13, 34), 'hps_refined': (47, 34),
                                  'kps_score': (81, 1)}, 82)}


def _per_item(det, dets, counts, pay, idle):
  """The plain builder: one dict per row, each value copied from the row."""
  out = []
  for b in range(dets.shape[0]):
    if b in idle:
      out.append(None)
      continue
    res = []
    for j in range(int(counts[b])):
      r = dets[b, j]
      item = {'score': float(r[0]), 'class': int(r[1]), 'ct': r[2:4].copy()}
      if det.has_tracking:
        item['tracking'] = r[4:6].copy()
      item['bbox'] = r[6:10].copy()
      for k, (o, w) in det.payload_layout.items():
        item[k] = float(pay[b, j, o]) if k in ('alpha', 'rot_y') else pay[b, j, o:o + w].copy()
      res.append(item)
    out.append(res)
  return out


@pytest.mark.parametrize('kind', list(_layouts()))
def test_results_equal_the_per_item_builder(kind):
  from centertrack_b200.device_detections import DeviceDetections
  from centertrack_b200.opts import opts
  task, layout, F = _layouts()[kind]
  opt = opts().init([task])
  B, K = 4, 6
  det = DeviceDetections(opt, B, K, F, layout, 64, 96, 'cpu')
  rng = np.random.RandomState(5)
  dets = rng.randn(B, K, L.CT_DET_FLOATS).astype(np.float32)
  dets[..., 1] = rng.randint(1, 11, (B, K))
  counts = np.array([0, K, 3, 2], np.int32)
  pay = rng.randn(B, K, det.Wp).astype(np.float32) if det.Wp else None
  want_keys = ['score', 'class', 'ct'] + (['tracking'] if kind == 'tracking' else []) + ['bbox'] + \
      {'ctdet': [], 'tracking': [], 'pose': ['hps'],
       'ddd': ['dep', 'dim', 'alpha', 'loc', 'rot_y', 'velocity', 'nuscenes_att']}[kind]
  for idle in ((), {3}):
    got = det.results(dets, counts, pay, idle)
    want = _per_item(det, dets, counts, pay, idle)
    assert [None if g is None else len(g) for g in got] == [0, K, 3, None if 3 in idle else 2]
    for g, w in zip(got, want):
      if w is None:
        assert g is None
        continue
      for a, e in zip(g, w):
        assert list(a) == want_keys
        for k in want_keys:
          assert type(a[k]) is type(e[k]) and np.array_equal(a[k], e[k]), (kind, k)
          assert np.shape(a[k]) == np.shape(e[k])
  # the values do not alias the tables passed in (the runner's pinned buffers, rewritten by later steps)
  got = det.results(dets, counts, pay)
  before = _per_item(det, dets, counts, pay, ())
  dets[:] = np.nan
  if pay is not None:
    pay[:] = np.nan
  for g, w in zip(got, before):
    for a, e in zip(g, w):
      for k in want_keys:
        assert np.array_equal(a[k], e[k]), (kind, k)
  if det.Wp:
    with pytest.raises(ValueError, match='payload_np'):
      det.results(dets, counts)
