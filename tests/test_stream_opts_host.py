"""Per-stream tracker settings on the host (no GPU): the resolution against opts.py's derivation, the refusals that run
before anything is enqueued, StreamState's options, and the _opts entry points in the header, the binding and their
argument checks."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from centertrack_b200 import _lib as L
from centertrack_b200.device_tracker import POST_OPTION_KEYS, DeviceTracker, resolve_options
from helpers import ROOT, make_opt

LAYOUT = {'tracking': (9, 2)}
F = 11

GRID = [[], ['--track_thresh', '0.1'], ['--track_thresh', '0.5'], ['--out_thresh', '0.2'], ['--out_thresh', '0.6'],
        ['--pre_thresh', '0.1', '--new_thresh', '0.7'], ['--track_thresh', '0.45', '--pre_thresh', '0.3'],
        ['--track_thresh', '0.2', '--out_thresh', '0.35', '--pre_thresh', '0.6', '--new_thresh', '0.25'],
        ['--max_age', '3', '--hungarian'], ['--public_det', '--max_age', '1']]


def _as_flags(args):
  f, i = {}, 0
  while i < len(args):
    k = args[i][2:]
    if k in ('hungarian', 'public_det'):
      f[k], i = True, i + 1
    else:
      f[k], i = (int(args[i + 1]) if k == 'max_age' else float(args[i + 1])), i + 2
  return f


@pytest.mark.parametrize('base', [[], ['--track_thresh', '0.4', '--pre_thresh', '0.5']])
@pytest.mark.parametrize('i', range(len(GRID)))
def test_resolution_equals_opts_init_of_the_same_flags(base, i):
  """opt_b = the runner's flags + the stream's, through opts().init: flags below and above track_thresh."""
  args = GRID[i]
  opt = make_opt('mot', base)
  got = resolve_options(opt, _as_flags(args))
  want = make_opt('mot', base + args)
  for k in ('out_thresh', 'new_thresh', 'pre_thresh', 'max_age', 'hungarian', 'public_det'):
    assert got[k] == getattr(want, k), (k, args)
  assert resolve_options(opt, None) == resolve_options(opt, {})
  # without a tracker: out_thresh alone, not derived (opts.py's non-tracking branch)
  det = make_opt('mot', base)
  det.task = 'ctdet'
  assert resolve_options(det, {'out_thresh': 0.05}, POST_OPTION_KEYS) == {'out_thresh': 0.05}


def test_resolution_refuses_other_keys_and_bad_values():
  opt = make_opt('mot')
  for k in ('K', 'flip_test', 'pre_hm', 'head_conv', 'reg_offset', 'input_h'):
    with pytest.raises(ValueError, match="'%s'" % k):
      resolve_options(opt, {k: 1})
  with pytest.raises(ValueError, match="'max_age'"):
    resolve_options(opt, {'max_age': 'x'}, POST_OPTION_KEYS)
  for k, v in (('hungarian', 1), ('public_det', 'yes'), ('max_age', 2.0), ('max_age', True), ('track_thresh', 'a'),
               ('out_thresh', float('nan')), ('new_thresh', None), ('pre_thresh', True)):
    with pytest.raises(ValueError, match=r"\['%s'\]: bad value" % k):
      resolve_options(opt, {k: v})
  with pytest.raises(ValueError, match='dict'):
    resolve_options(opt, [('max_age', 1)])


def _tracker(opt, stream_opts, B=3):
  return DeviceTracker(opt, B, 16, F, LAYOUT, 64, 64, 'cpu', max_public_dets=8, stream_opts=stream_opts)


def test_tracker_capacity_staging_and_records(built_lib):
  opt = make_opt('mot', ['--max_age', '1'])
  trk = _tracker(opt, [None, {'max_age': 4, 'hungarian': True}, {'track_thresh': 0.6}])
  assert trk.T == 16 * 5 and trk.max_age == 4 and trk.hungarian and not trk.public_det
  rec = (L.TrackOpts * 3).from_buffer_copy(trk.d_opts.numpy().tobytes())
  assert C.sizeof(L.TrackOpts) == 32
  assert [r.max_age for r in rec] == [1, 4, 1] and [r.hungarian for r in rec] == [0, 1, 0]
  assert rec[2].out_thresh == np.float32(0.6) and rec[0].out_thresh == np.float32(opt.out_thresh)
  with pytest.raises(ValueError, match='max_age 5 is above the 4'):
    trk.check_options({'max_age': 5}, 'options[1]')
  with pytest.raises(ValueError, match='stages no public detections'):
    trk.check_options({'public_det': True}, 'options[0]')
  assert trk.check_options({'max_age': 4})['max_age'] == 4
  with pytest.raises(ValueError, match=r'expected 3 entries'):
    _tracker(opt, [None, None])
  plain = _tracker(opt, None)
  assert plain.d_opts is None and plain.T == 32
  with pytest.raises(ValueError, match='built without stream_opts'):
    plain.check_options({'max_age': 1})


def _runner(stream_opts, opt=None, B=3):
  """A StreamRunner with nothing but a CPU tracker and the host state the step checks read."""
  from centertrack_b200.runner import StreamRunner
  r = object.__new__(StreamRunner)
  r.opt = opt or make_opt('mot', ['--max_age', '1'])
  r.B, r.H, r.W, r.t, r.idle_g, r.frames_mode, r.post = B, 64, 64, 0, None, False, None
  r.tracker = _tracker(r.opt, stream_opts, B)
  r.public = r.tracker.public_det
  return r


def test_runner_refusals_before_anything_is_enqueued(built_lib):
  """Each refusal of step_host fires before the runner touches a device buffer or stream (the fake runner has none:
  reaching them would raise AttributeError, not ValueError)."""
  import torch
  r = _runner([None, {'public_det': True}, {'max_age': 2}])
  img = torch.zeros((3, 3, 64, 64))
  pub = [None, np.zeros((1, 2), np.float32), None]
  cases = [
      (dict(options={0: {'max_age': 1}}), 'does not start a video'),                 # outside a start
      (dict(starts=[0], options={0: {'K': 50}}), "'K' cannot differ"),
      (dict(starts=[0], options={0: {'flip_test': True}}), "'flip_test' cannot differ"),
      (dict(starts=[0], options={0: {'max_age': 1.5}}), 'bad value'),
      (dict(starts=[0], options={0: {'max_age': 3}}), 'max_age 3 is above the 2'),
      (dict(public_dets=[np.zeros((1, 2), np.float32)] * 3), r'public_dets\[0\]: stream 0 runs without public_det'),
      (dict(public_dets=None), 'every step needs the public detections'),
  ]
  for kw, msg in cases:
    kw.setdefault('public_dets', pub)
    with pytest.raises(ValueError, match=msg):
      r.step_host(img, **kw)
  # a start turning public_det off: its entry must then be None
  with pytest.raises(ValueError, match=r'public_dets\[1\]'):
    r.step_host(img, public_dets=pub, starts=[1], options={1: {'public_det': False}})
  # public_det on a runner built without staging
  r2 = _runner([None, {'hungarian': True}, None])
  with pytest.raises(ValueError, match='stages no public detections'):
    r2.step_host(img, starts=[2], options={2: {'public_det': True}})
  # a runner without stream_opts refuses options
  r3 = _runner(None)
  with pytest.raises(ValueError, match='built without stream_opts'):
    r3.step_host(img, starts=[2], options={2: {'max_age': 1}})
  # the host state was not changed by any refused step
  assert [o['max_age'] for o in r.tracker.options] == [1, 1, 2]


def test_pre_dets_seeds_use_the_streams_new_thresh(built_lib):
  r = _runner([None, {'new_thresh': 0.8}, None], B=3)
  items = [{'score': s, 'class': 1, 'bbox': [1., 2., 10., 12.]} for s in (0.35, 0.5, 0.9)]
  now = r._step_options(r._check_options({2: {'track_thresh': 0.6}}, [2]))
  streams, seeds = r._check_starts([0, 1, 2], {0: items, 1: items, 2: items}, now)
  assert streams == [0, 1, 2] and [len(s) for s in seeds] == [3, 1, 1]       # new_thresh 0.3, 0.8, 0.6


def test_stream_state_round_trips_its_options(built_lib):
  from centertrack_b200.runner import StreamState
  o = resolve_options(make_opt('mot'), {'track_thresh': 0.45, 'hungarian': True})
  st = StreamState(None, (4, 4), np.eye(3, 4, dtype=np.float32), None, (0, 0), None, (64, 64), {}, None, 16, 'bgr',
                   options=o)
  assert st.options == o and st.options is not o
  r = _runner([None, {'max_age': 1}, None])
  assert r._restore_options({1: st}) == {1: o}
  big = StreamState(None, (4, 4), None, None, (0, 0), None, (64, 64), {}, None, 16, 'bgr', options=dict(o, max_age=9))
  with pytest.raises(ValueError, match=r'restore\[1\]: max_age 9'):
    r._restore_options({1: big})
  assert StreamState(None, (4, 4), None, None, None, None, (64, 64), {}, None, None, 'bgr').options is None


def test_opts_entry_points_are_declared_exported_and_check_their_arguments(built_lib):
  src = open(os.path.join(ROOT, 'include', 'ctb200.h')).read()
  for name in ('ct_track_step_opts', 'ct_track_start_opts', 'ct_track_restore_opts', 'ct_post_process_opts'):
    assert re.search(r'\bint %s\(' % name, src) and name in L.EXPORTS
  assert 'CTB200_ABI_VERSION 2' in src
  lib = L.lib()
  d = L.TrackDesc()
  d.B, d.K, d.F, d.max_tracks, d.rec_tracking = 2, 4, 11, 8, -1
  d.records = d.trans_out_inv = d.tracks = d.counts = 16
  opts = C.c_void_p(16)
  assert lib.ct_track_step_opts(C.byref(d), None, None, None, None, 0, None) == L.CT_ERR_INVALID
  assert b'null opts' in lib.ct_last_error()
  assert lib.ct_track_step_opts(C.byref(d), None, None, opts, None, -1, None) == L.CT_ERR_INVALID
  assert b'n_streams < 0' in lib.ct_last_error()
  assert lib.ct_track_step_opts(C.byref(d), None, None, opts, C.c_void_p(16), 0, None) == L.CT_ERR_INVALID
  a = L.TrackAssoc()
  a.public_det, a.max_public = 1, 4
  assert lib.ct_track_step_opts(C.byref(d), C.byref(a), None, opts, None, 0, None) == L.CT_ERR_INVALID
  assert b'public_det needs public_ct' in lib.ct_last_error()
  assert lib.ct_track_start_opts(C.byref(d), None, None, C.c_void_p(16), 1, None, None) == L.CT_ERR_INVALID
  assert b'null opts' in lib.ct_last_error()
  assert lib.ct_track_restore_opts(C.byref(d), None, None, C.c_void_p(16), 1, None, None, None) == L.CT_ERR_INVALID
  assert lib.ct_track_restore_opts(C.byref(d), None, opts, None, 1, None, None, None) == L.CT_ERR_INVALID
  assert b'null entry list' in lib.ct_last_error()
  dd = L.DetDesc()
  dd.n, dd.K, dd.F = 2, 4, 11
  dd.records = dd.trans_out_inv = dd.dets = dd.counts = 16
  assert lib.ct_post_process_opts(C.byref(dd), None, None, None, 2, None) == L.CT_ERR_INVALID
  assert b'null opts' in lib.ct_last_error()
  assert lib.ct_post_process_opts(C.byref(dd), None, opts, None, -1, None) == L.CT_ERR_INVALID


def test_one_resolution_rule_for_none_and_dicts_after_opt_changes():
  """An opt changed after opts().init: entries that set no threshold run opt's thresholds as they are (None, {} and
  a dict of other flags alike); a threshold flag re-derives from opt's current thresholds."""
  opt = make_opt('coco_tracking', ['--track_thresh', '0.2'])
  opt.out_thresh = 0.1                                       # below track_thresh, as a caller may set it
  base = resolve_options(opt, None)
  assert base['out_thresh'] == 0.1 and resolve_options(opt, {}) == base
  assert resolve_options(opt, {'hungarian': True}) == dict(base, hungarian=True)
  assert resolve_options(opt, {'max_age': 3})['out_thresh'] == 0.1
  got = resolve_options(opt, {'track_thresh': 0.05})
  assert (got['out_thresh'], got['pre_thresh'], got['new_thresh']) == (0.1, opt.pre_thresh, opt.new_thresh)
  got = resolve_options(opt, {'track_thresh': 0.4})
  assert (got['out_thresh'], got['pre_thresh'], got['new_thresh']) == (0.4, 0.4, 0.4)
  trk = _tracker(opt, [None, {}, {'hungarian': True}])
  assert [o['out_thresh'] for o in trk.options] == [0.1, 0.1, 0.1]
  # an unchanged opt: a threshold flag below the runner's track_thresh is opts().init's value
  fresh = make_opt('coco_tracking', ['--track_thresh', '0.4'])
  assert resolve_options(fresh, {'track_thresh': 0.1})['out_thresh'] == make_opt('coco_tracking', [
      '--track_thresh', '0.4', '--track_thresh', '0.1']).out_thresh == 0.1


def test_restore_takes_numpy_starts(built_lib):
  r = _runner([None, None, None])
  r.cap = None
  assert r._check_restore(None, r._streams_arg('starts', np.array([0, 2])), None) == {}
  assert r._streams_arg('starts', np.array([2, 0])) == [2, 0]
