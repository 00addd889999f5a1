"""Per-stream tracker state kept on the GPU between frames (SURVEY 8f-1): the reference's
`generic_post_process` affine (utils/post_process.py:21-91), `Tracker.step` association (utils/tracker.py:28-138:
greedy, `--hungarian`, `--public_det`) and the prior heat-map render of `Detector._get_additional_inputs`
(detector.py:254-290) as two launches on the decode records -- `ct_track_step` (`ct_track_step_assoc` for the
Hungarian / public-detection modes) and `ct_render_tracks` -- so that a stream never returns to the host between
frames: records(t) -> tracks(t) -> pre_hm(t+1) are all device-resident and CUDA-graph capturable (fixed launch shapes).
Every mode reproduces the host `Tracker` (centertrack_b200.tracker) row for row.
Results are rows of CT_TRK_FLOATS fp32 (score, class, ct, tracking, bbox, tracking_id, age, active) in the
reference's output order (matched detections, new tracks, coasting tracks).  Pose, 3D, velocity and attribute head
sets also get a parallel payload table [B,T,Wp] (`ct_track_step_payload`) with the fields generic_post_process adds
for them (hps, dep, dim, alpha, loc, rot_y, velocity, nuscenes_att); on 3D head sets `ct` is the amodal centre, as in
the reference.  `results()` turns host copies into the reference's list of dicts.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib as L
from .dataset_info import get_dataset
from .image import get_affine_transform

# widths of the record heads a payload field is computed from, as the reference's heads have them (opts.py)
_HEAD_WIDTHS = {'dep': 1, 'dim': 3, 'rot': 8, 'amodel_offset': 2}


def payload_layout(layout):
  """Decode record layout {head: (offset, width)} -> the payload row {field: (offset, width)}, in ct_track_payload's
  order: each field generic_post_process adds for the heads present (post_process.py:55-89).  {} for 2-D head sets."""
  for k, w in _HEAD_WIDTHS.items():
    if k in layout and layout[k][1] != w:
      raise ValueError('%s head with %d channels, expected %d' % (k, layout[k][1], w))
  fields = []
  if 'hps' in layout:
    fields.append(('hps', layout['hps'][1]))
  fields += [(f, w) for f, head, w in (('dep', 'dep', 1), ('dim', 'dim', 3), ('alpha', 'rot', 1)) if head in layout]
  if all(k in layout for k in ('rot', 'dep', 'dim')):
    fields += [('loc', 3), ('rot_y', 1)]
  fields += [(k, layout[k][1]) for k in ('velocity', 'nuscenes_att') if k in layout]
  out, off = {}, 0
  for f, w in fields:
    out[f] = (off, w)
    off += w
  return out


def seed_rows(items, new_thresh):
  """Tracker.init_track on a fresh tracker (utils/tracker.py:11-22) as track-table rows: the result dicts with
  score > new_thresh, in input order, get ids 1..n with age = 1 and active = 1; `ct` is the bbox centre when the item has
  none, computed in float64 as the reference does on its JSON-loaded results.  `tracking` is 0 when absent.
  -> float32 [n, CT_TRK_FLOATS].  ValueError when a kept item lacks score, class or bbox."""
  rows = []
  for item in items:
    if item['score'] <= new_thresh:
      continue
    try:
      bbox = [float(v) for v in item['bbox'][:4]]
      cls = item['class']
    except KeyError as e:
      raise ValueError('pre_dets: a seed needs score, class and bbox (missing %s)' % e)
    ct = item['ct'] if 'ct' in item else [(bbox[0] + bbox[2]) / 2, (bbox[1] + bbox[3]) / 2]
    r = np.zeros(L.CT_TRK_FLOATS, np.float32)
    r[L.CT_TRK_SCORE], r[L.CT_TRK_CLASS] = item['score'], cls
    r[L.CT_TRK_CT:L.CT_TRK_CT + 2] = np.asarray(ct, np.float64)[:2]
    r[L.CT_TRK_TRACKING:L.CT_TRK_TRACKING + 2] = np.asarray(item.get('tracking', (0., 0.)), np.float64)[:2]
    r[L.CT_TRK_BBOX:L.CT_TRK_BBOX + 4] = bbox
    r[L.CT_TRK_ID], r[L.CT_TRK_AGE], r[L.CT_TRK_ACTIVE] = len(rows) + 1, 1, 1
    rows.append(r)
  return np.stack(rows) if rows else np.zeros((0, L.CT_TRK_FLOATS), np.float32)


# The reference flags a StreamRunner stream may set for itself (stream_opts, options=): they act only in the per-stream
# kernels.  A runner without a tracker (device_post_process) takes out_thresh alone.
TRACK_OPTION_KEYS = ('track_thresh', 'out_thresh', 'pre_thresh', 'new_thresh', 'max_age', 'hungarian', 'public_det')
POST_OPTION_KEYS = ('out_thresh',)


def resolve_options(opt, flags, keys=TRACK_OPTION_KEYS, what='options'):
  """The settings of opt_b = opt with a stream's flags ({name: value} of `keys`, or None) applied -> {out_thresh,
  new_thresh, pre_thresh, max_age, hungarian, public_det}; None and {} give opt's own.  The one rule for every entry:
  flags that set no threshold leave opt's thresholds as they are (its current attributes, whatever changed them after
  opts().init).  A threshold flag (track_thresh, out_thresh, pre_thresh, new_thresh) re-derives all three as
  opts.py:97-99 does on tracking tasks, max(track_thresh, threshold), from the thresholds opts was given (opt.thresh_args) while
  those still derive to opt's current values -- so opt_b is opts().init of the runner's flags plus the stream's -- and
  from opt's current thresholds once opt was changed after init (or has no thresh_args).  Only out_thresh, without the
  derivation, when keys is POST_OPTION_KEYS.  ValueError naming the key for a key outside `keys` (such as K, flip_test,
  pre_hm or a head option, which change the network or the records) or a value of the wrong type."""
  flags = {} if flags is None else flags
  if not isinstance(flags, dict):
    raise ValueError('%s: expected a dict of per-stream flags or None, got %s' % (what, type(flags).__name__))
  for k, v in flags.items():
    if k not in keys:
      raise ValueError('%s: %r cannot differ between the streams of a runner; a stream may set %s' %
                       (what, k, ', '.join(keys)))
    if k in ('hungarian', 'public_det'):
      ok = isinstance(v, (bool, np.bool_))
    elif k == 'max_age':
      ok = isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_))
    else:
      ok = isinstance(v, (int, float, np.integer, np.floating)) and not isinstance(v, (bool, np.bool_)) and \
          np.isfinite(v)
    if not ok:
      raise ValueError('%s[%r]: bad value %r (%s)' % (what, k, v, 'a bool' if k in ('hungarian', 'public_det') else
                                                     'an int' if k == 'max_age' else 'a finite number'))
  if keys == POST_OPTION_KEYS:
    return {'out_thresh': float(flags.get('out_thresh', opt.out_thresh))}
  names = ('out_thresh', 'pre_thresh', 'new_thresh')
  now = {k: getattr(opt, k) for k in names}
  given = now
  if any(k in flags for k in names + ('track_thresh',)):
    tracking = 'tracking' in getattr(opt, 'task', 'tracking')
    derive = lambda v, track: {k: max(track, x) for k, x in v.items()} if tracking else dict(v)
    args = getattr(opt, 'thresh_args', None)
    if args is not None and derive(args, opt.track_thresh) == now:
      given = dict(args)                             # opt as opts().init left it: the thresholds as given
    else:
      given = dict(now)                              # opt changed after init: its current thresholds
    given.update((k, flags[k]) for k in names if k in flags)
    given = derive(given, flags.get('track_thresh', getattr(opt, 'track_thresh', 0.3)))
  return {'out_thresh': float(given['out_thresh']), 'new_thresh': float(given['new_thresh']),
          'pre_thresh': float(given['pre_thresh']), 'max_age': int(flags.get('max_age', opt.max_age)),
          'hungarian': bool(flags.get('hungarian', getattr(opt, 'hungarian', False))),
          'public_det': bool(flags.get('public_det', getattr(opt, 'public_det', False)))}


def opts_records(resolved):
  """Resolved settings (resolve_options), one per stream -> ct_track_opts [n] (ctypes array)."""
  arr = (L.TrackOpts * len(resolved))()
  for r, v in zip(arr, resolved):
    r.out_thresh = v['out_thresh']
    if 'max_age' in v:
      r.new_thresh, r.pre_thresh, r.max_age = v['new_thresh'], v['pre_thresh'], v['max_age']
      r.hungarian, r.public_det = int(v['hungarian']), int(v['public_det'])
  return arr


def plan_starts(B, T, new_thresh, has_payload, starts, pre_dets):
  """Checks one step's video starts and builds their seeds, before anything is enqueued.  starts: stream indices whose
  frame is a video's first; pre_dets: {stream: list of result dicts} seeding some of them (or None).  new_thresh: one
  threshold, or one per stream (each stream's seeds are filtered with its own).
  -> (streams list, [seed rows float32 [n_i, CT_TRK_FLOATS]] in the same order).  ValueError on a stream out of range
  or repeated, pre_dets for a stream that does not start, more kept seeds than the T rows of the track table, or
  pre_dets on a head set with payload fields (their seeds would need those fields)."""
  streams = []
  for s in starts:
    if isinstance(s, (bool, np.bool_)) or not isinstance(s, (int, np.integer)):
      raise ValueError('starts: stream indices must be integers, got %r' % (s,))
    s = int(s)
    if not 0 <= s < B:
      raise ValueError('starts: stream %d out of range [0, %d)' % (s, B))
    if s in streams:
      raise ValueError('starts: stream %d given twice' % s)
    streams.append(s)
  pre_dets = pre_dets or {}
  for s in pre_dets:
    if s not in streams:
      raise ValueError('pre_dets: stream %r does not start a video in this step' % (s,))
  if has_payload and pre_dets:
    raise ValueError('pre_dets: seeding is not supported on head sets with payload fields (pose, 3D, velocity, '
                     'attributes); start those streams without pre_dets')
  seeds = []
  for s in streams:
    rows = seed_rows(pre_dets.get(s, ()), new_thresh[s] if isinstance(new_thresh, (list, tuple)) else new_thresh)
    if len(rows) > T:
      raise ValueError('pre_dets[%d]: %d seeds above new_thresh, more than the %d rows of the track table' %
                       (s, len(rows), T))
    seeds.append(rows)
  return streams, seeds


def default_geometry(inp_h, inp_w):
  """(c, s) of a source image of exactly the network input size: DeviceTracker's default camera geometry."""
  return np.array([inp_w / 2., inp_h / 2.], np.float32), max(inp_h, inp_w) * 1.0


class DeviceTracker(object):

  def __init__(self, opt, B, K, rec_floats, layout, inp_h, inp_w, device, centers=None, scales=None, max_tracks=None,
               max_public_dets=512, calibs=None, stream_opts=None):
    """centers/scales: per-stream (c, s) of the source rectangle (Detector._input_geometry); default = a source image
    of exactly the network input size (the synthetic benchmark streams).  max_public_dets: with --public_det, the most
    public detections one stream may bring per frame (P, the row count of the public_ct buffers step() takes).
    calibs: per-stream [3,4] camera matrices for the 3D head sets (loc, rot_y); default = Detector._get_default_calib
    of a source image centred on c, with --test_focal_length or the dataset's rest_focal_length.
    stream_opts: None (every stream runs opt), or B entries, each None (opt) or a dict of TRACK_OPTION_KEYS flags that
    stream b runs with instead (resolve_options): its own thresholds, max_age, --hungarian and --public_det, through the
    _opts entry points and the device records d_opts.  The table's T rows then come from the largest max_age, public
    detections are staged when any stream has --public_det, and the Hungarian scratch is always allocated."""
    self.per_stream = stream_opts is not None
    if self.per_stream and len(stream_opts) != B:
      raise ValueError('stream_opts: expected %d entries (one per stream, None or a dict), got %d' %
                       (B, len(stream_opts)))
    self.options = [resolve_options(opt, f, what='stream_opts[%d]' % b)
                    for b, f in enumerate(stream_opts if self.per_stream else [None] * B)]
    self.hungarian = any(o['hungarian'] for o in self.options)
    self.public_det = any(o['public_det'] for o in self.options)
    self.max_age = max(o['max_age'] for o in self.options)     # the table's coasting capacity
    self.max_public = int(max_public_dets)
    if self.public_det and self.max_public <= 0:
      raise ValueError('--public_det needs max_public_dets > 0')
    self.opt, self.B, self.K, self.F = opt, B, K, rec_floats
    self.inp_h, self.inp_w = inp_h, inp_w
    self.device = torch.device(device)
    self.T = int(max_tracks or (K * (1 + max(0, self.max_age))))
    self.T = max(self.T, K)
    c0, s0 = default_geometry(inp_h, inp_w)
    t_in, t_out = self._trans_rows([c0 if centers is None else centers[b] for b in range(B)],
                                   [s0 if scales is None else scales[b] for b in range(B)])
    self.trans_out_inv = torch.from_numpy(t_out).to(self.device)
    self.trans_input = torch.from_numpy(t_in).to(self.device)
    self.tracks = torch.zeros((B, self.T, L.CT_TRK_FLOATS), dtype=torch.float32, device=self.device)
    self.counts = torch.zeros((B, 2), dtype=torch.int32, device=self.device)
    self.boxes = torch.zeros((B, self.T, 5), dtype=torch.float32, device=self.device)
    self.boxes[:, :, 3] = -1.0                       # no tracks yet: nothing to splat (first frame: pre_hm = 0)
    d = L.TrackDesc()
    d.B, d.K, d.F = B, K, rec_floats
    d.rec_tracking = layout['tracking'][0] if 'tracking' in layout else -1
    d.max_tracks = self.T
    d.out_thresh, d.new_thresh, d.pre_thresh = float(opt.out_thresh), float(opt.new_thresh), float(opt.pre_thresh)
    d.max_age = int(opt.max_age)
    d.inp_h, d.inp_w = inp_h, inp_w
    d.trans_out_inv, d.trans_input = self.trans_out_inv.data_ptr(), self.trans_input.data_ptr()
    d.tracks, d.counts, d.boxes = self.tracks.data_ptr(), self.counts.data_ptr(), self.boxes.data_ptr()
    self.desc = d
    a = L.TrackAssoc()
    a.hungarian, a.public_det, a.max_public = int(self.hungarian), int(self.public_det), self.max_public
    self.assoc = a
    self.payload_layout = payload_layout(layout)
    self.Wp = sum(w for _, w in self.payload_layout.values())
    self.payload = self.calib = self.pay = None
    if self.Wp:
      self.payload = torch.zeros((B, self.T, self.Wp), dtype=torch.float32, device=self.device)
      p = L.TrackPayload()
      p.width, p.payload = self.Wp, self.payload.data_ptr()
      rec = lambda k: layout[k][0] if k in layout else -1
      p.rec_hps = rec('hps_refined' if 'hps_refined' in layout else 'hps')      # as decode.views_from_records
      p.hps_floats = layout['hps'][1] if 'hps' in layout else 0
      p.rec_dep, p.rec_dim, p.rec_rot, p.rec_amodel_offset = rec('dep'), rec('dim'), rec('rot'), rec('amodel_offset')
      p.rec_velocity, p.velocity_floats = rec('velocity'), layout.get('velocity', (0, 0))[1]
      p.rec_nuscenes_att, p.att_floats = rec('nuscenes_att'), layout.get('nuscenes_att', (0, 0))[1]
      if 'loc' in self.payload_layout:
        self.calib = torch.from_numpy(self._calibs(opt, calibs, centers, inp_h, inp_w)).to(self.device)
        p.calib = self.calib.data_ptr()
      self.pay = p
    smem = L.lib().ct_track_payload_smem_bytes(K, self.T, self.Wp, int(self.hungarian or self.public_det or
                                                                         self.per_stream))
    if smem > 200 * 1024:
      raise ValueError('track table of %d rows does not fit in shared memory' % self.T)
    self.d_opts = None
    if self.per_stream:
      self.d_opts = torch.frombuffer(bytearray(self.opts_bytes()), dtype=torch.uint8).to(self.device)

  def opts_bytes(self):
    """The ct_track_opts records of the streams' current settings, as bytes."""
    return bytes(opts_records(self.options))

  def check_options(self, flags, what='options', resolved=False):
    """A stream's new settings (a dict of flags, resolved against opt; resolved=True: settings resolve_options already
    gave, as a StreamState carries them) -> the resolved settings.  ValueError for what resolve_options refuses, on a tracker built without
    stream_opts, for a max_age above the table's capacity, or --public_det on a tracker that stages no public
    detections."""
    if not self.per_stream:
      raise ValueError('%s: this runner was built without stream_opts: its streams all run opt (build it with '
                       'stream_opts to give streams their own tracker settings)' % what)
    o = dict(flags) if resolved else resolve_options(self.opt, flags, what=what)
    if o['max_age'] > self.max_age:
      raise ValueError('%s: max_age %d is above the %d the track table was sized for (T = K (1 + max_age) = %d rows); '
                       'give the runner a stream_opts entry with the largest max_age' % (what, o['max_age'],
                                                                                          self.max_age, self.T))
    if o['public_det'] and not self.public_det:
      raise ValueError('%s: public_det on a runner that stages no public detections (neither opt nor any stream_opts '
                       'entry has public_det)' % what)
    return o

  def _calibs(self, opt, calibs, centers, inp_h, inp_w):
    if calibs is not None:
      out = np.asarray(calibs, np.float32)
      if out.shape != (self.B, 3, 4):
        raise ValueError('calibs: expected %d camera matrices [3, 4], got shape %s' % (self.B, out.shape))
      return np.ascontiguousarray(out)
    f = opt.test_focal_length if getattr(opt, 'test_focal_length', -1) >= 0 else get_dataset(opt.dataset).rest_focal_length
    out = np.zeros((self.B, 3, 4), np.float32)
    for b in range(self.B):
      cx, cy = (inp_w / 2., inp_h / 2.) if centers is None else (float(centers[b][0]), float(centers[b][1]))
      out[b] = [[f, 0, cx, 0], [0, f, cy, 0], [0, 0, 1, 0]]      # Detector._get_default_calib(2 cx, 2 cy)
    return out

  def _trans_rows(self, centers, scales):
    """(c, s) per stream -> (trans_input float64 [n, 6], trans_out_inv float32 [n, 6]) rows."""
    down = getattr(self.opt, 'down_ratio', 4)
    out_w, out_h = self.inp_w // down, self.inp_h // down
    t_out = np.zeros((len(centers), 6), np.float32)
    t_in = np.zeros((len(centers), 6), np.float64)
    for i, (c, s) in enumerate(zip(centers, scales)):
      c = np.asarray(c, np.float32)
      t_out[i] = get_affine_transform(c, s, 0, (out_w, out_h), inv=1).astype(np.float32).reshape(6)
      t_in[i] = get_affine_transform(c, s, 0, [self.inp_w, self.inp_h]).reshape(6)
    return t_in, t_out

  def geometry_rows(self, centers, scales, calibs):
    """The camera geometry of n streams ((c, s) of their source rectangle and [3,4] camera matrices) -> the rows
    set_geometry writes: (float64 [n, 6] trans_input, float32 [n, 18] = trans_out_inv (6) then calib (12)), computed
    exactly as the constructor computes them."""
    t_in, t_out = self._trans_rows(centers, scales)
    cal = np.asarray(calibs, np.float32).reshape(len(t_out), 12)
    return t_in, np.concatenate([t_out, cal], axis=1)

  def set_geometry(self, streams, rows_in, rows_out):
    """trans_input, trans_out_inv (and calib on 3D head sets) of `streams` <- rows (geometry_rows, device tensors), on
    the current stream.  The descriptors keep pointing at the same tensors, so captured graphs read the new rows: call
    it between two steps, before start_device renders the streams' seeds."""
    for i, b in enumerate(streams):
      self.trans_input[b].copy_(rows_in[i])
      self.trans_out_inv[b].copy_(rows_out[i, :6])
      if self.calib is not None:
        self.calib[b].view(12).copy_(rows_out[i, 6:])

  def reset(self):
    """Detector.reset_tracking / Tracker.reset for every stream."""
    self.tracks.zero_()
    self.counts.zero_()
    if self.payload is not None:
      self.payload.zero_()
    self.boxes.zero_()
    self.boxes[:, :, 3] = -1.0

  def start(self, streams, seeds=None):
    """Detector.reset_tracking + Tracker.init_track(seeds[b]) on each stream b of `streams` alone, on the current
    stream: its tracks, counts and payload are cleared, the seeds written (seed_rows), and its boxes rendered from them,
    so that the next render() splats them.  seeds: {stream: list of result dicts} (pre_dets) or None.  ValueError as
    plan_starts."""
    streams, rows = plan_starts(self.B, self.T, [o['new_thresh'] for o in self.options], self.payload is not None,
                                streams, seeds)
    if not streams:
      return
    lst = torch.tensor([[s, len(r)] for s, r in zip(streams, rows)], dtype=torch.int32).to(self.device)
    seed = torch.from_numpy(np.concatenate(rows)).to(self.device) if sum(map(len, rows)) else None
    self.start_device(lst, len(streams), seed)

  def _opts(self, opts):
    """The device ct_track_opts records a launch reads: `opts` (a runner's per-slot copy), or d_opts."""
    return L.ptr(self.d_opts if opts is None else opts)

  def start_device(self, start_list, n_starts, seeds=None, opts=None):
    """ct_track_start on device buffers: start_list int32 [>= n_starts, 2] rows (stream, seed rows), seeds fp32
    [sum of n, CT_TRK_FLOATS] in start_list's order (or None).  No checks of the contents: see plan_starts.  With
    stream_opts: ct_track_start_opts on `opts` (device ct_track_opts [B], default d_opts)."""
    pay = C.byref(self.pay) if self.pay is not None else None
    if self.per_stream:
      L.check(L.lib().ct_track_start_opts(C.byref(self.desc), pay, self._opts(opts), L.ptr(start_list), n_starts,
                                          L.ptr(seeds), L.stream_ptr()), 'ct_track_start_opts')
      return
    L.check(L.lib().ct_track_start(C.byref(self.desc), pay, L.ptr(start_list), n_starts, L.ptr(seeds),
                                   L.stream_ptr()), 'ct_track_start')

  def restore_device(self, entries, n_entries, rows=None, payload_rows=None, opts=None):
    """ct_track_restore on device buffers: entries int32 [>= n_entries, 3] rows (stream, rows n, id_count), rows fp32
    [sum of n, CT_TRK_FLOATS] and payload_rows fp32 [sum of n, Wp] in entries' order (None when every n is 0).  The
    rows are written as they are, and each stream's boxes rendered from them with its own index and trans_input.
    With stream_opts: ct_track_restore_opts on `opts`, as start_device."""
    pay = C.byref(self.pay) if self.pay is not None else None
    if self.per_stream:
      L.check(L.lib().ct_track_restore_opts(C.byref(self.desc), pay, self._opts(opts), L.ptr(entries), n_entries,
                                            L.ptr(rows), L.ptr(payload_rows), L.stream_ptr()), 'ct_track_restore_opts')
      return
    L.check(L.lib().ct_track_restore(C.byref(self.desc), pay, L.ptr(entries), n_entries, L.ptr(rows),
                                     L.ptr(payload_rows), L.stream_ptr()), 'ct_track_restore')

  def public_buffers(self):
    """Zeroed device buffers of the shape step() takes with --public_det: public_ct [B,P,2] fp32, public_n [B] int32."""
    return (torch.zeros((self.B, self.max_public, 2), dtype=torch.float32, device=self.device),
            torch.zeros((self.B,), dtype=torch.int32, device=self.device))

  def step(self, records, public_ct=None, public_n=None, steps=None, opts=None):
    """records [B,K,F] (ct_decode) -> updates tracks/counts/boxes in place, on the current stream.
    With --public_det: public_ct [B,P,2] fp32 (each stream's public detection centres, image coordinates, first
    public_n[b] rows used) and public_n [B] int32, device tensors (P = max_public_dets).  The descriptor points at
    the buffers of this call, so a CUDA graph captured around it keeps reading them.  steps: optional [B] int32
    device tensor that receives the Dijkstra search steps of each stream's Hungarian solve.  With stream_opts: one
    ct_track_step_opts on `opts` (device ct_track_opts [B], default d_opts)."""
    if self.public_det and (public_ct is None or public_n is None):
      raise ValueError('--public_det: step() needs the public detections (public_ct, public_n)')
    assert records.is_cuda and records.dtype == torch.float32 and tuple(records.shape) == (self.B, self.K, self.F)
    self.desc.records = records.data_ptr()
    if self.pay is None and not (self.per_stream or self.hungarian or self.public_det or steps is not None):
      L.check(L.lib().ct_track_step(C.byref(self.desc), L.stream_ptr()), 'ct_track_step')
      return
    a = self.assoc
    a.public_ct = a.public_n = None
    if self.public_det:
      if not (public_ct.is_cuda and public_ct.dtype == torch.float32 and public_ct.is_contiguous() and
              tuple(public_ct.shape) == (self.B, self.max_public, 2)):
        raise ValueError('public_ct must be a contiguous fp32 CUDA tensor [%d, %d, 2]' % (self.B, self.max_public))
      if not (public_n.is_cuda and public_n.dtype == torch.int32 and tuple(public_n.shape) == (self.B,)):
        raise ValueError('public_n must be an int32 CUDA tensor [%d]' % self.B)
      a.public_ct, a.public_n = public_ct.data_ptr(), public_n.data_ptr()
    if steps is not None:
      assert steps.is_cuda and steps.dtype == torch.int32 and tuple(steps.shape) == (self.B,)
    a.steps = steps.data_ptr() if steps is not None else None
    if self.per_stream:
      L.check(L.lib().ct_track_step_opts(C.byref(self.desc), C.byref(a), C.byref(self.pay) if self.pay is not None
                                         else None, self._opts(opts), None, 0, L.stream_ptr()), 'ct_track_step_opts')
    elif self.pay is not None:
      L.check(L.lib().ct_track_step_payload(C.byref(self.desc), C.byref(a), C.byref(self.pay), L.stream_ptr()),
              'ct_track_step_payload')
    else:
      L.check(L.lib().ct_track_step_assoc(C.byref(self.desc), C.byref(a), L.stream_ptr()), 'ct_track_step_assoc')

  def render(self, pre_hm):
    """pre_hm [B,1,H,W] fp32 <- splat of the current tracks (what the NEXT frame's network reads)."""
    assert pre_hm.is_cuda and pre_hm.dtype == torch.float32 and tuple(pre_hm.shape) == (self.B, 1, self.inp_h, self.inp_w)
    L.check(L.lib().ct_render_tracks(L.ptr(self.boxes), self.B * self.T, L.ptr(pre_hm), self.B, self.inp_h,
                                     self.inp_w, L.stream_ptr()), 'ct_render_tracks')

  def step_mapped(self, records, streams, public_ct=None, public_n=None, opts=None):
    """step() on a compacted batch: records [n,K,F], streams int32 [>= n] device map (image i is stream streams[i];
    < 0: a padding image, nothing is written).  Streams that are not listed keep their tables byte for byte.
    public_ct / public_n stay indexed by the stream, as in step()."""
    if self.public_det and (public_ct is None or public_n is None):
      raise ValueError('--public_det: step_mapped() needs the public detections (public_ct, public_n)')
    n = records.shape[0]
    assert records.is_cuda and records.dtype == torch.float32 and records.is_contiguous() and \
        tuple(records.shape) == (n, self.K, self.F) and 0 < n <= self.B
    assert streams.is_cuda and streams.dtype == torch.int32 and streams.numel() >= n
    d = L.TrackDesc.from_buffer_copy(self.desc)
    d.B, d.records = n, records.data_ptr()
    a = L.TrackAssoc.from_buffer_copy(self.assoc)
    a.public_ct = a.public_n = a.steps = None
    if self.public_det:
      a.public_ct, a.public_n = public_ct.data_ptr(), public_n.data_ptr()
    pay = C.byref(self.pay) if self.pay is not None else None
    if self.per_stream:
      L.check(L.lib().ct_track_step_opts(C.byref(d), C.byref(a), pay, self._opts(opts), L.ptr(streams), self.B,
                                         L.stream_ptr()), 'ct_track_step_opts')
      return
    L.check(L.lib().ct_track_step_mapped(C.byref(d), C.byref(a), pay, L.ptr(streams), self.B, L.stream_ptr()),
            'ct_track_step_mapped')

  def render_mapped(self, pre_hm, image_of):
    """render() on a compacted batch: pre_hm [n,1,H,W] fp32 <- the tracks of stream s splatted into image
    image_of[s] (int32 [B] device map; < 0 or >= n: not rendered); every image of pre_hm is zeroed first."""
    n = pre_hm.shape[0]
    assert pre_hm.is_cuda and pre_hm.dtype == torch.float32 and tuple(pre_hm.shape) == (n, 1, self.inp_h, self.inp_w)
    assert image_of.is_cuda and image_of.dtype == torch.int32 and image_of.numel() == self.B
    L.check(L.lib().ct_render_tracks_mapped(L.ptr(self.boxes), self.B * self.T, L.ptr(image_of), self.B, L.ptr(pre_hm),
                                            n, self.inp_h, self.inp_w, L.stream_ptr()), 'ct_render_tracks_mapped')

  @property
  def d2h_bytes(self):
    return self.tracks.numel() * 4 + self.counts.numel() * 4 + (self.payload.numel() * 4 if self.Wp else 0)

  def results(self, tracks_np, counts_np, payload_np=None, idle=()):
    """Host copies -> [[{score, class, ct, tracking, bbox, tracking_id, age, active}, ...] per stream], plus the payload
    fields of the head set (payload_np [B,T,Wp], needed when it has any) with the host path's shapes: hps [2J],
    dep [1], dim [3], alpha, loc [3], rot_y, velocity, nuscenes_att.  idle: streams that had no frame in that step;
    their entry is None."""
    if self.Wp and payload_np is None:
      raise ValueError('results(): this head set has payload fields (%s): pass payload_np' %
                       ', '.join(self.payload_layout))
    out = []
    for b in range(tracks_np.shape[0]):
      if b in idle:
        out.append(None)
        continue
      n = int(counts_np[b, 0])
      rows = tracks_np[b, :n]
      res = [{'score': float(r[L.CT_TRK_SCORE]), 'class': int(r[L.CT_TRK_CLASS]),
              'ct': r[L.CT_TRK_CT:L.CT_TRK_CT + 2].copy(), 'tracking': r[L.CT_TRK_TRACKING:L.CT_TRK_TRACKING + 2].copy(),
              'bbox': r[L.CT_TRK_BBOX:L.CT_TRK_BBOX + 4].copy(), 'tracking_id': int(r[L.CT_TRK_ID]),
              'age': int(r[L.CT_TRK_AGE]), 'active': int(r[L.CT_TRK_ACTIVE])} for r in rows]
      for item, q in zip(res, payload_np[b, :n] if self.Wp else ()):
        for k, (o, w) in self.payload_layout.items():
          item[k] = float(q[o]) if k in ('alpha', 'rot_y') else q[o:o + w].copy()
      out.append(res)
    return out
