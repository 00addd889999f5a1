"""Per-stream detections of runners without a tracker, post-processed on the GPU: `Detector.post_process` +
`merge_outputs` (detector.py:356-377, utils/post_process.py:21-91) as one launch on the decode records
(`ct_post_process`).  Each stream's records with score > out_thresh become rows of CT_DET_FLOATS fp32 (score,
class + 1, ct, tracking, bbox) in its source pixels -- the first columns of DeviceTracker's track rows, computed by the
same device code -- and, on pose, 3D, velocity and attribute head sets, payload rows beside them with the fields
generic_post_process adds (hps, dep, dim, alpha, loc, rot_y, velocity, nuscenes_att); on 3D head sets `ct` is the
amodal centre, as in the reference.  `results()` turns host copies into the reference's list of dicts.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib as L
from .device_tracker import POST_OPTION_KEYS, DeviceTracker, default_geometry, opts_records, payload_layout, \
    resolve_options


class DeviceDetections(object):
  """The device tables of one runner's post-processed detections: dets [B,K,CT_DET_FLOATS], counts [B], the optional
  payload [B,K,Wp], and each stream's camera geometry (trans_out_inv [B,6], calib [B,3,4] on 3D head sets), built as
  DeviceTracker builds its own."""

  # the camera rows are DeviceTracker's: same (c, s) -> affine and default calib arithmetic
  _trans_rows = DeviceTracker._trans_rows
  _calibs = DeviceTracker._calibs
  geometry_rows = DeviceTracker.geometry_rows

  opts_bytes = DeviceTracker.opts_bytes
  _opts = DeviceTracker._opts

  def __init__(self, opt, B, K, rec_floats, layout, inp_h, inp_w, device, centers=None, scales=None, calibs=None,
               stream_opts=None):
    """centers/scales: per-stream (c, s) of the source rectangle; default = a source image of exactly the network
    input size.  calibs: per-stream [3,4] camera matrices for the 3D head sets (loc, rot_y); default as
    DeviceTracker's.  stream_opts: None, or B entries, each None (opt) or {'out_thresh': v}, the threshold stream b
    keeps its records above (ct_post_process_opts on the device records d_opts)."""
    self.per_stream = stream_opts is not None
    if self.per_stream and len(stream_opts) != B:
      raise ValueError('stream_opts: expected %d entries (one per stream, None or a dict), got %d' %
                       (B, len(stream_opts)))
    self.options = [resolve_options(opt, f, POST_OPTION_KEYS, 'stream_opts[%d]' % b)
                    for b, f in enumerate(stream_opts if self.per_stream else [None] * B)]
    self.opt, self.B, self.K, self.F = opt, B, K, rec_floats
    self.inp_h, self.inp_w = inp_h, inp_w
    self.device = torch.device(device)
    c0, s0 = default_geometry(inp_h, inp_w)
    _, t_out = self._trans_rows([c0 if centers is None else centers[b] for b in range(B)],
                                [s0 if scales is None else scales[b] for b in range(B)])
    self.trans_out_inv = torch.from_numpy(t_out).to(self.device)
    self.dets = torch.zeros((B, K, L.CT_DET_FLOATS), dtype=torch.float32, device=self.device)
    self.counts = torch.zeros((B,), dtype=torch.int32, device=self.device)
    self.has_tracking = 'tracking' in layout
    d = L.DetDesc()
    d.K, d.F = K, rec_floats
    d.rec_tracking = layout['tracking'][0] if self.has_tracking else -1
    d.out_thresh = float(opt.out_thresh)
    d.trans_out_inv, d.dets, d.counts = self.trans_out_inv.data_ptr(), self.dets.data_ptr(), self.counts.data_ptr()
    self.desc = d
    self.payload_layout = payload_layout(layout)
    self.Wp = sum(w for _, w in self.payload_layout.values())
    self.payload = self.calib = self.pay = None
    if self.Wp:
      self.payload = torch.zeros((B, K, self.Wp), dtype=torch.float32, device=self.device)
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
    self.d_opts = None
    if self.per_stream:
      self.d_opts = torch.frombuffer(bytearray(self.opts_bytes()), dtype=torch.uint8).to(self.device)

  def check_options(self, flags, what='options', resolved=False):
    """A stream's new setting ({'out_thresh': v}, or resolved as a StreamState carries it) -> the resolved setting;
    ValueError for another key, a bad value, or a runner built without stream_opts."""
    if not self.per_stream:
      raise ValueError('%s: this runner was built without stream_opts: its streams all run opt (build it with '
                       'stream_opts to give streams their own out_thresh)' % what)
    return dict(flags) if resolved else resolve_options(self.opt, flags, POST_OPTION_KEYS, what)

  def set_geometry(self, streams, rows_in, rows_out):
    """trans_out_inv (and calib on 3D head sets) of `streams` <- rows_out (geometry_rows, device tensors), on the
    current stream, as DeviceTracker.set_geometry (rows_in, the input affine, is not read here)."""
    for i, b in enumerate(streams):
      self.trans_out_inv[b].copy_(rows_out[i, :6])
      if self.calib is not None:
        self.calib[b].view(12).copy_(rows_out[i, 6:])

  def _launch(self, records, streams, opts=None):
    n = records.shape[0]
    assert records.is_cuda and records.dtype == torch.float32 and records.is_contiguous() and \
        tuple(records.shape) == (n, self.K, self.F) and 0 < n <= self.B
    self.desc.n, self.desc.records = n, records.data_ptr()
    pay = C.byref(self.pay) if self.pay is not None else None
    if self.per_stream:
      L.check(L.lib().ct_post_process_opts(C.byref(self.desc), pay, self._opts(opts), L.ptr(streams), self.B,
                                           L.stream_ptr()), 'ct_post_process_opts')
      return
    L.check(L.lib().ct_post_process(C.byref(self.desc), pay, L.ptr(streams), self.B, L.stream_ptr()),
            'ct_post_process')

  def step(self, records, opts=None):
    """records [B,K,F] (ct_decode) -> dets, counts (and payload) of every stream, on the current stream.  The
    descriptor points at the buffers of this call, so a CUDA graph captured around it keeps reading them.  With
    stream_opts: on `opts` (device ct_track_opts [B], default d_opts)."""
    self._launch(records, None, opts)

  def step_mapped(self, records, streams, opts=None):
    """step() on a compacted batch: records [n,K,F], streams int32 [>= n] device map (image i is stream streams[i];
    < 0: a padding image, nothing is written).  Streams that are not listed keep their rows byte for byte."""
    assert streams.is_cuda and streams.dtype == torch.int32 and streams.numel() >= records.shape[0]
    self._launch(records, streams, opts)

  @property
  def d2h_bytes(self):
    return self.dets.numel() * 4 + self.counts.numel() * 4 + (self.payload.numel() * 4 if self.Wp else 0)

  def results(self, dets_np, counts_np, payload_np=None, idle=()):
    """Host copies -> [[{score, class, ct, tracking, bbox}, ...] per stream] as Detector.post_process + merge_outputs
    give them (tracking only when the head set has it), plus the payload fields of the head set (payload_np [B,K,Wp],
    needed when it has any) with the host path's shapes: hps [2J], dep [1], dim [3], alpha, loc [3], rot_y, velocity,
    nuscenes_att.  idle: streams that had no frame in that step; their entry is None.  Each field is copied once per
    stream, and the items hold views of those copies (or Python scalars), never of the arrays passed in."""
    if self.Wp and payload_np is None:
      raise ValueError('results(): this head set has payload fields (%s): pass payload_np' %
                       ', '.join(self.payload_layout))
    out = []
    for b in range(dets_np.shape[0]):
      if b in idle:
        out.append(None)
        continue
      n = int(counts_np[b])
      rows = dets_np[b, :n]
      cols = {'score': rows[:, L.CT_TRK_SCORE].tolist(), 'class': rows[:, L.CT_TRK_CLASS].astype(np.int64).tolist(),
              'ct': rows[:, L.CT_TRK_CT:L.CT_TRK_CT + 2].copy()}
      if self.has_tracking:
        cols['tracking'] = rows[:, L.CT_TRK_TRACKING:L.CT_TRK_TRACKING + 2].copy()
      cols['bbox'] = rows[:, L.CT_TRK_BBOX:L.CT_TRK_BBOX + 4].copy()
      if self.Wp:
        q = payload_np[b, :n]
        for k, (o, w) in self.payload_layout.items():
          cols[k] = q[:, o].tolist() if k in ('alpha', 'rot_y') else q[:, o:o + w].copy()
      keys = list(cols)
      out.append([dict(zip(keys, vals)) for vals in zip(*(cols[k] for k in keys))])
    return out
