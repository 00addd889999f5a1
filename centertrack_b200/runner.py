"""StreamRunner: the batched, graph-captured form of `Detector.run`'s device half for B independent video streams
on one GPU (SURVEY 8e: streams shard across GPUs, replicas of the weights, no data-path collective).

One step = for every stream its current frame: network (pre_img = that stream's previous frame, kept on
the device exactly like detector.py:148) + fused sigmoid + fused decode -> one packed record buffer
[B,K,F].  THREE input slots rotate: step t reads slot t%3 (images) and slot (t-1)%3 (pre_images: the previous
step's images, never copied) while the copy stream uploads step t+1's frames into slot (t+1)%3 -- with two slots
the upload would have to wait for the step that still reads its target as pre_images.  One CUDA graph per slot
replays the whole step as a single launch.  The FIRST step of a stream uses the frame itself as pre_images
(detector.py:99-103).

Two ways to feed the prior heat-map (`--pre_hm`):
  * device_tracking=False: the caller supplies pre_hm per step (what Detector._get_additional_inputs renders on the
    host).  With the one-step software pipeline of `step_host` the caller cannot have seen records(t-1) when it
    submits step t, so a host-rendered pre_hm is necessarily one frame stale -- this mode is for detection-style
    pipelines and for measuring the hot path with given inputs.
  * device_tracking=True (SURVEY 8f-1): the reference's dependency chain closed ON THE DEVICE, inside the same graph:
        pre_hm(t) = splat(tracks(t-1))  ->  network + decode -> records(t)  ->  tracks(t) = Tracker.step(records(t))
    (`DeviceTracker`: ct_render_tracks, ct_track_step).  Exact reference semantics (no stale prior), no host round
    trip; the host uploads only the frame and downloads the track table (ids, boxes, ages), and for pose / 3D head sets
    the payload table beside it (hps, dep, dim, alpha, loc, rot_y, velocity, nuscenes_att).  Every association mode
    of the host Tracker runs there: greedy, `--hungarian`, and `--public_det`, whose public detections (the `ct`s of
    each frame's provided detections) are staged per input slot like the frames and uploaded with them.

The end-to-end form (`step_host`) takes HOST frames: pinned staging, H2D on a copy stream overlapped
with the previous step's compute, graph replay, D2H of the records (and tracks).

Frames mode (`frame_sizes`, `step_frames`) takes the raw uint8 BGR camera frames instead, one source size per stream:
the three slots hold the B frames ragged (16-byte aligned offsets) in pinned and device memory, and the step warps and
normalises them on the device exactly as Detector.pre_process_device does (cv2's fixed-point bilinear).  On the bf16
engine ct_pack_stem_frames writes the stem's packed bf16 input straight from slot t (images) and slot t-1 (pre_images,
warped again: no fp32 copy is kept); the fp32 and bf16x3 engines warp each stream into the fp32 image slot with
ct_warp_affine_normalize and run their plan unchanged.  The tracker gets each stream's (c, s) and default calib, so
tracks, public detections and 3D boxes are in that camera's pixels.

Video starts (`starts=`, `pre_dets=` of step_host / step_frames / load_device_inputs): a stream may begin a new video at
any step, as Detector.reset_tracking + Tracker.init_track(pre_dets) on that stream alone.  A start is rare (once per
video), so it is not in the graphs: a step that carries starts first runs a short prologue on the compute stream -- the
started streams' frames copied into the previous slot (their pre_images), then ct_track_start (reset, seeds, render
boxes) -- and then replays the same graph as any other step.  Steps without starts run exactly what they ran before.

Flip test (`opt.flip_test`, detector.py:225-226,285-286,311-332): the network runs on 2B images, the streams' frames
[0, B) and their mirrors [B, 2B), inside the same step.  pre_images is the previous step's 2B images, so the previous
frame's mirror comes free (detector.py:148).  Uploads, the device tracker's render and a caller's pre_hm fill the first
B images; ct_mirror_x writes the second half in the graph, or, in frames mode on the bf16 engine,
ct_pack_stem_frames_flip stores every packed pixel at its mirrored position too.  One ct_flip_merge_heads launch
averages the flipped heads into [B] buffers; decode and tracking then run at B on those and on the first half of the
other heads.  Records, tracks, uploads and downloads are the same size as without the flip.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib as L
from .dataset_info import get_dataset
from .decode import generic_decode
from .detector import default_calib, flip_output, flip_plan, frame_geometry
from .device_tracker import DeviceTracker, plan_starts


NS = 3          # input slots


class StreamRunner(object):

  def __init__(self, model, B, H, W, K=100, precision='bf16', device='cuda', use_graph=True, opt=None,
               device_tracking=False, max_public_dets=512, calibs=None, frame_sizes=None):
    """max_public_dets: with device_tracking and --public_det, the most public detections a stream may bring per
    frame (more raise ValueError; none is ever dropped).  calibs: with device_tracking on a 3D head set, one [3,4]
    camera matrix per stream (DeviceTracker's default otherwise; in frames mode Detector._get_default_calib of the
    stream's source size).  frame_sizes: B (height, width) source sizes, fixed for the runner's lifetime, to feed raw
    uint8 frames with step_frames; each must map to the network input (H, W) under opt's resolution policy
    (ValueError otherwise).  opt.flip_test: every stream's frame runs with its mirror (2B images per step) and the
    averaged heads are merged before decode, as Detector.process does; inputs and outputs keep their B shapes."""
    self.B, self.H, self.W, self.K = B, H, W, K
    self.device = torch.device(device)
    self.model = model
    self.opt = opt if opt is not None else getattr(model, 'opt', None)
    self.frames_mode = frame_sizes is not None
    if self.frames_mode:
      calibs = self._frame_geometry(frame_sizes, calibs)
    self.flip = bool(getattr(self.opt, 'flip_test', False))
    NB = 2 * B if self.flip else B                           # --flip_test: frames [0, B), their mirrors [B, 2B)
    self.eng = model.engine_for(NB, H, W, self.device, precision)
    self.eng.set_fused_activations(True)
    f32 = torch.float32
    self.img = [torch.zeros((NB, 3, H, W), dtype=f32, device=self.device) for _ in range(NS)]
    self.hm = [torch.zeros((NB, 1, H, W), dtype=f32, device=self.device) for _ in range(NS)]
    if self.flip:                                            # the averaged heads, merged per stream
      self.flip_plan = flip_plan(self.eng.outputs, get_dataset(self.opt.dataset).flip_idx, self.device)
      self.merged = {h: torch.zeros((B,) + tuple(self.eng.outputs[h].shape[1:]), dtype=f32, device=self.device)
                     for h in self.flip_plan}
    self._pack_mirror = self.flip and self.frames_mode and self.eng.use_halo   # the flip pack writes the mirrors
    self.h_img = [torch.zeros((B, 3, H, W), dtype=f32).pin_memory() for _ in range(NS)]
    self.h_hm = [torch.zeros((B, 1, H, W), dtype=f32).pin_memory() for _ in range(NS)]
    if self.frames_mode:      # frame slots: B uint8 frames at 16-byte aligned offsets, pinned staging + device
      self.u8 = [torch.zeros(self.slot_bytes, dtype=torch.uint8, device=self.device) for _ in range(NS)]
      self.h_u8 = [torch.zeros(self.slot_bytes, dtype=torch.uint8).pin_memory() for _ in range(NS)]
      self.minv = torch.from_numpy(np.stack([f.minv[:] for f in self.frames])).to(self.device)
    self.rec = None
    self.layout = None
    self.ws = None                                           # private decode workspace (captured by the graphs)
    self.use_graph = use_graph
    self.graphs = [None] * NS
    self.compute = torch.cuda.Stream(device=self.device)
    self.copy = torch.cuda.Stream(device=self.device)
    self.ev_in = [torch.cuda.Event() for _ in range(NS)]     # slot uploaded
    self.ev_done = [torch.cuda.Event() for _ in range(NS)]   # slot no longer read (neither as images nor pre_images)
    self.t = 0
    self.tracker = None
    self.device_tracking = device_tracking
    self._starts = [None] * NS                               # per slot: the streams whose frame starts a video
    self._start_bytes = 0                                    # start list + seed rows uploaded by the last step
    self.h_start = None                                      # per slot start list / seed staging, made on first use
    self._eager(0, first=True)                               # sizes the record buffer
    if device_tracking:
      assert self.opt is not None, 'device tracking needs opt (thresholds, max_age)'
      geo = {}
      if self.frames_mode:
        geo = dict(centers=[m['c'] for m in self._meta], scales=[m['s'] for m in self._meta])
      self.tracker = DeviceTracker(self.opt, B, K, self.rec.shape[2], self.layout, H, W, self.device,
                                   max_public_dets=max_public_dets, calibs=calibs, **geo)
    self.public = self.tracker is not None and self.tracker.public_det
    if self.public:                                          # per slot: device (public_ct, public_n) + pinned staging
      self.pub = [self.tracker.public_buffers() for _ in range(NS)]
      self.h_pub = [tuple(t.cpu().pin_memory() for t in p) for p in self.pub]
    torch.cuda.synchronize(self.device)
    self.h_rec = [torch.zeros_like(self.rec, device='cpu').pin_memory() for _ in range(2)]
    if self.tracker is not None:
      self.h_trk = [torch.zeros_like(self.tracker.tracks, device='cpu').pin_memory() for _ in range(2)]
      self.h_cnt = [torch.zeros_like(self.tracker.counts, device='cpu').pin_memory() for _ in range(2)]
      if self.tracker.payload is not None:
        self.h_pay = [torch.zeros_like(self.tracker.payload, device='cpu').pin_memory() for _ in range(2)]
    # launches of one step: the network plan + decode (+ memset-free: render + track step); frames mode: the pack op
    # becomes ct_pack_stem_frames (one launch per CT_FRAMES_PER_LAUNCH streams), or B warps come before the plan.
    # --flip_test: + the merge, + the mirrors of the images and pre_hm unless the flip pack writes them
    self.launches_per_step = self.eng.n_launches + 1 + (2 if device_tracking else 0)
    if self.frames_mode:
      self.launches_per_step += (-(-B // L.CT_FRAMES_PER_LAUNCH) - 1) if self.eng.use_halo else B
    if self.flip:
      self.launches_per_step += 1 + (0 if self._pack_mirror else 1 + int(self.eng.has_pre_hm))

  def _frame_geometry(self, frame_sizes, calibs):
    """Per-stream geometry of frames mode (Detector.pre_process_device's, through detector.frame_geometry): the
    ct_frame descriptors, the metas, the slot size.  -> the tracker's calibs."""
    opt, B = self.opt, self.B
    if opt is None:
      raise ValueError('frames mode needs opt (the resolution policy and the dataset mean / std)')
    if len(frame_sizes) != B:
      raise ValueError('frame_sizes: expected %d (height, width) pairs, got %d' % (B, len(frame_sizes)))
    if calibs is not None:
      calibs = np.asarray(calibs, np.float32)
      if calibs.shape != (B, 3, 4):
        raise ValueError('calibs: expected %d camera matrices [3, 4], got shape %s' % (B, calibs.shape))
    ds = get_dataset(opt.dataset)
    focal = opt.test_focal_length if getattr(opt, 'test_focal_length', -1) >= 0 else ds.rest_focal_length
    self.mean = np.ascontiguousarray(ds.mean, dtype=np.float32).reshape(3)
    self.std = np.ascontiguousarray(ds.std, dtype=np.float32).reshape(3)
    self.frames = (L.Frame * B)()
    self._meta = []
    off = 0
    for b, (h, w) in enumerate(frame_sizes):
      h, w = int(h), int(w)
      if h <= 0 or w <= 0:
        raise ValueError('frame_sizes[%d]: bad size %s' % (b, (h, w)))
      meta, minv = frame_geometry(opt, h, w)
      if (meta['inp_height'], meta['inp_width']) != (self.H, self.W):
        raise ValueError('frame_sizes[%d] = %s maps to a %dx%d network input under this resolution policy, not the '
                         "runner's %dx%d" % (b, (h, w), meta['inp_height'], meta['inp_width'], self.H, self.W))
      meta['calib'] = calibs[b] if calibs is not None else default_calib(focal, w, h)
      self._meta.append(meta)
      f = self.frames[b]
      f.offset, f.h, f.w, f.step = off, h, w, 3 * w
      f.minv[:] = minv.tolist()
      off += (h * w * 3 + 15) // 16 * 16
    self.frame_sizes = [(int(h), int(w)) for h, w in frame_sizes]
    self.slot_bytes = off
    return calibs if calibs is not None else np.stack([m['calib'] for m in self._meta]).astype(np.float32)

  def meta(self, b):
    """Frames mode: the meta dict Detector.pre_process returns for stream b's frames (c, s, sizes, trans_input,
    trans_output, calib) -- what generic_post_process needs when the records are post-processed on the host."""
    if not self.frames_mode:
      raise ValueError('meta(): the runner was not built with frame_sizes')
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in self._meta[b].items()}

  # one step, eager launches on the current stream
  def _eager(self, slot, first=False):
    if self.tracker is not None:
      self.tracker.render(self.hm[slot][:self.B])            # pre_hm(t) from tracks(t-1)
    prev = slot if first else (slot - 1) % NS
    if self.frames_mode and self.eng.use_halo:
      eng = self.eng
      pack = L.lib().ct_pack_stem_frames_flip if self.flip else L.lib().ct_pack_stem_frames
      L.check(pack(
          L.ptr(self.u8[slot]), L.ptr(self.u8[prev] if eng.has_pre_img else None), self.frames, self.B,
          C.c_void_p(self.mean.ctypes.data), C.c_void_p(self.std.ctypes.data),
          L.ptr(self.hm[slot] if eng.has_pre_hm else None), L.ptr(eng.stem_input), self.H, self.W, L.stream_ptr()),
          'ct_pack_stem_frames')
      out = dict(eng.forward_packed(eng.has_pre_img, eng.has_pre_hm))
    else:
      if self.frames_mode:
        self._warp_frames(slot)
      if self.flip:                  # the mirrored half; pre_images (img[prev]) was mirrored by its own step
        self._mirror(self.img[slot], 0, self.B)
        if self.eng.has_pre_hm:
          self._mirror(self.hm[slot], 0, self.B)
      out = dict(self.eng.forward(self.img[slot], self.img[prev], self.hm[slot]))
    if self.flip:
      out = flip_output(out, self.flip_plan, self.merged)
    if self.ws is None:
      cat = out['hm'].shape[1]
      J = out['hm_hp'].shape[1] if ('hm_hp' in out and 'hps' in out) else 0
      self.ws = torch.zeros(L.lib().ct_decode_workspace_bytes(self.B, cat, J, self.K), dtype=torch.uint8,
                            device=self.device)
    res = generic_decode(out, K=self.K, records_out=self.rec, workspace=self.ws)
    if self.rec is None:
      self.rec, self.layout = res.records, res.layout
    if self.tracker is not None:
      self.tracker.step(self.rec, *(self.pub[slot] if self.public else ()))    # tracks(t)
    return res

  def _mirror(self, x, b, n):
    """--flip_test: x[B+b : B+b+n] <- x[b : b+n] mirrored along W (ct_mirror_x), on the current stream."""
    _, c, h, w = x.shape
    L.check(L.lib().ct_mirror_x(L.ptr(x[b]), L.ptr(x[self.B + b]), n, c, h, w, L.stream_ptr()), 'ct_mirror_x')

  def _warp_frames(self, slot):
    """fp32 and bf16x3 engines: the slot's frames -> its fp32 image, one ct_warp_affine_normalize per stream."""
    lib, st = L.lib(), L.stream_ptr()
    src, dst = self.u8[slot].data_ptr(), self.img[slot]
    for b, f in enumerate(self.frames):
      L.check(lib.ct_warp_affine_normalize(C.c_void_p(src + f.offset), 1, f.h, f.w, f.step, L.ptr(self.minv[b]),
                                           C.c_void_p(self.mean.ctypes.data), C.c_void_p(self.std.ctypes.data),
                                           L.ptr(dst[b]), self.H, self.W, st), 'ct_warp_affine_normalize')

  def _graph(self, slot):
    if self.graphs[slot] is None:
      saved = None
      if self.tracker is not None:                           # capture must not disturb live stream state
        saved = [t.clone() for t in self._tracker_state()]
      s = torch.cuda.Stream(device=self.device)
      s.wait_stream(torch.cuda.current_stream())
      with torch.cuda.stream(s):
        self._eager(slot)
      torch.cuda.current_stream().wait_stream(s)
      g = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g):
        self._eager(slot)
      self.graphs[slot] = g
      if saved is not None:
        for t, v in zip(self._tracker_state(), saved):
          t.copy_(v)
    return self.graphs[slot]

  def _tracker_state(self):
    trk = self.tracker
    return [trk.tracks, trk.counts, trk.boxes] + ([trk.payload] if trk.payload is not None else [])

  def warm(self):
    for s in range(NS):
      if self.use_graph:
        self._graph(s)
      else:
        self._eager(s)
    if self.tracker is not None:
      self.tracker.reset()
    torch.cuda.synchronize(self.device)

  def reset_tracking(self):
    self.t = 0
    if self.tracker is not None:
      self.tracker.reset()

  def _check_public(self, public_dets):
    """public_dets: list of B arrays [P_b, 2] (the `ct` of each of the frame's public detections, image coordinates)
    -> list of B float32 arrays; ValueError when they are missing, unexpected, or more than max_public_dets."""
    if not self.public:
      if public_dets is not None:
        raise ValueError('public detections are only read by device tracking with --public_det')
      return None
    if public_dets is None:
      raise ValueError('--public_det: every step needs the public detections of its frames (public_dets)')
    if len(public_dets) != self.B:
      raise ValueError('public_dets: expected %d arrays (one per stream), got %d' % (self.B, len(public_dets)))
    out = []
    for b, p in enumerate(public_dets):
      a = np.asarray(p, np.float32)
      if a.size == 0:
        a = a.reshape(0, 2)
      if a.ndim != 2 or a.shape[1] != 2:
        raise ValueError('public_dets[%d]: expected [P, 2] centres, got shape %s' % (b, a.shape))
      if a.shape[0] > self.tracker.max_public:
        raise ValueError('public_dets[%d]: %d public detections, more than max_public_dets = %d' %
                         (b, a.shape[0], self.tracker.max_public))
      out.append(a)
    return out

  def _fill_public(self, dst, pub):
    ct, n = dst
    ct.zero_()
    for b, a in enumerate(pub):
      ct[b, :len(a)] = torch.from_numpy(a)
      n[b] = len(a)

  def _check_starts(self, starts, pre_dets):
    """starts (stream indices whose frame in this step is a video's first) and pre_dets ({stream: list of result
    dicts} seeding the tracker of some of them, in each stream's source pixels like the tracks) -> (streams, seed rows)
    or None.  ValueError (device_tracker.plan_starts) before anything is enqueued; without device tracking a start only
    switches pre_images, and pre_dets are refused."""
    if starts is None or len(starts) == 0:
      if pre_dets:
        raise ValueError('pre_dets: stream(s) %s do not start a video in this step' % sorted(pre_dets))
      return None
    if self.tracker is None:
      if pre_dets:
        raise ValueError('pre_dets seed the device tracker: this runner was built without device_tracking')
      return plan_starts(self.B, 0, 0.0, False, starts, None)
    trk = self.tracker
    return plan_starts(self.B, trk.T, self.opt.new_thresh, trk.payload is not None, starts, pre_dets)

  def _stage_starts(self, slot, plan):
    """The pinned staging of slot's start list (stream, seeds) and seed rows <- plan; -> (entries, seed rows).  The
    staging was last read by the upload of step t-3, which the last fetch() waited for."""
    if self.h_start is None:
      T = self.tracker.T
      self.h_start = [torch.zeros((self.B, 2), dtype=torch.int32).pin_memory() for _ in range(NS)]
      self.h_seed = [torch.zeros((self.B * T, L.CT_TRK_FLOATS), dtype=torch.float32).pin_memory() for _ in range(NS)]
      self.d_start = [torch.zeros((self.B, 2), dtype=torch.int32, device=self.device) for _ in range(NS)]
      self.d_seed = [torch.zeros((self.B * T, L.CT_TRK_FLOATS), dtype=torch.float32, device=self.device)
                     for _ in range(NS)]
    streams, seeds = plan
    n = 0
    for e, (s, rows) in enumerate(zip(streams, seeds)):
      self.h_start[slot][e, 0], self.h_start[slot][e, 1] = s, len(rows)
      self.h_seed[slot][n:n + len(rows)] = torch.from_numpy(rows)
      n += len(rows)
    return len(streams), n

  def _upload_starts(self, slot, plan, non_blocking):
    """Stages and uploads one step's starts for slot (the current stream is the upload's); -> the bytes uploaded."""
    self._starts[slot] = None
    if plan is None:
      return 0
    self._starts[slot] = plan[0]
    if self.tracker is None:
      return 0
    e, n = self._stage_starts(slot, plan)
    self.d_start[slot][:e].copy_(self.h_start[slot][:e], non_blocking=non_blocking)
    if n:
      self.d_seed[slot][:n].copy_(self.h_seed[slot][:n], non_blocking=non_blocking)
    return e * 8 + n * L.CT_TRK_FLOATS * 4

  def load_device_inputs(self, images, pre_hms, slot, public_dets=None, starts=None, pre_dets=None):
    """Copies step_device's inputs into `slot` on the current stream; starts / pre_dets as in step_host."""
    pub = self._check_public(public_dets)
    plan = self._check_starts(starts, pre_dets)
    self.img[slot][:self.B].copy_(images)
    if pre_hms is not None:
      self.hm[slot][:self.B].copy_(pre_hms)
    if pub is not None:
      self._fill_public(self.h_pub[slot], pub)
      self.pub[slot][0].copy_(self.h_pub[slot][0])
      self.pub[slot][1].copy_(self.h_pub[slot][1])
    self._start_bytes = self._upload_starts(slot, plan, non_blocking=False)

  def _start_prologue(self, slot, streams):
    """A step whose frames start new videos on `streams`, before the step itself (graph replay or eager), on the same
    stream: first-frame pre_images and the tracker start.  Outside the graphs: they stay the same for every step."""
    if self.t > 0:
      # pre_images of a started stream = its own frame: overwrite its part of the previous slot, which holds step t-1's
      # images.  Safe: that slot is read only by this step (as pre_images), after this prologue on the same stream, and
      # it is next written by the upload of step t+2, which waits for ev_done[prev], recorded after this step.
      prev = (slot - 1) % NS
      for b in streams:
        if self.frames_mode and self.eng.use_halo:          # the pack kernel warps (and mirrors) u8[prev] again
          f = self.frames[b]
          o, n = f.offset, f.h * f.w * 3
          self.u8[prev][o:o + n].copy_(self.u8[slot][o:o + n])
          continue
        if self.frames_mode:                                 # the plan reads img[prev]: warp this frame into it
          f = self.frames[b]
          L.check(L.lib().ct_warp_affine_normalize(
              C.c_void_p(self.u8[slot].data_ptr() + f.offset), 1, f.h, f.w, f.step, L.ptr(self.minv[b]),
              C.c_void_p(self.mean.ctypes.data), C.c_void_p(self.std.ctypes.data), L.ptr(self.img[prev][b]), self.H,
              self.W, L.stream_ptr()), 'ct_warp_affine_normalize')
        else:
          self.img[prev][b].copy_(self.img[slot][b])
        if self.flip:                                        # --flip_test: pre_images is the (frame, mirror) pair
          self._mirror(self.img[prev], b, 1)
    if self.tracker is not None:                             # reset + seeds + boxes: the step's render splats them
      self.tracker.start_device(self.d_start[slot], len(streams), self.d_seed[slot])

  def _launch(self, slot):
    streams, self._starts[slot] = self._starts[slot], None
    if streams:
      self._start_prologue(slot, streams)
    if self.t == 0:
      self._eager(slot, first=True)                          # first frame of the streams: pre_images = images
    elif self.use_graph:
      self._graph(slot).replay()
    else:
      self._eager(slot)

  def step_device(self):
    """Inputs already resident in the slot buffers; runs on the current stream."""
    slot = self.t % NS
    self._launch(slot)
    self.t += 1
    return self.rec

  def step_host(self, images, pre_hms=None, public_dets=None, starts=None, pre_dets=None):
    """images [B,3,H,W] (and pre_hms [B,1,H,W] unless device_tracking): float32 HOST tensors (what
    Detector.pre_process / _get_additional_inputs produce); with --public_det, public_dets = B arrays [P_b, 2] (the
    `ct`s of each frame's public detections).  starts: the streams whose frame in this step is a new video's first
    (Detector.reset_tracking on those streams alone: the frame is its own pre_images and the stream's tracker restarts
    empty, or from pre_dets = {stream: list of result dicts} as Tracker.init_track; the other streams are unaffected).
    Returns the records of the PREVIOUS call (None the first time) -- a one-step software pipeline: this step's H2D
    overlaps the previous step's compute."""
    pub = self._check_public(public_dets)
    plan = self._check_starts(starts, pre_dets)
    slot = self.t % NS
    if pub is not None:        # the slot's staging was last read by step t-3's upload, which the last fetch() waited for
      self._fill_public(self.h_pub[slot], pub)
    use_hm = self.tracker is None and pre_hms is not None
    src_img, src_hm = images, pre_hms
    if not images.is_pinned() or (use_hm and not pre_hms.is_pinned()):   # pageable input: stage through pinned memory
      self.h_img[slot].copy_(images)
      src_img = self.h_img[slot]
      if use_hm:
        self.h_hm[slot].copy_(pre_hms)
        src_hm = self.h_hm[slot]
    with torch.cuda.stream(self.copy):
      self.copy.wait_event(self.ev_done[slot])       # slot's old contents were last read as pre_images of step t-2
      self.img[slot][:self.B].copy_(src_img, non_blocking=True)
      if use_hm:
        self.hm[slot][:self.B].copy_(src_hm, non_blocking=True)
      if pub is not None:
        self.pub[slot][0].copy_(self.h_pub[slot][0], non_blocking=True)
        self.pub[slot][1].copy_(self.h_pub[slot][1], non_blocking=True)
      self._start_bytes = self._upload_starts(slot, plan, non_blocking=True)
      self.ev_in[slot].record(self.copy)
    return self._submit(slot)

  def _submit(self, slot):
    """The step of the uploaded slot on the compute stream and the D2H of its results; -> the previous step's
    records."""
    prev = self.fetch() if self.t > 0 else None
    with torch.cuda.stream(self.compute):
      self.compute.wait_event(self.ev_in[slot])
      self._launch(slot)
      self.h_rec[self.t & 1].copy_(self.rec, non_blocking=True)
      if self.tracker is not None:
        self.h_trk[self.t & 1].copy_(self.tracker.tracks, non_blocking=True)
        self.h_cnt[self.t & 1].copy_(self.tracker.counts, non_blocking=True)
        if self.tracker.payload is not None:
          self.h_pay[self.t & 1].copy_(self.tracker.payload, non_blocking=True)
      # this step's pre_images slot may be overwritten once this step is done
      self.ev_done[(slot - 1) % NS].record(self.compute)
    self.t += 1
    return prev

  def frame_buffers(self):
    """Frames mode: numpy views [h_b, w_b, 3] uint8 of the pinned staging the NEXT step_frames uploads, one per stream,
    for a decoder to write its frames in place; then call step_frames(None).  They may be written once the previous
    step_frames call has returned (its upload of three steps ago, which last read this staging, has completed by
    then) and until the next step_frames call."""
    if not self.frames_mode:
      raise ValueError('frame_buffers(): the runner was not built with frame_sizes')
    buf = self.h_u8[self.t % NS].numpy()
    return [buf[f.offset:f.offset + f.h * f.w * 3].reshape(f.h, f.w, 3) for f in self.frames]

  def step_frames(self, frames, pre_hms=None, public_dets=None, starts=None, pre_dets=None):
    """frames: B uint8 [h_b, w_b, 3] BGR arrays of the sizes given as frame_sizes, or None when they were written
    through frame_buffers().  pre_hms, public_dets, starts, pre_dets and the return value as in step_host; public
    detections and pre_dets are in each stream's source pixels, and so are the tracks.  ValueError on a wrong count,
    dtype or shape, or when the runner was not built with frame_sizes."""
    if not self.frames_mode:
      raise ValueError('step_frames: the runner was not built with frame_sizes (use step_host)')
    pub = self._check_public(public_dets)
    plan = self._check_starts(starts, pre_dets)
    slot = self.t % NS
    if frames is not None:
      if len(frames) != self.B:
        raise ValueError('frames: expected %d arrays (one per stream), got %d' % (self.B, len(frames)))
      for b, (a, (h, w)) in enumerate(zip(frames, self.frame_sizes)):
        if not isinstance(a, np.ndarray) or a.dtype != np.uint8:
          raise ValueError('frames[%d]: expected a uint8 numpy array, got %s' %
                           (b, getattr(a, 'dtype', type(a).__name__)))
        if a.shape != (h, w, 3):
          raise ValueError('frames[%d]: expected shape %s, got %s' % (b, (h, w, 3), a.shape))
      # the slot's staging was last read by step t-3's upload, which the last fetch() waited for
      for a, v in zip(frames, self.frame_buffers()):
        np.copyto(v, a)
    if pub is not None:
      self._fill_public(self.h_pub[slot], pub)
    use_hm = self.tracker is None and pre_hms is not None
    src_hm = pre_hms
    if use_hm and not pre_hms.is_pinned():
      self.h_hm[slot].copy_(pre_hms)
      src_hm = self.h_hm[slot]
    with torch.cuda.stream(self.copy):
      self.copy.wait_event(self.ev_done[slot])       # slot's old contents were last read as pre_images of step t-2
      self.u8[slot].copy_(self.h_u8[slot], non_blocking=True)
      if use_hm:
        self.hm[slot][:self.B].copy_(src_hm, non_blocking=True)
      if pub is not None:
        self.pub[slot][0].copy_(self.h_pub[slot][0], non_blocking=True)
        self.pub[slot][1].copy_(self.h_pub[slot][1], non_blocking=True)
      self._start_bytes = self._upload_starts(slot, plan, non_blocking=True)
      self.ev_in[slot].record(self.copy)
    return self._submit(slot)

  def fetch(self, copy=True):
    """Blocks until the last submitted step finished; returns its records as numpy [B,K,F].  A copy by default: the
    two pinned buffers are reused by the asynchronous D2H of later steps (copy=False hands out the pinned view, valid
    until the step after next is submitted)."""
    self.compute.synchronize()
    rec = self.h_rec[(self.t - 1) & 1].numpy()
    return rec.copy() if copy else rec

  def fetch_tracks(self):
    """(tracks [B,T,CT_TRK_FLOATS], counts [B,2]) of the last submitted step (device_tracking), as numpy copies."""
    self.compute.synchronize()
    i = (self.t - 1) & 1
    return self.h_trk[i].numpy().copy(), self.h_cnt[i].numpy().copy()

  def fetch_results(self):
    """The last submitted step's tracks (device_tracking) as the host path's per-stream lists of dicts
    (DeviceTracker.results), payload fields included."""
    self.compute.synchronize()
    i = (self.t - 1) & 1
    pay = self.h_pay[i].numpy() if self.tracker.payload is not None else None
    return self.tracker.results(self.h_trk[i].numpy(), self.h_cnt[i].numpy(), pay)

  def previous_results(self):
    """After a step_host / step_frames call: the tracks of the step before it, as fetch_results() gives them.  No wait:
    the call returned once that step had finished (its records are what the call returned), and its tables are not
    overwritten before the next call."""
    if self.t < 2:
      raise ValueError('previous_results(): fewer than two steps submitted')
    i = (self.t - 2) & 1
    pay = self.h_pay[i].numpy() if self.tracker.payload is not None else None
    return self.tracker.results(self.h_trk[i].numpy(), self.h_cnt[i].numpy(), pay)

  @property
  def h2d_bytes_per_step(self):
    """Bytes uploaded per step: the frames (and pre_hm / public detections); a step that starts videos with device
    tracking also uploads its start list and seed rows, counted here after that step is submitted."""
    pub = self.B * (self.tracker.max_public * 2 + 1) * 4 if self.public else 0
    hm = self.B * self.H * self.W * 4 if self.tracker is None else 0
    if self.frames_mode:
      return self.slot_bytes + hm + pub + self._start_bytes
    return self.B * 3 * self.H * self.W * 4 + hm + pub + self._start_bytes

  @property
  def d2h_bytes_per_step(self):
    return self.rec.numel() * 4 + (self.tracker.d2h_bytes if self.tracker is not None else 0)

  def views(self, rec_np):
    from .decode import views_from_records
    return {k: v.numpy() for k, v in views_from_records(torch.from_numpy(rec_np), self.layout).items()}
