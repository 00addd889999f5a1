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
  Without a tracker, device_post_process=True post-processes the records inside the same graph (`DeviceDetections`:
  ct_post_process, Detector.post_process + merge_outputs) and downloads each stream's detections with them, so a
  detection model (ctdet, ddd, multi_pose) needs no host generic_post_process either.

The end-to-end form (`step_host`) takes HOST frames: pinned staging, H2D on a copy stream overlapped
with the previous step's compute, graph replay, D2H of the records (and tracks).

Frames mode (`frame_sizes`, `step_frames`) takes the raw uint8 BGR camera frames instead, one source size per stream:
the three slots hold the B frames ragged (16-byte aligned offsets) in pinned and device memory, each slot's ct_frame
descriptors are a device array beside them, and the step warps and normalises the frames on the device exactly as
Detector.pre_process_device does (cv2's fixed-point bilinear).  On the bf16 engine ct_pack_stem_frames_dev writes the
stem's packed bf16 input straight from slot t (images) and slot t-1 (pre_images, warped again: no fp32 copy is kept);
the fp32 and bf16x3 engines warp every stream into the fp32 image slot with one ct_warp_frames_normalize and run their
plan unchanged.  The tracker gets each stream's (c, s) and default calib, so tracks, public detections and 3D boxes are
in that camera's pixels.  With max_frame_size, stream b's frame lives at b * cap in every slot, so a stream may take a
frame of another size, and a new camera, when it starts a video: the step uploads the slot's changed descriptors, and
a replayed graph reads them, without a recapture.
A capacity runner may take NV12 or I420 frames instead (`frame_format`, what video decoders emit): each [3h/2, w] frame
is uploaded as it is, half the bytes of BGR, and the device-descriptor kernels convert each bilinear tap to BGR with
cv2.cvtColor's fixed-point arithmetic, so the stream computes what it computes on the cv2-converted BGR frame.
Device frames (step_frames with CUDA tensors, what GPU decoders hand out): instead of the host staging and upload, one
ct_stage_frames on the copy stream copies every live stream's frame from the caller's tensors (any row pitch; RGB and
planar RGB written as BGR, NV12 / I420 planes written in cv2's layout) into its region of the slot.  Everything after
that -- packs, warps, graphs, start prologue, tracker -- reads the slot as it reads an uploaded one.

Video starts (`starts=`, `pre_dets=` of step_host / step_frames / load_device_inputs): a stream may begin a new video at
any step, as Detector.reset_tracking + Tracker.init_track(pre_dets) on that stream alone.  A start is rare (once per
video), so it is not in the graphs: a step that carries starts first runs a short prologue on the compute stream -- the
started streams' frames copied into the previous slot (their pre_images), then ct_track_start (reset, seeds, render
boxes) -- and then replays the same graph as any other step.  Steps without starts run exactly what they ran before.

Flip test (`opt.flip_test`, detector.py:225-226,285-286,311-332): the network runs on 2B images, the streams' frames
[0, B) and their mirrors [B, 2B), inside the same step.  pre_images is the previous step's 2B images, so the previous
frame's mirror comes free (detector.py:148).  Uploads, the device tracker's render and a caller's pre_hm fill the first
B images; ct_mirror_x writes the second half in the graph, or, in frames mode on the bf16 engine,
ct_pack_stem_frames_flip_dev stores every packed pixel at its mirrored position too.  One ct_flip_merge_heads launch
averages the flipped heads into [B] buffers; decode and tracking then run at B on those and on the first half of the
other heads.  Records, tracks, uploads and downloads are the same size as without the flip.

Idle streams (`idle_streams=g`, `step_frames(..., idle=)`, capacity frames runners): a step computes only the streams
that have a frame.  The live streams s_0 < ... < s_{n-1} are compacted into the first n images (image i = stream s_i),
the batch rounded up to a multiple of g (capped at B) with padding images whose invalid descriptors give zero input.
Every launch runs at that batch; the track step and the prior heat-map render map images to streams through per-slot
device maps (ct_track_step_mapped, ct_render_tracks_mapped), uploaded with the slot's descriptors when they change.
One CUDA graph per (slot, batch).  pre_images must not depend on an image index, so the fp32 and bf16x3 engines warp
the previous slot's frames again (the bf16 engine's pack already does).  An idle stream's tables, frame region and
camera rows are left as they are; it comes back with a video start, or continues its video (`resume=`): its last frame
is still in its region of the slot where it last had a frame (`last_slot`), and when that is not the previous slot one
ct_stage_frames on the copy stream copies it there before the step's upload, so the step reads it as pre_images.

Moving a video (`stream_state(b)`, `step_frames(..., restore={b: state})`, capacity runners): a StreamState holds a
stream's last frame, camera and track rows; restoring it into a stream of this or another runner is a video start at the
state's frame size and camera whose prologue stages that frame as pre_images and writes the rows verbatim
(ct_track_restore) instead of seeding them.

Per-stream tracker settings (`stream_opts`, `options=` at a video start, a StreamState's options): each stream may run
its own out_thresh / pre_thresh / new_thresh (derived from its track_thresh as opts.py derives them), max_age,
--hungarian and --public_det, so that stream b computes what Detector(opt_b).run computes.  They act only in the
per-stream kernels (ct_track_step_opts, ct_track_start_opts / _restore_opts, ct_post_process_opts), which read one
ct_track_opts record per stream from the slot's device copy; a slot's records are uploaded with its frames when they
changed, so the graphs are never recaptured.

Crops (`crop_size=(out_h, out_w)`, frames runners with device_tracking or device_post_process): the last launch of each
step, inside its graph, crops every active track (or kept detection) of every stream out of the frame slot the step
read -- one ct_crop_boxes, cv2.warpAffine of each box stretched to out_h x out_w, with the warp's taps and so 4:2:0
frames converted as cv2.cvtColor converts them -- into that slot's uint8 BGR crop buffer [B, K, out_h, out_w, 3].  The
graphs have fixed pointers, so there is one crop buffer per input slot: a step's crops stay put until its slot is
reused three steps later.  Only the crop counts [B] travel to the host, with the tables (fetch_crops).
With crop_format as well, the crops are written instead as the batch an embedding or classifier network reads: one
ct_crop_boxes_tensor (an offsets pass, then the crop pass) packs every stream's crops, stream after stream, into that
slot's [B * K, 3, out_h, out_w] tensor of the format's dtype, channel order and Normalize(mean, std), beside the slot's
row offsets [B + 1]; the uint8 buffers are not allocated.  In fp16 at B = 32, K = 100 and 256 x 128 crops a slot's batch
is 629 MB (1.9 GB for the three slots).
"""
import ctypes as C

import numpy as np
import torch

from . import _lib as L
from .dataset_info import get_dataset
from .decode import generic_decode
from .detector import default_calib, flip_output, flip_plan, frame_geometry
from .device_detections import DeviceDetections
from .device_tracker import DeviceTracker, default_geometry, plan_starts


NS = 3          # input slots
# idle_streams=True: the batch granule.  On an H100 (DESIGN §5) g = 4 was never faster than g = 1 and slower where it
# pads (n = 1, 2); a larger g only saves graphs.
IDLE_GRANULE = 1

# frame_format -> ct_frame.format
FRAME_FORMATS = {'bgr': L.CT_FRAME_BGR, 'nv12': L.CT_FRAME_NV12, 'i420': L.CT_FRAME_I420}


def frame_layout(fmt, h, w):
  """(array shape, bytes, row pitch) of an h x w source frame in format fmt: BGR is [h, w, 3]; NV12 and I420 are one
  [3h/2, w] uint8 array each (cv2's 4:2:0 layouts), half the bytes."""
  if fmt == 'bgr':
    return (h, w, 3), h * w * 3, 3 * w
  return (h * 3 // 2, w), h * w * 3 // 2, w


def frame_size_of(fmt, shape):
  """The (h, w) of a frame array of this shape in format fmt, or None when the shape is not one of fmt's: BGR
  [h, w, 3]; NV12 / I420 [R, w] with R a multiple of 3 (h = 2R/3) and w even."""
  shape = tuple(shape)
  if fmt == 'bgr':
    return shape[:2] if len(shape) == 3 and shape[2] == 3 else None
  if len(shape) != 2 or shape[0] % 3 or shape[1] % 2:
    return None
  return shape[0] // 3 * 2, shape[1]


# step_frames(layout=) of a device frame on a BGR runner -> ct_frame_src.layout
DEVICE_LAYOUTS = {'bgr': L.CT_SRC_BGR, 'rgb': L.CT_SRC_RGB, 'rgb_planar': L.CT_SRC_RGB_PLANAR}


def is_device_frame(x):
  """Whether a step_frames entry is a device frame (a torch tensor, or a tuple of plane tensors) rather than an array."""
  return isinstance(x, torch.Tensor) or (isinstance(x, tuple) and len(x) > 0 and
                                         all(isinstance(t, torch.Tensor) for t in x))


def device_frame_source(x, fmt, layout, device, what='frame'):
  """A device frame -> ((h, w), L.FrameSrc) for ct_stage_frames, reading only each tensor's dtype, device, shape,
  stride() and data_ptr().  fmt: the runner's frame_format; layout: 'bgr', 'rgb' ([h, w, 3]) or 'rgb_planar' ([3, h, w])
  on a BGR runner, 'bgr' on a 4:2:0 one.  NV12 / I420: one uint8 [3h/2, w] tensor in cv2's layout (I420 with rows of
  exactly w bytes, since its chroma half-rows are packed two to a row), or the planes (Y [h, w], UV [h/2, w]) /
  (Y [h, w], U [h/2, w/2], V [h/2, w/2]).  Rows may have any pitch; the innermost stride must be 1 (and 3 for the pixels
  of an interleaved frame).  ValueError naming `what` on a wrong dtype or device, strides, a pitch shorter than a row,
  plane shapes that disagree, or odd 4:2:0 sizes."""
  if fmt not in FRAME_FORMATS:
    raise ValueError('frame_format: expected one of %s, got %r' % (sorted(FRAME_FORMATS), fmt))
  if fmt == 'bgr' and layout not in DEVICE_LAYOUTS:
    raise ValueError('layout: expected one of %s, got %r' % (sorted(DEVICE_LAYOUTS), layout))
  if fmt != 'bgr' and layout != 'bgr':
    raise ValueError("layout=%r: a %s runner takes its own format only (layout='bgr')" % (layout, fmt.upper()))
  planes = x if isinstance(x, tuple) else (x,)
  device = torch.device(device)
  for i, t in enumerate(planes):
    name = what if len(planes) == 1 else '%s[%d]' % (what, i)
    if not isinstance(t, torch.Tensor):
      raise ValueError('%s: expected a torch tensor, got %s' % (name, type(t).__name__))
    if t.dtype != torch.uint8:
      raise ValueError('%s: expected a uint8 tensor, got %s' % (name, t.dtype))
    if t.device.type != device.type or (device.index is not None and t.device.index != device.index):
      raise ValueError("%s: on %s, not on the runner's device %s" % (name, t.device, device))

  def pitch(shape, stride, name, row):
    """The row pitch of a [rows, row] plane of these (shape, strides) (its innermost stride 1); a single row's pitch is
    its length."""
    if shape[1] > 1 and stride[1] != 1:
      raise ValueError('%s: the innermost stride must be 1, got strides %s' % (name, tuple(stride)))
    p = stride[0] if shape[0] > 1 else row
    if p < row:
      raise ValueError('%s: row pitch of %d bytes is shorter than a row of %d' % (name, p, row))
    return p

  src = L.FrameSrc()
  if fmt == 'bgr':
    if len(planes) != 1:
      raise ValueError('%s: a BGR runner takes one tensor per frame, got %d' % (what, len(planes)))
    if layout == 'rgb_planar':
      if x.dim() != 3 or x.shape[0] != 3:
        raise ValueError("%s: layout 'rgb_planar' expects shape [3, h, w], got %s" % (what, tuple(x.shape)))
      h, w = int(x.shape[1]), int(x.shape[2])
      if h <= 0 or w <= 0:
        raise ValueError('%s: empty frame of shape %s' % (what, tuple(x.shape)))
      p = pitch(x.shape[1:], x.stride()[1:], what, w)
      src.layout = L.CT_SRC_RGB_PLANAR
      for c in range(3):
        src.plane[c], src.pitch[c] = x.data_ptr() + c * x.stride(0), p
      return (h, w), src
    if x.dim() != 3 or x.shape[2] != 3:
      raise ValueError("%s: layout %r expects shape [h, w, 3], got %s" % (what, layout, tuple(x.shape)))
    h, w = int(x.shape[0]), int(x.shape[1])
    if h <= 0 or w <= 0:
      raise ValueError('%s: empty frame of shape %s' % (what, tuple(x.shape)))
    if x.stride(2) != 1 or (w > 1 and x.stride(1) != 3):
      raise ValueError('%s: the innermost stride must be 1 and the pixel stride 3, got strides %s' % (what, x.stride()))
    src.layout = DEVICE_LAYOUTS[layout]
    src.plane[0], src.pitch[0] = x.data_ptr(), (x.stride(0) if h > 1 else 3 * w)
    if src.pitch[0] < 3 * w:
      raise ValueError('%s: row pitch of %d bytes is shorter than a row of %d' % (what, src.pitch[0], 3 * w))
    return (h, w), src
  n_planes = 2 if fmt == 'nv12' else 3
  src.layout = L.CT_SRC_NV12 if fmt == 'nv12' else L.CT_SRC_I420
  if len(planes) == 1:                      # cv2's [3h/2, w] layout
    if x.dim() != 2 or x.shape[0] % 3 or x.shape[1] % 2 or x.shape[0] == 0 or x.shape[1] == 0:
      raise ValueError('%s: expected a %s frame of shape [3h/2, w] (rows a multiple of 3, w even), got %s' %
                       (what, fmt.upper(), tuple(x.shape)))
    h, w = int(x.shape[0]) // 3 * 2, int(x.shape[1])
    p = pitch(x.shape, x.stride(), what, w)
    if fmt == 'i420' and p != w:
      raise ValueError('%s: an I420 frame given as one tensor needs rows of exactly w = %d bytes (its chroma half-rows '
                       'are packed two to a row), got a pitch of %d; give a pitched surface as (Y, U, V) planes' %
                       (what, w, p))
    y = x.data_ptr()
    src.plane[0], src.pitch[0] = y, p
    if fmt == 'nv12':
      src.plane[1], src.pitch[1] = y + h * p, p
    else:
      src.plane[1], src.plane[2] = y + h * w, y + h * w + (h // 2) * (w // 2)
      src.pitch[1] = src.pitch[2] = w // 2
    return (h, w), src
  if len(planes) != n_planes:
    raise ValueError('%s: expected %s planes %s, got %d tensors' %
                     (what, fmt.upper(), '(Y, UV)' if fmt == 'nv12' else '(Y, U, V)', len(planes)))
  Y = planes[0]
  if Y.dim() != 2:
    raise ValueError('%s[0]: expected a 2-D plane, got shape %s' % (what, tuple(Y.shape)))
  h, w = int(Y.shape[0]), int(Y.shape[1])
  if h <= 0 or w <= 0 or h % 2 or w % 2:
    raise ValueError('%s[0]: Y plane of shape %s; %s frames have an even, non-zero height and width' %
                     (what, (h, w), fmt.upper()))
  want = [(h, w), (h // 2, w)] if fmt == 'nv12' else [(h, w), (h // 2, w // 2), (h // 2, w // 2)]
  for i, (t, s) in enumerate(zip(planes, want)):
    if tuple(t.shape) != s:
      raise ValueError('%s[%d]: expected shape %s for a Y plane of %s, got %s' % (what, i, s, (h, w), tuple(t.shape)))
    src.plane[i], src.pitch[i] = t.data_ptr(), pitch(t.shape, t.stride(), '%s[%d]' % (what, i), s[1])
  return (h, w), src


def check_crop_size(crop_size, frames_mode, tables):
  """crop_size of StreamRunner -> (out_h, out_w), or None when off.  ValueError for a size that is not two integers
  >= 1, or a runner without frames (frame_sizes) or without a tracker or device post-processing (tables), whose boxes
  and frames the crops come from."""
  if crop_size is None:
    return None
  hw = tuple(crop_size) if isinstance(crop_size, (tuple, list)) else None
  if hw is None or len(hw) != 2 or any(isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)) or v < 1
                                       for v in hw):
    raise ValueError('crop_size: expected (out_h, out_w), two integers >= 1, got %r' % (crop_size,))
  if not frames_mode:
    raise ValueError('crop_size: crops are cut from the camera frames; build the runner with frame_sizes (frames mode)')
  if not tables:
    raise ValueError('crop_size: crops are cut at the tracks or detections of the device tables; build the runner with '
                     'device_tracking or device_post_process')
  return int(hw[0]), int(hw[1])


CROP_DTYPES = {torch.float32: L.CT_CROP_F32, torch.float16: L.CT_CROP_F16, torch.bfloat16: L.CT_CROP_BF16}
CROP_ORDERS = {'rgb': L.CT_CROP_RGB, 'bgr': L.CT_CROP_BGR}


def check_crop_format(crop_format, crop_size):
  """crop_format of StreamRunner -> {'dtype', 'channels', 'mean', 'std'} with mean and std as fp32 tuples, or None when
  off.  ValueError without crop_size, for a value that is not a dict of exactly these keys, a dtype other than
  torch.float16 / bfloat16 / float32, channels other than 'rgb' / 'bgr', or a mean or std that is not three real
  numbers finite in fp32, or a std with an entry that is 0 in fp32 (torchvision's Normalize refuses it too)."""
  if crop_format is None:
    return None
  if crop_size is None:
    raise ValueError('crop_format: it describes the crops of crop_size; build the runner with crop_size too')
  keys = ('dtype', 'channels', 'mean', 'std')
  if not isinstance(crop_format, dict) or sorted(crop_format) != sorted(keys):
    raise ValueError('crop_format: expected a dict of exactly %s, got %r' % (', '.join(keys), crop_format))
  if not any(crop_format['dtype'] is t for t in CROP_DTYPES):
    raise ValueError('crop_format: dtype must be torch.float16, torch.bfloat16 or torch.float32, got %r' %
                     (crop_format['dtype'],))
  if not isinstance(crop_format['channels'], str) or crop_format['channels'] not in CROP_ORDERS:
    raise ValueError("crop_format: channels must be 'rgb' or 'bgr', got %r" % (crop_format['channels'],))
  out = dict(dtype=crop_format['dtype'], channels=crop_format['channels'])
  for key in ('mean', 'std'):
    v = crop_format[key]
    v = tuple(v) if isinstance(v, (tuple, list, np.ndarray)) else None
    if v is None or len(v) != 3 or any(isinstance(x, (bool, np.bool_)) or not isinstance(x, (int, float, np.integer,
                                                                                             np.floating)) for x in v):
      raise ValueError('crop_format: %s must be three real numbers, got %r' % (key, crop_format[key]))
    with np.errstate(over='ignore'):
      f32 = tuple(np.float32(x) for x in v)
    if not all(np.isfinite(f32)) or (key == 'std' and any(x == 0 for x in f32)):
      raise ValueError('crop_format: %s must be finite in fp32%s, got %r' % (key, ' and != 0' if key == 'std' else '',
                                                                            crop_format[key]))
    out[key] = tuple(float(x) for x in f32)
  return out


def _ints(streams):
  """The integer entries of a stream list, as a set (the others are refused by the list's own check)."""
  return {int(s) for s in streams if isinstance(s, (int, np.integer)) and not isinstance(s, (bool, np.bool_))}


class StreamState(object):
  """One stream of a capacity runner after the last step in which it had a frame (StreamRunner.stream_state), what
  step_frames(restore=) needs to continue its video on another stream or runner.
    frame            device uint8 tensor of that frame in frame_format's layout ([h, w, 3], or [3h/2, w] in 4:2:0)
    size             its (h, w)
    calib            float32 [3, 4] camera matrix
    tracks, counts, payload   tracking runners: the track rows [n, CT_TRK_FLOATS] (device), (n, id_count), and the
                     payload rows [n, Wp] (device) on head sets with payload fields; None otherwise
    options          the stream's resolved tracker settings (resolve_options: out_thresh, new_thresh, pre_thresh,
                     max_age, hungarian, public_det; out_thresh alone without a tracker), which restore= applies on a
                     runner built with stream_opts (one built without runs its own opt on every stream); None on a
                     runner that neither tracks nor post-processes
    input_size, record_layout, payload_layout, max_tracks, frame_format   the layout facts the importer checks
  A copy: the exporting runner may go on using the stream."""

  def __init__(self, frame, size, calib, tracks, counts, payload, input_size, record_layout, payload_layout, max_tracks,
               frame_format, options=None):
    self.frame, self.size, self.calib = frame, tuple(size), calib
    self.tracks, self.counts, self.payload = tracks, counts, payload
    self.input_size, self.record_layout, self.payload_layout = tuple(input_size), record_layout, payload_layout
    self.max_tracks, self.frame_format = max_tracks, frame_format
    self.options = dict(options) if options is not None else None


class StreamRunner(object):

  frame_format = 'bgr'
  post = None                                                # device_post_process: DeviceDetections
  crop = None                                                # crop_size: (out_h, out_w)
  crop_format = None                                         # crop_format: check_crop_format's dict

  def __init__(self, model, B, H, W, K=100, precision='bf16', device='cuda', use_graph=True, opt=None,
               device_tracking=False, max_public_dets=512, calibs=None, frame_sizes=None, max_frame_size=None,
               idle_streams=None, frame_format='bgr', device_post_process=False, stream_opts=None, crop_size=None,
               crop_format=None):
    """max_public_dets: with device_tracking and --public_det, the most public detections a stream may bring per
    frame (more raise ValueError; none is ever dropped).  calibs: with device_tracking on a 3D head set, one [3,4]
    camera matrix per stream (DeviceTracker's default otherwise; in frames mode Detector._get_default_calib of the
    stream's source size).  frame_sizes: B (height, width) source sizes to feed raw uint8 frames with step_frames; each
    must map to the network input (H, W) under opt's resolution policy (ValueError otherwise); the descriptors of the
    frames live on the device.  Without max_frame_size they are fixed for the runner's lifetime.  max_frame_size
    (h, w): every stream gets a frame region of h * w * 3 bytes in each slot, and may bring a frame of any size that
    fits it and maps to (H, W) when it starts a video (frame_sizes are then the first sizes).
    opt.flip_test: every stream's frame runs with its mirror (2B images per step) and the averaged heads are merged
    before decode, as Detector.process does; inputs and outputs keep their B shapes.
    idle_streams g >= 1, or True for g = IDLE_GRANULE (capacity frames runners only): step_frames(idle=) may leave
    streams without a frame, and a step computes only the live ones, in a batch rounded up to a multiple of g (see the
    module docstring).  None or False: off.
    frame_format: what step_frames and frame_buffers take -- 'bgr' (uint8 [h, w, 3]), or 'nv12' / 'i420' (one uint8
    [3h/2, w] array per frame in cv2's 4:2:0 layout, h and w even; needs max_frame_size, whose region is then
    h * w * 3 / 2 bytes).  A 4:2:0 frame is converted on the device, inside the warp, exactly as
    cv2.cvtColor(COLOR_YUV2BGR_NV12 / _I420) converts it: a stream gives what it gives on that BGR image.
    device_post_process (runners without device_tracking): each step also post-processes its records on the device
    (ct_post_process, inside the graph) into each stream's detections in its source pixels -- Detector.post_process +
    merge_outputs -- and downloads them with the records: fetch_results() / previous_results() give the host path's
    dicts, fetch_detections() the tables.  calibs then give the 3D head sets' cameras, as with device_tracking.
    stream_opts (device_tracking or device_post_process): None, every stream runs opt (the launches and bytes of a
    runner without it), or B entries, each None (opt) or a dict of the flags stream b runs with instead --
    track_thresh, out_thresh, pre_thresh, new_thresh, max_age, hungarian, public_det with a tracker (resolved against
    opt by device_tracker.resolve_options), out_thresh alone with device_post_process.  A stream changes them only at
    a video start (options= of step_host / step_frames / load_device_inputs) or with a restore.  The track table's
    rows come from the largest max_age among opt and these entries, and public detections are staged when opt or any
    entry has public_det.
    crop_size (out_h, out_w): frames runners with device_tracking or device_post_process; each step also crops every
    stream's active tracks (or kept detections) out of its frame on the device (fetch_crops, previous_crops).  None:
    off, the launches and bytes of a runner without it.
    crop_format (with crop_size): {'dtype': torch.float16 | torch.bfloat16 | torch.float32, 'channels': 'rgb' | 'bgr',
    'mean': (m0, m1, m2), 'std': (s0, s1, s2)}, mean and std in output-channel order; the crops come as one packed
    batch of that dtype, torchvision's Normalize(mean, std)(ToTensor()(crop)).to(dtype) of each crop in that channel
    order (fetch_crops).  None: the uint8 BGR crops."""
    if stream_opts is not None and not (device_tracking or device_post_process):
      raise ValueError('stream_opts: the per-stream settings act in the tracker or the device post-processing; build '
                       'the runner with device_tracking or device_post_process')
    if device_post_process and device_tracking:
      raise ValueError('device_post_process is for runners without a tracker: device_tracking already post-processes '
                       'the detections (fetch_results() gives its tracks)')
    self.crop_size = check_crop_size(crop_size, frame_sizes is not None, device_tracking or device_post_process)
    self.crop_format = check_crop_format(crop_format, crop_size)
    self.crop = None                                         # crop_size once the tables exist (_eager launches it)
    self.B, self.H, self.W, self.K = B, H, W, K
    self.device = torch.device(device)
    self.model = model
    self.opt = opt if opt is not None else getattr(model, 'opt', None)
    self.frames_mode = frame_sizes is not None
    if max_frame_size is not None and not self.frames_mode:
      raise ValueError('max_frame_size needs frame_sizes (frames mode)')
    if frame_format not in FRAME_FORMATS:
      raise ValueError('frame_format: expected one of %s, got %r' % (sorted(FRAME_FORMATS), frame_format))
    if frame_format != 'bgr' and max_frame_size is None:
      raise ValueError("frame_format=%r needs frame_sizes and max_frame_size (the device-descriptor frames path)" %
                       (frame_format,))
    self.frame_format = frame_format
    self.idle_g = None
    if idle_streams is True:                                 # on, with the default granule
      idle_streams = IDLE_GRANULE
    if idle_streams is not None and idle_streams is not False:
      if isinstance(idle_streams, np.bool_) or not isinstance(idle_streams, (int, np.integer)) or idle_streams < 1:
        raise ValueError('idle_streams: expected True or an integer batch granule >= 1, got %r' % (idle_streams,))
      if max_frame_size is None:
        raise ValueError('idle_streams needs a capacity frames runner (frame_sizes and max_frame_size)')
      self.idle_g = int(idle_streams)
    self._n = B                                              # the (padded) batch of the step being launched
    self.cap = self.max_frame_bytes = None
    if self.frames_mode:
      calibs = self._frame_geometry(frame_sizes, calibs, max_frame_size)
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
      # per slot: the device descriptors of its frames, their pinned staging and a host mirror.  The graphs read
      # d_frames[slot], so it is written in place and never reallocated.
      desc = torch.from_numpy(np.frombuffer(bytes(self.frames), np.uint8).copy())
      self.h_frames = [desc.clone().pin_memory() for _ in range(NS)]
      self.d_frames = [desc.to(self.device) for _ in range(NS)]
      self._desc_mirror = [bytes(self.frames)] * NS
    if self.idle_g is not None:  # per slot: streams [B] (image -> stream) then image_of [B] (stream -> image), int32
      ident = torch.arange(B, dtype=torch.int32).repeat(2)
      self.h_map = [ident.clone().pin_memory() for _ in range(NS)]
      self.d_map = [ident.to(self.device) for _ in range(NS)]
      self._map_mirror = [ident.numpy().tobytes()] * NS
      self._live = [None, None]                              # per D2H buffer: the live streams of its step
      self._was_idle = set()                                 # the streams idle in the last submitted step
      self.idle_graphs = {}                                  # (slot, batch) -> graph
      if not self.eng.use_halo and self.eng.has_pre_img:     # pre_images, warped again from the previous slot
        self.pre_img = torch.zeros((NB, 3, H, W), dtype=f32, device=self.device)
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
    self._restores = [None] * NS                             # per slot: {stream: StreamState} restored in its step
    self.last_slot = [None] * B                              # per stream: the slot of its last step with a frame
    self._start_bytes = 0                                    # start list + seed rows uploaded by the last step
    self.h_start = None                                      # per slot start list / seed staging, made on first use
    self.h_geo = None                                        # per slot camera geometry rows staging, made on first use
    self._geo = [None] * NS                                  # per slot: the streams whose geometry rows it carries
    self._frame_bytes = 0                                    # frame (+ descriptor) bytes of the last upload
    self._ev_read = None                                     # recorded after the last staging of device frames
    if self.frames_mode:
      self._frame_bytes = sum(e - a for a, e in self._upload_runs())
    self._eager(0, first=True)                               # sizes the record buffer
    if device_tracking:
      assert self.opt is not None, 'device tracking needs opt (thresholds, max_age)'
      geo = {}
      if self.frames_mode:
        geo = dict(centers=[m['c'] for m in self._meta], scales=[m['s'] for m in self._meta])
      self.tracker = DeviceTracker(self.opt, B, K, self.rec.shape[2], self.layout, H, W, self.device,
                                   max_public_dets=max_public_dets, calibs=calibs, stream_opts=stream_opts, **geo)
    elif device_post_process:
      assert self.opt is not None, 'device post-processing needs opt (out_thresh)'
      geo = {}
      if self.frames_mode:
        geo = dict(centers=[m['c'] for m in self._meta], scales=[m['s'] for m in self._meta])
      self.post = DeviceDetections(self.opt, B, K, self.rec.shape[2], self.layout, H, W, self.device, calibs=calibs,
                                   stream_opts=stream_opts, **geo)
    if self.crop_size is not None:   # per input slot: the slot's graphs write its crops; the counts go to the host
      if self.crop_format is None:
        self.crops = [torch.zeros((B, K) + self.crop_size + (3,), dtype=torch.uint8, device=self.device)
                      for _ in range(NS)]
      else:                          # the packed batch [B * K rows] and its row offsets [B + 1]
        self.crops = [torch.zeros((B * K, 3) + self.crop_size, dtype=self.crop_format['dtype'], device=self.device)
                      for _ in range(NS)]
        self.crop_offsets = [torch.zeros((B + 1,), dtype=torch.int32, device=self.device) for _ in range(NS)]
      self.crop_counts = torch.zeros((B,), dtype=torch.int32, device=self.device)
      self.h_crop_cnt = [torch.zeros((B,), dtype=torch.int32).pin_memory() for _ in range(2)]
      self.crop = self.crop_size
    self.d_opts = None
    tables = self._geo_tables()
    if self._per_stream():                        # per slot: device ct_track_opts [B], pinned staging, host mirror
      self.d_opts = [tables.d_opts.clone() for _ in range(NS)]
      self.h_opts = [tables.d_opts.cpu().pin_memory() for _ in range(NS)]
      self._opts_mirror = [tables.opts_bytes()] * NS
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
    if self.post is not None:
      self.h_det = [torch.zeros_like(self.post.dets, device='cpu').pin_memory() for _ in range(2)]
      self.h_det_cnt = [torch.zeros_like(self.post.counts, device='cpu').pin_memory() for _ in range(2)]
      if self.post.payload is not None:
        self.h_det_pay = [torch.zeros_like(self.post.payload, device='cpu').pin_memory() for _ in range(2)]
    # launches of one step: the network plan + decode (+ memset-free: render + track step); frames mode: the pack op
    # becomes ct_pack_stem_frames_dev, or one ct_warp_frames_normalize comes before the plan.
    # --flip_test: + the merge, + the mirrors of the images and pre_hm unless the flip pack writes them;
    # device_post_process: + ct_post_process; crop_size: + ct_crop_boxes, or with crop_format ct_crop_boxes_tensor's two
    self.launches_per_step = self.eng.n_launches + 1 + (2 if device_tracking else 0) + (1 if self.post else 0) + \
        ((2 if self.crop_format else 1) if self.crop else 0)
    if self.frames_mode:
      self.launches_per_step += 0 if self.eng.use_halo else 1
    if self.flip:
      self.launches_per_step += 1 + (0 if self._pack_mirror else 1 + int(self.eng.has_pre_hm))
    if self.idle_g is not None and not self.eng.use_halo and self.eng.has_pre_img:   # + the pre_images warp (+ mirror)
      self.launches_per_step += 1 + int(self.flip)

  def _frame_geometry(self, frame_sizes, calibs, max_frame_size=None):
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
    self.cap = self.max_frame_bytes = None
    if max_frame_size is not None:
      mh, mw = (int(v) for v in max_frame_size)
      if mh <= 0 or mw <= 0:
        raise ValueError('max_frame_size: bad size %s' % ((mh, mw),))
      self.max_frame_bytes = frame_layout(self.frame_format, mh, mw)[1]
      self.cap = (self.max_frame_bytes + 15) // 16 * 16        # stream b's frame lives at b * cap in every slot
    ds = get_dataset(opt.dataset)
    self.focal = opt.test_focal_length if getattr(opt, 'test_focal_length', -1) >= 0 else ds.rest_focal_length
    self.mean = np.ascontiguousarray(ds.mean, dtype=np.float32).reshape(3)
    self.std = np.ascontiguousarray(ds.std, dtype=np.float32).reshape(3)
    self.frames = (L.Frame * B)()
    self._meta = []
    off = 0
    for b, (h, w) in enumerate(frame_sizes):
      h, w = int(h), int(w)
      meta, minv = self._size_geometry('frame_sizes[%d]' % b, h, w)
      meta['calib'] = calibs[b] if calibs is not None else default_calib(self.focal, w, h)
      self._meta.append(meta)
      f = self.frames[b]
      _, nbytes, f.step = frame_layout(self.frame_format, h, w)
      f.offset, f.h, f.w, f.format = (off if self.cap is None else b * self.cap), h, w, FRAME_FORMATS[self.frame_format]
      f.minv[:] = minv.tolist()
      off += (nbytes + 15) // 16 * 16
    self._prev_meta = self._meta
    self.frame_sizes = [(int(h), int(w)) for h, w in frame_sizes]
    self.slot_bytes = off if self.cap is None else B * self.cap
    return calibs if calibs is not None else np.stack([m['calib'] for m in self._meta]).astype(np.float32)

  def _size_geometry(self, what, h, w):
    """(meta without calib, minv) of an h x w source frame; ValueError when it is empty, does not fit a capacity
    runner's frame region, is odd in a 4:2:0 format, or maps to another network input than (H, W)."""
    if h <= 0 or w <= 0:
      raise ValueError('%s: bad size %s' % (what, (h, w)))
    if self.frame_format != 'bgr' and (h % 2 or w % 2):
      raise ValueError('%s = %s: %s frames have an even height and width' % (what, (h, w), self.frame_format.upper()))
    nbytes = frame_layout(self.frame_format, h, w)[1]
    if self.cap is not None and nbytes > self.max_frame_bytes:
      raise ValueError('%s = %s: %d bytes, more than the %d of max_frame_size' % (what, (h, w), nbytes,
                                                                                 self.max_frame_bytes))
    meta, minv = frame_geometry(self.opt, h, w)
    if (meta['inp_height'], meta['inp_width']) != (self.H, self.W):
      raise ValueError('%s = %s maps to a %dx%d network input under this resolution policy, not the '
                       "runner's %dx%d" % (what, (h, w), meta['inp_height'], meta['inp_width'], self.H, self.W))
    return meta, minv

  def check_frame_size(self, size):
    """ValueError unless a stream of this runner can take frames of size (height, width) at a video start."""
    h, w = (int(v) for v in size)
    if self.cap is None:
      if (h, w) not in self.frame_sizes:
        raise ValueError('frame size %s: the streams take %s' % ((h, w), sorted(set(self.frame_sizes))))
      return
    self._size_geometry('frame size', h, w)

  def meta(self, b):
    """Frames mode: the meta dict Detector.pre_process returns for stream b's frame in the last submitted step (c, s,
    sizes, trans_input, trans_output, calib) -- what generic_post_process needs when the records are post-processed on
    the host."""
    if not self.frames_mode:
      raise ValueError('meta(): the runner was not built with frame_sizes')
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in self._meta[b].items()}

  def previous_meta(self, b):
    """Frames mode: meta(b) of the step whose records the last step_frames call returned (the step before the last
    submitted one), for generic_post_process of those records; as previous_results() is to fetch_results()."""
    if not self.frames_mode:
      raise ValueError('previous_meta(): the runner was not built with frame_sizes')
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in self._prev_meta[b].items()}

  def _check_calibs(self, calibs, streams):
    """calibs ({stream: [3, 4]} of started streams) -> {stream: float32 [3, 4]}; ValueError before anything is
    enqueued."""
    out = {}
    for s, k in (calibs or {}).items():
      if s not in streams:
        raise ValueError('calibs: stream %r does not start a video in this step' % (s,))
      k = np.asarray(k, np.float32)
      if k.shape != (3, 4):
        raise ValueError('calibs[%d]: expected a [3, 4] camera matrix, got shape %s' % (s, k.shape))
      out[s] = k
    return out

  def _check_sizes(self, sizes, streams):
    """This step's (h, w) per stream -> {stream: (meta without calib, minv)} of the streams whose size changes.
    ValueError (before anything is enqueued) for a change on a fixed-size runner or on a stream that does not start a
    video (its pre_hm boxes were rendered with its old trans_input), or a size _size_geometry refuses."""
    changed = {}
    for b, (hw, now) in enumerate(zip(sizes, self.frame_sizes)):
      if tuple(hw) == tuple(now):
        continue
      if self.cap is None:
        raise ValueError('frames[%d]: expected shape %s, got %s' % (b, tuple(now) + (3,), tuple(hw) + (3,)))
      if b not in streams:
        raise ValueError('frames[%d]: size %s differs from the stream\'s %s; a stream changes its frame size only when '
                         'it starts a video (starts=)' % (b, tuple(hw), tuple(now)))
      changed[b] = self._size_geometry('frames[%d]' % b, int(hw[0]), int(hw[1]))
    return changed

  def _plan_geometry(self, slot, changed, calibs, live=None):
    """Host state of one step's geometry changes (changed: _check_sizes, calibs: _check_calibs): the descriptors and
    metas of the changed streams, the slot's descriptor staging when its device copy differs, and the tracker rows of
    the streams whose camera changes.  live (idle-streams runners): the step's live streams, whose descriptors the
    slot holds in image order.  -> (descriptor bytes to upload or None, [(stream, c, s, calib)])."""
    rows = []
    if self.frames_mode:
      self._prev_meta = self._meta
      if changed or calibs:
        self._meta = list(self._meta)
      for b, (meta, minv) in changed.items():
        h, w = meta['height'], meta['width']
        f = self.frames[b]
        f.h, f.w, f.step = h, w, frame_layout(self.frame_format, h, w)[2]
        f.minv[:] = minv.tolist()
        meta['calib'] = calibs[b] if b in calibs else default_calib(self.focal, w, h)
        self._meta[b] = meta
        self.frame_sizes[b] = (h, w)
      for b, k in calibs.items():
        if b not in changed:
          self._meta[b] = dict(self._meta[b], calib=k)
      for b in sorted(set(changed) | set(calibs)):
        m = self._meta[b]
        rows.append((b, m['c'], m['s'], np.asarray(m['calib'], np.float32)))
    elif self._geo_tables() is not None:     # fp32 images of the input size: the default (c, s) throughout
      c, s = default_geometry(self.H, self.W)
      rows = [(b, c, s, k) for b, k in sorted(calibs.items())]
    desc = None
    if self.frames_mode:
      now = bytes(self.frames) if live is None else bytes(self._image_frames(live))
      if now != self._desc_mirror[slot]:
        desc = self._desc_mirror[slot] = now
    return desc, rows

  def _upload_runs(self, live=None):
    """Maximal runs [start, end) of the slot bytes this step's frames use: stream b's frame, padded to 16 bytes, at its
    offset, for every stream or the `live` ones.  One run of slot_bytes on a fixed runner (its frames are contiguous)
    and on a capacity runner whose streams are all at capacity."""
    runs = []
    for b, f in enumerate(self.frames):
      if live is not None and b not in live:
        continue
      a, e = f.offset, f.offset + (frame_layout(self.frame_format, f.h, f.w)[1] + 15) // 16 * 16
      if runs and runs[-1][1] == a:
        runs[-1][1] = e
      else:
        runs.append([a, e])
    return [tuple(r) for r in runs]

  def _image_frames(self, live):
    """Idle-streams runners: the slot's descriptors in image order (image i = stream live[i]); the padding images'
    are zero, which the frames kernels read as invalid (a zero input)."""
    arr = (L.Frame * self.B)()
    for i, b in enumerate(live):
      arr[i] = self.frames[b]
    return arr

  def _maps(self, live):
    """int32 [2B]: streams (image -> stream, -1 for padding) then image_of (stream -> image, -1 when idle)."""
    m = np.full(2 * self.B, -1, np.int32)
    m[:len(live)] = live
    m[self.B + np.asarray(live, np.int64)] = np.arange(len(live), dtype=np.int32)
    return m

  def padded_batch(self, n):
    """The network batch of a step with n live streams: n rounded up to a multiple of idle_streams, at most B."""
    g = self.idle_g or self.B
    return min(-(-n // g) * g, self.B)

  # one step, eager launches on the current stream, at the batch self._n (B but on an idle-streams runner)
  def _eager(self, slot, first=False):
    n = self._n
    NBn = 2 * n if self.flip else n
    if self.tracker is not None:                             # pre_hm(t) from tracks(t-1)
      if self.idle_g is None:
        self.tracker.render(self.hm[slot][:self.B])
      else:
        self.tracker.render_mapped(self.hm[slot][:n], self.d_map[slot][self.B:])
    prev = slot if first else (slot - 1) % NS
    if self.frames_mode and self.eng.use_halo:
      eng = self.eng
      cur, pre = L.ptr(self.u8[slot]), L.ptr(self.u8[prev] if eng.has_pre_img else None)
      ms = (C.c_void_p(self.mean.ctypes.data), C.c_void_p(self.std.ctypes.data),
            L.ptr(self.hm[slot] if eng.has_pre_hm else None), L.ptr(eng.stem_input), self.H, self.W, L.stream_ptr())
      # the slot's device descriptors: a replayed graph reads the geometry the slot holds
      pack = L.lib().ct_pack_stem_frames_flip_dev if self.flip else L.lib().ct_pack_stem_frames_dev
      L.check(pack(cur, pre, L.ptr(self.d_frames[slot]), n, self.slot_bytes, *ms), 'ct_pack_stem_frames_dev')
      out = dict(eng.forward_packed(eng.has_pre_img, eng.has_pre_hm, n=NBn))
    else:
      if self.frames_mode:
        self._warp_frames(slot)
      pre = self.img[prev]
      if self.idle_g is not None and self.eng.has_pre_img:   # the previous frames through this step's descriptors
        pre = self.pre_img
        self._warp_frames(slot, src=self.u8[prev], dst=pre)
      if self.flip:                  # the mirrored half; pre_images (img[prev]) was mirrored by its own step
        self._mirror(self.img[slot], 0, n, n)
        if self.eng.has_pre_hm:
          self._mirror(self.hm[slot], 0, n, n)
        if pre is not self.img[prev]:
          self._mirror(pre, 0, n, n)
      out = dict(self.eng.forward(self.img[slot][:NBn], pre[:NBn], self.hm[slot][:NBn], n=NBn))
    if self.flip:
      merged = self.merged if n == self.B else {h: m[:n] for h, m in self.merged.items()}
      out = flip_output(out, self.flip_plan, merged)
    if self.ws is None:
      cat = out['hm'].shape[1]
      J = out['hm_hp'].shape[1] if ('hm_hp' in out and 'hps' in out) else 0
      self.ws = torch.zeros(L.lib().ct_decode_workspace_bytes(self.B, cat, J, self.K), dtype=torch.uint8,
                            device=self.device)
    rec = self.rec if (self.rec is None or n == self.B) else self.rec[:n]
    res = generic_decode(out, K=self.K, records_out=rec, workspace=self._decode_ws(n))
    if self.rec is None:
      self.rec, self.layout = res.records, res.layout
    if self.tracker is not None:                             # tracks(t)
      pub = self.pub[slot] if self.public else ()
      if self.idle_g is None:
        self.tracker.step(self.rec, *pub, opts=self._slot_opts(slot))
      else:
        self.tracker.step_mapped(self.rec[:n], self.d_map[slot][:self.B], *pub, opts=self._slot_opts(slot))
    if self.post is not None:                                # each stream's detections in its source pixels
      if self.idle_g is None:
        self.post.step(self.rec, opts=self._slot_opts(slot))
      else:
        self.post.step_mapped(self.rec[:n], self.d_map[slot][:self.B], opts=self._slot_opts(slot))
    if self.crop is not None:                                # the boxes just written, cut from the frames just read
      self._crop(slot)
    return res

  def _crop(self, slot):
    """ct_crop_boxes (ct_crop_boxes_tensor with crop_format, its offsets into crop_offsets[slot]) of this step's tables
    from u8[slot] through the slot's device descriptors into crops[slot], at the step's batch (image i = stream
    d_map[slot][i] on an idle-streams runner), on the current stream."""
    d = L.CropDesc()
    d.buf, d.buf_bytes, d.frames = self.u8[slot].data_ptr(), self.slot_bytes, self.d_frames[slot].data_ptr()
    if self.tracker is not None:                             # the active prefix of each stream's track rows
      trk = self.tracker
      d.rows, d.row_floats, d.rows_per_stream = trk.tracks.data_ptr(), L.CT_TRK_FLOATS, trk.T
      d.counts, d.counts_stride, d.active_col = trk.counts.data_ptr(), 2, L.CT_TRK_ACTIVE
    else:                                                    # each stream's kept detections
      d.rows, d.row_floats, d.rows_per_stream = self.post.dets.data_ptr(), L.CT_DET_FLOATS, self.K
      d.counts, d.counts_stride, d.active_col = self.post.counts.data_ptr(), 1, -1
    d.K, d.out_h, d.out_w = self.K, self.crop[0], self.crop[1]
    d.out_counts = self.crop_counts.data_ptr()
    streams = L.ptr(self.d_map[slot][:self.B]) if self.idle_g is not None else None
    if self.crop_format is None:
      d.out = self.crops[slot].data_ptr()
      L.check(L.lib().ct_crop_boxes(C.byref(d), streams, self._n, self.B, L.stream_ptr()), 'ct_crop_boxes')
      return
    fmt, t = self.crop_format, L.CropTensor()
    t.type, t.order = CROP_DTYPES[fmt['dtype']], CROP_ORDERS[fmt['channels']]
    t.mean[:], t.std[:] = fmt['mean'], fmt['std']
    t.rows_cap, t.out, t.out_offsets = self.crops[slot].shape[0], self.crops[slot].data_ptr(), \
        self.crop_offsets[slot].data_ptr()
    L.check(L.lib().ct_crop_boxes_tensor(C.byref(d), C.byref(t), streams, self._n, self.B, L.stream_ptr()),
            'ct_crop_boxes_tensor')

  def _slot_opts(self, slot):
    """The device ct_track_opts records slot's step reads (stream_opts runners), or None."""
    return self.d_opts[slot] if getattr(self, 'd_opts', None) is not None else None

  def _check_options(self, options, streams):
    """options ({stream: flags} of streams that start a video in this step) -> {stream: resolved settings}; ValueError
    before anything is enqueued (a stream that does not start, or what check_options refuses)."""
    out = {}
    for s, flags in (options or {}).items():
      if s not in streams:
        raise ValueError('options: stream %r does not start a video in this step; a stream changes its tracker '
                         'settings only at a video start (starts=) or a restore' % (s,))
      tables = self._geo_tables()
      if tables is None:
        raise ValueError('options: the runner has neither device_tracking nor device_post_process, whose settings they '
                         'are')
      out[s] = tables.check_options(flags, 'options[%d]' % s)
    return out

  def _per_stream(self):
    """Whether the runner was built with stream_opts."""
    return getattr(self._geo_tables(), 'per_stream', False)

  def _step_options(self, planned):
    """Each stream's settings in this step (stream_opts runners; None otherwise): the current ones with `planned`
    ({stream: resolved}) applied."""
    if not self._per_stream():
      return None
    return [planned.get(b, o) for b, o in enumerate(self._geo_tables().options)]

  def _plan_options(self, slot, planned):
    """Applies planned settings to the host state; -> the slot's ct_track_opts bytes to upload when its device copy
    differs (staged in h_opts[slot]), else None."""
    if getattr(self, 'd_opts', None) is None:
      return None
    tables = self._geo_tables()
    for b, o in planned.items():
      tables.options[b] = o
    now = tables.opts_bytes()
    if now == self._opts_mirror[slot]:
      return None
    self._opts_mirror[slot] = now
    self.h_opts[slot].numpy()[:] = np.frombuffer(now, np.uint8)
    return now

  def _decode_ws(self, n):
    """The decode workspace of a batch n <= B.  ct_decode keeps n per-image counters at its start, which must be zero
    on entry (each image's last CTA resets its own), and its candidates from align256(4 n) on.  At n < B the view starts
    align256(4 B) - align256(4 n) bytes in, so that the candidates of every batch begin where the B-image layout's do
    and never overwrite a counter of another batch."""
    if n == self.B:
      return self.ws
    a = lambda x: (x + 255) // 256 * 256
    return self.ws[a(4 * self.B) - a(4 * n):]

  def _mirror(self, x, b, n, half=None):
    """--flip_test: x[half+b : half+b+n] <- x[b : b+n] mirrored along W (ct_mirror_x), on the current stream; half =
    the step's batch (B by default)."""
    _, c, h, w = x.shape
    half = self.B if half is None else half
    L.check(L.lib().ct_mirror_x(L.ptr(x[b]), L.ptr(x[half + b]), n, c, h, w, L.stream_ptr()), 'ct_mirror_x')

  def _warp_frames(self, slot, src=None, dst=None):
    """fp32 and bf16x3 engines: the slot's frames -> its fp32 image, one ct_warp_frames_normalize for all of them from
    the slot's device descriptors, at the step's batch.  src / dst: another frame slot through this slot's descriptors,
    into another image buffer."""
    src = self.u8[slot] if src is None else src
    dst = self.img[slot] if dst is None else dst
    L.check(L.lib().ct_warp_frames_normalize(L.ptr(src), L.ptr(self.d_frames[slot]), self._n, self.slot_bytes,
                                             C.c_void_p(self.mean.ctypes.data), C.c_void_p(self.std.ctypes.data),
                                             L.ptr(dst), self.H, self.W, L.stream_ptr()), 'ct_warp_frames_normalize')

  def _graph(self, slot):
    if self.idle_g is not None:                              # one graph per (slot, batch), captured on first use
      key = (slot, self._n)
      if key not in self.idle_graphs:
        self.idle_graphs[key] = self._capture(slot)
      return self.idle_graphs[key]
    if self.graphs[slot] is None:
      self.graphs[slot] = self._capture(slot)
    return self.graphs[slot]

  def _capture(self, slot):
    saved = None
    if self.tracker is not None:                             # capture must not disturb live stream state
      saved = [t.clone() for t in self._tracker_state()]
    s = torch.cuda.Stream(device=self.device)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
      self._eager(slot)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
      self._eager(slot)
    if saved is not None:
      for t, v in zip(self._tracker_state(), saved):
        t.copy_(v)
    return g

  def _geo_tables(self):
    """The device tables that hold per-stream camera rows (the tracker, or the post-processed detections), or None."""
    return self.tracker if self.tracker is not None else self.post

  def _tracker_state(self):
    trk = self.tracker
    return [trk.tracks, trk.counts, trk.boxes] + ([trk.payload] if trk.payload is not None else [])

  def batches(self):
    """The network batches a step may run at: B, or on an idle-streams runner every padded batch."""
    return [self.B] if self.idle_g is None else sorted({self.padded_batch(n) for n in range(1, self.B + 1)})

  def warm(self):
    for n in self.batches():
      self._n = n
      for s in range(NS):
        if self.use_graph:
          self._graph(s)
        else:
          self._eager(s)
    self._n = self.B
    if self.tracker is not None:
      self.tracker.reset()
    torch.cuda.synchronize(self.device)

  def reset_tracking(self):
    self.t = 0
    self.last_slot = [None] * self.B
    if self.idle_g is not None:
      self._was_idle = set()
    if self.tracker is not None:
      self.tracker.reset()

  def _check_public(self, public_dets, idle=(), options=None):
    """public_dets: list of B arrays [P_b, 2] (the `ct` of each of the frame's public detections, image coordinates)
    -> list of B float32 arrays; ValueError when they are missing, unexpected, or more than max_public_dets.  The
    entries of `idle` streams are ignored (and may be None).  options (stream_opts runners: each stream's settings in
    this step): a stream whose public_det is off must have a None entry."""
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
      private = options is not None and not options[b]['public_det']
      if private and p is not None and b not in idle:
        raise ValueError('public_dets[%d]: stream %d runs without public_det (its stream_opts / options); its entry '
                         'must be None' % (b, b))
      if b in idle or private:
        out.append(np.zeros((0, 2), np.float32))
        continue
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

  def _check_starts(self, starts, pre_dets, options=None):
    """starts (stream indices whose frame in this step is a video's first) and pre_dets ({stream: list of result
    dicts} seeding the tracker of some of them, in each stream's source pixels like the tracks) -> (streams, seed rows)
    or None.  ValueError (device_tracker.plan_starts) before anything is enqueued; without device tracking a start only
    switches pre_images, and pre_dets are refused.  options: each stream's settings in this step (stream_opts
    runners), whose new_thresh filters its seeds."""
    if starts is None or len(starts) == 0:
      if pre_dets:
        raise ValueError('pre_dets: stream(s) %s do not start a video in this step' % sorted(pre_dets))
      return None
    if self.tracker is None:
      if pre_dets:
        raise ValueError('pre_dets seed the device tracker: this runner was built without device_tracking')
      return plan_starts(self.B, 0, 0.0, False, starts, None)
    trk = self.tracker
    nt = [o['new_thresh'] for o in options] if options is not None else self.opt.new_thresh
    return plan_starts(self.B, trk.T, nt, trk.payload is not None, starts, pre_dets)

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

  def _upload_geometry(self, slot, rows, non_blocking):
    """Stages and uploads the tracker geometry rows of the streams whose camera changes in this step (_plan_geometry)
    for slot's start prologue (the current stream is the upload's); -> the bytes uploaded."""
    self._geo[slot] = None
    if not rows or self._geo_tables() is None:
      return 0
    if self.h_geo is None:
      self.h_geo = [(torch.zeros((self.B, 6), dtype=torch.float64).pin_memory(),
                     torch.zeros((self.B, 18), dtype=torch.float32).pin_memory()) for _ in range(NS)]
      self.d_geo_in = [torch.zeros((self.B, 6), dtype=torch.float64, device=self.device) for _ in range(NS)]
      self.d_geo_out = [torch.zeros((self.B, 18), dtype=torch.float32, device=self.device) for _ in range(NS)]
    streams, cs, ss, ks = zip(*rows)
    t_in, t_out = self._geo_tables().geometry_rows(cs, ss, ks)
    n = len(streams)
    h_in, h_out = self.h_geo[slot]
    h_in[:n], h_out[:n] = torch.from_numpy(t_in), torch.from_numpy(t_out)
    self.d_geo_in[slot][:n].copy_(h_in[:n], non_blocking=non_blocking)
    self.d_geo_out[slot][:n].copy_(h_out[:n], non_blocking=non_blocking)
    self._geo[slot] = list(streams)
    return n * (6 * 8 + 18 * 4)

  def load_device_inputs(self, images, pre_hms, slot, public_dets=None, starts=None, pre_dets=None, calibs=None,
                         options=None):
    """Copies step_device's inputs into `slot` on the current stream; starts / pre_dets / calibs / options as in
    step_host."""
    planned = self._check_options(options, self._streams_arg('starts', starts) if options else ())
    now = self._step_options(planned)
    pub = self._check_public(public_dets, (), now)
    plan = self._check_starts(starts, pre_dets, now)
    cal = self._check_calibs(calibs, plan[0] if plan else ())
    self.img[slot][:self.B].copy_(images)
    if pre_hms is not None:
      self.hm[slot][:self.B].copy_(pre_hms)
    if pub is not None:
      self._fill_public(self.h_pub[slot], pub)
      self.pub[slot][0].copy_(self.h_pub[slot][0])
      self.pub[slot][1].copy_(self.h_pub[slot][1])
    _, rows = self._plan_geometry(slot, {}, cal)
    ob = self._plan_options(slot, planned)
    if ob is not None:
      self.d_opts[slot].copy_(self.h_opts[slot])
    self._start_bytes = self._upload_starts(slot, plan, non_blocking=False) + \
        self._upload_geometry(slot, rows, non_blocking=False) + (len(ob) if ob is not None else 0)

  def _start_prologue(self, slot, streams, restores=None):
    """A step whose frames start new videos on `streams` or continue restored ones ({stream: StreamState}), before the
    step itself (graph replay or eager), on the same stream: first-frame pre_images, the restored streams' frames as
    theirs, and the tracker start and restore.  Outside the graphs: they stay the same for every step.  In the first
    step (t = 0) with restores, the step runs as a later one, so every other stream's frame is copied as a start's."""
    restores = restores or {}
    prev = (slot - 1) % NS
    if self.t > 0:
      own = list(streams)
    elif restores:
      live = self._live[self.t & 1] if self.idle_g is not None else range(self.B)
      own = [b for b in live if b not in restores]
    else:
      own = []
    if restores:
      # pre_images of a restored stream = the state's frame, staged into its region of the previous slot; safe as a
      # start's copy below: the region is read by step t-1 as its images, which comes first on this stream
      self._stage_states(prev, restores)
    for b in own + sorted(restores):
      # pre_images of a started stream = its own frame: overwrite its part of the previous slot, which holds step t-1's
      # images.  Safe: that slot is read only by this step (as pre_images), after this prologue on the same stream, and
      # it is next written by the upload of step t+2, which waits for ev_done[prev], recorded after this step.
      src = (self.u8[slot] if b in own else self.u8[prev]) if self.frames_mode else None
      # the pack kernel (or, on an idle-streams runner, the pre_images warp) reads u8[prev] again
      if self.frames_mode and (self.eng.use_halo or self.idle_g is not None):
        if b in own:
          f = self.frames[b]
          o, n = f.offset, frame_layout(self.frame_format, f.h, f.w)[1]
          self.u8[prev][o:o + n].copy_(self.u8[slot][o:o + n])
        continue
      if self.frames_mode:   # the plan reads img[prev]: warp this frame into it through the slot's device descriptor
        L.check(L.lib().ct_warp_frames_normalize(
            L.ptr(src), C.c_void_p(self.d_frames[slot].data_ptr() + b * C.sizeof(L.Frame)), 1,
            self.slot_bytes, C.c_void_p(self.mean.ctypes.data), C.c_void_p(self.std.ctypes.data),
            L.ptr(self.img[prev][b]), self.H, self.W, L.stream_ptr()), 'ct_warp_frames_normalize')
      else:
        self.img[prev][b].copy_(self.img[slot][b])
      if self.flip:                                        # --flip_test: pre_images is the (frame, mirror) pair
        self._mirror(self.img[prev], b, 1)
    geo, self._geo[slot] = self._geo[slot], None
    if geo:                                                  # new cameras: before the seeds' boxes are rendered
      self._geo_tables().set_geometry(geo, self.d_geo_in[slot], self.d_geo_out[slot])
    if self.tracker is not None and streams:                 # reset + seeds + boxes: the step's render splats them
      self.tracker.start_device(self.d_start[slot], len(streams), self.d_seed[slot], opts=self._slot_opts(slot))
    if self.tracker is not None and restores:                # the exported rows, boxes at this stream and camera
      self._restore_tracks(restores, self._slot_opts(slot))

  def _on_device(self, t):
    """t on the runner's device; a tensor of another device is copied over (on the current stream)."""
    if t.device != self.u8[0].device:
      return t.to(self.u8[0].device)
    t.record_stream(torch.cuda.current_stream(self.device))  # the caller may drop the state once step_frames returns
    return t

  def _stage_states(self, dst_slot, restores):
    """The restored streams' frames -> their regions of u8[dst_slot] (one ct_stage_frames), on the current stream."""
    bs = sorted(restores)
    frames = [self._on_device(restores[b].frame) for b in bs]
    srcs = (L.FrameSrc * len(bs))(*[device_frame_source(x, self.frame_format, 'bgr', x.device)[1] for x in frames])
    dst = (L.Frame * len(bs))(*[self.frames[b] for b in bs])
    L.check(L.lib().ct_stage_frames(srcs, dst, len(bs), L.ptr(self.u8[dst_slot]), self.slot_bytes, L.stream_ptr()),
            'ct_stage_frames')

  def _restore_tracks(self, restores, opts=None):
    """ct_track_restore of the restored streams' rows, on the current stream."""
    bs = sorted(restores)
    ent = torch.tensor([[b, restores[b].counts[0], restores[b].counts[1]] for b in bs], dtype=torch.int32)
    rows = [restores[b].tracks for b in bs if restores[b].counts[0]]
    pay = [restores[b].payload for b in bs if restores[b].counts[0]] if self.tracker.payload is not None else []
    rows = torch.cat([self._on_device(r) for r in rows]) if rows else None
    pay = torch.cat([self._on_device(p) for p in pay]) if pay else None
    self.tracker.restore_device(ent.to(self.device), len(bs), rows, pay, opts=opts)

  def _launch(self, slot):
    streams, self._starts[slot] = self._starts[slot], None
    restores, self._restores[slot] = self._restores[slot], None
    if streams or restores:
      self._start_prologue(slot, streams or [], restores)
    if self.t == 0 and not restores:
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

  def step_host(self, images, pre_hms=None, public_dets=None, starts=None, pre_dets=None, calibs=None, options=None):
    """images [B,3,H,W] (and pre_hms [B,1,H,W] unless device_tracking): float32 HOST tensors (what
    Detector.pre_process / _get_additional_inputs produce); with --public_det, public_dets = B arrays [P_b, 2] (the
    `ct`s of each frame's public detections).  starts: the streams whose frame in this step is a new video's first
    (Detector.reset_tracking on those streams alone: the frame is its own pre_images and the stream's tracker restarts
    empty, or from pre_dets = {stream: list of result dicts} as Tracker.init_track; the other streams are unaffected).
    calibs: {stream: [3, 4] camera matrix} of some started streams, their camera from this frame on (3D head sets:
    loc, rot_y); a started stream without one keeps its camera.
    options: {stream: flags} of some started streams (runners built with stream_opts): their tracker settings from this
    frame on, resolved against opt as the constructor's stream_opts entries are; a started stream without one keeps
    its settings.  ValueError, before anything is enqueued, for a stream that does not start, a key or value
    resolve_options refuses, a max_age above the track table's capacity, or public_det on a runner that stages no
    public detections.
    Returns the records of the PREVIOUS call (None the first time) -- a one-step software pipeline: this step's H2D
    overlaps the previous step's compute."""
    if self.idle_g is not None:
      raise ValueError('step_host: a runner built with idle_streams takes raw frames (step_frames)')
    planned = self._check_options(options, self._streams_arg('starts', starts) if options else ())
    now = self._step_options(planned)
    pub = self._check_public(public_dets, (), now)
    plan = self._check_starts(starts, pre_dets, now)
    cal = self._check_calibs(calibs, plan[0] if plan else ())
    slot = self.t % NS
    _, rows = self._plan_geometry(slot, {}, cal)
    ob = self._plan_options(slot, planned)
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
      self._start_bytes = self._upload_starts(slot, plan, non_blocking=True) + \
          self._upload_geometry(slot, rows, non_blocking=True) + self._upload_options(slot, ob)
      self.ev_in[slot].record(self.copy)
    return self._submit(slot)

  def _upload_options(self, slot, ob):
    """Uploads slot's staged ct_track_opts records (_plan_options) when they changed, on the current (copy) stream;
    -> the bytes uploaded."""
    if ob is None:
      return 0
    self.d_opts[slot].copy_(self.h_opts[slot], non_blocking=True)
    return len(ob)

  def _submit(self, slot):
    """The step of the uploaded slot on the compute stream and the D2H of its results; -> the previous step's
    records."""
    prev = self.fetch() if self.t > 0 else None
    with torch.cuda.stream(self.compute):
      self.compute.wait_event(self.ev_in[slot])
      self._launch(slot)
      if self._n == self.B:
        self.h_rec[self.t & 1].copy_(self.rec, non_blocking=True)
      else:                                          # the step's [n, K, F]; fetch() expands them to the streams
        self.h_rec[self.t & 1][:self._n].copy_(self.rec[:self._n], non_blocking=True)
      if self.tracker is not None:
        self.h_trk[self.t & 1].copy_(self.tracker.tracks, non_blocking=True)
        self.h_cnt[self.t & 1].copy_(self.tracker.counts, non_blocking=True)
        if self.tracker.payload is not None:
          self.h_pay[self.t & 1].copy_(self.tracker.payload, non_blocking=True)
      if self.post is not None:
        self.h_det[self.t & 1].copy_(self.post.dets, non_blocking=True)
        self.h_det_cnt[self.t & 1].copy_(self.post.counts, non_blocking=True)
        if self.post.payload is not None:
          self.h_det_pay[self.t & 1].copy_(self.post.payload, non_blocking=True)
      if self.crop is not None:
        self.h_crop_cnt[self.t & 1].copy_(self.crop_counts, non_blocking=True)
      # this step's pre_images slot may be overwritten once this step is done
      self.ev_done[(slot - 1) % NS].record(self.compute)
    self.t += 1
    return prev

  def frame_buffers(self, sizes=None):
    """Frames mode: numpy views [h_b, w_b, 3] uint8 ([3h_b/2, w_b] with frame_format 'nv12' or 'i420') of the pinned
    staging the NEXT step_frames uploads, one per stream,
    for a decoder to write its frames in place; then call step_frames(None).  They may be written once the previous
    step_frames call has returned (its upload of three steps ago, which last read this staging, has completed by
    then) and until the next step_frames call.  sizes ({stream: (h, w)}, capacity runners): the views of those streams
    at a new size, for frames that start a video; the next step_frames(None, starts=...) must start them."""
    if not self.frames_mode:
      raise ValueError('frame_buffers(): the runner was not built with frame_sizes')
    now = list(self.frame_sizes)
    for b, hw in (sizes or {}).items():
      if not 0 <= b < self.B:
        raise ValueError('sizes: stream %r out of range [0, %d)' % (b, self.B))
      hw = (int(hw[0]), int(hw[1]))
      if hw != now[b]:
        if self.cap is None:
          raise ValueError('sizes[%d]: the frame sizes of a runner built without max_frame_size are fixed' % b)
        self._size_geometry('sizes[%d]' % b, *hw)
      now[b] = hw
    self._pending_sizes = now
    return self._views(self.t % NS, now)

  def _views(self, slot, sizes):
    buf = self.h_u8[slot].numpy()
    views = []
    for f, (h, w) in zip(self.frames, sizes):
      shape, n, _ = frame_layout(self.frame_format, h, w)
      views.append(buf[f.offset:f.offset + n].reshape(shape))
    return views

  def _frame_sizes_of(self, frames, idle=()):
    """This step's (h, w) per stream: the shapes of `frames`, or the sizes of the last frame_buffers() call when None.
    ValueError on a wrong count or dtype, or a shape that is not [h, w, 3] ([3h/2, w] with R = 3h/2 a multiple of 3 and
    w even, in a 4:2:0 frame_format).  `idle` streams keep their size and their entries are not looked at."""
    if frames is None:
      sizes = list(getattr(self, '_pending_sizes', None) or self.frame_sizes)
      return [self.frame_sizes[b] if b in idle else hw for b, hw in enumerate(sizes)]
    if len(frames) != self.B:
      raise ValueError('frames: expected %d arrays (one per stream), got %d' % (self.B, len(frames)))
    sizes = []
    for b, (a, (h, w)) in enumerate(zip(frames, self.frame_sizes)):
      if b in idle:
        sizes.append((h, w))
        continue
      if not isinstance(a, np.ndarray) or a.dtype != np.uint8:
        raise ValueError('frames[%d]: expected a uint8 numpy array, got %s' %
                         (b, getattr(a, 'dtype', type(a).__name__)))
      if self.cap is None and a.shape != (h, w, 3):
        raise ValueError('frames[%d]: expected shape %s, got %s' % (b, (h, w, 3), a.shape))
      hw = frame_size_of(self.frame_format, a.shape)
      if hw is None and self.frame_format == 'bgr':
        raise ValueError('frames[%d]: expected shape [h, w, 3], got %s' % (b, a.shape))
      if hw is None:
        raise ValueError('frames[%d]: expected a %s frame of shape [3h/2, w] (rows a multiple of 3, w even), got %s' %
                         (b, self.frame_format.upper(), a.shape))
      sizes.append(hw)
    return sizes

  def _check_idle(self, idle, started, pre_hms):
    """idle (the streams without a frame in this step) -> the live streams, ascending, or None on a runner built
    without idle_streams.  ValueError before anything is enqueued: idle on such a runner, pre_hms on an idle-streams
    runner, a stream out of range or repeated, every stream idle, a stream both idle and started, or a stream that was
    idle in the last step and comes back without a video start."""
    if self.idle_g is None:
      if idle is not None:
        raise ValueError('idle: this runner was built without idle_streams')
      return None
    if pre_hms is not None:
      raise ValueError('pre_hms: a runner built with idle_streams renders its prior heat-maps itself (device_tracking) '
                       'or runs without them')
    gone = set()
    for s in idle or ():
      if isinstance(s, (bool, np.bool_)) or not isinstance(s, (int, np.integer)):
        raise ValueError('idle: stream indices must be integers, got %r' % (s,))
      s = int(s)
      if not 0 <= s < self.B:
        raise ValueError('idle: stream %d out of range [0, %d)' % (s, self.B))
      if s in gone:
        raise ValueError('idle: stream %d given twice' % s)
      gone.add(s)
    if len(gone) == self.B:
      raise ValueError('idle: every stream is idle; a step needs at least one frame')
    both = sorted(gone & set(started))
    if both:
      raise ValueError('idle: stream(s) %s also start a video in this step' % both)
    live = [b for b in range(self.B) if b not in gone]
    back = [b for b in live if b in self._was_idle and b not in started]
    if back:
      raise ValueError('stream(s) %s were idle in the last step: an idle stream comes back only with a video start '
                       '(starts=)' % back)
    return live

  def _streams_arg(self, what, streams):
    """A list of distinct stream indices in [0, B) (None: empty); ValueError otherwise."""
    out = []
    for s in (() if streams is None else streams):
      if isinstance(s, (bool, np.bool_)) or not isinstance(s, (int, np.integer)):
        raise ValueError('%s: stream indices must be integers, got %r' % (what, s))
      s = int(s)
      if not 0 <= s < self.B:
        raise ValueError('%s: stream %d out of range [0, %d)' % (what, s, self.B))
      if s in out:
        raise ValueError('%s: stream %d given twice' % (what, s))
      out.append(s)
    return out

  def _check_resume(self, resume, started, idle, restored):
    """resume (streams idle in the last step whose frame in this step continues their video) -> the streams, ascending.
    ValueError before anything is enqueued: resume on a runner without idle_streams, a stream that is also started,
    restored or idle, one that was live in the last step, or one without a frame since the runner was built or reset.
    (A frame of another size than the stream's last is refused by _check_sizes.)"""
    out = self._streams_arg('resume', resume)
    if not out:
      return []
    if self.idle_g is None:
      raise ValueError('resume: this runner was built without idle_streams (its streams are never idle)')
    for what, other in (('start a video (starts=)', started), ('are idle (idle=)', idle or ()),
                        ('are restored (restore=)', restored)):
      both = sorted(set(out) & _ints(other))
      if both:
        raise ValueError('resume: stream(s) %s also %s in this step' % (both, what))
    live = sorted(set(out) - self._was_idle)
    if live:
      raise ValueError('resume: stream(s) %s were live in the last step; resume continues a stream that was idle' %
                       live)
    new = [b for b in out if self.last_slot[b] is None]
    if new:
      raise ValueError('resume: stream(s) %s have had no frame since the runner was built or reset; they come back with '
                       'a video start' % new)
    return sorted(out)

  def _plan_resume(self, slot, live, resumed):
    """Host bookkeeping of step t = self.t in `slot`: the copies that put each resumed stream's last frame where this
    step reads pre_images -- [(stream, source slot, destination slot, byte offset, bytes)] for the streams whose last
    slot is not the previous slot (t-1) % 3 -- and then last_slot of this step's live streams (every stream when live is
    None) <- slot."""
    dst = (self.t - 1) % NS
    out = []
    for b in resumed:
      if self.last_slot[b] != dst:
        f = self.frames[b]
        out.append((b, self.last_slot[b], dst, f.offset, frame_layout(self.frame_format, f.h, f.w)[1]))
    for b in (range(self.B) if live is None else live):
      self.last_slot[b] = slot
    return out

  def _copy_resumed(self, copies):
    """One ct_stage_frames of the resumed streams' last frames (_resume_copies) from their last slots into the previous
    slot, on the current (copy) stream, before this step's frames are written."""
    srcs, dsts = (L.FrameSrc * len(copies))(), (L.Frame * len(copies))()
    for i, (b, s, _, o, n) in enumerate(copies):
      f = self.frames[b]
      view = self.u8[s][o:o + n].view(frame_layout(self.frame_format, f.h, f.w)[0])
      srcs[i], dsts[i] = device_frame_source(view, self.frame_format, 'bgr', view.device)[1], f
    L.check(L.lib().ct_stage_frames(srcs, dsts, len(copies), L.ptr(self.u8[copies[0][2]]), self.slot_bytes,
                                    L.stream_ptr()), 'ct_stage_frames')

  def _check_restore(self, restore, started, idle):
    """restore ({stream: StreamState}) -> {stream: StreamState}.  ValueError before anything is enqueued: a runner
    without max_frame_size, a stream out of range, also started or idle, or a state whose network input, record or
    payload layout, tracker or frame_format differ from this runner's, with more rows than the track table, or whose
    frame does not fit the capacity region or map to (H, W)."""
    if not restore:
      return {}
    if self.cap is None:
      raise ValueError('restore: needs a capacity frames runner (frame_sizes and max_frame_size)')
    out = {}
    for s in self._streams_arg('restore', list(restore)):
      st = restore[s]
      if not isinstance(st, StreamState):
        raise ValueError('restore[%d]: expected a StreamState (stream_state()), got %s' % (s, type(st).__name__))
      out[s] = st
    for what, other in (('start a video (starts=)', started), ('are idle (idle=)', idle or ())):
      both = sorted(set(out) & _ints(other))
      if both:
        raise ValueError('restore: stream(s) %s also %s in this step' % (both, what))
    pay = self.tracker.payload_layout if self.tracker is not None else None
    for s, st in sorted(out.items()):
      if st.input_size != (self.H, self.W):
        raise ValueError('restore[%d]: network input %s, the runner\'s is %s' % (s, st.input_size, (self.H, self.W)))
      if st.record_layout != self.layout:
        raise ValueError('restore[%d]: record layout %s differs from the runner\'s %s' % (s, st.record_layout,
                                                                                         self.layout))
      if st.frame_format != self.frame_format:
        raise ValueError('restore[%d]: frame_format %r, the runner\'s is %r' % (s, st.frame_format, self.frame_format))
      if (st.tracks is None) != (self.tracker is None):
        raise ValueError('restore[%d]: the state %s track table and the runner %s a tracker' %
                         (s, 'has no' if st.tracks is None else 'has a', 'has' if self.tracker else 'has no'))
      if st.payload_layout != pay:
        raise ValueError('restore[%d]: payload layout %s differs from the runner\'s %s' % (s, st.payload_layout, pay))
      if self.tracker is not None and not 0 <= st.counts[0] <= self.tracker.T:
        raise ValueError('restore[%d]: %d track rows, more than the %d of the track table' % (s, st.counts[0],
                                                                                            self.tracker.T))
      self._size_geometry('restore[%d]' % s, *st.size)
    return out

  def _restore_options(self, rest):
    """{stream: resolved settings} the restored states carry, on a runner built with stream_opts; ValueError as
    check_options.  A runner built without stream_opts runs its own opt on every stream, restored ones included."""
    tables = self._geo_tables()
    if not self._per_stream():
      return {}
    return {s: tables.check_options(st.options, 'restore[%d]' % s, resolved=True)
            for s, st in sorted(rest.items()) if st.options is not None}

  def stream_state(self, b):
    """Waits like fetch(), then returns stream b's StreamState after the last submitted step in which it had a frame:
    that frame (a device copy), its size and camera, and on a tracking runner its track rows, counts and payload rows.
    step_frames(restore={s: state}) on this or another runner continues the video on stream s from its next frame.
    ValueError on a runner without max_frame_size, or a stream that has had no frame since the runner was built or
    reset."""
    if self.cap is None:
      raise ValueError('stream_state: needs a capacity frames runner (frame_sizes and max_frame_size)')
    b = self._streams_arg('stream_state', [b])[0]
    s = self.last_slot[b]
    if s is None:
      raise ValueError('stream_state: stream %d has had no frame since the runner was built or reset' % b)
    self.compute.synchronize()
    f = self.frames[b]
    shape, n, _ = frame_layout(self.frame_format, f.h, f.w)
    trk = self.tracker
    counts = tuple(int(v) for v in trk.counts[b].cpu()) if trk is not None else None
    with torch.cuda.stream(self.compute):
      frame = self.u8[s][f.offset:f.offset + n].clone().view(shape)
      tracks = trk.tracks[b, :counts[0]].clone() if trk is not None else None
      pay = trk.payload[b, :counts[0]].clone() if trk is not None and trk.payload is not None else None
    self.compute.synchronize()
    return StreamState(frame, (f.h, f.w), np.array(self._meta[b]['calib'], np.float32).reshape(3, 4), tracks, counts,
                       pay, (self.H, self.W), dict(self.layout), trk.payload_layout if trk is not None else None,
                       trk.T if trk is not None else None, self.frame_format,
                       self._geo_tables().options[b] if self._geo_tables() is not None else None)

  def step_frames(self, frames, pre_hms=None, public_dets=None, starts=None, pre_dets=None, calibs=None, idle=None,
                  layout='bgr', resume=None, restore=None, options=None):
    """frames: B uint8 [h_b, w_b, 3] BGR arrays of the sizes given as frame_sizes (with frame_format 'nv12' / 'i420':
    [3h_b/2, w_b] arrays in that layout), or None when they were written through frame_buffers(), or B device frames
    (below).  pre_hms, public_dets, starts, pre_dets, calibs and the return value as in step_host;
    public detections and pre_dets are in each stream's source pixels, and so are the tracks.  On a runner built with
    max_frame_size, a stream in `starts` may bring a frame of another size (that fits the region and maps to (H, W));
    without a calibs entry it then gets Detector._get_default_calib of that size.  ValueError (before anything is
    enqueued) on a wrong count, dtype or shape, a size change that is not allowed, or when the runner was not built
    with frame_sizes.
    idle (runners built with idle_streams): the streams without a frame in this step; their frames and public_dets
    entries are ignored (and may be None), their tables, camera and frame region are left as they are, and their
    records come back zero and their fetch_results() entries None.  A stream idle in one step comes back with a video
    start, or in `resume`: its frame continues its video, and its records, tracks (ids, ages) and payload are those of
    the stream fed only the frames it delivered, one after the other (tracks age per frame, not per step).  A resumed
    frame has the size of the stream's last one.
    restore ({stream: StreamState}, capacity runners): each listed stream continues the video of the state
    (stream_state() of this or another runner, on any device) with this step's frame, of the state's size: a video start
    at the state's size and camera whose pre_images is the state's frame and whose tracker gets the state's rows as they
    are (ids, ages, id counter).  Refused, before anything is enqueued, together with starts, resume or idle for the
    same stream, or for a state of another network input, head set, track table or frame_format.
    Device frames (what GPU decoders hand out): uint8 CUDA tensors on the runner's device instead of arrays, for every
    stream with a frame in this step (a step never mixes the two).  A BGR runner takes [h, w, 3] with layout 'bgr' or
    'rgb', or [3, h, w] with layout 'rgb_planar'; an NV12 runner one [3h/2, w] tensor in cv2's layout or the planes
    (Y [h, w], UV [h/2, w]); an I420 runner one [3h/2, w] tensor of rows of exactly w bytes or the planes
    (Y [h, w], U [h/2, w/2], V [h/2, w/2]).  options as in step_host; a restored stream takes the state's options.
    Rows may have any pitch (views of wider or taller surfaces); the innermost
    stride must be 1 (device_frame_source).  One ct_stage_frames copies them into the slot on the runner's copy stream,
    after the work queued on the caller's current stream at this call (which writes the frames); nothing of them is
    uploaded, and the step computes bit for bit what it computes on the same frames given as arrays (RGB swapped to
    BGR).  The tensors may be freed after the call (the caching allocator keeps their memory until the copy has run), but
    memory the caller reuses itself, such as a decoder's surface pool, must not be written again before frames_read()
    has completed: make the decoder's stream wait on it."""
    if not self.frames_mode:
      raise ValueError('step_frames: the runner was not built with frame_sizes (use step_host)')
    planned = self._check_options(options, self._streams_arg('starts', starts) if options else ())
    rest = self._check_restore(restore, self._streams_arg('starts', starts), idle)
    planned.update(self._restore_options(rest))
    now = self._step_options(planned)
    plan = self._check_starts(starts, pre_dets, now)
    started = plan[0] if plan else ()
    resumed = self._check_resume(resume, started, idle, rest)
    live = self._check_idle(idle, list(started) + sorted(rest) + resumed, pre_hms)
    gone = () if live is None else set(range(self.B)) - set(live)
    pub = self._check_public(public_dets, gone, now)
    cal = self._check_calibs(calibs, started)
    cal.update((b, np.asarray(st.calib, np.float32)) for b, st in rest.items())   # a restore: the state's camera
    dev = None                                       # device frames: [(stream, ct_frame_src, tensors)]
    if frames is not None and self._device_step(frames, gone):
      sizes, dev = self._device_sources(frames, gone, layout)
    else:
      if layout != 'bgr':
        raise ValueError("layout=%r: applies to device frames; arrays are in the runner's frame_format" % (layout,))
      sizes = self._frame_sizes_of(frames, gone)
    for b, st in sorted(rest.items()):
      if tuple(sizes[b]) != st.size:
        raise ValueError('restore[%d]: the frame of this step is %s, the state\'s video %s' % (b, tuple(sizes[b]),
                                                                                             st.size))
    changed = self._check_sizes(sizes, list(started) + sorted(rest))
    slot = self.t % NS
    self._pending_sizes = None
    desc, rows = self._plan_geometry(slot, changed, cal, live)
    ob = self._plan_options(slot, planned)
    copies = self._plan_resume(slot, live, resumed)
    self._restores[slot] = rest or None
    maps = None
    if live is not None:
      self._was_idle = set(gone)
      self._n = self.padded_batch(len(live))
      self._live[self.t & 1] = live
      now = self._maps(live).tobytes()
      if now != self._map_mirror[slot]:
        maps = self._map_mirror[slot] = now
        self.h_map[slot].numpy()[:] = np.frombuffer(maps, np.int32)
    if frames is not None and dev is None:
      # the slot's staging was last read by step t-3's upload, which the last fetch() waited for
      for b, (a, v) in enumerate(zip(frames, self._views(slot, self.frame_sizes))):
        if b not in gone:
          np.copyto(v, a)
    if desc is not None:
      self.h_frames[slot].numpy()[:] = np.frombuffer(desc, np.uint8)
    if pub is not None:
      self._fill_public(self.h_pub[slot], pub)
    use_hm = self.tracker is None and pre_hms is not None
    src_hm = pre_hms
    if use_hm and not pre_hms.is_pinned():
      self.h_hm[slot].copy_(pre_hms)
      src_hm = self.h_hm[slot]
    caller = torch.cuda.current_stream(self.device)
    with torch.cuda.stream(self.copy):
      self.copy.wait_event(self.ev_done[slot])       # slot's old contents were last read as pre_images of step t-2
      if copies:                                     # resumed streams' last frames -> pre_images, before any frame of
        self._copy_resumed(copies)                   # this step is written (a source may be this slot: DESIGN §5)
      if dev is not None:                            # staged from the caller's tensors once its stream has written them
        self.copy.wait_stream(caller)
        self._stage_frames(slot, dev)
      self._frame_bytes = 0                          # the used bytes only, and the descriptors when they changed
      for a, e in (self._upload_runs(live) if dev is None else ()):
        self.u8[slot][a:e].copy_(self.h_u8[slot][a:e], non_blocking=True)
        self._frame_bytes += e - a
      if desc is not None:
        self.d_frames[slot].copy_(self.h_frames[slot], non_blocking=True)
        self._frame_bytes += len(desc)
      if maps is not None:
        self.d_map[slot].copy_(self.h_map[slot], non_blocking=True)
        self._frame_bytes += len(maps)
      if use_hm:
        self.hm[slot][:self.B].copy_(src_hm, non_blocking=True)
      if pub is not None:
        self.pub[slot][0].copy_(self.h_pub[slot][0], non_blocking=True)
        self.pub[slot][1].copy_(self.h_pub[slot][1], non_blocking=True)
      self._start_bytes = self._upload_starts(slot, plan, non_blocking=True) + \
          self._upload_geometry(slot, rows, non_blocking=True) + (12 * len(rest) if self.tracker is not None else 0) + \
          self._upload_options(slot, ob)
      self.ev_in[slot].record(self.copy)
    return self._submit(slot)

  def _device_step(self, frames, idle):
    """Whether this step's frames are device frames; ValueError on a wrong count or when the live streams' entries mix
    device tensors and arrays."""
    if len(frames) != self.B:
      raise ValueError('frames: expected %d arrays (one per stream), got %d' % (self.B, len(frames)))
    kinds = [(b, is_device_frame(a)) for b, a in enumerate(frames) if b not in idle]
    dev, host = [b for b, k in kinds if k], [b for b, k in kinds if not k]
    if dev and host:
      raise ValueError('frames: stream(s) %s bring device tensors and stream(s) %s host arrays; a step takes uint8 '
                       "tensors on the runner's device for all its streams or uint8 numpy arrays for all" % (dev, host))
    return bool(dev)

  def _device_sources(self, frames, idle, layout):
    """Device frames -> (this step's (h, w) per stream, [(stream, ct_frame_src, tensors)] of the live streams);
    ValueError (device_frame_source) before anything is enqueued.  `idle` streams keep their size."""
    sizes, out = [], []
    for b, (x, hw) in enumerate(zip(frames, self.frame_sizes)):
      if b in idle:
        sizes.append(hw)
        continue
      size, src = device_frame_source(x, self.frame_format, layout, self.u8[0].device, 'frames[%d]' % b)
      sizes.append(size)
      out.append((b, src, x if isinstance(x, tuple) else (x,)))
    return sizes, out

  def _stage_frames(self, slot, dev):
    """ct_stage_frames of the device frames `dev` (_device_sources) into u8[slot], each at its stream's region in the
    descriptor this step gives it, on the current (copy) stream; the source tensors are marked used by that stream."""
    n = len(dev)
    srcs = (L.FrameSrc * n)(*[s for _, s, _ in dev])
    dst = (L.Frame * n)(*[self.frames[b] for b, _, _ in dev])
    L.check(L.lib().ct_stage_frames(srcs, dst, n, L.ptr(self.u8[slot]), self.slot_bytes, L.stream_ptr()),
            'ct_stage_frames')
    for _, _, ts in dev:
      for t in ts:
        t.record_stream(self.copy)
    if self._ev_read is None:
      self._ev_read = torch.cuda.Event()
    self._ev_read.record(self.copy)

  def frames_read(self):
    """The torch.cuda.Event recorded on the copy stream after the last step_frames call that took device frames (None
    before the first): once it has completed, that call's source tensors have been read and their memory may be
    written again.  A decoder that recycles its surfaces makes its stream wait on it (stream.wait_event)."""
    return self._ev_read

  def fetch(self, copy=True):
    """Blocks until the last submitted step finished; returns its records as numpy [B,K,F].  A copy by default: the
    two pinned buffers are reused by the asynchronous D2H of later steps (copy=False hands out the pinned view, valid
    until the step after next is submitted)."""
    self.compute.synchronize()
    rec = self.h_rec[(self.t - 1) & 1].numpy()
    live = self._live_of(self.t - 1)
    if live is not None:                             # idle streams: zero rows
      out = np.zeros_like(rec)
      out[live] = rec[:len(live)]
      return out
    return rec.copy() if copy else rec

  def _live_of(self, t):
    """The live streams of step t (one of the last two), or None when every stream had a frame."""
    if self.idle_g is None:
      return None
    live = self._live[t & 1]
    return None if live is None or len(live) == self.B else live

  def _idle_of(self, t):
    live = self._live_of(t)
    return () if live is None else set(range(self.B)) - set(live)

  def _results(self, t):
    i = t & 1
    if self.post is not None:
      pay = self.h_det_pay[i].numpy() if self.post.payload is not None else None
      return self.post.results(self.h_det[i].numpy(), self.h_det_cnt[i].numpy(), pay, self._idle_of(t))
    if self.tracker is None:
      raise ValueError('results: the runner was built without device_tracking or device_post_process')
    pay = self.h_pay[i].numpy() if self.tracker.payload is not None else None
    return self.tracker.results(self.h_trk[i].numpy(), self.h_cnt[i].numpy(), pay, self._idle_of(t))

  def fetch_tracks(self):
    """(tracks [B,T,CT_TRK_FLOATS], counts [B,2]) of the last submitted step (device_tracking), as numpy copies."""
    self.compute.synchronize()
    i = (self.t - 1) & 1
    return self.h_trk[i].numpy().copy(), self.h_cnt[i].numpy().copy()

  def fetch_detections(self):
    """(dets [B,K,CT_DET_FLOATS], counts [B], payload [B,K,Wp] or None) of the last submitted step
    (device_post_process), as numpy copies: stream b's detections are its first counts[b] rows.  A stream that was idle
    in that step has count 0."""
    if self.post is None:
      raise ValueError('fetch_detections(): the runner was built without device_post_process')
    self.compute.synchronize()
    return self._detections(self.t - 1)

  def previous_detections(self):
    """After a step_host / step_frames call: fetch_detections() of the step before it, without a wait (as
    previous_results())."""
    if self.post is None:
      raise ValueError('previous_detections(): the runner was built without device_post_process')
    if self.t < 2:
      raise ValueError('previous_detections(): fewer than two steps submitted')
    return self._detections(self.t - 2)

  def _detections(self, t):
    i = t & 1
    cnt = self.h_det_cnt[i].numpy().copy()
    cnt[sorted(self._idle_of(t))] = 0
    pay = self.h_det_pay[i].numpy().copy() if self.post.payload is not None else None
    return self.h_det[i].numpy().copy(), cnt, pay

  def fetch_results(self):
    """The last submitted step's tracks (device_tracking), or detections (device_post_process), as the host path's
    per-stream lists of dicts (DeviceTracker.results, DeviceDetections.results), payload fields included; None for a
    stream that was idle in that step."""
    self.compute.synchronize()
    return self._results(self.t - 1)

  def previous_results(self):
    """After a step_host / step_frames call: the tracks (or detections) of the step before it, as fetch_results()
    gives them.  No wait: the call returned once that step had finished (its records are what the call returned), and
    its tables are not overwritten before the next call."""
    if self.t < 2:
      raise ValueError('previous_results(): fewer than two steps submitted')
    return self._results(self.t - 2)

  def fetch_crops(self):
    """(crops, counts) of the last submitted step (crop_size runners); waits as fetch_results() does.  crops: the
    device uint8 view [B, K, out_h, out_w, 3] of that step's crop buffer, BGR, crop k of stream b being the box of
    fetch_results()[b][k]; counts: numpy int32 [B], 0 for a stream that was idle in that step.  Crops at or beyond
    counts[b] are stale.  The view is not a copy: a step's crops stay unchanged until its input slot is reused, by the
    step submitted three steps later, whose graph rewrites them: they stay valid while the next two steps are submitted,
    and work the caller queues on its own stream that reads them must have finished before the third is.
    With crop_format: (batch, counts), batch being the device view [N, 3, out_h, out_w] of that step's packed batch in
    the format's dtype, N = counts.sum(): stream b's crops are batch[counts[:b].sum():counts[:b + 1].sum()], in the
    order above.  The same lifetime."""
    if self.crop is None:
      raise ValueError('fetch_crops(): the runner was built without crop_size')
    if self.t < 1:
      raise ValueError('fetch_crops(): no step submitted')
    self.compute.synchronize()
    return self._crops_of(self.t - 1)

  def previous_crops(self):
    """After a step_frames call: fetch_crops() of the step before it, without a wait (as previous_results())."""
    if self.crop is None:
      raise ValueError('previous_crops(): the runner was built without crop_size')
    if self.t < 2:
      raise ValueError('previous_crops(): fewer than two steps submitted')
    return self._crops_of(self.t - 2)

  def _crops_of(self, t):
    cnt = self.h_crop_cnt[t & 1].numpy().copy()
    cnt[sorted(self._idle_of(t))] = 0
    if self.crop_format is not None:                         # the idle streams have no rows in the batch
      return self.crops[t % NS][:int(cnt.sum())], cnt
    return self.crops[t % NS], cnt

  @property
  def h2d_bytes_per_step(self):
    """Bytes uploaded per step: the frames (and pre_hm / public detections); a step that starts videos with device
    tracking also uploads its start list and seed rows (and the tracker geometry rows of streams whose camera
    changes), counted here after that step is submitted.  A capacity runner uploads the bytes its streams' frames use,
    plus the slot's descriptors in a step where they changed; an idle-streams runner the live streams' frames, plus the
    descriptors and stream maps when they changed.  A frame's bytes are those of its frame_format: h * w * 3 / 2 in
    NV12 / I420.  A step fed device frames uploads none of its frames' bytes."""
    pub = self.B * (self.tracker.max_public * 2 + 1) * 4 if self.public else 0
    hm = self.B * self.H * self.W * 4 if self.tracker is None else 0
    if self.frames_mode:
      return self._frame_bytes + hm + pub + self._start_bytes
    return self.B * 3 * self.H * self.W * 4 + hm + pub + self._start_bytes

  @property
  def d2h_bytes_per_step(self):
    tables = self._geo_tables()
    return self.rec.numel() * 4 + (tables.d2h_bytes if tables is not None else 0) + (self.B * 4 if self.crop else 0)

  def views(self, rec_np):
    from .decode import views_from_records
    return {k: v.numpy() for k, v in views_from_records(torch.from_numpy(rec_np), self.layout).items()}
