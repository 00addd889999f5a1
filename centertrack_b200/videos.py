"""track_videos: many videos of different lengths through one StreamRunner, each video on one stream from its first
frame to its last -- the batched form of the reference's evaluation loop (src/test.py prefetch_test: reset_tracking and
init_track(pre_dets) at each video's first frame, then Detector.run on every frame).

A video goes to the first free stream (in frames mode, a free stream whose frame_sizes entry is the video's frame
size; on a runner built with max_frame_size, any free stream, whose frame size changes at the start) and starts there
with StreamRunner's `starts=` / `pre_dets=` / `calibs=`; when it ends, the stream takes the next video in the same step.
A stream with no video re-feeds its last frame and its results are dropped; on a runner built with idle_streams it is
marked idle instead, and the step computes only the streams that play a video.  In frames mode the videos' frames may
instead be device frames (CUDA tensors, StreamRunner.step_frames), all videos of one call being of one kind.  The runner's one-step pipeline is kept:
the upload of step t+1 overlaps step t, and step t's tracks are yielded after step t+1 is submitted.
"""
import numpy as np
import torch

from .runner import device_frame_source, frame_layout, frame_size_of, is_device_frame


class Video(object):
  """One video: `id`, `frames` (an iterable: uint8 [h, w, 3] BGR arrays in frames mode -- [3h/2, w] NV12 / I420 arrays
  on a runner of that frame_format, or device frames as step_frames takes them --, pre-processed fp32 [3, H, W] images otherwise), optional `pre_dets` (result dicts seeding the tracker at the first frame, as the reference's
  --load_results does), `public_dets` (per frame, the [P, 2] centres of its public detections, for --public_det) and
  `calib` (the [3, 4] camera matrix of its frames).  Without `calib` the video runs in whatever camera its stream
  has: Detector._get_default_calib of its frame size when that size differs from the stream's last one, otherwise the
  stream's current camera -- which may be the `calib` of the previous video on that stream.  When some videos of a
  dataset carry a calib, give every video one (e.g. detector.default_calib of its size) so that its camera does not
  depend on the stream it lands on.
  `options`: the tracker flags the video runs with (StreamRunner's options= at its start: track_thresh, out_thresh,
  pre_thresh, new_thresh, max_age, hungarian, public_det), on a runner built with stream_opts; on such a runner a video
  without options runs the runner's opt, whichever stream it lands on."""

  def __init__(self, id, frames, pre_dets=None, public_dets=None, calib=None, options=None):
    self.id, self.frames, self.pre_dets, self.public_dets = id, frames, pre_dets, public_dets
    self.calib, self.options = calib, options


class _Playing(object):
  """A video on a stream: its frame iterator, the frame the next step feeds, and that frame's index."""

  def __init__(self, video, it, first):
    self.video, self.it, self.frame, self.index = video, it, first, 0


def _as_video(v):
  return v if isinstance(v, Video) else Video(**v)


def _stream_crops(runner, cut, b):
  """Stream b's crops of fetch_crops()' (crops, counts): its rows of the packed batch with crop_format."""
  crops, counts = cut
  if getattr(runner, 'crop_format', None) is not None:
    start = int(counts[:b].sum())
    return crops[start:start + int(counts[b])]
  return crops[b, :counts[b]]


def track_videos(runner, videos, layout='bgr', crops=False):
  """runner: a StreamRunner with device tracking, or with device_post_process (detection models: each frame's
  detections, and no video may bring pre_dets); videos: an iterable of Video (or dicts of its fields).  Yields
  (video id, frame index, results) for every frame of every video exactly once, as its tracks come back; results is the
  list of dicts fetch_results() gives for that stream (in source pixels in frames mode).  layout: step_frames' layout of
  device frames.  ValueError for a video whose frame size no stream can take, a video whose frames are of another kind
  (device tensors or arrays) than the first video's, or a runner with neither device tracking nor device
  post-processing.
  crops=True (a runner built with crop_size): yields (video id, frame index, results, crops) instead, crops being that
  stream's device uint8 view [n, out_h, out_w, 3] of the frame's crops (StreamRunner.fetch_crops), n being the number
  of active tracks (the leading entries of results; every detection without a tracker) and crop k the box of
  results[k].  A step's items come after the next step is submitted, and the step submitted three steps
  later rewrites its crops: a view stays valid while the items of the next step are pulled, and becomes invalid when
  the first item of the step after that is pulled.  Copy (or consume) a crop before then.  With the runner's
  crop_format, crops is instead that stream's slice [n, 3, out_h, out_w] of the step's packed batch, with the same
  lifetime.  ValueError for crops other than True or False (the batch's format is the runner's crop_format)."""
  if runner.tracker is None and getattr(runner, 'post', None) is None:
    raise ValueError('track_videos: the runner needs device_tracking=True or device_post_process=True')
  if crops not in (True, False):
    raise ValueError('track_videos: crops must be True or False, got %r (build the runner with crop_format for a '
                     'normalised batch)' % (crops,))
  if crops and getattr(runner, 'crop', None) is None:
    raise ValueError('track_videos: crops=True needs a runner built with crop_size')
  if layout != 'bgr' and not runner.frames_mode:
    raise ValueError('track_videos: layout=%r needs a frames-mode runner' % (layout,))
  B = runner.B
  tables = runner.tracker if runner.tracker is not None else runner.post
  per_stream = getattr(tables, 'per_stream', False)
  capacity = runner.frames_mode and getattr(runner, 'max_frame_bytes', None) is not None
  idle_runner = getattr(runner, 'idle_g', None) is not None
  fmt = getattr(runner, 'frame_format', 'bgr')
  if runner.frames_mode:
    sizes = [tuple(s) for s in runner.frame_sizes]
  else:
    sizes = [(3, runner.H, runner.W)] * B

  kind = []                           # frames mode: [whether the videos bring device frames], set by the first video

  def size_of(frame):
    if runner.frames_mode and is_device_frame(frame):
      return device_frame_source(frame, fmt, layout, runner.u8[0].device)[0]
    shape = tuple(np.shape(frame))
    if not runner.frames_mode:
      return shape[-3:]
    return shape[:2] if fmt == 'bgr' else frame_size_of(fmt, shape)     # None: not a frame of that format

  def filler(size):
    """A frame of this size for a stream that never had a video, of the videos' kind."""
    if not runner.frames_mode:
      return torch.zeros(size)
    if not kind[0]:
      return np.zeros(frame_layout(fmt, *size)[0], np.uint8)
    shape = (3,) + tuple(size) if layout == 'rgb_planar' else frame_layout(fmt, *size)[0]
    return torch.zeros(shape, dtype=torch.uint8, device=runner.u8[0].device)

  source = iter(videos)
  pending = []                        # pulled, not yet placed: _Playing with index 0
  playing = [None] * B
  last = [None] * B                   # the frame each stream was last fed

  def pull():
    for v in source:
      v = _as_video(v)
      it = iter(v.frames)
      first = next(it, None)
      if first is None:               # no frames: nothing to yield
        continue
      if runner.frames_mode:
        dev = is_device_frame(first)
        if not kind:
          kind.append(dev)
        elif kind[0] != dev:
          raise ValueError('track_videos: video %r brings %s; the videos before it bring %s' %
                           (v.id, *(('device frames', 'arrays') if dev else ('arrays', 'device frames'))))
        if dev:
          try:
            size_of(first)
          except ValueError as e:
            raise ValueError('track_videos: video %r: %s' % (v.id, e))
      if size_of(first) is None:
        raise ValueError('track_videos: video %r: a frame of shape %s is not a %s frame [3h/2, w]' %
                         (v.id, np.shape(first), fmt.upper()))
      if capacity:
        try:
          runner.check_frame_size(size_of(first))
        except ValueError as e:
          raise ValueError('track_videos: video %r: %s' % (v.id, e))
      elif size_of(first) not in sizes:
        raise ValueError('track_videos: video %r has frames of size %s; the streams take %s' %
                         (v.id, size_of(first), sorted(set(sizes))))
      return _Playing(v, it, first)
    return None

  def place():
    """Pending videos in order, each to the first free stream of its size (any free stream on a capacity runner);
    then new videos while a stream is free (looking at most B videos ahead).  -> the streams that start a video."""
    started = []

    def put(p):
      for b in range(B):
        if playing[b] is None and (capacity or sizes[b] == size_of(p.frame)):
          playing[b] = p
          sizes[b] = size_of(p.frame)
          started.append(b)
          return True
      return False

    pending[:] = [p for p in pending if not put(p)]
    while None in playing and len(pending) < B:
      p = pull()
      if p is None:
        break
      if not put(p):
        pending.append(p)
    return started

  fed = None                          # (video id, frame index) per stream of the last submitted step
  while True:
    started = place()
    if all(p is None for p in playing):
      break
    frames, now = [], [None] * B
    for b, p in enumerate(playing):
      if p is not None:
        last[b] = p.frame
        now[b] = (p.video.id, p.index)
      elif idle_runner:               # no frame: the stream is idle in this step
        frames.append(None)
        continue
      elif last[b] is None:           # a stream that never had a video: any frame of its size
        last[b] = filler(sizes[b])
      frames.append(last[b])
    pre_dets = {b: playing[b].video.pre_dets for b in started if playing[b].video.pre_dets is not None}
    options = {b: playing[b].video.options or {} for b in started} if per_stream else \
        {b: playing[b].video.options for b in started if playing[b].video.options is not None}
    step_opts = runner._step_options({b: tables.check_options(o, 'video %r: options' % (playing[b].video.id,))
                                      for b, o in options.items()}) if per_stream else None
    public = None
    if runner.public:
      public = []
      for b, p in enumerate(playing):
        pd = p.video.public_dets if p is not None else None
        if per_stream and not step_opts[b]['public_det']:      # a stream without --public_det takes None
          public.append(None)
          continue
        public.append(np.zeros((0, 2), np.float32) if pd is None else pd[p.index])
    kw = dict(public_dets=public, starts=started, pre_dets=pre_dets or None)
    if options:
      kw['options'] = options
    if idle_runner:
      kw['idle'] = [b for b, p in enumerate(playing) if p is None]
    calibs = {b: playing[b].video.calib for b in started if playing[b].video.calib is not None}
    if calibs:
      kw['calibs'] = calibs
    if runner.frames_mode:
      if layout != 'bgr' or kind[0]:
        kw['layout'] = layout
      runner.step_frames(frames, **kw)
    else:
      runner.step_host(torch.stack([torch.as_tensor(f, dtype=torch.float32).reshape(sizes[0]) for f in frames]), **kw)
    if fed is not None:
      res = runner.previous_results()
      cut = runner.previous_crops() if crops else None
      for b, key in enumerate(fed):
        if key is not None:
          yield key + (res[b],) + ((_stream_crops(runner, cut, b),) if crops else ())
    fed = now
    for b, p in enumerate(playing):   # advance; a finished video frees its stream for the next step
      if p is not None:
        nxt = next(p.it, None)
        if nxt is None:
          playing[b] = None
        else:
          p.frame, p.index = nxt, p.index + 1
  if fed is not None:
    res = runner.fetch_results()
    cut = runner.fetch_crops() if crops else None
    for b, key in enumerate(fed):
      if key is not None:
        yield key + (res[b],) + ((_stream_crops(runner, cut, b),) if crops else ())
