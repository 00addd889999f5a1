"""track_videos: many videos of different lengths through one StreamRunner, each video on one stream from its first
frame to its last -- the batched form of the reference's evaluation loop (src/test.py prefetch_test: reset_tracking and
init_track(pre_dets) at each video's first frame, then Detector.run on every frame).

A video goes to the first free stream (in frames mode, a free stream whose frame_sizes entry is the video's frame
size) and starts there with StreamRunner's `starts=` / `pre_dets=`; when it ends, the stream takes the next video in the
same step.  A stream with no video re-feeds its last frame and its results are dropped.  The runner's one-step pipeline
is kept: the upload of step t+1 overlaps step t, and step t's tracks are yielded after step t+1 is submitted.
"""
import numpy as np
import torch


class Video(object):
  """One video: `id`, `frames` (an iterable: uint8 [h, w, 3] BGR arrays in frames mode, pre-processed fp32 [3, H, W]
  images otherwise), optional `pre_dets` (result dicts seeding the tracker at the first frame, as the reference's
  --load_results does) and `public_dets` (per frame, the [P, 2] centres of its public detections, for --public_det)."""

  def __init__(self, id, frames, pre_dets=None, public_dets=None):
    self.id, self.frames, self.pre_dets, self.public_dets = id, frames, pre_dets, public_dets


class _Playing(object):
  """A video on a stream: its frame iterator, the frame the next step feeds, and that frame's index."""

  def __init__(self, video, it, first):
    self.video, self.it, self.frame, self.index = video, it, first, 0


def _as_video(v):
  return v if isinstance(v, Video) else Video(**v)


def track_videos(runner, videos):
  """runner: a StreamRunner with device tracking; videos: an iterable of Video (or dicts of its fields).  Yields
  (video id, frame index, results) for every frame of every video exactly once, as its tracks come back; results is the
  list of dicts fetch_results() gives for that stream (in source pixels in frames mode).  ValueError for a video whose
  frame size no stream has, or a runner without device tracking."""
  if runner.tracker is None:
    raise ValueError('track_videos: the runner needs device_tracking=True')
  B = runner.B
  if runner.frames_mode:
    sizes = [tuple(s) for s in runner.frame_sizes]
  else:
    sizes = [(3, runner.H, runner.W)] * B

  def size_of(frame):
    shape = tuple(np.shape(frame))
    return shape[:2] if runner.frames_mode else shape[-3:]

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
      if size_of(first) not in sizes:
        raise ValueError('track_videos: video %r has frames of size %s; the streams take %s' %
                         (v.id, size_of(first), sorted(set(sizes))))
      return _Playing(v, it, first)
    return None

  def place():
    """Pending videos in order, each to the first free stream of its size; then new videos while a stream is free
    (looking at most B videos ahead).  -> the streams that start a video."""
    started = []

    def put(p):
      for b in range(B):
        if playing[b] is None and sizes[b] == size_of(p.frame):
          playing[b] = p
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
      elif last[b] is None:           # a stream that never had a video: any frame of its size
        last[b] = np.zeros(sizes[b] + (3,), np.uint8) if runner.frames_mode else torch.zeros(sizes[b])
      frames.append(last[b])
    pre_dets = {b: playing[b].video.pre_dets for b in started if playing[b].video.pre_dets is not None}
    public = None
    if runner.public:
      public = []
      for p in playing:
        pd = p.video.public_dets if p is not None else None
        public.append(np.zeros((0, 2), np.float32) if pd is None else pd[p.index])
    kw = dict(public_dets=public, starts=started, pre_dets=pre_dets or None)
    if runner.frames_mode:
      runner.step_frames(frames, **kw)
    else:
      runner.step_host(torch.stack([torch.as_tensor(f, dtype=torch.float32).reshape(sizes[0]) for f in frames]), **kw)
    if fed is not None:
      res = runner.previous_results()
      for b, key in enumerate(fed):
        if key is not None:
          yield key + (res[b],)
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
    for b, key in enumerate(fed):
      if key is not None:
        yield key + (res[b],)
