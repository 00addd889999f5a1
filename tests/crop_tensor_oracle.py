"""The reference of ct_crop_boxes_tensor's elements: torchvision's Normalize(mean, std)(ToTensor()(crop)).to(dtype) of
each uint8 crop on the CPU (tests/test_crop_tensor_host.py checks it against the documented formula in numpy), and the
packing rule: stream after stream, each stream's crops in result order."""
import numpy as np
import torch

IMAGENET = {'mean': (0.485, 0.456, 0.406), 'std': (0.229, 0.224, 0.225)}


def normalize(crops, dtype, channels, mean, std):
  """uint8 BGR crops [n, h, w, 3] (numpy) -> CPU tensor [n, 3, h, w] of dtype, channels 'rgb' or 'bgr'."""
  from torchvision import transforms as T
  crops = np.asarray(crops, np.uint8)
  if channels == 'rgb':
    crops = crops[..., ::-1]
  to_tensor, norm = T.ToTensor(), T.Normalize(mean, std)
  if len(crops) == 0:
    return torch.zeros((0, 3) + crops.shape[1:3], dtype=dtype)
  return torch.stack([norm(to_tensor(np.ascontiguousarray(c))) for c in crops]).to(dtype)


def pack(u8, counts, streams, dtype, channels, mean, std):
  """The packed batch of uint8 crops u8 [n_streams, K, h, w, 3] with counts [n_streams]: the streams listed in
  `streams`, ascending, each its first counts[b] crops -> (CPU tensor [N, 3, h, w], offsets int32 [n_streams + 1])."""
  counts = np.asarray(counts)
  n_streams = u8.shape[0]
  rows = np.array([int(counts[b]) if b in streams else 0 for b in range(n_streams)])
  offsets = np.concatenate([[0], np.cumsum(rows)]).astype(np.int32)
  parts = [u8[b, :rows[b]] for b in range(n_streams) if rows[b]]
  got = np.concatenate(parts) if parts else np.zeros((0,) + u8.shape[2:], np.uint8)
  return normalize(got, dtype, channels, mean, std), offsets


def bits(t):
  """The element bits of a tensor (NaN payloads and signed zeros compare exactly)."""
  t = t.contiguous()
  return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)
