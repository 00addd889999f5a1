"""Adversarial DCNv2 offset / mask maps (test infrastructure; numpy only, importable without a GPU).

catalogue(B, H, W, margin) writes one entry per (image, pixel, tap) of an om map [B, H, W, 27] (offsets 2k = dy,
2k + 1 = dx, then the nine masks, already sigmoid'd) from the categories below, spread by a fixed stride so that each
category meets image corners, edges, the interior, ragged 8 x 16 patches and every tap:

  normal        N(0, 3) offsets (the filler, two slots of the cycle)
  int_interior  exact integer positions inside the image
  int_last_row  exact integers on the last row: the y + 1 neighbour lies outside, its weight is exactly 0
  int_last_col  the same on the last column
  y_low, x_low  py (px) in {-1, -1 + 2^-20, -1 + 2^-8, -0.5, -2^-20}
  y_high,x_high py (px) in {H-1, H-1 + 2^-20, H - 0.5, H - 2^-20, H, H + 2^-20}
  frac          half- and quarter-pixel positions
  tie           a corner weight hy hx m that is an exact bf16 rounding tie (ly = 0, m in {1, 0.5}, hx = 0.5 +
                odd 2^-9 or 0.25 + odd 2^-10; half of them round down to even, half up), in y or in x
  win_y, win_x  floor(py) (floor(px)) on the first row of the pixel's CT_A_DCN_WIN window, one row above it, on the
                last row that holds the 2-row footprint, and one row below that
  far           py or px at +-(H + W + 5), +-1e4, +-3e38
  neg_zero      -0.0 offsets

Offsets are targets minus the tap's base position, rounded to fp32: the kernels then add them to the base in fp32, so
a fine fraction far from the origin lands a few ulps from its target, still on the adversarial side of the edge.
Masks are 0, 1, 2^-8 or 0.5 on half of the entries and uniform on the others (the tie entries keep theirs)."""
import numpy as np

CATEGORIES = ['normal', 'int_interior', 'int_last_row', 'int_last_col', 'y_low', 'x_low', 'y_high', 'x_high', 'frac',
              'tie', 'win_y', 'win_x', 'far', 'neg_zero']
_SLOTS = CATEGORIES + ['normal']          # 15 slots, visited with stride 7 (coprime)
TC_BM_Y, TC_BM_X = 8, 16                  # the window sampler's pixel patch
# the maps of tests/test_gpu_dcn_sampler.py (B, H, W): B of 1 - 3, so 128-row tiles straddle images
PROBE_SHAPES = [(1, 1, 1), (2, 1, 20), (3, 20, 1), (2, 7, 5), (1, 8, 16), (3, 9, 17), (2, 33, 61), (1, 64, 96)]


def window_origin(y, x, margin):
  """(first row, first column, rows, columns) of the CT_A_DCN_WIN window of the patch holding pixel (y, x)."""
  return (y // TC_BM_Y) * TC_BM_Y - 1 - margin, (x // TC_BM_X) * TC_BM_X - 1 - margin, \
      TC_BM_Y + 2 * margin + 3, TC_BM_X + 2 * margin + 3


def categories(B, H, W):
  """[B, H, W, 9] index into CATEGORIES of each entry."""
  e = np.arange(H * W * 9).reshape(1, H, W, 9) + np.zeros((B, 1, 1, 1), np.int64)
  b = np.arange(B).reshape(B, 1, 1, 1)
  slot = (e * 7 + b * 4) % len(_SLOTS)
  return np.array([CATEGORIES.index(s) for s in _SLOTS])[slot]


def regions(B, H, W):
  """[B, H, W, 9] labels: 0 interior, 1 edge, 2 corner; and a bool map of the pixels in ragged 8 x 16 patches."""
  y = np.arange(H).reshape(H, 1)
  x = np.arange(W).reshape(1, W)
  n = ((y == 0) | (y == H - 1)).astype(int) + ((x == 0) | (x == W - 1)).astype(int)
  reg = np.minimum(n, 2)
  ragged = ((H % 8 != 0) & (y >= H // 8 * 8)) | ((W % 16 != 0) & (x >= W // 16 * 16))
  shape = (B, H, W, 9)
  return np.broadcast_to(reg[None, :, :, None], shape), np.broadcast_to(ragged[None, :, :, None], shape)


def catalogue(B, H, W, margin=2, seed=0):
  """-> (om fp32 [B, H, W, 27], category index [B, H, W, 9])."""
  rng = np.random.default_rng(seed)
  cat = categories(B, H, W)
  shape = (B, H, W, 9)
  tap = np.broadcast_to(np.arange(9), shape)
  yy = np.broadcast_to(np.arange(H).reshape(1, H, 1, 1), shape)
  xx = np.broadcast_to(np.arange(W).reshape(1, 1, W, 1), shape)
  base_y, base_x = yy - 1 + tap // 3, xx - 1 + tap % 3
  n = B * H * W * 9

  def inside(size):           # a position with a quarter fraction whose footprint is (partly) in [0, size)
    return rng.integers(-1, size, n) + rng.choice([0.25, 0.5, 0.75], n)

  def ints(size):
    return rng.integers(0, max(size - 1, 1), n).astype(np.float64)

  py = (base_y + rng.normal(0, 3, shape)).reshape(-1)        # 'normal' everywhere, overwritten per category
  px = (base_x + rng.normal(0, 3, shape)).reshape(-1)
  m = rng.uniform(0, 1, n)
  fixed = rng.integers(0, 8, n)
  m = np.where(fixed == 0, 0.0, np.where(fixed == 1, 1.0, np.where(fixed == 2, 2.0 ** -8, np.where(fixed == 3, 0.5, m))))
  c = cat.reshape(-1)
  by, bx = base_y.reshape(-1).astype(np.float64), base_x.reshape(-1).astype(np.float64)
  pick = lambda vals: np.asarray(vals, np.float64)[rng.integers(0, len(vals), n)]

  def put(name, y, x):
    s = c == CATEGORIES.index(name)
    py[s], px[s] = y[s], x[s]
    return s

  put('int_interior', ints(H), ints(W))
  put('int_last_row', np.full(n, H - 1.0), ints(W))
  put('int_last_col', ints(H), np.full(n, W - 1.0))
  low, high = [-1.0, -1 + 2.0 ** -20, -1 + 2.0 ** -8, -0.5, -2.0 ** -20], [0.0, 2.0 ** -20, 0.5, 1 - 2.0 ** -20, 1.0, 1 + 2.0 ** -20]
  put('y_low', pick(low), inside(W))
  put('x_low', inside(H), pick(low))
  put('y_high', H - 1 + pick(high), inside(W))
  put('x_high', inside(H), W - 1 + pick(high))
  put('frac', rng.integers(-1, H, n) + pick([0.0, 0.25, 0.5, 0.75]), rng.integers(-1, W, n) + pick([0.0, 0.25, 0.5, 0.75]))
  # ties: ly = 0 on an integer row, hx a bf16 midpoint (or the same in x)
  odd = 2 * rng.integers(0, 32, n) + 1
  hx = np.where(rng.integers(0, 2, n) == 0, 0.5 + odd * 2.0 ** -9, 0.25 + odd * 2.0 ** -10)
  in_y, in_x = ints(H), ints(W)
  along_x = rng.integers(0, 2, n) == 0
  s = put('tie', np.where(along_x, in_y, rng.integers(-1, H, n) + (1 - hx)),
          np.where(along_x, rng.integers(-1, W, n) + (1 - hx), in_x))
  m[s] = np.where(rng.integers(0, 2, n) == 0, 1.0, 0.5)[s]
  # window-edge footprints
  wy0, wx0, ph, pw = window_origin(yy.reshape(-1), xx.reshape(-1), margin)
  rows = np.stack([wy0, wy0 - 1, wy0 + ph - 2, wy0 + ph - 1], 1)[np.arange(n), rng.integers(0, 4, n)]
  cols = np.stack([wx0, wx0 - 1, wx0 + pw - 2, wx0 + pw - 1], 1)[np.arange(n), rng.integers(0, 4, n)]
  fr = pick([0.0, 0.25, 0.5, 0.75, float(np.float32(1 / 3))])
  near_y, near_x = by + rng.uniform(-1.5, 1.5, n), bx + rng.uniform(-1.5, 1.5, n)
  put('win_y', rows + fr, near_x)
  put('win_x', near_y, cols + fr)
  far = np.asarray([H + W + 5.0, -(H + W + 5.0), 1e4, -1e4, 3e38, -3e38])[rng.integers(0, 6, n)]
  along_x = rng.integers(0, 2, n) == 0
  put('far', np.where(along_x, by, far), np.where(along_x, far, bx))
  dy = (py - by).astype(np.float32)
  dx = (px - bx).astype(np.float32)
  s = c == CATEGORIES.index('neg_zero')
  dy[s], dx[s] = -0.0, -0.0
  om = np.zeros((B, H, W, 27), np.float32)
  off = np.stack([dy.reshape(shape), dx.reshape(shape)], -1).reshape(B, H, W, 18)
  om[..., :18] = off
  om[..., 18:] = m.astype(np.float32).reshape(shape)
  return om, cat


def positions(om):
  """The sampling positions (py, px) [B, H, W, 9] fp32, as the kernels compute them: fp32 base + fp32 offset."""
  B, H, W, _ = om.shape
  tap = np.arange(9)
  by = (np.arange(H).reshape(1, H, 1, 1) - 1 + tap // 3).astype(np.float32)
  bx = (np.arange(W).reshape(1, 1, W, 1) - 1 + tap % 3).astype(np.float32)
  return by + om[..., 0:18:2], bx + om[..., 1:18:2]


def window_split(om, margin):
  """Per entry: 0 sample outside the image (value 0), 1 footprint inside the patch's window, 2 global fall-back."""
  B, H, W, _ = om.shape
  py, px = positions(om)
  valid = (py > -1) & (py < H) & (px > -1) & (px < W)
  with np.errstate(invalid='ignore', over='ignore'):
    y0 = np.floor(np.where(valid, py, 0)).astype(np.int64)
    x0 = np.floor(np.where(valid, px, 0)).astype(np.int64)
  yy = np.arange(H).reshape(1, H, 1, 1)
  xx = np.arange(W).reshape(1, 1, W, 1)
  wy0, wx0, ph, pw = window_origin(yy, xx, margin)
  win = (y0 >= wy0) & (y0 + 1 <= wy0 + ph - 1) & (x0 >= wx0) & (x0 + 1 <= wx0 + pw - 1)
  return np.where(valid, np.where(win, 1, 2), 0)
