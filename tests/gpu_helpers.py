"""GPU-side helpers shared by the -m gpu parity tests and tools/gpu_check.py: drive ct_conv_forward
through the C ABI on raw device buffers."""
import ctypes as C

import torch

from centertrack_b200 import _lib as L

dev = torch.device('cuda')


def conv_desc(engine, dtype, x_nchw, w, bias, stride, relu=True, residual=None, a_mode=L.CT_A_CONV, om=None,
              out_mode=L.CT_OUT_NHWC, n_tile=0, head_act=0, sig_from=1 << 30, ld_pad=0, ch_off=0, sum3=0):
  """-> (descriptor, output buffer, the device buffers the descriptor points to) of the launch run_conv makes."""
  lib = L.lib()
  B, Cin, H, W = x_nchw.shape
  O, _, k, _ = w.shape
  act = torch.bfloat16 if dtype == L.CT_BF16 else torch.float32
  ld_in = Cin + ld_pad
  xb = torch.zeros((B, H, W, ld_in), dtype=act, device=dev)
  xb[..., ch_off:ch_off + Cin] = x_nchw.permute(0, 2, 3, 1).to(act)
  pad = k // 2
  OH, OW = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
  if k % 2 == 0:                      # even kernel: padding on the top / left only (taps -k/2 .. k/2-1), 'same' output
    OH, OW = H, W
  if engine in (L.CT_ENGINE_TCGEN05, L.CT_ENGINE_TCGEN05_HALO, L.CT_ENGINE_TCGEN05_X3) and n_tile == 0:
    cap = 256 if engine == L.CT_ENGINE_TCGEN05 or (engine == L.CT_ENGINE_TCGEN05_X3 and a_mode != L.CT_A_DCN) else 128
    n_tile = min(cap, (O + 15) // 16 * 16)
  w32 = w.float().contiguous()
  pc, pkh, pkw = Cin, k, k
  if a_mode == L.CT_A_DCN_WIN:        # 64-channel-chunk-major K order (include/ctb200.h)
    nch = Cin // 64
    w32 = w32.reshape(O, nch, 64, 3, 3).permute(0, 2, 1, 3, 4).reshape(O, 64, nch * 3, 3).contiguous()
    pc, pkh, pkw = 64, nch * 3, 3
  nbytes = lib.ct_packed_weight_bytes(engine, O, pc, pkh, pkw, n_tile)
  wp = torch.empty(nbytes, dtype=torch.uint8)
  L.check(lib.ct_pack_weights(engine, C.c_void_p(w32.data_ptr()), O, pc, pkh, pkw, n_tile, C.c_void_p(wp.data_ptr())))
  wp = wp.to(dev)
  sh = bias.float().contiguous().to(dev)
  d = L.ConvDesc()
  d.engine, d.dtype, d.a_mode = engine, dtype, a_mode
  d.B, d.H, d.W, d.C_in, d.ld_in, d.C_out = B, H, W, Cin, ld_in, O
  d.KH = d.KW = k
  d.stride, d.pad, d.OH, d.OW = stride, pad, OH, OW
  d.out_mode, d.relu, d.head_act, d.sig_from, d.depth_scale, d.n_tile = out_mode, int(relu), head_act, sig_from, 1.0, n_tile
  d.epilogue_sum3 = sum3
  d.x = xb.data_ptr() + ch_off * xb.element_size()
  d.w, d.shift = wp.data_ptr(), sh.data_ptr()
  if residual is not None:
    rb = residual.permute(0, 2, 3, 1).contiguous().to(act).to(dev)
    d.residual, d.ld_res = rb.data_ptr(), O
  if om is not None:
    d.om, d.ld_om = om.data_ptr(), om.shape[-1]
  if out_mode == L.CT_OUT_NCHW_F32:
    out = torch.zeros((B, O, OH, OW), dtype=torch.float32, device=dev)
    d.out, d.ld_out = out.data_ptr(), 0
  elif out_mode == L.CT_OUT_NHWC_F32:
    out = torch.zeros((B, OH, OW, 32), dtype=torch.float32, device=dev)
    d.out, d.ld_out = out.data_ptr(), 32
  elif out_mode == L.CT_OUT_NHWC_S2D:
    oc = 16 if sum3 else O
    out = torch.zeros((B, OH // 2, OW // 2, 4 * oc), dtype=act, device=dev)
    d.out, d.ld_out = out.data_ptr(), oc
  else:
    oc = 16 if sum3 else O
    out = torch.zeros((B, OH, OW, oc), dtype=act, device=dev)
    d.out, d.ld_out = out.data_ptr(), oc
  return d, out, (xb, wp, sh, rb if residual is not None else None)


def packed_weights(engine, w, n_tile):
  """ct_pack_weights of w [O, I, kh, kw] (fp32, then bf16 RNE on the tensor-core engines) -> device blob."""
  lib = L.lib()
  w32 = w.detach().float().cpu().contiguous()
  O, I, kh, kw = w32.shape
  wp = torch.empty(lib.ct_packed_weight_bytes(engine, O, I, kh, kw, n_tile), dtype=torch.uint8)
  L.check(lib.ct_pack_weights(engine, C.c_void_p(w32.data_ptr()), O, I, kh, kw, n_tile, C.c_void_p(wp.data_ptr())))
  return wp.to(dev)


def heads_desc(x_nchw, w1, b1, heads, n2, ld_pad=0, ch_off=0, depth_scale=1.0):
  """The fused head launch as engine._fused_heads builds it: heads.0 = 3x3 64 -> n_heads x mid (+ b1, ReLU) on the
  halo engine at n_tile NH = 128 (mid 256) or 64 (mid 64), then per head a 1x1 mid -> C_out (+ bias, activation) at
  the common 1x1 n_tile n2, its weights zero-padded to n2 by the packer.  heads: [(w2 [C_out, mid, 1, 1], b2, act)].

  Every head's fp32 NCHW planes lie in one NaN-filled buffer, each followed by a guard band of n2 planes plus one
  tile row (16 image rows): any store from a ragged tile's out-of-image rows or columns C_out .. n2 - 1 lands in one.
  -> (descriptor, [head output views], buffer, [guard band slices of it], device buffers the descriptor points to)."""
  B, Cin, H, W = x_nchw.shape
  nh = 128 if w1.shape[0] // len(heads) == 256 else 64
  xb = torch.zeros((B, H, W, Cin + ld_pad), dtype=torch.bfloat16, device=dev)
  xb[..., ch_off:ch_off + Cin] = x_nchw.permute(0, 2, 3, 1).to(dev, torch.bfloat16)
  w1p = packed_weights(L.CT_ENGINE_TCGEN05_HALO, w1, nh)
  sh = b1.float().contiguous().to(dev)
  guard = (n2 * H * W + 16 * W + 3) // 4 * 4
  sizes = [B * w2.shape[0] * H * W for w2, _, _ in heads]
  offs, pos = [], guard
  for s in sizes:                                       # 16-byte aligned planes
    offs.append(pos)
    pos += (s + 3) // 4 * 4 + guard
  buf = torch.full((pos,), float('nan'), dtype=torch.float32, device=dev)
  table = (L.Head * len(heads))()
  keep, outs = [xb, w1p, sh, buf, table], []
  for t, (w2, b2, act), off, s in zip(table, heads, offs, sizes):
    wp, bb = packed_weights(L.CT_ENGINE_TCGEN05_HALO, w2, n2), b2.float().contiguous().to(dev)
    keep += [wp, bb]
    outs.append(buf[off:off + s].view(B, w2.shape[0], H, W))
    t.w, t.bias, t.out = wp.data_ptr(), bb.data_ptr(), outs[-1].data_ptr()
    t.C_out, t.n_tile, t.head_act = w2.shape[0], n2, act
  guards = [slice(0, offs[0])] + [slice(off + s, nxt) for off, s, nxt in zip(offs, sizes, offs[1:] + [pos])]
  d = L.ConvDesc()
  d.engine, d.dtype, d.a_mode = L.CT_ENGINE_TCGEN05_HALO, L.CT_BF16, L.CT_A_CONV
  d.B, d.H, d.W, d.C_in, d.ld_in, d.C_out = B, H, W, Cin, Cin + ld_pad, w1.shape[0]
  d.KH = d.KW = 3
  d.stride, d.pad, d.OH, d.OW = 1, 1, H, W
  d.out_mode, d.relu, d.sig_from, d.depth_scale, d.n_tile = L.CT_OUT_NCHW_F32, 1, 1 << 30, depth_scale, nh
  d.x = xb.data_ptr() + ch_off * xb.element_size()
  d.w, d.shift = w1p.data_ptr(), sh.data_ptr()
  d.n_heads, d.heads = len(heads), C.cast(table, C.POINTER(L.Head))
  return d, outs, buf, guards, keep


def run_conv(*args, **kwargs):
  d, out, _buffers = conv_desc(*args, **kwargs)
  L.check(L.lib().ct_conv_forward(C.byref(d), L.stream_ptr()), 'conv')
  torch.cuda.synchronize()
  if d.out_mode == L.CT_OUT_NCHW_F32:
    return out
  if d.out_mode == L.CT_OUT_NHWC_S2D:   # undo: [B, OH/2, OW/2, (sy, sx, c)] -> [B, c, OH, OW]
    B, h, w, c4 = out.shape
    return out.reshape(B, h, w, 2, 2, c4 // 4).permute(0, 5, 1, 3, 2, 4).reshape(B, c4 // 4, 2 * h, 2 * w).float()
  return out.permute(0, 3, 1, 2).float()


def conv_cases():
  # (name, B, Cin, Cout, H, W, k, stride, residual, ld_pad, ch_off)
  return [
      ('3x3 s1 64->64', 2, 64, 64, 24, 40, 3, 1, True, 0, 0),
      ('3x3 s2 32->64', 1, 32, 64, 32, 48, 3, 2, False, 0, 0),
      ('3x3 s1 16->16 (4 taps/slice)', 1, 16, 16, 40, 56, 3, 1, False, 0, 0),
      ('3x3 s2 16->32', 1, 16, 32, 40, 56, 3, 2, False, 0, 0),
      ('1x1 448->128 slice of concat', 1, 448, 128, 16, 24, 1, 1, False, 64, 32),
      ('3x3 s1 256->512 (2 n-tiles)', 1, 256, 512, 8, 12, 3, 1, True, 0, 0),
      ('3x3 s1 64->1024 (heads.0)', 1, 64, 1024, 16, 24, 3, 1, False, 0, 0),
      ('3x3 s2 32->64 (2-D pixel patches)', 2, 32, 64, 32, 64, 3, 2, False, 0, 0),
      ('3x3 s1 64->64 +res (2-D pixel patches)', 2, 64, 64, 16, 32, 3, 1, True, 16, 0),
  ]


