"""Drop-in for the reference's `model/networks/DCNv2/dcn_v2.py::DCN` (the un-vendored
CharlesShang/DCNv2 submodule; call sites dla.py:19,513, necks/dlaup.py:17,99, resdcn.py:20,242,
necks/msraup.py:20,105).

Same constructor signature, same parameter names (`weight`, `bias`, `conv_offset_mask.weight`,
`conv_offset_mask.bias` -> state-dict keys `...{proj,node}_i.conv.*`), same forward contract
`[B,C_in,H,W] -> [B,C_out,H,W]`, same initialisation as upstream (weight ~ U(+-1/sqrt(9*C_in)),
bias = 0, offset/mask conv zero).  forward runs two libctb200 launches (offset/mask 3x3 conv, then the
gather-into-tensor-core modulated deformable conv); there is no CPU path.
"""
import ctypes as C
import math

import torch
import torch.nn as nn

from . import _lib as L


def _pair(v):
  return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


class DCN(nn.Module):

  def __init__(self, in_channels, out_channels, kernel_size=(3, 3), stride=1, padding=1, dilation=1,
               deformable_groups=1):
    super(DCN, self).__init__()
    kh, kw = _pair(kernel_size)
    if (kh, kw) != (3, 3) or _pair(stride) != (1, 1) or _pair(padding) != (1, 1) or \
        _pair(dilation) != (1, 1) or deformable_groups != 1:
      raise NotImplementedError(
          'centertrack_b200.DCN implements the configuration every CenterTrack call site uses: '
          '3x3, stride 1, padding 1, dilation 1, deformable_groups 1')
    self.in_channels, self.out_channels = in_channels, out_channels
    self.kernel_size, self.stride, self.padding, self.dilation = (kh, kw), 1, 1, 1
    self.deformable_groups = deformable_groups
    self.weight = nn.Parameter(torch.empty(out_channels, in_channels, kh, kw))
    self.bias = nn.Parameter(torch.zeros(out_channels))
    self.conv_offset_mask = nn.Conv2d(in_channels, deformable_groups * 3 * kh * kw, kernel_size=(kh, kw),
                                      stride=1, padding=1, bias=True)
    self.precision = 'bf16'     # 'bf16' (wgmma) or 'fp32' (SIMT, reference accuracy)
    self._packed = None
    self.reset_parameters()

  def reset_parameters(self):
    stdv = 1. / math.sqrt(self.in_channels * self.kernel_size[0] * self.kernel_size[1])
    with torch.no_grad():
      self.weight.uniform_(-stdv, stdv)
      self.bias.zero_()
      self.conv_offset_mask.weight.zero_()
      self.conv_offset_mask.bias.zero_()
    self._packed = None

  def _load_from_state_dict(self, *args, **kwargs):
    self._packed = None
    return super(DCN, self)._load_from_state_dict(*args, **kwargs)

  def _pack(self, device, P):
    sms = torch.cuda.get_device_properties(device).multi_processor_count
    key = (self.precision, str(device), P >= sms * 128)
    if self._packed is not None and self._packed[0] == key:
      return self._packed[1]
    lib = L.lib()
    eng = L.CT_ENGINE_TCGEN05 if self.precision == 'bf16' else L.CT_ENGINE_SIMT

    def pack(w, n_tile):
      w32 = w.detach().to('cpu', torch.float32).contiguous()
      O, I, kh, kw = w32.shape
      n = lib.ct_packed_weight_bytes(eng, O, I, kh, kw, n_tile)
      dst = torch.empty(n, dtype=torch.uint8)
      L.check(lib.ct_pack_weights(eng, C.c_void_p(w32.data_ptr()), O, I, kh, kw, n_tile,
                                  C.c_void_p(dst.data_ptr())), 'ct_pack_weights')
      return dst.to(device)
    nt_main = min(256, (self.out_channels + 15) // 16 * 16)
    if eng == L.CT_ENGINE_TCGEN05 and nt_main > 64 and P < sms * 128:
      nt_main = 64
    packed = dict(
        n_om=32, n_main=nt_main,
        w_om=pack(self.conv_offset_mask.weight, 32), w_main=pack(self.weight, nt_main),
        b_om=self.conv_offset_mask.bias.detach().float().to(device).contiguous(),
        b_main=self.bias.detach().float().to(device).contiguous())
    self._packed = (key, packed)
    return packed

  def forward(self, x):
    if not x.is_cuda:
      raise RuntimeError('centertrack_b200.DCN runs on an H100 only (no CPU fallback); got a %s tensor'
                         % x.device)
    lib = L.lib()
    B, Cin, H, W = x.shape
    assert Cin == self.in_channels
    bf16 = self.precision == 'bf16'
    act = torch.bfloat16 if bf16 else torch.float32
    pk = self._pack(x.device, B * H * W)
    xn = x.detach().permute(0, 2, 3, 1).contiguous().to(act)            # NHWC
    om = torch.empty((B, H, W, 32), dtype=torch.float32, device=x.device)
    out = torch.empty((B, H, W, self.out_channels), dtype=act, device=x.device)
    d = L.ConvDesc()
    d.engine = L.CT_ENGINE_TCGEN05 if bf16 else L.CT_ENGINE_SIMT
    d.dtype = L.CT_BF16 if bf16 else L.CT_F32
    d.B, d.H, d.W, d.C_in, d.ld_in = B, H, W, Cin, Cin
    d.KH = d.KW = 3
    d.stride, d.pad, d.OH, d.OW = 1, 1, H, W
    d.x = xn.data_ptr()
    st = L.stream_ptr()
    # offset / mask conv -> fp32 NHWC [.,32] (ch 0..17 offsets, 18..26 sigmoid(mask))
    d.a_mode, d.C_out, d.out_mode, d.ld_out, d.sig_from = L.CT_A_CONV, 27, L.CT_OUT_NHWC_F32, 32, 18
    d.n_tile, d.w, d.shift, d.out = pk['n_om'], pk['w_om'].data_ptr(), pk['b_om'].data_ptr(), om.data_ptr()
    L.check(lib.ct_conv_forward(C.byref(d), st), 'DCN offset conv')
    # modulated deformable conv
    d.a_mode, d.C_out, d.out_mode, d.ld_out, d.sig_from = L.CT_A_DCN, self.out_channels, L.CT_OUT_NHWC, \
        self.out_channels, 1 << 30
    d.n_tile, d.w, d.shift, d.out = pk['n_main'], pk['w_main'].data_ptr(), pk['b_main'].data_ptr(), \
        out.data_ptr()
    d.om, d.ld_om = om.data_ptr(), 32
    L.check(lib.ct_conv_forward(C.byref(d), st), 'DCN main')
    return out.permute(0, 3, 1, 2).to(x.dtype)
