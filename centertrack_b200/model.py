"""Model factory + checkpoint I/O with the reference's surface (model/model.py:16-101):
`create_model(arch, head, head_conv, opt)`, `load_model(model, path, opt, optimizer=None)`,
`save_model(path, epoch, model, optimizer=None)`, `_network_factory`.

`DLASegB200` registers exactly the parameters/buffers of the reference's `DLASeg(34, ...)`
(dla.py:594-617 + base_model.py:14-65), so reference checkpoints load key-for-key (including the two
dead `base.level{3,4}.project.*` tensors and BatchNorm's `num_batches_tracked`), but holds no PyTorch
compute: `forward` hands the state_dict to a `DLA34Engine` plan of libctb200 launches.
Archs: `dla_34` (the default --arch, opts.py:82) with any `--dla_node` (dcn | conv | gcn, dla.py:588-592), and
`generic` with `--backbone dla34 --neck dlaup` (generic_network.py:29-107 over backbones/dla.py + necks/dlaup.py): the
same graph under the state-dict names `backbone.*` / `neck.{dla_up,ida_up}.*`, so it runs the same engine plan.
`resdcn` / `res` / `dlav0` and the resnet / mobilenet backbones or the msraup neck raise: their `BaseModel.forward`
has no `imgpre2feats` (resdcn.py:192-206), i.e. they cannot take the tracking inputs this path exists for.
"""
import torch
import torch.nn as nn

from .dcn import DCN
from .engine import DLA34Engine

BN_MOMENTUM = 0.1


def _bn(c):
  return nn.BatchNorm2d(c, momentum=BN_MOMENTUM)


class _Holder(nn.Module):
  """Parameter container; never called."""

  def forward(self, *a, **k):
    raise RuntimeError('parameter holder: compute runs in DLA34Engine')


def _block(cin, cout):                         # BasicBlock keys: conv1,bn1,conv2,bn2
  m = _Holder()
  m.conv1 = nn.Conv2d(cin, cout, 3, bias=False)
  m.bn1 = _bn(cout)
  m.conv2 = nn.Conv2d(cout, cout, 3, bias=False)
  m.bn2 = _bn(cout)
  return m


def _root(cin, cout):                          # Root keys: conv, bn
  m = _Holder()
  m.conv = nn.Conv2d(cin, cout, 1, bias=False)
  m.bn = _bn(cout)
  return m


def _tree(levels, cin, cout, level_root=False, root_dim=0):
  """Tree keys (dla.py:175-213): tree1, tree2, [root], [project.0/.1]."""
  m = _Holder()
  if root_dim == 0:
    root_dim = 2 * cout
  if level_root:
    root_dim += cin
  if levels == 1:
    m.tree1 = _block(cin, cout)
    m.tree2 = _block(cout, cout)
    m.root = _root(root_dim, cout)
  else:
    m.tree1 = _tree(levels - 1, cin, cout)
    m.tree2 = _tree(levels - 1, cout, cout, root_dim=root_dim + cout)
  if cin != cout:
    m.project = nn.Sequential(nn.Conv2d(cin, cout, 1, bias=False), _bn(cout))
  return m


def _stem(cin, cout):
  return nn.Sequential(nn.Conv2d(cin, cout, 7, bias=False), _bn(cout), nn.ReLU(inplace=True))


def _conv_level(cin, cout):
  return nn.Sequential(nn.Conv2d(cin, cout, 3, bias=False), _bn(cout), nn.ReLU(inplace=True))


def _deform(cin, cout):                        # DeformConv keys: actf.0, conv (DCN)
  m = _Holder()
  m.actf = nn.Sequential(_bn(cout), nn.ReLU(inplace=True))
  m.conv = DCN(cin, cout, kernel_size=(3, 3), stride=1, padding=1, dilation=1, deformable_groups=1)
  return m


def _conv_node(cin, cout):                     # Conv keys (dla.py:466-475): conv.0 (1x1), conv.1 (BN)
  m = _Holder()
  m.conv = nn.Sequential(nn.Conv2d(cin, cout, 1, bias=False), _bn(cout), nn.ReLU(inplace=True))
  return m


def _global_conv_node(cin, cout, k=7):         # GlobalConv keys (dla.py:477-503): gcl.{0,1}, gcr.{0,1}, act.0
  m = _Holder()
  m.gcl = nn.Sequential(nn.Conv2d(cin, cout, (k, 1), bias=False, padding=(k // 2, 0)),
                        nn.Conv2d(cout, cout, (1, k), bias=False, padding=(0, k // 2)))
  m.gcr = nn.Sequential(nn.Conv2d(cin, cout, (1, k), bias=False, padding=(0, k // 2)),
                        nn.Conv2d(cout, cout, (k, 1), bias=False, padding=(k // 2, 0)))
  m.act = nn.Sequential(_bn(cout), nn.ReLU(inplace=True))
  return m


DLA_NODE = {'dcn': (_deform, _deform), 'gcn': (_conv_node, _global_conv_node), 'conv': (_conv_node, _conv_node)}


def _fill_up_weights(up):
  """Bilinear initialisation of the (learnable) depthwise upsampling kernel (dla.py:454-463)."""
  w = up.weight.data
  k = w.size(2)
  f = (k + 1) // 2
  c = (2 * f - 1 - f % 2) / (2. * f)
  i = torch.arange(k, dtype=torch.float64)
  g = 1 - (i / f - c).abs()
  w[:] = (g[:, None] * g[None, :]).to(w.dtype)


def _ida(o, channels, up_f, node_type=(_deform, _deform)):    # IDAUp keys: proj_i, up_i, node_i
  m = _Holder()
  for i in range(1, len(channels)):
    f = int(up_f[i])
    setattr(m, 'proj_%d' % i, node_type[0](channels[i], o))
    up = nn.ConvTranspose2d(o, o, f * 2, stride=f, padding=f // 2, output_padding=0, groups=o, bias=False)
    _fill_up_weights(up)
    setattr(m, 'up_%d' % i, up)
    setattr(m, 'node_%d' % i, node_type[1](o, o))
  return m


def _dla34_backbone(opt):
  """DLA-34 `base` (dla.py:231-267 == backbones/dla.py:223-265): stems, level0..5."""
  base = _Holder()
  base.base_layer = _stem(3, 16)
  base.level0 = _conv_level(16, 16)
  base.level1 = _conv_level(16, 32)
  base.level2 = _tree(1, 32, 64, level_root=False)
  base.level3 = _tree(2, 64, 128, level_root=True)
  base.level4 = _tree(2, 128, 256, level_root=True)
  base.level5 = _tree(1, 256, 512, level_root=True)
  if opt is None or getattr(opt, 'pre_img', False):
    base.pre_img_layer = _stem(3, 16)
  if opt is None or getattr(opt, 'pre_hm', False):
    base.pre_hm_layer = _stem(1, 16)
  return base


def _dlaup_neck(node_type):
  """(dla_up, ida_up) of dla.py:549-566,606-617 == necks/dlaup.py:139-190.
  DLAUp: ida_0 sees [256,512], ida_1 [128,256,256], ida_2 [64,128,128,128]."""
  ch = [16, 32, 64, 128, 256, 512]
  dla_up = _Holder()
  channels, in_ch = ch[2:], list(ch[2:])
  scales = [1, 2, 4, 8]
  for i in range(3):
    j = -i - 2
    setattr(dla_up, 'ida_%d' % i, _ida(channels[j], in_ch[j:], [s // scales[j] for s in scales[j:]], node_type))
    scales[j + 1:] = [scales[j]] * len(scales[j + 1:])
    in_ch[j + 1:] = [channels[j]] * len(in_ch[j + 1:])
  return dla_up, _ida(64, ch[2:5], [1, 2, 4], node_type)


class _B200Net(nn.Module):
  """What the two archs share: the head modules (base_model.py:23-65 == generic_network.py:47-89), the engine cache
  and `forward`.  Subclasses register the trunk under the reference's names and say how those names map onto the
  engine's (`_engine_state_dict`)."""

  def _common_init(self, heads, opt):
    self.opt = opt
    self.heads = heads
    self.num_stacks = 1
    self.precision = getattr(opt, 'b200_precision', 'bf16') if opt is not None else 'bf16'
    self._engines = {}
    return DLA_NODE[getattr(opt, 'dla_node', 'dcn') if opt is not None else 'dcn']      # dla.py:588-592

  def _add_heads(self, heads, head_convs, opt):
    head_kernel = getattr(opt, 'head_kernel', 3) if opt is not None else 3
    prior_bias = getattr(opt, 'prior_bias', -4.6) if opt is not None else -4.6
    for head in heads:
      classes, hc = heads[head], head_convs[head]
      if len(hc) > 0:
        layers = [nn.Conv2d(64, hc[0], head_kernel, padding=head_kernel // 2, bias=True),
                  nn.ReLU(inplace=True)]
        for k in range(1, len(hc)):
          layers += [nn.Conv2d(hc[k - 1], hc[k], 1, bias=True), nn.ReLU(inplace=True)]
        layers.append(nn.Conv2d(hc[-1], classes, 1, bias=True))
        fc = nn.Sequential(*layers)
        if 'hm' in head:
          fc[-1].bias.data.fill_(prior_bias)
        else:
          for m in fc.modules():
            if isinstance(m, nn.Conv2d):
              nn.init.constant_(m.bias, 0)
      else:
        fc = nn.Conv2d(64, classes, 1, bias=True)
        if 'hm' in head:
          fc.bias.data.fill_(prior_bias)
        else:
          nn.init.constant_(fc.bias, 0)
      setattr(self, head, fc)

  def _engine_state_dict(self):
    """The module's tensors under the names the engine plan uses (DLASeg's: base.*, dla_up.*, ida_up.*, <head>.*)."""
    return self.state_dict()

  # -- engine cache ---------------------------------------------------------------------------
  def _load_from_state_dict(self, *args, **kwargs):
    self._engines = {}
    return super(_B200Net, self)._load_from_state_dict(*args, **kwargs)

  def invalidate(self):
    self._engines = {}

  MAX_ENGINES = 4       # resolutions kept alive (each holds a full activation plan on the GPU); LRU beyond that

  def _weights_version(self):
    """Changes whenever a parameter/buffer is written in place (tensor._version) or replaced (.half(), .to())."""
    return tuple((id(t), t._version, t.dtype) for t in list(self.parameters()) + list(self.buffers()))

  def engine_for(self, B, H, W, device, precision=None):
    precision = precision or self.precision
    ver = self._weights_version()
    if getattr(self, '_engines_version', None) != ver:        # in-place weight edits / dtype moves: repack
      self._engines = {}
      self._engines_version = ver
    key = (B, H, W, str(device), precision)
    eng = self._engines.pop(key, None)
    if eng is None:
      depth_scale = getattr(self.opt, 'depth_scale', 1.0) if self.opt is not None else 1.0
      eng = DLA34Engine(self._engine_state_dict(), self.heads, B, H, W, precision=precision, device=device,
                        depth_scale=depth_scale, dla_node=getattr(self.opt, 'dla_node', 'dcn') if self.opt is not None else 'dcn')
      while len(self._engines) >= self.MAX_ENGINES:           # --keep_res / --fix_short on variable-size inputs
        self._engines.pop(next(iter(self._engines)))
    self._engines[key] = eng                                  # most recently used last
    return eng

  def forward(self, x, pre_img=None, pre_hm=None):
    """-> [ {head: [B,c,H/4,W/4] fp32} ]  (list of num_stacks=1; base_model.py:73-91).  Raw head
    outputs (no sigmoid), like the reference module."""
    if not x.is_cuda:
      raise RuntimeError('centertrack_b200 model runs on an H100 only (no CPU fallback); input is on %s'
                         % x.device)
    B, _, H, W = x.shape
    eng = self.engine_for(B, H, W, x.device)
    if eng.fused_act:
      eng.set_fused_activations(False)
    f = lambda t: None if t is None else t.detach().float().contiguous()
    out = eng.forward(f(x), f(pre_img), f(pre_hm))
    z = {h: out[h].clone() for h in self.heads}
    if self.opt is not None and getattr(self.opt, 'model_output_list', False):
      return [[z[h] for h in sorted(self.heads)]]
    return [z]


class DLASegB200(_B200Net):
  """State-dict-compatible stand-in for DLASeg(34, heads, head_convs, opt) (dla.py:576-640)."""

  def __init__(self, num_layers, heads, head_convs, opt=None):
    super(DLASegB200, self).__init__()
    if num_layers != 34:
      raise NotImplementedError('only DLA-34 (arch dla_34) is on the H100 hot path')
    node_type = self._common_init(heads, opt)
    self.base = _dla34_backbone(opt)
    self.dla_up, self.ida_up = _dlaup_neck(node_type)
    self._add_heads(heads, head_convs, opt)


class _DLAUpNeck(_Holder):                     # necks/dlaup.py:170-190: `neck.dla_up.*`, `neck.ida_up.*`
  pass


class GenericNetworkB200(_B200Net):
  """State-dict-compatible stand-in for GenericNetwork(num_layers, heads, head_convs, opt=opt) with
  `--backbone dla34 --neck dlaup` (generic_network.py:29-107).  backbones/dla.py's DLA and necks/dlaup.py's DLASeg are
  the `base` / `dla_up` + `ida_up` of dla.py under other names (the forward is the same graph: x = base_layer(img)
  + pre_img_layer(pre) + pre_hm_layer(hm), level0..5, DLAUp, clone, IDAUp, take the last), so the tensors are handed
  to the same engine plan with `backbone.` -> `base.`, `neck.dla_up.` -> `dla_up.`, `neck.ida_up.` -> `ida_up.`.
  Note opts.py:295: `head_conv` defaults to 64 (not 256) when the arch name has no 'dla' in it."""

  RENAME = (('backbone.', 'base.'), ('neck.dla_up.', 'dla_up.'), ('neck.ida_up.', 'ida_up.'))

  def __init__(self, num_layers, heads, head_convs, num_stacks=1, opt=None):
    super(GenericNetworkB200, self).__init__()
    backbone = getattr(opt, 'backbone', 'dla34') if opt is not None else 'dla34'
    neck = getattr(opt, 'neck', 'dlaup') if opt is not None else 'dlaup'
    if backbone != 'dla34' or neck != 'dlaup':
      raise NotImplementedError('generic arch: only --backbone dla34 --neck dlaup is on the H100 hot path '
                                '(got %s / %s)' % (backbone, neck))
    print('Using generic model with backbone {} and neck {}'.format(backbone, neck))
    node_type = self._common_init(heads, opt)
    self.backbone = _dla34_backbone(opt)
    self.backbone.channels = [16, 32, 64, 128, 256, 512]
    self.neck = _DLAUpNeck()
    self.neck.dla_up, self.neck.ida_up = _dlaup_neck(node_type)
    self.neck.out_channel = 64
    self._add_heads(heads, head_convs, opt)

  def _engine_state_dict(self):
    out = {}
    for k, v in self.state_dict().items():
      for a, b in self.RENAME:
        if k.startswith(a):
          k = b + k[len(a):]
          break
      out[k] = v
    return out


def _unsupported(name):
  def make(*a, **k):
    raise NotImplementedError('arch %r is outside the H100 hot path (dla_34, or generic with --backbone dla34 '
                              '--neck dlaup): it has no imgpre2feats, i.e. no tracking inputs' % name)
  return make


_network_factory = {
    'dla': DLASegB200,
    'resdcn': _unsupported('resdcn'), 'res': _unsupported('res'),
    'dlav0': _unsupported('dlav0'), 'generic': GenericNetworkB200,
}


def create_model(arch, head, head_conv, opt=None):
  """model.py:24-29."""
  num_layers = int(arch[arch.find('_') + 1:]) if '_' in arch else 0
  arch = arch[:arch.find('_')] if '_' in arch else arch
  return _network_factory[arch](num_layers, heads=head, head_convs=head_conv, opt=opt)


def load_model(model, model_path, opt, optimizer=None):
  """model.py:31-90: strips `module.`, tolerates shape mismatches (skip / reuse_hm), strict=False."""
  start_epoch = 0
  checkpoint = torch.load(model_path, map_location=lambda storage, loc: storage)
  print('loaded {}, epoch {}'.format(model_path, checkpoint['epoch']))
  state_dict = {}
  for k, v in checkpoint['state_dict'].items():
    state_dict[k[7:] if k.startswith('module') and not k.startswith('module_list') else k] = v
  msd = model.state_dict()
  for k in list(state_dict):
    if k in msd:
      mismatch = state_dict[k].shape != msd[k].shape
      reset = getattr(opt, 'reset_hm', False) and k.startswith('hm') and state_dict[k].shape[0] in [80, 1]
      if mismatch or reset:
        if getattr(opt, 'reuse_hm', False):
          print('Reusing parameter {}, required shape{}, loaded shape{}.'.format(
              k, msd[k].shape, state_dict[k].shape))
          n = min(state_dict[k].shape[0], msd[k].shape[0])
          t = msd[k].clone()
          t[:n] = state_dict[k][:n]
          state_dict[k] = t
        else:
          print('Skip loading parameter {}, required shape{}, loaded shape{}.'.format(
              k, msd[k].shape, state_dict[k].shape))
          state_dict[k] = msd[k]
    else:
      print('Drop parameter {}.'.format(k))
  for k in msd:
    if k not in state_dict:
      print('No param {}.'.format(k))
      state_dict[k] = msd[k]
  model.load_state_dict(state_dict, strict=False)
  if hasattr(model, 'invalidate'):
    model.invalidate()
  if optimizer is not None and getattr(opt, 'resume', False):
    if 'optimizer' in checkpoint:
      start_epoch = checkpoint['epoch']
      start_lr = opt.lr
      for step in opt.lr_step:
        if start_epoch >= step:
          start_lr *= 0.1
      for pg in optimizer.param_groups:
        pg['lr'] = start_lr
      print('Resumed optimizer with start lr', start_lr)
    else:
      print('No optimizer parameters in checkpoint.')
  if optimizer is not None:
    return model, optimizer, start_epoch
  return model


def save_model(path, epoch, model, optimizer=None):
  """model.py:92-101."""
  sd = model.module.state_dict() if isinstance(model, torch.nn.DataParallel) else model.state_dict()
  data = {'epoch': epoch, 'state_dict': sd}
  if optimizer is not None:
    data['optimizer'] = optimizer.state_dict()
  torch.save(data, path)
