"""-m gpu: `--arch generic --backbone dla34 --neck dlaup` (generic_network.py:29-107) on the H100 against goldens made
by the reference's own GenericNetwork (tests/golden/net_generic_coco_tracking_64x96.npz, oracle/gen_golden.py::
gen_generic).  With --head_conv 256 the plan that runs is launch for launch the dla_34 one (CPU test
test_generic_arch_is_the_dla34_graph_under_other_names); the arch's own default head width is 64 (opts.py:295): the
fused first head conv becomes 64 -> 64 x n_heads and the 1x1 heads read 64-channel slices of it."""
import os

import numpy as np
import pytest
import torch

import ct_oracle as co
from centertrack_b200 import synthetic as wt
from helpers import load_generic_golden, make_model

pytestmark = pytest.mark.gpu
STAGES = ['base.level2', 'base.level5', 'dla_up.ida_0.node_1', 'dla_up.ida_2.node_3', 'ida_up.node_2']


def _run(extra, precision):
  opt, model, sd = make_model('coco_tracking', extra=['--arch', 'generic'] + extra)
  model = model.cuda()
  img, pre, hm = wt.synthetic_inputs(1, 64, 96)
  eng = model.engine_for(1, 64, 96, torch.device('cuda'), precision)
  out = {k: v.clone() for k, v in eng.forward(img.cuda(), pre.cuda(), hm.cuda()).items()}
  torch.cuda.synchronize()
  return opt, model, sd, eng, out, (img, pre, hm)


@pytest.mark.parametrize('precision', ['fp32', 'bf16x3'])
@pytest.mark.parametrize('tag,extra', [('hc256', ['--head_conv', '256']), ('hc64', [])])
def test_generic_network_matches_reference_golden(tag, extra, precision, golden_dir):
  """fp32 SIMT and bf16x3 tensor-core engines within north_star's 1e-3 of the reference GenericNetwork's fp32 outputs
  (heads and trunk stages), and the CUDA-graph replay bit-identical to the eager launches."""
  g = load_generic_golden(golden_dir)
  opt, model, sd, eng, out, (img, pre, hm) = _run(extra, precision)
  for h in opt.heads:
    ref = g['%s.head.%s' % (tag, h)]
    err = np.abs(out[h].cpu().numpy() - ref)
    scale = max(1.0, float(np.abs(ref).max()))
    assert err.max() <= 1e-3 * scale and err.mean() <= 2e-4 * scale, (tag, precision, h, err.max())
  for name in STAGES:
    ref = g['%s.stage.%s' % (tag, name)]
    got = eng.stage('feat' if name == 'ida_up.node_2' else name).detach().float().cpu().numpy()
    assert np.abs(got - ref).max() <= 1e-3 * max(1.0, float(np.abs(ref).max())), (tag, precision, name)
  eng.in_img.copy_(img); eng.in_pre.copy_(pre); eng.in_hm.copy_(hm)
  rep = eng.replay()
  torch.cuda.synchronize()
  assert all(torch.equal(out[h], rep[h]) for h in out)


def test_generic_module_forward_and_reference_checkpoint_names(tmp_path, golden_dir):
  """create_model('generic', ...)(x, pre_img, pre_hm)[-1] after a save_model / load_model round trip of a checkpoint
  with the reference GenericNetwork's key names (`backbone.*`, `neck.dla_up.*`, `neck.ida_up.*`, `module.` prefix)."""
  from centertrack_b200.model import create_model, load_model, save_model
  g = load_generic_golden(golden_dir)
  opt, model, sd = make_model('coco_tracking', extra=['--arch', 'generic', '--b200_precision', 'fp32'])
  path = str(tmp_path / 'generic.pth')
  torch.save({'epoch': 3, 'state_dict': {'module.' + k: v for k, v in sd.items()}}, path)
  fresh = create_model(opt.arch, opt.heads, opt.head_conv, opt=opt)
  fresh = load_model(fresh, path, opt).cuda().eval()
  img, pre, hm = wt.synthetic_inputs(1, 64, 96)
  with torch.no_grad():
    out = fresh(img.cuda(), pre.cuda(), hm.cuda())[-1]
  for h in opt.heads:
    ref = g['hc64.head.' + h]
    assert np.abs(out[h].cpu().numpy() - ref).max() <= 1e-3 * max(1.0, float(np.abs(ref).max())), h
  save_model(path, 4, fresh)
  assert sorted(torch.load(path)['state_dict'].keys()) == list(g['hc64.keys'])


def test_generic_bf16_engine_tracks_the_emulating_oracle():
  """The benchmarked bf16 wgmma engine on the 64-wide heads (halo engine: 3x3 64 -> 256, then 1x1 heads on
  64-channel slices with ld 256) against the oracle run with the engine's rounding points, same statistic and bound as
  the dla_34 test (mean |err| <= 0.2 std)."""
  opt, model, sd, eng, out, (img, pre, hm) = _run([], 'bf16')
  emu = co.GenericDLA34Oracle(sd, opt.heads, emulate_bf16=True).forward(img, pre, hm)
  for h in opt.heads:
    ref = emu[h].numpy().ravel()
    got = out[h].float().cpu().numpy().ravel()
    assert np.abs(got - ref).mean() <= 0.2 * max(float(ref.std()), 1e-6), h
