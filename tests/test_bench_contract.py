"""bench.py pieces that run without a GPU: the `--impl reference` arm's JSON line (the oracle port on the host cores,
one 64x96-free full-size frame per step is too slow here, so the contract is checked on the smallest legal run) and
the stock-PyTorch context leg on the CPU device (same code path as on the GPU, minus the CUDA synchronisations)."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_one_json_line_with_the_contract_keys():
  r = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--impl', 'reference', '--steps', '1', '--warmup', '0'],
                     capture_output=True, text=True, timeout=600, cwd=ROOT)
  assert r.returncode == 0, r.stderr[-2000:]
  lines = [l for l in r.stdout.splitlines() if l.strip()]
  assert len(lines) == 1, r.stdout
  d = json.loads(lines[0])
  assert d['impl'] == 'reference' and d['unit'] == 'frames/s' and d['higher_is_better'] is True
  assert d['metric'] == 'frames/sec (device-timed) DLA-34 512x512'
  assert d['value'] > 0 and d['steps'] == 1
  assert d['cpu_baseline']['kind'] == 'port' and d['cpu_baseline']['cores'] >= 1 and d['cpu_baseline']['value'] == d['value']
  assert d['e2e'] == {'value': d['value'], 'unit': 'frames/s', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0}


def test_stock_pytorch_context_leg_runs_on_the_cpu_device():
  sys.path.insert(0, ROOT)
  import bench
  from centertrack_b200 import synthetic as wt
  from helpers import make_model
  opt, model, sd = make_model('coco_tracking')
  saved = bench.K
  bench.K = 40
  try:
    r = bench.stock_pytorch_leg(sd, opt.heads, 2, 64, 96, torch.device('cpu'), wt, steps=1, warmup=0)
  finally:
    bench.K = saved
  assert r['kind'] == 'port' and r['fp32'] > 0 and r['bf16_autocast'] > 0 and r['frames_per_step'] == 2


def test_dump_outputs_writes_float_arrays_and_samples_the_large_ones(tmp_path):
  """--dump-outputs: one DIR/<name>.npy per array the timed step returns (records, track tables, track counts, head
  maps); floats as float32, integers as float64; an array above `max_elems` becomes a fixed seeded sample of that many
  values under <name>_sample.npy; the same inputs give the same files."""
  import numpy as np
  sys.path.insert(0, ROOT)
  import bench

  class Stub(object):
    pass

  g = torch.Generator().manual_seed(0)
  runner, runner.tracker, runner.eng = Stub(), Stub(), Stub()
  runner.rec = torch.randn(2, 100, 15, generator=g)
  runner.tracker.tracks = torch.randn(2, 100, 13, generator=g)
  runner.tracker.counts = torch.tensor([[3, 1], [0, 2]], dtype=torch.int32)
  runner.eng.outputs = {'hm': torch.rand(2, 80, 64, 64, generator=g), 'reg': torch.randn(2, 2, 8, 8, generator=g)}
  for d in ('a', 'b'):
    bench.dump_outputs(str(tmp_path / d), runner, True, max_elems=4096)
  names = sorted(os.listdir(tmp_path / 'a'))
  assert names == ['head_hm_sample.npy', 'head_reg.npy', 'records.npy', 'track_counts.npy', 'tracks.npy']
  for n in names:
    a, b = np.load(tmp_path / 'a' / n), np.load(tmp_path / 'b' / n)
    assert a.dtype == (np.float64 if n == 'track_counts.npy' else np.float32) and np.array_equal(a, b), n
  assert np.array_equal(np.load(tmp_path / 'a' / 'records.npy'), runner.rec.numpy())
  assert np.array_equal(np.load(tmp_path / 'a' / 'track_counts.npy'), [[3, 1], [0, 2]])
  hm = np.load(tmp_path / 'a' / 'head_hm_sample.npy')
  idx = np.sort(np.random.RandomState(0).randint(0, runner.eng.outputs['hm'].numel(), 4096))
  assert hm.shape == (4096,) and np.array_equal(hm, runner.eng.outputs['hm'].numpy().reshape(-1)[idx])
  # a dump that would exceed 64 MB in all is refused
  runner.eng.outputs = {'h%d' % i: torch.zeros(3 << 20) for i in range(16)}
  try:
    bench.dump_outputs(str(tmp_path / 'c'), runner, True)
    raise AssertionError('a dump above 64 MB must be refused')
  except RuntimeError as e:
    assert '64 MB' in str(e)
