"""The C-ABI library builds for sm_90a, loads without a GPU, and exports every symbol the public
header declares (no compute calls here)."""
import ctypes
import os
import re

from conftest import ROOT


def _declared():
  src = open(os.path.join(ROOT, 'include', 'ctb200.h')).read()
  src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
  return sorted(set(re.findall(r'\b(ct_[a-z0-9_]+)\s*\(', src)))


def test_header_declares_entry_points():
  names = _declared()
  for must in ('ct_conv_forward', 'ct_decode', 'ct_stem_forward', 'ct_maxpool2', 'ct_maxpool2_s2d', 'ct_upsample_add',
               'ct_pack_weights', 'ct_last_error'):
    assert must in names


def test_library_exports_every_declared_symbol(built_lib):
  lib = ctypes.CDLL(built_lib)
  for name in _declared():
    assert hasattr(lib, name), 'libctb200.so does not export %s' % name
  lib.ct_abi_version.restype = ctypes.c_int
  assert lib.ct_abi_version() == 1


def test_python_binding_lists_match_header(built_lib):
  from centertrack_b200 import _lib
  assert sorted(_lib.EXPORTS) == _declared()
  _lib.lib()     # argtypes/restype wiring must not raise


def test_sass_is_hopper_native(built_lib):
  """wgmma / TMA bulk copy / mbarrier must be in the SASS (HGMMA + WARPGROUP fences / UBLKCP / UTMALDG tensor loads /
  SYNCS mbarrier transactions)."""
  import shutil
  import subprocess
  if shutil.which('cuobjdump') is None:
    import pytest
    pytest.skip('cuobjdump not available')
  sass = subprocess.run(['cuobjdump', '-sass', built_lib], capture_output=True, text=True).stdout
  for mnemonic in ('HGMMA', 'WARPGROUP', 'UBLKCP', 'UTMALDG', 'SYNCS'):
    assert mnemonic in sass, mnemonic


def test_host_weight_packing_roundtrip(built_lib):
  """ct_pack_weights (host code, no GPU): SIMT layout k-major; tensor-core layout = 128B-swizzled tiles."""
  import numpy as np
  from centertrack_b200 import _lib as L
  lib = L.lib()
  rng = np.random.RandomState(0)
  O, I, k = 24, 16, 3
  w = rng.randn(O, I, k, k).astype(np.float32)
  n = lib.ct_packed_weight_bytes(L.CT_ENGINE_SIMT, O, I, k, k, 0)
  dst = np.zeros(n // 4, dtype=np.float32)
  assert lib.ct_pack_weights(L.CT_ENGINE_SIMT, w.ctypes.data, O, I, k, k, 0, dst.ctypes.data) == 0
  ldw = 64
  ref = np.zeros((k * k * I, ldw), np.float32)
  ref[:, :O] = w.transpose(2, 3, 1, 0).reshape(k * k * I, O)
  assert np.array_equal(dst.reshape(-1, ldw), ref)
  # tensor-core engine: de-swizzle and compare against bf16-rounded weights
  n_tile = 32
  n = lib.ct_packed_weight_bytes(L.CT_ENGINE_TCGEN05, O, I, k, k, n_tile)
  ks = (k * k * I + 63) // 64
  assert n == 1 * ks * n_tile * 64 * 2
  dst = np.zeros(n // 2, dtype=np.uint16)
  assert lib.ct_pack_weights(L.CT_ENGINE_TCGEN05, w.ctypes.data, O, I, k, k, n_tile, dst.ctypes.data) == 0
  tiles = dst.reshape(ks, n_tile, 8, 8)          # [slice][row][chunk][elem]
  wk = w.transpose(0, 2, 3, 1).reshape(O, k * k * I)   # k = tap*C_in + c
  import torch
  wk_bf16 = torch.from_numpy(wk).bfloat16().view(torch.int16).numpy().view(np.uint16)
  for r in range(O):
    for kk in range(k * k * I):
      s, j = divmod(kk, 64)
      chunk = (j // 8) ^ (r & 7)
      assert tiles[s, r, chunk, j % 8] == wk_bf16[r, kk]
  assert lib.ct_pack_weights(L.CT_ENGINE_TCGEN05, w.ctypes.data, O, I, k, k, 20, dst.ctypes.data) != 0
  assert b'n_tile' in lib.ct_last_error()


def test_product_path_refuses_to_run_without_a_gpu(built_lib):
  """No CPU fallback anywhere on the product path: every public entry point raises on host tensors / no device."""
  import sys
  import pytest
  import torch
  sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
  from helpers import make_model, make_opt
  from centertrack_b200.dcn import DCN
  from centertrack_b200.decode import generic_decode
  from centertrack_b200.detector import Detector
  opt, model, _ = make_model('coco_tracking')
  z = torch.zeros(1, 3, 64, 96)
  with pytest.raises(RuntimeError, match='no CPU fallback'):
    model(z, z, torch.zeros(1, 1, 64, 96))
  with pytest.raises(RuntimeError, match='no CPU fallback'):
    generic_decode({'hm': torch.rand(1, 2, 8, 8), 'reg': torch.rand(1, 2, 8, 8), 'wh': torch.rand(1, 2, 8, 8)}, K=4)
  with pytest.raises(RuntimeError, match='no CPU fallback'):
    DCN(64, 64)(torch.zeros(1, 64, 8, 8))
  with pytest.raises(RuntimeError, match='no CPU fallback'):
    Detector(make_opt('coco_tracking', ['--gpus', '-1']))


def test_argument_validation_returns_status_without_touching_the_gpu(built_lib):
  """Every entry point validates before it launches: bad descriptors come back as a negative ct_status with a
  message in ct_last_error(), nothing throws across the ABI (checked here on a machine with no GPU)."""
  import sys
  sys.path.insert(0, ROOT)
  from centertrack_b200 import _lib as L
  lib = L.lib()
  assert lib.ct_decode(ctypes.byref(L.DecodeDesc()), None) == -1 and b'null pointer' in lib.ct_last_error()
  assert lib.ct_conv_forward(ctypes.byref(L.ConvDesc()), None) == -1 and b'ct_conv_forward' in lib.ct_last_error()
  p = ctypes.c_void_p(16)
  assert lib.ct_upsample_add(p, None, p, p, L.CT_BF16, 1, 4, 4, 8, 3, 8, 8, 8, None) == -1
  assert b'upsample factor' in lib.ct_last_error()
  assert lib.ct_upsample_add(p, None, p, p, L.CT_BF16, 1, 4, 4, 12, 2, 12, 12, 12, None) == -1     # C % 8 != 0
  assert lib.ct_packed_weight_bytes(L.CT_ENGINE_TCGEN05, 64, 64, 3, 3, 24) == -1                     # n_tile % 16
  assert lib.ct_packed_weight_bytes(L.CT_ENGINE_TCGEN05, 64, 64, 3, 3, 64) == 64 * (9 * 64) * 2
  assert lib.ct_decode_workspace_bytes(2, 80, 0, 100) == 256 + 8 * 2 * 80 * 100
