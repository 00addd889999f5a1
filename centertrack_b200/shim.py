"""install(): make the reference's import names resolve to this package, so the reference's own
`src/demo.py` / `src/test.py` (which do `from detector import Detector`, `from opts import opts`, ...) run
unchanged on the H100 path.  See INTEGRATION.md.

    import centertrack_b200.shim as shim; shim.install()        # before importing the reference scripts
    # or, DCN only (keep the reference's PyTorch graph, swap its absent CUDA extension):
    shim.install_dcn_only()

How it works.  A `sys.meta_path` finder placed FIRST answers, lazily and only for the leaf modules this package
replaces, with the H100 implementation:

    detector                          -> centertrack_b200.detector      (Detector)
    model.model                       -> centertrack_b200.model         (create_model / load_model / save_model)
    model.decode                      -> centertrack_b200.decode        (generic_decode)
    utils.tracker                     -> centertrack_b200.tracker       (Tracker)
    model.networks.DCNv2.dcn_v2       -> centertrack_b200.dcn           (DCN; dla.py:18-22 imports it in a try)

Every other name -- `opts`, `logger`, `utils.utils`, `utils.debugger`, `utils.image`, `utils.post_process`,
`model.utils`, `dataset.dataset_factory`, `dataset.datasets.*` -- is left to the normal import machinery, i.e. to
the REFERENCE's own files once `src/lib` is on `sys.path` (the reference's `_init_paths` puts it there, whether
that happens before or after install(): nothing is resolved until it is imported).  Only when the reference is NOT
importable (stand-alone use of this package under the reference's names) do the parents `model`, `model.networks`,
`utils`, `dataset` fall back to empty synthetic packages and `opts`, `utils.image`, `utils.post_process`,
`dataset.dataset_factory` to this package's host-side mirrors.  (Round 1 registered empty packages eagerly, which
shadowed the reference's `utils.utils` / `model.utils` / `logger` and broke `src/test.py`.)
"""
import importlib
import importlib.abc
import importlib.machinery
import sys
import types

_ALWAYS = {
    'detector': 'centertrack_b200.detector',
    'model.model': 'centertrack_b200.model',
    'model.decode': 'centertrack_b200.decode',
    'utils.tracker': 'centertrack_b200.tracker',
    'model.networks.DCNv2.dcn_v2': 'centertrack_b200.dcn',
}
_DCN_ONLY = {'model.networks.DCNv2.dcn_v2': 'centertrack_b200.dcn'}
# used only when no other finder can supply the name (reference not importable)
_FALLBACK = {
    'opts': 'centertrack_b200.opts',
    'utils.image': 'centertrack_b200.image',
    'utils.post_process': 'centertrack_b200.post_process',
    'dataset.dataset_factory': 'centertrack_b200.dataset_info',
}
_PACKAGES = ('model', 'model.networks', 'model.networks.DCNv2', 'utils', 'dataset')


class _AliasLoader(importlib.abc.Loader):

  def __init__(self, target):
    self.target = target

  def create_module(self, spec):
    if self.target is None:                       # synthetic empty package
      m = types.ModuleType(spec.name)
      m.__path__ = []
      return m
    return importlib.import_module(self.target)   # the SAME module object under a second name

  def exec_module(self, module):
    pass


class B200Finder(importlib.abc.MetaPathFinder):

  def __init__(self, aliases):
    self.aliases = dict(aliases)
    self.full = aliases is _ALWAYS

  def _others(self, name, path, target):
    for f in sys.meta_path:
      if f is self or not hasattr(f, 'find_spec'):
        continue
      try:
        spec = f.find_spec(name, path, target)
      except Exception:
        spec = None
      if spec is not None:
        return spec
    return None

  def find_spec(self, name, path=None, target=None):
    if name in self.aliases:
      return importlib.machinery.ModuleSpec(name, _AliasLoader(self.aliases[name]))
    if name in _PACKAGES or (self.full and name in _FALLBACK):
      spec = self._others(name, path, target)
      if spec is not None:
        return None                                # the reference (or anything real) wins
      if name in _PACKAGES:
        return importlib.machinery.ModuleSpec(name, _AliasLoader(None), is_package=True)
      return importlib.machinery.ModuleSpec(name, _AliasLoader(_FALLBACK[name]))
    return None


def _installed():
  return [f for f in sys.meta_path if isinstance(f, B200Finder)]


def _install(aliases):
  for f in _installed():
    sys.meta_path.remove(f)
  for name in aliases:                             # a copy imported earlier (e.g. the reference's detector) must go
    sys.modules.pop(name, None)
  finder = B200Finder(aliases)
  sys.meta_path.insert(0, finder)
  importlib.invalidate_caches()
  return finder


def install_dcn_only():
  """Only `model.networks.DCNv2.dcn_v2.DCN`: the reference's own DLASeg then runs with our DCN kernels."""
  _install(_DCN_ONLY)
  return importlib.import_module('model.networks.DCNv2.dcn_v2')


def install():
  """-> {reference module name: product module} of the names that are always replaced."""
  _install(_ALWAYS)
  return {name: importlib.import_module(target) for name, target in _ALWAYS.items()}


def uninstall():
  for f in _installed():
    sys.meta_path.remove(f)
  for name in list(_ALWAYS) + list(_FALLBACK):
    m = sys.modules.get(name)
    if m is not None and getattr(m, '__name__', name) != name:
      sys.modules.pop(name, None)
