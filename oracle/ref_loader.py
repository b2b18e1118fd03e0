"""oracle/ref_loader.py -- import the UNMODIFIED reference python hot path on CPU.

TEST INFRASTRUCTURE ONLY.  Used by oracle/make_golden.py and oracle/make_ref_vectors.py where a reference checkout
exists (CL3D_REFERENCE, default /root/reference); never by the tests or the product.

Three shims make `<reference>/pytorch/{models,ops/pt_custom_ops/pt_utils.py,utils/config.py}` import
as they are (SURVEY.md section 8c):
  1. sys.modules['pt_custom_ops._ext'] = oracle.ext   (the reference's native ops are CUDA-only)
  2. an `easydict.EasyDict` stand-in                  (package not installed here)
  3. yaml.load with a default Loader                  (reference calls yaml.load(f), PyYAML >= 6 needs a Loader)
PseudoGrid.__init__ needs an initialised process group (models/utlis.py:186) and a writable kernel
directory ($JOB_LOG_DIR, models/utlis.py:158-167): a 1-rank gloo group and a temp dir are provided.
"""
import os
import sys
import tempfile
import types

REF_ROOT = os.path.join(os.environ.get("CL3D_REFERENCE", "/root/reference"), "pytorch")


def available():
    return os.path.isdir(os.path.join(REF_ROOT, "models"))


class _EasyDict(dict):
    def __init__(self, d=None, **kw):
        super().__init__()
        d = dict(d or {}, **kw)
        for k, v in d.items():
            setattr(self, k, v)

    def __setattr__(self, k, v):
        if isinstance(v, dict) and not isinstance(v, _EasyDict):
            v = _EasyDict(v)
        super().__setitem__(k, v)

    __setitem__ = __setattr__

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)


_loaded = {}


def load(ext_module=None):
    """Returns a namespace with the reference modules: .lao (local_aggregation_operators), .pt_utils,
    .config (the EasyDict global).  `ext_module` replaces pt_custom_ops._ext (default: oracle.ext)."""
    if "ns" in _loaded:
        return _loaded["ns"]
    if not available():
        raise ImportError(f"{REF_ROOT} is not present -- the tests use the tests/golden fixtures instead")
    from . import ext as oracle_ext
    ext_module = ext_module or oracle_ext
    pkg = types.ModuleType("pt_custom_ops")
    pkg.__path__ = []
    pkg._ext = ext_module
    sys.modules["pt_custom_ops"] = pkg
    sys.modules["pt_custom_ops._ext"] = ext_module
    if "easydict" not in sys.modules:
        try:
            import easydict  # noqa: F401
        except ImportError:
            m = types.ModuleType("easydict")
            m.EasyDict = _EasyDict
            sys.modules["easydict"] = m
    import yaml
    if not getattr(yaml, "_cl3d_patched", False):
        _orig = yaml.load

        def _load(stream, Loader=None):
            return _orig(stream, Loader=Loader or yaml.SafeLoader)

        yaml.load = _load
        yaml._cl3d_patched = True
    os.environ.setdefault("JOB_LOG_DIR", tempfile.mkdtemp(prefix="cl3d_ref_kernels_"))
    import torch.distributed as dist
    if not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29577")
        dist.init_process_group("gloo", rank=0, world_size=1)
    for p in (REF_ROOT, os.path.join(REF_ROOT, "ops", "pt_custom_ops")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import importlib
    pt_utils = importlib.import_module("pt_utils")
    lao = importlib.import_module("models.local_aggregation_operators")
    try:
        cfg = importlib.import_module("utils.config")
    except Exception:  # pragma: no cover
        cfg = None
    ns = types.SimpleNamespace(lao=lao, pt_utils=pt_utils, config_module=cfg, EasyDict=sys.modules["easydict"].EasyDict)
    _loaded["ns"] = ns
    return ns


def make_config(la_type, **over):
    """A fresh copy of the reference's default config (utils/config.py:77-103) with the LA family selected."""
    ns = load()
    import copy
    cfg = copy.deepcopy(ns.config_module.config)
    cfg.local_aggregation_type = la_type
    for k, v in over.items():
        if isinstance(v, dict):
            for kk, vv in v.items():
                cfg[k][kk] = vv
        else:
            cfg[k] = v
    return cfg
