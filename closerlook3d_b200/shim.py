"""Make the reference's own `models/`, `cfgs/` and `function/` run on this package with zero edits.

The reference reaches the hot path through two bare module names put on sys.path by its own files
(`from pt_utils import MaskedQueryAndGroup`, models/local_aggregation_operators.py:13; `from pt_utils import
MaskedMaxPool`, models/backbones/resnet.py:11; `MaskedUpsample`, models/heads/segmentation_head.py:12) and
through `from ..local_aggregation_operators import LocalAggregation` (resnet.py:3).  `install()` pre-seeds
sys.modules so that those imports resolve to this package's drop-in modules, and re-binds the reference's
MultiPartSegHeadResNet to this package's (same module tree, heads fused).  It also provides the two small
compatibility shims the reference needs on a current stack (easydict not installed; yaml.load without Loader).
"""
import importlib
import os
import sys
import types


def install(reference_pytorch_root=None):
    from . import local_aggregation_operators as lao
    from . import pt_utils
    sys.modules["pt_utils"] = pt_utils
    if "easydict" not in sys.modules:
        try:
            import easydict  # noqa: F401
        except ImportError:
            from .config import AttrDict

            class EasyDict(AttrDict):
                def __init__(self, d=None, **kw):
                    super().__init__()
                    for k, v in dict(d or {}, **kw).items():
                        self[k] = EasyDict(v) if isinstance(v, dict) and not isinstance(v, EasyDict) else v

                def __setattr__(self, k, v):
                    self[k] = EasyDict(v) if isinstance(v, dict) and not isinstance(v, EasyDict) else v

            m = types.ModuleType("easydict")
            m.EasyDict = EasyDict
            sys.modules["easydict"] = m
    import yaml
    if not getattr(yaml, "_cl3d_patched", False):
        _orig = yaml.load
        yaml.load = lambda stream, Loader=None: _orig(stream, Loader=Loader or yaml.SafeLoader)
        yaml._cl3d_patched = True
    if reference_pytorch_root:
        if reference_pytorch_root not in sys.path:
            sys.path.insert(0, reference_pytorch_root)
        # The operator module must be replaced BEFORE the reference's `models` package is imported: models/__init__
        # -> build -> backbones/resnet.py:3 runs `from ..local_aggregation_operators import LocalAggregation` during
        # that import, and a name bound by a from-import is not re-bound by a later sys.modules change.
        sys.modules["models.local_aggregation_operators"] = lao
        if os.path.isdir(os.path.join(reference_pytorch_root, "models")):
            pkg = importlib.import_module("models")
            pkg.local_aggregation_operators = lao
            # a `models` package imported before install() already holds the reference's classes: re-bind them
            for name, mod in list(sys.modules.items()):
                if mod is not None and (name == "models" or name.startswith("models.")) and mod is not lao:
                    for attr in ("LocalAggregation", "PosPool", "AdaptiveWeight", "PointWiseMLP", "PseudoGrid"):
                        if hasattr(mod, attr) and getattr(mod, attr) is not getattr(lao, attr):
                            setattr(mod, attr, getattr(lao, attr))
            # the part-segmentation head runs its S shape heads fused: models/build.py binds the class by name
            # (`from .heads import MultiPartSegHeadResNet`), so every module that holds it is re-bound
            from .backbone import MultiPartSegHeadResNet
            for name in ("models.heads.segmentation_head", "models.heads", "models.build"):
                try:
                    mod = importlib.import_module(name)
                except ImportError:
                    continue
                if hasattr(mod, "MultiPartSegHeadResNet"):
                    mod.MultiPartSegHeadResNet = MultiPartSegHeadResNet


def reference_config(yaml_path):
    """the reference's global config updated from one of its cfgs/*.yaml (utils/config.py:106-117)"""
    cfgmod = importlib.import_module("utils.config")
    cfgmod.update_config(yaml_path)
    return cfgmod.config
