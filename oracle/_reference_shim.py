"""Import the UNMODIFIED reference modules (TEST / MEASUREMENT INFRASTRUCTURE).

Where they come from: ``/root/reference`` in the authoring container; on the GPU box (where that path does not exist) the
byte copies staged by ``oracle/make_ref.py`` under ``oracle/_ref/`` (git-ignored, shipped by gpurun).

The reference package cannot be imported normally: ``stereo/modeling/__init__.py:4-31`` imports every trainer, which pulls
``easydict``, ``timm``, ``matplotlib`` (absent from this image).  Registering empty namespace modules for the package levels
lets the sub-modules we need import without running those ``__init__`` files (SURVEY.md section 8c); ``timm`` and FoundationStereo's
``Utils`` helper (needs imageio/open3d) are stubbed -- they are only dereferenced in constructors / code paths never taken here.
"""
import importlib
import os
import sys
import types

_HERE = os.path.dirname(os.path.abspath(__file__))


def _find_root():
    env = os.environ.get("OPENSTEREO_REFERENCE")
    for cand in ([env] if env else []) + ["/root/reference", os.path.join(_HERE, "_ref")]:
        if cand and os.path.isdir(os.path.join(cand, "stereo", "modeling")):
            return cand
    return "/root/reference"


REFERENCE_ROOT = _find_root()
IS_LIVE_TREE = os.path.isdir(os.path.join(REFERENCE_ROOT, ".git")) or REFERENCE_ROOT == "/root/reference"


def available():
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "stereo", "modeling"))


def _namespace(name, path):
    if name not in sys.modules:
        mod = types.ModuleType(name)
        mod.__path__ = [path]
        sys.modules[name] = mod


def load(dotted):
    """load('stereo.modeling.cost_volume.cost_volume') -> module object of the reference."""
    if not available():
        raise RuntimeError("reference tree not present at %s" % REFERENCE_ROOT)
    root = os.path.join(REFERENCE_ROOT, "stereo")
    _namespace("stereo", root)
    _namespace("stereo.modeling", os.path.join(root, "modeling"))
    _namespace("stereo.modeling.models", os.path.join(root, "modeling", "models"))
    for sub in ("fast_foundationstereo", "foundationstereo", "igevpp", "casnet"):
        _namespace("stereo.modeling.models." + sub, os.path.join(root, "modeling", "models", sub))
        _namespace("stereo.modeling.models.%s.core" % sub, os.path.join(root, "modeling", "models", sub, "core"))
    if "timm" not in sys.modules:       # a module imported now binds whichever timm this leaves in sys.modules
        try:
            importlib.import_module("timm")
        except Exception:
            install_timm_stub()
    if "Utils" not in sys.modules:      # fast_foundationstereo/core/submodule.py:7-8 (`from Utils import AMP_DTYPE`)
        import torch
        stub = types.ModuleType("Utils")
        stub.AMP_DTYPE = torch.float16
        sys.modules["Utils"] = stub
    return importlib.import_module(dotted)


def install_timm_stub():
    """StereoBase / LightStereo / IGEV build their 2D encoders with ``timm.create_model(..., pretrained=True,
    features_only=True)`` (stereobase/backbone.py:35) -- timm is not in this image and the pretrained weights need a network.
    The encoder is outside the hot path (SURVEY.md section 2.1 row 12), so tests and the config-3 bench substitute a
    structurally identical stand-in: same attribute names, strides and channel plan as MobileNetV2-100
    (conv_stem 3->32 /2, blocks 16, 24 /2, 32 /2, 64 /2, 96, 160 /2, 320), plain conv-BN-ReLU6 inside.  Everything from the
    encoder's outputs on is the reference's unmodified code."""
    import torch.nn as nn
    timm = sys.modules.get("timm")
    if timm is not None and hasattr(timm, "create_model"):
        return timm                                     # a real timm, or the stand-in already installed: modules hold it

    def cbr(cin, cout, stride):
        return nn.Sequential(nn.Conv2d(cin, cout, 3, stride, 1, bias=False), nn.BatchNorm2d(cout), nn.ReLU6(inplace=True))

    class _MobileNetV2Shape(nn.Module):
        def __init__(self):
            super().__init__()
            self.conv_stem = nn.Conv2d(3, 32, 3, 2, 1, bias=False)
            self.bn1 = nn.BatchNorm2d(32)
            self.act1 = nn.ReLU6(inplace=True)
            plan = [(32, 16, 1), (16, 24, 2), (24, 32, 2), (32, 64, 2), (64, 96, 1), (96, 160, 2), (160, 320, 1)]
            self.blocks = nn.Sequential(*[nn.Sequential(cbr(i, o, s)) for i, o, s in plan])

    def create_model(name, pretrained=False, features_only=False, **kwargs):
        if name != "mobilenetv2_100":
            raise NotImplementedError("timm stand-in only mirrors mobilenetv2_100 (asked for %s)" % name)
        return _MobileNetV2Shape()

    stub = types.ModuleType("timm")
    stub.create_model, stub._osb_stub = create_model, True
    sys.modules["timm"] = stub
    return stub


class AttrDict(dict):
    """Five-line stand-in for easydict (absent here): cfgs.MAX_DISP and cfgs.get(...)."""

    def __getattr__(self, key):
        try:
            val = self[key]
        except KeyError as exc:
            raise AttributeError(key) from exc
        return AttrDict(val) if isinstance(val, dict) else val


def load_cfg(relpath):
    import yaml
    with open(os.path.join(REFERENCE_ROOT, relpath)) as f:
        return AttrDict(yaml.safe_load(f))
