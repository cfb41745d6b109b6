"""Oracle: MonSter built by the reference's own class (TEST / MEASUREMENT INFRASTRUCTURE -- see oracle/__init__.py).

* ``monster(yaml, seed, encoder)``  the reference's MonSter, eval mode, from an unchanged YAML with seeded parameters.  Its
  constructor torch.load()s a Depth Anything V2 checkpoint (monster.py:293); while it runs, the loader is substituted by one that
  returns the state dict of a freshly built DepthAnythingV2 of the same encoder, so nothing is downloaded or read from disk.  Every
  parameter is then replaced by oracle/seeded_init.py's seeded values.  ``encoder`` overrides the YAML's (tests use ``vits`` to
  keep the CPU reference quick: the stereo path does not depend on it).
* matplotlib, imported by monster.py and unused, is stubbed where it is absent; without xformers the DINOv2 attention takes its
  plain fallback.
* ``amp_dtype(yaml)``  the autocast dtype MonSter's trainer runs a YAML under (trainer.py:58-84), or None without AMP.
"""
import contextlib
import sys
import types

import torch

from oracle import _reference_shim as shim
from oracle import seeded_init as si

UNIFORM_YAML = "cfgs/monster/monster_sceneflow_uniform.yaml"
AMP_YAML = "cfgs/monster/monster_sceneflow.yaml"
# As for IGEV (oracle/igev_rt.py): sharpen the classifier so that the initial disparity spreads over the range.
MONSTER_SCALE = {"classifier.weight": 8.0}

_MONO = {"vits": dict(encoder="vits", features=64, out_channels=[48, 96, 192, 384]),
         "vitb": dict(encoder="vitb", features=128, out_channels=[96, 192, 384, 768]),
         "vitl": dict(encoder="vitl", features=256, out_channels=[256, 512, 1024, 1024])}


def _stub_matplotlib():
    """monster.py:9 imports matplotlib.pyplot and never uses it; where matplotlib is absent, empty modules stand in."""
    try:
        import matplotlib.pyplot  # noqa: F401
    except ImportError:
        mpl = sys.modules.get("matplotlib") or types.ModuleType("matplotlib")
        mpl.pyplot = types.ModuleType("matplotlib.pyplot")
        sys.modules["matplotlib"], sys.modules["matplotlib.pyplot"] = mpl, mpl.pyplot


def load_reference(dotted):
    """Import a module of the reference's monster package (a directory without __init__.py)."""
    _stub_matplotlib()
    return shim.load(dotted)


@contextlib.contextmanager
def _checkpoint_from(state_dict):
    real = torch.load
    torch.load = lambda *args, **kwargs: state_dict
    try:
        yield
    finally:
        torch.load = real


def amp_dtype(yaml):
    opt = shim.load_cfg(yaml).OPTIMIZATION
    if not opt.get("AMP", False):
        return None
    return torch.bfloat16 if str(opt.get("AMP_DTYPE", "fp16")).lower() in ("bf16", "bfloat16") else torch.float16


def monster(yaml=UNIFORM_YAML, seed=7, encoder="vits"):
    """The reference's MonSter, eval mode, built from `yaml` unchanged (encoder overridden when given), seeded weights."""
    cfg = shim.load_cfg(yaml).MODEL
    if encoder is not None:
        cfg.encoder = encoder
    dpt = load_reference("stereo.modeling.models.monster.depth_anything_v2.dpt")
    with _checkpoint_from(dpt.DepthAnythingV2(**_MONO[cfg.encoder]).state_dict()):
        m = load_reference("stereo.modeling.models.monster.monster").MonSter(cfg).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=seed, scale=MONSTER_SCALE))
    return m
