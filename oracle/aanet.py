"""Oracle: AANet built by the reference's own class, and a CPU reference of its modulated deformable convolution (TEST /
MEASUREMENT INFRASTRUCTURE -- see oracle/__init__.py).

* ``aanet(yaml, seed, offset_scale)``  the reference's ``aanet``, eval mode, from an unchanged YAML with seeded parameters.  Its
  submodule imports ``stereo.libs.AANet.deform_conv``, whose wrapper imports the compiled ``deform_conv_cuda`` extension as a
  sibling module; ``load_reference`` registers the build that oracle/make_ref.py staged under oracle/_ref/ under that name
  first, so the import succeeds from the live reference tree and from the staged copy alike.  The seeded ``offset_conv`` weights
  and biases are multiplied by ``offset_scale``: the reference initialises them to zero, which makes every deformable layer a plain
  dilated convolution with mask 1 and would leave the gather untested.
* ``modulated_deform_conv(...)``  the forward of the reference's modulated_deform_conv (deform_conv.py:113-150) on CPU tensors,
  through ``torchvision.ops.deform_conv2d(mask=...)``: the reference refuses CPU tensors (deform_conv.py:135-136).  Same offset
  layout ((dy, dx) per tap, per deformable group), same zero outside (-1, H) x (-1, W) and per-corner bilinear weights.
"""
import importlib.util
import os
import sys

import torch

from oracle import _reference_shim as shim
from oracle import seeded_init as si
from oracle.make_ref import extension_path

EVAL_YAML = "cfgs/aanet/aanet_sceneflow.yaml"
_EXT = "stereo.libs.AANet.deform_conv.deform_conv_cuda"


def extension_available():
    return os.path.exists(extension_path())


def load_reference(dotted):
    """Import a module of the reference with the staged deform_conv_cuda build registered as the wrapper's sibling module."""
    if _EXT not in sys.modules:
        path = extension_path()
        if not os.path.exists(path):
            raise RuntimeError("the reference's deform_conv_cuda is not built (%s): run oracle/make_ref.py" % path)
        spec = importlib.util.spec_from_file_location(_EXT, path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        sys.modules[_EXT] = mod
    return shim.load(dotted)


def aanet_class():
    return load_reference("stereo.modeling.models.aanet.aanet").aanet


def aanet(yaml=EVAL_YAML, seed=5, offset_scale=1.0):
    """The reference's aanet, eval mode, built from `yaml` unchanged, seeded weights; offset_conv weights and biases times
    `offset_scale`."""
    m = aanet_class()(shim.load_cfg(yaml).MODEL).eval()
    sd = si.seeded_state_dict(m.state_dict(), seed=seed)
    for k in sd:
        if ".offset_conv." in k:
            sd[k] = sd[k] * offset_scale
    m.load_state_dict(sd)
    return m


def modulated_deform_conv(input, offset, mask, weight, bias=None, stride=1, padding=0, dilation=1, deformable_groups=None):
    """(B, Cin, H, W), (B, dg*18, Ho, Wo), (B, dg*9, Ho, Wo), (Cout, Cin, 3, 3) -> (B, Cout, Ho, Wo), groups = 1, in the inputs'
    dtype (fp64 inputs give an fp64 reference).  dg is read from the offsets' channels (deform_conv2d does the same)."""
    from torchvision.ops import deform_conv2d
    dg = offset.shape[1] // 18
    assert offset.shape[1] == 18 * dg and mask.shape[1] == 9 * dg and deformable_groups in (None, dg)
    return deform_conv2d(input, offset, weight, bias, stride=stride, padding=padding, dilation=dilation, mask=mask)
