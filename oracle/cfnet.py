"""Oracle: CFNet (stereo/modeling/models/cfnet) -- TEST / MEASUREMENT INFRASTRUCTURE (see oracle/__init__.py).

* ``reference_model``   the reference's own ``CFNet(cfg.MODEL)`` from the unchanged cfgs/cfnet/cfnet_sceneflow_part2.yaml, in eval
                        mode, with seeded weights (oracle/seeded_init.py) and the three regression heads sharpened (CFNET_SCALE)
* ``mish64``            fp64 Mish, x * tanh(softplus(x)) with F.softplus's threshold 20 (cfnet/submodule.py:99-106, 249-260)
* ``softargmin_var64``  fp64 softmax over D, expectation and variance about it: disparity_regression + disparity_variance
                        (integer planes) or the sum over disparity samples + disparity_variance_confidence
                        (cfnet/submodule.py:121-141, cfnet/cfnet.py:526-566)
"""
import torch

from . import _reference_shim as shim
from .seeded_init import seeded_state_dict

CFG = "cfgs/cfnet/cfnet_sceneflow_part2.yaml"
MODULE = "stereo.modeling.models.cfnet.cfnet"

# Sharpening factors for the seeded weights: on one 256x512 pair the un-sharpened logits of classif2 / confidence_classif1_s3 /
# confidence_classif1_s2 have a standard deviation of 0.022 / 0.14 / 0.056, so every softmax is nearly uniform; these bring them
# to 3.3 / 4.7 / 5.3, so that the disparity, its variance and the search ranges of the next stages really vary.
CFNET_SCALE = {"classif2.2.weight": 150.0, "confidence_classif1_s3.2.weight": 25.0, "confidence_classif1_s2.2.weight": 60.0}
SEED = 17


def reference_module():
    return shim.load(MODULE)


def reference_model(seed=SEED, scale=None, replace_mish=False):
    """The reference's CFNet built from the unchanged YAML, seeded, in eval mode, on the CPU."""
    mod = reference_module()
    cfg = shim.load_cfg(CFG)
    model = mod.CFNet(cfg.MODEL, replace_mish=replace_mish) if replace_mish else mod.CFNet(cfg.MODEL)
    model.load_state_dict(seeded_state_dict(model.state_dict(), seed=seed, scale=CFNET_SCALE if scale is None else scale))
    return model.eval()


def mish64(x):
    x = x.double()
    sp = torch.where(x > 20, x, torch.log1p(torch.exp(torch.clamp(x, max=20))))
    return x * torch.tanh(sp)


def softargmin_var64(cost, values=None):
    """cost (B, D, H, W) logits, values (B, D, H, W) or None (planes 0..D-1) -> (mean, variance), each (B, H, W), fp64."""
    c = cost.double()
    p = torch.softmax(c, dim=1)
    if values is None:
        v = torch.arange(c.shape[1], dtype=torch.float64, device=c.device).view(1, -1, 1, 1)
    else:
        v = values.double()
    mu = (p * v).sum(1)
    var = (p * (v - mu.unsqueeze(1)) ** 2).sum(1)
    return mu, var
