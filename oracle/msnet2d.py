"""Oracle: MSNet2D (stereo/modeling/models/msnet/MSNet2D.py) -- TEST / MEASUREMENT INFRASTRUCTURE (see oracle/__init__.py).

* ``reference_model``     the reference's own ``MSNet2D(cfg.MODEL)`` from the unchanged cfgs/msnet/msnet2d_sceneflow.yaml, in eval
                          mode, with seeded weights (oracle/seeded_init.py) and classif3's last conv sharpened (MSNET2D_SCALE)
* ``volume_loop``         the reference's 48-iteration volume loop (MSNet2D.py:143-162) on given preconv11 features, calling the
                          model's own interweave_tensors, conv3d and volume11
* ``interlaced_crops64``  fp64 gather of the library's cropped, block-interleaved inputs (include/openstereo_b200.h:
                          osb_interlaced_crops_fwd), written from its index formula
* ``stages``              the eval forward split where the library splits it: features, volume, aggregation logits, tail
"""
import torch
import torch.nn.functional as F

from . import _reference_shim as shim
from .msnet import load_reference
from .seeded_init import seeded_state_dict

CFG = "cfgs/msnet/msnet2d_sceneflow.yaml"
MODULE = "stereo.modeling.models.msnet.MSNet2D"

# With seeded_state_dict's N(0, 1/fan_in) weights volume11's 16 -> 1 conv varies by 0.006 around a BN shift of -0.13, so its
# ReLU zeroes the whole volume, and classif3's logits have a standard deviation of 0.33, so the softmax is nearly uniform.  These
# factors (and the seed) give, on random 128 x 256 images, a volume positive on 57% of its voxels with a standard deviation of 0.3,
# logits of standard deviation 3.9 and a disparity of standard deviation 20 px.
MSNET2D_SCALE = {"volume11.0.0.weight": 30.0, "classif3.2.weight": 10.0}
SEED = 22


def reference_module():
    return load_reference(MODULE)


def reference_model(seed=SEED, scale=None):
    """The reference's MSNet2D built from the unchanged YAML, seeded, in eval mode, on the CPU."""
    cfg = shim.load_cfg(CFG)
    model = reference_module().MSNet2D(cfg.MODEL)
    model.load_state_dict(seeded_state_dict(model.state_dict(), seed=seed, scale=MSNET2D_SCALE if scale is None else scale))
    return model.eval()


def volume_loop(model, feat_left, feat_right):
    """MSNet2D.py:143-162 verbatim on the preconv11 outputs -> volume (B, 48, H, W)."""
    interweave = load_reference("stereo.modeling.models.msnet.submodule").interweave_tensors
    featL, featR = feat_left, feat_right
    B, C, H, W = featL.shape
    volume = featL.new_zeros([B, model.num_groups, model.volume_size, H, W])
    for i in range(model.volume_size):
        if i > 0:
            x = interweave(featL[:, :, :, i:], featR[:, :, :, :-i])
            x = torch.unsqueeze(x, 1)
            x = model.conv3d(x)
            x = torch.squeeze(x, 2)
            x = model.volume11(x)
            volume[:, :, i, :, i:] = x
        else:
            x = interweave(featL, featR)
            x = torch.unsqueeze(x, 1)
            x = model.conv3d(x)
            x = torch.squeeze(x, 2)
            x = model.volume11(x)
            volume[:, :, i, :, :] = x
    return torch.squeeze(volume.contiguous(), 1)


def interlaced_crops64(left, right, ndisp):
    """[x_d (B, H, W - d, 2C) fp64]: x_d[b, h, w - d, 8j + k] = left[b, 4j + k, h, w], x_d[..., 8j + 4 + k] = right[b, 4j + k, h, w - d]."""
    left, right = left.double(), right.double()
    b, c, h, w = left.shape
    out = []
    for d in range(ndisp):
        lv = left[..., d:].reshape(b, c // 4, 4, h, w - d)
        rv = right[..., :w - d].reshape(b, c // 4, 4, h, w - d)
        out.append(torch.stack((lv, rv), 2).reshape(b, 2 * c, h, w - d).permute(0, 2, 3, 1).contiguous())
    return out


def stages(model, left, right):
    """The reference's eval forward cut at the library's stage boundaries -> dict of features, volume, logits, disp."""
    fl = model.preconv11(model.feature_extraction(left))
    fr = model.preconv11(model.feature_extraction(right))
    volume = volume_loop(model, fl, fr)
    cost0 = model.dres0(volume)
    cost0 = model.dres1(cost0) + cost0
    out3 = model.encoder_decoder3(model.encoder_decoder2(model.encoder_decoder1(cost0)))
    logits = model.classif3(out3)
    cost3 = torch.squeeze(F.interpolate(torch.unsqueeze(logits, 1), [model.maxdisp, left.shape[2], left.shape[3]], mode="trilinear"), 1)
    pred3 = F.softmax(cost3, dim=1)
    disp_values = torch.arange(0, model.maxdisp, dtype=pred3.dtype, device=pred3.device).view(1, model.maxdisp, 1, 1)
    return {"feat_left": fl, "feat_right": fr, "volume": volume, "logits": logits, "disp": torch.sum(pred3 * disp_values, 1)}
