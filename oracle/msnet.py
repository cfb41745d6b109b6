"""Oracle: MSNet3D's 3D part (TEST INFRASTRUCTURE -- see oracle/__init__.py).

* ``MobileV2Residual3D``  ``MobileV2_Residual_3D``, same state_dict keys            stereo/modeling/models/msnet/submodule.py:136-173
* ``Hourglass3D``         ``hourglass3D``                                           msnet/MSNet3D.py:10-46
* ``Aggregation``         the eval forward after the cost volume: dres0, dres1 (+ cost0), three hourglasses, classif3, the
                          trilinear x4 + softmax + regression (MSNet3D.py:118-161); its state_dict keys are the model's keys of
                          those modules
* ``eval_forward``        MSNet3D's eval forward (MSNet3D.py:110-161) around any feature extractor (the reference's own 2D
                          MobileNet is outside the hot path and is not restated)

Same aten calls in the same order as the reference, on fp32 CPU tensors; bit-equality is asserted by tools/make_golden.py and
tests/test_msnet_cpu.py.
"""
import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _reference_shim as shim
from .cost_volume import build_gwc_volume

# seeded_state_dict's N(0, 1/fan_in) weights leave MSNet3D's logits nearly flat (std 0.03 at 64 x 128): the softmax is then
# uniform and the disparity carries no signal.  Sharpening the last classifier conv gives logits of std ~4 and a disparity std of
# several pixels.
MSNET3D_SCALE = {"classif3.2.weight": 125.0}


def load_reference(dotted):
    """Import a module of the reference's msnet package without running its __init__ (which imports the trainer stack)."""
    shim._namespace("stereo.modeling.models.msnet", os.path.join(shim.REFERENCE_ROOT, "stereo", "modeling", "models", "msnet"))
    return shim.load(dotted)


def convbn_3d(in_channels, out_channels, kernel_size, stride, pad):
    return nn.Sequential(nn.Conv3d(in_channels, out_channels, kernel_size=kernel_size, stride=stride, padding=pad, bias=False),
                         nn.BatchNorm3d(out_channels))


class MobileV2Residual3D(nn.Module):
    def __init__(self, inp, oup, stride, expanse_ratio):
        super().__init__()
        self.stride = stride
        hidden_dim = round(inp * expanse_ratio)
        self.use_res_connect = self.stride == (1, 1, 1) and inp == oup      # False for an int stride, as in the reference
        if expanse_ratio == 1:
            self.conv = nn.Sequential(
                nn.Conv3d(hidden_dim, hidden_dim, 3, stride, 1, groups=hidden_dim, bias=False), nn.BatchNorm3d(hidden_dim),
                nn.ReLU6(inplace=True),
                nn.Conv3d(hidden_dim, oup, 1, 1, 0, bias=False), nn.BatchNorm3d(oup))
        else:
            self.conv = nn.Sequential(
                nn.Conv3d(inp, hidden_dim, 1, 1, 0, bias=False), nn.BatchNorm3d(hidden_dim), nn.ReLU6(inplace=True),
                nn.Conv3d(hidden_dim, hidden_dim, 3, stride, 1, groups=hidden_dim, bias=False), nn.BatchNorm3d(hidden_dim),
                nn.ReLU6(inplace=True),
                nn.Conv3d(hidden_dim, oup, 1, 1, 0, bias=False), nn.BatchNorm3d(oup))

    def forward(self, x):
        if self.use_res_connect:
            return x + self.conv(x)
        return self.conv(x)


class Hourglass3D(nn.Module):
    def __init__(self, in_channels):
        super().__init__()
        r = 2
        self.conv1 = MobileV2Residual3D(in_channels, in_channels * 2, 2, r)
        self.conv2 = MobileV2Residual3D(in_channels * 2, in_channels * 2, 1, r)
        self.conv3 = MobileV2Residual3D(in_channels * 2, in_channels * 4, 2, r)
        self.conv4 = MobileV2Residual3D(in_channels * 4, in_channels * 4, 1, r)
        self.conv5 = nn.Sequential(
            nn.ConvTranspose3d(in_channels * 4, in_channels * 2, 3, padding=1, output_padding=1, stride=2, bias=False),
            nn.BatchNorm3d(in_channels * 2))
        self.conv6 = nn.Sequential(
            nn.ConvTranspose3d(in_channels * 2, in_channels, 3, padding=1, output_padding=1, stride=2, bias=False),
            nn.BatchNorm3d(in_channels))
        self.redir1 = MobileV2Residual3D(in_channels, in_channels, 1, r)
        self.redir2 = MobileV2Residual3D(in_channels * 2, in_channels * 2, 1, r)

    def forward(self, x):
        conv1 = self.conv1(x)
        conv2 = self.conv2(conv1)
        conv3 = self.conv3(conv2)
        conv4 = self.conv4(conv3)
        conv5 = F.relu(self.conv5(conv4) + self.redir2(conv2), inplace=True)
        conv6 = F.relu(self.conv6(conv5) + self.redir1(x), inplace=True)
        return conv6


class Aggregation(nn.Module):
    """MSNet3D after the gwc volume (eval): volume (B, 40, D/4, H/4, W/4) -> logits (B, 1, D/4, H/4, W/4) with ``logits``, the
    disparity (B, H, W) with ``forward``."""

    def __init__(self, maxdisp=192, num_groups=40, hourglass_size=32, dres_expanse_ratio=3):
        super().__init__()
        self.maxdisp = maxdisp
        c, r = hourglass_size, dres_expanse_ratio
        self.dres0 = nn.Sequential(MobileV2Residual3D(num_groups, c, 1, r), MobileV2Residual3D(c, c, 1, r))
        self.dres1 = nn.Sequential(MobileV2Residual3D(c, c, 1, r), MobileV2Residual3D(c, c, 1, r))
        self.encoder_decoder1 = Hourglass3D(c)
        self.encoder_decoder2 = Hourglass3D(c)
        self.encoder_decoder3 = Hourglass3D(c)
        self.classif3 = nn.Sequential(convbn_3d(c, c, 3, 1, 1), nn.ReLU(inplace=True),
                                      nn.Conv3d(c, 1, kernel_size=3, padding=1, stride=1, bias=False, dilation=1))

    def logits(self, volume):
        cost0 = self.dres0(volume)
        cost0 = self.dres1(cost0) + cost0
        out1 = self.encoder_decoder1(cost0)
        out2 = self.encoder_decoder2(out1)
        out3 = self.encoder_decoder3(out2)
        return self.classif3(out3)

    def forward(self, volume, h, w):
        cost3 = F.interpolate(self.logits(volume), [self.maxdisp, h, w], mode="trilinear")
        cost3 = torch.squeeze(cost3, 1)
        pred3 = F.softmax(cost3, dim=1)
        disp_values = torch.arange(0, self.maxdisp, dtype=pred3.dtype, device=pred3.device).view(1, self.maxdisp, 1, 1)
        return torch.sum(pred3 * disp_values, 1, keepdim=False)


def aggregation_of(model):
    """An oracle Aggregation holding `model`'s (an MSNet3D) weights."""
    agg = Aggregation(maxdisp=model.maxdisp, num_groups=model.num_groups, hourglass_size=model.hourglass_size,
                      dres_expanse_ratio=model.dres_expanse_ratio)
    sd = model.state_dict()
    agg.load_state_dict({k: sd[k] for k in agg.state_dict()})
    return agg.eval()


def eval_forward(feature_extraction, agg, left, right, num_groups=40):
    """MSNet3D.forward in eval mode (MSNet3D.py:110-161) -> {'disp_pred': (B, H, W)}."""
    features_left = feature_extraction(left)
    features_right = feature_extraction(right)
    volume = build_gwc_volume(features_left, features_right, agg.maxdisp // 4, num_groups)
    return {"disp_pred": agg(volume, left.size()[2], left.size()[3])}
