"""Oracle: CasStereo (CasPSMNet / CasGwcNet) cost volumes and aggregation (TEST INFRASTRUCTURE -- see oracle/__init__.py).

* ``warped_concat_volume``       CasPSMNet ``GetCostVolume.forward``      stereo/modeling/models/casnet/cas_psm.py:286-318
* ``warped_gwc_concat_volume``   CasGwcNet ``GetCostVolume.forward``      stereo/modeling/models/casnet/cas_gwc.py:263-329
* ``CostAggregation``            eval branch of ``CostAggregation``       cas_psm.py:182-279 (identical in cas_gwc.py:159-256),
                                 hourglass cas_psm.py:6-43 (= gwcnet/hourglass.py, restated in oracle/aggregation.py)
* ``upsample_softargmin_values`` its tail: trilinear up-sampling of the classifier logits, softmax over D, expectation over
                                 the per-pixel hypotheses (cas_psm.py:268-274, casnet/submodule.py:22-24)

Same aten calls in the same order as the reference, on fp32 CPU tensors; bit-equality is asserted by tools/make_golden.py and
tests/test_cascade_cpu.py.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .aggregation import GwcHourglass, _gwc_cb
from .regression import disparity_regression_values

# Sharpening factors for oracle.seeded_init.seeded_state_dict(..., scale=...): on one 256x512 pair of the unchanged
# cfgs/casnet/casnet_psm_sceneflow.yaml the un-sharpened classif3 logit std of stages 1 / 2 is 0.035 / 0.046 (CasPSMNet) and
# 0.102 / 0.131 (CasGwcNet built from the same MODEL section); these bring both stages to ~4.
CASNET_SCALE = {"cost_agg.0.classif3.2.weight": 114.0, "cost_agg.1.classif3.2.weight": 87.0}
CASGWC_SCALE = {"cost_agg.0.classif3.2.weight": 39.0, "cost_agg.1.classif3.2.weight": 28.0}


def _sample_grid(height, width, disp, ndisp, like):
    """(B, D, H, W, 2) grid_sample grid of a column shift by `disp` and the (B, D, H, W) column index it was built from."""
    bs = disp.shape[0]
    rows, cols = torch.meshgrid([torch.arange(0, height, dtype=like.dtype, device=like.device),
                                 torch.arange(0, width, dtype=like.dtype, device=like.device)])
    rows = rows.reshape(1, 1, height, width).repeat(bs, ndisp, 1, 1)
    cols = cols.reshape(1, 1, height, width).repeat(bs, ndisp, 1, 1)
    gx = (cols - disp) / ((width - 1.0) / 2.0) - 1.0
    gy = rows / ((height - 1.0) / 2.0) - 1.0
    return torch.stack([gx, gy], dim=4), cols


def _warp(y, grid, ndisp):
    bs, channels, height, width = y.size()
    return F.grid_sample(y, grid.view(bs, ndisp * height, width, 2), mode='bilinear', padding_mode='zeros',
                         align_corners=True).view(bs, channels, ndisp, height, width)


def warped_concat_volume(x, y, disp, ndisp):
    """(B, 2C, D, H, W): [x repeated over D (unmasked) | y warped to column w - disp]."""
    bs, channels, height, width = x.size()
    volume = x.new().resize_(bs, channels * 2, ndisp, height, width).zero_()
    grid, _ = _sample_grid(height, width, disp, ndisp, x)
    volume[:, x.size()[1]:, :, :, :] = _warp(y, grid, ndisp)
    volume[:, :x.size()[1], :, :, :] = x.unsqueeze(2).repeat(1, 1, ndisp, 1, 1)
    return volume


def _masked_pair(x, y, disp, ndisp):
    """(x repeated over D and zeroed where w < disp, y warped), both (B, C, D, H, W)."""
    height, width = y.shape[2], y.shape[3]
    grid, cols = _sample_grid(height, width, disp, ndisp, x)
    yw = _warp(y, grid, ndisp)
    xw = x.unsqueeze(2).repeat(1, 1, ndisp, 1, 1).transpose(0, 1)
    xw[:, cols < disp] = 0
    return xw.transpose(0, 1), yw


def warped_gwc_concat_volume(features_left, features_right, disp, ndisp, num_groups):
    """(B, G + 2*Cc, D, H, W): [group-wise mean of x_warped * y_warped | x_warped | y_warped]."""
    x, y = features_left["gwc_feature"], features_right["gwc_feature"]
    bs, channels, height, width = x.size()
    xw, yw = _masked_pair(x, y, disp, ndisp)
    gwc = (xw * yw).view([bs, num_groups, channels // num_groups, ndisp, height, width]).mean(dim=2)
    x, y = features_left["concat_feature"], features_right["concat_feature"]
    bs, channels, height, width = x.size()
    concat = x.new().resize_(bs, channels * 2, ndisp, height, width).zero_()
    xw, yw = _masked_pair(x, y, disp, ndisp)
    concat[:, x.size()[1]:, :, :, :] = yw
    concat[:, :x.size()[1], :, :, :] = xw
    return torch.cat((gwc, concat), 1)


def upsample_softargmin_values(cost3, fine_d, fine_h, fine_w, disp_values):
    """(B, 1, D', H', W') logits -> (B, H, W) disparity."""
    cost3 = F.interpolate(cost3, [fine_d, fine_h, fine_w], mode='trilinear', align_corners=False)
    cost3 = torch.squeeze(cost3, 1)
    return disparity_regression_values(F.softmax(cost3, dim=1), disp_values)


def _head(c):
    return nn.Sequential(_gwc_cb(c, c, 3, 1, 1), nn.ReLU(inplace=True), nn.Conv3d(c, 1, kernel_size=3, padding=1, stride=1, bias=False))


class CostAggregation(nn.Module):
    """Same state_dict keys as the reference's CostAggregation(in_channels, base_channels); eval forward only."""

    def __init__(self, in_channels, base_channels=32):
        super().__init__()
        c = base_channels
        self.dres0 = nn.Sequential(_gwc_cb(in_channels, c, 3, 1, 1), nn.ReLU(inplace=True), _gwc_cb(c, c, 3, 1, 1),
                                   nn.ReLU(inplace=True))
        self.dres1 = nn.Sequential(_gwc_cb(c, c, 3, 1, 1), nn.ReLU(inplace=True), _gwc_cb(c, c, 3, 1, 1))
        self.dres2, self.dres3, self.dres4 = GwcHourglass(c), GwcHourglass(c), GwcHourglass(c)
        self.classif0, self.classif1, self.classif2, self.classif3 = _head(c), _head(c), _head(c), _head(c)

    def logits(self, cost):
        cost0 = self.dres0(cost)
        cost0 = self.dres1(cost0) + cost0
        out3 = self.dres4(self.dres3(self.dres2(cost0)))
        return self.classif3(out3)

    def forward(self, cost, fine_d, fine_h, fine_w, disp_range_samples):
        return upsample_softargmin_values(self.logits(cost), fine_d, fine_h, fine_w, disp_range_samples)
