"""Oracle: CoEx's attention cost volume, 3D aggregation and regression tail (TEST INFRASTRUCTURE -- see oracle/__init__.py).

* ``attention_volume``  AttentionCostVolume after its convolutions, last plane dropped
                        stereo/modeling/models/coex/coex_cost_processor.py:53-65,230 (CostVolume :10-35)
* ``Aggregation``       eval forward of ``Aggregation``, same state_dict keys     coex_cost_processor.py:68-237
                        (``BasicConv`` coex/submodule.py, ``channelAtt`` coex_cost_processor.py:68-80)
* ``nearest_index``     aten's source index of F.interpolate(mode='nearest') along one dimension (the resampling at :219-224)
* ``regression``        ``Regression.forward`` (eval) with ``upfeat``             coex/coex_disp_processor.py:8-65

Same aten calls in the same order as the reference, on fp32 CPU tensors; bit-equality is asserted by tools/make_golden.py and
tests/test_coex_cpu.py.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .cost_volume import coex_cost_volume

# seeded_state_dict needs no sharpening factor for CoEx: the top-k pooling picks indices whatever the logit scale, and one
# 256x512 pair of the unchanged cfgs/coex/coex_sceneflow_amp.yaml with seed 1 gives a disparity std of 16 px.


def attention_volume(x, y, maxdisp_lowres, head=1):
    """x, y: the desc outputs (B, C, H, W) -> (B, head, maxdisp_lowres, H, W)."""
    xn = x / torch.norm(x, 2, 1, True)
    yn = y / torch.norm(y, 2, 1, True)
    return coex_cost_volume(xn, yn, maxdisp_lowres, head)[:, :, :-1, :, :]


def nearest_index(out_size, in_size):
    """Source index of every output position of F.interpolate(mode='nearest') along one dimension (aten nearest_idx)."""
    if in_size == out_size:
        return list(range(out_size))
    if out_size == 2 * in_size:
        return [i >> 1 for i in range(out_size)]
    scale = np.float32(in_size) / np.float32(out_size)
    return [min(int(np.floor(np.float32(i) * scale)), in_size - 1) for i in range(out_size)]


def topk_pool(cost, k, stable=False):
    """Top k logits along D and their indices.  The reference's cost.sort(2, True) keeps exact ties in index order only while
    D <= 16 (aten's CPU sort falls back to insertion sort there); beyond that the order of equal values is the introsort's.
    stable=True gives the lower-index-first order at every D, the order the CUDA kernel implements."""
    _, ind = cost.sort(dim=2, descending=True, stable=True) if stable else cost.sort(2, True)
    ind = ind[:, :, :k]
    return torch.gather(cost, 2, ind), ind


def upfeat(disp4, prob, up_h=4, up_w=4):
    b, _, h, w = disp4.shape
    feat = F.unfold(disp4, 3, 1, 1).reshape(b, -1, h, w)
    feat = F.interpolate(feat, (h * up_h, w * up_w), mode='nearest').reshape(b, -1, 9, h * up_h, w * up_w)
    return (feat * prob.unsqueeze(1)).sum(2)


def regression(cost, spx, top_k, stable=False):
    """cost (B, 1, D, h, w) logits, spx (B, 9, 4h, 4w) probabilities -> (B, 4h, 4w) disparity; 2 <= top_k."""
    b = spx.shape[0]
    corr, ind = topk_pool(cost, top_k, stable)
    corr = F.softmax(corr, 2)
    disp4 = torch.sum(corr * ind, 2, keepdim=True)
    disp4 = disp4.reshape(b, 1, disp4.shape[-2], disp4.shape[-1])
    return upfeat(disp4, spx, 4, 4).squeeze(1) * 4


# ---------------------------------------------------------------------------------------------------------- aggregation
class BasicConv(nn.Module):
    """conv -> BN (when bn) -> LeakyReLU(0.01) (when relu); the BN module exists either way, as in the reference."""

    def __init__(self, cin, cout, deconv=False, is_3d=True, bn=True, relu=True, **kw):
        super().__init__()
        kind = {(True, True): nn.ConvTranspose3d, (False, True): nn.Conv3d, (True, False): nn.ConvTranspose2d,
                (False, False): nn.Conv2d}[(deconv, is_3d)]
        self.relu, self.use_bn = relu, bn
        self.conv = kind(cin, cout, bias=False, **kw)
        self.bn = nn.BatchNorm3d(cout) if is_3d else nn.BatchNorm2d(cout)
        self.LeakyReLU = nn.LeakyReLU()

    def forward(self, x):
        x = self.conv(x)
        x = self.bn(x) if self.use_bn else x
        return self.LeakyReLU(x) if self.relu else x


class ChannelAtt(nn.Module):
    """cv * sigmoid(1x1 conv(LeakyReLU(BN(1x1 conv(im))))) broadcast over D."""

    def __init__(self, cv_chan, im_chan):
        super().__init__()
        self.im_att = nn.Sequential(BasicConv(im_chan, im_chan // 2, is_3d=False, kernel_size=1, stride=1, padding=0),
                                    nn.Conv2d(im_chan // 2, cv_chan, 1))

    def forward(self, cv, im):
        return torch.sigmoid(self.im_att(im).unsqueeze(2)) * cv


class Aggregation(nn.Module):
    """CoEx's Aggregation with disparity stride 2 (the only stride the engine serves); eval forward only."""

    def __init__(self, max_disparity=192, matching_head=1, gce=True, channels=(16, 32, 48), blocks_num=(2, 2, 2),
                 spixel_branch_channels=(32, 48), im_chans=(16, 24, 32, 96, 160)):
        super().__init__()
        self.D = int(max_disparity // 4)
        self.gce = gce
        ch = [8] + list(channels)
        self.conv_stem = BasicConv(matching_head, 8, kernel_size=3, stride=1, padding=1)
        if gce:
            self.channelAttStem = ChannelAtt(8, 2 * im_chans[1] + spixel_branch_channels[1])
            self.channelAtt = nn.ModuleList()
            self.channelAttDown = nn.ModuleList()
        self.conv_down, self.conv_up, self.conv_skip, self.conv_agg = nn.ModuleList(), nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        for i in range(3):
            self.conv_down.append(nn.Sequential(*[BasicConv(ch[i] if n == 0 else ch[i + 1], ch[i + 1], kernel_size=3, padding=1,
                                                            stride=2 if n == 0 else 1) for n in range(blocks_num[i])]))
            if gce:
                self.channelAttDown.append(ChannelAtt(ch[i + 1], (1 if i == 2 else 2) * im_chans[i + 2]))
            last = i == 0
            self.conv_up.append(BasicConv(ch[i + 1], 1 if last else ch[i], deconv=True, bn=not last, relu=not last, kernel_size=4,
                                          padding=1, stride=2))
            self.conv_agg.append(nn.Sequential(BasicConv(ch[i], ch[i], kernel_size=3, padding=1, stride=1),
                                               BasicConv(ch[i], ch[i], kernel_size=3, padding=1, stride=1)))
            self.conv_skip.append(BasicConv(2 * ch[i], ch[i], kernel_size=1, padding=0, stride=1))
            if gce:
                self.channelAtt.append(ChannelAtt(ch[i], 2 * im_chans[i + 1]))

    def forward(self, img, cost):
        b, _, h, w = img[0].shape
        cost = self.conv_stem(cost.reshape(b, -1, self.D, h, w))
        if self.gce:
            cost = self.channelAttStem(cost, img[0])
        levels = [cost]
        for i in range(3):
            cost = self.conv_down[i](cost)
            if self.gce:
                cost = self.channelAttDown[i](cost, img[i + 1])
            levels.append(cost)
        for i in range(3):
            j = 2 - i                                            # conv_up[-i-1], skip level levels[-i-2]
            cost = self.conv_up[j](cost)
            skip = levels[j]
            if cost.shape != skip.shape:
                cost = F.interpolate(cost, size=tuple(skip.shape[-3:]), mode='nearest')
            if i == 2:
                break
            cost = self.conv_agg[j](self.conv_skip[j](torch.cat([cost, skip], 1)))
            if self.gce:
                cost = self.channelAtt[j](cost, img[-i - 2])
        return cost
