"""Host-side mirrors of the reference model classes for the hot path (GwcNet, PSMNet).

Same constructor arguments (a cfg object with MAX_DISP / USE_CONCAT_VOLUME / ...), same
``forward(inputs: dict) -> {'disp_pred': ...}`` contract (docs/4.how_to_create_your_model.md:8-23)
and the SAME state_dict keys as stereo/modeling/models/gwcnet/gwcnet.py:11-39 and
stereo/modeling/models/psmnet/psmnet.py:10-29, so an unchanged reference checkpoint loads with
``load_state_dict``.  They exist because the reference package itself is not importable on a
machine without easydict/timm (SURVEY.md section 8c); where it IS importable, use
``openstereo_b200.patch.patch(reference_model)`` instead and nothing here is needed.

Division of labour: the 2D feature extractors are out of the kernel scope (SURVEY.md section 2.1
row 12) and stay torch.nn/cuDNN -- except their 1/2-resolution front (eight 32->32 3x3 convs), which
reuses the wgmma conv kernel when the input is 256 rows high (_front_tc), and the residual stages, whose
3x3 convs (the stride-2 stage entry included) run on it when the 1/4-resolution map is 128 wide (_stage_tc); everything from the cost
volume to the disparity map runs in the sm_90a kernels through the engines of aggregation.py.  The 3D modules below are PARAMETER
CONTAINERS: they are never called, only read by the engines.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import aggregation as _agg
from . import ops
from .aggregation import GwcAggregation, PSMAggregation


USE_TC_BACKBONE = True      # the 2D extractor's 3x3 residual blocks on the wgmma kernels (False: everything 2D stays cuDNN)


def _cfg_get(cfgs, key, default=None):
    if isinstance(cfgs, dict):
        return cfgs.get(key, default)
    return getattr(cfgs, key, default)


# ------------------------------------------------------------------------------------------- 2D backbones (cuDNN)
def _cb(cin, cout, k, stride, pad, dilation, bias=False):
    return nn.Sequential(nn.Conv2d(cin, cout, kernel_size=k, stride=stride, padding=dilation if dilation > 1 else pad,
                                   dilation=dilation, bias=bias), nn.BatchNorm2d(cout))


def _front_tc_ok(net, x):
    """The 1/2-resolution front of the backbone (firstconv[1:], layer1: eight 32->32 3x3 convs, where cuDNN's best fp32
    kernel reaches ~8 TFLOP/s) can run on the wgmma conv kernel when the half-resolution HEIGHT is the 128-voxel M tile:
    a 2D conv commutes with transposing the image, so the kernel sees (rows = W/2, columns = H/2 = 128) and the 3x3 weights
    with kh/kw swapped, as a one-plane 3D conv (the kd != 1 phases are skipped for D = 1)."""
    return (getattr(net, "_osb_folded", False) and x.is_cuda and x.dim() == 4 and x.shape[2] == 2 * ops.TC_WIDTH and x.shape[3] % 2 == 0
            and _agg.USE_TENSOR_CORES and USE_TC_BACKBONE and x.dtype == torch.float32 and ops.conv3d_tc_kc(32, 32, ops.TC_WIDTH) == 32)


def _front_tc(net, x, nhwc=False):
    """firstconv + layer1 -> (B, 32, H/2, W/2) NCHW, or with nhwc=True the (B, H/2, W/2, 32) channels-last view of the last
    epilogue's (B, W/2, H/2 = 128, 32) output, which layer2 reads without a layout change (_stage_tc)."""
    convs = [m for m in net.firstconv.modules() if isinstance(m, nn.Conv2d)]
    blocks = list(net.layer1.children())
    y = F.relu(convs[0](x))                                                      # 3 -> 32, stride 2: stays cuDNN
    t = y.permute(0, 3, 2, 1).contiguous()                                       # (B, W/2, H/2 = 128, 32) channels-last
    t = _tc2d(net, convs[2], _tc2d(net, convs[1], t, ops.ACT_RELU, transpose=True), ops.ACT_RELU, transpose=True)
    for i, blk in enumerate(blocks):                                             # conv-bn-relu, conv-bn, += identity
        c1, c2 = _block_convs(blk)
        assert blk.downsample is None
        t = _tc2d(net, c2, _tc2d(net, c1, t, ops.ACT_RELU, transpose=True), ops.ACT_NONE, residual=t,
                  last=(i == len(blocks) - 1 and not nhwc), transpose=True)
    return t.transpose(1, 2) if nhwc else t.transpose(2, 3).contiguous()          # (B, 32, W/2, 128) -> (B, 32, 128, W/2)


def _front(net, x):
    """firstconv + layer1 -> (NCHW output, possibly a view; its channels-last view when the tensor-core front ran, else None)."""
    if not _front_tc_ok(net, x):
        return net.layer1(net.firstconv(x)), None
    t = _front_tc(net, x, nhwc=True)
    return t.permute(0, 3, 1, 2), t


def _tc2d(net, conv, t, act, residual=None, last=False, transpose=False, res_nhwc=True):
    """One BN-folded 3x3 Conv2d (stride 1 with dilation 1 or 2, or stride 2) on the wgmma kernels: t (B, rows, cols, Cin)
    channels-last with 128 OUTPUT columns; stride 2 runs as a one-plane stride-2 conv."""
    cache = net.__dict__.setdefault("_osb_tc2d", {})
    dil, s = conv.dilation[0], conv.stride[0]
    if id(conv) not in cache:
        assert conv.kernel_size == (3, 3) and conv.padding == (dil, dil) and conv.dilation == (dil, dil) and conv.stride == (s, s)
        assert s == 1 or (s == 2 and dil == 1 and not transpose)
        w5 = torch.zeros(conv.out_channels, conv.in_channels, 3, 3, 3, dtype=torch.float32, device=conv.weight.device)
        w2 = conv.weight.detach().float()
        w5[:, :, 1] = w2.transpose(2, 3) if transpose else w2                   # image transposed -> taps transposed
        if s == 2:
            wp = ops.pack_tc_weight(w5, 16, kw_order=(1, 0, 2))
        else:
            wp = ops.pack_tc_weight(w5, ops.conv2d_tc_kc(conv.in_channels, conv.out_channels, ops.TC_WIDTH, dil))
        cache[id(conv)] = (wp, None if conv.bias is None else conv.bias.detach().float().contiguous())
    wp, bias = cache[id(conv)]
    if s == 2:                                                                   # a stage entry's conv1: channels-last out
        assert residual is None and not last
        return ops.conv3d_k3_s2_tc(t.unsqueeze(1), wp, None, bias, None, act, out_ndhwc=True).squeeze(1)
    return ops.conv2d_k3_tc(t, wp, None, bias, residual, act, dil, out_nhwc=not last, res_nhwc=res_nhwc)


def _block_convs(blk):
    c1 = [m for m in blk.conv1.modules() if isinstance(m, nn.Conv2d)][0]
    c2 = [m for m in blk.conv2.modules() if isinstance(m, nn.Conv2d)][0]
    return c1, c2


def _block_tc_ok(blk, c):
    """An identity-shortcut BasicBlock whose two 3x3 convs (same dilation, c -> c channels) have a tensor-core kernel."""
    if blk.downsample is not None:
        return False
    c1, c2 = _block_convs(blk)
    dil = c1.dilation[0]
    return all(cv.kernel_size == (3, 3) and cv.stride == (1, 1) and cv.dilation == (dil, dil) and cv.padding == (dil, dil)
               and cv.in_channels == c and cv.out_channels == c for cv in (c1, c2)) and ops.conv2d_tc_kc(c, c, ops.TC_WIDTH, dil) != 0


def _downsample_conv(blk):
    """The 1x1 conv that is a BN-folded block's whole downsample branch, None for any other branch."""
    mods = [] if blk.downsample is None else [m for m in blk.downsample.modules() if not isinstance(m, nn.Sequential)]
    return mods[0] if len(mods) == 1 and isinstance(mods[0], nn.Conv2d) else None


def _entry_tc_ok(blk, c, h, w):
    """A stage's first block that changes stride or channels (c -> cout, input h x w): 3x3 conv1 (stride 1 or 2, dilation 1), 3x3
    conv2 (cout -> cout) and a 1x1 downsample of the same stride, where the output is 128 columns wide and both 3x3 convs have a
    tensor-core kernel (stride 2: the one-plane stride-2 conv, which needs even h and w)."""
    c1, c2 = _block_convs(blk)
    ds = _downsample_conv(blk)
    s, cout = c1.stride[0], c1.out_channels
    if ds is None or s not in (1, 2) or w != s * ops.TC_WIDTH:
        return False
    if not (ds.kernel_size == (1, 1) and ds.stride == (s, s) and ds.padding == (0, 0) and ds.groups == 1
            and ds.in_channels == c and ds.out_channels == cout):
        return False
    if not all(cv.kernel_size == (3, 3) and cv.dilation == (1, 1) and cv.padding == (1, 1) and cv.groups == 1 and cv.out_channels == cout
               for cv in (c1, c2)) or c1.stride != (s, s) or c1.in_channels != c or c2.stride != (1, 1) or c2.in_channels != cout:
        return False
    conv1_ok = ops.conv3d_s2_tc_supported(c, cout, 1, h, w) if s == 2 else ops.conv2d_tc_kc(c, cout, ops.TC_WIDTH, 1) != 0
    return conv1_ok and ops.conv2d_tc_kc(cout, cout, ops.TC_WIDTH, 1) != 0


def _entry_tc(net, blk, x, t, last):
    """An _entry_tc_ok block: conv1 + ReLU channels-last on the wgmma kernels from t (B, H, W, C); the downsample on the fp32 1x1
    kernel from x, the same input as NCHW (a view is fine: only the rows and columns it reads are copied); conv2 adds it in its
    epilogue."""
    c1, c2 = _block_convs(blk)
    ds = _downsample_conv(blk)
    cache = net.__dict__.setdefault("_osb_tc2d", {})
    if id(ds) not in cache:
        cache[id(ds)] = (ops.pack_conv_weight(ds.weight.unsqueeze(2)), None if ds.bias is None else ds.bias.detach().float().contiguous())
    wp, bias = cache[id(ds)]
    r = ops.conv3d_1x1(x[:, :, ::2, ::2].contiguous() if ds.stride[0] == 2 else x.contiguous(), wp, None, bias)   # (B, Cout, H', 128)
    return _tc2d(net, c2, _tc2d(net, c1, t, ops.ACT_RELU), ops.ACT_NONE, residual=r, last=last, res_nhwc=False)


def _stage_tc(net, stage, x, t=None, nhwc_out=False):
    """A residual stage (layer2 / layer3 / the dilated layer4 of the PSMNet-style extractor: gwcnet_backbone.py:38-60) on a
    feature map 128 columns wide at its output.  x: the NCHW input (a view is fine); t: the same input channels-last (B, H, W, C)
    when the layers before ran on the wgmma kernels, else None.  Returns (NCHW output, its channels-last copy or None).
    The identity-shortcut 3x3 blocks run on the wgmma kernels, channels-last in between.  The first block runs there too when it
    has an identity shortcut, or -- on a channels-last input -- as an _entry_tc block; a stage fed NCHW by cuDNN layers keeps
    its entry block on cuDNN.  With nhwc_out a stage that got a channels-last input hands one on: the last epilogue writes it and
    the NCHW output is its transpose; otherwise the last epilogue writes NCHW.  Any block without a kernel variant keeps the
    stage on the module's own layers (cuDNN)."""
    blocks = list(stage.children())
    usable = getattr(net, "_osb_folded", False) and x.is_cuda and x.dtype == torch.float32 and _agg.USE_TENSOR_CORES and USE_TC_BACKBONE
    c, h, w = x.shape[1:]
    entry = usable and t is not None and _entry_tc_ok(blocks[0], c, h, w)
    if entry:
        c = _block_convs(blocks[0])[1].out_channels
    elif not (usable and w == ops.TC_WIDTH and _block_tc_ok(blocks[0], c)):
        x, t = blocks[0](x.contiguous()), None
        blocks, c, w = blocks[1:], x.shape[1], x.shape[3]
    if not (usable and blocks and (entry or w == ops.TC_WIDTH) and all(_block_tc_ok(blk, c) for blk in blocks[entry:])):
        y = x.contiguous()
        for blk in blocks:
            y = blk(y)
        return y, None
    keep = nhwc_out and t is not None
    t = t.contiguous() if t is not None else ops.to_ndhwc(x.unsqueeze(2).contiguous()).squeeze(1)   # (B, H, W, C)
    for i, blk in enumerate(blocks):
        last = i == len(blocks) - 1 and not keep
        if i == 0 and entry:
            t = _entry_tc(net, blk, x, t, last)
        else:
            c1, c2 = _block_convs(blk)
            t = _tc2d(net, c2, _tc2d(net, c1, t, ops.ACT_RELU), ops.ACT_NONE, residual=t, last=last)
    return (t.permute(0, 3, 1, 2).contiguous(), t) if keep else (t, None)       # NCHW (B, C, H, 128)


def _lastconv_tc_ok(net, x):
    """lastconv = conv3x3(320->128)+BN+ReLU, conv1x1(128->12) (gwcnet_backbone.py:62-67): cuDNN picks an FFT algorithm for the
    320-channel 3x3 (2.1 ms); on the wgmma kernel it is the layer3 conv with 20 K chunks."""
    convs = [m for m in net.lastconv.modules() if isinstance(m, nn.Conv2d)]
    return (getattr(net, "_osb_folded", False) and x.is_cuda and x.dtype == torch.float32 and _agg.USE_TENSOR_CORES and USE_TC_BACKBONE
            and x.shape[3] == ops.TC_WIDTH and len(convs) == 2 and convs[0].kernel_size == (3, 3) and convs[0].stride == (1, 1)
            and convs[0].dilation == (1, 1) and convs[0].padding == (1, 1) and convs[1].kernel_size == (1, 1)
            and ops.conv2d_tc_kc(convs[0].in_channels, convs[0].out_channels, ops.TC_WIDTH, 1) != 0)


def _lastconv_tc(net, x):
    convs = [m for m in net.lastconv.modules() if isinstance(m, nn.Conv2d)]
    t = ops.to_ndhwc(x.unsqueeze(2).contiguous()).squeeze(1)                      # (B, H, 128, 320)
    return convs[1](_tc2d(net, convs[0], t, ops.ACT_RELU, last=True))             # 3x3 + ReLU on tensor cores, 1x1 on cuDNN


def gwc_extract(net, x):
    """feature_extraction.forward of gwcnet_backbone.py:80-93 on any module with its attribute names (this file's mirror or a
    BN-folded copy of the reference's own class): identical graph, the 3x3 residual blocks on the wgmma kernels where a
    variant serves the shape, everything else through the module's own layers (cuDNN)."""
    l2, t = _stage_tc(net, net.layer2, *_front(net, x), nhwc_out=True)
    l3, t = _stage_tc(net, net.layer3, l2, t, nhwc_out=True)
    l4, _ = _stage_tc(net, net.layer4, l3, t)
    gwc = torch.cat((l2, l3, l4), dim=1)
    out = {"gwc_feature": gwc}
    if net.concat_feature:
        out["concat_feature"] = _lastconv_tc(net, gwc) if _lastconv_tc_ok(net, gwc) else net.lastconv(gwc)
    return out


def psm_extract(net, x):
    """PSMNet._forward of psmnet_backbone.py:82-116 on any module with its attribute names (see gwc_extract)."""
    o4_0, t = _stage_tc(net, net.layer2, *_front(net, x), nhwc_out=True)
    o8, _ = _stage_tc(net, net.layer4, *_stage_tc(net, net.layer3, o4_0, t, nhwc_out=True))
    size = (o8.size()[2], o8.size()[3])
    up = [F.interpolate(getattr(net, "branch%d" % i)(o8), size, mode="bilinear", align_corners=True) for i in (1, 2, 3, 4)]
    cat = torch.cat((o4_0, o8, up[3], up[2], up[1], up[0]), 1)
    return _lastconv_tc(net, cat) if _lastconv_tc_ok(net, cat) else net.lastconv(cat)


class _ResBlock(nn.Module):
    """conv-bn-relu, conv-bn, += identity (no trailing relu): gwcnet_backbone.py:13-35, psmnet/submodule.py:219-243."""

    def __init__(self, conv1, conv2, downsample):
        super().__init__()
        self.conv1, self.conv2, self.downsample = conv1, conv2, downsample

    def forward(self, x):
        out = self.conv2(self.conv1(x))
        if self.downsample is not None:
            x = self.downsample(x)
        out += x
        return out


def _stage(make_block, make_down, inplanes, planes, blocks, stride):
    down = make_down(inplanes, planes, stride) if (stride != 1 or inplanes != planes) else None
    layers = [make_block(inplanes, planes, stride, down)]
    layers += [make_block(planes, planes, 1, None) for _ in range(1, blocks)]
    return nn.Sequential(*layers)


class _GwcFeatureExtraction(nn.Module):
    def __init__(self, concat_feature, concat_channels):
        super().__init__()
        self.concat_feature = concat_feature
        r = lambda: nn.ReLU(inplace=True)
        self.firstconv = nn.Sequential(_cb(3, 32, 3, 2, 1, 1), r(), _cb(32, 32, 3, 1, 1, 1), r(), _cb(32, 32, 3, 1, 1, 1), r())

        def block(dil):
            return lambda i, o, s, d: _ResBlock(nn.Sequential(_cb(i, o, 3, s, 1, dil), r()), _cb(o, o, 3, 1, 1, dil), d)

        down = lambda i, o, s: nn.Sequential(nn.Conv2d(i, o, kernel_size=1, stride=s, bias=False), nn.BatchNorm2d(o))
        self.layer1 = _stage(block(1), down, 32, 32, 3, 1)
        self.layer2 = _stage(block(1), down, 32, 64, 16, 2)
        self.layer3 = _stage(block(1), down, 64, 128, 3, 1)
        self.layer4 = _stage(block(2), down, 128, 128, 3, 1)
        if concat_feature:
            self.lastconv = nn.Sequential(_cb(320, 128, 3, 1, 1, 1), r(),
                                          nn.Conv2d(128, concat_channels, kernel_size=1, padding=0, stride=1, bias=False))

    def forward(self, x):
        return gwc_extract(self, x)


def _fold_conv_bn(module):
    """Copy of a 2D feature extractor with every eval-mode Conv2d+BatchNorm2d pair folded into one conv (the BN affine is
    absorbed into the weights/bias), so cuDNN runs one kernel where PyTorch would run conv, batch_norm as two.  The
    original module keeps the parameters (state_dict unchanged); the folded copy is runtime-only."""
    import copy
    from torch.nn.utils.fusion import fuse_conv_bn_eval
    inst_fwd = module.__dict__.pop("forward", None)              # a patch()-installed per-instance forward is not part of the net
    try:
        fused = copy.deepcopy(module).eval()
    finally:
        if inst_fwd is not None:
            module.__dict__["forward"] = inst_fwd

    def walk(m):
        for name, child in list(m.named_children()):
            if isinstance(child, nn.Sequential):
                mods = list(child.children())
                out, i = [], 0
                while i < len(mods):
                    if i + 1 < len(mods) and isinstance(mods[i], nn.Conv2d) and isinstance(mods[i + 1], nn.BatchNorm2d):
                        out.append(fuse_conv_bn_eval(mods[i], mods[i + 1]))
                        i += 2
                    else:
                        out.append(mods[i])
                        i += 1
                new = nn.Sequential(*out)
                setattr(m, name, new)
                walk(new)
            else:
                walk(child)
    walk(fused)
    for q in fused.parameters():
        q.requires_grad_(False)
    fused._osb_folded = not any(isinstance(m, nn.BatchNorm2d) for m in fused.modules())   # every BN absorbed: convs carry the affine
    return fused


class _FoldedRuntime:
    """Lazily (re)built BN-folded twin of a backbone; rebuilt when a parameter/buffer changes or moves."""

    def __init__(self, module):
        self.module, self.stamp, self.fused = module, None, None

    def get(self):
        m = self.module
        stamp = tuple((t._version, t.data_ptr()) for t in list(m.parameters()) + list(m.buffers()))
        if stamp != self.stamp:
            with torch.no_grad():
                self.fused = _fold_conv_bn(m)
            self.stamp = stamp
        return self.fused


class _GwcBackbone(nn.Module):
    def __init__(self, use_concat_volume, concat_channels):
        super().__init__()
        self.feature_extraction = _GwcFeatureExtraction(use_concat_volume, concat_channels)
        self._rt = None

    def forward(self, inputs):
        if self._rt is None:
            self._rt = _FoldedRuntime(self.feature_extraction)
        fe = self.feature_extraction if self.training else self._rt.get()
        # left and right share weights: one batched pass (B*2) instead of two (gwcnet_backbone.py:101-107)
        both = fe(torch.cat((inputs["left"], inputs["right"]), 0))
        b = inputs["left"].shape[0]
        return {"ref_feature": {k: v[:b] for k, v in both.items()}, "tgt_feature": {k: v[b:] for k, v in both.items()}}


class _PsmBackbone(nn.Module):
    def __init__(self):
        super().__init__()
        cbr = lambda i, o, k, s, p, d: nn.Sequential(*_cb(i, o, k, s, p, d), nn.ReLU(inplace=True))
        self.firstconv = nn.Sequential(cbr(3, 32, 3, 2, 1, 1), cbr(32, 32, 3, 1, 1, 1), cbr(32, 32, 3, 1, 1, 1))

        def block(pad, dil):
            return lambda i, o, s, d: _ResBlock(cbr(i, o, 3, s, pad, dil), _cb(o, o, 3, 1, pad, dil), d)

        down = lambda i, o, s: _cb(i, o, 1, s, 0, 1, bias=True)          # conv_bn default bias=True (psmnet_backbone.py:68-71)
        self.layer1 = _stage(block(1, 1), down, 32, 32, 3, 1)
        self.layer2 = _stage(block(1, 1), down, 32, 64, 16, 2)
        self.layer3 = _stage(block(1, 1), down, 64, 128, 3, 1)
        self.layer4 = _stage(block(2, 2), down, 128, 128, 3, 1)
        for i, k in zip((1, 2, 3, 4), (64, 32, 16, 8)):
            setattr(self, "branch%d" % i, nn.Sequential(nn.AvgPool2d((k, k), stride=(k, k)), cbr(128, 32, 1, 1, 0, 1)))
        self.lastconv = nn.Sequential(cbr(320, 128, 3, 1, 1, 1),
                                      nn.Conv2d(128, 32, kernel_size=1, padding=0, stride=1, dilation=1, bias=False))

    def _forward(self, x):
        return psm_extract(self, x)

    def forward(self, inputs):
        if getattr(self, "_rt", None) is None:
            object.__setattr__(self, "_rt", _FoldedRuntime(self))
        net = self if self.training else self._rt.get()
        both = psm_extract(net, torch.cat((inputs["left"], inputs["right"]), 0))
        b = inputs["left"].shape[0]
        return {"ref_feature": both[:b], "tgt_feature": both[b:]}


# ------------------------------------------------------------------------------ 3D parameter containers (never called)
def _cb3(cin, cout, k, s, p):
    return nn.Sequential(nn.Conv3d(cin, cout, kernel_size=k, stride=s, padding=p, bias=False), nn.BatchNorm3d(cout))


def _db3(cin, cout):
    return nn.Sequential(nn.ConvTranspose3d(cin, cout, 3, padding=1, output_padding=1, stride=2, bias=False), nn.BatchNorm3d(cout))


class _GwcHourglassParams(nn.Module):
    def __init__(self, c):
        super().__init__()
        r = lambda: nn.ReLU(inplace=True)
        self.conv1 = nn.Sequential(_cb3(c, 2 * c, 3, 2, 1), r())
        self.conv2 = nn.Sequential(_cb3(2 * c, 2 * c, 3, 1, 1), r())
        self.conv3 = nn.Sequential(_cb3(2 * c, 4 * c, 3, 2, 1), r())
        self.conv4 = nn.Sequential(_cb3(4 * c, 4 * c, 3, 1, 1), r())
        self.conv5, self.conv6 = _db3(4 * c, 2 * c), _db3(2 * c, c)
        self.redir1, self.redir2 = _cb3(c, c, 1, 1, 0), _cb3(2 * c, 2 * c, 1, 1, 0)


class GwcVolumeCostProcessor(nn.Module):
    """gwcnet_cost_processor.py:5-68 -- both volumes and the concat in one kernel launch."""

    def __init__(self, maxdisp=192, downsample=4, num_groups=40, use_concat_volume=True, *args, **kwargs):
        super().__init__()
        self.maxdisp, self.downsample, self.num_groups, self.use_concat_volume = maxdisp, downsample, num_groups, use_concat_volume

    def forward(self, inputs):
        lf, rf = inputs["ref_feature"], inputs["tgt_feature"]
        d = self.maxdisp // self.downsample
        if self.use_concat_volume:
            vol = ops.gwc_concat_volume(lf["gwc_feature"], rf["gwc_feature"], lf["concat_feature"], rf["concat_feature"],
                                        d, self.num_groups)
        else:
            vol = ops.build_gwc_volume(lf["gwc_feature"], rf["gwc_feature"], d, self.num_groups)
        return {"cost_volume": vol}


class GwcDispProcessor(nn.Module):
    """gwcnet_disp_processor.py:29-140 (inference branch); parameters under the reference's names."""

    def __init__(self, maxdisp=192, downsample=4, num_groups=40, use_concat_volume=True, concat_channels=12, *args, **kwargs):
        super().__init__()
        self.maxdisp = maxdisp
        cin = num_groups + (2 * concat_channels if use_concat_volume else 0)
        r = lambda: nn.ReLU(inplace=True)
        self.dres0 = nn.Sequential(_cb3(cin, 32, 3, 1, 1), r(), _cb3(32, 32, 3, 1, 1), r())
        self.dres1 = nn.Sequential(_cb3(32, 32, 3, 1, 1), r(), _cb3(32, 32, 3, 1, 1))
        self.dres2, self.dres3, self.dres4 = _GwcHourglassParams(32), _GwcHourglassParams(32), _GwcHourglassParams(32)
        for i in range(4):
            setattr(self, "classif%d" % i, nn.Sequential(_cb3(32, 32, 3, 1, 1), r(),
                                                         nn.Conv3d(32, 1, kernel_size=3, padding=1, stride=1, bias=False)))
        self._engine = None

    def forward(self, inputs):
        if self.training:
            raise RuntimeError("openstereo_b200.GwcDispProcessor implements the inference branch only (model.eval())")
        if self._engine is None:
            self._engine = GwcAggregation(self)
        h, w = inputs["left"].shape[2:]
        return {"inference_disp": {"disp_est": self._engine(inputs["cost_volume"], h, w)}}


class GwcNet(nn.Module):
    def __init__(self, cfgs):
        super().__init__()
        self.maxdisp = _cfg_get(cfgs, "MAX_DISP", 192)
        use_concat, cc = _cfg_get(cfgs, "USE_CONCAT_VOLUME", True), _cfg_get(cfgs, "CONCAT_CHANNELS", 12)
        ds, g = _cfg_get(cfgs, "DOWNSAMPLE", 4), _cfg_get(cfgs, "NUM_GROUPS", 40)
        self.Backbone = _GwcBackbone(use_concat, cc if use_concat else 0)
        self.CostProcessor = GwcVolumeCostProcessor(self.maxdisp, ds, g, use_concat)
        self.DispProcessor = GwcDispProcessor(self.maxdisp, ds, g, use_concat, cc)

    def forward(self, inputs):
        inputs.update(self.Backbone(inputs))                      # the reference mutates the dict too (gwcnet.py:30,32)
        inputs.update(self.CostProcessor(inputs))
        return {"disp_pred": self.DispProcessor(inputs)["inference_disp"]["disp_est"]}


# ---- PSMNet
def _cbr3(cin, cout, k=3, s=1, p=1):
    return nn.Sequential(nn.Conv3d(cin, cout, kernel_size=k, stride=s, padding=p, dilation=1, bias=False),
                         nn.BatchNorm3d(cout), nn.ReLU(inplace=True))


class _PsmHourglassParams(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv1, self.conv2 = _cbr3(c, 2 * c, 3, 2, 1), _cb3(2 * c, 2 * c, 3, 1, 1)
        self.conv3, self.conv4 = _cbr3(2 * c, 2 * c, 3, 2, 1), _cbr3(2 * c, 2 * c, 3, 1, 1)
        self.conv5, self.conv6 = _db3(2 * c, 2 * c), _db3(2 * c, c)


class _PsmAggregatorParams(nn.Module):
    def __init__(self, max_disp, in_planes=64):
        super().__init__()
        self.max_disp = max_disp
        self.dres0 = nn.Sequential(_cbr3(in_planes, 32), _cbr3(32, 32))
        self.dres1 = nn.Sequential(_cbr3(32, 32), _cb3(32, 32, 3, 1, 1))
        self.dres2, self.dres3, self.dres4 = _PsmHourglassParams(32), _PsmHourglassParams(32), _PsmHourglassParams(32)
        for i in (1, 2, 3):
            setattr(self, "classif%d" % i, nn.Sequential(_cbr3(32, 32), nn.Conv3d(32, 1, kernel_size=3, stride=1, padding=1, bias=False)))


class PSMCostProcessor(nn.Module):
    """psmnet_cost_processor.py:224-256.  Returns the three DISPARITY maps directly (the fused tail never
    materialises the (B,192,H,W) costs), under the keys disp1..3."""

    def __init__(self, max_disp=192, in_planes=64):
        super().__init__()
        self.max_disp = max_disp
        self.aggregator = _PsmAggregatorParams(max_disp, in_planes)
        self._engine = None

    def forward(self, inputs):
        if self.training:
            raise RuntimeError("openstereo_b200.PSMCostProcessor implements inference only (model.eval())")
        if self._engine is None:
            self._engine = PSMAggregation(self.aggregator)
        raw = ops.cat_fms(inputs["ref_feature"], inputs["tgt_feature"], max_disp=int(self.max_disp // 4))
        d1, d2, d3 = self._engine(raw)
        return {"disp1": d1, "disp2": d2, "disp3": d3}


class _PsmSoftArgminParams(nn.Module):
    def __init__(self, max_disp):
        super().__init__()
        self.disp_regression = nn.Conv3d(1, 1, (max_disp, 1, 1), 1, 0, bias=False)     # frozen linspace weight, kept for the checkpoint
        self.disp_regression.weight.data = torch.linspace(0, max_disp - 1, max_disp).view(1, 1, max_disp, 1, 1)
        self.disp_regression.weight.requires_grad = False


class PSMDispProcessor(nn.Module):
    def __init__(self, max_disp=192):
        super().__init__()
        self.disp_processor = _PsmSoftArgminParams(max_disp)

    def forward(self, inputs):
        return [inputs["disp1"], inputs["disp2"], inputs["disp3"]]


class PSMNet(nn.Module):
    def __init__(self, cfgs):
        super().__init__()
        self.maxdisp = _cfg_get(cfgs, "MAX_DISP", 192)
        self.Backbone = _PsmBackbone()
        self.CostProcessor = PSMCostProcessor(max_disp=self.maxdisp)
        self.DispProcessor = PSMDispProcessor(max_disp=self.maxdisp)

    def forward(self, inputs):
        inputs.update(self.Backbone(inputs))
        inputs.update(self.CostProcessor(inputs))
        disps = self.DispProcessor(inputs)
        return {"disp_pred": disps[-1], "train_preds": disps}
