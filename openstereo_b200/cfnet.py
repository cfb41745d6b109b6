"""CFNet (stereo/modeling/models/cfnet/cfnet.py, class cfnet) after its 2D feature extractor, on the library.

``CFNetEngine(model)`` runs the eval branch of ``cfnet.forward`` (cfnet.py:488-668) from the features on:

* stage 1   the three gwc + concatenation volumes at maxdisp // 8, 16, 32 (one ops.gwc_concat_volume launch each), dres0 / dres1
            at each scale, combine1 = hourglassup(32), dres3 = hourglass(32), classif2 and the soft-argmin with its variance
            (one osb_softargmin_var_fwd launch over the integer planes);
* s3, s2    the search range and the disparity samples: the sqrt of the variance, the gamma / beta bounds and their bilinear x2
            up-sampling restated term for term (they are inline in the reference's forward, so there is nothing to call;
            F.interpolate, which the reference's deprecated F.upsample alias calls), then the model's own generate_search_range and
            generate_disparity_samples (`.long()` included); the warped gwc + concatenation volume at those samples
            (osb_warped_gwc_concat_volume_ex_fwd with the left copy unmasked) with the samples appended as one more channel
            (torch.cat), confidence0..3, confidence_classif1 and the soft-argmin over the samples (with the variance at s3);
* the final bilinear x2 up-sampling of the s2 disparity.

Every 3D convolution (about 75 per forward) runs on the fp32 CUDA-core kernels of csrc/conv3d.cu with BN folded and Mish in the
epilogue (OSB_ACT_MISH), the residuals ``dres1(cost0) + cost0`` and ``FMish(conv(x) + redir(y))`` in the same launch.  No
tensor-core layer runs, so the engine polls no range guard.  Parameters are read through the reference's attribute names and
re-packed when they change; a module tree whose activations are not the reference's Mish (``CFNet(d, replace_mish=True)``) is
refused when the engine is built, naming the module.
"""
import torch
import torch.nn.functional as F

from . import ops
from .aggregation import _Engine, _Packed
from .ops import ACT_MISH, ACT_NONE


def _is_mish(m):
    return type(m).__name__ == "Mish"


def _convbn(m, fold):
    """convbn_3d = Sequential(Conv3d, BatchNorm3d) (cfnet/submodule.py:115-118) with the BN folded (fold=False: validation only,
    the module may still be in training mode), or a bare Conv3d."""
    if isinstance(m, torch.nn.Sequential):
        if len(m) != 2 or not isinstance(m[1], torch.nn.BatchNorm3d):
            raise NotImplementedError("patch(CFNet): %r is not the reference's convbn_3d" % (m,))
        return _Packed(m[0], m[1] if fold else None)
    return _Packed(m)


def _chain(seq, name, fold=True):
    """Sequential of convbn_3d / Conv3d / ConvTranspose3d + BatchNorm3d, each optionally followed by the reference's Mish ->
    [(packed layer, activation)].  Any other module (nn.ReLU in a model built with replace_mish=True) is refused, named."""
    mods, out, i = list(seq), [], 0
    while i < len(mods):
        m = mods[i]
        if isinstance(m, torch.nn.ConvTranspose3d) and i + 1 < len(mods) and isinstance(mods[i + 1], torch.nn.BatchNorm3d):
            out.append((_Packed(m, mods[i + 1] if fold else None), ACT_NONE))
            i += 2
            continue
        if _is_mish(m) and out and out[-1][1] == ACT_NONE:
            out[-1] = (out[-1][0], ACT_MISH)
        elif isinstance(m, (torch.nn.Sequential, torch.nn.Conv3d)):
            out.append((_convbn(m, fold), ACT_NONE))
        else:
            raise NotImplementedError("patch(CFNet): %s.%d is %s; the kernels implement the reference's Mish after a convolution "
                                      "(a model built with replace_mish=True is not served)" % (name, i, type(m).__name__))
        i += 1
    return out


def _run(chain, x, residual=None):
    """The chain's layers in order; `residual` is added before the last layer's activation (dres1(cost0) + cost0)."""
    for i, (layer, act) in enumerate(chain):
        x = _conv3d(layer, x, act, residual if i == len(chain) - 1 else None)
    return x


def _conv3d(layer, x, act=ACT_NONE, residual=None):
    if layer.transposed:
        return ops.deconv3d(x, layer.w, layer.scale, layer.shift, residual, layer.kernel, act)
    if layer.kernel == 1:
        return ops.conv3d_1x1(x, layer.w, layer.scale, layer.shift, residual, None, act)
    return ops.conv3d_k3(x, layer.w, layer.scale, layer.shift, residual, None, layer.stride, act)


# The Sequentials the engine runs (cfnet.py:288-402) and its five hourglasses
_CHAINS = ("dres0", "dres1", "dres0_5", "dres1_5", "dres0_6", "dres1_6", "confidence0_s3", "confidence1_s3", "confidence0_s2",
           "confidence1_s2", "classif2", "confidence_classif1_s3", "confidence_classif1_s2")
_HOURGLASSES = ("dres3", "confidence2_s3", "confidence3_s3", "confidence2_s2", "confidence3_s2")


def _single(chain, name):
    if len(chain) != 1:
        raise NotImplementedError("patch(CFNet): %s is not one convolution" % name)
    return chain[0][0]


class _Hourglass:
    """hourglass (cfnet.py:222-262): conv1..4 with Mish, conv5 / conv6 = FMish(deconv + redir) in one launch each."""

    def __init__(self, m, name, fold=True):
        self.c = {k: _chain(getattr(m, k), "%s.%s" % (name, k), fold) for k in ("conv1", "conv2", "conv3", "conv4")}
        self.conv5, self.conv6 = (_single(_chain(getattr(m, k), "%s.%s" % (name, k), fold), k) for k in ("conv5", "conv6"))
        self.redir1, self.redir2 = _convbn(m.redir1, fold), _convbn(m.redir2, fold)

    def __call__(self, x):
        conv2 = _run(self.c["conv2"], _run(self.c["conv1"], x))
        conv4 = _run(self.c["conv4"], _run(self.c["conv3"], conv2))
        conv5 = _conv3d(self.conv5, conv4, ACT_MISH, _conv3d(self.redir2, conv2))
        return _conv3d(self.conv6, conv5, ACT_MISH, _conv3d(self.redir1, x))


class _HourglassUp:
    """hourglassup (cfnet.py:170-219): conv1 / conv3 are plain stride-2 convolutions, their outputs concatenated with the next
    scale's cost (torch.cat) before combine1 / combine2; conv8 / conv9 = FMish(deconv + redir) in one launch each."""

    def __init__(self, m, name, fold=True):
        self.conv1, self.conv3 = _Packed(m.conv1), _Packed(m.conv3)
        self.c = {k: _chain(getattr(m, k), "%s.%s" % (name, k), fold) for k in ("conv2", "conv4", "combine1", "combine2")}
        self.conv8, self.conv9 = (_single(_chain(getattr(m, k), "%s.%s" % (name, k), fold), k) for k in ("conv8", "conv9"))
        self.redir1, self.redir2 = _convbn(m.redir1, fold), _convbn(m.redir2, fold)

    def __call__(self, x, feature4, feature5):
        conv1 = _run(self.c["combine1"], torch.cat((_conv3d(self.conv1, x), feature4), dim=1))
        conv2 = _run(self.c["conv2"], conv1)
        conv3 = _run(self.c["combine2"], torch.cat((_conv3d(self.conv3, conv2), feature5), dim=1))
        conv4 = _run(self.c["conv4"], conv3)
        conv8 = _conv3d(self.conv8, conv4, ACT_MISH, _conv3d(self.redir2, conv2))
        return _conv3d(self.conv9, conv8, ACT_MISH, _conv3d(self.redir1, x))


class CFNetEngine(_Engine):
    """Eval forward of the reference's cfnet after feature_extraction; see the module docstring.  Constructing it checks every
    module it will run, so an unsupported model is refused at once."""

    def __init__(self, model):
        super().__init__(model)
        with torch.no_grad():
            self._pack(fold=False)                                   # every layer's modules and hyper-parameters, checked now

    def _pack(self, fold=True):
        m = self.module
        self.chains = {name: _chain(getattr(m, name), name, fold) for name in _CHAINS}
        self.hourglasses = {name: _Hourglass(getattr(m, name), name, fold) for name in _HOURGLASSES}
        self.combine1 = _HourglassUp(m.combine1, "combine1", fold)

    @staticmethod
    def serves(data):
        """CUDA inference calls whose image height and width are multiples of 32 (the five-level feature pyramid)."""
        left, right = data["left"], data["right"]
        return left.dim() == 4 and left.shape == right.shape and left.shape[2] % 32 == 0 and left.shape[3] % 32 == 0

    # ---- the stages (tools/bench_configs.py c17 times them one by one)
    def volumes(self, fl, fr):
        """Stage-1 volumes: torch.cat((gwc_volume_s, concat_volume_s), 1) at maxdisp // 8, 16, 32 (cfnet.py:494-511)."""
        m = self.module
        return [ops.gwc_concat_volume(fl["gw%d" % s], fr["gw%d" % s], fl["concat_feature%d" % s], fr["concat_feature%d" % s],
                                      m.maxdisp // 2 ** (s - 1), m.num_groups).float() for s in (4, 5, 6)]

    def stage1(self, vol4, vol5, vol6):
        """cfnet.py:516-532 -> (pred2_s4 (B, 1, H/8, W/8), its standard deviation)."""
        c = self.chains
        cost = []
        for v, s in ((vol4, ""), (vol5, "_5"), (vol6, "_6")):
            c0 = _run(c["dres0" + s], v)
            cost.append(_run(c["dres1" + s], c0, residual=c0))
        out2 = self.hourglasses["dres3"](self.combine1(*cost))
        pred, var = ops.softargmin_var(_run(c["classif2"], out2).squeeze(1))
        return pred, var.sqrt()

    def samples(self, pred, std, gamma, beta, scale, sample_count, size):
        """The search range and the integer disparity samples of the next stage (cfnet.py:533-543, 567-577).  The bounds
        pred -/+ ((gamma + 1) std + beta) and their bilinear x2 up-sampling (align_corners) to `size` are restated term for term, in
        the reference's order: they are inline in its forward, and F.upsample is a deprecated alias of F.interpolate.  Then the
        model's own generate_search_range and generate_disparity_samples, `.long()` included.  -> (B, sample_count + 2, h, w) fp32."""
        m = self.module
        lo = F.interpolate((pred - (gamma + 1) * std - beta) * 2, size, mode="bilinear", align_corners=True)
        hi = F.interpolate((pred + (gamma + 1) * std + beta) * 2, size, mode="bilinear", align_corners=True)
        lo, hi = m.generate_search_range(sample_count + 1, lo, hi, scale=scale)
        return m.generate_disparity_samples(lo, hi, sample_count).float()

    def refine(self, fl, fr, samples, level, stage, num_groups, variance):
        """One refinement stage (s3: level 3, s2: level 2; cfnet.py:544-566, 578-597): the warped volume at `samples` with the samples
        appended, the confidence stack and the soft-argmin over the samples -> (pred (B, 1, h, w), standard deviation or None)."""
        c = self.chains
        vol = ops.warped_gwc_concat_volume(fl["gw%d" % level], fr["gw%d" % level], fl["concat_feature%d" % level],
                                           fr["concat_feature%d" % level], samples, num_groups, mask_left=False).float()
        vol = torch.cat((vol, samples.unsqueeze(1)), dim=1)
        c0 = _run(c["confidence0_" + stage], vol)
        c0 = _run(c["confidence1_" + stage], c0, residual=c0)
        out2 = self.hourglasses["confidence3_" + stage](self.hourglasses["confidence2_" + stage](c0))
        pred, var = ops.softargmin_var(_run(c["confidence_classif1_" + stage], out2).squeeze(1), samples, variance)
        return pred, None if var is None else var.sqrt()

    def __call__(self, fl, fr, h, w):
        """features_left / features_right (the reference's feature_extraction dicts) -> disparity (B, h, w) fp32."""
        m = self.module
        fl = {k: self._check(v) for k, v in fl.items()}
        fr = {k: self._check(v) for k, v in fr.items()}
        self._ensure(fl["gw4"].device)
        pred, std = self.stage1(*self.volumes(fl, fr))
        samples = self.samples(pred, std, m.gamma_s3.detach(), m.beta_s3.detach(), 2, m.sample_count_s3, [h // 4, w // 4])
        pred, std = self.refine(fl, fr, samples, 3, "s3", m.num_groups, True)
        samples = self.samples(pred, std, m.gamma_s2.detach(), m.beta_s2.detach(), 1, m.sample_count_s2, [h // 2, w // 2])
        pred, _ = self.refine(fl, fr, samples, 2, "s2", m.num_groups // 2, False)
        return F.interpolate(pred * 2, [h, w], mode="bilinear", align_corners=True).squeeze(1)
