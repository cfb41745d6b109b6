"""Hot-path engines: run the reference's 3D aggregation modules with the sm_90a kernels.

Each engine is built FROM an existing module tree (the reference's own ``GwcDispProcessor`` /
``PSMAggregator`` / StereoBase ``Hourglass``, or the host mirrors in host_models.py): it reads the
module's parameters by the reference's attribute names, pre-packs them once (weights to
(Cin, taps, Cout); eval BatchNorm folded to scale/shift) and then executes the forward graph as a
sequence of fused kernels.  cfg -> constructor -> load_state_dict stay untouched, so unchanged
checkpoints and YAML configs keep working (SURVEY.md section 8b).

Graphs restated (file:line of the reference forward each engine replaces):
  GwcAggregation        gwcnet/gwcnet_disp_processor.py:83-91,128-140 + gwcnet/hourglass.py:46-56
  CascadeAggregation    casnet/cas_psm.py:233-279 (CostAggregation, eval) + cas_psm.py:33-43
  PSMAggregation        psmnet/psmnet_cost_processor.py:181-221,108-132 + psmnet_disp_processor.py:107-118
  StereoBaseAggregation stereobase/hourglass.py:79-104 + stereobase_gru.py:161-164, and IGEV-RT's hourglass(8)
                        igev_rt/igev_rt_stereo.py:21-87 (the same graph built from IGEV's BasicConv / FeatureAtt)
  LightStereoAggregation lightstereo/aggregation.py:42-60 (Aggregation.forward), :94-101 (MobileV2Residual), :119-134 (AttentionModule)
  CoExAggregation       coex/coex_cost_processor.py:196-237 (Aggregation.forward), :68-80 (channelAtt)
  MSNet3DAggregation    msnet/MSNet3D.py:118-161 (eval forward after the volume), :10-46 (hourglass3D), submodule.py:136-173
  MSNet2DVolume         msnet/MSNet2D.py:143-162 (the 48-disparity volume loop)
  MSNet2DAggregation    msnet/MSNet2D.py:164-212 (eval forward after the volume), :10-45 (hourglass2D), submodule.py:94-133
  IGEVPPAggregation     igevpp/igevpp_stereo.py:69-94 (hourglass.forward), submodule.py:8-34 (BasicConv), :162-175 (FeatureAtt)
"""
import torch

from . import ops
from .ops import ACT_LEAKY, ACT_NONE, ACT_RELU, ACT_RELU6


class _Packed:
    """One conv/deconv (+BN) layer, packed for the kernels."""
    __slots__ = ("w", "scale", "shift", "stride", "kernel", "transposed", "cin", "cout", "_w5", "_tc")

    def __init__(self, conv, bn=None):
        self._tc = {}                                           # kind -> weight packed for the wgmma kernels (tc)
        self._w5 = conv.weight.detach() if conv.weight.dim() == 5 else None
        self.cin, self.cout = (conv.in_channels, conv.out_channels)
        self.transposed = isinstance(conv, (torch.nn.ConvTranspose3d, torch.nn.ConvTranspose2d))
        self.kernel = int(conv.kernel_size[0])
        self.stride = int(conv.stride[0])
        self._validate(conv)
        wt = conv.weight
        if wt.dim() == 4:                                       # Conv2d 1x1 (FeatureAtt)
            wt = wt.unsqueeze(2)
        if self.transposed:
            self.w = ops.pack_deconv_weight(wt)
        else:
            self.w = ops.pack_conv_weight(wt)
        if self.kernel == 1:
            self.w = self.w.reshape(self.w.shape[0], self.w.shape[2]).contiguous()
        self.scale, self.shift = (None, None)
        if bn is not None:
            if bn.training:
                raise RuntimeError("BatchNorm folding is only valid in eval mode (call model.eval())")
            self.scale, self.shift = ops.fold_bn(bn)
        if getattr(conv, "bias", None) is not None:
            bias = conv.bias.detach().float()
            self.shift = bias.contiguous() if self.shift is None else (self.shift + bias * self.scale).contiguous()


def _packed_validate(self, conv):
    """The kernels implement exactly the hyper-parameters of the three reference architectures (isotropic k in {1, 3} or the k4
    transposed conv, stride 1/2, padding k // 2, dilation 1, groups 1).  A module tree that deviates would silently compute a
    different convolution: refuse it instead."""
    ks, st = tuple(conv.kernel_size), tuple(conv.stride)
    ok = len(set(ks)) == 1 and len(set(st)) == 1 and tuple(conv.dilation) == (1,) * len(ks) and conv.groups == 1
    if self.transposed:
        op = tuple(conv.output_padding)
        ok = ok and ((ks[0] == 3 and st[0] == 2 and tuple(conv.padding) == (1,) * len(ks) and op == (1,) * len(ks))
                     or (ks[0] == 4 and st[0] == 2 and tuple(conv.padding) == (1,) * len(ks) and op == (0,) * len(ks)))
    else:
        ok = ok and ks[0] in (1, 3) and st[0] in (1, 2) and tuple(conv.padding) == (ks[0] // 2,) * len(ks)
        ok = ok and getattr(conv, "padding_mode", "zeros") == "zeros"
    if not ok:
        raise NotImplementedError("openstereo_b200: no kernel for %r (supported: Conv k1/k3, stride 1/2, padding k//2, dilation 1, "
                                  "groups 1; ConvTranspose k3 s2 p1 op1 or k4 s2 p1)" % (conv,))


def _packed_tc(self, kind):
    """This layer's weight packed for a tensor-core kernel family, packed on first use: kind 16 or 32 the stride-1 pack at that K
    chunk (a head narrower than 16 channels zero-padded to 16), "s2" the stride-2 pack, "dc" the transposed conv's, "c1" the taps of
    a one-channel head for conv3d_k3_c1_ndhwc, "head" a one-channel head with Cin zero-padded to a multiple of 32."""
    if kind not in self._tc:
        w = self._w5
        if kind == "s2":
            self._tc[kind] = ops.pack_tc_weight(w, 16, kw_order=(1, 0, 2))
        elif kind == "dc":
            self._tc[kind] = ops.pack_tc_deconv_weight(w)
        elif kind == "c1":
            self._tc[kind] = ops.pack_c1_weight(w)
        elif kind == "head":
            self._tc[kind] = ops.pack_tc_weight(_zero_padded(w, 1, _pad32(self.cin)), 32, pad_cout_to=16)
        else:
            self._tc[kind] = ops.pack_tc_weight(w, kind, pad_cout_to=16 if self.cout < 16 else None)
    return self._tc[kind]


def _zero_padded(w, n0, n1):
    """w (n0', n1', ...) zero-padded to (n0, n1, ...)."""
    out = w.new_zeros((n0, n1) + tuple(w.shape[2:]))
    out[:w.shape[0], :w.shape[1]] = w
    return out


def _pad32(c):
    return (c + 31) // 32 * 32


_Packed._validate = _packed_validate
_Packed.tc = _packed_tc


def _conv(layer, x, act=ACT_NONE, residual=None, gate=None):
    if layer.kernel == 1:
        return ops.conv3d_1x1(x, layer.w, layer.scale, layer.shift, residual, gate, act)
    return ops.conv3d_k3(x, layer.w, layer.scale, layer.shift, residual, gate, layer.stride, act)


USE_TENSOR_CORES = True      # set False to force every conv onto the fp32 CUDA-core kernels


def _tc_weight(layer, width):
    """hi/lo split weight of a 3x3x3 stride-1 layer for the tensor-core kernel variant serving `width`, or None."""
    if not USE_TENSOR_CORES or layer.transposed or layer.kernel != 3 or layer.stride != 1 or layer._w5 is None:
        return None
    kc = ops.conv3d_tc_kc(layer.cin, layer.cout, width)
    return layer.tc(kc) if kc else None


def _tc_ok(layer, width):
    return _tc_weight(layer, width) is not None


def _conv_tc(layer, x_ndhwc, act=ACT_NONE, residual=None, out_ndhwc=True, res_ndhwc=True, in_ncdhw=False, out_split=False):
    wt = _tc_weight(layer, x_ndhwc.shape[4] if in_ncdhw else x_ndhwc.shape[3])
    return ops.conv3d_k3_tc(x_ndhwc, wt, layer.scale, layer.shift, residual, act, out_ndhwc, res_ndhwc, in_ncdhw,
                            out_split=out_split)


def _split_chain_ok(width, *layers):
    """True when every layer runs on the W = 128 kernel, which reads and writes split activations (ops.to_split): a chain of
    them hands its intermediate tensors on in that form."""
    return USE_TENSOR_CORES and all(ops.conv3d_tc_kc(l.cin, l.cout, width) == 32 for l in layers)


def _stem_in(layer, volume, act, out_split=False):
    """First aggregation layer on an NCDHW cost volume: the W = 128 kernel reads NCDHW directly, other variants convert once."""
    if ops.conv3d_tc_kc(layer.cin, layer.cout, volume.shape[-1]) == 32:
        return _conv_tc(layer, volume, act, in_ncdhw=True, out_split=out_split)
    return _conv_tc(layer, ops.to_ndhwc(volume), act)


def _conv_auto(layer, x, act=ACT_NONE, residual=None):
    """3x3x3 conv (stride 1 or 2) on an NCDHW tensor, NCDHW result: tensor cores when a kernel variant exists for the
    shape, the fp32 CUDA-core kernel otherwise."""
    if layer.stride == 1 and _tc_ok(layer, x.shape[-1]):
        return _conv_tc(layer, ops.to_ndhwc(x), act, residual, out_ndhwc=False, res_ndhwc=False)
    if (USE_TENSOR_CORES and layer.stride == 2 and layer.kernel == 3 and not layer.transposed and layer._w5 is not None
            and ops.conv3d_s2_tc_supported(layer.cin, layer.cout, x.shape[2], x.shape[3], x.shape[4])):
        return ops.conv3d_k3_s2_tc(ops.to_ndhwc(x), layer.tc("s2"), layer.scale, layer.shift, residual, act)
    return _conv(layer, x, act, residual)


def _deconv(layer, x, act=ACT_NONE, residual=None):
    if (USE_TENSOR_CORES and layer.transposed and layer.kernel == 3 and layer._w5 is not None
            and ops.deconv3d_tc_supported(layer.cin, layer.cout, x.shape[-1])):
        return ops.deconv3d_k3_tc(ops.to_ndhwc(x), layer.tc("dc"), layer.scale, layer.shift, residual, act)
    return ops.deconv3d(x, layer.w, layer.scale, layer.shift, residual, layer.kernel, act)


def _versions(module):
    return tuple(p._version for p in module.parameters()) + tuple(b._version for b in module.buffers())


class _Engine:
    """Pre-pack on first use; re-pack when any parameter/buffer was modified in place or moved."""

    def __init__(self, module):
        self.module = module
        self._stamp = None

    def _watch(self, device):
        """fp16-range guard of the tensor-core convolutions: report a past overflow, schedule the next asynchronous read."""
        if USE_TENSOR_CORES:
            mon = ops.TcOverflowMonitor.get(device)
            mon.check()
            return mon
        return None

    def _ensure(self, device):
        stamp = (str(device), _versions(self.module), tuple(p.data_ptr() for p in self.module.parameters()))
        if stamp != self._stamp:
            if self.module.training:
                raise RuntimeError("openstereo_b200 engines run inference only: call model.eval()")
            with torch.no_grad():
                self._pack()
            self._stamp = stamp

    @staticmethod
    def _check(x):
        if not x.is_cuda:
            raise RuntimeError("openstereo_b200: not implemented on the CPU (no fallback); move the model to CUDA")
        return x.detach().float().contiguous()


# ------------------------------------------------------------------------------------------------------ GwcNet
class _GwcHourglass:
    def __init__(self, m):
        self.conv1, self.conv2 = _Packed(m.conv1[0][0], m.conv1[0][1]), _Packed(m.conv2[0][0], m.conv2[0][1])
        self.conv3, self.conv4 = _Packed(m.conv3[0][0], m.conv3[0][1]), _Packed(m.conv4[0][0], m.conv4[0][1])
        self.conv5, self.conv6 = _Packed(m.conv5[0], m.conv5[1]), _Packed(m.conv6[0], m.conv6[1])
        self.redir1, self.redir2 = _Packed(m.redir1[0], m.redir1[1]), _Packed(m.redir2[0], m.redir2[1])

    def __call__(self, x):
        c1 = _conv_auto(self.conv1, x, ACT_RELU)
        c2 = _conv_auto(self.conv2, c1, ACT_RELU)
        c3 = _conv_auto(self.conv3, c2, ACT_RELU)
        c4 = _conv_auto(self.conv4, c3, ACT_RELU)
        c5 = _deconv(self.conv5, c4, ACT_RELU, residual=_conv(self.redir2, c2))
        return _deconv(self.conv6, c5, ACT_RELU, residual=_conv(self.redir1, x))


def _hg_channels_last_ok(hg, x_shape_ndhwc):
    """True when every layer of a GwcNet hourglass has a tensor-core / channels-last kernel for this input."""
    if not USE_TENSOR_CORES:
        return False
    b, d, h, w, c = x_shape_ndhwc
    if d % 4 or h % 4 or w % 4:
        return False
    return (ops.conv3d_s2_tc_supported(hg.conv1.cin, hg.conv1.cout, d, h, w) and _tc_ok(hg.conv2, w // 2)
            and ops.conv3d_s2_tc_supported(hg.conv3.cin, hg.conv3.cout, d // 2, h // 2, w // 2) and _tc_ok(hg.conv4, w // 4)
            and ops.deconv3d_tc_supported(hg.conv5.cin, hg.conv5.cout, w // 4)
            and ops.deconv3d_tc_supported(hg.conv6.cin, hg.conv6.cout, w // 2)
            and (hg.redir1.cin, hg.redir1.cout) in ((32, 32), (64, 64)) and (hg.redir2.cin, hg.redir2.cout) in ((32, 32), (64, 64)))


def _gwc_hourglass_channels_last(hg, x):
    """GwcNet hourglass (gwcnet/hourglass.py:46-56) with every tensor channels-last: no layout conversion between layers."""
    c1 = ops.conv3d_k3_s2_tc(x, hg.conv1.tc("s2"), hg.conv1.scale, hg.conv1.shift, None, ACT_RELU, out_ndhwc=True)
    c2 = _conv_tc(hg.conv2, c1, ACT_RELU)
    c3 = ops.conv3d_k3_s2_tc(c2, hg.conv3.tc("s2"), hg.conv3.scale, hg.conv3.shift, None, ACT_RELU, out_ndhwc=True)
    c4 = _conv_tc(hg.conv4, c3, ACT_RELU)
    r2 = ops.conv1x1_ndhwc(c2, hg.redir2.w, hg.redir2.scale, hg.redir2.shift)
    c5 = ops.deconv3d_k3_tc(c4, hg.conv5.tc("dc"), hg.conv5.scale, hg.conv5.shift, r2, ACT_RELU, out_ndhwc=True, res_ndhwc=True)
    r1 = ops.conv1x1_ndhwc(x, hg.redir1.w, hg.redir1.scale, hg.redir1.shift)
    return ops.deconv3d_k3_tc(c5, hg.conv6.tc("dc"), hg.conv6.scale, hg.conv6.shift, r1, ACT_RELU, out_ndhwc=True, res_ndhwc=True)


def _classif3_channels_last(classif3, out):
    """classif3 (conv+BN+ReLU, then the 32 -> 1 conv) on a channels-last volume -> (B,1,D,H,W) logits.  The first conv must have a
    tensor-core variant for the width."""
    head0, cls = classif3
    width = out.shape[3]
    if _tc_ok(cls, width):                                         # 32 -> 1 head on the narrow (Cout <= 16) tensor-core variant
        mid = _conv_tc(head0, out, ACT_RELU, out_split=_split_chain_ok(width, head0, cls))
        return _conv_tc(cls, mid, ACT_NONE, out_ndhwc=False, res_ndhwc=False)
    if cls.cin == 32 and cls.cout == 1 and cls._w5 is not None and cls.stride == 1:
        head = _conv_tc(head0, out, ACT_RELU)                      # stays channels-last for the 1-channel head
        return ops.conv3d_k3_c1_ndhwc(head, cls.tc("c1"), cls.scale, cls.shift)
    head = _conv_tc(head0, out, ACT_RELU, out_ndhwc=False)
    return _conv(cls, head)


class GwcAggregation(_Engine):
    """Eval branch of GwcDispProcessor: volume (B,64,D',H',W') -> disparity (B,H,W)."""

    def _pack(self):
        m = self.module
        self.dres0 = [_Packed(m.dres0[0][0], m.dres0[0][1]), _Packed(m.dres0[2][0], m.dres0[2][1])]
        self.dres1 = [_Packed(m.dres1[0][0], m.dres1[0][1]), _Packed(m.dres1[2][0], m.dres1[2][1])]
        self.hg = [_GwcHourglass(m.dres2), _GwcHourglass(m.dres3), _GwcHourglass(m.dres4)]
        self.classif3 = [_Packed(m.classif3[0][0], m.classif3[0][1]), _Packed(m.classif3[2])]

    def logits(self, volume):
        volume = self._check(volume)
        self._ensure(volume.device)
        width = volume.shape[-1]
        stem_tc = all(_tc_ok(l, width) for l in (self.dres0[0], self.dres0[1], self.dres1[0], self.dres1[1]))
        b, _, dd, hh, ww = volume.shape
        if stem_tc and _tc_ok(self.classif3[0], width) and all(_hg_channels_last_ok(hg, (b, dd, hh, ww, 32)) for hg in self.hg):
            # everything from the volume to the classifier runs channels-last on the tensor cores: ONE layout conversion; inside
            # the W = 128 stem the activations stay split
            split = _split_chain_ok(width, self.dres0[0], self.dres0[1], self.dres1[0], self.dres1[1])
            c = _conv_tc(self.dres0[1], _stem_in(self.dres0[0], volume, ACT_RELU, out_split=split), ACT_RELU, out_split=split)
            out = _conv_tc(self.dres1[1], _conv_tc(self.dres1[0], c, ACT_RELU, out_split=split), ACT_NONE, residual=c)
            for hg in self.hg:
                out = _gwc_hourglass_channels_last(hg, out)
            return _classif3_channels_last(self.classif3, out)
        if stem_tc:
            # full-resolution stem on the tensor cores: channels-last inside, NCDHW handed to the hourglasses
            c = _conv_tc(self.dres0[1], _stem_in(self.dres0[0], volume, ACT_RELU), ACT_RELU)
            cost0 = _conv_tc(self.dres1[1], _conv_tc(self.dres1[0], c, ACT_RELU), ACT_NONE, residual=c, out_ndhwc=False)
        else:
            c = _conv(self.dres0[1], _conv(self.dres0[0], volume, ACT_RELU), ACT_RELU)
            cost0 = _conv(self.dres1[1], _conv(self.dres1[0], c, ACT_RELU), ACT_NONE, residual=c)
        out = cost0
        for hg in self.hg:
            out = hg(out)
        if _tc_ok(self.classif3[0], width):
            head = _conv_tc(self.classif3[0], ops.to_ndhwc(out), ACT_RELU, out_ndhwc=False)
        else:
            head = _conv(self.classif3[0], out, ACT_RELU)
        return _conv(self.classif3[1], head)

    def __call__(self, volume, h, w):
        mon = self._watch(volume.device)
        out = ops.upsample_softargmin(self.logits(volume), self.module.maxdisp, h, w, align_corners=False)
        if mon is not None:
            mon.poll()
        return out


class CascadeAggregation(GwcAggregation):
    """Eval branch of CasStereo's CostAggregation (casnet/cas_psm.py:233-279, the same class in cas_gwc.py:210-256): its
    layers and module indices are GwcDispProcessor's, so GwcAggregation.logits runs it as is; the tail weights fine bin d by
    the per-pixel hypothesis disp_range_samples[b, d, h, w] instead of d."""

    def __call__(self, cost, fine_d, fine_h, fine_w, disp_range_samples):
        mon = self._watch(cost.device)
        assert tuple(disp_range_samples.shape[1:]) == (fine_d, fine_h, fine_w)
        out = ops.upsample_softargmin_values(self.logits(cost), disp_range_samples, align_corners=False)
        if mon is not None:
            mon.poll()
        return out


# ------------------------------------------------------------------------------------------------------ PSMNet
class _PSMHourglass:
    def __init__(self, m):
        self.conv1, self.conv2 = _Packed(m.conv1[0], m.conv1[1]), _Packed(m.conv2[0], m.conv2[1])
        self.conv3, self.conv4 = _Packed(m.conv3[0], m.conv3[1]), _Packed(m.conv4[0], m.conv4[1])
        self.conv5, self.conv6 = _Packed(m.conv5[0], m.conv5[1]), _Packed(m.conv6[0], m.conv6[1])

    def __call__(self, x, presqu, postsqu, skip):
        out = _conv_auto(self.conv1, x, ACT_RELU)
        pre = _conv_auto(self.conv2, out, ACT_RELU, residual=postsqu)
        out = _conv_auto(self.conv4, _conv_auto(self.conv3, pre, ACT_RELU), ACT_RELU)
        post = _deconv(self.conv5, out, ACT_RELU, residual=presqu if presqu is not None else pre)
        # `out_i = hourglass(...) + cost0` (psmnet_cost_processor.py:188-194) rides on conv6's epilogue
        return _deconv(self.conv6, post, ACT_NONE, residual=skip), pre, post


def _psm_hg_channels_last_ok(hg, shape_ndhwc):
    """True when every layer of a PSMNet hourglass has a tensor-core kernel for this channels-last input."""
    if not USE_TENSOR_CORES:
        return False
    b, d, h, w, c = shape_ndhwc
    if d % 4 or h % 4 or w % 4 or any(l._w5 is None for l in (hg.conv1, hg.conv2, hg.conv3, hg.conv4, hg.conv5, hg.conv6)):
        return False
    return (ops.conv3d_s2_tc_supported(hg.conv1.cin, hg.conv1.cout, d, h, w) and _tc_ok(hg.conv2, w // 2)
            and ops.conv3d_s2_tc_supported(hg.conv3.cin, hg.conv3.cout, d // 2, h // 2, w // 2) and _tc_ok(hg.conv4, w // 4)
            and hg.conv5.kernel == 3 and hg.conv6.kernel == 3
            and ops.deconv3d_tc_supported(hg.conv5.cin, hg.conv5.cout, w // 4)
            and ops.deconv3d_tc_supported(hg.conv6.cin, hg.conv6.cout, w // 2))


def _psm_hourglass_channels_last(hg, x, presqu, postsqu, skip):
    """PSMNet hourglass (psmnet_cost_processor.py:108-132) with every tensor channels-last: the NCDHW route converted the layout in
    front of every layer.  Returns (out + skip, pre, post) like _PSMHourglass.__call__, all NDHWC."""
    out = ops.conv3d_k3_s2_tc(x, hg.conv1.tc("s2"), hg.conv1.scale, hg.conv1.shift, None, ACT_RELU, out_ndhwc=True)
    pre = _conv_tc(hg.conv2, out, ACT_RELU, residual=postsqu)
    out = ops.conv3d_k3_s2_tc(pre, hg.conv3.tc("s2"), hg.conv3.scale, hg.conv3.shift, None, ACT_RELU, out_ndhwc=True)
    out = _conv_tc(hg.conv4, out, ACT_RELU)
    post = ops.deconv3d_k3_tc(out, hg.conv5.tc("dc"), hg.conv5.scale, hg.conv5.shift, presqu if presqu is not None else pre, ACT_RELU,
                              out_ndhwc=True, res_ndhwc=True)
    out = ops.deconv3d_k3_tc(post, hg.conv6.tc("dc"), hg.conv6.scale, hg.conv6.shift, skip, ACT_NONE, out_ndhwc=True, res_ndhwc=True)
    return out, pre, post


class PSMAggregation(_Engine):
    """PSMAggregator + FasterSoftArgmin: raw concat volume -> [disp1, disp2, disp3], each (B,H,W)."""

    def _pack(self):
        m = self.module
        self.dres0 = [_Packed(m.dres0[0][0], m.dres0[0][1]), _Packed(m.dres0[1][0], m.dres0[1][1])]
        self.dres1 = [_Packed(m.dres1[0][0], m.dres1[0][1]), _Packed(m.dres1[1][0], m.dres1[1][1])]
        self.hg = [_PSMHourglass(m.dres2), _PSMHourglass(m.dres3), _PSMHourglass(m.dres4)]
        self.heads = [[_Packed(c[0][0], c[0][1]), _Packed(c[1])] for c in (m.classif1, m.classif2, m.classif3)]

    def logits(self, raw_cost):
        raw_cost = self._check(raw_cost)
        self._ensure(raw_cost.device)
        width = raw_cost.shape[-1]
        stem_tc = all(_tc_ok(l, width) for l in (self.dres0[0], self.dres0[1], self.dres1[0], self.dres1[1]))
        b, _, dd, hh, ww = raw_cost.shape
        if (stem_tc and all(_psm_hg_channels_last_ok(hg, (b, dd, hh, ww, 32)) for hg in self.hg)
                and all(_tc_ok(a, width) and _tc_ok(bb, width) for a, bb in self.heads)):
            # everything channels-last on the tensor cores: the stacked-hourglass skips (pre / post / cost0) never change layout
            c = _conv_tc(self.dres0[1], _stem_in(self.dres0[0], raw_cost, ACT_RELU), ACT_RELU)
            cost0 = _conv_tc(self.dres1[1], _conv_tc(self.dres1[0], c, ACT_RELU), ACT_NONE, residual=c)
            out1, pre1, post1 = _psm_hourglass_channels_last(self.hg[0], cost0, None, None, cost0)
            out2, pre2, post2 = _psm_hourglass_channels_last(self.hg[1], out1, pre1, post1, cost0)
            out3, _, _ = _psm_hourglass_channels_last(self.hg[2], out2, pre2, post2, cost0)
            costs, prev = [], None
            for (a, bb), x in zip(self.heads, (out1, out2, out3)):
                prev = _conv_tc(bb, _conv_tc(a, x, ACT_RELU), ACT_NONE, residual=prev, out_ndhwc=False, res_ndhwc=False)
                costs.append(prev)
            return costs
        if stem_tc:
            c = _conv_tc(self.dres0[1], _stem_in(self.dres0[0], raw_cost, ACT_RELU), ACT_RELU)
            cost0 = _conv_tc(self.dres1[1], _conv_tc(self.dres1[0], c, ACT_RELU), ACT_NONE, residual=c, out_ndhwc=False)
        else:
            c = _conv(self.dres0[1], _conv(self.dres0[0], raw_cost, ACT_RELU), ACT_RELU)
            cost0 = _conv(self.dres1[1], _conv(self.dres1[0], c, ACT_RELU), ACT_NONE, residual=c)
        out1, pre1, post1 = self.hg[0](cost0, None, None, cost0)
        out2, pre2, post2 = self.hg[1](out1, pre1, post1, cost0)
        out3, pre3, post3 = self.hg[2](out2, pre2, post2, cost0)

        def head(i, x, prev):
            a, b = self.heads[i]
            if _tc_ok(a, width) and _tc_ok(b, width):                   # both convs on tensor cores, channels-last in between
                return _conv_tc(b, _conv_tc(a, ops.to_ndhwc(x), ACT_RELU), ACT_NONE, residual=prev, out_ndhwc=False, res_ndhwc=False)
            if _tc_ok(a, width):
                return _conv(b, _conv_tc(a, ops.to_ndhwc(x), ACT_RELU, out_ndhwc=False), residual=prev)
            return _conv(b, _conv(a, x, ACT_RELU), residual=prev)

        cost1 = head(0, out1, None)
        cost2 = head(1, out2, cost1)
        cost3 = head(2, out3, cost2)
        return [cost1, cost2, cost3]

    def __call__(self, raw_cost):
        b, c, d, h, w = raw_cost.shape
        max_disp = self.module.max_disp
        mon = self._watch(raw_cost.device)
        out = [ops.upsample_softargmin(cost, max_disp, 4 * h, 4 * w, align_corners=True)
               for cost in self.logits(raw_cost)]
        if mon is not None:
            mon.poll()
        return out


# -------------------------------------------------------------------------------------------------- StereoBase
class _FeatureAtt:
    """FeatureAtt: StereoBase's (feat_att[0] a BasicConv2d with `.block`) or IGEV's (feat_att[0] an IGEV BasicConv), then a biased
    1x1 Conv2d."""

    def __init__(self, m):
        first = m.feat_att[0]
        if hasattr(first, "block"):
            blk = first.block
            self.a = _Packed(blk[0], blk[1])
            self.act = ACT_LEAKY if any(isinstance(l, torch.nn.LeakyReLU) for l in blk) else ACT_NONE
        else:
            self.a, self.act = _igev_basic_conv(first)
        self.b = _Packed(m.feat_att[1])

    def __call__(self, feat):
        hidden = ops.conv3d_1x1(feat, self.a.w, self.a.scale, self.a.shift, act=self.act)
        return ops.conv3d_1x1(hidden, self.b.w, self.b.scale, self.b.shift, sigmoid_out=True)   # (B, cv_chan, H, W)


def _igev_basic_conv(m):
    """IGEV's BasicConv (igev/submodule.py, igev_rt/submodule.py): `.conv`, then `.bn` only when `use_bn` (the module owns a `bn`
    even with bn=False), then nn.LeakyReLU() -- slope 0.01, created inside forward -- only when `relu` -> (_Packed, act)."""
    return _Packed(m.conv, m.bn if m.use_bn else None), ACT_LEAKY if m.relu else ACT_NONE


def _block(m):
    """(_Packed, act) of one hourglass layer: StereoBase's BasicConv3d / BasicDeconv3d (`.block` = conv, optional BN, optional
    LeakyReLU) or IGEV's BasicConv."""
    if not hasattr(m, "block"):
        return _igev_basic_conv(m)
    layers = list(m.block)
    bn = layers[1] if len(layers) > 1 and isinstance(layers[1], torch.nn.BatchNorm3d) else None
    act = ACT_LEAKY if any(isinstance(l, torch.nn.LeakyReLU) for l in layers) else ACT_NONE
    return _Packed(layers[0], bn), act


class StereoBaseAggregation(_Engine):
    """Hourglass(volume_channel, backbone_channels) with FeatureAtt gates: (B,C,D',H',W') + 2D features -> same shape.  Also runs
    IGEV-RT's hourglass(8): its 8/16/32/48-channel plan fails tc_route_ok, so every layer takes the fp32 CUDA-core kernels."""

    def _pack(self):
        m = self.module
        self.conv = {name: [_block(b) for b in getattr(m, name)] for name in ("conv1", "conv2", "conv3", "agg_0", "agg_1")}
        self.up = {name: _block(getattr(m, name)) for name in ("conv3_up", "conv2_up", "conv1_up")}
        self.att = {name: _FeatureAtt(getattr(m, "feature_att_" + name)) for name in ("8", "16", "32", "up_16", "up_8")}

    def _pair(self, name, x, gate):
        (l0, a0), (l1, a1) = self.conv[name]
        return _conv(l1, _conv(l0, x, a0), a1, gate=gate)

    def _agg(self, name, up, skip, gate):
        (l0, a0), (l1, a1), (l2, a2) = self.conv[name]
        # torch.cat((up, skip), 1) -> 1x1 conv, without materialising the concat (hourglass.py:91-92,96-97)
        x = ops.conv3d_1x1(up, l0.w, l0.scale, l0.shift, act=a0, x1=skip)
        return _conv(l2, _conv(l1, x, a1), a2, gate=gate)

    # ---- tensor-core route: channels-last, channel plan zero-padded to multiples of 32 (24 -> 32, 48 -> 64, 96) -------------------
    def tc_route_ok(self, shape):
        """True when the 1/8 and 1/16 levels and the two upper transposed convs of this hourglass have wgmma variants for an
        input volume of `shape` (B, C, D', H', W'); the 1/32 level (6 % of the MACs at config 3) stays on the CUDA-core kernels."""
        if not USE_TENSOR_CORES:
            return False
        b, c, d, h, w = shape
        if d % 8 or h % 8 or w % 8:
            return False
        (l10, _), (l11, _) = self.conv["conv1"]
        (l20, _), (l21, _) = self.conv["conv2"]
        if (l10.cin, l10.cout, l20.cout) != (c, 2 * c, 4 * c) or any(l._w5 is None for l in (l10, l11, l20, l21)):
            return False
        pc, p2, p4 = _pad32(c), _pad32(2 * c), _pad32(4 * c)
        return bool(ops.conv3d_s2_tc_supported(pc, p2, d, h, w) and ops.conv3d_tc_kc(p2, p2, w // 2) == 16
                    and ops.conv3d_s2_tc_supported(p2, p4, d // 2, h // 2, w // 2) and ops.conv3d_tc_kc(p4, p4, w // 4) == 16
                    and ops.deconv3d_k4_tc_supported(p4, p2, w // 4) and ops.deconv3d_k4_tc_supported(p2, pc, w // 2)
                    and (2 * p4, p4) in ((192, 96), (128, 64)) and (2 * p2, p2) in ((192, 96), (128, 64))
                    and self.up["conv2_up"][0].kernel == 4 and self.up["conv1_up"][0].kernel == 4)

    def _tc_pack(self):
        """Zero-padded tensor-core packs of the layers on the 1/8 and 1/16 levels (built once per _ensure stamp)."""
        if getattr(self, "_tcp_stamp", None) == self._stamp:
            return self._tcp
        P = _pad32

        def vec(v, n, fill):
            if v is None:
                return None
            out = v.new_full((n,), fill)
            out[:v.numel()] = v
            return out

        def pack(layer, transposed=False, kw_order=(0, 1, 2), bounds=None):
            """[(lo, weight, scale, shift)] per output-channel slice [lo, hi) of `bounds` (default: one slice of every channel) of the
            layer with Cin and Cout zero-padded to multiples of 32."""
            w = layer._w5                                                   # (Cout, Cin, 3, 3, 3); transposed (Cin, Cout, 4, 4, 4)
            wp = _zero_padded(w, P(w.shape[0]), P(w.shape[1]))
            n = wp.shape[1 if transposed else 0]
            sc, sh = vec(layer.scale, n, 1.0), vec(layer.shift, n, 0.0)
            out = []
            for lo, hi in bounds or ((0, n),):
                wt = (ops.pack_tc_deconv_weight(wp[:, lo:hi].contiguous()) if transposed
                      else ops.pack_tc_weight(wp[lo:hi].contiguous(), 16, kw_order=kw_order))
                out.append((lo, wt, None if sc is None else sc[lo:hi].contiguous(), None if sh is None else sh[lo:hi].contiguous()))
            return out

        def whole(layer, **kw):
            return pack(layer, **kw)[0][1:]

        def cat1x1(layer):
            w = layer.w                                                     # (C0 + C1, Cout), both slabs Cout channels wide
            cout = w.shape[1]
            wp = w.new_zeros((2 * P(cout), P(cout)))
            wp[:cout, :cout] = w[:cout]
            wp[P(cout):P(cout) + cout, :cout] = w[cout:]
            return (wp.contiguous(), vec(layer.scale, P(cout), 1.0), vec(layer.shift, P(cout), 0.0))

        t = {}
        for name in ("conv1", "conv2"):
            (l0, _), (l1, _) = self.conv[name]
            t[name] = (whole(l0, kw_order=(1, 0, 2)), whole(l1))
        for name in ("agg_0", "agg_1"):
            (l0, _), (l1, _), (l2, _) = self.conv[name]
            t[name] = (cat1x1(l0), whole(l1), whole(l2))
        for name in ("conv2_up", "conv1_up"):
            t[name] = whole(self.up[name][0], transposed=True)
        # 1/32 level: 6c = 144 runs as 160 = 96 + 64 output-channel slices (N = 3 * 160 exceeds one CTA's weight buffers), the
        # transposed conv back to 4c = 96 as 64 + 32 (N = 4 * 96 exceeds the wgmma N limit of 256): separately packed weight slices
        (l0, _), (l1, _) = self.conv["conv3"]
        lu = self.up["conv3_up"][0]
        if P(l0.cout) == 160 and P(l0.cin) == 96 and lu.kernel == 4 and all(l._w5 is not None for l in (l0, l1, lu)):
            t["conv3"] = (pack(l0, kw_order=(1, 0, 2), bounds=((0, 96), (96, 160))), pack(l1, bounds=((0, 96), (96, 160))))
            t["conv3_up"] = pack(lu, transposed=True, bounds=((0, 64), (64, 96)))
        self._tcp, self._tcp_stamp = t, self._stamp
        return t

    def _level32_tc_ok(self, shape):
        b, c, d, h, w = shape
        return bool(w // 8 == 16 and _pad32(6 * c) == 160 and _pad32(4 * c) == 96
                    and ops.conv3d_s2_tc_supported(96, 96, d // 4, h // 4, w // 4) and ops.conv3d_s2_tc_supported(96, 64, d // 4, h // 4, w // 4)
                    and ops.conv3d_tc_kc(160, 96, 16) == 16 and ops.conv3d_tc_kc(160, 64, 16) == 16
                    and ops.deconv3d_k4_tc_supported(160, 64, 16) and ops.deconv3d_k4_tc_supported(160, 32, 16))

    def _gate_nhwc(self, name, feat, channels):
        fa = self.att[name]                                                 # one launch: (B, H, W, C padded), padded channels 0
        if fa.a.w.shape[1] % 4 == 0 and fa.b.w.shape[1] % 4 == 0:
            return ops.feature_att_gate(feat, fa.a.w, fa.a.scale, fa.a.shift, fa.b.w, fa.b.scale, fa.b.shift, pad_to=channels,
                                        act1=fa.act)
        return ops.to_ndhwc(fa(feat).unsqueeze(2), pad_to=channels).squeeze(1)

    def _call_tc(self, x, feats):
        t = self._tc_pack()
        c = x.shape[1]
        pc, p2, p4 = _pad32(c), _pad32(2 * c), _pad32(4 * c)
        act = lambda name, i: self.conv[name][i][1]                         # noqa: E731
        xc = ops.to_ndhwc(x, pad_to=pc)
        (w0, sc0, sh0), (w1, sc1, sh1) = t["conv1"]
        c1 = ops.conv3d_k3_s2_tc(xc, w0, sc0, sh0, None, act("conv1", 0), out_ndhwc=True)
        conv1 = ops.conv3d_k3_tc(c1, w1, sc1, sh1, None, act("conv1", 1), gate=self._gate_nhwc("8", feats[1], p2))
        (w0, sc0, sh0), (w1, sc1, sh1) = t["conv2"]
        c2 = ops.conv3d_k3_s2_tc(conv1, w0, sc0, sh0, None, act("conv2", 0), out_ndhwc=True)
        conv2 = ops.conv3d_k3_tc(c2, w1, sc1, sh1, None, act("conv2", 1), gate=self._gate_nhwc("16", feats[2], p4))
        if "conv3" in t and self._level32_tc_ok(x.shape):
            # 1/32 level (768 voxels per pair at config 3: one 8 x 16 plane = one M tile) as output-channel slices
            b, d4, h4, w4, _ = conv2.shape
            s0, s1 = t["conv3"]
            y = conv2.new_empty((b, d4 // 2, h4 // 2, w4 // 2, 160))
            for lo, wt, sc, sh in s0:
                ops.tc_slice("s2", conv2, wt, sc, sh, y, lo, act("conv3", 0))
            g32 = self._gate_nhwc("32", feats[3], 160)
            conv3 = torch.empty_like(y)
            for lo, wt, sc, sh in s1:
                ops.tc_slice("s1", y, wt, sc, sh, conv3, lo, act("conv3", 1), gate=g32)
            up3 = conv2.new_empty((b, d4, h4, w4, p4))
            for lo, wt, sc, sh in t["conv3_up"]:
                ops.tc_slice("dc4", conv3, wt, sc, sh, up3, lo, self.up["conv3_up"][1])
        else:
            # 1/32 level on the fp32 CUDA-core kernels (NCDHW): 6 % of the MACs
            conv2_ncdhw = conv2[..., :4 * c].permute(0, 4, 1, 2, 3).contiguous()
            conv3 = self._pair("conv3", conv2_ncdhw, self.att["32"](feats[3]))
            l, a = self.up["conv3_up"]
            up3 = ops.to_ndhwc(_deconv(l, conv3, a), pad_to=p4)
        (wc, scc, shc), (w1, sc1, sh1), (w2, sc2, sh2) = t["agg_0"]
        y = ops.conv1x1_ndhwc_cat(up3, conv2, wc, scc, shc, act("agg_0", 0))
        y = ops.conv3d_k3_tc(y, w1, sc1, sh1, None, act("agg_0", 1))
        conv2 = ops.conv3d_k3_tc(y, w2, sc2, sh2, None, act("agg_0", 2), gate=self._gate_nhwc("up_16", feats[2], p4))
        wu, scu, shu = t["conv2_up"]
        up2 = ops.deconv3d_k4_tc(conv2, wu, scu, shu, None, self.up["conv2_up"][1])
        (wc, scc, shc), (w1, sc1, sh1), (w2, sc2, sh2) = t["agg_1"]
        y = ops.conv1x1_ndhwc_cat(up2, conv1, wc, scc, shc, act("agg_1", 0))
        y = ops.conv3d_k3_tc(y, w1, sc1, sh1, None, act("agg_1", 1))
        conv1 = ops.conv3d_k3_tc(y, w2, sc2, sh2, None, act("agg_1", 2), gate=self._gate_nhwc("up_8", feats[1], p2))
        wu, scu, shu = t["conv1_up"]
        return ops.deconv3d_k4_tc(conv1, wu, scu, shu, None, self.up["conv1_up"][1], out_ndhwc=False, cout_real=c)

    def __call__(self, x, features):
        x = self._check(x)
        self._ensure(x.device)
        feats = [self._check(f) for f in features]
        if self.tc_route_ok(x.shape):
            mon = self._watch(x.device)
            out = self._call_tc(x, feats)
            if mon is not None:
                mon.poll()
            return out
        g8, g16, g32 = self.att["8"](feats[1]), self.att["16"](feats[2]), self.att["32"](feats[3])
        conv1 = self._pair("conv1", x, g8)
        conv2 = self._pair("conv2", conv1, g16)
        conv3 = self._pair("conv3", conv2, g32)
        l, a = self.up["conv3_up"]
        conv2 = self._agg("agg_0", _deconv(l, conv3, a), conv2, self.att["up_16"](feats[2]))
        l, a = self.up["conv2_up"]
        conv1 = self._agg("agg_1", _deconv(l, conv2, a), conv1, self.att["up_8"](feats[1]))
        l, a = self.up["conv1_up"]
        return _deconv(l, conv1, a)


class StereoBaseCostHead(_Engine):
    """classifier Conv3d(C,1,3) -> softmax -> disparity_regression (stereobase_gru.py:101,163-164).
    ``module`` is the nn.Conv3d classifier."""

    def _pack(self):
        self.layer = _Packed(self.module)

    def logits(self, geo):
        """classifier(geo) alone: (B,C,D',H',W') -> (B,1,D',H',W') fp32 logits (IGEV-RT's softmax and regression follow it)."""
        geo = self._check(geo)
        self._ensure(geo.device)
        lay = self.layer
        cp = _pad32(lay.cin)
        if (USE_TENSOR_CORES and lay.cout == 1 and lay._w5 is not None and lay.kernel == 3 and lay.stride == 1
                and ops.conv3d_tc_kc(cp, 1, geo.shape[-1]) == 32):
            # 24 -> 1 head on the narrow tensor-core variant: channels zero-padded to 32 while the layout changes (one pass), the
            # generic CUDA-core conv is the slow path at config 3
            mon = self._watch(geo.device)
            logits = ops.conv3d_k3_tc(ops.to_ndhwc(geo, pad_to=cp), lay.tc("head"), lay.scale, lay.shift, None, ACT_NONE,
                                      out_ndhwc=False, res_ndhwc=False)
            if mon is not None:
                mon.poll()
        else:
            logits = _conv(lay, geo)                            # (B,1,D',H',W')
        return logits

    def __call__(self, geo, maxdisp_lowres):
        return ops.softargmin(self.logits(geo).squeeze(1), maxdisp_lowres, keepdim=True)


# -------------------------------------------------------------------------------------------------------- CoEx
def _basic_conv(m):
    """CoEx's BasicConv (coex/submodule.py): conv, then its BN only when use_bn, then LeakyReLU only when relu -> (_Packed, act)."""
    if m.relu and m.LeakyReLU.negative_slope != 0.01:
        raise NotImplementedError("openstereo_b200: LeakyReLU slope %g (the kernels apply 0.01)" % m.LeakyReLU.negative_slope)
    return _Packed(m.conv, m.bn if m.use_bn else None), ACT_LEAKY if m.relu else ACT_NONE


class _ChannelAtt:
    """channelAtt.im_att (coex_cost_processor.py:68-80): image features (B,Cim,H,W) -> sigmoid gate (B,Ccv,H,W), applied by
    the epilogue of the conv the reference multiplies it into."""

    def __init__(self, m):
        self.a, self.act = _basic_conv(m.im_att[0])
        self.b = _Packed(m.im_att[1])

    def __call__(self, im):
        hidden = ops.conv3d_1x1(im, self.a.w, self.a.scale, self.a.shift, act=self.act)
        return ops.conv3d_1x1(hidden, self.b.w, self.b.scale, self.b.shift, sigmoid_out=True)


class CoExAggregation(_Engine):
    """Eval forward of CoEx's Aggregation (coex_cost_processor.py:196-237): cost (B, head, D, h, w) and the image features ->
    logits (B, 1, D, h, w).  Every conv runs on the fp32 CUDA-core kernels; each channelAtt gate rides on the epilogue of the conv
    it follows; each conv_skip is a 1x1 conv over (up, skip) without the concatenation; where a transposed conv's output is larger
    than its skip level (an odd extent below it), nearest_resize3d brings it back like the reference's F.interpolate.
    conv_skip[0], conv_agg[0] and channelAtt[0] are never used by the forward and are not read."""

    def _pack(self):
        m = self.module
        self.gce = bool(m.gce)
        self.down = [[_basic_conv(c) for c in seq] for seq in m.conv_down]
        self.up = [_basic_conv(c) for c in m.conv_up]
        self.stem = _basic_conv(m.conv_stem)
        # indexed like the reference's up path: step i uses conv_skip[-i-1], conv_agg[-i-1], channelAtt[-i-1] for i = 0, 1
        self.skip = [_basic_conv(m.conv_skip[-i - 1]) for i in range(2)]
        self.agg = [[_basic_conv(c) for c in m.conv_agg[-i - 1]] for i in range(2)]
        if self.gce:
            self.att_stem = _ChannelAtt(m.channelAttStem)
            self.att_down = [_ChannelAtt(a) for a in m.channelAttDown]
            self.att = [_ChannelAtt(m.channelAtt[-i - 1]) for i in range(2)]

    def _seq(self, layers, x, att, im):
        """A chain of BasicConvs; the channelAtt gate (when gce) rides on the last one."""
        for n, (layer, act) in enumerate(layers):
            gate = att(im) if self.gce and n == len(layers) - 1 else None
            x = _conv(layer, x, act, gate=gate)
        return x

    def __call__(self, img, cost):
        cost = self._check(cost)
        self._ensure(cost.device)
        img = [self._check(f) for f in img]
        b, _, h, w = img[0].shape
        x = cost.reshape(b, -1, self.module.D, h, w)
        x = self._seq([self.stem], x, getattr(self, "att_stem", None), img[0])
        levels = [x]
        for i in range(3):
            x = self._seq(self.down[i], x, self.att_down[i] if self.gce else None, img[i + 1])
            levels.append(x)
        for i in range(3):
            layer, act = self.up[-i - 1]
            x = ops.deconv3d(x, layer.w, layer.scale, layer.shift, None, layer.kernel, act)
            skip = levels[-i - 2]
            if x.shape[2:] != skip.shape[2:]:
                x = ops.nearest_resize3d(x, skip.shape[2:])
            if i == 2:
                break
            sl, sa = self.skip[i]
            x = ops.conv3d_1x1(x, sl.w, sl.scale, sl.shift, act=sa, x1=skip)
            x = self._seq(self.agg[i], x, self.att[i] if self.gce else None, img[-i - 2])
        return x


# ------------------------------------------------------------------------------------------------------ MSNet3D
def _mbv2_check(m, name):
    """Refuse a MobileV2_Residual_3D (msnet/submodule.py:136-173) that osb_mbv2_block3d_fwd does not implement, naming it."""
    layers = list(m.conv)
    if len(layers) != 8:
        raise NotImplementedError("openstereo_b200: %s uses the expanse_ratio == 1 branch (no 1x1x1 expansion); only the expanding "
                                  "MobileV2_Residual_3D has a kernel" % name)
    pw, bn1, a1, dw, bn2, a2, pl, bn3 = layers
    conv, bn = torch.nn.Conv3d, torch.nn.BatchNorm3d
    ok = all(isinstance(l, conv) for l in (pw, dw, pl)) and all(isinstance(l, bn) for l in (bn1, bn2, bn3))
    ok = ok and all(isinstance(l, torch.nn.ReLU6) for l in (a1, a2))
    ok = ok and all(l.bias is None and tuple(l.dilation) == (1, 1, 1) and l.padding_mode == "zeros" for l in (pw, dw, pl))
    ok = ok and all(tuple(l.kernel_size) == (1, 1, 1) and tuple(l.stride) == (1, 1, 1) and tuple(l.padding) == (0, 0, 0)
                    and l.groups == 1 for l in (pw, pl))
    hid = pw.out_channels if ok else 0
    ok = ok and tuple(dw.kernel_size) == (3, 3, 3) and tuple(dw.padding) == (1, 1, 1) and dw.stride in ((1, 1, 1), (2, 2, 2))
    ok = ok and dw.in_channels == dw.out_channels == dw.groups == hid and pl.in_channels == hid
    if not ok:
        raise NotImplementedError("openstereo_b200: %s is not the block osb_mbv2_block3d_fwd implements (1x1x1 expand + BN + ReLU6, "
                                  "depthwise 3x3x3 stride 1/2 padding 1 with groups == hidden + BN + ReLU6, 1x1x1 project + BN, "
                                  "no bias, no dilation)" % name)
    key = (pw.in_channels, hid, pl.out_channels, dw.stride[0])
    if key not in _MBV2_CONFIGS:
        raise NotImplementedError("openstereo_b200: %s has (Cin, Chid, Cout, stride) = %s; osb_mbv2_block3d_fwd is instantiated for "
                                  "%s" % (name, key, sorted(_MBV2_CONFIGS)))


_MBV2_CONFIGS = {(40, 120, 32, 1), (32, 96, 32, 1), (32, 64, 32, 1), (32, 64, 64, 2), (64, 128, 64, 1), (64, 128, 128, 2),
                 (128, 256, 128, 1)}


class _MBV2Block3D:
    """MobileV2_Residual_3D packed for osb_mbv2_block3d_fwd: the three BNs folded, w_exp (Cin, Chid), w_dw (27, Chid),
    w_proj (Chid, Cout).  use_res_connect is honoured as the module computes it (False for every block MSNet3D builds: its int
    stride never equals (1, 1, 1))."""

    def __init__(self, m, name):
        _mbv2_check(m, name)
        pw, bn1, _, dw, bn2, _, pl, bn3 = list(m.conv)
        self.cin, self.hid, self.cout, self.stride = pw.in_channels, pw.out_channels, pl.out_channels, dw.stride[0]
        self.w_exp = pw.weight.detach().float().reshape(self.hid, self.cin).t().contiguous()
        self.w_dw = dw.weight.detach().float().reshape(self.hid, 27).t().contiguous()
        self.w_proj = pl.weight.detach().float().reshape(self.cout, self.hid).t().contiguous()
        self.bn = [ops.fold_bn(b) for b in (bn1, bn2, bn3)]
        if any(b.training for b in (bn1, bn2, bn3)):
            raise RuntimeError("BatchNorm folding is only valid in eval mode (call model.eval())")
        self.res = bool(m.use_res_connect)
        self.name = name

    def __call__(self, x, residual=None, in_ndhwc=False, out_ndhwc=False):
        if self.res:
            if residual is not None:
                raise NotImplementedError("openstereo_b200: %s adds its identity and a second residual" % self.name)
            assert out_ndhwc or not in_ndhwc
            residual = x if in_ndhwc == out_ndhwc else ops.to_ndhwc(x)
        (s1, b1), (s2, b2), (s3, b3) = self.bn
        return ops.mbv2_block3d(x, self.w_exp, s1, b1, self.w_dw, s2, b2, self.w_proj, s3, b3, residual, self.stride, in_ndhwc,
                                out_ndhwc)


class _MSNetHourglass:
    """hourglass3D (msnet/MSNet3D.py:10-46)."""

    def __init__(self, m, name):
        blk = lambda attr: _MBV2Block3D(getattr(m, attr), "%s.%s" % (name, attr))         # noqa: E731
        self.conv1, self.conv2, self.conv3, self.conv4 = blk("conv1"), blk("conv2"), blk("conv3"), blk("conv4")
        self.redir1, self.redir2 = blk("redir1"), blk("redir2")
        self.conv5, self.conv6 = _Packed(m.conv5[0], m.conv5[1]), _Packed(m.conv6[0], m.conv6[1])

    def __call__(self, x):
        """NCDHW; relu(conv5(conv4) + redir2(conv2)) and relu(conv6(conv5) + redir1(x)) in the transposed convs' epilogues."""
        c2 = self.conv2(self.conv1(x))
        c4 = self.conv4(self.conv3(c2))
        c5 = _deconv(self.conv5, c4, ACT_RELU, residual=self.redir2(c2))
        return _deconv(self.conv6, c5, ACT_RELU, residual=self.redir1(x))

    def channels_last(self, x):
        c2 = self.conv2(self.conv1(x, in_ndhwc=True, out_ndhwc=True), in_ndhwc=True, out_ndhwc=True)
        c4 = self.conv4(self.conv3(c2, in_ndhwc=True, out_ndhwc=True), in_ndhwc=True, out_ndhwc=True)
        r2 = self.redir2(c2, in_ndhwc=True, out_ndhwc=True)
        c5 = ops.deconv3d_k3_tc(c4, self.conv5.tc("dc"), self.conv5.scale, self.conv5.shift, r2, ACT_RELU, out_ndhwc=True,
                                res_ndhwc=True)
        r1 = self.redir1(x, in_ndhwc=True, out_ndhwc=True)
        return ops.deconv3d_k3_tc(c5, self.conv6.tc("dc"), self.conv6.scale, self.conv6.shift, r1, ACT_RELU, out_ndhwc=True,
                                  res_ndhwc=True)

    def channels_last_ok(self, shape):
        b, c, d, h, w = shape
        return (USE_TENSOR_CORES and d % 4 == 0 and h % 4 == 0 and w % 4 == 0
                and all(l._w5 is not None for l in (self.conv5, self.conv6))
                and ops.deconv3d_tc_supported(self.conv5.cin, self.conv5.cout, w // 4)
                and ops.deconv3d_tc_supported(self.conv6.cin, self.conv6.cout, w // 2))


class MSNet3DAggregation(_Engine):
    """Eval forward of MSNet3D after the cost volume (msnet/MSNet3D.py:118-161): dres0 -> dres1 (+ cost0) -> 3 x hourglass3D ->
    classif3 -> trilinear x4 + softmax + regression.  ``module`` is the MSNet3D model; its parameters are read by the reference's
    attribute names.  Every MobileV2_Residual_3D (22 per forward) is one osb_mbv2_block3d_fwd launch; dres1's `+ cost0` rides on
    its last block's residual operand.  Constructing the engine checks every block, so an unsupported model is refused at once."""

    def __init__(self, module):
        super().__init__(module)
        for name, m in self._blocks(module):
            _mbv2_check(m, name)

    @staticmethod
    def _blocks(m):
        for seq in ("dres0", "dres1"):
            for i, blk in enumerate(getattr(m, seq)):
                yield "%s.%d" % (seq, i), blk
        for hg in ("encoder_decoder1", "encoder_decoder2", "encoder_decoder3"):
            for attr in ("conv1", "conv2", "conv3", "conv4", "redir1", "redir2"):
                yield "%s.%s" % (hg, attr), getattr(getattr(m, hg), attr)

    def _pack(self):
        m = self.module
        self.dres0 = [_MBV2Block3D(b, "dres0.%d" % i) for i, b in enumerate(m.dres0)]
        self.dres1 = [_MBV2Block3D(b, "dres1.%d" % i) for i, b in enumerate(m.dres1)]
        self.hg = [_MSNetHourglass(getattr(m, n), n) for n in ("encoder_decoder1", "encoder_decoder2", "encoder_decoder3")]
        self.classif3 = [_Packed(m.classif3[0][0], m.classif3[0][1]), _Packed(m.classif3[2])]

    def logits(self, volume):
        volume = self._check(volume)
        self._ensure(volume.device)
        shape = (volume.shape[0], self.dres0[-1].cout) + tuple(volume.shape[2:])
        if all(hg.channels_last_ok(shape) for hg in self.hg) and _tc_ok(self.classif3[0], volume.shape[-1]):
            # the first block reads the NCDHW volume, every later tensor is channels-last
            c = self.dres0[0](volume, out_ndhwc=True)
            for blk in self.dres0[1:]:
                c = blk(c, in_ndhwc=True, out_ndhwc=True)
            out = c
            for i, blk in enumerate(self.dres1):
                out = blk(out, residual=c if i == len(self.dres1) - 1 else None, in_ndhwc=True, out_ndhwc=True)
            for hg in self.hg:
                out = hg.channels_last(out)
            return _classif3_channels_last(self.classif3, out)
        c = volume
        for blk in self.dres0:
            c = blk(c)
        out = c
        for i, blk in enumerate(self.dres1):
            out = blk(out, residual=c if i == len(self.dres1) - 1 else None)
        for hg in self.hg:
            out = hg(out)
        return _conv_auto(self.classif3[1], _conv_auto(self.classif3[0], out, ACT_RELU))

    def __call__(self, volume, h, w):
        mon = self._watch(volume.device)
        out = ops.upsample_softargmin(self.logits(volume), self.module.maxdisp, h, w, align_corners=False)
        if mon is not None:
            mon.poll()
        return out


# -------------------------------------------------------------------------------------------------- LightStereo
class _PW:
    """1x1 Conv2d (+BN or bias) packed for osb_conv3d_1x1_bn_act_fwd: weight (Cin, Cout)."""
    __slots__ = ("w", "scale", "shift")

    def __init__(self, conv, bn=None):
        self.w = conv.weight.detach().float().reshape(conv.out_channels, conv.in_channels).t().contiguous()
        self.scale, self.shift = ops.fold_bn(bn) if bn is not None else (None, None)
        if conv.bias is not None:
            bias = conv.bias.detach().float()
            self.shift = bias.contiguous() if self.shift is None else (self.shift + bias * self.scale).contiguous()


class _DW:
    """Depthwise Conv2d (+BN or bias)."""
    __slots__ = ("w", "scale", "shift", "stride")

    def __init__(self, conv, bn=None):
        assert conv.groups == conv.in_channels == conv.out_channels and conv.dilation == (1, 1)
        assert conv.padding == (conv.kernel_size[0] // 2, conv.kernel_size[1] // 2) and conv.stride[0] == conv.stride[1]
        self.w = conv.weight.detach().float().reshape(conv.out_channels, *conv.kernel_size).contiguous()
        self.stride = int(conv.stride[0])
        self.scale, self.shift = ops.fold_bn(bn) if bn is not None else (None, None)
        if conv.bias is not None:
            bias = conv.bias.detach().float()
            self.shift = bias.contiguous() if self.shift is None else (self.shift + bias * self.scale).contiguous()


class _InvertedResidual:
    """MobileV2Residual (lightstereo/aggregation.py:63-101): pw+BN+ReLU6 -> dw3x3+BN+ReLU6 -> pw+BN (+ identity)."""

    def __init__(self, m):
        self.pw = _PW(m.pwconv[0], m.pwconv[1])
        self.dw = _DW(m.dwconv[0], m.dwconv[1])
        self.pl = _PW(m.pwliner[0], m.pwliner[1])
        self.res = bool(m.use_res_connect)

    def __call__(self, x):
        h = ops.conv3d_1x1(x, self.pw.w, self.pw.scale, self.pw.shift, act=ACT_RELU6)
        h = ops.dwconv2d(h, self.dw.w, self.dw.scale, self.dw.shift, stride=self.dw.stride, act=ACT_RELU6)
        return ops.conv3d_1x1(h, self.pl.w, self.pl.scale, self.pl.shift, residual=x if self.res else None)


class _StripAttention:
    """AttentionModule (lightstereo/aggregation.py:104-134): cost * conv3(a + sum_k conv_k_2(conv_k_1(a))), a = conv0(feat)."""

    def __init__(self, m):
        self.conv0, self.conv3 = _PW(m.conv0), _PW(m.conv3)
        self.pairs = [(_DW(getattr(m, "conv%d_1" % i)), _DW(getattr(m, "conv%d_2" % i))) for i in range(3)]

    def __call__(self, cost, feat):
        a = ops.conv3d_1x1(feat, self.conv0.w, None, self.conv0.shift)
        acc = a
        for first, second in self.pairs:                        # acc = a + b0 + b1 + b2, accumulated by the second strip conv
            t = ops.dwconv2d(a, first.w, None, first.shift)
            acc = ops.dwconv2d(t, second.w, None, second.shift, residual=acc)
        return ops.conv3d_1x1(acc, self.conv3.w, None, self.conv3.shift, gate=cost)


class LightStereoAggregation(_Engine):
    """Aggregation.forward (lightstereo/aggregation.py:42-60): correlation volume (B, D/4, H/4, W/4) + left features at 1/4, 1/8,
    1/16 -> [(B, D/4, H/4, W/4)].  53 launches for LightStereo-S; no elementwise pass of its own (BN, ReLU6, shortcuts, the
    attention product and the final ReLUs all ride on the producing kernels)."""

    def _pack(self):
        m = self.module
        seq = lambda s: [_InvertedResidual(b) for b in s]
        self.conv0, self.conv2, self.conv4 = seq(m.conv0), seq(m.conv2), seq(m.conv4)
        self.conv1, self.conv3 = _InvertedResidual(m.conv1), _InvertedResidual(m.conv3)
        self.redir1, self.redir2 = _InvertedResidual(m.redir1), _InvertedResidual(m.redir2)
        self.up = []
        for blk in (m.conv5, m.conv6):
            sc, sh = ops.fold_bn(blk[1])
            self.up.append((ops.pack_deconv2d_weight(blk[0].weight), sc, sh))
        self.att = [_StripAttention(a) for a in (m.att0, m.att2, m.att4)] if m.left_att else None

    def __call__(self, x, features_left):
        x = self._check(x)
        self._ensure(x.device)
        feats = [self._check(f) for f in features_left]
        for blk in self.conv0:
            x = blk(x)
        if self.att:
            x = self.att[0](x, feats[0])
        half = self.conv1(x)
        for blk in self.conv2:
            half = blk(half)
        if self.att:
            half = self.att[1](half, feats[1])
        quarter = self.conv3(half)
        for blk in self.conv4:
            quarter = blk(quarter)
        if self.att:
            quarter = self.att[2](quarter, feats[2])
        w5, s5, b5 = self.up[0]
        up = ops.deconv2d_k3s2(quarter, w5, s5, b5, residual=self.redir2(half), act=ACT_RELU)
        w6, s6, b6 = self.up[1]
        return [ops.deconv2d_k3s2(up, w6, s6, b6, residual=self.redir1(x), act=ACT_RELU)]


# ------------------------------------------------------------------------------------------------------ MSNet2D
def msnet2d_volume_weights(conv3d):
    """The reference's depth-strided Conv3d chain (msnet/MSNet2D.py:73-81: k(8,3,3) s8, k(4,3,3) s4, k(2,3,3) s2, each + BN +
    ReLU) as three dense 3x3 Conv2d weights over the channel orders the library uses:
      layer-1 input   8j + t      the crop block j of ops.interlaced_crops: t < 4 left channel 4j+t (reference depth 8j + 2t),
                                  t >= 4 right channel 4j+t-4 (depth 8j + 2(t-4) + 1)
      layer-1 output  16j + c     channel c of reference depth j (eight blocks of the shared 8 -> 16 weight: block diagonal)
      layer-2 output  32e + c     channel c of depth e; input block 16(4e + k) + c' is channel c' of depth 4e + k
      layer-3 output  c           input 32k + c' is channel c' of depth k
    -> [(weight (Cout, Cin, 3, 3), scale, shift)] with the BN folded and the conv bias in the shift, fp32, on conv3d's device."""
    c1, b1, _, c2, b2, _, c3, b3, _ = conv3d
    w1, w2, w3 = (c.weight.detach().float() for c in (c1, c2, c3))
    n1, n2, n3 = w1.shape[0], w2.shape[0], w3.shape[0]
    depth = [2 * (t % 4) + t // 4 for t in range(8)]
    d1 = w1.new_zeros(8 * n1, 64, 3, 3)
    for j in range(8):
        d1[n1 * j:n1 * (j + 1), 8 * j:8 * (j + 1)] = w1[:, 0, depth]
    d2 = w2.new_zeros(2 * n2, 8 * n1, 3, 3)
    for e in range(2):
        d2[n2 * e:n2 * (e + 1), 4 * n1 * e:4 * n1 * (e + 1)] = w2.permute(0, 2, 1, 3, 4).reshape(n2, 4 * n1, 3, 3)
    d3 = w3.permute(0, 2, 1, 3, 4).reshape(n3, 2 * n2, 3, 3).contiguous()
    out = []
    for wd, conv, bn, rep in ((d1, c1, b1, 8), (d2, c2, b2, 2), (d3, c3, b3, 1)):
        if bn.training:
            raise RuntimeError("BatchNorm folding is only valid in eval mode (call model.eval())")
        scale, shift = ops.fold_bn(bn)
        if conv.bias is not None:
            shift = shift + conv.bias.detach().float() * scale
        out.append((wd.contiguous(), scale.repeat(rep).contiguous(), shift.repeat(rep).contiguous()))
    return out


def _msnet2d_check(model):
    """Refuse an MSNet2D whose volume network is not the one msnet2d_volume_weights restates, naming the module."""
    want = [((8, 3, 3), (8, 1, 1), 1, 16), ((4, 3, 3), (4, 1, 1), 16, 32), ((2, 3, 3), (2, 1, 1), 32, 16)]
    convs = [model.conv3d[i] for i in (0, 3, 6)] if len(model.conv3d) == 9 else []
    ok = len(convs) == 3 and all(
        isinstance(c, torch.nn.Conv3d) and (tuple(c.kernel_size), tuple(c.stride), c.in_channels, c.out_channels) == w
        and tuple(c.padding) == (0, 1, 1) and tuple(c.dilation) == (1, 1, 1) and c.groups == 1 for c, w in zip(convs, want))
    ok = ok and all(isinstance(model.conv3d[i], torch.nn.BatchNorm3d) for i in (1, 4, 7))
    ok = ok and all(isinstance(model.conv3d[i], torch.nn.ReLU) for i in (2, 5, 8))
    ok = ok and model.num_groups == 1 and model.volume_size == 48
    if not ok:
        raise NotImplementedError("openstereo_b200: MSNet2D.conv3d / num_groups / volume_size differ from the reference's "
                                  "(msnet/MSNet2D.py:55-81); no kernel plan for them")


class MSNet2DVolume(_Engine):
    """MSNet2D's volume loop (msnet/MSNet2D.py:143-162): featL, featR (B, 32, H, W) after preconv11 -> volume (B, 48, H, W).
    One osb_interlaced_crops_fwd launch writes the 48 cropped, interleaved inputs; per disparity d the three depth-strided Conv3ds
    run as dense 3x3 Conv2ds on the crop of width W - d (so their zero padding sits at its edges, as in the reference) and
    volume11 as a 1x1 conv, BN and ReLU folded into each epilogue.  A crop at least OSB_TC_MIN_WIDTH wide runs its 3x3 layers on
    the general-width wgmma kernels (3xFP16, fp32-accurate), a narrower one on the fp32 CUDA-core kernels.  Each volume11 result
    is copied into volume[:, d, :, d:] of a zeroed volume, so the columns w < d stay exactly 0."""

    def __init__(self, module):
        super().__init__(module)
        _msnet2d_check(module)

    def _pack(self):
        m = self.module
        self.layers = msnet2d_volume_weights(m.conv3d)
        w3, s3, b3 = self.layers[2]
        self.cout3 = _pad32(w3.shape[0])                        # the 16-channel layer runs zero-padded to 32 channels
        pad = lambda v: torch.cat((v, v.new_zeros(self.cout3 - v.numel())))     # noqa: E731
        self.cc = [ops.pack_conv_weight(self._at_kd1(w)) for w, _, _ in self.layers[:2]]
        self.cc.append(ops.pack_conv_weight(self._at_kd1(_zero_padded(w3, self.cout3, w3.shape[1]))))
        self.cc_affine = [(s, b) for _, s, b in self.layers[:2]] + [(pad(s3), pad(b3))]
        conv, bn = m.volume11[0][0], m.volume11[0][1]
        self.v11 = conv.weight.detach().float().reshape(1, -1).t()
        self.v11 = torch.cat((self.v11, self.v11.new_zeros(self.cout3 - self.v11.shape[0], 1))).contiguous()
        self.v11_scale, self.v11_shift = ops.fold_bn(bn)
        self._tc = {}

    @staticmethod
    def _at_kd1(w):
        w5 = w.new_zeros(w.shape[0], w.shape[1], 3, 3, 3)
        w5[:, :, 1] = w
        return w5

    def _tc_weight(self, i, width):
        w, _, _ = self.layers[i]
        kc = ops.conv2d_tc_kc(w.shape[1], self.cout3 if i == 2 else w.shape[0], width)
        if not kc:
            return None
        if (i, kc) not in self._tc:
            self._tc[(i, kc)] = ops.pack_tc_weight_2d(w, kc, pad_cout_to=self.cout3 if i == 2 else None)
        return self._tc[(i, kc)]

    def tc_width(self, width):
        """True when every 3x3 layer of a crop this wide runs on the tensor cores."""
        return USE_TENSOR_CORES and all(self._tc_weight(i, width) is not None for i in range(3))

    def front(self, x, width):
        """One crop (B, H, width, 64) channels-last -> the layer-3 output (B, cout3, H, width), channels 16.. zero."""
        if self.tc_width(width):
            for i, (_, s, b) in enumerate(self.layers):
                x = ops.conv2d_k3_tc(x, self._tc_weight(i, width), s, b, act=ACT_RELU, out_nhwc=i < 2)
            return x
        x = x.permute(0, 3, 1, 2).unsqueeze(2).contiguous()
        for w, (s, b) in zip(self.cc, self.cc_affine):
            x = ops.conv3d_k3(x, w, s, b, act=ACT_RELU)
        return x.squeeze(2)

    def __call__(self, feat_left, feat_right):
        fl, fr = self._check(feat_left), self._check(feat_right)
        self._ensure(fl.device)
        mon = self._watch(fl.device)
        b, _, h, w = fl.shape
        volume = torch.zeros((b, self.module.volume_size, h, w), dtype=torch.float32, device=fl.device)
        for d, x in enumerate(ops.interlaced_crops(fl, fr, min(self.module.volume_size, w))):
            y = ops.conv3d_1x1(self.front(x, w - d), self.v11, self.v11_scale, self.v11_shift, act=ACT_RELU)
            volume[:, d, :, d:].copy_(y[:, 0])
        if mon is not None:
            mon.poll()
        return volume


class _MBV2Block2D:
    """MobileV2_Residual (msnet/submodule.py:94-133): 1x1 + BN + ReLU6 -> depthwise 3x3 (stride 1/2) + BN + ReLU6 -> 1x1 + BN
    (+ identity when use_res_connect); `act` is applied after the identity, in the projection's epilogue."""

    def __init__(self, m, name):
        layers = list(m.conv)
        if len(layers) != 8 or not all(isinstance(layers[i], torch.nn.Conv2d) for i in (0, 3, 6)) or layers[0].kernel_size != (1, 1):
            raise NotImplementedError("openstereo_b200: %s is not an expanding MobileV2_Residual (1x1, depthwise 3x3, 1x1)" % name)
        pw, dw, pl = layers[0], layers[3], layers[6]
        if dw.groups != dw.in_channels or dw.kernel_size != (3, 3) or dw.dilation != (1, 1) or pl.kernel_size != (1, 1):
            raise NotImplementedError("openstereo_b200: %s has a dilated or non-depthwise 3x3; only dilation 1 has a kernel" % name)
        self.pw, self.dw, self.pl = _PW(pw, layers[1]), _DW(dw, layers[4]), _PW(pl, layers[7])
        self.res = bool(m.use_res_connect)

    def __call__(self, x, act=ACT_NONE):
        h = ops.conv3d_1x1(x, self.pw.w, self.pw.scale, self.pw.shift, act=ACT_RELU6)
        h = ops.dwconv2d(h, self.dw.w, self.dw.scale, self.dw.shift, stride=self.dw.stride, act=ACT_RELU6)
        return ops.conv3d_1x1(h, self.pl.w, self.pl.scale, self.pl.shift, residual=x if self.res else None, act=act)


class _Hourglass2D:
    """hourglass2D (msnet/MSNet2D.py:10-45): relu(conv5(conv4) + redir2(conv2)), relu(conv6(conv5) + redir1(x)) in the
    transposed convs' epilogues."""

    def __init__(self, m, name):
        blk = lambda attr: _MBV2Block2D(getattr(m, attr), "%s.%s" % (name, attr))          # noqa: E731
        self.conv1, self.conv2, self.conv3, self.conv4 = blk("conv1"), blk("conv2"), blk("conv3"), blk("conv4")
        self.redir1, self.redir2 = blk("redir1"), blk("redir2")
        self.up = []
        for attr in ("conv5", "conv6"):
            up = getattr(m, attr)[0]
            if (up.kernel_size, up.stride, up.padding, up.output_padding, up.dilation, up.groups) != ((3, 3), (2, 2), (1, 1), (1, 1),
                                                                                                      (1, 1), 1) or up.bias is not None:
                raise NotImplementedError("openstereo_b200: %s.%s is not ConvTranspose2d(k3, s2, p1, op1, bias=False)" % (name, attr))
            seq = getattr(m, attr)
            sc, sh = ops.fold_bn(seq[1])
            self.up.append((ops.pack_deconv2d_weight(seq[0].weight), sc, sh))

    def __call__(self, x):
        c2 = self.conv2(self.conv1(x))
        c4 = self.conv4(self.conv3(c2))
        (w5, s5, b5), (w6, s6, b6) = self.up
        c5 = ops.deconv2d_k3s2(c4, w5, s5, b5, residual=self.redir2(c2), act=ACT_RELU)
        return ops.deconv2d_k3s2(c5, w6, s6, b6, residual=self.redir1(x), act=ACT_RELU)


class MSNet2DAggregation(_Engine):
    """Eval forward of MSNet2D after the volume (msnet/MSNet2D.py:164-212): dres0 -> dres1 (+ cost0) -> 3 x hourglass2D ->
    classif3 -> trilinear x4 + softmax + regression (osb_upsample_softargmin_fwd, Dl = 48 -> maxdisp).  ``module`` is the MSNet2D
    model; its parameters are read by the reference's attribute names.  The ReLUs between the dres blocks ride on the blocks'
    projection epilogues; dres1's `+ cost0` follows its last block (that block already adds its own identity)."""

    def __init__(self, module):
        super().__init__(module)
        self._pack_blocks()

    def _pack_blocks(self):
        m = self.module
        self.dres0 = [_MBV2Block2D(m.dres0[i], "dres0.%d" % i) for i in (0, 2)]
        self.dres1 = [_MBV2Block2D(m.dres1[i], "dres1.%d" % i) for i in (0, 2)]
        self.hg = [_Hourglass2D(getattr(m, n), n) for n in ("encoder_decoder1", "encoder_decoder2", "encoder_decoder3")]
        cls = m.classif3
        self.classif3 = [(ops.pack_conv_weight(MSNet2DVolume._at_kd1(cls[0][0].weight.detach().float())),) + ops.fold_bn(cls[0][1]),
                         (ops.pack_conv_weight(MSNet2DVolume._at_kd1(cls[2].weight.detach().float())), None, None)]

    def _pack(self):
        self._pack_blocks()

    def logits(self, volume):
        """volume (B, 48, H, W) -> classif3's cost (B, 48, H, W)."""
        x = self._check(volume)
        self._ensure(x.device)
        cost0 = self.dres0[1](self.dres0[0](x, ACT_RELU), ACT_RELU)
        out = self.dres1[1](self.dres1[0](cost0, ACT_RELU))
        out += cost0
        for hg in self.hg:
            out = hg(out)
        (w0, s0, b0), (w1, _, _) = self.classif3
        out = ops.conv3d_k3(out.unsqueeze(2), w0, s0, b0, act=ACT_RELU)
        return ops.conv3d_k3(out, w1).squeeze(2)

    def __call__(self, volume, h, w):
        return ops.upsample_softargmin(self.logits(volume).unsqueeze(1), self.module.maxdisp, h, w, align_corners=False)


# ------------------------------------------------------------------------------------------------------ IGEV++
def _in_refusal(m, norm, relu):
    """Why IGEV++'s BasicConv `m` (igevpp/submodule.py:8-34: conv, InstanceNorm when use_in, LeakyReLU() made in forward when relu)
    is not the layer the instance-norm kernels run with flags (norm, relu), or None."""
    if bool(m.use_in) != norm or bool(m.relu) != relu:
        return "%r: IN=%s, relu=%s (the graph runs IN=%s, relu=%s)" % (m.conv, m.use_in, m.relu, norm, relu)
    inorm = m.IN
    if norm and (inorm.affine or inorm.track_running_stats or inorm.eps != 1e-5):
        return "%r: affine / tracked statistics / eps %g (eval normalises by each image's statistics with eps 1e-5)" % (inorm, inorm.eps)
    if norm and m.conv.bias is not None:
        return "%r: bias in front of the instance norm" % (m.conv,)
    slopes = [l.negative_slope for l in m.modules() if isinstance(l, torch.nn.LeakyReLU)]
    if any(s != 0.01 for s in slopes):
        return "LeakyReLU slope %s (the kernels apply 0.01)" % slopes
    try:
        _Packed(m.conv)
    except NotImplementedError as exc:
        return str(exc)
    return None


class _InstanceFeatureAtt:
    """IGEV++'s FeatureAtt (igevpp/submodule.py:162-175): feature map -> sigmoid(conv(leaky(instance_norm2d(conv(feat))))), two 1x1
    launches: the hidden layer with moments out, then the biased 1x1 on its normalised output with sigmoid_out."""

    def __init__(self, m):
        self.a, self.b = _Packed(m.feat_att[0].conv), _Packed(m.feat_att[1])

    def __call__(self, feat):
        hidden, stats = ops.conv3d_1x1_in(feat, self.a.w, moments=True)
        return ops.conv3d_1x1_in(hidden, self.b.w, in_stats0=stats, shift=self.b.shift, sigmoid_out=True)


_IGEVPP_CONVS = ("conv0", "conv1.0", "conv1.1", "conv2.0", "conv2.1", "conv3.0", "conv3.1", "conv3_up", "agg_0.0", "agg_0.1", "agg_0.2",
                 "conv2_up", "agg_1.0", "agg_1.1", "agg_1.2", "conv1_up")
_IGEVPP_GATES = ("4", "8", "16", "32", "up_16", "up_8")


class IGEVPPAggregation(_Engine):
    """IGEV++'s instance-normalised hourglass(8) (igevpp/igevpp_stereo.py:22-94): cost volume (B, C, D, H, W) + the four left
    feature maps -> (B, C, 2 * ceil(D / 2), ...), on the fp32 CUDA-core kernels.  Each BasicConv is conv -> InstanceNorm3d ->
    LeakyReLU(0.01): its convolution stores the raw output with the per-(b, channel) statistics (moments out) and every consumer
    normalises, activates and gates the tensor as it stages it (normalised input), so an instance-norm layer costs no pass over HBM
    of its own.  16 convolutions and 6 two-launch FeatureAtt gates: 28 launches.  conv1_up (IN=False, relu=False) writes the plain
    output."""

    def __init__(self, module):
        super().__init__(module)
        self._why = self._refusal()

    def _blocks(self):
        m = self.module
        for name in _IGEVPP_CONVS:
            mod = m
            for part in name.split("."):
                mod = mod[int(part)] if part.isdigit() else getattr(mod, part)
            yield name, mod

    def _refusal(self):
        m = self.module
        for name, blk in self._blocks():
            last = name == "conv1_up"
            why = _in_refusal(blk, not last, not last)
            if why:
                return "%s: %s" % (name, why)
        for g in _IGEVPP_GATES:
            fa = getattr(m, "feature_att_" + g).feat_att
            why = _in_refusal(fa[0], True, True)
            if why:
                return "feature_att_%s: %s" % (g, why)
            try:
                _Packed(fa[1])
            except NotImplementedError as exc:
                return "feature_att_%s: %s" % (g, exc)
        return None

    def serves(self, x, features):
        """True when the kernels run this call: every layer is the one they implement (no affine or tracked instance norm, slope
        0.01, the reference's kernel sizes, strides and flags) and the volume and the features have the shapes the graph
        concatenates and gates (the reference's own torch.cat and broadcast would refuse any other)."""
        if self._why is not None or x.dim() != 5 or len(features) < 4:
            return False
        if any(p.device != x.device for p in self.module.parameters()):
            return False
        b, c, d, h, w = x.shape
        l = dict(self._blocks())
        if c != l["conv0"].conv.in_channels or d * h * w > (1 << 24):        # moments count voxels exactly in fp32
            return False
        ext = [(d, h, w)]                                                      # extents of the four levels
        for _ in range(3):
            ext.append(tuple((e - 1) // 2 + 1 for e in ext[-1]))
        if any(tuple(2 * e for e in ext[k + 1]) != ext[k] for k in (1, 2)):   # the deconvs land on the skip levels of agg_0 / agg_1
            return False
        att = [self.module.feature_att_4, self.module.feature_att_8, self.module.feature_att_16, self.module.feature_att_32]
        return all(f.dim() == 4 and tuple(f.shape) == (b, a.feat_att[0].conv.in_channels) + e[1:]
                   for f, a, e in zip(features, att, ext))

    def _pack(self):
        self.l = {name: _Packed(blk.conv) for name, blk in self._blocks()}
        self.att = {g: _InstanceFeatureAtt(getattr(self.module, "feature_att_" + g)) for g in _IGEVPP_GATES}

    def __call__(self, x, features):
        if self._why is not None:
            raise NotImplementedError("openstereo_b200: IGEV++ hourglass: %s" % self._why)
        x = self._check(x)
        if any(p.device != x.device for p in self.module.parameters()):
            raise RuntimeError("openstereo_b200: IGEV++ hourglass: the module's parameters are not on %s" % x.device)
        self._ensure(x.device)
        f = [self._check(t) for t in features[:4]]
        l, att = self.l, self.att
        k3, dc, pw = ops.conv3d_k3_in, ops.deconv3d_in, ops.conv3d_1x1_in
        c0, s0 = k3(x, l["conv0"].w, moments=True)
        g4 = att["4"](f[0])
        y, s = k3(c0, l["conv1.0"].w, 2, s0, g4, moments=True)
        c1, s1 = k3(y, l["conv1.1"].w, 1, s, moments=True)
        g8 = att["8"](f[1])
        y, s = k3(c1, l["conv2.0"].w, 2, s1, g8, moments=True)
        c2, s2 = k3(y, l["conv2.1"].w, 1, s, moments=True)
        g16 = att["16"](f[2])
        y, s = k3(c2, l["conv3.0"].w, 2, s2, g16, moments=True)
        c3, s3 = k3(y, l["conv3.1"].w, 1, s, moments=True)
        g32 = att["32"](f[3])
        y, s = dc(c3, l["conv3_up"].w, 4, s3, g32, moments=True)
        # torch.cat((conv3_up, conv2), 1) -> agg_0 without the concat: the up slab has no gate, the skip slab feature_att_16's
        y, s = pw(y, l["agg_0.0"].w, s, None, c2, s2, g16, moments=True)
        y, s = k3(y, l["agg_0.1"].w, 1, s, moments=True)
        c2, s2 = k3(y, l["agg_0.2"].w, 1, s, moments=True)
        gu16 = att["up_16"](f[2])
        y, s = dc(c2, l["conv2_up"].w, 4, s2, gu16, moments=True)
        y, s = pw(y, l["agg_1.0"].w, s, None, c1, s1, g8, moments=True)
        y, s = k3(y, l["agg_1.1"].w, 1, s, moments=True)
        c1, s1 = k3(y, l["agg_1.2"].w, 1, s, moments=True)
        gu8 = att["up_8"](f[1])
        return dc(c1, l["conv1_up"].w, 4, s1, gu8)
