"""The rest of the IGEV-Stereo / StereoBase update block on the library (DESIGN.md section 4.16): the motion encoder
(igev/update.py:75-94 == stereobase/gru_blocks.py:233-251), the disparity head (igev/update.py:17-25 == gru_blocks.py:271-281) and
mask_feat_4 (igev/update.py:123-125 == gru_blocks.py:304-306).  The 3x3 layers run on the wgmma convolutions (osb_conv2d_k3_tc_fwd,
3xFP16 split) with channels-last fp32 intermediates, the three shapes they do not serve on the library's fp32 CUDA-core kernels:

    MotionEncoderEngine  one branch (disp (B,1,H,W), corr (B,Cc,H,W)) -> (B,C,H,W), at the widths of _ENCODER_PLANS:
        cor  = relu(convc2(relu(convc1(corr))))         osb_conv3d_1x1_bn_act_fwd on the lookup's NCHW output, pack, tc convc2
                                                        (zero-padded to `rows` output channels where it is narrower)
        dsp  = relu(convd2(relu(convd1(disp))))         convd1 (7x7, 1 -> Cd) as the depthwise osb_dwconv2d_fwd over disp
                                                        broadcast to Cd planes, pack, tc convd2
        part = conv(cor, W[:, :Cc2] | 0) + b            conv's weight zero-padded from C - 1 to C output channels, K split in two;
                                                        the cor half has zero columns for cor's pad channels
        out  = relu(conv(dsp, W[:, Cc2:]) + part)       NCHW output with the channels-last residual: relu(conv(cat(cor, dsp)))
        out[:, C - 1] = disp                            the reference's torch.cat([out, disp])
      BasicMotionEncoder (IGEV, StereoBase) and IGEV++'s BasicDispEncoder run one branch; MonSter's BasicMotionEncoder_mix2 runs
      one per layer suffix "" / "_mono" (its convc1 reads corr and flaw as two NCHW blocks, the concatenation is never built) and
      joins the two 64-channel halves by one torch.cat into the module's (B, 128, H, W) output.
    DispHeadEngine       net0 (B,128,H,W) -> (B,1,H,W)
        one channels-last pack; conv1 + bias + relu as two Cout 128 launches (one per half of its 256 channels, NCHW);
        conv2 + bias as two osb_conv3d_k3_bn_act_fwd launches (D = 1), the second adding the first as its residual
    MaskFeatEngine       net0 -> (B,Cout,H,W): one pack, one Cout 32 (IGEV, StereoBase) or Cout 64 (IGEV++) launch with bias + relu
                         and NCHW output
    GeoEncoderEngine     IGEV++'s geo_encoder0/1/2 (igevpp/update.py:72-80)

MonSter's mix2 update blocks (monster/update.py) use IGEV's ConvGRUs, disparity and mask heads; IGEV++'s update block
(igevpp/update.py) uses IGEV's ConvGRUs and disparity head.  All run on gru.ConvGRUEngine and the engines here as they are.

patch.py installs them as per-instance forward overrides of the update blocks' modules and runs the reference's own forward for
every shape or hyper-parameter no kernel serves (route_ok, the engines' serves()).
"""
import torch

from . import ops
from .aggregation import _Engine


def route_ok(w):
    """True when the wgmma kernels serve every tensor-core layer of the three modules at image width w (the 64 -> 64, 64 -> 128 and
    128 -> 128 layers on the 16-channel-chunk kernels, 128 -> 32 on any): W >= OSB_TC_MIN_WIDTH."""
    return (all(ops.conv2d_tc_kc(cin, cout, w) == 16 for cin, cout in ((64, 64), (64, 128), (128, 128)))
            and ops.conv2d_tc_kc(128, 32, w) != 0)


def _tc_serves(w, *shapes):
    """True when a wgmma instantiation serves every (Cin, Cout) 3x3 layer at image width w.  For the shapes of the IGEV++ engines
    (Cout 32 or 128) that is W >= OSB_TC_MIN_WIDTH."""
    return all(ops.conv2d_tc_kc(cin, cout, w) != 0 for cin, cout in shapes)


def _is_conv(c, cin, cout, k):
    return (isinstance(c, torch.nn.Conv2d) and c.in_channels == cin and c.out_channels == cout and c.kernel_size == (k, k)
            and c.padding == (k // 2, k // 2) and c.stride == (1, 1) and c.dilation == (1, 1) and c.groups == 1
            and c.padding_mode == "zeros")


def _bias(conv, pad_to=None):
    b = torch.zeros(conv.out_channels, device=conv.weight.device) if conv.bias is None else conv.bias.detach().float()
    if pad_to is not None:
        b = torch.cat((b, b.new_zeros(pad_to - b.numel())))
    return b.contiguous()


def _pad_rows(w, rows):
    """(Cout, Cin, k, k) -> (rows, Cin, k, k): zero output channels appended (they compute exact zeros)."""
    return torch.cat((w, w.new_zeros((rows - w.shape[0],) + tuple(w.shape[1:]))), 0)


def _conv_dtype(*tensors):
    """dtype of a reference Conv2d's output on these inputs: the autocast dtype where autocast is on, else the inputs' promotion."""
    if torch.is_autocast_enabled("cuda"):
        return torch.get_autocast_dtype("cuda")
    dtype = tensors[0].dtype
    for t in tensors[1:]:
        dtype = torch.promote_types(dtype, t.dtype)
    return dtype


def _f32(t):
    return t.detach().float().contiguous()


class _BlockEngine(_Engine):
    """An update-block module's forward on the library: re-pack if needed, report a past fp16 overflow of the tensor-core
    convolutions, run _run, schedule the next overflow read, return in _dtype(*args), the dtype the reference's forward returns.

    amp=True (patch(model, amp=True)): under CUDA autocast, fp16 or bf16, the engine's tensor-core 3x3 layers run at autocast
    accuracy -- one fp16 MMA per product (ops.conv2d_k3_tc precision="f16", DESIGN.md section 4.20) -- as the reference's autocast
    convolutions do.  fp16 operands serve bf16 autocast too: finer mantissa, and the same range guard as the fp32 mode.  Outside
    autocast, and with amp=False, every layer keeps the fp32-accurate product.  The CUDA-core layers, the dtypes returned and the
    overflow monitor are the same either way."""

    def __init__(self, module, amp=False):
        super().__init__(module)
        self.amp = bool(amp)

    def _precision(self):
        """precision= of this call's tensor-core launches."""
        return "f16" if self.amp and torch.is_autocast_enabled("cuda") else "fp32"

    def __call__(self, *args):
        device = args[0].device
        self._ensure(device)
        mon = ops.TcOverflowMonitor.get(device)
        mon.check()
        out = self._run(*args)
        mon.poll()
        return out.to(self._dtype(*args))

    def _dtype(self, *args):
        return _conv_dtype(*args)


# The layer plans MotionEncoderEngine serves, keyed by the output channels of convc1, convc2, convd1 and conv and by whether the
# module has the mix2 "_mono" branch -> (rows convc2 is packed with, the image widths the wgmma kernels serve at).  conv is packed
# with one more output row, a zero one: the kernel's output channel that disp is copied into.
_ENCODER_PLANS = {
    (64, 64, 64, 127, False): (64, route_ok),                                                      # BasicMotionEncoder
    (128, 96, 32, 127, False): (128, lambda w: _tc_serves(w, (128, 128), (32, 32), (32, 128))),    # BasicDispEncoder (no Cout 96)
    (64, 64, 64, 63, True): (64, route_ok),                                                        # BasicMotionEncoder_mix2
}


class MotionEncoderEngine(_BlockEngine):
    """BasicMotionEncoder.forward(disp, corr), BasicDispEncoder.forward(disp, corr) and BasicMotionEncoder_mix2.forward(disp, corr,
    flaw_stereo, disp_mono, corr_mono, flaw_mono) (monster/update.py:523-561) on the library (module docstring).  self.w holds one
    dict of packed weights per branch, named after the layers: c1 / bc1 (convc1), c2 / bc2, d1 / bd1, d2 / bd2, wc / wd / b
    (conv).  A one-branch module's dict is also the engine's attributes (engine.wc, ...)."""

    def _layout(self):
        """(convc1, convc2, convd1, conv output channels), the branch suffixes, the plan (None: not one of _ENCODER_PLANS)."""
        m = self.module
        widths = tuple(getattr(getattr(m, n, None), "out_channels", None) for n in ("convc1", "convc2", "convd1", "conv"))
        mix = hasattr(m, "conv_mono")
        return widths, ("", "_mono") if mix else ("",), _ENCODER_PLANS.get(widths + (mix,))

    @staticmethod
    def _branches(args, suffixes):
        """The forward's arguments as one (disp, corr[, flaw]) tuple per branch."""
        return [tuple(args)] if len(suffixes) == 1 else [tuple(args[:3]), tuple(args[3:])]

    def _pack(self):
        m = self.module
        (_, c2, _, out), suffixes, (rows, _) = self._layout()
        self.w = []
        for s in suffixes:
            convc1, convc2, convd1, convd2, conv = (getattr(m, n + s) for n in ("convc1", "convc2", "convd1", "convd2", "conv"))
            w = _pad_rows(conv.weight.detach().float(), out + 1)
            wc = torch.cat((w[:, :c2], w.new_zeros(out + 1, rows - c2, 3, 3)), 1)                   # cor's pad channels: zero
            self.w.append(dict(c1=convc1.weight.detach().float()[:, :, 0, 0].t().contiguous(), bc1=_bias(convc1),   # (Cin, Cc1)
                               c2=ops.pack_tc_weight_2d(_pad_rows(convc2.weight.detach().float(), rows), 16),
                               bc2=_bias(convc2, rows), d1=convd1.weight.detach().float()[:, 0].contiguous(),   # (Cd, 7, 7)
                               bd1=_bias(convd1), d2=ops.pack_tc_weight_2d(convd2.weight, 16), bd2=_bias(convd2),
                               wc=ops.pack_tc_weight_2d(wc, 16), wd=ops.pack_tc_weight_2d(w[:, c2:], 16), b=_bias(conv, out + 1),
                               convd2=convd2, d2_kc={}))
        if len(self.w) == 1:
            vars(self).update(self.w[0])

    @staticmethod
    def _convd2(p, w):
        """Branch p's convd2 packed for the K chunk of image width w: the 16-channel chunk, or one packed on first use (Cd 32 at
        W' = 128: 32)."""
        kc = ops.conv2d_tc_kc(p["d2"].cout, p["d2"].cout, w)
        if kc == p["d2"].kc:
            return p["d2"]
        if kc not in p["d2_kc"]:
            p["d2_kc"][kc] = ops.pack_tc_weight_2d(p["convd2"].weight, kc)
        return p["d2_kc"][kc]

    def serves(self, *args):
        m = self.module
        (c1, c2, cd, out), suffixes, plan = self._layout()
        disp = args[0]
        if plan is None or not all(t.dim() == 4 and t.shape[0] == disp.shape[0] and t.shape[2:] == disp.shape[2:] for t in args):
            return False
        branches = self._branches(args, suffixes)
        planes = [t.shape[1] for t in branches[0][1:]]                 # corr[, flaw]: the same in every branch
        if any(b[0].shape[1] != 1 or [t.shape[1] for t in b[1:]] != planes for b in branches):
            return False
        return (all(_is_conv(getattr(m, "convc1" + s), sum(planes), c1, 1) and _is_conv(getattr(m, "convc2" + s), c1, c2, 3)
                    and _is_conv(getattr(m, "convd1" + s), 1, cd, 7) and _is_conv(getattr(m, "convd2" + s), cd, cd, 3)
                    and _is_conv(getattr(m, "conv" + s), c2 + cd, out, 3) for s in suffixes)
                and plan[1](disp.shape[-1]))

    def _branch(self, p, d, corr, flaw=None, prec="fp32"):
        """One branch on the packed weights p: d is disp in fp32, channels-last intermediates, NCHW output."""
        cor = ops.conv3d_1x1(_f32(corr), p["c1"], None, p["bc1"], act=ops.ACT_RELU, x1=None if flaw is None else _f32(flaw))
        cor = ops.conv2d_k3_tc(ops.nchw_to_nhwc_cat([cor]), p["c2"], None, p["bc2"], act=ops.ACT_RELU, precision=prec)
        dsp = ops.dwconv2d(d.expand(-1, p["d1"].shape[0], -1, -1).contiguous(), p["d1"], None, p["bd1"], act=ops.ACT_RELU)
        dsp = ops.conv2d_k3_tc(ops.nchw_to_nhwc_cat([dsp]), self._convd2(p, d.shape[-1]), None, p["bd2"], act=ops.ACT_RELU,
                               precision=prec)
        part = ops.conv2d_k3_tc(cor, p["wc"], None, p["b"], precision=prec)
        out = ops.conv2d_k3_tc(dsp, p["wd"], None, None, part, ops.ACT_RELU, out_nhwc=False, res_nhwc=True, precision=prec)
        out[:, -1:].copy_(d)
        return out

    def _run(self, *args):
        prec = self._precision()
        outs = [self._branch(p, _f32(b[0]), *b[1:], prec=prec) for p, b in zip(self.w, self._branches(args, self._layout()[1]))]
        return outs[0] if len(outs) == 1 else torch.cat(outs, 1)

    def _dtype(self, *args):
        dtype = _conv_dtype(*args)                                     # promoted with every disp: the reference's torch.cat
        for b in self._branches(args, self._layout()[1]):
            dtype = torch.promote_types(dtype, b[0].dtype)
        return dtype


class DispHeadEngine(_BlockEngine):
    """DispHead.forward(x) = conv2(relu(conv1(x))) on the library (module docstring)."""

    def _pack(self):
        m = self.module
        w, b = m.conv1.weight, _bias(m.conv1)
        self.w1 = [ops.pack_tc_weight_2d(w[:128], 16), ops.pack_tc_weight_2d(w[128:], 16)]
        self.b1 = [b[:128].contiguous(), b[128:].contiguous()]
        w5 = m.conv2.weight.detach().float().new_zeros(1, 256, 3, 3, 3)
        w5[:, :, 1] = m.conv2.weight.detach().float()                          # 2D taps at kd = 1 of a D = 1 volume
        self.w2, self.b2 = [ops.pack_conv_weight(w5[:, :128]), ops.pack_conv_weight(w5[:, 128:])], _bias(m.conv2)

    def serves(self, x):
        m = self.module
        return (x.dim() == 4 and _is_conv(m.conv1, x.shape[1], 256, 3) and x.shape[1] == 128 and _is_conv(m.conv2, 256, 1, 3)
                and route_ok(x.shape[-1]))

    def _run(self, x):
        xn, prec = ops.nchw_to_nhwc_cat([_f32(x)]), self._precision()
        h0 = ops.conv2d_k3_tc(xn, self.w1[0], None, self.b1[0], act=ops.ACT_RELU, out_nhwc=False, precision=prec)
        h1 = ops.conv2d_k3_tc(xn, self.w1[1], None, self.b1[1], act=ops.ACT_RELU, out_nhwc=False, precision=prec)
        y = ops.conv3d_k3(h0.unsqueeze(2), self.w2[0], None, self.b2)
        return ops.conv3d_k3(h1.unsqueeze(2), self.w2[1], None, None, y).squeeze(2)


class MaskFeatEngine(_BlockEngine):
    """mask_feat_4 = Sequential(Conv2d(128, Cout, 3, padding=1), ReLU) on the library (module docstring): Cout 32 (IGEV-Stereo,
    StereoBase) or 64 (IGEV++)."""

    def _pack(self):
        self.w = {}                                                             # K chunk -> packed weight (Cout 32 at W' = 128: 32, else 16)
        self.b = _bias(self.module[0])

    def serves(self, x):
        m = self.module
        cout = getattr(m[0], "out_channels", 0) if len(m) else 0
        return (len(m) == 2 and isinstance(m[1], torch.nn.ReLU) and x.dim() == 4 and x.shape[1] == 128 and cout in (32, 64)
                and _is_conv(m[0], 128, cout, 3) and route_ok(x.shape[-1]) and ops.conv2d_tc_kc(128, cout, x.shape[-1]) != 0)

    def _run(self, x):
        kc = ops.conv2d_tc_kc(128, self.module[0].out_channels, x.shape[-1])
        if kc not in self.w:
            self.w[kc] = ops.pack_tc_weight_2d(self.module[0].weight, kc)
        return ops.conv2d_k3_tc(ops.nchw_to_nhwc_cat([_f32(x)]), self.w[kc], None, self.b, act=ops.ACT_RELU, out_nhwc=False,
                                precision=self._precision())                # kc = 32 (conv3d_tc.cu) keeps the 3-term product


class GeoEncoderEngine(_BlockEngine):
    """IGEV++'s GeoEncoder.forward(geo) = convg2(relu(convg1(geo))) (igevpp/update.py:72-80) on the library:

        x = relu(convg1(geo))       osb_conv3d_1x1_bn_act_fwd on the lookup's NCHW output, in place (geo_planes -> 128)
        y = convg2(x)               one channels-last pack, one Cout-128 wgmma launch with NCHW output: the 128 -> 96 weight and bias
                                    are zero-padded to 128 rows (there is no Cout-96 instantiation at W' = 128 or at general widths)
        return y[:, :96]            a view; channels 96..127 are exact zeros
    """

    def _pack(self):
        m = self.module
        self.g1, self.bg1 = m.convg1.weight.detach().float()[:, :, 0, 0].t().contiguous(), _bias(m.convg1)     # (Cin, 128)
        self.g2, self.bg2 = ops.pack_tc_weight_2d(_pad_rows(m.convg2.weight.detach().float(), 128), 16), _bias(m.convg2, 128)

    def serves(self, geo):
        m = self.module
        return (geo.dim() == 4 and _is_conv(m.convg1, geo.shape[1], 128, 1) and _is_conv(m.convg2, 128, 96, 3)
                and _tc_serves(geo.shape[-1], (128, 128)))

    def _run(self, geo):
        x = ops.conv3d_1x1(_f32(geo), self.g1, None, self.bg1, act=ops.ACT_RELU)
        return ops.conv2d_k3_tc(ops.nchw_to_nhwc_cat([x]), self.g2, None, self.bg2, out_nhwc=False, precision=self._precision())[:, :96]


# BasicDispEncoder's and BasicMotionEncoder_mix2's engine, by the module class's name
DispEncoderEngine = MixMotionEncoderEngine = MotionEncoderEngine
