"""The rest of the IGEV-Stereo / StereoBase update block on the library (DESIGN.md section 4.16): the motion encoder
(igev/update.py:75-94 == stereobase/gru_blocks.py:233-251), the disparity head (igev/update.py:17-25 == gru_blocks.py:271-281) and
mask_feat_4 (igev/update.py:123-125 == gru_blocks.py:304-306).  The 3x3 layers run on the wgmma convolutions (osb_conv2d_k3_tc_fwd,
3xFP16 split) with channels-last fp32 intermediates, the three shapes they do not serve on the library's fp32 CUDA-core kernels:

    MotionEncoderEngine  (disp (B,1,H,W), corr (B,Cc,H,W)) -> (B,128,H,W)
        cor  = relu(convc2(relu(convc1(corr))))         osb_conv3d_1x1_bn_act_fwd on the lookup's NCHW output, pack, tc Cout 64
        dsp  = relu(convd2(relu(convd1(disp))))         convd1 (7x7, 1 -> 64) as the depthwise osb_dwconv2d_fwd over disp
                                                        broadcast to 64 planes, pack, tc Cout 64
        part = conv(cor, W[:, :64]) + b                 conv's weight zero-padded from 127 to 128 output channels, K split in two
        out  = relu(conv(dsp, W[:, 64:]) + part)        NCHW output with the channels-last residual: relu(conv(cat(cor, dsp)))
        out[:, 127] = disp                              the reference's torch.cat([out, disp])
    DispHeadEngine       net0 (B,128,H,W) -> (B,1,H,W)
        one channels-last pack; conv1 + bias + relu as two Cout 128 launches (one per half of its 256 channels, NCHW);
        conv2 + bias as two osb_conv3d_k3_bn_act_fwd launches (D = 1), the second adding the first as its residual
    MaskFeatEngine       net0 -> (B,Cout,H,W): one pack, one Cout 32 (IGEV, StereoBase) or Cout 64 (IGEV++) launch with bias + relu
                         and NCHW output

MonSter's mix2 update blocks (monster/update.py) add MixMotionEncoderEngine (BasicMotionEncoder_mix2); their ConvGRUs, disparity and
mask heads are IGEV's modules.  IGEV++'s update block (igevpp/update.py) adds GeoEncoderEngine (geo_encoder0/1/2) and DispEncoderEngine (encoder); its ConvGRUs and
disparity head are IGEV's modules and run on gru.ConvGRUEngine and DispHeadEngine as they are.

patch.py installs them as per-instance forward overrides of update_block.encoder / disp_head / mask_feat_4 and runs the reference's
own forward for every shape or hyper-parameter no kernel serves (route_ok, the engines' serves()).
"""
import torch

from . import ops
from .aggregation import _Engine


def route_ok(w):
    """True when the wgmma kernels serve every tensor-core layer of the three modules at image width w (the 64 -> 64, 64 -> 128 and
    128 -> 128 layers on the 16-channel-chunk kernels, 128 -> 32 on any): W >= OSB_TC_MIN_WIDTH."""
    return (all(ops.conv2d_tc_kc(cin, cout, w) == 16 for cin, cout in ((64, 64), (64, 128), (128, 128)))
            and ops.conv2d_tc_kc(128, 32, w) != 0)


def _is_conv(c, cin, cout, k):
    return (isinstance(c, torch.nn.Conv2d) and c.in_channels == cin and c.out_channels == cout and c.kernel_size == (k, k)
            and c.padding == (k // 2, k // 2) and c.stride == (1, 1) and c.dilation == (1, 1) and c.groups == 1
            and c.padding_mode == "zeros")


def _bias(conv, pad_to=None):
    b = torch.zeros(conv.out_channels, device=conv.weight.device) if conv.bias is None else conv.bias.detach().float()
    if pad_to is not None:
        b = torch.cat((b, b.new_zeros(pad_to - b.numel())))
    return b.contiguous()


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


class MotionEncoderEngine(_Engine):
    """BasicMotionEncoder.forward(disp, corr) on the library (module docstring)."""

    def _pack(self):
        m = self.module
        w = m.conv.weight.detach().float()
        w = torch.cat((w, w.new_zeros((1,) + tuple(w.shape[1:]))), 0)           # 127 -> 128 output channels, row 127 zero
        self.c1, self.bc1 = m.convc1.weight.detach().float()[:, :, 0, 0].t().contiguous(), _bias(m.convc1)     # (Cin, 64)
        self.c2, self.bc2 = ops.pack_tc_weight_2d(m.convc2.weight, 16), _bias(m.convc2)
        self.d1, self.bd1 = m.convd1.weight.detach().float()[:, 0].contiguous(), _bias(m.convd1)            # (64, 7, 7)
        self.d2, self.bd2 = ops.pack_tc_weight_2d(m.convd2.weight, 16), _bias(m.convd2)
        self.wc, self.wd, self.b = ops.pack_tc_weight_2d(w[:, :64], 16), ops.pack_tc_weight_2d(w[:, 64:], 16), _bias(m.conv, 128)

    def serves(self, disp, corr):
        m = self.module
        return (disp.dim() == 4 and corr.dim() == 4 and disp.shape[1] == 1 and disp.shape[0] == corr.shape[0]
                and disp.shape[2:] == corr.shape[2:] and _is_conv(m.convc1, corr.shape[1], 64, 1) and _is_conv(m.convc2, 64, 64, 3)
                and _is_conv(m.convd1, 1, 64, 7) and _is_conv(m.convd2, 64, 64, 3) and _is_conv(m.conv, 128, 127, 3)
                and route_ok(disp.shape[-1]))

    def __call__(self, disp, corr):
        self._ensure(disp.device)
        mon = ops.TcOverflowMonitor.get(disp.device)
        mon.check()
        dtype = torch.promote_types(_conv_dtype(disp, corr), disp.dtype)        # the reference's torch.cat([out, disp])
        d = _f32(disp)
        cor = ops.conv3d_1x1(_f32(corr), self.c1, None, self.bc1, act=ops.ACT_RELU)
        cor = ops.conv2d_k3_tc(ops.nchw_to_nhwc_cat([cor]), self.c2, None, self.bc2, act=ops.ACT_RELU)
        dsp = ops.dwconv2d(d.expand(-1, 64, -1, -1).contiguous(), self.d1, None, self.bd1, act=ops.ACT_RELU)
        dsp = ops.conv2d_k3_tc(ops.nchw_to_nhwc_cat([dsp]), self.d2, None, self.bd2, act=ops.ACT_RELU)
        part = ops.conv2d_k3_tc(cor, self.wc, None, self.b)
        out = ops.conv2d_k3_tc(dsp, self.wd, None, None, part, ops.ACT_RELU, out_nhwc=False, res_nhwc=True)
        out[:, 127:].copy_(d)
        mon.poll()
        return out.to(dtype)


class DispHeadEngine(_Engine):
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

    def __call__(self, x):
        self._ensure(x.device)
        mon = ops.TcOverflowMonitor.get(x.device)
        mon.check()
        dtype = _conv_dtype(x)
        xn = ops.nchw_to_nhwc_cat([_f32(x)])
        h0 = ops.conv2d_k3_tc(xn, self.w1[0], None, self.b1[0], act=ops.ACT_RELU, out_nhwc=False)
        h1 = ops.conv2d_k3_tc(xn, self.w1[1], None, self.b1[1], act=ops.ACT_RELU, out_nhwc=False)
        y = ops.conv3d_k3(h0.unsqueeze(2), self.w2[0], None, self.b2)
        y = ops.conv3d_k3(h1.unsqueeze(2), self.w2[1], None, None, y).squeeze(2)
        mon.poll()
        return y.to(dtype)


class MaskFeatEngine(_Engine):
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

    def __call__(self, x):
        self._ensure(x.device)
        mon = ops.TcOverflowMonitor.get(x.device)
        mon.check()
        dtype = _conv_dtype(x)
        kc = ops.conv2d_tc_kc(128, self.module[0].out_channels, x.shape[-1])
        if kc not in self.w:
            self.w[kc] = ops.pack_tc_weight_2d(self.module[0].weight, kc)
        y = ops.conv2d_k3_tc(ops.nchw_to_nhwc_cat([_f32(x)]), self.w[kc], None, self.b, act=ops.ACT_RELU, out_nhwc=False)
        mon.poll()
        return y.to(dtype)


def _tc_serves(w, *shapes):
    """True when a wgmma instantiation serves every (Cin, Cout) 3x3 layer at image width w.  For the shapes of the IGEV++ engines
    (Cout 32 or 128) that is W >= OSB_TC_MIN_WIDTH."""
    return all(ops.conv2d_tc_kc(cin, cout, w) != 0 for cin, cout in shapes)


def _pad_rows(w, rows):
    """(Cout, Cin, k, k) -> (rows, Cin, k, k): zero output channels appended (they compute exact zeros)."""
    return torch.cat((w, w.new_zeros((rows - w.shape[0],) + tuple(w.shape[1:]))), 0)


class GeoEncoderEngine(_Engine):
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

    def __call__(self, geo):
        self._ensure(geo.device)
        mon = ops.TcOverflowMonitor.get(geo.device)
        mon.check()
        dtype = _conv_dtype(geo)
        x = ops.conv3d_1x1(_f32(geo), self.g1, None, self.bg1, act=ops.ACT_RELU)
        y = ops.conv2d_k3_tc(ops.nchw_to_nhwc_cat([x]), self.g2, None, self.bg2, out_nhwc=False)
        mon.poll()
        return y[:, :96].to(dtype)


class DispEncoderEngine(_Engine):
    """IGEV++'s BasicDispEncoder.forward(disp, corr) (igevpp/update.py:82-100) on the library, MotionEncoderEngine's plan at IGEV++'s
    widths:

        cor  = relu(convc2(relu(convc1(corr))))     convc1 (Cc -> 128) on the CUDA-core 1x1 from the NCHW input, pack, convc2
                                                    (128 -> 96) padded to 128 output channels (exact zeros), kept channels-last
        dsp  = relu(convd2(relu(convd1(disp))))     convd1 (7x7, 1 -> 32) as the depthwise kernel over disp broadcast to 32 planes,
                                                    pack, convd2 (32 -> 32) on the Cout-32 wgmma kernels
        part = conv(cor, W[:, :96] | 0) + b         conv's weight padded from 127 to 128 output channels; the cor half gets zero
                                                    columns for cor's 32 pad channels
        out  = relu(conv(dsp, W[:, 96:]) + part)    NCHW output with the channels-last residual: relu(conv(cat(cor, dsp)))
        out[:, 127] = disp                          the reference's torch.cat([out, disp])
    """

    def _pack(self):
        m = self.module
        self.c1, self.bc1 = m.convc1.weight.detach().float()[:, :, 0, 0].t().contiguous(), _bias(m.convc1)     # (Cin, 128)
        self.c2, self.bc2 = ops.pack_tc_weight_2d(_pad_rows(m.convc2.weight.detach().float(), 128), 16), _bias(m.convc2, 128)
        self.d1, self.bd1 = m.convd1.weight.detach().float()[:, 0].contiguous(), _bias(m.convd1)            # (32, 7, 7)
        self.d2, self.bd2 = {}, _bias(m.convd2)                                 # K chunk -> packed convd2 (W' = 128: 32, else 16)
        w = _pad_rows(m.conv.weight.detach().float(), 128)                      # 127 -> 128 output channels, row 127 zero
        wc = torch.cat((w[:, :96], w.new_zeros(128, 32, 3, 3)), 1)              # cor's pad channels 96..127 meet zero columns
        self.wc, self.wd, self.b = ops.pack_tc_weight_2d(wc, 16), ops.pack_tc_weight_2d(w[:, 96:], 16), _bias(m.conv, 128)

    def serves(self, disp, corr):
        m = self.module
        return (disp.dim() == 4 and corr.dim() == 4 and disp.shape[1] == 1 and disp.shape[0] == corr.shape[0]
                and disp.shape[2:] == corr.shape[2:] and _is_conv(m.convc1, corr.shape[1], 128, 1) and _is_conv(m.convc2, 128, 96, 3)
                and _is_conv(m.convd1, 1, 32, 7) and _is_conv(m.convd2, 32, 32, 3) and _is_conv(m.conv, 128, 127, 3)
                and _tc_serves(disp.shape[-1], (128, 128), (32, 32), (32, 128)))

    def __call__(self, disp, corr):
        self._ensure(disp.device)
        mon = ops.TcOverflowMonitor.get(disp.device)
        mon.check()
        dtype = torch.promote_types(_conv_dtype(disp, corr), disp.dtype)        # the reference's torch.cat([out, disp])
        d = _f32(disp)
        kc = ops.conv2d_tc_kc(32, 32, d.shape[-1])
        if kc not in self.d2:
            self.d2[kc] = ops.pack_tc_weight_2d(self.module.convd2.weight, kc)
        cor = ops.conv3d_1x1(_f32(corr), self.c1, None, self.bc1, act=ops.ACT_RELU)
        cor = ops.conv2d_k3_tc(ops.nchw_to_nhwc_cat([cor]), self.c2, None, self.bc2, act=ops.ACT_RELU)
        dsp = ops.dwconv2d(d.expand(-1, 32, -1, -1).contiguous(), self.d1, None, self.bd1, act=ops.ACT_RELU)
        dsp = ops.conv2d_k3_tc(ops.nchw_to_nhwc_cat([dsp]), self.d2[kc], None, self.bd2, act=ops.ACT_RELU)
        part = ops.conv2d_k3_tc(cor, self.wc, None, self.b)
        out = ops.conv2d_k3_tc(dsp, self.wd, None, None, part, ops.ACT_RELU, out_nhwc=False, res_nhwc=True)
        out[:, 127:].copy_(d)
        mon.poll()
        return out.to(dtype)


class MixMotionEncoderEngine(_Engine):
    """MonSter's BasicMotionEncoder_mix2.forward(disp, corr, flaw_stereo, disp_mono, corr_mono, flaw_mono) (monster/update.py:523-561)
    on the library, MotionEncoderEngine's plan once per branch (stereo: convc1 / convc2 / convd1 / convd2 / conv; mono: the *_mono
    layers):

        cor  = relu(convc2(relu(convc1(cat(corr, flaw)))))   convc1 (162 + 96 -> 64) on the CUDA-core 1x1 over its two NCHW inputs
                                                            (the concatenation is never built), pack, tc Cout 64
        dsp  = relu(convd2(relu(convd1(disp))))             convd1 (7x7, 1 -> 64) as the depthwise kernel over disp broadcast to
                                                            64 planes, pack, tc Cout 64
        part = conv(cor, W[:, :64]) + b                     conv's weight zero-padded from 63 to 64 output channels, K split in two
        out  = relu(conv(dsp, W[:, 64:]) + part)            NCHW output with the channels-last residual: relu(conv(cat(cor, dsp)))
        out[:, 63] = disp                                   the reference's cat: channel 63 <- disp, channel 127 <- disp_mono

    The two 64-channel NCHW halves are joined by one torch.cat into the module's (B, 128, H, W) output.
    """

    _BRANCHES = ("", "_mono")

    def _pack(self):
        m = self.module
        self.w = []
        for sfx in self._BRANCHES:
            c1, c2, d1, d2, conv = (getattr(m, n + sfx) for n in ("convc1", "convc2", "convd1", "convd2", "conv"))
            w = _pad_rows(conv.weight.detach().float(), 64)                      # 63 -> 64 output channels, row 63 zero
            self.w.append(dict(c1=c1.weight.detach().float()[:, :, 0, 0].t().contiguous(), bc1=_bias(c1),    # (Cin, 64)
                               c2=ops.pack_tc_weight_2d(c2.weight, 16), bc2=_bias(c2),
                               d1=d1.weight.detach().float()[:, 0].contiguous(), bd1=_bias(d1),               # (64, 7, 7)
                               d2=ops.pack_tc_weight_2d(d2.weight, 16), bd2=_bias(d2),
                               wc=ops.pack_tc_weight_2d(w[:, :64], 16), wd=ops.pack_tc_weight_2d(w[:, 64:], 16), b=_bias(conv, 64)))

    def serves(self, disp, corr, flaw, disp_mono, corr_mono, flaw_mono):
        m = self.module
        ts = (disp, corr, flaw, disp_mono, corr_mono, flaw_mono)
        if not all(t.dim() == 4 and t.shape[0] == disp.shape[0] and t.shape[2:] == disp.shape[2:] for t in ts):
            return False
        if disp.shape[1] != 1 or disp_mono.shape[1] != 1 or corr.shape[1] != corr_mono.shape[1] or flaw.shape[1] != flaw_mono.shape[1]:
            return False
        cin = corr.shape[1] + flaw.shape[1]
        return (all(_is_conv(getattr(m, "convc1" + s), cin, 64, 1) and _is_conv(getattr(m, "convc2" + s), 64, 64, 3)
                    and _is_conv(getattr(m, "convd1" + s), 1, 64, 7) and _is_conv(getattr(m, "convd2" + s), 64, 64, 3)
                    and _is_conv(getattr(m, "conv" + s), 128, 63, 3) for s in self._BRANCHES)
                and route_ok(disp.shape[-1]))

    def _branch(self, p, d, corr, flaw):
        cor = ops.conv3d_1x1(_f32(corr), p["c1"], None, p["bc1"], act=ops.ACT_RELU, x1=_f32(flaw))
        cor = ops.conv2d_k3_tc(ops.nchw_to_nhwc_cat([cor]), p["c2"], None, p["bc2"], act=ops.ACT_RELU)
        dsp = ops.dwconv2d(d.expand(-1, 64, -1, -1).contiguous(), p["d1"], None, p["bd1"], act=ops.ACT_RELU)
        dsp = ops.conv2d_k3_tc(ops.nchw_to_nhwc_cat([dsp]), p["d2"], None, p["bd2"], act=ops.ACT_RELU)
        part = ops.conv2d_k3_tc(cor, p["wc"], None, p["b"])
        out = ops.conv2d_k3_tc(dsp, p["wd"], None, None, part, ops.ACT_RELU, out_nhwc=False, res_nhwc=True)
        out[:, 63:].copy_(d)
        return out

    def __call__(self, disp, corr, flaw, disp_mono, corr_mono, flaw_mono):
        self._ensure(disp.device)
        mon = ops.TcOverflowMonitor.get(disp.device)
        mon.check()
        # the reference's torch.cat([out, disp, out_mono, disp_mono]) promotes the convolutions' dtype with both disparities'
        dtype = torch.promote_types(torch.promote_types(_conv_dtype(disp, corr, flaw, disp_mono, corr_mono, flaw_mono), disp.dtype),
                                    disp_mono.dtype)
        out = torch.cat((self._branch(self.w[0], _f32(disp), corr, flaw), self._branch(self.w[1], _f32(disp_mono), corr_mono, flaw_mono)), 1)
        mon.poll()
        return out.to(dtype)
