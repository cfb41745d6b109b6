"""ConvGRU update cell of IGEV-Stereo and StereoBase on the wgmma convolutions (igev/update.py:28-42 ==
stereobase/gru_blocks.py:254-268; DESIGN.md section 4.15):

    z  = sigmoid(convz([h, x]) + cz)
    r  = sigmoid(convr([h, x]) + cr)
    q  = tanh(convq([r * h, x]) + cq)
    h' = (1 - z) h + z q                                  x = torch.cat(x_list, 1)

Each conv's input channels split into the h block and the x block, and the partial sums chain through the epilogue's residual:

    zx = conv(x, Wz_x) + b_z + cz      rx = ...      qx = ...                      (three launches over x, NCHW context views)
    z  = sigmoid(conv(h, Wz_h) + zx)                 rh = sigmoid(conv(h, Wr_h) + rx) * h
    h' = h + z * (tanh(conv(rh, Wq_h) + qx) - h)                                   (NCHW output)

Same MACs as the reference; h and the x_list are packed channels-last once per call (osb_ncdhw_to_ndhwc_slice), every
intermediate stays channels-last fp32.  Hidden 128 at W >= OSB_TC_MIN_WIDTH only (route_ok); patch.py runs the reference's own
forward for every other shape.
"""
import torch

from . import ops
from .aggregation import _Engine

HIDDEN = 128


def route_ok(hidden, cin, w):
    """True when the wgmma kernels serve a ConvGRU with this hidden size, total input channels (h + x) and image width."""
    cx = cin - hidden
    return (hidden == HIDDEN and cx >= 16 and cx % 16 == 0 and ops.conv2d_tc_kc(hidden, hidden, w) == 16
            and ops.conv2d_tc_kc(cx, hidden, w) == 16)


def pack_gru_conv(conv, hidden):
    """One of convz / convr / convq -> (h block, x block, bias): the (Cout, hidden + Cx, 3, 3) weight's two column blocks, each
    packed as a one-plane 3x3x3 weight (taps at kd = 1) for the 16-channel-chunk kernels."""
    w = conv.weight.detach().float()
    bias = None if conv.bias is None else conv.bias.detach().float().contiguous()
    return ops.pack_tc_weight_2d(w[:, :hidden], 16), ops.pack_tc_weight_2d(w[:, hidden:], 16), bias


class ConvGRUEngine(_Engine):
    """Packs convz / convr / convq of a reference ConvGRU module (re-packed when a parameter changes) and runs its forward."""

    def _pack(self):
        m = self.module
        hidden = m.convz.out_channels
        self.w = {k: pack_gru_conv(getattr(m, "conv" + k), hidden) for k in "zrq"}

    def serves(self, h, x_list):
        cin = h.shape[1] + sum(t.shape[1] for t in x_list)
        c = self.module.convz
        return (c.kernel_size == (3, 3) and c.padding == (1, 1) and c.stride == (1, 1) and c.dilation == (1, 1) and c.in_channels == cin
                and route_ok(self.module.convz.out_channels, cin, h.shape[-1]))

    def __call__(self, h, cz, cr, cq, *x_list):
        self._ensure(h.device)
        mon = ops.TcOverflowMonitor.get(h.device)
        mon.check()
        dtype = torch.promote_types(torch.promote_types(h.dtype, cz.dtype), cq.dtype)   # the reference's result dtype

        def f32(t):
            return t.detach().float().contiguous()

        def ctx(t):                                      # NCHW context, a channel split() view read in place when it is fp32
            t = t.detach().float()
            return t if tuple(t.stride()[1:]) == (t.shape[2] * t.shape[3], t.shape[3], 1) else t.contiguous()

        hn = ops.nchw_to_nhwc_cat([f32(h)])
        xn = ops.nchw_to_nhwc_cat([f32(t) for t in x_list])
        (zh, zxw, zb), (rhw, rxw, rb), (qh, qxw, qb) = self.w["z"], self.w["r"], self.w["q"]
        zx = ops.conv2d_k3_tc_gru(xn, zxw, zb, ctx(cz), res_nhwc=False)
        rx = ops.conv2d_k3_tc_gru(xn, rxw, rb, ctx(cr), res_nhwc=False)
        qx = ops.conv2d_k3_tc_gru(xn, qxw, qb, ctx(cq), res_nhwc=False)
        z = ops.conv2d_k3_tc_gru(hn, zh, None, zx, ops.ACT_SIGMOID)
        rh = ops.conv2d_k3_tc_gru(hn, rhw, None, rx, ops.ACT_SIGMOID, mul=hn)
        out = ops.conv2d_k3_tc_gru(rh, qh, None, qx, ops.ACT_TANH, blend=(z, hn), out_nhwc=False)
        mon.poll()
        return out.to(dtype)
