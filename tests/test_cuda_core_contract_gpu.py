"""GPU: contract of every fp32 CUDA-core convolution (csrc/conv3d.cu, lightstereo.cu, msnet.cu, flavours.cu).

REGISTRY has one or more rows per instantiation or launch path (tests/test_host_logic_cpu.py checks that every launch_conv_k3 /
launch_deconv / launch_conv1x1_cat / launch_mbv2 template list and every kernel launched directly with <<< in those files has a
row).  Each row names the entry point family, the channels, a small input shape with partial tiles in every tiled dimension and
the instantiation it must reach, in the template spelling of the source.  For every row:
  routing      torch.profiler sees exactly one kernel of this library, the row's instantiation;
  accuracy     weights scaled per output channel by 2^k (k over [-12, 12]) times a non-power-of-two factor; folded BN, residual,
               activation, gate and sigmoid where the entry point has them, against an fp64 reference of the whole operation: error
               per output channel <= 1e-5 x that channel's max |want| (an error in a small channel cannot hide behind a large one);
               outputs that end in ReLU6 or a sigmoid measure the error against sum |w.x| instead (saturated_magnitude);
  store paths  entry points with a vec_ok rule (3-D conv, transposed conv, NCDHW 1x1) run once with every pointer 16-byte aligned
               and Wo % 4 == 0 (vector epilogue), then with the output, the residual and the gate each at a 4-byte offset (the rule
               sends the whole launch to the scalar epilogue): all runs pass the accuracy check and agree bit for bit;
  bounds       the output lives inside a buffer whose output region starts as NaN, guarded on each side by 4 KB of sentinels;
               every output element is written and no sentinel changes;
  determinism  two launches of the same row are bit-identical (no kernel here uses atomics: a difference is a race);
  item loop    the grid-stride channels-last 1x1 launchers run at persistent-grid caps 1, 7 and uncapped, so one CTA walks many
               tiles with its staged weights and pipelined loads carried over: outputs are bit-identical across caps.
test_refusals: every input an entry point refuses returns its error code and launches nothing.
"""
import re
import zlib
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ACT_NONE, ACT_RELU, ACT_LEAKY, ACT_RELU6 = 0, 1, 2, 3
OSB_EINVAL, OSB_EUNSUPPORTED = 1, 3
GUARD = 1024                            # sentinel floats on each side of an output region (4 KB, keeps 16-byte alignment)
SENTINEL = -1234.5
TOL = 1e-5                              # per-channel error bar, relative to the channel's max |want|

# fam: k3 = osb_conv3d_k3_bn_act_fwd, dc = osb_deconv3d_bn_act_fwd, pw = osb_conv3d_1x1_bn_act_fwd, nd = osb_conv1x1_ndhwc_fwd,
# cat = osb_conv1x1_ndhwc_cat_fwd, c1 = osb_conv3d_k3_c1_ndhwc_fwd, dw = osb_dwconv2d_fwd, dc2 = osb_deconv2d_k3s2_fwd,
# mb = osb_mbv2_block3d_fwd, fa = osb_feature_att_gate_fwd.  shape = INPUT (B, D, H, W), or (B, H, W) for the 2-D families.
# ep: epilogue operands (sc scale, sh shift, res residual, gate; fa: sc1 sh1 sc2 sh2).
Row = namedtuple("Row", "id fam variant cin cout shape opts")


def R(rid, fam, variant, cin, cout, shape, **opts):
    return Row(rid, fam, variant, cin, cout, shape, opts)


REGISTRY = [
    # conv3d.cu launch_conv_k3<S,TCO,NCG,TD,TH,CI>: output tile TD x TH x 32.  Stride 1: D 5, H 6, W 36 against 4 x 4 x 32; stride 2:
    # odd input extents 5 x 9 x 71 -> 3 x 5 x 36 against 2 x 4 x 32.  Cin 13 / 11 leaves a partial input-channel chunk.  The
    # 24-channel groups serve Cout % 24 == 0 && Cout % 32 != 0 (24, 48, 144); 96 is a multiple of 32 and takes the general branch.
    R("k3-co1-s1", "k3", "launch_conv_k3<1,1,1,4,4,8>", 13, 1, (2, 5, 6, 36), stride=1, ep="sc sh res gate", act=ACT_RELU),
    R("k3-co5-s1", "k3", "launch_conv_k3<1,1,1,4,4,8>", 13, 5, (2, 5, 6, 36), stride=1, ep="sh res", act=ACT_LEAKY),
    R("k3-co1-s2", "k3", "launch_conv_k3<2,1,1,2,4,4>", 11, 1, (2, 5, 9, 71), stride=2, ep="sc sh", act=ACT_NONE),
    R("k3-co3-s2", "k3", "launch_conv_k3<2,1,1,2,4,4>", 11, 3, (2, 5, 9, 71), stride=2, ep="sc gate", act=ACT_RELU),
    R("k3-co24-s1", "k3", "launch_conv_k3<1,8,3,4,4,8>", 13, 24, (2, 5, 6, 36), stride=1, ep="sh res", act=ACT_LEAKY),
    R("k3-co144-s1", "k3", "launch_conv_k3<1,8,3,4,4,8>", 13, 144, (2, 5, 6, 36), stride=1, ep="sc", act=ACT_NONE),
    R("k3-co144-s2", "k3", "launch_conv_k3<2,8,3,2,4,4>", 11, 144, (2, 5, 9, 71), stride=2, ep="sh res gate", act=ACT_RELU),
    R("k3-co48-s2", "k3", "launch_conv_k3<2,8,3,2,4,4>", 11, 48, (2, 5, 9, 71), stride=2, ep="sc sh res gate", act=ACT_LEAKY),
    R("k3-co96-s1", "k3", "launch_conv_k3<1,8,4,4,4,8>", 13, 96, (2, 5, 6, 36), stride=1, ep="sc sh res gate", act=ACT_LEAKY),
    R("k3-co96-s2", "k3", "launch_conv_k3<2,8,4,2,4,4>", 11, 96, (2, 5, 9, 71), stride=2, ep="sc res", act=ACT_LEAKY),
    R("k3-co40-s1", "k3", "launch_conv_k3<1,8,4,4,4,8>", 13, 40, (2, 5, 6, 36), stride=1, ep="sc res", act=ACT_RELU),
    R("k3-co64-s1", "k3", "launch_conv_k3<1,8,4,4,4,8>", 13, 64, (2, 5, 6, 36), stride=1, ep="sh gate", act=ACT_LEAKY),
    R("k3-co64-s2", "k3", "launch_conv_k3<2,8,4,2,4,4>", 11, 64, (2, 5, 9, 71), stride=2, ep="sc sh res gate", act=ACT_LEAKY),
    R("k3-co40-s2", "k3", "launch_conv_k3<2,8,4,2,4,4>", 11, 40, (2, 5, 9, 71), stride=2, ep="sh", act=ACT_RELU),
    # conv3d.cu launch_deconv<KS,CI>: output 2D x 2H x 2W = 6 x 6|10 x 68 against the 4 x 4 x 64 tile; Cout 20 / 12 against 16
    R("dc3", "dc", "launch_deconv<3,8>", 13, 20, (2, 3, 3, 34), k=3, ep="sc sh res", act=ACT_RELU),
    R("dc3-shift", "dc", "launch_deconv<3,8>", 13, 20, (2, 3, 3, 34), k=3, ep="sh", act=ACT_LEAKY),
    R("dc4", "dc", "launch_deconv<4,8>", 11, 12, (2, 3, 5, 34), k=4, ep="sc sh res", act=ACT_LEAKY),
    R("dc4-scale", "dc", "launch_deconv<4,8>", 11, 12, (2, 3, 5, 34), k=4, ep="sc res", act=ACT_RELU),
    # conv3d.cu conv3d_1x1_kernel: W % 8 != 0 (a partial voxel octet per row), Cout not a multiple of the 32-channel CTA
    R("pw-one", "pw", "conv3d_1x1_kernel", 40, 24, (2, 3, 5, 20), ep="sc sh res", act=ACT_RELU6),
    R("pw-two", "pw", "conv3d_1x1_kernel", 64, 40, (2, 3, 5, 20), c0=24, ep="sh gate", act=ACT_LEAKY),
    R("pw-wide", "pw", "conv3d_1x1_kernel", 300, 33, (2, 2, 3, 28), c0=136, ep="sc sh res gate", act=ACT_RELU, sigmoid=1),
    R("pw-2d", "pw", "conv3d_1x1_kernel", 48, 32, (2, 1, 7, 44), ep="sc sh", act=ACT_RELU6, sigmoid=1),
    # conv3d.cu channels-last 1x1, grid-stride over 32-voxel groups: V = 2030 / 1974, not multiples of 32
    R("nd32", "nd", "conv1x1_ndhwc_32_kernel", 32, 32, (2, 5, 7, 29), ep="sc sh", act=ACT_RELU),
    R("nd64", "nd", "conv1x1_ndhwc_kernel<64,64>", 64, 64, (2, 3, 7, 47), ep="sh", act=ACT_LEAKY),
    # conv3d.cu channels-last 1x1 over two slabs, persistent over 128-voxel tiles: V = 1000 / 777; unequal splits and one slab
    R("cat192", "cat", "launch_conv1x1_cat<192,96>", 192, 96, (2, 4, 5, 25), c0=64, ep="sc sh", act=ACT_LEAKY),
    R("cat128", "cat", "launch_conv1x1_cat<128,64>", 128, 64, (1, 3, 7, 37), c0=32, ep="sc", act=ACT_RELU),
    R("cat128-one", "cat", "launch_conv1x1_cat<128,64>", 128, 64, (1, 3, 7, 37), c0=128, ep="sh", act=ACT_NONE),
    # conv3d.cu classifier head, tile 2 x 4 x 32
    R("c1", "c1", "conv3d_k3_c1_ndhwc_kernel<32>", 32, 1, (2, 5, 7, 37), ep="sc sh"),
    R("c1-plain", "c1", "conv3d_k3_c1_ndhwc_kernel<32>", 32, 1, (1, 3, 5, 33), ep=""),
    # lightstereo.cu: tiles 32 x 8 output pixels (depthwise) / input pixels (transposed)
    R("dw3-s1", "dw", "dwconv2d_kernel", 12, 12, (2, 11, 37), k=(3, 3), stride=1, ep="sc sh res", act=ACT_RELU6),
    R("dw3-s2", "dw", "dwconv2d_kernel", 12, 12, (2, 19, 69), k=(3, 3), stride=2, ep="sc sh", act=ACT_RELU),
    R("dw1x7-s1", "dw", "dwconv2d_kernel", 10, 10, (2, 9, 41), k=(1, 7), stride=1, ep="sh res", act=ACT_NONE),
    R("dw11x1-s2", "dw", "dwconv2d_kernel", 10, 10, (2, 19, 69), k=(11, 1), stride=2, ep="sc res", act=ACT_LEAKY),
    R("dc2", "dc2", "deconv2d_k3s2_kernel", 40, 20, (2, 9, 35), ep="sc sh res", act=ACT_RELU),
    R("dc2-relu6", "dc2", "deconv2d_k3s2_kernel", 13, 8, (1, 8, 32), ep="sh", act=ACT_RELU6),
    # msnet.cu launch_mbv2<CIN,CHID,COUT,S,TH,TW>: output 5 x 6 x 19 (stride 1) / 3 x 5 x 10 (stride 2), partial in H and W; the
    # depth march is split into chunks at this grid size.  Every row runs NCDHW and NDHWC in and out, with and without residual.
    R("mb-40-120-32", "mb", "launch_mbv2<40,120,32,1,4,16>", 40, 32, (2, 5, 6, 19), chid=120, stride=1),
    R("mb-32-96-32", "mb", "launch_mbv2<32,96,32,1,4,16>", 32, 32, (2, 5, 6, 19), chid=96, stride=1),
    R("mb-32-64-32", "mb", "launch_mbv2<32,64,32,1,4,16>", 32, 32, (2, 5, 6, 19), chid=64, stride=1),
    R("mb-32-64-64-s2", "mb", "launch_mbv2<32,64,64,2,4,8>", 32, 64, (2, 5, 9, 19), chid=64, stride=2),
    R("mb-64-128-64", "mb", "launch_mbv2<64,128,64,1,4,8>", 64, 64, (2, 5, 6, 19), chid=128, stride=1),
    R("mb-64-128-128-s2", "mb", "launch_mbv2<64,128,128,2,4,4>", 64, 128, (2, 5, 9, 19), chid=128, stride=2),
    R("mb-128-256-128", "mb", "launch_mbv2<128,256,128,1,4,4>", 128, 128, (2, 5, 6, 19), chid=256, stride=1),
    # flavours.cu FeatureAtt gate, 8-pixel tiles (HW = 35 / 27): a padded channel plan, and hidden / output loops of several passes
    R("fa-pad", "fa", "feature_att_gate_kernel", 48, 24, (2, 5, 7), ch=24, cpad=32, ep="sc1 sh1 sh2", act=ACT_LEAKY),
    R("fa-wide", "fa", "feature_att_gate_kernel", 160, 144, (2, 3, 9), ch=80, cpad=160, ep="sh1 sc2 sh2", act=ACT_RELU),
]

VEC_RULE = ("k3", "dc", "pw")           # entry points whose vec_ok rule picks the vector or the scalar epilogue
CAPPED = ("nd", "cat")                  # launchers whose grid follows osb_set_persistent_grid_cap


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, ops
    return _lib, ops


@pytest.fixture
def grid_cap(osb):
    _, ops = osb
    yield ops.set_persistent_grid_cap
    ops.set_persistent_grid_cap(0)


def channel_scales(cout, g):
    """2^k x a non-power-of-two factor per output channel, k spread over [-12, 12]."""
    k = torch.linspace(-12, 12, cout).round()[torch.randperm(cout, generator=g)]
    return torch.ldexp(torch.ones(cout), k.int()) * (1.0 + 0.9 * torch.rand(cout, generator=g)) * 0.77


def activate(y, act):
    if act == ACT_RELU:
        return F.relu(y)
    if act == ACT_LEAKY:
        return F.leaky_relu(y, 0.01)
    if act == ACT_RELU6:
        return y.clamp(0.0, 6.0)
    return y


def bcast(v, ndim, cdim):
    shape = [1] * ndim
    shape[cdim] = -1
    return v.double().view(shape)


def ptr(t):
    return None if t is None else t.data_ptr()


class Case:
    """One launch of a row: device operands, the fp64 reference of its output (in the output's layout, channel axis `cdim`) and
    `fn(y, residual, gate)`, a direct call of the C entry point with caller-chosen output / residual / gate addresses."""

    def __init__(self, name, want, cdim, fn, res=None, gate=None, mag=None):
        self.name, self.want, self.cdim, self.fn, self.mag = name, want, cdim, fn, mag
        self.numel = want.numel()
        self.res = None if res is None else res.float().contiguous().cuda()
        self.gate = None if gate is None else gate.float().contiguous().cuda()
        self._keep = []

    def _shifted(self, t, off):
        """t's data at a 4 * off byte offset from a fresh allocation (off = 0: t itself)."""
        if t is None or off == 0:
            return ptr(t)
        buf = torch.empty(t.numel() + off, device="cuda")
        buf[off:].copy_(t.flatten())
        self._keep.append(buf)
        return buf.data_ptr() + 4 * off

    def guarded(self, y_off=0):
        """Fresh output buffer: sentinels | output region (NaN) | sentinels, the region starting 4 * y_off bytes past the guard."""
        buf = torch.full((GUARD + y_off + self.numel + GUARD,), SENTINEL, device="cuda")
        buf[GUARD + y_off:GUARD + y_off + self.numel] = float("nan")
        return buf

    def launch(self, y_off=0, res_off=0, gate_off=0):
        """-> (guarded buffer, index of the output region's first element in it)."""
        buf, lead = self.guarded(y_off), GUARD + y_off
        self.fn(buf.data_ptr() + 4 * lead, self._shifted(self.res, res_off), self._shifted(self.gate, gate_off))
        torch.cuda.synchronize()
        self._keep.clear()
        return buf, lead

    def check_bounds(self, buf, lead, what):
        bits = buf.view(torch.int32)
        sent = torch.tensor([SENTINEL]).view(torch.int32).item()
        assert (bits[:lead] == sent).all() and (bits[lead + self.numel:] == sent).all(), "%s: a store left the output region" % what
        inner = buf[lead:lead + self.numel]
        assert not torch.isnan(inner).any(), "%s: %d output elements never written" % (what, int(torch.isnan(inner).sum()))

    def channel_ratio(self, inner):
        """-> per output channel max |got - want| / max |want| (a channel whose reference is all zero must be exactly zero); for an
        output that ends in ReLU6 or a sigmoid the denominator also covers the channel's max of `mag` (saturated_magnitude)."""
        c = self.want.shape[self.cdim]
        per_channel = lambda t: t.movedim(self.cdim, 0).reshape(c, -1)          # noqa: E731
        got = per_channel(inner.double().cpu().view(self.want.shape))
        want = per_channel(self.want)
        err = (got - want).abs().amax(dim=1)
        scale = want.abs().amax(dim=1)
        if self.mag is not None:
            scale = torch.maximum(scale, per_channel(self.mag).amax(dim=1))
        ratio = err / scale.clamp(min=1e-300)
        ratio[(scale == 0) & (err == 0)] = 0.0
        return ratio


def epilogue_operands(row, g, out_shape, cdim, cs):
    """fp32 scale / shift / residual / gate of the row's `ep` list (None where absent); residual and shift scaled like the channel."""
    ep = row.opts.get("ep", "").split()
    c = out_shape[cdim]
    sc = torch.rand(c, generator=g) + 0.5 if "sc" in ep else None
    sh = 0.1 * cs * torch.randn(c, generator=g) if "sh" in ep else None
    res = 0.3 * bcast(cs, len(out_shape), cdim).float() * torch.randn(out_shape, generator=g) if "res" in ep else None
    return sc, sh, res


def ref_epilogue(conv, cdim, sc, sh, res, act, gate=None, sigmoid=False):
    """fp64: act(conv * sc + sh + res) * gate, then the optional sigmoid."""
    y = conv
    if sc is not None:
        y = y * bcast(sc, y.dim(), cdim)
    if sh is not None:
        y = y + bcast(sh, y.dim(), cdim)
    if res is not None:
        y = y + res.double()
    y = activate(y, act)
    if gate is not None:
        y = y * gate.double()
    return torch.sigmoid(y) if sigmoid else y


def saturated_magnitude(conv_abs, cdim, sc, sh, res, act, sigmoid=False):
    """Bar scale of an output that ends in ReLU6 or a sigmoid (None for any other).  Those cap a channel's max |want| at 6 (or 1)
    while its pre-activation sums, scaled per channel by up to 2^12, stay large: where such a sum cancels into the unclamped range,
    an fp32 sum correct to a few ulp of sum |w.x| is off by more than 1e-5 x max |want| (measured: up to 5e-5).  For these outputs
    a channel's bar scale also covers L x max(|scale| sum |w.x| + |shift| + |residual|), where conv_abs = sum |w.x| is the fp64
    convolution of |x| with |w| and L the activation's Lipschitz constant (1 for ReLU6, 1/4 for the sigmoid; the gate is <= 1)."""
    if act != ACT_RELU6 and not sigmoid:
        return None
    m = conv_abs
    if sc is not None:
        m = m * bcast(sc.abs(), m.dim(), cdim)
    if sh is not None:
        m = m + bcast(sh.abs(), m.dim(), cdim)
    if res is not None:
        m = m + res.double().abs()
    return 0.25 * m if sigmoid else m


def cases(osb, row, g):
    lib, ops = osb
    call, o = lib.call, row.opts
    s = lambda: torch.cuda.current_stream().cuda_stream           # noqa: E731
    act = o.get("act", ACT_NONE)
    ep = o.get("ep", "").split()
    cs = channel_scales(row.cout, g)
    dev = lambda t: None if t is None else t.float().contiguous().cuda()      # noqa: E731

    if row.fam in ("k3", "dc"):
        b, d, h, w = row.shape
        x = torch.randn(b, row.cin, d, h, w, generator=g)
        if row.fam == "k3":
            st, k = o["stride"], 3
            wt = torch.randn(row.cout, row.cin, 3, 3, 3, generator=g) * (27 * row.cin) ** -0.5 * cs.view(-1, 1, 1, 1, 1)
            conv = F.conv3d(x.double(), wt.double(), stride=st, padding=1)
            wp = ops.pack_conv_weight(wt).cuda()
        else:
            k = o["k"]
            wt = torch.randn(row.cin, row.cout, k, k, k, generator=g) * (row.cin * k ** 3 / 8) ** -0.5 * cs.view(1, -1, 1, 1, 1)
            conv = F.conv_transpose3d(x.double(), wt.double(), stride=2, padding=1, output_padding=1 if k == 3 else 0)
            wp = ops.pack_deconv_weight(wt).cuda()
        sc, sh, res = epilogue_operands(row, g, conv.shape, 1, cs)
        gate = None
        if "gate" in ep:                                            # (B, Cout, Ho, Wo), broadcast over the output depth
            gate = torch.sigmoid(torch.randn(b, row.cout, conv.shape[3], conv.shape[4], generator=g))
        want = ref_epilogue(conv, 1, sc, sh, res, act, None if gate is None else gate.unsqueeze(2))
        xd, scd, shd = dev(x), dev(sc), dev(sh)
        if row.fam == "k3":
            fn = lambda y, r, gt: call("osb_conv3d_k3_bn_act_fwd", xd.data_ptr(), wp.data_ptr(), ptr(scd), ptr(shd), r, gt, y, b,  # noqa
                                       row.cin, row.cout, d, h, w, st, act, s())
        else:
            fn = lambda y, r, gt: call("osb_deconv3d_bn_act_fwd", xd.data_ptr(), wp.data_ptr(), ptr(scd), ptr(shd), r, y, b,  # noqa
                                       row.cin, row.cout, d, h, w, k, act, s())
        return [Case(row.id, want, 1, fn, res, gate)]

    if row.fam == "pw":
        b, d, h, w = row.shape
        c0 = o.get("c0", row.cin)
        x = torch.randn(b, row.cin, d, h, w, generator=g)
        wt = torch.randn(row.cin, row.cout, generator=g) * row.cin ** -0.5 * cs.view(1, -1)
        conv = torch.einsum("bcdhw,co->bodhw", x.double(), wt.double())
        sc, sh, res = epilogue_operands(row, g, conv.shape, 1, cs)
        gate = torch.sigmoid(torch.randn(b, row.cout, h, w, generator=g)) if "gate" in ep else None
        want = ref_epilogue(conv, 1, sc, sh, res, act, None if gate is None else gate.unsqueeze(2), o.get("sigmoid", 0))
        mag = saturated_magnitude(torch.einsum("bcdhw,co->bodhw", x.double().abs(), wt.double().abs()), 1, sc, sh, res, act,
                                  o.get("sigmoid", 0))
        x0, x1 = dev(x[:, :c0]), dev(x[:, c0:]) if c0 < row.cin else None
        wp, scd, shd = dev(wt), dev(sc), dev(sh)
        fn = lambda y, r, gt: call("osb_conv3d_1x1_bn_act_fwd", x0.data_ptr(), ptr(x1), c0, wp.data_ptr(), ptr(scd), ptr(shd), r, gt,  # noqa
                                   y, b, row.cin, row.cout, d, h, w, act, o.get("sigmoid", 0), s())
        return [Case(row.id, want, 1, fn, res, gate, mag)]

    if row.fam in ("nd", "cat"):
        v = 1
        for n in row.shape:
            v *= n
        x = torch.randn(v, row.cin, generator=g)
        wt = torch.randn(row.cin, row.cout, generator=g) * row.cin ** -0.5 * cs.view(1, -1)
        conv = x.double() @ wt.double()
        sc, sh, _ = epilogue_operands(row, g, conv.shape, 1, cs)
        want = ref_epilogue(conv, 1, sc, sh, None, act)
        wp, scd, shd = dev(wt), dev(sc), dev(sh)
        if row.fam == "nd":
            xd = dev(x)
            fn = lambda y, r, gt: call("osb_conv1x1_ndhwc_fwd", xd.data_ptr(), wp.data_ptr(), ptr(scd), ptr(shd), y, v, row.cin,  # noqa
                                       row.cout, act, s())
        else:
            c0 = o["c0"]
            x0, x1 = dev(x[:, :c0]), dev(x[:, c0:]) if c0 < row.cin else None
            fn = lambda y, r, gt: call("osb_conv1x1_ndhwc_cat_fwd", x0.data_ptr(), ptr(x1), c0, row.cin - c0, wp.data_ptr(),  # noqa
                                       ptr(scd), ptr(shd), y, v, row.cout, act, s())
        return [Case(row.id, want, 1, fn)]

    if row.fam == "c1":
        b, d, h, w = row.shape
        x = torch.randn(b, row.cin, d, h, w, generator=g)
        wt = torch.randn(1, row.cin, 3, 3, 3, generator=g) * (27 * row.cin) ** -0.5 * 0.37
        conv = F.conv3d(x.double(), wt.double(), padding=1)
        sc, sh, _ = epilogue_operands(row, g, conv.shape, 1, torch.ones(1))
        want = ref_epilogue(conv, 1, sc, sh, None, ACT_NONE)
        xd, wp, scd, shd = dev(x.permute(0, 2, 3, 4, 1)), ops.pack_c1_weight(wt).cuda(), dev(sc), dev(sh)
        fn = lambda y, r, gt: call("osb_conv3d_k3_c1_ndhwc_fwd", xd.data_ptr(), wp.data_ptr(), ptr(scd), ptr(shd), y, b, row.cin,  # noqa
                                   d, h, w, s())
        return [Case(row.id, want, 1, fn)]

    if row.fam == "dw":
        b, h, w = row.shape
        (kh, kw), st = o["k"], o["stride"]
        x = torch.randn(b, row.cin, h, w, generator=g)
        wt = torch.randn(row.cin, kh, kw, generator=g) * (kh * kw) ** -0.5 * cs.view(-1, 1, 1)
        conv = F.conv2d(x.double(), wt.double().unsqueeze(1), stride=st, padding=(kh // 2, kw // 2), groups=row.cin)
        sc, sh, res = epilogue_operands(row, g, conv.shape, 1, cs)
        want = ref_epilogue(conv, 1, sc, sh, res, act)
        mag = saturated_magnitude(F.conv2d(x.double().abs(), wt.double().abs().unsqueeze(1), stride=st, padding=(kh // 2, kw // 2),
                                           groups=row.cin), 1, sc, sh, res, act)
        xd, wp, scd, shd = dev(x), dev(wt), dev(sc), dev(sh)
        fn = lambda y, r, gt: call("osb_dwconv2d_fwd", xd.data_ptr(), wp.data_ptr(), ptr(scd), ptr(shd), r, y, b, row.cin, h, w,  # noqa
                                   kh, kw, st, act, s())
        return [Case(row.id, want, 1, fn, res, mag=mag)]

    if row.fam == "dc2":
        b, h, w = row.shape
        x = torch.randn(b, row.cin, h, w, generator=g)
        wt = torch.randn(row.cin, row.cout, 3, 3, generator=g) * (row.cin * 9 / 4) ** -0.5 * cs.view(1, -1, 1, 1)
        conv = F.conv_transpose2d(x.double(), wt.double(), stride=2, padding=1, output_padding=1)
        sc, sh, res = epilogue_operands(row, g, conv.shape, 1, cs)
        want = ref_epilogue(conv, 1, sc, sh, res, act)
        mag = saturated_magnitude(F.conv_transpose2d(x.double().abs(), wt.double().abs(), stride=2, padding=1, output_padding=1), 1,
                                  sc, sh, res, act)
        xd, wp, scd, shd = dev(x), ops.pack_deconv2d_weight(wt).cuda(), dev(sc), dev(sh)
        fn = lambda y, r, gt: call("osb_deconv2d_k3s2_fwd", xd.data_ptr(), wp.data_ptr(), ptr(scd), ptr(shd), r, y, b, row.cin,  # noqa
                                   row.cout, h, w, act, s())
        return [Case(row.id, want, 1, fn, res, mag=mag)]

    if row.fam == "mb":
        b, d, h, w = row.shape
        chid, st = o["chid"], o["stride"]
        x = torch.randn(b, row.cin, d, h, w, generator=g)
        w_exp = torch.randn(row.cin, chid, generator=g) * row.cin ** -0.5
        w_dw = torch.randn(chid, 1, 3, 3, 3, generator=g) * 27 ** -0.5
        w_proj = torch.randn(chid, row.cout, generator=g) * chid ** -0.5 * cs.view(1, -1)
        s1, s2, s3 = (torch.rand(n, generator=g) + 0.5 for n in (chid, chid, row.cout))
        b1, b2 = 0.1 * torch.randn(chid, generator=g), 0.1 * torch.randn(chid, generator=g)
        b3 = 0.1 * cs * torch.randn(row.cout, generator=g)
        hid = activate(torch.einsum("bcdhw,ce->bedhw", x.double(), w_exp.double()) * bcast(s1, 5, 1) + bcast(b1, 5, 1), ACT_RELU6)
        hid = F.conv3d(hid, w_dw.double(), stride=st, padding=1, groups=chid)     # zero-pads the hidden tensor
        hid = activate(hid * bcast(s2, 5, 1) + bcast(b2, 5, 1), ACT_RELU6)
        proj = torch.einsum("bedhw,eo->bodhw", hid, w_proj.double()) * bcast(s3, 5, 1) + bcast(b3, 5, 1)
        res = 0.3 * cs.view(1, -1, 1, 1, 1) * torch.randn(proj.shape, generator=g)
        wd = [dev(t) for t in (w_exp, s1, b1, w_dw.view(chid, 27).t(), s2, b2, w_proj, s3, b3)]
        out = []
        for in_cl, out_cl, with_res in ((0, 0, 1), (1, 1, 1), (0, 1, 0), (1, 0, 0), (0, 0, 0), (1, 1, 0), (0, 1, 1), (1, 0, 1)):
            want = proj + res.double() if with_res else proj
            r = res if with_res else None
            if out_cl:
                want = want.permute(0, 2, 3, 4, 1).contiguous()
                r = None if r is None else r.permute(0, 2, 3, 4, 1)
            xd = dev(x.permute(0, 2, 3, 4, 1) if in_cl else x)

            def fn(y, rp, gt, xd=xd, in_cl=in_cl, out_cl=out_cl):
                call("osb_mbv2_block3d_fwd", xd.data_ptr(), *[t.data_ptr() for t in wd], rp, y, b, row.cin, chid, row.cout, d, h, w, st,
                     in_cl, out_cl, s())
            name = "%s %s->%s%s" % (row.id, "ndhwc" if in_cl else "ncdhw", "ndhwc" if out_cl else "ncdhw", " +res" if with_res else "")
            out.append(Case(name, want, 4 if out_cl else 1, fn, r))
        return out

    assert row.fam == "fa"
    b, h, w = row.shape
    ch, cv, cpad = o["ch"], row.cout, o["cpad"]
    feat = torch.randn(b, row.cin, h, w, generator=g)
    w1 = torch.randn(row.cin, ch, generator=g) * row.cin ** -0.5
    w2 = torch.randn(ch, cv, generator=g) * ch ** -0.5 * cs.view(1, -1)
    sc1 = torch.rand(ch, generator=g) + 0.5 if "sc1" in ep else None
    sh1 = 0.1 * torch.randn(ch, generator=g) if "sh1" in ep else None
    sc2 = torch.rand(cv, generator=g) + 0.5 if "sc2" in ep else None
    sh2 = 0.1 * cs * torch.randn(cv, generator=g) if "sh2" in ep else None
    hid = ref_epilogue(torch.einsum("bchw,ce->behw", feat.double(), w1.double()), 1, sc1, sh1, None, act)
    gate = ref_epilogue(torch.einsum("behw,ev->bhwv", hid, w2.double()), 3, sc2, sh2, None, ACT_NONE, sigmoid=True)
    want = torch.zeros(b, h, w, cpad, dtype=torch.float64)
    want[..., :cv] = gate
    mag = torch.zeros_like(want)
    mag[..., :cv] = saturated_magnitude(torch.einsum("behw,ev->bhwv", hid.abs(), w2.double().abs()), 3, sc2, sh2, None, ACT_NONE,
                                        sigmoid=True)
    fd, w1d, w2d = dev(feat), dev(w1), dev(w2)
    ps = [dev(t) for t in (sc1, sh1, sc2, sh2)]
    fn = lambda y, r, gt: call("osb_feature_att_gate_fwd", fd.data_ptr(), w1d.data_ptr(), ptr(ps[0]), ptr(ps[1]), w2d.data_ptr(),  # noqa
                               ptr(ps[2]), ptr(ps[3]), y, b, row.cin, ch, cv, cpad, h * w, act, s())
    return [Case(row.id, want, 3, fn, mag=mag)]


def seed(row, salt=0):
    return torch.Generator().manual_seed(salt + zlib.crc32(row.id.encode()) % 10000)


@pytest.mark.timeout(180)
@pytest.mark.parametrize("row", REGISTRY, ids=[r.id for r in REGISTRY])
def test_accuracy_store_paths_bounds_determinism(osb, grid_cap, row):
    worst = 0.0
    for case in cases(osb, row, seed(row)):
        runs = [("aligned", {}, 0), ("aligned again", {}, 0)]
        if row.fam in VEC_RULE:
            assert case.want.shape[-1] % 4 == 0, "%s: Wo %% 4 != 0 would send the aligned run to the scalar path" % case.name
            runs.append(("y+4", {"y_off": 1}, 0))
            if case.res is not None:
                runs.append(("residual+4", {"res_off": 1}, 0))
            if case.gate is not None:
                runs.append(("gate+4", {"gate_off": 1}, 0))
        if row.fam in CAPPED:
            runs += [("grid cap 1", {}, 1), ("grid cap 7", {}, 7)]
        first = None
        for label, offs, cap in runs:
            what = "%s, %s" % (case.name, label)
            grid_cap(cap)
            buf, lead = case.launch(**offs)
            case.check_bounds(buf, lead, what)
            inner = buf[lead:lead + case.numel]
            ratio = case.channel_ratio(inner)
            bad = (ratio > TOL).nonzero().flatten().tolist()
            assert not bad, "%s: channels %s exceed %g of their own max (err/max %s)" % (
                what, bad[:8], TOL, [float(ratio[c]) for c in bad[:8]])
            worst = max(worst, float(ratio.max()))
            bits = inner.view(torch.int32).clone()
            if first is None:
                first = bits
            else:
                assert torch.equal(first, bits), "%s: output differs bit-wise from the first aligned, uncapped run" % what
    print("\n%-18s worst per-channel err/max %.2e" % (row.id, worst))


def kernel_of(variant):
    """Registry spelling -> the __global__ function it launches, e.g. launch_deconv<3,8> -> deconv3d_kernel<3,8>."""
    for launcher, kernel in (("launch_conv_k3", "conv3d_k3_kernel"), ("launch_deconv", "deconv3d_kernel"),
                             ("launch_conv1x1_cat", "conv1x1_ndhwc_cat_kernel"), ("launch_mbv2", "mbv2_block3d_kernel")):
        if variant.startswith(launcher + "<"):
            return kernel + variant[len(launcher):]
    return variant


@pytest.mark.timeout(120)
@pytest.mark.parametrize("row", REGISTRY, ids=[r.id for r in REGISTRY])
def test_routing(osb, row):
    from torch.profiler import ProfilerActivity, profile
    case = cases(osb, row, seed(row, 3))[0]
    buf = case.guarded()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        case.fn(buf.data_ptr() + 4 * GUARD, ptr(case.res), ptr(case.gate))
        torch.cuda.synchronize()
    names = sorted({e.name.replace(" ", "") for e in prof.events() if "osb::" in e.name})
    want = re.compile(r"osb::%s\(" % re.escape(kernel_of(row.variant)))
    assert len(names) == 1 and want.search(names[0]), "%s: launched %s, expected %s" % (row.id, names, kernel_of(row.variant))


def refusals(P, s):
    """(what, expected error code, entry point, arguments); P is a 4 MB device buffer every pointer argument refers to."""
    mis = P + 4
    nd = "osb_conv1x1_ndhwc_fwd"
    cat = "osb_conv1x1_ndhwc_cat_fwd"
    mb = "osb_mbv2_block3d_fwd"
    mbw = (P,) * 10                                              # x, w_exp, scale1, shift1, w_dw, scale2, shift2, w_proj, scale3, shift3
    return [
        ("conv1x1_ndhwc 32->64", OSB_EUNSUPPORTED, nd, (P, P, None, None, P, 64, 32, 64, ACT_NONE, s)),
        ("conv1x1_ndhwc 64->32", OSB_EUNSUPPORTED, nd, (P, P, None, None, P, 64, 64, 32, ACT_NONE, s)),
        ("conv1x1_ndhwc 16->16", OSB_EUNSUPPORTED, nd, (P, P, None, None, P, 64, 16, 16, ACT_NONE, s)),
        ("conv1x1_ndhwc y+4", OSB_EINVAL, nd, (P, P, None, None, mis, 64, 32, 32, ACT_NONE, s)),
        ("conv1x1_ndhwc act 3", OSB_EINVAL, nd, (P, P, None, None, P, 64, 32, 32, ACT_RELU6, s)),
        ("conv1x1_ndhwc_cat 64+64->96", OSB_EUNSUPPORTED, cat, (P, P, 64, 64, P, None, None, P, 64, 96, ACT_NONE, s)),
        ("conv1x1_ndhwc_cat 96+96->64", OSB_EUNSUPPORTED, cat, (P, P, 96, 96, P, None, None, P, 64, 64, ACT_NONE, s)),
        ("conv1x1_ndhwc_cat 64+64->32", OSB_EUNSUPPORTED, cat, (P, P, 64, 64, P, None, None, P, 64, 32, ACT_NONE, s)),
        ("conv1x1_ndhwc_cat C0 % 4", OSB_EINVAL, cat, (P, P, 2, 126, P, None, None, P, 64, 64, ACT_NONE, s)),
        ("conv1x1_ndhwc_cat x1 null", OSB_EINVAL, cat, (P, None, 64, 64, P, None, None, P, 64, 64, ACT_NONE, s)),
        ("conv1x1_ndhwc_cat y+4", OSB_EINVAL, cat, (P, P, 64, 64, P, None, None, mis, 64, 64, ACT_NONE, s)),
        ("conv1x1_ndhwc_cat act 3", OSB_EINVAL, cat, (P, P, 64, 64, P, None, None, P, 64, 64, ACT_RELU6, s)),
        ("mbv2 (32,64,32,2)", OSB_EINVAL, mb, mbw + (None, P + 4096, 1, 32, 64, 32, 2, 2, 2, 2, 0, 0, s)),
        ("mbv2 (40,120,32,2)", OSB_EINVAL, mb, mbw + (None, P + 4096, 1, 40, 120, 32, 2, 2, 2, 2, 0, 0, s)),
        ("mbv2 (32,96,64,1)", OSB_EINVAL, mb, mbw + (None, P + 4096, 1, 32, 96, 64, 2, 2, 2, 1, 0, 0, s)),
        ("mbv2 y aliases x", OSB_EINVAL, mb, mbw + (None, P, 1, 40, 120, 32, 2, 2, 2, 1, 0, 0, s)),
        ("mbv2 stride 3", OSB_EINVAL, mb, mbw + (None, P + 4096, 1, 40, 120, 32, 2, 2, 2, 3, 0, 0, s)),
        ("mbv2 layout 2", OSB_EINVAL, mb, mbw + (None, P + 4096, 1, 40, 120, 32, 2, 2, 2, 1, 2, 0, s)),
        ("mbv2 channels-last y+4", OSB_EINVAL, mb, mbw + (None, P + 4100, 1, 40, 120, 32, 2, 2, 2, 1, 0, 1, s)),
        ("deconv2d_k3s2 y+4", OSB_EINVAL, "osb_deconv2d_k3s2_fwd", (P, P, None, None, None, mis, 1, 8, 8, 4, 4, ACT_NONE, s)),
        ("deconv2d_k3s2 residual+4", OSB_EINVAL, "osb_deconv2d_k3s2_fwd", (P, P, None, None, mis, P, 1, 8, 8, 4, 4, ACT_NONE, s)),
        ("deconv2d_k3s2 act 4", OSB_EINVAL, "osb_deconv2d_k3s2_fwd", (P, P, None, None, None, P, 1, 8, 8, 4, 4, 4, s)),
        ("conv3d_k3_c1_ndhwc Cin 16", OSB_EUNSUPPORTED, "osb_conv3d_k3_c1_ndhwc_fwd", (P, P, None, None, P, 1, 16, 2, 2, 2, s)),
        ("conv3d_k3_c1_ndhwc Cin 64", OSB_EUNSUPPORTED, "osb_conv3d_k3_c1_ndhwc_fwd", (P, P, None, None, P, 1, 64, 2, 2, 2, s)),
        ("conv3d_k3_c1_ndhwc x+4", OSB_EINVAL, "osb_conv3d_k3_c1_ndhwc_fwd", (mis, P, None, None, P, 1, 32, 2, 2, 2, s)),
        ("conv3d_k3 act 3", OSB_EINVAL, "osb_conv3d_k3_bn_act_fwd", (P, P, None, None, None, None, P, 1, 4, 8, 2, 2, 8, 1, ACT_RELU6, s)),
        ("conv3d_k3 act -1", OSB_EINVAL, "osb_conv3d_k3_bn_act_fwd", (P, P, None, None, None, None, P, 1, 4, 8, 2, 2, 8, 1, -1, s)),
        ("conv3d_k3 stride 3", OSB_EINVAL, "osb_conv3d_k3_bn_act_fwd", (P, P, None, None, None, None, P, 1, 4, 8, 2, 2, 8, 3, 0, s)),
        ("deconv3d act 3", OSB_EINVAL, "osb_deconv3d_bn_act_fwd", (P, P, None, None, None, P, 1, 4, 8, 2, 2, 2, 3, ACT_RELU6, s)),
        ("deconv3d kernel 2", OSB_EINVAL, "osb_deconv3d_bn_act_fwd", (P, P, None, None, None, P, 1, 4, 8, 2, 2, 2, 2, ACT_NONE, s)),
        ("conv3d_1x1 act 4", OSB_EINVAL, "osb_conv3d_1x1_bn_act_fwd", (P, None, 8, P, None, None, None, None, P, 1, 8, 8, 2, 2, 8, 4, 0, s)),
        ("conv3d_1x1 split without x1", OSB_EINVAL, "osb_conv3d_1x1_bn_act_fwd",
         (P, None, 4, P, None, None, None, None, P, 1, 8, 8, 2, 2, 8, ACT_NONE, 0, s)),
        ("dwconv2d act 4", OSB_EINVAL, "osb_dwconv2d_fwd", (P, P, None, None, None, P, 1, 4, 8, 8, 3, 3, 1, 4, s)),
        ("dwconv2d 2x3 kernel", OSB_EINVAL, "osb_dwconv2d_fwd", (P, P, None, None, None, P, 1, 4, 8, 8, 2, 3, 1, ACT_NONE, s)),
        ("dwconv2d stride 3", OSB_EINVAL, "osb_dwconv2d_fwd", (P, P, None, None, None, P, 1, 4, 8, 8, 3, 3, 3, ACT_NONE, s)),
        ("feature_att_gate act 3", OSB_EINVAL, "osb_feature_att_gate_fwd", (P, P, None, None, P, None, None, P, 1, 8, 8, 8, 8, 16, 3, s)),
        ("feature_att_gate Cpad < Cv", OSB_EINVAL, "osb_feature_att_gate_fwd",
         (P, P, None, None, P, None, None, P, 1, 8, 8, 8, 4, 16, ACT_LEAKY, s)),
        ("feature_att_gate Cv % 4", OSB_EINVAL, "osb_feature_att_gate_fwd",
         (P, P, None, None, P, None, None, P, 1, 8, 8, 6, 8, 16, ACT_LEAKY, s)),
    ]


@pytest.mark.timeout(60)
def test_refusals(osb):
    lib, _ = osb
    buf = torch.zeros(1 << 20, device="cuda")                   # 4 MB: every argument list above stays inside it
    torch.cuda.synchronize()
    for what, code, name, args in refusals(buf.data_ptr(), torch.cuda.current_stream().cuda_stream):
        before = lib.launch_count()
        rc = getattr(lib.lib, name)(*args)
        assert rc == code, "%s: %s returned %d, expected %d (%s)" % (what, name, rc, code, lib.lib.osb_last_error())
        assert lib.launch_count() == before, "%s: a refused call launched a kernel" % what
    torch.cuda.synchronize()
