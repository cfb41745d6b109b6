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
Instance-norm rows (fam in-k3 / in-dc / in-pw: osb_conv3d_k3_in_fwd, osb_deconv3d_in_fwd, osb_conv3d_1x1_in_fwd) cover every
instantiation the three entry points dispatch to, with partial tiles, rows of more than 64 CTAs along grid x (the slot-merge loop of
moments_out takes several passes) and rows whose channels carry a mean offset of about 30 standard deviations (opt `offset`):
  normalised input  leaky((x - mean) * rstd) * gate as the operand, ungated, gated, and gated with the scale / shift / activation
               (and output sigmoid) the entry point accepts: run through the checks above (both store paths, bounds, determinism);
  moments out  test_instance_norm_moments_out: raw output and per-(b, channel) (mean, rstd) of the stored output in sentinel-guarded
               buffers, aligned and with y 4 bytes off (scalar epilogue) and aligned again: outputs AND statistics bit-identical, the
               workspace's counters back to 0 after every launch; output per channel within 1e-5 of fp64, mean within 1e-5 of
               |mean| + std and rstd within 1e-5 of fp64 statistics of the stored output.
CONV_PARAMS_FIELDS classifies every field of struct ConvParams as an operand / geometry field or as the instance-norm mode
(tests/test_host_logic_cpu.py).
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
    # ---- instance-norm modes (conv3d.cu, in_params): dispatch_conv_k3's six instantiations, both transposed kernels, the 1x1 over
    # one slab, two slabs and in 2D.  slots: k3 72 (4 x 6 x 3 tiles of 32 x 4 x 4), dc 70 (2 x 7 x 5 of 64 x 4 x 4), pw 65 (4160 voxel
    # octets / 64).  offset: mean offset of the input channels, in standard deviations (cancellation in the statistics)
    R("in-k3-co3-s1", "in-k3", "launch_conv_k3<1,1,1,4,4,8>", 13, 3, (2, 5, 6, 36), stride=1, act=ACT_RELU),
    R("in-k3-co5-s2", "in-k3", "launch_conv_k3<2,1,1,2,4,4>", 11, 5, (2, 5, 9, 71), stride=2, act=ACT_LEAKY),
    R("in-k3-co24-s1", "in-k3", "launch_conv_k3<1,8,3,4,4,8>", 13, 24, (2, 5, 6, 36), stride=1, act=ACT_LEAKY),
    R("in-k3-co48-s2", "in-k3", "launch_conv_k3<2,8,3,2,4,4>", 11, 48, (2, 5, 9, 71), stride=2, act=ACT_RELU),
    R("in-k3-co8-s1", "in-k3", "launch_conv_k3<1,8,4,4,4,8>", 13, 8, (2, 5, 6, 36), stride=1, act=ACT_LEAKY),
    R("in-k3-co40-s1", "in-k3", "launch_conv_k3<1,8,4,4,4,8>", 16, 40, (2, 5, 6, 36), stride=1, act=ACT_RELU),
    R("in-k3-co64-w70", "in-k3", "launch_conv_k3<1,8,4,4,4,8>", 8, 64, (1, 7, 10, 70), stride=1, act=ACT_LEAKY),
    R("in-k3-slots", "in-k3", "launch_conv_k3<1,8,4,4,4,8>", 4, 16, (1, 9, 22, 100), stride=1, act=ACT_LEAKY),
    R("in-k3-cancel", "in-k3", "launch_conv_k3<1,8,4,4,4,8>", 13, 32, (2, 5, 6, 36), stride=1, act=ACT_RELU, offset=30.0),
    R("in-k3-co16-s2", "in-k3", "launch_conv_k3<2,8,4,2,4,4>", 11, 16, (2, 5, 9, 71), stride=2, act=ACT_LEAKY),
    R("in-k3-co64-s2", "in-k3", "launch_conv_k3<2,8,4,2,4,4>", 32, 64, (2, 3, 5, 17), stride=2, act=ACT_RELU),
    R("in-dc3", "in-dc", "launch_deconv<3,8>", 13, 20, (2, 3, 3, 34), k=3, act=ACT_RELU),
    R("in-dc3-slots", "in-dc", "launch_deconv<3,8>", 4, 8, (1, 9, 13, 40), k=3, act=ACT_LEAKY),
    R("in-dc4", "in-dc", "launch_deconv<4,8>", 12, 8, (2, 3, 5, 34), k=4, act=ACT_LEAKY),
    R("in-dc4-w9", "in-dc", "launch_deconv<4,8>", 64, 32, (1, 2, 3, 9), k=4, act=ACT_RELU),
    R("in-dc4-cancel", "in-dc", "launch_deconv<4,8>", 8, 16, (1, 3, 4, 32), k=4, act=ACT_LEAKY, offset=30.0),
    R("in-pw-one", "in-pw", "conv3d_1x1_kernel", 40, 24, (2, 3, 5, 20), act=ACT_RELU6),
    R("in-pw-two", "in-pw", "conv3d_1x1_kernel", 64, 32, (2, 3, 5, 20), c0=32, act=ACT_LEAKY, sigmoid=1),
    R("in-pw-two-w30", "in-pw", "conv3d_1x1_kernel", 32, 16, (2, 6, 9, 30), c0=16, act=ACT_RELU),
    R("in-pw-2d", "in-pw", "conv3d_1x1_kernel", 96, 48, (2, 1, 7, 44), act=ACT_LEAKY),
    R("in-pw-2d-wide", "in-pw", "conv3d_1x1_kernel", 48, 96, (2, 1, 7, 44), act=ACT_RELU6, sigmoid=1),
    R("in-pw-slots", "in-pw", "conv3d_1x1_kernel", 16, 40, (1, 8, 40, 100), c0=8, act=ACT_LEAKY),
    R("in-pw-cancel", "in-pw", "conv3d_1x1_kernel", 24, 32, (2, 3, 6, 24), c0=16, act=ACT_RELU, offset=30.0),
]

VEC_RULE = ("k3", "dc", "pw", "in-k3", "in-dc", "in-pw")   # entry points whose vec_ok rule picks the vector or the scalar epilogue
IN_FAMS = ("in-k3", "in-dc", "in-pw")

# Every field of struct ConvParams (csrc/conv3d.cu): "" = an operand, geometry or launch field of every row, "in" = the instance-norm
# modes, exercised by the in-* rows.  A field that is in neither fails tests/test_host_logic_cpu.py.
CONV_PARAMS_FIELDS = {
    **{f: "" for f in ("x x1 w scale shift residual gate y B Cin Cin0 Cout D H W Do Ho Wo tiles_w tiles_h tiles_d act sigmoid_out "
                       "vec_ok").split()},
    **{f: "in" for f in "in_stats in_gate in_stats1 in_gate1 stats part counter ws_floats ws_need".split()},
}


def in_grid(row):
    """(CTAs along grid x = moments slots, channel blocks along grid y) of an instance-norm row's launch."""
    b, d, h, w = row.shape
    if row.fam == "in-k3":
        s, tco, ncg, td, th = (int(v) for v in row.variant[len("launch_conv_k3<"):-1].split(",")[:5])
        do, ho, wo = (d - 1) // s + 1, (h - 1) // s + 1, (w - 1) // s + 1
        return -(-wo // 32) * -(-ho // th) * -(-do // td), -(-row.cout // (tco * ncg))
    if row.fam == "in-dc":
        return -(-2 * w // 64) * -(-2 * h // 4) * -(-2 * d // 4), -(-row.cout // 16)
    return -(-d * h * -(-w // 8) // 64), -(-row.cout // 32)
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

    if row.fam in IN_FAMS:
        return in_cases(osb, row, g)

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


def in_input(row, g, mean=1.0, spread=2.0):
    """Input of an instance-norm row: spread * N(0, 1) + mean, plus opt `offset` standard deviations on every other channel."""
    b, d, h, w = row.shape
    x = torch.randn(b, row.cin, d, h, w, generator=g) * spread + mean
    off = row.opts.get("offset", 0.0)
    if off:
        x[:, 0::2] += off * spread * torch.sign(torch.randn(1, (row.cin + 1) // 2, 1, 1, 1, generator=g))
    return x


def in_weight(row, g, cs):
    """-> (fp32 weight in the reference's layout, packed weight on the device)."""
    from openstereo_b200 import ops
    if row.fam == "in-k3":
        wt = torch.randn(row.cout, row.cin, 3, 3, 3, generator=g) * (27 * row.cin) ** -0.5 * cs.view(-1, 1, 1, 1, 1)
        return wt, ops.pack_conv_weight(wt).cuda()
    if row.fam == "in-dc":
        k = row.opts["k"]
        wt = torch.randn(row.cin, row.cout, k, k, k, generator=g) * (row.cin * k ** 3 / 8) ** -0.5 * cs.view(1, -1, 1, 1, 1)
        return wt, ops.pack_deconv_weight(wt).cuda()
    wt = torch.randn(row.cout, row.cin, 1, 1, 1, generator=g) * row.cin ** -0.5 * cs.view(-1, 1, 1, 1, 1)
    return wt, wt.reshape(row.cout, row.cin).t().contiguous().cuda()


def in_conv64(row, x, wt):
    """fp64 convolution of an instance-norm row (the zero padding applies to the normalised, gated tensor)."""
    x, wt = x.double(), wt.double()
    if row.fam == "in-k3":
        return F.conv3d(x, wt, stride=row.opts["stride"], padding=1)
    if row.fam == "in-dc":
        return F.conv_transpose3d(x, wt, stride=2, padding=1, output_padding=1 if row.opts["k"] == 3 else 0)
    return F.conv3d(x, wt)


def in_stats32(x):
    """(B, C, 2) fp32 (mean, rstd) of x computed in fp64: the normalised-input cases feed exact statistics."""
    y = x.double().flatten(2)
    return torch.stack([y.mean(2), 1 / torch.sqrt(y.var(2, unbiased=False) + 1e-5)], -1).float().contiguous()


def in_normalised64(x, st, gate):
    """leaky((x - mean) * rstd) * gate in fp64 with the fp32 statistics the kernel reads; gate (B, C, H, W) broadcast over D."""
    mean, rstd = st[..., 0].double().view(*st.shape[:2], 1, 1, 1), st[..., 1].double().view(*st.shape[:2], 1, 1, 1)
    y = F.leaky_relu((x.double() - mean) * rstd, 0.01)
    return y if gate is None else y * gate.double().unsqueeze(2)


def in_call(osb, row, xs, wp, stats_in, gates, y, stats_out=None, ws=None, sc=None, sh=None, act=ACT_NONE, sigmoid=0):
    """One launch of an instance-norm row.  xs / stats_in / gates: one entry per slab (the 1x1 takes two); pointers are addresses."""
    lib, _ = osb
    b, d, h, w = row.shape
    s = torch.cuda.current_stream().cuda_stream
    wsn = 0 if ws is None else ws[1]
    ws = None if ws is None else ws[0]
    if row.fam == "in-k3":
        lib.call("osb_conv3d_k3_in_fwd", xs[0], wp, sc, sh, stats_in[0], gates[0], y, stats_out, ws, wsn, b, row.cin, row.cout, d, h, w,
                 row.opts["stride"], act, s)
    elif row.fam == "in-dc":
        lib.call("osb_deconv3d_in_fwd", xs[0], wp, sc, sh, stats_in[0], gates[0], y, stats_out, ws, wsn, b, row.cin, row.cout, d, h, w,
                 row.opts["k"], act, s)
    else:
        c0 = row.opts.get("c0", row.cin)
        two = c0 < row.cin
        lib.call("osb_conv3d_1x1_in_fwd", xs[0], xs[1] if two else None, c0, wp, sc, sh, stats_in[0], gates[0],
                 stats_in[1] if two else None, gates[1] if two else None, y, stats_out, ws, wsn, b, row.cin, row.cout, d, h, w, act,
                 sigmoid, s)


def in_slabs(row, x):
    c0 = row.opts.get("c0", row.cin)
    return [x[:, :c0]] + ([x[:, c0:]] if c0 < row.cin else [])


def in_cases(osb, row, g):
    """Normalised-input cases of an instance-norm row: ungated, gated, gated + scale / shift / activation (+ output sigmoid)."""
    o = row.opts
    b, d, h, w = row.shape
    cs = channel_scales(row.cout, g)
    x = in_input(row, g)
    wt, wp = in_weight(row, g, cs)
    slabs = in_slabs(row, x)
    stats = [in_stats32(t) for t in slabs]
    gates = [torch.sigmoid(torch.randn(b, t.shape[1], h, w, generator=g)) for t in slabs]
    dev = lambda t: None if t is None else t.float().contiguous().cuda()      # noqa: E731
    xd, std = [dev(t) for t in slabs], [dev(t) for t in stats]
    out = []
    for name, gated, ep in (("ungated", False, False), ("gated", True, False), ("gated+epilogue", True, True)):
        gs = gates if gated else [None] * len(slabs)
        xn = torch.cat([in_normalised64(t, st, gt) for t, st, gt in zip(slabs, stats, gs)], 1)
        conv = in_conv64(row, xn, wt)
        sc = torch.rand(row.cout, generator=g) + 0.5 if ep else None
        sh = 0.1 * cs * torch.randn(row.cout, generator=g) if ep else None
        act, sig = (o.get("act", ACT_NONE), o.get("sigmoid", 0)) if ep else (ACT_NONE, 0)
        want = ref_epilogue(conv, 1, sc, sh, None, act, None, sig)
        mag = saturated_magnitude(in_conv64(row, xn.abs(), wt.abs()), 1, sc, sh, None, act, sig)
        gd, scd, shd = [dev(t) for t in gs], dev(sc), dev(sh)

        def fn(y, r, gt, gd=gd, scd=scd, shd=shd, act=act, sig=sig):
            in_call(osb, row, [t.data_ptr() for t in xd], wp.data_ptr(), [t.data_ptr() for t in std], [ptr(t) for t in gd], y,
                    sc=ptr(scd), sh=ptr(shd), act=act, sigmoid=sig)
        out.append(Case("%s %s" % (row.id, name), want, 1, fn, mag=mag))
    return out


def seed(row, salt=0):
    return torch.Generator().manual_seed(salt + zlib.crc32(row.id.encode()) % 10000)


@pytest.mark.timeout(180)
@pytest.mark.parametrize("row", REGISTRY, ids=[r.id for r in REGISTRY])
def test_accuracy_store_paths_bounds_determinism(osb, grid_cap, row):
    worst = 0.0
    for case in cases(osb, row, seed(row)):
        runs = [("aligned", {}, 0), ("aligned again", {}, 0)]
        if row.fam in VEC_RULE:
            assert case.want.shape[-1] % 4 == 0 or row.fam in IN_FAMS, "%s: Wo %% 4 != 0 would send the aligned run to the scalar path" % (
                case.name)
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
    for _ in range(2):                  # a profiling window that delivered no kernel record at all is taken once more
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            case.fn(buf.data_ptr() + 4 * GUARD, ptr(case.res), ptr(case.gate))
            torch.cuda.synchronize()
        names = sorted({e.name.replace(" ", "") for e in prof.events() if "osb::" in e.name})
        if names:
            break
    want = re.compile(r"osb::%s\(" % re.escape(kernel_of(row.variant)))
    assert len(names) == 1 and want.search(names[0]), "%s: launched %s, expected %s" % (row.id, names, kernel_of(row.variant))


IN_ROWS = [r for r in REGISTRY if r.fam in IN_FAMS]
STATS_TOL = 1e-5            # |mean - mean64| / (|mean64| + std64) and |rstd / rstd64 - 1|


@pytest.mark.timeout(120)
@pytest.mark.parametrize("row", IN_ROWS, ids=[r.id for r in IN_ROWS])
def test_instance_norm_moments_out(osb, row):
    lib, _ = osb
    g = seed(row, 5)
    b, d, h, w = row.shape
    x = in_input(row, g, mean=0.5, spread=1.0)
    wt, wp = in_weight(row, g, channel_scales(row.cout, g))
    want = in_conv64(row, x, wt)
    op, param = {"in-k3": (0, row.opts.get("stride")), "in-dc": (1, row.opts.get("k")), "in-pw": (2, 0)}[row.fam]
    need = lib.lib.osb_conv3d_in_workspace_floats(op, b, row.cout, d, h, w, param)
    slots, blocks = in_grid(row)
    assert need == 3 * b * row.cout * slots + b * blocks, "%s: workspace %d for %d slots" % (row.id, need, slots)
    n_y, n_s = want.numel(), 2 * b * row.cout
    # one buffer of sentinels: | y region (+1 float for the shifted run) | statistics | workspace |, GUARD sentinels around each
    o_y = GUARD
    o_s = o_y + (n_y + 1 + 3) // 4 * 4 + GUARD
    o_w = o_s + (n_s + 3) // 4 * 4 + GUARD
    buf = torch.full((o_w + (need + 3) // 4 * 4 + GUARD,), SENTINEL, device="cuda")
    buf[o_w:o_w + need] = 0.0                                     # zero-filled before its first use, reused by every launch
    xs = [t.contiguous().cuda() for t in in_slabs(row, x)]
    sent = torch.tensor([SENTINEL]).view(torch.int32).item()
    runs = []
    for what, y_off in (("aligned", 0), ("y+4", 1), ("aligned again", 0)):
        lead = o_y + y_off
        buf[o_y:o_y + n_y + 1] = SENTINEL
        buf[lead:lead + n_y] = float("nan")
        buf[o_s:o_s + n_s] = float("nan")
        in_call(osb, row, [t.data_ptr() for t in xs], wp.data_ptr(), [None, None], [None, None], buf.data_ptr() + 4 * lead,
                stats_out=buf.data_ptr() + 4 * o_s, ws=(buf.data_ptr() + 4 * o_w, need))
        torch.cuda.synchronize()
        outside = torch.ones(buf.numel(), dtype=torch.bool, device="cuda")
        outside[lead:lead + n_y] = False
        outside[o_s:o_s + n_s] = False
        outside[o_w:o_w + need] = False
        assert (buf.view(torch.int32)[outside] == sent).all(), "%s %s: a store left the output, statistics or workspace" % (row.id, what)
        y, st = buf[lead:lead + n_y], buf[o_s:o_s + n_s]
        assert not torch.isnan(y).any() and not torch.isnan(st).any(), "%s %s: outputs or statistics never written" % (row.id, what)
        assert (buf[o_w + need - b * blocks:o_w + need].view(torch.int32) == 0).all(), "%s %s: counters not re-armed" % (row.id, what)
        runs.append((y.view(torch.int32).clone(), st.view(torch.int32).clone()))
    for what, (y_bits, s_bits) in zip(("y+4 (scalar epilogue)", "aligned again"), runs[1:]):
        assert torch.equal(runs[0][0], y_bits), "%s: output of the %s run differs bit-wise" % (row.id, what)
        assert torch.equal(runs[0][1], s_bits), "%s: statistics of the %s run differ bit-wise" % (row.id, what)
    y = runs[0][0].view(torch.float32).cpu().double().view(want.shape)
    err = (y - want).abs().amax(dim=(0, 2, 3, 4))
    scale = want.abs().amax(dim=(0, 2, 3, 4))
    bad = (err > TOL * scale).nonzero().flatten().tolist()
    assert not bad, "%s: raw output channels %s exceed %g of their own max" % (row.id, bad[:8], TOL)
    yf = y.flatten(2)
    mean64, var64 = yf.mean(2), yf.var(2, unbiased=False)          # statistics OF THE STORED OUTPUT
    std64 = var64.sqrt()
    st = runs[0][1].view(torch.float32).cpu().double().view(b, row.cout, 2)
    err_m = ((st[..., 0] - mean64).abs() / (mean64.abs() + std64)).max().item()
    err_r = (st[..., 1] * torch.sqrt(var64 + 1e-5) - 1).abs().max().item()
    ratio = (mean64.abs() / std64).max().item()
    print("\n%-16s slots %d  max |mean| / std %.1f  mean err %.2e  rstd err %.2e" % (row.id, slots, ratio, err_m, err_r))
    if row.opts.get("offset") and row.fam == "in-pw":                # (k3 / dc: the zero padding spreads the means over the border)
        assert ratio >= 15, "%s: the cancellation row's channels have |mean| / std of at most %.1f" % (row.id, ratio)
    assert err_m <= STATS_TOL and err_r <= STATS_TOL, "%s: mean err %.2e, rstd err %.2e" % (row.id, err_m, err_r)


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
