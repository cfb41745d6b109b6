"""GPU: split NDHWC activations (ops.to_split / from_split, csrc/tc_common.cuh).  The encoding is checked bit for bit against a host
reimplementation of the hi/lo rule, saturation and the overflow count included (from the conversion and from a layer's epilogue);
a W = 128 layer fed split rows (TMA tensor copies, zero fill outside the image) gives exactly what it gives for the fp32 tensor, at
the first and last row and plane, odd H and D = 1; a chain of layers hands split tensors on without a conversion in between."""
import pytest
import torch
import torch.nn.functional as F

from openstereo_b200 import _lib, ops

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def host_split(x):
    """(B,D,H,W,C) fp32 -> (B,D,H,W,2C) fp16: per 16-channel granule [16 hi | 16 lo] of x * 16, round to nearest, saturating."""
    def sat(v):
        h = v.half()
        return torch.where(torch.isinf(h), torch.sign(v).half() * 65504.0, h)
    s = x.float() * 16.0
    hi = sat(s)
    lo = sat(s - hi.float())
    g = x.shape[-1] // 16
    both = torch.stack((hi.view(*x.shape[:4], g, 16), lo.view(*x.shape[:4], g, 16)), dim=4)   # (..., 2, g, 16)
    return both.permute(0, 1, 2, 3, 5, 4, 6).reshape(*x.shape[:4], 2 * x.shape[-1]).contiguous()


def split_of(x_ndhwc):
    return ops.to_split(x_ndhwc.permute(0, 4, 1, 2, 3).contiguous())


def rnd(g, *shape, scale=1.0):
    return torch.randn(*shape, device=DEV, generator=g) * scale


def test_round_trip_matches_host_rule():
    g = torch.Generator(device=DEV).manual_seed(0)
    x = rnd(g, 2, 3, 5, 16, 48) * torch.logspace(-9, 3, 48, device=DEV)                # tiny to large magnitudes
    x[0, 0, 0, 0, :4] = torch.tensor([0.0, -0.0, 4093.9, -4093.9], device=DEV)
    ops.tc_overflow_count(reset=True)
    s = split_of(x)
    assert s.dtype == torch.float16 and s.shape == (2, 3, 5, 16, 96)
    assert torch.equal(s.view(torch.int16), host_split(x).view(torch.int16))
    back = ops.from_split(s)
    h = host_split(x).view(*x.shape[:4], 3, 2, 16).float()
    assert torch.equal(back, ((h[..., 0, :] + h[..., 1, :]) / 16.0).reshape(x.shape))
    assert ((back - x).abs() <= torch.maximum(x.abs() * 2.0 ** -21, torch.tensor(2.0 ** -28, device=DEV))).all()
    assert ops.tc_overflow_count(reset=True) == 0


def test_saturation_and_overflow_flag():
    x = torch.zeros(1, 1, 1, 4, 16, device=DEV)
    x[0, 0, 0, 1, 3] = 5000.0
    x[0, 0, 0, 2, 7] = -1e6
    ops.tc_overflow_count(reset=True)
    s = split_of(x)
    assert torch.equal(s.view(torch.int16), host_split(x).view(torch.int16))
    assert s[0, 0, 0, 1, 3].item() == 65504.0 and s[0, 0, 0, 2, 7].item() == -65504.0
    assert ops.tc_overflow_count(reset=True) > 0


def test_overflow_flag_from_epilogue():
    g = torch.Generator(device=DEV).manual_seed(1)
    x = rnd(g, 1, 2, 2, 128, 32)
    wp = ops.pack_tc_weight(rnd(g, 32, 32, 3, 3, 3, scale=0.05), 32)
    ops.tc_overflow_count(reset=True)
    ops.conv3d_k3_tc(x, wp, torch.full((32,), 1e5, device=DEV), None, out_split=True)
    assert ops.tc_overflow_count(reset=True) > 0
    ops.conv3d_k3_tc(x, wp, None, None, out_split=True)
    assert ops.tc_overflow_count(reset=True) == 0


# (B, D, H) at W = 128: first / last rows and planes are TMA zero fill; odd H leaves the second tile of the last item below the
# image; D = 1 is the one-plane (2D) case
SHAPES = [(1, 1, 3), (2, 3, 5), (1, 4, 2), (1, 2, 1)]


@pytest.mark.parametrize("cin,cout", [(32, 32), (64, 32), (32, 1)])
@pytest.mark.parametrize("shape", SHAPES, ids=["d1-h3", "d3-h5", "d4-h2", "d2-h1"])
def test_split_input_is_bit_identical(shape, cin, cout):
    B, D, H = shape
    g = torch.Generator(device=DEV).manual_seed(2)
    x = rnd(g, B, D, H, 128, cin)
    w = rnd(g, cout, cin, 3, 3, 3, scale=0.05)
    head = cout < 16
    wp = ops.pack_tc_weight(w, 32, pad_cout_to=16 if head else None)
    sc = None if head else torch.rand(cout, device=DEV, generator=g) + 0.5
    sh = None if head else rnd(g, cout, scale=0.1)
    out_ndhwc = not head
    want = ops.conv3d_k3_tc(x, wp, sc, sh, None, ops.ACT_RELU, out_ndhwc=out_ndhwc)
    got = ops.conv3d_k3_tc(split_of(x), wp, sc, sh, None, ops.ACT_RELU, out_ndhwc=out_ndhwc)
    assert torch.equal(got, want)
    ref = F.relu(F.conv3d(x.permute(0, 4, 1, 2, 3).double(), w.double(), padding=1))
    if not head:
        ref = F.relu(F.conv3d(x.permute(0, 4, 1, 2, 3).double(), w.double(), padding=1) * sc.double().view(-1, 1, 1, 1)
                     + sh.double().view(-1, 1, 1, 1)).permute(0, 2, 3, 4, 1)
    assert (got.double() - ref).abs().max().item() < 1e-4 * max(1.0, ref.abs().max().item())
    if not head:                                                       # a split output holds exactly the encoded fp32 output
        assert torch.equal(ops.conv3d_k3_tc(split_of(x), wp, sc, sh, None, ops.ACT_RELU, out_split=True).view(torch.int16),
                           host_split(want).view(torch.int16))


def test_ncdhw_stem_writes_split():
    g = torch.Generator(device=DEV).manual_seed(3)
    x = rnd(g, 1, 64, 3, 5, 128)
    wp = ops.pack_tc_weight(rnd(g, 32, 64, 3, 3, 3, scale=0.05), 32)
    want = ops.conv3d_k3_tc(x, wp, None, None, None, ops.ACT_RELU, in_ncdhw=True)
    got = ops.conv3d_k3_tc(x, wp, None, None, None, ops.ACT_RELU, in_ncdhw=True, out_split=True)
    assert torch.equal(got.view(torch.int16), host_split(want).view(torch.int16))


def test_two_layer_chain_stays_split():
    """conv -> conv + residual, the residual being the first layer's split output: two launches and no conversion between them;
    the residual enters as (hi + lo) / 16, so the result matches the fp32 chain to the split's ~22 bits."""
    g = torch.Generator(device=DEV).manual_seed(4)
    x = rnd(g, 2, 3, 4, 128, 32)
    w1, w2 = (ops.pack_tc_weight(rnd(g, 32, 32, 3, 3, 3, scale=0.05), 32) for _ in range(2))
    xs = split_of(x)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    ops.profile_start()
    c = ops.conv3d_k3_tc(xs, w1, None, None, None, ops.ACT_RELU, out_split=True)
    y = ops.conv3d_k3_tc(c, w2, None, None, c, ops.ACT_NONE)
    names = ops.profile_stop()
    torch.cuda.synchronize()
    # both launches are recorded under the family's profile name, like the same layers on fp32 tensors
    assert _lib.launch_count() - n0 == 2 and list(names) == ["osb_conv3d_k3_tc_fwd"] and len(names["osb_conv3d_k3_tc_fwd"]) == 2
    assert c.dtype == torch.float16 and y.dtype == torch.float32 and y.shape == x.shape
    c32 = ops.conv3d_k3_tc(x, w1, None, None, None, ops.ACT_RELU)
    y32 = ops.conv3d_k3_tc(c32, w2, None, None, c32, ops.ACT_NONE)
    assert torch.equal(ops.conv3d_k3_tc(xs, w2, None, None, None, ops.ACT_NONE, out_split=False),
                       ops.conv3d_k3_tc(x, w2, None, None, None, ops.ACT_NONE))
    assert (y - y32).abs().max().item() <= 2.0 ** -18 * max(1.0, c32.abs().max().item())


def test_split_arguments_are_checked():
    g = torch.Generator(device=DEV).manual_seed(5)
    x = rnd(g, 1, 1, 2, 64, 64)                                        # W = 64: served by a 16-channel-chunk kernel
    wp = ops.pack_tc_weight(rnd(g, 64, 64, 3, 3, 3, scale=0.05), 16)
    with pytest.raises(Exception, match="split activations are served by the W = 128 kernel only"):
        ops.conv3d_k3_tc(x, wp, out_split=True)
    w32 = ops.pack_tc_weight(rnd(g, 32, 32, 3, 3, 3, scale=0.05), 32)
    with pytest.raises(ValueError, match="read as split activations"):     # a plain half tensor is not split activations
        ops.conv3d_k3_tc(rnd(g, 1, 1, 2, 128, 32).half(), w32)
