"""GPU: edge cases of the two-parity work items of conv3d_tcdc.cu.  A work item stages the input rows at offsets +1, 0 (and -1 for
k = 4) once for both output row parities; with H = 1 or D = 1 the rows and planes at offsets +-1 lie outside the input and are
staged as zeros.  Each case is checked against fp64 PyTorch and for bit-identity across persistent-grid caps."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import ops
    return ops


def rnd(seed, *shape, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def rel_close(got, want, tol, what):
    got = got.detach().cpu()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    err = ((got - want).abs().max() / (want.abs().max() + 1e-12)).item()
    assert err <= tol, "%s: rel err %g > %g" % (what, err, tol)


def _grid_caps(ops, fn):
    """fn() under persistent-grid caps 1, 7 and none: every cap must give the same bytes."""
    outs = []
    try:
        for cap in (1, 7, 0):
            ops.set_persistent_grid_cap(cap)
            outs.append(fn())
    finally:
        ops.set_persistent_grid_cap(0)
    return outs


@pytest.mark.parametrize("cin,cout,d,h,w", [
    (32, 64, 1, 1, 16),      # one input row and plane: offsets +1 and -1 both outside the input
    (32, 32, 1, 1, 64),
    (32, 64, 1, 3, 32),      # one plane, odd H
    (32, 32, 3, 1, 64),      # one row, several planes
])
def test_deconv3d_k4_tc_single_row_or_plane(ops, cin, cout, d, h, w):
    assert ops.deconv3d_k4_tc_supported(cin, cout, w)
    x, wt = rnd(900, 2, cin, d, h, w), rnd(901, cin, cout, 4, 4, 4, scale=0.2)
    want = F.conv_transpose3d(x.double(), wt.double(), stride=2, padding=1).float()
    xc, wp = ops.to_ndhwc(x.cuda()), ops.pack_tc_deconv_weight(wt.cuda())
    outs = _grid_caps(ops, lambda: ops.deconv3d_k4_tc(xc, wp).cpu())
    rel_close(outs[-1].permute(0, 4, 1, 2, 3), want, 1e-5, "k4 deconv ndhwc")
    assert all(torch.equal(o, outs[-1]) for o in outs), "grid caps disagree"
    rel_close(ops.deconv3d_k4_tc(xc, wp, out_ndhwc=False), want, 1e-5, "k4 deconv ncdhw")


@pytest.mark.parametrize("cin,cout,d,h,w", [
    (32, 64, 1, 1, 32),
    (32, 32, 1, 1, 64),
    (16, 32, 1, 1, 200),     # general width: two column tiles
    (32, 64, 2, 3, 32),      # odd H: the last row block is short
])
def test_deconv3d_k3_tc_single_row_or_plane(ops, cin, cout, d, h, w):
    assert ops.deconv3d_tc_supported(cin, cout, w)
    x, wt = rnd(910, 2, cin, d, h, w), rnd(911, cin, cout, 3, 3, 3, scale=0.2)
    want = F.conv_transpose3d(x.double(), wt.double(), stride=2, padding=1, output_padding=1).float()
    xc, wp = ops.to_ndhwc(x.cuda()), ops.pack_tc_deconv_weight(wt.cuda())
    outs = _grid_caps(ops, lambda: ops.deconv3d_k3_tc(xc, wp).cpu())
    rel_close(outs[-1], want, 1e-5, "k3 deconv ncdhw")
    assert all(torch.equal(o, outs[-1]) for o in outs), "grid caps disagree"
    rel_close(ops.deconv3d_k3_tc(xc, wp, out_ndhwc=True).permute(0, 4, 1, 2, 3), want, 1e-5, "k3 deconv ndhwc")
