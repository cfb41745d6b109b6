"""GPU: edge cases of the channel-pair work items of conv3d_tcs2.cu.  A work item is one output tile and two channel groups of 32,
one per consumer warpgroup, reading the same staged units.  With Cout = 96 the second warpgroup of a tile's last item has no group:
it still waits for and releases every unit and weight slot, and stores nothing.  Each case is checked against fp64 PyTorch and for
bit-identity across persistent-grid caps."""
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
    (32, 96, 4, 6, 64),      # odd number of channel groups: the last item has one idle warpgroup
    (32, 128, 4, 6, 64),     # two items per tile
    (32, 64, 2, 4, 128),     # one output plane: the kd = 0 phase is skipped
    (32, 96, 4, 2, 64),      # one output row: the only row block is short
    (16, 128, 2, 4, 300),    # general width: two column tiles
])
def test_conv3d_s2_tc_channel_pairs(ops, cin, cout, d, h, w):
    assert ops.conv3d_s2_tc_supported(cin, cout, d, h, w)
    x, wt = rnd(920, 2, cin, d, h, w), rnd(921, cout, cin, 3, 3, 3, scale=0.2)
    sc, sh = rnd(922, cout).abs() + 0.5, rnd(923, cout, scale=0.1)
    want = F.conv3d(x.double(), wt.double(), stride=2, padding=1)
    res = rnd(924, *want.shape)
    want_full = torch.relu(want * sc.double().view(1, -1, 1, 1, 1) + sh.double().view(1, -1, 1, 1, 1) + res.double()).float()
    want = want.float()
    xc, wp = ops.to_ndhwc(x.cuda()), ops.pack_tc_weight(wt.cuda(), 16, kw_order=(1, 0, 2))

    outs = _grid_caps(ops, lambda: ops.conv3d_k3_s2_tc(xc, wp, out_ndhwc=True).cpu())
    rel_close(outs[-1].permute(0, 4, 1, 2, 3), want, 1e-5, "ndhwc")
    assert all(torch.equal(o, outs[-1]) for o in outs), "grid caps disagree (ndhwc)"

    fn = lambda: ops.conv3d_k3_s2_tc(xc, wp, sc.cuda(), sh.cuda(), res.cuda(), ops.ACT_RELU).cpu()  # noqa: E731
    outs = _grid_caps(ops, fn)
    rel_close(outs[-1], want_full, 1e-5, "ncdhw + ncdhw residual")
    assert all(torch.equal(o, outs[-1]) for o in outs), "grid caps disagree (ncdhw)"


def test_conv3d_s2_tc_cout96_slice(ops):
    """Cout = 96 written as channels [64, 160) of a 160-channel channels-last tensor (W' = 16): the channels outside the slice keep
    their contents."""
    cin, cout, ctot, coff, d, h, w = 32, 96, 160, 64, 4, 10, 32
    assert ops.conv3d_s2_tc_supported(cin, cout, d, h, w)
    x, wt = rnd(930, 2, cin, d, h, w), rnd(931, cout, cin, 3, 3, 3, scale=0.2)
    sc, sh = rnd(932, cout).abs() + 0.5, rnd(933, cout, scale=0.1)
    want = F.conv3d(x.double(), wt.double(), stride=2, padding=1)
    want = (want * sc.double().view(1, -1, 1, 1, 1) + sh.double().view(1, -1, 1, 1, 1)).float().permute(0, 2, 3, 4, 1)
    xc, wp = ops.to_ndhwc(x.cuda()), ops.pack_tc_weight(wt.cuda(), 16, kw_order=(1, 0, 2))

    def run():
        y = torch.full((2, d // 2, h // 2, w // 2, ctot), -1234.5, device="cuda")
        return ops.tc_slice("s2", xc, wp, sc.cuda(), sh.cuda(), y, coff).cpu()

    outs = _grid_caps(ops, run)
    y = outs[-1]
    rel_close(y[..., coff:coff + cout], want, 1e-5, "slice")
    assert bool((y[..., :coff] == -1234.5).all()), "channels below the slice were written"
    assert all(torch.equal(o, y) for o in outs), "grid caps disagree"
