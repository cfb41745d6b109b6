"""GPU: the full-resolution tensor-core kernel (csrc/conv3d_tc.cu: W = 128, Cout = 32 or <= 16) computes two output rows per work
item, one per consumer warpgroup, from input rows 2p - 1 .. 2p + 2 staged once per phase.  The shapes here are the ones where that
pairing has edges the registry shapes of test_tc_contract_gpu.py do not reach: H = 1 (the second row of every item lies below the
image), H = 2 (one full item per plane), odd H with D > 1 on the register-staged (Cin = 64) rows, one plane with H = 3 (the
backbone front's class), the NCDHW input with odd H and the 32 -> 1 head (Cout padded to 16, NCDHW output) with odd H.  Each is
checked against fp64 at the contract tolerance and for bit-identity across persistent-grid caps."""
import pytest
import torch
import torch.nn.functional as F

from openstereo_b200 import ops

pytestmark = pytest.mark.gpu

# (id, cin, cout, (B, D, H, W), mode, variant); mode "ncdhw-in": the input goes in as (B, Cin, D, H, W); "head": a 32 -> cout <= 16
# classifier head (weights zero-padded to 16 rows, NCDHW output, no folded BN)
CASES = [
    ("h1", 32, 32, (1, 3, 1, 128), None, "tc<32>"),
    ("h2", 32, 32, (2, 2, 2, 128), None, "tc<32>"),
    ("regs-h5", 64, 32, (1, 3, 5, 128), None, "tc<32>"),
    ("1plane-h3", 32, 32, (2, 1, 3, 128), None, "tc<32>"),
    ("ncdhw-h5", 64, 32, (1, 3, 5, 128), "ncdhw-in", "tc<32>"),
    ("head-h3", 32, 1, (2, 3, 3, 128), "head", "tc<16>"),
]


def _run(cin, cout, shape, mode, seed=0):
    B, D, H, W = shape
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(seed)
    sc = torch.rand(cout, device=dev, generator=g) + 0.5
    sh = torch.randn(cout, device=dev, generator=g) * 0.1
    x = torch.randn(B, D, H, W, cin, device=dev, generator=g)
    w = torch.randn(cout, cin, 3, 3, 3, device=dev, generator=g) * 0.05
    ref = F.conv3d(x.permute(0, 4, 1, 2, 3).double(), w.double(), padding=1).permute(0, 2, 3, 4, 1)
    if mode == "head":
        wp = ops.pack_tc_weight(w, 32, pad_cout_to=16)
        run = lambda: ops.conv3d_k3_tc(x, wp, None, None, None, ops.ACT_NONE, out_ndhwc=False,  # noqa: E731
                                       res_ndhwc=False).permute(0, 2, 3, 4, 1)
        return run, ref
    wp = ops.pack_tc_weight(w, ops.conv3d_tc_kc(cin, cout, W))
    if mode == "ncdhw-in":
        xn = x.permute(0, 4, 1, 2, 3).contiguous()
        run = lambda: ops.conv3d_k3_tc(xn, wp, sc, sh, None, ops.ACT_NONE, out_ndhwc=True, in_ncdhw=True)  # noqa: E731
    else:
        run = lambda: ops.conv3d_k3_tc(x, wp, sc, sh, None, ops.ACT_NONE, out_ndhwc=True)  # noqa: E731
    return run, ref * sc.double() + sh.double()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_full_res_two_row_items(case):
    _, cin, cout, shape, mode, variant = case
    run, ref = _run(cin, cout, shape, mode)
    outs = []
    for cap in (1, 7, 0):
        prev = ops.set_persistent_grid_cap(cap)
        try:
            outs.append(run())
            torch.cuda.synchronize()
            assert ops.tc_last_variant() == variant
        finally:
            ops.set_persistent_grid_cap(prev)
    for y in outs[1:]:
        assert torch.equal(y, outs[0]), "output depends on the persistent grid"
    y = outs[0].double()
    assert torch.isfinite(y).all()
    err = (y - ref).abs().reshape(-1, cout).amax(0)
    scale = ref.abs().reshape(-1, cout).amax(0)
    assert (err <= 1e-5 * scale + 1e-7).all(), "max relative error %g" % (err / scale).max().item()
