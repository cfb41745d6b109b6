"""GPU: the stride-1 generic tensor-core kernel (csrc/conv3d_tcg.cu) computes two output tiles per work item, one per consumer
warpgroup.  The shapes here are the ones where that pairing has edges the registry shapes of test_tc_contract_gpu.py do not
reach: H = 1 (the second tile of every item lies below the image), H = 2, an even H whose last item is full, W = 16 with H < 16
(8 image rows per tile: the second tile lies wholly below the image), dilation 2 with odd H (rows h and h + 2 pair up) and a
general width.  Each is checked against fp64 at the contract tolerance and for bit-identity across persistent-grid caps."""
import pytest
import torch
import torch.nn.functional as F

from openstereo_b200 import ops

pytestmark = pytest.mark.gpu

# (id, cin, cout, (B, D, H, W), dilation, variant)
CASES = [
    ("w128-h1", 32, 64, (1, 3, 1, 128), 1, "tcg<64,16,128,1,1,0,0>"),
    ("w128-h2", 32, 128, (2, 2, 2, 128), 1, "tcg<128,16,128,1,1,0,0>"),
    ("w64-h8", 32, 64, (1, 2, 8, 64), 1, "tcg<64,16,64,1,1,0,0>"),
    ("w32-h6", 48, 128, (1, 2, 6, 32), 1, "tcg<128,16,32,1,1,0,0>"),
    ("w16-h6", 32, 64, (1, 3, 6, 16), 1, "tcg<64,16,16,1,1,0,1>"),
    ("w16-h9", 32, 96, (2, 2, 9, 16), 1, "tcg<96,16,16,1,1,0,1>"),
    ("w240-h3", 32, 64, (1, 2, 3, 240), 1, "tcg<64,16,128,1,1,1,0>"),
    ("dil2-h5", 32, 128, (2, 1, 5, 128), 2, "tcg<128,16,128,1,2,0,0>"),
    ("dil2-h1", 32, 128, (1, 1, 1, 128), 2, "tcg<128,16,128,1,2,0,0>"),
]


def _run(cin, cout, shape, dil, seed=0):
    B, D, H, W = shape
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(seed)
    sc = torch.rand(cout, device=dev, generator=g) + 0.5
    sh = torch.randn(cout, device=dev, generator=g) * 0.1
    if dil == 1:
        x = torch.randn(B, D, H, W, cin, device=dev, generator=g)
        w = torch.randn(cout, cin, 3, 3, 3, device=dev, generator=g) * 0.05
        wp = ops.pack_tc_weight(w, ops.conv3d_tc_kc(cin, cout, W))
        ref = F.conv3d(x.permute(0, 4, 1, 2, 3).double(), w.double(), padding=1).permute(0, 2, 3, 4, 1)
        run = lambda: ops.conv3d_k3_tc(x, wp, sc, sh, None, ops.ACT_NONE, out_ndhwc=True)  # noqa: E731
    else:
        x = torch.randn(B, H, W, cin, device=dev, generator=g)
        w2 = torch.randn(cout, cin, 3, 3, device=dev, generator=g) * 0.05
        w5 = torch.zeros(cout, cin, 3, 3, 3, device=dev)
        w5[:, :, 1] = w2
        wp = ops.pack_tc_weight(w5, ops.conv2d_tc_kc(cin, cout, W, dil))
        ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w2.double(), padding=dil, dilation=dil).permute(0, 2, 3, 1)
        run = lambda: ops.conv2d_k3_tc(x, wp, sc, sh, None, ops.ACT_NONE, dilation=dil)  # noqa: E731
    ref = ref * sc.double() + sh.double()
    return run, ref


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_two_tile_items(case):
    _, cin, cout, shape, dil, variant = case
    run, ref = _run(cin, cout, shape, dil)
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
