"""GPU: the tensor-core convolutions at GENERAL image widths (VERDICT round 1, weak #8 / next #7).

The whole-row tensor-core variants serve W' in {128, 64, 32} only (a 512-pixel-wide input).  The GW instantiations of conv3d_tcg.cu / conv3d_tcs2.cu / conv3d_tcdc.cu tile an image row into 128-column
segments with a one-column halo, so the reference's own timing shape (544x960 -> W' = 240, tools/measure.py:32), KITTI
(1248 -> 312) and IGEV's config-5 width (640 -> 160) take the tensor-core path.  Op level: against an fp64 convolution
(<= 1e-5 of the output scale, the bar of the whole-row variants); engine level: against the CPU oracle of the reference modules
(EPE <= 1e-3 px) and against the same engine on the fp32 CUDA-core kernels."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import aggregation as oagg     # noqa: E402
from oracle import seeded_init as si       # noqa: E402


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import aggregation, ops
    return aggregation, ops


def rnd(seed, *shape, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def rel_close(got, want, tol, what):
    got = got.detach().cpu()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    err = ((got - want).abs().max() / (want.abs().max() + 1e-12)).item()
    assert err <= tol, "%s: rel err %g > %g" % (what, err, tol)


def _bn(cout, seed):
    return torch.rand(cout, generator=torch.Generator().manual_seed(seed)) + 0.5, rnd(seed + 1, cout, scale=0.1)


def test_capability_queries(osb):
    _, ops = osb
    for w in (240, 312, 160, 120, 60, 78, 40, 24, 126, 127, 253):
        assert ops.conv3d_tc_kc(32, 32, w) == 16 and ops.conv3d_tc_kc(64, 64, w) == 16 and ops.conv3d_tc_kc(128, 128, w) == 16
        assert ops.deconv3d_tc_supported(64, 32, w) and ops.deconv3d_tc_supported(128, 64, w)
        if w % 2 == 0:
            assert ops.conv3d_s2_tc_supported(32, 64, 4, 4, 2 * w) and ops.conv3d_s2_tc_supported(64, 128, 4, 4, 2 * w)
    assert ops.conv3d_tc_kc(32, 32, 128) == 32 and ops.conv3d_tc_kc(64, 64, 64) == 16      # whole-row variants keep their shapes
    assert ops.conv3d_tc_kc(32, 32, 16) == 0 and not ops.deconv3d_tc_supported(64, 32, 16)   # too narrow: CUDA-core kernels
    assert ops.conv3d_tc_kc(32, 48, 240) == 0 and ops.conv3d_tc_kc(24, 32, 240) == 0


@pytest.mark.parametrize("b,cin,cout,d,h,w", [
    (1, 32, 32, 3, 7, 240),     # 544x960 (tools/measure.py) stem layer: two column tiles (126 + 114), ragged row block
    (1, 64, 32, 2, 6, 160),     # IGEV width, first aggregation layer 64 -> 32
    (1, 32, 32, 2, 3, 312),     # KITTI: three column tiles
    (2, 64, 64, 2, 5, 120),     # hourglass interior at 1/8 of a 960-wide input: one tile, 8 columns of padding
    (1, 128, 128, 2, 4, 60),    # 1/16 level: N = 3 x 128
    (1, 16, 64, 1, 3, 126),     # exactly one tile
    (1, 16, 64, 1, 3, 127),     # one column into the second tile
    (1, 32, 32, 1, 11, 253),    # one column into the third tile, three row blocks
    (2, 32, 32, 2, 2, 24),      # narrowest width served
    (1, 64, 32, 2, 4, 64),      # a whole-row width whose Cout (32 @ 64) has no whole-row variant: one column tile, half empty
])
def test_conv3d_tc_general_width(osb, b, cin, cout, d, h, w):
    _, ops = osb
    assert ops.conv3d_tc_kc(cin, cout, w) == 16
    x, wt = rnd(270, b, cin, d, h, w), rnd(271, cout, cin, 3, 3, 3, scale=0.2)
    sc, sh = _bn(cout, 272)
    want = F.conv3d(x.double(), wt.double(), padding=1).float()
    xc = ops.to_ndhwc(x.cuda())
    wp = ops.pack_tc_weight(wt.cuda(), 16)
    got = ops.conv3d_k3_tc(xc, wp, out_ndhwc=False)
    rel_close(got, want, 1e-5, "gw plain ncdhw-out")
    res = rnd(274, *want.shape)
    want2 = F.relu(want * sc.view(1, -1, 1, 1, 1) + sh.view(1, -1, 1, 1, 1) + res)
    got = ops.conv3d_k3_tc(xc, wp, sc.cuda(), sh.cuda(), res.cuda(), ops.ACT_RELU, out_ndhwc=False, res_ndhwc=False)
    rel_close(got, want2, 1e-5, "gw bn+res+relu ncdhw")
    got = ops.conv3d_k3_tc(xc, wp, sc.cuda(), sh.cuda(), res.permute(0, 2, 3, 4, 1).contiguous().cuda(), ops.ACT_RELU,
                           out_ndhwc=True, res_ndhwc=True)
    rel_close(got.permute(0, 4, 1, 2, 3), want2, 1e-5, "gw bn+res+relu ndhwc")


@pytest.mark.parametrize("b,cin,cout,d,h,w", [
    (1, 32, 64, 4, 8, 240),     # conv1 of the hourglass at W' = 240 -> 120
    (1, 64, 128, 2, 4, 120),    # conv3: 120 -> 60
    (1, 64, 64, 2, 6, 312),     # PSMNet conv1 on KITTI: 156 output columns = two tiles (127 + 29)
    (1, 16, 64, 2, 2, 254),     # 127 output columns: exactly one tile
    (2, 32, 64, 2, 10, 256),    # 128 output columns: the last one alone in the second tile; ragged row blocks
    (1, 32, 64, 2, 4, 48),      # narrowest output width served (24)
])
def test_conv3d_s2_tc_general_width(osb, b, cin, cout, d, h, w):
    _, ops = osb
    assert ops.conv3d_s2_tc_supported(cin, cout, d, h, w)
    x, wt = rnd(280, b, cin, d, h, w), rnd(281, cout, cin, 3, 3, 3, scale=0.2)
    sc, sh = _bn(cout, 282)
    want = F.conv3d(x.double(), wt.double(), stride=2, padding=1).float()
    xc = ops.to_ndhwc(x.cuda())
    wp = ops.pack_tc_weight(wt.cuda(), 16, kw_order=(1, 0, 2))
    got = ops.conv3d_k3_s2_tc(xc, wp)
    rel_close(got, want, 1e-5, "gw s2 plain")
    res = rnd(284, *want.shape)
    want2 = F.relu(want * sc.view(1, -1, 1, 1, 1) + sh.view(1, -1, 1, 1, 1) + res)
    got = ops.conv3d_k3_s2_tc(xc, wp, sc.cuda(), sh.cuda(), res.cuda(), ops.ACT_RELU)
    rel_close(got, want2, 1e-5, "gw s2 bn+res+relu")
    got = ops.conv3d_k3_s2_tc(xc, wp, sc.cuda(), sh.cuda(), None, ops.ACT_RELU, out_ndhwc=True)
    rel_close(got.permute(0, 4, 1, 2, 3), F.relu(want * sc.view(1, -1, 1, 1, 1) + sh.view(1, -1, 1, 1, 1)), 1e-5, "gw s2 ndhwc out")


@pytest.mark.parametrize("b,cin,cout,d,h,w", [
    (1, 128, 64, 2, 4, 60),     # conv5: 1/16 -> 1/8 of a 960-wide input
    (1, 64, 32, 2, 5, 120),     # conv6: 1/8 -> 1/4, ragged row blocks
    (2, 64, 64, 1, 3, 78),      # PSMNet conv5 on KITTI
    (1, 16, 32, 1, 2, 127),     # exactly one tile of input columns
    (1, 16, 64, 1, 2, 128),     # the last input column alone in the second tile (64 @ 128 has no whole-row variant)
    (1, 32, 32, 2, 7, 156),     # two tiles, 5-tile row blocks
    (1, 32, 32, 1, 3, 24),      # narrowest width served
])
def test_deconv3d_tc_general_width(osb, b, cin, cout, d, h, w):
    _, ops = osb
    assert ops.deconv3d_tc_supported(cin, cout, w)
    x, wt = rnd(290, b, cin, d, h, w), rnd(291, cin, cout, 3, 3, 3, scale=0.2)
    sc, sh = _bn(cout, 292)
    want = F.conv_transpose3d(x.double(), wt.double(), stride=2, padding=1, output_padding=1).float()
    xc = ops.to_ndhwc(x.cuda())
    wp = ops.pack_tc_deconv_weight(wt.cuda())
    got = ops.deconv3d_k3_tc(xc, wp)
    rel_close(got, want, 1e-5, "gw deconv plain")
    res = rnd(294, *want.shape)
    want2 = F.relu(want * sc.view(1, -1, 1, 1, 1) + sh.view(1, -1, 1, 1, 1) + res)
    got = ops.deconv3d_k3_tc(xc, wp, sc.cuda(), sh.cuda(), res.cuda(), ops.ACT_RELU)
    rel_close(got, want2, 1e-5, "gw deconv bn+res+relu")
    got = ops.deconv3d_k3_tc(xc, wp, sc.cuda(), sh.cuda(), res.permute(0, 2, 3, 4, 1).contiguous().cuda(), ops.ACT_RELU,
                             out_ndhwc=True, res_ndhwc=True)
    rel_close(got.permute(0, 4, 1, 2, 3), want2, 1e-5, "gw deconv ndhwc")


def test_output_outside_the_image_is_never_written(osb):
    """Column tiles overhang the image on the right: the 130-wide rows (a second tile with two valid columns) must match the fp64
    conv and stay finite.  That no masked store lands in the next row or beyond the tensor is checked with sentinel-guarded output
    buffers for every instantiation in tests/test_tc_contract_gpu.py."""
    _, ops = osb
    b, cin, cout, d, h, w = 1, 32, 32, 2, 3, 130
    x, wt = rnd(300, b, cin, d, h, w).cuda(), rnd(301, cout, cin, 3, 3, 3, scale=0.2).cuda()
    wp = ops.pack_tc_weight(wt, 16)
    a = ops.conv3d_k3_tc(ops.to_ndhwc(x), wp)                    # (B, D, H, W, C) channels-last
    # the same rows embedded in a wider, otherwise untouched image must come out identical where the receptive fields agree
    ref = F.conv3d(x.double(), wt.double(), padding=1).float().permute(0, 2, 3, 4, 1)
    rel_close(a, ref.cpu(), 1e-5, "130-wide rows")
    assert torch.isfinite(a).all()


@pytest.mark.parametrize("wq", [240, 160])
def test_gwc_aggregation_general_width(osb, wq):
    """GwcNet aggregation at W' = 240 (544x960, the reference's timing shape) / 160: every 3x3x3 layer on the column-tile tensor-core
    kernels, channels-last end to end; vs the CPU oracle and vs the fp32 CUDA-core path of the same engine."""
    agg, ops = osb
    m = oagg.GwcDispProcessor(maxdisp=32, downsample=4, num_groups=40, use_concat_volume=True, concat_channels=12).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=141, scale={"classif3.2.weight": 60.0}))
    vol = rnd(142, 1, 64, 8, 8, wq)
    with torch.no_grad():
        want_logits = m.aggregate(vol)
        want = m(vol, 32, 4 * wq)
    m.cuda()
    eng = agg.GwcAggregation(m)
    eng._ensure(torch.device("cuda", 0))
    assert agg._tc_ok(eng.dres0[0], wq) and agg._tc_ok(eng.hg[0].conv2, wq // 2) and agg._tc_ok(eng.hg[0].conv4, wq // 4)
    assert agg._hg_channels_last_ok(eng.hg[0], (1, 8, 8, wq, 32))
    from openstereo_b200 import _lib
    before = _lib.launch_count()
    got_logits = eng.logits(vol.cuda())
    launches = _lib.launch_count() - before
    err = ((got_logits.cpu() - want_logits).abs().max() / want_logits.abs().max()).item()
    assert err <= 5e-5, err
    e = (eng(vol.cuda(), 32, 4 * wq).cpu() - want).abs().mean().item()
    print("GwcNet aggregation at W'=%d: EPE vs oracle %.3e, %d launches" % (wq, e, launches))
    assert e <= 2e-4 and want.std() > 1.0
    agg.USE_TENSOR_CORES = False
    try:
        ref_logits = agg.GwcAggregation(m).logits(vol.cuda())
    finally:
        agg.USE_TENSOR_CORES = True
    assert ((got_logits - ref_logits).abs().max() / ref_logits.abs().max()).item() <= 5e-5


def test_psm_aggregation_general_width(osb):
    """PSMNet aggregation (three heads, stacked-hourglass skips) at KITTI's W' = 312 -> 156 -> 78, NCDHW between the layers."""
    agg, ops = osb
    m = oagg.PSMAggregator(32, 64).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=151, scale={
        "classif1.1.weight": 20.0, "classif2.1.weight": 20.0, "classif3.1.weight": 20.0}))
    vol = rnd(152, 1, 64, 8, 8, 312)
    with torch.no_grad():
        want = m.aggregate(vol)
    m.cuda()
    eng = agg.PSMAggregation(m)
    got = eng.logits(vol.cuda())
    assert agg._tc_ok(eng.dres0[0], 312) and agg._tc_ok(eng.hg[0].conv2, 156) and agg._tc_ok(eng.hg[0].conv4, 78)
    for g, w_ in zip(got, want):
        err = ((g.cpu() - w_).abs().max() / w_.abs().max()).item()
        assert err <= 5e-5, err
