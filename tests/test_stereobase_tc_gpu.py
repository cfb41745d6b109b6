"""GPU: the tensor-core pieces StereoBase's hourglass needs (VERDICT round 1, missing #6 / next #6; BASELINE config 3):
channel plan 24/48/96/144 (24 and 48 run zero-padded to 32 and 64), ConvTranspose3d(k4, s2, p1), LeakyReLU, FeatureAtt's sigmoid
gate in the conv epilogue, the 1x1 conv over a never-materialised channel concat.  Reference: stereobase/hourglass.py:7-104,
igev_blocks.py:35-48.  Op level vs fp64 PyTorch (<= 1e-5 of the output scale); engine level vs the CPU oracle of the reference
module and vs the engine's fp32 CUDA-core route."""
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


def test_to_ndhwc_pad(osb):
    _, ops = osb
    x = rnd(400, 2, 24, 3, 5, 7).cuda()
    y = ops.to_ndhwc(x, pad_to=32)
    assert y.shape == (2, 3, 5, 7, 32)
    assert torch.equal(y[..., :24], x.permute(0, 2, 3, 4, 1)) and (y[..., 24:] == 0).all()


@pytest.mark.parametrize("b,cin,cout,d,h,w", [(1, 96, 96, 2, 8, 32), (2, 64, 96, 1, 5, 32)])
def test_conv3d_tc_cout96_and_gate(osb, b, cin, cout, d, h, w):
    """4c = 96 channels at the 1/16 level, LeakyReLU, and the FeatureAtt gate (B,H,W,C) multiplied after the activation."""
    _, ops = osb
    assert ops.conv3d_tc_kc(cin, cout, w) == 16
    x, wt = rnd(410, b, cin, d, h, w), rnd(411, cout, cin, 3, 3, 3, scale=0.2)
    sc, sh = _bn(cout, 412)
    gate = torch.sigmoid(rnd(414, b, cout, h, w))
    want = F.leaky_relu(F.conv3d(x.double(), wt.double(), padding=1).float() * sc.view(1, -1, 1, 1, 1) + sh.view(1, -1, 1, 1, 1))
    xc = ops.to_ndhwc(x.cuda())
    wp = ops.pack_tc_weight(wt.cuda(), 16)
    got = ops.conv3d_k3_tc(xc, wp, sc.cuda(), sh.cuda(), None, ops.ACT_LEAKY)
    rel_close(got.permute(0, 4, 1, 2, 3), want, 1e-5, "cout96 leaky")
    got = ops.conv3d_k3_tc(xc, wp, sc.cuda(), sh.cuda(), None, ops.ACT_LEAKY, gate=gate.permute(0, 2, 3, 1).contiguous().cuda())
    rel_close(got.permute(0, 4, 1, 2, 3), want * gate.unsqueeze(2), 1e-5, "cout96 leaky * gate")


def test_conv3d_tc_gate_two_rows_per_tile(osb):
    """W = 64 (two image rows per M tile), 48 -> 48 zero-padded to 64 -> 64: padded channels stay exactly zero."""
    _, ops = osb
    b, c, cp, d, h, w = 2, 48, 64, 2, 6, 64
    x, wt = rnd(420, b, c, d, h, w), rnd(421, c, c, 3, 3, 3, scale=0.2)
    sc, sh = _bn(c, 422)
    gate = torch.sigmoid(rnd(424, b, c, h, w))
    want = F.leaky_relu(F.conv3d(x.double(), wt.double(), padding=1).float() * sc.view(1, -1, 1, 1, 1) + sh.view(1, -1, 1, 1, 1))
    want = want * gate.unsqueeze(2)
    wpad = torch.zeros(cp, cp, 3, 3, 3)
    wpad[:c, :c] = wt
    scp, shp = torch.ones(cp), torch.zeros(cp)
    scp[:c], shp[:c] = sc, sh
    gp = torch.zeros(b, h, w, cp)
    gp[..., :c] = gate.permute(0, 2, 3, 1)
    got = ops.conv3d_k3_tc(ops.to_ndhwc(x.cuda(), pad_to=cp), ops.pack_tc_weight(wpad.cuda(), 16), scp.cuda(), shp.cuda(), None,
                           ops.ACT_LEAKY, gate=gp.cuda())
    assert (got[..., c:] == 0).all()
    rel_close(got[..., :c].permute(0, 4, 1, 2, 3), want, 1e-5, "48->48 padded, gate")


def test_conv3d_s2_tc_cout96(osb):
    _, ops = osb
    b, cin, cout, d, h, w = 1, 64, 96, 4, 8, 64
    assert ops.conv3d_s2_tc_supported(cin, cout, d, h, w)
    x, wt = rnd(430, b, cin, d, h, w), rnd(431, cout, cin, 3, 3, 3, scale=0.2)
    sc, sh = _bn(cout, 432)
    want = F.leaky_relu(F.conv3d(x.double(), wt.double(), stride=2, padding=1).float() * sc.view(1, -1, 1, 1, 1) + sh.view(1, -1, 1, 1, 1))
    got = ops.conv3d_k3_s2_tc(ops.to_ndhwc(x.cuda()), ops.pack_tc_weight(wt.cuda(), 16, kw_order=(1, 0, 2)), sc.cuda(), sh.cuda(), None,
                              ops.ACT_LEAKY, out_ndhwc=True)
    rel_close(got.permute(0, 4, 1, 2, 3), want, 1e-5, "s2 cout96 leaky")


@pytest.mark.parametrize("b,cin,cout,d,h,w", [
    (1, 96, 64, 3, 8, 32),      # conv2_up: 4c -> 2c (48 packed as 64) at 1/16 -> 1/8
    (2, 64, 32, 2, 10, 64),     # conv1_up: 2c -> c (24 packed as 32) at 1/8 -> 1/4; ragged row blocks (8 rows per item)
    (1, 16, 32, 1, 3, 64),      # single input plane, short block
    (1, 32, 64, 1, 1, 32),      # one input row
])
def test_deconv3d_k4_tc(osb, b, cin, cout, d, h, w):
    _, ops = osb
    assert ops.deconv3d_k4_tc_supported(cin, cout, w)
    x, wt = rnd(440, b, cin, d, h, w), rnd(441, cin, cout, 4, 4, 4, scale=0.2)
    sc, sh = _bn(cout, 442)
    want = F.conv_transpose3d(x.double(), wt.double(), stride=2, padding=1).float()
    xc = ops.to_ndhwc(x.cuda())
    wp = ops.pack_tc_deconv_weight(wt.cuda())
    got = ops.deconv3d_k4_tc(xc, wp)
    rel_close(got.permute(0, 4, 1, 2, 3), want, 1e-5, "k4 deconv plain ndhwc")
    got = ops.deconv3d_k4_tc(xc, wp, out_ndhwc=False)
    rel_close(got, want, 1e-5, "k4 deconv plain ncdhw")
    want2 = F.leaky_relu(want * sc.view(1, -1, 1, 1, 1) + sh.view(1, -1, 1, 1, 1))
    got = ops.deconv3d_k4_tc(xc, wp, sc.cuda(), sh.cuda(), None, ops.ACT_LEAKY)
    rel_close(got.permute(0, 4, 1, 2, 3), want2, 1e-5, "k4 deconv bn+leaky")
    creal = cout - 8                                             # zero-padded plan: only the real channels reach an NCDHW output
    got = ops.deconv3d_k4_tc(xc, wp, out_ndhwc=False, cout_real=creal)
    rel_close(got, want[:, :creal].contiguous(), 1e-5, "k4 deconv ncdhw, real channels only")


def test_conv1x1_ndhwc_cat(osb):
    _, ops = osb
    for (c0, c1, cout, v) in ((96, 96, 96, 1000), (64, 64, 64, 777)):
        x0, x1 = rnd(450, v, c0), rnd(451, v, c1)
        wt = rnd(452, c0 + c1, cout, scale=0.1)
        sc, sh = _bn(cout, 453)
        want = F.leaky_relu((torch.cat((x0, x1), 1).double() @ wt.double()).float() * sc + sh)
        got = ops.conv1x1_ndhwc_cat(x0.cuda(), x1.cuda(), wt.cuda(), sc.cuda(), sh.cuda(), ops.ACT_LEAKY)
        rel_close(got, want, 1e-5, "1x1 over the concat %d+%d->%d" % (c0, c1, cout))


@pytest.mark.parametrize("b,cf,cv,h,w", [(2, 64, 48, 8, 16), (1, 192, 96, 5, 7), (1, 160, 144, 3, 5)])
def test_feature_att_gate_one_launch(osb, b, cf, cv, h, w):
    """sigmoid(conv1x1(leaky(bn(conv1x1(feat))))) written channels-last and zero-padded, vs PyTorch (igev_blocks.py:35-48)."""
    _, ops = osb
    ch, cp = cf // 2, (cv + 31) // 32 * 32
    feat = rnd(470, b, cf, h, w)
    w1, w2 = rnd(471, ch, cf, scale=0.2), rnd(472, cv, ch, scale=0.2)
    sc1, sh1 = _bn(ch, 473)
    bias = rnd(475, cv, scale=0.3)
    hid = F.leaky_relu(F.conv2d(feat.double(), w1.double()[:, :, None, None]).float() * sc1.view(1, -1, 1, 1) + sh1.view(1, -1, 1, 1))
    want = torch.sigmoid(F.conv2d(hid.double(), w2.double()[:, :, None, None]).float() + bias.view(1, -1, 1, 1))
    got = ops.feature_att_gate(feat.cuda(), w1.t().contiguous().cuda(), sc1.cuda(), sh1.cuda(), w2.t().contiguous().cuda(), None,
                               bias.cuda(), pad_to=cp)
    assert got.shape == (b, h, w, cp) and (got[..., cv:] == 0).all()
    assert (got[..., :cv].cpu() - want.permute(0, 2, 3, 1)).abs().max().item() <= 2e-6


@pytest.mark.parametrize("b,d,h", [(1, 2, 8), (2, 1, 5), (1, 3, 16)])
def test_channel_slices_at_width_16(osb, b, d, h):
    """The 1/32 level of StereoBase's hourglass: W' = 16 (eight image rows per M tile, two per epilogue warp), 6c = 144 channels
    run as 160 = 96 + 64 output-channel slices; stride-2 conv, stride-1 conv with gate, k4 transposed conv (96 = 64 + 32)."""
    _, ops = osb
    cin, ctot, w = 96, 160, 16
    # stride 2: (b, 96, 2d, 2h, 32) -> (b, 160, d, h, 16)
    x, wt = rnd(480, b, cin, 2 * d, 2 * h, 2 * w), rnd(481, ctot, cin, 3, 3, 3, scale=0.2)
    sc, sh = _bn(ctot, 482)
    want = F.leaky_relu(F.conv3d(x.double(), wt.double(), stride=2, padding=1).float() * sc.view(1, -1, 1, 1, 1) + sh.view(1, -1, 1, 1, 1))
    y = torch.full((b, d, h, w, ctot), float("nan"), device="cuda")
    xc = ops.to_ndhwc(x.cuda())
    for lo, hi in ((0, 96), (96, 160)):
        ops.tc_slice("s2", xc, ops.pack_tc_weight(wt[lo:hi].cuda(), 16, kw_order=(1, 0, 2)), sc[lo:hi].contiguous().cuda(),
                     sh[lo:hi].contiguous().cuda(), y, lo, ops.ACT_LEAKY)
    rel_close(y.permute(0, 4, 1, 2, 3), want, 1e-5, "s2 slices @16")
    # stride 1 with gate: 160 -> 160
    x1, wt1 = want, rnd(483, ctot, ctot, 3, 3, 3, scale=0.1)
    gate = torch.sigmoid(rnd(484, b, ctot, h, w))
    want1 = F.leaky_relu(F.conv3d(x1.double(), wt1.double(), padding=1).float() * sc.view(1, -1, 1, 1, 1) + sh.view(1, -1, 1, 1, 1))
    want1 = want1 * gate.unsqueeze(2)
    y1 = torch.full_like(y, float("nan"))
    gp = gate.permute(0, 2, 3, 1).contiguous().cuda()
    x1c = ops.to_ndhwc(x1.cuda())
    for lo, hi in ((0, 96), (96, 160)):
        ops.tc_slice("s1", x1c, ops.pack_tc_weight(wt1[lo:hi].cuda(), 16), sc[lo:hi].contiguous().cuda(), sh[lo:hi].contiguous().cuda(),
                     y1, lo, ops.ACT_LEAKY, gate=gp)
    rel_close(y1.permute(0, 4, 1, 2, 3), want1, 1e-5, "s1 slices + gate @16")
    # k4 transposed conv: 160 -> 96 at (d, h, 16) -> (2d, 2h, 32)
    wt2 = rnd(485, ctot, 96, 4, 4, 4, scale=0.1)
    sc2, sh2 = _bn(96, 486)
    want2 = F.leaky_relu(F.conv_transpose3d(want1.double(), wt2.double(), stride=2, padding=1).float() * sc2.view(1, -1, 1, 1, 1)
                         + sh2.view(1, -1, 1, 1, 1))
    y2 = torch.full((b, 2 * d, 2 * h, 2 * w, 96), float("nan"), device="cuda")
    x2c = ops.to_ndhwc(want1.cuda())
    for lo, hi in ((0, 64), (64, 96)):
        ops.tc_slice("dc4", x2c, ops.pack_tc_deconv_weight(wt2[:, lo:hi].contiguous().cuda()), sc2[lo:hi].contiguous().cuda(),
                     sh2[lo:hi].contiguous().cuda(), y2, lo, ops.ACT_LEAKY)
    rel_close(y2.permute(0, 4, 1, 2, 3), want2, 1e-5, "k4 deconv slices @16")


def _stereobase_case(osb, b, dq, hq, wq, seed):
    agg, ops = osb
    m = oagg.StereoBaseCostHead(24, [96, 64, 192, 160], max_disp=4 * dq).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=seed, scale={"classifier.weight": 150.0}))
    vol = rnd(seed + 1, b, 24, dq, hq, wq)
    feats = [rnd(seed + 2, b, 96, hq, wq), rnd(seed + 3, b, 64, hq // 2, wq // 2), rnd(seed + 4, b, 192, hq // 4, wq // 4),
             rnd(seed + 5, b, 160, hq // 8, wq // 8)]
    return m, vol, feats


def test_stereobase_hourglass_tensor_cores(osb):
    """Hourglass(24, [96, 64, 192, 160]) at W' = 128 (BASELINE config 3's width) on a short volume: tensor-core route vs the CPU oracle
    of the reference module and vs the fp32 CUDA-core route of the same engine."""
    agg, ops = osb
    m, vol, feats = _stereobase_case(osb, 1, 8, 16, 128, 460)
    with torch.no_grad():
        want_geo, want_disp = m(vol, feats)
    m.cuda()
    eng = agg.StereoBaseAggregation(m.cost_agg)
    fg = [f.cuda() for f in feats]
    eng._ensure(torch.device("cuda", 0))
    assert eng.tc_route_ok(vol.shape) and eng._level32_tc_ok(vol.shape)
    from openstereo_b200 import _lib
    before = _lib.launch_count()
    got = eng(vol.cuda(), fg)
    launches = _lib.launch_count() - before
    err = ((got.cpu() - want_geo).abs().max() / want_geo.abs().max()).item()
    print("StereoBase hourglass on the tensor cores: rel err vs oracle %.2e, %d launches" % (err, launches))
    assert err <= 5e-5
    agg.USE_TENSOR_CORES = False
    try:
        ref = agg.StereoBaseAggregation(m.cost_agg)(vol.cuda(), fg)
    finally:
        agg.USE_TENSOR_CORES = True
    assert ((got - ref).abs().max() / ref.abs().max()).item() <= 5e-5
    head = agg.StereoBaseCostHead(m.classifier)
    disp = head(got, 8)
    assert (disp.cpu() - want_disp).abs().mean().item() <= 1e-4
