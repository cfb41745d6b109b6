"""GPU: the first block of each residual stage of the 2D feature extractors (layer2[0]: 3x3 stride 2 32->64, layer3[0]: 3x3 64->128,
each with a 1x1 downsample) on the wgmma kernels, and the one-plane stride-2 convolution that serves layer2[0].conv1.

Op level: against an fp64 convolution (<= 1e-5 of the output scale, the bar of the other tensor-core tests).  Route level: against
the module's own block on the same BN-folded module (cuDNN fp32, TF32 off), with the tolerances of the backbone-route tests."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, aggregation, host_models, ops
    torch.backends.cudnn.allow_tf32 = False
    return _lib, aggregation, host_models, ops


def rnd(seed, *shape, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def rel_err(got, want):
    return ((got.detach().cpu() - want.detach().cpu()).abs().max() / (want.abs().max() + 1e-12)).item()


def _randomise_bn(m):
    with torch.no_grad():
        for mod in m.modules():                              # non-trivial BN statistics so that the folding matters
            if isinstance(mod, nn.BatchNorm2d):
                mod.running_mean.normal_(0, 0.2), mod.running_var.uniform_(0.5, 1.5)
                mod.weight.uniform_(0.5, 1.5), mod.bias.normal_(0, 0.2)
    return m


@pytest.mark.parametrize("b,cin,cout,h,w", [
    (2, 32, 64, 128, 256),      # layer2[0].conv1 at the bench shape: 128 output columns (the last one alone in a second column tile)
    (1, 32, 64, 6, 480),        # a general width: 240 output columns
    (1, 64, 128, 4, 96),        # 64 -> 128, 48 output columns
])
def test_conv3d_s2_tc_one_plane(osb, b, cin, cout, h, w):
    """D = 1 is a stride-2 3x3 Conv2d: one output plane from the kd = 1 taps, either output layout, with a residual."""
    _, _, _, ops = osb
    assert ops.conv3d_s2_tc_supported(cin, cout, 1, h, w) and not ops.conv3d_s2_tc_supported(cin, cout, 3, h, w)
    x, wt, bias = rnd(300, b, cin, h, w), rnd(301, cout, cin, 3, 3, scale=0.2), rnd(302, cout, scale=0.1)
    want = F.conv2d(x.double(), wt.double(), bias.double(), stride=2, padding=1)
    w5 = torch.zeros(cout, cin, 3, 3, 3)
    w5[:, :, 1] = wt
    wp = ops.pack_tc_weight(w5.cuda(), 16, kw_order=(1, 0, 2))
    xc = x.permute(0, 2, 3, 1).contiguous().cuda().unsqueeze(1)                   # (B, 1, H, W, Cin)
    got = ops.conv3d_k3_s2_tc(xc, wp, None, bias.cuda())
    assert got.shape == (b, cout, 1, h // 2, w // 2)
    assert rel_err(got[:, :, 0], want.float()) <= 1e-5
    got = ops.conv3d_k3_s2_tc(xc, wp, None, bias.cuda(), None, ops.ACT_RELU, out_ndhwc=True)
    assert got.shape == (b, 1, h // 2, w // 2, cout)
    assert rel_err(got[:, 0].permute(0, 3, 1, 2), F.relu(want).float()) <= 1e-5
    res = rnd(303, b, cout, h // 2, w // 2)
    got = ops.conv3d_k3_s2_tc(xc, wp, None, bias.cuda(), res.unsqueeze(2).cuda(), ops.ACT_RELU)
    assert rel_err(got[:, :, 0], F.relu(want + res.double()).float()) <= 1e-5
    got = ops.conv3d_k3_s2_tc(xc, wp, None, bias.cuda(), res.permute(0, 2, 3, 1).contiguous().unsqueeze(1).cuda(), ops.ACT_NONE,
                              out_ndhwc=True, res_ndhwc=True)
    assert rel_err(got[:, 0].permute(0, 3, 1, 2), (want + res.double()).float()) <= 1e-5


def _gwc(hm):
    torch.manual_seed(7)
    return hm._fold_conv_bn(_randomise_bn(hm._GwcFeatureExtraction(True, 12).eval())).cuda()


def _psm(hm):
    torch.manual_seed(8)
    return hm._fold_conv_bn(_randomise_bn(hm._PsmBackbone().eval())).cuda()


@pytest.mark.parametrize("model", ["gwc", "psm"])
def test_stage_entry_routes(osb, model):
    """layer2[0] (stride 2, from the (B, 32, 128, 256) map of a 256x512 input) and layer3[0] (64 -> 128) of the BN-folded
    extractor on the wgmma route, against the module's own block on cuDNN; then the whole stage on a channels-last input, which
    hands a channels-last copy of its output on when asked."""
    lib, _, hm, ops = osb
    f = _gwc(hm) if model == "gwc" else _psm(hm)
    with torch.no_grad():
        x2 = torch.relu(rnd(310, 2, 32, 128, 256)).cuda()
        x3 = f.layer2(x2)
        for stage, x in ((f.layer2, x2), (f.layer3, x3)):
            blk = stage[0]
            assert hm._entry_tc_ok(blk, x.shape[1], x.shape[2], x.shape[3])
            t = x.permute(0, 2, 3, 1).contiguous()
            got = hm._entry_tc(f, blk, x, t, last=True)
            want = blk(x)
            assert got.shape == want.shape and rel_err(got, want) <= 2e-5
            got = hm._entry_tc(f, blk, x, t, last=False)                       # channels-last out, as the next block reads it
            assert rel_err(got.permute(0, 3, 1, 2), want) <= 2e-5
            want = stage(x)
            n0 = lib.launch_count()
            got, gt = hm._stage_tc(f, stage, x, t, nhwc_out=True)
            assert lib.launch_count() - n0 == 3 + 2 * (len(stage) - 1)                # entry (conv1, 1x1, conv2) + identity blocks
            assert got.is_contiguous() and rel_err(got, want) <= 1e-4 and torch.equal(gt.permute(0, 3, 1, 2), got)
            got, gt = hm._stage_tc(f, stage, x, t)
            assert gt is None and rel_err(got, want) <= 1e-4
        # from the channels-last view the tensor-core front hands over, and its NCHW view
        t2 = x2.permute(0, 3, 2, 1).contiguous().transpose(1, 2)
        got, _ = hm._stage_tc(f, f.layer2, t2.permute(0, 3, 1, 2), t2)
        assert rel_err(got, x3) <= 1e-4
        # an NCHW input from cuDNN layers keeps the entry block on cuDNN: layout change + the identity blocks only
        n0 = lib.launch_count()
        got, gt = hm._stage_tc(f, f.layer2, x2, None, nhwc_out=True)
        assert lib.launch_count() - n0 == 1 + 30 and gt is None and rel_err(got, x3) <= 1e-4


def test_stage_entry_without_a_variant_stays_cudnn(osb):
    """A 96-column map has no tensor-core route: the stages give the module's result exactly."""
    _, _, hm, _ = osb
    f = _gwc(hm)
    with torch.no_grad():
        x2 = torch.relu(rnd(320, 2, 32, 64, 192)).cuda()
        x3 = f.layer2(x2)
        assert not hm._entry_tc_ok(f.layer2[0], 32, 64, 192) and not hm._entry_tc_ok(f.layer3[0], 64, 32, 96)
        t2 = x2.permute(0, 2, 3, 1).contiguous()
        t3 = x3.permute(0, 2, 3, 1).contiguous()
        assert torch.equal(hm._stage_tc(f, f.layer2, x2, t2, nhwc_out=True)[0], x3)
        assert torch.equal(hm._stage_tc(f, f.layer3, x3, t3, nhwc_out=True)[0], f.layer3(x3))
        assert torch.equal(hm._stage_tc(f, f.layer2, t2.permute(0, 3, 1, 2), t2)[0], x3)


def test_gwc_extract_calls_cudnn_only_outside_the_kernels(osb):
    """At 256x512 every 3x3 residual conv of the extractor, the stage entries included, runs on this library: nn.Conv2d is
    called only for firstconv[0] (3 -> 32) and lastconv's 1x1 (128 -> 12)."""
    _, _, hm, _ = osb
    f = _gwc(hm)
    called = []
    orig = nn.Conv2d.forward

    def counting(self, x):
        called.append(self)
        return orig(self, x)

    nn.Conv2d.forward = counting
    try:
        with torch.no_grad():
            hm.gwc_extract(f, rnd(330, 2, 3, 256, 512).cuda())
    finally:
        nn.Conv2d.forward = orig
    convs = [m for m in f.firstconv.modules() if isinstance(m, nn.Conv2d)][:1] + \
        [m for m in f.lastconv.modules() if isinstance(m, nn.Conv2d)][1:]
    assert [id(m) for m in called] == [id(m) for m in convs]
