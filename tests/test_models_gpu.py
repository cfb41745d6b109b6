"""GPU: module- and model-level parity.  The CUDA engines (openstereo_b200.aggregation / host_models) are fed the
SAME seeded, non-degenerate weights as the CPU oracle (oracle.seeded_init) and compared with the oracle's output and
with the committed golden vectors (which came from the unmodified reference).

Bar (BASELINE.json north_star): disparity EPE vs the reference <= 1e-3 px in fp32."""
import pytest
import torch

from conftest import load_golden

pytestmark = pytest.mark.gpu

from oracle import aggregation as oagg     # noqa: E402
from oracle import models as omodels       # noqa: E402
from oracle import seeded_init as si       # noqa: E402

EPE_BAR = 1e-3


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    import openstereo_b200
    from openstereo_b200 import aggregation, host_models, ops
    return openstereo_b200, aggregation, host_models, ops


def rel_err(got, want):
    return ((got.detach().cpu() - want).abs().max() / (want.abs().max() + 1e-12)).item()


def epe(got, want):
    return (got.detach().cpu() - want).abs().mean().item()


def test_gwc_hourglass_golden(osb):
    _, agg, _, _ = osb
    g = load_golden("gwc_hourglass_c8")
    m = oagg.GwcHourglass(8).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=g["seed"]))
    m.cuda()
    with torch.no_grad():
        hg = agg._GwcHourglass(m)
        got = hg(g["x"].cuda())
    assert rel_err(got, g["out"]) <= 1e-5


def test_gwc_disp_processor_golden(osb):
    _, agg, _, _ = osb
    g = load_golden("gwc_disp_processor")
    m = oagg.GwcDispProcessor(maxdisp=32, downsample=4, num_groups=4, use_concat_volume=True, concat_channels=2).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=g["seed"], scale={"classif3.2.weight": 60.0}))
    m.cuda()
    engine = agg.GwcAggregation(m)
    logits = engine.logits(g["volume"].cuda())
    assert rel_err(logits, g["logits"]) <= 2e-5
    disp = engine(g["volume"].cuda(), 32, 64)
    assert epe(disp, g["out"]) <= EPE_BAR * 0.1 and g["out"].std() > 1.0


def test_psm_aggregator_golden(osb):
    _, agg, _, _ = osb
    g = load_golden("psm_aggregator")
    m = oagg.PSMAggregator(32, 8).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=g["seed"], scale={
        "classif1.1.weight": 20.0, "classif2.1.weight": 20.0, "classif3.1.weight": 20.0}))
    m.cuda()
    engine = agg.PSMAggregation(m)
    c1, c2, c3 = engine.logits(g["raw"].cuda())
    assert rel_err(c1, g["cost1_low"]) <= 2e-5 and rel_err(c2, g["cost2_low"]) <= 2e-5 and rel_err(c3, g["cost3_low"]) <= 2e-5
    with torch.no_grad():
        want = m.cpu()(g["raw"])                                  # [cost3, cost2, cost1] upsampled (B,32,H,W)
    from oracle import regression as oreg
    m.cuda()
    disps = engine(g["raw"].cuda())
    assert epe(disps[2], oreg.faster_soft_argmin(want[0], 32)) <= EPE_BAR * 0.1


def test_stereobase_head_golden(osb):
    _, agg, _, _ = osb
    g = load_golden("stereobase_head")
    m = oagg.StereoBaseCostHead(8, [16, 16, 24, 20], max_disp=64).eval()
    sd = si.seeded_state_dict(m.state_dict(), seed=g["seed_head"], scale={"classifier.weight": 30.0})
    sd_h = si.seeded_state_dict(m.cost_agg.state_dict(), seed=g["seed_hourglass"])
    sd.update({"cost_agg." + k: v for k, v in sd_h.items()})
    m.load_state_dict(sd)
    m.cuda()
    feats = [g["f0"].cuda(), g["f1"].cuda(), g["f2"].cuda(), g["f3"].cuda()]
    geo = agg.StereoBaseAggregation(m.cost_agg)(g["volume"].cuda(), feats)
    assert rel_err(geo, g["geo"]) <= 2e-5
    init = agg.StereoBaseCostHead(m.classifier)(geo, 16)
    assert init.shape == g["init_disp"].shape
    assert (init.cpu() - g["init_disp"]).abs().max().item() <= 1e-4


def test_stereobase_config3_subgraph(osb):
    """Config 3 per-GPU shapes (gwc C=96 G=8 + concat C=8 -> Hourglass(24,[96,64,192,160]) -> classifier -> soft-argmin),
    batch 1, synthetic features; oracle on CPU."""
    _, agg, _, ops = osb
    from oracle import cost_volume as ocv
    gen = torch.Generator().manual_seed(7)
    r = lambda *s: torch.randn(*s, generator=gen)
    ml, mr, cl, cr = r(1, 96, 32, 64), r(1, 96, 32, 64), r(1, 8, 32, 64), r(1, 8, 32, 64)
    feats = [r(1, 96, 32, 64), r(1, 64, 16, 32), r(1, 192, 8, 16), r(1, 160, 4, 8)]
    m = oagg.StereoBaseCostHead(24, [96, 64, 192, 160], max_disp=192).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=9, scale={"classifier.weight": 150.0}))
    with torch.no_grad():
        vol = torch.cat((ocv.build_gwc_volume(ml, mr, 48, 8), ocv.build_concat_volume(cl, cr, 48)), 1)
        geo_want, init_want = m(vol, feats)
    m.cuda()
    vol_got = ops.gwc_concat_volume(ml.cuda(), mr.cuda(), cl.cuda(), cr.cuda(), 48, 8)
    assert (vol_got.cpu() - vol).abs().max().item() <= 1e-6
    geo = agg.StereoBaseAggregation(m.cost_agg)(vol_got, [f.cuda() for f in feats])
    assert rel_err(geo, geo_want) <= 5e-5
    init = agg.StereoBaseCostHead(m.classifier)(geo, 48)
    assert epe(init, init_want) <= EPE_BAR * 0.1 and init_want.std() > 0.5


def _gwcnet_pair(osb):
    _, _, hm, _ = osb
    oracle = omodels.GwcNet().eval()
    sd = si.seeded_state_dict(oracle.state_dict(), seed=1, scale=si.GWCNET_SCALE)
    oracle.load_state_dict(sd)
    mine = hm.GwcNet({"MAX_DISP": 192, "USE_CONCAT_VOLUME": True, "CONCAT_CHANNELS": 12, "DOWNSAMPLE": 4, "NUM_GROUPS": 40})
    mine.load_state_dict(sd)                                       # unchanged reference key names
    return oracle, mine.eval().cuda()


def test_gwcnet_golden_epe(osb):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    g = load_golden("gwcnet_64x128")
    oracle, mine = _gwcnet_pair(osb)
    with torch.no_grad():
        got = mine({"left": g["left"].cuda(), "right": g["right"].cuda()})["disp_pred"]
    assert got.shape == g["out"].shape and got.dtype == torch.float32
    e = epe(got, g["out"])
    print("GwcNet 64x128 EPE vs reference golden: %.3e" % e)
    assert e <= EPE_BAR and g["out"].std() > 10


def test_gwcnet_hot_path_isolated(osb):
    """Feed the ORACLE's backbone features to the CUDA hot path, so the comparison isolates volume + aggregation +
    soft-argmin from cuDNN-vs-MKLDNN differences in the (out-of-scope) 2D backbone."""
    g = load_golden("gwcnet_64x128")
    oracle, mine = _gwcnet_pair(osb)
    with torch.no_grad():
        lf, rf = oracle.Backbone(g["left"], g["right"])
        vol = oracle.CostProcessor(lf, rf)
        want = oracle.DispProcessor(vol, 64, 128)
        inputs = {"left": g["left"].cuda(),
                  "ref_feature": {k: v.cuda() for k, v in lf.items()}, "tgt_feature": {k: v.cuda() for k, v in rf.items()}}
        inputs.update(mine.CostProcessor(inputs))
        assert (inputs["cost_volume"].cpu() - vol).abs().max().item() <= 1e-5
        got = mine.DispProcessor(inputs)["inference_disp"]["disp_est"]
    e = epe(got, want)
    print("GwcNet hot path EPE vs oracle: %.3e (max %.3e)" % (e, (got.cpu() - want).abs().max().item()))
    assert e <= EPE_BAR * 0.2


def test_psmnet_golden_epe(osb):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    _, _, hm, _ = osb
    g = load_golden("psmnet_256x256")
    oracle = omodels.PSMNet().eval()
    sd = si.seeded_state_dict(oracle.state_dict(), seed=g["seed"], scale=si.PSMNET_SCALE, keep=si.PSMNET_KEEP)
    mine = hm.PSMNet({"MAX_DISP": 192})
    mine.load_state_dict(sd)
    mine.eval().cuda()
    with torch.no_grad():
        out = mine({"left": g["left"].cuda(), "right": g["right"].cuda()})
    assert len(out["train_preds"]) == 3                             # all three heads run in eval, like the reference
    e = epe(out["disp_pred"], g["out"])
    print("PSMNet 256x256 EPE vs reference golden: %.3e" % e)
    assert e <= EPE_BAR and g["out"].std() > 10


def test_engine_refuses_training_and_cpu(osb):
    _, agg, hm, _ = osb
    m = oagg.GwcDispProcessor(maxdisp=32, num_groups=4, concat_channels=2).cuda()
    m.train()
    with pytest.raises(RuntimeError, match="eval"):
        agg.GwcAggregation(m).logits(torch.randn(1, 8, 8, 8, 16, device="cuda"))
    m.eval()
    with pytest.raises(RuntimeError, match="CPU"):
        agg.GwcAggregation(m).logits(torch.randn(1, 8, 8, 8, 16))


def test_engine_repacks_after_weight_update(osb):
    _, agg, _, _ = osb
    m = oagg.GwcDispProcessor(maxdisp=32, num_groups=4, concat_channels=2).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=3))
    m.cuda()
    eng = agg.GwcAggregation(m)
    x = torch.randn(1, 8, 8, 8, 16, device="cuda")
    a = eng.logits(x).clone()
    with torch.no_grad():
        m.classif3[2].weight.mul_(2.0)
    b = eng.logits(x)
    assert torch.allclose(b, 2.0 * a, rtol=1e-5, atol=1e-6)


def test_gwc_aggregation_full_width_tensor_cores(osb):
    """W' = 128 (a 512-pixel-wide input): the stem and classifier convs run on the wgmma 3xFP16 kernel.  Compared with
    the CPU oracle on a short volume (D'=8, H'=10) and with the CUDA-core path of the same engine."""
    _, agg, _, _ = osb
    m = oagg.GwcDispProcessor(maxdisp=32, downsample=4, num_groups=40, use_concat_volume=True, concat_channels=12).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=41, scale={"classif3.2.weight": 60.0}))
    vol = torch.randn(1, 64, 8, 12, 128, generator=torch.Generator().manual_seed(42))
    with torch.no_grad():
        want_logits = m.aggregate(vol)
        want = m(vol, 48, 512)
    m.cuda()
    eng = agg.GwcAggregation(m)
    assert agg.USE_TENSOR_CORES and eng._ensure(torch.device("cuda", 0)) is None and agg._tc_ok(eng.dres0[0], 128)
    assert agg._tc_ok(eng.hg[0].conv2, 64) and agg._tc_ok(eng.hg[0].conv4, 32)     # hourglass interiors too
    assert agg._hg_channels_last_ok(eng.hg[0], (1, 8, 12, 128, 32))                 # ... with no layout change in between
    got_logits = eng.logits(vol.cuda())
    assert rel_err(got_logits, want_logits) <= 5e-5
    got = eng(vol.cuda(), 48, 512)
    e = epe(got, want)
    print("GwcNet aggregation (tensor-core stem) EPE vs oracle: %.3e" % e)
    assert e <= EPE_BAR * 0.2 and want.std() > 1.0
    agg.USE_TENSOR_CORES = False
    try:
        ref_logits = agg.GwcAggregation(m).logits(vol.cuda())
    finally:
        agg.USE_TENSOR_CORES = True
    assert rel_err(got_logits, ref_logits.cpu()) <= 5e-5


def test_backbone_front_tensor_cores(osb):
    """256-row inputs: firstconv[1:] + layer1 (eight 32->32 3x3 convs at 1/2 resolution) run on the wgmma conv kernel
    through the transposed-image mapping.  Compared with cuDNN on the same BN-folded weights and with the unfolded module
    on the CPU (fp32); 3xTF32 keeps fp32 accuracy, so the tolerance is the usual accumulation-order one."""
    _, agg, hm, _ = osb
    torch.manual_seed(7)
    m = hm._GwcFeatureExtraction(True, 12).eval()
    with torch.no_grad():
        for mod in m.modules():                              # non-trivial BN statistics so that the folding matters
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.running_mean.normal_(0, 0.2), mod.running_var.uniform_(0.5, 1.5)
                mod.weight.uniform_(0.5, 1.5), mod.bias.normal_(0, 0.2)
        x = torch.randn(2, 3, 256, 96)
        want_cpu = m.layer1(m.firstconv(x))
        x512 = torch.randn(1, 3, 32, 512)                    # 1/4-resolution width 128: layer2 / layer3 blocks on tensor cores
        want512 = m(x512)["gwc_feature"]
        f = hm._fold_conv_bn(m).cuda()
        xg = x.cuda()
        assert hm._front_tc_ok(f, xg) and not hm._front_tc_ok(f, xg[:, :, :128])
        got = hm._front_tc(f, xg)
        cudnn = f.layer1(f.firstconv(xg))
        assert got.shape == cudnn.shape == (2, 32, 128, 48) and got.is_contiguous()
        assert rel_err(got, cudnn.cpu()) <= 2e-5
        assert rel_err(got, want_cpu) <= 5e-5
        full = f(xg)                                         # the whole extractor takes the tensor-core front by itself
        agg.USE_TENSOR_CORES = False
        try:
            ref = f(xg)
        finally:
            agg.USE_TENSOR_CORES = True
        assert rel_err(full["gwc_feature"], ref["gwc_feature"].cpu()) <= 5e-5
        # residual stages: 15 + 2 + 3 (dilated) blocks of layer2 / layer3 / layer4 leave cuDNN when the 1/4-resolution map is 128 wide
        from openstereo_b200 import _lib
        before = _lib.launch_count()
        full512 = f(x512.cuda())
        got512 = full512["gwc_feature"]
        # layout change + convs of layer2, layer3, layer4 (dilated), lastconv's 320->128 3x3
        assert _lib.launch_count() - before == (1 + 30) + (1 + 4) + (1 + 6) + (1 + 1)
        assert rel_err(got512, want512) <= 1e-4
        assert rel_err(full512["concat_feature"], m(x512)["concat_feature"]) <= 1e-4
        agg.USE_TENSOR_CORES = False
        try:
            ref512 = f(x512.cuda())["gwc_feature"]
        finally:
            agg.USE_TENSOR_CORES = True
        assert rel_err(got512, ref512.cpu()) <= 1e-4
