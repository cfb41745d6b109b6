"""GPU: CasStereo (CasPSMNet / CasGwcNet) on the sm_90a kernels -- the warped cost volumes and the hypothesis-weighted tail
against the CPU oracle (oracle/cascade.py, pinned bit-exactly to the reference), CascadeAggregation at both stage shapes, the
tensor-core routing of its convolutions, and patch() on the unmodified reference classes."""
import pytest
import torch

from oracle import _reference_shim as shim
from oracle import cascade as ocas
from oracle import seeded_init as si

from conftest import load_golden

pytestmark = pytest.mark.gpu

EPE_BAR = 1e-3
VOLUME_BAR = 1e-6


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, ops
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return _lib, ops


def rnd(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def samples(seed, b, d, h, w):
    """Fractional, integer and negative hypotheses; columns w - disp below -1, in (-1, 0) and beyond W - 1."""
    g = torch.Generator().manual_seed(seed)
    disp = torch.rand(b, d, h, w, generator=g) * (w + 8) - 6
    disp[:, 0] = torch.randint(-3, w + 3, (b, h, w), generator=g).float()
    disp[:, 1] = torch.arange(w).float() + 0.5
    disp[:, 2] = torch.arange(w).float() - (w - 1) - 0.25
    return disp


def _check_volume(got, want, masked=None):
    err = (got.cpu() - want).abs().max().item()
    assert err <= VOLUME_BAR, err
    if masked is not None:
        assert (got.cpu()[masked] == 0).all()                           # masked entries are exact zeros
    return err


# ------------------------------------------------------------------------------------------------ volumes
def test_volume_golden(osb):
    _, ops = osb
    g = load_golden("cas_volume_psm")
    got = ops.warped_concat_volume(g["x"].cuda(), g["y"].cuda(), g["disp"].cuda(), mask_left=False)
    _check_volume(got, g["out"])
    g = load_golden("cas_volume_gwc")
    got = ops.warped_gwc_concat_volume(g["xg"].cuda(), g["yg"].cuda(), g["xc"].cuda(), g["yc"].cuda(), g["disp"].cuda(), g["groups"])
    _check_volume(got, g["out"])


@pytest.mark.parametrize("b,c,d,h,w", [(1, 32, 12, 5, 150), (2, 16, 12, 2, 37), (2, 32, 12, 37, 64), (1, 16, 5, 3, 2)])
def test_psm_volume_vs_oracle(osb, b, c, d, h, w):
    _, ops = osb
    x, y, disp = rnd(1, b, c, h, w), rnd(2, b, c, h, w), samples(3, b, d, h, w)
    want = ocas.warped_concat_volume(x, y, disp, d)
    got = ops.warped_concat_volume(x.cuda(), y.cuda(), disp.cuda(), mask_left=False)
    _check_volume(got, want)
    # mask_left=True is CasGwcNet's concatenation half: left copy zeroed where w < disp
    masked = torch.arange(w).float().view(1, 1, 1, w).expand(b, d, h, w) < disp
    got = ops.warped_concat_volume(x.cuda(), y.cuda(), disp.cuda(), mask_left=True)
    want = want.clone()
    want[:, :c].transpose(0, 1)[:, masked] = 0
    _check_volume(got, want, masked.unsqueeze(1).expand(b, 2 * c, d, h, w) & (torch.arange(2 * c) < c).view(1, -1, 1, 1, 1))


@pytest.mark.parametrize("b,cg,g,cc,d,h,w", [(1, 320, 40, 12, 12, 4, 150), (2, 160, 20, 6, 12, 2, 37), (2, 24, 2, 3, 5, 13, 21),
                                             (1, 80, 10, 3, 12, 37, 64)])
def test_gwc_volume_vs_oracle(osb, b, cg, g, cc, d, h, w):
    _, ops = osb
    fl = {"gwc_feature": rnd(4, b, cg, h, w), "concat_feature": rnd(5, b, cc, h, w)}
    fr = {"gwc_feature": rnd(6, b, cg, h, w), "concat_feature": rnd(7, b, cc, h, w)}
    disp = samples(8, b, d, h, w)
    want = ocas.warped_gwc_concat_volume(fl, fr, disp, d, g)
    got = ops.warped_gwc_concat_volume(fl["gwc_feature"].cuda(), fr["gwc_feature"].cuda(), fl["concat_feature"].cuda(),
                                       fr["concat_feature"].cuda(), disp.cuda(), g)
    masked = torch.arange(w).float().view(1, 1, 1, w).expand(b, d, h, w) < disp
    sel = (torch.arange(g + 2 * cc) < g + cc).view(1, -1, 1, 1, 1) & masked.unsqueeze(1)
    err = _check_volume(got, want, sel.expand_as(want))
    print("CasGwcNet volume Cg/G=%d/%d Cc=%d: max |err| %.2e" % (cg, g, cc, err))


# ------------------------------------------------------------------------------------------------ tail
@pytest.mark.parametrize("tag", ["x4", "x2"])
def test_tail_golden(osb, tag):
    _, ops = osb
    g = load_golden("cas_tail")
    got = ops.upsample_softargmin_values(g["cost_" + tag].cuda(), g["values_" + tag].cuda()).cpu()
    e = (got - g["out_" + tag]).abs()
    assert e.mean().item() <= 1e-4 and e.max().item() <= 5e-4


@pytest.mark.parametrize("fine_d,hl,wl,scale", [(48, 16, 32, 4), (24, 32, 64, 2)])
def test_tail_vs_oracle(osb, fine_d, hl, wl, scale):
    _, ops = osb
    logits = rnd(20, 2, 1, 12, hl, wl) * 4
    h, w = 4 * hl if scale == 4 else 2 * hl, 4 * wl if scale == 4 else 2 * wl
    vals = samples(21, 2, fine_d, h, w) * 2
    want = ocas.upsample_softargmin_values(logits, fine_d, h, w, vals)
    got = ops.upsample_softargmin_values(logits.cuda(), vals.cuda()).cpu()
    e = (got - want).abs()
    print("tail 12 -> %d: mean %.2e max %.2e px" % (fine_d, e.mean().item(), e.max().item()))
    assert e.mean().item() <= 1e-4 and e.max().item() <= 5e-4


# ------------------------------------------------------------------------------------------------ engine
def _agg(in_channels, seed):
    m = ocas.CostAggregation(in_channels, 32).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=seed, scale={"classif3.2.weight": 40.0}))
    return m


STAGES_256x512 = [(64, 48, 64, 128), (32, 24, 128, 256)]          # (volume channels, FineD, H', W') of stages 1 / 2


@pytest.mark.parametrize("cin,fine_d,hh,ww", STAGES_256x512)
def test_cascade_aggregation_vs_oracle(osb, cin, fine_d, hh, ww):
    _, ops = osb
    from openstereo_b200.aggregation import CascadeAggregation
    oracle = _agg(cin, 30)
    cost = rnd(31, 1, cin, 12, hh, ww).abs()
    scale = 4 if fine_d == 48 else 2
    base = torch.linspace(1.5, 45.5, fine_d).view(1, fine_d, 1, 1) if fine_d == 48 else torch.arange(fine_d).float().view(1, -1, 1, 1)
    vals = (base + rnd(32, 1, 1, hh * scale, ww * scale) * 3).contiguous()
    with torch.no_grad():
        want = oracle(cost, fine_d, hh * scale, ww * scale, vals)
        got = CascadeAggregation(oracle.cuda())(cost.cuda(), fine_d, hh * scale, ww * scale, vals.cuda()).cpu()
    e = (got - want).abs().mean().item()
    print("CascadeAggregation stage %s: EPE %.3e px vs oracle (disp std %.2f)" % ((cin, hh, ww), e, want.std().item()))
    assert want.std() > 1 and e <= EPE_BAR


FP32_CONV_ENTRIES = ("osb_conv3d_k3_bn_act_fwd", "osb_deconv3d_bn_act_fwd")


@pytest.mark.parametrize("cin,hh,ww", [(64, 64, 128), (32, 128, 256), (64, 128, 240), (32, 256, 480)])
def test_cascade_aggregation_routing(osb, cin, hh, ww):
    """Every 3x3x3 convolution (and transposed convolution) at the stage shapes of 256x512 and 512x960 runs on a tensor-core
    instantiation: the fp32 CUDA-core 3x3x3 entry points are never called."""
    _, ops = osb
    from openstereo_b200.aggregation import CascadeAggregation
    eng = CascadeAggregation(_agg(cin, 33).cuda())
    cost = torch.rand(1, cin, 12, hh, ww, device="cuda")
    with torch.no_grad():
        eng.logits(cost)                                                # pack outside the profiled call
        torch.cuda.synchronize()
        ops.profile_start()
        eng.logits(cost)
        torch.cuda.synchronize()
        calls = {k: len(v) for k, v in ops.profile_stop().items()}
    print("CascadeAggregation (%d, 12, %d, %d): %s; last tc variant %s" % (cin, hh, ww, calls, ops.tc_last_variant()))
    assert not any(name in calls for name in FP32_CONV_ENTRIES), calls


# ------------------------------------------------------------------------------------------------ patch() on the reference
needs_ref = pytest.mark.skipif(not shim.available(), reason="reference tree (oracle/_ref) not staged")


def _casnet(module):
    cfg = shim.load_cfg("cfgs/casnet/casnet_psm_sceneflow.yaml").MODEL
    mod = shim.load("stereo.modeling.models.casnet." + module)
    m = (mod.PSMNet if module == "cas_psm" else mod.GwcNet)(cfg).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=1, scale=ocas.CASNET_SCALE if module == "cas_psm" else ocas.CASGWC_SCALE))
    return m


def _inputs(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return {"left": torch.randn(b, 3, h, w, generator=g), "right": torch.randn(b, 3, h, w, generator=g)}


@needs_ref
@pytest.mark.parametrize("module,seed", [("cas_psm", 40), ("cas_gwc", 41)])
def test_patch_cascade_256x512(osb, module, seed):
    lib, _ = osb
    from openstereo_b200.patch import patch
    m = _casnet(module)
    x = _inputs(1, 256, 512, seed)
    with torch.no_grad():
        want = m(dict(x))["disp_pred"]
        patch(m.cuda())
        before = lib.launch_count()
        got = m({k: v.cuda() for k, v in x.items()})["disp_pred"]
        launches = lib.launch_count() - before
    e = (got.cpu() - want).abs().mean().item()
    print("patch(%s) 256x512 EPE vs the reference on CPU: %.3e px (disp std %.2f), %d launches" % (module, e, want.std().item(), launches))
    assert got.shape == want.shape and got.is_cuda
    assert launches >= 2 * (1 + 20 + 1) and want.std() > 1 and e <= EPE_BAR


@needs_ref
def test_patch_cascade_training_on_cuda(osb):
    """strict=False: a CUDA training call runs the reference's own code (no kernel of this library), gradients intact."""
    lib, _ = osb
    from openstereo_b200.patch import patch
    m = patch(_casnet("cas_psm").cuda(), strict=False).train()
    x = {k: v.cuda() for k, v in _inputs(2, 256, 256, 42).items()}
    before = lib.launch_count()
    out = m(dict(x))
    assert lib.launch_count() == before
    out["disp_pred"].mean().backward()
    assert any(p.grad is not None and p.grad.abs().sum() > 0 for n, p in m.named_parameters() if n.startswith("feature_extraction."))
    strict = patch(_casnet("cas_psm").cuda()).train()
    with pytest.raises(RuntimeError, match="CUDA inference only"):
        strict(dict(x))
