"""CPU: CasStereo (CasPSMNet / CasGwcNet) -- the oracle against its fixtures and the live reference, the new C-ABI entry
points, and patch()'s drop-in contract on the unmodified reference classes (no compute on a GPU here)."""
import pytest
import torch

from oracle import _reference_shim as shim
from oracle import cascade as ocas
from oracle import seeded_init as si

from conftest import load_golden

needs_ref = pytest.mark.skipif(not shim.available(), reason="reference tree not present")


def rnd(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


# ------------------------------------------------------------------------------------------ oracle vs fixtures
def test_oracle_volumes_golden():
    g = load_golden("cas_volume_psm")
    assert torch.equal(ocas.warped_concat_volume(g["x"], g["y"], g["disp"], g["disp"].shape[1]), g["out"])
    g = load_golden("cas_volume_gwc")
    fl, fr = {"gwc_feature": g["xg"], "concat_feature": g["xc"]}, {"gwc_feature": g["yg"], "concat_feature": g["yc"]}
    assert torch.equal(ocas.warped_gwc_concat_volume(fl, fr, g["disp"], g["disp"].shape[1], g["groups"]), g["out"])


@pytest.mark.parametrize("tag", ["x4", "x2"])
def test_oracle_tail_golden(tag):
    g = load_golden("cas_tail")
    vals = g["values_" + tag]
    out = ocas.upsample_softargmin_values(g["cost_" + tag], vals.shape[1], vals.shape[2], vals.shape[3], vals)
    assert torch.equal(out, g["out_" + tag])


# ------------------------------------------------------------------------------------------ oracle vs live reference
@needs_ref
@pytest.mark.parametrize("b,c,d,h,w", [(2, 5, 6, 7, 19), (1, 3, 12, 37, 9), (1, 4, 3, 2, 2)])
def test_oracle_pins_volumes(b, c, d, h, w):
    rpsm = shim.load("stereo.modeling.models.casnet.cas_psm")
    rgwc = shim.load("stereo.modeling.models.casnet.cas_gwc")
    disp = torch.rand(b, d, h, w, generator=torch.Generator().manual_seed(3)) * (w + 6) - 4
    x, y = rnd(1, b, c, h, w), rnd(2, b, c, h, w)
    assert torch.equal(rpsm.GetCostVolume()(x, y, disp, d), ocas.warped_concat_volume(x, y, disp, d))
    fl = {"gwc_feature": rnd(4, b, 2 * c, h, w), "concat_feature": rnd(5, b, c, h, w)}
    fr = {"gwc_feature": rnd(6, b, 2 * c, h, w), "concat_feature": rnd(7, b, c, h, w)}
    assert torch.equal(rgwc.GetCostVolume()(fl, fr, disp, d, c), ocas.warped_gwc_concat_volume(fl, fr, disp, d, c))


@needs_ref
@pytest.mark.parametrize("module", ["cas_psm", "cas_gwc"])
def test_oracle_pins_cost_aggregation(module):
    ref_cls = shim.load("stereo.modeling.models.casnet." + module).CostAggregation
    with torch.no_grad():
        ref, mine = ref_cls(16, 8).eval(), ocas.CostAggregation(16, 8).eval()
        assert list(ref.state_dict()) == list(mine.state_dict())
        sd = si.seeded_state_dict(ref.state_dict(), seed=8)
        ref.load_state_dict(sd), mine.load_state_dict(sd)
        cost, vals = rnd(9, 1, 16, 12, 8, 12), torch.rand(1, 48, 32, 48, generator=torch.Generator().manual_seed(10)) * 90 - 5
        assert torch.equal(ref(cost, 48, 32, 48, vals), mine(cost, 48, 32, 48, vals))


@needs_ref
def test_reference_casnet_reproduces_golden():
    g = load_golden("cas_psmnet_256x512")
    m = _casnet("cas_psm")
    assert si_checksum(m.state_dict()) == pytest.approx(g["checksum"], rel=1e-12)
    with torch.no_grad():
        out = m({"left": rnd(g["seed_left"], 1, 3, 256, 512), "right": rnd(g["seed_right"], 1, 3, 256, 512)})["disp_pred"]
    assert torch.equal(out[:, ::8, ::8], g["disp_sample"])


def si_checksum(sd):
    return float(sum(v.double().abs().sum() for v in sd.values()))


# ------------------------------------------------------------------------------------------ C ABI and ops
def test_new_entry_points_bound():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, ops
    for name in ("osb_warped_concat_volume_fwd", "osb_warped_gwc_concat_volume_fwd", "osb_upsample_softargmin_values_fwd"):
        assert name in _lib.SIGNATURES and hasattr(_lib.lib, name)
    with pytest.raises(ValueError, match="null pointer"):
        _lib.call("osb_warped_concat_volume_fwd", None, None, None, None, 1, 4, 2, 4, 4, 0, None)
    with pytest.raises(ValueError, match="must be >= 2"):            # the grid divides by (H - 1) / 2
        _lib.call("osb_warped_concat_volume_fwd", 16, 16, 16, 16, 1, 4, 2, 1, 4, 0, None)
    with pytest.raises(ValueError, match="not divisible"):
        _lib.call("osb_warped_gwc_concat_volume_fwd", 16, 16, 16, 16, 16, 16, 1, 12, 5, 3, 2, 4, 4, None)
    x, disp = torch.randn(1, 4, 3, 8), torch.randn(1, 2, 3, 8)
    with pytest.raises(RuntimeError, match="not implemented on the CPU"):
        ops.warped_concat_volume(x, x, disp)
    with pytest.raises(RuntimeError, match="not implemented on the CPU"):
        ops.upsample_softargmin_values(torch.randn(1, 1, 2, 3, 4), torch.randn(1, 8, 6, 8))
    with pytest.raises(RuntimeError, match="no backward"):
        ops.warped_concat_volume(x.requires_grad_(), x, disp)


# ------------------------------------------------------------------------------------------ patch() contract
def _casnet(module, scale=None):
    cfg = shim.load_cfg("cfgs/casnet/casnet_psm_sceneflow.yaml").MODEL
    mod = shim.load("stereo.modeling.models.casnet." + module)
    m = (mod.PSMNet if module == "cas_psm" else mod.GwcNet)(cfg).eval()
    scale = scale if scale is not None else (ocas.CASNET_SCALE if module == "cas_psm" else ocas.CASGWC_SCALE)
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=1, scale=scale))
    return m


def _inputs(h, w, seed, b=1):
    g = torch.Generator().manual_seed(seed)
    return {"left": torch.randn(b, 3, h, w, generator=g), "right": torch.randn(b, 3, h, w, generator=g)}


@needs_ref
@pytest.mark.parametrize("module", ["cas_psm", "cas_gwc"])
def test_patch_cascade_contract(module):
    from openstereo_b200.patch import patch
    m = _casnet(module)
    keys = list(m.state_dict().keys())
    x = _inputs(256, 256, 3)
    with torch.no_grad():
        want = m(dict(x))["disp_pred"]
        assert patch(m, strict=False) is m and m._osb_patched
        assert "forward" in vars(m.get_cv) and all("forward" in vars(a) for a in m.cost_agg)   # the cascade patcher ran
        assert patch(m, strict=False) is m                              # idempotent
        assert list(m.state_dict().keys()) == keys
        assert torch.equal(m(dict(x))["disp_pred"], want)               # CPU call delegated to the reference's own code
        strict = patch(_casnet(module))
        with pytest.raises(RuntimeError, match="CUDA inference only"):
            strict(dict(x))


@needs_ref
def test_patch_cascade_training_keeps_gradients():
    from openstereo_b200.patch import patch
    m = patch(_casnet("cas_psm"), strict=False).train()
    out = m(dict(_inputs(256, 256, 5, b=2)))                            # training BatchNorm needs > 1 value per channel
    loss = sum(out["stage%d" % (i + 1)][k].mean() for i in range(2) for k in ("pred0", "pred1", "pred2", "pred3"))
    loss.backward()
    grads = [p.grad for n, p in m.named_parameters() if n.startswith("cost_agg.") and ".classif3." in n]
    assert all(g is not None for g in grads) and any(g.abs().sum() > 0 for g in grads)
    assert any(p.grad is not None and p.grad.abs().sum() > 0 for n, p in m.named_parameters() if n.startswith("feature_extraction."))


@needs_ref
def test_patch_routes_by_defining_module():
    """CasStereo's classes share their names with psmnet.psmnet.PSMNet and gwcnet.gwcnet.GwcNet; each keeps its own patcher."""
    from openstereo_b200 import patch as P
    psm = shim.load("stereo.modeling.models.psmnet.psmnet").PSMNet(shim.load_cfg("cfgs/psmnet/psmnet_sceneflow.yaml").MODEL).eval()
    P.patch(psm, strict=False)
    assert "forward" in vars(psm.CostProcessor) and "forward" in vars(psm.DispProcessor.disp_processor)
    gwc = shim.load("stereo.modeling.models.gwcnet.gwcnet").GwcNet(shim.load_cfg("cfgs/gwcnet/gwcnet_sceneflow.yaml").MODEL).eval()
    P.patch(gwc, strict=False)
    assert "forward" in vars(gwc.CostProcessor) and "forward" in vars(gwc.DispProcessor)
    for module in ("cas_psm", "cas_gwc"):
        m = P.patch(_casnet(module, scale={}), strict=False)
        assert "forward" in vars(m.get_cv)
