"""CPU: CoEx -- the oracle against its fixtures and the live reference, the top-k tie order, aten's nearest index, the new C-ABI
entry points, and patch()'s drop-in contract on the unmodified reference class (no compute on a GPU here)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import _reference_shim as shim
from oracle import coex as ocx
from oracle import seeded_init as si

from conftest import load_golden

needs_ref = pytest.mark.skipif(not shim.available(), reason="reference tree not present")


def rnd(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def checksum(sd):
    return float(sum(v.double().abs().sum() for v in sd.values()))


# ------------------------------------------------------------------------------------------ oracle vs fixtures
def test_oracle_golden():
    g = load_golden("coex_attention")
    assert torch.equal(ocx.attention_volume(g["x"], g["y"], g["maxdisp"], g["head"]), g["out"])
    g = load_golden("coex_regression")
    for k in (2, 3):
        assert torch.equal(ocx.regression(g["cost"], g["spx"], k), g["out_k%d" % k])
        assert torch.equal(ocx.topk_pool(g["cost"], k)[1], g["ind_k%d" % k])
    g = load_golden("coex_nearest")
    for i in range(3):
        size = tuple(int(v) for v in g["size%d" % i])
        assert torch.equal(F.interpolate(g["x"], size=size, mode="nearest"), g["out%d" % i])


def test_oracle_aggregation_golden():
    g = load_golden("coex_aggregation")
    m = ocx.Aggregation(max_disparity=64).eval()
    sd = si.seeded_state_dict(m.state_dict(), seed=g["weight_seed"])
    assert checksum(sd) == pytest.approx(g["checksum"], rel=1e-12)
    m.load_state_dict(sd)
    with torch.no_grad():
        out = m([g["img0"], g["img1"], g["img2"], g["img3"]], g["cost"])
    assert torch.equal(out, g["out"])


def test_ties_choose_lower_index():
    cost = torch.tensor([1.0, 3.0, 3.0, 0.0, 3.0, 2.0, 3.0]).view(1, 1, 7, 1, 1)
    assert ocx.topk_pool(cost, 2)[1].flatten().tolist() == [1, 2]
    assert ocx.topk_pool(cost, 5)[1].flatten().tolist() == [1, 2, 4, 6, 5]
    g = load_golden("coex_regression")                                 # the fixture's logits hold many exact ties
    vals, ind = ocx.topk_pool(g["cost"], 3)
    tie = vals[:, :, 1:] == vals[:, :, :-1]
    assert tie.any() and (ind[:, :, 1:] > ind[:, :, :-1])[tie].all()


def test_cpu_sort_tie_order_beyond_16_planes():
    """aten's default CPU sort keeps exact ties in index order only up to 16 planes (its insertion-sort range); at CoEx's D = 48 the
    order of equal values is the introsort's, which is why the kernel's lower-index-first rule is pinned to the stable sort there."""
    for d, in_order in ((10, True), (16, True), (48, False)):
        ind = ocx.topk_pool(torch.zeros(1, 1, d, 1, 1), d)[1].flatten()
        assert torch.equal(ind, torch.arange(d)) == in_order
        assert torch.equal(ocx.topk_pool(torch.zeros(1, 1, d, 1, 1), d, stable=True)[1].flatten(), torch.arange(d))


@pytest.mark.parametrize("n_in,n_out", [(136, 135), (26, 25), (14, 13), (48, 48), (24, 48), (7, 3), (5, 13)])
def test_nearest_index_matches_interpolate(n_in, n_out):
    idx = ocx.nearest_index(n_out, n_in)
    for dim in range(3):
        shape, size = [3, 4, 5], [3, 4, 5]
        shape[dim], size[dim] = n_in, n_out
        x = rnd(dim, 1, 2, *shape)
        want = F.interpolate(x, size=tuple(size), mode="nearest")
        assert torch.equal(torch.index_select(x, 2 + dim, torch.tensor(idx)), want)


# ------------------------------------------------------------------------------------------ oracle vs live reference
@needs_ref
@pytest.mark.parametrize("k", [2, 3, 5, 8])
def test_oracle_pins_regression(k):
    rdp = shim.load("stereo.modeling.models.coex.coex_disp_processor")
    cost = torch.cat((rnd(1, 2, 1, 24, 5, 9), torch.randint(0, 3, (2, 1, 24, 5, 9), generator=torch.Generator().manual_seed(2)).float()), 2)
    spx = torch.softmax(rnd(3, 2, 9, 20, 36), 1)
    with torch.no_grad():
        assert torch.equal(rdp.Regression(192, k).eval()(cost, spx)[0], ocx.regression(cost, spx, k))


@needs_ref
@pytest.mark.parametrize("gce", [True, False])
def test_oracle_pins_aggregation(gce):
    rcp = shim.load("stereo.modeling.models.coex.coex_cost_processor")
    ref, mine = rcp.Aggregation(max_disparity=64, gce=gce).eval(), ocx.Aggregation(max_disparity=64, gce=gce).eval()
    assert sorted(ref.state_dict()) == sorted(mine.state_dict())
    sd = si.seeded_state_dict(ref.state_dict(), seed=5)
    ref.load_state_dict(sd), mine.load_state_dict(sd)
    img = [rnd(6, 1, 96, 13, 10), rnd(7, 1, 64, 7, 5), rnd(8, 1, 192, 4, 3), rnd(9, 1, 160, 2, 2)]
    cost = rnd(10, 1, 1, 16, 13, 10)
    with torch.no_grad():
        assert torch.equal(ref(img, cost), mine(img, cost))


# ------------------------------------------------------------------------------------------ C ABI and ops
def test_new_entry_points_bound():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, ops
    for name in ("osb_coex_regression_fwd", "osb_nearest_resize3d_fwd"):
        assert name in _lib.SIGNATURES and hasattr(_lib.lib, name)
    with pytest.raises(ValueError, match="null pointer"):
        _lib.call("osb_coex_regression_fwd", None, None, None, 1, 8, 2, 2, 2, 1, None)
    with pytest.raises(ValueError, match="top_k=1 not supported"):
        _lib.call("osb_coex_regression_fwd", 16, 16, 16, 1, 8, 2, 2, 1, 1, None)
    with pytest.raises(ValueError, match="exceeds"):
        _lib.call("osb_coex_regression_fwd", 16, 16, 16, 1, 4, 2, 2, 5, 1, None)
    with pytest.raises(ValueError, match="null pointer"):
        _lib.call("osb_nearest_resize3d_fwd", None, None, 1, 2, 2, 2, 2, 2, 2, None)
    with pytest.raises(RuntimeError, match="not implemented on the CPU"):
        ops.coex_regression(torch.randn(1, 1, 8, 2, 3), torch.randn(1, 9, 8, 12), 2)
    with pytest.raises(RuntimeError, match="not implemented on the CPU"):
        ops.nearest_resize3d(torch.randn(1, 2, 3, 4, 5), (3, 3, 3))
    with pytest.raises(RuntimeError, match="no backward"):
        ops.coex_regression(torch.randn(1, 1, 8, 2, 3, requires_grad=True), torch.randn(1, 9, 8, 12), 2)
    with pytest.raises(RuntimeError, match="no backward"):
        ops.coex_attention_volume(torch.randn(1, 4, 2, 3, requires_grad=True), torch.randn(1, 4, 2, 3), 2)


# ------------------------------------------------------------------------------------------ patch() contract
def _coex(**overrides):
    shim.install_timm_stub()
    cfg = shim.load_cfg("cfgs/coex/coex_sceneflow_amp.yaml").MODEL
    cfg.update(overrides)
    m = shim.load("stereo.modeling.models.coex.coex").CoEx(cfg).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=1))
    return m


def _inputs(h, w, seed, b=1):
    g = torch.Generator().manual_seed(seed)
    return {"left": torch.randn(b, 3, h, w, generator=g), "right": torch.randn(b, 3, h, w, generator=g)}


@needs_ref
def test_patch_coex_contract():
    from openstereo_b200.patch import patch, _patch_coex, _PATCHERS
    assert _PATCHERS["CoEx"] is _patch_coex
    m = _coex()
    keys = list(m.state_dict().keys())
    x = _inputs(128, 256, 3)
    with torch.no_grad():
        want = m(dict(x))["disp_pred"]
        assert patch(m, strict=False) is m and m._osb_patched
        assert all("forward" in vars(mod) for mod in (m.CostProcessor, m.DispProcessor, m.DispProcessor.regression))
        assert patch(m, strict=False) is m                              # idempotent
        assert list(m.state_dict().keys()) == keys
        assert torch.equal(m(dict(x))["disp_pred"], want)               # CPU call delegated to the reference's own code
        strict = patch(_coex())
        with pytest.raises(RuntimeError, match="CUDA inference only"):
            strict(dict(x))
        with pytest.raises(RuntimeError, match="CUDA inference only"):
            strict.DispProcessor.regression(torch.randn(1, 1, 48, 4, 5), torch.softmax(torch.randn(1, 9, 16, 20), 1))


@needs_ref
@pytest.mark.parametrize("setting,value", [("REGRESSION_TOPK", 1), ("REGRESSION_TOPK", 9), ("AGGREGATION_DISP_STRIDES", 1),
                                           ("MATCHING_WEIGHTED", True)])
def test_patch_coex_refuses_unsupported(setting, value):
    from openstereo_b200.patch import patch
    m = _coex(**{setting: value})
    with pytest.raises(NotImplementedError, match=setting):
        patch(m, strict=False)
    assert not getattr(m, "_osb_patched", False)
