"""CPU: CFNet's patch surface (routing, the per-instance override, state_dict, refusals), serves(), the OSB_ACT_MISH constant and
its Python twin, and the fp64 oracle (oracle/cfnet.py) against the reference's own formulas."""
import os
import re

import pytest
import torch
import torch.nn.functional as F

from oracle import _reference_shim as shim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not shim.available(), reason="reference tree not staged")


@pytest.fixture(scope="module")
def native():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import ops, patch
    return ops, patch


def test_mish_constant_and_its_twin(native):
    ops, _ = native
    text = open(os.path.join(ROOT, "include", "openstereo_b200.h")).read()
    assert int(re.search(r"#define OSB_ACT_MISH (\d+)", text).group(1)) == ops.ACT_MISH == 6
    consts = {int(v) for v in re.findall(r"#define OSB_ACT_\w+ (\d+)", text)}
    assert len(consts) == len(re.findall(r"#define OSB_ACT_\w+ (\d+)", text)), "two activations share a code"


@needs_ref
def test_patch_surface(native):
    from oracle.cfnet import reference_model
    _, patch = native
    m, other = reference_model(), reference_model()
    keys = list(m.state_dict())
    assert type(m).__name__ == "cfnet" and type(m).__module__.split(".")[-2:] == ["cfnet", "cfnet"]
    assert patch._MODULE_PATCHERS[("cfnet", "cfnet", "cfnet")] is patch._patch_cfnet
    patch.patch(m)
    assert list(m.state_dict()) == keys
    assert "forward" in vars(m) and "forward" not in vars(other), "the override is per instance"
    assert type(m).forward is type(other).forward
    with pytest.raises(RuntimeError, match="CUDA inference only"):          # CPU call, strict
        m({"left": torch.zeros(1, 3, 64, 128), "right": torch.zeros(1, 3, 64, 128)})
    assert patch.patch(m) is m                                             # patching twice is a no-op


@needs_ref
@pytest.mark.parametrize("kw", [{"amp": True}, {"aggregation": True}])
def test_refusals(native, kw):
    from oracle.cfnet import reference_model
    _, patch = native
    with pytest.raises(NotImplementedError):
        patch.patch(reference_model(), **kw)


@needs_ref
def test_swapped_mish_refused_by_name(native):
    from oracle.cfnet import reference_model
    _, patch = native
    with pytest.raises(NotImplementedError, match=r"dres0\.1 is ReLU"):
        patch.patch(reference_model(replace_mish=True))


@needs_ref
def test_training_mode_model_patches(native):
    from oracle.cfnet import reference_model
    _, patch = native
    m = reference_model().train()
    patch.patch(m, strict=False)                                           # BN is folded at the first CUDA inference call
    assert m.training


def test_serves(native):
    from openstereo_b200.cfnet import CFNetEngine
    ok = lambda h, w, b=1: CFNetEngine.serves({"left": torch.zeros(b, 3, h, w), "right": torch.zeros(b, 3, h, w)})   # noqa: E731
    assert ok(256, 512) and ok(512, 960, 4) and ok(32, 32)
    assert not ok(256, 500) and not ok(250, 512) and not ok(544, 970)
    assert not CFNetEngine.serves({"left": torch.zeros(1, 3, 64, 64), "right": torch.zeros(1, 3, 64, 32)})


@needs_ref
def test_oracle_against_the_reference_formulas():
    from oracle.cfnet import mish64, softargmin_var64
    sub = shim.load("stereo.modeling.models.cfnet.submodule")
    x = torch.cat([torch.linspace(-40, 40, 4001), torch.tensor([-1e-6, 0.0, 1e-6, 19.999, 20.0, 20.001])]).double()
    assert torch.allclose(mish64(x), sub.FMish(x), rtol=1e-15, atol=1e-300)
    assert torch.allclose(mish64(x), sub.Mish()(x), rtol=1e-15, atol=1e-300)
    g = torch.Generator().manual_seed(3)
    cost = torch.randn(2, 12, 5, 7, generator=g, dtype=torch.float64) * 3
    p = F.softmax(cost, dim=1)
    mu, var = softargmin_var64(cost)
    want = sub.disparity_regression(p, 12)
    assert torch.allclose(mu, want, rtol=1e-13, atol=1e-12)
    assert torch.allclose(var, sub.disparity_variance(p, 12, want.unsqueeze(1)).squeeze(1), rtol=1e-12, atol=1e-12)
    samples = torch.sort(torch.randint(0, 60, (2, 12, 5, 7), generator=g).double(), dim=1).values
    mu, var = softargmin_var64(cost, samples)
    want = torch.sum(p * samples, dim=1, keepdim=True)
    assert torch.allclose(mu, want.squeeze(1), rtol=1e-13, atol=1e-12)
    assert torch.allclose(var, sub.disparity_variance_confidence(p, samples, want).squeeze(1), rtol=1e-12, atol=1e-12)


def test_integer_round_trip_bound():
    """The warped-volume kernel's coordinate round trip (v / ((W - 1) / 2) - 1, then (g + 1) * ((W - 1) / 2), IEEE fp32) returns
    every integer column within 2^-23 (W - 1) of itself, and every integer row within 2^-23 (H - 1) (the same function of the
    extent): the bounds the GPU test and DESIGN.md section 4.22 state."""
    for w in list(range(2, 1100)) + [1920, 3840]:
        half = torch.tensor((w - 1.0) / 2.0, dtype=torch.float32)
        v = torch.arange(-3, w + 3, dtype=torch.float32)
        ix = ((v / half) - 1 + 1) * half
        assert float((ix - v).abs().max()) <= 2.0 ** -23 * (w - 1), w
