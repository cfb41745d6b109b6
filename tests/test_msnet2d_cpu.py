"""CPU: MSNet2D's patch surface (routing, the per-instance override, state_dict, refusals), the oracle against the reference's own
forward, the fp64 gather of the interlaced crops against the reference's interleave, and the dense 3x3 weights the volume
network runs as (aggregation.msnet2d_volume_weights) against the reference's Conv3d chain, in fp64."""
import pytest
import torch
import torch.nn.functional as F

from oracle import _reference_shim as shim

needs_ref = pytest.mark.skipif(not shim.available(), reason="reference tree not staged")


@pytest.fixture(scope="module")
def native():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import aggregation, patch
    return aggregation, patch


def _images(b, h, w, seed=1):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(b, 3, h, w, generator=g), torch.randn(b, 3, h, w, generator=g)


@needs_ref
def test_patch_surface(native):
    from oracle.msnet2d import reference_model
    _, patch = native
    m, other = reference_model(), reference_model()
    keys = list(m.state_dict())
    assert type(m).__name__ == "MSNet2D" and type(m).__module__.split(".")[-2:] == ["msnet", "MSNet2D"]
    assert patch._MODULE_PATCHERS[("msnet", "MSNet2D", "MSNet2D")] is patch._patch_msnet2d
    patch.patch(m)
    assert list(m.state_dict()) == keys
    assert "forward" in vars(m) and "forward" not in vars(other), "the override is per instance"
    assert type(m).forward is type(other).forward
    with pytest.raises(RuntimeError, match="CUDA inference only"):          # CPU call, strict
        m({"left": torch.zeros(1, 3, 64, 256), "right": torch.zeros(1, 3, 64, 256)})
    assert patch.patch(m) is m


@needs_ref
def test_training_mode_refused(native):
    from oracle.msnet2d import reference_model
    _, patch = native
    m = patch.patch(reference_model().train())
    with pytest.raises(RuntimeError, match="CUDA inference only"):
        m({"left": torch.zeros(1, 3, 64, 256), "right": torch.zeros(1, 3, 64, 256)})


@needs_ref
def test_non_strict_cpu_call_runs_the_reference(native):
    from oracle.msnet2d import reference_model
    _, patch = native
    l, r = _images(1, 64, 256)
    want = reference_model()({"left": l, "right": r})["disp_pred"]
    m = patch.patch(reference_model(), strict=False)
    with torch.no_grad():
        assert torch.equal(m({"left": l, "right": r})["disp_pred"], want)


@needs_ref
@pytest.mark.parametrize("kw", [{"amp": True}, {"aggregation": True}])
def test_refusals(native, kw):
    from oracle.msnet2d import reference_model
    _, patch = native
    with pytest.raises(NotImplementedError):
        patch.patch(reference_model(), **kw)


@needs_ref
def test_foreign_volume_network_refused_by_name(native):
    from oracle.msnet2d import reference_model
    _, patch = native
    m = reference_model()
    m.conv3d[3] = torch.nn.Conv3d(16, 32, kernel_size=(4, 3, 3), stride=[2, 1, 1], padding=[0, 1, 1])
    with pytest.raises(NotImplementedError, match="MSNet2D.conv3d"):
        patch.patch(m)
    m = reference_model()
    m.dres0[0].conv[3].dilation = (2, 2)
    with pytest.raises(NotImplementedError, match="dres0.0"):
        patch.patch(m)


@needs_ref
def test_oracle_stages_equal_the_reference_forward():
    from oracle.msnet2d import reference_model, stages
    m = reference_model()
    l, r = _images(2, 64, 256, seed=5)
    with torch.no_grad():
        s = stages(m, l, r)
        want = m({"left": l, "right": r})["disp_pred"]
    assert torch.equal(s["disp"], want)
    assert s["volume"].shape == (2, 48, 16, 64) and float(s["volume"].std()) > 0.05
    tri = torch.ones(48, 64).triu() == 0                                 # (d, w): w < d
    assert torch.all(s["volume"].permute(0, 2, 1, 3)[:, :, tri] == 0)


@needs_ref
def test_interlaced_crops64_is_the_reference_interleave():
    from oracle.msnet2d import interlaced_crops64
    sub = shim.load("stereo.modeling.models.msnet.submodule")
    g = torch.Generator().manual_seed(2)
    fl, fr = torch.randn(2, 32, 3, 20, generator=g), torch.randn(2, 32, 3, 20, generator=g)
    depth = [8 * j + 2 * (t % 4) + t // 4 for j in range(8) for t in range(8)]     # block order -> reference depth
    for d, x in enumerate(interlaced_crops64(fl, fr, 20)):
        ref = sub.interweave_tensors(fl[..., d:], fr[..., :20 - d]) if d else sub.interweave_tensors(fl, fr)
        assert torch.equal(x.permute(0, 3, 1, 2), ref.double()[:, depth])


@needs_ref
@pytest.mark.parametrize("width", [1, 2, 7, 30])
def test_block_weights_equal_the_conv3d_chain(native, width):
    """The dense 3x3 weights over the library's channel orders, applied in fp64 to the block-interleaved crop, give the reference's
    Conv3d + BN + ReLU chain on the interleaved tensor: the permutation, the block diagonals and the folded BN are exact."""
    aggregation, _ = native
    from oracle.msnet2d import interlaced_crops64, reference_model
    sub = shim.load("stereo.modeling.models.msnet.submodule")
    m = reference_model(seed=4).double()
    g = torch.Generator().manual_seed(width)
    fl, fr = torch.randn(1, 32, 5, width, generator=g, dtype=torch.float64), torch.randn(1, 32, 5, width, generator=g, dtype=torch.float64)
    with torch.no_grad():
        want = m.conv3d(sub.interweave_tensors(fl, fr).unsqueeze(1)).squeeze(2)
        layers = aggregation.msnet2d_volume_weights(m.float().conv3d)
    x = interlaced_crops64(fl, fr, 1)[0].permute(0, 3, 1, 2)
    for w, scale, shift in layers:
        x = F.relu(F.conv2d(x, w.double(), padding=1) * scale.double().view(1, -1, 1, 1) + shift.double().view(1, -1, 1, 1))
    assert x.shape == want.shape
    assert torch.allclose(x, want, rtol=1e-6, atol=1e-6)                  # BN folded in fp32, applied in fp64
