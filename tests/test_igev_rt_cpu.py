"""CPU: IGEV-RT -- the geometry-only lookup oracle against its fixture and the live reference, the new C-ABI entry point, and
patch()'s drop-in contract on the unmodified reference class (no compute on a GPU here)."""
import pytest
import torch

from oracle import _reference_shim as shim
from oracle import igev_rt as oigrt

from conftest import load_golden

needs_ref = pytest.mark.skipif(not shim.available(), reason="reference tree not present")


def rnd(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def _inputs(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return {"left": torch.rand(b, 3, h, w, generator=g) * 2 - 1, "right": torch.rand(b, 3, h, w, generator=g) * 2 - 1}


# ------------------------------------------------------------------------------------------ oracle vs fixture / live reference
def test_oracle_geo_volume_lookup_golden():
    g = load_golden("geo_volume_lookup")
    assert g["cases"] == 4
    seen = set()
    for i in range(g["cases"]):
        vol, disp, levels, radius = g["volume%d" % i], g["disp%d" % i], g["levels%d" % i], g["radius%d" % i]
        out = oigrt.GeoEncodingVolume(vol, num_levels=levels, radius=radius)(disp)
        assert torch.equal(out, g["out%d" % i]), i
        seen.add((levels, radius))
        # taps leave the row at both ends of the top level: exact zeros there
        assert (disp < -radius - 1).any() and (disp > vol.shape[2] + radius).any()
    assert {l for l, _ in seen} == {1, 2, 3} and {r for _, r in seen} == {2, 4}


@needs_ref
@pytest.mark.parametrize("levels,radius", [(1, 4), (2, 4), (3, 1), (2, 3)])
def test_oracle_pins_reference_geo_volume(levels, radius):
    rgeo = oigrt.load_reference("stereo.modeling.models.igev_rt.geometry")
    vol = rnd(5, 2, 6, 20, 3, 11)
    disp = torch.rand(2, 1, 3, 11, generator=torch.Generator().manual_seed(6)) * 34 - 7
    want = rgeo.Geo_Encoding_Volume(vol, num_levels=levels, radius=radius)(disp)
    assert torch.equal(oigrt.GeoEncodingVolume(vol, num_levels=levels, radius=radius)(disp), want)


# ------------------------------------------------------------------------------------------ host side
def test_entry_point_bound_and_declared():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, geo
    assert "osb_geo_volume_lookup_fwd" in _lib.SIGNATURES
    with pytest.raises(ValueError, match="null pointer"):
        _lib.call("osb_geo_volume_lookup_fwd", None, None, None, None, None, None, 1, 8, 48, 4, 4, 2, 4, None)
    with pytest.raises(ValueError, match="num_levels"):
        _lib.call("osb_geo_volume_lookup_fwd", 0x1000, None, None, None, 0x1000, 0x1000, 1, 8, 48, 4, 4, 5, 4, None)
    with pytest.raises(ValueError, match="level 1 is null"):
        _lib.call("osb_geo_volume_lookup_fwd", 0x1000, None, None, None, 0x1000, 0x1000, 1, 8, 48, 4, 4, 2, 4, None)
    assert geo.Geo_Encoding_Volume is geo.GeoEncodingVolume
    with pytest.raises(RuntimeError, match="CUDA tensors required"):
        geo.GeoEncodingVolume(rnd(1, 1, 8, 12, 2, 4))


def test_engine_reads_igev_layers():
    """The aggregation engine packs IGEV's BasicConv (BN only when use_bn, LeakyReLU only when relu) and its FeatureAtt."""
    from openstereo_b200 import aggregation as agg
    from openstereo_b200.ops import ACT_LEAKY, ACT_NONE
    sub = oigrt.load_reference("stereo.modeling.models.igev_rt.submodule")
    a = sub.BasicConv(8, 16, is_3d=True, bn=False, relu=True, kernel_size=3, padding=1, stride=2).eval()
    assert a.bn is not None                                     # owned even with bn=False: use_bn decides
    layer, act = agg._block(a)
    assert layer.scale is None and layer.shift is None and act == ACT_LEAKY and layer.stride == 2
    b = sub.BasicConv(16, 8, deconv=True, is_3d=True, bn=True, relu=False, kernel_size=(4, 4, 4), padding=(1, 1, 1),
                      stride=(2, 2, 2)).eval()
    layer, act = agg._block(b)
    assert layer.transposed and layer.kernel == 4 and layer.scale is not None and act == ACT_NONE
    fa = agg._FeatureAtt(sub.FeatureAtt(16, 64).eval())
    assert fa.act == ACT_LEAKY and fa.a.scale is not None and fa.b.scale is None and fa.b.shift is not None
    assert tuple(fa.a.w.shape) == (64, 32) and tuple(fa.b.w.shape) == (32, 16)


@needs_ref
def test_hourglass8_refuses_tensor_core_route():
    """At c = 8 the plan would pad 8 and 16 channels to 32: the engine keeps IGEV-RT's hourglass on the CUDA-core kernels."""
    from openstereo_b200 import aggregation as agg
    eng = agg.StereoBaseAggregation(oigrt.igev_rt().cost_agg)
    eng._pack()
    for shape in ((1, 8, 48, 64, 128), (8, 8, 48, 136, 240)):
        assert not eng.tc_route_ok(shape)


# ------------------------------------------------------------------------------------------ patch() on the reference class
@needs_ref
def test_patch_keeps_state_dict_and_refuses_cpu():
    from openstereo_b200.patch import patch
    m = oigrt.igev_rt()
    keys = list(m.state_dict().keys())
    patch(m)
    assert list(m.state_dict().keys()) == keys
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA inference only"):
        m(_inputs(1, 64, 128, 3))


@needs_ref
def test_patch_non_strict_cpu_equals_reference():
    from openstereo_b200.patch import patch
    x = _inputs(1, 64, 128, 4)
    with torch.no_grad():
        want = oigrt.igev_rt()(dict(x))["disp_pred"]
        got = patch(oigrt.igev_rt(), strict=False)(dict(x))["disp_pred"]
    assert want.shape == (1, 1, 64, 128) and want.std() > 0.1
    assert torch.equal(got, want)
