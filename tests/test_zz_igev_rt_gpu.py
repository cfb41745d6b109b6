"""GPU: IGEV-RT -- the geometry-only lookup against the reference class on the CPU (value, zeros outside the row; its store bounds,
refusals and fp64 accuracy are rows of test_kernel_contract_gpu.py), the combined lookup left as it was, and the hourglass(8) +
classifier engine against the reference modules.  patch() on the
whole reference model is in test_zz_igev_rt_fullsize_gpu.py.  Both files sort after the torch.profiler routing suites
(test_*_contract_gpu.py), so in one pytest process they run after those suites, like the other model-level files.

Lookup bar.  Each output is v0*w0 + v1*w1 with the reference's interpolation weights replayed operation by operation, so the only
freedom is how the two products are rounded and added (aten's vectorised CPU kernel may fuse them): at most 1 ulp of
|v0|*w0 + |v1|*w1, which is the same lookup run on |volume|."""
import pytest
import torch

from oracle import _reference_shim as shim
from oracle import igev_rt as oigrt

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not shim.available(), reason="reference tree (oracle/_ref) not staged")


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, aggregation, geo, ops
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return _lib, ops, geo, aggregation


def rnd(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def _disp(seed, b, h, w, d, radius):
    """Disparities from below -r - 4 to past D + r + 4: taps leave the row at both ends on every level."""
    disp = torch.rand(b, 1, h, w, generator=torch.Generator().manual_seed(seed)) * (d + 2 * radius + 8) - radius - 4
    disp[0, 0, 0, :4] = torch.tensor([0.0, d - 1.0, -radius - 2.5, d + radius + 2.5])
    return disp


def _combined_inputs():
    g = torch.Generator().manual_seed(60)
    f1, f2 = torch.randn(2, 16, 3, 130, generator=g), torch.randn(2, 16, 3, 130, generator=g)
    vol = torch.randn(2, 8, 48, 3, 130, generator=g)
    disp = torch.rand(2, 1, 3, 130, generator=g) * 60 - 6
    coords = torch.arange(130).float().reshape(1, 1, 130, 1).repeat(2, 3, 1, 1)
    return [t.cuda() for t in (f1, f2, vol, disp, coords)]


def test_combined_lookup_unchanged_by_geometry_only_mode(osb):
    """The combined lookup gives the same bits before and after the geometry-only mode runs in the process (this file's first
    test, so nothing earlier in it has called the geometry-only entry point)."""
    _, ops, geo, _ = osb
    f1, f2, vol, disp, coords = _combined_inputs()

    def combined():
        return [geo.CombinedGeoEncodingVolume(f1, f2, vol, num_levels=2, radius=r)(disp, coords).cpu() for r in (4, 2)]
    before = combined()
    for r in (4, 2):
        geo.GeoEncodingVolume(rnd(61, 1, 8, 48, 3, 130).cuda(), radius=r)(torch.rand(1, 1, 3, 130, device="cuda") * 40)
    after = combined()
    for r, a, b in zip((4, 2), before, after):
        assert torch.equal(a, b), r


# (B, C, D, H, W, levels, radius): radius 4 and the generic path, levels 1-4, widths off 128, B > 1
CASES = [(1, 8, 48, 3, 130, 2, 4), (2, 8, 48, 2, 200, 4, 4), (2, 5, 40, 3, 129, 3, 2), (1, 6, 24, 2, 77, 1, 1),
         (3, 4, 36, 2, 140, 2, 3), (2, 8, 48, 4, 96, 1, 4)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "B%dC%dD%dH%dW%d-L%d-r%d" % c)
def test_geo_volume_lookup_matches_reference(osb, case):
    _, ops, geo, _ = osb
    b, c, d, h, w, levels, radius = case
    rgeo = oigrt.load_reference("stereo.modeling.models.igev_rt.geometry")
    vol, disp = rnd(40, b, c, d, h, w), _disp(41, b, h, w, d, radius)
    want = rgeo.Geo_Encoding_Volume(vol, num_levels=levels, radius=radius)(disp)
    scale = rgeo.Geo_Encoding_Volume(vol.abs(), num_levels=levels, radius=radius)(disp)        # |v0|*w0 + |v1|*w1 per tap
    got = geo.Geo_Encoding_Volume(vol.cuda(), num_levels=levels, radius=radius)(disp.cuda())
    assert got.shape == want.shape == (b, levels * c * (2 * radius + 1), h, w) and got.dtype == torch.float32
    got = got.cpu()
    err = (got - want).abs()
    ulp = torch.nextafter(scale, torch.full_like(scale, float("inf"))) - scale
    assert (err <= ulp).all(), "max err %g ulps" % (err / ulp.clamp(min=1e-45)).max().item()
    assert (got[scale == 0] == 0).all() and (scale == 0).any()                     # taps outside the row: exact zeros
    print("%s: %.4f of the outputs bit-equal" % (case, (err == 0).float().mean().item()))


# ------------------------------------------------------------------------------------------ hourglass(8) + classifier engine
def _features(seed, b, h4, w4):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(b, ch, h4 // s, w4 // s, generator=g) for ch, s in ((96, 1), (64, 2), (192, 4), (160, 8))]


@needs_ref
@pytest.mark.parametrize("h,w", [(256, 512), (544, 960)])
def test_hourglass8_and_classifier_against_reference(osb, h, w):
    lib, ops, _, aggregation = osb
    m = oigrt.igev_rt()
    hg, cls = m.cost_agg, m.classifier
    b, d4, h4, w4 = 1, 48, h // 4, w // 4
    x = rnd(70, b, 8, d4, h4, w4)
    feats = _features(71, b, h4, w4)
    with torch.no_grad():
        want = cls(hg(x, feats))
        hg.cuda(), cls.cuda()
        eng, head = aggregation.StereoBaseAggregation(hg), aggregation.StereoBaseCostHead(cls)
        xg, fg = x.cuda(), [f.cuda() for f in feats]
        eng(xg, fg), head.logits(eng(xg, fg))                                            # pack both engines
        assert not eng.tc_route_ok(xg.shape)                                            # 8 / 16 channels: CUDA-core route
        before = lib.launch_count()
        geo = eng(xg, fg)
        mid = lib.launch_count()
        got = head.logits(geo)
        end = lib.launch_count()
    # 6 convs of conv1..conv3, 5 FeatureAtt gates x 2 1x1 convs, 3 transposed convs, agg_0 and agg_1 x 3 convs
    assert mid - before == 6 + 10 + 3 + 6
    head_tc = ops.conv3d_tc_kc(32, 1, w4) == 32                                         # narrow tensor-core head: pad + conv
    assert end - mid == (2 if head_tc else 1)
    err = (got.cpu() - want).abs().max().item() / want.abs().max().item()
    print("hourglass(8) + classifier %dx%d: max err %.2e of the logit scale, head on %s" % (h, w, err, "tensor cores" if head_tc
                                                                                          else "CUDA cores"))
    assert got.shape == want.shape and err <= 1e-5
