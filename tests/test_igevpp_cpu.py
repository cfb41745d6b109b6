"""CPU: IGEV++ -- the multi-range lookup oracle against its fixture and the live reference, the new C-ABI entry point's argument
checks, the weight packing of the new update-block engines (zero pad rows and columns), their serves() over widths and
hyper-parameters, and patch()'s drop-in contract on the unmodified reference class (no compute on a GPU here)."""
import pytest
import torch

from oracle import _reference_shim as shim
from oracle import igevpp as oigpp

from conftest import load_golden

needs_ref = pytest.mark.skipif(not shim.available(), reason="reference tree not present")


def rnd(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def _inputs(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return {"left": torch.rand(b, 3, h, w, generator=g) * 2 - 1, "right": torch.rand(b, 3, h, w, generator=g) * 2 - 1}


@pytest.fixture(scope="module")
def native():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib
    return _lib


# ------------------------------------------------------------------------------------------ oracle vs fixture / live reference
def test_oracle_multirange_lookup_golden():
    g = load_golden("igevpp_lookup")
    assert g["cases"] == 4
    seen, independent = set(), False
    for i in range(g["cases"]):
        levels, radius = g["levels%d" % i], g["radius%d" % i]
        v0, v1, v2, disp = g["vol0_%d" % i], g["vol1_%d" % i], g["vol2_%d" % i], g["disp%d" % i]
        b, _, d0, h, w = v0.shape
        coords = torch.arange(w).float().reshape(1, 1, w, 1).repeat(b, h, 1, 1)
        outs = oigpp.MultiRangeGeoEncodingVolume(v0, v1, v2, g["fmap1_%d" % i], g["fmap2_%d" % i], radius=radius,
                                                 num_levels=levels)(disp, coords)
        for name, out in zip(("feat0", "feat1", "feat2", "corr"), outs):
            assert torch.equal(out, g["%s%d" % (name, i)]), (i, name)
        seen.add((levels, radius))
        # taps leave the rows at both ends: below 0 and past 4 * D2 (geo_feat2 samples at disp / 4)
        assert (disp < -radius - 1).any() and (disp > 4 * v2.shape[2] + radius).any()
        independent |= v1.shape[2] != d0 >> 1 or v2.shape[2] != d0 >> 2
    assert {(2, 4), (2, 2), (1, 4)} <= seen and independent


@needs_ref
@pytest.mark.parametrize("levels,radius,d1,d2", [(1, 4, 13, 30), (2, 4, 48, 48), (2, 1, 9, 5), (2, 3, 24, 12)])
def test_oracle_pins_reference_multirange(levels, radius, d1, d2):
    rgeo = oigpp.load_reference("stereo.modeling.models.igevpp.geometry")
    v0, v1, v2 = rnd(5, 2, 6, 20, 3, 11), rnd(6, 2, 6, d1, 3, 11), rnd(7, 2, 6, d2, 3, 11)
    f1, f2 = rnd(8, 2, 4, 3, 11), rnd(9, 2, 4, 3, 11)
    disp = torch.rand(2, 1, 3, 11, generator=torch.Generator().manual_seed(10)) * 140 - 7
    coords = torch.arange(11).float().reshape(1, 1, 11, 1).repeat(2, 3, 1, 1)
    want = rgeo.Combined_Geo_Encoding_Volume(v0, v1, v2, f1, f2, radius=radius, num_levels=levels)(disp, coords)
    got = oigpp.MultiRangeGeoEncodingVolume(v0, v1, v2, f1, f2, radius=radius, num_levels=levels)(disp, coords)
    assert all(torch.equal(a, b) for a, b in zip(got, want))


# ------------------------------------------------------------------------------------------ host side
_P = 0x1000


def _args(**kw):
    """Arguments of osb_geo_multirange_lookup_fwd, every pointer a fake address; kw overrides by name."""
    names = ["geo0", "geo1", "geo2", "geo3", "vol1", "vol2", "corr0", "corr1", "corr2", "corr3", "disp", "coords", "out0", "out1",
             "out2", "out_corr", "B", "C", "D0", "D1", "D2", "H", "W", "W2", "levels", "radius", "stream"]
    vals = dict(geo0=_P, geo1=_P, geo2=None, geo3=None, vol1=_P, vol2=_P, corr0=_P, corr1=_P, corr2=None, corr3=None, disp=_P,
                coords=_P, out0=_P, out1=_P, out2=_P, out_corr=_P, B=1, C=8, D0=48, D1=48, D2=48, H=4, W=4, W2=4, levels=2, radius=4,
                stream=None)
    vals.update(kw)
    return [vals[n] for n in names]


@pytest.mark.parametrize("kw,match", [
    (dict(out_corr=None), "null pointer"), (dict(vol2=None), "null pointer"), (dict(coords=None), "null pointer"),
    (dict(geo1=None), "level 1 is null"), (dict(corr1=None), "level 1 is null"), (dict(levels=0), "num_levels"),
    (dict(levels=5), "num_levels"), (dict(radius=17), "radius"), (dict(radius=-1), "radius"), (dict(D0=3), "shorter than 2"),
    (dict(D2=1), "shorter than 2"), (dict(W2=3), "shorter than 2"), (dict(C=0), "empty shape"), (dict(D1=0), "empty shape"),
    (dict(B=2000), "grid dimension")])
def test_entry_point_argument_checks(native, kw, match):
    """Every refusal is an argument error raised before any CUDA call (the fake addresses are never touched)."""
    assert native.SIGNATURES["osb_geo_multirange_lookup_fwd"] == [native._f32p] * 16 + [native._i] * 10 + [native._s]
    with pytest.raises(ValueError, match=match):
        native.call("osb_geo_multirange_lookup_fwd", *_args(**kw))


def test_host_refuses_cpu_tensors(native):
    from openstereo_b200 import geo, ops
    v = rnd(1, 1, 8, 12, 2, 16)
    f = rnd(2, 1, 4, 2, 16)
    with pytest.raises(RuntimeError, match="CUDA tensors required"):
        geo.MultiRangeGeoEncodingVolume(v, v, v, f, f)
    with pytest.raises(RuntimeError, match="not implemented on the CPU"):
        ops.geo_multirange_lookup([v], v, v, [rnd(3, 1, 2, 16, 16)], rnd(4, 1, 1, 2, 16), torch.zeros(1, 2, 16), 4)


def _update_mods(seed):
    from types import SimpleNamespace
    torch.manual_seed(seed)
    m = shim.load("stereo.modeling.models.igevpp.update")
    args = SimpleNamespace(CORR_RADIUS=4)
    return m.GeoEncoder(144).eval(), m.GeoEncoder(72).eval(), m.BasicDispEncoder(args).eval()


@needs_ref
def test_weight_packing_pads_with_zeros(native):
    """convg2 / convc2 (96 rows) and conv (127 rows) are padded to 128 output channels with zero weights and zero biases; conv's cor
    half has zero columns for cor's 32 pad channels.  The packed TcWeight keeps the real rows to the hi + lo split's accuracy."""
    from openstereo_b200 import update
    g0, _, enc = _update_mods(1)
    ge, de = update.GeoEncoderEngine(g0), update.DispEncoderEngine(enc)
    ge._pack()
    de._pack()

    def unpack(tw):                                     # (3, cin/16, 3, 3*cout, 32) swizzled fp16 -> (cout, cin, 3, 3) of kd = 1
        kc, cout = tw.kc, tw.cout
        d = tw.data.float().view(3, -1, 3, 3 * cout, 2 * kc // 8, 8)
        rows = torch.arange(3 * cout)
        key = (rows & 7) if kc == 32 else ((rows >> 1) & 3)
        src = torch.arange(2 * kc // 8).view(1, -1) ^ key.view(-1, 1)
        inv = torch.empty_like(src)
        inv.scatter_(1, src, torch.arange(2 * kc // 8).expand_as(src).contiguous())
        d = torch.gather(d, 4, inv.view(1, 1, 1, 3 * cout, -1, 1).expand_as(d).contiguous()).reshape(3, -1, 3, 3 * cout, 2, kc)
        w = (d[..., 0, :] + d[..., 1, :])[1]            # (chunk, kh, 3*cout, kc) at kd = 1
        w = w.view(w.shape[0], 3, 3, cout, kc).permute(3, 0, 4, 1, 2).reshape(cout, -1, 3, 3)
        return w * (tw.inv.view(-1, 1, 1, 1) * 16)

    assert ge.g2.cout == 128 and ge.bg2.shape == (128,) and torch.equal(ge.bg2[96:], torch.zeros(32))
    w = unpack(ge.g2)
    assert torch.equal(w[96:], torch.zeros_like(w[96:]))
    assert torch.allclose(w[:96], g0.convg2.weight.float(), rtol=0, atol=1e-7)
    assert tuple(ge.g1.shape) == (144, 128) and torch.equal(ge.g1, g0.convg1.weight[:, :, 0, 0].t())
    c2 = unpack(de.c2)
    assert torch.equal(c2[96:], torch.zeros_like(c2[96:])) and torch.equal(de.bc2[96:], torch.zeros(32))
    wc, wd = unpack(de.wc), unpack(de.wd)
    assert wc.shape == (128, 128, 3, 3) and wd.shape == (128, 32, 3, 3)
    assert torch.equal(wc[:, 96:], torch.zeros_like(wc[:, 96:])) and torch.equal(wc[127], torch.zeros_like(wc[127]))
    assert torch.equal(wd[127], torch.zeros_like(wd[127])) and de.b[127] == 0
    assert torch.allclose(wc[:127, :96], enc.conv.weight[:, :96], rtol=0, atol=1e-7)
    assert torch.allclose(wd[:127], enc.conv.weight[:, 96:], rtol=0, atol=1e-7)
    assert tuple(de.c1.shape) == (114, 128) and tuple(de.d1.shape) == (32, 7, 7)


@needs_ref
def test_engines_serve_widths_and_hyper_parameters(native):
    """W' >= OSB_TC_MIN_WIDTH with the reference's hyper-parameters; any other width or layer shape runs the module's own forward."""
    from openstereo_b200 import update
    g0, g1, enc = _update_mods(2)
    ge0, ge1, de = update.GeoEncoderEngine(g0), update.GeoEncoderEngine(g1), update.DispEncoderEngine(enc)
    mask64 = torch.nn.Sequential(torch.nn.Conv2d(128, 64, 3, padding=1), torch.nn.ReLU(inplace=True))
    mask48 = torch.nn.Sequential(torch.nn.Conv2d(128, 48, 3, padding=1), torch.nn.ReLU(inplace=True))
    mf64, mf48 = update.MaskFeatEngine(mask64), update.MaskFeatEngine(mask48)
    for w in (16, 20, 23, 24, 32, 60, 64, 128, 160, 240):
        ok = w >= 24
        x = torch.zeros(1, 128, 2, w)
        assert ge0.serves(torch.zeros(1, 144, 2, w)) == ok and ge1.serves(torch.zeros(1, 72, 2, w)) == ok
        assert de.serves(torch.zeros(1, 1, 2, w), torch.zeros(1, 114, 2, w)) == ok
        assert mf64.serves(x) == ok and not mf48.serves(x)
    x = torch.zeros(1, 144, 2, 128)
    assert not ge0.serves(torch.zeros(1, 72, 2, 128)) and not ge1.serves(x)          # geo_planes must match convg1
    assert not de.serves(torch.zeros(1, 1, 2, 128), torch.zeros(1, 96, 2, 128))     # another CORR_RADIUS
    assert not de.serves(torch.zeros(2, 1, 2, 128), torch.zeros(1, 114, 2, 128))
    assert not ge0.serves(torch.zeros(144, 2, 128))


# ------------------------------------------------------------------------------------------ patch() on the reference class
@needs_ref
def test_patch_keeps_state_dict_overrides_per_instance_and_refuses_cpu():
    from openstereo_b200.patch import patch
    m, other = oigpp.igevpp(), oigpp.igevpp()
    keys = list(m.state_dict().keys())
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    patch(m)
    assert m._osb_patched and list(m.state_dict().keys()) == keys
    assert all(torch.equal(v, sd[k]) for k, v in m.state_dict().items())
    ub = m.update_block
    for name in ("gru04", "gru08", "gru16", "encoder", "geo_encoder0", "geo_encoder1", "geo_encoder2", "disp_head", "mask_feat_4"):
        assert "forward" in vars(getattr(ub, name)), name                   # per-instance override
        assert "forward" not in vars(getattr(other.update_block, name)), name
    assert "forward" in vars(m.classifier) and "forward" not in vars(m.cost_agg0) and "forward" not in vars(ub)
    for name in ("forward", "upsample_disp"):
        assert name in vars(m) and name not in vars(other)                  # the rebound methods, this instance only
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA inference only"):
        m(_inputs(1, 64, 128, 3))


@needs_ref
def test_patch_non_strict_cpu_equals_reference():
    from openstereo_b200.patch import patch
    x = _inputs(1, 64, 128, 4)
    with torch.no_grad():
        ref = oigpp.igevpp()
        ref.args.VALID_ITERS = 4
        want = ref(dict(x))["disp_pred"]
        pm = patch(oigpp.igevpp(), strict=False)
        pm.args.VALID_ITERS = 4
        got = pm(dict(x))["disp_pred"]
    assert want.shape == (1, 1, 64, 128) and want.std() > 0.1
    assert torch.equal(got, want)
