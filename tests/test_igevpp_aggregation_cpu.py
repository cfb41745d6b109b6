"""CPU: IGEV++'s instance-normalised hourglasses -- the engine's packing of IGEV++'s BasicConv (no BatchNorm, IN and ReLU flags),
its refusals (affine or tracked instance norms, another LeakyReLU slope, flags the graph does not run, shapes it cannot
concatenate), the argument checks of the three instance-norm entry points, and patch(model, aggregation=True)'s surface and
non-strict delegation on the unmodified reference class (no compute on a GPU here)."""
import pytest
import torch

from oracle import _reference_shim as shim
from oracle import igevpp as oigpp

needs_ref = pytest.mark.skipif(not shim.available(), reason="reference tree not present")


@pytest.fixture(scope="module")
def native():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib
    return _lib


def _hourglass(seed=1):
    torch.manual_seed(seed)
    return oigpp.load_reference("stereo.modeling.models.igevpp.igevpp_stereo").hourglass(8).eval()


def _hg_inputs(b, d, h, w, seed=2):
    g = torch.Generator().manual_seed(seed)
    ext = [(h, w)]
    for _ in range(3):
        ext.append(tuple((e - 1) // 2 + 1 for e in ext[-1]))
    return torch.randn(b, 8, d, h, w, generator=g), [torch.randn(b, c, *e, generator=g) for c, e in zip((96, 64, 192, 160), ext)]


# ------------------------------------------------------------------------------------------ entry points
_P = 0x1000


def _k3(**kw):
    a = dict(x=_P, w=_P, scale=None, shift=None, in_stats=None, in_gate=None, y=_P, stats=None, ws=None, ws_floats=0, B=1, Cin=8,
             Cout=8, D=4, H=4, W=8, stride=1, act=0, s=None)
    a.update(kw)
    return list(a.values())


def _pw(**kw):
    a = dict(x0=_P, x1=None, Cin0=8, w=_P, scale=None, shift=None, s0=None, g0=None, s1=None, g1=None, y=_P, stats=None, ws=None,
             ws_floats=0, B=1, Cin=8, Cout=8, D=4, H=4, W=8, act=0, sigmoid=0, s=None)
    a.update(kw)
    return list(a.values())


@pytest.mark.parametrize("name,args,match", [
    ("osb_conv3d_k3_in_fwd", _k3(x=None), "null pointer"),
    ("osb_conv3d_k3_in_fwd", _k3(stats=_P), "null pointer"),
    ("osb_conv3d_k3_in_fwd", _k3(D=0), "empty shape"),
    ("osb_conv3d_k3_in_fwd", _k3(stride=3), "stride"),
    ("osb_conv3d_k3_in_fwd", _k3(in_gate=_P), "statistics"),
    ("osb_conv3d_k3_in_fwd", _k3(stats=_P, ws=_P, act=2), "raw output"),
    ("osb_conv3d_k3_in_fwd", _k3(stats=_P, ws=_P, shift=_P), "raw output"),
    ("osb_conv3d_k3_in_fwd", _k3(in_stats=_P + 4), "aligned"),
    ("osb_conv3d_k3_in_fwd", _k3(D=512, H=256, W=256), "exact fp32 count"),
    ("osb_deconv3d_in_fwd", _k3(stride=2), "kernel 2"),
    ("osb_deconv3d_in_fwd", _k3(W=-1, stride=4), "empty shape"),
    ("osb_conv3d_1x1_in_fwd", _pw(x0=None), "null pointer"),
    ("osb_conv3d_1x1_in_fwd", _pw(Cin=16), "channel split"),
    ("osb_conv3d_1x1_in_fwd", _pw(s1=_P), "second slab"),
    ("osb_conv3d_1x1_in_fwd", _pw(stats=_P, ws=_P, sigmoid=1), "raw output"),
])
def test_entry_point_argument_checks(native, name, args, match):
    """Refused with OSB_EINVAL before any CUDA call (nothing here has a device)."""
    with pytest.raises(ValueError, match=match):
        native.call(name, *args)


def test_workspace_query(native):
    """3 floats per (b, channel, CTA) + one counter per (b, channel block), from the instantiation's tiles; -1 for bad arguments."""
    q = native.lib.osb_conv3d_in_workspace_floats
    # k3 stride 1, Cout 8 -> 32-channel groups, tiles 4 x 4 x 32: 48 x 64 x 128 -> 12 * 16 * 4 CTAs
    assert q(0, 2, 8, 48, 64, 128, 1) == 3 * 2 * 8 * 768 + 2
    # stride 2 tile 2 x 4 x 32 on the 24 x 32 x 64 output
    assert q(0, 1, 16, 48, 64, 128, 2) == 3 * 16 * (12 * 8 * 2) + 1
    # transposed k4: output 2x, tile 4 x 4 x 64, 16-channel groups
    assert q(1, 1, 32, 6, 8, 16, 4) == 3 * 32 * (3 * 4 * 1) + 2
    # 1x1: 64 octets of 8 columns per CTA, 32-channel groups
    assert q(2, 1, 48, 1, 64, 128, 0) == 3 * 48 * 16 + 2
    assert q(3, 1, 8, 4, 4, 8, 1) == -1 and q(0, 1, 8, 4, 4, 8, 3) == -1 and q(1, 1, 8, 4, 4, 8, 2) == -1 and q(2, 0, 8, 4, 4, 8, 0) == -1


# ------------------------------------------------------------------------------------------ the engine
@needs_ref
def test_engine_packs_basic_conv_without_batchnorm(native):
    from openstereo_b200.aggregation import IGEVPPAggregation, _in_refusal
    hg = _hourglass()
    eng = IGEVPPAggregation(hg)
    assert eng._why is None
    for name, blk in eng._blocks():
        assert not hasattr(blk, "bn") and isinstance(blk.IN, torch.nn.InstanceNorm3d)
        last = name == "conv1_up"
        assert _in_refusal(blk, not last, not last) is None and _in_refusal(blk, last, last) is not None, name
    eng._pack()
    assert len(eng.l) == 16 and all(p.scale is None and p.shift is None for p in eng.l.values())
    assert tuple(eng.l["conv0"].w.shape) == (8, 27, 8) and tuple(eng.l["conv3.0"].w.shape) == (32, 27, 64)
    assert tuple(eng.l["conv3_up"].w.shape) == (64, 64, 32) and eng.l["conv3_up"].transposed and eng.l["conv3_up"].kernel == 4
    assert tuple(eng.l["agg_0.0"].w.shape) == (64, 32) and tuple(eng.l["agg_1.0"].w.shape) == (32, 16)
    want = hg.conv1[0].conv.weight.permute(1, 2, 3, 4, 0).reshape(8, 27, 16)
    assert torch.equal(eng.l["conv1.0"].w, want)
    for g, (cf, cv) in zip(("4", "8", "16", "32", "up_16", "up_8"), ((96, 8), (64, 16), (192, 32), (160, 64), (192, 32), (64, 16))):
        a = eng.att[g]
        fa = getattr(hg, "feature_att_" + g).feat_att
        assert tuple(a.a.w.shape) == (cf, cf // 2) and a.a.shift is None
        assert tuple(a.b.w.shape) == (cf // 2, cv) and torch.equal(a.b.shift, fa[1].bias)
    x, f = _hg_inputs(1, 48, 64, 128)
    assert eng.serves(x, f)
    x, f = _hg_inputs(2, 47, 31, 63)
    assert eng.serves(x, f)
    assert not eng.serves(x[:, :, :, :30], f) and not eng.serves(x, f[:3]) and not eng.serves(x[:, :4], f)


@needs_ref
@pytest.mark.parametrize("change", ["affine", "tracked", "eps", "slope", "flags", "gate_affine", "dilation"])
def test_engine_refuses(native, change):
    from openstereo_b200.aggregation import IGEVPPAggregation
    hg = _hourglass()
    if change == "affine":
        hg.conv2[1].IN = torch.nn.InstanceNorm3d(32, affine=True)
    elif change == "tracked":
        hg.agg_1[2].IN = torch.nn.InstanceNorm3d(16, track_running_stats=True).eval()
    elif change == "eps":
        hg.conv0.IN = torch.nn.InstanceNorm3d(8, eps=1e-3)
    elif change == "slope":
        hg.conv3_up.act = torch.nn.LeakyReLU(0.1)
    elif change == "flags":
        hg.conv2_up.relu = False
    elif change == "gate_affine":
        hg.feature_att_up_8.feat_att[0].IN = torch.nn.InstanceNorm2d(32, affine=True)
    else:
        hg.conv3[1].conv.dilation = (2, 2, 2)
    eng = IGEVPPAggregation(hg)
    assert eng._why is not None
    x, f = _hg_inputs(1, 16, 16, 32)
    assert not eng.serves(x, f)
    with pytest.raises(NotImplementedError):
        eng(x, f)


# ------------------------------------------------------------------------------------------ patch()
def _inputs(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return {"left": torch.rand(b, 3, h, w, generator=g) * 2 - 1, "right": torch.rand(b, 3, h, w, generator=g) * 2 - 1}


def _surface(m):
    names = {n for n in ("forward", "upsample_disp") if n in vars(m)}
    for name, mod in m.named_modules():
        if "forward" in vars(mod):
            names.add(name + ".forward")
    return names


@needs_ref
def test_patch_aggregation_surface():
    """patch(m, aggregation=True) changes what patch(m) changes plus cost_agg0/1/2.forward; patch(m) leaves the hourglasses alone;
    the parameters and the state_dict are untouched."""
    from openstereo_b200.patch import patch
    plain, agg = patch(oigpp.igevpp()), oigpp.igevpp()
    sd = {k: v.clone() for k, v in agg.state_dict().items()}
    patch(agg, aggregation=True)
    assert _surface(agg) == _surface(plain) | {"cost_agg0.forward", "cost_agg1.forward", "cost_agg2.forward"}
    assert not {"cost_agg0.forward", "cost_agg1.forward", "cost_agg2.forward"} & _surface(plain)
    assert all(torch.equal(v, sd[k]) for k, v in agg.state_dict().items()) and list(agg.state_dict()) == list(sd)
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA inference only"):
        x, f = _hg_inputs(1, 16, 16, 32)
        agg.cost_agg0(x, f)


@needs_ref
def test_patch_aggregation_refused_on_other_models():
    from oracle import igev_rt as ort
    from openstereo_b200.patch import patch
    m = ort.igev_rt()
    with pytest.raises(NotImplementedError, match="IGEVRTtereo"):
        patch(m, aggregation=True)
    assert not getattr(m, "_osb_patched", False) and not any("forward" in vars(mod) for mod in m.modules())


@needs_ref
def test_patch_aggregation_non_strict_cpu_equals_reference():
    from openstereo_b200.patch import patch
    x = _inputs(1, 64, 128, 4)
    with torch.no_grad():
        ref = oigpp.igevpp()
        ref.args.VALID_ITERS = 4
        want = ref(dict(x))["disp_pred"]
        pm = patch(oigpp.igevpp(), strict=False, aggregation=True)
        pm.args.VALID_ITERS = 4
        got = pm(dict(x))["disp_pred"]
    assert want.shape == (1, 1, 64, 128) and want.std() > 0.1
    assert torch.equal(got, want)
