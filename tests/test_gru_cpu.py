"""CPU: the ConvGRU drop-in of IGEV-Stereo / StereoBase -- weight packing into the h / x column blocks, the route predicate, the new
C-ABI entry points' argument checks, and patch()'s contract on the unmodified reference classes (no compute on a GPU here)."""
import pytest
import torch

from oracle import _reference_shim as shim
from oracle import seeded_init as si

needs_ref = pytest.mark.skipif(not shim.available(), reason="reference tree not present")


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, gru, ops
    return _lib, gru, ops


def _unpack(tw):
    """TcWeight (16-channel chunks) -> the (Cout, Cin, 3, 3, 3) fp32 weight it holds: undo the swizzle, the layout and the scale."""
    k, nch, _, rows, two_kc = tw.data.shape
    kc = two_kc // 2
    cout = rows // 3
    cpr = two_kc // 8
    key = (torch.arange(rows) >> 1) & 3
    src = torch.arange(cpr).view(1, cpr) ^ key.view(-1, 1)                # the swizzle is an involution
    d = tw.data.view(k, nch, k, rows, cpr, 8)
    d = torch.gather(d, 4, src.view(1, 1, 1, rows, cpr, 1).expand(k, nch, k, rows, cpr, 8).contiguous())
    d = d.reshape(k, nch, k, 3, cout, 2, kc).float()                        # (kd, chunk, kh, kw, co, half, ci)
    w = (d[:, :, :, :, :, 0] + d[:, :, :, :, :, 1]).permute(4, 1, 5, 0, 2, 3).reshape(cout, nch * kc, k, k, 3)
    return w * (tw.inv * 16).view(-1, 1, 1, 1, 1)


def test_pack_round_trip(osb):
    _, gru, _ = osb
    torch.manual_seed(0)
    conv = torch.nn.Conv2d(128 + 256, 128, 3, padding=1)
    with torch.no_grad():
        conv.weight.mul_(torch.logspace(-3, 1, 128).view(-1, 1, 1, 1))   # per-channel scales across four decades
    wh, wx, bias = gru.pack_gru_conv(conv, 128)
    assert wh.data.shape == (3, 128 // 16, 3, 3 * 128, 32) and wx.data.shape == (3, 256 // 16, 3, 3 * 128, 32)
    assert torch.equal(bias, conv.bias.detach())
    for tw, block in ((wh, conv.weight[:, :128]), (wx, conv.weight[:, 128:])):
        w = _unpack(tw)
        assert torch.count_nonzero(w[:, :, 0]) == 0 and torch.count_nonzero(w[:, :, 2]) == 0   # one plane: taps at kd = 1
        ref = block.detach().double()
        err = (w[:, :, 1].double() - ref).abs()
        # f16_split: 2^-22 relative, 2^-25 absolute in the scaled units where the channel's max |w| lies in [2^14, 2^15)
        amax = ref.abs().amax(dim=(1, 2, 3), keepdim=True)
        assert (err <= ref.abs() * 2 ** -21 + amax * 2 ** -38).all()


@pytest.mark.parametrize("hidden,cin,w,ok", [
    (128, 384, 128, True), (128, 384, 160, True), (128, 384, 64, True), (128, 256, 32, True), (128, 384, 240, True),
    (128, 384, 24, True), (128, 384, 23, False), (128, 384, 16, False), (128, 384, 8, False),
    (96, 288, 128, False), (64, 192, 128, False), (128, 136, 128, False), (128, 128, 128, False)])
def test_route_predicate(osb, hidden, cin, w, ok):
    """Hidden 128 at every width of at least OSB_TC_MIN_WIDTH takes the wgmma kernels; everything else the reference's forward."""
    _, gru, _ = osb
    assert gru.route_ok(hidden, cin, w) is ok


def test_entry_points_declared_and_refuse_bad_arguments(osb):
    lib, _, _ = osb
    for name in ("osb_conv2d_k3_tc_gru_fwd", "osb_ncdhw_to_ndhwc_slice"):
        assert name in lib.SIGNATURES and hasattr(lib.lib, name)
    p, before = 0x1000, lib.launch_count()
    gru = lambda **kw: lib.call("osb_conv2d_k3_tc_gru_fwd", *[kw.get(k, d) for k, d in (
        ("x", p), ("w", p), ("scale", p), ("shift", None), ("res", p), ("mul", None), ("bz", None), ("bh", None), ("y", p),
        ("B", 2), ("Cin", 256), ("Cout", 128), ("H", 8), ("W", 128), ("act", 4), ("out", 1), ("rn", 0), ("rbs", 0), ("s", None))])
    with pytest.raises(ValueError, match="null pointer"):
        gru(x=None)
    with pytest.raises(ValueError, match="no Cout = 128 kernel"):
        gru(Cout=64)
    with pytest.raises(ValueError, match="no Cout = 128 kernel"):
        gru(W=16)
    with pytest.raises(ValueError, match="unknown activation 3"):
        gru(act=3)
    with pytest.raises(ValueError, match="16-byte aligned"):
        gru(mul=0x1004)
    with pytest.raises(ValueError, match="blend needs both"):
        gru(bz=p)
    with pytest.raises(ValueError, match="residual batch stride"):
        gru(rbs=128 * 8 * 128 - 4)
    with pytest.raises(ValueError, match="residual batch stride"):
        gru(rbs=384 * 8 * 128, rn=1)
    with pytest.raises(ValueError, match="residual batch stride"):
        gru(rbs=384 * 8 * 128, res=None)
    with pytest.raises(ValueError, match="null pointer"):
        lib.call("osb_ncdhw_to_ndhwc_slice", None, p, 1, 128, 1, 8, 64, 256, 0, None)
    with pytest.raises(ValueError, match="do not fit"):
        lib.call("osb_ncdhw_to_ndhwc_slice", p, p, 1, 128, 1, 8, 64, 256, 129, None)
    with pytest.raises(ValueError, match="do not fit"):
        lib.call("osb_ncdhw_to_ndhwc_slice", p, p, 1, 128, 1, 8, 64, 256, -1, None)
    assert lib.launch_count() == before


def _igev():
    shim.install_timm_stub()
    cfg = shim.load_cfg("cfgs/igev/igev_sceneflow_amp.yaml").MODEL
    m = shim.load("stereo.modeling.models.igev.igev_stereo").IGEVStereo(cfg).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=12, scale={"classifier.weight": 8.0}))
    return m


def _stereobase():
    shim.install_timm_stub()
    cfg = shim.load_cfg("cfgs/stereobase/stereobase_sceneflow.yaml").MODEL
    m = shim.load("stereo.modeling.models.stereobase.stereobase_gru").StereoBase(cfg).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=3, scale={"classifier.weight": 8.0}))
    return m


@needs_ref
@pytest.mark.parametrize("build", [_igev, _stereobase])
def test_patch_overrides_per_instance_and_refuses_cpu(osb, build):
    from openstereo_b200.patch import patch
    a, b = build(), build()
    keys = {k: v.clone() for k, v in a.state_dict().items()}
    patch(a)
    assert {k: v for k, v in a.state_dict().items()}.keys() == keys.keys()
    assert all(torch.equal(v, keys[k]) for k, v in a.state_dict().items())
    for name in ("gru04", "gru08", "gru16"):
        assert "forward" in vars(getattr(a.update_block, name))             # an instance attribute: the class is untouched
        assert "forward" not in vars(getattr(b.update_block, name))
    g = a.update_block.gru16
    h, c = torch.zeros(1, 128, 4, 32), torch.zeros(1, 384, 4, 32)
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA inference only"):
        g(h, *c.split(128, 1), torch.zeros(1, 128, 4, 32))


@needs_ref
def test_patch_non_strict_cpu_equals_reference(osb):
    """strict=False: every CPU call runs the reference's own code, bit for bit (StereoBase, 32 GRU iterations at 64x128)."""
    from openstereo_b200.patch import patch
    g = torch.Generator().manual_seed(5)
    x = {"left": torch.randn(1, 3, 64, 128, generator=g), "right": torch.randn(1, 3, 64, 128, generator=g)}
    with torch.no_grad():
        want = _stereobase()(dict(x))["disp_pred"]
        got = patch(_stereobase(), strict=False)(dict(x))["disp_pred"]
    assert torch.isfinite(want).all() and torch.equal(got, want)
