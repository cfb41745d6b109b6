"""CPU: the motion encoder / disp head / mask_feat_4 drop-in of IGEV-Stereo and StereoBase (update.py) -- weight packing, the route
predicate and the engines' shape / hyper-parameter checks, and patch()'s contract on the unmodified reference classes (no compute on
a GPU here)."""
import pytest
import torch

from oracle import _reference_shim as shim
from oracle import seeded_init as si

needs_ref = pytest.mark.skipif(not shim.available(), reason="reference tree not present")


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, ops, update
    return _lib, ops, update


def _unpack(tw):
    """TcWeight (16-channel chunks) -> the (Cout, Cin, 3, 3) fp32 2D weight it holds at kd = 1."""
    k, nch, _, rows, two_kc = tw.data.shape
    kc = two_kc // 2
    cout = rows // 3
    cpr = two_kc // 8
    key = (torch.arange(rows) >> 1) & 3
    src = torch.arange(cpr).view(1, cpr) ^ key.view(-1, 1)
    d = tw.data.view(k, nch, k, rows, cpr, 8)
    d = torch.gather(d, 4, src.view(1, 1, 1, rows, cpr, 1).expand(k, nch, k, rows, cpr, 8).contiguous())
    d = d.reshape(k, nch, k, 3, cout, 2, kc).float()
    w = (d[:, :, :, :, :, 0] + d[:, :, :, :, :, 1]).permute(4, 1, 5, 0, 2, 3).reshape(cout, nch * kc, k, k, 3)
    assert torch.count_nonzero(w[:, :, 0]) == 0 and torch.count_nonzero(w[:, :, 2]) == 0
    return (w * (tw.inv * 16).view(-1, 1, 1, 1, 1))[:, :, 1]


def _close(got, ref):
    ref = ref.detach().double()
    amax = ref.abs().amax(dim=(1, 2, 3), keepdim=True)
    return bool(((got.double() - ref).abs() <= ref.abs() * 2 ** -21 + amax * 2 ** -38).all())


class _Args:
    CORR_LEVELS, CORR_RADIUS = 2, 4


def _update_cls():
    return shim.load("stereo.modeling.models.igev.update")


@needs_ref
def test_encoder_pack_splits_k_and_pads_row_127(osb):
    _, ops, update = osb
    torch.manual_seed(0)
    enc = _update_cls().BasicMotionEncoder(_Args()).eval()
    eng = update.MotionEncoderEngine(enc)
    eng._pack()
    w = enc.conv.weight
    for tw, block in ((eng.wc, w[:, :64]), (eng.wd, w[:, 64:])):
        got = _unpack(tw)
        assert got.shape == (128, 64, 3, 3)
        assert torch.count_nonzero(got[127]) == 0                             # the zero-padded output channel
        assert _close(got[:127], block)
    assert eng.b.shape == (128,) and torch.equal(eng.b[:127], enc.conv.bias) and eng.b[127] == 0
    assert torch.equal(eng.c1, enc.convc1.weight[:, :, 0, 0].t())              # (Cin, Cout)
    assert torch.equal(eng.d1, enc.convd1.weight[:, 0])                        # the depthwise (64, 7, 7) weight
    assert _close(_unpack(eng.c2), enc.convc2.weight) and _close(_unpack(eng.d2), enc.convd2.weight)


@needs_ref
def test_disp_head_pack_halves(osb):
    _, ops, update = osb
    torch.manual_seed(1)
    head = _update_cls().DispHead(128, 256, 1).eval()
    eng = update.DispHeadEngine(head)
    eng._pack()
    for i in range(2):
        assert _close(_unpack(eng.w1[i]), head.conv1.weight[128 * i:128 * (i + 1)])
        assert torch.equal(eng.b1[i], head.conv1.bias[128 * i:128 * (i + 1)])
    for i in range(2):                                                          # (Cin, 27 taps, 1), 2D taps at kd = 1
        w = eng.w2[i].view(128, 3, 3, 3)
        assert torch.count_nonzero(w[:, 0]) == 0 and torch.count_nonzero(w[:, 2]) == 0
        assert torch.equal(w[:, 1], head.conv2.weight[0, 128 * i:128 * (i + 1)])


@pytest.mark.parametrize("w,ok", [(128, True), (160, True), (240, True), (64, True), (32, True), (24, True), (23, False), (16, False),
                                  (8, False)])
def test_route_predicate_widths(osb, w, ok):
    _, _, update = osb
    assert update.route_ok(w) is ok


@needs_ref
@pytest.mark.parametrize("case", ["ok", "narrow", "cor_planes", "kernel", "padding", "width127", "hidden96", "mask_width", "head_width"])
def test_engines_serve_only_the_reference_hyper_parameters(osb, case):
    """Every module hyper-parameter other than the reference's (and IGEV-RT's hidden-96 block) runs the reference's own forward."""
    _, _, update = osb
    mod = _update_cls()
    torch.manual_seed(2)
    enc, head = mod.BasicMotionEncoder(_Args()), mod.DispHead(128, 256, 1)
    mask = torch.nn.Sequential(torch.nn.Conv2d(128, 32, 3, padding=1), torch.nn.ReLU(inplace=True))
    b, h, w, cc, hid = 2, 5, 128, 162, 128
    if case == "narrow":
        w = 16
    elif case == "cor_planes":
        cc = 99
    elif case == "kernel":
        enc.convc2 = torch.nn.Conv2d(64, 64, 5, padding=2)
    elif case == "padding":
        enc.convd1 = torch.nn.Conv2d(1, 64, 7, padding=2)
    elif case == "width127":
        enc.conv = torch.nn.Conv2d(128, 126, 3, padding=1)
    elif case == "hidden96":
        hid = 96
        head, mask = mod.DispHead(96, 256, 1), torch.nn.Sequential(torch.nn.Conv2d(96, 32, 3, padding=1), torch.nn.ReLU())
    elif case == "mask_width":
        mask = torch.nn.Sequential(torch.nn.Conv2d(128, 16, 3, padding=1), torch.nn.ReLU())
    elif case == "head_width":
        head = mod.DispHead(128, 192, 1)
    disp, corr, net = torch.zeros(b, 1, h, w), torch.zeros(b, cc, h, w), torch.zeros(b, hid, h, w)
    got = (update.MotionEncoderEngine(enc).serves(disp, corr), update.DispHeadEngine(head).serves(net),
           update.MaskFeatEngine(mask).serves(net))
    want = {"ok": (True, True, True), "narrow": (False, False, False), "cor_planes": (False, True, True),
            "kernel": (False, True, True), "padding": (False, True, True), "width127": (False, True, True),
            "hidden96": (True, False, False), "mask_width": (True, True, False), "head_width": (True, False, True)}[case]
    assert got == want


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


def _igev_rt():
    shim.install_timm_stub()
    cfg = shim.load_cfg("cfgs/igev_rt/igev_rt_sceneflow_uniform.yaml").MODEL
    return shim.load("stereo.modeling.models.igev_rt.igev_rt_stereo").IGEVRTtereo(cfg).eval()


HEADS = ("encoder", "disp_head", "mask_feat_4")


@needs_ref
@pytest.mark.parametrize("build", [_igev, _stereobase])
def test_patch_overrides_per_instance_and_refuses_cpu(osb, build):
    from openstereo_b200.patch import patch
    a, b = build(), build()
    keys = {k: v.clone() for k, v in a.state_dict().items()}
    patch(a)
    assert a.state_dict().keys() == keys.keys() and all(torch.equal(v, keys[k]) for k, v in a.state_dict().items())
    for name in HEADS:
        assert "forward" in vars(getattr(a.update_block, name))             # an instance attribute: the class is untouched
        assert "forward" not in vars(getattr(b.update_block, name))
    ub = a.update_block
    with torch.no_grad():
        for call in (lambda: ub.encoder(torch.zeros(1, 1, 4, 32), torch.zeros(1, 162, 4, 32)),
                     lambda: ub.disp_head(torch.zeros(1, 128, 4, 32)), lambda: ub.mask_feat_4(torch.zeros(1, 128, 4, 32))):
            with pytest.raises(RuntimeError, match="CUDA inference only"):
                call()


@needs_ref
def test_patch_leaves_igev_rt_update_block_alone(osb):
    from openstereo_b200.patch import patch
    m = patch(_igev_rt())
    for name in HEADS + ("gru04", "gru08", "gru16"):
        mod = getattr(m.update_block, name, None)
        assert mod is None or "forward" not in vars(mod)


@needs_ref
def test_patch_non_strict_cpu_equals_reference(osb):
    """strict=False: every CPU call runs the reference's own code, bit for bit (IGEV, 32 GRU iterations at 64x128)."""
    from openstereo_b200.patch import patch
    g = torch.Generator().manual_seed(6)
    x = {"left": torch.rand(1, 3, 64, 128, generator=g) * 255, "right": torch.rand(1, 3, 64, 128, generator=g) * 255}
    with torch.no_grad():
        want = _igev()(dict(x))["disp_pred"]
        got = patch(_igev(), strict=False)(dict(x))["disp_pred"]
    assert torch.isfinite(want).all() and torch.equal(got, want)
