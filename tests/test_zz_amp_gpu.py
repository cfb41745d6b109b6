"""GPU: the autocast-precision mode of the stride-1 wgmma convolutions (OSB_PREC_F16, DESIGN.md section 4.20) and patch(model,
amp=True) -- at the C ABI per width class the update-block engines use, against fp64 and against F.conv2d's own fp16-autocast error on
the same inputs, with store bounds and the bits of the fp32 mode; the kappa * n count of the single-term MMAs; the fp16 range guard;
every update-block engine under fp16 and bf16 autocast; whole models under their AMP YAML; the training / autograd refusal.  Sorted
after the torch.profiler routing suites like the other model-level files."""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from oracle import _reference_shim as shim
from oracle import seeded_init as si

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not shim.available(), reason="reference tree (oracle/_ref) not staged")]

PREC_FP32, PREC_F16 = 0, 1
RATIO = 1.5          # the f16 mode's error may not exceed 1.5 x the error of the reference's autocast on the same inputs


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, ops
    from openstereo_b200.patch import patch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return _lib, ops, patch


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _guarded(n):
    pad = 64
    buf = torch.full((n + 2 * pad,), 12345.0, device="cuda")
    buf[pad:pad + n] = float("nan")
    return buf, buf[pad:pad + n], pad


def _guards_intact(buf, pad, n):
    return bool((buf[:pad] == 12345.0).all() and (buf[pad + n:] == 12345.0).all())


def _err(got, want):
    return (got.double().cpu() - want.cpu()).abs().mean().item()


# ------------------------------------------------------------------------------------------ the C ABI
# (W', Cin, Cout): the whole-row W' = 128 tiles, the general-width column tiles (160, 80, 40) and the multi-row tiles (64, 32)
ABI_CASES = [(w, cin, cout) for w in (128, 160, 80, 64, 40, 32) for cin, cout in ((64, 64), (128, 128))]


def _conv_case(cin, cout, w, seed, b=2, h=5):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, cin, h, w, generator=g)
    wt = torch.randn(cout, cin, 3, 3, generator=g) * (1.0 / (3 * cin ** 0.5))
    bias = torch.randn(cout, generator=g) * 0.1
    return x, wt, bias


def _autocast_conv(x, wt, bias):
    """F.conv2d under the reference's fp16 autocast, in float64 (its output is fp16)."""
    with torch.autocast("cuda", dtype=torch.float16):
        y = F.conv2d(x.cuda(), wt.cuda(), bias.cuda(), padding=1)
    assert y.dtype == torch.float16
    return y.double().cpu()


def _plain(lib, ops, x, wt, bias, res, prec, entry):
    b, cin, h, w = x.shape
    cout = wt.shape[0]
    tw = ops.pack_tc_weight_2d(wt.cuda(), 16)
    n = b * cout * h * w
    buf, y, pad = _guarded(n)
    xn, r = x.permute(0, 2, 3, 1).contiguous().cuda(), res.permute(0, 2, 3, 1).contiguous().cuda()
    args = [xn.data_ptr(), tw.data.data_ptr(), tw.eff_scale(None).data_ptr(), bias.cuda().data_ptr(), r.data_ptr(), y.data_ptr(), b,
            cin, cout, h, w, 1, ops.ACT_RELU, 0, 1]
    if entry == "new":
        lib.call("osb_conv2d_k3_tc_prec_fwd", *args, prec, _stream())
    else:
        lib.call("osb_conv2d_k3_tc_fwd", *args, _stream())
    torch.cuda.synchronize()
    assert torch.isfinite(y).all() and _guards_intact(buf, pad, n)
    return y.view(b, cout, h, w).clone(), ops.tc_last_variant()


@pytest.mark.parametrize("w,cin,cout", ABI_CASES)
def test_abi_conv_f16_against_fp64_and_autocast(osb, w, cin, cout):
    """relu(conv + bias + channels-last residual), NCHW output: the f16 mode's error against fp64 within 1.5 x F.conv2d's fp16
    autocast error; OSB_PREC_FP32 through the new entry point = the old entry point, bit for bit; sentinels intact."""
    lib, ops, _ = osb
    x, wt, bias = _conv_case(cin, cout, w, w + cout)
    res = torch.randn(x.shape[0], cout, x.shape[2], w, generator=torch.Generator().manual_seed(5))
    want = F.relu(F.conv2d(x.double(), wt.double(), bias.double(), padding=1) + res.double())
    amp = F.relu(_autocast_conv(x, wt, bias) + res.double())
    ops.tc_overflow_count(reset=True)
    f16, v16 = _plain(lib, ops, x, wt, bias, res, PREC_F16, "new")
    f32, v32 = _plain(lib, ops, x, wt, bias, res, PREC_FP32, "new")
    old, vold = _plain(lib, ops, x, wt, bias, res, None, "old")
    e16, e_amp, e32 = _err(f16, want), _err(amp, want), _err(f32, want)
    print("W=%d %d->%d %s: f16 %.3e, autocast %.3e, fp32 %.3e" % (w, cin, cout, v16, e16, e_amp, e32))
    assert v16 == v32 == vold and v16.startswith("tcg<")
    assert torch.equal(f32, old)
    assert e16 <= RATIO * e_amp and e32 < e16 / 20               # the single-term mode did run: fp32-accurate is far closer
    assert ops.tc_overflow_count(reset=True) == 0


def test_abi_conv3d_tc_route_keeps_the_three_term_product(osb):
    """Cout 32 at W' = 128 is served by conv3d_tc.cu (32-channel chunks), which has no single-term mode: OSB_PREC_F16 computes the
    OSB_PREC_FP32 result, bit for bit."""
    lib, ops, _ = osb
    x, wt, bias = _conv_case(128, 32, 128, 3)
    res = torch.randn(2, 32, 5, 128, generator=torch.Generator().manual_seed(6))
    f16, v16 = _plain(lib, ops, x, wt, bias, res, PREC_F16, "new")
    f32, v32 = _plain(lib, ops, x, wt, bias, res, PREC_FP32, "new")
    assert v16 == v32 == "tc<32>" and torch.equal(f16, f32)


GRU_MODES = ["sigmoid_mul", "tanh_blend"]


def _gru(lib, ops, xn, wt, shift, res_nchw, mode, mul, bz, bh, prec, entry):
    b, h, w, cin = xn.shape
    tw = ops.pack_tc_weight_2d(wt.cuda(), 16)
    n = b * 128 * h * w
    buf, y, pad = _guarded(n)
    act = ops.ACT_SIGMOID if mode == "sigmoid_mul" else ops.ACT_TANH
    args = [xn.data_ptr(), tw.data.data_ptr(), tw.eff_scale(None).data_ptr(), shift.data_ptr(), res_nchw.data_ptr(),
            mul.data_ptr() if mode == "sigmoid_mul" else None, bz.data_ptr() if mode == "tanh_blend" else None,
            bh.data_ptr() if mode == "tanh_blend" else None, y.data_ptr(), b, cin, 128, h, w, act, 1, 0, 0]
    if entry == "new":
        lib.call("osb_conv2d_k3_tc_gru_prec_fwd", *args, prec, _stream())
    else:
        lib.call("osb_conv2d_k3_tc_gru_fwd", *args, _stream())
    torch.cuda.synchronize()
    assert torch.isfinite(y).all() and _guards_intact(buf, pad, n)
    return y.view(b, h, w, 128).clone(), ops.tc_last_variant()


@pytest.mark.parametrize("mode", GRU_MODES)
@pytest.mark.parametrize("w", [128, 160, 80, 64, 40, 32])
def test_abi_gru_f16_against_fp64_and_autocast(osb, w, mode):
    """The ConvGRU epilogue modes (sigmoid + r * h, tanh + the blend) on the Cout = 128 instantiations: as the plain conv above."""
    lib, ops, _ = osb
    x, wt, shift = _conv_case(128, 128, w, 7 * w + len(mode))
    b, _, h, _ = x.shape
    g = torch.Generator().manual_seed(w)
    res = torch.randn(b, 128, h, w, generator=g)                       # NCHW context (cz / cr / cq)
    mul, bz, bh = (torch.rand(b, h, w, 128, generator=g) for _ in range(3))
    act = torch.sigmoid if mode == "sigmoid_mul" else torch.tanh

    def epilogue(conv):
        v = act(conv + res.double()).permute(0, 2, 3, 1)
        return v * mul.double() if mode == "sigmoid_mul" else bh.double() + bz.double() * (v - bh.double())
    want = epilogue(F.conv2d(x.double(), wt.double(), shift.double(), padding=1))
    amp = epilogue(_autocast_conv(x, wt, shift))
    xn = x.permute(0, 2, 3, 1).contiguous().cuda()
    ops_args = (xn, wt, shift.cuda(), res.cuda(), mode, mul.cuda(), bz.cuda(), bh.cuda())
    f16, v16 = _gru(lib, ops, *ops_args, PREC_F16, "new")
    f32, v32 = _gru(lib, ops, *ops_args, PREC_FP32, "new")
    old, vold = _gru(lib, ops, *ops_args, None, "old")
    e16, e_amp, e32 = _err(f16, want), _err(amp, want), _err(f32, want)
    print("GRU %s W=%d %s: f16 %.3e, autocast %.3e, fp32 %.3e" % (mode, w, v16, e16, e_amp, e32))
    assert v16 == v32 == vold and v16.startswith("tcg<128,")
    assert torch.equal(f32, old)
    assert e16 <= RATIO * e_amp and e32 < e16 / 20


def test_correction_counts_the_single_term_mmas(osb):
    """With kappa raised, the f16 output scales by 1 + kappa * n for n = the MMAs it issued (D = 1: Cin / 16 chunks x 3 kh taps),
    not the 3-term count (three times that); kappa is restored afterwards."""
    lib, ops, _ = osb
    x, wt, _ = _conv_case(128, 128, 160, 11)
    tw = ops.pack_tc_weight_2d(wt.cuda(), 16)
    xn = x.permute(0, 2, 3, 1).contiguous().cuda()
    kappa = 9e-7

    def run(prec):
        y = torch.empty(2, 5, 160, 128, device="cuda")
        lib.call("osb_conv2d_k3_tc_prec_fwd", xn.data_ptr(), tw.data.data_ptr(), tw.eff_scale(None).data_ptr(), None, None,
                 y.data_ptr(), 2, 128, 128, 5, 160, 1, ops.ACT_NONE, 1, 1, prec, _stream())
        torch.cuda.synchronize()
        return y.double()
    default = ops.set_rz_kappa(0.0)
    try:
        base = {p: run(p) for p in (PREC_F16, PREC_FP32)}
        ops.set_rz_kappa(kappa)
        raised = {p: run(p) for p in (PREC_F16, PREC_FP32)}
    finally:
        ops.set_rz_kappa(default)
    assert ops.set_rz_kappa(default) == default
    n1 = (128 // 16) * 3
    for p, n in ((PREC_F16, n1), (PREC_FP32, 3 * n1)):
        keep = base[p].abs() > 1e-2
        shrink = (raised[p][keep] / base[p][keep]).median().item() - 1.0
        print("precision %d: measured kappa * n = %.4e, expected %.4e" % (p, shrink, kappa * n))
        assert abs(shrink - kappa * n) <= 0.1 * kappa * n


@pytest.mark.parametrize("prec", [PREC_FP32, PREC_F16])
def test_range_guard_reports_in_both_modes(osb, prec):
    """An activation just beyond +-4094 raises the sticky overflow count in the single-term mode as in the 3-term mode."""
    lib, ops, _ = osb
    x, wt, bias = _conv_case(64, 64, 160, 13)
    ops.tc_overflow_count(reset=True)
    res = torch.zeros(2, 64, 5, 160)
    _plain(lib, ops, x, wt, bias, res, prec, "new")
    assert ops.tc_overflow_count(reset=True) == 0
    x[1, 7, 2, 33] = -4100.0
    _plain(lib, ops, x, wt, bias, res, prec, "new")
    assert ops.tc_overflow_count(reset=True) >= 1


# ------------------------------------------------------------------------------------------ the engines
def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _igev_update():
    return shim.load("stereo.modeling.models.igev.update")


class _Args:
    CORR_LEVELS, CORR_RADIUS = 2, 4


def _engine_cases(ops, w, seed):
    """(name, module, engine class, inputs) for every update-block engine at image width w, b = 2, h = 4."""
    from types import SimpleNamespace
    from openstereo_b200 import gru, update
    b, h = 2, 4
    g = _gen(seed)
    torch.manual_seed(seed)
    igev = _igev_update()
    pp = shim.load("stereo.modeling.models.igevpp.update")
    from oracle import monster as omon
    mon = omon.load_reference("stereo.modeling.models.monster.update")
    rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).cuda()   # noqa: E731
    disp = (torch.rand(b, 1, h, w, generator=g) * 48).cuda()
    net = torch.tanh(rnd(b, 128, h, w, scale=2.0))
    ctx = rnd(b, 384, h, w)
    corr = rnd(b, 2 * 9 * 9, h, w)                                      # (CORR_LEVELS * 2 levels) x (2r + 1) planes, r = 4
    cases = [
        ("ConvGRU", igev.ConvGRU(128, 256).eval(), gru.ConvGRUEngine, (net, *ctx.split(128, 1), rnd(b, 128, h, w), rnd(b, 128, h, w))),
        ("BasicMotionEncoder", igev.BasicMotionEncoder(_Args()).eval(), update.MotionEncoderEngine, (disp, corr)),
        ("DispHead", igev.DispHead(128, 256, 1).eval(), update.DispHeadEngine, (net,)),
        ("mask_feat_4", torch.nn.Sequential(torch.nn.Conv2d(128, 32, 3, padding=1), torch.nn.ReLU(inplace=True)).eval(),
         update.MaskFeatEngine, (net,)),
        ("GeoEncoder", pp.GeoEncoder(144).eval(), update.GeoEncoderEngine, (rnd(b, 144, h, w),)),
        ("BasicDispEncoder", pp.BasicDispEncoder(SimpleNamespace(CORR_RADIUS=4)).eval(), update.DispEncoderEngine,
         (disp, rnd(b, 96 + 18, h, w))),
        ("BasicMotionEncoder_mix2", mon.BasicMotionEncoder_mix2(SimpleNamespace(corr_levels=2, corr_radius=4)).eval(),
         update.MixMotionEncoderEngine, (disp, corr, rnd(b, 96, h, w), disp * 0.9, rnd(b, 162, h, w), rnd(b, 96, h, w))),
    ]
    return cases


def _f64(module):
    import copy
    return copy.deepcopy(module).double()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("w", [128, 160])
def test_engines_under_autocast_with_amp(osb, w, dtype):
    """Every update-block engine built with amp=True, installed as its module's forward, under fp16 and bf16 autocast: the output
    dtype is the reference module's there, and the error against the module in fp64 is within 1.5 x the reference module's own
    autocast error on the same inputs.  Outside autocast the amp engine computes the amp=False engine's result, bit for bit."""
    _, ops, _ = osb
    from openstereo_b200.patch import _override, _override_engine
    for name, ref, cls, args in _engine_cases(ops, w, 21 + w):
        ref = ref.cuda()
        mine = _f64(ref).float().cuda()
        eng = cls(mine, amp=True)
        if cls.__name__ == "ConvGRUEngine":
            _override(mine, "ConvGRU", True, eng, lambda h, cz, cr, cq, *x: eng.serves(h, x))
        else:
            _override_engine(mine, eng, True, name)
        assert eng.amp
        with torch.no_grad():
            want = _f64(ref)(*[a.double() for a in args])
            with torch.autocast("cuda", dtype=dtype):
                assert eng._precision() == "f16"
                assert eng.serves(*args) if cls.__name__ != "ConvGRUEngine" else eng.serves(args[0], args[4:])
                ref_out, got = ref(*args), mine(*args)
            plain = cls(_f64(ref).float().cuda())                          # outside autocast: amp=True computes amp=False's bits
            assert torch.equal(eng(*args), plain(*args))
        ops.tc_overflow_count(reset=True)
        e_got, e_ref = _err(got, want), _err(ref_out, want)
        print("%s W=%d %s: amp engine %.3e, reference autocast %.3e (%s)" % (name, w, dtype, e_got, e_ref, got.dtype))
        assert got.dtype == ref_out.dtype and got.shape == ref_out.shape and torch.isfinite(got).all()
        assert e_got <= RATIO * e_ref


# ------------------------------------------------------------------------------------------ whole models
def _igev(yaml="cfgs/igev/igev_sceneflow_amp.yaml"):
    shim.install_timm_stub()
    cfg = shim.load_cfg(yaml).MODEL
    m = shim.load("stereo.modeling.models.igev.igev_stereo").IGEVStereo(cfg).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=12, scale={"classifier.weight": 8.0}))
    return m


def _stereobase():
    shim.install_timm_stub()
    cfg = shim.load_cfg("cfgs/stereobase/stereobase_sceneflow.yaml").MODEL
    m = shim.load("stereo.modeling.models.stereobase.stereobase_gru").StereoBase(cfg).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=3, scale={"classifier.weight": 8.0}))
    return m


def _igevpp(amp):
    from oracle import igevpp as oigpp
    return oigpp.igevpp(oigpp.AMP_YAML if amp else oigpp.UNIFORM_YAML)


def _monster(amp):
    from oracle import monster as omon
    return omon.monster(omon.AMP_YAML if amp else omon.UNIFORM_YAML)


def _monster_dtype():
    from oracle import monster as omon
    return omon.amp_dtype(omon.AMP_YAML)


# name -> (build(amp YAML?), autocast dtype the AMP YAML's trainer wraps the forward in (None: the model autocasts itself),
#          input scale)
MODELS = {
    "IGEVStereo": (lambda amp: _igev(), lambda: torch.float16, 255.0),
    "StereoBase": (lambda amp: _stereobase(), lambda: torch.float16, 255.0),
    "IGEVPPStereo": (_igevpp, lambda: None, 1.0),
    "MonSter": (_monster, _monster_dtype, 1.0),
}


def _x(b, h, w, seed, scale):
    g = torch.Generator().manual_seed(seed)
    if scale == 1.0:
        return {"left": (torch.rand(b, 3, h, w, generator=g) * 2 - 1).cuda(), "right": (torch.rand(b, 3, h, w, generator=g) * 2 - 1).cuda()}
    return {"left": (torch.rand(b, 3, h, w, generator=g) * scale).cuda(), "right": (torch.rand(b, 3, h, w, generator=g) * scale).cuda()}


def _autocast(dtype):
    return torch.autocast("cuda", dtype=dtype) if dtype else contextlib.nullcontext()


@pytest.mark.parametrize("name", sorted(MODELS))
def test_whole_model_under_amp_yaml(osb, name):
    """256x512 under the AMP YAML: patch(amp=True)'s EPE against the unpatched fp32 model is at most 1.25 x the unpatched AMP model's
    EPE against it, + 1e-3 px, with the AMP model's output dtype.  With autocast off amp=True launches exactly what amp=False does
    (no single-term launch) and gives its disparities up to the run-to-run spread of the amp=False model itself: the reference's own
    layers need not repeat their bits from run to run; the engines' bits are compared in test_engines_under_autocast_with_amp."""
    lib, ops, patch = osb
    build, dtype_of, scale = MODELS[name]
    dtype = dtype_of()
    x = _x(1, 256, 512, 91, scale)
    with torch.no_grad():
        fp32 = build(False).cuda()(dict(x))["disp_pred"].float()
        with _autocast(dtype):
            amp = build(True).cuda()(dict(x))["disp_pred"]
            ops.profile_start()
            got = patch(build(True).cuda(), amp=True)(dict(x))["disp_pred"]
            prof = ops.profile_stop()
        e_amp, e_got = (amp.float() - fp32).abs().mean().item(), (got.float() - fp32).abs().mean().item()
        print("patch(%s, amp=True) under the AMP YAML (%s): EPE %.3e vs fp32 (unpatched AMP %.3e), dtype %s; f16 launches %s" % (
            name, dtype, e_got, e_amp, got.dtype, {k: len(v) for k, v in prof.items() if "prec" in k}))
        assert len(prof.get("osb_conv2d_k3_tc_gru_prec_fwd", [])) >= 32 * 18 and len(prof.get("osb_conv2d_k3_tc_prec_fwd", [])) > 0
        assert got.dtype == amp.dtype and torch.isfinite(got.float()).all() and fp32.std() > 0.5
        assert e_got <= 1.25 * e_amp + 1e-3
        runs = {}
        for amp_flag in (True, False):
            m = patch(build(False).cuda(), amp=amp_flag)
            ops.profile_start()
            out = m(dict(x))["disp_pred"]
            runs[amp_flag] = (out, {k: len(v) for k, v in ops.profile_stop().items()})
        (a, pa), (b, pb) = runs[True], runs[False]
        spread = (m(dict(x))["disp_pred"] - b).abs().max().item()
    diff = (a - b).abs().max().item()
    print("autocast off: amp=True vs amp=False max |diff| %.3e, amp=False run-to-run %.3e" % (diff, spread))
    assert pa == pb and not any("prec" in k for k in pa)
    assert diff <= 2 * spread


def test_training_and_autograd_never_reach_the_kernels(osb):
    """patch(amp=True) keeps the guard: under autocast, a training-mode or autograd-recording call raises in strict mode and runs the
    reference's code with strict=False."""
    lib, ops, patch = osb
    x = _x(1, 64, 128, 93, 255.0)
    m = patch(_igev().cuda(), amp=True)
    with torch.autocast("cuda", dtype=torch.float16):
        with pytest.raises(RuntimeError, match="CUDA inference only"):
            m(dict(x))                                                  # autograd recording through the parameters
        m.train()
        with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA inference only"):
            m(dict(x))
    c = patch(_igev().cuda(), strict=False, amp=True).train()
    before = lib.launch_count()
    with torch.autocast("cuda", dtype=torch.float16):
        out = c(dict(x))
    assert lib.launch_count() == before
    out["disp_pred"].float().mean().backward()
    assert c.update_block.gru04.convz.weight.grad is not None and c.update_block.encoder.conv.weight.grad is not None
