"""GPU: the motion encoder, disp head and mask_feat_4 of IGEV-Stereo / StereoBase on the library (update.py, DESIGN.md section
4.16) -- each engine against its reference module in float64, the K-split layer's NCHW output with a channels-last residual inside
store bounds, the launch sequences, the delegation of narrow widths, the training / autograd refusal, dtypes under autocast, the fp16-range guard and whole
models against the unpatched reference.  Sorted after the torch.profiler routing suites like the other model-level files."""
import pytest
import torch
import torch.nn.functional as F

from oracle import _reference_shim as shim
from oracle import seeded_init as si

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not shim.available(), reason="reference tree (oracle/_ref) not staged")]

TOL = 1e-5          # per element, of the summed |products| feeding it through every layer (the GRU tests' bar)


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, ops, update
    from openstereo_b200.patch import patch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return _lib, ops, update, patch


class _Args:
    CORR_LEVELS, CORR_RADIUS = 2, 4


def _mods(seed):
    torch.manual_seed(seed)
    m = shim.load("stereo.modeling.models.igev.update")
    enc, head = m.BasicMotionEncoder(_Args()).eval(), m.DispHead(128, 256, 1).eval()
    mask = torch.nn.Sequential(torch.nn.Conv2d(128, 32, 3, padding=1), torch.nn.ReLU(inplace=True)).eval()
    return enc, head, mask


def _inputs(ops, b, h, w, seed):
    """disp in 0..48, corr = one geometry-encoding lookup (ops.geo_lookup) of a seeded volume at that disparity, net0 = tanh(.)."""
    g = torch.Generator().manual_seed(seed)
    disp = (torch.rand(b, 1, h, w, generator=g) * 48).cuda()
    g0 = torch.randn(b, 8, 48, h, w, generator=g).cuda()
    c0 = (torch.randn(b, h, w, w, generator=g) * 4).cuda()
    coords = torch.arange(w, dtype=torch.float32, device="cuda").view(1, 1, w).expand(b, h, w).contiguous()
    corr = ops.geo_lookup([g0, ops.avgpool_pairs(g0, 2)], [c0, ops.avgpool_pairs(c0, 3)], disp, coords, 4)
    net = torch.tanh(torch.randn(b, 128, h, w, generator=g) * 2).cuda()
    return disp, corr, net


def _absconv(x, conv):
    return F.conv2d(x, conv.weight.double().abs(), conv.bias.double().abs(), padding=conv.padding)


def _magnitudes(enc, head, mask, disp, corr, net):
    """Per output element, the sum of |products| + |bias| through every layer, float64 (relu(|.|) = |.|)."""
    a = lambda t: t.double().abs()
    cor = _absconv(_absconv(a(corr), enc.convc1), enc.convc2)
    dsp = _absconv(_absconv(a(disp), enc.convd1), enc.convd2)
    m_enc = torch.cat([_absconv(torch.cat([cor, dsp], 1), enc.conv), a(disp)], 1)
    m_head = _absconv(_absconv(a(net), head.conv1), head.conv2)
    return m_enc, m_head, _absconv(a(net), mask[0])


def _check(name, got, want, mag):
    assert got.shape == want.shape and got.dtype == torch.float32 and torch.isfinite(got).all()
    err = (got.cpu().double() - want).abs()
    print("%s: max err %.3e, max err / magnitude %.3e" % (name, err.max(), (err / mag).max()))
    assert (err <= TOL * mag + 1e-6).all()


@pytest.mark.parametrize("w", [128, 160, 240])
def test_engines_against_reference_fp64(osb, w):
    _, ops, update, _ = osb
    enc, head, mask = _mods(w)
    disp, corr, net = _inputs(ops, 2, 5, w, w + 1)
    dc, cc, nc = disp.cpu().double(), corr.cpu().double(), net.cpu().double()
    with torch.no_grad():
        want = (enc.double()(dc, cc), head.double()(nc), mask.double()(nc))
        mags = _magnitudes(enc, head, mask, dc, cc, nc)
        engines = [cls(mod.float().cuda()) for cls, mod in ((update.MotionEncoderEngine, enc), (update.DispHeadEngine, head),
                                                            (update.MaskFeatEngine, mask))]
        assert engines[0].serves(disp, corr) and engines[1].serves(net) and engines[2].serves(net)
        got = (engines[0](disp, corr), engines[1](net), engines[2](net))
        torch.cuda.synchronize()
    for name, g, wt, m in zip(("encoder", "disp_head", "mask_feat_4"), got, want, mags):
        _check("%s W=%d" % (name, w), g, wt, m)
    assert torch.equal(got[0][:, 127:], disp)                              # the reference's torch.cat([out, disp]), bit for bit
    assert ops.tc_overflow_count(reset=True) == 0


def _guarded(n, dev="cuda"):
    pad = 64
    buf = torch.full((n + 2 * pad,), 12345.0, device=dev)
    buf[pad:pad + n] = float("nan")
    return buf, buf[pad:pad + n], pad


def _guards_intact(buf, pad, n):
    return bool((buf[:pad] == 12345.0).all() and (buf[pad + n:] == 12345.0).all())


def test_nchw_output_with_channels_last_residual(osb):
    """The encoder's K-split second launch: NCHW output, channels-last residual, ReLU after the residual, on the whole-row and the
    general-width Cout = 128 instantiations, inside sentinels."""
    lib, ops, _, _ = osb
    for w, variant in ((128, "tcg<128,16,128,1,1,0,0>"), (88, "tcg<128,16,128,1,1,1,0>")):
        g = torch.Generator().manual_seed(w)
        b, h = 2, 3
        x = torch.randn(b, 64, h, w, generator=g)
        wt = torch.randn(128, 64, 3, 3, generator=g) * 0.05
        res = torch.randn(b, h, w, 128, generator=g)
        tw = ops.pack_tc_weight_2d(wt.cuda(), 16)
        n = b * 128 * h * w
        buf, y, pad = _guarded(n)
        r, xn = res.cuda(), x.permute(0, 2, 3, 1).contiguous().cuda()
        lib.call("osb_conv2d_k3_tc_fwd", xn.data_ptr(), tw.data.data_ptr(), tw.eff_scale(None).data_ptr(), None, r.data_ptr(),
                 y.data_ptr(), b, 64, 128, h, w, 1, ops.ACT_RELU, 0, 1, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert ops.tc_last_variant() == variant
        assert torch.isfinite(y).all() and _guards_intact(buf, pad, n)
        got = y.view(b, 128, h, w)
        want = F.relu(F.conv2d(x.double(), wt.double(), padding=1) + res.permute(0, 3, 1, 2).double())
        mag = F.conv2d(x.double().abs(), wt.double().abs(), padding=1) + res.permute(0, 3, 1, 2).double().abs()
        assert ((got.cpu().double() - want).abs() <= TOL * mag + 1e-6).all()


@pytest.mark.parametrize("w,last", [(128, "tcg<128,16,128,1,1,0,0>"), (160, "tcg<128,16,128,1,1,1,0>")])
def test_launch_sequences(osb, w, last):
    lib, ops, update, _ = osb
    enc, head, mask = [m.cuda() for m in _mods(3)]
    disp, corr, net = _inputs(ops, 1, 4, w, 5)
    cases = [(update.MotionEncoderEngine(enc), (disp, corr), 8,
              {"osb_conv3d_1x1_bn_act_fwd": 1, "osb_dwconv2d_fwd": 1, "osb_ncdhw_to_ndhwc_slice": 2, "osb_conv2d_k3_tc_fwd": 4}, last),
             (update.DispHeadEngine(head), (net,), 5,
              {"osb_ncdhw_to_ndhwc_slice": 1, "osb_conv2d_k3_tc_fwd": 2, "osb_conv3d_k3_bn_act_fwd": 2}, last),
             (update.MaskFeatEngine(mask), (net,), 2, {"osb_ncdhw_to_ndhwc_slice": 1, "osb_conv2d_k3_tc_fwd": 1},
              "tc<32>" if w == 128 else "tcg<32,16,128,1,1,1,0>")]
    with torch.no_grad():
        for eng, args, launches, names, variant in cases:
            eng(*args)                                                      # packs the weights
            ops.profile_start()
            before = lib.launch_count()
            eng(*args)
            n = lib.launch_count() - before
            prof = ops.profile_stop()
            assert n == launches
            assert {k: len(v) for k, v in prof.items()} == names
            if variant:
                assert ops.tc_last_variant() == variant


def test_narrow_width_runs_the_reference(osb):
    """W = 16 < OSB_TC_MIN_WIDTH: the patched modules run the reference's own forward, no library launch."""
    lib, ops, update, _ = osb
    from openstereo_b200.patch import _override_engine
    enc, head, mask = [m.cuda() for m in _mods(4)]
    disp, corr, net = _inputs(ops, 2, 8, 16, 6)
    with torch.no_grad():
        want = (enc(disp, corr), head(net), mask(net))
        for mod, cls, what in ((enc, update.MotionEncoderEngine, "encoder"), (head, update.DispHeadEngine, "disp_head"),
                               (mask, update.MaskFeatEngine, "mask_feat_4")):
            _override_engine(mod, cls(mod), True, what)
        before = lib.launch_count()
        got = (enc(disp, corr), head(net), mask(net))
        assert lib.launch_count() == before
    assert all(torch.equal(a, b) for a, b in zip(got, want))


def test_training_and_autograd_never_reach_the_kernels(osb):
    lib, ops, update, _ = osb
    from openstereo_b200.patch import _override_engine
    disp, corr, net = _inputs(ops, 1, 4, 64, 2)
    loose, strict = [m.cuda() for m in _mods(1)], [m.cuda() for m in _mods(1)]
    for mods, st in ((loose, False), (strict, True)):
        for mod, cls in zip(mods, (update.MotionEncoderEngine, update.DispHeadEngine, update.MaskFeatEngine)):
            _override_engine(mod, cls(mod), st, type(mod).__name__)
    calls = lambda ms: (lambda: ms[0](disp, corr), lambda: ms[1](net), lambda: ms[2](net))
    before = lib.launch_count()
    for call, mod in zip(calls(loose), loose):
        out = call()                                                        # grad enabled, parameters require grad
        assert out.requires_grad
        out.sum().backward()
        assert next(mod.parameters()).grad is not None
        mod.train()
        with torch.no_grad():
            call()
    assert lib.launch_count() == before
    for call, mod in zip(calls(strict), strict):
        with pytest.raises(RuntimeError, match="CUDA inference only"):
            call()
        mod.train()
        with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA inference only"):
            call()


@pytest.mark.parametrize("disp_dtype", [torch.float32, torch.float16])
def test_dtypes_under_autocast(osb, disp_dtype):
    """Under fp16 autocast each output has the dtype the reference module returns there (the encoder's is torch.cat's promotion of
    the fp16 conv output and disp), and stays close to the fp32 reference."""
    _, ops, update, _ = osb
    from openstereo_b200.patch import _override_engine
    ref, mine = [m.cuda() for m in _mods(8)], [m.cuda() for m in _mods(8)]
    for mod, cls in zip(mine, (update.MotionEncoderEngine, update.DispHeadEngine, update.MaskFeatEngine)):
        _override_engine(mod, cls(mod), True, type(mod).__name__)
    disp, corr, net = _inputs(ops, 2, 6, 160, 9)
    disp = disp.to(disp_dtype)
    with torch.no_grad():
        want32 = (ref[0](disp.float(), corr), ref[1](net), ref[2](net))
        with torch.autocast("cuda", dtype=torch.float16):
            want = (ref[0](disp, corr), ref[1](net), ref[2](net))
            got = (mine[0](disp, corr), mine[1](net), mine[2](net))
    for g, w, w32 in zip(got, want, want32):
        assert g.dtype == w.dtype and g.shape == w.shape
        assert (g.float() - w32).abs().max().item() <= 2e-3 * max(1.0, w32.abs().max().item())


def test_overflow_monitor_raises(osb):
    _, ops, update, _ = osb
    _, _, mask = _mods(9)
    eng = update.MaskFeatEngine(mask.cuda())
    _, _, net = _inputs(ops, 1, 4, 64, 8)
    ops.tc_overflow_count(reset=True)
    with torch.no_grad():
        eng(net * 1e4)                                                      # |x| far beyond 4094
        torch.cuda.synchronize()
        with pytest.raises(RuntimeError, match="fp16 range"):
            eng(net)
        torch.cuda.synchronize()
    assert ops.tc_overflow_count(reset=True) == 0


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


NEW_ENTRIES = {"osb_conv3d_1x1_bn_act_fwd": 1, "osb_dwconv2d_fwd": 1, "osb_conv3d_k3_bn_act_fwd": 2,
               "osb_conv2d_k3_tc_fwd": 4 + 2 + 1}          # per update-block call: encoder, disp head, mask_feat_4


@pytest.mark.parametrize("name,build", [("IGEVStereo", _igev), ("StereoBase", _stereobase)])
def test_whole_model_against_unpatched(osb, name, build):
    """256x512 through the reference classes and patch(): the encoder and both heads ran on the library at least once per iteration,
    and disp_pred stays within the bar test_zz_gru_gpu.py uses against the unpatched model on GPU and CPU."""
    lib, ops, _, patch = osb
    m = build()
    g = torch.Generator().manual_seed(31)
    x = {"left": torch.rand(1, 3, 256, 512, generator=g) * 255, "right": torch.rand(1, 3, 256, 512, generator=g) * 255}
    with torch.no_grad():
        want_cpu = m(dict(x))["disp_pred"]
        m.cuda()
        xg = {k: v.cuda() for k, v in x.items()}
        want_gpu = m(dict(xg))["disp_pred"]
        patch(m)
        ops.profile_start()
        got = m(dict(xg))["disp_pred"]
        prof = ops.profile_stop()
    counts = {k: len(prof.get(k, [])) for k in NEW_ENTRIES}
    e_gpu = (got - want_gpu).abs().mean().item()
    e_cpu = (got.cpu() - want_cpu).abs().mean().item()
    floor = (want_gpu.cpu() - want_cpu).abs().mean().item()
    print("patch(%s) 256x512: EPE %.3e vs GPU ref, %.3e vs CPU ref (floor %.3e); launches %s" % (name, e_gpu, e_cpu, floor, counts))
    assert all(counts[k] >= 32 * n for k, n in NEW_ENTRIES.items())
    assert len(prof.get("osb_conv2d_k3_tc_gru_fwd", [])) % 6 == 0
    assert torch.isfinite(got).all()
    assert e_gpu <= max(10 * floor, 1e-2) and e_cpu <= max(10 * floor, 1e-2)


def test_igev_544x960_general_width(osb):
    """W' = 240: every new stage on the general-width instantiations; disp_pred finite and within the bar against unpatched fp32."""
    lib, ops, _, patch = osb
    m = _igev().cuda()
    g = torch.Generator().manual_seed(41)
    x = {"left": (torch.rand(1, 3, 544, 960, generator=g) * 255).cuda(), "right": (torch.rand(1, 3, 544, 960, generator=g) * 255).cuda()}
    with torch.no_grad():
        want = m(dict(x))["disp_pred"]
        patch(m)
        ops.profile_start()
        got = m(dict(x))["disp_pred"]
        prof = ops.profile_stop()
    e = (got - want).abs().mean().item()
    print("patch(IGEVStereo) 544x960: EPE %.3e vs GPU ref" % e)
    assert len(prof.get("osb_dwconv2d_fwd", [])) >= 32
    assert torch.isfinite(got).all() and e <= 1e-2
