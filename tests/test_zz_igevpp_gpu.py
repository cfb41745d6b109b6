"""GPU: IGEV++ on the library -- the multi-range lookup (one launch of geo_lookup_kernel's third mode) against the reference in float64
and fp32 with store bounds checked by sentinels, the combined and geometry-only modes' bits around multi-range calls, the new
update-block engines (geo encoders, disparity encoder, Cout-64 mask head) against their modules in float64, launch sequences, the
narrow-width delegation, autocast dtypes, the fp16-range guard, the training / autograd refusal, and the whole model under both YAMLs
against the unpatched model.  Sorted after the torch.profiler routing suites like the other model-level files."""
import pytest
import torch
import torch.nn.functional as F

from oracle import _reference_shim as shim
from oracle import igevpp as oigpp

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not shim.available(), reason="reference tree (oracle/_ref) not staged")]

TOL = 1e-5          # per element, of the summed |products| feeding it through every layer (the update-block tests' bar)


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, ops, update
    from openstereo_b200.patch import patch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return _lib, ops, update, patch


# ------------------------------------------------------------------------------------------ multi-range lookup
def _lookup_case(b, c, d0, d1, d2, h, w, levels, radius, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    v0, v1, v2 = (torch.randn(b, c, d, h, w, generator=g).to(dtype) for d in (d0, d1, d2))
    f1, f2 = torch.randn(b, 6, h, w, generator=g).to(dtype), torch.randn(b, 6, h, w, generator=g).to(dtype)
    top = 4 * max(d0, d1, d2) + 2 * radius + 8
    disp = (torch.rand(b, 1, h, w, generator=g) * top - radius - 4).to(dtype)
    disp[0, 0, 0, :3] = torch.tensor([-radius - 1.5, 4 * d2 + radius + 1.5, 2.5], dtype=dtype)
    coords = torch.arange(w).to(dtype).reshape(1, 1, w, 1).repeat(b, h, 1, 1)
    return v0, v1, v2, f1, f2, disp, coords


def _guarded(n):
    pad = 64
    buf = torch.full((n + 2 * pad,), 12345.0, device="cuda")
    buf[pad:pad + n] = float("nan")
    return buf, buf[pad:pad + n], pad


def _guards_intact(buf, pad, n):
    return bool((buf[:pad] == 12345.0).all() and (buf[pad + n:] == 12345.0).all())


CASES = [  # (B, C, D0, D1, D2, H, W, levels, radius)
    (2, 8, 48, 48, 48, 3, 131, 2, 4), (1, 8, 48, 13, 30, 2, 21, 1, 4), (3, 5, 24, 17, 9, 2, 9, 2, 2), (2, 4, 16, 24, 6, 3, 133, 2, 1),
    (1, 3, 20, 7, 33, 2, 40, 2, 3), (2, 8, 48, 48, 48, 2, 128, 1, 2)]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "x".join(map(str, c)))
def test_multirange_lookup_against_reference(osb, case):
    """One launch writes the reference's four tensors: within 2^-22 of the |v0|*w0 + |v1|*w1 magnitude of the fp32 reference class on
    the CPU (2^-20 for the correlation rows); against float64 within 3e-5 of that magnitude plus the largest sample (a weight's fp32
    coordinate rounding); exact zeros past the rows, no store outside any tensor."""
    lib, ops, _, _ = osb
    from openstereo_b200 import geo
    b, c, d0, d1, d2, h, w, levels, radius = case
    v0, v1, v2, f1, f2, disp, coords = _lookup_case(*case, seed=sum(case))
    ref = oigpp.load_reference("stereo.modeling.models.igevpp.geometry").Combined_Geo_Encoding_Volume
    want32 = ref(v0, v1, v2, f1, f2, radius=radius, num_levels=levels)(disp, coords)
    d64 = [t.double() for t in (v0, v1, v2, f1, f2)]
    want64 = oigpp.MultiRangeGeoEncodingVolume(*d64, radius=radius, num_levels=levels)(disp.double(), coords.double())
    mag = oigpp.MultiRangeGeoEncodingVolume(*[t.abs() for t in d64], radius=radius, num_levels=levels)(disp.double(), coords.double())
    vol = geo.MultiRangeGeoEncodingVolume(v0.cuda(), v1.cuda(), v2.cuda(), f1.cuda(), f2.cuda(), radius=radius, num_levels=levels)
    before = lib.launch_count()
    got = vol(disp.cuda(), coords.cuda())
    assert lib.launch_count() == before + 1
    t = 2 * radius + 1
    shapes = ((b, levels * c * t, h, w), (b, c * t, h, w), (b, c * t, h, w), (b, levels * t, h, w))
    from oracle.geo_lookup import all_pairs_correlation
    tops = [v0.abs().max().item(), v1.abs().max().item(), v2.abs().max().item(), all_pairs_correlation(f1, f2).abs().max().item()]
    for name, gt, w32, w64, m, shape, top in zip(("geo_feat0", "geo_feat1", "geo_feat2", "init_corr"), got, want32, want64, mag, shapes,
                                                 tops):
        assert gt.shape == shape and gt.dtype == torch.float32
        gc = gt.cpu()
        # fp32 replays the reference's fp32 coordinate round trip, so the tap weights carry its rounding: against float64 that
        # rounding (a few ulp of a coordinate up to 4 * D) is part of the bar; init_corr also carries the all-pairs GEMM's summation
        # order (cuBLAS on the GPU, CPU BLAS in the reference)
        tol = 2 ** -20 if name == "init_corr" else 2 ** -22
        assert ((gc.double() - w64).abs() <= 3e-5 * (m + top) + 1e-30).all(), name
        assert ((gc - w32).abs() <= tol * m.float() + 1e-30).all(), name
        assert torch.equal(gc[w64 == 0], w32[w64 == 0]), name                # taps past both ends: exact zeros
    # store bounds: the four outputs inside sentinels, one launch
    bufs = [_guarded(b * s[1] * h * w) for s in shapes]
    gp = [vol.geo_volume0_pyramid[i].data_ptr() if i < levels else None for i in range(4)]
    cp = [vol.init_corr_pyramid[i].data_ptr() if i < levels else None for i in range(4)]
    dg, cg = disp.cuda(), coords.cuda().reshape(b, h, w).contiguous()
    lib.call("osb_geo_multirange_lookup_fwd", *gp, vol.geo_volume1.data_ptr(), vol.geo_volume2.data_ptr(), *cp, dg.data_ptr(),
             cg.data_ptr(), *[y.data_ptr() for _, y, _ in bufs], b, c, d0, d1, d2, h, w, w, levels, radius,
             torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for (buf, y, pad), gt in zip(bufs, got):
        assert _guards_intact(buf, pad, y.numel()) and torch.equal(y.view_as(gt), gt)


def test_other_modes_keep_their_bits_around_multirange_calls(osb):
    """The combined (IGEV / StereoBase) and geometry-only (IGEV-RT) lookups compute the same bits before and after multi-range
    launches of the same kernel instantiations in the same process."""
    _, ops, _, _ = osb
    g = torch.Generator().manual_seed(3)
    b, c, d, h, w = 2, 8, 48, 3, 133
    g0 = torch.randn(b, c, d, h, w, generator=g).cuda()
    c0 = torch.randn(b, h, w, w, generator=g).cuda()
    disp = (torch.rand(b, 1, h, w, generator=g) * 60 - 6).cuda()
    coords = torch.arange(w, dtype=torch.float32, device="cuda").view(1, 1, w).expand(b, h, w).contiguous()
    gp, cpy = [g0, ops.avgpool_pairs(g0, 2)], [c0, ops.avgpool_pairs(c0, 3)]

    def run():
        return [ops.geo_lookup(gp, cpy, disp, coords, r) for r in (4, 2)] + [ops.geo_volume_lookup(gp, disp, r) for r in (4, 3)]
    first = run()
    for r in (4, 2):
        ops.geo_multirange_lookup(gp, g0, g0[:, :, :20].contiguous(), cpy, disp, coords, r)
    second = run()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(first, second))


# ------------------------------------------------------------------------------------------ update-block engines
def _mods(seed):
    from types import SimpleNamespace
    torch.manual_seed(seed)
    m = shim.load("stereo.modeling.models.igevpp.update")
    mask = torch.nn.Sequential(torch.nn.Conv2d(128, 64, 3, padding=1), torch.nn.ReLU(inplace=True))
    return (m.GeoEncoder(144).eval(), m.GeoEncoder(72).eval(), m.BasicDispEncoder(SimpleNamespace(CORR_RADIUS=4)).eval(),
            mask.eval())


def _inputs(ops, b, h, w, seed):
    """One multi-range lookup of seeded volumes (geo_feat0, geo_feat1, init_corr), disp in 0..48 and net0 = tanh(.)."""
    g = torch.Generator().manual_seed(seed)
    disp = (torch.rand(b, 1, h, w, generator=g) * 48).cuda()
    v = [torch.randn(b, 8, 48, h, w, generator=g).cuda() for _ in range(3)]
    c0 = (torch.randn(b, h, w, w, generator=g) * 4).cuda()
    coords = torch.arange(w, dtype=torch.float32, device="cuda").view(1, 1, w).expand(b, h, w).contiguous()
    f0, f1, _, corr = ops.geo_multirange_lookup([v[0], ops.avgpool_pairs(v[0], 2)], v[1], v[2], [c0, ops.avgpool_pairs(c0, 3)], disp,
                                                coords, 4)
    enc_in = torch.cat([torch.randn(b, 96, h, w, generator=g).cuda(), corr], 1)          # the blended geo_feat and init_corr
    net = torch.tanh(torch.randn(b, 128, h, w, generator=g) * 2).cuda()
    return f0, f1, disp, enc_in, net


def _absconv(x, conv):
    return F.conv2d(x, conv.weight.double().abs(), conv.bias.double().abs(), padding=conv.padding)


def _check(name, got, want, mag):
    assert got.shape == want.shape and got.dtype == torch.float32 and torch.isfinite(got).all()
    err = (got.cpu().double() - want).abs()
    print("%s: max err %.3e, max err / magnitude %.3e" % (name, err.max(), (err / mag).max()))
    assert (err <= TOL * mag + 1e-6).all()


@pytest.mark.parametrize("w", [128, 160, 240])
def test_engines_against_reference_fp64(osb, w):
    _, ops, update, _ = osb
    ge0, ge1, enc, mask = _mods(w)
    f0, f1, disp, enc_in, net = _inputs(ops, 2, 5, w, w + 1)
    a = lambda t: t.cpu().double().abs()
    with torch.no_grad():
        want = (ge0.double()(f0.cpu().double()), ge1.double()(f1.cpu().double()), enc.double()(disp.cpu().double(), enc_in.cpu().double()),
                mask.double()(net.cpu().double()))
        mags = (_absconv(_absconv(a(f0), ge0.convg1), ge0.convg2), _absconv(_absconv(a(f1), ge1.convg1), ge1.convg2),
                torch.cat([_absconv(torch.cat([_absconv(_absconv(a(enc_in), enc.convc1), enc.convc2),
                                               _absconv(_absconv(a(disp), enc.convd1), enc.convd2)], 1), enc.conv), a(disp)], 1),
                _absconv(a(net), mask[0]))
        engines = [cls(mod.float().cuda()) for cls, mod in ((update.GeoEncoderEngine, ge0), (update.GeoEncoderEngine, ge1),
                                                            (update.DispEncoderEngine, enc), (update.MaskFeatEngine, mask))]
        assert engines[0].serves(f0) and engines[1].serves(f1) and engines[2].serves(disp, enc_in) and engines[3].serves(net)
        got = (engines[0](f0), engines[1](f1), engines[2](disp, enc_in), engines[3](net))
        torch.cuda.synchronize()
    for name, g, wt, m in zip(("geo_encoder0", "geo_encoder1", "encoder", "mask_feat_4"), got, want, mags):
        _check("%s W=%d" % (name, w), g.contiguous(), wt, m)
    assert got[0].shape[1] == 96 and torch.equal(got[0]._base[:, 96:], torch.zeros_like(got[0]._base[:, 96:]))   # exact zero pad rows
    assert torch.equal(got[2][:, 127:], disp)                              # the reference's torch.cat([out, disp]), bit for bit
    assert ops.tc_overflow_count(reset=True) == 0


@pytest.mark.parametrize("w,last", [(128, "tcg<128,16,128,1,1,0,0>"), (160, "tcg<128,16,128,1,1,1,0>")])
def test_launch_sequences(osb, w, last):
    lib, ops, update, _ = osb
    ge0, _, enc, mask = [m.cuda() for m in _mods(3)]
    f0, _, disp, enc_in, net = _inputs(ops, 1, 4, w, 5)
    cases = [(update.GeoEncoderEngine(ge0), (f0,), 3,
              {"osb_conv3d_1x1_bn_act_fwd": 1, "osb_ncdhw_to_ndhwc_slice": 1, "osb_conv2d_k3_tc_fwd": 1}, last),
             (update.DispEncoderEngine(enc), (disp, enc_in), 8,
              {"osb_conv3d_1x1_bn_act_fwd": 1, "osb_dwconv2d_fwd": 1, "osb_ncdhw_to_ndhwc_slice": 2, "osb_conv2d_k3_tc_fwd": 4}, last),
             (update.MaskFeatEngine(mask), (net,), 2, {"osb_ncdhw_to_ndhwc_slice": 1, "osb_conv2d_k3_tc_fwd": 1},
              "tcg<64,16,128,1,1,0,0>" if w == 128 else "tcg<64,16,128,1,1,1,0>")]
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
            assert ops.tc_last_variant() == variant


@pytest.mark.parametrize("w,variant", [(128, "tc<32>"), (160, "tcg<32,16,128,1,1,1,0>")])
def test_mask_feat_cout32_launches_what_it_did(osb, w, variant):
    """IGEV's and StereoBase's Cout-32 mask head: one pack and one launch of the Cout-32 instantiation, as before Cout 64 was served."""
    lib, ops, update, _ = osb
    torch.manual_seed(4)
    mask = torch.nn.Sequential(torch.nn.Conv2d(128, 32, 3, padding=1), torch.nn.ReLU(inplace=True)).eval().cuda()
    net = torch.tanh(torch.randn(2, 128, 4, w, device="cuda"))
    eng = update.MaskFeatEngine(mask)
    with torch.no_grad():
        assert eng.serves(net)
        eng(net)
        ops.profile_start()
        before = lib.launch_count()
        y = eng(net)
        prof = ops.profile_stop()
        assert lib.launch_count() - before == 2
        assert {k: len(v) for k, v in prof.items()} == {"osb_ncdhw_to_ndhwc_slice": 1, "osb_conv2d_k3_tc_fwd": 1}
        assert ops.tc_last_variant() == variant and list(eng.w) == [ops.conv2d_tc_kc(128, 32, w)]
        assert (y - mask(net)).abs().max().item() <= 1e-4


def test_narrow_width_runs_the_reference(osb):
    """W = 16 < OSB_TC_MIN_WIDTH: the patched modules run the reference's own forward, no library launch."""
    lib, ops, update, _ = osb
    from openstereo_b200.patch import _override_engine
    ge0, ge1, enc, mask = [m.cuda() for m in _mods(4)]
    f0, f1, disp, enc_in, net = _inputs(ops, 2, 8, 16, 6)
    with torch.no_grad():
        want = (ge0(f0), ge1(f1), enc(disp, enc_in), mask(net))
        for mod, cls in ((ge0, update.GeoEncoderEngine), (ge1, update.GeoEncoderEngine), (enc, update.DispEncoderEngine),
                         (mask, update.MaskFeatEngine)):
            _override_engine(mod, cls(mod), True, type(mod).__name__)
        before = lib.launch_count()
        got = (ge0(f0), ge1(f1), enc(disp, enc_in), mask(net))
        assert lib.launch_count() == before
    assert all(torch.equal(a, b) for a, b in zip(got, want))


def test_training_and_autograd_never_reach_the_kernels(osb):
    lib, ops, update, _ = osb
    from openstereo_b200.patch import _override_engine
    f0, f1, disp, enc_in, net = _inputs(ops, 1, 4, 64, 2)
    classes = (update.GeoEncoderEngine, update.GeoEncoderEngine, update.DispEncoderEngine, update.MaskFeatEngine)
    loose, strict = [m.cuda() for m in _mods(1)], [m.cuda() for m in _mods(1)]
    for mods, st in ((loose, False), (strict, True)):
        for mod, cls in zip(mods, classes):
            _override_engine(mod, cls(mod), st, type(mod).__name__)
    calls = lambda ms: (lambda: ms[0](f0), lambda: ms[1](f1), lambda: ms[2](disp, enc_in), lambda: ms[3](net))
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


def test_dtypes_under_autocast(osb):
    """Under fp16 autocast each output has the dtype the reference module returns there (the encoder's is torch.cat's promotion of
    the fp16 conv output and the fp32 disp), and stays close to the fp32 reference."""
    _, ops, update, _ = osb
    from openstereo_b200.patch import _override_engine
    ref, mine = [m.cuda() for m in _mods(8)], [m.cuda() for m in _mods(8)]
    for mod, cls in zip(mine, (update.GeoEncoderEngine, update.GeoEncoderEngine, update.DispEncoderEngine, update.MaskFeatEngine)):
        _override_engine(mod, cls(mod), True, type(mod).__name__)
    f0, f1, disp, enc_in, net = _inputs(ops, 2, 6, 160, 9)
    calls = lambda ms: (ms[0](f0), ms[1](f1), ms[2](disp, enc_in), ms[3](net))
    with torch.no_grad():
        want32 = calls(ref)
        with torch.autocast("cuda", dtype=torch.float16):
            want, got = calls(ref), calls(mine)
    for g, w, w32 in zip(got, want, want32):
        assert g.dtype == w.dtype and g.shape == w.shape
        assert (g.float() - w32).abs().max().item() <= 2e-3 * max(1.0, w32.abs().max().item())


def test_overflow_monitor_raises(osb):
    _, ops, update, _ = osb
    ge0 = _mods(9)[0]
    eng = update.GeoEncoderEngine(ge0.cuda())
    f0 = _inputs(ops, 1, 4, 64, 8)[0]
    ops.tc_overflow_count(reset=True)
    with torch.no_grad():
        eng(f0 * 1e5)                                                       # convg1's output far beyond 4094
        torch.cuda.synchronize()
        with pytest.raises(RuntimeError, match="fp16 range"):
            eng(f0)
        torch.cuda.synchronize()
    assert ops.tc_overflow_count(reset=True) == 0


# ------------------------------------------------------------------------------------------ the whole model
def _x(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return {"left": torch.rand(b, 3, h, w, generator=g) * 2 - 1, "right": torch.rand(b, 3, h, w, generator=g) * 2 - 1}


def test_patched_forward_launch_count(osb):
    """256x512 (W' = 128), 32 iterations: per iteration one lookup, 3 x 6 ConvGRU launches + 3 x 2 packs of their inputs, 3 x 3 geo
    encoder launches, 8 encoder launches, 5 disp head and 2 mask head launches; once per forward the gwc volume, 3 classifiers,
    3 regressions, the two pyramid levels and the convex up-sampling."""
    lib, ops, _, patch = osb
    m = patch(oigpp.igevpp().cuda())
    xg = {k: v.cuda() for k, v in _x(1, 256, 512, 80).items()}
    with torch.no_grad():
        m(dict(xg))
        ops.profile_start()
        before = lib.launch_count()
        m(dict(xg))
        n = lib.launch_count() - before
        prof = ops.profile_stop()
    counts = {k: len(v) for k, v in prof.items()}
    print("patch(IGEV++) 256x512: %d launches %s" % (n, counts))
    assert counts["osb_geo_multirange_lookup_fwd"] == 32 and counts["osb_conv2d_k3_tc_gru_fwd"] == 32 * 18
    assert counts["osb_gwc_volume_fwd"] == 1 and counts["osb_softargmin_fwd"] == 3 and counts["osb_context_upsample_fwd"] == 1
    assert counts["osb_avgpool_pairs_fwd"] == 2 and counts["osb_dwconv2d_fwd"] == 32
    assert counts["osb_conv3d_1x1_bn_act_fwd"] == 32 * 4                  # convg1 x 3, convc1
    assert n == sum(counts.values())


@pytest.mark.parametrize("yaml", ["uniform", "amp"])
def test_whole_model_against_unpatched(osb, yaml):
    """256x512 through the reference class and patch().  fp32 (uniform YAML): within max(10 x the reference's GPU-vs-CPU floor,
    1e-2) px of the unpatched model on GPU and CPU.  AMP YAML: within twice the unpatched AMP model's own distance to the fp32 CPU
    reference."""
    lib, ops, _, patch = osb
    path = oigpp.UNIFORM_YAML if yaml == "uniform" else oigpp.AMP_YAML
    x = _x(1, 256, 512, 81)
    xg = {k: v.cuda() for k, v in x.items()}
    with torch.no_grad():
        want_cpu = oigpp.igevpp()(dict(x))["disp_pred"]
        if yaml == "uniform":
            m = oigpp.igevpp().cuda()
            want_gpu = m(dict(xg))["disp_pred"]
            got = patch(m)(dict(xg))["disp_pred"]
            e_gpu = (got - want_gpu).abs().mean().item()
            e_cpu = (got.cpu() - want_cpu).abs().mean().item()
            floor = (want_gpu.cpu() - want_cpu).abs().mean().item()
            print("patch(IGEV++) 256x512: EPE %.3e vs GPU ref, %.3e vs CPU ref (floor %.3e)" % (e_gpu, e_cpu, floor))
            assert got.dtype == torch.float32 and want_cpu.std() > 1.0
            assert e_gpu <= max(10 * floor, 1e-2) and e_cpu <= max(10 * floor, 1e-2)
        else:
            amp = oigpp.igevpp(path).cuda()(dict(xg))["disp_pred"]
            got = patch(oigpp.igevpp(path).cuda())(dict(xg))["disp_pred"]
            e_amp = (amp.cpu() - want_cpu).abs().mean().item()
            e_got = (got.cpu() - want_cpu).abs().mean().item()
            print("patch(IGEV++, AMP YAML) 256x512: EPE %.3e vs fp32 CPU (unpatched AMP %.3e)" % (e_got, e_amp))
            assert got.dtype == amp.dtype and e_got <= max(2 * e_amp, 1e-2)
    assert torch.isfinite(got).all() and got.shape == want_cpu.shape


def test_patch_is_per_instance_and_refuses_training(osb):
    lib, _, _, patch = osb
    a, b = patch(oigpp.igevpp(seed=9).cuda()), oigpp.igevpp(seed=9).cuda()
    for m in (a, b):
        m.args.VALID_ITERS = 4
    xg = {k: v.cuda() for k, v in _x(1, 64, 128, 82).items()}
    with torch.no_grad():
        before = lib.launch_count()
        out_b = b(dict(xg))["disp_pred"]
        assert lib.launch_count() == before                             # the unpatched instance runs nothing of this library
        out_a = a(dict(xg))["disp_pred"]
        assert lib.launch_count() > before
    assert (out_a - out_b).abs().mean().item() <= 1e-2
    with pytest.raises(RuntimeError, match="CUDA inference only"):
        a(dict(xg))                                                     # autograd recording through the parameters
    a.train()
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA inference only"):
        a(dict(xg))
    c = patch(oigpp.igevpp(seed=9).cuda(), strict=False).train()
    c.args.TRAIN_ITERS = 2
    before = lib.launch_count()
    out = c(dict(xg))
    assert lib.launch_count() == before
    out["disp_pred"].mean().backward()
    assert c.update_block.geo_encoder0.convg2.weight.grad is not None and c.update_block.encoder.conv.weight.grad is not None
