"""GPU: CFNet on the library (openstereo_b200/cfnet.py) and the two runtime modes it adds.

* Mish: every CUDA-core registry row of the k3, stride-2, transposed-k3 / k4 and 1x1 paths (tests/test_cuda_core_contract_gpu.py,
  imported read-only) re-run with act = OSB_ACT_MISH against fp64 conv + BN (+ residual) + Mish (+ gate) from the same fp32 inputs:
  error per output channel <= 1e-5 x the channel's max sum |terms| plus four ulp of Mish, both store paths, output inside
  NaN-filled regions between sentinels, determinism; the instance-norm, tensor-core, 2D and channels-last entry points refuse 6.
* The variance mode of the soft-argmin (osb_softargmin_var_fwd) is a row family of tests/test_kernel_contract_gpu.py ("var"), as
  are the unmasked warped volume at fractional samples (the cas rows with mask = 0) and both entry points' refusals.
* The warped volume with the left copy unmasked at CFNet's integer samples against the reference's SpatialTransformer +
  groupwise_correlation_4D + cat, and bit-identical to osb_warped_gwc_concat_volume_fwd with mask_left = 1.
* Each engine stage and the whole patched model against the reference (cuDNN fp32, TF32 off), and the guard.
"""
import re

import pytest
import torch
import torch.nn.functional as F

import test_cuda_core_contract_gpu as cc

pytestmark = pytest.mark.gpu

ACT_MISH = 6
ULP4 = 4 * 2.0 ** -24


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, ops
    return _lib, ops


@pytest.fixture(autouse=True)
def _fp32_reference():
    """cuDNN fp32 (TF32 off) with deterministic algorithms: the unpatched model is then the same from run to run, so the counts of
    the whole-model test (pixels whose .long() truncation falls the other way) do not move with cuDNN's algorithm choice."""
    cudnn, matmul = torch.backends.cudnn, torch.backends.cuda.matmul
    old = cudnn.allow_tf32, matmul.allow_tf32, cudnn.deterministic, cudnn.benchmark
    cudnn.allow_tf32 = matmul.allow_tf32 = False
    cudnn.deterministic, cudnn.benchmark = True, False
    yield
    cudnn.allow_tf32, matmul.allow_tf32, cudnn.deterministic, cudnn.benchmark = old


def mish64(x):
    from oracle.cfnet import mish64 as m
    return m(x)


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------------------------------ Mish
MISH_ROWS = [r for r in cc.REGISTRY if r.fam in ("k3", "dc", "pw")]


def mish_case(osb, row, g):
    """The registry row's launch with act = OSB_ACT_MISH: fp64 want = Mish(conv * sc + sh + res) * gate, mag = sum |terms|."""
    lib, ops = osb
    o, ep = row.opts, row.opts.get("ep", "").split()
    b, d, h, w = row.shape
    cs = cc.channel_scales(row.cout, g)
    x = torch.randn(b, row.cin, d, h, w, generator=g)
    if row.fam == "k3":
        st = o["stride"]
        wt = torch.randn(row.cout, row.cin, 3, 3, 3, generator=g) * (27 * row.cin) ** -0.5 * cs.view(-1, 1, 1, 1, 1)
        op = lambda a, k: F.conv3d(a, k, stride=st, padding=1)                          # noqa: E731
        wp = ops.pack_conv_weight(wt).cuda()
    elif row.fam == "dc":
        k = o["k"]
        wt = torch.randn(row.cin, row.cout, k, k, k, generator=g) * (row.cin * k ** 3 / 8) ** -0.5 * cs.view(1, -1, 1, 1, 1)
        op = lambda a, kk: F.conv_transpose3d(a, kk, stride=2, padding=1, output_padding=1 if k == 3 else 0)   # noqa: E731
        wp = ops.pack_deconv_weight(wt).cuda()
    else:
        wt = torch.randn(row.cin, row.cout, generator=g) * row.cin ** -0.5 * cs.view(1, -1)
        op = lambda a, kk: torch.einsum("bcdhw,co->bodhw", a, kk)                      # noqa: E731
        wp = wt.float().contiguous().cuda()
    conv = op(x.double(), wt.double())
    sc, sh, res = cc.epilogue_operands(row, g, conv.shape, 1, cs)
    gate = None
    if "gate" in ep:
        gate = torch.sigmoid(torch.randn(b, row.cout, conv.shape[3], conv.shape[4], generator=g))
    pre = cc.ref_epilogue(conv, 1, sc, sh, res, cc.ACT_NONE)
    want = mish64(pre) if gate is None else mish64(pre) * gate.double().unsqueeze(2)
    mag = cc.saturated_magnitude(op(x.double().abs(), wt.double().abs()), 1, sc, sh, res, cc.ACT_RELU6)   # sum |terms|
    dev = lambda t: None if t is None else t.float().contiguous().cuda()                # noqa: E731
    xd, scd, shd = dev(x), dev(sc), dev(sh)
    call = lib.call
    if row.fam == "k3":
        fn = lambda y, r, gt: call("osb_conv3d_k3_bn_act_fwd", xd.data_ptr(), wp.data_ptr(), cc.ptr(scd), cc.ptr(shd), r, gt, y, b,  # noqa
                                   row.cin, row.cout, d, h, w, st, ACT_MISH, _stream())
    elif row.fam == "dc":
        fn = lambda y, r, gt: call("osb_deconv3d_bn_act_fwd", xd.data_ptr(), wp.data_ptr(), cc.ptr(scd), cc.ptr(shd), r, y, b,  # noqa
                                   row.cin, row.cout, d, h, w, k, ACT_MISH, _stream())
    else:
        c0 = o.get("c0", row.cin)
        x0, x1 = dev(x[:, :c0]), dev(x[:, c0:]) if c0 < row.cin else None
        fn = lambda y, r, gt: call("osb_conv3d_1x1_bn_act_fwd", x0.data_ptr(), cc.ptr(x1), c0, wp.data_ptr(), cc.ptr(scd),  # noqa
                                   cc.ptr(shd), r, gt, y, b, row.cin, row.cout, d, h, w, ACT_MISH, 0, _stream())
    return cc.Case(row.id + " mish", want, 1, fn, res, gate, mag), pre


@pytest.mark.parametrize("row", MISH_ROWS, ids=[r.id for r in MISH_ROWS])
def test_mish_epilogue(osb, row):
    case, pre = mish_case(osb, row, cc.seed(row, salt=606))
    if row.cout >= 8:                                            # the per-channel scales span 2^-12 .. 2^12
        assert (pre.abs() > 20).any() and (pre.abs() < 1e-2).any(), "the row must reach softplus's threshold and the origin"
    first = None
    runs = [{}, {}, {"y_off": 1}] + ([{"res_off": 1}] if case.res is not None else []) + ([{"gate_off": 1}] if case.gate is not None else [])
    for offs in runs:
        buf, lead = case.launch(**offs)
        case.check_bounds(buf, lead, "%s %s" % (case.name, offs))
        inner = buf[lead:lead + case.numel]
        ratio = case.channel_ratio(inner)
        assert float(ratio.max()) <= cc.TOL + ULP4, "%s %s: err / max sum|terms| %g" % (case.name, offs, float(ratio.max()))
        bits = inner.view(torch.int32).clone()
        if first is None:
            first = bits
        else:
            assert torch.equal(first, bits), "%s %s: not bit-identical to the first run" % (case.name, offs)


def test_mish_refused_elsewhere(osb):
    """Every entry point without the Mish epilogue refuses act = 6 as an argument error, before any launch."""
    lib, _ = osb
    buf = torch.zeros(1 << 22, device="cuda")
    p = buf.data_ptr()
    s = _stream()
    calls = {
        "osb_conv3d_k3_in_fwd": (p, p, None, None, None, None, p, None, None, 0, 1, 8, 8, 2, 4, 32, 1, ACT_MISH, s),
        "osb_deconv3d_in_fwd": (p, p, None, None, None, None, p, None, None, 0, 1, 8, 8, 2, 4, 32, 3, ACT_MISH, s),
        "osb_conv3d_1x1_in_fwd": (p, None, 8, p, None, None, None, None, None, None, p, None, None, 0, 1, 8, 8, 2, 4, 32, ACT_MISH, 0, s),
        "osb_conv3d_k3_tc_fwd": (p, p, p, None, None, p, 1, 32, 32, 2, 4, 128, ACT_MISH, 1, 1, s),
        "osb_conv3d_k3_s2_tc_fwd": (p, p, p, None, None, p, 1, 32, 64, 2, 4, 128, ACT_MISH, 1, 1, s),
        "osb_deconv3d_k3_tc_fwd": (p, p, p, None, None, p, 1, 64, 32, 2, 4, 64, ACT_MISH, 1, 1, s),
        "osb_conv2d_k3_tc_fwd": (p, p, p, None, None, p, 1, 32, 64, 4, 128, 1, ACT_MISH, 1, 1, s),
        "osb_dwconv2d_fwd": (p, p, None, None, None, p, 1, 8, 8, 16, 3, 3, 1, ACT_MISH, s),
        "osb_deconv2d_k3s2_fwd": (p, p, None, None, None, p, 1, 8, 8, 8, 16, ACT_MISH, s),
        "osb_conv1x1_ndhwc_fwd": (p, p, None, None, p, 64, 32, 32, ACT_MISH, s),
        "osb_conv1x1_ndhwc_cat_fwd": (p, p, 64, 64, p, None, None, p, 128, 64, ACT_MISH, s),
    }
    for name, args in calls.items():
        before = lib.launch_count()
        with pytest.raises(ValueError, match="activation"):
            lib.call(name, *args)
        assert lib.launch_count() == before, name


# --------------------------------------------------------------------------------------------------------------- warped volume
def _reference_module():
    from oracle.cfnet import reference_module
    return reference_module()


def test_warped_volume_mask_left_one_is_the_cascade_entry_point(osb):
    lib, _ = osb
    g = torch.Generator().manual_seed(7)
    b, cg, gr, cc_, d, h, w = 2, 40, 10, 12, 5, 6, 45
    xg, yg = torch.randn(b, cg, h, w, generator=g).cuda(), torch.randn(b, cg, h, w, generator=g).cuda()
    xc, yc = torch.randn(b, cc_, h, w, generator=g).cuda(), torch.randn(b, cc_, h, w, generator=g).cuda()
    disp = (torch.rand(b, d, h, w, generator=g) * (w + 8) - 4).cuda()
    outs = []
    for name, extra in (("osb_warped_gwc_concat_volume_fwd", ()), ("osb_warped_gwc_concat_volume_ex_fwd", (1,))):
        out = torch.full((b, gr + 2 * cc_, d, h, w), float("nan"), device="cuda")
        lib.call(name, xg.data_ptr(), yg.data_ptr(), xc.data_ptr(), yc.data_ptr(), disp.data_ptr(), out.data_ptr(), b, cg, gr, cc_, d,
                 h, w, *extra, _stream())
        outs.append(out.view(torch.int32))
    assert torch.equal(outs[0], outs[1])
    before = lib.launch_count()
    with pytest.raises(ValueError):
        lib.call("osb_warped_gwc_concat_volume_ex_fwd", xg.data_ptr(), yg.data_ptr(), xc.data_ptr(), yc.data_ptr(), disp.data_ptr(),
                 outs[0].data_ptr(), b, cg, gr, cc_, d, h, w, 2, _stream())
    assert lib.launch_count() == before


def _roundtrip32(v, size):
    """The kernel's coordinate round trip (v / ((size - 1) / 2) - 1, then (g + 1) * ((size - 1) / 2)) in IEEE fp32."""
    half = torch.tensor((size - 1.0) / 2.0, dtype=torch.float32)
    return ((v / half) - 1 + 1) * half


# (B, Cg, G, Cc, D, H, W): CFNet's s3 / s2 layouts; H = 64 and 128 have rows whose round trip leaves the integer (15 and 21 of them)
@pytest.mark.parametrize("shape", [(2, 80, 20, 6, 12, 9, 64), (1, 160, 40, 12, 16, 64, 240), (1, 80, 20, 6, 12, 128, 480)])
def test_warped_volume_at_integer_samples(osb, shape):
    """mask_left = 0 at integer samples (past both edges included) against the reference's SpatialTransformer (exact gather,
    zeros outside [0, W - 1]) + groupwise_correlation_4D + cat.  The kernel samples bilinearly at the round-tripped coordinates,
    which land within 2^-23 (W - 1) of the integer column and 2^-23 (H - 1) of the integer row, so each warped feature is a convex
    combination of its 2x2 cell in which the taps other than the exact one weigh at most 2^-23 (W - 1 + H - 1): it is within that
    fraction of the largest difference between the exact tap and a feature of its 3x3 neighbourhood (zeros outside the image)."""
    _, ops = osb
    mod = _reference_module()
    b, cg, gr, cc_, d, h, w = shape
    rows = torch.arange(h, dtype=torch.float32)
    off_rows = int((_roundtrip32(rows, h) != rows).sum())
    assert off_rows == 0 or h >= 64
    if h >= 64:
        assert off_rows > 0, "the case must exercise rows whose round trip leaves the integer"
    g = torch.Generator().manual_seed(sum(shape))
    xg, yg = torch.randn(b, cg, h, w, generator=g).cuda(), torch.randn(b, cg, h, w, generator=g).cuda()
    xc, yc = torch.randn(b, cc_, h, w, generator=g).cuda(), torch.randn(b, cc_, h, w, generator=g).cuda()
    cols = torch.arange(w).view(1, 1, 1, w)
    target = torch.randint(-3, w + 3, (b, d, h, w), generator=g)     # the column each sample reads, past both edges
    samples = (cols - target).float().cuda()
    with torch.no_grad():
        got = ops.warped_gwc_concat_volume(xg, yg, xc, yc, samples, gr, mask_left=False)
        st = mod.SpatialTransformer()
        rc, lc = st(xc, yc, samples)
        rg, lg = st(xg, yg, samples)
        want = torch.cat((mod.groupwise_correlation_4D(lg, rg, gr), lc, rc), dim=1)
    # left copy: exact
    assert torch.equal(got[:, gr:gr + cc_], want[:, gr:gr + cc_])
    frac = 2.0 ** -23 * ((w - 1) + (h - 1))
    idx = (target.clamp(-2, w + 1) + 2).cuda()

    def nb_diff(y):
        """max |y[h + dy, t + dx] - y[h, t]| over the 3x3 neighbourhood of the gathered (row, column t), zeros outside the image,
        (B, C, D, H, W)."""
        yp = F.pad(y, (3, 3, 1, 1))
        centre = yp[:, :, 1:1 + h, 1:1 + w + 4]
        m = torch.zeros_like(centre)
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                m = torch.maximum(m, (yp[:, :, 1 + dy:1 + dy + h, 1 + dx:1 + dx + w + 4] - centre).abs())
        i5 = idx.unsqueeze(1).expand(-1, y.shape[1], -1, -1, -1)
        return torch.gather(m.unsqueeze(2).expand(-1, -1, d, -1, -1), 4, i5)

    ulp4 = 4 * 2.0 ** -24
    r_got, r_want = got[:, gr + cc_:], want[:, gr + cc_:]
    nbc = nb_diff(yc)
    bound = frac * nbc + ulp4 * (r_want.abs() + nbc)
    dev = (r_got - r_want).abs()
    assert bool((dev <= bound).all()), float((dev / bound.clamp(min=1e-30)).max())
    kk = cg // gr
    nbg = nb_diff(yg)
    tol_r = frac * nbg + ulp4 * (rg.abs() + nbg)
    lgv = lg.reshape(b, gr, kk, d, h, w)
    gbound = (lgv.abs() * tol_r.reshape(b, gr, kk, d, h, w)).mean(2) + 2 * ulp4 * (lgv * rg.reshape(b, gr, kk, d, h, w)).abs().mean(2)
    gdev = (got[:, :gr] - want[:, :gr]).abs()
    assert bool((gdev <= gbound).all()), float((gdev / gbound.clamp(min=1e-30)).max())
    print("\nH=%d (%d rows off the integer) W=%d: largest deviation of a warped feature %.3g (%.3g of its largest 3x3 neighbour "
          "difference); gwc %.3g" % (h, off_rows, w, float(dev.max()), float((dev / nbc.clamp(min=1e-30)).max()), float(gdev.max())))


# ------------------------------------------------------------------------------------------------------------- model / stages
@pytest.fixture(scope="module")
def models(osb):
    from oracle.cfnet import reference_model
    ref = reference_model().cuda()
    pat = reference_model().cuda()
    from openstereo_b200.patch import patch
    patch(pat)
    return ref, pat


def _pair(b, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    return {"left": torch.randn(b, 3, h, w, generator=g).cuda(), "right": torch.randn(b, 3, h, w, generator=g).cuda()}


class _SampleRecorder:
    """Records every generate_disparity_samples call of a model instance: the pre-truncation values and the integer samples."""

    def __init__(self, model):
        self.calls, self.model = [], model
        orig = model.generate_disparity_samples

        def rec(lo, hi, n=12):
            pre = torch.cat((torch.floor(lo), model.uniform_sampler(lo, hi, n), torch.ceil(hi)), dim=1)
            out = orig(lo, hi, n)
            self.calls.append((pre, out))
            return out
        model.generate_disparity_samples = rec

    def close(self):
        del self.model.generate_disparity_samples


def test_stages_against_the_reference(models):
    from openstereo_b200.cfnet import CFNetEngine
    ref, _ = models
    eng = CFNetEngine(ref)
    data = _pair(2, 256, 512, seed=3)
    m = ref
    with torch.no_grad():
        fl, fr = m.feature_extraction(data["left"]), m.feature_extraction(data["right"])
        eng._ensure(data["left"].device)
        vols = eng.volumes(fl, fr)
        for v, s in zip(vols, (4, 5, 6)):
            mod = _reference_module()
            want = torch.cat((mod.build_gwc_volume(fl["gw%d" % s], fr["gw%d" % s], m.maxdisp // 2 ** (s - 1), m.num_groups),
                              mod.build_concat_volume(fl["concat_feature%d" % s], fr["concat_feature%d" % s], m.maxdisp // 2 ** (s - 1))), 1)
            assert float((v - want).abs().max()) <= 1e-5 * float(want.abs().max())
        pred, std = eng.stage1(*vols)
        mod = _reference_module()
        c4 = m.dres0(vols[0]); c4 = m.dres1(c4) + c4
        c5 = m.dres0_5(vols[1]); c5 = m.dres1_5(c5) + c5
        c6 = m.dres0_6(vols[2]); c6 = m.dres1_6(c6) + c6
        cost = m.classif2(m.dres3(m.combine1(c4, c5, c6))).squeeze(1)
        p = F.softmax(cost, dim=1)
        want = mod.disparity_regression(p, m.maxdisp // 8).unsqueeze(1)
        want_std = mod.disparity_variance(p, m.maxdisp // 8, want).sqrt()
        assert float((pred - want).abs().max()) <= 1e-3 and float((pred - want).abs().mean()) <= 1e-4
        assert float((std - want_std).abs().mean()) <= 1e-4
        # s3 and s2 from the same samples
        for level, stage, groups, size in ((3, "s3", m.num_groups, 4), (2, "s2", m.num_groups // 2, 2)):
            d = m.sample_count_s3 if stage == "s3" else m.sample_count_s2
            lo = (torch.rand(2, 1, 256 // size, 512 // size, generator=torch.Generator().manual_seed(level)) * 100).cuda()
            samples = m.generate_disparity_samples(lo, lo + 20, d).float()
            got, got_std = eng.refine(fl, fr, samples, level, stage, groups, True)
            vc, _ = m.cost_volume_generator(fl["concat_feature%d" % level], fr["concat_feature%d" % level], samples, "concat")
            vg, sm = m.cost_volume_generator(fl["gw%d" % level], fr["gw%d" % level], samples, "gwc", groups)
            c0 = getattr(m, "confidence0_" + stage)(torch.cat((vg, vc, sm), 1))
            c0 = getattr(m, "confidence1_" + stage)(c0) + c0
            out2 = getattr(m, "confidence3_" + stage)(getattr(m, "confidence2_" + stage)(c0))
            p = F.softmax(getattr(m, "confidence_classif1_" + stage)(out2).squeeze(1), dim=1)
            want = torch.sum(p * samples, dim=1, keepdim=True)
            want_std = mod.disparity_variance_confidence(p, samples, want).sqrt()
            err = (got - want).abs()
            print("\n%s: max |pred - ref| %.3g px, mean %.3g" % (stage, float(err.max()), float(err.mean())))
            assert float(err.max()) <= 1e-2 and float(err.mean()) <= 1e-4
            assert float((got_std - want_std).abs().mean()) <= 1e-4


@pytest.mark.parametrize("hw", [(256, 512), (512, 960)])
def test_whole_model(models, hw):
    ref, pat = models
    data = _pair(2, *hw, seed=hw[0])
    recs = [_SampleRecorder(ref), _SampleRecorder(pat)]
    try:
        with torch.no_grad():
            want = ref(data)["disp_pred"]
            got = pat(data)["disp_pred"]
    finally:
        for r in recs:
            r.close()
    assert got.shape == want.shape == (2,) + hw and got.dtype == want.dtype
    epe = float((got - want).abs().mean())
    assert want.std() > 1.0
    stats, pixels, near = [], [], []
    for (pre, ref_s), (_, got_s) in zip(recs[0].calls, recs[1].calls):
        differ = (ref_s != got_s)
        dist = (pre - pre.round()).abs()
        pix = differ.any(1)
        pixels.append(pix)
        near.append((differ & (dist > 3e-4)).any(1) == 0)
        stats.append((int(pix.sum()), float(pix.float().mean()), float(dist[differ].max()) if differ.any() else 0.0))
    assert len(stats) == 2
    # s2 pixels whose samples differ although no sample's reference value lies near an integer: their distance (s2 pixels,
    # Chebyshev) to the nearest s3 pixel whose samples differed, whose different hypotheses the s3 aggregation carried to them
    far = (pixels[1] & ~near[1]).nonzero()
    s3_at = pixels[0].nonzero()
    reach = 0
    for bb, y, x in far.tolist():
        src = s3_at[s3_at[:, 0] == bb]
        assert len(src), "s2 samples differ away from an integer in an image whose s3 samples all agree"
        reach = max(reach, int(torch.maximum((2 * src[:, 1] - y).abs(), (2 * src[:, 2] - x).abs()).min()))
    print("\n%dx%d: EPE %.3g px; s3 / s2 samples differing at (pixels, share, largest distance of the reference's value from an "
          "integer there): %s; s2 pixels away from an integer lie within %d px of an s3 one" % (hw + (epe, stats, reach)))
    assert epe <= 1e-3
    # .long() truncation (DESIGN.md section 4.22): s3's samples differ only where the reference's value lies within stage 1's noise
    # of an integer (measured: at most 2.5e-4 from one, at 2.6e-4 .. 4.3e-4 of the pixels); s2's differ where its own value lies
    # that near an integer or next to an s3 pixel whose hypotheses differed
    assert stats[0][2] <= 3e-4, "s3 samples differ where the reference's value is not near an integer"
    assert stats[0][1] <= 6e-4 and stats[1][1] <= 6e-4
    assert reach <= 32, "s2 samples differ away from an integer and away from every s3 difference"


def test_guard(osb):
    from oracle.cfnet import reference_model
    from openstereo_b200.patch import patch
    data = _pair(1, 128, 256, seed=5)
    # training mode (its forward updates the BN statistics: separate instances)
    strict_t, loose_t = patch(reference_model().cuda().train()), patch(reference_model().cuda().train(), strict=False)
    with pytest.raises(RuntimeError, match="CUDA inference only"):
        strict_t(data)
    out = loose_t(data)
    assert isinstance(out, list) and len(out) == 9
    sum(o.mean() for o in out).backward()
    assert loose_t.classif2[2].weight.grad is not None and loose_t.confidence_classif1_s2[2].weight.grad is not None
    strict, loose = patch(reference_model().cuda()), patch(reference_model().cuda(), strict=False)
    unpatched = reference_model().cuda()
    # a recording autograd graph in eval mode
    rec = {k: v.clone().requires_grad_(True) for k, v in data.items()}
    with pytest.raises(RuntimeError, match="CUDA inference only"):
        strict(rec)
    d = loose(rec)["disp_pred"]
    assert d.grad_fn is not None
    with torch.no_grad():
        assert float((d.detach() - unpatched(data)["disp_pred"]).abs().max()) <= 1e-3
    # CPU calls: strict refuses; non-strict hands the call to the reference, which behaves exactly as unpatched
    cpu = {k: v.cpu() for k, v in data.items()}
    strict_cpu, loose_cpu, unpatched_cpu = (m.cpu() for m in (strict, loose, unpatched))
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="CUDA inference only"):
            strict_cpu(cpu)
        try:
            want = unpatched_cpu(cpu)
        except Exception as exc:                                   # the reference's own CPU behaviour (get_device() = -1)
            with pytest.raises(type(exc), match=re.escape(str(exc))):
                loose_cpu(cpu)
        else:
            assert torch.equal(loose_cpu(cpu)["disp_pred"], want["disp_pred"])
