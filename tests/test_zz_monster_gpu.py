"""GPU: MonSter on the library -- the disparity-warp mode of warped_volume_kernel against the reference's disp_warp (bit for bit,
store bounds inside sentinels, one launch, determinism, refusals that launch nothing), CasStereo's volume modes keeping their bits
around warp launches, MixMotionEncoderEngine against its module in float64 (the fp16-range guard, re-packing, bf16 autocast dtypes),
the patched forward's launch sequence, the whole model under both YAMLs against the unpatched model, and the training / autograd
refusal.  Sorted after the torch.profiler routing suites like the other model-level files."""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from oracle import _reference_shim as shim
from oracle import monster as omon

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


# ------------------------------------------------------------------------------------------ the disparity warp
def _warp_case(b, c, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    img = torch.randn(b, c, h, w, generator=g)
    disp = torch.rand(b, 1, h, w, generator=g) * (w + 16) - 8                 # negative, and beyond both edges
    disp[0, 0, 0, :4] = torch.tensor([0.0, -3.25, w + 5.5, 1.0])[:w]
    disp[-1, 0, -1, -2:] = torch.tensor([0.0, 2.0 * w])
    return img, disp


WARP_CASES = [(2, 5, 2, 17), (1, 3, 64, 131), (3, 96, 64, 128), (2, 9, 2, 9), (4, 16, 64, 33), (1, 96, 2, 128)]


def _guarded(n):
    pad = 64
    buf = torch.full((n + 2 * pad,), 12345.0, device="cuda")
    buf[pad:pad + n] = float("nan")
    return buf, buf[pad:pad + n], pad


@pytest.mark.parametrize("case", WARP_CASES, ids=lambda c: "x".join(map(str, c)))
def test_disp_warp_against_reference(osb, case):
    """Bit for bit the reference's disp_warp(img, disp)[0] on the CPU, one launch, deterministic, every store inside the output."""
    lib, ops, _, _ = osb
    warp = omon.load_reference("stereo.modeling.models.monster.warp")
    img, disp = _warp_case(*case, seed=sum(case))
    want = warp.disp_warp(img, disp.clone())[0]
    ig, dg = img.cuda(), disp.cuda()
    before = lib.launch_count()
    got = ops.disp_warp(ig, dg)
    assert lib.launch_count() == before + 1
    assert got.shape == img.shape and got.dtype == torch.float32
    assert torch.equal(got.cpu(), want)
    assert torch.equal(ops.disp_warp(ig, dg), got)
    buf, y, pad = _guarded(img.numel())
    lib.call("osb_disp_warp_fwd", ig.data_ptr(), dg.data_ptr(), y.data_ptr(), *case, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert bool((buf[:pad] == 12345.0).all() and (buf[pad + y.numel():] == 12345.0).all())
    assert torch.equal(y.view_as(got), got)


def test_disp_warp_refusals_launch_nothing(osb):
    lib, ops, _, _ = osb
    img, disp = torch.zeros(1, 4, 1, 16, device="cuda"), torch.zeros(1, 1, 1, 16, device="cuda")
    out = torch.zeros(1, 4, 1, 16, device="cuda")
    before = lib.launch_count()
    for b, c, h, w in ((1, 4, 1, 16), (1, 4, 2, 1), (0, 4, 2, 16), (1, 0, 2, 16)):
        with pytest.raises(ValueError):
            lib.call("osb_disp_warp_fwd", img.data_ptr(), disp.data_ptr(), out.data_ptr(), b, c, h, w, None)
    with pytest.raises(ValueError, match="do not match"):
        ops.disp_warp(img, torch.zeros(1, 2, 1, 16, device="cuda"))
    assert lib.launch_count() == before


def test_disp_warp_bf16_returns_the_input_dtype(osb):
    """bf16 features and disparities (the AMP YAML's): the kernel samples in fp32 and returns bf16, bit for bit the reference's
    warp of the same values in fp32 rounded to bf16.  The reference itself builds the grid in bf16 (meshgrid type_as(img)), so its
    own bf16 output differs by bf16's coordinate rounding; that distance is printed, not asserted."""
    _, ops, _, _ = osb
    warp = omon.load_reference("stereo.modeling.models.monster.warp")
    img, disp = _warp_case(2, 8, 16, 128, 5)
    img, disp = img.bfloat16(), disp.bfloat16()
    got = ops.disp_warp(img.cuda(), disp.cuda())
    want_bf16 = warp.disp_warp(img, disp.clone())[0]
    assert got.dtype == want_bf16.dtype == torch.bfloat16
    assert torch.equal(got.cpu(), warp.disp_warp(img.float(), disp.float())[0].bfloat16())
    print("disp_warp bf16: mean |kernel - reference's bf16 grid| %.3e" % (got.cpu().float() - want_bf16.float()).abs().mean().item())


def test_cascade_modes_keep_their_bits_around_warp_calls(osb):
    """CasPSMNet's and CasGwcNet's volumes (both mask settings, 5 to 10 channels per group, an odd width) compute the same bits
    before and after disparity-warp launches of the same kernel instantiations in the same process."""
    _, ops, _, _ = osb
    g = torch.Generator().manual_seed(4)

    def rnd(*shape):
        return torch.randn(*shape, generator=g).cuda()
    b, h, w = 2, 5, 37
    x, y = rnd(b, 12, h, w), rnd(b, 12, h, w)
    xg, yg = rnd(b, 40, h, w), rnd(b, 40, h, w)
    disp = (torch.rand(b, 6, h, w, generator=g) * 50 - 8).cuda()

    def run():
        return [ops.warped_concat_volume(x, y, disp, mask_left=m) for m in (False, True)] + \
               [ops.warped_gwc_concat_volume(xg, yg, x, y, disp, G) for G in (8, 4, 5)]
    first = run()
    for c in (5, 96):
        ops.disp_warp(rnd(b, c, h, w), disp[:, :1].contiguous())
    second = run()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(first, second))


# ------------------------------------------------------------------------------------------ MixMotionEncoderEngine
def _mix2(seed):
    from types import SimpleNamespace
    torch.manual_seed(seed)
    m = omon.load_reference("stereo.modeling.models.monster.update")
    return m.BasicMotionEncoder_mix2(SimpleNamespace(corr_levels=2, corr_radius=4)).eval()


def _enc_inputs(b, h, w, seed):
    """(disp, corr, flaw, disp_mono, corr_mono, flaw_mono): disparities in 0..48, lookup-like corr, feature differences."""
    g = torch.Generator().manual_seed(seed)
    return tuple(t.cuda() for t in (torch.rand(b, 1, h, w, generator=g) * 48, torch.randn(b, 162, h, w, generator=g),
                                    torch.randn(b, 96, h, w, generator=g), torch.rand(b, 1, h, w, generator=g) * 48,
                                    torch.randn(b, 162, h, w, generator=g), torch.randn(b, 96, h, w, generator=g)))


def _absconv(x, conv):
    return F.conv2d(x, conv.weight.double().abs(), conv.bias.double().abs(), padding=conv.padding)


def _magnitude(enc, args):
    a = [t.cpu().double().abs() for t in args]
    out = []
    for sfx, (d, corr, flaw) in (("", (a[0], a[1], a[2])), ("_mono", (a[3], a[4], a[5]))):
        m = lambda n: getattr(enc, n + sfx)
        cor = _absconv(_absconv(torch.cat([corr, flaw], 1), m("convc1")), m("convc2"))
        dsp = _absconv(_absconv(d, m("convd1")), m("convd2"))
        out += [_absconv(torch.cat([cor, dsp], 1), m("conv")), d]
    return torch.cat(out, 1)


@pytest.mark.parametrize("w", [128, 160, 240])
def test_mix_encoder_against_reference_fp64(osb, w):
    _, ops, update, _ = osb
    enc = _mix2(w)
    args = _enc_inputs(2, 5, w, w + 1)
    with torch.no_grad():
        want = enc.double()(*[t.cpu().double() for t in args])
        mag = _magnitude(enc, args)
        eng = update.MixMotionEncoderEngine(enc.float().cuda())
        assert eng.serves(*args)
        got = eng(*args)
        torch.cuda.synchronize()
    assert got.shape == (2, 128, 5, w) and got.dtype == torch.float32 and torch.isfinite(got).all()
    err = (got.cpu().double() - want).abs()
    print("mix2 encoder W=%d: max err %.3e, max err / magnitude %.3e" % (w, err.max(), (err / mag).max()))
    assert (err <= TOL * mag + 1e-6).all()
    assert torch.equal(got[:, 63:64], args[0]) and torch.equal(got[:, 127:], args[3])     # the reference's cat, bit for bit
    assert ops.tc_overflow_count(reset=True) == 0


def test_mix_encoder_pad_channel_is_exact_zero(osb):
    """conv's 64th (pad) output channel computes exact zeros before disp is written over it."""
    _, ops, update, _ = osb
    eng = update.MixMotionEncoderEngine(_mix2(3).cuda())
    args = _enc_inputs(1, 4, 128, 2)
    with torch.no_grad():
        eng._ensure(args[0].device)
        zero = torch.zeros_like(args[0])
        for p, (d, corr, flaw) in zip(eng.w, (args[:3], args[3:])):
            out = eng._branch(p, zero, corr, flaw)
            assert torch.equal(out[:, 63], torch.zeros_like(out[:, 63])) and out[:, :63].abs().sum() > 0


def test_mix_encoder_launch_sequence(osb):
    """Per branch: the 1x1 over corr and flaw (two inputs, no concatenation), the depthwise 7x7, two channels-last packs and four
    Cout-64 wgmma launches; the two halves are joined by one torch.cat (not a library launch)."""
    lib, ops, update, _ = osb
    for w, variant in ((128, "tcg<64,16,128,1,1,0,0>"), (160, "tcg<64,16,128,1,1,1,0>")):
        eng = update.MixMotionEncoderEngine(_mix2(4).cuda())
        args = _enc_inputs(1, 4, w, 5)
        with torch.no_grad():
            eng(*args)
            ops.profile_start()
            before = lib.launch_count()
            eng(*args)
            n = lib.launch_count() - before
            prof = ops.profile_stop()
        assert n == 16
        assert {k: len(v) for k, v in prof.items()} == {"osb_conv3d_1x1_bn_act_fwd": 2, "osb_dwconv2d_fwd": 2,
                                                         "osb_ncdhw_to_ndhwc_slice": 4, "osb_conv2d_k3_tc_fwd": 8}
        assert ops.tc_last_variant() == variant


def test_mix_encoder_guard_and_repack(osb):
    _, ops, update, _ = osb
    enc = _mix2(6).cuda()
    eng = update.MixMotionEncoderEngine(enc)
    args = _enc_inputs(1, 4, 128, 7)
    ops.tc_overflow_count(reset=True)
    with torch.no_grad():
        eng(args[0], args[1] * 1e5, *args[2:])                             # convc1's output far beyond 4094
        torch.cuda.synchronize()
        with pytest.raises(RuntimeError, match="fp16 range"):
            eng(*args)
        torch.cuda.synchronize()
        assert ops.tc_overflow_count(reset=True) == 0
        before = eng(*args)
        enc.conv_mono.weight.mul_(0.5)                                      # a parameter changes in place: re-pack
        after = eng(*args)
        want = enc(*args)
    assert torch.equal(after[:, :64], before[:, :64]) and not torch.equal(after[:, 64:], before[:, 64:])
    assert (after - want).abs().max().item() <= 1e-3 * max(1.0, want.abs().max().item())


def test_mix_encoder_dtypes_under_bf16_autocast(osb):
    """Under the AMP YAML's bf16 autocast the engine computes in fp32 and returns the module's dtype (torch.cat's promotion of the
    bf16 convolutions with the fp32 disparities); fp16 autocast as well."""
    _, ops, update, _ = osb
    from openstereo_b200.patch import _override_engine
    ref, mine = _mix2(8).cuda(), _mix2(8).cuda()
    _override_engine(mine, update.MixMotionEncoderEngine(mine), True, "encoder")
    args = _enc_inputs(2, 6, 160, 9)
    with torch.no_grad():
        want32 = ref(*args)
        for dtype in (torch.bfloat16, torch.float16):
            with torch.autocast("cuda", dtype=dtype):
                want, got = ref(*args), mine(*args)
                wb, gb = ref(*[t.to(dtype) for t in args]), mine(*[t.to(dtype) for t in args])
            assert got.dtype == want.dtype and gb.dtype == wb.dtype == dtype
            assert (got.float() - want32).abs().max().item() <= 1e-3 * max(1.0, want32.abs().max().item())


# ------------------------------------------------------------------------------------------ the whole model
def _x(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return {"left": torch.rand(b, 3, h, w, generator=g) * 2 - 1, "right": torch.rand(b, 3, h, w, generator=g) * 2 - 1}


def _autocast(dtype):
    return torch.autocast("cuda", dtype=dtype) if dtype else contextlib.nullcontext()


def test_patched_forward_launch_count(osb):
    """256x512 (W' = 128), 32 iterations (25 of update_block, 7 of the two mix2 blocks): 39 lookups, 14 warps and 39 x 18 ConvGRU
    launches; 25 IGEV encoders (one 1x1 and one depthwise each) and 14 mix2 encoders (two of each); once per forward the gwc
    volume, the regression and the two pyramid levels, and 8 convex up-samplings (the 7 mono up-samplings and the last stereo one)."""
    lib, ops, _, patch = osb
    m = patch(omon.monster().cuda())
    xg = {k: v.cuda() for k, v in _x(1, 256, 512, 80).items()}
    with torch.no_grad():
        m(dict(xg))
        ops.profile_start()
        before = lib.launch_count()
        m(dict(xg))
        n = lib.launch_count() - before
        prof = ops.profile_stop()
    counts = {k: len(v) for k, v in prof.items()}
    print("patch(MonSter) 256x512: %d launches %s" % (n, counts))
    assert counts["osb_geo_lookup_fwd"] == 39 and counts["osb_disp_warp_fwd"] == 14
    assert counts["osb_conv2d_k3_tc_gru_fwd"] == 39 * 18
    assert counts["osb_conv3d_1x1_bn_act_fwd"] == 25 + 14 * 2 and counts["osb_dwconv2d_fwd"] == 25 + 14 * 2
    assert counts["osb_gwc_volume_fwd"] == 1 and counts["osb_softargmin_fwd"] == 1 and counts["osb_avgpool_pairs_fwd"] == 2
    assert counts["osb_context_upsample_fwd"] == 8
    # per update-block pass: 8 (IGEV encoder) or 16 (mix2 encoder) + 4 disp head + 1 mask head wgmma / CUDA-core launches
    assert counts["osb_conv2d_k3_tc_fwd"] == 25 * 4 + 14 * 8 + 39 * 3 and counts["osb_conv3d_k3_bn_act_fwd"] == 39 * 2
    assert n == sum(counts.values())


@pytest.mark.parametrize("yaml", ["uniform", "amp"])
def test_whole_model_against_unpatched(osb, yaml):
    """256x512 through the reference class and patch().  fp32 (uniform YAML): within max(10 x the reference's GPU-vs-CPU floor,
    1e-2) px of the unpatched model on GPU and CPU.  AMP YAML (bf16 autocast): within twice the unpatched AMP model's own distance to
    the fp32 CPU reference, with the reference's output dtype."""
    lib, ops, _, patch = osb
    x = _x(1, 256, 512, 81)
    xg = {k: v.cuda() for k, v in x.items()}
    with torch.no_grad():
        want_cpu = omon.monster()(dict(x))["disp_pred"]
        if yaml == "uniform":
            m = omon.monster().cuda()
            want_gpu = m(dict(xg))["disp_pred"]
            got = patch(m)(dict(xg))["disp_pred"]
            e_gpu = (got - want_gpu).abs().mean().item()
            e_cpu = (got.cpu() - want_cpu).abs().mean().item()
            floor = (want_gpu.cpu() - want_cpu).abs().mean().item()
            print("patch(MonSter) 256x512: EPE %.3e vs GPU ref, %.3e vs CPU ref (floor %.3e)" % (e_gpu, e_cpu, floor))
            assert got.dtype == torch.float32 and want_cpu.std() > 1.0
            assert e_gpu <= max(10 * floor, 1e-2) and e_cpu <= max(10 * floor, 1e-2)
        else:
            dtype = omon.amp_dtype(omon.AMP_YAML)
            with _autocast(dtype):
                amp = omon.monster(omon.AMP_YAML).cuda()(dict(xg))["disp_pred"]
                got = patch(omon.monster(omon.AMP_YAML).cuda())(dict(xg))["disp_pred"]
            e_amp = (amp.float().cpu() - want_cpu).abs().mean().item()
            e_got = (got.float().cpu() - want_cpu).abs().mean().item()
            print("patch(MonSter, AMP YAML, %s) 256x512: EPE %.3e vs fp32 CPU (unpatched AMP %.3e), dtype %s" % (dtype, e_got, e_amp,
                                                                                                            got.dtype))
            assert got.dtype == amp.dtype and e_got <= max(2 * e_amp, 1e-2)
    assert torch.isfinite(got).all() and got.shape == want_cpu.shape


def test_patch_is_per_instance_and_refuses_training(osb):
    lib, _, _, patch = osb
    a, b = patch(omon.monster(seed=9).cuda()), omon.monster(seed=9).cuda()
    for m in (a, b):
        m.args.valid_iters = 9
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
    c = patch(omon.monster(seed=9).cuda(), strict=False).train()
    c.args.train_iters = 9
    before = lib.launch_count()
    out = c(dict(xg))
    assert lib.launch_count() == before
    out["disp_pred"].mean().backward()
    blk = c.update_block_mix_stereo
    assert blk.encoder.conv.weight.grad is not None and blk.gru04.convz.weight.grad is not None
