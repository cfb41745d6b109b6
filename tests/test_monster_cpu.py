"""CPU: MonSter -- the oracle builds the reference class from both YAMLs, a numpy replay of the disparity-warp kernel's arithmetic
equals the reference's disp_warp bit for bit, the new C-ABI entry point's argument checks, MixMotionEncoderEngine's weight packing
and serves(), and patch()'s drop-in contract on the unmodified reference class (no compute on a GPU here)."""
import numpy as np
import pytest
import torch

from oracle import _reference_shim as shim
from oracle import monster as omon

needs_ref = pytest.mark.skipif(not shim.available(), reason="reference tree not present")
F32 = np.float32


def _inputs(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return {"left": torch.rand(b, 3, h, w, generator=g) * 2 - 1, "right": torch.rand(b, 3, h, w, generator=g) * 2 - 1}


@pytest.fixture(scope="module")
def native():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib
    return _lib


# ------------------------------------------------------------------------------------------ the warp's arithmetic, replayed
def _fma(a, b, c):
    """fp32 fused multiply-add: the product of two fp32 values is exact in the 64-bit long double significand."""
    return (a.astype(np.longdouble) * b + c).astype(F32)


def _coord(v, size):
    """csrc/cascade.cu border_roundtrip: normalize_coords, fmaf(g + 1, size / 2, -0.5), clamp to [0, size - 1]."""
    sm1 = F32(size - 1)
    g = (F32(2) * (v / sm1)).astype(F32) - F32(1)
    u = _fma(g + F32(1), np.full_like(g, F32(size) / F32(2)), np.full_like(g, F32(-0.5)))
    return np.minimum(np.maximum(u, F32(0)), sm1).astype(F32)


def replay_disp_warp(img, disp):
    """What warped_volume_kernel's disparity-warp mode computes, operation by operation, in numpy fp32."""
    b, c, h, w = img.shape
    out = np.zeros_like(img)
    cols = np.arange(w, dtype=F32)
    for bi in range(b):
        for y in range(h):
            iy = _coord(np.full(w, F32(y)), h)
            ix = _coord((cols - disp[bi, 0, y]).astype(F32), w)
            fx, fy = np.floor(ix), np.floor(iy)
            x0, y0 = fx.astype(np.int64), fy.astype(np.int64)
            wx = (ix - fx).astype(F32)
            e = (F32(1) - wx).astype(F32)
            n = (iy - fy).astype(F32)
            s = (F32(1) - n).astype(F32)
            for ci in range(c):
                plane = img[bi, ci]

                def tap(yy, xx):
                    ok = (yy < h) & (xx < w)
                    return np.where(ok, plane[np.minimum(yy, h - 1), np.minimum(xx, w - 1)], F32(0)).astype(F32)
                acc = (tap(y0, x0) * (s * e)).astype(F32)
                acc = _fma(tap(y0, x0 + 1), s * wx, acc)
                acc = _fma(tap(y0 + 1, x0), n * e, acc)
                out[bi, ci, y] = _fma(tap(y0 + 1, x0 + 1), n * wx, acc)
    return out


def warp_case(b, c, h, w, seed):
    """Seeded features and disparities with disp = 0, negative disp and disp beyond both edges in every case."""
    g = torch.Generator().manual_seed(seed)
    img = torch.randn(b, c, h, w, generator=g)
    disp = torch.rand(b, 1, h, w, generator=g) * (w + 16) - 8
    disp[0, 0, 0, :4] = torch.tensor([0.0, -3.25, w + 5.5, 1.0])[:w]
    disp[-1, 0, -1, -2:] = torch.tensor([0.0, 2.0 * w])
    return img, disp


WARP_CASES = [(2, 5, 2, 17), (1, 3, 64, 131), (2, 4, 7, 128), (3, 9, 2, 9)]


@needs_ref
@pytest.mark.parametrize("case", WARP_CASES, ids=lambda c: "x".join(map(str, c)))
def test_warp_replay_equals_reference(case):
    warp = omon.load_reference("stereo.modeling.models.monster.warp")
    img, disp = warp_case(*case, seed=sum(case))
    want = warp.disp_warp(img, disp.clone())[0]
    got = replay_disp_warp(img.numpy(), disp.numpy())
    assert np.array_equal(got, want.numpy())
    # the border clamp is exercised on both sides: columns whose sample lies left of 0 and right of W - 1
    assert (disp > torch.arange(case[3]).float()).any() and (torch.arange(case[3]).float() - disp > case[3] - 1).any()


# ------------------------------------------------------------------------------------------ host side
_P = 0x1000


@pytest.mark.parametrize("kw,match", [
    (dict(img=None), "null pointer"), (dict(disp=None), "null pointer"), (dict(out=None), "null pointer"),
    (dict(H=1), "H=1"), (dict(W=1), "W=1"), (dict(B=0), "empty shape"), (dict(C=0), "Cc=0"),
    (dict(W=1 << 20), "shared memory")])
def test_entry_point_argument_checks(native, kw, match):
    """Every refusal is an argument error raised before any CUDA call (the fake addresses are never touched)."""
    assert native.SIGNATURES["osb_disp_warp_fwd"] == [native._f32p] * 3 + [native._i] * 4 + [native._s]
    vals = dict(img=_P, disp=_P, out=_P, B=1, C=8, H=4, W=16, stream=None)
    vals.update(kw)
    with pytest.raises(ValueError, match=match):
        native.call("osb_disp_warp_fwd", *[vals[k] for k in ("img", "disp", "out", "B", "C", "H", "W", "stream")])


def test_host_refuses_cpu_tensors(native):
    from openstereo_b200 import ops
    with pytest.raises(RuntimeError, match="not implemented on the CPU"):
        ops.disp_warp(torch.zeros(1, 4, 2, 8), torch.zeros(1, 1, 2, 8))


def _mix2(seed, **kw):
    from types import SimpleNamespace
    torch.manual_seed(seed)
    m = omon.load_reference("stereo.modeling.models.monster.update")
    return m.BasicMotionEncoder_mix2(SimpleNamespace(corr_levels=kw.get("levels", 2), corr_radius=kw.get("radius", 4))).eval()


@needs_ref
def test_weight_packing_pads_with_zeros(native):
    """conv / conv_mono (63 rows) are padded to 64 output channels with zero weights and zero biases; convc1 is kept whole over its
    258 input channels (the kernel reads corr and flaw as two blocks)."""
    from openstereo_b200 import update
    enc = _mix2(1)
    eng = update.MixMotionEncoderEngine(enc)
    eng._pack()
    for p, sfx in zip(eng.w, ("", "_mono")):
        conv = getattr(enc, "conv" + sfx)
        assert p["wc"].cout == 64 and p["wd"].cout == 64 and p["b"].shape == (64,) and p["b"][63] == 0
        assert torch.equal(p["b"][:63], conv.bias.float())
        assert tuple(p["c1"].shape) == (258, 64) and torch.equal(p["c1"], getattr(enc, "convc1" + sfx).weight[:, :, 0, 0].t())
        assert tuple(p["d1"].shape) == (64, 7, 7)


@needs_ref
def test_engine_serves_widths_and_hyper_parameters(native):
    """W' >= OSB_TC_MIN_WIDTH with the reference's hyper-parameters; any other width or layer shape runs the module's own forward."""
    from openstereo_b200 import update
    eng = update.MixMotionEncoderEngine(_mix2(2))
    other = update.MixMotionEncoderEngine(_mix2(2, radius=3))

    def args(w, cor=162, flaw=96, b=1):
        return (torch.zeros(b, 1, 2, w), torch.zeros(b, cor, 2, w), torch.zeros(b, flaw, 2, w), torch.zeros(1, 1, 2, w),
                torch.zeros(1, cor, 2, w), torch.zeros(1, flaw, 2, w))
    for w in (16, 20, 23, 24, 32, 60, 64, 128, 160, 240):
        assert eng.serves(*args(w)) == (w >= 24)
    assert not eng.serves(*args(128, cor=126))                                   # another corr_radius
    assert not eng.serves(*args(128, flaw=64))                                   # another flaw width
    assert not eng.serves(*args(128, b=2))
    assert not other.serves(*args(128)) and other.serves(*args(128, cor=126))


# ------------------------------------------------------------------------------------------ the oracle and patch()
@needs_ref
@pytest.mark.parametrize("yaml", [omon.UNIFORM_YAML, omon.AMP_YAML])
def test_oracle_builds_the_reference_class(yaml):
    m = omon.monster(yaml)
    assert type(m).__name__ == "MonSter" and not m.training and m.args.valid_iters == 32 and m.args.encoder == "vits"
    assert omon.amp_dtype(yaml) == (torch.bfloat16 if yaml == omon.AMP_YAML else None)
    again = omon.monster(yaml)
    assert all(torch.equal(a, b) for a, b in zip(m.state_dict().values(), again.state_dict().values()))


_OVERRIDDEN = ("gru04", "gru08", "gru16", "encoder", "disp_head", "mask_feat_4")


@needs_ref
def test_patch_keeps_state_dict_overrides_per_instance_and_refuses_cpu():
    from openstereo_b200.patch import patch
    m, other = omon.monster(), omon.monster()
    mod = omon.load_reference("stereo.modeling.models.monster.monster")
    g = dict(vars(mod))
    cls_dict = dict(vars(type(m)))
    keys = list(m.state_dict().keys())
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    patch(m)
    assert m._osb_patched and list(m.state_dict().keys()) == keys
    assert all(torch.equal(v, sd[k]) for k, v in m.state_dict().items())
    assert dict(vars(mod)) == g and dict(vars(type(m))) == cls_dict                # module globals and class untouched
    blocks = ("update_block", "update_block_mix_stereo", "update_block_mix_mono")
    expected = {"%s.%s" % (b, n) for b in blocks for n in _OVERRIDDEN}
    overridden = {name for name, sub in m.named_modules() if name and "forward" in vars(sub)}
    assert overridden == expected
    assert not any("forward" in vars(sub) for _, sub in other.named_modules())
    for name in ("_forward_pair", "upsample_disp"):
        assert name in vars(m) and name not in vars(other)                  # the rebound methods, this instance only
    assert "forward" not in vars(m)
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA inference only"):
        m(_inputs(1, 64, 128, 3))


@needs_ref
def test_patch_non_strict_cpu_equals_reference():
    from openstereo_b200.patch import patch
    x = _inputs(1, 64, 128, 4)
    with torch.no_grad():
        ref = omon.monster()
        ref.args.valid_iters = 9                                            # iterations 2..8 run the mix2 blocks and the warps
        want = ref(dict(x))["disp_pred"]
        pm = patch(omon.monster(), strict=False)
        pm.args.valid_iters = 9
        got = pm(dict(x))["disp_pred"]
    assert want.shape == (1, 1, 64, 128) and want.std() > 0.1
    assert torch.equal(got, want)
