"""GPU: the host side of every wgmma convolution wrapper, pinned call by call.  A recorder around _lib.call (which still forwards
each call) checks, for every layout combination a wrapper accepts, the one entry point it launches, the profile key it records
under, every non-pointer C argument, every pointer as an offset from the operand tensors, and the shape and dtype of y.  Each
wrapper must refuse a residual of the wrong shape before it launches anything."""
import pytest
import torch

from openstereo_b200 import _lib, ops

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


class _NonNull:
    """A pointer the test cannot name (a buffer the wrapper owns) but that must be set."""

    def __eq__(self, other):
        return other is not None

    def __repr__(self):
        return "<non-null>"


NONNULL = _NonNull()


def rnd(g, *shape, scale=1.0):
    return torch.randn(*shape, device=DEV, generator=g) * scale


def p(t, off=0):
    return None if t is None else t.data_ptr() + off


def stream():
    return torch.cuda.current_stream(DEV).cuda_stream


def weight(g, cout, cin, kc=16, kw_order=(0, 1, 2), pad_cout_to=None, k=3, twod=False):
    if twod:
        return ops.pack_tc_weight_2d(rnd(g, cout, cin, 3, 3, scale=0.05), kc, pad_cout_to=pad_cout_to)
    return ops.pack_tc_weight(rnd(g, cout, cin, k, k, k, scale=0.05), kc, kw_order=kw_order, pad_cout_to=pad_cout_to)


def bn(g, c):
    return rnd(g, c).abs() + 0.5, rnd(g, c, scale=0.1)


# Each case builds its operands and returns (run, entry point, profile key, expected C arguments of y, y shape, y dtype).
CASES = {}


def case(fn):
    CASES[fn.__name__] = fn
    return fn


# ---------------------------------------------------------------------------------------------------------- conv3d_k3_tc
def _s1(g, in_ncdhw, split_in, res):
    b, d, h, w, cin, cout = 1, 2, 4, 128, 32, 32
    wt = weight(g, cout, cin, 32)
    sc, sh = bn(g, cout)
    x = rnd(g, b, cin, d, h, w)
    xin = x if in_ncdhw else (ops.to_split(x) if split_in else x.permute(0, 2, 3, 4, 1).contiguous())
    r, res_ndhwc = None, True
    if res == "ndhwc":
        r = rnd(g, b, d, h, w, cout)
    elif res == "ncdhw":
        r, res_ndhwc = rnd(g, b, cout, d, h, w), False
    elif res == "split":
        r = ops.to_split(rnd(g, b, cout, d, h, w))
    return b, d, h, w, cin, cout, wt, sc, sh, xin, r, res_ndhwc


def _s1_case(in_ncdhw=False, split_in=False, out_ndhwc=True, res=None, out_split=False):
    def build():
        g = torch.Generator(device=DEV).manual_seed(1)
        b, d, h, w, cin, cout, wt, sc, sh, x, r, res_ndhwc = _s1(g, in_ncdhw, split_in, res)
        run = lambda: ops.conv3d_k3_tc(x, wt, sc, sh, r, ops.ACT_RELU, out_ndhwc, res_ndhwc, in_ncdhw, out_split=out_split)  # noqa: E731
        shape = (b, d, h, w, 2 * cout if out_split else cout) if out_ndhwc else (b, cout, d, h, w)
        dtype = torch.float16 if out_split else torch.float32
        if split_in or out_split or res == "split":
            lay = lambda split, ndhwc: ops.LAYOUT_SPLIT if split else (ops.LAYOUT_NDHWC if ndhwc else ops.LAYOUT_NCDHW)  # noqa: E731
            args = lambda y: [p(x), p(wt.data), p(wt.eff_scale(sc)), p(sh), p(r), p(y), b, cin, cout, d, h, w, ops.ACT_RELU,  # noqa: E731
                              lay(split_in, not in_ncdhw), lay(out_split, out_ndhwc), lay(res == "split", res_ndhwc), stream()]
            key = "osb_conv3d_k3_tc_ncdhw_fwd" if in_ncdhw else "osb_conv3d_k3_tc_fwd"
            return run, "osb_conv3d_k3_tc_split_fwd", key, args, shape, dtype
        name = "osb_conv3d_k3_tc_ncdhw_fwd" if in_ncdhw else "osb_conv3d_k3_tc_fwd"
        args = lambda y: [p(x), p(wt.data), p(wt.eff_scale(sc)), p(sh), p(r), p(y), b, cin, cout, d, h, w, ops.ACT_RELU,  # noqa: E731
                          int(out_ndhwc), int(res_ndhwc), stream()]
        return run, name, name, args, shape, dtype
    return build


for _name, _kw in {"ndhwc": {}, "ndhwc_to_ncdhw": dict(out_ndhwc=False), "ndhwc_res_ndhwc": dict(res="ndhwc"),
                   "ncdhw_res_ncdhw_out": dict(out_ndhwc=False, res="ncdhw"), "in_ncdhw": dict(in_ncdhw=True),
                   "in_ncdhw_out_ncdhw": dict(in_ncdhw=True, out_ndhwc=False), "split_in": dict(split_in=True),
                   "split_out": dict(out_split=True), "split_in_out": dict(split_in=True, out_split=True),
                   "split_res": dict(res="split"), "split_in_ncdhw_out": dict(split_in=True, out_ndhwc=False),
                   "split_in_out_res": dict(split_in=True, out_split=True, res="split"),
                   "in_ncdhw_split_out": dict(in_ncdhw=True, out_split=True),
                   "split_in_res_ndhwc": dict(split_in=True, res="ndhwc")}.items():
    CASES["conv3d_k3_tc_" + _name] = _s1_case(**_kw)


@case
def conv3d_k3_tc_gate():
    g = torch.Generator(device=DEV).manual_seed(2)
    b, d, h, w, cin, cout = 1, 2, 4, 64, 64, 64
    wt = weight(g, cout, cin, 16)
    sc, sh = bn(g, cout)
    x, r, gate = rnd(g, b, d, h, w, cin), rnd(g, b, d, h, w, cout), rnd(g, b, h, w, cout).sigmoid()
    run = lambda: ops.conv3d_k3_tc(x, wt, sc, sh, r, ops.ACT_LEAKY, gate=gate)  # noqa: E731
    args = lambda y: [p(x), p(wt.data), p(wt.eff_scale(sc)), p(sh), p(r), p(gate), p(y), b, cin, cout, d, h, w, ops.ACT_LEAKY,  # noqa: E731
                      stream()]
    return run, "osb_conv3d_k3_tc_gate_fwd", "osb_conv3d_k3_tc_gate_fwd", args, (b, d, h, w, cout), torch.float32


def _head(prepadded):
    def build():
        g = torch.Generator(device=DEV).manual_seed(3)
        b, d, h, w, cin = 1, 2, 4, 128, 32
        wt = weight(g, 1, cin, 32, pad_cout_to=16)
        sc, sh = bn(g, 1)
        shp = torch.cat((sh, sh.new_zeros(15))) if prepadded else sh
        x = rnd(g, b, d, h, w, cin)
        run = lambda: ops.conv3d_k3_tc(x, wt, sc, shp, None, ops.ACT_NONE, out_ndhwc=False, res_ndhwc=False)  # noqa: E731
        args = lambda y: [p(x), p(wt.data), p(wt.eff_scale(sc)), p(shp) if prepadded else NONNULL, None, p(y), b, cin, 1, d, h, w,  # noqa: E731
                          ops.ACT_NONE, 0, 0, stream()]
        return run, "osb_conv3d_k3_tc_fwd", "osb_conv3d_k3_tc_fwd", args, (b, 1, d, h, w), torch.float32
    return build


CASES["conv3d_k3_tc_padded_head"] = _head(False)
CASES["conv3d_k3_tc_padded_head_prepadded_shift"] = _head(True)


# ------------------------------------------------------------------------------------------- stride 2 and transposed, 3D
def _s2_case(out_ndhwc, res_ndhwc, with_res, d=2):
    def build():
        g = torch.Generator(device=DEV).manual_seed(4)
        b, h, w, cin, cout = 1, 4, 128, 32, 64
        wt = weight(g, cout, cin, 16, kw_order=(1, 0, 2))
        sc, sh = bn(g, cout)
        x = rnd(g, b, d, h, w, cin)
        do = max(1, d // 2)
        r = (rnd(g, b, do, h // 2, w // 2, cout) if res_ndhwc else rnd(g, b, cout, do, h // 2, w // 2)) if with_res else None
        run = lambda: ops.conv3d_k3_s2_tc(x, wt, sc, sh, r, ops.ACT_RELU, out_ndhwc, res_ndhwc)  # noqa: E731
        args = lambda y: [p(x), p(wt.data), p(wt.eff_scale(sc)), p(sh), p(r), p(y), b, cin, cout, d, h, w, ops.ACT_RELU,  # noqa: E731
                          int(out_ndhwc), int(res_ndhwc), stream()]
        shape = (b, do, h // 2, w // 2, cout) if out_ndhwc else (b, cout, do, h // 2, w // 2)
        return run, "osb_conv3d_k3_s2_tc_fwd", "osb_conv3d_k3_s2_tc_fwd", args, shape, torch.float32
    return build


CASES["conv3d_k3_s2_tc_ncdhw"] = _s2_case(False, False, False)
CASES["conv3d_k3_s2_tc_ndhwc_res_ndhwc"] = _s2_case(True, True, True)
CASES["conv3d_k3_s2_tc_ncdhw_res_ncdhw"] = _s2_case(False, False, True)
CASES["conv3d_k3_s2_tc_one_plane"] = _s2_case(True, False, False, d=1)


def _dc_case(k, out_ndhwc, res_ndhwc, with_res, creal=None):
    def build():
        g = torch.Generator(device=DEV).manual_seed(5)
        b, d, h, w, cin, cout = 1, 2, 2, 32, 64, 64
        wt = ops.pack_tc_deconv_weight(rnd(g, cin, cout, k, k, k, scale=0.05))
        sc, sh = bn(g, cout)
        x = rnd(g, b, d, h, w, cin)
        c = cout if creal is None else creal
        o = (2 * d, 2 * h, 2 * w)
        r = (rnd(g, b, *o, cout) if res_ndhwc else rnd(g, b, c, *o)) if with_res else None
        shape = (b, *o, cout) if out_ndhwc else (b, c, *o)
        if k == 3:
            run = lambda: ops.deconv3d_k3_tc(x, wt, sc, sh, r, ops.ACT_RELU, out_ndhwc, res_ndhwc)  # noqa: E731
            args = lambda y: [p(x), p(wt.data), p(wt.eff_scale(sc)), p(sh), p(r), p(y), b, cin, cout, d, h, w, ops.ACT_RELU,  # noqa: E731
                              int(out_ndhwc), int(res_ndhwc), stream()]
            return run, "osb_deconv3d_k3_tc_fwd", "osb_deconv3d_k3_tc_fwd", args, shape, torch.float32
        run = lambda: ops.deconv3d_k4_tc(x, wt, sc, sh, r, ops.ACT_RELU, out_ndhwc, res_ndhwc, cout_real=creal)  # noqa: E731
        args = lambda y: [p(x), p(wt.data), p(wt.eff_scale(sc)), p(sh), p(r), p(y), b, cin, cout, c, d, h, w, ops.ACT_RELU,  # noqa: E731
                          int(out_ndhwc), int(res_ndhwc), stream()]
        return run, "osb_deconv3d_k4_tc_fwd", "osb_deconv3d_k4_tc_fwd", args, shape, torch.float32
    return build


CASES["deconv3d_k3_tc_ncdhw"] = _dc_case(3, False, False, False)
CASES["deconv3d_k3_tc_ndhwc_res_ndhwc"] = _dc_case(3, True, True, True)
CASES["deconv3d_k3_tc_ncdhw_res_ncdhw"] = _dc_case(3, False, False, True)
CASES["deconv3d_k4_tc_ndhwc"] = _dc_case(4, True, True, False)
CASES["deconv3d_k4_tc_ndhwc_res_ndhwc"] = _dc_case(4, True, True, True)
CASES["deconv3d_k4_tc_ncdhw_real"] = _dc_case(4, False, False, False, creal=48)
CASES["deconv3d_k4_tc_ncdhw_real_res_ncdhw"] = _dc_case(4, False, False, True, creal=48)


# -------------------------------------------------------------------------------------------------------------- tc_slice
def _slice_case(kind, coff, gate=False):
    def build():
        g = torch.Generator(device=DEV).manual_seed(6)
        b = 1
        if kind == "s2":
            d, h, w, cin, cout, ctot = 2, 4, 32, 96, 96 if coff == 0 else 64, 160
            wt, o = weight(g, cout, cin, 16, kw_order=(1, 0, 2)), (d // 2, h // 2, w // 2)
            name = "osb_conv3d_k3_s2_tc_cs_fwd"
        elif kind == "s1":
            d, h, w, cin, cout, ctot = 2, 4, 16, 160, 96 if coff == 0 else 64, 160
            wt, o = weight(g, cout, cin, 16), (d, h, w)
            name = "osb_conv3d_k3_tc_cs_fwd"
        else:
            d, h, w, cin, cout, ctot = 1, 2, 16, 160, 64 if coff == 0 else 32, 96
            wt, o = ops.pack_tc_deconv_weight(rnd(g, cin, cout, 4, 4, 4, scale=0.05)), (2 * d, 2 * h, 2 * w)
            name = "osb_deconv3d_k4_tc_cs_fwd"
        sc, sh = bn(g, cout)
        x, y = rnd(g, b, d, h, w, cin), torch.zeros(b, *o, ctot, device=DEV)
        gt = rnd(g, b, h, w, ctot).sigmoid() if gate else None
        run = lambda: ops.tc_slice(kind, x, wt, sc, sh, y, coff, ops.ACT_LEAKY, gate=gt)  # noqa: E731
        head = [p(x), p(wt.data), p(wt.eff_scale(sc)), p(sh)]
        tail = [b, cin, cout, d, h, w, ops.ACT_LEAKY, ctot, stream()]
        if kind == "s1":
            args = lambda yy: head + [None, p(gt, 4 * coff), p(y, 4 * coff)] + tail  # noqa: E731
        else:
            args = lambda yy: head + [p(y, 4 * coff)] + tail  # noqa: E731

        def run_same_y():
            out = run()
            assert out is y
            return out
        return run_same_y, name, name, args, tuple(y.shape), torch.float32
    return build


CASES["tc_slice_s2_lo"] = _slice_case("s2", 0)
CASES["tc_slice_s2_hi"] = _slice_case("s2", 96)
CASES["tc_slice_s1_lo_gate"] = _slice_case("s1", 0, gate=True)
CASES["tc_slice_s1_hi_gate"] = _slice_case("s1", 96, gate=True)
CASES["tc_slice_s1_hi"] = _slice_case("s1", 96)
CASES["tc_slice_dc4_lo"] = _slice_case("dc4", 0)
CASES["tc_slice_dc4_hi"] = _slice_case("dc4", 64)


# ------------------------------------------------------------------------------------------------------------ conv2d_k3_tc
def _2d_case(cin, cout, out_nhwc, res, precision="fp32", dilation=1):
    def build():
        g = torch.Generator(device=DEV).manual_seed(7)
        b, h, w = 2, 4, 128
        kc = ops.conv2d_tc_kc(cin, cout, w, dilation)
        wt = weight(g, cout, cin, kc, twod=True)
        sc, sh = bn(g, cout)
        x = rnd(g, b, h, w, cin)
        r = {None: None, "nhwc": rnd(g, b, h, w, cout), "nchw": rnd(g, b, cout, h, w)}[res]
        res_nhwc = res != "nchw"
        run = lambda: ops.conv2d_k3_tc(x, wt, sc, sh, r, ops.ACT_RELU, dilation, out_nhwc, res_nhwc, precision)  # noqa: E731
        prec = ops.PRECISIONS[precision]
        name = "osb_conv2d_k3_tc_prec_fwd" if prec else "osb_conv2d_k3_tc_fwd"
        args = lambda y: ([p(x), p(wt.data), p(wt.eff_scale(sc)), p(sh), p(r), p(y), b, cin, cout, h, w, dilation, ops.ACT_RELU,  # noqa: E731
                           int(out_nhwc), int(res_nhwc)] + ([prec] if prec else []) + [stream()])
        return run, name, name, args, (b, h, w, cout) if out_nhwc else (b, cout, h, w), torch.float32
    return build


CASES["conv2d_k3_tc_nhwc"] = _2d_case(32, 32, True, None)
CASES["conv2d_k3_tc_nchw_res_nhwc"] = _2d_case(32, 32, False, "nhwc")
CASES["conv2d_k3_tc_nhwc_res_nchw"] = _2d_case(64, 64, True, "nchw")
CASES["conv2d_k3_tc_dilated"] = _2d_case(128, 128, True, "nhwc", dilation=2)
CASES["conv2d_k3_tc_f16"] = _2d_case(64, 64, False, "nhwc", precision="f16")
CASES["conv2d_k3_tc_f16_kc32"] = _2d_case(32, 32, True, None, precision="f16")


def _gru_case(res, out_nhwc, mode, precision="fp32"):
    def build():
        g = torch.Generator(device=DEV).manual_seed(8)
        b, h, w, cin, cout = 2, 4, 32, 64, 128
        wt = weight(g, cout, cin, 16, twod=True)
        sh = rnd(g, cout, scale=0.1)
        x = rnd(g, b, h, w, cin)
        r, rbs = None, 0
        if res == "nhwc":
            r = rnd(g, b, h, w, cout)
        elif res == "nchw":
            r = rnd(g, b, cout, h, w)
        elif res == "view":                                          # a channel split() of a wider NCHW tensor
            wide = rnd(g, b, 3 * cout, h, w)
            r = wide.split(cout, 1)[1]
            rbs = wide.stride(0)
        mul = rnd(g, b, h, w, cout) if mode == "mul" else None
        z, hh = (rnd(g, b, h, w, cout).sigmoid(), rnd(g, b, h, w, cout)) if mode == "blend" else (None, None)
        act = {"plain": ops.ACT_NONE, "mul": ops.ACT_SIGMOID, "blend": ops.ACT_TANH}[mode]
        res_nhwc = res == "nhwc"
        run = lambda: ops.conv2d_k3_tc_gru(x, wt, sh, r, act, mul, None if z is None else (z, hh), out_nhwc, res_nhwc,  # noqa: E731
                                           precision)
        prec = ops.PRECISIONS[precision]
        name = "osb_conv2d_k3_tc_gru_prec_fwd" if prec else "osb_conv2d_k3_tc_gru_fwd"
        args = lambda y: ([p(x), p(wt.data), p(wt.eff_scale(None)), p(sh), p(r), p(mul), p(z), p(hh), p(y), b, cin, cout, h, w,  # noqa: E731
                           act, int(out_nhwc), int(res_nhwc), rbs] + ([prec] if prec else []) + [stream()])
        return run, name, name, args, (b, h, w, cout) if out_nhwc else (b, cout, h, w), torch.float32
    return build


CASES["conv2d_k3_tc_gru_view_res"] = _gru_case("view", True, "plain")
CASES["conv2d_k3_tc_gru_nchw_res"] = _gru_case("nchw", True, "plain")
CASES["conv2d_k3_tc_gru_mul"] = _gru_case("nhwc", True, "mul")
CASES["conv2d_k3_tc_gru_blend_nchw_out"] = _gru_case("nhwc", False, "blend")
CASES["conv2d_k3_tc_gru_view_res_f16"] = _gru_case("view", True, "plain", precision="f16")
CASES["conv2d_k3_tc_gru_blend_f16"] = _gru_case(None, False, "blend", precision="f16")


def _md_case(cout, stride, out_nhwc, prepadded=False, mask_mode=ops.MASK_PROB):
    def build():
        g = torch.Generator(device=DEV).manual_seed(9)
        b, h, w, cin, dg, pad, dil = 2, 6, 20, 32, 2, 1, 1
        rows = ops.mdconv_packed_rows(cout)
        wt = ops.pack_tc_weight_2d(rnd(g, cout, cin, 3, 3, scale=0.05), 16, pad_cout_to=rows)
        sc, sh = bn(g, cout)
        shp = torch.cat((sh, sh.new_zeros(rows - cout))) if prepadded else sh
        ho, wo = (h + 2 * pad - 2 * dil - 1) // stride + 1, (w + 2 * pad - 2 * dil - 1) // stride + 1
        x = rnd(g, b, h, w, cin)
        om = rnd(g, b, dg * 27, ho, wo)
        off, mask = om[:, :dg * 18], om[:, dg * 18:]
        run = lambda: ops.mdconv2d_k3_tc(x, off, mask, wt, sc, shp, stride, pad, dil, dg, ops.ACT_RELU, mask_mode, out_nhwc)  # noqa: E731
        padded = rows != cout
        args = lambda y: [p(x), p(off), om.stride(0), p(mask), om.stride(0), mask_mode, p(wt.data), p(wt.eff_scale(sc)),  # noqa: E731
                          NONNULL if padded and not prepadded else p(shp), NONNULL if padded else p(y), b, cin, rows, h, w, stride, pad,
                          dil, dg, ops.ACT_RELU, int(out_nhwc), stream()]
        return (run, "osb_mdconv2d_k3_tc_fwd", "osb_mdconv2d_k3_tc_fwd", args, (b, ho, wo, cout) if out_nhwc else (b, cout, ho, wo),
                torch.float32)
    return build


CASES["mdconv2d_k3_tc_padded_plan"] = _md_case(16, 1, False)
CASES["mdconv2d_k3_tc_padded_plan_prepadded_shift"] = _md_case(16, 1, False, prepadded=True)
CASES["mdconv2d_k3_tc_nhwc_stride2"] = _md_case(32, 2, True, mask_mode=ops.MASK_DOUBLE_SIGMOID)
CASES["mdconv2d_k3_tc_nchw"] = _md_case(64, 1, False)


def _record(monkeypatch):
    calls, real = [], _lib.call

    def recorder(name, *args):
        calls.append((name, args))
        return real(name, *args)
    monkeypatch.setattr(_lib, "call", recorder)
    return calls


def _run(monkeypatch, build):
    run, name, key, args, shape, dtype = build()
    calls = _record(monkeypatch)
    ops.profile_start()
    try:
        y = run()
    finally:
        prof = ops.profile_stop()
    torch.cuda.synchronize()
    assert [n for n, _ in calls] == [name]
    assert list(prof) == [key]
    assert list(calls[0][1]) == args(y)
    assert tuple(y.shape) == shape and y.dtype == dtype
    return y


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_path(monkeypatch, name):
    _run(monkeypatch, CASES[name])


@pytest.mark.parametrize("pair", [("conv3d_k3_tc_padded_head", "conv3d_k3_tc_padded_head_prepadded_shift"),
                                  ("mdconv2d_k3_tc_padded_plan", "mdconv2d_k3_tc_padded_plan_prepadded_shift")])
def test_short_shift_is_zero_padded(monkeypatch, pair):
    """A shift with the layer's channels on a zero-padded plan runs exactly as the same shift padded with zeros by the caller."""
    a, b = (_run(monkeypatch, CASES[n]) for n in pair)
    assert torch.equal(a, b)


def _bad_residuals(g):
    """(wrapper call taking a residual, residual shape it needs, wrong shapes)."""
    x3 = rnd(g, 1, 2, 4, 128, 32)
    w32 = weight(g, 32, 32, 32)
    ws2 = weight(g, 64, 32, 16, kw_order=(1, 0, 2))
    x_dc = rnd(g, 1, 2, 2, 32, 64)
    wdc3 = ops.pack_tc_deconv_weight(rnd(g, 64, 64, 3, 3, 3, scale=0.05))
    wdc4 = ops.pack_tc_deconv_weight(rnd(g, 64, 64, 4, 4, 4, scale=0.05))
    x2 = rnd(g, 2, 4, 128, 32)
    w2 = weight(g, 32, 32, 32, twod=True)
    xg = rnd(g, 2, 4, 32, 64)
    wg = weight(g, 128, 64, 16, twod=True)
    return [
        (lambda r: ops.conv3d_k3_tc(x3, w32, None, None, r), [(1, 2, 4, 128, 16), (1, 32, 2, 4, 128), (1, 2, 4, 64, 32)]),
        (lambda r: ops.conv3d_k3_tc(x3, w32, None, None, r, out_ndhwc=False, res_ndhwc=False), [(1, 2, 4, 128, 32), (1, 16, 2, 4, 128)]),
        (lambda r: ops.conv3d_k3_s2_tc(x3, ws2, None, None, r), [(1, 1, 2, 64, 64), (1, 64, 2, 2, 64), (1, 32, 1, 2, 64)]),
        (lambda r: ops.conv3d_k3_s2_tc(x3, ws2, None, None, r, out_ndhwc=True, res_ndhwc=True), [(1, 64, 1, 2, 64)]),
        (lambda r: ops.deconv3d_k3_tc(x_dc, wdc3, None, None, r), [(1, 4, 4, 64, 64), (1, 64, 4, 4, 32)]),
        (lambda r: ops.deconv3d_k4_tc(x_dc, wdc4, None, None, r), [(1, 64, 4, 4, 64), (1, 4, 4, 64, 32)]),
        (lambda r: ops.deconv3d_k4_tc(x_dc, wdc4, None, None, r, out_ndhwc=False, res_ndhwc=False, cout_real=48),
         [(1, 64, 4, 4, 64), (1, 4, 4, 64, 48)]),
        (lambda r: ops.conv2d_k3_tc(x2, w2, None, None, r), [(2, 4, 128, 16), (2, 4, 64, 32)]),
        (lambda r: ops.conv2d_k3_tc(x2, w2, None, None, r, res_nhwc=False), [(2, 16, 4, 128)]),
        (lambda r: ops.conv2d_k3_tc_gru(xg, wg, None, r), [(2, 4, 32, 64), (2, 128, 4, 32)]),
        (lambda r: ops.conv2d_k3_tc_gru(xg, wg, None, r, res_nhwc=False), [(2, 4, 32, 128), (2, 64, 4, 32)]),
    ]


def test_wrong_residual_shape_is_refused_before_any_launch(monkeypatch):
    g = torch.Generator(device=DEV).manual_seed(10)
    cases = _bad_residuals(g)
    calls = _record(monkeypatch)
    for run, shapes in cases:
        for shape in shapes:
            with pytest.raises(AssertionError):
                run(torch.zeros(shape, device=DEV))
    assert calls == []
