"""GPU: IGEV++'s instance-normalised hourglasses on the library -- the two instance-norm modes of the fp32 CUDA-core convolutions
(moments out: per-(b, channel) statistics against float64 with partial tiles in every dimension, bit-identical reruns, no store
outside the output, the statistics or the workspace; normalised input: against F.instance_norm -> leaky_relu -> gate -> conv in
float64, border voxels included), the IGEVPPAggregation engine against a reference hourglass(8) in float64 with its launch sequence
pinned, and patch(model, aggregation=True) under both YAMLs against the unpatched model.  Sorted after the torch.profiler routing
suites like the other model-level files."""
import pytest
import torch
import torch.nn.functional as F

from oracle import _reference_shim as shim
from oracle import igevpp as oigpp

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not shim.available(), reason="reference tree (oracle/_ref) not staged")]

SENTINEL = -1234.5
GUARD = 256                 # sentinel floats on each side of every region the kernels write (1 KB, keeps 16-byte alignment)
STATS_TOL = 1e-5            # |mean - mean64| / (|mean64| + std64) and |rstd / rstd64 - 1|
CONV_TOL = 1e-5             # per element, of the summed |products| feeding it
ENGINE_TOL = 1e-3           # max |out - out64| / max |out64| through the 16 convolutions and 6 gates of one hourglass


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, aggregation, ops
    from openstereo_b200.patch import patch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return _lib, ops, aggregation, patch


class Guarded:
    """One device buffer of sentinels: regions handed out back to back, each 16-byte aligned between at least GUARD sentinels."""

    def __init__(self, sizes):
        offs, off = [], GUARD
        for n in sizes:
            offs.append(off)
            off += (n + 3) // 4 * 4 + GUARD
        self.buf = torch.full((off,), SENTINEL, device="cuda")
        self.views = [self.buf[o:o + n] for o, n in zip(offs, sizes)]
        self.outside = torch.ones(off, dtype=torch.bool, device="cuda")
        for o, n in zip(offs, sizes):
            self.outside[o:o + n] = False

    def intact(self):
        return bool((self.buf[self.outside] == SENTINEL).all())


def _rnd(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).cuda()


def _in64(x, stats, gate):
    """leaky(instance_norm(x)) * gate in float64 with the given (mean, rstd)."""
    x = x.double()
    mean, rstd = stats[..., 0].double(), stats[..., 1].double()
    shape = mean.shape + (1,) * (x.dim() - 2)
    y = F.leaky_relu((x - mean.view(shape)) * rstd.view(shape), 0.01)
    if gate is not None:
        y = y * (gate.double().unsqueeze(2) if x.dim() == 5 else gate.double())
    return y


def _stats64(y):
    y = y.double().flatten(2)
    mean, var = y.mean(2), y.var(2, unbiased=False)
    return mean, var


def _stats32(x):
    """(B, C, 2) float32 (mean, rstd) of x, computed in float64 (the normalised-input tests feed exact statistics)."""
    mean, var = _stats64(x)
    return torch.stack([mean, 1 / torch.sqrt(var + 1e-5)], -1).float().contiguous()


# (family, Cin, Cout, input shape (B, D, H, W), stride / kernel, c0): partial tiles in every dimension of every instantiation the
# hourglass reaches -- launch_conv_k3<1,8,4,4,4,8> (tile 4 x 4 x 32, Cout 8..64), launch_conv_k3<2,8,4,2,4,4> (2 x 4 x 32),
# launch_deconv<4,8> (4 x 4 x 64 outputs), conv3d_1x1_kernel over one and two slabs and in 2D (64 voxel octets of 8 columns)
CASES = [
    ("k3", 13, 8, (2, 5, 6, 36), 1, None), ("k3", 16, 40, (2, 5, 6, 36), 1, None), ("k3", 8, 64, (1, 7, 10, 70), 1, None),
    ("k3", 11, 16, (2, 5, 9, 71), 2, None), ("k3", 32, 64, (2, 3, 5, 17), 2, None),
    ("dc", 12, 8, (2, 3, 5, 34), 4, None), ("dc", 64, 32, (1, 2, 3, 9), 4, None),
    ("pw", 64, 32, (2, 3, 5, 20), 0, 32), ("pw", 32, 16, (2, 6, 9, 30), 0, 16), ("pw", 96, 48, (2, 1, 7, 44), 0, None),
    ("pw", 40, 24, (2, 3, 5, 20), 0, 40),
]


def _case_id(c):
    return "%s-%d-%d-%s-%d%s" % (c[0], c[1], c[2], "x".join(map(str, c[3])), c[4], "" if c[5] in (None, c[1]) else "-c0%d" % c[5])


def _run(lib, ops, fam, x, w, y, stats, ws, in_stats=None, in_gate=None, x1=None, in_stats1=None, in_gate1=None, param=1):
    s = torch.cuda.current_stream().cuda_stream
    p = lambda t: None if t is None else t.data_ptr()                                   # noqa: E731
    b, cin = x.shape[:2]
    d, h, wd = x.shape[2:]
    cout = w.shape[-1]
    if fam == "k3":
        lib.call("osb_conv3d_k3_in_fwd", x.data_ptr(), w.data_ptr(), None, None, p(in_stats), p(in_gate), y.data_ptr(), p(stats), p(ws),
                 0 if ws is None else ws.numel(), b, cin, cout, d, h, wd, param, 0, s)
    elif fam == "dc":
        lib.call("osb_deconv3d_in_fwd", x.data_ptr(), w.data_ptr(), None, None, p(in_stats), p(in_gate), y.data_ptr(), p(stats), p(ws),
                 0 if ws is None else ws.numel(), b, cin, cout, d, h, wd, param, 0, s)
    else:
        c1 = 0 if x1 is None else x1.shape[1]
        lib.call("osb_conv3d_1x1_in_fwd", x.data_ptr(), p(x1), cin, w.data_ptr(), None, None, p(in_stats), p(in_gate), p(in_stats1),
                 p(in_gate1), y.data_ptr(), p(stats), p(ws), 0 if ws is None else ws.numel(), b, cin + c1, cout, d, h, wd, 0, 0, s)


def _weights(g, fam, cin, cout, param):
    from openstereo_b200 import ops
    if fam == "k3":
        wt = _rnd(g, cout, cin, 3, 3, 3, scale=0.2)
        return wt, ops.pack_conv_weight(wt)
    if fam == "dc":
        wt = _rnd(g, cin, cout, param, param, param, scale=0.2)
        return wt, ops.pack_deconv_weight(wt)
    wt = _rnd(g, cout, cin, 1, 1, 1, scale=0.2)
    return wt, wt.reshape(cout, cin).t().contiguous()


def _out_shape(fam, b, cout, d, h, w, param):
    if fam == "k3":
        return (b, cout, (d - 1) // param + 1, (h - 1) // param + 1, (w - 1) // param + 1)
    if fam == "dc":
        return (b, cout, 2 * d, 2 * h, 2 * w)
    return (b, cout, d, h, w)


def _conv64(fam, x, wt, param):
    if fam == "k3":
        return F.conv3d(x, wt.double(), stride=param, padding=1)
    if fam == "dc":
        return F.conv_transpose3d(x, wt.double(), stride=2, padding=1)
    return F.conv3d(x, wt.double())


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_moments_out(osb, case):
    """Raw output within CONV_TOL of the float64 conv; per-(b, channel) mean and rstd within STATS_TOL of float64 statistics of the
    stored output; a rerun gives the same bits; the sentinels around the output, the statistics and the workspace are intact and the
    workspace's counters are back to 0."""
    lib, ops, _, _ = osb
    fam, cin, cout, (b, d, h, w), param, c0 = case
    g = torch.Generator().manual_seed(sum(case[3]) + cin + cout)
    wt, wp = _weights(g, fam, cin, cout, param)
    x = _rnd(g, b, cin, d, h, w) + 0.5
    c0 = c0 or cin
    oshape = _out_shape(fam, b, cout, d, h, w, param)
    need = lib.lib.osb_conv3d_in_workspace_floats({"k3": 0, "dc": 1, "pw": 2}[fam], b, cout, d, h, w, param)
    assert need > 0
    n_y = oshape[0] * oshape[1] * oshape[2] * oshape[3] * oshape[4]
    buf = Guarded([n_y, b * cout * 2, need])
    yv, sv, wv = buf.views
    wv.zero_()
    runs = []
    for _ in range(2):
        if fam == "pw" and c0 < cin:
            _run(lib, ops, fam, x[:, :c0].contiguous(), wp, yv, sv, wv, x1=x[:, c0:].contiguous())
        else:
            _run(lib, ops, fam, x, wp, yv, sv, wv, param=param)
        torch.cuda.synchronize()
        runs.append((yv.clone(), sv.clone()))
    assert buf.intact()
    blocks = -(-cout // {"k3": 32, "dc": 16, "pw": 32}[fam])
    assert bool((wv[need - b * blocks:].view(torch.int32) == 0).all())                 # the counters re-armed themselves
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    y = runs[0][0].view(oshape)
    want = _conv64(fam, x.double(), wt, param)
    mag = _conv64(fam, x.double().abs(), wt.abs(), param)
    assert ((y.double() - want).abs() <= CONV_TOL * mag + 1e-6).all()
    mean64, var64 = _stats64(y)
    st = runs[0][1].view(b, cout, 2).double()
    std64 = var64.sqrt()
    err_m = ((st[..., 0] - mean64).abs() / (mean64.abs() + std64)).max().item()
    err_r = (st[..., 1] * torch.sqrt(var64 + 1e-5) - 1).abs().max().item()
    print("%s: mean err %.2e, rstd err %.2e" % (_case_id(case), err_m, err_r))
    assert err_m <= STATS_TOL and err_r <= STATS_TOL


NORM_CASES = [c for c in CASES if c[0] != "pw"] + [
    ("pw", 64, 32, (2, 3, 5, 20), 0, 32), ("pw", 32, 16, (2, 6, 9, 30), 0, 16), ("pw", 48, 96, (2, 1, 7, 44), 0, None)]


@pytest.mark.parametrize("case", NORM_CASES, ids=_case_id)
@pytest.mark.parametrize("gated", [False, True])
def test_normalised_input(osb, case, gated):
    """conv(leaky(instance_norm(x)) * gate) against float64, border voxels included (the padding is 0 after normalisation); the
    1x1 over two slabs normalises each slab by its own statistics and gates only the second, as agg_0 / agg_1 do."""
    lib, ops, _, _ = osb
    fam, cin, cout, (b, d, h, w), param, c0 = case
    g = torch.Generator().manual_seed(3 * sum(case[3]) + cin + cout + gated)
    wt, wp = _weights(g, fam, cin, cout, param)
    x = _rnd(g, b, cin, d, h, w, scale=2.0) + 1.0
    c0 = c0 or cin
    gate = torch.sigmoid(_rnd(g, b, cin, h, w)) if gated else None
    y = torch.full(_out_shape(fam, b, cout, d, h, w, param), SENTINEL, device="cuda")
    if fam == "pw" and c0 < cin:
        xa, xb = x[:, :c0].contiguous(), x[:, c0:].contiguous()
        sa, sb = _stats32(xa), _stats32(xb)
        gb = gate[:, c0:].contiguous() if gated else None
        _run(lib, ops, fam, xa, wp, y, None, None, sa, None, xb, sb, gb)
        xn = torch.cat([_in64(xa, sa, None), _in64(xb, sb, gb)], 1)
    else:
        st = _stats32(x)
        xin = x[:, :, 0] if (fam == "pw" and d == 1) else x
        _run(lib, ops, fam, x, wp, y, None, None, st, gate, param=param)
        xn = _in64(xin, st, gate)
        if xn.dim() == 4:
            xn = xn.unsqueeze(2)
    torch.cuda.synchronize()
    want = _conv64(fam, xn, wt, param)
    mag = _conv64(fam, xn.abs(), wt.abs(), param)
    err = ((y.double() - want).abs() / (mag + 1e-6)).max().item()
    print("%s gated=%s: max err / magnitude %.2e" % (_case_id(case), gated, err))
    assert err <= CONV_TOL


def test_entry_points_refuse(osb):
    lib, ops, _, _ = osb
    s = torch.cuda.current_stream().cuda_stream
    x = torch.zeros(1, 8, 4, 4, 8, device="cuda")
    w = torch.zeros(8, 27, 8, device="cuda")
    y = torch.empty(1, 8, 4, 4, 8, device="cuda")
    st = torch.empty(1, 8, 2, device="cuda")
    ws = torch.zeros(4, device="cuda")
    P = lambda t: t.data_ptr()                                                          # noqa: E731
    before = lib.launch_count()
    with pytest.raises(ValueError, match="workspace"):
        lib.call("osb_conv3d_k3_in_fwd", P(x), P(w), None, None, None, None, P(y), P(st), P(ws), 4, 1, 8, 8, 4, 4, 8, 1, 0, s)
    with pytest.raises(ValueError, match="null pointer"):
        lib.call("osb_conv3d_k3_in_fwd", P(x), P(w), None, None, None, None, P(y), P(st), None, 0, 1, 8, 8, 4, 4, 8, 1, 0, s)
    with pytest.raises(ValueError, match="empty shape"):
        lib.call("osb_deconv3d_in_fwd", P(x), P(w), None, None, None, None, P(y), None, None, 0, 1, 8, 8, 0, 4, 8, 4, 0, s)
    with pytest.raises(ValueError, match="raw output"):
        lib.call("osb_conv3d_1x1_in_fwd", P(x), None, 8, P(w), None, None, None, None, None, None, P(y), P(st), P(ws), 4, 1, 8, 8,
                 4, 4, 8, 0, 1, s)
    with pytest.raises(ValueError, match="grid too large"):
        lib.call("osb_conv3d_1x1_in_fwd", P(x), None, 8, P(w), None, None, None, None, None, None, P(y), None, None, 0, 70000, 8, 8,
                 4, 4, 8, 0, 0, s)
    assert lib.launch_count() == before
    assert lib.lib.osb_conv3d_in_workspace_floats(3, 1, 8, 4, 4, 8, 1) == -1


# ------------------------------------------------------------------------------------------ the engine
def _hourglass(seed):
    torch.manual_seed(seed)
    return oigpp.load_reference("stereo.modeling.models.igevpp.igevpp_stereo").hourglass(8).eval().cuda()


def _hg_inputs(b, d, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, 8, d, h, w, generator=g)
    ext = [(h, w)]
    for _ in range(3):
        ext.append(tuple((e - 1) // 2 + 1 for e in ext[-1]))
    feats = [torch.randn(b, c, *e, generator=g) for c, e in zip((96, 64, 192, 160), ext)]
    return x, feats


SEQUENCE = (["osb_conv3d_k3_in_fwd"] + ["osb_conv3d_1x1_in_fwd"] * 2 + ["osb_conv3d_k3_in_fwd"] * 2 + ["osb_conv3d_1x1_in_fwd"] * 2
            + ["osb_conv3d_k3_in_fwd"] * 2 + ["osb_conv3d_1x1_in_fwd"] * 2 + ["osb_conv3d_k3_in_fwd"] * 2 + ["osb_conv3d_1x1_in_fwd"] * 2
            + ["osb_deconv3d_in_fwd", "osb_conv3d_1x1_in_fwd"] + ["osb_conv3d_k3_in_fwd"] * 2 + ["osb_conv3d_1x1_in_fwd"] * 2
            + ["osb_deconv3d_in_fwd", "osb_conv3d_1x1_in_fwd"] + ["osb_conv3d_k3_in_fwd"] * 2 + ["osb_conv3d_1x1_in_fwd"] * 2
            + ["osb_deconv3d_in_fwd"])


@pytest.mark.parametrize("shape", [(1, 48, 64, 128), (2, 47, 31, 63), (1, 24, 16, 40)], ids=lambda s: "x".join(map(str, s)))
def test_engine_against_hourglass_fp64(osb, shape):
    """IGEVPPAggregation on one seeded reference hourglass(8): the model's real shape (D' = 48 at 1/4 of 256x512) and odd D/H/W,
    within ENGINE_TOL of the module in float64; 28 launches in the pinned order (16 convolutions, 6 gates of two 1x1 launches)."""
    lib, ops, aggregation, _ = osb
    hg = _hourglass(sum(shape))
    x, feats = _hg_inputs(*shape, seed=sum(shape) + 1)
    eng = aggregation.IGEVPPAggregation(hg)
    xg, fg = x.cuda(), [f.cuda() for f in feats]
    assert eng.serves(xg, fg)
    with torch.no_grad():
        got = eng(xg, fg)
        torch.cuda.synchronize()
        order = []
        real_call = lib.call
        lib.call = lambda name, *a: (order.append(name), real_call(name, *a))[1]
        try:
            before = lib.launch_count()
            again = eng(xg, fg)
            n = lib.launch_count() - before
        finally:
            lib.call = real_call
        want = hg.double().cuda()(xg.double(), [f.double() for f in fg])
    assert order == SEQUENCE and n == 28
    assert torch.equal(got, again)
    b, _, d, h, w = x.shape
    assert got.shape == want.shape == (b, 8, 2 * ((d + 1) // 2), 2 * ((h + 1) // 2), 2 * ((w + 1) // 2))
    err = (got.double() - want).abs().max().item() / want.abs().max().item()
    print("hourglass(8) %s: max err / max |out| %.2e" % ("x".join(map(str, shape)), err))
    assert err <= ENGINE_TOL


def test_engine_refusals(osb):
    """Affine or tracked instance norms, another LeakyReLU slope and shapes the graph cannot concatenate are not served; the patched
    module then runs its own forward."""
    _, _, aggregation, patch = osb
    x, feats = _hg_inputs(1, 16, 16, 32, 3)
    xg, fg = x.cuda(), [f.cuda() for f in feats]
    assert aggregation.IGEVPPAggregation(_hourglass(1)).serves(xg, fg)
    assert not aggregation.IGEVPPAggregation(_hourglass(1).cpu()).serves(xg, fg)          # parameters elsewhere
    assert not aggregation.IGEVPPAggregation(_hourglass(1)).serves(xg[:, :, :, :15], fg)
    assert not aggregation.IGEVPPAggregation(_hourglass(1)).serves(xg, fg[:3])
    hg = _hourglass(1)
    hg.conv2[1].IN = torch.nn.InstanceNorm3d(32, affine=True)
    assert not aggregation.IGEVPPAggregation(hg).serves(xg, fg)
    hg = _hourglass(1)
    hg.feature_att_16.feat_att[0].IN = torch.nn.InstanceNorm2d(96, track_running_stats=True).eval()
    assert not aggregation.IGEVPPAggregation(hg).serves(xg, fg)
    hg = _hourglass(1)
    hg.agg_0[1].slope = torch.nn.LeakyReLU(0.2)
    assert not aggregation.IGEVPPAggregation(hg).serves(xg, fg)


# ------------------------------------------------------------------------------------------ the whole model
def _x(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return {"left": torch.rand(b, 3, h, w, generator=g) * 2 - 1, "right": torch.rand(b, 3, h, w, generator=g) * 2 - 1}


@pytest.mark.parametrize("yaml", ["uniform", "amp"])
def test_whole_model_with_aggregation(osb, yaml):
    """256x512.  Uniform YAML: patch(m, aggregation=True) within max(10 x the reference's GPU-vs-CPU floor, 1e-2) px EPE of the
    unpatched model on the GPU; the three hourglasses run 3 x 28 launches of the instance-norm entry points.  AMP YAML: the
    reference's output dtype and an EPE to the fp32 CPU reference within twice the unpatched AMP model's."""
    lib, ops, _, patch = osb
    path = oigpp.UNIFORM_YAML if yaml == "uniform" else oigpp.AMP_YAML
    x = _x(1, 256, 512, 91)
    xg = {k: v.cuda() for k, v in x.items()}
    with torch.no_grad():
        want_cpu = oigpp.igevpp()(dict(x))["disp_pred"]
        if yaml == "uniform":
            m = oigpp.igevpp().cuda()
            want_gpu = m(dict(xg))["disp_pred"]
            pm = patch(m, aggregation=True)
            ops.profile_start()
            got = pm(dict(xg))["disp_pred"]
            prof = ops.profile_stop()
            counts = {k: len(v) for k, v in prof.items()}
            assert counts["osb_conv3d_k3_in_fwd"] == 3 * 11 and counts["osb_deconv3d_in_fwd"] == 3 * 3
            assert counts["osb_conv3d_1x1_in_fwd"] == 3 * 14
            e_gpu = (got - want_gpu).abs().mean().item()
            floor = (want_gpu.cpu() - want_cpu).abs().mean().item()
            print("patch(IGEV++, aggregation=True) 256x512: EPE %.3e vs GPU ref (floor %.3e)" % (e_gpu, floor))
            assert got.dtype == torch.float32 and want_cpu.std() > 1.0
            assert e_gpu <= max(10 * floor, 1e-2)
        else:
            amp = oigpp.igevpp(path).cuda()(dict(xg))["disp_pred"]
            got = patch(oigpp.igevpp(path).cuda(), aggregation=True)(dict(xg))["disp_pred"]
            e_amp = (amp.cpu() - want_cpu).abs().mean().item()
            e_got = (got.cpu() - want_cpu).abs().mean().item()
            print("patch(IGEV++, AMP YAML, aggregation=True) 256x512: EPE %.3e vs fp32 CPU (unpatched AMP %.3e)" % (e_got, e_amp))
            assert got.dtype == amp.dtype and e_got <= max(2 * e_amp, 1e-2)
    assert torch.isfinite(got).all() and got.shape == want_cpu.shape


def test_aggregation_guard(osb):
    """The hourglass overrides follow the same rule as every override: strict mode refuses training and recording calls,
    strict=False hands them to the reference (gradients intact)."""
    lib, _, _, patch = osb
    a = patch(oigpp.igevpp(seed=9).cuda(), aggregation=True)
    x, feats = _hg_inputs(1, 16, 16, 32, 4)
    xg, fg = x.cuda(), [f.cuda() for f in feats]
    with torch.no_grad():
        before = lib.launch_count()
        a.cost_agg0(xg, fg)
        assert lib.launch_count() == before + 28
    with pytest.raises(RuntimeError, match="CUDA inference only"):
        a.cost_agg1(xg, fg)                                                  # autograd records through the parameters
    c = patch(oigpp.igevpp(seed=9).cuda(), strict=False, aggregation=True)
    before = lib.launch_count()
    c.cost_agg2(xg, fg).mean().backward()
    assert lib.launch_count() == before and c.cost_agg2.conv0.conv.weight.grad is not None
