"""GPU: the ConvGRU of IGEV-Stereo / StereoBase on the wgmma convolutions (gru.py, DESIGN.md section 4.15) -- the engine against
the reference ConvGRU in float64, the delegation of shapes without a kernel, every new epilogue mode at the C ABI with store
bounds, fp16 under autocast, the launch sequence, the fp16-range guard, whole models against the unpatched reference, and the
training / autograd refusal.  Sorted after the torch.profiler routing suites like the other model-level files."""
import pytest
import torch

from oracle import _reference_shim as shim
from oracle import seeded_init as si

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not shim.available(), reason="reference tree (oracle/_ref) not staged")]

EPE_BAR = 1e-3
TOL = 1e-5          # per element, of the summed |products| feeding it (the other wgmma layers' bar)


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, gru, ops
    from openstereo_b200.patch import patch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return _lib, gru, ops, patch


def _convgru_cls():
    return shim.load("stereo.modeling.models.igev.update").ConvGRU


def _cell(cx, seed):
    torch.manual_seed(seed)
    return _convgru_cls()(128, cx).eval()


def _operands(b, cx_parts, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    hid = torch.tanh(torch.randn(b, 128, h, w, generator=g) * 2)
    ctx = torch.randn(b, 384, h, w, generator=g)                        # cz, cr, cq: split() views, as the models pass them
    xs = [torch.randn(b, c, h, w, generator=g) for c in cx_parts]
    return hid, list(ctx.split(128, 1)), xs


def _magnitude(cell, hid, cz, cr, cq, xs):
    """Per element, the sum of |products| (and |bias| + |context|) entering each gate's pre-activation, float64."""
    import torch.nn.functional as F
    a = lambda t: t.double().abs()
    hx = torch.cat([a(hid)] + [a(t) for t in xs], 1)
    m = sum(F.conv2d(hx, a(c.weight), a(c.bias), padding=1) for c in (cell.convz, cell.convr, cell.convq))
    return m + a(cz) + a(cr) + a(cq)


@pytest.mark.parametrize("cx_parts", [(128, 128), (128, 128), (128,)], ids=["gru04", "gru08", "gru16"])
@pytest.mark.parametrize("w", [128, 64, 32, 240, 60])
@pytest.mark.parametrize("b", [1, 3])
def test_engine_against_reference_fp64(osb, cx_parts, w, b):
    _, gru, ops, _ = osb
    cell = _cell(sum(cx_parts), 7 + w + b)
    hid, (cz, cr, cq), xs = _operands(b, cx_parts, 5, w, w * 10 + b)
    with torch.no_grad():
        want = cell.double()(hid.double(), cz.double(), cr.double(), cq.double(), *[t.double() for t in xs])
        mag = _magnitude(cell, hid, cz, cr, cq, xs)
        cell = cell.float().cuda()
        eng = gru.ConvGRUEngine(cell)
        assert eng.serves(hid, xs)
        ctx = torch.cat([cz, cr, cq], 1).cuda()
        gz, gr, gq = ctx.split(128, 1)
        assert b == 1 or not gz.is_contiguous()
        got = eng(hid.cuda(), gz, gr, gq, *[t.cuda() for t in xs])
        torch.cuda.synchronize()
    assert got.shape == want.shape and got.dtype == torch.float32
    err = (got.cpu().double() - want).abs()
    assert torch.isfinite(got).all() and (err <= TOL * mag + 1e-6).all(), "max err %g, max err/mag %g" % (err.max(), (err / mag).max())
    assert ops.tc_overflow_count(reset=True) == 0


def test_narrow_width_runs_the_reference(osb):
    """W = 16 < OSB_TC_MIN_WIDTH: no kernel serves it, the patched module runs the reference's own forward (no library launch)."""
    lib, _, _, _ = osb
    from openstereo_b200.patch import _override_convgru
    from openstereo_b200.gru import ConvGRUEngine
    cell = _cell(128, 3).cuda()
    hid, ctx, xs = [t for t in _operands(2, (128,), 8, 16, 4)]
    args = [hid.cuda()] + [c.cuda() for c in ctx] + [t.cuda() for t in xs]
    with torch.no_grad():
        want = cell(*args)
        _override_convgru(cell, ConvGRUEngine(cell), strict=True)
        before = lib.launch_count()
        got = cell(*args)
        assert lib.launch_count() == before
    assert torch.equal(got, want)


def _sentinel_buf(n, dev):
    pad = 64
    buf = torch.full((n + 2 * pad,), 12345.0, device=dev)
    buf[pad:pad + n] = float("nan")
    return buf, pad


@pytest.mark.parametrize("w,variant", [(128, "tcg<128,16,128,1,1,0,0>"), (32, "tcg<128,16,32,1,1,0,0>"),
                                       (160, "tcg<128,16,128,1,1,1,0>")])
@pytest.mark.parametrize("mode", ["sigmoid", "tanh", "mul", "blend", "bstride", "blend_nhwc"])
def test_epilogue_modes_c_abi(osb, w, variant, mode):
    """Each new mode on every Cout = 128 instantiation: every output element written (NaN-filled buffer), no sentinel touched, and
    the value equal to the mode's formula on a float64 reference conv."""
    import torch.nn.functional as F
    lib, gru, ops, _ = osb
    dev = torch.device("cuda")
    b, cin, h = 2, 64, 6
    g = torch.Generator().manual_seed(w)
    x = torch.randn(b, cin, h, w, generator=g)
    wt, bias = torch.randn(128, cin, 3, 3, generator=g) * 0.05, torch.randn(128, generator=g)
    wide = torch.randn(b, 384, h, w, generator=g)
    res = wide[:, 128:256]                                                   # NCHW view, batch stride 384 H W
    m, z, hh = (torch.rand(b, h, w, 128, generator=g) for _ in range(3))
    w5 = torch.zeros(128, cin, 3, 3, 3)
    w5[:, :, 1] = wt
    tw = ops.pack_tc_weight(w5.cuda(), 16)
    xn = x.permute(0, 2, 3, 1).contiguous().cuda()
    pre = F.conv2d(x.double(), wt.double(), bias.double(), padding=1)       # (B, 128, H, W)
    kw = dict(act=ops.ACT_NONE, mul=None, z=None, hh=None, res=None, res_nhwc=1, out_nhwc=1, rbs=0)
    if mode == "sigmoid":
        kw.update(act=ops.ACT_SIGMOID, res=res.permute(0, 2, 3, 1).contiguous())
        want = torch.sigmoid(pre + res.double())
    elif mode == "tanh":
        kw.update(act=ops.ACT_TANH, out_nhwc=0)
        want = torch.tanh(pre)
    elif mode == "mul":
        kw.update(act=ops.ACT_SIGMOID, mul=m)
        want = torch.sigmoid(pre) * m.permute(0, 3, 1, 2).double()
    elif mode in ("blend", "blend_nhwc"):
        kw.update(act=ops.ACT_TANH, z=z, hh=hh, out_nhwc=int(mode == "blend_nhwc"))
        zz, hd = z.permute(0, 3, 1, 2).double(), hh.permute(0, 3, 1, 2).double()
        want = hd + zz * (torch.tanh(pre) - hd)
    else:
        kw.update(res_nhwc=0, res="view", rbs=384 * h * w)
        want = pre + res.double()
    wide_g = wide.cuda()
    r = kw["res"]
    r = wide_g[:, 128:256] if isinstance(r, str) else (None if r is None else r.cuda())
    n = b * 128 * h * w
    buf, pad = _sentinel_buf(n, dev)
    y = buf[pad:pad + n]
    keep = [None if kw[k] is None else kw[k].cuda() for k in ("mul", "z", "hh")]   # alive until the kernel has run
    bias_g, scale_g = bias.cuda(), tw.eff_scale(None)
    lib.call("osb_conv2d_k3_tc_gru_fwd", xn.data_ptr(), tw.data.data_ptr(), scale_g.data_ptr(), bias_g.data_ptr(),
             None if r is None else r.data_ptr(), *[None if t is None else t.data_ptr() for t in keep],
             y.data_ptr(), b, cin, 128, h, w, kw["act"], kw["out_nhwc"], kw["res_nhwc"], kw["rbs"], torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert ops.tc_last_variant() == variant
    assert torch.isfinite(y).all(), "unwritten output elements"
    assert (buf[:pad] == 12345.0).all() and (buf[pad + n:] == 12345.0).all(), "store outside the output"
    got = (y.view(b, h, w, 128).permute(0, 3, 1, 2) if kw["out_nhwc"] else y.view(b, 128, h, w)).cpu().double()
    mag = F.conv2d(x.double().abs(), wt.double().abs(), bias.double().abs(), padding=1) + 1
    assert ((got - want).abs() <= TOL * mag).all(), (got - want).abs().max()


def test_slice_pack_writes_its_channels_only(osb):
    lib, _, ops, _ = osb
    g = torch.Generator().manual_seed(1)
    parts = [torch.randn(2, c, 5, 37, generator=g).cuda() for c in (128, 96, 32)]
    got = ops.nchw_to_nhwc_cat(parts)
    assert torch.equal(got, torch.cat(parts, 1).permute(0, 2, 3, 1))
    y = torch.full((2, 5, 37, 300), 7.0, device="cuda")
    lib.call("osb_ncdhw_to_ndhwc_slice", parts[1].data_ptr(), y.data_ptr(), 2, 96, 1, 5, 37, 300, 150, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert torch.equal(y[..., 150:246], parts[1].permute(0, 2, 3, 1))
    assert (y[..., :150] == 7).all() and (y[..., 246:] == 7).all()


def test_fp16_under_autocast(osb):
    """The AMP YAML hands fp16 tensors in: the engine computes in fp32 and returns fp16, close to the fp32 reference."""
    _, _, _, patch = osb
    from openstereo_b200.patch import _override_convgru
    from openstereo_b200.gru import ConvGRUEngine
    cell = _cell(256, 5).cuda()
    hid, ctx, xs = _operands(2, (128, 128), 8, 160, 6)
    with torch.no_grad():
        want = cell(hid.cuda(), *[c.cuda() for c in ctx], *[t.cuda() for t in xs])
        _override_convgru(cell, ConvGRUEngine(cell), strict=True)
        with torch.autocast("cuda", dtype=torch.float16):
            got = cell(hid.cuda().half(), *[c.cuda().half() for c in ctx], *[t.cuda().half() for t in xs])
    assert got.dtype == torch.float16
    assert (got.float() - want).abs().max().item() <= 5e-3


@pytest.mark.parametrize("w,variant", [(128, "tcg<128,16,128,1,1,0,0>"), (32, "tcg<128,16,32,1,1,0,0>"),
                                       (80, "tcg<128,16,128,1,1,1,0>")])
def test_launch_sequence(osb, w, variant):
    """One call = one channels-last pack of h, one per x_list tensor, and six convolutions on one instantiation."""
    lib, gru, ops, _ = osb
    cell = _cell(256, 2).cuda()
    eng = gru.ConvGRUEngine(cell)
    hid, ctx, xs = _operands(1, (128, 128), 4, w, 3)
    args = [hid.cuda()] + [c.cuda() for c in ctx] + [t.cuda() for t in xs]
    with torch.no_grad():
        eng(*args)                                                          # packs the weights
        ops.profile_start()
        before = lib.launch_count()
        eng(*args)
        launches = lib.launch_count() - before
        prof = ops.profile_stop()
    assert launches == 1 + 2 + 6
    assert {k: len(v) for k, v in prof.items()} == {"osb_ncdhw_to_ndhwc_slice": 3, "osb_conv2d_k3_tc_gru_fwd": 6}
    assert ops.tc_last_variant() == variant


def test_overflow_monitor_raises(osb):
    _, gru, ops, _ = osb
    cell = _cell(128, 9).cuda()
    eng = gru.ConvGRUEngine(cell)
    hid, ctx, xs = _operands(1, (128,), 4, 64, 8)
    args = [hid.cuda()] + [c.cuda() for c in ctx]
    ops.tc_overflow_count(reset=True)
    with torch.no_grad():
        eng(*args, xs[0].cuda() * 1e4)                                      # |x| far beyond 4094
        torch.cuda.synchronize()
        with pytest.raises(RuntimeError, match="fp16 range"):
            eng(*args, xs[0].cuda())
        torch.cuda.synchronize()
    assert ops.tc_overflow_count(reset=True) == 0                          # the monitor reset the counter when it raised


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


@pytest.mark.parametrize("name,build,calls", [("IGEVStereo", _igev, 32 * 3), ("StereoBase", _stereobase, 32 * 3)])
def test_whole_model_against_unpatched(osb, name, build, calls):
    """256x512 through the reference classes and patch(): the GRUs ran on the library (six convolutions per call, at least one call
    per GRU and iteration), and disp_pred stays within the bar test_patch_gpu.py sets for these recurrent models."""
    lib, _, ops, patch = osb
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
    n = len(prof.get("osb_conv2d_k3_tc_gru_fwd", []))
    e_gpu = (got - want_gpu).abs().mean().item()
    e_cpu = (got.cpu() - want_cpu).abs().mean().item()
    floor = (want_gpu.cpu() - want_cpu).abs().mean().item()
    print("patch(%s) 256x512 with the GRUs: EPE %.3e vs GPU ref, %.3e vs CPU ref (floor %.3e); %d GRU convolutions"
          % (name, e_gpu, e_cpu, floor, n))
    assert n % 6 == 0 and n >= 6 * calls
    assert torch.isfinite(got).all()
    assert e_gpu <= max(10 * floor, 1e-2) and e_cpu <= max(10 * floor, 1e-2)


def test_training_and_autograd_never_reach_the_kernels(osb):
    lib, _, _, _ = osb
    from openstereo_b200.patch import _override_convgru
    from openstereo_b200.gru import ConvGRUEngine
    hid, ctx, xs = _operands(1, (128,), 4, 64, 2)
    args = [hid.cuda()] + [c.cuda() for c in ctx] + [t.cuda() for t in xs]
    loose, strict = _cell(128, 1).cuda(), _cell(128, 1).cuda()
    _override_convgru(loose, ConvGRUEngine(loose), strict=False)
    _override_convgru(strict, ConvGRUEngine(strict), strict=True)
    before = lib.launch_count()
    out = loose(*args)                                                      # grad enabled, parameters require grad
    assert out.requires_grad
    out.sum().backward()
    assert loose.convz.weight.grad is not None
    loose.train()
    with torch.no_grad():
        loose(*args)
    assert lib.launch_count() == before
    with pytest.raises(RuntimeError, match="CUDA inference only"):
        strict(*args)
    strict.train()
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA inference only"):
        strict(*args)
