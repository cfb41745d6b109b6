"""GPU: AANet on the library -- the reference's own DCNv2 extension against the torchvision oracle, the modulated deformable gather
mode of the general-width wgmma convolutions against float64 (every packed width, strides 1 and 2, widths that are not multiples
of the tile, store bounds inside sentinels, determinism, the instantiation it reports, refusals that launch nothing), the
bottleneck engine against its module, and the whole patched model against the unpatched one with offsets that leave the image."""
import pytest
import torch

from oracle import _reference_shim as shim
from oracle import aanet as oa

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not shim.available() or not oa.extension_available(),
                                                  reason="reference tree or its deform_conv_cuda build (oracle/_ref) not staged")]

TOL = 1e-5          # per element, of the summed |products| feeding it (the tensor-core contract's bar)


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, ops
    from openstereo_b200.patch import patch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return _lib, ops, patch


def _case(b, cin, cout, h, w, stride, dil, dg, seed, spread=4.0):
    g = torch.Generator().manual_seed(seed)
    ho, wo = (h + 2 * dil - 2 * dil - 1) // stride + 1, (w + 2 * dil - 2 * dil - 1) // stride + 1
    x = torch.randn(b, cin, h, w, generator=g)
    off = torch.randn(b, dg * 18, ho, wo, generator=g) * spread
    off[:, 0::7] = torch.randint(-3, 4, off[:, 0::7].shape, generator=g).float()     # integer offsets
    off[0, :2, 0, :3] = torch.tensor([[-1e3, 0.0, 2.5e3], [3.0, -1e3, 0.5]])          # beyond every edge
    logits = torch.randn(b, dg * 9, ho, wo, generator=g) * 2
    wgt = torch.randn(cout, cin, 3, 3, generator=g) / (3 * cin ** 0.5)
    bias = torch.randn(cout, generator=g) * 0.1
    return x, off, logits, wgt, bias, (ho, wo)


def _fp32_positions(off, stride, pad, dil):
    """The offsets as the kernels (this library's and the reference's) apply them: each sample position is the fp32 sum of the
    integer tap position and the offset, so a float64 oracle fed these offsets samples the same points."""
    b, c, ho, wo = off.shape
    ys = torch.arange(ho, dtype=torch.float64).view(1, 1, ho, 1) * stride - pad
    xs = torch.arange(wo, dtype=torch.float64).view(1, 1, 1, wo) * stride - pad
    out = off.double().clone()
    for tap in range(9):
        kh, kw = divmod(tap, 3)
        for base, k in ((ys + kh * dil, 0), (xs + kw * dil, 1)):
            sl = out[:, k + 2 * tap::18]
            sl.copy_((base.float() + off[:, k + 2 * tap::18].float()).double() - base)
    return out


def _bar(x, off, mask, wgt, stride, pad, dil):
    return oa.modulated_deform_conv(x.abs().double(), off.double(), mask.abs().double(), wgt.abs().double(), None, stride, pad, dil)


@pytest.mark.parametrize("stride", [1, 2])
def test_reference_extension_equals_torchvision_oracle(stride):
    ref = oa.load_reference("stereo.libs.AANet.deform_conv")
    x, off, logits, wgt, bias, _ = _case(2, 32, 32, 13, 37, stride, 2, 2, seed=3 + stride)
    mask = torch.sigmoid(logits)
    dev = torch.device("cuda")
    with torch.no_grad():
        got = ref.modulated_deform_conv(x.to(dev), off.to(dev), mask.to(dev), wgt.to(dev), bias.to(dev), stride, 2, 2, 1, 2).cpu()
    want = oa.modulated_deform_conv(x.double(), _fp32_positions(off, stride, 2, 2), mask.double(), wgt.double(), bias.double(),
                                    stride, 2, 2)
    bar = _bar(x, off, mask, wgt, stride, 2, 2)
    assert ((got.double() - want).abs() <= 1e-5 * bar + 1e-5).all()


# (cout, cin, h, w, stride, dilation, dg): every packed width (16 rides the 32-row instantiation), widths below, at and across
# the 126-column tile step, strides 1 and 2, a 16-channel chunk spanning two deformable groups (cin 16, dg 2)
CASES = [(16, 16, 9, 45, 1, 2, 2), (32, 32, 7, 130, 1, 1, 1), (64, 64, 6, 127, 2, 2, 2), (128, 128, 5, 252, 1, 2, 2),
         (32, 48, 11, 20, 2, 1, 1), (64, 32, 4, 300, 1, 3, 4)]


@pytest.mark.parametrize("cout,cin,h,w,stride,dil,dg", CASES)
def test_gather_mode_against_float64(osb, cout, cin, h, w, stride, dil, dg):
    _, ops, _ = osb
    x, off, logits, wgt, bias, (ho, wo) = _case(2, cin, cout, h, w, stride, dil, dg, seed=cout + w)
    dev = torch.device("cuda")
    mask = torch.sigmoid(logits)
    with torch.no_grad():
        got = ops.modulated_deform_conv(x.to(dev), off.to(dev), mask.to(dev), wgt.to(dev), bias.to(dev), stride, dil, dil, 1, dg)
    assert got.shape == (2, cout, ho, wo) and got.dtype == torch.float32
    assert ops.tc_last_variant() == "tcg<%d,16,128,1,1,1,0>" % ops.mdconv_packed_rows(cout)
    want = oa.modulated_deform_conv(x.double(), _fp32_positions(off, stride, dil, dil), mask.double(), wgt.double(), bias.double(),
                                    stride, dil, dil)
    bar = _bar(x, off, mask, wgt, stride, dil, dil)
    err = (got.cpu().double() - want).abs()
    assert (err <= TOL * bar + 1e-6).all(), "max err %g" % err.max()
    assert ops.tc_overflow_count(dev, reset=True) == 0


@pytest.mark.parametrize("cout,cin,h,w,stride,dil,dg", CASES)
def test_gather_mode_stores_inside_sentinels(osb, cout, cin, h, w, stride, dil, dg):
    """NCHW output (the engine's layout) at the packed width, written into a NaN-filled buffer between sentinel guards: every
    element is written, nothing outside the tensor is, and the values are those of the functional call."""
    _lib, ops, _ = osb
    x, off, logits, wgt, bias, (ho, wo) = _case(2, cin, cout, h, w, stride, dil, dg, seed=cout + w)
    dev = torch.device("cuda")
    rows = ops.mdconv_packed_rows(cout)
    wp = ops.pack_tc_weight_2d(wgt.to(dev), 16, pad_cout_to=rows)
    xn = x.to(dev).permute(0, 2, 3, 1).contiguous()
    off, mask = off.to(dev), torch.sigmoid(logits).to(dev)
    shift = torch.cat((bias, bias.new_zeros(rows - cout))).to(dev)
    n, guard = 2 * rows * ho * wo, 256
    buf = torch.full((n + 2 * guard,), float("nan"), device=dev)
    buf[:guard], buf[-guard:] = 7.0, 7.0
    y = buf[guard:guard + n]
    rc = _lib.lib.osb_mdconv2d_k3_tc_fwd(xn.data_ptr(), off.data_ptr(), off.stride(0), mask.data_ptr(), mask.stride(0), 0,
                                        wp.data.data_ptr(), wp.eff_scale(None).data_ptr(), shift.data_ptr(), y.data_ptr(), 2, cin,
                                        rows, h, w, stride, dil, dil, dg, ops.ACT_NONE, 0, torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert (buf[:guard] == 7).all() and (buf[-guard:] == 7).all() and not torch.isnan(y).any()
    with torch.no_grad():
        want = ops.modulated_deform_conv(x.to(dev), off, mask, wgt.to(dev), bias.to(dev), stride, dil, dil, 1, dg)
    assert torch.equal(y.view(2, rows, ho, wo)[:, :cout], want)
    if rows > cout:                                       # the zero-padded rows: conv 0 + shift 0
        assert (y.view(2, rows, ho, wo)[:, cout:] == 0).all()


def test_double_sigmoid_mask_from_one_offset_conv_output(osb):
    """The engine's call: offsets and mask logits as channel slices of one tensor, 2 * sigmoid applied in the loader, folded BN and
    ReLU, NCHW and NHWC stores inside NaN-filled buffers between sentinels; two launches are bit-identical."""
    _, ops, _ = osb
    x, off, logits, wgt, bias, (ho, wo) = _case(2, 64, 64, 10, 140, 1, 2, 2, seed=11)
    dev = torch.device("cuda")
    om = torch.cat((off, logits), 1).to(dev)
    wp = ops.pack_tc_weight_2d(wgt.to(dev), 16)
    scale, shift = torch.rand(64, device=dev) + 0.5, torch.randn(64, device=dev) * 0.1
    xn = x.to(dev).permute(0, 2, 3, 1).contiguous()
    want = oa.modulated_deform_conv(x.double(), _fp32_positions(off, 1, 2, 2), 2 * torch.sigmoid(logits.double()), wgt.double(),
                                    None, 1, 2, 2)
    want = torch.relu(want * scale.cpu().double().view(1, -1, 1, 1) + shift.cpu().double().view(1, -1, 1, 1))
    bar = _bar(x, off, 2 * torch.sigmoid(logits), wgt, 1, 2, 2) * scale.cpu().double().view(1, -1, 1, 1)
    outs = []
    for _ in range(2):
        y = ops.mdconv2d_k3_tc(xn, om[:, :36], om[:, 36:], wp, scale, shift, 1, 2, 2, 2, ops.ACT_RELU, ops.MASK_DOUBLE_SIGMOID)
        outs.append(y)
    assert torch.equal(outs[0], outs[1])
    assert ((outs[0].cpu().double() - want).abs() <= TOL * bar + 1e-6).all()
    # NHWC store: every element written, no write outside
    n = 2 * ho * wo * 64
    buf = torch.full((n + 2 * 64,), float("nan"), device=dev)
    buf[:64], buf[-64:] = 7.0, 7.0
    y = buf[64:64 + n].view(2, ho, wo, 64)
    rc = _lib_call(osb, xn, om, wp, scale, shift, y, 1)
    assert rc == 0
    torch.cuda.synchronize()
    assert (buf[:64] == 7).all() and (buf[-64:] == 7).all() and not torch.isnan(y).any()
    assert torch.equal(y.permute(0, 3, 1, 2), outs[0])


def _lib_call(osb, xn, om, wp, scale, shift, y, out_nhwc, **kw):
    _lib, ops, _ = osb
    b, h, w, cin = xn.shape
    a = dict(offset=om.data_ptr(), obs=om.stride(0), mask=om.data_ptr() + 36 * om.stride(1) * 4, mbs=om.stride(0), mode=1, cout=wp.cout,
             stride=1, pad=2, dil=2, dg=2, act=ops.ACT_RELU, b=b, cin=cin, h=h, w=w)
    a.update(kw)
    return _lib.lib.osb_mdconv2d_k3_tc_fwd(xn.data_ptr(), a["offset"], a["obs"], a["mask"], a["mbs"], a["mode"], wp.data.data_ptr(),
                                          wp.eff_scale(scale).data_ptr(), shift.data_ptr(), y.data_ptr(), a["b"], a["cin"], a["cout"],
                                          a["h"], a["w"], a["stride"], a["pad"], a["dil"], a["dg"], a["act"], out_nhwc,
                                          torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("kw", [dict(cout=96), dict(cout=16), dict(stride=3), dict(dg=3), dict(cin=24), dict(mode=2),
                                dict(act=4), dict(obs=10), dict(mbs=10), dict(offset=0), dict(pad=-1), dict(dil=0)])
def test_refusals_launch_nothing(osb, kw):
    _lib, ops, _ = osb
    dev = torch.device("cuda")
    x, off, logits, wgt, _, (ho, wo) = _case(1, 64, 64, 6, 40, 1, 2, 2, seed=2)
    om = torch.cat((off, logits), 1).to(dev)
    wp = ops.pack_tc_weight_2d(wgt.to(dev), 16)
    scale, shift = torch.ones(64, device=dev), torch.zeros(64, device=dev)
    y = torch.full((1, 64, ho, wo), 3.0, device=dev)
    before = _lib.lib.osb_launch_count()
    assert _lib_call(osb, x.to(dev).permute(0, 2, 3, 1).contiguous(), om, wp, scale, shift, y, 0, **kw) == 1    # OSB_EINVAL
    assert _lib.lib.osb_launch_count() == before
    torch.cuda.synchronize()
    assert (y == 3).all()


def test_functional_refusals(osb):
    _, ops, _ = osb
    dev = torch.device("cuda")
    x, off, logits, wgt, _, _ = _case(1, 32, 32, 6, 40, 1, 1, 1, seed=4)
    args = [x.to(dev), off.to(dev), torch.sigmoid(logits).to(dev), wgt.to(dev)]
    with pytest.raises(RuntimeError, match="no backward"):
        ops.modulated_deform_conv(args[0].requires_grad_(), *args[1:], None, 1, 1, 1)
    with pytest.raises(ValueError):
        ops.modulated_deform_conv(*[a.detach() for a in args], None, 1, 1, 1, groups=2)
    with pytest.raises(TypeError):
        ops.modulated_deform_conv(args[0].detach().half(), *args[1:], None, 1, 1, 1)


def _inputs(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    left = torch.randn(b, 3, h, w, generator=g)
    right = torch.roll(left, 5, -1) + 0.1 * torch.randn(b, 3, h, w, generator=g)
    return left.cuda(), right.cuda()


def _install_engines(m):
    """Every deformable bottleneck's forward through the gather mode, behind patch()'s guard (patch() itself keeps the reference's
    extension for them)."""
    from openstereo_b200.aanet import DeformBottleneckEngine
    from openstereo_b200.patch import _override
    blocks = [mod for mod in m.modules() if type(mod).__name__ in ("DeformBottleneck", "DeformSimpleBottleneck")]
    for mod in blocks:
        engine = DeformBottleneckEngine(mod)
        _override(mod, "AANet " + type(mod).__name__, True, engine, engine.serves)
    return blocks


@pytest.mark.parametrize("engines", [False, True])
@pytest.mark.parametrize("b,h,w", [(2, 192, 384), (1, 576, 960)])
def test_whole_model_patched_equals_unpatched(osb, b, h, w, engines):
    _, ops, patch = osb
    # offset_conv scaled so that offsets span several pixels and leave the image (the default init zeroes it)
    ref = oa.aanet(offset_scale=30.0).cuda()
    lib = patch(oa.aanet(offset_scale=30.0).cuda())
    if engines:
        assert len(_install_engines(lib)) == 15
    left, right = _inputs(b, h, w, seed=h)
    seen = []
    hook = ref.feature_extractor.layer3[0].conv2.offset_conv.register_forward_hook(lambda mod, i, o: seen.append(o[:, :36].abs().amax()))
    with torch.no_grad():
        want = ref({"left": left, "right": right})
        got = lib({"left": left, "right": right})
    hook.remove()
    assert seen[0] > 8, "offsets must leave a neighbourhood of the tap"
    assert len(got["disp_preds"]) == len(want["disp_preds"])
    for g_, w_ in zip(got["disp_preds"], want["disp_preds"]):
        assert g_.shape == w_.shape and g_.dtype == w_.dtype
        assert (g_ - w_).abs().mean().item() <= 1e-3
    assert (got["disp_pred"] - want["disp_pred"]).abs().mean().item() <= 1e-3
    assert want["disp_pred"].std() > 0.5
    assert ops.tc_overflow_count(left.device, reset=True) == 0


def test_engine_serves_every_deformable_block(osb):
    _, ops, patch = osb
    m = patch(oa.aanet(offset_scale=30.0).cuda())
    from openstereo_b200.aanet import DeformBottleneckEngine
    assert not any("forward" in vars(x) for x in m.modules() if type(x).__name__ in ("DeformBottleneck", "DeformSimpleBottleneck"))
    blocks = _install_engines(m)
    left, right = _inputs(1, 96, 192, seed=1)
    with torch.no_grad():
        feat = m.feature_extractor.conv1(left)
        assert all(DeformBottleneckEngine(blk).serves(feat) for blk in blocks)
    m.train()
    with pytest.raises(RuntimeError, match="CUDA inference only"):
        m({"left": left, "right": right})
