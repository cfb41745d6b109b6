"""GPU: IGEV++'s instance-normalised hourglasses on the library -- the refusals of the instance-norm entry points (their kernel-level
contract, moments out and normalised input, is in test_cuda_core_contract_gpu.py), the IGEVPPAggregation engine against a reference
hourglass(8) in float64 with its launch sequence pinned, and patch(model, aggregation=True) under both YAMLs against the unpatched
model.  Sorted after the torch.profiler routing suites like the other model-level files."""
import pytest
import torch

from oracle import _reference_shim as shim
from oracle import igevpp as oigpp

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not shim.available(), reason="reference tree (oracle/_ref) not staged")]

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
