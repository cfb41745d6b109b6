"""GPU: MSNet3D on the sm_90a kernels -- the fused MobileV2_Residual_3D block (osb_mbv2_block3d_fwd) against the CPU oracle
(oracle/msnet.py, pinned bit-exactly to the reference) for all seven block configs, MSNet3DAggregation on both routes, and patch()
on the unmodified reference class."""
import copy

import pytest
import torch

from oracle import _reference_shim as shim
from oracle import msnet as oms
from oracle import seeded_init as si

from conftest import load_golden

pytestmark = pytest.mark.gpu

REL_BAR = 1e-5                  # max |err| / max |want|
EPE_BAR = 1e-3                  # px

# (Cin, Chid, Cout, stride): every MobileV2_Residual_3D config MSNet3D builds
CONFIGS = [(40, 120, 32, 1), (32, 96, 32, 1), (32, 64, 32, 1), (32, 64, 64, 2), (64, 128, 64, 1), (64, 128, 128, 2),
           (128, 256, 128, 1)]


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, ops
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return _lib, ops


def rnd(seed, *shape):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def block(cin, chid, cout, stride, seed, shift1=None):
    m = oms.MobileV2Residual3D(cin, cout, stride, chid / cin).eval()
    sd = si.seeded_state_dict(m.state_dict(), seed=seed)
    if shift1 is not None:                      # BN1 bias such that relu6(shift1) is ~3: a wrongly padded halo shows as O(1) errors
        sd["conv.1.bias"] = torch.full_like(sd["conv.1.bias"], shift1)
    m.load_state_dict(sd)
    assert m.conv[0].out_channels == chid
    return m


def rel_err(got, want):
    return ((got - want).abs().max() / want.abs().max()).item()


def to_cl(t):
    return t.permute(0, 2, 3, 4, 1).contiguous()


def run_block(m, x, residual=None, in_cl=False, out_cl=False):
    from openstereo_b200.aggregation import _MBV2Block3D
    eng = _MBV2Block3D(copy.deepcopy(m).cuda(), "block")
    xin = to_cl(x) if in_cl else x
    res = None if residual is None else (to_cl(residual) if out_cl else residual)
    with torch.no_grad():
        y = eng(xin.cuda(), None if res is None else res.cuda(), in_ndhwc=in_cl, out_ndhwc=out_cl).cpu()
    return y.permute(0, 4, 1, 2, 3) if out_cl else y


# ------------------------------------------------------------------------------------------------ the block kernel
@pytest.mark.parametrize("cfg", CONFIGS, ids=lambda c: "%d-%d-%d-s%d" % c)
@pytest.mark.parametrize("dhw", [(7, 9, 37), (8, 10, 36)], ids=["odd", "even"])
def test_block_vs_oracle(osb, cfg, dhw):
    cin, chid, cout, stride = cfg
    m = block(cin, chid, cout, stride, seed=sum(cfg))
    x = rnd(1, 2, cin, *dhw)
    with torch.no_grad():
        want = m(x)
    got = run_block(m, x)
    err = rel_err(got, want)
    print("mbv2_block3d %s D,H,W=%s: max rel err %.2e" % (cfg, dhw, err))
    assert got.shape == want.shape and err <= REL_BAR


@pytest.mark.parametrize("cfg", [(32, 96, 32, 1), (32, 64, 64, 2), (128, 256, 128, 1)], ids=lambda c: "%d-%d-%d-s%d" % c)
@pytest.mark.parametrize("in_cl,out_cl", [(False, True), (True, True), (True, False)])
@pytest.mark.parametrize("with_res", [False, True])
def test_block_layouts_and_residual(osb, cfg, in_cl, out_cl, with_res):
    cin, chid, cout, stride = cfg
    m = block(cin, chid, cout, stride, seed=7)
    x = rnd(2, 2, cin, 5, 11, 19)
    with torch.no_grad():
        want = m(x)
    res = rnd(3, *want.shape) if with_res else None
    if with_res:
        want = want + res
    got = run_block(m, x, res, in_cl, out_cl)
    assert got.shape == want.shape and rel_err(got, want) <= REL_BAR


@pytest.mark.parametrize("cfg", [(40, 120, 32, 1), (32, 64, 64, 2), (64, 128, 128, 2)], ids=lambda c: "%d-%d-%d-s%d" % c)
def test_hidden_padding_is_zero(osb, cfg):
    """BN1's shift near +3 makes relu6(shift1) ~ 3 everywhere: zero-padding the INPUT instead of the hidden tensor would put O(1)
    errors on every border voxel."""
    cin, chid, cout, stride = cfg
    m = block(cin, chid, cout, stride, seed=11, shift1=3.0)
    x = rnd(4, 1, cin, 6, 7, 13) * 0.1
    with torch.no_grad():
        want = m(x)
    got = run_block(m, x)
    assert rel_err(got, want) <= REL_BAR


@pytest.mark.parametrize("cfg", [(32, 96, 32, 1), (64, 128, 64, 1)], ids=lambda c: "%d-%d-%d-s%d" % c)
@pytest.mark.parametrize("cl", [False, True])
def test_block_use_res_connect_forced(osb, cfg, cl):
    cin, chid, cout, stride = cfg
    m = block(cin, chid, cout, stride, seed=13)
    m.use_res_connect = True
    x = rnd(5, 2, cin, 7, 9, 37)
    with torch.no_grad():
        want = m(x)
        assert not torch.equal(want, m.conv(x))
    got = run_block(m, x, in_cl=cl, out_cl=cl)
    assert rel_err(got, want) <= REL_BAR


def test_block_golden(osb):
    g = load_golden("msnet_block")
    for i, cfg in enumerate(((40, 120, 32, 1), (32, 64, 64, 2))):
        m = block(*cfg, seed=g["seed%d" % i])
        got = run_block(m, g["x%d" % i])
        assert rel_err(got, g["out%d" % i]) <= REL_BAR


# ------------------------------------------------------------------------------------------------ aggregation engine
def _aggregation(seed):
    m = oms.Aggregation().eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=seed, scale=oms.MSNET3D_SCALE))
    return m


def _check_engine(osb, shape, expect_deconv, seed=20):
    _, ops = osb
    from openstereo_b200.aggregation import MSNet3DAggregation
    m = _aggregation(seed)
    vol = rnd(seed + 1, *shape)
    with torch.no_grad():
        want = m.logits(vol)
        eng = MSNet3DAggregation(m.cuda())
        ops.profile_start()
        got = eng.logits(vol.cuda())
        torch.cuda.synchronize()
        prof = ops.profile_stop()
    err = rel_err(got.cpu(), want)
    print("MSNet3DAggregation %s: max rel err %.2e, launches %s" % (shape, err, {k: len(v) for k, v in prof.items()}))
    assert got.shape == want.shape and err <= REL_BAR
    assert len(prof["osb_mbv2_block3d_fwd"]) == 22
    assert len(prof.get(expect_deconv, [])) == 6
    return prof


def test_engine_ncdhw_route(osb):
    prof = _check_engine(osb, (1, 40, 48, 16, 32), "osb_deconv3d_bn_act_fwd")
    assert "osb_deconv3d_k3_tc_fwd" not in prof


def test_engine_channels_last_route(osb):
    prof = _check_engine(osb, (2, 40, 48, 64, 128), "osb_deconv3d_k3_tc_fwd")
    assert "osb_ncdhw_to_ndhwc" not in prof                          # the first block reads the NCDHW volume itself


def test_engine_general_width_route(osb):
    _check_engine(osb, (1, 40, 48, 128, 240), "osb_deconv3d_k3_tc_fwd")


def test_engine_without_tensor_cores(osb):
    from openstereo_b200 import aggregation as agg
    saved, agg.USE_TENSOR_CORES = agg.USE_TENSOR_CORES, False
    try:
        prof = _check_engine(osb, (2, 40, 48, 64, 128), "osb_deconv3d_bn_act_fwd")
    finally:
        agg.USE_TENSOR_CORES = saved
    assert not any("_tc_" in k for k in prof)


def test_engine_disparity(osb):
    from openstereo_b200.aggregation import MSNet3DAggregation
    m = _aggregation(21)
    vol = rnd(22, 1, 40, 12, 16, 32)
    with torch.no_grad():
        want = m(vol, 64, 128)
        got = MSNet3DAggregation(m.cuda())(vol.cuda(), 64, 128).cpu()
    assert got.shape == want.shape and (got - want).abs().mean().item() <= EPE_BAR


# ------------------------------------------------------------------------------------------------ patch() on the reference
needs_ref = pytest.mark.skipif(not shim.available(), reason="reference tree (oracle/_ref) not staged")


def msnet3d(seed=1):
    cfg = shim.load_cfg("cfgs/msnet/msnet3d_sceneflow.yaml").MODEL
    m = oms.load_reference("stereo.modeling.models.msnet.MSNet3D").MSNet3D(cfg).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=seed, scale=oms.MSNET3D_SCALE))
    return m


def inputs(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return {"left": torch.randn(b, 3, h, w, generator=g), "right": torch.randn(b, 3, h, w, generator=g)}


def patched_vs_reference(lib, b, h, w, seed):
    """-> (EPE px, reference disparity std): the reference on the CPU vs patch() on the GPU."""
    from openstereo_b200.patch import patch
    m = msnet3d()
    keys = list(m.state_dict().keys())
    x = inputs(b, h, w, seed)
    with torch.no_grad():
        want = m(dict(x))["disp_pred"]
        patch(m.cuda())
        before = lib.launch_count()
        got = m({k: v.cuda() for k, v in x.items()})["disp_pred"]
        launches = lib.launch_count() - before
    assert list(m.state_dict().keys()) == keys
    assert got.shape == want.shape and got.is_cuda and launches >= 22 + 6 + 4
    epe = (got.cpu() - want).abs().mean().item()
    print("patch(MSNet3D) B=%d %dx%d: EPE %.3e px vs the reference on the CPU (disp std %.2f), %d launches"
          % (b, h, w, epe, want.std().item(), launches))
    return epe, want.std().item()


@needs_ref
def test_patch_msnet3d_256x512(osb):
    lib, _ = osb
    epe, std = patched_vs_reference(lib, 1, 256, 512, 30)
    assert std > 1 and epe <= EPE_BAR


@needs_ref
def test_patch_msnet3d_golden(osb):
    from openstereo_b200.patch import patch
    g = load_golden("msnet3d_model")
    m = patch(msnet3d(g["weight_seed"]).cuda())
    with torch.no_grad():
        got = m({"left": g["left"].cuda(), "right": g["right"].cuda()})["disp_pred"].cpu()
    assert (got - g["disp"]).abs().mean().item() <= EPE_BAR


@needs_ref
def test_patch_msnet3d_delegates_recording_and_training(osb):
    """strict=False: a CUDA call that autograd records, or a training call, runs the reference's own forward (no launch of this
    library) with gradients matching the unpatched model's; strict=True refuses both loudly."""
    lib, _ = osb
    from openstereo_b200.patch import patch
    x = {k: v.cuda() for k, v in inputs(1, 64, 128, 31).items()}
    ref = msnet3d().cuda()
    m = patch(msnet3d().cuda(), strict=False)
    for train in (False, True):
        ref.train(train), m.train(train)
        for mod in (ref, m):
            mod.zero_grad()
        before = lib.launch_count()
        out = m(dict(x))["disp_pred"]
        assert lib.launch_count() == before and out.requires_grad
        out.mean().backward()
        ref(dict(x))["disp_pred"].mean().backward()
        pairs = [(n, p.grad, q.grad) for (n, p), (_, q) in zip(m.named_parameters(), ref.named_parameters())]
        assert all((gp is None) == (gq is None) for _, gp, gq in pairs)
        gp = torch.cat([a.flatten() for _, a, b in pairs if b is not None])
        gq = torch.cat([b.flatten() for _, a, b in pairs if b is not None])
        # the reference's own backward is not bit-reproducible on the GPU (cuDNN weight gradients and the trilinear backward
        # accumulate in a run-dependent order, and ReLU6 clips flip on near-ties): compare the whole gradient in the L2 norm
        assert ((gp - gq).norm() / gq.norm()).item() <= 1e-2
    strict = patch(msnet3d().cuda())
    with pytest.raises(RuntimeError, match="CUDA inference only"):
        strict(dict(x))
    with pytest.raises(RuntimeError, match="CUDA inference only"):
        strict.train()(dict(x))
