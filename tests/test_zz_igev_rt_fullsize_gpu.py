"""GPU: patch() on the unmodified IGEV-RT reference class (igev_rt/igev_rt_stereo.py, IGEVRTtereo) under both YAMLs, whole-model
forwards at 256x512 against the unpatched model on the CPU and on the GPU, per-instance patching and the training / autograd
refusal.  The kernel-level IGEV-RT tests (lookup, engine) are in test_zz_igev_rt_gpu.py; these whole-model runs come last, with the
other full-size model tests."""
import pytest
import torch

from oracle import _reference_shim as shim
from oracle import igev_rt as oigrt

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not shim.available(), reason="reference tree (oracle/_ref) not staged")


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, ops
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return _lib, ops


# ------------------------------------------------------------------------------------------ patch() on the reference class
def _inputs(b, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return {"left": torch.rand(b, 3, h, w, generator=g) * 2 - 1, "right": torch.rand(b, 3, h, w, generator=g) * 2 - 1}


@needs_ref
def test_patch_igev_rt_reference_class(osb):
    """The uniform YAML's model at 256x512: volume, hourglass, classifier, regression, 8 lookups and the up-sampling run in this
    library; the 8 GRU iterations amplify any fp32 reordering, so the bound follows the reference's own GPU-vs-CPU floor."""
    lib, ops = osb
    from openstereo_b200.patch import patch
    m = oigrt.igev_rt()
    x = _inputs(1, 256, 512, 80)
    with torch.no_grad():
        want_cpu = m(dict(x))["disp_pred"]
        m.cuda()
        xg = {k: v.cuda() for k, v in x.items()}
        want_gpu = m(dict(xg))["disp_pred"]
        patch(m)
        m(dict(xg))
        before = lib.launch_count()
        got = m(dict(xg))["disp_pred"]
        launches = lib.launch_count() - before
    e_gpu = (got - want_gpu).abs().mean().item()
    floor = (want_gpu.cpu() - want_cpu).abs().mean().item()
    print("patch(IGEV-RT) 256x512: EPE %.3e vs GPU ref (reference GPU-vs-CPU floor %.3e); %d launches" % (e_gpu, floor, launches))
    head = 2 if ops.conv3d_tc_kc(32, 1, 128) == 32 else 1
    # volume + hourglass (25) + classifier + regression + pyramid level + 8 lookups + convex up-sampling
    assert launches == 1 + 25 + head + 1 + 1 + 8 + 1
    assert got.shape == want_gpu.shape and got.dtype == torch.float32 and torch.isfinite(got).all()
    assert want_cpu.std() > 1.0
    assert e_gpu <= max(10 * floor, 1e-2)


@needs_ref
def test_patch_igev_rt_amp_yaml(osb):
    """The AMP YAML: fp16 reaches the patched calls, which compute in fp32 and hand fp16 back.  The patched model stays within
    twice the unpatched AMP model's own distance to the fp32 CPU reference."""
    from openstereo_b200.patch import patch
    ref = oigrt.igev_rt(oigrt.AMP_YAML)
    x = _inputs(1, 256, 512, 81)
    with torch.no_grad():
        want_cpu = ref(dict(x))["disp_pred"]
        ref.cuda()
        xg = {k: v.cuda() for k, v in x.items()}
        amp = ref(dict(xg))["disp_pred"]
        pm = patch(oigrt.igev_rt(oigrt.AMP_YAML).cuda())
        got = pm(dict(xg))["disp_pred"]
    e_amp = (amp.cpu() - want_cpu).abs().mean().item()
    e_got = (got.cpu() - want_cpu).abs().mean().item()
    print("patch(IGEV-RT, AMP YAML) 256x512: EPE %.3e vs fp32 CPU (unpatched AMP %.3e)" % (e_got, e_amp))
    assert torch.isfinite(got).all() and got.shape == amp.shape
    assert e_got <= max(2 * e_amp, 1e-2)


@needs_ref
def test_patch_igev_rt_is_per_instance_and_refuses_training(osb):
    lib, _ = osb
    from openstereo_b200.patch import patch
    a, b = patch(oigrt.igev_rt(seed=9).cuda()), oigrt.igev_rt(seed=9).cuda()
    xg = {k: v.cuda() for k, v in _inputs(1, 64, 128, 82).items()}
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
    # strict=False: a training call runs the reference's code, gradients intact
    c = patch(oigrt.igev_rt(seed=9).cuda(), strict=False).train()
    before = lib.launch_count()
    out = c(dict(xg))
    assert lib.launch_count() == before
    (out["init_disp"].mean() + out["disp_pred"].mean()).backward()          # the GRU loop detaches disp: init_disp carries the head
    assert c.classifier.weight.grad is not None and c.cost_agg.conv1[0].conv.weight.grad is not None
