"""GPU: patch()'s routing rule on the module overrides that own parameters, and the rebound scale-4 context_upsample.

A module in eval() mode whose parameters require grad, called with grad enabled on operands that do not (features of a frozen
backbone computed under no_grad), is not a CUDA inference call: the kernels would cut the parameters' gradients.  strict=True
refuses it; strict=False runs the reference's forward, so the parameters get their gradients and the library launches nothing.
The operands are the ones the model itself hands the module in a no_grad forward on CUDA."""
import pytest
import torch

from oracle import _reference_shim as shim
from oracle import cascade as ocas
from oracle import igev_rt as oigrt
from oracle import igevpp as oigpp
from oracle import seeded_init as si

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not shim.available(), reason="reference tree (oracle/_ref) not staged")]

_M = "stereo.modeling.models."


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib
    from openstereo_b200.patch import patch
    return _lib, patch


def _cfg_model(cfg, dotted, cls, **seeding):
    shim.install_timm_stub()
    m = getattr(shim.load(dotted), cls)(shim.load_cfg(cfg).MODEL).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), **seeding))
    return m


def _gwcnet():
    return _cfg_model("cfgs/gwcnet/gwcnet_sceneflow.yaml", _M + "gwcnet.gwcnet", "GwcNet", seed=1, scale=si.GWCNET_SCALE)


def _psmnet():
    return _cfg_model("cfgs/psmnet/psmnet_sceneflow.yaml", _M + "psmnet.psmnet", "PSMNet", seed=1, scale=si.PSMNET_SCALE,
                      keep=si.PSMNET_KEEP)


def _stereobase():
    return _cfg_model("cfgs/stereobase/stereobase_sceneflow.yaml", _M + "stereobase.stereobase_gru", "StereoBase", seed=3,
                      scale={"classifier.weight": 8.0})


def _lightstereo():
    return _cfg_model("cfgs/lightstereo/lightstereo_s_sceneflow.yaml", _M + "lightstereo.lightstereo", "LightStereo", seed=11)


def _igev():
    return _cfg_model("cfgs/igev/igev_sceneflow_amp.yaml", _M + "igev.igev_stereo", "IGEVStereo", seed=12,
                      scale={"classifier.weight": 8.0})


def _cascade(module, scale):
    return lambda: _cfg_model("cfgs/casnet/casnet_psm_sceneflow.yaml", _M + "casnet." + module,
                              "PSMNet" if module == "cas_psm" else "GwcNet", seed=1, scale=scale)


# (model, the overridden module's path); every one owns parameters that the kernels would cut off
CASES = [(_gwcnet, "DispProcessor"), (_psmnet, "CostProcessor"), (_stereobase, "cost_agg"), (_lightstereo, "cost_agg"),
         (oigrt.igev_rt, "cost_agg"), (oigrt.igev_rt, "classifier"), (oigpp.igevpp, "classifier"),
         (_cascade("cas_psm", ocas.CASNET_SCALE), "cost_agg.0"), (_cascade("cas_psm", ocas.CASNET_SCALE), "cost_agg.1"),
         (_cascade("cas_gwc", ocas.CASGWC_SCALE), "cost_agg.0"), (_cascade("cas_gwc", ocas.CASGWC_SCALE), "cost_agg.1")]


class _Captured(Exception):
    pass


def _operands(model, path):
    """The (args, kwargs) the model's no_grad CUDA forward passes to model.<path> on its first call."""
    got = []

    def hook(mod, args, kwargs):
        got.append((args, kwargs))
        raise _Captured                                              # the rest of the forward is not needed

    handle = model.get_submodule(path).register_forward_pre_hook(hook, with_kwargs=True)
    g = torch.Generator().manual_seed(3)
    x = {k: (torch.rand(1, 3, 256, 512, generator=g) * 2 - 1).cuda() for k in ("left", "right")}
    try:
        with torch.no_grad(), pytest.raises(_Captured):
            model(x)
    finally:
        handle.remove()
    return got[0]


def _tensors(x):
    if isinstance(x, torch.Tensor):
        yield x
    elif isinstance(x, (list, tuple)):
        for v in x:
            yield from _tensors(v)
    elif isinstance(x, dict):
        for v in x.values():
            yield from _tensors(v)


@pytest.mark.parametrize("build,path", CASES, ids=["GwcNet", "PSMNet", "StereoBase", "LightStereo", "IGEV-RT-cost_agg",
                                                    "IGEV-RT-classifier", "IGEV++", "CasPSMNet-0", "CasPSMNet-1", "CasGwcNet-0",
                                                    "CasGwcNet-1"])
def test_trainable_module_never_reaches_the_kernels(osb, build, path):
    lib, patch = osb
    strict, loose = patch(build().cuda()), patch(build().cuda(), strict=False)
    args, kwargs = _operands(strict, path)
    assert not any(t.requires_grad for t in _tensors((args, kwargs))) and torch.is_grad_enabled()
    mod = loose.get_submodule(path)
    assert not mod.training and all(p.requires_grad for p in mod.parameters()) and any(True for _ in mod.parameters())
    with pytest.raises(RuntimeError, match="CUDA inference only"):
        strict.get_submodule(path)(*args, **kwargs)
    before = lib.launch_count()
    out = [t for t in _tensors(mod(*args, **kwargs)) if t.requires_grad]
    assert lib.launch_count() == before and out
    sum(t.float().sum() for t in out).backward()
    assert any(p.grad is not None and p.grad.abs().sum() > 0 for p in mod.parameters())


@pytest.mark.parametrize("build", [_lightstereo, _igev])
def test_strict_context_upsample_at_another_scale_runs_the_reference(osb, build):
    """The kernel serves scale 4 only: a CUDA inference call at scale 2 is the reference's, in strict mode too.  LightStereo's
    context_upsample takes a scale; IGEV's takes none and rejects the argument itself."""
    lib, patch = osb
    model = patch(build().cuda())
    rebound = model.forward.__globals__["context_upsample"]
    reference = type(model).forward.__globals__["context_upsample"]
    assert rebound is not reference
    g = torch.Generator().manual_seed(4)
    disp, weights = torch.rand(1, 1, 8, 16, generator=g).cuda(), torch.rand(1, 9, 16, 32, generator=g).cuda()
    with torch.no_grad():
        try:
            want = reference(disp, weights, 2)
        except TypeError as exc:
            want = exc
        before = lib.launch_count()
        if isinstance(want, TypeError):
            with pytest.raises(TypeError, match="positional argument"):
                rebound(disp, weights, 2)
        else:
            assert torch.equal(rebound(disp, weights, 2), want)
        assert lib.launch_count() == before
    assert isinstance(want, TypeError) == (build is _igev)
