"""CPU: patch(model, amp=True) -- which models take it, what it installs, that every update-block engine receives the flag -- and the
C ABI of the autocast-precision entry points (osb_conv2d_k3_tc_prec_fwd, osb_conv2d_k3_tc_gru_prec_fwd)."""
import ctypes
import os
import re

import pytest
import torch

from oracle import _reference_shim as shim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not shim.available(), reason="reference tree not present")
_M = "stereo.modeling.models."


@pytest.fixture(scope="module")
def native():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib
    return _lib


def _cfg_model(cfg, dotted, cls):
    shim.install_timm_stub()
    return getattr(shim.load(dotted), cls)(shim.load_cfg(cfg).MODEL)


def _oracle(name, fn, **kw):
    def build():
        import importlib
        return getattr(importlib.import_module("oracle." + name), fn)(**kw)
    return build


AMP_MODELS = {
    "StereoBase": lambda: _cfg_model("cfgs/stereobase/stereobase_sceneflow.yaml", _M + "stereobase.stereobase_gru", "StereoBase"),
    "IGEVStereo": lambda: _cfg_model("cfgs/igev/igev_sceneflow_amp.yaml", _M + "igev.igev_stereo", "IGEVStereo"),
    "IGEV++": _oracle("igevpp", "igevpp"),
    "MonSter": _oracle("monster", "monster"),
}
_UPDATE_BLOCKS = {"StereoBase": ("update_block",), "IGEVStereo": ("update_block",), "IGEV++": ("update_block",),
                  "MonSter": ("update_block", "update_block_mix_stereo", "update_block_mix_mono")}


def _instance_attributes(model):
    return {"%s.%s" % (path, name) if path else name for path, sub in model.named_modules() for name in vars(sub)}


def _engines(model):
    """Every update-block engine the patch installed: the engine a module's guarded forward closes over."""
    from openstereo_b200.update import _BlockEngine
    out = []
    for _, sub in model.named_modules():
        fwd = vars(sub).get("forward")
        for cell in getattr(fwd, "__closure__", None) or ():
            try:
                v = cell.cell_contents
            except ValueError:
                continue
            if isinstance(v, _BlockEngine):
                out.append(v)
    return out


@needs_ref
@pytest.mark.parametrize("name", sorted(AMP_MODELS))
def test_amp_accepted_installs_the_same_overrides_and_reaches_every_engine(name):
    from openstereo_b200.patch import patch
    plain, amp = AMP_MODELS[name]().eval(), AMP_MODELS[name]().eval()
    assert patch(plain) is plain and patch(amp, amp=True) is amp
    assert _instance_attributes(amp) == _instance_attributes(plain)
    e_plain, e_amp = _engines(plain), _engines(amp)
    per_block = 9 if name == "IGEV++" else 6                   # gru04/08/16, encoder, disp_head, mask_feat_4 (+ geo_encoder0..2)
    assert len(e_amp) == len(e_plain) == per_block * len(_UPDATE_BLOCKS[name])
    assert all(e.amp for e in e_amp) and not any(e.amp for e in e_plain)
    assert {type(e) for e in e_amp} == {type(e) for e in e_plain}
    # outside autocast an amp engine asks for the fp32-accurate product
    assert {e._precision() for e in e_amp} == {"fp32"}


@needs_ref
def test_amp_combines_with_igevpp_aggregation():
    from openstereo_b200.patch import patch
    plain = patch(AMP_MODELS["IGEV++"]().eval(), aggregation=True)
    amp = patch(AMP_MODELS["IGEV++"]().eval(), aggregation=True, amp=True)
    assert _instance_attributes(amp) == _instance_attributes(plain)
    assert {"cost_agg0.forward", "cost_agg1.forward", "cost_agg2.forward"} <= _instance_attributes(amp)
    assert all(e.amp for e in _engines(amp))


def _named(name, module="stereo.modeling.models.x.x"):
    cls = type(name, (torch.nn.Module,), {"__module__": module})
    return cls()


@pytest.mark.parametrize("name", ["GwcNet", "PSMNet", "LightStereo", "IGEVRTtereo", "CoEx", "MSNet3D"])
def test_amp_refused_for_every_other_patcher(name):
    from openstereo_b200.patch import _PATCHERS, patch
    assert name in _PATCHERS
    m = _named(name)
    with pytest.raises(NotImplementedError, match=r"patch\(%s, amp=True\)" % name):
        patch(m, amp=True)
    assert not getattr(m, "_osb_patched", False)


@pytest.mark.parametrize("module,name", [("stereo.modeling.models.casnet.cas_psm", "PSMNet"),
                                         ("stereo.modeling.models.casnet.cas_gwc", "GwcNet")])
def test_amp_refused_for_casstereo(module, name):
    from openstereo_b200.patch import patch
    with pytest.raises(NotImplementedError, match=r"patch\(%s, amp=True\)" % name):
        patch(_named(name, module), amp=True)


def test_every_patcher_is_covered():
    """The refusal list above and the four amp models are every entry of _PATCHERS."""
    from openstereo_b200.patch import _AMP_PATCHERS, _PATCHERS
    amp = {k for k, v in _PATCHERS.items() if v in _AMP_PATCHERS}
    assert amp == {"StereoBase", "IGEVStereo", "IGEVPPStereo", "MonSter"}
    assert set(_PATCHERS) - amp == {"GwcNet", "PSMNet", "LightStereo", "IGEVRTtereo", "CoEx", "MSNet3D"}


def _prototype(name):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "openstereo_b200.h")).read(), flags=re.S)
    m = re.search(r"int\s+%s\s*\(([^)]*)\)" % name, text)
    assert m, name
    return [p.strip() for p in m.group(1).replace("\n", " ").split(",")]


@pytest.mark.parametrize("new,old", [("osb_conv2d_k3_tc_prec_fwd", "osb_conv2d_k3_tc_fwd"),
                                     ("osb_conv2d_k3_tc_gru_prec_fwd", "osb_conv2d_k3_tc_gru_fwd")])
def test_abi_declares_the_precision_entry_points(native, new, old):
    """The old prototype plus `int precision` before the stream; exported; bound with that arity."""
    p_new, p_old = _prototype(new), _prototype(old)
    assert len(p_new) == len(p_old) + 1 == len(native.SIGNATURES[new])
    assert p_new[:-2] == p_old[:-1] and p_new[-2] == "int precision" and p_new[-1] == p_old[-1]
    assert native.SIGNATURES[new] == native.SIGNATURES[old][:-1] + [ctypes.c_int, ctypes.c_void_p]
    assert hasattr(ctypes.CDLL(native.LIB_PATH), new)
    text = open(os.path.join(ROOT, "include", "openstereo_b200.h")).read()
    assert re.search(r"#define OSB_PREC_FP32 0\b", text) and re.search(r"#define OSB_PREC_F16 1\b", text)


@pytest.mark.parametrize("precision", [-1, 2, 16])
def test_abi_refuses_an_unknown_precision_before_any_launch(native, precision):
    a = 0x1000                                                  # never dereferenced: the check comes first
    with pytest.raises(ValueError, match="unknown precision %d" % precision):
        native.call("osb_conv2d_k3_tc_prec_fwd", a, a, a, None, None, a, 1, 64, 64, 4, 128, 1, 0, 1, 1, precision, None)
    with pytest.raises(ValueError, match="unknown precision %d" % precision):
        native.call("osb_conv2d_k3_tc_gru_prec_fwd", a, a, None, None, None, None, None, None, a, 1, 64, 128, 4, 128, 0, 1, 1, 0,
                    precision, None)


def test_ops_refuses_an_unknown_precision(native):
    from openstereo_b200 import ops
    x = torch.zeros(1, 4, 128, 64)
    for fn in (ops.conv2d_k3_tc, ops.conv2d_k3_tc_gru):
        with pytest.raises(ValueError, match="precision"):
            fn(x, None, precision="bf16")
