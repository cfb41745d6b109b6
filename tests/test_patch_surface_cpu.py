"""CPU: what patch() rebinds on each supported class -- the exact instance attributes it adds or replaces, per sub-module, on the
UNMODIFIED reference classes -- and the oracle's timm stand-in, which has to be one object whichever of shim.load() and
install_timm_stub() runs first."""
import sys

import pytest
import torch

from oracle import _reference_shim as shim

pytestmark = pytest.mark.skipif(not shim.available(), reason="reference tree not present")

_UPDATE = ("gru04", "gru08", "gru16", "encoder", "disp_head", "mask_feat_4")


def _update(block, names=_UPDATE):
    return {"%s.%s.forward" % (block, n) for n in names}


def _cfg_model(cfg, dotted, cls):
    shim.install_timm_stub()
    return getattr(shim.load(dotted), cls)(shim.load_cfg(cfg).MODEL)


def _oracle(name, fn):
    def build():
        import importlib
        return getattr(importlib.import_module("oracle." + name), fn)()
    return build


_M = "stereo.modeling.models."
MODELS = {
    "GwcNet": (lambda: _cfg_model("cfgs/gwcnet/gwcnet_sceneflow.yaml", _M + "gwcnet.gwcnet", "GwcNet"),
               {"Backbone.forward", "CostProcessor.forward", "CostProcessor.build_gwc_volume", "CostProcessor.build_concat_volume",
                "DispProcessor.forward"}),
    "PSMNet": (lambda: _cfg_model("cfgs/psmnet/psmnet_sceneflow.yaml", _M + "psmnet.psmnet", "PSMNet"),
               {"Backbone.forward", "CostProcessor.forward", "CostProcessor.cat_func", "DispProcessor.disp_processor.forward"}),
    "StereoBase": (lambda: _cfg_model("cfgs/stereobase/stereobase_sceneflow.yaml", _M + "stereobase.stereobase_gru", "StereoBase"),
                   {"forward", "upsample_disp", "cost_agg.forward"} | _update("update_block")),
    "LightStereo": (lambda: _cfg_model("cfgs/lightstereo/lightstereo_s_sceneflow.yaml", _M + "lightstereo.lightstereo",
                                       "LightStereo"),
                    {"forward", "cost_agg.forward"}),
    "IGEVStereo": (lambda: _cfg_model("cfgs/igev/igev_sceneflow_amp.yaml", _M + "igev.igev_stereo", "IGEVStereo"),
                   {"forward", "upsample_disp"} | _update("update_block")),
    "IGEV-RT": (_oracle("igev_rt", "igev_rt"), {"forward", "upsample_disp", "cost_agg.forward", "classifier.forward"}),
    "IGEV++": (_oracle("igevpp", "igevpp"),
               {"forward", "upsample_disp", "classifier.forward"}
               | _update("update_block", _UPDATE + ("geo_encoder0", "geo_encoder1", "geo_encoder2"))),
    "MonSter": (_oracle("monster", "monster"),
                {"_forward_pair", "upsample_disp"} | _update("update_block") | _update("update_block_mix_stereo")
                | _update("update_block_mix_mono")),
    "CoEx": (lambda: _cfg_model("cfgs/coex/coex_sceneflow_amp.yaml", _M + "coex.coex", "CoEx"),
             {"CostProcessor.forward", "DispProcessor.forward", "DispProcessor.regression.forward"}),
    "MSNet3D": (lambda: _cfg_model("cfgs/msnet/msnet3d_sceneflow.yaml", _M + "msnet.MSNet3D", "MSNet3D"), {"forward"}),
    "CasPSMNet": (lambda: _cfg_model("cfgs/casnet/casnet_psm_sceneflow.yaml", _M + "casnet.cas_psm", "PSMNet"),
                  {"get_cv.forward", "cost_agg.0.forward", "cost_agg.1.forward"}),
    "CasGwcNet": (lambda: _cfg_model("cfgs/casnet/casnet_psm_sceneflow.yaml", _M + "casnet.cas_gwc", "GwcNet"),
                  {"get_cv.forward", "cost_agg.0.forward", "cost_agg.1.forward"}),
}


def _instance_attributes(model):
    return {(path, name): value for path, sub in model.named_modules() for name, value in vars(sub).items()}


@pytest.mark.parametrize("name", sorted(MODELS))
def test_patch_rebinds_exactly(name):
    """The attributes patch() adds, or replaces by another object (PSMNet's cat_func), on every sub-module of the instance; the
    idempotence flag aside.  Everything else -- the class, the other sub-modules, parameters and buffers -- stays as it was."""
    from openstereo_b200.patch import patch
    build, want = MODELS[name]
    model = build().eval()
    before = _instance_attributes(model)
    patch(model)
    after = _instance_attributes(model)
    changed = {("%s.%s" % key if key[0] else key[1]) for key, v in after.items() if key not in before or before[key] is not v}
    assert changed - {"_osb_patched"} == want and model._osb_patched
    assert before.keys() <= after.keys()


def test_timm_stand_in_is_one_object(monkeypatch):
    """A reference module that shim.load() imports while timm is absent binds the stand-in install_timm_stub() returns later."""
    for key in [k for k in sys.modules if k == "timm" or k.startswith(_M + "stereobase")]:
        monkeypatch.delitem(sys.modules, key)
    backbone = shim.load(_M + "stereobase.backbone")
    assert shim.install_timm_stub() is backbone.timm is sys.modules["timm"]
    cfg = shim.load_cfg("cfgs/stereobase/stereobase_sceneflow.yaml").MODEL
    model = shim.load(_M + "stereobase.stereobase_gru").StereoBase(cfg)
    assert isinstance(model, torch.nn.Module)
