"""patch(model): make an UNMODIFIED OpenStereo model instance (GwcNet / PSMNet / StereoBase / LightStereo / IGEVStereo / IGEV-RT /
IGEV++ / MonSter / CoEx / MSNet3D / MSNet2D, CasStereo's CasPSMNet / CasGwcNet, AANet and CFNet, built by the reference's own classes from an unchanged cfg YAML) run its cost-volume
hot path on the sm_90a kernels.

The reference has no operator registry; names are bound three different ways (SURVEY.md section 8b), and each needs its own
rebinding.  What each model rebinds:

* GwcNet      ``Backbone.forward``; ``CostProcessor.forward`` and its bound ``build_gwc_volume`` / ``build_concat_volume``
              (gwcnet_cost_processor.py:58-64); ``DispProcessor.forward`` (gwcnet_disp_processor.py:83-140)
* PSMNet      ``Backbone.forward``; ``CostProcessor.forward`` and ``cat_func``, the functools.partial of ``cat_fms`` captured at
              construction (psmnet_cost_processor.py:227-232); ``FasterSoftArgmin.forward``
* StereoBase  reference globals used by the model's methods (stereobase_gru.py:5-6,10-11): build_gwc_volume, build_concat_volume,
              disparity_regression, CombinedGeoEncodingVolume, context_upsample (any scale); ``cost_agg`` (Hourglass) forward;
              the update block
* LightStereo globals (lightstereo.py:4-6): correlation_volume, disparity_regression, context_upsample (scale 4); ``cost_agg``
* IGEVStereo  globals (igev_stereo.py:1-3): build_gwc_volume, disparity_regression, context_upsample (scale 4),
              Combined_Geo_Encoding_Volume; the update block
* MonSter     IGEVStereo's globals (monster.py:1-8) and disp_warp; ``update_block``, ``update_block_mix_stereo`` and
              ``update_block_mix_mono``
* IGEV-RT     globals (igev_rt_stereo.py:1-6): build_gwc_volume, disparity_regression (strided), Geo_Encoding_Volume,
              context_upsample ((B, 1, 4h, 4w)); ``cost_agg`` and ``classifier`` forward
* IGEV++      globals (igevpp_stereo.py:4-8): build_gwc_volume, disparity_regression (strided), Combined_Geo_Encoding_Volume
              (multi-range), context_upsample ((B, 1, 4h, 4w)); ``classifier`` forward; the update block with ``geo_encoder0..2``;
              with aggregation=True also ``cost_agg0 / cost_agg1 / cost_agg2`` forward
* CasStereo   ``get_cv`` (GetCostVolume) and every ``cost_agg[i]`` (CostAggregation) forward
* CoEx        ``CostProcessor`` / ``DispProcessor`` / ``DispProcessor.regression`` forward
* AANet       ``cost_volume`` and ``disparity_estimation`` forward; the ``disp_warp`` global of every ``refinement[i]``
              (aanet/submodule.py:748, 801-824)
* MSNet3D     one monolithic ``forward`` (MSNet3D.py:110-161), no processor modules: ``model.forward``, which keeps the
              reference's ``feature_extraction``
* MSNet2D     the same: ``model.forward`` (MSNet2D.py:134-212), which keeps ``feature_extraction`` and ``preconv11``
* CFNet       the same: ``model.forward`` (cfnet.py:488-668), which keeps ``feature_extraction`` and the reference's search-range
              and sampling code between the stages

"The update block" is the per-instance ``forward`` of its ``gru04 / gru08 / gru16`` (gru.py) and ``encoder / disp_head /
mask_feat_4`` (update.py).  A module override is a per-instance ``forward`` attribute.  A reference global is rebound by giving the
instance private copies of the methods of its class that use the name, with a private globals dict (_rebind_methods): the module
itself, and therefore every other instance, is untouched.  Parameters stay where they are (the engines read them through the
reference's attribute names), so ``state_dict()`` / ``load_state_dict()`` and checkpoints are untouched.

Every rebinding routes each call by one rule (_guard).  A call is a CUDA inference call when every operand is on a CUDA device,
the owning module is in eval mode (for a reference global: the model), autograd records on no operand (``torch.no_grad()`` as in
trainer_template.py:260-283, or no operand requires grad) and, for a module override, not on one of the module's own parameters
either.  The kernels have no backward, so any other call must NOT reach them silently:
  strict=True  (default) it RAISES -- there is no CPU / autograd path in this package;
  strict=False           it runs the reference's own original code, gradients intact (tools/train.py).
A CUDA inference call that no kernel serves (a shape or hyper-parameter outside the kernels' envelope) runs the reference's own
code in both modes.  Every other call runs the library.

Precision.  By default every patched layer computes fp32-accurate results, under autocast too, and returns the reference's dtypes.
``patch(model, amp=True)`` (IGEVStereo, StereoBase, IGEV++, MonSter) lets the update block's tensor-core 3x3 convolutions run at
the accuracy the reference's AMP YAMLs ask for: inside ``torch.autocast("cuda", ...)`` (fp16 or bf16) they issue one fp16 MMA per
product instead of the three of the fp32-accurate split (gru.py, update.py: _BlockEngine; DESIGN.md section 4.20).  Outside
autocast ``amp=True`` computes exactly what ``amp=False`` does.  The overrides installed, the shapes served and the dtypes returned
are the same either way.
"""
import functools
import types

import torch

from . import ops
from .aggregation import (CascadeAggregation, GwcAggregation, IGEVPPAggregation, PSMAggregation, StereoBaseAggregation,
                          StereoBaseCostHead)
from .geo import CombinedGeoEncodingVolume, GeoEncodingVolume, MultiRangeGeoEncodingVolume
from .gru import ConvGRUEngine
from .update import DispHeadEngine, GeoEncoderEngine, MaskFeatEngine, MotionEncoderEngine


def _tensors(args):
    for a in args:
        if isinstance(a, torch.Tensor):
            yield a
        elif isinstance(a, (list, tuple)):
            yield from _tensors(a)
        elif isinstance(a, dict):
            yield from _tensors(a.values())


def _recording(*args):
    """True when autograd would record an op on these operands (the kernels would silently cut the graph)."""
    return torch.is_grad_enabled() and any(t.requires_grad for t in _tensors(args))


def _trainable(module):
    """True when autograd would record through the module's own parameters (a kernel call would cut them off)."""
    return torch.is_grad_enabled() and any(p.requires_grad for p in module.parameters())


def _refuse(what):
    raise RuntimeError("openstereo_b200: %s is patched for CUDA inference only (model.eval() on a CUDA device, under "
                       "torch.no_grad() or with no operand requiring grad); use patch(model, strict=False) to delegate "
                       "training / CPU calls to the reference implementation" % what)


def _guard(what, strict, fast, orig, owner, serves=None, operands=None, own_params=False):
    """The rule of the module docstring as a callable with orig's signature: `fast` for a CUDA inference call that serves(*args)
    accepts (None: every one), else orig, or a refusal naming `what`.  owner: the module whose mode counts (None: no mode check);
    operands(*args): the tensors the rule looks at (None: every argument); own_params: the parameter condition of a module
    override."""
    def call(*args, **kwargs):
        ts = list(_tensors(operands(*args, **kwargs) if operands else (args, kwargs)))
        if (not ts or not all(t.is_cuda for t in ts) or (owner is not None and owner.training) or _recording(*ts)
                or (own_params and _trainable(owner))):
            if strict:
                _refuse(what)
            return orig(*args, **kwargs)
        if serves is not None and not serves(*args, **kwargs):
            return orig(*args, **kwargs)                            # no kernel for this call: the reference's computation
        return fast(*args, **kwargs)
    return call


def _override(mod, what, strict, fast, serves=None, operands=None):
    """Install _guard(...) over the module's own forward as its per-instance forward."""
    mod.forward = _guard(what, strict, fast, mod.forward, mod, serves, operands, own_params=True)


def _rebind_methods(model, overrides):
    """Give `model` private copies of the methods of its class that use any name in `overrides` as a module global: same code
    object, closure and defaults, but a globals dict with the overrides applied.  The module namespace and the class are not
    modified, so other instances (patched or not) are unaffected."""
    for name, fn in vars(type(model)).items():
        if isinstance(fn, types.FunctionType) and set(fn.__code__.co_names) & set(overrides):
            g = dict(fn.__globals__)
            g.update(overrides)
            copy = types.FunctionType(fn.__code__, g, fn.__name__, fn.__defaults__, fn.__closure__)
            copy.__kwdefaults__ = fn.__kwdefaults__
            setattr(model, name, types.MethodType(copy, model))


# The library's side of each reference global, one per name and signature, as (fast, serves) for _guard.  The geometry factories
# are the library's classes, which take the reference classes' arguments.
def _gwc_volume(ref, tgt, maxdisp, groups):
    return ops.build_gwc_volume(ref, tgt, maxdisp, groups)


def _concat_volume(ref, tgt, maxdisp):
    return ops.build_concat_volume(ref, tgt, maxdisp)


def _correlation_volume(left, right, max_disp):
    return ops.correlation_volume(left, right, max_disp)


def _regression(x, maxdisp):
    return ops.disparity_regression(x, maxdisp)


def _regression_interval(prob, maxdisp, interval):                  # IGEV-RT / IGEV++: the strided regression
    return ops.disparity_regression_interval(prob, maxdisp, interval)


def _upsample(disp_low, up_weights, scale_factor=4):
    return ops.context_upsample(disp_low, up_weights, scale_factor).to(disp_low.dtype)


def _upsample_keepdim(disp_low, up_weights):                        # IGEV-RT / IGEV++: keeps dim 1, (B, 1, 4h, 4w)
    return ops.context_upsample(disp_low, up_weights, 4).unsqueeze(1).to(disp_low.dtype)


def _disp_warp(img, disp, padding_mode="border"):
    """(warped, None): the valid mask (disp_warp(...)[1]) is not computed; the only method the patch rebinds that calls
    disp_warp, MonSter's _forward_pair, takes [0]."""
    return ops.disp_warp(img, disp), None


_GWC, _CONCAT, _CORR = (_gwc_volume, None), (_concat_volume, None), (_correlation_volume, None)
_REGRESSION, _REGRESSION_INTERVAL = (_regression, None), (_regression_interval, None)
_UPSAMPLE, _UPSAMPLE_KEEPDIM = (_upsample, None), (_upsample_keepdim, None)
_UPSAMPLE_4 = (_upsample, lambda disp_low, up_weights, scale_factor=4: scale_factor == 4)
_COMBINED_GEO = (CombinedGeoEncodingVolume, None)
_IGEV_GLOBALS = {"build_gwc_volume": _GWC, "disparity_regression": _REGRESSION, "context_upsample": _UPSAMPLE_4,
                 "Combined_Geo_Encoding_Volume": _COMBINED_GEO}


def _rebind_globals(model, strict, table):
    """table: {name of a global of the model's module: (fast, serves)} -> the model's methods see the guarded callables."""
    g = type(model).forward.__globals__
    _rebind_methods(model, {name: _guard(name, strict, fast, g[name], model, serves) for name, (fast, serves) in table.items()})


def _override_engine(mod, engine, strict, what):
    """Install an update-block engine (update.py) as the module's guarded forward: the calls engine.serves() accepts run it."""
    _override(mod, what, strict, engine, engine.serves)


def _override_convgru(mod, engine, strict):
    """Install a gru.ConvGRUEngine as the ConvGRU module's guarded forward(h, cz, cr, cq, *x_list)."""
    _override(mod, "ConvGRU", strict, engine, lambda h, cz, cr, cq, *x_list: engine.serves(h, x_list))


_UPDATE_ENGINES = {"encoder": MotionEncoderEngine, "geo_encoder0": GeoEncoderEngine, "geo_encoder1": GeoEncoderEngine,
                   "geo_encoder2": GeoEncoderEngine, "disp_head": DispHeadEngine, "mask_feat_4": MaskFeatEngine}
_IGEV_UPDATE = ("gru04", "gru08", "gru16", "encoder", "disp_head", "mask_feat_4")


def _patch_update_block(block, strict, names=_IGEV_UPDATE, amp=False):
    """Per-instance ``forward`` overrides of the update block's modules `names`: the ConvGRUs ``gru04 / gru08 / gru16`` on
    gru.ConvGRUEngine, the others on their update.py engine, each built with `amp` (autocast-precision tensor-core layers).  CUDA
    inference calls the kernels serve (the engines' serves()) run the engine, the other shapes and hyper-parameters the reference's
    own forward."""
    for name in names:
        mod = getattr(block, name)
        if name.startswith("gru"):
            _override_convgru(mod, ConvGRUEngine(mod, amp), strict)
        else:
            _override_engine(mod, _UPDATE_ENGINES[name](mod, amp), strict, name)


def _patch_backbone(bb, net, extract, split):
    """2D feature extractor (gwcnet_backbone.py:96-107 / psmnet_backbone.py:118-126; not a SURVEY section-8 row, but inside the
    measured forward): CUDA inference calls run a BN-folded twin of `net` whose identity-shortcut 3x3 residual blocks use the
    wgmma conv kernels where a variant serves the shape (host_models.gwc_extract / psm_extract; every other layer is the
    module's own cuDNN conv), left and right images in ONE batched pass (the weights are shared).  Parameters stay in `net`;
    the twin is rebuilt when they change.  Any other call (CPU, training, autograd recording, fp16 or unequal images) runs the
    reference's forward, in strict mode too: the cost processor that follows refuses such a call."""
    from . import host_models
    rt = host_models._FoldedRuntime(net)

    def fast(inputs):
        left = inputs["left"]
        return split(extract(rt.get(), torch.cat((left, inputs["right"]), 0)), left.shape[0])

    _override(bb, "Backbone", False, fast,
              serves=lambda inputs: inputs["left"].dtype == torch.float32 and inputs["left"].shape == inputs["right"].shape,
              operands=lambda inputs: (inputs["left"], inputs["right"]))


def _split_dict(both, b):
    return {"ref_feature": {k: v[:b] for k, v in both.items()}, "tgt_feature": {k: v[b:] for k, v in both.items()}}


def _split_tensor(both, b):
    return {"ref_feature": both[:b], "tgt_feature": both[b:]}


def _features(inputs):
    return inputs["ref_feature"], inputs["tgt_feature"]


def _patch_gwcnet(model, strict, backbone=True):
    if backbone:
        from .host_models import gwc_extract
        _patch_backbone(model.Backbone, model.Backbone.feature_extraction, gwc_extract, _split_dict)
    cp, dp = model.CostProcessor, model.DispProcessor
    cp_orig = cp.forward                                                 # the reference's bound method
    gwc_orig, cat_orig = cp.build_gwc_volume, cp.build_concat_volume
    engine = GwcAggregation(dp)

    def cost_orig(inputs):                                               # the reference's forward calls the reference's builders
        saved = cp.build_gwc_volume, cp.build_concat_volume
        cp.build_gwc_volume, cp.build_concat_volume = gwc_orig, cat_orig
        try:
            return cp_orig(inputs)
        finally:
            cp.build_gwc_volume, cp.build_concat_volume = saved

    def cost_fast(inputs):
        lf, rf = _features(inputs)
        d = cp.maxdisp // cp.downsample
        if cp.use_concat_volume:
            vol = ops.gwc_concat_volume(lf["gwc_feature"], rf["gwc_feature"], lf["concat_feature"],
                                        rf["concat_feature"], d, cp.num_groups)
        else:
            vol = ops.build_gwc_volume(lf["gwc_feature"], rf["gwc_feature"], d, cp.num_groups)
        return {"cost_volume": vol}

    cp.forward = _guard("GwcVolumeCostProcessor", strict, cost_fast, cost_orig, cp, operands=_features, own_params=True)
    _override(dp, "GwcDispProcessor", strict,
              lambda inputs: {"inference_disp": {"disp_est": engine(inputs["cost_volume"], *inputs["left"].shape[2:])}},
              operands=lambda inputs: (inputs["cost_volume"],))
    # the two volume builders stay callable on their own, with the reference's method signatures
    cp.build_gwc_volume = _guard("build_gwc_volume", strict,
                                 lambda ref, tgt: ops.build_gwc_volume(ref, tgt, cp.maxdisp // cp.downsample, cp.num_groups),
                                 gwc_orig, None)
    cp.build_concat_volume = _guard("build_concat_volume", strict,
                                    lambda ref, tgt: ops.build_concat_volume(ref, tgt, cp.maxdisp // cp.downsample), cat_orig, None)
    return model


class FusedCost:
    """What the patched PSMCostProcessor hands to PSMDispProcessor in place of a (B, 192, H, W) cost tensor: the fused tail
    (trilinear x4 + softmax + expectation in one kernel) already produced the disparity and the full-resolution cost is never
    materialised.  The patched FasterSoftArgmin recognises it; any other consumer gets a loud AttributeError/TypeError
    instead of a silently wrong tensor."""
    __slots__ = ("disp",)

    def __init__(self, disp):
        self.disp = disp


def _patch_psmnet(model, strict, backbone=True):
    if backbone:
        from .host_models import psm_extract
        _patch_backbone(model.Backbone, model.Backbone, psm_extract, _split_tensor)
    cp, dp = model.CostProcessor, model.DispProcessor
    cp_orig = cp.forward
    engine = PSMAggregation(cp.aggregator)
    max_disp = cp.aggregator.max_disp
    cat_orig = cp.cat_func                                          # functools.partial(cat_fms, ...) of the reference

    def cost_orig(inputs):                                          # the reference's forward calls the reference's cat_func
        saved, cp.cat_func = cp.cat_func, cat_orig
        try:
            return cp_orig(inputs)
        finally:
            cp.cat_func = saved

    def cat_fms(l, r):
        return ops.cat_fms(l, r, max_disp=int(max_disp // 4), start_disp=0, dilation=1)

    def cost_fast(inputs):
        d1, d2, d3 = engine(cat_fms(*_features(inputs)))
        return {"cost1": FusedCost(d1), "cost2": FusedCost(d2), "cost3": FusedCost(d3)}

    cp.forward = _guard("PSMCostProcessor", strict, cost_fast, cost_orig, cp, operands=_features, own_params=True)
    cp.cat_func = _guard("cat_fms", strict, cat_fms, cat_orig, None)
    sa = dp.disp_processor                                          # FasterSoftArgmin: keep the frozen Conv3d parameter
    soft_argmin = _guard("FasterSoftArgmin", strict, lambda cost: ops.faster_soft_argmin(
        cost, sa.max_disp, sa.start_disp, sa.dilation, sa.alpha, sa.normalize), sa.forward, None)
    sa.forward = lambda cost: cost.disp if isinstance(cost, FusedCost) else soft_argmin(cost)
    return model


def _patch_stereobase(model, strict, backbone=True, amp=False):
    # SURVEY.md section 8(f) rows 1 and 3: the per-GRU-iteration lookup and the convex up-sampling (stereobase_gru.py:172-209)
    _rebind_globals(model, strict, {"build_gwc_volume": _GWC, "build_concat_volume": _CONCAT, "disparity_regression": _REGRESSION,
                                    "CombinedGeoEncodingVolume": _COMBINED_GEO, "context_upsample": _UPSAMPLE})
    agg = StereoBaseAggregation(model.cost_agg)
    _override(model.cost_agg, "StereoBase Hourglass", strict, lambda x, features, return_multi=False: agg(x, features).to(x.dtype),
              serves=lambda x, features, return_multi=False: not return_multi)
    _patch_update_block(model.update_block, strict, amp=amp)
    return model


def _patch_lightstereo(model, strict, backbone=True):
    """LightStereo (BASELINE config 4; lightstereo/lightstereo.py:44-70): correlation_volume, the 2D `Aggregation` hourglass
    (cost_agg), disparity_regression and context_upsample; backbone / refine heads stay the reference's cuDNN code."""
    from .aggregation import LightStereoAggregation
    _rebind_globals(model, strict, {"correlation_volume": _CORR, "disparity_regression": _REGRESSION,
                                    "context_upsample": _UPSAMPLE_4})
    engine = LightStereoAggregation(model.cost_agg)
    _override(model.cost_agg, "LightStereo Aggregation", strict,
              lambda x, features_left: [t.to(x.dtype) for t in engine(x, features_left[:3])],
              operands=lambda x, features_left: (x, features_left[:3]))
    return model


def _patch_igev(model, strict, backbone=True, amp=False):
    """IGEV-Stereo (BASELINE config 5; igev/igev_stereo.py:136-213): the gwc volume, the soft-argmin regression of the initial
    disparity, the per-GRU-iteration lookup of the combined geometry-encoding volume, the three ConvGRUs of the update block
    (``update_block.gru04 / gru08 / gru16``, gru.py), its motion encoder and disp / mask heads (``update_block.encoder / disp_head /
    mask_feat_4``, update.py) and the convex up-sampling.  The hourglass(8) and the feature nets stay the reference's cuDNN code.
    Under autocast (the AMP YAML) the update block computes in fp32 and returns the reference's dtypes; with amp=True its
    tensor-core layers compute at autocast accuracy instead (module docstring)."""
    _rebind_globals(model, strict, _IGEV_GLOBALS)
    _patch_update_block(model.update_block, strict, amp=amp)
    return model


def _patch_monster(model, strict, backbone=True, amp=False):
    """MonSter (monster/monster.py, class MonSter): the stereo branch's IGEV-shaped hot path -- the gwc volume, the soft-argmin
    regression of the initial disparity, every lookup of the combined geometry-encoding volume (at disp, and at disp_mono_4x in
    the last 7 iterations), the disparity warps of features_right[0] (``disp_warp``; the kernel replays the border padding only),
    the ConvGRUs, motion encoders and disp / mask heads of ``update_block``, ``update_block_mix_stereo`` and
    ``update_block_mix_mono`` and the convex up-sampling.  The Depth Anything encoder and decoders, feat_transfer*, the stems,
    corr_stem / corr_feature_att / cost_agg, the classifier, compute_scale_shift, REMP and the update blocks' own forward stay the
    reference's code; `backbone` has no effect.  Under autocast (the AMP YAML, bf16) every patched call computes in fp32 and
    returns the reference's dtypes; with amp=True the update blocks' tensor-core layers compute at autocast accuracy instead."""
    warp = (_disp_warp, lambda img, disp, padding_mode="border": padding_mode == "border")
    _rebind_globals(model, strict, dict(_IGEV_GLOBALS, disp_warp=warp))
    for block in (model.update_block, model.update_block_mix_stereo, model.update_block_mix_mono):
        _patch_update_block(block, strict, amp=amp)
    return model


def _patch_igev_rt(model, strict, backbone=True):
    """IGEV-RT (igev_rt/igev_rt_stereo.py:146-206, class IGEVRTtereo): the gwc volume, the hourglass(8) (``cost_agg.forward``), the
    classifier Conv3d(8 -> 1) (``classifier.forward``, which returns logits: the reference's own softmax follows), the strided
    regression of the initial disparity, the per-GRU-iteration lookup of the geometry-only encoding volume and the convex
    up-sampling.  The feature nets, hnet / cnet and the ConvGRU update block stay the reference's code; `backbone` has no effect.
    Under autocast (the AMP YAML) fp16 tensors arrive: every call computes in fp32 and returns the caller's dtype."""
    _rebind_globals(model, strict, {"build_gwc_volume": _GWC, "disparity_regression": _REGRESSION_INTERVAL,
                                    "Geo_Encoding_Volume": (GeoEncodingVolume, None), "context_upsample": _UPSAMPLE_KEEPDIM})
    agg, head = StereoBaseAggregation(model.cost_agg), StereoBaseCostHead(model.classifier)
    _override(model.cost_agg, "IGEV-RT hourglass", strict, lambda x, features: agg(x, features).to(x.dtype))
    _override(model.classifier, "IGEV-RT classifier", strict, lambda x: head.logits(x).to(x.dtype))
    return model


def _patch_igevpp(model, strict, backbone=True, aggregation=False, amp=False):
    """IGEV++ (igevpp/igevpp_stereo.py:162-249, class IGEVPPStereo): the gwc volume, the classifier Conv3d(8 -> 1) of the three
    disparity ranges (``classifier.forward``, which returns logits: the reference's own softmax follows), the strided regressions of
    the three initial disparities, the per-GRU-iteration multi-range lookup (one launch), the update block's ConvGRUs, geometry
    encoders, disparity encoder, disparity head and mask head, and the convex up-sampling.  With aggregation=True also the three
    instance-normalised hourglasses (``cost_agg0 / cost_agg1 / cost_agg2.forward``, aggregation.IGEVPPAggregation); calls whose
    layers or shapes the kernels do not implement run the module's own forward.  patch0 / patch1, the feature nets, cnet,
    selective_conv, disp_conv and BasicMultiUpdateBlock.forward itself (the selective-weight blend, cat, pool2x, interp) stay the
    reference's code, and so do the hourglasses by default; `backbone` has no effect.  Under autocast (the AMP YAML) every call
    computes in fp32 and returns the reference's dtypes; with amp=True the update block's tensor-core layers compute at autocast
    accuracy instead (the hourglasses stay fp32-accurate)."""
    _rebind_globals(model, strict, {"build_gwc_volume": _GWC, "disparity_regression": _REGRESSION_INTERVAL,
                                    "Combined_Geo_Encoding_Volume": (MultiRangeGeoEncodingVolume, None),
                                    "context_upsample": _UPSAMPLE_KEEPDIM})
    head = StereoBaseCostHead(model.classifier)
    _override(model.classifier, "IGEV++ classifier", strict, lambda x: head.logits(x).to(x.dtype))
    _patch_update_block(model.update_block, strict, _IGEV_UPDATE + ("geo_encoder0", "geo_encoder1", "geo_encoder2"), amp=amp)
    if aggregation:
        for name in ("cost_agg0", "cost_agg1", "cost_agg2"):
            eng = IGEVPPAggregation(getattr(model, name))
            _override(getattr(model, name), "IGEV++ " + name, strict, lambda x, features, eng=eng: eng(x, features).to(x.dtype),
                      serves=eng.serves)
    return model


def _patch_cascade(model, strict, backbone=True):
    """CasStereo (casnet/cas_psm.py PSMNet = CasPSMNet, casnet/cas_gwc.py GwcNet = CasGwcNet): every stage's warped cost volume
    (``get_cv.forward``) and every stage's aggregation + hypothesis-weighted soft-argmin (``cost_agg[i].forward``).  The FPN
    feature extractor and get_disp_range_samples stay the reference's code inside model.forward; `backbone` has no effect."""
    if type(model).__module__.rsplit(".", 1)[-1] == "cas_gwc":
        def cost_volume(features_left, features_right, disp_range_samples, ndisp, num_groups):
            assert disp_range_samples.shape[1] == ndisp
            vol = ops.warped_gwc_concat_volume(features_left["gwc_feature"], features_right["gwc_feature"],
                                               features_left["concat_feature"], features_right["concat_feature"],
                                               disp_range_samples, num_groups)
            return vol.to(features_left["gwc_feature"].dtype)
        _override(model.get_cv, "CasGwcNet GetCostVolume", strict, cost_volume)
    else:
        def cost_volume(x, y, disp_range_samples, ndisp):
            assert disp_range_samples.shape[1] == ndisp
            return ops.warped_concat_volume(x, y, disp_range_samples, mask_left=False)
        _override(model.get_cv, "CasPSMNet GetCostVolume", strict, cost_volume)
    for agg_mod in model.cost_agg:
        _patch_cascade_agg(agg_mod, strict)
    return model


def _patch_cascade_agg(agg_mod, strict):
    engine = CascadeAggregation(agg_mod)

    def aggregate(cost, FineD, FineH, FineW, disp_range_samples):   # the reference's names: model.forward passes them by keyword
        return engine(cost, FineD, FineH, FineW, disp_range_samples).to(cost.dtype)

    _override(agg_mod, "CasStereo CostAggregation", strict, aggregate)


def _patch_coex(model, strict, backbone=True):
    """CoEx (coex/coex.py): the attention cost volume and the 3D aggregation (``CostProcessor.forward``), the top-k regression
    with the superpixel up-sampling (``DispProcessor.forward``, and ``regression.forward`` for direct callers).  The MobileNet
    encoder, FeatUp, the stems and the superpixel branch convs stay the reference's code; `backbone` has no effect."""
    from .aggregation import CoExAggregation
    cp, dp = model.CostProcessor, model.DispProcessor
    reg = dp.regression
    if not 2 <= reg.top_k <= 8:
        raise NotImplementedError("patch(CoEx): REGRESSION_TOPK=%d is not supported (2..8; the reference's k = 1 branch gathers "
                                  "index D, which is out of range)" % reg.top_k)
    if cp.aggregation_disp_strides != 2:
        raise NotImplementedError("patch(CoEx): AGGREGATION_DISP_STRIDES=%r is not supported (2: the isotropic stride-2 "
                                  "convolutions of the kernels)" % (cp.aggregation_disp_strides,))
    if cp.matching_weighted:
        raise NotImplementedError("patch(CoEx): MATCHING_WEIGHTED=True is not supported")
    cv = cp.cost_volume
    engine = CoExAggregation(cp.cost_agg)

    def cost_fast(inputs):
        x, y = _features(inputs)
        xd, yd = cv.desc(cv.conv(x[0])), cv.desc(cv.conv(y[0]))       # the reference's own 2D convolutions
        cost = ops.coex_attention_volume(xd, yd, cv.costVolume.maxdisp - 1, cv.head)
        return {"cost_volume": engine(x, cost).to(x[0].dtype)}

    def disp_fast(inputs):
        cost = inputs["cost_volume"]
        xspx = dp.spx_2(dp.spx_4(inputs["ref_feature"][0]), inputs["stem_2x"])
        # the raw superpixel logits go into the kernel, which applies the reference's softmax over the 9 channels itself
        disp_pred = ops.coex_regression(cost, dp.spx(xspx), reg.top_k, spx_is_logits=True).to(cost.dtype)
        ref_img, tgt_img = inputs["left"], inputs["right"]
        output = {"inference_disp": {"disp_est": disp_pred},
                  "visual_summary": {"image/test/image_c": torch.cat([ref_img[0], tgt_img[0]], dim=1),
                                     "image/test/disp_c": disp_pred[0]}}
        if "disp_gt" in inputs:
            output["visual_summary"] = {"image/val/image_c": torch.cat([ref_img[0], tgt_img[0]], dim=1),
                                        "image/val/disp_c": torch.cat([inputs["disp_gt"][0], disp_pred[0]], dim=0)}
        return output

    _override(cp, "CoExCostProcessor", strict, cost_fast, operands=_features)
    _override(dp, "CoExDispProcessor", strict, disp_fast,
              operands=lambda inputs: (inputs["cost_volume"], inputs["ref_feature"], inputs["stem_2x"]))
    _override(reg, "CoEx Regression", strict, lambda cost, spg: [ops.coex_regression(cost, spg, reg.top_k).to(cost.dtype)])
    return model


def _aanet_disp_warp(img, disp, padding_mode="border"):
    """(warped, None) with the reference's precondition (aanet/submodule.py:811); StereoDRNetRefinement.forward takes [0]."""
    assert disp.min() >= 0
    return ops.disp_warp(img, disp), None


def _patch_aanet(model, strict, backbone=True):
    """AANet (aanet/aanet.py, class aanet): the correlation pyramid (``cost_volume.forward``: one correlation volume per scale at
    max_disp // 2^s), the soft-argmin of every scale (``disparity_estimation.forward``; match_similarity=False runs the reference's
    code) and the disparity warp of each StereoDRNet refinement (its ``disp_warp`` global).  The deformable bottlenecks keep the
    reference's DCNv2 extension, which the model cannot be built without and which is faster than the tensor-core gather mode
    (aanet.DeformBottleneckEngine, DESIGN.md section 4.21): that engine is not installed here.  The FPN, the bottlenecks, the
    cross-scale fusion layers and the refinements' convolutions stay the reference's code; `backbone` has no effect."""
    cv = model.cost_volume

    def cost_volume(left_feature_pyramid, right_feature_pyramid):
        return [ops.correlation_volume(l, r, cv.max_disp // (2 ** s))
                for s, (l, r) in enumerate(zip(left_feature_pyramid, right_feature_pyramid))]

    _override(cv, "AANet CostVolumePyramid", strict, cost_volume,
              serves=lambda left, right: cv.feature_similarity == "correlation")
    de = model.disparity_estimation
    _override(de, "AANet DisparityEstimation", strict, lambda cost: ops.softargmin(cost, cost.shape[1], keepdim=False),
              serves=lambda cost: de.match_similarity and cost.dim() == 4)
    for ref in model.refinement:
        orig = type(ref).forward.__globals__["disp_warp"]
        _rebind_methods(ref, {"disp_warp": _guard("disp_warp", strict, _aanet_disp_warp, orig, ref,
                                                  lambda img, disp, padding_mode="border": padding_mode == "border")})
    return model


def _patch_msnet3d(model, strict, backbone=True):
    """MSNet3D (msnet/MSNet3D.py): everything after the 2D features in the eval forward -- the gwc volume, the MobileV2_Residual_3D
    blocks (one fused launch each), the hourglass transposed convs, classif3 and the trilinear x4 + softmax + regression tail
    (``model.forward``, per instance).  The MobileNet 2D feature extractor stays the reference's code; `backbone` has no effect.
    A block the kernel does not implement is refused here, naming it."""
    from .aggregation import MSNet3DAggregation
    engine = MSNet3DAggregation(model)

    def forward(data):
        left, right = data["left"], data["right"]
        fl, fr = model.feature_extraction(left), model.feature_extraction(right)
        volume = ops.build_gwc_volume(fl, fr, model.maxdisp // 4, model.num_groups)
        return {"disp_pred": engine(volume, left.shape[2], left.shape[3]).to(left.dtype)}

    _override(model, "MSNet3D", strict, forward, operands=lambda data: (data["left"], data["right"]))
    return model


def _patch_msnet2d(model, strict, backbone=True):
    """MSNet2D (msnet/MSNet2D.py): everything after preconv11 in the eval forward (``model.forward``, per instance) -- the
    48-disparity volume loop (aggregation.MSNet2DVolume: the interlaced crops in one launch, the three depth-strided Conv3ds as 3x3
    Conv2ds per crop, volume11), then dres0 / dres1, the three hourglass2Ds, classif3 and the trilinear x4 + softmax + regression
    tail (aggregation.MSNet2DAggregation).  ``feature_extraction`` and ``preconv11`` stay the reference's code; `backbone` has no
    effect.  A volume network or block the kernels do not implement is refused here, naming it."""
    from .aggregation import MSNet2DAggregation, MSNet2DVolume
    volume, engine = MSNet2DVolume(model), MSNet2DAggregation(model)

    def forward(data):
        left, right = data["left"], data["right"]
        fl = model.preconv11(model.feature_extraction(left))
        fr = model.preconv11(model.feature_extraction(right))
        return {"disp_pred": engine(volume(fl, fr), left.shape[2], left.shape[3]).to(left.dtype)}

    _override(model, "MSNet2D", strict, forward, operands=lambda data: (data["left"], data["right"]))
    return model


def _patch_cfnet(model, strict, backbone=True):
    """CFNet (cfnet/cfnet.py, class cfnet, built by the CFNet(d) factory): everything after the 2D features in the eval forward
    (``model.forward``, per instance) -- the three stage-1 volumes, the warped volumes of the s3 / s2 refinements, every 3D
    convolution with its Mish epilogue and the three soft-argmin tails with their variances (cfnet.CFNetEngine).  The Mish feature
    extractor and the model's generate_search_range / generate_disparity_samples stay the reference's code; the bounds and
    their up-sampling, inline in the reference's forward, are restated term for term; `backbone` has no effect.  A model built with replace_mish=True is refused here, naming the module."""
    from .cfnet import CFNetEngine
    engine = CFNetEngine(model)

    def forward(data):
        left, right = data["left"], data["right"]
        fl, fr = model.feature_extraction(left), model.feature_extraction(right)
        return {"disp_pred": engine(fl, fr, left.shape[2], left.shape[3]).to(left.dtype)}

    _override(model, "CFNet", strict, forward, serves=engine.serves, operands=lambda data: (data["left"], data["right"]))
    return model


# Models routed by (package, module, class) of their defining module: CasStereo's classes are also named PSMNet / GwcNet, and
# AANet's and CFNet's classes are the bare lowercase `aanet` / `cfnet`; MSNet2D is routed the same way
_MODULE_PATCHERS = {("casnet", "cas_psm", "PSMNet"): _patch_cascade, ("casnet", "cas_gwc", "GwcNet"): _patch_cascade,
                    ("aanet", "aanet", "aanet"): _patch_aanet, ("cfnet", "cfnet", "cfnet"): _patch_cfnet,
                    ("msnet", "MSNet2D", "MSNet2D"): _patch_msnet2d}

_PATCHERS = {"GwcNet": _patch_gwcnet, "PSMNet": _patch_psmnet, "StereoBase": _patch_stereobase, "LightStereo": _patch_lightstereo,
             "IGEVStereo": _patch_igev, "IGEVRTtereo": _patch_igev_rt,
             "IGEVPPStereo": _patch_igevpp, "MonSter": _patch_monster, "CoEx": _patch_coex, "MSNet3D": _patch_msnet3d}
# the patchers whose update blocks take amp=True
_AMP_PATCHERS = (_patch_stereobase, _patch_igev, _patch_igevpp, _patch_monster)


def patch(model, strict=True, backbone=True, aggregation=False, amp=False):
    """Rebind the hot path of a reference model instance in place and return it.  backbone=True (default) also routes the
    GwcNet / PSMNet 2D extractor's residual blocks to the wgmma conv kernels in CUDA inference calls (_patch_backbone);
    backbone=False leaves the extractor entirely to the reference's cuDNN code.  For the CasStereo models (casnet.cas_psm.PSMNet,
    casnet.cas_gwc.GwcNet), AANet (aanet.aanet.aanet) and CFNet (cfnet.cfnet.cfnet) `backbone` has no effect: their 2D extractor
    always runs the reference's code.  aggregation=True (IGEV++ only) also runs the three instance-normalised hourglasses on the
    library; off by default.  amp=True (IGEVStereo, StereoBase, IGEVPPStereo, MonSter) runs the update blocks' tensor-core convolutions at autocast accuracy -- one fp16 MMA per
    product -- inside torch.autocast("cuda"), for users of the AMP YAMLs; outside autocast it changes nothing.  Off by default:
    every patched layer is then fp32-accurate under autocast too."""
    if not isinstance(model, torch.nn.Module):
        raise TypeError("patch() expects an nn.Module")
    name = type(model).__name__
    key = tuple(type(model).__module__.split(".")[-2:]) + (name,)
    if key in _MODULE_PATCHERS:
        patcher = _MODULE_PATCHERS[key]
    elif name in _PATCHERS:
        patcher = _PATCHERS[name]
    else:
        raise NotImplementedError("patch(): no hot-path drop-in for %s (supported: %s, CasStereo's casnet.cas_psm.PSMNet / "
                                  "casnet.cas_gwc.GwcNet, aanet.aanet.aanet, cfnet.cfnet.cfnet and msnet.MSNet2D.MSNet2D)" % (name, sorted(_PATCHERS)))
    if aggregation:
        if patcher is not _patch_igevpp:
            raise NotImplementedError("patch(%s, aggregation=True): only IGEVPPStereo has an aggregation option" % name)
        patcher = functools.partial(_patch_igevpp, aggregation=True)
    if amp:
        if patcher not in _AMP_PATCHERS and getattr(patcher, "func", None) not in _AMP_PATCHERS:
            raise NotImplementedError("patch(%s, amp=True): only the update blocks of %s have an autocast-precision mode"
                                      % (name, ", ".join(sorted(k for k, v in _PATCHERS.items() if v in _AMP_PATCHERS))))
        patcher = functools.partial(patcher, amp=True)
    if getattr(model, "_osb_patched", False):
        return model
    patcher(model, strict, backbone)
    model._osb_patched = True
    return model
