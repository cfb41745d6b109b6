"""patch(model): make an UNMODIFIED OpenStereo model instance (GwcNet / PSMNet / StereoBase / LightStereo / IGEVStereo / IGEV-RT /
IGEV++ / MonSter / CoEx / MSNet3D, and CasStereo's CasPSMNet / CasGwcNet, built by the reference's own classes from an unchanged cfg YAML) run its cost-volume
hot path on the sm_90a kernels.

The reference has no operator registry; names are bound three different ways (SURVEY.md section 8b), and each
needs its own rebinding:

* GwcNet      bound methods on ``CostProcessor`` (gwcnet_cost_processor.py:58-64) and the ``DispProcessor``
              forward (gwcnet_disp_processor.py:83-140)                    -> per-instance ``forward`` override
* PSMNet      ``cat_fms`` captured by functools.partial at construction (psmnet_cost_processor.py:227-232),
              aggregator + FasterSoftArgmin modules                          -> ``CostProcessor.forward`` / ``FasterSoftArgmin.forward``
* LightStereo / IGEVStereo  like StereoBase: names imported into lightstereo.py:4-6 / igev_stereo.py:1-3 (``from .submodule import *``)
* IGEV-RT     like IGEVStereo (igev_rt_stereo.py:1-6), plus per-instance ``cost_agg`` / ``classifier`` forward overrides
* MonSter     like IGEVStereo (monster.py:1-8, plus ``disp_warp``), and the ConvGRU / encoder / head overrides on all three update
              blocks (the two mix2 blocks' encoders on MixMotionEncoderEngine)
* IGEV++      like IGEVStereo (igevpp_stereo.py:4-8), plus a per-instance ``classifier`` forward override and the update block's
              ``gru04 / gru08 / gru16 / encoder / geo_encoder0..2 / disp_head / mask_feat_4`` forward overrides
* CasStereo   ``get_cv`` (GetCostVolume) and ``cost_agg[i]`` (CostAggregation) modules  -> per-instance ``forward`` overrides
* CoEx        ``CostProcessor`` / ``DispProcessor`` / ``DispProcessor.regression`` modules -> per-instance ``forward`` overrides
* MSNet3D     one monolithic ``forward`` (MSNet3D.py:110-161), no processor modules   -> per-instance ``model.forward`` override that
                                                                                keeps the reference's ``feature_extraction``
* StereoBase  functions imported INTO the module namespace (stereobase_gru.py:5-6,10-11) and the ``cost_agg``
              Hourglass                                                      -> per-INSTANCE copies of the methods that use those names,
                                                                                with a private globals dict (the module itself, and
                                                                                therefore every other StereoBase instance, is untouched)
* StereoBase / IGEVStereo ConvGRUs ``update_block.gru04 / gru08 / gru16``   -> per-instance ``forward`` overrides (gru.py)
* StereoBase / IGEVStereo ``update_block.encoder / disp_head / mask_feat_4``  -> per-instance ``forward`` overrides (update.py)

Parameters stay where they are (the engines read them through the reference's attribute names), so
``state_dict()`` / ``load_state_dict()`` and checkpoints are untouched.

When is a call accelerated?  Only when it is a CUDA inference call: every tensor on a CUDA device, the module in eval
mode, and autograd not recording (``torch.no_grad()`` as in trainer_template.py:260-283, or no operand requires grad).
The kernels have no backward, so anything else must NOT reach them silently:
  strict=True  (default) such a call RAISES -- there is no CPU / autograd path in this package;
  strict=False           such a call runs the reference's own original Python code, gradients intact (tools/train.py).
"""
import types

import torch

from . import ops
from .aggregation import CascadeAggregation, GwcAggregation, PSMAggregation, StereoBaseAggregation, StereoBaseCostHead
from .geo import CombinedGeoEncodingVolume, GeoEncodingVolume, MultiRangeGeoEncodingVolume


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


def _accelerable(module, *args):
    ts = list(_tensors(args))
    return (module is None or not module.training) and bool(ts) and all(t.is_cuda for t in ts) and not _recording(*ts)


def _refuse(what):
    raise RuntimeError("openstereo_b200: %s is patched for CUDA inference only (model.eval() on a CUDA device, under "
                       "torch.no_grad() or with no operand requiring grad); use patch(model, strict=False) to delegate "
                       "training / CPU calls to the reference implementation" % what)


def _patch_backbone(bb, net, extract, split):
    """2D feature extractor (gwcnet_backbone.py:96-107 / psmnet_backbone.py:118-126; not a SURVEY section-8 row, but inside the
    measured forward): CUDA inference calls run a BN-folded twin of `net` whose identity-shortcut 3x3 residual blocks use the
    wgmma conv kernels where a variant serves the shape (host_models.gwc_extract / psm_extract; every other layer is the
    module's own cuDNN conv), left and right images in ONE batched pass (the weights are shared).  Parameters stay in `net`;
    the twin is rebuilt when they change.  Any other call (CPU, training, autograd recording) runs the reference's forward."""
    from . import host_models
    rt = host_models._FoldedRuntime(net)
    orig = bb.forward

    def forward(self, inputs):
        left, right = inputs["left"], inputs["right"]
        trainable = torch.is_grad_enabled() and any(q.requires_grad for q in net.parameters())   # the folded twin would cut them off
        if trainable or not (_accelerable(self, left, right) and left.dtype == torch.float32 and left.shape == right.shape):
            return orig(inputs)
        both = extract(rt.get(), torch.cat((left, right), 0))
        return split(both, left.shape[0])

    bb.forward = types.MethodType(forward, bb)


def _split_dict(both, b):
    return {"ref_feature": {k: v[:b] for k, v in both.items()}, "tgt_feature": {k: v[b:] for k, v in both.items()}}


def _split_tensor(both, b):
    return {"ref_feature": both[:b], "tgt_feature": both[b:]}


def _patch_gwcnet(model, strict, backbone=True):
    if backbone:
        from .host_models import gwc_extract
        _patch_backbone(model.Backbone, model.Backbone.feature_extraction, gwc_extract, _split_dict)
    cp, dp = model.CostProcessor, model.DispProcessor
    cp_orig, dp_orig = cp.forward, dp.forward                                 # the reference's bound methods
    gwc_orig, cat_orig = cp.build_gwc_volume, cp.build_concat_volume
    engine = GwcAggregation(dp)

    def cost_forward(self, inputs):
        lf, rf = inputs["ref_feature"], inputs["tgt_feature"]
        if not _accelerable(self, lf, rf):
            if strict:
                _refuse("GwcVolumeCostProcessor")
            saved = self.build_gwc_volume, self.build_concat_volume            # the reference's forward calls these two
            self.build_gwc_volume, self.build_concat_volume = gwc_orig, cat_orig
            try:
                return cp_orig(inputs)
            finally:
                self.build_gwc_volume, self.build_concat_volume = saved
        d = self.maxdisp // self.downsample
        if self.use_concat_volume:
            vol = ops.gwc_concat_volume(lf["gwc_feature"], rf["gwc_feature"], lf["concat_feature"],
                                        rf["concat_feature"], d, self.num_groups)
        else:
            vol = ops.build_gwc_volume(lf["gwc_feature"], rf["gwc_feature"], d, self.num_groups)
        return {"cost_volume": vol}

    def disp_forward(self, inputs):
        if not _accelerable(self, inputs["cost_volume"]):
            return dp_orig(inputs) if not strict else _refuse("GwcDispProcessor")
        h, w = inputs["left"].shape[2:]
        return {"inference_disp": {"disp_est": engine(inputs["cost_volume"], h, w)}}

    cp.forward = types.MethodType(cost_forward, cp)
    dp.forward = types.MethodType(disp_forward, dp)

    # the two volume builders stay callable on their own, with the reference's method signatures
    def build_gwc(ref, tgt):
        if _accelerable(None, ref, tgt):
            return ops.build_gwc_volume(ref, tgt, cp.maxdisp // cp.downsample, cp.num_groups)
        return gwc_orig(ref, tgt) if not strict else _refuse("build_gwc_volume")

    def build_concat(ref, tgt):
        if _accelerable(None, ref, tgt):
            return ops.build_concat_volume(ref, tgt, cp.maxdisp // cp.downsample)
        return cat_orig(ref, tgt) if not strict else _refuse("build_concat_volume")

    cp.build_gwc_volume, cp.build_concat_volume = build_gwc, build_concat
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

    def cost_forward(self, inputs):
        lf, rf = inputs["ref_feature"], inputs["tgt_feature"]
        if not _accelerable(self, lf, rf):
            if strict:
                _refuse("PSMCostProcessor")
            saved, self.cat_func = self.cat_func, cat_orig
            try:
                return cp_orig(inputs)
            finally:
                self.cat_func = saved
        raw = ops.cat_fms(lf, rf, max_disp=int(max_disp // 4), start_disp=0, dilation=1)
        d1, d2, d3 = engine(raw)
        return {"cost1": FusedCost(d1), "cost2": FusedCost(d2), "cost3": FusedCost(d3)}

    cp.forward = types.MethodType(cost_forward, cp)

    def cat_func(l, r):
        if _accelerable(None, l, r):
            return ops.cat_fms(l, r, max_disp=int(max_disp // 4), start_disp=0, dilation=1)
        return cat_orig(l, r) if not strict else _refuse("cat_fms")

    cp.cat_func = cat_func
    sa = dp.disp_processor                                          # FasterSoftArgmin: keep the frozen Conv3d parameter
    sa_orig = sa.forward

    def sa_forward(self, cost):
        if isinstance(cost, FusedCost):
            return cost.disp
        if _accelerable(None, cost):
            return ops.faster_soft_argmin(cost, self.max_disp, self.start_disp, self.dilation, self.alpha, self.normalize)
        return sa_orig(cost) if not strict else _refuse("FasterSoftArgmin")

    sa.forward = types.MethodType(sa_forward, sa)
    return model


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


def _patch_convgru(block, strict):
    """Per-instance ``forward`` overrides of ``gru04 / gru08 / gru16`` of an IGEV / StereoBase BasicMultiUpdateBlock: CUDA inference
    calls the wgmma kernels serve (gru.route_ok) run gru.ConvGRUEngine; the other shapes run the reference's own forward."""
    from .gru import ConvGRUEngine
    for name in ("gru04", "gru08", "gru16"):
        mod = getattr(block, name)
        _override_convgru(mod, ConvGRUEngine(mod), strict)


def _patch_update_heads(block, strict, encoder=None):
    """Per-instance ``forward`` overrides of ``encoder / disp_head / mask_feat_4`` of an IGEV / StereoBase / MonSter update block:
    CUDA inference calls the kernels serve (update.route_ok, the engines' serves()) run update.py's engines; the other shapes and
    hyper-parameters run the reference's own forward.  `encoder`: the engine class of ``encoder`` (default MotionEncoderEngine)."""
    from .update import DispHeadEngine, MaskFeatEngine, MotionEncoderEngine
    for name, cls in (("encoder", encoder or MotionEncoderEngine), ("disp_head", DispHeadEngine), ("mask_feat_4", MaskFeatEngine)):
        mod = getattr(block, name)
        _override_engine(mod, cls(mod), strict, name)


def _override_engine(mod, engine, strict, what):
    orig = mod.forward

    def forward(self, *args):
        if _trainable(self) or not _accelerable(self, *args):
            return orig(*args) if not strict else _refuse(what)
        if not engine.serves(*args):
            return orig(*args)                                      # no kernel for this shape: the reference computation
        return engine(*args)

    mod.forward = types.MethodType(forward, mod)


def _override_convgru(mod, engine, strict):
    orig = mod.forward

    def forward(self, h, cz, cr, cq, *x_list):
        if _trainable(self) or not _accelerable(self, h, cz, cr, cq, *x_list):
            return orig(h, cz, cr, cq, *x_list) if not strict else _refuse("ConvGRU")
        if not engine.serves(h, x_list):
            return orig(h, cz, cr, cq, *x_list)                     # no kernel for this shape: today's reference computation
        return engine(h, cz, cr, cq, *x_list)

    mod.forward = types.MethodType(forward, mod)


def _patch_stereobase(model, strict, backbone=True):
    g = type(model).forward.__globals__                            # stereo.modeling.models.stereobase.stereobase_gru namespace
    hg = model.cost_agg
    hg_orig = hg.forward
    agg = StereoBaseAggregation(hg)
    orig = {n: g[n] for n in ("build_gwc_volume", "build_concat_volume", "disparity_regression", "CombinedGeoEncodingVolume",
                              "context_upsample")}

    def gwc(ref, tgt, maxdisp, groups):
        if _accelerable(model, ref, tgt):
            return ops.build_gwc_volume(ref, tgt, maxdisp, groups)
        return orig["build_gwc_volume"](ref, tgt, maxdisp, groups) if not strict else _refuse("build_gwc_volume")

    def concat(ref, tgt, maxdisp):
        if _accelerable(model, ref, tgt):
            return ops.build_concat_volume(ref, tgt, maxdisp)
        return orig["build_concat_volume"](ref, tgt, maxdisp) if not strict else _refuse("build_concat_volume")

    def regression(x, maxdisp):
        if _accelerable(model, x):
            return ops.disparity_regression(x, maxdisp)
        return orig["disparity_regression"](x, maxdisp) if not strict else _refuse("disparity_regression")

    # SURVEY.md section 8(f) rows 1 and 3: the per-GRU-iteration lookup and the convex up-sampling (stereobase_gru.py:172-209)
    def geo_factory(fmap1, fmap2, volume, num_levels=2, radius=4):
        fast = _accelerable(model, fmap1, fmap2, volume)
        if not fast and strict:
            _refuse("CombinedGeoEncodingVolume")
        cls = CombinedGeoEncodingVolume if fast else orig["CombinedGeoEncodingVolume"]
        return cls(fmap1, fmap2, volume, num_levels=num_levels, radius=radius)

    def upsample(disp_low, up_weights, scale_factor=4):
        if _accelerable(model, disp_low, up_weights):
            return ops.context_upsample(disp_low, up_weights, scale_factor).to(disp_low.dtype)
        return orig["context_upsample"](disp_low, up_weights, scale_factor) if not strict else _refuse("context_upsample")

    _rebind_methods(model, {"build_gwc_volume": gwc, "build_concat_volume": concat, "disparity_regression": regression,
                            "CombinedGeoEncodingVolume": geo_factory, "context_upsample": upsample})

    def hg_forward(self, x, features, return_multi=False):
        if return_multi or not _accelerable(self, x, features):
            return hg_orig(x, features, return_multi) if not strict else _refuse("StereoBase Hourglass")
        return agg(x, features).to(x.dtype)

    hg.forward = types.MethodType(hg_forward, hg)
    _patch_convgru(model.update_block, strict)
    _patch_update_heads(model.update_block, strict)
    return model


def _volume_tail_overrides(model, strict, orig, with_corr):
    """Guarded replacements of the module-global hot-path functions LightStereo / IGEV import into their model module."""
    out = {}
    if with_corr:
        def corr(left, right, max_disp):
            if _accelerable(model, left, right):
                return ops.correlation_volume(left, right, max_disp)
            return orig["correlation_volume"](left, right, max_disp) if not strict else _refuse("correlation_volume")
        out["correlation_volume"] = corr
    else:
        def gwc(ref, tgt, maxdisp, groups):
            if _accelerable(model, ref, tgt):
                return ops.build_gwc_volume(ref, tgt, maxdisp, groups)
            return orig["build_gwc_volume"](ref, tgt, maxdisp, groups) if not strict else _refuse("build_gwc_volume")
        out["build_gwc_volume"] = gwc

    def regression(x, maxdisp):
        if _accelerable(model, x):
            return ops.disparity_regression(x, maxdisp)
        return orig["disparity_regression"](x, maxdisp) if not strict else _refuse("disparity_regression")

    def upsample(disp_low, up_weights, scale_factor=4):
        if scale_factor == 4 and _accelerable(model, disp_low, up_weights):
            return ops.context_upsample(disp_low, up_weights, 4).to(disp_low.dtype)
        if strict:
            _refuse("context_upsample")
        return orig["context_upsample"](disp_low, up_weights) if scale_factor == 4 else orig["context_upsample"](disp_low, up_weights, scale_factor)

    out["disparity_regression"], out["context_upsample"] = regression, upsample
    return out


def _patch_lightstereo(model, strict, backbone=True):
    """LightStereo (BASELINE config 4; lightstereo/lightstereo.py:44-70): correlation_volume, the 2D `Aggregation` hourglass
    (cost_agg), disparity_regression and context_upsample; backbone / refine heads stay the reference's cuDNN code."""
    from .aggregation import LightStereoAggregation
    g = type(model).forward.__globals__
    orig = {n: g[n] for n in ("correlation_volume", "disparity_regression", "context_upsample")}
    _rebind_methods(model, _volume_tail_overrides(model, strict, orig, with_corr=True))
    agg_mod = model.cost_agg
    agg_orig = agg_mod.forward
    engine = LightStereoAggregation(agg_mod)

    def agg_forward(self, x, features_left):
        if not _accelerable(self, x, features_left[:3]):
            return agg_orig(x, features_left) if not strict else _refuse("LightStereo Aggregation")
        return [t.to(x.dtype) for t in engine(x, features_left[:3])]

    agg_mod.forward = types.MethodType(agg_forward, agg_mod)
    return model


def _patch_igev(model, strict, backbone=True):
    """IGEV-Stereo (BASELINE config 5; igev/igev_stereo.py:136-213): the gwc volume, the soft-argmin regression of the initial
    disparity, the per-GRU-iteration lookup of the combined geometry-encoding volume, the three ConvGRUs of the update block
    (``update_block.gru04 / gru08 / gru16``, gru.py), its motion encoder and disp / mask heads (``update_block.encoder / disp_head /
    mask_feat_4``, update.py) and the convex up-sampling.  The hourglass(8) and the feature nets stay the reference's cuDNN code.
    Under autocast (the AMP YAML) the update block computes in fp32 and returns the reference's dtypes."""
    g = type(model).forward.__globals__
    orig = {n: g[n] for n in ("build_gwc_volume", "disparity_regression", "context_upsample", "Combined_Geo_Encoding_Volume")}
    over = _volume_tail_overrides(model, strict, orig, with_corr=False)
    over["Combined_Geo_Encoding_Volume"] = _igev_geo_factory(model, strict, orig["Combined_Geo_Encoding_Volume"])
    _rebind_methods(model, over)
    _patch_convgru(model.update_block, strict)
    _patch_update_heads(model.update_block, strict)
    return model


def _igev_geo_factory(model, strict, orig_cls):
    """Guarded replacement of IGEV's Combined_Geo_Encoding_Volume (igev/geometry.py, and MonSter's copy of it)."""
    def geo_factory(fmap1, fmap2, volume, num_levels=2, radius=4):
        fast = _accelerable(model, fmap1, fmap2, volume)
        if not fast and strict:
            _refuse("Combined_Geo_Encoding_Volume")
        cls = CombinedGeoEncodingVolume if fast else orig_cls
        return cls(fmap1, fmap2, volume, num_levels=num_levels, radius=radius)
    return geo_factory


def _patch_monster(model, strict, backbone=True):
    """MonSter (monster/monster.py, class MonSter): the stereo branch's IGEV-shaped hot path -- the gwc volume, the soft-argmin
    regression of the initial disparity, every lookup of the combined geometry-encoding volume (at disp, and at disp_mono_4x in
    the last 7 iterations), the disparity warps of features_right[0] (``disp_warp``), the ConvGRUs, motion encoders and disp /
    mask heads of ``update_block``, ``update_block_mix_stereo`` and ``update_block_mix_mono`` (the mix2 blocks' encoders on
    update.MixMotionEncoderEngine) and the convex up-sampling.  The Depth Anything encoder and decoders, feat_transfer*, the stems,
    corr_stem / corr_feature_att / cost_agg, the classifier, compute_scale_shift, REMP and the update blocks' own forward stay the
    reference's code; `backbone` has no effect.  Under autocast (the AMP YAML, bf16) every patched call computes in fp32 and
    returns the reference's dtypes."""
    from .update import MixMotionEncoderEngine
    g = type(model).forward.__globals__
    orig = {n: g[n] for n in ("build_gwc_volume", "disparity_regression", "context_upsample", "Combined_Geo_Encoding_Volume",
                              "disp_warp")}
    over = _volume_tail_overrides(model, strict, orig, with_corr=False)
    over["Combined_Geo_Encoding_Volume"] = _igev_geo_factory(model, strict, orig["Combined_Geo_Encoding_Volume"])

    def warp(img, disp, padding_mode="border"):
        """disp_warp(img, disp) -> (warped, None) on the library.  The valid mask (disp_warp(...)[1]) is not computed: the only
        method the patch rebinds that calls disp_warp, _forward_pair, takes [0]."""
        if not _accelerable(model, img, disp):
            return orig["disp_warp"](img, disp, padding_mode) if not strict else _refuse("disp_warp")
        if padding_mode != "border":
            return orig["disp_warp"](img, disp, padding_mode)           # the kernel replays the border padding only
        return ops.disp_warp(img, disp), None

    over["disp_warp"] = warp
    _rebind_methods(model, over)
    _patch_convgru(model.update_block, strict)
    _patch_update_heads(model.update_block, strict)
    for block in (model.update_block_mix_stereo, model.update_block_mix_mono):
        _patch_convgru(block, strict)
        _patch_update_heads(block, strict, encoder=MixMotionEncoderEngine)
    return model


def _patch_igev_rt(model, strict, backbone=True):
    """IGEV-RT (igev_rt/igev_rt_stereo.py:146-206, class IGEVRTtereo): the gwc volume, the hourglass(8) (``cost_agg.forward``), the
    classifier Conv3d(8 -> 1) (``classifier.forward``, which returns logits: the reference's own softmax follows), the strided
    regression of the initial disparity, the per-GRU-iteration lookup of the geometry-only encoding volume and the convex
    up-sampling.  The feature nets, hnet / cnet and the ConvGRU update block stay the reference's code; `backbone` has no effect.
    Under autocast (the AMP YAML) fp16 tensors arrive: every call computes in fp32 and returns the caller's dtype."""
    g = type(model).forward.__globals__
    orig = {n: g[n] for n in ("build_gwc_volume", "disparity_regression", "Geo_Encoding_Volume", "context_upsample")}

    def gwc(ref, tgt, maxdisp, groups):
        if _accelerable(model, ref, tgt):
            return ops.build_gwc_volume(ref, tgt, maxdisp, groups)
        return orig["build_gwc_volume"](ref, tgt, maxdisp, groups) if not strict else _refuse("build_gwc_volume")

    def regression(prob, maxdisp, interval):
        if _accelerable(model, prob):
            return ops.disparity_regression_interval(prob, maxdisp, interval)
        return orig["disparity_regression"](prob, maxdisp, interval) if not strict else _refuse("disparity_regression")

    def geo_factory(geo_volume, num_levels=2, radius=4):
        fast = _accelerable(model, geo_volume)
        if not fast and strict:
            _refuse("Geo_Encoding_Volume")
        cls = GeoEncodingVolume if fast else orig["Geo_Encoding_Volume"]
        return cls(geo_volume, num_levels=num_levels, radius=radius)

    def upsample(disp_low, up_weights):                               # IGEV-RT's version keeps dim 1: (B, 1, 4h, 4w)
        if _accelerable(model, disp_low, up_weights):
            return ops.context_upsample(disp_low, up_weights, 4).unsqueeze(1).to(disp_low.dtype)
        return orig["context_upsample"](disp_low, up_weights) if not strict else _refuse("context_upsample")

    _rebind_methods(model, {"build_gwc_volume": gwc, "disparity_regression": regression, "Geo_Encoding_Volume": geo_factory,
                            "context_upsample": upsample})

    hg, cls_mod = model.cost_agg, model.classifier
    hg_orig, cls_orig = hg.forward, cls_mod.forward
    agg, head = StereoBaseAggregation(hg), StereoBaseCostHead(cls_mod)

    def hg_forward(self, x, features):
        if not _accelerable(self, x, features):
            return hg_orig(x, features) if not strict else _refuse("IGEV-RT hourglass")
        return agg(x, features).to(x.dtype)

    def cls_forward(self, x):
        if not _accelerable(self, x):
            return cls_orig(x) if not strict else _refuse("IGEV-RT classifier")
        return head.logits(x).to(x.dtype)

    hg.forward = types.MethodType(hg_forward, hg)
    cls_mod.forward = types.MethodType(cls_forward, cls_mod)
    return model


def _patch_igevpp(model, strict, backbone=True):
    """IGEV++ (igevpp/igevpp_stereo.py:162-249, class IGEVPPStereo): the gwc volume, the classifier Conv3d(8 -> 1) of the three
    disparity ranges (``classifier.forward``, which returns logits: the reference's own softmax follows), the strided regressions of
    the three initial disparities, the per-GRU-iteration multi-range lookup (one launch), the update block's ConvGRUs, geometry
    encoders, disparity encoder, disparity head and mask head, and the convex up-sampling.  The instance-normalised hourglasses,
    patch0 / patch1, the feature nets, cnet, selective_conv, disp_conv and BasicMultiUpdateBlock.forward itself (the selective-weight
    blend, cat, pool2x, interp) stay the reference's code; `backbone` has no effect.  Under autocast (the AMP YAML) every call
    computes in fp32 and returns the reference's dtypes."""
    g = type(model).forward.__globals__
    orig = {n: g[n] for n in ("build_gwc_volume", "disparity_regression", "Combined_Geo_Encoding_Volume", "context_upsample")}

    def gwc(ref, tgt, maxdisp, groups):
        if _accelerable(model, ref, tgt):
            return ops.build_gwc_volume(ref, tgt, maxdisp, groups)
        return orig["build_gwc_volume"](ref, tgt, maxdisp, groups) if not strict else _refuse("build_gwc_volume")

    def regression(prob, maxdisp, interval):
        if _accelerable(model, prob):
            return ops.disparity_regression_interval(prob, maxdisp, interval)
        return orig["disparity_regression"](prob, maxdisp, interval) if not strict else _refuse("disparity_regression")

    def geo_factory(geo_volume0, geo_volume1, geo_volume2, init_fmap1, init_fmap2, radius=4, num_levels=2):
        fast = _accelerable(model, geo_volume0, geo_volume1, geo_volume2, init_fmap1, init_fmap2)
        if not fast and strict:
            _refuse("Combined_Geo_Encoding_Volume")
        cls = MultiRangeGeoEncodingVolume if fast else orig["Combined_Geo_Encoding_Volume"]
        return cls(geo_volume0, geo_volume1, geo_volume2, init_fmap1, init_fmap2, radius=radius, num_levels=num_levels)

    def upsample(disp_low, up_weights):                               # IGEV++'s version keeps dim 1: (B, 1, 4h, 4w)
        if _accelerable(model, disp_low, up_weights):
            return ops.context_upsample(disp_low, up_weights, 4).unsqueeze(1).to(disp_low.dtype)
        return orig["context_upsample"](disp_low, up_weights) if not strict else _refuse("context_upsample")

    _rebind_methods(model, {"build_gwc_volume": gwc, "disparity_regression": regression, "Combined_Geo_Encoding_Volume": geo_factory,
                            "context_upsample": upsample})

    cls_mod = model.classifier
    cls_orig, head = cls_mod.forward, StereoBaseCostHead(cls_mod)

    def cls_forward(self, x):
        if not _accelerable(self, x):
            return cls_orig(x) if not strict else _refuse("IGEV++ classifier")
        return head.logits(x).to(x.dtype)

    cls_mod.forward = types.MethodType(cls_forward, cls_mod)

    from .update import DispEncoderEngine, DispHeadEngine, GeoEncoderEngine, MaskFeatEngine
    block = model.update_block
    _patch_convgru(block, strict)
    for name, cls in (("encoder", DispEncoderEngine), ("geo_encoder0", GeoEncoderEngine), ("geo_encoder1", GeoEncoderEngine),
                      ("geo_encoder2", GeoEncoderEngine), ("disp_head", DispHeadEngine), ("mask_feat_4", MaskFeatEngine)):
        mod = getattr(block, name)
        _override_engine(mod, cls(mod), strict, name)
    return model


def _patch_cascade(model, strict, backbone=True):
    """CasStereo (casnet/cas_psm.py PSMNet = CasPSMNet, casnet/cas_gwc.py GwcNet = CasGwcNet): every stage's warped cost volume
    (``get_cv.forward``) and every stage's aggregation + hypothesis-weighted soft-argmin (``cost_agg[i].forward``).  The FPN
    feature extractor and get_disp_range_samples stay the reference's code inside model.forward; `backbone` has no effect."""
    gcv = model.get_cv
    gcv_orig = gcv.forward
    if type(model).__module__.rsplit(".", 1)[-1] == "cas_gwc":
        def cv_forward(self, features_left, features_right, disp_range_samples, ndisp, num_groups):
            if not _accelerable(self, features_left, features_right, disp_range_samples):
                if strict:
                    _refuse("CasGwcNet GetCostVolume")
                return gcv_orig(features_left, features_right, disp_range_samples, ndisp, num_groups)
            assert disp_range_samples.shape[1] == ndisp
            vol = ops.warped_gwc_concat_volume(features_left["gwc_feature"], features_right["gwc_feature"],
                                               features_left["concat_feature"], features_right["concat_feature"],
                                               disp_range_samples, num_groups)
            return vol.to(features_left["gwc_feature"].dtype)
    else:
        def cv_forward(self, x, y, disp_range_samples, ndisp):
            if not _accelerable(self, x, y, disp_range_samples):
                if strict:
                    _refuse("CasPSMNet GetCostVolume")
                return gcv_orig(x, y, disp_range_samples, ndisp)
            assert disp_range_samples.shape[1] == ndisp
            return ops.warped_concat_volume(x, y, disp_range_samples, mask_left=False)
    gcv.forward = types.MethodType(cv_forward, gcv)

    for agg_mod in model.cost_agg:
        _patch_cascade_agg(agg_mod, strict)
    return model


def _patch_cascade_agg(agg_mod, strict):
    agg_orig = agg_mod.forward
    engine = CascadeAggregation(agg_mod)

    def agg_forward(self, cost, FineD, FineH, FineW, disp_range_samples):
        if not _accelerable(self, cost, disp_range_samples):
            if strict:
                _refuse("CasStereo CostAggregation")
            return agg_orig(cost, FineD, FineH, FineW, disp_range_samples)
        return engine(cost, FineD, FineH, FineW, disp_range_samples).to(cost.dtype)

    agg_mod.forward = types.MethodType(agg_forward, agg_mod)


def _trainable(module):
    """True when autograd would record through the module's own parameters (a kernel call would cut them off)."""
    return torch.is_grad_enabled() and any(p.requires_grad for p in module.parameters())


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
    cp_orig, dp_orig, reg_orig = cp.forward, dp.forward, reg.forward

    def cost_forward(self, inputs):
        x, y = inputs["ref_feature"], inputs["tgt_feature"]
        if _trainable(self) or not _accelerable(self, x, y):
            return cp_orig(inputs) if not strict else _refuse("CoExCostProcessor")
        xd, yd = cv.desc(cv.conv(x[0])), cv.desc(cv.conv(y[0]))       # the reference's own 2D convolutions
        cost = ops.coex_attention_volume(xd, yd, cv.costVolume.maxdisp - 1, cv.head)
        return {"cost_volume": engine(x, cost).to(x[0].dtype)}

    def disp_forward(self, inputs):
        cost = inputs["cost_volume"]
        if _trainable(self) or not _accelerable(self, cost, inputs["ref_feature"], inputs["stem_2x"]):
            return dp_orig(inputs) if not strict else _refuse("CoExDispProcessor")
        xspx = self.spx_2(self.spx_4(inputs["ref_feature"][0]), inputs["stem_2x"])
        # the raw superpixel logits go into the kernel, which applies the reference's softmax over the 9 channels itself
        disp_pred = ops.coex_regression(cost, self.spx(xspx), self.regression.top_k, spx_is_logits=True).to(cost.dtype)
        ref_img, tgt_img = inputs["left"], inputs["right"]
        output = {"inference_disp": {"disp_est": disp_pred},
                  "visual_summary": {"image/test/image_c": torch.cat([ref_img[0], tgt_img[0]], dim=1),
                                     "image/test/disp_c": disp_pred[0]}}
        if "disp_gt" in inputs:
            output["visual_summary"] = {"image/val/image_c": torch.cat([ref_img[0], tgt_img[0]], dim=1),
                                        "image/val/disp_c": torch.cat([inputs["disp_gt"][0], disp_pred[0]], dim=0)}
        return output

    def reg_forward(self, cost, spg):
        if not _accelerable(self, cost, spg):
            return reg_orig(cost, spg) if not strict else _refuse("CoEx Regression")
        return [ops.coex_regression(cost, spg, self.top_k).to(cost.dtype)]

    cp.forward = types.MethodType(cost_forward, cp)
    dp.forward = types.MethodType(disp_forward, dp)
    reg.forward = types.MethodType(reg_forward, reg)
    return model


def _patch_msnet3d(model, strict, backbone=True):
    """MSNet3D (msnet/MSNet3D.py): everything after the 2D features in the eval forward -- the gwc volume, the MobileV2_Residual_3D
    blocks (one fused launch each), the hourglass transposed convs, classif3 and the trilinear x4 + softmax + regression tail
    (``model.forward``, per instance).  The MobileNet 2D feature extractor stays the reference's code; `backbone` has no effect.
    A block the kernel does not implement is refused here, naming it."""
    from .aggregation import MSNet3DAggregation
    engine = MSNet3DAggregation(model)
    orig = model.forward                                              # the reference's bound method

    def forward(self, data):
        left, right = data["left"], data["right"]
        if _trainable(self) or not _accelerable(self, left, right):
            return orig(data) if not strict else _refuse("MSNet3D")
        fl, fr = self.feature_extraction(left), self.feature_extraction(right)
        volume = ops.build_gwc_volume(fl, fr, self.maxdisp // 4, self.num_groups)
        return {"disp_pred": engine(volume, left.shape[2], left.shape[3]).to(left.dtype)}

    model.forward = types.MethodType(forward, model)
    return model


# CasStereo's classes are also named PSMNet / GwcNet: they are told apart by the module that defines them
_CASCADE_MODULES = {("casnet", "cas_psm"): "PSMNet", ("casnet", "cas_gwc"): "GwcNet"}

_PATCHERS = {"GwcNet": _patch_gwcnet, "PSMNet": _patch_psmnet, "StereoBase": _patch_stereobase, "LightStereo": _patch_lightstereo,
             "IGEVStereo": _patch_igev, "IGEVRTtereo": _patch_igev_rt,
             "IGEVPPStereo": _patch_igevpp, "MonSter": _patch_monster, "CoEx": _patch_coex, "MSNet3D": _patch_msnet3d}


def patch(model, strict=True, backbone=True):
    """Rebind the hot path of a reference model instance in place and return it.  backbone=True (default) also routes the
    GwcNet / PSMNet 2D extractor's residual blocks to the wgmma conv kernels in CUDA inference calls (_patch_backbone);
    backbone=False leaves the extractor entirely to the reference's cuDNN code.  For the CasStereo models (casnet.cas_psm.PSMNet,
    casnet.cas_gwc.GwcNet) `backbone` has no effect: their FPN extractor always runs the reference's code."""
    if not isinstance(model, torch.nn.Module):
        raise TypeError("patch() expects an nn.Module")
    name = type(model).__name__
    if _CASCADE_MODULES.get(tuple(type(model).__module__.split(".")[-2:])) == name:
        patcher = _patch_cascade
    elif name in _PATCHERS:
        patcher = _PATCHERS[name]
    else:
        raise NotImplementedError("patch(): no hot-path drop-in for %s (supported: %s, and CasStereo's casnet.cas_psm.PSMNet / "
                                  "casnet.cas_gwc.GwcNet)" % (name, sorted(_PATCHERS)))
    if getattr(model, "_osb_patched", False):
        return model
    patcher(model, strict, backbone)
    model._osb_patched = True
    return model
