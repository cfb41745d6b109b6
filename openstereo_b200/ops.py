"""Reference-facing operators: same names, argument meaning and error behaviour as the OpenStereo
functions they replace, executed by the sm_90a kernels in libopenstereo_b200.so.

PyTorch is plumbing here: it owns device memory (tensor.data_ptr()) and the stream
(torch.cuda.current_stream()).  All arithmetic happens in the hand-written kernels.  There is no
CPU path: a non-CUDA tensor raises, exactly like the reference's own native ops
(stereo/modeling/models/nmrf/ops/src/ms_deform_attn.h:29-38 -> "Not implemented on the CPU").
"""
import math

import torch

from . import _lib

ACT_NONE, ACT_RELU, ACT_LEAKY, ACT_RELU6 = 0, 1, 2, 3
TC_WIDTH = 128      # image width (at 1/4 resolution) handled by the tensor-core conv kernel
TC_KC = 32          # input channels per K chunk of the tensor-core conv (128-byte K-major rows)


_LAUNCH_DEVICE = [None]      # device index of the tensors of the launch being assembled (set by _stream, read by _call)


def _stream(t):
    """cudaStream_t of the CURRENT stream of the device `t` lives on (not of the current device: a model moved to cuda:1 without
    torch.cuda.set_device(1) must still launch on device 1 -- the reference's aten ops are device-guarded the same way)."""
    _LAUNCH_DEVICE[0] = t.device.index
    return torch.cuda.current_stream(t.device).cuda_stream


def _same_device(*tensors):
    devs = {t.device for t in tensors if t is not None}
    if len(devs) > 1:
        raise RuntimeError("openstereo_b200: operands live on different devices: %s" % sorted(str(d) for d in devs))


# Optional live timing: CUDA events recorded on the launching stream around every entry-point call.
_PROFILE = None


def profile_start():
    global _PROFILE
    _PROFILE = {}


def profile_stop():
    """-> {entry point name: [(start_event, stop_event), ...]}; call torch.cuda.synchronize() before reading."""
    global _PROFILE
    out, _PROFILE = _PROFILE, None
    return out or {}


def _call(name, *args, profile_as=None):
    """profile_as: the name the profile records the launch under (default: the entry point), so that an entry point serving
    another layout of the same layers keeps the existing record of those layers."""
    dev = _LAUNCH_DEVICE[0]
    if dev is not None and dev != torch.cuda.current_device():
        with torch.cuda.device(dev):                     # device guard: kernels launch where their operands live
            return _call_on_current(name, args, profile_as or name)
    return _call_on_current(name, args, profile_as or name)


def _call_on_current(name, args, key):
    if _PROFILE is None:
        return _lib.call(name, *args)
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    _lib.call(name, *args)
    stop.record()
    _PROFILE.setdefault(key, []).append((start, stop))


def _prep(t, name):
    """-> (contiguous fp32 CUDA tensor, original dtype).  Half/bf16 inputs (StereoBase under autocast,
    cfgs/stereobase/stereobase_sceneflow.yaml:50) are up-converted on load; outputs are cast back."""
    if not isinstance(t, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor" % name)
    if not t.is_cuda:
        raise RuntimeError("%s: not implemented on the CPU (openstereo_b200 has no CPU fallback)" % name)
    if t.dtype not in (torch.float32, torch.float16, torch.bfloat16):
        raise TypeError("%s: unsupported dtype %s" % (name, t.dtype))
    return t.detach().float().contiguous(), t.dtype


def _ptr(t):
    return None if t is None else t.data_ptr()


def _recording(*tensors):
    """True when autograd is recording on one of the operands: the call must go through openstereo_b200.autograd (the plain
    path detaches its inputs)."""
    return torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in tensors)


def _grad_operands(*tensors):
    for t in tensors:
        if not t.is_cuda:
            raise RuntimeError("openstereo_b200: not implemented on the CPU (openstereo_b200 has no CPU fallback)")
    return [t.float() for t in tensors]


# --------------------------------------------------------------------------- cost volumes
def build_gwc_volume(refimg_fea, targetimg_fea, maxdisp, num_groups):
    """stereo/modeling/cost_volume/cost_volume.py:68-78 -> (B, num_groups, maxdisp, H, W)."""
    if _recording(refimg_fea, targetimg_fea):
        from .autograd import GwcVolumeFn
        assert refimg_fea.dim() == 4 and refimg_fea.shape == targetimg_fea.shape and refimg_fea.shape[1] % num_groups == 0
        r, t = _grad_operands(refimg_fea, targetimg_fea)
        return GwcVolumeFn.apply(r, t, int(maxdisp), int(num_groups), False).to(refimg_fea.dtype)
    ref, dt = _prep(refimg_fea, "refimg_fea")
    tgt, _ = _prep(targetimg_fea, "targetimg_fea")
    assert ref.dim() == 4 and ref.shape == tgt.shape
    _same_device(ref, tgt)
    b, c, h, w = ref.shape
    assert c % num_groups == 0                       # cost_volume.py:61
    out = torch.empty((b, num_groups, maxdisp, h, w), dtype=torch.float32, device=ref.device)
    if out.numel():
        _call("osb_gwc_volume_fwd", ref.data_ptr(), tgt.data_ptr(), out.data_ptr(), b, c, h, w, maxdisp,
                  num_groups, _stream(out))
    return out.to(dt)


def build_concat_volume(refimg_fea, targetimg_fea, maxdisp, mask_left=True):
    """cost_volume.py:81-92 -> (B, 2C, maxdisp, H, W); mask_left=False is igev/submodule.py:216-227."""
    if _recording(refimg_fea, targetimg_fea):
        from .autograd import ConcatVolumeFn
        assert refimg_fea.dim() == 4 and refimg_fea.shape == targetimg_fea.shape
        r, t = _grad_operands(refimg_fea, targetimg_fea)
        return ConcatVolumeFn.apply(r, t, int(maxdisp), bool(mask_left)).to(refimg_fea.dtype)
    ref, dt = _prep(refimg_fea, "refimg_fea")
    tgt, _ = _prep(targetimg_fea, "targetimg_fea")
    assert ref.dim() == 4 and ref.shape == tgt.shape
    _same_device(ref, tgt)
    b, c, h, w = ref.shape
    out = torch.empty((b, 2 * c, maxdisp, h, w), dtype=torch.float32, device=ref.device)
    if out.numel():
        _call("osb_concat_volume_fwd", ref.data_ptr(), tgt.data_ptr(), out.data_ptr(), b, c, h, w, maxdisp,
                  1 if mask_left else 0, _stream(out))
    return out.to(dt)


def cat_fms(reference_fm, target_fm, max_disp=192, start_disp=0, dilation=1):
    """psmnet/psmnet_cost_processor.py:9-50.  PSMNet only ever calls it with start_disp=0, dilation=1
    (:227-232), where it equals build_concat_volume; other samplings are not on the hot path."""
    if start_disp != 0 or dilation != 1:
        raise NotImplementedError("cat_fms: only start_disp=0, dilation=1 (the PSMNet configuration) is accelerated")
    return build_concat_volume(reference_fm, target_fm, max_disp)


def correlation_volume(left_feature, right_feature, max_disp):
    """cost_volume.py:32-41 -> (B, max_disp, H, W)."""
    if _recording(left_feature, right_feature):
        from .autograd import GwcVolumeFn
        assert left_feature.dim() == 4 and left_feature.shape == right_feature.shape
        l, r = _grad_operands(left_feature, right_feature)
        return GwcVolumeFn.apply(l, r, int(max_disp), 1, False).squeeze(1).to(left_feature.dtype)
    l, dt = _prep(left_feature, "left_feature")
    r, _ = _prep(right_feature, "right_feature")
    assert l.dim() == 4 and l.shape == r.shape
    _same_device(l, r)
    b, c, h, w = l.shape
    out = torch.empty((b, max_disp, h, w), dtype=torch.float32, device=l.device)
    if out.numel():
        _call("osb_corr_volume_fwd", l.data_ptr(), r.data_ptr(), out.data_ptr(), b, c, h, w, max_disp, _stream(out))
    return out.to(dt)


def build_gwc_volume_normalized(refimg_fea, targetimg_fea, maxdisp, num_groups):
    """FoundationStereo's L2-normalised group-wise correlation volume (foundationstereo/core/submodule.py:422-461):
    every group's channel vector is F.normalize'd (eps 1e-12) before the dot product, which is a SUM over the group."""
    ref, dt = _prep(refimg_fea, "refimg_fea")
    tgt, _ = _prep(targetimg_fea, "targetimg_fea")
    assert ref.dim() == 4 and ref.shape == tgt.shape
    _same_device(ref, tgt)
    b, c, h, w = ref.shape
    assert c % num_groups == 0
    out = torch.empty((b, num_groups, maxdisp, h, w), dtype=torch.float32, device=ref.device)
    if out.numel():
        rn, tn = torch.empty_like(ref), torch.empty_like(tgt)
        _call("osb_group_l2_normalize_fwd", ref.data_ptr(), rn.data_ptr(), b, c, h, w, num_groups, 1e-12, _stream(out))
        _call("osb_group_l2_normalize_fwd", tgt.data_ptr(), tn.data_ptr(), b, c, h, w, num_groups, 1e-12, _stream(out))
        _call("osb_gwc_volume_sum_fwd", rn.data_ptr(), tn.data_ptr(), out.data_ptr(), b, c, h, w, maxdisp, num_groups, _stream(out))
    return out.to(dt)


def coex_cost_volume(x, y, maxdisp, group=1):
    """CoExCostVolume(maxdisp, group)(x, y), cost_volume/cost_volume.py:9-29 -> (B, group, maxdisp + 1, H, W):
    cost[b,g,d,h,w] = sum_k x[b,gK+k,h,w] * y[b,gK+k,h,w-d], zero where w < d (the module's left zero padding)."""
    if _recording(x, y):
        from .autograd import GwcVolumeFn
        assert x.dim() == 4 and x.shape == y.shape and x.shape[1] % group == 0
        a, b_ = _grad_operands(x, y)
        return GwcVolumeFn.apply(a, b_, int(maxdisp) + 1, int(group), True).to(x.dtype)
    xs, dt = _prep(x, "x")
    ys, _ = _prep(y, "y")
    assert xs.dim() == 4 and xs.shape == ys.shape
    _same_device(xs, ys)
    b, c, h, w = xs.shape
    assert c % group == 0
    out = torch.empty((b, group, maxdisp + 1, h, w), dtype=torch.float32, device=xs.device)
    if out.numel():
        _call("osb_gwc_volume_sum_fwd", xs.data_ptr(), ys.data_ptr(), out.data_ptr(), b, c, h, w, maxdisp + 1, group, _stream(out))
    return out.to(dt)


def build_sub_volume(feat_l, feat_r, maxdisp):
    """cost_volume/cost_volume.py:108-117 -> (B, maxdisp, H, W): L1 distance between the left features and the right features
    shifted by d; columns w < d see a zero right feature."""
    l, dt = _prep(feat_l, "feat_l")
    r, _ = _prep(feat_r, "feat_r")
    assert l.dim() == 4 and l.shape == r.shape
    _same_device(l, r)
    b, c, h, w = l.shape
    out = torch.empty((b, maxdisp, h, w), dtype=torch.float32, device=l.device)
    if out.numel():
        _call("osb_sub_volume_fwd", l.data_ptr(), r.data_ptr(), out.data_ptr(), b, c, h, w, maxdisp, _stream(out))
    return out.to(dt)


def gwc_concat_volume(ref_gwc, tgt_gwc, ref_cat, tgt_cat, maxdisp, num_groups):
    """GwcVolumeCostProcessor.forward (gwcnet_cost_processor.py:55-68): both volumes and the
    torch.cat in one launch -> (B, G + 2*Cc, maxdisp, H, W)."""
    rg, dt = _prep(ref_gwc, "ref_gwc")
    tg, _ = _prep(tgt_gwc, "tgt_gwc")
    rc, _ = _prep(ref_cat, "ref_cat")
    tc, _ = _prep(tgt_cat, "tgt_cat")
    assert rg.shape == tg.shape and rc.shape == tc.shape and rg.shape[0] == rc.shape[0] and rg.shape[2:] == rc.shape[2:]
    _same_device(rg, tg, rc, tc)
    b, cg, h, w = rg.shape
    cc = rc.shape[1]
    assert cg % num_groups == 0
    out = torch.empty((b, num_groups + 2 * cc, maxdisp, h, w), dtype=torch.float32, device=rg.device)
    if out.numel():
        _call("osb_gwc_concat_volume_fwd", rg.data_ptr(), tg.data_ptr(), rc.data_ptr(), tc.data_ptr(),
                  out.data_ptr(), b, cg, cc, h, w, maxdisp, num_groups, _stream(out))
    return out.to(dt)


def _no_autograd(name, *tensors):
    if _recording(*tensors):
        raise RuntimeError("openstereo_b200.ops.%s has no backward: call it under torch.no_grad() or on operands that do not "
                           "require grad" % name)


def warped_concat_volume(x, y, disp_samples, mask_left=False):
    """CasPSMNet's GetCostVolume.forward (casnet/cas_psm.py:286-318) -> (B, 2C, D, H, W): channels [:C] are x repeated over D
    (zeroed where w < disp when mask_left), channels [C:] are y sampled at column w - disp[b, d, h, w] like
    F.grid_sample(bilinear, zeros, align_corners=True).  disp_samples: (B, D, H, W), any real values.  No backward."""
    _no_autograd("warped_concat_volume", x, y, disp_samples)
    xs, dt = _prep(x, "x")
    ys, _ = _prep(y, "y")
    ds, _ = _prep(disp_samples, "disp_samples")
    assert xs.dim() == 4 and xs.shape == ys.shape and ds.dim() == 4
    b, c, h, w = xs.shape
    assert ds.shape[0] == b and ds.shape[2:] == (h, w)
    _same_device(xs, ys, ds)
    d = ds.shape[1]
    out = torch.empty((b, 2 * c, d, h, w), dtype=torch.float32, device=xs.device)
    if out.numel():
        _call("osb_warped_concat_volume_fwd", xs.data_ptr(), ys.data_ptr(), ds.data_ptr(), out.data_ptr(), b, c, d, h, w,
              1 if mask_left else 0, _stream(out))
    return out.to(dt)


def warped_gwc_concat_volume(x_gwc, y_gwc, x_cat, y_cat, disp_samples, num_groups):
    """CasGwcNet's GetCostVolume.forward (casnet/cas_gwc.py:263-329) -> (B, G + 2*Cc, D, H, W): the group-wise correlation of
    the masked left and warped right gwc features, then [masked left | warped right] concatenation features, in one launch.
    No backward."""
    _no_autograd("warped_gwc_concat_volume", x_gwc, y_gwc, x_cat, y_cat, disp_samples)
    xg, dt = _prep(x_gwc, "x_gwc")
    yg, _ = _prep(y_gwc, "y_gwc")
    xc, _ = _prep(x_cat, "x_cat")
    yc, _ = _prep(y_cat, "y_cat")
    ds, _ = _prep(disp_samples, "disp_samples")
    assert xg.dim() == 4 and xg.shape == yg.shape and xc.shape == yc.shape and ds.dim() == 4
    b, cg, h, w = xg.shape
    cc = xc.shape[1]
    assert xc.shape[0] == b and xc.shape[2:] == (h, w) and ds.shape[0] == b and ds.shape[2:] == (h, w)
    assert cg % num_groups == 0                                  # cas_gwc.py:312
    _same_device(xg, yg, xc, yc, ds)
    d = ds.shape[1]
    out = torch.empty((b, num_groups + 2 * cc, d, h, w), dtype=torch.float32, device=xg.device)
    if out.numel():
        _call("osb_warped_gwc_concat_volume_fwd", xg.data_ptr(), yg.data_ptr(), xc.data_ptr(), yc.data_ptr(), ds.data_ptr(),
              out.data_ptr(), b, cg, num_groups, cc, d, h, w, _stream(out))
    return out.to(dt)


def disp_warp(img, disp):
    """MonSter's disp_warp(img, disp)[0] (monster/warp.py) -> (B, C, H, W) in img's dtype: img (B, C, H, W) sampled at column
    w - disp[b, 0, h, w] like its F.grid_sample(bilinear, padding_mode='border', align_corners=False), computed in fp32 (the
    reference's interp runs with autocast off).  disp: (B, 1, H, W), any real values.  One launch; no backward."""
    _no_autograd("disp_warp", img, disp)
    x, dt = _prep(img, "img")
    d, _ = _prep(disp, "disp")
    if x.dim() != 4 or tuple(d.shape) != (x.shape[0], 1) + tuple(x.shape[2:]):
        raise ValueError("disp_warp: img %s and disp %s do not match (B, C, H, W) / (B, 1, H, W)" % (tuple(x.shape), tuple(d.shape)))
    _same_device(x, d)
    b, c, h, w = x.shape
    out = torch.empty_like(x)
    if out.numel():
        _call("osb_disp_warp_fwd", x.data_ptr(), d.data_ptr(), out.data_ptr(), b, c, h, w, _stream(out))
    return out.to(dt)


# --------------------------------------------------------------------------- soft-argmin tails
def softargmin(cost, maxdisp, keepdim=True, alpha=1.0, start=0.0, step=1.0, normalize=True):
    """disparity_regression(F.softmax(cost, 1), maxdisp) in one pass (stereobase_gru.py:163-164)."""
    if _recording(cost):
        from .autograd import SoftArgminFn
        assert cost.dim() == 4 and cost.shape[1] == maxdisp
        (cg,) = _grad_operands(cost)
        out = SoftArgminFn.apply(cg, float(alpha), float(start), float(step), bool(normalize)).to(cost.dtype)
        return out.unsqueeze(1) if keepdim else out
    c, dt = _prep(cost, "cost")
    assert len(c.shape) == 4                          # disp_regression.py:9
    b, d, h, w = c.shape
    assert d == maxdisp
    out = torch.empty((b, h, w), dtype=torch.float32, device=c.device)
    if out.numel():
        _call("osb_softargmin_fwd", c.data_ptr(), out.data_ptr(), b, d, h, w, float(alpha), float(start),
                  float(step), 1 if normalize else 0, _stream(out))
    out = out.to(dt)
    return out.unsqueeze(1) if keepdim else out


def disparity_regression(x, maxdisp, keepdim=True):
    """disp_pred/disp_regression.py:8-12 (keepdim=True) / gwcnet_disp_processor.py:22-26 (False):
    sum_d x[:, d] * d on an already-normalised x."""
    return softargmin(x, maxdisp, keepdim=keepdim, normalize=False)


def disparity_regression_interval(prob, maxdisp, interval):
    """IGEV++'s strided expectation (igevpp/submodule.py:147-151): sum_k prob[:, k] * (k * interval) over the
    maxdisp // interval hypotheses 0, interval, 2*interval, ...; prob is already normalised.  -> (B, 1, H, W)."""
    assert len(prob.shape) == 4
    return softargmin(prob, maxdisp // interval, keepdim=True, start=0.0, step=float(interval), normalize=False)


def disparity_regression_values(prob, disp_values):
    """CasStereo's expectation over per-pixel hypothesis planes (casnet/submodule.py:22-24): sum_d prob * disp_values -> (B, H, W)."""
    p, dt = _prep(prob, "prob")
    v, _ = _prep(disp_values, "disp_values")
    assert len(p.shape) == 4 and p.shape == v.shape
    _same_device(p, v)
    b, d, h, w = p.shape
    out = torch.empty((b, h, w), dtype=torch.float32, device=p.device)
    if out.numel():
        _call("osb_regression_values_fwd", p.data_ptr(), v.data_ptr(), out.data_ptr(), b, d, h, w, _stream(out))
    return out.to(dt)


def faster_soft_argmin(cost_volume, max_disp, start_disp=0, dilation=1, alpha=1.0, normalize=True):
    """FasterSoftArgmin.forward, psmnet/psmnet_disp_processor.py:51-74 -> (B, H, W)."""
    if cost_volume.dim() != 4:
        raise ValueError('expected 4D input (got {}D input)'.format(cost_volume.dim()))
    n = (max_disp + dilation - 1) // dilation
    end = start_disp + max_disp - 1
    step = (end - start_disp) / (n - 1) if n > 1 else 0.0       # torch.linspace(start, end, n)
    return softargmin(cost_volume, n, keepdim=False, alpha=alpha, start=start_disp, step=step, normalize=normalize)


def upsample_softargmin(cost, maxdisp, out_h, out_w, align_corners=False):
    """F.interpolate(cost, [maxdisp, H, W], 'trilinear') -> squeeze -> softmax -> regression, fused
    (gwcnet_disp_processor.py:129-133; psmnet_cost_processor.py:203-214 with align_corners=True).
    cost: (B, 1, D', H', W') -> (B, H, W)."""
    c, dt = _prep(cost, "cost")
    assert c.dim() == 5 and c.shape[1] == 1
    b, _, dl, hl, wl = c.shape
    out = torch.empty((b, out_h, out_w), dtype=torch.float32, device=c.device)
    if out.numel():
        _call("osb_upsample_softargmin_fwd", c.data_ptr(), out.data_ptr(), b, dl, hl, wl, maxdisp, out_h, out_w,
                  1 if align_corners else 0, _stream(out))
    return out.to(dt)


def upsample_softargmin_values(cost, disp_values, align_corners=False):
    """CasStereo's CostAggregation eval tail (casnet/cas_psm.py:268-274): F.upsample(cost, [D, H, W], 'trilinear') -> squeeze
    -> softmax over D -> sum_d p * disp_values, fused.  cost: (B, 1, D', H', W'), disp_values: (B, D, H, W) -> (B, H, W).
    No backward."""
    _no_autograd("upsample_softargmin_values", cost, disp_values)
    c, dt = _prep(cost, "cost")
    v, _ = _prep(disp_values, "disp_values")
    assert c.dim() == 5 and c.shape[1] == 1 and v.dim() == 4 and v.shape[0] == c.shape[0]
    _same_device(c, v)
    b, _, dl, hl, wl = c.shape
    _, d, h, w = v.shape
    out = torch.empty((b, h, w), dtype=torch.float32, device=c.device)
    if out.numel():
        _call("osb_upsample_softargmin_values_fwd", c.data_ptr(), v.data_ptr(), out.data_ptr(), b, dl, hl, wl, d, h, w,
              1 if align_corners else 0, _stream(out))
    return out.to(dt)


def coex_attention_volume(x, y, maxdisp, head=1):
    """CoEx's AttentionCostVolume after its convolutions (coex/coex_cost_processor.py:53-65 with the last plane dropped at :230):
    x / ||x||_2 and y / ||y||_2 over ALL channels, then cost[b,g,d,h,w] = sum over group g's channels of x_n[.., w] * y_n[.., w-d]
    for d < maxdisp, zero where w < d.  x, y (B,C,H,W) -> (B, head, maxdisp, H, W).  No backward."""
    _no_autograd("coex_attention_volume", x, y)
    xs, dt = _prep(x, "x")
    ys, _ = _prep(y, "y")
    assert xs.dim() == 4 and xs.shape == ys.shape
    _same_device(xs, ys)
    b, c, h, w = xs.shape
    assert c % head == 0
    out = torch.empty((b, head, maxdisp, h, w), dtype=torch.float32, device=xs.device)
    if out.numel():
        xn, yn = torch.empty_like(xs), torch.empty_like(ys)
        _call("osb_group_l2_normalize_fwd", xs.data_ptr(), xn.data_ptr(), b, c, h, w, 1, 0.0, _stream(out))
        _call("osb_group_l2_normalize_fwd", ys.data_ptr(), yn.data_ptr(), b, c, h, w, 1, 0.0, _stream(out))
        _call("osb_gwc_volume_sum_fwd", xn.data_ptr(), yn.data_ptr(), out.data_ptr(), b, c, h, w, maxdisp, head, _stream(out))
    return out.to(dt)


def _aligned16(t):
    return t if t.data_ptr() % 16 == 0 else t.clone()


def coex_regression(cost, spx, top_k, spx_is_logits=False):
    """CoEx's Regression.forward (eval) with upfeat (coex/coex_disp_processor.py:8-65) in one launch: cost (B,1,D,h,w) logits,
    spx (B,9,4h,4w) superpixel probabilities (or logits with spx_is_logits=True, fusing the softmax over the 9 channels) ->
    disparity (B,4h,4w).  The top k logits along D (2 <= top_k <= 8) with ties to the lower index.  No backward."""
    _no_autograd("coex_regression", cost, spx)
    c, dt = _prep(cost, "cost")
    s, _ = _prep(spx, "spx")
    assert c.dim() == 5 and c.shape[1] == 1 and s.dim() == 4
    b, _, d, h, w = c.shape
    assert tuple(s.shape) == (b, 9, 4 * h, 4 * w), (tuple(s.shape), tuple(c.shape))
    _same_device(c, s)
    out = torch.empty((b, 4 * h, 4 * w), dtype=torch.float32, device=c.device)
    if out.numel():
        _call("osb_coex_regression_fwd", c.data_ptr(), _aligned16(s).data_ptr(), out.data_ptr(), b, d, h, w, int(top_k),
              1 if spx_is_logits else 0, _stream(out))
    return out.to(dt)


def nearest_resize3d(x, size):
    """F.interpolate(x, size=(D, H, W), mode='nearest') for a (B,C,D,H,W) volume, bit-equal (a gather with aten's source index).
    No backward."""
    _no_autograd("nearest_resize3d", x)
    xs, dt = _prep(x, "x")
    assert xs.dim() == 5 and len(size) == 3
    b, c, di, hi, wi = xs.shape
    do, ho, wo = (int(v) for v in size)
    out = torch.empty((b, c, do, ho, wo), dtype=torch.float32, device=xs.device)
    if out.numel():
        _call("osb_nearest_resize3d_fwd", xs.data_ptr(), out.data_ptr(), b * c, di, hi, wi, do, ho, wo, _stream(out))
    return out.to(dt)


def mbv2_block3d(x, w_exp, scale1, shift1, w_dw, scale2, shift2, w_proj, scale3, shift3, residual=None, stride=1,
                 in_ndhwc=False, out_ndhwc=False):
    """MSNet3D's MobileV2_Residual_3D (msnet/submodule.py:136-173) in one launch: 1x1x1 expand + BN + ReLU6, depthwise 3x3x3
    (stride 1 or 2, padding 1) + BN + ReLU6, 1x1x1 project + BN, + residual.  BNs folded to (scale, shift); w_exp (Cin, Chid),
    w_dw (27, Chid) tap-major, w_proj (Chid, Cout).  x (B,Cin,D,H,W), or (B,D,H,W,Cin) with in_ndhwc; the result and the residual
    are (B,Cout,Do,Ho,Wo), or (B,Do,Ho,Wo,Cout) with out_ndhwc, n_o = ceil(n / stride).  CUDA fp32 contiguous tensors.  No backward."""
    _no_autograd("mbv2_block3d", x, w_exp, w_dw, w_proj, residual)
    ts = [x, w_exp, scale1, shift1, w_dw, scale2, shift2, w_proj, scale3, shift3] + ([] if residual is None else [residual])
    for t in ts:
        if not t.is_cuda:
            raise RuntimeError("mbv2_block3d: not implemented on the CPU (openstereo_b200 has no CPU fallback)")
        assert t.dtype == torch.float32 and t.is_contiguous()
    _same_device(*ts)
    assert x.dim() == 5
    if in_ndhwc:
        b, d, h, w, cin = x.shape
    else:
        b, cin, d, h, w = x.shape
    chid, cout = w_exp.shape[1], w_proj.shape[1]
    assert tuple(w_exp.shape) == (cin, chid) and tuple(w_dw.shape) == (27, chid) and tuple(w_proj.shape) == (chid, cout)
    do, ho, wo = (d - 1) // stride + 1, (h - 1) // stride + 1, (w - 1) // stride + 1
    shape = (b, do, ho, wo, cout) if out_ndhwc else (b, cout, do, ho, wo)
    y = torch.empty(shape, dtype=torch.float32, device=x.device)
    if residual is not None:
        assert tuple(residual.shape) == shape
    _call("osb_mbv2_block3d_fwd", x.data_ptr(), w_exp.data_ptr(), scale1.data_ptr(), shift1.data_ptr(), w_dw.data_ptr(),
          scale2.data_ptr(), shift2.data_ptr(), w_proj.data_ptr(), scale3.data_ptr(), shift3.data_ptr(), _ptr(residual), y.data_ptr(),
          b, cin, chid, cout, d, h, w, int(stride), 1 if in_ndhwc else 0, 1 if out_ndhwc else 0, _stream(y))
    return y


def epe_partial(disp_pred, disp_gt, maxdisp):
    """Per-image {sum |pred-gt| over 0<gt<maxdisp, #valid} -> (B, 2) fp32
    (metric_per_image.py:32-41 with the mask of trainer_template.py:288)."""
    p, _ = _prep(disp_pred, "disp_pred")
    g, _ = _prep(disp_gt, "disp_gt")
    assert p.shape == g.shape and p.dim() == 3
    b = p.shape[0]
    out = torch.empty((b, 2), dtype=torch.float32, device=p.device)
    _call("osb_epe_partial_fwd", p.data_ptr(), g.data_ptr(), out.data_ptr(), b, p.shape[1] * p.shape[2],
              float(maxdisp), _stream(out))
    return out


def epe_per_image(disp_pred, disp_gt, maxdisp):
    part = epe_partial(disp_pred, disp_gt, maxdisp)
    return torch.where(part[:, 1] > 0, part[:, 0] / part[:, 1], torch.zeros_like(part[:, 0]))


# --------------------------------------------------------------------------- 3D aggregation primitives
def pack_conv_weight(weight):
    """(Cout, Cin, k, k, k) Conv3d parameter -> (Cin, k^3, Cout) contiguous fp32."""
    co, ci = weight.shape[:2]
    return weight.detach().float().permute(1, 2, 3, 4, 0).reshape(ci, -1, co).contiguous()


def pack_deconv_weight(weight):
    """(Cin, Cout, k, k, k) ConvTranspose3d parameter -> (Cin, k^3, Cout) contiguous fp32."""
    ci, co = weight.shape[:2]
    return weight.detach().float().permute(0, 2, 3, 4, 1).reshape(ci, -1, co).contiguous()


def fold_bn(bn):
    """Eval-mode BatchNorm -> (scale, shift) with y = x*scale + shift."""
    scale = (bn.weight.detach().float() / torch.sqrt(bn.running_var.detach().float() + bn.eps))
    shift = bn.bias.detach().float() - bn.running_mean.detach().float() * scale
    return scale.contiguous(), shift.contiguous()


def conv3d_k3(x, w_packed, scale=None, shift=None, residual=None, gate=None, stride=1, act=ACT_NONE):
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 5
    b, cin, d, h, w = x.shape
    assert w_packed.shape[0] == cin and w_packed.shape[1] == 27
    cout = w_packed.shape[2]
    do, ho, wo = (d - 1) // stride + 1, (h - 1) // stride + 1, (w - 1) // stride + 1
    y = torch.empty((b, cout, do, ho, wo), dtype=torch.float32, device=x.device)
    if residual is not None:
        assert residual.shape == y.shape and residual.is_contiguous()
    if gate is not None:
        assert gate.shape == (b, cout, ho, wo) and gate.is_contiguous()
    _call("osb_conv3d_k3_bn_act_fwd", x.data_ptr(), w_packed.data_ptr(), _ptr(scale), _ptr(shift), _ptr(residual),
              _ptr(gate), y.data_ptr(), b, cin, cout, d, h, w, stride, act, _stream(y))
    return y


def deconv3d(x, w_packed, scale=None, shift=None, residual=None, kernel=3, act=ACT_NONE):
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 5
    b, cin, d, h, w = x.shape
    assert w_packed.shape[0] == cin and w_packed.shape[1] == kernel ** 3
    cout = w_packed.shape[2]
    y = torch.empty((b, cout, 2 * d, 2 * h, 2 * w), dtype=torch.float32, device=x.device)
    if residual is not None:
        assert residual.shape == y.shape and residual.is_contiguous()
    _call("osb_deconv3d_bn_act_fwd", x.data_ptr(), w_packed.data_ptr(), _ptr(scale), _ptr(shift), _ptr(residual),
              y.data_ptr(), b, cin, cout, d, h, w, kernel, act, _stream(y))
    return y


def conv3d_1x1(x0, w_packed, scale=None, shift=None, residual=None, gate=None, act=ACT_NONE, x1=None,
               sigmoid_out=False):
    """1x1x1 conv over the channel concat of x0 (and x1).  4-D inputs are treated as D=1 volumes."""
    squeeze = x0.dim() == 4
    if squeeze:
        x0 = x0.unsqueeze(2)
        x1 = None if x1 is None else x1.unsqueeze(2)
    assert x0.is_cuda and x0.dtype == torch.float32 and x0.is_contiguous()
    b, c0, d, h, w = x0.shape
    cin = c0 + (0 if x1 is None else x1.shape[1])
    if x1 is not None:
        assert x1.is_contiguous() and x1.shape[0] == b and x1.shape[2:] == x0.shape[2:]
    assert w_packed.shape[0] == cin
    cout = w_packed.shape[-1]
    y = torch.empty((b, cout, d, h, w), dtype=torch.float32, device=x0.device)
    _call("osb_conv3d_1x1_bn_act_fwd", x0.data_ptr(), _ptr(x1), c0, w_packed.data_ptr(), _ptr(scale), _ptr(shift),
              _ptr(residual), _ptr(gate), y.data_ptr(), b, cin, cout, d, h, w, act, 1 if sigmoid_out else 0, _stream(y))
    return y.squeeze(2) if squeeze else y


# --------------------------------------------------------------------------- tensor-core conv (wgmma, 3xFP16 split)
def conv3d_tc_supported(cin, cout, w, stride=1):
    return bool(_lib.lib.osb_conv3d_tc_supported(int(cin), int(cout), int(w), int(stride)))


def conv3d_tc_kc(cin, cout, w, stride=1):
    """K chunk (16 / 32) of the tensor-core kernel variant serving this shape, 0 if there is none."""
    return int(_lib.lib.osb_conv3d_tc_kc(int(cin), int(cout), int(w), int(stride)))


def tc_operand_kind():
    """MMA kind of the tensor-core convolutions: "f16" (3xFP16 operand split, csrc/tc_common.cuh)."""
    return "f16"


TC_ACT_SCALE_LOG2 = 4        # activations are staged as x * 2^4 (csrc/tc_common.cuh: TC_ACT_SCALE); |x| must stay below 4094
TC_WEIGHT_TOP_LOG2 = 15      # per output channel, weights are scaled so that max |w| * 2^e lies in [2^14, 2^15)


def set_rz_kappa(kappa):
    """Override the accumulator round-towards-zero correction constant of the tensor-core convs (include/openstereo_b200.h:
    osb_set_rz_kappa); returns the previous value.  Calibration / bisect only."""
    return float(_lib.lib.osb_set_rz_kappa(float(kappa)))


def set_persistent_grid_cap(cap):
    """Clamp the grid of the persistent kernels (tensor-core convs, volume constructors) to `cap` CTAs, 0 = no cap (include/
    openstereo_b200.h: osb_set_persistent_grid_cap); returns the previous cap.  Tests only: cap = 1 runs every work item on one CTA."""
    return int(_lib.lib.osb_set_persistent_grid_cap(int(cap)))


def tc_last_variant():
    """Template arguments of the tensor-core conv instantiation this thread launched last, e.g. "tcg<64,16,64,1,1,0,1>"."""
    return (_lib.lib.osb_tc_last_variant() or b"").decode()


def volume_last_variant():
    """Cost-volume kernel this thread launched last, e.g. "volume<1,0,tma>" (VEC, K4, TMA or plain-load staging)."""
    return (_lib.lib.osb_volume_last_variant() or b"").decode()


def tc_overflow_count(device=None, reset=False):
    """Number of loader threads (since the last reset) that staged an activation outside the fp16 range of the tensor-core
    convolutions (|x| >= 4094).  Synchronises the current stream of `device`.  0 = every result is valid."""
    import ctypes
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    out = ctypes.c_uint(0)
    with torch.cuda.device(dev):
        rc = _lib.lib.osb_tc_overflow_count(torch.cuda.current_stream(dev).cuda_stream, 1 if reset else 0, ctypes.byref(out))
    if rc != 0:
        raise RuntimeError("osb_tc_overflow_count: %s" % (_lib.lib.osb_last_error() or b"").decode())
    return int(out.value)


class TcOverflowMonitor:
    """Asynchronous watch on the fp16-range counter (include/openstereo_b200.h: osb_tc_overflow_poll).  An engine calls poll()
    after its last kernel (a 4-byte device->pinned-host copy on the current stream, no synchronisation) and check() before its
    next forward: once the copy has landed, a non-zero count raises -- an activation left the +-4094 range of the tensor-core
    convolutions and the previous result was computed from saturated operands."""
    _instances = {}

    @classmethod
    def get(cls, device):
        dev = torch.device(device)
        if dev.index not in cls._instances:
            cls._instances[dev.index] = cls(dev)
        return cls._instances[dev.index]

    def __init__(self, device):
        self.device = device
        self.host = torch.zeros(1, dtype=torch.int32).pin_memory()
        self.event = None

    def poll(self):
        stream = torch.cuda.current_stream(self.device)
        with torch.cuda.device(self.device):
            rc = _lib.lib.osb_tc_overflow_poll(stream.cuda_stream, self.host.data_ptr())
        if rc != 0:
            raise RuntimeError("osb_tc_overflow_poll: %s" % (_lib.lib.osb_last_error() or b"").decode())
        self.event = torch.cuda.Event()
        self.event.record(stream)

    def check(self):
        if self.event is not None and self.event.query():
            self.event = None
            n = int(self.host.item()) & 0xFFFFFFFF
            if n:
                tc_overflow_count(self.device, reset=True)
                raise RuntimeError("openstereo_b200: %d loader threads met activations outside the fp16 range of the tensor-core "
                                   "convolutions (|x| >= 4094); the previous result is invalid.  Run those layers with "
                                   "aggregation.USE_TENSOR_CORES = False" % n)


def f16_split(w):
    """fp32 tensor (already scaled into the fp16 range) -> (hi, lo) fp16 with hi = rn(w), lo = rn(w - hi):
    |w - hi - lo| <= 2^-22 |w| while lo stays a normal fp16 number (|w| >= 2^-3), 2^-25 absolute below that."""
    w = w.contiguous()
    hi = w.to(torch.float16)
    lo = (w - hi.float()).to(torch.float16)
    return hi, lo


class TcWeight:
    """A conv weight packed for the wgmma kernels: `data` fp16 [3 kd][Cin/kc][3 kh][3*Cout (kw-major)][kc hi | kc lo] of
    w * 2^e_c with the 16-byte chunks of every row stored in the wgmma swizzle order (pack_tc_weight), and `inv` = 2^-(e_c + TC_ACT_SCALE_LOG2) per output channel -- the exact factor the epilogue must apply.
    `cout` is the packed row count per kw slice (narrow heads are zero-padded to 16), `cout_real` the layer's channels."""
    __slots__ = ("data", "inv", "kc", "cout", "cout_real", "ksize", "_eff")

    def __init__(self, data, inv, kc, cout, cout_real=None, ksize=3):
        self.data, self.inv, self.kc, self.cout, self._eff = data, inv, kc, cout, None
        self.cout_real = cout if cout_real is None else cout_real
        self.ksize = ksize                                                  # 3, or 4 for the k4-s2 transposed conv

    def eff_scale(self, scale):
        """Epilogue scale vector: folded-BN scale (or 1) times the exact power-of-two un-scaling of this weight."""
        key = None if scale is None else (scale.data_ptr(), scale._version)
        if self._eff is None or self._eff[0] != key:
            if scale is not None and scale.numel() < self.inv.numel():            # zero-padded head: pad the BN scale too
                scale = torch.cat((scale.float(), scale.new_ones(self.inv.numel() - scale.numel()).float()))
            eff = self.inv if scale is None else scale.float() * self.inv
            self._eff = (key, eff.contiguous())
        return self._eff[1]


def pack_tc_weight(weight, kc=None, kw_order=(0, 1, 2), pad_cout_to=None):
    """(Cout, Cin, k, k, k) fp32 Conv3d parameter (k = 3, or 4 for the k4-s2 transposed conv) -> TcWeight (see there).  Per output
    channel the weights are scaled by the power of two that puts max |w| into [2^14, 2^15) (exact; undone by TcWeight.inv), then
    split with f16_split.  kw_order lists the kw slices in the order the kernel stacks them along N."""
    w = weight.detach().float()
    cout_real, cin = w.shape[:2]
    k = int(w.shape[2])
    if pad_cout_to is not None and cout_real < pad_cout_to:             # narrow classifier heads ride the COUT = 16 kernel variant
        w = torch.cat((w, w.new_zeros((pad_cout_to - cout_real,) + tuple(w.shape[1:]))), 0)
    cout = w.shape[0]
    kc = TC_KC if kc is None else kc
    assert kc in (16, 32) and cin % kc == 0 and k in (3, 4) and tuple(w.shape[2:]) == (k, k, k) and len(kw_order) == k
    amax = w.abs().amax(dim=(1, 2, 3, 4))
    _, ex = torch.frexp(amax)                                           # amax = m * 2^ex, m in [0.5, 1)
    e = torch.where(amax > 0, TC_WEIGHT_TOP_LOG2 - ex, torch.zeros_like(ex)).clamp(-40, 40)
    ws = torch.ldexp(w, e.view(-1, 1, 1, 1, 1))
    hi, lo = f16_split(ws)
    both = torch.stack((hi, lo), 0)                                    # (2, co, ci, kd, kh, kw)
    both = both[..., list(kw_order)]                                   # stride-2 kernel wants kw slices as (1, 0, 2)
    both = both.contiguous().view(2, cout, cin // kc, kc, k, k, k)     # (half, co, chunk, ci, kd, kh, kw)
    both = both.permute(4, 2, 5, 6, 1, 0, 3)                           # (kd, chunk, kh, kw, co, half, ci)
    data = both.reshape(k, cin // kc, k, k * cout, 2 * kc).contiguous()
    # Pre-swizzle: the kernels copy a (kd, chunk, kh) slice into shared memory with ONE 1-D TMA bulk copy, so global memory already
    # holds the wgmma K-major swizzled layout: 16-byte chunk c of row n sits at chunk c ^ (n & 7) (128-byte rows, SWIZZLE_128B) or
    # c ^ ((n >> 1) & 3) (64-byte rows, SWIZZLE_64B) -- an XOR within the row, i.e. a gather with an involutive index.
    cpr = (2 * kc) // 8                                                 # 16-byte chunks per row (8 halfs each)
    rows = torch.arange(k * cout, device=data.device)
    key = (rows & 7) if kc == 32 else ((rows >> 1) & 3)
    src = torch.arange(cpr, device=data.device).view(1, cpr) ^ key.view(-1, 1)              # (rows, cpr): chunk stored at position c
    data = data.view(k, cin // kc, k, k * cout, cpr, 8)
    data = torch.gather(data, 4, src.view(1, 1, 1, k * cout, cpr, 1).expand(k, cin // kc, k, k * cout, cpr, 8).contiguous())
    data = data.reshape(k, cin // kc, k, k * cout, 2 * kc).contiguous()
    inv = torch.ldexp(torch.ones_like(amax), -(e + TC_ACT_SCALE_LOG2))
    return TcWeight(data, inv.contiguous(), kc, cout, cout_real, ksize=k)


def _tc_args(w_split, cin, kc, scale):
    assert isinstance(w_split, TcWeight) and w_split.kc == kc
    k = w_split.ksize
    assert tuple(w_split.data.shape) == (k, cin // kc, k, k * w_split.cout, 2 * kc) and w_split.data.dtype == torch.float16
    assert w_split.data.is_contiguous() and w_split.data.is_cuda
    return w_split.data.data_ptr(), w_split.eff_scale(scale)


def to_ndhwc(x, pad_to=None):
    """(B,C,D,H,W) -> (B,D,H,W,C) contiguous fp32, on the device; pad_to > C appends zero channels (channel plans that are not
    multiples of 16 run on the tensor-core kernels zero-padded)."""
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 5
    b, c, d, h, w = x.shape
    cp = c if pad_to is None else int(pad_to)
    assert cp >= c
    y = torch.empty((b, d, h, w, cp), dtype=torch.float32, device=x.device)
    if cp == c:
        _call("osb_ncdhw_to_ndhwc", x.data_ptr(), y.data_ptr(), b, c, d, h, w, _stream(y))
    else:
        _call("osb_ncdhw_to_ndhwc_pad", x.data_ptr(), y.data_ptr(), b, c, cp, d, h, w, _stream(y))
    return y


# Split NDHWC activations (include/openstereo_b200.h, csrc/tc_common.cuh): a channels-last (B,D,H,W,C) fp32 tensor held as
# (B,D,H,W,2C) fp16, per voxel granules of 16 channels [16 hi | 16 lo] of x * 2^4 -- the operand rows of the wgmma layers, so a
# layer that reads one skips the conversion of its input.  Same bytes as the fp32 tensor; values keep about 22 significant bits.
SPLIT_GRANULE = 16
LAYOUT_NCDHW, LAYOUT_NDHWC, LAYOUT_SPLIT = 0, 1, 2


def is_split(t):
    """True for a split NDHWC activation (fp16, channels last, 2C entries per voxel)."""
    return t.dtype == torch.float16 and t.dim() == 5


def to_split(x):
    """(B,C,D,H,W) fp32 -> split NDHWC (B,D,H,W,2C) fp16, C a multiple of 16.  Values outside +-4094 saturate and raise
    tc_overflow_count."""
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 5
    b, c, d, h, w = x.shape
    assert c % SPLIT_GRANULE == 0, "split activations need a multiple of %d channels" % SPLIT_GRANULE
    y = torch.empty((b, d, h, w, 2 * c), dtype=torch.float16, device=x.device)
    _call("osb_ncdhw_to_split", x.data_ptr(), y.data_ptr(), b, c, d, h, w, _stream(y))
    return y


def from_split(x_split):
    """split (B,D,H,W,2C) fp16 -> (B,D,H,W,C) fp32 channels-last, each value (hi + lo) / 16 as the kernels decode it.  For tests
    and inspection: the layers read split tensors directly."""
    assert is_split(x_split) and x_split.shape[4] % (2 * SPLIT_GRANULE) == 0
    g = x_split.shape[4] // (2 * SPLIT_GRANULE)
    v = x_split.view(*x_split.shape[:4], g, 2, SPLIT_GRANULE).float()
    return ((v[..., 0, :] + v[..., 1, :]) * (1.0 / 16)).reshape(*x_split.shape[:4], g * SPLIT_GRANULE).contiguous()


def conv3d_k3_tc(x_ndhwc, w_split, scale=None, shift=None, residual=None, act=ACT_NONE, out_ndhwc=True, res_ndhwc=True,
                 in_ncdhw=False, gate=None, out_split=False):
    """3x3x3 stride-1 conv + folded BN + residual + activation on the tensor cores.  x_ndhwc: (B,D,H,W,Cin), or the NCDHW
    tensor (B,Cin,D,H,W) with in_ncdhw=True (W = 128 layers only: the cost volume goes in as the volume kernel wrote it).
    W = 128 layers also take x and a channels-last residual as split activations (to_split), and out_split=True returns y as one;
    a split residual enters as (hi + lo) / 16."""
    assert x_ndhwc.is_cuda and x_ndhwc.dtype in (torch.float32, torch.float16) and x_ndhwc.is_contiguous() and x_ndhwc.dim() == 5
    in_split = is_split(x_ndhwc)
    assert not (in_split and in_ncdhw)
    if in_ncdhw:
        b, cin, d, h, w = x_ndhwc.shape
    else:
        b, d, h, w, cin = x_ndhwc.shape
        if in_split:
            cin = w_split.data.shape[1] * w_split.kc
            if x_ndhwc.shape[4] != 2 * cin:
                raise ValueError("conv3d_k3_tc: an fp16 input is read as split activations (ops.to_split), 2 * Cin = %d entries per "
                                 "voxel for this weight; got %d" % (2 * cin, x_ndhwc.shape[4]))
    cout = w_split.cout_real
    kc = conv3d_tc_kc(cin, cout, w)
    assert kc
    wptr, scale = _tc_args(w_split, cin, kc, scale)
    if shift is not None and shift.numel() < w_split.cout:               # zero-padded head
        shift = torch.cat((shift.float(), shift.new_zeros(w_split.cout - shift.numel()).float()))
    res_split = residual is not None and is_split(residual)
    if residual is not None:
        want = (b, d, h, w, 2 * cout if res_split else cout) if res_ndhwc else (b, cout, d, h, w)
        assert tuple(residual.shape) == want and residual.is_contiguous() and (res_split or residual.dtype == torch.float32)
    if in_split or out_split or res_split:
        assert gate is None and (out_ndhwc or not out_split)
        shape = (b, d, h, w, 2 * cout if out_split else cout) if out_ndhwc else (b, cout, d, h, w)
        y = torch.empty(shape, dtype=torch.float16 if out_split else torch.float32, device=x_ndhwc.device)
        layout = lambda split, ndhwc: LAYOUT_SPLIT if split else (LAYOUT_NDHWC if ndhwc else LAYOUT_NCDHW)
        # profiled as the fp32 entry point reading the same input layout would be: the same kernel and the same layers
        _call("osb_conv3d_k3_tc_split_fwd", x_ndhwc.data_ptr(), wptr, _ptr(scale), _ptr(shift), _ptr(residual), y.data_ptr(),
              b, cin, cout, d, h, w, act, layout(in_split, not in_ncdhw), layout(out_split, out_ndhwc), layout(res_split, res_ndhwc),
              _stream(y), profile_as="osb_conv3d_k3_tc_ncdhw_fwd" if in_ncdhw else "osb_conv3d_k3_tc_fwd")
        return y
    shape = (b, d, h, w, cout) if out_ndhwc else (b, cout, d, h, w)
    y = torch.empty(shape, dtype=torch.float32, device=x_ndhwc.device)
    assert not in_ncdhw or kc == 32
    if gate is not None:                                                     # FeatureAtt: (B,H,W,Cout) multiplier after the activation
        assert kc == 16 and out_ndhwc and res_ndhwc and not in_ncdhw
        assert tuple(gate.shape) == (b, h, w, cout) and gate.is_contiguous() and gate.dtype == torch.float32 and gate.is_cuda
        _call("osb_conv3d_k3_tc_gate_fwd", x_ndhwc.data_ptr(), wptr, _ptr(scale), _ptr(shift), _ptr(residual), gate.data_ptr(),
              y.data_ptr(), b, cin, cout, d, h, w, act, _stream(y))
        return y
    _call("osb_conv3d_k3_tc_ncdhw_fwd" if in_ncdhw else "osb_conv3d_k3_tc_fwd", x_ndhwc.data_ptr(), wptr, _ptr(scale), _ptr(shift), _ptr(residual),
          y.data_ptr(), b, cin, cout, d, h, w, act, 1 if out_ndhwc else 0, 1 if res_ndhwc else 0, _stream(y))
    return y


def conv3d_s2_tc_supported(cin, cout, d, h, w):
    return bool(_lib.lib.osb_conv3d_s2_tc_supported(int(cin), int(cout), int(d), int(h), int(w)))


def conv3d_k3_s2_tc(x_ndhwc, w_split, scale=None, shift=None, residual=None, act=ACT_NONE, out_ndhwc=False, res_ndhwc=False):
    """3x3x3 STRIDE-2 conv + folded BN + residual + activation on the tensor cores.  x_ndhwc: (B,D,H,W,Cin), even D,H,W, or D = 1:
    a stride-2 3x3 Conv2d as one plane (its taps at kd = 1 of the weight, one output plane);
    w_split = pack_tc_weight(weight, 16, kw_order=(1, 0, 2))."""
    assert x_ndhwc.is_cuda and x_ndhwc.dtype == torch.float32 and x_ndhwc.is_contiguous() and x_ndhwc.dim() == 5
    b, d, h, w, cin = x_ndhwc.shape
    cout = w_split.cout
    wptr, scale = _tc_args(w_split, cin, 16, scale)
    do, ho, wo = max(1, d // 2), h // 2, w // 2
    shape = (b, do, ho, wo, cout) if out_ndhwc else (b, cout, do, ho, wo)
    y = torch.empty(shape, dtype=torch.float32, device=x_ndhwc.device)
    if residual is not None:
        want = (b, do, ho, wo, cout) if res_ndhwc else (b, cout, do, ho, wo)
        assert tuple(residual.shape) == want and residual.is_contiguous()
    _call("osb_conv3d_k3_s2_tc_fwd", x_ndhwc.data_ptr(), wptr, _ptr(scale), _ptr(shift), _ptr(residual),
          y.data_ptr(), b, cin, cout, d, h, w, act, 1 if out_ndhwc else 0, 1 if res_ndhwc else 0, _stream(y))
    return y


def deconv3d_tc_supported(cin, cout, w):
    return bool(_lib.lib.osb_deconv3d_tc_supported(int(cin), int(cout), int(w)))


def pack_tc_deconv_weight(weight):
    """(Cin, Cout, 3, 3, 3) ConvTranspose3d parameter -> TcWeight, 16-channel chunks, kw slices ordered (1, 2, 0):
    even output columns come from tap 1, odd ones from taps 2 (same input column) and 0 (next input column).
    (Cin, Cout, 4, 4, 4) (k4 s2 p1): kw slices (1, 3, 2, 0) -- even columns taps 1 (same input column) and 3 (previous one), odd
    columns taps 2 (same) and 0 (next)."""
    w = weight.detach().float().permute(1, 0, 2, 3, 4).contiguous()
    return pack_tc_weight(w, 16, kw_order=(1, 2, 0) if w.shape[2] == 3 else (1, 3, 2, 0))


def deconv3d_k4_tc_supported(cin, cout, w):
    return bool(_lib.lib.osb_deconv3d_k4_tc_supported(int(cin), int(cout), int(w)))


def deconv3d_k4_tc(x_ndhwc, w_split, scale=None, shift=None, residual=None, act=ACT_NONE, out_ndhwc=True, res_ndhwc=True,
                   cout_real=None):
    """ConvTranspose3d(k4, s2, p1) + folded BN + residual + activation on the tensor cores.  x_ndhwc: (B,D,H,W,Cin); cout_real <
    packed Cout (zero-padded channel plan) is allowed for an NCDHW output, which then holds only the real channels."""
    assert x_ndhwc.is_cuda and x_ndhwc.dtype == torch.float32 and x_ndhwc.is_contiguous() and x_ndhwc.dim() == 5
    b, d, h, w, cin = x_ndhwc.shape
    cout = w_split.cout
    creal = cout if cout_real is None else int(cout_real)
    assert w_split.ksize == 4 and (out_ndhwc is False or creal == cout)
    wptr, scale = _tc_args(w_split, cin, 16, scale)
    shape = (b, 2 * d, 2 * h, 2 * w, cout) if out_ndhwc else (b, creal, 2 * d, 2 * h, 2 * w)
    y = torch.empty(shape, dtype=torch.float32, device=x_ndhwc.device)
    if residual is not None:
        want = (b, 2 * d, 2 * h, 2 * w, cout) if res_ndhwc else (b, creal, 2 * d, 2 * h, 2 * w)
        assert tuple(residual.shape) == want and residual.is_contiguous()
    _call("osb_deconv3d_k4_tc_fwd", x_ndhwc.data_ptr(), wptr, _ptr(scale), _ptr(shift), _ptr(residual),
          y.data_ptr(), b, cin, cout, creal, d, h, w, act, 1 if out_ndhwc else 0, 1 if res_ndhwc else 0, _stream(y))
    return y


def tc_slice(kind, x_ndhwc, w_split, scale, shift, y, coff, act=ACT_NONE, gate=None):
    """One output-channel SLICE of a tensor-core conv (include/openstereo_b200.h: *_cs_fwd): channels [coff, coff + w_split.cout) of
    the preallocated channels-last `y` (..., Ctot).  kind: "s1" (3x3x3 stride 1, optional (B,H,W,Ctot) gate), "s2" (stride 2) or
    "dc4" (ConvTranspose3d k4 s2 p1).  scale / shift: this slice's folded BN."""
    assert x_ndhwc.is_cuda and x_ndhwc.dtype == torch.float32 and x_ndhwc.is_contiguous() and x_ndhwc.dim() == 5
    assert y.is_contiguous() and y.dtype == torch.float32 and y.dim() == 5
    b, d, h, w, cin = x_ndhwc.shape
    cout, ctot = w_split.cout, y.shape[-1]
    assert 0 <= coff and coff + cout <= ctot and coff % 4 == 0
    wptr, scale = _tc_args(w_split, cin, 16, scale)
    yp = y.data_ptr() + 4 * coff
    if kind == "s1":
        assert tuple(y.shape[:4]) == (b, d, h, w)
        gp = None
        if gate is not None:
            assert tuple(gate.shape) == (b, h, w, ctot) and gate.is_contiguous()
            gp = gate.data_ptr() + 4 * coff
        _call("osb_conv3d_k3_tc_cs_fwd", x_ndhwc.data_ptr(), wptr, _ptr(scale), _ptr(shift), None, gp, yp, b, cin, cout, d, h, w, act,
              ctot, _stream(y))
    elif kind == "s2":
        assert tuple(y.shape[:4]) == (b, d // 2, h // 2, w // 2) and gate is None
        _call("osb_conv3d_k3_s2_tc_cs_fwd", x_ndhwc.data_ptr(), wptr, _ptr(scale), _ptr(shift), yp, b, cin, cout, d, h, w, act, ctot,
              _stream(y))
    else:
        assert kind == "dc4" and tuple(y.shape[:4]) == (b, 2 * d, 2 * h, 2 * w) and gate is None and w_split.ksize == 4
        _call("osb_deconv3d_k4_tc_cs_fwd", x_ndhwc.data_ptr(), wptr, _ptr(scale), _ptr(shift), yp, b, cin, cout, d, h, w, act, ctot,
              _stream(y))
    return y


def feature_att_gate(feat, w1, scale1, shift1, w2, scale2, shift2, pad_to=None, act1=ACT_LEAKY):
    """FeatureAtt's gate (igev_blocks.py:35-48) in one launch: feat (B,Cf,H,W) NCHW -> sigmoid gate (B,H,W,Cpad) channels-last,
    zero beyond the Cv real channels.  w1 (Cf,Ch), w2 (Ch,Cv) packed (Cin, Cout)."""
    assert feat.is_cuda and feat.dtype == torch.float32 and feat.is_contiguous() and feat.dim() == 4
    b, cf, h, w = feat.shape
    ch, cv = w1.shape[1], w2.shape[1]
    assert w1.shape[0] == cf and w2.shape[0] == ch and w1.is_contiguous() and w2.is_contiguous()
    cp = cv if pad_to is None else int(pad_to)
    gate = torch.empty((b, h, w, cp), dtype=torch.float32, device=feat.device)
    _call("osb_feature_att_gate_fwd", feat.data_ptr(), w1.data_ptr(), _ptr(scale1), _ptr(shift1), w2.data_ptr(), _ptr(scale2),
          _ptr(shift2), gate.data_ptr(), b, cf, ch, cv, cp, h * w, act1, _stream(gate))
    return gate


def conv1x1_ndhwc_cat(x0, x1, w_packed, scale=None, shift=None, act=ACT_NONE):
    """Channels-last 1x1x1 conv over torch.cat((x0, x1), -1) without materialising it: (..., C0), (..., C1) -> (..., Cout);
    w_packed (C0 + C1, Cout)."""
    assert x0.is_cuda and x0.dtype == torch.float32 and x0.is_contiguous() and x1.is_contiguous() and x0.shape[:-1] == x1.shape[:-1]
    c0, c1 = x0.shape[-1], x1.shape[-1]
    cin, cout = w_packed.shape
    assert cin == c0 + c1 and w_packed.is_contiguous()
    y = torch.empty(x0.shape[:-1] + (cout,), dtype=torch.float32, device=x0.device)
    _call("osb_conv1x1_ndhwc_cat_fwd", x0.data_ptr(), x1.data_ptr(), c0, c1, w_packed.data_ptr(), _ptr(scale), _ptr(shift),
          y.data_ptr(), x0.numel() // c0, cout, act, _stream(y))
    return y


def deconv3d_k3_tc(x_ndhwc, w_split, scale=None, shift=None, residual=None, act=ACT_NONE, out_ndhwc=False, res_ndhwc=False):
    """ConvTranspose3d(k3, s2, p1, op1) + folded BN + residual + activation on the tensor cores.  x_ndhwc: (B,D,H,W,Cin)."""
    assert x_ndhwc.is_cuda and x_ndhwc.dtype == torch.float32 and x_ndhwc.is_contiguous() and x_ndhwc.dim() == 5
    b, d, h, w, cin = x_ndhwc.shape
    cout = w_split.cout
    wptr, scale = _tc_args(w_split, cin, 16, scale)
    shape = (b, 2 * d, 2 * h, 2 * w, cout) if out_ndhwc else (b, cout, 2 * d, 2 * h, 2 * w)
    y = torch.empty(shape, dtype=torch.float32, device=x_ndhwc.device)
    if residual is not None:
        want = (b, 2 * d, 2 * h, 2 * w, cout) if res_ndhwc else (b, cout, 2 * d, 2 * h, 2 * w)
        assert tuple(residual.shape) == want and residual.is_contiguous()
    _call("osb_deconv3d_k3_tc_fwd", x_ndhwc.data_ptr(), wptr, _ptr(scale), _ptr(shift), _ptr(residual),
          y.data_ptr(), b, cin, cout, d, h, w, act, 1 if out_ndhwc else 0, 1 if res_ndhwc else 0, _stream(y))
    return y


def conv1x1_ndhwc(x_ndhwc, w_packed, scale=None, shift=None, act=ACT_NONE):
    """Channels-last 1x1x1 conv: x (..., Cin) -> (..., Cout); w_packed (Cin, Cout)."""
    assert x_ndhwc.is_cuda and x_ndhwc.dtype == torch.float32 and x_ndhwc.is_contiguous()
    cin, cout = w_packed.shape
    assert x_ndhwc.shape[-1] == cin
    y = torch.empty(x_ndhwc.shape[:-1] + (cout,), dtype=torch.float32, device=x_ndhwc.device)
    _call("osb_conv1x1_ndhwc_fwd", x_ndhwc.data_ptr(), w_packed.data_ptr(), _ptr(scale), _ptr(shift), y.data_ptr(),
          x_ndhwc.numel() // cin, cin, cout, act, _stream(y))
    return y


def pack_c1_weight(weight):
    """(1, Cin, 3, 3, 3) Conv3d parameter -> (27, Cin) tap-major fp32 for conv3d_k3_c1_ndhwc."""
    assert weight.dim() == 5 and weight.shape[0] == 1 and tuple(weight.shape[2:]) == (3, 3, 3)
    return weight.detach().float()[0].permute(1, 2, 3, 0).reshape(27, -1).contiguous()


def conv3d_k3_c1_ndhwc(x_ndhwc, w_taps, scale=None, shift=None):
    """Single-output-channel 3x3x3 conv (classifier head) on a channels-last volume: (B,D,H,W,Cin) -> (B,1,D,H,W)."""
    assert x_ndhwc.is_cuda and x_ndhwc.dtype == torch.float32 and x_ndhwc.is_contiguous() and x_ndhwc.dim() == 5
    b, d, h, w, cin = x_ndhwc.shape
    assert w_taps.shape == (27, cin) and w_taps.is_contiguous()
    y = torch.empty((b, 1, d, h, w), dtype=torch.float32, device=x_ndhwc.device)
    _call("osb_conv3d_k3_c1_ndhwc_fwd", x_ndhwc.data_ptr(), w_taps.data_ptr(), _ptr(scale), _ptr(shift), y.data_ptr(), b, cin, d, h, w,
          _stream(y))
    return y


# ------------------------------------------------------------------ SURVEY.md section 8(f) row 2: LightStereo 2D aggregation
def dwconv2d(x, weight, scale=None, shift=None, residual=None, stride=1, act=ACT_NONE, out=None):
    """Depthwise Conv2d (groups = C, padding = k // 2) + per-channel scale/shift + residual + activation
    (lightstereo/aggregation.py:80-84 dwconv, :109-117 strip convs).  x (B,C,H,W); weight (C,1,KH,KW) or (C,KH,KW)."""
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 4
    b, c, h, w = x.shape
    kh, kw = weight.shape[-2:]
    wt = weight.detach().float().reshape(c, kh, kw).contiguous()
    ho, wo = (h - 1) // stride + 1, (w - 1) // stride + 1
    y = torch.empty((b, c, ho, wo), dtype=torch.float32, device=x.device) if out is None else out
    if residual is not None:
        assert residual.shape == y.shape and residual.is_contiguous()
    _call("osb_dwconv2d_fwd", x.data_ptr(), wt.data_ptr(), _ptr(scale), _ptr(shift), _ptr(residual), y.data_ptr(), b, c, h, w,
          int(kh), int(kw), int(stride), act, _stream(y))
    return y


def pack_deconv2d_weight(weight):
    """(Cin, Cout, 3, 3) ConvTranspose2d parameter -> (Cin, 9, Cout) contiguous fp32."""
    ci, co = weight.shape[:2]
    assert tuple(weight.shape[2:]) == (3, 3)
    return weight.detach().float().permute(0, 2, 3, 1).reshape(ci, 9, co).contiguous()


def deconv2d_k3s2(x, w_packed, scale=None, shift=None, residual=None, act=ACT_NONE):
    """ConvTranspose2d(k3, s2, p1, op1) + folded BN + residual + activation (lightstereo/aggregation.py:28-34,58-59)."""
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 4
    b, cin, h, w = x.shape
    assert w_packed.shape[0] == cin and w_packed.shape[1] == 9
    cout = w_packed.shape[2]
    y = torch.empty((b, cout, 2 * h, 2 * w), dtype=torch.float32, device=x.device)
    if residual is not None:
        assert residual.shape == y.shape and residual.is_contiguous()
    _call("osb_deconv2d_k3s2_fwd", x.data_ptr(), w_packed.data_ptr(), _ptr(scale), _ptr(shift), _ptr(residual), y.data_ptr(), b, cin,
          cout, h, w, act, _stream(y))
    return y


# ------------------------------------------------------------------ SURVEY.md section 8(f): GRU-iteration lookups
def avgpool_pairs(x, axis):
    """Average adjacent pairs along `axis` (a trailing odd element is dropped) == F.avg_pool2d(.., [1, 2], stride=[1, 2])
    applied along that axis (igev/geometry.py:24-30)."""
    assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
    axis = axis % x.dim()
    n = x.shape[axis]
    outer, inner = math.prod(x.shape[:axis]), math.prod(x.shape[axis + 1:])
    y = torch.empty(x.shape[:axis] + (n // 2,) + x.shape[axis + 1:], dtype=torch.float32, device=x.device)
    _call("osb_avgpool_pairs_fwd", x.data_ptr(), y.data_ptr(), outer, n, inner, _stream(y))
    return y


def geo_lookup(geo_levels, corr_levels, disp, coords, radius):
    """One lookup of the combined geometry-encoding volume (igev/geometry.py:32-57): geo_levels[i] (B,C,D>>i,H,W),
    corr_levels[i] (B,H,W,W2>>i), disp (B,1,H,W), coords (B,H,W[,1]) -> (B, L*(C+1)*(2r+1), H, W)."""
    levels = len(geo_levels)
    assert levels == len(corr_levels) and 1 <= levels <= 4
    b, c, d, h, w = geo_levels[0].shape
    w2 = corr_levels[0].shape[-1]
    for i in range(levels):
        g, cr = geo_levels[i], corr_levels[i]
        assert g.is_cuda and g.dtype == torch.float32 and g.is_contiguous() and tuple(g.shape) == (b, c, d >> i, h, w)
        assert cr.is_cuda and cr.dtype == torch.float32 and cr.is_contiguous() and tuple(cr.shape) == (b, h, w, w2 >> i)
    disp = disp.contiguous().float()
    coords = coords.reshape(b, h, w).contiguous().float()
    assert tuple(disp.shape) == (b, 1, h, w)
    out = torch.empty((b, levels * (c + 1) * (2 * radius + 1), h, w), dtype=torch.float32, device=disp.device)
    gp = [geo_levels[i].data_ptr() if i < levels else None for i in range(4)]
    cp = [corr_levels[i].data_ptr() if i < levels else None for i in range(4)]
    _call("osb_geo_lookup_fwd", *gp, *cp, disp.data_ptr(), coords.data_ptr(), out.data_ptr(), b, c, d, h, w, w2, levels, radius,
          _stream(out))
    return out


def geo_volume_lookup(geo_levels, disp, radius):
    """One lookup of IGEV-RT's geometry-only encoding volume (igev_rt/geometry.py:18-33): geo_levels[i] (B,C,D>>i,H,W),
    disp (B,1,H,W) -> (B, L*C*(2r+1), H, W), level-major, then channel, then tap."""
    levels = len(geo_levels)
    assert 1 <= levels <= 4
    b, c, d, h, w = geo_levels[0].shape
    for i in range(levels):
        g = geo_levels[i]
        assert g.is_cuda and g.dtype == torch.float32 and g.is_contiguous() and tuple(g.shape) == (b, c, d >> i, h, w)
    disp = disp.contiguous().float()
    assert tuple(disp.shape) == (b, 1, h, w)
    _same_device(geo_levels[0], disp)
    out = torch.empty((b, levels * c * (2 * radius + 1), h, w), dtype=torch.float32, device=disp.device)
    gp = [geo_levels[i].data_ptr() if i < levels else None for i in range(4)]
    _call("osb_geo_volume_lookup_fwd", *gp, disp.data_ptr(), out.data_ptr(), b, c, d, h, w, levels, radius, _stream(out))
    return out


def geo_multirange_lookup(geo_levels, vol1, vol2, corr_levels, disp, coords, radius):
    """One lookup of IGEV++'s multi-range encoding volume (igevpp/geometry.py:35-77), one launch: geo_levels[i] (B,C,D0>>i,H,W),
    vol1 (B,C,D1,H,W), vol2 (B,C,D2,H,W), corr_levels[i] (B,H,W,W2>>i), disp (B,1,H,W), coords (B,H,W[,1]) ->
    (geo_feat0 (B, L*C*T, H, W), geo_feat1 (B, C*T, H, W) at disp/2, geo_feat2 (B, C*T, H, W) at disp/4, init_corr (B, L*T, H, W)),
    T = 2r+1, fp32 whatever the input dtype."""
    levels = len(geo_levels)
    if not (1 <= levels <= 4 and levels == len(corr_levels)):
        raise ValueError("geo_multirange_lookup: 1..4 pyramid levels of both the volume and the correlation expected")
    geo = [_prep(g, "geo_multirange_lookup")[0] for g in geo_levels]
    corr = [_prep(cr, "geo_multirange_lookup")[0] for cr in corr_levels]
    (v1, _), (v2, _) = _prep(vol1, "geo_multirange_lookup"), _prep(vol2, "geo_multirange_lookup")
    disp, _ = _prep(disp, "geo_multirange_lookup")
    b, c, d0, h, w = geo[0].shape
    coords, _ = _prep(coords.reshape(b, h, w), "geo_multirange_lookup")
    w2 = corr[0].shape[-1]
    for i in range(levels):
        if tuple(geo[i].shape) != (b, c, d0 >> i, h, w) or tuple(corr[i].shape) != (b, h, w, w2 >> i):
            raise ValueError("geo_multirange_lookup: pyramid level %d has shape %s / %s" % (i, tuple(geo[i].shape), tuple(corr[i].shape)))
    if v1.shape[:2] != (b, c) or v1.shape[3:] != (h, w) or v2.shape[:2] != (b, c) or v2.shape[3:] != (h, w):
        raise ValueError("geo_multirange_lookup: range volumes %s / %s do not match %s" % (tuple(v1.shape), tuple(v2.shape), (b, c, h, w)))
    if tuple(disp.shape) != (b, 1, h, w):
        raise ValueError("geo_multirange_lookup: disp has shape %s, expected %s" % (tuple(disp.shape), (b, 1, h, w)))
    _same_device(*geo, *corr, v1, v2, disp, coords)
    t = 2 * radius + 1
    out0 = torch.empty((b, levels * c * t, h, w), dtype=torch.float32, device=disp.device)
    out1 = torch.empty((b, c * t, h, w), dtype=torch.float32, device=disp.device)
    out2 = torch.empty((b, c * t, h, w), dtype=torch.float32, device=disp.device)
    out_corr = torch.empty((b, levels * t, h, w), dtype=torch.float32, device=disp.device)
    gp = [geo[i].data_ptr() if i < levels else None for i in range(4)]
    cp = [corr[i].data_ptr() if i < levels else None for i in range(4)]
    _call("osb_geo_multirange_lookup_fwd", *gp, v1.data_ptr(), v2.data_ptr(), *cp, disp.data_ptr(), coords.data_ptr(),
          out0.data_ptr(), out1.data_ptr(), out2.data_ptr(), out_corr.data_ptr(), b, c, d0, v1.shape[2], v2.shape[2], h, w, w2, levels,
          radius, _stream(out0))
    return out0, out1, out2, out_corr


def context_upsample(disp_low, up_weights, scale_factor=4):
    """stereobase/igev_blocks.py:51-63: disp_low (B,1,h,w), up_weights (B,9,s*h,s*w) -> (B, s*h, s*w)."""
    assert disp_low.is_cuda and disp_low.dim() == 4 and disp_low.shape[1] == 1
    b, _, h, w = disp_low.shape
    assert tuple(up_weights.shape) == (b, 9, h * scale_factor, w * scale_factor)
    disp_low, up_weights = disp_low.contiguous().float(), up_weights.contiguous().float()
    out = torch.empty((b, h * scale_factor, w * scale_factor), dtype=torch.float32, device=disp_low.device)
    _call("osb_context_upsample_fwd", disp_low.data_ptr(), up_weights.data_ptr(), out.data_ptr(), b, h, w, scale_factor, _stream(out))
    return out


def conv2d_tc_kc(cin, cout, w, dilation=1):
    """K chunk of the tensor-core kernel serving a 3x3 Conv2d of this shape (0 = none)."""
    return int(_lib.lib.osb_conv2d_tc_kc(int(cin), int(cout), int(w), int(dilation)))


def pack_tc_weight_2d(weight, kc):
    """(Cout, Cin, 3, 3) Conv2d weight -> TcWeight of the one-plane 3x3x3 weight that holds its taps at kd = 1 (conv2d_k3_tc)."""
    w2 = weight.detach().float()
    w5 = w2.new_zeros(w2.shape[0], w2.shape[1], 3, 3, 3)
    w5[:, :, 1] = w2
    return pack_tc_weight(w5, kc)


def conv2d_k3_tc(x_nhwc, w_split, scale=None, shift=None, residual=None, act=ACT_NONE, dilation=1, out_nhwc=True, res_nhwc=True):
    """3x3 Conv2d (stride 1, padding = dilation) + folded BN + residual + activation on the tensor cores.  x_nhwc (B,H,W,Cin);
    w_split = pack_tc_weight of the 3x3x3 weight that holds the 2D taps at kd = 1."""
    assert x_nhwc.is_cuda and x_nhwc.dtype == torch.float32 and x_nhwc.is_contiguous() and x_nhwc.dim() == 4
    b, h, w, cin = x_nhwc.shape
    cout = w_split.cout
    kc = conv2d_tc_kc(cin, cout, w, dilation)
    assert kc
    wptr, scale = _tc_args(w_split, cin, kc, scale)
    y = torch.empty((b, h, w, cout) if out_nhwc else (b, cout, h, w), dtype=torch.float32, device=x_nhwc.device)
    if residual is not None:
        assert residual.is_contiguous() and residual.numel() == y.numel()
    _call("osb_conv2d_k3_tc_fwd", x_nhwc.data_ptr(), wptr, _ptr(scale), _ptr(shift), _ptr(residual), y.data_ptr(), b, cin,
          cout, h, w, dilation, act, int(out_nhwc), int(res_nhwc), _stream(y))
    return y


# --------------------------------------------------------------------------- ConvGRU update (gru.py)
ACT_SIGMOID, ACT_TANH = 4, 5     # include/openstereo_b200.h: OSB_ACT_SIGMOID / OSB_ACT_TANH, osb_conv2d_k3_tc_gru_fwd only


def nchw_to_nhwc_cat(tensors):
    """[(B,C_i,H,W) fp32 contiguous] -> (B,H,W,sum C_i) fp32: the channel concatenation, written channels-last one slice per tensor
    (osb_ncdhw_to_ndhwc_slice) without materialising the NCHW torch.cat."""
    b, _, h, w = tensors[0].shape
    total = sum(t.shape[1] for t in tensors)
    y = torch.empty((b, h, w, total), dtype=torch.float32, device=tensors[0].device)
    coff = 0
    for t in tensors:
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.dim() == 4 and (t.shape[0], *t.shape[2:]) == (b, h, w)
        _call("osb_ncdhw_to_ndhwc_slice", t.data_ptr(), y.data_ptr(), b, t.shape[1], 1, h, w, total, coff, _stream(y))
        coff += t.shape[1]
    return y


def conv2d_k3_tc_gru(x_nhwc, w_split, shift=None, residual=None, act=ACT_NONE, mul=None, blend=None, out_nhwc=True, res_nhwc=True):
    """3x3 Conv2d (stride 1, padding 1) with the ConvGRU epilogue on the tensor cores (osb_conv2d_k3_tc_gru_fwd), Cout = 128:
        v = act(conv(x) + shift + residual);  v = v * mul;  y = h + z * (v - h) with (z, h) = blend.
    x_nhwc (B,H,W,Cin); mul and the blend operands (B,H,W,128) channels-last; an NCHW residual (res_nhwc=False) may be a channel
    split() view of a wider (B, C', H, W) tensor (its batch stride goes to the kernel, no copy)."""
    assert x_nhwc.is_cuda and x_nhwc.dtype == torch.float32 and x_nhwc.is_contiguous() and x_nhwc.dim() == 4
    b, h, w, cin = x_nhwc.shape
    cout = w_split.cout
    wptr, scale = _tc_args(w_split, cin, 16, None)
    y = torch.empty((b, h, w, cout) if out_nhwc else (b, cout, h, w), dtype=torch.float32, device=x_nhwc.device)
    rbs = 0
    if residual is not None:
        assert residual.is_cuda and residual.dtype == torch.float32
        if res_nhwc:
            assert tuple(residual.shape) == (b, h, w, cout) and residual.is_contiguous()
        else:
            assert tuple(residual.shape) == (b, cout, h, w) and tuple(residual.stride()[1:]) == (h * w, w, 1)
            rbs = 0 if residual.is_contiguous() else residual.stride(0)
    z, hh = blend if blend is not None else (None, None)
    for t in (mul, z, hh):
        assert t is None or (tuple(t.shape) == (b, h, w, cout) and t.is_contiguous() and t.dtype == torch.float32 and t.is_cuda)
    _call("osb_conv2d_k3_tc_gru_fwd", x_nhwc.data_ptr(), wptr, _ptr(scale), _ptr(shift), _ptr(residual), _ptr(mul), _ptr(z), _ptr(hh),
          y.data_ptr(), b, cin, cout, h, w, act, int(out_nhwc), int(res_nhwc), rbs, _stream(y))
    return y
