#!/usr/bin/env python
"""Hot-path timings at the OTHER BASELINE.json configurations (bench.py is the contract line for configs[1], GwcNet):

    python tools/bench_configs.py [--only c1,c3,c4,c5] [--iters 10]

  c1  PSMNet cfgs/psmnet, 1 pair 256x512 D=192: whole-model forward of the host mirror (pairs/s) + EPE vs the CPU oracle
  c3  StereoBase cfgs/stereobase, 4 pairs/GPU (batch 32 over 8 GPUs) @256x512: the hot sub-graph on synthetic features --
      gwc (C=96, G=8) + concat (C=8) volume -> Hourglass(24, [96,64,192,160]) with FeatureAtt gates -> classifier -> softmax ->
      regression (stereobase_gru.py:139-164)
  c4  LightStereo-S cfgs/lightstereo, batch 16 @320x736: correlation_volume (C=24... the 1/4 features) -> Aggregation(48, [1,2,4],
      expanse 4, left attention) -> softmax/regression -> context_upsample (lightstereo.py:51-62)
  c5  IGEV cfgs/igev, batch 8 @480x640: gwc volume (C=96, G=8, D'=48) + 16 GRU-iteration lookups of the combined geometry
      encoding volume (igev_stereo.py:158,181-193; geometry.py:32-57) + 16 context up-samplings
  c6  CasPSMNet cfgs/casnet (the reference's class + patch()), batch 10 @512x960: whole-model forward next to the unpatched model
      on the same GPU, per-stage volume / aggregation / tail times  (python tools/bench_configs.py --only c6)
  c7  CoEx cfgs/coex (the reference's class + patch()), batch 8 @256x512 and @540x960: whole-model forward next to the unpatched
      model on the same GPU, per-stage volume / aggregation / regression times, the fused tail against the reference's tail
      (python tools/bench_configs.py --only c7)
  c8  MSNet3D cfgs/msnet/msnet3d_sceneflow.yaml (the reference's class + patch()), batch 8 @256x512 and @512x960: whole-model
      forward next to the unpatched model on the same GPU (timed alternately), per-stage volume / aggregation / tail times, and
      per MobileV2_Residual_3D config the fused block's time, TFLOP/s and GB/s  (python tools/bench_configs.py --only c8)
  c9  IGEV-RT cfgs/igev_rt (the reference's class + patch()), batch 8 @256x512 and @544x960: the uniform YAML's model patched and
      unpatched, timed alternately, the unpatched AMP YAML's model for context, per-stage times (volume, cost_agg, classifier, the 8
      lookups, everything else) and the lookups' GB/s  (python tools/bench_configs.py --only c9)
  c10 the ConvGRUs of IGEVStereo (cfgs/igev AMP YAML @480x640) and StereoBase (cfgs/stereobase @256x512), batch 8 (the reference's
      classes + patch()): ms in the three ConvGRUs and per forward, patched / cuDNN fp32 / fp16 autocast in alternating rotation,
      the GRU stage's TFLOP/s and the EPE against the unpatched model  (python tools/bench_configs.py --only c10)
  c11 the rest of the same update blocks (motion encoder, disp head, mask_feat_4), same models, shapes and rotation as c10: ms per
      forward in each of the six update-block modules, the three new stages' TFLOP/s and the EPE against the unpatched model
      (python tools/bench_configs.py --only c11)
  c12 IGEV++ (reference class + patch()), B=8 @256x512, 32 iterations: patched / cuDNN fp32 / AMP YAML / patched AMP YAML in
      alternating rotation, ms per forward in the lookups, ConvGRUs, geo + disp encoders, heads and the rest, and the EPE against
      the unpatched fp32 model  (python tools/bench_configs.py --only c12)
  c13 MonSter (reference class + patch(), ViT-L Depth Anything encoder), B=8 @256x512, 32 iterations: patched uniform YAML / cuDNN
      fp32 / the AMP YAML's bf16 autocast / patched AMP YAML in alternating rotation, ms per forward in the lookups, ConvGRUs,
      motion encoders, heads, warps and the rest, and the EPE against the unpatched fp32 model
      (python tools/bench_configs.py --only c13 > results/h100_c13_monster.jsonl)
Each line: this library (CUDA events, L2 flushed between iterations by the working set itself: every config streams > 126 MB per
step) next to the SAME graph of the oracle modules (bit-equal restatements of the reference: identical aten calls) on this GPU with
cuDNN fp32 (TF32 off) -- SURVEY.md section 8d's GPU comparator -- and the max abs / EPE difference between the two.
Test / measurement infrastructure: imports oracle/ as the checker and comparator."""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import __graft_entry__                                  # noqa: E402
__graft_entry__.build()
from openstereo_b200 import aggregation as agg          # noqa: E402
from openstereo_b200 import geo, host_models, ops       # noqa: E402
from oracle import aggregation as oagg                  # noqa: E402
from oracle import cascade as ocas                      # noqa: E402
from oracle import cost_volume as ocv                   # noqa: E402
from oracle import geo_lookup as ogeo                   # noqa: E402
from oracle import lightstereo as olight                # noqa: E402
from oracle import models as omodels                    # noqa: E402
from oracle import regression as oreg                   # noqa: E402
from oracle import seeded_init as si                    # noqa: E402

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
# under torchrun (python -m torch.distributed.run --nproc-per-node N tools/bench_configs.py --only c3): one process per GPU, every
# rank times the same per-GPU workload (weak scaling: BASELINE config 3 is batch 32 over 8 GPUs = 4 pairs per GPU), the step time is
# the max over ranks, rank 0 prints the aggregate
WORLD = int(os.environ.get("WORLD_SIZE", "1"))
RANK = int(os.environ.get("RANK", "0"))
DEV = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
torch.cuda.set_device(DEV)
if WORLD > 1:
    import torch.distributed as dist
    dist.init_process_group("nccl", device_id=DEV)


def over_ranks(ms):
    """max over ranks of a per-rank time (ms)"""
    if WORLD == 1:
        return ms
    t = torch.tensor([ms], device=DEV, dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def timeit(fn, iters, warm=3):
    for _ in range(warm):
        out = fn()
    torch.cuda.synchronize()
    if WORLD > 1:
        dist.barrier()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters, out


NO_REF = bool(os.environ.get("OSB_NO_REF"))         # launch lists under ncu: skip the cuDNN comparator


def rnd(gen, *shape, scale=1.0):
    return (torch.randn(*shape, generator=gen) * scale).to(DEV)


def emit(**kw):
    if RANK == 0:
        print(json.dumps(kw), flush=True)


def c1(iters):
    oracle = omodels.PSMNet(192).eval()
    sd = si.seeded_state_dict(oracle.state_dict(), seed=1, scale=si.PSMNET_SCALE, keep=si.PSMNET_KEEP)
    oracle.load_state_dict(sd)
    mine = host_models.PSMNet({"MAX_DISP": 192}).eval()
    mine.load_state_dict(sd)
    mine.to(DEV)
    g = torch.Generator().manual_seed(7)
    x = {"left": torch.randn(1, 3, 256, 512, generator=g), "right": torch.randn(1, 3, 256, 512, generator=g)}
    xg = {k: v.to(DEV) for k, v in x.items()}
    with torch.no_grad():
        want = oracle(dict(x))["disp_pred"]
        ms, got = timeit(lambda: mine(dict(xg))["disp_pred"], iters)
        oracle.to(DEV)
        ms_ref, ref_gpu = timeit(lambda: oracle(dict(xg))["disp_pred"], max(2, iters // 3), warm=1)
    emit(config="c1 PSMNet 1 pair 256x512 D=192", ms_per_step=round(ms, 3), pairs_per_s=round(1e3 / ms, 2),
         reference_cudnn_fp32_ms=round(ms_ref, 2), speedup_vs_reference_gpu=round(ms_ref / ms, 2),
         epe_vs_cpu_oracle_px=float("%.3e" % (got.cpu() - want).abs().mean().item()), overflow_count=ops.tc_overflow_count())


def c3(iters, B=4):
    gen = torch.Generator().manual_seed(7)
    ml, mr, cl, cr = rnd(gen, B, 96, 64, 128), rnd(gen, B, 96, 64, 128), rnd(gen, B, 8, 64, 128), rnd(gen, B, 8, 64, 128)
    feats = [rnd(gen, B, 96, 64, 128), rnd(gen, B, 64, 32, 64), rnd(gen, B, 192, 16, 32), rnd(gen, B, 160, 8, 16)]
    m = oagg.StereoBaseCostHead(24, [96, 64, 192, 160], max_disp=192).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=9, scale={"classifier.weight": 150.0}))
    m.to(DEV)
    hg, head = agg.StereoBaseAggregation(m.cost_agg), agg.StereoBaseCostHead(m.classifier)

    def ours():
        vol = ops.gwc_concat_volume(ml, mr, cl, cr, 48, 8)
        return head(hg(vol, feats), 48)

    def ref():
        vol = torch.cat((ocv.build_gwc_volume(ml, mr, 48, 8), ocv.build_concat_volume(cl, cr, 48)), 1)
        return m(vol, feats)[1]

    with torch.no_grad():
        ms, got = timeit(ours, iters, warm=1 if NO_REF else 3)
        ms = over_ranks(ms)
        ms_ref, want = (float("nan"), got) if NO_REF else timeit(ref, max(2, iters // 3), warm=1)
    emit(config="c3 StereoBase hot sub-graph, B=%d/GPU @256x512 (volume -> Hourglass(24)+FeatureAtt -> classifier -> soft-argmin)" % B,
         n_gpus=WORLD, ms_per_step=round(ms, 3), pairs_per_s=round(WORLD * B * 1e3 / ms, 2), reference_cudnn_fp32_ms=round(ms_ref, 2),
         speedup_vs_reference_gpu=round(ms_ref / ms, 2), init_disp_epe_vs_reference_gpu_px=float("%.3e" % (got - want).abs().mean().item()),
         gmac_per_pair=23.48)


def c4(iters, B=16):
    gen = torch.Generator().manual_seed(11)
    h, w = 80, 184
    fl, fr = rnd(gen, B, 24, h, w), rnd(gen, B, 24, h, w)
    feats = [fl, rnd(gen, B, 32, h // 2, w // 2), rnd(gen, B, 96, h // 4, w // 4)]
    spx = torch.softmax(rnd(gen, B, 9, 4 * h, 4 * w), 1)
    m = olight.Aggregation(in_channels=48, left_att=True, blocks=[1, 2, 4], expanse_ratio=4, backbone_channels=[24, 32, 96]).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=6))
    m.to(DEV)
    eng = agg.LightStereoAggregation(m)

    def ours():
        vol = ops.correlation_volume(fl, fr, 48)
        enc = eng(vol, feats)[0]
        init = ops.softargmin(enc, 48, keepdim=True)
        return ops.context_upsample(init * 4.0, spx, 4)

    def ref():
        vol = ocv.correlation_volume(fl, fr, 48)
        enc = m(vol, feats)[0]
        init = oreg.disparity_regression(F.softmax(enc, 1), 48)
        return ogeo.context_upsample(init * 4.0, spx)

    with torch.no_grad():
        ms, got = timeit(ours, iters)
        ms_ref, want = timeit(ref, max(2, iters // 3), warm=1)
    emit(config="c4 LightStereo-S hot path, B=%d @320x736 (corr volume -> 2D aggregation -> soft-argmin -> context_upsample)" % B,
         ms_per_step=round(ms, 3), pairs_per_s=round(B * 1e3 / ms, 2), reference_cudnn_fp32_ms=round(ms_ref, 2),
         speedup_vs_reference_gpu=round(ms_ref / ms, 2), disp_epe_vs_reference_gpu_px=float("%.3e" % (got - want.reshape(got.shape)).abs().mean().item()),
         disparity_std_px=round(want.std().item(), 2))


def c5(iters, B=8, gru_iters=16):
    gen = torch.Generator().manual_seed(13)
    h, w, d = 120, 160, 48
    ml, mr = rnd(gen, B, 96, h, w), rnd(gen, B, 96, h, w)
    f1, f2 = rnd(gen, B, 96, h, w), rnd(gen, B, 96, h, w)
    cv = rnd(gen, B, 8, d, h, w)                                              # stands in for the hourglass(8) output
    disp = (torch.rand(B, 1, h, w, generator=gen) * (d - 1)).to(DEV)
    coords = torch.arange(w, device=DEV).float().reshape(1, 1, w, 1).repeat(B, h, 1, 1)
    spx = torch.softmax(rnd(gen, B, 9, 4 * h, 4 * w), 1)

    def ours():
        vol = ops.build_gwc_volume(ml, mr, d, 8)
        gv = geo.CombinedGeoEncodingVolume(f1, f2, cv, num_levels=2, radius=4)
        out = None
        for _ in range(gru_iters):
            feat = gv(disp, coords)
            out = ops.context_upsample(disp * 4.0, spx, 4)
        return vol, feat, out

    def ref():
        vol = ocv.build_gwc_volume(ml, mr, d, 8)
        gv = ogeo.GeoEncodingVolume(f1, f2, cv, num_levels=2, radius=4)
        out = None
        for _ in range(gru_iters):
            feat = gv(disp, coords)
            out = ogeo.context_upsample(disp * 4.0, spx)
        return vol, feat, out

    with torch.no_grad():
        ms, got = timeit(ours, iters)
        ms_ref, want = timeit(ref, max(2, iters // 3), warm=1)
    emit(config="c5 IGEV hot path, B=%d @480x640: gwc volume (C=96,G=8,D'=48) + %d x (geo-volume lookup + context_upsample)" % (B, gru_iters),
         ms_per_step=round(ms, 3), pairs_per_s=round(B * 1e3 / ms, 2), reference_cudnn_fp32_ms=round(ms_ref, 2),
         speedup_vs_reference_gpu=round(ms_ref / ms, 2),
         max_abs_diff={"volume": float("%.2e" % (got[0] - want[0]).abs().max().item()),
                       "lookup": float("%.2e" % (got[1] - want[1]).abs().max().item()),
                       "upsample": float("%.2e" % (got[2] - want[2].reshape(got[2].shape)).abs().max().item())})


def gw(iters):
    """GwcNet hot path (gwc+concat volume -> 3D aggregation -> fused tail) at widths the whole-row tensor-core kernels do not serve:
    the reference's own timing shape 1x3x544x960 (tools/measure.py:32, W' = 240) and a KITTI crop 384x1248 (W' = 312).  Three
    columns: column-tile tensor-core kernels, the fp32 CUDA-core kernels of the same engine (what round 1 ran at these widths) and the
    oracle modules on cuDNN fp32."""
    for (h, w) in ((544, 960), (384, 1248)):
        gen = torch.Generator().manual_seed(17)
        hq, wq = h // 4, w // 4
        ml, mr = rnd(gen, 1, 320, hq, wq), rnd(gen, 1, 320, hq, wq)
        cl, cr = rnd(gen, 1, 12, hq, wq), rnd(gen, 1, 12, hq, wq)
        m = oagg.GwcDispProcessor(maxdisp=192, downsample=4, num_groups=40, use_concat_volume=True, concat_channels=12).eval()
        m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=41, scale={"classif3.2.weight": 60.0}))
        m.to(DEV)
        eng = agg.GwcAggregation(m)

        def ours():
            return eng(ops.gwc_concat_volume(ml, mr, cl, cr, 48, 40), h, w)

        def ref():
            vol = torch.cat((ocv.build_gwc_volume(ml, mr, 48, 40), ocv.build_concat_volume(cl, cr, 48)), 1)
            return m(vol, h, w)

        with torch.no_grad():
            ms, got = timeit(ours, iters)
            agg.USE_TENSOR_CORES = False
            try:
                ms_cc, got_cc = timeit(lambda: agg.GwcAggregation(m)(ops.gwc_concat_volume(ml, mr, cl, cr, 48, 40), h, w), max(2, iters // 3), warm=1)
            finally:
                agg.USE_TENSOR_CORES = True
            ms_ref, want = timeit(ref, max(2, iters // 3), warm=1)
        emit(config="gw GwcNet hot path, 1 pair @%dx%d D=192 (W' = %d: column-tile tensor-core kernels)" % (h, w, wq),
             ms_per_step=round(ms, 3), pairs_per_s=round(1e3 / ms, 2), cuda_core_kernels_ms=round(ms_cc, 2),
             reference_cudnn_fp32_ms=round(ms_ref, 2), speedup_vs_cuda_core=round(ms_cc / ms, 2),
             speedup_vs_reference_gpu=round(ms_ref / ms, 2),
             epe_vs_reference_gpu_px=float("%.3e" % (got - want.reshape(got.shape)).abs().mean().item()),
             epe_vs_cuda_core_px=float("%.3e" % (got - got_cc).abs().mean().item()), disparity_std_px=round(want.std().item(), 2),
             overflow_count=ops.tc_overflow_count())


def c6(iters, B=10, h=512, w=960):
    """CasPSMNet (the reference's own class, cfgs/casnet/casnet_psm_sceneflow.yaml unchanged, seeded weights) at the cfg's eval
    crop and evaluator batch: patch() next to the unpatched model on this GPU (cuDNN fp32, TF32 off).  Per stage: the warped
    volume (GB/s on its algorithmic bytes), the aggregation (useful TFLOP/s on the 3D convolutions' MACs) and the fused tail."""
    from oracle import _reference_shim as shim
    from openstereo_b200.patch import patch
    cfg = shim.load_cfg("cfgs/casnet/casnet_psm_sceneflow.yaml").MODEL
    m = shim.load("stereo.modeling.models.casnet.cas_psm").PSMNet(cfg).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=1, scale=ocas.CASNET_SCALE))
    m.to(DEV)
    gen = torch.Generator().manual_seed(19)
    x = {"left": rnd(gen, B, 3, h, w), "right": rnd(gen, B, 3, h, w)}
    with torch.no_grad():
        ms_ref, want = timeit(lambda: m(dict(x))["disp_pred"], max(2, iters // 3), warm=1)
        patch(m)
        ms, got = timeit(lambda: m(dict(x))["disp_pred"], iters)
        # per-stage split: CUDA events around each stage's volume / aggregation call, the tail's own entry point inside it
        events = []

        def timed(mod, tag):
            inner = mod.forward

            def fwd(*args, **kw):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                out = inner(*args, **kw)
                b.record()
                events.append((tag, a, b))
                return out
            mod.forward = fwd
        timed(m.get_cv, "volume")
        for i, agg_mod in enumerate(m.cost_agg):
            timed(agg_mod, "agg%d" % i)
        ops.profile_start()
        m(dict(x))
        torch.cuda.synchronize()
        prof = ops.profile_stop()
    tails = [a.elapsed_time(b) for a, b in prof.get("osb_upsample_softargmin_values_fwd", [])]
    vols = [a.elapsed_time(b) for tag, a, b in events if tag == "volume"]
    aggs = [a.elapsed_time(b) for tag, a, b in events if tag.startswith("agg")]
    stages = []
    for i, (cin, hq, wq, gmac) in enumerate(((32, h // 4, w // 4, 109.0), (16, h // 2, w // 2, 395.0))):
        vol_bytes = 4 * (2 * B * cin * hq * wq + B * 12 * hq * wq + B * 2 * cin * 12 * hq * wq)
        agg_ms = aggs[i] - tails[i]
        stages.append({"stage": i + 1, "volume_shape": [B, 2 * cin, 12, hq, wq], "volume_ms": round(vols[i], 3),
                       "volume_GBps": round(vol_bytes / vols[i] / 1e6, 1), "volume_frac_of_3350GBps": round(vol_bytes / vols[i] / 1e6 / 3350, 3),
                       "aggregation_ms": round(agg_ms, 3), "aggregation_useful_tflops": round(2 * gmac * B / agg_ms, 1),
                       "tail_ms": round(tails[i], 3)})
    emit(config="c6 CasPSMNet cfgs/casnet/casnet_psm_sceneflow.yaml, B=%d @%dx%d (reference class + patch())" % (B, h, w),
         gpu="%s, %.0f W power limit" % (torch.cuda.get_device_name(DEV), _power_limit_w()),
         ms_per_step=round(ms, 3), pairs_per_s=round(B * 1e3 / ms, 2), reference_cudnn_fp32_ms=round(ms_ref, 2),
         reference_pairs_per_s=round(B * 1e3 / ms_ref, 2), speedup_vs_reference_gpu=round(ms_ref / ms, 2),
         epe_vs_reference_gpu_px=float("%.3e" % (got - want).abs().mean().item()), disparity_std_px=round(want.std().item(), 2),
         stages=stages, overflow_count=ops.tc_overflow_count())


def c7(iters, B=8):
    """CoEx (the reference's own class, cfgs/coex/coex_sceneflow_amp.yaml unchanged, seeded weights) at the cfg's eval size
    540x960 and at 256x512, evaluator batch 8: patch() next to the unpatched model on this GPU (cuDNN fp32, TF32 off).  Per stage:
    the attention volume, the 3D aggregation and the regression tail; the fused tail's GB/s on its algorithmic bytes and its time
    next to the reference's tail (softmax over the 9 superpixel planes + Regression.forward) on the same inputs."""
    from oracle import _reference_shim as shim
    from openstereo_b200.patch import patch
    shim.install_timm_stub()
    cfg = shim.load_cfg("cfgs/coex/coex_sceneflow_amp.yaml").MODEL
    cls = shim.load("stereo.modeling.models.coex.coex").CoEx
    for (h, w) in ((256, 512), (540, 960)):
        m = cls(cfg).eval()
        m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=1))
        m.to(DEV)
        gen = torch.Generator().manual_seed(23)
        x = {"left": rnd(gen, B, 3, h, w), "right": rnd(gen, B, 3, h, w)}
        cp, dp = m.CostProcessor, m.DispProcessor
        seen = {}

        def grab(mod, args):
            seen["cost"] = args[0]["cost_volume"]
        hook = dp.register_forward_pre_hook(grab)
        with torch.no_grad():
            ms_ref, want = timeit(lambda: m(dict(x))["disp_pred"], max(2, iters // 3), warm=1)
            ref_stages = _stage_times(lambda: m(dict(x)), {"volume": cp.cost_volume, "aggregation": cp.cost_agg,
                                                         "regression": dp.regression})
            # the reference's tail on the inputs it sees in this model: softmax over the 9 superpixel planes, then Regression
            inputs = dict(x)
            inputs.update(m.Backbone(inputs))
            xspx = dp.spx_2(dp.spx_4(inputs["ref_feature"][0]), inputs["stem_2x"])
            spx_logits = dp.spx(xspx)
            cost = seen["cost"]
            ms_ref_tail, _ = timeit(lambda: dp.regression(cost, F.softmax(spx_logits, 1)), iters)
            patch(m)
            ms, got = timeit(lambda: m(dict(x))["disp_pred"], iters)
            ms_tail, _ = timeit(lambda: ops.coex_regression(cost, spx_logits, dp.regression.top_k, spx_is_logits=True), iters)
            stages = _stage_times(lambda: m(dict(x)), {"aggregation": agg.CoExAggregation}, volume_fn="coex_attention_volume")
            ops.profile_start()
            m(dict(x))
            torch.cuda.synchronize()
            prof = ops.profile_stop()
        hook.remove()
        stages["regression"] = round(sum(a.elapsed_time(b) for a, b in prof["osb_coex_regression_fwd"]), 3)
        hq, wq = cost.shape[-2:]
        tail_bytes = 4 * (B * cost.shape[2] * hq * wq + 9 * B * 16 * hq * wq + B * 16 * hq * wq)
        emit(config="c7 CoEx cfgs/coex/coex_sceneflow_amp.yaml, B=%d @%dx%d (reference class + patch())" % (B, h, w),
             gpu="%s, %.0f W power limit" % (torch.cuda.get_device_name(DEV), _power_limit_w()),
             ms_per_step=round(ms, 3), pairs_per_s=round(B * 1e3 / ms, 2), reference_cudnn_fp32_ms=round(ms_ref, 2),
             reference_pairs_per_s=round(B * 1e3 / ms_ref, 2), speedup_vs_reference_gpu=round(ms_ref / ms, 2),
             stage_ms=stages, reference_stage_ms=ref_stages,
             regression_tail_ms=round(ms_tail, 4), reference_tail_ms=round(ms_ref_tail, 4),
             regression_tail_GBps=round(tail_bytes / ms_tail / 1e6, 1), regression_tail_frac_of_3350GBps=round(tail_bytes / ms_tail / 1e6 / 3350, 3),
             epe_vs_reference_gpu_px=float("%.3e" % (got - want).abs().mean().item()), disparity_std_px=round(want.std().item(), 2))


def _mbv2_rows(eng, prof, B, d, h, w):
    """Per (Cin, Chid, Cout, stride) config of the fused MobileV2_Residual_3D block: launches, kernel ms, fp32 TFLOP/s on the
    algorithmic MACs Vin*Cin*Chid + Vout*27*Chid + Vout*Chid*Cout, GB/s on the algorithmic bytes 4*(Vin*Cin + Vout*Cout [+ Vout*Cout
    residual]), and which bound (67 TFLOP/s fp32, 3.35 TB/s HBM) is the larger."""
    blocks = list(eng.dres0) + list(eng.dres1)
    for hg in eng.hg:
        blocks += [hg.conv1, hg.conv2, hg.conv3, hg.conv4, hg.redir2, hg.redir1]           # launch order
    events = prof["osb_mbv2_block3d_fwd"]
    assert len(events) == len(blocks) == 22
    rows = {}
    for blk, (a, b) in zip(blocks, events):
        dims_in = _mbv2_dims(eng, blk, d, h, w)
        vin = B * dims_in[0] * dims_in[1] * dims_in[2]
        vout = B * ((dims_in[0] - 1) // blk.stride + 1) * ((dims_in[1] - 1) // blk.stride + 1) * ((dims_in[2] - 1) // blk.stride + 1)
        res = blk is eng.dres1[-1]
        macs = vin * blk.cin * blk.hid + vout * 27 * blk.hid + vout * blk.hid * blk.cout
        byts = 4 * (vin * blk.cin + vout * blk.cout * (2 if res else 1))
        key = "%d-%d-%d-s%d" % (blk.cin, blk.hid, blk.cout, blk.stride)
        r = rows.setdefault(key, {"launches": 0, "ms": 0.0, "macs": 0, "bytes": 0})
        r["launches"] += 1
        r["ms"] += a.elapsed_time(b)
        r["macs"] += macs
        r["bytes"] += byts
    for key, r in rows.items():
        tflops = 2 * r["macs"] / r["ms"] / 1e9
        gbps = r["bytes"] / r["ms"] / 1e6
        r.update(ms=round(r["ms"], 3), TFLOPs=round(tflops, 2), GBps=round(gbps, 1),
                 bound="fp32 FMA" if 2 * r["macs"] / 67e12 > r["bytes"] / 3.35e12 else "HBM",
                 frac_of_bound=round(max(tflops / 67.0, gbps / 3350.0), 3))
        del r["macs"], r["bytes"]
    return rows


def _mbv2_dims(eng, blk, d, h, w):
    """Input extents of a block of MSNet3DAggregation for a (d, h, w) volume: full resolution except inside the hourglasses."""
    for hg in eng.hg:
        if blk in (hg.conv1, hg.redir1):
            return (d, h, w)
        if blk in (hg.conv2, hg.conv3, hg.redir2):
            return (-(-d // 2), -(-h // 2), -(-w // 2))
        if blk is hg.conv4:
            return (-(-d // 4), -(-h // 4), -(-w // 4))
    return (d, h, w)


def c8(iters, B=8):
    """MSNet3D (the reference's own class, cfgs/msnet/msnet3d_sceneflow.yaml unchanged, seeded and sharpened weights) at 256x512 and
    at the cfg's eval crop 512x960, batch 8: patch() against the unpatched model on this GPU (cuDNN fp32, TF32 off), timed
    alternately in the same process; per-stage times of the patched forward (volume, aggregation, tail) from CUDA events around
    each launch; per block config the fused kernel's time and rates (_mbv2_rows)."""
    from oracle import msnet as oms
    from openstereo_b200.patch import patch
    from oracle import _reference_shim as shim
    shim_cfg = shim.load_cfg("cfgs/msnet/msnet3d_sceneflow.yaml").MODEL
    cls = oms.load_reference("stereo.modeling.models.msnet.MSNet3D").MSNet3D
    for (h, w) in ((256, 512), (512, 960)):
        ref = cls(shim_cfg).eval()
        ref.load_state_dict(si.seeded_state_dict(ref.state_dict(), seed=1, scale=oms.MSNET3D_SCALE))
        ref.to(DEV)
        pm = cls(shim_cfg).eval()
        pm.load_state_dict(ref.state_dict())
        patch(pm.to(DEV))
        gen = torch.Generator().manual_seed(23)
        x = {"left": rnd(gen, B, 3, h, w), "right": rnd(gen, B, 3, h, w)}
        with torch.no_grad():
            ms_ref, ms = [], []
            for _ in range(3):                                          # alternate: the two share the GPU's state
                t, want = timeit(lambda: ref(dict(x))["disp_pred"], max(1, iters // 5), warm=1)
                ms_ref.append(t)
                t, got = timeit(lambda: pm(dict(x))["disp_pred"], iters, warm=2)
                ms.append(t)
            ms_ref, ms = sorted(ms_ref)[1], sorted(ms)[1]
            ops.profile_start()
            pm(dict(x))
            torch.cuda.synchronize()
            prof = ops.profile_stop()
        eng = agg.MSNet3DAggregation(pm)                                # the same blocks, in the patched forward's launch order
        eng._ensure(DEV)
        span = lambda name: round(sum(a.elapsed_time(b) for a, b in prof.get(name, [])), 3)         # noqa: E731
        total = round(sum(a.elapsed_time(b) for evs in prof.values() for a, b in evs), 3)
        stages = {"volume": span("osb_gwc_volume_fwd"), "tail": span("osb_upsample_softargmin_fwd")}
        stages["aggregation"] = round(total - stages["volume"] - stages["tail"], 3)
        stages["mbv2_blocks"] = span("osb_mbv2_block3d_fwd")
        d4, h4, w4 = shim_cfg.MAX_DISP // 4, h // 4, w // 4
        emit(config="c8 MSNet3D cfgs/msnet/msnet3d_sceneflow.yaml, B=%d @%dx%d (reference class + patch())" % (B, h, w),
             gpu="%s, %.0f W power limit" % (torch.cuda.get_device_name(DEV), _power_limit_w()),
             ms_per_step=round(ms, 3), pairs_per_s=round(B * 1e3 / ms, 2), reference_cudnn_fp32_ms=round(ms_ref, 2),
             reference_pairs_per_s=round(B * 1e3 / ms_ref, 2), speedup_vs_reference_gpu=round(ms_ref / ms, 2),
             stage_ms=stages, block_configs=_mbv2_rows(eng, prof, B, d4, h4, w4),
             epe_vs_reference_gpu_px=float("%.3e" % (got - want).abs().mean().item()), disparity_std_px=round(want.std().item(), 2))
        del ref, pm, eng, prof
        torch.cuda.empty_cache()


def c9(iters, B=8):
    """IGEV-RT (the reference's own class, cfgs/igev_rt YAMLs unchanged, seeded weights with the classifier sharpened) at 256x512 and
    at SceneFlow's 540x960 after DivisiblePad 32 (544x960), batch 8.  The uniform (fp32) YAML's model with and without patch() is
    timed alternately in one process, with the unpatched AMP YAML's model (fp16 autocast) in the same rotation for context.  Stage
    times of the patched forward come from CUDA events around ops.build_gwc_volume, cost_agg, classifier and the lookups; the rest
    of the step (feature nets, hnet / cnet, the ConvGRU, regression, up-sampling) is "other".  Lookup GB/s counts the algorithmic
    bytes: the output written, 2r+2 samples per (pixel, channel, level) read once and the disparity read once per channel row."""
    from oracle import igev_rt as oigrt
    from openstereo_b200.patch import patch
    for (h, w) in ((256, 512), (544, 960)):
        ref = oigrt.igev_rt(oigrt.UNIFORM_YAML).to(DEV)
        amp = oigrt.igev_rt(oigrt.AMP_YAML).to(DEV)
        pm = patch(oigrt.igev_rt(oigrt.UNIFORM_YAML).to(DEV))
        cfg = pm.args
        gen = torch.Generator().manual_seed(29)
        x = {"left": rnd(gen, B, 3, h, w), "right": rnd(gen, B, 3, h, w)}
        with torch.no_grad():
            ms_ref, ms_amp, ms = [], [], []
            for _ in range(3):                                          # alternate: the three share the GPU's state
                t, want = timeit(lambda: ref(dict(x))["disp_pred"], max(1, iters // 2), warm=1)
                ms_ref.append(t)
                t, got_amp = timeit(lambda: amp(dict(x))["disp_pred"], max(1, iters // 2), warm=1)
                ms_amp.append(t)
                t, got = timeit(lambda: pm(dict(x))["disp_pred"], iters, warm=2)
                ms.append(t)
            ms_ref, ms_amp, ms = sorted(ms_ref)[1], sorted(ms_amp)[1], sorted(ms)[1]
            stages = _stage_times(lambda: pm(dict(x)), {"cost_agg": pm.cost_agg, "classifier": pm.classifier,
                                                        "lookups": geo.GeoEncodingVolume}, volume_fn="build_gwc_volume")
        stages["other"] = round(ms - sum(stages.values()), 3)
        c, d4, h4, w4 = 8, cfg.MAX_DISP // 4, h // 4, w // 4
        levels, r = cfg.CORR_LEVELS, cfg.CORR_RADIUS
        rows = B * levels * c * h4 * w4                                 # (pixel, channel, level) rows of one lookup
        lookup_bytes = 4 * (rows * (2 * r + 1) + rows * (2 * r + 2) + rows)
        n_lookups = cfg.VALID_ITERS
        emit(config="c9 IGEV-RT cfgs/igev_rt, B=%d @%dx%d (reference class + patch())" % (B, h, w),
             gpu="%s, %.0f W power limit" % (torch.cuda.get_device_name(DEV), _power_limit_w()),
             ms_per_step=round(ms, 3), pairs_per_s=round(B * 1e3 / ms, 2),
             reference_uniform_fp32_ms=round(ms_ref, 2), reference_uniform_pairs_per_s=round(B * 1e3 / ms_ref, 2),
             reference_amp_fp16_ms=round(ms_amp, 2), reference_amp_pairs_per_s=round(B * 1e3 / ms_amp, 2),
             speedup_vs_reference_uniform=round(ms_ref / ms, 3), speedup_vs_reference_amp=round(ms_amp / ms, 3),
             stage_ms=stages, lookups=n_lookups,
             lookup_gb_per_s=round(n_lookups * lookup_bytes / (stages["lookups"] * 1e-3) / 1e9, 1) if stages.get("lookups") else None,
             epe_vs_reference_uniform_px=float("%.3e" % (got - want).abs().mean().item()),
             epe_amp_reference_vs_uniform_px=float("%.3e" % (got_amp - want).abs().mean().item()),
             disparity_std_px=round(want.std().item(), 2))
        del ref, amp, pm
        torch.cuda.empty_cache()


def _gru_stage(run, block):
    """One run of `run` with CUDA events around every call of block.gru04 / gru08 / gru16: (ms in the three ConvGRUs, their MACs)."""
    events, macs = [], [0]
    mods = [getattr(block, n) for n in ("gru04", "gru08", "gru16")]
    saved = [vars(m).get("forward") for m in mods]

    def wrap(inner):
        def fwd(h, *rest):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            cin = h.shape[1] + sum(t.shape[1] for t in rest[3:])
            macs[0] += 3 * h.shape[0] * h.shape[2] * h.shape[3] * h.shape[1] * cin * 9
            a.record()
            out = inner(h, *rest)
            b.record()
            events.append((a, b))
            return out
        return fwd
    for m in mods:
        m.forward = wrap(m.forward)
    try:
        run()
        torch.cuda.synchronize()
    finally:
        for m, s in zip(mods, saved):
            if s is None:
                del m.forward
            else:
                m.forward = s
    return sum(a.elapsed_time(b) for a, b in events), macs[0]


def c10(iters, B=8):
    """The ConvGRUs of IGEV-Stereo (cfgs/igev AMP YAML, config 5's 480x640) and StereoBase (cfgs/stereobase, 256x512), batch 8, the
    reference's classes with the timm stand-in the tests use.  Three variants timed in alternating rotation: patch() (the GRUs on the
    wgmma kernels, fp32), unpatched cuDNN fp32 with TF32 off, and unpatched under fp16 autocast.  Per variant: whole-forward ms and
    the ms spent in the three ConvGRUs (CUDA events around every gru04 / gru08 / gru16 call); the GRU stage's useful fp32-equivalent
    TFLOP/s counts 2 x its MACs (three 3x3 convs of Cin = hidden + inputs per call); EPE of patched against unpatched fp32."""
    from oracle import _reference_shim as shim
    from openstereo_b200.patch import patch
    shim.install_timm_stub()

    def build(which):
        if which == "igev":
            cfg = shim.load_cfg("cfgs/igev/igev_sceneflow_amp.yaml").MODEL
            m = shim.load("stereo.modeling.models.igev.igev_stereo").IGEVStereo(cfg).eval()
            m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=12, scale={"classifier.weight": 8.0}))
        else:
            cfg = shim.load_cfg("cfgs/stereobase/stereobase_sceneflow.yaml").MODEL
            m = shim.load("stereo.modeling.models.stereobase.stereobase_gru").StereoBase(cfg).eval()
            m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=3, scale={"classifier.weight": 8.0}))
        return m.to(DEV)

    for which, name, (h, w) in (("igev", "IGEVStereo", (480, 640)), ("stereobase", "StereoBase", (256, 512))):
        ref, pm = build(which), patch(build(which))
        gen = torch.Generator().manual_seed(31)
        x = {"left": (torch.rand(B, 3, h, w, generator=gen) * 255).to(DEV), "right": (torch.rand(B, 3, h, w, generator=gen) * 255).to(DEV)}
        variants = {"patched": (pm, False), "cudnn_fp32": (ref, False), "amp_fp16": (ref, True)}

        def fwd(m, amp):
            with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
                return m(dict(x))["disp_pred"]
        ms = {k: [] for k in variants}
        gru_ms = {k: [] for k in variants}
        outs, macs = {}, 0
        with torch.no_grad():
            for _ in range(3):                                          # alternate: the three share the GPU's state
                for k, (m, amp) in variants.items():
                    t, outs[k] = timeit(lambda: fwd(m, amp), max(1, iters // 5), warm=1)
                    ms[k].append(t)
                    g, macs = _gru_stage(lambda: fwd(m, amp), m.update_block)
                    gru_ms[k].append(g)
        med = lambda v: sorted(v)[1]
        emit(config="c10 ConvGRUs of %s, B=%d @%dx%d (reference class + patch())" % (name, B, h, w),
             gpu="%s, %.0f W power limit" % (torch.cuda.get_device_name(DEV), _power_limit_w()),
             gru_ms={k: round(med(v), 2) for k, v in gru_ms.items()},
             forward_ms={k: round(med(v), 2) for k, v in ms.items()},
             gru_share_of_forward={k: round(med(gru_ms[k]) / med(ms[k]), 3) for k in variants},
             gru_gmac=round(macs / 1e9, 1),
             gru_tflops_fp32_equivalent={k: round(2 * macs / (med(v) * 1e-3) / 1e12, 1) for k, v in gru_ms.items()},
             gru_speedup_vs_cudnn_fp32=round(med(gru_ms["cudnn_fp32"]) / med(gru_ms["patched"]), 2),
             gru_speedup_vs_amp_fp16=round(med(gru_ms["amp_fp16"]) / med(gru_ms["patched"]), 2),
             epe_patched_vs_cudnn_fp32_px=float("%.3e" % (outs["patched"] - outs["cudnn_fp32"]).abs().mean().item()),
             epe_amp_vs_cudnn_fp32_px=float("%.3e" % (outs["amp_fp16"].float() - outs["cudnn_fp32"]).abs().mean().item()),
             disparity_std_px=round(outs["cudnn_fp32"].std().item(), 2))
        del ref, pm
        torch.cuda.empty_cache()


# MACs per 1/4-resolution pixel and call (igev/update.py:17-25,75-94,123-125): convc1 1x1 Cc -> 64, convc2 / convd2 3x3 64 -> 64,
# convd1 7x7 1 -> 64, conv 3x3 128 -> 127; DispHead 3x3 128 -> 256 -> 1; mask_feat_4 3x3 128 -> 32
_UPDATE_MACS = {"encoder": lambda cc: cc * 64 + 2 * 64 * 64 * 9 + 49 * 64 + 128 * 127 * 9,
                "disp_head": lambda cc: 128 * 256 * 9 + 256 * 9, "mask_feat_4": lambda cc: 128 * 32 * 9}


def _update_stages(run, block):
    """One run of `run` with CUDA events around every call of the six update-block modules: {module: ms}, {module: MACs}."""
    names = ("encoder", "disp_head", "mask_feat_4", "gru04", "gru08", "gru16")
    events, macs = [], {n: 0 for n in _UPDATE_MACS}
    mods = {n: getattr(block, n) for n in names}
    saved = {n: vars(m).get("forward") for n, m in mods.items()}

    def wrap(name, inner):
        def fwd(*args):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            if name in _UPDATE_MACS:
                x = args[-1]                                        # corr (encoder) or net0: (B, C, H, W)
                macs[name] += _UPDATE_MACS[name](x.shape[1]) * x.shape[0] * x.shape[2] * x.shape[3]
            a.record()
            out = inner(*args)
            b.record()
            events.append((name, a, b))
            return out
        return fwd
    for n, m in mods.items():
        m.forward = wrap(n, m.forward)
    try:
        run()
        torch.cuda.synchronize()
    finally:
        for n, m in mods.items():
            if saved[n] is None:
                del m.forward
            else:
                m.forward = saved[n]
    ms = {n: 0.0 for n in names}
    for n, a, b in events:
        ms[n] += a.elapsed_time(b)
    return ms, macs


def c11(iters, B=8):
    """The motion encoder, disp head and mask_feat_4 of IGEV-Stereo (cfgs/igev AMP YAML, 480x640) and StereoBase (cfgs/stereobase,
    256x512), batch 8, the reference's classes: the variants of c10 (patch(), unpatched cuDNN fp32 with TF32 off, unpatched fp16
    autocast) in alternating rotation, medians of three.  Per variant: whole-forward ms, ms in each update-block module (CUDA events
    around every call), the three new stages' useful TFLOP/s (2 x the MACs of _UPDATE_MACS), EPE of each variant against fp32."""
    from oracle import _reference_shim as shim
    from openstereo_b200.patch import patch
    shim.install_timm_stub()

    def build(which):
        if which == "igev":
            cfg = shim.load_cfg("cfgs/igev/igev_sceneflow_amp.yaml").MODEL
            m = shim.load("stereo.modeling.models.igev.igev_stereo").IGEVStereo(cfg).eval()
            m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=12, scale={"classifier.weight": 8.0}))
        else:
            cfg = shim.load_cfg("cfgs/stereobase/stereobase_sceneflow.yaml").MODEL
            m = shim.load("stereo.modeling.models.stereobase.stereobase_gru").StereoBase(cfg).eval()
            m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=3, scale={"classifier.weight": 8.0}))
        return m.to(DEV)

    new = tuple(_UPDATE_MACS)
    for which, name, (h, w) in (("igev", "IGEVStereo", (480, 640)), ("stereobase", "StereoBase", (256, 512))):
        ref, pm = build(which), patch(build(which))
        gen = torch.Generator().manual_seed(31)
        x = {"left": (torch.rand(B, 3, h, w, generator=gen) * 255).to(DEV), "right": (torch.rand(B, 3, h, w, generator=gen) * 255).to(DEV)}
        variants = {"patched": (pm, False), "cudnn_fp32": (ref, False), "amp_fp16": (ref, True)}

        def fwd(m, amp):
            with torch.autocast("cuda", dtype=torch.float16, enabled=amp):
                return m(dict(x))["disp_pred"]
        ms = {k: [] for k in variants}
        stage = {k: [] for k in variants}
        outs, macs = {}, {}
        with torch.no_grad():
            for _ in range(3):                                          # alternate: the three share the GPU's state
                for k, (m, amp) in variants.items():
                    t, outs[k] = timeit(lambda: fwd(m, amp), max(1, iters // 5), warm=1)
                    ms[k].append(t)
                    st, macs = _update_stages(lambda: fwd(m, amp), m.update_block)
                    stage[k].append(st)
        med = lambda v: sorted(v)[1]
        stage_ms = {k: {n: round(med([s[n] for s in v]), 2) for n in v[0]} for k, v in stage.items()}
        new_ms = {k: round(sum(v[n] for n in new), 2) for k, v in stage_ms.items()}
        emit(config="c11 motion encoder + disp head + mask_feat_4 of %s, B=%d @%dx%d (reference class + patch())" % (name, B, h, w),
             gpu="%s, %.0f W power limit" % (torch.cuda.get_device_name(DEV), _power_limit_w()),
             forward_ms={k: round(med(v), 2) for k, v in ms.items()},
             stage_ms=stage_ms,
             new_stages_ms=new_ms,
             new_stages_gmac={n: round(v / 1e9, 1) for n, v in macs.items()},
             new_stages_tflops_fp32_equivalent={k: {n: round(2 * macs[n] / (v[n] * 1e-3) / 1e12, 1) for n in new}
                                                for k, v in stage_ms.items()},
             new_stages_speedup_vs_cudnn_fp32=round(new_ms["cudnn_fp32"] / new_ms["patched"], 2),
             new_stages_speedup_vs_amp_fp16=round(new_ms["amp_fp16"] / new_ms["patched"], 2),
             epe_patched_vs_cudnn_fp32_px=float("%.3e" % (outs["patched"] - outs["cudnn_fp32"]).abs().mean().item()),
             epe_amp_vs_cudnn_fp32_px=float("%.3e" % (outs["amp_fp16"].float() - outs["cudnn_fp32"]).abs().mean().item()),
             disparity_std_px=round(outs["cudnn_fp32"].std().item(), 2))
        del ref, pm
        torch.cuda.empty_cache()


def c12(iters, B=8, h=256, w=512):
    """IGEV++ (igevpp/igevpp_stereo.py, the reference's class with the timm stand-in), batch 8 at 256x512 (W' = 128), 32 GRU
    iterations.  Variants in alternating rotation, medians of three: patch() of the uniform-YAML model (fp32), the unpatched
    uniform-YAML model (cuDNN fp32, TF32 off), the unpatched AMP-YAML model (the reference's own fp16 autocast) and patch() of the
    AMP-YAML model.  Per variant: whole-forward ms and ms per forward in the lookups (CUDA events around every lookup call), the
    three ConvGRUs, the three geo encoders + the disparity encoder, the disparity + mask heads, and everything else; EPE of each
    variant against the unpatched fp32 model."""
    from oracle import igevpp as oigpp
    from openstereo_b200 import geo
    from openstereo_b200.patch import patch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    ref_geo = oigpp.load_reference("stereo.modeling.models.igevpp.geometry").Combined_Geo_Encoding_Volume
    variants = {"patched": patch(oigpp.igevpp().to(DEV)), "cudnn_fp32": oigpp.igevpp().to(DEV),
                "amp_fp16": oigpp.igevpp(oigpp.AMP_YAML).to(DEV), "patched_amp_yaml": patch(oigpp.igevpp(oigpp.AMP_YAML).to(DEV))}
    gen = torch.Generator().manual_seed(31)
    x = {"left": (torch.rand(B, 3, h, w, generator=gen) * 2 - 1).to(DEV), "right": (torch.rand(B, 3, h, w, generator=gen) * 2 - 1).to(DEV)}
    groups = {"lookups": ("lookup",), "convgrus": ("gru04", "gru08", "gru16"),
              "geo_and_disp_encoders": ("geo_encoder0", "geo_encoder1", "geo_encoder2", "encoder"), "heads": ("disp_head", "mask_feat_4")}
    ms = {k: [] for k in variants}
    stage = {k: [] for k in variants}
    outs = {}
    with torch.no_grad():
        for _ in range(3):                                              # alternate: the variants share the GPU's state
            for k, m in variants.items():
                t, outs[k] = timeit(lambda: m(dict(x))["disp_pred"], max(1, iters // 5), warm=1)
                ms[k].append(t)
                ub = m.update_block
                targets = {n: getattr(ub, n) for g in list(groups.values())[1:] for n in g}
                targets["lookup"] = geo.MultiRangeGeoEncodingVolume if k.startswith("patched") else ref_geo
                st = _stage_times(lambda: m(dict(x)), targets)
                stage[k].append({g: sum(st.get(n, 0.0) for n in names) for g, names in groups.items()})
    med = lambda v: sorted(v)[1]
    stage_ms = {k: {g: round(med([s[g] for s in v]), 2) for g in groups} for k, v in stage.items()}
    for k in stage_ms:
        stage_ms[k]["everything_else"] = round(med(ms[k]) - sum(stage_ms[k][g] for g in groups), 2)
    fp32 = outs["cudnn_fp32"].float()
    emit(config="c12 IGEV++ refinement loop, B=%d @%dx%d, 32 iterations (reference class + patch())" % (B, h, w),
         gpu="%s, %.0f W power limit" % (torch.cuda.get_device_name(DEV), _power_limit_w()),
         forward_ms={k: round(med(v), 2) for k, v in ms.items()},
         stage_ms_per_forward=stage_ms,
         epe_vs_cudnn_fp32_px={k: float("%.3e" % (o.float() - fp32).abs().mean().item()) for k, o in outs.items() if k != "cudnn_fp32"},
         disparity_std_px=round(fp32.std().item(), 2))
    del variants
    torch.cuda.empty_cache()


def c13(iters, B=8, h=256, w=512):
    """MonSter (monster/monster.py, the reference's class; oracle/monster.py supplies seeded weights for its Depth Anything V2
    ViT-L), batch 8 at 256x512 (W' = 128), 32 GRU iterations.  Variants in alternating rotation, medians of three: patch() of the
    uniform-YAML model (fp32), the unpatched uniform-YAML model (cuDNN fp32, TF32 off), the unpatched AMP-YAML model under the bf16
    autocast its trainer uses and patch() of the AMP-YAML model under the same autocast.  Per variant: whole-forward ms and ms per
    forward in the 39 lookups, the ConvGRUs, the motion encoders and the disp + mask heads of the three update blocks, the 14
    disparity warps, and everything else; EPE of each variant against the unpatched fp32 model."""
    import contextlib
    from oracle import monster as omon
    from openstereo_b200 import geo
    from openstereo_b200.patch import patch
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    ref_mod = omon.load_reference("stereo.modeling.models.monster.monster")
    ref_geo = omon.load_reference("stereo.modeling.models.monster.geometry").Combined_Geo_Encoding_Volume
    amp = omon.amp_dtype(omon.AMP_YAML)
    variants = {"patched": (patch(omon.monster(encoder="vitl").to(DEV)), None),
                "cudnn_fp32": (omon.monster(encoder="vitl").to(DEV), None),
                "amp_bf16": (omon.monster(omon.AMP_YAML, encoder="vitl").to(DEV), amp),
                "patched_amp_yaml": (patch(omon.monster(omon.AMP_YAML, encoder="vitl").to(DEV)), amp)}
    gen = torch.Generator().manual_seed(37)
    x = {"left": (torch.rand(B, 3, h, w, generator=gen) * 2 - 1).to(DEV), "right": (torch.rand(B, 3, h, w, generator=gen) * 2 - 1).to(DEV)}
    blocks = ("update_block", "update_block_mix_stereo", "update_block_mix_mono")
    groups = {"lookups": ("lookup",), "convgrus": ("gru04", "gru08", "gru16"), "encoders": ("encoder",),
              "heads": ("disp_head", "mask_feat_4"), "warps": ("warp",)}
    ms = {k: [] for k in variants}
    stage = {k: [] for k in variants}
    outs = {}

    def forward(m, dtype):
        with torch.autocast("cuda", dtype=dtype) if dtype else contextlib.nullcontext():
            return m(dict(x))["disp_pred"]

    def stage_times(k, m, dtype):
        targets = {"%s.%s" % (b, n): getattr(getattr(m, b), n) for b in blocks for names in list(groups.values())[1:4] for n in names}
        targets["lookup"] = geo.CombinedGeoEncodingVolume if k.startswith("patched") else ref_geo
        if k.startswith("patched"):
            return _stage_times(lambda: forward(m, dtype), targets, volume_fn="disp_warp")
        inner = ref_mod.disp_warp                                     # the unpatched _forward_pair reads the module global
        ref_mod.disp_warp = lambda *a, **kw: _timed_call(events, inner, *a, **kw)
        events = []
        try:
            st = _stage_times(lambda: forward(m, dtype), targets)
        finally:
            ref_mod.disp_warp = inner
        st["volume"] = round(sum(a.elapsed_time(b) for a, b in events), 3)
        return st

    with torch.no_grad():
        for _ in range(3):                                              # alternate: the variants share the GPU's state
            for k, (m, dtype) in variants.items():
                t, outs[k] = timeit(lambda: forward(m, dtype), max(1, iters // 5), warm=1)
                ms[k].append(t)
                st = stage_times(k, m, dtype)
                st["warp"] = st.pop("volume", 0.0)
                stage[k].append({g: sum(v for n, v in st.items() if n.rsplit(".", 1)[-1] in names) for g, names in groups.items()})
    med = lambda v: sorted(v)[1]
    stage_ms = {k: {g: round(med([s[g] for s in v]), 2) for g in groups} for k, v in stage.items()}
    for k in stage_ms:
        stage_ms[k]["everything_else"] = round(med(ms[k]) - sum(stage_ms[k][g] for g in groups), 2)
    fp32 = outs["cudnn_fp32"].float()
    emit(config="c13 MonSter refinement loop, B=%d @%dx%d, 32 iterations, vitl (reference class + patch())" % (B, h, w),
         gpu="%s, %.0f W power limit" % (torch.cuda.get_device_name(DEV), _power_limit_w()),
         forward_ms={k: round(med(v), 2) for k, v in ms.items()},
         stage_ms_per_forward=stage_ms,
         epe_vs_cudnn_fp32_px={k: float("%.3e" % (o.float() - fp32).abs().mean().item()) for k, o in outs.items() if k != "cudnn_fp32"},
         output_dtype={k: str(o.dtype) for k, o in outs.items()},
         disparity_std_px=round(fp32.std().item(), 2))
    del variants
    torch.cuda.empty_cache()


def _timed_call(events, fn, *args, **kw):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn(*args, **kw)
    b.record()
    events.append((a, b))
    return out


def _stage_times(run, targets, volume_fn=None):
    """One run of `run` with CUDA events around the forward of each target (a module, or a class whose __call__ is wrapped) and,
    with volume_fn, around ops.<volume_fn>: {stage: ms}."""
    events, restore = [], []

    def wrap(tag, inner):
        def fwd(*args, **kw):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = inner(*args, **kw)
            b.record()
            events.append((tag, a, b))
            return out
        return fwd
    for tag, t in targets.items():
        if isinstance(t, type):
            inner = t.__call__
            t.__call__ = wrap(tag, inner)
            restore.append(lambda t=t, inner=inner: setattr(t, "__call__", inner))
        else:
            inner = t.forward
            t.forward = wrap(tag, inner)
            restore.append(lambda t=t, inner=inner: setattr(t, "forward", inner))
    if volume_fn:
        inner = getattr(ops, volume_fn)
        setattr(ops, volume_fn, wrap("volume", inner))
        restore.append(lambda inner=inner: setattr(ops, volume_fn, inner))
    try:
        run()
        torch.cuda.synchronize()
    finally:
        for r in restore:
            r()
    out = {}
    for tag, a, b in events:
        out[tag] = round(out.get(tag, 0.0) + a.elapsed_time(b), 3)
    return out


def _power_limit_w():
    try:
        import subprocess
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(DEV.index or 0)],
                             capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return float("nan")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="c1,c3,c4,c5,gw")
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    for name in a.only.split(","):
        try:
            {"c1": c1, "c3": c3, "c4": c4, "c5": c5, "gw": gw, "c6": c6, "c7": c7, "c8": c8, "c9": c9, "c10": c10, "c11": c11,
             "c12": c12, "c13": c13}[name](a.iters)
        except Exception as exc:                                               # one config must not hide the others
            emit(config=name, error=repr(exc)[:300])
    if WORLD > 1:
        dist.destroy_process_group()
