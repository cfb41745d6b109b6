#!/usr/bin/env python
"""Generate tests/golden/*.npz by running the UNMODIFIED reference (authoring container only).

    python tools/make_golden.py            # needs /root/reference

For every case: seeded inputs -> the reference's own function/module (imported through
oracle/_reference_shim.py) -> outputs saved next to the inputs.  While generating, the script also
asserts that the oracle restatement is BIT-EQUAL to the reference on the same inputs; that is what
"the oracle is pinned against outputs of the reference itself" means (oracle/__init__.py).

Module weights are not stored (GwcNet is 27 MB): they are regenerated from
``oracle.seeded_init.seeded_state_dict(seed)``, and a checksum of the generated state_dict is stored
so a drift of torch's CPU RNG would be detected instead of silently changing the test.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import _reference_shim as shim                      # noqa: E402
from oracle import aggregation as oagg                          # noqa: E402
from oracle import cascade as ocas                              # noqa: E402
from oracle import coex as ocx                                  # noqa: E402
from oracle import cost_volume as ocv                           # noqa: E402
from oracle import geo_lookup as ogeo                           # noqa: E402
from oracle import igev_rt as oigrt                             # noqa: E402
from oracle import igevpp as oigpp                              # noqa: E402
from oracle import lightstereo as olight                        # noqa: E402
from oracle import models as omodels                            # noqa: E402
from oracle import msnet as oms                                 # noqa: E402
from oracle import regression as oreg                           # noqa: E402
from oracle import seeded_init as si                            # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def rnd(seed, *shape, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def checksum(sd):
    return float(sum(v.double().abs().sum() for v in sd.values()))


def save(name, **arrays):
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, name + ".npz")
    np.savez_compressed(path, **{k: (v.detach().numpy() if torch.is_tensor(v) else np.asarray(v))
                                 for k, v in arrays.items()})
    print("%-34s %8.1f KB" % (name, os.path.getsize(path) / 1024))


def must_equal(a, b, what):
    if not torch.equal(a, b):
        raise SystemExit("oracle != reference for %s (max diff %g)" % (what, (a - b).abs().max()))


def volumes():
    rcv = shim.load("stereo.modeling.cost_volume.cost_volume")
    rgw = shim.load("stereo.modeling.models.gwcnet.gwcnet_cost_processor")
    rpsm = shim.load("stereo.modeling.models.psmnet.psmnet_cost_processor")
    rigev = shim.load("stereo.modeling.models.igev.submodule")
    # (name, B, C, H, W, D, G)
    for name, b, c, h, w, d, g in [("gwc_small", 2, 24, 5, 20, 6, 4), ("gwc_d_gt_w", 1, 16, 3, 7, 10, 2),
                                   ("gwc_k12", 1, 96, 4, 33, 12, 8), ("gwc_k8_w128", 1, 64, 2, 128, 48, 8)]:
        l, r = rnd(1, b, c, h, w), rnd(2, b, c, h, w)
        ref = rcv.build_gwc_volume(l, r, d, g)
        must_equal(ref, ocv.build_gwc_volume(l, r, d, g), name)
        # the GwcNet method copy is the same function (gwcnet_cost_processor.py:22-39)
        proc = rgw.GwcVolumeCostProcessor(maxdisp=d * 4, downsample=4, num_groups=g)
        must_equal(ref, proc.build_gwc_volume(l, r), name + "/method")
        save(name, left=l, right=r, maxdisp=d, groups=g, out=ref)
    for name, b, c, h, w, d in [("concat_small", 2, 6, 5, 20, 6), ("concat_d_gt_w", 1, 4, 3, 7, 10),
                                ("concat_c12_w128", 1, 12, 2, 128, 48)]:
        l, r = rnd(3, b, c, h, w), rnd(4, b, c, h, w)
        ref = rcv.build_concat_volume(l, r, d)
        must_equal(ref, ocv.build_concat_volume(l, r, d), name)
        must_equal(ref, rpsm.cat_fms(l, r, max_disp=d), name + "/cat_fms")
        must_equal(ref, ocv.cat_fms(l, r, max_disp=d), name + "/cat_fms oracle")
        unmasked = rigev.build_concat_volume(l, r, d)
        must_equal(unmasked, ocv.build_concat_volume(l, r, d, mask_left=False), name + "/unmasked")
        save(name, left=l, right=r, maxdisp=d, out=ref, out_unmasked=unmasked)
    l, r = rnd(5, 2, 24, 6, 23), rnd(6, 2, 24, 6, 23)
    ref = rcv.correlation_volume(l, r, 9)
    must_equal(ref, ocv.correlation_volume(l, r, 9), "corr")
    save("corr_small", left=l, right=r, maxdisp=9, out=ref)
    # fused gwc+concat as GwcVolumeCostProcessor.forward returns it
    lg, rg, lc, rc = rnd(7, 1, 32, 4, 40), rnd(8, 1, 32, 4, 40), rnd(9, 1, 3, 4, 40), rnd(10, 1, 3, 4, 40)
    proc = rgw.GwcVolumeCostProcessor(maxdisp=64, downsample=4, num_groups=4, use_concat_volume=True)
    ref = proc({"ref_feature": {"gwc_feature": lg, "concat_feature": lc},
                "tgt_feature": {"gwc_feature": rg, "concat_feature": rc}})["cost_volume"]
    must_equal(ref, ocv.gwc_concat_volume(lg, rg, lc, rc, 16, 4), "fused")
    save("gwc_concat_fused", lg=lg, rg=rg, lc=lc, rc=rc, maxdisp=16, groups=4, out=ref)
    # cat_fms with start_disp / dilation (only the oracle restates these; PSMNet never uses them)
    l, r = rnd(11, 1, 4, 3, 17), rnd(12, 1, 4, 3, 17)
    for tag, kw in [("neg", dict(max_disp=8, start_disp=-3, dilation=1)), ("dil", dict(max_disp=9, start_disp=0, dilation=2))]:
        ref = rpsm.cat_fms(l, r, **kw)
        must_equal(ref, ocv.cat_fms(l, r, **kw), "cat_fms " + tag)
        save("cat_fms_" + tag, left=l, right=r, out=ref, **kw)


def regression():
    rreg = shim.load("stereo.modeling.disp_pred.disp_regression")
    rgdp = shim.load("stereo.modeling.models.gwcnet.gwcnet_disp_processor")
    rpdp = shim.load("stereo.modeling.models.psmnet.psmnet_disp_processor")
    rmet = shim.load("stereo.evaluation.metric_per_image") if os.path.exists(
        os.path.join(shim.REFERENCE_ROOT, "stereo/evaluation/metric_per_image.py")) else None
    import torch.nn.functional as F
    cost = rnd(20, 2, 12, 4, 9, scale=3.0)
    prob = F.softmax(cost, dim=1)
    ref_keep = rreg.disparity_regression(prob, 12)
    ref_flat = rgdp.disparity_regression(prob, 12)
    must_equal(ref_keep, oreg.disparity_regression(prob, 12, keepdim=True), "regression keepdim")
    must_equal(ref_flat, oreg.disparity_regression(prob, 12, keepdim=False), "regression flat")
    must_equal(ref_keep, oreg.softargmin(cost, 12), "softargmin")
    save("softargmin_small", cost=cost, prob=prob, maxdisp=12, out_keepdim=ref_keep, out_flat=ref_flat)
    fsa = rpdp.FasterSoftArgmin(max_disp=16)
    cost = rnd(21, 2, 16, 3, 5, scale=2.0)
    ref = fsa(cost)
    must_equal(ref, oreg.faster_soft_argmin(cost, 16), "faster soft argmin")
    save("faster_softargmin", cost=cost, maxdisp=16, out=ref)
    # fused tails: trilinear x4 -> softmax -> regression
    low = rnd(22, 2, 1, 6, 5, 7, scale=3.0)
    up = F.interpolate(low, [24, 20, 28], mode="trilinear")
    ref_gwc = rgdp.disparity_regression(F.softmax(torch.squeeze(up, 1), dim=1), 24)
    must_equal(ref_gwc, oreg.upsample_softargmin(low, 24, 20, 28, align_corners=False), "gwc tail")
    up = F.interpolate(low, [24, 20, 28], mode="trilinear", align_corners=True)
    ref_psm = rpdp.FasterSoftArgmin(max_disp=24)(torch.squeeze(up, 1))
    must_equal(ref_psm, oreg.upsample_softargmin(low, 24, 20, 28, align_corners=True, psm_tail=True), "psm tail")
    save("upsample_softargmin", cost=low, maxdisp=24, out_h=20, out_w=28, out_gwc=ref_gwc, out_psm=ref_psm)
    if rmet is not None:
        pred, gt = rnd(23, 3, 6, 8).abs() * 40, rnd(24, 3, 6, 8).abs() * 60
        gt[2] = 500.0                                  # an image with no valid pixel
        mask = (gt < 192) & (gt > 0)
        ref = rmet.epe_metric(pred, gt, mask)
        must_equal(ref, oreg.epe_per_image(pred, gt, mask), "epe")
        save("epe_per_image", pred=pred, gt=gt, out=ref)


def modules():
    rgh = shim.load("stereo.modeling.models.gwcnet.hourglass")
    rgdp = shim.load("stereo.modeling.models.gwcnet.gwcnet_disp_processor")
    rpcp = shim.load("stereo.modeling.models.psmnet.psmnet_cost_processor")
    rsbh = shim.load("stereo.modeling.models.stereobase.hourglass")
    with torch.no_grad():
        # GwcNet hourglass, 8 channels
        ref, mine = rgh.Hourglass(8).eval(), oagg.GwcHourglass(8).eval()
        sd = si.seeded_state_dict(ref.state_dict(), seed=31)
        ref.load_state_dict(sd), mine.load_state_dict(sd)
        x = rnd(32, 1, 8, 8, 8, 12)
        y = ref(x)
        must_equal(y, mine(x), "gwc hourglass")
        save("gwc_hourglass_c8", x=x, out=y, seed=31, sd_checksum=checksum(sd))
        # GwcDispProcessor eval branch
        kw = dict(maxdisp=32, downsample=4, num_groups=4, use_concat_volume=True, concat_channels=2)
        ref, mine = rgdp.GwcDispProcessor(**kw).eval(), oagg.GwcDispProcessor(**kw).eval()
        sd = si.seeded_state_dict(ref.state_dict(), seed=33, scale={"classif3.2.weight": 60.0})
        ref.load_state_dict(sd), mine.load_state_dict(sd)
        vol = rnd(34, 1, 8, 8, 8, 16)
        left = torch.zeros(1, 3, 32, 64)
        y = ref({"cost_volume": vol, "left": left})["inference_disp"]["disp_est"]
        must_equal(y, mine(vol, 32, 64), "gwc disp processor")
        save("gwc_disp_processor", volume=vol, out=y, logits=mine.aggregate(vol), seed=33, sd_checksum=checksum(sd))
        # PSMAggregator
        ref, mine = rpcp.PSMAggregator(max_disp=32, in_planes=8).eval(), oagg.PSMAggregator(32, 8).eval()
        sd = si.seeded_state_dict(ref.state_dict(), seed=35,
                                  scale={"classif1.1.weight": 20.0, "classif2.1.weight": 20.0, "classif3.1.weight": 20.0})
        ref.load_state_dict(sd), mine.load_state_dict(sd)
        raw = rnd(36, 1, 8, 8, 8, 16)
        ys, ms = ref(raw), mine(raw)
        for a, b in zip(ys, ms):
            must_equal(a, b, "psm aggregator")
        low = mine.aggregate(raw)
        save("psm_aggregator", raw=raw, cost3_low=low[2], cost2_low=low[1], cost1_low=low[0], seed=35,
             sd_checksum=checksum(sd))
        # StereoBase hourglass + classifier + softargmin
        bc = [16, 16, 24, 20]
        ref = rsbh.Hourglass(8, bc).eval()
        mine = oagg.StereoBaseCostHead(8, bc, max_disp=64).eval()
        sd_h = si.seeded_state_dict(ref.state_dict(), seed=37)
        ref.load_state_dict(sd_h)
        sd = si.seeded_state_dict(mine.state_dict(), seed=38, scale={"classifier.weight": 30.0})
        sd.update({"cost_agg." + k: v for k, v in sd_h.items()})
        mine.load_state_dict(sd)
        vol = rnd(39, 1, 8, 16, 16, 32)
        feats = [rnd(40, 1, 16, 16, 32), rnd(41, 1, 16, 8, 16), rnd(42, 1, 24, 4, 8), rnd(43, 1, 20, 2, 4)]
        geo = ref(vol, feats)
        geo2, init_disp = mine(vol, feats)
        must_equal(geo, geo2, "stereobase hourglass")
        save("stereobase_head", volume=vol, f0=feats[0], f1=feats[1], f2=feats[2], f3=feats[3], geo=geo,
             init_disp=init_disp, seed_hourglass=37, seed_head=38, sd_checksum=checksum(sd))


def models():
    with torch.no_grad():
        cfg = shim.load_cfg("cfgs/gwcnet/gwcnet_sceneflow.yaml").MODEL
        ref = shim.load("stereo.modeling.models.gwcnet.gwcnet").GwcNet(cfg).eval()
        mine = omodels.GwcNet(cfg.MAX_DISP, cfg.USE_CONCAT_VOLUME, cfg.CONCAT_CHANNELS, cfg.DOWNSAMPLE,
                              cfg.NUM_GROUPS).eval()
        assert list(ref.state_dict().keys()) == list(mine.state_dict().keys())
        sd = si.seeded_state_dict(ref.state_dict(), seed=1, scale=si.GWCNET_SCALE)
        ref.load_state_dict(sd), mine.load_state_dict(sd)
        x = {"left": rnd(50, 1, 3, 64, 128), "right": rnd(51, 1, 3, 64, 128)}
        y = ref(dict(x))["disp_pred"]
        must_equal(y, mine(dict(x))["disp_pred"], "GwcNet")
        save("gwcnet_64x128", left=x["left"], right=x["right"], out=y, seed=1, sd_checksum=checksum(sd))

        cfg = shim.load_cfg("cfgs/psmnet/psmnet_sceneflow.yaml").MODEL
        ref = shim.load("stereo.modeling.models.psmnet.psmnet").PSMNet(cfg).eval()
        mine = omodels.PSMNet(cfg.MAX_DISP).eval()
        assert list(ref.state_dict().keys()) == list(mine.state_dict().keys())
        sd = si.seeded_state_dict(ref.state_dict(), seed=1, scale=si.PSMNET_SCALE, keep=si.PSMNET_KEEP)
        ref.load_state_dict(sd), mine.load_state_dict(sd)
        # inputs are rounded to fp16-representable values so they can be stored compactly and exactly
        x = {"left": rnd(52, 1, 3, 256, 256).half().float(), "right": rnd(53, 1, 3, 256, 256).half().float()}
        y = ref(dict(x))
        m = mine(dict(x))
        for a, b in zip(y["train_preds"], m["train_preds"]):
            must_equal(a, b, "PSMNet")
        save("psmnet_256x256", left=x["left"].half(), right=x["right"].half(), out=y["disp_pred"], seed=1,
             sd_checksum=checksum(sd))


def lookups():
    """SURVEY.md section 8(f) rows 1 and 3: geometry-encoding volume lookup and context up-sampling."""
    rgeo = shim.load("stereo.modeling.models.igev.geometry")
    rsb = shim.load("stereo.modeling.models.stereobase.gru_blocks")
    rblk = shim.load("stereo.modeling.models.stereobase.igev_blocks")
    # (name, B, C_feat, C_geo, D, H, W, levels, radius)
    for name, b, cf, cg, d, h, w, levels, radius in (("geo_lookup_small", 2, 6, 8, 12, 3, 10, 2, 4),
                                                     ("geo_lookup_3lvl", 1, 4, 3, 17, 2, 21, 3, 2)):
        f1, f2 = rnd(60, b, cf, h, w), rnd(61, b, cf, h, w)
        vol = rnd(62, b, cg, d, h, w)
        # disparities inside, at the borders of and beyond the volume; two iterations like the GRU loop
        disp = torch.rand(b, 1, h, w, generator=torch.Generator().manual_seed(63)) * (d + 6) - 3
        disp[0, 0, 0, :3] = torch.tensor([0.0, d - 1.0, 2.5])
        coords = torch.arange(w).float().reshape(1, 1, w, 1).repeat(b, h, 1, 1)
        ref = rgeo.Combined_Geo_Encoding_Volume(f1, f2, vol, num_levels=levels, radius=radius)
        ref2 = rsb.CombinedGeoEncodingVolume(f1, f2, vol, num_levels=levels, radius=radius)
        mine = ogeo.GeoEncodingVolume(f1, f2, vol, num_levels=levels, radius=radius)
        out = ref(disp, coords)
        must_equal(out, ref2(disp, coords), name + " igev vs stereobase class")
        must_equal(out, mine(disp, coords), name)
        must_equal(ref.init_corr_pyramid[-1], mine.corr_pyramid[-1], name + " corr pyramid")
        must_equal(ref.geo_volume_pyramid[-1], mine.geo_pyramid[-1], name + " geo pyramid")
        save(name, fmap1=f1, fmap2=f2, volume=vol, disp=disp, coords=coords, levels=levels, radius=radius, out=out,
             geo_last=ref.geo_volume_pyramid[-1], corr_last=ref.init_corr_pyramid[-1])
    low = rnd(64, 2, 1, 5, 7).abs() * 20
    wts = torch.softmax(rnd(65, 2, 9, 20, 28), dim=1)
    ref = rblk.context_upsample(low, wts)
    must_equal(ref, ogeo.context_upsample(low, wts), "context_upsample")
    save("context_upsample", disp_low=low, up_weights=wts, scale=4, out=ref)


def lightstereo():
    """SURVEY.md section 8(f) row 2: LightStereo's 2D aggregation (cfgs/lightstereo: in_channels 48, blocks [4, 8, 14], expanse 4
    in LightStereo-M; a reduced [1, 2, 2] stack with every block kind keeps the fixture small)."""
    ragg = shim.load("stereo.modeling.models.lightstereo.aggregation")
    with torch.no_grad():
        args = dict(in_channels=12, left_att=True, blocks=[1, 2, 2], expanse_ratio=4, backbone_channels=[10, 14, 18])
        ref, mine = ragg.Aggregation(**args).eval(), olight.Aggregation(**args).eval()
        assert list(ref.state_dict().keys()) == list(mine.state_dict().keys())
        sd = si.seeded_state_dict(ref.state_dict(), seed=5)
        ref.load_state_dict(sd), mine.load_state_dict(sd)
        x = rnd(86, 2, 12, 8, 20)
        feats = [rnd(87, 2, 10, 8, 20), rnd(88, 2, 14, 4, 10), rnd(89, 2, 18, 2, 5)]
        y = ref(x, feats)[0]
        must_equal(y, mine(x, feats)[0], "LightStereo aggregation")
        if not y.std() > 1e-3:
            raise SystemExit("degenerate LightStereo fixture (std %g)" % y.std())
        save("lightstereo_aggregation", x=x, f0=feats[0], f1=feats[1], f2=feats[2], out=y, seed=5, sd_checksum=checksum(sd))


def flavours():
    """SURVEY.md section 8(f) row 4: the remaining volume / regression flavours (oracle pinned ahead of the kernels)."""
    import torch.nn.functional as F
    rcv = shim.load("stereo.modeling.cost_volume.cost_volume")
    import types
    for missing in ("trimesh", "imageio", "open3d", "transformations"):     # imported at module level by foundationstereo/Utils.py,
        if missing not in sys.modules:                                      # never dereferenced by the two functions used here
            try:
                __import__(missing)
            except Exception:
                sys.modules[missing] = types.ModuleType(missing)
    rfs = shim.load("stereo.modeling.models.foundationstereo.core.submodule")
    rpp = shim.load("stereo.modeling.models.igevpp.submodule")
    rcas = shim.load("stereo.modeling.models.casnet.submodule")
    l, r = rnd(80, 2, 24, 3, 17), rnd(81, 2, 24, 3, 17)
    ref = rfs.build_gwc_volume(l, r, 9, 4)
    must_equal(ref, ocv.build_gwc_volume_normalized(l, r, 9, 4), "normalised gwc volume")
    save("gwc_normalized", left=l, right=r, maxdisp=9, groups=4, out=ref)
    ref = rcv.CoExCostVolume(6, group=3)(l, r)
    must_equal(ref, ocv.coex_cost_volume(l, r, 6, 3), "CoEx volume")
    save("coex_volume", left=l, right=r, maxdisp=6, group=3, out=ref)
    ls, rs = rnd(82, 1, 5, 2, 6), rnd(83, 1, 5, 2, 6)
    ref = rcv.build_corr_volume(ls, rs, 9)                          # 9 > W = 6: exercises the unshifted else-branch
    must_equal(ref, ocv.build_corr_volume(ls, rs, 9), "corr volume (d >= W quirk)")
    save("corr_volume_quirk", left=ls, right=rs, maxdisp=9, out=ref)
    prob = F.softmax(rnd(84, 2, 12, 3, 5, scale=2.0), dim=1)
    ref = rpp.disparity_regression(prob, 48, 4)
    must_equal(ref, oreg.disparity_regression_interval(prob, 48, 4), "interval regression")
    vals = rnd(85, 2, 12, 3, 5).abs() * 30
    ref2 = rcas.disparity_regression(prob, vals)
    must_equal(ref2, oreg.disparity_regression_values(prob, vals), "explicit-hypothesis regression")
    save("regression_flavours", prob=prob, maxdisp=48, interval=4, out_interval=ref, values=vals, out_values=ref2)


def cascade_samples(seed, b, d, h, w):
    """Per-pixel hypotheses covering every case of the warped volume: fractional, integer and negative samples, and columns
    w - disp beyond both image edges (below -1, in (-1, 0), above W - 1)."""
    g = torch.Generator().manual_seed(seed)
    disp = torch.rand(b, d, h, w, generator=g) * (w + 8) - 6
    disp[:, 0] = torch.randint(-3, w + 3, (b, h, w), generator=g).float()           # integer samples
    disp[:, 1] = torch.arange(w).float() + 0.5                                      # column -0.5: between -1 and 0
    disp[:, 2] = torch.arange(w).float() - (w - 1) - 0.25                           # column W - 0.75: beyond the right edge
    return disp


def cascade():
    """CasStereo: both GetCostVolume variants at a height whose row coordinates partly come back off-integer, the
    CostAggregation tail at x4 and x2, and a seeded CasPSMNet at 256x512 (a strided sample of its disparity map)."""
    rpsm = shim.load("stereo.modeling.models.casnet.cas_psm")
    rgwc = shim.load("stereo.modeling.models.casnet.cas_gwc")
    b, d, h, w = 2, 5, 13, 21
    assert any((hh / ((h - 1.0) / 2.0) - 1.0 + 1) * ((h - 1) / 2) != hh for hh in range(h))
    disp = cascade_samples(90, b, d, h, w)
    x, y = rnd(91, b, 6, h, w), rnd(92, b, 6, h, w)
    ref = rpsm.GetCostVolume()(x, y, disp, d)
    must_equal(ref, ocas.warped_concat_volume(x, y, disp, d), "CasPSMNet volume")
    save("cas_volume_psm", x=x, y=y, disp=disp, out=ref)
    fl = {"gwc_feature": rnd(93, b, 8, h, w), "concat_feature": rnd(94, b, 3, h, w)}
    fr = {"gwc_feature": rnd(95, b, 8, h, w), "concat_feature": rnd(96, b, 3, h, w)}
    ref = rgwc.GetCostVolume()(fl, fr, disp, d, 2)
    must_equal(ref, ocas.warped_gwc_concat_volume(fl, fr, disp, d, 2), "CasGwcNet volume")
    save("cas_volume_gwc", xg=fl["gwc_feature"], yg=fr["gwc_feature"], xc=fl["concat_feature"], yc=fr["concat_feature"],
         disp=disp, groups=2, out=ref)
    with torch.no_grad():
        agg = rpsm.CostAggregation(8, 8).eval()
        agg.load_state_dict(si.seeded_state_dict(agg.state_dict(), seed=97))
        arrays = {}
        for tag, (fd, hl, wl) in (("x4", (48, 5, 7)), ("x2", (24, 10, 14))):
            logits = rnd(98, 1, 1, 12, hl, wl, scale=3.0)
            vals = cascade_samples(99, 1, fd, 20, 28) * 4
            want = ocas.upsample_softargmin_values(logits, fd, 20, 28, vals)
            agg.classif3 = _Const(logits)                                           # feed the tail known logits
            must_equal(agg(torch.zeros(1, 8, 4, 4, 4), fd, 20, 28, vals), want, "CasStereo tail " + tag)
            arrays.update({"cost_" + tag: logits, "values_" + tag: vals, "out_" + tag: want})
        save("cas_tail", **arrays)
        cfg = shim.load_cfg("cfgs/casnet/casnet_psm_sceneflow.yaml").MODEL
        m = rpsm.PSMNet(cfg).eval()
        sd = si.seeded_state_dict(m.state_dict(), seed=1, scale=ocas.CASNET_SCALE)
        m.load_state_dict(sd)
        left, right = rnd(100, 1, 3, 256, 512), rnd(101, 1, 3, 256, 512)
        out = m({"left": left, "right": right})["disp_pred"]
        save("cas_psmnet_256x512", seed_left=100, seed_right=101, weight_seed=1, checksum=checksum(sd), disp_sample=out[:, ::8, ::8],
             disp_mean=out.mean(), disp_std=out.std())


def coex_tie_logits(seed, b, d, h, w):
    """Small-integer logits: many exact ties along D, so the fixtures pin the order of equal values in the top-k selection."""
    return torch.randint(-3, 3, (b, 1, d, h, w), generator=torch.Generator().manual_seed(seed)).float()


def coex():
    rcp = shim.load("stereo.modeling.models.coex.coex_cost_processor")
    rdp = shim.load("stereo.modeling.models.coex.coex_disp_processor")
    with torch.no_grad():
        # attention volume: the reference module's own forward vs the oracle on the module's desc outputs
        att = rcp.AttentionCostVolume(32, 20, 12, head=2).eval()
        att.load_state_dict(si.seeded_state_dict(att.state_dict(), seed=110))
        l, r = rnd(111, 2, 20, 6, 19), rnd(112, 2, 20, 6, 19)
        ref = att(l, r)[:, :, :-1]
        xd, yd = att.desc(att.conv(l)), att.desc(att.conv(r))
        must_equal(ref, ocx.attention_volume(xd, yd, 8, 2), "CoEx attention volume")
        save("coex_attention", x=xd, y=yd, maxdisp=8, head=2, out=ref)
        # regression + upfeat, probabilities in; tie-heavy logits, k = 2 and 3
        arrays = {}
        cost = coex_tie_logits(113, 2, 10, 5, 7)
        spx = torch.softmax(rnd(114, 2, 9, 20, 28, scale=2.0), 1)
        for k in (2, 3):
            reg = rdp.Regression(40, k).eval()
            ref = reg(cost, spx)[0]
            must_equal(ref, ocx.regression(cost, spx, k), "CoEx regression k=%d" % k)
            arrays["out_k%d" % k] = ref
            arrays["ind_k%d" % k] = ocx.topk_pool(cost, k)[1]
        save("coex_regression", cost=cost, spx=spx, **arrays)
        # nearest resampling along each dimension, including the 136 -> 135 of CoEx's 540 x 960 evaluation size
        x = rnd(115, 1, 1, 7, 136, 12)
        arrays = {"x": x}
        for i, size in enumerate(((6, 135, 24), (14, 13, 12), (7, 136, 5))):
            y = torch.nn.functional.interpolate(x, size=size, mode="nearest")
            want = x[:, :, ocx.nearest_index(size[0], 7)][:, :, :, ocx.nearest_index(size[1], 136)][..., ocx.nearest_index(size[2], 12)]
            must_equal(y, want, "nearest index %s" % (size,))
            arrays["size%d" % i], arrays["out%d" % i] = torch.tensor(size), y
        save("coex_nearest", **arrays)
        # a small Aggregation (D = 16, 10 x 12 image: both upper levels mismatch their skip, 2 -> 3 rows and 3 -> 5)
        ref_agg = rcp.Aggregation(max_disparity=64).eval()
        mine = ocx.Aggregation(max_disparity=64).eval()
        assert sorted(ref_agg.state_dict()) == sorted(mine.state_dict())
        sd = si.seeded_state_dict(ref_agg.state_dict(), seed=116)
        ref_agg.load_state_dict(sd), mine.load_state_dict(sd)
        img = [rnd(117, 1, 96, 10, 12), rnd(118, 1, 64, 5, 6), rnd(119, 1, 192, 3, 3), rnd(120, 1, 160, 2, 2)]
        cost = rnd(121, 1, 1, 16, 10, 12, scale=0.3)
        ref = ref_agg(img, cost)
        must_equal(ref, mine(img, cost), "CoEx Aggregation")
        save("coex_aggregation", weight_seed=116, checksum=checksum(sd), img0=img[0], img1=img[1], img2=img[2], img3=img[3], cost=cost,
             out=ref)


def msnet():
    rsub = oms.load_reference("stereo.modeling.models.msnet.submodule")
    rm3 = oms.load_reference("stereo.modeling.models.msnet.MSNet3D")
    with torch.no_grad():
        # two MobileV2_Residual_3D blocks on odd extents: the first block of dres0 and a stride-2 hourglass block
        arrays = {}
        for i, (cin, chid, cout, stride) in enumerate(((40, 120, 32, 1), (32, 64, 64, 2))):
            ref = rsub.MobileV2_Residual_3D(cin, cout, stride, chid / cin).eval()
            mine = oms.MobileV2Residual3D(cin, cout, stride, chid / cin).eval()
            assert not ref.use_res_connect and sorted(ref.state_dict()) == sorted(mine.state_dict())
            seed = 130 + i
            sd = si.seeded_state_dict(ref.state_dict(), seed=seed)
            ref.load_state_dict(sd), mine.load_state_dict(sd)
            x = rnd(132 + i, 1, cin, 5, 7, 9)
            out = ref(x)
            must_equal(out, mine(x), "MobileV2_Residual_3D %s" % ((cin, chid, cout, stride),))
            arrays.update({"seed%d" % i: seed, "x%d" % i: x, "out%d" % i: out})
        save("msnet_block", **arrays)
        # the 3D part of the model (every block, the three hourglasses, classif3, the tail) on a small volume
        cfg = shim.load_cfg("cfgs/msnet/msnet3d_sceneflow.yaml").MODEL
        model = rm3.MSNet3D(cfg).eval()
        agg = oms.Aggregation().eval()
        sd = si.seeded_state_dict(agg.state_dict(), seed=134, scale=oms.MSNET3D_SCALE)
        agg.load_state_dict(sd)
        for name, mod in (("dres0", model.dres0), ("dres1", model.dres1), ("encoder_decoder1", model.encoder_decoder1),
                          ("classif3", model.classif3)):
            mod.load_state_dict({k[len(name) + 1:]: v for k, v in sd.items() if k.startswith(name + ".")})
        vol = rnd(135, 1, 40, 8, 8, 8)
        hg = model.encoder_decoder1(model.dres0(vol))
        must_equal(hg, agg.encoder_decoder1(agg.dres0(vol)), "hourglass3D")
        logits = agg.logits(vol)
        disp = agg(vol, 32, 32)
        save("msnet_aggregation", weight_seed=134, checksum=checksum(sd), volume=vol, logits=logits, disp=disp)
        # the whole model from the unchanged YAML, seeded and sharpened: the reference's forward vs the restated eval forward
        model.load_state_dict(si.seeded_state_dict(model.state_dict(), seed=1, scale=oms.MSNET3D_SCALE))
        g = torch.Generator().manual_seed(136)
        left, right = torch.randn(1, 3, 64, 128, generator=g), torch.randn(1, 3, 64, 128, generator=g)
        disp = model({"left": left, "right": right})["disp_pred"]
        must_equal(disp, oms.eval_forward(model.feature_extraction, oms.aggregation_of(model), left, right)["disp_pred"],
                   "MSNet3D eval forward")
        save("msnet3d_model", weight_seed=1, checksum=checksum(model.state_dict()), left=left, right=right, disp=disp,
             disp_std=disp.std())


# (B, C, D, H, W, levels, radius) of tests/golden/geo_volume_lookup.npz, case i stored under keys suffixed with i
GEO_VOLUME_CASES = ((2, 8, 48, 3, 10, 2, 4), (1, 3, 17, 2, 21, 1, 4), (1, 5, 24, 2, 9, 3, 4), (2, 4, 20, 3, 7, 3, 2))


def igev_rt():
    """IGEV-RT's geometry-only encoding volume (igev_rt/geometry.py): the reference class against the oracle, bit for bit.  The
    disparities run from below -r to past D + r, so taps leave the row at both ends on every level."""
    rgeo = oigrt.load_reference("stereo.modeling.models.igev_rt.geometry")
    arrays = {}
    for i, (b, c, d, h, w, levels, radius) in enumerate(GEO_VOLUME_CASES):
        vol = rnd(140 + i, b, c, d, h, w)
        disp = torch.rand(b, 1, h, w, generator=torch.Generator().manual_seed(150 + i)) * (d + 2 * radius + 8) - radius - 4
        disp[0, 0, 0, :5] = torch.tensor([0.0, d - 1.0, 2.5, -radius - 1.5, d + radius + 1.5])
        ref = rgeo.Geo_Encoding_Volume(vol, num_levels=levels, radius=radius)
        out = ref(disp)
        must_equal(out, oigrt.GeoEncodingVolume(vol, num_levels=levels, radius=radius)(disp), "geo_volume_lookup case %d" % i)
        assert out.shape == (b, levels * c * (2 * radius + 1), h, w)
        arrays.update({"volume%d" % i: vol, "disp%d" % i: disp, "levels%d" % i: levels, "radius%d" % i: radius, "out%d" % i: out})
    save("geo_volume_lookup", cases=len(GEO_VOLUME_CASES), **arrays)


# (B, C, D0, D1, D2, H, W, levels, radius) of tests/golden/igevpp_lookup.npz, case i stored under keys suffixed with i
IGEVPP_CASES = ((1, 8, 48, 48, 48, 2, 10, 2, 4), (1, 3, 20, 13, 30, 2, 21, 1, 4), (1, 5, 24, 17, 9, 2, 9, 2, 2),
                (2, 4, 16, 24, 6, 3, 7, 2, 4))


def igevpp():
    """IGEV++'s multi-range encoding volume (igevpp/geometry.py): the reference class against the oracle, bit for bit.  The
    disparities run from below -r to past 4 * max(D) + r, so taps leave every row at both ends; D1 and D2 differ from D0 >> i."""
    rgeo = oigpp.load_reference("stereo.modeling.models.igevpp.geometry")
    arrays = {}
    for i, (b, c, d0, d1, d2, h, w, levels, radius) in enumerate(IGEVPP_CASES):
        v0, v1, v2 = rnd(170 + i, b, c, d0, h, w), rnd(180 + i, b, c, d1, h, w), rnd(190 + i, b, c, d2, h, w)
        f1, f2 = rnd(200 + i, b, 6, h, w), rnd(210 + i, b, 6, h, w)
        top = 4 * max(d0, d1, d2) + 2 * radius + 8
        disp = torch.rand(b, 1, h, w, generator=torch.Generator().manual_seed(220 + i)) * top - radius - 4
        disp[0, 0, 0, :5] = torch.tensor([0.0, d0 - 1.0, 2.5, -radius - 1.5, 4 * d2 + radius + 1.5])
        coords = torch.arange(w).float().reshape(1, 1, w, 1).repeat(b, h, 1, 1)
        ref = rgeo.Combined_Geo_Encoding_Volume(v0, v1, v2, f1, f2, radius=radius, num_levels=levels)
        outs = ref(disp, coords)
        mine = oigpp.MultiRangeGeoEncodingVolume(v0, v1, v2, f1, f2, radius=radius, num_levels=levels)(disp, coords)
        t = 2 * radius + 1
        for name, a, m, shape in zip(("feat0", "feat1", "feat2", "corr"), outs, mine,
                                     ((b, levels * c * t, h, w), (b, c * t, h, w), (b, c * t, h, w), (b, levels * t, h, w))):
            must_equal(a, m, "igevpp_lookup case %d %s" % (i, name))
            assert a.shape == shape, (name, a.shape, shape)
            arrays["%s%d" % (name, i)] = a
        arrays.update({"vol0_%d" % i: v0, "vol1_%d" % i: v1, "vol2_%d" % i: v2, "fmap1_%d" % i: f1, "fmap2_%d" % i: f2,
                       "disp%d" % i: disp, "levels%d" % i: levels, "radius%d" % i: radius})
    save("igevpp_lookup", cases=len(IGEVPP_CASES), **arrays)


class _Const(torch.nn.Module):
    def __init__(self, t):
        super().__init__()
        self.t = t

    def forward(self, _):
        return self.t


SECTIONS = ["volumes", "regression", "modules", "models", "lookups", "flavours", "lightstereo", "cascade", "coex", "msnet", "igev_rt", "igevpp"]

if __name__ == "__main__":
    if not shim.available():
        raise SystemExit("reference tree not found; golden vectors can only be generated in the authoring container")
    torch.set_num_threads(os.cpu_count() or 1)
    for name in sys.argv[1:] or SECTIONS:                       # e.g. `python tools/make_golden.py cascade`
        globals()[name]()
    print("all oracle restatements bit-equal to the reference; golden vectors written to", OUT)
