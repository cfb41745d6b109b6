"""Oracle: IGEV++'s multi-range geometry encoding volume (TEST INFRASTRUCTURE -- see oracle/__init__.py).

* ``MultiRangeGeoEncodingVolume``  restates ``Combined_Geo_Encoding_Volume`` stereo/modeling/models/igevpp/geometry.py:6-87 (+
  ``bilinear_sampler`` igevpp/utils.py): the combined lookup of oracle/geo_lookup.py over a pair-averaged pyramid of the first
  volume, plus one bilinear lookup each of the second volume at dx + disp / 2 and the third at dx + disp / 4 (no pyramid, their own
  plane counts), returned as four separate tensors.
* ``igevpp(yaml, seed)``  the reference's own IGEVPPStereo built from an unchanged YAML with the timm stand-in and seeded weights.

Same aten calls in the same order as the reference, so the lookup is bit-equal on CPU (asserted by tools/make_golden.py).
"""
import torch
import torch.nn.functional as F

from oracle import _reference_shim as shim
from oracle import seeded_init as si
from oracle.geo_lookup import _sample_rows, all_pairs_correlation

UNIFORM_YAML = "cfgs/igevpp/igevpp_sceneflow_uniform.yaml"
AMP_YAML = "cfgs/igevpp/igevpp_sceneflow_amp.yaml"
# As for IGEV-RT (oracle/igev_rt.py): sharpen the shared classifier so that the three initial disparities spread over the range.
IGEVPP_SCALE = {"classifier.weight": 8.0}


class MultiRangeGeoEncodingVolume:
    def __init__(self, geo_volume0, geo_volume1, geo_volume2, init_fmap1, init_fmap2, radius=4, num_levels=2):
        self.num_levels, self.radius = num_levels, radius
        corr = all_pairs_correlation(init_fmap1, init_fmap2)
        b, c, d0, h, w = geo_volume0.shape
        geo = geo_volume0.permute(0, 3, 4, 1, 2).reshape(b * h * w, c, 1, d0)
        self.vol1 = geo_volume1.permute(0, 3, 4, 1, 2).reshape(b * h * w, c, 1, geo_volume1.shape[2])
        self.vol2 = geo_volume2.permute(0, 3, 4, 1, 2).reshape(b * h * w, c, 1, geo_volume2.shape[2])
        corr = corr.reshape(b * h * w, 1, 1, corr.shape[-1])
        self.geo_pyramid, self.corr_pyramid = [geo], [corr]
        for _ in range(num_levels - 1):
            geo = F.avg_pool2d(geo, [1, 2], stride=[1, 2])
            self.geo_pyramid.append(geo)
            corr = F.avg_pool2d(corr, [1, 2], stride=[1, 2])
            self.corr_pyramid.append(corr)

    def __call__(self, disp, coords):
        r = self.radius
        b, _, h, w = disp.shape
        dx = torch.linspace(-r, r, 2 * r + 1).view(1, 1, 2 * r + 1, 1).to(disp.device)
        d = disp.reshape(b * h * w, 1, 1, 1)
        feat1 = _sample_rows(self.vol1, dx + d / 2).view(b, h, w, -1)
        feat2 = _sample_rows(self.vol2, dx + d / 4).view(b, h, w, -1)
        feat0, corr = [], []
        for lvl in range(self.num_levels):
            feat0.append(_sample_rows(self.geo_pyramid[lvl], dx + d / 2 ** lvl).view(b, h, w, -1))
            x = coords.reshape(b * h * w, 1, 1, 1) / 2 ** lvl - d / 2 ** lvl + dx
            corr.append(_sample_rows(self.corr_pyramid[lvl], x).view(b, h, w, -1))

        def nchw(t):
            return t.permute(0, 3, 1, 2).contiguous().float()
        return nchw(torch.cat(feat0, dim=-1)), nchw(feat1), nchw(feat2), nchw(torch.cat(corr, dim=-1))


def load_reference(dotted):
    """Import a module of the reference's igevpp package (a directory without __init__.py)."""
    return shim.load(dotted)


def igevpp(yaml=UNIFORM_YAML, seed=7):
    """The reference's IGEVPPStereo, eval mode, built from `yaml` unchanged, with seeded weights (classifier sharpened)."""
    shim.install_timm_stub()
    cfg = shim.load_cfg(yaml).MODEL
    m = load_reference("stereo.modeling.models.igevpp.igevpp_stereo").IGEVPPStereo(cfg).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=seed, scale=IGEVPP_SCALE))
    return m
