"""Oracle: IGEV-RT's geometry-only encoding volume (TEST INFRASTRUCTURE -- see oracle/__init__.py).

* ``GeoEncodingVolume``  restates ``Geo_Encoding_Volume`` stereo/modeling/models/igev_rt/geometry.py:6-33 (+ ``bilinear_sampler``
  igev_rt/utils.py): the combined lookup of oracle/geo_lookup.py without the all-pairs correlation rows -- a pair-averaged pyramid
  of the geometry volume along the disparity axis, and per GRU iteration 2r+1 bilinear taps per level at dx + disp / 2^i.
* ``igev_rt(yaml, seed)``  the reference's own IGEVRTtereo built from an unchanged YAML with the timm stand-in and seeded weights.

Same aten calls in the same order as the reference, so the lookup is bit-equal on CPU (asserted by tools/make_golden.py).
"""
import torch
import torch.nn.functional as F

from oracle import _reference_shim as shim
from oracle import seeded_init as si
from oracle.geo_lookup import _sample_rows

UNIFORM_YAML = "cfgs/igev_rt/igev_rt_sceneflow_uniform.yaml"
AMP_YAML = "cfgs/igev_rt/igev_rt_sceneflow_amp.yaml"
# Un-sharpened classifier logits are nearly flat, so the initial disparity would sit at the middle of the range everywhere; this
# factor spreads them over a few units, as tests/test_patch_gpu.py's _igev() does for IGEVStereo.
IGEV_RT_SCALE = {"classifier.weight": 8.0}


class GeoEncodingVolume:
    def __init__(self, geo_volume, num_levels=2, radius=4):
        self.num_levels, self.radius = num_levels, radius
        b, c, d, h, w = geo_volume.shape
        geo = geo_volume.permute(0, 3, 4, 1, 2).reshape(b * h * w, c, 1, d)
        self.geo_pyramid = [geo]
        for _ in range(num_levels - 1):
            geo = F.avg_pool2d(geo, [1, 2], stride=[1, 2])
            self.geo_pyramid.append(geo)

    def __call__(self, disp):
        r = self.radius
        b, _, h, w = disp.shape
        dx = torch.linspace(-r, r, 2 * r + 1).view(1, 1, 2 * r + 1, 1).to(disp.device)
        feats = []
        for lvl in range(self.num_levels):
            x = dx + disp.reshape(b * h * w, 1, 1, 1) / 2 ** lvl
            feats.append(_sample_rows(self.geo_pyramid[lvl], x).view(b, h, w, -1))
        return torch.cat(feats, dim=-1).permute(0, 3, 1, 2).contiguous().float()


def load_reference(dotted):
    """Import a module of the reference's igev_rt package (a directory without __init__.py)."""
    return shim.load(dotted)


def igev_rt(yaml=UNIFORM_YAML, seed=7):
    """The reference's IGEVRTtereo, eval mode, built from `yaml` unchanged, with seeded weights (classifier sharpened)."""
    shim.install_timm_stub()
    cfg = shim.load_cfg(yaml).MODEL
    m = load_reference("stereo.modeling.models.igev_rt.igev_rt_stereo").IGEVRTtereo(cfg).eval()
    m.load_state_dict(si.seeded_state_dict(m.state_dict(), seed=seed, scale=IGEV_RT_SCALE))
    return m
