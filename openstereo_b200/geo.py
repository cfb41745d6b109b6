"""Host-side mirrors of the reference's geometry-encoding volumes (SURVEY.md section 8(f) row 1).

``CombinedGeoEncodingVolume(init_fmap1, init_fmap2, geo_volume, num_levels=2, radius=4)`` and ``obj(disp, coords)`` have
the reference's signature and return value (stereo/modeling/models/stereobase/gru_blocks.py:169-229;
``Combined_Geo_Encoding_Volume`` stereo/modeling/models/igev/geometry.py:7-66 is the same class under IGEV's name).  What
differs is the data layout: the geometry volume stays (B, C, D, H, W) -- no (B*H*W, C, 1, D) permuted copy -- the pyramid
is built by the pair-average kernel, and one gather kernel per GRU iteration writes the (B, L*(C+1)*(2r+1), H, W) feature
map directly instead of grid tensors + 2L grid_sample calls + cat + permute.  CUDA only: there is no CPU fallback.

``GeoEncodingVolume(geo_volume, num_levels=2, radius=4)`` and ``obj(disp)`` are IGEV-RT's geometry-only variant
(``Geo_Encoding_Volume`` stereo/modeling/models/igev_rt/geometry.py:6-33): the same pyramid and taps without the correlation
rows, (B, L*C*(2r+1), H, W).

``MultiRangeGeoEncodingVolume(geo_volume0, geo_volume1, geo_volume2, init_fmap1, init_fmap2, radius=4, num_levels=2)`` and
``obj(disp, coords)`` are IGEV++'s multi-range variant (``Combined_Geo_Encoding_Volume`` stereo/modeling/models/igevpp/geometry.py:
6-87): the geo_volume0 pyramid, two single-level volumes sampled at disp / 2 and disp / 4, and the correlation rows, returned as
the reference's four tensors from one launch.
"""
import torch

from . import ops


class CombinedGeoEncodingVolume:
    def __init__(self, init_fmap1, init_fmap2, geo_volume, num_levels=2, radius=4):
        if not (geo_volume.is_cuda and init_fmap1.is_cuda and init_fmap2.is_cuda):
            raise RuntimeError("CombinedGeoEncodingVolume: CUDA tensors required (the reference class serves CPU tensors)")
        self.num_levels, self.radius = int(num_levels), int(radius)
        self.geo_volume_pyramid = _volume_pyramid(geo_volume, self.num_levels)
        # MonSter builds the volume inside its AMP YAML's bf16 autocast, where einsum would return bf16: the lookup reads fp32
        with torch.autocast("cuda", enabled=False):
            self.init_corr_pyramid = self.corr_pyramid(init_fmap1, init_fmap2, self.num_levels)

    def __call__(self, disp, coords):
        return ops.geo_lookup(self.geo_volume_pyramid, self.init_corr_pyramid, disp, coords, self.radius)

    @staticmethod
    def corr(fmap1, fmap2):
        """All-pairs row correlation (gru_blocks.py:222-229): a batched fp32 GEMM, left to cuBLAS."""
        b, _, h, w1 = fmap1.shape
        w2 = fmap2.shape[-1]
        corr = torch.einsum('aijk,aijh->ajkh', fmap1, fmap2)
        return corr.reshape(b, h, w1, 1, w2).contiguous()

    @classmethod
    def corr_pyramid(cls, fmap1, fmap2, num_levels):
        """[(B, H, W1, W2 >> i)]: the all-pairs correlation and its pair-averaged levels along the right-image column."""
        corr = cls.corr(fmap1.float(), fmap2.float())                             # (B, H, W1, 1, W2)
        b, h, w1, _, w2 = corr.shape
        pyramid = [corr.reshape(b, h, w1, w2)]
        for _ in range(num_levels - 1):
            pyramid.append(ops.avgpool_pairs(pyramid[-1], 3))
        return pyramid


def _volume_pyramid(volume, num_levels):
    """[(B, C, D >> i, H, W)]: the volume in its native layout and its pair-averaged levels along the disparity axis."""
    pyramid = [volume.float().contiguous()]
    for _ in range(num_levels - 1):
        pyramid.append(ops.avgpool_pairs(pyramid[-1], 2))
    return pyramid


class GeoEncodingVolume:
    def __init__(self, geo_volume, num_levels=2, radius=4):
        if not geo_volume.is_cuda:
            raise RuntimeError("GeoEncodingVolume: CUDA tensors required (the reference class serves CPU tensors)")
        self.num_levels, self.radius = int(num_levels), int(radius)
        self.geo_volume_pyramid = _volume_pyramid(geo_volume, self.num_levels)

    def __call__(self, disp):
        return ops.geo_volume_lookup(self.geo_volume_pyramid, disp, self.radius)


class MultiRangeGeoEncodingVolume:
    """IGEV++'s Combined_Geo_Encoding_Volume (igevpp/geometry.py:6-87): the pyramid of geo_volume0, geo_volume1 and geo_volume2 as
    they are (each with its own plane count) and the correlation pyramid; obj(disp, coords) -> (geo_feat0, geo_feat1, geo_feat2,
    init_corr) from one launch.  Note the reference's argument order: radius before num_levels."""

    def __init__(self, geo_volume0, geo_volume1, geo_volume2, init_fmap1, init_fmap2, radius=4, num_levels=2):
        if not all(t.is_cuda for t in (geo_volume0, geo_volume1, geo_volume2, init_fmap1, init_fmap2)):
            raise RuntimeError("MultiRangeGeoEncodingVolume: CUDA tensors required (the reference class serves CPU tensors)")
        self.num_levels, self.radius = int(num_levels), int(radius)
        self.geo_volume0_pyramid = _volume_pyramid(geo_volume0, self.num_levels)
        self.geo_volume1 = geo_volume1.float().contiguous()
        self.geo_volume2 = geo_volume2.float().contiguous()
        self.init_corr_pyramid = CombinedGeoEncodingVolume.corr_pyramid(init_fmap1, init_fmap2, self.num_levels)

    def __call__(self, disp, coords):
        return ops.geo_multirange_lookup(self.geo_volume0_pyramid, self.geo_volume1, self.geo_volume2, self.init_corr_pyramid, disp,
                                         coords, self.radius)


Combined_Geo_Encoding_Volume = CombinedGeoEncodingVolume          # IGEV's spelling (igev/geometry.py:7)
Geo_Encoding_Volume = GeoEncodingVolume                           # IGEV-RT's spelling (igev_rt/geometry.py:6)
context_upsample = ops.context_upsample
