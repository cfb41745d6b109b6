"""GPU: contract of every kernel that is not a convolution -- cost volumes, regression tails, lookups and backward passes
(csrc/volume.cu, softargmin.cu, backward.cu, geo.cu, cascade.cu, coex.cu, flavours.cu and the layout pass of conv3d_tc.cu).

REGISTRY has one or more rows per instantiation (tests/test_host_logic_cpu.py checks that every __global__ instantiation those
files can launch has a row).  Each row names the family, the instantiation it must reach in the template spelling of the source
and a small shape with partial tiles, chunks and units in every tiled dimension.  For every row:
  routing      torch.profiler sees exactly one kernel of this library, the row's instantiation; volume runs also assert
               osb_volume_last_variant(), which names the vector-epilogue and the TMA-or-plain-load staging choices;
  accuracy     an fp64 reference of the whole operation from the same fp32 inputs.  Features, cascade features and the gradient
               weights of the backward kernels are scaled per correlation group or channel by 2^k (k over [-12, 12]) times a
               non-power-of-two factor.  Three kinds of bar, none over the whole tensor:
                 products and sums   error <= 1e-5 x the output channel's max of the fp64 magnitude sum |terms| (cancellation
                                     can make |want| small while the fp32 rounding stays proportional to sum |terms|); the geo,
                                     context and regression-values taps use each element's own sum |terms|, which is stricter;
                 copies and gathers  bit-exact: the concat volume and the concat halves of the fused volume, the left copies of
                                     the warped volumes, nearest_resize3d, avgpool_pairs, the layout pass with its zero
                                     channels, and the exact zeros of every masked triangle;
                 soft-argmin family  per pixel, see soft_model();
  bounds       the output region starts as NaN between 4 KB sentinel guards: every element is written and no sentinel changes;
               a backward launch with one gradient pointer null leaves that gradient's region unwritten;
  store paths  where a kernel picks its loads and stores by alignment (the volume's vec_ok and use_tma, context_upsample's
               vector branch) the row runs aligned and with pointers moved 4 bytes: bit-identical, and each run passes the bar;
  item loop    volume rows run at persistent-grid caps 1, 5 and uncapped, bit-identical; the grid-stride rows of avgpool_pairs
               and nearest_resize3d have totals above their SM-count-based grid caps;
  determinism  two launches are bit-identical, except epe_partial_kernel, whose float atomics add block partial sums in
               arrival order: its error sum gets the bar of the sum instead (its counts are integers and stay exact).
test_volume_item_order_0: the other work-item order, read once per process, in a child process, bit-identical to order 1.
test_volume_input_types: fp16 / bf16 inputs through ops.*: output in the input type, equal to the rounded fp32 result.
test_refusals: every input an entry point refuses returns OSB_EINVAL and launches nothing.
"""
import math
import os
import re
import subprocess
import sys
import zlib
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OSB_EINVAL = 1
GUARD = 1024                            # sentinel floats on each side of an output region (4 KB, keeps 16-byte alignment)
SENTINEL = -1234.5
TOL = 1e-5                              # products and sums: error / (channel max of sum |terms|)
TOL_SOFT = 4.0                          # soft-argmin family: error / soft_model()
U = 2.0 ** -24                          # unit roundoff of fp32
F64 = torch.float64

Row = namedtuple("Row", "id fam variant shape opts")


def R(rid, fam, variant, shape, **opts):
    return Row(rid, fam, variant, shape, opts)


def V(vec, k4):
    return "volume_kernel<%s,%s>" % ("true" if vec else "false", "true" if k4 else "false")


# vol shapes: gwc / sum / corr (B, G, K, H, W, D); cat (B, C, H, W, D); fused (B, G, K, Cc, H, W, D).  A work item is one row,
# 128 columns, 64 disparities and GU = min(G, 8) groups, halved while GU * K > 128.
REGISTRY = [
    R("vol-gwc-k1", "vol", V(1, 0), (1, 8, 1, 3, 128, 65), entry="gwc"),                 # D = 65: a second chunk of one plane
    R("vol-gwc-k3-w5", "vol", V(0, 0), (2, 5, 3, 3, 5, 3), entry="gwc"),
    R("vol-gwc-k4-w5", "vol", V(0, 1), (1, 3, 4, 2, 5, 3), entry="gwc"),
    R("vol-gwc-k12-w260", "vol", V(1, 1), (1, 6, 12, 2, 260, 64), entry="gwc"),           # three column tiles, the last partial
    R("vol-gwc-k40-w129", "vol", V(0, 1), (1, 5, 40, 2, 129, 65), entry="gwc"),           # GU = 2: last unit holds one group
    R("vol-gwc-k40-b2", "vol", V(1, 1), (2, 3, 40, 2, 132, 70), entry="gwc"),             # last unit's TMA box reads image b+1
    R("vol-gwc-k144", "vol", V(1, 1), (1, 2, 144, 2, 128, 33), entry="gwc"),              # largest K: GU = 1, 221 KB ring
    R("vol-gwc-g11-b2", "vol", V(1, 1), (2, 11, 4, 3, 68, 20), entry="gwc"),              # G % GU = 3
    R("vol-gwc-d-gt-w", "vol", V(1, 1), (1, 4, 8, 2, 20, 40), entry="gwc"),               # planes d >= W are all zero
    R("vol-sum-k12", "vol", V(1, 1), (2, 3, 12, 2, 64, 29), entry="sum"),
    R("vol-sum-k3", "vol", V(1, 0), (1, 4, 3, 2, 36, 9), entry="sum"),
    R("vol-corr-k7", "vol", V(1, 0), (2, 1, 7, 3, 132, 65), entry="corr"),
    R("vol-cat-masked", "vol", V(0, 1), (2, 11, 2, 129, 65), entry="cat", mask=1),
    R("vol-cat-unmasked", "vol", V(1, 1), (2, 6, 2, 128, 64), entry="cat", mask=0),
    R("vol-cat-d-gt-w", "vol", V(1, 1), (1, 5, 2, 12, 20), entry="cat", mask=1),
    R("vol-fused-k4", "vol", V(1, 1), (2, 10, 4, 6, 2, 128, 65), entry="fused"),
    R("vol-fused-k3", "vol", V(1, 0), (1, 5, 3, 5, 2, 132, 48), entry="fused"),
    R("vol-fused-k3-w129", "vol", V(0, 0), (1, 5, 3, 4, 2, 129, 20), entry="fused"),
    # softargmin.cu softargmin_kernel (B, D, H, W): 8-bin chunks; 185 pixels per image, not a multiple of the 256-thread block
    R("sa-d1", "sa", "softargmin_kernel", (2, 1, 5, 37)),
    R("sa-d7-alpha-1", "sa", "softargmin_kernel", (2, 7, 5, 37), alpha=-1.0),
    R("sa-d8-interval", "sa", "softargmin_kernel", (2, 8, 5, 37), start=-3.5, step=0.75),
    R("sa-d9-last", "sa", "softargmin_kernel", (2, 9, 5, 37), peak_last=1),              # arg-max in the last, one-bin chunk
    R("sa-d9-inf", "sa", "softargmin_kernel", (2, 9, 5, 37), inf=1),
    R("sa-d192-spread", "sa", "softargmin_kernel", (1, 192, 5, 37), spread=60.0, offset=1e4),
    R("sa-d193-last", "sa", "softargmin_kernel", (1, 193, 5, 37), peak_last=1, alpha=0.5, start=1.0, step=0.5),
    R("sa-d193-inf", "sa", "softargmin_kernel", (1, 193, 3, 37), inf=1, spread=60.0),
    R("sa-d9-raw", "sa", "softargmin_kernel", (2, 9, 5, 37), norm=0),
    R("sa-d192-raw", "sa", "softargmin_kernel", (1, 192, 5, 37), norm=0, alpha=-1.0, start=2.0, step=0.5),
    # upsample_softargmin_kernel (B, Dl, Hl, Wl, D, H, W): 128-column tiles; shared tables of D + Dl + 1 words (48 KB)
    R("up-x4", "up", "upsample_softargmin_kernel<false>", (2, 12, 5, 40, 48, 20, 160), align=0),
    R("up-x4-align", "up", "upsample_softargmin_kernel<false>", (2, 12, 5, 40, 48, 20, 160), align=1),
    R("up-ratio", "up", "upsample_softargmin_kernel<false>", (1, 10, 5, 33, 37, 17, 130), align=0),
    R("up-ratio-align", "up", "upsample_softargmin_kernel<false>", (1, 10, 5, 33, 37, 17, 130), align=1),
    R("up-spread", "up", "upsample_softargmin_kernel<false>", (1, 12, 3, 10, 48, 12, 40), align=0, spread=60.0, offset=1e4),
    R("up-ones", "up", "upsample_softargmin_kernel<false>", (2, 1, 1, 1, 7, 3, 5), align=0),
    R("up-h1-align", "up", "upsample_softargmin_kernel<false>", (1, 3, 2, 4, 9, 1, 13), align=1),
    R("up-dmax", "up", "upsample_softargmin_kernel<false>", (1, 4, 2, 3, 12283, 2, 3), align=0),   # D + Dl + 1 = 12288 words
    R("upv-x4", "up", "upsample_softargmin_kernel<true>", (2, 12, 5, 40, 48, 20, 160), align=0, values=1),
    R("upv-ratio-align", "up", "upsample_softargmin_kernel<true>", (1, 10, 5, 33, 37, 17, 130), align=1, values=1),
    R("epe", "epe", "epe_partial_kernel", (3, 50001), maxdisp=192.0),
    # backward.cu (B, G, K, H, W, D) / (B, C, H, W, D) / (B, D, H, W): 128-column blocks
    R("bwd-gwc-mean", "bgwc", "gwc_volume_bwd_kernel", (2, 3, 4, 3, 133, 40), reduce_sum=0),
    R("bwd-gwc-sum", "bgwc", "gwc_volume_bwd_kernel", (1, 5, 2, 2, 37, 45), reduce_sum=1),     # D > W
    R("bwd-cat-masked", "bcat", "concat_volume_bwd_kernel", (2, 5, 3, 133, 40), mask=1),
    R("bwd-cat-unmasked", "bcat", "concat_volume_bwd_kernel", (1, 4, 2, 37, 45), mask=0),
    R("bwd-sa", "bsa", "softargmin_bwd_kernel", (2, 24, 5, 37)),
    R("bwd-sa-interval", "bsa", "softargmin_bwd_kernel", (2, 13, 5, 37), alpha=-0.7, start=2.0, step=0.5),
    R("bwd-sa-raw", "bsa", "softargmin_bwd_kernel", (1, 13, 5, 37), norm=0, alpha=1.3, start=-1.0, step=0.25),
    # geo.cu geo_lookup (B, C, D, H, W, W2, levels): output (B, L * (C + 1) * (2r + 1), H, W), 128-column blocks
    R("geo-r4-l4", "geo", "geo_lookup_kernel<4>", (2, 3, 48, 3, 130, 136, 4), radius=4, cross=1),
    R("geo-r4-l1", "geo", "geo_lookup_kernel<4>", (1, 2, 8, 2, 21, 20, 1), radius=4),
    R("geo-r0-l2", "geo", "geo_lookup_kernel<0>", (1, 3, 16, 2, 40, 44, 2), radius=0),
    R("geo-r1-l3", "geo", "geo_lookup_kernel<0>", (2, 2, 24, 2, 33, 30, 3), radius=1),
    R("geo-r3-l4", "geo", "geo_lookup_kernel<0>", (1, 2, 32, 3, 131, 140, 4), radius=3),
    R("pool-small", "pool", "avgpool_pairs_kernel", (3, 7, 35)),                         # odd n: the last element is dropped
    R("pool-multipass", "pool", "avgpool_pairs_kernel", (3, 11, 0)),                     # inner from the SM count: > 2 grid passes
    # context_upsample (B, h, w, s): one thread per 4 output columns, 512 columns per block
    R("ctx-s1", "ctx", "context_upsample_kernel", (2, 5, 12, 1)),
    R("ctx-s2", "ctx", "context_upsample_kernel", (2, 4, 10, 2)),
    R("ctx-s3", "ctx", "context_upsample_kernel", (1, 3, 12, 3)),
    R("ctx-s3-odd", "ctx", "context_upsample_kernel", (1, 3, 11, 3)),
    R("ctx-s4", "ctx", "context_upsample_kernel", (2, 3, 40, 4)),
    R("ctx-s8", "ctx", "context_upsample_kernel", (1, 2, 70, 8)),                         # 560 columns: two blocks
    # cascade.cu warped volumes (B, Cg, G, Cc, D, H, W): one CTA per (image row, unit).  It stages one right row per channel
    # where the row coordinate round trip returns the integer (every row at H = 5), two where it does not (some rows at H = 6, 7, 10)
    R("cas-cat-h5", "cas", "warped_volume_kernel<8>", (2, 0, 0, 11, 5, 5, 37), mask=0, two=0),
    R("cas-cat-h6-mask", "cas", "warped_volume_kernel<8>", (1, 0, 0, 8, 4, 6, 40), mask=1, two=1),
    R("cas-gwc-k8", "cas", "warped_volume_kernel<8>", (2, 16, 2, 5, 4, 10, 40), two=1),
    R("cas-gwc-k9", "cas", "warped_volume_kernel<16>", (1, 27, 3, 3, 5, 5, 36), two=0),
    R("cas-gwc-k16", "cas", "warped_volume_kernel<16>", (1, 32, 2, 10, 3, 7, 33), two=1),
    R("cas-gwc-wmax", "cas", "warped_volume_kernel<16>", (1, 16, 1, 1, 2, 2, 1816)),     # 16 x 2 rows x 1816 floats = 227 KB
    R("cas-cat-wmax", "cas", "warped_volume_kernel<8>", (1, 0, 0, 1, 2, 2, 3632), mask=1),
    # coex.cu regression (B, D, h, w): tiles of 16 x 32 low-resolution pixels
    R("coex-k2", "coex", "coex_regression_kernel<2>", (2, 2, 5, 9), k=2, logits=1),
    R("coex-k3", "coex", "coex_regression_kernel<3>", (1, 3, 17, 33), k=3, logits=1, ties=1),
    R("coex-k4", "coex", "coex_regression_kernel<4>", (2, 4, 5, 9), k=4, logits=0),
    R("coex-k5", "coex", "coex_regression_kernel<5>", (1, 5, 17, 33), k=5, logits=0, ties=1),
    R("coex-k6", "coex", "coex_regression_kernel<6>", (2, 6, 5, 9), k=6, logits=1, ties=1),
    R("coex-k7", "coex", "coex_regression_kernel<7>", (1, 7, 6, 35), k=7, logits=1),
    R("coex-k8", "coex", "coex_regression_kernel<8>", (2, 8, 5, 9), k=8, logits=0),
    R("coex-k4-d24-ties", "coex", "coex_regression_kernel<4>", (2, 24, 17, 33), k=4, logits=1, ties=1),
    R("coex-k2-d48", "coex", "coex_regression_kernel<2>", (1, 48, 6, 35), k=2, logits=0, ties=1),
    # nearest_resize3d (N, Di, Hi, Wi, Do, Ho, Wo): equal, doubled and general ratios; N = 0 takes N from the SM count
    R("near-mixed", "near", "nearest_resize3d_kernel", (3, 4, 5, 9, 4, 10, 13)),
    R("near-down", "near", "nearest_resize3d_kernel", (2, 9, 7, 10, 4, 7, 20)),
    R("near-multipass", "near", "nearest_resize3d_kernel", (0, 5, 6, 12, 10, 13, 25)),
    # flavours.cu
    R("l2n-k8", "l2n", "group_l2_normalize_kernel", (2, 3, 8, 5, 37)),
    R("l2n-k1", "l2n", "group_l2_normalize_kernel", (1, 4, 1, 3, 21)),
    R("sub-d21-w13", "sub", "sub_volume_kernel", (2, 7, 3, 13, 21)),                     # D % 8 != 0, D > W
    R("sub-w140", "sub", "sub_volume_kernel", (1, 5, 2, 140, 16)),
    R("rv", "rv", "regression_values_kernel", (2, 19, 5, 37)),
    # conv3d_tc.cu layout pass (B, C, Cpad, D, H, W): 32 x 32 transpose tiles
    R("pad-24-32", "pad", "ncdhw_to_ndhwc_kernel", (2, 24, 32, 3, 5, 7)),
    R("pad-40", "pad", "ncdhw_to_ndhwc_kernel", (1, 40, 40, 2, 3, 11)),
    R("pad-48-64", "pad", "ncdhw_to_ndhwc_kernel", (1, 48, 64, 2, 5, 9)),
]
BY_ID = {r.id: r for r in REGISTRY}


@pytest.fixture(scope="module")
def osb():
    import __graft_entry__
    __graft_entry__.build()
    from openstereo_b200 import _lib, ops
    return _lib, ops


@pytest.fixture
def grid_cap(osb):
    _, ops = osb
    yield ops.set_persistent_grid_cap
    ops.set_persistent_grid_cap(0)


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


def scales(n, g, lo=-12, hi=12):
    """2^k x a non-power-of-two factor per channel, k spread over [lo, hi]."""
    k = torch.linspace(lo, hi, n).round()[torch.randperm(n, generator=g)]
    return torch.ldexp(torch.ones(n), k.int()) * (1.0 + 0.9 * torch.rand(n, generator=g)) * 0.77


def per(t, s, dim):
    shape = [1] * t.dim()
    shape[dim] = -1
    return t * s.view(shape)


def chanmax(mag, *keep):
    """Max of `mag` over every dim but `keep`, broadcastable to mag."""
    dims = [d for d in range(mag.dim()) if d not in keep]
    return mag.amax(dim=dims, keepdim=True) if dims else mag


def f32(x):
    return torch.as_tensor(x, dtype=torch.float32)


def soft_model(p, x, v, out, lam, S, dim=1):
    """Per-pixel error model of the soft-argmin family, out = sum_j p_j v_j with p = softmax(x) over `dim`:
        E = gamma_D sum_j p_j |v_j| + sum_j p_j |v_j - out| eps_j,   eps_j = 2^-24 (|x_j - m| + lam_j (8 + 2 S) + 8),
    gamma_D = D 2^-24 covering the fp32 sums over D bins, eps_j the relative error of p_j: the exponential of a rounded argument
    x_j - m (|x_j - m| ulps), the rounding of the logit itself (lam_j = sum |terms| of x_j: the logit for the plain kernel, the
    trilinear interpolation of |cost| for the up-sampling tails, up to 8 roundings each) and, where the logit is interpolated,
    the fp32 source coordinate (one ulp of coordinates up to S moves the weight of neighbours up to 2 lam_j apart).  A term
    2^-100 (max |v| + 1) covers exponentials that underflow in fp32.  The bar is TOL_SOFT x E."""
    m = x.amax(dim=dim, keepdim=True)
    live = p > 0
    dx = torch.where(live, (x - m).abs(), torch.zeros_like(x))
    lam = torch.where(live, lam, torch.zeros_like(lam))
    eps = U * (dx + lam * (8 + 2 * S) + 8)
    D = x.shape[dim]
    E = D * U * (p * v.abs()).sum(dim) + (p * (v - out.unsqueeze(dim)).abs() * eps).sum(dim)
    return E + 2.0 ** -100 * (v.abs().amax(dim) + 1)


def axis(n_in, n_out, align):
    """aten's linear source index in fp32 (softargmin.cu Axis::locate): (i0, i1, lambda)."""
    dst = torch.arange(n_out, dtype=torch.float32)
    if align:
        scale = f32(n_in - 1) / f32(n_out - 1) if n_out > 1 else f32(0.0)
        src = scale * dst
    else:
        scale = f32(n_in) / f32(n_out)
        src = torch.clamp(scale * (dst + 0.5) - 0.5, min=0.0)
    i0 = torch.clamp(src.long(), max=n_in - 1)
    i1 = i0 + (i0 < n_in - 1).long()
    return i0, i1, (src - i0.float()).double()


def lerp(t, dim, ax):
    i0, i1, lam = ax
    shape = [1] * t.dim()
    shape[dim] = -1
    lam = lam.view(shape)
    return t.index_select(dim, i0) * (1 - lam) + t.index_select(dim, i1) * lam


def trilinear(cost, axes):
    for dim, ax in zip((1, 2, 3), axes):
        cost = lerp(cost, dim, ax)
    return cost


def roundtrip_geo(x, n):
    """geo.cu roundtrip: x -> 2x/(n-1) - 1 -> (g + 1) * (0.5 (n - 1)), every step rounded to fp32."""
    g = (f32(2.0) * x) / f32(n - 1) - f32(1.0)
    return (g + f32(1.0)) * (f32(0.5) * f32(n - 1))


def roundtrip_cas(v, half):
    """cascade.cu cas_roundtrip: grid value v/half - 1 and aten's unnormalisation (g + 1) * half, in fp32."""
    g = v / half - f32(1.0)
    return (g + f32(1.0)) * half


class Case:
    """One launch of a row.  `want` is the fp64 reference in the output layout; `scale` (broadcastable to want) the magnitude the
    error is measured against, with bar `tol`; `exact` marks elements that must equal want bit for bit; `skip` marks elements the
    launch must leave unwritten.  fn(y, P) calls the C entry point with output address y; P(name) is the device address of input
    `name`, moved 4 bytes when the run shifts it."""

    def __init__(self, name, want, scale, fn, inputs, tol=TOL, exact=None, skip=None, det_scale=None, info=None):
        self.name, self.want, self.scale, self.fn, self.inputs, self.tol = name, want, scale, fn, inputs, tol
        self.exact = torch.zeros(want.shape, dtype=torch.bool) if exact is None else exact.expand(want.shape)
        self.skip = torch.zeros(want.shape, dtype=torch.bool) if skip is None else skip
        self.det_scale = det_scale              # None: repeated launches must be bit-identical
        self.info = info or {}
        self.numel = want.numel()
        self._dev = None

    def dev(self):
        if self._dev is None:
            self._dev = {k: v.contiguous().cuda() for k, v in self.inputs.items()}
        return self._dev

    def guarded(self, y_off=0):
        buf = torch.full((GUARD + y_off + self.numel + GUARD,), SENTINEL, device="cuda")
        buf[GUARD + y_off:GUARD + y_off + self.numel] = float("nan")
        return buf

    def launch(self, y_off=0, shift=()):
        """-> (guarded buffer, index of the output region's first element in it)."""
        dev, keep = self.dev(), []

        def P(name):
            t = dev[name]
            if name not in shift:
                return t.data_ptr()
            buf = torch.empty(t.numel() + 1, device="cuda")
            buf[1:].copy_(t.flatten())
            keep.append(buf)
            return buf.data_ptr() + 4

        buf, lead = self.guarded(y_off), GUARD + y_off
        self.fn(buf.data_ptr() + 4 * lead, P)
        torch.cuda.synchronize()
        return buf, lead

    def check(self, buf, lead, what):
        """Bounds, unwritten and exact elements, the bar; -> worst error / scale over the barred elements (inner on the CPU)."""
        bits = buf.view(torch.int32).cpu()
        sent = torch.tensor([SENTINEL]).view(torch.int32).item()
        assert (bits[:lead] == sent).all() and (bits[lead + self.numel:] == sent).all(), "%s: a store left the output region" % what
        got = buf[lead:lead + self.numel].cpu().view(self.want.shape)
        nan = torch.isnan(got)
        assert nan[self.skip].all(), "%s: %d elements of a gradient that was not asked for were written" % (
            what, int((~nan[self.skip]).sum()))
        live = ~self.skip
        assert not nan[live].any(), "%s: %d output elements never written" % (what, int(nan[live].sum()))
        ex = self.exact & live
        if ex.any():
            bad = got[ex].view(torch.int32) != self.want[ex].float().view(torch.int32)
            assert not bad.any(), "%s: %d elements that must be exact differ (first got %s want %s)" % (
                what, int(bad.sum()), got[ex][bad][:4].tolist(), self.want[ex][bad][:4].tolist())
        m = live & ~self.exact
        if not m.any():
            return 0.0
        err = (got.double() - self.want).abs()[m]
        sc = self.scale.expand(self.want.shape)[m]
        ratio = torch.where(sc > 0, err / sc.clamp(min=1e-300), torch.where(err > 0, math.inf, 0.0))
        worst = float(ratio.max())
        if worst > self.tol:
            i = int(ratio.argmax())
            raise AssertionError("%s: error %.3e = %.3e x the bar's scale %.3e (allowed %g); got %r want %r; %d elements over" % (
                what, float(err[i]), worst, float(sc[i]), self.tol, float(got[m][i]), float(self.want[m][i]),
                int((ratio > self.tol).sum())))
        return worst


# ------------------------------------------------------------------------------------------------------------- references
def gwc_ref(ref, tgt, G, D, s):
    """vol[b,g,d,h,w] = s sum_k ref[b,gK+k,h,w] tgt[b,gK+k,h,w-d] (w >= d, else 0); -> (vol, sum |terms|)."""
    B, C, H, W = ref.shape
    K = C // G
    r, t = ref.double(), tgt.double()
    vol, mag = torch.zeros(B, G, D, H, W, dtype=F64), torch.zeros(B, G, D, H, W, dtype=F64)
    for d in range(min(D, W)):
        p = (r[..., d:] * t[..., :W - d]).view(B, G, K, H, W - d)
        vol[:, :, d, :, d:] = p.sum(2) * s
        mag[:, :, d, :, d:] = p.abs().sum(2) * s
    return vol, mag


def tri(D, W):
    """(D, W) mask of the w < d triangle."""
    return torch.arange(W).view(1, W) < torch.arange(D).view(D, 1)


def cat_ref(ref, tgt, D, mask):
    B, C, H, W = ref.shape
    t = tri(D, W).view(1, 1, D, 1, W)
    left = ref.double().unsqueeze(2).expand(B, C, D, H, W).clone()
    if mask:
        left = left.masked_fill(t, 0.0)
    right = torch.zeros(B, C, D, H, W, dtype=F64)
    for d in range(min(D, W)):
        right[:, :, d, :, d:] = tgt[..., :W - d].double()
    return torch.cat([left, right], 1)


def volume_variant(K, W, shift=(), y_off=0, gwc=True):
    vec = W % 4 == 0 and y_off == 0 and not {"ref", "rc"} & set(shift)
    tma = gwc and W % 4 == 0 and "tgt" not in shift
    return "volume<%d,%d,%s>" % (vec, K % 4 == 0, "tma" if tma else "ldg")


def disp_mixture(g, shape, lo, hi):
    """Hypotheses: uniform in [lo, hi] (negative and beyond the far edge), exact integers and half-integers."""
    u = lo + (hi - lo) * torch.rand(shape, generator=g)
    pick = torch.rand(shape, generator=g)
    u = torch.where(pick < 0.3, u.round(), u)
    return torch.where((pick >= 0.3) & (pick < 0.45), u.floor() + 0.5, u)


def cases(osb, row, g):
    lib, ops = osb
    call = lambda *a: lib.call(*a)                                # noqa: E731
    s = lambda: torch.cuda.current_stream().cuda_stream          # noqa: E731
    o, fam = row.opts, row.fam
    rn = lambda *shape: torch.randn(*shape, generator=g)         # noqa: E731

    if fam == "vol":
        e = o["entry"]
        if e == "cat":
            B, C, H, W, D = row.shape
            G = K = Cg = 0
            Cc = C
        elif e == "fused":
            B, G, K, Cc, H, W, D = row.shape
            Cg = G * K
        else:
            B, G, K, H, W, D = row.shape
            Cg, Cc = G * K, 0
        inputs, parts, mags, exact = {}, [], [], []
        if Cg:
            ref = rn(B, G, K, H, W) * scales(G, g).view(1, G, 1, 1, 1)                 # per correlation group
            tgt = per(rn(B, Cg, H, W), 1.0 + 0.5 * torch.rand(Cg, generator=g), 1)
            ref = ref.reshape(B, Cg, H, W)
            vol, mag = gwc_ref(ref, tgt, G, D, 1.0 if e == "sum" else 1.0 / K)
            parts.append(vol), mags.append(chanmax(mag, 1)), exact.append(tri(D, W).view(1, 1, D, 1, W).expand(vol.shape))
            inputs.update(ref=ref, tgt=tgt)
        if Cc:
            rc, tc = per(rn(B, Cc, H, W), scales(Cc, g), 1), per(rn(B, Cc, H, W), scales(Cc, g), 1)
            cv = cat_ref(rc, tc, D, o.get("mask", 1))
            parts.append(cv), mags.append(torch.ones(1, 2 * Cc, 1, 1, 1, dtype=F64)), exact.append(torch.ones(cv.shape, dtype=torch.bool))
            inputs.update(rc=rc, tc=tc)
        want = torch.cat(parts, 1)
        scale = torch.cat([m.expand(1, p.shape[1], 1, 1, 1) for m, p in zip(mags, parts)], 1)
        ex = torch.cat(exact, 1)
        if e == "corr":
            want, scale, ex = want.squeeze(1), scale.squeeze(1), ex.squeeze(1)
        mask = o.get("mask", 1)
        fns = {
            "gwc": lambda y, P: call("osb_gwc_volume_fwd", P("ref"), P("tgt"), y, B, Cg, H, W, D, G, s()),
            "sum": lambda y, P: call("osb_gwc_volume_sum_fwd", P("ref"), P("tgt"), y, B, Cg, H, W, D, G, s()),
            "corr": lambda y, P: call("osb_corr_volume_fwd", P("ref"), P("tgt"), y, B, Cg, H, W, D, s()),
            "cat": lambda y, P: call("osb_concat_volume_fwd", P("rc"), P("tc"), y, B, Cc, H, W, D, mask, s()),
            "fused": lambda y, P: call("osb_gwc_concat_volume_fwd", P("ref"), P("tgt"), P("rc"), P("tc"), y, B, Cg, Cc, H, W, D, G,
                                       s()),
        }
        return [Case(row.id, want, scale, fns[e], inputs, exact=ex, info=dict(K=K, W=W, gwc=Cg > 0))]

    if fam == "sa":
        B, D, H, W = row.shape
        alpha, start, step, norm = o.get("alpha", 1.0), o.get("start", 0.0), o.get("step", 1.0), o.get("norm", 1)
        cost = o.get("offset", 0.0) + o.get("spread", 3.0) * (2 * torch.rand(B, D, H, W, generator=g) - 1)
        if o.get("peak_last"):
            cost[:, D - 1, ::2] += 0.5 * o.get("spread", 3.0) + 8.0
        if o.get("inf"):
            hit = torch.rand(B, D, H, W, generator=g) < 0.4
            hit[:, D // 2] = False                                  # every pixel keeps a finite bin
            cost = cost.masked_fill(hit, -math.inf)
        x = (cost * f32(alpha)).double()                            # the fp32 logits
        v = (f32(start) + f32(step) * torch.arange(D, dtype=torch.float32)).double().view(1, D, 1, 1)
        v = v.expand(B, D, H, W)
        if norm:
            p = torch.softmax(x, 1)
            want = (p * v).sum(1)
            scale, tol = soft_model(p, x, v, want, x.abs(), 0), TOL_SOFT
        else:
            want = (x * v).sum(1)
            scale, tol = (D + 2) * U * (x * v).abs().sum(1), TOL_SOFT
        fn = lambda y, P: call("osb_softargmin_fwd", P("cost"), y, B, D, H, W, alpha, start, step, norm, s())      # noqa: E731
        return [Case(row.id, want, scale, fn, {"cost": cost}, tol=tol)]

    if fam == "up":
        B, Dl, Hl, Wl, D, H, W = row.shape
        align = o["align"]
        cost = o.get("offset", 0.0) + o.get("spread", 4.0) * rn(B, Dl, Hl, Wl)
        axes = (axis(Dl, D, align), axis(Hl, H, align), axis(Wl, W, align))
        x = trilinear(cost.double(), axes)
        lam = trilinear(cost.double().abs(), axes)
        p = torch.softmax(x, 1)
        inputs = {"cost": cost}
        if o.get("values"):
            values = 50.0 * (2 * torch.rand(B, D, H, W, generator=g) - 1)          # non-monotone, negative hypotheses
            v = values.double()
            inputs["values"] = values
            fn = lambda y, P: call("osb_upsample_softargmin_values_fwd", P("cost"), P("values"), y, B, Dl, Hl, Wl, D, H, W,  # noqa
                                   align, s())
        else:
            v = torch.arange(D, dtype=F64).view(1, D, 1, 1).expand(B, D, H, W)
            fn = lambda y, P: call("osb_upsample_softargmin_fwd", P("cost"), y, B, Dl, Hl, Wl, D, H, W, align, s())  # noqa: E731
        want = (p * v).sum(1)
        scale = soft_model(p, x * math.log2(math.e), v, want, lam * math.log2(math.e), max(Dl, Hl, Wl))
        return [Case(row.id, want, scale, fn, inputs, tol=TOL_SOFT)]

    if fam == "epe":
        B, HW = row.shape
        maxdisp = o["maxdisp"]
        gt = 220 * torch.rand(B, HW, generator=g) - 10                # about a fifth outside (0, maxdisp)
        pred = gt + 3 * rn(B, HW)
        valid = (gt > 0) & (gt < maxdisp)
        terms = ((gt - pred).abs().double() * valid)
        want = torch.stack([terms.sum(1), valid.double().sum(1)], 1)
        scale = torch.stack([HW * U * terms.sum(1), torch.ones(B, dtype=F64)], 1)
        exact = torch.zeros(B, 2, dtype=torch.bool)
        exact[:, 1] = True                                            # counts: integers below 2^24, exact in fp32
        fn = lambda y, P: call("osb_epe_partial_fwd", P("pred"), P("gt"), y, B, HW, maxdisp, s())     # noqa: E731
        return [Case(row.id, want, scale, fn, {"pred": pred, "gt": gt}, tol=1.0, exact=exact, det_scale=scale)]

    if fam in ("bgwc", "bcat"):
        if fam == "bgwc":
            B, G, K, H, W, D = row.shape
            C = G * K
            ref, tgt = rn(B, C, H, W), rn(B, C, H, W)
            gvol = rn(B, G, D, H, W) * scales(G, g).view(1, G, 1, 1, 1)             # gradient weights per group
            sc = 1.0 if o["reduce_sum"] else 1.0 / K
            gv = gvol.double().repeat_interleave(K, dim=1)
            gl = gr = gv
            a_ref, a_tgt = tgt.double(), ref.double()
            inputs = {"gvol": gvol, "ref": ref, "tgt": tgt}
        else:
            B, C, H, W, D = row.shape
            gvol = rn(B, 2 * C, D, H, W) * scales(2 * C, g).view(1, 2 * C, 1, 1, 1)
            sc = 1.0
            gl, gr = gvol[:, :C].double(), gvol[:, C:].double()
            a_ref = a_tgt = torch.ones(B, C, H, W, dtype=F64)
            inputs = {"gvol": gvol}
        grf, gtg = torch.zeros(B, C, H, W, dtype=F64), torch.zeros(B, C, H, W, dtype=F64)
        mrf, mtg = torch.zeros_like(grf), torch.zeros_like(gtg)
        for d in range(D):
            if d < W:
                a = gl[:, :, d, :, d:] * a_ref[..., :W - d]                          # d(ref)[w] += gvol[d, w] * tgt[w - d]
                grf[..., d:] += a * sc
                mrf[..., d:] += a.abs() * sc
                b = gr[:, :, d, :, d:] * a_tgt[..., d:]                              # d(tgt)[w] += gvol[d, w + d] * ref[w + d]
                gtg[..., :W - d] += b * sc
                mtg[..., :W - d] += b.abs() * sc
            if fam == "bcat" and not o["mask"]:
                grf += gl[:, :, d] if d >= W else gl[:, :, d].masked_fill(torch.arange(W) >= d, 0.0)
                mrf += (gl[:, :, d] if d >= W else gl[:, :, d].masked_fill(torch.arange(W) >= d, 0.0)).abs()
        want = torch.stack([grf, gtg])
        scale = torch.stack([chanmax(mrf, 1), chanmax(mtg, 1)])
        n = B * C * H * W
        out = []
        for mode in ("both", "ref only", "tgt only"):
            skip = torch.zeros(want.shape, dtype=torch.bool)
            if mode == "ref only":
                skip[1] = True
            if mode == "tgt only":
                skip[0] = True

            def fn(y, P, mode=mode):
                yr = None if mode == "tgt only" else y
                yt = None if mode == "ref only" else y + 4 * n
                if fam == "bgwc":
                    call("osb_gwc_volume_bwd", P("gvol"), P("ref"), P("tgt"), yr, yt, B, C, H, W, D, G, o["reduce_sum"], s())
                else:
                    call("osb_concat_volume_bwd", P("gvol"), yr, yt, B, C, H, W, D, o["mask"], s())
            out.append(Case("%s %s" % (row.id, mode), want, scale, fn, inputs, skip=skip))
        return out

    if fam == "bsa":
        B, D, H, W = row.shape
        alpha, start, step, norm = o.get("alpha", 1.0), o.get("start", 0.0), o.get("step", 1.0), o.get("norm", 1)
        cost = 4 * rn(B, D, H, W)
        k = torch.randint(-12, 13, (B, H, W), generator=g)
        gout = torch.ldexp(torch.ones(B, H, W), k.int()) * (1.0 + 0.9 * torch.rand(B, H, W, generator=g)) * 0.77 * torch.sign(rn(B, H, W))
        x = (cost * f32(alpha)).double()
        v = (f32(start) + f32(step) * torch.arange(D, dtype=torch.float32)).double().view(1, D, 1, 1).expand(B, D, H, W)
        ga = (gout.double() * alpha).unsqueeze(1)
        if norm:
            p = torch.softmax(x, 1)
            outf = (p * v).sum(1, keepdim=True)
            want = ga * p * (v - outf)
            E = soft_model(p, x, v, outf.squeeze(1), x.abs(), 0).unsqueeze(1)
            eps = U * (2 * (x - x.amax(1, keepdim=True)).abs() + x.abs() + 16)
            scale = ga.abs() * (p * (v - outf).abs() * (eps + (D + 4) * U) + p * E) + ga.abs() * (v.abs() + outf.abs() + 1) * 2.0 ** -100
        else:
            want = ga * v
            scale = 4 * U * want.abs()
        fn = lambda y, P: call("osb_softargmin_bwd", P("cost"), P("gout"), y, B, D, H, W, alpha, start, step, norm, s())  # noqa: E731
        return [Case(row.id, want, scale, fn, {"cost": cost, "gout": gout}, tol=TOL_SOFT)]

    if fam == "geo":
        B, C, D, H, W, W2, L = row.shape
        r = o["radius"]
        T = 2 * r + 1
        geo = [per(rn(B, C, D >> i, H, W), scales(C, g), 1) for i in range(L)]
        corr = [rn(B, H, W, W2 >> i) * 3.1 for i in range(L)]
        disp = disp_mixture(g, (B, 1, H, W), -6.0, D + 6.0)
        coords = torch.arange(W, dtype=torch.float32).view(1, 1, W).expand(B, H, W).contiguous()
        want = torch.zeros(B, L, C + 1, T, H, W, dtype=F64)
        mag = torch.zeros_like(want)
        fallback = 0
        for lvl in range(L):
            sc = f32(1.0 / (1 << lvl))
            dq = disp[:, 0] * sc                                              # (B, H, W)
            for c in range(C + 1):
                if c < C:
                    n, base = D >> lvl, dq
                    data = geo[lvl][:, c].double()                               # (B, n, H, W): sample along dim 1
                else:
                    n, base = W2 >> lvl, coords * sc - dq
                    data = corr[lvl].double().permute(0, 3, 1, 2)               # (B, n, H, W)
                first = torch.floor(roundtrip_geo(f32(-r) + base, n))
                for k in range(T):
                    ix = roundtrip_geo(f32(k - r) + base, n)
                    fl = torch.floor(ix)
                    if r == 4:
                        fallback += int((fl != first + k).sum())
                    w1, w0 = (ix - fl).double(), ((fl + f32(1.0)) - ix).double()
                    i0 = fl.long()
                    vals = []
                    for i in (i0, i0 + 1):
                        ok = (i >= 0) & (i < n)
                        vals.append(torch.gather(data, 1, i.clamp(0, n - 1).unsqueeze(1)).squeeze(1) * ok)
                    want[:, lvl, c, k] = vals[0] * w0 + vals[1] * w1
                    mag[:, lvl, c, k] = (vals[0] * w0).abs() + (vals[1] * w1).abs()
        if o.get("cross"):
            assert fallback > 0, "%s: no tap crosses an integer in the coordinate round trip" % row.id
        want, mag = want.view(B, L * (C + 1) * T, H, W), mag.view(B, L * (C + 1) * T, H, W)
        inputs = {"disp": disp, "coords": coords}
        for i in range(L):
            inputs["geo%d" % i], inputs["corr%d" % i] = geo[i], corr[i]

        def fn(y, P):
            gp = [P("geo%d" % i) if i < L else None for i in range(4)]
            cp = [P("corr%d" % i) if i < L else None for i in range(4)]
            call("osb_geo_lookup_fwd", *gp, *cp, P("disp"), P("coords"), y, B, C, D, H, W, W2, L, r, s())
        return [Case(row.id, want, mag, fn, inputs)]

    if fam == "pool":
        outer, n, inner = row.shape
        if inner == 0:                                                  # above the grid cap: SM count x 32 blocks x 256
            inner = (5 * sm_count() * 32 * 256) // (2 * outer * (n // 2)) + 37
        x = rn(outer, n, inner)
        h = n // 2
        want = ((x[:, 0:2 * h:2] + x[:, 1:2 * h:2]) * 0.5).double()          # fp32 sum, exact halving
        fn = lambda y, P: call("osb_avgpool_pairs_fwd", P("x"), y, outer, n, inner, s())       # noqa: E731
        return [Case(row.id, want, None, fn, {"x": x}, exact=torch.ones(want.shape, dtype=torch.bool))]

    if fam == "ctx":
        B, h, w, sf = row.shape
        H, W = h * sf, w * sf
        disp = per(rn(B, h, w), scales(h, g), 1)                          # per low-resolution row
        up = rn(B, 9, H, W)
        dp = F.pad(disp.double(), (1, 1, 1, 1))
        yi, xi = torch.arange(H) // sf, torch.arange(W) // sf
        want = torch.zeros(B, H, W, dtype=F64)
        mag = torch.zeros_like(want)
        for k in range(9):
            nb = dp[:, yi + k // 3][:, :, xi + k % 3]
            want += up[:, k].double() * nb
            mag += (up[:, k].double() * nb).abs()
        fn = lambda y, P: call("osb_context_upsample_fwd", P("disp"), P("up"), y, B, h, w, sf, s())   # noqa: E731
        return [Case(row.id, want, mag, fn, {"disp": disp, "up": up}, info=dict(vec=W % 4 == 0 and sf % 4 == 0))]

    if fam == "cas":
        B, Cg, G, Cc, D, H, W = row.shape
        K = Cg // G if Cg else 0
        xc, yc = per(rn(B, Cc, H, W), scales(Cc, g), 1), per(rn(B, Cc, H, W), scales(Cc, g), 1)
        disp = disp_mixture(g, (B, D, H, W), -3.0, W + 3.0)
        half_w, half_h = f32((W - 1.0) / 2.0), f32((H - 1.0) / 2.0)
        iy = roundtrip_cas(torch.arange(H, dtype=torch.float32), half_h)      # (H,)
        fy = torch.floor(iy)
        ny = iy - fy
        if "two" in o:
            assert bool((ny != 0).any()) == bool(o["two"]), "%s: row coordinates do not stage the rows the row expects" % row.id
        sy = f32(1.0) - ny
        fw = torch.arange(W, dtype=torch.float32).view(1, 1, 1, W)
        ix = roundtrip_cas(fw - disp, half_w)                                # (B, D, H, W)
        inside = (ix > -2.0) & (ix < W + 1.0)
        fx = torch.floor(ix)
        wx = ix - fx
        ex = f32(1.0) - wx
        syv, nyv = sy.view(1, 1, H, 1), ny.view(1, 1, H, 1)
        wts = [syv * ex, syv * wx, nyv * ex, nyv * wx]                        # nw, ne, sw, se in fp32
        x0 = fx.long()

        def warp(y):
            """-> (taps, sum |terms|), (B, C, D, H, W)."""
            Cn = y.shape[1]
            taps, mg = torch.zeros(B, Cn, D, H, W, dtype=F64), torch.zeros(B, Cn, D, H, W, dtype=F64)
            for t, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
                yy = fy.long() + dy                                           # (H,)
                rows = y.double()[:, :, yy.clamp(0, H - 1)] * ((yy >= 0) & (yy < H)).view(1, 1, H, 1)   # (B, C, H, W)
                xx = x0 + dx
                okx = ((xx >= 0) & (xx < W) & inside).unsqueeze(1)
                idx = xx.clamp(0, W - 1).unsqueeze(1).expand(B, Cn, D, H, W)
                v = torch.gather(rows.unsqueeze(2).expand(B, Cn, D, H, W), 4, idx) * okx
                term = v * wts[t].double().unsqueeze(1)
                taps += term
                mg += term.abs()
            return taps, mg
        masked = (fw < disp).unsqueeze(1)                                    # (B, 1, D, H, W)
        parts, mags, exact, inputs = [], [], [], {"xc": xc, "yc": yc, "disp": disp}
        if Cg:
            xg, yg = per(rn(B, Cg, H, W), scales(Cg, g), 1), per(rn(B, Cg, H, W), scales(Cg, g), 1)
            tg, mg = warp(yg)
            xl = xg.double().unsqueeze(2)
            vol = (xl * tg).view(B, G, K, D, H, W).sum(2) / K
            vm = (xl.abs() * mg).view(B, G, K, D, H, W).sum(2) / K
            vol = vol.masked_fill(masked, 0.0)
            parts.append(vol), mags.append(chanmax(vm, 1)), exact.append(masked.expand(vol.shape))
            inputs.update(xg=xg, yg=yg)
        mask_left = 1 if Cg else o.get("mask", 0)
        left = xc.double().unsqueeze(2).expand(B, Cc, D, H, W)
        if mask_left:
            left = left.masked_fill(masked, 0.0)
        tc, mc = warp(yc)
        parts += [left, tc]
        mags += [torch.ones(1, Cc, 1, 1, 1, dtype=F64), chanmax(mc, 1)]
        exact += [torch.ones(left.shape, dtype=torch.bool), torch.zeros(tc.shape, dtype=torch.bool)]
        want = torch.cat(parts, 1)
        scale = torch.cat([m.expand(1, p.shape[1], 1, 1, 1) for m, p in zip(mags, parts)], 1)
        if Cg:
            fn = lambda y, P: call("osb_warped_gwc_concat_volume_fwd", P("xg"), P("yg"), P("xc"), P("yc"), P("disp"), y, B, Cg, G,  # noqa
                                   Cc, D, H, W, s())
        else:
            fn = lambda y, P: call("osb_warped_concat_volume_fwd", P("xc"), P("yc"), P("disp"), y, B, Cc, D, H, W, mask_left, s())  # noqa
        return [Case(row.id, want, scale, fn, inputs, exact=torch.cat(exact, 1))]

    if fam == "coex":
        B, D, h, w = row.shape
        k, logits = o["k"], o["logits"]
        cost = (rn(B, 1, D, h, w) * 2).round() / 2 if o.get("ties") else 3 * rn(B, 1, D, h, w)
        spx = 2 * rn(B, 9, 4 * h, 4 * w)
        if not logits:
            spx = torch.softmax(spx, 1)
        vals, idx = torch.sort(cost.double(), dim=2, descending=True, stable=True)
        p = torch.softmax(vals[:, :, :k], 2)
        d4 = (p * idx[:, :, :k].double()).sum(2)[:, 0]                       # (B, h, w)
        q = torch.softmax(spx.double(), 1) if logits else spx.double()
        dp = F.pad(d4, (1, 1, 1, 1))
        yi, xi = torch.arange(4 * h) // 4, torch.arange(4 * w) // 4
        want = torch.zeros(B, 4 * h, 4 * w, dtype=F64)
        scale = torch.zeros_like(want)
        ds = (spx.double() - spx.double().amax(1, keepdim=True)).abs() if logits else torch.zeros_like(q)
        for t in range(9):
            nb = dp[:, yi + t // 3][:, :, xi + t % 3]
            want += 4 * nb * q[:, t]
            # disp_4 carries ~(k + 2) roundings of values up to D; each weight (k + 9) roundings plus its softmax argument
            scale += 4 * U * q[:, t].abs() * (D * (k + 2) + nb.abs() * (k + 12 + ds[:, t]))
        fn = lambda y, P: call("osb_coex_regression_fwd", P("cost"), P("spx"), y, B, D, h, w, k, logits, s())     # noqa: E731
        return [Case(row.id, want, scale, fn, {"cost": cost, "spx": spx}, tol=TOL_SOFT)]

    if fam == "near":
        N, Di, Hi, Wi, Do, Ho, Wo = row.shape
        if N == 0:                                                      # above the grid cap: SM count x 8 blocks x 256
            N = (5 * sm_count() * 8 * 256) // (2 * Do * Ho * Wo) + 1
        x = rn(N, Di, Hi, Wi)
        want = F.interpolate(x.unsqueeze(1), size=(Do, Ho, Wo), mode="nearest")[:, 0].double()
        fn = lambda y, P: call("osb_nearest_resize3d_fwd", P("x"), y, N, Di, Hi, Wi, Do, Ho, Wo, s())   # noqa: E731
        return [Case(row.id, want, None, fn, {"x": x}, exact=torch.ones(want.shape, dtype=torch.bool))]

    if fam == "l2n":
        B, G, K, H, W = row.shape
        x = rn(B, G, K, H, W) * scales(G, g).view(1, G, 1, 1, 1)
        x[:, 0, :, 0] = 0.0                                             # a zero vector: 0 / eps
        x[:, -1, :, 1] *= 1e-14 / x[:, -1, :, 1].abs().amax()           # norm below eps: x / eps
        x = x.reshape(B, G * K, H, W)
        eps = float(f32(1e-12))
        xv = x.double().view(B, G, K, H, W)
        want = (xv / xv.norm(dim=2, keepdim=True).clamp(min=eps)).view(B, G * K, H, W)
        fn = lambda y, P: call("osb_group_l2_normalize_fwd", P("x"), y, B, G * K, H, W, G, 1e-12, s())    # noqa: E731
        return [Case(row.id, want, want.abs(), fn, {"x": x}, exact=(x == 0))]

    if fam == "sub":
        B, C, H, W, D = row.shape
        l, r = per(rn(B, C, H, W), scales(C, g), 1), per(rn(B, C, H, W), scales(C, g), 1)
        want = torch.zeros(B, D, H, W, dtype=F64)
        mag = torch.zeros_like(want)
        ld, rd = l.double(), r.double()
        for d in range(D):
            rs = torch.zeros_like(rd)
            if d < W:
                rs[..., d:] = rd[..., :W - d]
            want[:, d] = (ld - rs).abs().sum(1)
            mag[:, d] = (ld.abs() + rs.abs()).sum(1)
        fn = lambda y, P: call("osb_sub_volume_fwd", P("l"), P("r"), y, B, C, H, W, D, s())      # noqa: E731
        return [Case(row.id, want, chanmax(mag, 1), fn, {"l": l, "r": r})]

    if fam == "rv":
        B, D, H, W = row.shape
        prob = torch.softmax(3 * rn(B, D, H, W), 1)
        values = 40 * rn(B, D, H, W)
        want = (prob.double() * values.double()).sum(1)
        mag = (prob.double() * values.double()).abs().sum(1)
        fn = lambda y, P: call("osb_regression_values_fwd", P("prob"), P("values"), y, B, D, H, W, s())     # noqa: E731
        return [Case(row.id, want, mag, fn, {"prob": prob, "values": values})]

    assert fam == "pad"
    B, C, Cp, D, H, W = row.shape
    x = rn(B, C, D, H, W)
    want = torch.zeros(B, D, H, W, Cp, dtype=F64)
    want[..., :C] = x.permute(0, 2, 3, 4, 1).double()
    fn = lambda y, P: call("osb_ncdhw_to_ndhwc_pad", P("x"), y, B, C, Cp, D, H, W, s())          # noqa: E731
    return [Case(row.id, want, None, fn, {"x": x}, exact=torch.ones(want.shape, dtype=torch.bool))]


def seed(row, salt=0):
    return torch.Generator().manual_seed(salt + zlib.crc32(row.id.encode()) % 10000)


def runs_of(row, case):
    """(label, launch kwargs, grid cap, expected volume variant or None)."""
    runs = [("aligned", {}, 0), ("aligned again", {}, 0)]
    if row.fam == "vol":
        if case.info["W"] % 4 == 0:
            runs += [("out+4", {"y_off": 1}, 0), ("ref+4", {"shift": ("ref", "rc")}, 0), ("tgt+4", {"shift": ("tgt", "tc")}, 0),
                     ("ref+4 tgt+4", {"shift": ("ref", "rc", "tgt", "tc")}, 0)]
        runs += [("grid cap 1", {}, 1), ("grid cap 5", {}, 5)]
    if row.fam == "ctx" and case.info["vec"]:
        runs += [("out+4", {"y_off": 1}, 0), ("up+4", {"shift": ("up",)}, 0)]
    return runs


@pytest.mark.timeout(300)
@pytest.mark.parametrize("row", REGISTRY, ids=[r.id for r in REGISTRY])
def test_accuracy_store_paths_bounds_determinism(osb, grid_cap, row):
    _, ops = osb
    worst = 0.0
    for case in cases(osb, row, seed(row)):
        first = None
        for label, kw, cap in runs_of(row, case):
            what = "%s, %s" % (case.name, label)
            grid_cap(cap)
            buf, lead = case.launch(**kw)
            if row.fam == "vol":
                want_v = volume_variant(case.info["K"], case.info["W"], kw.get("shift", ()), kw.get("y_off", 0), case.info["gwc"])
                assert ops.volume_last_variant() == want_v, "%s: ran %s, expected %s" % (what, ops.volume_last_variant(), want_v)
            worst = max(worst, case.check(buf, lead, what))
            inner = buf[lead:lead + case.numel].cpu()
            if first is None:
                first = inner
            elif case.det_scale is None:
                assert torch.equal(first.view(torch.int32), inner.view(torch.int32)), "%s: differs bit-wise from the first run" % what
            else:
                diff = (first.double() - inner.double()).abs().view(case.want.shape)
                assert (diff <= 2 * case.det_scale).all(), "%s: repeated launches differ beyond the bar of the sum" % what
    print("\n%-22s %-5s worst err/scale %.2e (bar %g)" % (row.id, row.fam, worst, TOL_SOFT if row.fam in ("sa", "up", "bsa", "coex")
                                                          else (1.0 if row.fam == "epe" else TOL)))


def profiled_kernels(osb, case, what):
    """-> names (spaces removed) of the kernels of this library the profiler saw for one call of case.fn."""
    from torch.profiler import ProfilerActivity, profile
    lib, _ = osb
    dev = case.dev()
    buf = case.guarded()
    names = []
    for _ in range(3):
        torch.cuda.synchronize()
        before = lib.launch_count()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            case.fn(buf.data_ptr() + 4 * GUARD, lambda name: dev[name].data_ptr())
            torch.cuda.synchronize()
        assert lib.launch_count() - before == 1, "%s: %d launches for one call" % (what, lib.launch_count() - before)
        names = sorted({e.name.replace(" ", "") for e in prof.events() if "osb::" in e.name})
        if names:
            break
    return names


@pytest.mark.timeout(120)
@pytest.mark.parametrize("row", REGISTRY, ids=[r.id for r in REGISTRY])
def test_routing(osb, row):
    """One call is one launch (the library's launch counter) of the row's instantiation (torch.profiler).  In a few sessions per
    thousand the profiler's activity-buffer request lands inside cudaLaunchKernel (which then takes about 1 ms) and the session
    holds the launch's API record but no device record, although the kernel ran (measured on an H100 with the parent commit's
    library as well).  Only a session with no kernel of this library recorded is repeated, at most three times; a session
    that records any kernel is judged as it is."""
    names = profiled_kernels(osb, cases(osb, row, seed(row, 3))[0], row.id)
    want = re.compile(r"osb::%s\(" % re.escape(row.variant))
    assert len(names) == 1 and want.search(names[0]), "%s: launched %s, expected %s" % (row.id, names, row.variant)


@pytest.mark.timeout(300)
def test_volume_item_order_0(osb, tmp_path):
    """OSB_VOLUME_ORDER=0 (unit fastest) is read once per process: a child process computes a fused row in that order, and its
    output must equal order 1's bit for bit.  subprocess.run waits for the child and kills it on timeout."""
    row = BY_ID["vol-fused-k4"]
    case = cases(osb, row, seed(row))[0]
    buf, lead = case.launch()
    case.check(buf, lead, "order 1")
    mine = buf[lead:lead + case.numel].cpu()
    B, G, K, Cc, H, W, D = row.shape
    torch.save({k: v for k, v in case.inputs.items()}, str(tmp_path / "in.pt"))
    script = ("import sys, torch\n"
              "from openstereo_b200 import ops\n"
              "t = torch.load(sys.argv[1] + '/in.pt')\n"
              "c = {k: v.cuda() for k, v in t.items()}\n"
              "out = ops.gwc_concat_volume(c['ref'], c['tgt'], c['rc'], c['tc'], %d, %d)\n"
              "torch.save(out.cpu(), sys.argv[1] + '/out.pt')\n" % (D, G))
    env = dict(os.environ, OSB_VOLUME_ORDER="0", PYTHONPATH=os.pathsep.join([ROOT] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    res = subprocess.run([sys.executable, "-c", script, str(tmp_path)], env=env, cwd=ROOT, timeout=240, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    other = torch.load(str(tmp_path / "out.pt")).flatten()
    assert torch.equal(other.view(torch.int32), mine.view(torch.int32)), "order 0 and order 1 differ"


@pytest.mark.timeout(120)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("entry", ["gwc", "sum", "corr", "cat", "fused"])
def test_volume_input_types(osb, entry, dtype):
    """fp16 / bf16 features through ops.*: the output has the input type and equals the fp32 result of the same (exactly
    up-converted) features, rounded to that type; and that is within the type's rounding of the fp64 reference."""
    _, ops = osb
    g = torch.Generator().manual_seed(7 + len(entry))
    B, C, Cc, H, W, D, G = 2, 12, 5, 3, 36, 11, 3
    a = [(torch.randn(B, n, H, W, generator=g) * 2).to(dtype).cuda() for n in (C, C, Cc, Cc)]
    run = {"gwc": lambda t: ops.build_gwc_volume(t[0], t[1], D, G),
           "sum": lambda t: ops.coex_cost_volume(t[0], t[1], D - 1, G),
           "corr": lambda t: ops.correlation_volume(t[0], t[1], D),
           "cat": lambda t: ops.build_concat_volume(t[2], t[3], D),
           "fused": lambda t: ops.gwc_concat_volume(t[0], t[1], t[2], t[3], D, G)}[entry]
    got = run(a)
    assert got.dtype == dtype
    full = run([t.float() for t in a])
    assert full.dtype == torch.float32
    assert torch.equal(got, full.to(dtype)), "%s: %s output is not the rounded fp32 result" % (entry, dtype)
    r, t = a[0].double().cpu(), a[1].double().cpu()
    parts = []
    if entry in ("gwc", "sum", "corr", "fused"):
        vol, mag = gwc_ref(r, t, 1 if entry == "corr" else G, D, 1.0 if entry == "sum" else 1.0 / (C // (1 if entry == "corr" else G)))
        parts.append((vol, chanmax(mag, 1)))
    if entry in ("cat", "fused"):
        cv = cat_ref(a[2].double().cpu(), a[3].double().cpu(), D, 1)
        parts.append((cv, torch.zeros(1, dtype=F64)))
    want = torch.cat([p for p, _ in parts], 1)
    scale = torch.cat([m.expand(1, p.shape[1], 1, 1, 1) for p, m in parts], 1)
    gd = got.double().cpu().view(want.shape)
    rel = torch.finfo(dtype).eps / 2
    assert ((gd - want).abs() <= rel * want.abs() + TOL * scale).all(), "%s: %s output beyond the type's rounding" % (entry, dtype)


def refusals(P, s):
    """(what, entry point, arguments); P is a 4 MB device buffer every pointer argument refers to."""
    mis = P + 4
    gb, cb, sb = "osb_gwc_volume_bwd", "osb_concat_volume_bwd", "osb_softargmin_bwd"
    geo = "osb_geo_lookup_fwd"
    lv = (P,) * 8                                                       # geo0..3, corr0..3
    cx, cg = "osb_warped_concat_volume_fwd", "osb_warped_gwc_concat_volume_fwd"
    co = "osb_coex_regression_fwd"
    return [
        ("gwc_volume empty W", "osb_gwc_volume_fwd", (P, P, P, 1, 8, 4, 0, 4, 2, s)),
        ("gwc_volume empty D", "osb_gwc_volume_fwd", (P, P, P, 1, 8, 4, 8, 0, 2, s)),
        ("gwc_volume C % G", "osb_gwc_volume_fwd", (P, P, P, 1, 9, 4, 8, 4, 2, s)),
        ("gwc_volume K 145", "osb_gwc_volume_fwd", (P, P, P, 1, 145, 2, 8, 4, 1, s)),
        ("gwc_volume K 145 x 2", "osb_gwc_volume_fwd", (P, P, P, 1, 290, 2, 8, 4, 2, s)),
        ("gwc_volume_sum C % G", "osb_gwc_volume_sum_fwd", (P, P, P, 1, 10, 4, 8, 4, 3, s)),
        ("gwc_volume_sum empty B", "osb_gwc_volume_sum_fwd", (P, P, P, 0, 8, 4, 8, 4, 2, s)),
        ("corr_volume empty H", "osb_corr_volume_fwd", (P, P, P, 1, 8, 0, 8, 4, s)),
        ("corr_volume K 145", "osb_corr_volume_fwd", (P, P, P, 1, 145, 2, 8, 4, s)),
        ("concat_volume empty D", "osb_concat_volume_fwd", (P, P, P, 1, 4, 4, 8, 0, 1, s)),
        ("concat_volume C 0", "osb_concat_volume_fwd", (P, P, P, 1, 0, 4, 8, 4, 1, s)),
        ("gwc_concat_volume Cc 0", "osb_gwc_concat_volume_fwd", (P, P, P, P, P, 1, 8, 0, 4, 8, 4, 2, s)),
        ("gwc_concat_volume C % G", "osb_gwc_concat_volume_fwd", (P, P, P, P, P, 1, 9, 4, 4, 8, 4, 2, s)),
        ("softargmin empty D", "osb_softargmin_fwd", (P, P, 1, 0, 4, 4, 1.0, 0.0, 1.0, 1, s)),
        ("upsample_softargmin empty", "osb_upsample_softargmin_fwd", (P, P, 1, 4, 2, 3, 16, 0, 3, 0, s)),
        ("upsample_softargmin table", "osb_upsample_softargmin_fwd", (P, P, 1, 4, 2, 3, 12284, 2, 3, 0, s)),
        ("upsample_softargmin_values table", "osb_upsample_softargmin_values_fwd", (P, P, P, 1, 4, 2, 3, 12284, 2, 3, 0, s)),
        ("upsample_softargmin_values empty", "osb_upsample_softargmin_values_fwd", (P, P, P, 1, 0, 2, 3, 16, 2, 3, 0, s)),
        ("epe_partial empty", "osb_epe_partial_fwd", (P, P, P, 1, 0, 192.0, s)),
        ("gwc_volume_bwd C*H 65792", gb, (P, P, P, P, P, 1, 256, 257, 8, 4, 2, 0, s)),
        ("gwc_volume_bwd C % G", gb, (P, P, P, P, P, 1, 9, 4, 8, 4, 2, 0, s)),
        ("gwc_volume_bwd no gradient", gb, (P, P, P, None, None, 1, 8, 4, 8, 4, 2, 0, s)),
        ("gwc_volume_bwd empty D", gb, (P, P, P, P, P, 1, 8, 4, 8, 0, 2, 0, s)),
        ("concat_volume_bwd C*H 65792", cb, (P, P, P, 1, 256, 257, 8, 4, 1, s)),
        ("concat_volume_bwd no gradient", cb, (P, None, None, 1, 8, 4, 8, 4, 1, s)),
        ("concat_volume_bwd empty W", cb, (P, P, P, 1, 8, 4, 0, 4, 1, s)),
        ("softargmin_bwd empty", sb, (P, P, P, 1, 0, 4, 4, 1.0, 0.0, 1.0, 1, s)),
        ("geo_lookup 0 levels", geo, lv + (P, P, P, 1, 2, 16, 2, 8, 8, 0, 4, s)),
        ("geo_lookup 5 levels", geo, lv + (P, P, P, 1, 2, 64, 2, 8, 64, 5, 4, s)),
        ("geo_lookup radius 17", geo, lv + (P, P, P, 1, 2, 64, 2, 8, 64, 2, 17, s)),
        ("geo_lookup radius -1", geo, lv + (P, P, P, 1, 2, 64, 2, 8, 64, 2, -1, s)),
        ("geo_lookup D pyramid", geo, lv + (P, P, P, 1, 2, 7, 2, 8, 64, 3, 4, s)),
        ("geo_lookup W2 pyramid", geo, lv + (P, P, P, 1, 2, 64, 2, 8, 7, 3, 4, s)),
        ("geo_lookup null level", geo, (P, None, P, P, P, P, P, P, P, P, P, 1, 2, 64, 2, 8, 64, 2, 4, s)),
        ("geo_lookup empty", geo, lv + (P, P, P, 1, 0, 64, 2, 8, 64, 2, 4, s)),
        ("avgpool_pairs n 1", "osb_avgpool_pairs_fwd", (P, P, 4, 1, 4, s)),
        ("context_upsample scale 0", "osb_context_upsample_fwd", (P, P, P, 1, 4, 4, 0, s)),
        ("warped_concat H 1", cx, (P, P, P, P, 1, 4, 2, 1, 8, 0, s)),
        ("warped_concat W 1", cx, (P, P, P, P, 1, 4, 2, 4, 1, 0, s)),
        ("warped_concat empty D", cx, (P, P, P, P, 1, 4, 0, 4, 8, 0, s)),
        ("warped_concat W 3633", cx, (P, P, P, P, 1, 1, 2, 2, 3633, 1, s)),
        ("warped_gwc K 17", cg, (P, P, P, P, P, P, 1, 17, 1, 4, 2, 4, 8, s)),
        ("warped_gwc Cg % G", cg, (P, P, P, P, P, P, 1, 10, 3, 4, 2, 4, 8, s)),
        ("warped_gwc W 1817", cg, (P, P, P, P, P, P, 1, 16, 1, 1, 2, 2, 1817, s)),
        ("warped_gwc Cc 0", cg, (P, P, P, P, P, P, 1, 16, 2, 0, 2, 4, 8, s)),
        ("coex top_k 1", co, (P, P, P, 1, 8, 4, 4, 1, 1, s)),
        ("coex top_k 9", co, (P, P, P, 1, 16, 4, 4, 9, 1, s)),
        ("coex top_k 5 > D 4", co, (P, P, P, 1, 4, 4, 4, 5, 1, s)),
        ("coex spx+4", co, (P, mis, P, 1, 8, 4, 4, 2, 1, s)),
        ("coex out+4", co, (P, P, mis, 1, 8, 4, 4, 2, 1, s)),
        ("coex empty", co, (P, P, P, 1, 8, 0, 4, 2, 1, s)),
        ("nearest_resize3d empty", "osb_nearest_resize3d_fwd", (P, P, 1, 2, 2, 2, 0, 2, 2, s)),
        ("group_l2_normalize C % G", "osb_group_l2_normalize_fwd", (P, P, 1, 10, 4, 4, 3, 1e-12, s)),
        ("group_l2_normalize empty", "osb_group_l2_normalize_fwd", (P, P, 1, 8, 0, 4, 2, 1e-12, s)),
        ("sub_volume empty", "osb_sub_volume_fwd", (P, P, P, 1, 4, 4, 8, 0, s)),
        ("sub_volume B*H 65536", "osb_sub_volume_fwd", (P, P, P, 2, 4, 32768, 8, 4, s)),
        ("regression_values empty", "osb_regression_values_fwd", (P, P, P, 1, 0, 4, 4, s)),
        ("ncdhw_to_ndhwc_pad Cpad < C", "osb_ncdhw_to_ndhwc_pad", (P, P, 1, 8, 4, 2, 2, 2, s)),
    ]


@pytest.mark.timeout(60)
def test_refusals(osb):
    lib, _ = osb
    buf = torch.zeros(1 << 20, device="cuda")                   # 4 MB: every argument list above stays inside it
    torch.cuda.synchronize()
    for what, name, args in refusals(buf.data_ptr(), torch.cuda.current_stream().cuda_stream):
        before = lib.launch_count()
        rc = getattr(lib.lib, name)(*args)
        assert rc == OSB_EINVAL, "%s: %s returned %d, expected %d (%s)" % (what, name, rc, OSB_EINVAL, lib.lib.osb_last_error())
        assert lib.launch_count() == before, "%s: a refused call launched a kernel" % what
    torch.cuda.synchronize()
