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
                                     the warped volumes, the interlaced crops, nearest_resize3d, avgpool_pairs, the layout pass
                                     with its zero channels, and the exact zeros of every masked triangle;
                 soft-argmin family  per pixel, see soft_model();
  bounds       the output region starts as NaN between 4 KB sentinel guards: every element is written and no sentinel changes;
               a backward launch with one gradient pointer null, or a variance launch with var_out null, leaves that output's
               region unwritten;
  store paths  where a kernel picks its loads and stores by alignment (the volume's vec_ok and use_tma, context_upsample's
               vector branch) the row runs aligned and with pointers moved 4 bytes: bit-identical, and each run passes the bar;
  item loop    volume and crop rows run at persistent-grid caps 1, 5 and uncapped, bit-identical; the grid-stride rows of
               avgpool_pairs and nearest_resize3d have totals above their SM-count-based grid caps;
  determinism  two launches are bit-identical, except epe_partial_kernel, whose float atomics add block partial sums in
               arrival order: its error sum gets the bar of the sum instead (its counts are integers and stay exact).
Runtime modes are row families of their own (NONCONV_MODE_VARIANTS; NONCONV_KERNEL_PARAMS classifies every parameter of every
kernel above, a by-value struct parameter field by field, as an operand or as the mode it selects, and MODE_REQUIREMENTS lists the
edges each family's rows must cover):
  crop         the interlaced crops (VolParams::crop): all D crops in one guarded buffer, bit-exact against the fp64 gather;
               aligned, with the left or the right input moved 4 bytes (a moved left input takes volume_kernel<false,true>),
               at grid caps 1 and 5; three column tiles and two disparity chunks, D = W, the largest C whose rows fit;
  var          the soft-argmin variance (softargmin_kernel's values / var_out): mean and variance in one guarded buffer; the
               variance is summed about the kernel's fp32 mean, so its bar adds the mean's bar squared; the var_out-NULL run's
               mean equals the full run's bit for bit, and with values NULL too it is osb_softargmin_fwd's result;
  geov         the geometry-only lookup (corr[0] == NULL): geo_model without correlation rows, a grid z of exactly 65535;
  geomr        the multi-range lookup: four outputs, one case each, the other three written to guarded scratch; vol2's taps
               leave both ends; D1 != D2, D1 = D2 = 2, W2 != W, a grid z of exactly 65535;
  warp         the disparity warp (border = 1): border_roundtrip replayed in fp32, disparities past both edges, 227 KB of rows;
  slice        the channel slice of a channels-last concatenation: exact inside the slice, the other channels still NaN;
  split        the split NDHWC conversion: every 32-bit word of hi/lo halves exact, tc_overflow_count >= 1 after a saturating
               row and 0 after the others.
The cas rows with mask = 0 run the fused warped volume through its _ex entry point with the left copy and the correlation
unmasked (CFNet), at fractional samples, on both instantiations.
test_volume_item_order_0: the other work-item order, read once per process, in a child process, bit-identical to order 1, for a
fused volume and for interlaced crops (through ops.interlaced_crops, whose views must have the crops' shapes).
test_warped_ex_mask_left_1: the _ex entry point with mask_left = 1 is osb_warped_gwc_concat_volume_fwd bit for bit.
test_volume_input_types: fp16 / bf16 inputs through ops.*: output in the input type, equal to the rounded fp32 result.
test_refusals: every input an entry point refuses returns OSB_EINVAL and launches nothing, and a valid launch after them all
returns OSB_OK (no refusal leaves a CUDA error behind for the next launch to report).
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
OSB_OK, OSB_EINVAL = 0, 1
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
    # interlaced-crops mode (VolParams::crop, osb_interlaced_crops_fwd) (B, C, H, W, D): the D crops (B, H, W - d, 2C) back to back.
    # A work item stages C left and C right rows of one 128-column tile, 1288 C + 16 bytes
    R("crop-w260-d70", "crop", V(1, 1), (2, 8, 3, 260, 70)),           # three column tiles, the last partial; two disparity chunks
    R("crop-d-eq-w", "crop", V(0, 1), (1, 4, 2, 131, 131)),            # the last crop is one column wide
    R("crop-c180", "crop", V(1, 1), (1, 180, 2, 40, 9)),               # 231 856 bytes staged: the largest C that fits 227 KB
    R("crop-msnet2d", "crop", V(1, 1), (2, 32, 3, 240, 48)),           # MSNet2D's own shape at 1/4 of 960
    R("crop-b3-w61", "crop", V(0, 1), (3, 8, 2, 61, 17)),
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
    # variance mode (values / var_out, osb_softargmin_var_fwd) (B, D, H, W): the sa rows' costs; values = 1 reads sorted non-integer
    # samples, some negative (CFNet's), values NULL the planes 0 .. D - 1.  No pixel count is a multiple of the 256-thread block
    R("var-d1", "var", "softargmin_kernel", (2, 1, 5, 37)),                         # the variance must be exactly 0
    R("var-d1-values", "var", "softargmin_kernel", (2, 1, 5, 37), values=1),
    R("var-d9-inf", "var", "softargmin_kernel", (2, 9, 5, 37), inf=1),               # a one-bin last chunk with -inf bins
    R("var-d9-inf-values", "var", "softargmin_kernel", (2, 9, 7, 37), inf=1, values=1, peak_last=1),
    R("var-d193-inf-values", "var", "softargmin_kernel", (1, 193, 3, 37), inf=1, spread=60.0, values=1),
    R("var-d48-spread", "var", "softargmin_kernel", (1, 48, 5, 37), spread=60.0, offset=1e4),
    R("var-d192-spread-values", "var", "softargmin_kernel", (1, 192, 5, 37), spread=60.0, offset=1e4, values=1),
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
    # geometry-only mode (corr[0] == NULL, osb_geo_volume_lookup_fwd) (B, C, D, H, W, levels): output (B, L * C * (2r + 1), H, W)
    R("geov-r4-l4", "geov", "geo_lookup_kernel<4>", (2, 3, 48, 3, 130, 4), radius=4, cross=1),
    R("geov-r4-l1", "geov", "geo_lookup_kernel<4>", (1, 2, 8, 2, 21, 1), radius=4),
    R("geov-r0-l2", "geov", "geo_lookup_kernel<0>", (1, 3, 16, 2, 40, 2), radius=0),
    R("geov-r2-l3-b3", "geov", "geo_lookup_kernel<0>", (3, 2, 24, 2, 131, 3), radius=2),
    R("geov-zmax", "geov", "geo_lookup_kernel<0>", (257, 85, 8, 1, 3, 3), radius=1),        # grid z = B * L * C = 65535
    # multi-range mode (out_corr != NULL, osb_geo_multirange_lookup_fwd) (B, C, D0, D1, D2, H, W, W2, levels): four outputs, the
    # geo_volume0 pyramid, vol1 at disp / 2, vol2 at disp / 4 and the correlation rows
    R("geomr-r4-l4", "geomr", "geo_lookup_kernel<4>", (2, 3, 48, 13, 7, 2, 130, 136, 4), radius=4, cross=1),
    R("geomr-r4-l1-d2", "geomr", "geo_lookup_kernel<4>", (1, 2, 8, 2, 2, 3, 21, 20, 1), radius=4),
    R("geomr-r0-l2", "geomr", "geo_lookup_kernel<0>", (1, 3, 16, 6, 10, 2, 40, 44, 2), radius=0),
    R("geomr-r3-l3", "geomr", "geo_lookup_kernel<0>", (2, 2, 24, 12, 5, 2, 131, 140, 3), radius=3),
    R("geomr-zmax", "geomr", "geo_lookup_kernel<0>", (771, 28, 4, 3, 5, 1, 3, 6, 1), radius=1),   # B * (L * C + 2C + L) = 65535
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
    # the left copy and the correlation unmasked (osb_warped_gwc_concat_volume_ex_fwd, mask_left = 0: CFNet)
    R("cas-gwc-k8-unmasked", "cas", "warped_volume_kernel<8>", (2, 24, 3, 5, 4, 10, 40), mask=0, two=1),
    R("cas-gwc-wmax-unmasked", "cas", "warped_volume_kernel<16>", (1, 32, 2, 3, 2, 6, 1816), mask=0, two=1),   # 227 KB of rows
    # disparity-warp mode (border = 1, osb_disp_warp_fwd) (B, C, H, W): units of 8 channels; every row coordinate is an integer at
    # H = 2 (and 3), not at the heights below
    R("warp-c5-h2", "warp", "warped_volume_kernel<8>", (2, 5, 2, 17), two=0),
    R("warp-c8-w131", "warp", "warped_volume_kernel<8>", (1, 8, 7, 131), two=1),
    R("warp-c19", "warp", "warped_volume_kernel<8>", (2, 19, 6, 40), two=1),              # three units, the last one partial
    R("warp-wmax", "warp", "warped_volume_kernel<8>", (1, 8, 4, 3632), two=1),            # 8 x 2 rows x 3632 floats = 227 KB, all staged
    R("warp-w2", "warp", "warped_volume_kernel<8>", (1, 1, 5, 2), two=1),
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
    # channel slice (osb_ncdhw_to_ndhwc_slice) (B, C, D, H, W, ystride, coff): channels coff .. coff + C - 1 of voxels of ystride
    R("slice-96-at-150", "slice", "ncdhw_to_ndhwc_kernel", (2, 96, 1, 5, 37, 300, 150)),
    R("slice-5-at-3", "slice", "ncdhw_to_ndhwc_kernel", (1, 5, 2, 3, 11, 13, 3)),
    R("slice-40-whole", "slice", "ncdhw_to_ndhwc_kernel", (1, 40, 2, 3, 7, 40, 0)),
    R("slice-33-at-37-last", "slice", "ncdhw_to_ndhwc_kernel", (2, 33, 1, 4, 9, 70, 37)),  # odd C and offset, ends at the last channel
    # split output (osb_ncdhw_to_split) (B, C, D, H, W): split NDHWC, 2C fp16 per voxel
    R("split-c16", "split", "ncdhw_to_ndhwc_kernel", (2, 16, 3, 5, 7)),
    R("split-c48", "split", "ncdhw_to_ndhwc_kernel", (1, 48, 2, 3, 11)),                  # two transpose tiles of channels
    R("split-c32-sat", "split", "ncdhw_to_ndhwc_kernel", (2, 32, 2, 3, 9), sat=1),        # |x| >= 4094 and subnormal lo halves
]
BY_ID = {r.id: r for r in REGISTRY}

# Runtime modes of the kernels above.  Each mode is one row family; NONCONV_MODE_VARIANTS lists the instantiations its entry point
# reaches, and its rows must reach exactly those (tests/test_host_logic_cpu.py).
NONCONV_MODE_VARIANTS = {
    "crop": {V(1, 1), V(0, 1)},                                         # interlaced crops (MSNet2D): VolParams::crop
    "var": {"softargmin_kernel"},                                       # soft-argmin variance (CFNet): values / var_out
    "geov": {"geo_lookup_kernel<4>", "geo_lookup_kernel<0>"},           # geometry-only (IGEV-RT): corr[0] == NULL
    "geomr": {"geo_lookup_kernel<4>", "geo_lookup_kernel<0>"},          # multi-range (IGEV++): out_corr != NULL
    "warp": {"warped_volume_kernel<8>"},                                # disparity warp (MonSter, AANet): border = 1
    "slice": {"ncdhw_to_ndhwc_kernel"},                                 # channel slice of a channels-last concatenation
    "split": {"ncdhw_to_ndhwc_kernel"},                                 # split NDHWC output
}


def _plain(names):
    return {n: "" for n in names.split()}


# Every parameter of every kernel above (the __global__ functions of the registry's sources, tests/test_host_logic_cpu.py), a
# by-value struct parameter replaced by its fields, spelled as the kernel reads them ("p.crop", "ad.align"): "" = an operand,
# geometry field or flag the plain rows exercise, otherwise the mode whose rows exercise it.  A parameter that is not here fails
# tests/test_host_logic_cpu.py.  p.order is the work-item order: order 1 in every row, order 0 in test_volume_item_order_0.
NONCONV_KERNEL_PARAMS = {
    "volume_kernel": {
        **_plain("tgt_map total_items"),
        **{"p." + f: "" for f in ("ref_g tgt_g ref_c tgt_c out B Cg Cc H W D G K Ctot oc_cat GU n_gwc_units n_cat_units w_tiles "
                                  "d_chunks mask_left use_tma vec_ok order inv_k").split()},
        "p.crop": "crop",
    },
    "softargmin_kernel": {**_plain("cost out D HW total alpha start step normalize"), "values": "var", "var_out": "var"},
    "upsample_softargmin_kernel": {**_plain("cost out Dl Hl Wl D H W values"),
                                   **{"%s.%s" % (a, f): "" for a in ("ad", "ah", "aw") for f in ("scale", "in", "align")}},
    "epe_partial_kernel": _plain("pred gt out HW maxdisp"),
    "gwc_volume_bwd_kernel": _plain("gvol ref tgt gref gtgt C H W D G s"),
    "concat_volume_bwd_kernel": _plain("gvol gref gtgt C H W D mask_left"),
    "softargmin_bwd_kernel": _plain("cost gout gcost D hw total alpha start step normalize"),
    "geo_lookup_kernel": {
        **{"p." + f: "" for f in "geo disp coords out B C D H W W2 levels radius".split()},
        "p.corr": "geov",
        **{"p." + f: "geomr" for f in "vol1 vol2 out1 out2 out_corr D1 D2".split()},
    },
    "avgpool_pairs_kernel": _plain("x y outer n inner"),
    "context_upsample_kernel": _plain("disp up out h w s"),
    "warped_volume_kernel": {
        **{"p." + f: "" for f in ("xg yg xc yc disp out B Cg G K Cc D H W Ctot oc_cat n_gwc_units n_cat_units mask_left half_w "
                                  "half_h").split()},
        **{"p." + f: "warp" for f in "border wm1 hm1".split()},
    },
    "coex_regression_kernel": {"p." + f: "" for f in "cost spx out B D h w logits".split()},
    "nearest_resize3d_kernel": _plain("x y total Di Hi Wi Do Ho Wo"),
    "group_l2_normalize_kernel": _plain("x y K hw total eps"),
    "sub_volume_kernel": _plain("l r out C H W D"),
    "regression_values_kernel": _plain("prob values out D hw total"),
    "ncdhw_to_ndhwc_kernel": {**_plain("x y C Cp vol"), "ys": "split", "overflow": "split", "ystride": "slice", "coff": "slice"},
}


def grid_z(row):
    """Grid z of a geo_lookup_kernel launch: one CTA row per (batch item, row of the output)."""
    if row.fam == "geov":
        B, C, D, H, W, L = row.shape
        return B * L * C
    B, C, D0, D1, D2, H, W, W2, L = row.shape
    return B * (L * C + 2 * C + L)


def _pow2(n):
    return n & (n - 1) == 0


def crop_smem(C):
    """Shared memory of an interlaced-crops CTA (volume.cu crop_smem_bytes): a left row of 128 + 1 and a right row of 192 + 1
    floats per channel, and 16 bytes of mbarriers."""
    return C * (129 + 193) * 4 + 16


SMEM_OPT_IN = 227 * 1024


# What each mode's rows must include between them (tests/test_host_logic_cpu.py): every requirement is met by at least one row.
MODE_REQUIREMENTS = {
    "crop": {
        "three column tiles, the last one partial, and two disparity chunks": lambda r: 256 < r.shape[3] < 384 and r.shape[3] % 128
        and 64 < r.shape[4] <= 128,
        "D = W with W % 4 != 0 at C = 4": lambda r: r.shape[4] == r.shape[3] and r.shape[3] % 4 and r.shape[1] == 4,
        "the largest C whose staged rows fit": lambda r: crop_smem(r.shape[1]) <= SMEM_OPT_IN < crop_smem(r.shape[1] + 4),
        "MSNet2D's shape at 1/4 of 960": lambda r: r.shape[1:] == (32, 3, 240, 48),
        "B > 1 at an odd width": lambda r: r.shape[0] > 1 and r.shape[3] % 2,
    },
    "var": {
        "D = 1": lambda r: r.shape[1] == 1,
        "-inf bins with a one-bin last chunk at D = 9": lambda r: r.shape[1] == 9 and r.opts.get("inf"),
        "-inf bins with a one-bin last chunk at D = 193": lambda r: r.shape[1] == 193 and r.opts.get("inf"),
        "offset 1e4 with spread 60": lambda r: r.opts.get("offset") == 1e4 and r.opts.get("spread") == 60.0,
        "values (also run with var_out NULL)": lambda r: r.opts.get("values"),
        "values NULL": lambda r: not r.opts.get("values"),
        "a pixel count not a multiple of 256": lambda r: (r.shape[0] * r.shape[2] * r.shape[3]) % 256,
    },
    "geov": {
        "radius 4 over 4 levels with taps that take the fallback read": lambda r: r.opts["radius"] == 4 and r.shape[5] == 4 and r.opts.get("cross"),
        "radius 4 at one level": lambda r: r.opts["radius"] == 4 and r.shape[5] == 1,
        "radius 0": lambda r: r.opts["radius"] == 0,
        "a generic radius other than 0 at B = 3 and a partial 128-column block": lambda r: r.opts["radius"] not in (0, 4) and r.shape[0] == 3
        and r.shape[4] % 128 not in (0, r.shape[4]),
        "grid z = 65535": lambda r: grid_z(r) == 65535,
    },
    "geomr": {
        "radius 4 over 4 levels with taps that take the fallback read": lambda r: r.opts["radius"] == 4 and r.shape[8] == 4 and r.opts.get("cross"),
        "radius 4 at one level with D1 = D2 = 2": lambda r: r.opts["radius"] == 4 and r.shape[8] == 1 and r.shape[3] == r.shape[4] == 2,
        "radius 0": lambda r: r.opts["radius"] == 0,
        "radius 3": lambda r: r.opts["radius"] == 3,
        "D1 != D2, neither a power of two": lambda r: r.shape[3] != r.shape[4] and not _pow2(r.shape[3]) and not _pow2(r.shape[4]),
        "W2 != W": lambda r: r.shape[7] != r.shape[6],
        "grid z = 65535": lambda r: grid_z(r) == 65535,
    },
    "warp": {
        "a partial unit at H = 2": lambda r: r.shape[1] % 8 and r.shape[2] == 2,
        "three units, the last one partial": lambda r: r.shape[1] > 16 and r.shape[1] % 8,
        "227 KB of staged rows, two per channel": lambda r: r.shape[1] >= 8 and 8 * 2 * r.shape[3] * 4 == 227 * 1024 and r.opts["two"],
        "W = 2": lambda r: r.shape[3] == 2,
    },
    "slice": {
        "odd channel count and offset, ending at the voxel's last channel": lambda r: r.shape[1] % 2 and r.shape[6] % 2
        and r.shape[6] + r.shape[1] == r.shape[5],
        "a slice that is the whole voxel": lambda r: r.shape[6] == 0 and r.shape[1] == r.shape[5],
        "three channel tiles in the middle of the voxel": lambda r: r.shape[1] > 64 and 0 < r.shape[6] < r.shape[5] - r.shape[1],
    },
    "split": {
        "one granule": lambda r: r.shape[1] == 16,
        "two transpose tiles of channels": lambda r: r.shape[1] > 32,
        "saturation and subnormal lo halves": lambda r: r.opts.get("sat"),
    },
}


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


def lerp_taps(data, n, base, r):
    """Taps k = 0 .. 2r of grid_sample's linear interpolation (align_corners=True, zero padding) of data (B, C, n, H, W) along dim
    2 at base + (k - r), base (B, H, W) in fp32, the coordinate round-tripped as geo.cu does -> (taps (B, C, T, H, W), sum |terms|,
    number of taps whose floor is not the first tap's floor + k: those take the kernel's fallback read)."""
    B, Cn, _, H, W = data.shape
    first = torch.floor(roundtrip_geo(f32(-r) + base, n))
    taps, mags, cross = [], [], 0
    for k in range(2 * r + 1):
        ix = roundtrip_geo(f32(k - r) + base, n)
        fl = torch.floor(ix)
        cross += int((fl != first + k).sum())
        w1, w0 = (ix - fl).double().unsqueeze(1), ((fl + f32(1.0)) - ix).double().unsqueeze(1)
        i0 = fl.long()
        vals = []
        for i in (i0, i0 + 1):
            ok = ((i >= 0) & (i < n)).unsqueeze(1)
            idx = i.clamp(0, n - 1).view(B, 1, 1, H, W).expand(B, Cn, 1, H, W)
            vals.append(torch.gather(data, 2, idx).squeeze(2) * ok)
        taps.append(vals[0] * w0 + vals[1] * w1)
        mags.append((vals[0] * w0).abs() + (vals[1] * w1).abs())
    return torch.stack(taps, 2), torch.stack(mags, 2), cross


def geo_model(vols, corr, disp, coords, r):
    """fp64 model of geo_lookup_kernel.  vols: [(volume (B, C, n, H, W), shift)], each sampled at disp / 2^shift; corr: None (no
    correlation row) or, per vols entry i, (B, H, W, W2 >> i) sampled at coords / 2^i - disp / 2^i.  -> (want (B, len(vols),
    C [+ 1], 2r + 1, H, W), sum |terms|, taps that take the fallback read)."""
    wants, mags, cross = [], [], 0
    for i, (vol, shift) in enumerate(vols):
        sc = f32(1.0 / (1 << shift))
        dq = disp[:, 0] * sc                                                  # (B, H, W)
        rows = [(vol.double(), vol.shape[2], dq)]
        if corr is not None:
            rows.append((corr[i].double().permute(0, 3, 1, 2).unsqueeze(1), corr[i].shape[3], coords * sc - dq))
        parts = [lerp_taps(data, n, base, r) for data, n, base in rows]
        wants.append(torch.cat([p[0] for p in parts], 1))
        mags.append(torch.cat([p[1] for p in parts], 1))
        cross += sum(p[2] for p in parts)
    return torch.stack(wants, 1), torch.stack(mags, 1), cross


def roundtrip_cas(v, half):
    """cascade.cu cas_roundtrip: grid value v/half - 1 and aten's unnormalisation (g + 1) * half, in fp32."""
    g = v / half - f32(1.0)
    return (g + f32(1.0)) * half


def roundtrip_border(v, size):
    """cascade.cu border_roundtrip: the grid value 2 (v / (size - 1)) - 1 in fp32, then fmaf(g + 1, size / 2, -0.5) and the clamp to
    [0, size - 1].  The fmaf's product is exact in fp64 and so is its sum whenever the result is >= 0 (below 0 the clamp takes over),
    so one rounding to fp32 replays it.  -> (coordinate, (clamped below anywhere, clamped above anywhere))."""
    g = f32(2.0) * (v / f32(size - 1)) - f32(1.0)
    u = ((g + f32(1.0)).double() * (size / 2.0) - 0.5).float()
    return u.clamp(0.0, size - 1.0), (bool((u < 0).any()), bool((u > size - 1).any()))


def host_split(x):
    """(..., C) fp32 -> (..., 2C) fp16 split channels-last: per 16-channel granule [16 hi | 16 lo] of s = 16 x, hi = fp16_rn(s),
    lo = fp16_rn(s - hi), each saturating to +-65504."""
    def sat(v):
        h = v.half()
        return torch.where(torch.isinf(h), torch.sign(v).half() * 65504.0, h)
    s = x.contiguous().float() * 16.0
    hi = sat(s)
    lo = sat(s - hi.float())
    lead, C = s.shape[:-1], s.shape[-1]
    both = torch.stack((hi.view(*lead, C // 16, 16), lo.view(*lead, C // 16, 16)), -2)              # (..., granule, hi / lo, 16)
    return both.reshape(*lead, 2 * C)


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
        assert nan[self.skip].all(), "%s: %d elements the launch must leave unwritten were written" % (
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
    """osb_volume_last_variant() of a volume launch: vector stores when W % 4 == 0 and the left inputs and the output are 16-byte
    aligned; TMA staging only for correlation units (gwc) with W % 4 == 0 and an aligned right input.  Concatenation-only launches,
    the interlaced crops among them (K = 0, gwc = False), always stage with plain loads."""
    vec = W % 4 == 0 and y_off == 0 and not {"ref", "rc"} & set(shift)
    tma = gwc and W % 4 == 0 and "tgt" not in shift
    return "volume<%d,%d,%s>" % (vec, K % 4 == 0, "tma" if tma else "ldg")


def disp_mixture(g, shape, lo, hi):
    """Hypotheses: uniform in [lo, hi] (negative and beyond the far edge), exact integers and half-integers."""
    u = lo + (hi - lo) * torch.rand(shape, generator=g)
    pick = torch.rand(shape, generator=g)
    u = torch.where(pick < 0.3, u.round(), u)
    return torch.where((pick >= 0.3) & (pick < 0.45), u.floor() + 0.5, u)


def soft_cost(o, shape, g):
    """Costs of the soft-argmin rows (B, D, H, W): offset + spread x U(-1, 1); peak_last puts the arg-max of every other row of
    pixels in the last bin; inf sets about 40% of the bins to -inf, every pixel keeping bin D // 2 finite."""
    B, D, H, W = shape
    cost = o.get("offset", 0.0) + o.get("spread", 3.0) * (2 * torch.rand(B, D, H, W, generator=g) - 1)
    if o.get("peak_last"):
        cost[:, D - 1, ::2] += 0.5 * o.get("spread", 3.0) + 8.0
    if o.get("inf"):
        hit = torch.rand(B, D, H, W, generator=g) < 0.4
        hit[:, D // 2] = False
        cost = cost.masked_fill(hit, -math.inf)
    return cost


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

    if fam == "crop":
        from oracle.msnet2d import interlaced_crops64
        B, C, H, W, D = row.shape
        rc, tc = per(rn(B, C, H, W), scales(C, g), 1), per(rn(B, C, H, W), scales(C, g), 1)
        want = torch.cat([x.reshape(-1) for x in interlaced_crops64(rc, tc, D)])
        fn = lambda y, P: call("osb_interlaced_crops_fwd", P("rc"), P("tc"), y, B, C, H, W, D, s())     # noqa: E731
        return [Case(row.id, want, None, fn, {"rc": rc, "tc": tc}, exact=torch.ones(want.shape, dtype=torch.bool),
                     info=dict(K=0, W=W, gwc=False))]

    if fam == "var":
        B, D, H, W = row.shape
        n = B * H * W
        cost = soft_cost(o, row.shape, g)
        inputs = {"cost": cost}
        if o.get("values"):                                         # sorted, non-integer, some negative
            lo = 200.0 * torch.rand(B, 1, H, W, generator=g) - 20.0
            inputs["values"] = lo + torch.sort(3.0 * D * torch.rand(B, D, H, W, generator=g), dim=1).values
            v = inputs["values"].double()
        else:
            v = torch.arange(D, dtype=F64).view(1, D, 1, 1).expand(B, D, H, W)
        x = cost.double()                                           # the kernel reads the logits as they are: no rounding
        p = torch.softmax(x, 1)
        mu = (p * v).sum(1)
        dev2 = (v - mu.unsqueeze(1)) ** 2
        var = (p * dev2).sum(1)
        none = torch.zeros_like(x)
        e_mu = soft_model(p, x, v, mu, none, 0)
        # summed about the kernel's mean m: sum p (v - m)^2 = var + (m - mu)^2, and |m - mu| <= TOL_SOFT e_mu
        e_var = soft_model(p, x, dev2, var, none, 0) + TOL_SOFT * e_mu ** 2
        want, scale = torch.stack([mu, var]), torch.stack([e_mu, e_var])
        exact = torch.full(want.shape, D == 1)                      # p = 1: the mean is v_0 and the variance 0, both exact
        no_var = torch.zeros(want.shape, dtype=torch.bool)
        no_var[1] = True                                            # the variance region: a mean-only launch leaves it unwritten

        def vals(P):
            return P("values") if "values" in inputs else None

        def full(y, P):                                             # mean at y, variance after it
            call("osb_softargmin_var_fwd", P("cost"), vals(P), y, y + 4 * n, B, D, H, W, s())

        def mean_only(y, P):
            call("osb_softargmin_var_fwd", P("cost"), vals(P), y, None, B, D, H, W, s())

        def plain(y, P):
            call("osb_softargmin_fwd", P("cost"), y, B, D, H, W, 1.0, 0.0, 1.0, 1, s())
        # same_as: the mean must equal the first case's mean bit for bit
        out = [Case(row.id, want, scale, full, inputs, tol=TOL_SOFT, exact=exact),
               Case(row.id + " var_out NULL", want, scale, mean_only, inputs, tol=TOL_SOFT, exact=exact, skip=no_var,
                    info=dict(same_as=row.id))]
        if "values" not in inputs:                                  # both NULL above: that is the plain kernel's launch
            out.append(Case(row.id + " osb_softargmin_fwd", want, scale, plain, inputs, tol=TOL_SOFT, exact=exact, skip=no_var,
                            info=dict(same_as=row.id)))
        return out

    if fam == "sa":
        B, D, H, W = row.shape
        alpha, start, step, norm = o.get("alpha", 1.0), o.get("start", 0.0), o.get("step", 1.0), o.get("norm", 1)
        cost = soft_cost(o, row.shape, g)
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

    if fam in ("geo", "geov", "geomr"):
        if fam == "geomr":
            B, C, D, D1, D2, H, W, W2, L = row.shape
        elif fam == "geov":
            B, C, D, H, W, L = row.shape
            W2 = 0
        else:
            B, C, D, H, W, W2, L = row.shape
        r = o["radius"]
        T = 2 * r + 1
        geo = [per(rn(B, C, D >> i, H, W), scales(C, g), 1) for i in range(L)]
        corr = [rn(B, H, W, W2 >> i) * 3.1 for i in range(L)] if W2 else None
        coords = torch.arange(W, dtype=torch.float32).view(1, 1, W).expand(B, H, W).contiguous()
        inputs = {"geo%d" % i: geo[i] for i in range(L)}
        gp = lambda P: [P("geo%d" % i) if i < L else None for i in range(4)]           # noqa: E731
        cp = lambda P: [P("corr%d" % i) if i < L else None for i in range(4)]          # noqa: E731
        if corr is not None:
            inputs.update({"corr%d" % i: corr[i] for i in range(L)}, coords=coords)
        if fam == "geomr":                              # half the pixels reach past vol2's far end (disp / 4 > D2 + r)
            near, far = disp_mixture(g, (B, 1, H, W), -6.0, D + 6.0), disp_mixture(g, (B, 1, H, W), -6.0, 4 * max(D, D1, D2) + 8.0)
            disp = torch.where(torch.rand(B, 1, H, W, generator=g) < 0.5, near, far)
        else:
            disp = disp_mixture(g, (B, 1, H, W), -6.0, D + 6.0)
        inputs["disp"] = disp
        want, mag, cross = geo_model([(geo[i], i) for i in range(L)], corr, disp, coords, r)      # (B, L, C [+ 1], T, H, W)
        if fam == "geo":
            want, mag = want.view(B, L * (C + 1) * T, H, W), mag.view(B, L * (C + 1) * T, H, W)

            def fn(y, P):
                call("osb_geo_lookup_fwd", *gp(P), *cp(P), P("disp"), P("coords"), y, B, C, D, H, W, W2, L, r, s())
            out = [Case(row.id, want, mag, fn, inputs)]
        elif fam == "geov":
            want, mag = want.view(B, L * C * T, H, W), mag.view(B, L * C * T, H, W)

            def fn(y, P):
                call("osb_geo_volume_lookup_fwd", *gp(P), P("disp"), y, B, C, D, H, W, L, r, s())
            out = [Case(row.id, want, mag, fn, inputs)]
        else:
            vol1, vol2 = per(rn(B, C, D1, H, W), scales(C, g), 1), per(rn(B, C, D2, H, W), scales(C, g), 1)
            inputs.update(vol1=vol1, vol2=vol2)
            w12, m12, cross12 = geo_model([(vol1, 1), (vol2, 2)], None, disp, None, r)             # (B, 2, C, T, H, W)
            cross += cross12
            q = disp / 4
            assert bool((q - r < -1).any() and (q + r > D2).any()), "%s: vol2's taps do not leave both ends" % row.id
            # geo_feat0 (B, L * C * T, H, W), geo_feat1 and geo_feat2 (B, C * T, H, W), init_corr (B, L * T, H, W)
            outs = [(want[:, :, :C], mag[:, :, :C]), (w12[:, 0], m12[:, 0]), (w12[:, 1], m12[:, 1]), (want[:, :, C], mag[:, :, C])]
            outs = [(w.reshape(B, -1, H, W), m.reshape(B, -1, H, W)) for w, m in outs]
            sizes = [w.numel() for w, _ in outs]
            out = []
            for j, name in enumerate(("geo_feat0", "geo_feat1", "geo_feat2", "init_corr")):
                def fn(y, P, j=j):
                    """Output j at y, the other three in scratch between sentinel guards (their own cases check them)."""
                    scratch = [torch.full((2 * GUARD + n,), SENTINEL, device="cuda") for n in sizes]
                    ys = [y if i == j else scratch[i].data_ptr() + 4 * GUARD for i in range(4)]
                    call("osb_geo_multirange_lookup_fwd", *gp(P), P("vol1"), P("vol2"), *cp(P), P("disp"), P("coords"), *ys,
                         B, C, D, D1, D2, H, W, W2, L, r, s())
                    torch.cuda.synchronize()
                out.append(Case("%s %s" % (row.id, name), outs[j][0], outs[j][1], fn, inputs))
        if o.get("cross"):
            assert cross > 0, "%s: no tap crosses an integer in the coordinate round trip" % row.id
        return out

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
        mask_left = o.get("mask", 1) if Cg else o.get("mask", 0)             # with Cg > 0 it masks the correlation too
        if Cg:
            xg, yg = per(rn(B, Cg, H, W), scales(Cg, g), 1), per(rn(B, Cg, H, W), scales(Cg, g), 1)
            tg, mg = warp(yg)
            xl = xg.double().unsqueeze(2)
            vol = (xl * tg).view(B, G, K, D, H, W).sum(2) / K
            vm = (xl.abs() * mg).view(B, G, K, D, H, W).sum(2) / K
            zeros = masked if mask_left else torch.zeros_like(masked)
            vol = vol.masked_fill(zeros, 0.0)
            parts.append(vol), mags.append(chanmax(vm, 1)), exact.append(zeros.expand(vol.shape))
            inputs.update(xg=xg, yg=yg)
        left = xc.double().unsqueeze(2).expand(B, Cc, D, H, W)
        if mask_left:
            left = left.masked_fill(masked, 0.0)
        tc, mc = warp(yc)
        parts += [left, tc]
        mags += [torch.ones(1, Cc, 1, 1, 1, dtype=F64), chanmax(mc, 1)]
        exact += [torch.ones(left.shape, dtype=torch.bool), torch.zeros(tc.shape, dtype=torch.bool)]
        want = torch.cat(parts, 1)
        scale = torch.cat([m.expand(1, p.shape[1], 1, 1, 1) for m, p in zip(mags, parts)], 1)
        if Cg and "mask" in o:
            fn = lambda y, P: call("osb_warped_gwc_concat_volume_ex_fwd", P("xg"), P("yg"), P("xc"), P("yc"), P("disp"), y, B, Cg,  # noqa
                                   G, Cc, D, H, W, mask_left, s())
        elif Cg:
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

    if fam == "warp":
        B, C, H, W = row.shape
        img = per(rn(B, C, H, W), scales(C, g), 1)
        disp = disp_mixture(g, (B, 1, H, W), -(W // 2) - 3.0, W + W // 2 + 3.0)
        disp[0, 0, 0, 0], disp[-1, 0, -1, -1] = W + 2.5, -W - 1.0            # column coordinates below 0 and past W - 1
        iy, bites_y = roundtrip_border(torch.arange(H, dtype=torch.float32), H)
        fy = torch.floor(iy)
        ny = iy - fy
        assert bool((ny != 0).any()) == bool(o["two"]), "%s: row coordinates do not stage the rows the row expects" % row.id
        ix, bites = roundtrip_border(torch.arange(W, dtype=torch.float32) - disp[:, 0], W)       # (B, H, W)
        assert bites[0] and bites[1], "%s: the border clamp does not bite on both sides" % row.id
        fx = torch.floor(ix)
        wx = ix - fx
        ex, sy = f32(1.0) - wx, (f32(1.0) - ny).view(1, H, 1)
        nyv = ny.view(1, H, 1)
        wts = [sy * ex, sy * wx, nyv * ex, nyv * wx]                          # nw, ne, sw, se in fp32
        want, mag = torch.zeros(B, C, H, W, dtype=F64), torch.zeros(B, C, H, W, dtype=F64)
        for t, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
            yy = (fy.long() + dy).clamp(max=H - 1)                            # row H is only reached with weight 0
            xx = fx.long() + dx                                               # (B, H, W) in [0, W]; column W reads as zero
            rows = img.double()[:, :, yy]                                     # (B, C, H, W)
            v = torch.gather(rows, 3, xx.clamp(max=W - 1).unsqueeze(1).expand(B, C, H, W)) * (xx < W).unsqueeze(1)
            term = v * wts[t].double().unsqueeze(1)
            want += term
            mag += term.abs()
        fn = lambda y, P: call("osb_disp_warp_fwd", P("img"), P("disp"), y, B, C, H, W, s())          # noqa: E731
        return [Case(row.id, want, mag, fn, {"img": img, "disp": disp})]

    if fam == "slice":
        B, C, D, H, W, ys, coff = row.shape
        x = per(rn(B, C, D, H, W), scales(C, g), 1)
        want = torch.zeros(B, D, H, W, ys, dtype=F64)
        want[..., coff:coff + C] = x.permute(0, 2, 3, 4, 1).double()
        inside = torch.zeros(ys, dtype=torch.bool)
        inside[coff:coff + C] = True
        fn = lambda y, P: call("osb_ncdhw_to_ndhwc_slice", P("x"), y, B, C, D, H, W, ys, coff, s())   # noqa: E731
        return [Case(row.id, want, None, fn, {"x": x}, exact=inside, skip=~inside.expand(want.shape))]

    if fam == "split":
        B, C, D, H, W = row.shape
        sat = o.get("sat", 0)
        x = per(rn(B, C, D, H, W), scales(C, g, -24 if sat else -12, 8), 1).clamp(-4000.0, 4000.0)
        if sat:                                            # 16 x 4094 = 65504 is the largest fp16; the others saturate
            x.view(-1)[:6] = torch.tensor([4094.0, -4094.0, 4094.5, -5000.0, 1e6, -1e30])
        want = host_split(x.permute(0, 2, 3, 4, 1)).view(torch.int32).view(torch.float32).double()   # (B, D, H, W, C) words

        def fn(y, P):
            ops.tc_overflow_count(reset=True)
            call("osb_ncdhw_to_split", P("x"), y, B, C, D, H, W, s())
            n = ops.tc_overflow_count(reset=True)
            assert (n >= 1) if sat else (n == 0), "%s: overflow count %d after the conversion" % (row.id, n)
        return [Case(row.id, want, None, fn, {"x": x}, exact=torch.ones(want.shape, dtype=torch.bool))]

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
    if row.fam == "crop":                       # a moved output is refused (test_refusals); a moved left input drops vec_ok
        runs += [("rc+4", {"shift": ("rc",)}, 0), ("tc+4", {"shift": ("tc",)}, 0), ("grid cap 1", {}, 1), ("grid cap 5", {}, 5)]
    if row.fam == "ctx" and case.info["vec"]:
        runs += [("out+4", {"y_off": 1}, 0), ("up+4", {"shift": ("up",)}, 0)]
    return runs


@pytest.mark.timeout(300)
@pytest.mark.parametrize("row", REGISTRY, ids=[r.id for r in REGISTRY])
def test_accuracy_store_paths_bounds_determinism(osb, grid_cap, row):
    _, ops = osb
    worst = 0.0
    firsts = {}
    for case in cases(osb, row, seed(row)):
        first = None
        for label, kw, cap in runs_of(row, case):
            what = "%s, %s" % (case.name, label)
            grid_cap(cap)
            buf, lead = case.launch(**kw)
            if row.fam in ("vol", "crop"):
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
        firsts[case.name] = first
        if "same_as" in case.info:              # the written elements must equal that case's bit for bit
            other, live = firsts[case.info["same_as"]], ~case.skip.flatten()
            assert torch.equal(first[live].view(torch.int32), other[live].view(torch.int32)), "%s: differs bit-wise from %s" % (
                case.name, case.info["same_as"])
    print("\n%-22s %-5s worst err/scale %.2e (bar %g)" % (row.id, row.fam, worst, TOL_SOFT if row.fam in ("sa", "var", "up", "bsa", "coex")
                                                          else (1.0 if row.fam == "epe" else TOL)))


def profiled_kernels(osb, case, what):
    """-> names (spaces removed) of the kernels of this library the profiler saw for one call of case.fn."""
    from torch.profiler import ProfilerActivity, profile
    lib, _ = osb
    dev = case.dev()
    buf = case.guarded()
    names = []
    for _ in range(10):
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
    library as well).  Such sessions can come several in a row (an H100 run of this file once had three empty sessions in a
    row for one row), so only a session with no kernel of this library recorded is repeated, at most ten times; a session
    that records any kernel is judged as it is."""
    names = profiled_kernels(osb, cases(osb, row, seed(row, 3))[0], row.id)
    want = re.compile(r"osb::%s\(" % re.escape(row.variant))
    assert len(names) == 1 and want.search(names[0]), "%s: launched %s, expected %s" % (row.id, names, row.variant)


@pytest.mark.timeout(300)
def test_volume_item_order_0(osb, tmp_path):
    """OSB_VOLUME_ORDER=0 (unit fastest) is read once per process: a child process computes a fused row and a crop row in that
    order, and each output must equal order 1's bit for bit; the crops go through ops.interlaced_crops, whose views must be the
    (B, H, W - d, 2C) images back to back.  subprocess.run waits for the child and kills it on timeout."""
    mine = {}
    for rid in ("vol-fused-k4", "crop-w260-d70"):
        row = BY_ID[rid]
        case = cases(osb, row, seed(row))[0]
        buf, lead = case.launch()
        case.check(buf, lead, "%s, order 1" % rid)
        mine[rid] = buf[lead:lead + case.numel].cpu()
        torch.save({k: v for k, v in case.inputs.items()}, str(tmp_path / ("%s.pt" % rid)))
    B, G, K, Cc, H, W, D = BY_ID["vol-fused-k4"].shape
    cB, cC, cH, cW, cD = BY_ID["crop-w260-d70"].shape
    script = ("import sys, torch\n"
              "from openstereo_b200 import ops\n"
              "t = torch.load(sys.argv[1] + '/vol-fused-k4.pt')\n"
              "c = {k: v.cuda() for k, v in t.items()}\n"
              "out = ops.gwc_concat_volume(c['ref'], c['tgt'], c['rc'], c['tc'], %d, %d)\n"
              "torch.save(out.cpu(), sys.argv[1] + '/vol-fused-k4.out.pt')\n"
              "t = torch.load(sys.argv[1] + '/crop-w260-d70.pt')\n"
              "views = ops.interlaced_crops(t['rc'].cuda(), t['tc'].cuda(), %d)\n"
              "torch.save([v.cpu() for v in views], sys.argv[1] + '/crop-w260-d70.out.pt')\n" % (D, G, cD))
    env = dict(os.environ, OSB_VOLUME_ORDER="0", PYTHONPATH=os.pathsep.join([ROOT] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    res = subprocess.run([sys.executable, "-c", script, str(tmp_path)], env=env, cwd=ROOT, timeout=240, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    other = torch.load(str(tmp_path / "vol-fused-k4.out.pt")).flatten()
    assert torch.equal(other.view(torch.int32), mine["vol-fused-k4"].view(torch.int32)), "fused volume: order 0 and order 1 differ"
    views = torch.load(str(tmp_path / "crop-w260-d70.out.pt"))
    assert [tuple(v.shape) for v in views] == [(cB, cH, cW - d, 2 * cC) for d in range(cD)]
    other = torch.cat([v.flatten() for v in views])
    assert torch.equal(other.view(torch.int32), mine["crop-w260-d70"].view(torch.int32)), "crops: order 0 and order 1 differ"


@pytest.mark.timeout(120)
def test_warped_ex_mask_left_1(osb):
    """osb_warped_gwc_concat_volume_ex_fwd with mask_left = 1 passes the masked cas model and is osb_warped_gwc_concat_volume_fwd
    bit for bit, on both instantiations, with the inputs of the unmasked rows."""
    lib, _ = osb
    for rid in ("cas-gwc-k8-unmasked", "cas-gwc-wmax-unmasked"):
        row = BY_ID[rid]
        B, Cg, G, Cc, D, H, W = row.shape
        case = cases(osb, row._replace(opts=dict(row.opts, mask=1)), seed(row))[0]      # the _ex launch, the masked model
        ex, lead = case.launch()
        case.check(ex, lead, "%s, mask_left = 1" % rid)
        dev = case.dev()
        buf = case.guarded()
        lib.call("osb_warped_gwc_concat_volume_fwd", *(dev[k].data_ptr() for k in ("xg", "yg", "xc", "yc", "disp")),
                 buf.data_ptr() + 4 * GUARD, B, Cg, G, Cc, D, H, W, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert torch.equal(ex.view(torch.int32), buf.view(torch.int32)), "%s: _ex with mask_left = 1 differs from the cascade entry" % rid


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
    gv, l4 = "osb_geo_volume_lookup_fwd", (P,) * 4
    mr = "osb_geo_multirange_lookup_fwd"

    def mrp(vol1=P, out_corr=P):
        """geo0..3, vol1, vol2, corr0..3, disp, coords, out0, out1, out2, out_corr"""
        return (P,) * 4 + (vol1, P) + (P,) * 4 + (P, P, P, P, P, out_corr)
    cx, cg, dw = "osb_warped_concat_volume_fwd", "osb_warped_gwc_concat_volume_fwd", "osb_disp_warp_fwd"
    cgx = "osb_warped_gwc_concat_volume_ex_fwd"
    co = "osb_coex_regression_fwd"
    ic, sv = "osb_interlaced_crops_fwd", "osb_softargmin_var_fwd"
    return [
        ("interlaced_crops C 6", ic, (P, P, P, 1, 6, 2, 16, 4, s)),
        ("interlaced_crops C 184", ic, (P, P, P, 1, 184, 2, 16, 4, s)),            # 237 008 bytes of staged rows
        ("interlaced_crops D 0", ic, (P, P, P, 1, 8, 2, 16, 0, s)),
        ("interlaced_crops D 17 > W 16", ic, (P, P, P, 1, 8, 2, 16, 17, s)),
        ("interlaced_crops out+4", ic, (P, P, mis, 1, 8, 2, 16, 4, s)),
        ("interlaced_crops null right", ic, (P, None, P, 1, 8, 2, 16, 4, s)),
        ("softargmin_var null cost", sv, (None, None, P, P, 1, 4, 2, 2, s)),
        ("softargmin_var null output", sv, (P, None, None, P, 1, 4, 2, 2, s)),
        ("softargmin_var D 0", sv, (P, None, P, P, 1, 0, 2, 2, s)),
        ("softargmin_var empty B", sv, (P, P, P, None, 0, 4, 2, 2, s)),
        ("warped_gwc_ex mask_left 2", cgx, (P, P, P, P, P, P, 1, 16, 2, 4, 2, 4, 8, 2, s)),
        ("warped_gwc_ex K 17", cgx, (P, P, P, P, P, P, 1, 17, 1, 4, 2, 4, 8, 0, s)),
        ("warped_gwc_ex W 1817", cgx, (P, P, P, P, P, P, 1, 16, 1, 1, 2, 2, 1817, 0, s)),

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
        ("geo_lookup B*L*(C+1) 65536", geo, lv + (P, P, P, 256, 255, 64, 2, 8, 64, 1, 4, s)),
        ("geo_volume_lookup 0 levels", gv, l4 + (P, P, 1, 2, 16, 2, 8, 0, 4, s)),
        ("geo_volume_lookup 5 levels", gv, l4 + (P, P, 1, 2, 64, 2, 8, 5, 4, s)),
        ("geo_volume_lookup radius 17", gv, l4 + (P, P, 1, 2, 64, 2, 8, 2, 17, s)),
        ("geo_volume_lookup radius -1", gv, l4 + (P, P, 1, 2, 64, 2, 8, 2, -1, s)),
        ("geo_volume_lookup D pyramid", gv, l4 + (P, P, 1, 2, 7, 2, 8, 3, 4, s)),
        ("geo_volume_lookup null level", gv, (P, None, P, P, P, P, 1, 2, 64, 2, 8, 2, 4, s)),
        ("geo_volume_lookup empty", gv, l4 + (P, P, 1, 2, 64, 0, 8, 2, 4, s)),
        ("geo_volume_lookup B*L*C 65536", gv, l4 + (P, P, 16, 1024, 16, 2, 8, 4, 4, s)),
        ("geo_multirange D1 1", mr, mrp() + (1, 2, 64, 1, 8, 2, 8, 64, 2, 4, s)),
        ("geo_multirange D2 1", mr, mrp() + (1, 2, 64, 8, 1, 2, 8, 64, 2, 4, s)),
        ("geo_multirange null vol1", mr, mrp(vol1=None) + (1, 2, 64, 8, 8, 2, 8, 64, 2, 4, s)),
        ("geo_multirange null out_corr", mr, mrp(out_corr=None) + (1, 2, 64, 8, 8, 2, 8, 64, 2, 4, s)),
        ("geo_multirange W2 pyramid", mr, mrp() + (1, 2, 64, 8, 8, 2, 8, 7, 3, 4, s)),
        ("geo_multirange radius 17", mr, mrp() + (1, 2, 64, 8, 8, 2, 8, 64, 2, 17, s)),
        ("geo_multirange grid z 65536", mr, mrp() + (256, 85, 64, 8, 8, 2, 8, 64, 1, 4, s)),       # 256 x (85 + 170 + 1)
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
        ("disp_warp H 1", dw, (P, P, P, 1, 4, 1, 16, s)),
        ("disp_warp W 1", dw, (P, P, P, 1, 4, 2, 1, s)),
        ("disp_warp W 3633", dw, (P, P, P, 1, 1, 2, 3633, s)),
        ("disp_warp C 0", dw, (P, P, P, 1, 0, 2, 16, s)),
        ("disp_warp empty B", dw, (P, P, P, 0, 4, 2, 16, s)),
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
        ("ncdhw_to_ndhwc_slice B 65536", "osb_ncdhw_to_ndhwc_slice", (P, P, 65536, 4, 1, 2, 2, 4, 0, s)),
        ("ncdhw_to_split C 24", "osb_ncdhw_to_split", (P, P, 1, 24, 1, 2, 2, s)),
        ("ncdhw_to_split B 65536", "osb_ncdhw_to_split", (P, P, 65536, 16, 1, 2, 2, s)),
    ]


@pytest.mark.timeout(60)
def test_refusals(osb):
    lib, ops = osb
    buf = torch.zeros(1 << 20, device="cuda")                   # 4 MB: every argument list above stays inside it
    torch.cuda.synchronize()
    s = torch.cuda.current_stream().cuda_stream
    for what, name, args in refusals(buf.data_ptr(), s):
        before = lib.launch_count()
        rc = getattr(lib.lib, name)(*args)
        assert rc == OSB_EINVAL, "%s: %s returned %d, expected %d (%s)" % (what, name, rc, OSB_EINVAL, lib.lib.osb_last_error())
        assert lib.launch_count() == before, "%s: a refused call launched a kernel" % what
    small = torch.zeros(1, 8, 2, 16, device="cuda")
    for c, nd in ((184, 4), (6, 4), (8, 0), (8, 17)):           # ops.interlaced_crops refuses the same shapes before any launch
        before = lib.launch_count()
        with pytest.raises(ValueError, match="interlaced_crops"):
            ops.interlaced_crops(small.new_zeros(1, c, 2, 16), small.new_zeros(1, c, 2, 16), nd)
        assert lib.launch_count() == before, "ops.interlaced_crops C %d ndisp %d launched a kernel" % (c, nd)
    # a valid launch after every refusal: OSB_OK, so no refused call left a CUDA error for the next launch's check to report
    before = lib.launch_count()
    rc = lib.lib.osb_interlaced_crops_fwd(small.data_ptr(), small.data_ptr(), buf.data_ptr(), 1, 8, 2, 16, 4, s)
    assert rc == OSB_OK, "a valid launch after the refusals returned %d (%s)" % (rc, lib.lib.osb_last_error())
    assert lib.launch_count() == before + 1
    torch.cuda.synchronize()
