/*
 * openstereo_b200.h -- C ABI of the H100-native cost-volume hot path for OpenStereo.
 *
 * Drop-in boundary.  The reference (XiandaGuo/OpenStereo) has no operator registry: the hot path is
 * a set of plain Python callables on torch.Tensor (SURVEY.md section 8b).  The reference's own
 * convention for native ops is "a compiled extension called from a thin Python wrapper on the
 * current CUDA stream" (stereo/libs/AANet/deform_conv/deform_conv.py:9,44-56;
 * stereo/modeling/models/nmrf/ops/functions/ms_deform_attn_func.py:11-47).  This header is that
 * extension's surface, expressed as a C ABI: plain device pointers, sizes and a stream handle --
 * no torch types.  openstereo_b200/ops.py binds it with ctypes; INTEGRATION.md shows the stub a
 * reference maintainer would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to dense fp32 data in the reference's layout
 *     (NCHW features, NCDHW volumes), unless the name ends in _host;
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream);
 *   - inputs are borrowed and never written; outputs are caller-allocated;
 *   - return value 0 = success, otherwise an OSB_E* code; osb_last_error() returns a
 *     thread-local message.  Nothing falls back to a CPU path: without a CUDA device every
 *     compute entry point fails with OSB_ECUDA.
 */
#ifndef OPENSTEREO_B200_H_
#define OPENSTEREO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OSB_OK 0
#define OSB_EINVAL 1  /* bad shape / argument (the reference raises AssertionError / ValueError) */
#define OSB_ECUDA 2   /* CUDA runtime / driver error, incl. "no device" */
#define OSB_EUNSUPPORTED 3

#define OSB_ACT_NONE 0
#define OSB_ACT_RELU 1
#define OSB_ACT_LEAKY 2 /* LeakyReLU(0.01), nn.LeakyReLU default used by StereoBase */
#define OSB_ACT_RELU6 3 /* nn.ReLU6 of LightStereo's MobileV2Residual; accepted by the CUDA-core 1x1, depthwise and 2D kernels */
#define OSB_ACT_SIGMOID 4 /* the ConvGRU gates (torch.sigmoid / torch.tanh); accepted by osb_conv2d_k3_tc_gru_fwd */
#define OSB_ACT_TANH 5
/* CFNet's Mish, v * tanh(softplus(v)) with F.softplus's threshold 20 (cfnet/submodule.py:249-260), applied after the residual:
 * FMish(conv(x) + redir(y)) is one launch.  Accepted by osb_conv3d_k3_bn_act_fwd, osb_deconv3d_bn_act_fwd and
 * osb_conv3d_1x1_bn_act_fwd only; every other entry point returns OSB_EINVAL for it. */
#define OSB_ACT_MISH 6

/* Precision of the tensor-core products (osb_conv2d_k3_tc_prec_fwd, osb_conv2d_k3_tc_gru_prec_fwd) */
#define OSB_PREC_FP32 0 /* fp32-accurate 3xFP16 split products (the default of every other entry point) */
#define OSB_PREC_F16 1  /* one fp16 MMA per product, a_hi * b_hi: autocast precision (DESIGN.md section 4.20) */

typedef void* osb_stream_t;

int osb_abi_version(void);
const char* osb_last_error(void);
/* Number of kernels this library has launched in this process (bench.py reports it). */
uint64_t osb_launch_count(void);
/* fp16 range guard of the tensor-core convolutions.  They compute every fp32 product as three kind::f16 MMAs on operands split
 * into fp16 (hi, lo) pairs (csrc/tc_common.cuh): activations are staged as x * 16, so |x| must stay below 65504 / 16 = 4094
 * (weights are pre-scaled per output channel on the host and cannot overflow).  Conversions saturate and every loader thread
 * that met a larger value increments a sticky per-device counter.  osb_tc_overflow_count copies it to *count (host memory),
 * optionally resets it, and synchronises `stream`; osb_tc_overflow_flag returns its device address (for an asynchronous read). */
int osb_tc_overflow_count(osb_stream_t stream, int reset, unsigned int* count);
/* Asynchronous variant: enqueue a 4-byte copy of the counter into PINNED host memory on `stream` and return at once (the caller
 * reads *host_pinned after an event recorded behind it has completed; the Python engines do that at the start of their next call). */
int osb_tc_overflow_poll(osb_stream_t stream, unsigned int* host_pinned);
const unsigned int* osb_tc_overflow_flag(void);
/* Expected round-towards-zero loss per accumulating tensor-core MMA, undone by the conv epilogues (csrc/tc_common.cuh: rz_kappa;
 * DESIGN.md section 2.1).  Process-wide; returns the previous value; 0 switches the correction off; values outside [0, 1e-6) are
 * ignored.  The default 1.57e-8 is calibrated on the H100 (DESIGN.md section 2.1: it removes 87-100 % of the layer-level bias
 * against fp64).  The setter exists for calibration and tests (tools/parity_bisect.py, tests/test_tc_contract_gpu.py). */
float osb_set_rz_kappa(float kappa);
/* Test hooks of the persistent kernels (the tensor-core convolutions, the volume constructors and the grid-stride channels-last
 * 1x1 convolutions osb_conv1x1_ndhwc_fwd / osb_conv1x1_ndhwc_cat_fwd), process-wide.
 * osb_set_persistent_grid_cap clamps their grid to `cap` CTAs (0 = no cap, the default: one CTA per resident slot) and returns the
 * previous cap.  Every CTA walks the work items it = blockIdx.x, blockIdx.x + gridDim.x, ..., so cap = 1 makes one CTA compute every
 * item in order; an item's result does not depend on the CTA that computes it, so outputs are bit-identical for any cap.
 * osb_tc_last_variant returns the template arguments of the tensor-core instantiation this thread launched last, e.g.
 * "tcg<64,16,64,1,1,0,1>" (COUT, KC, W, TILES, DIL, GW, GATE), "tc<32>", "tcs2<...>", "tcdc<...>"; "" before the first launch. */
int osb_set_persistent_grid_cap(int cap);
const char* osb_tc_last_variant(void);
/* The cost-volume kernel this thread launched last, as "volume<VEC,K4,STAGE>": VEC = 1 for 16-byte loads and stores of the left
 * features and the output (W % 4 == 0, ref and out 16-byte aligned), K4 = 1 when the channels per group are a multiple of 4
 * (or the volume is concatenation only), STAGE = tma when the right features are staged by TMA tile loads (W % 4 == 0, tgt
 * 16-byte aligned), ldg when by plain loads; "" before the first launch. */
const char* osb_volume_last_variant(void);

/* ---------------------------------------------------------------- cost-volume constructors --- */

/* build_gwc_volume(refimg_fea, targetimg_fea, maxdisp, num_groups)
 *   stereo/modeling/cost_volume/cost_volume.py:68-78, gwcnet/gwcnet_cost_processor.py:22-39
 * ref,tgt: (B,C,H,W) -> out: (B,G,D,H,W); out[b,g,d,h,w] = mean_k ref[b,gK+k,h,w]*tgt[b,gK+k,h,w-d]
 * for w >= d, exact 0 otherwise.  C % G != 0 -> OSB_EINVAL (reference: assert, cost_volume.py:61). */
int osb_gwc_volume_fwd(const float* ref, const float* tgt, float* out, int B, int C, int H, int W,
                       int D, int G, osb_stream_t stream);

/* build_concat_volume(refimg_fea, targetimg_fea, maxdisp)   cost_volume.py:81-92
 * == cat_fms(start_disp=0, dilation=1)                       psmnet/psmnet_cost_processor.py:9-50
 * out: (B,2C,D,H,W).  mask_left=1: canonical form (left half zero for w<d);
 * mask_left=0: IGEV-family form (igev/submodule.py:216-227). */
int osb_concat_volume_fwd(const float* ref, const float* tgt, float* out, int B, int C, int H,
                          int W, int D, int mask_left, osb_stream_t stream);

/* GwcVolumeCostProcessor.forward: torch.cat((gwc, concat), 1) written in ONE pass
 *   gwcnet/gwcnet_cost_processor.py:55-68, stereobase/stereobase_gru.py:142-160
 * out: (B, G + 2*Cc, D, H, W). */
int osb_gwc_concat_volume_fwd(const float* ref_gwc, const float* tgt_gwc, const float* ref_cat,
                              const float* tgt_cat, float* out, int B, int Cg, int Cc, int H, int W,
                              int D, int G, osb_stream_t stream);

/* correlation_volume(left, right, max_disp)   cost_volume.py:32-41   out: (B,D,H,W) */
int osb_corr_volume_fwd(const float* left, const float* right, float* out, int B, int C, int H,
                        int W, int D, osb_stream_t stream);

/* MSNet2D's per-disparity inputs (msnet/MSNet2D.py:145-159: interweave_tensors(featL[..., d:], featR[..., :-d])), cropped and
 * channels-last, written by the concat path of the volume kernel: for d = 0 .. D-1 the image
 *     out_d[b, h, w - d, 8j + k]     = left[b, 4j + k, h, w]
 *     out_d[b, h, w - d, 8j + 4 + k] = right[b, 4j + k, h, w - d]        (w = d .. W-1, j < C/4, k < 4)
 * of shape (B, H, W - d, 2C), the D images back to back (image d starts at B*H*2C*(d*W - d*(d-1)/2) floats).  Block j holds the
 * four left and four right channels that the reference's interleave puts at depths 8j .. 8j+7, left first.  C % 4 == 0,
 * C <= 180 (a CTA stages one left and one right row per channel, 1288 C + 16 bytes of shared memory, 227 KB at most),
 * 1 <= D <= W, out 16-byte aligned.  The columns w < d are not stored anywhere: each image is exactly the reference's crop. */
int osb_interlaced_crops_fwd(const float* left, const float* right, float* out, int B, int C, int H, int W, int D,
                             osb_stream_t stream);

/* ------------------------------------------------------------------------ soft-argmin tails --- */

/* softmax over D fused with the expectation (one pass over the cost):
 *   disparity_regression(F.softmax(x,1), D)    disp_pred/disp_regression.py:8-12,
 *                                              gwcnet/gwcnet_disp_processor.py:22-26
 *   FasterSoftArgmin.forward                   psmnet/psmnet_disp_processor.py:51-74
 * cost: (B,D,H,W) -> out: (B,H,W); sample value of bin d is start + d*step; cost is multiplied by
 * alpha first; normalize=0 skips the softmax (sum_d cost*value). */
int osb_softargmin_fwd(const float* cost, float* out, int B, int D, int H, int W, float alpha,
                       float start, float step, int normalize, osb_stream_t stream);

/* Soft-argmin with the candidates' values and the variance of the distribution (CFNet, cfnet/cfnet.py:526-566,
 * cfnet/submodule.py:121-141): p = softmax over D of cost (B,D,H,W),
 *   disp_out[b,h,w] = mu = sum_d p_d v_d,   var_out[b,h,w] = sum_d p_d (v_d - mu)^2   (disparity_variance(_confidence))
 * with v_d = values[b,d,h,w] (CFNet's disparity samples), or v_d = d when values is NULL.  var_out may be NULL (no variance);
 * the variance is a second pass over the cost about the mu of the same launch.  With values and var_out NULL, disp_out is
 * osb_softargmin_fwd(cost, disp_out, B, D, H, W, 1, 0, 1, 1) bit for bit.  disp_out / var_out: (B,H,W) = (B,1,H,W). */
int osb_softargmin_var_fwd(const float* cost, const float* values, float* disp_out, float* var_out, int B, int D, int H, int W,
                           osb_stream_t stream);

/* F.interpolate(cost,[D,H,W],'trilinear',align_corners) -> softmax(dim=1) -> expectation, fused;
 * the upsampled (B,D,H,W) tensor is never materialised.
 *   gwcnet/gwcnet_disp_processor.py:129-133 (align_corners=0)
 *   psmnet/psmnet_cost_processor.py:203-214 + psmnet_disp_processor.py:64-73 (align_corners=1)
 * cost: (B,1,Dl,Hl,Wl) -> out: (B,H,W). */
int osb_upsample_softargmin_fwd(const float* cost, float* out, int B, int Dl, int Hl, int Wl, int D,
                                int H, int W, int align_corners, osb_stream_t stream);

/* osb_upsample_softargmin_fwd with per-pixel hypothesis values: the expectation is sum_d p[b,d,h,w] * values[b,d,h,w]
 * instead of sum_d p * d.  CasStereo's CostAggregation eval tail (casnet/cas_psm.py:268-274, cas_gwc.py:245-251):
 * F.upsample(cost3, [D,H,W], 'trilinear', align_corners) -> softmax(dim=1) -> disparity_regression(p, values).
 * cost: (B,1,Dl,Hl,Wl), values: (B,D,H,W) -> out: (B,H,W). */
int osb_upsample_softargmin_values_fwd(const float* cost, const float* values, float* out, int B, int Dl, int Hl, int Wl,
                                       int D, int H, int W, int align_corners, osb_stream_t stream);

/* epe_metric partial sums   stereo/evaluation/metric_per_image.py:32-41 with the eval mask of
 * trainer_template.py:288 (0 < gt < maxdisp).  out: (B,2) = {sum |pred-gt| over valid, #valid}. */
int osb_epe_partial_fwd(const float* pred, const float* gt, float* out, int B, int HW, float maxdisp,
                        osb_stream_t stream);

/* ------------------------------------------------------------------------- 3D aggregation ----- */

/* Conv3d(k=3, pad=1, stride in {1,2}, bias=False) + folded eval BatchNorm3d + optional residual +
 * activation + optional channel gate:
 *     y = act( conv(x) * scale[co] + shift[co] + residual ) * gate[b,co,h,w]
 *   convbn_3d gwcnet/hourglass.py:5-16; conv3d_bn(_relu) psmnet/submodule.py:68-83,160-177;
 *   BasicConv3d common/basic_block_3d.py:5-20; FeatureAtt stereobase/igev_blocks.py:35-48.
 * x: (B,Cin,D,H,W); w_packed: (Cin,27,Cout) = weight.permute(1,2,3,4,0) of the (Cout,Cin,3,3,3)
 * parameter; scale/shift: (Cout) or NULL (= 1 / 0); residual: like y or NULL;
 * gate: (B,Cout,Ho,Wo) already sigmoid-ed, or NULL.  y: (B,Cout,Do,Ho,Wo), Do=(D-1)/stride+1. */
int osb_conv3d_k3_bn_act_fwd(const float* x, const float* w_packed, const float* scale,
                             const float* shift, const float* residual, const float* gate, float* y,
                             int B, int Cin, int Cout, int D, int H, int W, int stride, int act,
                             osb_stream_t stream);

/* ConvTranspose3d(stride=2, bias=False) + folded BN + residual + activation.
 *   kernel=3: padding=1, output_padding=1 (gwcnet/hourglass.py:35-41, psmnet deconv3d_bn)
 *   kernel=4: padding=1                   (stereobase/hourglass.py:39-49)
 * x: (B,Cin,D,H,W) -> y: (B,Cout,2D,2H,2W); w_packed: (Cin,k^3,Cout) = weight.permute(0,2,3,4,1)
 * of the (Cin,Cout,k,k,k) parameter. */
int osb_deconv3d_bn_act_fwd(const float* x, const float* w_packed, const float* scale,
                            const float* shift, const float* residual, float* y, int B, int Cin,
                            int Cout, int D, int H, int W, int kernel, int act, osb_stream_t stream);

/* Conv3d(k=1) + folded BN + residual + activation + gate (redir1/2 gwcnet/hourglass.py:43-44,
 * agg_0[0]/agg_1[0] stereobase/hourglass.py:51-66).  Also serves the 2D 1x1 convs of FeatureAtt
 * with D=1.  x may be given as two channel slabs (x0: Cin0 channels, x1: Cin-Cin0 channels) so the
 * torch.cat of stereobase/hourglass.py:91,96 is never materialised; x1 NULL -> single input.
 * w_packed: (Cin,Cout).  sigmoid_out=1 applies a final sigmoid (FeatureAtt gate). */
int osb_conv3d_1x1_bn_act_fwd(const float* x0, const float* x1, int Cin0, const float* w_packed,
                              const float* scale, const float* shift, const float* residual,
                              const float* gate, float* y, int B, int Cin, int Cout, int D, int H,
                              int W, int act, int sigmoid_out, osb_stream_t stream);

/* Instance-normalised variants of the three convolutions above (IGEV++'s BasicConv: conv -> InstanceNorm -> LeakyReLU(0.01),
 * igevpp/submodule.py:8-34), same kernels and instantiations.  Two modes, each on when its pointers are given:
 *   normalised input: every in-bounds input element of channel c is staged as
 *       leaky((x - in_stats[b,c,0]) * in_stats[b,c,1]) * in_gate[b,c,h,w]        (in_gate NULL: no gate; broadcast over D)
 *     and out-of-bounds taps stay 0 (the reference pads the normalised, gated tensor).  The 1x1 takes one pair per slab.
 *   moments out: y is stored raw (scale, shift, act and sigmoid_out must be 0 / NULL) and stats_out[b,co] = (mean, 1/sqrt(var +
 *     1e-5)) of y over D*H*W, biased variance as F.instance_norm, computed in the same launch: per-CTA partials (count, sum, M2)
 *     in their own workspace slots, merged in slot order (Chan et al.) by the last CTA of each (b, channel block).
 * in_stats / stats_out: (B, C, 2) fp32, 8-byte aligned.  workspace: workspace_floats >= osb_conv3d_in_workspace_floats(...)
 * floats, 16-byte aligned, zero-filled before its first use (its counters return to 0 after every launch).  Where the counters
 * sit depends on the op and the shapes, so a workspace may only be reused by launches of the same op and shapes, and never by
 * launches that may run concurrently.  D*H*W of the output <= 2^24. */
int osb_conv3d_k3_in_fwd(const float* x, const float* w_packed, const float* scale, const float* shift,
                         const float* in_stats, const float* in_gate, float* y, float* stats_out, float* workspace,
                         long long workspace_floats, int B, int Cin, int Cout, int D, int H, int W, int stride, int act,
                         osb_stream_t stream);
int osb_deconv3d_in_fwd(const float* x, const float* w_packed, const float* scale, const float* shift,
                        const float* in_stats, const float* in_gate, float* y, float* stats_out, float* workspace,
                        long long workspace_floats, int B, int Cin, int Cout, int D, int H, int W, int kernel, int act,
                        osb_stream_t stream);
int osb_conv3d_1x1_in_fwd(const float* x0, const float* x1, int Cin0, const float* w_packed, const float* scale,
                          const float* shift, const float* in_stats0, const float* in_gate0, const float* in_stats1,
                          const float* in_gate1, float* y, float* stats_out, float* workspace, long long workspace_floats,
                          int B, int Cin, int Cout, int D, int H, int W, int act, int sigmoid_out, osb_stream_t stream);
/* Workspace (floats) the moments-out launch of op 0 = osb_conv3d_k3_in_fwd (param = stride), 1 = osb_deconv3d_in_fwd (param =
 * kernel) or 2 = osb_conv3d_1x1_in_fwd (param ignored) needs for INPUT extents D, H, W; -1 for invalid arguments. */
int osb_conv3d_in_workspace_floats(int op, int B, int Cout, int D, int H, int W, int param);

/* ------------------------------------------------------- tensor-core (wgmma) variant of the 3x3x3 conv ----- */

/* Same operator as osb_conv3d_k3_bn_act_fwd (stride 1) for the full-resolution layers, computed on the Hopper (wgmma) tensor
 * cores with 3xFP16 operand splitting (fp32-accurate, see csrc/tc_common.cuh, conv3d_tc.cu, conv3d_tcg.cu).  Supported shapes:
 * osb_conv3d_tc_supported / osb_conv3d_tc_kc.  x is CHANNELS-LAST (B,D,H,W,Cin) fp32; w_split is the host-split fp16 weight
 * tensor [3 kd][Cin/kc][3 kh][3*Cout (kw-major)][kc hi | kc lo] of w * 2^e_c (ops.pack_tc_weight; e_c per output channel);
 * `scale` (REQUIRED here, Cout floats) must already contain the exact inverse 2^-(e_c + 4) times the folded-BN scale
 * (TcWeight.eff_scale).  y and residual are fp32, NCDHW or NDHWC according to out_ndhwc / res_ndhwc. */
int osb_conv3d_tc_supported(int Cin, int Cout, int W, int stride);
/* General widths: every W >= OSB_TC_MIN_WIDTH that has no whole-row variant is served by 128-column tiles of one image row with a
 * one-column halo (conv3d_tcg.cu / conv3d_tcs2.cu / conv3d_tcdc.cu, GW instantiations): 240 (the reference's 544x960 timing shape,
 * tools/measure.py:32), 312 (KITTI), 160 (IGEV) ... -- stride 1: Cout 32|64|128; stride 2: Cout 64|128; transposed: Cout 32|64. */
#define OSB_TC_MIN_WIDTH 24
int osb_tc_general_width(int W);
/* K chunk (16 or 32 input channels per operand tile) the weight tensor must be packed with; 0 = unsupported shape.
 * Variants: W=128/Cout=32 (kc 32); W=64/Cout=64, W=32/Cout=64|128 (kc 16, M tile = 128/W image rows); general widths (kc 16). */
int osb_conv3d_tc_kc(int Cin, int Cout, int W, int stride);
int osb_conv3d_k3_tc_fwd(const float* x_ndhwc, const void* w_split, const float* scale, const float* shift,
                         const float* residual, float* y, int B, int Cin, int Cout, int D, int H, int W, int act,
                         int out_ndhwc, int res_ndhwc, osb_stream_t stream);
/* Same with FeatureAtt's gate fused: y = act(bn(conv(x)) + residual) * gate, gate_nhwc (B,H,W,Cout) = sigmoid(att) broadcast over D
 * (stereobase/hourglass.py:80-99, igev_blocks.py:35-48).  Channels-last y / residual, 16-channel-chunk variants only. */
int osb_conv3d_k3_tc_gate_fwd(const float* x_ndhwc, const void* w_split, const float* scale, const float* shift,
                              const float* residual, const float* gate_nhwc, float* y, int B, int Cin, int Cout, int D, int H, int W,
                              int act, osb_stream_t stream);
/* Same, reading an NCDHW input (B,Cin,D,H,W) -- the cost volume exactly as osb_gwc_concat_volume_fwd / build_*_volume return it --
 * so the first aggregation layer needs no layout-conversion pass.  Served by the W = 128 variant (Cout = 32 or <= 16). */
int osb_conv3d_k3_tc_ncdhw_fwd(const float* x_ncdhw, const void* w_split, const float* scale, const float* shift,
                               const float* residual, float* y, int B, int Cin, int Cout, int D, int H, int W, int act,
                               int out_ndhwc, int res_ndhwc, osb_stream_t stream);
/* Split NDHWC activations: a channels-last (B,D,H,W,C) tensor stored as (B,D,H,W,2C) fp16 -- the bytes of the fp32 tensor, so
 * the pointers below are typed float* --, per voxel granules of 16 channels [16 hi | 16 lo] with hi = fp16_rn(16x),
 * lo = fp16_rn(16x - hi) (saturating; a value outside +-4094 raises the overflow count of osb_tc_overflow_count).  The W = 128
 * wgmma layers read it with TMA tensor copies and write it from their epilogues, so that layers chained through it skip the
 * conversion of their input; a split residual is read as (hi + lo) / 16.  Layout codes: */
#define OSB_LAYOUT_NCDHW 0
#define OSB_LAYOUT_NDHWC 1
#define OSB_LAYOUT_SPLIT 2
/* NCDHW fp32 (B,C,D,H,W) -> split NDHWC, C a multiple of 16. */
int osb_ncdhw_to_split(const float* x, float* y_split, int B, int C, int D, int H, int W, osb_stream_t stream);
/* osb_conv3d_k3_tc_fwd / _ncdhw_fwd with each of x, y and residual in any of the layouts above (W = 128; Cout = 32 for a split
 * y or residual; a split y needs a channels-last residual). */
int osb_conv3d_k3_tc_split_fwd(const float* x, const void* w_split, const float* scale, const float* shift, const float* residual,
                               float* y, int B, int Cin, int Cout, int D, int H, int W, int act, int in_layout, int out_layout,
                               int res_layout, osb_stream_t stream);
/* Stride-2 variant (the down-sampling convs of the hourglasses): x (B,D,H,W,Cin) channels-last with even D,H,W ->
 * y (B,Cout,D/2,H/2,W/2) or channels-last.  D = 1 is a stride-2 3x3 Conv2d (the backbone's stage entry): one output plane from
 * the kd = 1 taps.  w_split like above but with the kw slices stored in the order (1,0,2)
 * (ops.pack_tc_weight(..., kw_order=(1,0,2))), 16-channel K chunks.  Supported: W=128/Cout=64, W=64/Cout=64|128. */
int osb_conv3d_s2_tc_supported(int Cin, int Cout, int D, int H, int W);
int osb_conv3d_k3_s2_tc_fwd(const float* x_ndhwc, const void* w_split, const float* scale, const float* shift,
                            const float* residual, float* y, int B, int Cin, int Cout, int D, int H, int W, int act,
                            int out_ndhwc, int res_ndhwc, osb_stream_t stream);
/* ConvTranspose3d(k=3, stride=2, padding=1, output_padding=1) on the tensor cores: x (B,D,H,W,Cin) channels-last ->
 * y (B,Cout,2D,2H,2W) or channels-last.  w_split = ops.pack_tc_deconv_weight(weight): the (Cin,Cout,3,3,3) parameter split
 * hi/lo (fp16), 16-channel K chunks, kw slices stored as (1,2,0).  Supported: W=32/Cout=64 (conv5), W=64/Cout=32 (conv6). */
int osb_deconv3d_tc_supported(int Cin, int Cout, int W);
int osb_deconv3d_k3_tc_fwd(const float* x_ndhwc, const void* w_split, const float* scale, const float* shift,
                           const float* residual, float* y, int B, int Cin, int Cout, int D, int H, int W, int act,
                           int out_ndhwc, int res_ndhwc, osb_stream_t stream);
/* ConvTranspose3d(k=4, stride=2, padding=1) on the tensor cores -- BasicDeconv3d of StereoBase's hourglass
 * (stereobase/hourglass.py:35-60 conv3_up / conv2_up / conv1_up): x (B,D,H,W,Cin) channels-last -> y (B,2D,2H,2W,Cout) channels-last
 * or (B,cout_real,2D,2H,2W).  w_split = ops.pack_tc_deconv_weight of the (Cin,Cout,4,4,4) parameter, kw slices stored as (1,3,2,0).
 * Cout is the PACKED channel count (zero-padded channel plans: 24 -> 32, 48 -> 64); cout_real <= Cout real channels are written /
 * added when the output / residual is NCDHW.  Supported: W=32/Cout=64, W=64/Cout=32, W=16/Cout=64|32. */
int osb_deconv3d_k4_tc_supported(int Cin, int Cout, int W);
int osb_deconv3d_k4_tc_fwd(const float* x_ndhwc, const void* w_split, const float* scale, const float* shift,
                           const float* residual, float* y, int B, int Cin, int Cout, int cout_real, int D, int H, int W, int act,
                           int out_ndhwc, int res_ndhwc, osb_stream_t stream);
/* Channel-SLICE variants (suffix _cs): the launch computes Cout consecutive channels of a wider channels-last tensor whose voxels
 * hold `ystride` >= Cout floats; y (and residual / gate_nhwc) point at the slice's first channel.  Channel plans whose kw-stacked
 * N = 3*Cout (4*Cout for the k4 transposed conv) exceeds what one CTA can hold -- StereoBase's 6c = 144 (run as 160 = 96 + 64) --
 * are produced by two launches over output-channel slices of separately packed weights.  Channels-last in and out. */
int osb_conv3d_k3_tc_cs_fwd(const float* x_ndhwc, const void* w_split, const float* scale, const float* shift, const float* residual,
                            const float* gate_nhwc, float* y, int B, int Cin, int Cout, int D, int H, int W, int act, int ystride,
                            osb_stream_t stream);
int osb_conv3d_k3_s2_tc_cs_fwd(const float* x_ndhwc, const void* w_split, const float* scale, const float* shift, float* y, int B,
                               int Cin, int Cout, int D, int H, int W, int act, int ystride, osb_stream_t stream);
int osb_deconv3d_k4_tc_cs_fwd(const float* x_ndhwc, const void* w_split, const float* scale, const float* shift, float* y, int B,
                              int Cin, int Cout, int D, int H, int W, int act, int ystride, osb_stream_t stream);
/* Channels-last 1x1x1 conv over the channel concatenation of two tensors (torch.cat((up, skip), 1) -> Conv3d(k=1) of
 * stereobase/hourglass.py:91-92,96-97, never materialised): x0 (voxels,C0), x1 (voxels,C1) or NULL -> y (voxels,Cout);
 * w_packed (C0+C1, Cout).  192 -> 96 and 128 -> 64. */
int osb_conv1x1_ndhwc_cat_fwd(const float* x0, const float* x1, int C0, int C1, const float* w_packed, const float* scale,
                              const float* shift, float* y, long long voxels, int Cout, int act, osb_stream_t stream);
/* Channels-last 1x1x1 conv + folded BN + activation (the redir branches when the aggregation runs channels-last):
 * x (voxels, Cin) -> y (voxels, Cout); w_packed (Cin, Cout).  32->32 and 64->64. */
int osb_conv1x1_ndhwc_fwd(const float* x, const float* w_packed, const float* scale, const float* shift, float* y,
                          long long voxels, int Cin, int Cout, int act, osb_stream_t stream);
/* Classifier head Conv3d(Cin, 1, 3, 1, 1) (gwcnet_disp_processor.py:60-70 classif*[2]) on a channels-last input:
 * x (B,D,H,W,Cin) -> y (B,1,D,H,W) = (B,D,H,W); w_taps (27, Cin) tap-major [kd][kh][kw][ci]; scale/shift: optional 1-element
 * arrays (folded BN / bias).  Cin = 32. */
int osb_conv3d_k3_c1_ndhwc_fwd(const float* x_ndhwc, const float* w_taps, const float* scale, const float* shift, float* y, int B,
                               int Cin, int D, int H, int W, osb_stream_t stream);
/* 3x3 Conv2d (stride 1, padding = dilation, dilation 1 or 2) + folded BN + residual + activation on the tensor cores, for the
 * residual blocks of the PSMNet-style feature extractor (BasicBlock gwcnet_backbone.py:13-35, layers :38-60;
 * psmnet/submodule.py:219-243): x (B,H,W,Cin) channels-last, w_split = the 3x3x3 tensor-core packing of the 2D weight placed
 * at kd = 1, y (B,H,W,Cout) or (B,Cout,H,W).  dilation 1 = osb_conv3d_k3_tc_fwd with D = 1; dilation 2: W = 128, Cout = 128.
 * osb_conv2d_tc_kc returns the K chunk of the serving kernel (0 = unsupported). */
int osb_conv2d_tc_kc(int Cin, int Cout, int W, int dilation);
int osb_conv2d_k3_tc_fwd(const float* x_nhwc, const void* w_split, const float* scale, const float* shift, const float* residual,
                         float* y, int B, int Cin, int Cout, int H, int W, int dilation, int act, int out_nhwc, int res_nhwc,
                         osb_stream_t stream);
/* osb_conv2d_k3_tc_fwd (dilation 1) with the epilogue of one ConvGRU step (igev/update.py:28-42, stereobase/gru_blocks.py:254-268),
 * for Cout = 128 (the hidden size) and the widths the 16-channel-chunk kernels serve (osb_conv2d_tc_kc(Cin, 128, W, 1) == 16: W >= 24):
 *     v = act(conv(x) * scale + shift + residual),  act also OSB_ACT_SIGMOID / OSB_ACT_TANH
 *     v = v * mul                                    (mul_nhwc non-NULL: the GRU's r * h)
 *     y = blend_h + blend_z * (v - blend_h)          (both non-NULL: h' = (1 - z) h + z q)
 * mul_nhwc, blend_z_nhwc, blend_h_nhwc: (B,H,W,Cout) channels-last fp32.  res_bstride: floats between the batches of an NCHW
 * residual (res_nhwc = 0), >= Cout*H*W -- a channel split() view of a wider (B, C', H, W) tensor -- or 0 for Cout*H*W.  With every
 * new operand NULL and a standard activation the result is osb_conv2d_k3_tc_fwd's, bit for bit. */
int osb_conv2d_k3_tc_gru_fwd(const float* x_nhwc, const void* w_split, const float* scale, const float* shift, const float* residual,
                             const float* mul_nhwc, const float* blend_z_nhwc, const float* blend_h_nhwc, float* y, int B, int Cin,
                             int Cout, int H, int W, int act, int out_nhwc, int res_nhwc, long long res_bstride, osb_stream_t stream);
/* osb_conv2d_k3_tc_fwd and osb_conv2d_k3_tc_gru_fwd with the precision of the products, `precision` = OSB_PREC_FP32 (the result is
 * the entry point without it, bit for bit) or OSB_PREC_F16: the single-term mode of the 16-channel-chunk kernels (csrc/conv3d_tcg.cu),
 * activations staged as fp16(x * 16) alone -- the same range guard (|x| < 4094, the overflow counter) -- and one fp16 MMA per product
 * with fp32 accumulation, the accuracy of the reference's fp16 / bf16 autocast.  Scale, shift, residual, activation, gate and blend
 * stay fp32.  A shape the selector routes to csrc/conv3d_tc.cu (Cout <= 32 at W = 128: osb_conv2d_tc_kc(...) == 32) keeps the
 * 3-term product under either value.  Any other value of `precision` returns OSB_EINVAL before any launch. */
int osb_conv2d_k3_tc_prec_fwd(const float* x_nhwc, const void* w_split, const float* scale, const float* shift, const float* residual,
                              float* y, int B, int Cin, int Cout, int H, int W, int dilation, int act, int out_nhwc, int res_nhwc,
                              int precision, osb_stream_t stream);
int osb_conv2d_k3_tc_gru_prec_fwd(const float* x_nhwc, const void* w_split, const float* scale, const float* shift,
                                  const float* residual, const float* mul_nhwc, const float* blend_z_nhwc, const float* blend_h_nhwc,
                                  float* y, int B, int Cin, int Cout, int H, int W, int act, int out_nhwc, int res_nhwc,
                                  long long res_bstride, int precision, osb_stream_t stream);
/* Modulated deformable 3x3 convolution (DCNv2, groups = 1) + folded BN + activation on the tensor cores: the forward of the
 * reference's ModulatedDeformConvFunction (libs/AANet/deform_conv/deform_conv.py:113-150) as a gather mode of the general-width
 * csrc/conv3d_tcg.cu instantiations (DESIGN.md section 4.21):
 *     y[b,o,ho,wo] = act(scale[o] * sum_{c,tap} w[o,c,tap] * m * bilinear(x[b,:,:,c], ho*stride - padding + kh*dilation + dy,
 *                                                                           wo*stride - padding + kw*dilation + dx) + shift[o])
 * tap = 3 kh + kw; deformable group g = c / (Cin / deformable_groups); dy / dx = offset[b, 18 g + 2 tap + {0, 1}, ho, wo];
 * m = mask[b, 9 g + tap, ho, wo], or 2 * sigmoid(that) with mask_mode = OSB_MASK_DOUBLE_SIGMOID (AANet's DeformConv2d with
 * double_mask, applied to the raw offset_conv logits).  A sample outside (-1, H) x (-1, W) is 0, and each bilinear corner outside
 * the image is 0 (dmcn_im2col_bilinear).  x (B,H,W,Cin) channels-last; offset and mask NCHW over the output extents (Ho, Wo) =
 * ((H + 2 padding - 2 dilation - 1) / stride + 1, ...), offset_bstride / mask_bstride floats between their batches (>= dg*18*Ho*Wo
 * / dg*9*Ho*Wo, so both may be channel slices of one (B, dg*27, Ho, Wo) tensor); w_split = the 2D packing at kd = 1 (Cout rows:
 * 32, 64 or 128; a 16-channel layer is packed zero-padded to 32 rows and its caller keeps the first 16 output channels);
 * y (B,Ho,Wo,Cout) or (B,Cout,Ho,Wo).  Products are 3xFP16 (fp32-accurate); the staged operand m * bilinear(x) must stay below 4094 in magnitude
 * (the overflow counter; with m <= 2, |x| < 2047).  Cin % 16 == 0, Cin % deformable_groups == 0 with a multiple of 4 channels per
 * group, stride 1 or 2, padding >= 0, dilation >= 1, act OSB_ACT_NONE / RELU / LEAKY; anything else returns OSB_EINVAL before any
 * launch.  osb_tc_last_variant names the instantiation ("tcg<64,16,128,1,1,1,0>"). */
#define OSB_MASK_PROB 0           /* the mask is used as given */
#define OSB_MASK_DOUBLE_SIGMOID 1 /* the mask holds logits: m = 2 * sigmoid(mask) */
int osb_mdconv2d_k3_tc_fwd(const float* x_nhwc, const float* offset, long long offset_bstride, const float* mask,
                           long long mask_bstride, int mask_mode, const void* w_split, const float* scale, const float* shift, float* y,
                           int B, int Cin, int Cout, int H, int W, int stride, int padding, int dilation,
                           int deformable_groups, int act, int out_nhwc, osb_stream_t stream);
/* ---- SURVEY.md section 8(f) row 4: remaining volume / regression flavours of the model zoo -------------------------------------
 * osb_gwc_volume_sum_fwd: osb_gwc_volume_fwd with a plain SUM over the K channels of a group instead of the mean:
 *   - CoExCostVolume(maxdisp, group)(x, y) (cost_volume/cost_volume.py:9-29) = sum flavour with D = maxdisp + 1, G = group;
 *   - FoundationStereo's L2-normalised volume (foundationstereo/core/submodule.py:422-461) = sum flavour on features that
 *     osb_group_l2_normalize_fwd normalised per group first (y = x / max(||x_group||_2, eps), aten F.normalize, eps 1e-12).
 * osb_sub_volume_fwd: build_sub_volume (cost_volume.py:108-117): out[b,d,h,w] = sum_c |L[..,w] - R[..,w-d]| (R = 0 for w < d).
 * osb_regression_values_fwd: sum_d prob[b,d,h,w] * values[b,d,h,w] -> (B,H,W) (casnet/submodule.py:22-24). */
int osb_gwc_volume_sum_fwd(const float* ref, const float* tgt, float* out, int B, int C, int H, int W, int D, int G,
                           osb_stream_t stream);
int osb_group_l2_normalize_fwd(const float* x, float* y, int B, int C, int H, int W, int G, float eps, osb_stream_t stream);
int osb_sub_volume_fwd(const float* left, const float* right, float* out, int B, int C, int H, int W, int D, osb_stream_t stream);
int osb_regression_values_fwd(const float* prob, const float* values, float* out, int B, int D, int H, int W, osb_stream_t stream);

/* ---- CasStereo warped cost volumes (casnet/cas_psm.py:286-318, casnet/cas_gwc.py:263-329) --------------------------------
 * The right features are sampled at fractional per-pixel hypotheses disp (B,D,H,W) exactly like
 *   F.grid_sample(y, ((w - disp)/((W-1)/2) - 1, h/((H-1)/2) - 1), 'bilinear', padding_mode='zeros', align_corners=True)
 * (coordinate round trip replayed in fp32); disp may be fractional, negative or beyond either edge.  H >= 2, W >= 2.
 * osb_warped_concat_volume_fwd: CasPSMNet's GetCostVolume: x, y (B,C,H,W) -> out (B,2C,D,H,W) = [x repeated over D | warped y];
 *   mask_left = 1 zeroes the left copy where w < disp (CasGwcNet's concatenation half).
 * osb_warped_gwc_concat_volume_fwd: CasGwcNet's GetCostVolume: out (B, G + 2*Cc, D, H, W) =
 *   [mean over each group's Cg/G channels of x_warped * y_warped | x_warped | y_warped], x_warped = 0 where w < disp;
 *   Cg % G == 0, Cg/G <= 16.
 * One launch each, every output element written once (no memset). */
int osb_warped_concat_volume_fwd(const float* x, const float* y, const float* disp, float* out, int B, int C, int D, int H, int W,
                                 int mask_left, osb_stream_t stream);
int osb_warped_gwc_concat_volume_fwd(const float* xg, const float* yg, const float* xc, const float* yc, const float* disp,
                                     float* out, int B, int Cg, int G, int Cc, int D, int H, int W, osb_stream_t stream);
/* osb_warped_gwc_concat_volume_fwd with the left masking as an argument: mask_left = 1 is that entry point bit for bit;
 * mask_left = 0 leaves x unmasked in both the correlation and the concatenation half -- CFNet's cost_volume_generator
 * (cfnet/cfnet.py:463-486, SpatialTransformer + groupwise_correlation_4D + cat, cfnet/submodule.py:167-173, 315-361), whose
 * right features are gathered at integer samples with zeros outside [0, W-1].  The bilinear coordinate round trip lands within
 * 2^-23 (W - 1) of the integer column and 2^-23 (H - 1) of the integer row (rows too: at H = 64 / 128 / 256, 15 / 21 / 63 rows
 * come back off the integer), so each warped feature differs from that exact gather by at most 2^-23 (W - 1 + H - 1) times the
 * largest difference between the gathered feature and one of its 3x3 neighbours (DESIGN.md section 4.22). */
int osb_warped_gwc_concat_volume_ex_fwd(const float* xg, const float* yg, const float* xc, const float* yc, const float* disp,
                                        float* out, int B, int Cg, int G, int Cc, int D, int H, int W, int mask_left,
                                        osb_stream_t stream);
/* osb_disp_warp_fwd: MonSter's disp_warp(img, disp)[0] (monster/warp.py): img (B,C,H,W), disp (B,1,H,W) -> out (B,C,H,W), img
 *   sampled at column w - disp like F.grid_sample(bilinear, padding_mode='border', align_corners=False) of MonSter's
 *   normalize_coords grid, bit for bit with the reference on the CPU.  The same kernel as the two above, one launch; H >= 2, W >= 2. */
int osb_disp_warp_fwd(const float* img, const float* disp, float* out, int B, int C, int H, int W, osb_stream_t stream);

/* ---- CoEx (coex/coex_disp_processor.py:8-65, coex/coex_cost_processor.py:219-224) -------------------------------------------
 * osb_coex_regression_fwd: Regression.forward (eval) + upfeat in one launch: cost (B,1,D,h,w) logits, spx (B,9,4h,4w) ->
 *   out (B,4h,4w).  Per low-resolution pixel the top_k largest logits along D (2 <= top_k <= 8, top_k <= D; among equal values
 *   the lower index first, like the reference's stable descending sort), their softmax and disp_4 = sum_j p_j * index_j; then
 *   out[b,Y,X] = 4 * sum_{t<9} disp_4[b, Y/4 + t/3 - 1, X/4 + t%3 - 1] * p_t[b,Y,X] with zero outside the image.
 *   spx_is_logits = 1: p = softmax of spx over its 9 channels; 0: spx already holds the probabilities.  spx and out 16-byte aligned.
 * osb_nearest_resize3d_fwd: F.interpolate(x, size=(Do,Ho,Wo), mode='nearest') on N = B*C planes (Di,Hi,Wi) -> (Do,Ho,Wo), with
 *   aten's source index per dimension (dst; dst >> 1 when out = 2*in; else min(floor(dst * ((float)in / out)), in - 1)). */
int osb_coex_regression_fwd(const float* cost, const float* spx, float* out, int B, int D, int h, int w, int top_k, int spx_is_logits,
                            osb_stream_t stream);
int osb_nearest_resize3d_fwd(const float* x, float* y, int N, int Di, int Hi, int Wi, int Do, int Ho, int Wo, osb_stream_t stream);

/* ---- MSNet3D (msnet/submodule.py:136-173) ------------------------------------------------------------------------------------
 * osb_mbv2_block3d_fwd: one whole MobileV2_Residual_3D block in one launch, IEEE fp32 on the CUDA cores:
 *   y = scale3 * (w_proj . relu6(scale2 * dw3x3x3_stride(relu6(scale1 * (w_exp . x) + shift1)) + shift2)) + shift3 [+ residual]
 *   (the three eval BatchNorms folded to per-channel scale/shift).  The expanded tensor never reaches global memory.
 *   x (B,Cin,D,H,W) with in_layout = 0 or (B,D,H,W,Cin) with in_layout = 1; y and the optional residual (NULL = none) are
 *   (B,Cout,Do,Ho,Wo) with out_layout = 0 or (B,Do,Ho,Wo,Cout) with out_layout = 1, where n_o = ceil(n / stride) (k3, padding 1).
 *   w_exp (Cin, Chid), w_dw (27, Chid) with tap = (kd * 3 + kh) * 3 + kw, w_proj (Chid, Cout).  The depthwise conv zero-pads
 *   the HIDDEN tensor: outside the volume the expanded value is 0, not relu6(shift1).  Any D, H, W >= 1.
 *   Instantiated (Cin, Chid, Cout, stride): (40,120,32,1) (32,96,32,1) (32,64,32,1) (32,64,64,2) (64,128,64,1) (64,128,128,2)
 *   (128,256,128,1); anything else is OSB_EINVAL.  Weights and BN vectors 16-byte aligned, and y / residual too when
 *   out_layout = 1; y must not alias x. */
int osb_mbv2_block3d_fwd(const float* x, const float* w_exp, const float* scale1, const float* shift1, const float* w_dw,
                         const float* scale2, const float* shift2, const float* w_proj, const float* scale3, const float* shift3,
                         const float* residual, float* y, int B, int Cin, int Chid, int Cout, int D, int H, int W, int stride,
                         int in_layout, int out_layout, osb_stream_t stream);

/* Backward (adjoint) kernels so the volume constructors and the soft-argmin stay differentiable under tools/train.py
 * (openstereo_b200/autograd.py wraps them in torch.autograd.Function).  grad_ref / grad_tgt may be NULL when not needed.
 *   osb_gwc_volume_bwd     adjoint of osb_gwc_volume_fwd (reduce_sum = 0) / osb_gwc_volume_sum_fwd (1): grad_vol (B,G,D,H,W)
 *   osb_concat_volume_bwd  adjoint of osb_concat_volume_fwd: grad_vol (B,2C,D,H,W)
 *   osb_softargmin_bwd     adjoint of osb_softargmin_fwd w.r.t. cost: grad_out (B,H,W) -> grad_cost (B,D,H,W) */
int osb_gwc_volume_bwd(const float* grad_vol, const float* ref, const float* tgt, float* grad_ref, float* grad_tgt, int B, int C,
                       int H, int W, int D, int G, int reduce_sum, osb_stream_t stream);
int osb_concat_volume_bwd(const float* grad_vol, float* grad_ref, float* grad_tgt, int B, int C, int H, int W, int D, int mask_left,
                          osb_stream_t stream);
int osb_softargmin_bwd(const float* cost, const float* grad_out, float* grad_cost, int B, int D, int H, int W, float alpha,
                       float start, float step, int normalize, osb_stream_t stream);

/* ---- SURVEY.md section 8(f) row 2: LightStereo 2D cost aggregation (lightstereo/aggregation.py:7-134) ------------------------------
 * Depthwise Conv2d (groups = C), kernel KH x KW (odd, <= 21), padding (KH/2, KW/2), stride 1 or 2, NCHW fp32:
 *   y[b,c,oh,ow] = act(scale[c] * sum_{i,j} w[c,i,j] * x[b,c,oh*s+i-KH/2,ow*s+j-KW/2] + shift[c] + residual[b,c,oh,ow])
 * the 3x3 dwconv of MobileV2Residual (:80-84, folded BN + ReLU6) and the strip convolutions of AttentionModule
 * (:109-117: 1x7/7x1, 1x11/11x1, 1x21/21x1 with bias = shift; the branch sum `attn + attn_0 + ...` rides on `residual`).
 * w: (C, KH, KW) contiguous; scale/shift/residual optional; y may alias residual. */
int osb_dwconv2d_fwd(const float* x, const float* w, const float* scale, const float* shift, const float* residual, float* y, int B,
                     int C, int H, int W, int KH, int KW, int stride, int act, osb_stream_t stream);
/* ConvTranspose2d(k=3, stride=2, padding=1, output_padding=1, bias=False) + folded BN + residual + activation
 * (lightstereo/aggregation.py:28-34,58-59: conv5 / conv6 with `F.relu(conv5(conv4) + redir2(conv2))`): x (B,Cin,H,W) ->
 * y (B,Cout,2H,2W); w_packed (Cin, 9, Cout) = ops.pack_deconv2d_weight of the (Cin,Cout,3,3) parameter. */
int osb_deconv2d_k3s2_fwd(const float* x, const float* w_packed, const float* scale, const float* shift, const float* residual,
                          float* y, int B, int Cin, int Cout, int H, int W, int act, osb_stream_t stream);

/* ---- SURVEY.md section 8(f) rows 1 and 3: GRU-iteration lookups of IGEV / StereoBase ------------------------------------
 * Pair-average along the middle axis of a (outer, n, inner) array -> (outer, n/2, inner): the F.avg_pool2d(.., [1,2],
 * stride=[1,2]) pyramid of Combined_Geo_Encoding_Volume.__init__ (igev/geometry.py:24-30, stereobase/gru_blocks.py:187-193)
 * on the volume's native (B,C,D,H,W) layout (outer=B*C, n=D, inner=H*W) and on the all-pairs correlation
 * (outer=B*H*W1, n=W2, inner=1). */
int osb_avgpool_pairs_fwd(const float* x, float* y, long long outer, int n, long long inner, osb_stream_t stream);
/* Combined_Geo_Encoding_Volume.__call__ (igev/geometry.py:32-57) == CombinedGeoEncodingVolume.__call__
 * (stereobase/gru_blocks.py:195-220): per pyramid level i < num_levels, 2*radius+1 zero-padded bilinear taps of
 *   geo_i (B, C, D>>i, H, W) at d = disp/2^i + dx            -> channels [i*(C+1)*T + c*T + k]
 *   corr_i (B, H, W, W2>>i) at x = coords/2^i - disp/2^i + dx -> channels [i*(C+1)*T + C*T + k],   T = 2*radius+1
 * disp (B,1,H,W), coords (B,H,W), out (B, num_levels*(C+1)*T, H, W).  Unused level pointers are NULL. */
int osb_geo_lookup_fwd(const float* geo0, const float* geo1, const float* geo2, const float* geo3, const float* corr0,
                       const float* corr1, const float* corr2, const float* corr3, const float* disp, const float* coords,
                       float* out, int B, int C, int D, int H, int W, int W2, int num_levels, int radius, osb_stream_t stream);
/* Geo_Encoding_Volume.__call__ (igev_rt/geometry.py:18-33, IGEV-RT): the same lookup of the geometry volume alone, no correlation
 * row.  Per level i < num_levels, 2*radius+1 zero-padded bilinear taps of geo_i (B, C, D>>i, H, W) at d = dx + disp/2^i
 *   -> channels [i*C*T + c*T + k],   T = 2*radius+1
 * disp (B,1,H,W), out (B, num_levels*C*T, H, W).  Unused level pointers are NULL. */
int osb_geo_volume_lookup_fwd(const float* geo0, const float* geo1, const float* geo2, const float* geo3, const float* disp,
                              float* out, int B, int C, int D, int H, int W, int num_levels, int radius, osb_stream_t stream);
/* IGEV++'s multi-range Combined_Geo_Encoding_Volume.__call__ (igevpp/geometry.py:35-77) in one launch, T = 2*radius+1:
 *   geo_i (B, C, D0>>i, H, W), i < num_levels, at d = dx + disp/2^i   -> out0     (B, num_levels*C*T, H, W), [i*C*T + c*T + k]
 *   vol1  (B, C, D1, H, W)  at d = dx + disp/2                          -> out1     (B, C*T, H, W),            [c*T + k]
 *   vol2  (B, C, D2, H, W)  at d = dx + disp/4                          -> out2     (B, C*T, H, W),            [c*T + k]
 *   corr_i (B, H, W, W2>>i) at x = coords/2^i - disp/2^i + dx           -> out_corr (B, num_levels*T, H, W),   [i*T + k]
 * geo_i is the pair-averaged pyramid of the first volume; D1 and D2 are independent of D0.  disp (B,1,H,W), coords (B,H,W).
 * Unused level pointers are NULL. */
int osb_geo_multirange_lookup_fwd(const float* geo0, const float* geo1, const float* geo2, const float* geo3, const float* vol1,
                                  const float* vol2, const float* corr0, const float* corr1, const float* corr2, const float* corr3,
                                  const float* disp, const float* coords, float* out0, float* out1, float* out2, float* out_corr,
                                  int B, int C, int D0, int D1, int D2, int H, int W, int W2, int num_levels, int radius,
                                  osb_stream_t stream);
/* context_upsample (stereobase/igev_blocks.py:51-63, igev/submodule.py:253-265): disp_low (B,1,h,w), up_weights
 * (B,9,scale*h,scale*w) -> out (B, scale*h, scale*w) = sum over the 3x3 low-resolution neighbourhood (zero padded). */
int osb_context_upsample_fwd(const float* disp_low, const float* up_weights, float* out, int B, int h, int w, int scale,
                             osb_stream_t stream);
/* (B,C,D,H,W) -> (B,D,H,W,C) layout change feeding the tensor-core conv. */
int osb_ncdhw_to_ndhwc(const float* x, float* y, int B, int C, int D, int H, int W, osb_stream_t stream);
/* Same with the channel axis zero-padded to Cpad >= C: y (B,D,H,W,Cpad) -- channel plans that are not multiples of 16 (StereoBase's
 * 24 / 48) run on the tensor-core kernels as 32 / 64 with zero weights on the padding. */
int osb_ncdhw_to_ndhwc_pad(const float* x, float* y, int B, int C, int Cpad, int D, int H, int W, osb_stream_t stream);
/* Same into channels coff .. coff + C - 1 of y (B,D,H,W,ystride), ystride >= coff + C; the other channels are left as they are
 * (the ConvGRU's torch.cat of its inputs, written channels-last without materialising the NCHW concatenation). */
int osb_ncdhw_to_ndhwc_slice(const float* x, float* y, int B, int C, int D, int H, int W, int ystride, int coff, osb_stream_t stream);
/* FeatureAtt gate in one launch (igev_blocks.py:35-48 as used by stereobase/hourglass.py:62-99):
 * gate_nhwc (B,H,W,Cpad) = sigmoid(conv1x1(act1(bn(conv1x1(feat_nchw (B,Cf,H,W)))))), channels Cv..Cpad-1 zero.
 * w1_packed (Cf,Ch), w2_packed (Ch,Cv); scale/shift = folded BN / bias (NULL = identity).  HW = H*W. */
int osb_feature_att_gate_fwd(const float* feat_nchw, const float* w1_packed, const float* scale1, const float* shift1,
                             const float* w2_packed, const float* scale2, const float* shift2, float* gate_nhwc, int B,
                             int Cf, int Ch, int Cv, int Cpad, int HW, int act1, osb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* OPENSTEREO_B200_H_ */
