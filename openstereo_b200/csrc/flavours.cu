// SURVEY.md section 8(f) row 4: the remaining volume / regression flavours of the model zoo.
//   group_l2_normalize   F.normalize over each correlation group's channel vector (foundationstereo/core/submodule.py:422-431),
//                        the pre-pass of the L2-normalised gwc volume (then osb_gwc_volume_sum_fwd on the normalised features)
//   sub_volume           build_sub_volume, cost_volume/cost_volume.py:108-117 (L1 distance volume, StereoBase USE_SUB_VOLUME)
//   regression_values    sum_d prob * disp_values with per-pixel hypothesis planes (casnet/submodule.py:22-24)
// All three are HBM-bound elementwise / small-reduction kernels: one pass over their inputs, coalesced along W.
#include "common.cuh"

namespace osb {

// y[b, g*K + k, h, w] = x[...] / max(||x[b, g*K .. g*K + K - 1, h, w]||_2, eps)      (aten normalize: eps 1e-12, clamp_min)
__global__ void __launch_bounds__(256) group_l2_normalize_kernel(const float* __restrict__ x, float* __restrict__ y, int K, size_t hw,
                                                                  size_t total, float eps) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;       // index over (b, g, h*w)
  if (i >= total) return;
  const size_t bg = i / hw, pix = i % hw;
  const float* xp = x + bg * K * hw + pix;
  float ss = 0.f;
  for (int k = 0; k < K; ++k) {
    const float v = __ldg(xp + (size_t)k * hw);
    ss = fmaf(v, v, ss);
  }
  const float denom = fmaxf(sqrtf(ss), eps);
  float* yp = y + bg * K * hw + pix;
  for (int k = 0; k < K; ++k) yp[(size_t)k * hw] = __ldg(xp + (size_t)k * hw) / denom;
}

// cost[b, d, h, w] = sum_c |L[b,c,h,w] - R[b,c,h,w-d]|  (w >= d),   sum_c |L[b,c,h,w]|  (w < d)
// thread = one (b, h, w) and a chunk of 8 hypotheses kept in registers; L is read once per channel, R as 8 neighbouring columns.
__global__ void __launch_bounds__(128) sub_volume_kernel(const float* __restrict__ l, const float* __restrict__ r, float* __restrict__ out,
                                                          int C, int H, int W, int D) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  const int h = blockIdx.y % H, b = blockIdx.y / H;
  const int d0 = blockIdx.z * 8;
  if (w >= W) return;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  const size_t hw = (size_t)H * W;
  const float* lp = l + ((size_t)b * C * H + h) * W + w;
  const float* rp = r + ((size_t)b * C * H + h) * W;
  for (int c = 0; c < C; ++c) {
    const float lv = __ldg(lp + c * hw);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int x = w - (d0 + j);
      const float rv = x >= 0 ? __ldg(rp + c * hw + x) : 0.f;
      acc[j] += fabsf(lv - rv);
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j)
    if (d0 + j < D) out[(((size_t)b * D + d0 + j) * H + h) * W + w] = acc[j];
}

__global__ void __launch_bounds__(256) regression_values_kernel(const float* __restrict__ prob, const float* __restrict__ values,
                                                                 float* __restrict__ out, int D, size_t hw, size_t total) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;       // index over (b, h*w)
  if (i >= total) return;
  const size_t b = i / hw, pix = i % hw;
  const float* pp = prob + b * D * hw + pix;
  const float* vp = values + b * D * hw + pix;
  float acc = 0.f;
  for (int d = 0; d < D; ++d) acc = fmaf(__ldg(pp + (size_t)d * hw), __ldg(vp + (size_t)d * hw), acc);
  out[i] = acc;
}

}  // namespace osb

extern "C" {

int osb_group_l2_normalize_fwd(const float* x, float* y, int B, int C, int H, int W, int G, float eps, osb_stream_t stream) {
  using namespace osb;
  OSB_REQUIRE(x && y, "group_l2_normalize: null pointer");
  OSB_REQUIRE(B > 0 && C > 0 && H > 0 && W > 0 && G > 0, "group_l2_normalize: empty shape");
  OSB_REQUIRE(C % G == 0, "groupwise_correlation: C=%d not divisible by num_groups=%d", C, G);
  const size_t hw = (size_t)H * W, total = (size_t)B * G * hw;
  group_l2_normalize_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, y, C / G, hw, total, eps);
  count_launch();
  return check_launch("group_l2_normalize_kernel");
}

int osb_sub_volume_fwd(const float* left, const float* right, float* out, int B, int C, int H, int W, int D, osb_stream_t stream) {
  using namespace osb;
  OSB_REQUIRE(left && right && out, "sub_volume: null pointer");
  OSB_REQUIRE(B > 0 && C > 0 && H > 0 && W > 0 && D > 0, "sub_volume: empty shape");
  OSB_REQUIRE((long long)B * H <= 65535 && (D + 7) / 8 <= 65535, "sub_volume: grid too large");
  dim3 grid((W + 127) / 128, B * H, (D + 7) / 8);
  sub_volume_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(left, right, out, C, H, W, D);
  count_launch();
  return check_launch("sub_volume_kernel");
}

int osb_regression_values_fwd(const float* prob, const float* values, float* out, int B, int D, int H, int W, osb_stream_t stream) {
  using namespace osb;
  OSB_REQUIRE(prob && values && out, "regression_values: null pointer");
  OSB_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0, "regression_values: empty shape");
  const size_t hw = (size_t)H * W, total = (size_t)B * hw;
  regression_values_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(prob, values, out, D, hw, total);
  count_launch();
  return check_launch("regression_values_kernel");
}
}

// ------------------------------------------------------------------------------------------ FeatureAtt gate, one launch
// igev_blocks.py:35-48 (FeatureAtt.feat_att) as used by stereobase/hourglass.py:62-99:
//     gate = sigmoid(Conv2d(Cf/2 -> Cv, 1, bias)(LeakyReLU(BN(Conv2d(Cf -> Cf/2, 1)(feat)))))
// written CHANNELS-LAST and zero-padded, (B, H, W, Cpad), the operand the tensor-core conv epilogues multiply by
// (tc_common.cuh: store_ndhwc_chunk32 gate0).  The unfused path was two 1x1-conv launches plus a layout conversion per gate --
// 15 launches of latency-bound work per StereoBase forward.
// CTA = 8 consecutive pixels of one image x 128 threads (16 channel groups x 8 pixels): the feature tile [Cf][8] is staged in shared
// memory, a thread produces 4 channels of one pixel at a time (one LDG.128 of the (Cin, Cout)-packed weights per input channel,
// shared by the 8 pixel lanes).  A first version with 32-pixel tiles left the 1/16-resolution gates on 64 CTAs: 244 us.
namespace osb {

constexpr int FA_PT = 8;                      // pixels per CTA: small tiles -> B*H*W/8 CTAs (the 1/16 maps have 512 pixels per image)

__global__ void __launch_bounds__(128) feature_att_gate_kernel(const float* __restrict__ feat, const float* __restrict__ w1,
                                                               const float* __restrict__ sc1, const float* __restrict__ sh1,
                                                               const float* __restrict__ w2, const float* __restrict__ sc2,
                                                               const float* __restrict__ sh2, float* __restrict__ gate, int Cf,
                                                               int Ch, int Cv, int Cpad, int HW, int act1) {
  extern __shared__ __align__(16) float fa_smem[];
  float* fs = fa_smem;                        // [Cf][PT]
  float* hs = fs + Cf * FA_PT;                // [Ch][PT]
  float* os = hs + Ch * FA_PT;                // [PT][Cpad + 4]
  const int OS = Cpad + 4;
  const int px = threadIdx.x % FA_PT, grp = threadIdx.x / FA_PT;      // 8 pixels x 16 channel groups
  constexpr int NG = 128 / FA_PT;
  const int tiles = (HW + FA_PT - 1) / FA_PT;
  const int b = blockIdx.x / tiles, p0 = (blockIdx.x % tiles) * FA_PT;
  const int np = min(FA_PT, HW - p0);
  const float* fb = feat + (size_t)b * Cf * HW + p0;
  for (int i = threadIdx.x; i < Cf * FA_PT; i += 128) fs[i] = (i % FA_PT) < np ? __ldg(fb + (size_t)(i / FA_PT) * HW + (i % FA_PT)) : 0.f;
  for (int i = threadIdx.x; i < FA_PT * OS; i += 128) os[i] = 0.f;     // padded channels stay zero
  __syncthreads();
  for (int hc = grp * 4; hc < Ch; hc += 4 * NG) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 8
    for (int c = 0; c < Cf; ++c) {
      const float x = fs[c * FA_PT + px];
      const float4 w = __ldg(reinterpret_cast<const float4*>(w1 + (size_t)c * Ch + hc));
      a0 = fmaf(x, w.x, a0), a1 = fmaf(x, w.y, a1), a2 = fmaf(x, w.z, a2), a3 = fmaf(x, w.w, a3);
    }
    float v[4] = {a0, a1, a2, a3};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float t = fmaf(v[j], sc1 ? __ldg(sc1 + hc + j) : 1.f, sh1 ? __ldg(sh1 + hc + j) : 0.f);
      if (act1 == OSB_ACT_LEAKY) t = t > 0.f ? t : 0.01f * t;
      else if (act1 == OSB_ACT_RELU) t = fmaxf(t, 0.f);
      hs[(hc + j) * FA_PT + px] = t;
    }
  }
  __syncthreads();
  for (int oc = grp * 4; oc < Cv; oc += 4 * NG) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 8
    for (int c = 0; c < Ch; ++c) {
      const float x = hs[c * FA_PT + px];
      const float4 w = __ldg(reinterpret_cast<const float4*>(w2 + (size_t)c * Cv + oc));
      a0 = fmaf(x, w.x, a0), a1 = fmaf(x, w.y, a1), a2 = fmaf(x, w.z, a2), a3 = fmaf(x, w.w, a3);
    }
    float v[4] = {a0, a1, a2, a3};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float t = fmaf(v[j], sc2 ? __ldg(sc2 + oc + j) : 1.f, sh2 ? __ldg(sh2 + oc + j) : 0.f);
      os[px * OS + oc + j] = 1.f / (1.f + expf(-t));
    }
  }
  __syncthreads();
  float* gb = gate + ((size_t)b * HW + p0) * Cpad;
  const int q4 = Cpad / 4;
  for (int i = threadIdx.x; i < np * q4; i += 128) {
    const int p = i / q4, c4 = i % q4;
    reinterpret_cast<float4*>(gb)[i] = *reinterpret_cast<const float4*>(os + p * OS + 4 * c4);
  }
}

}  // namespace osb

extern "C" int osb_feature_att_gate_fwd(const float* feat_nchw, const float* w1_packed, const float* scale1, const float* shift1,
                                        const float* w2_packed, const float* scale2, const float* shift2, float* gate_nhwc, int B,
                                        int Cf, int Ch, int Cv, int Cpad, int HW, int act1, osb_stream_t stream) {
  using namespace osb;
  OSB_REQUIRE(feat_nchw && w1_packed && w2_packed && gate_nhwc, "feature_att_gate: null pointer");
  OSB_REQUIRE(B > 0 && Cf > 0 && Ch > 0 && Cv > 0 && HW > 0 && Ch % 4 == 0 && Cv % 4 == 0 && Cpad % 4 == 0 && Cpad >= Cv,
              "feature_att_gate: bad shape (hidden / output channels must be multiples of 4)");
  OSB_REQUIRE(act1 >= 0 && act1 <= 2, "feature_att_gate: unknown activation %d", act1);
  OSB_REQUIRE(((reinterpret_cast<uintptr_t>(w1_packed) | reinterpret_cast<uintptr_t>(w2_packed) | reinterpret_cast<uintptr_t>(gate_nhwc)) & 15) == 0,
              "feature_att_gate: pointers must be 16-byte aligned");
  const size_t smem = ((size_t)(Cf + Ch) * FA_PT + (size_t)FA_PT * (Cpad + 4)) * sizeof(float);
  OSB_REQUIRE(smem <= 200 * 1024, "feature_att_gate: %d + %d channels exceed the shared-memory tile", Cf, Ch);
  static PerDeviceFlag configured;
  if (!configured.here()) {
    cudaError_t e = cudaFuncSetAttribute(feature_att_gate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) {
      set_error("feature_att_gate: cannot reserve shared memory: %s", cudaGetErrorString(e));
      return OSB_ECUDA;
    }
    configured.here() = true;
  }
  const long long blocks = (long long)B * ((HW + FA_PT - 1) / FA_PT);
  OSB_REQUIRE(blocks < (1ll << 31), "feature_att_gate: too many tiles");
  feature_att_gate_kernel<<<(unsigned)blocks, 128, smem, (cudaStream_t)stream>>>(feat_nchw, w1_packed, scale1, shift1, w2_packed, scale2,
                                                                                 shift2, gate_nhwc, Cf, Ch, Cv, Cpad, HW, act1);
  count_launch();
  return check_launch("feature_att_gate_kernel");
}
