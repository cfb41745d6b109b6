// CoEx (stereo/modeling/models/coex/) for sm_90a: the fused regression tail and the nearest resampling of the aggregation.
//
//   Regression.forward (eval) + upfeat      coex/coex_disp_processor.py:8-65
//   F.interpolate(mode='nearest') in 3D     coex/coex_cost_processor.py:219-224 (a transposed conv's output vs its skip level)
//
// ---- regression tail ------------------------------------------------------------------------------------------------------
// The reference sorts the whole (B,1,D,h,w) logit tensor along D, gathers the top k, takes their softmax and the expectation of
// the indices (disp_4), then up-samples disp_4 x4 with the superpixel weights: a softmax over 9 full-resolution logit planes, a
// 3x3 unfold, a nearest x4 interpolate of the 9 unfolded planes, a product and a sum -- about ten full-resolution passes for one
// output plane.  Here ONE launch reads every logit and every superpixel value once and writes the output once.
//
// A CTA owns a tile of kTileH x kTileW low-resolution pixels.  Phase 1: its threads compute disp_4 for the tile plus a 1-pixel
// halo (zero outside the image: the unfold's padding) into shared memory, each streaming D through a K-entry register list sorted
// by value.  A new value enters only when it is strictly larger than an entry, so among equal values the lower index stays first
// -- the order of the reference's stable cost.sort(2, descending=True) on the CPU.  Phase 2: a thread owns 4 consecutive
// full-resolution columns, which share one low-resolution column and therefore one 3x3 neighbourhood of disp_4; it reads the 9
// superpixel values of those columns as float4s (a warp reads 512 contiguous bytes per plane) and writes one float4.
//
// Arithmetic follows the reference's operation order: softmax over the k values as max, exp(v - max), sum in j order, divide;
// disp_4 = sum_j p_j * (float)index_j in j order; optional softmax over the 9 superpixel logits likewise; out = 4 * sum_t
// disp_4[neighbour t] * p_t in t order (products and sums rounded separately, no contraction).
//
// Roofline: HBM-bound.  Algorithmic bytes = 4 * (B*D*h*w + 9*B*16*h*w + B*16*h*w) (the logits, the superpixel planes, the output).
//
// ---- nearest resampling ---------------------------------------------------------------------------------------------------
// A gather with aten's nearest index per dimension (UpSample.h nearest_idx): dst when in == out, dst >> 1 when out == 2*in, else
// min((int)floorf(dst * ((float)in / out)), in - 1).  Bit-equal to F.interpolate(mode='nearest').
#include <algorithm>

#include "common.cuh"

namespace osb {

constexpr int kRegThreads = 256;
constexpr int kTileH = 16, kTileW = 32;                  // low-resolution pixels per CTA
constexpr int kHaloH = kTileH + 2, kHaloW = kTileW + 2;

struct RegressionParams {
  const float* cost;   // (B, 1, D, h, w)
  const float* spx;    // (B, 9, 4h, 4w): logits or probabilities
  float* out;          // (B, 4h, 4w)
  int B, D, h, w;
  int logits;
};

template <int K>
__device__ __forceinline__ float topk_disparity(const float* __restrict__ col, size_t plane, int D) {
  float vals[K];
  int idx[K];
#pragma unroll
  for (int j = 0; j < K; ++j) vals[j] = 0.f, idx[j] = 0;
#pragma unroll 4
  for (int d = 0; d < D; ++d) {
    float cv = __ldg(col + (size_t)d * plane);
    int ci = d;
    bool moving = false;
#pragma unroll
    for (int j = 0; j < K; ++j) {
      // slot j is empty (d <= j), or the carried value beats it strictly, or an insertion above is pushing entries down
      if (moving || d <= j || cv > vals[j]) {
        moving = true;
        const float tv = vals[j];
        const int ti = idx[j];
        vals[j] = cv, idx[j] = ci;
        cv = tv, ci = ti;
      }
    }
  }
  const float m = vals[0];                               // the list is sorted: its first value is the max
  float e[K], s = 0.f;
#pragma unroll
  for (int j = 0; j < K; ++j) {
    e[j] = expf(__fsub_rn(vals[j], m));
    s = __fadd_rn(s, e[j]);
  }
  float disp = 0.f;
#pragma unroll
  for (int j = 0; j < K; ++j) disp = __fadd_rn(disp, __fmul_rn(__fdiv_rn(e[j], s), (float)idx[j]));
  return disp;
}

template <int K>
__global__ void __launch_bounds__(kRegThreads) coex_regression_kernel(const RegressionParams p) {
  __shared__ float s_disp[kHaloH][kHaloW];
  const int b = blockIdx.z;
  const int y0 = blockIdx.y * kTileH, x0 = blockIdx.x * kTileW;
  const size_t plane = (size_t)p.h * p.w;
  const float* cost = p.cost + (size_t)b * p.D * plane;

  // ---- phase 1: disp_4 of the tile and its halo ----
  for (int i = threadIdx.x; i < kHaloH * kHaloW; i += kRegThreads) {
    const int ly = i / kHaloW, lx = i - ly * kHaloW;
    const int y = y0 + ly - 1, x = x0 + lx - 1;
    float v = 0.f;
    if (y >= 0 && y < p.h && x >= 0 && x < p.w) v = topk_disparity<K>(cost + (size_t)y * p.w + x, plane, p.D);
    s_disp[ly][lx] = v;
  }
  __syncthreads();

  // ---- phase 2: 4 x 4 full-resolution pixels per tile cell, 4 columns (one float4) per thread and step ----
  const int H4 = 4 * p.h, W4 = 4 * p.w;
  const size_t fplane = (size_t)H4 * W4;
  const float* spx = p.spx + (size_t)b * 9 * fplane;
  float* out = p.out + (size_t)b * fplane;
  for (int i = threadIdx.x; i < 4 * kTileH * kTileW; i += kRegThreads) {
    const int fy = i / kTileW, lx = i - fy * kTileW;     // full-resolution row within the tile, low-resolution column
    const int Y = 4 * y0 + fy, x = x0 + lx;
    if (Y >= H4 || x >= p.w) continue;
    const int ly = fy >> 2;
    float nb[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) nb[t] = s_disp[ly + t / 3][lx + t % 3];
    const size_t off = (size_t)Y * W4 + 4 * x;
    float4 q[9];
#pragma unroll
    for (int t = 0; t < 9; ++t) q[t] = __ldcs(reinterpret_cast<const float4*>(spx + t * fplane + off));
    if (p.logits) {
      float4 m = q[0];
#pragma unroll
      for (int t = 1; t < 9; ++t) m.x = fmaxf(m.x, q[t].x), m.y = fmaxf(m.y, q[t].y), m.z = fmaxf(m.z, q[t].z), m.w = fmaxf(m.w, q[t].w);
      float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int t = 0; t < 9; ++t) {
        q[t].x = expf(__fsub_rn(q[t].x, m.x)), q[t].y = expf(__fsub_rn(q[t].y, m.y));
        q[t].z = expf(__fsub_rn(q[t].z, m.z)), q[t].w = expf(__fsub_rn(q[t].w, m.w));
        s.x = __fadd_rn(s.x, q[t].x), s.y = __fadd_rn(s.y, q[t].y), s.z = __fadd_rn(s.z, q[t].z), s.w = __fadd_rn(s.w, q[t].w);
      }
#pragma unroll
      for (int t = 0; t < 9; ++t)
        q[t].x = __fdiv_rn(q[t].x, s.x), q[t].y = __fdiv_rn(q[t].y, s.y), q[t].z = __fdiv_rn(q[t].z, s.z), q[t].w = __fdiv_rn(q[t].w, s.w);
    }
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      acc.x = __fadd_rn(acc.x, __fmul_rn(nb[t], q[t].x)), acc.y = __fadd_rn(acc.y, __fmul_rn(nb[t], q[t].y));
      acc.z = __fadd_rn(acc.z, __fmul_rn(nb[t], q[t].z)), acc.w = __fadd_rn(acc.w, __fmul_rn(nb[t], q[t].w));
    }
    __stcs(reinterpret_cast<float4*>(out + off), make_float4(4.f * acc.x, 4.f * acc.y, 4.f * acc.z, 4.f * acc.w));
  }
}

// aten's nearest source index (aten/src/ATen/native/UpSample.h: nearest_idx with the scale (float)in / out)
__device__ __forceinline__ int nearest_src(int dst, int in, int out) {
  if (in == out) return dst;
  if (out == 2 * in) return dst >> 1;
  const float scale = __fdiv_rn((float)in, (float)out);
  return min((int)floorf(__fmul_rn((float)dst, scale)), in - 1);
}

__global__ void __launch_bounds__(256) nearest_resize3d_kernel(const float* __restrict__ x, float* __restrict__ y, long long total,
                                                               int Di, int Hi, int Wi, int Do, int Ho, int Wo) {
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int ow = (int)(i % Wo);
    long long r = i / Wo;
    const int oh = (int)(r % Ho);
    r /= Ho;
    const int od = (int)(r % Do);
    const long long n = r / Do;
    const int id = nearest_src(od, Di, Do), ih = nearest_src(oh, Hi, Ho), iw = nearest_src(ow, Wi, Wo);
    y[i] = __ldg(x + ((n * Di + id) * Hi + ih) * Wi + iw);
  }
}

}  // namespace osb

extern "C" {

int osb_coex_regression_fwd(const float* cost, const float* spx, float* out, int B, int D, int h, int w, int top_k,
                            int spx_is_logits, osb_stream_t stream) {
  using namespace osb;
  OSB_REQUIRE(cost && spx && out, "coex_regression: null pointer");
  OSB_REQUIRE(B > 0 && D > 0 && h > 0 && w > 0, "coex_regression: empty shape B=%d D=%d h=%d w=%d", B, D, h, w);
  OSB_REQUIRE(top_k >= 2 && top_k <= 8, "coex_regression: top_k=%d not supported (2..8)", top_k);
  OSB_REQUIRE(top_k <= D, "coex_regression: top_k=%d exceeds the %d disparity planes", top_k, D);
  OSB_REQUIRE((reinterpret_cast<uintptr_t>(spx) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
              "coex_regression: spx and out must be 16-byte aligned");
  OSB_REQUIRE((h + kTileH - 1) / kTileH <= 65535 && B <= 65535, "coex_regression: grid too large");
  RegressionParams p{cost, spx, out, B, D, h, w, spx_is_logits ? 1 : 0};
  const dim3 grid((w + kTileW - 1) / kTileW, (h + kTileH - 1) / kTileH, B);
  const cudaStream_t s = (cudaStream_t)stream;
  switch (top_k) {
    case 2: coex_regression_kernel<2><<<grid, kRegThreads, 0, s>>>(p); break;
    case 3: coex_regression_kernel<3><<<grid, kRegThreads, 0, s>>>(p); break;
    case 4: coex_regression_kernel<4><<<grid, kRegThreads, 0, s>>>(p); break;
    case 5: coex_regression_kernel<5><<<grid, kRegThreads, 0, s>>>(p); break;
    case 6: coex_regression_kernel<6><<<grid, kRegThreads, 0, s>>>(p); break;
    case 7: coex_regression_kernel<7><<<grid, kRegThreads, 0, s>>>(p); break;
    default: coex_regression_kernel<8><<<grid, kRegThreads, 0, s>>>(p); break;
  }
  count_launch();
  return check_launch("coex_regression_kernel");
}

int osb_nearest_resize3d_fwd(const float* x, float* y, int N, int Di, int Hi, int Wi, int Do, int Ho, int Wo, osb_stream_t stream) {
  using namespace osb;
  OSB_REQUIRE(x && y, "nearest_resize3d: null pointer");
  OSB_REQUIRE(N > 0 && Di > 0 && Hi > 0 && Wi > 0 && Do > 0 && Ho > 0 && Wo > 0, "nearest_resize3d: empty shape");
  const long long total = (long long)N * Do * Ho * Wo;
  const long long blocks = std::min<long long>((total + 255) / 256, (long long)sm_count() * 8);
  nearest_resize3d_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, y, total, Di, Hi, Wi, Do, Ho, Wo);
  count_launch();
  return check_launch("nearest_resize3d_kernel");
}
}
