// Soft-argmin tails for sm_90a: softmax over the disparity axis fused with the expectation, with or without the
// trilinear x4 up-sampling in front of it, and the per-image EPE partial sums.
//
//   disparity_regression(F.softmax(x, 1), D)   stereo/modeling/disp_pred/disp_regression.py:8-12
//                                              stereo/modeling/models/gwcnet/gwcnet_disp_processor.py:22-26
//   FasterSoftArgmin.forward                   stereo/modeling/models/psmnet/psmnet_disp_processor.py:51-74
//   F.interpolate(..., 'trilinear') -> softmax -> regression
//                                              gwcnet_disp_processor.py:129-133, psmnet_cost_processor.py:203-214
//   epe_metric                                 stereo/evaluation/metric_per_image.py:32-41
//
// The reference materialises the (B,192,H,W) probability tensor four times (interpolate, softmax, mul, sum =
// 100.7 MB/pair each); here one thread owns one output pixel and keeps a running (max, sum, weighted sum).
#include "common.cuh"

namespace osb {

// ------------------------------------------------------------------------------------------------ plain soft-argmin
// Variance mode of softargmin_kernel for one pixel: p = softmax_d(cost), mu = sum_d p_d v_d with v_d = vals[d * HW] (or d when
// vals is NULL), then var = sum_d p_d (v_d - mu)^2, CFNet's disparity_variance / disparity_variance_confidence
// (cfnet/submodule.py:128-141).  Pass 1 is the plain kernel's loop (alpha 1, start 0, step 1), so with vals NULL mu is its result
// bit for bit; pass 2 re-reads the cost and sums exp(x_d - max) (v_d - mu)^2 about that mu (no E[v^2] - mu^2 cancellation).
// Out of line: the plain instantiation's code is unchanged.
static __device__ __noinline__ void softargmin_var(const float* __restrict__ p, const float* __restrict__ vals, float* __restrict__ mu_out,
                                                   float* __restrict__ var_out, int D, size_t HW) {
  float m = -INFINITY, s = 0.f, t = 0.f;
  for (int d0 = 0; d0 < D; d0 += 8) {
    float x[8];
    float cm = -INFINITY;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      x[i] = (d0 + i < D) ? __ldg(p + (size_t)(d0 + i) * HW) : -INFINITY;
      cm = fmaxf(cm, x[i]);
    }
    const float nm = fmaxf(m, cm);
    if (nm == -INFINITY) continue;
    const float sc = expf(m - nm);
    s *= sc, t *= sc;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float e = expf(x[i] - nm);
      s += e;
      const float v = vals ? (d0 + i < D ? __ldg(vals + (size_t)(d0 + i) * HW) : 0.f) : (float)(d0 + i);
      t = fmaf(e, v, t);
    }
    m = nm;
  }
  const float mu = t / s;
  *mu_out = mu;
  if (!var_out) return;
  float s2 = 0.f, q = 0.f;
  for (int d = 0; d < D; ++d) {
    const float e = expf(__ldg(p + (size_t)d * HW) - m);
    const float dv = (vals ? __ldg(vals + (size_t)d * HW) : (float)d) - mu;
    s2 += e;
    q = fmaf(e, dv * dv, q);
  }
  *var_out = q / s2;
}

// cost (B,D,H,W): one pass, online softmax in chunks of 8 bins (one rescale per chunk).  Consecutive threads own
// consecutive pixels, so every load of a warp is one 128-byte line; 8 independent loads are in flight per thread.
// Variance mode (values or var_out non-NULL; osb_softargmin_var_fwd, always normalised): CFNet's regression tails.
__global__ void __launch_bounds__(256) softargmin_kernel(const float* __restrict__ cost, float* __restrict__ out, int D,
                                                         size_t HW, size_t total, float alpha, float start, float step,
                                                         int normalize, const float* __restrict__ values,
                                                         float* __restrict__ var_out) {
  const size_t pix = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= total) return;
  const size_t b = pix / HW, hw = pix - b * HW;
  const float* p = cost + b * (size_t)D * HW + hw;
  if (values || var_out) {
    softargmin_var(p, values ? values + b * (size_t)D * HW + hw : nullptr, out + pix, var_out ? var_out + pix : nullptr, D, HW);
    return;
  }
  if (!normalize) {
    float t = 0.f;
    for (int d = 0; d < D; ++d) t = fmaf(__ldg(p + (size_t)d * HW) * alpha, start + step * (float)d, t);
    out[pix] = t;
    return;
  }
  float m = -INFINITY, s = 0.f, t = 0.f;
  for (int d0 = 0; d0 < D; d0 += 8) {
    float v[8];
    float cm = -INFINITY;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      v[i] = (d0 + i < D) ? __ldg(p + (size_t)(d0 + i) * HW) * alpha : -INFINITY;
      cm = fmaxf(cm, v[i]);
    }
    const float nm = fmaxf(m, cm);
    if (nm == -INFINITY) continue;                     // every logit so far is -inf
    const float sc = expf(m - nm);                     // exp(-inf) = 0 on the first chunk
    s *= sc, t *= sc;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float e = expf(v[i] - nm);                 // padded bins: exp(-inf) = 0
      s += e;
      t = fmaf(e, start + step * (float)(d0 + i), t);
    }
    m = nm;
  }
  out[pix] = t / s;
}

// ------------------------------------------------------------------------------- fused trilinear + soft-argmin
// PyTorch's source-index rule (aten/src/ATen/native/UpSample.h, area_pixel_compute_source_index), in fp32 like aten:
//   align_corners: src = dst * (in-1)/(out-1);  else: src = max((dst + 0.5) * in/out - 0.5, 0)
struct Axis {
  float scale;
  int in, align;
  __device__ __forceinline__ void locate(int dst, int& i0, int& i1, float& l1) const {
    float src = align ? scale * (float)dst : fmaxf(scale * ((float)dst + 0.5f) - 0.5f, 0.f);
    i0 = min((int)src, in - 1);
    i1 = i0 + (i0 < in - 1 ? 1 : 0);
    l1 = src - (float)i0;
  }
};
__host__ inline Axis make_axis(int in, int out, int align) {
  Axis a;
  a.in = in, a.align = align;
  if (align)
    a.scale = out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f;
  else
    a.scale = (float)in / (float)out;
  return a;
}

// cost (B,Dl,Hl,Wl) low-res logits -> out (B,H,W).  aten nests the interpolation W innermost, D outermost, so the
// per-pixel bilinear value t(c) of coarse slice c is computed once and the fine samples whose lower neighbour is c are
// lerps between t(c) and t(c+1).  A lerp never exceeds max(t(c), t(c+1)), so the running maximum is updated once per
// coarse interval (one extra exp per interval instead of one per sample).  The fine->coarse map depends on d only; it
// is tabulated once per CTA in shared memory (lambda per fine sample, first fine sample per coarse interval).
// Logits are pre-scaled by log2(e) so every exponential is a single MUFU.EX2.
// VALUES: the value of fine bin d is values[b,d,h,w] (CasStereo's per-pixel hypotheses, casnet/cas_psm.py:268-274) instead
// of d; `values` is unused otherwise.
template <bool VALUES>
__global__ void __launch_bounds__(128) upsample_softargmin_kernel(const float* __restrict__ cost, float* __restrict__ out,
                                                                  int Dl, int Hl, int Wl, int D, int H, int W, Axis ad,
                                                                  Axis ah, Axis aw, const float* __restrict__ values) {
  extern __shared__ float s_tab[];
  float* s_lam = s_tab;                                  // [D]   weight of the upper neighbour
  int* s_first = reinterpret_cast<int*>(s_tab + D);      // [Dl+1] first fine sample of coarse interval c
  for (int c = threadIdx.x; c <= Dl; c += blockDim.x) s_first[c] = D;
  __syncthreads();
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    int i0, i1, p0 = -1, p1;
    float l1, pl;
    ad.locate(d, i0, i1, l1);
    if (d > 0) ad.locate(d - 1, p0, p1, pl);
    s_lam[d] = l1;
    for (int c = p0 + 1; c <= i0; ++c) s_first[c] = d;   // i0 is non-decreasing in d
  }
  __syncthreads();

  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int y = blockIdx.y;
  const int b = blockIdx.z;
  if (x >= W) return;
  int y0, y1, x0, x1;
  float ly, lx;
  ah.locate(y, y0, y1, ly);
  aw.locate(x, x0, x1, lx);
  constexpr float kLog2e = 1.4426950408889634f;
  const float hy = (1.f - ly) * kLog2e, hx = 1.f - lx;
  ly *= kLog2e;
  const size_t slice = (size_t)Hl * Wl;
  const float* base = cost + (size_t)b * Dl * slice;
  const float* p00 = base + (size_t)y0 * Wl + x0;
  const float* p01 = base + (size_t)y0 * Wl + x1;
  const float* p10 = base + (size_t)y1 * Wl + x0;
  const float* p11 = base + (size_t)y1 * Wl + x1;
  // raw corner values of one coarse slice; combined later so the loads have a whole interval to land
  float a0 = __ldg(p00), a1 = __ldg(p01), a2 = __ldg(p10), a3 = __ldg(p11);
  float t0 = hy * (hx * a0 + lx * a1) + ly * (hx * a2 + lx * a3);
  if (Dl > 1) {
    a0 = __ldg(p00 + slice), a1 = __ldg(p01 + slice), a2 = __ldg(p10 + slice), a3 = __ldg(p11 + slice);
  }
  const float* vpix = VALUES ? values + (size_t)b * D * H * W + (size_t)y * W + x : nullptr;
  float m = -INFINITY, s = 0.f, t = 0.f;
  for (int c = 0; c < Dl; ++c) {
    const float t1 = (c + 1 < Dl) ? hy * (hx * a0 + lx * a1) + ly * (hx * a2 + lx * a3) : t0;
    if (c + 2 < Dl) {                                    // prefetch slice c+2
      const size_t o = (size_t)(c + 2) * slice;
      a0 = __ldg(p00 + o), a1 = __ldg(p01 + o), a2 = __ldg(p10 + o), a3 = __ldg(p11 + o);
    }
    const int dbeg = s_first[c], dend = s_first[c + 1];
    if (dbeg < dend) {
      const float nm = fmaxf(m, fmaxf(t0, t1));
      const float sc = exp2f(m - nm);                    // exp2(-inf) = 0 on the first interval
      s *= sc, t *= sc;
      m = nm;
      const float dt = t1 - t0, tm = t0 - m;
      float fd = (float)dbeg;
      for (int d = dbeg; d < dend; ++d) {
        const float e = exp2f(fmaf(s_lam[d], dt, tm));   // (1-l)*t0 + l*t1 - m
        s += e;
        t = fmaf(e, VALUES ? __ldg(vpix + (size_t)d * H * W) : fd, t);
        fd += 1.f;
      }
    }
    t0 = t1;
  }
  out[((size_t)b * H + y) * W + x] = t / s;
}

// ------------------------------------------------------------------------------------------- per-image EPE partials
__global__ void __launch_bounds__(256) epe_partial_kernel(const float* __restrict__ pred, const float* __restrict__ gt,
                                                          float* __restrict__ out, int HW, float maxdisp) {
  const int b = blockIdx.y;
  const float* p = pred + (size_t)b * HW;
  const float* g = gt + (size_t)b * HW;
  float err = 0.f, cnt = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += gridDim.x * blockDim.x) {
    const float gv = __ldg(g + i);
    if (gv > 0.f && gv < maxdisp) {
      err += fabsf(gv - __ldg(p + i));
      cnt += 1.f;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    err += __shfl_xor_sync(0xffffffffu, err, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  __shared__ float se[8], sc[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) se[warp] = err, sc[warp] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    float e = 0.f, c = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) e += se[i], c += sc[i];
    atomicAdd(out + 2 * b + 0, e);
    atomicAdd(out + 2 * b + 1, c);
  }
}

}  // namespace osb

extern "C" {

int osb_softargmin_fwd(const float* cost, float* out, int B, int D, int H, int W, float alpha, float start, float step,
                       int normalize, osb_stream_t stream) {
  OSB_REQUIRE(cost && out, "softargmin: null pointer");
  OSB_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0, "softargmin: empty shape B=%d D=%d H=%d W=%d", B, D, H, W);
  const size_t HW = (size_t)H * W, total = HW * B;
  const unsigned blocks = (unsigned)((total + 255) / 256);
  osb::softargmin_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(cost, out, D, HW, total, alpha, start, step, normalize, nullptr,
                                                                    nullptr);
  osb::count_launch();
  return osb::check_launch("softargmin_kernel");
}

int osb_softargmin_var_fwd(const float* cost, const float* values, float* disp_out, float* var_out, int B, int D, int H, int W,
                           osb_stream_t stream) {
  OSB_REQUIRE(cost && disp_out, "softargmin_var: null pointer");
  OSB_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0, "softargmin_var: empty shape B=%d D=%d H=%d W=%d", B, D, H, W);
  const size_t HW = (size_t)H * W, total = HW * B;
  const unsigned blocks = (unsigned)((total + 255) / 256);
  osb::softargmin_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(cost, disp_out, D, HW, total, 1.f, 0.f, 1.f, 1, values, var_out);
  osb::count_launch();
  return osb::check_launch("softargmin_kernel");
}

int osb_upsample_softargmin_fwd(const float* cost, float* out, int B, int Dl, int Hl, int Wl, int D, int H, int W,
                                int align_corners, osb_stream_t stream) {
  OSB_REQUIRE(cost && out, "upsample_softargmin: null pointer");
  OSB_REQUIRE(B > 0 && Dl > 0 && Hl > 0 && Wl > 0 && D > 0 && H > 0 && W > 0, "upsample_softargmin: empty shape");
  OSB_REQUIRE(H <= 65535 && B <= 65535, "upsample_softargmin: grid too large");
  dim3 grid((W + 127) / 128, H, B);
  OSB_REQUIRE((size_t)(D + Dl + 1) * 4 <= 48 * 1024, "upsample_softargmin: D=%d too large for the shared tables", D);
  osb::upsample_softargmin_kernel<false><<<grid, 128, (size_t)(D + Dl + 1) * 4, (cudaStream_t)stream>>>(
      cost, out, Dl, Hl, Wl, D, H, W, osb::make_axis(Dl, D, align_corners), osb::make_axis(Hl, H, align_corners),
      osb::make_axis(Wl, W, align_corners), nullptr);
  osb::count_launch();
  return osb::check_launch("upsample_softargmin_kernel");
}

int osb_upsample_softargmin_values_fwd(const float* cost, const float* values, float* out, int B, int Dl, int Hl, int Wl, int D,
                                       int H, int W, int align_corners, osb_stream_t stream) {
  OSB_REQUIRE(cost && values && out, "upsample_softargmin_values: null pointer");
  OSB_REQUIRE(B > 0 && Dl > 0 && Hl > 0 && Wl > 0 && D > 0 && H > 0 && W > 0, "upsample_softargmin_values: empty shape");
  OSB_REQUIRE(H <= 65535 && B <= 65535, "upsample_softargmin_values: grid too large");
  dim3 grid((W + 127) / 128, H, B);
  OSB_REQUIRE((size_t)(D + Dl + 1) * 4 <= 48 * 1024, "upsample_softargmin_values: D=%d too large for the shared tables", D);
  osb::upsample_softargmin_kernel<true><<<grid, 128, (size_t)(D + Dl + 1) * 4, (cudaStream_t)stream>>>(
      cost, out, Dl, Hl, Wl, D, H, W, osb::make_axis(Dl, D, align_corners), osb::make_axis(Hl, H, align_corners),
      osb::make_axis(Wl, W, align_corners), values);
  osb::count_launch();
  return osb::check_launch("upsample_softargmin_kernel<values>");
}

int osb_epe_partial_fwd(const float* pred, const float* gt, float* out, int B, int HW, float maxdisp, osb_stream_t stream) {
  OSB_REQUIRE(pred && gt && out, "epe_partial: null pointer");
  OSB_REQUIRE(B > 0 && HW > 0 && B <= 65535, "epe_partial: bad shape B=%d HW=%d", B, HW);
  cudaError_t e = cudaMemsetAsync(out, 0, sizeof(float) * 2 * B, (cudaStream_t)stream);
  if (e != cudaSuccess) {
    osb::set_error("epe_partial: memset failed: %s", cudaGetErrorString(e));
    return OSB_ECUDA;
  }
  int bx = (HW + 256 * 8 - 1) / (256 * 8);
  if (bx < 1) bx = 1;
  if (bx > 64) bx = 64;
  osb::epe_partial_kernel<<<dim3(bx, B), 256, 0, (cudaStream_t)stream>>>(pred, gt, out, HW, maxdisp);
  osb::count_launch();
  return osb::check_launch("epe_partial_kernel");
}
}
