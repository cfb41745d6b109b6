// Warped cost volumes of the cascade models (CasStereo: CasPSMNet / CasGwcNet) for sm_90a.
//
//   GetCostVolume.forward  stereo/modeling/models/casnet/cas_psm.py:286-318   [x repeated over D | grid_sample(y)]
//   GetCostVolume.forward  stereo/modeling/models/casnet/cas_gwc.py:263-329   [gwc(x_warped, y_warped) | x_warped | y_warped]
//
// Every stage of a cascade samples the right features at a fractional, per-pixel hypothesis disp[b,d,h,w] (arbitrary per
// (b, d, h, w): not linear in d, possibly negative or beyond either edge) through
//   F.grid_sample(y, grid, 'bilinear', padding_mode='zeros', align_corners=True),  grid = ((w - disp)/((W-1)/2) - 1, h/((H-1)/2) - 1)
// and CasGwcNet zeroes the left features where w < disp.  The reference materialises meshgrid repeats, the (B,D,H,W,2) grid,
// a warped copy of the right features, a repeated copy of the left, their product and a torch.cat; here ONE launch writes
// the final (B, Cout, D, H, W) fp32 volume, every element exactly once (masked entries as exact zeros, so no memset).
//
// Work decomposition.  A CTA owns one image row (b, h) and one "unit": a correlation group (K channels) or a chunk of <= 8
// concatenation channels.  The row coordinate of the grid is the same for the whole row, so the CTA stages the unit's right
// feature rows y0 = floor(iy) and, when the coordinate round trip left the integer, y0 + 1 in shared memory (zero rows
// outside the image).  A thread owns one column at a time: it keeps the unit's left values in registers across the D
// planes, computes the column coordinate and the four bilinear weights once per plane, and gathers its two (or four) taps
// per channel from shared memory.  Consecutive threads own consecutive columns, so every store of a warp is one 128-byte
// row segment of an output plane.
//
// Arithmetic.  The coordinate round trip is replayed operation by operation (grid value, then aten's unnormalisation
// (g + 1) * ((size - 1) / 2)), and the interpolation follows aten's vectorised CPU grid sampler: weights nw = s*e,
// ne = s*w, sw = n*e, se = n*w, then v_nw*nw, fused multiply-adds of the ne, sw and se taps in that order.  The warped
// right features therefore match the reference bit for bit; the group mean sums the K products in order and divides by K.
//
// Disparity-warp mode (border = 1, MonSter's disp_warp, monster/warp.py): a concatenation unit with D = 1 that writes only the
// warped right features to an NCHW (B, C, H, W) output.  The grid is MonSter's normalize_coords, g = 2 * (v / (size - 1)) - 1
// with v = w - disp for x and v = h for y, sampled with align_corners=False and padding_mode='border'.  aten's vectorised CPU
// sampler unnormalises that as (g + 1) * (size / 2) - 0.5, which its build contracts into one fused multiply-add, then clamps
// to [0, size - 1] before the floor; the kernel does the same, so the warped features match the reference's CPU disp_warp bit
// for bit.  The row coordinate is not an integer here (about h * H / (H - 1) - 0.5), so rows y0 and y0 + 1 are both real taps.
//
// Roofline: HBM-bound.  Algorithmic bytes = 4*(2*B*C*H*W + B*D*H*W + B*Cout*D*H*W)  (both feature maps of each pair,
// the hypotheses, the volume).
#include "common.cuh"

namespace osb {

constexpr int kCasThreads = 128;
constexpr int kCasCatChunk = 8;   // concatenation channels per unit

struct WarpParams {
  const float* xg;     // gwc features (B, Cg, H, W): left / right; NULL when Cg = 0
  const float* yg;
  const float* xc;     // concatenation features (B, Cc, H, W)
  const float* yc;
  const float* disp;   // (B, D, H, W) hypotheses at the volume's resolution
  float* out;          // (B, Ctot, D, H, W)
  int B, Cg, G, K, Cc, D, H, W;
  int Ctot, oc_cat;    // output channels; first concatenation channel (= G)
  int n_gwc_units, n_cat_units;
  int mask_left;       // zero the left copy where w < disp (CasGwcNet) or not (CasPSMNet)
  int border;          // disparity-warp mode: MonSter's coordinates, border padding, warped right features only
  float half_w, half_h;  // (W - 1) / 2, (H - 1) / 2
  float wm1, hm1;        // W - 1, H - 1
};

// grid value and grid_sample's unnormalisation of it (align_corners=True), IEEE fp32 without contraction
__device__ __forceinline__ float cas_roundtrip(float v, float half) {
  const float g = __fsub_rn(__fdiv_rn(v, half), 1.f);
  return __fmul_rn(__fadd_rn(g, 1.f), half);
}

// MonSter's normalize_coords, then grid_sample's align_corners=False unnormalisation as aten's vectorised CPU sampler computes
// it, fmaf(g + 1, size / 2, -0.5), and the border clamp to [0, size - 1]; IEEE fp32 otherwise without contraction
__device__ __forceinline__ float border_roundtrip(float v, float sizem1) {
  const float g = __fsub_rn(__fmul_rn(2.f, __fdiv_rn(v, sizem1)), 1.f);
  const float u = fmaf(__fadd_rn(g, 1.f), __fmul_rn(__fadd_rn(sizem1, 1.f), 0.5f), -0.5f);
  return fminf(fmaxf(u, 0.f), sizem1);
}

// KMAX: compile-time bound of the channels a unit stages (gwc: K; concatenation: kCasCatChunk)
template <int KMAX>
__global__ void __launch_bounds__(kCasThreads) warped_volume_kernel(const WarpParams p) {
  extern __shared__ __align__(16) float s_rows[];         // [KMAX][2][W]: rows y0 and y0 + 1 of each staged channel
  const int units = p.n_gwc_units + p.n_cat_units;
  const int unit = blockIdx.x % units;
  const int h = (blockIdx.x / units) % p.H;
  const int b = blockIdx.x / (units * p.H);
  const bool gwc = unit < p.n_gwc_units;
  const int nch = gwc ? p.K : min(kCasCatChunk, p.Cc - (unit - p.n_gwc_units) * kCasCatChunk);
  const int c0 = gwc ? unit * p.K : (unit - p.n_gwc_units) * kCasCatChunk;   // first input channel of the unit
  const float* xsrc = (gwc ? p.xg : p.xc) + (((size_t)b * (gwc ? p.Cg : p.Cc) + c0) * p.H + h) * p.W;
  const float* ysrc = (gwc ? p.yg : p.yc) + ((size_t)b * (gwc ? p.Cg : p.Cc) + c0) * p.H * p.W;
  const size_t HW = (size_t)p.H * p.W;

  // row coordinate: the same for every sample of this CTA
  const float iy = p.border ? border_roundtrip((float)h, p.hm1) : cas_roundtrip((float)h, p.half_h);
  const float fy = floorf(iy);
  const int y0 = (int)fy;
  const float n = __fsub_rn(iy, fy), s = __fsub_rn(1.f, n);
  const bool two = n != 0.f;                                 // a tap with weight n*(...) = 0 adds exactly nothing

  for (int idx = threadIdx.x; idx < nch * (two ? 2 : 1) * p.W; idx += kCasThreads) {
    const int c = idx / ((two ? 2 : 1) * p.W), rem = idx - c * (two ? 2 : 1) * p.W;
    const int r = rem / p.W, w = rem - r * p.W;
    const int row = y0 + r;
    s_rows[((size_t)c * 2 + r) * p.W + w] = (row >= 0 && row < p.H) ? __ldg(ysrc + c * HW + (size_t)row * p.W + w) : 0.f;
  }
  __syncthreads();

  if (p.border) {      // disparity warp: D = 1, the warped right features only, (B, C, H, W); its own loop keeps the volume path's code
    const float* dsrc = p.disp + (size_t)b * HW + (size_t)h * p.W;
    float* dst = p.out + ((size_t)b * p.Cc + c0) * HW + (size_t)h * p.W;
    for (int w = threadIdx.x; w < p.W; w += kCasThreads) {
      const float ix = border_roundtrip(__fsub_rn((float)w, __ldg(dsrc + w)), p.wm1);   // in [0, W - 1]: x0 is a real column
      const float fx = floorf(ix);
      const int x0 = (int)fx;
      const float wx = __fsub_rn(ix, fx), e = __fsub_rn(1.f, wx);
      const float nw = __fmul_rn(s, e), ne = __fmul_rn(s, wx), sw = __fmul_rn(n, e), se = __fmul_rn(n, wx);
      const bool in1 = x0 + 1 < p.W;
#pragma unroll
      for (int c = 0; c < KMAX; ++c) {
        if (c < nch) {
          const float* r0 = s_rows + (size_t)c * 2 * p.W;
          float acc = __fmul_rn(r0[x0], nw);
          acc = fmaf(in1 ? r0[x0 + 1] : 0.f, ne, acc);
          if (two) {
            const float* r1 = r0 + p.W;
            acc = fmaf(r1[x0], sw, acc);
            acc = fmaf(in1 ? r1[x0 + 1] : 0.f, se, acc);
          }
          __stcs(dst + c * HW + w, acc);
        }
      }
    }
    return;
  }

  const float* dsrc = p.disp + (size_t)b * p.D * HW + (size_t)h * p.W;
  const float kf = (float)p.K;
  for (int w = threadIdx.x; w < p.W; w += kCasThreads) {
    float xl[KMAX];
#pragma unroll
    for (int c = 0; c < KMAX; ++c) xl[c] = c < nch ? __ldg(xsrc + c * HW + w) : 0.f;
    const float fw = (float)w;
    for (int d = 0; d < p.D; ++d) {
      const float sd = __ldg(dsrc + (size_t)d * HW + w);
      const float ix = cas_roundtrip(__fsub_rn(fw, sd), p.half_w);
      const bool masked = fw < sd;                           // CasGwcNet: x_warped[:, mw < disp] = 0
      float taps[KMAX];
      if (ix > -2.f && ix < (float)p.W + 1.f) {              // else both neighbours lie outside: zeros padding
        const float fx = floorf(ix);
        const int x0 = (int)fx;
        const float wx = __fsub_rn(ix, fx), e = __fsub_rn(1.f, wx);
        const float nw = __fmul_rn(s, e), ne = __fmul_rn(s, wx), sw = __fmul_rn(n, e), se = __fmul_rn(n, wx);
        const bool in0 = x0 >= 0 && x0 < p.W, in1 = x0 + 1 >= 0 && x0 + 1 < p.W;
#pragma unroll
        for (int c = 0; c < KMAX; ++c) {
          if (c < nch) {
            const float* r0 = s_rows + (size_t)c * 2 * p.W;
            float acc = __fmul_rn(in0 ? r0[x0] : 0.f, nw);
            acc = fmaf(in1 ? r0[x0 + 1] : 0.f, ne, acc);
            if (two) {
              const float* r1 = r0 + p.W;
              acc = fmaf(in0 ? r1[x0] : 0.f, sw, acc);
              acc = fmaf(in1 ? r1[x0 + 1] : 0.f, se, acc);
            }
            taps[c] = acc;
          }
        }
      } else {
#pragma unroll
        for (int c = 0; c < KMAX; ++c) taps[c] = 0.f;
      }
      if (gwc) {
        float acc = 0.f;
#pragma unroll
        for (int c = 0; c < KMAX; ++c)
          if (c < nch) acc = __fadd_rn(acc, __fmul_rn(xl[c], taps[c]));
        const int g = unit;
        __stcs(p.out + (((size_t)b * p.Ctot + g) * p.D + d) * HW + (size_t)h * p.W + w, masked ? 0.f : __fdiv_rn(acc, kf));
      } else {
        const bool zero_left = p.mask_left && masked;
#pragma unroll
        for (int c = 0; c < KMAX; ++c) {
          if (c < nch) {
            const int oc = p.oc_cat + c0 + c;
            __stcs(p.out + (((size_t)b * p.Ctot + oc) * p.D + d) * HW + (size_t)h * p.W + w, zero_left ? 0.f : xl[c]);
            __stcs(p.out + (((size_t)b * p.Ctot + oc + p.Cc) * p.D + d) * HW + (size_t)h * p.W + w, taps[c]);
          }
        }
      }
    }
  }
}

static int launch_warped(const WarpParams& p0, cudaStream_t stream) {
  WarpParams p = p0;
  OSB_REQUIRE(p.B > 0 && p.D > 0, "warped_volume: empty shape B=%d D=%d", p.B, p.D);
  OSB_REQUIRE(p.H >= 2 && p.W >= 2, "warped_volume: H=%d W=%d (the grid divides by (H-1)/2 and (W-1)/2: both must be >= 2)",
              p.H, p.W);
  OSB_REQUIRE(p.Cg >= 0 && p.Cc > 0, "warped_volume: Cg=%d Cc=%d", p.Cg, p.Cc);
  p.K = 0;
  if (p.Cg > 0) {
    OSB_REQUIRE(p.G > 0 && p.Cg % p.G == 0, "warped_gwc_volume: Cg=%d not divisible by num_groups=%d", p.Cg, p.G);
    p.K = p.Cg / p.G;
    OSB_REQUIRE(p.K <= 16, "warped_gwc_volume: %d channels per group exceed the 16 supported", p.K);
  } else {
    p.G = 0;
  }
  p.Ctot = p.border ? p.Cc : p.G + 2 * p.Cc;
  p.oc_cat = p.G;
  p.n_gwc_units = p.G;
  p.n_cat_units = (p.Cc + kCasCatChunk - 1) / kCasCatChunk;
  p.half_w = (float)((p.W - 1.0) / 2.0);
  p.half_h = (float)((p.H - 1.0) / 2.0);
  p.wm1 = (float)(p.W - 1);
  p.hm1 = (float)(p.H - 1);
  const int kmax = p.K > 8 ? 16 : 8;
  const size_t smem = (size_t)kmax * 2 * p.W * sizeof(float);
  OSB_REQUIRE(smem <= 227 * 1024, "warped_volume: W=%d needs %zu bytes of shared memory for %d staged channel rows (227 KB max)",
              p.W, smem, 2 * kmax);
  const long long blocks = (long long)(p.n_gwc_units + p.n_cat_units) * p.H * p.B;
  OSB_REQUIRE(blocks < (1ll << 31), "warped_volume: too many CTAs (%lld)", blocks);
  using Fn = void (*)(const WarpParams);
  const Fn kernel = kmax == 16 ? warped_volume_kernel<16> : warped_volume_kernel<8>;
  static size_t configured_all[64][2] = {};                   // cudaFuncSetAttribute is per device
  size_t& configured = configured_all[device_index() & 63][kmax == 16 ? 1 : 0];
  if (smem > 48 * 1024 && smem > configured) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
      set_error("warped_volume: cannot reserve %zu bytes of shared memory: %s", smem, cudaGetErrorString(e));
      return OSB_ECUDA;
    }
    configured = smem;
  }
  kernel<<<(unsigned)blocks, kCasThreads, smem, stream>>>(p);
  count_launch();
  return check_launch("warped_volume_kernel");
}

}  // namespace osb

extern "C" {

int osb_warped_concat_volume_fwd(const float* x, const float* y, const float* disp, float* out, int B, int C, int D, int H, int W,
                                 int mask_left, osb_stream_t stream) {
  OSB_REQUIRE(x && y && disp && out, "warped_concat_volume: null pointer");
  osb::WarpParams p{};
  p.xc = x, p.yc = y, p.disp = disp, p.out = out;
  p.B = B, p.Cg = 0, p.G = 0, p.Cc = C, p.D = D, p.H = H, p.W = W, p.mask_left = mask_left ? 1 : 0;
  return osb::launch_warped(p, (cudaStream_t)stream);
}

int osb_warped_gwc_concat_volume_fwd(const float* xg, const float* yg, const float* xc, const float* yc, const float* disp,
                                     float* out, int B, int Cg, int G, int Cc, int D, int H, int W, osb_stream_t stream) {
  OSB_REQUIRE(xg && yg && xc && yc && disp && out, "warped_gwc_concat_volume: null pointer");
  OSB_REQUIRE(Cg > 0, "warped_gwc_concat_volume: Cg=%d", Cg);
  osb::WarpParams p{};
  p.xg = xg, p.yg = yg, p.xc = xc, p.yc = yc, p.disp = disp, p.out = out;
  p.B = B, p.Cg = Cg, p.G = G, p.Cc = Cc, p.D = D, p.H = H, p.W = W, p.mask_left = 1;
  return osb::launch_warped(p, (cudaStream_t)stream);
}

int osb_disp_warp_fwd(const float* img, const float* disp, float* out, int B, int C, int H, int W, osb_stream_t stream) {
  OSB_REQUIRE(img && disp && out, "disp_warp: null pointer");
  osb::WarpParams p{};
  p.yc = img, p.disp = disp, p.out = out;
  p.B = B, p.Cg = 0, p.G = 0, p.Cc = C, p.D = 1, p.H = H, p.W = W, p.border = 1;
  return osb::launch_warped(p, (cudaStream_t)stream);
}
}
