// Geometry-encoding volume lookup and convex ("context") up-sampling: SURVEY.md section 8(f) rows 1 and 3, the GRU-iteration
// hot spots of IGEV / StereoBase.
//   * geo_lookup_kernel     Combined_Geo_Encoding_Volume.__call__  stereo/modeling/models/igev/geometry.py:32-57 ==
//                           CombinedGeoEncodingVolume.__call__     stereo/modeling/models/stereobase/gru_blocks.py:195-220
//                           (bilinear_sampler = grid_sample(align_corners=True, zeros) igev/utils.py:61-79)
//                           and, with no correlation rows, Geo_Encoding_Volume.__call__ stereo/modeling/models/igev_rt/geometry.py:18-33
//   * avgpool_pairs_kernel  the F.avg_pool2d(.., [1,2], stride=[1,2]) pyramid of geometry.py:24-30
//   * context_upsample_kernel  context_upsample  stereo/modeling/models/stereobase/igev_blocks.py:51-63
// The reference materialises, per GRU iteration and level, a (B*H*W, C, 1, D) permuted copy of the volume (once), two grid
// tensors, two grid_sample outputs, a cat and a permute (~100 MB written per iteration at config 5).  Here the geometry
// volume stays in its native (B, C, D, H, W) layout -- neighbouring pixels have neighbouring disparities, so a warp's taps
// for one (channel, tap) hit one or two 128-byte rows -- and one kernel writes the (B, L*(C+1)*(2r+1), H, W) feature map
// directly.  HBM/gather-bound: (C+1)*(2r+1)*L floats written per pixel, about as many sectors read.
#include <algorithm>

#include "common.cuh"

namespace osb {

constexpr int GEO_MAX_LEVELS = 4;

struct GeoParams {
  const float* geo[GEO_MAX_LEVELS];    // level i: (B, C, D >> i, H, W)
  const float* corr[GEO_MAX_LEVELS];   // level i: (B, H, W, W2 >> i); all NULL = geometry-only lookup (no correlation row)
  const float* disp;                   // (B, 1, H, W)
  const float* coords;                 // (B, H, W) left-image x coordinate of every pixel (unused when geometry-only)
  float* out;                          // (B, L * (C + 1) * (2r + 1), H, W), geometry-only (B, L * C * (2r + 1), H, W),
                                       // multi-range (B, L * C * (2r + 1), H, W): the geo_volume0 pyramid rows only
  // multi-range mode (IGEV++'s Combined_Geo_Encoding_Volume), on when out_corr != NULL: two more single-level volumes, each
  // with its own plane count, sampled at dx + disp / 2 and dx + disp / 4, and the correlation rows in a tensor of their own
  const float* vol1;                   // (B, C, D1, H, W)
  const float* vol2;                   // (B, C, D2, H, W)
  float* out1;                         // (B, C * (2r + 1), H, W)
  float* out2;                         // (B, C * (2r + 1), H, W)
  float* out_corr;                     // (B, L * (2r + 1), H, W)
  int B, C, D, H, W, W2, levels, radius, D1, D2;
};

// The reference turns a pixel coordinate into a normalised grid value and grid_sample turns it back
// (align_corners=True): x -> 2x/(L-1) - 1 -> ((g + 1)/2)(L-1).  The round trip is replayed operation by operation (IEEE
// fp32, no contraction possible between a division and a subtraction) so that the interpolation weights carry the same
// rounding as the reference's.
__device__ __forceinline__ float roundtrip(float x, int len) {
  const float g = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, x), (float)(len - 1)), 1.f);
  return __fmul_rn(__fadd_rn(g, 1.f), 0.5f * (float)(len - 1));
}

// zero-padded linear interpolation of a strided row
__device__ __forceinline__ float lerp_row(const float* __restrict__ row, size_t stride, int len, float ix) {
  const float fl = floorf(ix);
  const int i0 = (int)fl;
  const float w1 = __fsub_rn(ix, fl), w0 = __fsub_rn(__fadd_rn(fl, 1.f), ix);
  const float v0 = (i0 >= 0 && i0 < len) ? __ldg(row + (size_t)i0 * stride) : 0.f;
  const float v1 = (i0 + 1 >= 0 && i0 + 1 < len) ? __ldg(row + (size_t)(i0 + 1) * stride) : 0.f;
  return __fadd_rn(__fmul_rn(v0, w0), __fmul_rn(v1, w1));
}

// One thread = one pixel x one "row" (a geometry channel of a level, or a level's correlation row): 2r+1 taps that, up to
// coordinate rounding, slide over one window of 2r+2 consecutive samples.  The window is loaded once (zero padded) and each
// tap picks its two samples from registers; a tap whose floor() does not land on window slot k (possible only when the
// coordinate round trip moves it across an integer) falls back to a direct read.  RADIUS = 0 is the generic path.  With
// corr[0] == NULL (IGEV-RT's Geo_Encoding_Volume) a level has only its C geometry rows: a runtime mode, not an instantiation.
// With out_corr != NULL (IGEV++'s multi-range Combined_Geo_Encoding_Volume) a batch item has L*C rows of the geo[] pyramid, C rows
// of vol1, C rows of vol2 and L correlation rows, each written to its own output tensor: a third runtime mode.
template <int RADIUS>
__global__ void __launch_bounds__(128) geo_lookup_kernel(const GeoParams p) {
  const int w = blockIdx.x * 128 + threadIdx.x;
  const int h = blockIdx.y;
  if (w >= p.W) return;
  const size_t hw = (size_t)p.H * p.W, pix = (size_t)h * p.W + w;
  const int radius = RADIUS > 0 ? RADIUS : p.radius;
  const int taps = 2 * radius + 1;
  // this thread's row: batch item b, pyramid level lvl, sampled at disp / 2^shift; geometry channel c of a volume of len planes
  // (vol1 / vol2 when src > 0), or the correlation row of level lvl
  int b, lvl, c, shift, src = 0;
  bool is_corr;
  float* o;
  if (p.out_corr == nullptr) {
    const int rows = p.corr[0] != nullptr ? p.C + 1 : p.C;
    b = blockIdx.z / (p.levels * rows);
    const int lr = blockIdx.z % (p.levels * rows);
    lvl = lr / rows, c = lr % rows, shift = lvl, is_corr = c == p.C;
    o = p.out + (((size_t)b * p.levels + lvl) * rows * taps + (size_t)c * taps) * hw + pix;
  } else {
    const int rows = p.levels * p.C + 2 * p.C + p.levels;
    b = blockIdx.z / rows;
    int r = blockIdx.z % rows;
    if (r < p.levels * p.C) {                          // geo_feat0: level, then channel, then tap
      lvl = r / p.C, c = r % p.C, shift = lvl, is_corr = false;
      o = p.out + (((size_t)b * p.levels + lvl) * p.C + c) * taps * hw + pix;
    } else if ((r -= p.levels * p.C) < 2 * p.C) {      // geo_feat1 at disp / 2, geo_feat2 at disp / 4
      lvl = 0, c = r % p.C, src = 1 + r / p.C, shift = src, is_corr = false;
      o = (src == 1 ? p.out1 : p.out2) + ((size_t)b * p.C + c) * taps * hw + pix;
    } else {                                           // init_corr
      lvl = r - 2 * p.C, c = 0, shift = lvl, is_corr = true;
      o = p.out_corr + ((size_t)b * p.levels + lvl) * taps * hw + pix;
    }
  }
  const float disp = __ldg(p.disp + (size_t)b * hw + pix);
  const float scale = 1.f / (float)(1 << shift);       // exact
  const float dq = disp * scale;                       // disp / 2^shift, exact
  const float* row;
  size_t stride;
  int len;
  float base;                                          // tap k samples at base + (k - radius): the reference adds dx + base for
                                                       // the geometry rows and base + dx for the correlation (same fp32 sum)
  // constant indices only: a runtime index would make the compiler copy the pointer arrays to local memory
  if (!is_corr) {
    const float* geo = src == 1 ? p.vol1 : src == 2 ? p.vol2
                     : lvl == 0 ? p.geo[0] : lvl == 1 ? p.geo[1] : lvl == 2 ? p.geo[2] : p.geo[3];
    len = src == 1 ? p.D1 : src == 2 ? p.D2 : p.D >> lvl;
    row = geo + ((size_t)b * p.C + c) * len * hw + pix;
    stride = hw;
    base = dq;                                         // geometry.py:22-26 adds dx + disp / 2^i: the same fp32 sum
  } else {
    const float* corr = lvl == 0 ? p.corr[0] : lvl == 1 ? p.corr[1] : lvl == 2 ? p.corr[2] : p.corr[3];
    len = p.W2 >> lvl;
    row = corr + ((size_t)b * hw + pix) * len;
    stride = 1;
    base = __fsub_rn(__ldg(p.coords + (size_t)b * hw + pix) * scale, dq);            // coords / 2^lvl - disp / 2^lvl
  }
  if (RADIUS > 0) {
    constexpr int T = 2 * RADIUS + 1;
    const float x0 = roundtrip(__fadd_rn((float)(-RADIUS), base), len);
    const int i0 = (int)floorf(x0);
    float win[T + 1];
#pragma unroll
    for (int j = 0; j <= T; ++j) {
      const int i = i0 + j;
      win[j] = (i >= 0 && i < len) ? __ldg(row + (size_t)i * stride) : 0.f;
    }
#pragma unroll
    for (int k = 0; k < T; ++k) {
      const float ix = roundtrip(__fadd_rn((float)(k - RADIUS), base), len);
      const float fl = floorf(ix);
      float v;
      if ((int)fl == i0 + k) {
        const float w1 = __fsub_rn(ix, fl), w0 = __fsub_rn(__fadd_rn(fl, 1.f), ix);
        v = __fadd_rn(__fmul_rn(win[k], w0), __fmul_rn(win[k + 1], w1));
      } else {
        v = lerp_row(row, stride, len, ix);
      }
      o[(size_t)k * hw] = v;
    }
  } else {
    for (int k = 0; k < taps; ++k)
      o[(size_t)k * hw] = lerp_row(row, stride, len, roundtrip(__fadd_rn((float)(k - radius), base), len));
  }
}

// y[o, k, i] = (x[o, 2k, i] + x[o, 2k+1, i]) / 2 for k < n/2 (a trailing odd element is dropped, as avg_pool2d does)
__global__ void __launch_bounds__(256) avgpool_pairs_kernel(const float* __restrict__ x, float* __restrict__ y, size_t outer, int n,
                                                            size_t inner) {
  const int half = n / 2;
  const size_t total = outer * half * inner;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (size_t)gridDim.x * 256) {
    const size_t in = i % inner, k = (i / inner) % half, o = i / (inner * half);
    const float* src = x + (o * n + 2 * k) * inner + in;
    y[i] = __fmul_rn(__fadd_rn(__ldg(src), __ldg(src + inner)), 0.5f);
  }
}

// out[b, Y, X] = sum_k up[b, k, Y, X] * disp_low[b, Y/s + k/3 - 1, X/s + k%3 - 1]   (zero padded), one thread = 4 columns
__global__ void __launch_bounds__(128) context_upsample_kernel(const float* __restrict__ disp, const float* __restrict__ up,
                                                               float* __restrict__ out, int h, int w, int s) {
  const int H = h * s, W = w * s;
  const int X = (blockIdx.x * 128 + threadIdx.x) * 4, Y = blockIdx.y, b = blockIdx.z;
  if (X >= W) return;
  const float* dl = disp + (size_t)b * h * w;
  const float* u = up + (size_t)b * 9 * H * W + (size_t)Y * W + X;
  float* o = out + ((size_t)b * H + Y) * W + X;
  const int y0 = Y / s;
  const bool vec = (W % 4 == 0) && (s % 4 == 0) && ((reinterpret_cast<uintptr_t>(u) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(o) & 15) == 0) && (((size_t)H * W) % 4 == 0);
  if (vec) {                                           // the four columns share one low-resolution cell
    const int x0 = X / s;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const int yy = y0 + k / 3 - 1, xx = x0 + k % 3 - 1;
      const float d = (yy >= 0 && yy < h && xx >= 0 && xx < w) ? __ldg(dl + (size_t)yy * w + xx) : 0.f;
      const float4 wv = __ldg(reinterpret_cast<const float4*>(u + (size_t)k * H * W));
      acc.x = fmaf(wv.x, d, acc.x), acc.y = fmaf(wv.y, d, acc.y), acc.z = fmaf(wv.z, d, acc.z), acc.w = fmaf(wv.w, d, acc.w);
    }
    *reinterpret_cast<float4*>(o) = acc;
  } else {
    for (int j = 0; j < 4 && X + j < W; ++j) {
      const int x0 = (X + j) / s;
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const int yy = y0 + k / 3 - 1, xx = x0 + k % 3 - 1;
        const float d = (yy >= 0 && yy < h && xx >= 0 && xx < w) ? __ldg(dl + (size_t)yy * w + xx) : 0.f;
        acc = fmaf(__ldg(u + (size_t)k * H * W + j), d, acc);
      }
      o[j] = acc;
    }
  }
}

}  // namespace osb

extern "C" {

int osb_avgpool_pairs_fwd(const float* x, float* y, long long outer, int n, long long inner, osb_stream_t stream) {
  using namespace osb;
  OSB_REQUIRE(x && y, "avgpool_pairs: null pointer");
  OSB_REQUIRE(outer > 0 && n >= 2 && inner > 0, "avgpool_pairs: bad shape outer=%lld n=%d inner=%lld", outer, n, inner);
  const long long total = outer * (n / 2) * inner;
  const unsigned blocks = (unsigned)std::min<long long>((total + 255) / 256, (long long)osb::sm_count() * 32);
  avgpool_pairs_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(x, y, (size_t)outer, n, (size_t)inner);
  count_launch();
  return check_launch("avgpool_pairs_kernel");
}

int osb_geo_lookup_fwd(const float* geo0, const float* geo1, const float* geo2, const float* geo3, const float* corr0,
                       const float* corr1, const float* corr2, const float* corr3, const float* disp, const float* coords,
                       float* out, int B, int C, int D, int H, int W, int W2, int num_levels, int radius, osb_stream_t stream) {
  using namespace osb;
  OSB_REQUIRE(disp && coords && out, "geo_lookup: null pointer");
  OSB_REQUIRE(B > 0 && C > 0 && D > 0 && H > 0 && W > 0 && W2 > 0, "geo_lookup: empty shape");
  OSB_REQUIRE(num_levels >= 1 && num_levels <= GEO_MAX_LEVELS, "geo_lookup: num_levels %d outside 1..%d", num_levels, GEO_MAX_LEVELS);
  OSB_REQUIRE(radius >= 0 && radius <= 16, "geo_lookup: radius %d outside 0..16", radius);
  OSB_REQUIRE((D >> (num_levels - 1)) >= 2 && (W2 >> (num_levels - 1)) >= 2, "geo_lookup: pyramid level shorter than 2 samples");
  OSB_REQUIRE(H <= 65535 && B <= 65535, "geo_lookup: H and B must fit a grid dimension");
  GeoParams p{};
  const float* g[GEO_MAX_LEVELS] = {geo0, geo1, geo2, geo3};
  const float* c[GEO_MAX_LEVELS] = {corr0, corr1, corr2, corr3};
  for (int i = 0; i < num_levels; ++i) {
    OSB_REQUIRE(g[i] && c[i], "geo_lookup: pyramid level %d is null", i);
    p.geo[i] = g[i], p.corr[i] = c[i];
  }
  p.disp = disp, p.coords = coords, p.out = out;
  p.B = B, p.C = C, p.D = D, p.H = H, p.W = W, p.W2 = W2, p.levels = num_levels, p.radius = radius;
  OSB_REQUIRE((long long)B * num_levels * (C + 1) <= 65535, "geo_lookup: B * levels * (C + 1) must fit a grid dimension");
  dim3 grid((W + 127) / 128, H, B * num_levels * (C + 1));
  if (radius == 4) geo_lookup_kernel<4><<<grid, 128, 0, (cudaStream_t)stream>>>(p);      // IGEV / StereoBase default (corr_radius 4)
  else geo_lookup_kernel<0><<<grid, 128, 0, (cudaStream_t)stream>>>(p);
  count_launch();
  return check_launch("geo_lookup_kernel");
}

int osb_geo_volume_lookup_fwd(const float* geo0, const float* geo1, const float* geo2, const float* geo3, const float* disp,
                              float* out, int B, int C, int D, int H, int W, int num_levels, int radius, osb_stream_t stream) {
  using namespace osb;
  OSB_REQUIRE(disp && out, "geo_volume_lookup: null pointer");
  OSB_REQUIRE(B > 0 && C > 0 && D > 0 && H > 0 && W > 0, "geo_volume_lookup: empty shape");
  OSB_REQUIRE(num_levels >= 1 && num_levels <= GEO_MAX_LEVELS, "geo_volume_lookup: num_levels %d outside 1..%d", num_levels,
              GEO_MAX_LEVELS);
  OSB_REQUIRE(radius >= 0 && radius <= 16, "geo_volume_lookup: radius %d outside 0..16", radius);
  OSB_REQUIRE((D >> (num_levels - 1)) >= 2, "geo_volume_lookup: pyramid level shorter than 2 samples");
  OSB_REQUIRE(H <= 65535 && B <= 65535, "geo_volume_lookup: H and B must fit a grid dimension");
  GeoParams p{};                                       // p.corr stays NULL: the kernel's geometry-only mode
  const float* g[GEO_MAX_LEVELS] = {geo0, geo1, geo2, geo3};
  for (int i = 0; i < num_levels; ++i) {
    OSB_REQUIRE(g[i], "geo_volume_lookup: pyramid level %d is null", i);
    p.geo[i] = g[i];
  }
  p.disp = disp, p.coords = nullptr, p.out = out;
  p.B = B, p.C = C, p.D = D, p.H = H, p.W = W, p.W2 = 0, p.levels = num_levels, p.radius = radius;
  OSB_REQUIRE((long long)B * num_levels * C <= 65535, "geo_volume_lookup: B * levels * C must fit a grid dimension");
  dim3 grid((W + 127) / 128, H, B * num_levels * C);
  if (radius == 4) geo_lookup_kernel<4><<<grid, 128, 0, (cudaStream_t)stream>>>(p);      // IGEV-RT default (CORR_RADIUS 4)
  else geo_lookup_kernel<0><<<grid, 128, 0, (cudaStream_t)stream>>>(p);
  count_launch();
  return check_launch("geo_lookup_kernel");
}

int osb_geo_multirange_lookup_fwd(const float* geo0, const float* geo1, const float* geo2, const float* geo3, const float* vol1,
                                  const float* vol2, const float* corr0, const float* corr1, const float* corr2, const float* corr3,
                                  const float* disp, const float* coords, float* out0, float* out1, float* out2, float* out_corr,
                                  int B, int C, int D0, int D1, int D2, int H, int W, int W2, int num_levels, int radius,
                                  osb_stream_t stream) {
  using namespace osb;
  OSB_REQUIRE(vol1 && vol2 && disp && coords && out0 && out1 && out2 && out_corr, "geo_multirange_lookup: null pointer");
  OSB_REQUIRE(B > 0 && C > 0 && D0 > 0 && D1 > 0 && D2 > 0 && H > 0 && W > 0 && W2 > 0, "geo_multirange_lookup: empty shape");
  OSB_REQUIRE(num_levels >= 1 && num_levels <= GEO_MAX_LEVELS, "geo_multirange_lookup: num_levels %d outside 1..%d", num_levels,
              GEO_MAX_LEVELS);
  OSB_REQUIRE(radius >= 0 && radius <= 16, "geo_multirange_lookup: radius %d outside 0..16", radius);
  OSB_REQUIRE((D0 >> (num_levels - 1)) >= 2 && (W2 >> (num_levels - 1)) >= 2 && D1 >= 2 && D2 >= 2,
              "geo_multirange_lookup: a volume or pyramid level shorter than 2 samples");
  OSB_REQUIRE(H <= 65535 && B <= 65535, "geo_multirange_lookup: H and B must fit a grid dimension");
  OSB_REQUIRE((long long)B * (num_levels * C + 2 * C + num_levels) <= 65535,
              "geo_multirange_lookup: B * (levels * C + 2 * C + levels) must fit a grid dimension");
  GeoParams p{};
  const float* g[GEO_MAX_LEVELS] = {geo0, geo1, geo2, geo3};
  const float* c[GEO_MAX_LEVELS] = {corr0, corr1, corr2, corr3};
  for (int i = 0; i < num_levels; ++i) {
    OSB_REQUIRE(g[i] && c[i], "geo_multirange_lookup: pyramid level %d is null", i);
    p.geo[i] = g[i], p.corr[i] = c[i];
  }
  p.vol1 = vol1, p.vol2 = vol2, p.disp = disp, p.coords = coords;
  p.out = out0, p.out1 = out1, p.out2 = out2, p.out_corr = out_corr;                    // out_corr != NULL: the multi-range mode
  p.B = B, p.C = C, p.D = D0, p.D1 = D1, p.D2 = D2, p.H = H, p.W = W, p.W2 = W2, p.levels = num_levels, p.radius = radius;
  dim3 grid((W + 127) / 128, H, B * (num_levels * C + 2 * C + num_levels));
  if (radius == 4) geo_lookup_kernel<4><<<grid, 128, 0, (cudaStream_t)stream>>>(p);      // IGEV++ default (CORR_RADIUS 4)
  else geo_lookup_kernel<0><<<grid, 128, 0, (cudaStream_t)stream>>>(p);
  count_launch();
  return check_launch("geo_lookup_kernel");
}

int osb_context_upsample_fwd(const float* disp_low, const float* up_weights, float* out, int B, int h, int w, int scale,
                             osb_stream_t stream) {
  using namespace osb;
  OSB_REQUIRE(disp_low && up_weights && out, "context_upsample: null pointer");
  OSB_REQUIRE(B > 0 && h > 0 && w > 0 && scale >= 1, "context_upsample: bad shape");
  OSB_REQUIRE((long long)h * scale <= 65535 && B <= 65535, "context_upsample: output height and B must fit a grid dimension");
  dim3 grid((w * scale + 511) / 512, h * scale, B);
  context_upsample_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(disp_low, up_weights, out, h, w, scale);
  count_launch();
  return check_launch("context_upsample_kernel");
}
}
