// MSNet3D (stereo/modeling/models/msnet/) for sm_90a: one launch per MobileV2_Residual_3D block (msnet/submodule.py:136-173).
//
//   y = BN3(W_proj . relu6(BN2(dw3x3x3_stride(relu6(BN1(W_exp . x)))))) [+ residual]
//
// The reference materialises the expanded tensor twice per block (after the expansion and after the depthwise conv), each time
// followed by separate BN and ReLU6 passes.  Here the expanded tensor never leaves shared memory.
//
// A CTA owns a TH x TW tile of output rows/columns and marches along the output depth (a chunk of it when the grid would otherwise
// be short of two CTAs per SM).  It keeps a ring of the 3 expanded input planes the depthwise conv needs, over the tile's input
// halo ((S*(TH-1)+3) x (S*(TW-1)+3) voxels, all Chid channels).  Per output plane:
//   1. expand the new input plane(s) (one at stride 1, two at stride 2): stage x over the halo in shared memory, then a
//      halo x Chid register-tiled product (4 voxels x 4 channels per thread), folded BN1, ReLU6, into the ring slot of that plane;
//   2. depthwise 3x3x3 from the ring (4 output columns x 4 channels per thread), folded BN2, ReLU6, into a [voxel][channel] tile;
//   3. project (2 voxels x 4 output channels per thread, K = Chid), folded BN3, the optional residual, store.
// Only the H/W halo of the expansion is recomputed (1.7x at 4 x 16, stride 1); along D each input plane is expanded once per chunk.
//
// Padding rule: the depthwise conv zero-pads the HIDDEN tensor.  Halo voxels outside the volume (and whole planes outside [0, D))
// are written as exact zeros, not relu6(shift1) -- which is what expanding a zero-padded input would give.
//
// Stride 2 gives ceil(n / 2) outputs per dimension (k3, padding 1).  Any D, H, W works: partial tiles compute on zero halo and
// store only the voxels inside the output.
//
// Arithmetic: IEEE fp32 FMAs on the CUDA cores; the three BatchNorms are folded to scale/shift on the host.  Weights are read
// through the read-only path (w_exp (Cin, Chid), w_dw (27, Chid) tap-major, w_proj (Chid, Cout)); they stay in L1/L2.
#include "common.cuh"

namespace osb {

constexpr int kMbThreads = 256;

struct Mbv2Params {
  const float* x;
  const float* w_exp;
  const float* s1;
  const float* b1;
  const float* w_dw;
  const float* s2;
  const float* b2;
  const float* w_proj;
  const float* s3;
  const float* b3;
  const float* res;
  float* y;
  int D, H, W, Do, Ho, Wo;
  int tiles_w, dchunk;
  int in_cl, out_cl;  // 1 = NDHWC, 0 = NCDHW
};

template <int CIN, int CHID, int COUT, int S, int TH, int TW>
struct MbCfg {
  static constexpr int HH = S * (TH - 1) + 3, HW = S * (TW - 1) + 3;  // input halo of the tile
  static constexpr int P = HH * HW, P4 = (P + 3) / 4 * 4;
  static constexpr int TV = TH * TW;
  static constexpr int HS = CHID + 4;  // row stride of the depthwise output tile (padded: conflict-free reads in phase 3)
  static constexpr int RING = 3 * P * CHID;
  static constexpr int XS = CIN * P4;
  static constexpr int H2 = TV * HS;
  static constexpr int SCRATCH = XS > H2 ? XS : H2;  // x staging (phase 1) and the depthwise tile (phases 2-3) alias
  static constexpr size_t SMEM = (size_t)(RING + SCRATCH) * sizeof(float);
  static_assert(CHID % 4 == 0 && COUT % 4 == 0 && TW % 4 == 0, "channel quads and 4-column runs");
  static_assert(SMEM <= 227 * 1024, "shared memory");
};

__device__ __forceinline__ float relu6f(float v) { return fminf(fmaxf(v, 0.f), 6.f); }

__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

__device__ __forceinline__ void fma4(float (&a)[4], float s, const float4& w) {
  a[0] = fmaf(s, w.x, a[0]), a[1] = fmaf(s, w.y, a[1]), a[2] = fmaf(s, w.z, a[2]), a[3] = fmaf(s, w.w, a[3]);
}

// Phase 1: expanded input plane z -> ring slot (z mod 3), [halo voxel][Chid].
template <int CIN, int CHID, int COUT, int S, int TH, int TW>
__device__ __forceinline__ void mb_expand(const Mbv2Params& p, float* ring, float* xs, int b, int z, int iy0, int ix0) {
  using C = MbCfg<CIN, CHID, COUT, S, TH, TW>;
  float* slot = ring + ((z + 3) % 3) * (C::P * CHID);
  if (z < 0 || z >= p.D) {  // a plane of the hidden tensor's zero padding
    for (int i = threadIdx.x; i < C::P * CHID / 4; i += kMbThreads) reinterpret_cast<float4*>(slot)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    return;
  }
  const size_t plane = (size_t)p.H * p.W;
  if (!p.in_cl) {
    for (int i = threadIdx.x; i < CIN * C::P4; i += kMbThreads) {
      const int ci = i / C::P4, q = i - ci * C::P4;
      const int hy = q / C::HW, hx = q - hy * C::HW;
      const int yy = iy0 + hy, xx = ix0 + hx;
      float v = 0.f;
      if (q < C::P && yy >= 0 && yy < p.H && xx >= 0 && xx < p.W)
        v = __ldg(p.x + (((size_t)b * CIN + ci) * p.D + z) * plane + (size_t)yy * p.W + xx);
      xs[i] = v;
    }
  } else {
    for (int i = threadIdx.x; i < CIN * C::P4; i += kMbThreads) {
      const int q = i / CIN, ci = i - q * CIN;
      const int hy = q / C::HW, hx = q - hy * C::HW;
      const int yy = iy0 + hy, xx = ix0 + hx;
      float v = 0.f;
      if (q < C::P && yy >= 0 && yy < p.H && xx >= 0 && xx < p.W)
        v = __ldg(p.x + ((((size_t)b * p.D + z) * p.H + yy) * p.W + xx) * CIN + ci);
      xs[ci * C::P4 + q] = v;
    }
  }
  __syncthreads();
  constexpr int NQ = CHID / 4, NG = C::P4 / 4;
  for (int it = threadIdx.x; it < NQ * NG; it += kMbThreads) {
    const int cq = it % NQ, g = it / NQ;
    float acc[4][4] = {};
    const float* xp = xs + 4 * g;
    const float* wp = p.w_exp + 4 * cq;
#pragma unroll 8
    for (int ci = 0; ci < CIN; ++ci) {
      const float4 xv = *reinterpret_cast<const float4*>(xp + ci * C::P4);
      const float4 wv = ld4(wp + ci * CHID);
      fma4(acc[0], xv.x, wv), fma4(acc[1], xv.y, wv), fma4(acc[2], xv.z, wv), fma4(acc[3], xv.w, wv);
    }
    const float4 sc = ld4(p.s1 + 4 * cq), sh = ld4(p.b1 + 4 * cq);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int q = 4 * g + j;
      if (q >= C::P) break;
      const int hy = q / C::HW, hx = q - hy * C::HW;
      const int yy = iy0 + hy, xx = ix0 + hx;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (yy >= 0 && yy < p.H && xx >= 0 && xx < p.W)
        v = make_float4(relu6f(fmaf(acc[j][0], sc.x, sh.x)), relu6f(fmaf(acc[j][1], sc.y, sh.y)), relu6f(fmaf(acc[j][2], sc.z, sh.z)),
                        relu6f(fmaf(acc[j][3], sc.w, sh.w)));
      *reinterpret_cast<float4*>(slot + q * CHID + 4 * cq) = v;
    }
  }
  __syncthreads();
}

template <int CIN, int CHID, int COUT, int S, int TH, int TW>
__global__ void __launch_bounds__(kMbThreads, 1) mbv2_block3d_kernel(const Mbv2Params p) {
  using C = MbCfg<CIN, CHID, COUT, S, TH, TW>;
  extern __shared__ float4 smem4[];
  float* ring = reinterpret_cast<float*>(smem4);
  float* scratch = ring + C::RING;  // x staging [Cin][P4] in phase 1, depthwise output [TV][HS] in phases 2-3
  const int b = blockIdx.z;
  const int ty = blockIdx.x / p.tiles_w, tx = blockIdx.x - ty * p.tiles_w;
  const int oh0 = ty * TH, ow0 = tx * TW;
  const int iy0 = S * oh0 - 1, ix0 = S * ow0 - 1;
  const int od0 = blockIdx.y * p.dchunk;
  const int od1 = min(od0 + p.dchunk, p.Do);
  constexpr int NQ = CHID / 4, RUNS = TW / 4, NO = COUT / 4;
  constexpr int NCOL = 3 * S + 3;  // halo columns under 4 output columns

  if (S == 1) {
    mb_expand<CIN, CHID, COUT, S, TH, TW>(p, ring, scratch, b, od0 - 1, iy0, ix0);
    mb_expand<CIN, CHID, COUT, S, TH, TW>(p, ring, scratch, b, od0, iy0, ix0);
  } else {
    mb_expand<CIN, CHID, COUT, S, TH, TW>(p, ring, scratch, b, 2 * od0 - 1, iy0, ix0);
  }
  for (int od = od0; od < od1; ++od) {
    if (S == 1) {
      mb_expand<CIN, CHID, COUT, S, TH, TW>(p, ring, scratch, b, od + 1, iy0, ix0);
    } else {
      mb_expand<CIN, CHID, COUT, S, TH, TW>(p, ring, scratch, b, 2 * od, iy0, ix0);
      mb_expand<CIN, CHID, COUT, S, TH, TW>(p, ring, scratch, b, 2 * od + 1, iy0, ix0);
    }
    // ---- phase 2: depthwise 3x3x3, 4 output columns x 4 channels per item ----
    float* h2 = scratch;
    for (int it = threadIdx.x; it < TH * RUNS * NQ; it += kMbThreads) {
      const int cq = it % NQ, r = it / NQ;
      const int run = r % RUNS, row = r / RUNS;
      float acc[4][4] = {};
#pragma unroll
      for (int kd = 0; kd < 3; ++kd) {
        const float* sl = ring + ((S * od - 1 + kd + 3) % 3) * (C::P * CHID);
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
          const float* rp = sl + ((S * row + kh) * C::HW + S * 4 * run) * CHID + 4 * cq;
          float4 in[NCOL];
#pragma unroll
          for (int c = 0; c < NCOL; ++c) in[c] = *reinterpret_cast<const float4*>(rp + c * CHID);
#pragma unroll
          for (int kw = 0; kw < 3; ++kw) {
            const float4 w = ld4(p.w_dw + ((kd * 3 + kh) * 3 + kw) * CHID + 4 * cq);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const float4 v = in[S * j + kw];
              acc[j][0] = fmaf(v.x, w.x, acc[j][0]), acc[j][1] = fmaf(v.y, w.y, acc[j][1]);
              acc[j][2] = fmaf(v.z, w.z, acc[j][2]), acc[j][3] = fmaf(v.w, w.w, acc[j][3]);
            }
          }
        }
      }
      const float4 sc = ld4(p.s2 + 4 * cq), sh = ld4(p.b2 + 4 * cq);
#pragma unroll
      for (int j = 0; j < 4; ++j)
        *reinterpret_cast<float4*>(h2 + (row * TW + 4 * run + j) * C::HS + 4 * cq) =
            make_float4(relu6f(fmaf(acc[j][0], sc.x, sh.x)), relu6f(fmaf(acc[j][1], sc.y, sh.y)), relu6f(fmaf(acc[j][2], sc.z, sh.z)),
                        relu6f(fmaf(acc[j][3], sc.w, sh.w)));
    }
    __syncthreads();
    // ---- phase 3: projection, 2 voxels x 4 output channels per item ----
    for (int it = threadIdx.x; it < (C::TV / 2) * NO; it += kMbThreads) {
      const int oq = it % NO, v0 = 2 * (it / NO);
      float acc[2][4] = {};
      const float* h0 = h2 + v0 * C::HS;
      const float* wp = p.w_proj + 4 * oq;
#pragma unroll 4
      for (int c = 0; c < CHID; c += 4) {
        const float4 a0 = *reinterpret_cast<const float4*>(h0 + c);
        const float4 a1 = *reinterpret_cast<const float4*>(h0 + C::HS + c);
        const float4 w0 = ld4(wp + (c + 0) * COUT), w1 = ld4(wp + (c + 1) * COUT);
        const float4 w2 = ld4(wp + (c + 2) * COUT), w3 = ld4(wp + (c + 3) * COUT);
        fma4(acc[0], a0.x, w0), fma4(acc[0], a0.y, w1), fma4(acc[0], a0.z, w2), fma4(acc[0], a0.w, w3);
        fma4(acc[1], a1.x, w0), fma4(acc[1], a1.y, w1), fma4(acc[1], a1.z, w2), fma4(acc[1], a1.w, w3);
      }
      const float4 sc = ld4(p.s3 + 4 * oq), sh = ld4(p.b3 + 4 * oq);
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int v = v0 + j;
        const int oh = oh0 + v / TW, ow = ow0 + v % TW;
        if (oh >= p.Ho || ow >= p.Wo) continue;
        float o[4] = {fmaf(acc[j][0], sc.x, sh.x), fmaf(acc[j][1], sc.y, sh.y), fmaf(acc[j][2], sc.z, sh.z), fmaf(acc[j][3], sc.w, sh.w)};
        if (p.out_cl) {
          const size_t off = ((((size_t)b * p.Do + od) * p.Ho + oh) * p.Wo + ow) * COUT + 4 * oq;
          if (p.res) {
            const float4 r = ld4(p.res + off);
            o[0] += r.x, o[1] += r.y, o[2] += r.z, o[3] += r.w;
          }
          *reinterpret_cast<float4*>(p.y + off) = make_float4(o[0], o[1], o[2], o[3]);
        } else {
          const size_t vol = (size_t)p.Do * p.Ho * p.Wo;
          const size_t off = ((size_t)b * COUT + 4 * oq) * vol + ((size_t)od * p.Ho + oh) * p.Wo + ow;
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            float v = o[k];
            if (p.res) v += __ldg(p.res + off + k * vol);
            p.y[off + k * vol] = v;
          }
        }
      }
    }
    __syncthreads();  // the depthwise tile aliases the next expansion's x staging
  }
}

template <int CIN, int CHID, int COUT, int S, int TH, int TW>
int launch_mbv2(Mbv2Params p, int B, cudaStream_t stream) {
  using C = MbCfg<CIN, CHID, COUT, S, TH, TW>;
  auto kernel = mbv2_block3d_kernel<CIN, CHID, COUT, S, TH, TW>;
  static PerDeviceFlag configured;
  if (!configured.here()) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM);
    if (e != cudaSuccess) {
      set_error("mbv2_block3d: cannot reserve %zu bytes of shared memory: %s", C::SMEM, cudaGetErrorString(e));
      return OSB_ECUDA;
    }
    configured.here() = true;
  }
  const int tiles_h = (p.Ho + TH - 1) / TH, tiles_w = (p.Wo + TW - 1) / TW;
  p.tiles_w = tiles_w;
  // split the depth march while the grid is short of two CTAs per SM (each extra chunk re-expands 2 or 3 planes)
  const long long ctas = (long long)tiles_h * tiles_w * B, want = 2ll * sm_count();
  int dchunk = p.Do;
  while (dchunk > 4 && ctas * ((p.Do + dchunk - 1) / dchunk) < want) dchunk = (dchunk + 1) / 2;
  p.dchunk = dchunk;
  const dim3 grid((unsigned)(tiles_h * tiles_w), (unsigned)((p.Do + dchunk - 1) / dchunk), (unsigned)B);
  kernel<<<grid, kMbThreads, C::SMEM, stream>>>(p);
  count_launch();
  return check_launch("mbv2_block3d_kernel");
}

}  // namespace osb

extern "C" {

int osb_mbv2_block3d_fwd(const float* x, const float* w_exp, const float* scale1, const float* shift1, const float* w_dw,
                         const float* scale2, const float* shift2, const float* w_proj, const float* scale3, const float* shift3,
                         const float* residual, float* y, int B, int Cin, int Chid, int Cout, int D, int H, int W, int stride,
                         int in_layout, int out_layout, osb_stream_t stream) {
  using namespace osb;
  OSB_REQUIRE(x && w_exp && scale1 && shift1 && w_dw && scale2 && shift2 && w_proj && scale3 && shift3 && y,
              "mbv2_block3d: null pointer");
  OSB_REQUIRE(B > 0 && D > 0 && H > 0 && W > 0, "mbv2_block3d: empty shape B=%d D=%d H=%d W=%d", B, D, H, W);
  OSB_REQUIRE(B <= 65535, "mbv2_block3d: B=%d exceeds the grid", B);
  OSB_REQUIRE(stride == 1 || stride == 2, "mbv2_block3d: stride=%d (1 or 2)", stride);
  OSB_REQUIRE((in_layout == 0 || in_layout == 1) && (out_layout == 0 || out_layout == 1),
              "mbv2_block3d: layouts must be 0 (NCDHW) or 1 (NDHWC), got in=%d out=%d", in_layout, out_layout);
  OSB_REQUIRE(static_cast<const void*>(y) != static_cast<const void*>(x), "mbv2_block3d: y must not alias x");
  const void* aligned[] = {w_exp, scale1, shift1, w_dw, scale2, shift2, w_proj, scale3, shift3, out_layout ? y : nullptr,
                           out_layout ? residual : nullptr};
  for (const void* q : aligned) OSB_REQUIRE((reinterpret_cast<uintptr_t>(q) & 15) == 0, "mbv2_block3d: weights, BN vectors and "
                                            "a channels-last y / residual must be 16-byte aligned");
  Mbv2Params p{};
  p.x = x, p.w_exp = w_exp, p.s1 = scale1, p.b1 = shift1, p.w_dw = w_dw, p.s2 = scale2, p.b2 = shift2;
  p.w_proj = w_proj, p.s3 = scale3, p.b3 = shift3, p.res = residual, p.y = y;
  p.D = D, p.H = H, p.W = W;
  p.Do = (D - 1) / stride + 1, p.Ho = (H - 1) / stride + 1, p.Wo = (W - 1) / stride + 1;
  p.in_cl = in_layout, p.out_cl = out_layout;
  const cudaStream_t s = (cudaStream_t)stream;
  // the seven (Cin, Chid, Cout, stride) blocks MSNet3D builds (MSNet3D.py:13-27,63-69); output tile TH x TW per config
  if (Cin == 40 && Chid == 120 && Cout == 32 && stride == 1) return launch_mbv2<40, 120, 32, 1, 4, 16>(p, B, s);
  if (Cin == 32 && Chid == 96 && Cout == 32 && stride == 1) return launch_mbv2<32, 96, 32, 1, 4, 16>(p, B, s);
  if (Cin == 32 && Chid == 64 && Cout == 32 && stride == 1) return launch_mbv2<32, 64, 32, 1, 4, 16>(p, B, s);
  if (Cin == 32 && Chid == 64 && Cout == 64 && stride == 2) return launch_mbv2<32, 64, 64, 2, 4, 8>(p, B, s);
  if (Cin == 64 && Chid == 128 && Cout == 64 && stride == 1) return launch_mbv2<64, 128, 64, 1, 4, 8>(p, B, s);
  if (Cin == 64 && Chid == 128 && Cout == 128 && stride == 2) return launch_mbv2<64, 128, 128, 2, 4, 4>(p, B, s);
  if (Cin == 128 && Chid == 256 && Cout == 128 && stride == 1) return launch_mbv2<128, 256, 128, 1, 4, 4>(p, B, s);
  OSB_REQUIRE(false, "mbv2_block3d: (Cin, Chid, Cout, stride) = (%d, %d, %d, %d) is not instantiated (MSNet3D's blocks: (40,120,32,1) "
              "(32,96,32,1) (32,64,32,1) (32,64,64,2) (64,128,64,1) (64,128,128,2) (128,256,128,1))", Cin, Chid, Cout, stride);
  return OSB_EINVAL;
}
}
