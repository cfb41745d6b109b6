// Fused cost-volume constructor for sm_90a.
//
// Replaces the reference's Python loops of slice assignments
//   build_gwc_volume     stereo/modeling/cost_volume/cost_volume.py:68-78
//   build_concat_volume  stereo/modeling/cost_volume/cost_volume.py:81-92  (cat_fms, psmnet_cost_processor.py:9-50)
//   correlation_volume   stereo/modeling/cost_volume/cost_volume.py:32-41
//   torch.cat((gwc, concat), 1)  gwcnet_cost_processor.py:65
// with ONE launch that writes every output row exactly once (zeros of the w<d triangle included, so no memset).
//
// Work decomposition.  A work item is one image row (b, h), one 128-column tile, one chunk of <=64 disparities and one
// "unit" of GU output channels; the kernel is persistent (2 CTAs per SM, grid = a multiple of the SM count) and each CTA
// walks the item list through a two-stage shared-memory ring, so the TMA load of the next item overlaps the FMAs and
// stores of the current one.  Within an item warp = one output channel (a correlation group or a concat channel), lane = four
// consecutive columns (a 16-byte quad), so every store instruction of a warp is one contiguous 512-byte row segment.
//
// gwc unit: the right-image rows of the unit's GU*K feature channels are staged in shared memory by ONE TMA tile load
// (box 192 x 1 x GU*K, start column w0 - d0 - 64; the hardware zero-fills the negative / out-of-range columns, which is
// exactly the reference's "columns w<d stay zero").  Each lane keeps a 4(d-quads) x 4(d) x 4(w) accumulator block in
// registers: per feature channel it reads its left quad straight from global (no reuse across lanes -> no smem) and
// five right quads from shared memory (a 20-float sliding window) and issues 64 FMAs.
// concat unit: pure shifted copy; right rows are staged per warp in the same shared buffer.
//
// Roofline: HBM-bound.  Algorithmic bytes = 4*(2*B*C*H*W + B*Cout*D*H*W)  (BASELINE.md section 3).
#include <cstdlib>

#include "common.cuh"

namespace osb {

constexpr int kTileW = 128;   // columns per CTA
constexpr int kChunkD = 64;   // disparities per CTA
constexpr int kRowW = kTileW + kChunkD;  // staged right-row width (192 floats)
constexpr int kJG = 4;        // d-quads held in registers per pass (16 disparities)

struct VolParams {
  const float* ref_g;
  const float* tgt_g;
  const float* ref_c;
  const float* tgt_c;
  float* out;
  int B, Cg, Cc, H, W, D, G, K;
  int Ctot, oc_cat;
  int GU, n_gwc_units, n_cat_units, w_tiles, d_chunks;
  int mask_left, use_tma, vec_ok;
  int order;           // work-item order: 0 = unit fastest, 1 = image row fastest (adjacent CTAs write adjacent 512-byte rows)
  float inv_k;
};

__device__ __forceinline__ float4 load_quad(const float* row, int w, int W, bool vec) {
  // row points at column 0 of a feature row; returns columns w..w+3 (zero beyond W).
  if (vec && w + 3 < W) return __ldg(reinterpret_cast<const float4*>(row + w));
  float4 v;
  v.x = (w + 0 < W) ? __ldg(row + w + 0) : 0.f;
  v.y = (w + 1 < W) ? __ldg(row + w + 1) : 0.f;
  v.z = (w + 2 < W) ? __ldg(row + w + 2) : 0.f;
  v.w = (w + 3 < W) ? __ldg(row + w + 3) : 0.f;
  return v;
}

__device__ __forceinline__ void store_quad(float* row, int w, int W, bool vec, float4 v) {
  if (vec && w + 3 < W) {
    st_cs_f4(row + w, v);
  } else {
    if (w + 0 < W) __stcs(row + w + 0, v.x);
    if (w + 1 < W) __stcs(row + w + 1, v.y);
    if (w + 2 < W) __stcs(row + w + 2, v.z);
    if (w + 3 < W) __stcs(row + w + 3, v.w);
  }
}

struct Item {
  int unit, h, b, w0, d0;
};
__device__ __forceinline__ Item decode_item(const VolParams& p, int it) {
  Item i;
  const int units = p.n_gwc_units + p.n_cat_units;
  if (p.order == 1) {                               // rows fastest: CTAs resident together fill neighbouring rows of one (c, d) plane
    i.h = it % p.H;
    it /= p.H;
    i.unit = it % units;
    it /= units;
  } else {
    i.unit = it % units;
    it /= units;
    i.h = it % p.H;
    it /= p.H;
  }
  i.d0 = (it % p.d_chunks) * kChunkD;
  it /= p.d_chunks;
  i.w0 = (it % p.w_tiles) * kTileW;
  i.b = it / p.w_tiles;
  return i;
}

// Persistent kernel: gridDim.x = resident CTAs (2 per SM); each CTA walks the item list with a 2-stage shared-memory
// ring.  While the warps compute item i out of buffer s, the TMA engine is already filling buffer s^1 for item i+grid.
template <bool VEC, bool K4>
__global__ void __launch_bounds__(256, 2) volume_kernel(const __grid_constant__ CUtensorMap tgt_map, const VolParams p,
                                                        const int total_items) {
  extern __shared__ __align__(128) float smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rows = p.n_gwc_units > 0 ? p.GU * p.K : p.GU;          // staged channel rows per buffer
  const size_t buf_floats = (size_t)rows * kRowW;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 2 * buf_floats);
  const size_t HW = (size_t)p.H * p.W;
  constexpr bool vec = VEC;
  const uint32_t tx_bytes = (uint32_t)rows * kRowW * 4u;

  if (p.use_tma && threadIdx.x == 0) {
    tma_prefetch_desc(&tgt_map);
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
    fence_mbar_init();
  }
  __syncthreads();

  auto issue_tma = [&](int it, int stage) {                         // thread 0 only
    const Item n = decode_item(p, it);
    if (n.unit < p.n_gwc_units) {
      fence_proxy_async();                                          // generic-proxy accesses of this buffer are done
      mbar_arrive_expect_tx(&bars[stage], tx_bytes);
      tma_load_3d(smem + stage * buf_floats, &tgt_map, &bars[stage], n.w0 - n.d0 - kChunkD, n.h,
                  n.b * p.Cg + n.unit * p.GU * p.K);
    }
  };

  int stage = 0;
  uint32_t phase0 = 0, phase1 = 0;
  if (p.use_tma && threadIdx.x == 0 && (int)blockIdx.x < total_items) issue_tma(blockIdx.x, 0);

  for (int it = blockIdx.x; it < total_items; it += gridDim.x, stage ^= 1) {
    const Item cur = decode_item(p, it);
    const int nxt = it + gridDim.x;
    if (p.use_tma && threadIdx.x == 0 && nxt < total_items) issue_tma(nxt, stage ^ 1);
    float* buf = smem + stage * buf_floats;
    const int h = cur.h, b = cur.b, w0 = cur.w0, d0 = cur.d0;
    const int wq = w0 + 4 * lane;                                   // first column of this lane's quad
    const int nd = min(kChunkD, p.D - d0);
    const int nquads = (nd + 3) >> 2;
    const int col0 = w0 - d0 - kChunkD;                             // global column of staged column 0

    if (cur.unit < p.n_gwc_units) {
      // ---------------------------------------------------------------- group-wise correlation unit
      const int g0 = cur.unit * p.GU;
      if (p.use_tma) {
        if (stage == 0) {
          mbar_wait(&bars[0], phase0);
          phase0 ^= 1;
        } else {
          mbar_wait(&bars[1], phase1);
          phase1 ^= 1;
        }
      } else {
        const int live = min(rows, p.Cg - g0 * p.K);
        for (int idx = threadIdx.x; idx < live * kRowW; idx += blockDim.x) {
          const int r = idx / kRowW, c = idx - r * kRowW;
          const int gw = col0 + c;
          float v = 0.f;
          if (gw >= 0 && gw < p.W) v = __ldg(p.tgt_g + ((size_t)(b * p.Cg + g0 * p.K + r) * p.H + h) * p.W + gw);
          buf[idx] = v;
        }
        __syncthreads();
      }
      const int g = g0 + warp;
      if (g < p.G && wq < p.W) {
        const float* lrow = p.ref_g + ((size_t)(b * p.Cg + g * p.K) * p.H + h) * p.W;
        const float* rbase = buf + (size_t)warp * p.K * kRowW;
        float* obase = p.out + (((size_t)(b * p.Ctot + g) * p.D) * p.H + h) * p.W;   // + d*HW
        for (int j0 = 0; j0 < nquads; j0 += kJG) {
          float acc[kJG][4][4];
#pragma unroll
          for (int jj = 0; jj < kJG; ++jj)
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
              for (int a = 0; a < 4; ++a) acc[jj][i][a] = 0.f;
          const int win = kChunkD + 4 * (lane - j0) - 16;           // first float of the 20-float window, in [0, 172]
          for (int k0 = 0; k0 < p.K; k0 += 4) {
            float4 lq[4];                                           // four independent global loads in flight
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
              lq[kk] = (K4 || k0 + kk < p.K) ? load_quad(lrow + (size_t)(k0 + kk) * HW, wq, p.W, vec) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
              if (K4 || k0 + kk < p.K) {
                // the 1/K of the mean is folded into the left operand (4 multiplies per channel instead of 64 per pass)
                const float l[4] = {lq[kk].x * p.inv_k, lq[kk].y * p.inv_k, lq[kk].z * p.inv_k, lq[kk].w * p.inv_k};
                float r[20];
                const float4* rp = reinterpret_cast<const float4*>(rbase + (size_t)(k0 + kk) * kRowW + win);
#pragma unroll
                for (int n = 0; n < 5; ++n) {
                  const float4 t = rp[n];
                  r[4 * n + 0] = t.x, r[4 * n + 1] = t.y, r[4 * n + 2] = t.z, r[4 * n + 3] = t.w;
                }
#pragma unroll
                for (int jj = 0; jj < kJG; ++jj)
#pragma unroll
                  for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int a = 0; a < 4; ++a) acc[jj][i][a] = fmaf(l[a], r[16 - 4 * jj + a - i], acc[jj][i][a]);
              }
            }
          }
#pragma unroll
          for (int jj = 0; jj < kJG; ++jj) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int d = d0 + 4 * (j0 + jj) + i;
              if (4 * (j0 + jj) + i < nd) {
                float4 v;
                v.x = (wq + 0 >= d) ? acc[jj][i][0] : 0.f;
                v.y = (wq + 1 >= d) ? acc[jj][i][1] : 0.f;
                v.z = (wq + 2 >= d) ? acc[jj][i][2] : 0.f;
                v.w = (wq + 3 >= d) ? acc[jj][i][3] : 0.f;
                store_quad(obase + (size_t)d * HW, wq, p.W, vec, v);
              }
            }
          }
        }
      }
    } else {
      // ---------------------------------------------------------------- concatenation unit (shifted copy)
      const int oc = (cur.unit - p.n_gwc_units) * p.GU + warp;
      if (oc < 2 * p.Cc) {
        const bool left = oc < p.Cc;
        float* obase = p.out + (((size_t)(b * p.Ctot + p.oc_cat + oc) * p.D) * p.H + h) * p.W;
        if (left) {
          if (wq < p.W) {
            const float4 v = load_quad(p.ref_c + ((size_t)(b * p.Cc + oc) * p.H + h) * p.W, wq, p.W, vec);
            for (int dd = 0; dd < nd; ++dd) {
              const int d = d0 + dd;
              float4 o = v;
              if (p.mask_left) {
                o.x = (wq + 0 >= d) ? v.x : 0.f;
                o.y = (wq + 1 >= d) ? v.y : 0.f;
                o.z = (wq + 2 >= d) ? v.z : 0.f;
                o.w = (wq + 3 >= d) ? v.w : 0.f;
              }
              store_quad(obase + (size_t)d * HW, wq, p.W, vec, o);
            }
          }
        } else {
          float* row = buf + (size_t)warp * kRowW;
          const float* src = p.tgt_c + ((size_t)(b * p.Cc + (oc - p.Cc)) * p.H + h) * p.W;
          for (int c = lane; c < kRowW; c += 32) {
            const int gw = col0 + c;
            row[c] = (gw >= 0 && gw < p.W) ? __ldg(src + gw) : 0.f;
          }
          __syncwarp();
          if (wq < p.W) {
            for (int j = 0; j < nquads; ++j) {
              const float4 lo = *reinterpret_cast<const float4*>(row + kChunkD + 4 * (lane - j) - 4);
              const float4 hi = *reinterpret_cast<const float4*>(row + kChunkD + 4 * (lane - j));
              const float wv[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const int d = d0 + 4 * j + i;
                if (4 * j + i < nd) {
                  float4 o;                                         // columns w<d read the zero-filled halo
                  o.x = wv[4 - i], o.y = wv[5 - i], o.z = wv[6 - i], o.w = wv[7 - i];
                  store_quad(obase + (size_t)d * HW, wq, p.W, vec, o);
                }
              }
            }
          }
        }
      }
    }
    __syncthreads();                                                // buffer `stage` may be refilled from now on
  }
}

static thread_local const char* g_volume_variant = "";   // osb_volume_last_variant

static int launch_volume(const float* ref_g, const float* tgt_g, const float* ref_c, const float* tgt_c, float* out,
                         int B, int Cg, int Cc, int H, int W, int D, int G, int mask_left, cudaStream_t stream, int reduce_sum = 0) {
  OSB_REQUIRE(B > 0 && H > 0 && W > 0 && D > 0, "volume: empty shape B=%d H=%d W=%d D=%d", B, H, W, D);
  OSB_REQUIRE(Cg >= 0 && Cc >= 0 && (Cg > 0 || Cc > 0), "volume: no channels");
  int K = 0;
  if (Cg > 0) {
    OSB_REQUIRE(G > 0 && Cg % G == 0, "groupwise_correlation: C=%d not divisible by num_groups=%d", Cg, G);
    K = Cg / G;
    OSB_REQUIRE(K <= 144, "volume: %d channels per group exceeds the 144 supported (two-stage 192-float rows in 227 KB)", K);
  } else {
    G = 0;
  }
  VolParams p{};
  p.ref_g = ref_g, p.tgt_g = tgt_g, p.ref_c = ref_c, p.tgt_c = tgt_c, p.out = out;
  p.B = B, p.Cg = Cg, p.Cc = Cc, p.H = H, p.W = W, p.D = D, p.G = G, p.K = K;
  p.Ctot = G + 2 * Cc, p.oc_cat = G;
  int GU = 8;
  if (Cg > 0) {
    GU = G < 8 ? G : 8;
    while (GU > 1 && GU * K > 128) GU >>= 1;
  }
  p.GU = GU;
  p.n_gwc_units = Cg > 0 ? (G + GU - 1) / GU : 0;
  p.n_cat_units = Cc > 0 ? (2 * Cc + GU - 1) / GU : 0;
  p.w_tiles = (W + kTileW - 1) / kTileW;
  p.d_chunks = (D + kChunkD - 1) / kChunkD;
  p.mask_left = mask_left;
  {
    static const int order = [] {                   // OSB_VOLUME_ORDER=0 restores the round-1 item order (A/B in tools/kbench.py)
      const char* e = getenv("OSB_VOLUME_ORDER");
      return e ? atoi(e) : 1;
    }();
    p.order = order;
  }
  p.inv_k = K > 0 ? (reduce_sum ? 1.0f : 1.0f / (float)K) : 0.f;   // reduce_sum: plain sum over the group's channels (CoEx, L2-normalised gwc)
  auto aligned16 = [](const void* q) { return q == nullptr || (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  p.vec_ok = (W % 4 == 0) && aligned16(ref_g) && aligned16(ref_c) && aligned16(out);
  const int rows = Cg > 0 ? GU * K : GU;
  size_t smem = 2 * (size_t)rows * kRowW * sizeof(float) + 16;    // two-stage ring + two mbarriers
  CUtensorMap map{};
  p.use_tma = 0;
  if (Cg > 0 && W % 4 == 0 && aligned16(tgt_g) && rows <= 256) {
    // tensor (B*Cg, H, W) fp32; box = 192 columns x 1 row x GU*K channels
    if (make_tensor_map_3d(&map, tgt_g, (uint64_t)W, (uint64_t)H, (uint64_t)B * Cg, (uint64_t)W * 4, (uint64_t)H * W * 4,
                           kRowW, 1, (uint32_t)rows))
      p.use_tma = 1;
  }
  using KernelFn = void (*)(const CUtensorMap, const VolParams, const int);
  const bool k4 = (K % 4 == 0);                                   // K = 0 (concat only) counts as a multiple
  const int variant = (p.vec_ok ? 2 : 0) | (k4 ? 1 : 0);
  static const KernelFn kernels[4] = {volume_kernel<false, false>, volume_kernel<false, true>, volume_kernel<true, false>,
                                      volume_kernel<true, true>};
  KernelFn kernel = kernels[variant];
  static size_t configured_all[64][4] = {};                       // per device: cudaFuncSetAttribute is per device
  size_t* configured = configured_all[device_index() & 63];
  if (smem > configured[variant]) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
      set_error("volume: cannot reserve %zu bytes of shared memory: %s", smem, cudaGetErrorString(e));
      return OSB_ECUDA;
    }
    configured[variant] = smem;
  }
  const long long total = (long long)(p.n_gwc_units + p.n_cat_units) * H * B * p.w_tiles * p.d_chunks;
  OSB_REQUIRE(total < (1ll << 31), "volume: too many work items (%lld)", total);
  static const char* const names[8] = {"volume<0,0,ldg>", "volume<0,0,tma>", "volume<0,1,ldg>", "volume<0,1,tma>",
                                       "volume<1,0,ldg>", "volume<1,0,tma>", "volume<1,1,ldg>", "volume<1,1,tma>"};
  g_volume_variant = names[2 * variant + p.use_tma];
  int per_sm = 0;
  cudaError_t oe = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, 32 * GU, smem);
  if (oe != cudaSuccess || per_sm < 1) {
    set_error("volume: occupancy query failed (%s), smem=%zu", cudaGetErrorString(oe), smem);
    (void)cudaGetLastError();
    return OSB_ECUDA;
  }
  long long grid = (long long)sm_count() * per_sm;                // persistent: every CTA resident, multiple of the SM count
  if (grid > total) grid = total;
  grid = cap_persistent_grid(grid);
  kernel<<<(unsigned)grid, 32 * GU, smem, stream>>>(map, p, (int)total);
  count_launch();
  return check_launch("volume_kernel");
}

}  // namespace osb

extern "C" {

const char* osb_volume_last_variant(void) { return osb::g_volume_variant; }

int osb_gwc_volume_fwd(const float* ref, const float* tgt, float* out, int B, int C, int H, int W, int D, int G,
                       osb_stream_t stream) {
  OSB_REQUIRE(ref && tgt && out, "gwc_volume: null pointer");
  OSB_REQUIRE(C > 0, "gwc_volume: C=%d", C);
  return osb::launch_volume(ref, tgt, nullptr, nullptr, out, B, C, 0, H, W, D, G, 1, (cudaStream_t)stream);
}

int osb_gwc_volume_sum_fwd(const float* ref, const float* tgt, float* out, int B, int C, int H, int W, int D, int G,
                           osb_stream_t stream) {
  OSB_REQUIRE(ref && tgt && out, "gwc_volume_sum: null pointer");
  OSB_REQUIRE(C > 0, "gwc_volume_sum: C=%d", C);
  return osb::launch_volume(ref, tgt, nullptr, nullptr, out, B, C, 0, H, W, D, G, 1, (cudaStream_t)stream, 1);
}

int osb_concat_volume_fwd(const float* ref, const float* tgt, float* out, int B, int C, int H, int W, int D,
                          int mask_left, osb_stream_t stream) {
  OSB_REQUIRE(ref && tgt && out, "concat_volume: null pointer");
  OSB_REQUIRE(C > 0, "concat_volume: C=%d", C);
  return osb::launch_volume(nullptr, nullptr, ref, tgt, out, B, 0, C, H, W, D, 0, mask_left, (cudaStream_t)stream);
}

int osb_gwc_concat_volume_fwd(const float* ref_gwc, const float* tgt_gwc, const float* ref_cat, const float* tgt_cat,
                              float* out, int B, int Cg, int Cc, int H, int W, int D, int G, osb_stream_t stream) {
  OSB_REQUIRE(ref_gwc && tgt_gwc && ref_cat && tgt_cat && out, "gwc_concat_volume: null pointer");
  OSB_REQUIRE(Cg > 0 && Cc > 0, "gwc_concat_volume: Cg=%d Cc=%d", Cg, Cc);
  return osb::launch_volume(ref_gwc, tgt_gwc, ref_cat, tgt_cat, out, B, Cg, Cc, H, W, D, G, 1, (cudaStream_t)stream);
}

int osb_corr_volume_fwd(const float* left, const float* right, float* out, int B, int C, int H, int W, int D,
                        osb_stream_t stream) {
  OSB_REQUIRE(left && right && out, "corr_volume: null pointer");
  OSB_REQUIRE(C > 0, "corr_volume: C=%d", C);
  // correlation_volume == build_gwc_volume(..., num_groups=1).squeeze(1)  (SURVEY.md section 4.3)
  return osb::launch_volume(left, right, nullptr, nullptr, out, B, C, 0, H, W, D, 1, 1, (cudaStream_t)stream);
}
}
