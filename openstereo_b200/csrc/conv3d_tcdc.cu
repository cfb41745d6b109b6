// Tensor-core (Hopper wgmma) ConvTranspose3d k=3, stride 2, padding 1, output_padding 1: the up-sampling convs of the hourglasses
//   conv5 128->64 / 64->64 (1/16 -> 1/8 res) and conv6 64->32 (1/8 -> 1/4 res): gwcnet/hourglass.py:35-41,
//   psmnet/psmnet_cost_processor.py:99-106 (deconv3d_bn).
// Per dimension an output index o gathers  o even (=2m): tap k=1 from input m;  o odd (=2m+1): k=0 from m+1 and k=2 from m.
// Same machinery as conv3d_tcg.cu / conv3d_tcs2.cu (3xFP16 split, LDG-staged swizzled operands, warp-specialised persistent CTA,
// one accumulator tile of G = 32 output channels per consumer warpgroup).  A work item is plane od, R = 128/Win consecutive input
// rows j, all 2*Win output columns, and BOTH output row parities: consumer warpgroup t accumulates output rows oh = 2j + t.  For
// each valid tap pair (kd, kh) the operand tile is the R input rows j + (t + 1 - kh) / 2 of input plane id, un-shifted in w, and
// one MMA with the kw slices stacked along N gives
//   E[m] = A[m].W1 -> output column 2m,      P2[m] = A[m].W2 and P0[m] = A[m].W0 -> output column 2m+1 = P2[m] + P0[m+1];
// the epilogue does that single right shift (zero at m = Win-1: the column beyond the input) and writes both columns.
// A (kd, chunk) phase stages the units of input row offsets +1, 0 (k4: and -1) once, in that order, and both warpgroups read
// them: parity 1 meets offset +1 through kh = 0 and offset 0 through kh = 2, parity 0 offset 0 through kh = 1 -- 2 stagings for
// 3 MMA chains.  Each tile gets the same MMA sequence (kh ascending) as a one-parity item would, hence the same kappa * n.
// Both parities share od, so items of one od have the same kd taps (1 or 2, alternating with od parity, the fastest index).
// GENERAL WIDTHS (GW = true, W = 128 instantiations; see conv3d_tcg.cu): an M tile is a 128-column segment of one INPUT row of
// runtime width Wr starting at input column ct * 127; tile column 127 is the halo that provides P0[m+1] (zero beyond the image) and
// its two output columns are not stored.
// KS = 4: ConvTranspose3d(k=4, s=2, p=1) of StereoBase's hourglass (stereobase/hourglass.py:35-60 conv*_up): per dimension
//   o = 2m: taps k=1 (input m) and k=3 (input m-1);   o = 2m+1: taps k=2 (input m) and k=0 (input m+1)
// -- every tile has 2 x 2 (kd, kh) tap pairs, a phase stages 3 units for 4 chains, the four kw slices are stacked along N as
// [W1 | W3 | W2 | W0] and the epilogue forms  even[m] = P1[m] + P3[m-1],  odd[m] = P2[m] + P0[m+1]  (one left and one right shift).
//
// Warp roles (512 threads, 1 CTA/SM, persistent; setmaxnreg moves the registers, tc_common.cuh): warps 0-7 = two consumer
// warpgroups (output row parity 0 and 1), warps 8-11 = A-unit loaders, warp 12 = weight-slice producer, warps 13-15 idle.
#include "tc_common.cuh"

namespace osb {

struct TcdcParams {
  const float* x;          // (B, D, H, W, Cin) channels-last
  const void* w;           // fp16 [3 kd][Cin/KC][3 kh][3*Cout][KC hi | KC lo]  (ops.pack_tc_weight)
  const float* scale;
  const float* shift;
  const float* residual;
  float* y;
  int B, D, H, Cin;        // INPUT extent D x H x W; output is 2D x 2H x 2W
  int act;
  float kappa;       // expected round-towards-zero loss per accumulating MMA (tc_common.cuh)
  unsigned int* overflow;  // sticky fp16-range flag (tc_common.cuh)
  int out_ndhwc, res_ndhwc;
  int items, hblocks;
  int Wr, ctiles;          // general-width instantiations: INPUT width and column tiles per row (whole-row kernels: W, 1)
  int ystride;             // channels per voxel of the channels-last y / residual (0 = COUT); > COUT: this launch writes a channel slice
  int cout_real;           // channels of an NCDHW output / residual (<= COUT: zero-padded channel plans write only the real ones)
};

template <int COUT, int KC, int W, int TILES, bool GW = false, int KS_ = 3>     // W = INPUT width, KS_ = kernel size (3 or 4)
struct TcdcCfg {
  static_assert(!GW || W == 128, "general-width tiles are 128-column segments of one input row");
  static_assert(KS_ == 3 || (KS_ == 4 && !GW), "kernel size 3 (any width) or 4 (whole-row tiles)");
  static constexpr int KS = KS_;
  static constexpr int HALO = GW ? 1 : 0;                   // halo columns on the RIGHT of a column tile
  static constexpr int CSTEP = 128 - HALO;                  // input columns a column tile produces outputs for
  static constexpr int R = 128 / W;                         // input rows (= output rows of one parity) per M tile
  static constexpr int ROWB = KC * 4;                       // bytes per K-major operand row: [KC fp16 hi | KC fp16 lo]
  static constexpr int UNIT_BYTES = 128 * ROWB;
  static constexpr int N3 = KS_ * COUT;                     // kw slices stacked along N
  static constexpr int G = 32;                              // output channels per work item
  static constexpr int NG = COUT / G;                       // channel groups
  static constexpr int NGK = KS_ * G;                       // wgmma N: the KS kw blocks of one channel group
  static constexpr int B_SLICE = N3 * ROWB;                 // one kh weight slice in global memory (hi and lo halves of every row)
  static constexpr int B_SUB = NGK * ROWB;                  // the part of it one item reads
  // Staged accumulator tile per warpgroup: k3 stages all three kw blocks at once; k4's four do not fit next to its 2 x 4 weight
  // slices, so it stages two blocks per pass, [P3 | P0] (the shifted ones) and then [P1 | P2].
  static constexpr int SCOLS = KS_ == 3 ? NGK : 2 * G;
  static constexpr int LD = SCOLS + 4;                      // floats per row of a staged accumulator tile
  static constexpr int NU = KS_ - 1;                        // units per (kd, chunk) phase: input row offsets +1, 0 (k4: and -1)
  // A-unit ring.  NLW loader warps (8-11) fill the units round-robin (unit u belongs to loader u mod NLW) into a ring as deep as
  // shared memory allows (at most 10 units).  Each loader warp enumerates ONLY ITS OWN units: a walk over the whole (tile, tap)
  // sequence by every warp, picking every NLW-th unit, makes that scalar control flow the bound of these kernels.
  static constexpr int NLW = 4;
  static constexpr int XCHG_FLOATS = 2 * 4 * 2 * 32;        // per consumer warpgroup: [2][4 quadrants][2 sides][32]
  static constexpr int FIXED_SMEM = 1024 + TC_BSLOTS * KS_ * B_SUB + TC_WGS * 128 * LD * 4 + 1024 + TC_WGS * XCHG_FLOATS * 4 + 3 * COUT * 4;
  static constexpr int STAGES = (232448 - FIXED_SMEM) / UNIT_BYTES < 10 ? (232448 - FIXED_SMEM) / UNIT_BYTES : 10;
  static_assert(STAGES >= NLW, "the ring must hold at least one unit per loader warp");
  static constexpr int HBLK = TILES * R;                    // input rows per work item
  static constexpr int KSTEPS = KC / 16;                    // K = 16 fp16 channels per MMA
  static constexpr int A_OFF = 0;
  static constexpr int B_OFF = A_OFF + STAGES * UNIT_BYTES;
  static constexpr int STAGE_OFF = B_OFF + TC_BSLOTS * KS_ * B_SUB;   // [TC_WGS][128][LD] fp32 accumulator tiles
  static constexpr int BAR_OFF = STAGE_OFF + TC_WGS * 128 * LD * 4;
  static constexpr int THREADS = TC_WG_THREADS;             // consumers 0-7 | A loaders 8-11 | weight producer 12, idle 13-15
  static constexpr size_t SMEM = 1024 + (size_t)BAR_OFF + 1024 + TC_WGS * XCHG_FLOATS * 4 + 3 * COUT * 4;
  static_assert(SMEM <= 232448, "shared memory budget of one CTA exceeded");
  static_assert(TILES == 1, "a consumer warpgroup holds one accumulator tile");
  static_assert(COUT % G == 0, "output channels come in groups of 32");
  static_assert(32 * LD >= TP_WARP_FLOATS, "store_ndhwc_chunk32 transposes through the warp's own rows of the staging tile");
  static_assert(B_SUB % 1024 == 0 && UNIT_BYTES % 1024 == 0, "operand tiles must stay 1024-byte aligned");
  // weight slice through which the tile of row parity t reads unit u (input row offset 1 - u), or -1: output row 2j + t gathers
  // tap kh from input row j + (t + 1 - kh) / 2
  static constexpr int kh_of(int u, int t) { return (t - 1 + 2 * u >= 0 && t - 1 + 2 * u < KS_) ? t - 1 + 2 * u : -1; }
};

// work item = (image b, output plane od, block of TILES*R input rows, column tile); the column tile and then od vary fastest, so
// that the 1-tap (even od) and 2-tap (odd od) items are interleaved over the persistent CTAs
struct ItemDc {
  int b, od, j0, ct, nkd;
};
// output index o gathers tap k from input (o + 1 - k) / 2 when that is an integer inside [0, n)
__device__ __forceinline__ bool kd_valid(int od, int kd, int D) {
  const int num = od + 1 - kd;
  return !(num & 1) && num >= 0 && (num >> 1) < D;
}
// rows outside the image are staged as zeros rather than skipped, so only the parity decides
__device__ __forceinline__ bool kh_valid(int ph, int kh) { return ((ph + 1 - kh) & 1) == 0; }
template <class C>
__device__ __forceinline__ ItemDc decode_dc(const TcdcParams& p, int it) {
  ItemDc w;
  w.ct = 0;
  if (C::HALO) {                                    // general widths: the column tile varies fastest
    w.ct = it % p.ctiles;
    it /= p.ctiles;
  }
  const int Do = 2 * p.D;
  w.od = it % Do;
  it /= Do;
  w.j0 = (it % p.hblocks) * C::HBLK;
  w.b = it / p.hblocks;
  w.nkd = 0;
#pragma unroll
  for (int k = 0; k < C::KS; ++k) w.nkd += kd_valid(w.od, k, p.D) ? 1 : 0;   // input planes feeding plane od
  return w;
}

// Accumulator column blocks GA and GB (G = 32 columns each) of a finished 128 x N tile into staged columns [0, 32) and [32, 64),
// or (ADD) added to the values staged there.  Fragment layout as in wg_stage (tc_common.cuh): register 4j + r holds column
// 8j + 2(l%4) + r%2.
template <int N, int GA, int GB, bool ADD>
__device__ __forceinline__ void dc_stage_pair(float* stage, int ld, const float (&acc)[2][N / 2], int wq, int lane) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float* r0 = stage + (64 * h + 16 * wq + (lane >> 2)) * ld + 2 * (lane & 3);
#pragma unroll
    for (int g = 0; g < 2; ++g)
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = (g ? GB : GA) * 4 + jj;
#pragma unroll
        for (int r = 0; r < 2; ++r) {               // rows lane/4 and lane/4 + 8 of the fragment
          float2* d = reinterpret_cast<float2*>(r0 + 8 * r * ld + 32 * g + 8 * jj);
          float2 v = make_float2(acc[h][4 * j + 2 * r], acc[h][4 * j + 2 * r + 1]);
          if (ADD) {
            const float2 s = *d;
            v = make_float2(s.x + v.x, s.y + v.y);
          }
          *d = v;
        }
      }
  }
}

template <int COUT, int KC, int W, int TILES, bool GW = false, int KS = 3>
__global__ void __launch_bounds__(TcdcCfg<COUT, KC, W, TILES, GW, KS>::THREADS, 1) conv3d_tcdc_kernel(const TcdcParams p) {
  using C = TcdcCfg<COUT, KC, W, TILES, GW, KS>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte aligned; offsetting smem_raw itself keeps every derived pointer in the shared window (LDS/STS, see conv3d_tc.cu)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* a_buf = smem + C::A_OFF;
  uint8_t* b_buf = smem + C::B_OFF;
  float* stage = reinterpret_cast<float*>(smem + C::STAGE_OFF);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::BAR_OFF);
  uint64_t* a_ready = bars;                         // [STAGES] loaders -> consumers  (32 arrivals: one warp)
  uint64_t* a_empty = a_ready + C::STAGES;          // [STAGES] consumers -> loaders  (8 arrivals: one per consumer warp)
  uint64_t* b_full = a_empty + C::STAGES;           // [2][KS]  weight producer -> consumers (expect_tx + bulk-copy bytes)
  uint64_t* b_empty = b_full + TC_BSLOTS * KS;      // [2][KS]  consumers -> weight producer (8 arrivals)
  float* xchg = reinterpret_cast<float*>(smem + C::BAR_OFF + 1024);   // [TC_WGS][XCHG_FLOATS]
  float* s_scale = xchg + TC_WGS * C::XCHG_FLOATS;
  float* s_shift = s_scale + COUT;
  float* zeros = s_shift + COUT;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nchunk = p.Cin / KC;
  const int Wp = GW ? p.Wr : W;                     // INPUT width (the output is 2 * Wp wide)
  const int YS = (W < 32 && p.ystride) ? p.ystride : COUT;   // (compile-time COUT in the wide instantiations: slices exist at W' = 16 only)      // channel stride of the channels-last output / residual

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(&a_ready[s], 32);                     // one loader warp fills a unit
      mbar_init(&a_empty[s], 4 * TC_WGS);
    }
    for (int k = 0; k < TC_BSLOTS * KS; ++k) {
      mbar_init(&b_full[k], 1);
      mbar_init(&b_empty[k], 4 * TC_WGS);
    }
    fence_mbar_init();
  }
  for (int c = threadIdx.x; c < COUT; c += blockDim.x) {
    s_scale[c] = p.scale ? p.scale[c] : 1.f;
    s_shift[c] = p.shift ? p.shift[c] : 0.f;
    zeros[c] = 0.f;
  }
  __syncthreads();

  // ---------------------------------------------------------------------------------------------- consumer warpgroups
  // Warpgroup wg issues the wgmmas of output row parity wg into its 128 x KS*G register tile (output channels cg .. cg + 31 of every
  // kw tap) from the units and weight slices both warpgroups read, then runs the epilogue of that tile.
  if (warp < 4 * TC_WGS) {
    setmaxnreg_inc<TC_CONSUMER_REGS>();
    const int wg = warp >> 2;                        // output row parity of this warpgroup's tile
    stage += wg * 128 * C::LD;
    xchg += wg * C::XCHG_FLOATS;
    const int bar_stage = 1 + 2 * wg, bar_xchg = 2 + 2 * wg;   // this warpgroup's named barriers
    const uint64_t dbase = (KC == 32) ? desc_sw128_base() : desc_sw64_base();
    constexpr uint32_t A_HALF = 64 * C::ROWB / 16;  // descriptor offset of operand rows 64..127
    const uint32_t b16 = (smem_u32(b_buf) & 0x3FFFF) >> 4;
    const int q = warp & 3;                          // epilogue: this warp owns tile rows 32q .. 32q + 31
    const int m = q * 32 + lane;                     // operand row owned by this thread
    const int rr = m / W, wcol = m % W;              // input row inside the tile, input column
    const bool has_right_q = (((q + 1) * 32) % W) != 0;   // the next quadrant continues the same image row
    const bool has_left_q = ((q * 32) % W) != 0;          // (k4 only) the previous quadrant does
    const int Do = 2 * p.D, Ho = 2 * p.H;
    const int Wo = 2 * Wp;
    uint32_t unitc = 0, phc = 0, exc = 0;
    for (int it = blockIdx.x; it < p.items; it += gridDim.x) {
      const int cg = (it % C::NG) * C::G;            // output channel group of this item
      const ItemDc w = decode_dc<C>(p, it / C::NG);
      float ev[32], od_[32];
      float acc[2][C::NGK / 2];
      uint32_t accum = 0;
      for (int kd = 0; kd < KS; ++kd) {
        if (!kd_valid(w.od, kd, p.D)) continue;
        for (int ch = 0; ch < nchunk; ++ch, ++phc) {
          const uint32_t bset = (phc & 1) * KS, bpar = (phc >> 1) & 1;   // weight buffers alternate between phases
          // The slices of the other row parity: wait for their fill and release them.  Every warpgroup waits for and releases each
          // slice and unit of a phase, so neither can arrive on a later phase of a buffer than the one being filled.
#pragma unroll
          for (int kh = 0; kh < KS; ++kh) {
            if (kh_valid(wg, kh)) continue;
            mbar_wait(&b_full[bset + kh], bpar);
            wg_release(&b_empty[bset + kh], lane);
          }
#pragma unroll
          for (int u = 0; u < C::NU; ++u) {
            const uint32_t slot = unitc % C::STAGES, par = (unitc / C::STAGES) & 1;
            mbar_wait(&a_ready[slot], par);
            const int kh = C::kh_of(u, wg);
            if (kh >= 0) {                         // warpgroup-uniform
              mbar_wait(&b_full[bset + kh], bpar);
              const uint64_t da0 = dbase | (uint64_t)((smem_u32(a_buf + slot * C::UNIT_BYTES) & 0x3FFFF) >> 4);
              const uint64_t db0 = dbase | (uint64_t)(b16 + ((bset + kh) * C::B_SUB) / 16);
              wg_fence();
#pragma unroll
              for (int ks = 0; ks < C::KSTEPS; ++ks)
                wg_mma_split<C::NGK>(acc, da0 + TcK<KC>::A_KSTEP * ks, A_HALF, TcK<KC>::A_LO, db0 + 2 * ks, TcK<KC>::B_LO, ks > 0 ? 1u : accum);
              wg_commit();
              wg_wait_all();
              accum = 1;
              wg_release(&b_empty[bset + kh], lane);
            }
            wg_release(&a_empty[slot], lane);
            ++unitc;
          }
        }
      }
      const int j = w.j0 + rr;                       // input row of this thread's voxel
      const bool live = j < p.H;
      const int oh = 2 * j + wg;
      // general widths: input column of this thread's tile column; the halo column and columns beyond the image are not stored
      const int col = GW ? w.ct * C::CSTEP + m : wcol;
      const bool cvalid = !GW || (m < C::CSTEP && col < Wp);
      const uint32_t vmask = GW ? __ballot_sync(0xffffffffu, cvalid) : 0xffffffffu;
      const size_t vox = (((size_t)w.b * Do + w.od) * Ho + oh) * Wo + 2 * col;         // NDHWC index of the EVEN output voxel
      if (live && cvalid && p.residual && p.res_ndhwc) {
        // the residual streams from HBM: start pulling this thread's two voxels (2*COUT floats, contiguous) into L2 while
        // the tile is being staged, so the loads after the transpose do not expose the DRAM latency per tile
        const float* rp = p.residual + vox * YS;
#pragma unroll
        for (int k = 0; k < 2 * COUT; k += 32) asm volatile("prefetch.global.L2 [%0];" ::"l"(rp + k));
      }
      // tap pairs of this tile: (1 or 2 kd) x (1 or 2 kh); each adds chunks x k-steps x 3 MMAs (tc_common.cuh: rz_kappa)
      const float corr = 1.f + p.kappa * (float)(w.nkd * (KS == 4 ? 2 : wg + 1) * nchunk * C::KSTEPS * 3);
      float* srow = stage + m * C::LD;             // this voxel's staged accumulator columns
      float* xb = xchg + (exc & 1) * (4 * 2 * 32);
      ++exc;
      named_bar_sync(bar_stage, 128);              // every warp is done with the previous tile's staged rows
      if constexpr (KS == 3) {
        // staged column blocks [E (kw=1) | P2 (kw=2) | P0 (kw=0)]
        wg_stage<C::NGK>(stage, C::LD, acc, q, lane);
        named_bar_sync(bar_stage, 128);
        if (lane == 0) {                           // P0 of this quadrant's first column
#pragma unroll
          for (int i = 0; i < 32; i += 4)
            *reinterpret_cast<float4*>(xb + (q * 2) * 32 + i) = *reinterpret_cast<const float4*>(srow + 2 * C::G + i);
        }
        named_bar_sync(bar_xchg, 128);
        const float* xr = has_right_q ? xb + ((q + 1) * 2) * 32 : zeros;
#pragma unroll
        for (int i0 = 0; i0 < 32; i0 += 4) {        // neighbour values loaded unconditionally, merged with selects (no branches)
          const float4 r4 = *reinterpret_cast<const float4*>(xr + i0);
          const float4 e4 = *reinterpret_cast<const float4*>(srow + i0);
          const float4 p24 = *reinterpret_cast<const float4*>(srow + C::G + i0);
          const float4 p04 = *reinterpret_cast<const float4*>(srow + 2 * C::G + i0);
          const float re[4] = {r4.x, r4.y, r4.z, r4.w};
          const float e[4] = {e4.x, e4.y, e4.z, e4.w}, p2[4] = {p24.x, p24.y, p24.z, p24.w}, p0[4] = {p04.x, p04.y, p04.z, p04.w};
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int i = i0 + k;
            float right = __shfl_down_sync(0xffffffffu, p0[k], 1);   // P0 of input column m+1
            right = (lane == 31) ? re[k] : right;                    // zero beyond the last input column
            if (W < 32) right = (wcol == W - 1) ? 0.f : right;       // row seams inside the warp
            ev[i] = e[k] * corr;
            od_[i] = (p2[k] + right) * corr;
          }
        }
      } else {
        // k4, pass 1: the two shifted blocks [P3 | P0].  Each thread writes its shifted values back over its own staged row (the
        // neighbours' values arrive by shuffle and through xb), so that the outputs are not held in registers next to the P1 and P2
        // accumulators.
        dc_stage_pair<C::NGK, 1, 3, false>(stage, C::LD, acc, q, lane);
        named_bar_sync(bar_stage, 128);
        if (lane == 31) {                          // P3 of this quadrant's last column
#pragma unroll
          for (int i = 0; i < 32; i += 4)
            *reinterpret_cast<float4*>(xb + (q * 2 + 1) * 32 + i) = *reinterpret_cast<const float4*>(srow + i);
        }
        if (lane == 0) {                           // P0 of this quadrant's first column
#pragma unroll
          for (int i = 0; i < 32; i += 4)
            *reinterpret_cast<float4*>(xb + (q * 2) * 32 + i) = *reinterpret_cast<const float4*>(srow + C::G + i);
        }
        named_bar_sync(bar_xchg, 128);
        const float* xl = has_left_q ? xb + ((q - 1) * 2 + 1) * 32 : zeros;
        const float* xr = has_right_q ? xb + ((q + 1) * 2) * 32 : zeros;
#pragma unroll
        for (int i0 = 0; i0 < 32; i0 += 4) {
          const float4 l4 = *reinterpret_cast<const float4*>(xl + i0);
          const float4 r4 = *reinterpret_cast<const float4*>(xr + i0);
          const float4 p34 = *reinterpret_cast<const float4*>(srow + i0);
          const float4 p04 = *reinterpret_cast<const float4*>(srow + C::G + i0);
          const float le[4] = {l4.x, l4.y, l4.z, l4.w}, re[4] = {r4.x, r4.y, r4.z, r4.w};
          const float p3[4] = {p34.x, p34.y, p34.z, p34.w}, p0[4] = {p04.x, p04.y, p04.z, p04.w};
          float e[4], o[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float left = __shfl_up_sync(0xffffffffu, p3[k], 1);      // P3 of input column m-1
            const float right = __shfl_down_sync(0xffffffffu, p0[k], 1);   // P0 of input column m+1
            e[k] = (lane == 0) ? le[k] : left;           // zero before the first input column
            o[k] = (lane == 31) ? re[k] : right;         // zero beyond the last one
            if (W < 32) {                                // row seams inside the warp are image edges
              e[k] = (wcol == 0) ? 0.f : e[k];
              o[k] = (wcol == W - 1) ? 0.f : o[k];
            }
          }
          *reinterpret_cast<float4*>(srow + i0) = make_float4(e[0], e[1], e[2], e[3]);
          *reinterpret_cast<float4*>(srow + C::G + i0) = make_float4(o[0], o[1], o[2], o[3]);
        }
        // pass 2: the aligned blocks [P1 | P2] added in place: the tile then holds  P3[m-1] + P1[m] | P0[m+1] + P2[m]
        named_bar_sync(bar_stage, 128);            // every warp has written its shifted values
        dc_stage_pair<C::NGK, 0, 2, true>(stage, C::LD, acc, q, lane);
        named_bar_sync(bar_stage, 128);
#pragma unroll
        for (int i0 = 0; i0 < 32; i0 += 4) {
          const float4 e4 = *reinterpret_cast<const float4*>(srow + i0);
          const float4 o4 = *reinterpret_cast<const float4*>(srow + C::G + i0);
          const float e[4] = {e4.x, e4.y, e4.z, e4.w}, o[4] = {o4.x, o4.y, o4.z, o4.w};
#pragma unroll
          for (int k = 0; k < 4; ++k) ev[i0 + k] = e[k] * corr, od_[i0 + k] = o[k] * corr;
        }
      }
      const size_t plane = (size_t)Do * Ho * Wo;                                   // NCDHW channel stride
      const size_t ncdhw0 = (size_t)w.b * p.cout_real * plane + ((size_t)w.od * Ho + oh) * Wo + 2 * col;
      // coalesced channels-last path (BN/residual/act inside); W < 32: the warp's two input rows map to output rows that are
      // not adjacent in memory -> per-thread stores below
      if (W >= 32 && live && p.out_ndhwc && (!p.residual || p.res_ndhwc)) {
        // lane k owns output voxels (vox0 + 2k) and (vox0 + 2k + 1): two transposes with a 2-voxel lane stride
        float* y0 = p.y + (vox - 2 * lane) * YS + cg;
        const float* r0 = p.residual ? p.residual + (vox - 2 * lane) * YS + cg : nullptr;
        store_ndhwc_chunk32(stage + q * 32 * C::LD, lane, ev, y0, r0, 2 * YS, s_scale + cg, s_shift + cg, p.act, vmask);
        store_ndhwc_chunk32(stage + q * 32 * C::LD, lane, od_, y0 + YS, r0 ? r0 + YS : nullptr, 2 * YS, s_scale + cg,
                            s_shift + cg, p.act, vmask);
      } else if (live && cvalid) {
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          ev[i] = fmaf(ev[i], s_scale[cg + i], s_shift[cg + i]);
          od_[i] = fmaf(od_[i], s_scale[cg + i], s_shift[cg + i]);
        }
        if (p.residual) {
          if (p.res_ndhwc) {
            const float4* rp = reinterpret_cast<const float4*>(p.residual + vox * YS + cg);
            const float4* rq = reinterpret_cast<const float4*>(p.residual + (vox + 1) * YS + cg);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float4 a = __ldg(rp + i), bq = __ldg(rq + i);
              ev[4 * i] += a.x, ev[4 * i + 1] += a.y, ev[4 * i + 2] += a.z, ev[4 * i + 3] += a.w;
              od_[4 * i] += bq.x, od_[4 * i + 1] += bq.y, od_[4 * i + 2] += bq.z, od_[4 * i + 3] += bq.w;
            }
          } else {
#pragma unroll
            for (int i = 0; i < 32; ++i) {
              if (cg + i >= p.cout_real) continue;
              const float2 rv = __ldg(reinterpret_cast<const float2*>(p.residual + ncdhw0 + (size_t)(cg + i) * plane));
              ev[i] += rv.x, od_[i] += rv.y;
            }
          }
        }
        if (p.act == OSB_ACT_RELU) {
#pragma unroll
          for (int i = 0; i < 32; ++i) ev[i] = fmaxf(ev[i], 0.f), od_[i] = fmaxf(od_[i], 0.f);
        } else if (p.act == OSB_ACT_LEAKY) {
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            ev[i] = ev[i] > 0.f ? ev[i] : 0.01f * ev[i];
            od_[i] = od_[i] > 0.f ? od_[i] : 0.01f * od_[i];
          }
        }
        if (p.out_ndhwc) {
          float4* yp = reinterpret_cast<float4*>(p.y + vox * YS + cg);
          float4* yq = reinterpret_cast<float4*>(p.y + (vox + 1) * YS + cg);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            yp[i] = make_float4(ev[4 * i], ev[4 * i + 1], ev[4 * i + 2], ev[4 * i + 3]);
            yq[i] = make_float4(od_[4 * i], od_[4 * i + 1], od_[4 * i + 2], od_[4 * i + 3]);
          }
        } else {
#pragma unroll
          for (int i = 0; i < 32; ++i)             // columns 2w, 2w+1 of consecutive lanes: 256 contiguous bytes per warp
            if (cg + i < p.cout_real) *reinterpret_cast<float2*>(p.y + ncdhw0 + (size_t)(cg + i) * plane) = make_float2(ev[i], od_[i]);
        }
      }
    }
  }
  // ---------------------------------------------------------------------------------------------- A-unit loaders
  // One loader WARP per unit, units round-robin over the NLW loader warps (unit u -> warp u % NLW, ring slot u % STAGES), so NLW
  // units' global loads are in flight per SM; a slot is refilled in unit order (the a_empty wait of use n cannot be overtaken: use
  // n + 1 of that slot belongs to a warp that has not filled it yet, so no mbarrier phase is skipped); with all loader warps on one
  // unit at a time they would sit on the load latency.  Each warp enumerates ONLY its own units (see the Cfg note): one runtime
  // loop, one copy of the body (unrolled bodies bloat the kernel's code).
  else if (warp < 4 * TC_WGS + C::NLW) {
    setmaxnreg_dec<TC_LOADER_REGS>();
    const int lw = warp - 4 * TC_WGS;
    static_assert(KC == 16, "lane_voxel / unit-row mapping below is written for 64-byte operand rows");
    constexpr int CPR = KC / 4;                      // fp32 16-byte chunks per voxel of the K chunk
    constexpr int VPL = 32 / CPR;                    // voxels covered by one warp-wide LDG.128
    constexpr int NLD = 128 / VPL;                   // loads per lane per unit
    static_assert(W % VPL == 0, "a load instruction must not straddle image rows");
    const int v0 = lane_voxel<KC>(lane), c = lane % CPR;   // permuted voxel order: conflict-free STS.64 (tc_common.cuh)
    float amax = 0.f;
    uint32_t ubase = 0;                              // global index of the current phase's first unit
    int first = lw;                                  // this warp's first local unit index in the current phase: (ubase + first) % NLW == lw
    auto fill = [&](const float* base, size_t rstride, size_t cstride, int h_first, int h_step, uint32_t u, int col0) {
      // base: this lane's address for load 0; load j covers operand rows VPL*j .. VPL*j + VPL - 1 = columns (VPL*j) % W ..
      // of tile row (VPL*j) / W, read from image row h_first + h_step * tile row (rstride / cstride floats per tile row / column).
      // General widths: col0 = INPUT column of load 0 (columns >= Wp are zero: beyond the image).
      float4 v[NLD];
#pragma unroll
      for (int j = 0; j < NLD; ++j) {
        const int hin = h_first + h_step * ((VPL * j) / W);
        const size_t off = (size_t)((VPL * j) / W) * rstride + (size_t)((VPL * j) % W) * cstride;
        bool ok = hin >= 0 && hin < p.H;
        if (GW) ok = ok && (unsigned)(col0 + VPL * j) < (unsigned)Wp;
        v[j] = ok ? __ldg(reinterpret_cast<const float4*>(base + (ptrdiff_t)off)) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      const uint32_t slot = u % C::STAGES, ph = (u / C::STAGES) & 1;   // u = global unit index
      mbar_wait_relaxed(&a_empty[slot], ph ^ 1);
      uint8_t* tile = a_buf + slot * C::UNIT_BYTES;
#pragma unroll
      for (int j = 0; j < NLD; ++j) stage_f16_split<KC>(tile, v0 + VPL * j, c, v[j], amax);
      fence_proxy_async();
      mbar_arrive(&a_ready[slot]);
    };
    for (int it = blockIdx.x; it < p.items; it += gridDim.x) {
      const ItemDc w = decode_dc<C>(p, it / C::NG);   // every channel group of a tile stages the same units
      for (int kd = 0; kd < KS; ++kd) {
        if (!kd_valid(w.od, kd, p.D)) continue;
        const int id = (w.od + 1 - kd) >> 1;         // input plane feeding output plane od through tap kd
        const float* plane = p.x + ((size_t)w.b * p.D + id) * p.H * (size_t)Wp * p.Cin;
        const int col0 = w.ct * C::CSTEP + v0;       // INPUT column of this lane's first load (whole-row kernels: v0)
        for (int ch = 0; ch < nchunk; ++ch) {
#pragma unroll 1
          for (int j = first; j < C::NU; j += C::NLW) {
            // unit j = the R input rows at offset 1 - j from the item's block (rows outside the image are zeros)
            const int h_first = w.j0 + 1 - j;
            const float* base = plane + ((ptrdiff_t)h_first * Wp + col0) * p.Cin + ch * KC + c * 4;
            fill(base, (size_t)Wp * p.Cin, (size_t)p.Cin, h_first, 1, ubase + j, col0);
          }
          ubase += C::NU;
          first = (first + C::NLW - C::NU % C::NLW) % C::NLW;
        }
      }
    }
    tc_report_overflow(p.overflow, amax);
  }
  // ---------------------------------------------------------------------------------------------- weight-slice producer
  // One elected lane streams the item's channel group of the pre-swizzled (kd, chunk, kh) slices -- KS G-row kw blocks, 1-D bulk
  // copies -- into the two buffer sets, up to a whole phase ahead of the MMAs (tc_common.cuh: bulk_g2s).  Every kh slice serves one
  // of the two row parities in every phase.  The other warps of this warpgroup are idle: they only hand their registers back.
  else {
    setmaxnreg_dec<TC_PRODUCER_REGS>();
    if (warp == 4 * TC_WGS + C::NLW && elect_one()) {
      const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(p.w);
      uint32_t phc = 0;
      for (int it = blockIdx.x; it < p.items; it += gridDim.x) {
        const int cg = (it % C::NG) * C::G;
        const ItemDc w = decode_dc<C>(p, it / C::NG);
        for (int kd = 0; kd < KS; ++kd) {
          if (!kd_valid(w.od, kd, p.D)) continue;         // same phase enumeration as the consumers and the A loaders
          for (int ch = 0; ch < nchunk; ++ch, ++phc) {
            for (int kh = 0; kh < KS; ++kh) {
              const uint32_t slot = (phc & 1) * KS + kh;
              const size_t slice = ((size_t)kd * nchunk + ch) * KS + kh;
              mbar_wait_relaxed(&b_empty[slot], ((phc >> 1) & 1) ^ 1);
              mbar_arrive_expect_tx(&b_full[slot], C::B_SUB);
#pragma unroll
              for (int kw = 0; kw < KS; ++kw)
                bulk_g2s(b_buf + slot * C::B_SUB + kw * C::G * C::ROWB, wsrc + slice * C::B_SLICE + (size_t)(kw * COUT + cg) * C::ROWB,
                         C::G * C::ROWB, &b_full[slot]);
            }
          }
        }
      }
    }
    __syncwarp();
  }
}

template <int COUT, int KC, int W, int TILES, bool GW = false, int KS = 3>
static int launch_tcdc(const TcArgs& a, cudaStream_t stream) {
  using C = TcdcCfg<COUT, KC, W, TILES, GW, KS>;
  TcdcParams p{};
  p.ystride = a.ystride, p.cout_real = a.cout_real;
  p.hblocks = (a.H + C::HBLK - 1) / C::HBLK;
  p.Wr = GW ? a.W : W;
  p.ctiles = GW ? (a.W + C::CSTEP - 1) / C::CSTEP : 1;
  static const std::string variant = tc_variant_name("tcdc<%d,%d,%d,%d,%d,%d>", COUT, KC, W, TILES, (int)GW, KS);
  return launch_persistent<conv3d_tcdc_kernel<COUT, KC, W, TILES, GW, KS>>(   // both row parities per item
      a, p, (long long)a.B * (2 * a.D) * p.hblocks * p.ctiles * C::NG, C::SMEM, variant.c_str(), stream);
}

// The instantiation that serves a transposed conv of kernel size `ks` (INPUT width W), writing a channel slice; null when there is
// none.
static TcLaunch select_deconv3d_tc(int ks, int Cin, int Cout, int W, bool slice) {
  if (Cin % 16 != 0 || Cin < 16) return nullptr;
  if (ks == 4) {
    if (W == 16 && Cout == 64) return launch_tcdc<64, 16, 16, 1, false, 4>;   // StereoBase conv3_up: 6c -> 4c = 96 as slices 64 + 32
    if (W == 16 && Cout == 32) return launch_tcdc<32, 16, 16, 1, false, 4>;
    if (slice) return nullptr;                                              // channel slices are instantiated for W = 16 only
    if (W == 32 && Cout == 64) return launch_tcdc<64, 16, 32, 1, false, 4>;
    if (W == 64 && Cout == 32) return launch_tcdc<32, 16, 64, 1, false, 4>;
    return nullptr;
  }
  if (ks != 3 || slice) return nullptr;
  if (W == 32 && Cout == 64) return launch_tcdc<64, 16, 32, 1>;
  if (W == 64 && Cout == 32) return launch_tcdc<32, 16, 64, 1>;
  if (!osb_tc_general_width(W)) return nullptr;
  if (Cout == 64) return launch_tcdc<64, 16, 128, 1, true>;                 // 128-column tiles of the INPUT row
  if (Cout == 32) return launch_tcdc<32, 16, 128, 1, true>;
  return nullptr;
}

static int deconv3d_tc_impl(int ks, TcArgs a, cudaStream_t stream) {
  OSB_REQUIRE(select_deconv3d_tc(ks, a.Cin, a.Cout, a.W, false), "deconv3d_k%d_tc: unsupported shape Cin=%d Cout=%d W=%d", ks, a.Cin,
              a.Cout, a.W);
  const TcLaunch launch = select_deconv3d_tc(ks, a.Cin, a.Cout, a.W, a.slice());
  const int rc = check_tc_args(ks == 4 ? "deconv3d_k4_tc" : "deconv3d_k3_tc", a, launch);
  return rc != OSB_OK ? rc : launch(a, stream);
}

}  // namespace osb

extern "C" {

int osb_deconv3d_tc_supported(int Cin, int Cout, int W) { return osb::select_deconv3d_tc(3, Cin, Cout, W, false) ? 1 : 0; }

int osb_deconv3d_k4_tc_supported(int Cin, int Cout, int W) { return osb::select_deconv3d_tc(4, Cin, Cout, W, false) ? 1 : 0; }

int osb_deconv3d_k4_tc_fwd(const float* x_ndhwc, const void* w_split, const float* scale, const float* shift,
                           const float* residual, float* y, int B, int Cin, int Cout, int cout_real, int D, int H, int W, int act,
                           int out_ndhwc, int res_ndhwc, osb_stream_t stream) {
  return osb::deconv3d_tc_impl(4, {x_ndhwc, w_split, scale, shift, residual, nullptr, y, B, Cin, Cout, D, H, W, act, out_ndhwc, res_ndhwc,
                                   0, 0, cout_real}, (cudaStream_t)stream);
}

int osb_deconv3d_k4_tc_cs_fwd(const float* x_ndhwc, const void* w_split, const float* scale, const float* shift, float* y, int B,
                              int Cin, int Cout, int D, int H, int W, int act, int ystride, osb_stream_t stream) {
  return osb::deconv3d_tc_impl(4, {x_ndhwc, w_split, scale, shift, nullptr, nullptr, y, B, Cin, Cout, D, H, W, act, 1, 1, 0, ystride,
                                   Cout}, (cudaStream_t)stream);
}

int osb_deconv3d_k3_tc_fwd(const float* x_ndhwc, const void* w_split, const float* scale, const float* shift,
                           const float* residual, float* y, int B, int Cin, int Cout, int D, int H, int W, int act,
                           int out_ndhwc, int res_ndhwc, osb_stream_t stream) {
  return osb::deconv3d_tc_impl(3, {x_ndhwc, w_split, scale, shift, residual, nullptr, y, B, Cin, Cout, D, H, W, act, out_ndhwc, res_ndhwc,
                                   0, 0, Cout}, (cudaStream_t)stream);
}
}
