// Tensor-core (Hopper wgmma) implicit-GEMM Conv3d 3x3x3, stride 1, pad 1, for the full-resolution layers of the hourglass
// aggregation (W = 128 output columns = one 128-row M tile).  fp32-accurate through 3xFP16 operand splitting (tc_common.cuh):
//   a*b ~= a_lo*b_hi + a_hi*b_lo + a_hi*b_hi   on wgmma (fp16 operands), fp32 accumulation in registers.
// Activations are split while they are staged (fp32 in HBM -> [hi | lo] fp16 rows in shared memory); weights are split
// and pre-scaled once on the host.  Plain TF32 / BF16 / FP16 operands break the 1e-3 px EPE bar (SURVEY.md section 4.3);
// the split keeps it (tests/test_zz_fullsize_gpu.py).
//
// Replaces the same reference modules as conv3d.cu (convbn_3d + ReLU of gwcnet/hourglass.py:5-16,
// gwcnet_disp_processor.py:40-81; conv3d_bn(_relu) psmnet/submodule.py:68-83,160-177) for layers with W == 128.
//
// GEMM mapping.  Activations are channels-last (B, D, H, W, Cin): an A tile is "the 128 voxels of one image row x 32
// input channels", K-major with 128-byte rows in the canonical SWIZZLE_128B layout.
//   * the three kw taps are NOT realised by shifting A (that would need halo columns and unaligned tiles); instead the
//     three weight slices are stacked along N -- one MMA of N = 3*Cout produces P_kw[m] = A[m] . B_kw for kw = 0,1,2 --
//     and the epilogue forms D[m] = P_0[m-1] + P_1[m] + P_2[m+1] with warp shuffles (zero padding at m = -1 / 128 is
//     implicit because a row tile spans the whole image width).
//   * kh taps: output row h needs input rows h-1, h, h+1, staged through a shared-memory ring; row r of a phase meets weight
//     slice kh = r.
//   * an operand row is 128 bytes = two split granules [16 hi | 16 lo | 16 hi | 16 lo] fp16, SWIZZLE_128B; a K = 16 MMA step
//     is 32 bytes, so the hi k-steps sit at descriptor offsets +0, +4 and the lo ones at +2, +6 (16-byte units) of the SAME tile
//     (weight rows stay [32 hi | 32 lo]: hi +0, +2, lo +4, +6).
//   * kd taps and 32-channel Cin chunks are phases of one work item; the three kh weight slices of a phase are double-buffered.
// Work item = (image b, output plane d, output rows 2p and 2p + 1): TWO accumulator tiles of 128 x 3*Cout fp32, one per consumer
// warpgroup, each held in that warpgroup's registers as two m64 halves (96 registers per thread for Cout = 32).  A phase stages
// input rows 2p - 1 .. 2p + 2 once and both warpgroups read them: warpgroup t meets phase row r with weight slice kh = r - t
// (0 <= r - t <= 2), so an input row is staged twice per two output rows instead of three times per output row, and each weight
// slice a phase streams serves both output rows.
//
// Operand staging.  A split NDHWC input (tc_common.cuh) is already in operand form: one elected lane of the loader warpgroup
// copies each row with a TMA tensor copy (128-byte swizzle, zero fill for rows outside the image) straight into the ring.  fp32
// inputs go through the converters: the loader warps read coalesced float4 from global/L2 (or the raw rows a bulk-copy producer
// staged), convert to the hi/lo fp16 pair, write the row in the same granule order with the 128-byte swizzle applied by hand (two
// conflict-free STS.64) and publish the tile to the tensor core through fence.proxy.async + mbarrier.
//
// Warp roles (512 threads, 1 CTA/SM, persistent; setmaxnreg moves the registers, tc_common.cuh): warps 0-7 = two consumer
// warpgroups (wgmma issue, then the epilogue of the finished tile on the accumulator fragments: kw un-shift by shuffles, BN /
// residual / activation, stores through a per-warp 16-row tile; tc_common.cuh: frag_unshift, frag_epilogue), warps 8-11 = A-row
// loaders, warp 12 = weight-slice producer (one elected
// lane issuing 1-D bulk copies of the pre-swizzled slices into two buffer sets), warp 13 = raw-row producer (bulk copies of
// whole fp32 input rows ahead of the converters), warps 14-15 idle.
//
// Shared memory (Cout = 32): A ring 4 x 16 KB | weights 2 x 3 x 12 KB | raw rows 2 x 16 KB | per warpgroup a double-buffered
// seam-row buffer (4 KB) | per consumer warp a 16 x 40 fp32 output tile (2.5 KB) = 202,240 of the 232,448 bytes a CTA may have.
#include <type_traits>

#include "tc_common.cuh"

namespace osb {

constexpr int TC_W = 128;          // image width handled (M tile)
constexpr int TC_KC = 32;          // input channels per phase: 128-byte K-major rows [32 hi | 32 lo] fp16, SWIZZLE_128B
constexpr int TC_TILES = TC_WGS;   // output rows (accumulator tiles) per work item: one per consumer warpgroup
constexpr int TC_ROWS = TC_TILES + 2;
constexpr int TC_STAGES = 4;       // A-row ring depth (converted fp16 hi|lo tiles)
constexpr int TC_RAW = 2;          // raw fp32 rows staged by 1-D TMA bulk copies ahead of the converters (Cin = 32 channels-last layers)
constexpr int TC_ROW_BYTES = TC_W * TC_KC * 4;     // 16384: one staged input row (hi and lo halves of every voxel)

struct TcParams {
  CUtensorMap xmap;        // in_split: the input as split NDHWC rows (make_tensor_map_split)
  const float* x;          // (B, D, H, W, Cin) channels-last
  const void* w;           // fp16 [3 kd][Cin/32][3 kh][3*Cout][32 hi | 32 lo]  (ops.pack_tc_weight)
  const float* scale;
  const float* shift;
  const float* residual;
  float* y;
  int B, D, H, Cin, Cout;
  int act;
  float kappa;       // expected round-towards-zero loss per accumulating MMA (tc_common.cuh)
  unsigned int* overflow;  // sticky fp16-range flag (tc_common.cuh)
  int out_ndhwc, res_ndhwc;
  int bulk_rows;     // input rows staged by TMA bulk copies, TC_RAW deep: Cin == 32 channels-last (one 16 KB copy per row) or NCDHW
                     // (32 copies of 512 bytes, one per channel plane)
  int in_ncdhw;      // the INPUT is (B, Cin, D, H, W): the first aggregation layer reads the cost volume as the volume kernel wrote it
  int in_split, out_split, res_split;   // x / y / residual are split NDHWC (tc_common.cuh)
  int items, hblocks;
};

template <int COUT>
struct TcCfg {
  static constexpr int N3 = 3 * COUT;                      // kw-stacked MMA N
  static constexpr int B_SLICE = N3 * TC_KC * 4;           // one kh weight slice, rows [hi | lo] (12288 B for Cout = 32)
  static constexpr int XCHG_FLOATS = 2 * frag_xchg_floats<COUT, 1>();   // per consumer warpgroup: double-buffered seam rows
  static constexpr int A_OFF = 0;
  static constexpr int B_OFF = A_OFF + TC_STAGES * TC_ROW_BYTES;      // [2][3 kh]
  static constexpr int RAW_OFF = B_OFF + TC_BSLOTS * 3 * B_SLICE;    // [TC_RAW] raw fp32 input rows
  static constexpr int BAR_OFF = RAW_OFF + TC_RAW * TC_ROW_BYTES;
  static constexpr size_t SMEM = 1024 + (size_t)BAR_OFF + 256 + TC_WGS * XCHG_FLOATS * 4 + 4 * TC_WGS * FRAG_TP_FLOATS * 4 + 2 * COUT * 4;
  static_assert(B_SLICE % 1024 == 0, "weight slices must stay 1024-byte aligned");
  static_assert(SMEM <= 232448, "shared memory budget of one CTA exceeded");
};

template <int COUT>
__global__ void __launch_bounds__(TC_WG_THREADS, 1) conv3d_tc_kernel(const __grid_constant__ TcParams p) {
  using C = TcCfg<COUT>;
  constexpr int N3 = C::N3;
  constexpr int B_SLICE = C::B_SLICE;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte aligned (SWIZZLE_128B atoms).  Offsetting smem_raw itself, not a round-tripped integer address, keeps every derived
  // pointer in the shared window: the compiler emits LDS/STS with 32-bit addresses instead of generic 64-bit ones.
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* a_buf = smem + C::A_OFF;
  uint8_t* b_buf = smem + C::B_OFF;
  uint8_t* raw_buf = smem + C::RAW_OFF;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::BAR_OFF);
  uint64_t* a_ready = bars;                         // [STAGES] loaders -> consumers  (128 arrivals)
  uint64_t* a_empty = a_ready + TC_STAGES;          // [STAGES] consumers -> loaders  (8 arrivals: one per consumer warp)
  uint64_t* b_full = a_empty + TC_STAGES;           // [2][3]   weight producer -> consumers (expect_tx + bulk-copy bytes)
  uint64_t* b_empty = b_full + TC_BSLOTS * 3;       // [2][3]   consumers -> weight producer (8 arrivals)
  uint64_t* raw_full = b_empty + TC_BSLOTS * 3;     // [RAW]    row producer -> converters (expect_tx + bulk-copy bytes, or a plain arrive)
  uint64_t* raw_empty = raw_full + TC_RAW;          // [RAW]    converters -> row producer (128 arrivals)
  float* xchg = reinterpret_cast<float*>(smem + C::BAR_OFF + 256);   // [TC_WGS][XCHG_FLOATS] boundary exchange
  float* tiles = xchg + TC_WGS * C::XCHG_FLOATS;           // [8 consumer warps][FRAG_TP_FLOATS] output tiles
  float* s_scale = tiles + 4 * TC_WGS * FRAG_TP_FLOATS;     // [COUT]
  float* s_shift = s_scale + COUT;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nchunk = p.Cin / TC_KC;

  if (threadIdx.x == 0) {
    for (int s = 0; s < TC_STAGES; ++s) {
      mbar_init(&a_ready[s], p.in_split ? 1 : 128);   // one expect_tx arrival of the TMA issuer, or every converter thread
      mbar_init(&a_empty[s], 4 * TC_WGS);
    }
    for (int k = 0; k < TC_BSLOTS * 3; ++k) {
      mbar_init(&b_full[k], 1);
      mbar_init(&b_empty[k], 4 * TC_WGS);
    }
    for (int k = 0; k < TC_RAW; ++k) {
      mbar_init(&raw_full[k], 1);
      mbar_init(&raw_empty[k], 128);
    }
    fence_mbar_init();
  }
  for (int c = threadIdx.x; c < COUT; c += blockDim.x) {
    s_scale[c] = p.scale ? p.scale[c] : 1.f;
    s_shift[c] = p.shift ? p.shift[c] : 0.f;
  }
  __syncthreads();
  // The rows a CTA stages form one flat sequence (item, kd, chunk, r).  `RowIter` walks it; loads run TWO rows ahead of
  // the stores (software pipeline in registers) so that a full L2/HBM round trip is always in flight.
  struct RowIter {
    int it, kd, ch, r;
  };
  auto advance = [&](RowIter& s) {                  // -> false when the sequence is exhausted
    for (;;) {
      if (s.it >= p.items) return false;
      if (++s.r < TC_ROWS) return true;
      s.r = -1;
      if (++s.ch < nchunk) continue;
      s.ch = 0;
      const int d = (s.it / p.hblocks) % p.D;
      for (++s.kd; s.kd < 3; ++s.kd) {
        const int din = d + s.kd - 1;
        if (din >= 0 && din < p.D) break;
      }
      if (s.kd < 3) continue;
      s.it += gridDim.x;
      if (s.it >= p.items) return false;
      const int d2 = (s.it / p.hblocks) % p.D;
      s.kd = (d2 == 0) ? 1 : 0;                     // first input plane that exists
    }
  };
  // ---------------------------------------------------------------------------------------------- consumer warpgroups
  // Warpgroup wg accumulates output row 2p + wg of the item from the rows and weight slices both warpgroups read, then runs the
  // epilogue of that row on the accumulator fragments (tc_common.cuh: frag_unshift, frag_epilogue).
  if (warp < 4 * TC_WGS) {
    setmaxnreg_inc<TC_CONSUMER_REGS>();
    const int wg = warp >> 2;
    xchg += wg * C::XCHG_FLOATS;
    const int bar_xchg = 1 + wg;                     // this warpgroup's named barrier
    constexpr uint32_t A_HALF = 64 * TC_KC * 4 / 16;  // descriptor offset of operand rows 64..127
    const uint64_t dbase = desc_sw128_base();
    // Descriptors differ only in their 14-bit start-address field (bits 0-13, units of 16 bytes).
    const uint32_t b16 = (smem_u32(b_buf) & 0x3FFFF) >> 4;
    const int q = warp & 3;                          // warp of the warpgroup
    uint32_t rowc = 0, phc = 0, exc = 0;
    for (int it = blockIdx.x; it < p.items; it += gridDim.x) {
      const int d = (it / p.hblocks) % p.D;
      const int b = it / (p.hblocks * p.D);
      const int h = (it % p.hblocks) * TC_TILES + wg;
      // the residual streams from HBM / L2: pull one voxel's channels per thread into L2 while the row is being accumulated
      if (h < p.H && p.residual && p.res_ndhwc)
        asm volatile("prefetch.global.L2 [%0];" ::"l"(p.residual + ((((size_t)b * p.D + d) * p.H + h) * TC_W + q * 32 + lane) * COUT));
      float acc[2][N3 / 2];
      uint32_t accum = 0;
      for (int kd = 0; kd < 3; ++kd) {
        const int din = d + kd - 1;
        if (din < 0 || din >= p.D) continue;
        for (int ch = 0; ch < nchunk; ++ch, ++phc) {
          const uint32_t bslot = (phc & 1) * 3;     // weight buffers alternate between phases
#pragma unroll
          for (int r = 0; r < TC_ROWS; ++r) {
            // Every warpgroup waits for each row's fill and releases it, including the row its own tile does not read, so neither
            // can arrive on a later phase of a slot than the one being filled.
            const uint32_t s = rowc % TC_STAGES, par = (rowc / TC_STAGES) & 1;
            mbar_wait(&a_ready[s], par);
            const int kh = r - wg;                  // input row r of the phase meets weight slice kh for output row 2p + wg
            if (kh >= 0 && kh < 3) {
              mbar_wait(&b_full[bslot + kh], (phc >> 1) & 1);
              const uint64_t da0 = dbase | (uint64_t)((smem_u32(a_buf + s * TC_ROW_BYTES) & 0x3FFFF) >> 4);
              const uint64_t db0 = dbase | (uint64_t)(b16 + (bslot + kh) * (B_SLICE / 16));
              wg_fence();
#pragma unroll
              for (int ks = 0; ks < TcK<TC_KC>::KSTEPS; ++ks)
                wg_mma_split<N3>(acc, da0 + TcK<TC_KC>::A_KSTEP * ks, A_HALF, TcK<TC_KC>::A_LO, db0 + 2 * ks, TcK<TC_KC>::B_LO,
                                 ks > 0 ? 1u : accum);
              wg_commit();
              wg_wait_all();
              accum = 1;
              wg_release(&b_empty[bslot + kh], lane);   // the weight slice is free once these MMAs have read it
            }
            wg_release(&a_empty[s], lane);
            ++rowc;
          }
        }
      }
      // A tile below the image (odd H) received its MMAs and releases like any other and stores nothing.  The branch is
      // warpgroup-uniform and the epilogue's barrier and seam buffer are this warpgroup's own.
      if (h >= p.H) continue;
      // MMAs each P_kw accumulator received: (existing kd planes) x chunks x 3 kh x k-steps x 3 split terms
      const float corr = 1.f + p.kappa * (float)(((d > 0) + 1 + (d + 1 < p.D)) * nchunk * 3 * TcK<TC_KC>::KSTEPS * 3);
      frag_unshift<COUT, 1, TC_W>(acc, xchg + (exc & 1) * (C::XCHG_FLOATS / 2), q, lane, corr, bar_xchg);
      ++exc;
      const size_t row0 = (((size_t)b * p.D + d) * p.H + h) * TC_W;                // NDHWC voxel index of column 0
      const size_t plane = (size_t)p.D * p.H * TC_W;                               // NCDHW channel stride
      const size_t ncdhw0 = (size_t)b * p.Cout * plane + ((size_t)d * p.H + h) * TC_W;   // p.Cout <= COUT real channels
      auto rows = [&](int m, ptrdiff_t& yo, ptrdiff_t& ro, ptrdiff_t& go) {      // m = image column
        yo = p.out_ndhwc ? (ptrdiff_t)(row0 + m) * COUT : (ptrdiff_t)(ncdhw0 + m);
        ro = p.res_ndhwc ? (ptrdiff_t)(row0 + m) * COUT : (ptrdiff_t)(ncdhw0 + m);
        go = 0;
        return true;
      };
      frag_epilogue<COUT>(acc, lane, q, tiles + warp * FRAG_TP_FLOATS, s_scale, s_shift, p.act, p.y, p.out_ndhwc ? 1 : plane, p.residual, p.res_ndhwc ? 1 : plane,
                          nullptr, rows, COUT == 32 ? 32 : p.Cout, p.out_split, p.res_split, p.overflow);
    }
  }
  // ---------------------------------------------------------------------------------------------- A-row loaders
  else if (warp < 4 * TC_WGS + 4) {
    setmaxnreg_dec<TC_LOADER_REGS>();
    if (p.in_split) {
      // split rows: one elected lane of warp 8 copies each row of the sequence with a TMA tensor copy of the chunk's two granules
      // x 128 columns; rows above / below the image fall outside the map and arrive as zeros (the conv's padding)
      if (warp == 4 * TC_WGS && elect_one()) {
        RowIter ld{(int)blockIdx.x, 0, 0, -1};
        if (ld.it < p.items) ld.kd = (((ld.it / p.hblocks) % p.D) == 0) ? 1 : 0;
        uint32_t rowc = 0;
        while (advance(ld)) {
          const int hb = ld.it % p.hblocks;
          const int d = (ld.it / p.hblocks) % p.D;
          const int b = ld.it / (p.hblocks * p.D);
          const uint32_t s = rowc % TC_STAGES, par = (rowc / TC_STAGES) & 1;
          mbar_wait_relaxed(&a_empty[s], par ^ 1);
          mbar_arrive_expect_tx(&a_ready[s], TC_ROW_BYTES);
          tma_load_4d(a_buf + s * TC_ROW_BYTES, &p.xmap, &a_ready[s], 2 * TC_KC * ld.ch, 0, hb * TC_TILES - 1 + ld.r, b * p.D + d + ld.kd - 1);
          ++rowc;
        }
      }
      __syncwarp();
      return;
    }
    const int lt = threadIdx.x - 4 * TC_WGS * 32;    // 0..127
    const int vsel = lt >> 3, c16 = lt & 7;          // this thread's voxel (mod 16) and fp32 16-byte chunk of the 32-channel slice
    // voxel order inside a half-warp alternates bit 1 of the column: a granule-ordered row puts its hi halves in chunks {0,1,4,5}
    // and its lo halves in {2,3,6,7}, and only rows differing in bit 1 swizzle those onto disjoint banks (conflict-free STS.64)
    const int vcol = ((vsel & 1) << 1) | ((vsel >> 1) & 1) | (vsel & 12);
    float amax = 0.f;
    // The two input layouts run separate copies of the loops below (NCDHW is a compile-time flag), so that each copy keeps only
    // its own layout's swizzled store offsets live: both fit the loaders' register budget (TC_LOADER_REGS) without spilling.
    auto run = [&](auto in_ncdhw) {
      constexpr bool NCDHW = decltype(in_ncdhw)::value;
      const size_t row_stride = (size_t)TC_W * p.Cin;  // floats per image row
      auto load_row = [&](const RowIter& s, float4 (&v)[8]) {
        const int hb = s.it % p.hblocks;
        const int d = (s.it / p.hblocks) % p.D;
        const int b = s.it / (p.hblocks * p.D);
        const int hin = hb * TC_TILES - 1 + s.r, din = d + s.kd - 1;
        if (hin >= 0 && hin < p.H && NCDHW) {
          // NCDHW input: this thread stages voxel (column) lt for all eight channel quads; every LDG.32 of a warp is one
          // contiguous 128-byte row segment of a channel plane.  v[j] holds channels 4*qj .. 4*qj+3, qj = j ^ ((lt >> 3) & 1)
          // (the swap keeps the STS.64 of lanes 8 apart -- same swizzled chunk -- on different 8-byte halves).
          const size_t plane = (size_t)p.D * p.H * TC_W;
          const float* src = p.x + (((size_t)b * p.Cin + s.ch * TC_KC) * p.D + din) * p.H * TC_W + (size_t)hin * TC_W + lt;
          // channels in plane order (one running address), then the quad swap as register selects
#pragma unroll
          for (int j = 0; j < 8; ++j, src += 4 * plane)
            v[j] = make_float4(__ldg(src), __ldg(src + plane), __ldg(src + 2 * plane), __ldg(src + 3 * plane));
          const bool swap = (lt >> 3) & 1;
#pragma unroll
          for (int j = 0; j < 8; j += 2) {
            const float4 e = v[j], o = v[j + 1];
            v[j] = swap ? o : e;
            v[j + 1] = swap ? e : o;
          }
        } else if (hin >= 0 && hin < p.H) {             // rows outside the image are the conv's zero padding
          const float* src = p.x + (((size_t)b * p.D + din) * p.H + hin) * row_stride + s.ch * TC_KC + c16 * 4 + vcol * p.Cin;
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = __ldg(reinterpret_cast<const float4*>(src + 16 * j * p.Cin));
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      };
      uint32_t rowc = 0;
      auto store_row = [&](const float4 (&v)[8]) {
        const uint32_t s = rowc % TC_STAGES, par = (rowc / TC_STAGES) & 1;
        mbar_wait_relaxed(&a_empty[s], par ^ 1);        // the MMAs that read this slot last time have completed
        uint8_t* tile = a_buf + s * TC_ROW_BYTES;
        if (NCDHW) {
#pragma unroll
          for (int j = 0; j < 8; ++j) stage_f16_split<TC_KC>(tile, lt, j ^ ((lt >> 3) & 1), v[j], amax);
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) stage_f16_split<TC_KC>(tile, vcol + 16 * j, c16, v[j], amax);   // tile row = image column
        }
        fence_proxy_async();                            // generic-proxy writes -> visible to the tensor core (async proxy)
        mbar_arrive(&a_ready[s]);
        ++rowc;
      };
      RowIter ld{(int)blockIdx.x, 0, 0, -1};
      if (ld.it < p.items) ld.kd = (((ld.it / p.hblocks) % p.D) == 0) ? 1 : 0;
      if (p.bulk_rows) {
        // The row producer (warp 13) keeps TC_RAW rows of raw fp32 in flight with 16 KB TMA bulk copies; these four warps only
        // convert: LDS.128 (a warp reads 512 contiguous bytes) -> fp16 hi|lo -> swizzled STS.64.  No load latency on this path.
        uint32_t rawc = 0;
        while (advance(ld)) {
          const int hb = ld.it % p.hblocks;
          const int hin = hb * TC_TILES - 1 + ld.r;
          const uint32_t slot = rawc % TC_RAW, par = (rawc / TC_RAW) & 1;
          mbar_wait_relaxed(&raw_full[slot], par);
          float4 v[8];
          if (hin >= 0 && hin < p.H && NCDHW) {    // raw slot = [32 channels][128 columns]: this thread's column, 8 channel quads
            const float* src = reinterpret_cast<const float*>(raw_buf + slot * TC_ROW_BYTES) + lt;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float* q = src + 4 * (j ^ ((lt >> 3) & 1)) * TC_W;
              v[j] = make_float4(q[0], q[TC_W], q[2 * TC_W], q[3 * TC_W]);
            }
          } else if (hin >= 0 && hin < p.H) {
            const float* src = reinterpret_cast<const float*>(raw_buf + slot * TC_ROW_BYTES) + c16 * 4;
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = *reinterpret_cast<const float4*>(src + (vcol + 16 * j) * TC_KC);
          } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
          }
          store_row(v);                                 // consumes v: the reads of the raw slot are complete behind it
          mbar_arrive(&raw_empty[slot]);
          ++rawc;
        }
        tc_report_overflow(p.overflow, amax);
        amax = 0.f;
      }
      float4 va[8], vb[8];
      bool has_a = !p.bulk_rows && advance(ld);
      if (has_a) load_row(ld, va);
      bool has_b = has_a && advance(ld);
      if (has_b) load_row(ld, vb);
      while (has_a) {
        store_row(va);
        has_a = has_b && advance(ld);
        if (has_a) load_row(ld, va);
        if (!has_b) break;
        store_row(vb);
        has_b = has_a && advance(ld);
        if (has_b) load_row(ld, vb);
      }
      tc_report_overflow(p.overflow, amax);
    };
    if (p.in_ncdhw) run(std::true_type{});
    else run(std::false_type{});
  }
  // ---------------------------------------------------------------------------------------------- producer warpgroup
  // Warp 12 is the weight-slice producer, warp 13 the raw-row producer (bulk-copied input rows only); warps 14-15 are idle and
  // only hand their registers back.
  else {
    setmaxnreg_dec<TC_PRODUCER_REGS>();
    // weight-slice producer: one elected lane streams the pre-swizzled (kd, chunk, kh) slices with 1-D bulk copies into the two
    // buffer sets; it runs up to a whole phase ahead of the MMAs.
    if (warp == 4 * TC_WGS + 4 && elect_one()) {
      const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(p.w);
      uint32_t phc = 0;
      for (int it = blockIdx.x; it < p.items; it += gridDim.x) {
        const int d = (it / p.hblocks) % p.D;
        for (int kd = 0; kd < 3; ++kd) {
          const int din = d + kd - 1;
          if (din < 0 || din >= p.D) continue;
          for (int ch = 0; ch < nchunk; ++ch, ++phc) {
            for (int kh = 0; kh < 3; ++kh) {
              const uint32_t slot = (phc & 1) * 3 + kh;
              const size_t slice = ((size_t)kd * nchunk + ch) * 3 + kh;
              mbar_wait_relaxed(&b_empty[slot], ((phc >> 1) & 1) ^ 1);   // the MMAs that read this buffer two phases ago are done
              mbar_arrive_expect_tx(&b_full[slot], B_SLICE);
              bulk_g2s(b_buf + slot * B_SLICE, wsrc + slice * B_SLICE, B_SLICE, &b_full[slot]);
            }
          }
        }
      }
    }
    // raw-row producer: bulk copies of whole fp32 input rows, TC_RAW ahead of the converters
    else if (warp == 4 * TC_WGS + 5 && p.bulk_rows && elect_one()) {
      RowIter ld{(int)blockIdx.x, 0, 0, -1};
      if (ld.it < p.items) ld.kd = (((ld.it / p.hblocks) % p.D) == 0) ? 1 : 0;
      uint32_t rawc = 0;
      while (advance(ld)) {
        const int hb = ld.it % p.hblocks;
        const int d = (ld.it / p.hblocks) % p.D;
        const int b = ld.it / (p.hblocks * p.D);
        const int hin = hb * TC_TILES - 1 + ld.r, din = d + ld.kd - 1;
        const uint32_t slot = rawc % TC_RAW, par = (rawc / TC_RAW) & 1;
        mbar_wait_relaxed(&raw_empty[slot], par ^ 1);
        if (hin >= 0 && hin < p.H && p.in_ncdhw) {      // NCDHW: 32 channel planes, each contributes one 512-byte image row
          const size_t plane = (size_t)p.D * p.H * TC_W;
          const float* src = p.x + (((size_t)b * p.Cin + ld.ch * TC_KC) * p.D + din) * p.H * TC_W + (size_t)hin * TC_W;
          mbar_arrive_expect_tx(&raw_full[slot], TC_ROW_BYTES);
          for (int c = 0; c < TC_KC; ++c)
            bulk_g2s(raw_buf + slot * TC_ROW_BYTES + c * (TC_W * 4), src + c * plane, TC_W * 4, &raw_full[slot]);
        } else if (hin >= 0 && hin < p.H) {             // one image row = 128 voxels x 32 channels x 4 B, contiguous
          const float* src = p.x + (((size_t)b * p.D + din) * p.H + hin) * (size_t)(TC_W * TC_KC);
          mbar_arrive_expect_tx(&raw_full[slot], TC_ROW_BYTES);
          bulk_g2s(raw_buf + slot * TC_ROW_BYTES, src, TC_ROW_BYTES, &raw_full[slot]);
        } else {
          mbar_arrive(&raw_full[slot]);                 // zero-padding row: nothing to copy, the converters write zeros
        }
        ++rawc;
      }
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------- layout conversion kernels
// NCDHW -> NDHWC through a 32x32 shared-memory transpose (both sides coalesced); with `ys`, to split NDHWC instead of y (each
// value's hi and lo halves, out-of-range values reported on `overflow`).  y voxels hold `ystride` >= Cp floats and the Cp channels
// land at channel `coff` of each, so that several NCDHW tensors fill one channels-last concatenation.
__global__ void __launch_bounds__(256) ncdhw_to_ndhwc_kernel(const float* __restrict__ x, float* __restrict__ y, int C, int Cp,
                                                             size_t vol, uint16_t* __restrict__ ys, unsigned int* overflow,
                                                             int ystride, int coff) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const size_t v0 = (size_t)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;       // 32 x 8
  float amax = 0.f;
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i;
    const size_t v = v0 + tx;
    tile[i][tx] = (c < C && v < vol) ? __ldg(x + ((size_t)b * C + c) * vol + v) : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const size_t v = v0 + i;
    const int c = c0 + tx;
    if (c >= Cp || v >= vol) continue;
    if (!ys) {
      y[((size_t)b * vol + v) * ystride + coff + c] = tile[tx][i];      // channels C .. Cp-1: zero padding
      continue;
    }
    const float s = tile[tx][i] * TC_ACT_SCALE;
    const uint32_t hl = cvt_f16x2_sat(s, s - f16x2_to_float2(cvt_f16x2_sat(s, 0.f)).x);   // {hi, lo}
    uint16_t* vox = ys + ((size_t)b * vol + v) * 2 * Cp;
    vox[split_index(c)] = (uint16_t)(hl & 0xFFFFu);
    vox[split_index(c) + SPLIT_GRANULE] = (uint16_t)(hl >> 16);
    amax = fmaxf(amax, fabsf(s));
  }
  if (ys) tc_report_overflow(overflow, amax);
}

template <int COUT>
int launch_tc(const TcArgs& a, cudaStream_t stream) {
  TcParams p{};
  p.Cout = a.Cout, p.in_ncdhw = a.in_ncdhw;
  p.in_split = a.in_split, p.out_split = a.out_split, p.res_split = a.res_split;
  p.bulk_rows = !a.in_split && (a.in_ncdhw || a.Cin == TC_KC);   // fp32 channels-last Cin = 64 rows are strided: register-staged
  if (a.in_split && !make_tensor_map_split(&p.xmap, a.x, a.Cin, TC_W, a.H, a.B * a.D, TC_KC)) return OSB_ECUDA;
  p.hblocks = (a.H + TC_TILES - 1) / TC_TILES;
  static const std::string variant = tc_variant_name("tc<%d>", COUT);
  return launch_persistent<conv3d_tc_kernel<COUT>>(a, p, (long long)a.B * a.D * p.hblocks, TcCfg<COUT>::SMEM, variant.c_str(), stream);
}
template int launch_tc<32>(const TcArgs&, cudaStream_t);
template int launch_tc<16>(const TcArgs&, cudaStream_t);   // classifier heads (32 -> 1): NCDHW output only

}  // namespace osb

extern "C" {

// Widths served by the general-width (column-tile) instantiations of conv3d_tcg.cu / conv3d_tcs2.cu / conv3d_tcdc.cu: any row of
// at least OSB_TC_MIN_WIDTH voxels (below that a 128-column tile is mostly padding and the fp32 CUDA-core kernels win).
int osb_tc_general_width(int W) { return W >= OSB_TC_MIN_WIDTH ? 1 : 0; }

// K-chunk (input channels per operand tile) of the kernel variant that serves a shape; 0 = no tensor-core variant.
int osb_conv3d_tc_kc(int Cin, int Cout, int W, int stride) {
  return stride == 1 ? osb::select_conv3d_tc(Cin, Cout, W, 1, false, false).kc : 0;
}

int osb_conv3d_tc_supported(int Cin, int Cout, int W, int stride) { return osb_conv3d_tc_kc(Cin, Cout, W, stride) != 0; }

int osb_ncdhw_to_ndhwc_pad(const float* x, float* y, int B, int C, int Cpad, int D, int H, int W, osb_stream_t stream) {
  using namespace osb;
  OSB_REQUIRE(x && y, "ncdhw_to_ndhwc: null pointer");
  OSB_REQUIRE(B > 0 && C > 0 && Cpad >= C && D > 0 && H > 0 && W > 0 && B <= 65535, "ncdhw_to_ndhwc: bad shape");
  const size_t vol = (size_t)D * H * W;
  dim3 grid((unsigned)((vol + 31) / 32), (Cpad + 31) / 32, B);
  ncdhw_to_ndhwc_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, y, C, Cpad, vol, nullptr, nullptr, Cpad, 0);
  count_launch();
  return check_launch("ncdhw_to_ndhwc_kernel");
}

int osb_ncdhw_to_split(const float* x, float* y_split, int B, int C, int D, int H, int W, osb_stream_t stream) {
  using namespace osb;
  OSB_REQUIRE(x && y_split, "ncdhw_to_split: null pointer");
  OSB_REQUIRE(B > 0 && C > 0 && C % SPLIT_GRANULE == 0 && D > 0 && H > 0 && W > 0 && B <= 65535,
              "ncdhw_to_split: bad shape (C must be a multiple of %d)", SPLIT_GRANULE);
  unsigned int* flag = tc_overflow_flag();
  if (!flag) return OSB_ECUDA;
  const size_t vol = (size_t)D * H * W;
  dim3 grid((unsigned)((vol + 31) / 32), (C + 31) / 32, B);
  ncdhw_to_ndhwc_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, nullptr, C, C, vol, reinterpret_cast<uint16_t*>(y_split), flag, C, 0);
  count_launch();
  return check_launch("ncdhw_to_ndhwc_kernel");
}

int osb_ncdhw_to_ndhwc(const float* x, float* y, int B, int C, int D, int H, int W, osb_stream_t stream) {
  return osb_ncdhw_to_ndhwc_pad(x, y, B, C, C, D, H, W, stream);
}

int osb_ncdhw_to_ndhwc_slice(const float* x, float* y, int B, int C, int D, int H, int W, int ystride, int coff, osb_stream_t stream) {
  using namespace osb;
  OSB_REQUIRE(x && y, "ncdhw_to_ndhwc_slice: null pointer");
  OSB_REQUIRE(B > 0 && C > 0 && D > 0 && H > 0 && W > 0 && B <= 65535, "ncdhw_to_ndhwc_slice: bad shape");
  OSB_REQUIRE(coff >= 0 && ystride >= coff + C, "ncdhw_to_ndhwc_slice: channels %d .. %d do not fit a voxel of %d", coff, coff + C - 1,
              ystride);
  const size_t vol = (size_t)D * H * W;
  dim3 grid((unsigned)((vol + 31) / 32), (C + 31) / 32, B);
  ncdhw_to_ndhwc_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, y, C, C, vol, nullptr, nullptr, ystride, coff);
  count_launch();
  return check_launch("ncdhw_to_ndhwc_kernel");
}

static int conv3d_k3_tc_impl(osb::TcArgs a, int dilation, osb_stream_t stream) {
  using namespace osb;
  const int kc = select_conv3d_tc(a.Cin, a.Cout, a.W, dilation, false, false).kc;
  OSB_REQUIRE(kc, "conv3d_k3_tc: unsupported shape Cin=%d Cout=%d W=%d dilation=%d", a.Cin, a.Cout, a.W, dilation);
  OSB_REQUIRE(!a.in_ncdhw || kc == 32, "conv3d_k3_tc: NCDHW input is served by the W = 128 kernel only");
  OSB_REQUIRE((!a.ystride && !a.gate) || kc == 16, "conv3d_k3_tc: a channel slice or gate needs the 16-channel-chunk kernels");
  OSB_REQUIRE(a.Cout > 16 || (!a.out_ndhwc && (!a.residual || !a.res_ndhwc)), "conv3d_k3_tc: Cout <= 16 writes (and adds) NCDHW tensors only");
  OSB_REQUIRE(!(a.in_split || a.out_split || a.res_split) || (kc == 32 && !a.ystride && !a.gate),
              "conv3d_k3_tc: split activations are served by the W = 128 kernel only");
  OSB_REQUIRE(!a.in_split || !a.in_ncdhw, "conv3d_k3_tc: an input is either NCDHW or split");
  OSB_REQUIRE((!a.out_split || a.out_ndhwc) && (!a.res_split || a.res_ndhwc), "conv3d_k3_tc: split tensors are channels-last");
  OSB_REQUIRE(!(a.out_split || a.res_split) || (a.out_ndhwc && (!a.residual || a.res_ndhwc)),
              "conv3d_k3_tc: a split output or residual needs a channels-last output and residual");
  const TcLaunch launch = select_conv3d_tc(a.Cin, a.Cout, a.W, dilation, a.gate != nullptr, a.slice()).launch;
  const int rc = check_tc_args("conv3d_k3_tc", a, launch);
  return rc != OSB_OK ? rc : launch(a, (cudaStream_t)stream);
}

int osb_conv3d_k3_tc_fwd(const float* x_ndhwc, const void* w_split, const float* scale, const float* shift,
                         const float* residual, float* y, int B, int Cin, int Cout, int D, int H, int W, int act,
                         int out_ndhwc, int res_ndhwc, osb_stream_t stream) {
  return conv3d_k3_tc_impl({x_ndhwc, w_split, scale, shift, residual, nullptr, y, B, Cin, Cout, D, H, W, act, out_ndhwc, res_ndhwc, 0, 0,
                            Cout}, 1, stream);
}

int osb_conv3d_k3_tc_gate_fwd(const float* x_ndhwc, const void* w_split, const float* scale, const float* shift,
                              const float* residual, const float* gate_nhwc, float* y, int B, int Cin, int Cout, int D, int H, int W,
                              int act, osb_stream_t stream) {
  OSB_REQUIRE(gate_nhwc, "conv3d_k3_tc_gate: null gate");
  return conv3d_k3_tc_impl({x_ndhwc, w_split, scale, shift, residual, gate_nhwc, y, B, Cin, Cout, D, H, W, act, 1, 1, 0, 0, Cout}, 1,
                           stream);
}

int osb_conv3d_k3_tc_cs_fwd(const float* x_ndhwc, const void* w_split, const float* scale, const float* shift, const float* residual,
                            const float* gate_nhwc, float* y, int B, int Cin, int Cout, int D, int H, int W, int act, int ystride,
                            osb_stream_t stream) {
  return conv3d_k3_tc_impl({x_ndhwc, w_split, scale, shift, residual, gate_nhwc, y, B, Cin, Cout, D, H, W, act, 1, 1, 0, ystride, Cout},
                           1, stream);
}

int osb_conv3d_k3_tc_ncdhw_fwd(const float* x_ncdhw, const void* w_split, const float* scale, const float* shift,
                               const float* residual, float* y, int B, int Cin, int Cout, int D, int H, int W, int act,
                               int out_ndhwc, int res_ndhwc, osb_stream_t stream) {
  return conv3d_k3_tc_impl({x_ncdhw, w_split, scale, shift, residual, nullptr, y, B, Cin, Cout, D, H, W, act, out_ndhwc, res_ndhwc, 1, 0,
                            Cout}, 1, stream);
}

int osb_conv3d_k3_tc_split_fwd(const float* x, const void* w_split, const float* scale, const float* shift, const float* residual,
                               float* y, int B, int Cin, int Cout, int D, int H, int W, int act, int in_layout, int out_layout,
                               int res_layout, osb_stream_t stream) {
  auto known = [](int l) { return l == OSB_LAYOUT_NCDHW || l == OSB_LAYOUT_NDHWC || l == OSB_LAYOUT_SPLIT; };
  OSB_REQUIRE(known(in_layout) && known(out_layout) && known(res_layout), "conv3d_k3_tc_split: unknown layout");
  osb::TcArgs a{x, w_split, scale, shift, residual, nullptr, y, B, Cin, Cout, D, H, W, act, out_layout != OSB_LAYOUT_NCDHW, res_layout != OSB_LAYOUT_NCDHW,
                in_layout == OSB_LAYOUT_NCDHW, 0, Cout};
  a.in_split = in_layout == OSB_LAYOUT_SPLIT, a.out_split = out_layout == OSB_LAYOUT_SPLIT, a.res_split = res_layout == OSB_LAYOUT_SPLIT;
  return conv3d_k3_tc_impl(a, 1, stream);
}

int osb_conv2d_tc_kc(int Cin, int Cout, int W, int dilation) { return osb::select_conv3d_tc(Cin, Cout, W, dilation, false, false).kc; }

int osb_conv2d_k3_tc_gru_fwd(const float* x_nhwc, const void* w_split, const float* scale, const float* shift, const float* residual,
                             const float* mul_nhwc, const float* blend_z_nhwc, const float* blend_h_nhwc, float* y, int B, int Cin,
                             int Cout, int H, int W, int act, int out_nhwc, int res_nhwc, long long res_bstride, osb_stream_t stream) {
  // the ConvGRU epilogue is compiled into conv3d_tcg.cu's Cout = 128 instantiations (TcgCfg::GRU)
  OSB_REQUIRE(Cout == 128 && osb::select_conv3d_tc(Cin, Cout, W, 1, false, false).kc == 16,
              "conv2d_k3_tc_gru: no Cout = 128 kernel of conv3d_tcg.cu serves Cin=%d Cout=%d W=%d", Cin, Cout, W);
  osb::TcArgs a{x_nhwc, w_split, scale, shift, residual, nullptr, y, B, Cin, Cout, 1, H, W, act, out_nhwc, res_nhwc, 0, 0, Cout};
  a.gru = 1, a.mul = mul_nhwc, a.blend_z = blend_z_nhwc, a.blend_h = blend_h_nhwc, a.res_bstride = res_bstride;
  return conv3d_k3_tc_impl(a, 1, stream);
}

int osb_conv2d_k3_tc_fwd(const float* x_nhwc, const void* w_split, const float* scale, const float* shift, const float* residual,
                         float* y, int B, int Cin, int Cout, int H, int W, int dilation, int act, int out_nhwc, int res_nhwc,
                         osb_stream_t stream) {
  return conv3d_k3_tc_impl({x_nhwc, w_split, scale, shift, residual, nullptr, y, B, Cin, Cout, 1, H, W, act, out_nhwc, res_nhwc, 0, 0,
                            Cout}, dilation, stream);
}
}
