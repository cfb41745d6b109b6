// Generic tensor-core (Hopper wgmma) Conv3d 3x3x3 stride 1 for the hourglass-interior layers whose image width is below the
// 128-row M tile: an M tile is R = 128 / W consecutive image rows (W = 64 -> 2 rows, W = 32 -> 4 rows).
//   conv2 64->64 @ 1/8 res, conv4 128->128 (GwcNet) / 64->64 (PSMNet) @ 1/16 res:
//   gwcnet/hourglass.py:25-32, psmnet/psmnet_cost_processor.py:86-98.
// Same scheme as conv3d_tc.cu (3xFP16 split, kw taps stacked along N and un-shifted in the epilogue, LDG-staged swizzled
// operands, warp-specialised persistent CTA with a consumer warpgroup that issues the wgmmas and runs the epilogue), generalised:
//   * an A "unit" is R consecutive input rows starting at block row s; tap kh of output tile t reads the unit with
//     s = t * R + kh - 1.  A work item is two such tiles, one per consumer warpgroup (TcgCfg::NT, tile_of): each unit and
//     weight slice is staged once and read by both, so the units between the two tiles and the whole weight stream serve two
//     output tiles;
//   * K chunks are 16 channels (64-byte rows [16 hi | 16 lo] fp16, SWIZZLE_64B: one K = 16 MMA step each);
//   * a work item covers G = 32 output channels: the accumulator tile is 128 x 3G = 96 fp32 columns (96 registers per consumer
//     thread), and the weight producer streams only the three G-row kw blocks of each slice (contiguous in shared memory, so one
//     N = 96 wgmma covers them); wider layers are COUT / G items per tile;
//   * the epilogue's +-1 column shift never crosses an image-row boundary (tile rows are whole image rows).
// GENERAL WIDTHS (GW = true, W = 128 instantiations): an M tile is a 128-column SEGMENT of one image row of runtime width Wr,
// starting at column ct * (128 - 2 DIL) - DIL: the first / last DIL tile columns are a halo (loaded like any other column, zero
// outside the image -- the conv's padding), the kw-stacked partial sums are un-shifted across the whole tile exactly as before and
// only the 128 - 2 DIL interior columns that exist in the image are stored.  Work items gain a column-tile index (fastest), so
// widths such as 240 (the reference's 544x960 timing shape), 312 (KITTI) or 160 take the tensor-core path with 1.6 % halo overhead.
// SINGLE-TERM MODE (runtime, TcArgs::terms == 1; DESIGN.md section 4.20): the loaders stage only the hi part of each operand row
// (same scale, saturation and overflow flag), the consumers issue one a_hi * b_hi MMA per half and K step instead of three, and the
// kappa * n correction counts those MMAs.  The weight pack is the same; its lo half is not read.  Epilogues are unchanged (fp32).
// MODULATED DEFORMABLE GATHER (runtime, TcgParams::dcn, general-width instantiations only; DESIGN.md section 4.21): the 3x3 DCNv2
// convolution of deform_conv_cuda_kernel.cu:571 (modulated_deformable_im2col + GEMM) as one launch.  Tiles are those of the 2D
// convolution (128 output columns of one row; the halo columns are gathered and not stored).  The loader warps stage, per
// (16-channel chunk, tap, tile), one unit of mask * bilinear(x) at the tap's offset position for the tile's 128 pixels, split hi / lo
// as any operand row; the consumer issues one N = G MMA chain per unit with the tap's kw block of the unchanged weight slice into
// the P0 accumulators, which move to P1 for the epilogue (no kw un-shift).  The weight stream, ring, epilogue and stores are those
// of the one-plane 2D convolution.
#include <type_traits>

#include "tc_common.cuh"

namespace osb {

struct TcgParams {
  const float* x;          // (B, D, H, W, Cin) channels-last
  const void* w;           // fp16 [3 kd][Cin/KC][3 kh][3*Cout][KC hi | KC lo]  (ops.pack_tc_weight)
  const float* scale;
  const float* shift;
  const float* residual;
  const float* gate;       // optional (B, H, W, Cout) channels-last multiplier applied after the activation: FeatureAtt's gate
                           // (NDHWC output only), or the ConvGRU's h of r * h (TcArgs::mul)
  const float* blend_z;    // optional ConvGRU blend operands (B, H, W, Cout) channels-last: y = blend_h + blend_z * (y - blend_h)
  const float* blend_h;
  long long res_bstride;   // floats between the batches of an NCDHW residual (0 = COUT * D * H * W)
  float* y;
  int B, D, H, Cin;
  int act;
  float kappa;       // expected round-towards-zero loss per accumulating MMA (tc_common.cuh)
  unsigned int* overflow;  // sticky fp16-range flag (tc_common.cuh)
  int out_ndhwc, res_ndhwc;
  int items, hblocks;      // items = (b, d, row block, column tile) x output channel groups
  int Wr, ctiles;          // general-width instantiations: image width and column tiles per row (whole-row kernels: W, 1)
  int ystride;             // channels per voxel of the channels-last y / residual / gate tensors (0 = COUT); > COUT when this launch
                           // produces a channel SLICE of a wider tensor (pointers pre-offset to the slice's first channel)
  int terms;               // split terms per product (TcArgs::terms): 3, or 1 = hi parts only (staged and multiplied)
  // modulated deformable gather (TcArgs::dcn; general-width instantiations): x is the (B, Hin, Win, Cin) input, H / Wr the output
  int dcn;
  const float* offset;
  const float* mask;
  long long off_bstride, mask_bstride;
  int Hin, Win, stride, pad, dil, cpg, mask_mode;   // cpg: input channels per deformable group
};

template <int COUT, int KC, int W, int TILES, int DIL = 1, bool GW = false>
struct TcgCfg {
  static_assert(!GW || W == 128, "general-width tiles are 128-column segments of one image row");
  // Cout = 128, dilation 1 (hidden 128 at every width): the ConvGRU epilogue (tc_common.cuh: frag_epilogue, TcArgs::gru)
  static constexpr bool GRU = COUT == 128 && DIL == 1;
  static constexpr int HALO = GW ? DIL : 0;                 // halo columns on each side of a column tile
  static constexpr int CSTEP = 128 - 2 * HALO;              // image columns a column tile produces
  // DIL = 2: dilated 2D convs of the backbone (layer4 of gwcnet_backbone.py:38-60, psmnet_backbone.py) as one-plane volumes:
  // tap kh of output row t reads input row t + (kh-1)*DIL, the kw-stacked partial sums are un-shifted by DIL columns.
  static_assert(DIL == 1 || (W == 128 && DIL == 2 && COUT >= 64), "dilation 2 is instantiated for full-width rows only");
  static constexpr int R = 128 / W;                         // image rows per M tile
  static constexpr int ROWB = KC * 4;                       // bytes per K-major operand row: [KC fp16 hi | KC fp16 lo]
  static constexpr int UNIT_BYTES = 128 * ROWB;
  static constexpr int N3 = 3 * COUT;
  static constexpr int G = 32;                              // output channels per work item
  static constexpr int NG = COUT / G;                       // channel groups
  static constexpr int NG3 = 3 * G;                         // wgmma N: the three kw blocks of one channel group
  static constexpr int B_SLICE = N3 * ROWB;                 // one kh weight slice in global memory (hi and lo halves of every row)
  static constexpr int B_SUB = NG3 * ROWB;                  // the part of it one item reads
  // Work item = NT output tiles, tile t (consumer warpgroup t) at image rows row0 + t * TS .. + R - 1.  DIL = 1: consecutive row
  // blocks, so the units of rows between the tiles feed both.  DIL = 2: rows h and h + 2, whose taps share two of their three units
  // (adjacent rows share none); row blocks then interleave, hb = 2k + j -> rows 4k + j and 4k + j + 2.
  static constexpr int NT = TC_WGS * TILES;
  static constexpr int TS = R * DIL;
  static constexpr int HSPAN = NT * TS;                     // image rows covered by DIL interleaved row blocks
  __host__ __device__ static constexpr int row0(int hb) { return (hb / DIL) * HSPAN + (hb % DIL) * R; }
  __host__ static int hblocks(int H) { return DIL * ((H + HSPAN - 1) / HSPAN); }
  // A-unit ring.  NLW loader warps (8-11) fill the units round-robin (unit u belongs to loader u mod NLW) into a ring as deep as
  // shared memory allows (at most 10 units).  Each loader warp enumerates ONLY ITS OWN units: a walk over the whole (tile, tap)
  // sequence by every warp, picking every NLW-th unit, makes that scalar control flow the bound of these kernels.
  static constexpr int NLW = 4;
  static constexpr int XCHG_FLOATS = 2 * frag_xchg_floats<G, DIL>();   // per consumer warpgroup: double-buffered seam rows
  static constexpr int FIXED_SMEM = 1024 + TC_BSLOTS * 3 * B_SUB + 1024 + TC_WGS * XCHG_FLOATS * 4 + 4 * TC_WGS * FRAG_TP_FLOATS * 4 +
                                    2 * COUT * 4;
  static constexpr int STAGES = (232448 - FIXED_SMEM) / UNIT_BYTES < 10 ? (232448 - FIXED_SMEM) / UNIT_BYTES : 10;
  static_assert(STAGES >= NLW, "the ring must hold at least one unit per loader warp");
  static constexpr int S_FIRST = -DIL;                      // unit start rows run from S_FIRST to S_LAST (block-relative)
  static constexpr int S_LAST = (NT - 1) * TS + DIL;
  static constexpr int KSTEPS = KC / 16;                    // K = 16 fp16 channels per MMA
  static constexpr int A_OFF = 0;
  static constexpr int B_OFF = A_OFF + STAGES * UNIT_BYTES;
  static constexpr int BAR_OFF = B_OFF + TC_BSLOTS * 3 * B_SUB;
  static constexpr int THREADS = TC_WG_THREADS;             // consumers 0-7 | A loaders 8-11 | weight producer 12, idle 13-15
  static constexpr size_t SMEM = 1024 + (size_t)BAR_OFF + 1024 + TC_WGS * XCHG_FLOATS * 4 + 4 * TC_WGS * FRAG_TP_FLOATS * 4 + 2 * COUT * 4;
  static_assert(SMEM <= 232448, "shared memory budget of one CTA exceeded");
  static_assert(TILES == 1, "a consumer warpgroup holds one accumulator tile");
  static_assert(DIL == 1 || R == 1, "interleaved row blocks assume one image row per tile");
  static_assert(COUT % G == 0, "output channels come in groups of 32");
  static_assert(B_SUB % 1024 == 0 && UNIT_BYTES % 1024 == 0, "operand tiles must stay 1024-byte aligned");
  // tile fed by unit s through tap kh, or -1
  static constexpr int tile_of(int s, int kh) {
    const int num = s - (kh - 1) * DIL;
    return (num >= 0 && num % TS == 0 && num / TS < NT) ? num / TS : -1;
  }
  static constexpr bool used(int s) { return tile_of(s, 0) >= 0 || tile_of(s, 1) >= 0 || tile_of(s, 2) >= 0; }
  // units of one (kd, chunk) phase in issue order: their number and the start row of the j-th one
  static constexpr int units_per_phase() {
    int n = 0;
    for (int s = S_FIRST; s <= S_LAST; ++s) n += used(s) ? 1 : 0;
    return n;
  }
  static constexpr int NU = units_per_phase();
  static constexpr int unit_s(int j) {
    int k = 0;
    for (int s = S_FIRST; s <= S_LAST; ++s)
      if (used(s)) {
        if (k == j) return s;
        ++k;
      }
    return S_LAST;
  }
};

template <int COUT, int KC, int W, int TILES, int DIL = 1, bool GW = false, bool GATE = false>
__global__ void __launch_bounds__(TcgCfg<COUT, KC, W, TILES, DIL, GW>::THREADS, 1) conv3d_tcg_kernel(const TcgParams p) {
  using C = TcgCfg<COUT, KC, W, TILES, DIL, GW>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* a_buf = smem + C::A_OFF;
  uint8_t* b_buf = smem + C::B_OFF;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::BAR_OFF);
  uint64_t* a_ready = bars;                         // [STAGES] loaders -> consumer   (32 arrivals: one warp)
  uint64_t* a_empty = a_ready + C::STAGES;          // [STAGES] consumers -> loaders  (8 arrivals: one per consumer warp)
  uint64_t* b_full = a_empty + C::STAGES;           // [2][3]   weight producer -> consumers (expect_tx + bulk-copy bytes)
  uint64_t* b_empty = b_full + TC_BSLOTS * 3;       // [2][3]   consumers -> weight producer (8 arrivals)
  float* xchg = reinterpret_cast<float*>(smem + C::BAR_OFF + 1024);   // [TC_WGS][XCHG_FLOATS]
  float* tiles = xchg + TC_WGS * C::XCHG_FLOATS;       // [8 consumer warps][FRAG_TP_FLOATS] output tiles
  float* s_scale = tiles + 4 * TC_WGS * FRAG_TP_FLOATS;
  float* s_shift = s_scale + COUT;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nchunk = p.Cin / KC;
  const int Wp = GW ? p.Wr : W;                     // image width = row pitch in voxels
  const int YS = (W < 32 && p.ystride) ? p.ystride : COUT;   // (compile-time COUT in the wide instantiations: slices exist at W' = 16 only)      // channel stride of the channels-last output / residual / gate
  const int ctiles = GW ? p.ctiles : 1;             // work item = (b, d, row block, column tile), column tile fastest
  const bool dcn = GW && p.dcn;                     // modulated deformable gather (same tiles, halo columns gathered and not stored)

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(&a_ready[s], 32);                     // one loader warp fills a unit
      mbar_init(&a_empty[s], 4 * TC_WGS);
    }
    for (int k = 0; k < TC_BSLOTS * 3; ++k) {
      mbar_init(&b_full[k], 1);
      mbar_init(&b_empty[k], 4 * TC_WGS);
    }
    fence_mbar_init();
  }
  for (int c = threadIdx.x; c < COUT; c += blockDim.x) {
    s_scale[c] = p.scale ? p.scale[c] : 1.f;
    s_shift[c] = p.shift ? p.shift[c] : 0.f;
  }
  __syncthreads();

  // ---------------------------------------------------------------------------------------------- consumer warpgroups
  // Warpgroup wg issues the wgmmas of tile wg of the item into its 128 x 96 register tile (output channels cg .. cg + 31 of all
  // three kw taps) from the units and weight slices both warpgroups read, then runs the epilogue of that tile on the accumulator
  // fragments (tc_common.cuh: frag_unshift, frag_epilogue).
  if (warp < 4 * TC_WGS) {
    setmaxnreg_inc<TC_CONSUMER_REGS>();
    const int wg = warp >> 2;
    xchg += wg * C::XCHG_FLOATS;
    const int bar_xchg = 1 + wg;                     // this warpgroup's named barrier
    const uint64_t dbase = (KC == 32) ? desc_sw128_base() : desc_sw64_base();
    constexpr uint32_t A_HALF = 64 * C::ROWB / 16;  // descriptor offset of operand rows 64..127
    const uint32_t b16 = (smem_u32(b_buf) & 0x3FFFF) >> 4;
    const int q = warp & 3;                          // warp of the warpgroup
    // The item loop, written once and entered on the (launch-uniform) mode: the gather's copy has its own MMA loop and epilogue, so
    // that its registers do not weigh on the convolution's copy, which is the code of the instantiations without the mode.
    auto items = [&](auto gather_c) {
      constexpr bool GATHER = decltype(gather_c)::value;
      uint32_t unitc = 0, phc = 0, exc = 0;
      for (int it = blockIdx.x; it < p.items; it += gridDim.x) {
        const int cg = (it % C::NG) * C::G;            // output channel group of this item
        const int it0 = it / C::NG;
        const int ct = it0 % ctiles;
        const int hb = (it0 / ctiles) % p.hblocks;
        const int d = (it0 / (ctiles * p.hblocks)) % p.D;
        const int b = it0 / (ctiles * p.hblocks * p.D);
        // Tile row m -> image row h (a tile below the image, odd H or H not a multiple of the item's rows, received its MMAs and
        // releases like any other and stores nothing) and column (general widths: halo columns and columns beyond the image are not
        // stored).  Returns whether the row is stored.
        auto tile_row = [&](int m, int& h, int& col) {
          h = C::row0(hb) + wg * C::TS + m / W;
          col = GW ? ct * C::CSTEP - C::HALO + m : m % W;
          return h < p.H && (!GW || (m >= C::HALO && m < 128 - C::HALO && col < Wp));
        };
        {
          // the residual and the gate stream from HBM / L2: pull one voxel's channel group per thread into L2 while the tile is
          // being accumulated
          int h, col;
          if (tile_row(q * 32 + lane, h, col)) {
            const ptrdiff_t vox = (((ptrdiff_t)b * p.D + d) * p.H + h) * Wp + col;
            if (p.residual && p.res_ndhwc) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.residual + vox * YS + cg));
            if (GATE && p.gate) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.gate + (((ptrdiff_t)b * p.H + h) * Wp + col) * YS + cg));
          }
        }
        float acc[2][C::NG3 / 2];
        // The MMA loop of one item, written once for both modes and entered per item on the (CTA-uniform) mode: each copy issues one
        // fixed wgmma sequence, so no code path inside the loop has to reconcile two (a per-unit branch costs a synchronising dummy wgmma
        // at every merge).  HI: single-term mode, a_hi * b_hi only.
        auto mma_item = [&](auto hi_c) {
          constexpr bool HI = decltype(hi_c)::value;
          uint32_t accum = 0;
          for (int kd = 0; kd < 3; ++kd) {
            const int din = d + kd - 1;
            if (din < 0 || din >= p.D) continue;
            for (int ch = 0; ch < nchunk; ++ch, ++phc) {
  #pragma unroll
              for (int s = C::S_FIRST; s <= C::S_LAST; ++s) {
                if (!C::used(s)) continue;
                const uint32_t slot = unitc % C::STAGES, par = (unitc / C::STAGES) & 1;
                mbar_wait(&a_ready[slot], par);
                const uint64_t da0 = dbase | (uint64_t)((smem_u32(a_buf + slot * C::UNIT_BYTES) & 0x3FFFF) >> 4);
  #pragma unroll
                for (int kh = 0; kh < 3; ++kh) {
                  if (C::tile_of(s, kh) != wg) continue;   // unit s meets slice kh for tile wg when s == wg * TS + (kh - 1) * DIL
                  const uint32_t bslot = (phc & 1) * 3 + kh;
                  mbar_wait(&b_full[bslot], (phc >> 1) & 1);
                  const uint64_t db0 = dbase | (uint64_t)(b16 + (bslot * C::B_SUB) / 16);
                  wg_fence();
  #pragma unroll
                  for (int ks = 0; ks < C::KSTEPS; ++ks) {
                    if constexpr (HI) wg_mma_hi<C::NG3>(acc, da0 + TcK<KC>::A_KSTEP * ks, A_HALF, db0 + 2 * ks, ks > 0 ? 1u : accum);
                    else wg_mma_split<C::NG3>(acc, da0 + TcK<KC>::A_KSTEP * ks, A_HALF, TcK<KC>::A_LO, db0 + 2 * ks, TcK<KC>::B_LO, ks > 0 ? 1u : accum);
                  }
                  wg_commit();
                  wg_wait_all();
                  accum = 1;
                  wg_release(&b_empty[bslot], lane);
                }
                wg_release(&a_empty[slot], lane);
                ++unitc;
              }
            }
          }
        };
        // The gather's MMA loop: per chunk, units (tap, tile) in that order, tap-major; this warpgroup multiplies its own tile's units
        // with the tap's kw block of slice kh and releases every unit.  All nine taps accumulate into the P0 registers (columns
        // 0 .. G - 1 of the 3G-wide tile: a 16-register block at the start of each half, which keeps the consumers' register
        // allocation -- an N = G chain into the P1 block spilled); they move to P1, which the epilogue reads.
        auto mma_gather = [&]() {
          uint32_t accum = 0;
          for (int ch = 0; ch < nchunk; ++ch, ++phc) {
  #pragma unroll
            for (int tap = 0; tap < 9; ++tap) {
              const int kh = tap / 3, kw = tap % 3;
  #pragma unroll
              for (int t = 0; t < C::NT; ++t) {
                const uint32_t slot = unitc % C::STAGES, par = (unitc / C::STAGES) & 1;
                mbar_wait(&a_ready[slot], par);
                if (t == wg) {
                  const uint32_t bslot = (phc & 1) * 3 + kh;
                  mbar_wait(&b_full[bslot], (phc >> 1) & 1);
                  const uint64_t da0 = dbase | (uint64_t)((smem_u32(a_buf + slot * C::UNIT_BYTES) & 0x3FFFF) >> 4);
                  const uint64_t db0 = dbase | (uint64_t)(b16 + (bslot * C::B_SUB + kw * C::G * C::ROWB) / 16);
                  wg_fence();
  #pragma unroll
                  for (int ks = 0; ks < C::KSTEPS; ++ks)
  #pragma unroll
                    for (int h = 0; h < 2; ++h) {
                      float(&p1)[C::G / 2] = *reinterpret_cast<float(*)[C::G / 2]>(&acc[h][0]);
                      const uint64_t da = da0 + TcK<KC>::A_KSTEP * ks + h * A_HALF, db = db0 + 2 * ks;
                      wgmma_f16<C::G>(p1, da + TcK<KC>::A_LO, db, ks > 0 ? 1u : accum);   // small terms first, as wg_mma_split
                      wgmma_f16<C::G>(p1, da, db + TcK<KC>::B_LO, 1);
                      wgmma_f16<C::G>(p1, da, db, 1);
                    }
                  wg_commit();
                  wg_wait_all();
                  accum = 1;
                  if (kw == 2) wg_release(&b_empty[bslot], lane);
                }
                wg_release(&a_empty[slot], lane);
                ++unitc;
              }
            }
          }
        };
        if constexpr (GATHER) {
          mma_gather();
          // n = MMAs issued into the P1 accumulators: chunks x 9 taps x k-steps x 3 split terms (tc_common.cuh: rz_kappa)
          const float corr = 1.f + p.kappa * (float)(nchunk * 9 * C::KSTEPS * 3);
  #pragma unroll
          for (int h = 0; h < 2; ++h)
  #pragma unroll
            for (int i = 0; i < C::G / 2; ++i) acc[h][C::G / 2 + i] = acc[h][i] * corr;
        } else {
          if (p.terms == 1) mma_item(std::true_type{});
          else mma_item(std::false_type{});
          // n = MMAs issued into each accumulator: kd planes x chunks x 3 kh taps x k-steps x split terms (tc_common.cuh: rz_kappa)
          const float corr = 1.f + p.kappa * (float)(((d > 0) + 1 + (d + 1 < p.D)) * nchunk * 3 * C::KSTEPS * p.terms);
          frag_unshift<C::G, DIL, W>(acc, xchg + (exc & 1) * (C::XCHG_FLOATS / 2), q, lane, corr, bar_xchg);
          ++exc;
        }
        const size_t plane = (size_t)p.D * p.H * Wp;                                 // NCDHW channel stride
        const ptrdiff_t rbs = (C::GRU && p.res_bstride) ? (ptrdiff_t)p.res_bstride : (ptrdiff_t)(COUT * plane);   // NCDHW residual batch stride
        auto rows = [&](int m, ptrdiff_t& yo, ptrdiff_t& ro, ptrdiff_t& go) {
          int h, col;
          const bool ok = tile_row(m, h, col);
          const ptrdiff_t vox = (((ptrdiff_t)b * p.D + d) * p.H + h) * Wp + col;     // NDHWC voxel index
          const ptrdiff_t sp = ((ptrdiff_t)d * p.H + h) * Wp + col;                  // offset inside an NCDHW channel plane
          yo = p.out_ndhwc ? vox * YS : (ptrdiff_t)b * COUT * plane + sp;
          ro = p.res_ndhwc ? vox * YS : (ptrdiff_t)b * rbs + sp;
          go = (((ptrdiff_t)b * p.H + h) * Wp + col) * YS;
          return ok;
        };
        frag_epilogue<C::G, C::GRU>(acc, lane, q, tiles + warp * FRAG_TP_FLOATS, s_scale + cg, s_shift + cg, p.act, p.y + (p.out_ndhwc ? (size_t)cg : cg * plane),
                            p.out_ndhwc ? 1 : plane, p.residual ? p.residual + (p.res_ndhwc ? (size_t)cg : cg * plane) : nullptr,
                            p.res_ndhwc ? 1 : plane, ((GATE || C::GRU) && p.gate) ? p.gate + cg : nullptr, rows, C::G, false, false, nullptr,
                          p.blend_z ? p.blend_z + cg : nullptr, p.blend_h ? p.blend_h + cg : nullptr);
      }
    };
    if (dcn) items(std::true_type{});
    else items(std::false_type{});
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
      // General widths: col0 = image column of load 0 (may be -HALO .. or beyond Wr: those columns are zero padding).
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
      if (p.terms == 1) {                            // the hi part alone: the single-term MMAs read nothing else
#pragma unroll
        for (int j = 0; j < NLD; ++j) stage_f16_hi<KC>(tile, v0 + VPL * j, c, v[j], amax);
      } else {
#pragma unroll
        for (int j = 0; j < NLD; ++j) stage_f16_split<KC>(tile, v0 + VPL * j, c, v[j], amax);
      }
      fence_proxy_async();
      mbar_arrive(&a_ready[slot]);
    };
    // The gather's unit (chunk ch, tap, tile t): operand row v = output pixel (row h, column col) of tile t, its 4-channel quad c of
    // chunk ch = mask * bilinear sample of x at the tap's offset position, as modulated_deformable_im2col_gpu_kernel and
    // dmcn_im2col_bilinear compute it (deform_conv_cuda_kernel.cu:468-497, 571-633): zero outside (-1, Hin) x (-1, Win), each corner
    // checked on its own.  A quad never spans two deformable groups (cpg % 4 == 0, checked by the entry point).
    auto fill_gather = [&](int b, int h, int col_first, int ch, int tap, uint32_t u) {
      const int kh = tap / 3, kw = tap % 3;
      const int cin = ch * KC + c * 4, g = cin / p.cpg;
      const size_t plane = (size_t)p.H * Wp;
      const float* off = p.offset + b * p.off_bstride + (size_t)(g * 18 + 2 * tap) * plane + (size_t)h * Wp;
      const float* msk = p.mask + b * p.mask_bstride + (size_t)(g * 9 + tap) * plane + (size_t)h * Wp;
      const float* img = p.x + (size_t)b * p.Hin * p.Win * p.Cin + cin;
      const int hb0 = h * p.stride - p.pad + kh * p.dil;
      const uint32_t slot = u % C::STAGES, ph = (u / C::STAGES) & 1;
      mbar_wait_relaxed(&a_empty[slot], ph ^ 1);
      uint8_t* tile = a_buf + slot * C::UNIT_BYTES;
#pragma unroll 4
      for (int j = 0; j < NLD; ++j) {
        const int col = col_first + VPL * j;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (h < p.H && (unsigned)col < (unsigned)Wp) {
          const float dy = __ldg(off + col), dx = __ldg(off + plane + col), ml = __ldg(msk + col);
          const float m = p.mask_mode ? 2.f * (1.f / (1.f + expf(-ml))) : ml;
          const float hi = (float)hb0 + dy, wi = (float)(col * p.stride - p.pad + kw * p.dil) + dx;
          if (hi > -1.f && wi > -1.f && hi < (float)p.Hin && wi < (float)p.Win) {
            const int hl = (int)floorf(hi), wl = (int)floorf(wi), hh = hl + 1, wh = wl + 1;
            const float lh = hi - hl, lw = wi - wl, uh = 1.f - lh, uw = 1.f - lw;
            const float w1 = uh * uw, w2 = uh * lw, w3 = lh * uw, w4 = lh * lw;
            const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
            auto at = [&](int y, int x) { return __ldg(reinterpret_cast<const float4*>(img + ((size_t)y * p.Win + x) * p.Cin)); };
            const float4 v1 = (hl >= 0 && wl >= 0) ? at(hl, wl) : z;
            const float4 v2 = (hl >= 0 && wh <= p.Win - 1) ? at(hl, wh) : z;
            const float4 v3 = (hh <= p.Hin - 1 && wl >= 0) ? at(hh, wl) : z;
            const float4 v4 = (hh <= p.Hin - 1 && wh <= p.Win - 1) ? at(hh, wh) : z;
            v.x = (w1 * v1.x + w2 * v2.x + w3 * v3.x + w4 * v4.x) * m;
            v.y = (w1 * v1.y + w2 * v2.y + w3 * v3.y + w4 * v4.y) * m;
            v.z = (w1 * v1.z + w2 * v2.z + w3 * v3.z + w4 * v4.z) * m;
            v.w = (w1 * v1.w + w2 * v2.w + w3 * v3.w + w4 * v4.w) * m;
          }
        }
        stage_f16_split<KC>(tile, v0 + VPL * j, c, v, amax);   // amax sees the modulated operand: |m| <= 2 doubles the input's range
      }
      fence_proxy_async();
      mbar_arrive(&a_ready[slot]);
    };
    if (dcn) {
      constexpr int NUG = 9 * C::NT;                 // units per chunk: (tap, tile), tap-major as the consumers take them
#pragma unroll 1
      for (int it = blockIdx.x; it < p.items; it += gridDim.x) {
        const int it0 = it / C::NG;
        const int ct = it0 % ctiles;
        const int hb = (it0 / ctiles) % p.hblocks;
        const int b = it0 / (ctiles * p.hblocks);
#pragma unroll 1
        for (int ch = 0; ch < nchunk; ++ch) {
#pragma unroll 1
          for (int j = first; j < NUG; j += C::NLW)
            fill_gather(b, C::row0(hb) + (j % C::NT) * C::TS, ct * C::CSTEP - C::HALO + v0, ch, j / C::NT, ubase + j);
          ubase += NUG;
          first = (first + C::NLW - NUG % C::NLW) % C::NLW;
        }
      }
    } else
    for (int it = blockIdx.x; it < p.items; it += gridDim.x) {
      const int it0 = it / C::NG;                    // every channel group of a tile stages the same units
      const int ct = it0 % ctiles;
      const int hb = (it0 / ctiles) % p.hblocks;
      const int d = (it0 / (ctiles * p.hblocks)) % p.D;
      const int b = it0 / (ctiles * p.hblocks * p.D);
      const int h0 = C::row0(hb);
      const int col0 = ct * C::CSTEP - C::HALO + v0;   // image column of this lane's first load (whole-row kernels: v0)
      for (int kd = 0; kd < 3; ++kd) {
        const int din = d + kd - 1;
        if (din < 0 || din >= p.D) continue;
        const float* plane = p.x + ((size_t)b * p.D + din) * p.H * (size_t)Wp * p.Cin;
        for (int ch = 0; ch < nchunk; ++ch) {
#pragma unroll 1
          for (int j = first; j < C::NU; j += C::NLW) {
            // unit = R consecutive image rows starting at h0 + s: operand row v is voxel (h0 + s) * W + v of the plane
            const int s = C::unit_s(j);
            const float* base = plane + ((ptrdiff_t)(h0 + s) * Wp + col0) * p.Cin + ch * KC + c * 4;
            fill(base, (size_t)Wp * p.Cin, (size_t)p.Cin, h0 + s, 1, ubase + j, col0);
          }
          ubase += C::NU;
          first = (first + C::NLW - C::NU % C::NLW) % C::NLW;
        }
      }
    }
    tc_report_overflow(p.overflow, amax);
  }
  // ---------------------------------------------------------------------------------------------- weight-slice producer
  // One elected lane streams the item's channel group of the pre-swizzled (kd, chunk, kh) slices -- three G-row kw blocks, 1-D
  // bulk copies -- into the two buffer sets, up to a whole phase ahead of the MMAs (tc_common.cuh: bulk_g2s).  The blocks keep
  // their row index mod 8, so the swizzle applied by the packer stays valid.  The other warps of this warpgroup are idle: they only
  // hand their registers back.
  else {
    setmaxnreg_dec<TC_PRODUCER_REGS>();
    if (warp == 4 * TC_WGS + C::NLW && elect_one()) {
      const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(p.w);
      uint32_t phc = 0;
      for (int it = blockIdx.x; it < p.items; it += gridDim.x) {
        const int cg = (it % C::NG) * C::G;
        const int d = (it / C::NG / (ctiles * p.hblocks)) % p.D;
        for (int kd = 0; kd < 3; ++kd) {
          const int din = d + kd - 1;
          if (din < 0 || din >= p.D) continue;
          for (int ch = 0; ch < nchunk; ++ch, ++phc) {
            for (int kh = 0; kh < 3; ++kh) {
              const uint32_t slot = (phc & 1) * 3 + kh;
              const size_t slice = ((size_t)kd * nchunk + ch) * 3 + kh;
              mbar_wait_relaxed(&b_empty[slot], ((phc >> 1) & 1) ^ 1);
              mbar_arrive_expect_tx(&b_full[slot], C::B_SUB);
#pragma unroll
              for (int kw = 0; kw < 3; ++kw)
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

template <int COUT, int KC, int W, int TILES, int DIL = 1, bool GW = false, bool GATE = false>
static int launch_tcg(const TcArgs& a, cudaStream_t stream) {
  using C = TcgCfg<COUT, KC, W, TILES, DIL, GW>;
  TcgParams p{};
  p.gate = a.gate ? a.gate : a.mul, p.ystride = a.ystride, p.terms = a.terms;
  p.blend_z = a.blend_z, p.blend_h = a.blend_h, p.res_bstride = a.res_bstride;
  p.hblocks = C::hblocks(a.H);
  p.Wr = GW ? a.W : W;
  p.ctiles = GW ? (a.W + C::CSTEP - 1) / C::CSTEP : 1;
  p.dcn = a.dcn, p.offset = a.dcn_offset, p.mask = a.dcn_mask, p.off_bstride = a.dcn_off_bstride, p.mask_bstride = a.dcn_mask_bstride;
  p.Hin = a.dcn_h, p.Win = a.dcn_w, p.stride = a.dcn_stride, p.pad = a.dcn_pad, p.dil = a.dcn_dil, p.mask_mode = a.dcn_mask_mode;
  p.cpg = a.Cin / a.dcn_dg;
  static const std::string variant = tc_variant_name("tcg<%d,%d,%d,%d,%d,%d,%d>", COUT, KC, W, TILES, DIL, (int)GW, (int)GATE);
  return launch_persistent<conv3d_tcg_kernel<COUT, KC, W, TILES, DIL, GW, GATE>>(
      a, p, (long long)a.B * a.D * p.hblocks * p.ctiles * C::NG, C::SMEM, variant.c_str(), stream);
}

TcLaunch select_mdconv_tc(int Cout) {
  // the general-width instantiations of select_conv3d_tc below
  if (Cout == 32) return launch_tcg<32, 16, 128, 1, 1, true>;
  if (Cout == 64) return launch_tcg<64, 16, 128, 1, 1, true>;
  if (Cout == 128) return launch_tcg<128, 16, 128, 1, 1, true>;
  return nullptr;
}

TcRoute select_conv3d_tc(int Cin, int Cout, int W, int dilation, bool gate, bool slice) {
  if (dilation == 1 && W == 128 && Cin % 32 == 0 && Cin >= 32 && !gate && !slice) {   // conv3d_tc.cu
    if (Cout == 32) return {launch_tc<32>, 32};
    if (Cout >= 1 && Cout <= 16) return {launch_tc<16>, 32};   // narrow heads: weights zero-padded to 16 rows
  }
  if (Cin % 16 != 0 || Cin < 16) return {};
  if (dilation == 2)                                            // 2D backbone stages as one-plane volumes
    return (W == 128 && Cout == 128 && !gate && !slice) ? TcRoute{launch_tcg<128, 16, 128, 1, 2>, 16} : TcRoute{};
  if (dilation != 1) return {};
  if (W == 16) {                      // StereoBase 1/32 level: 6c = 144 -> 160 channels as two slices (96 + 64), 8 image rows per tile
    if (Cout == 96) return {launch_tcg<96, 16, 16, 1, 1, false, true>, 16};
    if (Cout == 64) return {launch_tcg<64, 16, 16, 1, 1, false, true>, 16};
    return {};
  }
  if (slice) return {};                                         // channel slices are instantiated for W = 16 only
  if (gate) {
    if (W == 64 && Cout == 64) return {launch_tcg<64, 16, 64, 1, 1, false, true>, 16};   // StereoBase 1/8 level (FeatureAtt gate)
    if (W == 32 && Cout == 96) return {launch_tcg<96, 16, 32, 1, 1, false, true>, 16};   // ... 1/16 level
    return {};
  }
  if (W == 64 && Cout == 64) return {launch_tcg<64, 16, 64, 1>, 16};
  if (W == 32 && Cout == 64) return {launch_tcg<64, 16, 32, 1>, 16};
  if (W == 32 && Cout == 128) return {launch_tcg<128, 16, 32, 1>, 16};
  if (W == 32 && Cout == 96) return {launch_tcg<96, 16, 32, 1>, 16};         // StereoBase 1/16 level (4c = 96)
  if (W == 128 && Cout == 64) return {launch_tcg<64, 16, 128, 1>, 16};       // 2D backbone stages as one-plane volumes
  if (W == 128 && Cout == 128) return {launch_tcg<128, 16, 128, 1>, 16};
  if (!osb_tc_general_width(W)) return {};
  // every other width: 128-column tiles with a one-column halo
  if (Cout == 32) return {launch_tcg<32, 16, 128, 1, 1, true>, 16};
  if (Cout == 64) return {launch_tcg<64, 16, 128, 1, 1, true>, 16};
  if (Cout == 128) return {launch_tcg<128, 16, 128, 1, 1, true>, 16};
  return {};
}

}  // namespace osb
