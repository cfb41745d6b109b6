// Tensor-core (Hopper wgmma) Conv3d 3x3x3 STRIDE 2, pad 1: the down-sampling convs of the hourglasses
//   conv1 32->64 (1/4 -> 1/8 res) and conv3 64->128 / 64->64 (1/8 -> 1/16 res): gwcnet/hourglass.py:19-29,
//   psmnet/psmnet_cost_processor.py:79-94.
// Same machinery as conv3d_tcg.cu (3xFP16 split, LDG-staged swizzled operands, warp-specialised persistent CTA, one accumulator tile
// of G = 32 output channels per consumer warpgroup, taps stacked along N and recombined in the epilogue); what changes is the gather:
//   out[ow] = in[2ow-1].W0 + in[2ow].W1 + in[2ow+1].W2.  With E[j] = in[2j] (even columns) and O[j] = in[2j+1] (odd columns)
//   this is  out[ow] = E[ow].W1 + O[ow].W2 + O[ow-1].W0 ,  so per (output tile, kd, kh) the loaders stage TWO operand tiles
//   -- the even and the odd columns of the RO = 128/Wo input rows 2*oh + kh - 1 -- and the issuer runs
//   E x W1 (N = G) into accumulator columns [0,G) and O x [W0 | W2] (N = 2G) into [G, 3G); the epilogue
//   adds P1[ow] + P2[ow] + P0[ow-1] (a single left shift, zero at ow = 0 = the conv's left padding).
// Weight slices are packed with the kw order (1, 0, 2) so both MMAs read contiguous rows.
// A work item is one output tile and a PAIR of channel groups: consumer warpgroup t computes output channels (2 * pair + t) * G ..,
// from the same staged units.  Neighbouring output row blocks share at most one of their three kh input rows at stride 2, two
// channel groups of one tile share all of them, so pairing by channel group halves the units staged per output channel.  With an odd
// number of groups (Cout = 96) the second warpgroup of a tile's last item has no group: it waits for and releases every unit and
// weight slot like the other one, and issues no MMAs and stores nothing.
// GENERAL WIDTHS (GW = true, W = 128 instantiations; see conv3d_tcg.cu): an M tile is a 128-column segment of one OUTPUT row of
// runtime width Wr starting at output column ct * 127 - 1; tile column 0 is the halo that provides O[ow-1] (zero at ow = -1) and is
// not stored.
//
// Warp roles (512 threads, 1 CTA/SM, persistent; setmaxnreg moves the registers, tc_common.cuh): warps 0-7 = two consumer
// warpgroups (channel group 2 * pair and 2 * pair + 1), warps 8-11 = A-unit loaders, warp 12 = weight-slice producer, warps 13-15 idle.
#include "tc_common.cuh"

namespace osb {

struct Tcs2Params {
  const float* x;          // (B, D, H, W, Cin) channels-last
  const void* w;           // fp16 [3 kd][Cin/KC][3 kh][3*Cout][KC hi | KC lo]  (ops.pack_tc_weight)
  const float* scale;
  const float* shift;
  const float* residual;
  float* y;
  int B, D, H, Cin;        // INPUT extent D x H x (2*WO); output is Do x H/2 x WO
  int Do;                  // D/2, or 1 for D = 1 (a one-plane 2D conv: only the kd = 1 taps meet the input)
  int act;
  float kappa;       // expected round-towards-zero loss per accumulating MMA (tc_common.cuh)
  unsigned int* overflow;  // sticky fp16-range flag (tc_common.cuh)
  int out_ndhwc, res_ndhwc;
  int items, hblocks;
  int Wr, ctiles;          // general-width instantiations: OUTPUT width and column tiles per row (whole-row kernels: W, 1)
  int ystride;             // channels per voxel of the channels-last y / residual (0 = COUT); > COUT: this launch writes a channel slice
};

template <int COUT, int KC, int W, int TILES, bool GW = false>     // W = OUTPUT width
struct Tcs2Cfg {
  static_assert(!GW || W == 128, "general-width tiles are 128-column segments of one output row");
  static constexpr int HALO = GW ? 1 : 0;                   // halo columns on the LEFT of a column tile
  static constexpr int CSTEP = 128 - HALO;                  // output columns a column tile produces
  static constexpr int R = 128 / W;                         // OUTPUT image rows per M tile
  static constexpr int ROWB = KC * 4;                       // bytes per K-major operand row: [KC fp16 hi | KC fp16 lo]
  static constexpr int UNIT_BYTES = 128 * ROWB;
  static constexpr int N3 = 3 * COUT;
  static constexpr int G = 32;                              // output channels per consumer warpgroup
  static constexpr int NG = COUT / G;                       // channel groups
  static constexpr int NP = (NG + TC_WGS - 1) / TC_WGS;     // channel-group pairs = work items per output tile
  static constexpr int B_SLICE = N3 * ROWB;                 // one kh weight slice in global memory (hi and lo halves of every row)
  static constexpr int B_SUB = 3 * G * ROWB;                // the part of it one channel group reads: [W1 | W0 | W2]
  static constexpr int B_SLOT = TC_WGS * B_SUB;             // one weight buffer: the B_SUB blocks of both groups of a pair
  // Staged accumulator tile per warpgroup: [P1 | P0 | P2] of PC output channels per pass.  Two [128][3G + 4] tiles do not fit next to
  // a full ring and the doubled weight slots, so the epilogue stages its 3G accumulator columns in two passes of 16 channels.
  static constexpr int PC = 16;
  static constexpr int NPASS = G / PC;
  static constexpr int LD = 3 * PC + 4;                     // floats per row of a staged accumulator tile
  static constexpr int XCHG_FLOATS = 2 * 4 * PC;            // per consumer warpgroup: [2 buffers][4 quadrants][PC]
  // A-unit ring.  NLW loader warps (8-11) fill the units round-robin (unit u belongs to loader u mod NLW) into a ring as deep as
  // shared memory allows (at most 10 units).  Each loader warp enumerates ONLY ITS OWN units: a walk over the whole (tile, tap)
  // sequence by every warp, picking every NLW-th unit, makes that scalar control flow the bound of these kernels.
  static constexpr int NLW = 4;
  static constexpr int FIXED_SMEM = 1024 + TC_BSLOTS * 3 * B_SLOT + TC_WGS * 128 * LD * 4 + 1024 + TC_WGS * XCHG_FLOATS * 4 + 3 * COUT * 4;
  static constexpr int STAGES = (232448 - FIXED_SMEM) / UNIT_BYTES < 10 ? (232448 - FIXED_SMEM) / UNIT_BYTES : 10;
  static_assert(STAGES >= NLW, "the ring must hold at least one unit per loader warp");
  static constexpr int NU = TILES * 3 * 2;                   // units of one (kd, chunk) phase: (tile, kh, column parity)
  static constexpr int HBLK = TILES * R;                    // output rows per work item
  static constexpr int KSTEPS = KC / 16;                    // K = 16 fp16 channels per MMA
  static constexpr int A_OFF = 0;
  static constexpr int B_OFF = A_OFF + STAGES * UNIT_BYTES;
  static constexpr int STAGE_OFF = B_OFF + TC_BSLOTS * 3 * B_SLOT;   // [TC_WGS][128][LD] fp32 accumulator tiles
  static constexpr int BAR_OFF = STAGE_OFF + TC_WGS * 128 * LD * 4;
  static constexpr int THREADS = TC_WG_THREADS;             // consumers 0-7 | A loaders 8-11 | weight producer 12, idle 13-15
  static constexpr size_t SMEM = 1024 + (size_t)BAR_OFF + 1024 + TC_WGS * XCHG_FLOATS * 4 + 3 * COUT * 4;
  static_assert(SMEM <= 232448, "shared memory budget of one CTA exceeded");
  static_assert(TILES == 1, "a consumer warpgroup holds one accumulator tile");
  static_assert(COUT % G == 0, "output channels come in groups of 32");
  static_assert(32 * LD >= TP_WARP_FLOATS, "store_ndhwc_chunk32 transposes through the warp's own rows of the staging tile");
  static_assert(B_SUB % 1024 == 0 && UNIT_BYTES % 1024 == 0, "operand tiles must stay 1024-byte aligned");
};

// Accumulator columns [C0, C0 + 16) of a finished 128 x N tile into staged columns [dst, dst + 16) of a [128][ld] tile.  Fragment
// layout as in wg_stage (tc_common.cuh): register 4j + r holds column 8j + 2(l%4) + r%2.  C0 must be a compile-time constant after
// unrolling (it indexes the accumulator registers).
template <int N>
__device__ __forceinline__ void s2_stage16(float* stage, int ld, const float (&acc)[2][N / 2], int c0, int dst, int wq, int lane) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float* r0 = stage + (64 * h + 16 * wq + (lane >> 2)) * ld + 2 * (lane & 3) + dst;
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
      const int j = c0 / 8 + jj;
      *reinterpret_cast<float2*>(r0 + 8 * jj) = make_float2(acc[h][4 * j], acc[h][4 * j + 1]);
      *reinterpret_cast<float2*>(r0 + 8 * ld + 8 * jj) = make_float2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
    }
  }
}

template <int COUT, int KC, int W, int TILES, bool GW = false>
__global__ void __launch_bounds__(Tcs2Cfg<COUT, KC, W, TILES, GW>::THREADS, 1) conv3d_tcs2_kernel(const Tcs2Params p) {
  using C = Tcs2Cfg<COUT, KC, W, TILES, GW>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte aligned; offsetting smem_raw itself keeps every derived pointer in the shared window (LDS/STS, see conv3d_tc.cu)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* a_buf = smem + C::A_OFF;
  uint8_t* b_buf = smem + C::B_OFF;
  float* stage = reinterpret_cast<float*>(smem + C::STAGE_OFF);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::BAR_OFF);
  uint64_t* a_ready = bars;                         // [STAGES] loaders -> consumers  (32 arrivals: one warp)
  uint64_t* a_empty = a_ready + C::STAGES;          // [STAGES] consumers -> loaders  (8 arrivals: one per consumer warp)
  uint64_t* b_full = a_empty + C::STAGES;           // [2][3]   weight producer -> consumers (expect_tx + bulk-copy bytes)
  uint64_t* b_empty = b_full + TC_BSLOTS * 3;       // [2][3]   consumers -> weight producer (8 arrivals)
  float* xchg = reinterpret_cast<float*>(smem + C::BAR_OFF + 1024);   // [TC_WGS][XCHG_FLOATS]
  float* s_scale = xchg + TC_WGS * C::XCHG_FLOATS;
  float* s_shift = s_scale + COUT;
  float* zeros = s_shift + COUT;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nchunk = p.Cin / KC;
  const int Wp = GW ? p.Wr : W;                     // OUTPUT width (the input is 2 * Wp wide)
  const int YS = (W < 32 && p.ystride) ? p.ystride : COUT;   // (compile-time COUT in the wide instantiations: slices exist at W' = 16 only)      // channel stride of the channels-last output / residual
  const int ctiles = GW ? p.ctiles : 1;             // work item = (b, od, row block, column tile, channel-group pair), pair fastest

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
    zeros[c] = 0.f;
  }
  __syncthreads();

  // ---------------------------------------------------------------------------------------------- consumer warpgroups
  // Warpgroup wg issues the wgmmas of channel group 2 * pair + wg -- E x W1 (N = G) and O x [W0 | W2] (N = 2G) -- into its 128-row
  // register tile from the units and weight slots both warpgroups read, then runs the epilogue of that tile.
  if (warp < 4 * TC_WGS) {
    setmaxnreg_inc<TC_CONSUMER_REGS>();
    const int wg = warp >> 2;
    stage += wg * 128 * C::LD;
    xchg += wg * C::XCHG_FLOATS;
    const int bar_stage = 1 + 2 * wg, bar_xchg = 2 + 2 * wg;   // this warpgroup's named barriers
    const uint64_t dbase = (KC == 32) ? desc_sw128_base() : desc_sw64_base();
    constexpr uint32_t A_HALF = 64 * C::ROWB / 16;  // descriptor offset of operand rows 64..127
    const uint32_t b16 = (smem_u32(b_buf) & 0x3FFFF) >> 4;
    const int Do = p.Do, Ho = p.H / 2;
    const int q = warp & 3;                          // epilogue: this warp owns tile rows 32q .. 32q + 31
    const int m = q * 32 + lane;                     // operand row owned by this thread
    const int rr = m / W, wcol = m % W;              // image row inside the tile, image column
    const bool has_left_q = ((q * 32) % W) != 0;     // the quadrant to the left continues the same image row
    uint32_t unitc = 0, phc = 0, exc = 0;
    for (int it = blockIdx.x; it < p.items; it += gridDim.x) {
      const int g = (it % C::NP) * TC_WGS + wg;      // output channel group of this warpgroup's tile
      const bool has_group = g < C::NG;              // false: the second warpgroup of the last pair of an odd NG (warpgroup-uniform)
      const int cg = g * C::G;
      const int it0 = it / C::NP;
      const int ct = it0 % ctiles;
      const int hb = (it0 / ctiles) % p.hblocks;
      const int d = (it0 / (ctiles * p.hblocks)) % Do;
      const int b = it0 / (ctiles * p.hblocks * Do);
      float acc_e[2][C::G / 2], acc_o[2][C::G];     // accumulator columns [P1 | P0 | P2]
      uint32_t accum_e = 0, accum_o = 0;
      for (int kd = 0; kd < 3; ++kd) {
        const int din = 2 * d + kd - 1;
        if (din < 0 || din >= p.D) continue;
        for (int ch = 0; ch < nchunk; ++ch, ++phc) {
#pragma unroll
          for (int kh = 0; kh < 3; ++kh) {
            const uint32_t bslot = (phc & 1) * 3 + kh;
#pragma unroll
            for (int par = 0; par < 2; ++par) {       // par 0: even input columns (kw = 1); par 1: odd columns (kw = 0, 2)
              // Both warpgroups wait for every unit and weight slot before releasing it, the one without a group included, so
              // neither can arrive on a later phase of a slot than the one being filled.
              const uint32_t slot = unitc % C::STAGES, ph = (unitc / C::STAGES) & 1;
              mbar_wait(&a_ready[slot], ph);
              if (par == 0) mbar_wait(&b_full[bslot], (phc >> 1) & 1);   // first use of slice kh in this phase
              if (has_group) {
                const uint64_t da0 = dbase | (uint64_t)((smem_u32(a_buf + slot * C::UNIT_BYTES) & 0x3FFFF) >> 4);
                // this group's block of the slot, rows [W1 (G) | W0 (G) | W2 (G)]
                const uint64_t db0 = dbase | (uint64_t)(b16 + (bslot * C::B_SLOT + wg * C::B_SUB + (par ? C::G * C::ROWB : 0)) / 16);
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < C::KSTEPS; ++ks) {
                  if (par == 0) wg_mma_split<C::G>(acc_e, da0 + TcK<KC>::A_KSTEP * ks, A_HALF, TcK<KC>::A_LO, db0 + 2 * ks, TcK<KC>::B_LO, ks > 0 ? 1u : accum_e);
                  else wg_mma_split<2 * C::G>(acc_o, da0 + TcK<KC>::A_KSTEP * ks, A_HALF, TcK<KC>::A_LO, db0 + 2 * ks, TcK<KC>::B_LO, ks > 0 ? 1u : accum_o);
                }
                wg_commit();
                wg_wait_all();
                if (par == 0) accum_e = 1;
                else accum_o = 1;
              }
              wg_release(&a_empty[slot], lane);
              if (par == 1) wg_release(&b_empty[bslot], lane);          // last use of slice kh in this phase
              ++unitc;
            }
          }
        }
      }
      if (!has_group) continue;                      // warpgroup-uniform; the epilogue's barriers are this warpgroup's own
      const int h = hb * C::HBLK + rr;               // output row of this thread's voxel
      const bool live = h < Ho;
      // general widths: output column of this thread's tile column; the halo column and columns beyond the image are not stored
      const int col = GW ? ct * C::CSTEP - C::HALO + m : wcol;
      const bool cvalid = !GW || (m >= C::HALO && col < Wp);
      const uint32_t vmask = GW ? __ballot_sync(0xffffffffu, cvalid) : 0xffffffffu;
      // input planes 2d-1, 2d, 2d+1: the first is missing for d = 0 (tc_common.cuh: rz_kappa)
      const float corr = 1.f + p.kappa * (float)(((d > 0) + 1 + (2 * d + 1 < p.D)) * nchunk * 3 * C::KSTEPS * 3);
      const ptrdiff_t vox = (((ptrdiff_t)b * Do + d) * Ho + h) * Wp + col;       // NDHWC voxel index (output)
      const size_t plane = (size_t)Do * Ho * Wp;                                 // NCDHW channel stride (output)
      const ptrdiff_t ncdhw0 = (ptrdiff_t)b * COUT * plane + ((ptrdiff_t)d * Ho + h) * Wp + col;
      float out[32];
#pragma unroll
      for (int pass = 0; pass < C::NPASS; ++pass) {
        named_bar_sync(bar_stage, 128);              // every warp is done with the rows staged before (previous pass or tile)
        s2_stage16<C::G>(stage, C::LD, acc_e, pass * C::PC, 0, q, lane);                  // P1 (kw = 1, even columns)
        s2_stage16<2 * C::G>(stage, C::LD, acc_o, pass * C::PC, C::PC, q, lane);          // P0 (kw = 0)
        s2_stage16<2 * C::G>(stage, C::LD, acc_o, C::G + pass * C::PC, 2 * C::PC, q, lane);   // P2 (kw = 2)
        named_bar_sync(bar_stage, 128);
        const float* srow = stage + m * C::LD;       // [P1 | P0 | P2] of this pass's channels
        float* xb = xchg + (exc & 1) * (4 * C::PC);
        ++exc;
        if (lane == 31) {                            // P0 of this quadrant's last column
#pragma unroll
          for (int i = 0; i < C::PC; i += 4)
            *reinterpret_cast<float4*>(xb + q * C::PC + i) = *reinterpret_cast<const float4*>(srow + C::PC + i);
        }
        named_bar_sync(bar_xchg, 128);
        const float* xl = has_left_q ? xb + (q - 1) * C::PC : zeros;
#pragma unroll
        for (int i0 = 0; i0 < C::PC; i0 += 4) {      // neighbour values loaded unconditionally, merged with selects (no branches)
          const float4 l4 = *reinterpret_cast<const float4*>(xl + i0);
          const float4 p14 = *reinterpret_cast<const float4*>(srow + i0);
          const float4 p04 = *reinterpret_cast<const float4*>(srow + C::PC + i0);
          const float4 p24 = *reinterpret_cast<const float4*>(srow + 2 * C::PC + i0);
          const float le[4] = {l4.x, l4.y, l4.z, l4.w};
          const float p0[4] = {p04.x, p04.y, p04.z, p04.w}, p1[4] = {p14.x, p14.y, p14.z, p14.w}, p2[4] = {p24.x, p24.y, p24.z, p24.w};
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            float left = __shfl_up_sync(0xffffffffu, p0[k], 1);   // P0 of output column ow-1
            left = (lane == 0) ? le[k] : left;                    // zero at ow = 0 (left padding)
            if (W < 32) left = (wcol == 0) ? 0.f : left;          // row seams inside the warp
            out[pass * C::PC + i0 + k] = ((left + p1[k]) + p2[k]) * corr;
          }
        }
      }
      const uint32_t vm = (W < 32) ? __ballot_sync(0xffffffffu, live) : (live ? vmask : 0u);   // voxels of this warp that exist
      if (vm && p.out_ndhwc && (!p.residual || p.res_ndhwc)) {     // coalesced channels-last path (BN/residual/act inside)
        store_ndhwc_chunk32(stage + q * 32 * C::LD, lane, out, p.y + (vox - lane) * YS + cg,
                            p.residual ? p.residual + (vox - lane) * YS + cg : nullptr, YS, s_scale + cg, s_shift + cg, p.act, vm);
      } else if (live && cvalid) {
#pragma unroll
        for (int i = 0; i < 32; ++i) out[i] = fmaf(out[i], s_scale[cg + i], s_shift[cg + i]);
        if (p.residual) {
          if (p.res_ndhwc) {
            const float4* rp = reinterpret_cast<const float4*>(p.residual + vox * YS + cg);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float4 rv = __ldg(rp + i);
              out[4 * i] += rv.x, out[4 * i + 1] += rv.y, out[4 * i + 2] += rv.z, out[4 * i + 3] += rv.w;
            }
          } else {
#pragma unroll
            for (int i = 0; i < 32; ++i) out[i] += __ldg(p.residual + ncdhw0 + (size_t)(cg + i) * plane);
          }
        }
        if (p.act == OSB_ACT_RELU) {
#pragma unroll
          for (int i = 0; i < 32; ++i) out[i] = fmaxf(out[i], 0.f);
        } else if (p.act == OSB_ACT_LEAKY) {
#pragma unroll
          for (int i = 0; i < 32; ++i) out[i] = out[i] > 0.f ? out[i] : 0.01f * out[i];
        }
        if (p.out_ndhwc) {
          float4* yp = reinterpret_cast<float4*>(p.y + vox * YS + cg);
#pragma unroll
          for (int i = 0; i < 8; ++i) yp[i] = make_float4(out[4 * i], out[4 * i + 1], out[4 * i + 2], out[4 * i + 3]);
        } else {
#pragma unroll
          for (int i = 0; i < 32; ++i) p.y[ncdhw0 + (size_t)(cg + i) * plane] = out[i];
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
    const int WI = 2 * Wp;                           // input width
    const int Do = p.Do;
    uint32_t ubase = 0;                              // global index of the current phase's first unit
    int first = lw;                                  // this warp's first local unit index in the current phase: (ubase + first) % NLW == lw
    auto fill = [&](const float* base, size_t rstride, size_t cstride, int h_first, int h_step, uint32_t u, int col0) {
      // base: this lane's address for load 0; load j covers operand rows VPL*j .. VPL*j + VPL - 1 = columns (VPL*j) % W ..
      // of tile row (VPL*j) / W, read from image row h_first + h_step * tile row (rstride / cstride floats per tile row / column).
      // General widths: col0 = OUTPUT column of load 0 (-1 = the left halo; columns outside [0, Wp) are zero padding).
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
      const int it0 = it / C::NP;                    // every channel-group pair of a tile stages the same units
      const int ct = it0 % ctiles;
      const int hb = (it0 / ctiles) % p.hblocks;
      const int od = (it0 / (ctiles * p.hblocks)) % Do;
      const int b = it0 / (ctiles * p.hblocks * Do);
      const int h0 = hb * C::HBLK;                   // first OUTPUT row of the block
      const int col0 = ct * C::CSTEP - C::HALO + v0; // OUTPUT column of this lane's first load (whole-row kernels: v0)
      for (int kd = 0; kd < 3; ++kd) {
        const int din = 2 * od + kd - 1;
        if (din < 0 || din >= p.D) continue;
        const float* plane = p.x + ((size_t)b * p.D + din) * p.H * (size_t)WI * p.Cin;
        for (int ch = 0; ch < nchunk; ++ch) {
#pragma unroll 1
          for (int j = first; j < C::NU; j += C::NLW) {       // local unit index = (t * 3 + kh) * 2 + par
            const int t = j / 6, kh = (j >> 1) % 3, par = j & 1;
            // operand row v = output voxel (row h0 + t*R + v / W, column v % W) reading input (2*row + kh - 1, 2*col + par)
            const int h_first = 2 * (h0 + t * C::R) + kh - 1;
            const float* base = plane + ((ptrdiff_t)h_first * WI + 2 * col0 + par) * p.Cin + ch * KC + c * 4;
            fill(base, (size_t)2 * WI * p.Cin, (size_t)2 * p.Cin, h_first, 2, ubase + j, col0);
          }
          ubase += C::NU;
          first = (first + C::NLW - C::NU % C::NLW) % C::NLW;
        }
      }
    }
    tc_report_overflow(p.overflow, amax);
  }
  // ---------------------------------------------------------------------------------------------- weight-slice producer
  // One elected lane streams the item's channel groups of the pre-swizzled (kd, chunk, kh) slices -- per group three G-row blocks
  // [W1 | W0 | W2], 1-D bulk copies -- into the two buffer sets, up to a whole phase ahead of the MMAs (tc_common.cuh: bulk_g2s).
  // The last pair of an odd NG has one group: one block, and expect_tx counts only its bytes.  The other warps of this warpgroup
  // are idle: they only hand their registers back.
  else {
    setmaxnreg_dec<TC_PRODUCER_REGS>();
    if (warp == 4 * TC_WGS + C::NLW && elect_one()) {
      const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(p.w);
      uint32_t phc = 0;
      for (int it = blockIdx.x; it < p.items; it += gridDim.x) {
        const int g0 = (it % C::NP) * TC_WGS;        // first channel group of the pair
        const int ngr = min(TC_WGS, C::NG - g0);     // groups in the pair
        const int od = (it / C::NP / (ctiles * p.hblocks)) % p.Do;
        for (int kd = 0; kd < 3; ++kd) {
          const int din = 2 * od + kd - 1;              // must enumerate the same phases as the consumers and the loaders
          if (din < 0 || din >= p.D) continue;
          for (int ch = 0; ch < nchunk; ++ch, ++phc) {
            for (int kh = 0; kh < 3; ++kh) {
              const uint32_t slot = (phc & 1) * 3 + kh;
              const size_t slice = ((size_t)kd * nchunk + ch) * 3 + kh;
              mbar_wait_relaxed(&b_empty[slot], ((phc >> 1) & 1) ^ 1);
              mbar_arrive_expect_tx(&b_full[slot], ngr * C::B_SUB);
              for (int t = 0; t < ngr; ++t)
#pragma unroll
                for (int kw = 0; kw < 3; ++kw)
                  bulk_g2s(b_buf + slot * C::B_SLOT + t * C::B_SUB + kw * C::G * C::ROWB,
                           wsrc + slice * C::B_SLICE + (size_t)(kw * COUT + (g0 + t) * C::G) * C::ROWB, C::G * C::ROWB, &b_full[slot]);
            }
          }
        }
      }
    }
    __syncwarp();
  }
}

template <int COUT, int KC, int W, int TILES, bool GW = false>
static int launch_tcs2(const TcArgs& a, cudaStream_t stream) {
  using C = Tcs2Cfg<COUT, KC, W, TILES, GW>;
  Tcs2Params p{};
  p.ystride = a.ystride;
  p.Do = a.D == 1 ? 1 : a.D / 2;
  p.hblocks = (a.H / 2 + C::HBLK - 1) / C::HBLK;
  p.Wr = GW ? a.W / 2 : W;
  p.ctiles = GW ? (p.Wr + C::CSTEP - 1) / C::CSTEP : 1;
  static const std::string variant = tc_variant_name("tcs2<%d,%d,%d,%d,%d>", COUT, KC, W, TILES, (int)GW);
  return launch_persistent<conv3d_tcs2_kernel<COUT, KC, W, TILES, GW>>(   // two channel groups per item
      a, p, (long long)a.B * p.Do * p.hblocks * p.ctiles * C::NP, C::SMEM, variant.c_str(), stream);
}

// The instantiation that serves a stride-2 shape (INPUT extents; template W = output width), writing a channel slice; null when
// there is none.  D = 1 is a one-plane 2D conv (the backbone's stride-2 stage entry): one output plane from the kd = 1 taps.
static TcLaunch select_conv3d_s2_tc(int Cin, int Cout, int D, int H, int W, bool slice) {
  if (Cin % 16 != 0 || Cin < 16 || (D % 2 && D != 1) || H % 2 || W % 2) return nullptr;
  if (W == 32 && Cout == 96) return launch_tcs2<96, 16, 16, 1>;       // StereoBase conv3[0]: 4c -> 6c as two channel slices
  if (W == 32 && Cout == 64) return launch_tcs2<64, 16, 16, 1>;
  if (slice) return nullptr;                                           // channel slices are instantiated for W = 16 only
  if (W == 128 && Cout == 64) return launch_tcs2<64, 16, 64, 1>;
  if (W == 64 && Cout == 64) return launch_tcs2<64, 16, 32, 1>;
  if (W == 64 && Cout == 128) return launch_tcs2<128, 16, 32, 1>;
  if (W == 64 && Cout == 96) return launch_tcs2<96, 16, 32, 1>;       // StereoBase conv2[0]: 2c -> 4c = 96
  if (!osb_tc_general_width(W / 2)) return nullptr;
  if (Cout == 64) return launch_tcs2<64, 16, 128, 1, true>;           // 128-column tiles of the OUTPUT row
  if (Cout == 128) return launch_tcs2<128, 16, 128, 1, true>;
  return nullptr;
}

static int conv3d_k3_s2_tc_impl(TcArgs a, cudaStream_t stream) {
  OSB_REQUIRE(select_conv3d_s2_tc(a.Cin, a.Cout, a.D, a.H, a.W, false), "conv3d_k3_s2_tc: unsupported shape Cin=%d Cout=%d D=%d H=%d W=%d",
              a.Cin, a.Cout, a.D, a.H, a.W);
  const TcLaunch launch = select_conv3d_s2_tc(a.Cin, a.Cout, a.D, a.H, a.W, a.slice());
  const int rc = check_tc_args("conv3d_k3_s2_tc", a, launch);
  return rc != OSB_OK ? rc : launch(a, stream);
}

}  // namespace osb

extern "C" {

int osb_conv3d_s2_tc_supported(int Cin, int Cout, int D, int H, int W) {
  return osb::select_conv3d_s2_tc(Cin, Cout, D, H, W, false) ? 1 : 0;
}

int osb_conv3d_k3_s2_tc_fwd(const float* x_ndhwc, const void* w_split, const float* scale, const float* shift,
                            const float* residual, float* y, int B, int Cin, int Cout, int D, int H, int W, int act,
                            int out_ndhwc, int res_ndhwc, osb_stream_t stream) {
  return osb::conv3d_k3_s2_tc_impl({x_ndhwc, w_split, scale, shift, residual, nullptr, y, B, Cin, Cout, D, H, W, act, out_ndhwc, res_ndhwc,
                                    0, 0, Cout}, (cudaStream_t)stream);
}

int osb_conv3d_k3_s2_tc_cs_fwd(const float* x_ndhwc, const void* w_split, const float* scale, const float* shift, float* y, int B,
                               int Cin, int Cout, int D, int H, int W, int act, int ystride, osb_stream_t stream) {
  return osb::conv3d_k3_s2_tc_impl({x_ndhwc, w_split, scale, shift, nullptr, nullptr, y, B, Cin, Cout, D, H, W, act, 1, 1, 0, ystride,
                                    Cout}, (cudaStream_t)stream);
}
}
