// Shared device helpers of the Hopper (wgmma) convolution kernels (conv3d_tc.cu: W = 128 specialisation; conv3d_tcg.cu: generic
// multi-row tiles; conv3d_tcs2.cu, conv3d_tcdc.cu).  See conv3d_tc.cu for the design notes.
#pragma once
#include "common.cuh"

namespace osb {

// ------------------------------------------------------------------------------------------------ small PTX wrappers
// Wait used by the helper roles (loaders, weight producer): they run AHEAD of the consumer warpgroup and would otherwise burn
// issue slots of the shared schedulers in a tight try_wait loop; back off between probes.
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  for (;;) {
    asm volatile(
        "{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (done) return;
    __nanosleep(64);
  }
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// K-major, SWIZZLE_128B wgmma shared-memory matrix descriptor: 8-row atoms of 1024 bytes (SBO), start address 0.
__device__ __forceinline__ uint64_t desc_sw128_base() {
  uint64_t d = 0;
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// K-major SWIZZLE_64B descriptor base (64-byte rows, 512-byte 8-row atoms)
__device__ __forceinline__ uint64_t desc_sw64_base() {
  uint64_t d = 0;
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(512 >> 4) << 32;
  d |= (uint64_t)2 << 62;
  return d;
}

// ------------------------------------------------------------------------------------------------ wgmma
// D (64 x N, fp32, registers of the issuing warpgroup) (+)= A (64 x 16 fp16, K-major, shared) * B (N x 16 fp16, K-major, shared)^T.
// `accumulate` = 0 overwrites D.  Every thread of the warpgroup executes it (warpgroup-uniform control flow).
template <int N>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate);
template <>
__device__ __forceinline__ void wgmma_f16<32>(float (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}

template <>
__device__ __forceinline__ void wgmma_f16<48>(float (&d)[24], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %26, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}

template <>
__device__ __forceinline__ void wgmma_f16<64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}

template <>
__device__ __forceinline__ void wgmma_f16<96>(float (&d)[48], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %50, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}

template <>
__device__ __forceinline__ void wgmma_f16<128>(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// One K = 16 step of the 3xFP16 product (below) into a 128-row accumulator tile held as two m64 halves: half h reads operand rows
// 64h .. 64h + 63 (a_half = their descriptor offset in 16-byte units), a_lo / b_lo = descriptor offset of the lo half of the k-step
// in an A / B row (they differ for 32-channel rows: A rows are split granules, B rows [32 hi | 32 lo], see TcK).
template <int N>
__device__ __forceinline__ void wg_mma_split(float (&acc)[2][N / 2], uint64_t da, uint32_t a_half, uint32_t a_lo, uint64_t db,
                                             uint32_t b_lo, uint32_t accumulate) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    wgmma_f16<N>(acc[h], da + h * a_half + a_lo, db, accumulate);   // small terms first
    wgmma_f16<N>(acc[h], da + h * a_half, db + b_lo, 1);
    wgmma_f16<N>(acc[h], da + h * a_half, db, 1);
  }
}
// Consumer-side release of a ring slot / weight buffer read by the wgmmas just waited for: one arrival per consumer warp (barrier
// count 4 x consumer warpgroups).  With two consumer warpgroups, each releases every slot it is handed, including the ones its own
// tile does not read, and only after waiting for that slot's fill, so neither can arrive on a later phase than the one being filled.
__device__ __forceinline__ void wg_release(uint64_t* bar, int lane) {
  if (lane == 0) mbar_arrive(bar);
}
// Accumulator fragment of wgmma m64nN (f32): register 4j + r of lane l in warp w of the warpgroup holds row 16w + l/4 + 8(r/2),
// column 8j + 2(l%4) + r%2.  The epilogues of conv3d_tcs2.cu / conv3d_tcdc.cu own one voxel (tile row) per thread, so their finished
// tiles go through shared memory:
// `stage` is [128 rows][ld floats], ld = N + 4 (rows 16 B apart in bank space: the per-row LDS.128 of a warp are conflict-free).
template <int N>
__device__ __forceinline__ void wg_stage(float* stage, int ld, const float (&acc)[2][N / 2], int wq, int lane) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float* r0 = stage + (64 * h + 16 * wq + (lane >> 2)) * ld + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
      *reinterpret_cast<float2*>(r0 + 8 * j) = make_float2(acc[h][4 * j], acc[h][4 * j + 1]);
      *reinterpret_cast<float2*>(r0 + 8 * ld + 8 * j) = make_float2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
    }
  }
}
// 16 consecutive staged accumulator columns of one tile row
__device__ __forceinline__ void stage_ld16(const float* row, uint32_t* r) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 v = reinterpret_cast<const float4*>(row)[i];
    r[4 * i] = __float_as_uint(v.x), r[4 * i + 1] = __float_as_uint(v.y), r[4 * i + 2] = __float_as_uint(v.z), r[4 * i + 3] = __float_as_uint(v.w);
  }
}

// 1-D bulk copy global -> shared through the TMA engine (SASS UBLKCP), completion counted in bytes on an mbarrier.  The weight
// slices are stored PRE-SWIZZLED in global memory (ops.pack_tc_weight), so one elected thread can stream them with no register
// staging, any number of slices in flight, where LDG/STS weight loaders would expose one full L2 round trip per slice.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// 16-byte asynchronous copy global -> shared (LDGSTS) with zero fill when !valid: the A-unit loaders keep several units of raw
// fp32 rows in flight per warp WITHOUT holding them in registers (each lane later reads back exactly the bytes it copied, so no
// cross-lane synchronisation beyond cp.async.wait_group is needed).
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
  const uint32_t n = valid ? 16u : 0u;
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(n) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
constexpr int TC_BSLOTS = 2;       // weight-slice buffers per kh tap: the producer runs one (kd, chunk) phase ahead of the MMAs
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int threads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
// Warp roles of the stride-1 kernels (conv3d_tc.cu, conv3d_tcg.cu): 512 threads = two consumer warpgroups (one 128 x 3G
// accumulator tile each) | one warpgroup of A loaders | one warpgroup of bulk-copy producers (single elected lanes) and idle warps.
// The CTA starts at 128 registers per thread; setmaxnreg moves them to the consumers: 2 x 128 x 184 + 128 x 112 + 128 x 32 = 65536.
constexpr int TC_WGS = 2;                 // consumer warpgroups per CTA: each owns one output tile of a work item
constexpr int TC_CONSUMER_REGS = 184;
constexpr int TC_LOADER_REGS = 112;
constexpr int TC_PRODUCER_REGS = 32;
constexpr int TC_WG_THREADS = 512;
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
// One lane of a fully converged warp (control flow stays warp-uniform; only the bulk-copy issue is predicated on the elected lane).
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n.reg .pred p;\nelect.sync _|p, 0xffffffff;\nselp.u32 %0, 1, 0, p;\n}\n" : "=r"(pred));
  return pred != 0;
}
// 3xFP16 operand split (fp32-accurate products on the 16-bit tensor-core rate).
//   x * s  =  hi + lo + r,   hi = fp16_rn(x*s),  lo = fp16_rn(x*s - hi),   |r| <= max(2^-22 |x*s|, 2^-25)
// and every product is issued as  a_lo*b_hi + a_hi*b_lo + a_hi*b_hi  on wgmma (fp16 operands) with fp32 accumulation in registers
// (the dropped lo*lo term is <= 2^-22 of the product; both roundings are to nearest, so the residual is zero-mean).  fp16
// carries the same 11 significant bits as TF32, so the accuracy equals a 3xTF32 scheme while an MMA instruction covers K = 16
// channels instead of 8: half the MMAs, half the operand bytes in shared memory.  What fp16 lacks is exponent range, hence the
// power-of-two scales: activations are staged as x * TC_ACT_SCALE (|x| < 65504 / TC_ACT_SCALE = 4094 is representable; smaller
// magnitudes keep 22 significant bits down to |x| ~ 2^-7 and an ABSOLUTE error of 2^-29 below that), weights are pre-scaled per
// output channel on the host so that max |w| lands in [2^14, 2^15) (ops.pack_tc_weight), and the epilogue's folded-BN scale
// carries the exact inverse 2^-(e_c + 4).  Conversions saturate (no inf/NaN poisoning) and a sticky device flag records any
// |x * s| > 65504 (osb_tc_overflow_count; the Python engines check it and refuse to return silently wrong results).
constexpr float TC_ACT_SCALE = 16.f;
constexpr float TC_F16_MAX = 65504.f;
// {lo 16 bits: fp16(a), hi 16 bits: fp16(b)}, round to nearest even, saturating to +-65504
__device__ __forceinline__ uint32_t cvt_f16x2_sat(float a, float b) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
__device__ __forceinline__ float2 f16x2_to_float2(uint32_t h) {
  float2 f;
  asm("{\n.reg .b16 l, u;\nmov.b32 {l, u}, %2;\ncvt.f32.f16 %0, l;\ncvt.f32.f16 %1, u;\n}\n" : "=f"(f.x), "=f"(f.y) : "r"(h));
  return f;
}
// four fp32 channels -> 4 fp16 hi parts + 4 fp16 lo parts of x * TC_ACT_SCALE; amax tracks max |x * s| for the overflow flag
__device__ __forceinline__ void f16_split4(const float4 v, uint2& hi, uint2& lo, float& amax) {
  const float x0 = v.x * TC_ACT_SCALE, x1 = v.y * TC_ACT_SCALE, x2 = v.z * TC_ACT_SCALE, x3 = v.w * TC_ACT_SCALE;
  amax = fmaxf(amax, fmaxf(fmaxf(fabsf(x0), fabsf(x1)), fmaxf(fabsf(x2), fabsf(x3))));
  hi.x = cvt_f16x2_sat(x0, x1);
  hi.y = cvt_f16x2_sat(x2, x3);
  const float2 h01 = f16x2_to_float2(hi.x), h23 = f16x2_to_float2(hi.y);
  lo.x = cvt_f16x2_sat(x0 - h01.x, x1 - h01.y);
  lo.y = cvt_f16x2_sat(x2 - h23.x, x3 - h23.y);
}
unsigned int* tc_overflow_flag();      // api.cu: device address of the sticky overflow counter of the CURRENT device
__device__ __forceinline__ void tc_report_overflow(unsigned int* flag, float amax) {
  if (amax > TC_F16_MAX) atomicAdd(flag, 1u);
}

// The tensor core's fp32 accumulation truncates (rounds towards zero) rather than rounding to nearest.  Each MMA therefore
// shrinks the running sum by ~c * ulp, and because E[partial sum after i of n MMAs | final] = (i/n) * final, an accumulator that
// received n MMAs comes out as final * (1 - kappa * n) plus zero-mean noise.  The shrink is coherent from layer to layer, the
// noise is not -- so the epilogue undoes the EXPECTED loss: raw sum * (1 + kappa * n), n = MMAs issued into that accumulator for
// this work item.  kappa is a calibration constant (tools/parity_bisect.py --layers); osb_set_rz_kappa() overrides it.
float rz_kappa();           // api.cu


// byte offset of 16-byte chunk `c` of K-major row `row` inside a swizzled operand tile
template <int KC>
__device__ __forceinline__ int swz_offset(int row, int c) {
  if constexpr (KC == 32) return row * 128 + ((c ^ (row & 7)) << 4);          // SWIZZLE_128B
  else return row * 64 + ((c ^ ((row >> 1) & 3)) << 4);                        // SWIZZLE_64B
}


// ------------------------------------------------------------------------------- split NDHWC activations
// The format the wgmma layers hand each other channels-last activations in: per voxel, channel granules of 16, each
// [16 fp16 hi | 16 fp16 lo] (64 bytes) of x * TC_ACT_SCALE split as f16_split4 does.  A (B, D, H, W, C) tensor is stored as
// (B, D, H, W, 2C) fp16: the bytes of the fp32 tensor, so voxel and channel-group offsets counted in floats (a multiple of 16
// channels) address the same bytes.  An operand row of KC channels is KC / 16 whole granules: a TMA tensor copy of it lands in
// shared memory exactly as the converters stage it (stage_f16_split), and the MMAs read the same values either way.
constexpr int SPLIT_GRANULE = 16;
// fp16 index, inside its voxel, of the hi part of channel c (the lo part follows SPLIT_GRANULE halves later)
__device__ __forceinline__ int split_index(int c) { return (c / SPLIT_GRANULE) * 2 * SPLIT_GRANULE + c % SPLIT_GRANULE; }
// encode four channels c .. c + 3 (c % 4 == 0) of one voxel
__device__ __forceinline__ void split_store4(uint16_t* vox, int c, const float4 v, float& amax) {
  uint2 hi, lo;
  f16_split4(v, hi, lo, amax);
  *reinterpret_cast<uint2*>(vox + split_index(c)) = hi;
  *reinterpret_cast<uint2*>(vox + split_index(c) + SPLIT_GRANULE) = lo;
}
// decode four channels: (hi + lo) * 2^-4, about 22 significant bits of the value that was encoded
__device__ __forceinline__ float4 split_load4(const uint16_t* vox, int c) {
  const uint2 hi = __ldg(reinterpret_cast<const uint2*>(vox + split_index(c)));
  const uint2 lo = __ldg(reinterpret_cast<const uint2*>(vox + split_index(c) + SPLIT_GRANULE));
  const float2 h01 = f16x2_to_float2(hi.x), h23 = f16x2_to_float2(hi.y), l01 = f16x2_to_float2(lo.x), l23 = f16x2_to_float2(lo.y);
  constexpr float inv = 1.f / TC_ACT_SCALE;
  return make_float4((h01.x + l01.x) * inv, (h01.y + l01.y) * inv, (h23.x + l23.x) * inv, (h23.y + l23.y) * inv);
}

// Stage four fp32 channels (fp32 16-byte chunk `q` of the KC-channel slice of operand row `row`) into a swizzled operand tile whose
// K-major rows hold KC / 16 split granules = 4*KC bytes (the layout of a split NDHWC row): hi part to 16-byte chunk
// 4(q/4) + (q%4)/2, lo part two chunks later, 8 bytes each.
template <int KC>
__device__ __forceinline__ void stage_f16_split(uint8_t* tile, int row, int q, const float4 v, float& amax) {
  uint2 hi, lo;
  f16_split4(v, hi, lo, amax);
  const int sub = (q & 1) << 3, chunk = 4 * (q >> 2) + ((q >> 1) & 1);
  *reinterpret_cast<uint2*>(tile + swz_offset<KC>(row, chunk) + sub) = hi;
  *reinterpret_cast<uint2*>(tile + swz_offset<KC>(row, chunk + 2) + sub) = lo;
}
// Lane -> operand row inside a warp-wide load of VPL = 128 / KC voxels (KC/4 lanes each), permuted so that the two STS.64 of
// stage_f16_split are bank-conflict free per half-warp: SWIZZLE_128B rows (KC = 32, granule order) must differ in bit 1, SWIZZLE_64B rows
// (KC = 16) must be {r, r+1, r+4, r+5}.  Global loads stay whole 16-byte chunks of whole voxels either way.
template <int KC>
__device__ __forceinline__ int lane_voxel(int lane) {
  if constexpr (KC == 32) return (((lane >> 3) & 1) << 1) | (lane >> 4);                       // 4 voxels: 0,2 | 1,3 (caller adds the rest)
  else return ((lane >> 2) & 1) | (((lane >> 3) & 1) << 2) | ((lane >> 4) << 1);               // 8 voxels: 0,1,4,5 | 2,3,6,7
}
// MMAs issued per accumulator per staged (unit, weight slice): k-steps of 16 channels x 3 split terms.  Descriptor start-address
// offsets in 16-byte units: k-step ks of an A row (split granules) is hi at A_KSTEP * ks, lo A_LO further; of a B row
// ([KC hi | KC lo], ops.pack_tc_weight) hi at 2 * ks, lo B_LO further.  For KC = 16 both layouts are the same.
template <int KC>
struct TcK {
  static constexpr int KSTEPS = KC / 16;
  static constexpr int A_KSTEP = 4;
  static constexpr int A_LO = 2;
  static constexpr int B_LO = KC / 8;
};

// ------------------------------------------------------------------------------- fragment-resident stride-1 epilogue
// conv3d_tc.cu / conv3d_tcg.cu: a 128 x 3G accumulator tile holds the kw-stacked partial sums [P0 | P1 | P2] of G output channels,
// and out[m] = P0[m - DIL] + P1[m] + P2[m + DIL].  In the fragment layout above, P0, P1 and P2 of one (row, channel) sit in
// registers 4j + r, 4(j + G/8) + r and 4(j + G/4) + r of the same thread, and rows m -+ DIL sit DIL lane quads away in the same
// warp, or DIL rows across the boundary of the warp's 16-row group.  So the un-shift runs on the registers: one shuffle per
// neighbour value (the sending lane picks which of its two row registers the receiver needs), and only the DIL seam rows of each
// 16-row group go through a small shared buffer.
// Seam buffer of one warpgroup, per exchange: [8 row groups (group 4h + w = rows 64h + 16w ..)][2 sides][DIL rows][G channels]:
// side 0 = P0 of the group's last DIL rows, side 1 = P2 of its first DIL rows.  Callers double-buffer it, so that a warp already
// publishing the next item's seams cannot overwrite values another warp has still to read.
template <int G, int DIL>
constexpr int frag_xchg_floats() { return 8 * 2 * DIL * G; }
// On return register 4(j + G/8) + r of acc[h] (the P1 registers) holds ((left + P1) + right) * corr for row 64h + 16wq + l/4 +
// 8(r/2), channel 8j + 2(l%4) + r%2.  Neighbours outside the image row (tile rows with m % W < DIL or >= W - DIL, W = tile row
// width) are +0, as the zero padding of the conv.  `bar`: this warpgroup's named barrier between the seam writes and reads.
template <int G, int DIL, int W>
__device__ __forceinline__ void frag_unshift(float (&acc)[2][3 * G / 2], float* xb, int wq, int lane, float corr, int bar) {
  constexpr int SIDE = DIL * G;
  const int l4 = lane >> 2, c0 = 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float* grp = xb + (4 * h + wq) * 2 * SIDE;
    if (l4 >= 8 - DIL) {
#pragma unroll
      for (int j = 0; j < G / 8; ++j)
        *reinterpret_cast<float2*>(grp + (l4 - 8 + DIL) * G + 8 * j + c0) = make_float2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
    }
    if (l4 < DIL) {
#pragma unroll
      for (int j = 0; j < G / 8; ++j)
        *reinterpret_cast<float2*>(grp + SIDE + l4 * G + 8 * j + c0) =
            make_float2(acc[h][4 * (j + G / 4)], acc[h][4 * (j + G / 4) + 1]);
    }
  }
  named_bar_sync(bar, 128);
  const int src_l = (lane - 4 * DIL) & 31, src_r = (lane + 4 * DIL) & 31;
  // a sender whose left-shuffle receiver wraps around to lanes 0 .. 4 DIL - 1 holds that receiver's hi-row neighbour in its lo row
  // register; likewise for the right shuffle
  const bool wrap_l = l4 >= 8 - DIL, wrap_r = l4 < DIL;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int g = 4 * h + wq;
    // seam values, loaded unconditionally from clamped addresses and merged with selects
    const float* xl = xb + (g > 0 ? g - 1 : 0) * 2 * SIDE + (l4 < DIL ? l4 : 0) * G + c0;
    const float* xr = xb + (g < 7 ? g + 1 : 7) * 2 * SIDE + SIDE + (l4 >= 8 - DIL ? l4 - 8 + DIL : 0) * G + c0;
    const int mlo = (64 * h + 16 * wq + l4) % W, mhi = (64 * h + 16 * wq + 8 + l4) % W;
#pragma unroll
    for (int j = 0; j < G / 8; ++j) {
      const float2 sl = *reinterpret_cast<const float2*>(xl + 8 * j);
      const float2 sr = *reinterpret_cast<const float2*>(xr + 8 * j);
#pragma unroll
      for (int c2 = 0; c2 < 2; ++c2) {
        const float p0lo = acc[h][4 * j + c2], p0hi = acc[h][4 * j + 2 + c2];
        const float p2lo = acc[h][4 * (j + G / 4) + c2], p2hi = acc[h][4 * (j + G / 4) + 2 + c2];
        float llo = __shfl_sync(0xffffffffu, p0lo, src_l);
        float lhi = __shfl_sync(0xffffffffu, wrap_l ? p0lo : p0hi, src_l);
        float rlo = __shfl_sync(0xffffffffu, wrap_r ? p2hi : p2lo, src_r);
        float rhi = __shfl_sync(0xffffffffu, p2hi, src_r);
        llo = (l4 < DIL) ? (c2 ? sl.y : sl.x) : llo;
        rhi = (l4 >= 8 - DIL) ? (c2 ? sr.y : sr.x) : rhi;
        llo = (mlo < DIL) ? 0.f : llo;
        lhi = (mhi < DIL) ? 0.f : lhi;
        rlo = (mlo >= W - DIL) ? 0.f : rlo;
        rhi = (mhi >= W - DIL) ? 0.f : rhi;
        float& olo = acc[h][4 * (j + G / 8) + c2];
        float& ohi = acc[h][4 * (j + G / 8) + 2 + c2];
        olo = ((llo + olo) + rlo) * corr;
        ohi = ((lhi + ohi) + rhi) * corr;
      }
    }
  }
}
// The ConvGRU gate activations (OSB_ACT_SIGMOID, OSB_ACT_TANH) with IEEE expf / tanhf: torch.sigmoid / torch.tanh to a few ulp.
static __device__ __noinline__ float gru_act(float v, int act) { return act == OSB_ACT_SIGMOID ? 1.f / (1.f + expf(-v)) : tanhf(v); }
// Channels-last output tile of one consumer warp: 16 fragment rows x 32 channels.  40 floats per row: the STS.64 of a half-warp
// (rows l/4, channel pairs 2(l%4)) hit distinct banks, and rows stay 16-byte aligned for the LDS.128 reads.
constexpr int FRAG_TP_STRIDE = 40;
constexpr int FRAG_TP_FLOATS = 16 * FRAG_TP_STRIDE;
// Folded BN, residual, activation and gate on the un-shifted fragments (frag_unshift), in that order, then the stores.  Row (h, rh)
// of this thread is tile row 64h + 16wq + l/4 + 8rh.  y / res / gate point at channel 0 of the tile's channel group;
// rows(m, yo, ro, go) sets tile row m's offsets into them and returns whether the row is stored.  ycs / rcs are the channel
// strides (1: channels-last, else NCDHW planes); nch: channels of the group that exist (channels-last callers pass G); sc / sh:
// the group's folded BN in shared memory; gate: channels-last only.
//   * channels-last output and residual (G = 32): the warp passes each m64 half's 16 rows through its own tile `tbuf`
//     (FRAG_TP_FLOATS), so that every LDG.128 / STG.128 of the warp covers 4 whole 128-byte rows: a store straight from the
//     fragments (32 bytes of each of 8 rows per instruction) needs 4x the L1 wavefronts on the data path the MMAs' operand reads
//     also use.  BN, residual, activation and gate run on the transposed values, where a lane's 4 channels are fixed.
//   * otherwise straight from the fragments: NCDHW planes take 8 consecutive voxels of 4 channels per warp instruction.
// y_split / res_split: the channels-last output / residual is split NDHWC (G = 32 only; offsets still count floats, which address
// the same bytes); a split output reports values outside the fp16 range on `overflow`.
// GRU (conv3d_tcg.cu's Cout = 128 instantiations, the ConvGRU update): act may also be OSB_ACT_SIGMOID / OSB_ACT_TANH, and bz / bh
// are channels-last operands at the gate's offsets; when set, the value after the gate becomes the blend bh + bz * (v - bh) =
// (1 - z) h + z q.  With either, the values are stored straight from the fragments.  Compiled out of every other instantiation.
template <int G, bool GRU = false, class Rows>
__device__ __forceinline__ void frag_epilogue(const float (&acc)[2][3 * G / 2], int lane, int wq, float* tbuf, const float* sc,
                                              const float* sh, int act, float* y, size_t ycs, const float* res, size_t rcs,
                                              const float* gate, Rows rows, int nch, bool y_split = false, bool res_split = false,
                                              unsigned int* overflow = nullptr, const float* bz = nullptr, const float* bh = nullptr) {
  const int c0 = 2 * (lane & 3), l4 = lane >> 2;
  if constexpr (G == 32) {
    // the GRU's multiplier and blend run on the path below: in this one they would make the Cout = 128 instantiations spill
    if (ycs == 1 && (!res || rcs == 1) && !(GRU && (gate || bz))) {
      const int c4 = 4 * (lane & 7), sub = lane >> 3;
      const float4 a = *reinterpret_cast<const float4*>(sc + c4);
      const float4 b = *reinterpret_cast<const float4*>(sh + c4);
      float amax = 0.f;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        __syncwarp();                                   // the previous half's readers are done with the tile
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int rh = 0; rh < 2; ++rh)
            *reinterpret_cast<float2*>(tbuf + (8 * rh + l4) * FRAG_TP_STRIDE + 8 * j + c0) =
                make_float2(acc[h][4 * (j + 4) + 2 * rh], acc[h][4 * (j + 4) + 2 * rh + 1]);
        __syncwarp();
        float4 o[4];
        ptrdiff_t yo[4], ro[4], go[4];
        bool ok[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {                   // tile row 4i + sub, channels c4 .. c4 + 3
          ok[i] = rows(64 * h + 16 * wq + 4 * i + sub, yo[i], ro[i], go[i]);
          o[i] = *reinterpret_cast<const float4*>(tbuf + (4 * i + sub) * FRAG_TP_STRIDE + c4);
          o[i].x = fmaf(o[i].x, a.x, b.x), o[i].y = fmaf(o[i].y, a.y, b.y), o[i].z = fmaf(o[i].z, a.z, b.z), o[i].w = fmaf(o[i].w, a.w, b.w);
        }
        if (res) {
          float4 r[4];
#pragma unroll
          for (int i = 0; i < 4; ++i)
            r[i] = !ok[i] ? make_float4(0.f, 0.f, 0.f, 0.f)
                 : res_split ? split_load4(reinterpret_cast<const uint16_t*>(res + ro[i]), c4)
                             : __ldg(reinterpret_cast<const float4*>(res + ro[i] + c4));
#pragma unroll
          for (int i = 0; i < 4; ++i) o[i].x += r[i].x, o[i].y += r[i].y, o[i].z += r[i].z, o[i].w += r[i].w;
        }
        if (act == OSB_ACT_RELU) {
#pragma unroll
          for (int i = 0; i < 4; ++i) o[i].x = fmaxf(o[i].x, 0.f), o[i].y = fmaxf(o[i].y, 0.f), o[i].z = fmaxf(o[i].z, 0.f), o[i].w = fmaxf(o[i].w, 0.f);
        } else if (act == OSB_ACT_LEAKY) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            o[i].x = o[i].x > 0.f ? o[i].x : 0.01f * o[i].x, o[i].y = o[i].y > 0.f ? o[i].y : 0.01f * o[i].y;
            o[i].z = o[i].z > 0.f ? o[i].z : 0.01f * o[i].z, o[i].w = o[i].w > 0.f ? o[i].w : 0.01f * o[i].w;
          }
        } else if (GRU && (act == OSB_ACT_SIGMOID || act == OSB_ACT_TANH)) {
#pragma unroll
          for (int i = 0; i < 4; ++i)
            o[i].x = gru_act(o[i].x, act), o[i].y = gru_act(o[i].y, act), o[i].z = gru_act(o[i].z, act), o[i].w = gru_act(o[i].w, act);
        }
        if (!GRU && gate) {
          float4 g[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) g[i] = ok[i] ? __ldg(reinterpret_cast<const float4*>(gate + go[i] + c4)) : make_float4(1.f, 1.f, 1.f, 1.f);
#pragma unroll
          for (int i = 0; i < 4; ++i) o[i].x *= g[i].x, o[i].y *= g[i].y, o[i].z *= g[i].z, o[i].w *= g[i].w;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if (!ok[i]) continue;
          if (y_split) split_store4(reinterpret_cast<uint16_t*>(y + yo[i]), c4, o[i], amax);
          else *reinterpret_cast<float4*>(y + yo[i] + c4) = o[i];
        }
      }
      if (y_split) tc_report_overflow(overflow, amax);
      return;
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    // one m64 half at a time, its residual and gate loads batched ahead of its stores (the compiler does not move a load across
    // a store that may alias it, so per-element loads would expose one memory latency each)
    float2 rv[G / 8][2], gv[G / 8][2];
#pragma unroll
    for (int j = 0; j < G / 8; ++j)
#pragma unroll
      for (int rh = 0; rh < 2; ++rh) {
        const int c = 8 * j + c0;
        ptrdiff_t yo, ro, go;
        const bool live = rows(64 * h + 16 * wq + l4 + 8 * rh, yo, ro, go);
        rv[j][rh] = make_float2(0.f, 0.f);
        gv[j][rh] = make_float2(1.f, 1.f);
        if (res) {
          if (rcs == 1) {
            if (live) rv[j][rh] = __ldg(reinterpret_cast<const float2*>(res + ro + c));
          } else {
            if (live && c < nch) rv[j][rh].x = __ldg(res + ro + (size_t)c * rcs);
            if (live && c + 1 < nch) rv[j][rh].y = __ldg(res + ro + (size_t)(c + 1) * rcs);
          }
        }
        if (!GRU && gate && live) gv[j][rh] = __ldg(reinterpret_cast<const float2*>(gate + go + c));
      }
#pragma unroll
    for (int j = 0; j < G / 8; ++j) {
      const int c = 8 * j + c0;
      const float2 a = *reinterpret_cast<const float2*>(sc + c);
      const float2 b = *reinterpret_cast<const float2*>(sh + c);
#pragma unroll
      for (int rh = 0; rh < 2; ++rh) {
        ptrdiff_t yo, ro, go;
        const bool live = rows(64 * h + 16 * wq + l4 + 8 * rh, yo, ro, go);
        float v0 = fmaf(acc[h][4 * (j + G / 8) + 2 * rh], a.x, b.x);
        float v1 = fmaf(acc[h][4 * (j + G / 8) + 2 * rh + 1], a.y, b.y);
        if (res) v0 += rv[j][rh].x, v1 += rv[j][rh].y;
        if (act == OSB_ACT_RELU) {
          v0 = fmaxf(v0, 0.f), v1 = fmaxf(v1, 0.f);
        } else if (act == OSB_ACT_LEAKY) {
          v0 = v0 > 0.f ? v0 : 0.01f * v0, v1 = v1 > 0.f ? v1 : 0.01f * v1;
        } else if (GRU && (act == OSB_ACT_SIGMOID || act == OSB_ACT_TANH)) {
          v0 = gru_act(v0, act), v1 = gru_act(v1, act);
        }
        if (!GRU && gate) v0 *= gv[j][rh].x, v1 *= gv[j][rh].y;
        if (!live) continue;
        if (GRU && gate) {                              // loaded where it is used: batched like gv, the GRU operands would spill
          const float2 m = __ldg(reinterpret_cast<const float2*>(gate + go + c));
          v0 *= m.x, v1 *= m.y;
        }
        if (GRU && bz) {
          const float2 z = __ldg(reinterpret_cast<const float2*>(bz + go + c));
          const float2 hv = __ldg(reinterpret_cast<const float2*>(bh + go + c));
          v0 = hv.x + z.x * (v0 - hv.x), v1 = hv.y + z.y * (v1 - hv.y);
        }
        if (ycs == 1) {
          *reinterpret_cast<float2*>(y + yo + c) = make_float2(v0, v1);
        } else {
          if (c < nch) y[yo + (size_t)c * ycs] = v0;
          if (c + 1 < nch) y[yo + (size_t)(c + 1) * ycs] = v1;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------- coalesced channels-last epilogue output
// An epilogue thread owns ONE voxel and all of its channels.  Storing those directly makes every STG.128 of a warp touch
// 32 different 128-byte lines (16 B of each) -- 8x the L1 wavefronts of a coalesced store, on the data pipe the tensor
// core's operand reads also use.  Instead the warp transposes its
// 32 voxels x 32 channels through a private shared-memory tile so one instruction covers 4 voxels x 128 contiguous bytes;
// folded BN, the channels-last residual and the activation are applied after the transpose, where a lane's four channels
// are the same for every voxel (scale/shift sit in registers instead of one LDS per channel).
constexpr int TP_STRIDE = 36;                       // floats per tile row: 144 B keeps STS.128 / LDS.128 conflict-free
constexpr int TP_WARP_FLOATS = 32 * TP_STRIDE;      // 4608 B per epilogue warp (the kernels reuse the warp's own rows of the staged
                                                    // accumulator tile, which the warp has read into registers by then)

// sum[32]: raw accumulator sums of this lane's voxel for channels [c, c+32).  y0 / res0 point at channel c of the voxel
// owned by lane 0; lane k's voxel lies vstride floats further per lane.  sc / sh point at channel c of the folded BN.
// vmask: bit k set = the voxel of lane k exists in the output (general-width column tiles mask their halo columns and the part of
// the last tile beyond the image; whole-row tiles pass all ones and the tests fold away).
// gate0: optional channels-last multiplier of lane 0's voxel (same voxel stride), applied AFTER the activation -- FeatureAtt's
// sigmoid(att) * cv of stereobase/hourglass.py:80-99 / igev_blocks.py:35-48 with the gate stored as (B, H, W, C).
__device__ __forceinline__ void store_ndhwc_chunk32(float* tbuf, int lane, const float (&sum)[32], float* y0, const float* res0,
                                                    size_t vstride, const float* sc, const float* sh, int act,
                                                    uint32_t vmask = 0xffffffffu, const float* gate0 = nullptr) {
  const int c4 = 4 * (lane & 7), sub = lane >> 3;
  __syncwarp();                                     // the previous chunk's readers are done with the tile
  float4* row = reinterpret_cast<float4*>(tbuf + lane * TP_STRIDE);
#pragma unroll
  for (int i = 0; i < 8; ++i) row[i] = make_float4(sum[4 * i], sum[4 * i + 1], sum[4 * i + 2], sum[4 * i + 3]);
  __syncwarp();
  const float4 a = *reinterpret_cast<const float4*>(sc + c4);
  const float4 b = *reinterpret_cast<const float4*>(sh + c4);
  float4 o[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    o[j] = *reinterpret_cast<const float4*>(tbuf + (4 * j + sub) * TP_STRIDE + c4);
    o[j].x = fmaf(o[j].x, a.x, b.x), o[j].y = fmaf(o[j].y, a.y, b.y), o[j].z = fmaf(o[j].z, a.z, b.z), o[j].w = fmaf(o[j].w, a.w, b.w);
  }
  if (res0) {
    float4 r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j)
      r[j] = ((vmask >> (4 * j + sub)) & 1u) ? __ldg(reinterpret_cast<const float4*>(res0 + (size_t)(4 * j + sub) * vstride + c4))
                                             : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j].x += r[j].x, o[j].y += r[j].y, o[j].z += r[j].z, o[j].w += r[j].w;
  }
  if (act == OSB_ACT_RELU) {
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j].x = fmaxf(o[j].x, 0.f), o[j].y = fmaxf(o[j].y, 0.f), o[j].z = fmaxf(o[j].z, 0.f), o[j].w = fmaxf(o[j].w, 0.f);
  } else if (act == OSB_ACT_LEAKY) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o[j].x = o[j].x > 0.f ? o[j].x : 0.01f * o[j].x, o[j].y = o[j].y > 0.f ? o[j].y : 0.01f * o[j].y;
      o[j].z = o[j].z > 0.f ? o[j].z : 0.01f * o[j].z, o[j].w = o[j].w > 0.f ? o[j].w : 0.01f * o[j].w;
    }
  }
  if (gate0) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (!((vmask >> (4 * j + sub)) & 1u)) continue;
      const float4 g = __ldg(reinterpret_cast<const float4*>(gate0 + (size_t)(4 * j + sub) * vstride + c4));
      o[j].x *= g.x, o[j].y *= g.y, o[j].z *= g.z, o[j].w *= g.w;
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j)
    if ((vmask >> (4 * j + sub)) & 1u) *reinterpret_cast<float4*>(y0 + (size_t)(4 * j + sub) * vstride + c4) = o[j];
}

// ------------------------------------------------------------------------------------------------ host: check and launch
// Arguments of a tensor-core conv entry point (include/openstereo_b200.h).  Extents are those of the INPUT.
struct TcArgs {
  const float* x;
  const void* w;
  const float* scale;
  const float* shift;
  const float* residual;
  const float* gate;       // stride 1: FeatureAtt gate (B, H, W, Cout) channels-last, or null
  float* y;
  int B, Cin, Cout, D, H, W;
  int act, out_ndhwc, res_ndhwc;
  int in_ncdhw;            // stride 1: the input is (B, Cin, D, H, W)
  int ystride;             // channels per voxel of the channels-last y / residual / gate (0 = Cout)
  int cout_real;           // channels an NCDHW output / residual holds (< Cout: a zero-padded channel plan)
  float kappa;             // set by check_tc_args
  unsigned int* overflow;  // set by check_tc_args
  int in_split = 0, out_split = 0, res_split = 0;   // stride 1, W = 128: the channels-last x / y / residual is split NDHWC
  // ConvGRU epilogue (osb_conv2d_k3_tc_gru_fwd, conv3d_tcg.cu only): gru = 1 admits OSB_ACT_SIGMOID / OSB_ACT_TANH and the operands
  // below, each (B,H,W,Cout) channels-last: y = act(...) * mul, then y = blend_h + blend_z * (y - blend_h).  res_bstride: floats
  // between the batches of an NCDHW residual (0 = Cout*D*H*W), so that a channel split() view of a wider tensor needs no copy.
  int gru = 0;
  const float* mul = nullptr;
  const float* blend_z = nullptr;
  const float* blend_h = nullptr;
  long long res_bstride = 0;
  bool slice() const { return ystride != 0 && ystride != Cout; }
};
// Launcher of one instantiation: the result of a family's selector (null: no instantiation serves the arguments).
using TcLaunch = int (*)(const TcArgs&, cudaStream_t);

// The checks every tensor-core entry point runs after its family's shape rules and before any CUDA call: pointers (the kernels'
// loaders and stores use 128-bit accesses and bulk copies), extents, activation, the layouts a channel slice, a gate or a
// zero-padded channel plan need (OSB_EINVAL); a selector result for the requested gate / channel slice (OSB_EUNSUPPORTED); then
// the overflow flag of the current device (OSB_ECUDA).
inline int check_tc_args(const char* what, TcArgs& a, TcLaunch launch) {
  auto aligned = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  OSB_REQUIRE(a.x && a.w && a.y, "%s: null pointer", what);
  OSB_REQUIRE(a.B > 0 && a.D > 0 && a.H > 0, "%s: empty shape", what);
  OSB_REQUIRE(a.act >= 0 && (a.act <= 2 || (a.gru && (a.act == OSB_ACT_SIGMOID || a.act == OSB_ACT_TANH))), "%s: unknown activation %d",
              what, a.act);
  OSB_REQUIRE(aligned(a.x) && aligned(a.w) && aligned(a.y) && aligned(a.residual) && aligned(a.gate) && aligned(a.mul) &&
              aligned(a.blend_z) && aligned(a.blend_h), "%s: pointers must be 16-byte aligned", what);
  OSB_REQUIRE(!a.blend_z == !a.blend_h, "%s: the blend needs both z and h", what);
  OSB_REQUIRE(a.res_bstride == 0 || (a.residual && !a.res_ndhwc && a.res_bstride >= (long long)a.Cout * a.D * a.H * a.W),
              "%s: a residual batch stride (%lld) needs an NCDHW residual and at least Cout*D*H*W floats", what, a.res_bstride);
  const bool channels_last = a.out_ndhwc && (!a.residual || a.res_ndhwc);
  OSB_REQUIRE(a.ystride == 0 || (a.ystride >= a.Cout && a.ystride % 4 == 0 && channels_last),
              "%s: a channel slice (ystride %d) needs channels-last tensors", what, a.ystride);
  OSB_REQUIRE(!a.gate || channels_last, "%s: the gate operand needs a channels-last output (and residual)", what);
  OSB_REQUIRE(a.cout_real == a.Cout || (a.cout_real >= 1 && a.cout_real < a.Cout && !a.out_ndhwc && (!a.residual || !a.res_ndhwc)),
              "%s: only NCDHW tensors may hold fewer (%d) channels than the packed %d", what, a.cout_real, a.Cout);
  if (!launch) {
    set_error("%s: no instantiation serves Cout=%d W=%d with gate=%d ystride=%d", what, a.Cout, a.W, a.gate != nullptr, a.ystride);
    return OSB_EUNSUPPORTED;
  }
  a.kappa = rz_kappa();
  a.overflow = tc_overflow_flag();
  return a.overflow ? OSB_OK : OSB_ECUDA;   // tc_overflow_flag has set the message
}

// Launch of a persistent tensor-core kernel over `items` work items (CTAs walk it = blockIdx.x, + gridDim.x, ...): one CTA per SM
// at most (its shared memory is taken), the grid capped by osb_set_persistent_grid_cap.  Fills the fields every Params struct has
// from `a`; the family launcher has set the rest.  `variant` is what osb_tc_last_variant reports.  A template on the kernel, so
// that every instantiation has its own per-device "shared memory configured" flag.
template <auto KERNEL, class P>
int launch_persistent(const TcArgs& a, P p, long long items, size_t smem, const char* variant, cudaStream_t stream) {
  OSB_REQUIRE(items < (1ll << 31), "%s: too many work items", variant);
  static PerDeviceFlag configured;
  if (!configured.here()) {
    const cudaError_t e = cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
      set_error("%s: cannot reserve %zu bytes of shared memory: %s", variant, smem, cudaGetErrorString(e));
      return OSB_ECUDA;
    }
    configured.here() = true;
  }
  p.x = a.x, p.w = a.w, p.scale = a.scale, p.shift = a.shift, p.residual = a.residual, p.y = a.y;
  p.B = a.B, p.D = a.D, p.H = a.H, p.Cin = a.Cin, p.act = a.act, p.out_ndhwc = a.out_ndhwc, p.res_ndhwc = a.res_ndhwc;
  p.kappa = a.kappa, p.overflow = a.overflow;
  p.items = (int)items;
  const int sms = sm_count();
  set_tc_variant(variant);
  KERNEL<<<(int)cap_persistent_grid(p.items < sms ? p.items : sms), TC_WG_THREADS, smem, stream>>>(p);
  count_launch();
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    cudaFuncAttributes fa{};
    (void)cudaFuncGetAttributes(&fa, KERNEL);
    set_error("%s: launch failed: %s (threads %d, kernel maxThreadsPerBlock %d, regs %d, static smem %zu, dynamic smem %zu, "
              "max dynamic %d)", variant, cudaGetErrorString(e), TC_WG_THREADS, fa.maxThreadsPerBlock, fa.numRegs,
              fa.sharedSizeBytes, smem, fa.maxDynamicSharedSizeBytes);
    return OSB_ECUDA;
  }
  return OSB_OK;
}

// The stride-1 family's selector (conv3d_tcg.cu): the instantiation of conv3d_tc.cu or conv3d_tcg.cu that serves Conv3d k3 s1 p1
// (dilation 2: the one-plane 2D conv), with a gate / writing a channel slice, and its K chunk; {nullptr, 0} when there is none.
struct TcRoute {
  TcLaunch launch;
  int kc;
};
TcRoute select_conv3d_tc(int Cin, int Cout, int W, int dilation, bool gate, bool slice);
template <int COUT>
int launch_tc(const TcArgs& a, cudaStream_t stream);   // conv3d_tc.cu

}  // namespace osb
