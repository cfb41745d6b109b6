// Shared helpers for the sm_90a kernels of the OpenStereo cost-volume hot path.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <string>

#include "../../include/openstereo_b200.h"

namespace osb {

// ---- error plumbing (api.cu owns the storage) -------------------------------------------------
void set_error(const char* fmt, ...);
void count_launch(int n = 1);
int check_launch(const char* what);  // cudaGetLastError -> OSB_OK / OSB_ECUDA (+message)
int device_index();                   // current CUDA device (0 when the query fails)
int sm_count();                       // multiprocessors of the CURRENT device (cached per device)
// Grid of a persistent kernel (CTAs walk `for (it = blockIdx.x; it < items; it += gridDim.x)`): `grid` clamped to the cap set by
// osb_set_persistent_grid_cap, so tests can make one CTA run many work items in a row.
long long cap_persistent_grid(long long grid);
// Template arguments of a tensor-core instantiation, spelled as osb_tc_last_variant returns them; each launcher formats its name
// once (a function-local static) and records it on every launch with set_tc_variant (this thread only; `name` must outlive it).
std::string tc_variant_name(const char* fmt, ...);
void set_tc_variant(const char* name);
// Per-device "already configured" flag: cudaFuncSetAttribute is per device, a process may drive several
// (DataParallel, model.to('cuda:1')); a plain `static bool` would configure only the first one.
struct PerDeviceFlag {
  bool done[64] = {};
  bool& here() { return done[device_index() & 63]; }
};

#define OSB_REQUIRE(cond, ...)          \
  do {                                  \
    if (!(cond)) {                      \
      ::osb::set_error(__VA_ARGS__);    \
      return OSB_EINVAL;                \
    }                                   \
  } while (0)

// ---- small device helpers ---------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// 3-D TMA tile load global -> shared, completion signalled on an mbarrier (SASS: UTMALDG).
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
// 4-D TMA tile load (coordinates innermost-first; boxes partly or wholly outside the tensor are zero-filled)
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// streaming (evict-first) 128-bit store: the volumes are written once and read by the next kernel
// from HBM/L2, never re-read by this one.
__device__ __forceinline__ void st_cs_f4(float* p, float4 v) { __stcs(reinterpret_cast<float4*>(p), v); }

// ---- host-side TMA descriptor factory (api.cu) ------------------------------------------------
// dims/strides innermost-first, fp32 elements, zero OOB fill, no swizzle.  Returns false (and sets the error)
// when the driver entry point is missing or the encode fails.
bool make_tensor_map_3d(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_bytes,
                        uint64_t stride2_bytes, uint32_t box0, uint32_t box1, uint32_t box2);
// Split NDHWC activations (tc_common.cuh) of a (B, D, H, W, C) tensor as a 4-D fp16 map (2C, W, H, B*D), box = `kc` channels'
// granules x W voxels x 1 x 1, zero fill outside, the wgmma operand swizzle (kc = 32: 128 B, kc = 16: 64 B).
bool make_tensor_map_split(CUtensorMap* out, const void* base, int C, int W, int H, int BD, int kc);

}  // namespace osb
