// C-ABI plumbing: error strings, launch accounting and the TMA descriptor factory.
#include <atomic>
#include <cstdarg>
#include <cstring>

#include "common.cuh"

namespace osb {

static thread_local char g_error[512] = "";
static std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
}

static std::atomic<float> g_rz_kappa{1.57e-8f};   // default of osb_set_rz_kappa (include/openstereo_b200.h)
float rz_kappa() { return g_rz_kappa.load(std::memory_order_relaxed); }

static std::atomic<int> g_grid_cap{0};            // osb_set_persistent_grid_cap; 0 = no cap
long long cap_persistent_grid(long long grid) {
  const int cap = g_grid_cap.load(std::memory_order_relaxed);
  return (cap > 0 && grid > cap) ? cap : grid;
}

std::string tc_variant_name(const char* fmt, ...) {
  char buf[64];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  return buf;
}
static thread_local const char* g_tc_variant = "";
void set_tc_variant(const char* name) { g_tc_variant = name; }

// Sticky fp16-range counter of the tensor-core convolutions (tc_common.cuh): one zero-initialised unsigned int per device,
// allocated on first use, incremented by every loader thread that staged a value beyond +-65504 / TC_ACT_SCALE.
static std::atomic<unsigned int*> g_overflow[64];
unsigned int* tc_overflow_flag() {
  const int dev = device_index() & 63;
  unsigned int* p = g_overflow[dev].load(std::memory_order_acquire);
  if (p) return p;
  unsigned int* fresh = nullptr;
  if (cudaMalloc(&fresh, sizeof(unsigned int)) != cudaSuccess || cudaMemset(fresh, 0, sizeof(unsigned int)) != cudaSuccess) {
    set_error("tc_overflow_flag: %s", cudaGetErrorString(cudaGetLastError()));
    return nullptr;
  }
  unsigned int* expected = nullptr;
  if (!g_overflow[dev].compare_exchange_strong(expected, fresh, std::memory_order_acq_rel)) {
    (void)cudaFree(fresh);
    return expected;
  }
  return fresh;
}

int device_index() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    (void)cudaGetLastError();
    return 0;
  }
  return dev;
}

int sm_count() {
  static std::atomic<int> cache[64];
  const int dev = device_index();
  int n = cache[dev & 63].load(std::memory_order_relaxed);
  if (n > 0) return n;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) {
    (void)cudaGetLastError();
    n = 132;
  }
  cache[dev & 63].store(n, std::memory_order_relaxed);
  return n;
}

void count_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) return OSB_OK;
  set_error("%s: launch failed: %s", what, cudaGetErrorString(e));
  return OSB_ECUDA;
}

// cuTensorMapEncodeTiled is a driver-API symbol; fetch it through the runtime so the library does not link libcuda.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess) {
      (void)cudaGetLastError();
      return (EncodeTiledFn) nullptr;
    }
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

bool make_tensor_map_3d(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2, uint64_t stride1_bytes,
                        uint64_t stride2_bytes, uint32_t box0, uint32_t box1, uint32_t box2) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled not available from the driver");
    return false;
  }
  const cuuint64_t dims[3] = {d0, d1, d2};
  const cuuint64_t strides[2] = {stride1_bytes, stride2_bytes};
  const cuuint32_t box[3] = {box0, box1, box2};
  const cuuint32_t elem[3] = {1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(base), dims, strides, box, elem,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
    return false;
  }
  return true;
}

bool make_tensor_map_split(CUtensorMap* out, const void* base, int C, int W, int H, int BD, int kc) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled not available from the driver");
    return false;
  }
  const uint64_t vox = 2ull * C * sizeof(uint16_t);                  // bytes per voxel
  const cuuint64_t dims[4] = {2ull * C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)BD};
  const cuuint64_t strides[3] = {vox, vox * W, vox * W * H};
  const cuuint32_t box[4] = {2u * kc, (cuuint32_t)W, 1, 1};
  const cuuint32_t elem[4] = {1, 1, 1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, elem,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, kc == 32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled (split activations) failed with CUresult %d", (int)r);
    return false;
  }
  return true;
}

}  // namespace osb

extern "C" {
int osb_abi_version(void) { return 1; }
const char* osb_last_error(void) { return osb::g_error; }
uint64_t osb_launch_count(void) { return osb::g_launches.load(std::memory_order_relaxed); }
float osb_set_rz_kappa(float kappa) {
  const float old = osb::g_rz_kappa.load(std::memory_order_relaxed);
  if (kappa >= 0.f && kappa < 1e-6f) osb::g_rz_kappa.store(kappa, std::memory_order_relaxed);
  return old;
}
int osb_set_persistent_grid_cap(int cap) { return osb::g_grid_cap.exchange(cap > 0 ? cap : 0, std::memory_order_relaxed); }
const char* osb_tc_last_variant(void) { return osb::g_tc_variant; }
int osb_tc_overflow_count(osb_stream_t stream, int reset, unsigned int* count) {
  using namespace osb;
  OSB_REQUIRE(count, "tc_overflow_count: null pointer");
  unsigned int* flag = tc_overflow_flag();
  if (!flag) return OSB_ECUDA;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemcpyAsync(count, flag, sizeof(unsigned int), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess && reset) e = cudaMemsetAsync(flag, 0, sizeof(unsigned int), st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    set_error("tc_overflow_count: %s", cudaGetErrorString(e));
    return OSB_ECUDA;
  }
  return OSB_OK;
}
const unsigned int* osb_tc_overflow_flag(void) { return osb::tc_overflow_flag(); }
int osb_tc_overflow_poll(osb_stream_t stream, unsigned int* host_pinned) {
  using namespace osb;
  OSB_REQUIRE(host_pinned, "tc_overflow_poll: null pointer");
  unsigned int* flag = tc_overflow_flag();
  if (!flag) return OSB_ECUDA;
  cudaError_t e = cudaMemcpyAsync(host_pinned, flag, sizeof(unsigned int), cudaMemcpyDeviceToHost, (cudaStream_t)stream);
  if (e != cudaSuccess) {
    set_error("tc_overflow_poll: %s", cudaGetErrorString(e));
    return OSB_ECUDA;
  }
  return OSB_OK;
}
}
