// wvn-b200: host-side helpers (error string, tensor-map encoding).
#include "host_common.h"

#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <mutex>
#include <vector>

namespace wvn {

static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

const char* last_error() { return g_err; }

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || p == nullptr) return nullptr;
  fn = reinterpret_cast<PFN_encodeTiled>(p);
  return fn;
}

int make_tmap_bf16_2d(CUtensorMap* out, const void* gptr, uint64_t inner, uint64_t outer,
                      uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return set_error(WVN_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  if (box_inner * 2 != 128) return set_error(WVN_ERR_INVALID, "tensor map: inner box must be 128 bytes");
  if (box_outer > 256) return set_error(WVN_ERR_INVALID, "tensor map: outer box must be <= 256");
  if ((reinterpret_cast<uintptr_t>(gptr) & 15) != 0 || (row_stride_bytes & 15) != 0)
    return set_error(WVN_ERR_INVALID, "tensor map: base/stride must be 16-byte aligned (ptr=%p stride=%llu)", gptr,
                     (unsigned long long)row_stride_bytes);
  cuuint64_t gdim[2] = {inner, outer};
  cuuint64_t gstride[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(gptr), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(WVN_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d (inner=%llu outer=%llu)", (int)r,
                     (unsigned long long)inner, (unsigned long long)outer);
  return WVN_OK;
}

int make_tmap_2d(CUtensorMap* out, const void* gptr, int elem_bytes, uint64_t inner, uint64_t outer,
                 uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer, int swizzle_bytes) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return set_error(WVN_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  if (elem_bytes != 2 && elem_bytes != 4) return set_error(WVN_ERR_INVALID, "tensor map: element size %d", elem_bytes);
  if (swizzle_bytes != 0 && box_inner * elem_bytes != static_cast<uint32_t>(swizzle_bytes))
    return set_error(WVN_ERR_INVALID, "tensor map: inner box (%u B) must equal the swizzle span (%d B)",
                     box_inner * elem_bytes, swizzle_bytes);
  if (box_outer > 256 || (reinterpret_cast<uintptr_t>(gptr) & 15) != 0 || (row_stride_bytes & 15) != 0)
    return set_error(WVN_ERR_INVALID, "tensor map: bad box / alignment (ptr=%p stride=%llu)", gptr,
                     (unsigned long long)row_stride_bytes);
  cuuint64_t gdim[2] = {inner, outer};
  cuuint64_t gstride[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUresult r = fn(out, elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                  const_cast<void*>(gptr), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(WVN_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d (inner=%llu outer=%llu)", (int)r,
                     (unsigned long long)inner, (unsigned long long)outer);
  return WVN_OK;
}

int sm_count() {
  static int n = 0;
  if (n) return n;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  return n;
}

static std::atomic<long long> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
long long launch_count() { return g_launches.load(); }

namespace {
struct ProfRec { int cat; cudaEvent_t a, b; };
std::mutex g_prof_mu;
int g_prof_mask = 0;  // bit c = category c is timed
std::vector<ProfRec> g_prof;
std::vector<cudaEvent_t> g_pool;
cudaEvent_t g_open[PROF_NUM] = {nullptr, nullptr};
cudaEvent_t get_event() {
  if (!g_pool.empty()) { cudaEvent_t e = g_pool.back(); g_pool.pop_back(); return e; }
  cudaEvent_t e = nullptr;
  cudaEventCreate(&e);
  return e;
}
}  // namespace

void prof_enable(int category_mask) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof_mask = category_mask;
}

void prof_begin(int cat, cudaStream_t s) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (!((g_prof_mask >> cat) & 1)) return;
  g_open[cat] = get_event();
  cudaEventRecord(g_open[cat], s);
}

void prof_end(int cat, cudaStream_t s) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (g_open[cat] == nullptr) return;
  cudaEvent_t b = get_event();
  cudaEventRecord(b, s);
  g_prof.push_back({cat, g_open[cat], b});
  g_open[cat] = nullptr;
}

int prof_collect(float* ms_by_cat, long long* launches_by_cat) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  for (int i = 0; i < PROF_NUM; ++i) { ms_by_cat[i] = 0.f; launches_by_cat[i] = 0; }
  for (auto& r : g_prof) {
    cudaError_t e = cudaEventSynchronize(r.b);
    if (e != cudaSuccess) return set_error(WVN_ERR_CUDA, "profiler: %s", cudaGetErrorString(e));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, r.a, r.b);
    ms_by_cat[r.cat] += ms;
    launches_by_cat[r.cat] += 1;
    g_pool.push_back(r.a);
    g_pool.push_back(r.b);
  }
  g_prof.clear();
  return WVN_OK;
}

}  // namespace wvn
