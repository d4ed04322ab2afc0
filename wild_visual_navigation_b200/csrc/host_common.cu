// wvn-b200: host-side helpers (error string, tensor-map encoding, device buffers and arenas, weight stores).
#include "host_common.h"

#include <cuda_bf16.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <mutex>
#include <vector>

#include "gemm.h"

namespace {

// fp32 rows [rows, dim] -> bf16 rows [rows, ld] (padding columns left untouched = zero)
__global__ void cast_rows_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long rows, int dim,
                                 long long ld) {
  const long long n = rows * dim;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / dim;
    const int c = static_cast<int>(i - r * dim);
    dst[r * ld + c] = __float2bfloat16_rn(src[i]);
  }
}

}  // namespace

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

int cast_rows_to_bf16(const float* src, void* dst, long long rows, int dim, long long ld, int max_blocks,
                      cudaStream_t s) {
  const int blocks = static_cast<int>(std::min<long long>((rows * dim + 255) / 256, max_blocks));
  cast_rows_kernel<<<blocks, 256, 0, s>>>(src, reinterpret_cast<__nv_bfloat16*>(dst), rows, dim, ld);
  WVN_CHECK_LAUNCH("cast_rows_kernel");
  return WVN_OK;
}

int DevBuf::alloc(size_t n) {
  release();
  void* q = nullptr;
  WVN_CHECK_CUDA(cudaMalloc(&q, n ? n : 1));
  p = q;
  bytes = n;
  WVN_CHECK_CUDA(cudaMemset(p, 0, n ? n : 1));
  return WVN_OK;
}

void DevBuf::release() {
  if (p) cudaFree(p);
  p = nullptr;
  bytes = 0;
}

int carve(DevBuf* buf, const std::function<void(Carver&)>& layout, const char* who) {
  Carver count;
  layout(count);
  const int rc = buf->alloc(count.bytes);
  if (rc != WVN_OK) {
    const std::string why = last_error();
    return set_error(rc, "%s: arena of %zu bytes: %s", who, count.bytes, why.c_str());
  }
  Carver pieces;
  pieces.base = static_cast<char*>(buf->p);
  layout(pieces);
  return WVN_OK;
}

constexpr size_t kStageBytes = 8u << 20;

int WeightStore::add(const std::string& name, long long rows, int cols, bool bf16) {
  if (!stage.p) WVN_PROPAGATE(stage.alloc(kStageBytes));
  const long long ld = bf16 ? gemm_w_pitch(cols) : cols;
  Weight& wt = w[name];
  WVN_PROPAGATE(wt.buf.alloc(static_cast<size_t>(rows * ld) * (bf16 ? 2 : 4)));
  wt.numel = rows * cols;
  wt.bf16 = bf16;
  wt.cols = cols;
  wt.ld = static_cast<int>(ld);
  return WVN_OK;
}

int WeightStore::set(const char* name, const float* data, long long numel) {
  auto it = w.find(name);
  WVN_REQUIRE(it != w.end(), "set_weight: unknown weight '%s'", name);
  Weight& wt = it->second;
  WVN_REQUIRE(wt.numel == numel, "set_weight: '%s' expects %lld elements, got %lld", name, wt.numel, numel);
  cudaPointerAttributes attr;
  bool on_device = false;
  if (cudaPointerGetAttributes(&attr, data) == cudaSuccess)
    on_device = (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged);
  else
    cudaGetLastError();
  // fp32 destination: copy straight in; bf16 destination: stage (if host) + cast on device
  if (!wt.bf16) {
    WVN_CHECK_CUDA(
        cudaMemcpy(wt.buf.p, data, numel * 4, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
  } else {
    // stage whole rows, cast each into its row of the pitched storage
    const long long chunk_rows = static_cast<long long>(stage.bytes / 4) / wt.cols;
    const long long rows = numel / wt.cols;
    for (long long r0 = 0; r0 < rows; r0 += chunk_rows) {
      const long long n = std::min(chunk_rows, rows - r0);
      const float* src = data + r0 * wt.cols;
      if (!on_device) {
        WVN_CHECK_CUDA(cudaMemcpy(stage.p, src, n * wt.cols * 4, cudaMemcpyHostToDevice));
        src = reinterpret_cast<const float*>(stage.p);
      }
      WVN_PROPAGATE(cast_rows_to_bf16(src, reinterpret_cast<__nv_bfloat16*>(wt.buf.p) + r0 * wt.ld, n, wt.cols, wt.ld,
                                      4096, 0));
      WVN_CHECK_CUDA(cudaStreamSynchronize(0));
    }
  }
  wt.loaded = true;
  return WVN_OK;
}

int WeightStore::check_loaded(const char* what, const char* skip_prefix) const {
  for (auto& kv : w) {
    if (skip_prefix && kv.first.rfind(skip_prefix, 0) == 0) continue;
    if (!kv.second.loaded) return set_error(WVN_ERR_STATE, "%s: weight '%s' was never set", what, kv.first.c_str());
  }
  return WVN_OK;
}

}  // namespace wvn
