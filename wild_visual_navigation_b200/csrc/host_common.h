// wvn-b200: host-side helpers shared by the translation units of libwvn_b200.so
// (error reporting, TMA tensor-map encoding through the driver entry point, device buffers and arenas, weight stores).
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <functional>
#include <map>
#include <string>

namespace wvn {

// Error codes returned through the C ABI (0 = ok).
enum : int {
  WVN_OK = 0,
  WVN_ERR_INVALID = -1,   // bad argument / unsupported shape
  WVN_ERR_CUDA = -2,      // CUDA runtime / driver error (message in wvn_last_error())
  WVN_ERR_NO_DEVICE = -3, // no sm_90 device
  WVN_ERR_STATE = -4,     // handle in the wrong state (e.g. weights missing)
};

int set_error(int code, const char* fmt, ...);
const char* last_error();

#define WVN_CHECK_CUDA(expr)                                                                          \
  do {                                                                                                \
    cudaError_t _e = (expr);                                                                          \
    if (_e != cudaSuccess)                                                                            \
      return ::wvn::set_error(::wvn::WVN_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                              __FILE__, __LINE__);                                                    \
  } while (0)

#define WVN_CHECK_LAUNCH(name)                                                                        \
  do {                                                                                                \
    ::wvn::count_launch();                                                                            \
    cudaError_t _e = cudaGetLastError();                                                              \
    if (_e != cudaSuccess)                                                                            \
      return ::wvn::set_error(::wvn::WVN_ERR_CUDA, "launch of %s failed: %s (%s:%d)", name,           \
                              cudaGetErrorString(_e), __FILE__, __LINE__);                            \
  } while (0)

#define WVN_REQUIRE(cond, ...)                                                     \
  do {                                                                             \
    if (!(cond)) return ::wvn::set_error(::wvn::WVN_ERR_INVALID, __VA_ARGS__);     \
  } while (0)

#define WVN_PROPAGATE(expr)      \
  do {                           \
    int _r = (expr);             \
    if (_r != 0) return _r;      \
  } while (0)

// 2D bf16 row-major tensor [outer, inner] with row pitch `row_stride_bytes`, tiled in
// boxes of [box_outer, box_inner] with the 128-byte swizzle (box_inner must be 64).
int make_tmap_bf16_2d(CUtensorMap* out, const void* gptr, uint64_t inner, uint64_t outer,
                      uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer);

// Generic 2D row-major tensor map: elem_bytes in {2 (bf16), 4 (fp32)}; swizzle_bytes in {0, 64, 128}
// (the inner box must span exactly swizzle_bytes when swizzling).
int make_tmap_2d(CUtensorMap* out, const void* gptr, int elem_bytes, uint64_t inner, uint64_t outer,
                 uint64_t row_stride_bytes, uint32_t box_inner, uint32_t box_outer, int swizzle_bytes);

int sm_count();

// Kernel-launch counter (every launch of one of this library's kernels) and an optional
// CUDA-event profiler used by bench.py to time the dominant kernels inside a real step.
void count_launch();
long long launch_count();
enum ProfCategory : int { PROF_ATTENTION = 0, PROF_GEMM = 1, PROF_NUM = 2 };
void prof_enable(int category_mask);
void prof_begin(int cat, cudaStream_t s);
void prof_end(int cat, cudaStream_t s);
// Synchronises, sums elapsed ms per category, clears the record list.
int prof_collect(float* ms_by_cat, long long* launches_by_cat);

inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

// fp32 rows [rows, dim] -> bf16 rows `ld` apart on the device (the pad columns are left untouched), in at most
// `max_blocks` blocks of 256 threads.
int cast_rows_to_bf16(const float* src, void* dst, long long rows, int dim, long long ld, int max_blocks,
                      cudaStream_t s);

// Device memory that frees itself.  alloc() zero-fills (pitched rows rely on their pad columns being zero) and frees
// what the buffer held before.
struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;

  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
  ~DevBuf() { release(); }
  int alloc(size_t n);

 private:
  void release();
};

// One walk over a device arena's layout, run twice: with a null base the carver only counts bytes, with a base it
// hands out the same pieces in the same order.  Every piece starts on a 256-byte boundary.
struct Carver {
  char* base = nullptr;
  size_t bytes = 0;
  template <class T>
  T* take(size_t n) {   // n elements of T
    T* p = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
    bytes += (n * sizeof(T) + 255) / 256 * 256;
    return p;
  }
};
// Sizes `buf` by one layout walk, allocates it (zero-filled) and walks again to hand out the pointers.  A failure names
// `who`.
int carve(DevBuf* buf, const std::function<void(Carver&)>& layout, const char* who);

// A handle's named weights: device storage sized at create, filled by set() from fp32 host or device data.
struct WeightStore {
  struct Weight {
    DevBuf buf;            // fp32 dense, or bf16 rows of `cols` elements stored `ld` apart (pad columns zero)
    long long numel = 0;
    bool bf16 = false;
    bool loaded = false;
    int cols = 0, ld = 0;
  };
  std::map<std::string, Weight> w;
  DevBuf stage;            // host data on its way to a bf16 weight

  // `rows` x `cols` elements; bf16 rows are stored at the GEMM's W pitch gemm_w_pitch(cols)
  int add(const std::string& name, long long rows, int cols, bool bf16);
  // Copies fp32 `data` (host or device): fp32 storage as is, bf16 storage cast on the device into its pitched rows,
  // through `stage` when the source is host memory.  With `src_row`, stored row r is row src_row(r, rows) of `data`.
  int set(const char* name, const float* data, long long numel, long long (*src_row)(long long, long long) = nullptr);
  // null for a name that was never added
  template <class T>
  T* ptr(const std::string& name) const {
    auto it = w.find(name);
    return it == w.end() ? nullptr : reinterpret_cast<T*>(it->second.buf.p);
  }
  // WVN_ERR_STATE naming the first weight never set; names starting with `skip_prefix` (when given) are not checked
  int check_loaded(const char* what, const char* skip_prefix = nullptr) const;
};

}  // namespace wvn
