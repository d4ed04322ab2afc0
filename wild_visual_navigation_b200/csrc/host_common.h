// wvn-b200: host-side helpers shared by the translation units of libwvn_b200.so
// (error reporting, TMA tensor-map encoding through the driver entry point).
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

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

}  // namespace wvn
