// Shared helpers of libnts_b200: error handling, launch accounting, vector types.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <functional>

#include "nts_b200.h"

namespace nts {

// thread-local last-error text (nts_last_error)
char *last_error_buffer();
bool abort_on_error();
void count_launch();

inline int fail(int code, const char *what, const char *file, int line) {
  snprintf(last_error_buffer(), 512, "%s (%s:%d)", what, file, line);
  if (abort_on_error()) {
    fprintf(stderr, "libnts_b200: %s\n", last_error_buffer());
    exit(1); // the reference's convention, cuda/ntsCUDAGraphOP.cu:13-19
  }
  return code;
}

#define NTS_CUDA_OK(expr)                                                                         \
  do {                                                                                            \
    cudaError_t nts_e_ = (expr);                                                                  \
    if (nts_e_ != cudaSuccess)                                                                    \
      return ::nts::fail((int)nts_e_, cudaGetErrorString(nts_e_), __FILE__, __LINE__);            \
  } while (0)

#define NTS_ARG_CHECK(cond, msg)                                                                  \
  do {                                                                                            \
    if (!(cond))                                                                                  \
      return ::nts::fail(-1, msg, __FILE__, __LINE__);                                            \
  } while (0)

// after every kernel launch: count it and surface launch-configuration errors
#define NTS_LAUNCH_CHECK()                                                                        \
  do {                                                                                            \
    ::nts::count_launch();                                                                        \
    NTS_CUDA_OK(cudaGetLastError());                                                              \
  } while (0)

inline cudaStream_t as_stream(void *s) { return reinterpret_cast<cudaStream_t>(s); }

inline bool aligned_to(const void *p, size_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

int sm_count();

// Minimum of two timed run() calls after one warm-up call, with CUDA events on st (synchronises).  Returns run()'s
// error, or nonzero when an event call fails.
int time_min_of_two(const std::function<int()> &run, cudaStream_t st, float *ms);

// Gathers of nts_plan.cu for the exchange engine, on rows of an explicit stride (lds elements of the input type);
// flags as for nts_gather_plan_run_ex / _run_bf16_ex (0: accumulate).  FP32 rows, and BF16 gathers of FP32 or BF16
// rows.  Plus the conversion pass that writes BF16 rows of stride ld (ld % 8 == 0, zero past F, dst 16-byte aligned).
int run_plan(nts_gather_plan *pl, const float *input, uint32_t lds, float *output, uint32_t F, int flags,
             cudaStream_t st);
int run_plan_bf16(nts_gather_plan *pl, const void *input, int dtype, uint32_t lds, float *output, uint32_t F,
                  cudaStream_t st, int flags = 0);
int to_bf16_rows(const void *src, int dtype, uint32_t lds, void *dst, uint32_t n_rows, uint32_t F, uint32_t ld,
                 cudaStream_t st);

// BF16 layout rule of the fused GAT layer (K7): rows of ld values, ld % 8 == 0 and >= F; with heads > 1 every head is a
// whole number of 16-byte chunks (D % 8 == 0) and ld == F.  Returns 0 or the argument error.
int check_gat_bf16_layout(uint32_t F, uint32_t ld, uint32_t heads);

struct __align__(16) float8v {
  float4 lo, hi;
};

template <int VEC> struct Vec;
template <> struct Vec<1> { using type = float; };
template <> struct Vec<2> { using type = float2; };
template <> struct Vec<4> { using type = float4; };
template <> struct Vec<8> { using type = float8v; };

// What one lane loads for VEC values of a row of element type T, and widen(), which turns it into the FP32 vector
// Vec<VEC>.  A BF16 value is the upper half of the FP32 with the same bits, so widening is exact (one shift or mask);
// for FP32 rows both are the identity.
template <class T, int VEC> struct Ld { using type = typename Vec<VEC>::type; };
template <> struct Ld<__nv_bfloat16, 2> { using type = uint32_t; };
template <> struct Ld<__nv_bfloat16, 4> { using type = uint2; };
template <> struct Ld<__nv_bfloat16, 8> { using type = uint4; };
__device__ __forceinline__ float widen(float v) { return v; }
__device__ __forceinline__ float2 widen(float2 v) { return v; }
__device__ __forceinline__ float4 widen(float4 v) { return v; }
__device__ __forceinline__ float2 widen(uint32_t u) {
  return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}
__device__ __forceinline__ float4 widen(uint2 u) {
  const float2 a = widen(u.x), b = widen(u.y);
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ float8v widen(uint4 u) { return {widen(make_uint2(u.x, u.y)), widen(make_uint2(u.z, u.w))}; }

// GAT attention logits (K7, K10): leaky_relu, and the segment maximum merged with one atomic
__device__ __forceinline__ float leaky(float x, float slope) { return x > 0.f ? x : x * slope; }
__device__ __forceinline__ void atomic_max_float(float *addr, float v) {
  // IEEE-754 order trick: non-negative floats order like signed ints, negative floats inversely like unsigned ints;
  // one `red` instead of a CAS loop (v + 0.f turns -0.0 into +0.0, NaN never reaches here)
  v += 0.f;
  if (v >= 0.f)
    atomicMax(reinterpret_cast<int *>(addr), __float_as_int(v));
  else
    atomicMin(reinterpret_cast<unsigned int *>(addr), __float_as_uint(v));
}

// A plan of parts (checked by the caller) with its slab count, and with hubs_allowed (a single part) its hub counts
// and schedule, chosen by timing candidates for width feature_size in run mode run_flags (0 or NTS_PLAN_OVERWRITE),
// as FP32 gathers or, with bf16, as BF16 gathers of BF16 rows (nts_plan.cu)
nts_gather_plan *tune_plan(const nts_plan_part *parts, int n_parts, nts_vid_t n_rows, nts_vid_t gather_rows,
                           nts_vid_t feature_size, bool bf16, int run_flags, bool hubs_allowed, cudaStream_t st);

} // namespace nts
