// Shared helpers of libnts_b200: error handling, launch accounting, vector types.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

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

// BF16 gathers of nts_plan.cu for the exchange engine: rows of an explicit stride (lds elements of the input type),
// and the conversion pass that writes BF16 rows of stride ld (ld % 8 == 0, zero past F, dst 16-byte aligned)
int run_plan_bf16(nts_gather_plan *pl, const void *input, int dtype, uint32_t lds, float *output, uint32_t F,
                  cudaStream_t st);
int to_bf16_rows(const void *src, int dtype, uint32_t lds, void *dst, uint32_t n_rows, uint32_t F, uint32_t ld,
                 cudaStream_t st);

template <int VEC> struct Vec;
template <> struct Vec<1> { using type = float; };
template <> struct Vec<2> { using type = float2; };
template <> struct Vec<4> { using type = float4; };

} // namespace nts

// nts_gather_plan_create_parts with the slab count measured on BF16 gathers when bf16 != 0 (nts_plan.cu)
extern "C" nts_gather_plan *nts_plan_create_parts_typed(const nts_plan_part *parts, int n_parts, nts_vid_t n_rows,
                                                        nts_vid_t gather_rows, int n_slabs, nts_vid_t feature_size,
                                                        int bf16, void *stream);
