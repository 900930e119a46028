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

// The widest vector (4, 2 or 1 floats) that rows of F floats allow at every one of the pointers (a null one counts as
// aligned).  The width for several pointers is the minimum of their single widths.
template <class... P> inline int pick_vec(uint32_t F, const P *...p) {
  if (F % 4 == 0 && (aligned_to(p, 16) && ...))
    return 4;
  if (F % 2 == 0 && (aligned_to(p, 8) && ...))
    return 2;
  return 1;
}

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

// Arithmetic on the Vec<VEC> types: a = 0, a += w * x, *p += a (plain read-modify-write) and *p += a as no-return
// vector reductions (sm_90+: one L2 atomic transaction per 8 / 16 bytes)
__device__ __forceinline__ void zero_vec(float &a) { a = 0.f; }
__device__ __forceinline__ void zero_vec(float2 &a) { a = make_float2(0.f, 0.f); }
__device__ __forceinline__ void zero_vec(float4 &a) { a = make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ void zero_vec(float8v &a) {
  zero_vec(a.lo);
  zero_vec(a.hi);
}
__device__ __forceinline__ void fma_vec(float &a, float w, float x) { a = fmaf(w, x, a); }
__device__ __forceinline__ void fma_vec(float2 &a, float w, float2 x) {
  a.x = fmaf(w, x.x, a.x);
  a.y = fmaf(w, x.y, a.y);
}
__device__ __forceinline__ void fma_vec(float4 &a, float w, float4 x) {
  a.x = fmaf(w, x.x, a.x);
  a.y = fmaf(w, x.y, a.y);
  a.z = fmaf(w, x.z, a.z);
  a.w = fmaf(w, x.w, a.w);
}
__device__ __forceinline__ void fma_vec(float8v &a, float w, float8v x) {
  fma_vec(a.lo, w, x.lo);
  fma_vec(a.hi, w, x.hi);
}
__device__ __forceinline__ void rmw_add(float *p, float a) { *p = *p + a; }
__device__ __forceinline__ void rmw_add(float2 *p, float2 a) {
  float2 o = *p;
  o.x += a.x;
  o.y += a.y;
  *p = o;
}
__device__ __forceinline__ void rmw_add(float4 *p, float4 a) {
  float4 o = *p;
  o.x += a.x;
  o.y += a.y;
  o.z += a.z;
  o.w += a.w;
  *p = o;
}
__device__ __forceinline__ void rmw_add(float8v *p, float8v a) {
  rmw_add(&p->lo, a.lo);
  rmw_add(&p->hi, a.hi);
}
__device__ __forceinline__ void red_add(float *p, float a) { atomicAdd(p, a); }
__device__ __forceinline__ void red_add(float2 *p, float2 a) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a.x), "f"(a.y) : "memory");
}
__device__ __forceinline__ void red_add(float4 *p, float4 a) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a.x), "f"(a.y), "f"(a.z), "f"(a.w)
               : "memory");
}
__device__ __forceinline__ void red_add(float8v *p, float8v a) {
  red_add(&p->lo, a.lo);
  red_add(&p->hi, a.hi);
}

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

// One element of Parameter::learnC2G_with_decay_Adam (core/NtsScheduler.hpp:774-781), every operation explicitly
// rounded, in the reference's order:
//   W_g = W * weight_decay + grad;  M = beta1*M + (1-beta1)*W_g;  V = beta2*V + (1-beta2)*W_g*W_g;
//   W   = W - alpha * M / (sqrt(V) + epsilon)
// The dense update (nts_adam_update) and the embedding's row-sparse one (K11) both call it, so a row of either gets
// the same bits from the same inputs.
__device__ __forceinline__ void adam_element(float &w, float &m, float &v, float grad, float weight_decay, float beta1,
                                             float beta2, float alpha, float epsilon) {
  const float wg = __fadd_rn(__fmul_rn(w, weight_decay), grad);
  m = __fadd_rn(__fmul_rn(beta1, m), __fmul_rn(__fsub_rn(1.f, beta1), wg));
  v = __fadd_rn(__fmul_rn(beta2, v), __fmul_rn(__fmul_rn(__fsub_rn(1.f, beta2), wg), wg));
  w = __fsub_rn(w, __fdiv_rn(__fmul_rn(alpha, m), __fadd_rn(__fsqrt_rn(v), epsilon)));
}

// Segment search: the largest r in [0, n_rows) with off[r] <= e  (requires off[0] <= e < off[n_rows])
__device__ __forceinline__ uint32_t find_row(const uint32_t *__restrict__ off, uint32_t n_rows, uint32_t e) {
  uint32_t lo = 0, hi = n_rows; // invariant: off[lo] <= e < off[hi]
  while (hi - lo > 1) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (__ldg(off + mid) <= e)
      lo = mid;
    else
      hi = mid;
  }
  return lo;
}

// Tables sharded by global row ranges: shard o holds the ids [off[o], off[o+1]) of up to kMaxShards shards.
constexpr int kMaxShards = 32;

// The table's n_shards + 1 offsets and n_shards shard pointers staged in shared memory by the whole block; also(i)
// stages entry i of tables that share the offsets.
template <class P, class Also>
__device__ __forceinline__ void stage_shard_table(uint32_t *s_off, const P **s_shard, const uint32_t *__restrict__ off,
                                             const P *const *__restrict__ shards, int n_shards, Also also) {
  for (int i = threadIdx.x; i <= n_shards; i += blockDim.x) {
    s_off[i] = __ldg(off + i);
    if (i < n_shards) {
      s_shard[i] = shards[i];
      also(i);
    }
  }
  __syncthreads();
}
template <class P>
__device__ __forceinline__ void stage_shard_table(uint32_t *s_off, const P **s_shard, const uint32_t *__restrict__ off,
                                             const P *const *__restrict__ shards, int n_shards) {
  stage_shard_table(s_off, s_shard, off, shards, n_shards, [](int) {});
}

// The owner of id: the last shard o with s_off[o] <= id, so an empty shard (s_off[o] == s_off[o+1]) is never chosen
__device__ __forceinline__ int find_shard(const uint32_t *s_off, int n_shards, uint32_t id) {
  int lo = 0, hi = n_shards;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (s_off[mid] <= id)
      lo = mid;
    else
      hi = mid;
  }
  return lo;
}

// mbarrier / bulk-copy (TMA, SASS UBLKCP) PTX: global -> shared copies whose completion is counted on an mbarrier
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile("{\n\t"
               ".reg .pred p;\n\t"
               "WAIT_%=:\n\t"
               "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
               "@p bra DONE_%=;\n\t"
               "bra WAIT_%=;\n\t"
               "DONE_%=:\n\t"
               "}" ::"r"(smem_u32(bar)),
               "r"(parity)
               : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// The columns col .. col+3 (col < F) of a chunk that are < F, written into a row of an FP32 output of row stride F
// with stores of VEC floats (the output's rows are 16-byte aligned only when F % 4 == 0).  store_chunk_checked also
// checks the first column: the two forms compile differently unless the caller's own col < F check is visible.
template <int VEC> __device__ __forceinline__ void store_chunk(float *o, uint32_t col, uint32_t F, float4 a) {
  if constexpr (VEC == 4) {
    *reinterpret_cast<float4 *>(o + col) = a;
  } else if constexpr (VEC == 2) {
    *reinterpret_cast<float2 *>(o + col) = make_float2(a.x, a.y);
    if (col + 2 < F)
      *reinterpret_cast<float2 *>(o + col + 2) = make_float2(a.z, a.w);
  } else {
    o[col] = a.x;
    if (col + 1 < F)
      o[col + 1] = a.y;
    if (col + 2 < F)
      o[col + 2] = a.z;
    if (col + 3 < F)
      o[col + 3] = a.w;
  }
}
template <int VEC>
__device__ __forceinline__ void store_chunk_checked(float *__restrict__ o, uint32_t col, uint32_t F, float4 a) {
  if constexpr (VEC == 4) {
    *reinterpret_cast<float4 *>(o + col) = a;
  } else if constexpr (VEC == 2) {
    float2 *p = reinterpret_cast<float2 *>(o + col);
    p[0] = make_float2(a.x, a.y);
    if (col + 2 < F)
      p[1] = make_float2(a.z, a.w);
  } else {
    const float v[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int i = 0; i < 4; i++)
      if (col + i < F)
        o[col + i] = v[i];
  }
}
// *p += a: a plain read-modify-write when `whole` (the caller is the only writer), else a reduction
template <class V> __device__ __forceinline__ void add_vec(V *p, V a, bool whole) {
  if (whole)
    rmw_add(p, a);
  else
    red_add(p, a);
}
// o[col .. col+7] (+)= a for the columns < Fo of a row of Fo floats (K1 on BF16 rows: the output's width need not be a
// multiple of the 8-value chunk).  Whole chunks go as 16- or 8-byte vectors when Fo and the row allow them.
__device__ __forceinline__ void flush_cols(float *o, uint32_t col, uint32_t Fo, const float8v &a, bool whole) {
  const float v[8] = {a.lo.x, a.lo.y, a.lo.z, a.lo.w, a.hi.x, a.hi.y, a.hi.z, a.hi.w};
  const uintptr_t align = reinterpret_cast<uintptr_t>(o);
  if ((Fo & 3u) == 0 && (align & 15u) == 0) { // col and Fo multiples of 4: whole float4s
#pragma unroll
    for (int i = 0; i < 8; i += 4)
      if (col + i < Fo)
        add_vec(reinterpret_cast<float4 *>(o + col + i), make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]), whole);
  } else if ((Fo & 1u) == 0 && (align & 7u) == 0) {
#pragma unroll
    for (int i = 0; i < 8; i += 2)
      if (col + i < Fo)
        add_vec(reinterpret_cast<float2 *>(o + col + i), make_float2(v[i], v[i + 1]), whole);
  } else {
#pragma unroll
    for (int i = 0; i < 8; i++)
      if (col + i < Fo)
        add_vec(o + col + i, v[i], whole);
  }
}

// A plan of parts (checked by the caller) with its slab count, and with hubs_allowed (a single part) its hub counts
// and schedule, chosen by timing candidates for width feature_size in run mode run_flags (0 or NTS_PLAN_OVERWRITE),
// as FP32 gathers or, with bf16, as BF16 gathers of BF16 rows (nts_plan.cu)
nts_gather_plan *tune_plan(const nts_plan_part *parts, int n_parts, nts_vid_t n_rows, nts_vid_t gather_rows,
                           nts_vid_t feature_size, bool bf16, int run_flags, bool hubs_allowed, cudaStream_t st);

} // namespace nts
