// Segmented weighted gather-sum whose sources are rows of a table sharded by global row ranges (K9, full-neighbour
// inference of sampled GCN, DESIGN.md §3 K9):
//
//   out[r, :F] += sum_{e in [off[r], off[r+1])} w[e] * row(idx[e]),   row(g) = shards[o][g - shard_off[o], :F]
//
// for the shard o with shard_off[o] <= g < shard_off[o+1].  The shards are those of feature_table.ShardedFeatureTable:
// up to 32 row ranges, local or peer memory, FP32 rows of a pitch % 4 == 0 or BF16 rows of a pitch % 8 == 0, every
// shard 16-byte aligned, so a lane always loads 16 bytes (4 FP32 or 8 BF16 values, widened exactly).
//
// The walk is K1's (nts_aggregate.cu): work is split by edges, a (virtual) warp owns the edge quantum [q*Q, (q+1)*Q)
// of one column tile, finds its first row by binary search over the offsets and keeps a register accumulator per lane;
// a row inside the quantum is written with one read-modify-write, a row cut by a quantum boundary is finished with
// vector `red.global.add`.  What differs is the staging of an edge: lane j of the group loads edge j's (index, weight),
// finds the index's shard once by binary search over the <= 33 offsets staged in shared memory, and forms the 64-bit
// address of the source row; the group's lanes then take (address, weight) by shuffle.  So the search runs once per
// edge and column tile, never once per lane.  Rows of at most 16 / 8 loads split a warp into G = 2 / 4 virtual warps
// with quanta of their own (rows of F = 41 are 11 FP32 or 6 BF16 loads), wider rows take K loads per lane and
// column tiles of at most 4 * 32 loads.
#include "nts_common.cuh"

namespace nts {
namespace {

constexpr int kWarps = 8;
constexpr int kMaxShards = 32;

__device__ __forceinline__ void acc_add(float4 &a, float w, uint4 v, float) {
  a.x = fmaf(w, __uint_as_float(v.x), a.x);
  a.y = fmaf(w, __uint_as_float(v.y), a.y);
  a.z = fmaf(w, __uint_as_float(v.z), a.z);
  a.w = fmaf(w, __uint_as_float(v.w), a.w);
}
__device__ __forceinline__ void acc_add(float8v &a, float w, uint4 v, __nv_bfloat16) {
  const float8v x = widen(v);
  a.lo.x = fmaf(w, x.lo.x, a.lo.x);
  a.lo.y = fmaf(w, x.lo.y, a.lo.y);
  a.lo.z = fmaf(w, x.lo.z, a.lo.z);
  a.lo.w = fmaf(w, x.lo.w, a.lo.w);
  a.hi.x = fmaf(w, x.hi.x, a.hi.x);
  a.hi.y = fmaf(w, x.hi.y, a.hi.y);
  a.hi.z = fmaf(w, x.hi.z, a.hi.z);
  a.hi.w = fmaf(w, x.hi.w, a.hi.w);
}
__device__ __forceinline__ void acc_zero(float4 &a) { a = make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ void acc_zero(float8v &a) {
  acc_zero(a.lo);
  acc_zero(a.hi);
}

__device__ __forceinline__ void add4(float *p, float4 a, bool whole) {
  if (whole) {
    float4 o = *reinterpret_cast<float4 *>(p);
    o.x += a.x;
    o.y += a.y;
    o.z += a.z;
    o.w += a.w;
    *reinterpret_cast<float4 *>(p) = o;
  } else {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a.x), "f"(a.y), "f"(a.z), "f"(a.w)
                 : "memory");
  }
}
__device__ __forceinline__ void add2(float *p, float a, float b, bool whole) {
  if (whole) {
    float2 o = *reinterpret_cast<float2 *>(p);
    o.x += a;
    o.y += b;
    *reinterpret_cast<float2 *>(p) = o;
  } else {
    asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
  }
}
__device__ __forceinline__ void add1(float *p, float a, bool whole) {
  if (whole)
    *p = *p + a;
  else
    atomicAdd(p, a);
}

// o[col .. col+3] (+)= a for the columns < F of a row; svec (4, 2 or 1, uniform over the launch) is the widest store
// that F and the output's alignment allow
__device__ __forceinline__ void flush4(float *o, uint32_t col, uint32_t F, float4 a, int svec, bool whole) {
  if (svec == 4) {
    add4(o + col, a, whole); // F % 4 == 0: a chunk is whole or entirely past F (not flushed)
  } else if (svec == 2) {
    add2(o + col, a.x, a.y, whole);
    if (col + 2 < F)
      add2(o + col + 2, a.z, a.w, whole);
  } else {
    add1(o + col, a.x, whole);
    if (col + 1 < F)
      add1(o + col + 1, a.y, whole);
    if (col + 2 < F)
      add1(o + col + 2, a.z, whole);
    if (col + 3 < F)
      add1(o + col + 3, a.w, whole);
  }
}
__device__ __forceinline__ void flush_acc(float *o, uint32_t col, uint32_t F, const float4 &a, int svec, bool whole) {
  flush4(o, col, F, a, svec, whole);
}
__device__ __forceinline__ void flush_acc(float *o, uint32_t col, uint32_t F, const float8v &a, int svec, bool whole) {
  flush4(o, col, F, a.lo, svec, whole);
  if (col + 4 < F)
    flush4(o, col + 4, F, a.hi, svec, whole);
}

// largest r in [0, n_rows) with off[r] <= e  (requires off[0] <= e < off[n_rows])
__device__ __forceinline__ uint32_t find_row(const uint32_t *__restrict__ off, uint32_t n_rows, uint32_t e) {
  uint32_t lo = 0, hi = n_rows;
  while (hi - lo > 1) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (__ldg(off + mid) <= e)
      lo = mid;
    else
      hi = mid;
  }
  return lo;
}

// T: the shards' element type; K: 16-byte loads per lane per column tile; U: edges whose loads are issued before
// their FMAs; G: virtual warps per warp (K == 1 only); MINB: __launch_bounds__ min CTAs/SM
template <class T, int K, int U, int G, int MINB>
__global__ void __launch_bounds__(kWarps * 32, MINB)
    sharded_gather_sum_kernel(float *__restrict__ out, const unsigned char *const *__restrict__ shards,
                              const uint32_t *__restrict__ shard_off, int n_shards, uint32_t row_bytes,
                              const float *__restrict__ w, const uint32_t *__restrict__ idx,
                              const uint32_t *__restrict__ off, uint32_t n_rows, uint32_t e_begin, uint32_t e_end,
                              uint32_t F, uint32_t Q, uint32_t tiles, uint32_t tile_vecs, int svec) {
  static_assert(G == 1 || K == 1, "virtual warps hold one load per lane");
  constexpr uint32_t VEC = 16 / sizeof(T);
  constexpr uint32_t GS = 32 / G;
  using Acc = typename Vec<VEC>::type;
  __shared__ uint32_t s_off[kMaxShards + 1];
  __shared__ const unsigned char *s_shard[kMaxShards];
  for (int i = threadIdx.x; i <= n_shards; i += blockDim.x) {
    s_off[i] = __ldg(shard_off + i);
    if (i < n_shards)
      s_shard[i] = shards[i];
  }
  __syncthreads();

  const uint32_t lane = threadIdx.x & (GS - 1);
  const unsigned gmask = G == 1 ? 0xffffffffu : (((1u << GS) - 1u) << ((threadIdx.x & 31u) & ~(GS - 1u)));
  const uint64_t gwarp = (uint64_t)blockIdx.x * (kWarps * G) + threadIdx.x / GS;
  const uint32_t tile = (uint32_t)(gwarp % tiles);
  const uint64_t e0_64 = e_begin + (gwarp / tiles) * (uint64_t)Q;
  if (e0_64 >= e_end)
    return;
  const uint32_t e0 = (uint32_t)e0_64;
  const uint32_t e1 = e_end - e0 > Q ? e0 + Q : e_end;

  const uint32_t nvec = (F + VEC - 1) / VEC;
  const uint32_t c0 = tile * tile_vecs + lane; // this lane's first load of a row
  bool act[K];
#pragma unroll
  for (int k = 0; k < K; k++)
    act[k] = k * GS + lane < tile_vecs && c0 + k * GS < nvec;

  uint32_t row = find_row(off, n_rows, e0);
  uint32_t row_end = __ldg(off + row + 1);
  bool row_started_inside = __ldg(off + row) >= e0;
  Acc acc[K];
#pragma unroll
  for (int k = 0; k < K; k++)
    acc_zero(acc[k]);

  auto flush = [&](bool whole) {
    float *o = out + (size_t)row * F;
#pragma unroll
    for (int k = 0; k < K; k++) {
      if (act[k])
        flush_acc(o, (c0 + k * GS) * VEC, F, acc[k], svec, whole);
      acc_zero(acc[k]);
    }
  };
  auto advance = [&](uint32_t ee) { // ee >= row_end: the current row ends inside the quantum
    flush(row_started_inside);
    do {
      row++;
      row_end = __ldg(off + row + 1);
    } while (ee >= row_end);
    row_started_inside = true;
  };

  for (uint32_t e = e0; e < e1; e += GS) {
    const uint32_t cnt = min(GS, e1 - e);
    unsigned long long my_row = 0;
    float my_w = 1.f;
    if (lane < cnt) { // the edge's shard, once: binary search over the staged offsets
      const uint32_t id = __ldg(idx + e + lane);
      int lo = 0, hi = n_shards;
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (s_off[mid] <= id)
          lo = mid;
        else
          hi = mid;
      }
      my_row = reinterpret_cast<unsigned long long>(s_shard[lo]) + (unsigned long long)(id - s_off[lo]) * row_bytes;
      if (w)
        my_w = __ldg(w + e + lane);
    }
    uint32_t j = 0;
    for (; j + U <= cnt; j += U) {
      uint4 v[U][K];
      float wu[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const uint4 *p = reinterpret_cast<const uint4 *>(__shfl_sync(gmask, my_row, j + u, GS)) + c0;
        wu[u] = __shfl_sync(gmask, my_w, j + u, GS);
#pragma unroll
        for (int k = 0; k < K; k++)
          if (act[k])
            v[u][k] = __ldg(p + k * GS);
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        if (e + j + u >= row_end)
          advance(e + j + u);
#pragma unroll
        for (int k = 0; k < K; k++)
          if (act[k])
            acc_add(acc[k], wu[u], v[u][k], T());
      }
    }
    for (; j < cnt; j++) {
      const uint4 *p = reinterpret_cast<const uint4 *>(__shfl_sync(gmask, my_row, j, GS)) + c0;
      const float wj = __shfl_sync(gmask, my_w, j, GS);
      uint4 v1[K];
#pragma unroll
      for (int k = 0; k < K; k++)
        if (act[k])
          v1[k] = __ldg(p + k * GS);
      if (e + j >= row_end)
        advance(e + j);
#pragma unroll
      for (int k = 0; k < K; k++)
        if (act[k])
          acc_add(acc[k], wj, v1[k], T());
    }
  }
  // the last row of the quantum is whole only if it started inside and ends at or before e1
  flush(row_started_inside && row_end <= e1);
}

struct Shape {
  int k, u, g, minb;
  uint32_t tiles, tile_vecs;
};

// One load per lane up to rows of 32 loads (G virtual warps for rows of <= 8 / 16), K <= 4 loads per lane beyond,
// in column tiles of at most 4 * 32 loads.  (U, MINB) follow K1's points for the same register footprint.
Shape pick_shape(uint32_t nvec) {
  Shape s;
  const uint32_t chunks = (nvec + 31) / 32;
  s.tiles = (chunks + 3) / 4;
  s.tile_vecs = (nvec + s.tiles - 1) / s.tiles;
  s.k = (int)((s.tile_vecs + 31) / 32);
  s.tiles = (nvec + s.tile_vecs - 1) / s.tile_vecs;
  s.g = s.k == 1 && s.tiles == 1 ? (nvec <= 8 ? 4 : (nvec <= 16 ? 2 : 1)) : 1;
  s.u = s.k <= 2 ? 4 : 2;
  s.minb = s.k == 1 ? 4 : (s.k == 2 ? 2 : 1);
  return s;
}

template <class T, int K, int U, int G, int MINB>
int launch(const Shape &s, float *out, const void *const *shards, const uint32_t *shard_off, int n_shards,
           uint32_t row_bytes, const float *w, const uint32_t *idx, const uint32_t *off, uint32_t n_rows,
           uint32_t e_begin, uint32_t e_end, uint32_t F, int svec, cudaStream_t st) {
  // edges per virtual warp: 512 / G, halved (down to 32) until the grid has 64 virtual warps per SM
  uint32_t Q = 512u / G;
  const uint64_t n_edges = e_end - e_begin, want = (uint64_t)sm_count() * 64;
  while (Q > 32 && (n_edges + Q - 1) / Q * s.tiles < want)
    Q >>= 1;
  const uint64_t vwarps = (n_edges + Q - 1) / Q * s.tiles;
  const uint64_t blocks = (vwarps + kWarps * G - 1) / (kWarps * G);
  NTS_ARG_CHECK(blocks <= 0x7fffffffull, "nts_segment_gather_sum_sharded: grid too large");
  sharded_gather_sum_kernel<T, K, U, G, MINB><<<(unsigned)blocks, kWarps * 32, 0, st>>>(
      out, reinterpret_cast<const unsigned char *const *>(shards), shard_off, n_shards, row_bytes, w, idx, off, n_rows,
      e_begin, e_end, F, Q, s.tiles, s.tile_vecs, svec);
  NTS_LAUNCH_CHECK();
  return 0;
}

template <class T>
int dispatch(float *out, const void *const *shards, const uint32_t *shard_off, int n_shards, uint32_t pitch,
             const float *w, const uint32_t *idx, const uint32_t *off, uint32_t n_rows, uint32_t e_begin,
             uint32_t e_end, uint32_t F, cudaStream_t st) {
  constexpr uint32_t VEC = 16 / sizeof(T);
  const Shape s = pick_shape((F + VEC - 1) / VEC);
  const int svec = (F % 4 == 0 && aligned_to(out, 16)) ? 4 : ((F % 2 == 0 && aligned_to(out, 8)) ? 2 : 1);
  const uint32_t row_bytes = pitch * (uint32_t)sizeof(T);
#define NTS_K9_CASE(K_, U_, G_, B_)                                                                                   \
  if (s.k == K_ && s.u == U_ && s.g == G_ && s.minb == B_)                                                          \
    return launch<T, K_, U_, G_, B_>(s, out, shards, shard_off, n_shards, row_bytes, w, idx, off, n_rows, e_begin,  \
                                     e_end, F, svec, st);
  NTS_K9_CASE(1, 4, 4, 4)
  NTS_K9_CASE(1, 4, 2, 4)
  NTS_K9_CASE(1, 4, 1, 4)
  NTS_K9_CASE(2, 4, 1, 2)
  NTS_K9_CASE(3, 2, 1, 1)
  NTS_K9_CASE(4, 2, 1, 1)
#undef NTS_K9_CASE
  return fail(-1, "nts_segment_gather_sum_sharded: no instantiation for this row width", __FILE__, __LINE__);
}

} // namespace
} // namespace nts

extern "C" int nts_segment_gather_sum_sharded(float *output, const void *const *shards, int shard_dtype,
                                              const nts_vid_t *shard_offsets, int n_shards, nts_vid_t shard_pitch,
                                              const float *weight, const nts_vid_t *indices, const nts_vid_t *offsets,
                                              nts_vid_t n_rows, uint64_t edge_begin, uint64_t edge_end,
                                              nts_vid_t feature_size, void *stream) {
  NTS_ARG_CHECK(edge_begin <= edge_end, "nts_segment_gather_sum_sharded: edge range is reversed");
  if (n_rows == 0 || edge_begin == edge_end || feature_size == 0)
    return 0;
  NTS_ARG_CHECK(shard_dtype == NTS_DTYPE_F32 || shard_dtype == NTS_DTYPE_BF16,
                "nts_segment_gather_sum_sharded: shard_dtype must be NTS_DTYPE_F32 or NTS_DTYPE_BF16");
  NTS_ARG_CHECK(shard_pitch >= feature_size && shard_pitch % (shard_dtype == NTS_DTYPE_BF16 ? 8 : 4) == 0,
                "nts_segment_gather_sum_sharded: shard_pitch must be >= feature_size and a multiple of 4 (FP32) or "
                "8 (BF16) values");
  NTS_ARG_CHECK(n_shards >= 1 && n_shards <= nts::kMaxShards, "nts_segment_gather_sum_sharded needs 1..32 shards");
  NTS_ARG_CHECK(output && shards && shard_offsets && indices && offsets,
                "null pointer passed to nts_segment_gather_sum_sharded");
  NTS_ARG_CHECK(nts::aligned_to(output, 4) && nts::aligned_to(shards, 8),
                "nts_segment_gather_sum_sharded needs a 4-byte aligned output and an 8-byte aligned shard array");
  NTS_ARG_CHECK(edge_end < 0xffffffffull, "nts_segment_gather_sum_sharded: edge positions must fit uint32 offsets");
  NTS_ARG_CHECK((uint64_t)shard_pitch * (shard_dtype == NTS_DTYPE_BF16 ? 2 : 4) < 0xffffffffull,
                "nts_segment_gather_sum_sharded: shard rows must be shorter than 4 GiB");
  cudaStream_t st = nts::as_stream(stream);
  if (shard_dtype == NTS_DTYPE_BF16)
    return nts::dispatch<__nv_bfloat16>(output, shards, shard_offsets, n_shards, shard_pitch, weight, indices, offsets,
                                        n_rows, (uint32_t)edge_begin, (uint32_t)edge_end, feature_size, st);
  return nts::dispatch<float>(output, shards, shard_offsets, n_shards, shard_pitch, weight, indices, offsets, n_rows,
                              (uint32_t)edge_begin, (uint32_t)edge_end, feature_size, st);
}
