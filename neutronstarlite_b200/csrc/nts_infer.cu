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
//
// K10 (full-neighbour inference of sampled GAT, DESIGN.md §3 K8) runs the same walk with the attention weight
//   a[e, h] = exp(leaky_relu(s[src(e), h] + d[r, h]) - seg_max[r, h]) / seg_sum[r, h]
// in place of w[e] (the ShardedAttention policy), after edge-balanced statistics passes over the same CSC piece whose
// source scores s are read by global id from a score table with the row table's shard offsets.
#include <algorithm>

#include "nts_common.cuh"

namespace nts {
namespace {

constexpr int kWarps = 8;

// a += w * (the 16-byte load v as FP32 values: 4 floats, or 8 BF16 values widened)
__device__ __forceinline__ void acc_add(float4 &a, float w, uint4 v, float) {
  fma_vec(a, w, make_float4(__uint_as_float(v.x), __uint_as_float(v.y), __uint_as_float(v.z), __uint_as_float(v.w)));
}
__device__ __forceinline__ void acc_add(float8v &a, float w, uint4 v, __nv_bfloat16) { fma_vec(a, w, widen(v)); }

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

// Weight policies of the walk.  The lane that stages an edge turns (edge, shard, local row) into a Staged value that
// the group's lanes take by shuffle; a lane turns it into one value per load k while the row loads are in flight
// (pre), and into the edge's weight for load k once the edge's row is current (weight).  load_row runs whenever the
// walk reaches a new row.
//
// PlainWeight (K9): w[e], or 1 when w is null.
template <int K> struct PlainWeight {
  static constexpr int kTables = 1; // shard tables staged in shared memory
  using Params = const float *; // w
  using Staged = float;
  static constexpr float kIdle = 1.f;
  Params p;
  template <uint32_t GS, uint32_t VEC> __device__ __forceinline__ void init(uint32_t, const bool *) {}
  __device__ __forceinline__ void stage_table(const unsigned char **, int) const {}
  __device__ __forceinline__ Staged stage(uint32_t e, uint32_t lane, const unsigned char *const *, int,
                                          uint32_t) const {
    return p ? __ldg(p + e + lane) : 1.f;
  }
  __device__ __forceinline__ float pre(Staged s, int) const { return s; }
  __device__ __forceinline__ void load_row(uint32_t) {}
  __device__ __forceinline__ float weight(float w, int) const { return w; }
};

// ShardedAttention (K10): a[e, h] = exp(leaky_relu(s[src(e), h] + d[row, h]) - m[row, h]) / z[row, h], h the head of
// load k.  The score table shares the row table's shard offsets, so the staging lane's shard search also gives the
// source's score row, whose address the lanes take by shuffle; each lane reads its own head's score.
struct AttentionParams {
  const unsigned char *const *score_shards;
  uint32_t score_row_bytes;
  const float *d, *m, *z; // [n_rows, H]: destination scores, segment maxima, segment sums
  uint32_t H, D;
  float slope;
};
template <int K> struct ShardedAttention {
  static constexpr int kTables = 2;
  using Params = AttentionParams;
  using Staged = unsigned long long; // address of the source's score row
  static constexpr unsigned long long kIdle = 0;
  Params p;
  uint32_t h[K]; // the head of each load
  float dk[K], mk[K], izk[K];

  // load k of a lane covers columns [(c0 + k * GS) * VEC, + VEC), inside one head
  template <uint32_t GS, uint32_t VEC> __device__ __forceinline__ void init(uint32_t c0, const bool *act) {
#pragma unroll
    for (int k = 0; k < K; k++)
      h[k] = act[k] ? (c0 + k * GS) * VEC / p.D : 0u;
  }
  __device__ __forceinline__ void stage_table(const unsigned char **s_score, int i) const {
    s_score[i] = p.score_shards[i];
  }
  __device__ __forceinline__ Staged stage(uint32_t, uint32_t, const unsigned char *const *s_score, int o,
                                          uint32_t local) const {
    return reinterpret_cast<unsigned long long>(s_score[o]) + (unsigned long long)local * p.score_row_bytes;
  }
  __device__ __forceinline__ float pre(Staged s, int k) const { return __ldg(reinterpret_cast<const float *>(s) + h[k]); }
  __device__ __forceinline__ void load_row(uint32_t row) {
#pragma unroll
    for (int k = 0; k < K; k++) {
      const size_t o = (size_t)row * p.H + h[k];
      dk[k] = __ldg(p.d + o);
      mk[k] = __ldg(p.m + o);
      izk[k] = 1.f / __ldg(p.z + o);
    }
  }
  __device__ __forceinline__ float weight(float s, int k) const {
    return expf(leaky(s + dk[k], p.slope) - mk[k]) * izk[k];
  }
};

// T: the shards' element type; W: the weight policy; K: 16-byte loads per lane per column tile; U: edges whose loads
// are issued before their FMAs; G: virtual warps per warp (K == 1 only); MINB: __launch_bounds__ min CTAs/SM
template <class T, template <int> class W, int K, int U, int G, int MINB>
__global__ void __launch_bounds__(kWarps * 32, MINB)
    sharded_gather_sum_kernel(float *__restrict__ out, const unsigned char *const *__restrict__ shards,
                              const uint32_t *__restrict__ shard_off, int n_shards, uint32_t row_bytes,
                              const typename W<K>::Params prm,
                              const uint32_t *__restrict__ idx, const uint32_t *__restrict__ off, uint32_t n_rows,
                              uint32_t e_begin, uint32_t e_end, uint32_t F, uint32_t Q, uint32_t tiles,
                              uint32_t tile_vecs, int svec) {
  static_assert(G == 1 || K == 1, "virtual warps hold one load per lane");
  constexpr uint32_t VEC = 16 / sizeof(T);
  constexpr uint32_t GS = 32 / G;
  using Acc = typename Vec<VEC>::type;
  using Staged = typename W<K>::Staged;
  W<K> wp{prm};
  __shared__ uint32_t s_off[kMaxShards + 1];
  __shared__ const unsigned char *s_shard[W<K>::kTables * kMaxShards]; // row shards, then the policy's
  stage_shard_table(s_off, s_shard, shard_off, shards, n_shards,
                    [&](int i) { wp.stage_table(s_shard + kMaxShards, i); });

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
  wp.template init<GS, VEC>(c0, act);

  uint32_t row = find_row(off, n_rows, e0);
  uint32_t row_end = __ldg(off + row + 1);
  bool row_started_inside = __ldg(off + row) >= e0;
  wp.load_row(row);
  Acc acc[K];
#pragma unroll
  for (int k = 0; k < K; k++)
    zero_vec(acc[k]);

  auto flush = [&](bool whole) {
    float *o = out + (size_t)row * F;
#pragma unroll
    for (int k = 0; k < K; k++) {
      if (act[k])
        flush_acc(o, (c0 + k * GS) * VEC, F, acc[k], svec, whole);
      zero_vec(acc[k]);
    }
  };
  auto advance = [&](uint32_t ee) { // ee >= row_end: the current row ends inside the quantum
    flush(row_started_inside);
    do {
      row++;
      row_end = __ldg(off + row + 1);
    } while (ee >= row_end);
    row_started_inside = true;
    wp.load_row(row);
  };

  for (uint32_t e = e0; e < e1; e += GS) {
    const uint32_t cnt = min(GS, e1 - e);
    unsigned long long my_row = 0;
    Staged my_w = W<K>::kIdle;
    if (lane < cnt) { // the edge's shard, once: binary search over the staged offsets
      const uint32_t id = __ldg(idx + e + lane);
      const int lo = find_shard(s_off, n_shards, id);
      my_row = reinterpret_cast<unsigned long long>(s_shard[lo]) + (unsigned long long)(id - s_off[lo]) * row_bytes;
      my_w = wp.stage(e, lane, s_shard + kMaxShards, lo, id - s_off[lo]);
    }
    uint32_t j = 0;
    for (; j + U <= cnt; j += U) {
      uint4 v[U][K];
      float wu[U][K];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const uint4 *p = reinterpret_cast<const uint4 *>(__shfl_sync(gmask, my_row, j + u, GS)) + c0;
        const Staged su = __shfl_sync(gmask, my_w, j + u, GS);
#pragma unroll
        for (int k = 0; k < K; k++) {
          if (act[k])
            v[u][k] = __ldg(p + k * GS);
          // pre() runs for idle loads too (head 0 of a real score row): K9's register allocation stays as it was
          wu[u][k] = wp.pre(su, k);
        }
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        if (e + j + u >= row_end)
          advance(e + j + u);
#pragma unroll
        for (int k = 0; k < K; k++)
          if (act[k])
            acc_add(acc[k], wp.weight(wu[u][k], k), v[u][k], T());
      }
    }
    for (; j < cnt; j++) {
      const uint4 *p = reinterpret_cast<const uint4 *>(__shfl_sync(gmask, my_row, j, GS)) + c0;
      const Staged sj = __shfl_sync(gmask, my_w, j, GS);
      uint4 v1[K];
      float w1[K];
#pragma unroll
      for (int k = 0; k < K; k++) {
        if (act[k])
          v1[k] = __ldg(p + k * GS);
        w1[k] = wp.pre(sj, k);
      }
      if (e + j >= row_end)
        advance(e + j);
#pragma unroll
      for (int k = 0; k < K; k++)
        if (act[k])
          acc_add(acc[k], wp.weight(w1[k], k), v1[k], T());
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

template <class T, template <int> class W, int K, int U, int G, int MINB>
int launch(const Shape &s, float *out, const void *const *shards, const uint32_t *shard_off, int n_shards,
           uint32_t row_bytes, const typename W<K>::Params &prm, const uint32_t *idx, const uint32_t *off,
           uint32_t n_rows, uint32_t e_begin, uint32_t e_end, uint32_t F, int svec, cudaStream_t st, const char *who) {
  // edges per virtual warp: 512 / G, halved (down to 32) until the grid has 64 virtual warps per SM
  uint32_t Q = 512u / G;
  const uint64_t n_edges = e_end - e_begin, want = (uint64_t)sm_count() * 64;
  while (Q > 32 && (n_edges + Q - 1) / Q * s.tiles < want)
    Q >>= 1;
  const uint64_t vwarps = (n_edges + Q - 1) / Q * s.tiles;
  const uint64_t blocks = (vwarps + kWarps * G - 1) / (kWarps * G);
  if (blocks > 0x7fffffffull)
    return fail(-1, who, __FILE__, __LINE__);
  sharded_gather_sum_kernel<T, W, K, U, G, MINB><<<(unsigned)blocks, kWarps * 32, 0, st>>>(
      out, reinterpret_cast<const unsigned char *const *>(shards), shard_off, n_shards, row_bytes, prm, idx, off,
      n_rows, e_begin, e_end, F, Q, s.tiles, s.tile_vecs, svec);
  NTS_LAUNCH_CHECK();
  return 0;
}

// who: the entry's name, for its errors
template <class T, template <int> class W>
int dispatch(float *out, const void *const *shards, const uint32_t *shard_off, int n_shards, uint32_t pitch,
             const typename W<1>::Params &prm, const uint32_t *idx, const uint32_t *off, uint32_t n_rows,
             uint32_t e_begin, uint32_t e_end, uint32_t F, cudaStream_t st, const char *who) {
  constexpr uint32_t VEC = 16 / sizeof(T);
  const Shape s = pick_shape((F + VEC - 1) / VEC);
  const int svec = pick_vec(F, out);
  const uint32_t row_bytes = pitch * (uint32_t)sizeof(T);
#define NTS_K9_CASE(K_, U_, G_, B_)                                                                                   \
  if (s.k == K_ && s.u == U_ && s.g == G_ && s.minb == B_)                                                          \
    return launch<T, W, K_, U_, G_, B_>(s, out, shards, shard_off, n_shards, row_bytes, prm, idx, off, n_rows,      \
                                        e_begin, e_end, F, svec, st, who);
  NTS_K9_CASE(1, 4, 4, 4)
  NTS_K9_CASE(1, 4, 2, 4)
  NTS_K9_CASE(1, 4, 1, 4)
  NTS_K9_CASE(2, 4, 1, 2)
  NTS_K9_CASE(3, 2, 1, 1)
  NTS_K9_CASE(4, 2, 1, 1)
#undef NTS_K9_CASE
  return fail(-1, who, __FILE__, __LINE__);
}

// ---- K10: softmax statistics over sharded scores ---------------------------------------------------------------
// gat_edge_stats_kernel's edge-balanced passes (nts_edge_ops.cu) on a CSC piece of absolute edge positions
// [e_begin, e_end) whose sources' scores are read by global id from score shards: lane = (edge slot el, head h), a
// warp owns a quantum of 512 consecutive edges whatever rows they belong to, and every lane merges its running
// (max | sum) with one atomic when its row changes or the quantum ends (combined over the warp first when the whole
// warp is in one row).  PASS 0: maxima onto -inf, PASS 1: sums of exp(logit - max) onto 0; the init pass presets
// both and gives empty segments (0, 1).  The H lanes of one edge search the same staged offsets (broadcast reads).
__global__ void __launch_bounds__(kWarps * 32)
    sharded_stats_init_kernel(float *__restrict__ seg_max, float *__restrict__ seg_sum,
                              const uint32_t *__restrict__ off, uint32_t n_rows, uint32_t H) {
  const uint64_t n = (uint64_t)n_rows * H;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t r = (uint32_t)(i / H);
    const bool empty = __ldg(off + r + 1) == __ldg(off + r);
    seg_max[i] = empty ? 0.f : -INFINITY;
    seg_sum[i] = empty ? 1.f : 0.f;
  }
}

template <int H, int PASS>
__global__ void __launch_bounds__(kWarps * 32)
    sharded_stats_kernel(float *__restrict__ seg_max, float *__restrict__ seg_sum,
                         const unsigned char *const *__restrict__ score_shards, const uint32_t *__restrict__ shard_off,
                         int n_shards, uint32_t score_row_bytes, const float *__restrict__ d_att,
                         const uint32_t *__restrict__ idx, const uint32_t *__restrict__ off, uint32_t n_rows,
                         uint32_t e_begin, uint32_t e_end, float slope) {
  static_assert(32 % H == 0, "H must divide the warp size");
  constexpr uint32_t kEdgesPerStep = 32 / H;
  constexpr int kUnroll = 4;
  constexpr uint32_t kQuantum = 512;
  __shared__ uint32_t s_off[kMaxShards + 1];
  __shared__ const unsigned char *s_shard[kMaxShards];
  stage_shard_table(s_off, s_shard, shard_off, score_shards, n_shards);

  const uint32_t lane = threadIdx.x & 31;
  const uint32_t h = lane % H, el = lane / H;
  const uint64_t nwarps = (uint64_t)gridDim.x * kWarps;
  for (uint64_t qw = (uint64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); e_begin + qw * kQuantum < e_end;
       qw += nwarps) {
    const uint32_t e0 = e_begin + (uint32_t)(qw * kQuantum);
    const uint32_t e1 = e_end - e0 > kQuantum ? e0 + kQuantum : e_end;
    uint32_t row = find_row(off, n_rows, e0);
    uint32_t row_end = __ldg(off + row + 1);
    float dv, mx = 0.f, acc;
    auto load_row = [&]() {
      dv = __ldg(d_att + (size_t)row * H + h);
      if (PASS == 1)
        mx = seg_max[(size_t)row * H + h]; // written by the previous launch
      acc = PASS == 0 ? -INFINITY : 0.f;
    };
    auto merge = [&](float v) {
      if (PASS == 0) {
        if (v > -INFINITY)
          atomic_max_float(seg_max + (size_t)row * H + h, v);
      } else if (v != 0.f) {
        atomicAdd(seg_sum + (size_t)row * H + h, v);
      }
    };
    auto score = [&](uint32_t e) {
      const uint32_t id = __ldg(idx + e);
      const int lo = find_shard(s_off, n_shards, id);
      return __ldg(reinterpret_cast<const float *>(s_shard[lo] + (size_t)(id - s_off[lo]) * score_row_bytes) + h);
    };
    load_row();
    for (uint32_t eb = e0 + el; eb < e1; eb += kEdgesPerStep * kUnroll) {
      float sv[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; u++) {
        const uint32_t e = eb + u * kEdgesPerStep;
        sv[u] = e < e1 ? score(e) : 0.f;
      }
#pragma unroll
      for (int u = 0; u < kUnroll; u++) {
        const uint32_t e = eb + u * kEdgesPerStep;
        if (e < e1) {
          if (e >= row_end) {
            merge(acc);
            do {
              row++;
              row_end = __ldg(off + row + 1);
            } while (e >= row_end);
            load_row();
          }
          const float x = leaky(sv[u] + dv, slope);
          acc = PASS == 0 ? fmaxf(acc, x) : acc + expf(x - mx);
        }
      }
    }
    // end of the quantum: when every lane is still in the same row, combine the lanes of one head first
    const uint32_t row0 = __shfl_sync(0xffffffffu, row, 0);
    if (__all_sync(0xffffffffu, row == row0)) {
#pragma unroll
      for (int o = 16; o >= H; o >>= 1) {
        const float other = __shfl_xor_sync(0xffffffffu, acc, o);
        acc = PASS == 0 ? fmaxf(acc, other) : acc + other;
      }
      if (el == 0)
        merge(acc);
    } else {
      merge(acc);
    }
  }
}

template <int H>
int launch_stats(float *seg_max, float *seg_sum, const void *const *score_shards, const uint32_t *shard_off,
                 int n_shards, uint32_t score_row_bytes, const float *d_att, const uint32_t *idx, const uint32_t *off,
                 uint32_t n_rows, uint32_t e_begin, uint32_t e_end, float slope, cudaStream_t st) {
  const auto sh = reinterpret_cast<const unsigned char *const *>(score_shards);
  const uint64_t quanta = (e_end - e_begin + 511) / 512;
  const unsigned grid = (unsigned)std::min<uint64_t>((quanta + kWarps - 1) / kWarps, (uint64_t)sm_count() * 16);
  sharded_stats_kernel<H, 0><<<grid, kWarps * 32, 0, st>>>(seg_max, seg_sum, sh, shard_off, n_shards,
                                                           score_row_bytes, d_att, idx, off, n_rows, e_begin, e_end,
                                                           slope);
  NTS_LAUNCH_CHECK();
  sharded_stats_kernel<H, 1><<<grid, kWarps * 32, 0, st>>>(seg_max, seg_sum, sh, shard_off, n_shards,
                                                           score_row_bytes, d_att, idx, off, n_rows, e_begin, e_end,
                                                           slope);
  NTS_LAUNCH_CHECK();
  return 0;
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
  static const char kWho[] = "nts_segment_gather_sum_sharded: no instantiation for this row width, or grid too large";
  if (shard_dtype == NTS_DTYPE_BF16)
    return nts::dispatch<__nv_bfloat16, nts::PlainWeight>(output, shards, shard_offsets, n_shards, shard_pitch,
                                                          {weight}, indices, offsets, n_rows, (uint32_t)edge_begin,
                                                          (uint32_t)edge_end, feature_size, st, kWho);
  return nts::dispatch<float, nts::PlainWeight>(output, shards, shard_offsets, n_shards, shard_pitch, {weight}, indices,
                                                offsets, n_rows, (uint32_t)edge_begin, (uint32_t)edge_end,
                                                feature_size, st, kWho);
}

// Layout checks K10's two entries share: the score shards (FP32 rows of score_pitch >= heads, score_pitch % 4 == 0)
// over the same 1..32 row ranges as the rows, uint32 edge positions.
static int check_k10(const char *who, const void *const *score_shards, const nts_vid_t *shard_offsets, int n_shards,
                     nts_vid_t score_pitch, const float *dst_score, const nts_vid_t *indices,
                     const nts_vid_t *offsets, uint64_t edge_end, nts_vid_t heads) {
  if (!(n_shards >= 1 && n_shards <= nts::kMaxShards))
    return nts::fail(-1, who, __FILE__, __LINE__);
  NTS_ARG_CHECK(heads >= 1 && score_pitch >= heads && score_pitch % 4 == 0,
                "K10: score_pitch must be >= heads >= 1 and a multiple of 4");
  NTS_ARG_CHECK(score_shards && shard_offsets && dst_score && indices && offsets, "null pointer passed to K10");
  NTS_ARG_CHECK(nts::aligned_to(score_shards, 8), "K10 needs an 8-byte aligned score shard array");
  NTS_ARG_CHECK(edge_end < 0xffffffffull, "K10: edge positions must fit uint32 offsets");
  NTS_ARG_CHECK((uint64_t)score_pitch * 4 < 0xffffffffull, "K10: score rows must be shorter than 4 GiB");
  return 0;
}

extern "C" int nts_gat_softmax_stats_sharded(float *seg_max, float *seg_sum, const void *const *score_shards,
                                             const nts_vid_t *shard_offsets, int n_shards, nts_vid_t score_pitch,
                                             const float *dst_score, const nts_vid_t *indices,
                                             const nts_vid_t *offsets, nts_vid_t n_rows, uint64_t edge_begin,
                                             uint64_t edge_end, nts_vid_t heads, float negative_slope, void *stream) {
  NTS_ARG_CHECK(edge_begin <= edge_end, "nts_gat_softmax_stats_sharded: edge range is reversed");
  if (n_rows == 0)
    return 0;
  if (const int rc = check_k10("nts_gat_softmax_stats_sharded needs 1..32 shards", score_shards, shard_offsets,
                               n_shards, score_pitch, dst_score, indices, offsets, edge_end, heads))
    return rc;
  NTS_ARG_CHECK(heads <= 32 && 32 % heads == 0, "nts_gat_softmax_stats_sharded: heads must divide 32");
  NTS_ARG_CHECK(seg_max && seg_sum, "null pointer passed to nts_gat_softmax_stats_sharded");
  cudaStream_t st = nts::as_stream(stream);
  const uint64_t n = (uint64_t)n_rows * heads;
  const unsigned grid = (unsigned)std::min<uint64_t>((n + 255) / 256, (uint64_t)nts::sm_count() * 16);
  nts::sharded_stats_init_kernel<<<grid, nts::kWarps * 32, 0, st>>>(seg_max, seg_sum, offsets, n_rows, heads);
  NTS_LAUNCH_CHECK();
  if (edge_begin == edge_end)
    return 0;
  const uint32_t rb = score_pitch * 4, eb = (uint32_t)edge_begin, ee = (uint32_t)edge_end;
#define NTS_K10_STATS(H_)                                                                                             \
  case H_:                                                                                                            \
    return nts::launch_stats<H_>(seg_max, seg_sum, score_shards, shard_offsets, n_shards, rb, dst_score, indices,    \
                                 offsets, n_rows, eb, ee, negative_slope, st);
  switch (heads) {
    NTS_K10_STATS(1)
    NTS_K10_STATS(2)
    NTS_K10_STATS(4)
    NTS_K10_STATS(8)
    NTS_K10_STATS(16)
    NTS_K10_STATS(32)
  }
#undef NTS_K10_STATS
  return 0;
}

extern "C" int nts_gat_aggregate_sharded(float *output, const void *const *shards, int shard_dtype,
                                         const nts_vid_t *shard_offsets, int n_shards, nts_vid_t shard_pitch,
                                         const void *const *score_shards, nts_vid_t score_pitch,
                                         const float *dst_score, const float *seg_max, const float *seg_sum,
                                         const nts_vid_t *indices, const nts_vid_t *offsets, nts_vid_t n_rows,
                                         uint64_t edge_begin, uint64_t edge_end, nts_vid_t feature_size,
                                         nts_vid_t heads, float negative_slope, void *stream) {
  NTS_ARG_CHECK(edge_begin <= edge_end, "nts_gat_aggregate_sharded: edge range is reversed");
  if (n_rows == 0 || edge_begin == edge_end || feature_size == 0)
    return 0;
  if (const int rc = check_k10("nts_gat_aggregate_sharded needs 1..32 shards", score_shards, shard_offsets, n_shards,
                               score_pitch, dst_score, indices, offsets, edge_end, heads))
    return rc;
  NTS_ARG_CHECK(shard_dtype == NTS_DTYPE_F32 || shard_dtype == NTS_DTYPE_BF16,
                "nts_gat_aggregate_sharded: shard_dtype must be NTS_DTYPE_F32 or NTS_DTYPE_BF16");
  const uint32_t VEC = shard_dtype == NTS_DTYPE_BF16 ? 8 : 4;
  NTS_ARG_CHECK(shard_pitch >= feature_size && shard_pitch % VEC == 0,
                "nts_gat_aggregate_sharded: shard_pitch must be >= feature_size and a multiple of 4 (FP32) or 8 (BF16) "
                "values");
  NTS_ARG_CHECK(feature_size % heads == 0, "nts_gat_aggregate_sharded: feature_size must be a multiple of heads");
  NTS_ARG_CHECK(heads == 1 || (feature_size / heads) % VEC == 0,
                "nts_gat_aggregate_sharded: with heads > 1 the head width must be a multiple of 4 (FP32) or 8 (BF16) "
                "values, so that every 16-byte load lies inside one head");
  NTS_ARG_CHECK(output && shards && seg_max && seg_sum, "null pointer passed to nts_gat_aggregate_sharded");
  NTS_ARG_CHECK(nts::aligned_to(output, 4) && nts::aligned_to(shards, 8),
                "nts_gat_aggregate_sharded needs a 4-byte aligned output and an 8-byte aligned shard array");
  NTS_ARG_CHECK((uint64_t)shard_pitch * (VEC == 8 ? 2 : 4) < 0xffffffffull,
                "nts_gat_aggregate_sharded: shard rows must be shorter than 4 GiB");
  const nts::AttentionParams prm = {reinterpret_cast<const unsigned char *const *>(score_shards), score_pitch * 4,
                                    dst_score, seg_max, seg_sum, heads, feature_size / heads, negative_slope};
  cudaStream_t st = nts::as_stream(stream);
  static const char kWho[] = "nts_gat_aggregate_sharded: no instantiation for this row width, or grid too large";
  if (shard_dtype == NTS_DTYPE_BF16)
    return nts::dispatch<__nv_bfloat16, nts::ShardedAttention>(output, shards, shard_offsets, n_shards, shard_pitch,
                                                               prm, indices, offsets, n_rows, (uint32_t)edge_begin,
                                                               (uint32_t)edge_end, feature_size, st, kWho);
  return nts::dispatch<float, nts::ShardedAttention>(output, shards, shard_offsets, n_shards, shard_pitch, prm,
                                                     indices, offsets, n_rows, (uint32_t)edge_begin,
                                                     (uint32_t)edge_end, feature_size, st, kWho);
}
