// K8: neighbour sampling for mini-batch training (nts_sampler) - the blocks of the reference's SampledSubgraph
// (core/ntsSampler.hpp, core/FullyRepGraph.hpp) built on the GPU, deterministically.
//
// Per hop, with n_dst destinations and fanout k:
//   count    one thread per destination: min(indeg, k); a CUB exclusive scan gives the block's column_offset
//   select   one warp per destination: every slot when indeg <= k, else Floyd's k-subset of the slots drawn from a
//            counter hash of (seed, step, hop, global dst, j), written in ascending slot order; every kept edge's global
//            source id and weight go to the block, and (source id, edge position) to a padded n_dst * k pair array
//            whose unused pairs carry the key V
//   sort     one stable CUB radix sort of the pairs by source id
//   finish   head flags + an inclusive scan number the distinct sources in ascending id order: the next hop's
//            destinations, each edge's local source id, and the transposed block (the sorted order is the transposed
//            edge order, stable by edge position), in one pass
// then one 12-byte device-to-host copy (edge count, source count, bad-seed flag) sizes the next hop.  No atomics on
// floats anywhere; the only atomic is the bad-seed flag.
//
// NTS_SAMPLER_INCLUDE_DST: the count pass also appends one marker pair (destination id, kMarker | i) per destination
// after the n_dst * k edge pairs, so the same sort puts every destination among the sources; the stable sort leaves a
// key's markers after its edges.  One inclusive scan over 64-bit flags (head count in the high word, marker count in
// the low word) gives each pair its local source id and each edge pair its transposed position (sorted position minus
// the markers before it), so the transposed block is still stable by edge position.  Markers write dst_pos.
//
// nts_sampler_create_sharded: count and select read a destination's CSC from the shard that owns it (ShardTable);
// the draws use the global destination id, so the blocks are those of the whole-graph sampler.
#include <cub/cub.cuh>

#include <vector>

#include "nts_common.cuh"

namespace {

using u32 = uint32_t;
using u64 = uint64_t;

constexpr int kMaxFanout = 64;
constexpr int kMaxHops = 8;
constexpr int kSelectWarps = 8;
constexpr int kThreads = 256;
using nts::kMaxShards;               // nts_sampler_create_sharded
constexpr u32 kMarker = 0x80000000u;   // value bit of a destination marker pair (edge positions are < 2^31)

__host__ __device__ __forceinline__ u64 splitmix64(u64 z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// The CSC sharded by destination ranges (nts_sampler_create_sharded): shard o holds destinations [off[o], off[o+1])
// with local column offsets; row ids are global.  The table lives in the sampler's device memory.  count_kernel and
// select_kernel take it as a last parameter, unused (null) by their whole-graph instantiations, whose code is that of
// the whole-graph kernels they were before the sharded twins existed.
struct ShardTable {
  u32 n;
  u32 off[kMaxShards + 1];
  const u32 *col[kMaxShards];
  const u32 *row[kMaxShards];
  const float *w[kMaxShards];
};

// The table staged in shared memory, once per block and before any thread of the block returns.
__device__ __forceinline__ const ShardTable &stage_shards(const ShardTable *__restrict__ table) {
  __shared__ ShardTable s;
  const u32 n = table->n;
  for (u32 i = threadIdx.x; i <= n; i += blockDim.x) {
    s.off[i] = table->off[i];
    if (i < n) {
      s.col[i] = table->col[i];
      s.row[i] = table->row[i];
      s.w[i] = table->w[i];
    }
  }
  if (threadIdx.x == 0) s.n = n;
  __syncthreads();
  return s;
}

// The owner of v < V is the last shard with off[o] <= v, so an empty shard (off[o] == off[o+1]) is never chosen; v's
// in-edges are slots [base, base + deg) of the owner's row / w.
__device__ __forceinline__ int shard_of(const ShardTable &t, u32 v, u32 &base, u32 &deg) {
  const int lo = nts::find_shard(t.off, (int)t.n, v);
  const u32 lv = v - t.off[lo];
  base = t.col[lo][lv];
  deg = t.col[lo][lv + 1] - base;
  return lo;
}

template <bool kSharded>
__global__ void count_kernel(const u32 *__restrict__ dst, u32 n_dst, const u32 *__restrict__ g_col, u32 V, u32 k,
                             u32 *__restrict__ cnt, u32 *__restrict__ bad, u32 *__restrict__ marker_keys,
                             u32 *__restrict__ marker_vals, const ShardTable *__restrict__ shards) {
  const ShardTable *t = nullptr;
  if constexpr (kSharded) t = &stage_shards(shards);
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n_dst) return;
  u32 c = 0;
  if (i < n_dst) {
    const u32 v = dst[i];
    if (v < V) {
      u32 deg;
      if constexpr (kSharded) {
        u32 base;
        shard_of(*t, v, base, deg);
      } else {
        deg = g_col[v + 1] - g_col[v];
      }
      c = min(deg, k);
    } else {
      atomicOr(bad, 1u);
    }
    if (marker_keys) {            // NTS_SAMPLER_INCLUDE_DST; a bad id sorts with the unused pairs
      marker_keys[i] = min(v, V);
      marker_vals[i] = kMarker | (u32)i;
    }
  }
  cnt[i] = c;   // cnt[n_dst] = 0: the exclusive scan's last element is the edge count
}

template <bool kSharded>
__global__ void __launch_bounds__(kSelectWarps * 32)
select_kernel(const u32 *__restrict__ dst, u32 n_dst, const u32 *__restrict__ g_col, const u32 *__restrict__ g_row,
              const float *__restrict__ g_w, u32 V, u32 k, u64 step_key, u32 hop, const u32 *__restrict__ col,
              u32 *__restrict__ row_global, float *__restrict__ weight, u32 *__restrict__ edge_dst,
              u32 *__restrict__ keys, u32 *__restrict__ vals, const ShardTable *__restrict__ shards) {
  __shared__ u32 chosen[kSelectWarps][kMaxFanout];
  const ShardTable *t = nullptr;
  if constexpr (kSharded) t = &stage_shards(shards);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const u32 d = blockIdx.x * kSelectWarps + warp;
  if (d >= n_dst) return;   // warp-uniform
  const u32 v = dst[d];
  u32 base = 0, deg = 0;
  const u32 *row = g_row;
  const float *w = g_w;
  if (v < V) {
    if constexpr (kSharded) {
      const int o = shard_of(*t, v, base, deg);
      row = t->row[o];
      w = t->w[o];
    } else {
      base = g_col[v];
      deg = g_col[v + 1] - base;
    }
  }
  const u32 e0 = col[d];
  const u64 p0 = (u64)d * k;
  auto emit = [&](u32 i, u32 slot) {
    const u32 e = e0 + i;
    const u32 s = row[base + slot];
    row_global[e] = s;
    weight[e] = w[base + slot];
    edge_dst[e] = d;
    keys[p0 + i] = s;
    vals[p0 + i] = e;
  };
  const u32 kept = min(deg, k);
  if (deg <= k) {
    for (u32 i = lane; i < deg; i += 32) emit(i, i);
  } else {
    // Floyd: for j = deg-k .. deg-1, t = draw(j+1); add j if t is already chosen, else t.  Every lane computes the
    // same draw; the membership test is spread over the lanes.
    u32 *S = chosen[warp];
    const u64 dst_key = splitmix64(step_key ^ (((u64)hop << 32) | v));
    for (u32 i = 0; i < k; ++i) {
      const u32 j = deg - k + i;
      const u32 h = (u32)(splitmix64(dst_key ^ (u64)j) >> 32);
      const u32 t = (u32)(((u64)h * (u64)(j + 1)) >> 32);
      bool hit = false;
      for (u32 q = lane; q < i; q += 32) hit |= S[q] == t;
      hit = __any_sync(0xffffffffu, hit);
      if (lane == 0) S[i] = hit ? j : t;
      __syncwarp();
    }
    // ascending slot order: the chosen slots are distinct, so a slot's rank is the number of smaller ones
    for (u32 a = lane; a < k; a += 32) {
      const u32 x = S[a];
      u32 r = 0;
      for (u32 b = 0; b < k; ++b) r += S[b] < x;
      emit(r, x);
    }
  }
  for (u32 i = kept + lane; i < k; i += 32) keys[p0 + i] = V;   // unused pairs sort past every source id
}

__global__ void head_kernel(const u32 *__restrict__ skeys, u64 n_pad, const u32 *__restrict__ col, u32 n_dst,
                            u32 *__restrict__ flag) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pad) return;
  flag[i] = i < col[n_dst] && (i == 0 || skeys[i] != skeys[i - 1]);
}

__global__ void finish_kernel(const u32 *__restrict__ skeys, const u32 *__restrict__ svals,
                              const u32 *__restrict__ pos, u64 n_pad, const u32 *__restrict__ col, u32 n_dst,
                              const u32 *__restrict__ edge_dst, const float *__restrict__ weight,
                              u32 *__restrict__ row_local, u32 *__restrict__ src, u32 *__restrict__ row_offset,
                              u32 *__restrict__ col_t, float *__restrict__ w_t, u32 *__restrict__ counts) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  const u32 n_edges = col[n_dst];
  if (i == 0 && n_edges == 0) {
    row_offset[0] = 0;
    counts[0] = 0;
    counts[1] = 0;
  }
  if (i >= n_edges || i >= n_pad) return;
  const u32 l = pos[i] - 1, e = svals[i];
  row_local[e] = l;
  col_t[i] = edge_dst[e];
  w_t[i] = weight[e];
  if (i == 0 || skeys[i] != skeys[i - 1]) {
    src[l] = skeys[i];
    row_offset[l] = (u32)i;
  }
  if (i + 1 == n_edges) {
    row_offset[l + 1] = n_edges;
    counts[0] = n_edges;
    counts[1] = l + 1;
  }
}

// NTS_SAMPLER_INCLUDE_DST: flag[i] = (head << 32) | marker over the n_tot sorted pairs; keys >= V (unused pairs, bad
// seeds) are neither
__global__ void head_dst_kernel(const u32 *__restrict__ skeys, const u32 *__restrict__ svals, u64 n_tot, u32 V,
                                u64 *__restrict__ flag) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_tot) return;
  const u32 key = skeys[i];
  const bool valid = key < V;
  const bool head = valid && (i == 0 || key != skeys[i - 1]);
  const bool marker = valid && (svals[i] & kMarker);
  flag[i] = ((u64)head << 32) | (u64)marker;
}

__global__ void finish_dst_kernel(const u32 *__restrict__ skeys, const u32 *__restrict__ svals,
                                  const u64 *__restrict__ pos, u64 n_tot, const u32 *__restrict__ col, u32 n_dst,
                                  u32 V, const u32 *__restrict__ edge_dst, const float *__restrict__ weight,
                                  u32 *__restrict__ row_local, u32 *__restrict__ src, u32 *__restrict__ row_offset,
                                  u32 *__restrict__ col_t, float *__restrict__ w_t, u32 *__restrict__ dst_pos,
                                  u32 *__restrict__ counts) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  const u32 n_edges = col[n_dst];
  if (i == 0 && (n_tot == 0 || skeys[0] >= V)) {
    row_offset[0] = 0;
    counts[0] = 0;
    counts[1] = 0;
  }
  if (i >= n_tot) return;
  const u32 key = skeys[i];
  if (key >= V) return;
  const u64 p = pos[i];
  const u32 l = (u32)(p >> 32) - 1, val = svals[i];
  const u32 mk = val >> 31;
  const u32 t = (u32)i - (u32)p + mk;   // edge pairs before sorted position i: its transposed position
  if (mk) {
    dst_pos[val & ~kMarker] = l;
  } else {
    row_local[val] = l;
    col_t[t] = edge_dst[val];
    w_t[t] = weight[val];
  }
  if (i == 0 || key != skeys[i - 1]) {
    src[l] = key;
    row_offset[l] = t;
  }
  if (i + 1 == n_tot || skeys[i + 1] >= V) {
    row_offset[l + 1] = n_edges;
    counts[0] = n_edges;
    counts[1] = l + 1;
  }
}

// nts_sample_transpose: the destination of every edge, and lower bounds of each source in the sorted keys
__global__ void edge_dst_kernel(const u32 *__restrict__ col, u32 n_dst, u32 *__restrict__ edge_dst,
                                u32 *__restrict__ iota) {
  const u32 d = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
  if (d >= n_dst) return;
  for (u32 e = col[d] + (threadIdx.x & 31); e < col[d + 1]; e += 32) {
    edge_dst[e] = d;
    iota[e] = e;
  }
}

__global__ void lower_bound_kernel(const u32 *__restrict__ skeys, u64 n, u32 n_src, u32 *__restrict__ row_offset) {
  const u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (s > n_src) return;
  u64 lo = 0, hi = n;
  while (lo < hi) {
    const u64 mid = (lo + hi) >> 1;
    if (skeys[mid] < s) lo = mid + 1; else hi = mid;
  }
  row_offset[s] = (u32)lo;
}

__global__ void permute_kernel(const u32 *__restrict__ svals, u64 n, const u32 *__restrict__ edge_dst,
                               const float *__restrict__ weight, u32 *__restrict__ col_t, float *__restrict__ w_t) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u32 e = svals[i];
  col_t[i] = edge_dst[e];
  w_t[i] = weight[e];
}

// nts_merge_chunk_csc: a rank's chunk CSCs (same destinations, chunk o's sources before chunk o+1's) merged into
// one CSC per destination in chunk order.  count: each destination's in-degree over the chunks; a scan; copy: a warp
// per destination appends each chunk's slots.
struct ChunkCscs {
  int n;
  const u32 *col[kMaxShards];
  const u32 *row[kMaxShards];
  const float *w[kMaxShards];
};

__global__ void merge_count_kernel(const ChunkCscs c, u32 n_dst, u32 *__restrict__ deg, u32 *__restrict__ bad) {
  const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n_dst) return;
  u32 n = 0;
  if (i < n_dst)
    for (int o = 0; o < c.n; ++o) {
      const u32 d = c.col[o][i + 1] - c.col[o][i];
      if (d && (!c.row[o] || !c.w[o])) atomicOr(bad, 1u);   // a chunk with edges passed without its arrays
      n += d;
    }
  deg[i] = n;   // deg[n_dst] = 0: the exclusive scan's last element is the edge count
}

__global__ void merge_copy_kernel(const ChunkCscs c, u32 n_dst, const u32 *__restrict__ out_col,
                                  u32 *__restrict__ out_row, float *__restrict__ out_w) {
  const u32 d = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (d >= n_dst) return;
  u32 e = out_col[d];
  for (int o = 0; o < c.n; ++o) {
    const u32 b = c.col[o][d], n = c.col[o][d + 1] - b;
    for (u32 j = lane; j < n; j += 32) {
      out_row[e + j] = c.row[o][b + j];
      out_w[e + j] = c.w[o][b + j];
    }
    e += n;
  }
}

inline unsigned blocks_for(u64 n, int threads = kThreads) { return (unsigned)((n + threads - 1) / threads); }

inline int bits_for(u32 v) {
  int b = 1;
  while (b < 32 && (v >> b) != 0) ++b;
  return b;
}

} // namespace

struct nts_sampler {
  const u32 *g_col = nullptr, *g_row = nullptr;
  const float *g_w = nullptr;
  ShardTable *shards = nullptr;   // nts_sampler_create_sharded: the shard table in device memory, else null
  u32 V = 0;
  u32 max_seeds = 0;
  int hops = 0;
  bool include_dst = false;   // NTS_SAMPLER_INCLUDE_DST
  u32 fanout[kMaxHops] = {};
  u64 cap_dst[kMaxHops] = {}, cap_pad[kMaxHops] = {}, cap_src[kMaxHops] = {};
  struct Hop {
    u32 *dst = nullptr, *col = nullptr, *row_local = nullptr, *row_global = nullptr, *edge_dst = nullptr;
    float *weight = nullptr, *w_t = nullptr;
    u32 *src = nullptr, *row_offset = nullptr, *col_t = nullptr;
    u32 *dst_pos = nullptr;   // include_dst only
    u32 n_dst = 0, n_src = 0;
    u64 n_edges = 0;
  } hop[kMaxHops];
  bool sampled = false;
  // scratch shared by the hops
  u32 *cnt = nullptr, *keys = nullptr, *keys_alt = nullptr, *vals = nullptr, *vals_alt = nullptr, *flag = nullptr,
      *pos = nullptr, *counts = nullptr;
  u64 *flag64 = nullptr, *pos64 = nullptr;   // include_dst: replace flag / pos
  void *tmp = nullptr;
  size_t tmp_bytes = 0;
  u32 *counts_host = nullptr;
  std::vector<void *> allocs;
  u64 bytes = 0;

  template <class T> int alloc(T **p, u64 n) {
    const size_t b = (size_t)std::max<u64>(n, 1) * sizeof(T);
    NTS_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(p), b));
    allocs.push_back(*p);
    bytes += b;
    return 0;
  }
  ~nts_sampler() {
    for (void *p : allocs) cudaFree(p);
    if (counts_host) cudaFreeHost(counts_host);
  }
};

namespace {

int sampler_setup(nts_sampler *s, cudaStream_t st) {
  u64 max_dst = 0, max_pad = 0;
  for (int h = 0; h < s->hops; ++h) {
    s->cap_dst[h] = h == 0 ? s->max_seeds : s->cap_src[h - 1];
    // include_dst: one marker pair per destination after the edge pairs, and up to n_dst more sources
    s->cap_pad[h] = s->cap_dst[h] * (s->fanout[h] + (s->include_dst ? 1 : 0));
    s->cap_src[h] = std::min<u64>(s->V, s->cap_pad[h]);
    NTS_ARG_CHECK(s->cap_pad[h] < (1ull << 31),
                  s->include_dst ? "sampler worst case n_dst * (fanout + 1) reaches 2^31 pairs in one hop"
                                 : "sampler worst case n_dst * fanout reaches 2^31 edges in one hop");
    max_dst = std::max(max_dst, s->cap_dst[h]);
    max_pad = std::max(max_pad, s->cap_pad[h]);
  }
  for (int h = 0; h < s->hops; ++h) {
    nts_sampler::Hop &H = s->hop[h];
    if (h == 0) {
      if (int rc = s->alloc(&H.dst, s->cap_dst[0])) return rc;
    } else {
      H.dst = s->hop[h - 1].src;
    }
    const u64 E = s->cap_pad[h], S = s->cap_src[h];
    int rc = 0;
    if ((rc = s->alloc(&H.col, s->cap_dst[h] + 1)) || (rc = s->alloc(&H.row_local, E)) ||
        (rc = s->alloc(&H.row_global, E)) || (rc = s->alloc(&H.edge_dst, E)) || (rc = s->alloc(&H.weight, E)) ||
        (rc = s->alloc(&H.w_t, E)) || (rc = s->alloc(&H.col_t, E)) || (rc = s->alloc(&H.src, S)) ||
        (rc = s->alloc(&H.row_offset, S + 1)))
      return rc;
    if (s->include_dst && (rc = s->alloc(&H.dst_pos, s->cap_dst[h]))) return rc;
  }
  int rc = 0;
  if ((rc = s->alloc(&s->cnt, max_dst + 1)) || (rc = s->alloc(&s->keys, max_pad)) ||
      (rc = s->alloc(&s->keys_alt, max_pad)) || (rc = s->alloc(&s->vals, max_pad)) ||
      (rc = s->alloc(&s->vals_alt, max_pad)) || (rc = s->alloc(&s->counts, 4)))
    return rc;
  if (s->include_dst) {
    if ((rc = s->alloc(&s->flag64, max_pad)) || (rc = s->alloc(&s->pos64, max_pad))) return rc;
  } else if ((rc = s->alloc(&s->flag, max_pad)) || (rc = s->alloc(&s->pos, max_pad))) {
    return rc;
  }
  // CUB scratch for the largest scan and sort (queried again, and checked, at every call)
  size_t b0 = 0, b1 = 0, b2 = 0;
  cub::DoubleBuffer<u32> kd(s->keys, s->keys_alt), vd(s->vals, s->vals_alt);
  NTS_CUDA_OK(cub::DeviceScan::ExclusiveSum(nullptr, b0, s->cnt, s->cnt, (int64_t)(max_dst + 1), st));
  if (s->include_dst)
    NTS_CUDA_OK(cub::DeviceScan::InclusiveSum(nullptr, b1, s->flag64, s->pos64, (int64_t)std::max<u64>(max_pad, 1),
                                              st));
  else
    NTS_CUDA_OK(cub::DeviceScan::InclusiveSum(nullptr, b1, s->flag, s->pos, (int64_t)std::max<u64>(max_pad, 1), st));
  NTS_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, b2, kd, vd, (int64_t)std::max<u64>(max_pad, 1), 0, 32, st));
  s->tmp_bytes = std::max(b0, std::max(b1, b2));
  if ((rc = s->alloc(reinterpret_cast<char **>(&s->tmp), s->tmp_bytes))) return rc;
  NTS_CUDA_OK(cudaMallocHost(reinterpret_cast<void **>(&s->counts_host), 4 * sizeof(u32)));
  return 0;
}

int check_tmp(const nts_sampler *s, size_t need) {
  NTS_ARG_CHECK(need <= s->tmp_bytes, "sampler CUB scratch smaller than a call needs");
  return 0;
}

template <class T> int inclusive_sum(nts_sampler *s, const T *in, T *out, u64 n, cudaStream_t st) {
  size_t need = 0;
  NTS_CUDA_OK(cub::DeviceScan::InclusiveSum(nullptr, need, in, out, (int64_t)n, st));
  if (int rc = check_tmp(s, need)) return rc;
  NTS_CUDA_OK(cub::DeviceScan::InclusiveSum(s->tmp, need, in, out, (int64_t)n, st));
  return 0;
}

int sample_hop(nts_sampler *s, int h, u64 step_key, cudaStream_t st) {
  nts_sampler::Hop &H = s->hop[h];
  const u32 n_dst = H.n_dst, k = s->fanout[h];
  const bool inc = s->include_dst;
  const u64 n_pad = (u64)n_dst * k;
  const u64 n_sort = inc ? n_pad + n_dst : n_pad;   // include_dst: the marker pairs follow the edge pairs
  u32 *const mk = inc ? s->keys + n_pad : nullptr, *const mv = inc ? s->vals + n_pad : nullptr;
  const unsigned count_grid = blocks_for((u64)n_dst + 1);
  if (s->shards)
    count_kernel<true><<<count_grid, kThreads, 0, st>>>(H.dst, n_dst, nullptr, s->V, k, s->cnt, s->counts + 2, mk, mv,
                                                        s->shards);
  else
    count_kernel<false><<<count_grid, kThreads, 0, st>>>(H.dst, n_dst, s->g_col, s->V, k, s->cnt, s->counts + 2, mk,
                                                         mv, nullptr);
  NTS_LAUNCH_CHECK();
  size_t need = 0;
  NTS_CUDA_OK(cub::DeviceScan::ExclusiveSum(nullptr, need, s->cnt, H.col, (int64_t)n_dst + 1, st));
  if (int rc = check_tmp(s, need)) return rc;
  NTS_CUDA_OK(cub::DeviceScan::ExclusiveSum(s->tmp, need, s->cnt, H.col, (int64_t)n_dst + 1, st));
  const u32 *skeys = s->keys, *svals = s->vals;
  if (n_dst > 0) {
    const unsigned grid = (n_dst + kSelectWarps - 1) / kSelectWarps;
    if (s->shards)
      select_kernel<true><<<grid, kSelectWarps * 32, 0, st>>>(H.dst, n_dst, nullptr, nullptr, nullptr, s->V, k,
                                                              step_key, (u32)h, H.col, H.row_global, H.weight,
                                                              H.edge_dst, s->keys, s->vals, s->shards);
    else
      select_kernel<false><<<grid, kSelectWarps * 32, 0, st>>>(H.dst, n_dst, s->g_col, s->g_row, s->g_w, s->V, k,
                                                               step_key, (u32)h, H.col, H.row_global, H.weight,
                                                               H.edge_dst, s->keys, s->vals, nullptr);
    NTS_LAUNCH_CHECK();
    cub::DoubleBuffer<u32> kd(s->keys, s->keys_alt), vd(s->vals, s->vals_alt);
    const int end_bit = bits_for(s->V);
    NTS_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, need, kd, vd, (int64_t)n_sort, 0, end_bit, st));
    if (int rc = check_tmp(s, need)) return rc;
    NTS_CUDA_OK(cub::DeviceRadixSort::SortPairs(s->tmp, need, kd, vd, (int64_t)n_sort, 0, end_bit, st));
    skeys = kd.Current();
    svals = vd.Current();
    if (inc) {
      head_dst_kernel<<<blocks_for(n_sort), kThreads, 0, st>>>(skeys, svals, n_sort, s->V, s->flag64);
      NTS_LAUNCH_CHECK();
      if (int rc = inclusive_sum(s, s->flag64, s->pos64, n_sort, st)) return rc;
    } else {
      head_kernel<<<blocks_for(n_pad), kThreads, 0, st>>>(skeys, n_pad, H.col, n_dst, s->flag);
      NTS_LAUNCH_CHECK();
      if (int rc = inclusive_sum(s, s->flag, s->pos, n_pad, st)) return rc;
    }
  }
  if (inc)
    finish_dst_kernel<<<blocks_for(std::max<u64>(n_sort, 1)), kThreads, 0, st>>>(
        skeys, svals, s->pos64, n_sort, H.col, n_dst, s->V, H.edge_dst, H.weight, H.row_local, H.src, H.row_offset,
        H.col_t, H.w_t, H.dst_pos, s->counts);
  else
    finish_kernel<<<blocks_for(std::max<u64>(n_pad, 1)), kThreads, 0, st>>>(
        skeys, svals, s->pos, n_pad, H.col, n_dst, H.edge_dst, H.weight, H.row_local, H.src, H.row_offset, H.col_t,
        H.w_t, s->counts);
  NTS_LAUNCH_CHECK();
  NTS_CUDA_OK(cudaMemcpyAsync(s->counts_host, s->counts, 3 * sizeof(u32), cudaMemcpyDeviceToHost, st));
  NTS_CUDA_OK(cudaStreamSynchronize(st));
  NTS_ARG_CHECK(s->counts_host[2] == 0, "a seed vertex id is >= the graph's vertex count");
  H.n_edges = s->counts_host[0];
  H.n_src = s->counts_host[1];
  return 0;
}

} // namespace

extern "C" {

nts_sampler *nts_sampler_create(const nts_vid_t *column_offset, const nts_vid_t *row_indices, const float *edge_weight,
                                nts_vid_t n_vertices, uint64_t n_edges, nts_vid_t max_seeds, int hops,
                                const int *fanout, void *stream) {
  return nts_sampler_create_ex(column_offset, row_indices, edge_weight, n_vertices, n_edges, max_seeds, hops, fanout,
                               0, stream);
}

} // extern "C"

namespace {

nts_sampler *sampler_fail(const char *msg) {
  nts::fail(-1, msg, __FILE__, __LINE__);
  return nullptr;
}

// the argument checks both constructors share; null when the arguments are valid
const char *sampler_args_error(int hops, const int *fanout) {
  if (hops < 1 || hops > kMaxHops) return "sampler hops must be in 1..8";
  if (!fanout) return "sampler fanout is null";
  for (int h = 0; h < hops; ++h)
    if (fanout[h] < 1 || fanout[h] > kMaxFanout) return "sampler fanout must be in 1..64";
  return nullptr;
}

// a sampler over s's graph (set by the caller): parameters, then the scratch for max_seeds seeds
nts_sampler *sampler_init(nts_sampler *s, u32 V, nts_vid_t max_seeds, int hops, const int *fanout, uint32_t flags,
                          void *stream) {
  s->include_dst = (flags & NTS_SAMPLER_INCLUDE_DST) != 0;
  s->V = V;
  s->max_seeds = max_seeds;
  s->hops = hops;
  for (int h = 0; h < hops; ++h) s->fanout[h] = (u32)fanout[h];
  if (sampler_setup(s, nts::as_stream(stream)) != 0) {
    delete s;
    return nullptr;
  }
  return s;
}

} // namespace

extern "C" {

nts_sampler *nts_sampler_create_ex(const nts_vid_t *column_offset, const nts_vid_t *row_indices,
                                   const float *edge_weight, nts_vid_t n_vertices, uint64_t n_edges,
                                   nts_vid_t max_seeds, int hops, const int *fanout, uint32_t flags, void *stream) {
  if (const char *why = sampler_args_error(hops, fanout)) return sampler_fail(why);
  if (n_vertices == 0 || n_vertices >= (1u << 31)) return sampler_fail("sampler needs 1 <= V < 2^31");
  if (n_edges >= (1ull << 32)) return sampler_fail("sampler needs fewer than 2^32 edges");
  if (!column_offset || (n_edges && (!row_indices || !edge_weight)))
    return sampler_fail("null graph array passed to sampler");
  if (flags & ~(uint32_t)NTS_SAMPLER_INCLUDE_DST) return sampler_fail("unknown sampler flag bits");
  nts_sampler *s = new nts_sampler;
  s->g_col = column_offset;
  s->g_row = row_indices;
  s->g_w = edge_weight;
  return sampler_init(s, n_vertices, max_seeds, hops, fanout, flags, stream);
}

nts_sampler *nts_sampler_create_sharded(const nts_vid_t *const *column_offsets, const nts_vid_t *const *row_indices,
                                        const float *const *edge_weights, const nts_vid_t *shard_offsets,
                                        int n_shards, nts_vid_t max_seeds, int hops, const int *fanout,
                                        uint32_t flags, void *stream) {
  if (const char *why = sampler_args_error(hops, fanout)) return sampler_fail(why);
  if (n_shards < 1 || n_shards > kMaxShards) return sampler_fail("sharded sampler needs 1..32 shards");
  if (!column_offsets || !row_indices || !edge_weights || !shard_offsets)
    return sampler_fail("null shard array passed to sampler");
  if (shard_offsets[0] != 0) return sampler_fail("shard offsets must start at 0");
  for (int o = 0; o < n_shards; ++o) {
    if (shard_offsets[o + 1] < shard_offsets[o]) return sampler_fail("shard offsets must be non-decreasing");
    if (shard_offsets[o + 1] > shard_offsets[o] && (!column_offsets[o] || !row_indices[o] || !edge_weights[o]))
      return sampler_fail("null graph array of a non-empty shard passed to sampler");
  }
  const u32 V = shard_offsets[n_shards];
  if (V == 0 || V >= (1u << 31)) return sampler_fail("sampler needs 1 <= V < 2^31");
  if (flags & ~(uint32_t)NTS_SAMPLER_INCLUDE_DST) return sampler_fail("unknown sampler flag bits");
  ShardTable t{};
  t.n = (u32)n_shards;
  for (int o = 0; o <= n_shards; ++o) t.off[o] = shard_offsets[o];
  for (int o = 0; o < n_shards; ++o) {
    t.col[o] = column_offsets[o];
    t.row[o] = row_indices[o];
    t.w[o] = edge_weights[o];
  }
  nts_sampler *s = new nts_sampler;
  cudaStream_t st = nts::as_stream(stream);
  cudaError_t e = cudaSuccess;
  if (s->alloc(&s->shards, 1) != 0 ||
      (e = cudaMemcpyAsync(s->shards, &t, sizeof(t), cudaMemcpyHostToDevice, st)) != cudaSuccess ||
      (e = cudaStreamSynchronize(st)) != cudaSuccess) {   // t is on this stack frame
    if (e != cudaSuccess) nts::fail((int)e, cudaGetErrorString(e), __FILE__, __LINE__);
    delete s;
    return nullptr;
  }
  return sampler_init(s, V, max_seeds, hops, fanout, flags, stream);
}

int nts_sampler_sample(nts_sampler *s, const nts_vid_t *seeds, nts_vid_t n_seeds, uint64_t seed, uint64_t step,
                       void *stream) {
  NTS_ARG_CHECK(s != nullptr, "sampler is null");
  NTS_ARG_CHECK(n_seeds <= s->max_seeds, "more seeds than the sampler was created for");
  NTS_ARG_CHECK(n_seeds == 0 || seeds != nullptr, "seeds is null");
  cudaStream_t st = nts::as_stream(stream);
  s->sampled = false;
  NTS_CUDA_OK(cudaMemsetAsync(s->counts, 0, 4 * sizeof(u32), st));
  if (n_seeds) NTS_CUDA_OK(cudaMemcpyAsync(s->hop[0].dst, seeds, n_seeds * sizeof(u32), cudaMemcpyDeviceToDevice, st));
  const u64 step_key = splitmix64(splitmix64(seed) ^ step);
  for (int h = 0; h < s->hops; ++h) {
    s->hop[h].n_dst = h == 0 ? n_seeds : s->hop[h - 1].n_src;
    if (int rc = sample_hop(s, h, step_key, st)) return rc;
  }
  s->sampled = true;
  return 0;
}

int nts_sampler_hop_view(const nts_sampler *s, int hop, nts_sample_hop_view *v) {
  NTS_ARG_CHECK(s != nullptr && v != nullptr, "null sampler or view");
  NTS_ARG_CHECK(hop >= 0 && hop < s->hops, "hop out of range");
  NTS_ARG_CHECK(s->sampled, "the sampler holds no complete sample");
  const nts_sampler::Hop &H = s->hop[hop];
  v->n_dst = H.n_dst;
  v->n_src = H.n_src;
  v->n_edges = H.n_edges;
  v->dst = H.dst;
  v->column_offset = H.col;
  v->row_indices = H.row_local;
  v->row_global = H.row_global;
  v->weight = H.weight;
  v->src = H.src;
  v->row_offset = H.row_offset;
  v->column_indices = H.col_t;
  v->weight_backward = H.w_t;
  return 0;
}

int nts_sampler_hop_dst_pos(const nts_sampler *s, int hop, const nts_vid_t **dst_pos) {
  NTS_ARG_CHECK(s != nullptr && dst_pos != nullptr, "null sampler or dst_pos");
  NTS_ARG_CHECK(s->include_dst, "the sampler was created without NTS_SAMPLER_INCLUDE_DST");
  NTS_ARG_CHECK(hop >= 0 && hop < s->hops, "hop out of range");
  NTS_ARG_CHECK(s->sampled, "the sampler holds no complete sample");
  *dst_pos = s->hop[hop].dst_pos;
  return 0;
}

uint64_t nts_sampler_bytes(const nts_sampler *s) { return s ? s->bytes : 0; }

int nts_sampler_destroy(nts_sampler *s) {
  delete s;
  return 0;
}

int nts_sample_transpose(const nts_vid_t *column_offset, const nts_vid_t *row_indices, const float *weight,
                         nts_vid_t n_dst, nts_vid_t n_src, uint64_t n_edges, nts_vid_t *row_offset,
                         nts_vid_t *column_indices, float *weight_backward, void *stream) {
  NTS_ARG_CHECK(n_edges < (1ull << 31), "transpose needs fewer than 2^31 edges");
  NTS_ARG_CHECK(row_offset != nullptr, "row_offset is null");
  NTS_ARG_CHECK(n_edges == 0 || (column_offset && row_indices && weight && column_indices && weight_backward),
                "null block array passed to nts_sample_transpose");
  cudaStream_t st = nts::as_stream(stream);
  if (n_edges == 0) {
    NTS_CUDA_OK(cudaMemsetAsync(row_offset, 0, ((size_t)n_src + 1) * sizeof(u32), st));
    return 0;
  }
  // edge_dst, iota, sorted keys, sorted values, CUB scratch: stream-ordered temporaries
  size_t sort_bytes = 0;
  cub::DoubleBuffer<u32> kd(nullptr, nullptr), vd(nullptr, nullptr);
  const int end_bit = bits_for(n_src);
  NTS_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, kd, vd, (int64_t)n_edges, 0, end_bit, st));
  const size_t E4 = ((n_edges * sizeof(u32) + 255) / 256) * 256;
  char *t = nullptr;
  NTS_CUDA_OK(cudaMallocAsync(reinterpret_cast<void **>(&t), 5 * E4 + sort_bytes, st));
  u32 *edge_dst = reinterpret_cast<u32 *>(t), *iota = reinterpret_cast<u32 *>(t + E4),
      *kalt = reinterpret_cast<u32 *>(t + 2 * E4), *valt = reinterpret_cast<u32 *>(t + 3 * E4),
      *kin = reinterpret_cast<u32 *>(t + 4 * E4);
  int rc = 0;
  do {
    if (n_dst) {
      edge_dst_kernel<<<(n_dst + 7) / 8, 256, 0, st>>>(column_offset, n_dst, edge_dst, iota);
      ::nts::count_launch();
      if (cudaGetLastError() != cudaSuccess) { rc = nts::fail(-1, "edge_dst_kernel launch failed", __FILE__, __LINE__); break; }
    }
    cudaError_t e = cudaMemcpyAsync(kin, row_indices, n_edges * sizeof(u32), cudaMemcpyDeviceToDevice, st);
    if (e != cudaSuccess) { rc = nts::fail((int)e, cudaGetErrorString(e), __FILE__, __LINE__); break; }
    cub::DoubleBuffer<u32> k2(kin, kalt), v2(iota, valt);
    e = cub::DeviceRadixSort::SortPairs(t + 5 * E4, sort_bytes, k2, v2, (int64_t)n_edges, 0, end_bit, st);
    if (e != cudaSuccess) { rc = nts::fail((int)e, cudaGetErrorString(e), __FILE__, __LINE__); break; }
    lower_bound_kernel<<<blocks_for((u64)n_src + 1), kThreads, 0, st>>>(k2.Current(), n_edges, n_src, row_offset);
    ::nts::count_launch();
    permute_kernel<<<blocks_for(n_edges), kThreads, 0, st>>>(v2.Current(), n_edges, edge_dst, weight, column_indices,
                                                              weight_backward);
    ::nts::count_launch();
    e = cudaGetLastError();
    if (e != cudaSuccess) { rc = nts::fail((int)e, cudaGetErrorString(e), __FILE__, __LINE__); break; }
  } while (0);
  cudaError_t e = cudaFreeAsync(t, st);
  if (rc == 0 && e != cudaSuccess) rc = nts::fail((int)e, cudaGetErrorString(e), __FILE__, __LINE__);
  return rc;
}

int nts_merge_chunk_csc(const nts_vid_t *const *column_offsets, const nts_vid_t *const *row_indices,
                        const float *const *edge_weights, int n_chunks, nts_vid_t n_dst, uint64_t n_edges,
                        nts_vid_t *column_offset, nts_vid_t *row_indices_out, float *edge_weight_out, void *stream) {
  NTS_ARG_CHECK(n_chunks >= 1 && n_chunks <= kMaxShards, "nts_merge_chunk_csc needs 1..32 chunks");
  NTS_ARG_CHECK(column_offsets && row_indices && edge_weights && column_offset, "null array passed to nts_merge_chunk_csc");
  NTS_ARG_CHECK(n_edges < (1ull << 32), "nts_merge_chunk_csc needs fewer than 2^32 edges");
  NTS_ARG_CHECK(n_edges == 0 || (row_indices_out && edge_weight_out), "null output passed to nts_merge_chunk_csc");
  ChunkCscs c{};
  c.n = n_chunks;
  for (int o = 0; o < n_chunks; ++o) {
    NTS_ARG_CHECK(column_offsets[o] != nullptr, "null chunk column_offset passed to nts_merge_chunk_csc");
    c.col[o] = column_offsets[o];
    c.row[o] = row_indices[o];
    c.w[o] = edge_weights[o];
  }
  cudaStream_t st = nts::as_stream(stream);
  size_t scan_bytes = 0;
  NTS_CUDA_OK(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const u32 *)nullptr, (u32 *)nullptr,
                                            (int64_t)n_dst + 1, st));
  const size_t deg_bytes = (((size_t)n_dst + 1) * sizeof(u32) + 255) / 256 * 256;
  char *t = nullptr;
  NTS_CUDA_OK(cudaMallocAsync(reinterpret_cast<void **>(&t), deg_bytes + 256 + scan_bytes, st));
  u32 *deg = reinterpret_cast<u32 *>(t), *bad = reinterpret_cast<u32 *>(t + deg_bytes);
  // the scanned edge count and the bad-array flag, read back before the copy writes n_edges slots
  u32 check[2] = {0, 0};
  cudaError_t e = cudaMemsetAsync(bad, 0, sizeof(u32), st);
  if (e == cudaSuccess) {
    merge_count_kernel<<<blocks_for((u64)n_dst + 1), kThreads, 0, st>>>(c, n_dst, deg, bad);
    ::nts::count_launch();
    e = cudaGetLastError();
  }
  if (e == cudaSuccess)
    e = cub::DeviceScan::ExclusiveSum(t + deg_bytes + 256, scan_bytes, deg, column_offset, (int64_t)n_dst + 1, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(check, column_offset + n_dst, sizeof(u32), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(check + 1, bad, sizeof(u32), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  int rc = 0;
  if (e != cudaSuccess) {
    rc = nts::fail((int)e, cudaGetErrorString(e), __FILE__, __LINE__);
  } else if (check[1]) {
    rc = nts::fail(-1, "nts_merge_chunk_csc: null row / weight array of a chunk with edges", __FILE__, __LINE__);
  } else if (check[0] != n_edges) {
    rc = nts::fail(-1, "nts_merge_chunk_csc: n_edges differs from the chunks' edge count", __FILE__, __LINE__);
  } else if (n_dst) {
    merge_copy_kernel<<<(n_dst + 7) / 8, 256, 0, st>>>(c, n_dst, column_offset, row_indices_out, edge_weight_out);
    ::nts::count_launch();
    e = cudaGetLastError();
    if (e != cudaSuccess) rc = nts::fail((int)e, cudaGetErrorString(e), __FILE__, __LINE__);
  }
  e = cudaFreeAsync(t, st);   // stream-ordered: after the kernels that read it
  if (rc == 0 && e != cudaSuccess) return nts::fail((int)e, cudaGetErrorString(e), __FILE__, __LINE__);
  return rc;
}

} // extern "C"
