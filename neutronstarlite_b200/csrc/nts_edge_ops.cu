// Edge-granular operators of the GAT path for sm_90a: mirror/destination <-> edge-message copies,
// per-destination edge softmax (multi-column, max-subtracted) and the fused-aggregation backward.
//
// Replaces cuda/ntsCUDADistKernel.cuh:23-95,166-260 and the `scatter_grad_back_to_messaage` kernel
// (cuda/ntsCUDAFuseKernel.cuh:492-506) of the reference.  These kernels are HBM-bound streams over
// [E, F] messages: every one moves whole rows with the widest vector the row alignment allows, is
// split by EDGES (a warp owns a quantum of consecutive edges and finds its destination rows by
// binary search over column_offset), and uses atomics only where two edges of different
// destinations meet in one mirror row.
#include <algorithm>

#include "nts_common.cuh"

namespace nts {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr uint32_t kEdgeQuantum = 64; // consecutive edges per warp

// mirror slot of edge e: through the MirrorIndex table, or directly when the index array already holds slots
__device__ __forceinline__ uint32_t slot_at(const uint32_t *__restrict__ row_idx,
                                            const uint32_t *__restrict__ mirror_index, size_t e) {
  const uint32_t id = __ldg(row_idx + e);
  return mirror_index ? __ldg(mirror_index + id) : id;
}

__device__ __forceinline__ float vec_dot(float a, float b) { return a * b; }
__device__ __forceinline__ float vec_dot(float2 a, float2 b) { return fmaf(a.x, b.x, a.y * b.y); }
__device__ __forceinline__ float vec_dot(float4 a, float4 b) {
  return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, a.w * b.w)));
}
__device__ __forceinline__ float vec_dot(float8v a, float8v b) {
  return fmaf(a.lo.x, b.lo.x, fmaf(a.lo.y, b.lo.y, fmaf(a.lo.z, b.lo.z, fmaf(a.lo.w, b.lo.w, vec_dot(a.hi, b.hi)))));
}
__device__ __forceinline__ float vec_scale(float a, float s) { return a * s; }
__device__ __forceinline__ float2 vec_scale(float2 a, float s) { return make_float2(a.x * s, a.y * s); }
__device__ __forceinline__ float4 vec_scale(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ float8v vec_scale(float8v a, float s) { return {vec_scale(a.lo, s), vec_scale(a.hi, s)}; }
__device__ __forceinline__ float vec_add(float a, float b) { return a + b; }
__device__ __forceinline__ float2 vec_add(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float4 vec_add(float4 a, float4 b) {
  return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}
__device__ __forceinline__ float8v vec_add(float8v a, float8v b) { return {vec_add(a.lo, b.lo), vec_add(a.hi, b.hi)}; }

// ---- row movers ------------------------------------------------------------------------------------------
// mode 0: dst[r,:]        = src[map(r),:]
// mode 1: dst[map(r),:]  += src[r,:]   (map unique -> plain read-modify-write)
// mode 2: dst[map(r),:]  += src[r,:]   (atomic)
// map(r) = map2 ? map2[map1[r]] : map1[r]
template <int VEC, int MODE>
__global__ void __launch_bounds__(kThreads)
    move_rows_kernel(float *__restrict__ dst, const float *__restrict__ src, const uint32_t *__restrict__ map1,
                     const uint32_t *__restrict__ map2, uint64_t n_rows, const uint32_t *__restrict__ n_rows_dev,
                     uint32_t F) {
  using V = typename Vec<VEC>::type;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t nvec = F / VEC;
  if (n_rows_dev)
    n_rows = __ldg(n_rows_dev); // e.g. E_p = column_offset[Vp], kept on the device
  const uint64_t warp0 = (uint64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  const uint64_t nwarps = (uint64_t)gridDim.x * kWarps;
  for (uint64_t r = warp0; r < n_rows; r += nwarps) {
    uint32_t m = __ldg(map1 + r);
    if (map2)
      m = __ldg(map2 + m);
    if (MODE == 0) {
      const V *s = reinterpret_cast<const V *>(src + (size_t)m * F);
      V *d = reinterpret_cast<V *>(dst + (size_t)r * F);
      for (uint32_t c = lane; c < nvec; c += 32)
        d[c] = __ldg(s + c);
    } else {
      const V *s = reinterpret_cast<const V *>(src + (size_t)r * F);
      V *d = reinterpret_cast<V *>(dst + (size_t)m * F);
      for (uint32_t c = lane; c < nvec; c += 32) {
        V v = __ldg(s + c);
        if (MODE == 1)
          d[c] = vec_add(d[c], v);
        else
          red_add(d + c, v);
      }
    }
  }
}

// ---- row gather from a table sharded by global row ranges ----------------------------------------------------
// dst[k,:F] = shards[o][ids[k] - off[o], :F], o = the shard with off[o] <= ids[k] < off[o+1] (binary search over the
// offsets staged in shared memory; empty shards have off[o] == off[o+1] and are never chosen).  Shard rows are `pitch`
// floats with pitch % 4 == 0 and every shard 16-byte aligned, so each lane loads whole float4s, the last one of a row
// reaching into its padding; stores are SVEC floats wide (dst is [n, F], so F's alignment decides).  A row takes
// LANES lanes (a virtual warp of a warp for rows of at most 8 / 16 float4s, as in the planned kernel), and each lane
// issues up to kGatherUnroll loads before it stores them.
constexpr int kGatherUnroll = 4;

template <int LANES, int SVEC>
__global__ void __launch_bounds__(kThreads)
    gather_rows_sharded_kernel(float *__restrict__ dst, const float *const *__restrict__ shards,
                               const uint32_t *__restrict__ offsets, int n_shards, uint32_t pitch,
                               const uint32_t *__restrict__ ids, uint32_t n, uint32_t F) {
  __shared__ uint32_t s_off[kMaxShards + 1];
  __shared__ const float *s_shard[kMaxShards];
  stage_shard_table(s_off, s_shard, offsets, shards, n_shards);
  constexpr uint32_t kRowsPerBlock = kThreads / LANES;
  const uint32_t sub = threadIdx.x & (LANES - 1);
  const uint32_t nvec = (F + 3) / 4;
  for (uint64_t k = (uint64_t)blockIdx.x * kRowsPerBlock + threadIdx.x / LANES; k < n;
       k += (uint64_t)gridDim.x * kRowsPerBlock) {
    const uint32_t id = __ldg(ids + k);
    const int lo = find_shard(s_off, n_shards, id);
    const float4 *s = reinterpret_cast<const float4 *>(s_shard[lo] + (size_t)(id - s_off[lo]) * pitch);
    float *d = dst + (size_t)k * F;
    for (uint32_t c0 = sub; c0 < nvec; c0 += kGatherUnroll * LANES) {
      float4 v[kGatherUnroll];
#pragma unroll
      for (int u = 0; u < kGatherUnroll; u++)
        if (c0 + u * LANES < nvec)
          v[u] = __ldg(s + c0 + u * LANES);
#pragma unroll
      for (int u = 0; u < kGatherUnroll; u++)
        if (c0 + u * LANES < nvec)
          store_chunk<SVEC>(d, 4 * (c0 + u * LANES), F, v[u]);
    }
  }
}

template <int LANES>
static void launch_gather_rows_sharded(int svec, unsigned grid, cudaStream_t st, float *dst, const float *const *shards,
                                       const uint32_t *offsets, int n_shards, uint32_t pitch, const uint32_t *ids,
                                       uint32_t n, uint32_t F) {
  if (svec == 4)
    gather_rows_sharded_kernel<LANES, 4><<<grid, kThreads, 0, st>>>(dst, shards, offsets, n_shards, pitch, ids, n, F);
  else if (svec == 2)
    gather_rows_sharded_kernel<LANES, 2><<<grid, kThreads, 0, st>>>(dst, shards, offsets, n_shards, pitch, ids, n, F);
  else
    gather_rows_sharded_kernel<LANES, 1><<<grid, kThreads, 0, st>>>(dst, shards, offsets, n_shards, pitch, ids, n, F);
}

// The BF16 twin: shard rows of `pitch` BF16 values (pitch % 8 == 0), one 16-byte load per 8 values.  SVEC == 0 copies
// them into BF16 rows of stride ld_out (ld_out % 8 == 0, dst 16-byte aligned): whole chunks, so the columns
// [F, 8 ceil(F/8)) receive the shard's pad.  SVEC = 4 / 2 / 1 widens them into FP32 [n, F] with stores of SVEC floats.
// Same shard staging and search as gather_rows_sharded_kernel; LANES lanes per row of ceil(F/8) chunks.
template <int LANES, int SVEC>
__global__ void __launch_bounds__(kThreads)
    gather_rows_sharded_bf16_kernel(void *__restrict__ dst, uint32_t ld_out, const uint4 *const *__restrict__ shards,
                                    const uint32_t *__restrict__ offsets, int n_shards, uint32_t pitch,
                                    const uint32_t *__restrict__ ids, uint32_t n, uint32_t F) {
  __shared__ uint32_t s_off[kMaxShards + 1];
  __shared__ const uint4 *s_shard[kMaxShards];
  stage_shard_table(s_off, s_shard, offsets, shards, n_shards);
  constexpr uint32_t kRowsPerBlock = kThreads / LANES;
  const uint32_t sub = threadIdx.x & (LANES - 1);
  const uint32_t nvec = (F + 7) / 8;
  for (uint64_t k = (uint64_t)blockIdx.x * kRowsPerBlock + threadIdx.x / LANES; k < n;
       k += (uint64_t)gridDim.x * kRowsPerBlock) {
    const uint32_t id = __ldg(ids + k);
    const int lo = find_shard(s_off, n_shards, id);
    const uint4 *s = s_shard[lo] + (size_t)(id - s_off[lo]) * (pitch / 8);
    for (uint32_t c0 = sub; c0 < nvec; c0 += kGatherUnroll * LANES) {
      uint4 v[kGatherUnroll];
#pragma unroll
      for (int u = 0; u < kGatherUnroll; u++)
        if (c0 + u * LANES < nvec)
          v[u] = __ldg(s + c0 + u * LANES);
#pragma unroll
      for (int u = 0; u < kGatherUnroll; u++) {
        const uint32_t c = c0 + u * LANES;
        if (c < nvec) {
          if constexpr (SVEC == 0) {
            reinterpret_cast<uint4 *>(dst)[(size_t)k * (ld_out / 8) + c] = v[u];
          } else {
            float *d = reinterpret_cast<float *>(dst) + (size_t)k * F;
            const float8v x = widen(v[u]);
            store_chunk<SVEC>(d, 8 * c, F, x.lo);
            if (8 * c + 4 < F)
              store_chunk<SVEC>(d, 8 * c + 4, F, x.hi);
          }
        }
      }
    }
  }
}

template <int LANES>
static void launch_gather_rows_sharded_bf16(int svec, unsigned grid, cudaStream_t st, void *dst, uint32_t ld_out,
                                            const uint4 *const *shards, const uint32_t *offsets, int n_shards,
                                            uint32_t pitch, const uint32_t *ids, uint32_t n, uint32_t F) {
  if (svec == 0)
    gather_rows_sharded_bf16_kernel<LANES, 0><<<grid, kThreads, 0, st>>>(dst, ld_out, shards, offsets, n_shards, pitch,
                                                                         ids, n, F);
  else if (svec == 4)
    gather_rows_sharded_bf16_kernel<LANES, 4><<<grid, kThreads, 0, st>>>(dst, ld_out, shards, offsets, n_shards, pitch,
                                                                         ids, n, F);
  else if (svec == 2)
    gather_rows_sharded_bf16_kernel<LANES, 2><<<grid, kThreads, 0, st>>>(dst, ld_out, shards, offsets, n_shards, pitch,
                                                                         ids, n, F);
  else
    gather_rows_sharded_bf16_kernel<LANES, 1><<<grid, kThreads, 0, st>>>(dst, ld_out, shards, offsets, n_shards, pitch,
                                                                         ids, n, F);
}

// msg[e,:] (=|+=) x[dst(e),:] : destination row broadcast over its CSC segment
template <int VEC, bool ACCUM>
__global__ void __launch_bounds__(kThreads)
    segment_broadcast_kernel(float *__restrict__ msg, const float *__restrict__ x, const uint32_t *__restrict__ off,
                             uint32_t n_rows, uint32_t F) {
  using V = typename Vec<VEC>::type;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t nvec = F / VEC;
  const uint32_t n_edges = __ldg(off + n_rows); // E_p stays on the device: no host read-back
  const uint64_t nwarps = (uint64_t)gridDim.x * kWarps;
  for (uint64_t qw = (uint64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); qw * kEdgeQuantum < n_edges; qw += nwarps) {
  const uint32_t e0 = (uint32_t)(qw * kEdgeQuantum);
  const uint32_t e1 = (uint32_t)min((uint64_t)n_edges, (uint64_t)e0 + kEdgeQuantum);
  uint32_t row = find_row(off, n_rows, e0);
  uint32_t row_end = __ldg(off + row + 1);
  for (uint32_t e = e0; e < e1; e++) {
    while (e >= row_end) {
      row++;
      row_end = __ldg(off + row + 1);
    }
    const V *s = reinterpret_cast<const V *>(x + (size_t)row * F);
    V *d = reinterpret_cast<V *>(msg + (size_t)e * F);
    for (uint32_t c = lane; c < nvec; c += 32) {
      V v = __ldg(s + c);
      d[c] = ACCUM ? vec_add(d[c], v) : v;
    }
  }
  } // quantum loop
}

// y[d,:] += sum_{e->d} msg[e,:]: edge-quantum segmented sum of a contiguous stream; boundary rows use atomics
template <int VEC>
__global__ void __launch_bounds__(kThreads)
    segment_sum_kernel(float *__restrict__ y, const float *__restrict__ msg, const uint32_t *__restrict__ off,
                       uint32_t n_rows, uint32_t F) {
  using V = typename Vec<VEC>::type;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t nvec = F / VEC;
  const uint32_t n_edges = __ldg(off + n_rows); // E_p stays on the device: no host read-back
  const uint64_t nwarps = (uint64_t)gridDim.x * kWarps;
  for (uint64_t qw = (uint64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); qw * kEdgeQuantum < n_edges; qw += nwarps) {
  const uint32_t e0 = (uint32_t)(qw * kEdgeQuantum);
  const uint32_t e1 = (uint32_t)min((uint64_t)n_edges, (uint64_t)e0 + kEdgeQuantum);
  // columns are processed in passes of 32 vectors so that the accumulator stays in one register set
  for (uint32_t cbase = 0; cbase < nvec; cbase += 32) {
    const uint32_t c = cbase + lane;
    const bool act = c < nvec;
    uint32_t row = find_row(off, n_rows, e0);
    uint32_t row_end = __ldg(off + row + 1);
    bool inside = __ldg(off + row) >= e0;
    V acc;
    memset(&acc, 0, sizeof(V));
    for (uint32_t e = e0; e < e1; e++) {
      if (e >= row_end) {
        if (act) {
          V *o = reinterpret_cast<V *>(y + (size_t)row * F) + c;
          if (inside)
            *o = vec_add(*o, acc);
          else
            red_add(o, acc);
        }
        memset(&acc, 0, sizeof(V));
        do {
          row++;
          row_end = __ldg(off + row + 1);
        } while (e >= row_end);
        inside = true;
      }
      if (act)
        acc = vec_add(acc, __ldg(reinterpret_cast<const V *>(msg + (size_t)e * F) + c));
    }
    if (act) {
      V *o = reinterpret_cast<V *>(y + (size_t)row * F) + c;
      if (inside && row_end <= e1)
        *o = vec_add(*o, acc);
      else
        red_add(o, acc);
    }
  }
  } // quantum loop
}

// ---- edge softmax ------------------------------------------------------------------------------------------
// One CTA walks a block of destination rows.  Small segments are handled one per warp, segments with
// more than kHubDegree edges by the whole CTA.  H = number of columns (heads); element (e,h) at m[e*H+h].
constexpr uint32_t kRowsPerCta = 64;
constexpr uint32_t kHubDegree = 4096;

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <bool IS_MAX> __device__ __forceinline__ float block_reduce(float v, float *scratch) {
  v = IS_MAX ? warp_max(v) : warp_sum(v);
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __syncthreads(); // scratch reuse
  if (lane == 0)
    scratch[wid] = v;
  __syncthreads();
  float r = scratch[0];
#pragma unroll
  for (int i = 1; i < kWarps; i++)
    r = IS_MAX ? fmaxf(r, scratch[i]) : r + scratch[i];
  return r;
}

// forward: a = exp(m - max) / sum exp(m - max) per (segment, column); cache gets a copy of a
template <bool BACKWARD>
__global__ void __launch_bounds__(kThreads)
    edge_softmax_kernel(float *__restrict__ out, const float *__restrict__ in0, const float *__restrict__ in1,
                        float *__restrict__ cache, const uint32_t *__restrict__ off, uint32_t n_rows, uint32_t H) {
  // forward : in0 = m,      in1 unused, out = a, cache = a
  // backward: in0 = g_out,  in1 = a (cached), out = g_in = a*g - a*sum(a*g)
  __shared__ float scratch[kWarps];
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t r0 = blockIdx.x * kRowsPerCta;
  const uint32_t r1 = min(n_rows, r0 + kRowsPerCta);
  for (uint32_t r = r0; r < r1; r++) {
    const uint32_t b = __ldg(off + r), e = __ldg(off + r + 1);
    const uint32_t deg = e - b;
    if (deg == 0)
      continue;
    const bool hub = deg > kHubDegree; // block-uniform
    if (!hub && ((r - r0) % kWarps) != wid)
      continue;
    const uint32_t tid = hub ? threadIdx.x : lane;
    const uint32_t nthr = hub ? kThreads : 32;
    for (uint32_t h = 0; h < H; h++) {
      const float *x0 = in0 + (size_t)b * H + h;
      if (!BACKWARD) {
        float mx = -INFINITY;
        for (uint32_t i = tid; i < deg; i += nthr)
          mx = fmaxf(mx, __ldg(x0 + (size_t)i * H));
        mx = hub ? block_reduce<true>(mx, scratch) : warp_max(mx);
        float s = 0.f;
        for (uint32_t i = tid; i < deg; i += nthr)
          s += expf(__ldg(x0 + (size_t)i * H) - mx);
        s = hub ? block_reduce<false>(s, scratch) : warp_sum(s);
        const float inv = 1.f / s;
        for (uint32_t i = tid; i < deg; i += nthr) {
          float a = expf(__ldg(x0 + (size_t)i * H) - mx) * inv;
          out[((size_t)b + i) * H + h] = a;
          if (cache)
            cache[((size_t)b + i) * H + h] = a;
        }
      } else {
        const float *a0 = in1 + (size_t)b * H + h;
        float dot = 0.f;
        for (uint32_t i = tid; i < deg; i += nthr)
          dot = fmaf(__ldg(x0 + (size_t)i * H), __ldg(a0 + (size_t)i * H), dot);
        dot = hub ? block_reduce<false>(dot, scratch) : warp_sum(dot);
        for (uint32_t i = tid; i < deg; i += nthr) {
          float a = __ldg(a0 + (size_t)i * H);
          float g = __ldg(x0 + (size_t)i * H);
          out[((size_t)b + i) * H + h] = a * g - a * dot;
        }
      }
    }
  }
}

// ---- fused GAT aggregation backward ----------------------------------------------------------------------
//   a_grad[e]               = < mirror[slot(e),:], g[dst(e),:] >      (warp-shuffle reduction)
//   mirror_grad[slot(e),:] += a[e] * g[dst(e),:]                      (vector red.global.add)
template <int VEC>
__global__ void __launch_bounds__(kThreads)
    fuse_weight_backward_kernel(float *__restrict__ mirror_grad, float *__restrict__ a_grad,
                                const float *__restrict__ mirror, const float *__restrict__ a,
                                const float *__restrict__ g, const uint32_t *__restrict__ row_idx,
                                const uint32_t *__restrict__ off, const uint32_t *__restrict__ mirror_index,
                                uint32_t n_rows, uint32_t F, uint32_t heads) {
  using V = typename Vec<VEC>::type;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t head_vecs = F / VEC / heads; // vectors per head (host guarantees divisibility)
  const uint32_t n_edges = __ldg(off + n_rows); // E_p stays on the device: no host read-back
  const uint64_t nwarps = (uint64_t)gridDim.x * kWarps;
  for (uint64_t qw = (uint64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); qw * kEdgeQuantum < n_edges; qw += nwarps) {
    const uint32_t e0 = (uint32_t)(qw * kEdgeQuantum);
    const uint32_t e1 = (uint32_t)min((uint64_t)n_edges, (uint64_t)e0 + kEdgeQuantum);
    uint32_t row = find_row(off, n_rows, e0);
    uint32_t row_end = __ldg(off + row + 1);
    for (uint32_t e = e0; e < e1; e++) {
      while (e >= row_end) {
        row++;
        row_end = __ldg(off + row + 1);
      }
      const uint32_t slot = slot_at(row_idx, mirror_index, e);
      const V *gm = reinterpret_cast<const V *>(g + (size_t)row * F);
      const V *mm = reinterpret_cast<const V *>(mirror + (size_t)slot * F);
      V *dm = reinterpret_cast<V *>(mirror_grad + (size_t)slot * F);
      for (uint32_t h = 0; h < heads; h++) {
        const float ae = __ldg(a + (size_t)e * heads + h);
        float dot = 0.f;
        for (uint32_t c = h * head_vecs + lane; c < (h + 1) * head_vecs; c += 32) {
          V gv = __ldg(gm + c);
          dot += vec_dot(__ldg(mm + c), gv);
          red_add(dm + c, vec_scale(gv, ae));
        }
        dot = warp_sum(dot);
        if (lane == 0)
          a_grad[(size_t)e * heads + h] = dot;
      }
    }
  } // quantum loop
}

// ---- fully fused GAT layer (K7): attention logits are never materialised ------------------------------------------
//   logit[e,h] = leaky_relu(s[slot(e),h] + d[dst(e),h]);  a = softmax over the destination segment
// stats kernel: seg_max[d,h], seg_sum[d,h] (sum of exp(logit - max)); empty segments get (0, 1).

__global__ void __launch_bounds__(kThreads)
    gat_softmax_stats_kernel(float *__restrict__ seg_max, float *__restrict__ seg_sum, const float *__restrict__ s_att,
                             const float *__restrict__ d_att, const uint32_t *__restrict__ row_idx,
                             const uint32_t *__restrict__ off, const uint32_t *__restrict__ mirror_index,
                             uint32_t n_rows, uint32_t H, float slope) {
  __shared__ float scratch[kWarps];
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t r0 = blockIdx.x * kRowsPerCta;
  const uint32_t r1 = min(n_rows, r0 + kRowsPerCta);
  for (uint32_t r = r0; r < r1; r++) {
    const uint32_t b = __ldg(off + r), e = __ldg(off + r + 1);
    const uint32_t deg = e - b;
    const bool hub = deg > kHubDegree; // block-uniform
    if (!hub && ((r - r0) % kWarps) != wid)
      continue;
    const uint32_t tid = hub ? threadIdx.x : lane;
    const uint32_t nthr = hub ? kThreads : 32;
    for (uint32_t h = 0; h < H; h++) {
      if (deg == 0) {
        if (tid == 0) {
          seg_max[(size_t)r * H + h] = 0.f;
          seg_sum[(size_t)r * H + h] = 1.f;
        }
        continue;
      }
      const float dv = __ldg(d_att + (size_t)r * H + h);
      float mx = -INFINITY;
      for (uint32_t i = tid; i < deg; i += nthr) {
        const uint32_t slot = slot_at(row_idx, mirror_index, b + i);
        mx = fmaxf(mx, leaky(__ldg(s_att + (size_t)slot * H + h) + dv, slope));
      }
      mx = hub ? block_reduce<true>(mx, scratch) : warp_max(mx);
      float sum = 0.f;
      for (uint32_t i = tid; i < deg; i += nthr) {
        const uint32_t slot = slot_at(row_idx, mirror_index, b + i);
        sum += expf(leaky(__ldg(s_att + (size_t)slot * H + h) + dv, slope) - mx);
      }
      sum = hub ? block_reduce<false>(sum, scratch) : warp_sum(sum);
      if (tid == 0) {
        seg_max[(size_t)r * H + h] = mx;
        seg_sum[(size_t)r * H + h] = sum;
      }
    }
  }
}

// Edge-balanced statistics (H divides 32): a warp owns a quantum of consecutive EDGES whatever rows they belong to,
// lane = (edge slot, head); every lane keeps a running (max | sum) for the row its edges are in and merges it with
// one atomic when its row changes or the quantum ends (combined across the lanes first when the whole warp sits in
// one row - the hub case).  PASS 0: maxima (seg_max pre-set to -inf), PASS 1: sums of exp(logit - max) (seg_sum
// pre-set to 0); gat_stats_init_kernel presets both and gives empty segments (0, 1).
__global__ void __launch_bounds__(kThreads)
    gat_stats_init_kernel(float *__restrict__ seg_max, float *__restrict__ seg_sum, const uint32_t *__restrict__ off,
                          uint32_t n_rows, uint32_t H) {
  const uint64_t n = (uint64_t)n_rows * H;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t r = (uint32_t)(i / H);
    const bool empty = __ldg(off + r + 1) == __ldg(off + r);
    seg_max[i] = empty ? 0.f : -INFINITY;
    seg_sum[i] = empty ? 1.f : 0.f;
  }
}

template <int H, int PASS>
__global__ void __launch_bounds__(kThreads)
    gat_edge_stats_kernel(float *__restrict__ seg_max, float *__restrict__ seg_sum, const float *__restrict__ s_att,
                          const float *__restrict__ d_att, const uint32_t *__restrict__ row_idx,
                          const uint32_t *__restrict__ off, const uint32_t *__restrict__ mirror_index,
                          uint32_t n_rows, float slope) {
  static_assert(32 % H == 0, "H must divide the warp size");
  constexpr uint32_t kEdgesPerStep = 32 / H;
  constexpr int kUnroll = 4;
  constexpr uint32_t kQuantum = 512;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t h = lane % H, el = lane / H;
  const uint32_t n_edges = __ldg(off + n_rows);
  const uint64_t nwarps = (uint64_t)gridDim.x * kWarps;
  for (uint64_t qw = (uint64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); qw * kQuantum < n_edges; qw += nwarps) {
    const uint32_t e0 = (uint32_t)(qw * kQuantum);
    const uint32_t e1 = (uint32_t)min((uint64_t)n_edges, (uint64_t)e0 + kQuantum);
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
    load_row();
    for (uint32_t eb = e0 + el; eb < e1; eb += kEdgesPerStep * kUnroll) {
      float sv[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; u++) {
        const uint32_t e = eb + u * kEdgesPerStep;
        sv[u] = e < e1 ? __ldg(s_att + (size_t)slot_at(row_idx, mirror_index, e) * H + h) : 0.f;
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

// Single-pass backward when a head is a power-of-two number of vectors <= 32 (e.g. 8 heads x 8 columns): every lane
// owns vector column(s) c = lane + 32k of the row, its head is c / head_vecs, per-head dot products are segmented
// xor-shuffle reductions, the first lane of each head group issues the score-gradient atomics.
template <int VEC, int KB>
__global__ void __launch_bounds__(kThreads)
    gat_fused_backward_seg_kernel(float *__restrict__ mirror_grad, float *__restrict__ s_grad,
                                  float *__restrict__ d_grad, const float *__restrict__ mirror,
                                  const float *__restrict__ s_att, const float *__restrict__ d_att,
                                  const float *__restrict__ seg_max, const float *__restrict__ seg_sum,
                                  const float *__restrict__ out_dot_g, const float *__restrict__ g,
                                  const uint32_t *__restrict__ row_idx, const uint32_t *__restrict__ off,
                                  const uint32_t *__restrict__ mirror_index, uint32_t n_rows, uint32_t F, uint32_t H,
                                  float slope) {
  using V = typename Vec<VEC>::type;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t nvec = F / VEC;
  const uint32_t head_vecs = nvec / H; // power of two, <= 32
  const bool leader = (lane % head_vecs) == 0;
  uint32_t hk[KB];
  bool act[KB];
#pragma unroll
  for (int k = 0; k < KB; k++) {
    act[k] = lane + 32 * k < nvec;
    hk[k] = act[k] ? (lane + 32 * k) / head_vecs : 0u;
  }
  const uint32_t n_edges = __ldg(off + n_rows);
  const uint64_t nwarps = (uint64_t)gridDim.x * kWarps;
  for (uint64_t qw = (uint64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); qw * kEdgeQuantum < n_edges; qw += nwarps) {
    const uint32_t e0 = (uint32_t)(qw * kEdgeQuantum);
    const uint32_t e1 = (uint32_t)min((uint64_t)n_edges, (uint64_t)e0 + kEdgeQuantum);
    uint32_t row = find_row(off, n_rows, e0);
    uint32_t row_end = __ldg(off + row + 1);
    float d_acc[KB], dv[KB], mv[KB], iz[KB], og[KB];
    auto load_row = [&]() {
#pragma unroll
      for (int k = 0; k < KB; k++) {
        const size_t rh = (size_t)row * H + hk[k];
        dv[k] = __ldg(d_att + rh);
        mv[k] = __ldg(seg_max + rh);
        iz[k] = 1.f / __ldg(seg_sum + rh);
        og[k] = __ldg(out_dot_g + rh);
        d_acc[k] = 0.f;
      }
    };
    auto flush_row = [&]() {
#pragma unroll
      for (int k = 0; k < KB; k++)
        if (act[k] && leader && d_acc[k] != 0.f)
          atomicAdd(d_grad + (size_t)row * H + hk[k], d_acc[k]);
    };
    load_row();
    for (uint32_t eb = e0; eb < e1; eb += 32) {
      // indices and mirror slots of 32 edges at once (coalesced), broadcast per edge by shuffle; the mirror row of
      // edge j+1 is requested before edge j is processed (the random gather is the long-latency load)
      const uint32_t cnt = min(32u, e1 - eb);
      uint32_t my_slot = 0;
      if (lane < cnt)
        my_slot = slot_at(row_idx, mirror_index, eb + lane);
      V m_next[KB];
      {
        const uint32_t s0 = __shfl_sync(0xffffffffu, my_slot, 0);
        const V *mm0 = reinterpret_cast<const V *>(mirror + (size_t)s0 * F);
#pragma unroll
        for (int k = 0; k < KB; k++)
          if (act[k])
            m_next[k] = __ldg(mm0 + lane + 32 * k);
      }
      for (uint32_t j = 0; j < cnt; j++) {
        const uint32_t e = eb + j;
        if (e >= row_end) {
          flush_row();
          do {
            row++;
            row_end = __ldg(off + row + 1);
          } while (e >= row_end);
          load_row();
        }
        const uint32_t slot = __shfl_sync(0xffffffffu, my_slot, j);
        V m_cur[KB];
#pragma unroll
        for (int k = 0; k < KB; k++)
          m_cur[k] = m_next[k];
        if (j + 1 < cnt) {
          const uint32_t s1 = __shfl_sync(0xffffffffu, my_slot, j + 1);
          const V *mm1 = reinterpret_cast<const V *>(mirror + (size_t)s1 * F);
#pragma unroll
          for (int k = 0; k < KB; k++)
            if (act[k])
              m_next[k] = __ldg(mm1 + lane + 32 * k);
        }
        const V *gm = reinterpret_cast<const V *>(g + (size_t)row * F);
        V *dm = reinterpret_cast<V *>(mirror_grad + (size_t)slot * F);
#pragma unroll
        for (int k = 0; k < KB; k++) {
          const uint32_t c = lane + 32 * k;
          float dot = 0.f, pre = 0.f, a = 0.f;
          if (act[k]) {
            const V gv = __ldg(gm + c);
            dot = vec_dot(m_cur[k], gv);
            pre = __ldg(s_att + (size_t)slot * H + hk[k]) + dv[k];
            a = expf(leaky(pre, slope) - mv[k]) * iz[k];
            red_add(dm + c, vec_scale(gv, a));
          }
          // per-head dot: lanes of one head are contiguous and head_vecs is a power of two
          for (uint32_t o = head_vecs >> 1; o > 0; o >>= 1)
            dot += __shfl_xor_sync(0xffffffffu, dot, o);
          if (act[k] && leader) {
            const float d_pre = a * (dot - og[k]) * (pre > 0.f ? 1.f : slope);
            atomicAdd(s_grad + (size_t)slot * H + hk[k], d_pre);
            d_acc[k] += d_pre;
          }
        }
      }
    }
    flush_row();
  } // quantum loop
}

// backward of the fused layer, one pass over the edges:
//   a        = exp(logit - m) / z                              (recomputed)
//   d_a      = < mirror[slot, head h], g[dst, head h] >        (warp-shuffle reduction)
//   d_logit  = a * (d_a - <out[dst,h], g[dst,h]>)              (softmax backward; the segment sum is a per-vertex dot)
//   d_pre    = d_logit * leaky_relu'(pre)
//   s_grad[slot,h] += d_pre (atomic),  d_grad[dst,h] += d_pre (per-row register sum, one atomic per row/quantum)
//   mirror_grad[slot, head h] += a * g[dst, head h]            (vector red)
template <int VEC>
__global__ void __launch_bounds__(kThreads)
    gat_fused_backward_kernel(float *__restrict__ mirror_grad, float *__restrict__ s_grad, float *__restrict__ d_grad,
                              const float *__restrict__ mirror, const float *__restrict__ s_att,
                              const float *__restrict__ d_att, const float *__restrict__ seg_max,
                              const float *__restrict__ seg_sum, const float *__restrict__ out_dot_g,
                              const float *__restrict__ g, const uint32_t *__restrict__ row_idx,
                              const uint32_t *__restrict__ off, const uint32_t *__restrict__ mirror_index,
                              uint32_t n_rows, uint32_t F, uint32_t H, float slope) {
  using V = typename Vec<VEC>::type;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t head_vecs = F / VEC / H;
  const uint32_t n_edges = __ldg(off + n_rows);
  const uint64_t nwarps = (uint64_t)gridDim.x * kWarps;
  for (uint64_t qw = (uint64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); qw * kEdgeQuantum < n_edges; qw += nwarps) {
    const uint32_t e0 = (uint32_t)(qw * kEdgeQuantum);
    const uint32_t e1 = (uint32_t)min((uint64_t)n_edges, (uint64_t)e0 + kEdgeQuantum);
    for (uint32_t h = 0; h < H; h++) { // one head at a time: the per-row accumulator is a single register
      uint32_t row = find_row(off, n_rows, e0);
      uint32_t row_end = __ldg(off + row + 1);
      float d_acc = 0.f;
      for (uint32_t e = e0; e < e1; e++) {
        if (e >= row_end) {
          if (lane == 0 && d_acc != 0.f)
            atomicAdd(d_grad + (size_t)row * H + h, d_acc);
          d_acc = 0.f;
          do {
            row++;
            row_end = __ldg(off + row + 1);
          } while (e >= row_end);
        }
        const uint32_t slot = slot_at(row_idx, mirror_index, e);
        const size_t rh = (size_t)row * H + h;
        const float pre = __ldg(s_att + (size_t)slot * H + h) + __ldg(d_att + rh);
        const float a = expf(leaky(pre, slope) - __ldg(seg_max + rh)) / __ldg(seg_sum + rh);
        const V *gm = reinterpret_cast<const V *>(g + (size_t)row * F) + h * head_vecs;
        const V *mm = reinterpret_cast<const V *>(mirror + (size_t)slot * F) + h * head_vecs;
        V *dm = reinterpret_cast<V *>(mirror_grad + (size_t)slot * F) + h * head_vecs;
        float dot = 0.f;
        for (uint32_t c = lane; c < head_vecs; c += 32) {
          V gv = __ldg(gm + c);
          dot += vec_dot(__ldg(mm + c), gv);
          red_add(dm + c, vec_scale(gv, a));
        }
        dot = warp_sum(dot);
        const float d_pre = a * (dot - __ldg(out_dot_g + rh)) * (pre > 0.f ? 1.f : slope);
        if (lane == 0)
          atomicAdd(s_grad + (size_t)slot * H + h, d_pre);
        d_acc += d_pre;
      }
      if (lane == 0 && d_acc != 0.f)
        atomicAdd(d_grad + (size_t)row * H + h, d_acc);
    }
  } // quantum loop
}

// ---- K7 backward without per-edge atomics: one destination-major and one source-major pass -------------------------
// The single-pass kernels above are destination-major, so every edge issues a vector `red` into its SOURCE's gradient
// row and a scalar atomic into its source's score gradient; on a power-law graph those collide on hub sources.  The two
// passes below walk the same edges twice, each time in the order in which ITS outputs are segment sums, so both keep
// register accumulators and write once per row (plain read-modify-write when the row lies inside the warp's edge
// quantum, `red`/atomicAdd only for rows cut by a quantum boundary):
//   destination-major (CSC): gathers mirror[slot(e)] and src_score[slot(e)], row constants g[dst], pack[dst]
//                            -> dst_score_grad[dst,h] = sum_e d_pre(e,h)
//   source-major (CSR):      gathers g[dst(e)] and pack[dst(e)], row constants mirror[slot], src_score[slot]
//                            -> mirror_grad[slot] = sum_e a(e,h) g[dst(e)],  src_score_grad[slot,h] = sum_e d_pre(e,h)
// pack[v,h] = { dst_score, seg_max + log(seg_sum), <out[v,h], g[v,h]>, 0 } so that one 16-byte load carries everything
// an edge needs about its destination:  a = exp(leaky(s + d) - lse),  d_pre = a (dot - <out,g>) leaky'(s + d).
constexpr uint32_t kBwdQuantum = 256;

__global__ void __launch_bounds__(kThreads)
    gat_pack_dst_kernel(float4 *__restrict__ pack, const float *__restrict__ d_att, const float *__restrict__ seg_max,
                        const float *__restrict__ seg_sum, const float *__restrict__ out_dot_g, uint64_t n) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    pack[i] = make_float4(__ldg(d_att + i), __ldg(seg_max + i) + logf(__ldg(seg_sum + i)), __ldg(out_dot_g + i), 0.f);
}

// VEC floats per lane load, KB chunks of 32 vectors per row, U edges gathered before any arithmetic.
// ONEHEAD: heads == 1, any row width (the dot product is a full-warp sum); otherwise a head is a power-of-two number
// of vectors <= 32 and per-head dots are segmented xor-shuffle sums (lanes of one head are contiguous).
// T: element type of `gathered` and `row_vals` (float, or __nv_bfloat16 with VEC in {2, 4, 8}: the rows are widened to
// FP32 in registers; F is then the BF16 row stride ld, which the FP32 `vec_out` shares).  Everything else is FP32.
template <int VEC, int KB, int U, bool SRC_MAJOR, bool ONEHEAD, class T = float>
__global__ void __launch_bounds__(kThreads)
    gat_backward_pass_kernel(float *__restrict__ vec_out, float *__restrict__ score_out,
                             const T *__restrict__ gathered, const T *__restrict__ row_vals,
                             const float *__restrict__ src_score, const float4 *__restrict__ dst_pack,
                             const uint32_t *__restrict__ col, const uint32_t *__restrict__ off,
                             const uint32_t *__restrict__ col_map, uint32_t n_rows, uint32_t F, uint32_t H,
                             float slope) {
  using V = typename Vec<VEC>::type;
  using L = typename Ld<T, VEC>::type; // what a lane loads per vector (FP32: V itself)
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t nvec = F / VEC;
  const uint32_t head_vecs = ONEHEAD ? 32u : nvec / H;
  uint32_t hk[KB];
  bool act[KB], lead[KB];
#pragma unroll
  for (int k = 0; k < KB; k++) {
    act[k] = lane + 32 * k < nvec;
    hk[k] = (ONEHEAD || !act[k]) ? 0u : (lane + 32 * k) / head_vecs;
    lead[k] = ONEHEAD ? (lane == 0 && k == 0) : (act[k] && (lane % head_vecs) == 0);
  }
  const uint32_t n_edges = __ldg(off + n_rows);
  const uint64_t nwarps = (uint64_t)gridDim.x * kWarps;
  for (uint64_t qw = (uint64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); qw * kBwdQuantum < n_edges; qw += nwarps) {
    const uint32_t e0 = (uint32_t)(qw * kBwdQuantum);
    const uint32_t e1 = (uint32_t)min((uint64_t)n_edges, (uint64_t)e0 + kBwdQuantum);
    uint32_t row = find_row(off, n_rows, e0);
    uint32_t row_begin = __ldg(off + row), row_end = __ldg(off + row + 1);
    V yv[KB], mg[KB];
    float rs[KB], acc[KB];
    float4 rp[KB];
    auto load_row = [&]() {
      const L *yr = reinterpret_cast<const L *>(row_vals + (size_t)row * F);
#pragma unroll
      for (int k = 0; k < KB; k++) {
        acc[k] = 0.f;
        if (act[k])
          yv[k] = widen(__ldg(yr + lane + 32 * k));
        if constexpr (SRC_MAJOR) {
          rs[k] = __ldg(src_score + (size_t)row * H + hk[k]);
          zero_vec(mg[k]);
        } else {
          rp[k] = __ldg(dst_pack + (size_t)row * H + hk[k]);
        }
      }
    };
    auto flush_row = [&]() {
      const bool whole = row_begin >= e0 && row_end <= e1; // no other warp touches this row
#pragma unroll
      for (int k = 0; k < KB; k++) {
        if constexpr (SRC_MAJOR) {
          if (act[k]) {
            V *o = reinterpret_cast<V *>(vec_out + (size_t)row * F) + lane + 32 * k;
            if (whole)
              *o = vec_add(*o, mg[k]);
            else
              red_add(o, mg[k]);
          }
        }
        if (lead[k]) {
          float *o = score_out + (size_t)row * H + hk[k];
          if (whole)
            *o += acc[k];
          else if (acc[k] != 0.f)
            atomicAdd(o, acc[k]);
        }
      }
    };
    load_row();
    for (uint32_t eb = e0; eb < e1; eb += 32) {
      const uint32_t cnt = min(32u, e1 - eb);
      uint32_t my_idx = 0;
      if (lane < cnt) {
        my_idx = __ldg(col + eb + lane);
        if (col_map)
          my_idx = __ldg(col_map + my_idx);
      }
      for (uint32_t j = 0; j < cnt; j += U) {
        L xv[U][KB];
        float es[U][KB];
        float4 ep[U][KB];
#pragma unroll
        for (int u = 0; u < U; u++) {
          const uint32_t idx = __shfl_sync(0xffffffffu, my_idx, min(j + u, cnt - 1));
          const L *xr = reinterpret_cast<const L *>(gathered + (size_t)idx * F);
#pragma unroll
          for (int k = 0; k < KB; k++) {
            if (act[k])
              xv[u][k] = __ldg(xr + lane + 32 * k);
            if constexpr (SRC_MAJOR)
              ep[u][k] = __ldg(dst_pack + (size_t)idx * H + hk[k]);
            else
              es[u][k] = __ldg(src_score + (size_t)idx * H + hk[k]);
          }
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
          const uint32_t e = eb + j + u;
          if (e >= e1)
            break;
          if (e >= row_end) {
            flush_row();
            do {
              row++;
              row_begin = row_end;
              row_end = __ldg(off + row + 1);
            } while (e >= row_end);
            load_row();
          }
          float dotk[KB];
#pragma unroll
          for (int k = 0; k < KB; k++)
            dotk[k] = act[k] ? vec_dot(widen(xv[u][k]), yv[k]) : 0.f;
          if constexpr (ONEHEAD) {
            float t = dotk[0];
#pragma unroll
            for (int k = 1; k < KB; k++)
              t += dotk[k];
            t = warp_sum(t);
#pragma unroll
            for (int k = 0; k < KB; k++)
              dotk[k] = t;
          } else {
#pragma unroll
            for (int k = 0; k < KB; k++)
              for (uint32_t o = head_vecs >> 1; o > 0; o >>= 1)
                dotk[k] += __shfl_xor_sync(0xffffffffu, dotk[k], o);
          }
#pragma unroll
          for (int k = 0; k < KB; k++) {
            const float sc = SRC_MAJOR ? rs[k] : es[u][k];
            const float4 pk = SRC_MAJOR ? ep[u][k] : rp[k];
            const float pre = sc + pk.x;
            const float a = expf(leaky(pre, slope) - pk.y);
            if constexpr (SRC_MAJOR) {
              if (act[k])
                mg[k] = vec_add(mg[k], vec_scale(widen(xv[u][k]), a));
            }
            acc[k] += a * (dotk[k] - pk.z) * (pre > 0.f ? 1.f : slope);
          }
        }
      }
    }
    flush_row();
  } // quantum loop
}

// ---- (vid,row) records read from mapped pinned host memory ---------------------------------------------------
template <bool ACCUM>
__global__ void __launch_bounds__(kThreads)
    records_kernel(float *__restrict__ dst, const float *__restrict__ records, uint32_t n_records, uint32_t F,
                   uint32_t start, uint32_t end) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warp0 = (uint64_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
  const uint64_t nwarps = (uint64_t)gridDim.x * kWarps;
  const size_t stride = (size_t)F + 1;
  for (uint64_t k = warp0; k < n_records; k += nwarps) {
    const float *rec = records + k * stride;
    const uint32_t vid = reinterpret_cast<const uint32_t *>(rec)[0];
    if (vid < start || vid >= end)
      continue;
    float *d = dst + (size_t)(vid - start) * F;
    for (uint32_t c = lane; c < F; c += 32) {
      float v = rec[1 + c];
      if (ACCUM)
        atomicAdd(d + c, v);
      else
        d[c] = v;
    }
  }
}

// ---- launch helpers ----------------------------------------------------------------------------------------
// persistent-style grid: enough CTAs to fill every SM several times over, work is grid-strided
static unsigned stream_grid(uint64_t rows) {
  uint64_t blocks = (rows + kWarps - 1) / kWarps;
  uint64_t cap = (uint64_t)sm_count() * 16;
  if (blocks > cap)
    blocks = cap;
  if (blocks == 0)
    blocks = 1;
  return (unsigned)blocks;
}
static unsigned full_grid() { return (unsigned)(sm_count() * 16); }

template <int MODE>
static int move_rows(float *dst, const float *src, const uint32_t *map1, const uint32_t *map2, uint64_t n_rows,
                     const uint32_t *n_rows_dev, uint32_t F, cudaStream_t st) {
  if ((n_rows == 0 && !n_rows_dev) || F == 0)
    return 0;
  NTS_ARG_CHECK(dst && src && map1, "null pointer passed to row mover");
  int vec = pick_vec(F, dst, src);
  unsigned grid = n_rows_dev ? full_grid() : stream_grid(n_rows);
  if (vec == 4)
    move_rows_kernel<4, MODE><<<grid, kThreads, 0, st>>>(dst, src, map1, map2, n_rows, n_rows_dev, F);
  else if (vec == 2)
    move_rows_kernel<2, MODE><<<grid, kThreads, 0, st>>>(dst, src, map1, map2, n_rows, n_rows_dev, F);
  else
    move_rows_kernel<1, MODE><<<grid, kThreads, 0, st>>>(dst, src, map1, map2, n_rows, n_rows_dev, F);
  NTS_LAUNCH_CHECK();
  return 0;
}

} // namespace nts

using namespace nts;

extern "C" {

int nts_gather_rows(float *dst, const float *src, const nts_vid_t *rows, nts_vid_t n_rows, nts_vid_t feature_size,
                    void *stream) {
  return move_rows<0>(dst, src, rows, nullptr, n_rows, nullptr, feature_size, as_stream(stream));
}

int nts_gather_rows_sharded(float *dst, const float *const *shards, const nts_vid_t *shard_offsets, int n_shards,
                            nts_vid_t shard_pitch, const nts_vid_t *ids, nts_vid_t n, nts_vid_t feature_size,
                            void *stream) {
  if (n == 0 || feature_size == 0)
    return 0;
  NTS_ARG_CHECK(dst && shards && shard_offsets && ids, "null pointer passed to nts_gather_rows_sharded");
  NTS_ARG_CHECK(n_shards >= 1 && n_shards <= kMaxShards, "nts_gather_rows_sharded needs 1..32 shards");
  NTS_ARG_CHECK(shard_pitch % 4 == 0 && shard_pitch >= feature_size,
                "nts_gather_rows_sharded: shard_pitch must be a multiple of 4 and at least feature_size");
  const uint32_t F = feature_size, nvec = (F + 3) / 4;
  const int svec = pick_vec(F, dst);
  const int lanes = nvec <= 8 ? 8 : (nvec <= 16 ? 16 : 32);
  const uint64_t rows_per_block = kThreads / lanes;
  const uint64_t cap = (uint64_t)sm_count() * 16;
  const unsigned grid = (unsigned)std::min<uint64_t>((n + rows_per_block - 1) / rows_per_block, cap);
  cudaStream_t st = as_stream(stream);
  if (lanes == 8)
    launch_gather_rows_sharded<8>(svec, grid, st, dst, shards, shard_offsets, n_shards, shard_pitch, ids, n, F);
  else if (lanes == 16)
    launch_gather_rows_sharded<16>(svec, grid, st, dst, shards, shard_offsets, n_shards, shard_pitch, ids, n, F);
  else
    launch_gather_rows_sharded<32>(svec, grid, st, dst, shards, shard_offsets, n_shards, shard_pitch, ids, n, F);
  NTS_LAUNCH_CHECK();
  return 0;
}

int nts_gather_rows_sharded_bf16(void *dst, int dst_dtype, nts_vid_t dst_ld, const void *const *shards,
                                 const nts_vid_t *shard_offsets, int n_shards, nts_vid_t shard_pitch,
                                 const nts_vid_t *ids, nts_vid_t n, nts_vid_t feature_size, void *stream) {
  NTS_ARG_CHECK(dst_dtype == NTS_DTYPE_BF16 || dst_dtype == NTS_DTYPE_F32,
                "nts_gather_rows_sharded_bf16: dst_dtype must be NTS_DTYPE_BF16 or NTS_DTYPE_F32");
  NTS_ARG_CHECK(shard_pitch % 8 == 0 && shard_pitch >= feature_size,
                "nts_gather_rows_sharded_bf16: shard_pitch must be a multiple of 8 and at least feature_size");
  NTS_ARG_CHECK(dst_dtype == NTS_DTYPE_F32 ? dst_ld == feature_size : (dst_ld % 8 == 0 && dst_ld >= feature_size),
                "nts_gather_rows_sharded_bf16: dst_ld must be feature_size (FP32) or a multiple of 8 >= feature_size "
                "(BF16)");
  if (n == 0 || feature_size == 0)
    return 0;
  NTS_ARG_CHECK(dst && shards && shard_offsets && ids, "null pointer passed to nts_gather_rows_sharded_bf16");
  NTS_ARG_CHECK(n_shards >= 1 && n_shards <= kMaxShards, "nts_gather_rows_sharded_bf16 needs 1..32 shards");
  NTS_ARG_CHECK(dst_dtype == NTS_DTYPE_F32 || aligned_to(dst, 16),
                "nts_gather_rows_sharded_bf16: BF16 rows need a 16-byte aligned dst");
  const uint32_t F = feature_size, nvec = (F + 7) / 8;
  const int svec = dst_dtype == NTS_DTYPE_BF16 ? 0 : pick_vec(F, dst);
  const int lanes = nvec <= 8 ? 8 : (nvec <= 16 ? 16 : 32);
  const uint64_t rows_per_block = kThreads / lanes;
  const uint64_t cap = (uint64_t)sm_count() * 16;
  const unsigned grid = (unsigned)std::min<uint64_t>((n + rows_per_block - 1) / rows_per_block, cap);
  cudaStream_t st = as_stream(stream);
  const uint4 *const *sh = reinterpret_cast<const uint4 *const *>(shards);
  if (lanes == 8)
    launch_gather_rows_sharded_bf16<8>(svec, grid, st, dst, dst_ld, sh, shard_offsets, n_shards, shard_pitch, ids, n, F);
  else if (lanes == 16)
    launch_gather_rows_sharded_bf16<16>(svec, grid, st, dst, dst_ld, sh, shard_offsets, n_shards, shard_pitch, ids, n,
                                        F);
  else
    launch_gather_rows_sharded_bf16<32>(svec, grid, st, dst, dst_ld, sh, shard_offsets, n_shards, shard_pitch, ids, n,
                                        F);
  NTS_LAUNCH_CHECK();
  return 0;
}

int nts_scatter_add_rows(float *dst, const float *src, const nts_vid_t *rows, nts_vid_t n_rows,
                         nts_vid_t feature_size, void *stream) {
  return move_rows<1>(dst, src, rows, nullptr, n_rows, nullptr, feature_size, as_stream(stream));
}

int nts_scatter_add_rows_atomic(float *dst, const float *src, const nts_vid_t *rows, nts_vid_t n_rows,
                                nts_vid_t feature_size, void *stream) {
  return move_rows<2>(dst, src, rows, nullptr, n_rows, nullptr, feature_size, as_stream(stream));
}

// The edge count E_p = column_offset[batch_size] is read by the kernels on the device (the reference keeps
// e_size on the host inside deviceCSC; its Cuda_Stream signatures do not pass it).
int nts_scatter_src_mirror_to_msg(float *message, const float *src_mirror_feature, const nts_vid_t *row_indices,
                                  const nts_vid_t *column_offset, const nts_vid_t *mirror_index,
                                  nts_vid_t batch_size, nts_vid_t feature_size, void *stream) {
  if (batch_size == 0)
    return 0;
  NTS_ARG_CHECK(column_offset && mirror_index, "null graph pointer");
  return move_rows<0>(message, src_mirror_feature, row_indices, mirror_index, 0, column_offset + batch_size,
                      feature_size, as_stream(stream));
}

int nts_gather_msg_to_src_mirror(float *src_mirror_feature, const float *message, const nts_vid_t *row_indices,
                                 const nts_vid_t *column_offset, const nts_vid_t *mirror_index,
                                 nts_vid_t batch_size, nts_vid_t feature_size, void *stream) {
  if (batch_size == 0)
    return 0;
  NTS_ARG_CHECK(column_offset && mirror_index, "null graph pointer");
  return move_rows<2>(src_mirror_feature, message, row_indices, mirror_index, 0, column_offset + batch_size,
                      feature_size, as_stream(stream));
}

static int segment_broadcast(float *msg, const float *x, const nts_vid_t *column_offset, nts_vid_t batch_size,
                             nts_vid_t F, bool accum, cudaStream_t st) {
  if (batch_size == 0 || F == 0)
    return 0;
  NTS_ARG_CHECK(msg && x && column_offset, "null pointer passed to segment broadcast");
  int vec = pick_vec(F, msg, x);
  unsigned grid = full_grid();
#define NTS_BCAST(V_)                                                                                     \
  if (accum)                                                                                              \
    segment_broadcast_kernel<V_, true><<<grid, kThreads, 0, st>>>(msg, x, column_offset, batch_size, F);  \
  else                                                                                                    \
    segment_broadcast_kernel<V_, false><<<grid, kThreads, 0, st>>>(msg, x, column_offset, batch_size, F);
  if (vec == 4) {
    NTS_BCAST(4)
  } else if (vec == 2) {
    NTS_BCAST(2)
  } else {
    NTS_BCAST(1)
  }
#undef NTS_BCAST
  NTS_LAUNCH_CHECK();
  return 0;
}

int nts_scatter_dst_to_msg(float *message, const float *dst_feature, const nts_vid_t *row_indices,
                           const nts_vid_t *column_offset, nts_vid_t batch_size, nts_vid_t feature_size,
                           void *stream) {
  (void)row_indices;
  return segment_broadcast(message, dst_feature, column_offset, batch_size, feature_size, false, as_stream(stream));
}

int nts_scatter_grad_back_to_message(const float *input, float *message_grad, const nts_vid_t *row_indices,
                                     const nts_vid_t *column_offset, nts_vid_t batch_size, nts_vid_t feature_size,
                                     void *stream) {
  (void)row_indices;
  return segment_broadcast(message_grad, input, column_offset, batch_size, feature_size, true, as_stream(stream));
}

int nts_gather_msg_to_dst(float *dst_feature, const float *message, const nts_vid_t *row_indices,
                          const nts_vid_t *column_offset, nts_vid_t batch_size, nts_vid_t feature_size,
                          void *stream) {
  (void)row_indices;
  cudaStream_t st = as_stream(stream);
  if (batch_size == 0 || feature_size == 0)
    return 0;
  NTS_ARG_CHECK(dst_feature && message && column_offset, "null pointer passed to gather_msg_to_dst");
  int vec = pick_vec(feature_size, dst_feature, message);
  unsigned grid = full_grid();
  if (vec == 4)
    segment_sum_kernel<4><<<grid, kThreads, 0, st>>>(dst_feature, message, column_offset, batch_size, feature_size);
  else if (vec == 2)
    segment_sum_kernel<2><<<grid, kThreads, 0, st>>>(dst_feature, message, column_offset, batch_size, feature_size);
  else
    segment_sum_kernel<1><<<grid, kThreads, 0, st>>>(dst_feature, message, column_offset, batch_size, feature_size);
  NTS_LAUNCH_CHECK();
  return 0;
}

int nts_edge_softmax_forward(float *msg_output, const float *msg_input, float *msg_cached,
                             const nts_vid_t *row_indices, const nts_vid_t *column_offset, nts_vid_t batch_size,
                             nts_vid_t feature_size, void *stream) {
  (void)row_indices;
  if (batch_size == 0 || feature_size == 0)
    return 0;
  NTS_ARG_CHECK(msg_output && msg_input && column_offset, "null pointer passed to edge softmax");
  unsigned grid = (batch_size + kRowsPerCta - 1) / kRowsPerCta;
  edge_softmax_kernel<false><<<grid, kThreads, 0, as_stream(stream)>>>(msg_output, msg_input, nullptr, msg_cached,
                                                                       column_offset, batch_size, feature_size);
  NTS_LAUNCH_CHECK();
  return 0;
}

int nts_edge_softmax_backward(float *msg_input_grad, const float *msg_output_grad, const float *msg_cached,
                              const nts_vid_t *row_indices, const nts_vid_t *column_offset, nts_vid_t batch_size,
                              nts_vid_t feature_size, void *stream) {
  (void)row_indices;
  if (batch_size == 0 || feature_size == 0)
    return 0;
  NTS_ARG_CHECK(msg_input_grad && msg_output_grad && msg_cached && column_offset,
                "null pointer passed to edge softmax backward");
  unsigned grid = (batch_size + kRowsPerCta - 1) / kRowsPerCta;
  edge_softmax_kernel<true><<<grid, kThreads, 0, as_stream(stream)>>>(msg_input_grad, msg_output_grad, msg_cached,
                                                                      nullptr, column_offset, batch_size,
                                                                      feature_size);
  NTS_LAUNCH_CHECK();
  return 0;
}

int nts_aggregate_dst_fuse_weight_backward_heads(float *mirror_grad, float *edge_weight_grad, const float *mirror,
                                                 const float *edge_weight, const float *dst_grad,
                                                 const nts_vid_t *row_indices, const nts_vid_t *column_offset,
                                                 const nts_vid_t *mirror_index, nts_vid_t batch_size,
                                                 nts_vid_t feature_size, nts_vid_t heads, void *stream) {
  cudaStream_t st = as_stream(stream);
  if (batch_size == 0 || feature_size == 0)
    return 0;
  NTS_ARG_CHECK(mirror_grad && edge_weight_grad && mirror && edge_weight && dst_grad && row_indices &&
                    column_offset && mirror_index,
                "null pointer passed to fuse-weight backward");
  NTS_ARG_CHECK(heads >= 1 && feature_size % heads == 0, "feature_size must be a multiple of heads");
  int vec = pick_vec(feature_size, mirror_grad, mirror, dst_grad);
  while (vec > 1 && (feature_size / heads) % vec != 0)
    vec >>= 1;
  unsigned grid = full_grid();
  if (vec == 4)
    fuse_weight_backward_kernel<4><<<grid, kThreads, 0, st>>>(mirror_grad, edge_weight_grad, mirror, edge_weight,
                                                              dst_grad, row_indices, column_offset, mirror_index,
                                                              batch_size, feature_size, heads);
  else if (vec == 2)
    fuse_weight_backward_kernel<2><<<grid, kThreads, 0, st>>>(mirror_grad, edge_weight_grad, mirror, edge_weight,
                                                              dst_grad, row_indices, column_offset, mirror_index,
                                                              batch_size, feature_size, heads);
  else
    fuse_weight_backward_kernel<1><<<grid, kThreads, 0, st>>>(mirror_grad, edge_weight_grad, mirror, edge_weight,
                                                              dst_grad, row_indices, column_offset, mirror_index,
                                                              batch_size, feature_size, heads);
  NTS_LAUNCH_CHECK();
  return 0;
}

int nts_aggregate_dst_fuse_weight_backward(float *mirror_grad, float *edge_weight_grad, const float *mirror,
                                           const float *edge_weight, const float *dst_grad,
                                           const nts_vid_t *row_indices, const nts_vid_t *column_offset,
                                           const nts_vid_t *mirror_index, nts_vid_t batch_size,
                                           nts_vid_t feature_size, void *stream) {
  return nts_aggregate_dst_fuse_weight_backward_heads(mirror_grad, edge_weight_grad, mirror, edge_weight, dst_grad,
                                                      row_indices, column_offset, mirror_index, batch_size,
                                                      feature_size, 1, stream);
}

int nts_gat_softmax_stats(float *seg_max, float *seg_sum, const float *src_score, const float *dst_score,
                          const nts_vid_t *row_indices, const nts_vid_t *column_offset, const nts_vid_t *mirror_index,
                          nts_vid_t batch_size, nts_vid_t heads, float negative_slope, void *stream) {
  if (batch_size == 0 || heads == 0)
    return 0;
  NTS_ARG_CHECK(seg_max && seg_sum && src_score && dst_score && row_indices && column_offset,
                "null pointer passed to gat_softmax_stats");
  unsigned grid = (batch_size + kRowsPerCta - 1) / kRowsPerCta;
  cudaStream_t st = as_stream(stream);
#define NTS_STATS(H_)                                                                                           \
  do {                                                                                                          \
    gat_stats_init_kernel<<<stream_grid(((uint64_t)batch_size * heads + kThreads - 1) / kThreads), kThreads, 0, \
                            st>>>(seg_max, seg_sum, column_offset, batch_size, heads);                          \
    count_launch();                                                                                             \
    gat_edge_stats_kernel<H_, 0><<<full_grid(), kThreads, 0, st>>>(seg_max, seg_sum, src_score, dst_score,      \
                                                                     row_indices, column_offset, mirror_index,   \
                                                                     batch_size, negative_slope);                \
    count_launch();                                                                                             \
    gat_edge_stats_kernel<H_, 1><<<full_grid(), kThreads, 0, st>>>(seg_max, seg_sum, src_score, dst_score,      \
                                                                     row_indices, column_offset, mirror_index,   \
                                                                     batch_size, negative_slope);                \
  } while (0)
  switch (heads) { // edge-balanced kernels when the head count divides the warp
  case 1: NTS_STATS(1); break;
  case 2: NTS_STATS(2); break;
  case 4: NTS_STATS(4); break;
  case 8: NTS_STATS(8); break;
  case 16: NTS_STATS(16); break;
  case 32: NTS_STATS(32); break;
  default:
    gat_softmax_stats_kernel<<<grid, kThreads, 0, st>>>(seg_max, seg_sum, src_score, dst_score, row_indices,
                                                        column_offset, mirror_index, batch_size, heads,
                                                        negative_slope);
  }
#undef NTS_STATS
  NTS_LAUNCH_CHECK();
  return 0;
}

int nts_gat_fused_aggregate_backward(float *mirror_grad, float *src_score_grad, float *dst_score_grad,
                                     const float *mirror, const float *src_score, const float *dst_score,
                                     const float *seg_max, const float *seg_sum, const float *out_dot_grad,
                                     const float *dst_grad, const nts_vid_t *row_indices,
                                     const nts_vid_t *column_offset, const nts_vid_t *mirror_index,
                                     nts_vid_t batch_size, nts_vid_t feature_size, nts_vid_t heads,
                                     float negative_slope, void *stream) {
  cudaStream_t st = as_stream(stream);
  if (batch_size == 0 || feature_size == 0)
    return 0;
  NTS_ARG_CHECK(mirror_grad && src_score_grad && dst_score_grad && mirror && src_score && dst_score && seg_max &&
                    seg_sum && out_dot_grad && dst_grad && row_indices && column_offset,
                "null pointer passed to fused GAT backward");
  NTS_ARG_CHECK(heads >= 1 && feature_size % heads == 0, "feature_size must be a multiple of heads");
  int vec = pick_vec(feature_size, mirror_grad, mirror, dst_grad);
  while (vec > 1 && (feature_size / heads) % vec != 0)
    vec >>= 1;
  unsigned grid = full_grid();
  // single-pass kernel: prefer the vector width that keeps the most lanes busy, needs a power-of-two number of
  // vectors per head (<= 32) and at most 4 chunks per lane
  {
    int sv = vec;
    while (sv > 1 && feature_size / sv < 32)
      sv >>= 1;
    const uint32_t nvec = feature_size / sv, hv = nvec / heads;
    const bool pow2 = hv >= 1 && (hv & (hv - 1)) == 0 && hv <= 32 && hv * heads == nvec;
    const uint32_t kb = (nvec + 31) / 32;
    if (pow2 && kb <= 4) {
#define NTS_GATS(V_, K_)                                                                                         \
  gat_fused_backward_seg_kernel<V_, K_><<<grid, kThreads, 0, st>>>(                                              \
      mirror_grad, src_score_grad, dst_score_grad, mirror, src_score, dst_score, seg_max, seg_sum, out_dot_grad, \
      dst_grad, row_indices, column_offset, mirror_index, batch_size, feature_size, heads, negative_slope)
#define NTS_GATS_K(V_)                                                                                           \
  if (kb == 1)                                                                                                   \
    NTS_GATS(V_, 1);                                                                                             \
  else if (kb == 2)                                                                                              \
    NTS_GATS(V_, 2);                                                                                             \
  else                                                                                                           \
    NTS_GATS(V_, 4)
      if (sv == 4) {
        NTS_GATS_K(4);
      } else if (sv == 2) {
        NTS_GATS_K(2);
      } else {
        NTS_GATS_K(1);
      }
#undef NTS_GATS_K
#undef NTS_GATS
      NTS_LAUNCH_CHECK();
      return 0;
    }
  }
#define NTS_GATB(V_)                                                                                           \
  gat_fused_backward_kernel<V_><<<grid, kThreads, 0, st>>>(mirror_grad, src_score_grad, dst_score_grad, mirror, \
                                                           src_score, dst_score, seg_max, seg_sum, out_dot_grad, \
                                                           dst_grad, row_indices, column_offset, mirror_index,  \
                                                           batch_size, feature_size, heads, negative_slope)
  if (vec == 4)
    NTS_GATB(4);
  else if (vec == 2)
    NTS_GATB(2);
  else
    NTS_GATB(1);
#undef NTS_GATB
  NTS_LAUNCH_CHECK();
  return 0;
}

int nts_gat_fused_aggregate_backward_two_pass(float *mirror_grad, float *src_score_grad, float *dst_score_grad,
                                              float *dst_pack, const float *mirror, const float *src_score,
                                              const float *dst_score, const float *seg_max, const float *seg_sum,
                                              const float *out_dot_grad, const float *dst_grad,
                                              const nts_vid_t *row_indices, const nts_vid_t *column_offset,
                                              const nts_vid_t *mirror_index, const nts_vid_t *slot_row_offset,
                                              const nts_vid_t *slot_column_indices, nts_vid_t batch_size,
                                              nts_vid_t mirror_size, nts_vid_t feature_size, nts_vid_t heads,
                                              float negative_slope, void *stream) {
  cudaStream_t st = as_stream(stream);
  if (batch_size == 0 || feature_size == 0 || mirror_size == 0)
    return 0;
  NTS_ARG_CHECK(mirror_grad && src_score_grad && dst_score_grad && dst_pack && mirror && src_score && dst_score &&
                    seg_max && seg_sum && out_dot_grad && dst_grad && row_indices && column_offset &&
                    slot_row_offset && slot_column_indices,
                "null pointer passed to fused GAT backward (two pass)");
  NTS_ARG_CHECK(heads >= 1 && feature_size % heads == 0, "feature_size must be a multiple of heads");
  NTS_ARG_CHECK((reinterpret_cast<uintptr_t>(dst_pack) & 15) == 0, "dst_pack must be 16-byte aligned");
  int vec = pick_vec(feature_size, mirror_grad, mirror, dst_grad);
  while (vec > 1 && (feature_size / heads) % vec != 0)
    vec >>= 1;
  while (vec > 1 && feature_size / vec < 32) // keep all 32 lanes busy on narrow rows
    vec >>= 1;
  const uint32_t nvec = feature_size / vec, hv = nvec / heads;
  const uint32_t kb = (nvec + 31) / 32;
  const bool one = heads == 1;
  const bool pow2 = hv >= 1 && (hv & (hv - 1)) == 0 && hv <= 32;
  if (kb > 4 || !(one || pow2)) // shapes the register-accumulator passes do not cover: single pass with atomics
    return nts_gat_fused_aggregate_backward(mirror_grad, src_score_grad, dst_score_grad, mirror, src_score, dst_score,
                                            seg_max, seg_sum, out_dot_grad, dst_grad, row_indices, column_offset,
                                            mirror_index, batch_size, feature_size, heads, negative_slope, stream);
  const uint64_t n_pack = (uint64_t)batch_size * heads;
  gat_pack_dst_kernel<<<stream_grid((n_pack + kThreads - 1) / kThreads), kThreads, 0, st>>>(
      reinterpret_cast<float4 *>(dst_pack), dst_score, seg_max, seg_sum, out_dot_grad, n_pack);
  NTS_LAUNCH_CHECK();
  const unsigned grid = full_grid();
  const float4 *pk = reinterpret_cast<const float4 *>(dst_pack);
#define NTS_GAT2(V_, K_, U_, ONE_)                                                                                   \
  do {                                                                                                               \
    gat_backward_pass_kernel<V_, K_, U_, false, ONE_><<<grid, kThreads, 0, st>>>(                                    \
        nullptr, dst_score_grad, mirror, dst_grad, src_score, pk, row_indices, column_offset, mirror_index,          \
        batch_size, feature_size, heads, negative_slope);                                                            \
    count_launch();                                                                                                  \
    gat_backward_pass_kernel<V_, K_, U_, true, ONE_><<<grid, kThreads, 0, st>>>(                                     \
        mirror_grad, src_score_grad, dst_grad, mirror, src_score, pk, slot_column_indices, slot_row_offset, nullptr, \
        mirror_size, feature_size, heads, negative_slope);                                                           \
  } while (0)
#define NTS_GAT2_K(V_, ONE_)                                                                                         \
  do {                                                                                                               \
    if (kb == 1)                                                                                                     \
      NTS_GAT2(V_, 1, 4, ONE_);                                                                                      \
    else if (kb == 2)                                                                                                \
      NTS_GAT2(V_, 2, 2, ONE_);                                                                                      \
    else                                                                                                             \
      NTS_GAT2(V_, 4, 1, ONE_);                                                                                      \
  } while (0)
#define NTS_GAT2_V(ONE_)                                                                                             \
  do {                                                                                                               \
    if (vec == 4)                                                                                                    \
      NTS_GAT2_K(4, ONE_);                                                                                           \
    else if (vec == 2)                                                                                               \
      NTS_GAT2_K(2, ONE_);                                                                                           \
    else                                                                                                             \
      NTS_GAT2_K(1, ONE_);                                                                                           \
  } while (0)
  if (one)
    NTS_GAT2_V(true);
  else
    NTS_GAT2_V(false);
#undef NTS_GAT2_V
#undef NTS_GAT2_K
#undef NTS_GAT2
  NTS_LAUNCH_CHECK();
  return 0;
}

int nts_gat_fused_aggregate_backward_two_pass_bf16(float *mirror_grad, float *src_score_grad, float *dst_score_grad,
                                                   float *dst_pack, const void *mirror, const float *src_score,
                                                   const float *dst_score, const float *seg_max, const float *seg_sum,
                                                   const float *out_dot_grad, const void *dst_grad,
                                                   const nts_vid_t *row_indices, const nts_vid_t *column_offset,
                                                   const nts_vid_t *mirror_index, const nts_vid_t *slot_row_offset,
                                                   const nts_vid_t *slot_column_indices, nts_vid_t batch_size,
                                                   nts_vid_t mirror_size, nts_vid_t feature_size, nts_vid_t ld,
                                                   nts_vid_t heads, float negative_slope, void *stream) {
  if (const int rc = check_gat_bf16_layout(feature_size, ld, heads))
    return rc;
  // the shape rule of the FP32 passes on rows of ld BF16 values: 2, 4 or 8 values per lane (as wide as keeps 32 lanes
  // busy), a power-of-two number of vectors per head (<= 32) and at most 4 chunks per lane; there is no fallback
  int vec = 8;
  while (vec > 2 && ld / vec < 32)
    vec >>= 1;
  const uint32_t nvec = ld / vec, hv = nvec / heads;
  const uint32_t kb = (nvec + 31) / 32;
  const bool one = heads == 1;
  NTS_ARG_CHECK(kb <= 4 && (one || (hv >= 1 && (hv & (hv - 1)) == 0 && hv <= 32)),
                "no BF16 two-pass GAT backward for this shape (heads > 1 need a power-of-two number of vectors per "
                "head, rows at most 1024 values)");
  cudaStream_t st = as_stream(stream);
  if (batch_size == 0 || feature_size == 0 || mirror_size == 0)
    return 0;
  NTS_ARG_CHECK(mirror_grad && src_score_grad && dst_score_grad && dst_pack && mirror && src_score && dst_score &&
                    seg_max && seg_sum && out_dot_grad && dst_grad && row_indices && column_offset &&
                    slot_row_offset && slot_column_indices,
                "null pointer passed to fused GAT backward (two pass, BF16)");
  NTS_ARG_CHECK(aligned_to(mirror_grad, 16) && aligned_to(mirror, 16) && aligned_to(dst_grad, 16) &&
                    aligned_to(dst_pack, 16),
                "BF16 fused GAT backward needs 16-byte aligned mirror_grad, mirror, dst_grad and dst_pack");
  const uint64_t n_pack = (uint64_t)batch_size * heads;
  gat_pack_dst_kernel<<<stream_grid((n_pack + kThreads - 1) / kThreads), kThreads, 0, st>>>(
      reinterpret_cast<float4 *>(dst_pack), dst_score, seg_max, seg_sum, out_dot_grad, n_pack);
  NTS_LAUNCH_CHECK();
  const unsigned grid = full_grid();
  const float4 *pk = reinterpret_cast<const float4 *>(dst_pack);
  const __nv_bfloat16 *m16 = static_cast<const __nv_bfloat16 *>(mirror);
  const __nv_bfloat16 *g16 = static_cast<const __nv_bfloat16 *>(dst_grad);
#define NTS_GAT2B(V_, K_, UD_, US_, ONE_)                                                                            \
  do {                                                                                                               \
    gat_backward_pass_kernel<V_, K_, UD_, false, ONE_, __nv_bfloat16><<<grid, kThreads, 0, st>>>(                    \
        nullptr, dst_score_grad, m16, g16, src_score, pk, row_indices, column_offset, mirror_index, batch_size, ld,   \
        heads, negative_slope);                                                                                      \
    count_launch();                                                                                                  \
    gat_backward_pass_kernel<V_, K_, US_, true, ONE_, __nv_bfloat16><<<grid, kThreads, 0, st>>>(                     \
        mirror_grad, src_score_grad, g16, m16, src_score, pk, slot_column_indices, slot_row_offset, nullptr,         \
        mirror_size, ld, heads, negative_slope);                                                                     \
  } while (0)
  // vec = 2 / 4 only on rows of fewer than 128 / 256 values (kb <= 2); vec = 8 for the wider ones.  U per pass is the
  // FP32 choice except where that point spills with BF16 rows (single-head passes: dst-major VEC 2 x KB 1 at U = 8,
  // src-major 2 x 2 and 8 x 2 at U = 4, all spill-free)
#define NTS_GAT2B_ONE(ONE_)                                                                                          \
  do {                                                                                                               \
    if (vec == 2) {                                                                                                  \
      if (kb == 1)                                                                                                   \
        NTS_GAT2B(2, 1, ONE_ ? 8 : 4, 4, ONE_);                                                                      \
      else                                                                                                           \
        NTS_GAT2B(2, 2, 2, ONE_ ? 4 : 2, ONE_);                                                                      \
    } else if (vec == 4) {                                                                                           \
      if (kb == 1)                                                                                                   \
        NTS_GAT2B(4, 1, 4, 4, ONE_);                                                                                 \
      else                                                                                                           \
        NTS_GAT2B(4, 2, 2, 2, ONE_);                                                                                 \
    } else if (kb == 1) {                                                                                            \
      NTS_GAT2B(8, 1, 4, 4, ONE_);                                                                                   \
    } else if (kb == 2) {                                                                                            \
      NTS_GAT2B(8, 2, 2, ONE_ ? 4 : 2, ONE_);                                                                        \
    } else {                                                                                                         \
      NTS_GAT2B(8, 4, 1, 1, ONE_);                                                                                   \
    }                                                                                                                \
  } while (0)
  if (one)
    NTS_GAT2B_ONE(true);
  else
    NTS_GAT2B_ONE(false);
#undef NTS_GAT2B_ONE
#undef NTS_GAT2B
  NTS_LAUNCH_CHECK();
  return 0;
}

int nts_deserialize_records(float *mirror, const float *records, nts_vid_t n_records, nts_vid_t feature_size,
                            nts_vid_t partition_start, nts_vid_t partition_end, void *stream) {
  if (n_records == 0)
    return 0;
  NTS_ARG_CHECK(mirror && records, "null pointer passed to deserialize_records");
  records_kernel<false><<<stream_grid(n_records), kThreads, 0, as_stream(stream)>>>(
      mirror, records, n_records, feature_size, partition_start, partition_end);
  NTS_LAUNCH_CHECK();
  return 0;
}

int nts_aggregate_records(float *aggregate, const float *records, nts_vid_t n_records, nts_vid_t feature_size,
                          nts_vid_t partition_start, nts_vid_t partition_end, void *stream) {
  if (n_records == 0)
    return 0;
  NTS_ARG_CHECK(aggregate && records, "null pointer passed to aggregate_records");
  records_kernel<true><<<stream_grid(n_records), kThreads, 0, as_stream(stream)>>>(
      aggregate, records, n_records, feature_size, partition_start, partition_end);
  NTS_LAUNCH_CHECK();
  return 0;
}

} // extern "C"
