// nts_gather_plan: a chunk's (offsets, indices, weight) arrays preprocessed ONCE for repeated aggregation, and the
// kernel that consumes them.  Same contraction as segment_gather_sum_kernel (nts_aggregate.cu) -
//
//   out[r,:] += sum_{e in [off[r], off[r+1])} in[row(e),:] * w[e]
//
// i.e. Cuda_Stream::Gather_By_Dst_From_Src / Gather_By_Src_From_Dst (cuda/ntsCUDAGraphOP.cu:157-281) - but with the
// three things a profile of that kernel asks for (it is bound by the L1 data stage every gathered byte crosses, and
// re-reads the feature matrix from DRAM many times over):
//
//   1. source-slab bucketing.  Edges are regrouped by (slab of the gathered row, output row): slab s holds the
//      edges whose gathered row lies in rows [s*slab_rows, (s+1)*slab_rows) of the input matrix, sized so that one
//      slab of the matrix stays resident in the 50 MB L2.  One launch per slab, in stream order, so at any moment
//      the CTAs in flight gather from ONE slab; the output row of a (slab, row) segment is finished with a plain
//      read-modify-write exactly like the unbucketed kernel (launches never overlap, so no extra atomics).
//      The bucketing is a stable sort by (slab, row): inside a segment the edges keep the order of the reference
//      layout (core/PartitionedGraph.hpp:389-405), summation order per output element changes only in where the
//      partial sums of the slabs are added.
//   2. (row, weight) pairs.  The base / slot lookup is applied at plan time and row index and weight are stored
//      interleaved, so the per-edge broadcast read from shared memory is ONE 8-byte LDS instead of two 4-byte ones,
//      and the TMA bulk copy (cp.async.bulk -> SASS UBLKCP) stages one array per CTA instead of two.
//   3. 16-byte feature loads for every width.  An input whose row pitch is a multiple of 4 floats is gathered in
//      place; rows whose byte length is not a multiple of 16 (a contiguous F = 602 input: 2408 B) are copied once per
//      call into a workspace with rows padded to a multiple of 4 floats, so the gather always uses float4 loads on
//      16-byte aligned rows and one warp covers up to 640 columns: 19 + 1 data-stage wavefronts per edge at F = 602
//      instead of 21.6 + 4.
//
// Plan construction (hand-written kernels + one CUB radix sort) replaces nothing in the reference: its chunks are
// built on the host by single-threaded loops (core/PartitionedGraph.hpp:324-420) and never re-bucketed.
//
// BF16 gathers (nts_gather_plan_run_bf16_ex): the gathered operand is read as BF16 rows (round-to-nearest-even of the
// FP32 input, one conversion pass per call into the plan's workspace at a stride of ceil(F/8)*8) and widened to FP32
// in registers; weights, accumulators and outputs stay FP32.  A 16-byte load then carries 8 values instead of 4, so
// every gathered edge moves half the bytes through L2 and the L1 data stage.
#include <cub/cub.cuh>
#include <cuda_bf16.h>

#include <algorithm>
#include <type_traits>
#include <vector>

#include "nts_common.cuh"

struct nts_gather_plan {
  uint32_t n_rows = 0;         // output rows
  uint64_t n_edges = 0;
  uint32_t gather_rows = 0;    // rows of the gathered matrix
  int slabs = 1;
  uint32_t slab_rows = 0;
  uint2 *pairs = nullptr;      // [n_edges] {gathered row, weight bits}, slab-major, then output row, then original order
  uint32_t *voff = nullptr;    // [slabs * n_rows + 1] offsets of the (slab, row) segments
  std::vector<uint64_t> slab_edge; // [slabs + 1] host copy of voff[s * n_rows]
  float *workspace = nullptr;  // padded copy of the input when its rows are not 16-byte multiples / aligned
  size_t workspace_floats = 0;
  __nv_bfloat16 *workspace_bf16 = nullptr; // BF16 copy of the input for BF16 gathers (rows padded to 8 values)
  size_t workspace_bf16_elems = 0;
  // dense hub blocks (nts_gather_plan_create_hybrid); the slab-bucketed pairs hold the remaining edges only
  int hub_cols = 0, hub_rows = 0;
  uint32_t *hub_col_ids = nullptr; // [hub_cols] gathered rows of the column block, most referenced first
  uint32_t *hub_row_ids = nullptr; // [hub_rows] output rows of the row block, longest segment first
  uint32_t lda_c = 0, lda_r = 0;   // n_rows / hub_rows rounded up to a multiple of 4 (16-byte operand rows)
  float *dense = nullptr;          // D_c^T [hub_cols x lda_c], then D_r^T [gather_rows x lda_r]: summed edge weights
  size_t dense_floats = 0;
  int overlap = 0;                 // 1: the row block runs inside the slab launches (planned_slab_hub_kernel)
  int last_grid = 0, last_launches = 0, last_k = 0, last_u = 0, last_outv = 0;
  float tuned_ms = 0.f;        // measured plans (tune_plan): time of the winning candidate
};

namespace nts {

static int g_plan_u = 0, g_plan_minb = 0, g_plan_q = 0, g_plan_variant = 0; // measurement hooks (NTS_PLAN_TUNE="U,MINB[,Q]"), 0 = default

// ---- plan construction kernels -----------------------------------------------------------------------------------
// The mapped (gathered) row of edge e of a part: index_add + (slot_of[idx[e]] or idx[e] - index_base)
__device__ __forceinline__ uint32_t plan_gathered_row(const nts_plan_part &pt, uint32_t e) {
  const uint32_t id = __ldg(pt.indices + e);
  return (pt.slot_of ? __ldg(pt.slot_of + id) : id - pt.index_base) + pt.index_add;
}

constexpr uint32_t kNoHub = 0xffffffffu;

// Edge e of part pt is plan edge e_off + e, its output row row_add + (part-local row):
// key[e_off + e] = slab(gathered row) * n_rows + output row, val[e_off + e] = e_off + e.
// KeyT = uint64_t (a single part with hub blocks): an edge whose gathered row is a hub column goes to cell (slot, row)
// of the column block D_c^T [hub_cols x lda_c]; else an edge of a hub row goes to cell (gathered row, slot) of the row
// block D_r^T [gather_rows x lda_r]; both as n_keys + the cell's offset in the dense buffer, so they sort past every
// residual (slab, row) key and voff[n_keys] is the residual edge count.
template <class KeyT>
__global__ void plan_keys_kernel(nts_plan_part pt, uint32_t e_off, uint32_t n_rows, uint32_t slab_rows, uint32_t slabs,
                                 const uint32_t *__restrict__ col_slot, const uint32_t *__restrict__ row_slot,
                                 uint32_t lda_c, uint64_t dc_cells, uint32_t lda_r, KeyT *__restrict__ key,
                                 uint32_t *__restrict__ val) {
  for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < pt.n_edges; e += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t r = find_row(pt.offsets, pt.n_rows, (uint32_t)e) + pt.row_add;
    const uint32_t g = plan_gathered_row(pt, (uint32_t)e);
    uint32_t s = g / slab_rows;
    if (s >= slabs)
      s = slabs - 1;
    KeyT k = (KeyT)s * n_rows + r;
    if constexpr (sizeof(KeyT) == 8) {
      const uint64_t n_keys = (uint64_t)slabs * n_rows;
      const uint32_t cs = __ldg(col_slot + g), rs = __ldg(row_slot + r);
      if (cs != kNoHub)
        k = n_keys + (uint64_t)cs * lda_c + r;
      else if (rs != kNoHub)
        k = n_keys + dc_cells + (uint64_t)g * lda_r + rs;
    }
    key[e_off + e] = k;
    val[e_off + e] = e_off + (uint32_t)e;
  }
}

// pairs[i] = {gathered row, weight} of plan edge perm[i] (perm == nullptr: identity); parts: the device copy of the
// plan's parts, whose edges are numbered consecutively in the order given
__global__ void plan_pairs_kernel(const uint32_t *__restrict__ perm, const nts_plan_part *__restrict__ parts,
                                  uint32_t n_edges, uint2 *__restrict__ pairs) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_edges; i += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t e = perm ? __ldg(perm + i) : (uint32_t)i;
    const nts_plan_part *pt = parts;
    for (; e >= pt->n_edges; pt++)
      e -= (uint32_t)pt->n_edges;
    const float wt = pt->weight ? __ldg(pt->weight + e) : 1.f;
    pairs[i] = make_uint2(plan_gathered_row(*pt, e), __float_as_uint(wt));
  }
}

// voff[k] = number of sorted keys < k, k in [0, n_keys]
template <class KeyT>
__global__ void plan_offsets_kernel(const KeyT *__restrict__ sorted_key, uint32_t n_edges, uint32_t n_keys,
                                    uint32_t *__restrict__ voff) {
  for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k <= n_keys; k += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = n_edges; // first position with key >= k
    while (lo < hi) {
      uint32_t mid = lo + ((hi - lo) >> 1);
      if (__ldg(sorted_key + mid) < (KeyT)k)
        lo = mid + 1;
      else
        hi = mid;
    }
    voff[k] = lo;
  }
}

// ---- hub blocks (nts_gather_plan_create_hybrid) --------------------------------------------------------------------
// cnt[g] = number of edges that gather row g (integer atomics: the counts are exact and order-independent)
__global__ void plan_ref_count_kernel(const uint32_t *__restrict__ idx, const uint32_t *__restrict__ slot_of,
                                      uint32_t base, uint32_t n_edges, uint32_t *__restrict__ cnt) {
  for (uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_edges; e += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t id = __ldg(idx + e);
    atomicAdd(cnt + (slot_of ? __ldg(slot_of + id) : id - base), 1u);
  }
}

// One warp per run of equal dense keys (a cell): dense[key - n_keys] = sum of the run's weights, lane-strided partial
// sums then a fixed butterfly, so two builds give bit-identical cells.
__global__ void plan_cell_sum_kernel(const uint64_t *__restrict__ cell_key, const uint32_t *__restrict__ run_start,
                                     const uint32_t *__restrict__ run_len, uint32_t n_runs,
                                     const uint32_t *__restrict__ perm, const float *__restrict__ w, uint64_t n_keys,
                                     float *__restrict__ dense) {
  const uint32_t lane = threadIdx.x & 31;
  for (uint64_t run = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; run < n_runs;
       run += ((uint64_t)gridDim.x * blockDim.x) >> 5) {
    const uint32_t b = __ldg(run_start + run), n = __ldg(run_len + run);
    float s = 0.f;
    for (uint32_t j = lane; j < n; j += 32)
      s += w ? __ldg(w + __ldg(perm + b + j)) : 1.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
      s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0)
      dense[__ldg(cell_key + run) - n_keys] = s;
  }
}

// dst[r, 0:ld] = {src[r, 0:F], 0...} for src rows of stride lds   (ld = F rounded up to a multiple of 4; one warp per
// row piece)
__global__ void pad_rows_kernel(const float *__restrict__ src, uint32_t lds, float *__restrict__ dst, uint32_t n_rows,
                                uint32_t F, uint32_t ld) {
  const uint64_t total = (uint64_t)n_rows * ld;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t r = i / ld;
    const uint32_t c = (uint32_t)(i - r * ld);
    dst[i] = c < F ? __ldg(src + r * lds + c) : 0.f;
  }
}

// dst[r, 0:ld] = {bf16(src[r, 0:F]), 0...}   (ld % 8 == 0; one thread per 16-byte chunk of 8 output values)
// S = float: round to nearest even (cvt.rn.bf16x2.f32, what torch's .to(torch.bfloat16) executes on the GPU);
// S = __nv_bfloat16: the values are copied as they are (re-strided / realigned BF16 input).
template <class S>
__global__ void bf16_rows_kernel(const S *__restrict__ src, uint32_t lds, uint4 *__restrict__ dst, uint32_t n_rows,
                                 uint32_t F, uint32_t ld) {
  const uint32_t ld8 = ld / 8;
  const uint64_t total = (uint64_t)n_rows * ld8;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t r = i / ld8;
    const uint32_t c = (uint32_t)(i - r * ld8) * 8;
    const S *s = src + r * lds;
    uint32_t w[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const uint32_t c0 = c + 2 * j, c1 = c0 + 1;
      if constexpr (std::is_same<S, float>::value) {
        const __nv_bfloat162 h = __floats2bfloat162_rn(c0 < F ? __ldg(s + c0) : 0.f, c1 < F ? __ldg(s + c1) : 0.f);
        w[j] = *reinterpret_cast<const uint32_t *>(&h);
      } else {
        const uint16_t *u = reinterpret_cast<const uint16_t *>(s);
        w[j] = (c0 < F ? (uint32_t)__ldg(u + c0) : 0u) | ((c1 < F ? (uint32_t)__ldg(u + c1) : 0u) << 16);
      }
    }
    dst[i] = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

// ---- the aggregation kernel ----------------------------------------------------------------------------------------
constexpr int kPlanWarps = 8;

// Output columns 4c .. 4c+3 of one accumulator chunk, OUTV floats per store (the output keeps the caller's row
// stride F, so its rows are 16-byte aligned only when F % 4 == 0).
template <int OUTV, bool ATOMIC>
__device__ __forceinline__ void flush_chunk(float *__restrict__ orow, uint32_t col, uint32_t F, float4 a) {
  if constexpr (OUTV == 4) {
    float4 *p = reinterpret_cast<float4 *>(orow + col);
    if constexpr (ATOMIC) {
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a.x), "f"(a.y), "f"(a.z), "f"(a.w)
                   : "memory");
    } else {
      float4 o = *p;
      o.x += a.x, o.y += a.y, o.z += a.z, o.w += a.w;
      *p = o;
    }
  } else if constexpr (OUTV == 2) {
    float2 *p = reinterpret_cast<float2 *>(orow + col);
    if constexpr (ATOMIC) {
      asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a.x), "f"(a.y) : "memory");
      if (col + 2 < F)
        asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p + 1), "f"(a.z), "f"(a.w) : "memory");
    } else {
      float2 o = p[0];
      o.x += a.x, o.y += a.y;
      p[0] = o;
      if (col + 2 < F) {
        float2 o1 = p[1];
        o1.x += a.z, o1.y += a.w;
        p[1] = o1;
      }
    }
  } else {
    const float v[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int i = 0; i < 4; i++)
      if (col + i < F) {
        if constexpr (ATOMIC)
          atomicAdd(orow + col + i, v[i]);
        else
          orow[col + i] += v[i];
      }
  }
}

// Gathered element types.  A chunk is the 16 bytes one lane loads per column step: 4 floats, or 8 BF16 values that are
// widened to FP32 in registers (a BF16 value is the upper half of the FP32 with the same bits: exact, one ALU op).
template <class T> struct GatherT;
template <> struct GatherT<float> {
  using chunk = float4;
  static constexpr int V = 4;
  __device__ static __forceinline__ void widen(const float4 &c, float (&v)[4]) {
    v[0] = c.x, v[1] = c.y, v[2] = c.z, v[3] = c.w;
  }
};
template <> struct GatherT<__nv_bfloat16> {
  using chunk = uint4;
  static constexpr int V = 8;
  __device__ static __forceinline__ void widen(const uint4 &c, float (&v)[8]) {
    const uint32_t u[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
    for (int i = 0; i < 4; i++) {
      v[2 * i] = __uint_as_float(u[i] << 16);
      v[2 * i + 1] = __uint_as_float(u[i] & 0xffff0000u);
    }
  }
};

// T    : gathered element type (float | __nv_bfloat16); a chunk holds V = 4 | 8 values
// K    : chunks per lane per column tile (a tile covers K*32*V values)
// U    : edges whose K loads are issued before any FMA (U*K independent 16-byte loads per lane)
// OUTV : floats per output store (4 when F % 4 == 0 and the output is 16-byte aligned, else 2 or 1)
// MINB : __launch_bounds__ minimum CTAs per SM
// G    : virtual warps per warp.  Rows of at most 16 / 8 chunks (FP32: F <= 64 / 32) would leave half / three quarters
//        of the lanes idle, so a warp is split into G independent groups of 32/G lanes, each with its own edge quantum,
//        row bookkeeping and accumulators (the kernel has no warp-wide shuffles: all state is per lane already).
// Warp g owns the edge quantum [e_begin + q*Q, ...) of column tile t (g = q*tiles + t); the (row, weight) pairs of the
// CTA's edge span are staged in shared memory by one cp.async.bulk, completion on an mbarrier.  `vblock` is the CTA's
// index among the gather CTAs of the launch (blockIdx.x in planned_gather_sum_kernel).
template <class T, int K, int U, int OUTV, int G>
__device__ __forceinline__ void planned_gather_body(unsigned char *smem_raw, uint32_t vblock,
                                                    const typename GatherT<T>::chunk *__restrict__ in, uint32_t ldc,
                                                    float *__restrict__ out, uint32_t F,
                                                    const uint2 *__restrict__ pairs, const uint32_t *__restrict__ off,
                                                    uint32_t n_rows, uint32_t e_begin, uint32_t e_end, uint32_t Q,
                                                    uint32_t tiles, uint32_t tile_vecs) {
  static_assert(G == 1 || K == 1, "virtual warps are for rows narrower than a warp");
  using Chunk = typename GatherT<T>::chunk;
  constexpr int V = GatherT<T>::V;
  constexpr uint32_t GS = 32 / G;                       // lanes per virtual warp
  const uint32_t lane = threadIdx.x & (GS - 1);         // lane within the virtual warp
  const uint32_t vwarp_in_block = threadIdx.x / GS;
  const uint64_t gwarp = (uint64_t)vblock * (kPlanWarps * G) + vwarp_in_block;
  const uint32_t tile = (uint32_t)(gwarp % tiles);
  const uint64_t q = gwarp / tiles;
  const uint64_t e0_64 = e_begin + q * (uint64_t)Q;

  uint64_t *bar = reinterpret_cast<uint64_t *>(smem_raw);
  uint2 *s_pair = reinterpret_cast<uint2 *>(smem_raw + 16);
  uint32_t cta_e_base = 0, bulk_bytes = 0;
  {
    const uint64_t cta_w0 = (uint64_t)vblock * (kPlanWarps * G);
    const uint64_t first_q = cta_w0 / tiles;
    const uint64_t last_q = (cta_w0 + kPlanWarps * G - 1) / tiles;
    uint64_t ce0 = e_begin + first_q * (uint64_t)Q;
    uint64_t ce1 = e_begin + (last_q + 1) * (uint64_t)Q;
    if (ce1 > e_end)
      ce1 = e_end;
    if (ce0 < ce1) {
      cta_e_base = (uint32_t)(ce0 & ~1ull); // 16-byte aligned start (8-byte elements, array 16-byte aligned)
      const uint32_t n_el = (uint32_t)(ce1 - cta_e_base);
      bulk_bytes = (n_el * 8u) & ~15u;      // whole 16-byte units through the bulk engine, a last odd element by a plain load
      if (threadIdx.x == 0) {
        mbar_init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        if (n_el & 1u)
          s_pair[n_el - 1] = __ldg(pairs + cta_e_base + n_el - 1);
      }
      __syncthreads();
      if (threadIdx.x == 0 && bulk_bytes) {
        mbar_expect_tx(bar, bulk_bytes);
        bulk_g2s(s_pair, pairs + cta_e_base, bulk_bytes, bar);
      }
    }
  }
  if (e0_64 >= e_end)
    return;
  const uint32_t e0 = (uint32_t)e0_64;
  const uint32_t e1 = (e0_64 + Q < e_end) ? e0 + Q : e_end;

  const uint32_t c0 = tile * tile_vecs + lane; // first chunk column of this lane
  bool act[K];
#pragma unroll
  for (int k = 0; k < K; k++)
    act[k] = (k * GS + lane) < tile_vecs && (c0 + k * GS) < ldc;

  uint32_t row = find_row(off, n_rows, e0);
  uint32_t row_end = __ldg(off + row + 1);
  bool row_started_inside = __ldg(off + row) >= e0;

  float acc[K][V];
#pragma unroll
  for (int k = 0; k < K; k++)
#pragma unroll
    for (int j = 0; j < V; j++)
      acc[k][j] = 0.f;

  auto flush = [&](bool whole) {
    float *orow = out + (size_t)row * F;
#pragma unroll
    for (int k = 0; k < K; k++) {
#pragma unroll
      for (int h = 0; h < V; h += 4) { // the output keeps OUTV-float stores: a BF16 chunk flushes as two float4
        const uint32_t col = (c0 + k * GS) * V + h;
        const float4 a = make_float4(acc[k][h], acc[k][h + 1], acc[k][h + 2], acc[k][h + 3]);
        if (act[k] && col < F) {
          if (whole)
            flush_chunk<OUTV, false>(orow, col, F, a);
          else
            flush_chunk<OUTV, true>(orow, col, F, a);
        }
      }
#pragma unroll
      for (int j = 0; j < V; j++)
        acc[k][j] = 0.f;
    }
  };
  auto advance = [&](uint32_t ee) {
    flush(row_started_inside);
    do {
      row++;
      row_end = __ldg(off + row + 1);
    } while (ee >= row_end);
    row_started_inside = true;
  };

  if (bulk_bytes)
    mbar_wait(bar, 0);

  const uint2 *sp = s_pair - cta_e_base;
  uint32_t e = e0;
  auto fma_chunk = [&](int k, float w, const Chunk &c) {
    float x[V];
    GatherT<T>::widen(c, x);
#pragma unroll
    for (int j = 0; j < V; j++)
      acc[k][j] = fmaf(w, x[j], acc[k][j]);
  };
  for (; e + U <= e1; e += U) {
    Chunk v[U][K];
    float wu[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const uint2 pr = sp[e + u];
      wu[u] = __uint_as_float(pr.y);
      const Chunk *p = in + (size_t)pr.x * ldc + c0;
#pragma unroll
      for (int k = 0; k < K; k++)
        if (act[k])
          v[u][k] = __ldg(p + k * GS);
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (e + u >= row_end)
        advance(e + u);
#pragma unroll
      for (int k = 0; k < K; k++)
        if (act[k])
          fma_chunk(k, wu[u], v[u][k]);
    }
  }
  for (; e < e1; e++) {
    const uint2 pr = sp[e];
    const float wj = __uint_as_float(pr.y);
    const Chunk *p = in + (size_t)pr.x * ldc + c0;
    Chunk v1[K];
#pragma unroll
    for (int k = 0; k < K; k++)
      if (act[k])
        v1[k] = __ldg(p + k * GS);
    if (e >= row_end)
      advance(e);
#pragma unroll
    for (int k = 0; k < K; k++)
      if (act[k])
        fma_chunk(k, wj, v1[k]);
  }
  flush(row_started_inside && row_end <= e1);
}

template <class T, int K, int U, int OUTV, int MINB, int G = 1>
__global__ void __launch_bounds__(kPlanWarps * 32, MINB)
    planned_gather_sum_kernel(const typename GatherT<T>::chunk *__restrict__ in, uint32_t ldc, float *__restrict__ out,
                              uint32_t F, const uint2 *__restrict__ pairs, const uint32_t *__restrict__ off,
                              uint32_t n_rows, uint32_t e_begin, uint32_t e_end, uint32_t Q, uint32_t tiles,
                              uint32_t tile_vecs) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  planned_gather_body<T, K, U, OUTV, G>(smem_raw, blockIdx.x, in, ldc, out, F, pairs, off, n_rows, e_begin, e_end, Q,
                                        tiles, tile_vecs);
}

struct PlanShape;
// ---- experiment the north star asks for: feature ROWS staged in shared memory by TMA ----------------------------------
// Same work split and row bookkeeping, but the gathered row never passes through registers on its way in: lane 0 of
// each warp issues one cp.async.bulk (SASS UBLKCP) per edge that copies the row's tile (16-byte aligned thanks to the
// padded workspace) into a per-warp ring of STAGES shared-memory buffers, completion on one mbarrier per stage; the
// warp waits, reads its chunks with 16-byte LDS, accumulates, and re-arms the stage for edge e + STAGES.
// Kept as variant 1 of nts_gather_plan_set_variant for measurement (tools/k1_sweep.py --tma; 3-10x slower than
// variant 0 on an H100): bulk copies bypass L1, which serves
// the hub rows of a skewed graph, and every gathered byte still crosses the shared-memory data stage once.
template <int K, int STAGES, int OUTV, int MINB>
__global__ void __launch_bounds__(kPlanWarps * 32, MINB)
    planned_gather_sum_tma_kernel(const float4 *__restrict__ in, uint32_t ld4, float *__restrict__ out, uint32_t F,
                                  const uint2 *__restrict__ pairs, const uint32_t *__restrict__ off, uint32_t n_rows,
                                  uint32_t e_begin, uint32_t e_end, uint32_t Q, uint32_t tiles, uint32_t tile_vecs,
                                  uint32_t pair_bytes) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp_in_block = threadIdx.x >> 5;
  const uint64_t gwarp = (uint64_t)blockIdx.x * kPlanWarps + warp_in_block;
  const uint32_t tile = (uint32_t)(gwarp % tiles);
  const uint64_t q = gwarp / tiles;
  const uint64_t e0_64 = e_begin + q * (uint64_t)Q;

  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint64_t *bar = reinterpret_cast<uint64_t *>(smem_raw);
  uint2 *s_pair = reinterpret_cast<uint2 *>(smem_raw + 16);
  // per-warp ring: STAGES barriers, then STAGES row buffers of tile_vecs float4
  const uint32_t ring_bytes = 8u * STAGES + 8u * (STAGES & 1) + STAGES * tile_vecs * 16u;
  unsigned char *ring = smem_raw + 16 + pair_bytes + (size_t)warp_in_block * ring_bytes;
  uint64_t *sbar = reinterpret_cast<uint64_t *>(ring);
  float4 *sbuf = reinterpret_cast<float4 *>(ring + 8u * STAGES + 8u * (STAGES & 1));
  uint32_t cta_e_base = 0, bulk_bytes = 0;
  {
    const uint64_t cta_w0 = (uint64_t)blockIdx.x * kPlanWarps;
    const uint64_t first_q = cta_w0 / tiles;
    const uint64_t last_q = (cta_w0 + kPlanWarps - 1) / tiles;
    uint64_t ce0 = e_begin + first_q * (uint64_t)Q;
    uint64_t ce1 = e_begin + (last_q + 1) * (uint64_t)Q;
    if (ce1 > e_end)
      ce1 = e_end;
    if (lane == 0)
      for (int s = 0; s < STAGES; s++)
        mbar_init(sbar + s, 1);
    if (ce0 < ce1) {
      cta_e_base = (uint32_t)(ce0 & ~1ull);
      const uint32_t n_el = (uint32_t)(ce1 - cta_e_base);
      bulk_bytes = (n_el * 8u) & ~15u;
      if (threadIdx.x == 0) {
        mbar_init(bar, 1);
        if (n_el & 1u)
          s_pair[n_el - 1] = __ldg(pairs + cta_e_base + n_el - 1);
      }
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    if (threadIdx.x == 0 && bulk_bytes) {
      mbar_expect_tx(bar, bulk_bytes);
      bulk_g2s(s_pair, pairs + cta_e_base, bulk_bytes, bar);
    }
  }
  if (e0_64 >= e_end)
    return;
  const uint32_t e0 = (uint32_t)e0_64;
  const uint32_t e1 = (e0_64 + Q < e_end) ? e0 + Q : e_end;
  const uint32_t c0 = tile * tile_vecs + lane;
  const uint32_t my_vecs = min(tile_vecs, ld4 - tile * tile_vecs); // float4 of this tile that exist in the row
  const uint32_t row_bytes = my_vecs * 16u;
  bool act[K];
#pragma unroll
  for (int k = 0; k < K; k++)
    act[k] = (k * 32 + lane) < my_vecs;

  uint32_t row = find_row(off, n_rows, e0);
  uint32_t row_end = __ldg(off + row + 1);
  bool row_started_inside = __ldg(off + row) >= e0;
  float4 acc[K];
#pragma unroll
  for (int k = 0; k < K; k++)
    zero_vec(acc[k]);
  auto flush = [&](bool whole) {
    float *orow = out + (size_t)row * F;
#pragma unroll
    for (int k = 0; k < K; k++) {
      const uint32_t col = (c0 + k * 32) * 4;
      if (act[k] && col < F) {
        if (whole)
          flush_chunk<OUTV, false>(orow, col, F, acc[k]);
        else
          flush_chunk<OUTV, true>(orow, col, F, acc[k]);
      }
      zero_vec(acc[k]);
    }
  };
  auto advance = [&](uint32_t ee) {
    flush(row_started_inside);
    do {
      row++;
      row_end = __ldg(off + row + 1);
    } while (ee >= row_end);
    row_started_inside = true;
  };
  if (bulk_bytes)
    mbar_wait(bar, 0);
  const uint2 *sp = s_pair - cta_e_base;
  auto issue = [&](uint32_t e, uint32_t stage) { // lane 0 only
    const uint32_t src_row = sp[e].x;
    mbar_expect_tx(sbar + stage, row_bytes);
    bulk_g2s(sbuf + (size_t)stage * tile_vecs, in + (size_t)src_row * ld4 + tile * tile_vecs, row_bytes, sbar + stage);
  };
  if (lane == 0)
    for (uint32_t s = 0; s < STAGES && e0 + s < e1; s++)
      issue(e0 + s, s);
  uint32_t stage = 0, parity = 0;
  for (uint32_t e = e0; e < e1; e++) {
    const float w = __uint_as_float(sp[e].y);
    mbar_wait(sbar + stage, parity);
    const float4 *b = sbuf + (size_t)stage * tile_vecs + lane;
    float4 v[K];
#pragma unroll
    for (int k = 0; k < K; k++)
      if (act[k])
        v[k] = b[k * 32];
    if (e >= row_end)
      advance(e);
#pragma unroll
    for (int k = 0; k < K; k++)
      if (act[k])
        fma_vec(acc[k], w, v[k]);
    __syncwarp(); // every lane has consumed the stage (its values are in registers and used): it may be overwritten
    if (lane == 0 && e + STAGES < e1)
      issue(e + STAGES, stage);
    if (++stage == STAGES) {
      stage = 0;
      parity ^= 1u;
    }
  }
  flush(row_started_inside && row_end <= e1);
}

template <int K, int STAGES, int OUTV, int MINB>
static int launch_planned_tma(nts_gather_plan *pl, const PlanShape &sh, const float4 *in, uint32_t ld4, float *out,
                              uint32_t F, uint32_t Q, cudaStream_t st);

struct PlanShape {
  int k, u, outv, minb, g;
  uint32_t tiles, tile_vecs;
};

template <class T, int K, int U, int OUTV, int MINB, int G = 1>
static int launch_planned(nts_gather_plan *pl, const PlanShape &sh, const T *in_rows, uint32_t ldc, float *out,
                          uint32_t F, uint32_t Q, cudaStream_t st) {
  auto kern = planned_gather_sum_kernel<T, K, U, OUTV, MINB, G>;
  const auto *in = reinterpret_cast<const typename GatherT<T>::chunk *>(in_rows);
  const size_t smem = 16 + ((size_t)kPlanWarps * G * Q + 4) * 8;
  NTS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  pl->last_launches = 0;
  for (int s = 0; s < pl->slabs; s++) {
    const uint64_t eb = pl->slab_edge[s], ee = pl->slab_edge[s + 1];
    if (ee <= eb)
      continue;
    const uint64_t quanta = (ee - eb + Q - 1) / Q;
    const uint64_t blocks = (quanta * sh.tiles + kPlanWarps * G - 1) / (kPlanWarps * G);
    NTS_ARG_CHECK(blocks <= 0x7fffffffull, "aggregation grid too large");
    kern<<<(unsigned)blocks, kPlanWarps * 32, smem, st>>>(in, ldc, out, F, pl->pairs, pl->voff + (size_t)s * pl->n_rows,
                                                          pl->n_rows, (uint32_t)eb, (uint32_t)ee, Q, sh.tiles,
                                                          sh.tile_vecs);
    NTS_LAUNCH_CHECK();
    pl->last_grid = (int)blocks;
    pl->last_launches++;
  }
  return 0;
}

template <int K, int STAGES, int OUTV, int MINB>
static int launch_planned_tma(nts_gather_plan *pl, const PlanShape &sh, const float4 *in, uint32_t ld4, float *out,
                              uint32_t F, uint32_t Q, cudaStream_t st) {
  auto kern = planned_gather_sum_tma_kernel<K, STAGES, OUTV, MINB>;
  const uint32_t pair_bytes = (kPlanWarps * Q + 4) * 8;
  const uint32_t ring_bytes = 8u * STAGES + 8u * (STAGES & 1) + STAGES * sh.tile_vecs * 16u;
  const size_t smem = 16 + pair_bytes + (size_t)kPlanWarps * ring_bytes;
  NTS_ARG_CHECK(smem <= 227 * 1024, "row-staging ring does not fit shared memory");
  NTS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  pl->last_launches = 0;
  for (int s = 0; s < pl->slabs; s++) {
    const uint64_t eb = pl->slab_edge[s], ee = pl->slab_edge[s + 1];
    if (ee <= eb)
      continue;
    const uint64_t quanta = (ee - eb + Q - 1) / Q;
    const uint64_t blocks = (quanta * sh.tiles + kPlanWarps - 1) / kPlanWarps;
    NTS_ARG_CHECK(blocks <= 0x7fffffffull, "aggregation grid too large");
    kern<<<(unsigned)blocks, kPlanWarps * 32, smem, st>>>(in, ld4, out, F, pl->pairs, pl->voff + (size_t)s * pl->n_rows,
                                                          pl->n_rows, (uint32_t)eb, (uint32_t)ee, Q, sh.tiles,
                                                          sh.tile_vecs, pair_bytes);
    NTS_LAUNCH_CHECK();
    pl->last_grid = (int)blocks;
    pl->last_launches++;
  }
  return 0;
}

#define NTS_PLAN_TMA_CASE(K_, S_, B_)                                                                               \
  if (sh.k == K_ && stages == S_ && sh.minb == B_) {                                                                \
    if (sh.outv == 4)                                                                                               \
      return launch_planned_tma<K_, S_, 4, B_>(pl, sh, in4, ld4, out, F, Q, st);                                    \
    if (sh.outv == 2)                                                                                               \
      return launch_planned_tma<K_, S_, 2, B_>(pl, sh, in4, ld4, out, F, Q, st);                                    \
    return launch_planned_tma<K_, S_, 1, B_>(pl, sh, in4, ld4, out, F, Q, st);                                      \
  }

#define NTS_PLAN_CASE_G(U_, B_, G_)                                                                                 \
  if (sh.k == 1 && sh.u == U_ && sh.minb == B_ && sh.g == G_) {                                                     \
    if (sh.outv == 4)                                                                                               \
      return launch_planned<T, 1, U_, 4, B_, G_>(pl, sh, in, ldc, out, F, Q, st);                                   \
    if (sh.outv == 2)                                                                                               \
      return launch_planned<T, 1, U_, 2, B_, G_>(pl, sh, in, ldc, out, F, Q, st);                                   \
    return launch_planned<T, 1, U_, 1, B_, G_>(pl, sh, in, ldc, out, F, Q, st);                                     \
  }

#define NTS_PLAN_CASE(K_, U_, B_)                                                                                   \
  if (sh.k == K_ && sh.u == U_ && sh.minb == B_) {                                                                  \
    if (sh.outv == 4)                                                                                               \
      return launch_planned<T, K_, U_, 4, B_>(pl, sh, in, ldc, out, F, Q, st);                                       \
    if (sh.outv == 2)                                                                                               \
      return launch_planned<T, K_, U_, 2, B_>(pl, sh, in, ldc, out, F, Q, st);                                       \
    return launch_planned<T, K_, U_, 1, B_>(pl, sh, in, ldc, out, F, Q, st);                                         \
  }

// ---- dense hub blocks: FP32 SIMT GEMM (FFMA only, no tensor cores) ----------------------------------------------------
//   out[rowmap(m), n] += sum_{k in this CTA's K range} At[k, m] * B[colmap(k), n]      m < M, n < F
// At is the block stored K-major ([K x lda], lda % 4 == 0, columns M..lda zero), B rows are ldb floats, 16-byte
// aligned (the input or the padded workspace; values past F only reach accumulators of columns >= F, which the
// epilogue never writes), so both operand tiles are rows of 16-byte chunks that
// cp.async copies straight into double-buffered shared memory (zero-filled past the edges).  128 x 128 x 16 tiles,
// 256 threads, 8 x 8 outputs per thread.  Column block: colmap = hub columns, rowmap = identity, one CTA per output
// tile -> plain read-modify-write, or with STORE a plain store of the tile (overwrite runs: M = every output row, so
// the column block writes each output element exactly once and initialises the output for the launches after it).
// Row block: colmap = identity, rowmap = hub rows, split-K -> vector red.
// blockIdx.x = (split * m_tiles + m_tile) * n_tiles + n_tile: the N tiles of one A tile run back to back (A from L2).
constexpr int kHubBM = 128, kHubBN = 128, kHubBK = 16, kHubThreads = 256;

__device__ __forceinline__ void p_cp_async16(void *smem_dst, const void *gmem_src, bool full) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src),
               "r"(full ? 16 : 0)
               : "memory");
}

// TB = __nv_bfloat16: B rows are BF16 (ldb % 8 == 0), cp.async fills half-size B tiles and the values are widened to
// FP32 at the shared-memory read; A, the accumulators and the FFMA math are those of the FP32 instantiation.
// TN = outputs per thread along N: 8 (128 x 128 tile, 8 x 8 per thread, the stand-alone kernel's) or 4 (128 x 64 tile,
// 8 x 4 per thread: half the accumulators, for the fused slab launches whose gather runs 3 or 4 CTAs per SM).
// KKU = unroll of the 16-step loop over one K tile.
// Tile `tile` = (split * m_tiles + m_tile) * n_tiles + n_tile covers K rows [k_lo + split * k_split, ...) cut at k_hi.
template <int TN, class TB> struct HubSmem {
  static constexpr uint32_t kBN = 16 * TN;
  float As[2][kHubBK][kHubBM];
  TB Bs[2][kHubBK][kBN];
};

template <class TB, int OUTV, bool SPLIT, bool STORE, int TN, int KKU>
__device__ __forceinline__ void hub_gemm_tile(HubSmem<TN, TB> &sm, uint32_t tile, const float *__restrict__ At,
                                              uint32_t lda, uint32_t M, uint32_t k_lo, uint32_t k_hi, uint32_t k_split,
                                              const TB *__restrict__ B, uint32_t ldb,
                                              const uint32_t *__restrict__ colmap, float *__restrict__ out, uint32_t F,
                                              const uint32_t *__restrict__ rowmap, uint32_t m_tiles, uint32_t n_tiles) {
  static_assert(!(SPLIT && STORE), "split-K partials must be added, not stored");
  constexpr bool kBf16 = std::is_same<TB, __nv_bfloat16>::value;
  constexpr uint32_t kBV = 16 / sizeof(TB); // B values per 16-byte chunk
  constexpr uint32_t kBN = HubSmem<TN, TB>::kBN;
  constexpr uint32_t kBChunks = kHubBK * kBN / kBV; // 512 / 256 (FP32 / BF16, TN = 8), 256 / 128 (TN = 4)
  auto &As = sm.As;
  auto &Bs = sm.Bs;
  const uint32_t t = threadIdx.x;
  const uint32_t n_tile = tile % n_tiles, rest = tile / n_tiles;
  const uint32_t m0 = (rest % m_tiles) * kHubBM, n0 = n_tile * kBN;
  const uint32_t k_begin = k_lo + (rest / m_tiles) * k_split;
  const uint32_t k_end = min(k_hi, k_begin + k_split);
  if (k_begin >= k_end)
    return;
  const uint32_t n_kt = (k_end - k_begin + kHubBK - 1) / kHubBK;

  auto load = [&](uint32_t kt, int buf) {
#pragma unroll
    for (int i = 0; i < 2; i++) { // 512 16-byte chunks per A tile, 2 per thread
      const uint32_t c = t + i * kHubThreads, kk = c >> 5, c4 = (c & 31) * 4;
      const uint32_t k = k_begin + kt * kHubBK + kk;
      const bool a_ok = k < k_end && m0 + c4 < lda;
      p_cp_async16(&As[buf][kk][c4], a_ok ? At + (size_t)k * lda + m0 + c4 : At, a_ok);
    }
#pragma unroll
    for (int i = 0; i < (int)((kBChunks + kHubThreads - 1) / kHubThreads); i++) {
      constexpr uint32_t kRowChunks = kBN / kBV;
      const uint32_t c = t + i * kHubThreads, kk = c / kRowChunks, cv = (c % kRowChunks) * kBV;
      if (kBChunks % kHubThreads != 0 && c >= kBChunks)
        break;
      const uint32_t k = k_begin + kt * kHubBK + kk;
      const bool b_ok = k < k_end && n0 + cv < ldb;
      const uint32_t brow = b_ok ? (colmap ? __ldg(colmap + k) : k) : 0;
      p_cp_async16(&Bs[buf][kk][cv], B + (size_t)brow * ldb + (b_ok ? n0 + cv : 0), b_ok);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  auto read_b4 = [&](int buf, int kk, uint32_t n) -> float4 { // B values n .. n+3 of row kk as FP32
    if constexpr (kBf16) {
      const uint2 u = *reinterpret_cast<const uint2 *>(&Bs[buf][kk][n]);
      return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                         __uint_as_float(u.y & 0xffff0000u));
    } else {
      return *reinterpret_cast<const float4 *>(&Bs[buf][kk][n]);
    }
  };

  const uint32_t tx = t & 15, ty = t >> 4;
  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; i++)
#pragma unroll
    for (int j = 0; j < TN; j++)
      acc[i][j] = 0.f;

  load(0, 0);
  for (uint32_t kt = 0; kt < n_kt; kt++) {
    const int buf = kt & 1;
    if (kt + 1 < n_kt) {
      load(kt + 1, buf ^ 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
#pragma unroll(KKU)
    for (int kk = 0; kk < kHubBK; kk++) {
      const float4 a0 = *reinterpret_cast<const float4 *>(&As[buf][kk][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4 *>(&As[buf][kk][64 + ty * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float b[TN];
#pragma unroll
      for (int h = 0; h < TN / 4; h++) {
        const float4 bh = read_b4(buf, kk, h * 64 + tx * 4);
        b[4 * h] = bh.x, b[4 * h + 1] = bh.y, b[4 * h + 2] = bh.z, b[4 * h + 3] = bh.w;
      }
#pragma unroll
      for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = 0; j < TN; j++)
          acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < 8; i++) {
    const uint32_t m = m0 + (i >> 2) * 64 + ty * 4 + (i & 3);
    if (m >= M)
      continue;
    float *orow = out + (size_t)(rowmap ? __ldg(rowmap + m) : m) * F;
#pragma unroll
    for (int j = 0; j < TN / 4; j++) {
      const uint32_t col = n0 + j * 64 + tx * 4;
      const float4 a = make_float4(acc[i][j * 4], acc[i][j * 4 + 1], acc[i][j * 4 + 2], acc[i][j * 4 + 3]);
      if (col < F) {
        if constexpr (STORE)
          store_chunk_checked<OUTV>(orow, col, F, a);
        else
          flush_chunk<OUTV, SPLIT>(orow, col, F, a);
      }
    }
  }
}

// STORE: every tile has a non-empty K range (the column block's K = hub_cols >= 1), so no output tile is skipped.
template <class TB, int OUTV, bool SPLIT, bool STORE>
__global__ void __launch_bounds__(kHubThreads, 2)
    hub_block_gemm_kernel(const float *__restrict__ At, uint32_t lda, uint32_t M, uint32_t K, uint32_t k_split,
                          const TB *__restrict__ B, uint32_t ldb, const uint32_t *__restrict__ colmap,
                          float *__restrict__ out, uint32_t F, const uint32_t *__restrict__ rowmap, uint32_t m_tiles,
                          uint32_t n_tiles) {
  __shared__ __align__(16) HubSmem<8, TB> sm;
  hub_gemm_tile<TB, OUTV, SPLIT, STORE, 8, kHubBK>(sm, blockIdx.x, At, lda, M, 0, K, k_split, B, ldb, colmap, out, F,
                                                   rowmap, m_tiles, n_tiles);
}

// Split-K length of the row block (M = hub_rows, K = gather_rows): about 4 waves of 2 CTAs per SM over the whole K,
// at least 16 K tiles per CTA.
static uint32_t hub_row_k_split(uint32_t K, uint32_t m_tiles, uint32_t n_tiles) {
  const uint64_t want = (uint64_t)sm_count() * 2 * 4;
  const uint64_t splits = (want + (uint64_t)m_tiles * n_tiles - 1) / ((uint64_t)m_tiles * n_tiles);
  const uint32_t k_split = (uint32_t)((K + splits - 1) / splits);
  return std::max<uint32_t>((k_split + kHubBK - 1) / kHubBK * kHubBK, 16 * kHubBK);
}

// rows = false: the column block only (the row block runs inside the fused slab launches).  overwrite: the column
// block stores its tiles instead of adding them (it covers every output element, and it launches first).
template <class TB, int OUTV>
static int launch_hub_blocks(nts_gather_plan *pl, const TB *in, uint32_t ldb, float *out, uint32_t F, bool rows,
                             bool overwrite, cudaStream_t st) {
  const uint32_t n_tiles = (F + kHubBN - 1) / kHubBN;
  if (pl->hub_cols) { // column block: M = n_rows, K = hub_cols
    const uint32_t m_tiles = (pl->n_rows + kHubBM - 1) / kHubBM;
    const uint64_t blocks = (uint64_t)m_tiles * n_tiles;
    NTS_ARG_CHECK(blocks <= 0x7fffffffull, "hub column block grid too large");
    auto kern = overwrite ? hub_block_gemm_kernel<TB, OUTV, false, true> : hub_block_gemm_kernel<TB, OUTV, false, false>;
    kern<<<(unsigned)blocks, kHubThreads, 0, st>>>(pl->dense, pl->lda_c, pl->n_rows, (uint32_t)pl->hub_cols,
                                                   (uint32_t)pl->hub_cols, in, ldb, pl->hub_col_ids, out, F, nullptr,
                                                   m_tiles, n_tiles);
    NTS_LAUNCH_CHECK();
  }
  if (pl->hub_rows && rows) { // row block: M = hub_rows, K = gather_rows
    const uint32_t m_tiles = (pl->hub_rows + kHubBM - 1) / kHubBM;
    const uint32_t K = pl->gather_rows;
    const uint32_t k_split = hub_row_k_split(K, m_tiles, n_tiles);
    const uint64_t splits = (K + k_split - 1) / k_split;
    hub_block_gemm_kernel<TB, OUTV, true, false><<<(unsigned)(splits * m_tiles * n_tiles), kHubThreads, 0, st>>>(
        pl->dense + (size_t)pl->hub_cols * pl->lda_c, pl->lda_r, (uint32_t)pl->hub_rows, K, k_split, in, ldb, nullptr,
        out, F, pl->hub_row_ids, m_tiles, n_tiles);
    NTS_LAUNCH_CHECK();
  }
  return 0;
}

// ---- fused slab launches (nts_gather_plan.overlap): the row block's tiles run inside the slab launches --------------
// The row block is FFMA-bound, the residual gather bound by gathered rows moving from L2 to the SMs; run one after the
// other, each leaves idle what the other needs.  They can share a launch because they write disjoint output rows: the
// row block takes every non-column-block edge of its hub rows (plan_keys_kernel), so those rows have empty residual
// segments and no gather warp writes them, while the row block writes hub rows only.  Its split-K is cut at the slab
// boundaries, so the tiles in slab s's launch read B rows [s * slab_rows, (s+1) * slab_rows) of the gathered matrix:
// the rows slab s's gather is making L2-resident.  (The column block writes every output row with a plain
// read-modify-write, so it stays a launch of its own, before the first slab.)
struct HubRowArgs {
  const float *At;                  // D_r^T [gather_rows x lda]
  uint32_t lda, M;                  // M = hub rows
  uint32_t k_lo, k_hi, k_split;     // this slab's gathered rows [k_lo, k_hi), split-K length
  const uint32_t *rowmap;           // hub row ids
  uint32_t m_tiles, n_tiles, n_gemm; // n_gemm = row-block tiles of this launch (splits * m_tiles * n_tiles)
  uint32_t period;                  // grid / n_gemm (>= 1)
};

// Every period-th block (period = floor(grid / n_gemm)) of the first n_gemm * period is a row-block tile, the rest are
// gather CTAs: the tiles are spread through the grid (CTAs start in about blockIdx order) instead of forming a head
// or a tail.  The GEMM body has half the accumulators (TN = 4) at 3 or 4 CTAs per SM, where the 8 x 8 body would not
// fit the gather's register budget; its K-tile loop is unrolled 4-fold, not 16-fold, for the same reason.
template <class T, int K, int U, int OUTV, int MINB, int G>
__global__ void __launch_bounds__(kPlanWarps * 32, MINB)
    planned_slab_hub_kernel(const typename GatherT<T>::chunk *__restrict__ in, uint32_t ldc, float *__restrict__ out,
                            uint32_t F, const uint2 *__restrict__ pairs, const uint32_t *__restrict__ off,
                            uint32_t n_rows, uint32_t e_begin, uint32_t e_end, uint32_t Q, uint32_t tiles,
                            uint32_t tile_vecs, const HubRowArgs hub) {
  static_assert(kPlanWarps * 32 == kHubThreads, "both bodies run 256 threads");
  constexpr int TN = MINB <= 2 ? 8 : 4;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const uint32_t b = blockIdx.x, grp = b / hub.period;
  if (grp < hub.n_gemm && b - grp * hub.period == hub.period - 1)
    hub_gemm_tile<T, OUTV, true, false, TN, TN == 8 ? kHubBK : 4>(
        *reinterpret_cast<HubSmem<TN, T> *>(smem_raw), grp, hub.At, hub.lda, hub.M, hub.k_lo, hub.k_hi, hub.k_split,
        reinterpret_cast<const T *>(in), ldc * GatherT<T>::V, nullptr, out, F, hub.rowmap, hub.m_tiles, hub.n_tiles);
  else
    planned_gather_body<T, K, U, OUTV, G>(smem_raw, b - min(grp, hub.n_gemm), in, ldc, out, F, pairs, off, n_rows,
                                          e_begin, e_end, Q, tiles, tile_vecs);
}

template <class T, int K, int U, int OUTV, int MINB, int G = 1>
static int launch_fused(nts_gather_plan *pl, const PlanShape &sh, const T *in_rows, uint32_t ldc, float *out,
                        uint32_t F, uint32_t Q, cudaStream_t st) {
  constexpr int TN = MINB <= 2 ? 8 : 4;
  auto kern = planned_slab_hub_kernel<T, K, U, OUTV, MINB, G>;
  const auto *in = reinterpret_cast<const typename GatherT<T>::chunk *>(in_rows);
  const size_t smem = std::max(16 + ((size_t)kPlanWarps * G * Q + 4) * 8, sizeof(HubSmem<TN, T>));
  NTS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  HubRowArgs hub;
  hub.At = pl->dense + (size_t)pl->hub_cols * pl->lda_c;
  hub.lda = pl->lda_r;
  hub.M = (uint32_t)pl->hub_rows;
  hub.rowmap = pl->hub_row_ids;
  hub.m_tiles = (hub.M + kHubBM - 1) / kHubBM;
  hub.n_tiles = (F + 16 * TN - 1) / (16 * TN);
  hub.k_split = hub_row_k_split(pl->gather_rows, hub.m_tiles, hub.n_tiles);
  pl->last_launches = 0;
  for (int s = 0; s < pl->slabs; s++) {
    // slab s gathers rows [s * slab_rows, (s+1) * slab_rows); the last one runs to gather_rows
    // (plan_hybrid_keys_kernel clamps the slab index to slabs - 1)
    hub.k_lo = (uint32_t)std::min<uint64_t>((uint64_t)s * pl->slab_rows, pl->gather_rows);
    hub.k_hi = s + 1 == pl->slabs ? pl->gather_rows
                                  : (uint32_t)std::min<uint64_t>((uint64_t)(s + 1) * pl->slab_rows, pl->gather_rows);
    const uint64_t splits = hub.k_hi > hub.k_lo ? (hub.k_hi - hub.k_lo + hub.k_split - 1) / hub.k_split : 0;
    const uint64_t n_gemm = splits * hub.m_tiles * hub.n_tiles;
    const uint64_t eb = pl->slab_edge[s], ee = pl->slab_edge[s + 1];
    const uint64_t quanta = ee > eb ? (ee - eb + Q - 1) / Q : 0;
    const uint64_t blocks = n_gemm + (quanta * sh.tiles + kPlanWarps * G - 1) / (kPlanWarps * G);
    if (!blocks)
      continue;
    NTS_ARG_CHECK(blocks <= 0x7fffffffull, "aggregation grid too large");
    hub.n_gemm = (uint32_t)n_gemm;
    hub.period = n_gemm ? (uint32_t)(blocks / n_gemm) : 1;
    kern<<<(unsigned)blocks, kPlanWarps * 32, smem, st>>>(in, ldc, out, F, pl->pairs, pl->voff + (size_t)s * pl->n_rows,
                                                          pl->n_rows, (uint32_t)eb, (uint32_t)ee, Q, sh.tiles,
                                                          sh.tile_vecs, hub);
    NTS_LAUNCH_CHECK();
    pl->last_grid = (int)blocks;
    pl->last_launches++;
  }
  return 0;
}

// The fused schedule exists at the (chunks, U, occupancy, virtual warps) points run_gather picks by default.
#define NTS_PLAN_FUSED_CASE(K_, U_, B_, G_)                                                                         \
  if (sh.k == K_ && sh.u == U_ && sh.minb == B_ && sh.g == G_) {                                                    \
    if (sh.outv == 4)                                                                                               \
      return launch_fused<T, K_, U_, 4, B_, G_>(pl, sh, in, ldc, out, F, Q, st);                                    \
    if (sh.outv == 2)                                                                                               \
      return launch_fused<T, K_, U_, 2, B_, G_>(pl, sh, in, ldc, out, F, Q, st);                                    \
    return launch_fused<T, K_, U_, 1, B_, G_>(pl, sh, in, ldc, out, F, Q, st);                                      \
  }

// The gather of rows already in the kernel's layout: `in` holds gather_rows rows of ld values of T, 16-byte aligned,
// ld % V == 0 (columns F..ld are read but never reach an output).  Dense hub blocks first, then the residual edges'
// slab launches (stream order); with pl->overlap the row block runs inside the slab launches instead
// (planned_slab_hub_kernel).  overwrite: output = A in instead of output += A in; the column block stores the first
// value of every output element, or, in a plan without hub columns, the output is zeroed first.
template <class T>
static int run_gather(nts_gather_plan *pl, const T *in, uint32_t ld, float *output, uint32_t F, bool overwrite,
                      cudaStream_t st) {
  constexpr bool kBf16 = std::is_same<T, __nv_bfloat16>::value;
  PlanShape sh;
  const uint32_t ldc = ld / GatherT<T>::V; // 16-byte chunks per row
  const uint32_t chunks = (ldc + 31) / 32;
  const uint32_t kmax = 5;
  sh.tiles = (chunks + kmax - 1) / kmax;
  sh.tile_vecs = (ldc + sh.tiles - 1) / sh.tiles;
  sh.k = (int)((sh.tile_vecs + 31) / 32);
  sh.tiles = (ldc + sh.tile_vecs - 1) / sh.tile_vecs;
  sh.outv = pick_vec(F, output);
  const bool fused = pl->overlap && pl->hub_rows;
  NTS_ARG_CHECK(!fused || g_plan_variant == 0, "the fused slab launches use the register-staging gather (variant 0)");
  if (overwrite && !pl->hub_cols)
    NTS_CUDA_OK(cudaMemsetAsync(output, 0, (size_t)pl->n_rows * F * sizeof(float), st));
  if (pl->hub_cols || pl->hub_rows) {
    const int rc = sh.outv == 4   ? launch_hub_blocks<T, 4>(pl, in, ld, output, F, !fused, overwrite, st)
                   : sh.outv == 2 ? launch_hub_blocks<T, 2>(pl, in, ld, output, F, !fused, overwrite, st)
                                  : launch_hub_blocks<T, 1>(pl, in, ld, output, F, !fused, overwrite, st);
    if (rc)
      return rc;
  }
  sh.g = ldc <= 8 ? 4 : (ldc <= 16 ? 2 : 1); // rows narrower than half / a quarter of a warp: virtual warps
  if (g_plan_variant == 1 || getenv("NTS_PLAN_NO_SUBWARP"))
    sh.g = 1;
  // (U, min CTAs/SM): U*K 16-byte loads in flight per lane
  // defaults = the largest U that compiles without spills at the occupancy point (ptxas -v); measured points for
  // the headline shapes measured on an H100 with tools/k1_sweep.py (unbucketed, Zipf graph of config B):
  // k = 5, F = 602: U=4 at 2 CTAs/SM 24.9 ms vs U=1 at 3 CTAs 25.1 / U=4 at 1 CTA 27.1 / U=2 at 3 CTAs 32.7;
  // k = 1, F = 128: U=4 at 4 CTAs 3.98 ms vs U=8 at 3 CTAs 4.37 / U=16 at 2 CTAs 5.5
  sh.minb = sh.k >= 3 ? 2 : (sh.k == 2 ? 3 : 4);
  sh.u = sh.k == 4 ? 2 : 4;
  if constexpr (kBf16) {
    // BF16 rows (8 values per chunk: F = 602 is k = 3, F = 128 is k = 1 with 2 virtual warps), measured on an H100
    // SXM at 700 W with tools/gather_dtype_sweep.py --tune (BF16-tuned plans of config B, whole call):
    // k = 3, F = 602: U=2 at 3 CTAs/SM 10.16 ms vs U=4 at 2 CTAs 10.56 / U=6 at 1 CTA 13.77;
    // k = 1, F = 128 (G = 2): U=4 at 4 CTAs 1.74 ms vs U=8 at 2 CTAs 2.06 (forward and backward alike)
    sh.minb = sh.k >= 4 ? 2 : (sh.k >= 2 ? 3 : 4);
    sh.u = sh.k == 1 ? 4 : 2;
  }
  {
    static int env_read = 0;
    if (!env_read) {
      env_read = 1;
      if (const char *t = getenv("NTS_PLAN_TUNE"))
        sscanf(t, "%d,%d,%d", &g_plan_u, &g_plan_minb, &g_plan_q);
    }
    if (g_plan_u > 0)
      sh.u = g_plan_u;
    if (g_plan_minb > 0)
      sh.minb = g_plan_minb;
  }
  uint32_t Q = g_plan_q > 0 ? (uint32_t)g_plan_q : 512u / sh.g; // the CTA's staged span stays 8 * 512 pairs
  if (g_plan_q <= 0) { // shrink for small inputs so every slab launch still fills the SMs
    const uint64_t per_slab = pl->slab_edge[pl->slabs] / (uint64_t)pl->slabs + 1; // residual edges (no hub blocks)
    const uint64_t want_warps = (uint64_t)sm_count() * 64 * sh.g;
    while (Q > 32 && ((per_slab + Q - 1) / Q) * sh.tiles < want_warps)
      Q >>= 1;
  }
  Q = (Q + 31u) & ~31u;
  if (Q * sh.g > 1024)
    Q = (1024 / sh.g) & ~31u;
  pl->last_k = sh.k, pl->last_u = sh.u, pl->last_outv = sh.outv;
  float *out = output;
  if (fused) {
    if constexpr (kBf16) {
      NTS_PLAN_FUSED_CASE(1, 4, 4, 2)
      NTS_PLAN_FUSED_CASE(1, 4, 4, 4)
      NTS_PLAN_FUSED_CASE(1, 4, 4, 1)
      NTS_PLAN_FUSED_CASE(2, 2, 3, 1)
      NTS_PLAN_FUSED_CASE(3, 2, 3, 1)
      NTS_PLAN_FUSED_CASE(4, 2, 2, 1)
      NTS_PLAN_FUSED_CASE(5, 2, 2, 1)
    } else {
      NTS_PLAN_FUSED_CASE(1, 4, 4, 2)
      NTS_PLAN_FUSED_CASE(1, 4, 4, 4)
      NTS_PLAN_FUSED_CASE(1, 4, 4, 1)
      NTS_PLAN_FUSED_CASE(2, 4, 3, 1)
      NTS_PLAN_FUSED_CASE(3, 4, 2, 1)
      NTS_PLAN_FUSED_CASE(4, 2, 2, 1)
      NTS_PLAN_FUSED_CASE(5, 4, 2, 1)
    }
    return fail(-1, "no fused slab/hub-row instantiation for this (chunks, U, occupancy) point", __FILE__, __LINE__);
  }
  if constexpr (kBf16) {
    // only points that compile without spills (a BF16 chunk holds 8 accumulators: U*K loads cost what they do in
    // FP32, the accumulators twice as much)
    NTS_PLAN_CASE_G(4, 4, 2)
    NTS_PLAN_CASE_G(4, 4, 4)
    NTS_PLAN_CASE_G(8, 2, 2)
    NTS_PLAN_CASE_G(8, 2, 4)
    if (sh.g != 1)
      return fail(-1, "no BF16 virtual-warp instantiation for this (U, occupancy) point", __FILE__, __LINE__);
    NTS_PLAN_CASE(1, 4, 4)
    NTS_PLAN_CASE(1, 8, 2)
    NTS_PLAN_CASE(2, 2, 3)
    NTS_PLAN_CASE(2, 4, 2)
    NTS_PLAN_CASE(3, 4, 2)
    NTS_PLAN_CASE(3, 2, 3)
    NTS_PLAN_CASE(3, 6, 1)
    NTS_PLAN_CASE(4, 2, 2)
    NTS_PLAN_CASE(4, 4, 2)
    NTS_PLAN_CASE(5, 2, 2)
    return fail(-1, "no BF16 planned-aggregation instantiation for this (chunks, U, occupancy) point", __FILE__,
                __LINE__);
  } else {
  const float4 *in4 = reinterpret_cast<const float4 *>(in);
  const uint32_t ld4 = ldc;
  if (g_plan_variant == 1) { // TMA row staging (measurement variant): U = ring depth
    // occupancy as for variant 0 (or set_tuning's): 4 / 3 / 2 CTAs per SM at 1 / 2 / 3+ chunks per lane, each with a
    // ring of 4 stages (2 at 4 chunks) at the default U
    const int stages = sh.u >= 8 ? 8 : (sh.u >= 4 ? 4 : 2);
    NTS_PLAN_TMA_CASE(1, 8, 4)
    NTS_PLAN_TMA_CASE(1, 4, 4)
    NTS_PLAN_TMA_CASE(1, 8, 3)
    NTS_PLAN_TMA_CASE(2, 4, 3)
    NTS_PLAN_TMA_CASE(2, 4, 2)
    NTS_PLAN_TMA_CASE(3, 4, 2)
    NTS_PLAN_TMA_CASE(4, 4, 2)
    NTS_PLAN_TMA_CASE(4, 2, 2)
    NTS_PLAN_TMA_CASE(5, 4, 2)
    NTS_PLAN_TMA_CASE(5, 2, 2)
    NTS_PLAN_TMA_CASE(5, 4, 1)
    NTS_PLAN_TMA_CASE(5, 8, 1)
    return fail(-1, "no TMA row-staging instantiation for this (chunks, stages, occupancy) point", __FILE__, __LINE__);
  }
  NTS_PLAN_CASE_G(4, 4, 2)
  NTS_PLAN_CASE_G(4, 4, 4)
  NTS_PLAN_CASE_G(8, 3, 2)
  NTS_PLAN_CASE_G(8, 3, 4)
  if (sh.g != 1)
    return fail(-1, "no virtual-warp instantiation for this (U, occupancy) point", __FILE__, __LINE__);
  NTS_PLAN_CASE(1, 8, 4)
  NTS_PLAN_CASE(1, 4, 4)
  NTS_PLAN_CASE(1, 8, 3)
  NTS_PLAN_CASE(1, 16, 2)
  NTS_PLAN_CASE(2, 4, 3)
  NTS_PLAN_CASE(2, 8, 2)
  NTS_PLAN_CASE(3, 4, 3)
  NTS_PLAN_CASE(3, 4, 2)
  NTS_PLAN_CASE(4, 2, 2)
  NTS_PLAN_CASE(4, 4, 2)
  NTS_PLAN_CASE(5, 2, 2)
  NTS_PLAN_CASE(5, 1, 3)
  NTS_PLAN_CASE(5, 2, 3)
  NTS_PLAN_CASE(5, 4, 1)
  NTS_PLAN_CASE(5, 4, 2)
  return fail(-1, "no planned-aggregation instantiation for this (chunks, U, occupancy) point", __FILE__, __LINE__);
  }
}

// Workspace of at least `elems` values of E (grown, never shrunk; shared by every width that runs the plan).
template <class E> static int ensure_workspace(E *&ws, size_t &have, size_t elems) {
  if (elems <= have)
    return 0;
  if (ws)
    NTS_CUDA_OK(cudaFree(ws));
  ws = nullptr;
  have = 0;
  NTS_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(&ws), elems * sizeof(E)));
  have = elems;
  return 0;
}

// Argument checks and the runs with nothing to gather, shared by the FP32 and BF16 entries: *done = the run is
// complete (an empty overwrite run still zeroes its output).  Returns 0 or the error.
static int run_prologue(nts_gather_plan *pl, const void *input, uint32_t lds, float *output, uint32_t F, int flags,
                        bool *done, cudaStream_t st) {
  *done = true;
  NTS_ARG_CHECK((flags & ~(NTS_PLAN_OVERWRITE | NTS_PLAN_COPY_INPUT)) == 0, "unknown plan run flags");
  if (pl->n_rows == 0 || F == 0)
    return 0;
  if (pl->n_edges == 0) {
    if (flags & NTS_PLAN_OVERWRITE) {
      NTS_ARG_CHECK(output != nullptr, "null output pointer");
      NTS_CUDA_OK(cudaMemsetAsync(output, 0, (size_t)pl->n_rows * F * sizeof(float), st));
    }
    return 0;
  }
  NTS_ARG_CHECK(input && output, "null feature pointer");
  NTS_ARG_CHECK(lds >= F, "row stride below the feature width");
  *done = false;
  return 0;
}

// FP32 rows of stride lds.  16-byte loads need 16-byte aligned rows: the input is gathered in place when lds % 4 == 0
// and it is aligned (the gather then reads columns F..lds of every row, the last one included, but never writes them
// to an output); otherwise, or with NTS_PLAN_COPY_INPUT, from a zero-padded copy (ld = F rounded up to 4).
int run_plan(nts_gather_plan *pl, const float *input, uint32_t lds, float *output, uint32_t F, int flags,
             cudaStream_t st) {
  bool done = false;
  if (const int rc = run_prologue(pl, input, lds, output, F, flags, &done, st))
    return rc;
  if (done)
    return 0;
  if (lds % 4 == 0 && aligned_to(input, 16) && !(flags & NTS_PLAN_COPY_INPUT))
    return run_gather<float>(pl, input, lds, output, F, flags & NTS_PLAN_OVERWRITE, st);
  const uint32_t ld = (F + 3u) & ~3u;
  if (const int rc = ensure_workspace(pl->workspace, pl->workspace_floats, (size_t)pl->gather_rows * ld))
    return rc;
  const uint64_t total = (uint64_t)pl->gather_rows * ld;
  const unsigned blocks = (unsigned)std::min<uint64_t>((total + 255) / 256, (uint64_t)sm_count() * 32);
  pad_rows_kernel<<<blocks, 256, 0, st>>>(input, lds, pl->workspace, pl->gather_rows, F, ld);
  NTS_LAUNCH_CHECK();
  return run_gather<float>(pl, pl->workspace, ld, output, F, flags & NTS_PLAN_OVERWRITE, st);
}

// dst[r, 0:ld] = {bf16(src[r, 0:F]), 0...} for rows of stride lds (elements of src's type); ld % 8 == 0
int to_bf16_rows(const void *src, int dtype, uint32_t lds, void *dst, uint32_t n_rows, uint32_t F, uint32_t ld,
                 cudaStream_t st) {
  NTS_ARG_CHECK(dtype == NTS_DTYPE_F32 || dtype == NTS_DTYPE_BF16, "input dtype must be NTS_DTYPE_F32 or NTS_DTYPE_BF16");
  NTS_ARG_CHECK(ld % 8 == 0 && ld >= F && lds >= F && aligned_to(dst, 16), "bad BF16 row layout");
  if (!n_rows || !F)
    return 0;
  const uint64_t total = (uint64_t)n_rows * (ld / 8);
  const unsigned blocks = (unsigned)std::min<uint64_t>((total + 255) / 256, (uint64_t)sm_count() * 32);
  uint4 *d = static_cast<uint4 *>(dst);
  if (dtype == NTS_DTYPE_F32)
    bf16_rows_kernel<float><<<blocks, 256, 0, st>>>(static_cast<const float *>(src), lds, d, n_rows, F, ld);
  else
    bf16_rows_kernel<__nv_bfloat16><<<blocks, 256, 0, st>>>(static_cast<const __nv_bfloat16 *>(src), lds, d, n_rows,
                                                            F, ld);
  NTS_LAUNCH_CHECK();
  return 0;
}

// BF16 gathers on rows of stride lds elements: an FP32 input is rounded into the BF16 workspace (stride ld = F rounded
// up to 8); a BF16 input is gathered in place when its stride is a whole number of 16-byte chunks and it is aligned
// (values between F and lds are never written to an output column), else (or with NTS_PLAN_COPY_INPUT) re-strided
// into the workspace.  flags: NTS_PLAN_OVERWRITE / NTS_PLAN_COPY_INPUT as for nts_gather_plan_run_ex.
int run_plan_bf16(nts_gather_plan *pl, const void *input, int dtype, uint32_t lds, float *output, uint32_t F,
                  cudaStream_t st, int flags) {
  NTS_ARG_CHECK(dtype == NTS_DTYPE_F32 || dtype == NTS_DTYPE_BF16, "input dtype must be NTS_DTYPE_F32 or NTS_DTYPE_BF16");
  NTS_ARG_CHECK(g_plan_variant == 0, "the TMA row-staging variant (nts_gather_plan_set_variant(1)) gathers FP32 rows only");
  bool done = false;
  if (const int rc = run_prologue(pl, input, lds, output, F, flags, &done, st))
    return rc;
  if (done)
    return 0;
  const bool overwrite = flags & NTS_PLAN_OVERWRITE;
  if (dtype == NTS_DTYPE_BF16 && lds % 8 == 0 && aligned_to(input, 16) && !(flags & NTS_PLAN_COPY_INPUT))
    return run_gather<__nv_bfloat16>(pl, static_cast<const __nv_bfloat16 *>(input), lds, output, F, overwrite, st);
  const uint32_t ld = (F + 7u) & ~7u;
  if (const int rc = ensure_workspace(pl->workspace_bf16, pl->workspace_bf16_elems, (size_t)pl->gather_rows * ld))
    return rc;
  if (const int rc = to_bf16_rows(input, dtype, lds, pl->workspace_bf16, pl->gather_rows, F, ld, st))
    return rc;
  return run_gather<__nv_bfloat16>(pl, pl->workspace_bf16, ld, output, F, overwrite, st);
}

// Slab-count bound for gathered rows of row_bytes bytes each (FP32: F rounded up to 4 floats, BF16: to 8 values).
static int pick_slabs_for_rows(nts_vid_t gather_rows, uint64_t n_edges, nts_vid_t n_rows, uint64_t row_bytes,
                               uint64_t l2_budget_bytes) {
  if (!l2_budget_bytes)
    l2_budget_bytes = 16ull << 20; // a third of the 50 MB L2: the slab stays resident next to the streamed outputs
  const uint64_t bytes = (uint64_t)gather_rows * row_bytes;
  uint64_t s = (bytes + l2_budget_bytes - 1) / l2_budget_bytes;
  // every (slab, row) segment costs one read-modify-write of the output row: keep >= 16 edges per segment on average
  const uint64_t by_degree = n_rows ? n_edges / ((uint64_t)n_rows * 16ull) : 1;
  if (s > by_degree)
    s = by_degree;
  if (s > 64)
    s = 64;
  return s < 1 ? 1 : (int)s;
}

// Exact reference counts of the gathered rows and segment lengths of the output rows, on the host.
static bool hub_counts(const nts_vid_t *offsets, const nts_vid_t *indices, const nts_vid_t *slot_of, nts_vid_t base,
                       uint32_t n_rows, uint32_t E, uint32_t gather_rows, std::vector<uint32_t> &col_cnt,
                       std::vector<uint32_t> &seg, cudaStream_t st) {
  uint32_t *cnt = nullptr;
  std::vector<uint32_t> off(n_rows + 1);
  col_cnt.assign(gather_rows, 0);
  const unsigned blocks = (unsigned)std::min<uint64_t>(((uint64_t)E + 255) / 256, (uint64_t)sm_count() * 32);
  bool ok = cudaMalloc(reinterpret_cast<void **>(&cnt), (size_t)gather_rows * 4) == cudaSuccess &&
            cudaMemsetAsync(cnt, 0, (size_t)gather_rows * 4, st) == cudaSuccess;
  if (ok && E) {
    plan_ref_count_kernel<<<blocks, 256, 0, st>>>(indices, slot_of, base, E, cnt);
    count_launch();
  }
  ok = ok && cudaMemcpyAsync(col_cnt.data(), cnt, (size_t)gather_rows * 4, cudaMemcpyDeviceToHost, st) == cudaSuccess &&
       cudaMemcpyAsync(off.data(), offsets, ((size_t)n_rows + 1) * 4, cudaMemcpyDeviceToHost, st) == cudaSuccess &&
       cudaStreamSynchronize(st) == cudaSuccess;
  cudaFree(cnt);
  seg.resize(n_rows);
  for (uint32_t r = 0; r < n_rows; r++)
    seg[r] = off[r + 1] - off[r];
  return ok;
}

// The h ids of largest count, ties broken by the smaller id (deterministic), largest first.
static std::vector<uint32_t> top_ids(const std::vector<uint32_t> &cnt, size_t h) {
  std::vector<uint32_t> ids(cnt.size());
  for (size_t i = 0; i < ids.size(); i++)
    ids[i] = (uint32_t)i;
  h = std::min(h, ids.size());
  std::partial_sort(ids.begin(), ids.begin() + h, ids.end(),
                    [&](uint32_t a, uint32_t b) { return cnt[a] != cnt[b] ? cnt[a] > cnt[b] : a < b; });
  ids.resize(h);
  return ids;
}

static nts_gather_plan *refuse_plan(const char *what) {
  fail(-1, what, __FILE__, __LINE__);
  return nullptr;
}

// The sorted layout of pl (pairs and voff allocated, d_parts the device copy of the parts): one stable LSD radix sort
// of all edges by key, so the edges of one (slab, row) segment or one dense cell keep the order of the parts and each
// part its own edge order; then the residual pairs in sorted order, the segment offsets and the host copy of the slab
// boundaries.  KeyT = uint32_t: (slab, row) keys only.  KeyT = uint64_t: hub columns / hub rows of the single part are
// picked, the sort also splits off the edges of the two dense blocks and each dense cell is the sum of its edges'
// weights.
template <class KeyT>
static bool sort_plan(nts_gather_plan *pl, const nts_plan_part *parts, int n_parts, const nts_plan_part *d_parts,
                      int n_hub_cols, int n_hub_rows, cudaStream_t st) {
  constexpr bool hubs = sizeof(KeyT) == 8;
  const uint32_t E = (uint32_t)pl->n_edges, n_rows = pl->n_rows, G = pl->gather_rows;
  const uint64_t n_keys = (uint64_t)pl->slabs * n_rows;
  uint64_t dc_cells = 0;
  uint32_t *d_col_slot = nullptr, *d_row_slot = nullptr, *d_runs = nullptr;
  bool ok = true;
  if (hubs) {
    const nts_plan_part &pt = parts[0];
    std::vector<uint32_t> col_cnt, seg;
    if (!hub_counts(pt.offsets, pt.indices, pt.slot_of, pt.index_base, n_rows, E, G, col_cnt, seg, st))
      return false;
    const std::vector<uint32_t> cols = top_ids(col_cnt, (size_t)n_hub_cols), rows = top_ids(seg, (size_t)n_hub_rows);
    pl->hub_cols = (int)cols.size();
    pl->hub_rows = (int)rows.size();
    pl->lda_c = (n_rows + 3u) & ~3u;
    pl->lda_r = ((uint32_t)pl->hub_rows + 3u) & ~3u;
    dc_cells = (uint64_t)pl->hub_cols * pl->lda_c;
    pl->dense_floats = dc_cells + (pl->hub_rows ? (uint64_t)G * pl->lda_r : 0);
    std::vector<uint32_t> col_slot(G, kNoHub), row_slot(n_rows, kNoHub);
    for (size_t i = 0; i < cols.size(); i++)
      col_slot[cols[i]] = (uint32_t)i;
    for (size_t i = 0; i < rows.size(); i++)
      row_slot[rows[i]] = (uint32_t)i;
    ok = cudaMalloc(reinterpret_cast<void **>(&pl->dense), pl->dense_floats * 4) == cudaSuccess &&
         cudaMalloc(reinterpret_cast<void **>(&pl->hub_col_ids), cols.size() * 4 + 4) == cudaSuccess &&
         cudaMalloc(reinterpret_cast<void **>(&pl->hub_row_ids), rows.size() * 4 + 4) == cudaSuccess &&
         cudaMalloc(reinterpret_cast<void **>(&d_col_slot), (size_t)G * 4 + 4) == cudaSuccess &&
         cudaMalloc(reinterpret_cast<void **>(&d_row_slot), (size_t)n_rows * 4 + 4) == cudaSuccess &&
         cudaMalloc(reinterpret_cast<void **>(&d_runs), 4) == cudaSuccess &&
         cudaMemcpyAsync(pl->hub_col_ids, cols.data(), cols.size() * 4, cudaMemcpyHostToDevice, st) == cudaSuccess &&
         cudaMemcpyAsync(pl->hub_row_ids, rows.data(), rows.size() * 4, cudaMemcpyHostToDevice, st) == cudaSuccess &&
         cudaMemcpyAsync(d_col_slot, col_slot.data(), (size_t)G * 4, cudaMemcpyHostToDevice, st) == cudaSuccess &&
         cudaMemcpyAsync(d_row_slot, row_slot.data(), (size_t)n_rows * 4, cudaMemcpyHostToDevice, st) == cudaSuccess &&
         cudaMemsetAsync(pl->dense, 0, pl->dense_floats * 4, st) == cudaSuccess;
  }
  int bits = 1;
  while (bits < (int)(8 * sizeof(KeyT)) && (1ull << bits) < n_keys + pl->dense_floats)
    bits++;
  KeyT *key_in = nullptr, *key_out = nullptr;
  uint32_t *val_in = nullptr, *val_out = nullptr;
  void *tmp = nullptr;
  size_t tmp_bytes = 0;
  ok = ok && cudaMalloc(reinterpret_cast<void **>(&key_in), (size_t)E * sizeof(KeyT)) == cudaSuccess &&
       cudaMalloc(reinterpret_cast<void **>(&key_out), (size_t)E * sizeof(KeyT)) == cudaSuccess &&
       cudaMalloc(reinterpret_cast<void **>(&val_in), (size_t)E * 4) == cudaSuccess &&
       cudaMalloc(reinterpret_cast<void **>(&val_out), (size_t)E * 4) == cudaSuccess &&
       cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, key_in, key_out, val_in, val_out, (int64_t)E, 0, bits, st) ==
           cudaSuccess &&
       cudaMalloc(&tmp, tmp_bytes ? tmp_bytes : 16) == cudaSuccess;
  uint32_t e_off = 0;
  for (int k = 0; k < n_parts && ok; k++) {
    const nts_plan_part &pt = parts[k];
    if (!pt.n_edges)
      continue;
    const unsigned blocks = (unsigned)std::min<uint64_t>((pt.n_edges + 255) / 256, (uint64_t)sm_count() * 32);
    plan_keys_kernel<KeyT><<<blocks, 256, 0, st>>>(pt, e_off, n_rows, pl->slab_rows, (uint32_t)pl->slabs, d_col_slot,
                                                   d_row_slot, pl->lda_c, dc_cells, pl->lda_r, key_in, val_in);
    count_launch();
    e_off += (uint32_t)pt.n_edges;
  }
  ok = ok && cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, key_in, key_out, val_in, val_out, (int64_t)E, 0, bits,
                                             st) == cudaSuccess;
  if (ok) {
    const unsigned kb = (unsigned)std::min<uint64_t>((n_keys + 256) / 256, (uint64_t)sm_count() * 32);
    plan_offsets_kernel<KeyT><<<kb, 256, 0, st>>>(key_out, E, (uint32_t)n_keys, pl->voff);
    count_launch();
    std::vector<uint32_t> h(pl->slabs + 1);
    ok = cudaStreamSynchronize(st) == cudaSuccess;
    for (int s = 0; s <= pl->slabs && ok; s++)
      ok = cudaMemcpy(&h[s], pl->voff + (size_t)s * n_rows, 4, cudaMemcpyDeviceToHost) == cudaSuccess;
    for (int s = 0; s <= pl->slabs; s++)
      pl->slab_edge[s] = h[s];
  }
  const uint32_t n_res = (uint32_t)pl->slab_edge[pl->slabs], n_dense = E - n_res;
  if (ok && n_res) {
    const unsigned blocks = (unsigned)std::min<uint64_t>(((uint64_t)n_res + 255) / 256, (uint64_t)sm_count() * 32);
    plan_pairs_kernel<<<blocks, 256, 0, st>>>(val_out, d_parts, n_res, pl->pairs);
    count_launch();
  }
  if constexpr (hubs) {
    if (ok && n_dense) { // runs of equal cell keys: (key, length), start = exclusive sum of the lengths (integers)
      uint32_t n_runs = 0;
      size_t b1 = 0, b2 = 0;
      ok = cub::DeviceRunLengthEncode::Encode(nullptr, b1, key_out + n_res, key_in, val_in, d_runs, (int64_t)n_dense,
                                              st) == cudaSuccess &&
           cub::DeviceScan::ExclusiveSum(nullptr, b2, val_in, d_col_slot, (int64_t)n_dense, st) == cudaSuccess;
      if (ok && std::max(b1, b2) > tmp_bytes) {
        cudaFree(tmp);
        tmp_bytes = std::max(b1, b2);
        ok = cudaMalloc(&tmp, tmp_bytes) == cudaSuccess;
      }
      uint32_t *run_start = nullptr;
      ok = ok && cudaMalloc(reinterpret_cast<void **>(&run_start), (size_t)n_dense * 4) == cudaSuccess &&
           cub::DeviceRunLengthEncode::Encode(tmp, b1, key_out + n_res, key_in, val_in, d_runs, (int64_t)n_dense, st) ==
               cudaSuccess &&
           cudaMemcpyAsync(&n_runs, d_runs, 4, cudaMemcpyDeviceToHost, st) == cudaSuccess &&
           cudaStreamSynchronize(st) == cudaSuccess &&
           cub::DeviceScan::ExclusiveSum(tmp, b2, val_in, run_start, (int64_t)n_runs, st) == cudaSuccess;
      if (ok) {
        const unsigned rb = (unsigned)std::min<uint64_t>(((uint64_t)n_runs * 32 + 255) / 256, (uint64_t)sm_count() * 32);
        plan_cell_sum_kernel<<<rb, 256, 0, st>>>(key_in, run_start, val_in, n_runs, val_out + n_res, parts[0].weight,
                                                 n_keys, pl->dense);
        count_launch();
        ok = cudaStreamSynchronize(st) == cudaSuccess;
      }
      cudaFree(run_start);
    }
  }
  cudaFree(key_in), cudaFree(key_out), cudaFree(val_in), cudaFree(val_out), cudaFree(tmp);
  cudaFree(d_col_slot), cudaFree(d_row_slot), cudaFree(d_runs);
  return ok;
}

// The plan builder: the edges of parts (a single chunk is one part with row_add = index_add = 0) bucketed by (slab,
// output row), with n_hub_cols / n_hub_rows dense hub blocks beside the residual (a single part only).  The caller has
// checked the parts' arrays and row ranges.
static nts_gather_plan *build_plan(const nts_plan_part *parts, int n_parts, nts_vid_t n_rows, nts_vid_t gather_rows,
                                   int n_slabs, int n_hub_cols, int n_hub_rows, cudaStream_t st) {
  uint64_t total = 0;
  for (int k = 0; k < n_parts; k++)
    total += parts[k].n_edges;
  if (total >= 0xffffffffull)
    return refuse_plan("plan edge count must fit uint32 offsets");
  if (n_slabs < 1 || gather_rows == 0)
    n_slabs = 1;
  if ((uint64_t)n_slabs * n_rows >= 0xffffffffull)
    return refuse_plan("slabs * rows must fit 32-bit segment keys");
  const bool hubs = gather_rows > 0 && (n_hub_cols > 0 || n_hub_rows > 0);
  if (hubs && n_parts != 1)
    return refuse_plan("hub blocks need a plan of a single part");
  nts_gather_plan *pl = new nts_gather_plan();
  pl->n_rows = n_rows;
  pl->n_edges = total;
  pl->gather_rows = gather_rows;
  pl->slabs = n_slabs;
  pl->slab_rows = gather_rows ? (gather_rows + n_slabs - 1) / n_slabs : 1;
  pl->slab_edge.assign(n_slabs + 1, 0);
  if (n_rows == 0 || total == 0)
    return pl;
  const uint32_t E = (uint32_t)total;
  nts_plan_part *d_parts = nullptr;
  bool ok = cudaMalloc(reinterpret_cast<void **>(&pl->pairs), (size_t)E * sizeof(uint2)) == cudaSuccess &&
            cudaMalloc(reinterpret_cast<void **>(&pl->voff), ((size_t)n_slabs * n_rows + 1) * 4) == cudaSuccess &&
            cudaMalloc(reinterpret_cast<void **>(&d_parts), n_parts * sizeof(nts_plan_part)) == cudaSuccess &&
            cudaMemcpyAsync(d_parts, parts, n_parts * sizeof(nts_plan_part), cudaMemcpyHostToDevice, st) == cudaSuccess;
  if (ok && n_slabs == 1 && !hubs && n_parts == 1 && parts[0].row_add == 0 && parts[0].n_rows == n_rows) {
    // one part in its own row order: the stable sort would leave every edge in place
    const unsigned blocks = (unsigned)std::min<uint64_t>(((uint64_t)E + 255) / 256, (uint64_t)sm_count() * 32);
    plan_pairs_kernel<<<blocks, 256, 0, st>>>(nullptr, d_parts, E, pl->pairs);
    count_launch();
    ok = cudaMemcpyAsync(pl->voff, parts[0].offsets, ((size_t)n_rows + 1) * 4, cudaMemcpyDeviceToDevice, st) ==
         cudaSuccess;
    pl->slab_edge[1] = E;
  } else if (ok) {
    ok = hubs ? sort_plan<uint64_t>(pl, parts, n_parts, d_parts, n_hub_cols, n_hub_rows, st)
              : sort_plan<uint32_t>(pl, parts, n_parts, d_parts, 0, 0, st);
  }
  if (ok)
    ok = cudaStreamSynchronize(st) == cudaSuccess && cudaGetLastError() == cudaSuccess;
  cudaFree(d_parts);
  if (!ok) {
    nts_gather_plan_destroy(pl);
    return refuse_plan("nts_gather_plan: device allocation or preprocessing failed");
  }
  return pl;
}

// Slab count by measurement.  Whether bucketing pays depends on how skewed the gathered rows are (hub sources stay in
// L1/L2 by themselves: on an H100, the Zipf graph of config B at F=602 takes 24.8 ms unbucketed, 19.5 ms with 4 slabs
// and 25.5 ms with 16; with uniform endpoints 87.1 ms vs 39.0 ms at 16 slabs) and on the degree distribution of the output rows (every non-empty
// (slab, row) segment costs a read-modify-write of the output row) - so the candidates 1, 2, 4, ... up to the
// size-based bound are built and timed on the real arrays (zero features: the access pattern does not depend on the
// values), 1 warm + 2 timed launches each, and the fastest is kept.  One-time cost per (chunk, direction, width).
//
// Then the dense hub blocks, by coordinate descent from the best plain plan: hub columns 32, 64, ... with no hub rows,
// then hub rows 32, 64, ... with the chosen columns (each stops at the first candidate that is not faster), then the
// slab count of the residual at half and twice the plain plan's: at most 12 more timed builds.  NTS_PLAN_HUBS=0
// (measurement override) skips this.  Only rows with more than kHubFloor edges per cell of their column / row of the
// block are candidates, which keeps uniform and sparse inputs hub-free without any timing: on an H100 SXM (700 W) the
// F=602 gather of config B averages ~170 ps per edge (19.4 ms for 114.8 M edges), a dense cell costs 2 * 608 flop,
// ~18 ps at the 67 TFLOP/s FP32 data-sheet rate, so below ~0.1 edge per cell a column cannot pay for itself even at
// peak; 0.05 leaves a factor of two for the timed search to settle.
static constexpr double kHubFloor = 0.05;
static constexpr int kHubMax = 512;

nts_gather_plan *tune_plan(const nts_plan_part *parts, int n_parts, nts_vid_t n_rows, nts_vid_t gather_rows,
                           nts_vid_t feature_size, bool bf16, int run_flags, bool hubs_allowed, cudaStream_t st) {
  uint64_t n_edges = 0;
  for (int k = 0; k < n_parts; k++)
    n_edges += parts[k].n_edges;
  const uint64_t row_bytes = bf16 ? ((feature_size + 7ull) & ~7ull) * 2ull : ((feature_size + 3ull) & ~3ull) * 4ull;
  const int s_max = pick_slabs_for_rows(gather_rows, n_edges, n_rows, row_bytes, 16ull << 20);
  const char *hub_env = getenv("NTS_PLAN_HUBS");
  const bool try_hubs = hubs_allowed && !(hub_env && strcmp(hub_env, "0") == 0) && n_rows > 0 && gather_rows > 0;
  nts_gather_plan *best = build_plan(parts, n_parts, n_rows, gather_rows, 1, 0, 0, st);
  if (!best || (s_max <= 1 && !try_hubs) || n_edges == 0 || feature_size == 0)
    return best;
  float *x = nullptr, *y = nullptr;
  const size_t xb = (size_t)gather_rows * feature_size * (bf16 ? 2 : sizeof(float)),
               yb = (size_t)n_rows * feature_size * sizeof(float);
  bool ok = cudaMalloc(reinterpret_cast<void **>(&x), xb) == cudaSuccess &&
            cudaMalloc(reinterpret_cast<void **>(&y), yb) == cudaSuccess &&
            cudaMemsetAsync(x, 0, xb, st) == cudaSuccess && cudaMemsetAsync(y, 0, yb, st) == cudaSuccess;
  auto time_plan = [&](nts_gather_plan *pl, float *ms) {
    return time_min_of_two([&] {
      return bf16 ? run_plan_bf16(pl, x, NTS_DTYPE_BF16, feature_size, y, feature_size, st, run_flags)
                  : run_plan(pl, x, feature_size, y, feature_size, run_flags, st);
    }, st, ms) == 0;
  };
  float best_ms = 0.f;
  ok = ok && time_plan(best, &best_ms);
  // build and time one candidate, keep it if it is faster: 1 = kept, 0 = not kept (*ms its time), -1 = failed
  auto consider = [&](int s, int hc, int hr, float *ms, int overlap = 0) -> int {
    nts_gather_plan *pl = build_plan(parts, n_parts, n_rows, gather_rows, s, hc, hr, st);
    if (pl)
      pl->overlap = overlap;
    if (!pl || !time_plan(pl, ms)) {
      nts_gather_plan_destroy(pl);
      return -1;
    }
    if (*ms < best_ms) {
      nts_gather_plan_destroy(best);
      best = pl;
      best_ms = *ms;
      return 1;
    }
    nts_gather_plan_destroy(pl);
    return 0;
  };
  for (int s = 2; ok && s_max > 1; s *= 2) {
    const int cand = s > s_max ? s_max : s;
    float ms = 0.f;
    const int r = consider(cand, 0, 0, &ms);
    if (r < 0 || (r == 0 && ms > 1.1f * best_ms)) // getting worse: larger slab counts only add read-modify-writes
      break;
    if (cand == s_max)
      break;
  }
  if (ok && try_hubs) {
    const nts_plan_part &pt = parts[0];
    std::vector<uint32_t> col_cnt, seg;
    ok = hub_counts(pt.offsets, pt.indices, pt.slot_of, pt.index_base, n_rows, (uint32_t)n_edges, gather_rows, col_cnt,
                    seg, st);
    int n_c = 0, n_r = 0;
    for (uint32_t c : col_cnt)
      n_c += c > kHubFloor * n_rows;
    for (uint32_t s : seg)
      n_r += s > kHubFloor * gather_rows;
    const int plain_slabs = best->slabs;
    float ms = 0.f;
    for (int c = 32; ok && c <= std::min(n_c, kHubMax); c *= 2)
      if (consider(best->slabs, c, 0, &ms) != 1)
        break;
    for (int r = 32; ok && r <= std::min(n_r, kHubMax); r *= 2)
      if (consider(best->slabs, best->hub_cols, r, &ms) != 1)
        break;
    if (best->hub_cols || best->hub_rows) {
      const int hc = best->hub_cols, hr = best->hub_rows;
      for (int s : {plain_slabs / 2, std::min(plain_slabs * 2, s_max)})
        if (s >= 1 && s != plain_slabs && s != best->slabs)
          consider(s, hc, hr, &ms);
    }
    // Then the schedule: the row block inside the slab launches against before them, for the chosen counts; when the
    // fused schedule wins, more hub rows may pay under it, so the hub-row search continues upward under it.
    // NTS_PLAN_OVERLAP=0 (measurement override) keeps the sequential schedule.
    const char *ov_env = getenv("NTS_PLAN_OVERLAP");
    if (ok && best->hub_rows && !(ov_env && strcmp(ov_env, "0") == 0)) {
      best->overlap = 1;
      float fused_ms = 0.f;
      if (time_plan(best, &fused_ms) && fused_ms < best_ms) {
        best_ms = fused_ms;
        for (int r = 2 * best->hub_rows; r <= std::min(n_r, kHubMax); r *= 2)
          if (consider(best->slabs, best->hub_cols, r, &ms, 1) != 1)
            break;
      } else {
        best->overlap = 0;
      }
    }
  }
  cudaFree(x), cudaFree(y);
  best->tuned_ms = best_ms;
  return best;
}

} // namespace nts

using namespace nts;

extern "C" {

int nts_gather_plan_pick_slabs(nts_vid_t gather_rows, uint64_t n_edges, nts_vid_t n_rows, nts_vid_t feature_size,
                               uint64_t l2_budget_bytes) {
  return pick_slabs_for_rows(gather_rows, n_edges, n_rows, ((feature_size + 3ull) & ~3ull) * 4ull, l2_budget_bytes);
}

// The arguments of a single-chunk entry as a plan part; false (error set) when they are refused.
static bool chunk_part(const nts_vid_t *offsets, const nts_vid_t *indices, const float *weight,
                       const nts_vid_t *slot_of, nts_vid_t index_base, nts_vid_t n_rows, uint64_t n_edges,
                       nts_plan_part *pt) {
  if (n_rows && n_edges && !(offsets && indices)) {
    refuse_plan("null graph array");
    return false;
  }
  *pt = {offsets, indices, weight, slot_of, index_base, 0, n_rows, 0, n_edges};
  return true;
}

nts_gather_plan *nts_gather_plan_create_hybrid(const nts_vid_t *offsets, const nts_vid_t *indices,
                                               const float *weight, const nts_vid_t *slot_of, nts_vid_t index_base,
                                               nts_vid_t n_rows, uint64_t n_edges, nts_vid_t gather_rows, int n_slabs,
                                               int n_hub_cols, int n_hub_rows, void *stream) {
  nts_plan_part pt;
  if (!chunk_part(offsets, indices, weight, slot_of, index_base, n_rows, n_edges, &pt))
    return nullptr;
  if (n_hub_cols < 0 || n_hub_rows < 0)
    return refuse_plan("negative hub count");
  return build_plan(&pt, 1, n_rows, gather_rows, n_slabs, n_hub_cols, n_hub_rows, as_stream(stream));
}

nts_gather_plan *nts_gather_plan_create_tuned_ex(const nts_vid_t *offsets, const nts_vid_t *indices,
                                                 const float *weight, const nts_vid_t *slot_of, nts_vid_t index_base,
                                                 nts_vid_t n_rows, uint64_t n_edges, nts_vid_t gather_rows,
                                                 nts_vid_t feature_size, int gather_dtype, int run_flags,
                                                 void *stream) {
  if ((gather_dtype != NTS_DTYPE_F32 && gather_dtype != NTS_DTYPE_BF16) || (run_flags & ~NTS_PLAN_OVERWRITE))
    return refuse_plan("nts_gather_plan_create_tuned_ex: gather_dtype must be NTS_DTYPE_F32 or NTS_DTYPE_BF16, "
                       "run_flags 0 or NTS_PLAN_OVERWRITE");
  nts_plan_part pt;
  if (!chunk_part(offsets, indices, weight, slot_of, index_base, n_rows, n_edges, &pt))
    return nullptr;
  return tune_plan(&pt, 1, n_rows, gather_rows, feature_size, gather_dtype == NTS_DTYPE_BF16, run_flags, true,
                   as_stream(stream));
}

nts_gather_plan *nts_gather_plan_create_parts(const nts_plan_part *parts, int n_parts, nts_vid_t n_rows,
                                              nts_vid_t gather_rows, int n_slabs, nts_vid_t feature_size, void *stream) {
  if (!parts || n_parts < 1)
    return refuse_plan("no plan parts");
  for (int k = 0; k < n_parts; k++) {
    if (parts[k].n_edges && !(parts[k].offsets && parts[k].indices))
      return refuse_plan("null graph array in a plan part");
    if ((uint64_t)parts[k].row_add + parts[k].n_rows > n_rows)
      return refuse_plan("plan part rows exceed the output rows");
  }
  if (n_slabs >= 1)
    return build_plan(parts, n_parts, n_rows, gather_rows, n_slabs, 0, 0, as_stream(stream));
  return tune_plan(parts, n_parts, n_rows, gather_rows, feature_size, false, 0, false, as_stream(stream));
}

float nts_gather_plan_tuned_ms(const nts_gather_plan *pl) { return pl ? pl->tuned_ms : 0.f; }

int nts_gather_plan_destroy(nts_gather_plan *pl) {
  if (!pl)
    return 0;
  cudaFree(pl->pairs);
  cudaFree(pl->voff);
  cudaFree(pl->workspace);
  cudaFree(pl->workspace_bf16);
  cudaFree(pl->dense);
  cudaFree(pl->hub_col_ids);
  cudaFree(pl->hub_row_ids);
  delete pl;
  return 0;
}

int nts_gather_plan_slabs(const nts_gather_plan *pl) { return pl ? pl->slabs : 0; }

int nts_gather_plan_hubs(const nts_gather_plan *pl, int *cols, int *rows) {
  NTS_ARG_CHECK(pl != nullptr, "null plan");
  if (cols)
    *cols = pl->hub_cols;
  if (rows)
    *rows = pl->hub_rows;
  return 0;
}

int nts_gather_plan_overlap(const nts_gather_plan *pl) { return pl ? pl->overlap : 0; }

int nts_gather_plan_set_overlap(nts_gather_plan *pl, int overlap) {
  NTS_ARG_CHECK(pl != nullptr, "null plan");
  NTS_ARG_CHECK(overlap == 0 || overlap == 1, "overlap must be 0 (sequential) or 1 (fused slab launches)");
  pl->overlap = overlap;
  return 0;
}

uint64_t nts_gather_plan_bytes(const nts_gather_plan *pl) {
  if (!pl)
    return 0;
  return pl->n_edges * 8ull + ((uint64_t)pl->slabs * pl->n_rows + 1) * 4ull + pl->workspace_floats * 4ull +
         pl->workspace_bf16_elems * 2ull + pl->dense_floats * 4ull + ((uint64_t)pl->hub_cols + pl->hub_rows) * 4ull;
}

int nts_gather_plan_last_launch(const nts_gather_plan *pl, int *launches, int *grid, int *k, int *u, int *outv) {
  NTS_ARG_CHECK(pl != nullptr, "null plan");
  if (launches)
    *launches = pl->last_launches;
  if (grid)
    *grid = pl->last_grid;
  if (k)
    *k = pl->last_k;
  if (u)
    *u = pl->last_u;
  if (outv)
    *outv = pl->last_outv;
  return 0;
}

int nts_gather_plan_run_ex(nts_gather_plan *pl, const float *input, nts_vid_t input_ld, float *output,
                           nts_vid_t feature_size, int flags, void *stream) {
  NTS_ARG_CHECK(input_ld >= feature_size, "input row pitch below the feature width");
  NTS_ARG_CHECK(output != nullptr || feature_size == 0, "null output pointer");
  NTS_ARG_CHECK(pl != nullptr, "null plan");
  return run_plan(pl, input, input_ld, output, feature_size, flags, as_stream(stream));
}

int nts_gather_plan_run_bf16_ex(nts_gather_plan *pl, const void *input, int input_dtype, nts_vid_t input_ld,
                                float *output, nts_vid_t feature_size, int flags, void *stream) {
  NTS_ARG_CHECK(input_ld >= feature_size, "input row pitch below the feature width");
  NTS_ARG_CHECK(output != nullptr || feature_size == 0, "null output pointer");
  NTS_ARG_CHECK(pl != nullptr, "null plan");
  return run_plan_bf16(pl, input, input_dtype, input_ld, output, feature_size, as_stream(stream), flags);
}

int nts_rows_to_bf16(const void *src, int src_dtype, nts_vid_t lds, void *dst, nts_vid_t n_rows, nts_vid_t feature_size,
                     nts_vid_t ld, void *stream) {
  NTS_ARG_CHECK((src && dst) || n_rows == 0 || feature_size == 0, "null pointer passed to nts_rows_to_bf16");
  return to_bf16_rows(src, src_dtype, lds, dst, n_rows, feature_size, ld, as_stream(stream));
}

int nts_gather_plan_set_variant(int variant) {
  NTS_ARG_CHECK(variant == 0 || variant == 1, "variant must be 0 (register staging) or 1 (TMA row staging)");
  g_plan_variant = variant;
  return 0;
}

int nts_gather_plan_set_tuning(int u, int min_blocks, int edges_per_warp) {
  NTS_ARG_CHECK(u >= 0 && min_blocks >= 0 && edges_per_warp >= 0 && edges_per_warp <= 4096, "bad tuning point");
  g_plan_u = u;
  g_plan_minb = min_blocks;
  g_plan_q = edges_per_warp;
  return 0;
}

} // extern "C"
