// Segmented weighted gather-sum (the SpMM-like neighbour aggregation) for sm_90a.
//
//   out[r,:] += sum_{e in [off[r], off[r+1])} in[src(e),:] * w[e]
//
// replaces the eight `aggregate_kernel_from_{src,dst}_*` kernels of the reference
// (cuda/ntsCUDAFuseKernel.cuh:147-487) and their launchers (cuda/ntsCUDAGraphOP.cu:157-281).
//
// Design (see DESIGN.md "K1"): HBM/L2-bound gather.  Work is split by EDGES, not rows: warp g owns
// the edge quantum [q*Q, (q+1)*Q) of column tile t (g = q*tiles + t), finds its first row with a
// binary search over the offsets, and walks the edges keeping a register accumulator of K vector
// chunks per lane.  Feature rows are read with 4/8/16-byte vector loads (width picked from F and the
// pointer alignment: F=602 rows are only 8-byte aligned), U edges are loaded before any FMA so
// every lane keeps U*K independent loads in flight.  A row that lies entirely inside the quantum is
// written with one non-atomic read-modify-write; a row cut by a quantum boundary (hubs) is finished
// with vector `red.global.add` atomics.  No row-degree assumptions, no per-edge atomics, 64-bit
// address arithmetic throughout.
//
// Two index/weight staging variants:
//   variant 1 (shuffle): each lane loads one edge's (index, weight) coalesced, broadcast by __shfl.
//   variant 2 (bulk):    one thread per CTA issues `cp.async.bulk` (TMA, SASS UBLKCP) copies of the
//                        CTA's index and weight tiles into shared memory, completion on an mbarrier;
//                        warps then read (index, weight) with broadcast LDS.  DEFAULT (H100, F=602
//                        Reddit-shaped launch: 26.4 vs 27.7 ms; F=128: 4.77 vs 4.93 ms).
//
// Template parameters of segment_gather_sum_kernel<VEC,K,U,BULK,MINB,HM>: VEC floats per lane load, K vector
// chunks per lane (a warp covers 32*VEC*K columns per tile), U edges whose loads are issued before their FMAs,
// BULK = variant 2, MINB = __launch_bounds__ min CTAs/SM (register cap), HM = head mode: 0 one weight per edge,
// 1 the weight array is [E,H] and each lane picks its column's head, 2 the weight is recomputed on the fly from the
// per-vertex attention scores and softmax statistics (the fused GAT layer, nts_edge_ops.cu K7).
// (U, MINB) per shape come from tools/tune_aggregate.py sweeps; NTS_AGG_TUNE / NTS_AGG_TILES are
// measurement hooks read once at first launch, not product configuration.
#include <type_traits>

#include "nts_common.cuh"

namespace nts {

static int g_variant = 0;          // 0 = auto
static int g_edges_per_warp = 0;   // 0 = auto
static int g_last_grid = 0, g_last_block = 0, g_last_smem = 0, g_last_variant = 0;
static int g_last_vec = 0, g_last_k = 0, g_last_u = 0, g_last_minb = 0, g_last_tiles = 0; // instantiation of the last launch

constexpr int kWarpsPerBlock = 8;

// Fused GAT attention (K7): instead of loading a per-edge weight, recompute it from per-vertex scores
//   a[e,h] = exp(leaky_relu(s[slot(e),h] + d[row,h]) - m[row,h]) / z[row,h]      (column tile t = head h)
// m / z are the per-(destination, head) softmax statistics produced by gat_softmax_stats_kernel.
struct AttParams {
  const float *s; // [M, H] source scores (mirror rows)
  const float *d; // [V, H] destination scores
  const float *m; // [V, H] segment max of the logits
  const float *z; // [V, H] segment sum of exp(logit - m)
  float slope;    // leaky_relu negative slope
};
__device__ __forceinline__ float att_weight(float s, float d, float m, float inv_z, float slope) {
  return expf(leaky(s + d, slope) - m) * inv_z;
}

// ---- the kernel --------------------------------------------------------------------------------------------
// VEC  : floats per vector load (1, 2, 4); feature_size % VEC == 0 and rows VEC*4-byte aligned
// K    : vector chunks per lane per column tile (a tile covers K*32*VEC floats)
// U    : edges loaded before the FMAs start (memory-level parallelism = U*K loads per lane)
// BULK : stage index/weight tiles with cp.async.bulk + mbarrier (variant 2)
// MINB : minimum resident CTAs per SM handed to __launch_bounds__ (register cap = 65536 / (256*MINB))
// HM   : head mode.  0 = one weight per edge (or none);
//                    1 = multi-head weights w[E, H]: every lane scales its columns with the weight of the head
//                        that owns them (head of column c = c / D), loaded per lane (lanes of one head broadcast);
//                    2 = fused GAT attention: the weight is recomputed from per-vertex scores (AttParams).
//        For HM != 0 a lane's K chunks may belong to different heads, so weights / row constants are per chunk.
// G    : virtual warps per warp (BULK only): rows of at most 16 vectors leave half of the lanes idle, so the warp is
//        split into G independent groups of 32/G lanes, each with its own edge quantum and row state (the BULK
//        variant has no warp-wide shuffles; all bookkeeping is per lane).  Used by the fused GAT layers (F = 64).
// T    : gathered element type.  float, or __nv_bfloat16 with VEC = 8: one 16-byte load carries 8 BF16 values that are
//        widened to FP32 in registers, and F is the BF16 row stride ld (a multiple of 8).  In the fused GAT layer
//        (HM == 2) the FP32 output shares that stride.  In head mode 0 (K1 on BF16 rows, kNarrowOut) the output is
//        [n_rows, Fo] contiguous with Fo <= ld carried in `heads` (unused by HM 0 otherwise): a lane's chunks cover
//        ceil(Fo / 8) chunks of the row and its flush writes only columns < Fo.
template <int VEC, int K, int U, bool BULK, int MINB = 1, int HM = 0, int G = 1, class T = float>
__global__ void __launch_bounds__(kWarpsPerBlock * 32, MINB)
    segment_gather_sum_kernel(const T *__restrict__ in, float *__restrict__ out, const float *__restrict__ w,
                              const uint32_t *__restrict__ idx, const uint32_t *__restrict__ off,
                              const uint32_t *__restrict__ slot_of, uint32_t base, uint32_t n_rows,
                              uint64_t n_edges64, uint32_t F, uint32_t Q, uint32_t tiles, uint32_t tile_vecs,
                              uint32_t tile_major, uint32_t heads, AttParams att, uint32_t e_begin, uint32_t out_mod) {
  static_assert(!(HM == 1 && BULK), "[E, H] weight matrices are not bulk-staged (indices of HM 0 / 2 are)");
  static_assert(G == 1 || (BULK && K == 1), "virtual warps need the shuffle-free variant and one chunk per lane");
  static_assert(std::is_same<T, float>::value || (HM != 1 && VEC == 8), "BF16 rows: head mode 0 or 2, 8 per chunk");
  constexpr bool kNarrowOut = !std::is_same<T, float>::value && HM == 0;
  using V = typename Vec<VEC>::type;
  using L = typename Ld<T, VEC>::type; // what a lane loads per chunk (FP32: V itself)
  constexpr uint32_t GS = 32 / G;
  constexpr uint32_t kVW = kWarpsPerBlock * G; // (virtual) warps per CTA
  const uint32_t n_edges = (uint32_t)n_edges64;
  const uint32_t lane = threadIdx.x & (GS - 1);
  const uint32_t warp_in_block = threadIdx.x / GS;
  const uint32_t nvec = kNarrowOut ? (heads + VEC - 1) / VEC : F / VEC;

  // quantum / column tile owned by this warp.
  //   interleaved (tile_major = 0): consecutive warps = the column tiles of one quantum (they share index loads)
  //   tile-major  (tile_major = 1): all quanta of tile 0 first, then tile 1, ...: at any moment the CTAs in flight
  //     touch one column slab of the feature matrix, which is sized to stay resident in the 50 MB L2.
  //     Warps per tile are padded to a multiple of the CTA size so a CTA never straddles two tiles.
  const uint64_t gwarp = (uint64_t)blockIdx.x * kVW + warp_in_block;
  // the launch covers edges [e_begin, n_edges64) of the arrays (e_begin = off[0]; 0 except for row-range launches)
  const uint64_t n_quanta = (n_edges64 - e_begin + Q - 1) / Q;
  const uint64_t wpt = (n_quanta + kVW - 1) / kVW * kVW;
  const uint32_t tile = tile_major ? (uint32_t)(gwarp / wpt) : (uint32_t)(gwarp % tiles);
  const uint64_t q = tile_major ? gwarp % wpt : gwarp / tiles;
  const uint64_t e0_64 = e_begin + q * (uint64_t)Q;

  // BULK staging buffers: indices+weights of every edge this CTA touches
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint32_t *s_idx = nullptr;
  float *s_w = nullptr;
  uint32_t cta_e_base = 0; // first staged edge (16-byte aligned element index)
  uint32_t bulk_bytes = 0;
  if constexpr (BULK) {
    // CTA edge span: quanta of warps 0..kVW-1
    const uint64_t cta_w0 = (uint64_t)blockIdx.x * kVW;
    const uint64_t first_q = tile_major ? cta_w0 % wpt : cta_w0 / tiles;
    const uint64_t last_q = tile_major ? first_q + kVW - 1 : (cta_w0 + kVW - 1) / tiles;
    uint64_t ce0 = e_begin + first_q * (uint64_t)Q;
    uint64_t ce1 = e_begin + (last_q + 1) * (uint64_t)Q;
    if (ce1 > n_edges)
      ce1 = n_edges;
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem_raw);
    const uint32_t span_cap = kVW * Q + 8; // elements reserved per array (host sizes smem to this)
    s_idx = reinterpret_cast<uint32_t *>(smem_raw + 16);
    s_w = reinterpret_cast<float *>(smem_raw + 16 + (size_t)span_cap * 4);
    if (ce0 < ce1) {
      cta_e_base = (uint32_t)(ce0 & ~3ull); // 16-byte aligned start (arrays are 16-byte aligned)
      const uint32_t n_el = (uint32_t)(ce1 - cta_e_base);
      bulk_bytes = (n_el * 4u) & ~15u;      // whole 16-byte units go through the bulk engine ...
      const uint32_t bulk_el = bulk_bytes / 4u;
      if (threadIdx.x == 0) {
        mbar_init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      }
      if (threadIdx.x < n_el - bulk_el) {   // ... the last < 4 elements by plain loads (never read past the array)
        s_idx[bulk_el + threadIdx.x] = __ldg(idx + cta_e_base + bulk_el + threadIdx.x);
        if (w)
          s_w[bulk_el + threadIdx.x] = __ldg(w + cta_e_base + bulk_el + threadIdx.x);
      }
      __syncthreads();
      if (threadIdx.x == 0 && bulk_bytes) {
        mbar_expect_tx(bar, w ? 2 * bulk_bytes : bulk_bytes);
        bulk_g2s(s_idx, idx + cta_e_base, bulk_bytes, bar);
        if (w)
          bulk_g2s(s_w, w + cta_e_base, bulk_bytes, bar);
      }
    }
  }

  if (e0_64 >= n_edges64) {
    return; // (BULK: a CTA whose later warps have no work still issued/awaited nothing they need)
  }
  const uint32_t e0 = (uint32_t)e0_64;
  const uint32_t e1 = (e0_64 + Q < n_edges64) ? e0 + Q : n_edges;

  // column tile handled by this warp
  const uint32_t c0 = tile * tile_vecs + lane; // first vector column of this lane
  bool act[K];
  uint32_t hk[K]; // head that owns chunk k of this lane (HM != 0)
#pragma unroll
  for (int k = 0; k < K; k++) {
    act[k] = (k * GS + lane) < tile_vecs && (c0 + k * GS) < nvec;
    hk[k] = 0;
    if constexpr (HM != 0)
      hk[k] = act[k] ? ((c0 + k * GS) * VEC) / (F / heads) : 0u;
  }

  // first row of the quantum (overlaps with the bulk copy in flight)
  uint32_t row = find_row(off, n_rows, e0);
  uint32_t row_end = __ldg(off + row + 1);
  bool row_started_inside = __ldg(off + row) >= e0;

  V acc[K];
#pragma unroll
  for (int k = 0; k < K; k++)
    zero_vec(acc[k]);

  // per-row attention constants of the heads of this lane's chunks (HM == 2)
  float att_d[K], att_m[K], att_iz[K];
  auto load_att_row = [&]() {
    if constexpr (HM == 2) {
#pragma unroll
      for (int k = 0; k < K; k++) {
        const size_t o = (size_t)(out_mod ? row % out_mod : row) * heads + hk[k];
        att_d[k] = __ldg(att.d + o);
        att_m[k] = __ldg(att.m + o);
        att_iz[k] = 1.f / __ldg(att.z + o);
      }
    }
  };
  load_att_row();

  // slab-bucketed launches (out_mod != 0): `row` is a virtual row (slab * out_mod + output row); the slabs of one
  // output row are processed by different warps, possibly at the same time, so every flush is a reduction
  auto flush = [&](bool whole) {
    const uint32_t orow = out_mod ? row % out_mod : row;
    whole = whole && !out_mod;
    if constexpr (kNarrowOut) {
#pragma unroll
      for (int k = 0; k < K; k++) {
        if (act[k])
          flush_cols(out + (size_t)orow * heads, (c0 + k * GS) * 8u, heads, acc[k], whole);
        zero_vec(acc[k]);
      }
    } else {
      V *o = reinterpret_cast<V *>(out + (size_t)orow * F) + c0;
#pragma unroll
      for (int k = 0; k < K; k++) {
        if (act[k]) {
          if (whole)
            rmw_add(o + k * GS, acc[k]);
          else
            red_add(o + k * GS, acc[k]);
        }
        zero_vec(acc[k]);
      }
    }
  };
  // move to the row containing edge ee (ee >= row_end on entry)
  auto advance = [&](uint32_t ee) {
    flush(row_started_inside); // row_end <= ee < e1: the row ends inside the quantum
    do {
      row++;
      row_end = __ldg(off + row + 1);
    } while (ee >= row_end);
    row_started_inside = true;
    load_att_row();
  };
  // weight of (edge value, chunk k) in the accumulate phase
  auto weight_of = [&](float raw, int k) -> float {
    if constexpr (HM == 2)
      return att_weight(raw, att_d[k], att_m[k], att_iz[k], att.slope);
    else
      return raw;
  };

  if constexpr (BULK) {
    if (bulk_bytes)
      mbar_wait(reinterpret_cast<uint64_t *>(smem_raw), 0);
  }

  for (uint32_t e = e0; e < e1; e += 32) {
    const uint32_t cnt = min(32u, e1 - e);
    uint32_t my_src = 0;
    float my_w = 1.f;
    if constexpr (!BULK) {
      if (lane < cnt) {
        uint32_t id = __ldg(idx + e + lane);
        my_src = slot_of ? __ldg(slot_of + id) : id - base;
        if constexpr (HM == 0)
          if (w)
            my_w = __ldg(w + e + lane);
      }
    }
    uint32_t j = 0;
    // full groups of U edges: U*K independent vector loads per lane, then the FMAs
    for (; j + U <= cnt; j += U) {
      L v[U][K];
      float wu[U][HM == 0 ? 1 : K];
#pragma unroll
      for (int u = 0; u < U; u++) {
        uint32_t s;
        if constexpr (BULK) {
          uint32_t id = s_idx[e + j + u - cta_e_base];
          s = slot_of ? __ldg(slot_of + id) : id - base;
          if constexpr (HM == 0)
            wu[u][0] = w ? s_w[e + j + u - cta_e_base] : 1.f;
        } else {
          s = __shfl_sync(0xffffffffu, my_src, j + u);
          if constexpr (HM == 0)
            wu[u][0] = __shfl_sync(0xffffffffu, my_w, j + u);
        }
        const L *p = reinterpret_cast<const L *>(in + (size_t)s * F) + c0;
#pragma unroll
        for (int k = 0; k < K; k++) {
          if (act[k])
            v[u][k] = __ldg(p + k * GS);
          if constexpr (HM == 1)
            wu[u][k] = act[k] ? __ldg(w + (size_t)(e + j + u) * heads + hk[k]) : 0.f;
          if constexpr (HM == 2)
            wu[u][k] = act[k] ? __ldg(att.s + (size_t)s * heads + hk[k]) : 0.f;
        }
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        const uint32_t ee = e + j + u;
        if (ee >= row_end)
          advance(ee);
#pragma unroll
        for (int k = 0; k < K; k++)
          if (act[k])
            fma_vec(acc[k], weight_of(wu[u][HM == 0 ? 0 : k], k), widen(v[u][k]));
      }
    }
    // remainder (< U edges)
    for (; j < cnt; j++) {
      uint32_t s;
      float wj[HM == 0 ? 1 : K];
      if constexpr (BULK) {
        uint32_t id = s_idx[e + j - cta_e_base];
        s = slot_of ? __ldg(slot_of + id) : id - base;
        if constexpr (HM == 0)
          wj[0] = w ? s_w[e + j - cta_e_base] : 1.f;
      } else {
        s = __shfl_sync(0xffffffffu, my_src, j);
        if constexpr (HM == 0)
          wj[0] = __shfl_sync(0xffffffffu, my_w, j);
      }
      const L *p = reinterpret_cast<const L *>(in + (size_t)s * F) + c0;
      L v1[K];
#pragma unroll
      for (int k = 0; k < K; k++) {
        if (act[k])
          v1[k] = __ldg(p + k * GS);
        if constexpr (HM == 1)
          wj[k] = act[k] ? __ldg(w + (size_t)(e + j) * heads + hk[k]) : 0.f;
        if constexpr (HM == 2)
          wj[k] = act[k] ? __ldg(att.s + (size_t)s * heads + hk[k]) : 0.f;
      }
      const uint32_t ee = e + j;
      if (ee >= row_end)
        advance(ee);
#pragma unroll
      for (int k = 0; k < K; k++)
        if (act[k])
          fma_vec(acc[k], weight_of(wj[HM == 0 ? 0 : k], k), widen(v1[k]));
    }
  }
  // last row of the quantum: whole only if it started inside and also ends at/before e1
  flush(row_started_inside && row_end <= e1);
}

// ---- host-side dispatch ---------------------------------------------------------------------------------
struct LaunchShape {
  int vec, k, u, minb;
  uint32_t tiles, tile_vecs, tile_major, heads;
  int g = 1;            // virtual warps per warp (fused attention on rows of <= 16 vectors)
  uint32_t e_begin = 0; // first edge of the launch (row-range launches), offsets[0]
  uint32_t out_mod = 0; // != 0: offsets index virtual rows slab * out_mod + row (slab-bucketed arrays)
};

static LaunchShape pick_shape(const float *in, const float *out, uint32_t F, uint32_t heads) {
  LaunchShape s;
  s.heads = heads ? heads : 1;
  s.vec = pick_vec(F, in, out);
  if (heads > 1) // a head's columns must be a whole number of vectors
    while (s.vec > 1 && (F / heads) % s.vec != 0)
      s.vec >>= 1;
  const uint32_t nvec = F / s.vec;
  const uint32_t chunks = (nvec + 31) / 32;
  const uint32_t kmax = (s.vec == 4) ? 4 : 5;
  s.tiles = (chunks + kmax - 1) / kmax;
  s.tile_major = 0;
  // experiment / tuning hook: NTS_AGG_TILES="tiles,tile_major"
  if (const char *e = getenv("NTS_AGG_TILES")) {
    int t = 0, m = 0;
    if (sscanf(e, "%d,%d", &t, &m) == 2 && t >= 1 && (uint32_t)t <= chunks && (chunks + t - 1) / t <= kmax) {
      s.tiles = (uint32_t)t;
      s.tile_major = m ? 1u : 0u;
    }
  }
  s.tile_vecs = (nvec + s.tiles - 1) / s.tiles;
  s.k = (int)((s.tile_vecs + 31) / 32);
  s.tiles = (nvec + s.tile_vecs - 1) / s.tile_vecs;
  // (U, min CTAs/SM): measured on an H100 for the headline shapes (NTS_PLAN=0 tools/tune_aggregate.py, the
  // Reddit-shaped graph), generic rule otherwise
  s.minb = 1;
  int budget = 40 / (s.k * s.vec);
  s.u = budget >= 8 ? 8 : (budget >= 4 ? 4 : 2);
  if (s.vec == 2 && s.k == 5) { // F=602: 26.4 ms vs 26.2 (U=4, 1 CTA) / 26.3 (U=4, 2 CTAs) / 27.1 (U=2, 3 CTAs)
    s.u = 2;
    s.minb = 2;
  } else if (s.vec == 4 && s.k == 1) { // F=128: 4.77 ms vs 6.0 (U=8, 4 CTAs) / 6.1 (U=8, 1 CTA) / 6.7 (U=16, 2)
    s.u = 4;
    s.minb = 4;
  }
  if (const char *tune = getenv("NTS_AGG_TUNE")) {
    int tu = 0, tb = 0;
    if (sscanf(tune, "%d,%d", &tu, &tb) == 2) {
      s.u = tu;
      s.minb = tb;
    }
  }
  return s;
}

static const AttParams kNoAtt = {nullptr, nullptr, nullptr, nullptr, 0.f};

template <int VEC, int K, int U, int MINB>
static int launch_shape(bool bulk, const LaunchShape &sh, const float *in, float *out, const float *w,
                        const uint32_t *idx, const uint32_t *off, const uint32_t *slot_of, uint32_t base,
                        uint32_t n_rows, uint64_t n_edges, uint32_t F, uint32_t Q, cudaStream_t st,
                        const AttParams *att = nullptr) {
  const uint64_t quanta = (n_edges - sh.e_begin + Q - 1) / Q;
  uint64_t warps;
  if (sh.tile_major)
    warps = (quanta + kWarpsPerBlock - 1) / kWarpsPerBlock * kWarpsPerBlock * sh.tiles;
  else
    warps = quanta * sh.tiles;
  const uint64_t blocks = (warps + kWarpsPerBlock - 1) / kWarpsPerBlock;
  NTS_ARG_CHECK(blocks <= 0x7fffffffull, "aggregation grid too large");
  g_last_grid = (int)blocks;
  g_last_block = kWarpsPerBlock * 32;
  g_last_vec = VEC, g_last_k = K, g_last_u = U, g_last_minb = MINB, g_last_tiles = (int)sh.tiles;
  if (att || sh.heads > 1) {
    if constexpr (MINB == 1) { // per-head kernels exist for the untuned occupancy points only
      g_last_smem = 0;
      if constexpr (K == 1) {
        if (att && bulk && sh.g == 2) { // rows of <= 16 vectors: two virtual warps per warp
          constexpr int G2 = 2;
          size_t span_cap = (size_t)kWarpsPerBlock * G2 * Q + 8;
          size_t smem = 16 + 2 * span_cap * 4;
          auto kern = segment_gather_sum_kernel<VEC, K, U, true, 1, 2, G2>;
          NTS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
          g_last_smem = (int)smem;
          const uint64_t vblocks = (warps + kWarpsPerBlock * G2 - 1) / (kWarpsPerBlock * G2);
          g_last_grid = (int)vblocks;
          kern<<<(unsigned)vblocks, kWarpsPerBlock * 32, smem, st>>>(in, out, nullptr, idx, off, slot_of, base, n_rows,
                                                                     n_edges, F, Q, sh.tiles, sh.tile_vecs,
                                                                     sh.tile_major, sh.heads, *att, sh.e_begin,
                                                                     sh.out_mod);
          NTS_LAUNCH_CHECK();
          return 0;
        }
      }
      if (att && bulk) { // fused attention with TMA-staged index tiles (no weight array to stage)
        size_t span_cap = (size_t)kWarpsPerBlock * Q + 8;
        size_t smem = 16 + 2 * span_cap * 4;
        auto kern = segment_gather_sum_kernel<VEC, K, U, true, 1, 2>;
        NTS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        g_last_smem = (int)smem;
        kern<<<(unsigned)blocks, kWarpsPerBlock * 32, smem, st>>>(in, out, nullptr, idx, off, slot_of, base, n_rows,
                                                                  n_edges, F, Q, sh.tiles, sh.tile_vecs, sh.tile_major,
                                                                  sh.heads, *att, sh.e_begin, sh.out_mod);
      } else if (att)
        segment_gather_sum_kernel<VEC, K, U, false, 1, 2><<<(unsigned)blocks, kWarpsPerBlock * 32, 0, st>>>(
            in, out, nullptr, idx, off, slot_of, base, n_rows, n_edges, F, Q, sh.tiles, sh.tile_vecs, sh.tile_major,
            sh.heads, *att, sh.e_begin, sh.out_mod);
      else
        segment_gather_sum_kernel<VEC, K, U, false, 1, 1><<<(unsigned)blocks, kWarpsPerBlock * 32, 0, st>>>(
            in, out, w, idx, off, slot_of, base, n_rows, n_edges, F, Q, sh.tiles, sh.tile_vecs, sh.tile_major,
            sh.heads, kNoAtt, sh.e_begin, sh.out_mod);
      NTS_LAUNCH_CHECK();
      return 0;
    } else {
      return fail(-1, "no per-head kernel for this occupancy point", __FILE__, __LINE__);
    }
  }
  if (bulk) {
    size_t span_cap = (size_t)kWarpsPerBlock * Q + 8;
    size_t smem = 16 + 2 * span_cap * 4;
    auto kern = segment_gather_sum_kernel<VEC, K, U, true, MINB>;
    NTS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    g_last_smem = (int)smem;
    kern<<<(unsigned)blocks, kWarpsPerBlock * 32, smem, st>>>(in, out, w, idx, off, slot_of, base, n_rows, n_edges, F,
                                                              Q, sh.tiles, sh.tile_vecs, sh.tile_major, 1u, kNoAtt, sh.e_begin,
                                                              sh.out_mod);
  } else {
    g_last_smem = 0;
    segment_gather_sum_kernel<VEC, K, U, false, MINB><<<(unsigned)blocks, kWarpsPerBlock * 32, 0, st>>>(
        in, out, w, idx, off, slot_of, base, n_rows, n_edges, F, Q, sh.tiles, sh.tile_vecs, sh.tile_major, 1u,
        kNoAtt, sh.e_begin, sh.out_mod);
  }
  NTS_LAUNCH_CHECK();
  return 0;
}

#define NTS_CASE(V_, K_, U_, B_)                                                                               \
  if (s.vec == V_ && s.k == K_ && s.u == U_ && s.minb == B_)                                                    \
    return launch_shape<V_, K_, U_, B_>(bulk, s, in, out, w, idx, off, slot_of, base, n_rows, n_edges, F, Q, st, att);

static int segment_gather_sum(const float *in, float *out, const float *w, const uint32_t *idx, const uint32_t *off,
                              const uint32_t *slot_of, uint32_t base, uint32_t n_rows, uint64_t n_edges, uint32_t F,
                              cudaStream_t st, uint32_t heads = 1, const AttParams *att = nullptr,
                              uint64_t e_begin = 0, uint32_t out_mod = 0) {
  // n_edges is the END of the edge range [e_begin, n_edges) (= the edge count for whole-array launches)
  if (n_rows == 0 || n_edges <= e_begin || F == 0)
    return 0;
  NTS_ARG_CHECK(in && out && idx && off, "null pointer passed to segment_gather_sum");
  NTS_ARG_CHECK(n_edges < 0xffffffffull, "chunk edge count must fit uint32 offsets");
  if (heads > 1 && !att) {
    NTS_ARG_CHECK(w != nullptr, "multi-head aggregation needs the [E, heads] weight matrix");
    NTS_ARG_CHECK(F % heads == 0, "feature_size must be a multiple of heads");
  }
  LaunchShape s = pick_shape(in, out, F, heads);
  s.e_begin = (uint32_t)e_begin;
  s.out_mod = out_mod;
  if (heads > 1 || att) { // per-head kernels: untuned occupancy point
    s.minb = 1;
    int budget = 40 / (s.k * s.vec);
    s.u = budget >= 8 ? 8 : (budget >= 4 ? 4 : 2);
    if (att && s.k == 1 && s.tiles == 1 && F / s.vec <= 16 && !s.tile_major && !getenv("NTS_AGG_NO_SUBWARP"))
      s.g = 2;
  }
  // edges per warp: multiple of 32; shrink for small inputs so the grid still fills every SM
  uint32_t Q = g_edges_per_warp > 0 ? (uint32_t)g_edges_per_warp : 512u / (uint32_t)s.g;
  if (g_edges_per_warp <= 0) {
    const uint64_t want_warps = (uint64_t)sm_count() * 64;
    while (Q > 32 && ((n_edges - e_begin + Q - 1) / Q) * s.tiles < want_warps)
      Q >>= 1;
  }
  Q = (Q + 31u) & ~31u;
  if (s.g > 1 && Q * s.g > 1024) // the CTA's staged index span must keep fitting shared memory
    Q = (1024u / s.g) & ~31u;
  int variant = g_variant == 0 ? 2 : g_variant; // measured on an H100: bulk-staged indices are ~3-5% faster
  bool bulk = variant == 2 && (att || heads <= 1); // [E, H] weight matrices are not bulk-staged
  // the bulk copies need 16-byte aligned index/weight arrays (cudaMalloc gives 256)
  if (bulk && !(aligned_to(idx, 16) && (!w || aligned_to(w, 16)))) {
    bulk = false;
    variant = 1;
  }
  g_last_variant = variant;
  // default (U, MINB) points
  NTS_CASE(4, 1, 4, 4)
  NTS_CASE(4, 2, 4, 1)
  NTS_CASE(4, 3, 2, 1)
  NTS_CASE(4, 4, 2, 1)
  NTS_CASE(2, 1, 8, 1)
  NTS_CASE(2, 2, 8, 1)
  NTS_CASE(2, 3, 4, 1)
  NTS_CASE(2, 4, 4, 1)
  NTS_CASE(2, 5, 2, 2)
  NTS_CASE(1, 1, 8, 1)
  NTS_CASE(1, 2, 8, 1)
  NTS_CASE(1, 3, 8, 1)
  NTS_CASE(1, 4, 8, 1)
  NTS_CASE(1, 5, 8, 1)
  // extra points reachable through NTS_AGG_TUNE / NTS_AGG_TILES (tuning sweeps, tools/tune_aggregate.py)
  NTS_CASE(4, 1, 8, 1)
  NTS_CASE(4, 1, 8, 4)
  NTS_CASE(4, 1, 16, 2)
  NTS_CASE(4, 1, 8, 3)
  NTS_CASE(2, 5, 4, 1)
  NTS_CASE(2, 5, 2, 3)
  NTS_CASE(2, 5, 4, 2)
  NTS_CASE(2, 4, 2, 3)
  NTS_CASE(2, 4, 4, 2)
  NTS_CASE(2, 3, 2, 3)
  NTS_CASE(2, 3, 4, 3)
  NTS_CASE(2, 3, 4, 2)
  NTS_CASE(2, 2, 4, 3)
  NTS_CASE(2, 2, 4, 4)
  NTS_CASE(2, 2, 8, 2)
  NTS_CASE(2, 2, 8, 3)
  NTS_CASE(2, 1, 8, 4)
  NTS_CASE(2, 1, 8, 3)
  NTS_CASE(2, 1, 16, 2)
  return fail(-1, "no kernel instantiation for this (vector width, chunks, U, occupancy) point", __FILE__, __LINE__);
}

// ---- K7 forward on BF16 mirror rows --------------------------------------------------------------------------------
int check_gat_bf16_layout(uint32_t F, uint32_t ld, uint32_t heads) {
  NTS_ARG_CHECK(heads >= 1 && F % heads == 0, "feature_size must be a multiple of heads");
  NTS_ARG_CHECK(ld % 8 == 0 && ld >= F, "BF16 rows need a stride ld >= feature_size with ld % 8 == 0");
  NTS_ARG_CHECK(heads == 1 || ((F / heads) % 8 == 0 && ld == F),
                "BF16 rows with heads > 1 need a head width D % 8 == 0 (a 16-byte chunk never straddles two heads) "
                "and ld == feature_size");
  return 0;
}

template <int K, int U, int G>
static int launch_gat_bf16(const LaunchShape &sh, const __nv_bfloat16 *in, float *out, const uint32_t *idx,
                           const uint32_t *off, const uint32_t *slot_of, uint32_t n_rows, uint64_t n_edges,
                           uint32_t ld, uint32_t Q, const AttParams &att, cudaStream_t st) {
  constexpr uint32_t kVW = kWarpsPerBlock * G;
  const uint64_t warps = (n_edges + Q - 1) / Q * sh.tiles;
  const uint64_t blocks = (warps + kVW - 1) / kVW;
  NTS_ARG_CHECK(blocks <= 0x7fffffffull, "aggregation grid too large");
  const size_t smem = 16 + 2 * ((size_t)kVW * Q + 8) * 4;
  auto kern = segment_gather_sum_kernel<8, K, U, true, 1, 2, G, __nv_bfloat16>;
  NTS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  g_last_grid = (int)blocks;
  g_last_block = kWarpsPerBlock * 32;
  g_last_smem = (int)smem;
  g_last_variant = 2;
  g_last_vec = 8, g_last_k = K, g_last_u = U, g_last_minb = 1, g_last_tiles = (int)sh.tiles;
  kern<<<(unsigned)blocks, kWarpsPerBlock * 32, smem, st>>>(in, out, nullptr, idx, off, slot_of, 0, n_rows, n_edges,
                                                            ld, Q, sh.tiles, sh.tile_vecs, 0, sh.heads, att, 0, 0);
  NTS_LAUNCH_CHECK();
  return 0;
}

// Chunks of 8 values: K <= 4 chunks per lane per column tile; rows of at most 16 / 8 chunks (F <= 128 / 64) split the
// warp into G = 2 / 4 virtual warps (config D's 64-wide layers are 8 chunks: one head of 8 per lane at D = 8).
// NTS_GAT_BF16_TUNE="U,G" is a measurement hook (tools/gat_dtype_sweep.py --tune) for the one-chunk rows.
static int gat_forward_bf16(const __nv_bfloat16 *in, float *out, const uint32_t *idx, const uint32_t *off,
                            const uint32_t *slot_of, uint32_t n_rows, uint64_t n_edges, uint32_t ld,
                            uint32_t heads, const AttParams &att, cudaStream_t st) {
  LaunchShape s;
  s.heads = heads;
  s.vec = 8;
  const uint32_t nvec = ld / 8;
  const uint32_t chunks = (nvec + 31) / 32;
  s.tiles = (chunks + 3) / 4;
  s.tile_vecs = (nvec + s.tiles - 1) / s.tiles;
  s.k = (int)((s.tile_vecs + 31) / 32);
  s.tiles = (nvec + s.tile_vecs - 1) / s.tile_vecs;
  s.tile_major = 0;
  s.minb = 1;
  s.g = (s.k == 1 && s.tiles == 1) ? (nvec <= 8 ? 4 : (nvec <= 16 ? 2 : 1)) : 1;
  // U measured on config D's one-chunk rows (H100 SXM, 700 W, tools/gat_dtype_sweep.py --tune): G = 4 at U = 2 / 4 / 8
  // 4.63 / 4.80 / 5.47 ms per 64-wide call, 3.59 / 3.69 / 4.34 ms at 41 wide; G = 2 and G = 1 are slower at every U
  s.u = s.k == 1 ? 2 : (s.k == 2 ? 4 : 2);
  if (const char *tune = getenv("NTS_GAT_BF16_TUNE")) {
    int tu = 0, tg = 0;
    if (s.k == 1 && s.tiles == 1 && sscanf(tune, "%d,%d", &tu, &tg) == 2 && tg >= 1 && (uint32_t)(32 / tg) >= nvec) {
      s.u = tu;
      s.g = tg;
    }
  }
  uint32_t Q = 512u / (uint32_t)s.g; // edges per (virtual) warp, shrunk for small inputs as in segment_gather_sum
  const uint64_t want_warps = (uint64_t)sm_count() * 64;
  while (Q > 32 && ((n_edges + Q - 1) / Q) * s.tiles < want_warps)
    Q >>= 1;
  Q = (Q + 31u) & ~31u;
  if (Q * s.g > 1024)
    Q = (1024u / s.g) & ~31u;
#define NTS_GAT16(K_, U_, G_)                                                                                    \
  if (s.k == K_ && s.u == U_ && s.g == G_)                                                                       \
    return launch_gat_bf16<K_, U_, G_>(s, in, out, idx, off, slot_of, n_rows, n_edges, ld, Q, att, st);
  NTS_GAT16(1, 2, 1)
  NTS_GAT16(1, 4, 1)
  NTS_GAT16(1, 8, 1)
  NTS_GAT16(1, 2, 2)
  NTS_GAT16(1, 4, 2)
  NTS_GAT16(1, 8, 2)
  NTS_GAT16(1, 2, 4)
  NTS_GAT16(1, 4, 4)
  NTS_GAT16(1, 8, 4)
  NTS_GAT16(2, 4, 1)
  NTS_GAT16(3, 2, 1)
  NTS_GAT16(4, 2, 1)
#undef NTS_GAT16
  return fail(-1, "no BF16 fused-GAT instantiation for this (chunks, U, virtual warps) point", __FILE__, __LINE__);
}

// ---- K1 on BF16 rows (head mode 0) -----------------------------------------------------------------------------------
// out[r, :F] += sum_e w_e * float(in[idx[e], :F]) with BF16 rows of stride ld (ld % 8 == 0, ld >= F, 16-byte aligned)
// and a contiguous FP32 output [n_rows, F].  Same edge quanta, staging variants and atomics as the FP32 K1.
template <int K, int U, int MINB, int G>
static int launch_k1_bf16(bool bulk, const LaunchShape &sh, const __nv_bfloat16 *in, float *out, const float *w,
                          const uint32_t *idx, const uint32_t *off, uint32_t n_rows, uint64_t n_edges, uint32_t ld,
                          uint32_t F, uint32_t Q, cudaStream_t st) {
  constexpr uint32_t kVW = kWarpsPerBlock * G;
  const uint64_t warps = (n_edges + Q - 1) / Q * sh.tiles;
  const uint64_t blocks = (warps + kVW - 1) / kVW;
  NTS_ARG_CHECK(blocks <= 0x7fffffffull, "aggregation grid too large");
  g_last_grid = (int)blocks;
  g_last_block = kWarpsPerBlock * 32;
  g_last_variant = bulk ? 2 : 1;
  g_last_vec = 8, g_last_k = K, g_last_u = U, g_last_minb = MINB, g_last_tiles = (int)sh.tiles;
  if (bulk) {
    const size_t smem = 16 + 2 * ((size_t)kVW * Q + 8) * 4;
    auto kern = segment_gather_sum_kernel<8, K, U, true, MINB, 0, G, __nv_bfloat16>;
    NTS_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    g_last_smem = (int)smem;
    kern<<<(unsigned)blocks, kWarpsPerBlock * 32, smem, st>>>(in, out, w, idx, off, nullptr, 0, n_rows, n_edges, ld, Q,
                                                              sh.tiles, sh.tile_vecs, 0, F, kNoAtt, 0, 0);
  } else {
    if constexpr (G == 1) {
      g_last_smem = 0;
      segment_gather_sum_kernel<8, K, U, false, MINB, 0, 1, __nv_bfloat16><<<(unsigned)blocks, kWarpsPerBlock * 32, 0,
                                                                              st>>>(
          in, out, w, idx, off, nullptr, 0, n_rows, n_edges, ld, Q, sh.tiles, sh.tile_vecs, 0, F, kNoAtt, 0, 0);
    } else {
      return fail(-1, "virtual warps need the bulk-staged variant", __FILE__, __LINE__);
    }
  }
  NTS_LAUNCH_CHECK();
  return 0;
}

// Chunks of 8 values, K <= 4 per lane per column tile; rows of at most 16 chunks (F <= 128: F = 41 and 37 are 6 and 5
// chunks, F = 128 is 16) split the warp into G = 2 virtual warps under the bulk-staged variant, F = 602 (76 chunks) is
// K = 3.  (U, MINB, G) measured on sampled config B blocks (H100 SXM, 700 W, tools/sample_dtype_sweep.py): at F = 41
// G = 4 / 2 / 1 took 43.4 / 36.2 / 30.7 us at (U 4, MINB 4) and G = 2 took 30.7 us at MINB 2 (a block's few edges
// already shrink the quantum to 32, so G divides the grid); F = 602 U = 4 / 2: 73.5 / 75.4 us.  NTS_K1_BF16_TUNE="U,MINB,G"
// is a measurement hook, whose G applies only to a one-chunk row under the bulk variant that it fits.
static int segment_gather_sum_bf16(const __nv_bfloat16 *in, uint32_t ld, float *out, const float *w,
                                   const uint32_t *idx, const uint32_t *off, uint32_t n_rows, uint64_t n_edges,
                                   uint32_t F, cudaStream_t st) {
  LaunchShape s;
  s.vec = 8;
  s.heads = 1;
  s.tile_major = 0;
  const uint32_t nvec = (F + 7) / 8;
  const uint32_t chunks = (nvec + 31) / 32;
  s.tiles = (chunks + 3) / 4;
  s.tile_vecs = (nvec + s.tiles - 1) / s.tiles;
  s.k = (int)((s.tile_vecs + 31) / 32);
  s.tiles = (nvec + s.tile_vecs - 1) / s.tile_vecs;
  int variant = g_variant == 0 ? 2 : g_variant;
  // the bulk copies need 16-byte aligned index/weight arrays (cudaMalloc gives 256)
  if (variant == 2 && !(aligned_to(idx, 16) && (!w || aligned_to(w, 16))))
    variant = 1;
  const bool bulk = variant == 2;
  const bool narrow = bulk && s.k == 1 && s.tiles == 1;
  s.g = narrow && nvec <= 16 ? 2 : 1;
  s.u = s.k <= 3 ? 4 : 2;
  s.minb = s.k == 4 ? 1 : 2;
  if (const char *tune = getenv("NTS_K1_BF16_TUNE")) {
    int tu = 0, tb = 0, tg = 0;
    if (sscanf(tune, "%d,%d,%d", &tu, &tb, &tg) == 3) {
      s.u = tu;
      s.minb = tb;
      if (narrow && tg >= 1 && (uint32_t)(32 / tg) >= nvec)
        s.g = tg;
    }
  }
  uint32_t Q = g_edges_per_warp > 0 ? (uint32_t)g_edges_per_warp : 512u / (uint32_t)s.g;
  if (g_edges_per_warp <= 0) {
    const uint64_t want_warps = (uint64_t)sm_count() * 64;
    while (Q > 32 && ((n_edges + Q - 1) / Q) * s.tiles < want_warps)
      Q >>= 1;
  }
  Q = (Q + 31u) & ~31u;
  if (s.g > 1 && Q * s.g > 1024) // the CTA's staged index span must keep fitting shared memory
    Q = (1024u / s.g) & ~31u;
#define NTS_BF16_CASE(K_, U_, B_, G_)                                                                              \
  if (s.k == K_ && s.u == U_ && s.minb == B_ && s.g == G_)                                                         \
    return launch_k1_bf16<K_, U_, B_, G_>(bulk, s, in, out, w, idx, off, n_rows, n_edges, ld, F, Q, st);
  // default points
  NTS_BF16_CASE(1, 4, 2, 2)
  NTS_BF16_CASE(1, 4, 2, 1)
  NTS_BF16_CASE(2, 4, 2, 1)
  NTS_BF16_CASE(3, 4, 2, 1)
  NTS_BF16_CASE(4, 2, 1, 1)
  // extra points reachable through NTS_K1_BF16_TUNE
  NTS_BF16_CASE(1, 4, 4, 4)
  NTS_BF16_CASE(1, 4, 4, 2)
  NTS_BF16_CASE(1, 4, 4, 1)
  NTS_BF16_CASE(1, 2, 4, 4)
  NTS_BF16_CASE(1, 8, 2, 4)
  NTS_BF16_CASE(1, 4, 2, 4)
  NTS_BF16_CASE(1, 2, 4, 2)
  NTS_BF16_CASE(1, 8, 2, 2)
  NTS_BF16_CASE(3, 2, 2, 1)
  NTS_BF16_CASE(3, 2, 1, 1)
  NTS_BF16_CASE(3, 4, 1, 1)
#undef NTS_BF16_CASE
  return fail(-1, "no BF16 K1 instantiation for this (chunks, U, occupancy, virtual warps) point", __FILE__, __LINE__);
}

} // namespace nts

extern "C" {

int nts_segment_gather_sum(const float *input, float *output, const float *weight, const nts_vid_t *indices,
                           const nts_vid_t *offsets, nts_vid_t index_base, nts_vid_t n_rows, uint64_t n_edges,
                           nts_vid_t feature_size, void *stream) {
  return nts::segment_gather_sum(input, output, weight, indices, offsets, nullptr, index_base, n_rows, n_edges,
                                 feature_size, nts::as_stream(stream));
}

int nts_segment_gather_sum_range(const float *input, float *output, const float *weight, const nts_vid_t *indices,
                                 const nts_vid_t *offsets, const nts_vid_t *slot_of, nts_vid_t index_base,
                                 nts_vid_t n_rows, uint64_t edge_begin, uint64_t edge_end, nts_vid_t feature_size,
                                 void *stream) {
  NTS_ARG_CHECK(edge_begin <= edge_end, "edge range is reversed");
  return nts::segment_gather_sum(input, output, weight, indices, offsets, slot_of, index_base, n_rows, edge_end,
                                 feature_size, nts::as_stream(stream), 1, nullptr, edge_begin, 0);
}

int nts_segment_gather_sum_slots(const float *input, float *output, const float *weight, const nts_vid_t *indices,
                                 const nts_vid_t *offsets, const nts_vid_t *slot_of, nts_vid_t n_rows,
                                 uint64_t n_edges, nts_vid_t feature_size, void *stream) {
  NTS_ARG_CHECK(slot_of != nullptr, "slot table is null");
  return nts::segment_gather_sum(input, output, weight, indices, offsets, slot_of, 0, n_rows, n_edges, feature_size,
                                 nts::as_stream(stream));
}

int nts_segment_gather_sum_heads(const float *input, float *output, const float *weight, const nts_vid_t *indices,
                                 const nts_vid_t *offsets, const nts_vid_t *slot_of, nts_vid_t index_base,
                                 nts_vid_t n_rows, uint64_t n_edges, nts_vid_t feature_size, nts_vid_t heads,
                                 void *stream) {
  NTS_ARG_CHECK(heads >= 1, "heads must be >= 1");
  return nts::segment_gather_sum(input, output, weight, indices, offsets, slot_of, index_base, n_rows, n_edges,
                                 feature_size, nts::as_stream(stream), heads);
}

int nts_gat_fused_aggregate_forward(const float *mirror, float *output, const float *src_score,
                                    const float *dst_score, const float *seg_max, const float *seg_sum,
                                    const nts_vid_t *row_indices, const nts_vid_t *column_offset,
                                    const nts_vid_t *mirror_index, nts_vid_t batch_size, uint64_t n_edges,
                                    nts_vid_t feature_size, nts_vid_t heads, float negative_slope, void *stream) {
  NTS_ARG_CHECK(heads >= 1 && feature_size % heads == 0, "feature_size must be a multiple of heads");
  NTS_ARG_CHECK(src_score && dst_score && seg_max && seg_sum, "null pointer passed to fused GAT forward");
  nts::AttParams att = {src_score, dst_score, seg_max, seg_sum, negative_slope};
  return nts::segment_gather_sum(mirror, output, nullptr, row_indices, column_offset, mirror_index, 0, batch_size,
                                 n_edges, feature_size, nts::as_stream(stream), heads, &att);
}

int nts_gat_fused_aggregate_forward_bf16(const void *mirror, float *output, const float *src_score,
                                         const float *dst_score, const float *seg_max, const float *seg_sum,
                                         const nts_vid_t *row_indices, const nts_vid_t *column_offset,
                                         const nts_vid_t *mirror_index, nts_vid_t batch_size, uint64_t n_edges,
                                         nts_vid_t feature_size, nts_vid_t ld, nts_vid_t heads, float negative_slope,
                                         void *stream) {
  if (const int rc = nts::check_gat_bf16_layout(feature_size, ld, heads))
    return rc;
  if (batch_size == 0 || n_edges == 0 || feature_size == 0)
    return 0;
  NTS_ARG_CHECK(mirror && output && src_score && dst_score && seg_max && seg_sum && row_indices && column_offset,
                "null pointer passed to fused GAT forward (BF16)");
  NTS_ARG_CHECK(nts::aligned_to(mirror, 16) && nts::aligned_to(output, 16) && nts::aligned_to(row_indices, 16),
                "BF16 fused GAT forward needs 16-byte aligned mirror, output and row_indices");
  NTS_ARG_CHECK(n_edges < 0xffffffffull, "chunk edge count must fit uint32 offsets");
  nts::AttParams att = {src_score, dst_score, seg_max, seg_sum, negative_slope};
  return nts::gat_forward_bf16(static_cast<const __nv_bfloat16 *>(mirror), output, row_indices, column_offset,
                               mirror_index, batch_size, n_edges, ld, heads, att, nts::as_stream(stream));
}

int nts_segment_gather_sum_bf16(const void *input, nts_vid_t input_ld, float *output, const float *weight,
                                const nts_vid_t *indices, const nts_vid_t *offsets, nts_vid_t n_rows, uint64_t n_edges,
                                nts_vid_t feature_size, void *stream) {
  NTS_ARG_CHECK(input_ld % 8 == 0 && input_ld >= feature_size,
                "BF16 rows need a stride input_ld >= feature_size with input_ld % 8 == 0");
  if (n_rows == 0 || n_edges == 0 || feature_size == 0)
    return 0;
  NTS_ARG_CHECK(input && output && indices && offsets, "null pointer passed to nts_segment_gather_sum_bf16");
  NTS_ARG_CHECK(nts::aligned_to(input, 16), "nts_segment_gather_sum_bf16 needs a 16-byte aligned input");
  NTS_ARG_CHECK(n_edges < 0xffffffffull, "chunk edge count must fit uint32 offsets");
  return nts::segment_gather_sum_bf16(static_cast<const __nv_bfloat16 *>(input), input_ld, output, weight, indices,
                                      offsets, n_rows, n_edges, feature_size, nts::as_stream(stream));
}

int nts_gather_by_dst_from_src(const float *input, float *output, const float *weight_forward,
                               const nts_vid_t *row_indices, const nts_vid_t *column_offset, nts_vid_t src_start,
                               nts_vid_t src_end, nts_vid_t dst_start, nts_vid_t dst_end, nts_vid_t edges,
                               nts_vid_t batch_size, nts_vid_t feature_size, int with_weight, void *stream) {
  (void)src_end;
  (void)dst_start;
  (void)dst_end;
  if (batch_size == 0 || edges == 0 || feature_size == 0) // empty chunk / empty partition: nothing to add
    return 0;
  NTS_ARG_CHECK(!with_weight || weight_forward, "with_weight set but weight pointer is null");
  return nts::segment_gather_sum(input, output, with_weight ? weight_forward : nullptr, row_indices, column_offset,
                                 nullptr, src_start, batch_size, edges, feature_size, nts::as_stream(stream));
}

int nts_gather_by_src_from_dst(const float *input, float *output, const float *weight_backward,
                               const nts_vid_t *row_offset, const nts_vid_t *column_indices, nts_vid_t src_start,
                               nts_vid_t src_end, nts_vid_t dst_start, nts_vid_t dst_end, nts_vid_t edges,
                               nts_vid_t batch_size, nts_vid_t feature_size, int with_weight, void *stream) {
  (void)src_start;
  (void)src_end;
  (void)dst_end;
  if (batch_size == 0 || edges == 0 || feature_size == 0)
    return 0;
  NTS_ARG_CHECK(!with_weight || weight_backward, "with_weight set but weight pointer is null");
  return nts::segment_gather_sum(input, output, with_weight ? weight_backward : nullptr, column_indices, row_offset,
                                 nullptr, dst_start, batch_size, edges, feature_size, nts::as_stream(stream));
}

int nts_aggregate_set_variant(int variant, int edges_per_warp) {
  NTS_ARG_CHECK(variant >= 0 && variant <= 2, "variant must be 0 (auto), 1 (shuffle) or 2 (bulk)");
  NTS_ARG_CHECK(edges_per_warp >= 0 && edges_per_warp <= 4096, "edges_per_warp out of range");
  nts::g_variant = variant;
  nts::g_edges_per_warp = edges_per_warp;
  return 0;
}

int nts_aggregate_last_launch(int *grid, int *block, int *smem_bytes, int *variant) {
  if (grid)
    *grid = nts::g_last_grid;
  if (block)
    *block = nts::g_last_block;
  if (smem_bytes)
    *smem_bytes = nts::g_last_smem;
  if (variant)
    *variant = nts::g_last_variant;
  return 0;
}

int nts_aggregate_last_shape(int *vec, int *k, int *u, int *min_blocks, int *tiles) {
  if (vec)
    *vec = nts::g_last_vec;
  if (k)
    *k = nts::g_last_k;
  if (u)
    *u = nts::g_last_u;
  if (min_blocks)
    *min_blocks = nts::g_last_minb;
  if (tiles)
    *tiles = nts::g_last_tiles;
  return 0;
}

} // extern "C"
