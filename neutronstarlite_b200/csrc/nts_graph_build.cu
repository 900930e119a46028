// Chunk construction on the device: the arrays of nts_graph_host.cpp (CSC_segment_pinned per source partition,
// MirrorIndex, the whole-partition CSC; core/PartitionedGraph.hpp:105-143,295-420) built on the GPU, either from the
// reference's packed binary edge file ({u32 src, u32 dst}, dep/gemini/type.hpp:100-106), streamed in blocks so no
// process holds the edge list, or from edge arrays already on the device.
//
//   pass 1   degrees with multiplicity (raw, then clamped to >= 1) over all edges; any id >= V is an error
//   offsets  the reference's partitioner on the raw out-degree (nts::partition_offsets_from_out_degree), or given
//   pass 2   the owned edges (destination in [po[rank], po[rank+1])) compacted into 64-bit keys (dst_local, src)
//   dist     MirrorIndex = inclusive scan of "v is the source of an owned edge" shifted by one; the whole-partition
//            CSC = one sort of the pass-2 keys
//   chunks   edges bucketed by source partition, then per chunk one key sort (dst_local, src_local) -> CSC and
//            one key sort (src_local, dst_local) -> CSR.  Keys never exceed 62 bits for V < 2^31 and any P.
//
// Orders are the host builder's: CSC (dst, src) ascending, CSR (src, dst) ascending, duplicates kept.  Equal keys are
// identical edges, so the sorts need not be stable and the atomic compaction order does not show in any output.
// Weights are nts_norm_degree (core/ntsBaseOp.hpp:194-197) written with explicitly rounded intrinsics, so contraction
// or fast-math flags cannot change a bit.
//
// Device scratch beyond the returned arrays: two u64 key arrays (16 B per owned edge), CUB's temporary storage and, in
// the streaming passes only, two staging buffers capped at V records each (16 B per vertex), so the peak stays below
// 40 B per owned edge + 16 B per vertex.  The pinned host blocks are host memory.
#include <cub/cub.cuh>
#include <errno.h>
#include <stdarg.h>
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <vector>

#include "nts_common.cuh"

namespace nts {
// the reference's vertex-chunk partitioner over the raw out-degree (nts_graph_host.cpp)
int partition_offsets_from_out_degree(const uint32_t *out_degree_raw, uint64_t n_edges, uint32_t V, int P,
                                      uint32_t *partition_offset);
} // namespace nts

struct nts_graph_build {
  uint32_t V = 0;
  int P = 0, rank = 0, dist = 0;
  std::vector<uint32_t> po;             // [P+1]
  std::vector<uint64_t> chunk_start;    // [P+1], chunk i's edges at [chunk_start[i], chunk_start[i+1])
  uint64_t owned_edges = 0;
  uint32_t owned_mirrors = 0;
  uint64_t scratch_now = 0, scratch_peak = 0;
  double seconds[4] = {0, 0, 0, 0};     // degrees pass, owned-edge pass, chunks, distributed artefacts
  uint32_t *out_deg = nullptr, *in_deg = nullptr;       // [V], clamped
  uint32_t *col_off = nullptr;                          // P x [Vp+1]
  uint32_t *row_off = nullptr;                          // chunk i at po[i] + i, [Vi+1]
  uint8_t *source_active = nullptr;                     // chunk i at po[i], [Vi]
  uint32_t *row_indices = nullptr, *column_indices = nullptr;
  float *w_fwd = nullptr, *w_bwd = nullptr;             // [owned_edges]
  uint32_t *mirror_index = nullptr;                     // [V+1]
  uint32_t *whole_col = nullptr, *whole_rows = nullptr; // [Vp+1], [owned_edges]
  uint32_t Vp() const { return po[rank + 1] - po[rank]; }
};

namespace {

using u64 = unsigned long long;

const uint64_t kMaxStageRecords = 1ull << 22;
const int kThreads = 256;

inline int bitwidth(uint64_t x) { return x ? 64 - __builtin_clzll(x) : 0; }

inline unsigned grid_for(uint64_t n) {
  const uint64_t cap = (uint64_t)nts::sm_count() * 16;
  return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((n + kThreads - 1) / kThreads, cap));
}

__device__ __forceinline__ float norm_degree(uint32_t out_src, uint32_t in_dst) {
  return __fdiv_rn(1.0f, __fmul_rn(__double2float_rn(__dsqrt_rn((double)out_src)),
                                   __double2float_rn(__dsqrt_rn((double)in_dst))));
}

// edge i as 64-bit ids: packed {u32 src, u32 dst} records, or two arrays of int32 / int64 (negative -> huge -> >= V)
struct PackedEdges {
  const uint2 *e;
  __device__ __forceinline__ void get(uint64_t i, uint64_t &s, uint64_t &d) const {
    const uint2 r = e[i];
    s = r.x, d = r.y;
  }
};
template <class T> struct SplitEdges {
  const T *s, *d;
  __device__ __forceinline__ void get(uint64_t i, uint64_t &so, uint64_t &dd) const {
    so = (uint64_t)(int64_t)s[i], dd = (uint64_t)(int64_t)d[i];
  }
};

template <class Src> __global__ void degree_kernel(Src e, uint64_t n, uint32_t V, uint32_t *out, uint32_t *in, int *err) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t s, d;
    e.get(i, s, d);
    if (s >= V || d >= V) {
      *err = 1;
      continue;
    }
    atomicAdd(out + s, 1u);
    atomicAdd(in + d, 1u);
  }
}

// owned edges -> keys[pos] = (d - v0) << bv | s, pos from one warp-aggregated atomic; keys == nullptr only counts
template <class Src>
__global__ void owned_kernel(Src e, uint64_t n, uint32_t V, uint32_t v0, uint32_t v1, int bv, u64 *keys, u64 cap,
                             u64 *counter, int *err) {
  const unsigned lane = threadIdx.x & 31;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x - lane); base < n; base += stride) {
    const uint64_t i = base + lane;
    uint64_t s = 0, d = 0;
    bool keep = false;
    if (i < n) {
      e.get(i, s, d);
      if (s >= V || d >= V)
        *err = 1;
      else
        keep = d >= v0 && d < v1;
    }
    const unsigned mask = __ballot_sync(0xffffffffu, keep);
    if (!mask)
      continue;
    u64 first = 0;
    if (lane == __ffs(mask) - 1)
      first = atomicAdd(counter, (u64)__popc(mask));
    first = __shfl_sync(0xffffffffu, first, __ffs(mask) - 1);
    const u64 pos = first + __popc(mask & ((1u << lane) - 1));
    if (keep && keys && pos < cap)
      keys[pos] = ((u64)(d - v0) << bv) | s;
  }
}

__global__ void clamp_kernel(uint32_t *a, uint32_t n) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    a[i] = max(a[i], 1u);
}

// caller-supplied degrees: must already be clamped, >= 1 and < 2^32
template <class T> __global__ void take_degrees_kernel(const T *src, uint32_t *dst, uint32_t n, int *err) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const int64_t v = (int64_t)src[i];
    if (v < 1 || v > (int64_t)0xffffffffll)
      *err = 1;
    dst[i] = (uint32_t)v;
  }
}

__global__ void range_sum_kernel(const uint32_t *a, uint32_t n, u64 *sum) {
  u64 acc = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    acc += a[i];
  for (int o = 16; o; o >>= 1)
    acc += __shfl_down_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0 && acc)
    atomicAdd(sum, acc);
}

__device__ __forceinline__ int partition_of(const uint32_t *po, int P, uint32_t s) {
  int lo = 0, hi = P; // po[lo] <= s < po[lo+1]; empty partitions are skipped by the search
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (po[mid] <= s)
      lo = mid;
    else
      hi = mid;
  }
  return lo;
}

// chunk histogram (count != nullptr) or the bucket scatter (cursor != nullptr) of the pass-2 keys by source partition;
// the scatter re-keys an edge of chunk i as (dst_local << bs[i]) | (src - po[i])
__global__ void bucket_kernel(const u64 *keys, uint64_t n, int bv, const uint32_t *po, int P, const uint8_t *bs,
                              u64 *count, u64 *cursor, u64 *out) {
  const unsigned lane = threadIdx.x & 31;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const u64 vmask = (1ull << bv) - 1;
  for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x - lane); base < n; base += stride) {
    const uint64_t i = base + lane;
    const bool live = i < n;
    u64 k = 0;
    int c = -1;
    if (live) {
      k = keys[i];
      c = partition_of(po, P, (uint32_t)(k & vmask));
    }
    const unsigned peers = __match_any_sync(0xffffffffu, c);
    const int leader = __ffs(peers) - 1;
    u64 first = 0;
    if (live && lane == (unsigned)leader)
      first = atomicAdd(count ? count + c : cursor + c, (u64)__popc(peers));
    first = __shfl_sync(0xffffffffu, first, leader);
    if (live && out) {
      const u64 dl = k >> bv, s = k & vmask;
      out[first + __popc(peers & ((1u << lane) - 1))] = (dl << bs[c]) | (s - po[c]);
    }
  }
}

// off[0..nseg] of the sorted keys' segments (segment = key >> shift): off[s] = first position with segment >= s
__global__ void boundary_kernel(const u64 *keys, uint64_t n, int shift, uint32_t nseg, uint32_t *off) {
  for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t <= n; t += (uint64_t)gridDim.x * blockDim.x) {
    const int64_t prev = t == 0 ? -1 : (int64_t)(keys[t - 1] >> shift);
    const int64_t cur = t == n ? (int64_t)nseg : (int64_t)(keys[t] >> shift);
    for (int64_t s = prev + 1; s <= cur; s++)
      off[s] = (uint32_t)t;
  }
}

// CSC of one chunk from its sorted (dst_local, src_local) keys: source ids, forward weights, and the CSR keys
// (src_local, dst_local) for the second sort
__global__ void emit_csc_kernel(const u64 *keys, uint64_t n, int bs, int bd, uint32_t s0, uint32_t v0,
                                const uint32_t *out_deg, const uint32_t *in_deg, uint32_t *rows, float *w, u64 *csr_keys) {
  const u64 smask = (1ull << bs) - 1;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const u64 k = keys[i];
    const uint32_t sl = (uint32_t)(k & smask), dl = (uint32_t)(k >> bs);
    rows[i] = s0 + sl;
    w[i] = norm_degree(out_deg[s0 + sl], in_deg[v0 + dl]);
    csr_keys[i] = ((u64)sl << bd) | dl;
  }
}

__global__ void emit_csr_kernel(const u64 *keys, uint64_t n, int bd, uint32_t s0, uint32_t v0, const uint32_t *out_deg,
                                const uint32_t *in_deg, uint32_t *cols, float *w) {
  const u64 dmask = (1ull << bd) - 1;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const u64 k = keys[i];
    const uint32_t dl = (uint32_t)(k & dmask), sl = (uint32_t)(k >> bd);
    cols[i] = v0 + dl;
    w[i] = norm_degree(out_deg[s0 + sl], in_deg[v0 + dl]);
  }
}

__global__ void source_active_kernel(const uint32_t *row_off, uint32_t n, uint8_t *active) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    active[i] = row_off[i + 1] > row_off[i] ? 1 : 0;
}

__global__ void mark_sources_kernel(const u64 *keys, uint64_t n, int bv, uint32_t *flags) {
  const u64 vmask = (1ull << bv) - 1;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    flags[(keys[i] & vmask) + 1] = 1;
}

__global__ void low_bits_kernel(const u64 *keys, uint64_t n, int bv, uint32_t *out) {
  const u64 vmask = (1ull << bv) - 1;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    out[i] = (uint32_t)(keys[i] & vmask);
}

// ---- inclusive scan of u32 (MirrorIndex): tile sums, scan of the sums (recursively), tile scans ------------------
const int kScanThreads = 512, kScanItems = 8, kScanTile = kScanThreads * kScanItems;

__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t *total) {
  __shared__ uint32_t warp_sums[kScanThreads / 32];
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t inc = v;
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= (unsigned)o)
      inc += t;
  }
  if (lane == 31)
    warp_sums[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = lane < kScanThreads / 32 ? warp_sums[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= (unsigned)o)
        w += t;
    }
    if (lane < kScanThreads / 32)
      warp_sums[lane] = w;
  }
  __syncthreads();
  const uint32_t before = (warp ? warp_sums[warp - 1] : 0) + inc - v;
  if (total)
    *total = warp_sums[kScanThreads / 32 - 1];
  return before;
}

__global__ void __launch_bounds__(kScanThreads) tile_sum_kernel(const uint32_t *x, uint64_t n, uint32_t *sums) {
  const uint64_t base = (uint64_t)blockIdx.x * kScanTile + (uint64_t)threadIdx.x * kScanItems;
  uint32_t s = 0;
  for (int k = 0; k < kScanItems; k++)
    s += base + k < n ? x[base + k] : 0;
  uint32_t total;
  block_exclusive_scan(s, &total);
  if (threadIdx.x == 0)
    sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kScanThreads) tile_scan_kernel(uint32_t *x, uint64_t n, const uint32_t *sums_inc) {
  const uint64_t base = (uint64_t)blockIdx.x * kScanTile + (uint64_t)threadIdx.x * kScanItems;
  uint32_t v[kScanItems], s = 0;
  for (int k = 0; k < kScanItems; k++) {
    v[k] = base + k < n ? x[base + k] : 0;
    s += v[k];
  }
  uint32_t run = block_exclusive_scan(s, nullptr) + (blockIdx.x ? sums_inc[blockIdx.x - 1] : 0);
  for (int k = 0; k < kScanItems; k++) {
    run += v[k];
    if (base + k < n)
      x[base + k] = run;
  }
}

// ---- host side ------------------------------------------------------------------------------------------------------
int err_msg(const char *fmt, ...) __attribute__((format(printf, 1, 2)));
int err_msg(const char *fmt, ...) {
  char buf[400];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  return nts::fail(-1, buf, __FILE__, __LINE__);
}

// scratch allocations, tracked so the builder can report its peak
struct Scratch {
  nts_graph_build *b;
  std::vector<void *> live;
  std::vector<size_t> sizes;
  explicit Scratch(nts_graph_build *b_) : b(b_) {}
  template <class T> cudaError_t alloc(T **p, size_t count) {
    const size_t bytes = std::max<size_t>(count * sizeof(T), 16);
    cudaError_t e = cudaMalloc(reinterpret_cast<void **>(p), bytes);
    if (e != cudaSuccess)
      return e;
    live.push_back(*p), sizes.push_back(bytes);
    b->scratch_now += bytes;
    b->scratch_peak = std::max(b->scratch_peak, b->scratch_now);
    return cudaSuccess;
  }
  void release(void *p) {
    for (size_t k = 0; k < live.size(); k++)
      if (live[k] == p) {
        cudaFree(p);
        b->scratch_now -= sizes[k];
        live.erase(live.begin() + k), sizes.erase(sizes.begin() + k);
        return;
      }
  }
  ~Scratch() {
    for (void *p : live)
      cudaFree(p);
    b->scratch_now = 0;
  }
};

int scan_inclusive(uint32_t *x, uint64_t n, Scratch &sc, cudaStream_t st) {
  if (n == 0)
    return 0;
  const uint64_t tiles = (n + kScanTile - 1) / kScanTile;
  uint32_t *sums = nullptr;
  if (tiles > 1) {
    NTS_CUDA_OK(sc.alloc(&sums, tiles));
    tile_sum_kernel<<<(unsigned)tiles, kScanThreads, 0, st>>>(x, n, sums);
    NTS_LAUNCH_CHECK();
    if (int rc = scan_inclusive(sums, tiles, sc, st))
      return rc;
  }
  tile_scan_kernel<<<(unsigned)tiles, kScanThreads, 0, st>>>(x, n, sums);
  NTS_LAUNCH_CHECK();
  if (sums) {
    NTS_CUDA_OK(cudaStreamSynchronize(st));
    sc.release(sums);
  }
  return 0;
}

double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// streams a packed edge file through two pinned host blocks of block_edges records (pread) and two device staging
// buffers (cudaMemcpyAsync on a copy stream): the read of a block overlaps the kernels on the previous one
struct FileStream {
  int fd = -1;
  uint64_t n = 0, block = 0, stage = 0;
  uint2 *pinned[2] = {nullptr, nullptr};
  uint2 *dev[2] = {nullptr, nullptr};
  cudaStream_t copy = nullptr;
  cudaEvent_t pinned_free[2] = {}, stage_free[2] = {}, copied[2] = {};
  cudaStream_t st = nullptr;
  Scratch *sc = nullptr;

  ~FileStream() {
    if (copy)
      cudaStreamSynchronize(copy);
    if (st)
      cudaStreamSynchronize(st);
    for (int k = 0; k < 2; k++) {
      if (pinned[k])
        cudaFreeHost(pinned[k]);
      if (dev[k])
        sc->release(dev[k]);
      if (pinned_free[k])
        cudaEventDestroy(pinned_free[k]);
      if (stage_free[k])
        cudaEventDestroy(stage_free[k]);
      if (copied[k])
        cudaEventDestroy(copied[k]);
    }
    if (copy)
      cudaStreamDestroy(copy);
    if (fd >= 0)
      close(fd);
  }

  int open_file(const char *path, uint64_t block_edges, uint32_t V) {
    fd = open(path, O_RDONLY);
    if (fd < 0)
      return err_msg("cannot open edge file '%s': %s", path, strerror(errno));
    struct stat stt;
    if (fstat(fd, &stt) != 0)
      return err_msg("cannot stat edge file '%s': %s", path, strerror(errno));
    if (stt.st_size % 8 != 0)
      return err_msg("edge file '%s' has %lld bytes, not a multiple of 8 ({u32 src, u32 dst} records)", path,
                     (long long)stt.st_size);
    n = (uint64_t)stt.st_size / 8;
    block = std::min<uint64_t>(block_edges, std::max<uint64_t>(n, 1));
    stage = std::min<uint64_t>(std::min<uint64_t>(block, kMaxStageRecords), V);
    return 0;
  }

  int setup(Scratch &s, cudaStream_t stream) {
    sc = &s;
    st = stream;
    if (n == 0)
      return 0;
    NTS_CUDA_OK(cudaStreamCreateWithFlags(&copy, cudaStreamNonBlocking));
    for (int k = 0; k < 2; k++) {
      NTS_CUDA_OK(cudaHostAlloc(reinterpret_cast<void **>(&pinned[k]), block * 8, cudaHostAllocDefault));
      NTS_CUDA_OK(s.alloc(&dev[k], stage));
      NTS_CUDA_OK(cudaEventCreateWithFlags(&pinned_free[k], cudaEventDisableTiming));
      NTS_CUDA_OK(cudaEventCreateWithFlags(&stage_free[k], cudaEventDisableTiming));
      NTS_CUDA_OK(cudaEventCreateWithFlags(&copied[k], cudaEventDisableTiming));
    }
    return 0;
  }

  // one pass over the file: launch(const uint2 *edges, uint64_t count) on st per staged piece
  template <class F> int pass(F launch) {
    uint64_t piece = 0;
    for (uint64_t b = 0, k = 0; b < n; b += block, k++) {
      const uint64_t cnt = std::min(block, n - b);
      uint2 *buf = pinned[k & 1];
      NTS_CUDA_OK(cudaEventSynchronize(pinned_free[k & 1]));
      char *dst = reinterpret_cast<char *>(buf);
      const size_t want = cnt * 8;
      size_t done = 0;
      while (done < want) {
        const ssize_t r = pread(fd, dst + done, want - done, (off_t)(b * 8 + done));
        if (r < 0 && errno == EINTR)
          continue;
        if (r <= 0)
          return err_msg("short read of the edge file at byte %llu: %s", (unsigned long long)(b * 8 + done),
                         r < 0 ? strerror(errno) : "end of file");
        done += (size_t)r;
      }
      for (uint64_t o = 0; o < cnt; o += stage, piece++) {
        const uint64_t m = std::min(stage, cnt - o);
        const int j = (int)(piece & 1);
        NTS_CUDA_OK(cudaStreamWaitEvent(copy, stage_free[j], 0));
        NTS_CUDA_OK(cudaMemcpyAsync(dev[j], buf + o, m * 8, cudaMemcpyHostToDevice, copy));
        NTS_CUDA_OK(cudaEventRecord(copied[j], copy));
        NTS_CUDA_OK(cudaStreamWaitEvent(st, copied[j], 0));
        if (int rc = launch((const uint2 *)dev[j], m))
          return rc;
        NTS_CUDA_OK(cudaEventRecord(stage_free[j], st));
      }
      NTS_CUDA_OK(cudaEventRecord(pinned_free[k & 1], copy));
    }
    NTS_CUDA_OK(cudaStreamSynchronize(st));
    return 0;
  }
};

int check_common(uint32_t V, int P, int rank, const nts_vid_t *po, int flags) {
  if (V == 0 || V >= (1u << 31))
    return err_msg("vertices = %u: must be in [1, 2^31) (ids live in int32 device tensors)", V);
  if (P < 1)
    return err_msg("partitions = %d: must be >= 1", P);
  if (rank < 0 || rank >= P)
    return err_msg("rank %d out of range for %d partitions", rank, P);
  if (flags & ~NTS_GRAPH_BUILD_DIST)
    return err_msg("unknown flags 0x%x", flags);
  if (po) {
    if (po[0] != 0 || po[P] != V)
      return err_msg("partition_offset must run from 0 to V = %u (got %u .. %u)", V, po[0], po[P]);
    for (int i = 0; i < P; i++)
      if (po[i + 1] < po[i])
        return err_msg("partition_offset decreases at %d", i);
  }
  return 0;
}

int read_flag(int *d_err, cudaStream_t st, int *flag) {
  NTS_CUDA_OK(cudaMemcpyAsync(flag, d_err, sizeof(int), cudaMemcpyDeviceToHost, st));
  NTS_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

template <class T> int sort_keys(cub::DoubleBuffer<T> &db, uint64_t n, int end_bit, void *tmp, size_t tmp_bytes,
                                 cudaStream_t st) {
  if (n < 2 || end_bit == 0)
    return 0;
  NTS_CUDA_OK(cub::DeviceRadixSort::SortKeys(tmp, tmp_bytes, db, (int64_t)n, 0, end_bit, st));
  return 0;
}

// everything after the degrees and the partition offsets: pass 2 (owned(keys, cap, counter) writes the pass-2 keys),
// the distributed artefacts and the chunks
template <class Owned> int build_rest(nts_graph_build *b, Scratch &sc, cudaStream_t st, Owned owned) {
  const uint32_t V = b->V, v0 = b->po[b->rank], v1 = b->po[b->rank + 1], Vp = v1 - v0;
  const int P = b->P, bv = bitwidth(V - 1), bd = bitwidth(Vp ? Vp - 1 : 0);
  const uint64_t E = b->owned_edges;
  double t0 = now_s();

  u64 *A = nullptr, *B = nullptr, *counter = nullptr, *cursor = nullptr;
  int *d_err = nullptr;
  uint32_t *d_po = nullptr;
  uint8_t *d_bs = nullptr;
  NTS_CUDA_OK(sc.alloc(&A, E));
  NTS_CUDA_OK(sc.alloc(&counter, P + 1));
  NTS_CUDA_OK(sc.alloc(&d_err, 1));
  NTS_CUDA_OK(cudaMemsetAsync(counter, 0, sizeof(u64) * (P + 1), st));
  NTS_CUDA_OK(cudaMemsetAsync(d_err, 0, sizeof(int), st));
  if (int rc = owned(A, (u64)E, counter + P, d_err))
    return rc;
  u64 got = 0;
  int flag = 0;
  NTS_CUDA_OK(cudaMemcpyAsync(&got, counter + P, sizeof(u64), cudaMemcpyDeviceToHost, st));
  if (int rc = read_flag(d_err, st, &flag))
    return rc;
  if (flag)
    return err_msg("an edge has a vertex id >= V = %u", V);
  if (got != E)
    return err_msg("the owned-edge pass found %llu edges, the degrees promise %llu (did the input change?)", got,
                   (u64)E);
  b->seconds[1] = now_s() - t0;

  // chunk sizes
  std::vector<uint8_t> bs(P);
  for (int i = 0; i < P; i++) {
    const uint32_t Vi = b->po[i + 1] - b->po[i];
    bs[i] = (uint8_t)bitwidth(Vi ? Vi - 1 : 0);
  }
  NTS_CUDA_OK(sc.alloc(&d_po, P + 1));
  NTS_CUDA_OK(sc.alloc(&d_bs, P));
  NTS_CUDA_OK(cudaMemcpyAsync(d_po, b->po.data(), sizeof(uint32_t) * (P + 1), cudaMemcpyHostToDevice, st));
  NTS_CUDA_OK(cudaMemcpyAsync(d_bs, bs.data(), P, cudaMemcpyHostToDevice, st));
  std::vector<u64> counts(P, 0);
  if (E) {
    bucket_kernel<<<grid_for(E), kThreads, 0, st>>>(A, E, bv, d_po, P, d_bs, counter, nullptr, nullptr);
    NTS_LAUNCH_CHECK();
    NTS_CUDA_OK(cudaMemcpyAsync(counts.data(), counter, sizeof(u64) * P, cudaMemcpyDeviceToHost, st));
    NTS_CUDA_OK(cudaStreamSynchronize(st));
  }
  b->chunk_start.assign(P + 1, 0);
  for (int i = 0; i < P; i++)
    b->chunk_start[i + 1] = b->chunk_start[i] + counts[i];

  // returned arrays
  NTS_CUDA_OK(cudaMalloc(&b->col_off, sizeof(uint32_t) * (size_t)P * (Vp + 1)));
  NTS_CUDA_OK(cudaMalloc(&b->row_off, sizeof(uint32_t) * ((size_t)V + P)));
  NTS_CUDA_OK(cudaMalloc(&b->source_active, V));
  NTS_CUDA_OK(cudaMalloc(&b->row_indices, sizeof(uint32_t) * std::max<uint64_t>(E, 1)));
  NTS_CUDA_OK(cudaMalloc(&b->column_indices, sizeof(uint32_t) * std::max<uint64_t>(E, 1)));
  NTS_CUDA_OK(cudaMalloc(&b->w_fwd, sizeof(float) * std::max<uint64_t>(E, 1)));
  NTS_CUDA_OK(cudaMalloc(&b->w_bwd, sizeof(float) * std::max<uint64_t>(E, 1)));

  NTS_CUDA_OK(sc.alloc(&B, E));
  void *tmp = nullptr;
  size_t tmp_bytes = 0;
  if (E >= 2) {
    cub::DoubleBuffer<u64> q(A, B);
    NTS_CUDA_OK(cub::DeviceRadixSort::SortKeys(nullptr, tmp_bytes, q, (int64_t)E, 0, 64, st));
    NTS_CUDA_OK(sc.alloc(reinterpret_cast<char **>(&tmp), tmp_bytes));
  }

  u64 *cur = A, *alt = B; // cur holds the pass-2 keys
  if (b->dist) {
    t0 = now_s();
    NTS_CUDA_OK(cudaMalloc(&b->mirror_index, sizeof(uint32_t) * ((size_t)V + 1)));
    NTS_CUDA_OK(cudaMalloc(&b->whole_col, sizeof(uint32_t) * ((size_t)Vp + 1)));
    NTS_CUDA_OK(cudaMalloc(&b->whole_rows, sizeof(uint32_t) * std::max<uint64_t>(E, 1)));
    NTS_CUDA_OK(cudaMemsetAsync(b->mirror_index, 0, sizeof(uint32_t) * ((size_t)V + 1), st));
    if (E) {
      mark_sources_kernel<<<grid_for(E), kThreads, 0, st>>>(cur, E, bv, b->mirror_index);
      NTS_LAUNCH_CHECK();
    }
    if (int rc = scan_inclusive(b->mirror_index, (uint64_t)V + 1, sc, st))
      return rc;
    NTS_CUDA_OK(cudaMemcpyAsync(&b->owned_mirrors, b->mirror_index + V, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    cub::DoubleBuffer<u64> q(cur, alt);
    if (int rc = sort_keys(q, E, bv + bd, tmp, tmp_bytes, st))
      return rc;
    cur = q.Current(), alt = q.Alternate();
    if (E) {
      low_bits_kernel<<<grid_for(E), kThreads, 0, st>>>(cur, E, bv, b->whole_rows);
      NTS_LAUNCH_CHECK();
      boundary_kernel<<<grid_for(E + 1), kThreads, 0, st>>>(cur, E, bv, Vp, b->whole_col);
      NTS_LAUNCH_CHECK();
    } else {
      NTS_CUDA_OK(cudaMemsetAsync(b->whole_col, 0, sizeof(uint32_t) * ((size_t)Vp + 1), st));
    }
    NTS_CUDA_OK(cudaStreamSynchronize(st));
    b->seconds[3] = now_s() - t0;
  }

  t0 = now_s();
  if (E) {
    NTS_CUDA_OK(cudaMemcpyAsync(counter, b->chunk_start.data(), sizeof(u64) * P, cudaMemcpyHostToDevice, st));
    cursor = counter;
    bucket_kernel<<<grid_for(E), kThreads, 0, st>>>(cur, E, bv, d_po, P, d_bs, nullptr, cursor, alt);
    NTS_LAUNCH_CHECK();
    std::swap(cur, alt);
  }
  for (int i = 0; i < P; i++) {
    const uint32_t s0 = b->po[i], Vi = b->po[i + 1] - s0;
    const uint64_t e0 = b->chunk_start[i], Ei = counts[i];
    uint32_t *col = b->col_off + (size_t)i * (Vp + 1), *ro = b->row_off + s0 + i;
    if (Ei == 0) {
      NTS_CUDA_OK(cudaMemsetAsync(col, 0, sizeof(uint32_t) * ((size_t)Vp + 1), st));
      NTS_CUDA_OK(cudaMemsetAsync(ro, 0, sizeof(uint32_t) * ((size_t)Vi + 1), st));
      if (Vi)
        NTS_CUDA_OK(cudaMemsetAsync(b->source_active + s0, 0, Vi, st));
      continue;
    }
    cub::DoubleBuffer<u64> csc(cur + e0, alt + e0);
    if (int rc = sort_keys(csc, Ei, bs[i] + bd, tmp, tmp_bytes, st))
      return rc;
    emit_csc_kernel<<<grid_for(Ei), kThreads, 0, st>>>(csc.Current(), Ei, bs[i], bd, s0, v0, b->out_deg, b->in_deg,
                                                       b->row_indices + e0, b->w_fwd + e0, csc.Alternate());
    NTS_LAUNCH_CHECK();
    boundary_kernel<<<grid_for(Ei + 1), kThreads, 0, st>>>(csc.Current(), Ei, bs[i], Vp, col);
    NTS_LAUNCH_CHECK();
    cub::DoubleBuffer<u64> csr(csc.Alternate(), csc.Current());
    if (int rc = sort_keys(csr, Ei, bs[i] + bd, tmp, tmp_bytes, st))
      return rc;
    emit_csr_kernel<<<grid_for(Ei), kThreads, 0, st>>>(csr.Current(), Ei, bd, s0, v0, b->out_deg, b->in_deg,
                                                       b->column_indices + e0, b->w_bwd + e0);
    NTS_LAUNCH_CHECK();
    boundary_kernel<<<grid_for(Ei + 1), kThreads, 0, st>>>(csr.Current(), Ei, bd, Vi, ro);
    NTS_LAUNCH_CHECK();
    source_active_kernel<<<grid_for(Vi), kThreads, 0, st>>>(ro, Vi, b->source_active + s0);
    NTS_LAUNCH_CHECK();
  }
  NTS_CUDA_OK(cudaStreamSynchronize(st));
  b->seconds[2] = now_s() - t0;
  return 0;
}

int finish_offsets(nts_graph_build *b, const nts_vid_t *po, uint64_t n_edges, const uint32_t *raw_out_dev,
                   cudaStream_t st) {
  b->po.assign(b->P + 1, 0);
  if (po) {
    std::copy(po, po + b->P + 1, b->po.begin());
    return 0;
  }
  std::vector<uint32_t> raw(b->V);
  NTS_CUDA_OK(cudaMemcpyAsync(raw.data(), raw_out_dev, sizeof(uint32_t) * b->V, cudaMemcpyDeviceToHost, st));
  NTS_CUDA_OK(cudaStreamSynchronize(st));
  if (nts::partition_offsets_from_out_degree(raw.data(), n_edges, b->V, b->P, b->po.data()) != 0)
    return err_msg("partitioner failed for V = %u, P = %d", b->V, b->P);
  return 0;
}

int check_owned(nts_graph_build *b) {
  if (b->owned_edges >= (1ull << 31))
    return err_msg("rank %d owns %llu edges: at most 2^31 - 1 per rank (edge_size is an int)", b->rank,
                   (u64)b->owned_edges);
  return 0;
}

int build_from_file(nts_graph_build *b, const char *path, const nts_vid_t *po, uint64_t block_edges,
                    cudaStream_t st) {
  Scratch sc(b);
  FileStream fs;
  if (int rc = fs.open_file(path, block_edges, b->V))
    return rc;
  const uint32_t V = b->V;
  int *d_err = nullptr;
  u64 *d_sum = nullptr;
  NTS_CUDA_OK(cudaMalloc(&b->out_deg, sizeof(uint32_t) * V));
  NTS_CUDA_OK(cudaMalloc(&b->in_deg, sizeof(uint32_t) * V));
  NTS_CUDA_OK(sc.alloc(&d_err, 1));
  NTS_CUDA_OK(sc.alloc(&d_sum, 1));
  NTS_CUDA_OK(cudaMemsetAsync(b->out_deg, 0, sizeof(uint32_t) * V, st));
  NTS_CUDA_OK(cudaMemsetAsync(b->in_deg, 0, sizeof(uint32_t) * V, st));
  NTS_CUDA_OK(cudaMemsetAsync(d_err, 0, sizeof(int), st));
  NTS_CUDA_OK(cudaMemsetAsync(d_sum, 0, sizeof(u64), st));
  if (int rc = fs.setup(sc, st))
    return rc;

  double t0 = now_s();
  int rc = fs.pass([&](const uint2 *e, uint64_t m) -> int {
    degree_kernel<<<grid_for(m), kThreads, 0, st>>>(PackedEdges{e}, m, V, b->out_deg, b->in_deg, d_err);
    NTS_LAUNCH_CHECK();
    return 0;
  });
  if (rc)
    return rc;
  int flag = 0;
  if ((rc = read_flag(d_err, st, &flag)))
    return rc;
  if (flag)
    return err_msg("edge file '%s' has a vertex id >= V = %u", path, V);
  if ((rc = finish_offsets(b, po, fs.n, b->out_deg, st)))
    return rc;
  const uint32_t v0 = b->po[b->rank], v1 = b->po[b->rank + 1];
  if (v1 > v0) {
    range_sum_kernel<<<grid_for(v1 - v0), kThreads, 0, st>>>(b->in_deg + v0, v1 - v0, d_sum);
    NTS_LAUNCH_CHECK();
  }
  clamp_kernel<<<grid_for(V), kThreads, 0, st>>>(b->out_deg, V);
  NTS_LAUNCH_CHECK();
  clamp_kernel<<<grid_for(V), kThreads, 0, st>>>(b->in_deg, V);
  NTS_LAUNCH_CHECK();
  u64 owned = 0;
  NTS_CUDA_OK(cudaMemcpyAsync(&owned, d_sum, sizeof(u64), cudaMemcpyDeviceToHost, st));
  NTS_CUDA_OK(cudaStreamSynchronize(st));
  b->owned_edges = owned;
  b->seconds[0] = now_s() - t0;
  if ((rc = check_owned(b)))
    return rc;
  const int bv = bitwidth(V - 1);
  return build_rest(b, sc, st, [&](u64 *keys, u64 cap, u64 *counter, int *err) -> int {
    return fs.pass([&](const uint2 *e, uint64_t m) -> int {
      owned_kernel<<<grid_for(m), kThreads, 0, st>>>(PackedEdges{e}, m, V, v0, v1, bv, keys, cap, counter, err);
      NTS_LAUNCH_CHECK();
      return 0;
    });
  });
}

template <class T>
int build_from_device(nts_graph_build *b, const T *src, const T *dst, uint64_t n_edges, const nts_vid_t *po,
                      const T *out_degree, const T *in_degree, cudaStream_t st) {
  Scratch sc(b);
  const uint32_t V = b->V;
  const SplitEdges<T> edges{src, dst};
  int *d_err = nullptr;
  u64 *d_count = nullptr;
  NTS_CUDA_OK(cudaMalloc(&b->out_deg, sizeof(uint32_t) * V));
  NTS_CUDA_OK(cudaMalloc(&b->in_deg, sizeof(uint32_t) * V));
  NTS_CUDA_OK(sc.alloc(&d_err, 1));
  NTS_CUDA_OK(sc.alloc(&d_count, 1));
  NTS_CUDA_OK(cudaMemsetAsync(d_err, 0, sizeof(int), st));
  NTS_CUDA_OK(cudaMemsetAsync(d_count, 0, sizeof(u64), st));
  double t0 = now_s();
  int rc = 0, flag = 0;
  if (out_degree) {
    take_degrees_kernel<<<grid_for(V), kThreads, 0, st>>>(out_degree, b->out_deg, V, d_err);
    NTS_LAUNCH_CHECK();
    take_degrees_kernel<<<grid_for(V), kThreads, 0, st>>>(in_degree, b->in_deg, V, d_err);
    NTS_LAUNCH_CHECK();
    if ((rc = read_flag(d_err, st, &flag)))
      return rc;
    if (flag)
      return err_msg("given degrees must lie in [1, 2^32) (clamped degrees with multiplicity)");
  } else {
    NTS_CUDA_OK(cudaMemsetAsync(b->out_deg, 0, sizeof(uint32_t) * V, st));
    NTS_CUDA_OK(cudaMemsetAsync(b->in_deg, 0, sizeof(uint32_t) * V, st));
    if (n_edges) {
      degree_kernel<<<grid_for(n_edges), kThreads, 0, st>>>(edges, n_edges, V, b->out_deg, b->in_deg, d_err);
      NTS_LAUNCH_CHECK();
    }
    if ((rc = read_flag(d_err, st, &flag)))
      return rc;
    if (flag)
      return err_msg("an edge has a vertex id >= V = %u", V);
  }
  if ((rc = finish_offsets(b, po, n_edges, b->out_deg, st)))
    return rc;
  if (!out_degree) {
    clamp_kernel<<<grid_for(V), kThreads, 0, st>>>(b->out_deg, V);
    NTS_LAUNCH_CHECK();
    clamp_kernel<<<grid_for(V), kThreads, 0, st>>>(b->in_deg, V);
    NTS_LAUNCH_CHECK();
  }
  const uint32_t v0 = b->po[b->rank], v1 = b->po[b->rank + 1];
  const int bv = bitwidth(V - 1);
  if (n_edges) {
    owned_kernel<<<grid_for(n_edges), kThreads, 0, st>>>(edges, n_edges, V, v0, v1, bv, (u64 *)nullptr, 0, d_count,
                                                         d_err);
    NTS_LAUNCH_CHECK();
  }
  u64 owned = 0;
  NTS_CUDA_OK(cudaMemcpyAsync(&owned, d_count, sizeof(u64), cudaMemcpyDeviceToHost, st));
  if ((rc = read_flag(d_err, st, &flag)))
    return rc;
  if (flag)
    return err_msg("an edge has a vertex id >= V = %u", V);
  b->owned_edges = owned;
  b->seconds[0] = now_s() - t0;
  if ((rc = check_owned(b)))
    return rc;
  return build_rest(b, sc, st, [&](u64 *keys, u64 cap, u64 *counter, int *err) -> int {
    if (n_edges) {
      owned_kernel<<<grid_for(n_edges), kThreads, 0, st>>>(edges, n_edges, V, v0, v1, bv, keys, cap, counter, err);
      NTS_LAUNCH_CHECK();
    }
    return 0;
  });
}

nts_graph_build *finish(nts_graph_build *b, int rc) {
  if (rc == 0)
    return b;
  nts_graph_build_destroy(b);
  return nullptr;
}

} // namespace

extern "C" {

nts_graph_build *nts_graph_build_from_file(const char *path, nts_vid_t V, int P, int rank,
                                           const nts_vid_t *partition_offset, uint64_t block_edges, int flags,
                                           void *stream) {
  if (!path) {
    err_msg("edge file path is NULL");
    return nullptr;
  }
  if (block_edges == 0) {
    err_msg("block_edges must be >= 1");
    return nullptr;
  }
  if (check_common(V, P, rank, partition_offset, flags))
    return nullptr;
  nts_graph_build *b = new nts_graph_build;
  b->V = V, b->P = P, b->rank = rank, b->dist = flags & NTS_GRAPH_BUILD_DIST;
  return finish(b, build_from_file(b, path, partition_offset, block_edges, nts::as_stream(stream)));
}

nts_graph_build *nts_graph_build_from_device(const void *src, const void *dst, int index_dtype, uint64_t n_edges,
                                             nts_vid_t V, int P, int rank, const nts_vid_t *partition_offset,
                                             const void *out_degree, const void *in_degree, int flags, void *stream) {
  if (index_dtype != NTS_INDEX_I32 && index_dtype != NTS_INDEX_I64) {
    err_msg("index_dtype %d: must be NTS_INDEX_I32 or NTS_INDEX_I64", index_dtype);
    return nullptr;
  }
  if (n_edges && (!src || !dst)) {
    err_msg("src / dst are NULL for %llu edges", (unsigned long long)n_edges);
    return nullptr;
  }
  if (!out_degree != !in_degree) {
    err_msg("give both degree arrays or neither");
    return nullptr;
  }
  if (out_degree && !partition_offset && P > 1) {
    err_msg("partition_offset is required with given degrees and partitions > 1 (the partitioner needs the raw "
            "out-degree)");
    return nullptr;
  }
  if (check_common(V, P, rank, partition_offset, flags))
    return nullptr;
  nts_graph_build *b = new nts_graph_build;
  b->V = V, b->P = P, b->rank = rank, b->dist = flags & NTS_GRAPH_BUILD_DIST;
  const cudaStream_t st = nts::as_stream(stream);
  int rc;
  if (index_dtype == NTS_INDEX_I32)
    rc = build_from_device(b, (const int32_t *)src, (const int32_t *)dst, n_edges, partition_offset,
                           (const int32_t *)out_degree, (const int32_t *)in_degree, st);
  else
    rc = build_from_device(b, (const int64_t *)src, (const int64_t *)dst, n_edges, partition_offset,
                           (const int64_t *)out_degree, (const int64_t *)in_degree, st);
  return finish(b, rc);
}

int nts_graph_build_info(const nts_graph_build *b, nts_vid_t *partition_offset, uint64_t *chunk_edges,
                         nts_vid_t *owned_mirrors, uint64_t *scratch_peak_bytes, double *pass_seconds) {
  NTS_ARG_CHECK(b, "graph build handle is NULL");
  if (partition_offset)
    std::copy(b->po.begin(), b->po.end(), partition_offset);
  if (chunk_edges)
    for (int i = 0; i < b->P; i++)
      chunk_edges[i] = b->chunk_start[i + 1] - b->chunk_start[i];
  if (owned_mirrors)
    *owned_mirrors = b->owned_mirrors;
  if (scratch_peak_bytes)
    *scratch_peak_bytes = b->scratch_peak;
  if (pass_seconds)
    std::copy(b->seconds, b->seconds + 4, pass_seconds);
  return 0;
}

static int copy_out(void *dst, const void *src, size_t bytes, cudaStream_t st) {
  if (dst && bytes)
    NTS_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st));
  return 0;
}

int nts_graph_build_export_chunk(const nts_graph_build *b, int i, nts_vid_t *column_offset, nts_vid_t *row_indices,
                                 float *edge_weight_forward, nts_vid_t *row_offset, nts_vid_t *column_indices,
                                 float *edge_weight_backward, unsigned char *source_active, void *stream) {
  NTS_ARG_CHECK(b, "graph build handle is NULL");
  NTS_ARG_CHECK(i >= 0 && i < b->P, "chunk index out of range");
  const cudaStream_t st = nts::as_stream(stream);
  const uint32_t Vp = b->Vp(), s0 = b->po[i], Vi = b->po[i + 1] - s0;
  const uint64_t e0 = b->chunk_start[i], Ei = b->chunk_start[i + 1] - e0;
  int rc = 0;
  (void)((rc = copy_out(column_offset, b->col_off + (size_t)i * (Vp + 1), 4 * ((size_t)Vp + 1), st)) ||
         (rc = copy_out(row_indices, b->row_indices + e0, 4 * Ei, st)) ||
         (rc = copy_out(edge_weight_forward, b->w_fwd + e0, 4 * Ei, st)) ||
         (rc = copy_out(row_offset, b->row_off + s0 + i, 4 * ((size_t)Vi + 1), st)) ||
         (rc = copy_out(column_indices, b->column_indices + e0, 4 * Ei, st)) ||
         (rc = copy_out(edge_weight_backward, b->w_bwd + e0, 4 * Ei, st)) ||
         (rc = copy_out(source_active, b->source_active + s0, Vi, st)));
  return rc;
}

int nts_graph_build_export_dist(const nts_graph_build *b, nts_vid_t *mirror_index, nts_vid_t *column_offset,
                                nts_vid_t *row_indices, void *stream) {
  NTS_ARG_CHECK(b, "graph build handle is NULL");
  NTS_ARG_CHECK(b->dist, "the graph was built without NTS_GRAPH_BUILD_DIST");
  const cudaStream_t st = nts::as_stream(stream);
  int rc = 0;
  (void)((rc = copy_out(mirror_index, b->mirror_index, 4 * ((size_t)b->V + 1), st)) ||
         (rc = copy_out(column_offset, b->whole_col, 4 * ((size_t)b->Vp() + 1), st)) ||
         (rc = copy_out(row_indices, b->whole_rows, 4 * b->owned_edges, st)));
  return rc;
}

int nts_graph_build_export_degrees(const nts_graph_build *b, nts_vid_t *out_degree, nts_vid_t *in_degree,
                                   void *stream) {
  NTS_ARG_CHECK(b, "graph build handle is NULL");
  const cudaStream_t st = nts::as_stream(stream);
  int rc = 0;
  (void)((rc = copy_out(out_degree, b->out_deg, 4 * (size_t)b->V, st)) ||
         (rc = copy_out(in_degree, b->in_deg, 4 * (size_t)b->V, st)));
  return rc;
}

int nts_graph_build_destroy(nts_graph_build *b) {
  if (!b)
    return 0;
  for (void *p : {(void *)b->out_deg, (void *)b->in_deg, (void *)b->col_off, (void *)b->row_off,
                  (void *)b->source_active, (void *)b->row_indices, (void *)b->column_indices, (void *)b->w_fwd,
                  (void *)b->w_bwd, (void *)b->mirror_index, (void *)b->whole_col, (void *)b->whole_rows})
    if (p)
      cudaFree(p);
  delete b;
  return 0;
}

} // extern "C"
