// nts_exchange: the data plane of the device-resident partition-boundary exchange, in C++ behind the C ABI.
//
// Replaces the GPU drivers of the reference engine - Graph::sync_compute_decoupled (forward, core/graph.hpp:3639-3719)
// and Graph::compute_sync_decoupled (backward, :3455-3622) - and the host-staged NtsGraphCommunicator they drive
// (comm/network.cpp:159-844).  Peer-memory ("p2p") transport, PUSH model, pipelined per source partition like the
// reference's ring (aggregate chunk (p+s) while chunk (p+s+1) is in flight, core/graph.hpp:3678-3719):
//
//   forward   send side (high-priority side streams, ring order p-1, p-2, ...): a peer that reads only some of my rows
//             is served by the persistent gather kernel, which gathers them straight from the caller's tensor and
//             STORES them into the peer's receive window over NVLink (CUDA-IPC mapping; no window copy of X, no
//             packing pass); a peer that reads ALL my rows gets one contiguous copy-engine transfer (no SM time);
//             either way pushed[p] is then raised in the peer's flags.  Receive side (main stream): the local chunk,
//             then either one aggregation launch per source partition (p+s) as soon as ITS flag is up (pipeline), or
//             ONE launch over all remote chunks once every flag is up (merged) - chosen once per width from measured
//             launch times (decide_mode).
//   backward  partial gradients of the active sources of every remote chunk (per chunk, or in one merged launch) into a
//             local staging; the copy engines push each slice into its owner's window; the local chunk overlaps with
//             the pushes; one scatter-add of everything received.
//   mirrors   DistGPUGetDepNbrOp forward / backward on the same windows (nts_exchange_fetch_mirrors / return_mirror_grads).
//
// Cross-GPU ordering: epoch-numbered flags in peer memory, release / acquire at system scope:
//   pushed[j]   (in my flags)  = last epoch for which rank j's rows have landed in my window,
//   consumed[j] (in my flags)  = last epoch whose window contents rank j has finished reading.
// The receive window has n_buffers (1 or 2) epoch-alternating buffers: before writing epoch e into peer j's window
// the pusher waits for consumed[j] >= e - n_buffers.  Every wait is bounded (NTS_EXCHANGE_TIMEOUT_MS, default 30 s):
// on expiry the kernel records what it was waiting for in a host-mapped word and traps, so a dead or failed peer
// surfaces as a CUDA error with a message instead of a hang.
// The CONTROL plane (row lists, IPC handles, barriers) stays with the caller - torch.distributed in this repo, MPI in
// the reference's host code - so this file depends on neither.
#include <algorithm>
#include <vector>

#include "nts_common.cuh"

namespace nts {
constexpr int kMaxPeers = 32;

struct PushTarget {
  const uint32_t *rows;          // local row ids to send (nullptr: rows are contiguous from `src_row0`)
  uint32_t n_rows, src_row0;
  float *dst;                    // first destination row in the peer's window (peer address)
  uint32_t *pushed_flag;         // peer address: flags[p] of that peer
  const uint32_t *consumed_flag; // local address: flags[P + j]
};
struct PushArgs {
  PushTarget t[kMaxPeers];
  int n;
  uint32_t epoch, wait_epoch; // wait for consumed >= wait_epoch (0: nothing to wait for)
};
} // namespace nts

struct nts_exchange {
  int P = 1, p = 0;
  nts_exchange_desc d;
  std::vector<nts_exchange_chunk> chunks;
  std::vector<uint32_t> need_count, send_count, recv_offs, srecv_offs, fwd_push_off, bwd_push_off;
  std::vector<char> send_all;         // [P] peer j reads ALL my rows in order: its forward push is one contiguous copy
  uint32_t recv_total = 0, send_total = 0;
  // exported receive window + flags
  float *window = nullptr;
  size_t buf_floats = 0; // floats per epoch buffer
  int n_buffers = 0;
  uint32_t *flags = nullptr;          // [2P]: pushed[P], consumed[P]
  uint32_t *tickets = nullptr;        // [P] CTA arrival counters of the push kernel (local)
  int *err_host = nullptr, *err_dev = nullptr; // host-mapped diagnostics of a timed-out wait
  std::vector<float *> peer_window;
  std::vector<uint32_t *> peer_flags;
  uint32_t **d_peer_flags = nullptr;
  bool peers_open = false;
  uint32_t epoch = 0;
  float *bsend = nullptr;             // backward partials [recv_total, F] (local)
  size_t bsend_cap = 0;
  float *stage16 = nullptr;           // BF16 gathers: this rank's X (forward) or dY (backward) as BF16 rows of stride
  size_t stage16_cap = 0;             // ld = ceil(F/8)*8, in floats (ld/2 per row)
  cudaStream_t comm = nullptr;
  std::vector<cudaStream_t> dma;      // [P] one stream per peer for copy-engine pushes: the copies to different peers
  std::vector<cudaEvent_t> ev_dma;    //     run on different copy engines at once (one engine alone does not fill NVLink)
  std::vector<char> dma_used;         //     streams used by the current call (joined back into `comm` at its end)
  cudaEvent_t ev_main = nullptr, ev_comm = nullptr;
  std::vector<cudaEvent_t> ev_peer;   // backward: partial of chunk i finished
  // preprocessed aggregation per chunk direction (created on first use; nullptr = plain kernel)
  std::vector<std::vector<std::pair<int, nts_gather_plan *>>> plan_fwd, plan_bwd; // [P] -> (plan_key(F, type), plan)
  // receive-side strategy per (direction, width), decided once from measured launch times (decide_mode):
  // 1 = pipeline (one launch per source partition as its rows land), 2 = merged (one launch over all remote chunks)
  struct Mode {
    int F, mode;
    bool bf16;
    nts_gather_plan *merged;
    float pipeline_ms, merged_ms; // the two estimates the decision was taken on
  };
  std::vector<Mode> mode_fwd, mode_bwd;
  int forced_mode = 0;                // NTS_EXCHANGE_MODE=pipeline|merged
  uint64_t plan_min_edges = 1u << 20;
  unsigned long long timeout_ns = 30ull * 1000000000ull;
  int push_ctas = 0;
  // optional per-phase timeline of the last forward (nts_exchange_set_trace): events on both streams
  bool trace = false;
  std::vector<cudaEvent_t> tev; // [0] call start, [1] push begin, [2] push end, [3] local chunk done,
                                // then per ring step s: [4+2(s-1)] rows of (p+s) have landed, [5+2(s-1)] chunk aggregated
  // which paths the last call took (nts_exchange_last_paths): host bookkeeping, filled while the call is enqueued
  struct Paths {
    int kind = 0, epoch = 0, buffer = 0, mode = 0, vec = 0, staging = 0;
    uint32_t kernel_peers = 0, dma_peers = 0, plan_chunks = 0;
  } last;
};

namespace nts {

__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t *p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t *p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
// spin until *flag >= value; on timeout record {code, index, wanted, seen} and trap
__device__ __forceinline__ void bounded_wait_geq(const uint32_t *flag, uint32_t value, unsigned long long timeout_ns,
                                                 int *err, int code, int index) {
  uint32_t v = ld_acquire_sys(flag);
  if (v >= value)
    return;
  const unsigned long long t0 = globaltimer_ns();
  while ((v = ld_acquire_sys(flag)) < value) {
    __nanosleep(200);
    if (globaltimer_ns() - t0 > timeout_ns) {
      if (err) {
        err[1] = index;
        err[2] = (int)value;
        err[3] = (int)v;
        __threadfence_system();
        err[0] = code;
        __threadfence_system();
      }
      __trap();
    }
  }
}

// wait for pushed[i] >= epoch for the listed partitions (one thread each)
__global__ void wait_pushed_kernel(const uint32_t *flags, uint32_t mask, uint32_t epoch, unsigned long long timeout_ns,
                                   int *err) {
  const int i = threadIdx.x;
  if (i < kMaxPeers && ((mask >> i) & 1u))
    bounded_wait_geq(flags + i, epoch, timeout_ns, err, 1, i);
}

// contiguous slices travel by the copy engines (cudaMemcpyAsync into the peer's window, no SM time): a one-thread wait
// before and a one-thread flag store after the copy, in stream order
__global__ void wait_consumed_kernel(const uint32_t *flag, uint32_t epoch, unsigned long long timeout_ns, int *err,
                                     int index) {
  bounded_wait_geq(flag, epoch, timeout_ns, err, 2, index);
}
__global__ void signal_pushed_kernel(uint32_t *peer_flag, uint32_t epoch) {
  __threadfence_system();
  st_release_sys(peer_flag, epoch);
}

// consumed[p] = epoch in every peer's flags
__global__ void signal_consumed_kernel(uint32_t *const *peer_flags, int P, int p, uint32_t value) {
  const int j = threadIdx.x;
  if (j >= P || j == p)
    return;
  __threadfence_system();
  st_release_sys(peer_flags[j] + P + p, value);
}

// The persistent push kernel: all CTAs work through the targets in order; a target's flag is raised by the last CTA
// to finish its share of that target's rows.  VEC floats per lane access (rows are F floats, F % VEC == 0, both
// sides VEC*4-byte aligned); 4-8 independent loads in flight per lane (four rows per warp step).
template <int VEC>
__global__ void __launch_bounds__(256)
    push_rows_kernel(const PushArgs a, const float *__restrict__ src, uint32_t F, uint32_t *tickets,
                     unsigned long long timeout_ns, int *err) {
  using V = typename Vec<VEC>::type;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps_per_cta = blockDim.x >> 5;
  const uint32_t gwarp = blockIdx.x * warps_per_cta + (threadIdx.x >> 5);
  const uint32_t n_warps = gridDim.x * warps_per_cta;
  const uint32_t nvec = F / VEC;
  for (int k = 0; k < a.n; k++) {
    const PushTarget t = a.t[k];
    if (t.n_rows) {
      if (a.wait_epoch && threadIdx.x == 0)
        bounded_wait_geq(t.consumed_flag, a.wait_epoch, timeout_ns, err, 2, k);
      __syncthreads();
      // four rows per warp step: 4 (narrow rows) or 8 independent loads per lane are in flight before the first store
      for (uint32_t r0 = gwarp * 4; r0 < t.n_rows; r0 += n_warps * 4) {
        const V *s[4];
        V *d[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const uint32_t r = min(r0 + k, t.n_rows - 1);
          const uint32_t srow = t.rows ? __ldg(t.rows + r) : t.src_row0 + r;
          s[k] = reinterpret_cast<const V *>(src + (size_t)srow * F);
          d[k] = reinterpret_cast<V *>(t.dst + (size_t)r * F);
        }
        const uint32_t live = min(4u, t.n_rows - r0);
        uint32_t c = lane;
        for (; c + 32 < nvec; c += 64) {
          V v[4][2];
#pragma unroll
          for (int k = 0; k < 4; k++) {
            v[k][0] = __ldg(s[k] + c);
            v[k][1] = __ldg(s[k] + c + 32);
          }
#pragma unroll
          for (int k = 0; k < 4; k++)
            if ((uint32_t)k < live) {
              d[k][c] = v[k][0];
              d[k][c + 32] = v[k][1];
            }
        }
        if (c < nvec) {
          V v[4];
#pragma unroll
          for (int k = 0; k < 4; k++)
            v[k] = __ldg(s[k] + c);
#pragma unroll
          for (int k = 0; k < 4; k++)
            if ((uint32_t)k < live)
              d[k][c] = v[k];
        }
      }
      __threadfence_system(); // my stores to the peer are ordered before the ticket below
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      const uint32_t ticket = atomicAdd(tickets + k, 1u);
      if (ticket == gridDim.x - 1) { // every CTA has finished this target
        tickets[k] = 0;
        __threadfence_system();
        st_release_sys(t.pushed_flag, a.epoch);
      }
    }
  }
}

} // namespace nts

using namespace nts;

#define NTS_TRY(expr)                                                                                               \
  do {                                                                                                              \
    int nts_rc_ = (expr);                                                                                           \
    if (nts_rc_ != 0)                                                                                               \
      return nts_rc_;                                                                                               \
  } while (0)

static int grow(float **buf, size_t *cap, size_t floats) {
  if (floats <= *cap)
    return 0;
  if (*buf)
    NTS_CUDA_OK(cudaFree(*buf));
  *buf = nullptr;
  NTS_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(buf), floats * sizeof(float)));
  *cap = floats;
  return 0;
}

// a timed-out wait left a record: turn the launch failure into a message
static int check_wait_error(nts_exchange *ex, int rc) {
  if (ex->err_host && ex->err_host[0]) {
    char msg[256];
    snprintf(msg, sizeof(msg),
             "exchange wait timed out on rank %d: %s %d (wanted epoch %d, saw %d) - a peer died, failed or fell out of step",
             ex->p, ex->err_host[0] == 1 ? "no rows pushed by partition" : "window not consumed by push target",
             ex->err_host[1], ex->err_host[2], ex->err_host[3]);
    return fail(rc ? rc : -1, msg, __FILE__, __LINE__);
  }
  return rc;
}

static int launch_push(nts_exchange *ex, const PushArgs &a, const float *src, uint32_t F, cudaStream_t st) {
  int vec = pick_vec(F, src);
  for (int k = 0; k < a.n; k++)
    vec = std::min(vec, pick_vec(F, a.t[k].dst));
  const int ctas = ex->push_ctas;
  ex->last.vec = vec;
  if (vec == 4)
    push_rows_kernel<4><<<ctas, 256, 0, st>>>(a, src, F, ex->tickets, ex->timeout_ns, ex->err_dev);
  else if (vec == 2)
    push_rows_kernel<2><<<ctas, 256, 0, st>>>(a, src, F, ex->tickets, ex->timeout_ns, ex->err_dev);
  else
    push_rows_kernel<1><<<ctas, 256, 0, st>>>(a, src, F, ex->tickets, ex->timeout_ns, ex->err_dev);
  NTS_LAUNCH_CHECK();
  return 0;
}

// One contiguous slice into peer j's window through the copy engines: [wait until j has consumed the buffer] -> peer
// copy -> raise pushed[p] at j.  n_rows == 0 still raises the flag (every rank signals every peer every call).
static int dma_push(nts_exchange *ex, int j, const float *src, size_t dst_row, uint32_t n_rows, uint32_t F, size_t buf,
                    uint32_t epoch, uint32_t wait_epoch, cudaStream_t from) {
  // fork: peer j's own stream continues after everything enqueued on `from` so far; dma_join() merges it back
  cudaStream_t st = ex->dma[j];
  NTS_CUDA_OK(cudaEventRecord(ex->ev_dma[j], from));
  NTS_CUDA_OK(cudaStreamWaitEvent(st, ex->ev_dma[j], 0));
  ex->dma_used[j] = 1;
  ex->last.dma_peers |= 1u << j;
  if (n_rows) {
    if (wait_epoch) {
      wait_consumed_kernel<<<1, 1, 0, st>>>(ex->flags + ex->P + j, wait_epoch, ex->timeout_ns, ex->err_dev, j);
      NTS_LAUNCH_CHECK();
    }
    NTS_CUDA_OK(cudaMemcpyAsync(ex->peer_window[j] + buf + dst_row * F, src, (size_t)n_rows * F * sizeof(float),
                                cudaMemcpyDeviceToDevice, st));
  }
  signal_pushed_kernel<<<1, 1, 0, st>>>(ex->peer_flags[j] + ex->p, epoch);
  NTS_LAUNCH_CHECK();
  return 0;
}

// `into` waits for every copy-engine push issued since the last join
static int dma_join(nts_exchange *ex, cudaStream_t into) {
  for (int j = 0; j < ex->P; j++)
    if (ex->dma_used[j]) {
      NTS_CUDA_OK(cudaEventRecord(ex->ev_dma[j], ex->dma[j]));
      NTS_CUDA_OK(cudaStreamWaitEvent(into, ex->ev_dma[j], 0));
      ex->dma_used[j] = 0;
    }
  return 0;
}

// Forward-style push of my rows to every peer in ring order p-1, p-2, ...: peers that read ALL my rows get one
// copy-engine transfer each, the others share persistent gather kernels (consecutive ones batched into one launch).
static int push_my_rows(nts_exchange *ex, const float *x, uint32_t F, size_t buf, uint32_t epoch, uint32_t wait_epoch) {
  const int P = ex->P, p = ex->p;
  PushArgs a;
  a.n = 0;
  a.epoch = epoch;
  a.wait_epoch = wait_epoch;
  for (int s = 1; s < P; s++) {
    const int j = (p - s + P) % P;
    if (ex->send_all[j]) {
      if (a.n) {
        NTS_TRY(launch_push(ex, a, x, F, ex->comm));
        a.n = 0;
      }
      NTS_TRY(dma_push(ex, j, x, ex->fwd_push_off[j], ex->send_count[j], F, buf, epoch, wait_epoch, ex->comm));
      continue;
    }
    ex->last.kernel_peers |= 1u << j;
    PushTarget &t = a.t[a.n++];
    t.rows = ex->d.send_rows_all + ex->srecv_offs[j];
    t.n_rows = ex->send_count[j];
    t.src_row0 = 0;
    t.dst = ex->peer_window[j] + buf + (size_t)ex->fwd_push_off[j] * F;
    t.pushed_flag = ex->peer_flags[j] + p;
    t.consumed_flag = ex->flags + P + j;
  }
  if (a.n)
    NTS_TRY(launch_push(ex, a, x, F, ex->comm));
  return 0;
}

// How a call gathers: FP32 rows of stride F, or BF16 rows of stride ld = ceil(F/8)*8 (FP32 accumulation).
struct GatherType {
  bool bf16;
  uint32_t ld; // row stride of the gathered input in elements
};
static int plan_key(uint32_t F, bool bf16) { return bf16 ? -(int)F : (int)F; } // plans are tuned per (width, type)

// aggregation of one chunk direction: preprocessed plan for big chunks (and for every BF16 gather), the plain kernel
// otherwise
static int aggregate_chunk(nts_exchange *ex, int i, bool forward, const void *in_rows, float *out, uint32_t F,
                           cudaStream_t st, GatherType gt = {false, 0}) {
  const float *in = static_cast<const float *>(in_rows);
  // chunk p is the local one: its "slots" are the global source ids of my own partition (base = dst_start) and its
  // "compact" row offsets are the plain row_offset over all my vertices
  const nts_exchange_chunk &c = ex->chunks[i];
  const bool local = i == ex->p;
  const uint32_t n_rows = (forward || local) ? ex->d.owned_vertices : ex->need_count[i];
  const uint32_t gather_rows = (forward && !local) ? ex->need_count[i] : ex->d.owned_vertices;
  if (!c.edges || !n_rows)
    return 0;
  const nts_vid_t *off = forward ? c.column_offset : c.row_offset_compact;
  const nts_vid_t *idx = forward ? c.slots : c.column_indices;
  const float *w = forward ? c.weight_forward : c.weight_backward;
  const uint32_t base = (forward && !local) ? 0u : ex->d.dst_start;
  if (c.edges >= ex->plan_min_edges || gt.bf16) {
    std::vector<std::pair<int, nts_gather_plan *>> &plans = (forward ? ex->plan_fwd : ex->plan_bwd)[i];
    nts_gather_plan *pl = nullptr;
    for (auto &e : plans)
      if (e.first == plan_key(F, gt.bf16))
        pl = e.second;
    if (!pl) { // first use of this width and type: slab and hub counts by measurement, built once and kept
      const nts_plan_part pt = {off, idx, w, nullptr, base, 0, n_rows, 0, c.edges};
      pl = tune_plan(&pt, 1, n_rows, gather_rows, F, gt.bf16, 0, true, st);
      if (!pl)
        return -1;
      int hc = 0, hr = 0, ehc = 0, ehr = 0;
      nts_gather_plan_hubs(pl, &hc, &hr);
      for (auto &e : plans) // another width settled on the same slab and hub counts: share its arrays
        if (nts_gather_plan_slabs(e.second) == nts_gather_plan_slabs(pl) &&
            nts_gather_plan_hubs(e.second, &ehc, &ehr) == 0 && ehc == hc && ehr == hr) {
          nts_gather_plan_destroy(pl);
          pl = e.second;
          break;
        }
      plans.emplace_back(plan_key(F, gt.bf16), pl);
    }
    ex->last.plan_chunks |= 1u << i;
    if (gt.bf16)
      return run_plan_bf16(pl, in_rows, NTS_DTYPE_BF16, gt.ld, out, F, st);
    return run_plan(pl, in, F, out, F, 0, st);
  }
  return nts_segment_gather_sum(in, out, w, idx, off, base, n_rows, c.edges, F, st);
}

// Pipeline or merged?  One launch per source partition hides the transfer behind the earlier chunks, but small
// launches run at a fraction of the large-launch rate (config B at 8 GPUs: 1.8 M-edge chunks);
// one merged launch is efficient but can only start when ALL rows have landed.  Decided once per (direction, width)
// from MEASURED launch times on scratch inputs (L = local chunk, c_i = remote chunks, M = merged launch) and the
// transfer time T of the bytes this rank receives (forward) / sends (backward) at 300 GB/s
// (two thirds of NVLink 4's 450 GB/s per direction on H100):
//   forward : pipeline ~ L + max(sum c_i, T - L)        merged ~ max(L, T) + M
//   backward: pipeline ~ sum c_i + max(L, T / (P-1))    merged ~ M + max(L, T)
// Each rank decides for itself (it only changes how a rank consumes its own window / fills its own staging).
//   (BF16 gathers: decided per (direction, width, type) on BF16 launches; T from the bytes actually pushed: BF16 rows
//    of ld = ceil(F/8)*8 values forward, FP32 partials backward)
static int decide_mode(nts_exchange *ex, bool forward, uint32_t F, cudaStream_t st, nts_exchange::Mode **out,
                       GatherType gt = {false, 0}) {
  std::vector<nts_exchange::Mode> &modes = forward ? ex->mode_fwd : ex->mode_bwd;
  for (auto &m : modes)
    if (m.F == (int)F && m.bf16 == gt.bf16) {
      *out = &m;
      return 0;
    }
  modes.push_back({(int)F, 1, gt.bf16, nullptr, 0.f, 0.f});
  nts_exchange::Mode &m = modes.back();
  *out = &m;
  const int P = ex->P, p = ex->p;
  const uint32_t Vp = ex->d.owned_vertices;
  uint64_t remote_edges = 0;
  int n_remote = 0;
  for (int i = 0; i < P; i++)
    if (i != p && ex->chunks[i].edges && ex->need_count[i]) {
      remote_edges += ex->chunks[i].edges;
      n_remote++;
    }
  if (ex->forced_mode == 1 || n_remote < 2 || !Vp || !ex->recv_total)
    return 0; // nothing to merge (or pipeline forced)
  // merged plan over all remote chunks (slab count measured)
  std::vector<nts_plan_part> parts;
  for (int i = 0; i < P; i++) {
    if (i == p || !ex->chunks[i].edges || !ex->need_count[i])
      continue;
    const nts_exchange_chunk &c = ex->chunks[i];
    nts_plan_part pt = {};
    if (forward) {
      pt.offsets = c.column_offset, pt.indices = c.slots, pt.weight = c.weight_forward;
      pt.index_base = 0, pt.index_add = ex->recv_offs[i], pt.n_rows = Vp, pt.row_add = 0;
    } else {
      pt.offsets = c.row_offset_compact, pt.indices = c.column_indices, pt.weight = c.weight_backward;
      pt.index_base = ex->d.dst_start, pt.index_add = 0, pt.n_rows = ex->need_count[i], pt.row_add = ex->recv_offs[i];
    }
    pt.n_edges = c.edges;
    parts.push_back(pt);
  }
  const uint32_t out_rows = forward ? Vp : ex->recv_total, in_rows = forward ? ex->recv_total : Vp;
  m.merged = tune_plan(parts.data(), (int)parts.size(), out_rows, in_rows, F, gt.bf16, 0, false, st);
  if (!m.merged)
    return -1;
  if (ex->forced_mode == 2) {
    m.mode = 2;
    return 0;
  }
  // measure: scratch inputs (zeros: the access pattern does not depend on the values)
  const size_t rows_max = std::max<size_t>(ex->recv_total, Vp);
  const size_t a_bytes = rows_max * std::max<size_t>((size_t)F * sizeof(float), gt.bf16 ? (size_t)gt.ld * 2 : 0);
  float *a = nullptr, *b = nullptr;
  NTS_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(&a), a_bytes));
  if (cudaMalloc(reinterpret_cast<void **>(&b), rows_max * F * sizeof(float)) != cudaSuccess) {
    cudaFree(a);
    return fail(-1, "scratch allocation for the exchange mode measurement failed", __FILE__, __LINE__);
  }
  cudaMemsetAsync(a, 0, a_bytes, st);
  cudaMemsetAsync(b, 0, rows_max * F * sizeof(float), st);
  float L = 0.f, M = 0.f, sum_c = 0.f;
  int rc = time_min_of_two([&]() { return aggregate_chunk(ex, p, forward, a, b, F, st, gt); }, st, &L);
  if (!rc)
    rc = time_min_of_two([&]() {
      return gt.bf16 ? run_plan_bf16(m.merged, a, NTS_DTYPE_BF16, gt.ld, b, F, st) : run_plan(m.merged, a, F, b, F, 0, st);
    }, st, &M);
  for (int i = 0; i < P && !rc; i++) {
    if (i == p || !ex->chunks[i].edges || !ex->need_count[i])
      continue;
    float c = 0.f;
    rc = time_min_of_two([&]() { return aggregate_chunk(ex, i, forward, a, b, F, st, gt); }, st, &c);
    sum_c += c;
  }
  cudaFree(a);
  cudaFree(b);
  if (rc)
    return rc;
  if (!ex->chunks[p].edges)
    L = 0.f;
  const double row_bytes = (forward && gt.bf16) ? gt.ld * 2.0 : F * 4.0;
  const float T = (float)((double)ex->recv_total * row_bytes / 300e9 * 1e3); // ms
  if (forward) {
    m.pipeline_ms = L + std::max(sum_c, T - L);
    m.merged_ms = std::max(L, T) + M;
  } else {
    m.pipeline_ms = sum_c + std::max(L, T / (float)(P - 1));
    m.merged_ms = M + std::max(L, T);
  }
  m.mode = m.merged_ms < m.pipeline_ms ? 2 : 1;
  if (m.mode == 1) { // the merged plan is not needed: release its arrays
    nts_gather_plan_destroy(m.merged);
    m.merged = nullptr;
  }
  return 0;
}

extern "C" {

nts_exchange *nts_exchange_create(const nts_exchange_desc *desc) {
  if (!desc || desc->partitions < 1 || desc->partitions > kMaxPeers || desc->rank < 0 ||
      desc->rank >= desc->partitions) {
    fail(-1, "bad exchange descriptor (1 <= partitions <= 32)", __FILE__, __LINE__);
    return nullptr;
  }
  nts_exchange *ex = new nts_exchange();
  ex->d = *desc;
  const int P = ex->P = desc->partitions, p = ex->p = desc->rank;
  if (P > 1 && !(desc->chunks && desc->need_count && desc->send_count && desc->fwd_push_offset &&
                 desc->bwd_push_offset)) {
    fail(-1, "exchange descriptor lacks the per-partition arrays", __FILE__, __LINE__);
    delete ex;
    return nullptr;
  }
  ex->need_count.assign(P, 0), ex->send_count.assign(P, 0), ex->fwd_push_off.assign(P, 0), ex->bwd_push_off.assign(P, 0);
  ex->chunks.assign(P, nts_exchange_chunk{});
  for (int i = 0; i < P && P > 1; i++) {
    if (i == p)
      continue;
    ex->need_count[i] = desc->need_count[i];
    ex->send_count[i] = desc->send_count[i];
    ex->fwd_push_off[i] = desc->fwd_push_offset[i];
    ex->bwd_push_off[i] = desc->bwd_push_offset[i];
    ex->chunks[i] = desc->chunks[i];
  }
  {
    nts_exchange_chunk &c = ex->chunks[p];
    c.column_offset = desc->local_column_offset;
    c.slots = desc->local_row_indices;
    c.weight_forward = desc->local_weight_forward;
    c.row_offset_compact = desc->local_row_offset;
    c.column_indices = desc->local_column_indices;
    c.weight_backward = desc->local_weight_backward;
    c.edges = desc->local_edges;
  }
  ex->recv_offs.assign(P + 1, 0), ex->srecv_offs.assign(P + 1, 0);
  for (int i = 0; i < P; i++) {
    ex->recv_offs[i + 1] = ex->recv_offs[i] + ex->need_count[i];
    ex->srecv_offs[i + 1] = ex->srecv_offs[i] + ex->send_count[i];
  }
  ex->recv_total = ex->recv_offs[P];
  ex->send_total = ex->srecv_offs[P];
  ex->send_all.assign(P, 0);
  if (P > 1 && ex->send_total && desc->send_rows_all && !getenv("NTS_EXCHANGE_NO_DMA")) {
    std::vector<uint32_t> rows(ex->send_total);
    if (cudaMemcpy(rows.data(), desc->send_rows_all, rows.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost) == cudaSuccess)
      for (int j = 0; j < P; j++) {
        if (j == p || ex->send_count[j] != desc->owned_vertices || !desc->owned_vertices)
          continue;
        bool ident = true;
        const uint32_t *r = rows.data() + ex->srecv_offs[j];
        for (uint32_t k = 0; k < ex->send_count[j] && ident; k++)
          ident = r[k] == k;
        ex->send_all[j] = ident;
      }
  }
  ex->peer_window.assign(P, nullptr);
  ex->peer_flags.assign(P, nullptr);
  ex->plan_fwd.resize(P), ex->plan_bwd.resize(P);
  ex->ev_peer.assign(P, nullptr);
  if (const char *t = getenv("NTS_EXCHANGE_TIMEOUT_MS")) {
    const long ms = atol(t);
    if (ms > 0)
      ex->timeout_ns = (unsigned long long)ms * 1000000ull;
  }
  if (const char *t = getenv("NTS_EXCHANGE_MODE"))
    ex->forced_mode = !strcmp(t, "pipeline") ? 1 : (!strcmp(t, "merged") ? 2 : 0);
  if (const char *t = getenv("NTS_EXCHANGE_PLAN_MIN_EDGES"))
    ex->plan_min_edges = strtoull(t, nullptr, 10);
  ex->push_ctas = std::max(8, sm_count() / 2); // enough memory-level parallelism for NVLink, half of the SMs at most
  if (const char *t = getenv("NTS_EXCHANGE_PUSH_CTAS")) {
    const int n = atoi(t);
    if (n > 0)
      ex->push_ctas = n;
  }
  int lo = 0, hi = 0;
  bool ok = cudaDeviceGetStreamPriorityRange(&lo, &hi) == cudaSuccess &&
            cudaMalloc(reinterpret_cast<void **>(&ex->flags), sizeof(uint32_t) * 2 * P) == cudaSuccess &&
            cudaMemset(ex->flags, 0, sizeof(uint32_t) * 2 * P) == cudaSuccess &&
            cudaMalloc(reinterpret_cast<void **>(&ex->tickets), sizeof(uint32_t) * kMaxPeers) == cudaSuccess &&
            cudaMemset(ex->tickets, 0, sizeof(uint32_t) * kMaxPeers) == cudaSuccess &&
            cudaMalloc(reinterpret_cast<void **>(&ex->d_peer_flags), sizeof(uint32_t *) * P) == cudaSuccess &&
            cudaHostAlloc(reinterpret_cast<void **>(&ex->err_host), 4 * sizeof(int), cudaHostAllocMapped) == cudaSuccess &&
            cudaHostGetDevicePointer(reinterpret_cast<void **>(&ex->err_dev), ex->err_host, 0) == cudaSuccess &&
            cudaStreamCreateWithPriority(&ex->comm, cudaStreamNonBlocking, hi) == cudaSuccess &&
            cudaEventCreateWithFlags(&ex->ev_main, cudaEventDisableTiming) == cudaSuccess &&
            cudaEventCreateWithFlags(&ex->ev_comm, cudaEventDisableTiming) == cudaSuccess;
  for (int i = 0; i < P && ok; i++)
    ok = cudaEventCreateWithFlags(&ex->ev_peer[i], cudaEventDisableTiming) == cudaSuccess;
  ex->dma.assign(P, nullptr), ex->ev_dma.assign(P, nullptr), ex->dma_used.assign(P, 0);
  for (int i = 0; i < P && ok && P > 1; i++)
    ok = cudaStreamCreateWithPriority(&ex->dma[i], cudaStreamNonBlocking, hi) == cudaSuccess &&
         cudaEventCreateWithFlags(&ex->ev_dma[i], cudaEventDisableTiming) == cudaSuccess;
  if (ok) {
    memset(ex->err_host, 0, 4 * sizeof(int));
    ok = cudaDeviceSynchronize() == cudaSuccess;
  }
  if (!ok) {
    fail(-1, "exchange resource allocation failed", __FILE__, __LINE__);
    delete ex;
    return nullptr;
  }
  return ex;
}

int nts_exchange_release_peers(nts_exchange *ex) {
  NTS_ARG_CHECK(ex != nullptr, "null engine");
  NTS_CUDA_OK(cudaDeviceSynchronize()); // my pushes into the peers' windows and my reads of my own are done
  if (ex->peers_open) {
    for (int j = 0; j < ex->P; j++)
      if (j != ex->p) {
        NTS_CUDA_OK(cudaIpcCloseMemHandle(ex->peer_window[j]));
        NTS_CUDA_OK(cudaIpcCloseMemHandle(ex->peer_flags[j]));
      }
    ex->peers_open = false;
  }
  return 0;
}

int nts_exchange_destroy(nts_exchange *ex) {
  if (!ex)
    return 0;
  cudaDeviceSynchronize();
  if (ex->peers_open)
    for (int j = 0; j < ex->P; j++)
      if (j != ex->p) {
        cudaIpcCloseMemHandle(ex->peer_window[j]);
        cudaIpcCloseMemHandle(ex->peer_flags[j]);
      }
  for (auto *side : {&ex->plan_fwd, &ex->plan_bwd})
    for (auto &per_chunk : *side) {
      std::vector<nts_gather_plan *> freed; // widths may share a plan
      for (auto &e : per_chunk)
        if (std::find(freed.begin(), freed.end(), e.second) == freed.end()) {
          nts_gather_plan_destroy(e.second);
          freed.push_back(e.second);
        }
    }
  for (auto *side : {&ex->mode_fwd, &ex->mode_bwd})
    for (auto &m : *side)
      nts_gather_plan_destroy(m.merged);
  cudaFree(ex->window);
  cudaFree(ex->flags);
  cudaFree(ex->tickets);
  cudaFree(ex->d_peer_flags);
  cudaFree(ex->bsend);
  cudaFree(ex->stage16);
  if (ex->err_host)
    cudaFreeHost(ex->err_host);
  if (ex->comm)
    cudaStreamDestroy(ex->comm);
  if (ex->ev_main)
    cudaEventDestroy(ex->ev_main);
  if (ex->ev_comm)
    cudaEventDestroy(ex->ev_comm);
  for (cudaEvent_t e : ex->ev_peer)
    if (e)
      cudaEventDestroy(e);
  for (cudaEvent_t e : ex->tev)
    if (e)
      cudaEventDestroy(e);
  for (cudaStream_t q : ex->dma)
    if (q)
      cudaStreamDestroy(q);
  for (cudaEvent_t e : ex->ev_dma)
    if (e)
      cudaEventDestroy(e);
  delete ex;
  return 0;
}

// Floats ONE epoch buffer of the receive window must hold for feature width F: the rows I read from peers (forward)
// or the partial gradients peers return for my rows (backward).
uint64_t nts_exchange_required_floats(const nts_exchange *ex, nts_vid_t feature_size) {
  uint64_t rows = std::max(ex->recv_total, ex->send_total);
  if (rows == 0)
    rows = 1;
  return rows * (uint64_t)feature_size;
}

// The same for BF16 gathers: forward rows arrive as BF16 at the padded stride ceil(F/8)*8 (ceil(F/8)*4 floats, more
// than F for F < 4), backward partials as FP32 rows of F floats.
uint64_t nts_exchange_required_floats_bf16(const nts_exchange *ex, nts_vid_t feature_size) {
  const uint64_t row16 = ((feature_size + 7ull) / 8ull) * 4ull;
  return std::max<uint64_t>(std::max<uint64_t>(ex->recv_total, 1) * row16, nts_exchange_required_floats(ex, feature_size));
}

uint64_t nts_exchange_capacity_floats(const nts_exchange *ex) { return ex ? ex->buf_floats : 0; }

// (Re)allocate the exported receive window: n_buffers epoch buffers of floats_per_buffer floats.
// CONTRACT (collective): a window may only be replaced when no rank still maps it or writes into it.  Sequence on
// EVERY rank: nts_exchange_release_peers -> barrier (caller's control plane) -> nts_exchange_reserve ->
// nts_exchange_handles -> (all-gather of the handles) -> nts_exchange_open_peers -> barrier.
int nts_exchange_reserve(nts_exchange *ex, uint64_t floats_per_buffer, int n_buffers) {
  NTS_ARG_CHECK(ex && (n_buffers == 1 || n_buffers == 2), "bad argument (n_buffers must be 1 or 2)");
  NTS_ARG_CHECK(!ex->peers_open, "nts_exchange_release_peers (and a barrier) must precede nts_exchange_reserve");
  NTS_CUDA_OK(cudaDeviceSynchronize());
  if (ex->window)
    NTS_CUDA_OK(cudaFree(ex->window));
  ex->window = nullptr;
  ex->buf_floats = 0;
  // every epoch buffer starts 256-byte aligned, like the first: the push kernel's vector width must not depend on
  // the epoch's parity
  floats_per_buffer = (floats_per_buffer + 63) & ~63ull;
  NTS_CUDA_OK(cudaMalloc(reinterpret_cast<void **>(&ex->window), floats_per_buffer * n_buffers * sizeof(float)));
  ex->buf_floats = floats_per_buffer;
  ex->n_buffers = n_buffers;
  return 0;
}

int nts_exchange_handles(nts_exchange *ex, unsigned char window_handle[NTS_IPC_HANDLE_BYTES],
                         unsigned char flags_handle[NTS_IPC_HANDLE_BYTES]) {
  NTS_ARG_CHECK(ex && ex->window && ex->flags, "window not allocated");
  cudaIpcMemHandle_t h;
  NTS_CUDA_OK(cudaIpcGetMemHandle(&h, ex->window));
  memcpy(window_handle, &h, sizeof(h));
  NTS_CUDA_OK(cudaIpcGetMemHandle(&h, ex->flags));
  memcpy(flags_handle, &h, sizeof(h));
  return 0;
}

// handles: P consecutive 64-byte window handles and P consecutive flag handles (own entries ignored)
int nts_exchange_open_peers(nts_exchange *ex, const unsigned char *window_handles, const unsigned char *flag_handles) {
  NTS_ARG_CHECK(ex && window_handles && flag_handles, "null argument");
  NTS_ARG_CHECK(!ex->peers_open, "peers already open");
  const int P = ex->P, p = ex->p;
  for (int j = 0; j < P; j++) {
    if (j == p) {
      ex->peer_window[j] = ex->window;
      ex->peer_flags[j] = ex->flags;
      continue;
    }
    cudaIpcMemHandle_t h;
    void *ptr = nullptr;
    memcpy(&h, window_handles + (size_t)j * NTS_IPC_HANDLE_BYTES, sizeof(h));
    NTS_CUDA_OK(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
    ex->peer_window[j] = static_cast<float *>(ptr);
    memcpy(&h, flag_handles + (size_t)j * NTS_IPC_HANDLE_BYTES, sizeof(h));
    NTS_CUDA_OK(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
    ex->peer_flags[j] = static_cast<uint32_t *>(ptr);
  }
  NTS_CUDA_OK(cudaMemcpy(ex->d_peer_flags, ex->peer_flags.data(), sizeof(uint32_t *) * P, cudaMemcpyHostToDevice));
  ex->peers_open = true;
  return 0;
}

static int ready_for(nts_exchange *ex, nts_vid_t F, bool bf16 = false) {
  NTS_ARG_CHECK(ex->peers_open && ex->n_buffers >= 1 &&
                    (bf16 ? nts_exchange_required_floats_bf16(ex, F) : nts_exchange_required_floats(ex, F)) <=
                        ex->buf_floats,
                "exchange window not reserved / peers not opened for this feature width");
  return 0;
}

// BF16 gathers: this rank's rows (X forward, dY backward) as BF16 at stride ld, converted once per call into the
// staging buffer - or used as they are when they already are BF16 rows of 16-byte multiples, aligned.  Returns the
// rows to push / gather from.
static int stage_bf16(nts_exchange *ex, const void *src, int dtype, uint32_t F, GatherType gt, cudaStream_t st,
                      const void **rows) {
  const uint32_t n = ex->d.owned_vertices;
  if (dtype == NTS_DTYPE_BF16 && gt.ld == F && aligned_to(src, 16)) {
    ex->last.staging = 2;
    *rows = src;
    return 0;
  }
  ex->last.staging = 1;
  NTS_TRY(grow(&ex->stage16, &ex->stage16_cap, (size_t)(n ? n : 1) * (gt.ld / 2)));
  NTS_TRY(to_bf16_rows(src, dtype, F, ex->stage16, n, F, gt.ld, st));
  *rows = ex->stage16;
  return 0;
}

// The receive mode of a forward / backward call.  decide_mode's timing runs aggregate chunks too, so the plan record
// starts here; a merged launch gathers every remote chunk that has edges through the merged plan.
static void record_mode(nts_exchange *ex, const nts_exchange::Mode &m) {
  ex->last.mode = m.mode;
  ex->last.plan_chunks = 0;
  if (m.mode == 2)
    for (int i = 0; i < ex->P; i++)
      if (i != ex->p && ex->chunks[i].edges && ex->need_count[i])
        ex->last.plan_chunks |= 1u << i;
}

static int forward_impl(nts_exchange *ex, const void *x_in, int x_dtype, float *y, nts_vid_t F, void *stream,
                        bool bf16 = false) {
  const nts_exchange_desc &d = ex->d;
  const float *x = static_cast<const float *>(x_in);
  // a rank that owns no vertices (the 1024-aligned partitioner leaves such ranks on small graphs) has no rows to
  // push or produce, but still takes part in the flag protocol below
  NTS_ARG_CHECK(d.owned_vertices == 0 || (x && y), "null feature pointer");
  cudaStream_t st = as_stream(stream);
  const int P = ex->P, p = ex->p;
  ex->last = {};
  ex->last.kind = 1;
  NTS_ARG_CHECK(!bf16 || P > 1, "BF16 gathers on one partition run through nts_gather_plan_run_bf16_ex");
  if (P == 1)
    return nts_gather_by_dst_from_src(x, y, d.local_weight_forward, d.local_row_indices, d.local_column_offset,
                                      d.dst_start, d.dst_start + d.owned_vertices, d.dst_start,
                                      d.dst_start + d.owned_vertices, d.local_edges, d.owned_vertices, F, 1, stream);
  NTS_TRY(ready_for(ex, F, bf16));
  // BF16: rows travel and are gathered as BF16 at stride ld; the push moves them as rows of Fw = ld/2 floats
  const GatherType gt = {bf16, bf16 ? ((F + 7u) & ~7u) : F};
  const uint32_t Fw = bf16 ? gt.ld / 2 : F;
  if (bf16 && d.owned_vertices) {
    const void *rows = nullptr;
    NTS_TRY(stage_bf16(ex, x_in, x_dtype, F, gt, st, &rows));
    x = static_cast<const float *>(rows);
  }
  const uint32_t epoch = ++ex->epoch;
  const size_t buf = (size_t)(epoch % ex->n_buffers) * ex->buf_floats;
  const uint32_t wait_epoch = epoch > (uint32_t)ex->n_buffers ? epoch - ex->n_buffers : 0u;
  ex->last.epoch = (int)epoch, ex->last.buffer = (int)(epoch % ex->n_buffers);
  const bool tr = ex->trace && (int)ex->tev.size() >= 4 + 2 * (P - 1);
  NTS_CUDA_OK(cudaEventRecord(ex->ev_main, st)); // x is ready
  if (tr)
    NTS_CUDA_OK(cudaEventRecord(ex->tev[0], st));
  NTS_CUDA_OK(cudaStreamWaitEvent(ex->comm, ex->ev_main, 0));
  if (tr)
    NTS_CUDA_OK(cudaEventRecord(ex->tev[1], ex->comm));
  // ---- side stream: my rows to every peer, ring order p-1, p-2, ... (the peer that needs them first)
  NTS_TRY(push_my_rows(ex, x, Fw, buf, epoch, wait_epoch));
  NTS_TRY(dma_join(ex, ex->comm));
  if (tr)
    NTS_CUDA_OK(cudaEventRecord(ex->tev[2], ex->comm));
  // ---- main stream: local chunk, then the remote chunks - one launch per partition as its rows arrive (pipeline) or
  // one launch over all of them once everything has landed (merged); measured once per width, see decide_mode
  nts_exchange::Mode *mode = nullptr;
  NTS_TRY(decide_mode(ex, true, F, st, &mode, gt));
  record_mode(ex, *mode);
  NTS_TRY(aggregate_chunk(ex, p, true, x, y, F, st, gt));
  if (tr)
    NTS_CUDA_OK(cudaEventRecord(ex->tev[3], st));
  if (mode->mode == 2) {
    uint32_t mask = 0;
    for (int j = 0; j < P; j++)
      if (j != p)
        mask |= 1u << j;
    wait_pushed_kernel<<<1, 32, 0, st>>>(ex->flags, mask, epoch, ex->timeout_ns, ex->err_dev);
    NTS_LAUNCH_CHECK();
    if (tr)
      NTS_CUDA_OK(cudaEventRecord(ex->tev[4], st));
    if (bf16)
      NTS_TRY(run_plan_bf16(mode->merged, ex->window + buf, NTS_DTYPE_BF16, gt.ld, y, F, st));
    else
      NTS_TRY(run_plan(mode->merged, ex->window + buf, F, y, F, 0, st));
    if (tr)
      for (int s = 1; s < P; s++) { // the merged launch is reported under ring step 1, the other steps read 0
        NTS_CUDA_OK(cudaEventRecord(ex->tev[5 + 2 * (s - 1)], st));
        if (s + 1 < P)
          NTS_CUDA_OK(cudaEventRecord(ex->tev[4 + 2 * s], st));
      }
  } else {
    for (int s = 1; s < P; s++) {
      const int i = (p + s) % P;
      wait_pushed_kernel<<<1, 32, 0, st>>>(ex->flags, 1u << i, epoch, ex->timeout_ns, ex->err_dev);
      NTS_LAUNCH_CHECK();
      if (tr)
        NTS_CUDA_OK(cudaEventRecord(ex->tev[4 + 2 * (s - 1)], st));
      if (ex->need_count[i])
        NTS_TRY(aggregate_chunk(ex, i, true, ex->window + buf + (size_t)ex->recv_offs[i] * Fw, y, F, st, gt));
      if (tr)
        NTS_CUDA_OK(cudaEventRecord(ex->tev[5 + 2 * (s - 1)], st));
    }
  }
  signal_consumed_kernel<<<1, 32, 0, st>>>(ex->d_peer_flags, P, p, epoch);
  NTS_LAUNCH_CHECK();
  // the next call on `st` may overwrite x: it must not start before the push kernel has read it
  NTS_CUDA_OK(cudaEventRecord(ex->ev_comm, ex->comm));
  NTS_CUDA_OK(cudaStreamWaitEvent(st, ex->ev_comm, 0));
  return 0;
}

static int backward_impl(nts_exchange *ex, const float *g, float *dx, nts_vid_t F, void *stream, bool bf16 = false) {
  const nts_exchange_desc &d = ex->d;
  NTS_ARG_CHECK(d.owned_vertices == 0 || (g && dx), "null gradient pointer");
  cudaStream_t st = as_stream(stream);
  const int P = ex->P, p = ex->p;
  ex->last = {};
  ex->last.kind = 2;
  NTS_ARG_CHECK(!bf16 || P > 1, "BF16 gathers on one partition run through nts_gather_plan_run_bf16_ex");
  if (P == 1)
    return nts_gather_by_src_from_dst(g, dx, d.local_weight_backward, d.local_row_offset, d.local_column_indices,
                                      d.dst_start, d.dst_start + d.owned_vertices, d.dst_start,
                                      d.dst_start + d.owned_vertices, d.local_edges, d.owned_vertices, F, 1, stream);
  NTS_TRY(ready_for(ex, F, bf16));
  // BF16: dY converted once into BF16 rows of stride ld, every chunk gathers from them; partials stay FP32
  const GatherType gt = {bf16, bf16 ? ((F + 7u) & ~7u) : F};
  const void *gin = g;
  if (bf16 && d.owned_vertices)
    NTS_TRY(stage_bf16(ex, g, NTS_DTYPE_F32, F, gt, st, &gin));
  const uint32_t epoch = ++ex->epoch;
  const size_t buf = (size_t)(epoch % ex->n_buffers) * ex->buf_floats;
  const uint32_t wait_epoch = epoch > (uint32_t)ex->n_buffers ? epoch - ex->n_buffers : 0u;
  ex->last.epoch = (int)epoch, ex->last.buffer = (int)(epoch % ex->n_buffers);
  NTS_TRY(grow(&ex->bsend, &ex->bsend_cap, (size_t)(ex->recv_total ? ex->recv_total : 1) * F));
  if (ex->recv_total)
    NTS_CUDA_OK(cudaMemsetAsync(ex->bsend, 0, (size_t)ex->recv_total * F * sizeof(float), st));
  nts_exchange::Mode *mode = nullptr;
  NTS_TRY(decide_mode(ex, false, F, st, &mode, gt));
  record_mode(ex, *mode);
  if (mode->mode == 2) {
    // ---- merged: ONE launch computes the partial gradients of the active sources of all remote chunks, then every
    // slice goes to its owner through the copy engines
    if (bf16)
      NTS_TRY(run_plan_bf16(mode->merged, gin, NTS_DTYPE_BF16, gt.ld, ex->bsend, F, st));
    else
      NTS_TRY(run_plan(mode->merged, g, F, ex->bsend, F, 0, st));
    NTS_CUDA_OK(cudaEventRecord(ex->ev_peer[p], st));
    NTS_CUDA_OK(cudaStreamWaitEvent(ex->comm, ex->ev_peer[p], 0));
    for (int s = 1; s < P; s++) {
      const int i = (p + s) % P;
      NTS_TRY(dma_push(ex, i, ex->bsend + (size_t)ex->recv_offs[i] * F, ex->bwd_push_off[i], ex->need_count[i], F, buf,
                       epoch, wait_epoch, ex->comm));
    }
  } else {
    // ---- pipeline: per remote chunk (p+1, p+2, ...) the partial gradients of its active sources, pushed to the
    // owner while the next chunk computes
    for (int s = 1; s < P; s++) {
      const int i = (p + s) % P;
      float *slice = ex->bsend + (size_t)ex->recv_offs[i] * F;
      if (ex->need_count[i])
        NTS_TRY(aggregate_chunk(ex, i, false, gin, slice, F, st, gt));
      NTS_CUDA_OK(cudaEventRecord(ex->ev_peer[i], st));
      NTS_CUDA_OK(cudaStreamWaitEvent(ex->comm, ex->ev_peer[i], 0));
      NTS_TRY(dma_push(ex, i, ex->bsend + (size_t)ex->recv_offs[i] * F, ex->bwd_push_off[i], ex->need_count[i], F, buf,
                       epoch, wait_epoch, ex->comm));
    }
  }
  // ---- local chunk overlaps with the pushes; then everything the peers computed for my rows
  NTS_TRY(aggregate_chunk(ex, p, false, gin, dx, F, st, gt));
  uint32_t mask = 0;
  for (int j = 0; j < P; j++)
    if (j != p)
      mask |= 1u << j;
  wait_pushed_kernel<<<1, 32, 0, st>>>(ex->flags, mask, epoch, ex->timeout_ns, ex->err_dev);
  NTS_LAUNCH_CHECK();
  if (ex->send_total)
    NTS_TRY(nts_scatter_add_rows_atomic(dx, ex->window + buf, d.send_rows_all, ex->send_total, F, st));
  signal_consumed_kernel<<<1, 32, 0, st>>>(ex->d_peer_flags, P, p, epoch);
  NTS_LAUNCH_CHECK();
  // bsend is rewritten by the next backward on `st`: the pushes must have read it
  NTS_TRY(dma_join(ex, ex->comm));
  NTS_CUDA_OK(cudaEventRecord(ex->ev_comm, ex->comm));
  NTS_CUDA_OK(cudaStreamWaitEvent(st, ex->ev_comm, 0));
  return 0;
}

// mirror[M, F] = the feature row of every source of a local in-edge, in MirrorIndex order (partition 0's active rows,
// partition 1's, ...; core/PartitionedGraph.hpp:295-305): remote rows arrive through the same push as the forward
// exchange, the own partition's rows by a local gather.
static int fetch_impl(nts_exchange *ex, const float *x, float *mirror, nts_vid_t F, void *stream) {
  const nts_exchange_desc &d = ex->d;
  cudaStream_t st = as_stream(stream);
  const int P = ex->P, p = ex->p;
  const uint32_t own = d.local_need_count;
  ex->last = {};
  ex->last.kind = 3;
  NTS_ARG_CHECK(own == 0 || d.local_need, "exchange descriptor lacks local_need (rows of this partition it reads itself)");
  if (P == 1)
    return own ? nts_gather_rows(mirror, x, d.local_need, own, F, stream) : 0;
  NTS_TRY(ready_for(ex, F));
  const uint32_t epoch = ++ex->epoch;
  const size_t buf = (size_t)(epoch % ex->n_buffers) * ex->buf_floats;
  const uint32_t wait_epoch = epoch > (uint32_t)ex->n_buffers ? epoch - ex->n_buffers : 0u;
  ex->last.epoch = (int)epoch, ex->last.buffer = (int)(epoch % ex->n_buffers);
  NTS_CUDA_OK(cudaEventRecord(ex->ev_main, st));
  NTS_CUDA_OK(cudaStreamWaitEvent(ex->comm, ex->ev_main, 0));
  NTS_TRY(push_my_rows(ex, x, F, buf, epoch, wait_epoch));
  NTS_TRY(dma_join(ex, ex->comm));
  const size_t before = ex->recv_offs[p]; // staged rows of the partitions before mine
  if (own)
    NTS_TRY(nts_gather_rows(mirror + before * F, x, d.local_need, own, F, st));
  uint32_t mask = 0;
  for (int j = 0; j < P; j++)
    if (j != p)
      mask |= 1u << j;
  wait_pushed_kernel<<<1, 32, 0, st>>>(ex->flags, mask, epoch, ex->timeout_ns, ex->err_dev);
  NTS_LAUNCH_CHECK();
  if (before)
    NTS_CUDA_OK(cudaMemcpyAsync(mirror, ex->window + buf, before * F * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (ex->recv_total > before)
    NTS_CUDA_OK(cudaMemcpyAsync(mirror + (before + own) * F, ex->window + buf + before * F,
                                (ex->recv_total - before) * (size_t)F * sizeof(float), cudaMemcpyDeviceToDevice, st));
  signal_consumed_kernel<<<1, 32, 0, st>>>(ex->d_peer_flags, P, p, epoch);
  NTS_LAUNCH_CHECK();
  NTS_CUDA_OK(cudaEventRecord(ex->ev_comm, ex->comm));
  NTS_CUDA_OK(cudaStreamWaitEvent(st, ex->ev_comm, 0));
  return 0;
}

// dx[v, :] += the mirror gradients every partition holds for my vertex v (dx zeroed by the caller): slices of
// mirror_grad go straight from the caller's buffer into the owners' windows.
static int return_impl(nts_exchange *ex, const float *gm, float *dx, nts_vid_t F, void *stream) {
  const nts_exchange_desc &d = ex->d;
  cudaStream_t st = as_stream(stream);
  const int P = ex->P, p = ex->p;
  const uint32_t own = d.local_need_count;
  ex->last = {};
  ex->last.kind = 4;
  NTS_ARG_CHECK(own == 0 || d.local_need, "exchange descriptor lacks local_need");
  if (P == 1)
    return own ? nts_scatter_add_rows(dx, gm, d.local_need, own, F, stream) : 0;
  NTS_TRY(ready_for(ex, F));
  const uint32_t epoch = ++ex->epoch;
  const size_t buf = (size_t)(epoch % ex->n_buffers) * ex->buf_floats;
  const size_t before = ex->recv_offs[p];
  const uint32_t wait_epoch = epoch > (uint32_t)ex->n_buffers ? epoch - ex->n_buffers : 0u;
  ex->last.epoch = (int)epoch, ex->last.buffer = (int)(epoch % ex->n_buffers);
  NTS_CUDA_OK(cudaEventRecord(ex->ev_main, st));
  NTS_CUDA_OK(cudaStreamWaitEvent(ex->comm, ex->ev_main, 0));
  for (int s = 1; s < P; s++) {
    const int i = (p + s) % P; // partition i's block of the mirror-gradient matrix goes to its owner
    NTS_TRY(dma_push(ex, i, gm + (size_t)(ex->recv_offs[i] + (i > p ? own : 0u)) * F, ex->bwd_push_off[i],
                     ex->need_count[i], F, buf, epoch, wait_epoch, ex->comm));
  }
  if (own)
    NTS_TRY(nts_scatter_add_rows(dx, gm + before * F, d.local_need, own, F, st));
  uint32_t mask = 0;
  for (int j = 0; j < P; j++)
    if (j != p)
      mask |= 1u << j;
  wait_pushed_kernel<<<1, 32, 0, st>>>(ex->flags, mask, epoch, ex->timeout_ns, ex->err_dev);
  NTS_LAUNCH_CHECK();
  if (ex->send_total)
    NTS_TRY(nts_scatter_add_rows_atomic(dx, ex->window + buf, d.send_rows_all, ex->send_total, F, st));
  signal_consumed_kernel<<<1, 32, 0, st>>>(ex->d_peer_flags, P, p, epoch);
  NTS_LAUNCH_CHECK();
  NTS_TRY(dma_join(ex, ex->comm));
  NTS_CUDA_OK(cudaEventRecord(ex->ev_comm, ex->comm));
  NTS_CUDA_OK(cudaStreamWaitEvent(st, ex->ev_comm, 0));
  return 0;
}

// Per-phase device timeline of forward calls (bench.py exchange_timeline): enable, run ONE forward, read.
int nts_exchange_set_trace(nts_exchange *ex, int enable) {
  NTS_ARG_CHECK(ex != nullptr, "null engine");
  if (enable && ex->tev.empty()) {
    ex->tev.assign(4 + 2 * (ex->P > 1 ? ex->P - 1 : 0), nullptr);
    for (cudaEvent_t &e : ex->tev)
      NTS_CUDA_OK(cudaEventCreate(&e));
  }
  ex->trace = enable != 0;
  return 0;
}

// ms[0] push kernel (side stream), ms[1] local chunk, then per ring step s = 1..P-1: ms[2s] time the main stream sat
// waiting for the rows of partition (p+s) after it was ready for them, ms[2s+1] aggregation of chunk (p+s);
// ms[2P] whole call on the main stream (2P+1 entries).  Synchronises the device.
int nts_exchange_last_timeline(nts_exchange *ex, float *ms, int capacity) {
  NTS_ARG_CHECK(ex && ms && ex->trace && !ex->tev.empty(), "tracing is not enabled");
  const int P = ex->P, n = 2 * P + 1;
  NTS_ARG_CHECK(capacity >= n, "timeline buffer too small (2P+1 floats)");
  NTS_CUDA_OK(cudaDeviceSynchronize());
  NTS_CUDA_OK(cudaEventElapsedTime(&ms[0], ex->tev[1], ex->tev[2]));
  NTS_CUDA_OK(cudaEventElapsedTime(&ms[1], ex->tev[0], ex->tev[3]));
  cudaEvent_t prev = ex->tev[3];
  for (int s = 1; s < P; s++) {
    NTS_CUDA_OK(cudaEventElapsedTime(&ms[2 * s], prev, ex->tev[4 + 2 * (s - 1)]));
    NTS_CUDA_OK(cudaEventElapsedTime(&ms[2 * s + 1], ex->tev[4 + 2 * (s - 1)], ex->tev[5 + 2 * (s - 1)]));
    prev = ex->tev[5 + 2 * (s - 1)];
  }
  NTS_CUDA_OK(cudaEventElapsedTime(&ms[2 * P], ex->tev[0], prev));
  return 0;
}

int nts_exchange_last_paths(const nts_exchange *ex, int *kind, int *epoch, int *buffer, int *mode,
                            uint32_t *kernel_peers, uint32_t *dma_peers, int *push_vec, uint32_t *plan_chunks,
                            int *bf16_staging) {
  NTS_ARG_CHECK(ex != nullptr, "null engine");
  const nts_exchange::Paths &r = ex->last;
  if (kind)
    *kind = r.kind;
  if (epoch)
    *epoch = r.epoch;
  if (buffer)
    *buffer = r.buffer;
  if (mode)
    *mode = r.mode;
  if (kernel_peers)
    *kernel_peers = r.kernel_peers;
  if (dma_peers)
    *dma_peers = r.dma_peers;
  if (push_vec)
    *push_vec = r.vec;
  if (plan_chunks)
    *plan_chunks = r.plan_chunks;
  if (bf16_staging)
    *bf16_staging = r.staging;
  return 0;
}

int nts_exchange_fetch_mirrors(nts_exchange *ex, const float *x, float *mirror, nts_vid_t F, void *stream) {
  // (a rank without in-edges has an empty mirror matrix: NULL is fine then, it still takes part in the protocol)
  NTS_ARG_CHECK(ex && (x || ex->d.owned_vertices == 0) && (mirror || ex->recv_total + ex->d.local_need_count == 0),
                "null argument");
  return check_wait_error(ex, fetch_impl(ex, x, mirror, F, stream));
}

int nts_exchange_return_mirror_grads(nts_exchange *ex, const float *mirror_grad, float *dx, nts_vid_t F, void *stream) {
  NTS_ARG_CHECK(ex && (mirror_grad || ex->recv_total + ex->d.local_need_count == 0) &&
                    (dx || ex->d.owned_vertices == 0),
                "null argument");
  return check_wait_error(ex, return_impl(ex, mirror_grad, dx, F, stream));
}

// Y_p += sum_i A_{p<-i} X_i.  `y` must be zeroed by the caller (accumulate semantics, like every aggregation entry).
int nts_exchange_forward(nts_exchange *ex, const float *x, float *y, nts_vid_t F, void *stream) {
  NTS_ARG_CHECK(ex != nullptr, "null engine");
  return check_wait_error(ex, forward_impl(ex, x, NTS_DTYPE_F32, y, F, stream));
}

// dX_p += sum_j A_{j<-p}^T dY_j.  `dx` must be zeroed by the caller.
int nts_exchange_backward(nts_exchange *ex, const float *g, float *dx, nts_vid_t F, void *stream) {
  NTS_ARG_CHECK(ex != nullptr, "null engine");
  return check_wait_error(ex, backward_impl(ex, g, dx, F, stream));
}

// BF16 gathers with FP32 accumulation (nts_gather_plan_run_bf16_ex's contract) across partitions: the rows travel as BF16
int nts_exchange_forward_bf16(nts_exchange *ex, const void *x, int x_dtype, float *y, nts_vid_t F, void *stream) {
  NTS_ARG_CHECK(ex != nullptr, "null engine");
  NTS_ARG_CHECK(x_dtype == NTS_DTYPE_F32 || x_dtype == NTS_DTYPE_BF16, "x_dtype must be NTS_DTYPE_F32 or NTS_DTYPE_BF16");
  return check_wait_error(ex, forward_impl(ex, x, x_dtype, y, F, stream, true));
}

int nts_exchange_backward_bf16(nts_exchange *ex, const float *g, float *dx, nts_vid_t F, void *stream) {
  NTS_ARG_CHECK(ex != nullptr, "null engine");
  return check_wait_error(ex, backward_impl(ex, g, dx, F, stream, true));
}

} // extern "C"
