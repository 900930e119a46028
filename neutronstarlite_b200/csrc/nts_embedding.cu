// K11: row-sparse Adam on a learnable embedding table sharded over the ranks of one node (feature_table.ShardedEmbedding).
//
// Every rank q has an outbox, one buffer its peers map over CUDA IPC:
//   [0, 16)                      uint32 count n_q (the rest of the 16 bytes unused)
//   [16, 16 + 16*ceil(cap/4))    n_q strictly ascending global row ids (uint32)
//   then                         n_q gradient rows of `pitch` floats (pad columns zero)
// One step on the owner of rows [lo, hi) is two launches on one stream, and neither needs the host to know a count:
//   mark:   every rank's outbox ids, grid-stride over the device-side counts; an id in [lo, hi) sets bit q of its row's
//           mask (atomicOr), its position in outbox q is recorded, and the first bit set appends the row to `touched`
//   update: one (virtual) warp per touched row sums the contributors' gradient rows in ascending rank order, starting
//           from the first contributor's row, applies adam_element to the row and its M and V, and clears the mask.
// A row's result depends only on its contributors' rows and its own state: the order of `touched` does not matter.
#include "nts_common.cuh"

namespace nts {
namespace {

constexpr int kThreads = 256;
constexpr int kBlocksPerSm = 8;

__device__ __forceinline__ const uint32_t *outbox_ids(const void *box) {
  return reinterpret_cast<const uint32_t *>(static_cast<const char *>(box) + 16);
}
__device__ __forceinline__ const float4 *outbox_rows(const void *box, uint32_t capacity) {
  return reinterpret_cast<const float4 *>(static_cast<const char *>(box) + 16 + 16 * (((uint64_t)capacity + 3) / 4));
}

__global__ void __launch_bounds__(kThreads)
    embedding_mark_kernel(const void *const *__restrict__ outboxes, int n_ranks, uint32_t lo, uint32_t hi,
                          uint32_t *__restrict__ mask, uint32_t *__restrict__ positions,
                          uint32_t *__restrict__ touched) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (int q = 0; q < n_ranks; q++) {
    const void *box = outboxes[q];
    const uint32_t n = *static_cast<const uint32_t *>(box);
    const uint32_t *ids = outbox_ids(box);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
      const uint32_t id = ids[i];
      if (id < lo || id >= hi)
        continue;
      const uint32_t r = id - lo;
      positions[(size_t)r * n_ranks + q] = i;
      if (atomicOr(mask + r, 1u << q) == 0)
        touched[1 + atomicAdd(touched, 1u)] = r;
    }
  }
}

// LANES lanes (a power of two <= 32) per touched row, each owning the row's float4 columns c = sub, sub + LANES, ...
template <int LANES>
__global__ void __launch_bounds__(kThreads)
    embedding_update_kernel(float *__restrict__ rows, float *__restrict__ M, float *__restrict__ V,
                            uint32_t *__restrict__ mask, const uint32_t *__restrict__ positions,
                            const uint32_t *__restrict__ touched, const void *const *__restrict__ outboxes,
                            int n_ranks, uint32_t capacity, uint32_t pitch, uint32_t F, float weight_decay,
                            float beta1, float beta2, float alpha, float epsilon) {
  __shared__ const float4 *s_rows[kMaxShards];
  for (int q = threadIdx.x; q < n_ranks; q += blockDim.x)
    s_rows[q] = outbox_rows(outboxes[q], capacity);
  __syncthreads();
  constexpr uint32_t kRowsPerBlock = kThreads / LANES;
  const uint32_t lane = threadIdx.x & 31, sub = threadIdx.x & (LANES - 1);
  const uint32_t group = LANES == 32 ? 0xffffffffu : ((1u << LANES) - 1) << (lane & ~(LANES - 1));
  const uint32_t n = __ldcg(touched); // the mark launch's atomics left it in L2
  const uint32_t nvec = (F + 3) / 4, vpitch = pitch / 4;
  for (uint32_t k = blockIdx.x * kRowsPerBlock + threadIdx.x / LANES; k < n; k += gridDim.x * kRowsPerBlock) {
    const uint32_t r = touched[1 + k];
    // the group's first lane reads and clears the row's mask; every lane of the group takes the same k
    uint32_t bits = 0;
    if (sub == 0) {
      bits = mask[r];
      mask[r] = 0;
    }
    bits = __shfl_sync(group, bits, 0, LANES);
    const int q0 = __ffs(bits) - 1;
    const float4 *g0 = s_rows[q0] + (size_t)positions[(size_t)r * n_ranks + q0] * vpitch;
    float4 *w4 = reinterpret_cast<float4 *>(rows + (size_t)r * pitch);
    float4 *m4 = reinterpret_cast<float4 *>(M + (size_t)r * pitch);
    float4 *v4 = reinterpret_cast<float4 *>(V + (size_t)r * pitch);
    for (uint32_t c = sub; c < nvec; c += LANES) {
      float4 g = g0[c];
      for (uint32_t rest = bits & (bits - 1); rest; rest &= rest - 1) {
        const int q = __ffs(rest) - 1;
        const float4 h = s_rows[q][(size_t)positions[(size_t)r * n_ranks + q] * vpitch + c];
        g.x = __fadd_rn(g.x, h.x);
        g.y = __fadd_rn(g.y, h.y);
        g.z = __fadd_rn(g.z, h.z);
        g.w = __fadd_rn(g.w, h.w);
      }
      float4 w = w4[c], m = m4[c], v = v4[c];
      // the pad columns of the last vector (4c + j >= F) keep their values
      adam_element(w.x, m.x, v.x, g.x, weight_decay, beta1, beta2, alpha, epsilon);
      if (4 * c + 1 < F)
        adam_element(w.y, m.y, v.y, g.y, weight_decay, beta1, beta2, alpha, epsilon);
      if (4 * c + 2 < F)
        adam_element(w.z, m.z, v.z, g.z, weight_decay, beta1, beta2, alpha, epsilon);
      if (4 * c + 3 < F)
        adam_element(w.w, m.w, v.w, g.w, weight_decay, beta1, beta2, alpha, epsilon);
      w4[c] = w;
      m4[c] = m;
      v4[c] = v;
    }
  }
}

template <int LANES>
void launch_update(unsigned grid, cudaStream_t st, float *rows, float *M, float *V, uint32_t *mask,
                   const uint32_t *positions, const uint32_t *touched, const void *const *outboxes, int n_ranks,
                   uint32_t capacity, uint32_t pitch, uint32_t F, float wd, float b1, float b2, float alpha,
                   float eps) {
  embedding_update_kernel<LANES><<<grid, kThreads, 0, st>>>(rows, M, V, mask, positions, touched, outboxes, n_ranks,
                                                            capacity, pitch, F, wd, b1, b2, alpha, eps);
}

} // namespace
} // namespace nts

using namespace nts;

extern "C" int nts_embedding_step(float *rows, float *adam_m, float *adam_v, uint32_t *mask, uint32_t *positions,
                                  uint32_t *touched, const void *const *outboxes, int n_ranks, nts_vid_t capacity,
                                  nts_vid_t row_lo, nts_vid_t row_hi, nts_vid_t pitch, nts_vid_t feature_size,
                                  float weight_decay, float beta1, float beta2, float alpha, float epsilon,
                                  void *stream) {
  NTS_ARG_CHECK(n_ranks >= 1 && n_ranks <= kMaxShards, "nts_embedding_step: n_ranks must be in [1, 32]");
  NTS_ARG_CHECK(row_lo <= row_hi, "nts_embedding_step: row_lo > row_hi");
  if (row_lo == row_hi)
    return 0;
  NTS_ARG_CHECK(feature_size > 0 && pitch % 4 == 0 && pitch >= feature_size,
                "nts_embedding_step: pitch must be a multiple of 4 and >= feature_size > 0");
  NTS_ARG_CHECK(rows && adam_m && adam_v && mask && positions && touched && outboxes,
                "null pointer passed to nts_embedding_step");
  NTS_ARG_CHECK(aligned_to(rows, 16) && aligned_to(adam_m, 16) && aligned_to(adam_v, 16),
                "nts_embedding_step: rows, M and V must be 16-byte aligned");
  cudaStream_t st = as_stream(stream);
  const unsigned grid = (unsigned)(sm_count() * kBlocksPerSm);
  NTS_CUDA_OK(cudaMemsetAsync(touched, 0, sizeof(uint32_t), st));
  embedding_mark_kernel<<<grid, kThreads, 0, st>>>(outboxes, n_ranks, row_lo, row_hi, mask, positions, touched);
  NTS_LAUNCH_CHECK();
  const uint32_t nvec = (feature_size + 3) / 4;
  auto run = nvec > 16 ? launch_update<32> : nvec > 8 ? launch_update<16> : nvec > 4 ? launch_update<8>
                                                                                   : launch_update<4>;
  run(grid, st, rows, adam_m, adam_v, mask, positions, touched, outboxes, n_ranks, capacity, pitch, feature_size,
      weight_decay, beta1, beta2, alpha, epsilon);
  NTS_LAUNCH_CHECK();
  return 0;
}
