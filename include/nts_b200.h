/* nts_b200.h - C ABI of libnts_b200.so: NeutronStar's sparse neighbour-aggregation hot path,
 * hand-written for NVIDIA H100 (sm_90a).
 *
 * This is the drop-in boundary.  Every entry point replaces one member of the reference's device
 * interface `cuda/ntsCUDA.hpp` (free functions :25-47, `deviceCSC` :49-95, `Cuda_Stream` :97-217,
 * implemented by `cuda/ntsCUDAGraphOP.cu`); the reference interface it stands in for is cited at
 * each declaration.  The C++ surface of that header (class `Cuda_Stream`, ...) is provided on top
 * of this ABI by `include/nts_cuda_compat.hpp` so the reference's host code links unchanged - see
 * INTEGRATION.md.
 *
 * Conventions
 *  - plain pointers and sizes; all device pointers are CUDA device (or mapped/peer) addresses,
 *    `stream` is a `cudaStream_t` passed as `void*` (NULL = the legacy default stream);
 *  - feature matrices are row-major contiguous float32 [rows, feature_size], borrowed, never
 *    re-laid-out (the reference borrows torch storage the same way, core/NtsScheduler.hpp:505-515);
 *  - vertex ids / offsets are uint32 (`VertexId_CUDA`, cuda/cuda_type.h:21); all address
 *    arithmetic is 64-bit (the reference's 32-bit `feature_size*batch_size` products overflow for
 *    V*F >= 2^32, cuda/ntsCUDAFuseKernel.cuh:280,299);
 *  - aggregation kernels ACCUMULATE into `output` (caller zeroes), exactly like the reference
 *    (cuda/ntsCUDAFuseKernel.cuh:272-309; tensors come zero-filled from NtsScheduler::NewKeyTensor);
 *  - every call is asynchronous on `stream` unless stated; launch errors are checked;
 *  - return value: 0 on success, otherwise the cudaError_t (or -1 for argument errors).  The
 *    message is available from nts_last_error().  With NTS_B200_ABORT_ON_ERROR=1 in the
 *    environment the library prints the message and exit(1)s instead - the reference's convention
 *    (cuda/ntsCUDAGraphOP.cu:13-19).
 *  - there is no CPU fallback anywhere in this library.
 */
#ifndef NTS_B200_H
#define NTS_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef uint32_t nts_vid_t; /* VertexId_CUDA, cuda/cuda_type.h:21 */

/* ---- library / device ----------------------------------------------------------------------- */
int nts_version(void);                 /* ABI version, currently 1 */
const char *nts_last_error(void);      /* thread-local text of the last failure */
int nts_device_count(void);
int nts_set_device(int device);        /* the reference never calls cudaSetDevice (always device 0) */
int nts_device_sm_count(int *sm_count);
int nts_device_synchronize(void);      /* ::CUDA_DEVICE_SYNCHRONIZE(), ntsCUDA.hpp:46 */
int nts_device_reset(void);            /* ::ResetDevice(), ntsCUDA.hpp:47 */

/* ---- memory (ntsCUDA.hpp:25-45) ---------------------------------------------------------------- */
void *nts_malloc_device(size_t bytes);            /* ::cudaMallocGPU / allocate_gpu_buffer / allocate_gpu_edge */
int nts_free_device(void *ptr);                   /* ::FreeBuffer / ::FreeEdge */
void *nts_malloc_pinned(size_t bytes);            /* ::cudaMallocPinned (cudaHostAllocMapped) */
int nts_free_pinned(void *ptr);                   /* ::ntsFreeHost */
void *nts_pinned_device_pointer(void *host_ptr);  /* ::getDevicePointer */
int nts_memcpy_h2d(void *dst_device, const void *src_host, size_t bytes, void *stream, int sync);
                                                  /* ::move_data_in / move_edge_in / move_bytes_in */
int nts_memcpy_d2h(void *dst_host, const void *src_device, size_t bytes, void *stream, int sync);
                                                  /* ::move_result_out */
int nts_memcpy_d2d(void *dst_device, const void *src_device, size_t bytes, void *stream);
int nts_zero(void *device_ptr, size_t bytes, void *stream); /* ::zero_buffer */

/* ---- streams / events (Cuda_Stream ctor, destory_Stream, CUDA_DEVICE_SYNCHRONIZE; ntsCUDA.hpp:97-103) */
void *nts_stream_create(int non_blocking);
int nts_stream_destroy(void *stream);
int nts_stream_synchronize(void *stream);
void *nts_event_create(int with_timing);
int nts_event_destroy(void *event);
int nts_event_record(void *event, void *stream);
int nts_stream_wait_event(void *stream, void *event);
int nts_event_elapsed_ms(void *start, void *stop, float *ms);

/* ---- the hot path: segmented weighted gather-sum (SpMM-like) --------------------------------------
 * output[r, :] += sum_{e in [offsets[r], offsets[r+1])} input[indices[e] - index_base, :] * (weight ? weight[e] : 1)
 *
 * Forward  = Cuda_Stream::Gather_By_Dst_From_Src[_Optim] (ntsCUDA.hpp:125-138, ntsCUDAGraphOP.cu:157-211):
 *            offsets = column_offset[Vdst+1], indices = row_indices (GLOBAL source ids), index_base = src_start.
 * Backward = Cuda_Stream::Gather_By_Src_From_Dst[_Optim] (ntsCUDA.hpp:139-152, ntsCUDAGraphOP.cu:213-281):
 *            offsets = row_offset[Vsrc+1], indices = column_indices (GLOBAL destination ids), index_base = dst_start.
 * The two named wrappers keep the reference's parameter list (minus the unused tensor_weight flag).
 */
int nts_segment_gather_sum(const float *input, float *output, const float *weight,
                           const nts_vid_t *indices, const nts_vid_t *offsets, nts_vid_t index_base,
                           nts_vid_t n_rows, uint64_t n_edges, nts_vid_t feature_size, void *stream);

int nts_gather_by_dst_from_src(const float *input, float *output, const float *weight_forward,
                               const nts_vid_t *row_indices, const nts_vid_t *column_offset,
                               nts_vid_t src_start, nts_vid_t src_end, nts_vid_t dst_start,
                               nts_vid_t dst_end, nts_vid_t edges, nts_vid_t batch_size,
                               nts_vid_t feature_size, int with_weight, void *stream);

int nts_gather_by_src_from_dst(const float *input, float *output, const float *weight_backward,
                               const nts_vid_t *row_offset, const nts_vid_t *column_indices,
                               nts_vid_t src_start, nts_vid_t src_end, nts_vid_t dst_start,
                               nts_vid_t dst_end, nts_vid_t edges, nts_vid_t batch_size,
                               nts_vid_t feature_size, int with_weight, void *stream);

/* Row-range launch of the same contraction: `offsets` points at the first row of the range (offsets[0] ==
 * edge_begin, offsets[n_rows] == edge_end), `output` at its first output row; indices / weight stay the whole
 * arrays (addressed by absolute edge position), row(e) = slot_of ? slot_of[indices[e]] : indices[e] - index_base.
 * Output rows outside the range are not touched, so a chunk can be aggregated one block of rows at a time. */
int nts_segment_gather_sum_range(const float *input, float *output, const float *weight, const nts_vid_t *indices,
                                 const nts_vid_t *offsets, const nts_vid_t *slot_of, nts_vid_t index_base,
                                 nts_vid_t n_rows, uint64_t edge_begin, uint64_t edge_end, nts_vid_t feature_size,
                                 void *stream);

/* K1 on BF16 rows with FP32 accumulation: output[r, 0:F] += sum_e weight[e] * float(input[indices[e], 0:F]) (weight
 * NULL: 1), F = feature_size.  `input` holds BF16 rows of stride input_ld values (input_ld % 8 == 0, >= F, 16-byte
 * aligned; columns F..input_ld-1 are never added); `output` is FP32 [n_rows, F] contiguous.  Accumulates like
 * nts_segment_gather_sum (rows cut by edge quanta finish with atomics); row addresses are 64-bit.  The layout
 * conditions are checked first; n_rows == 0 or n_edges == 0 then launches nothing.  FP32 operands are rounded with
 * nts_rows_to_bf16. */
int nts_segment_gather_sum_bf16(const void *input, nts_vid_t input_ld, float *output, const float *weight,
                                const nts_vid_t *indices, const nts_vid_t *offsets, nts_vid_t n_rows, uint64_t n_edges,
                                nts_vid_t feature_size, void *stream);

/* ---- preprocessed aggregation: nts_gather_plan --------------------------------------------------------------------
 * The arrays of one chunk direction (CSC: column_offset / row_indices / edge_weight_forward; CSR: row_offset /
 * column_indices / edge_weight_backward; core/GraphSegment.h:52-139) regrouped ONCE on the device for repeated
 * aggregation: edges bucketed by (slab of the gathered row, output row) with a stable sort so that one slab of the
 * feature matrix stays L2-resident per launch, (row, weight) stored as interleaved pairs, gathers from 16-byte
 * aligned (padded) rows.  The reference has no counterpart (its chunks are consumed as built); results equal
 * nts_segment_gather_sum up to fp32 re-association across slabs.  `gather_rows` = rows of the gathered matrix
 * (every mapped index must be < gather_rows); n_slabs = 0/1 disables the bucketing (pairs only).
 * The plan owns copies of everything it needs: the input arrays may be released after create returns
 * (create synchronises `stream`). */
typedef struct nts_gather_plan nts_gather_plan;
int nts_gather_plan_pick_slabs(nts_vid_t gather_rows, uint64_t n_edges, nts_vid_t n_rows, nts_vid_t feature_size,
                               uint64_t l2_budget_bytes /* 0 = default */);
/* A plan of one chunk with up to two dense FP32 hub blocks beside the slab-bucketed residual: the n_hub_cols most
 * referenced gathered rows (ties: smaller id) become a column block [n_rows x n_hub_cols] that takes every edge
 * gathering one of them, the n_hub_rows longest output rows a row block [n_hub_rows x gather_rows] that takes their
 * remaining edges; each dense cell holds the sum of its edges' weights.  A run computes the blocks as GEMMs before the
 * slab launches.  Counts above the rows available are clamped (nts_gather_plan_hubs reports the result); 0, 0 = no
 * hub blocks. */
nts_gather_plan *nts_gather_plan_create_hybrid(const nts_vid_t *offsets, const nts_vid_t *indices,
                                               const float *weight, const nts_vid_t *slot_of, nts_vid_t index_base,
                                               nts_vid_t n_rows, uint64_t n_edges, nts_vid_t gather_rows, int n_slabs,
                                               int n_hub_cols, int n_hub_rows, void *stream);
/* A plan of one chunk with the slab count chosen by MEASUREMENT on the real arrays at this feature width (candidates
 * 1, 2, 4, ... built and timed once; hub-dominated graphs prefer no bucketing, uniform ones 8-16 slabs), then the hub
 * counts of nts_gather_plan_create_hybrid the same way among rows dense enough to be candidates (NTS_PLAN_HUBS=0:
 * none).  The candidates are timed as gathers of gather_dtype: NTS_DTYPE_F32, or NTS_DTYPE_BF16 (BF16 rows; the L2
 * slab bound counts 2-byte rows), in the run mode the plan will be used in: run_flags 0 (accumulate) or
 * NTS_PLAN_OVERWRITE. */
nts_gather_plan *nts_gather_plan_create_tuned_ex(const nts_vid_t *offsets, const nts_vid_t *indices,
                                                 const float *weight, const nts_vid_t *slot_of, nts_vid_t index_base,
                                                 nts_vid_t n_rows, uint64_t n_edges, nts_vid_t gather_rows,
                                                 nts_vid_t feature_size, int gather_dtype, int run_flags,
                                                 void *stream);
/* Several chunks merged into ONE plan: part-local output row r becomes row_add + r, a mapped index g becomes index_add
 * + g; inside a (slab, row) segment the parts follow each other in the order given.  n_slabs = 0 measures the slab
 * count for feature_size on accumulating FP32 gathers.  Merged plans have no hub blocks.  Used by the exchange engine
 * to aggregate all remote chunks of a rank in one launch. */
typedef struct nts_plan_part {
  const nts_vid_t *offsets, *indices;   /* [n_rows+1], [n_edges] of this part */
  const float *weight;                  /* [n_edges] or NULL */
  const nts_vid_t *slot_of;             /* optional slot table applied to the indices */
  nts_vid_t index_base, index_add, n_rows, row_add;
  uint64_t n_edges;
} nts_plan_part;
nts_gather_plan *nts_gather_plan_create_parts(const nts_plan_part *parts, int n_parts, nts_vid_t n_rows,
                                              nts_vid_t gather_rows, int n_slabs, nts_vid_t feature_size, void *stream);
float nts_gather_plan_tuned_ms(const nts_gather_plan *plan); /* time of the winning candidate of a measured plan */
int nts_gather_plan_destroy(nts_gather_plan *plan);
int nts_gather_plan_slabs(const nts_gather_plan *plan);
int nts_gather_plan_hubs(const nts_gather_plan *plan, int *cols, int *rows); /* hub columns / rows of the plan */
/* Schedule of the hub-row block: 0 = its own launch before the slab launches, 1 = its tiles run inside the slab
 * launches that gather the same rows (it writes only hub rows, which have no residual edges).  Measured plans pick the
 * faster (NTS_PLAN_OVERLAP=0 forces 0); other plans start at 0.  Plans without hub rows ignore it. */
int nts_gather_plan_overlap(const nts_gather_plan *plan);
int nts_gather_plan_set_overlap(nts_gather_plan *plan, int overlap);
uint64_t nts_gather_plan_bytes(const nts_gather_plan *plan);
/* Run flags of the _ex entries.
 * NTS_PLAN_ACCUMULATE (0): output[r,:] += sum_e input[row(e),:] * w(e), one launch per non-empty slab, in stream order.
 * NTS_PLAN_OVERWRITE: output[r,:] = sum_e ... instead of +=; output may hold anything before the call (NaN included).
 *   The hub column block, which covers every output element and runs first, stores instead of adding; a plan without
 *   hub columns zeroes the output first.  Each element gets the value an accumulating run into zeros gives, up to the
 *   sign of a zero.
 * NTS_PLAN_COPY_INPUT: gather from a zero-padded copy of the input even where it could be gathered in place (for an
 *   input whose storage ends before the last row's input_ld-th value). */
enum { NTS_PLAN_ACCUMULATE = 0, NTS_PLAN_OVERWRITE = 1, NTS_PLAN_COPY_INPUT = 2 };
/* Run a plan on input rows of pitch input_ld floats (>= feature_size).  The input is gathered in place when
 * input_ld % 4 == 0 and it is 16-byte aligned: the gather then reads all input_ld values of every row, the last one
 * included, and never writes values past feature_size to an output.  Otherwise its rows are copied into the plan's
 * zero-padded workspace first (the copy reads feature_size values per row).  The output keeps the pitch
 * feature_size.  input_ld < feature_size and a null output are rejected. */
int nts_gather_plan_run_ex(nts_gather_plan *plan, const float *input, nts_vid_t input_ld, float *output,
                           nts_vid_t feature_size, int flags, void *stream);
int nts_gather_plan_last_launch(const nts_gather_plan *plan, int *launches, int *grid, int *k, int *u, int *outv);
/* BF16 gathers with FP32 accumulation: output[r,:] += sum_e w(e) * float(bf16(input[row(e),:])) (or = with
 * NTS_PLAN_OVERWRITE).  bf16() rounds to nearest even (what torch's x.to(torch.bfloat16) computes, incl. inf, NaN and
 * subnormals); weights, accumulation and output stay FP32.  Input rows of pitch input_ld elements of input_dtype:
 * an NTS_DTYPE_F32 input is converted once per call into the plan's BF16 workspace (rows padded to a multiple of 8
 * values); an NTS_DTYPE_BF16 input is gathered in place when input_ld % 8 == 0 and it is 16-byte aligned, else
 * re-strided into the workspace.  Flags as for nts_gather_plan_run_ex.  Hub blocks read BF16 rows and compute in
 * FP32.  Returns an error under nts_gather_plan_set_variant(1) (the TMA row-staging variant is FP32 only). */
enum { NTS_DTYPE_F32 = 0, NTS_DTYPE_BF16 = 1 };
int nts_gather_plan_run_bf16_ex(nts_gather_plan *plan, const void *input, int input_dtype, nts_vid_t input_ld,
                                float *output, nts_vid_t feature_size, int flags, void *stream);
int nts_gather_plan_set_tuning(int u, int min_blocks, int edges_per_warp); /* measurement hook, 0 = default */
/* 0 = gathered rows through registers (default); 1 = rows staged in shared memory by per-row cp.async.bulk (TMA) into
 * a per-warp ring, U of set_tuning = ring depth - the north star's "feature tiles via TMA", kept for measurement */
int nts_gather_plan_set_variant(int variant);

/* Same contraction with the source row taken through a slot table instead of `index - base`:
 * row = slot_of[indices[e]].  Used with MirrorIndex (core/PartitionedGraph.hpp:295-305) for the fused
 * GAT aggregation, DistAggregateDstFuseWeight::forward (core/ntsDistCPUGraphOp.hpp:516-546), and with
 * the compact receive-staging slots of the multi-GPU exchange. */
int nts_segment_gather_sum_slots(const float *input, float *output, const float *weight,
                                 const nts_vid_t *indices, const nts_vid_t *offsets,
                                 const nts_vid_t *slot_of, nts_vid_t n_rows, uint64_t n_edges,
                                 nts_vid_t feature_size, void *stream);

/* Multi-head fused GAT aggregation: weight is [n_edges, heads] row-major, feature_size = heads * D and head h scales
 * columns [h*D, (h+1)*D):  output[r, hD+c] += sum_e weight[e,h] * input[row(e), hD+c],  row(e) = slot_of ?
 * slot_of[indices[e]] : indices[e] - index_base.  heads = 1 is the single-head operator above.  (The reference's
 * DistAggregateDstFuseWeight has one head; 8 heads is config D of BASELINE.json.) */
int nts_segment_gather_sum_heads(const float *input, float *output, const float *weight,
                                 const nts_vid_t *indices, const nts_vid_t *offsets, const nts_vid_t *slot_of,
                                 nts_vid_t index_base, nts_vid_t n_rows, uint64_t n_edges,
                                 nts_vid_t feature_size, nts_vid_t heads, void *stream);

/* Tuning / introspection of the aggregation kernel (does not change results beyond fp32
 * re-association): variant 0 = auto, see DESIGN.md "kernel variants". */
int nts_aggregate_set_variant(int variant, int edges_per_warp);
int nts_aggregate_last_launch(int *grid, int *block, int *smem_bytes, int *variant);
/* Template point of the last launch: floats (BF16 values for the BF16 fused GAT forward and
 * nts_segment_gather_sum_bf16) per vector load, vector chunks per lane, edges loaded before their FMAs (U),
 * __launch_bounds__ minimum CTAs per SM, and column tiles.  Virtual warps show in nts_aggregate_last_launch's grid. */
int nts_aggregate_last_shape(int *vec, int *k, int *u, int *min_blocks, int *tiles);
uint64_t nts_kernel_launch_count(void); /* kernels launched by this library since load */

/* ---- edge-granular operators (GAT building blocks) -------------------------------------------------
 * All take the whole-partition CSC of core/PartitionedGraph.hpp:105-143 (column_offset[Vp+1], row_indices[Ep]
 * global source ids) as uploaded by `deviceCSC` (ntsCUDA.hpp:49-95). `batch_size` = Vp. */
/* msg[e,:] = mirror[mirror_index[row_indices[e]],:]      Cuda_Stream::Scatter_Src_Mirror_to_Msg (ntsCUDA.hpp:154) */
int nts_scatter_src_mirror_to_msg(float *message, const float *src_mirror_feature,
                                  const nts_vid_t *row_indices, const nts_vid_t *column_offset,
                                  const nts_vid_t *mirror_index, nts_vid_t batch_size,
                                  nts_vid_t feature_size, void *stream);
/* mirror_grad[mirror_index[row_indices[e]],:] += msg[e,:]  Cuda_Stream::Gather_Msg_To_Src_Mirror (ntsCUDA.hpp:159) */
int nts_gather_msg_to_src_mirror(float *src_mirror_feature, const float *message,
                                 const nts_vid_t *row_indices, const nts_vid_t *column_offset,
                                 const nts_vid_t *mirror_index, nts_vid_t batch_size,
                                 nts_vid_t feature_size, void *stream);
/* msg[e,:] = dst_feature[dst(e),:]                         Cuda_Stream::Scatter_Dst_to_Msg (ntsCUDA.hpp:164) */
int nts_scatter_dst_to_msg(float *message, const float *dst_feature, const nts_vid_t *row_indices,
                           const nts_vid_t *column_offset, nts_vid_t batch_size,
                           nts_vid_t feature_size, void *stream);
/* dst_feature[d,:] += sum_{e->d} msg[e,:]                  Cuda_Stream::Gather_Msg_to_Dst (ntsCUDA.hpp:168) */
int nts_gather_msg_to_dst(float *dst_feature, const float *message, const nts_vid_t *row_indices,
                          const nts_vid_t *column_offset, nts_vid_t batch_size,
                          nts_vid_t feature_size, void *stream);
/* a[seg,h] = softmax_seg(m[seg,h]) per destination segment and column h (max-subtracted; oracle =
 * DistEdgeSoftMax::forward core/ntsDistCPUGraphOp.hpp:449-470); msg_cached receives a copy.
 * Cuda_Stream::Edge_Softmax_Forward_Block (ntsCUDA.hpp:172) - the reference kernel handles 1 column only. */
int nts_edge_softmax_forward(float *msg_output, const float *msg_input, float *msg_cached,
                             const nts_vid_t *row_indices, const nts_vid_t *column_offset,
                             nts_vid_t batch_size, nts_vid_t feature_size, void *stream);
/* g_in[e,h] = a[e,h]*g[e,h] - a[e,h]*sum_seg(g*a)            Cuda_Stream::Edge_Softmax_Backward_Block (ntsCUDA.hpp:177) */
int nts_edge_softmax_backward(float *msg_input_grad, const float *msg_output_grad,
                              const float *msg_cached, const nts_vid_t *row_indices,
                              const nts_vid_t *column_offset, nts_vid_t batch_size,
                              nts_vid_t feature_size, void *stream);
/* message_grad[e,:] += input[dst(e),:]                     Cuda_Stream::Scatter_Grad_Back_To_Message (ntsCUDA.hpp:194) */
int nts_scatter_grad_back_to_message(const float *input, float *message_grad,
                                     const nts_vid_t *row_indices, const nts_vid_t *column_offset,
                                     nts_vid_t batch_size, nts_vid_t feature_size, void *stream);

/* Fused GAT aggregation backward, DistAggregateDstFuseWeight::backward (core/ntsDistCPUGraphOp.hpp:548-589)
 * WITHOUT the reference's spurious extra unweighted add (:572):
 *   mirror_grad[slot(e),:] += a[e] * g[dst(e),:]        (needs mirror_grad zeroed by the caller)
 *   a_grad[e]               = < mirror[slot(e),:], g[dst(e),:] >  */
int nts_aggregate_dst_fuse_weight_backward(float *mirror_grad, float *edge_weight_grad,
                                           const float *mirror, const float *edge_weight,
                                           const float *dst_grad, const nts_vid_t *row_indices,
                                           const nts_vid_t *column_offset,
                                           const nts_vid_t *mirror_index, nts_vid_t batch_size,
                                           nts_vid_t feature_size, void *stream);
/* multi-head form: edge_weight / edge_weight_grad are [E, heads], head h owns columns [h*D, (h+1)*D) */
int nts_aggregate_dst_fuse_weight_backward_heads(float *mirror_grad, float *edge_weight_grad,
                                                 const float *mirror, const float *edge_weight,
                                                 const float *dst_grad, const nts_vid_t *row_indices,
                                                 const nts_vid_t *column_offset,
                                                 const nts_vid_t *mirror_index, nts_vid_t batch_size,
                                                 nts_vid_t feature_size, nts_vid_t heads, void *stream);

/* ---- fully fused GAT layer (K7): edge logits / attention are never materialised ---------------------------------
 * The flow of toolkits/GAT_CPU_DIST_OPTM.hpp:196-241 (per-vertex scores -> leaky_relu -> edge softmax ->
 * DistAggregateDstFuseWeight) with a[e,h] = softmax_seg(leaky_relu(src_score[slot(e),h] + dst_score[dst(e),h]))
 * recomputed inside the kernels; slot(e) = mirror_index[row_indices[e]] (or row_indices[e] itself when mirror_index
 * is NULL, i.e. the caller has applied the lookup once), head h owns columns [h*D,(h+1)*D), D <= 512.
 *   stats    : seg_max[d,h], seg_sum[d,h]                                   ([batch_size, heads] each)
 *   forward  : output[d, hD+c] += sum_e a[e,h] * mirror[slot(e), hD+c]
 *   backward : mirror_grad[slot,hD+c] += a*g[d,hD+c];  src_score_grad[slot,h] += dpre;  dst_score_grad[d,h] += dpre
 *              with dpre = a*(<mirror[slot,h],g[d,h]> - out_dot_grad[d,h]) * leaky_relu'(pre) and
 *              out_dot_grad[d,h] = <output[d,h], g[d,h]> supplied by the caller (a per-vertex dot product).
 *   The three gradient outputs must be zeroed by the caller. */
int nts_gat_softmax_stats(float *seg_max, float *seg_sum, const float *src_score, const float *dst_score,
                          const nts_vid_t *row_indices, const nts_vid_t *column_offset,
                          const nts_vid_t *mirror_index, nts_vid_t batch_size, nts_vid_t heads,
                          float negative_slope, void *stream);
int nts_gat_fused_aggregate_forward(const float *mirror, float *output, const float *src_score,
                                    const float *dst_score, const float *seg_max, const float *seg_sum,
                                    const nts_vid_t *row_indices, const nts_vid_t *column_offset,
                                    const nts_vid_t *mirror_index, nts_vid_t batch_size, uint64_t n_edges,
                                    nts_vid_t feature_size, nts_vid_t heads, float negative_slope, void *stream);
int nts_gat_fused_aggregate_backward(float *mirror_grad, float *src_score_grad, float *dst_score_grad,
                                     const float *mirror, const float *src_score, const float *dst_score,
                                     const float *seg_max, const float *seg_sum, const float *out_dot_grad,
                                     const float *dst_grad, const nts_vid_t *row_indices,
                                     const nts_vid_t *column_offset, const nts_vid_t *mirror_index,
                                     nts_vid_t batch_size, nts_vid_t feature_size, nts_vid_t heads,
                                     float negative_slope, void *stream);
/* Same results without per-edge atomics: a destination-major pass over the CSC (dst_score_grad) and a source-major
 * pass over the CSR of the same edges keyed by MIRROR SLOT (mirror_grad, src_score_grad), both with register
 * accumulators.  slot_row_offset[mirror_size+1] / slot_column_indices[E] (local destination ids) list the out-edges
 * of every mirror slot; dst_pack is a 16-byte-aligned workspace of batch_size*heads*4 floats.  Shapes the passes do
 * not cover (heads > 1 with a non-power-of-two head width in vectors, rows wider than 128 vectors) fall back to
 * nts_gat_fused_aggregate_backward.  The three gradient outputs must be zeroed by the caller. */
int nts_gat_fused_aggregate_backward_two_pass(float *mirror_grad, float *src_score_grad, float *dst_score_grad,
                                              float *dst_pack, const float *mirror, const float *src_score,
                                              const float *dst_score, const float *seg_max, const float *seg_sum,
                                              const float *out_dot_grad, const float *dst_grad,
                                              const nts_vid_t *row_indices, const nts_vid_t *column_offset,
                                              const nts_vid_t *mirror_index, const nts_vid_t *slot_row_offset,
                                              const nts_vid_t *slot_column_indices, nts_vid_t batch_size,
                                              nts_vid_t mirror_size, nts_vid_t feature_size, nts_vid_t heads,
                                              float negative_slope, void *stream);
/* K7 with BF16 gathers and FP32 accumulation.  With m~ = bf16(mirror) and g~ = bf16(grad_out) (round to nearest even,
 * as torch's x.to(torch.bfloat16)) the layer computes the FP32 layer's function and gradients at the rounded operands:
 *   forward  : output[d, hD+c] += sum_e a[e,h] * m~[slot(e), hD+c]      (a from the FP32 scores and statistics)
 *   backward : mirror_grad[slot] += a*g~[d];  dpre = a*(<m~[slot,h], g~[d,h]> - out_dot_grad[d,h]) * leaky_relu'(pre)
 *              with out_dot_grad[d,h] = <output[d,h], g~[d,h]> (g~, not grad_out: the two passes rely on
 *              sum_e a*<m~, g~> = <output, g~>).
 * BF16 rows (mirror, dst_grad) have ld values each: ld % 8 == 0, ld >= feature_size, columns past feature_size zero;
 * with heads > 1, D = feature_size / heads must be a multiple of 8 and ld == feature_size.  The FP32 output and
 * mirror_grad have the same row stride ld.  Scores, statistics, dst_pack and the score gradients are FP32.  mirror,
 * output, mirror_grad, dst_grad, dst_pack and row_indices must be 16-byte aligned.  The backward additionally needs a
 * power-of-two number of vectors per head and rows of at most 1024 values; there is no fallback: other shapes return
 * an error.  The gradient outputs must be zeroed by the caller. */
int nts_gat_fused_aggregate_forward_bf16(const void *mirror, float *output, const float *src_score,
                                         const float *dst_score, const float *seg_max, const float *seg_sum,
                                         const nts_vid_t *row_indices, const nts_vid_t *column_offset,
                                         const nts_vid_t *mirror_index, nts_vid_t batch_size, uint64_t n_edges,
                                         nts_vid_t feature_size, nts_vid_t ld, nts_vid_t heads, float negative_slope,
                                         void *stream);
int nts_gat_fused_aggregate_backward_two_pass_bf16(float *mirror_grad, float *src_score_grad, float *dst_score_grad,
                                                   float *dst_pack, const void *mirror, const float *src_score,
                                                   const float *dst_score, const float *seg_max, const float *seg_sum,
                                                   const float *out_dot_grad, const void *dst_grad,
                                                   const nts_vid_t *row_indices, const nts_vid_t *column_offset,
                                                   const nts_vid_t *mirror_index, const nts_vid_t *slot_row_offset,
                                                   const nts_vid_t *slot_column_indices, nts_vid_t batch_size,
                                                   nts_vid_t mirror_size, nts_vid_t feature_size, nts_vid_t ld,
                                                   nts_vid_t heads, float negative_slope, void *stream);
/* dst[r, 0:ld] = {bf16(src[r, 0:feature_size]), 0 ...} for n_rows rows of stride lds (elements of src_dtype,
 * NTS_DTYPE_F32 rounded to nearest even, NTS_DTYPE_BF16 copied); ld % 8 == 0, ld >= feature_size, dst 16-byte aligned.
 * The conversion pass of nts_gather_plan_run_bf16_ex, exported for the BF16 rows of the K7 entries above. */
int nts_rows_to_bf16(const void *src, int src_dtype, nts_vid_t lds, void *dst, nts_vid_t n_rows, nts_vid_t feature_size,
                     nts_vid_t ld, void *stream);

/* ---- (vid,row) message records: the reference's host-staged exchange format (comm/network.h:143-149) ---
 * record k = { uint32 vid; float row[feature_size]; }, read through mapped pinned host memory. */
/* mirror[vid - partition_start,:] = record.row if vid in [partition_start, partition_end)
 * Cuda_Stream::deSerializeToGPU (ntsCUDA.hpp:113, ntsCUDATransferKernel.cuh:70-93) */
int nts_deserialize_records(float *mirror, const float *records, nts_vid_t n_records,
                            nts_vid_t feature_size, nts_vid_t partition_start,
                            nts_vid_t partition_end, void *stream);
/* Y[vid - partition_start,:] += record.row
 * Cuda_Stream::aggregate_comm_result_debug (ntsCUDA.hpp:117, ntsCUDATransferKernel.cuh:49-68) */
int nts_aggregate_records(float *aggregate, const float *records, nts_vid_t n_records,
                          nts_vid_t feature_size, nts_vid_t partition_start,
                          nts_vid_t partition_end, void *stream);

/* ---- dense-row exchange helpers of the exchange engine (replace the record format on NVLink) ----------- */
/* dst[k,:] = src[rows[k],:]   (sender-side compaction of mirror rows / pull from a peer's mapped buffer) */
int nts_gather_rows(float *dst, const float *src, const nts_vid_t *rows, nts_vid_t n_rows,
                    nts_vid_t feature_size, void *stream);
/* dst[k,:] = shards[o][ids[k] - shard_offsets[o], :feature_size] for k < n, o the shard that owns ids[k]: a gather by
 * global row id from a table split into n_shards (1..32) row ranges [shard_offsets[o], shard_offsets[o+1]) (device
 * array of n_shards+1 non-decreasing values; empty shards allowed), shard o stored at `shards[o]` (device array of
 * pointers, local or peer memory, each 16-byte aligned) with shard_pitch floats per row (shard_pitch % 4 == 0,
 * >= feature_size).  dst is [n, feature_size] contiguous.  Ids may repeat and come in any order; every id must lie in
 * [shard_offsets[0], shard_offsets[n_shards]) (not checked on the device).  n == 0 launches nothing. */
int nts_gather_rows_sharded(float *dst, const float *const *shards, const nts_vid_t *shard_offsets, int n_shards,
                            nts_vid_t shard_pitch, const nts_vid_t *ids, nts_vid_t n, nts_vid_t feature_size,
                            void *stream);
/* The same gather from BF16 shards: shard rows of shard_pitch BF16 values (shard_pitch % 8 == 0, >= feature_size; every
 * shard 16-byte aligned), read 16 bytes at a time.  dst_dtype NTS_DTYPE_BF16: dst holds BF16 rows of stride dst_ld
 * (dst_ld % 8 == 0, >= feature_size, dst 16-byte aligned) and gets a plain copy of columns [0, 8*ceil(F/8)) (the
 * columns past feature_size get the shard's pad values, later columns are not written).  NTS_DTYPE_F32: dst is FP32
 * [n, feature_size] contiguous (dst_ld == feature_size) and gets the rows widened exactly.  Ids as above; n == 0
 * launches nothing. */
int nts_gather_rows_sharded_bf16(void *dst, int dst_dtype, nts_vid_t dst_ld, const void *const *shards,
                                 const nts_vid_t *shard_offsets, int n_shards, nts_vid_t shard_pitch,
                                 const nts_vid_t *ids, nts_vid_t n, nts_vid_t feature_size, void *stream);
/* K9: the weighted gather-sum of K1 with its sources read by global id from a sharded table:
 * output[r, :F] += sum_{e in [offsets[r], offsets[r+1])} w(e) * row(indices[e]) for r < n_rows (w = weight[e], or 1
 * when weight is NULL), row(g) = row g - shard_offsets[o] of shards[o] for the shard o that owns g.  Shards as for
 * nts_gather_rows_sharded (1..32 row ranges, empty ones allowed, each 16-byte aligned) with rows of shard_pitch values
 * of shard_dtype: NTS_DTYPE_F32 (shard_pitch % 4 == 0) or NTS_DTYPE_BF16 (shard_pitch % 8 == 0, widened exactly,
 * FP32 accumulation); shard_pitch >= F, and columns past F are never added.  `offsets` holds absolute edge positions
 * (offsets[0] == edge_begin, offsets[n_rows] == edge_end), and indices / weight are addressed by absolute edge
 * position, as for nts_segment_gather_sum_range; every index must lie in [shard_offsets[0], shard_offsets[n_shards])
 * (not checked on the device).  `output` is FP32 [n_rows, F] contiguous, zeroed by the caller.  Work is split by
 * edges; rows cut by an edge quantum finish with atomics.  n_rows == 0 or an empty edge range launches nothing and
 * looks at no pointer; layout errors return an error and launch nothing. */
int nts_segment_gather_sum_sharded(float *output, const void *const *shards, int shard_dtype,
                                   const nts_vid_t *shard_offsets, int n_shards, nts_vid_t shard_pitch,
                                   const float *weight, const nts_vid_t *indices, const nts_vid_t *offsets,
                                   nts_vid_t n_rows, uint64_t edge_begin, uint64_t edge_end, nts_vid_t feature_size,
                                   void *stream);
/* K10: full-neighbour GAT attention over a sharded table, for the destinations r < n_rows of a CSC piece addressed as
 * for K9 (offsets[0] == edge_begin, offsets[n_rows] == edge_end, indices by absolute edge position, global ids).  The
 * sources' scores s[g, h] are FP32 rows of score_pitch values (score_pitch >= heads, % 4 == 0) in score_shards, which
 * share the row shards' shard_offsets (1..32 ranges), so one shard search per edge serves both; dst_score is the
 * local [n_rows, heads] d[r, h].  logit(e, h) = leaky_relu(s[indices[e], h] + d[r, h], negative_slope).
 * nts_gat_softmax_stats_sharded writes seg_max[r, h] = max_e logit and seg_sum[r, h] = sum_e exp(logit - seg_max)
 * ([n_rows, heads] FP32; empty segments get (0, 1)); heads must divide 32.  n_rows == 0 launches nothing and looks at
 * no pointer; an empty edge range only writes (0, 1).
 * nts_gat_aggregate_sharded adds output[r, h*D:(h+1)*D] += sum_e a(e, h) * row(indices[e])[h*D:(h+1)*D], with
 * a = exp(logit - seg_max) / seg_sum and D = feature_size / heads, rows as for K9 (FP32, or BF16 widened exactly with
 * FP32 accumulation).  Every 16-byte load must lie inside one head: with heads > 1, D % 4 == 0 (FP32) or D % 8 == 0
 * (BF16).  output is FP32 [n_rows, feature_size] contiguous, zeroed by the caller.  n_rows == 0, an empty edge range
 * or feature_size == 0 launches nothing and looks at no pointer.  For both, layout errors return an error and launch
 * nothing, and edge positions must fit uint32. */
int nts_gat_softmax_stats_sharded(float *seg_max, float *seg_sum, const void *const *score_shards,
                                  const nts_vid_t *shard_offsets, int n_shards, nts_vid_t score_pitch,
                                  const float *dst_score, const nts_vid_t *indices, const nts_vid_t *offsets,
                                  nts_vid_t n_rows, uint64_t edge_begin, uint64_t edge_end, nts_vid_t heads,
                                  float negative_slope, void *stream);
int nts_gat_aggregate_sharded(float *output, const void *const *shards, int shard_dtype,
                              const nts_vid_t *shard_offsets, int n_shards, nts_vid_t shard_pitch,
                              const void *const *score_shards, nts_vid_t score_pitch, const float *dst_score,
                              const float *seg_max, const float *seg_sum, const nts_vid_t *indices,
                              const nts_vid_t *offsets, nts_vid_t n_rows, uint64_t edge_begin, uint64_t edge_end,
                              nts_vid_t feature_size, nts_vid_t heads, float negative_slope, void *stream);
/* dst[rows[k],:] += src[k,:]  (receiver-side add of partial gradients; rows must be unique) */
int nts_scatter_add_rows(float *dst, const float *src, const nts_vid_t *rows, nts_vid_t n_rows,
                         nts_vid_t feature_size, void *stream);
/* same with vector red.global.add: rows may repeat (partials of several senders merged into one launch) */
int nts_scatter_add_rows_atomic(float *dst, const float *src, const nts_vid_t *rows, nts_vid_t n_rows,
                                nts_vid_t feature_size, void *stream);

/* ---- parameter update (SURVEY 8 f1) ------------------------------------------------------------------------------------
 * Parameter::learnC2G_with_decay_Adam (core/NtsScheduler.hpp:774-781) as ONE kernel, in place on W / M / V:
 *   W_g = W*weight_decay + grad;  M = beta1*M + (1-beta1)*W_g;  V = beta2*V + (1-beta2)*W_g*W_g;
 *   W  -= alpha * M / (sqrt(V) + epsilon)
 * alpha / beta1 / beta2 are the CURRENT values of the reference's schedule (Parameter::next(), :727-736).  `grad` is the
 * all-reduced gradient (Parameter::all_reduce_to_gradient, :719-722 - ncclAllReduce here instead of .cpu() + MPI). */
int nts_adam_update(float *W, float *M, float *V, const float *grad, uint64_t n, float weight_decay, float beta1,
                    float beta2, float alpha, float epsilon, void *stream);
/* K11: one row-sparse Adam step of an embedding table sharded by row ranges, on the owner of rows [row_lo, row_hi).
 * Every one of the n_ranks (1..32) ranks q has an outbox at outboxes[q] (device array of pointers, local or peer
 * memory, each 16-byte aligned) laid out as: a uint32 count n_q at byte 0; n_q <= capacity strictly ascending global
 * row ids (uint32) from byte 16; n_q gradient rows of `pitch` floats from byte 16 + 16*ceil(capacity/4).  For every
 * row g in [row_lo, row_hi) named by at least one outbox, the gradient is the sum of its contributors' rows in
 * ascending rank order (the first contributor's row plus the next, and so on, in float32), and columns [0,
 * feature_size) of rows[g - row_lo], adam_m[..] and adam_v[..] (rows of `pitch` floats, pitch % 4 == 0, >= feature_size,
 * 16-byte aligned) get nts_adam_update's arithmetic with that gradient, bit for bit; every other row and every pad
 * column keeps its bits.  Scratch of the owner: mask[row_hi - row_lo] (uint32, zero on entry and on return),
 * positions[(row_hi - row_lo) * n_ranks] (uint32) and touched[1 + row_hi - row_lo] (uint32).  Two launches on
 * `stream`, grid-stride over the device-side counts (the host needs no count).  The outboxes must be complete before
 * the step starts and stay unchanged until it ends; no other rank may read rows [row_lo, row_hi) meanwhile.  An empty
 * range launches nothing and looks at no pointer. */
int nts_embedding_step(float *rows, float *adam_m, float *adam_v, uint32_t *mask, uint32_t *positions,
                       uint32_t *touched, const void *const *outboxes, int n_ranks, nts_vid_t capacity,
                       nts_vid_t row_lo, nts_vid_t row_hi, nts_vid_t pitch, nts_vid_t feature_size,
                       float weight_decay, float beta1, float beta2, float alpha, float epsilon, void *stream);

/* ---- peer memory (CUDA IPC) for the NVLink exchange ------------------------------------------------------ */
#define NTS_IPC_HANDLE_BYTES 64
int nts_ipc_get_handle(void *device_ptr, unsigned char handle[NTS_IPC_HANDLE_BYTES]);
void *nts_ipc_open_handle(const unsigned char handle[NTS_IPC_HANDLE_BYTES]);
int nts_ipc_close_handle(void *peer_ptr);
/* cross-GPU flag signalling on IPC-mapped uint32 flags (release/acquire at system scope) */
int nts_signal_set(uint32_t *flag, uint32_t value, void *stream);
int nts_signal_wait_geq(const uint32_t *flag, uint32_t value, void *stream);

/* ---- the exchange engine: data plane of the distributed fused aggregation (peer-memory transport) ---------------------
 * Replaces Graph::sync_compute_decoupled / compute_sync_decoupled (core/graph.hpp:3455-3719) and the host-staged
 * NtsGraphCommunicator (comm/network.cpp:159-844).  PUSH model over CUDA-IPC windows, one pipeline stage per source
 * partition in the reference's ring order (core/graph.hpp:3678-3683): the owner of a row stores it straight into the
 * reader's receive window over NVLink and raises an epoch flag; the reader aggregates chunk (p+s) as soon as the rows
 * of partition (p+s) have landed (csrc/nts_exchange.cu documents the protocol).
 * The caller owns the CONTROL plane: it builds the plan arrays (who needs which rows;
 * neutronstarlite_b200/exchange.py::ExchangePlan or nts_exchange_plan_* below) and moves the two 64-byte IPC handles
 * per rank between processes (torch.distributed here, MPI in the reference's host code); the engine owns windows,
 * flags, streams, events and the launch sequence.  All pointers are device pointers that must outlive the engine;
 * per-partition arrays have `partitions` entries (own entry ignored).  Row layouts ("partition order"): the receive
 * staging of rank r holds the rows it reads from partition 0, 1, ... (r skipped), need_count[i] rows each; the
 * gradient staging holds what ranks 0, 1, ... (r skipped) return, send_count[j] rows each = the order of
 * send_rows_all. */
typedef struct nts_exchange nts_exchange;
typedef struct nts_exchange_chunk {          /* remote chunk i: sources in partition i -> my destinations */
  const nts_vid_t *column_offset;            /* [V_p+1]  graph_chunks[i]->column_offset_gpu */
  const nts_vid_t *slots;                    /* [E_i]    row_indices remapped to 0..need_count[i]-1 (rank in need list) */
  const float *weight_forward;               /* [E_i]    graph_chunks[i]->edge_weight_forward_gpu */
  const nts_vid_t *row_offset_compact;       /* [need_count[i]+1] row_offset restricted to the active sources */
  const nts_vid_t *column_indices;           /* [E_i]    graph_chunks[i]->column_indices_gpu (global destination ids) */
  const float *weight_backward;              /* [E_i]    graph_chunks[i]->edge_weight_backward_gpu */
  uint64_t edges;
} nts_exchange_chunk;
typedef struct nts_exchange_desc {
  int partitions, rank;
  nts_vid_t owned_vertices, dst_start;      /* V_p and partition_offset[rank] */
  /* local chunk (sources in this partition): CSC + CSR of CSC_segment_pinned */
  const nts_vid_t *local_column_offset, *local_row_indices, *local_row_offset, *local_column_indices;
  const float *local_weight_forward, *local_weight_backward;
  nts_vid_t local_edges;
  const nts_exchange_chunk *chunks;         /* [P] remote chunks (host array of device pointers) */
  const nts_vid_t *need_count;              /* [P] rows of partition i that I read (= active sources of chunk i) */
  const nts_vid_t *send_count;              /* [P] rows of mine that rank j reads */
  const nts_vid_t *send_rows_all;           /* device: concatenation over j != rank (ascending) of those local row ids */
  const nts_vid_t *fwd_push_offset;         /* [P] first row of MY rows inside rank j's receive staging */
  const nts_vid_t *bwd_push_offset;         /* [P] first row of MY partials inside rank i's gradient staging */
  /* rows of MY partition that are sources of my own in-edges (active sources of the local chunk, ascending); only
   * the mirror fetch below needs them */
  const nts_vid_t *local_need;              /* device */
  nts_vid_t local_need_count;
} nts_exchange_desc;

nts_exchange *nts_exchange_create(const nts_exchange_desc *desc);
int nts_exchange_destroy(nts_exchange *ex);
/* floats ONE epoch buffer of the receive window needs at this width; take the MAX over ranks before reserving */
uint64_t nts_exchange_required_floats(const nts_exchange *ex, nts_vid_t feature_size);
/* window floats per epoch buffer for BF16 calls of width F (BF16 rows at stride ceil(F/8)*8 forward, FP32 partials
 * backward): reserve this much before nts_exchange_forward_bf16 / nts_exchange_backward_bf16 */
uint64_t nts_exchange_required_floats_bf16(const nts_exchange *ex, nts_vid_t feature_size);
uint64_t nts_exchange_capacity_floats(const nts_exchange *ex);
/* Replacing the exported window is COLLECTIVE and must not race with peers that still map or write it.  On every
 * rank: nts_exchange_release_peers (drains this rank's device work, closes its mappings of the peers' windows) ->
 * barrier -> nts_exchange_reserve (frees / allocates; n_buffers = 2 lets a rank run one exchange ahead of a slow
 * peer, 1 halves the memory) -> nts_exchange_handles -> all-gather of the handles -> nts_exchange_open_peers ->
 * barrier.  Reserve once for the widest layer to keep cudaMalloc out of the epoch loop. */
int nts_exchange_release_peers(nts_exchange *ex);
int nts_exchange_reserve(nts_exchange *ex, uint64_t floats_per_buffer, int n_buffers);
int nts_exchange_handles(nts_exchange *ex, unsigned char window_handle[64], unsigned char flags_handle[64]);
int nts_exchange_open_peers(nts_exchange *ex, const unsigned char *window_handles, const unsigned char *flag_handles);
/* Y_p += sum_i A_{p<-i} X_i  (ForwardGPUfuseOp::forward, core/ntsDistGPUFusedGraphOp.hpp:56-73); y zeroed by caller.
 * Every rank must issue the same sequence of forward / backward calls (SPMD, like the reference's ring). */
int nts_exchange_forward(nts_exchange *ex, const float *x, float *y, nts_vid_t feature_size, void *stream);
/* dX_p += sum_j A_{j<-p}^T dY_j (ForwardGPUfuseOp::backward, :75-90); dx zeroed by caller */
int nts_exchange_backward(nts_exchange *ex, const float *g, float *dx, nts_vid_t feature_size, void *stream);
/* BF16 gathers with FP32 accumulation (the contract of nts_gather_plan_run_bf16_ex) across partitions.  Forward: the
 * sender rounds its X (NTS_DTYPE_F32, or NTS_DTYPE_BF16 used as is when F % 8 == 0 and 16-byte aligned) once per call
 * into BF16 rows of stride ceil(F/8)*8 and pushes them (half the bytes), every chunk gathers BF16 rows.  Backward: dY
 * is rounded once locally; partial gradients are computed, pushed and added in FP32.  Every chunk runs through a plan
 * tuned per (width, type); the pipelined-vs-merged choice is made per (direction, width, type). */
int nts_exchange_forward_bf16(nts_exchange *ex, const void *x, int x_dtype, float *y, nts_vid_t feature_size,
                              void *stream);
int nts_exchange_backward_bf16(nts_exchange *ex, const float *g, float *dx, nts_vid_t feature_size, void *stream);
/* per-phase device timeline of the last forward (measurement): [0] push kernel, [1] local chunk, then per ring step
 * s: [2s] wait for the rows of partition (p+s), [2s+1] aggregation of chunk (p+s); [2P] whole call.  2P+1 floats (ms);
 * nts_exchange_last_timeline synchronises the device */
int nts_exchange_set_trace(nts_exchange *ex, int enable);
int nts_exchange_last_timeline(nts_exchange *ex, float *ms, int capacity);
/* What the last call on this engine did (host bookkeeping, known once the call returns; null outputs are skipped):
 * kind 1 forward, 2 backward, 3 mirror fetch, 4 mirror return (0: no call yet); its epoch and window buffer
 * (epoch % n_buffers); mode 1 = pipeline, 2 = merged receive (0 for fetch / return); kernel_peers / dma_peers = bit j
 * set when peer j was served by the push kernel / by a copy-engine push (a peer that reads none of my rows still gets
 * its flag from one of them); push_vec = floats per lane access of the push kernel (0: no kernel push); plan_chunks =
 * bit i set when chunk i was aggregated through an nts_gather_plan (its own or the merged one) rather than K1;
 * bf16_staging = 0 for FP32 gathers, 1 when this rank's operand was converted into BF16 staging rows, 2 when BF16
 * input rows were used as they are.  A single-partition engine reports only the kind. */
int nts_exchange_last_paths(const nts_exchange *ex, int *kind, int *epoch, int *buffer, int *mode,
                            uint32_t *kernel_peers, uint32_t *dma_peers, int *push_vec, uint32_t *plan_chunks,
                            int *bf16_staging);
/* DistGPUGetDepNbrOp (core/ntsDistGPUGraphOp.hpp:48-143) on the same windows - the reference moves the whole feature
 * matrix GPU -> host -> MPI -> host -> GPU.  forward: mirror[MirrorIndex[s], :] = X[s, :] for every source s of a local
 * in-edge ([owned_mirrors, F], partition order); backward: dx[v, :] += every partition's mirror gradient of my vertex
 * v (dx zeroed by the caller). */
int nts_exchange_fetch_mirrors(nts_exchange *ex, const float *x, float *mirror, nts_vid_t feature_size, void *stream);
int nts_exchange_return_mirror_grads(nts_exchange *ex, const float *mirror_grad, float *dx, nts_vid_t feature_size,
                                     void *stream);

/* ---- exchange plan builder (host C++): the reference's chunks -> the arrays of nts_exchange_desc ------------------------
 * C++ twin of neutronstarlite_b200/exchange.py::ExchangePlan for hosts without Python (the reference's own host
 * code: include/nts_dropin/core/ntsDistGPUFusedGraphOp.hpp).  One nts_host_chunk per source partition i describes
 * CSC_segment_pinned `graph_chunks[i]` of this rank (core/GraphSegment.h:52-139) through its HOST arrays:
 * column_offset[V_p+1] / row_indices[E_i] (global source ids) / edge_weight_forward, row_offset[V_i+1] /
 * column_indices[E_i] (global destination ids) / edge_weight_backward, src_range, dst_range, edge_size.
 * Sequence:  create -> pack_needs -> (caller moves every rank's pack to every rank) -> set_peer_needs for each
 * peer -> finalize -> create_from_plan (uploads; the plan owns the device copies and must outlive the engine).
 * The merged arrays of the view (one CSC / one compact CSR over all remote chunks) serve transports that aggregate
 * all remote chunks in one launch (the NCCL all-to-all path); the peer-memory engine works per chunk. */
typedef struct nts_host_chunk {
  const nts_vid_t *column_offset, *row_indices, *row_offset, *column_indices;
  const float *edge_weight_forward, *edge_weight_backward;
  nts_vid_t src_start, src_end, dst_start, dst_end;
  uint64_t edges;
} nts_host_chunk;
typedef struct nts_exchange_plan nts_exchange_plan;
nts_exchange_plan *nts_exchange_plan_create(const nts_host_chunk *chunks, int partitions, int rank);
void nts_exchange_plan_destroy(nts_exchange_plan *plan);
/* rows of partition i (local ids, ascending) that have an edge into this rank's partition = what it reads from i */
const nts_vid_t *nts_exchange_plan_need(const nts_exchange_plan *plan, int i, nts_vid_t *count);
/* this rank's lists in wire form: need_counts[P] (own entry 0) and the lists concatenated in partition order */
uint64_t nts_exchange_plan_packed_rows(const nts_exchange_plan *plan);
int nts_exchange_plan_pack_needs(const nts_exchange_plan *plan, nts_vid_t *need_counts, nts_vid_t *need_rows);
/* rank j's wire form, as received */
int nts_exchange_plan_set_peer_needs(nts_exchange_plan *plan, int j, const nts_vid_t *need_counts,
                                     const nts_vid_t *need_rows);
int nts_exchange_plan_finalize(nts_exchange_plan *plan);
/* host view of the finalized plan (tests, other transports); pointers live as long as the plan */
typedef struct nts_exchange_plan_view {
  int partitions, rank;
  nts_vid_t owned_vertices, recv_total, send_total, backward_rows;
  uint64_t remote_edges;
  const nts_vid_t *need_count, *send_count, *peer_bwd_offset;   /* [P] each */
  const nts_vid_t *fwd_push_offset, *bwd_push_offset;           /* [P] each, see nts_exchange_desc */
  const nts_vid_t *remote_column_offset, *remote_slots;         /* [V_p+1], [remote_edges] */
  const float *remote_weight;
  const nts_vid_t *backward_offsets, *backward_indices;         /* [backward_rows+1], [remote_edges] */
  const float *backward_weight;
  const nts_vid_t *send_rows_all;                               /* [send_total] */
} nts_exchange_plan_view;
int nts_exchange_plan_get_view(const nts_exchange_plan *plan, nts_exchange_plan_view *view);
/* per remote chunk i of the finalized plan (host arrays, live as long as the plan): row_indices as ranks in the need
 * list [E_i], row_offset restricted to the active sources [need_count[i]+1] */
int nts_exchange_plan_chunk(const nts_exchange_plan *plan, int i, const nts_vid_t **slots,
                            const nts_vid_t **row_offset_compact);
/* DEVICE arrays of CSC_segment_pinned graph_chunks[i] as uploaded by CopyGraphToDevice (core/GraphSegment.cpp:178-220),
 * one entry per source partition; the plan uploads the derived arrays itself and must outlive the engine */
typedef struct nts_device_chunk {
  const nts_vid_t *column_offset, *row_indices, *row_offset, *column_indices;
  const float *edge_weight_forward, *edge_weight_backward;
} nts_device_chunk;
nts_exchange *nts_exchange_create_from_plan(nts_exchange_plan *plan, const nts_device_chunk *device_chunks);

/* ---- host-side graph preparation (C++ with OpenMP; no device involved) -----------------------------------
 * Restates the layout contract of core/graph.hpp:1185-1211 (partitioner), :4396-4401 (degree clamp),
 * core/ntsBaseOp.hpp:194-197 (edge weight) and core/PartitionedGraph.hpp:324-420 (per-source-partition chunks). */
/* degrees with multiplicity over packed {u32 src,u32 dst} edges, clamped to >= 1 */
int nts_host_degrees(const nts_vid_t *edges_src_dst, uint64_t n_edges, nts_vid_t n_vertices,
                     nts_vid_t *out_degree, nts_vid_t *in_degree);
/* partition_offset[P+1] */
int nts_host_partition_offsets(const nts_vid_t *edges_src_dst, uint64_t n_edges, nts_vid_t n_vertices,
                               int partitions, nts_vid_t *partition_offset);
/* number of edges of chunk (src partition i -> dst partition p) for every i: counts[P] */
int nts_host_chunk_edge_counts(const nts_vid_t *edges_src_dst, uint64_t n_edges,
                               const nts_vid_t *partition_offset, int partitions, int rank,
                               uint64_t *counts);
/* build chunk i of rank p into caller-allocated arrays:
 * column_offset[Vp+1], row_indices[Ei], edge_weight_forward[Ei], row_offset[Vi+1], column_indices[Ei],
 * edge_weight_backward[Ei], source_active[Vi] (bytes) */
int nts_host_build_chunk(const nts_vid_t *edges_src_dst, uint64_t n_edges, nts_vid_t n_vertices,
                         const nts_vid_t *partition_offset, int partitions, int rank, int src_partition,
                         const nts_vid_t *out_degree, const nts_vid_t *in_degree,
                         nts_vid_t *column_offset, nts_vid_t *row_indices, float *edge_weight_forward,
                         nts_vid_t *row_offset, nts_vid_t *column_indices, float *edge_weight_backward,
                         unsigned char *source_active);
/* MirrorIndex[V+1] of rank p (core/PartitionedGraph.hpp:295-305); returns owned_mirrors through *owned */
int nts_host_mirror_index(const nts_vid_t *edges_src_dst, uint64_t n_edges, nts_vid_t n_vertices,
                          const nts_vid_t *partition_offset, int rank, nts_vid_t *mirror_index,
                          nts_vid_t *owned);

/* ---- device-side graph preparation: nts_graph_build -------------------------------------------------------------------
 * The arrays of the host builder above, for one rank, built on the GPU.  From a packed binary edge file ({u32 src,
 * u32 dst} records; edge count = file size / 8) read twice in blocks of block_edges records - pass 1 degrees, pass 2
 * the owned edges - so no process holds the edge list; or from edge arrays already on the device (int32 or int64;
 * only the edges whose destination this rank owns are required when the GLOBAL clamped degrees are given, in the
 * same type).  partition_offset (HOST array [P+1]) may be NULL: the reference's partitioner then runs on the raw
 * out-degree (with given degrees it is required for P > 1).  Limits: 1 <= V < 2^31, owned edges < 2^31; an id >= V is
 * an error, never clamped.  Outputs are bit-identical to nts_host_build_chunk / nts_host_mirror_index (CSC (dst, src)
 * ascending, CSR (src, dst) ascending, weights of nts_norm_degree).  Device scratch beyond the returned arrays stays
 * below 40 B per owned edge + 16 B per vertex.  Both builders synchronise `stream` and return NULL on failure
 * (nts_last_error() says why); exports are asynchronous copies on `stream` into caller-allocated device arrays, and
 * any export pointer may be NULL (arrays of length 0 included). */
typedef struct nts_graph_build nts_graph_build;
enum { NTS_GRAPH_BUILD_DIST = 1 };              /* also build MirrorIndex and the whole-partition CSC */
enum { NTS_INDEX_I32 = 0, NTS_INDEX_I64 = 1 };  /* element type of device edge and degree arrays */
nts_graph_build *nts_graph_build_from_file(const char *path, nts_vid_t n_vertices, int partitions, int rank,
                                           const nts_vid_t *partition_offset, uint64_t block_edges, int flags,
                                           void *stream);
nts_graph_build *nts_graph_build_from_device(const void *src, const void *dst, int index_dtype, uint64_t n_edges,
                                             nts_vid_t n_vertices, int partitions, int rank,
                                             const nts_vid_t *partition_offset, const void *out_degree,
                                             const void *in_degree, int flags, void *stream);
/* partition_offset[P+1], chunk_edges[P], owned_mirrors (0 without NTS_GRAPH_BUILD_DIST), the peak device scratch in
 * bytes, and pass_seconds[4] = {degrees, owned edges, chunks, distributed artefacts}; every output may be NULL */
int nts_graph_build_info(const nts_graph_build *build, nts_vid_t *partition_offset, uint64_t *chunk_edges,
                         nts_vid_t *owned_mirrors, uint64_t *scratch_peak_bytes, double *pass_seconds);
/* chunk i (sources in partition i): column_offset[Vp+1], row_indices[Ei], edge_weight_forward[Ei], row_offset[Vi+1],
 * column_indices[Ei], edge_weight_backward[Ei], source_active[Vi] */
int nts_graph_build_export_chunk(const nts_graph_build *build, int i, nts_vid_t *column_offset, nts_vid_t *row_indices,
                                 float *edge_weight_forward, nts_vid_t *row_offset, nts_vid_t *column_indices,
                                 float *edge_weight_backward, unsigned char *source_active, void *stream);
/* MirrorIndex[V+1], whole-partition column_offset[Vp+1] and row_indices[owned edges] (needs NTS_GRAPH_BUILD_DIST) */
int nts_graph_build_export_dist(const nts_graph_build *build, nts_vid_t *mirror_index, nts_vid_t *column_offset,
                                nts_vid_t *row_indices, void *stream);
/* clamped degrees with multiplicity, out_degree[V] and in_degree[V] */
int nts_graph_build_export_degrees(const nts_graph_build *build, nts_vid_t *out_degree, nts_vid_t *in_degree,
                                   void *stream);
int nts_graph_build_destroy(nts_graph_build *build);

/* ---- neighbour sampling for mini-batch training: nts_sampler ---------------------------------------------------------
 * The blocks of the reference's SampledSubgraph (core/ntsSampler.hpp, core/FullyRepGraph.hpp), built on the GPU from the
 * CSC of a single-partition graph: column_offset[V+1], row_indices[E] (global source ids, ascending inside a
 * destination) and edge_weight[E] (nts_norm_degree).  Hop 0's destinations are the seeds; each hop's destinations are
 * the previous hop's distinct sources.  Destination d keeps min(indeg(d), fanout[h]) of its edge slots (multi-edges
 * are distinct slots): all of them, or a uniform subset chosen by Floyd's algorithm with the draw
 * t = (hash(seed, step, h, d, j) * (j + 1)) >> 32 for j = deg-k .. deg-1, where hash is the upper half of a splitmix64
 * chain (DESIGN.md §3 K8 states it exactly).  Kept slots are written in ascending slot order, so a sample is a pure
 * function of (graph, seed, step, h, d).  A hop's sources are its distinct source ids ascending; local source ids
 * index them.  Scratch is allocated once, at create, for max_seeds seeds; 1 <= fanout[h] <= 64, 1 <= hops <= 8.
 * nts_sampler_sample synchronises `stream` once per hop (to read the hop's edge and source counts) and reports a seed
 * >= V as an error after hop 0.  Hop views point into the sampler's memory and stay valid until the next sample.
 *
 * NTS_SAMPLER_INCLUDE_DST (nts_sampler_create_ex): every hop's sources include its destinations, the block layout a
 * layer needs when a destination reads its own previous-layer row (a GAT layer's destination score).  A hop keeps
 * exactly the edges, weights and slot order of the default mode (no self-loop edge is added); its sources are the
 * distinct ids of (kept sources U destinations), ascending, and nts_sampler_hop_dst_pos gives dst_pos[n_dst], each
 * destination's local index in src (src[dst_pos[i]] == dst[i]).  Hop h+1's destinations are hop h's sources, so the
 * destination set only grows with depth.  Scratch is sized for n_dst * (fanout + 1) pairs per hop.  With flags = 0
 * the sampler is nts_sampler_create's, byte for byte. */
#define NTS_SAMPLER_INCLUDE_DST 1u
typedef struct nts_sampler nts_sampler;
typedef struct nts_sample_hop_view {
  nts_vid_t n_dst, n_src;
  uint64_t n_edges;
  const nts_vid_t *dst;            /* [n_dst]  global destination ids */
  const nts_vid_t *column_offset;  /* [n_dst+1] */
  const nts_vid_t *row_indices;    /* [n_edges] local source ids (into src) */
  const nts_vid_t *row_global;     /* [n_edges] global source ids */
  const float *weight;             /* [n_edges] edge_weight at the kept slots, bit for bit */
  const nts_vid_t *src;            /* [n_src]  distinct global source ids, ascending */
  const nts_vid_t *row_offset;     /* [n_src+1] transposed block, edges of a source in edge order */
  const nts_vid_t *column_indices; /* [n_edges] local destination of each transposed edge */
  const float *weight_backward;    /* [n_edges] */
} nts_sample_hop_view;
nts_sampler *nts_sampler_create(const nts_vid_t *column_offset, const nts_vid_t *row_indices, const float *edge_weight,
                                nts_vid_t n_vertices, uint64_t n_edges, nts_vid_t max_seeds, int hops,
                                const int *fanout, void *stream);
/* flags: 0 or NTS_SAMPLER_INCLUDE_DST; other bits are an argument error.  nts_sampler_create is flags = 0. */
nts_sampler *nts_sampler_create_ex(const nts_vid_t *column_offset, const nts_vid_t *row_indices,
                                   const float *edge_weight, nts_vid_t n_vertices, uint64_t n_edges,
                                   nts_vid_t max_seeds, int hops, const int *fanout, uint32_t flags, void *stream);
/* The same sampler over a CSC sharded by destination ranges: shard o holds destinations [shard_offsets[o],
 * shard_offsets[o+1]) as column_offsets[o][local dst + 1] (local offsets), row_indices[o] (global source ids) and
 * edge_weights[o], in the slot order of the whole-graph CSC, so the blocks equal nts_sampler_create_ex's on the
 * concatenated shards bit for bit.  The shard arrays may be any device memory the stream's device can read, peer
 * memory included.  column_offsets / row_indices / edge_weights are host arrays of n_shards device pointers and
 * shard_offsets a host array of n_shards + 1 ids; all are copied at create.  1 <= n_shards <= 32; shard_offsets start
 * at 0 and do not decrease; V = shard_offsets[n_shards]; empty shards may have null arrays; every shard has fewer than
 * 2^32 edges.  Used with nts_sampler_sample / _hop_view / _hop_dst_pos / _bytes / _destroy. */
nts_sampler *nts_sampler_create_sharded(const nts_vid_t *const *column_offsets, const nts_vid_t *const *row_indices,
                                        const float *const *edge_weights, const nts_vid_t *shard_offsets,
                                        int n_shards, nts_vid_t max_seeds, int hops, const int *fanout,
                                        uint32_t flags, void *stream);
int nts_sampler_sample(nts_sampler *sampler, const nts_vid_t *seeds, nts_vid_t n_seeds, uint64_t seed, uint64_t step,
                       void *stream);
int nts_sampler_hop_view(const nts_sampler *sampler, int hop, nts_sample_hop_view *view);
/* *dst_pos = the hop's dst_pos[n_dst] (device, local source index of every destination); an error unless the sampler
 * was created with NTS_SAMPLER_INCLUDE_DST.  Valid until the next sample, like the hop view. */
int nts_sampler_hop_dst_pos(const nts_sampler *sampler, int hop, const nts_vid_t **dst_pos);
/* peak device bytes the sampler holds (scratch and hop storage) */
uint64_t nts_sampler_bytes(const nts_sampler *sampler);
int nts_sampler_destroy(nts_sampler *sampler);
/* The transposed block of any block whose local sources are in [0, n_src), in any order: row_offset[n_src+1],
 * column_indices[n_edges] (local destinations) and weight_backward[n_edges], edges of a source in edge order (one
 * stable radix sort; sources without edges get empty segments).  Temporary memory is stream-ordered. */
int nts_sample_transpose(const nts_vid_t *column_offset, const nts_vid_t *row_indices, const float *weight,
                         nts_vid_t n_dst, nts_vid_t n_src, uint64_t n_edges, nts_vid_t *row_offset,
                         nts_vid_t *column_indices, float *weight_backward, void *stream);

/* One weighted CSC from a rank's n_chunks chunk CSCs over the same n_dst destinations (PartitionedGraph's chunks:
 * column_offsets[o][n_dst+1], row_indices[o] and edge_weights[o] device arrays of chunk o): destination d's slots are
 * chunk 0's, then chunk 1's, ..., each in its chunk's order, which for the reference's chunks is the slot order of the
 * single-partition CSC.  Outputs: column_offset[n_dst+1], row_indices_out / edge_weight_out [n_edges], where n_edges
 * (< 2^32) is the sum of the chunks' edges.  The pointer arrays are host arrays; 1 <= n_chunks <= 32; row / weight
 * arrays of chunks without edges may be null.  Before any slot is copied the stream is synchronised once to check the
 * scanned edge count against n_edges and that no chunk with edges has a null array: either is an error, and only
 * column_offset has been written.  Temporary memory is stream-ordered. */
int nts_merge_chunk_csc(const nts_vid_t *const *column_offsets, const nts_vid_t *const *row_indices,
                        const float *const *edge_weights, int n_chunks, nts_vid_t n_dst, uint64_t n_edges,
                        nts_vid_t *column_offset, nts_vid_t *row_indices_out, float *edge_weight_out, void *stream);

/* ---- feature / label / mask tables (GNNDatum, core/ntsDataloador.hpp) ----------------------------------------------------
 * Text tables exactly as GNNDatum::readFeature_Label_Mask (:156-221) reads them - "id f0 .. fF-1", "id label",
 * "id train|val|eval|test", the k-th label / mask record belongs to the k-th feature record - parsed in parallel;
 * rows with id in [v_begin, v_end) land at id - v_begin (mask: train 0, val/eval 1, test 2, other 3).  label_path /
 * mask_path (and their outputs) may be NULL.  Returns 0, or a negative code (-2/-3/-4 unreadable file, -5 malformed). */
int nts_host_read_feature_label_mask(const char *feature_path, const char *label_path, const char *mask_path,
                                     nts_vid_t feature_size, nts_vid_t v_begin, nts_vid_t v_end, float *features,
                                     int64_t *labels, int32_t *masks);
/* rows [v_begin, v_end) of a packed float32 [V, feature_size] table (the twin of the packed binary edge file) */
int nts_host_read_feature_binary(const char *path, nts_vid_t feature_size, nts_vid_t v_begin, nts_vid_t v_end,
                                 float *features);

#ifdef __cplusplus
}
#endif
#endif /* NTS_B200_H */
