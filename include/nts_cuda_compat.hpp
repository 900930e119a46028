// nts_cuda_compat.hpp - the C++ face of the drop-in boundary.
//
// The reference's host code (core/NtsScheduler.hpp:151-357, core/GraphSegment.cpp:76-220,320-334,
// comm/network.cpp:52-101, core/graph.hpp:275-280, core/ntsDistGPUGraphOp.hpp:145-361) talks to the device
// through `cuda/ntsCUDA.hpp`: a handful of free functions (:25-47), `deviceCSC` (:49-95) and `Cuda_Stream`
// (:97-217).  This header re-declares that surface - same names, same parameter order and meaning, same
// "print and exit(1)" error convention (cuda/ntsCUDAGraphOP.cu:13-19) - as thin inline forwards to the C ABI of
// libnts_b200.so (include/nts_b200.h), so that reference translation units compile and link unchanged while
// every kernel they launch is the sm_90a implementation of this repository.
//
// Not reproduced on purpose:
//   * the reference's "_Optim" kernels overwrite instead of accumulate and overrun rows by one
//     (cuda/ntsCUDAFuseKernel.cuh:203-204,264,381,441); here plain and _Optim entry points run the same kernel;
//   * the reference GPU edge softmax has no max subtraction (cuda/ntsCUDADistKernel.cuh:192); ours matches the
//     CPU operator (core/ntsDistCPUGraphOp.hpp:463) instead;
//   * Gather_By_Dst_From_Message is declared but never defined in the reference (a link error if it were ever
//     used); here it is defined with the semantics of the kernel it was meant to launch.
#pragma once

#include <cstdio>
#include <cstdlib>

#include "nts_b200.h"

#if defined(CUDA_ENABLE) && CUDA_ENABLE
// the reference header pulls the CUDA runtime in (cuda/ntsCUDA.hpp:10-12) and comm/network.cpp:56,87 calls
// cudaFreeHost directly, so a drop-in has to do the same
#include "cuda_runtime.h"
#elif !defined(__CUDACC__) && !defined(CUDART_VERSION) && !defined(__DRIVER_TYPES_H__)
// without the toolkit headers only the stream type is needed, by name (ntsCUDA.hpp:102)
struct CUstream_st;
typedef struct CUstream_st *cudaStream_t;
#endif

#ifndef NTS_B200_DROPIN_CUDA_TYPE_H
typedef uint32_t VertexId_CUDA;
#endif

enum graph_type { CSR, CSC, PAIR };
enum weight_type { NULL_TYPE, SCALA_TYPE, TENSOR_TYPE };

namespace nts_compat {
inline void must(int rc, const char *what) {
  if (rc != 0) {
    std::fprintf(stderr, "nts_b200 %s failed: %s\n", what, nts_last_error());
    std::exit(1);
  }
}
template <class T> inline T *must_ptr(T *p, const char *what) {
  if (!p) {
    std::fprintf(stderr, "nts_b200 %s failed: %s\n", what, nts_last_error());
    std::exit(1);
  }
  return p;
}
} // namespace nts_compat

// ---- free functions (ntsCUDA.hpp:25-47) -------------------------------------------------------------------
inline void ntsFreeHost(void *buffer) { nts_compat::must(nts_free_pinned(buffer), "ntsFreeHost"); }
inline void *cudaMallocPinned(long size_of_bytes) {
  return nts_compat::must_ptr(nts_malloc_pinned((size_t)size_of_bytes), "cudaMallocPinned");
}
inline void *getDevicePointer(void *host_data_to_device) {
  return nts_compat::must_ptr(nts_pinned_device_pointer(host_data_to_device), "getDevicePointer");
}
inline void *cudaMallocGPU(long size_of_bytes) {
  return nts_compat::must_ptr(nts_malloc_device((size_t)size_of_bytes), "cudaMallocGPU");
}
// rows [src, dst) of width feature_size, device -> host
inline void move_result_out(float *output, float *input, int src, int dst, int feature_size, bool sync = true) {
  nts_compat::must(nts_memcpy_d2h(output, input, (size_t)(dst - src) * feature_size * sizeof(float), nullptr, sync),
                   "move_result_out");
}
inline void move_data_in(float *d_pointer, float *h_pointer, int start, int end, int feature_size,
                         bool sync = true) {
  nts_compat::must(
      nts_memcpy_h2d(d_pointer, h_pointer, (size_t)(end - start) * feature_size * sizeof(float), nullptr, sync),
      "move_data_in");
}
inline void move_edge_in(VertexId_CUDA *d_pointer, VertexId_CUDA *h_pointer, VertexId_CUDA start,
                         VertexId_CUDA end, int feature_size, bool sync = true) {
  nts_compat::must(nts_memcpy_h2d(d_pointer, h_pointer,
                                  (size_t)(end - start) * feature_size * sizeof(VertexId_CUDA), nullptr, sync),
                   "move_edge_in");
}
inline void move_bytes_in(void *d_pointer, void *h_pointer, long bytes, bool sync = true) {
  nts_compat::must(nts_memcpy_h2d(d_pointer, h_pointer, (size_t)bytes, nullptr, sync), "move_bytes_in");
}
inline void allocate_gpu_buffer(float **input, int size) {
  *input = (float *)nts_compat::must_ptr(nts_malloc_device(sizeof(float) * (size_t)size), "allocate_gpu_buffer");
}
inline void allocate_gpu_edge(VertexId_CUDA **input, int size) {
  *input = (VertexId_CUDA *)nts_compat::must_ptr(nts_malloc_device(sizeof(VertexId_CUDA) * (size_t)size),
                                                 "allocate_gpu_edge");
}
// (the reference's aggregate_comm_result is a debug kernel with no callers; kept as a no-op symbol)
inline void aggregate_comm_result(float *, float *, int, int, int, bool = true) {}
inline void FreeBuffer(float *buffer) { nts_compat::must(nts_free_device(buffer), "FreeBuffer"); }
inline void FreeEdge(VertexId_CUDA *buffer) { nts_compat::must(nts_free_device(buffer), "FreeEdge"); }
inline void zero_buffer(float *buffer, int size) {
  nts_compat::must(nts_zero(buffer, sizeof(float) * (size_t)size, nullptr), "zero_buffer");
  nts_compat::must(nts_device_synchronize(), "zero_buffer");
}
inline void CUDA_DEVICE_SYNCHRONIZE() { nts_compat::must(nts_device_synchronize(), "CUDA_DEVICE_SYNCHRONIZE"); }
inline void ResetDevice() { nts_compat::must(nts_device_reset(), "ResetDevice"); }

// ---- deviceCSC (ntsCUDA.hpp:49-95): whole-partition CSC (+ MirrorIndex) resident on the device ------------------
class deviceCSC {
public:
  VertexId_CUDA *column_offset = nullptr;
  VertexId_CUDA *row_indices = nullptr;
  VertexId_CUDA *mirror_index = nullptr;
  VertexId_CUDA v_size = 0;
  VertexId_CUDA e_size = 0;
  VertexId_CUDA mirror_size = 0;
  bool require_mirror = false;

  deviceCSC() {}
  ~deviceCSC() {}
  void init(VertexId_CUDA v_size_, VertexId_CUDA e_size_, bool require_mirror_ = false,
            VertexId_CUDA mirror_size_ = 0) {
    v_size = v_size_;
    e_size = e_size_;
    require_mirror = require_mirror_;
    column_offset = (VertexId_CUDA *)cudaMallocGPU((long)(v_size_ + 1) * (long)sizeof(VertexId_CUDA));
    row_indices = (VertexId_CUDA *)cudaMallocGPU((long)e_size_ * (long)sizeof(VertexId_CUDA));
    if (require_mirror_) {
      mirror_size = mirror_size_;
      mirror_index = (VertexId_CUDA *)cudaMallocGPU((long)mirror_size_ * (long)sizeof(VertexId_CUDA));
    }
  }
  void load_from_host(VertexId_CUDA *h_column_offset, VertexId_CUDA *h_row_indices,
                      VertexId_CUDA *h_mirror_index) {
    load_from_host(h_column_offset, h_row_indices);
    move_bytes_in(mirror_index, h_mirror_index, (long)mirror_size * (long)sizeof(VertexId_CUDA));
  }
  void load_from_host(VertexId_CUDA *h_column_offset, VertexId_CUDA *h_row_indices) {
    move_bytes_in(column_offset, h_column_offset, (long)(v_size + 1) * (long)sizeof(VertexId_CUDA));
    move_bytes_in(row_indices, h_row_indices, (long)e_size * (long)sizeof(VertexId_CUDA));
  }
  void release() {
    FreeEdge(column_offset);
    FreeEdge(row_indices);
    if (require_mirror)
      FreeEdge(mirror_index);
    column_offset = row_indices = mirror_index = nullptr;
  }
};

// ---- Cuda_Stream (ntsCUDA.hpp:97-217): one CUDA stream + one method per kernel family -------------------------
class Cuda_Stream {
public:
  cudaStream_t stream;

  // blocking stream, like the reference's cudaStreamCreate (ntsCUDAGraphOP.cu:60-63): ordered against the
  // legacy default stream that libtorch uses
  Cuda_Stream() { stream = (cudaStream_t)nts_compat::must_ptr(nts_stream_create(0), "Cuda_Stream"); }
  void destory_Stream() { nts_compat::must(nts_stream_destroy(stream), "destory_Stream"); }
  cudaStream_t getStream() { return stream; }
  void CUDA_DEVICE_SYNCHRONIZE() { nts_compat::must(nts_stream_synchronize(stream), "CUDA_DEVICE_SYNCHRONIZE"); }

  void move_result_out(float *output, float *input, VertexId_CUDA src, VertexId_CUDA dst, int feature_size,
                       bool sync = true) {
    nts_compat::must(
        nts_memcpy_d2h(output, input, (size_t)(dst - src) * feature_size * sizeof(float), stream, sync),
        "move_result_out");
  }
  void move_data_in(float *d_pointer, float *h_pointer, VertexId_CUDA start, VertexId_CUDA end,
                    int feature_size, bool sync = true) {
    nts_compat::must(
        nts_memcpy_h2d(d_pointer, h_pointer, (size_t)(end - start) * feature_size * sizeof(float), stream, sync),
        "move_data_in");
  }
  void move_edge_in(VertexId_CUDA *d_pointer, VertexId_CUDA *h_pointer, VertexId_CUDA start, VertexId_CUDA end,
                    int feature_size, bool sync = true) {
    nts_compat::must(nts_memcpy_h2d(d_pointer, h_pointer,
                                    (size_t)(end - start) * feature_size * sizeof(VertexId_CUDA), stream, sync),
                     "move_edge_in");
  }
  void aggregate_comm_result(float *, float *, VertexId_CUDA, int, int, bool = true) {}

  void deSerializeToGPU(float *input_gpu_buffer, float *input_buffer, VertexId_CUDA data_size,
                        VertexId_CUDA feature_size, VertexId_CUDA partition_start, VertexId_CUDA partition_end,
                        bool sync) {
    nts_compat::must(nts_deserialize_records(input_gpu_buffer, input_buffer, data_size, feature_size,
                                             partition_start, partition_end, stream),
                     "deSerializeToGPU");
    if (sync)
      CUDA_DEVICE_SYNCHRONIZE();
  }
  void aggregate_comm_result_debug(float *aggregate_buffer, float *input_buffer, VertexId_CUDA data_size,
                                   VertexId_CUDA feature_size, VertexId_CUDA partition_start,
                                   VertexId_CUDA partition_end, bool sync) {
    nts_compat::must(nts_aggregate_records(aggregate_buffer, input_buffer, data_size, feature_size,
                                           partition_start, partition_end, stream),
                     "aggregate_comm_result_debug");
    if (sync)
      CUDA_DEVICE_SYNCHRONIZE();
  }

  // fused vertex aggregation -------------------------------------------------------------------------------
  void Gather_By_Dst_From_Src(float *input, float *output, float *weight_forward, VertexId_CUDA *row_indices,
                              VertexId_CUDA *column_offset, VertexId_CUDA src_start, VertexId_CUDA src_end,
                              VertexId_CUDA dst_start, VertexId_CUDA dst_end, VertexId_CUDA edges,
                              VertexId_CUDA batch_size, VertexId_CUDA feature_size, bool with_weight = false,
                              bool tensor_weight = false) {
    (void)tensor_weight;
    nts_compat::must(nts_gather_by_dst_from_src(input, output, weight_forward, row_indices, column_offset,
                                                src_start, src_end, dst_start, dst_end, edges, batch_size,
                                                feature_size, with_weight ? 1 : 0, stream),
                     "Gather_By_Dst_From_Src");
  }
  void Gather_By_Dst_From_Src_Optim(float *input, float *output, float *weight_forward,
                                    VertexId_CUDA *row_indices, VertexId_CUDA *column_offset,
                                    VertexId_CUDA src_start, VertexId_CUDA src_end, VertexId_CUDA dst_start,
                                    VertexId_CUDA dst_end, VertexId_CUDA edges, VertexId_CUDA batch_size,
                                    VertexId_CUDA feature_size, bool with_weight = false,
                                    bool tensor_weight = false) {
    Gather_By_Dst_From_Src(input, output, weight_forward, row_indices, column_offset, src_start, src_end,
                           dst_start, dst_end, edges, batch_size, feature_size, with_weight, tensor_weight);
  }
  void Gather_By_Src_From_Dst(float *input, float *output, float *weight_backward, VertexId_CUDA *row_offset,
                              VertexId_CUDA *column_indices, VertexId_CUDA src_start, VertexId_CUDA src_end,
                              VertexId_CUDA dst_start, VertexId_CUDA dst_end, VertexId_CUDA edges,
                              VertexId_CUDA batch_size, VertexId_CUDA feature_size, bool with_weight = false,
                              bool tensor_weight = false) {
    (void)tensor_weight;
    nts_compat::must(nts_gather_by_src_from_dst(input, output, weight_backward, row_offset, column_indices,
                                                src_start, src_end, dst_start, dst_end, edges, batch_size,
                                                feature_size, with_weight ? 1 : 0, stream),
                     "Gather_By_Src_From_Dst");
  }
  void Gather_By_Src_From_Dst_Optim(float *input, float *output, float *weight_backward,
                                    VertexId_CUDA *row_offset, VertexId_CUDA *column_indices,
                                    VertexId_CUDA src_start, VertexId_CUDA src_end, VertexId_CUDA dst_start,
                                    VertexId_CUDA dst_end, VertexId_CUDA edges, VertexId_CUDA batch_size,
                                    VertexId_CUDA feature_size, bool with_weight = false,
                                    bool tensor_weight = false) {
    Gather_By_Src_From_Dst(input, output, weight_backward, row_offset, column_indices, src_start, src_end,
                           dst_start, dst_end, edges, batch_size, feature_size, with_weight, tensor_weight);
  }

  // edge-granular operators (GAT path) --------------------------------------------------------------------
  void Scatter_Src_Mirror_to_Msg(float *message, float *src_mirror_feature, VertexId_CUDA *row_indices,
                                 VertexId_CUDA *column_offset, VertexId_CUDA *mirror_index,
                                 VertexId_CUDA batch_size, VertexId_CUDA feature_size) {
    nts_compat::must(nts_scatter_src_mirror_to_msg(message, src_mirror_feature, row_indices, column_offset,
                                                   mirror_index, batch_size, feature_size, stream),
                     "Scatter_Src_Mirror_to_Msg");
  }
  void Gather_Msg_To_Src_Mirror(float *src_mirror_feature, float *message, VertexId_CUDA *row_indices,
                                VertexId_CUDA *column_offset, VertexId_CUDA *mirror_index,
                                VertexId_CUDA batch_size, VertexId_CUDA feature_size) {
    nts_compat::must(nts_gather_msg_to_src_mirror(src_mirror_feature, message, row_indices, column_offset,
                                                  mirror_index, batch_size, feature_size, stream),
                     "Gather_Msg_To_Src_Mirror");
  }
  void Scatter_Dst_to_Msg(float *message, float *dst_feature, VertexId_CUDA *row_indices,
                          VertexId_CUDA *column_offset, VertexId_CUDA batch_size, VertexId_CUDA feature_size) {
    nts_compat::must(
        nts_scatter_dst_to_msg(message, dst_feature, row_indices, column_offset, batch_size, feature_size, stream),
        "Scatter_Dst_to_Msg");
  }
  void Gather_Msg_to_Dst(float *dst_feature, float *message, VertexId_CUDA *row_indices,
                         VertexId_CUDA *column_offset, VertexId_CUDA batch_size, VertexId_CUDA feature_size) {
    nts_compat::must(
        nts_gather_msg_to_dst(dst_feature, message, row_indices, column_offset, batch_size, feature_size, stream),
        "Gather_Msg_to_Dst");
  }
  void Edge_Softmax_Forward_Block(float *msg_output, float *msg_input, float *msg_cached,
                                  VertexId_CUDA *row_indices, VertexId_CUDA *column_offset,
                                  VertexId_CUDA batch_size, VertexId_CUDA feature_size) {
    nts_compat::must(nts_edge_softmax_forward(msg_output, msg_input, msg_cached, row_indices, column_offset,
                                              batch_size, feature_size, stream),
                     "Edge_Softmax_Forward_Block");
  }
  void Edge_Softmax_Backward_Block(float *msg_input_grad, float *msg_output_grad, float *msg_cached,
                                   VertexId_CUDA *row_indices, VertexId_CUDA *column_offset,
                                   VertexId_CUDA batch_size, VertexId_CUDA feature_size) {
    nts_compat::must(nts_edge_softmax_backward(msg_input_grad, msg_output_grad, msg_cached, row_indices,
                                               column_offset, batch_size, feature_size, stream),
                     "Edge_Softmax_Backward_Block");
  }
  // Declared by the reference (ntsCUDA.hpp:186-192) and called from NtsScheduler::GatherByDstFromMessage
  // (core/NtsScheduler.hpp:192-211) but never defined in cuda/ntsCUDAGraphOP.cu; the intended kernel
  // (aggregate_kernel_from_message_without_weight_sum, cuda/ntsCUDAFuseKernel.cuh:562-577) is
  // output[d,:] += sum_{e->d} message[e,:] with (src, dst) = (row_indices, column_offset) - our Gather_Msg_to_Dst.
  void Gather_By_Dst_From_Message(float *input, float *output, VertexId_CUDA *src, VertexId_CUDA *dst,
                                  VertexId_CUDA src_start, VertexId_CUDA src_end, VertexId_CUDA dst_start,
                                  VertexId_CUDA dst_end, VertexId_CUDA edges, VertexId_CUDA batch_size,
                                  VertexId_CUDA feature_size, bool with_weight = false,
                                  bool tensor_weight = false) {
    (void)src_start; (void)src_end; (void)dst_start; (void)dst_end; (void)edges; (void)with_weight;
    (void)tensor_weight;
    nts_compat::must(nts_gather_msg_to_dst(output, input, src, dst, batch_size, feature_size, stream),
                     "Gather_By_Dst_From_Message");
  }
  void Scatter_Grad_Back_To_Message(float *input, float *message_grad, VertexId_CUDA *row_indices,
                                    VertexId_CUDA *column_offset, VertexId_CUDA src_start, VertexId_CUDA src_end,
                                    VertexId_CUDA dst_start, VertexId_CUDA dst_end, VertexId_CUDA edges,
                                    VertexId_CUDA batch_size, VertexId_CUDA feature_size,
                                    bool with_weight = true) {
    (void)src_start; (void)src_end; (void)dst_start; (void)dst_end; (void)edges; (void)with_weight;
    nts_compat::must(nts_scatter_grad_back_to_message(input, message_grad, row_indices, column_offset, batch_size,
                                                      feature_size, stream),
                     "Scatter_Grad_Back_To_Message");
  }
};
