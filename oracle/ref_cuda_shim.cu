// TEST / BENCH INFRASTRUCTURE ONLY.  extern "C" handles around the UNMODIFIED reference CUDA launchers
// (cuda/ntsCUDAGraphOP.cu, compiled from the reference sources for sm_90a by oracle/Makefile into
// oracle/_ref/libnts_refcuda.so) so that bench.py can time "the reference's own GPU kernels on an H100"
// next to ours (BASELINE.md section 3, item 7).  Nothing here is part of the product.
#define CUDA_ENABLE 1
#include "ntsCUDA.hpp"

extern "C" {

void *refcuda_stream_create() { return new Cuda_Stream(); }
// (Cuda_Stream::getStream() is declared but never defined in the reference: read the public member instead)
void *refcuda_stream_handle(void *s) { return (void *)static_cast<Cuda_Stream *>(s)->stream; }
void refcuda_stream_sync(void *s) { static_cast<Cuda_Stream *>(s)->CUDA_DEVICE_SYNCHRONIZE(); }

// optim = 0: aggregate_kernel_from_src_with_weight (global atomicAdd per edge element), the path
// NtsScheduler::GatherByDstFromSrc takes for F > 512 or when optim_kernel_enable is false;
// optim = 1: the shared-memory "_optim_nts" kernels (F <= 512 only).
void refcuda_gather_by_dst_from_src(void *s, float *in, float *out, float *w, unsigned *row_indices,
                                    unsigned *column_offset, unsigned src_s, unsigned src_e, unsigned dst_s,
                                    unsigned dst_e, unsigned edges, unsigned batch, unsigned F, int with_weight,
                                    int optim) {
  Cuda_Stream *cs = static_cast<Cuda_Stream *>(s);
  if (optim)
    cs->Gather_By_Dst_From_Src_Optim(in, out, w, row_indices, column_offset, src_s, src_e, dst_s, dst_e, edges,
                                     batch, F, with_weight != 0);
  else
    cs->Gather_By_Dst_From_Src(in, out, w, row_indices, column_offset, src_s, src_e, dst_s, dst_e, edges, batch, F,
                               with_weight != 0);
}

void refcuda_gather_by_src_from_dst(void *s, float *in, float *out, float *w, unsigned *row_offset,
                                    unsigned *column_indices, unsigned src_s, unsigned src_e, unsigned dst_s,
                                    unsigned dst_e, unsigned edges, unsigned batch, unsigned F, int with_weight,
                                    int optim) {
  Cuda_Stream *cs = static_cast<Cuda_Stream *>(s);
  if (optim)
    cs->Gather_By_Src_From_Dst_Optim(in, out, w, row_offset, column_indices, src_s, src_e, dst_s, dst_e, edges,
                                     batch, F, with_weight != 0);
  else
    cs->Gather_By_Src_From_Dst(in, out, w, row_offset, column_indices, src_s, src_e, dst_s, dst_e, edges, batch, F,
                               with_weight != 0);
}
}
