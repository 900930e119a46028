/* Drop-in stand-in for the reference's cuda/cuda_type.h (typedef :21, launch constants :22-25).
 * The library's kernels size their own grids from the SM count; the four launch constants are kept only so
 * that reference code which names them keeps compiling. */
#ifndef NTS_B200_DROPIN_CUDA_TYPE_H
#define NTS_B200_DROPIN_CUDA_TYPE_H
#include <stdint.h>
typedef uint32_t VertexId_CUDA;
static const int CUDA_NUM_THREADS = 256;
static const int CUDA_NUM_BLOCKS = 132 * 8;
static const int CUDA_NUM_THREADS_SOFTMAX = 256;
static const int CUDA_NUM_BLOCKS_SOFTMAX = 132 * 8;
#endif
