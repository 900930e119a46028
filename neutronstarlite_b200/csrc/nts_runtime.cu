// Runtime plumbing of libnts_b200: error state, device/stream/event/memory helpers (the free functions of
// cuda/ntsCUDA.hpp:25-47 and the stream half of `Cuda_Stream`, cuda/ntsCUDAGraphOP.cu:23-130,413-528),
// CUDA-IPC peer mappings and system-scope flag signalling for the NVLink exchange.
#include "nts_common.cuh"

#include <algorithm>
#include <atomic>

namespace nts {

static thread_local char t_last_error[512] = "";
static std::atomic<uint64_t> g_launches{0};

char *last_error_buffer() { return t_last_error; }

bool abort_on_error() {
  static int cached = -1;
  if (cached < 0) {
    const char *e = getenv("NTS_B200_ABORT_ON_ERROR");
    cached = (e && e[0] == '1') ? 1 : 0;
  }
  return cached == 1;
}

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64)
    return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132; // H100 SXM
    cached[dev] = n;
  }
  return cached[dev];
}

int time_min_of_two(const std::function<int()> &run, cudaStream_t st, float *ms) {
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  *ms = 1e30f;
  int rc = 0;
  if (cudaEventCreate(&e0) != cudaSuccess || cudaEventCreate(&e1) != cudaSuccess)
    rc = fail(-1, "event creation for a timed run failed", __FILE__, __LINE__);
  for (int it = 0; it < 3 && !rc; it++) {
    float t = 0.f;
    if (cudaEventRecord(e0, st) != cudaSuccess || (rc = run()) != 0 || cudaEventRecord(e1, st) != cudaSuccess ||
        cudaEventSynchronize(e1) != cudaSuccess || cudaEventElapsedTime(&t, e0, e1) != cudaSuccess)
      rc = rc ? rc : -1;
    else if (it > 0 && t < *ms)
      *ms = t;
  }
  if (e0)
    cudaEventDestroy(e0);
  if (e1)
    cudaEventDestroy(e1);
  return rc;
}

__global__ void signal_set_kernel(uint32_t *flag, uint32_t value) {
  // everything issued before this kernel on the stream is visible to the peer before the flag flips
  __threadfence_system();
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(flag), "r"(value) : "memory");
}

__global__ void signal_wait_kernel(const uint32_t *flag, uint32_t value) {
  uint32_t v;
  do {
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
    if (v < value)
      __nanosleep(200);
  } while (v < value);
}

// Parameter::learnC2G_with_decay_Adam (core/NtsScheduler.hpp:774-781) in one pass: the reference issues six
// element-wise libtorch ops (each a kernel and a temporary); same arithmetic, same order of operations per element
// (adam_element, nts_common.cuh)
__global__ void adam_update_kernel(float *__restrict__ W, float *__restrict__ M, float *__restrict__ V,
                                   const float *__restrict__ grad, uint64_t n, float weight_decay, float beta1,
                                   float beta2, float alpha, float epsilon) {
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    float w = W[i], m = M[i], v = V[i];
    adam_element(w, m, v, grad[i], weight_decay, beta1, beta2, alpha, epsilon);
    M[i] = m;
    V[i] = v;
    W[i] = w;
  }
}

} // namespace nts

using namespace nts;

extern "C" {

int nts_version(void) { return 1; }
const char *nts_last_error(void) { return last_error_buffer(); }
uint64_t nts_kernel_launch_count(void) { return g_launches.load(); }

int nts_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess)
    return 0;
  return n;
}
int nts_set_device(int device) {
  NTS_CUDA_OK(cudaSetDevice(device));
  return 0;
}
int nts_device_sm_count(int *out) {
  NTS_ARG_CHECK(out, "null output pointer");
  int dev = 0;
  NTS_CUDA_OK(cudaGetDevice(&dev));
  NTS_CUDA_OK(cudaDeviceGetAttribute(out, cudaDevAttrMultiProcessorCount, dev));
  return 0;
}
int nts_device_synchronize(void) {
  NTS_CUDA_OK(cudaDeviceSynchronize());
  return 0;
}
int nts_device_reset(void) {
  NTS_CUDA_OK(cudaDeviceReset());
  return 0;
}

void *nts_malloc_device(size_t bytes) {
  void *p = nullptr;
  cudaError_t e = cudaMalloc(&p, bytes ? bytes : 1);
  if (e != cudaSuccess) {
    fail((int)e, cudaGetErrorString(e), __FILE__, __LINE__);
    return nullptr;
  }
  return p;
}
int nts_free_device(void *ptr) {
  if (ptr)
    NTS_CUDA_OK(cudaFree(ptr));
  return 0;
}
void *nts_malloc_pinned(size_t bytes) {
  void *p = nullptr;
  cudaError_t e = cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocMapped);
  if (e != cudaSuccess) {
    fail((int)e, cudaGetErrorString(e), __FILE__, __LINE__);
    return nullptr;
  }
  return p;
}
int nts_free_pinned(void *ptr) {
  if (ptr)
    NTS_CUDA_OK(cudaFreeHost(ptr));
  return 0;
}
void *nts_pinned_device_pointer(void *host_ptr) {
  void *d = nullptr;
  cudaError_t e = cudaHostGetDevicePointer(&d, host_ptr, 0);
  if (e != cudaSuccess) {
    fail((int)e, cudaGetErrorString(e), __FILE__, __LINE__);
    return nullptr;
  }
  return d;
}

int nts_memcpy_h2d(void *dst, const void *src, size_t bytes, void *stream, int sync) {
  if (bytes == 0)
    return 0;
  NTS_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, as_stream(stream)));
  if (sync)
    NTS_CUDA_OK(cudaStreamSynchronize(as_stream(stream)));
  return 0;
}
int nts_memcpy_d2h(void *dst, const void *src, size_t bytes, void *stream, int sync) {
  if (bytes == 0)
    return 0;
  NTS_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, as_stream(stream)));
  if (sync)
    NTS_CUDA_OK(cudaStreamSynchronize(as_stream(stream)));
  return 0;
}
int nts_memcpy_d2d(void *dst, const void *src, size_t bytes, void *stream) {
  if (bytes == 0)
    return 0;
  NTS_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, as_stream(stream)));
  return 0;
}
int nts_zero(void *ptr, size_t bytes, void *stream) {
  if (bytes == 0)
    return 0;
  NTS_CUDA_OK(cudaMemsetAsync(ptr, 0, bytes, as_stream(stream)));
  return 0;
}

void *nts_stream_create(int non_blocking) {
  cudaStream_t s = nullptr;
  cudaError_t e = cudaStreamCreateWithFlags(&s, non_blocking ? cudaStreamNonBlocking : cudaStreamDefault);
  if (e != cudaSuccess) {
    fail((int)e, cudaGetErrorString(e), __FILE__, __LINE__);
    return nullptr;
  }
  return s;
}
int nts_stream_destroy(void *stream) {
  if (stream)
    NTS_CUDA_OK(cudaStreamDestroy(as_stream(stream)));
  return 0;
}
int nts_stream_synchronize(void *stream) {
  NTS_CUDA_OK(cudaStreamSynchronize(as_stream(stream)));
  return 0;
}
void *nts_event_create(int with_timing) {
  cudaEvent_t ev = nullptr;
  cudaError_t e = cudaEventCreateWithFlags(&ev, with_timing ? cudaEventDefault : cudaEventDisableTiming);
  if (e != cudaSuccess) {
    fail((int)e, cudaGetErrorString(e), __FILE__, __LINE__);
    return nullptr;
  }
  return ev;
}
int nts_event_destroy(void *event) {
  if (event)
    NTS_CUDA_OK(cudaEventDestroy(reinterpret_cast<cudaEvent_t>(event)));
  return 0;
}
int nts_event_record(void *event, void *stream) {
  NTS_CUDA_OK(cudaEventRecord(reinterpret_cast<cudaEvent_t>(event), as_stream(stream)));
  return 0;
}
int nts_stream_wait_event(void *stream, void *event) {
  NTS_CUDA_OK(cudaStreamWaitEvent(as_stream(stream), reinterpret_cast<cudaEvent_t>(event), 0));
  return 0;
}
int nts_event_elapsed_ms(void *start, void *stop, float *ms) {
  NTS_ARG_CHECK(ms, "null output pointer");
  NTS_CUDA_OK(cudaEventSynchronize(reinterpret_cast<cudaEvent_t>(stop)));
  NTS_CUDA_OK(cudaEventElapsedTime(ms, reinterpret_cast<cudaEvent_t>(start), reinterpret_cast<cudaEvent_t>(stop)));
  return 0;
}

int nts_ipc_get_handle(void *device_ptr, unsigned char handle[NTS_IPC_HANDLE_BYTES]) {
  static_assert(sizeof(cudaIpcMemHandle_t) == NTS_IPC_HANDLE_BYTES, "IPC handle size");
  cudaIpcMemHandle_t h;
  NTS_CUDA_OK(cudaIpcGetMemHandle(&h, device_ptr));
  memcpy(handle, &h, sizeof(h));
  return 0;
}
void *nts_ipc_open_handle(const unsigned char handle[NTS_IPC_HANDLE_BYTES]) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  void *p = nullptr;
  cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) {
    fail((int)e, cudaGetErrorString(e), __FILE__, __LINE__);
    return nullptr;
  }
  return p;
}
int nts_ipc_close_handle(void *peer_ptr) {
  if (peer_ptr)
    NTS_CUDA_OK(cudaIpcCloseMemHandle(peer_ptr));
  return 0;
}
int nts_adam_update(float *W, float *M, float *V, const float *grad, uint64_t n, float weight_decay, float beta1,
                    float beta2, float alpha, float epsilon, void *stream) {
  if (n == 0)
    return 0;
  NTS_ARG_CHECK(W && M && V && grad, "null pointer passed to nts_adam_update");
  const unsigned blocks = (unsigned)std::min<uint64_t>((n + 255) / 256, (uint64_t)sm_count() * 8);
  adam_update_kernel<<<blocks, 256, 0, as_stream(stream)>>>(W, M, V, grad, n, weight_decay, beta1, beta2, alpha, epsilon);
  NTS_LAUNCH_CHECK();
  return 0;
}

int nts_signal_set(uint32_t *flag, uint32_t value, void *stream) {
  NTS_ARG_CHECK(flag, "null flag");
  signal_set_kernel<<<1, 1, 0, as_stream(stream)>>>(flag, value);
  NTS_LAUNCH_CHECK();
  return 0;
}
int nts_signal_wait_geq(const uint32_t *flag, uint32_t value, void *stream) {
  NTS_ARG_CHECK(flag, "null flag");
  signal_wait_kernel<<<1, 1, 0, as_stream(stream)>>>(flag, value);
  NTS_LAUNCH_CHECK();
  return 0;
}

} // extern "C"
