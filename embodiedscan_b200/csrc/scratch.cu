// esb200 — stream-ordered scratch memory and the fixed-order reducer behind every multi-block floating-point sum of the
// library: partial sums are never combined with float atomics, so a training step computes the same bits on every run.
#include <mutex>

#include "common.cuh"

namespace {

__global__ void sum_partial_rows_kernel(const float* __restrict__ part, int n_parts, long long width, float* __restrict__ out,
                                        int accumulate) {
  const long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (j >= width) return;
  float s = accumulate ? out[j] : 0.f;
  for (int p = 0; p < n_parts; ++p) s += part[(long long)p * width + j];
  out[j] = s;
}

}  // namespace

int esb_sm_count() {
  static int sms[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 64) return 132;
  if (sms[dev] == 0) {
    int n = 132;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    sms[dev] = n;
  }
  return sms[dev];
}

namespace {
// The library's own stream-ordered pool per device (the device's default pool and its settings stay untouched). Blocks a
// step frees stay mapped up to the release threshold, so the next step reuses them without new mappings; above it the pool
// returns memory at synchronisation.
constexpr unsigned long long kScratchKeepBytes = 512ull << 20;
std::mutex g_pool_mutex;
cudaMemPool_t g_pool[64] = {};

cudaMemPool_t scratch_pool(int dev, cudaStream_t s) {
  if (dev < 0 || dev >= 64) return nullptr;
  std::lock_guard<std::mutex> lock(g_pool_mutex);
  if (g_pool[dev] == nullptr) {
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(s, &st);
    if (st != cudaStreamCaptureStatusNone) return nullptr;     // created by the first call outside a capture
    cudaMemPoolProps props = {};
    props.allocType = cudaMemAllocationTypePinned;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = dev;
    cudaMemPool_t pool = nullptr;
    if (cudaMemPoolCreate(&pool, &props) != cudaSuccess) return nullptr;
    unsigned long long keep = kScratchKeepBytes;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    g_pool[dev] = pool;
  }
  return g_pool[dev];
}
}  // namespace

cudaError_t esb_scratch_alloc(void** p, size_t bytes, cudaStream_t s) {
  int dev = 0;
  cudaGetDevice(&dev);
  const size_t n = bytes > 0 ? bytes : 16;
  cudaMemPool_t pool = scratch_pool(dev, s);
  // inside a capture before the first eager call the allocation becomes a graph allocation node either way
  return pool != nullptr ? cudaMallocFromPoolAsync(p, n, pool, s) : cudaMallocAsync(p, n, s);
}

cudaError_t esb_scratch_free(void* p, cudaStream_t s) { return cudaFreeAsync(p, s); }

int esb_sum_partial_rows(const float* part, int n_parts, long long width, float* out, int accumulate, cudaStream_t s) {
  if (width == 0) return ESB_OK;
  sum_partial_rows_kernel<<<esb_div_up(width, 256), 256, 0, s>>>(part, n_parts, width, out, accumulate);
  ESB_CUDA_LAUNCH_CHECK("sum_partial_rows_kernel");
  return ESB_OK;
}
