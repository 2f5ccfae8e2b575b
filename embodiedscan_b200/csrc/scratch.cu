// esb200 — stream-ordered scratch memory and the fixed-order reducer behind every multi-block floating-point sum of the
// library: partial sums are never combined with float atomics, so a training step computes the same bits on every run.
#include <mutex>

#include "common.cuh"

namespace {

constexpr int kSumThreads = 256;
constexpr int kSumLoads = 8;                          // independent loads in flight per thread and tile
constexpr int kSumTile = kSumThreads * kSumLoads;     // floats per shared-memory tile

// s + tile[0] + tile[1] + ... + tile[n - 1], in that order (1 <= n <= kSumTile). A loss sum is one such chain per tile,
// one dependent add per part (~450k parts for the focal loss of a C2 step): the 16-byte reads of the next 16 parts are
// issued before the adds of the current 16, and reads past n (still inside the tile) are never added.
__device__ __forceinline__ float add_chain_contiguous(const float* __restrict__ tile, int n, float s) {
  const float4* q = reinterpret_cast<const float4*>(tile);
  float4 a[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) a[u] = q[u];
  int r = 0;
  for (; r + 16 <= n; r += 16) {
    const int nx = min(r + 16, kSumTile - 16) / 4;
    float4 b[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) b[u] = q[nx + u];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      s = __fadd_rn(s, a[u].x);
      s = __fadd_rn(s, a[u].y);
      s = __fadd_rn(s, a[u].z);
      s = __fadd_rn(s, a[u].w);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) a[u] = b[u];
  }
  const float rest[16] = {a[0].x, a[0].y, a[0].z, a[0].w, a[1].x, a[1].y, a[1].z, a[1].w,
                          a[2].x, a[2].y, a[2].z, a[2].w, a[3].x, a[3].y, a[3].z, a[3].w};
#pragma unroll
  for (int u = 0; u < 16; ++u)
    if (r + u < n) s = __fadd_rn(s, rest[u]);
  return s;
}

// Block b finishes the `cw` columns j = b * cw + c, c < cw (cw a power of two dividing kSumThreads). The finishers'
// callers have few columns and many parts (a loss sum has one column and thousands of parts), so the whole block loads:
// tiles of kSumTile / cw parts x cw columns, every thread kSumLoads independent coalesced loads, through shared memory to
// thread c, which adds its column in part order, each add rounded on its own. The next tile is in flight in the loaders'
// registers while the current one is added. accumulate: 0 = out[j] = the sum from +0; 1 = the chain starts from out[j];
// 2 = out[j] + the finished sum from +0, one rounded add (how a gradient slot receives one backward pass's sum).
__global__ void __launch_bounds__(kSumThreads) sum_partial_rows_kernel(const float* __restrict__ part, int n_parts,
                                                                       long long width, float* __restrict__ out,
                                                                       int accumulate, int cw) {
  __shared__ __align__(16) float tile[kSumTile];
  const int t = threadIdx.x;
  const int rows = kSumTile / cw, rstep = kSumThreads / cw;
  const int r0 = t / cw;
  const long long j = blockIdx.x * (long long)cw + (t & (cw - 1));
  const bool col_ok = j < width;
  const bool adder = t < cw && col_ok;
  float v[kSumLoads];
  auto load = [&](int p0) {
#pragma unroll
    for (int k = 0; k < kSumLoads; ++k) {
      const int p = p0 + r0 + k * rstep;
      v[k] = col_ok && p < n_parts ? part[(long long)p * width + j] : 0.f;
    }
  };
  float s = adder && accumulate == 1 ? out[j] : 0.f;
  if (n_parts > 0) load(0);
  for (int p0 = 0; p0 < n_parts; p0 += rows) {
    __syncthreads();                                  // the adders are done with the previous tile
#pragma unroll
    for (int k = 0; k < kSumLoads; ++k) tile[t + k * kSumThreads] = v[k];   // = row r0 + k * rstep, column t % cw
    __syncthreads();
    if (p0 + rows < n_parts) load(p0 + rows);
    if (adder && cw == 1) {
      s = add_chain_contiguous(tile, min(rows, n_parts - p0), s);
    } else if (adder) {
      // 16 parts per group; the next group's reads (clamped inside the tile) are requested before this group's adds
      const int n = min(rows, n_parts - p0);
      const float* col = tile + t;
      float a[16];
#pragma unroll
      for (int u = 0; u < 16; ++u) a[u] = col[min(u, n - 1) * cw];
      int r = 0;
      for (; r + 16 <= n; r += 16) {
        float b[16];
#pragma unroll
        for (int u = 0; u < 16; ++u) b[u] = col[min(r + 16 + u, n - 1) * cw];
#pragma unroll
        for (int u = 0; u < 16; ++u) s = __fadd_rn(s, a[u]);
#pragma unroll
        for (int u = 0; u < 16; ++u) a[u] = b[u];
      }
      for (int u = 0; r + u < n; ++u) s = __fadd_rn(s, col[(r + u) * cw]);
    }
  }
  if (adder) out[j] = accumulate == 2 ? __fadd_rn(out[j], s) : s;
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
  // Narrow sums: 8 columns per block, so a tile is 256 parts deep and its add chain (~4 cycles per part) outlasts the
  // next tile's load latency. Wide sums: widen the blocks until the grid is at most ~8 blocks per SM.
  int cw = 1;
  while (cw < 8 && cw < width) cw *= 2;
  while (cw < kSumThreads && (width + cw - 1) / cw > 8LL * esb_sm_count()) cw *= 2;
  sum_partial_rows_kernel<<<esb_div_up(width, cw), kSumThreads, 0, s>>>(part, n_parts, width, out, accumulate, cw);
  ESB_CUDA_LAUNCH_CHECK("sum_partial_rows_kernel");
  return ESB_OK;
}
