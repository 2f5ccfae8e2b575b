// Point-set chamfer distance (embodiedscan/models/losses/chamfer_distance.py:13-79) without the (B, N, M) distance
// tensor the reference builds: nearest neighbours in both directions, then a deterministic backward.
//
// Forward: one thread per query point; the other set streams through shared-memory tiles. Each pair costs C criterion
// evaluations, so the work is O(B * N * M * C) and the memory O(B * (N + M)).
// Backward: a point's gradient is its own term plus the terms of every point that chose it as nearest neighbour. Those
// reverse terms are gathered, not scattered: the (batch, chosen index) keys are sorted stably and each point sums its
// segment in query-index order, so two runs give the same bits (no float atomics).
#include <cub/cub.cuh>
#include "common.cuh"

namespace {

constexpr int CD_THREADS = 256;

// dist[b, i] = min_j sum_c crit(q[b, i, c] - r[b, j, c]), idx[b, i] = the lowest such j
template <int C, int MODE>
__global__ void __launch_bounds__(CD_THREADS)
chamfer_nn_kernel(const float* __restrict__ q, const float* __restrict__ r, int Nq, int Nr, float* __restrict__ dist,
                  long long* __restrict__ idx) {
  __shared__ float tile[CD_THREADS * C];
  const int b = blockIdx.y;
  const int i = blockIdx.x * CD_THREADS + threadIdx.x;
  const float* qb = q + (size_t)b * Nq * C;
  const float* rb = r + (size_t)b * Nr * C;
  float x[C];
#pragma unroll
  for (int c = 0; c < C; ++c) x[c] = i < Nq ? qb[(size_t)i * C + c] : 0.f;
  float best = INFINITY;
  int bj = 0;
  for (int t0 = 0; t0 < Nr; t0 += CD_THREADS) {
    const int n = min(CD_THREADS, Nr - t0);
    __syncthreads();
    for (int k = threadIdx.x; k < n * C; k += CD_THREADS) tile[k] = rb[(size_t)t0 * C + k];
    __syncthreads();
#pragma unroll 4
    for (int j = 0; j < n; ++j) {
      float d = esb_cd_crit<MODE>(x[0] - tile[j * C]);
#pragma unroll
      for (int c = 1; c < C; ++c) d += esb_cd_crit<MODE>(x[c] - tile[j * C + c]);
      if (d < best) { best = d; bj = t0 + j; }      // strict: the first minimum wins, as torch.min
    }
  }
  if (i < Nq) {
    dist[(size_t)b * Nq + i] = best;
    idx[(size_t)b * Nq + i] = bj;
  }
}

// sort keys: the global row of the chosen neighbour; values: the global row of the query (ascending before the sort)
__global__ void chamfer_keys_kernel(const long long* __restrict__ idx1, const long long* __restrict__ idx2, int B, int N,
                                    int M, unsigned* __restrict__ k1, int* __restrict__ v1, unsigned* __restrict__ k2,
                                    int* __restrict__ v2) {
  const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long n1 = (long long)B * N, n2 = (long long)B * M;
  if (t < n1) {
    const int b = (int)(t / N);
    k1[t] = (unsigned)((long long)b * M + idx1[t]);
    v1[t] = (int)t;
  } else if (t < n1 + n2) {
    const long long u = t - n1;
    const int b = (int)(u / M);
    k2[u] = (unsigned)((long long)b * N + idx2[u]);
    v2[u] = (int)u;
  }
}

__device__ __forceinline__ int lower_bound_u(const unsigned* __restrict__ a, int n, unsigned key) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// One thread per point of either set (rows 0 .. B*N-1: src, then B*M rows: dst). A pair (p, q) with distance
// sum_c crit(p - q) sends g * crit'(p - q) to p and g * crit'(q - p) to q.
//   own term:     g_own[p] * crit'(p - other[own_idx[p]])
//   reverse term: sum over the sorted segment of queries q that chose p, in query order, of g_q[q] * crit'(p - q)
template <int C, int MODE>
__global__ void chamfer_grad_kernel(const float* __restrict__ src, const float* __restrict__ dst,
                                    const long long* __restrict__ idx1, const long long* __restrict__ idx2,
                                    const float* __restrict__ g1, const float* __restrict__ g2, int B, int N, int M,
                                    const unsigned* __restrict__ k1s, const int* __restrict__ v1s,
                                    const unsigned* __restrict__ k2s, const int* __restrict__ v2s,
                                    float* __restrict__ grad_src, float* __restrict__ grad_dst) {
  const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long n1 = (long long)B * N, n2 = (long long)B * M;
  if (t >= n1 + n2) return;
  const bool is_src = t < n1;
  const long long row = is_src ? t : t - n1;                   // global row in its own set
  const int n_own = is_src ? N : M, n_other = is_src ? M : N;
  const int b = (int)(row / n_own);
  const float* own = is_src ? src : dst;
  const float* other = is_src ? dst : src;
  const long long* own_idx = is_src ? idx1 : idx2;
  const float* g_own = is_src ? g1 : g2;
  const float* g_rev = is_src ? g2 : g1;
  // queries that chose this point are the other set's rows, sorted by the key b * n_own + local index = row
  const unsigned* ks = is_src ? k2s : k1s;
  const int* vs = is_src ? v2s : v1s;
  const int n_keys = (int)(is_src ? n2 : n1);
  float p[C], acc[C];
#pragma unroll
  for (int c = 0; c < C; ++c) { p[c] = own[row * C + c]; acc[c] = 0.f; }
  if (g_own != nullptr) {
    const float g = g_own[row];
    const float* o = other + ((long long)b * n_other + own_idx[row]) * C;
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] = g * esb_cd_dcrit<MODE>(p[c] - o[c]);
  }
  if (g_rev != nullptr) {
    for (int k = lower_bound_u(ks, n_keys, (unsigned)row); k < n_keys && ks[k] == (unsigned)row; ++k) {
      const long long qrow = vs[k];
      const float g = g_rev[qrow];
      const float* o = other + qrow * C;
#pragma unroll
      for (int c = 0; c < C; ++c) acc[c] += g * esb_cd_dcrit<MODE>(p[c] - o[c]);
    }
  }
  float* out = (is_src ? grad_src : grad_dst) + row * C;
#pragma unroll
  for (int c = 0; c < C; ++c) out[c] = acc[c];
}

template <int C, int MODE>
void launch_nn(const float* src, const float* dst, int B, int N, int M, float* dist1, float* dist2, long long* idx1,
               long long* idx2, cudaStream_t s) {
  chamfer_nn_kernel<C, MODE><<<dim3(esb_div_up(N, CD_THREADS), B), CD_THREADS, 0, s>>>(src, dst, N, M, dist1, idx1);
  chamfer_nn_kernel<C, MODE><<<dim3(esb_div_up(M, CD_THREADS), B), CD_THREADS, 0, s>>>(dst, src, M, N, dist2, idx2);
}

template <int C, int MODE>
void launch_grad(const float* src, const float* dst, const long long* idx1, const long long* idx2, const float* g1,
                 const float* g2, int B, int N, int M, const unsigned* k1s, const int* v1s, const unsigned* k2s,
                 const int* v2s, float* grad_src, float* grad_dst, cudaStream_t s) {
  const long long rows = (long long)B * N + (long long)B * M;
  chamfer_grad_kernel<C, MODE><<<esb_div_up(rows, 256), 256, 0, s>>>(src, dst, idx1, idx2, g1, g2, B, N, M, k1s, v1s,
                                                                     k2s, v2s, grad_src, grad_dst);
}

// compile-time (C, MODE) dispatch: C in [1, 8], MODE in ESB_CD_*
template <template <int, int> class F, typename... A>
void dispatch(int C, int mode, A... a) {
#define ESB_CD_CASE(CC)                                                                 \
  case CC:                                                                              \
    if (mode == ESB_CD_L1) F<CC, ESB_CD_L1>::run(a...);                                 \
    else if (mode == ESB_CD_L2) F<CC, ESB_CD_L2>::run(a...);                            \
    else F<CC, ESB_CD_SMOOTH_L1>::run(a...);                                            \
    break;
  switch (C) {
    ESB_CD_CASE(1) ESB_CD_CASE(2) ESB_CD_CASE(3) ESB_CD_CASE(4)
    ESB_CD_CASE(5) ESB_CD_CASE(6) ESB_CD_CASE(7) ESB_CD_CASE(8)
  }
#undef ESB_CD_CASE
}
template <int C, int MODE>
struct NnOp {
  template <typename... A>
  static void run(A... a) { launch_nn<C, MODE>(a...); }
};
template <int C, int MODE>
struct GradOp {
  template <typename... A>
  static void run(A... a) { launch_grad<C, MODE>(a...); }
};

}  // namespace

#define ESB_CD_CHECK_ARGS(fn)                                                                                      \
  ESB_CHECK_ARG(B >= 1 && N >= 1 && M >= 1, fn ": empty point set (B=%d N=%d M=%d)", B, N, M);                     \
  ESB_CHECK_ARG(C >= 1 && C <= 8, fn ": C must be in [1, 8], got %d", C);                                          \
  ESB_CHECK_ARG(mode == ESB_CD_L1 || mode == ESB_CD_L2 || mode == ESB_CD_SMOOTH_L1, fn ": bad mode %d", mode);     \
  ESB_CHECK_ARG((long long)B * N < (1LL << 31) && (long long)B * M < (1LL << 31), fn ": too many points")

extern "C" int esb_chamfer_fwd(const float* src, const float* dst, int B, int N, int M, int C, int mode, float* dist1,
                               float* dist2, long long* idx1, long long* idx2, void* stream) {
  ESB_CD_CHECK_ARGS("esb_chamfer_fwd");
  ESB_CHECK_ARG(B <= 65535, "esb_chamfer_fwd: B must be <= 65535");
  dispatch<NnOp>(C, mode, src, dst, B, N, M, dist1, dist2, idx1, idx2, (cudaStream_t)stream);
  ESB_CUDA_LAUNCH_CHECK("chamfer_nn_kernel");
  return ESB_OK;
}

extern "C" int esb_chamfer_bwd(const float* src, const float* dst, const long long* idx1, const long long* idx2,
                               const float* g1, const float* g2, int B, int N, int M, int C, int mode, float* grad_src,
                               float* grad_dst, void* stream_) {
  ESB_CD_CHECK_ARGS("esb_chamfer_bwd");
  cudaStream_t stream = (cudaStream_t)stream_;
  const int n1 = B * N, n2 = B * M;
  // keys < B * max(N, M) < 2^31: sort only the bits they use
  int end_bit = 1;
  while (end_bit < 32 && ((long long)1 << end_bit) < (long long)B * (N > M ? N : M)) ++end_bit;
  size_t t1 = 0, t2 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, t1, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr,
                                  (int*)nullptr, n1, 0, end_bit, stream);
  cub::DeviceRadixSort::SortPairs(nullptr, t2, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr,
                                  (int*)nullptr, n2, 0, end_bit, stream);
  const size_t a1 = esb_align((size_t)n1 * 4), a2 = esb_align((size_t)n2 * 4), at = esb_align(t1 > t2 ? t1 : t2);
  uint8_t* ws = nullptr;
  ESB_CUDA_CALL(esb_scratch_alloc((void**)&ws, 4 * a1 + 4 * a2 + at, stream));
  unsigned* k1 = (unsigned*)ws;
  unsigned* k1s = (unsigned*)(ws + a1);
  int* v1 = (int*)(ws + 2 * a1);
  int* v1s = (int*)(ws + 3 * a1);
  uint8_t* p2 = ws + 4 * a1;
  unsigned* k2 = (unsigned*)p2;
  unsigned* k2s = (unsigned*)(p2 + a2);
  int* v2 = (int*)(p2 + 2 * a2);
  int* v2s = (int*)(p2 + 3 * a2);
  void* temp = p2 + 4 * a2;
  chamfer_keys_kernel<<<esb_div_up((long long)n1 + n2, 256), 256, 0, stream>>>(idx1, idx2, B, N, M, k1, v1, k2, v2);
  cudaError_t e = cudaPeekAtLastError();
  size_t tb = t1;
  if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(temp, tb, k1, k1s, v1, v1s, n1, 0, end_bit, stream);
  tb = t2;
  if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(temp, tb, k2, k2s, v2, v2s, n2, 0, end_bit, stream);
  if (e == cudaSuccess) {
    dispatch<GradOp>(C, mode, src, dst, idx1, idx2, g1, g2, B, N, M, (const unsigned*)k1s, (const int*)v1s,
                     (const unsigned*)k2s, (const int*)v2s, grad_src, grad_dst, stream);
    e = cudaPeekAtLastError();
  }
  if (e != cudaSuccess) {
    esb_scratch_free(ws, stream);
    esb_set_error("esb_chamfer_bwd: %s", cudaGetErrorString(e));
    return ESB_ECUDA;
  }
  ESB_CUDA_CALL(esb_scratch_free(ws, stream));
  return ESB_OK;
}
