// esb200 — sparse 3D convolution, SIMT (CUDA-core) path: fp32 parity arithmetic and the fallback for channel
// counts the tensor-core path does not tile (Cin=3 stem). Replaces ME.MinkowskiConvolution forward/backward
// (†upstream MinkowskiEngine) as called from embodiedscan/models/backbones/mink_resnet.py:58-62,104-108 and
// embodiedscan/models/dense_heads/fcaf3d_head.py:919-946.
//
// Output-stationary implicit GEMM: a CTA owns 64 output rows x 64 output channels and loops over the kernel
// offsets k, gathering the neighbour input rows nbr[k][o] (or zero) — no atomics, every output written once,
// deterministic. dgrad is the same kernel run on the input-stationary map with W read transposed.
// wgrad reduces over the compacted (in,out) pair list of each offset.
//
// Roofline (pair model, BASELINE.md §3): bytes = P*(Cin+Cout)*e + 8P + K*Cin*Cout*e ; flops = 2*P*Cin*Cout.
#include "common.cuh"

namespace {

constexpr int TM = 64;   // output rows per CTA
constexpr int TN = 64;   // output channels per CTA
constexpr int KC = 16;   // reduction chunk (input channels)

template <typename T>
__device__ __forceinline__ void load4(const T* p, bool vec, int valid, float out[4]);

template <>
__device__ __forceinline__ void load4<float>(const float* p, bool vec, int valid, float out[4]) {
  if (vec && valid >= 4) {
    float4 v = *reinterpret_cast<const float4*>(p);
    out[0] = v.x; out[1] = v.y; out[2] = v.z; out[3] = v.w;
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) out[j] = j < valid ? p[j] : 0.f;
  }
}
template <>
__device__ __forceinline__ void load4<__nv_bfloat16>(const __nv_bfloat16* p, bool vec, int valid, float out[4]) {
  if (vec && valid >= 4) {
    uint2 v = *reinterpret_cast<const uint2*>(p);
    __nv_bfloat162 a = *reinterpret_cast<__nv_bfloat162*>(&v.x);
    __nv_bfloat162 b = *reinterpret_cast<__nv_bfloat162*>(&v.y);
    out[0] = __low2float(a); out[1] = __high2float(a); out[2] = __low2float(b); out[3] = __high2float(b);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) out[j] = j < valid ? __bfloat162float(p[j]) : 0.f;
  }
}

// y[o, :] = sum_k x[nbr[k][o], :] @ W_k      (W_k = w[k] (Cin,Cout), or w[k]^T with w[k] (Cout,Cin) if WT)
template <typename T, bool WT>
__global__ void __launch_bounds__(256)
spconv_fwd_kernel(const T* __restrict__ x, const T* __restrict__ w, const int* __restrict__ nbr, T* __restrict__ y,
                  int n_out, int cin, int cout, int K, int accumulate) {
  __shared__ __align__(16) float As[KC][TM + 4];
  __shared__ __align__(16) float Bs[KC][TN + 4];
  __shared__ int rows[TM];

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.x * TM, n0 = blockIdx.y * TN;
  const bool vec_in = (cin & 3) == 0, vec_out = (cout & 3) == 0;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k = 0; k < K; ++k) {
    int r = -1;
    if (tid < TM && m0 + tid < n_out) r = nbr[(long long)k * n_out + m0 + tid];
    if (tid < TM) rows[tid] = r;
    if (!__syncthreads_or(r >= 0)) continue;  // nobody in this tile has neighbour k (also publishes rows[])
    const T* wk = w + (long long)k * cin * cout;
    for (int c0 = 0; c0 < cin; c0 += KC) {
      {  // A: 64 rows x 16 channels, 4 channels per thread
        int row = tid >> 2, ch = (tid & 3) * 4;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        int src = rows[row];
        int valid = cin - (c0 + ch);
        if (src >= 0 && valid > 0) load4<T>(x + (long long)src * cin + c0 + ch, vec_in, valid, v);
#pragma unroll
        for (int j = 0; j < 4; ++j) As[ch + j][row] = v[j];
      }
      if (!WT) {  // B[kc][col] = wk[c0+kc][n0+col]
        int kc = tid >> 4, col = (tid & 15) * 4;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        int valid = cout - (n0 + col);
        if (c0 + kc < cin && valid > 0) load4<T>(wk + (long long)(c0 + kc) * cout + n0 + col, vec_out, valid, v);
#pragma unroll
        for (int j = 0; j < 4; ++j) Bs[kc][col + j] = v[j];
      } else {  // B[kc][col] = wk[n0+col][c0+kc]  (w[k] stored (Cout, Cin))
        int col = tid >> 2, kc = (tid & 3) * 4;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        int valid = cin - (c0 + kc);
        if (n0 + col < cout && valid > 0) load4<T>(wk + (long long)(n0 + col) * cin + c0 + kc, vec_in, valid, v);
#pragma unroll
        for (int j = 0; j < 4; ++j) Bs[kc + j][col] = v[j];
      }
      __syncthreads();
#pragma unroll
      for (int kc = 0; kc < KC; ++kc) {
        float4 a = *reinterpret_cast<const float4*>(&As[kc][ty * 4]);
        float4 b = *reinterpret_cast<const float4*>(&Bs[kc][tx * 4]);
        float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int row = m0 + ty * 4 + i;
    if (row >= n_out) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int col = n0 + tx * 4 + j;
      if (col < cout) {
        long long idx = (long long)row * cout + col;
        float v = acc[i][j];
        if (accumulate) v += esb_to_float<T>(y[idx]);
        y[idx] = esb_from_float<T>(v);
      }
    }
  }
}

// dw[k] (Cin,Cout) += sum_{p in pairs(k)} x[pin[p], :]^T dy[pout[p], :]
template <typename T>
__global__ void __launch_bounds__(256)
spconv_wgrad_kernel(const T* __restrict__ x, const T* __restrict__ dy, const int* __restrict__ pair_in,
                    const int* __restrict__ pair_out, const int* __restrict__ k_offsets, float* __restrict__ dw,
                    int cin, int cout, int splits) {
  __shared__ __align__(16) float As[KC][TM + 4];
  __shared__ __align__(16) float Bs[KC][TN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int k = blockIdx.x / splits, sp = blockIdx.x - k * splits;
  const int ci0 = blockIdx.y * TM, co0 = blockIdx.z * TN;
  const int p_beg = k_offsets[k], p_end = k_offsets[k + 1];
  const int np = p_end - p_beg;
  if (np <= 0) return;
  const int per = (np + splits - 1) / splits;
  const int s_beg = p_beg + sp * per;
  const int s_end = min(p_end, s_beg + per);
  if (s_beg >= s_end) return;
  const bool vec_in = (cin & 3) == 0, vec_out = (cout & 3) == 0;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int p0 = s_beg; p0 < s_end; p0 += KC) {
    {  // 16 pairs x 64 channels each for A (x rows) and B (dy rows); thread: pair = tid/16, ch = (tid%16)*4
      int pp = tid >> 4, ch = (tid & 15) * 4;
      float va[4] = {0.f, 0.f, 0.f, 0.f}, vb[4] = {0.f, 0.f, 0.f, 0.f};
      if (p0 + pp < s_end) {
        int ri = pair_in[p0 + pp], ro = pair_out[p0 + pp];
        int valid_a = cin - (ci0 + ch), valid_b = cout - (co0 + ch);
        if (valid_a > 0) load4<T>(x + (long long)ri * cin + ci0 + ch, vec_in, valid_a, va);
        if (valid_b > 0) load4<T>(dy + (long long)ro * cout + co0 + ch, vec_out, valid_b, vb);
      }
      *reinterpret_cast<float4*>(&As[pp][ch]) = make_float4(va[0], va[1], va[2], va[3]);
      *reinterpret_cast<float4*>(&Bs[pp][ch]) = make_float4(vb[0], vb[1], vb[2], vb[3]);
    }
    __syncthreads();
#pragma unroll
    for (int kc = 0; kc < KC; ++kc) {
      float4 a = *reinterpret_cast<const float4*>(&As[kc][ty * 4]);
      float4 b = *reinterpret_cast<const float4*>(&Bs[kc][tx * 4]);
      float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
  // this split's partial of dW[k]: part[sp][k] (zeroed by the host: splits without pairs leave it untouched)
  float* dwk = dw + ((long long)sp * gridDim.x / splits + k) * cin * cout;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int ci = ci0 + ty * 4 + i;
    if (ci >= cin) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int co = co0 + tx * 4 + j;
      if (co < cout) dwk[(long long)ci * cout + co] = acc[i][j];
    }
  }
}

}  // namespace

// x (n_in,cin), w (K,cin,cout) [or (K,cout,cin) when w_transposed], nbr (K,n_out) -> y (n_out,cout)
extern "C" int esb_spconv_fwd(const void* x, const void* w, const int* nbr, void* y, long long n_out, int cin, int cout,
                              int K, int w_transposed, int accumulate, int dtype, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  ESB_CHECK_ARG(cin > 0 && cout > 0 && K > 0, "esb_spconv_fwd: bad channel/kernel sizes");
  ESB_CHECK_ARG(dtype == ESB_F32 || dtype == ESB_BF16, "esb_spconv_fwd: dtype must be f32 or bf16");
  if (n_out == 0) return ESB_OK;
  dim3 grid(esb_div_up(n_out, TM), esb_div_up(cout, TN));
#define LAUNCH(T, WT)                                                                                          \
  spconv_fwd_kernel<T, WT><<<grid, 256, 0, stream>>>((const T*)x, (const T*)w, nbr, (T*)y, (int)n_out, cin, cout, K, \
                                                      accumulate)
  if (dtype == ESB_F32) {
    if (w_transposed) LAUNCH(float, true); else LAUNCH(float, false);
  } else {
    if (w_transposed) LAUNCH(__nv_bfloat16, true); else LAUNCH(__nv_bfloat16, false);
  }
#undef LAUNCH
  ESB_CUDA_LAUNCH_CHECK("spconv_fwd_kernel");
  return ESB_OK;
}

// dw (K,cin,cout) fp32 += the weight gradient (zeroed by the caller for a plain gradient); the pair splits' partials are
// added in split order.
extern "C" int esb_spconv_wgrad(const void* x, const void* dy, const int* pair_in, const int* pair_out,
                                const int* k_offsets, float* dw, long long n_pairs_hint, int cin, int cout, int K,
                                int dtype, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  ESB_CHECK_ARG(cin > 0 && cout > 0 && K > 0, "esb_spconv_wgrad: bad channel/kernel sizes");
  ESB_CHECK_ARG(dtype == ESB_F32 || dtype == ESB_BF16, "esb_spconv_wgrad: dtype must be f32 or bf16");
  int ci_t = esb_div_up(cin, TM), co_t = esb_div_up(cout, TN);
  // aim for ~4 CTAs/SM over the SMs, but keep >= 256 pairs per split
  long long per_k = n_pairs_hint / K + 1;
  int splits = (int)(4LL * esb_sm_count() / ((long long)K * ci_t * co_t));
  int max_by_pairs = (int)(per_k / 256) + 1;
  if (splits > max_by_pairs) splits = max_by_pairs;
  if (splits < 1) splits = 1;
  if (splits > 64) splits = 64;
  dim3 grid(K * splits, ci_t, co_t);
  const long long width = (long long)K * cin * cout;
  float* part = nullptr;
  ESB_CUDA_CALL(esb_scratch_alloc((void**)&part, sizeof(float) * splits * width, stream));
  ESB_CUDA_CALL(cudaMemsetAsync(part, 0, sizeof(float) * splits * width, stream));
  if (dtype == ESB_F32)
    spconv_wgrad_kernel<float><<<grid, 256, 0, stream>>>((const float*)x, (const float*)dy, pair_in, pair_out,
                                                          k_offsets, part, cin, cout, splits);
  else
    spconv_wgrad_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)dy,
                                                                  pair_in, pair_out, k_offsets, part, cin, cout, splits);
  ESB_CUDA_LAUNCH_CHECK("spconv_wgrad_kernel");
  int rc = esb_sum_partial_rows(part, splits, width, dw, 1, stream);
  ESB_CUDA_CALL(esb_scratch_free(part, stream));
  return rc;
}
