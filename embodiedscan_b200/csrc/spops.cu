// esb200 — row-feature operators around the sparse convolutions: strided max pooling, segmented
// normalisation (BatchNorm over all rows = 1 segment, InstanceNorm = 1 segment per scan) fused with the
// residual add and the activation. Replace ME.MinkowskiMaxPooling / MinkowskiInstanceNorm / MinkowskiBatchNorm /
// MinkowskiReLU / MinkowskiELU (†upstream) as used at embodiedscan/models/backbones/mink_resnet.py:64-69 and
// embodiedscan/models/dense_heads/fcaf3d_head.py:919-947. All HBM/L2-bound, vectorised along channels.
#include "common.cuh"

namespace {

// ---------------- max pooling over a kernel map ----------------
template <typename T>
__global__ void maxpool_fwd_kernel(const T* __restrict__ x, const int* __restrict__ nbr, T* __restrict__ y,
                                   int* __restrict__ arg, long long n_out, int C, int K) {
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t >= n_out * C) return;
  long long o = t / C;
  int c = (int)(t - o * C);
  float best = -INFINITY;
  int best_i = -1;
  for (int k = 0; k < K; ++k) {
    int i = nbr[(long long)k * n_out + o];
    if (i < 0) continue;
    float v = esb_to_float<T>(x[(long long)i * C + c]);
    if (best_i < 0 || v > best) {
      best = v;
      best_i = i;
    }
  }
  y[t] = esb_from_float<T>(best_i >= 0 ? best : 0.f);
  arg[t] = best_i;
}

template <typename T>
__global__ void maxpool_bwd_kernel(const T* __restrict__ dy, const int* __restrict__ arg, T* __restrict__ dx,
                                   long long n_out, int C) {
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t >= n_out * C) return;
  int c = (int)(t % C);
  int i = arg[t];
  // k2/s2 windows do not overlap: every (input row, channel) is the argmax of at most one output.
  if (i >= 0) dx[(long long)i * C + c] = dy[t];
}

// seg_off == NULL means ONE segment covering all n_total rows (BatchNorm): no host->device offset upload per call
__device__ __forceinline__ int seg_begin(const int* __restrict__ seg_off, int s) { return seg_off ? seg_off[s] : 0; }
__device__ __forceinline__ int seg_end(const int* __restrict__ seg_off, int s, int n_total) {
  return seg_off ? seg_off[s + 1] : n_total;
}

// ---------------- segmented column statistics ----------------
// pass 1: sum over rows of each segment; pass 2 (centered): sum (x-mean)^2. Block (bx, s, cz) writes its partial to
// out[bx][s][c]; esb_sum_partial_rows adds the row blocks in order.
template <typename T, int MODE>  // MODE 0: sum x ; 1: sum (x - mean[s][c])^2
__global__ void seg_colstat_kernel(const T* __restrict__ x, const int* __restrict__ seg_off, const float* __restrict__ mean,
                                   float* __restrict__ out, int C, int rows_per_block, int n_total) {
  __shared__ float red[8][33];
  const int s = blockIdx.y;
  const int c = blockIdx.z * 32 + threadIdx.x;
  const int r_beg = seg_begin(seg_off, s) + blockIdx.x * rows_per_block;
  const int r_end = min(seg_end(seg_off, s, n_total), r_beg + rows_per_block);
  float acc = 0.f;
  if (c < C) {
    float mu = MODE == 1 ? mean[s * C + c] : 0.f;
    for (int r = r_beg + threadIdx.y; r < r_end; r += 8) {
      float v = esb_to_float<T>(x[(long long)r * C + c]);
      if (MODE == 1) {
        v -= mu;
        acc = fmaf(v, v, acc);
      } else {
        acc += v;
      }
    }
  }
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float t = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) t += red[j][threadIdx.x];
    out[((long long)blockIdx.x * gridDim.y + s) * C + c] = t;
  }
}

// mean = sum / n ; (in place)
__global__ void seg_finalize_mean_kernel(float* __restrict__ sum, const int* __restrict__ seg_off, int S, int C,
                                         int n_total) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= S * C) return;
  int s = t / C;
  int n = seg_end(seg_off, s, n_total) - seg_begin(seg_off, s);
  sum[t] = n > 0 ? sum[t] / (float)n : 0.f;
}
// var(biased) -> rstd ; optionally update running stats (momentum, unbiased var) like nn.BatchNorm1d
__global__ void seg_finalize_rstd_kernel(const float* __restrict__ mean, float* __restrict__ var_to_rstd,
                                         const int* __restrict__ seg_off, int S, int C, float eps,
                                         float* __restrict__ running_mean, float* __restrict__ running_var,
                                         float momentum, int n_total) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= S * C) return;
  int s = t / C;
  int n = seg_end(seg_off, s, n_total) - seg_begin(seg_off, s);
  float var = n > 0 ? var_to_rstd[t] / (float)n : 0.f;
  if (running_mean != nullptr && S == 1) {
    float unbiased = n > 1 ? var * (float)n / (float)(n - 1) : var;
    running_mean[t] = (1.f - momentum) * running_mean[t] + momentum * mean[t];
    running_var[t] = (1.f - momentum) * running_var[t] + momentum * unbiased;
  }
  var_to_rstd[t] = rsqrtf(var + eps);
}

__device__ __forceinline__ float act_fwd(float z, int act) {
  if (act == 1) return fmaxf(z, 0.f);
  if (act == 2) return z > 0.f ? z : expm1f(z);
  return z;
}
// derivative of the activation expressed through its OUTPUT y
__device__ __forceinline__ float act_bwd_from_out(float y, int act) {
  if (act == 1) return y > 0.f ? 1.f : 0.f;
  if (act == 2) return y > 0.f ? 1.f : y + 1.f;
  return 1.f;
}

// y = act((x - mean) * rstd * gamma + beta + res)
template <typename T>
__global__ void norm_apply_kernel(const T* __restrict__ x, const T* __restrict__ res, const int* __restrict__ row_seg,
                                  const float* __restrict__ mean, const float* __restrict__ rstd,
                                  const float* __restrict__ gamma, const float* __restrict__ beta, T* __restrict__ y,
                                  long long N, int C, int act) {
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t >= N * C) return;
  long long r = t / C;
  int c = (int)(t - r * C);
  int s = row_seg ? row_seg[r] : 0;
  float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
  float z = (esb_to_float<T>(x[t]) - mean[s * C + c]) * rstd[s * C + c] * g + b;
  if (res) z += esb_to_float<T>(res[t]);
  y[t] = esb_from_float<T>(act_fwd(z, act));
}

// 8-wide helpers (16 B for bf16, 2 x 16 B for fp32)
template <typename T>
__device__ __forceinline__ void load8(const T* p, float v[8]);
template <>
__device__ __forceinline__ void load8<float>(const float* p, float v[8]) {
  float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <>
__device__ __forceinline__ void load8<__nv_bfloat16>(const __nv_bfloat16* p, float v[8]) {
  uint4 raw = *reinterpret_cast<const uint4*>(p);
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
  for (int i = 0; i < 4; ++i) { v[2 * i] = __low2float(h[i]); v[2 * i + 1] = __high2float(h[i]); }
}
template <typename T>
__device__ __forceinline__ void store8(T* p, const float v[8]);
template <>
__device__ __forceinline__ void store8<float>(float* p, const float v[8]) {
  reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}
template <>
__device__ __forceinline__ void store8<__nv_bfloat16>(__nv_bfloat16* p, const float v[8]) {
  uint4 o;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = o;
}

// y = act((x - mean) * rstd * gamma + beta + res), 8 channels per thread (C % 8 == 0)
template <typename T>
__global__ void norm_apply_vec8_kernel(const T* __restrict__ x, const T* __restrict__ res, const int* __restrict__ row_seg,
                                       const float* __restrict__ mean, const float* __restrict__ rstd,
                                       const float* __restrict__ gamma, const float* __restrict__ beta, T* __restrict__ y,
                                       long long n_vec, int C, int act) {
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t >= n_vec) return;
  const int cv = C >> 3;
  const long long r = t / cv;
  const int c0 = (int)(t - r * cv) << 3;
  const int s = row_seg ? row_seg[r] : 0;
  float v[8], rr[8];
  load8<T>(x + t * 8, v);
  if (res) load8<T>(res + t * 8, rr);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = c0 + i;
    float z = (v[i] - mean[s * C + c]) * rstd[s * C + c] * (gamma ? gamma[c] : 1.f) + (beta ? beta[c] : 0.f);
    if (res) z += rr[i];
    v[i] = act_fwd(z, act);
  }
  store8<T>(y + t * 8, v);
}

template <typename T>
__global__ void norm_bwd_apply_vec8_kernel(const T* __restrict__ x, const T* __restrict__ y, const T* __restrict__ dy,
                                           const int* __restrict__ row_seg, const int* __restrict__ seg_off,
                                           const float* __restrict__ mean, const float* __restrict__ rstd,
                                           const float* __restrict__ gamma, const float* __restrict__ sg,
                                           const float* __restrict__ sgx, T* __restrict__ dx, T* __restrict__ dres,
                                           long long N, long long n_vec, int C, int act) {
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t >= n_vec) return;
  const int cv = C >> 3;
  const long long r = t / cv;
  const int c0 = (int)(t - r * cv) << 3;
  const int s = row_seg ? row_seg[r] : 0;
  const float inv_n = 1.f / (float)max(seg_end(seg_off, s, (int)N) - seg_begin(seg_off, s), 1);
  float xv[8], yv[8], gv[8], ov[8];
  load8<T>(x + t * 8, xv);
  load8<T>(y + t * 8, yv);
  load8<T>(dy + t * 8, gv);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = c0 + i;
    float g = gv[i] * act_bwd_from_out(yv[i], act);
    float rs = rstd[s * C + c];
    float xh = (xv[i] - mean[s * C + c]) * rs;
    ov[i] = (gamma ? gamma[c] : 1.f) * rs * (g - sg[s * C + c] * inv_n - xh * sgx[s * C + c] * inv_n);
    gv[i] = g;
  }
  store8<T>(dx + t * 8, ov);
  if (dres) store8<T>(dres + t * 8, gv);
}

// backward reduce: sg[s][c] = sum g ; sgx[s][c] = sum g * xhat, with g = dy * act'(y); partials per row block as above
template <typename T>
__global__ void norm_bwd_reduce_kernel(const T* __restrict__ x, const T* __restrict__ y, const T* __restrict__ dy,
                                       const int* __restrict__ seg_off, const float* __restrict__ mean,
                                       const float* __restrict__ rstd, float* __restrict__ sg, float* __restrict__ sgx,
                                       int C, int rows_per_block, int act, int n_total) {
  __shared__ float red0[8][33];
  __shared__ float red1[8][33];
  const int s = blockIdx.y;
  const int c = blockIdx.z * 32 + threadIdx.x;
  const int r_beg = seg_begin(seg_off, s) + blockIdx.x * rows_per_block;
  const int r_end = min(seg_end(seg_off, s, n_total), r_beg + rows_per_block);
  float a0 = 0.f, a1 = 0.f;
  if (c < C) {
    float mu = mean[s * C + c], rs = rstd[s * C + c];
    for (int r = r_beg + threadIdx.y; r < r_end; r += 8) {
      long long idx = (long long)r * C + c;
      float g = esb_to_float<T>(dy[idx]) * act_bwd_from_out(esb_to_float<T>(y[idx]), act);
      float xh = (esb_to_float<T>(x[idx]) - mu) * rs;
      a0 += g;
      a1 = fmaf(g, xh, a1);
    }
  }
  red0[threadIdx.y][threadIdx.x] = a0;
  red1[threadIdx.y][threadIdx.x] = a1;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float t0 = 0.f, t1 = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      t0 += red0[j][threadIdx.x];
      t1 += red1[j][threadIdx.x];
    }
    sg[((long long)blockIdx.x * gridDim.y + s) * C + c] = t0;
    sgx[((long long)blockIdx.x * gridDim.y + s) * C + c] = t1;
  }
}

// dx = gamma*rstd*(g - mean_s(g) - xhat*mean_s(g*xhat)) ; dres = g
template <typename T>
__global__ void norm_bwd_apply_kernel(const T* __restrict__ x, const T* __restrict__ y, const T* __restrict__ dy,
                                      const int* __restrict__ row_seg, const int* __restrict__ seg_off,
                                      const float* __restrict__ mean, const float* __restrict__ rstd,
                                      const float* __restrict__ gamma, const float* __restrict__ sg,
                                      const float* __restrict__ sgx, T* __restrict__ dx, T* __restrict__ dres,
                                      long long N, int C, int act) {
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t >= N * C) return;
  long long r = t / C;
  int c = (int)(t - r * C);
  int s = row_seg ? row_seg[r] : 0;
  float inv_n = 1.f / (float)max(seg_end(seg_off, s, (int)N) - seg_begin(seg_off, s), 1);
  float g = esb_to_float<T>(dy[t]) * act_bwd_from_out(esb_to_float<T>(y[t]), act);
  float rs = rstd[s * C + c];
  float xh = (esb_to_float<T>(x[t]) - mean[s * C + c]) * rs;
  float gm = gamma ? gamma[c] : 1.f;
  float v = gm * rs * (g - sg[s * C + c] * inv_n - xh * sgx[s * C + c] * inv_n);
  dx[t] = esb_from_float<T>(v);
  if (dres) dres[t] = esb_from_float<T>(g);
}

// plain activation (used where no normalisation precedes it)
template <typename T>
__global__ void act_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, long long n, int act) {
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t < n) y[t] = esb_from_float<T>(act_fwd(esb_to_float<T>(x[t]), act));
}

// y = act(x + bias[c] + res) over (rows, C) row-major (an NHWC activation is exactly that), 8 channels per thread.
// Replaces cuDNN's broadcast bias add + the separate residual add + ReLU of the folded conv+BN blocks (3 passes -> 1).
template <typename T>
__global__ void bias_act_kernel(const T* __restrict__ x, const float* __restrict__ bias, const T* __restrict__ res,
                                T* __restrict__ y, long long n_vec, int C, int act) {
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t >= n_vec) return;
  const int cv = C / 8;
  const int c0 = (int)(t % cv) * 8;
  float v[8], r[8];
  if (sizeof(T) == 2) {
    uint4 raw = reinterpret_cast<const uint4*>(x)[t];
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
    for (int i = 0; i < 4; ++i) { v[2 * i] = __low2float(h[i]); v[2 * i + 1] = __high2float(h[i]); }
    if (res) {
      uint4 rr = reinterpret_cast<const uint4*>(res)[t];
      const __nv_bfloat162* g = reinterpret_cast<const __nv_bfloat162*>(&rr);
#pragma unroll
      for (int i = 0; i < 4; ++i) { r[2 * i] = __low2float(g[i]); r[2 * i + 1] = __high2float(g[i]); }
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) { v[i] = esb_to_float<T>(x[t * 8 + i]); r[i] = res ? esb_to_float<T>(res[t * 8 + i]) : 0.f; }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = act_fwd(v[i] + (bias ? bias[c0 + i] : 0.f) + (res ? r[i] : 0.f), act);
  if (sizeof(T) == 2) {
    uint4 o;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
    reinterpret_cast<uint4*>(y)[t] = o;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) y[t * 8 + i] = esb_from_float<T>(v[i]);
  }
}

// dx = dy * act'(y) expressed through the OUTPUT y (8 elements per thread)
template <typename T>
__global__ void act_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ y, T* __restrict__ dx, long long n,
                               int act) {
  long long t = (blockIdx.x * (long long)blockDim.x + threadIdx.x) * 8;
  if (t + 8 <= n) {
    float g[8], o[8];
    load8<T>(dy + t, g);
    load8<T>(y + t, o);
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i] *= act_bwd_from_out(o[i], act);
    store8<T>(dx + t, g);
  } else {
    for (int i = 0; i < 8; ++i)
      if (t + i < n)
        dx[t + i] = esb_from_float<T>(esb_to_float<T>(dy[t + i]) * act_bwd_from_out(esb_to_float<T>(y[t + i]), act));
  }
}

// ---------------- fused BatchNorm statistics (one segment, bf16 rows) ----------------
// ONE pass over x: sum and sum of squares of v = x - pivot (pivot = row 0 of the column: keeps E[v^2] - E[v]^2 free of the
// catastrophic cancellation a raw single-pass variance has when |mean| >> std), accumulated per block in shared memory and
// added to stats[0] (sum v), stats[1] (sum v^2). The apply kernel turns them into mean / rstd on the fly.
template <typename T>
__global__ void bn_stats_kernel(const T* __restrict__ x, long long N, int C, int rows_per_block, float* __restrict__ part) {
  extern __shared__ float sh[];                    // [rstep][2][C]: one slot per row lane, summed in lane order
  const int tpr = C / 8;                           // threads per row (16-byte pieces)
  const int c = (threadIdx.x % tpr) * 8;
  const int rsub = threadIdx.x / tpr, rstep = blockDim.x / tpr;
  const long long r_beg = (long long)blockIdx.x * rows_per_block;
  const long long r_end = r_beg + rows_per_block < N ? r_beg + rows_per_block : N;
  float piv[8], sum[8], sq[8];
  load8<T>(x + c, piv);
#pragma unroll
  for (int e = 0; e < 8; ++e) sum[e] = sq[e] = 0.f;
  if (rsub < rstep) {
    for (long long r = r_beg + rsub; r < r_end; r += rstep) {
      float v[8];
      load8<T>(x + r * C + c, v);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float d = v[e] - piv[e];
        sum[e] += d;
        sq[e] = fmaf(d, d, sq[e]);
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      sh[(2 * rsub) * C + c + e] = sum[e];
      sh[(2 * rsub + 1) * C + c + e] = sq[e];
    }
  }
  __syncthreads();
  // this block's partial: part[blockIdx][0 .. C) = sum, [C .. 2C) = sum of squares
  for (int i = threadIdx.x; i < 2 * C; i += blockDim.x) {
    const int k = i < C ? 0 : 1, ci = i < C ? i : i - C;
    float t = 0.f;
    for (int r = 0; r < rstep; ++r) t += sh[(2 * r + k) * C + ci];
    part[(long long)blockIdx.x * 2 * C + i] = t;
  }
}

// y = act((x - mean) * rstd * gamma + beta + res) with mean / rstd derived from the raw sums of bn_stats_kernel; block 0 also
// publishes mean -> stats[2], rstd -> stats[3] (what the backward pass reads) and updates the running statistics.
template <typename T>
__global__ void bn_apply_fused_kernel(const T* __restrict__ x, const T* __restrict__ res, long long N, int C,
                                      const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                      float* __restrict__ running_mean, float* __restrict__ running_var, float momentum, int act,
                                      float* __restrict__ stats, T* __restrict__ y) {
  const float inv_n = 1.f / (float)N;
  if (blockIdx.x == 0) {
    for (int i = threadIdx.x; i < C; i += blockDim.x) {
      const float m = stats[i] * inv_n;
      const float var = fmaxf(stats[C + i] * inv_n - m * m, 0.f);
      const float mean = esb_to_float<T>(x[i]) + m;
      stats[2 * C + i] = mean;
      stats[3 * C + i] = rsqrtf(var + eps);
      if (running_mean != nullptr) {
        const float unbiased = N > 1 ? var * (float)N / (float)(N - 1) : var;
        running_mean[i] = (1.f - momentum) * running_mean[i] + momentum * mean;
        running_var[i] = (1.f - momentum) * running_var[i] + momentum * unbiased;
      }
    }
  }
  const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const int cv = C / 8;
  if (t >= N * cv) return;
  const long long r = t / cv;
  const int c = (int)(t - r * cv) * 8;
  float v[8], piv[8], rs[8];
  load8<T>(x + r * C + c, v);
  load8<T>(x + c, piv);
  if (res != nullptr) load8<T>(res + r * C + c, rs);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float m = stats[c + e] * inv_n;
    const float var = fmaxf(stats[C + c + e] * inv_n - m * m, 0.f);
    const float g = gamma ? gamma[c + e] : 1.f, b = beta ? beta[c + e] : 0.f;
    float z = (v[e] - (piv[e] + m)) * rsqrtf(var + eps) * g + b;
    if (res != nullptr) z += rs[e];
    v[e] = act_fwd(z, act);
  }
  store8<T>(y + r * C + c, v);
}

// out[r, :] = a[ia(r), :] + b[ib[r], :] with ia(r) = ia ? ia[r] : (r < na ? r : -1); a negative index contributes zeros.
// One thread per (row, 8-channel piece): the row gather of unions (A + B on different coordinate maps), of their gradients
// and of every `x[idx]` on the path; each output element is written once (no atomics).
template <typename T>
__global__ void gather2_rows_kernel(const T* __restrict__ a, const int* __restrict__ ia, long long na, const T* __restrict__ b,
                                    const int* __restrict__ ib, T* __restrict__ out, long long n_vec, int C) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_vec) return;
  const int cv = C / 8;
  const long long r = i / cv;
  const int c = (int)(i - r * cv) * 8;
  const long long ra = ia ? (long long)ia[r] : (r < na ? r : -1);
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] = 0.f;
  if (ra >= 0) load8<T>(a + ra * C + c, v);
  if (b != nullptr) {
    const int rb = ib[r];
    if (rb >= 0) {
      float w[8];
      load8<T>(b + (long long)rb * C + c, w);
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] += w[e];
    }
  }
  store8<T>(out + r * C + c, v);
}

}  // namespace

#define DISPATCH_T(dtype, ...)                         \
  if (dtype == ESB_F32) {                              \
    using T = float;                                   \
    __VA_ARGS__;                                       \
  } else {                                             \
    using T = __nv_bfloat16;                           \
    __VA_ARGS__;                                       \
  }

extern "C" int esb_maxpool_fwd(const void* x, const int* nbr, void* y, int* arg, long long n_out, int C, int K,
                               int dtype, void* stream) {
  if (n_out == 0) return ESB_OK;
  DISPATCH_T(dtype, (maxpool_fwd_kernel<T><<<esb_div_up(n_out * C, 256), 256, 0, (cudaStream_t)stream>>>(
                        (const T*)x, nbr, (T*)y, arg, n_out, C, K)));
  ESB_CUDA_LAUNCH_CHECK("maxpool_fwd_kernel");
  return ESB_OK;
}

// dx must be zero-initialised by the caller.
extern "C" int esb_maxpool_bwd(const void* dy, const int* arg, void* dx, long long n_out, int C, int dtype,
                               void* stream) {
  if (n_out == 0) return ESB_OK;
  DISPATCH_T(dtype, (maxpool_bwd_kernel<T><<<esb_div_up(n_out * C, 256), 256, 0, (cudaStream_t)stream>>>(
                        (const T*)dy, arg, (T*)dx, n_out, C)));
  ESB_CUDA_LAUNCH_CHECK("maxpool_bwd_kernel");
  return ESB_OK;
}

// Segmented normalisation forward.
//  seg_off (S+1) device int32 row offsets (rows of a segment are contiguous); row_seg (N) segment id per row or NULL
//  when S==1. mean/rstd (S,C) fp32 outputs (saved for backward). gamma/beta may be NULL. res may be NULL.
//  running_mean/var (C) updated when non-NULL and S==1 (BatchNorm training semantics, unbiased running var).
// seg_off may be NULL when S == 1 (one segment = all N rows).
extern "C" int esb_norm_fwd(const void* x, const void* res, const int* seg_off, const int* row_seg, int S,
                            long long N, int max_seg_rows, int C, const float* gamma, const float* beta, float eps,
                            float* running_mean, float* running_var, float momentum, int act, float* mean, float* rstd,
                            void* y, int dtype, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  ESB_CHECK_ARG(S >= 1 && C >= 1, "esb_norm_fwd: bad S/C");
  ESB_CHECK_ARG(seg_off != nullptr || S == 1, "esb_norm_fwd: seg_off may be NULL only for a single segment");
  ESB_CUDA_CALL(cudaMemsetAsync(mean, 0, sizeof(float) * S * C, stream));
  ESB_CUDA_CALL(cudaMemsetAsync(rstd, 0, sizeof(float) * S * C, stream));
  if (N == 0) return ESB_OK;
  const int rpb = 256;
  dim3 grid(esb_div_up(max_seg_rows > 0 ? max_seg_rows : 1, rpb), S, esb_div_up(C, 32)), block(32, 8);
  int fin = esb_div_up(S * C, 256);
  float* part = nullptr;
  ESB_CUDA_CALL(esb_scratch_alloc((void**)&part, sizeof(float) * grid.x * S * C, stream));
  int rc = ESB_OK;
  DISPATCH_T(dtype, {
    seg_colstat_kernel<T, 0><<<grid, block, 0, stream>>>((const T*)x, seg_off, nullptr, part, C, rpb, (int)N);
    rc = esb_sum_partial_rows(part, (int)grid.x, (long long)S * C, mean, 0, stream);
    seg_finalize_mean_kernel<<<fin, 256, 0, stream>>>(mean, seg_off, S, C, (int)N);
    seg_colstat_kernel<T, 1><<<grid, block, 0, stream>>>((const T*)x, seg_off, mean, part, C, rpb, (int)N);
    if (rc == ESB_OK) rc = esb_sum_partial_rows(part, (int)grid.x, (long long)S * C, rstd, 0, stream);
    seg_finalize_rstd_kernel<<<fin, 256, 0, stream>>>(mean, rstd, seg_off, S, C, eps, running_mean, running_var, momentum,
                                                      (int)N);
    if (C % 8 == 0)
      norm_apply_vec8_kernel<T><<<esb_div_up(N * (C / 8), 256), 256, 0, stream>>>(
          (const T*)x, (const T*)res, row_seg, mean, rstd, gamma, beta, (T*)y, N * (C / 8), C, act);
    else
      norm_apply_kernel<T><<<esb_div_up(N * C, 256), 256, 0, stream>>>((const T*)x, (const T*)res, row_seg, mean, rstd,
                                                                       gamma, beta, (T*)y, N, C, act);
  });
  ESB_CUDA_CALL(esb_scratch_free(part, stream));
  if (rc != ESB_OK) return rc;
  ESB_CUDA_LAUNCH_CHECK("esb_norm_fwd");
  return ESB_OK;
}

// Inference-mode normalisation with given statistics (BatchNorm eval): mean/rstd (1,C) supplied by the caller.
extern "C" int esb_norm_apply(const void* x, const void* res, const int* row_seg, long long N, int C,
                              const float* mean, const float* rstd, const float* gamma, const float* beta, int act,
                              void* y, int dtype, void* stream) {
  if (N == 0) return ESB_OK;
  DISPATCH_T(dtype, (norm_apply_kernel<T><<<esb_div_up(N * C, 256), 256, 0, (cudaStream_t)stream>>>(
                        (const T*)x, (const T*)res, row_seg, mean, rstd, gamma, beta, (T*)y, N, C, act)));
  ESB_CUDA_LAUNCH_CHECK("norm_apply_kernel");
  return ESB_OK;
}

// Backward: dgamma = sgx summed over segments, dbeta = sg summed over segments (the host sums the (S,C) arrays).
extern "C" int esb_norm_bwd(const void* x, const void* y, const void* dy, const int* seg_off, const int* row_seg, int S,
                            long long N, int max_seg_rows, int C, const float* mean, const float* rstd,
                            const float* gamma, int act, float* sg, float* sgx, void* dx, void* dres, int zero_sums,
                            int dtype, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  // zero_sums = 0: sg/sgx are the (already zeroed, used once per step) gradient slots of beta/gamma in the flat arena
  if (zero_sums) {
    ESB_CUDA_CALL(cudaMemsetAsync(sg, 0, sizeof(float) * S * C, stream));
    ESB_CUDA_CALL(cudaMemsetAsync(sgx, 0, sizeof(float) * S * C, stream));
  }
  if (N == 0) return ESB_OK;
  const int rpb = 256;
  dim3 grid(esb_div_up(max_seg_rows > 0 ? max_seg_rows : 1, rpb), S, esb_div_up(C, 32)), block(32, 8);
  const long long width = (long long)S * C;
  float* part = nullptr;
  ESB_CUDA_CALL(esb_scratch_alloc((void**)&part, sizeof(float) * 2 * grid.x * width, stream));
  int rc = ESB_OK;
  DISPATCH_T(dtype, {
    norm_bwd_reduce_kernel<T><<<grid, block, 0, stream>>>((const T*)x, (const T*)y, (const T*)dy, seg_off, mean, rstd,
                                                          part, part + grid.x * width, C, rpb, act, (int)N);
    rc = esb_sum_partial_rows(part, (int)grid.x, width, sg, 1, stream);
    if (rc == ESB_OK) rc = esb_sum_partial_rows(part + grid.x * width, (int)grid.x, width, sgx, 1, stream);
    if (C % 8 == 0)
      norm_bwd_apply_vec8_kernel<T><<<esb_div_up(N * (C / 8), 256), 256, 0, stream>>>(
          (const T*)x, (const T*)y, (const T*)dy, row_seg, seg_off, mean, rstd, gamma, sg, sgx, (T*)dx, (T*)dres, N,
          N * (C / 8), C, act);
    else
      norm_bwd_apply_kernel<T><<<esb_div_up(N * C, 256), 256, 0, stream>>>(
          (const T*)x, (const T*)y, (const T*)dy, row_seg, seg_off, mean, rstd, gamma, sg, sgx, (T*)dx, (T*)dres, N, C, act);
  });
  ESB_CUDA_CALL(esb_scratch_free(part, stream));
  if (rc != ESB_OK) return rc;
  ESB_CUDA_LAUNCH_CHECK("esb_norm_bwd");
  return ESB_OK;
}

extern "C" int esb_act_fwd(const void* x, void* y, long long n, int act, int dtype, void* stream) {
  if (n == 0) return ESB_OK;
  DISPATCH_T(dtype, (act_fwd_kernel<T><<<esb_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>((const T*)x, (T*)y, n, act)));
  ESB_CUDA_LAUNCH_CHECK("act_fwd_kernel");
  return ESB_OK;
}

// y = act(x + bias[c] + res), x/res/y (rows, C) row-major with C % 8 == 0; y may alias x. bias fp32 (C) or NULL.
extern "C" int esb_bias_act_fwd(const void* x, const float* bias, const void* res, void* y, long long rows, int C, int act,
                                int dtype, void* stream) {
  ESB_CHECK_ARG(C % 8 == 0, "esb_bias_act_fwd: C must be a multiple of 8");
  long long n_vec = rows * (C / 8);
  if (n_vec == 0) return ESB_OK;
  DISPATCH_T(dtype, (bias_act_kernel<T><<<esb_div_up(n_vec, 256), 256, 0, (cudaStream_t)stream>>>(
                        (const T*)x, bias, (const T*)res, (T*)y, n_vec, C, act)));
  ESB_CUDA_LAUNCH_CHECK("bias_act_kernel");
  return ESB_OK;
}

extern "C" int esb_act_bwd(const void* dy, const void* y, void* dx, long long n, int act, int dtype, void* stream) {
  if (n == 0) return ESB_OK;
  DISPATCH_T(dtype, (act_bwd_kernel<T><<<esb_div_up(n, 256 * 8), 256, 0, (cudaStream_t)stream>>>(
                        (const T*)dy, (const T*)y, (T*)dx, n, act)));
  ESB_CUDA_LAUNCH_CHECK("act_bwd_kernel");
  return ESB_OK;
}

// out (n, C) = a[ia] + b[ib] row-wise (see gather2_rows_kernel). ia may be NULL (identity on the first na rows), b / ib may be
// NULL (plain gather). C % 8 == 0.
extern "C" int esb_gather2_rows(const void* a, const int* ia, long long na, const void* b, const int* ib, void* out, long long n,
                                int C, int dtype, void* stream) {
  ESB_CHECK_ARG(C > 0 && C % 8 == 0, "esb_gather2_rows: C must be a positive multiple of 8");
  ESB_CHECK_ARG((b == nullptr) == (ib == nullptr), "esb_gather2_rows: b and ib go together");
  const long long n_vec = n * (C / 8);
  if (n_vec == 0) return ESB_OK;
  DISPATCH_T(dtype, (gather2_rows_kernel<T><<<esb_div_up(n_vec, 256), 256, 0, (cudaStream_t)stream>>>(
                        (const T*)a, ia, na, (const T*)b, ib, (T*)out, n_vec, C)));
  ESB_CUDA_LAUNCH_CHECK("gather2_rows_kernel");
  return ESB_OK;
}

// BatchNorm (one segment) forward in TWO launches: one statistics pass + one apply pass (esb_norm_fwd takes five: two
// centred passes with their finalisation kernels, the parity arithmetic). stats (4, C) fp32: [sum v, sum v^2, mean, rstd];
// rows 2 and 3 are the saved tensors of the backward pass. x / res / y (N, C), C % 8 == 0, 16 <= C <= 2048.
extern "C" int esb_batchnorm_fwd_fused(const void* x, const void* res, long long N, int C, const float* gamma, const float* beta,
                                       float eps, float* running_mean, float* running_var, float momentum, int act, float* stats,
                                       void* y, int dtype, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  ESB_CHECK_ARG(C % 8 == 0 && C >= 8 && C <= 2048, "esb_batchnorm_fwd_fused: C must be a multiple of 8 in [8, 2048]");
  ESB_CUDA_CALL(cudaMemsetAsync(stats, 0, sizeof(float) * 2 * C, stream));
  if (N == 0) return ESB_OK;
  long long rpb = (N + 2 * esb_sm_count() - 1) / (2 * esb_sm_count());
  if (rpb < 64) rpb = 64;
  const int grid_a = esb_div_up(N, rpb);
  const long long n_vec = N * (C / 8);
  const int rstep = 256 / (C / 8);
  float* part = nullptr;
  ESB_CUDA_CALL(esb_scratch_alloc((void**)&part, sizeof(float) * 2 * C * grid_a, stream));
  DISPATCH_T(dtype, (bn_stats_kernel<T><<<grid_a, 256, 2 * rstep * C * sizeof(float), stream>>>((const T*)x, N, C, (int)rpb, part)));
  ESB_CUDA_LAUNCH_CHECK("bn_stats_kernel");
  int rc = esb_sum_partial_rows(part, grid_a, 2LL * C, stats, 0, stream);
  ESB_CUDA_CALL(esb_scratch_free(part, stream));
  if (rc != ESB_OK) return rc;
  DISPATCH_T(dtype, (bn_apply_fused_kernel<T><<<esb_div_up(n_vec, 256), 256, 0, stream>>>(
                        (const T*)x, (const T*)res, N, C, gamma, beta, eps, running_mean, running_var, momentum, act, stats,
                        (T*)y)));
  ESB_CUDA_LAUNCH_CHECK("bn_apply_fused_kernel");
  return ESB_OK;
}

// ---------------- FCAF3D head epilogue (fcaf3d_head.py:1116-1149 after the three 1x1 convolutions) ----------------
// `out` (N, W) bf16 is the one padded head GEMM: columns [0, n_cls) class logits without bias, column n_cls the centre-ness,
// the next n_reg columns the box regression, the rest zero padding. One warp per row writes
//   cls   (N, n_cls) bf16 = out + bf16(bias)                     (conv_cls bias)
//   centre(N, 1)     fp32
//   bbox  (N, n_reg) fp32: columns [0, n_exp) max(exp(s * x), lo) (the Scale layer, exp and clamp(min=lo)), the rest x
//   prune (N, 1)     fp32 = max over the class logits            (the pruning score of the parent level)
// HBM-bound: 2 B * W read + 2 B * n_cls + 4 B * (2 + n_reg) written per row.
__global__ void __launch_bounds__(256) head_split_fwd_kernel(const __nv_bfloat16* __restrict__ out,
                                                             const float* __restrict__ bias, const float* __restrict__ scale,
                                                             long long N, int W, int n_cls, int n_reg, int n_exp, float lo,
                                                             __nv_bfloat16* __restrict__ cls, float* __restrict__ centre,
                                                             float* __restrict__ bbox, float* __restrict__ prune) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  const float s = *scale;
  for (long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < N; row += warps) {
    const __nv_bfloat16* o = out + row * W;
    float m = -INFINITY;
    for (int c = lane; c < n_cls; c += 32) {
      const float b = __bfloat162float(__float2bfloat16(bias[c]));
      const __nv_bfloat16 v = __float2bfloat16(__bfloat162float(o[c]) + b);
      cls[row * n_cls + c] = v;
      m = fmaxf(m, __bfloat162float(v));
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, d));
    if (lane == 0) {
      prune[row] = m;
      centre[row] = __bfloat162float(o[n_cls]);
    }
    if (lane < n_reg) {
      const float x = __bfloat162float(o[n_cls + 1 + lane]);
      bbox[row * n_reg + lane] = lane < n_exp ? fmaxf(expf(s * x), lo) : x;
    }
  }
}

// Backward of the above: dout (N, W) bf16 (padding columns zero), dbias (n_cls) += column sums of dcls, dscale += the Scale
// gradient. clamp(min=lo) passes the gradient where exp(s x) >= lo. n_cls <= 512 (16 class columns per lane).
__global__ void __launch_bounds__(256) head_split_bwd_kernel(const __nv_bfloat16* __restrict__ out,
                                                             const __nv_bfloat16* __restrict__ dcls,
                                                             const float* __restrict__ dcentre, const float* __restrict__ dbbox,
                                                             const float* __restrict__ scale, long long N, int W, int n_cls,
                                                             int n_reg, int n_exp, float lo, __nv_bfloat16* __restrict__ dout,
                                                             float* __restrict__ dbias, float* __restrict__ dscale) {
  extern __shared__ float s_bias[];                  // n_cls block-level column sums
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  const float s = *scale;
  for (int c = threadIdx.x; c < n_cls; c += blockDim.x) s_bias[c] = 0.f;
  __syncthreads();
  float acc[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) acc[k] = 0.f;
  float ds = 0.f;
  const int used = n_cls + 1 + n_reg;
  for (long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < N; row += warps) {
    __nv_bfloat16* d = dout + row * W;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const int c = lane + 32 * k;
      if (c < n_cls) {
        const __nv_bfloat16 g = dcls[row * n_cls + c];
        d[c] = g;
        acc[k] += __bfloat162float(g);
      }
    }
    if (lane == 0) d[n_cls] = __float2bfloat16(dcentre[row]);
    if (lane < n_reg) {
      float g = dbbox[row * n_reg + lane];
      if (lane < n_exp) {
        const float x = __bfloat162float(out[row * W + n_cls + 1 + lane]);
        const float e = expf(s * x);
        if (e >= lo) {
          ds += g * e * x;
          g = g * e * s;
        } else {
          g = 0.f;
        }
      }
      d[n_cls + 1 + lane] = __float2bfloat16(g);
    }
    for (int c = used + lane; c < W; c += 32) d[c] = __float2bfloat16(0.f);
  }
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const int c = lane + 32 * k;
    if (c < n_cls && acc[k] != 0.f) atomicAdd(&s_bias[c], acc[k]);
  }
#pragma unroll
  for (int d2 = 16; d2 > 0; d2 >>= 1) ds += __shfl_xor_sync(0xffffffffu, ds, d2);
  if (lane == 0 && ds != 0.f) atomicAdd(dscale, ds);
  __syncthreads();
  for (int c = threadIdx.x; c < n_cls; c += blockDim.x)
    if (s_bias[c] != 0.f) atomicAdd(&dbias[c], s_bias[c]);
}

static int head_split_grid(long long N) {
  long long g = esb_div_up(N, 8);                    // 8 warps (rows) per block
  const long long cap = 4LL * esb_sm_count();
  return (int)(g < cap ? g : cap);
}

extern "C" int esb_head_split_fwd(const void* out, const float* bias, const float* scale, long long N, int W, int n_cls,
                                  int n_reg, int n_exp, float lo, void* cls, float* centre, float* bbox, float* prune,
                                  void* stream) {
  ESB_CHECK_ARG(n_cls >= 1 && n_reg >= 0 && n_reg <= 32 && n_exp <= n_reg && n_cls + 1 + n_reg <= W,
                "esb_head_split_fwd: need n_cls >= 1, n_exp <= n_reg <= 32 and n_cls + 1 + n_reg <= W");
  if (N == 0) return ESB_OK;
  head_split_fwd_kernel<<<head_split_grid(N), 256, 0, (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)out, bias, scale, N, W, n_cls, n_reg, n_exp, lo, (__nv_bfloat16*)cls, centre, bbox, prune);
  ESB_CUDA_LAUNCH_CHECK("head_split_fwd_kernel");
  return ESB_OK;
}

// dbias (n_cls) and dscale (1) are ACCUMULATED into: the caller zeroes them.
extern "C" int esb_head_split_bwd(const void* out, const void* dcls, const float* dcentre, const float* dbbox,
                                  const float* scale, long long N, int W, int n_cls, int n_reg, int n_exp, float lo, void* dout,
                                  float* dbias, float* dscale, void* stream) {
  ESB_CHECK_ARG(n_cls >= 1 && n_cls <= 512 && n_reg >= 0 && n_reg <= 32 && n_exp <= n_reg && n_cls + 1 + n_reg <= W,
                "esb_head_split_bwd: need 1 <= n_cls <= 512, n_exp <= n_reg <= 32 and n_cls + 1 + n_reg <= W");
  if (N == 0) return ESB_OK;
  head_split_bwd_kernel<<<head_split_grid(N), 256, n_cls * sizeof(float), (cudaStream_t)stream>>>(
      (const __nv_bfloat16*)out, (const __nv_bfloat16*)dcls, dcentre, dbbox, scale, N, W, n_cls, n_reg, n_exp, lo,
      (__nv_bfloat16*)dout, dbias, dscale);
  ESB_CUDA_LAUNCH_CHECK("head_split_bwd_kernel");
  return ESB_OK;
}
