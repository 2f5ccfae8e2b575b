// esb200 — direct (SIMT, fp32-accumulate) NHWC 2D convolution, its two gradients and the stem's max pooling.
// Two jobs on the per-view image backbone (SURVEY §8 row a5; mmdet.ResNet called at
// embodiedscan/models/detectors/sparse_featfusion_single_stage.py:130-136):
//   * the fp32 PARITY arithmetic of every 2D convolution (the wgmma kernels of conv_tma.cu / conv2d_tc.cu take bf16
//     operands; fp32 FMA is what the 1e-3 bound of BASELINE.json is checked in), forward, dgrad and wgrad;
//   * the 7x7/2 stem on the 3-channel image in either dtype (Cin = 3 cannot feed a 16-byte TMA box) and the 3x3/2 max pool.
// Layouts: x (n,H,W,cin), w OHWI (cout,kh,kw,cin), y (n,Ho,Wo,cout); T = float or bf16, accumulation fp32.
// Roofline: fp32 FMA for the stem (147 x 16 FMA per output pixel), HBM for the pool.
#include "common.cuh"

namespace {

constexpr int CO_T = 16;     // output channels per thread
constexpr int R_CHUNK = 64;  // reduction elements staged per pass

// thread = one output pixel x CO_T output channels; the filter chunk is broadcast from shared memory
template <typename T>
__global__ void __launch_bounds__(128)
conv2d_direct_fwd_kernel(const T* __restrict__ x, const T* __restrict__ w, const float* __restrict__ bias,
                         const T* __restrict__ res, T* __restrict__ y, long long M, int H, int W, int cin, int Ho, int Wo,
                         int cout, int kh, int kw, int stride, int pad, int relu) {
  __shared__ float ws[R_CHUNK][CO_T];
  const long long m = (long long)blockIdx.x * 128 + threadIdx.x;
  const int co0 = blockIdx.y * CO_T;
  const int R = kh * kw * cin;
  const bool live = m < M;
  int iy0 = 0, ix0 = 0;
  const T* ximg = x;
  if (live) {
    const long long n = m / ((long long)Ho * Wo);
    const int rem = (int)(m - n * (long long)Ho * Wo);
    const int oy = rem / Wo, ox = rem - oy * Wo;
    iy0 = oy * stride - pad;
    ix0 = ox * stride - pad;
    ximg = x + n * (long long)H * W * cin;
  }
  float acc[CO_T];
#pragma unroll
  for (int c = 0; c < CO_T; ++c) acc[c] = 0.f;
  for (int r0 = 0; r0 < R; r0 += R_CHUNK) {
    __syncthreads();
    for (int i = threadIdx.x; i < R_CHUNK * CO_T; i += 128) {
      const int rr = i / CO_T, c = i - rr * CO_T;
      ws[rr][c] = (r0 + rr < R && co0 + c < cout) ? esb_to_float(w[(long long)(co0 + c) * R + r0 + rr]) : 0.f;
    }
    __syncthreads();
    if (live) {
      const int rend = min(R_CHUNK, R - r0);
      int tap = r0 / cin, ci = r0 - tap * cin;
      int ky = tap / kw, kx = tap - ky * kw;
      for (int rr = 0; rr < rend; ++rr) {
        const int iy = iy0 + ky, ix = ix0 + kx;
        if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
          const float xv = esb_to_float(ximg[((long long)iy * W + ix) * cin + ci]);
#pragma unroll
          for (int c = 0; c < CO_T; ++c) acc[c] = fmaf(xv, ws[rr][c], acc[c]);
        }
        if (++ci == cin) {
          ci = 0;
          if (++kx == kw) { kx = 0; ++ky; }
        }
      }
    }
  }
  if (!live) return;
#pragma unroll
  for (int c = 0; c < CO_T; ++c) {
    if (co0 + c < cout) {
      float v = acc[c];
      if (bias != nullptr) v += bias[co0 + c];
      if (res != nullptr) v += esb_to_float(res[m * cout + co0 + c]);
      if (relu) v = fmaxf(v, 0.f);
      y[m * cout + co0 + c] = esb_from_float<T>(v);
    }
  }
}

// thread = one INPUT pixel x CO_T input channels: dx[m, ci] = sum over taps, co of dy[src(m, tap), co] * w[co, tap, ci]
template <typename T>
__global__ void __launch_bounds__(128)
conv2d_direct_dgrad_kernel(const T* __restrict__ dy, const T* __restrict__ w, T* __restrict__ dx, long long M, int H, int W,
                           int cin, int Ho, int Wo, int cout, int kh, int kw, int stride, int pad) {
  __shared__ float ws[R_CHUNK][CO_T];            // [co within chunk][ci]
  const long long m = (long long)blockIdx.x * 128 + threadIdx.x;
  const int ci0 = blockIdx.y * CO_T;
  const bool live = m < M;
  int iy = 0, ix = 0;
  const T* dyimg = dy;
  if (live) {
    const long long n = m / ((long long)H * W);
    const int rem = (int)(m - n * (long long)H * W);
    iy = rem / W;
    ix = rem - iy * W;
    dyimg = dy + n * (long long)Ho * Wo * cout;
  }
  float acc[CO_T];
#pragma unroll
  for (int c = 0; c < CO_T; ++c) acc[c] = 0.f;
  const int R = kh * kw * cin;
  for (int tap = 0; tap < kh * kw; ++tap) {
    const int ky = tap / kw, kx = tap - ky * kw;
    const int ny = iy + pad - ky, nx = ix + pad - kx;
    const int oy = ny / stride, ox = nx / stride;
    const bool hit = live && ny >= 0 && nx >= 0 && oy * stride == ny && ox * stride == nx && oy < Ho && ox < Wo;
    for (int c0 = 0; c0 < cout; c0 += R_CHUNK) {
      __syncthreads();
      for (int i = threadIdx.x; i < R_CHUNK * CO_T; i += 128) {
        const int rr = i / CO_T, c = i - rr * CO_T;
        ws[rr][c] = (c0 + rr < cout && ci0 + c < cin) ? esb_to_float(w[(long long)(c0 + rr) * R + tap * cin + ci0 + c]) : 0.f;
      }
      __syncthreads();
      if (hit) {
        const T* src = dyimg + ((long long)oy * Wo + ox) * cout + c0;
        const int rend = min(R_CHUNK, cout - c0);
        for (int rr = 0; rr < rend; ++rr) {
          const float g = esb_to_float(src[rr]);
#pragma unroll
          for (int c = 0; c < CO_T; ++c) acc[c] = fmaf(g, ws[rr][c], acc[c]);
        }
      }
    }
  }
  if (!live) return;
#pragma unroll
  for (int c = 0; c < CO_T; ++c)
    if (ci0 + c < cin) dx[m * cin + ci0 + c] = esb_from_float<T>(acc[c]);
}

// dw[co, tap, ci] += sum over a slice of output pixels of dy[m, co] * x[src(m, tap), ci]; thread = (ci, co) of one tap,
// blockIdx.z = pixel slice (fp32 atomics across slices)
template <typename T>
__global__ void __launch_bounds__(256)
conv2d_direct_wgrad_kernel(const T* __restrict__ x, const T* __restrict__ dy, float* __restrict__ dw, long long M, int H, int W,
                           int cin, int Ho, int Wo, int cout, int kh, int kw, int stride, int pad, int slice) {
  const int tap = blockIdx.y;
  const int ky = tap / kw, kx = tap - ky * kw;
  const int pairs = cin * cout;
  const int p = blockIdx.x * 256 + threadIdx.x;
  if (p >= pairs) return;
  const int co = p / cin, ci = p - co * cin;      // consecutive threads: consecutive ci (contiguous x reads)
  const long long m_beg = (long long)blockIdx.z * slice;
  const long long m_end = m_beg + slice < M ? m_beg + slice : M;
  const long long HoWo = (long long)Ho * Wo;
  float acc = 0.f;
  for (long long m = m_beg; m < m_end; ++m) {
    const long long n = m / HoWo;
    const int rem = (int)(m - n * HoWo);
    const int oy = rem / Wo, ox = rem - oy * Wo;
    const int iy = oy * stride - pad + ky, ix = ox * stride - pad + kx;
    if (iy < 0 || iy >= H || ix < 0 || ix >= W) continue;
    acc = fmaf(esb_to_float(dy[m * cout + co]), esb_to_float(x[((n * H + iy) * (long long)W + ix) * cin + ci]), acc);
  }
  atomicAdd(dw + ((long long)co * kh * kw + tap) * cin + ci, acc);
}

// 3x3 / stride 2 / pad 1 style max pooling on NHWC, 8 channels (one 16-byte piece for bf16) per thread
template <typename T, int VEC>
__global__ void maxpool2d_nhwc_kernel(const T* __restrict__ x, T* __restrict__ y, long long total, int H, int W, int C, int Ho,
                                      int Wo, int k, int stride, int pad) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int cv = C / VEC;
  const int c = (int)(i % cv) * VEC;
  long long t = i / cv;
  const int ox = (int)(t % Wo); t /= Wo;
  const int oy = (int)(t % Ho);
  const long long n = t / Ho;
  float best[VEC];
#pragma unroll
  for (int e = 0; e < VEC; ++e) best[e] = -INFINITY;
  for (int dy = 0; dy < k; ++dy) {
    const int iy = oy * stride - pad + dy;
    if (iy < 0 || iy >= H) continue;
    for (int dx = 0; dx < k; ++dx) {
      const int ix = ox * stride - pad + dx;
      if (ix < 0 || ix >= W) continue;
      const T* src = x + ((n * H + iy) * (long long)W + ix) * C + c;
      if (VEC == 8 && sizeof(T) == 2) {
        const uint4 v = *reinterpret_cast<const uint4*>(src);
        const __nv_bfloat162* hp = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __bfloat1622float2(hp[e]);
          best[2 * e] = fmaxf(best[2 * e], f.x);
          best[2 * e + 1] = fmaxf(best[2 * e + 1], f.y);
        }
      } else {
#pragma unroll
        for (int e = 0; e < VEC; ++e) best[e] = fmaxf(best[e], esb_to_float(src[e]));
      }
    }
  }
  T* dst = y + ((n * Ho + oy) * (long long)Wo + ox) * C + c;
#pragma unroll
  for (int e = 0; e < VEC; ++e) dst[e] = esb_from_float<T>(best[e]);
}

}  // namespace

#define ESB_DTYPE_SWITCH(dtype, ...)                                  \
  if ((dtype) == ESB_F32) { using T = float; __VA_ARGS__ }            \
  else if ((dtype) == ESB_BF16) { using T = __nv_bfloat16; __VA_ARGS__ } \
  else { esb_set_error("unsupported dtype code %d", (int)(dtype)); return ESB_EINVAL; }

extern "C" int esb_conv2d_direct_fwd(const void* x, const void* w_ohwi, const float* bias, const void* residual, void* y,
                                     int n_img, int H, int W, int cin, int cout, int kh, int kw, int stride, int pad, int relu,
                                     int dtype, void* stream) {
  ESB_CHECK_ARG(cin > 0 && cout > 0 && kh >= 1 && kw >= 1 && stride >= 1 && pad >= 0, "esb_conv2d_direct_fwd: bad geometry");
  const int Ho = (H + 2 * pad - kh) / stride + 1, Wo = (W + 2 * pad - kw) / stride + 1;
  ESB_CHECK_ARG(Ho > 0 && Wo > 0, "esb_conv2d_direct_fwd: empty output");
  const long long M = (long long)n_img * Ho * Wo;
  if (M == 0) return ESB_OK;
  dim3 grid(esb_div_up(M, 128), esb_div_up(cout, CO_T));
  ESB_DTYPE_SWITCH(dtype, conv2d_direct_fwd_kernel<T><<<grid, 128, 0, (cudaStream_t)stream>>>(
      (const T*)x, (const T*)w_ohwi, bias, (const T*)residual, (T*)y, M, H, W, cin, Ho, Wo, cout, kh, kw, stride, pad, relu);)
  ESB_CUDA_LAUNCH_CHECK("conv2d_direct_fwd_kernel");
  return ESB_OK;
}

extern "C" int esb_conv2d_direct_dgrad(const void* dy, const void* w_ohwi, void* dx, int n_img, int H, int W, int cin, int cout,
                                       int kh, int kw, int stride, int pad, int dtype, void* stream) {
  ESB_CHECK_ARG(cin > 0 && cout > 0 && kh >= 1 && kw >= 1 && stride >= 1 && pad >= 0, "esb_conv2d_direct_dgrad: bad geometry");
  const int Ho = (H + 2 * pad - kh) / stride + 1, Wo = (W + 2 * pad - kw) / stride + 1;
  ESB_CHECK_ARG(Ho > 0 && Wo > 0, "esb_conv2d_direct_dgrad: empty output");
  const long long M = (long long)n_img * H * W;
  if (M == 0) return ESB_OK;
  dim3 grid(esb_div_up(M, 128), esb_div_up(cin, CO_T));
  ESB_DTYPE_SWITCH(dtype, conv2d_direct_dgrad_kernel<T><<<grid, 128, 0, (cudaStream_t)stream>>>(
      (const T*)dy, (const T*)w_ohwi, (T*)dx, M, H, W, cin, Ho, Wo, cout, kh, kw, stride, pad);)
  ESB_CUDA_LAUNCH_CHECK("conv2d_direct_dgrad_kernel");
  return ESB_OK;
}

// dw_ohwi (cout,kh,kw,cin) fp32, ZEROED BY THE CALLER (pixel slices accumulate with fp32 atomics)
extern "C" int esb_conv2d_direct_wgrad(const void* x, const void* dy, float* dw_ohwi, int n_img, int H, int W, int cin, int cout,
                                       int kh, int kw, int stride, int pad, int dtype, void* stream) {
  ESB_CHECK_ARG(cin > 0 && cout > 0 && kh >= 1 && kw >= 1 && stride >= 1 && pad >= 0, "esb_conv2d_direct_wgrad: bad geometry");
  const int Ho = (H + 2 * pad - kh) / stride + 1, Wo = (W + 2 * pad - kw) / stride + 1;
  ESB_CHECK_ARG(Ho > 0 && Wo > 0, "esb_conv2d_direct_wgrad: empty output");
  const long long M = (long long)n_img * Ho * Wo;
  if (M == 0) return ESB_OK;
  const int pair_blocks = esb_div_up((long long)cin * cout, 256);
  long long slices = (4LL * esb_sm_count() * 8) / ((long long)pair_blocks * kh * kw) + 1;   // enough CTAs to fill the device
  if (slices > 1024) slices = 1024;
  int slice = (int)((M + slices - 1) / slices);
  if (slice < 64) slice = 64;
  dim3 grid(pair_blocks, kh * kw, esb_div_up(M, slice));
  ESB_DTYPE_SWITCH(dtype, conv2d_direct_wgrad_kernel<T><<<grid, 256, 0, (cudaStream_t)stream>>>(
      (const T*)x, (const T*)dy, dw_ohwi, M, H, W, cin, Ho, Wo, cout, kh, kw, stride, pad, slice);)
  ESB_CUDA_LAUNCH_CHECK("conv2d_direct_wgrad_kernel");
  return ESB_OK;
}

extern "C" int esb_maxpool2d_nhwc(const void* x, void* y, int n_img, int H, int W, int C, int k, int stride, int pad, int dtype,
                                  void* stream) {
  ESB_CHECK_ARG(C > 0 && k >= 1 && stride >= 1 && pad >= 0 && pad < k, "esb_maxpool2d_nhwc: bad geometry");
  const int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
  ESB_CHECK_ARG(Ho > 0 && Wo > 0, "esb_maxpool2d_nhwc: empty output");
  if (n_img == 0) return ESB_OK;
  if (dtype == ESB_BF16 && C % 8 == 0) {
    const long long total = (long long)n_img * Ho * Wo * (C / 8);
    maxpool2d_nhwc_kernel<__nv_bfloat16, 8><<<esb_div_up(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16*)x, (__nv_bfloat16*)y, total, H, W, C, Ho, Wo, k, stride, pad);
  } else {
    const long long total = (long long)n_img * Ho * Wo * C;
    ESB_DTYPE_SWITCH(dtype, maxpool2d_nhwc_kernel<T, 1><<<esb_div_up(total, 256), 256, 0, (cudaStream_t)stream>>>(
        (const T*)x, (T*)y, total, H, W, C, Ho, Wo, k, stride, pad);)
  }
  ESB_CUDA_LAUNCH_CHECK("maxpool2d_nhwc_kernel");
  return ESB_OK;
}
