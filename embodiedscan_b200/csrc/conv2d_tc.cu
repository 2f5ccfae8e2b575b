// esb200 — dense 2D convolution on the Hopper tensor cores (wgmma), bf16 in / fp32 accumulate:
// the per-view image backbone (SURVEY §8 row a5: mmdet.ResNet(depth=50, base_channels=16) called at
// embodiedscan/models/detectors/sparse_featfusion_single_stage.py:130-136) as an implicit GEMM with the frozen
// BatchNorm folded into the weights and bias + residual + ReLU fused into the epilogue.
//
// STATUS: superseded on the measured path by conv_tma.cu (TMA-fed); kept as its cp.async baseline and as the dgrad for
// strides above 2.
//
// GEMM view: M = n_img*Ho*Wo output pixels, N = Cout, reduction R = kh*kw*Cin ordered (ky, kx, ci) — i.e. the weight
// in OHWI (= PyTorch channels_last) layout IS the K-major B operand, row n = output channel, R contiguous, zero padded
// to R_pad (multiple of 64) by the host. A is never materialised (no im2col buffer): a CTA owns 128 output pixels x
// N_TILE channels and gathers, per 64-wide reduction chunk, eight 16-byte pieces per pixel straight from the NHWC
// activations with cp.async (zero-fill outside the image / beyond R), into the 128B-swizzled K-major layout the
// sparse kernel uses. Thin layers (Cin = 16, 32) pack 4 or 2 filter taps into one 64-wide chunk, so a 3x3x16 filter
// is 3 chunks instead of 9. Same thread roles as spconv_tc.cu: threads 0-255 = two consumer warpgroups issuing wgmma
// (64 pixels each, accumulator in registers, written to shared memory at the end of the tile), threads 256-383 gather
// then run the epilogue (thread = pixel); full/empty mbarrier ring.
//
// The input gradient is the same kernel in transposed-gather mode; the weight gradient is a second kernel below with
// the pixels as the reduction dimension (split-K).
//
// Roofline: HBM. Algorithmic bytes per image = (H*W*Cin + Ho*Wo*Cout [+ residual]) * 2 + R_pad*Cout*2.
#include "tc_common.cuh"

using namespace esb_tc;

namespace {

template <int N_TILE, int STAGES>
__global__ void __launch_bounds__(384, 1)
conv2d_tc_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ wt,
                     const float* __restrict__ bias, const __nv_bfloat16* __restrict__ res,
                     __nv_bfloat16* __restrict__ y, long long M, int H, int W, int cin, int Ho, int Wo, int cout, int kh,
                     int kw, int stride, int pad, int r_pad, int relu, int transposed) {
  constexpr int B_STAGE_BYTES = N_TILE * 128;
  constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  constexpr int LAG = STAGES - 2;
  constexpr int NCONS = 256;
  constexpr int PITCH = N_TILE + 4;                // floats per accumulator-image row
  static_assert(TC_M * PITCH * 4 <= STAGES * STAGE_BYTES, "the accumulator image reuses the stage buffers");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = (uint64_t*)(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* accum_bar = empty_bar + STAGES;
  float* img = reinterpret_cast<float*>(smem);

  const long long tile = blockIdx.x;
  const int n0 = blockIdx.y * N_TILE;
  const int total = r_pad / TC_BK;                 // >= 1

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 128);
      mbar_init(&empty_bar[s], NCONS / 32);
    }
    mbar_init(accum_bar, NCONS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (threadIdx.x >= NCONS) {
    // ---------------- producers: 8 lanes fetch the 8 x 16 B pieces of one pixel's chunk (see spconv_tc.cu) ----------
    const int t = threadIdx.x - NCONS;
    const int sub = t & 7, rgrp = t >> 3;
    const uint32_t sw = (uint32_t)(rgrp & 7);
    const uint32_t a_thread_off = (uint32_t)((rgrp >> 3) * 1024 + (rgrp & 7) * 128) + ((sub ^ sw) << 4);
    const int taps = kh * kw;
    int iy0[8], ix0[8];
    long long img_off[8];                          // element offset of the pixel's image in x, or -1 beyond M
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const long long m = tile * TC_M + rgrp + 16 * i;
      if (m < M) {
        const long long n = m / ((long long)Ho * Wo);
        const int rem = (int)(m - n * (long long)Ho * Wo);
        const int oy = rem / Wo, ox = rem - oy * Wo;
        // forward: source pixel = row pixel * stride - pad + tap.  transposed (dgrad): rows are pixels of the conv's
        // INPUT grid and the source is dy: source pixel = (row pixel + pad - tap) / stride when that division is exact.
        iy0[i] = transposed ? oy + pad : oy * stride - pad;
        ix0[i] = transposed ? ox + pad : ox * stride - pad;
        img_off[i] = n * (long long)H * W * cin;
      } else {
        iy0[i] = ix0[i] = 0;
        img_off[i] = -1;
      }
    }
    for (int it = 0; it < total; ++it) {
      const int s = it % STAGES;
      if (it >= STAGES) mbar_wait(&empty_bar[s], ((it / STAGES) - 1) & 1);
      // this thread's 8 reduction elements of the chunk all belong to one filter tap (cin % 8 == 0)
      const int r0 = it * TC_BK + sub * 8;
      const int tap = r0 / cin, ch = r0 - tap * cin;
      const int ky = tap / kw, kx = tap - ky * kw;
      const bool tap_ok = tap < taps;
      const uint32_t a_base = smem_u32(smem + s * STAGE_BYTES) + a_thread_off;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        int iy, ix;
        bool ok = tap_ok && img_off[i] >= 0;
        if (!transposed) {
          iy = iy0[i] + ky;
          ix = ix0[i] + kx;
        } else {
          const int ny = iy0[i] - ky, nx = ix0[i] - kx;
          iy = ny / stride;
          ix = nx / stride;
          ok = ok && ny >= 0 && nx >= 0 && iy * stride == ny && ix * stride == nx;
        }
        ok = ok && iy >= 0 && iy < H && ix >= 0 && ix < W;
        const __nv_bfloat16* src = ok ? x + img_off[i] + ((long long)iy * W + ix) * cin + ch : x;
        cp_async16_ca(a_base + i * 2048, src, ok ? 16 : 0);
      }
      const uint32_t b_base = smem_u32(smem + s * STAGE_BYTES + A_STAGE_BYTES);
#pragma unroll
      for (int q = 0; q < N_TILE / 16; ++q) {
        const int idx = q * 128 + t;
        const int n = idx >> 3, j = idx & 7;
        const bool ok = n0 + n < cout;
        cp_async16_cg(b_base + (n >> 3) * 1024 + (n & 7) * 128 + ((j ^ (n & 7)) << 4),
                      ok ? wt + (long long)(n0 + n) * r_pad + it * TC_BK + j * 8 : wt, ok ? 16 : 0);
      }
      cp_async_commit();
      if (it >= LAG) {
        cp_async_wait<LAG>();
        fence_proxy_async();
        mbar_arrive(&full_bar[(it - LAG) % STAGES]);
      }
    }
    cp_async_wait<0>();
    fence_proxy_async();
    for (int d = (total > LAG ? total - LAG : 0); d < total; ++d) mbar_arrive(&full_bar[d % STAGES]);

    // ---------------- epilogue: + bias, + residual, ReLU, bf16 ----------------
    const long long row = tile * TC_M + t;                  // accumulator-image row = pixel of the tile
    mbar_wait(accum_bar, 0);
#pragma unroll 1
    for (int c0 = 0; c0 < N_TILE; c0 += 32) {
      uint32_t v[32];
      img_ld<32>(img, PITCH, t, c0, v);
      if (row < M) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int c = n0 + c0 + 8 * q;
          if (c < cout) {                                   // cout % 8 == 0: a group of 8 is all in or all out
            float f[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) f[e] = __uint_as_float(v[8 * q + e]);
            if (bias != nullptr) {
              const float4 b0 = *reinterpret_cast<const float4*>(bias + c);
              const float4 b1 = *reinterpret_cast<const float4*>(bias + c + 4);
              f[0] += b0.x; f[1] += b0.y; f[2] += b0.z; f[3] += b0.w;
              f[4] += b1.x; f[5] += b1.y; f[6] += b1.z; f[7] += b1.w;
            }
            if (res != nullptr) {
              const uint4 r = *reinterpret_cast<const uint4*>(res + row * cout + c);
              const __nv_bfloat162* rp = reinterpret_cast<const __nv_bfloat162*>(&r);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float2 rf = __bfloat1622float2(rp[e]);
                f[2 * e] += rf.x;
                f[2 * e + 1] += rf.y;
              }
            }
            if (relu) {
#pragma unroll
              for (int e = 0; e < 8; ++e) f[e] = fmaxf(f[e], 0.f);
            }
            uint4 o;
            o.x = pack_bf16(__float_as_uint(f[0]), __float_as_uint(f[1]));
            o.y = pack_bf16(__float_as_uint(f[2]), __float_as_uint(f[3]));
            o.z = pack_bf16(__float_as_uint(f[4]), __float_as_uint(f[5]));
            o.w = pack_bf16(__float_as_uint(f[6]), __float_as_uint(f[7]));
            *reinterpret_cast<uint4*>(y + row * cout + c) = o;
          }
        }
      }
    }
  } else {
    // ---------------- consumers: warpgroup wg owns pixels 64 wg .. 64 wg + 63 of the tile ----------------
    const int wg = threadIdx.x >> 7;
    float acc[N_TILE / 2];
    for (int it = 0; it < total; ++it) {
      const int s = it % STAGES;
      mbar_wait(&full_bar[s], (it / STAGES) & 1);
      const uint32_t a_addr = smem_u32(smem + s * STAGE_BYTES) + wg * 8192;
      const uint32_t b_addr = smem_u32(smem + s * STAGE_BYTES) + A_STAGE_BYTES;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < TC_BK / 16; ++kk)
        wgmma_bf16<N_TILE, 0, 0>(acc, make_desc(a_addr + kk * 32, 16, 1024), make_desc(b_addr + kk * 32, 16, 1024), it > 0 || kk > 0);
      wgmma_commit();
      wgmma_wait<1>();
      if (it > 0 && (threadIdx.x & 31) == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
    }
    wgmma_wait<0>();
    acc_fence<N_TILE / 2>(acc);
    asm volatile("bar.sync 2, %0;" ::"n"(NCONS) : "memory");
    acc_store<N_TILE>(acc, img, PITCH, wg * 64, threadIdx.x & 127);
    mbar_arrive(accum_bar);
  }
}

template <int N_TILE, int STAGES>
int launch_conv2d(const void* x, const void* wt, const float* bias, const void* res, void* y, long long M, int H, int W,
                  int cin, int Ho, int Wo, int cout, int kh, int kw, int stride, int pad, int r_pad, int relu,
                  int transposed, cudaStream_t stream) {
  size_t smem = (size_t)STAGES * (A_STAGE_BYTES + N_TILE * 128) + 1024 + 256;
  auto kern = conv2d_tc_fwd_kernel<N_TILE, STAGES>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { esb_set_error("conv2d_tc_fwd: smem attr: %s", cudaGetErrorString(e)); return ESB_ECUDA; }
  dim3 grid(esb_div_up(M, TC_M), esb_div_up(cout, N_TILE));
  kern<<<grid, 384, smem, stream>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)wt, bias, (const __nv_bfloat16*)res,
                                    (__nv_bfloat16*)y, M, H, W, cin, Ho, Wo, cout, kh, kw, stride, pad, r_pad, relu, transposed);
  return ESB_OK;
}


// ------------------------------------------------------------------------------------------------------------
// wgrad: dW^T[r, co] += sum over output pixels m of A[m, r] * dy[m, co], r = (ky, kx, ci) — the same implicit A as the
// forward pass, now MN-major on both sides with the PIXELS as the reduction dimension (64 per stage), exactly the
// operand arrangement of spconv_tc_wgrad_kernel with the pair list replaced by index arithmetic.
// CTA = (chunk of pixels: split-K) x (128-wide slice of r) x (N_TILE slice of Cout); fp32 atomics into dW^T.
// ------------------------------------------------------------------------------------------------------------
template <int N_TILE, int STAGES>
__global__ void __launch_bounds__(384, 1)
conv2d_tc_wgrad_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy, float* __restrict__ dw,
                       long long M, int H, int W, int cin, int Ho, int Wo, int cout, int kh, int kw, int stride, int pad,
                       int chunk_pixels) {
  constexpr int A_BYTES = 64 * 256;              // 64 pixels x 128 reduction elements (2 M-atoms of 64)
  constexpr int B_BYTES = 64 * N_TILE * 2;
  constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  constexpr int LAG = STAGES - 2;
  constexpr int NCONS = 256;
  constexpr int PITCH = N_TILE + 4;
  static_assert(128 * PITCH * 4 <= STAGES * STAGE_BYTES, "the accumulator image reuses the stage buffers");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = (uint64_t*)(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* accum_bar = empty_bar + STAGES;

  const long long s_beg = (long long)blockIdx.x * chunk_pixels;
  const long long s_end = s_beg + chunk_pixels < M ? s_beg + chunk_pixels : M;
  if (s_beg >= M) return;                          // uniform for the whole CTA
  const int total = (int)((s_end - s_beg + 63) / 64);
  const int R = kh * kw * cin;
  const int r0 = blockIdx.y * 128, co0 = blockIdx.z * N_TILE;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 128);
      mbar_init(&empty_bar[s], NCONS / 32);
    }
    mbar_init(accum_bar, NCONS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (threadIdx.x >= NCONS) {
    const int t = threadIdx.x - NCONS;
    const int warp = t >> 5;
    // thread t moves 16-byte piece (t & 15) of pixel rows kk = (t >> 4) + 8 q, q = 0..7; its 8 reduction elements
    // r = r0 + 8 (t & 15) .. +7 lie in ONE filter tap (cin % 8 == 0), fixed for the whole kernel
    const int mc = t & 15, kk0 = t >> 4;
    const int r = r0 + mc * 8;
    const int tap = r / cin, ch = r - tap * cin;
    const int ky = tap / kw, kx = tap - ky * kw;
    const bool r_ok = r < R;
    const long long HoWo = (long long)Ho * Wo;
    for (int it = 0; it < total; ++it) {
      const int s = it % STAGES;
      if (it >= STAGES) mbar_wait(&empty_bar[s], ((it / STAGES) - 1) & 1);
      const uint32_t a_base = smem_u32(smem + s * STAGE_BYTES);
      const uint32_t b_base = a_base + A_BYTES;
      const long long m0 = s_beg + (long long)it * 64;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int kk = kk0 + 8 * q;
        const long long m = m0 + kk;
        bool ok = r_ok && m < s_end;
        const __nv_bfloat16* src = x;
        if (ok) {
          const long long n = m / HoWo;
          const int rem = (int)(m - n * HoWo);
          const int oy = rem / Wo, ox = rem - oy * Wo;
          const int iy = oy * stride - pad + ky, ix = ox * stride - pad + kx;
          ok = iy >= 0 && iy < H && ix >= 0 && ix < W;
          if (ok) src = x + ((n * H + iy) * (long long)W + ix) * cin + ch;
        }
        // canonical MN-major SW128: atom(mi, kj) at mi*8192 + kj*1024, row kk%8, 16 B chunk index ^ row
        const uint32_t dst = a_base + (mc >> 3) * 8192 + (kk >> 3) * 1024 + (kk & 7) * 128 + (((mc & 7) ^ (kk & 7)) << 4);
        cp_async16_cg(dst, src, ok ? 16 : 0);
      }
#pragma unroll
      for (int q = 0; q < N_TILE / 16; ++q) {
        const int idx = q * 128 + t;
        const int kk = idx / (N_TILE / 8), nc = idx % (N_TILE / 8);
        const long long m = m0 + kk;
        const bool ok = m < s_end && co0 + nc * 8 < cout;
        const uint32_t dst = b_base + (nc >> 3) * 8192 + (kk >> 3) * 1024 + (kk & 7) * 128 + (((nc & 7) ^ (kk & 7)) << 4);
        cp_async16_cg(dst, ok ? dy + m * cout + co0 + nc * 8 : dy, ok ? 16 : 0);
      }
      cp_async_commit();
      if (it >= LAG) {
        cp_async_wait<LAG>();
        fence_proxy_async();
        mbar_arrive(&full_bar[(it - LAG) % STAGES]);
      }
    }
    cp_async_wait<0>();
    fence_proxy_async();
    for (int d = (total > LAG ? total - LAG : 0); d < total; ++d) mbar_arrive(&full_bar[d % STAGES]);

    // epilogue: image row = reduction element r (within the 128 slice), column = co; a warp stores contiguous runs of one
    // row of this pixel chunk's partial of dW^T (the host adds the chunks in order)
    mbar_wait(accum_bar, 0);
    const float* stg = reinterpret_cast<const float*>(smem);
    const int lane = t & 31;
    for (int i = 0; i < 32; ++i) {
      const int rl = warp * 32 + i;
      const int rr = r0 + rl;
      if (rr >= R) break;
      float* dwrow = dw + ((long long)blockIdx.x * R + rr) * cout + co0;
#pragma unroll
      for (int c = lane * 4; c < N_TILE; c += 128)
        if (co0 + c < cout)                              // cout % 8 == 0: a float4 is all in or all out
          *reinterpret_cast<float4*>(dwrow + c) = *reinterpret_cast<const float4*>(stg + rl * PITCH + c);
    }
  } else {
    // consumers: warpgroup wg owns reduction rows r0 + 64 wg .. (the second MN atom of the A tile)
    const int wg = threadIdx.x >> 7;
    float acc[N_TILE / 2];
    for (int it = 0; it < total; ++it) {
      const int s = it % STAGES;
      mbar_wait(&full_bar[s], (it / STAGES) & 1);
      const uint32_t a_addr = smem_u32(smem + s * STAGE_BYTES) + wg * 8192;
      const uint32_t b_addr = smem_u32(smem + s * STAGE_BYTES) + A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)              // 16 pixels per MMA = two 8-row K groups = 2048 B
        wgmma_bf16<N_TILE, 1, 1>(acc, make_desc(a_addr + kk * 2048, 8192, 1024), make_desc(b_addr + kk * 2048, 8192, 1024), it > 0 || kk > 0);
      wgmma_commit();
      wgmma_wait<1>();
      if (it > 0 && (threadIdx.x & 31) == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
    }
    wgmma_wait<0>();
    acc_fence<N_TILE / 2>(acc);
    asm volatile("bar.sync 2, %0;" ::"n"(NCONS) : "memory");
    acc_store<N_TILE>(acc, reinterpret_cast<float*>(smem), PITCH, wg * 64, threadIdx.x & 127);
    mbar_arrive(accum_bar);
  }
}

template <int N_TILE, int STAGES>
int launch_conv2d_wgrad(const void* x, const void* dy, float* dw, long long M, int H, int W, int cin, int Ho, int Wo,
                        int cout, int kh, int kw, int stride, int pad, int chunk_pixels, cudaStream_t stream) {
  size_t smem = (size_t)STAGES * (64 * 256 + 64 * N_TILE * 2) + 1024 + 256;
  auto kern = conv2d_tc_wgrad_kernel<N_TILE, STAGES>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { esb_set_error("conv2d_tc_wgrad: smem attr: %s", cudaGetErrorString(e)); return ESB_ECUDA; }
  dim3 grid(esb_div_up(M, chunk_pixels), esb_div_up(kh * kw * cin, 128), esb_div_up(cout, N_TILE));
  const long long width = (long long)kh * kw * cin * cout;     // every pixel chunk writes a whole partial of dW^T
  float* part = nullptr;
  ESB_CUDA_CALL(esb_scratch_alloc((void**)&part, sizeof(float) * grid.x * width, stream));
  kern<<<grid, 384, smem, stream>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)dy, part, M, H, W, cin, Ho, Wo, cout, kh,
                                    kw, stride, pad, chunk_pixels);
  int rc = esb_sum_partial_rows(part, (int)grid.x, width, dw, 1, stream);
  ESB_CUDA_CALL(esb_scratch_free(part, stream));
  return rc;
}

}  // namespace

static int conv2d_dispatch(const void* x, const void* w, const float* bias, const void* residual, void* y, long long M,
                           int Hs, int Ws, int cs, int Hr, int Wr, int cr, int kh, int kw, int stride, int pad, int r_pad,
                           int relu, int transposed, cudaStream_t stream) {
  const long long row_tiles = (M + TC_M - 1) / TC_M;
  int rc;
#define ESB_C2D(NT, ST) \
  launch_conv2d<NT, ST>(x, w, bias, residual, y, M, Hs, Ws, cs, Hr, Wr, cr, kh, kw, stride, pad, r_pad, relu, transposed, stream)
  if (cr > 128 && row_tiles * ((cr + 255) / 256) >= esb_sm_count())
    rc = ESB_C2D(256, 4);
  else if (cr > 64)
    rc = ESB_C2D(128, 4);
  else if (cr > 32)
    rc = ESB_C2D(64, 4);
  else
    rc = ESB_C2D(32, 4);
#undef ESB_C2D
  if (rc != ESB_OK) return rc;
  ESB_CUDA_LAUNCH_CHECK("conv2d_tc_fwd_kernel");
  return ESB_OK;
}

extern "C" int esb_conv2d_tc_fwd(const void* x, const void* w_ohwi, const float* bias, const void* residual, void* y,
                                 int n_img, int H, int W, int cin, int cout, int kh, int kw, int stride, int pad,
                                 int r_pad, int relu, void* stream_) {
  ESB_CHECK_ARG(cin > 0 && cin % 8 == 0, "esb_conv2d_tc_fwd: Cin must be a positive multiple of 8 (16-byte pieces)");
  ESB_CHECK_ARG(cout > 0 && cout % 8 == 0, "esb_conv2d_tc_fwd: Cout must be a positive multiple of 8");
  ESB_CHECK_ARG(kh >= 1 && kw >= 1 && stride >= 1 && pad >= 0, "esb_conv2d_tc_fwd: bad filter geometry");
  ESB_CHECK_ARG(r_pad % 64 == 0 && r_pad >= kh * kw * cin, "esb_conv2d_tc_fwd: r_pad must be kh*kw*Cin rounded up to 64");
  const int Ho = (H + 2 * pad - kh) / stride + 1, Wo = (W + 2 * pad - kw) / stride + 1;
  ESB_CHECK_ARG(Ho > 0 && Wo > 0, "esb_conv2d_tc_fwd: empty output");
  const long long M = (long long)n_img * Ho * Wo;
  if (M == 0) return ESB_OK;
  return conv2d_dispatch(x, w_ohwi, bias, residual, y, M, H, W, cin, Ho, Wo, cout, kh, kw, stride, pad, r_pad, relu, 0,
                         (cudaStream_t)stream_);
}

// Input gradient of the same convolution with the SAME kernel in transposed-gather mode: rows are the pixels of the
// conv's input grid, the source is dy (n_img,Ho,Wo,cout), and w_ihwo (cin, r_pad) holds the filter as
// (ci | ky, kx, co), rows zero padded from kh*kw*cout to r_pad. dx (n_img,H,W,cin) is written once (no atomics).
extern "C" int esb_conv2d_tc_dgrad(const void* dy, const void* w_ihwo, void* dx, int n_img, int H, int W, int cin,
                                   int cout, int kh, int kw, int stride, int pad, int r_pad, void* stream_) {
  ESB_CHECK_ARG(cin > 0 && cin % 8 == 0 && cout > 0 && cout % 8 == 0, "esb_conv2d_tc_dgrad: channels must be multiples of 8");
  ESB_CHECK_ARG(kh >= 1 && kw >= 1 && stride >= 1 && pad >= 0, "esb_conv2d_tc_dgrad: bad filter geometry");
  ESB_CHECK_ARG(r_pad % 64 == 0 && r_pad >= kh * kw * cout, "esb_conv2d_tc_dgrad: r_pad must be kh*kw*Cout rounded up to 64");
  const int Ho = (H + 2 * pad - kh) / stride + 1, Wo = (W + 2 * pad - kw) / stride + 1;
  ESB_CHECK_ARG(Ho > 0 && Wo > 0, "esb_conv2d_tc_dgrad: empty output");
  const long long M = (long long)n_img * H * W;
  if (M == 0) return ESB_OK;
  return conv2d_dispatch(dy, w_ihwo, nullptr, nullptr, dx, M, Ho, Wo, cout, H, W, cin, kh, kw, stride, pad, r_pad, 0, 1,
                         (cudaStream_t)stream_);
}

// Weight gradient: dw_t (kh*kw*cin, cout) fp32 += the gradient (zeroed by the caller; split-K partials are added in order),
// row r = (ky, kx, ci) like the forward's reduction index: dW[co, ci, ky, kx] = dw_t[(ky*kw + kx)*cin + ci, co].
extern "C" int esb_conv2d_tc_wgrad(const void* x, const void* dy, float* dw_t, int n_img, int H, int W, int cin, int cout,
                                   int kh, int kw, int stride, int pad, void* stream_) {
  ESB_CHECK_ARG(cin > 0 && cin % 8 == 0 && cout > 0 && cout % 8 == 0, "esb_conv2d_tc_wgrad: channels must be multiples of 8");
  ESB_CHECK_ARG(kh >= 1 && kw >= 1 && stride >= 1 && pad >= 0, "esb_conv2d_tc_wgrad: bad filter geometry");
  const int Ho = (H + 2 * pad - kh) / stride + 1, Wo = (W + 2 * pad - kw) / stride + 1;
  ESB_CHECK_ARG(Ho > 0 && Wo > 0, "esb_conv2d_tc_wgrad: empty output");
  const long long M = (long long)n_img * Ho * Wo;
  if (M == 0) return ESB_OK;
  const int n_tile = cout > 64 ? 128 : 64;
  // ~4 waves of 2 CTAs per SM over the (r-slice, channel-tile) grid; chunks of whole 64-pixel stages
  const long long tiles = (long long)esb_div_up(kh * kw * cin, 128) * esb_div_up(cout, n_tile);
  const long long target_chunks = (4LL * 2 * esb_sm_count() + tiles - 1) / tiles;
  long long cp = (M + target_chunks - 1) / target_chunks;
  cp = (cp + 63) / 64 * 64;
  if (cp < 512) cp = 512;
  if (cp > 65536) cp = 65536;
  int rc = n_tile == 128
               ? launch_conv2d_wgrad<128, 3>(x, dy, dw_t, M, H, W, cin, Ho, Wo, cout, kh, kw, stride, pad, (int)cp, (cudaStream_t)stream_)
               : launch_conv2d_wgrad<64, 4>(x, dy, dw_t, M, H, W, cin, Ho, Wo, cout, kh, kw, stride, pad, (int)cp, (cudaStream_t)stream_);
  if (rc != ESB_OK) return rc;
  ESB_CUDA_LAUNCH_CHECK("conv2d_tc_wgrad_kernel");
  return ESB_OK;
}
