// esb200 — colour-frame resize of the configs' MultiViewPipeline step `Resize(scale=(w, h), keep_ratio=False)`
// (configs/detection/mv-det3d_8xb4_embodiedscan-3d-284class-9dof.py:143,171 -> mmcv imresize -> cv2.resize with
// INTER_LINEAR), for all views of a scan in one launch: (V,H,W,3) uint8 HWC as decoded -> (V,3,h,w) uint8 CHW as
// Pack3DDetInputs stacks it (the layout esb_img_normalize reads). Channels are not reordered.
//
// Bit for bit cv2's 8-bit fixed point (imgproc/src/resize.cpp, restated in oracle/resize_ref.py):
//  - per axis, output index d: f = float((d + 0.5) * scale - 0.5) with scale = 1 / (out / in) in double,
//    s = floor(f), f -= s, coefficients rint((1 - f) * 2048) and rint(f * 2048) (float32, each rounded on its own).
//    Columns outside [0, in - 1) take s = clamp, f = 0; rows keep their coefficients and clamp only the row index.
//    Every step is an explicitly rounded intrinsic, so no FMA contraction changes a coefficient.
//  - horizontal S = p0 * c0 + p1 * c1, vertical (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2.
//  - an exact 2x downscale on both axes is cv2's INTER_AREA fast path, (a + b + c + d + 2) >> 2 per 2x2 block;
//    equal sizes are a layout change only.
// The coefficients are computed where they are used rather than copied from a host table: the same IEEE operations
// give the same integers, and the call needs no host-to-device copy.
// One CTA owns a 128 x 16 output tile of one view; a thread keeps its column's taps in registers for all 16 rows,
// the rows' taps are computed once per CTA. Stores are coalesced along each output row of each channel plane.
#include "common.cuh"

namespace {

constexpr int kTileW = 128, kTileH = 16;
enum ResizeMode { kCopy = 0, kLinear = 1, kArea2x = 2 };

struct Taps {
  int i0, i1, c0, c1;
};

__device__ __forceinline__ Taps linear_taps(int d, int n_out, int n_in, bool clamp_coef) {
  const double scale = __ddiv_rn(1.0, __ddiv_rn((double)n_out, (double)n_in));
  float f = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5));
  int s = (int)floorf(f);
  f = __fsub_rn(f, (float)s);
  if (clamp_coef && (s < 0 || s >= n_in - 1)) f = 0.f;
  Taps t;
  t.i0 = min(max(s, 0), n_in - 1);
  t.i1 = min(max(s + 1, 0), n_in - 1);
  t.c0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  t.c1 = __float2int_rn(__fmul_rn(f, 2048.f));
  return t;
}

template <int MODE>
__global__ void __launch_bounds__(kTileW) resize_u8_kernel(const unsigned char* __restrict__ src, int H, int W,
                                                           unsigned char* __restrict__ dst, int h, int w) {
  __shared__ int4 row_taps[kTileH];
  const int x = blockIdx.x * kTileW + threadIdx.x;
  const int y0 = blockIdx.y * kTileH;
  const int rows = min(kTileH, h - y0);
  const unsigned char* s = src + (long long)blockIdx.z * H * W * 3;
  const long long plane = (long long)h * w;
  unsigned char* d = dst + (long long)blockIdx.z * 3 * plane + (long long)y0 * w + x;
  if (MODE == kLinear) {
    if (threadIdx.x < rows) {
      const Taps t = linear_taps(y0 + threadIdx.x, h, H, false);
      row_taps[threadIdx.x] = make_int4(t.i0, t.i1, t.c0, t.c1);
    }
    __syncthreads();
  }
  if (x >= w) return;
  if (MODE == kCopy) {
    const unsigned char* p = s + ((long long)y0 * W + x) * 3;
    for (int r = 0; r < rows; ++r, p += (long long)W * 3, d += w) {
#pragma unroll
      for (int c = 0; c < 3; ++c) d[c * plane] = __ldg(p + c);
    }
  } else if (MODE == kArea2x) {
    const unsigned char* p = s + ((long long)2 * y0 * W + 2 * x) * 3;
    for (int r = 0; r < rows; ++r, p += (long long)2 * W * 3, d += w) {
      const unsigned char* q = p + (long long)W * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int sum = __ldg(p + c) + __ldg(p + 3 + c) + __ldg(q + c) + __ldg(q + 3 + c);
        d[c * plane] = (unsigned char)((sum + 2) >> 2);
      }
    }
  } else {
    const Taps tx = linear_taps(x, w, W, true);
    const int o0 = tx.i0 * 3, o1 = tx.i1 * 3;
    for (int r = 0; r < rows; ++r, d += w) {
      const int4 ty = row_taps[r];
      const unsigned char* p0 = s + (long long)ty.x * W * 3;
      const unsigned char* p1 = s + (long long)ty.y * W * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int s0 = __ldg(p0 + o0 + c) * tx.c0 + __ldg(p0 + o1 + c) * tx.c1;
        const int s1 = __ldg(p1 + o0 + c) * tx.c0 + __ldg(p1 + o1 + c) * tx.c1;
        d[c * plane] = (unsigned char)((((ty.z * (s0 >> 4)) >> 16) + ((ty.w * (s1 >> 4)) >> 16) + 2) >> 2);
      }
    }
  }
}

// cv2 runs INTER_LINEAR as INTER_AREA when both scales 1 / (out / in) round to exactly the integer 2
bool is_area_2x(int H, int W, int h, int w) {
  const double sx = 1.0 / ((double)w / W), sy = 1.0 / ((double)h / H);
  return sx == 2.0 && sy == 2.0;
}

}  // namespace

extern "C" int esb_img_resize_linear_u8(const unsigned char* src, int V, int H, int W, int h, int w,
                                        unsigned char* dst, void* stream) {
  ESB_CHECK_ARG(V >= 0 && V <= 65535, "esb_img_resize_linear_u8: V = %d outside [0, 65535]", V);
  ESB_CHECK_ARG(H > 0 && W > 0 && h > 0 && w > 0, "esb_img_resize_linear_u8: empty frame (%dx%d -> %dx%d)", W, H, w, h);
  ESB_CHECK_ARG(h <= 65535 * kTileH, "esb_img_resize_linear_u8: h = %d too large", h);
  if (V == 0) return ESB_OK;
  const dim3 grid(esb_div_up(w, kTileW), esb_div_up(h, kTileH), V);
  cudaStream_t s = (cudaStream_t)stream;
  if (h == H && w == W)
    resize_u8_kernel<kCopy><<<grid, kTileW, 0, s>>>(src, H, W, dst, h, w);
  else if (is_area_2x(H, W, h, w))
    resize_u8_kernel<kArea2x><<<grid, kTileW, 0, s>>>(src, H, W, dst, h, w);
  else
    resize_u8_kernel<kLinear><<<grid, kTileW, 0, s>>>(src, H, W, dst, h, w);
  ESB_CUDA_LAUNCH_CHECK("resize_u8_kernel");
  return ESB_OK;
}
