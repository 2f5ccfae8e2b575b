// esb200 — point painting (SURVEY §8 row a6): project voxel centres into the V views of their scan, fetch the
// nearest image-feature vector per view, zero/mean over valid views. One fused kernel replaces
// batch_point_sample + apply_3d_transformation + batch_points_cam2img + F.grid_sample(nearest)
// (embodiedscan/models/layers/fusion_layers/point_fusion.py:208-311, :20-107;
//  embodiedscan/structures/bbox_3d/utils.py:289-332) and the per-sample/per-level Python loop at
// embodiedscan/models/detectors/sparse_featfusion_single_stage.py:142-207.
//
// Index selection is integer-critical: every fp32 operation below is an explicit round-to-nearest
// intrinsic in the reference's evaluation order (no FMA contraction), mirrored 1:1 by oracle/fusion_ref.py.
// Quirks kept (SURVEY H4): the SUM runs over every view whose nearest pixel is inside the feature map, while the
// divisor counts only views passing the strict 0<x<w, 0<y<h, depth>0 test in padded-pixel units.
// HBM-bound: per point 12 B coords + v̄·C·e gathered + C·e written; a warp owns a point, lanes split channels.
#include <cub/cub.cuh>
#include "common.cuh"

#define ESB_PAINT_MAX_OPS 8
// op codes of the reversed 3D augmentation flow
#define ESB_OP_T 0
#define ESB_OP_S 1
#define ESB_OP_R 2
#define ESB_OP_HF 3
#define ESB_OP_VF 4

struct EsbPaintMeta {  // one per scan, 4-byte fields only (mirrored by ctypes in the host package)
  float sx, sy;        // img_scale_factor (w, h)
  float ox, oy;        // img_crop_offset (w, h)
  float ori_w;         // img_shape[1] (pre-padding width, used by flip)
  int flip;
  int n_ops;
  int op[ESB_PAINT_MAX_OPS];
  float param[ESB_PAINT_MAX_OPS][9];  // T: t[3] (already negated) ; S: s (already inverted) ; R: 3x3 row-major (already inverted)
};

namespace {

__device__ __forceinline__ void apply_ops(const EsbPaintMeta& m, float& x, float& y, float& z) {
  for (int i = 0; i < m.n_ops; ++i) {
    const float* p = m.param[i];
    switch (m.op[i]) {
      case ESB_OP_T: x = __fadd_rn(x, p[0]); y = __fadd_rn(y, p[1]); z = __fadd_rn(z, p[2]); break;
      case ESB_OP_S: x = __fmul_rn(x, p[0]); y = __fmul_rn(y, p[0]); z = __fmul_rn(z, p[0]); break;
      case ESB_OP_R: {  // points @ R : x' = x*R00 + y*R10 + z*R20
        float nx = __fadd_rn(__fadd_rn(__fmul_rn(x, p[0]), __fmul_rn(y, p[3])), __fmul_rn(z, p[6]));
        float ny = __fadd_rn(__fadd_rn(__fmul_rn(x, p[1]), __fmul_rn(y, p[4])), __fmul_rn(z, p[7]));
        float nz = __fadd_rn(__fadd_rn(__fmul_rn(x, p[2]), __fmul_rn(y, p[5])), __fmul_rn(z, p[8]));
        x = nx; y = ny; z = nz;
      } break;
      case ESB_OP_HF: x = -x; break;
      case ESB_OP_VF: y = -y; break;
      default: break;
    }
  }
}

// returns pixel linear index (iy*Wf+ix) or -1 when the nearest pixel is outside the map; *valid = reference's flag
__device__ __forceinline__ int project(const float* __restrict__ P, const EsbPaintMeta& m, float x, float y, float z,
                                       float pad_h, float pad_w, int Hf, int Wf, int* valid) {
  // [x y z 1] @ P^T, sequential products/sums
  float X = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, P[0]), __fmul_rn(y, P[1])), __fmul_rn(z, P[2])), P[3]);
  float Y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, P[4]), __fmul_rn(y, P[5])), __fmul_rn(z, P[6])), P[7]);
  float Z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, P[8]), __fmul_rn(y, P[9])), __fmul_rn(z, P[10])), P[11]);
  float zc = fmaxf(Z, 1e-3f);
  float u = __fdiv_rn(X, zc), v = __fdiv_rn(Y, zc);
  u = __fsub_rn(__fmul_rn(u, m.sx), m.ox);
  v = __fsub_rn(__fmul_rn(v, m.sy), m.oy);
  if (m.flip) u = __fsub_rn(m.ori_w, u);
  *valid = (u < pad_w) && (u > 0.f) && (v < pad_h) && (v > 0.f) && (Z > 0.f);
  float gx = __fsub_rn(__fmul_rn(__fdiv_rn(u, pad_w), 2.f), 1.f);
  float gy = __fsub_rn(__fmul_rn(__fdiv_rn(v, pad_h), 2.f), 1.f);
  // ATen grid_sampler_unnormalize(align_corners=True): ((g + 1) / 2) * (size - 1); nearest = nearbyint
  float fx = __fmul_rn(__fdiv_rn(__fadd_rn(gx, 1.f), 2.f), (float)(Wf - 1));
  float fy = __fmul_rn(__fdiv_rn(__fadd_rn(gy, 1.f), 2.f), (float)(Hf - 1));
  if (!(fabsf(fx) < 1e8f) || !(fabsf(fy) < 1e8f)) return -1;
  int ix = (int)nearbyintf(fx), iy = (int)nearbyintf(fy);
  if (ix < 0 || ix >= Wf || iy < 0 || iy >= Hf) return -1;
  return iy * Wf + ix;
}

// A point is either a voxel row (coords int32 [b,x,y,z] -> xyz * voxel_size) or, when fpts != NULL, an explicit fp32
// location fpts[n] of scan fbatch[n] (NULL: scan 0) — the prior-grid centres of the occupancy model
// (embodiedscan/models/detectors/dense_fusion_occ.py:156-202).
__device__ __forceinline__ void point_of(const int* __restrict__ coords, const float* __restrict__ fpts,
                                         const int* __restrict__ fbatch, long long n, float voxel_size,
                                         const EsbPaintMeta* __restrict__ metas, int* b, float* x, float* y, float* z) {
  if (fpts != nullptr) {
    *b = fbatch ? fbatch[n] : 0;
    *x = fpts[3 * n]; *y = fpts[3 * n + 1]; *z = fpts[3 * n + 2];
  } else {
    int4 c = reinterpret_cast<const int4*>(coords)[n];
    *b = c.x;
    *x = __fmul_rn((float)c.y, voxel_size);
    *y = __fmul_rn((float)c.z, voxel_size);
    *z = __fmul_rn((float)c.w, voxel_size);
  }
  apply_ops(metas[*b], *x, *y, *z);
}

// feat: (B*V, Hf, Wf, C) channels-last ; out: (N, C)
template <typename T>
__global__ void paint_fwd_kernel(const int* __restrict__ coords, const float* __restrict__ fpts,
                                 const int* __restrict__ fbatch, long long N, float voxel_size,
                                 const EsbPaintMeta* __restrict__ metas, const float* __restrict__ proj, int V,
                                 const T* __restrict__ feat, int Hf, int Wf, int C, float pad_h, float pad_w,
                                 T* __restrict__ out, int* __restrict__ valid_count) {
  const int lane = threadIdx.x & 31;
  const long long n = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  if (n >= N) return;
  int b; float x, y, z;
  point_of(coords, fpts, fbatch, n, voxel_size, metas, &b, &x, &y, &z);
  const EsbPaintMeta& m = metas[b];
  float acc[16];  // up to C = 512 : 16 channels per lane, channel = lane + 32*j ... stored strided
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = 0.f;
  int count = 0;
  for (int vb = 0; vb < V; vb += 32) {
    int v = vb + lane, pix = -1, ok = 0;
    if (v < V) pix = project(proj + ((long long)b * V + v) * 16, m, x, y, z, pad_h, pad_w, Hf, Wf, &ok);
    count += __popc(__ballot_sync(0xffffffffu, ok));
    unsigned hit = __ballot_sync(0xffffffffu, pix >= 0);
    while (hit) {
      int j = __ffs(hit) - 1;
      hit &= hit - 1;
      int pj = __shfl_sync(0xffffffffu, pix, j);
      const T* src = feat + (((long long)b * V + vb + j) * Hf * Wf + pj) * C;
#pragma unroll
      for (int q = 0; q < 16; ++q) {
        int c = lane + 32 * q;
        if (c < C) acc[q] += esb_to_float<T>(src[c]);
      }
    }
  }
  float inv = count > 0 ? 1.f / (float)count : 0.f;
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    int c = lane + 32 * q;
    if (c < C) out[n * C + c] = esb_from_float<T>(count > 0 ? acc[q] * inv : 0.f);
  }
  if (lane == 0 && valid_count) valid_count[n] = count;
}

// Backward, deterministic: a point's gradient dout[n] / count goes to the nearest pixel of every view that sees it. Pass 1
// writes one (pixel key, point) pair per (point, view) — key = (b*V + v)*Hf*Wf + pixel, or ~0u for a view that does not see
// the point; a stable radix sort groups the pairs by pixel with the points of a pixel in index order; pass 2 (one warp per
// pixel) adds them in that order, so dfeat does not depend on scheduling.
template <typename T>
__global__ void paint_bwd_pairs_kernel(const int* __restrict__ coords, const float* __restrict__ fpts,
                                       const int* __restrict__ fbatch, long long N, float voxel_size,
                                       const EsbPaintMeta* __restrict__ metas, const float* __restrict__ proj, int V, int Hf,
                                       int Wf, float pad_h, float pad_w, unsigned* __restrict__ keys, int* __restrict__ pts,
                                       float* __restrict__ inv_count) {
  const int lane = threadIdx.x & 31;
  const long long n = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  if (n >= N) return;
  int b; float x, y, z;
  point_of(coords, fpts, fbatch, n, voxel_size, metas, &b, &x, &y, &z);
  const EsbPaintMeta& m = metas[b];
  int count = 0;
  for (int vb = 0; vb < V; vb += 32) {
    int v = vb + lane, pix = -1, ok = 0;
    if (v < V) pix = project(proj + ((long long)b * V + v) * 16, m, x, y, z, pad_h, pad_w, Hf, Wf, &ok);
    count += __popc(__ballot_sync(0xffffffffu, ok));
    if (v < V) {
      keys[n * V + v] = pix >= 0 ? (unsigned)(((long long)b * V + v) * Hf * Wf + pix) : ~0u;
      pts[n * V + v] = (int)n;
    }
  }
  if (lane == 0) inv_count[n] = count > 0 ? 1.f / (float)count : 0.f;
}

template <typename T>
__global__ void paint_bwd_sum_kernel(const unsigned* __restrict__ keys, const int* __restrict__ pts, long long n_pairs,
                                     const float* __restrict__ inv_count, const T* __restrict__ dout, int C,
                                     float* __restrict__ dfeat) {
  const int lane = threadIdx.x & 31;
  const long long i = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  if (i >= n_pairs) return;
  const unsigned key = keys[i];
  if (key == ~0u || (i > 0 && keys[i - 1] == key)) return;          // not the first pair of a seen pixel
  float acc[16];
#pragma unroll
  for (int q = 0; q < 16; ++q) acc[q] = 0.f;
  for (long long j = i; j < n_pairs && keys[j] == key; ++j) {
    const long long n = pts[j];
    const float inv = inv_count[n];
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      const int c = lane + 32 * q;
      if (c < C) acc[q] += esb_to_float<T>(dout[n * C + c]) * inv;
    }
  }
  float* dst = dfeat + (long long)key * C;
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    const int c = lane + 32 * q;
    if (c < C) dst[c] += acc[q];
  }
}

}  // namespace

extern "C" int esb_paint_meta_bytes() { return (int)sizeof(EsbPaintMeta); }

extern "C" int esb_paint_fwd(const int* coords, const float* fpts, const int* fbatch, long long N, float voxel_size,
                             const void* metas, const float* proj,
                             int V, const void* feat, int Hf, int Wf, int C, float pad_h, float pad_w, void* out,
                             int* valid_count, int dtype, void* stream) {
  ESB_CHECK_ARG(C >= 1 && C <= 512, "esb_paint_fwd: C must be in [1,512]");
  ESB_CHECK_ARG(V >= 1, "esb_paint_fwd: V must be >= 1");
  if (N == 0) return ESB_OK;
  int grid = esb_div_up(N * 32, 256);
  if (dtype == ESB_F32)
    paint_fwd_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>(coords, fpts, fbatch, N, voxel_size, (const EsbPaintMeta*)metas, proj,
                                                                     V, (const float*)feat, Hf, Wf, C, pad_h, pad_w,
                                                                     (float*)out, valid_count);
  else
    paint_fwd_kernel<__nv_bfloat16><<<grid, 256, 0, (cudaStream_t)stream>>>(
        coords, fpts, fbatch, N, voxel_size, (const EsbPaintMeta*)metas, proj, V, (const __nv_bfloat16*)feat, Hf, Wf, C, pad_h, pad_w,
        (__nv_bfloat16*)out, valid_count);
  ESB_CUDA_LAUNCH_CHECK("paint_fwd_kernel");
  return ESB_OK;
}

// dfeat (fp32, the layout of feat) += d out / d feat; zero-initialised by the caller for a plain gradient.
extern "C" int esb_paint_bwd(const int* coords, const float* fpts, const int* fbatch, long long N, float voxel_size,
                             const void* metas, const float* proj,
                             int V, const void* dout, int Hf, int Wf, int C, float pad_h, float pad_w, float* dfeat,
                             int dtype, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  ESB_CHECK_ARG(C >= 1 && C <= 512, "esb_paint_bwd: C must be in [1,512]");
  if (N == 0) return ESB_OK;
  const long long n_pairs = N * V;
  ESB_CHECK_ARG(n_pairs < (1LL << 31), "esb_paint_bwd: too many (point, view) pairs");
  // pixel keys stay below 2^32 - 1 (the "not seen" marker) for feature maps of fewer than 4G pixels in all
  size_t temp_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr,
                                  (int*)nullptr, (int)n_pairs, 0, 32, stream);
  const size_t a_pairs = esb_align((size_t)n_pairs * 4);
  uint8_t* ws = nullptr;
  ESB_CUDA_CALL(esb_scratch_alloc((void**)&ws, 4 * a_pairs + esb_align((size_t)N * 4) + esb_align(temp_bytes), stream));
  unsigned* keys = (unsigned*)ws;
  unsigned* keys_s = (unsigned*)(ws + a_pairs);
  int* pts = (int*)(ws + 2 * a_pairs);
  int* pts_s = (int*)(ws + 3 * a_pairs);
  float* inv = (float*)(ws + 4 * a_pairs);
  void* temp = ws + 4 * a_pairs + esb_align((size_t)N * 4);
  const int grid = esb_div_up(N * 32, 256), grid2 = esb_div_up(n_pairs * 32, 256);
  if (dtype == ESB_F32)
    paint_bwd_pairs_kernel<float><<<grid, 256, 0, stream>>>(coords, fpts, fbatch, N, voxel_size, (const EsbPaintMeta*)metas, proj,
                                                            V, Hf, Wf, pad_h, pad_w, keys, pts, inv);
  else
    paint_bwd_pairs_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(coords, fpts, fbatch, N, voxel_size, (const EsbPaintMeta*)metas,
                                                                    proj, V, Hf, Wf, pad_h, pad_w, keys, pts, inv);
  ESB_CUDA_LAUNCH_CHECK("paint_bwd_pairs_kernel");
  cudaError_t e = cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys, keys_s, pts, pts_s, (int)n_pairs, 0, 32, stream);
  if (e != cudaSuccess) {
    esb_scratch_free(ws, stream);
    esb_set_error("esb_paint_bwd: sort: %s", cudaGetErrorString(e));
    return ESB_ECUDA;
  }
  if (dtype == ESB_F32)
    paint_bwd_sum_kernel<float><<<grid2, 256, 0, stream>>>(keys_s, pts_s, n_pairs, inv, (const float*)dout, C, dfeat);
  else
    paint_bwd_sum_kernel<__nv_bfloat16><<<grid2, 256, 0, stream>>>(keys_s, pts_s, n_pairs, inv, (const __nv_bfloat16*)dout, C,
                                                                   dfeat);
  ESB_CUDA_LAUNCH_CHECK("paint_bwd_sum_kernel");
  ESB_CUDA_CALL(esb_scratch_free(ws, stream));
  return ESB_OK;
}
