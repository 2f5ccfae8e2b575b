// esb200 — flat-arena optimiser step: global grad-norm (clip_grad max_norm=10, norm_type=2) and AdamW
// (lr 1e-3, weight_decay 1e-4; configs/detection/mv-det3d_8xb4_embodiedscan-3d-284class-9dof.py:219-223) over ONE
// contiguous fp32 parameter buffer and ONE contiguous gradient buffer (the same buffer NCCL all-reduces in
// buckets). Two launches per step instead of ~600 per-tensor kernels; pure HBM streaming: 16 B read + 12 B written
// per parameter. No host sync: the clip coefficient and step count stay on the device.
#include "common.cuh"

namespace {

__global__ void sumsq_kernel(const float* __restrict__ g, long long n, float* __restrict__ out) {
  float acc = 0.f;
  long long stride = (long long)gridDim.x * blockDim.x * 4;
  for (long long i = (blockIdx.x * (long long)blockDim.x + threadIdx.x) * 4; i < n; i += stride) {
    if (i + 3 < n) {
      float4 v = *reinterpret_cast<const float4*>(g + i);
      acc += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    } else {
      for (long long j = i; j < n; ++j) acc += g[j] * g[j];
    }
  }
  acc = esb_warp_sum(acc);
  __shared__ float red[32];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = esb_warp_sum(v);
    if (threadIdx.x == 0) out[blockIdx.x] = v;             // one partial per block, summed in block order
  }
}

// state[0] = sum of squares (input), state[1] = total norm (output), state[2] = clip coefficient (output)
__global__ void clip_coef_kernel(float* state, float max_norm, float world_scale) {
  float norm = sqrtf(state[0]) * world_scale;
  state[1] = norm;
  float coef = max_norm / (norm + 1e-6f);
  state[2] = max_norm > 0.f ? fminf(coef, 1.f) : 1.f;
}

// decoupled weight decay exactly as torch.optim.AdamW: p *= 1 - lr*wd ; p -= lr/bc1 * m / (sqrt(v)/sqrt(bc2) + eps)
// grad_scale folds the 1/world_size of the DDP mean and the clip coefficient (state[2]).
__global__ void adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                             float* __restrict__ v, const float* __restrict__ lr_mult, long long n, float lr, float beta1,
                             float beta2, float eps, float wd, float bc1, float bc2_sqrt, float grad_scale,
                             const float* __restrict__ state) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  float scale = grad_scale * (state ? state[2] : 1.f);
  float lm = lr_mult ? lr_mult[i] : 1.f;
  if (lm == 0.f) return;  // frozen parameter
  float gi = g[i] * scale;
  float mi = beta1 * m[i] + (1.f - beta1) * gi;
  float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
  m[i] = mi;
  v[i] = vi;
  float l = lr * lm;
  float pi = p[i] * (1.f - l * wd);
  float denom = sqrtf(vi) / bc2_sqrt + eps;
  p[i] = pi - (l / bc1) * (mi / denom);
}

template <typename T>
__global__ void cast_kernel(const float* __restrict__ src, T* __restrict__ dst, long long n) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) dst[i] = esb_from_float<T>(src[i]);
}

}  // namespace

// state: 3 device floats. Call with world_scale = 1/world_size when `grad` holds a SUM over ranks.
extern "C" int esb_grad_clip_coef(const float* grad, long long n, float max_norm, float world_scale, float* state,
                                  void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  ESB_CUDA_CALL(cudaMemsetAsync(state, 0, 3 * sizeof(float), stream));
  if (n > 0) {
    int grid = esb_div_up(n, 256 * 4 * 8);
    if (grid > esb_sm_count() * 8) grid = esb_sm_count() * 8;
    if (grid < 1) grid = 1;
    float* part = nullptr;
    ESB_CUDA_CALL(esb_scratch_alloc((void**)&part, (size_t)grid * sizeof(float), stream));
    sumsq_kernel<<<grid, 256, 0, stream>>>(grad, n, part);
    int rc = esb_sum_partial_rows(part, grid, 1, state, 0, stream);
    ESB_CUDA_CALL(esb_scratch_free(part, stream));
    if (rc != ESB_OK) return rc;
  }
  clip_coef_kernel<<<1, 1, 0, stream>>>(state, max_norm, world_scale);
  ESB_CUDA_LAUNCH_CHECK("esb_grad_clip_coef");
  return ESB_OK;
}

extern "C" int esb_adamw_step(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, const float* lr_mult,
                              long long n, float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                              float grad_scale, const float* clip_state, void* stream) {
  ESB_CHECK_ARG(step >= 1, "esb_adamw_step: step counts from 1");
  if (n == 0) return ESB_OK;
  float bc1 = 1.f - powf(beta1, (float)step);
  float bc2_sqrt = sqrtf(1.f - powf(beta2, (float)step));
  adamw_kernel<<<esb_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, lr_mult, n, lr, beta1,
                                                                      beta2, eps, weight_decay, bc1, bc2_sqrt,
                                                                      grad_scale, clip_state);
  ESB_CUDA_LAUNCH_CHECK("adamw_kernel");
  return ESB_OK;
}

// fp32 master arena -> bf16 compute copy (one launch for the whole model)
extern "C" int esb_cast_f32_to_bf16(const float* src, void* dst, long long n, void* stream) {
  if (n == 0) return ESB_OK;
  cast_kernel<__nv_bfloat16><<<esb_div_up(n, 256), 256, 0, (cudaStream_t)stream>>>(src, (__nv_bfloat16*)dst, n);
  ESB_CUDA_LAUNCH_CHECK("cast_kernel");
  return ESB_OK;
}
