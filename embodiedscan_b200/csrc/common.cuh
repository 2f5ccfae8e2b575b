// esb200 — shared device/host helpers for the sm_90a kernels behind libesb200.so.
// Buffers that cross the C ABI belong to the caller (PyTorch host); the only memory the library takes itself is the
// stream-ordered scratch of its deterministic reductions.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/esb200.h"  // the compiler checks every definition against the published ABI

void esb_set_error(const char* fmt, ...);

#define ESB_CHECK_ARG(cond, ...)                      \
  do {                                                \
    if (!(cond)) {                                    \
      esb_set_error(__VA_ARGS__);                     \
      return ESB_EINVAL;                              \
    }                                                 \
  } while (0)

#define ESB_CUDA_LAUNCH_CHECK(name)                                        \
  do {                                                                     \
    cudaError_t _e = cudaPeekAtLastError();                                \
    if (_e != cudaSuccess) {                                               \
      esb_set_error("%s: CUDA error %s", name, cudaGetErrorString(_e));    \
      return ESB_ECUDA;                                                    \
    }                                                                      \
  } while (0)

#define ESB_CUDA_CALL(expr)                                                \
  do {                                                                     \
    cudaError_t _e = (expr);                                               \
    if (_e != cudaSuccess) {                                               \
      esb_set_error("%s: CUDA error %s", #expr, cudaGetErrorString(_e));   \
      return ESB_ECUDA;                                                    \
    }                                                                      \
  } while (0)

static inline int esb_div_up(long long a, long long b) { return (int)((a + b - 1) / b); }
static inline size_t esb_align(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }
// ---- deterministic reductions (scratch.cu) --------------------------------------------------------------------------
// Kernels never combine partial sums with float atomics (their order, and so the rounding, would change from run to run):
// each block / split writes its partial to stream-ordered scratch memory and one of the reducers below adds the partials
// in index order. The scratch comes from the device's stream-ordered pool and is released on the same stream.
cudaError_t esb_scratch_alloc(void** p, size_t bytes, cudaStream_t s);
cudaError_t esb_scratch_free(void* p, cudaStream_t s);
// out[j] (+)= sum over p = 0 .. n_parts-1 of part[p * width + j], in that order. accumulate = 0 overwrites out; 1 starts the
// add chain from out[j]; 2 finishes the sum from +0 and adds it to out[j] with one rounded add (gradient slots, see
// esb_norm_bwd: the slot then receives exactly what autograd's `grad += fresh` would add)
int esb_sum_partial_rows(const float* part, int n_parts, long long width, float* out, int accumulate, cudaStream_t s);

// streaming multiprocessors of the current device (grid sizing; read once per device)
int esb_sm_count();

// ---- chamfer criteria (ESB_CD_*), per coordinate: torch l1_loss / mse_loss / smooth_l1_loss(beta=1), reduction none --
// The products are rounded on their own (no FMA contraction), as ATen rounds them, so nearest-neighbour choices agree.
template <int MODE>
__device__ __forceinline__ float esb_cd_crit(float x) {
  if constexpr (MODE == ESB_CD_L1) {
    return fabsf(x);
  } else if constexpr (MODE == ESB_CD_L2) {
    return __fmul_rn(x, x);
  } else {
    const float a = fabsf(x);
    return a < 1.f ? __fmul_rn(0.5f * a, a) : a - 0.5f;
  }
}
// derivative of esb_cd_crit: sign(x) with sign(0) = 0, 2x, x clamped to [-1, 1]
template <int MODE>
__device__ __forceinline__ float esb_cd_dcrit(float x) {
  if constexpr (MODE == ESB_CD_L1) {
    return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f);
  } else if constexpr (MODE == ESB_CD_L2) {
    return 2.f * x;
  } else {
    return fminf(fmaxf(x, -1.f), 1.f);
  }
}


// ---- coordinate key packing: [b:16 | x:16 | y:16 | z:16], xyz biased by 2^15 ----
#define ESB_EMPTY_KEY 0xFFFFFFFFFFFFFFFFull
#define ESB_COORD_BIAS 32768

__host__ __device__ __forceinline__ uint64_t esb_pack_key(int b, int x, int y, int z) {
  return ((uint64_t)(uint16_t)b << 48) | ((uint64_t)(uint16_t)(x + ESB_COORD_BIAS) << 32) |
         ((uint64_t)(uint16_t)(y + ESB_COORD_BIAS) << 16) | (uint64_t)(uint16_t)(z + ESB_COORD_BIAS);
}
__host__ __device__ __forceinline__ bool esb_coord_in_range(int b, int x, int y, int z) {
  return b >= 0 && b < 65535 && x >= -ESB_COORD_BIAS && x < ESB_COORD_BIAS && y >= -ESB_COORD_BIAS &&
         y < ESB_COORD_BIAS && z >= -ESB_COORD_BIAS && z < ESB_COORD_BIAS;
}
__host__ __device__ __forceinline__ uint32_t esb_hash64(uint64_t k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return (uint32_t)k;
}

#ifdef __CUDACC__
// floor division by a positive divisor (C division truncates toward zero).
__device__ __forceinline__ int esb_floor_div(int a, int d) {
  int q = a / d;
  return (a % d != 0 && a < 0) ? q - 1 : q;
}

__device__ __forceinline__ int esb_hash_find(const unsigned long long* __restrict__ keys,
                                             const int* __restrict__ vals, uint32_t mask, uint64_t key) {
  uint32_t slot = esb_hash64(key) & mask;
  for (uint32_t probe = 0; probe <= mask; ++probe) {
    unsigned long long k = keys[slot];
    if (k == key) return vals[slot];
    if (k == ESB_EMPTY_KEY) return -1;
    slot = (slot + 1) & mask;
  }
  return -1;
}

template <typename T>
__device__ __forceinline__ float esb_to_float(T v);
template <>
__device__ __forceinline__ float esb_to_float<float>(float v) { return v; }
template <>
__device__ __forceinline__ float esb_to_float<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T>
__device__ __forceinline__ T esb_from_float(float v);
template <>
__device__ __forceinline__ float esb_from_float<float>(float v) { return v; }
template <>
__device__ __forceinline__ __nv_bfloat16 esb_from_float<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ float esb_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float esb_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
#endif
