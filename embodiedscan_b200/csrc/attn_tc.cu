// esb200 — multi-head attention core of the grounding decoder (SURVEY §8 row a15: text<->3D cross-attention, self-attention
// and text cross-attention of embodiedscan/models/layers/ground_transformer/decoder.py:89-95,151-177; 8 heads of 32 channels,
// 256 queries, up to ~3.5k keys, key padding mask) as flash-attention tiles on wgmma fed by TMA, forward AND backward.
//
// forward  (one CTA = 128 queries of one (scan, head)): Q, K, V tiles arrive as 64B-swizzled TMA boxes; two consumer
//   warpgroups own 64 queries each. S = Q K^T is one wgmma pair (m64, N=128 keys, K=32) into registers; the four lanes that
//   hold a query row keep its running maximum / sum in the exp2 domain, write P (bf16) as the K-major 128B-swizzled A operand;
//   O_tile = P V is eight more wgmma with V read as the MN-major B operand (no transpose); O is rescaled in registers. Stores O
//   (bf16) and the log-sum-exp.
// backward (one CTA = 128 keys of one (scan, head), loop over query tiles): S^T = K Q^T and dP^T = V dO^T in registers of the
//   warpgroup that owns the key rows, which recomputes P^T and dS^T = P^T o (dP^T - delta) * scale and stores both as K-major
//   A tiles; dV += P^T dO and dK += dS^T Q accumulate in registers over all query tiles (dO, Q read MN-major);
//   dQ_tile = dS K reads the SAME dS^T tile as the MN-major A operand and K as the MN-major B operand and is stored to this
//   key tile's partial of dQ; the host adds the key tiles in order.
// Layout: q (B,H,Lq,32), k / v (B,H,Lk,32) bf16 contiguous; key_pad (B,Lk) uint8, 1 = ignore; lse (B,H,Lq) natural log.
// Roofline: tensor pipe for long key sets, launch / latency bound at decoder sizes (256 x 3.5k x 32 per head).
#include "tc_common.cuh"

using namespace esb_tc;

namespace {

constexpr int AT_D = 32;                    // head dimension
constexpr int AT_CONS = 256;                // two consumer warpgroups
constexpr int AT_THREADS = AT_CONS + 32;    // + the TMA producer warp
constexpr float LOG2E = 1.4426950408889634f;

__device__ __forceinline__ uint32_t swz128(uint32_t row, uint32_t piece) { return row * 128u + ((piece ^ (row & 7u)) << 4); }
// byte offset of element (row, col) of a [128 rows][128 cols] bf16 tile stored as two K-major 128B-swizzled 64-column chunks
__device__ __forceinline__ uint32_t tile_off(int row, int col) {
  return (uint32_t)(col >> 6) * 16384u + swz128((uint32_t)row, (uint32_t)((col & 63) >> 3)) + (uint32_t)(col & 7) * 2u;
}

// ------------------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(AT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmq, const __grid_constant__ CUtensorMap tmk,
                const __grid_constant__ CUtensorMap tmv, const unsigned char* __restrict__ key_pad,
                __nv_bfloat16* __restrict__ o, float* __restrict__ lse, int H, int Lq, int Lk, float scale) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* q_s = smem;                        // 128 x 64 B
  uint8_t* k_s = smem + 8192;                 // 2 stages x 8 KB
  uint8_t* v_s = smem + 8192 * 3;             // 2 stages x 8 KB
  uint8_t* p_s = smem + 8192 * 5;             // 2 chunks x 16 KB (offset 40960: 1024-aligned)
  uint64_t* bars = (uint64_t*)(p_s + 32768);
  uint64_t *q_full = bars, *kv_full = bars + 1, *kv_empty = bars + 3;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int bh = blockIdx.y, b = bh / H;
  const int q0 = blockIdx.x * 128;
  const int n_kt = (Lk + 127) / 128;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < 2; ++s) { mbar_init(&kv_full[s], 1); mbar_init(&kv_empty[s], AT_CONS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tma_prefetch_desc(&tmq); tma_prefetch_desc(&tmk); tma_prefetch_desc(&tmv);
  }
  __syncthreads();

  if (threadIdx.x >= AT_CONS) {
    if (lane == 0) {
      mbar_expect_tx(q_full, 8192);
      tma_load_2d(&tmq, q_full, smem_u32(q_s), 0, bh * Lq + q0);
      for (int j = 0; j < n_kt; ++j) {
        const int s = j & 1;
        mbar_wait(&kv_empty[s], ((j >> 1) & 1) ^ 1);
        mbar_expect_tx(&kv_full[s], 16384);
        tma_load_2d(&tmk, &kv_full[s], smem_u32(k_s + s * 8192), 0, bh * Lk + j * 128);
        tma_load_2d(&tmv, &kv_full[s], smem_u32(v_s + s * 8192), 0, bh * Lk + j * 128);
      }
    }
    return;
  }
  // ---- consumers: warpgroup wg owns queries 64 wg .. 64 wg + 63 of the tile; this thread holds rows ra and ra + 8 ----
  const int wg = threadIdx.x >> 7;
  const int ra = wg * 64 + 16 * (warp & 3) + (lane >> 2);
  const int cq = 2 * (lane & 3);                             // first of this thread's two columns in every 8-column block
  const float sc2 = scale * LOG2E;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};    // running maximum (exp2 domain) / this thread's partial sum
  float acc[AT_D / 2], sacc[64], oacc[AT_D / 2];
#pragma unroll
  for (int e = 0; e < AT_D / 2; ++e) acc[e] = 0.f;
  mbar_wait(q_full, 0);
  const uint32_t qa = smem_u32(q_s) + wg * 4096, pa = smem_u32(p_s) + wg * 8192;
  for (int j = 0; j < n_kt; ++j) {
    const int s = j & 1;
    mbar_wait(&kv_full[s], (j >> 1) & 1);
    const uint32_t ka = smem_u32(k_s + s * 8192), va = smem_u32(v_s + s * 8192);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 2; ++kk)
      wgmma_bf16<128, 0, 0>(sacc, make_desc_sw(qa + kk * 32, 16, 512, SW64), make_desc_sw(ka + kk * 32, 16, 512, SW64), kk > 0);
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence<64>(sacc);
    // key mask of this thread's 32 columns (identical for every query row)
    uint32_t dead = 0;
#pragma unroll
    for (int jb = 0; jb < 16; ++jb)
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int kj = j * 128 + 8 * jb + cq + u;
        if (kj >= Lk || (key_pad != nullptr && key_pad[(long long)b * Lk + kj])) dead |= 1u << (2 * jb + u);
      }
    float alpha[2], m_use[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = m[h];
#pragma unroll
      for (int jb = 0; jb < 16; ++jb)
#pragma unroll
        for (int u = 0; u < 2; ++u)
          if (!((dead >> (2 * jb + u)) & 1)) mx = fmaxf(mx, sacc[4 * jb + 2 * h + u] * sc2);
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      m_use[h] = mx == -INFINITY ? 0.f : mx;
      alpha[h] = exp2f(m[h] - m_use[h]);                     // m = -inf -> 0
      m[h] = mx;
    }
    // probabilities -> bf16 A operand in shared memory (this warpgroup's rows only)
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int jb = 0; jb < 16; ++jb)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float p0 = ((dead >> (2 * jb)) & 1) ? 0.f : exp2f(sacc[4 * jb + 2 * h] * sc2 - m_use[h]);
        const float p1 = ((dead >> (2 * jb + 1)) & 1) ? 0.f : exp2f(sacc[4 * jb + 2 * h + 1] * sc2 - m_use[h]);
        rs[h] += p0 + p1;
        *reinterpret_cast<uint32_t*>(p_s + tile_off(ra + 8 * h, 8 * jb + cq)) = pack_bf16(__float_as_uint(p0), __float_as_uint(p1));
      }
#pragma unroll
    for (int h = 0; h < 2; ++h) l[h] = l[h] * alpha[h] + rs[h];
    fence_proxy_async();
    asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");   // the warpgroup's P rows are complete
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
      wgmma_bf16<AT_D, 0, 1>(oacc, make_desc_sw(pa + (kk >> 2) * 16384 + (kk & 3) * 32, 16, 1024, SW128),
                             make_desc_sw(va + kk * 1024, 2048, 512, SW64), kk > 0);
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence<AT_D / 2>(oacc);
    if (lane == 0) mbar_arrive(&kv_empty[s]);
#pragma unroll
    for (int e = 0; e < AT_D / 2; ++e) acc[e] = acc[e] * alpha[(e >> 1) & 1] + oacc[e];
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
    const int qi = q0 + ra + 8 * h;
    if (qi < Lq) {
      const float inv = l[h] > 0.f ? 1.f / l[h] : 0.f;
      __nv_bfloat16* dst = o + ((long long)bh * Lq + qi) * AT_D;
#pragma unroll
      for (int jb = 0; jb < AT_D / 8; ++jb)
        *reinterpret_cast<uint32_t*>(dst + 8 * jb + cq) =
            pack_bf16(__float_as_uint(acc[4 * jb + 2 * h] * inv), __float_as_uint(acc[4 * jb + 2 * h + 1] * inv));
      if ((lane & 3) == 0) lse[(long long)bh * Lq + qi] = l[h] > 0.f ? (m[h] + log2f(l[h])) * 0.6931471805599453f : -INFINITY;
    }
  }
}

// delta[bh, q] = sum_d dO * O  (fp32)
__global__ void attn_delta_kernel(const __nv_bfloat16* __restrict__ o, const __nv_bfloat16* __restrict__ dout,
                                  float* __restrict__ delta, long long rows) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows) return;
  float s = 0.f;
  const uint4* a = reinterpret_cast<const uint4*>(o + i * AT_D);
  const uint4* g = reinterpret_cast<const uint4*>(dout + i * AT_D);
#pragma unroll
  for (int h = 0; h < 4; ++h) {
    const uint4 x = a[h], y = g[h];
    const __nv_bfloat162* xp = reinterpret_cast<const __nv_bfloat162*>(&x);
    const __nv_bfloat162* yp = reinterpret_cast<const __nv_bfloat162*>(&y);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 xf = __bfloat1622float2(xp[e]), yf = __bfloat1622float2(yp[e]);
      s = fmaf(xf.x, yf.x, s);
      s = fmaf(xf.y, yf.y, s);
    }
  }
  delta[i] = s;
}

// ------------------------------------------------------------------------------------------------------------
// backward
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(AT_THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmq, const __grid_constant__ CUtensorMap tmk,
                const __grid_constant__ CUtensorMap tmv, const __grid_constant__ CUtensorMap tmdo,
                const unsigned char* __restrict__ key_pad, const float* __restrict__ lse, const float* __restrict__ delta,
                float* __restrict__ dq, __nv_bfloat16* __restrict__ dk, __nv_bfloat16* __restrict__ dv, int H, int Lq, int Lk,
                float scale) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* k_s = smem;                        // 8 KB
  uint8_t* v_s = smem + 8192;                 // 8 KB
  uint8_t* q_s = smem + 16384;                // 2 stages x 8 KB
  uint8_t* do_s = smem + 32768;               // 2 stages x 8 KB
  uint8_t* pt_s = smem + 49152;               // P^T: 2 chunks x 16 KB (1024-aligned)
  uint8_t* ds_s = smem + 49152 + 32768;       // dS^T
  float* lse2_all = (float*)(smem + 49152 + 65536);        // 2 x 128: lse * log2e of the query tile (tiles alternate buffers)
  float* delta_all = lse2_all + 256;
  uint64_t* bars = (uint64_t*)(delta_all + 256);
  uint64_t *kv_full = bars, *qd_full = bars + 1, *qd_empty = bars + 3;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int bh = blockIdx.y, b = bh / H;
  const int k0 = blockIdx.x * 128;
  const int n_qt = (Lq + 127) / 128;

  if (threadIdx.x == 0) {
    mbar_init(kv_full, 1);
    for (int s = 0; s < 2; ++s) { mbar_init(&qd_full[s], 1); mbar_init(&qd_empty[s], AT_CONS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tma_prefetch_desc(&tmq); tma_prefetch_desc(&tmk); tma_prefetch_desc(&tmv); tma_prefetch_desc(&tmdo);
  }
  __syncthreads();

  if (threadIdx.x >= AT_CONS) {
    if (lane == 0) {
      mbar_expect_tx(kv_full, 16384);
      tma_load_2d(&tmk, kv_full, smem_u32(k_s), 0, bh * Lk + k0);
      tma_load_2d(&tmv, kv_full, smem_u32(v_s), 0, bh * Lk + k0);
      for (int i = 0; i < n_qt; ++i) {
        const int s = i & 1;
        mbar_wait(&qd_empty[s], ((i >> 1) & 1) ^ 1);
        mbar_expect_tx(&qd_full[s], 16384);
        tma_load_2d(&tmq, &qd_full[s], smem_u32(q_s + s * 8192), 0, bh * Lq + i * 128);
        tma_load_2d(&tmdo, &qd_full[s], smem_u32(do_s + s * 8192), 0, bh * Lq + i * 128);
      }
    }
    return;
  }
  // ---- consumers: warpgroup wg owns keys 64 wg .. 64 wg + 63 (S^T, dP^T, dV, dK rows) and queries 64 wg .. of every query
  // tile (dQ rows); this thread holds fragment rows ra and ra + 8 ----
  const int t = threadIdx.x, wg = t >> 7;
  const int ra = wg * 64 + 16 * (warp & 3) + (lane >> 2);
  const int cq = 2 * (lane & 3);
  bool k_dead[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int kj = k0 + ra + 8 * h;
    k_dead[h] = kj >= Lk || (key_pad != nullptr && key_pad[(long long)b * Lk + kj]);
  }
  const float sc2 = scale * LOG2E;
  float sacc[64], pacc[64], dvacc[AT_D / 2], dkacc[AT_D / 2], dqacc[AT_D / 2];
  const uint32_t ka = smem_u32(k_s), va = smem_u32(v_s), pa = smem_u32(pt_s), sa = smem_u32(ds_s);
  mbar_wait(kv_full, 0);
  for (int i = 0; i < n_qt; ++i) {
    const int s = i & 1;
    float* lse2_s = lse2_all + (i & 1) * 128;
    float* delta_s = delta_all + (i & 1) * 128;
    if (t < 128) {
      const int qi = i * 128 + t;
      lse2_s[t] = qi < Lq ? lse[(long long)bh * Lq + qi] * LOG2E : INFINITY;     // +inf -> p = 0 for absent queries
      delta_s[t] = qi < Lq ? delta[(long long)bh * Lq + qi] : 0.f;
    }
    // lse2 / delta of this tile are written; both warpgroups are past tile i - 1 (its dQ MMA read every row of dS^T)
    asm volatile("bar.sync 1, %0;" ::"n"(AT_CONS) : "memory");
    mbar_wait(&qd_full[s], (i >> 1) & 1);
    const uint32_t qa = smem_u32(q_s + s * 8192), da = smem_u32(do_s + s * 8192);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 2; ++kk)
      wgmma_bf16<128, 0, 0>(sacc, make_desc_sw(ka + wg * 4096 + kk * 32, 16, 512, SW64), make_desc_sw(qa + kk * 32, 16, 512, SW64),
                            kk > 0);
#pragma unroll
    for (int kk = 0; kk < 2; ++kk)
      wgmma_bf16<128, 0, 0>(pacc, make_desc_sw(va + wg * 4096 + kk * 32, 16, 512, SW64), make_desc_sw(da + kk * 32, 16, 512, SW64),
                            kk > 0);
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence<64>(sacc);
    acc_fence<64>(pacc);
#pragma unroll
    for (int jb = 0; jb < 16; ++jb)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float p[2], ds[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int c = 8 * jb + cq + u, e = 4 * jb + 2 * h + u;
          const float ex = k_dead[h] ? 0.f : exp2f(sacc[e] * sc2 - lse2_s[c]);
          p[u] = ex;
          ds[u] = ex * (pacc[e] - delta_s[c]) * scale;
        }
        const uint32_t off = tile_off(ra + 8 * h, 8 * jb + cq);
        *reinterpret_cast<uint32_t*>(pt_s + off) = pack_bf16(__float_as_uint(p[0]), __float_as_uint(p[1]));
        *reinterpret_cast<uint32_t*>(ds_s + off) = pack_bf16(__float_as_uint(ds[0]), __float_as_uint(ds[1]));
      }
    fence_proxy_async();
    asm volatile("bar.sync 1, %0;" ::"n"(AT_CONS) : "memory");   // P^T and dS^T of this query tile are complete
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {                           // reduction over the 128 queries of the tile
      const uint32_t a_off = wg * 8192 + (kk >> 2) * 16384 + (kk & 3) * 32;
      wgmma_bf16<AT_D, 0, 1>(dvacc, make_desc_sw(pa + a_off, 16, 1024, SW128), make_desc_sw(da + kk * 1024, 2048, 512, SW64),
                             i > 0 || kk > 0);
      wgmma_bf16<AT_D, 0, 1>(dkacc, make_desc_sw(sa + a_off, 16, 1024, SW128), make_desc_sw(qa + kk * 1024, 2048, 512, SW64),
                             i > 0 || kk > 0);
    }
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)                             // reduction over the 128 keys of this CTA
      wgmma_bf16<AT_D, 1, 1>(dqacc, make_desc_sw(sa + wg * 16384 + kk * 2048, 16384, 1024, SW128),
                             make_desc_sw(ka + kk * 1024, 2048, 512, SW64), kk > 0);
    wgmma_commit();
    wgmma_wait<0>();
    acc_fence<AT_D / 2>(dvacc);
    acc_fence<AT_D / 2>(dkacc);
    acc_fence<AT_D / 2>(dqacc);
    if (lane == 0) mbar_arrive(&qd_empty[s]);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int qi = i * 128 + ra + 8 * h;
      if (qi < Lq) {
        float* dst = dq + (((long long)blockIdx.x * gridDim.y + bh) * Lq + qi) * AT_D;     // partial of key tile blockIdx.x
#pragma unroll
        for (int jb = 0; jb < AT_D / 8; ++jb)
          *reinterpret_cast<float2*>(dst + 8 * jb + cq) = make_float2(dqacc[4 * jb + 2 * h], dqacc[4 * jb + 2 * h + 1]);
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int kj = k0 + ra + 8 * h;
    if (kj < Lk) {
      __nv_bfloat16* pv = dv + ((long long)bh * Lk + kj) * AT_D;
      __nv_bfloat16* pk = dk + ((long long)bh * Lk + kj) * AT_D;
#pragma unroll
      for (int jb = 0; jb < AT_D / 8; ++jb) {
        *reinterpret_cast<uint32_t*>(pv + 8 * jb + cq) =
            pack_bf16(__float_as_uint(dvacc[4 * jb + 2 * h]), __float_as_uint(dvacc[4 * jb + 2 * h + 1]));
        *reinterpret_cast<uint32_t*>(pk + 8 * jb + cq) =
            pack_bf16(__float_as_uint(dkacc[4 * jb + 2 * h]), __float_as_uint(dkacc[4 * jb + 2 * h + 1]));
      }
    }
  }
}

int rows32_map(CUtensorMap* tm, const void* base, long long rows) {      // (rows, 32) bf16: boxes of 128 rows, 64B swizzle
  unsigned long long dims[2] = {AT_D, (unsigned long long)(rows > 0 ? rows : 1)};
  unsigned long long str[1] = {AT_D * 2};
  unsigned box[2] = {AT_D, 128};
  return esb_tma_encode(tm, base, 2, dims, str, box, nullptr, 64);
}

}  // namespace

// o (B,H,Lq,32) = softmax(q k^T * scale + key padding) v ; lse (B,H,Lq) fp32 = log-sum-exp of the scaled scores (-inf for a query
// whose keys are all padded: its output row is zero).
extern "C" int esb_attn_fwd(const void* q, const void* k, const void* v, const unsigned char* key_pad, void* o, float* lse, int B,
                            int H, int Lq, int Lk, float scale, void* stream_) {
  ESB_CHECK_ARG(B > 0 && H > 0 && Lq > 0 && Lk > 0, "esb_attn_fwd: empty problem");
  CUtensorMap tmq, tmk, tmv;
  int rc = rows32_map(&tmq, q, (long long)B * H * Lq);
  if (rc == ESB_OK) rc = rows32_map(&tmk, k, (long long)B * H * Lk);
  if (rc == ESB_OK) rc = rows32_map(&tmv, v, (long long)B * H * Lk);
  if (rc != ESB_OK) return rc;
  const size_t smem = 8192 * 5 + 32768 + 8 * 8 + 1024;
  cudaError_t e = cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { esb_set_error("esb_attn_fwd: smem attr: %s", cudaGetErrorString(e)); return ESB_ECUDA; }
  dim3 grid((Lq + 127) / 128, B * H);
  attn_fwd_kernel<<<grid, AT_THREADS, smem, (cudaStream_t)stream_>>>(tmq, tmk, tmv, key_pad, (__nv_bfloat16*)o, lse, H, Lq, Lk, scale);
  ESB_CUDA_LAUNCH_CHECK("attn_fwd_kernel");
  return ESB_OK;
}

// dq (B,H,Lq,32) fp32 += the query gradient (zeroed by the caller; the key tiles' partials are added in order); dk, dv
// (B,H,Lk,32) bf16 written once;
// delta (B,H,Lq) fp32 workspace.
extern "C" int esb_attn_bwd(const void* q, const void* k, const void* v, const unsigned char* key_pad, const void* o,
                            const void* dout, const float* lse, float* delta, float* dq, void* dk, void* dv, int B, int H, int Lq,
                            int Lk, float scale, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  ESB_CHECK_ARG(B > 0 && H > 0 && Lq > 0 && Lk > 0, "esb_attn_bwd: empty problem");
  CUtensorMap tmq, tmk, tmv, tmdo;
  int rc = rows32_map(&tmq, q, (long long)B * H * Lq);
  if (rc == ESB_OK) rc = rows32_map(&tmk, k, (long long)B * H * Lk);
  if (rc == ESB_OK) rc = rows32_map(&tmv, v, (long long)B * H * Lk);
  if (rc == ESB_OK) rc = rows32_map(&tmdo, dout, (long long)B * H * Lq);
  if (rc != ESB_OK) return rc;
  const long long rows = (long long)B * H * Lq;
  attn_delta_kernel<<<esb_div_up(rows, 256), 256, 0, stream>>>((const __nv_bfloat16*)o, (const __nv_bfloat16*)dout, delta, rows);
  ESB_CUDA_LAUNCH_CHECK("attn_delta_kernel");
  const size_t smem = 49152 + 65536 + 2048 + 8 * 8 + 1024;
  cudaError_t e = cudaFuncSetAttribute(attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { esb_set_error("esb_attn_bwd: smem attr: %s", cudaGetErrorString(e)); return ESB_ECUDA; }
  dim3 grid((Lk + 127) / 128, B * H);
  const long long width = rows * AT_D;
  float* part = nullptr;
  ESB_CUDA_CALL(esb_scratch_alloc((void**)&part, sizeof(float) * grid.x * width, stream));
  attn_bwd_kernel<<<grid, AT_THREADS, smem, stream>>>(tmq, tmk, tmv, tmdo, key_pad, lse, delta, part, (__nv_bfloat16*)dk,
                                                      (__nv_bfloat16*)dv, H, Lq, Lk, scale);
  ESB_CUDA_LAUNCH_CHECK("attn_bwd_kernel");
  rc = esb_sum_partial_rows(part, (int)grid.x, width, dq, 1, stream);
  ESB_CUDA_CALL(esb_scratch_free(part, stream));
  return rc;
}
