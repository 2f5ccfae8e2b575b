// esb200 — sparse 3D convolution on the Hopper tensor cores (wgmma), bf16 in / fp32 accumulate.
// The throughput path for ME.MinkowskiConvolution forward / dgrad / wgrad (†upstream MinkowskiEngine; call sites
// embodiedscan/models/backbones/mink_resnet.py:58-62,104-108, embodiedscan/models/dense_heads/fcaf3d_head.py:919-946).
//
// forward / dgrad (spconv_tc_fwd_kernel): output-stationary implicit GEMM. A CTA owns 128 output rows x N_TILE output
// channels; for every kernel offset k that any row of the tile uses (per-tile bit mask) and every 64-channel slice of
// Cin it stages
//     A = the 128 gathered neighbour rows (cp.async 16 B, zero-filled where the neighbour is absent) and
//     B = W_k^T slice (N_TILE x 64, K-major)
// into 128B-swizzled shared memory; two consumer warpgroups issue wgmma (m64, N=N_TILE, K=16), 64 rows each, accumulating
// in registers; at the end of the tile they write the accumulator to shared memory (over the idle stage buffers) and the
// epilogue writes each output row once (no atomics, deterministic).
// Thread roles: threads 0-255 = the two consumer warpgroups; threads 256-383 = gather producers, then epilogue (thread =
// tile row). Full/empty mbarrier ring between producers and consumers; a consumer releases a stage once the wgmma group
// that read it has retired.
//
// wgrad (spconv_tc_wgrad_kernel): dW_k = X_k^T dY_k over the compacted pair list of offset k. Both operands are the
// gathered rows themselves, i.e. MN-major (M = Cin, N = Cout contiguous, reduction over pairs), staged in the
// canonical MN-major 128B-swizzle layout; split over pair ranges, each split's tile stored to scratch and the splits of an
// offset added to dW in order (spconv_wgrad_reduce_kernel).
//
// Roofline: pair model bytes = P*(Cin+Cout)*2 + 8P + K*Cin*Cout*2 (BASELINE.md §3); the gather is L2-fed.
#include "tc_common.cuh"

using namespace esb_tc;

namespace {

// per-tile (128 rows) bit mask of the kernel offsets that have at least one valid neighbour
__global__ void tile_mask_kernel(const int* __restrict__ nbr, int K, int n, uint32_t* __restrict__ masks) {
  const int tile = blockIdx.x, r = threadIdx.x;
  const int row = tile * TC_M + r;
  uint32_t m = 0;
  if (row < n)
    for (int k = 0; k < K; ++k)
      if (nbr[(long long)k * n + row] >= 0) m |= 1u << k;
  m = __reduce_or_sync(0xffffffffu, m);
  __shared__ uint32_t s[4];
  if ((r & 31) == 0) s[r >> 5] = m;
  __syncthreads();
  if (r == 0) masks[tile] = s[0] | s[1] | s[2] | s[3];
}

// ------------------------------------------------------------------------------------------------------------
// forward / dgrad
// ------------------------------------------------------------------------------------------------------------
// B_MN = false: wt is (K, cout, cin)  (W_k^T, reduction dim contiguous  -> K-major B; used by dgrad with wt = W itself)
// B_MN = true : wt is (K, cin, cout)  (W_k as stored, output dim contiguous -> MN-major B; used by forward, no transpose)
// The filter tile of every stage is ONE tiled TMA box (cp.async.bulk.tensor) issued by the first producer — the
// 128B-swizzled layouts wgmma reads are what the tensor map writes; the gathered rows arrive through cp.async.
template <int N_TILE, int STAGES, bool B_MN>
__global__ void __launch_bounds__(384, 1)
spconv_tc_fwd_kernel(const __nv_bfloat16* __restrict__ x, const __grid_constant__ CUtensorMap tmw,
                     const int* __restrict__ nbr, const uint32_t* __restrict__ masks, __nv_bfloat16* __restrict__ y,
                     int n_out, int cin, int cout, int K) {
  constexpr int A_BYTES = A_STAGE_BYTES;
  constexpr int B_STAGE_BYTES = N_TILE * 128;
  constexpr int STAGE_BYTES = A_BYTES + B_STAGE_BYTES;
  constexpr int LAG = STAGES - 2;                 // stages kept in flight per producer thread before it signals
  constexpr int NPROD = 128;
  constexpr int NCONS = 256;
  constexpr int PITCH = N_TILE + 4;               // floats per accumulator-image row
  static_assert(TC_M * PITCH * 4 <= STAGES * STAGE_BYTES, "the accumulator image reuses the stage buffers");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = (uint64_t*)(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* accum_bar = empty_bar + STAGES;
  float* img = reinterpret_cast<float*>(smem);
  __shared__ int idx_s[2][NPROD];

  const int tile = blockIdx.x;                     // 128 output rows
  const int n0 = blockIdx.y * N_TILE;
  const uint32_t mask = masks[tile];
  const int nchunk = cin / TC_BK;
  const int total = __popc(mask) * nchunk;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], NPROD + 1);          // every producer thread + the expect_tx arrival of the filter box
      mbar_init(&empty_bar[s], NCONS / 32);        // one arrival per consumer warp
    }
    mbar_init(accum_bar, NCONS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tma_prefetch_desc(&tmw);
  }
  __syncthreads();

  if (threadIdx.x >= NCONS) {
    // ---------------- producers ----------------
    // Lane mapping: 8 consecutive lanes fetch the 8 x 16 B chunks of ONE gathered row, so a warp-wide cp.async touches
    // 4 rows x 128 B (4 L1 wavefronts) instead of 32 different rows (32 wavefronts: the round-1a L1TEX bottleneck).
    // Producer t owns chunk (t & 7) of rows (t >> 3) + 16 i, i = 0..7.
    const int t = threadIdx.x - NCONS;
    const int sub = t & 7, rgrp = t >> 3;
    const uint32_t sw = (uint32_t)(rgrp & 7);
    const uint32_t a_thread_off = (uint32_t)((rgrp >> 3) * 1024 + (rgrp & 7) * 128) + ((sub ^ sw) << 4);
    int it = 0, kcount = 0;
    const int my_row = tile * TC_M + t;
    // the neighbour index of the NEXT offset is loaded while the stages of the current one are in flight
    int v_next = (mask && my_row < n_out) ? nbr[(long long)(__ffs(mask) - 1) * n_out + my_row] : -1;
    for (uint32_t mk = mask; mk; mk &= mk - 1, ++kcount) {
      const int k = __ffs(mk) - 1;
      int* idx_buf = idx_s[kcount & 1];
      idx_buf[t] = v_next;
      asm volatile("bar.sync 1, %0;" ::"n"(NPROD) : "memory");     // producers only
      {
        const uint32_t rest = mk & (mk - 1);
        v_next = (rest && my_row < n_out) ? nbr[(long long)(__ffs(rest) - 1) * n_out + my_row] : -1;
      }
      int src[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) src[i] = idx_buf[rgrp + 16 * i];
      for (int c = 0; c < nchunk; ++c, ++it) {
        const int s = it % STAGES;
        if (it >= STAGES) mbar_wait(&empty_bar[s], ((it / STAGES) - 1) & 1);
        const uint32_t stage_base = smem_u32(smem + s * STAGE_BYTES);
        if (t == 0) {        // the filter tile of this stage: one (B_MN: N_TILE / 64) tiled TMA box(es)
          mbar_expect_tx(&full_bar[s], B_STAGE_BYTES);
          const uint32_t b_base = stage_base + A_BYTES;
          if (B_MN) {        // stored kernel (K*cin rows, cout columns): 64 reduction rows x 64 columns per box
#pragma unroll
            for (int a = 0; a < N_TILE / 64; ++a) tma_load_2d(&tmw, &full_bar[s], b_base + a * 8192, n0 + a * 64, k * cin + c * TC_BK);
          } else {           // (K*cout rows, cin columns): N_TILE output rows x 64 reduction columns
            tma_load_2d(&tmw, &full_bar[s], b_base, c * TC_BK, k * cout + n0);
          }
        }
        const uint32_t a_base = stage_base + a_thread_off;
#pragma unroll
        for (int i = 0; i < 8; ++i)
          cp_async16_ca(a_base + i * 2048, x + (long long)(src[i] >= 0 ? src[i] : 0) * cin + c * TC_BK + sub * 8,
                        src[i] >= 0 ? 16 : 0);
        cp_async_commit();
        if (it >= LAG) {
          cp_async_wait<LAG>();
          fence_proxy_async();
          mbar_arrive(&full_bar[(it - LAG) % STAGES]);
        }
      }
    }
    // drain the last LAG stages
    cp_async_wait<0>();
    fence_proxy_async();
    for (int d = (total > LAG ? total - LAG : 0); d < total; ++d) mbar_arrive(&full_bar[d % STAGES]);

    // ---------------- epilogue ----------------
    const int row = tile * TC_M + t;                 // accumulator-image row = row within the tile
    if (total > 0) mbar_wait(accum_bar, 0);
    __nv_bfloat16* yrow = y + (long long)row * cout + n0;
#pragma unroll 1
    for (int c0 = 0; c0 < N_TILE; c0 += 32) {
      uint32_t v[32];
      if (total > 0) {
        img_ld<32>(img, PITCH, t, c0, v);
      } else {
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = 0u;
      }
      if (row < n_out) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          uint4 o;
          o.x = pack_bf16(v[8 * q + 0], v[8 * q + 1]);
          o.y = pack_bf16(v[8 * q + 2], v[8 * q + 3]);
          o.z = pack_bf16(v[8 * q + 4], v[8 * q + 5]);
          o.w = pack_bf16(v[8 * q + 6], v[8 * q + 7]);
          *reinterpret_cast<uint4*>(yrow + c0 + 8 * q) = o;
        }
      }
    }
  } else if (total > 0) {
    // ---------------- consumers: warpgroup wg owns rows 64 wg .. 64 wg + 63 ----------------
    const int wg = threadIdx.x >> 7;
    float acc[N_TILE / 2];
    for (int it = 0; it < total; ++it) {
      const int s = it % STAGES;
      mbar_wait(&full_bar[s], (it / STAGES) & 1);
      const uint32_t a_addr = smem_u32(smem + s * STAGE_BYTES) + wg * 8192;
      const uint32_t b_addr = smem_u32(smem + s * STAGE_BYTES) + A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < TC_BK / 16; ++kk) {
        const uint64_t bd = B_MN ? make_desc(b_addr + kk * 2048, 8192, 1024) : make_desc(b_addr + kk * 32, 16, 1024);
        wgmma_bf16<N_TILE, 0, B_MN ? 1 : 0>(acc, make_desc(a_addr + kk * 32, 16, 1024), bd, it > 0 || kk > 0);
      }
      wgmma_commit();
      wgmma_wait<1>();                             // the group of stage it - 1 has retired: release its buffers
      if (it > 0 && (threadIdx.x & 31) == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
    }
    wgmma_wait<0>();
    acc_fence<N_TILE / 2>(acc);
    asm volatile("bar.sync 2, %0;" ::"n"(NCONS) : "memory");     // every wgmma has read its stage: the image may overwrite them
    acc_store<N_TILE>(acc, img, PITCH, wg * 64, threadIdx.x & 127);
    mbar_arrive(accum_bar);
  }
}

// ------------------------------------------------------------------------------------------------------------
// wgrad: dW[k] (Cin, Cout) += sum over pairs p of offset k of x[pin[p], :]^T dy[pout[p], :]
// CTA = (offset k, pair split) x (128-channel slice of Cin) x (N_TILE slice of Cout); reduction dim = pairs (64 / stage)
// ------------------------------------------------------------------------------------------------------------
template <int N_TILE, int STAGES>
__global__ void __launch_bounds__(384, 1)
spconv_tc_wgrad_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy,
                       const int* __restrict__ pair_in, const int* __restrict__ pair_out,
                       const int* __restrict__ k_offsets, float* __restrict__ part, int cin, int cout, int K,
                       int chunk_pairs) {
  constexpr int A_BYTES = 64 * 256;              // 64 pairs x 128 channels (2 M-atoms of 64 ch)
  constexpr int B_BYTES = 64 * N_TILE * 2;
  constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  constexpr int LAG = STAGES - 2;
  constexpr int NCONS = 256;
  constexpr int PITCH = N_TILE + 4;                 // floats; +4 keeps the per-lane float4 reads conflict-free
  static_assert(128 * PITCH * 4 <= STAGES * STAGE_BYTES, "the accumulator image reuses the stage buffers");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = (uint64_t*)(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* accum_bar = empty_bar + STAGES;

  // Work item = one chunk of `chunk_pairs` consecutive pairs of ONE offset (uniform work per CTA: no heavy-offset tail).
  // blockIdx.x enumerates chunks offset by offset; CTAs past the last chunk exit.
  int k = 0, chunk = blockIdx.x, p_beg = 0, p_end = 0;
  for (; k < K; ++k) {
    p_beg = k_offsets[k];
    p_end = k_offsets[k + 1];
    const int nch = (p_end - p_beg + chunk_pairs - 1) / chunk_pairs;
    if (chunk < nch) break;
    chunk -= nch;
  }
  if (k >= K) return;                              // uniform for the whole CTA
  const int ci0 = blockIdx.y * 128, co0 = blockIdx.z * N_TILE;
  const int s_beg = p_beg + chunk * chunk_pairs;
  const int s_end = min(p_end, s_beg + chunk_pairs);
  const int total = (s_end - s_beg + 63) / 64;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 128);
      mbar_init(&empty_bar[s], NCONS / 32);
    }
    mbar_init(accum_bar, NCONS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int a_ch = min(128, cin - ci0);            // valid channels of the A slice (64 or 128)

  if (threadIdx.x >= NCONS) {
    const int t = threadIdx.x - NCONS;
    const int warp = t >> 5;
    // thread t moves chunk (t & 15) of pair rows kk = (t >> 4) + 8 q, q = 0..7 (16 consecutive lanes = one 256 B row);
    // the pair indices of stage it+1 are fetched while the copies of stage it are in flight (index-load latency was
    // 55% of the stall samples in the round-1a profile).
    const int mc = t & 15, kk0 = t >> 4;
    const bool a_ok_ch = mc * 8 < a_ch;
    int ri[8], ro[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int p = s_beg + kk0 + 8 * q;
      ri[q] = p < s_end ? pair_in[p] : -1;
      ro[q] = p < s_end ? pair_out[p] : -1;
    }
    for (int it = 0; it < total; ++it) {
      const int s = it % STAGES;
      if (it >= STAGES) mbar_wait(&empty_bar[s], ((it / STAGES) - 1) & 1);
      const uint32_t a_base = smem_u32(smem + s * STAGE_BYTES);
      const uint32_t b_base = a_base + A_BYTES;
      // canonical MN-major SW128: atom(mi, kj) at mi*8192 + kj*1024, row kk%8, 16 B chunk index ^ row
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int kk = kk0 + 8 * q;
        const bool ok = ri[q] >= 0 && a_ok_ch;
        const uint32_t dst = a_base + (mc >> 3) * 8192 + (kk >> 3) * 1024 + (kk & 7) * 128 + (((mc & 7) ^ (kk & 7)) << 4);
        cp_async16_cg(dst, x + (long long)(ok ? ri[q] : 0) * cin + ci0 + mc * 8, ok ? 16 : 0);
      }
#pragma unroll
      for (int q = 0; q < N_TILE / 16; ++q) {
        const int idx = q * 128 + t;
        const int kk = idx / (N_TILE / 8), nc = idx % (N_TILE / 8);
        // N_TILE = 128: kk = kk0 + 8 q (register ro[q]); N_TILE = 64: kk = (t >> 3) + 16 q -> fetch through ro when aligned
        int rr;
        if (N_TILE == 128) {
          rr = ro[q];
        } else {
          const int p = s_beg + it * 64 + kk;
          rr = p < s_end ? pair_out[p] : -1;
        }
        const uint32_t dst = b_base + (nc >> 3) * 8192 + (kk >> 3) * 1024 + (kk & 7) * 128 + (((nc & 7) ^ (kk & 7)) << 4);
        cp_async16_cg(dst, dy + (long long)(rr >= 0 ? rr : 0) * cout + co0 + nc * 8, rr >= 0 ? 16 : 0);
      }
      cp_async_commit();
      if (it + 1 < total) {   // prefetch the next stage's pair indices
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const int p = s_beg + (it + 1) * 64 + kk0 + 8 * q;
          ri[q] = p < s_end ? pair_in[p] : -1;
          ro[q] = p < s_end ? pair_out[p] : -1;
        }
      }
      if (it >= LAG) {
        cp_async_wait<LAG>();
        fence_proxy_async();
        mbar_arrive(&full_bar[(it - LAG) % STAGES]);
      }
    }
    cp_async_wait<0>();
    fence_proxy_async();
    for (int d = (total > LAG ? total - LAG : 0); d < total; ++d) mbar_arrive(&full_bar[d % STAGES]);

    // epilogue: image row = ci (within the 128 slice), column = co. A warp stores whole 512-byte runs of one row of this
    // chunk's partial part[chunk] (cin, cout).
    mbar_wait(accum_bar, 0);
    const float* stg = reinterpret_cast<const float*>(smem);
    const int lane = t & 31;
    for (int rr = 0; rr < 32; ++rr) {
      const int r = warp * 32 + rr;
      const int ci = ci0 + r;
      if (ci >= cin) break;
      float* dwrow = part + ((long long)blockIdx.x * cin + ci) * cout + co0;
#pragma unroll
      for (int c = lane * 4; c < N_TILE; c += 128)
        *reinterpret_cast<float4*>(dwrow + c) = *reinterpret_cast<const float4*>(stg + r * PITCH + c);
    }
  } else {
    // consumers: warpgroup wg owns the 64 input channels ci0 + 64 wg .. (the second MN atom of the A tile)
    const int wg = threadIdx.x >> 7;
    float acc[N_TILE / 2];
    for (int it = 0; it < total; ++it) {
      const int s = it % STAGES;
      mbar_wait(&full_bar[s], (it / STAGES) & 1);
      const uint32_t a_addr = smem_u32(smem + s * STAGE_BYTES) + wg * 8192;
      const uint32_t b_addr = smem_u32(smem + s * STAGE_BYTES) + A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)             // 16 pairs per MMA = two 8-row K groups = 2048 B
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

// dw[k] += the partials of the chunks of offset k, in chunk order (chunks enumerate offset by offset, as in the kernel above).
// slot = 0: the add chain starts from dw[k]. slot = 1 (gradient slots): the chunks are added from +0 and the finished sum is
// added to dw[k] with one rounded add, as autograd's `grad += fresh`.
// Thread = 4 consecutive columns of one offset (cin * cout is a multiple of 4096; the scratch partials are 16-byte aligned):
// the 16-byte loads of 8 chunks are in flight before their in-order adds, one add chain per column.
__global__ void spconv_wgrad_reduce_kernel(const float* __restrict__ part, const int* __restrict__ k_offsets, float* __restrict__ dw,
                                           int cin, int cout, int K, int chunk_pairs, int slot) {
  constexpr int D = 8;
  const long long e = (blockIdx.x * (long long)blockDim.x + threadIdx.x) * 4;
  const long long per_k = (long long)cin * cout;
  if (e >= per_k * K) return;
  const int k = (int)(e / per_k);
  const long long j = e - k * per_k;
  int c0 = 0;
  for (int kk = 0; kk < k; ++kk) c0 += (k_offsets[kk + 1] - k_offsets[kk] + chunk_pairs - 1) / chunk_pairs;
  const int nch = (k_offsets[k + 1] - k_offsets[k] + chunk_pairs - 1) / chunk_pairs;
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  if (!slot) {
#pragma unroll
    for (int q = 0; q < 4; ++q) s[q] = dw[e + q];
  }
  const float4* src = reinterpret_cast<const float4*>(part + (long long)c0 * per_k + j);
  const long long stride = per_k / 4;
  for (int c = 0; c < nch; c += D) {
    float4 v[D];
#pragma unroll
    for (int u = 0; u < D; ++u)
      if (c + u < nch) v[u] = src[(c + u) * stride];
#pragma unroll
    for (int u = 0; u < D; ++u)
      if (c + u < nch) {
        s[0] = __fadd_rn(s[0], v[u].x);
        s[1] = __fadd_rn(s[1], v[u].y);
        s[2] = __fadd_rn(s[2], v[u].z);
        s[3] = __fadd_rn(s[3], v[u].w);
      }
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) dw[e + q] = slot ? __fadd_rn(dw[e + q], s[q]) : s[q];
}

template <int N_TILE, int STAGES, bool B_MN>
int launch_fwd(const void* x, const CUtensorMap& tmw, const int* nbr, const unsigned* masks, void* y, long long n_out, int cin,
               int cout, int K, cudaStream_t stream) {
  size_t smem = (size_t)STAGES * (A_STAGE_BYTES + N_TILE * 128) + 1024 + 256;
  auto kern = spconv_tc_fwd_kernel<N_TILE, STAGES, B_MN>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { esb_set_error("spconv_tc_fwd: smem attr: %s", cudaGetErrorString(e)); return ESB_ECUDA; }
  dim3 grid(esb_div_up(n_out, TC_M), cout / N_TILE);
  kern<<<grid, 384, smem, stream>>>((const __nv_bfloat16*)x, tmw, nbr, masks, (__nv_bfloat16*)y, (int)n_out, cin,
                                              cout, K);
  return ESB_OK;
}

template <int N_TILE, int STAGES>
int launch_wgrad(const void* x, const void* dy, const int* pin, const int* pout, const int* koff, float* part, int cin,
                 int cout, int K, int n_chunks, int chunk_pairs, cudaStream_t stream) {
  size_t smem = (size_t)STAGES * (64 * 256 + 64 * N_TILE * 2) + 1024 + 256;
  auto kern = spconv_tc_wgrad_kernel<N_TILE, STAGES>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { esb_set_error("spconv_tc_wgrad: smem attr: %s", cudaGetErrorString(e)); return ESB_ECUDA; }
  dim3 grid(n_chunks, esb_div_up(cin, 128), cout / N_TILE);
  kern<<<grid, 384, smem, stream>>>((const __nv_bfloat16*)x, (const __nv_bfloat16*)dy, pin, pout, koff, part, cin, cout, K,
                                    chunk_pairs);
  return ESB_OK;
}

}  // namespace

// masks: ceil(n/128) uint32, bit k set when any row of the tile has a neighbour through offset k
extern "C" int esb_kmap_tile_masks(const int* nbr, int K, long long n, unsigned* masks, void* stream) {
  ESB_CHECK_ARG(K >= 1 && K <= 32, "esb_kmap_tile_masks: K must be in [1,32]");
  if (n == 0) return ESB_OK;
  tile_mask_kernel<<<esb_div_up(n, TC_M), 128, 0, (cudaStream_t)stream>>>(nbr, K, (int)n, masks);
  ESB_CUDA_LAUNCH_CHECK("tile_mask_kernel");
  return ESB_OK;
}

// bf16 tensor-core forward / dgrad. x (n_in,cin) ; nbr (K,n_out) ; masks from esb_kmap_tile_masks(nbr) ; y (n_out,cout).
// w_layout 0: w is (K,cout,cin) (reduction dim contiguous) ; w_layout 1: w is (K,cin,cout) (output dim contiguous).
// Forward passes the stored kernel with w_layout 1; dgrad passes the same tensor with roles swapped and w_layout 0.
// Requires cin % 64 == 0 and cout % 64 == 0.
extern "C" int esb_spconv_tc_fwd(const void* x, const void* wt, const int* nbr, const unsigned* masks, void* y,
                                 long long n_out, int cin, int cout, int K, int w_layout, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  ESB_CHECK_ARG(cin % 64 == 0 && cout % 64 == 0 && cin > 0 && cout > 0, "esb_spconv_tc_fwd: channels must be multiples of 64");
  ESB_CHECK_ARG(K >= 1 && K <= 27, "esb_spconv_tc_fwd: K must be in [1,27]");
  if (n_out == 0) return ESB_OK;
  int rc;
  // wide tiles amortise the gather; narrow tiles when there are too few row tiles to fill the SMs
  const int sms = esb_sm_count();
  long long row_tiles = (n_out + TC_M - 1) / TC_M;
  const int n_tile = (cout % 256 == 0 && row_tiles * (cout / 256) >= sms) ? 256
                     : (cout % 128 == 0 && row_tiles * (cout / 128) >= sms) ? 128 : 64;
  CUtensorMap tmw;
  {
    unsigned long long dims[2], str[1];
    unsigned box[2];
    if (w_layout) {   // (K*cin rows, cout columns): 64 x 64 boxes
      dims[0] = (unsigned long long)cout; dims[1] = (unsigned long long)K * cin; str[0] = (unsigned long long)cout * 2;
      box[0] = 64; box[1] = 64;
    } else {          // (K*cout rows, cin columns): N_TILE rows x 64 columns
      dims[0] = (unsigned long long)cin; dims[1] = (unsigned long long)K * cout; str[0] = (unsigned long long)cin * 2;
      box[0] = 64; box[1] = (unsigned)n_tile;
    }
    rc = esb_tma_encode(&tmw, wt, 2, dims, str, box, nullptr, 128);
    if (rc != ESB_OK) return rc;
  }
#define ESB_TC_LAUNCH(NT, ST)                                                                       \
  (w_layout ? launch_fwd<NT, ST, true>(x, tmw, nbr, masks, y, n_out, cin, cout, K, stream)         \
            : launch_fwd<NT, ST, false>(x, tmw, nbr, masks, y, n_out, cin, cout, K, stream))
  if (n_tile == 256)
    rc = ESB_TC_LAUNCH(256, 4);
  else if (n_tile == 128)
    rc = ESB_TC_LAUNCH(128, 4);
  else
    rc = ESB_TC_LAUNCH(64, 4);
#undef ESB_TC_LAUNCH
  if (rc != ESB_OK) return rc;
  ESB_CUDA_LAUNCH_CHECK("spconv_tc_fwd_kernel");
  return ESB_OK;
}

namespace {
int spconv_tc_wgrad(const void* x, const void* dy, const int* pair_in, const int* pair_out, const int* k_offsets, float* dw,
                    long long n_pairs_hint, int cin, int cout, int K, int slot, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  ESB_CHECK_ARG(cin % 64 == 0 && cout % 64 == 0 && cin > 0 && cout > 0, "esb_spconv_tc_wgrad: channels must be multiples of 64");
  int n_tile = (cout % 128 == 0) ? 128 : 64;
  // n_pairs_hint is an upper bound of the pair count (K * n_out); aim at ~4 waves of 2 CTAs/SM over the channel tiles
  long long tiles = (long long)esb_div_up(cin, 128) * (cout / n_tile);
  long long target_chunks = (4LL * 2 * esb_sm_count() + tiles - 1) / tiles;
  long long cp = (n_pairs_hint / 2 + target_chunks - 1) / target_chunks;   // maps are ~40% dense: hint/2 ~ real pairs
  cp = (cp + 63) / 64 * 64;
  if (cp < 512) cp = 512;
  if (cp > 16384) cp = 16384;
  int chunk_pairs = (int)cp;
  int n_chunks = (int)(n_pairs_hint / chunk_pairs) + K + 1;               // upper bound; surplus CTAs exit immediately
  float* part = nullptr;
  ESB_CUDA_CALL(esb_scratch_alloc((void**)&part, sizeof(float) * n_chunks * cin * cout, stream));
  int rc = n_tile == 128
               ? launch_wgrad<128, 3>(x, dy, pair_in, pair_out, k_offsets, part, cin, cout, K, n_chunks, chunk_pairs, stream)
               : launch_wgrad<64, 4>(x, dy, pair_in, pair_out, k_offsets, part, cin, cout, K, n_chunks, chunk_pairs, stream);
  if (rc == ESB_OK) {
    spconv_wgrad_reduce_kernel<<<esb_div_up((long long)K * cin * cout / 4, 256), 256, 0, stream>>>(part, k_offsets, dw, cin, cout,
                                                                                                 K, chunk_pairs, slot);
  }
  ESB_CUDA_CALL(esb_scratch_free(part, stream));
  if (rc != ESB_OK) return rc;
  ESB_CUDA_LAUNCH_CHECK("spconv_tc_wgrad_kernel");
  return ESB_OK;
}
}  // namespace

// bf16 tensor-core wgrad over pair lists; dw (K,cin,cout) fp32 += the weight gradient (zeroed by the caller for a plain
// gradient). The pair chunks of an offset are added in chunk order, starting from dw: the result does not depend on
// scheduling.
extern "C" int esb_spconv_tc_wgrad(const void* x, const void* dy, const int* pair_in, const int* pair_out,
                                   const int* k_offsets, float* dw, long long n_pairs_hint, int cin, int cout, int K,
                                   void* stream) {
  return spconv_tc_wgrad(x, dy, pair_in, pair_out, k_offsets, dw, n_pairs_hint, cin, cout, K, 0, stream);
}

// The same into a gradient slot that may hold earlier backward passes: the chunks are added in chunk order from +0 and
// dw = dw + that sum, one rounded add per element (on a zeroed dw: the bits of esb_spconv_tc_wgrad).
extern "C" int esb_spconv_tc_wgrad_slot(const void* x, const void* dy, const int* pair_in, const int* pair_out,
                                        const int* k_offsets, float* dw, long long n_pairs_hint, int cin, int cout, int K,
                                        void* stream) {
  return spconv_tc_wgrad(x, dy, pair_in, pair_out, k_offsets, dw, n_pairs_hint, cin, cout, K, 1, stream);
}
