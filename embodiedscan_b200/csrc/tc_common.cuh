// esb200 — wgmma / mbarrier / cp.async / TMA primitives shared by every tensor-core kernel of the library
// (spconv_tc.cu, conv2d_tc.cu, conv_tma.cu, attn_tc.cu): ONE copy of the descriptor encoders.
#pragma once
#include <cuda.h>            // CUtensorMap (types only: the encoder is fetched through cudaGetDriverEntryPoint)
#include "common.cuh"
#include "wgmma.cuh"

namespace esb_tc {

constexpr int TC_M = 128;
constexpr int TC_BK = 64;                      // bf16 elements per smem row = 128 B = one swizzle row
constexpr int A_STAGE_BYTES = TC_M * 128;      // 16 KB

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void cp_async16_ca(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async16_cg(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// ---- warpgroup MMA (wgmma) ------------------------------------------------------------------------------------------
// A 128-row accumulator tile is owned by two consumer warpgroups, 64 rows each (wgmma is m64); the fragment lives in
// registers and is written once per tile to a row-major fp32 image in shared memory (acc_store), which the epilogue
// threads read row by row (img_ld) — thread = tile row, as the epilogues of these kernels are written.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void acc_fence(float* d) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int R>
__device__ __forceinline__ void acc_zero(float* d) {
#pragma unroll
  for (int i = 0; i < R; ++i) d[i] = 0.f;
}
// m64nN fp32 fragment layout: element i of thread t (0..127 in the warpgroup) is row 16*(t/32) + (t%32)/4 + 8*((i/2)%2),
// column 8*(i/4) + 2*(t%4) + i%2.
template <int N>
__device__ __forceinline__ void acc_store(const float* d, float* img, int pitch, int row0, int t) {
  const int r = row0 + 16 * (t >> 5) + ((t & 31) >> 2), c = 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    *reinterpret_cast<float2*>(img + r * pitch + 8 * j + c) = make_float2(d[4 * j], d[4 * j + 1]);
    *reinterpret_cast<float2*>(img + (r + 8) * pitch + 8 * j + c) = make_float2(d[4 * j + 2], d[4 * j + 3]);
  }
}
// NCOL consecutive fp32 of row `row` starting at column `col` (16-byte aligned) into v[0..NCOL-1]
template <int NCOL>
__device__ __forceinline__ void img_ld(const float* img, int pitch, int row, int col, uint32_t v[32]) {
#pragma unroll
  for (int q = 0; q < NCOL / 4; ++q) {
    const float4 f = *reinterpret_cast<const float4*>(img + row * pitch + col + 4 * q);
    v[4 * q] = __float_as_uint(f.x); v[4 * q + 1] = __float_as_uint(f.y);
    v[4 * q + 2] = __float_as_uint(f.z); v[4 * q + 3] = __float_as_uint(f.w);
  }
}
__device__ __forceinline__ uint32_t pack_bf16(uint32_t lo_f32_bits, uint32_t hi_f32_bits) {
  __nv_bfloat162 h = __floats2bfloat162_rn(__uint_as_float(lo_f32_bits), __uint_as_float(hi_f32_bits));
  return *reinterpret_cast<uint32_t*>(&h);
}

// ---- shared-memory matrix descriptor (wgmma): start>>4 | LBO>>4 <<16 | SBO>>4 <<32 | layout type <<62 ----------------
constexpr uint32_t SW128 = 1, SW64 = 2, SW32 = 3;     // layout types: 128B / 64B / 32B swizzle
__device__ __forceinline__ uint64_t make_desc_sw(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout_type) {
  return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32) |
         ((uint64_t)layout_type << 62);
}
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return make_desc_sw(smem_addr, lbo_bytes, sbo_bytes, SW128);
}
// layout type of a row of `row_bytes` bytes (32 / 64 / 128): one swizzle span per row
__host__ __device__ __forceinline__ uint32_t mma_layout_of(int row_bytes) { return row_bytes >= 128 ? SW128 : row_bytes == 64 ? SW64 : SW32; }

// ---- TMA (cp.async.bulk.tensor) -------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* m, uint64_t* bar, uint32_t dst, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(dst), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap* m, uint64_t* bar, uint32_t dst, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
               ::"r"(dst), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* m, uint64_t* bar, uint32_t dst, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
               ::"r"(dst), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_5d(const CUtensorMap* m, uint64_t* bar, uint32_t dst, int c0, int c1, int c2, int c3,
                                            int c4) {
  asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
               ::"r"(dst), "l"(m), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(m), "r"(src), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(m), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2, int c3, int c4) {
  asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
               ::"l"(m), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

}  // namespace esb_tc

// ---- host side: tensor-map encoder (driver entry point, no libcuda link dependency) --------------------------------------
// Returns 0 on success. dims/strides innermost first; strides[i] = byte stride of dimension i+1; swizzle bytes 0/32/64/128.
int esb_tma_encode(CUtensorMap* out, const void* base, int rank, const unsigned long long* dims,
                   const unsigned long long* strides_bytes, const unsigned* box, const unsigned* elem_strides,
                   int swizzle_bytes);

