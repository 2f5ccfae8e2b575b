// esb200 — dense NHWC convolution as a persistent TMA + wgmma implicit GEMM (bf16 in, fp32 accumulate).
// The per-view image backbone of the hot path (SURVEY §8 row a5: mmdet.ResNet(depth=50, base_channels=16), called at
// embodiedscan/models/detectors/sparse_featfusion_single_stage.py:130-136; config
// configs/detection/mv-det3d_8xb4_embodiedscan-3d-284class-9dof.py:24-34) with the frozen BatchNorm folded into the
// weights and bias + residual + ReLU fused into the epilogue. The same kernel is the input gradient of every stride-1
// convolution (flipped taps, weights read as the MN-major B operand: no transposed copy of the filter exists).
//
// GEMM view: M = output pixels, N = output channels, reduction = (filter tap, input channel).
//   * A CTA is persistent: it walks output tiles  (TN images x TH rows x TW columns <= 128 pixels) x (N_TILE channels).
//   * A operand: for every filter tap ONE tiled TMA load of the box {bc channels, TW, TH, TN} of the NHWC activation tensor
//     at the tap's spatial offset. Zero padding = TMA out-of-bounds fill; stride-2 convolutions use the tensor map's element
//     strides. The box lands in shared memory as the K-major [pixel][channel] tile wgmma reads; thin layers (16 / 32
//     channels) use the 32B / 64B swizzle modes and several taps share one pipeline stage.
//   * B operand: 2-D TMA box of the OHWI filter matrix (row = output channel, columns = (tap, input channel)).
//   * Two consumer warpgroups issue wgmma (m64, N=N_TILE, K=16), 64 tile rows each, accumulating in registers; at the end of
//     a tile they write the accumulator to a shared-memory image, so the epilogue of tile i overlaps the loads and MMAs of
//     tile i+1 (the registers are the second accumulator buffer).
//   * Epilogue warps: image row -> + bias (+ residual) (ReLU) -> bf16 -> swizzled shared tile -> TMA store (the store
//     clips partial tiles; no per-thread global stores).
// Thread roles: 0..255 = consumer warpgroups, 256..287 = TMA producer warp, 288..415 = epilogue (thread = tile row).
//
// Roofline: HBM. Algorithmic bytes = (N*H*W*Cin + N*Ho*Wo*Cout [+ residual]) * 2 + kh*kw*Cin*Cout*2 per launch.
#include "tc_common.cuh"

using namespace esb_tc;

namespace {

struct ConvGeom {
  int tiles_w, tiles_h, tiles_d, tiles_n, n_blocks;   // tile grid; n_blocks = Cout / N_TILE
  int TW, TH, TD, TN;                        // output pixels per tile along w, h, d, image (2-D convolutions: d = 1)
  int Wo, Ho, Do, N;                         // output extent
  int stride;                                // spacing of the A-box origin per output pixel (element strides of the tensor map)
  int cin, bc, nchunk, group;                // reduction channels per tap, channels per sub-tile, cin / bc, sub-tiles per stage
  int cout, relu;
  int stages;
  // filter taps as a table: input offset of the tap relative to (output pixel * stride) and its index in the stored filter.
  // forward: (kx - pad, ky - pad, tap); stride-1 dgrad: flipped taps; stride-2 dgrad: the taps of one output parity class.
  int ntaps;
  short tap_dx[27], tap_dy[27], tap_dz[27], tap_w[27];
};

constexpr int EPI_THREADS = 128;
constexpr int NCONS = 256;                          // two consumer warpgroups
constexpr int PROD0 = NCONS, EPI0 = NCONS + 32;     // first thread of the producer warp / of the epilogue warps
constexpr int THREADS = EPI0 + EPI_THREADS;

__device__ __forceinline__ uint32_t swz(uint32_t off, uint32_t mask) { return off ^ (((off >> 7) & mask) << 4); }

template <int N_TILE, bool B_MN>
__global__ void __launch_bounds__(THREADS, 1)
conv_tma_kernel(const __grid_constant__ CUtensorMap tmx, const __grid_constant__ CUtensorMap tmw,
                const __grid_constant__ CUtensorMap tmy, const float* __restrict__ bias,
                const __nv_bfloat16* __restrict__ res, const ConvGeom g) {
  constexpr int CB_COLS = N_TILE < 64 ? N_TILE : 64;          // columns per TMA store (one swizzle span)
  constexpr int CB_ROW_BYTES = CB_COLS * 2;
  constexpr int CB_BYTES = 128 * CB_ROW_BYTES;
  constexpr uint32_t CB_MASK = CB_ROW_BYTES == 128 ? 7u : CB_ROW_BYTES == 64 ? 3u : 1u;
  constexpr int B_STAGE_BYTES = N_TILE * 128;
  constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  constexpr int PITCH = N_TILE + 4;                            // floats per accumulator-image row

  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const int STAGES = g.stages;
  uint8_t* cbuf = smem + STAGES * STAGE_BYTES;                 // 2 x CB_BYTES, 1024-aligned (STAGE_BYTES % 1024 == 0)
  float* img = reinterpret_cast<float*>(cbuf + 2 * CB_BYTES);  // 128 x PITCH accumulator image
  uint64_t* full_bar = (uint64_t*)(img + 128 * PITCH);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* tfull_bar = empty_bar + STAGES;                    // image written (consumers -> epilogue)
  uint64_t* tempty_bar = tfull_bar + 1;                        // image drained (epilogue -> consumers)

  const int lane = threadIdx.x & 31;
  const int n_sub = g.ntaps * g.nchunk;                        // sub-tiles (tap, channel chunk) per output tile
  const int n_it = (n_sub + g.group - 1) / g.group;            // pipeline stages per output tile
  const int bcb = g.bc * 2;                                    // bytes per sub-tile row
  const int rows_box = g.TW * g.TH * g.TD * g.TN;
  const uint32_t a_sub_bytes = (uint32_t)rows_box * bcb;       // what TMA delivers (<= 128 rows)
  const uint32_t b_sub_bytes = (uint32_t)N_TILE * bcb;
  const int n_work = g.tiles_w * g.tiles_h * g.tiles_d * g.tiles_n * g.n_blocks;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], NCONS / 32);
    }
    mbar_init(tfull_bar, NCONS);
    mbar_init(tempty_bar, EPI_THREADS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tma_prefetch_desc(&tmx);
    tma_prefetch_desc(&tmw);
    tma_prefetch_desc(&tmy);
  }
  __syncthreads();

  if (threadIdx.x >= PROD0 && threadIdx.x < EPI0) {
    // ------------------------------------------------ TMA producer ------------------------------------------------
    if (lane == 0) {
      uint32_t it = 0;
      for (int work = blockIdx.x; work < n_work; work += gridDim.x) {
        int t = work;
        const int tw = t % g.tiles_w; t /= g.tiles_w;
        const int th = t % g.tiles_h; t /= g.tiles_h;
        const int td = t % g.tiles_d; t /= g.tiles_d;
        const int tn = t % g.tiles_n; t /= g.tiles_n;
        const int n0 = t * N_TILE;
        const int x0 = tw * g.TW * g.stride, y0 = th * g.TH * g.stride, z0 = td * g.TD * g.stride, img0 = tn * g.TN;
        for (int i = 0; i < n_it; ++i, ++it) {
          const int s = it % STAGES;
          mbar_wait(&empty_bar[s], ((it / STAGES) & 1) ^ 1);
          const int q0 = i * g.group;
          const int cnt = min(g.group, n_sub - q0);
          mbar_expect_tx(&full_bar[s], (uint32_t)cnt * (a_sub_bytes + b_sub_bytes));
          const uint32_t a_base = smem_u32(smem + s * STAGE_BYTES);
          const uint32_t b_base = a_base + A_STAGE_BYTES;
          for (int j = 0; j < cnt; ++j) {
            const int q = q0 + j;
            const int tap = q / g.nchunk, ch = (q - tap * g.nchunk) * g.bc;
            tma_load_5d(&tmx, &full_bar[s], a_base + j * (128 * bcb), ch, x0 + g.tap_dx[tap], y0 + g.tap_dy[tap],
                        z0 + g.tap_dz[tap], img0);
            const int wtap = g.tap_w[tap];
            if (!B_MN) {           // rows = output channels, columns = (tap, input channel): K-major B
              tma_load_2d(&tmw, &full_bar[s], b_base + j * b_sub_bytes, wtap * g.cin + ch, n0);
            } else {               // rows = reduction channels, columns = (tap, output channel): MN-major B, <= 64 columns per box
              constexpr int NA = N_TILE < 64 ? N_TILE : 64;
#pragma unroll
              for (int a = 0; a < N_TILE / NA; ++a)
                tma_load_2d(&tmw, &full_bar[s], b_base + j * b_sub_bytes + a * (g.bc * NA * 2), wtap * g.cout + n0 + a * NA, ch);
            }
          }
        }
      }
    }
  } else if (threadIdx.x < NCONS) {
    // ------------------------------------------------ consumers ------------------------------------------------
    const int wg = threadIdx.x >> 7;                           // tile rows 64 wg .. 64 wg + 63
    const uint32_t a_layout = mma_layout_of(bcb);
    uint32_t it = 0, tcount = 0;
    float acc[N_TILE / 2];
    for (int work = blockIdx.x; work < n_work; work += gridDim.x, ++tcount) {
      int prev = -1;
      for (int i = 0; i < n_it; ++i, ++it) {
        const int s = it % STAGES;
        mbar_wait(&full_bar[s], (it / STAGES) & 1);
        const uint32_t a_base = smem_u32(smem + s * STAGE_BYTES);
        const uint32_t b_base = a_base + A_STAGE_BYTES;
        const int cnt = min(g.group, n_sub - i * g.group);
        wgmma_fence();
        for (int j = 0; j < cnt; ++j) {
          const uint32_t a_sub = a_base + j * (128 * bcb) + wg * (64 * bcb), b_sub = b_base + j * b_sub_bytes;
          for (int kk = 0; kk < g.bc / 16; ++kk) {
            const uint64_t ad = make_desc_sw(a_sub + kk * 32, 16, 8 * bcb, a_layout);
            const int accumulate = i > 0 || j > 0 || kk > 0;
            if (!B_MN) {
              wgmma_bf16<N_TILE, 0, 0>(acc, ad, make_desc_sw(b_sub + kk * 32, 16, 8 * bcb, a_layout), accumulate);
            } else {
              constexpr int NAB = (N_TILE < 64 ? N_TILE : 64) * 2;     // bytes per MN-major row (one atom of columns)
              wgmma_bf16<N_TILE, 0, 1>(acc, ad, make_desc_sw(b_sub + kk * 16 * NAB, g.bc * NAB, 8 * NAB, mma_layout_of(NAB)),
                                       accumulate);
            }
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                                       // the group of the previous stage has retired
        if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
        prev = s;
      }
      wgmma_wait<0>();
      acc_fence<N_TILE / 2>(acc);
      if (lane == 0) mbar_arrive(&empty_bar[prev]);
      mbar_wait(tempty_bar, (tcount & 1) ^ 1);                 // the epilogue has drained the previous tile's image
      acc_store<N_TILE>(acc, img, PITCH, wg * 64, threadIdx.x & 127);
      mbar_arrive(tfull_bar);
    }
  } else {
    // ------------------------------------------------ epilogue ------------------------------------------------
    const int et = threadIdx.x - EPI0;                         // 0..127
    const int m = et;                                          // tile row = image row
    uint32_t tcount = 0, cb = 0;
    for (int work = blockIdx.x; work < n_work; work += gridDim.x, ++tcount) {
      int t = work;
      const int tw = t % g.tiles_w; t /= g.tiles_w;
      const int th = t % g.tiles_h; t /= g.tiles_h;
      const int td = t % g.tiles_d; t /= g.tiles_d;
      const int tn = t % g.tiles_n; t /= g.tiles_n;
      const int n0 = t * N_TILE;
      const int ow0 = tw * g.TW, oh0 = th * g.TH, od0 = td * g.TD, img0 = tn * g.TN;
      // this thread's output pixel
      int mr = m;
      const int mw = mr % g.TW; mr /= g.TW;
      const int mh = mr % g.TH; mr /= g.TH;
      const int md = mr % g.TD;
      const int mi = mr / g.TD;
      const bool valid = m < rows_box && img0 + mi < g.N && od0 + md < g.Do && oh0 + mh < g.Ho && ow0 + mw < g.Wo;
      const long long pix = (((long long)(img0 + mi) * g.Do + (od0 + md)) * g.Ho + (oh0 + mh)) * g.Wo + (ow0 + mw);
      mbar_wait(tfull_bar, tcount & 1);
#pragma unroll 1
      for (int c0 = 0; c0 < N_TILE; c0 += CB_COLS, cb ^= 1) {
        if (et == 0) tma_store_wait_read<1>();                 // the store issued from this buffer two chunks ago has read it
        asm volatile("bar.sync 1, 128;" ::: "memory");
        uint8_t* crow = cbuf + cb * CB_BYTES;
#pragma unroll 1
        for (int c1 = 0; c1 < CB_COLS; c1 += 32) {
          constexpr int W32 = CB_COLS < 32 ? CB_COLS : 32;     // columns handled per image read (16 or 32)
          uint32_t v[32];
          img_ld<W32>(img, PITCH, m, c0 + c1, v);
          if (c0 + CB_COLS >= N_TILE && c1 + 32 >= CB_COLS) mbar_arrive(tempty_bar);   // last read of this tile's image
#pragma unroll
          for (int q = 0; q < W32 / 8; ++q) {
            const int c = n0 + c0 + c1 + 8 * q;
            float f[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) f[e] = __uint_as_float(v[8 * q + e]);
            if (bias != nullptr) {
              const float4 b0 = *reinterpret_cast<const float4*>(bias + c);
              const float4 b1 = *reinterpret_cast<const float4*>(bias + c + 4);
              f[0] += b0.x; f[1] += b0.y; f[2] += b0.z; f[3] += b0.w;
              f[4] += b1.x; f[5] += b1.y; f[6] += b1.z; f[7] += b1.w;
            }
            if (res != nullptr && valid) {
              const uint4 r = *reinterpret_cast<const uint4*>(res + pix * g.cout + c);
              const __nv_bfloat162* rp = reinterpret_cast<const __nv_bfloat162*>(&r);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float2 rf = __bfloat1622float2(rp[e]);
                f[2 * e] += rf.x;
                f[2 * e + 1] += rf.y;
              }
            }
            if (g.relu) {
#pragma unroll
              for (int e = 0; e < 8; ++e) f[e] = fmaxf(f[e], 0.f);
            }
            uint4 o;
            o.x = pack_bf16(__float_as_uint(f[0]), __float_as_uint(f[1]));
            o.y = pack_bf16(__float_as_uint(f[2]), __float_as_uint(f[3]));
            o.z = pack_bf16(__float_as_uint(f[4]), __float_as_uint(f[5]));
            o.w = pack_bf16(__float_as_uint(f[6]), __float_as_uint(f[7]));
            const uint32_t off = swz((uint32_t)(m * CB_ROW_BYTES + (c1 + 8 * q) * 2), CB_MASK);
            *reinterpret_cast<uint4*>(crow + off) = o;
          }
        }
        fence_proxy_async();                                   // generic-proxy writes -> visible to the TMA store
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (et == 0) {
          tma_store_5d(&tmy, smem_u32(crow), n0 + c0, ow0, oh0, od0, img0);
          tma_store_commit();
        }
      }
    }
    if (et == 0) tma_store_wait<0>();                          // global writes complete before the kernel ends
  }
}

// pick the output-tile extent (TW x TH x TD x TN <= 128 pixels) that wastes the fewest MMA rows over the whole output
void choose_tile(int Wo, int Ho, int Do, int N, int* TW, int* TH, int* TD, int* TN) {
  double best = -1.0;
  *TW = *TH = *TD = *TN = 1;
  for (int tw = 1; tw <= Wo && tw <= 128; ++tw)
    for (int th = 1; th <= Ho && tw * th <= 128; ++th)
      for (int td = 1; td <= Do && tw * th * td <= 128; ++td) {
        int tn = 1;
        if (tw == Wo && th == Ho && td == Do) tn = 128 / (tw * th * td) < N ? 128 / (tw * th * td) : N;
        const long long tiles = (long long)esb_div_up(Wo, tw) * esb_div_up(Ho, th) * esb_div_up(Do, td) * esb_div_up(N, tn);
        const double eff = (double)Wo * Ho * Do * N / ((double)tiles * 128.0) + 1e-6 * tw;   // ties: longer contiguous rows
        if (eff > best) { best = eff; *TW = tw; *TH = th; *TD = td; *TN = tn; }
      }
}

template <int N_TILE, bool B_MN>
int launch(const CUtensorMap& tmx, const CUtensorMap& tmw, const CUtensorMap& tmy, const float* bias, const void* res,
           ConvGeom g, cudaStream_t stream) {
  constexpr int CB_COLS = N_TILE < 64 ? N_TILE : 64;
  constexpr int STAGE_BYTES = A_STAGE_BYTES + N_TILE * 128;
  constexpr int IMG_BYTES = 128 * (N_TILE + 4) * 4;
  // the stage ring runs ahead ACROSS output tiles (persistent CTA), so its depth is set by shared memory, not by the filter:
  // one CTA per SM, whatever the 227 KB per block leave after the accumulator image and the two store buffers
  const int budget = 227 * 1024 - IMG_BYTES - 2 * 128 * CB_COLS * 2 - 2048;
  int stages = budget / STAGE_BYTES;
  stages = stages > 6 ? 6 : stages < 2 ? 2 : stages;
  g.stages = stages;
  const size_t smem = (size_t)stages * STAGE_BYTES + 2 * 128 * CB_COLS * 2 + IMG_BYTES + (2 * stages + 2) * 8 + 1024;
  auto kern = conv_tma_kernel<N_TILE, B_MN>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { esb_set_error("conv_tma: smem attr (%zu B): %s", smem, cudaGetErrorString(e)); return ESB_ECUDA; }
  const long long n_work = (long long)g.tiles_w * g.tiles_h * g.tiles_d * g.tiles_n * g.n_blocks;
  long long grid = esb_sm_count();
  if (grid > n_work) grid = n_work;
  kern<<<(unsigned)grid, THREADS, smem, stream>>>(tmx, tmw, tmy, bias, (const __nv_bfloat16*)res, g);
  return ESB_OK;
}

// One launch: `in` (N, Di, Hi, Wi, Ci) -> `out` viewed as (N, Do, Ho, Wo, Co) with the given byte strides (a parity class of dx
// is a strided view), taps from the table in `g`. taps_total = taps of the stored filter (extent of its tensor map).
// 2-D convolutions are the Di = Do = 1 case of the same rank-5 tensor maps.
int conv_tma_run(const void* in, const void* w, const float* bias, const void* res, void* out, int N, int Di, int Hi, int Wi,
                 int Ci, int Do, int Ho, int Wo, int Co, int taps_total, int stride, int relu, bool dgrad, ConvGeom g,
                 unsigned long long out_sw, unsigned long long out_sh, unsigned long long out_sd, unsigned long long out_sn,
                 cudaStream_t stream) {
  g.Wo = Wo; g.Ho = Ho; g.Do = Do; g.N = N;
  g.stride = stride;
  g.cin = Ci; g.cout = Co; g.relu = relu;
  g.bc = Ci >= 64 ? 64 : Ci;
  g.nchunk = Ci / g.bc;
  g.group = 64 / g.bc;
  choose_tile(Wo, Ho, Do, N, &g.TW, &g.TH, &g.TD, &g.TN);
  g.tiles_w = esb_div_up(Wo, g.TW); g.tiles_h = esb_div_up(Ho, g.TH); g.tiles_d = esb_div_up(Do, g.TD);
  g.tiles_n = esb_div_up(N, g.TN);
  const int n_tile = Co >= 128 ? 128 : Co;                     // 64 accumulator registers per consumer thread at most
  g.n_blocks = Co / n_tile;
  const int sd = Di > 1 ? stride : 1;          // a depth-1 (2-D) problem has nothing to stride over
  CUtensorMap tmx, tmw, tmy;
  {   // activations: {C, W, H, D, N}, box {bc, span_w, span_h, span_d, TN}, element strides {1, s, s, s, 1}
    unsigned long long dims[5] = {(unsigned long long)Ci, (unsigned long long)Wi, (unsigned long long)Hi, (unsigned long long)Di,
                                  (unsigned long long)N};
    unsigned long long str[4] = {(unsigned long long)Ci * 2, (unsigned long long)Wi * Ci * 2, (unsigned long long)Hi * Wi * Ci * 2,
                                 (unsigned long long)Di * Hi * Wi * Ci * 2};
    unsigned box[5] = {(unsigned)g.bc, (unsigned)((g.TW - 1) * stride + 1), (unsigned)((g.TH - 1) * stride + 1),
                       (unsigned)((g.TD - 1) * sd + 1), (unsigned)g.TN};
    unsigned es[5] = {1, (unsigned)stride, (unsigned)stride, (unsigned)sd, 1};
    int rc = esb_tma_encode(&tmx, in, 5, dims, str, box, es, g.bc * 2 >= 128 ? 128 : g.bc * 2);
    if (rc != ESB_OK) return rc;
  }
  if (!dgrad) {   // O..I (Co, taps*Ci): box {bc, n_tile}
    unsigned long long dims[2] = {(unsigned long long)taps_total * Ci, (unsigned long long)Co};
    unsigned long long str[1] = {(unsigned long long)taps_total * Ci * 2};
    unsigned box[2] = {(unsigned)g.bc, (unsigned)n_tile};
    int rc = esb_tma_encode(&tmw, w, 2, dims, str, box, nullptr, g.bc * 2 >= 128 ? 128 : g.bc * 2);
    if (rc != ESB_OK) return rc;
  } else {        // the forward filter (rows = its output channels = this GEMM's reduction) read as the MN-major B operand
    const int na = n_tile < 64 ? n_tile : 64;
    unsigned long long dims[2] = {(unsigned long long)taps_total * Co, (unsigned long long)Ci};
    unsigned long long str[1] = {(unsigned long long)taps_total * Co * 2};
    unsigned box[2] = {(unsigned)na, (unsigned)g.bc};
    int rc = esb_tma_encode(&tmw, w, 2, dims, str, box, nullptr, na * 2);
    if (rc != ESB_OK) return rc;
  }
  {   // output store: {Co, Wo, Ho, Do, N} with the caller's strides, box {<=64 channels, TW, TH, TD, TN}
    const int cb = n_tile < 64 ? n_tile : 64;
    unsigned long long dims[5] = {(unsigned long long)Co, (unsigned long long)Wo, (unsigned long long)Ho, (unsigned long long)Do,
                                  (unsigned long long)N};
    unsigned long long str[4] = {out_sw, out_sh, out_sd, out_sn};
    unsigned box[5] = {(unsigned)cb, (unsigned)g.TW, (unsigned)g.TH, (unsigned)g.TD, (unsigned)g.TN};
    int rc = esb_tma_encode(&tmy, out, 5, dims, str, box, nullptr, cb * 2);
    if (rc != ESB_OK) return rc;
  }
  int rc;
#define ESB_CT(NT)                                                                       \
  (dgrad ? launch<NT, true>(tmx, tmw, tmy, bias, res, g, stream) : launch<NT, false>(tmx, tmw, tmy, bias, res, g, stream))
  switch (n_tile) {
    case 16: rc = ESB_CT(16); break;
    case 32: rc = ESB_CT(32); break;
    case 64: rc = ESB_CT(64); break;
    case 128: rc = ESB_CT(128); break;
    default: esb_set_error("conv_tma: unsupported output channel count %d (16, 32, 64 or a multiple of 128)", Co); return ESB_EINVAL;
  }
#undef ESB_CT
  if (rc != ESB_OK) return rc;
  ESB_CUDA_LAUNCH_CHECK("conv_tma_kernel");
  return ESB_OK;
}

bool channels_ok(int c) { return c == 16 || c == 32 || (c >= 64 && c % 64 == 0); }

}  // namespace

namespace {

// forward of a (kd, kh, kw) convolution on (n, D, H, W, cin); kd = D = 1 for the 2-D entry point
int conv_fwd_any(const char* who, const void* x, const void* w, const float* bias, const void* residual, void* y, int n, int D,
                 int H, int W, int cin, int cout, int kd, int kh, int kw, int stride, int pad, int relu, cudaStream_t stream) {
  const int pd = kd > 1 ? pad : 0;
  if (!(channels_ok(cin) && channels_ok(cout))) { esb_set_error("%s: channels must be 16, 32 or a multiple of 64", who); return ESB_EINVAL; }
  if (!(cout <= 256 ? (cout & (cout - 1)) == 0 : cout % 256 == 0)) {
    esb_set_error("%s: Cout must be a power of two <= 256 or a multiple of 256", who);
    return ESB_EINVAL;
  }
  if (!(kd >= 1 && kh >= 1 && kw >= 1 && kd * kh * kw <= 27 && stride >= 1 && stride <= 8 && pad >= 0)) {
    esb_set_error("%s: bad filter geometry (at most 27 taps)", who);
    return ESB_EINVAL;
  }
  const int Do = (D + 2 * pd - kd) / (D > 1 ? stride : 1) + 1, Ho = (H + 2 * pad - kh) / stride + 1, Wo = (W + 2 * pad - kw) / stride + 1;
  if (Do <= 0 || Ho <= 0 || Wo <= 0) { esb_set_error("%s: empty output", who); return ESB_EINVAL; }
  if (n == 0) return ESB_OK;
  ConvGeom g{};
  for (int kz = 0; kz < kd; ++kz)
    for (int ky = 0; ky < kh; ++ky)
      for (int kx = 0; kx < kw; ++kx) {
        g.tap_dx[g.ntaps] = (short)(kx - pad);
        g.tap_dy[g.ntaps] = (short)(ky - pad);
        g.tap_dz[g.ntaps] = (short)(kz - pd);
        g.tap_w[g.ntaps] = (short)g.ntaps;
        ++g.ntaps;
      }
  const unsigned long long px = (unsigned long long)cout * 2;
  return conv_tma_run(x, w, bias, residual, y, n, D, H, W, cin, Do, Ho, Wo, cout, kd * kh * kw, stride, relu, false, g, px,
                      (unsigned long long)Wo * px, (unsigned long long)Ho * Wo * px, (unsigned long long)Do * Ho * Wo * px, stream);
}

// input gradient, stride 1 or 2: one launch per parity class of dx (see esb_conv2d_tma_dgrad)
int conv_dgrad_any(const char* who, const void* dy, const void* w, void* dx, int n, int D, int H, int W, int cin, int cout, int kd,
                   int kh, int kw, int stride, int pad, cudaStream_t stream) {
  const int pd = kd > 1 ? pad : 0, sd = D > 1 ? stride : 1;
  if (!(channels_ok(cin) && channels_ok(cout))) { esb_set_error("%s: channels must be 16, 32 or a multiple of 64", who); return ESB_EINVAL; }
  if (!(cin <= 256 ? (cin & (cin - 1)) == 0 : cin % 256 == 0)) {
    esb_set_error("%s: Cin must be a power of two <= 256 or a multiple of 256", who);
    return ESB_EINVAL;
  }
  if (!(kd >= 1 && kh >= 1 && kw >= 1 && kd * kh * kw <= 27 && pad >= 0 && pad < kh && pad < kw && (stride == 1 || stride == 2))) {
    esb_set_error("%s: bad filter geometry", who);
    return ESB_EINVAL;
  }
  const int Do = (D + 2 * pd - kd) / sd + 1, Ho = (H + 2 * pad - kh) / stride + 1, Wo = (W + 2 * pad - kw) / stride + 1;
  if (Do <= 0 || Ho <= 0 || Wo <= 0) { esb_set_error("%s: empty output", who); return ESB_EINVAL; }
  if (n == 0) return ESB_OK;
  const unsigned long long px = (unsigned long long)cin * 2, row = (unsigned long long)W * px, slab = (unsigned long long)H * row,
                           img = (unsigned long long)D * slab;
  if (stride == 2 && (kh < 2 || kw < 2 || (D > 1 && kd < 2)))   // a 1-wide filter leaves whole parity classes of dx untouched
    ESB_CUDA_CALL(cudaMemsetAsync(dx, 0, (size_t)n * img, stream));
  for (int pz = 0; pz < sd; ++pz)
    for (int ph = 0; ph < stride; ++ph)
      for (int pw = 0; pw < stride; ++pw) {
        const int Dc = (D - pz + sd - 1) / sd, Hc = (H - ph + stride - 1) / stride, Wc = (W - pw + stride - 1) / stride;
        if (Dc <= 0 || Hc <= 0 || Wc <= 0) continue;
        ConvGeom g{};
        for (int kz = 0; kz < kd; ++kz)
          for (int ky = 0; ky < kh; ++ky)
            for (int kx = 0; kx < kw; ++kx) {
              // dy pixel = (stride * i + n) / stride for class pixel i; only taps of matching parity contribute
              const int nz = pz + pd - kz, ny = ph + pad - ky, nx = pw + pad - kx;
              if (((nz % sd) + sd) % sd != 0 || ((ny % stride) + stride) % stride != 0 || ((nx % stride) + stride) % stride != 0) continue;
              g.tap_dx[g.ntaps] = (short)(nx >= 0 ? nx / stride : -((-nx) / stride));
              g.tap_dy[g.ntaps] = (short)(ny >= 0 ? ny / stride : -((-ny) / stride));
              g.tap_dz[g.ntaps] = (short)(nz >= 0 ? nz / sd : -((-nz) / sd));
              g.tap_w[g.ntaps] = (short)((kz * kh + ky) * kw + kx);
              ++g.ntaps;
            }
        if (g.ntaps == 0) continue;                             // no tap reaches this class: zeroed by the memset above
        uint8_t* base = (uint8_t*)dx + (unsigned long long)pz * slab + (unsigned long long)ph * row + (unsigned long long)pw * px;
        int rc = conv_tma_run(dy, w, nullptr, nullptr, base, n, Do, Ho, Wo, cout, Dc, Hc, Wc, cin, kd * kh * kw, 1, 0, true, g,
                              (unsigned long long)stride * px, (unsigned long long)stride * row, (unsigned long long)sd * slab, img,
                              stream);
        if (rc != ESB_OK) return rc;
      }
  return ESB_OK;
}

}  // namespace

// y (n,Ho,Wo,cout) = act(conv(x (n,H,W,cin), w_ohwi (cout,kh,kw,cin)) + bias + residual), NHWC bf16, fp32 accumulate.
// bias fp32 (cout) or NULL; residual bf16 (n,Ho,Wo,cout) or NULL. cin, cout in {16, 32, 64k}; cout <= 256 or a multiple of 256.
extern "C" int esb_conv2d_tma_fwd(const void* x, const void* w_ohwi, const float* bias, const void* residual, void* y,
                                  int n_img, int H, int W, int cin, int cout, int kh, int kw, int stride, int pad, int relu,
                                  void* stream_) {
  return conv_fwd_any("esb_conv2d_tma_fwd", x, w_ohwi, bias, residual, y, n_img, 1, H, W, cin, cout, 1, kh, kw, stride, pad, relu,
                      (cudaStream_t)stream_);
}

// The same kernel on (n, D, H, W, cin) volumes (rank-5 tensor maps): the dense Conv3d stack of the occupancy neck
// (embodiedscan/models/necks/imvoxel_neck.py:86-129). w_odhwi (cout, k, k, k, cin), NDHWC bf16.
extern "C" int esb_conv3d_tma_fwd(const void* x, const void* w_odhwi, const float* bias, const void* residual, void* y, int n,
                                  int D, int H, int W, int cin, int cout, int k, int stride, int pad, int relu, void* stream_) {
  return conv_fwd_any("esb_conv3d_tma_fwd", x, w_odhwi, bias, residual, y, n, D, H, W, cin, cout, k, k, k, stride, pad, relu,
                      (cudaStream_t)stream_);
}

// Input gradient of a convolution with stride 1 or 2: dx (n,H,W,cin) from dy (n,Ho,Wo,cout) and the forward filter w_ohwi as
// stored (read as the MN-major B operand). Stride 1: one launch with the taps flipped. Stride 2: dx splits into the four
// parity classes of (h, w); each class is a stride-1 convolution of dy with the taps of matching parity, stored through a
// tensor map whose strides skip every other pixel — every dx element is still written exactly once, no atomics, no memset
// except for classes no tap reaches (1x1 / stride 2).
extern "C" int esb_conv2d_tma_dgrad(const void* dy, const void* w_ohwi, void* dx, int n_img, int H, int W, int cin, int cout,
                                    int kh, int kw, int stride, int pad, void* stream_) {
  return conv_dgrad_any("esb_conv2d_tma_dgrad", dy, w_ohwi, dx, n_img, 1, H, W, cin, cout, 1, kh, kw, stride, pad,
                        (cudaStream_t)stream_);
}

extern "C" int esb_conv3d_tma_dgrad(const void* dy, const void* w_odhwi, void* dx, int n, int D, int H, int W, int cin, int cout,
                                    int k, int stride, int pad, void* stream_) {
  return conv_dgrad_any("esb_conv3d_tma_dgrad", dy, w_odhwi, dx, n, D, H, W, cin, cout, k, k, k, stride, pad,
                        (cudaStream_t)stream_);
}

// ------------------------------------------------------------------------------------------------------------
// The 7x7 / stride 2 / pad 3 stem on the 3-channel image (Cin = 3 cannot feed a 16-byte TMA box): the CTA stages the
// input patch of a 16 x 8 output tile in shared memory with coalesced loads, every thread lays out ITS pixel's 147-tap row
// as the K-major 128B-swizzled A operand (im2col in shared memory, never in HBM), the warpgroup issues ten wgmma
// (m64, N=16, K=16) per 64-row half against the filter resident in shared memory, writes the accumulator over the idle A tile,
// and every thread adds the folded-BN bias to ITS pixel, applies ReLU and stores 32 contiguous bytes.
// Persistent over tiles. Roofline: HBM (image in, 16-channel map out).
// ------------------------------------------------------------------------------------------------------------
namespace {

constexpr int ST_TW = 16, ST_TH = 8;                 // output tile
constexpr int ST_PW = 112, ST_PH = 2 * ST_TH + 5;    // patch: 112 bf16 per row (1 pad + 37 pixels x 3), 21 rows
constexpr int ST_K = 147, ST_KPAD = 160;             // 7*7*3 taps, padded to 10 x K16

__global__ void __launch_bounds__(128)
stem7x7_tc_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w, const float* __restrict__ bias,
                  __nv_bfloat16* __restrict__ y, int n_img, int H, int W, int Ho, int Wo, int relu) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* a_tile = smem;                                   // 3 chunks x (128 rows x 128 B) = 48 KB
  uint8_t* b_tile = smem + 3 * 16384;                       // 3 chunks x (16 rows x 128 B) = 6 KB
  __nv_bfloat16* patch = (__nv_bfloat16*)(b_tile + 3 * 2048);   // 21 x 112 bf16
  float* acc_img = reinterpret_cast<float*>(a_tile);          // 128 x 20 fp32 accumulator image over the idle A tile
  constexpr int PITCH = 20;

  const int t = threadIdx.x;
  // filter: (16, 147) bf16 -> K-major SW128 rows of three 64-wide chunks, zero beyond 147
  for (int i = t; i < 16 * 24; i += 128) {                  // 16 rows x 24 pieces of 8 elements
    const int n = i / 24, j = i - n * 24;                   // j = 16-byte piece index along K (0..23; 20..23 are padding)
    uint32_t v[4] = {0u, 0u, 0u, 0u};
    __nv_bfloat16* vp = reinterpret_cast<__nv_bfloat16*>(v);
    for (int e = 0; e < 8; ++e) {
      const int k = j * 8 + e;
      if (k < ST_K) vp[e] = w[n * ST_K + k];
    }
    const int c = j >> 3, jj = j & 7;
    *reinterpret_cast<uint4*>(b_tile + c * 2048 + n * 128 + ((jj ^ (n & 7)) << 4)) = make_uint4(v[0], v[1], v[2], v[3]);
  }
  __syncthreads();

  const int tiles_w = (Wo + ST_TW - 1) / ST_TW, tiles_h = (Ho + ST_TH - 1) / ST_TH;
  const int n_tiles = tiles_w * tiles_h * n_img;
  const int tx = t & 15, ty = t >> 4;                       // this thread's pixel inside the tile (row m = t)
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    int r = tile;
    const int twi = r % tiles_w; r /= tiles_w;
    const int thi = r % tiles_h;
    const int img = r / tiles_h;
    const int ox0 = twi * ST_TW, oy0 = thi * ST_TH;
    // ---- input patch: rows 2*oy0-3 .. +20, elements (2*ox0-3)*3 - 1 .. +111 of the (W*3)-element image rows; 4-byte words
    const int g0 = (2 * ox0 - 3) * 3 - 1;                   // even: words never straddle the row ends (W*3 is even)
    const __nv_bfloat16* ximg = x + (long long)img * H * W * 3;
    for (int i = t; i < ST_PH * (ST_PW / 2); i += 128) {
      const int pr = i / (ST_PW / 2), pw = i - pr * (ST_PW / 2);
      const int iy = 2 * oy0 - 3 + pr, g = g0 + 2 * pw;
      uint32_t v = 0u;
      if (iy >= 0 && iy < H && g >= 0 && g + 1 < W * 3) v = *reinterpret_cast<const uint32_t*>(ximg + (long long)iy * W * 3 + g);
      reinterpret_cast<uint32_t*>(patch)[pr * (ST_PW / 2) + pw] = v;
    }
    __syncthreads();
    // ---- im2col in shared memory: row t of A = the 7 x 21 window of this pixel, k = ky*21 + kx*3 + c
    {
      const __nv_bfloat16* base = patch + (2 * ty) * ST_PW + 6 * tx + 1;
      const uint32_t row_off = (uint32_t)((t >> 3) * 1024 + (t & 7) * 128);
#pragma unroll
      for (int j = 0; j < ST_KPAD / 8; ++j) {               // 20 pieces of 8 elements
        uint32_t v[4];
#pragma unroll
        for (int h = 0; h < 4; ++h) {
          const int k0 = j * 8 + 2 * h, k1 = k0 + 1;
          const uint32_t lo = k0 < ST_K ? (uint32_t)__bfloat16_as_ushort(base[(k0 / 21) * ST_PW + (k0 % 21)]) : 0u;
          const uint32_t hi = k1 < ST_K ? (uint32_t)__bfloat16_as_ushort(base[(k1 / 21) * ST_PW + (k1 % 21)]) : 0u;
          v[h] = lo | (hi << 16);
        }
        const int c = j >> 3, jj = j & 7;
        *reinterpret_cast<uint4*>(a_tile + c * 16384 + row_off + ((jj ^ (t & 7)) << 4)) = make_uint4(v[0], v[1], v[2], v[3]);
      }
    }
    fence_proxy_async();
    __syncthreads();
    {
      const uint32_t a_addr = smem_u32(a_tile), b_addr = smem_u32(b_tile);
      float acc[2][8];
      wgmma_fence();
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int kk = 0; kk < ST_KPAD / 16; ++kk)
          wgmma_bf16<16, 0, 0>(acc[h], make_desc(a_addr + h * 8192 + (kk >> 2) * 16384 + (kk & 3) * 32, 16, 1024),
                               make_desc(b_addr + (kk >> 2) * 2048 + (kk & 3) * 32, 16, 1024), kk > 0);
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence<8>(acc[0]);
      acc_fence<8>(acc[1]);
      __syncthreads();                                      // every MMA has read the A tile: the image may overwrite it
      acc_store<16>(acc[0], acc_img, PITCH, 0, t);
      acc_store<16>(acc[1], acc_img, PITCH, 64, t);
      __syncthreads();
    }
    uint32_t v[32];
    img_ld<16>(acc_img, PITCH, t, 0, v);
    const int ox = ox0 + tx, oy = oy0 + ty;
    if (ox < Wo && oy < Ho) {
      uint32_t o[8];
#pragma unroll
      for (int h = 0; h < 8; ++h) {
        float f0 = __uint_as_float(v[2 * h]) + bias[2 * h], f1 = __uint_as_float(v[2 * h + 1]) + bias[2 * h + 1];
        if (relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
        o[h] = pack_bf16(__float_as_uint(f0), __float_as_uint(f1));
      }
      uint4* dst = reinterpret_cast<uint4*>(y + (((long long)img * Ho + oy) * Wo + ox) * 16);
      dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
      dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
    }
    __syncthreads();          // the patch and the A tile are rewritten by the next iteration; image reads are done
  }
}

}  // namespace

// Stem of the image backbone: y (n,Ho,Wo,16) = act(conv7x7/2/3(x (n,H,W,3), w_ohwi (16,7,7,3)) + bias), bf16 NHWC.
extern "C" int esb_stem7x7_tc(const void* x, const void* w_ohwi, const float* bias, void* y, int n_img, int H, int W, int relu,
                              void* stream_) {
  ESB_CHECK_ARG(n_img >= 0 && H > 0 && W > 0 && (W * 3) % 2 == 0, "esb_stem7x7_tc: W*3 must be even (4-byte patch loads)");
  ESB_CHECK_ARG(bias != nullptr, "esb_stem7x7_tc: bias (16 fp32) is required");
  if (n_img == 0) return ESB_OK;
  const int Ho = (H + 6 - 7) / 2 + 1, Wo = (W + 6 - 7) / 2 + 1;
  const size_t smem = 3 * 16384 + 3 * 2048 + ((ST_PH * ST_PW * 2 + 15) & ~15) + 1024;
  cudaError_t e = cudaFuncSetAttribute(stem7x7_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { esb_set_error("esb_stem7x7_tc: smem attr: %s", cudaGetErrorString(e)); return ESB_ECUDA; }
  const long long n_tiles = (long long)esb_div_up(Wo, ST_TW) * esb_div_up(Ho, ST_TH) * n_img;
  long long grid = (long long)esb_sm_count() * 3;
  if (grid > n_tiles) grid = n_tiles;
  stem7x7_tc_kernel<<<(unsigned)grid, 128, smem, (cudaStream_t)stream_>>>(
      (const __nv_bfloat16*)x, (const __nv_bfloat16*)w_ohwi, bias, (__nv_bfloat16*)y, n_img, H, W, Ho, Wo, relu);
  ESB_CUDA_LAUNCH_CHECK("stem7x7_tc_kernel");
  return ESB_OK;
}

// ------------------------------------------------------------------------------------------------------------
// Weight gradient of the dense NHWC convolution, TMA-fed: dW^T[(tap, ci), co] = sum over output pixels of
// x[pixel shifted by tap, ci] * dy[pixel, co]. The pixels are the reduction dimension: a pipeline stage holds a box of exactly
// 64 output pixels (TN x TH x TW, powers of two) of dy and, for every (tap, channel slice) "atom" of the CTA's 128-row slice
// of the filter, the same box of x at the tap's offset (zero padding and ragged edges = TMA out-of-bounds zeros on BOTH
// operands, stride 2 = element strides). Both boxes land as [pixel][channel] rows = the MN-major operands wgmma takes
// directly (no transpose anywhere). A CTA accumulates its share of the pixel tiles in registers and stores its 128 x N_TILE
// fp32 tile to its split's partial of dW^T; the host adds the splits in order.
// CTA = (pixel-tile range) x (128-row slice of (tap, ci)) x (N_TILE slice of co). Threads: 0..255 consumers (64 filter rows
// per warpgroup), 256..287 producer, 288..415 epilogue.
// ------------------------------------------------------------------------------------------------------------
namespace {

struct WgradGeom {
  int tiles_w, tiles_h, tiles_d, tiles_n;     // pixel-tile grid over the OUTPUT pixels
  int TW, TH, TD, TN;                // TW*TH*TD*TN == 64
  int kd, kh, kw, stride, sd, pad, pd;   // sd / pd: stride / padding along depth (1 / 0 for 2-D convolutions)
  int cin, cout, aw, atoms_per_slice, chunks_per_tap;   // aw = channels per atom = min(cin, 64)
  int stages, tiles_per_cta;
};

template <int N_TILE>
__global__ void __launch_bounds__(THREADS, 1)
conv_tma_wgrad_kernel(const __grid_constant__ CUtensorMap tmx, const __grid_constant__ CUtensorMap tmdy,
                      float* __restrict__ dw, const WgradGeom g) {
  constexpr int NA = N_TILE < 64 ? N_TILE : 64;                // columns per B atom
  constexpr int A_BYTES = 64 * 256;                            // 64 pixels x 128 filter rows
  constexpr int B_BYTES = 64 * N_TILE * 2;
  constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  constexpr int PITCH = N_TILE + 4;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const int STAGES = g.stages;
  uint64_t* full_bar = (uint64_t*)(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* accum_bar = empty_bar + STAGES;
  float* img = reinterpret_cast<float*>(smem);                 // accumulator image over the idle stage buffers

  const int lane = threadIdx.x & 31;
  const int taps = g.kd * g.kh * g.kw;
  const int n_tiles = g.tiles_w * g.tiles_h * g.tiles_d * g.tiles_n;
  const int t_beg = blockIdx.x * g.tiles_per_cta;
  const int t_end = min(n_tiles, t_beg + g.tiles_per_cta);
  if (t_beg >= n_tiles) return;                                // uniform for the whole CTA
  const int total = t_end - t_beg;
  const int slice = blockIdx.y, co0 = blockIdx.z * N_TILE;
  const int awb = g.aw * 2;                                    // bytes per A row
  const int atom0 = slice * g.atoms_per_slice;
  const int n_atoms_total = taps * g.chunks_per_tap;
  const int n_valid = min(g.atoms_per_slice, n_atoms_total - atom0);
  const uint32_t a_atom_bytes = 64u * awb;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], NCONS / 32);
    }
    mbar_init(accum_bar, NCONS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    tma_prefetch_desc(&tmx);
    tma_prefetch_desc(&tmdy);
  }
  __syncthreads();

  if (threadIdx.x >= PROD0 && threadIdx.x < EPI0) {
    if (lane == 0) {
      for (int it = 0; it < total; ++it) {
        int t = t_beg + it;
        const int tw = t % g.tiles_w; t /= g.tiles_w;
        const int th = t % g.tiles_h; t /= g.tiles_h;
        const int td = t % g.tiles_d; t /= g.tiles_d;
        const int ox0 = tw * g.TW, oy0 = th * g.TH, oz0 = td * g.TD, img0 = t * g.TN;
        const int s = it % STAGES;
        mbar_wait(&empty_bar[s], ((it / STAGES) & 1) ^ 1);
        mbar_expect_tx(&full_bar[s], (uint32_t)n_valid * a_atom_bytes + B_BYTES);
        const uint32_t a_base = smem_u32(smem + s * STAGE_BYTES);
        const uint32_t b_base = a_base + A_BYTES;
        for (int a = 0; a < n_valid; ++a) {
          const int ga = atom0 + a;
          const int tap = ga / g.chunks_per_tap, ch0 = (ga - tap * g.chunks_per_tap) * g.aw;
          const int kz = tap / (g.kh * g.kw), kr = tap - kz * (g.kh * g.kw);
          const int ky = kr / g.kw, kx = kr - ky * g.kw;
          tma_load_5d(&tmx, &full_bar[s], a_base + a * a_atom_bytes, ch0, ox0 * g.stride - g.pad + kx, oy0 * g.stride - g.pad + ky,
                      oz0 * g.sd - g.pd + kz, img0);
        }
#pragma unroll
        for (int b = 0; b < N_TILE / NA; ++b)
          tma_load_5d(&tmdy, &full_bar[s], b_base + b * (64 * NA * 2), co0 + b * NA, ox0, oy0, oz0, img0);
      }
    }
  } else if (threadIdx.x < NCONS) {
    // consumers: warpgroup wg owns filter rows 64 wg .. 64 wg + 63 of the slice (64 / aw atoms further along the A tile)
    const int wg = threadIdx.x >> 7;
    const uint32_t a_layout = mma_layout_of(awb), b_layout = mma_layout_of(NA * 2);
    float acc[N_TILE / 2];
    for (int it = 0; it < total; ++it) {
      const int s = it % STAGES;
      mbar_wait(&full_bar[s], (it / STAGES) & 1);
      const uint32_t a_addr = smem_u32(smem + s * STAGE_BYTES) + wg * (64 / g.aw) * a_atom_bytes;
      const uint32_t b_addr = smem_u32(smem + s * STAGE_BYTES) + A_BYTES;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)                           // 16 pixels per MMA
        wgmma_bf16<N_TILE, 1, 1>(acc, make_desc_sw(a_addr + kk * 16 * awb, a_atom_bytes, 8 * awb, a_layout),
                                 make_desc_sw(b_addr + kk * 16 * (NA * 2), 64 * NA * 2, 8 * (NA * 2), b_layout), it > 0 || kk > 0);
      wgmma_commit();
      wgmma_wait<1>();
      if (it > 0 && lane == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
    }
    wgmma_wait<0>();
    acc_fence<N_TILE / 2>(acc);
    asm volatile("bar.sync 2, %0;" ::"n"(NCONS) : "memory");  // every wgmma has read its stage: the image may overwrite them
    acc_store<N_TILE>(acc, img, PITCH, wg * 64, threadIdx.x & 127);
    mbar_arrive(accum_bar);
  } else {
    // epilogue: image row = filter row of the slice, column = co
    const int quad = (threadIdx.x - EPI0) >> 5;
    mbar_wait(accum_bar, 0);
    const float* stg = img;
    const int rows_valid = n_valid * g.aw;                       // accumulator rows backed by loaded atoms
    for (int rr = 0; rr < 32; ++rr) {
      const int r = quad * 32 + rr;
      if (r >= rows_valid) break;
      // row r of the slice = atom r / aw, channel r % aw  ->  filter row (tap * cin + ch)
      const int ga = atom0 + r / g.aw;
      const int tap = ga / g.chunks_per_tap, ch = (ga - tap * g.chunks_per_tap) * g.aw + (r % g.aw);
      float* dwrow = dw + (((long long)blockIdx.x * g.kd * g.kh * g.kw + tap) * g.cin + ch) * g.cout + co0;
      for (int c = lane * 4; c < N_TILE; c += 128)
        *reinterpret_cast<float4*>(dwrow + c) = *reinterpret_cast<const float4*>(stg + r * PITCH + c);
    }
  }
}

template <int N_TILE>
int launch_wgrad_tma(const CUtensorMap& tmx, const CUtensorMap& tmdy, float* dw, WgradGeom g, int slices, int n_blocks,
                     cudaStream_t stream) {
  constexpr int STAGE_BYTES = 64 * 256 + 64 * N_TILE * 2;
  int stages = (100 * 1024) / STAGE_BYTES;
  const int need = (128 * (N_TILE + 4) * 4 + STAGE_BYTES - 1) / STAGE_BYTES;      // the epilogue reuses the stage buffers
  stages = stages < need ? need : stages > 6 ? 6 : stages;
  g.stages = stages;
  const size_t smem = (size_t)stages * STAGE_BYTES + (2 * stages + 1) * 8 + 16 + 1024;
  auto kern = conv_tma_wgrad_kernel<N_TILE>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) { esb_set_error("conv_tma_wgrad: smem attr: %s", cudaGetErrorString(e)); return ESB_ECUDA; }
  const long long n_tiles = (long long)g.tiles_w * g.tiles_h * g.tiles_d * g.tiles_n;
  // ~2 CTAs per SM in total; every CTA walks a contiguous range of pixel tiles
  long long splits = (2LL * esb_sm_count() + (long long)slices * n_blocks - 1) / ((long long)slices * n_blocks);
  if (splits > n_tiles) splits = n_tiles;
  if (splits < 1) splits = 1;
  g.tiles_per_cta = (int)((n_tiles + splits - 1) / splits);
  dim3 grid((unsigned)((n_tiles + g.tiles_per_cta - 1) / g.tiles_per_cta), slices, n_blocks);
  // every split writes a whole partial of dW^T (its slices x channel blocks cover all rows and columns)
  const long long width = (long long)g.kd * g.kh * g.kw * g.cin * g.cout;
  float* part = nullptr;
  ESB_CUDA_CALL(esb_scratch_alloc((void**)&part, sizeof(float) * grid.x * width, stream));
  kern<<<grid, THREADS, smem, stream>>>(tmx, tmdy, part, g);
  int rc = esb_sum_partial_rows(part, (int)grid.x, width, dw, 1, stream);
  ESB_CUDA_CALL(esb_scratch_free(part, stream));
  return rc;
}

}  // namespace

namespace {

int conv_wgrad_any(const char* who, const void* x, const void* dy, float* dw_t, int n_img, int D, int H, int W, int cin, int cout,
                   int kd, int kh, int kw, int stride, int pad, cudaStream_t stream) {
  if (!(channels_ok(cin) && channels_ok(cout))) { esb_set_error("%s: channels must be 16, 32 or a multiple of 64", who); return ESB_EINVAL; }
  if (!(kd >= 1 && kh >= 1 && kw >= 1 && stride >= 1 && stride <= 8 && pad >= 0)) { esb_set_error("%s: bad filter geometry", who); return ESB_EINVAL; }
  const int pd = kd > 1 ? pad : 0, sd = D > 1 ? stride : 1;
  const int Do = (D + 2 * pd - kd) / sd + 1, Ho = (H + 2 * pad - kh) / stride + 1, Wo = (W + 2 * pad - kw) / stride + 1;
  if (Do <= 0 || Ho <= 0 || Wo <= 0) { esb_set_error("%s: empty output", who); return ESB_EINVAL; }
  if (n_img == 0) return ESB_OK;
  WgradGeom g{};
  g.kd = kd; g.kh = kh; g.kw = kw; g.stride = stride; g.sd = sd; g.pad = pad; g.pd = pd; g.cin = cin; g.cout = cout;
  g.aw = cin < 64 ? cin : 64;
  g.atoms_per_slice = 128 / g.aw;
  g.chunks_per_tap = cin / g.aw;
  // pixel box of exactly 64 output pixels (powers of two): the one wasting the fewest zero-filled pixels
  double best = -1.0;
  for (int tw = 1; tw <= 64; tw *= 2)
    for (int th = 1; tw * th <= 64; th *= 2)
      for (int td = 1; tw * th * td <= 64; td *= 2) {
        const int tn = 64 / (tw * th * td);
        if (tn > 1 && (tw < Wo || th < Ho || td < Do)) continue;   // several images per box only for whole (padded) volumes
        if (td > 1 && Do == 1) continue;
        const double tiles = (double)esb_div_up(Wo, tw) * esb_div_up(Ho, th) * esb_div_up(Do, td) * esb_div_up(n_img, tn);
        const double eff = (double)Wo * Ho * Do * n_img / (tiles * 64.0) + 1e-6 * tw;
        if (eff > best) { best = eff; g.TW = tw; g.TH = th; g.TD = td; g.TN = tn; }
      }
  g.tiles_w = esb_div_up(Wo, g.TW); g.tiles_h = esb_div_up(Ho, g.TH); g.tiles_d = esb_div_up(Do, g.TD);
  g.tiles_n = esb_div_up(n_img, g.TN);
  const int n_tile = cout >= 128 ? 128 : cout;
  const int n_blocks = cout / n_tile;
  const int slices = esb_div_up(kd * kh * kw * g.chunks_per_tap, g.atoms_per_slice);
  CUtensorMap tmx, tmdy;
  {
    unsigned long long dims[5] = {(unsigned long long)cin, (unsigned long long)W, (unsigned long long)H, (unsigned long long)D,
                                  (unsigned long long)n_img};
    unsigned long long str[4] = {(unsigned long long)cin * 2, (unsigned long long)W * cin * 2, (unsigned long long)H * W * cin * 2,
                                 (unsigned long long)D * H * W * cin * 2};
    unsigned box[5] = {(unsigned)g.aw, (unsigned)((g.TW - 1) * stride + 1), (unsigned)((g.TH - 1) * stride + 1),
                       (unsigned)((g.TD - 1) * sd + 1), (unsigned)g.TN};
    unsigned es[5] = {1, (unsigned)stride, (unsigned)stride, (unsigned)sd, 1};
    int rc = esb_tma_encode(&tmx, x, 5, dims, str, box, es, g.aw * 2);
    if (rc != ESB_OK) return rc;
  }
  {
    const int na = n_tile < 64 ? n_tile : 64;
    unsigned long long dims[5] = {(unsigned long long)cout, (unsigned long long)Wo, (unsigned long long)Ho, (unsigned long long)Do,
                                  (unsigned long long)n_img};
    unsigned long long str[4] = {(unsigned long long)cout * 2, (unsigned long long)Wo * cout * 2,
                                 (unsigned long long)Ho * Wo * cout * 2, (unsigned long long)Do * Ho * Wo * cout * 2};
    unsigned box[5] = {(unsigned)na, (unsigned)g.TW, (unsigned)g.TH, (unsigned)g.TD, (unsigned)g.TN};
    int rc = esb_tma_encode(&tmdy, dy, 5, dims, str, box, nullptr, na * 2);
    if (rc != ESB_OK) return rc;
  }
  int rc;
  switch (n_tile) {
    case 16: rc = launch_wgrad_tma<16>(tmx, tmdy, dw_t, g, slices, n_blocks, stream); break;
    case 32: rc = launch_wgrad_tma<32>(tmx, tmdy, dw_t, g, slices, n_blocks, stream); break;
    case 64: rc = launch_wgrad_tma<64>(tmx, tmdy, dw_t, g, slices, n_blocks, stream); break;
    case 128: rc = launch_wgrad_tma<128>(tmx, tmdy, dw_t, g, slices, n_blocks, stream); break;
    default: esb_set_error("%s: unsupported Cout %d", who, cout); return ESB_EINVAL;
  }
  if (rc != ESB_OK) return rc;
  ESB_CUDA_LAUNCH_CHECK("conv_tma_wgrad_kernel");
  return ESB_OK;
}

}  // namespace

// dw_t (kh*kw*cin, cout) fp32 += the weight gradient (zeroed by the caller): dW[co, ci, ky, kx] = dw_t[(ky*kw + kx)*cin + ci, co].
// x (n,H,W,cin), dy (n,Ho,Wo,cout) bf16 NHWC; cin, cout in {16, 32, 64, 128, 256, 512, ...}.
extern "C" int esb_conv2d_tma_wgrad(const void* x, const void* dy, float* dw_t, int n_img, int H, int W, int cin, int cout,
                                    int kh, int kw, int stride, int pad, void* stream_) {
  return conv_wgrad_any("esb_conv2d_tma_wgrad", x, dy, dw_t, n_img, 1, H, W, cin, cout, 1, kh, kw, stride, pad,
                        (cudaStream_t)stream_);
}

// 3-D: dw_t (k*k*k*cin, cout) fp32 += the gradient (zeroed by the caller), row = ((kz*k + ky)*k + kx)*cin + ci; x (n,D,H,W,cin), dy NDHWC bf16.
extern "C" int esb_conv3d_tma_wgrad(const void* x, const void* dy, float* dw_t, int n, int D, int H, int W, int cin, int cout, int k,
                                    int stride, int pad, void* stream_) {
  return conv_wgrad_any("esb_conv3d_tma_wgrad", x, dy, dw_t, n, D, H, W, cin, cout, k, k, k, stride, pad, (cudaStream_t)stream_);
}
