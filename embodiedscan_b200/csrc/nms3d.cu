// esb200 — class-agnostic greedy NMS on the exact 9-DoF 3D IoU with a score threshold and a per-label cap: the final
// box filter of the reference's demo (`nms_filter`, demo/demo.py:84-130), which there is an N x N
// pytorch3d.ops.box3d_overlap call followed by an O(N^2) Python double loop on the host. Batched over scans (segments).
//
//   for i in candidates, score-descending (stable):
//     if kept_of_label[label[i]] >= topk_per_class: continue
//     if score[i] < score_thr:                      continue
//     if any(iou3d(i, j) > iou_thr for j in selected): continue
//     selected.append(i); kept_of_label[label[i]] += 1
//
// A candidate skipped by the cap or the score threshold never suppresses anything; `selected` comes back in selection
// order. Candidates arrive already score-sorted inside each segment (the host sorts; ties keep input order).
//
// Two kernels.
//  * nms3d_pair_kernel: one CTA per (segment, 64-row block, 64-column block) of the upper triangle. The 64 + 64 boxes are
//    staged in shared memory once (centre, half extents, rotation from the ZXY Euler angles, the 8 corners, circumscribed
//    radius). Every pair is first tested for (a) disjoint circumscribed spheres and (b) a separating axis among the 15
//    candidates of two oriented boxes; either proves the intersection empty, so the IoU is 0 and cannot exceed
//    iou_thr >= 0. Survivors are compacted into a shared list and only they run the exact clipping of iou3d.cuh, the
//    same instructions esb_box3d_overlap executes. The result is one bit per pair; no N x N float matrix exists.
//  * nms3d_greedy_kernel: one CTA per segment walks the candidates in order; the removed words and the per-label kept
//    counters live in shared memory and the threads OR a kept row's mask words into `removed` in parallel.
// Everything after the comparison `iou > iou_thr` is integer, so the kept list is deterministic.
//
// Degenerate boxes (pytorch3d raises on them): a box with a size <= 0 or any non-finite value has IoU 0 with every box.
// It can be kept, it never suppresses and it is never suppressed.
#include "iou3d.cuh"

namespace {

constexpr int TILE = 64;
constexpr int PAIR_THREADS = 128;
constexpr int KSTRIDE = 25;  // 24 corner floats per box, padded against shared-memory bank conflicts

struct StagedBoxes {            // structure of arrays over the 2 * TILE boxes of a CTA: rows first, then columns
  float c[3][2 * TILE];         // centre
  float h[3][2 * TILE];         // half extents
  float R[9][2 * TILE];         // rotation, row-major: column a is the box's axis a in world coordinates
  float rad[2 * TILE];          // circumscribed-sphere radius
  float k[2 * TILE * KSTRIDE];  // corners in the container's order (geometry.box_corners_container)
  unsigned char valid[2 * TILE];
};

// R = Rz(alpha) @ Rx(beta) @ Ry(gamma), the pytorch3d 'ZXY' convention of geometry.euler_angles_to_matrix
__device__ void stage_box(StagedBoxes& sb, int slot, const float* __restrict__ b) {
  float v[9];
  bool ok = b != nullptr;
  for (int q = 0; q < 9; ++q) {
    v[q] = ok ? b[q] : 0.f;
    ok = ok && isfinite(v[q]);
  }
  ok = ok && v[3] > 0.f && v[4] > 0.f && v[5] > 0.f;
  sb.valid[slot] = ok ? 1 : 0;
  if (!ok) return;
  float sa, ca, sbt, cb, sc, cc;
  sincosf(v[6], &sa, &ca);
  sincosf(v[7], &sbt, &cb);
  sincosf(v[8], &sc, &cc);
  const float R[9] = {ca * cc - sa * sbt * sc, -sa * cb, ca * sc + sa * sbt * cc,
                      sa * cc + ca * sbt * sc, ca * cb,  sa * sc - ca * sbt * cc,
                      -cb * sc,                sbt,      cb * cc};
  for (int q = 0; q < 9; ++q) sb.R[q][slot] = R[q];
  for (int a = 0; a < 3; ++a) {
    sb.c[a][slot] = v[a];
    sb.h[a][slot] = 0.5f * v[3 + a];
  }
  sb.rad[slot] = 0.5f * sqrtf(v[3] * v[3] + v[4] * v[4] + v[5] * v[5]);
  // 0:(0,0,0) 1:(0,0,1) 2:(0,1,1) 3:(0,1,0) 4:(1,0,0) 5:(1,0,1) 6:(1,1,1) 7:(1,1,0), minus 0.5, times the size
  const int bits[8] = {0, 1, 3, 2, 4, 5, 7, 6};
  for (int q = 0; q < 8; ++q) {
    const float lx = ((bits[q] >> 2) & 1 ? 0.5f : -0.5f) * v[3];
    const float ly = ((bits[q] >> 1) & 1 ? 0.5f : -0.5f) * v[4];
    const float lz = ((bits[q] >> 0) & 1 ? 0.5f : -0.5f) * v[5];
    for (int a = 0; a < 3; ++a)
      sb.k[slot * KSTRIDE + 3 * q + a] = v[a] + R[3 * a] * lx + R[3 * a + 1] * ly + R[3 * a + 2] * lz;
  }
}

// True when one of the 15 axes (3 + 3 face normals, 9 edge cross products) separates boxes i and j. The slack keeps
// fp32 rounding and near-parallel edges (cross product ~ 0) on the "not separated" side, where the exact clipping decides.
__device__ bool separated(const StagedBoxes& sb, int i, int j) {
  float Rm[3][3], Ab[3][3], t[3];
  const float d[3] = {sb.c[0][j] - sb.c[0][i], sb.c[1][j] - sb.c[1][i], sb.c[2][j] - sb.c[2][i]};
  const float ha[3] = {sb.h[0][i], sb.h[1][i], sb.h[2][i]}, hb[3] = {sb.h[0][j], sb.h[1][j], sb.h[2][j]};
  for (int a = 0; a < 3; ++a) {
    t[a] = d[0] * sb.R[a][i] + d[1] * sb.R[3 + a][i] + d[2] * sb.R[6 + a][i];
    for (int b = 0; b < 3; ++b) {
      Rm[a][b] = sb.R[a][i] * sb.R[b][j] + sb.R[3 + a][i] * sb.R[3 + b][j] + sb.R[6 + a][i] * sb.R[6 + b][j];
      Ab[a][b] = fabsf(Rm[a][b]) + 1e-6f;
    }
  }
  const float rel = 1.f + 1e-5f, abs_slack = 1e-6f;
  for (int a = 0; a < 3; ++a)
    if (fabsf(t[a]) > (ha[a] + hb[0] * Ab[a][0] + hb[1] * Ab[a][1] + hb[2] * Ab[a][2]) * rel + abs_slack) return true;
  for (int b = 0; b < 3; ++b)
    if (fabsf(t[0] * Rm[0][b] + t[1] * Rm[1][b] + t[2] * Rm[2][b]) >
        (ha[0] * Ab[0][b] + ha[1] * Ab[1][b] + ha[2] * Ab[2][b] + hb[b]) * rel + abs_slack)
      return true;
  for (int a = 0; a < 3; ++a) {
    const int a1 = (a + 1) % 3, a2 = (a + 2) % 3;
    for (int b = 0; b < 3; ++b) {
      const int b1 = (b + 1) % 3, b2 = (b + 2) % 3;
      const float ra = ha[a1] * Ab[a2][b] + ha[a2] * Ab[a1][b];
      const float rb = hb[b1] * Ab[a][b2] + hb[b2] * Ab[a][b1];
      if (fabsf(t[a2] * Rm[a1][b] - t[a1] * Rm[a2][b]) > (ra + rb) * rel + abs_slack) return true;
    }
  }
  return false;
}

// mask: per segment (max_seg, W) uint64, bit c of word (i, w) = candidate w * 64 + c is suppressed by candidate i (> i
// only). Words left of a row's diagonal block are never written and never read. stats: per segment 3 counters.
__global__ void __launch_bounds__(PAIR_THREADS)
nms3d_pair_kernel(const float* __restrict__ boxes, const int* __restrict__ seg_off, int max_seg, int W, float iou_thr,
                  unsigned long long* __restrict__ mask, unsigned long long* __restrict__ stats) {
  const int cb = blockIdx.x, rb = blockIdx.y, s = blockIdx.z;
  const int beg = seg_off[s], n = seg_off[s + 1] - beg;
  if (cb < rb || cb * TILE >= n) return;
  __shared__ StagedBoxes sb;
  __shared__ unsigned long long s_mask[TILE];
  __shared__ unsigned short s_list[TILE * TILE];
  __shared__ int s_nlist;
  __shared__ unsigned int s_cnt[3];
  const int tid = threadIdx.x;
  {
    const int g = (tid < TILE ? rb * TILE + tid : cb * TILE + tid - TILE);
    stage_box(sb, tid, g < n ? boxes + (size_t)(beg + g) * 9 : nullptr);
  }
  if (tid < TILE) s_mask[tid] = 0ull;
  if (tid < 3) s_cnt[tid] = 0u;
  if (tid == 0) s_nlist = 0;
  __syncthreads();

  unsigned int tested = 0, past_sphere = 0, past_sat = 0;
  for (int p = tid; p < TILE * TILE; p += PAIR_THREADS) {
    const int r = p >> 6, c = p & 63;
    if (cb * TILE + c <= rb * TILE + r) continue;                 // strict upper triangle
    if (!sb.valid[r] || !sb.valid[TILE + c]) continue;            // out of range or degenerate: IoU 0
    ++tested;
    const float dx = sb.c[0][TILE + c] - sb.c[0][r], dy = sb.c[1][TILE + c] - sb.c[1][r],
                dz = sb.c[2][TILE + c] - sb.c[2][r];
    const float reach = (sb.rad[r] + sb.rad[TILE + c]) * (1.f + 1e-5f) + 1e-6f;
    if (dx * dx + dy * dy + dz * dz > reach * reach) continue;
    ++past_sphere;
    if (separated(sb, r, TILE + c)) continue;
    ++past_sat;
    s_list[atomicAdd(&s_nlist, 1)] = (unsigned short)p;
  }
  for (int o = 16; o > 0; o >>= 1) {
    tested += __shfl_xor_sync(0xffffffffu, tested, o);
    past_sphere += __shfl_xor_sync(0xffffffffu, past_sphere, o);
    past_sat += __shfl_xor_sync(0xffffffffu, past_sat, o);
  }
  if ((tid & 31) == 0) {
    atomicAdd(&s_cnt[0], tested);
    atomicAdd(&s_cnt[1], past_sphere);
    atomicAdd(&s_cnt[2], past_sat);
  }
  __syncthreads();

  // the survivors, evenly over the threads; the candidate (column, lower score) is box A as in the reference's iou[i][j]
  const int nlist = s_nlist;
  for (int q = tid; q < nlist; q += PAIR_THREADS) {
    const int p = s_list[q], r = p >> 6, c = p & 63;
    float vol, iou;
    box3d_pair_overlap(sb.k + (TILE + c) * KSTRIDE, sb.k + r * KSTRIDE, &vol, &iou);
    if (iou > iou_thr) atomicOr(&s_mask[r], 1ull << c);
  }
  __syncthreads();
  if (tid < TILE && rb * TILE + tid < n)
    mask[((size_t)s * max_seg + rb * TILE + tid) * W + cb] = s_mask[tid];
  if (tid < 3 && s_cnt[tid]) atomicAdd(&stats[3 * s + tid], (unsigned long long)s_cnt[tid]);
}

__global__ void __launch_bounds__(256)
nms3d_greedy_kernel(const unsigned long long* __restrict__ mask, const float* __restrict__ scores,
                    const int* __restrict__ labels, const int* __restrict__ seg_off, int max_seg, int W, float score_thr,
                    int topk, int num_classes, int* __restrict__ keep, int* __restrict__ n_keep) {
  extern __shared__ unsigned long long sm[];
  unsigned long long* removed = sm;          // (W)
  int* kept_of_label = (int*)(sm + W);       // (num_classes)
  __shared__ int s_lab[64];
  __shared__ unsigned int s_ok[2];
  const int s = blockIdx.x, tid = threadIdx.x;
  const int beg = seg_off[s], n = seg_off[s + 1] - beg;
  const unsigned long long* mseg = mask + (size_t)s * max_seg * W;
  const int nw = (n + 63) / 64;
  for (int x = tid; x < nw; x += blockDim.x) removed[x] = 0ull;
  for (int x = tid; x < num_classes; x += blockDim.x) kept_of_label[x] = 0;
  int nk = 0;
  for (int w = 0; w < nw; ++w) {
    __syncthreads();
    if (tid < 64) {
      const int i = w * 64 + tid;
      bool ok = i < n && !(scores[beg + i] < score_thr);
      const int lab = ok ? labels[beg + i] : 0;
      ok = ok && lab >= 0 && lab < num_classes;                  // a label outside the table is never kept
      s_lab[tid] = lab;
      const unsigned int b = __ballot_sync(0xffffffffu, ok);
      if ((tid & 31) == 0) s_ok[tid >> 5] = b;
    }
    __syncthreads();
    const unsigned long long ok64 = (unsigned long long)s_ok[0] | ((unsigned long long)s_ok[1] << 32);
    unsigned long long visited = 0ull;
    while (true) {                                                // every read below is block-uniform
      const unsigned long long cur = ok64 & ~removed[w] & ~visited;
      if (!cur) break;
      const int b = __ffsll((long long)cur) - 1;
      visited |= (2ull << b) - 1ull;
      const int lab = s_lab[b];
      if (kept_of_label[lab] >= topk) continue;                   // capped: skipped, suppresses nothing
      __syncthreads();                                            // all threads have read `removed` / the counter
      const int i = w * 64 + b;
      const unsigned long long* row = mseg + (size_t)i * W;
      for (int x = w + tid; x < nw; x += blockDim.x) removed[x] |= row[x];
      if (tid == 0) {
        keep[beg + nk] = beg + i;
        ++kept_of_label[lab];
      }
      ++nk;
      __syncthreads();
    }
  }
  if (tid == 0) n_keep[s] = nk;
}

size_t stats_bytes(int S) { return esb_align((size_t)S * 3 * sizeof(unsigned long long)); }

}  // namespace

extern "C" size_t esb_nms3d_9dof_workspace_bytes(int M, int S, int max_seg) {
  (void)M;
  if (S <= 0 || max_seg <= 0) return 0;
  const size_t W = (size_t)(max_seg + 63) / 64;
  return stats_bytes(S) + (size_t)S * max_seg * W * sizeof(unsigned long long);
}

extern "C" int esb_nms3d_9dof(const float* boxes9, const float* scores, const int* labels, const int* seg_off, int S,
                              int max_seg, float iou_thr, float score_thr, int topk_per_class, int num_classes,
                              int* keep, int* n_keep, void* ws, size_t ws_bytes, void* stream) {
  ESB_CHECK_ARG(iou_thr >= 0.f, "esb_nms3d_9dof: iou_thr must be >= 0 (the early rejects rely on IoU 0 never suppressing)");
  ESB_CHECK_ARG(S >= 0 && S <= 65535 && max_seg >= 0, "esb_nms3d_9dof: 0 <= S <= 65535 segments, max_seg >= 0");
  ESB_CHECK_ARG(num_classes >= 1 && topk_per_class >= 0, "esb_nms3d_9dof: num_classes >= 1 and topk_per_class >= 0");
  if (S == 0) return ESB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (max_seg == 0) {
    ESB_CUDA_CALL(cudaMemsetAsync(n_keep, 0, (size_t)S * sizeof(int), st));
    return ESB_OK;
  }
  const int W = (max_seg + 63) / 64;
  ESB_CHECK_ARG(W <= 65535, "esb_nms3d_9dof: segment too long");
  ESB_CHECK_ARG(ws_bytes >= esb_nms3d_9dof_workspace_bytes(0, S, max_seg), "esb_nms3d_9dof: workspace too small");
  const size_t smem = (size_t)W * sizeof(unsigned long long) + (size_t)num_classes * sizeof(int);
  ESB_CHECK_ARG(smem <= 200 * 1024, "esb_nms3d_9dof: removed words + label counters exceed shared memory");
  unsigned long long* stats = (unsigned long long*)ws;
  unsigned long long* mask = (unsigned long long*)((char*)ws + stats_bytes(S));
  ESB_CUDA_CALL(cudaMemsetAsync(stats, 0, stats_bytes(S), st));
  nms3d_pair_kernel<<<dim3(W, W, S), PAIR_THREADS, 0, st>>>(boxes9, seg_off, max_seg, W, iou_thr, mask, stats);
  ESB_CUDA_LAUNCH_CHECK("nms3d_pair_kernel");
  if (smem > 48 * 1024)
    ESB_CUDA_CALL(cudaFuncSetAttribute(nms3d_greedy_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  nms3d_greedy_kernel<<<S, 256, smem, st>>>(mask, scores, labels, seg_off, max_seg, W, score_thr, topk_per_class,
                                            num_classes, keep, n_keep);
  ESB_CUDA_LAUNCH_CHECK("nms3d_greedy_kernel");
  return ESB_OK;
}
