// esb200 — exact 9-DoF oriented-box 3D IoU (SURVEY §8 row a12). Replaces pytorch3d.ops.box3d_overlap (†upstream
// pytorch3d 0.7.x `iou_box3d`) as reached through EulerInstance3DBoxes.overlaps
// (embodiedscan/structures/bbox_3d/euler_box3d.py:103-135; callers: match_cost.py:108, indoor_eval.py:127,
// grounding_metric.py:106). Same contract: corners (N,8,3) x (M,8,3) in the container's corner order -> (vol, iou).
//
// The clipping arithmetic lives in iou3d.cuh. One thread per (i, j) pair; latency-bound, tiny data.
//
// esb_box3d_best_overlap is the same pair arithmetic reduced on the device: each query box is clipped only against the
// targets of its own range (the same-label ground truth of its scan in indoor_eval, a prompt's targets in the grounding
// metric) and keeps the best IoU and the index of the box that gives it, instead of an n1 x n2 matrix on the host.
#include "iou3d.cuh"

namespace {

__global__ void box3d_overlap_kernel(const float* __restrict__ c1, int n1, const float* __restrict__ c2, int n2,
                                     float* __restrict__ vol, float* __restrict__ iou) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n1 * n2) return;
  int i = t / n2, j = t - i * n2;
  box3d_pair_overlap(c1 + i * 24, c2 + j * 24, vol + t, iou + t);
}

// torch.max's choice between two candidates (value, original index): a NaN beats any number (the first NaN wins), otherwise
// the larger value, ties to the smaller index. A total order, so the result does not depend on the walk order.
__device__ __forceinline__ bool beats(float v, int j, float b, int a) {
  if (a < 0) return true;
  if (isnan(v)) return !isnan(b) || j < a;
  if (isnan(b)) return false;
  return v > b || (v == b && j < a);
}

// One thread per query: its range qbeg[i]..qend[i] of tidx is walked in full, every pair through box3d_pair_overlap.
__global__ void box3d_best_overlap_kernel(const float* __restrict__ cq, int m, const float* __restrict__ ct,
                                          const int* __restrict__ tidx, const int* __restrict__ qbeg,
                                          const int* __restrict__ qend, float* __restrict__ best, int* __restrict__ arg) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const float* q = cq + (size_t)i * 24;
  float b = -INFINITY;
  int a = -1;
  for (int k = qbeg[i], e = qend[i]; k < e; ++k) {
    int j = tidx[k];
    float vol, iou;
    box3d_pair_overlap(q, ct + (size_t)j * 24, &vol, &iou);
    if (beats(iou, j, b, a)) b = iou, a = j;
  }
  best[i] = b;
  arg[i] = a;
}

}  // namespace


// corners1 (n1,8,3), corners2 (n2,8,3) fp32 -> vol (n1,n2), iou (n1,n2)
extern "C" int esb_box3d_overlap(const float* corners1, int n1, const float* corners2, int n2, float* vol, float* iou,
                                 void* stream) {
  if ((long long)n1 * n2 == 0) return ESB_OK;
  box3d_overlap_kernel<<<esb_div_up((long long)n1 * n2, 64), 64, 0, (cudaStream_t)stream>>>(corners1, n1, corners2, n2, vol,
                                                                                          iou);
  ESB_CUDA_LAUNCH_CHECK("box3d_overlap_kernel");
  return ESB_OK;
}

// query corners (m,8,3), target corners (g,8,3) fp32; query i is compared with targets tidx[qbeg[i] .. qend[i]) ->
// best[i] (max IoU, -inf for an empty range), arg[i] (the target index that gives it, -1 for an empty range)
extern "C" int esb_box3d_best_overlap(const float* qcorners, int m, const float* tcorners, const int* tidx,
                                      const int* qbeg, const int* qend, float* best, int* arg, void* stream) {
  if (m == 0) return ESB_OK;
  box3d_best_overlap_kernel<<<esb_div_up(m, 64), 64, 0, (cudaStream_t)stream>>>(qcorners, m, tcorners, tidx, qbeg, qend,
                                                                                best, arg);
  ESB_CUDA_LAUNCH_CHECK("box3d_best_overlap_kernel");
  return ESB_OK;
}
