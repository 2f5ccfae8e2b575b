// esb200 — exact 9-DoF oriented-box 3D IoU (SURVEY §8 row a12). Replaces pytorch3d.ops.box3d_overlap (†upstream
// pytorch3d 0.7.x `iou_box3d`) as reached through EulerInstance3DBoxes.overlaps
// (embodiedscan/structures/bbox_3d/euler_box3d.py:103-135; callers: match_cost.py:108, indoor_eval.py:127,
// grounding_metric.py:106). Same contract: corners (N,8,3) x (M,8,3) in the container's corner order -> (vol, iou).
//
// The clipping arithmetic lives in iou3d.cuh. One thread per (i, j) pair; latency-bound, tiny data.
#include "iou3d.cuh"

namespace {

__global__ void box3d_overlap_kernel(const float* __restrict__ c1, int n1, const float* __restrict__ c2, int n2,
                                     float* __restrict__ vol, float* __restrict__ iou) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n1 * n2) return;
  int i = t / n2, j = t - i * n2;
  box3d_pair_overlap(c1 + i * 24, c2 + j * 24, vol + t, iou + t);
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
