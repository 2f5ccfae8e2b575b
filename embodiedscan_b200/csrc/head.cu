// esb200 — FCAF3D (RotMat) head kernels: target assignment / centerness (SURVEY §8 row a9) and the sigmoid focal
// loss over the (Np,284) class logits (row a10). One fused pipeline replaces the ~15 dense (Np,Ng,*) temporaries
// of FCAF3DHeadRotMat.get_targets (embodiedscan/models/dense_heads/fcaf3d_head.py:1578-1664), _get_face_distances
// (:1527-1557) and _get_centerness (:1559-1576); focal follows mmcv.ops.sigmoid_focal_loss (†upstream mmcv
// 2.0.0rc4, CUDA semantics: label -1 = no positive class) as wrapped by mmdet.FocalLoss (cfg :46-52).
//
// Selection outputs (cls targets, box index) are integer-exact against the oracle: every float compare uses the
// same rounded operation sequence (no FMA contraction). Compulsory traffic per scan: Np*12 + Ng*72 + Np*48 B.
#include "common.cuh"

namespace {

struct FaceDist { float d[6]; };

// boxes: (Ng,9) = gravity centre(3), size(3), euler(3) ; rneg: (Ng,9) = euler_angles_to_matrix(-euler,'ZXY') row-major
__device__ __forceinline__ FaceDist face_distances(const float* __restrict__ box, const float* __restrict__ R, float px,
                                                   float py, float pz) {
  float sx = __fsub_rn(px, box[0]), sy = __fsub_rn(py, box[1]), sz = __fsub_rn(pz, box[2]);
  // shift @ R^T  (rotation_3d_in_euler(shift, -angles))
  float rx = __fadd_rn(__fadd_rn(__fmul_rn(sx, R[0]), __fmul_rn(sy, R[1])), __fmul_rn(sz, R[2]));
  float ry = __fadd_rn(__fadd_rn(__fmul_rn(sx, R[3]), __fmul_rn(sy, R[4])), __fmul_rn(sz, R[5]));
  float rz = __fadd_rn(__fadd_rn(__fmul_rn(sx, R[6]), __fmul_rn(sy, R[7])), __fmul_rn(sz, R[8]));
  float cx = __fadd_rn(box[0], rx), cy = __fadd_rn(box[1], ry), cz = __fadd_rn(box[2], rz);
  float hx = __fdiv_rn(box[3], 2.f), hy = __fdiv_rn(box[4], 2.f), hz = __fdiv_rn(box[5], 2.f);
  FaceDist f;
  f.d[0] = __fadd_rn(__fsub_rn(cx, box[0]), hx);
  f.d[1] = __fsub_rn(__fadd_rn(box[0], hx), cx);
  f.d[2] = __fadd_rn(__fsub_rn(cy, box[1]), hy);
  f.d[3] = __fsub_rn(__fadd_rn(box[1], hy), cy);
  f.d[4] = __fadd_rn(__fsub_rn(cz, box[2]), hz);
  f.d[5] = __fsub_rn(__fadd_rn(box[2], hz), cz);
  return f;
}
__device__ __forceinline__ bool inside_box(const FaceDist& f) {
  float m = fminf(fminf(fminf(f.d[0], f.d[1]), fminf(f.d[2], f.d[3])), fminf(f.d[4], f.d[5]));
  return m > 0.f;
}
__device__ __forceinline__ float centerness_of(const FaceDist& f) {
  float a = __fdiv_rn(fminf(f.d[0], f.d[1]), fmaxf(f.d[0], f.d[1]));
  float b = __fdiv_rn(fminf(f.d[2], f.d[3]), fmaxf(f.d[2], f.d[3]));
  float c = __fdiv_rn(fminf(f.d[4], f.d[5]), fmaxf(f.d[4], f.d[5]));
  // x_min / x_max * y_min / y_max * z_min / z_max, evaluated left to right
  float t = __fmul_rn(a, fminf(f.d[2], f.d[3]));
  t = __fdiv_rn(t, fmaxf(f.d[2], f.d[3]));
  t = __fmul_rn(t, fminf(f.d[4], f.d[5]));
  t = __fdiv_rn(t, fmaxf(f.d[4], f.d[5]));
  (void)b; (void)c;
  return __fsqrt_rn(t);
}

// All scans of the batch in one pipeline: points of a level are rows of every scan in natural (map) order,
// pt_batch[p] names the scan; boxes of scan b are rows [box_off[b], box_off[b+1]) of the concatenated box arrays.
__device__ __forceinline__ int level_of(const int* __restrict__ level_off, int L, int p) {
  int lvl = 0;
  while (lvl + 1 < L && p >= level_off[lvl + 1]) ++lvl;
  return lvl;
}

// counts[l*NgT + g] = number of level-l points of g's scan inside box g
__global__ void count_inside_kernel(const float* __restrict__ pts, const int* __restrict__ level_off, int L, int Np,
                                    const int* __restrict__ pt_batch, const float* __restrict__ boxes,
                                    const float* __restrict__ rneg, const int* __restrict__ box_off, int NgT,
                                    int* __restrict__ counts) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= Np) return;
  int b = pt_batch ? pt_batch[p] : 0;
  int g = box_off[b] + blockIdx.y;
  if (g >= box_off[b + 1]) return;
  FaceDist f = face_distances(boxes + g * 9, rneg + g * 9, pts[3 * p], pts[3 * p + 1], pts[3 * p + 2]);
  if (inside_box(f)) atomicAdd(&counts[level_of(level_off, L, p) * NgT + g], 1);
}

// best_level[g] per fcaf3d_head.py:1628-1634
__global__ void best_level_kernel(const int* __restrict__ counts, int L, int Ng, int assign_thr, int* __restrict__ best) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= Ng) return;
  int first = -1;
  for (int l = 0; l < L; ++l)
    if (counts[l * Ng + b] < assign_thr) { first = l; break; }
  int lower_index = (first < 0 ? 0 : first) - 1;   // argmax of an all-false mask is 0
  if (lower_index < 0) lower_index = 0;
  best[b] = first < 0 ? L - 1 : lower_index;
}

// top[g] = (k+1)-th largest of the masked centerness column of box g (fcaf3d_head.py:1643-1650), k+1 = kth.
// One CTA per box. Candidates (points of g's scan in g's best level, inside the box) are compacted into shared memory in
// ONE pass over the level; the kth rounds of "next largest in (value desc, index asc) order" then run over that list.
// Boxes with more than TOPK_CAP candidates fall back to rescanning the level each round.
constexpr int TOPK_CAP = 4096;

constexpr int TOPK_THREADS = 1024;

__global__ void __launch_bounds__(TOPK_THREADS)
topk_threshold_kernel(const float* __restrict__ pts, const int* __restrict__ level_off, const int* __restrict__ pt_batch,
                      const int* __restrict__ n_pts_of_scan, const float* __restrict__ boxes,
                      const float* __restrict__ rneg, const int* __restrict__ box_off, int B,
                      const int* __restrict__ best, int kth, float* __restrict__ top) {
  __shared__ float c_val[TOPK_CAP];
  __shared__ int c_idx[TOPK_CAP];
  __shared__ float s_val[TOPK_THREADS];
  __shared__ int s_idx[TOPK_THREADS];
  __shared__ float prev_v;
  __shared__ int prev_i;
  __shared__ int n_cand;
  const int g = blockIdx.x, tid = threadIdx.x;
  int scan = 0;
  while (scan + 1 < B && g >= box_off[scan + 1]) ++scan;
  const int lvl = best[g];
  const int p_beg = level_off[lvl], p_end = level_off[lvl + 1];
  const float* box = boxes + g * 9;
  const float* R = rneg + g * 9;
  const int k_eff = min(kth, n_pts_of_scan[scan]);
  if (tid == 0) { prev_v = INFINITY; prev_i = -1; n_cand = 0; }
  __syncthreads();
  for (int p = p_beg + tid; p < p_end; p += TOPK_THREADS) {
    if (pt_batch && pt_batch[p] != scan) continue;
    FaceDist f = face_distances(box, R, pts[3 * p], pts[3 * p + 1], pts[3 * p + 2]);
    if (!inside_box(f)) continue;
    int slot = atomicAdd(&n_cand, 1);
    if (slot < TOPK_CAP) { c_val[slot] = centerness_of(f); c_idx[slot] = p; }
  }
  __syncthreads();
  const int nc = n_cand;
  if (nc < k_eff) {  // the k-th largest entry is one of the -1 fillers
    if (tid == 0) top[g] = -1.f;
    return;
  }
  const bool in_smem = nc <= TOPK_CAP;
  for (int round = 0; round < k_eff; ++round) {
    float bv = -INFINITY;
    int bi = -1;
    const float pv = prev_v;
    const int pi = prev_i;
    if (in_smem) {
      for (int c = tid; c < nc; c += TOPK_THREADS) {
        float v = c_val[c];
        int p = c_idx[c];
        bool after = (v < pv) || (v == pv && p > pi);
        if (after && (bi < 0 || v > bv || (v == bv && p < bi))) { bv = v; bi = p; }
      }
    } else {
      for (int p = p_beg + tid; p < p_end; p += TOPK_THREADS) {
        if (pt_batch && pt_batch[p] != scan) continue;
        FaceDist f = face_distances(box, R, pts[3 * p], pts[3 * p + 1], pts[3 * p + 2]);
        if (!inside_box(f)) continue;
        float v = centerness_of(f);
        bool after = (v < pv) || (v == pv && p > pi);
        if (after && (bi < 0 || v > bv || (v == bv && p < bi))) { bv = v; bi = p; }
      }
    }
    s_val[tid] = bv;
    s_idx[tid] = bi;
    __syncthreads();
    for (int s = TOPK_THREADS / 2; s > 0; s >>= 1) {
      if (tid < s) {
        float ov = s_val[tid + s];
        int oi = s_idx[tid + s];
        bool take = oi >= 0 && (s_idx[tid] < 0 || ov > s_val[tid] || (ov == s_val[tid] && oi < s_idx[tid]));
        if (take) { s_val[tid] = ov; s_idx[tid] = oi; }
      }
      __syncthreads();
    }
    if (tid == 0) { prev_v = s_val[0]; prev_i = s_idx[0]; }
    __syncthreads();
  }
  if (tid == 0) top[g] = prev_v;
}

// number of points of each scan (torch.topk's `min(k+1, len(centerness))` uses the scan's total point count)
__global__ void count_scan_points_kernel(const int* __restrict__ pt_batch, int Np, int B, int* __restrict__ n_pts_of_scan) {
  __shared__ int hist[64];
  for (int i = threadIdx.x; i < 64; i += blockDim.x) hist[i] = 0;
  __syncthreads();
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < Np) {
    int b = pt_batch ? pt_batch[p] : 0;
    if (b < 64) atomicAdd(&hist[b], 1); else atomicAdd(&n_pts_of_scan[b], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < min(B, 64); i += blockDim.x)
    if (hist[i]) atomicAdd(&n_pts_of_scan[i], hist[i]);
}

// per point: min-volume box among (inside & best level & centerness > top[g]) over the boxes of its scan;
// first index wins ties.
__global__ void assign_kernel(const float* __restrict__ pts, const int* __restrict__ level_off, int L, int Np,
                              const int* __restrict__ pt_batch, const float* __restrict__ boxes,
                              const float* __restrict__ rneg, const long long* __restrict__ labels,
                              const int* __restrict__ box_off, const int* __restrict__ best,
                              const float* __restrict__ top, float* __restrict__ center_t, float* __restrict__ bbox_t,
                              long long* __restrict__ cls_t, int* __restrict__ box_idx) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= Np) return;
  const int lvl = level_of(level_off, L, p);
  const int b = pt_batch ? pt_batch[p] : 0;
  const int g_beg = box_off[b], g_end = box_off[b + 1];
  float px = pts[3 * p], py = pts[3 * p + 1], pz = pts[3 * p + 2];
  const float FMAX = 1e8f;
  float min_vol = FMAX;
  int min_ind = g_beg;
  float cent_sel = -1.f, cent0 = -1.f;
  for (int g = g_beg; g < g_end; ++g) {
    const float* box = boxes + g * 9;
    FaceDist f = face_distances(box, rneg + g * 9, px, py, pz);
    bool in = inside_box(f);
    bool lv = best[g] == lvl;
    float c = (in && lv) ? centerness_of(f) : -1.f;
    if (g == g_beg) cent0 = c;
    if (in && lv && c > top[g]) {
      float vol = __fmul_rn(__fmul_rn(box[3], box[4]), box[5]);
      if (vol < min_vol) { min_vol = vol; min_ind = g; cent_sel = c; }
    }
  }
  bool pos = min_vol < FMAX;
  if (g_end == g_beg) {  // scan without boxes: pseudo targets (fcaf3d_head.py:1601-1605)
    center_t[p] = 0.f;
#pragma unroll
    for (int j = 0; j < 9; ++j) bbox_t[p * 9 + j] = 0.f;
    cls_t[p] = -1;
    if (box_idx) box_idx[p] = -1;
    return;
  }
  // negatives inherit argmin over an all-1e8 row = the scan's first box (reference behaviour; unused by the loss)
  center_t[p] = pos ? cent_sel : cent0;
#pragma unroll
  for (int j = 0; j < 9; ++j) bbox_t[p * 9 + j] = boxes[min_ind * 9 + j];
  cls_t[p] = pos ? labels[min_ind] : -1;
  if (box_idx) box_idx[p] = pos ? min_ind : -1;
}

// ---------------- sigmoid focal loss (mmcv CUDA semantics) ----------------
__device__ __forceinline__ float sigmoidf(float x) { return 1.f / (1.f + expf(-x)); }
// x^gamma with the configured gamma = 2 as a multiply (general powf is ~20x the cost of the rest of the element)
__device__ __forceinline__ float pow_gamma(float x, float gamma) { return gamma == 2.f ? x * x : powf(x, gamma); }

template <typename T>
__global__ void focal_fwd_kernel(const T* __restrict__ logits, const long long* __restrict__ target, long long n, int C,
                                 float gamma, float alpha, const float* __restrict__ row_w, float* __restrict__ loss_sum) {
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  float l = 0.f;
  if (t < n * C) {
    long long r = t / C;
    int c = (int)(t - r * C);
    float p = sigmoidf(esb_to_float<T>(logits[t]));
    if (target[r] == c)
      l = -alpha * pow_gamma(1.f - p, gamma) * logf(fmaxf(p, 1.17549435e-38f));
    else
      l = -(1.f - alpha) * pow_gamma(p, gamma) * logf(fmaxf(1.f - p, 1.17549435e-38f));
    if (row_w) l *= row_w[r];
  }
  l = esb_warp_sum(l);
  __shared__ float red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = l;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += red[i];
    loss_sum[blockIdx.x] = s;                              // one partial per block, summed in block order
  }
}

// grad[t] = scale[0] * dloss/dlogit ; scale is a device scalar (grad_out / avg_factor) so no host sync is needed
template <typename T>
__global__ void focal_bwd_kernel(const T* __restrict__ logits, const long long* __restrict__ target, long long n, int C,
                                 float gamma, float alpha, const float* __restrict__ row_w,
                                 const float* __restrict__ scale, T* __restrict__ grad) {
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t >= n * C) return;
  long long r = t / C;
  int c = (int)(t - r * C);
  float p = sigmoidf(esb_to_float<T>(logits[t]));
  float g;
  if (target[r] == c)
    g = -alpha * pow_gamma(1.f - p, gamma) * (1.f - p - gamma * p * logf(fmaxf(p, 1.17549435e-38f)));
  else
    g = -(1.f - alpha) * pow_gamma(p, gamma) * (gamma * (1.f - p) * logf(fmaxf(1.f - p, 1.17549435e-38f)) - p);
  grad[t] = esb_from_float<T>(g * scale[0] * (row_w ? row_w[r] : 1.f));
}


// ---------------- fused box-regression loss (decode + decoupled corner chamfer), value AND gradient ----------------
// One thread per positive location. Replaces, for the positives of the whole batch, _bbox_pred_to_bbox
// (fcaf3d_head.py:1454-1525: 6 face distances + 6D rotation -> centre/size/Euler ZXY), ortho_6d_2_Mat (:1739-1750),
// pytorch3d matrix_to_euler_angles / euler_angles_to_matrix ('ZXY'), bbox_to_corners (chamfer_distance.py:160-203) and
// the four decoupled BBoxCDLoss terms (fcaf3d_head.py:1224-1281; L1 chamfer, src->dst only) — ~600 tiny launches of
// autograd ops in the reference formulation. The gradient w.r.t. the 12 regression channels is carried by forward-mode
// dual numbers, so the backward pass is a single scale of the stored gradient.
struct Dual {
  float v;
  float d[12];
};
__device__ __forceinline__ Dual dconst(float v) {
  Dual r; r.v = v;
#pragma unroll
  for (int i = 0; i < 12; ++i) r.d[i] = 0.f;
  return r;
}
__device__ __forceinline__ Dual dvar(float v, int idx) { Dual r = dconst(v); r.d[idx] = 1.f; return r; }
__device__ __forceinline__ Dual operator+(const Dual& a, const Dual& b) {
  Dual r; r.v = a.v + b.v;
#pragma unroll
  for (int i = 0; i < 12; ++i) r.d[i] = a.d[i] + b.d[i];
  return r;
}
__device__ __forceinline__ Dual operator-(const Dual& a, const Dual& b) {
  Dual r; r.v = a.v - b.v;
#pragma unroll
  for (int i = 0; i < 12; ++i) r.d[i] = a.d[i] - b.d[i];
  return r;
}
__device__ __forceinline__ Dual operator-(const Dual& a) {
  Dual r; r.v = -a.v;
#pragma unroll
  for (int i = 0; i < 12; ++i) r.d[i] = -a.d[i];
  return r;
}
__device__ __forceinline__ Dual operator*(const Dual& a, const Dual& b) {
  Dual r; r.v = a.v * b.v;
#pragma unroll
  for (int i = 0; i < 12; ++i) r.d[i] = a.d[i] * b.v + a.v * b.d[i];
  return r;
}
__device__ __forceinline__ Dual operator*(const Dual& a, float s) {
  Dual r; r.v = a.v * s;
#pragma unroll
  for (int i = 0; i < 12; ++i) r.d[i] = a.d[i] * s;
  return r;
}
__device__ __forceinline__ Dual operator+(const Dual& a, float s) { Dual r = a; r.v += s; return r; }
__device__ __forceinline__ Dual operator/(const Dual& a, const Dual& b) {
  Dual r;
  float inv = 1.f / b.v;
  r.v = a.v * inv;
#pragma unroll
  for (int i = 0; i < 12; ++i) r.d[i] = (a.d[i] - r.v * b.d[i]) * inv;
  return r;
}
__device__ __forceinline__ Dual dsqrt(const Dual& a) {
  Dual r; r.v = sqrtf(a.v);
  float g = a.v > 0.f ? 0.5f / r.v : 0.f;
#pragma unroll
  for (int i = 0; i < 12; ++i) r.d[i] = a.d[i] * g;
  return r;
}
__device__ __forceinline__ Dual dsin(const Dual& a) { float c = cosf(a.v); Dual r = a * c; r.v = sinf(a.v); return r; }
__device__ __forceinline__ Dual dcos(const Dual& a) { float s = -sinf(a.v); Dual r = a * s; r.v = cosf(a.v); return r; }
__device__ __forceinline__ Dual dasin(const Dual& a) {
  float g = rsqrtf(fmaxf(1.f - a.v * a.v, 1e-12f));
  Dual r = a * g; r.v = asinf(a.v); return r;
}
__device__ __forceinline__ Dual datan2(const Dual& y, const Dual& x) {   // d = (x dy - y dx) / (x^2 + y^2)
  float inv = 1.f / fmaxf(x.v * x.v + y.v * y.v, 1e-30f);
  Dual r; r.v = atan2f(y.v, x.v);
#pragma unroll
  for (int i = 0; i < 12; ++i) r.d[i] = (x.v * y.d[i] - y.v * x.d[i]) * inv;
  return r;
}
struct Dual3 { Dual x, y, z; };
__device__ __forceinline__ Dual3 dcross(const Dual3& a, const Dual3& b) {
  Dual3 r;
  r.x = a.y * b.z - a.z * b.y;
  r.y = a.z * b.x - a.x * b.z;
  r.z = a.x * b.y - a.y * b.x;
  return r;
}
__device__ __forceinline__ Dual3 dnormalize(const Dual3& a) {   // v / (|v| + 1e-8)
  Dual n = dsqrt(a.x * a.x + a.y * a.y + a.z * a.z) + 1e-8f;
  Dual3 r; r.x = a.x / n; r.y = a.y / n; r.z = a.z / n;
  return r;
}
// R = Rz(a) Rx(b) Ry(c) (pytorch3d 'ZXY'), row-major m[9]
__device__ __forceinline__ void euler_to_mat(const Dual& a, const Dual& b, const Dual& c, Dual m[9]) {
  Dual ca = dcos(a), sa = dsin(a), cb = dcos(b), sb = dsin(b), cc = dcos(c), sc = dsin(c);
  Dual a00 = ca, a01 = -(sa * cb), a02 = sa * sb;
  Dual a10 = sa, a11 = ca * cb, a12 = -(ca * sb);
  Dual a21 = sb, a22 = cb;     // a20 = 0
  m[0] = a00 * cc - a02 * sc; m[1] = a01; m[2] = a00 * sc + a02 * cc;
  m[3] = a10 * cc - a12 * sc; m[4] = a11; m[5] = a10 * sc + a12 * cc;
  m[6] = -(a22 * sc);         m[7] = a21; m[8] = a22 * cc;
}
__device__ __forceinline__ void euler_to_mat_f(float a, float b, float c, float m[9]) {
  float ca = cosf(a), sa = sinf(a), cb = cosf(b), sb = sinf(b), cc = cosf(c), sc = sinf(c);
  float a00 = ca, a01 = -sa * cb, a02 = sa * sb, a10 = sa, a11 = ca * cb, a12 = -ca * sb, a21 = sb, a22 = cb;
  m[0] = a00 * cc - a02 * sc; m[1] = a01; m[2] = a00 * sc + a02 * cc;
  m[3] = a10 * cc - a12 * sc; m[4] = a11; m[5] = a10 * sc + a12 * cc;
  m[6] = -a22 * sc;           m[7] = a21; m[8] = a22 * cc;
}
// sum over the 8 corners of min_j L1(src corner, dst corner j); src = (centre, size, euler) duals, dst precomputed
__device__ Dual corner_chamfer(const Dual ctr[3], const Dual size[3], const Dual eul[3], const float dst[24]) {
  Dual m[9];
  euler_to_mat(eul[0], eul[1], eul[2], m);
  Dual total = dconst(0.f);
  const float sx[8] = {1, 1, 1, 1, -1, -1, -1, -1}, sy[8] = {1, 1, -1, -1, 1, 1, -1, -1}, sz[8] = {1, -1, 1, -1, 1, -1, 1, -1};
#pragma unroll 1
  for (int i = 0; i < 8; ++i) {
    Dual hx = size[0] * (0.5f * sx[i]), hy = size[1] * (0.5f * sy[i]), hz = size[2] * (0.5f * sz[i]);
    Dual cx = ctr[0] + (hx * m[0] + hy * m[1] + hz * m[2]);
    Dual cy = ctr[1] + (hx * m[3] + hy * m[4] + hz * m[5]);
    Dual cz = ctr[2] + (hx * m[6] + hy * m[7] + hz * m[8]);
    float best = INFINITY;
    int bj = 0;
    for (int j = 0; j < 8; ++j) {
      float dsum = fabsf(cx.v - dst[3 * j]) + fabsf(cy.v - dst[3 * j + 1]) + fabsf(cz.v - dst[3 * j + 2]);
      if (dsum < best) { best = dsum; bj = j; }
    }
    float gx = cx.v > dst[3 * bj] ? 1.f : (cx.v < dst[3 * bj] ? -1.f : 0.f);
    float gy = cy.v > dst[3 * bj + 1] ? 1.f : (cy.v < dst[3 * bj + 1] ? -1.f : 0.f);
    float gz = cz.v > dst[3 * bj + 2] ? 1.f : (cz.v < dst[3 * bj + 2] ? -1.f : 0.f);
    total.v += best;
#pragma unroll
    for (int q = 0; q < 12; ++q) total.d[q] += gx * cx.d[q] + gy * cy.d[q] + gz * cz.d[q];
  }
  return total;
}

__global__ void __launch_bounds__(64)
bbox_cd_loss_kernel(const float* __restrict__ points, const float* __restrict__ bbox_pred, const float* __restrict__ tgt,
                    const float* __restrict__ row_w, float w0, float w1, float w2, float w3, int P,
                    float* __restrict__ loss_out, float* __restrict__ grad) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  float lval = 0.f;
  if (p < P) {
    Dual in[12];
#pragma unroll
    for (int i = 0; i < 12; ++i) in[i] = dvar(bbox_pred[p * 12 + i], i);
    // decode
    Dual3 shift;
    shift.x = (in[1] - in[0]) * 0.5f; shift.y = (in[3] - in[2]) * 0.5f; shift.z = (in[5] - in[4]) * 0.5f;
    Dual3 xr{in[6], in[7], in[8]}, yr{in[9], in[10], in[11]};
    Dual3 y = dnormalize(yr);
    Dual3 z = dnormalize(dcross(xr, y));
    Dual3 x = dcross(y, z);
    Dual eul[3];
    eul[1] = dasin(y.z);                 // beta  = asin(M[2][1])
    eul[0] = datan2(-y.x, y.y);          // alpha = atan2(-M[0][1], M[1][1])
    eul[2] = datan2(-x.z, z.z);          // gamma = atan2(-M[2][0], M[2][2])
    Dual m[9];
    euler_to_mat(eul[0], eul[1], eul[2], m);
    Dual pc[3], ps[3];
    pc[0] = (shift.x * m[0] + shift.y * m[1] + shift.z * m[2]) + points[3 * p];
    pc[1] = (shift.x * m[3] + shift.y * m[4] + shift.z * m[5]) + points[3 * p + 1];
    pc[2] = (shift.x * m[6] + shift.y * m[7] + shift.z * m[8]) + points[3 * p + 2];
    ps[0] = in[0] + in[1]; ps[1] = in[2] + in[3]; ps[2] = in[4] + in[5];
    // target corners
    const float* t = tgt + p * 9;
    float tm[9], dst[24];
    euler_to_mat_f(t[6], t[7], t[8], tm);
    const float sx[8] = {1, 1, 1, 1, -1, -1, -1, -1}, sy[8] = {1, 1, -1, -1, 1, 1, -1, -1}, sz[8] = {1, -1, 1, -1, 1, -1, 1, -1};
    for (int j = 0; j < 8; ++j) {
      float hx = 0.5f * sx[j] * t[3], hy = 0.5f * sy[j] * t[4], hz = 0.5f * sz[j] * t[5];
      dst[3 * j] = t[0] + hx * tm[0] + hy * tm[1] + hz * tm[2];
      dst[3 * j + 1] = t[1] + hx * tm[3] + hy * tm[4] + hz * tm[5];
      dst[3 * j + 2] = t[2] + hx * tm[6] + hy * tm[7] + hz * tm[8];
    }
    Dual tc[3] = {dconst(t[0]), dconst(t[1]), dconst(t[2])};
    Dual ts[3] = {dconst(t[3]), dconst(t[4]), dconst(t[5])};
    Dual te[3] = {dconst(t[6]), dconst(t[7]), dconst(t[8])};
    Dual acc = dconst(0.f);
    if (w0 != 0.f) acc = acc + corner_chamfer(pc, ts, te, dst) * w0;
    if (w1 != 0.f) acc = acc + corner_chamfer(tc, ps, te, dst) * w1;
    if (w2 != 0.f) acc = acc + corner_chamfer(tc, ts, eul, dst) * w2;
    if (w3 != 0.f) acc = acc + corner_chamfer(pc, ps, eul, dst) * w3;
    float w = row_w[p];
    lval = acc.v * w;
#pragma unroll
    for (int i = 0; i < 12; ++i) grad[p * 12 + i] = acc.d[i] * w;
  }
  lval = esb_warp_sum(lval);
  __shared__ float red[2];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = lval;
  __syncthreads();
  if (threadIdx.x == 0) loss_out[blockIdx.x] = red[0] + red[1];   // one partial per 64-thread block, summed in block order
}

}  // namespace

extern "C" size_t esb_fcaf3d_targets_workspace_bytes(int L, int NgT, int B) {
  return esb_align((size_t)L * NgT * 4) + 2 * esb_align((size_t)NgT * 4) + esb_align((size_t)B * 4);
}

// One launch pipeline for all B scans of the batch.
//  points (Np,3) fp32, level by level (level_off: L+1 device ints); pt_batch (Np) scan of each point (NULL: one scan);
//  boxes (NgT,9) gravity centre/size/euler and rneg (NgT,9) = R(-euler), labels (NgT) int64, concatenated over scans with
//  box_off (B+1) device ints; max_ng = largest per-scan box count (host-known).
//  Outputs: center_t (Np), bbox_t (Np,9), cls_t (Np) int64 (-1 = background), box_idx (Np) global box row or NULL.
extern "C" int esb_fcaf3d_targets(const float* points, const int* level_off, int L, int Np, const int* pt_batch,
                                  const float* boxes, const float* rneg, const long long* labels, const int* box_off,
                                  int B, int NgT, int max_ng, int assign_thr, int center_thr, float* center_t,
                                  float* bbox_t, long long* cls_t, int* box_idx, void* ws, size_t ws_bytes,
                                  void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  ESB_CHECK_ARG(L >= 1 && Np >= 0 && B >= 1 && NgT >= 0, "esb_fcaf3d_targets: bad sizes");
  if (ws_bytes < esb_fcaf3d_targets_workspace_bytes(L, NgT, B)) {
    esb_set_error("esb_fcaf3d_targets: workspace too small");
    return ESB_ENOMEM;
  }
  if (Np == 0) return ESB_OK;
  char* p = (char*)ws;
  int* counts = (int*)p;      p += esb_align((size_t)L * NgT * 4);
  int* best = (int*)p;        p += esb_align((size_t)NgT * 4);
  float* top = (float*)p;     p += esb_align((size_t)NgT * 4);
  int* n_pts_of_scan = (int*)p;
  if (NgT > 0) {
    ESB_CUDA_CALL(cudaMemsetAsync(counts, 0, (size_t)L * NgT * 4, stream));
    ESB_CUDA_CALL(cudaMemsetAsync(n_pts_of_scan, 0, (size_t)B * 4, stream));
    dim3 g1(esb_div_up(Np, 256), max_ng > 0 ? max_ng : 1);
    count_inside_kernel<<<g1, 256, 0, stream>>>(points, level_off, L, Np, pt_batch, boxes, rneg, box_off, NgT, counts);
    count_scan_points_kernel<<<esb_div_up(Np, 1024), 1024, 0, stream>>>(pt_batch, Np, B, n_pts_of_scan);
    best_level_kernel<<<esb_div_up(NgT, 128), 128, 0, stream>>>(counts, L, NgT, assign_thr, best);
    topk_threshold_kernel<<<NgT, TOPK_THREADS, 0, stream>>>(points, level_off, pt_batch, n_pts_of_scan, boxes, rneg, box_off, B,
                                                    best, center_thr + 1, top);
  }
  assign_kernel<<<esb_div_up(Np, 128), 128, 0, stream>>>(points, level_off, L, Np, pt_batch, boxes, rneg, labels, box_off,
                                                          best, top, center_t, bbox_t, cls_t, box_idx);
  ESB_CUDA_LAUNCH_CHECK("esb_fcaf3d_targets");
  return ESB_OK;
}

// loss_sum: device fp32 scalar, accumulated (caller zeroes). logits (n,C) row-major.
// row_w: optional (n) per-row weight (e.g. 1 / n_pos of the row's scan)
extern "C" int esb_focal_loss_fwd(const void* logits, const long long* target, long long n, int C, float gamma,
                                  float alpha, const float* row_w, float* loss_sum, int dtype, void* stream) {
  if (n == 0) return ESB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  int grid = esb_div_up(n * C, 256);
  float* part = nullptr;
  ESB_CUDA_CALL(esb_scratch_alloc((void**)&part, (size_t)grid * sizeof(float), s));
  if (dtype == ESB_F32)
    focal_fwd_kernel<float><<<grid, 256, 0, s>>>((const float*)logits, target, n, C, gamma, alpha, row_w, part);
  else
    focal_fwd_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>((const __nv_bfloat16*)logits, target, n, C, gamma, alpha, row_w, part);
  ESB_CUDA_LAUNCH_CHECK("focal_fwd_kernel");
  int rc = esb_sum_partial_rows(part, grid, 1, loss_sum, 1, s);
  ESB_CUDA_CALL(esb_scratch_free(part, s));
  return rc;
}

extern "C" int esb_focal_loss_bwd(const void* logits, const long long* target, long long n, int C, float gamma,
                                  float alpha, const float* row_w, const float* scale_dev, void* grad, int dtype,
                                  void* stream) {
  if (n == 0) return ESB_OK;
  int grid = esb_div_up(n * C, 256);
  if (dtype == ESB_F32)
    focal_bwd_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>((const float*)logits, target, n, C, gamma, alpha,
                                                                     row_w, scale_dev, (float*)grad);
  else
    focal_bwd_kernel<__nv_bfloat16><<<grid, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)logits, target, n, C, gamma,
                                                                             alpha, row_w, scale_dev, (__nv_bfloat16*)grad);
  ESB_CUDA_LAUNCH_CHECK("focal_bwd_kernel");
  return ESB_OK;
}

// Fused decode + decoupled corner-chamfer box loss over P positives:
//   loss_out (device fp32, accumulated; caller zeroes) = sum_p row_w[p] * sum_v w[v] * sum_{8 corners} min_j L1
//   grad (P,12) = d loss / d bbox_pred. Variants v: (pred centre), (pred size), (pred euler), (all predicted).
extern "C" int esb_bbox_cd_loss(const float* points, const float* bbox_pred, const float* targets, const float* row_w,
                                const float* w4_host, int P, float* loss_out, float* grad, void* stream) {
  if (P == 0) return ESB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const int grid = esb_div_up(P, 64);
  float* part = nullptr;
  ESB_CUDA_CALL(esb_scratch_alloc((void**)&part, (size_t)grid * sizeof(float), s));
  bbox_cd_loss_kernel<<<grid, 64, 0, s>>>(points, bbox_pred, targets, row_w, w4_host[0], w4_host[1], w4_host[2], w4_host[3], P,
                                          part, grad);
  ESB_CUDA_LAUNCH_CHECK("bbox_cd_loss_kernel");
  int rc = esb_sum_partial_rows(part, grid, 1, loss_out, 1, s);
  ESB_CUDA_CALL(esb_scratch_free(part, s));
  return rc;
}
