// esb200 — differentiable rotated 3D IoU of one-to-one box pairs: mmcv.ops.diff_iou_rotated_3d (mmcv 2.0.0rc4,
// †upstream) as RotatedIoU3DLoss calls it (embodiedscan/models/losses/rotated_iou_loss.py:14-91). Boxes are rows
// (x, y, z, w, l, h, alpha, ...) with z the box centre; columns past 7 are ignored.
//
// Per pair, one thread:
//   BEV corners (+-w/2, +-l/2) in the order (+,+), (-,+), (-,-), (+,-), rotated counter-clockwise by alpha;
//   24 candidate vertices: A's corners inside B (0-3), B's corners inside A (4-7), the intersections of A's edge i with
//   B's edge j (8 + 4 i + j, strict 0 < t, u < 1, parallel edges none); the inside test keeps normalised projections on
//   the two edges from corner 0 inside (-1e-6, 1 + 1e-6);
//   the valid vertices sorted by angle about their mean (stable: equal angles keep candidate order), the shoelace area
//   of that cycle (0 below 3 vertices);
//   inter = area * clamp(min(top) - max(bottom), 0), iou = inter / (Va + Vb - inter), no epsilon.
// The backward recomputes the geometry and applies the chain rule by hand: shoelace -> vertices -> corners (a corner
// vertex) or the four edge end points (an intersection, a rational function of them) -> (x, y, w, l, alpha); z overlap
// and volumes -> (z, h, w, l). The sort order is not differentiated. At ties of min / max the gradient is split in half
// and clamp passes it at exactly 0, as torch autograd does.
//
// Geometry runs in coordinates relative to A's centre (x, y and z), so fp32 never cancels metres against centimetres.
// The candidates and the sort live in a per-thread local array (24 x 13 B); every output of a pair is written by its
// own thread, with no atomics and no cross-thread sums, so the results are bit-reproducible.
#include "common.cuh"

namespace {

constexpr int kCand = 24;

// Every quotient uses the fast division (2 ulp, far inside the IoU bound): the IEEE division's slow-path subroutine
// makes the backward kernel save registers to local memory around its calls.
#ifdef __CUDA_ARCH__
#define FDIV(x, y) __fdividef(x, y)
#else
#define FDIV(x, y) ((x) / (y))
#endif
constexpr int kThreads = 128;

struct Pair {
  float ca[4][2], cb[4][2];  // BEV corners, relative to A's centre
  float ra[4][2], rb[4][2];  // corner offsets from their own box's centre (rotated half extents)
  float sa, ca_, sb, cb_;    // sin / cos of the two yaws
};

struct Poly {
  int n;
  float x[kCand], y[kCand], ang[kCand];
  unsigned char id[kCand];
};

__host__ __device__ __forceinline__ void corners(float cx, float cy, float w, float l, float s, float c,
                                                 float off[4][2], float out[4][2]) {
  const float sx[4] = {0.5f, -0.5f, -0.5f, 0.5f}, sy[4] = {0.5f, 0.5f, -0.5f, -0.5f};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float px = sx[k] * w, py = sy[k] * l;
    off[k][0] = px * c - py * s;
    off[k][1] = px * s + py * c;
    out[k][0] = cx + off[k][0];
    out[k][1] = cy + off[k][1];
  }
}

__host__ __device__ __forceinline__ bool inside(const float p[2], const float q[4][2]) {
  const float abx = q[1][0] - q[0][0], aby = q[1][1] - q[0][1];
  const float adx = q[3][0] - q[0][0], ady = q[3][1] - q[0][1];
  const float amx = p[0] - q[0][0], amy = p[1] - q[0][1];
  // projection / |edge|^2 in (-1e-6, 1 + 1e-6), multiplied out (a zero-length edge admits nothing, as its NaN would)
  const float pab = abx * amx + aby * amy, nab = abx * abx + aby * aby;
  const float pad = adx * amx + ady * amy, nad = adx * adx + ady * ady;
  return pab > -1e-6f * nab && pab < (1.f + 1e-6f) * nab && pad > -1e-6f * nad && pad < (1.f + 1e-6f) * nad;
}

// edge p1 -> p2 of A against edge p3 -> p4 of B: t along A's edge, or false
__host__ __device__ __forceinline__ bool intersect(const float p1[2], const float p2[2], const float p3[2],
                                                   const float p4[2], float* t_out) {
  const float num = (p1[0] - p2[0]) * (p3[1] - p4[1]) - (p1[1] - p2[1]) * (p3[0] - p4[0]);
  if (num == 0.f) return false;
  const float t = FDIV((p1[0] - p3[0]) * (p3[1] - p4[1]) - (p1[1] - p3[1]) * (p3[0] - p4[0]), num);
  const float u = -FDIV((p1[0] - p2[0]) * (p1[1] - p3[1]) - (p1[1] - p2[1]) * (p1[0] - p3[0]), num);
  *t_out = t;
  return t > 0.f && t < 1.f && u > 0.f && u < 1.f;
}

__host__ __device__ __forceinline__ void setup(const float* a, const float* b, Pair& g) {
  sincosf(a[6], &g.sa, &g.ca_);
  sincosf(b[6], &g.sb, &g.cb_);
  corners(0.f, 0.f, a[3], a[4], g.sa, g.ca_, g.ra, g.ca);
  corners(b[0] - a[0], b[1] - a[1], b[3], b[4], g.sb, g.cb_, g.rb, g.cb);
}

// the valid candidates, sorted by angle about their mean; returns the signed shoelace sum (twice the signed area)
__host__ __device__ __forceinline__ float polygon(const Pair& g, Poly& poly) {
  int n = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (inside(g.ca[k], g.cb)) {
      poly.x[n] = g.ca[k][0]; poly.y[n] = g.ca[k][1]; poly.id[n] = (unsigned char)k; ++n;
    }
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (inside(g.cb[k], g.ca)) {
      poly.x[n] = g.cb[k][0]; poly.y[n] = g.cb[k][1]; poly.id[n] = (unsigned char)(4 + k); ++n;
    }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float* p1 = g.ca[i];
      const float* p2 = g.ca[(i + 1) & 3];
      float t;
      if (intersect(p1, p2, g.cb[j], g.cb[(j + 1) & 3], &t)) {
        poly.x[n] = p1[0] + t * (p2[0] - p1[0]);
        poly.y[n] = p1[1] + t * (p2[1] - p1[1]);
        poly.id[n] = (unsigned char)(8 + 4 * i + j);
        ++n;
      }
    }
  poly.n = n;
  if (n < 3) return 0.f;
  float mx = 0.f, my = 0.f;
  for (int k = 0; k < n; ++k) { mx += poly.x[k]; my += poly.y[k]; }
  mx = FDIV(mx, (float)n);
  my = FDIV(my, (float)n);
  // sort key: a pseudo-angle, strictly increasing with the angle about the mean over [-pi/2, 3pi/2): the cyclic order
  // of atan2 (only the cycle's starting vertex may differ, which changes neither the area nor its gradient)
  for (int k = 0; k < n; ++k) {
    const float dx = poly.x[k] - mx, dy = poly.y[k] - my;
    const float r = FDIV(dy, fabsf(dx) + fabsf(dy));
    poly.ang[k] = dx < 0.f ? 2.f - r : r;
  }
  // insertion sort, strict comparison: equal angles keep candidate order
  for (int k = 1; k < n; ++k) {
    const float ak = poly.ang[k], xk = poly.x[k], yk = poly.y[k];
    const unsigned char ik = poly.id[k];
    int m = k - 1;
    while (m >= 0 && poly.ang[m] > ak) {
      poly.ang[m + 1] = poly.ang[m]; poly.x[m + 1] = poly.x[m]; poly.y[m + 1] = poly.y[m]; poly.id[m + 1] = poly.id[m];
      --m;
    }
    poly.ang[m + 1] = ak; poly.x[m + 1] = xk; poly.y[m + 1] = yk; poly.id[m + 1] = ik;
  }
  float s = 0.f;
  for (int k = 0; k < n; ++k) {
    const int k1 = k + 1 == n ? 0 : k + 1;
    s += poly.x[k] * poly.y[k1] - poly.y[k] * poly.x[k1];
  }
  return s;
}

struct ZOverlap {
  float d;      // min(top) - max(bottom), before the clamp
  float wa_top; // share of A in the min of the tops: 1, 0.5 (tie) or 0
  float wa_bot; // share of A in the max of the bottoms
};

__host__ __device__ __forceinline__ ZOverlap z_overlap(const float* a, const float* b) {
  const float dz = b[2] - a[2];
  const float at = 0.5f * a[5], ab = -0.5f * a[5];
  const float bt = dz + 0.5f * b[5], bb = dz - 0.5f * b[5];
  ZOverlap z;
  z.wa_top = at < bt ? 1.f : (at == bt ? 0.5f : 0.f);
  z.wa_bot = ab > bb ? 1.f : (ab == bb ? 0.5f : 0.f);
  z.d = fminf(at, bt) - fmaxf(ab, bb);
  return z;
}

__host__ __device__ __forceinline__ float pair_iou(const float* a, const float* b) {
  Pair g;
  Poly poly;
  setup(a, b, g);
  const float area = 0.5f * fabsf(polygon(g, poly));
  const ZOverlap z = z_overlap(a, b);
  const float inter = area * fmaxf(z.d, 0.f);
  return FDIV(inter, a[3] * a[4] * a[5] + b[3] * b[4] * b[5] - inter);
}

// corner gradients gc -> (x, y, z, w, l, h, alpha) of one box; wt / wb: its share in min(top) / max(bottom)
__host__ __device__ __forceinline__ void box_grad(const float* bx, const float gc[4][2], const float r[4][2], float sn,
                                                  float cs, float g_d, float wt, float wb, float g_vol, float* out) {
  const float sx[4] = {0.5f, -0.5f, -0.5f, 0.5f}, sy[4] = {0.5f, 0.5f, -0.5f, -0.5f};
  float gx = 0.f, gy = 0.f, gw = 0.f, gl = 0.f, gal = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    gx += gc[k][0];
    gy += gc[k][1];
    gw += sx[k] * (gc[k][0] * cs + gc[k][1] * sn);
    gl += sy[k] * (gc[k][1] * cs - gc[k][0] * sn);
    gal += gc[k][1] * r[k][0] - gc[k][0] * r[k][1];
  }
  out[0] = gx;
  out[1] = gy;
  out[2] = g_d * (wt - wb);
  out[3] = gw + g_vol * bx[4] * bx[5];
  out[4] = gl + g_vol * bx[3] * bx[5];
  out[5] = g_d * 0.5f * (wt + wb) + g_vol * bx[3] * bx[4];
  out[6] = gal;
}

// d iou / d (x, y, z, w, l, h, alpha) of both boxes, scaled by g_iou; gb may be null
__host__ __device__ __forceinline__ void pair_iou_grad(const float* a, const float* b, float g_iou, float* ga,
                                                       float* gb) {
  Pair g;
  Poly poly;
  setup(a, b, g);
  const float s = polygon(g, poly);
  const float area = 0.5f * fabsf(s);
  const ZOverlap z = z_overlap(a, b);
  const float ov = fmaxf(z.d, 0.f);
  const float inter = area * ov;
  const float va = a[3] * a[4] * a[5], vb = b[3] * b[4] * b[5];
  const float uni = va + vb - inter;
  const float inv_u2 = FDIV(1.f, uni * uni);
  const float g_inter = g_iou * (va + vb) * inv_u2;  // d(I/U)/dI with U = Va + Vb - I
  const float g_vol = -g_iou * inter * inv_u2;
  const float g_area = g_inter * ov;
  const float g_d = z.d >= 0.f ? g_inter * area : 0.f;

  float gca[4][2] = {}, gcb[4][2] = {};
  const int n = poly.n;
  if (n >= 3 && s != 0.f) {
    const float gs = g_area * (s > 0.f ? 0.5f : -0.5f);
    for (int k = 0; k < n; ++k) {
      const int kn = k + 1 == n ? 0 : k + 1, kp = k == 0 ? n - 1 : k - 1;
      const float gx = gs * (poly.y[kn] - poly.y[kp]);
      const float gy = gs * (poly.x[kp] - poly.x[kn]);
      const int id = poly.id[k];
      if (id < 4) {
        gca[id][0] += gx; gca[id][1] += gy;
      } else if (id < 8) {
        gcb[id - 4][0] += gx; gcb[id - 4][1] += gy;
      } else {
        const int i = (id - 8) >> 2, j = (id - 8) & 3, i1 = (i + 1) & 3, j1 = (j + 1) & 3;
        const float x1 = g.ca[i][0], y1 = g.ca[i][1], x2 = g.ca[i1][0], y2 = g.ca[i1][1];
        const float x3 = g.cb[j][0], y3 = g.cb[j][1], x4 = g.cb[j1][0], y4 = g.cb[j1][1];
        const float num = (x1 - x2) * (y3 - y4) - (y1 - y2) * (x3 - x4);
        const float t = FDIV((x1 - x3) * (y3 - y4) - (y1 - y3) * (x3 - x4), num);
        // P = p1 + t (p2 - p1), t = N / D
        const float gt = gx * (x2 - x1) + gy * (y2 - y1);
        const float gN = FDIV(gt, num), gD = -gN * t;
        gca[i][0] += (1.f - t) * gx + gN * (y3 - y4) + gD * (y3 - y4);
        gca[i][1] += (1.f - t) * gy - gN * (x3 - x4) - gD * (x3 - x4);
        gca[i1][0] += t * gx - gD * (y3 - y4);
        gca[i1][1] += t * gy + gD * (x3 - x4);
        gcb[j][0] += gN * (y4 - y1) - gD * (y1 - y2);
        gcb[j][1] += gN * (x1 - x4) + gD * (x1 - x2);
        gcb[j1][0] += gN * (y1 - y3) + gD * (y1 - y2);
        gcb[j1][1] += -gN * (x1 - x3) - gD * (x1 - x2);
      }
    }
  }

  box_grad(a, gca, g.ra, g.sa, g.ca_, g_d, z.wa_top, z.wa_bot, g_vol, ga);
  if (gb != nullptr) box_grad(b, gcb, g.rb, g.sb, g.cb_, g_d, 1.f - z.wa_top, 1.f - z.wa_bot, g_vol, gb);
}

__global__ void __launch_bounds__(kThreads) rotated_iou3d_fwd_kernel(const float* __restrict__ a, int lda,
                                                                     const float* __restrict__ b, int ldb, long long n,
                                                                     float* __restrict__ iou) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  float ra[7], rb[7];
#pragma unroll
  for (int c = 0; c < 7; ++c) {
    ra[c] = a[p * lda + c];
    rb[c] = b[p * ldb + c];
  }
  iou[p] = pair_iou(ra, rb);
}

__global__ void __launch_bounds__(kThreads) rotated_iou3d_bwd_kernel(const float* __restrict__ a, int lda,
                                                                     const float* __restrict__ b, int ldb, long long n,
                                                                     const float* __restrict__ grad_iou,
                                                                     float* __restrict__ grad_a,
                                                                     float* __restrict__ grad_b) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  float ra[7], rb[7], ga[7], gb[7];
#pragma unroll
  for (int c = 0; c < 7; ++c) {
    ra[c] = a[p * lda + c];
    rb[c] = b[p * ldb + c];
  }
  pair_iou_grad(ra, rb, grad_iou[p], ga, grad_b != nullptr ? gb : nullptr);
#pragma unroll
  for (int c = 0; c < 7; ++c) grad_a[p * 7 + c] = ga[c];
  if (grad_b != nullptr) {
#pragma unroll
    for (int c = 0; c < 7; ++c) grad_b[p * 7 + c] = gb[c];
  }
}

}  // namespace


extern "C" int esb_rotated_iou3d_fwd(const float* a, int lda, const float* b, int ldb, long long n, float* iou,
                                     void* stream) {
  ESB_CHECK_ARG(lda >= 7 && ldb >= 7, "esb_rotated_iou3d_fwd: row strides must be >= 7, got %d and %d", lda, ldb);
  ESB_CHECK_ARG(n >= 0, "esb_rotated_iou3d_fwd: negative pair count %lld", n);
  if (n == 0) return ESB_OK;
  rotated_iou3d_fwd_kernel<<<esb_div_up(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(a, lda, b, ldb, n, iou);
  ESB_CUDA_LAUNCH_CHECK("rotated_iou3d_fwd_kernel");
  return ESB_OK;
}

extern "C" int esb_rotated_iou3d_bwd(const float* a, int lda, const float* b, int ldb, long long n,
                                     const float* grad_iou, float* grad_a, float* grad_b, void* stream) {
  ESB_CHECK_ARG(lda >= 7 && ldb >= 7, "esb_rotated_iou3d_bwd: row strides must be >= 7, got %d and %d", lda, ldb);
  ESB_CHECK_ARG(n >= 0, "esb_rotated_iou3d_bwd: negative pair count %lld", n);
  if (n == 0) return ESB_OK;
  rotated_iou3d_bwd_kernel<<<esb_div_up(n, kThreads), kThreads, 0, (cudaStream_t)stream>>>(a, lda, b, ldb, n, grad_iou,
                                                                                          grad_a, grad_b);
  ESB_CUDA_LAUNCH_CHECK("rotated_iou3d_bwd_kernel");
  return ESB_OK;
}
