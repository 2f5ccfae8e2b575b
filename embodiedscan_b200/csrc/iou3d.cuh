// esb200 — device arithmetic of the exact 9-DoF box intersection, shared by esb_box3d_overlap (iou3d.cu) and the 3D-IoU
// NMS (nms3d.cu) so that both decide every pair with the same instructions.
//
// Intersection of two convex boxes by polygon clipping + the divergence theorem: the faces of A∩B are the faces of A
// clipped by B's six half-spaces plus the faces of B clipped (strictly) by A's, and
//     V = 1/3 * sum_faces (n_f . p_f) * area_f        (coordinates relative to A's centre).
// Strict clipping on one side keeps coplanar faces from being counted twice (identical boxes give IoU 1).
#pragma once
#include "common.cuh"

namespace {

struct V3 { float x, y, z; };
__device__ __forceinline__ V3 operator-(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ V3 operator+(V3 a, V3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ V3 operator*(V3 a, float s) { return {a.x * s, a.y * s, a.z * s}; }
__device__ __forceinline__ float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ V3 cross(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }

struct Box {
  V3 c;        // centre
  V3 n[3];     // unit axes
  float h[3];  // half extents
};

// corner order of EulerInstance3DBoxes.corners: unravel(2,2,2)[[0,1,3,2,4,5,7,6]] - 0.5
//   0:(0,0,0) 1:(0,0,1) 2:(0,1,1) 3:(0,1,0) 4:(1,0,0) 5:(1,0,1) 6:(1,1,1) 7:(1,1,0)
__device__ Box box_from_corners(const float* k, V3 origin) {
  V3 p[8];
  V3 c{0.f, 0.f, 0.f};
  for (int i = 0; i < 8; ++i) {
    p[i] = V3{k[3 * i], k[3 * i + 1], k[3 * i + 2]} - origin;
    c = c + p[i];
  }
  Box b;
  b.c = c * 0.125f;
  V3 e[3] = {p[4] - p[0], p[3] - p[0], p[1] - p[0]};
  for (int a = 0; a < 3; ++a) {
    float len = sqrtf(dot(e[a], e[a]));
    b.h[a] = 0.5f * len;
    b.n[a] = e[a] * (len > 0.f ? 1.f / len : 0.f);
  }
  return b;
}

constexpr int MAXV = 16;

// clip convex polygon by the half-space n.x <= d (strict: n.x < d)
__device__ int clip(const V3* in, int n_in, V3 n, float d, bool strict, V3* out) {
  int n_out = 0;
  for (int i = 0; i < n_in; ++i) {
    V3 a = in[i], b = in[(i + 1) % n_in];
    float da = dot(n, a) - d, db = dot(n, b) - d;
    bool ina = strict ? da < -1e-7f : da <= 1e-7f;
    bool inb = strict ? db < -1e-7f : db <= 1e-7f;
    if (ina) out[n_out++] = a;
    if (ina != inb) {
      float t = da / (da - db);
      out[n_out++] = a + (b - a) * t;
    }
    if (n_out >= MAXV - 1) break;
  }
  return n_out;
}

// contribution of the faces of P clipped by Q to 3 * volume
__device__ float faces_clipped(const Box& P, const Box& Q, bool strict) {
  float acc = 0.f;
  for (int a = 0; a < 3; ++a)
    for (int sgn = -1; sgn <= 1; sgn += 2) {
      V3 n = P.n[a] * (float)sgn;
      V3 fc = P.c + n * P.h[a];
      V3 u = P.n[(a + 1) % 3] * P.h[(a + 1) % 3], v = P.n[(a + 2) % 3] * P.h[(a + 2) % 3];
      V3 poly[MAXV], tmp[MAXV];
      poly[0] = fc - u - v; poly[1] = fc + u - v; poly[2] = fc + u + v; poly[3] = fc - u + v;
      int np = 4;
      for (int b = 0; b < 3 && np > 0; ++b)
        for (int s2 = -1; s2 <= 1 && np > 0; s2 += 2) {
          V3 m = Q.n[b] * (float)s2;
          float d = dot(m, Q.c) + Q.h[b];
          np = clip(poly, np, m, d, strict, tmp);
          for (int i = 0; i < np; ++i) poly[i] = tmp[i];
        }
      if (np < 3) continue;
      V3 av{0.f, 0.f, 0.f};
      for (int i = 1; i + 1 < np; ++i) av = av + cross(poly[i] - poly[0], poly[i + 1] - poly[0]);
      float area = 0.5f * fabsf(dot(av, n));
      acc += dot(n, fc) * area;
    }
  return acc;
}

// corners ka, kb (8,3) in the container's corner order -> intersection volume and IoU of the pair
__device__ void box3d_pair_overlap(const float* ka, const float* kb, float* vol, float* iou) {
  V3 origin{0.f, 0.f, 0.f};
  for (int q = 0; q < 8; ++q) origin = origin + V3{ka[3 * q], ka[3 * q + 1], ka[3 * q + 2]};
  origin = origin * 0.125f;                       // work relative to A's centre: small numbers in the divergence sum
  Box A = box_from_corners(ka, origin), B = box_from_corners(kb, origin);
  float va = 8.f * A.h[0] * A.h[1] * A.h[2], vb = 8.f * B.h[0] * B.h[1] * B.h[2];
  // quick reject: centre distance vs bounding spheres
  V3 dc = B.c - A.c;
  float ra = sqrtf(A.h[0] * A.h[0] + A.h[1] * A.h[1] + A.h[2] * A.h[2]);
  float rb = sqrtf(B.h[0] * B.h[0] + B.h[1] * B.h[1] + B.h[2] * B.h[2]);
  float v = 0.f;
  if (dot(dc, dc) < (ra + rb) * (ra + rb)) {
    v = (faces_clipped(A, B, false) + faces_clipped(B, A, true)) * (1.f / 3.f);
    v = fminf(fmaxf(v, 0.f), fminf(va, vb));
  }
  *vol = v;
  *iou = v / fmaxf(va + vb - v, 1e-12f);
}

}  // namespace
