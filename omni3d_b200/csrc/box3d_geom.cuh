// box3d_geom.cuh — per-lane geometry of the oriented-box 3D IoU (sm_90a device code; the
// functions are __host__ __device__ so tests/csrc/geom_host_harness.cpp can run them on the
// CPU and compare bit-for-bit with the oracle without a GPU).
//
// Replaces the arithmetic of pytorch3d._C.iou_box3d as the reference calls it at
// cubercnn/evaluation/omni3d_evaluation.py:155 (triangle-vs-plane clipping, coplanar de-dup,
// tetrahedral volume).  All predicates are evaluated with the same fp32 operation order as the
// serial CPU algorithm and this translation unit is compiled with -fmad=false, so the integer
// face counts — and in fact vol/iou — are bit-identical to the CPU path.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define C3D_HD __host__ __device__ __forceinline__
#else
#define C3D_HD static inline
#endif

namespace c3d {

constexpr float kEps = 1e-8f;   // kEpsilon
constexpr float dEps = 1e-3f;   // coplanarity
constexpr float aEps = 1e-4f;   // area

struct V3 { float x, y, z; };
struct Tri { V3 a, b, c; };

C3D_HD V3 mk(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
C3D_HD V3 operator+(V3 a, V3 b) { return mk(a.x + b.x, a.y + b.y, a.z + b.z); }
C3D_HD V3 operator-(V3 a, V3 b) { return mk(a.x - b.x, a.y - b.y, a.z - b.z); }
C3D_HD V3 operator*(float s, V3 a) { return mk(s * a.x, s * a.y, s * a.z); }
C3D_HD V3 operator/(V3 a, float s) { return mk(a.x / s, a.y / s, a.z / s); }
C3D_HD float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
C3D_HD V3 cross(V3 a, V3 b) {
  return mk(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
C3D_HD float norm(V3 a) { return sqrtf(dot(a, a)); }
C3D_HD V3 unit_normal(V3 e0, V3 e1) {
  V3 n = cross(e0, e1);
  return n / fmaxf(norm(n), kEps);
}

// box topology (corner order of DATA.md:109-131 / math_util.py:151-167), packed 4 bits per index
//   planes: {0,1,2,3},{3,2,6,7},{0,1,5,4},{0,3,7,4},{1,2,6,5},{4,5,6,7}
//   tris  : {0,1,2},{0,3,2},{4,5,6},{4,6,7},{1,5,6},{1,6,2},{0,4,7},{0,7,3},{3,2,6},{3,6,7},{0,1,5},{0,4,5}
C3D_HD int plane_vert(int p, int k) {
  const uint32_t T[6] = {0x3210u, 0x7623u, 0x4510u, 0x4730u, 0x5621u, 0x7654u};
  return (T[p] >> (4 * k)) & 0xF;
}
C3D_HD int tri_vert(int t, int k) {
  const uint32_t T[12] = {0x210u, 0x230u, 0x654u, 0x764u, 0x651u, 0x261u,
                          0x740u, 0x370u, 0x623u, 0x763u, 0x510u, 0x540u};
  return (T[t] >> (4 * k)) & 0xF;
}

// unit normal of a triangle from the best-conditioned pair of (vertex - centroid); first max wins
C3D_HD V3 tri_normal(const Tri& t) {
  V3 ctr = ((t.a + t.b) + t.c) / 3.0f;
  V3 a = t.a - ctr, b = t.b - ctr, c = t.c - ctr;
  float d01 = norm(cross(a, b)), d02 = norm(cross(a, c)), d12 = norm(cross(b, c));
  // sequence (0,1),(0,2),(1,2) with strict '>' against a running max starting at -1
  V3 e0 = a, e1 = b; float m = d01;
  if (d02 > m) { m = d02; e0 = a; e1 = c; }
  if (d12 > m) { m = d12; e0 = b; e1 = c; }
  return unit_normal(e0, e1);
}

// inward unit normal + centre of one box face (4 verts), oriented toward box centre `bc`
C3D_HD void plane_from_quad(V3 q0, V3 q1, V3 q2, V3 q3, V3 bc, V3* pc_out, V3* n_out) {
  V3 pc = (((q0 + q1) + q2) + q3) / 4.0f;
  V3 e[4] = {q0 - pc, q1 - pc, q2 - pc, q3 - pc};
  V3 n = mk(0.f, 0.f, 0.f);
  float m = -1.0f;
  for (int i = 0; i < 3; ++i)
    for (int j = i + 1; j < 4; ++j) {
      float d = norm(cross(e[i], e[j]));
      if (d > m) { m = d; n = unit_normal(e[i], e[j]); }
    }
  float c = dot(bc - pc, n);
  if (c < 0.0f) n = -1.0f * n;
  *pc_out = pc; *n_out = n;
}

C3D_HD V3 plane_edge_intersection(V3 pc, V3 n, V3 p0, V3 p1) {
  // The reference normalises the edge direction only to test |dot(direc, n)| >= dEps (edge not parallel to the plane).
  // Conservative shortcut with the outcome of that test unchanged: with dd = p1 - p0, bot = dot(dd, n) and |n| = 1 the
  // tested quantity is |bot| / |dd| up to a few ulp (~1e-6 absolute); when bot^2 >= 4e-6 |dd|^2 (|bot|/|dd| >= 2e-3, twice
  // the threshold) and |dd| is far above kEps, the exact evaluation is certainly >= 1e-3 and the square root + three
  // divisions are skipped; everything closer to the threshold takes the reference's arithmetic.
  V3 dd = p1 - p0;
  float bot = dot(dd, n);
  float len2 = dot(dd, dd);
  bool not_parallel;
  if (len2 > 1e-12f && bot * bot >= 4e-6f * len2) {
    not_parallel = true;
  } else {
    V3 direc = dd / fmaxf(norm(dd), kEps);
    not_parallel = fabsf(dot(direc, n)) >= dEps;
  }
  V3 p = (p1 + p0) / 2.0f;
  if (not_parallel) {
    float top = -1.0f * dot(p0 - pc, n);
    float a = top / bot;
    p = p0 + a * dd;
  }
  return p;
}

// Full "triangle coplanar with box face" test (tri normal ‖ plane normal, and the most distant
// tri/face vertex pair lies in the plane).  q = the face's 4 vertices.
C3D_HD bool coplanar_tri_plane_full(const Tri& t, const V3* q, V3 n) {
  V3 nt = tri_normal(t);
  bool check1 = fabsf(dot(nt, n)) > 1.0f - dEps;
  if (!check1) return false;
  const V3 tv[3] = {t.a, t.b, t.c};
  float best = -1.0f; int bi = 0, bj = 0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j) {
      V3 d = tv[i] - q[j];
      float dist = dot(d, d);
      if (dist > best) { best = dist; bi = i; bj = j; }
    }
  V3 d = tv[bi] - q[bj];
  d = d / fmaxf(norm(d), kEps);
  return fabsf(dot(d, n)) < dEps;
}

// Conservative reject for the test above: true => provably NOT coplanar (check1 fails with a
// wide margin on a well-conditioned triangle), so the expensive path can be skipped without
// changing the outcome.  cos^2 threshold 0.98 vs the real 0.998; conditioning guard keeps the
// rounding of the reference's normal far inside that margin.
C3D_HD bool surely_not_parallel(const Tri& t, V3 n) {
  V3 e1 = t.b - t.a, e2 = t.c - t.a, e3 = t.c - t.b;
  V3 N = cross(e1, e2);
  float NN = dot(N, N);
  float L2 = fmaxf(fmaxf(dot(e1, e1), dot(e2, e2)), dot(e3, e3));
  float C2 = fmaxf(fmaxf(dot(t.a, t.a), dot(t.b, t.b)), dot(t.c, t.c));
  float dn = dot(N, n);
  return (NN > 1e-6f * (C2 + L2) * L2) && (dn * dn < 0.98f * NN);
}

// Sutherland–Hodgman step for ONE triangle against ONE inward-oriented face plane.
// Returns the number of output triangles (0,1,2) written to o0,o1 (order as the CPU algorithm).
C3D_HD int clip_tri(const Tri& t, V3 pc, V3 n, const V3* q, Tri* o0, Tri* o1) {
  bool cop = surely_not_parallel(t, n) ? false : coplanar_tri_plane_full(t, q, n);
  bool in0 = dot(t.a - pc, n) >= 0.0f;
  bool in1 = dot(t.b - pc, n) >= 0.0f;
  bool in2 = dot(t.c - pc, n) >= 0.0f;
  int nin = (int)in0 + (int)in1 + (int)in2;
  if (cop || nin == 3) { *o0 = t; return 1; }
  if (nin == 0) return 0;
  // nin == 2, one vertex out:  (vout, vin1, vin2) = (v2,v0,v1) | (v1,v0,v2) | (v0,v1,v2); p1 = [vin1,vout], p2 = [vin2,vout]
  //                            -> (vin1, p1, vin2), (p1, p2, vin2)
  // nin == 1, two vertices out: (vin, vout1, vout2) = (v0,v1,v2) | (v2,v0,v1) | (v1,v0,v2); p1 = [vin,vout1], p2 = [vin,vout2]
  //                            -> (vin, p1, p2)
  // Both cases intersect two edges: the end points are selected first and the two intersections are evaluated in code
  // common to both (a warp's lanes in different cases stay converged through the expensive part); same operations on
  // the same operands as the two-branch form, hence the same bits.
  const bool two_in = (nin == 2);
  V3 a0, a1, b0, b1;
  if (two_in) {
    V3 vout = !in2 ? t.c : (!in1 ? t.b : t.a);
    a0 = !in0 ? t.b : t.a;   // vin1
    b0 = !in2 ? t.b : t.c;   // vin2
    a1 = vout; b1 = vout;
  } else {
    V3 vin = in0 ? t.a : (in2 ? t.c : t.b);
    a0 = vin; b0 = vin;
    a1 = in0 ? t.b : t.a;    // vout1
    b1 = in2 ? t.b : t.c;    // vout2
  }
  V3 p1 = plane_edge_intersection(pc, n, a0, a1);
  V3 p2 = plane_edge_intersection(pc, n, b0, b1);
  if (two_in) {
    o0->a = a0; o0->b = p1; o0->c = b0;
    o1->a = p1; o1->b = p2; o1->c = b0;
    return 2;
  }
  o0->a = a0; o0->b = p1; o0->c = p2;
  return 1;
}

C3D_HD float tri_area(const Tri& t) { return norm(cross(t.b - t.a, t.c - t.a)) / 2.0f; }

// tri–tri coplanarity given precomputed unit normals (the cheap dot test first; identical result)
C3D_HD bool coplanar_tri_tri(const Tri& t1, V3 n1, const Tri& t2, V3 n2) {
  bool check1 = fabsf(dot(n1, n2)) > 1.0f - dEps;
  if (!check1) return false;
  const V3 a[3] = {t1.a, t1.b, t1.c};
  const V3 b[3] = {t2.a, t2.b, t2.c};
  float best = -1.0f; int bi = 0, bj = 0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      V3 d = a[i] - b[j];
      float dist = dot(d, d);
      if (dist > best) { best = dist; bi = i; bj = j; }
    }
  V3 d = a[bi] - b[bj];
  d = d / fmaxf(norm(d), kEps);
  return (fabsf(dot(d, n1)) < dEps) || (fabsf(dot(d, n2)) < dEps);
}

// |det|/6 of a triangle about centre c
C3D_HD float tet_volume(const Tri& t, V3 c) {
  V3 a = t.a - c, b = t.b - c, d = t.c - c;
  return fabsf(dot(a, cross(b, d))) / 6.0f;
}

// ---- per-box record (64 floats = 256 B, built once per box by the prep kernel) ----
//   [0..23]  8 corners xyz
//   [24..59] 6 faces: centre xyz, inward unit normal xyz
//   [60..62] box centre (mean of corners)    [63] box volume (12 tets about the centre)
constexpr int kRecFloats = 64;

C3D_HD void build_box_record(const float* __restrict__ corners, float* __restrict__ rec,
                             float* sphere4 /* cx,cy,cz,r or null */) {
  V3 c[8];
  for (int i = 0; i < 8; ++i) {
    c[i] = mk(corners[3 * i], corners[3 * i + 1], corners[3 * i + 2]);
    rec[3 * i] = c[i].x; rec[3 * i + 1] = c[i].y; rec[3 * i + 2] = c[i].z;
  }
  V3 s = mk(0.f, 0.f, 0.f);
  for (int i = 0; i < 8; ++i) s = s + c[i];
  V3 bc = s / 8.0f;
  for (int p = 0; p < 6; ++p) {
    V3 pc, n;
    plane_from_quad(c[plane_vert(p, 0)], c[plane_vert(p, 1)], c[plane_vert(p, 2)],
                    c[plane_vert(p, 3)], bc, &pc, &n);
    float* o = rec + 24 + 6 * p;
    o[0] = pc.x; o[1] = pc.y; o[2] = pc.z; o[3] = n.x; o[4] = n.y; o[5] = n.z;
  }
  float vol = 0.0f;
  for (int t = 0; t < 12; ++t) {
    Tri tr; tr.a = c[tri_vert(t, 0)]; tr.b = c[tri_vert(t, 1)]; tr.c = c[tri_vert(t, 2)];
    vol = vol + tet_volume(tr, bc);
  }
  rec[60] = bc.x; rec[61] = bc.y; rec[62] = bc.z; rec[63] = vol;
  if (sphere4) {
    float r2 = 0.0f;
    for (int i = 0; i < 8; ++i) { V3 d = c[i] - bc; r2 = fmaxf(r2, dot(d, d)); }
    sphere4[0] = bc.x; sphere4[1] = bc.y; sphere4[2] = bc.z;
    sphere4[3] = sqrtf(r2) * 1.0009765625f + 1e-6f;   // padded bounding radius
  }
}

// centre (mean of corners) + padded bounding radius only: the SAME arithmetic as build_box_record's sphere
C3D_HD void box_sphere(const float* __restrict__ corners, float* sphere4) {
  V3 c[8];
  for (int i = 0; i < 8; ++i) c[i] = mk(corners[3 * i], corners[3 * i + 1], corners[3 * i + 2]);
  V3 s = mk(0.f, 0.f, 0.f);
  for (int i = 0; i < 8; ++i) s = s + c[i];
  V3 bc = s / 8.0f;
  float r2 = 0.0f;
  for (int i = 0; i < 8; ++i) { V3 d = c[i] - bc; r2 = fmaxf(r2, dot(d, d)); }
  sphere4[0] = bc.x; sphere4[1] = bc.y; sphere4[2] = bc.z;
  sphere4[3] = sqrtf(r2) * 1.0009765625f + 1e-6f;
}

// Row validity of a dt box (omni3d_evaluation.py:65-104): returns bit0 = coplanar_ok,
// bit1 = nonzero_ok.  NB the reference sums the six face offsets before abs() (:83-86).
C3D_HD int check_box(const float* __restrict__ corners, float eps_coplanar, float eps_nonzero) {
  V3 c[8];
  for (int i = 0; i < 8; ++i) c[i] = mk(corners[3 * i], corners[3 * i + 1], corners[3 * i + 2]);
  float acc = 0.0f;
  for (int p = 0; p < 6; ++p) {
    V3 v0 = c[plane_vert(p, 0)], v1 = c[plane_vert(p, 1)], v2 = c[plane_vert(p, 2)],
       v3 = c[plane_vert(p, 3)];
    V3 e0 = v1 - v0; e0 = e0 / fmaxf(norm(e0), 1e-12f);
    V3 e1 = v2 - v0; e1 = e1 / fmaxf(norm(e1), 1e-12f);
    V3 n = cross(e0, e1); n = n / fmaxf(norm(n), 1e-12f);
    V3 d = v3 - v0;
    acc += d.x * n.x; acc += d.y * n.y; acc += d.z * n.z;
  }
  int ok = (fabsf(acc) < eps_coplanar) ? 1 : 0;
  bool nz = true;
  for (int t = 0; t < 12; ++t) {
    V3 v0 = c[tri_vert(t, 0)], v1 = c[tri_vert(t, 1)], v2 = c[tri_vert(t, 2)];
    float area = norm(cross(v1 - v0, v2 - v0)) / 2.0f;
    if (!(area > eps_nonzero)) nz = false;
  }
  return ok | (nz ? 2 : 0);
}

}  // namespace c3d
