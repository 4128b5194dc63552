// roi_geom.cuh — sample geometry of the multi-level ROIAlign (aligned=True, adaptive sampling), shared by the forward
// and the backward kernels so that both round alike, and compiled for the host by tests/csrc/roi_align_host_harness.cpp,
// which walks the backward's contributions in the kernel's order and must produce the same fp32 maps bit for bit.
//
// Each operation is written out (fmaf and the round-to-nearest add / subtract / multiply / divide) as the forward has
// always compiled it, so no contraction a compiler might choose differently in one place can change a weight.  On the
// host the rounded operations are the plain IEEE ones; the harness is compiled with -ffp-contract=off.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define C3D_RG __host__ __device__ __forceinline__
#else
#define C3D_RG static inline
#endif

namespace c3d {

C3D_RG float rg_add(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
C3D_RG float rg_sub(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
C3D_RG float rg_mul(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
C3D_RG float rg_div(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}

// a NaN / Inf box (diverging step) must not become an out-of-range level or image index: such RoIs pool zeros and get
// no gradient
C3D_RG bool roi_in_range(const float* roi, int num_images, int num_levels) {
  const float fb = roi[0], fl = roi[1];
  return fb >= 0.f && fb < (float)num_images && fl >= 0.f && fl < (float)num_levels && isfinite(roi[2]) &&
         isfinite(roi[3]) && isfinite(roi[4]) && isfinite(roi[5]);
}

struct RoiGeom { float sw, sh, rw, rh, bw, bh, cnt; int gw, gh; };

C3D_RG RoiGeom roi_geom(const float* roi, float sc, int PH, int PW) {
  RoiGeom g;
  g.sw = fmaf(roi[2], sc, -0.5f);
  g.sh = fmaf(roi[3], sc, -0.5f);
  g.rw = rg_sub(fmaf(roi[4], sc, -0.5f), g.sw);
  g.rh = rg_sub(fmaf(roi[5], sc, -0.5f), g.sh);
  g.bw = rg_div(g.rw, (float)PW);
  g.bh = rg_div(g.rh, (float)PH);
  g.gw = (int)ceilf(g.bw);
  g.gh = (int)ceilf(g.bh);
  g.cnt = fmaxf((float)(g.gh * g.gw), 1.f);
  return g;
}

// coordinate of sample i of n in bin p of size b that starts the RoI at s: s + p * b + (i + 0.5) * b / n
C3D_RG float sample_at(float s, int p, float b, int i, int n) {
  return rg_add(fmaf((float)p, b, s), rg_div(rg_mul(rg_add((float)i, 0.5f), b), (float)n));
}

struct Tap { int y0, y1, x0, x1; float w1, w2, w3, w4; bool valid; };

C3D_RG Tap make_tap(float y, float x, int H, int W) {
  Tap t;
  t.valid = !(y < -1.0f || y > (float)H || x < -1.0f || x > (float)W);
  if (y <= 0.f) y = 0.f;
  if (x <= 0.f) x = 0.f;
  int yl = (int)y, xl = (int)x, yh, xh;
  if (yl >= H - 1) { yh = yl = H - 1; y = (float)yl; } else yh = yl + 1;
  if (xl >= W - 1) { xh = xl = W - 1; x = (float)xl; } else xh = xl + 1;
  const float ly = rg_sub(y, (float)yl), lx = rg_sub(x, (float)xl), hy = rg_sub(1.f, ly), hx = rg_sub(1.f, lx);
  t.y0 = yl; t.y1 = yh; t.x0 = xl; t.x1 = xh;
  t.w1 = rg_mul(hy, hx); t.w2 = rg_mul(hy, lx); t.w3 = rg_mul(ly, hx); t.w4 = rg_mul(ly, lx);
  return t;
}

}  // namespace c3d
