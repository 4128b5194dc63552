// TEST HARNESS (not product): the exact fp32 gradient maps of the ROIAlign backward (c3d_roi_align_bwd), from the
// product's sample geometry (omni3d_b200/csrc/roi_geom.cuh, compiled for the host).  One serial walk over the
// contributions in (RoI, ph, pw, iy, ix, tap) order, each applied as acc = fmaf(w, g, acc) with g = dout / count, gives
// every map element the chain the kernel promises, so the kernel's maps must equal these bit for bit.
// Build: g++ -O2 -ffp-contract=off -fPIC -shared.
#include <cmath>
#include <cstddef>
#include <vector>
#include "../../omni3d_b200/csrc/roi_geom.cuh"
using namespace c3d;

// rois [R][6]; dout [R][PH][PW][C] as floats (the bf16 values); grad[l]: fp32 (N, H[l], W[l], C), overwritten
extern "C" void harness_roi_align_bwd(const float* rois, int R, const float* dout, int C, int PH, int PW, int N,
                                      int num_levels, const int* H, const int* W, const float* scale, float** grad) {
  for (int l = 0; l < num_levels; ++l)
    for (size_t i = 0, n = (size_t)N * H[l] * W[l] * C; i < n; ++i) grad[l][i] = 0.f;
  std::vector<float> g(C);
  for (int r = 0; r < R; ++r) {
    const float* roi = rois + (size_t)r * 6;
    if (!roi_in_range(roi, N, num_levels)) continue;
    const int b = (int)roi[0], lvl = (int)roi[1], h = H[lvl], w = W[lvl];
    const RoiGeom geo = roi_geom(roi, scale[lvl], PH, PW);
    float* map = grad[lvl] + (size_t)b * h * w * C;
    for (int ph = 0; ph < PH; ++ph)
      for (int pw = 0; pw < PW; ++pw) {
        const float* d = dout + (((size_t)r * PH + ph) * PW + pw) * C;
        for (int c = 0; c < C; ++c) g[c] = rg_div(d[c], geo.cnt);
        for (int iy = 0; iy < geo.gh; ++iy) {
          const float y = sample_at(geo.sh, ph, geo.bh, iy, geo.gh);
          for (int ix = 0; ix < geo.gw; ++ix) {
            const float x = sample_at(geo.sw, pw, geo.bw, ix, geo.gw);
            const Tap t = make_tap(y, x, h, w);
            if (!t.valid) continue;
            const int py[4] = {t.y0, t.y0, t.y1, t.y1}, px[4] = {t.x0, t.x1, t.x0, t.x1};
            const float wt[4] = {t.w1, t.w2, t.w3, t.w4};
            for (int k = 0; k < 4; ++k) {
              float* p = map + ((size_t)py[k] * w + px[k]) * C;
              for (int c = 0; c < C; ++c) p[c] = std::fmaf(wt[k], g[c], p[c]);
            }
          }
        }
      }
  }
}
