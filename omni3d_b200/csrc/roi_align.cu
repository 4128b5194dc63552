// roi_align.cu — multi-level ROIAlign (aligned=True, adaptive sampling) on NHWC bf16 feature maps.
//
// Replaces detectron2 ROIPooler / ROIAlignV2 as used by the box pooler (roi_heads.py:267) and the cube
// pooler (roi_heads.py:362, built :166-171): 7x7 bins, sampling_ratio 0, FPN levels p2..p6 chosen by
// floor(4 + log2(sqrt(area)/224 + 1e-8)) clamped to [2,6].
// One warp per output bin; each lane owns 8 consecutive channels, so every bilinear tap is a single
// fully-coalesced 16-byte-per-lane read of the pixel's channel vector (no tensor cores: gather work).
// Backward is a gather: a block owns an (image, level, 8-row band) of the gradient map and adds, per 8 x 8 pixel tile in
// shared memory, the contributions of the RoIs that touch it in (RoI, bin, sample, tap) order — no atomics, so the
// gradient is the same on every run.
#include <cuda_bf16.h>
#include <stdlib.h>
#include "c3d_common.cuh"

namespace c3d {
using bf16 = __nv_bfloat16;

struct RoiLevels {
  const bf16* feat[5];
  float* grad[5];
  int H[5], W[5];
  float scale[5];
  int num_levels;
  int num_images;
};

struct Tap { int y0, y1, x0, x1; float w1, w2, w3, w4; bool valid; };

__device__ __forceinline__ Tap make_tap(float y, float x, int H, int W) {
  Tap t;
  t.valid = !(y < -1.0f || y > (float)H || x < -1.0f || x > (float)W);
  if (y <= 0.f) y = 0.f;
  if (x <= 0.f) x = 0.f;
  int yl = (int)y, xl = (int)x, yh, xh;
  if (yl >= H - 1) { yh = yl = H - 1; y = (float)yl; } else yh = yl + 1;
  if (xl >= W - 1) { xh = xl = W - 1; x = (float)xl; } else xh = xl + 1;
  float ly = y - yl, lx = x - xl, hy = 1.f - ly, hx = 1.f - lx;
  t.y0 = yl; t.y1 = yh; t.x0 = xl; t.x1 = xh;
  t.w1 = hy * hx; t.w2 = hy * lx; t.w3 = ly * hx; t.w4 = ly * lx;
  return t;
}

__device__ __forceinline__ void acc8(float (&a)[8], const bf16* p, float w) {
  uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) { float2 f = __bfloat1622float2(h[i]); a[2 * i] += w * f.x; a[2 * i + 1] += w * f.y; }
}

// a NaN / Inf box (diverging step) must not become an out-of-range level or image index: such RoIs pool zeros and get
// no gradient
__device__ __forceinline__ bool roi_sane(const float* roi, const RoiLevels& L) {
  const float fb = roi[0], fl = roi[1];
  return fb >= 0.f && (L.num_images <= 0 || fb < (float)L.num_images) && fl >= 0.f && fl < (float)L.num_levels &&
         isfinite(roi[2]) && isfinite(roi[3]) && isfinite(roi[4]) && isfinite(roi[5]);
}

// rois: [R][6] = (batch, level, x1, y1, x2, y2) fp32
__global__ void roi_align_kernel(RoiLevels L, const float* __restrict__ rois, int R, int C, int PH, int PW,
                                 bf16* __restrict__ out) {
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  const long long nbins = (long long)R * PH * PW;
  for (long long bin = (long long)blockIdx.x * warps_per_block + (threadIdx.x >> 5); bin < nbins;
       bin += (long long)gridDim.x * warps_per_block) {
    const int pw = (int)(bin % PW), ph = (int)((bin / PW) % PH), r = (int)(bin / ((long long)PW * PH));
    const float* roi = rois + (size_t)r * 6;
    if (!roi_sane(roi, L)) {
      for (int c = lane * 8; c < C; c += 256) *reinterpret_cast<uint4*>(out + (size_t)bin * C + c) = make_uint4(0, 0, 0, 0);
      continue;
    }
    const int b = (int)roi[0], lvl = (int)roi[1];
    const float sc = L.scale[lvl];
    const int H = L.H[lvl], W = L.W[lvl];
    const float sw = roi[2] * sc - 0.5f, sh = roi[3] * sc - 0.5f;
    const float rw = roi[4] * sc - 0.5f - sw, rh = roi[5] * sc - 0.5f - sh;
    const float bh = rh / PH, bw = rw / PW;
    const int gh = (int)ceilf(rh / PH), gw = (int)ceilf(rw / PW);
    const float cnt = fmaxf((float)(gh * gw), 1.f);
    const bf16* base = L.feat[lvl] + (size_t)b * H * W * C;
    for (int c = lane * 8; c < C; c += 256) {
      float a[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) a[k] = 0.f;
      for (int iy = 0; iy < gh; ++iy) {
        const float y = sh + ph * bh + (iy + 0.5f) * bh / (float)gh;
        for (int ix = 0; ix < gw; ++ix) {
          const float x = sw + pw * bw + (ix + 0.5f) * bw / (float)gw;
          Tap t = make_tap(y, x, H, W);
          if (!t.valid) continue;
          acc8(a, base + ((size_t)t.y0 * W + t.x0) * C + c, t.w1); acc8(a, base + ((size_t)t.y0 * W + t.x1) * C + c, t.w2);
          acc8(a, base + ((size_t)t.y1 * W + t.x0) * C + c, t.w3); acc8(a, base + ((size_t)t.y1 * W + t.x1) * C + c, t.w4);
        }
      }
      uint4 u;
      __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
      for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(a[2 * i] / cnt, a[2 * i + 1] / cnt);
      *reinterpret_cast<uint4*>(out + (size_t)bin * C + c) = u;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Backward (gather).  Grid = (sum over levels of ceil(H / 8) bands, images).  The block first lists, in index order, the
// RoIs of its image and level whose pixel footprint reaches its band (kListCap at a time), then walks the band's 8 x 8
// tiles: thread t owns channel cc + t of a [64 px][256 ch] fp32 shared-memory tile, every thread replays the same
// (RoI, bin, sample, tap) sequence and adds w * dout / count for the taps that fall in the tile, and a touched tile is
// added to the fp32 map.  Each map element thus receives its contributions in one fixed order.
constexpr int kTile = 8, kTileC = 256, kListCap = 2048;
constexpr int kBwdSmem = kTile * kTile * kTileC * 4;

__global__ void __launch_bounds__(kTileC)
roi_align_bwd_kernel(RoiLevels L, const float* __restrict__ rois, int R, int C, int PH, int PW, const bf16* __restrict__ dout) {
  extern __shared__ float sacc[];                   // [64 px][kTileC]
  __shared__ int slist[kListCap];
  __shared__ int s_wc[kTileC / 32];
  __shared__ int s_n, s_touch;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int b = blockIdx.y;
  int lvl = 0, band = blockIdx.x;
  while (lvl < L.num_levels - 1 && band >= (L.H[lvl] + kTile - 1) / kTile) { band -= (L.H[lvl] + kTile - 1) / kTile; ++lvl; }
  const int H = L.H[lvl], W = L.W[lvl];
  if (band * kTile >= H) return;
  const float sc = L.scale[lvl];
  const int ty0 = band * kTile, ty1 = min(H, ty0 + kTile) - 1;
  float* gmap = L.grad[lvl] + (size_t)b * H * W * C;
  for (int r0 = 0; r0 < R;) {
    // ---- the next window of matching RoIs, in index order
    if (tid == 0) s_n = 0;
    __syncthreads();
    int r = r0;
    while (r < R) {
      const int idx = r + tid;
      bool pred = false;
      if (idx < R) {
        const float* roi = rois + (size_t)idx * 6;
        if (roi_sane(roi, L) && (int)roi[0] == b && (int)roi[1] == lvl) {
          const float sh = roi[3] * sc - 0.5f, eh = roi[5] * sc - 0.5f;
          pred = (int)floorf(sh) - 1 <= ty1 && (int)floorf(eh) + 1 >= ty0;
        }
      }
      const unsigned bal = __ballot_sync(0xffffffffu, pred);
      if (lane == 0) s_wc[wid] = __popc(bal);
      __syncthreads();
      int before = 0, total = 0;
      for (int w = 0; w < kTileC / 32; ++w) { total += s_wc[w]; if (w < wid) before += s_wc[w]; }
      const int n0 = s_n;
      const bool fits = n0 + total <= kListCap;           // same value in every thread
      if (fits && pred) slist[n0 + before + __popc(bal & ((1u << lane) - 1u))] = idx;
      __syncthreads();
      if (!fits) break;
      if (tid == 0) s_n = n0 + total;
      __syncthreads();
      r += kTileC;
    }
    r0 = r;
    const int n = s_n;
    // ---- the band's tiles
    for (int tx0 = 0; tx0 < W; tx0 += kTile) {
      const int tx1 = min(W, tx0 + kTile) - 1;
      for (int cc = 0; cc < C; cc += kTileC) {
        const int c = cc + tid;
        const bool cin = c < C;
        for (int p = 0; p < kTile * kTile; ++p) sacc[p * kTileC + tid] = 0.f;
        if (tid == 0) s_touch = 0;
        __syncthreads();
        for (int li = 0; li < n; ++li) {
          const int ri = slist[li];
          const float* roi = rois + (size_t)ri * 6;
          const float sw = roi[2] * sc - 0.5f, sh = roi[3] * sc - 0.5f;
          const float rw = roi[4] * sc - 0.5f - sw, rh = roi[5] * sc - 0.5f - sh;
          if ((int)floorf(sw) - 1 > tx1 || (int)floorf(sw + rw) + 1 < tx0) continue;
          const float bh = rh / PH, bw = rw / PW;
          const int gh = (int)ceilf(rh / PH), gw = (int)ceilf(rw / PW);
          const float cnt = fmaxf((float)(gh * gw), 1.f);
          for (int ph = 0; ph < PH; ++ph) {
            if ((int)floorf(sh + ph * bh) - 1 > ty1 || (int)floorf(sh + (ph + 1) * bh) + 1 < ty0) continue;
            for (int pw = 0; pw < PW; ++pw) {
              if ((int)floorf(sw + pw * bw) - 1 > tx1 || (int)floorf(sw + (pw + 1) * bw) + 1 < tx0) continue;
              const float g = cin ? __bfloat162float(dout[(((size_t)ri * PH + ph) * PW + pw) * C + c]) / cnt : 0.f;
              for (int iy = 0; iy < gh; ++iy) {
                const float y = sh + ph * bh + (iy + 0.5f) * bh / (float)gh;
                for (int ix = 0; ix < gw; ++ix) {
                  const float x = sw + pw * bw + (ix + 0.5f) * bw / (float)gw;
                  const Tap t = make_tap(y, x, H, W);
                  if (!t.valid) continue;
                  const int ys[4] = {t.y0, t.y0, t.y1, t.y1}, xs[4] = {t.x0, t.x1, t.x0, t.x1};
                  const float ws[4] = {t.w1, t.w2, t.w3, t.w4};
#pragma unroll
                  for (int j = 0; j < 4; ++j)
                    if (ys[j] >= ty0 && ys[j] <= ty1 && xs[j] >= tx0 && xs[j] <= tx1) {
                      sacc[((ys[j] - ty0) * kTile + (xs[j] - tx0)) * kTileC + tid] += ws[j] * g;
                      if (tid == 0) s_touch = 1;
                    }
                }
              }
            }
          }
        }
        __syncthreads();
        if (s_touch && cin) {
          for (int p = 0; p < kTile * kTile; ++p) {
            const int py = ty0 + p / kTile, px = tx0 + p % kTile;
            if (py <= ty1 && px <= tx1) gmap[((size_t)py * W + px) * C + c] += sacc[p * kTileC + tid];
          }
        }
        __syncthreads();
      }
    }
  }
}

static int32_t run(bool bwd, const c3d_roi_levels* lv, const float* rois, int R, int C, int PH, int PW, void* out,
                   const void* dout, cudaStream_t st) {
  if (!lv || lv->num_levels < 1 || lv->num_levels > 5 || C % 8 != 0) return set_error(C3D_EINVAL, "roi_align: bad args");
  if (R == 0) return C3D_OK;
  RoiLevels L;
  L.num_levels = lv->num_levels;
  L.num_images = lv->num_images;
  for (int i = 0; i < 5; ++i) {
    L.feat[i] = (const bf16*)lv->feat[i]; L.grad[i] = (float*)lv->grad[i];
    L.H[i] = lv->H[i]; L.W[i] = lv->W[i]; L.scale[i] = lv->scale[i];
  }
  if (!bwd) {
    long long nbins = (long long)R * PH * PW;
    long long blocks = (nbins + 7) / 8;
    if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
    roi_align_kernel<<<(unsigned)blocks, 256, 0, st>>>(L, rois, R, C, PH, PW, (bf16*)out);
    return check_launch("roi_align");
  }
  if (L.num_images <= 0) return set_error(C3D_EINVAL, "roi_align bwd: num_images must be set");
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(roi_align_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kBwdSmem);
    if (e != cudaSuccess) return set_error(C3D_ECUDA, "roi_align bwd smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  int bands = 0;
  for (int i = 0; i < L.num_levels; ++i) bands += (L.H[i] + kTile - 1) / kTile;
  roi_align_bwd_kernel<<<dim3((unsigned)bands, (unsigned)L.num_images), kTileC, kBwdSmem, st>>>(L, rois, R, C, PH, PW, (const bf16*)dout);
  return check_launch("roi_align bwd");
}
}  // namespace c3d

extern "C" int32_t c3d_roi_align_fwd(const c3d_roi_levels* levels, const float* rois, int32_t R, int32_t C,
                                     int32_t pooled_h, int32_t pooled_w, void* out, void* stream) {
  if (!rois && R > 0) return c3d::set_error(C3D_EINVAL, "roi_align: null rois");
  return c3d::run(false, levels, rois, R, C, pooled_h, pooled_w, out, nullptr, (cudaStream_t)stream);
}
extern "C" int32_t c3d_roi_align_bwd(const c3d_roi_levels* levels, const float* rois, int32_t R, int32_t C,
                                     int32_t pooled_h, int32_t pooled_w, const void* dout, void* stream) {
  if (!rois && R > 0) return c3d::set_error(C3D_EINVAL, "roi_align: null rois");
  return c3d::run(true, levels, rois, R, C, pooled_h, pooled_w, nullptr, dout, (cudaStream_t)stream);
}
