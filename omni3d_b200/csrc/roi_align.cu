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

// Sample geometry, shared by the forward and the backward so that both round alike.  Each operation is written out
// (fmaf, __fadd_rn, __fmul_rn, __fdiv_rn) as the forward has always compiled it, so no contraction the compiler might
// choose differently in one kernel can change a weight.
struct RoiGeom { float sw, sh, rw, rh, bw, bh, cnt; int gw, gh; };

__device__ __forceinline__ RoiGeom roi_geom(const float* roi, float sc, int PH, int PW) {
  RoiGeom g;
  g.sw = fmaf(roi[2], sc, -0.5f);
  g.sh = fmaf(roi[3], sc, -0.5f);
  g.rw = __fsub_rn(fmaf(roi[4], sc, -0.5f), g.sw);
  g.rh = __fsub_rn(fmaf(roi[5], sc, -0.5f), g.sh);
  g.bw = __fdiv_rn(g.rw, (float)PW);
  g.bh = __fdiv_rn(g.rh, (float)PH);
  g.gw = (int)ceilf(g.bw);
  g.gh = (int)ceilf(g.bh);
  g.cnt = fmaxf((float)(g.gh * g.gw), 1.f);
  return g;
}

// coordinate of sample i of n in bin p of size b that starts the RoI at s: s + p * b + (i + 0.5) * b / n
__device__ __forceinline__ float sample_at(float s, int p, float b, int i, int n) {
  return __fadd_rn(fmaf((float)p, b, s), __fdiv_rn(__fmul_rn(__fadd_rn((float)i, 0.5f), b), (float)n));
}

struct Tap { int y0, y1, x0, x1; float w1, w2, w3, w4; bool valid; };

__device__ __forceinline__ Tap make_tap(float y, float x, int H, int W) {
  Tap t;
  t.valid = !(y < -1.0f || y > (float)H || x < -1.0f || x > (float)W);
  if (y <= 0.f) y = 0.f;
  if (x <= 0.f) x = 0.f;
  int yl = (int)y, xl = (int)x, yh, xh;
  if (yl >= H - 1) { yh = yl = H - 1; y = (float)yl; } else yh = yl + 1;
  if (xl >= W - 1) { xh = xl = W - 1; x = (float)xl; } else xh = xl + 1;
  const float ly = __fsub_rn(y, (float)yl), lx = __fsub_rn(x, (float)xl), hy = __fsub_rn(1.f, ly), hx = __fsub_rn(1.f, lx);
  t.y0 = yl; t.y1 = yh; t.x0 = xl; t.x1 = xh;
  t.w1 = __fmul_rn(hy, hx); t.w2 = __fmul_rn(hy, lx); t.w3 = __fmul_rn(ly, hx); t.w4 = __fmul_rn(ly, lx);
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
  return fb >= 0.f && fb < (float)L.num_images && fl >= 0.f && fl < (float)L.num_levels &&
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
    const int H = L.H[lvl], W = L.W[lvl];
    const RoiGeom g = roi_geom(roi, L.scale[lvl], PH, PW);
    const float cnt = g.cnt;
    const bf16* base = L.feat[lvl] + (size_t)b * H * W * C;
    for (int c = lane * 8; c < C; c += 256) {
      float a[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) a[k] = 0.f;
      for (int iy = 0; iy < g.gh; ++iy) {
        const float y = sample_at(g.sh, ph, g.bh, iy, g.gh);
        for (int ix = 0; ix < g.gw; ++ix) {
          const float x = sample_at(g.sw, pw, g.bw, ix, g.gw);
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
// Backward: a gather with no atomics, in two launches.
//
// roi_bucket_kernel lists the RoI indices of every (image, level) in index order (a stable counting sort).
//
// roi_align_bwd_kernel: grid = (sum over levels of ceil(H / 8) bands, images).  A block owns one (image, level, 8-row
// band) of the gradient map and walks the band's 8 x 8 pixel tiles.  For a tile it reads its bucket 256 RoIs at a time
// and lists the bins of those RoIs that can reach the tile, as "slots" (kSlots at a time, in (RoI, ph, pw) order).
// The threads then split the (slot, iy, ix) samples among themselves; each computes its sample's four taps once and
// keeps those that fall in the tile as (pixel, slot, weight) entries, compacted in (sample, tap) order.  Thread t owns
// channel cc + t: it stages g = dout / count of every slot for its channel and walks the entries, adding w * g to its
// column of a [64 px][256 ch] fp32 tile in shared memory.  Every element of the map thus receives
// acc = fmaf(w, g, acc), starting from +0, over (RoI, ph, pw, iy, ix, tap) in that order, as one chain, and is stored
// once, zeros included: the maps need no clearing.  Storing the chain is the same as adding it to a zeroed map, since
// the chain is never -0.
// (Up to version 2 of the ABI the kernel added to the map and split a band's RoIs into lists of 2048, adding each list's
// sum separately; results can differ from that only where more than 2048 RoIs of one image and level reach one band.
// Training samples at most 512 RoIs per image.)
constexpr int kTile = 8, kTileC = 256, kSlots = 32, kEntCap = 4 * kTileC;
constexpr int kBucketThreads = 1024, kBucketWarps = kBucketThreads / 32;

struct BwdSmem {
  float acc[kTile * kTile][kTileC];  // the tile: [pixel][channel - cc]
  float g[kSlots][kTileC];           // dout / count of each slot
  int2 ent[kEntCap];                 // (pixel | slot << 6, weight bits) in (sample, tap) order
  int roi[kTileC];                   // the window of the bucket: RoI index,
  int rect[kTileC];                  //   first ph | first pw << 8 | bins per row << 16,
  int bins[kTileC + 1];              //   exclusive prefix of the bins that can reach the tile
  float sh[kSlots], sw[kSlots], bh[kSlots], bw[kSlots], cnt[kSlots];
  int gh[kSlots], gw[kSlots], ph[kSlots], pw[kSlots], ri[kSlots], iy[kSlots], ix[kSlots], nix[kSlots];
  int items[kSlots + 1];             // exclusive prefix of the samples of each slot
  int warp[kTileC / 32];
};

__device__ __forceinline__ int warp_inclusive_scan(int x, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  return x;
}

// exclusive prefix of v over the block's kTileC threads; ends with a __syncthreads, reads s_warp after it
__device__ __forceinline__ int block_exclusive_scan(int v, int* s_warp, int& total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int x = warp_inclusive_scan(v, lane);
  if (lane == 31) s_warp[wid] = x;
  __syncthreads();
  int before = 0;
  total = 0;
#pragma unroll
  for (int w = 0; w < kTileC / 32; ++w) {
    const int t = s_warp[w];
    if (w < wid) before += t;
    total += t;
  }
  return before + x - v;
}

__device__ __forceinline__ int roi_bucket(const float* roi, const RoiLevels& L) {
  return roi_sane(roi, L) ? (int)roi[0] * L.num_levels + (int)roi[1] : -1;
}

// One block.  Warp w takes the w-th contiguous slice of [0, R) and counts its keys into wk[w][key]; the counts become
// start offsets (bucket by bucket, and warp by warp inside a bucket), and a second pass places every index.
// wk: kBucketWarps x nb ints of scratch; off: nb + 1 bucket offsets; idx: the bucketed RoI indices.
__global__ void __launch_bounds__(kBucketThreads)
roi_bucket_kernel(RoiLevels L, const float* __restrict__ rois, int R, int nb, int* __restrict__ wk, int* __restrict__ off,
                  int* __restrict__ idx) {
  __shared__ int s_part[kBucketWarps];
  __shared__ int s_carry;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int i = tid; i < kBucketWarps * nb; i += kBucketThreads) wk[i] = 0;
  if (tid == 0) s_carry = 0;
  __syncthreads();
  const int per = (R + kBucketWarps - 1) / kBucketWarps;
  const int lo = min(R, wid * per), hi = min(R, lo + per);
  int* mine = wk + (size_t)wid * nb;
  for (int r0 = lo; r0 < hi; r0 += 32) {
    const int r = r0 + lane;
    const int k = r < hi ? roi_bucket(rois + (size_t)r * 6, L) : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, k);
    if (k >= 0 && lane == __ffs(peers) - 1) atomicAdd(&mine[k], __popc(peers));
  }
  __syncthreads();
  for (int k0 = 0; k0 < nb; k0 += kBucketThreads) {
    const int k = k0 + tid;
    int tot = 0;
    if (k < nb)
      for (int w = 0; w < kBucketWarps; ++w) tot += wk[(size_t)w * nb + k];
    const int x = warp_inclusive_scan(tot, lane);
    if (lane == 31) s_part[wid] = x;
    __syncthreads();
    int run = s_carry + x - tot, chunk = 0;
    for (int w = 0; w < kBucketWarps; ++w) {
      if (w < wid) run += s_part[w];
      chunk += s_part[w];
    }
    if (k < nb) {
      off[k] = run;
      for (int w = 0; w < kBucketWarps; ++w) {
        const int c = wk[(size_t)w * nb + k];
        wk[(size_t)w * nb + k] = run;
        run += c;
      }
    }
    __syncthreads();
    if (tid == 0) s_carry += chunk;
    __syncthreads();
  }
  if (tid == 0) off[nb] = s_carry;
  for (int r0 = lo; r0 < hi; r0 += 32) {
    const int r = r0 + lane;
    const int k = r < hi ? roi_bucket(rois + (size_t)r * 6, L) : -1;
    const unsigned peers = __match_any_sync(0xffffffffu, k);
    const int leader = __ffs(peers) - 1;
    int base = 0;
    if (k >= 0 && lane == leader) base = atomicAdd(&mine[k], __popc(peers));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (k >= 0) idx[base + __popc(peers & ((1u << lane) - 1u))] = r;
  }
}

// samples i in [first, last] of the n samples (spacing st) of a bin starting at s whose taps can reach rows / columns
// [t0, t1]: the sample coordinate must lie in [t0 - 1, t1 + 1] (taps at floor and floor + 1 of the coordinate clamped into
// the map), widened by two samples plus the rounding of the coordinate
__device__ __forceinline__ void sample_range(float s, float st, int n, int t0, int t1, int& first, int& count) {
  const float slop = 2.f + 1e-5f * fabsf(s) / st;
  const float lo = ceilf(((float)t0 - 1.f - s) / st - 0.5f - slop), hi = floorf(((float)t1 + 1.f - s) / st - 0.5f + slop);
  first = (int)fmaxf(lo, 0.f);
  const int last = (int)fminf(hi, (float)(n - 1));
  count = max(0, last - first + 1);
}

__global__ void __launch_bounds__(kTileC, 2)
roi_align_bwd_kernel(RoiLevels L, const float* __restrict__ rois, const int* __restrict__ off, const int* __restrict__ idx,
                     int C, int PH, int PW, const bf16* __restrict__ dout) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  BwdSmem& S = *reinterpret_cast<BwdSmem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31;
  const int b = blockIdx.y;
  int lvl = 0, band = blockIdx.x;
  while (lvl < L.num_levels - 1 && band >= (L.H[lvl] + kTile - 1) / kTile) { band -= (L.H[lvl] + kTile - 1) / kTile; ++lvl; }
  const int H = L.H[lvl], W = L.W[lvl];
  if (band * kTile >= H) return;
  const float sc = L.scale[lvl];
  const int ty0 = band * kTile, ty1 = min(H, ty0 + kTile) - 1;
  const int key = b * L.num_levels + lvl;
  const int* list = idx + off[key];
  const int n = off[key + 1] - off[key];
  float* gmap = L.grad[lvl] + (size_t)b * H * W * C;
  for (int tx0 = 0; tx0 < W; tx0 += kTile) {
    const int tx1 = min(W, tx0 + kTile) - 1;
    for (int cc = 0; cc < C; cc += kTileC) {
      const int c = cc + tid;
#pragma unroll 8
      for (int p = 0; p < kTile * kTile; ++p) S.acc[p][tid] = 0.f;
      for (int w0 = 0; w0 < n; w0 += kTileC) {
        // ---- the bins of the next kTileC RoIs whose footprint, one pixel wider, overlaps the tile
        int nbin = 0, rect = 0, ri = 0;
        if (w0 + tid < n) {
          ri = list[w0 + tid];
          const RoiGeom g = roi_geom(rois + (size_t)ri * 6, sc, PH, PW);
          if (g.gh > 0 && g.gw > 0) {
            int ph0 = PH, ph1 = -1, pw0 = PW, pw1 = -1;
            for (int ph = 0; ph < PH; ++ph)
              if ((int)floorf(g.sh + ph * g.bh) - 1 <= ty1 && (int)floorf(g.sh + (ph + 1) * g.bh) + 1 >= ty0) {
                ph0 = min(ph0, ph);
                ph1 = ph;
              }
            for (int pw = 0; pw < PW; ++pw)
              if ((int)floorf(g.sw + pw * g.bw) - 1 <= tx1 && (int)floorf(g.sw + (pw + 1) * g.bw) + 1 >= tx0) {
                pw0 = min(pw0, pw);
                pw1 = pw;
              }
            if (ph1 >= ph0 && pw1 >= pw0) {
              nbin = (ph1 - ph0 + 1) * (pw1 - pw0 + 1);
              rect = ph0 | pw0 << 8 | (pw1 - pw0 + 1) << 16;
            }
          }
        }
        int nbins;
        const int first = block_exclusive_scan(nbin, S.warp, nbins);
        S.roi[tid] = ri;
        S.rect[tid] = rect;
        S.bins[tid] = first;
        if (tid == 0) S.bins[kTileC] = nbins;
        __syncthreads();
        for (int s0 = 0; s0 < nbins; s0 += kSlots) {
          const int ns = min(kSlots, nbins - s0);
          // ---- slot setup, one lane per slot: which RoI and bin, and which of its samples can reach the tile
          if (tid < 32) {
            int items = 0;
            if (lane < ns) {
              const int bin = s0 + lane;
              int lo = 0, hi = kTileC;                         // the last window RoI whose bins start at or before `bin`
              while (hi - lo > 1) {
                const int mid = (lo + hi) >> 1;
                if (S.bins[mid] <= bin) lo = mid; else hi = mid;
              }
              const int rc = S.rect[lo], r = S.roi[lo], local = bin - S.bins[lo], npw = rc >> 16;
              const int ph = (rc & 255) + local / npw, pw = ((rc >> 8) & 255) + local % npw;
              const RoiGeom g = roi_geom(rois + (size_t)r * 6, sc, PH, PW);
              int iy0, niy, ix0, nix;
              sample_range(fmaf((float)ph, g.bh, g.sh), __fdiv_rn(g.bh, (float)g.gh), g.gh, ty0, ty1, iy0, niy);
              sample_range(fmaf((float)pw, g.bw, g.sw), __fdiv_rn(g.bw, (float)g.gw), g.gw, tx0, tx1, ix0, nix);
              S.sh[lane] = g.sh; S.sw[lane] = g.sw; S.bh[lane] = g.bh; S.bw[lane] = g.bw; S.cnt[lane] = g.cnt;
              S.gh[lane] = g.gh; S.gw[lane] = g.gw; S.ph[lane] = ph; S.pw[lane] = pw; S.ri[lane] = r;
              S.iy[lane] = iy0; S.ix[lane] = ix0; S.nix[lane] = nix;
              items = niy * nix;
            }
            S.items[lane + 1] = warp_inclusive_scan(items, lane);
            if (lane == 0) S.items[0] = 0;
          }
          __syncthreads();
          // ---- g = dout / count of every slot, for this thread's channel
          for (int s = 0; s < ns; ++s)
            S.g[s][tid] = c < C ? __fdiv_rn(__bfloat162float(dout[(((size_t)S.ri[s] * PH + S.ph[s]) * PW + S.pw[s]) * C + c]), S.cnt[s])
                                : 0.f;
          const int nitems = S.items[ns];
          for (int i0 = 0; i0 < nitems; i0 += kTileC) {
            // ---- one sample per thread: its taps that fall in the tile, compacted in (sample, tap) order
            const int k = i0 + tid;
            unsigned mask = 0;
            int slot = 0;
            Tap t = {};
            if (k < nitems) {
              int lo = 0, hi = ns;
              while (hi - lo > 1) {
                const int mid = (lo + hi) >> 1;
                if (S.items[mid] <= k) lo = mid; else hi = mid;
              }
              slot = lo;
              const int local = k - S.items[slot], nx = S.nix[slot];
              const float y = sample_at(S.sh[slot], S.ph[slot], S.bh[slot], S.iy[slot] + local / nx, S.gh[slot]);
              const float x = sample_at(S.sw[slot], S.pw[slot], S.bw[slot], S.ix[slot] + local % nx, S.gw[slot]);
              t = make_tap(y, x, H, W);
              if (t.valid) {
                const bool r0 = t.y0 >= ty0 && t.y0 <= ty1, r1 = t.y1 >= ty0 && t.y1 <= ty1;
                const bool c0 = t.x0 >= tx0 && t.x0 <= tx1, c1 = t.x1 >= tx0 && t.x1 <= tx1;
                mask = (r0 && c0) | (r0 && c1) << 1 | (r1 && c0) << 2 | (r1 && c1) << 3;
              }
            }
            int nent;
            int q = block_exclusive_scan(__popc(mask), S.warp, nent);
            const int tag = slot << 6;
            if (mask & 1) S.ent[q++] = make_int2(tag | (t.y0 - ty0) * kTile + (t.x0 - tx0), __float_as_int(t.w1));
            if (mask & 2) S.ent[q++] = make_int2(tag | (t.y0 - ty0) * kTile + (t.x1 - tx0), __float_as_int(t.w2));
            if (mask & 4) S.ent[q++] = make_int2(tag | (t.y1 - ty0) * kTile + (t.x0 - tx0), __float_as_int(t.w3));
            if (mask & 8) S.ent[q] = make_int2(tag | (t.y1 - ty0) * kTile + (t.x1 - tx0), __float_as_int(t.w4));
            __syncthreads();
            // ---- this thread's channel, entry by entry
            for (int e = 0; e < nent; ++e) {
              const int2 en = S.ent[e];
              float& a = S.acc[en.x & 63][tid];
              a = fmaf(__int_as_float(en.y), S.g[en.x >> 6][tid], a);
            }
            __syncthreads();
          }
          __syncthreads();
        }
      }
      if (c < C) {
        for (int p = 0; p < kTile * kTile; ++p) {
          const int py = ty0 + p / kTile, px = tx0 + p % kTile;
          if (py <= ty1 && px <= tx1) gmap[((size_t)py * W + px) * C + c] = S.acc[p][tid];
        }
      }
    }
  }
}

static int32_t run(bool bwd, const c3d_roi_levels* lv, const float* rois, int R, int C, int PH, int PW, void* out,
                   const void* dout, cudaStream_t st) {
  if (!lv || lv->num_levels < 1 || lv->num_levels > 5 || C % 8 != 0) return set_error(C3D_EINVAL, "roi_align: bad args");
  if (R < 0) return set_error(C3D_EINVAL, "roi_align: negative R");
  if (lv->num_images <= 0) return set_error(C3D_EINVAL, "roi_align: num_images must be set");
  RoiLevels L;
  L.num_levels = lv->num_levels;
  L.num_images = lv->num_images;
  for (int i = 0; i < 5; ++i) {
    L.feat[i] = (const bf16*)lv->feat[i]; L.grad[i] = (float*)lv->grad[i];
    L.H[i] = lv->H[i]; L.W[i] = lv->W[i]; L.scale[i] = lv->scale[i];
  }
  if (!bwd) {
    if (R == 0) return C3D_OK;
    long long nbins = (long long)R * PH * PW;
    long long blocks = (nbins + 7) / 8;
    if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
    roi_align_kernel<<<(unsigned)blocks, 256, 0, st>>>(L, rois, R, C, PH, PW, (bf16*)out);
    return check_launch("roi_align");
  }
  if (PH < 1 || PW < 1 || PH > 255 || PW > 255) return set_error(C3D_EINVAL, "roi_align bwd: pooled size outside [1, 255]");
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(roi_align_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BwdSmem));
    if (e != cudaSuccess) return set_error(C3D_ECUDA, "roi_align bwd smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  // the RoI buckets live in stream-ordered scratch: offsets (nb + 1), per-warp counts (kBucketWarps x nb), indices (R)
  const int nb = L.num_images * L.num_levels;
  int* off = nullptr;
  cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&off), ((size_t)(kBucketWarps + 1) * nb + 1 + R) * sizeof(int), st);
  if (e != cudaSuccess) return set_error(C3D_ECUDA, "roi_align bwd buckets: %s", cudaGetErrorString(e));
  int* wk = off + nb + 1;
  int* idx = wk + (size_t)kBucketWarps * nb;
  roi_bucket_kernel<<<1, kBucketThreads, 0, st>>>(L, rois, R, nb, wk, off, idx);
  int32_t rc = check_launch("roi_align bwd buckets");
  if (rc == C3D_OK) {
    int bands = 0;
    for (int i = 0; i < L.num_levels; ++i) bands += (L.H[i] + kTile - 1) / kTile;
    roi_align_bwd_kernel<<<dim3((unsigned)bands, (unsigned)L.num_images), kTileC, sizeof(BwdSmem), st>>>(
        L, rois, off, idx, C, PH, PW, (const bf16*)dout);
    rc = check_launch("roi_align bwd");
  }
  e = cudaFreeAsync(off, st);
  if (rc == C3D_OK && e != cudaSuccess) rc = set_error(C3D_ECUDA, "roi_align bwd buckets free: %s", cudaGetErrorString(e));
  return rc;
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
