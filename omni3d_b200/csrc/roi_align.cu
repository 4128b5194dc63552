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
#include "roi_geom.cuh"

namespace c3d {
using bf16 = __nv_bfloat16;

struct RoiLevels {
  const bf16* feat[5];
  float* grad[5];
  int H[5], W[5];
  float scale[5];
  int num_levels;
  int num_images;
  int grad_bf16;
};

__device__ __forceinline__ void acc8(float (&a)[8], const bf16* p, float w) {
  uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) { float2 f = __bfloat1622float2(h[i]); a[2 * i] += w * f.x; a[2 * i + 1] += w * f.y; }
}

__device__ __forceinline__ bool roi_sane(const float* roi, const RoiLevels& L) {
  return roi_in_range(roi, L.num_images, L.num_levels);
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
// roi_bucket_kernel lists the RoI indices of every (image, level) in index order (a stable counting sort), and with each
// one the rows and columns its bins can reach (a conservative rectangle, computed once per RoI).
//
// roi_align_bwd_kernel: grid = (sum over levels of the 8 x 8 pixel tiles of a map, images).  A block owns one tile of
// one (image, level) gradient map.  It reads the bucket 256 RoIs at a time, drops those whose rectangle misses the tile,
// and lists the bins of the rest that can reach the tile, as "slots" (kSlots at a time, in (RoI, ph, pw) order).  The
// threads stage g = dout / count of every slot (16 bytes of dout per load) and split the (slot, iy, ix) samples among
// themselves; each computes its sample's four taps once and keeps those that fall in the tile as (pixel, slot, weight)
// entries, compacted in (sample, tap) order.  Thread t owns channel cc + t and walks the entries, adding w * g to its
// column of a [64 px][256 ch] fp32 tile in shared memory.  Every element of the map thus receives
// acc = fmaf(w, g, acc), starting from +0, over (RoI, ph, pw, iy, ix, tap) in that order, as one chain, and is stored
// once, zeros included, as fp32 or rounded once to bf16: the maps need no clearing.  Storing the chain is the same as
// adding it to a zeroed map, since the chain is never -0.
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

// Rows [x, y] and columns [z, w] of the map that the bins of a RoI can reach, as the tile kernel tests its bins: bin ph
// is kept for tile rows [t0, t1] when floor(sh + ph * bh) - 1 <= t1 and floor(sh + (ph + 1) * bh) + 1 >= t0.  Those
// bounds grow with ph, so every kept bin lies within floor(sh) - 1 and floor(sh + PH * bh) + 1; one more row on the far
// side covers a different rounding of sh + PH * bh.  Floats, so that no bound of a huge box overflows an int.  A RoI
// with no samples gets an empty rectangle.
__device__ __forceinline__ float4 roi_reach(const float* roi, float sc, int PH, int PW) {
  const RoiGeom g = roi_geom(roi, sc, PH, PW);
  if (g.gh <= 0 || g.gw <= 0) return make_float4(INFINITY, -INFINITY, INFINITY, -INFINITY);
  return make_float4(floorf(g.sh) - 1.f, floorf(fmaf((float)PH, g.bh, g.sh)) + 2.f,
                     floorf(g.sw) - 1.f, floorf(fmaf((float)PW, g.bw, g.sw)) + 2.f);
}

// One block.  Warp w takes the w-th contiguous slice of [0, R) and counts its keys into wk[w][key]; the counts become
// start offsets (bucket by bucket, and warp by warp inside a bucket), and a second pass places every index.
// wk: kBucketWarps x nb ints of scratch; off: nb + 1 bucket offsets; idx: the bucketed RoI indices; reach: their
// roi_reach rectangles, in the same order.
__global__ void __launch_bounds__(kBucketThreads)
roi_bucket_kernel(RoiLevels L, const float* __restrict__ rois, int R, int nb, int PH, int PW, int* __restrict__ wk,
                  int* __restrict__ off, int* __restrict__ idx, float4* __restrict__ reach) {
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
    if (k >= 0) {
      const int at = base + __popc(peers & ((1u << lane) - 1u));
      const float* roi = rois + (size_t)r * 6;
      idx[at] = r;
      reach[at] = roi_reach(roi, L.scale[(int)roi[1]], PH, PW);
    }
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

__device__ __forceinline__ void store_grad(float* p, float v) { *p = v; }
__device__ __forceinline__ void store_grad(bf16* p, float v) { *p = __float2bfloat16_rn(v); }

template <typename OutT>
__global__ void __launch_bounds__(kTileC, 2)
roi_align_bwd_kernel(RoiLevels L, const float* __restrict__ rois, const int* __restrict__ off, const int* __restrict__ idx,
                     const float4* __restrict__ reach, int C, int PH, int PW, const bf16* __restrict__ dout) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  BwdSmem& S = *reinterpret_cast<BwdSmem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31;
  const int b = blockIdx.y;
  int lvl = 0, tile = blockIdx.x;
  auto tiles_of = [&](int l) { return ((L.H[l] + kTile - 1) / kTile) * ((L.W[l] + kTile - 1) / kTile); };
  while (lvl < L.num_levels - 1 && tile >= tiles_of(lvl)) { tile -= tiles_of(lvl); ++lvl; }
  if (tile >= tiles_of(lvl)) return;
  const int H = L.H[lvl], W = L.W[lvl];
  const float sc = L.scale[lvl];
  const int ntx = (W + kTile - 1) / kTile;
  const int ty0 = tile / ntx * kTile, ty1 = min(H, ty0 + kTile) - 1;
  const int tx0 = tile % ntx * kTile, tx1 = min(W, tx0 + kTile) - 1;
  const int key = b * L.num_levels + lvl;
  const int* list = idx + off[key];
  const float4* lreach = reach + off[key];
  const int n = off[key + 1] - off[key];
  OutT* gmap = reinterpret_cast<OutT*>(L.grad[lvl]) + (size_t)b * H * W * C;
  for (int cc = 0; cc < C; cc += kTileC) {
    const int c = cc + tid;
#pragma unroll 8
    for (int p = 0; p < kTile * kTile; ++p) S.acc[p][tid] = 0.f;
    for (int w0 = 0; w0 < n; w0 += kTileC) {
      // ---- the bins of the next kTileC RoIs whose footprint, one pixel wider, overlaps the tile
      int nbin = 0, rect = 0, ri = 0;
      if (w0 + tid < n) {
        const float4 rc = lreach[w0 + tid];
        if (rc.x <= (float)ty1 && rc.y >= (float)ty0 && rc.z <= (float)tx1 && rc.w >= (float)tx0) {
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
      }
      int nbins;
      const int first = block_exclusive_scan(nbin, S.warp, nbins);
      if (nbins == 0) {            // uniform: no RoI of this window reaches the tile
        __syncthreads();
        continue;
      }
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
        // ---- g = dout / count of every slot: 8 channels per load, the slots spread over all threads.  x / 1 == x, so
        // the common single-sample bin skips the division.
        for (int j = tid; j < ns * (kTileC / 8); j += kTileC) {
          const int s = j / (kTileC / 8), q = j % (kTileC / 8) * 8;
          float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
          if (cc + q < C) {
            const uint4 u = __ldg(reinterpret_cast<const uint4*>(
                dout + (((size_t)S.ri[s] * PH + S.ph[s]) * PW + S.pw[s]) * C + cc + q));
            const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
            for (int i = 0; i < 4; ++i) { const float2 f = __bfloat1622float2(h[i]); v[2 * i] = f.x; v[2 * i + 1] = f.y; }
            const float cnt = S.cnt[s];
            if (cnt != 1.f) {
#pragma unroll
              for (int i = 0; i < 8; ++i) v[i] = __fdiv_rn(v[i], cnt);
            }
          }
          float4* dst = reinterpret_cast<float4*>(&S.g[s][q]);
          dst[0] = make_float4(v[0], v[1], v[2], v[3]);
          dst[1] = make_float4(v[4], v[5], v[6], v[7]);
        }
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
        if (py <= ty1 && px <= tx1) store_grad(gmap + ((size_t)py * W + px) * C + c, S.acc[p][tid]);
      }
    }
    __syncthreads();
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
  L.grad_bf16 = lv->grad_bf16;
  if (!bwd) {
    if (R == 0) return C3D_OK;
    long long nbins = (long long)R * PH * PW;
    long long blocks = (nbins + 7) / 8;
    if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
    roi_align_kernel<<<(unsigned)blocks, 256, 0, st>>>(L, rois, R, C, PH, PW, (bf16*)out);
    return check_launch("roi_align");
  }
  if (PH < 1 || PW < 1 || PH > 255 || PW > 255) return set_error(C3D_EINVAL, "roi_align bwd: pooled size outside [1, 255]");
  if (L.grad_bf16 != 0 && L.grad_bf16 != 1) return set_error(C3D_EINVAL, "roi_align bwd: grad_bf16 must be 0 or 1");
  if (R > 0 && reinterpret_cast<uintptr_t>(dout) % 16 != 0)
    return set_error(C3D_EINVAL, "roi_align bwd: dout must be 16-byte aligned");
  auto* kernel = L.grad_bf16 ? roi_align_bwd_kernel<bf16> : roi_align_bwd_kernel<float>;
  static bool attr[2] = {false, false};
  if (!attr[L.grad_bf16]) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BwdSmem));
    if (e != cudaSuccess) return set_error(C3D_ECUDA, "roi_align bwd smem attr: %s", cudaGetErrorString(e));
    attr[L.grad_bf16] = true;
  }
  // the RoI buckets live in stream-ordered scratch: reach rectangles (R float4), offsets (nb + 1), per-warp counts
  // (kBucketWarps x nb), indices (R)
  const int nb = L.num_images * L.num_levels;
  float4* reach = nullptr;
  cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&reach),
                                  (size_t)R * sizeof(float4) + ((size_t)(kBucketWarps + 1) * nb + 1 + R) * sizeof(int), st);
  if (e != cudaSuccess) return set_error(C3D_ECUDA, "roi_align bwd buckets: %s", cudaGetErrorString(e));
  int* off = reinterpret_cast<int*>(reach + R);
  int* wk = off + nb + 1;
  int* idx = wk + (size_t)kBucketWarps * nb;
  roi_bucket_kernel<<<1, kBucketThreads, 0, st>>>(L, rois, R, nb, PH, PW, wk, off, idx, reach);
  int32_t rc = check_launch("roi_align bwd buckets");
  if (rc == C3D_OK) {
    int tiles = 0;
    for (int i = 0; i < L.num_levels; ++i) tiles += ((L.H[i] + kTile - 1) / kTile) * ((L.W[i] + kTile - 1) / kTile);
    kernel<<<dim3((unsigned)tiles, (unsigned)L.num_images), kTileC, sizeof(BwdSmem), st>>>(L, rois, off, idx, reach, C, PH,
                                                                                          PW, (const bf16*)dout);
    rc = check_launch("roi_align bwd");
  }
  e = cudaFreeAsync(reach, st);
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
