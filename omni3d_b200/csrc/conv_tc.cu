// conv_tc.cu — NHWC bf16 implicit-GEMM convolution on the Hopper tensor cores (sm_90a, wgmma).
//
// Replaces the cuDNN convolutions the reference reaches through nn.Conv2d in
//   cubercnn/modeling/backbone/dla.py:43-51,159-161,211-214,241-243,287-297 (DLA34 bottom-up),
//   detectron2 FPN lateral/output convs (built at dla.py:500-506, resnet.py:88-95) and
//   detectron2 StandardRPNHead (configs/Base.yaml:49)
// for forward and (with flipped/transposed weights) data-gradient passes.
//
// GEMM view: M = output pixels, N = Cout, K = KH*KW*Cin.  One CTA computes 128-pixel x BLOCK_N tiles.
// A (activations): for every filter tap one 4-D TMA box [1][TH][TW][BLOCK_K] at the tap's shifted coordinates —
// TMA out-of-bounds zero fill *is* the convolution padding and the element-stride field *is* the convolution
// stride — landing in shared memory as the canonical K-major 128B/64B/32B-swizzled wgmma operand (TH*TW <= 128
// rows).  B (weights, [Cout][KH*KW*Cin] bf16): 2-D TMA box.  Warp-specialised and persistent: warp 8 = TMA producer
// over an mbarrier ring of STAGES slots; warps 0-7 = two consumer warpgroups, each accumulating 64 of the 128 tile
// rows in registers with wgmma (M = 64, N = BLOCK_N) and running the epilogue of its rows (bias / addend / ReLU /
// BatchNorm partial statistics -> bf16|fp32 NHWC stores) while the producer already streams the next tile.
#include <cuda.h>
#include <cuda_bf16.h>
#include <stdlib.h>
#include <string.h>
#include "c3d_common.cuh"
#include "ptx_sm90.cuh"

namespace c3d {

using bf16 = __nv_bfloat16;

constexpr int kConsumerWarps = 8;                       // two consumer warpgroups
constexpr int kGemmThreads = 32 * kConsumerWarps + 32;  // + one TMA producer warp (warp 8)

struct ConvKParams {
  int N, Ho, Wo, Cout;
  int KH, KW, stride, pad;
  int TH, TW, tiles_h, tiles_w;
  int kc_blocks;             // Cin / BLOCK_K
  int Cin;
  const float* bias;         // [Cout] or null
  int relu;
  int out_fp32;
  int add_mode;              // 0 none, 1 same-size, 2 nearest-up2 (addend (N,Ho/2,Wo/2,Cout)), 3 in place
  const bf16* addend;
  void* out;
  long long out_pix_stride;  // elements
  long long out_img_stride, out_h_stride, out_w_stride, out_off;   // output pixel index = img*is + ho*hs + wo*ws + off
  int split_c;               // 0, or: output channels >= split_c live split_off elements further (second output row of the
  long long split_off;       // merged stride-2 data gradient: channel j of pixel (h,w) = dx[2h + j / split_c][2w + ..])
  float* stats;              // [tiles_m][2][Cout] partial (sum, sum of squares) or null
};

template <int BLOCK_N, int BLOCK_K, int STAGES>
struct ConvSmem {
  static constexpr int kABytes = 128 * BLOCK_K * 2;
  static constexpr int kBBytes = BLOCK_N * BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kTileBytes = ((kStageBytes + 1023) / 1024) * 1024;
  static constexpr int kBarOffset = STAGES * kTileBytes;
  static constexpr int kRedOffset = kBarOffset + 256;                      // BatchNorm partial sums [8 warps][2][BLOCK_N]
  static constexpr int kTotal = kRedOffset + kConsumerWarps * 2 * BLOCK_N * 4 + 1024 /*align slack*/;
};

// Epilogue of the 64 rows (output pixels) of a 128 x BLOCK_N tile that consumer warpgroup `wg` accumulated.  A thread
// holds two pixels (rows 16w + l/4 and +8) and, per 8-channel block j, the channel pair 8j + 2(l%4): every store is a
// bf16x2 / float2 of one pixel; the four lanes of a quad cover 8 consecutive channels.
template <int BLOCK_N>
__device__ __forceinline__ void conv_epilogue_tile(const ConvKParams& P, const float (&acc)[BLOCK_N / 2], const int warp,
                                                   const int lane, const int img, const int ho0, const int wo0,
                                                   const int n0, const int tile_m, float* red) {
  bool valid[2];
  long long pix[2], apix[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    const int ty = r / P.TW, tx = r - ty * P.TW;
    const int ho = ho0 + ty, wo = wo0 + tx;
    valid[h] = (r < P.TH * P.TW) && (ho < P.Ho) && (wo < P.Wo);
    pix[h] = (long long)img * P.out_img_stride + (long long)ho * P.out_h_stride + (long long)wo * P.out_w_stride + P.out_off;
    apix[h] = 0;
    if (P.add_mode == 1) apix[h] = ((long long)img * P.Ho + ho) * P.Wo + wo;
    else if (P.add_mode == 2) apix[h] = ((long long)img * (P.Ho >> 1) + (ho >> 1)) * (P.Wo >> 1) + (wo >> 1);
  }
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int c = n0 + 8 * j + cq;                                   // channel pair (c, c + 1)
    if (P.stats) {
      // per-channel sum / sum of squares over the valid rows (raw fp32 accumulators): the two rows of a thread, then
      // the 8 row groups of the warp (lanes with equal l%4); fixed order => deterministic
      const float a0 = valid[0] ? acc[4 * j] : 0.f, a1 = valid[0] ? acc[4 * j + 1] : 0.f;
      const float b0 = valid[1] ? acc[4 * j + 2] : 0.f, b1 = valid[1] ? acc[4 * j + 3] : 0.f;
      float s0 = a0 + b0, s1 = a1 + b1, q0 = a0 * a0 + b0 * b0, q1 = a1 * a1 + b1 * b1;
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        q0 += __shfl_xor_sync(0xffffffffu, q0, o);
        q1 += __shfl_xor_sync(0xffffffffu, q1, o);
      }
      if (lane < 4) {
        float* rs = red + (warp * 2) * BLOCK_N + 8 * j + cq;
        rs[0] = s0; rs[1] = s1; rs[BLOCK_N] = q0; rs[BLOCK_N + 1] = q1;
      }
    }
    if (c >= P.Cout) continue;
    const long long coff = c + ((P.split_c && c >= P.split_c) ? P.split_off : 0);   // channel offset inside the pixel
    float2 bv = make_float2(0.f, 0.f);
    if (P.bias) bv = make_float2(__ldg(P.bias + c), __ldg(P.bias + c + 1));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (!valid[h]) continue;
      float v0 = acc[4 * j + 2 * h] + bv.x, v1 = acc[4 * j + 2 * h + 1] + bv.y;
      if (P.add_mode) {
        const bf16* ap = P.add_mode == 3 ? reinterpret_cast<const bf16*>(P.out) + pix[h] * P.out_pix_stride + coff
                                         : P.addend + apix[h] * P.Cout + c;
        const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(ap));
        v0 += a.x; v1 += a.y;
      }
      if (P.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
      if (P.out_fp32)
        *reinterpret_cast<float2*>(reinterpret_cast<float*>(P.out) + pix[h] * P.out_pix_stride + coff) = make_float2(v0, v1);
      else
        *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<bf16*>(P.out) + pix[h] * P.out_pix_stride + coff) =
            __floats2bfloat162_rn(v0, v1);
    }
  }
  if (P.stats) {
    ptx::named_bar_sync(1, 32 * kConsumerWarps);
    float* dst = P.stats + (size_t)tile_m * 2 * P.Cout;
    for (int i = threadIdx.x; i < 2 * BLOCK_N; i += 32 * kConsumerWarps) {
      const int which = i / BLOCK_N, cc = i - which * BLOCK_N;
      float a = 0.f;
#pragma unroll
      for (int w = 0; w < kConsumerWarps; ++w) a += red[(w * 2 + which) * BLOCK_N + cc];
      if (n0 + cc < P.Cout) dst[which * P.Cout + n0 + cc] = a;
    }
    ptx::named_bar_sync(1, 32 * kConsumerWarps);       // red is reused by this CTA's next tile
  }
}

// Persistent kernel: CTA b walks the (m-tile, n-tile) work items b, b + gridDim.x, ...  The stage ring runs across tile
// boundaries, so the producer loads the next tile while the consumers are in the epilogue of the current one.
template <int BLOCK_N, int BLOCK_K, int STAGES, int CPS>
__global__ void __launch_bounds__(kGemmThreads, CPS)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
               const ConvKParams P, const int tiles_m, const int n_tiles) {
  using S = ConvSmem<BLOCK_N, BLOCK_K, STAGES>;
  constexpr int kSwizzle = BLOCK_K * 2;                       // bytes per smem row = swizzle span
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::kBarOffset);
  uint64_t* empty_bar = full_bar + STAGES;
  float* red = reinterpret_cast<float*>(smem + S::kRedOffset);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_kb = P.KH * P.KW * P.kc_blocks;
  const int total = tiles_m * n_tiles;

  if (warp == kConsumerWarps && lane == 0) {
    ptx::prefetch_tensormap(&tmap_x);
    ptx::prefetch_tensormap(&tmap_w);
    for (int s = 0; s < STAGES; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], kConsumerWarps); }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    // ===== TMA producer =====
    if (ptx::elect_one()) {
      const uint32_t a_bytes = (uint32_t)(P.TH * P.TW * BLOCK_K * 2);
      int stage = 0; uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
        const int tile_m = tile / n_tiles, n0 = (tile - tile_m * n_tiles) * BLOCK_N;
        const int tw_i = tile_m % P.tiles_w, th_i = (tile_m / P.tiles_w) % P.tiles_h;
        const int img = tile_m / (P.tiles_w * P.tiles_h);
        const int hi0 = th_i * P.TH * P.stride - P.pad, wi0 = tw_i * P.TW * P.stride - P.pad;
        int tap = 0, kc = 0, kh = 0, kw = 0;
        for (int kb = 0; kb < num_kb; ++kb) {
          ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * S::kTileBytes;
          ptx::mbar_expect_tx(&full_bar[stage], a_bytes + (uint32_t)S::kBBytes);
          ptx::tma_load_4d(sa, &tmap_x, &full_bar[stage], kc * BLOCK_K, wi0 + kw, hi0 + kh, img);
          ptx::tma_load_2d(sa + S::kABytes, &tmap_w, &full_bar[stage], tap * P.Cin + kc * BLOCK_K, n0);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
          if (++kc == P.kc_blocks) { kc = 0; ++tap; if (++kw == P.KW) { kw = 0; ++kh; } }
        }
      }
    }
  } else {
    // ===== consumer warpgroups: rows 64 * (warp / 4) .. +63 of every tile =====
    constexpr uint32_t lt = ptx::swizzle_layout_type(kSwizzle);
    const uint32_t a_row0 = (uint32_t)((warp >> 2) * 64 * kSwizzle);
    float acc[BLOCK_N / 2];
    int stage = 0; uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x) {
      const int tile_m = tile / n_tiles, n0 = (tile - tile_m * n_tiles) * BLOCK_N;
      const int tw_i = tile_m % P.tiles_w, th_i = (tile_m / P.tiles_w) % P.tiles_h;
      const int img = tile_m / (P.tiles_w * P.tiles_h);
      int prev = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        ptx::mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = ptx::smem_u32(smem + stage * S::kTileBytes);
        const uint64_t da = ptx::make_smem_desc(sa + a_row0, 16, 8 * kSwizzle, lt);
        const uint64_t db = ptx::make_smem_desc(sa + S::kABytes, 16, 8 * kSwizzle, lt);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / 16; ++k)   // 16 bf16 = 32 bytes along K inside the swizzle span: +2 in (addr>>4)
          ptx::wgmma_bf16<BLOCK_N, 0, 0>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb | k) != 0 ? 1u : 0u);
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>();                    // the previous K block's MMAs are done: its slot can be refilled
        if (prev >= 0) { __syncwarp(); if (lane == 0) ptx::mbar_arrive(&empty_bar[prev]); }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      ptx::wgmma_wait<0>();
      ptx::fence_regs(acc);
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&empty_bar[prev]);
      conv_epilogue_tile<BLOCK_N>(P, acc, warp, lane, img, th_i * P.TH, tw_i * P.TW, n0, tile_m, red);
    }
  }
}

// ---- host side --------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}
static CUtensorMapSwizzle swz(int bytes) {
  return bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
}

// choose the output tile (TH x TW <= 128 rows) maximising useful rows
static void pick_tile(int Ho, int Wo, int stride, int* TH, int* TW) {
  double best = -1; int bth = 1, btw = 1;
  for (int tw = 1; tw <= 128 && tw <= Wo; ++tw) {
    if (tw * stride > 256) break;
    int th = 128 / tw; if (th > Ho) th = Ho;
    if (th * stride > 256) th = 256 / stride;
    if (th < 1) continue;
    long long tiles = (long long)((Ho + th - 1) / th) * ((Wo + tw - 1) / tw);
    double eff = (double)Ho * Wo / (double)(tiles * 128);
    if (eff > best + 1e-9 || (eff > best - 1e-9 && tw > btw)) { best = eff; bth = th; btw = tw; }
  }
  *TH = bth; *TW = btw;
}

template <int BN, int BK, int ST, int CPS>
static int32_t launch_conv(const CUtensorMap& mx, const CUtensorMap& mw, const ConvKParams& P, int tiles_m, int n_tiles,
                           cudaStream_t st) {
  using S = ConvSmem<BN, BK, ST>;
  static_assert(CPS * (S::kTotal + 1024) <= 228 * 1024, "conv: shared memory of CPS CTAs exceeds the SM");
  auto kern = conv_tc_kernel<BN, BK, ST, CPS>;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kTotal);
    if (e != cudaSuccess) return set_error(C3D_ECUDA, "conv smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  long long total = (long long)tiles_m * n_tiles;
  long long grid = (long long)kNumSMs * CPS;
  if (grid > total) grid = total;
  kern<<<(unsigned)grid, kGemmThreads, S::kTotal, st>>>(mx, mw, P, tiles_m, n_tiles);
  return check_launch("conv_tc_kernel");
}


// ------------------------------------------------------------------------------------------------
// Weight gradient: dW[co][kh][kw][ci] += sum_pixels dY[p][co] * X[p*stride + tap - pad][ci].
// GEMM view: M = Cout (128 per CTA: 64 per consumer warpgroup), N = (tap, ci) columns — up to 256 per CTA, made of
// whole TMA boxes [pixels][cw channels] (cw = 64/32/16), so small-Cin layers put SEVERAL TAPS side by side in N and dY
// is re-read ceil(taps*Cin/256) times instead of `taps` times — K = pixels.  Both operands are "MN-major" for the
// tensor core (the contiguous NHWC channel axis is M resp. N, pixels are K): the same 4-D TMA boxes as the forward pass
// are consumed through transposed wgmma descriptors.  Grid = (pixel-range split, column group, co tile); split-K
// partials are stored per split and summed in split order by wgrad_reduce_kernel, so the result does not depend on the
// order in which CTAs finish.
struct WgradKParams {
  int N, Ho, Wo, Cout, Cin;
  int KH, KW, stride, pad;
  int RH, RW, tiles_h, tiles_w;
  int num_tiles, tiles_per_split;
  int cw, nci, boxes_per_cta, total_boxes;   // B boxes: width cw channels, nci = Cin / cw per tap
  int ca, a_chunks_max;                      // A boxes: width ca channels
  float* dw;                                 // fp32 gradient (+=), or null when `part` is set
  float* part;                               // split-K partials [splits][welems] (plain stores), reduced in split order
  long long welems;
  int oihw;                                  // 0: dw is [Cout][KH][KW][Cin]; 1: [Cout][Cin][KH][KW] (master layout)
  int big, mc;                               // 1: 5-D tensor maps — ONE box carries all channel chunks of dY (and mc chunks of X)
  int lin;                                   // 1: fully-connected layer (c3d_linear_wgrad): x is (rows, KH*KW*Cin) with the
                                             // features in (tap, ci) order — box b reads channels [b*cw, (b+1)*cw) with no
                                             // spatial shift; KH/KW/Cin only drive the epilogue's master-layout index
};

// two pipeline stages of kPix pixels (GEMM K) x up to kCols GEMM columns per CTA (192 KB)
struct WgradSmem {
  static constexpr int kStages = 2, kPix = 128, kCols = 256;
  static constexpr int kABytes = kPix * 128 * 2;           // up to two [kPix px][64 ch] chunks (or narrower)
  static constexpr int kBBytes = kPix * kCols * 2;         // kCols columns x kPix pixels
  static constexpr int kStageBytes = kABytes + kBBytes;    // 96 KB
  static constexpr int kBarOffset = kStages * kStageBytes;
  static constexpr int kTotal = kBarOffset + 256 + 1024;
};

// main loop + epilogue of one consumer warpgroup with an NB-column accumulator (NB >= the CTA's columns rounded up to
// 64; the extra columns read stale shared memory and are never stored)
template <int NB>
__device__ __forceinline__ void wgrad_consume(const WgradKParams& P, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                              const int t_begin, const int t_end, const int warp, const int lane,
                                              const int co0, const int box0, const int ncols, const uint32_t a_box_bytes,
                                              const uint32_t b_box_bytes) {
  using S = WgradSmem;
  const int wg = warp >> 2;
  const bool active = co0 + wg * 64 < P.Cout;        // this warpgroup's 64 output channels exist
  float acc[NB / 2];
#pragma unroll
  for (int i = 0; i < NB / 2; ++i) acc[i] = 0.f;
  const uint32_t lt_a = ptx::swizzle_layout_type(P.ca * 2), lt_b = ptx::swizzle_layout_type(P.cw * 2);
  const int ksteps = (P.RH * P.RW) / 16;
  // MN-major descriptors: LBO = distance between channel chunks, SBO = 8 pixel rows
  const uint32_t a_sbo = 8 * P.ca * 2, b_sbo = 8 * P.cw * 2;
  const uint32_t a_kstep = (16 * P.ca * 2) >> 4, b_kstep = (16 * P.cw * 2) >> 4;
  const uint32_t a_off = (uint32_t)(wg * (64 / P.ca)) * a_box_bytes;   // first dY chunk of this warpgroup's channels
  int stage = 0; uint32_t phase = 0;
  int prev = -1;
  for (int t = t_begin; t < t_end; ++t) {
    ptx::mbar_wait(&full_bar[stage], phase);
    if (active) {
      const uint32_t sa = ptx::smem_u32(smem + stage * S::kStageBytes);
      const uint64_t da = ptx::make_smem_desc(sa + a_off, a_box_bytes, a_sbo, lt_a);
      const uint64_t db = ptx::make_smem_desc(sa + S::kABytes, b_box_bytes, b_sbo, lt_b);
      ptx::wgmma_fence();
      for (int k = 0; k < ksteps; ++k)
        ptx::wgmma_bf16<NB, 1, 1>(acc, da + (uint64_t)(a_kstep * k), db + (uint64_t)(b_kstep * k), 1u);
      ptx::wgmma_commit();
      ptx::wgmma_wait<1>();
    }
    if (prev >= 0) { __syncwarp(); if (lane == 0) ptx::mbar_arrive(&empty_bar[prev]); }
    prev = stage;
    if (++stage == S::kStages) { stage = 0; phase ^= 1; }
  }
  ptx::wgmma_wait<0>();
  ptx::fence_regs(acc);
  __syncwarp();
  if (lane == 0) ptx::mbar_arrive(&empty_bar[prev]);
  if (!active) return;
  const int taps = P.KH * P.KW;
#pragma unroll
  for (int j = 0; j < NB / 8; ++j) {
    const int n = 8 * j + 2 * (lane & 3);             // column pair (n, n + 1): same box, consecutive ci
    if (n >= ncols) continue;
    const int box = box0 + n / P.cw;
    const int tap = box / P.nci, ci = (box - tap * P.nci) * P.cw + (n % P.cw);
    if (ci >= P.Cin) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int co = co0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
      if (co >= P.Cout) continue;
      const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      // one writer per element: a plain store of this split's partial, or (single split) dw +=
      float* base = P.part ? P.part + (size_t)blockIdx.x * P.welems : P.dw;
      if (P.oihw) {
        float* dst = base + ((size_t)co * P.Cin + ci) * taps + tap;
        if (P.part) { dst[0] = v0; dst[taps] = v1; } else { dst[0] += v0; dst[taps] += v1; }
      } else {
        float2* dst = reinterpret_cast<float2*>(base + ((size_t)co * taps + tap) * P.Cin + ci);
        if (P.part) *dst = make_float2(v0, v1);
        else { float2 o = *dst; o.x += v0; o.y += v1; *dst = o; }
      }
    }
  }
}

// dw[e] += sum over s of part[s][e], summed in s order (deterministic split-K reduction)
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, int nparts, long long welems, float* __restrict__ dw) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < welems; e += (long long)gridDim.x * blockDim.x) {
    float a = 0.f;
    for (int s = 0; s < nparts; ++s) a += part[(size_t)s * welems + e];
    dw[e] += a;
  }
}
// runs `launch(part)` with a stream-ordered partial buffer of nparts x welems floats (null when nparts == 1: the kernel
// then adds into dw itself), then reduces the partials into dw in a fixed order
template <typename F>
static int32_t with_ordered_partials(int nparts, long long welems, float* dw, cudaStream_t st, F launch) {
  if (nparts <= 1) return launch(nullptr);
  float* part = nullptr;
  cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&part), (size_t)nparts * welems * sizeof(float), st);
  if (e != cudaSuccess) return set_error(C3D_ECUDA, "wgrad partials: %s", cudaGetErrorString(e));
  int32_t rc = launch(part);
  if (rc == C3D_OK) {
    long long blocks = (welems + 255) / 256;
    if (blocks > 8LL * kNumSMs) blocks = 8LL * kNumSMs;
    wgrad_reduce_kernel<<<(unsigned)blocks, 256, 0, st>>>(part, nparts, welems, dw);
    rc = check_launch("wgrad_reduce_kernel");
  }
  e = cudaFreeAsync(part, st);
  if (rc == C3D_OK && e != cudaSuccess) rc = set_error(C3D_ECUDA, "wgrad partials free: %s", cudaGetErrorString(e));
  return rc;
}

__global__ void __launch_bounds__(kGemmThreads, 1)
conv_wgrad_tc_kernel(const __grid_constant__ CUtensorMap tmap_dy, const __grid_constant__ CUtensorMap tmap_x,
                     const WgradKParams P) {
  using S = WgradSmem;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::kBarOffset);
  uint64_t* empty_bar = full_bar + S::kStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  const int split = blockIdx.x, group = blockIdx.y, co_tile = blockIdx.z;
  const int co0 = co_tile * 128;
  const int box0 = group * P.boxes_per_cta;
  const int nb = min(P.boxes_per_cta, P.total_boxes - box0);       // boxes (taps x ci chunks) of this CTA
  const int ncols = nb * P.cw;                                     // GEMM N (multiple of 16, <= S::kCols)
  const int t_begin = split * P.tiles_per_split;
  const int t_end = min(P.num_tiles, t_begin + P.tiles_per_split);
  if (t_begin >= t_end) return;
  const int R = P.RH * P.RW;
  int a_chunks = (P.Cout - co0 + P.ca - 1) / P.ca;
  if (a_chunks > P.a_chunks_max) a_chunks = P.a_chunks_max;
  // distance between channel chunks in shared memory: a full kPix-pixel slot per box, or (5-D boxes) the dense box pitch
  const uint32_t a_box_bytes = (uint32_t)((P.big ? R : S::kPix) * P.ca * 2), b_box_bytes = (uint32_t)((P.big ? R : S::kPix) * P.cw * 2);

  if (warp == kConsumerWarps && lane == 0) {
    ptx::prefetch_tensormap(&tmap_dy); ptx::prefetch_tensormap(&tmap_x);
    for (int s = 0; s < S::kStages; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], kConsumerWarps); }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    if (ptx::elect_one()) {
      int stage = 0; uint32_t phase = 0;
      const uint32_t bytes = (uint32_t)(R * 2 * ((P.big ? P.a_chunks_max : a_chunks) * P.ca + nb * P.cw));
      for (int t = t_begin; t < t_end; ++t) {
        const int tw_i = t % P.tiles_w, th_i = (t / P.tiles_w) % P.tiles_h, img = t / (P.tiles_w * P.tiles_h);
        const int ho0 = th_i * P.RH, wo0 = tw_i * P.RW;
        ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sa = smem + stage * S::kStageBytes;
        uint8_t* sb = sa + S::kABytes;
        ptx::mbar_expect_tx(&full_bar[stage], bytes);
        if (P.big) {
          ptx::tma_load_5d(sa, &tmap_dy, &full_bar[stage], 0, wo0, ho0, co0 / P.ca, img);
          for (int b = 0; b < nb; b += P.mc) {
            const int box = box0 + b;
            const int tap = box / P.nci, chunk = box - tap * P.nci;
            const int kh = tap / P.KW, kw = tap - kh * P.KW;
            if (P.lin)
              ptx::tma_load_5d(sb + b * b_box_bytes, &tmap_x, &full_bar[stage], 0, wo0, ho0, box, img);
            else
              ptx::tma_load_5d(sb + b * b_box_bytes, &tmap_x, &full_bar[stage], 0, wo0 * P.stride + kw - P.pad,
                               ho0 * P.stride + kh - P.pad, chunk, img);
          }
        } else {
          for (int c = 0; c < a_chunks; ++c)
            ptx::tma_load_4d(sa + c * a_box_bytes, &tmap_dy, &full_bar[stage], co0 + P.ca * c, wo0, ho0, img);
          for (int b = 0; b < nb; ++b) {
            const int box = box0 + b;
            const int tap = box / P.nci, chunk = box - tap * P.nci;
            const int kh = tap / P.KW, kw = tap - kh * P.KW;
            if (P.lin)
              ptx::tma_load_4d(sb + b * b_box_bytes, &tmap_x, &full_bar[stage], box * P.cw, wo0, ho0, img);
            else
              ptx::tma_load_4d(sb + b * b_box_bytes, &tmap_x, &full_bar[stage], chunk * P.cw,
                               wo0 * P.stride + kw - P.pad, ho0 * P.stride + kh - P.pad, img);
          }
        }
        if (++stage == S::kStages) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    if (ncols > 192)
      wgrad_consume<256>(P, smem, full_bar, empty_bar, t_begin, t_end, warp, lane, co0, box0, ncols, a_box_bytes, b_box_bytes);
    else if (ncols > 128)
      wgrad_consume<192>(P, smem, full_bar, empty_bar, t_begin, t_end, warp, lane, co0, box0, ncols, a_box_bytes, b_box_bytes);
    else if (ncols > 64)
      wgrad_consume<128>(P, smem, full_bar, empty_bar, t_begin, t_end, warp, lane, co0, box0, ncols, a_box_bytes, b_box_bytes);
    else
      wgrad_consume<64>(P, smem, full_bar, empty_bar, t_begin, t_end, warp, lane, co0, box0, ncols, a_box_bytes, b_box_bytes);
  }
}

// pixel box for wgrad: RH*RW must be a multiple of 16 (wgmma K) and <= WgradSmem::kPix
static void pick_tile_k(int Ho, int Wo, int stride, int* RH, int* RW) {
  constexpr int max_pix = WgradSmem::kPix;
  double best = -1; int bth = 1, btw = 16;
  for (int tw = 1; tw <= max_pix; ++tw) {
    if (tw * stride > 256) break;
    if (tw > Wo && tw != 16) continue;
    for (int th = 1; th * tw <= max_pix; ++th) {
      if ((th * tw) % 16 != 0 || th * stride > 256) continue;
      long long tiles = (long long)((Ho + th - 1) / th) * ((Wo + tw - 1) / tw);
      double eff = (double)Ho * Wo / (double)(tiles * th * tw) * (th * tw >= 64 ? 1.0 : 0.9);
      if (eff > best + 1e-9 || (eff > best - 1e-9 && th * tw > bth * btw)) { best = eff; bth = th; btw = tw; }
    }
  }
  *RH = bth; *RW = btw;
}

}  // namespace c3d

#include "conv_halo.cuh"

using namespace c3d;

extern "C" int32_t c3d_conv2d_tiles(const c3d_conv_desc* d, int32_t* tiles_m, int32_t* TH, int32_t* TW) {
  if (!d) return set_error(C3D_EINVAL, "null desc");
  int Ho = d->out_h > 0 ? d->out_h : (d->H + 2 * d->pad - d->KH) / d->stride + 1;
  int Wo = d->out_w > 0 ? d->out_w : (d->W + 2 * d->pad - d->KW) / d->stride + 1;
  if (halo_fwd_eligible(d)) {          // one partial-statistics row per persistent CTA
    if (TH) *TH = 1;
    if (TW) *TW = 128;
    if (tiles_m) *tiles_m = halo_fwd_grid(d);
    return C3D_OK;
  }
  int th, tw;
  pick_tile(Ho, Wo, d->stride, &th, &tw);
  if (TH) *TH = th;
  if (TW) *TW = tw;
  if (tiles_m) *tiles_m = d->N * ((Ho + th - 1) / th) * ((Wo + tw - 1) / tw);
  return C3D_OK;
}

extern "C" int32_t c3d_conv2d_fwd(const c3d_conv_desc* d, const void* x, const void* w, const float* bias,
                                  const void* addend, void* y, float* stats, void* stream) {
  if (!d || !x || !w || !y) return set_error(C3D_EINVAL, "conv2d: null pointer");
  const int Cin = d->Cin, Cout = d->Cout;
  if (halo_fwd_eligible(d)) return launch_halo_fwd(d, x, w, bias, y, stats, static_cast<cudaStream_t>(stream));
  if (Cin % 16 != 0 || Cin <= 0) return set_error(C3D_EINVAL, "conv2d: Cin=%d must be a multiple of 16", Cin);
  if (Cout % 16 != 0 || Cout <= 0) return set_error(C3D_EINVAL, "conv2d: Cout=%d must be a multiple of 16", Cout);
  if (d->stride < 1 || d->stride > 2) return set_error(C3D_EINVAL, "conv2d: stride %d unsupported", d->stride);
  const int BK = (Cin % 64 == 0) ? 64 : (Cin % 32 == 0 ? 32 : 16);
  int BN = 128;
  if (Cout % 128 != 0) BN = (Cout % 64 == 0) ? 64 : (Cout % 32 == 0 ? 32 : 16);
  // N = 256 (one CTA per SM, 128 accumulator registers per thread) for the layers with several 64-deep K blocks; the
  // 1x1 layers over <= 64 channels are memory-bound and keep two CTAs per SM
  if (BK == 64 && !(d->KH == 1 && Cin <= 64) && Cout % 256 == 0) BN = 256;
  const int Ho = d->out_h > 0 ? d->out_h : (d->H + 2 * d->pad - d->KH) / d->stride + 1;
  const int Wo = d->out_w > 0 ? d->out_w : (d->W + 2 * d->pad - d->KW) / d->stride + 1;
  if (d->add_mode == 2 && ((Ho & 1) || (Wo & 1))) return set_error(C3D_EINVAL, "conv2d: up2 addend needs even output");
  if ((d->add_mode == 1 || d->add_mode == 2) && !addend) return set_error(C3D_EINVAL, "conv2d: addend missing");
  if (d->add_mode == 3 && d->out_fp32) return set_error(C3D_EINVAL, "conv2d: in-place accumulate needs a bf16 output");
  if (d->add_mode < 0 || d->add_mode > 3) return set_error(C3D_EINVAL, "conv2d: add_mode %d", d->add_mode);
  if (d->y_split_c && (d->y_split_c % 16 != 0 || d->add_mode == 1 || d->add_mode == 2 || stats))
    return set_error(C3D_EINVAL, "conv2d: y_split_c must be a multiple of 16 without addend / statistics");
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error(C3D_ECUDA, "cuTensorMapEncodeTiled unavailable");

  ConvKParams P;
  P.N = d->N; P.Ho = Ho; P.Wo = Wo; P.Cout = Cout; P.KH = d->KH; P.KW = d->KW; P.stride = d->stride; P.pad = d->pad;
  pick_tile(Ho, Wo, d->stride, &P.TH, &P.TW);
  P.tiles_h = (Ho + P.TH - 1) / P.TH; P.tiles_w = (Wo + P.TW - 1) / P.TW;
  P.kc_blocks = Cin / BK; P.Cin = Cin;
  P.bias = bias; P.relu = d->relu; P.out_fp32 = d->out_fp32; P.add_mode = d->add_mode;
  P.addend = static_cast<const bf16*>(addend);
  P.out = y; P.out_pix_stride = d->y_pix_stride ? d->y_pix_stride : Cout;
  if (d->y_img_stride) {
    P.out_img_stride = d->y_img_stride; P.out_h_stride = d->y_h_stride; P.out_w_stride = d->y_w_stride; P.out_off = d->y_offset;
  } else {
    P.out_img_stride = (long long)Ho * Wo; P.out_h_stride = Wo; P.out_w_stride = 1; P.out_off = 0;
  }
  P.split_c = d->y_split_c; P.split_off = d->y_split_off;
  P.stats = stats;

  CUtensorMap mx, mw;
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)d->N};
    cuuint64_t strides[3] = {(cuuint64_t)Cin * 2, (cuuint64_t)Cin * 2 * d->W,
                             (cuuint64_t)Cin * 2 * (d->x_img_stride ? d->x_img_stride : (long long)d->W * d->H)};
    cuuint32_t box[4] = {(cuuint32_t)BK, (cuuint32_t)(P.TW * d->stride), (cuuint32_t)(P.TH * d->stride), 1};
    cuuint32_t estr[4] = {1, (cuuint32_t)d->stride, (cuuint32_t)d->stride, 1};
    CUresult r = enc(&mx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(x), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swz(BK * 2), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(C3D_ECUDA, "encode x tensormap failed: %d", (int)r);
  }
  {
    const long long Kt = (long long)d->KH * d->KW * Cin;
    cuuint64_t dims[2] = {(cuuint64_t)Kt, (cuuint64_t)Cout};
    cuuint64_t strides[1] = {(cuuint64_t)Kt * 2};
    cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)BN};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&mw, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(w), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swz(BK * 2), CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(C3D_ECUDA, "encode w tensormap failed: %d", (int)r);
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int tiles_m = d->N * P.tiles_h * P.tiles_w, n_tiles = Cout / BN;
  // (BN, BK) -> pipeline stages, CTAs per SM: N = 256 fills the register file with one CTA; the others run two CTAs so
  // that one CTA's epilogue overlaps the other's main loop
#define C3D_CONV_CASE(bn, bk, stg, cps) \
  if (BN == bn && BK == bk) return launch_conv<bn, bk, stg, cps>(mx, mw, P, tiles_m, n_tiles, st);
  C3D_CONV_CASE(256, 64, 4, 1)
  C3D_CONV_CASE(128, 64, 3, 2)
  C3D_CONV_CASE(64, 64, 4, 2)
  C3D_CONV_CASE(32, 64, 4, 2)
  C3D_CONV_CASE(16, 64, 4, 2)
  C3D_CONV_CASE(128, 32, 6, 2)
  C3D_CONV_CASE(64, 32, 6, 2)
  C3D_CONV_CASE(32, 32, 6, 2)
  C3D_CONV_CASE(16, 32, 6, 2)
  C3D_CONV_CASE(128, 16, 8, 2)
  C3D_CONV_CASE(64, 16, 8, 2)
  C3D_CONV_CASE(32, 16, 8, 2)
  C3D_CONV_CASE(16, 16, 8, 2)
#undef C3D_CONV_CASE
  return set_error(C3D_EINVAL, "conv2d: no kernel for BN=%d BK=%d", BN, BK);
}

// lin_c > 0: fully-connected layer — d describes the layer as a 1x1 conv over (1,1,rows) "pixels" with d->Cin input
// features that are laid out as (lin_pp taps) x (lin_c channels); the epilogue then addresses dw as [Cout][lin_c][lin_pp]
// when oihw (the nn.Linear master weight over a (C,P,P)-flattened input) or [Cout][lin_pp][lin_c] otherwise.
static int32_t wgrad_impl(const c3d_conv_desc* d, const void* x, const void* dy, float* dw, int32_t oihw, void* stream,
                          int lin_c, int lin_pp) {
  if (!d || !x || !dy || !dw) return set_error(C3D_EINVAL, "wgrad: null pointer");
  const int Cin = d->Cin, Cout = d->Cout;
  if (!lin_c && halo_wgrad_eligible(d)) return launch_halo_wgrad(d, x, dy, dw, oihw, static_cast<cudaStream_t>(stream));
  if (Cin % 16 != 0 || Cout % 16 != 0) return set_error(C3D_EINVAL, "wgrad: channels must be multiples of 16");
  if (d->stride < 1 || d->stride > 2) return set_error(C3D_EINVAL, "wgrad: stride %d unsupported", d->stride);
  const int Ho = (d->H + 2 * d->pad - d->KH) / d->stride + 1;
  const int Wo = (d->W + 2 * d->pad - d->KW) / d->stride + 1;
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error(C3D_ECUDA, "cuTensorMapEncodeTiled unavailable");
  WgradKParams P;
  P.N = d->N; P.Ho = Ho; P.Wo = Wo; P.Cout = Cout; P.Cin = Cin;
  P.KH = d->KH; P.KW = d->KW; P.stride = d->stride; P.pad = d->pad;
  P.lin = lin_c > 0;
  if (P.lin) {
    if (d->KH != 1 || d->KW != 1 || d->stride != 1 || d->pad != 0 || lin_c % 16 != 0 || (long long)lin_c * lin_pp != Cin)
      return set_error(C3D_EINVAL, "linear wgrad: bad feature factorisation %d x %d != %d", lin_c, lin_pp, Cin);
    P.Cin = lin_c; P.KH = lin_pp; P.KW = 1;      // epilogue index space: (tap = p, ci = c); the loader ignores kh / kw
  }
  pick_tile_k(Ho, Wo, d->stride, &P.RH, &P.RW);
  P.tiles_h = (Ho + P.RH - 1) / P.RH; P.tiles_w = (Wo + P.RW - 1) / P.RW;
  P.num_tiles = d->N * P.tiles_h * P.tiles_w;
  const int taps = P.KH * P.KW;
  const int Cin_e = P.Cin;                       // channels per tap in the epilogue's index space
  P.cw = (Cin_e % 64 == 0) ? 64 : (Cin_e % 32 == 0 ? 32 : 16);
  P.nci = Cin_e / P.cw;
  P.boxes_per_cta = WgradSmem::kCols / P.cw;
  P.total_boxes = taps * P.nci;
  P.ca = (Cout % 64 == 0) ? 64 : (Cout % 32 == 0 ? 32 : 16);
  P.a_chunks_max = 128 / P.ca;    // chunks beyond Cout are not loaded (those D rows are never stored)
  const int groups = (P.total_boxes + P.boxes_per_cta - 1) / P.boxes_per_cta;
  const int co_tiles = (Cout + 127) / 128;
  // split-K over pixels (1 CTA/SM): every split adds a 128 x N partial to the ordered reduction, so big weight tensors get exactly one
  // wave of CTAs (<= kNumSMs) while small ones (<= 64K elements: the pixel-heavy early layers) get ~4 waves for balance
  long long base = (long long)groups * co_tiles;
  const long long welems = (long long)Cout * taps * Cin_e;
  int splits = welems <= 65536 ? (int)((4LL * kNumSMs + base - 1) / base) : (int)(kNumSMs / base);
  if (splits > P.num_tiles) splits = P.num_tiles;
  if (splits < 1) splits = 1;
  P.tiles_per_split = (P.num_tiles + splits - 1) / splits;
  splits = (P.num_tiles + P.tiles_per_split - 1) / P.tiles_per_split;
  P.dw = dw;
  P.part = nullptr;
  P.welems = welems;
  P.oihw = oihw;
  const long long yps = d->y_pix_stride ? d->y_pix_stride : Cout;
  CUtensorMap mdy, mx;
  // 5-D maps (channel-chunk axis OUTSIDE the pixel axes): one box = [chunks][RH][RW][64 ch], the MN-major operand layout
  // with LBO = RH*RW*128 B — a third of the TMA instructions per stage (the loop is bound by boxes issued, not bytes)
  P.big = 0; P.mc = 1;
  {
    const int nchunks_x = P.lin ? P.total_boxes : P.nci;
    int mc = P.boxes_per_cta;
    while (mc > 1 && nchunks_x % mc != 0) mc >>= 1;
    const int nca = (Cout + P.ca - 1) / P.ca;
    const long long ximg = d->x_img_stride ? d->x_img_stride : (long long)d->W * d->H;
    cuuint64_t dy_dims[5] = {(cuuint64_t)P.ca, (cuuint64_t)Wo, (cuuint64_t)Ho, (cuuint64_t)nca, (cuuint64_t)d->N};
    cuuint64_t dy_str[4] = {(cuuint64_t)yps * 2, (cuuint64_t)yps * 2 * Wo, (cuuint64_t)P.ca * 2, (cuuint64_t)yps * 2 * Wo * Ho};
    cuuint32_t dy_box[5] = {(cuuint32_t)P.ca, (cuuint32_t)P.RW, (cuuint32_t)P.RH, (cuuint32_t)P.a_chunks_max, 1};
    cuuint32_t one5[5] = {1, 1, 1, 1, 1};
    cuuint64_t x_dims[5] = {(cuuint64_t)P.cw, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)nchunks_x, (cuuint64_t)d->N};
    cuuint64_t x_str[4] = {(cuuint64_t)Cin * 2, (cuuint64_t)Cin * 2 * d->W, (cuuint64_t)P.cw * 2, (cuuint64_t)Cin * 2 * ximg};
    cuuint32_t x_box[5] = {(cuuint32_t)P.cw, (cuuint32_t)(P.RW * d->stride), (cuuint32_t)(P.RH * d->stride), (cuuint32_t)mc, 1};
    cuuint32_t x_es[5] = {1, (cuuint32_t)d->stride, (cuuint32_t)d->stride, 1, 1};
    CUresult r1 = enc(&mdy, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(dy), dy_dims, dy_str, dy_box, one5,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, swz(P.ca * 2), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CUresult r2 = enc(&mx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(x), x_dims, x_str, x_box, x_es,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, swz(P.cw * 2), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r1 == CUDA_SUCCESS && r2 == CUDA_SUCCESS) { P.big = 1; P.mc = mc; }
    else {
      static bool warned = false;
      if (!warned) { fprintf(stderr, "c3d wgrad: 5-D tensor map rejected (%d, %d), using per-chunk boxes\n", (int)r1, (int)r2); warned = true; }
    }
  }
  if (!P.big) {
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cout, (cuuint64_t)Wo, (cuuint64_t)Ho, (cuuint64_t)d->N};
    cuuint64_t strides[3] = {(cuuint64_t)yps * 2, (cuuint64_t)yps * 2 * Wo, (cuuint64_t)yps * 2 * Wo * Ho};
    cuuint32_t box[4] = {(cuuint32_t)P.ca, (cuuint32_t)P.RW, (cuuint32_t)P.RH, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(&mdy, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(dy), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swz(P.ca * 2), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(C3D_ECUDA, "encode dy tensormap failed: %d", (int)r);
  }
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)d->N};
    cuuint64_t strides[3] = {(cuuint64_t)Cin * 2, (cuuint64_t)Cin * 2 * d->W,
                             (cuuint64_t)Cin * 2 * (d->x_img_stride ? d->x_img_stride : (long long)d->W * d->H)};
    cuuint32_t box[4] = {(cuuint32_t)P.cw, (cuuint32_t)(P.RW * d->stride), (cuuint32_t)(P.RH * d->stride), 1};
    cuuint32_t estr[4] = {1, (cuuint32_t)d->stride, (cuuint32_t)d->stride, 1};
    CUresult r = enc(&mx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(x), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swz(P.cw * 2), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(C3D_ECUDA, "encode x tensormap failed: %d", (int)r);
  }
  }
  dim3 grid((unsigned)splits, (unsigned)groups, (unsigned)co_tiles);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(conv_wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         WgradSmem::kTotal);
    if (e != cudaSuccess) return set_error(C3D_ECUDA, "wgrad smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  return with_ordered_partials(splits, welems, dw, st, [&](float* part) -> int32_t {
    WgradKParams Q = P;
    Q.part = part;
    conv_wgrad_tc_kernel<<<grid, kGemmThreads, WgradSmem::kTotal, st>>>(mdy, mx, Q);
    return check_launch("conv_wgrad_tc_kernel");
  });
}

extern "C" int32_t c3d_conv2d_wgrad(const c3d_conv_desc* d, const void* x, const void* dy, float* dw, int32_t oihw,
                                    void* stream) {
  return wgrad_impl(d, x, dy, dw, oihw, stream, 0, 0);
}

// ------------------------------------------------------------------------------------------------
// Fully-connected layers of the box head / cube head (detectron2 FastRCNNConvFCHead, configs/Base.yaml:67-70;
// cubercnn/modeling/roi_heads/cube_head.py:63-73,108-144) on the SAME wgmma kernels: a linear layer over `rows`
// feature vectors is the 1x1 convolution of a (1, 1, rows, K) "image" — 128-row M tiles, persistent CTAs, BLOCK_N 256,
// bias + ReLU fused in the epilogue; the weight gradient is the split-K MN-major GEMM of conv_wgrad_tc_kernel.
namespace c3d {
// fp32 master (N, K = C*PP) whose input features are ordered (c, p) [nn.Linear over a (C,P,P)-flattened NCHW RoI] ->
// bf16 (N, K') with K' ordered (p, c) [the NHWC-flattened RoI the ROIAlign kernel produces].  PP == 1: plain cast.
__global__ void pack_linear_rows_kernel(const float* __restrict__ w, int N, int C, int PP, bf16* __restrict__ out) {
  extern __shared__ float tile[];                       // [64 channels][PP]
  const int n = blockIdx.y, c0 = blockIdx.x * 64;
  const int nc = min(64, C - c0);
  const float* src = w + ((size_t)n * C + c0) * PP;
  for (int i = threadIdx.x; i < nc * PP; i += blockDim.x) tile[i] = src[i];
  __syncthreads();
  bf16* dst = out + (size_t)n * C * PP + c0;
  for (int i = threadIdx.x; i < nc * PP; i += blockDim.x) {
    const int p = i / nc, c = i - p * nc;
    dst[(size_t)p * C + c] = __float2bfloat16(tile[c * PP + p]);
  }
}
// bf16 (R, Cc) -> bf16 (Cc, R)
__global__ void transpose_bf16_kernel(const bf16* __restrict__ in, int R, int Cc, bf16* __restrict__ out) {
  __shared__ bf16 t[64][66];
  const int r0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
  for (int i = threadIdx.y; i < 64; i += blockDim.y) {
    const int r = r0 + i;
    for (int j = threadIdx.x; j < 64; j += blockDim.x)
      if (r < R && c0 + j < Cc) t[i][j] = in[(size_t)r * Cc + c0 + j];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 64; i += blockDim.y) {
    const int c = c0 + i;
    for (int j = threadIdx.x; j < 64; j += blockDim.x)
      if (c < Cc && r0 + j < R) out[(size_t)c * R + r0 + j] = t[j][i];
  }
}
// the layer over nseg blocks of seg_rows rows as a 1x1 convolution of nseg (1, seg_rows) "images" with K input and N
// output channels; block b starts at row b * seg_stride of the strided operand, which the caller places.  d->N == 0:
// nothing to compute.
static int32_t linear_desc(c3d_conv_desc* d, int32_t nseg, int64_t seg_rows, int64_t seg_stride, int K, int N) {
  memset(d, 0, sizeof(*d));
  if (nseg <= 0 || seg_rows <= 0) return C3D_OK;
  if (seg_rows > 0x7fffffffLL) return set_error(C3D_EINVAL, "linear: seg_rows %lld exceeds INT32_MAX", (long long)seg_rows);
  if (seg_stride < seg_rows) return set_error(C3D_EINVAL, "linear: seg_stride < seg_rows");
  d->N = nseg; d->H = 1; d->W = (int32_t)seg_rows; d->Cin = K; d->Cout = N; d->KH = 1; d->KW = 1; d->stride = 1; d->pad = 0;
  return C3D_OK;
}
}  // namespace c3d

extern "C" int32_t c3d_pack_linear_weight(const float* w, int32_t N, int32_t K, int32_t C, int32_t PP, void* w_bf16,
                                          void* wt_bf16, void* stream) {
  if (!w || !w_bf16 || !wt_bf16 || N <= 0 || K <= 0) return set_error(C3D_EINVAL, "pack_linear_weight: bad args");
  if (C <= 0 || PP <= 0) { C = K; PP = 1; }
  if ((long long)C * PP != K || PP > 256) return set_error(C3D_EINVAL, "pack_linear_weight: C*PP != K");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  dim3 g((C + 63) / 64, N);
  pack_linear_rows_kernel<<<g, 256, 64 * PP * sizeof(float), st>>>(w, N, C, PP, (bf16*)w_bf16);
  dim3 gt((K + 63) / 64, (N + 63) / 64);
  transpose_bf16_kernel<<<gt, dim3(32, 8), 0, st>>>((const bf16*)w_bf16, N, K, (bf16*)wt_bf16);
  return check_launch("pack_linear_weight");
}

extern "C" int32_t c3d_linear_fwd(const void* x, const void* w, const float* bias, void* y, int32_t nseg, int64_t seg_rows,
                                  int64_t seg_stride, int32_t K, int32_t N, int32_t relu, int32_t out_fp32, void* stream) {
  c3d_conv_desc d;
  const int32_t rc = linear_desc(&d, nseg, seg_rows, seg_stride, K, N);
  if (rc != C3D_OK || d.N == 0) return rc;
  d.x_img_stride = seg_stride;
  d.relu = relu; d.out_fp32 = out_fp32;
  return c3d_conv2d_fwd(&d, x, w, bias, nullptr, y, nullptr, stream);
}

extern "C" int32_t c3d_linear_dgrad(const void* dy, const void* wt, void* dx, int32_t nseg, int64_t seg_rows,
                                    int64_t seg_stride, int32_t N, int32_t K, int32_t accumulate, void* stream) {
  c3d_conv_desc d;
  const int32_t rc = linear_desc(&d, nseg, seg_rows, seg_stride, N, K);   // dx = dy . W: 1x1 conv with weight W^T (K, N)
  if (rc != C3D_OK || d.N == 0) return rc;
  d.y_img_stride = seg_stride; d.y_h_stride = seg_rows; d.y_w_stride = 1; d.y_offset = 0;
  d.add_mode = accumulate ? 3 : 0;
  return c3d_conv2d_fwd(&d, dy, wt, nullptr, nullptr, dx, nullptr, stream);
}

extern "C" int32_t c3d_linear_wgrad(const void* x, const void* dy, float* dw, int32_t nseg, int64_t seg_rows,
                                    int64_t seg_stride, int32_t K, int32_t N, int32_t C, int32_t PP, void* stream) {
  c3d_conv_desc d;
  const int32_t rc = linear_desc(&d, nseg, seg_rows, seg_stride, K, N);
  if (rc != C3D_OK || d.N == 0) return rc;
  d.x_img_stride = seg_stride;
  if (C <= 0 || PP <= 0) { C = K; PP = 1; }
  return wgrad_impl(&d, x, dy, dw, PP > 1, stream, C, PP);
}
