// conv_halo.cuh — "thin-channel" stride-1 convolutions (Cin, Cout <= 32) on wgmma with a rolling halo of input
// rows in shared memory.  Included by conv_tc.cu (same translation unit: shares the tensor-map encoder).
//
// Why a second kernel: for the 640x640 stem (7x7, 3->16) and level0 (3x3, 16->16) of DLA-34
// (cubercnn/modeling/backbone/dla.py:287-297) the tap-per-TMA-box implicit GEMM of conv_tc_kernel moves
// taps x 128 px x Cin x 2 B through L2->smem per 128 output pixels (196 KB for the stem) while the math is tiny:
// the layer would be L2->SM bandwidth bound far above its HBM roofline.  Here every input row is brought to shared
// memory ONCE per 128-pixel strip, as planes of 8 channels ([plane][pixel][8 ch], 16 B per pixel), and the tensor
// core reads its A operand *in place* through no-swizzle (INTERLEAVE) wgmma descriptors:
//   K-major canonical form  ((8,m),(T,2)) : ((16 B, SBO), (1, LBO))        (cute GMMA::Layout_K_INTER_Atom)
//   rows = consecutive pixels (16 B apart, SBO = 128 B per group of 8), the two 8-wide K chunks of one MMA are
//   either two channel planes (LBO = plane bytes) or — for the 8-channel stem — two adjacent taps (LBO = 16 B).
// A filter tap is therefore just a different descriptor start address (+kw*16 B, other ring slot for kh): no
// im2col copy exists anywhere.  The CTA walks down a strip, so each new output row costs ONE new input row of TMA.
//
// The weight gradient uses the same resident rows as an MN-major operand: M = 8 pixel shifts (= kw) x 8 channels,
// K = pixels, N = Cout from dY staged the same way; one register accumulator per (kh, plane) accumulates over every
// row the CTA visits and is stored once as the CTA's partial; the partials are summed in CTA order.
#pragma once

namespace c3d {

struct HaloParams {
  int N, H, W, Cin, Cout, KH, KW, pad;
  int P;                      // input channel planes (Cin / 8)
  int BW;                     // pixels per ring-slot row (multiple of 8)
  int R;                      // ring slots
  int ksteps;                 // MMAs (K = 16) per output row
  int strips;                 // ceil(W / 128)
  int rows_per_chunk, chunks_per_col, total_chunks;
  const bf16* w;              // [Cout][KH][KW][Cin] bf16
  const float* bias;
  int relu, out_fp32;
  void* out;
  long long out_pix_stride, out_img_stride, out_h_stride, out_w_stride, out_off;
  float* stats;               // [gridDim.x][2][Cout] or null
  // weight gradient only
  int PO;                     // output channel planes (Cout / 8)
  int RD;                     // dY ring slots
  float* dw;
  float* part;                // per-CTA partials [gridDim.x][welems], summed in CTA order (null: a single CTA adds into dw)
  long long welems;
  int oihw;
};

// descriptor halves: lo = start>>4 | (LBO>>4)<<16, hi = SBO>>4 | layout none (interleave)
__device__ __forceinline__ uint64_t halo_desc(uint32_t lo, uint32_t hi) { return ((uint64_t)hi << 32) | (uint64_t)lo; }
__host__ __device__ constexpr uint32_t halo_desc_hi(uint32_t sbo_bytes) { return (sbo_bytes >> 4) & 0x3FFFu; }

// ------------------------------------------------------------------------------------------------------------
// forward / data-gradient: y[n,y,x,:] = sum_taps W[:,kh,kw,:] . x[n, y+kh-pad, x+kw-pad, :]
// warp 8 = TMA producer; warps 0-7 = two consumer warpgroups, pixels 0..63 / 64..127 of the strip row (M = 64 each).
// CH = Cout / 16 (1 or 2).
// KS / CIN > 0 fix the filter size and input channels at compile time so that the per-MMA descriptor arithmetic folds
// to immediates.  KS = CIN = 0 is the generic (slow) fallback.
template <int CH, int KS, int CIN>
__global__ void __launch_bounds__(kGemmThreads, CH == 1 ? 3 : 2)
conv_halo_fwd_kernel(const __grid_constant__ CUtensorMap tmap_x, const HaloParams P) {
  constexpr int kCout = CH * 16;
  const int KH = KS > 0 ? KS : P.KH, KW = KH;
  const int Cin = CIN > 0 ? CIN : P.Cin;
  const int BW = KS > 1 ? 136 : P.BW;
  const int NP = Cin >> 3;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  const int plane_bytes = BW * 16;
  const int slot_bytes = NP * plane_bytes;
  const int wimg_bytes = P.ksteps * kCout * 32;
  uint8_t* wimg = smem;
  uint8_t* ring = smem + ((wimg_bytes + 127) & ~127);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(ring + (size_t)P.R * slot_bytes);
  uint64_t* empty_bar = full_bar + P.R;
  float* red = reinterpret_cast<float*>(empty_bar + P.R);         // [8 warps][2][kCout]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int KWP = (KW + 1) >> 1;                                  // tap pairs per filter row (Cin == 8 mode)
  const bool pair_mode = (Cin == 8);
  const int PQ = Cin >= 16 ? (Cin >> 4) : 1;

  // weight image: [kstep][Cout/8][2 K-chunks][8 rows][8 elems] = canonical no-swizzle K-major B operand
  for (int idx = threadIdx.x; idx < P.ksteps * kCout * 2; idx += blockDim.x) {
    const int j = idx & 1, co = (idx >> 1) % kCout, s = (idx >> 1) / kCout;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (pair_mode) {
      const int kh = s / KWP, kw = 2 * (s - kh * KWP) + j;
      if (kw < KW) v = *reinterpret_cast<const uint4*>(P.w + ((size_t)(co * KH + kh) * KW + kw) * 8);
    } else {
      const int tap = s / PQ, q = s - tap * PQ;
      v = *reinterpret_cast<const uint4*>(P.w + ((size_t)co * KH * KW + tap) * Cin + (2 * q + j) * 8);
    }
    *reinterpret_cast<uint4*>(wimg + (size_t)s * kCout * 32 + (co >> 3) * 256 + j * 128 + (co & 7) * 16) = v;
  }
  ptx::fence_proxy_async();

  if (warp == kConsumerWarps && lane == 0) {
    ptx::prefetch_tensormap(&tmap_x);
    for (int s = 0; s < P.R; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], kConsumerWarps); }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    if (ptx::elect_one()) {
      uint32_t slot = 0, par = 0;
      for (int c = blockIdx.x; c < P.total_chunks; c += gridDim.x) {
        const int col = c / P.chunks_per_col, cy = c - col * P.chunks_per_col;
        const int n = col / P.strips, xs = col - n * P.strips;
        const int y0 = cy * P.rows_per_chunk;
        const int rows = min(P.rows_per_chunk, P.H - y0);
        const int x0 = xs * 128 - P.pad;
        for (int i = 0; i < rows + KH - 1; ++i) {
          ptx::mbar_wait(&empty_bar[slot], par ^ 1u);
          ptx::mbar_expect_tx(&full_bar[slot], (uint32_t)slot_bytes);
          uint8_t* dst = ring + (size_t)slot * slot_bytes;
#pragma unroll
          for (int p = 0; p < NP; ++p)
            ptx::tma_load_4d(dst + p * plane_bytes, &tmap_x, &full_bar[slot], p * 8, x0, y0 - P.pad + i, n);
          if (++slot == (uint32_t)P.R) { slot = 0; par ^= 1u; }
        }
      }
    }
  } else {
    const uint32_t R = (uint32_t)P.R;
    const uint32_t slot_u = (uint32_t)slot_bytes >> 4;                         // descriptor address units (16 B)
    // A: this warpgroup's 64 pixels start 64 x 16 B into the row
    const uint32_t a_lo0 = ((ptx::smem_u32(ring) >> 4) + (uint32_t)((warp >> 2) * 64)) |
                           ((pair_mode ? 1u : ((uint32_t)plane_bytes >> 4)) << 16);
    const uint32_t b_lo0 = (ptx::smem_u32(wimg) >> 4) | (8u << 16);           // LBO 128 B
    constexpr uint32_t a_hi = halo_desc_hi(128), b_hi = halo_desc_hi(256);
    const int cq = 2 * (lane & 3);
    uint32_t slot0 = 0;                      // ring slot of the first input row of the current output row
    uint32_t rslot = 0, rpar = 0;            // next ring slot to wait for
    float s1[4 * CH], s2[4 * CH];            // statistics of this thread's channels (8j + cq, +1)
#pragma unroll
    for (int i = 0; i < 4 * CH; ++i) { s1[i] = 0.f; s2[i] = 0.f; }
    for (int c = blockIdx.x; c < P.total_chunks; c += gridDim.x) {
      const int col = c / P.chunks_per_col, cy = c - col * P.chunks_per_col;
      const int n = col / P.strips, xs = col - n * P.strips;
      const int y0 = cy * P.rows_per_chunk;
      const int rows = min(P.rows_per_chunk, P.H - y0);
      int xh[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) xh[h] = xs * 128 + (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
      for (int j = 0; j < rows; ++j) {
        const int need = j == 0 ? KH : 1;
        for (int t = 0; t < need; ++t) {
          ptx::mbar_wait(&full_bar[rslot], rpar);
          if (++rslot == R) { rslot = 0; rpar ^= 1u; }
        }
        float acc[kCout / 2];
        uint32_t sl = slot0;
        int s = 0;
        ptx::wgmma_fence();
#pragma unroll
        for (int kh = 0; kh < KH; ++kh) {
          const uint32_t row_lo = a_lo0 + sl * slot_u;
          if (pair_mode) {
#pragma unroll
            for (int pp = 0; pp < KWP; ++pp, ++s)
              ptx::wgmma_bf16<kCout, 0, 0>(acc, halo_desc(row_lo + (uint32_t)(2 * pp), a_hi),
                                            halo_desc(b_lo0 + (uint32_t)(s * kCout * 2), b_hi), s != 0 ? 1u : 0u);
          } else {
#pragma unroll
            for (int kw = 0; kw < KW; ++kw)
#pragma unroll
              for (int q = 0; q < PQ; ++q, ++s)
                ptx::wgmma_bf16<kCout, 0, 0>(acc, halo_desc(row_lo + (uint32_t)(2 * q) * ((uint32_t)plane_bytes >> 4) + (uint32_t)kw, a_hi),
                                              halo_desc(b_lo0 + (uint32_t)(s * kCout * 2), b_hi), s != 0 ? 1u : 0u);
          }
          if (++sl == R) sl = 0;
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        ptx::fence_regs(acc);
        // the oldest row of the window is no longer needed
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&empty_bar[slot0]);
        if (++slot0 == R) slot0 = 0;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (xh[h] >= P.W) continue;
          const long long pix = (long long)n * P.out_img_stride + (long long)(y0 + j) * P.out_h_stride +
                                (long long)xh[h] * P.out_w_stride + P.out_off;
#pragma unroll
          for (int jb = 0; jb < 2 * CH; ++jb) {
            const int c0 = 8 * jb + cq;
            float v0 = acc[4 * jb + 2 * h], v1 = acc[4 * jb + 2 * h + 1];
            if (P.stats) {
              s1[2 * jb] += v0; s1[2 * jb + 1] += v1;
              s2[2 * jb] += v0 * v0; s2[2 * jb + 1] += v1 * v1;
            }
            if (P.bias) { v0 += __ldg(P.bias + c0); v1 += __ldg(P.bias + c0 + 1); }
            if (P.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            if (P.out_fp32)
              *reinterpret_cast<float2*>(reinterpret_cast<float*>(P.out) + pix * P.out_pix_stride + c0) = make_float2(v0, v1);
            else
              *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<bf16*>(P.out) + pix * P.out_pix_stride + c0) =
                  __floats2bfloat162_rn(v0, v1);
          }
        }
      }
      for (int t = 0; t < KH - 1; ++t) {                         // rows only the finished chunk used
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&empty_bar[slot0]);
        if (++slot0 == R) slot0 = 0;
      }
    }
    if (P.stats) {          // one partial-statistics row per CTA (BatchNorm batch statistics, fp32 partials)
#pragma unroll
      for (int i = 0; i < 4 * CH; ++i) {
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
          s1[i] += __shfl_xor_sync(0xffffffffu, s1[i], o);
          s2[i] += __shfl_xor_sync(0xffffffffu, s2[i], o);
        }
      }
      if (lane < 4) {
#pragma unroll
        for (int jb = 0; jb < 2 * CH; ++jb)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            red[(warp * 2 + 0) * kCout + 8 * jb + cq + e] = s1[2 * jb + e];
            red[(warp * 2 + 1) * kCout + 8 * jb + cq + e] = s2[2 * jb + e];
          }
      }
      ptx::named_bar_sync(1, 32 * kConsumerWarps);
      const int m = threadIdx.x;
      if (m < 2 * kCout) {
        const int which = m / kCout, ci = m - which * kCout;
        float a = 0.f;
#pragma unroll
        for (int w = 0; w < kConsumerWarps; ++w) a += red[(w * 2 + which) * kCout + ci];
        P.stats[(size_t)blockIdx.x * 2 * kCout + which * kCout + ci] = a;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// weight gradient: dW[co][kh][kw][ci] += sum_{n,y,x} dY[n,y,x,co] * X[n, y+kh-pad, x+kw-pad, ci]
// One input row X[i] meets the KH gradient rows dY[i-KH+1 .. i] that use it: those rows sit in CONSECUTIVE ring slots
// (the first KH-1 slots are mirrored behind the ring, so a window never wraps).  Per input row and plane p:
//   D_b[m = (kw shift, ci)][n = co] += X_row^T . dY_row(j),  K = 16 pixels,  for every dY row j of the window,
// where accumulator b = KH-1-kh holds kh = i - j.  At the first/last rows of a chunk the window is clipped to the
// chunk's own rows, so every (row, kh) pair is counted once.  Consumer warpgroup p owns input-channel plane p
// (M = 8 shifts x 8 channels = 64; KW <= 7) and keeps its KH accumulators in registers for the CTA's lifetime.
template <int KS, int CIN, int CO>
__global__ void __launch_bounds__(CIN / 8 * 128 + 32, 1)
conv_halo_wgrad_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_dy,
                       const HaloParams P) {
  constexpr int KH = KS;
  constexpr int NP = CIN >> 3;
  constexpr int kWarps = 4 * NP;                            // consumer warps; warp kWarps = TMA producer
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  constexpr int plane_bytes = 144 * 16;                     // P.BW == 144 always for the weight gradient
  constexpr int slot_bytes = NP * plane_bytes;
  constexpr int dy_plane_bytes = 128 * 16;
  constexpr int dy_slot_bytes = (CO / 8) * dy_plane_bytes;
  uint8_t* ring = smem;
  uint8_t* dyring = ring + (size_t)P.R * slot_bytes;                        // RD slots + KH-1 mirror slots
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(dyring + (size_t)(P.RD + KH - 1) * dy_slot_bytes);
  uint64_t* empty_bar = full_bar + P.R;
  uint64_t* dfull_bar = empty_bar + P.R;
  uint64_t* dempty_bar = dfull_bar + P.RD;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (warp == kWarps && lane == 0) {
    ptx::prefetch_tensormap(&tmap_x); ptx::prefetch_tensormap(&tmap_dy);
    for (int s = 0; s < P.R; ++s) { ptx::mbar_init(&full_bar[s], 1); ptx::mbar_init(&empty_bar[s], kWarps); }
    for (int s = 0; s < P.RD; ++s) { ptx::mbar_init(&dfull_bar[s], 1); ptx::mbar_init(&dempty_bar[s], kWarps); }
    ptx::fence_barrier_init();
  }
  __syncthreads();

  if (warp == kWarps) {
    if (ptx::elect_one()) {
      uint32_t slot = 0, par = 0, ds = 0, dpar = 0;
      for (int c = blockIdx.x; c < P.total_chunks; c += gridDim.x) {
        const int col = c / P.chunks_per_col, cy = c - col * P.chunks_per_col;
        const int n = col / P.strips, xs = col - n * P.strips;
        const int y0 = cy * P.rows_per_chunk;
        const int rows = min(P.rows_per_chunk, P.H - y0);
        const int x0 = xs * 128;
        for (int i = 0; i < rows + KH - 1; ++i) {
          if (i < rows) {                                   // dY row i is first needed together with input row i
            ptx::mbar_wait(&dempty_bar[ds], dpar ^ 1u);
            const bool mirror = ds < (uint32_t)(KH - 1);
            ptx::mbar_expect_tx(&dfull_bar[ds], (uint32_t)dy_slot_bytes * (mirror ? 2u : 1u));
            uint8_t* dd = dyring + (size_t)ds * dy_slot_bytes;
            for (int p = 0; p < CO / 8; ++p) {
              ptx::tma_load_4d(dd + p * dy_plane_bytes, &tmap_dy, &dfull_bar[ds], p * 8, x0, y0 + i, n);
              if (mirror)
                ptx::tma_load_4d(dd + (size_t)P.RD * dy_slot_bytes + p * dy_plane_bytes, &tmap_dy, &dfull_bar[ds], p * 8, x0,
                                 y0 + i, n);
            }
            if (++ds == (uint32_t)P.RD) { ds = 0; dpar ^= 1u; }
          }
          ptx::mbar_wait(&empty_bar[slot], par ^ 1u);
          ptx::mbar_expect_tx(&full_bar[slot], (uint32_t)slot_bytes);
          uint8_t* dst = ring + (size_t)slot * slot_bytes;
#pragma unroll
          for (int p = 0; p < NP; ++p)
            ptx::tma_load_4d(dst + p * plane_bytes, &tmap_x, &full_bar[slot], p * 8, x0 - P.pad, y0 - P.pad + i, n);
          if (++slot == (uint32_t)P.R) { slot = 0; par ^= 1u; }
        }
      }
    }
  } else {
    const int p = warp >> 2;                 // input-channel plane of this warpgroup
    const uint32_t R = (uint32_t)P.R, RD = (uint32_t)P.RD;
    constexpr uint32_t slot_u = (uint32_t)slot_bytes >> 4, dy_slot_u = (uint32_t)dy_slot_bytes >> 4;
    // A: MN-major, MN chunk (pixel shift) stride 16 B ("SBO"), K group (8 px) stride 128 B ("LBO")
    const uint32_t a_lo0 = ((ptx::smem_u32(ring) >> 4) + (uint32_t)(p * (plane_bytes >> 4))) | (8u << 16);
    // B: MN-major, MN chunk (8 output channels) stride = dY plane
    const uint32_t b_lo0 = (ptx::smem_u32(dyring) >> 4) | (8u << 16);
    constexpr uint32_t a_hi = halo_desc_hi(16), b_hi = halo_desc_hi(dy_plane_bytes);
    float acc[KH][CO / 2];
#pragma unroll
    for (int b = 0; b < KH; ++b)
#pragma unroll
      for (int i = 0; i < CO / 2; ++i) acc[b][i] = 0.f;
    uint32_t xslot = 0, xpar = 0;            // input-row FIFO
    uint32_t dwait = 0, dwpar = 0;           // next dY slot to wait for
    uint32_t dlo = 0;                        // ring slot of the oldest dY row still in use
    for (int c = blockIdx.x; c < P.total_chunks; c += gridDim.x) {
      const int cy = c % P.chunks_per_col;
      const int y0 = cy * P.rows_per_chunk;
      const int rows = min(P.rows_per_chunk, P.H - y0);
      for (int i = 0; i < rows + KH - 1; ++i) {
        if (i < rows) {
          ptx::mbar_wait(&dfull_bar[dwait], dwpar);
          if (++dwait == RD) { dwait = 0; dwpar ^= 1u; }
        }
        ptx::mbar_wait(&full_bar[xslot], xpar);
        const int jlo = max(0, i - KH + 1), jhi = min(rows - 1, i);
        const int nvalid = jhi - jlo + 1;
        const int blo = KH - 1 - i + jlo;                  // accumulator of dY row jlo (kh = i - jlo)
        const uint32_t dy_lo = b_lo0 + dlo * dy_slot_u;    // dlo is the slot of row jlo (rows below jlo are released)
        const uint32_t row_lo = a_lo0 + xslot * slot_u;
        ptx::wgmma_fence();
#pragma unroll
        for (int b = 0; b < KH; ++b) {
          const int t = b - blo;                           // window row of accumulator b
          if (t < 0 || t >= nvalid) continue;
#pragma unroll
          for (int k = 0; k < 8; ++k)
            ptx::wgmma_bf16<CO, 1, 1>(acc[b], halo_desc(row_lo + (uint32_t)(k * 16), a_hi),
                                       halo_desc(dy_lo + (uint32_t)t * dy_slot_u + (uint32_t)(k * 16), b_hi), 1u);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
#pragma unroll
        for (int b = 0; b < KH; ++b) ptx::fence_regs(acc[b]);
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&empty_bar[xslot]);
        if (++xslot == R) { xslot = 0; xpar ^= 1u; }
        if (i >= KH - 1) {                                 // dY row i-KH+1 has met its last input row
          if (lane == 0) ptx::mbar_arrive(&dempty_bar[dlo]);
          if (++dlo == RD) dlo = 0;
        }
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = (warp & 3) * 16 + (lane >> 2) + 8 * h;
      const int kw = m >> 3, ci = p * 8 + (m & 7);
      if (kw >= P.KW) continue;
#pragma unroll
      for (int b = 0; b < KH; ++b) {
        const int kh = KH - 1 - b;
#pragma unroll
        for (int jb = 0; jb < CO / 8; ++jb)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int co = 8 * jb + 2 * (lane & 3) + e;
            const size_t off = P.oihw ? (((size_t)co * P.Cin + ci) * P.KH + kh) * P.KW + kw
                                      : (((size_t)co * P.KH + kh) * P.KW + kw) * P.Cin + ci;
            if (P.part) P.part[(size_t)blockIdx.x * P.welems + off] = acc[b][4 * jb + 2 * h + e];
            else P.dw[off] += acc[b][4 * jb + 2 * h + e];
          }
      }
    }
  }
}

// ---- host side ---------------------------------------------------------------------------------------------
// pure function of the descriptor (c3d_conv2d_tiles must agree with c3d_conv2d_fwd)
static bool halo_fwd_eligible(const c3d_conv_desc* d) {
  if (d->stride != 1 || d->KH != d->KW || !(d->KH & 1) || 2 * d->pad != d->KH - 1) return false;
  if (d->out_h > 0 || d->out_w > 0 || d->add_mode != 0) return false;
  if (!(d->Cin == 8 || d->Cin == 16 || d->Cin == 32)) return false;
  if (!(d->Cout == 16 || d->Cout == 32)) return false;
  if ((d->W < 128 && d->Cin != 8) || d->KH > 7) return false;   // NHWC8 input exists only for this kernel
  return true;
}
static bool halo_wgrad_eligible(const c3d_conv_desc* d) {
  if (d->stride != 1 || d->KH != d->KW || !(d->KH & 1) || 2 * d->pad != d->KH - 1) return false;
  if (!(d->Cin == 8 || d->Cin == 16 || d->Cin == 32)) return false;
  if (!(d->Cout == 16 || d->Cout == 32)) return false;
  if (d->y_pix_stride != 0 && d->y_pix_stride != d->Cout) return false;
  if (d->W < 128 && d->Cin != 8) return false;
  return (d->KH == 7 && d->Cin == 8) || (d->KH == 3 && d->Cin >= 16);     // the compiled instances
}
// ring depth: the TMA rows are only 2-4 KB, so hiding ~1.5 us of L2/HBM latency at ~40 B/ns per SM needs tens of rows in flight
static int halo_ring_rows(int window, int slot_bytes, int budget) {
  int pf = budget / slot_bytes - window;
  if (pf > 48) pf = 48;
  if (pf < 2) pf = 2;
  return window + pf;
}
static int halo_fwd_ctas_per_sm(int Cout) { return Cout == 16 ? 3 : 2; }     // = __launch_bounds__ of the instances
static void halo_chunking(const c3d_conv_desc* d, HaloParams* P, int ctas_per_sm, int* grid) {
  P->strips = (d->W + 127) / 128;
  P->rows_per_chunk = d->H < 32 ? d->H : 32;
  P->chunks_per_col = (d->H + P->rows_per_chunk - 1) / P->rows_per_chunk;
  P->total_chunks = d->N * P->strips * P->chunks_per_col;
  const int slots = kNumSMs * ctas_per_sm;
  *grid = P->total_chunks < slots ? P->total_chunks : slots;
}
static int halo_fwd_grid(const c3d_conv_desc* d) {
  HaloParams P; int grid;
  halo_chunking(d, &P, halo_fwd_ctas_per_sm(d->Cout), &grid);
  return grid;
}
static CUresult halo_tensormap(PFN_encodeTiled enc, CUtensorMap* m, const void* base, int C, int W, int H, int N, int boxw) {
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)C * 2 * W, (cuuint64_t)C * 2 * W * H};
  cuuint32_t box[4] = {8, (cuuint32_t)boxw, 1, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

template <int CH, int KS, int CIN>
static int32_t launch_halo_fwd_inst(const CUtensorMap& mx, const HaloParams& P, int grid, size_t smem, cudaStream_t st) {
  auto kern = conv_halo_fwd_kernel<CH, KS, CIN>;
  static size_t cur = 0;
  if (smem > cur) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return set_error(C3D_ECUDA, "halo smem attr: %s", cudaGetErrorString(e));
    cur = smem;
  }
  kern<<<grid, kGemmThreads, smem, st>>>(mx, P);
  return check_launch("conv_halo_fwd_kernel");
}

static int32_t launch_halo_fwd(const c3d_conv_desc* d, const void* x, const void* w, const float* bias, void* y,
                               float* stats, cudaStream_t st) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error(C3D_ECUDA, "cuTensorMapEncodeTiled unavailable");
  HaloParams P;
  memset(&P, 0, sizeof(P));
  int grid;
  const int ctas = halo_fwd_ctas_per_sm(d->Cout);
  halo_chunking(d, &P, ctas, &grid);
  P.N = d->N; P.H = d->H; P.W = d->W; P.Cin = d->Cin; P.Cout = d->Cout; P.KH = d->KH; P.KW = d->KW; P.pad = d->pad;
  P.P = d->Cin / 8;
  P.BW = (128 + d->KW - 1 + 7) / 8 * 8;
  P.R = halo_ring_rows(d->KH, P.P * P.BW * 16, ctas == 3 ? 48 * 1024 : 64 * 1024);
  P.ksteps = d->Cin == 8 ? d->KH * ((d->KW + 1) / 2) : d->KH * d->KW * (d->Cin / 16);
  P.w = static_cast<const bf16*>(w); P.bias = bias; P.relu = d->relu; P.out_fp32 = d->out_fp32; P.out = y;
  P.out_pix_stride = d->y_pix_stride ? d->y_pix_stride : d->Cout;
  if (d->y_img_stride) {
    P.out_img_stride = d->y_img_stride; P.out_h_stride = d->y_h_stride; P.out_w_stride = d->y_w_stride; P.out_off = d->y_offset;
  } else {
    P.out_img_stride = (long long)d->H * d->W; P.out_h_stride = d->W; P.out_w_stride = 1; P.out_off = 0;
  }
  P.stats = stats;
  CUtensorMap mx;
  CUresult r = halo_tensormap(enc, &mx, x, d->Cin, d->W, d->H, d->N, P.BW);
  if (r != CUDA_SUCCESS) return set_error(C3D_ECUDA, "encode halo x tensormap failed: %d", (int)r);
  const int wimg = (P.ksteps * d->Cout * 32 + 127) & ~127;
  const size_t smem = 128 + (size_t)wimg + (size_t)P.R * P.P * P.BW * 16 + (size_t)(2 * P.R) * 8 +
                      kConsumerWarps * 2 * d->Cout * sizeof(float) + 64;
  if (smem > 200 * 1024) return set_error(C3D_EINVAL, "halo conv: smem %zu too large", smem);
#define C3D_HALO_F(ch, ks, cin) \
  if (d->Cout == ch * 16 && d->KH == ks && d->Cin == cin) return launch_halo_fwd_inst<ch, ks, cin>(mx, P, grid, smem, st);
  C3D_HALO_F(1, 7, 8)
  C3D_HALO_F(1, 3, 16)
  C3D_HALO_F(1, 3, 32)
  C3D_HALO_F(2, 7, 8)
  C3D_HALO_F(2, 3, 16)
  C3D_HALO_F(2, 3, 32)
#undef C3D_HALO_F
  if (d->Cout == 16) return launch_halo_fwd_inst<1, 0, 0>(mx, P, grid, smem, st);
  return launch_halo_fwd_inst<2, 0, 0>(mx, P, grid, smem, st);
}

template <int KS, int CIN, int CO>
static int32_t launch_halo_wgrad_inst(const CUtensorMap& mx, const CUtensorMap& mdy, const HaloParams& P, int grid, size_t smem,
                                      cudaStream_t st) {
  auto kern = conv_halo_wgrad_kernel<KS, CIN, CO>;
  static size_t cur = 0;
  if (smem > cur) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return set_error(C3D_ECUDA, "halo wgrad smem attr: %s", cudaGetErrorString(e));
    cur = smem;
  }
  return with_ordered_partials(grid, P.welems, P.dw, st, [&](float* part) -> int32_t {
    HaloParams Q = P;
    Q.part = part;
    kern<<<grid, CIN / 8 * 128 + 32, smem, st>>>(mx, mdy, Q);
    return check_launch("conv_halo_wgrad_kernel");
  });
}

static int32_t launch_halo_wgrad(const c3d_conv_desc* d, const void* x, const void* dy, float* dw, int oihw,
                                 cudaStream_t st) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) return set_error(C3D_ECUDA, "cuTensorMapEncodeTiled unavailable");
  HaloParams P;
  memset(&P, 0, sizeof(P));
  P.N = d->N; P.H = d->H; P.W = d->W; P.Cin = d->Cin; P.Cout = d->Cout; P.KH = d->KH; P.KW = d->KW; P.pad = d->pad;
  P.P = d->Cin / 8; P.PO = d->Cout / 8;
  P.BW = 144;
  P.R = halo_ring_rows(0, P.P * P.BW * 16, 16 * 1024);             // input rows are a plain FIFO here
  P.RD = halo_ring_rows(d->KH, P.PO * 128 * 16, 0);                // window of KH rows + 2 in flight
  P.dw = dw; P.oihw = oihw;
  P.welems = (long long)d->Cout * d->KH * d->KW * d->Cin;
  const size_t smem = 128 + (size_t)P.R * P.P * P.BW * 16 + (size_t)(P.RD + d->KH - 1) * P.PO * 128 * 16 +
                      (size_t)(2 * P.R + 2 * P.RD) * 8 + 64;
  if (smem > 200 * 1024) return set_error(C3D_EINVAL, "halo wgrad: smem %zu too large", smem);
  int ctas = (int)((227 * 1024) / (smem + 1024));                  // co-resident CTAs by shared memory
  if (ctas > 4) ctas = 4;
  if (ctas < 1) ctas = 1;
  int grid;
  halo_chunking(d, &P, ctas, &grid);
  CUtensorMap mx, mdy;
  CUresult r = halo_tensormap(enc, &mx, x, d->Cin, d->W, d->H, d->N, P.BW);
  if (r != CUDA_SUCCESS) return set_error(C3D_ECUDA, "encode halo x tensormap failed: %d", (int)r);
  r = halo_tensormap(enc, &mdy, dy, d->Cout, d->W, d->H, d->N, 128);
  if (r != CUDA_SUCCESS) return set_error(C3D_ECUDA, "encode halo dy tensormap failed: %d", (int)r);
#define C3D_HALO_W(ks, cin, co) \
  if (d->KH == ks && d->Cin == cin && d->Cout == co) return launch_halo_wgrad_inst<ks, cin, co>(mx, mdy, P, grid, smem, st);
  C3D_HALO_W(7, 8, 16)
  C3D_HALO_W(7, 8, 32)
  C3D_HALO_W(3, 16, 16)
  C3D_HALO_W(3, 16, 32)
  C3D_HALO_W(3, 32, 16)
  C3D_HALO_W(3, 32, 32)
#undef C3D_HALO_W
  return set_error(C3D_EINVAL, "halo wgrad: no kernel for %dx%d, Cin %d, Cout %d", d->KH, d->KW, d->Cin, d->Cout);
}

}  // namespace c3d
