// nhwc_ops.cu — HBM-bound NHWC bf16 kernels around the tensor-core convolutions (sm_90a):
// train-mode BatchNorm (finalize / apply+residual+ReLU / backward reduce+apply), 2x2 max-pool,
// image normalisation + channel padding, fused SGD-momentum with finite check.
//
// Replaces the ATen/cuDNN calls behind nn.BatchNorm2d + ReLU + residual add
// (cubercnn/modeling/backbone/dla.py:17,58-66,168-172), nn.MaxPool2d (dla.py:209),
// GeneralizedRCNN.preprocess_image (called at rcnn3d.py:46,87) and the optimizer step +
// per-parameter finite check (tools/train_net.py:226-252, cubercnn/solver/build.py:47-56).
// All kernels: 16-byte vector loads (8 bf16 channels per thread), channel-innermost coalescing,
// grid = multiple of the SM count with grid-stride loops; no tensor cores (byte work).
#include <cuda_bf16.h>
#include "c3d_common.cuh"

namespace c3d {
using bf16 = __nv_bfloat16;

struct V8 { float v[8]; };
__device__ __forceinline__ V8 ld8(const bf16* p) {
  uint4 u = *reinterpret_cast<const uint4*>(p);
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
  V8 r;
#pragma unroll
  for (int i = 0; i < 4; ++i) { float2 f = __bfloat1622float2(h[i]); r.v[2 * i] = f.x; r.v[2 * i + 1] = f.y; }
  return r;
}
__device__ __forceinline__ void st8(bf16* p, const V8& a) {
  uint4 u;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(a.v[2 * i], a.v[2 * i + 1]);
  *reinterpret_cast<uint4*>(p) = u;
}
static inline int grid_for(long long work_items, int threads) {
  long long b = (work_items + threads - 1) / threads;
  long long cap = (long long)kNumSMs * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

// ---- BatchNorm forward ------------------------------------------------------------------------
// Column sums of a [rows][cols] fp32 matrix in fixed order (deterministic): stage 1 = slabs of rows per
// block (64 columns x 4 row lanes), doubles out; the LAST block then finishes over the <= kSlabs slabs
// (colsum_finalize_kernel below).
constexpr int kSlabs = 64;
// partial: [rows][2][C] per-tile (sum, sumsq) from the conv epilogue -> slab sums -> statistics.
// Second stage of the column sums: <= kSlabs rows of doubles.  A block is 32 channels x 8 row lanes; every lane sums
// each 8th slab (16 loads instead of a 128-long serial chain), then the 8 partials are combined through shared memory.
// Returns the two sums (offsets off0 / off1 inside a slab row; pass off1 < 0 for a single sum) to row-lane 0.
__device__ __forceinline__ void slab_sums(const double* slab, int slabs, size_t row_stride, int off0, int off1,
                                          int c, bool active, double* s_out, double* t_out) {
  __shared__ double sh[2][8][32];
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  double s = 0.0, t = 0.0;
  if (active) {
    // L2 loads (the slabs were written by other blocks), all of a lane's <= kSlabs / 8 rows in flight at once: this runs in
    // the ONE last block of a column group, so its load latency is the tail of every BatchNorm layer
    double vs[kSlabs / 8], vt[kSlabs / 8];
#pragma unroll
    for (int i = 0; i < kSlabs / 8; ++i) {
      const int r = ry + 8 * i;
      const bool in = r < slabs;
      vs[i] = in ? __ldcg(slab + (size_t)r * row_stride + off0 + c) : 0.0;
      vt[i] = (in && off1 >= 0) ? __ldcg(slab + (size_t)r * row_stride + off1 + c) : 0.0;
    }
#pragma unroll
    for (int i = 0; i < kSlabs / 8; ++i) { s += vs[i]; t += vt[i]; }
  }
  sh[0][ry][cx] = s; sh[1][ry][cx] = t;
  __syncthreads();
  if (ry == 0) {
#pragma unroll
    for (int k = 1; k < 8; ++k) { s += sh[0][k][cx]; t += sh[1][k][cx]; }
  }
  *s_out = s; *t_out = t;
}


// out = [relu]( (y - mean) * rstd * gamma + beta [+ residual] ), P pixels x C channels
// thread layout of the streaming BN kernels: tx = channel vector (8 channels, fixed for the thread's lifetime so the
// per-channel constants live in registers), ty = pixel row lane; pixels are strided by gridDim * rows_per_block.  No
// integer division and no parameter loads inside the loop: these kernels must sustain ~1.4 16-byte vectors per clock
// per SM to reach HBM speed, so the loop body is kept to the loads, 8 FMAs and the store.
__global__ void __launch_bounds__(256)
bn_apply_kernel(const bf16* __restrict__ y, const float* __restrict__ mean, const float* __restrict__ rstd,
                const float* __restrict__ gamma, const float* __restrict__ beta, const bf16* __restrict__ residual, int relu,
                bf16* __restrict__ out, long long P, int C) {
  const int cv = C >> 3;
  const int tx = threadIdx.x % cv, ty = threadIdx.x / cv;
  const int rows_per_block = blockDim.x / cv;
  if (ty >= rows_per_block) return;
  const int c = tx << 3;
  float m[8], sc[8], bt[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) { m[k] = mean[c + k]; sc[k] = rstd[c + k] * gamma[c + k]; bt[k] = beta[c + k]; }
  const long long step = (long long)gridDim.x * rows_per_block;
  for (long long p = (long long)blockIdx.x * rows_per_block + ty; p < P; p += step) {
    V8 a = ld8(y + p * C + c);
    V8 o;
    if (residual) {
      V8 r = ld8(residual + p * C + c);
#pragma unroll
      for (int k = 0; k < 8; ++k) o.v[k] = __fmaf_rn(a.v[k] - m[k], sc[k], bt[k]) + r.v[k];
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) o.v[k] = __fmaf_rn(a.v[k] - m[k], sc[k], bt[k]);
    }
    if (relu) {
#pragma unroll
      for (int k = 0; k < 8; ++k) o.v[k] = fmaxf(o.v[k], 0.f);
    }
    st8(out + p * C + c, o);
  }
}

// ---- BatchNorm backward -----------------------------------------------------------------------
// dz = dout * (out > 0 if relu);  partial[block][0][c] = sum dz, partial[block][1][c] = sum dz * y  (the finalisation
// turns the second sum into sum dz * xhat = rstd * (sum dz*y - mean * sum dz) in fp64).
// Register diet (ptxas): with mean / rstd / scale / shift / coefficients held per thread these kernels
// needed 86-90 registers => 2 CTAs of 256 threads per SM => too few loads in flight for HBM (they ran at ~60 % of the copy
// bandwidth and got SLOWER when the ReLU-mask recomputation added 16 more).  Now the mask constants live in shared memory
// (3 x C floats, read as two LDS.128 per array per pixel) and the arithmetic needs no per-channel constant at all (reduce) or
// three fused ones (apply): <= 64 registers => 4 CTAs per SM.
constexpr int kBnMaxC = 2048;
__device__ __forceinline__ void bn_mask_consts(float* cm, const float* __restrict__ mean, const float* __restrict__ rstd,
                                               const float* __restrict__ gamma, const float* __restrict__ beta, int C) {
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    cm[i] = mean[i]; cm[kBnMaxC + i] = rstd[i] * gamma[i]; cm[2 * kBnMaxC + i] = beta[i];
  }
}
// zero d where the forward's fma(y - mean, rstd*gamma, beta) was not positive (bit-identical recomputation)
__device__ __forceinline__ void bn_remask(V8& d, const V8& yy, const float* cm, int c) {
  const float4 m0 = *reinterpret_cast<const float4*>(cm + c), m1 = *reinterpret_cast<const float4*>(cm + c + 4);
  const float4 s0 = *reinterpret_cast<const float4*>(cm + kBnMaxC + c), s1 = *reinterpret_cast<const float4*>(cm + kBnMaxC + c + 4);
  const float4 b0 = *reinterpret_cast<const float4*>(cm + 2 * kBnMaxC + c), b1 = *reinterpret_cast<const float4*>(cm + 2 * kBnMaxC + c + 4);
  const float m[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
  const float sc[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
  const float bt[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
  for (int k = 0; k < 8; ++k) if (!(__fmaf_rn(yy.v[k] - m[k], sc[k], bt[k]) > 0.f)) d.v[k] = 0.f;
}

template <int THREADS>
__global__ void __launch_bounds__(THREADS, 4)
bn_bwd_reduce_kernel(const bf16* __restrict__ dout, const bf16* __restrict__ out, const bf16* __restrict__ y,
                     const float* __restrict__ mean, const float* __restrict__ rstd, int relu, float* __restrict__ partial,
                     long long P, int C, long long dout_stride, const float* __restrict__ gamma,
                     const float* __restrict__ beta) {
  // `out == nullptr` with relu: the layer has no residual, so its ReLU mask is a function of y alone
  __shared__ float cm[3 * kBnMaxC];
  __shared__ float sm[2][THREADS][8 + 1];
  const bool remask = relu && out == nullptr;
  if (remask) bn_mask_consts(cm, mean, rstd, gamma, beta, C);
  __syncthreads();
  const int cv = C >> 3;
  const int tx = threadIdx.x % cv, ty = threadIdx.x / cv;
  const int rows_per_block = THREADS / cv;
  const int c = tx << 3;
  float s[8], t[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) { s[k] = 0.f; t[k] = 0.f; }
  const bf16* yc = y + c;          // hoisted: the loop then fits the 64-register bound of 4 CTAs per SM without spilling
  if (ty < rows_per_block) {
    for (long long p = (long long)blockIdx.x * rows_per_block + ty; p < P; p += (long long)gridDim.x * rows_per_block) {
      V8 d = ld8(dout + p * dout_stride + c);
      const V8 yy = ld8(yc + p * C);
      if (remask) bn_remask(d, yy, cm, c);
      else if (relu) {
        const V8 o = ld8(out + p * C + c);
#pragma unroll
        for (int k = 0; k < 8; ++k) if (!(o.v[k] > 0.f)) d.v[k] = 0.f;
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) { s[k] += d.v[k]; t[k] = __fmaf_rn(d.v[k], yy.v[k], t[k]); }
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) { sm[0][threadIdx.x][k] = s[k]; sm[1][threadIdx.x][k] = t[k]; }
  __syncthreads();
  // fixed-order reduction over ty for each channel (deterministic)
  for (int idx = threadIdx.x; idx < 2 * C; idx += THREADS) {
    const int which = idx / C, ch = idx - which * C;
    const int vx = ch >> 3, k = ch & 7;
    float acc = 0.f;
    for (int r = 0; r < rows_per_block; ++r) acc += sm[which][r * cv + vx][k];
    partial[((size_t)blockIdx.x * 2 + which) * C + ch] = acc;
  }
}

// dy = A*dz + B*y + K with A = gamma*rstd, B = -A*rstd*mean(dz*xhat), K = -A*mean(dz) - B*mean  (== gamma*rstd*(dz - mean(dz)
// - xhat*mean(dz*xhat)), coefficients from the finalisation);  optionally dres = dz
__global__ void __launch_bounds__(256, 4)
bn_bwd_apply_kernel(const bf16* __restrict__ dout, const bf16* __restrict__ out, const bf16* __restrict__ y,
                    const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ coef, int relu,
                    bf16* __restrict__ dy, bf16* __restrict__ dres, long long P, int C, long long dout_stride,
                    long long dres_stride, const float* __restrict__ gamma,
                    const float* __restrict__ beta, int dres_acc) {
  __shared__ float cm[3 * kBnMaxC];
  const bool remask = relu && out == nullptr;
  if (remask) bn_mask_consts(cm, mean, rstd, gamma, beta, C);
  __syncthreads();
  const int cv = C >> 3;
  const int tx = threadIdx.x % cv, ty = threadIdx.x / cv;
  const int rows_per_block = blockDim.x / cv;
  if (ty >= rows_per_block) return;
  const int c = tx << 3;
  float cA[8], cB[8], cK[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) { cA[k] = coef[c + k]; cB[k] = coef[C + c + k]; cK[k] = coef[2 * C + c + k]; }
  const long long step = (long long)gridDim.x * rows_per_block;
  for (long long p = (long long)blockIdx.x * rows_per_block + ty; p < P; p += step) {
    V8 d = ld8(dout + p * dout_stride + c);
    const V8 yy = ld8(y + p * C + c);
    if (remask) bn_remask(d, yy, cm, c);
    else if (relu) {
      const V8 o = ld8(out + p * C + c);
#pragma unroll
      for (int k = 0; k < 8; ++k) if (!(o.v[k] > 0.f)) d.v[k] = 0.f;
    }
    V8 g;
#pragma unroll
    for (int k = 0; k < 8; ++k) g.v[k] = __fmaf_rn(cA[k], d.v[k], __fmaf_rn(cB[k], yy.v[k], cK[k]));
    st8(dy + p * C + c, g);
    if (dres) {
      if (dres_acc) {                  // the residual branch's gradient already holds other contributions: add in fp32
        const V8 r = ld8(dres + p * dres_stride + c);
#pragma unroll
        for (int k = 0; k < 8; ++k) d.v[k] += r.v[k];
      }
      st8(dres + p * dres_stride + c, d);
    }
  }
}

// ---- column sums + finalisation in ONE launch ------------------------------------------------------------------------
// The three consumers of the slab sums (BatchNorm statistics, BatchNorm backward coefficients, bias gradient) used to be a
// second launch of (C/32) tiny blocks behind colsum_stage1: ~100 extra launches of 5-10 us per step (1.2 ms with the
// stage-1 kernels).  Here the LAST stage-1 block to finish (ticket counter zeroed by a 4-byte memset node in
// front of the launch) runs the finalisation for all channels, in the same fixed order as before => same bits.
struct FinArgs {
  int mode;                  // 0 BatchNorm statistics, 1 BatchNorm backward coefficients, 2 bias gradient
  int C;
  double count;
  float eps, momentum;
  float* running_mean; float* running_var; float* mean_out; float* rstd_out;      // mode 0
  const float* gamma; const float* rstd; const float* mean; float* coef; float* dgamma; float* dbeta; int frozen;   // mode 1
  float* dbias;                                                                    // mode 2
};

__global__ void colsum_finalize_kernel(const float* __restrict__ m, int rows, int cols, int rows_per_slab,
                                       double* __restrict__ out /*[gridDim.y][cols]*/, unsigned int* __restrict__ ticket,
                                       const FinArgs A) {
  // a block owns 64 columns x one slab of rows.  Modes 0/1 (two sums per channel): the 64 columns are channels
  // [32 bx, 32 bx + 32) of BOTH halves, so the last block of a column group can finalise its 32 channels on its own —
  // all column groups finish in parallel (a single last block for all channels serialised ~30 us per layer).
  const int C = A.C, j = threadIdx.x & 63, lane = threadIdx.x >> 6;      // lane = 0..3 row lane
  const int ch = A.mode == 2 ? blockIdx.x * 64 + j : blockIdx.x * 32 + (j & 31);
  const int col = A.mode == 2 ? ch : (j >> 5) * C + ch;
  const bool ok = ch < C;
  const int r0 = blockIdx.y * rows_per_slab;
  const int r1 = min(rows, r0 + rows_per_slab);
  double acc = 0.0;
  if (ok)
    for (int r = r0 + lane; r < r1; r += 4) acc += (double)m[(size_t)r * cols + col];
  __shared__ double sm[4][64];
  __shared__ int s_last;
  sm[lane][j] = acc;
  __syncthreads();
  if (lane == 0 && ok) out[(size_t)blockIdx.y * cols + col] = ((sm[0][j] + sm[1][j]) + sm[2][j]) + sm[3][j];
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(ticket + blockIdx.x, 1u) == gridDim.y - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const int slabs = gridDim.y;
  const int ry = threadIdx.x >> 5;
  const int ngroups = A.mode == 2 ? 2 : 1;
  for (int gi = 0; gi < ngroups; ++gi) {
    const int c = (A.mode == 2 ? blockIdx.x * 64 + gi * 32 : blockIdx.x * 32) + (threadIdx.x & 31);
    double s, t;
    if (A.mode == 2) slab_sums(out, slabs, (size_t)C, 0, -1, c, c < C, &s, &t);
    else slab_sums(out, slabs, (size_t)2 * C, 0, C, c, c < C, &s, &t);
    if (c < C && ry == 0) {
      if (A.mode == 0) {
        double mean = s / A.count;
        double var = t / A.count - mean * mean;
        if (var < 0.0) var = 0.0;
        A.mean_out[c] = (float)mean;
        A.rstd_out[c] = (float)(1.0 / sqrt(var + (double)A.eps));
        if (A.running_mean) {
          double unbiased = A.count > 1.0 ? var * A.count / (A.count - 1.0) : var;
          A.running_mean[c] = (float)((1.0 - A.momentum) * A.running_mean[c] + A.momentum * mean);
          A.running_var[c] = (float)((1.0 - A.momentum) * A.running_var[c] + A.momentum * unbiased);
        }
      } else if (A.mode == 1) {
        // s = sum dz, t = sum dz*y  ->  sum dz*xhat = rstd * (t - mean * s)
        const double rs = (double)A.rstd[c], mu = (double)A.mean[c];
        const double tx = rs * (t - mu * s);
        const double a = (double)A.gamma[c] * rs;
        // frozen (eval-mode / freeze_bn) statistics do not depend on the batch: dy = gamma * rstd * dz
        const double c1 = A.frozen ? 0.0 : s / A.count, c2 = A.frozen ? 0.0 : tx / A.count;
        const double bq = -a * rs * c2;
        A.coef[c] = (float)a;
        A.coef[C + c] = (float)bq;
        A.coef[2 * C + c] = (float)(-a * c1 - bq * mu);
        if (A.dgamma) A.dgamma[c] += (float)tx;
        if (A.dbeta) A.dbeta[c] += (float)s;
      } else {
        A.dbias[c] += (float)s;
      }
    }
    __syncthreads();          // slab_sums' shared buffer is reused by the next channel group
  }
}
static inline int32_t launch_colsum_finalize(const float* m, int rows, int cols, double* scratch, const FinArgs& A,
                                             cudaStream_t st) {
  int slabs = rows < kSlabs ? rows : kSlabs;
  int rps = (rows + slabs - 1) / slabs;
  slabs = (rows + rps - 1) / rps;
  // the ticket lives behind the slab sums (c3d_bn_scratch_bytes reserves it)
  unsigned int* ticket = reinterpret_cast<unsigned int*>(scratch + (size_t)kSlabs * cols);
  const int groups = A.mode == 2 ? (A.C + 63) / 64 : (A.C + 31) / 32;        // one ticket per column group (<= 64)
  cudaError_t e = cudaMemsetAsync(ticket, 0, sizeof(unsigned int) * groups, st);
  if (e != cudaSuccess) return set_error(C3D_ECUDA, "colsum ticket: %s", cudaGetErrorString(e));
  dim3 grid(groups, slabs);
  colsum_finalize_kernel<<<grid, 256, 0, st>>>(m, rows, cols, rps, scratch, ticket, A);
  return C3D_OK;
}

// ---- bias / ReLU backward for the bias convs (FPN, RPN head) -----------------------------------------
// dz = dout * (out > 0 if relu) written as bf16; partial[block][c] = sum over the block's pixels of dz (dbias)
template <int THREADS, typename TIN, typename TOUT>
__global__ void bias_act_bwd_kernel(const TIN* __restrict__ dout, const TOUT* __restrict__ out, int relu,
                                    bf16* __restrict__ dz, float* __restrict__ partial, long long P, int C) {
  const int cv = C >> 3;
  const int tx = threadIdx.x % cv, ty = threadIdx.x / cv;
  const int rows_per_block = THREADS / cv;
  const int c = tx << 3;
  float s[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) s[k] = 0.f;
  auto load = [&](const auto* p) {
    V8 r;
    if constexpr (sizeof(*p) == 2) { r = ld8(reinterpret_cast<const bf16*>(p)); }
    else {
      const float4* q = reinterpret_cast<const float4*>(p);
      float4 a = q[0], b = q[1];
      r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w; r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
    }
    return r;
  };
  if (ty < rows_per_block) {
    for (long long p = (long long)blockIdx.x * rows_per_block + ty; p < P; p += (long long)gridDim.x * rows_per_block) {
      V8 d = load(dout + p * C + c);
      if (relu) {
        V8 o = load(out + p * C + c);
#pragma unroll
        for (int k = 0; k < 8; ++k) if (!(o.v[k] > 0.f)) d.v[k] = 0.f;
      }
      if (dz) st8(dz + p * C + c, d);       // (no ReLU and a bf16 dout: dz == dout, the caller passes NULL and keeps dout)
#pragma unroll
      for (int k = 0; k < 8; ++k) s[k] += d.v[k];
    }
  }
  __shared__ float sm[THREADS][8 + 1];
#pragma unroll
  for (int k = 0; k < 8; ++k) sm[threadIdx.x][k] = s[k];
  __syncthreads();
  for (int ch = threadIdx.x; ch < C; ch += THREADS) {
    const int vx = ch >> 3, k = ch & 7;
    float acc = 0.f;
    for (int r = 0; r < rows_per_block; ++r) acc += sm[r * cv + vx][k];
    partial[(size_t)blockIdx.x * C + ch] = acc;
  }
}

// dsmall[n,h,w,c] = sum of the 2x2 block of dbig (gradient of nearest x2 upsampling), bf16 in/out
__global__ void sumpool2_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int N, int H, int W, int C) {
  const int Ho = H >> 1, Wo = W >> 1, cv = C >> 3;
  const long long total = (long long)N * Ho * Wo * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) << 3;
    long long p = i / cv;
    const int wo = (int)(p % Wo); p /= Wo;
    const int ho = (int)(p % Ho);
    const int n = (int)(p / Ho);
    const long long base = ((long long)n * H + 2 * ho) * W + 2 * wo;
    V8 a = ld8(x + base * C + c), b = ld8(x + (base + 1) * C + c);
    V8 d = ld8(x + (base + W) * C + c), e = ld8(x + (base + W + 1) * C + c);
    V8 o;
#pragma unroll
    for (int k = 0; k < 8; ++k) o.v[k] = (a.v[k] + b.v[k]) + (d.v[k] + e.v[k]);
    st8(y + (((long long)n * Ho + ho) * Wo + wo) * C + c, o);
  }
}

// z (N,2Ho,2Wo,C) = dy scattered to the even positions, zeros elsewhere (input of the stride-2 data gradient)
__global__ void zero_stuff2_kernel(const bf16* __restrict__ dy, bf16* __restrict__ z, int N, int Ho, int Wo, int H,
                                   int W, int C) {
  const int cv = C >> 3;
  const long long total = (long long)N * H * W * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) << 3;
    long long p = i / cv;
    const int w = (int)(p % W); p /= W;
    const int h = (int)(p % H);
    const int n = (int)(p / H);
    V8 o;
#pragma unroll
    for (int k = 0; k < 8; ++k) o.v[k] = 0.f;
    if (!(h & 1) && !(w & 1) && (h >> 1) < Ho && (w >> 1) < Wo)
      o = ld8(dy + (((long long)n * Ho + (h >> 1)) * Wo + (w >> 1)) * C + c);
    st8(z + i * 8, o);
  }
}

// ---- 2x2 stride-2 max pool (NHWC) -------------------------------------------------------------
__global__ void maxpool2_fwd_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int N, int H, int W, int C) {
  const int Ho = H >> 1, Wo = W >> 1, cv = C >> 3;
  const long long total = (long long)N * Ho * Wo * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) << 3;
    long long p = i / cv;
    const int wo = (int)(p % Wo); p /= Wo;
    const int ho = (int)(p % Ho);
    const int n = (int)(p / Ho);
    const long long base = ((long long)n * H + 2 * ho) * W + 2 * wo;
    V8 a = ld8(x + base * C + c), b = ld8(x + (base + 1) * C + c);
    V8 d = ld8(x + (base + W) * C + c), e = ld8(x + (base + W + 1) * C + c);
    V8 o;
#pragma unroll
    for (int k = 0; k < 8; ++k) o.v[k] = fmaxf(fmaxf(a.v[k], b.v[k]), fmaxf(d.v[k], e.v[k]));
    st8(y + (((long long)n * Ho + ho) * Wo + wo) * C + c, o);
  }
}
// dx (N,H,W,C) = dy routed to the first maximal element of each window (row-major window order)
template <bool ACC>
__global__ void maxpool2_bwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ dy, bf16* __restrict__ dx,
                                    int N, int H, int W, int C, long long dy_stride, long long dx_stride) {
  const int Ho = H >> 1, Wo = W >> 1, cv = C >> 3;
  const long long total = (long long)N * Ho * Wo * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) << 3;
    long long p = i / cv;
    const int wo = (int)(p % Wo); p /= Wo;
    const int ho = (int)(p % Ho);
    const int n = (int)(p / Ho);
    const long long base = ((long long)n * H + 2 * ho) * W + 2 * wo;
    const long long off[4] = {base, base + 1, base + W, base + W + 1};
    V8 v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = ld8(x + off[j] * C + c);
    V8 g = ld8(dy + (((long long)n * Ho + ho) * Wo + wo) * dy_stride + c);
    V8 o[4];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      int best = 0; float bv = v[0].v[k];
#pragma unroll
      for (int j = 1; j < 4; ++j) if (v[j].v[k] > bv) { bv = v[j].v[k]; best = j; }
#pragma unroll
      for (int j = 0; j < 4; ++j) o[j].v[k] = (j == best) ? g.v[k] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (ACC) {                       // dx already holds the gradient of x's other consumers
        const V8 r = ld8(dx + off[j] * dx_stride + c);
#pragma unroll
        for (int k = 0; k < 8; ++k) o[j].v[k] += r.v[k];
      }
      st8(dx + off[j] * dx_stride + c, o[j]);
    }
  }
}

// ---- 3x3 stride-2 pad-1 max pool (NHWC): the torchvision ResNet stem pool (resnet.py:17-27 -> nn.MaxPool2d(3,2,1)) ----
__device__ __forceinline__ int pool3_out(int n) { return (n - 1) / 2 + 1; }      // floor((n + 2 - 3) / 2) + 1
__global__ void maxpool3s2_fwd_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int N, int H, int W, int C) {
  const int Ho = pool3_out(H), Wo = pool3_out(W), cv = C >> 3;
  const long long total = (long long)N * Ho * Wo * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) << 3;
    long long p = i / cv;
    const int wo = (int)(p % Wo); p /= Wo;
    const int ho = (int)(p % Ho);
    const int n = (int)(p / Ho);
    V8 o;
#pragma unroll
    for (int k = 0; k < 8; ++k) o.v[k] = -INFINITY;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int h = 2 * ho - 1 + kh;
      if (h < 0 || h >= H) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int w = 2 * wo - 1 + kw;
        if (w < 0 || w >= W) continue;
        V8 a = ld8(x + (((long long)n * H + h) * W + w) * C + c);
#pragma unroll
        for (int k = 0; k < 8; ++k) o.v[k] = fmaxf(o.v[k], a.v[k]);
      }
    }
    st8(y + (((long long)n * Ho + ho) * Wo + wo) * C + c, o);
  }
}
// dx[h,w] = sum over the (<= 4) windows containing (h,w) whose FIRST maximal element (row-major window order, the
// order ATen's max_pool2d resolves ties in) is (h,w), of dy[window].  Gather form: no atomics, no saved indices.
__global__ void maxpool3s2_bwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ dy, bf16* __restrict__ dx,
                                      int N, int H, int W, int C, long long dy_stride) {
  const int Ho = pool3_out(H), Wo = pool3_out(W), cv = C >> 3;
  const long long total = (long long)N * H * W * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % cv) << 3;
    long long p = i / cv;
    const int w = (int)(p % W); p /= W;
    const int h = (int)(p % H);
    const int n = (int)(p / H);
    const bf16* xn = x + (long long)n * H * W * C + c;
    const V8 me = ld8(xn + ((long long)h * W + w) * C);
    V8 acc;
#pragma unroll
    for (int k = 0; k < 8; ++k) acc.v[k] = 0.f;
    // windows ho with 2*ho-1 <= h <= 2*ho+1
    for (int ho = h >> 1; ho <= (h + 1) >> 1; ++ho) {
      if (ho >= Ho) continue;
      for (int wo = w >> 1; wo <= (w + 1) >> 1; ++wo) {
        if (wo >= Wo) continue;
        const int my = (h - (2 * ho - 1)) * 3 + (w - (2 * wo - 1));      // my position in that window's scan order
        bool win[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) win[k] = true;
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
          const int hh = 2 * ho - 1 + kh;
          if (hh < 0 || hh >= H) continue;
#pragma unroll
          for (int kw = 0; kw < 3; ++kw) {
            const int ww = 2 * wo - 1 + kw;
            const int pos = kh * 3 + kw;
            if (ww < 0 || ww >= W || pos == my) continue;
            const V8 o = ld8(xn + ((long long)hh * W + ww) * C);
#pragma unroll
            for (int k = 0; k < 8; ++k)       // an earlier element wins ties, a later one must be strictly larger
              if (pos < my ? (o.v[k] >= me.v[k]) : (o.v[k] > me.v[k])) win[k] = false;
          }
        }
        const V8 g = ld8(dy + (((long long)n * Ho + ho) * Wo + wo) * dy_stride + c);
#pragma unroll
        for (int k = 0; k < 8; ++k) if (win[k]) acc.v[k] += g.v[k];
      }
    }
    st8(dx + (((long long)n * H + h) * W + w) * C + c, acc);
  }
}

// ---- weight re-pack: fp32 OIHW / OHWI master -> bf16 OHWI (forward), bf16 rotated/transposed (data gradient) and the
// stride-2 phase sub-kernels (include/c3d.h c3d_pack_desc) ----
// Element i of D's source writes its forward-pack entry, its rotated / transposed data-gradient entry and — for 3x3
// stride-2 layers — its entry in the phase sub-kernel it belongs to (parity 0 uses tap [1], parity 1 taps [2, 0]).
__device__ __forceinline__ void pack_conv_weight_element(const c3d_pack_desc& D, long long i) {
  int kw, kh, ci, co;
  if (D.src_is_ohwi) {
    ci = (int)(i % D.Cin); long long t = i / D.Cin;
    kw = (int)(t % D.KW); t /= D.KW;
    kh = (int)(t % D.KH); co = (int)(t / D.KH);
  } else {
    kw = (int)(i % D.KW); long long t = i / D.KW;
    kh = (int)(t % D.KH); t /= D.KH;
    ci = (int)(t % D.Cin); co = (int)(t / D.Cin);
  }
  const bf16 v = __float2bfloat16(D.src[i]);
  if (D.fwd) static_cast<bf16*>(D.fwd)[(((long long)co * D.KH + kh) * D.KW + kw) * D.Cin + ci] = v;
  if (D.dgrad) static_cast<bf16*>(D.dgrad)[(((long long)ci * D.KH + (D.KH - 1 - kh)) * D.KW + (D.KW - 1 - kw)) * D.Cout + co] = v;
  if (D.phase[0]) {               // 3x3 only: parity a = (kh != 1), position inside the phase: kh 1 -> 0 | kh 2 -> 0, kh 0 -> 1
    const int a = kh != 1, b = kw != 1;
    const int ph = a ? (kh == 2 ? 0 : 1) : 0, pw = b ? (kw == 2 ? 0 : 1) : 0;
    // merged_phases: every phase is a 2x2 row block of one (4*Cin, 2, 2, Cout) weight (include/c3d.h c3d_pack_desc)
    const int KHp = (a || D.merged_phases) ? 2 : 1, KWp = (b || D.merged_phases) ? 2 : 1;
    static_cast<bf16*>(D.phase[a * 2 + b])[(((long long)ci * KHp + ph) * KWp + pw) * D.Cout + co] = v;
  }
}

// one weight; the descriptor travels in the kernel parameters (no host->device copy: the launch can be graph-captured)
__global__ void pack_conv_weight_desc_kernel(const c3d_pack_desc D, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    pack_conv_weight_element(D, i);
}

// every conv weight of a model in ONE launch: element e belongs to the descriptor with the last start <= e
__global__ void pack_conv_weights_batched_kernel(const c3d_pack_desc* __restrict__ descs, int n, long long total) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    int lo = 0, hi = n;
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (descs[mid].start <= e) lo = mid; else hi = mid; }
    const c3d_pack_desc D = descs[lo];
    pack_conv_weight_element(D, e - D.start);
  }
}

// ---- image normalisation: (3,H,W) fp32 / uint8 BGR -> (Hp,Wp,Cp) bf16 NHWC slots, zero padded -------------
// all images of a batch in ONE launch (blockIdx.y = image; pointers and sizes travel in the kernel parameters)
constexpr int kPreBatch = 64;
struct PreBatch { const void* img[kPreBatch]; int H[kPreBatch]; int W[kPreBatch]; };
template <typename T>
__global__ void preprocess_batch_kernel(const PreBatch B, bf16* __restrict__ out, int Hp, int Wp, int Cp, float m0, float m1,
                                        float m2, float s0, float s1, float s2) {
  const int n = blockIdx.y;
  const T* __restrict__ img = static_cast<const T*>(B.img[n]);
  const int H = B.H[n], W = B.W[n];
  const long long total = (long long)Hp * Wp;
  bf16* base = out + (size_t)n * total * Cp;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int w = (int)(i % Wp), h = (int)(i / Wp);
    float v0 = 0.f, v1 = 0.f, v2 = 0.f;
    if (h < H && w < W) {
      const long long o = (long long)h * W + w;
      v0 = ((float)img[o] - m0) / s0;
      v1 = ((float)img[(long long)H * W + o] - m1) / s1;
      v2 = ((float)img[2LL * H * W + o] - m2) / s2;
    }
    bf16* dst = base + i * Cp;
    for (int c = 0; c < Cp; c += 8) {
      V8 z;
#pragma unroll
      for (int k = 0; k < 8; ++k) z.v[k] = 0.f;
      if (c == 0) { z.v[0] = v0; z.v[1] = v1; z.v[2] = v2; }
      st8(dst + c, z);
    }
  }
}

// ---- fused SGD momentum (+weight decay) with finite check ----------------------------------------
// flags[0] != 0 on entry => skip (another rank or the loss check vetoed the step).  The finite scan is a
// separate tiny pass (grad_finite_kernel) so that all ranks can agree before anyone updates.
__global__ void grad_finite_kernel(const float* __restrict__ g, long long n, int* __restrict__ flag) {
  int bad = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float v = g[i];
    if (!(fabsf(v) <= 3.402823466e38f)) bad = 1;     // NaN or Inf
  }
  if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicOr(flag, 1);
}
__global__ void sgd_momentum_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ mom,
                                    long long n, float lr, const float* __restrict__ lr_dev, float momentum, float wd,
                                    float grad_scale, const int* __restrict__ skip_flag) {
  if (skip_flag && *skip_flag) return;
  if (lr_dev) lr = *lr_dev;                  // learning rate in device memory: the launch can live in a CUDA graph
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float d = g[i] * grad_scale + wd * p[i];
    float b = momentum * mom[i] + d;        // torch.optim.SGD: buf = momentum*buf + d (dampening 0)
    mom[i] = b;
    p[i] = p[i] - lr * b;
  }
}

}  // namespace c3d

using namespace c3d;
#define C3D_REQ(cond, msg) do { if (!(cond)) return set_error(C3D_EINVAL, msg); } while (0)

extern "C" size_t c3d_bn_scratch_bytes(int32_t C) {      // slab sums + the last-block ticket behind them
  return ((size_t)kSlabs * 2 * (size_t)(C > 0 ? C : 0) + 64) * sizeof(double);
}
extern "C" int32_t c3d_bn_finalize(const float* partial, int32_t rows, int32_t C, double count, float eps,
                                   float momentum, float* running_mean, float* running_var, float* mean_out,
                                   float* rstd_out, void* scratch, void* stream) {
  C3D_REQ(partial && mean_out && rstd_out && scratch && rows > 0 && C > 0, "bn_finalize: bad args");
  FinArgs A{};
  A.mode = 0; A.C = C; A.count = count; A.eps = eps; A.momentum = momentum;
  A.running_mean = running_mean; A.running_var = running_var; A.mean_out = mean_out; A.rstd_out = rstd_out;
  int32_t rc = launch_colsum_finalize(partial, rows, 2 * C, (double*)scratch, A, (cudaStream_t)stream);
  if (rc != C3D_OK) return rc;
  return check_launch("bn_finalize");
}
extern "C" int32_t c3d_bn_apply(const void* y, const float* mean, const float* rstd, const float* gamma,
                                const float* beta, const void* residual, int32_t relu, void* out, int64_t P,
                                int32_t C, void* stream) {
  C3D_REQ(y && mean && rstd && gamma && beta && out && C % 8 == 0, "bn_apply: bad args");
  if (P == 0) return C3D_OK;
  C3D_REQ(C <= 2048, "bn_apply: C too large");
  bn_apply_kernel<<<grid_for(P * (C / 8), 256), 256, 0, (cudaStream_t)stream>>>(
      (const bf16*)y, mean, rstd, gamma, beta, (const bf16*)residual, relu, (bf16*)out, P, C);
  return check_launch("bn_apply");
}
extern "C" int32_t c3d_bn_bwd_blocks(int64_t P, int32_t C) {
  if (C % 8 != 0 || C > 2048) return 0;
  int rows = 256 / (C / 8); if (rows < 1) rows = 1;
  long long b = (P + rows * 8LL - 1) / (rows * 8LL);
  if (b > kNumSMs * 4) b = kNumSMs * 4;
  if (b < 1) b = 1;
  return (int32_t)b;
}
extern "C" int32_t c3d_bn_bwd(const void* dout, const void* out, const void* y, const float* mean, const float* rstd,
                              const float* gamma, const float* beta, int32_t relu, int32_t frozen_stats,
                              float* partial /*[blocks][2][C]*/, float* coef /*[3][C]*/,
                              float* dgamma, float* dbeta, void* dy, void* dres, int64_t P, int32_t C,
                              int64_t dout_stride, int64_t dres_stride, void* scratch, void* stream) {
  const int dres_acc = (relu >> 1) & 1;          // flags: bit 0 = ReLU, bit 1 = dres += (instead of =)
  relu &= 1;
  C3D_REQ(dout && y && mean && rstd && gamma && partial && coef && dy && scratch && C % 8 == 0 && C <= 2048,
          "bn_bwd: bad args");
  C3D_REQ(!relu || out || beta, "bn_bwd: relu needs the forward output, or beta to recompute its sign from y");
  if (P == 0) return C3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int blocks = c3d_bn_bwd_blocks(P, C);
  const long long ds = dout_stride ? dout_stride : C;
  if (C / 8 <= 256)
    bn_bwd_reduce_kernel<256><<<blocks, 256, 0, st>>>((const bf16*)dout, (const bf16*)out, (const bf16*)y, mean, rstd,
                                                       relu, partial, P, C, ds, gamma, beta);
  else
    return set_error(C3D_EINVAL, "bn_bwd: C too large");
  FinArgs A{};
  A.mode = 1; A.C = C; A.count = (double)P; A.gamma = gamma; A.rstd = rstd; A.mean = mean; A.coef = coef; A.dgamma = dgamma; A.dbeta = dbeta;
  A.frozen = frozen_stats;
  int32_t rc = launch_colsum_finalize(partial, blocks, 2 * C, (double*)scratch, A, st);
  if (rc != C3D_OK) return rc;
  bn_bwd_apply_kernel<<<grid_for(P * (C / 8), 256), 256, 0, st>>>((const bf16*)dout, (const bf16*)out, (const bf16*)y,
                                                                   mean, rstd, coef, relu, (bf16*)dy, (bf16*)dres, P, C,
                                                                   ds, dres_stride ? dres_stride : C, gamma, beta, dres_acc);
  return check_launch("bn_bwd");
}
extern "C" int32_t c3d_maxpool2_fwd(const void* x, void* y, int32_t N, int32_t H, int32_t W, int32_t C, void* stream) {
  C3D_REQ(x && y && C % 8 == 0 && H % 2 == 0 && W % 2 == 0, "maxpool2: bad args");
  long long work = (long long)N * (H / 2) * (W / 2) * (C / 8);
  if (work == 0) return C3D_OK;
  maxpool2_fwd_kernel<<<grid_for(work, 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)x, (bf16*)y, N, H, W, C);
  return check_launch("maxpool2_fwd");
}
extern "C" int32_t c3d_maxpool2_bwd(const void* x, const void* dy, void* dx, int32_t N, int32_t H, int32_t W, int32_t C,
                                    int64_t dy_stride, int64_t dx_stride, int32_t accumulate, void* stream) {
  C3D_REQ(x && dy && dx && C % 8 == 0 && H % 2 == 0 && W % 2 == 0, "maxpool2_bwd: bad args");
  long long work = (long long)N * (H / 2) * (W / 2) * (C / 8);
  if (work == 0) return C3D_OK;
  auto kern = accumulate ? maxpool2_bwd_kernel<true> : maxpool2_bwd_kernel<false>;
  kern<<<grid_for(work, 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)x, (const bf16*)dy, (bf16*)dx, N, H, W, C,
                                                              dy_stride ? dy_stride : C, dx_stride ? dx_stride : C);
  return check_launch("maxpool2_bwd");
}
extern "C" int32_t c3d_maxpool3s2_fwd(const void* x, void* y, int32_t N, int32_t H, int32_t W, int32_t C, void* stream) {
  C3D_REQ(x && y && C % 8 == 0 && H >= 1 && W >= 1, "maxpool3s2: bad args");
  long long work = (long long)N * ((H - 1) / 2 + 1) * ((W - 1) / 2 + 1) * (C / 8);
  if (work == 0) return C3D_OK;
  maxpool3s2_fwd_kernel<<<grid_for(work, 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)x, (bf16*)y, N, H, W, C);
  return check_launch("maxpool3s2_fwd");
}
extern "C" int32_t c3d_maxpool3s2_bwd(const void* x, const void* dy, void* dx, int32_t N, int32_t H, int32_t W,
                                      int32_t C, int64_t dy_stride, void* stream) {
  C3D_REQ(x && dy && dx && C % 8 == 0 && H >= 1 && W >= 1, "maxpool3s2_bwd: bad args");
  long long work = (long long)N * H * W * (C / 8);
  if (work == 0) return C3D_OK;
  maxpool3s2_bwd_kernel<<<grid_for(work, 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)x, (const bf16*)dy, (bf16*)dx,
                                                                               N, H, W, C, dy_stride ? dy_stride : C);
  return check_launch("maxpool3s2_bwd");
}
extern "C" int32_t c3d_pack_conv_weights_batched(const void* descs_dev, int32_t n, int64_t total_elems, void* stream) {
  C3D_REQ(descs_dev && n > 0 && total_elems > 0, "pack_conv_weights_batched: bad args");
  pack_conv_weights_batched_kernel<<<grid_for(total_elems, 256), 256, 0, (cudaStream_t)stream>>>(
      static_cast<const c3d_pack_desc*>(descs_dev), n, total_elems);
  return check_launch("pack_conv_weights_batched");
}
extern "C" int32_t c3d_preprocess_batch(const void* const* imgs_host, const int32_t* H_host, const int32_t* W_host, int32_t N,
                                        int32_t is_u8, void* out, int32_t Hp, int32_t Wp, int32_t Cp, const float* mean3_host,
                                        const float* std3_host, void* stream) {
  C3D_REQ(imgs_host && H_host && W_host && out && mean3_host && std3_host && Cp % 8 == 0 && N >= 0, "preprocess_batch: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  for (int n0 = 0; n0 < N; n0 += kPreBatch) {
    const int nb = N - n0 < kPreBatch ? N - n0 : kPreBatch;
    PreBatch B;
    for (int i = 0; i < nb; ++i) {
      C3D_REQ(imgs_host[n0 + i] && H_host[n0 + i] <= Hp && W_host[n0 + i] <= Wp, "preprocess_batch: image larger than the slot");
      B.img[i] = imgs_host[n0 + i]; B.H[i] = H_host[n0 + i]; B.W[i] = W_host[n0 + i];
    }
    int bx = grid_for((long long)Hp * Wp, 256);
    if (bx > 4 * kNumSMs) bx = 4 * kNumSMs;
    bf16* o = (bf16*)out + (size_t)n0 * Hp * Wp * Cp;
    if (is_u8)
      preprocess_batch_kernel<uint8_t><<<dim3(bx, nb), 256, 0, st>>>(B, o, Hp, Wp, Cp, mean3_host[0], mean3_host[1], mean3_host[2],
                                                                     std3_host[0], std3_host[1], std3_host[2]);
    else
      preprocess_batch_kernel<float><<<dim3(bx, nb), 256, 0, st>>>(B, o, Hp, Wp, Cp, mean3_host[0], mean3_host[1], mean3_host[2],
                                                                   std3_host[0], std3_host[1], std3_host[2]);
  }
  return check_launch("preprocess_batch");
}
extern "C" int32_t c3d_grad_finite(const float* g, int64_t n, int32_t* flag, void* stream) {
  C3D_REQ(g && flag, "grad_finite: bad args");
  if (n == 0) return C3D_OK;
  grad_finite_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(g, n, flag);
  return check_launch("grad_finite");
}
extern "C" int32_t c3d_sgd_momentum(float* p, const float* g, float* mom, int64_t n, float lr, const float* lr_dev,
                                    float momentum, float weight_decay, float grad_scale, const int32_t* skip_flag,
                                    void* stream) {
  C3D_REQ(p && g && mom, "sgd: bad args");
  if (n == 0) return C3D_OK;
  sgd_momentum_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(p, g, mom, n, lr, lr_dev, momentum,
                                                                           weight_decay, grad_scale, skip_flag);
  return check_launch("sgd");
}

extern "C" int32_t c3d_bias_act_bwd(const void* dout, const void* out, int32_t relu, int32_t dtype_flags, void* dz,
                                    float* partial /*[c3d_bn_bwd_blocks(P,C)][C]*/, float* dbias, int64_t P, int32_t C,
                                    void* scratch, void* stream) {
  C3D_REQ(dout && partial && scratch && C % 8 == 0 && C <= 2048, "bias_act_bwd: bad args");
  C3D_REQ(!relu || out, "bias_act_bwd: relu needs the forward output");
  C3D_REQ(dz || (!relu && !(dtype_flags & 1)), "bias_act_bwd: dz may be NULL only without ReLU and with a bf16 dout (dz == dout)");
  if (P == 0) return C3D_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int blocks = c3d_bn_bwd_blocks(P, C);
  // dtype_flags: bit 0 = dout is fp32, bit 1 = out is fp32 (the forward output keeps its own dtype: a ReLU conv saves
  // a bf16 `out` even when its consumer hands back an fp32 gradient)
  const bool din32 = dtype_flags & 1, out32 = dtype_flags & 2;
#define C3D_BAB(TI, TO) bias_act_bwd_kernel<256, TI, TO><<<blocks, 256, 0, st>>>((const TI*)dout, (const TO*)out, relu, \
                                                                                 (bf16*)dz, partial, P, C)
  if (din32 && out32) C3D_BAB(float, float);
  else if (din32) C3D_BAB(float, bf16);
  else if (out32) C3D_BAB(bf16, float);
  else C3D_BAB(bf16, bf16);
#undef C3D_BAB
  if (dbias) {
    FinArgs A{};
    A.mode = 2; A.C = C; A.dbias = dbias;
    int32_t rc = launch_colsum_finalize(partial, blocks, C, (double*)scratch, A, st);
    if (rc != C3D_OK) return rc;
  }
  return check_launch("bias_act_bwd");
}
extern "C" int32_t c3d_sumpool2(const void* x, void* y, int32_t N, int32_t H, int32_t W, int32_t C, void* stream) {
  C3D_REQ(x && y && C % 8 == 0 && H % 2 == 0 && W % 2 == 0, "sumpool2: bad args");
  long long work = (long long)N * (H / 2) * (W / 2) * (C / 8);
  if (work == 0) return C3D_OK;
  sumpool2_kernel<<<grid_for(work, 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)x, (bf16*)y, N, H, W, C);
  return check_launch("sumpool2");
}
extern "C" int32_t c3d_zero_stuff2(const void* dy, void* z, int32_t N, int32_t Ho, int32_t Wo, int32_t H, int32_t W,
                                   int32_t C, void* stream) {
  C3D_REQ(dy && z && C % 8 == 0, "zero_stuff2: bad args");
  long long work = (long long)N * H * W * (C / 8);
  if (work == 0) return C3D_OK;
  zero_stuff2_kernel<<<grid_for(work, 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)dy, (bf16*)z, N, Ho, Wo, H, W, C);
  return check_launch("zero_stuff2");
}

extern "C" int32_t c3d_pack_conv_weight(const c3d_pack_desc* desc_host, void* stream) {
  C3D_REQ(desc_host && desc_host->src, "pack_conv_weight: null source");
  const c3d_pack_desc D = *desc_host;
  const bool phases = D.phase[0] || D.phase[1] || D.phase[2] || D.phase[3];
  C3D_REQ(D.fwd || D.dgrad || phases, "pack_conv_weight: no output");
  C3D_REQ(!phases || (D.phase[0] && D.phase[1] && D.phase[2] && D.phase[3] && D.KH == 3 && D.KW == 3),
          "pack_conv_weight: phase outputs need all four buffers and a 3x3 weight");
  C3D_REQ(D.Cout >= 0 && D.Cin >= 0 && D.KH >= 0 && D.KW >= 0, "pack_conv_weight: negative size");
  const long long total = (long long)D.Cout * D.Cin * D.KH * D.KW;
  if (total == 0) return C3D_OK;
  pack_conv_weight_desc_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(D, total);
  return check_launch("pack_conv_weight");
}
