// select_ops.cu — selection / sampling kernels of the RPN and ROI-head glue (one launch each, no host sync).
//
//   topk_segments_kernel     sorted top-k of many (image, segment) rows in one launch: per-level RPN pre-NMS top-k
//                            (detectron2 find_top_rpn_proposals via cubercnn/modeling/proposal_generator/rpn.py:221-284,
//                            configs/Base.yaml:51-54), the score sort of the concatenated candidates, the top-M of the
//                            inference candidates (fast_rcnn.py:57-116) and the Gumbel top-k of the anchor sampler.
//                            Radix select (11/11/10 bits) on order-preserving keys -> compaction into shared memory ->
//                            bitonic sort.  Replaces ATen mbtopk / radix-sort launches.
//   label_sample_kernel      ROIHeads3D.label_and_sample_proposals (cubercnn/modeling/roi_heads/roi_heads.py:826-929) for
//                            one image per block: IoU matcher (+ appended GT), ignore-region rule, IoU-weighted sampling
//                            without replacement (Gumbel top-k == torch.multinomial in distribution), fg-first slot
//                            compaction and the gather of the matched GT fields.  Replaces ~180 ATen launches.
//   anchor_sample_*          RPNWithIgnore.label_and_sample_anchors' sampling part (rpn.py:62-105, 275-328).
// IoU arithmetic: explicit round-to-nearest intrinsics in the operation order of the torch formulation
// (omni3d_b200/cubercnn/rpn.py pairwise_iou / pairwise_ioa) => labels / matches are bit-identical to it.
#include <stdint.h>
#include "c3d_common.cuh"

namespace c3d {

// ---- counter-based RNG: Philox4x32-10 (Salmon et al., SC'11), one call -> 4 x 32 random bits -----------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    const uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0; key.y += W1;
  }
  return ctr;
}
// uniform in (0, 1): never 0 or 1, so log(-log(u)) is finite
__device__ __forceinline__ float u01(uint32_t x) { return ((float)(x >> 8) + 0.5f) * (1.0f / 16777216.0f); }
// Gumbel-max key of weight w > 0: arg-top-k of log(w) + G  ==  sampling without replacement with probabilities ~ w
__device__ __forceinline__ float gumbel_key(float w, uint32_t bits) { return __logf(w) - __logf(-__logf(u01(bits))); }

// order-preserving float -> uint32 (larger float => larger key; +NaN sorts above +inf like torch.topk)
__device__ __forceinline__ uint32_t fkey(float v) {
  const uint32_t u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float fkey_inv(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// bitonic sort of n2 (power of two) 64-bit words in shared memory, DESCENDING; all threads of the block participate
__device__ void bitonic_desc(unsigned long long* s, int n2) {
  for (int size = 2; size <= n2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < (n2 >> 1); i += blockDim.x) {
        const int lo = 2 * i - (i & (stride - 1));
        const int hi = lo + stride;
        const bool up = (lo & size) == 0;
        const unsigned long long a = s[lo], b = s[hi];
        if ((a < b) == up) { s[lo] = b; s[hi] = a; }
      }
      __syncthreads();
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
constexpr int kTopkMaxSeg = 8;
struct TopkSeg {
  const float* vals;        // row b at vals + b * row_stride
  long long row_stride;
  int n, k, out_col;
};
struct TopkParams {
  TopkSeg seg[kTopkMaxSeg];
  int out_stride;           // elements per image row of out_vals / out_idx
  float* out_vals;          // [B][out_stride]
  int* out_idx;             // [B][out_stride] int32 (index inside the segment's row), may be null
  long long* out_idx64;     // same as int64 (torch index dtype), may be null
  int* out_count;           // [B][nseg] number of finite (> -inf) selected values, may be null
  int nseg;
};

__global__ void __launch_bounds__(1024)
topk_segments_kernel(const TopkParams P) {
  extern __shared__ unsigned long long sel[];            // [k2] (key << 32 | ~index)
  __shared__ int hist[2048];
  __shared__ int s_digit, s_need, s_cnt_gt, s_fin;
  __shared__ int s_weq[32];                             // per-warp counts of elements equal to the threshold
  const int b = blockIdx.x;
  const TopkSeg S = P.seg[blockIdx.y];
  const float* v = S.vals + (long long)b * S.row_stride;
  const int n = S.n, k = S.k < S.n ? S.k : S.n;
  int k2 = 1;
  while (k2 < k) k2 <<= 1;
  if (k2 < 2) k2 = 2;
  const int tid = threadIdx.x;

  uint32_t T = 0;          // key of the k-th largest element
  int need = 0;            // how many elements equal to T belong to the top-k
  if (k < n) {
    uint32_t prefix = 0, mask = 0;
    int want = k;
    const int shifts[3] = {21, 10, 0}, bits[3] = {11, 11, 10};
    for (int pass = 0; pass < 3; ++pass) {
      const int sh = shifts[pass], nb = 1 << bits[pass];
      for (int i = tid; i < nb; i += blockDim.x) hist[i] = 0;
      __syncthreads();
      for (int i = tid; i < n; i += blockDim.x) {
        const uint32_t u = fkey(v[i]);
        if ((u & mask) == prefix) atomicAdd(&hist[(u >> sh) & (nb - 1)], 1);
      }
      __syncthreads();
      if (tid < 32) {                                     // one warp: find the digit holding the want-th largest
        const int per = nb / 32;
        int mine = 0;
        for (int j = 0; j < per; ++j) mine += hist[tid * per + j];
        // suffix sums over lanes (lane 31 = largest digits)
        int suf = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int t = __shfl_down_sync(0xffffffffu, suf, o);
          if (tid + o < 32) suf += t;
        }
        const int above = suf - mine;                     // elements in strictly higher lanes
        const bool here = above < want && suf >= want;
        if (here) {
          int c = above, d = tid * per + per - 1;
          for (; d >= tid * per; --d) { c += hist[d]; if (c >= want) break; }
          s_digit = d;
          s_need = want - (c - hist[d]);
        }
      }
      __syncthreads();
      prefix |= (uint32_t)s_digit << sh;
      mask |= (uint32_t)(nb - 1) << sh;
      want = s_need;
      __syncthreads();
    }
    T = prefix;
    need = want;
  }
  if (tid == 0) { s_cnt_gt = 0; s_fin = 0; }
  for (int i = tid; i < k2; i += blockDim.x) sel[i] = 0ull;       // padding sorts last
  __syncthreads();
  int fin = 0;
  const uint32_t ninf = fkey(-INFINITY);
  if (k < n) {
    // elements above T land in any order (the sort below orders them by (key, index)); of the elements EQUAL to T the
    // `need` lowest indices are kept — counted in index order (block-wide prefix over the tile), never in atomic
    // arrival order, so the selected set is the same on every run
    const int base_eq = k - need;
    const int lane = tid & 31, wid = tid >> 5, nw = (blockDim.x + 31) >> 5;
    int eq_before = 0;                                        // tied elements in earlier tiles
    for (int i0 = 0; i0 < n; i0 += blockDim.x) {
      const int i = i0 + tid;
      const uint32_t u = i < n ? fkey(v[i]) : 0u;
      const bool eq = i < n && u == T;
      const unsigned bal = __ballot_sync(0xffffffffu, eq);
      if (lane == 0) s_weq[wid] = __popc(bal);
      __syncthreads();
      int before = eq_before, tile = 0;
      for (int w = 0; w < nw; ++w) { const int c = s_weq[w]; tile += c; if (w < wid) before += c; }
      __syncthreads();                                        // s_weq is rewritten by the next tile
      eq_before += tile;
      int pos = -1;
      if (i < n && u > T) pos = atomicAdd(&s_cnt_gt, 1);
      else if (eq) { const int e = before + __popc(bal & ((1u << lane) - 1u)); if (e < need) pos = base_eq + e; }
      if (pos >= 0) { sel[pos] = ((unsigned long long)u << 32) | (uint32_t)(~(uint32_t)i); fin += u > ninf; }
    }
  } else {
    for (int i = tid; i < n; i += blockDim.x) {
      const uint32_t u = fkey(v[i]);
      sel[i] = ((unsigned long long)u << 32) | (uint32_t)(~(uint32_t)i);
      fin += u > ninf;
    }
  }
  if (P.out_count) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) fin += __shfl_xor_sync(0xffffffffu, fin, o);
    if ((tid & 31) == 0 && fin) atomicAdd(&s_fin, fin);
  }
  __syncthreads();
  bitonic_desc(sel, k2);
  const long long o0 = (long long)b * P.out_stride + S.out_col;
  for (int j = tid; j < S.k; j += blockDim.x) {
    float val = -INFINITY; int idx = 0;
    if (j < k) { const unsigned long long w = sel[j]; val = fkey_inv((uint32_t)(w >> 32)); idx = (int)(~(uint32_t)w); }
    P.out_vals[o0 + j] = val;
    if (P.out_idx) P.out_idx[o0 + j] = idx;
    if (P.out_idx64) P.out_idx64[o0 + j] = idx;
  }
  if (P.out_count && tid == 0) P.out_count[b * P.nseg + blockIdx.y] = s_fin;
}

// ------------------------------------------------------------------------------------------------------------------
// ROIHeads3D.label_and_sample_proposals, one image per block
__device__ __forceinline__ float area4(const float4 b) { return __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y)); }

struct LabelSampleParams {
  const float4* prop_boxes;      // [B][P]
  const int* prop_count;         // [B]
  const float4* gt_boxes;        // [B][G]
  const long long* gt_classes;   // [B][G]  (< 0: ignore region)
  const unsigned char* gt_present;   // [B][G]
  const float* gt_boxes3D;       // [B][G][9]
  const float* gt_poses;         // [B][G][9]
  int B, P, G, K, S, Fcap, append_gt;
  float iou_thresh, ignore_thresh;
  const unsigned long long* rng; // [2] = seed, step counter
  // pre-sampling outputs [B][P+G] (may be null)
  long long* matched_idx; float* matched_iou; long long* labels;
  // sampled outputs [B][S]
  float4* s_boxes; unsigned char* s_valid; long long* s_classes; float4* s_gt_boxes; float* s_gt_boxes3D; float* s_gt_poses;
  long long* s_index;            // index into [proposals | appended GT], may be null
  float* stats;                  // [2] += (#fg samples, #bg samples) summed over images
};

constexpr int kLsMaxN = 2048, kLsMaxG = 256;

__global__ void __launch_bounds__(1024)
label_sample_kernel(const LabelSampleParams Q) {
  __shared__ unsigned long long key[kLsMaxN];
  __shared__ short s_cls[kLsMaxN], s_midx[kLsMaxN];
  __shared__ float4 sg[kLsMaxG];
  __shared__ float sga[kLsMaxG];
  __shared__ short sgc[kLsMaxG];                 // class, -1 ignore, -2 absent
  __shared__ int c_bg, c_fgc, c_bgc, f_ign, f_valid;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int P = Q.P, G = Q.G, n = P + (Q.append_gt ? G : 0);
  if (tid == 0) { c_bg = 0; c_fgc = 0; c_bgc = 0; f_ign = 0; f_valid = 0; }
  __syncthreads();
  for (int g = tid; g < G; g += blockDim.x) {
    const float4 v = Q.gt_boxes[(size_t)b * G + g];
    sg[g] = v; sga[g] = area4(v);
    const bool pres = Q.gt_present[(size_t)b * G + g] != 0;
    const long long c = Q.gt_classes[(size_t)b * G + g];
    sgc[g] = (short)(!pres ? -2 : (c < 0 ? -1 : (c > 32000 ? 32000 : c)));
    if (pres && c < 0) f_ign = 1;
    if (pres && c >= 0) f_valid = 1;
  }
  __syncthreads();
  const int pc = Q.prop_count[b];
  float4 box[2]; float viou[2], vioa[2]; int vidx[2]; bool pvalid[2], fg[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int j = tid + r * 1024;
    pvalid[r] = false; fg[r] = false; viou[r] = 0.f; vioa[r] = 0.f; vidx[r] = 0; box[r] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (j >= n) continue;
    if (j < P) { box[r] = Q.prop_boxes[(size_t)b * P + j]; pvalid[r] = j < pc; }
    else { box[r] = sg[j - P]; pvalid[r] = sgc[j - P] >= 0; }
    const float ab = area4(box[r]);
    float best = -1.f, ioa = 0.f; int bi = 0;
    for (int g = 0; g < G; ++g) {
      const float4 q = sg[g];
      const float w = fmaxf(__fsub_rn(fminf(q.z, box[r].z), fmaxf(q.x, box[r].x)), 0.f);
      const float h = fmaxf(__fsub_rn(fminf(q.w, box[r].w), fmaxf(q.y, box[r].y)), 0.f);
      const float inter = __fmul_rn(w, h);
      const short c = sgc[g];
      if (c >= 0) {
        const float iou = inter > 0.f ? __fdiv_rn(inter, __fsub_rn(__fadd_rn(sga[g], ab), inter)) : 0.f;
        if (iou > best) { best = iou; bi = g; }
      } else if (c == -1) {
        ioa = fmaxf(ioa, inter > 0.f ? __fdiv_rn(inter, ab) : 0.f);
      }
    }
    // torch: (B,G,P) IoU with non-valid GT rows set to -1, max over G -> first maximum; all rows -1 => index 0
    viou[r] = best; vioa[r] = ioa; vidx[r] = bi;
    fg[r] = best >= Q.iou_thresh;
    if (!fg[r] && pvalid[r]) atomicAdd(&c_bg, 1);
  }
  __syncthreads();
  const bool ign_rule = c_bg > 1 && f_ign && f_valid;
  const unsigned long long seed = Q.rng ? Q.rng[0] : 0ull, step = Q.rng ? Q.rng[1] : 0ull;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int j = tid + r * 1024;
    if (j >= kLsMaxN) continue;
    unsigned long long kk = ~0ull;                    // group 3: not a candidate (sorts last)
    if (j < n) {
      const bool bgr = !fg[r] && pvalid[r];
      const bool hit = bgr && vioa[r] >= Q.ignore_thresh && ign_rule;
      int cls = fg[r] ? (int)sgc[vidx[r]] : Q.K;
      if (fg[r] && cls < 0) cls = Q.K;              // cannot happen (only valid GT compete); keeps the index sane
      if (hit || !pvalid[r]) cls = -1;
      const float miou = fmaxf(viou[r], 0.f);
      s_cls[j] = (short)cls; s_midx[j] = (short)vidx[r];
      if (Q.labels) {
        Q.matched_idx[(size_t)b * n + j] = vidx[r];
        Q.matched_iou[(size_t)b * n + j] = miou;
        Q.labels[(size_t)b * n + j] = cls;
      }
      if (cls >= 0) {
        const bool isfg = cls < Q.K;
        atomicAdd(isfg ? &c_fgc : &c_bgc, 1);
        const uint4 rb = philox4x32_10(make_uint4((uint32_t)step, (uint32_t)(step >> 32), (uint32_t)(b * kLsMaxN + j), 0x50524F50u),
                                       make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
        const float gk = gumbel_key(__fadd_rn(miou, 1e-4f), rb.x);
        // ascending sort key: group (0 fg, 1 bg) | inverted Gumbel key | candidate index
        kk = ((unsigned long long)(isfg ? 0 : 1) << 43) | ((unsigned long long)(uint32_t)(~fkey(gk)) << 11) | (unsigned)j;
      }
    }
    key[j] = ~kk;                                       // bitonic_desc on the complement == ascending on kk
  }
  __syncthreads();
  bitonic_desc(key, kLsMaxN);
  const int nfg_all = c_fgc, nbg_all = c_bgc;
  const int num_fg = min(nfg_all, Q.Fcap), num_bg = min(nbg_all, Q.S - num_fg);
  for (int s = tid; s < Q.S; s += blockDim.x) {
    int src = -1;
    if (s < num_fg) src = s;
    else if (s < num_fg + num_bg) src = nfg_all + (s - num_fg);
    const size_t o = (size_t)b * Q.S + s;
    int j = 0, cls = -1, gi = 0;
    if (src >= 0) { j = (int)((~key[src]) & 2047ull); cls = s_cls[j]; gi = s_midx[j]; }
    float4 bx = make_float4(0.f, 0.f, 0.f, 0.f);
    if (src >= 0) bx = j < P ? Q.prop_boxes[(size_t)b * P + j] : sg[j - P];
    Q.s_boxes[o] = bx;
    Q.s_valid[o] = src >= 0;
    Q.s_classes[o] = cls;
    Q.s_gt_boxes[o] = sg[gi];
    if (Q.s_index) Q.s_index[o] = src >= 0 ? j : 0;
    const float* g3 = Q.gt_boxes3D + ((size_t)b * G + gi) * 9;
    const float* gp = Q.gt_poses + ((size_t)b * G + gi) * 9;
#pragma unroll
    for (int t = 0; t < 9; ++t) { Q.s_gt_boxes3D[o * 9 + t] = g3[t]; Q.s_gt_poses[o * 9 + t] = gp[t]; }
  }
  if (tid == 0 && Q.stats) { atomicAdd(Q.stats, (float)num_fg); atomicAdd(Q.stats + 1, (float)num_bg); }
}

// ------------------------------------------------------------------------------------------------------------------
// RPN anchor sampling: Gumbel keys of the positive / negative candidates (the top-k runs on topk_segments_kernel)
__global__ void anchor_sample_keys_kernel(const signed char* __restrict__ lab, const float* __restrict__ miou, int B, long long A,
                                          const unsigned long long* __restrict__ rng, float* __restrict__ keys /*[B][2][A]*/,
                                          int* __restrict__ counts /*[B][2]*/) {
  const int b = blockIdx.y;
  const unsigned long long seed = rng ? rng[0] : 0ull, step = rng ? rng[1] : 0ull;
  int np = 0, nn = 0;
  for (long long a = (long long)blockIdx.x * blockDim.x + threadIdx.x; a < A; a += (long long)gridDim.x * blockDim.x) {
    const signed char l = lab[(size_t)b * A + a];
    const uint4 rb = philox4x32_10(make_uint4((uint32_t)step, (uint32_t)(step >> 32), (uint32_t)a, 0x414E4300u + (uint32_t)b),
                                   make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
    const float gk = gumbel_key(__fadd_rn(miou[(size_t)b * A + a], 1e-4f), rb.x);
    keys[((size_t)b * 2 + 0) * A + a] = l == 1 ? gk : -INFINITY;
    keys[((size_t)b * 2 + 1) * A + a] = l == 0 ? gk : -INFINITY;
    np += l == 1; nn += l == 0;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { np += __shfl_xor_sync(0xffffffffu, np, o); nn += __shfl_xor_sync(0xffffffffu, nn, o); }
  if ((threadIdx.x & 31) == 0) { if (np) atomicAdd(counts + b * 2, np); if (nn) atomicAdd(counts + b * 2 + 1, nn); }
}

// labels of one image: -1 everywhere, sampled negatives 0 (or -1 inside an ignore region), sampled positives and the
// best anchor of every valid GT 1 (rpn.py:62-105)
__global__ void __launch_bounds__(1024)
anchor_sample_finish_kernel(const signed char* __restrict__ lab, const float* __restrict__ ioa, const int* __restrict__ topk_idx /*[B][2][kk]*/,
                            const int* __restrict__ counts, const int* __restrict__ best_idx /*[B][G]*/,
                            const unsigned char* __restrict__ gt_valid, const unsigned char* __restrict__ gt_ign, int G, long long A,
                            int kk, int cap_pos, int n_total, float ignore_thresh, signed char* __restrict__ out,
                            unsigned long long* __restrict__ rng_bump) {
  const int b = blockIdx.x, tid = threadIdx.x;
  signed char* o = out + (size_t)b * A;
  for (long long a = tid; a < A; a += blockDim.x) o[a] = -1;
  __shared__ int any_ign;
  if (tid == 0) any_ign = 0;
  __syncthreads();
  for (int g = tid; g < G; g += blockDim.x) if (gt_ign[(size_t)b * G + g]) any_ign = 1;
  __syncthreads();
  const int num_pos = min(counts[b * 2], cap_pos);
  const int num_neg = min(counts[b * 2 + 1], n_total - num_pos);
  const bool rule = num_neg > 1 && any_ign;
  const int* ip = topk_idx + (size_t)b * 2 * kk;
  for (int j = tid; j < num_neg && j < kk; j += blockDim.x) {
    const int a = ip[kk + j];
    o[a] = (rule && ioa[(size_t)b * A + a] >= ignore_thresh) ? -1 : 0;
  }
  for (int j = tid; j < num_pos && j < kk; j += blockDim.x) o[ip[j]] = 1;
  for (int g = tid; g < G; g += blockDim.x) {
    if (!gt_valid[(size_t)b * G + g]) continue;
    const int a = best_idx[(size_t)b * G + g];
    if (a >= 0 && a < A && lab[(size_t)b * A + a] == 1) o[a] = 1;
  }
  if (rng_bump && b == 0 && tid == 0) rng_bump[1] += 1;       // next step draws fresh noise (CUDA-graph replay safe)
}

__global__ void rng_bump_kernel(unsigned long long* rng) { rng[1] += 1; }

// ------------------------------------------------------------------------------------------------------------------
// fast_rcnn_inference_single_image, steps before the NMS (cubercnn/modeling/roi_heads/fast_rcnn.py:76-100) for all images:
// drop proposals with a non-finite score or box, clip the per-class boxes to the image, keep (proposal, class) pairs with
// score > thresh.  One warp per proposal.  Candidate (p, k) lives at index p*K + k (= filter_mask.nonzero() order).
__global__ void det_candidates_kernel(const float* __restrict__ probs /*[B][P][K+1]*/, const float4* __restrict__ boxes /*[B][P][K]*/,
                                      const int* __restrict__ prop_count, const float* __restrict__ hw /*[B][2]*/, int B, int P,
                                      int K, float thresh, float* __restrict__ cand_score /*[B][P*K]*/,
                                      float4* __restrict__ cand_boxes, int* __restrict__ maxc_bits /*[B]*/, int* __restrict__ total /*[B]*/) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * P) return;
  const int b = warp / P, p = warp - b * P;
  const float* pr = probs + (size_t)warp * (K + 1);
  const float4* bx = boxes + (size_t)warp * K;
  bool ok = p < prop_count[b];
  for (int k = lane; k <= K; k += 32) ok = ok && isfinite(pr[k]);
  for (int k = lane; k < K; k += 32) { const float4 v = bx[k]; ok = ok && isfinite(v.x) && isfinite(v.y) && isfinite(v.z) && isfinite(v.w); }
  ok = __all_sync(0xffffffffu, ok);
  const float H = hw[2 * b], W = hw[2 * b + 1];
  float mx = 0.f; int cnt = 0;
  for (int k = lane; k < K; k += 32) {
    float4 v = bx[k];
    v.x = fminf(fmaxf(v.x, 0.f), W); v.y = fminf(fmaxf(v.y, 0.f), H);
    v.z = fminf(fmaxf(v.z, 0.f), W); v.w = fminf(fmaxf(v.w, 0.f), H);
    const float s = pr[k];
    const bool keep = ok && s > thresh;
    const size_t o = ((size_t)b * P + p) * K + k;
    cand_score[o] = keep ? s : -INFINITY;
    cand_boxes[o] = v;
    if (keep) { mx = fmaxf(mx, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w))); ++cnt; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); cnt += __shfl_xor_sync(0xffffffffu, cnt, o); }
  if (lane == 0 && cnt) { atomicMax(maxc_bits + b, __float_as_int(mx)); atomicAdd(total + b, cnt); }
}

}  // namespace c3d

using namespace c3d;

extern "C" int32_t c3d_topk_segments(const c3d_topk_seg* segs, int32_t nseg, int32_t B, int32_t out_stride, float* out_vals,
                                     int32_t* out_idx, int64_t* out_idx64, int32_t* out_count, void* stream) {
  if (!segs || nseg < 1 || nseg > kTopkMaxSeg || !out_vals) return set_error(C3D_EINVAL, "topk: bad args");
  if (B <= 0) return C3D_OK;
  TopkParams P;
  int kmax = 1;
  for (int s = 0; s < nseg; ++s) {
    if (!segs[s].vals || segs[s].n < 1 || segs[s].k < 1 || segs[s].k > 8192)
      return set_error(C3D_EINVAL, "topk: segment %d needs 1 <= k <= 8192 (k=%d, n=%d)", s, segs[s].k, segs[s].n);
    P.seg[s].vals = segs[s].vals; P.seg[s].row_stride = segs[s].row_stride; P.seg[s].n = segs[s].n; P.seg[s].k = segs[s].k;
    P.seg[s].out_col = segs[s].out_col;
    const int k = segs[s].k < segs[s].n ? segs[s].k : segs[s].n;
    if (k > kmax) kmax = k;
  }
  int k2 = 2;
  while (k2 < kmax) k2 <<= 1;
  P.out_stride = out_stride; P.out_vals = out_vals; P.out_idx = out_idx; P.out_idx64 = reinterpret_cast<long long*>(out_idx64);
  P.out_count = out_count; P.nseg = nseg;
  const size_t smem = (size_t)k2 * 8;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(topk_segments_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 8);
    if (e != cudaSuccess) return set_error(C3D_ECUDA, "topk smem attr: %s", cudaGetErrorString(e));
    attr = true;
  }
  dim3 grid((unsigned)B, (unsigned)nseg);
  topk_segments_kernel<<<grid, 1024, smem, static_cast<cudaStream_t>(stream)>>>(P);
  return check_launch("topk_segments");
}

extern "C" int32_t c3d_label_sample_proposals(const c3d_label_sample_args* a, void* stream) {
  if (!a || !a->prop_boxes || !a->prop_count || !a->gt_boxes || !a->gt_classes || !a->gt_present || !a->gt_boxes3D ||
      !a->gt_poses || !a->s_boxes || !a->s_valid || !a->s_classes || !a->s_gt_boxes || !a->s_gt_boxes3D || !a->s_gt_poses)
    return set_error(C3D_EINVAL, "label_sample_proposals: null pointer");
  const int n = a->P + (a->append_gt ? a->G : 0);
  if (a->B < 1 || a->G < 1 || a->G > kLsMaxG || n > kLsMaxN || a->S < 1 || a->Fcap < 0 || a->Fcap > a->S || a->K > 32000)
    return set_error(C3D_EINVAL, "label_sample_proposals: P+G=%d (max %d), G=%d (max %d)", n, kLsMaxN, a->G, kLsMaxG);
  if ((a->labels != nullptr) != (a->matched_idx != nullptr) || (a->labels != nullptr) != (a->matched_iou != nullptr))
    return set_error(C3D_EINVAL, "label_sample_proposals: pre-sampling outputs come as a triple");
  LabelSampleParams Q;
  Q.prop_boxes = reinterpret_cast<const float4*>(a->prop_boxes); Q.prop_count = a->prop_count;
  Q.gt_boxes = reinterpret_cast<const float4*>(a->gt_boxes); Q.gt_classes = reinterpret_cast<const long long*>(a->gt_classes);
  Q.gt_present = a->gt_present; Q.gt_boxes3D = a->gt_boxes3D; Q.gt_poses = a->gt_poses;
  Q.B = a->B; Q.P = a->P; Q.G = a->G; Q.K = a->K; Q.S = a->S; Q.Fcap = a->Fcap; Q.append_gt = a->append_gt;
  Q.iou_thresh = a->iou_thresh; Q.ignore_thresh = a->ignore_thresh;
  Q.rng = reinterpret_cast<const unsigned long long*>(a->rng);
  Q.matched_idx = reinterpret_cast<long long*>(a->matched_idx); Q.matched_iou = a->matched_iou;
  Q.labels = reinterpret_cast<long long*>(a->labels);
  Q.s_boxes = reinterpret_cast<float4*>(a->s_boxes); Q.s_valid = a->s_valid; Q.s_classes = reinterpret_cast<long long*>(a->s_classes);
  Q.s_gt_boxes = reinterpret_cast<float4*>(a->s_gt_boxes); Q.s_gt_boxes3D = a->s_gt_boxes3D; Q.s_gt_poses = a->s_gt_poses;
  Q.s_index = reinterpret_cast<long long*>(a->s_index); Q.stats = a->stats;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  label_sample_kernel<<<a->B, 1024, 0, st>>>(Q);
  if (a->rng && a->bump_rng) rng_bump_kernel<<<1, 1, 0, st>>>(reinterpret_cast<unsigned long long*>(const_cast<uint64_t*>(a->rng)));
  return check_launch("label_sample_proposals");
}

extern "C" int32_t c3d_anchor_sample_keys(const int8_t* labels01, const float* matched_iou, int32_t B, int64_t A,
                                          const uint64_t* rng, float* keys, int32_t* counts, void* stream) {
  if (!labels01 || !matched_iou || !keys || !counts || B < 1 || A < 1) return set_error(C3D_EINVAL, "anchor_sample_keys: bad args");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaMemsetAsync(counts, 0, sizeof(int) * 2 * B, st);
  if (e != cudaSuccess) return set_error(C3D_ECUDA, "anchor_sample_keys: %s", cudaGetErrorString(e));
  int bx = (int)((A + 255) / 256);
  if (bx > 4 * kNumSMs) bx = 4 * kNumSMs;
  anchor_sample_keys_kernel<<<dim3(bx, B), 256, 0, st>>>(reinterpret_cast<const signed char*>(labels01), matched_iou, B, A,
                                                         reinterpret_cast<const unsigned long long*>(rng), keys, counts);
  return check_launch("anchor_sample_keys");
}

extern "C" int32_t c3d_anchor_sample_finish(const int8_t* labels01, const float* max_ioa, const int32_t* topk_idx,
                                            const int32_t* counts, const int32_t* best_idx, const uint8_t* gt_valid,
                                            const uint8_t* gt_ign, int32_t B, int32_t G, int64_t A, int32_t k, int32_t cap_pos,
                                            int32_t n_total, float ignore_thresh, int8_t* out_labels, uint64_t* rng_bump,
                                            void* stream) {
  if (!labels01 || !max_ioa || !topk_idx || !counts || !best_idx || !gt_valid || !gt_ign || !out_labels || B < 1 || G < 1)
    return set_error(C3D_EINVAL, "anchor_sample_finish: bad args");
  anchor_sample_finish_kernel<<<B, 1024, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const signed char*>(labels01), max_ioa, topk_idx, counts, best_idx, gt_valid, gt_ign, G, A, k, cap_pos,
      n_total, ignore_thresh, reinterpret_cast<signed char*>(out_labels), reinterpret_cast<unsigned long long*>(rng_bump));
  return check_launch("anchor_sample_finish");
}

extern "C" int32_t c3d_det_candidates(const float* probs, const float* boxes, const int32_t* prop_count, const float* image_hw,
                                      int32_t B, int32_t P, int32_t K, float score_thresh, float* cand_score, float* cand_boxes,
                                      float* maxc, int32_t* total, void* stream) {
  if (!probs || !boxes || !prop_count || !image_hw || !cand_score || !cand_boxes || !maxc || !total || B < 1 || P < 1 || K < 1)
    return set_error(C3D_EINVAL, "det_candidates: bad args");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaError_t e = cudaMemsetAsync(maxc, 0, sizeof(float) * B, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(total, 0, sizeof(int) * B, st);
  if (e != cudaSuccess) return set_error(C3D_ECUDA, "det_candidates: %s", cudaGetErrorString(e));
  const long long threads = (long long)B * P * 32;
  det_candidates_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(probs, reinterpret_cast<const float4*>(boxes), prop_count,
                                                                        image_hw, B, P, K, score_thresh, cand_score,
                                                                        reinterpret_cast<float4*>(cand_boxes),
                                                                        reinterpret_cast<int*>(maxc), total);
  return check_launch("det_candidates");
}
