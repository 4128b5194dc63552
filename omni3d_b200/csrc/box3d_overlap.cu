// box3d_overlap.cu — oriented-box 3D IoU for H100 (sm_90a).  Compile with -fmad=false.
//
// Replaces pytorch3d._C.iou_box3d (cubercnn/evaluation/omni3d_evaluation.py:155) and the
// reference wrapper box3d_overlap (omni3d_evaluation.py:106-166).
//
// Design (not the one-thread-per-pair layout of the stock CUDA op):
//   prep kernel   one thread per box: 256-byte record (corners, 6 inward face planes, centre,
//                 volume) + a padded bounding sphere + the dt-row validity flags.
//   filter kernel one thread per 4 consecutive pairs: bounding-sphere test (+ dt-row validity); disjoint
//                 spheres => exactly vol=iou=0, 0 faces, written with 16-byte stores at HBM rate; the
//                 surviving pair indices are appended to a queue (one atomic per warp).  Paired mode fuses
//                 prep + filter: the raw corners are staged through shared memory with coalesced loads
//                 and a rejected pair costs 192 B in + 4..12 B out, nothing else.
//   clip kernel   persistent warps walk the survivor queue with a static stride, ONE PAIR PER WARP (so
//                 1 000 live pairs already occupy 1 000 warps): lanes 0-15 clip box1's triangles by
//                 box2's planes while lanes 16-31 clip box2's triangles by box1's planes, triangle
//                 lists live in shared memory (SoA, conflict-free), compaction by ballot/popc keeps
//                 the serial order, so face counts, vol and iou are bit-identical to the serial CPU
//                 algorithm.
//   overflow      pairs whose intermediate list exceeds the shared-memory capacity (P≈1e-5 on
//                 random dense boxes) are queued and redone by a small kernel with
//                 global-memory lists.
// No tensor cores (byte/ALU work); HBM traffic = 96 B per box + 4..12 B per pair.
#include "box3d_geom.cuh"
#include "c3d_common.cuh"

namespace c3d {

constexpr int kCap = 64;           // triangles per side in shared memory
constexpr int kCapBig = 256;       // per side in the global-memory fallback
constexpr int kWarpsPerBlock = 4;
constexpr int kSidePad = 16;        // the second box's record / triangle buffers start 16 banks later: lanes 16-31 never hit lanes 0-15's banks
constexpr int kRecSmem = 128 + kSidePad;
__host__ __device__ constexpr int kBufSmem(int cap) { return 4 * 9 * cap + kSidePad; }
constexpr int kFallbackWarps = 296;
constexpr unsigned kFull = 0xffffffffu;
constexpr long long kMaxOverflowQueue = 1ll << 22;

struct Ctrl {            // lives at the head of the workspace (zeroed by a memset node at the start of a call)
  unsigned int n_live;     // survivors of the current batch (filter kernel appends, clip kernel reads)
  unsigned int n_overflow;
  int n_bad[2];
  unsigned int next_overflow;
  unsigned int pad[3];
};
constexpr long long kBatchPairs = 1ll << 24;   // pairs per filter/clip round (bounds the survivor queue: 64 MB of u32)

// ------------------------------------------------------------------------------------------
__global__ void iou3d_prep_kernel(const float* __restrict__ b1, int n1, const float* __restrict__ b2,
                                  int n2, float* __restrict__ rec, float4* __restrict__ sph,
                                  uint8_t* __restrict__ rowflags, float eps_c, float eps_nz,
                                  int do_check) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n1 + n2) return;
  const float* src = i < n1 ? b1 + 24 * (size_t)i : b2 + 24 * (size_t)(i - n1);
  float r[kRecFloats];
  float s4[4];
  build_box_record(src, r, s4);
  float4* dst = reinterpret_cast<float4*>(rec + (size_t)i * kRecFloats);
#pragma unroll
  for (int k = 0; k < kRecFloats / 4; ++k) dst[k] = make_float4(r[4 * k], r[4 * k + 1], r[4 * k + 2], r[4 * k + 3]);
  sph[i] = make_float4(s4[0], s4[1], s4[2], s4[3]);
  if (i < n1 && rowflags) {
    int f = do_check ? check_box(src, eps_c, eps_nz) : 3;
    rowflags[i] = (uint8_t)f;
  }
}

// Paired mode (pair k = boxes1[k] x boxes2[k]): every box belongs to exactly one pair, so building the 256-byte record of a
// box whose pair is rejected by the bounding-sphere test is wasted work and wasted HBM traffic — in the sparse regime that
// is ~all of them.  Fused prep + filter, one thread per PAIR: the block's 128 + 128 boxes are staged through shared memory
// with coalesced 16-byte loads (rows padded to 25 words: conflict-free per-thread reads), both spheres come from the raw
// corners, rejected pairs get their zeros here; only surviving pairs get records + a queue entry.
// Traffic per rejected pair: 192 B in + 4..12 B out.
constexpr int kPairedBlock = 128;
constexpr int kRowPad = 25;
__global__ void __launch_bounds__(kPairedBlock)
iou3d_prep_paired_kernel(const float* __restrict__ b1, const float* __restrict__ b2, long long k0, int nbatch, int n,
                         float* __restrict__ rec, float4* __restrict__ sph, float* __restrict__ vol,
                         float* __restrict__ iou, int* __restrict__ nfaces, unsigned* __restrict__ queue, Ctrl* ctrl) {
  __shared__ float sbox[2][kPairedBlock * kRowPad];
  const int tid = threadIdx.x;
  const long long kb = k0 + (long long)blockIdx.x * kPairedBlock;        // first pair of the block
  const int nblk = (int)min((long long)kPairedBlock, k0 + nbatch - kb);
  const float* g[2] = {b1 + 24 * kb, b2 + 24 * kb};
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    if ((reinterpret_cast<uintptr_t>(g[s]) & 15) == 0) {
      const float4* g4 = reinterpret_cast<const float4*>(g[s]);
      for (int q = tid; q < nblk * 6; q += kPairedBlock) {
        const float4 v = __ldg(g4 + q);
        const int row = q / 6, col = (q - row * 6) * 4;
        float* d = &sbox[s][row * kRowPad + col];
        d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
      }
    } else {
      for (int q = tid; q < nblk * 24; q += kPairedBlock) {
        const int row = q / 24;
        sbox[s][row * kRowPad + (q - row * 24)] = __ldg(g[s] + q);
      }
    }
  }
  __syncthreads();
  bool live = false;
  const long long k = kb + tid;
  if (tid < nblk) {
    const float* s1 = &sbox[0][tid * kRowPad];
    const float* s2 = &sbox[1][tid * kRowPad];
    float c1[4], c2[4];
    box_sphere(s1, c1);
    box_sphere(s2, c2);
    const float dx = c1[0] - c2[0], dy = c1[1] - c2[1], dz = c1[2] - c2[2];
    const float rs = c1[3] + c2[3];
    live = (dx * dx + dy * dy + dz * dz) <= rs * rs;
    if (!live) {
      iou[k] = 0.f;
      if (vol) vol[k] = 0.f;
      if (nfaces) nfaces[k] = 0;
    } else {
      float r[kRecFloats];
      float s4[4];
      build_box_record(s1, r, s4);
      float4* dst = reinterpret_cast<float4*>(rec + (size_t)k * kRecFloats);
#pragma unroll
      for (int q = 0; q < kRecFloats / 4; ++q) dst[q] = make_float4(r[4 * q], r[4 * q + 1], r[4 * q + 2], r[4 * q + 3]);
      build_box_record(s2, r, s4);
      dst = reinterpret_cast<float4*>(rec + (size_t)(n + k) * kRecFloats);
#pragma unroll
      for (int q = 0; q < kRecFloats / 4; ++q) dst[q] = make_float4(r[4 * q], r[4 * q + 1], r[4 * q + 2], r[4 * q + 3]);
    }
  }
  const unsigned m = __ballot_sync(kFull, live);
  if (m) {
    const int lane = tid & 31;
    unsigned base = 0;
    if (lane == 0) base = atomicAdd(&ctrl->n_live, (unsigned)__popc(m));
    base = __shfl_sync(kFull, base, 0);
    if (live) queue[base + __popc(m & ((1u << lane) - 1u))] = (unsigned)(k - k0);
  }
}

__global__ void iou3d_count_bad_kernel(const uint8_t* __restrict__ rowflags, int n1, Ctrl* ctrl,
                                       int* __restrict__ n_bad_out) {
  // single block; tiny
  __shared__ int s[2];
  if (threadIdx.x == 0) { s[0] = 0; s[1] = 0; }
  __syncthreads();
  int c0 = 0, c1 = 0;
  for (int i = threadIdx.x; i < n1; i += blockDim.x) {
    int f = rowflags[i];
    c0 += !(f & 1); c1 += !(f & 2);
  }
  atomicAdd(&s[0], c0); atomicAdd(&s[1], c1);
  __syncthreads();
  if (threadIdx.x == 0) {
    ctrl->n_bad[0] = s[0]; ctrl->n_bad[1] = s[1];
    if (n_bad_out) { n_bad_out[0] = s[0]; n_bad_out[1] = s[1]; }
  }
}

// ------------------------------------------------------------------------------------------
// One pair per warp.  `rec` = 2x64 floats (both box records, shared memory), `buf` = 4 triangle
// buffers of 9*CAP floats each laid out [side][pingpong][comp][slot].  Returns (on every lane)
// nf >= 0 and vol/iou, or nf = -1 on capacity overflow.
template <int CAP>
__device__ __forceinline__ int process_pair(const float* __restrict__ recA, const float* __restrict__ recB,
                                            float* rec, float* buf, int lane, float* vol_o, float* iou_o) {
  const int side = lane >> 4, hl = lane & 15;
  // 1. records -> shared
  constexpr int RB = 64 + kSidePad;          // second record
  constexpr int SB = 2 * 9 * CAP + kSidePad;  // second side's ping-pong buffers
  rec[lane] = recA[lane]; rec[lane + 32] = recA[lane + 32];
  rec[RB + lane] = recB[lane]; rec[RB + lane + 32] = recB[lane + 32];
  __syncwarp();
  const float* rT = rec + RB * side;        // box whose triangles this half clips
  const float* rP = rec + RB * (1 - side);  // box whose planes clip them
  float* sb = buf + (size_t)side * SB;
  int cur = 0;
  // 2. the 12 box triangles
  if (hl < 12) {
    float* d = sb;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      int v = tri_vert(hl, k);
      d[(3 * k + 0) * CAP + hl] = rT[3 * v + 0];
      d[(3 * k + 1) * CAP + hl] = rT[3 * v + 1];
      d[(3 * k + 2) * CAP + hl] = rT[3 * v + 2];
    }
  }
  int n = 12;
  __syncwarp();
  // 3. six clipping planes
  bool ovf = false;
  for (int p = 0; p < 6; ++p) {
    const float* pl = rP + 24 + 6 * p;
    V3 pc = mk(pl[0], pl[1], pl[2]), nn = mk(pl[3], pl[4], pl[5]);
    V3 q[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      int v = plane_vert(p, k);
      q[k] = mk(rP[3 * v], rP[3 * v + 1], rP[3 * v + 2]);
    }
    const float* src = sb + cur * 9 * CAP;
    float* dst = sb + (cur ^ 1) * 9 * CAP;
    int nother = __shfl_xor_sync(kFull, n, 16);
    int nmax = max(n, nother);
    int m = 0;
    for (int base = 0; base < nmax; base += 16) {
      int t = base + hl;
      int k = 0;
      Tri o0, o1;
      if (t < n) {
        Tri tr;
        tr.a = mk(src[0 * CAP + t], src[1 * CAP + t], src[2 * CAP + t]);
        tr.b = mk(src[3 * CAP + t], src[4 * CAP + t], src[5 * CAP + t]);
        tr.c = mk(src[6 * CAP + t], src[7 * CAP + t], src[8 * CAP + t]);
        k = clip_tri(tr, pc, nn, q, &o0, &o1);
      }
      unsigned b1 = (__ballot_sync(kFull, k >= 1) >> (16 * side)) & 0xffffu;
      unsigned b2 = (__ballot_sync(kFull, k == 2) >> (16 * side)) & 0xffffu;
      unsigned lower = (1u << hl) - 1u;
      int off = m + __popc(b1 & lower) + __popc(b2 & lower);
      int tot = __popc(b1) + __popc(b2);
      bool o = (m + tot > CAP);
      if (__any_sync(kFull, o)) { ovf = true; break; }
      if (k >= 1) {
        dst[0 * CAP + off] = o0.a.x; dst[1 * CAP + off] = o0.a.y; dst[2 * CAP + off] = o0.a.z;
        dst[3 * CAP + off] = o0.b.x; dst[4 * CAP + off] = o0.b.y; dst[5 * CAP + off] = o0.b.z;
        dst[6 * CAP + off] = o0.c.x; dst[7 * CAP + off] = o0.c.y; dst[8 * CAP + off] = o0.c.z;
      }
      if (k == 2) {
        int f = off + 1;
        dst[0 * CAP + f] = o1.a.x; dst[1 * CAP + f] = o1.a.y; dst[2 * CAP + f] = o1.a.z;
        dst[3 * CAP + f] = o1.b.x; dst[4 * CAP + f] = o1.b.y; dst[5 * CAP + f] = o1.b.z;
        dst[6 * CAP + f] = o1.c.x; dst[7 * CAP + f] = o1.c.y; dst[8 * CAP + f] = o1.c.z;
      }
      m += tot;
    }
    if (ovf) break;
    n = m; cur ^= 1;
    __syncwarp();
    nother = __shfl_xor_sync(kFull, n, 16);
    if (n == 0 && nother == 0) break;   // warp-uniform
  }
  if (ovf) { *vol_o = 0.f; *iou_o = 0.f; return -1; }
  const int n1 = __shfl_sync(kFull, n, 0), n2 = __shfl_sync(kFull, n, 16);
  if (n1 + n2 == 0) { *vol_o = 0.f; *iou_o = 0.f; return 0; }

  // 4. de-dup: drop box2-side triangles coplanar with a (non-degenerate) box1-side triangle
  const float* L1 = buf + cur * 9 * CAP;                   // final box1-side list
  const float* L2 = buf + SB + cur * 9 * CAP;              // final box2-side list
  float* F1 = buf + (cur ^ 1) * 9 * CAP;                   // scratch (free ping-pong halves)
  float* F2 = buf + SB + (cur ^ 1) * 9 * CAP;
  auto load_tri = [&](const float* L, int t) {
    Tri tr;
    tr.a = mk(L[0 * CAP + t], L[1 * CAP + t], L[2 * CAP + t]);
    tr.b = mk(L[3 * CAP + t], L[4 * CAP + t], L[5 * CAP + t]);
    tr.c = mk(L[6 * CAP + t], L[7 * CAP + t], L[8 * CAP + t]);
    return tr;
  };
  for (int idx = lane; idx < n1 + n2; idx += 32) {
    bool s0 = idx < n1;
    int t = s0 ? idx : idx - n1;
    Tri tr = load_tri(s0 ? L1 : L2, t);
    V3 nr = tri_normal(tr);
    float* F = s0 ? F1 : F2;
    F[0 * CAP + t] = nr.x; F[1 * CAP + t] = nr.y; F[2 * CAP + t] = nr.z;
    if (s0) F[3 * CAP + t] = tri_area(tr);
  }
  __syncwarp();
  int* fin2 = reinterpret_cast<int*>(F2 + 3 * CAP);        // final index of each box2-side tri or -1
  float* cx = F1 + 4 * CAP; float* cy = F1 + 6 * CAP;      // final-order arrays, 2*CAP each
  float* cz = F2 + 4 * CAP; float* vt = F2 + 6 * CAP;
  int nf = n1;
  for (int base = 0; base < n2; base += 32) {
    int b = base + lane;
    bool keep = false;
    if (b < n2) {
      keep = true;
      Tri t2 = load_tri(L2, b);
      V3 nb = mk(F2[0 * CAP + b], F2[1 * CAP + b], F2[2 * CAP + b]);
      for (int a = 0; a < n1; ++a) {
        V3 na = mk(F1[0 * CAP + a], F1[1 * CAP + a], F1[2 * CAP + a]);
        if (fabsf(dot(na, nb)) > 1.0f - dEps) {      // cheap half of the test first (same result)
          if (F1[3 * CAP + a] > aEps && coplanar_tri_tri(load_tri(L1, a), na, t2, nb)) { keep = false; break; }
        }
      }
    }
    unsigned kb = __ballot_sync(kFull, keep);
    if (b < n2) fin2[b] = keep ? nf + __popc(kb & ((1u << lane) - 1u)) : -1;
    nf += __popc(kb);
  }
  __syncwarp();
  // 5. centroids in final order, then the serial (bit-exact) sums
  for (int idx = lane; idx < n1 + n2; idx += 32) {
    bool s0 = idx < n1;
    int t = s0 ? idx : idx - n1;
    int f = s0 ? t : fin2[t];
    if (f >= 0) {
      Tri tr = load_tri(s0 ? L1 : L2, t);
      cx[f] = (tr.a.x + tr.b.x + tr.c.x) / 3.0f;
      cy[f] = (tr.a.y + tr.b.y + tr.c.y) / 3.0f;
      cz[f] = (tr.a.z + tr.b.z + tr.c.z) / 3.0f;
    }
  }
  __syncwarp();
  float acc = 0.0f;
  if (lane < 3) {
    const float* arr = lane == 0 ? cx : (lane == 1 ? cy : cz);
    for (int f = 0; f < nf; ++f) acc += arr[f];
    acc = acc / nf;
  }
  V3 pc = mk(__shfl_sync(kFull, acc, 0), __shfl_sync(kFull, acc, 1), __shfl_sync(kFull, acc, 2));
  for (int idx = lane; idx < n1 + n2; idx += 32) {
    bool s0 = idx < n1;
    int t = s0 ? idx : idx - n1;
    int f = s0 ? t : fin2[t];
    if (f >= 0) vt[f] = tet_volume(load_tri(s0 ? L1 : L2, t), pc);
  }
  __syncwarp();
  float vol = 0.0f, iou = 0.0f;
  if (lane == 0) {
    for (int f = 0; f < nf; ++f) vol = vol + vt[f];
    iou = vol / (rec[63] + rec[RB + 63] - vol);
  }
  *vol_o = __shfl_sync(kFull, vol, 0);
  *iou_o = __shfl_sync(kFull, iou, 0);
  __syncwarp();
  return nf;
}

struct PairArgs {
  const float* rec;        // (n1+n2) x 64
  const float4* sph;       // (n1+n2)
  const uint8_t* rowflags; // n1 or null (null => all rows valid)
  long long npairs;
  int n1, n2;              // paired mode: n2 == 0
  float* vol; float* iou; int* nfaces;
  Ctrl* ctrl;
  unsigned long long* overflow;   // queue of pair indices
  unsigned overflow_cap;
  // segmented (CSR) mode: `ngroups` independent (dt group x gt group) blocks in one launch — Omni3Deval.computeIoU's
  // one call per (image, category) (omni3d_evaluation.py:1339-1343,1401-1412).  pair k belongs to group g with
  // pair_off[g] <= k < pair_off[g+1]; inside it row-major over (dt_off[g+1]-dt_off[g]) x (gt_off[g+1]-gt_off[g]).
  const long long* pair_off; const int* dt_off; const int* gt_off; int ngroups;
};

__device__ __forceinline__ void pair_to_ij(const PairArgs& A, long long k, int* i, int* j) {
  if (A.ngroups > 0) {
    int lo = 0, hi = A.ngroups;                              // last g with pair_off[g] <= k
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (__ldg(A.pair_off + mid) <= k) lo = mid; else hi = mid; }
    const int d0 = __ldg(A.dt_off + lo), g0 = __ldg(A.gt_off + lo), ng = __ldg(A.gt_off + lo + 1) - g0;
    const long long r = k - __ldg(A.pair_off + lo);
    *i = d0 + (int)(r / ng); *j = A.n1 + g0 + (int)(r % ng);
    return;
  }
  if (A.n2 == 0) { *i = (int)k; *j = (int)k + A.n1; }      // paired: box2 records follow box1's
  else { *i = (int)(k / A.n2); *j = A.n1 + (int)(k % A.n2); }
}

// Sphere test (+ dt-row validity) of the pairs [k0, k0 + nbatch): 4 consecutive pairs per thread, zeros written with one
// 16-byte store per output array (the arrays are 16-byte aligned and k0 is a multiple of 4 whenever `vec` is set),
// survivors appended to the queue as offsets from k0 (one atomic per warp).
__global__ void __launch_bounds__(256)
iou3d_filter_kernel(PairArgs A, long long k0, int nbatch, unsigned* __restrict__ queue, int vec) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long kq = k0 + 4 * t;
  const int cnt = (int)max(0ll, min(4ll, k0 + nbatch - kq));
  unsigned livemask = 0;
  if (cnt > 0) {
    int i = 0, j = 0;
    pair_to_ij(A, kq, &i, &j);
    float4 s1 = __ldg(A.sph + i);
    bool rowok = A.rowflags ? (A.rowflags[i] == 3) : true;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (u < cnt) {
        if (u > 0) {
          if (A.ngroups > 0) {
            const int pi = i;
            pair_to_ij(A, kq + u, &i, &j);
            if (i != pi) { s1 = __ldg(A.sph + i); rowok = A.rowflags ? (A.rowflags[i] == 3) : true; }
          } else if (A.n2 == 0) {                           // paired records: (k, n1 + k)
            ++i; ++j; s1 = __ldg(A.sph + i); rowok = A.rowflags ? (A.rowflags[i] == 3) : true;
          } else {
            ++j;                                            // cross mode, row-major (n2 >= 1)
            if (j == A.n1 + A.n2) { j = A.n1; ++i; s1 = __ldg(A.sph + i); rowok = A.rowflags ? (A.rowflags[i] == 3) : true; }
          }
        }
        const float4 s2 = __ldg(A.sph + j);
        const float dx = s1.x - s2.x, dy = s1.y - s2.y, dz = s1.z - s2.z;
        const float rs = s1.w + s2.w;
        if (((dx * dx + dy * dy + dz * dz) <= rs * rs) && rowok) livemask |= 1u << u;
      }
    }
    if (vec && cnt == 4) {
      *reinterpret_cast<float4*>(A.iou + kq) = make_float4(0.f, 0.f, 0.f, 0.f);
      if (A.vol) *reinterpret_cast<float4*>(A.vol + kq) = make_float4(0.f, 0.f, 0.f, 0.f);
      if (A.nfaces) *reinterpret_cast<int4*>(A.nfaces + kq) = make_int4(0, 0, 0, 0);
    } else {
      for (int u = 0; u < cnt; ++u) {
        A.iou[kq + u] = 0.f;
        if (A.vol) A.vol[kq + u] = 0.f;
        if (A.nfaces) A.nfaces[kq + u] = 0;
      }
    }
  }
  // queue append: exclusive warp scan of the per-thread survivor counts
  const int lane = threadIdx.x & 31;
  const int mine = __popc(livemask);
  int incl = mine;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int v = __shfl_up_sync(kFull, incl, d);
    if (lane >= d) incl += v;
  }
  const int total = __shfl_sync(kFull, incl, 31);
  if (total == 0) return;
  unsigned base = 0;
  if (lane == 31) base = atomicAdd(&A.ctrl->n_live, (unsigned)total);
  base = __shfl_sync(kFull, base, 31);
  unsigned pos = base + (unsigned)(incl - mine);
  const unsigned rel = (unsigned)(kq - k0);
#pragma unroll
  for (int u = 0; u < 4; ++u)
    if (livemask & (1u << u)) queue[pos++] = rel + u;
}

// Survivor queue -> one pair per warp, static stride over the queue (no atomics; the per-pair work varies ~3x, the
// queue order is effectively random, so the tail is a few per cent once every warp holds tens of pairs).
__global__ void __launch_bounds__(32 * kWarpsPerBlock)
iou3d_clip_kernel(PairArgs A, long long k0, const unsigned* __restrict__ queue) {
  extern __shared__ __align__(16) float smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* rec = smem + warp * (kRecSmem + kBufSmem(kCap));
  float* buf = rec + kRecSmem;
  const unsigned n_live = A.ctrl->n_live;
  const unsigned W = gridDim.x * kWarpsPerBlock;
  for (unsigned q = warp * gridDim.x + blockIdx.x; q < n_live; q += W) {
    const long long k = k0 + (long long)__ldg(queue + q);
    int i, j;
    pair_to_ij(A, k, &i, &j);
    float v, u;
    int nf = process_pair<kCap>(A.rec + (size_t)i * kRecFloats, A.rec + (size_t)j * kRecFloats, rec, buf, lane, &v, &u);
    if (lane == 0) {
      if (nf < 0) {
        unsigned slot = atomicAdd(&A.ctrl->n_overflow, 1u);
        if (slot < A.overflow_cap) A.overflow[slot] = (unsigned long long)k;
        else { v = __int_as_float(0x7fc00000); u = v; }   // queue full: flagged NaN / nfaces -1
      }
      A.iou[k] = u;
      if (A.vol) A.vol[k] = v;
      if (A.nfaces) A.nfaces[k] = nf;
    }
  }
}

// rare path: same routine, triangle lists in global memory (one slab per warp)
__global__ void __launch_bounds__(32)
iou3d_overflow_kernel(PairArgs A, float* slabs) {
  __shared__ float rec[kRecSmem];
  const int lane = threadIdx.x;
  float* buf = slabs + (size_t)blockIdx.x * kBufSmem(kCapBig);
  const unsigned n = min(A.ctrl->n_overflow, A.overflow_cap);
  while (true) {
    unsigned q = 0;
    if (lane == 0) q = atomicAdd(&A.ctrl->next_overflow, 1u);
    q = __shfl_sync(kFull, q, 0);
    if (q >= n) break;
    long long k = (long long)A.overflow[q];
    int i, j;
    pair_to_ij(A, k, &i, &j);
    float v, u;
    int nf = process_pair<kCapBig>(A.rec + (size_t)i * kRecFloats, A.rec + (size_t)j * kRecFloats, rec,
                                   buf, lane, &v, &u);
    if (lane == 0) {
      if (nf < 0) { v = __int_as_float(0x7fc00000); u = v; }
      A.iou[k] = u;
      if (A.vol) A.vol[k] = v;
      if (A.nfaces) A.nfaces[k] = nf;
    }
    __syncwarp();
  }
}

// ---- workspace layout -------------------------------------------------------------------------
struct WsLayout {
  size_t ctrl, rec, sph, flags, overflow, slabs, queue, total;
};
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
static WsLayout ws_layout_pairs(int64_t n1, int64_t n2, int64_t npairs);
static WsLayout ws_layout(int64_t n1, int64_t n2) {
  return ws_layout_pairs(n1, n2 == 0 ? n1 : n2, n2 == 0 ? n1 : n1 * n2);
}
static WsLayout ws_layout_pairs(int64_t n1, int64_t m2, int64_t npairs) {
  WsLayout L;
  int64_t nb = n1 + m2;
  size_t o = 0;
  L.ctrl = o; o = align_up(o + sizeof(Ctrl), 256);
  L.rec = o; o = align_up(o + (size_t)nb * kRecFloats * 4, 256);
  L.sph = o; o = align_up(o + (size_t)nb * 16, 256);
  L.flags = o; o = align_up(o + (size_t)n1, 256);
  L.overflow = o; o = align_up(o + (size_t)(npairs < kMaxOverflowQueue ? npairs : kMaxOverflowQueue) * 8, 256);
  L.slabs = o; o = align_up(o + (size_t)kFallbackWarps * kBufSmem(kCapBig) * 4, 256);
  L.queue = o; o = align_up(o + (size_t)(npairs < kBatchPairs ? npairs : kBatchPairs) * 4, 256);
  L.total = o;
  return L;
}

struct SegInfo { const int64_t* pair_off; const int32_t* dt_off; const int32_t* gt_off; int32_t ngroups; int64_t total_pairs; };

static int32_t run_iou(const float* b1, int64_t n1, const float* b2, int64_t n2, bool paired,
                       bool do_check, float eps_c, float eps_nz, float* vol, float* iou, int32_t* nfaces,
                       int32_t* n_bad, void* ws, size_t ws_bytes, cudaStream_t st, const SegInfo* seg = nullptr) {
  if (n1 < 0 || n2 < 0) return set_error(C3D_EINVAL, "negative box count");
  int64_t m2 = paired ? n1 : n2;
  int64_t npairs = seg ? seg->total_pairs : (paired ? n1 : n1 * n2);
  if (n1 + m2 > (int64_t)INT32_MAX / 2 || npairs > ((int64_t)1 << 36))
    return set_error(C3D_EINVAL, "problem too large (%lld x %lld)", (long long)n1, (long long)m2);
  if (npairs == 0 && !(do_check && n1 > 0)) {
    if (n_bad) cudaMemsetAsync(n_bad, 0, 2 * sizeof(int32_t), st);
    return check_launch("iou3d memset");
  }
  if (!b1 || (!b2 && !paired && n2 > 0) || (!iou && npairs > 0) || !ws)
    return set_error(C3D_EINVAL, "null pointer");
  WsLayout L = seg ? ws_layout_pairs(n1, n2, npairs) : ws_layout(n1, paired ? 0 : n2);
  if (ws_bytes < L.total)
    return set_error(C3D_EWORKSPACE, "workspace %zu < required %zu", ws_bytes, L.total);
  if ((reinterpret_cast<uintptr_t>(ws) & 255) != 0) return set_error(C3D_EINVAL, "workspace must be 256-byte aligned");
  char* w = static_cast<char*>(ws);
  Ctrl* ctrl = reinterpret_cast<Ctrl*>(w + L.ctrl);
  float* rec = reinterpret_cast<float*>(w + L.rec);
  float4* sph = reinterpret_cast<float4*>(w + L.sph);
  uint8_t* flags = reinterpret_cast<uint8_t*>(w + L.flags);
  int nb = (int)(n1 + m2);
  unsigned* queue = reinterpret_cast<unsigned*>(w + L.queue);
  cudaMemsetAsync(ctrl, 0, sizeof(Ctrl), st);
  const bool fused_paired = paired && !do_check && !seg;
  if (!fused_paired)
    iou3d_prep_kernel<<<(nb + 127) / 128, 128, 0, st>>>(b1, (int)n1, b2, (int)m2, rec, sph, flags, eps_c,
                                                        eps_nz, do_check ? 1 : 0);
  if (do_check) iou3d_count_bad_kernel<<<1, 256, 0, st>>>(flags, (int)n1, ctrl, n_bad);
  if (npairs > 0) {
    PairArgs A;
    A.rec = rec; A.sph = sph; A.rowflags = do_check ? flags : nullptr;
    A.npairs = npairs; A.n1 = (int)n1; A.n2 = paired ? 0 : (int)n2;
    A.vol = vol; A.iou = iou; A.nfaces = nfaces; A.ctrl = ctrl;
    A.overflow = reinterpret_cast<unsigned long long*>(w + L.overflow);
    A.overflow_cap = (unsigned)(npairs < kMaxOverflowQueue ? npairs : kMaxOverflowQueue);
    A.pair_off = nullptr; A.dt_off = nullptr; A.gt_off = nullptr; A.ngroups = 0;
    if (seg) {
      A.pair_off = reinterpret_cast<const long long*>(seg->pair_off); A.dt_off = seg->dt_off; A.gt_off = seg->gt_off;
      A.ngroups = seg->ngroups;
    }
    size_t smem = (size_t)kWarpsPerBlock * (kRecSmem + kBufSmem(kCap)) * sizeof(float);
    static bool attr_set = false;
    if (!attr_set) {
      cudaFuncSetAttribute(iou3d_clip_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      attr_set = true;
    }
    int blocks_per_sm = (int)((227 * 1024) / (smem + 1024));
    if (blocks_per_sm > 8) blocks_per_sm = 8;
    const long long maxgrid = (long long)kNumSMs * blocks_per_sm;
    const int vec = ((reinterpret_cast<uintptr_t>(iou) | reinterpret_cast<uintptr_t>(vol) |
                      reinterpret_cast<uintptr_t>(nfaces)) & 15) == 0;
    for (long long k0 = 0; k0 < npairs; k0 += kBatchPairs) {
      const int nbatch = (int)(npairs - k0 < kBatchPairs ? npairs - k0 : kBatchPairs);
      if (k0 > 0) cudaMemsetAsync(&ctrl->n_live, 0, sizeof(unsigned), st);
      if (fused_paired)
        iou3d_prep_paired_kernel<<<(nbatch + kPairedBlock - 1) / kPairedBlock, kPairedBlock, 0, st>>>(
            b1, b2, k0, nbatch, (int)n1, rec, sph, vol, iou, nfaces, queue, ctrl);
      else
        iou3d_filter_kernel<<<(unsigned)(((nbatch + 3) / 4 + 255) / 256), 256, 0, st>>>(A, k0, nbatch, queue, vec);
      long long grid = ((long long)nbatch + kWarpsPerBlock - 1) / kWarpsPerBlock;   // one pair per warp at most
      if (grid > maxgrid) grid = maxgrid;
      iou3d_clip_kernel<<<(unsigned)grid, 32 * kWarpsPerBlock, smem, st>>>(A, k0, queue);
    }
    iou3d_overflow_kernel<<<kFallbackWarps, 32, 0, st>>>(A, reinterpret_cast<float*>(w + L.slabs));
  }
  return check_launch("iou3d launch");
}

}  // namespace c3d

extern "C" size_t c3d_iou_box3d_workspace_bytes(int64_t n1, int64_t n2) {
  if (n1 < 0 || n2 < 0) return 0;
  return c3d::ws_layout(n1, n2).total;
}
extern "C" int32_t c3d_iou_box3d(const float* boxes1, int64_t n1, const float* boxes2, int64_t n2,
                                 float* vol, float* iou, int32_t* nfaces, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  if (n2 == 0 || n1 == 0) return C3D_OK;   // empty output
  return c3d::run_iou(boxes1, n1, boxes2, n2, false, false, 0.f, 0.f, vol, iou, nfaces, nullptr, workspace,
                      workspace_bytes, static_cast<cudaStream_t>(stream));
}
extern "C" int32_t c3d_iou_box3d_paired(const float* boxes1, const float* boxes2, int64_t n, float* vol,
                                        float* iou, int32_t* nfaces, void* workspace,
                                        size_t workspace_bytes, void* stream) {
  if (n == 0) return C3D_OK;
  return c3d::run_iou(boxes1, n, boxes2, 0, true, false, 0.f, 0.f, vol, iou, nfaces, nullptr, workspace,
                      workspace_bytes, static_cast<cudaStream_t>(stream));
}
extern "C" int32_t c3d_box3d_overlap(const float* boxes_dt, int64_t n_dt, const float* boxes_gt,
                                     int64_t n_gt, float eps_coplanar, float eps_nonzero, float* iou,
                                     int32_t* n_bad, void* workspace, size_t workspace_bytes, void* stream) {
  if (n_dt == 0) {
    if (n_bad) cudaMemsetAsync(n_bad, 0, 2 * sizeof(int32_t), static_cast<cudaStream_t>(stream));
    return C3D_OK;
  }
  return c3d::run_iou(boxes_dt, n_dt, boxes_gt, n_gt, false, true, eps_coplanar, eps_nonzero, nullptr, iou,
                      nullptr, n_bad, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

extern "C" size_t c3d_box3d_overlap_segmented_workspace_bytes(int64_t n_dt, int64_t n_gt, int64_t total_pairs) {
  if (n_dt < 0 || n_gt < 0 || total_pairs < 0) return 0;
  return c3d::ws_layout_pairs(n_dt, n_gt, total_pairs).total;
}
extern "C" int32_t c3d_box3d_overlap_segmented(const float* boxes_dt, int64_t n_dt, const float* boxes_gt, int64_t n_gt,
                                               const int32_t* dt_off, const int32_t* gt_off, const int64_t* pair_off,
                                               int32_t num_groups, int64_t total_pairs, float eps_coplanar,
                                               float eps_nonzero, float* iou, int32_t* n_bad, void* workspace,
                                               size_t workspace_bytes, void* stream) {
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (num_groups < 0 || total_pairs < 0) return c3d::set_error(C3D_EINVAL, "segmented overlap: negative sizes");
  if (n_dt == 0 || num_groups == 0) {
    if (n_bad) cudaMemsetAsync(n_bad, 0, 2 * sizeof(int32_t), st);
    return C3D_OK;
  }
  if (!dt_off || !gt_off || !pair_off) return c3d::set_error(C3D_EINVAL, "segmented overlap: null offsets");
  c3d::SegInfo seg{pair_off, dt_off, gt_off, num_groups, total_pairs};
  return c3d::run_iou(boxes_dt, n_dt, boxes_gt, n_gt, false, true, eps_coplanar, eps_nonzero, nullptr, iou, nullptr, n_bad,
                      workspace, workspace_bytes, st, &seg);
}
