// nms.cu — batched greedy NMS for all images of a batch in two launches, fully on the device.
//
// Replaces torchvision.ops.nms (reached through detectron2 batched_nms in find_top_rpn_proposals,
// SURVEY.md A.3; configs/Base.yaml:51-54) whose CUDA path copies the suppression mask to the host and
// scans it there (one host sync per image).  Boxes arrive sorted by score (descending) per image and
// already shifted by the per-level "coordinate trick" offsets, so IoU > thr (same fp32 formula as
// torchvision's devIoU) reproduces its keep list exactly.
//   kernel 1: 64x64 tiles of the upper-triangular suppression bit matrix (one uint64 per row/tile);
//   kernel 2: one warp per image walks the rows in score order keeping the live "removed" bitset in
//             registers (4 words per lane, up to 8192 candidates), writes the first `max_keep` survivors.
#include <stdlib.h>
#include "c3d_common.cuh"

namespace c3d {

__device__ __forceinline__ bool iou_gt(const float4 a, const float4 b, float thr) {
  float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z);
  float top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
  float width = fmaxf(right - left, 0.f), height = fmaxf(bottom - top, 0.f);
  float inter = width * height;
  float sa = (a.z - a.x) * (a.w - a.y);
  float sb = (b.z - b.x) * (b.w - b.y);
  return (inter / (sa + sb - inter)) > thr;
}

__device__ __forceinline__ float4 shift(float4 b, float off) {
  return make_float4(b.x + off, b.y + off, b.z + off, b.w + off);
}

// cats (may be null): per-box category as float; maxc: per-image max coordinate.  Images with
// 4*nvalid <= trick_max_numel use torchvision's coordinate trick (boxes shifted by cat*(maxc+1)), larger
// ones plain per-category suppression — exactly torchvision.ops.batched_nms's two code paths.
__global__ void nms_mask_kernel(const float4* __restrict__ boxes, const int* __restrict__ nvalid, int n, int words,
                                float thr, const float* __restrict__ cats, const float* __restrict__ maxc,
                                int trick_max_numel, unsigned long long* __restrict__ mask) {
  const int b = blockIdx.z, row_blk = blockIdx.y, col_blk = blockIdx.x;
  if (col_blk < row_blk) return;
  const int nv = nvalid[b];
  const int row0 = row_blk * 64, col0 = col_blk * 64;
  if (row0 >= nv || col0 >= nv) return;
  __shared__ float4 cb[64];
  __shared__ float cc[64];
  const int t = threadIdx.x;
  const float4* bx = boxes + (size_t)b * n;
  const float* cx = cats ? cats + (size_t)b * n : nullptr;
  const bool trick = cx && (4 * nv <= trick_max_numel);
  const float scale = trick ? (maxc[b] + 1.0f) : 0.f;
  if (col0 + t < nv) {
    float c = cx ? cx[col0 + t] : 0.f;
    cc[t] = c;
    cb[t] = trick ? shift(bx[col0 + t], c * scale) : bx[col0 + t];
  }
  __syncthreads();
  const int i = row0 + t;
  if (i < nv) {
    const float myc = cx ? cx[i] : 0.f;
    const float4 me = trick ? shift(bx[i], myc * scale) : bx[i];
    unsigned long long bits = 0;
    const int ncol = min(64, nv - col0);
    const int start = (row_blk == col_blk) ? t + 1 : 0;
    for (int j = start; j < ncol; ++j)
      // different categories never suppress each other: per-category mode by definition, coordinate-trick mode because
      // the shifted boxes are disjoint (IoU 0 <= thr) — skip the IoU arithmetic for ~(levels-1)/levels of the pairs
      if (cc[j] == myc && iou_gt(me, cb[j], thr)) bits |= 1ULL << j;
    mask[((size_t)b * n + i) * words + col_blk] = bits;
  }
}

// Greedy scan of one score-ordered list of m rows by ONE warp, 64 rows at a time: the chunk's own keeps are resolved from
// its diagonal mask word alone (64 register-only steps: one shuffle each), then the kept rows' remaining words are OR-ed
// into the live "removed" bitset (word w on lane w % 32, slot w / 32) with independent, pipelined loads — instead of one
// dependent global load per kept row (a 1000-keep scan was ~0.7 ms of pure L2 latency).  Returns the keep mask of every
// chunk through `emit(chunk, keepbits)`; stops after max_keep keeps.  rows: mask + row*words, only words >= row/64 valid.
template <typename Emit>
__device__ __forceinline__ int nms_scan_chunks(const unsigned long long* __restrict__ rows, int m, int words, int max_keep,
                                               int lane, Emit emit) {
  unsigned long long r0 = 0, r1 = 0, r2 = 0, r3 = 0;
  const int wc = (m + 63) >> 6;
  int cnt = 0;
  for (int c = 0; c < wc && cnt < max_keep; ++c) {
    const int base = c << 6, nrows = min(64, m - base);
    const unsigned long long d0 = lane < nrows ? rows[(size_t)(base + lane) * words + c] : 0ull;
    const unsigned long long d1 = lane + 32 < nrows ? rows[(size_t)(base + lane + 32) * words + c] : 0ull;
    const int slot = c >> 5, owner = c & 31;
    unsigned long long cur = slot == 0 ? r0 : (slot == 1 ? r1 : (slot == 2 ? r2 : r3));
    cur = __shfl_sync(0xffffffffu, cur, owner);
    unsigned long long keep = 0ull;
    int room = max_keep - cnt;
    for (int i = 0; i < nrows && room > 0; ++i) {
      const unsigned long long di = __shfl_sync(0xffffffffu, i < 32 ? d0 : d1, i & 31);
      if (!((cur >> i) & 1ull)) { keep |= 1ull << i; cur |= di; --room; }
    }
    emit(c, keep);
    cnt += __popcll(keep);
    // OR the kept rows' later words into the live bitset.  The rows are independent of each other: the loads of kUn kept rows
    // are issued before any of them is consumed (one kept row at a time was one L2 round trip per kept row — 1000 keeps x
    // ~600 cycles per kept row)
    constexpr int kUn = 8;
    const bool w0 = lane > c && lane < wc, w1 = lane + 32 > c && lane + 32 < wc, w2 = lane + 64 > c && lane + 64 < wc,
               w3 = lane + 96 > c && lane + 96 < wc;
    unsigned long long k = keep;
    while (k) {
      unsigned long long t0[kUn], t1[kUn], t2[kUn], t3[kUn];
#pragma unroll
      for (int u = 0; u < kUn; ++u) {
        t0[u] = t1[u] = t2[u] = t3[u] = 0ull;
        if (k) {
          const int i = __ffsll((long long)k) - 1;
          k &= k - 1;
          const unsigned long long* row = rows + (size_t)(base + i) * words;
          if (w0) t0[u] = row[lane];
          if (w1) t1[u] = row[lane + 32];
          if (w2) t2[u] = row[lane + 64];
          if (w3) t3[u] = row[lane + 96];
        }
      }
#pragma unroll
      for (int u = 0; u < kUn; ++u) { r0 |= t0[u]; r1 |= t1[u]; r2 |= t2[u]; r3 |= t3[u]; }
    }
  }
  return cnt;
}

__global__ void nms_scan_kernel(const unsigned long long* __restrict__ mask, const int* __restrict__ nvalid, int n,
                                int words, int max_keep, int* __restrict__ keep_idx, int* __restrict__ keep_cnt) {
  const int b = blockIdx.x, lane = threadIdx.x;
  const int nv = nvalid[b];
  int* out = keep_idx + (size_t)b * max_keep;
  int written = 0;
  const int cnt = nms_scan_chunks(mask + (size_t)b * n * words, nv, words, max_keep, lane, [&](int c, unsigned long long keep) {
    // survivors of this chunk, in order: lane l owns rows l and l + 32
    const unsigned lo = (unsigned)keep, hi = (unsigned)(keep >> 32);
    if ((lo >> lane) & 1u) out[written + __popc(lo & ((1u << lane) - 1u))] = (c << 6) + lane;
    if ((hi >> lane) & 1u) out[written + __popc(lo) + __popc(hi & ((1u << lane) - 1u))] = (c << 6) + 32 + lane;
    written += __popcll(keep);
  });
  for (int k = cnt + lane; k < max_keep; k += 32) out[k] = -1;
  if (lane == 0) keep_cnt[b] = cnt;
}

// ------------------------------------------------------------------------------------------------------------
// Grouped variant: boxes of different categories never suppress each other, so the candidates of an image are first
// split (stably, i.e. still in score order) into their categories and every category is solved on its own:
//   G  one block per image: per-category counts, offsets and the permutation (category-major, score order inside)
//   M  64x64 suppression tiles inside each category only   (5 levels x 2000 boxes: 3.4x fewer pairs than 8300^2 / 2)
//   S  one warp per (image, category) greedy scan           (5x more warps, each over <= 2000 instead of 8300 rows)
//   C  one warp per image: survivors back in global score order, first max_keep
// Results are identical to the single-list kernels above (same IoU arithmetic, same coordinate-trick shifts).
constexpr int kMaxCat = 16;

__global__ void __launch_bounds__(32 * kMaxCat)
nms_group_kernel(const float* __restrict__ cats, const int* __restrict__ nvalid, int n, int ncat, int* __restrict__ perm,
                 int* __restrict__ cat_off /*[B][kMaxCat+1]*/, unsigned char* __restrict__ keepflag) {
  const int b = blockIdx.x, c = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nv = nvalid[b];
  const float* cx = cats + (size_t)b * n;
  __shared__ int cnt[kMaxCat + 1];
  for (int i = threadIdx.x; i < nv; i += blockDim.x) keepflag[(size_t)b * n + i] = 0;
  int mine = 0;
  if (c < ncat)
    for (int i0 = 0; i0 < nv; i0 += 32) {
      const int i = i0 + lane;
      const bool f = i < nv && (int)cx[i] == c;
      mine += __popc(__ballot_sync(0xffffffffu, f));
    }
  if (lane == 0) cnt[c] = c < ncat ? mine : 0;
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int k = 0; k < kMaxCat; ++k) { const int v = cnt[k]; cnt[k] = acc; acc += v; }
    cnt[kMaxCat] = acc;
  }
  __syncthreads();
  if (threadIdx.x <= kMaxCat) cat_off[(size_t)b * (kMaxCat + 1) + threadIdx.x] = cnt[threadIdx.x];
  if (c < ncat) {
    int base = cnt[c];
    for (int i0 = 0; i0 < nv; i0 += 32) {
      const int i = i0 + lane;
      const bool f = i < nv && (int)cx[i] == c;
      const unsigned m = __ballot_sync(0xffffffffu, f);
      if (f) perm[(size_t)b * n + base + __popc(m & ((1u << lane) - 1u))] = i;
      base += __popc(m);
    }
  }
}

__global__ void nms_mask_grouped_kernel(const float4* __restrict__ boxes, const int* __restrict__ nvalid, int n, int words,
                                        float thr, const float* __restrict__ maxc, int trick_max_numel,
                                        const int* __restrict__ perm, const int* __restrict__ cat_off, int ncat,
                                        unsigned long long* __restrict__ mask) {
  const int b = blockIdx.z / ncat, c = blockIdx.z % ncat;
  const int off = cat_off[(size_t)b * (kMaxCat + 1) + c], m = cat_off[(size_t)b * (kMaxCat + 1) + c + 1] - off;
  if (m <= 0) return;
  const int nv = nvalid[b];
  const bool trick = 4 * nv <= trick_max_numel;
  const float sh = trick ? (float)c * (maxc[b] + 1.0f) : 0.f;
  const float4* bx = boxes + (size_t)b * n;
  const int* pm = perm + (size_t)b * n + off;
  const int tiles = (m + 63) / 64;
  __shared__ float4 cb[64];
  const int t = threadIdx.x;
  for (int row_blk = blockIdx.y; row_blk < tiles; row_blk += gridDim.y)
    for (int col_blk = blockIdx.x; col_blk < tiles; col_blk += gridDim.x) {
      if (col_blk < row_blk) continue;
      const int row0 = row_blk * 64, col0 = col_blk * 64;
      __syncthreads();
      if (col0 + t < m) cb[t] = trick ? shift(bx[pm[col0 + t]], sh) : bx[pm[col0 + t]];
      __syncthreads();
      const int i = row0 + t;
      if (i < m) {
        const float4 me = trick ? shift(bx[pm[i]], sh) : bx[pm[i]];
        unsigned long long bits = 0;
        const int ncol = min(64, m - col0);
        const int start = (row_blk == col_blk) ? t + 1 : 0;
        for (int j = start; j < ncol; ++j)
          if (iou_gt(me, cb[j], thr)) bits |= 1ULL << j;
        mask[((size_t)b * n + off + i) * words + col_blk] = bits;
      }
    }
}

__global__ void nms_scan_grouped_kernel(const unsigned long long* __restrict__ mask, int n, int words, int max_keep,
                                        const int* __restrict__ perm, const int* __restrict__ cat_off, int ncat,
                                        unsigned char* __restrict__ keepflag) {
  const int b = blockIdx.x / ncat, c = blockIdx.x % ncat, lane = threadIdx.x;
  const int off = cat_off[(size_t)b * (kMaxCat + 1) + c], m = cat_off[(size_t)b * (kMaxCat + 1) + c + 1] - off;
  if (m <= 0) return;
  const int* pm = perm + (size_t)b * n + off;
  unsigned char* kf = keepflag + (size_t)b * n;
  nms_scan_chunks(mask + ((size_t)b * n + off) * words, m, words, max_keep, lane, [&](int c, unsigned long long keep) {
    if ((keep >> lane) & 1ull) kf[pm[(c << 6) + lane]] = 1;
    if ((keep >> (lane + 32)) & 1ull) kf[pm[(c << 6) + 32 + lane]] = 1;
  });
}

__global__ void nms_compact_kernel(const unsigned char* __restrict__ keepflag, const int* __restrict__ nvalid, int n,
                                   int max_keep, int* __restrict__ keep_idx, int* __restrict__ keep_cnt) {
  const int b = blockIdx.x, lane = threadIdx.x;
  const int nv = nvalid[b];
  int* out = keep_idx + (size_t)b * max_keep;
  int cnt = 0;
  for (int i0 = 0; i0 < nv && cnt < max_keep; i0 += 32) {
    const int i = i0 + lane;
    const bool f = i < nv && keepflag[(size_t)b * n + i];
    const unsigned mk = __ballot_sync(0xffffffffu, f);
    const int pos = cnt + __popc(mk & ((1u << lane) - 1u));
    if (f && pos < max_keep) out[pos] = i;
    cnt += __popc(mk);
  }
  if (cnt > max_keep) cnt = max_keep;
  for (int k = cnt + lane; k < max_keep; k += 32) out[k] = -1;
  if (lane == 0) keep_cnt[b] = cnt;
}

}  // namespace c3d

extern "C" size_t c3d_nms_workspace_bytes(int32_t B, int32_t n) {
  if (B < 0 || n < 0) return 0;
  size_t words = (size_t)(n + 63) / 64;
  // suppression bit matrix + (grouped path) permutation, keep flags and per-category offsets
  return (size_t)B * n * words * 8 + 256 + (size_t)B * n * 4 + (size_t)B * n + (size_t)B * (c3d::kMaxCat + 1) * 4 + 256;
}

static int32_t nms_impl(const float* boxes, const int32_t* nvalid, const float* cats, const float* maxc,
                        int32_t trick_max_numel, int32_t B, int32_t n, float iou_thresh, int32_t max_keep,
                        int32_t* keep_idx, int32_t* keep_cnt, void* workspace, size_t workspace_bytes, void* stream,
                        int ncat, int max_per_cat) {
  using namespace c3d;
  if (B == 0 || n == 0) return C3D_OK;
  if (!boxes || !nvalid || !keep_idx || !keep_cnt || !workspace) return set_error(C3D_EINVAL, "nms: null pointer");
  if (n > 8192) return set_error(C3D_EINVAL, "nms: at most 8192 candidates per image (got %d)", n);
  if (workspace_bytes < c3d_nms_workspace_bytes(B, n)) return set_error(C3D_EWORKSPACE, "nms: workspace too small");
  const int words = (n + 63) / 64;
  cudaStream_t st = (cudaStream_t)stream;
  // rows whose diagonal tile is skipped (beyond nvalid) are never read; no memset needed because the scan
  // only reads words >= i/64 of rows i < nvalid, all of which kernel 1 writes when col0 < nvalid.
  if (cats && !maxc) return set_error(C3D_EINVAL, "nms: cats given without maxc");
  if (cats && ncat > 0 && ncat <= kMaxCat) {
    // workspace: [mask][perm int32 B*n][cat_off int32 B*(kMaxCat+1)][keepflag u8 B*n]
    uint8_t* base = (uint8_t*)workspace + (((size_t)B * n * words * 8 + 255) & ~(size_t)255);
    int* perm = (int*)base;
    int* cat_off = perm + (size_t)B * n;
    unsigned char* keepflag = (unsigned char*)(cat_off + (size_t)B * (kMaxCat + 1));
    nms_group_kernel<<<B, 32 * kMaxCat, 0, st>>>(cats, nvalid, n, ncat, perm, cat_off, keepflag);
    int tiles = ((max_per_cat > 0 ? (max_per_cat < n ? max_per_cat : n) : n) + 63) / 64;
    if (tiles > 64) tiles = 64;                          // the kernel strides over further tiles if a category is larger
    dim3 gm(tiles, tiles, B * ncat);
    nms_mask_grouped_kernel<<<gm, 64, 0, st>>>((const float4*)boxes, nvalid, n, words, iou_thresh, maxc, trick_max_numel,
                                               perm, cat_off, ncat, (unsigned long long*)workspace);
    nms_scan_grouped_kernel<<<B * ncat, 32, 0, st>>>((const unsigned long long*)workspace, n, words, max_keep, perm,
                                                     cat_off, ncat, keepflag);
    nms_compact_kernel<<<B, 32, 0, st>>>(keepflag, nvalid, n, max_keep, keep_idx, keep_cnt);
    return check_launch("nms_batched (grouped)");
  }
  dim3 grid(words, words, B);
  nms_mask_kernel<<<grid, 64, 0, st>>>((const float4*)boxes, nvalid, n, words, iou_thresh, cats, maxc,
                                       trick_max_numel, (unsigned long long*)workspace);
  nms_scan_kernel<<<B, 32, 0, st>>>((const unsigned long long*)workspace, nvalid, n, words, max_keep, keep_idx,
                                    keep_cnt);
  return check_launch("nms_batched");
}

extern "C" int32_t c3d_nms_batched(const float* boxes, const int32_t* nvalid, const float* cats, const float* maxc,
                                   int32_t trick_max_numel, int32_t B, int32_t n, float iou_thresh,
                                   int32_t max_keep, int32_t* keep_idx, int32_t* keep_cnt, void* workspace,
                                   size_t workspace_bytes, void* stream) {
  return nms_impl(boxes, nvalid, cats, maxc, trick_max_numel, B, n, iou_thresh, max_keep, keep_idx, keep_cnt, workspace,
                  workspace_bytes, stream, 0, 0);
}
extern "C" int32_t c3d_nms_batched_grouped(const float* boxes, const int32_t* nvalid, const float* cats, const float* maxc,
                                           int32_t trick_max_numel, int32_t B, int32_t n, float iou_thresh,
                                           int32_t max_keep, int32_t ncat, int32_t max_per_cat_hint, int32_t* keep_idx,
                                           int32_t* keep_cnt, void* workspace, size_t workspace_bytes, void* stream) {
  if (!cats) return c3d::set_error(C3D_EINVAL, "nms grouped: cats missing");
  if (ncat < 1 || ncat > c3d::kMaxCat) return c3d::set_error(C3D_EINVAL, "nms grouped: ncat=%d outside [1, %d]", ncat, c3d::kMaxCat);
  return nms_impl(boxes, nvalid, cats, maxc, trick_max_numel, B, n, iou_thresh, max_keep, keep_idx, keep_cnt, workspace,
                  workspace_bytes, stream, ncat, max_per_cat_hint);
}
