// augment_ops.cu — device side of the input pipeline (SURVEY 8f-3): the image part of DatasetMapper3D
// (cubercnn/data/dataset_mapper.py:22-35: read_image -> T.AugInput -> ResizeShortestEdge + RandomFlip -> CHW uint8 tensor).
//
// detectron2's ResizeTransform resizes uint8 images with Pillow (Image.resize(..., BILINEAR)): a separable triangle filter
// whose support grows with the down-scale factor, evaluated in 22-bit fixed point with a uint8 intermediate image between
// the horizontal and the vertical pass.  The coefficients are computed on the host exactly like Pillow's
// precompute_coeffs / normalize_coeffs_8bpc (omni3d_b200/data.py); these kernels apply them — integer arithmetic only, so
// the result is BIT-IDENTICAL to Pillow's (tests compare against Pillow itself).  The horizontal flip of RandomFlip and the
// HWC -> CHW transposition of dataset_mapper.py:35 are folded into the second pass.  Byte work, HBM / L2 bound: no tensor cores.
#include <stdint.h>
#include "c3d_common.cuh"

namespace c3d {

// resample along one axis: out[o][i][c] = clip8((2^21 + sum_x src[o][lo_i + x][c] * kk[i][x]) >> 22)
//   src / dst are addressed through element strides (axis, other, channel), so the same kernel does the horizontal pass
//   (HWC -> HWC), the vertical pass (HWC -> CHW) and mirrors the OTHER axis when asked to (horizontal flip in pass 2).
__global__ void resample_u8_kernel(const uint8_t* __restrict__ src, long long s_a, long long s_o, long long s_c,
                                   uint8_t* __restrict__ dst, long long d_a, long long d_o, long long d_c, int n_out,
                                   int other_lo, int other_hi, int n_other, int C, const int* __restrict__ bounds,
                                   const int* __restrict__ kk, int ksize, int mirror_other) {
  const long long total = (long long)(other_hi - other_lo) * n_out * C;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(t % C);
    long long r = t / C;
    const int i = (int)(r % n_out);
    const int o = other_lo + (int)(r / n_out);
    const int lo = bounds[2 * i], n = bounds[2 * i + 1];
    const int* k = kk + (size_t)i * ksize;
    const uint8_t* p = src + (long long)o * s_o + (long long)lo * s_a + (long long)c * s_c;
    int acc = 1 << 21;
    for (int x = 0; x < n; ++x) acc += (int)p[(long long)x * s_a] * k[x];
    acc >>= 22;
    acc = acc < 0 ? 0 : (acc > 255 ? 255 : acc);
    const int oo = mirror_other ? (n_other - 1 - o) : o;
    dst[(long long)oo * d_o + (long long)i * d_a + (long long)c * d_c] = (uint8_t)acc;
  }
}

}  // namespace c3d

using namespace c3d;

extern "C" int32_t c3d_resize_bilinear_u8(const uint8_t* img_hwc, int32_t H, int32_t W, int32_t C, const int32_t* bounds_h,
                                          const int32_t* kk_h, int32_t ksize_h, const int32_t* bounds_v, const int32_t* kk_v,
                                          int32_t ksize_v, int32_t new_h, int32_t new_w, int32_t row_first, int32_t row_last,
                                          int32_t flip, uint8_t* tmp_hwc, uint8_t* out_chw, void* stream) {
  if (!img_hwc || !bounds_h || !kk_h || !bounds_v || !kk_v || !tmp_hwc || !out_chw || H < 1 || W < 1 || C < 1 || new_h < 1 ||
      new_w < 1 || ksize_h < 1 || ksize_v < 1 || row_first < 0 || row_last > H || row_first >= row_last)
    return set_error(C3D_EINVAL, "resize_bilinear_u8: bad args");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  auto blocks = [](long long n) { long long b = (n + 255) / 256; return (unsigned)(b > kNumSMs * 16 ? kNumSMs * 16 : (b < 1 ? 1 : b)); };
  // pass 1 (horizontal): img (H,W,C) -> tmp (H,new_w,C), only the rows the vertical pass reads
  resample_u8_kernel<<<blocks((long long)(row_last - row_first) * new_w * C), 256, 0, st>>>(
      img_hwc, C, (long long)W * C, 1, tmp_hwc, C, (long long)new_w * C, 1, new_w, row_first, row_last, H, C, bounds_h, kk_h,
      ksize_h, 0);
  // pass 2 (vertical): tmp (H,new_w,C) -> out (C,new_h,new_w); other axis = x, mirrored for the horizontal flip
  resample_u8_kernel<<<blocks((long long)new_w * new_h * C), 256, 0, st>>>(
      tmp_hwc, (long long)new_w * C, C, 1, out_chw, new_w, 1, (long long)new_h * new_w, new_h, 0, new_w, new_w, C, bounds_v,
      kk_v, ksize_v, flip ? 1 : 0);
  return check_launch("resize_bilinear_u8");
}
