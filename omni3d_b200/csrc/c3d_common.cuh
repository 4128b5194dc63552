// c3d_common.cuh — error plumbing shared by the C-ABI translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdio.h>
#include "../../include/c3d.h"

namespace c3d {
char* last_error_buf();          // thread-local, 512 bytes
int32_t set_error(int32_t code, const char* fmt, ...);
inline int32_t check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(C3D_ECUDA, "%s: %s", what, cudaGetErrorString(e));
  return C3D_OK;
}
constexpr int kNumSMs = 132;     // H100 SXM
}  // namespace c3d
