// GEMM weights of the spectral transforms (griffin_lim.cu, features.cu): one [N][K] matrix held as fp32 rows (fp32 / tf32
// math modes) and as power-of-two-scaled fp16 hi / lo planes (f16 / 3xF16), and the tap-GEMM call over it.
#pragma once
#include "operand_planes.cuh"

namespace fs2 {

struct VWeight {               // w: N * K floats; hi, lo: N * K halfs each; sc = [scale, 1 / scale]
  float* w = nullptr; __half* hi = nullptr; __half* lo = nullptr; float* sc = nullptr;
  int N = 0, K = 0;
};

// fill w's buffers from src [SR][SC] (its transpose when `transpose`), zero-padded to [N][K]: fp32 rows, scale, planes
int vweight_pack(VWeight& w, const float* src, int SR, int SC, int transpose, cudaStream_t st);

// out [B*L][w.N] = act(a [B*L][w.K] . w^T), a as fp32 rows (fp32 / tf32) or as hi (+ lo) planes (f16 / 3xF16); rows
// t >= lens[b] are written as 0 (and skipped by the tensor-core kernel)
int vweight_gemm(int math_mode, const VWeight& w, const void* a, int B, int L, int act, const int64_t* lens, float* out,
                 cudaStream_t st);

}  // namespace fs2
