// GEMM weights of the signal modules (melgan.cu, waveglow.cu, griffin_lim.cu, features.cu): one [taps][N][K] matrix held
// as fp32 rows (fp32 / tf32 math modes) and as power-of-two-scaled fp16 hi / lo planes (f16 / 3xF16), with an optional
// bias [N]; the tap-GEMM call over it; and the device arena a module's weights are carved from.
#pragma once
#include "operand_planes.cuh"

namespace fs2 {

struct VWeight {               // w: taps * N * K floats; hi, lo: as many halfs each; sc = [scale, 1 / scale]; bias: N floats or null
  float* w = nullptr; __half* hi = nullptr; __half* lo = nullptr; float* sc = nullptr; float* bias = nullptr;
  int N = 0, K = 0, taps = 1;
};

// w's buffers for its taps, N and K, in the order w, hi, lo, sc (, bias [N] when `bias`)
void vweight_carve(Bump& b, VWeight& w, bool bias);

// the power-of-two scale and the fp16 planes of w, from its fp32 rows w.w
int vweight_planes(const VWeight& w, cudaStream_t st);

// fill w's buffers from src [SR][SC] (its transpose when `transpose`), zero-padded to [N][K]: fp32 rows, scale, planes
int vweight_pack(VWeight& w, const float* src, int SR, int SC, int transpose, cudaStream_t st);

// out [B*L][w.N] = act(a [B*L][w.K] (w.taps taps at dilation dil) . w^T + w.bias) (+ resid [B*L][w.N]), a as fp32 rows
// (fp32 / tf32) or as hi (+ lo) planes (f16 / 3xF16); rows t >= lens[b] are written as 0 (and skipped by the tensor-core
// kernel).  outp (plane modes, nullable): the result's operand planes as well, with the lo plane in 3xF16
int vweight_gemm(int math_mode, const VWeight& w, const void* a, int B, int L, int act, const int64_t* lens, float* out,
                 cudaStream_t st, const float* resid = nullptr, int dil = 1, __half* outp = nullptr);

// (Re)allocates *arena for what carve(Bump&) places in it: carve runs on a counting Bump, the old arena is freed once the
// stream has drained, and carve runs again on the new arena to set the pointers
template <typename Carve>
int arena_carve(void** arena, cudaStream_t st, Carve carve) {
  Bump count(nullptr, 0);
  carve(count);
  if (*arena) { FS2_CUDA_CHECK(cudaStreamSynchronize(st)); FS2_CUDA_CHECK(cudaFree(*arena)); *arena = nullptr; }
  FS2_CUDA_CHECK(cudaMalloc(arena, count.off + 256));
  Bump b(*arena, (size_t)-1);
  carve(b);
  return FS2_OK;
}

}  // namespace fs2
