// The library's GEMM weights (the acoustic model in api.cu, the train convolutions in train.cu and the signal modules
// melgan.cu, hifigan.cu, bigvgan.cu, waveglow.cu, griffin_lim.cu, features.cu): one [taps][N][K] matrix held as fp32 rows (fp32 / tf32 math modes)
// and as power-of-two-scaled fp16 hi / lo planes (f16 / 3xF16), with an optional bias [N]; the tap-GEMM call over it, the
// one place that maps a math mode to a tap-GEMM family; and the device arena a module's weights are carved from.
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

// A convolution's GEMM rows from its folded torch-layout weight wt, element (tap j, row n, column c) at
// dst[j * tap_stride + n * row_stride + c] for j < taps, n < N, c < Cin.  u == 0: Conv1d wt [N][Cin][taps].  u >= 2:
// ConvTranspose1d wt [Cin][Cout][2u] (stride u, padding u / 2) as a polyphase matrix of taps = 3 and N = u Cout rows, row
// r Cout + co being output phase r and tap j reading input row t + j - 1 (zeros where the phase does not read it).
int conv_pack(const float* wt, int N, int Cin, int taps, int Cout, int u, long tap_stride, long row_stride, float* dst, cudaStream_t st);

// w (its N, K and buffers set) from a convolution's torch-layout tensors: conv_pack into w.w at row stride w.K, taps side
// by side along K (tap_stride = Cin, w.taps = 1) or as tap matrices (tap_stride = N K, w.taps = taps); bias [N] =
// b[n % Cout]; scale and planes.  wt2, b2 (nullable): a second 1-tap convolution of the same rows, packed in columns
// [Cin, 2 Cin) and its bias added, so that one GEMM over [x | y] computes wt . x + wt2 . y.
int vweight_pack_conv(const VWeight& w, const float* wt, const float* b, int Cin, int Cout, int taps, int u, long tap_stride, cudaStream_t st,
                      const float* wt2 = nullptr, const float* b2 = nullptr);

// dst [A'][B'][k] = src [A][B][k] zero-padded (a torch-layout convolution weight, or with B = k = 1 a bias, or with k = 1
// rows of a [rows][B] matrix; A' <= A or B' <= B crops)
int pad3(const float* src, int A, int Bn, int k, float* dst, int Ap, int Bp, cudaStream_t st);

// The TapGemm of out [B*L][w.N] = act(a [B*L][w.K] (w.taps taps at dilation dil) . w^T + w.bias) (+ resid [B*L][w.N]), a as
// fp32 rows (fp32 / tf32) or as hi (+ lo) planes (f16 / 3xF16); rows t >= lens[b] are written as 0 (and skipped by the
// tensor-core kernel).  outp (plane modes, nullable; ignored in the others): the result's operand planes as well, with the
// lo plane in 3xF16
TapGemm vweight_gemm_args(int math_mode, const VWeight& w, const void* a, int B, int L, int act, const int64_t* lens,
                          float* out, const float* resid = nullptr, int dil = 1, __half* outp = nullptr);

// runs g on the tap-GEMM family of math_mode
int tap_gemm(const TapGemm& g, int math_mode, cudaStream_t st);

// The row limits of a call whose GEMMs have up to `rows` rows: below 2^31 (int32 row indices) and, in fp32, at most
// kTapGemmFp32MaxRows.  The error reads "<who>: <formula> = <rows> <noun> rows exceed ...".
int check_rows(const char* who, const char* formula, const char* noun, long rows, int math_mode);

// tap_gemm(vweight_gemm_args(...))
int vweight_gemm(int math_mode, const VWeight& w, const void* a, int B, int L, int act, const int64_t* lens, float* out,
                 cudaStream_t st, const float* resid = nullptr, int dil = 1, __half* outp = nullptr);

// (Re)allocates *arena (*cap bytes) for what carve(Bump&) places in it.  carve returns FS2_OK or an error code; it runs on a
// counting Bump first, and an error there returns before anything is freed.  An arena already large enough is reused;
// otherwise the old one is freed once the stream has drained and a new one allocated.  carve then runs again on the arena
// to set the pointers.
template <typename Carve>
int arena_carve(void** arena, size_t* cap, cudaStream_t st, Carve carve) {
  Bump count(nullptr, 0);
  int rc = carve(count);
  if (rc) return rc;
  const size_t need = count.off + 256;
  if (need > *cap) {
    if (*arena) { FS2_CUDA_CHECK(cudaStreamSynchronize(st)); FS2_CUDA_CHECK(cudaFree(*arena)); *arena = nullptr; *cap = 0; }
    FS2_CUDA_CHECK(cudaMalloc(arena, need));
    *cap = need;
  }
  Bump b(*arena, *cap);
  return carve(b);
}

// a stream-ordered temporary for the single-layer entries: carve(Bump&) on a counting pass, then on the allocation; the
// caller releases *base with cudaFreeAsync on the same stream
template <typename Carve>
int temp_carve(void** base, cudaStream_t st, Carve carve) {
  Bump count(nullptr, 0);
  carve(count);
  FS2_CUDA_CHECK(cudaMallocAsync(base, count.off + 256, st));
  Bump b(*base, count.off + 256);
  carve(b);
  return FS2_OK;
}

}  // namespace fs2
