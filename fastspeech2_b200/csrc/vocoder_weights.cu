// The library's GEMM weights and tap-GEMM call (vocoder_weights.cuh).
#include <string.h>

#include "vocoder_weights.cuh"

namespace fs2 {
namespace {

// dst [DR][DC] = src [SR][SC] (or its transpose), zero-padded
__global__ void pad_pack_kernel(const float* __restrict__ src, int SR, int SC, int transpose, float* __restrict__ dst, int DR, int DC) {
  const long total = (long)DR * DC;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int r = (int)(i / DC), c = (int)(i % DC);
    const int sr = transpose ? c : r, sc = transpose ? r : c;
    dst[i] = sr < SR && sc < SC ? src[(long)sr * SC + sc] : 0.f;
  }
}

// Element (tap j, row n, column c) of a convolution's GEMM weight, at dst[j * tap_stride + n * row_stride + c], from the
// folded torch-layout weight:
//   u == 0  Conv1d w [N][Cin][taps]            -> w[n][c][j]
//   u >= 2  ConvTranspose1d w [Cin][Cout][2u]  -> row n = r Cout + co is output phase r, taps = 3, tap j reading input row
//           t + j - 1: w[c][co][k(r, j)] (0 where phase r does not read that row), k = r + u/2 + u (j = 0), r + u/2 (j = 1)
//           for r < u/2; r + u/2 (j = 1), r + u/2 - u (j = 2) for r >= u/2
__global__ void conv_pack_kernel(const float* __restrict__ w, int N, int Cin, int taps, int Cout, int u, long tap_stride, long row_stride,
                                 float* __restrict__ dst) {
  const long nc = (long)N * Cin, total = nc * taps;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int j = (int)(i / nc);
    const long rem = i - (long)j * nc;
    const int n = (int)(rem / Cin), c = (int)(rem - (long)n * Cin);
    float v;
    if (u == 0) {
      v = w[((long)n * Cin + c) * taps + j];
    } else {
      const int r = n / Cout, co = n - r * Cout, p = u / 2;
      const int kk = r < p ? (j == 1 ? r + p : j == 0 ? r + p + u : -1) : (j == 2 ? r + p - u : j == 1 ? r + p : -1);
      v = kk >= 0 ? w[((long)c * Cout + co) * (2 * u) + kk] : 0.f;
    }
    dst[j * tap_stride + n * row_stride + c] = v;
  }
}

// dst[n] = b[n % Cout] (+ b2[n])
__global__ void conv_bias_kernel(const float* __restrict__ b, const float* __restrict__ b2, int N, int Cout, float* __restrict__ dst) {
  for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < N; n += gridDim.x * blockDim.x) dst[n] = b2 ? b[n % Cout] + b2[n] : b[n % Cout];
}

// dst [A'][B'][k] = src [A][B][k] zero-padded (a torch-layout convolution weight, or with B = k = 1 a bias, or with
// k = 1 rows of a [rows][B] matrix; A' <= A or B' <= B crops)
__global__ void pad3_kernel(const float* __restrict__ src, int A, int Bn, int k, float* __restrict__ dst, int Ap, int Bp) {
  const long total = (long)Ap * Bp * k;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long ab = i / k;
    const int j = (int)(i - ab * k), a = (int)(ab / Bp), bb = (int)(ab - (long)a * Bp);
    dst[i] = a < A && bb < Bn ? src[((long)a * Bn + bb) * k + j] : 0.f;
  }
}

}  // namespace

void vweight_carve(Bump& b, VWeight& w, bool bias) {
  const size_t n = (size_t)w.taps * w.N * w.K;
  w.w = b.floats(n); w.hi = (__half*)b.bytes(n * 2); w.lo = (__half*)b.bytes(n * 2); w.sc = b.floats(2);
  w.bias = bias ? b.floats(w.N) : nullptr;
}

int vweight_planes(const VWeight& w, cudaStream_t st) {
  const long n = (long)w.taps * w.N * w.K;
  int rc = weight_scale(w.w, n, w.sc, w.sc + 1, st); if (rc) return rc;
  return split_f16(w.w, w.hi, w.lo, n, w.sc, st);
}

int vweight_pack(VWeight& w, const float* src, int SR, int SC, int transpose, cudaStream_t st) {
  const long n = (long)w.N * w.K;
  pad_pack_kernel<<<grid_for(n, 256), 256, 0, st>>>(src, SR, SC, transpose, w.w, w.N, w.K);
  FS2_LAUNCH_CHECK();
  return vweight_planes(w, st);
}

int conv_pack(const float* wt, int N, int Cin, int taps, int Cout, int u, long tap_stride, long row_stride, float* dst, cudaStream_t st) {
  conv_pack_kernel<<<grid_for((long)taps * N * Cin, 256), 256, 0, st>>>(wt, N, Cin, taps, Cout, u, tap_stride, row_stride, dst);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int vweight_pack_conv(const VWeight& w, const float* wt, const float* b, int Cin, int Cout, int taps, int u, long tap_stride, cudaStream_t st,
                      const float* wt2, const float* b2) {
  int rc = conv_pack(wt, w.N, Cin, taps, Cout, u, tap_stride, w.K, w.w, st);
  if (!rc && wt2) rc = conv_pack(wt2, w.N, Cin, taps, Cout, u, tap_stride, w.K, w.w + Cin, st);
  if (rc) return rc;
  conv_bias_kernel<<<grid_for(w.N, 256), 256, 0, st>>>(b, b2, w.N, Cout, w.bias);
  FS2_LAUNCH_CHECK();
  return vweight_planes(w, st);
}

int pad3(const float* src, int A, int Bn, int k, float* dst, int Ap, int Bp, cudaStream_t st) {
  pad3_kernel<<<grid_for((long)Ap * Bp * k, 256), 256, 0, st>>>(src, A, Bn, k, dst, Ap, Bp);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

TapGemm vweight_gemm_args(int math_mode, const VWeight& w, const void* a, int B, int L, int act, const int64_t* lens,
                          float* out, const float* resid, int dil, __half* outp) {
  TapGemm g;
  memset(&g, 0, sizeof(g));
  g.B = B; g.L = L; g.K = w.K; g.N = w.N; g.taps = w.taps; g.dil = dil; g.act = act; g.out = out; g.ldo = w.N; g.lens = lens;
  g.w = w.w; g.bias = w.bias; g.resid = resid; g.ldr = w.N; g.a_inv = 1.0f; g.ldx = w.K;
  if (math_mode == FS2_MATH_FP32 || math_mode == FS2_MATH_TF32) {
    g.x = (const float*)a;
    return g;
  }
  g.xp = (const __half*)a; g.w_hi = w.hi; g.w_lo = w.lo; g.w_inv = w.sc + 1; g.a_inv = kPlaneInv;
  g.precise = math_mode == FS2_MATH_3XTF32;
  if (outp) { g.outp = outp; g.ldo_p = w.N; g.outp_lo = g.precise; }
  return g;
}

int tap_gemm(const TapGemm& g, int math_mode, cudaStream_t st) {
  if (math_mode == FS2_MATH_FP32) return tap_gemm_fp32(g, st);
  if (math_mode == FS2_MATH_TF32) return tap_gemm_tf32(g, st);
  return tap_gemm_planes(g, st);
}

int check_rows(const char* who, const char* formula, const char* noun, long rows, int math_mode) {
  FS2_REQUIRE(rows < (1L << 31), "%s: %s = %ld %s rows exceed the int32 row index", who, formula, rows, noun);
  FS2_REQUIRE(math_mode != FS2_MATH_FP32 || rows <= kTapGemmFp32MaxRows, "%s: %s = %ld %s rows exceed fp32 mode's limit of %ld", who,
              formula, rows, noun, kTapGemmFp32MaxRows);
  return FS2_OK;
}

int vweight_gemm(int math_mode, const VWeight& w, const void* a, int B, int L, int act, const int64_t* lens, float* out,
                 cudaStream_t st, const float* resid, int dil, __half* outp) {
  return tap_gemm(vweight_gemm_args(math_mode, w, a, B, L, act, lens, out, resid, dil, outp), math_mode, st);
}

}  // namespace fs2
