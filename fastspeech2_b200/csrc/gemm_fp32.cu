// fp32 "tap GEMM": every Linear / Conv1d of the path as one shared-memory-staged kernel.
//
//   out[b,t,n] = act( sum_{j<taps} sum_{k<K} x[b, t+(j-pad)*dil, k] * w[j][n][k] + bias[n] ) (+ resid[b,t,n])
//
// Replaces nn.Linear (attention.py:48-50,74; encoder.py:119; fastspeech.py:153) and nn.Conv1d
// (modules.py:225-234, duration_predictor.py:48-55, variance_predictor.py:24-33,
// modules.py:283-348) of the reference.  Activations are [B, time, channel] with channels
// innermost, so a k-tap convolution is `taps` GEMMs that read the same matrix at shifted rows;
// rows outside [0, L) of the *same utterance* are zero ("same" padding at tensor edges only --
// padded time steps inside the rectangle are real inputs, SURVEY.md section 8a row a7; in per-utterance mode,
// TapGemm::lens, the epilogue writes them as zeros instead, so the next convolution's padding is the utterance's own).
//
// This is the exact-fp32 family (FMA on CUDA cores): used for the encoder and the predictors
// in every mode (their outputs feed round()/bucketize(), where tf32 noise would flip integers)
// and for the whole path in FS2_MATH_FP32.  Roofline: FP32 FMA pipe (compute bound, AI >> ridge).
//
// Tiling: CTA 128x128 outputs, BK=16, 256 threads, 8x8 register tile per thread (two 4-wide
// groups 64 apart in both directions so the LDS.128 reads are conflict free), operands staged
// transposed in shared memory ([k][m] / [k][n]) with register double buffering of the next
// global tile.  Global loads are 16-byte vectors along k (coalesced 64-byte runs per row).
#include "common.cuh"

namespace fs2 {
namespace {

constexpr int BM = 128, BN = 128, BK = 16, PADM = 4;
constexpr int NTHREADS = 256;

template <int ACT, bool HAS_RES>
__global__ void __launch_bounds__(NTHREADS, 2)
tap_gemm_fp32_kernel(TapGemm g) {
  __shared__ __align__(16) float As[2][BK][BM + PADM];
  __shared__ __align__(16) float Bs[2][BK][BN + PADM];

  const int tid = threadIdx.x;
  const int M = g.B * g.L;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int pad = (g.taps - 1) / 2, dil = g.dil > 1 ? g.dil : 1;

  // loader mapping: 4 threads cover one 16-float row chunk; rows lr and lr+64
  const int lr = tid >> 2, lk = (tid & 3) * 4;
  int a_t[2]; long a_base[2]; bool a_ok[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    int m = m0 + lr + 64 * i;
    a_ok[i] = m < M;
    int b = a_ok[i] ? m / g.L : 0;
    a_t[i] = a_ok[i] ? m - b * g.L : 0;
    a_base[i] = (long)b * g.L;
  }
  bool b_ok[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) b_ok[i] = (n0 + lr + 64 * i) < g.N;

  const int kchunks = g.K / BK;
  const int steps = g.taps * kchunks;

  float4 ra[2], rb[2];
  auto load_global = [&](int s) {
    int j = s / kchunks, k0 = (s - j * kchunks) * BK;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      int ts = a_t[i] + (j - pad) * dil;
      if (a_ok[i] && ts >= 0 && ts < g.L)
        ra[i] = __ldg(reinterpret_cast<const float4*>(g.x + (a_base[i] + ts) * g.ldx + k0 + lk));
      else
        ra[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (b_ok[i])
        rb[i] = __ldg(reinterpret_cast<const float4*>(g.w + ((long)j * g.N + n0 + lr + 64 * i) * g.K + k0 + lk));
      else
        rb[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store_shared = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      int r = lr + 64 * i;
      As[buf][lk + 0][r] = ra[i].x; As[buf][lk + 1][r] = ra[i].y; As[buf][lk + 2][r] = ra[i].z; As[buf][lk + 3][r] = ra[i].w;
      Bs[buf][lk + 0][r] = rb[i].x; Bs[buf][lk + 1][r] = rb[i].y; Bs[buf][lk + 2][r] = rb[i].z; Bs[buf][lk + 3][r] = rb[i].w;
    }
  };

  const int ty = tid >> 4, tx = tid & 15;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  load_global(0);
  store_shared(0);
  __syncthreads();

  for (int s = 0; s < steps; ++s) {
    const int buf = s & 1;
    if (s + 1 < steps) load_global(s + 1);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
      float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + tx * 4]);
      float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (s + 1 < steps) {
      store_shared(buf ^ 1);   // buf^1 was last read in iteration s-1, fenced by the barrier below
      __syncthreads();
    }
  }

  // epilogue: bias, activation, residual; 16-byte stores
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= M) continue;
    const bool padded = g.lens && m % g.L >= g.lens[m / g.L];   // per-utterance mode: exact zeros past the utterance
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int n = n0 + h * 64 + tx * 4;
      if (n >= g.N) continue;
      float4 v = make_float4(acc[i][h * 4 + 0], acc[i][h * 4 + 1], acc[i][h * 4 + 2], acc[i][h * 4 + 3]);
      if (g.bias) {
        float4 bv = __ldg(reinterpret_cast<const float4*>(g.bias + n));
        v.x += bv.x; v.y += bv.y; v.z += bv.z; v.w += bv.w;
      }
      if (ACT == ACT_RELU) {
        v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
      } else if (ACT == ACT_TANH) {
        v.x = tanhf(v.x); v.y = tanhf(v.y); v.z = tanhf(v.z); v.w = tanhf(v.w);
      }
      if (HAS_RES) {
        float4 rv = __ldg(reinterpret_cast<const float4*>(g.resid + (long)m * g.ldr + n));
        v.x += rv.x; v.y += rv.y; v.z += rv.z; v.w += rv.w;
      }
      if (padded) v = make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(g.out + (long)m * g.ldo + n) = v;
    }
  }
}

template <int ACT>
int launch(const TapGemm& g, cudaStream_t st) {
  dim3 grid((g.N + BN - 1) / BN, (g.B * g.L + BM - 1) / BM);
  if (g.resid) tap_gemm_fp32_kernel<ACT, true><<<grid, NTHREADS, 0, st>>>(g);
  else tap_gemm_fp32_kernel<ACT, false><<<grid, NTHREADS, 0, st>>>(g);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace

int tap_gemm_fp32(const TapGemm& g, cudaStream_t st) {
  FS2_REQUIRE(g.K % BK == 0 && g.N % 4 == 0, "tap_gemm_fp32: K (%d) must be a multiple of 16 and N (%d) of 4", g.K, g.N);
  FS2_REQUIRE(g.ldx % 4 == 0 && g.ldo % 4 == 0 && (!g.resid || g.ldr % 4 == 0), "tap_gemm_fp32: row strides must be 16-byte multiples");
  FS2_REQUIRE((g.taps & 1) == 1 && g.taps >= 1, "tap_gemm_fp32: taps must be odd");
  if ((long)g.B * g.L == 0) return FS2_OK;
  switch (g.act) {
    case ACT_NONE: return launch<ACT_NONE>(g, st);
    case ACT_RELU: return launch<ACT_RELU>(g, st);
    case ACT_TANH: return launch<ACT_TANH>(g, st);
  }
  set_error("tap_gemm_fp32: unknown activation %d", g.act);
  return FS2_ERR_INVALID;
}

}  // namespace fs2
