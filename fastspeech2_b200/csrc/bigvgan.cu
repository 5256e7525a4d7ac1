// BigVGAN's anti-aliased activation (DESIGN.md section 18): the Activation1d(Snake / SnakeBeta) kernels that BigVGAN runs
// on HiFi-GAN's generator chain (hifigan.cu) in place of its lrelu, before every block convolution and before conv_post.
// The chain, its window plan, its weights and BigVGAN's C entries are hifigan.cu's; this file holds the activation
// producer, the head, the activation parameters and the single-activation entry.
//
// Activation1d (alias-free torch's, per channel): up = 2 conv_transpose1d(replicate_pad(x, 5), f_up, stride 2)[15 : -15],
// s = Snake(up) = up + inv sin^2(alpha up) (inv = 1 / (alpha + 1e-9), or 1 / (beta + 1e-9) for SnakeBeta), out =
// conv1d(replicate_pad(s, (5, 6)), f_down, stride 2).  So 2x sample m of an utterance of n rows is u[m] = 2 sum_j
// x[clamp(j)] f_up[m + 5 - 2j] (six taps: j = m/2 - 3 .. m/2 + 2 for even m, (m-1)/2 - 2 .. (m-1)/2 + 3 for odd m), and
// out[t] = sum_k f_down[k] s[clamp(2t + k - 5)] with k = 0 .. 11, clamp to [0, 2n); out[t] reads rows t - 5 .. t + 5.
// Replicate padding is index clamping: to [0, len) of the buffer, which at an utterance edge is the utterance's edge and
// at a window side that is not one stays inside the buffer (those rows are wrong within the margin the plan absorbs).
//
// A width that is not a multiple of 32 runs zero-padded to C' = ceil32(C): the padded channels have alpha' = inv = 0, so
// they stay exactly 0 (Snake(0) = 0).  Every producer computes an element from its own utterance's rows below lens_s in a
// fixed arithmetic order that does not depend on where the row sits in its tile, so per-utterance results depend neither
// on the batch nor on the window.
#include <math.h>

#include "bigvgan.cuh"
#include "operand_planes.cuh"
#include "vocoder_weights.cuh"
#include "vocoder_window.cuh"

namespace fs2 {
namespace {

constexpr int kPostTaps = 7;                // conv_post's taps
constexpr int kChunk = 32, kQ = kChunk / 4; // channels per activation tile, and their float4 quads
constexpr int kActTile = 64;                // output rows per CTA of the activation producer
constexpr int kPostTile = 64;               // audio samples per CTA of the post kernel
constexpr float kSnakeEps = 1e-9f;          // Snake's no_div_by_zero

// The Activation1d of rows [l0, l0 + T) of one utterance's buffer x (local row 0 at x, rows C floats apart; combined as
// (x + r) / nk, r nullable) for channels [c0, c0 + 32), input rows clamped to [0, len) (len >= 1): x rows l0 - 5 ..
// l0 + T + 4 staged once, their 2x samples and Snake values computed once, then the 12-tap down filter.  emit(i, q, v):
// output row l0 + i, channels c0 + 4 q .. c0 + 4 q + 3.  Every thread of the CTA calls it; it ends without a barrier.
template <int T, typename Emit>
__device__ __forceinline__ void act_tile(const float* __restrict__ x, const float* __restrict__ r, int nk, int C, int c0, int l0, int len,
                                         const float* __restrict__ prm, int Cp, const float* __restrict__ f, float4* xs, float4* ss,
                                         Emit emit) {
  constexpr int XR = T + 2 * kAct, SR = 2 * T + 2 * kAct;
  const float fk = (float)nk;
  for (int i = threadIdx.x; i < XR * kQ; i += blockDim.x) {
    const int row = i / kQ, q = i - row * kQ;
    const long off = (long)min(max(l0 - kAct + row, 0), len - 1) * C + c0 + 4 * q;
    float4 v = __ldg(reinterpret_cast<const float4*>(x + off));
    if (r) {
      const float4 u = __ldg(reinterpret_cast<const float4*>(r + off));
      v = make_float4(v.x + u.x, v.y + u.y, v.z + u.z, v.w + u.w);
    }
    if (nk != 1) v = make_float4(v.x / fk, v.y / fk, v.z / fk, v.w / fk);
    xs[i] = v;
  }
  __syncthreads();
  const float* fu = f;
  const float* fd = f + kFilt;
  for (int i = threadIdx.x; i < SR * kQ; i += blockDim.x) {
    const int mi = i / kQ, q = i - mi * kQ;
    const int m = min(max(2 * l0 - kAct + mi, 0), 2 * len - 1), p = m >> 1, odd = m & 1;
    // u[m] = 2 sum_jj x[j] f_up[2 jj + 1 - odd], j = p + 2 + odd - jj: staged row j - (l0 - 5)
    const int j0 = p + 2 + odd - (l0 - kAct);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int jj = 0; jj < 6; ++jj) {
      const float w = fu[2 * jj + 1 - odd];
      const float4 v = xs[(j0 - jj) * kQ + q];
      acc = make_float4(fmaf(w, v.x, acc.x), fmaf(w, v.y, acc.y), fmaf(w, v.z, acc.z), fmaf(w, v.w, acc.w));
    }
    const float4 a = __ldg(reinterpret_cast<const float4*>(prm + c0) + q);
    const float4 iv = __ldg(reinterpret_cast<const float4*>(prm + Cp + c0) + q);
    float4 s;
    float u, sn;
    u = 2.f * acc.x; sn = sinf(a.x * u); s.x = fmaf(iv.x, sn * sn, u);
    u = 2.f * acc.y; sn = sinf(a.y * u); s.y = fmaf(iv.y, sn * sn, u);
    u = 2.f * acc.z; sn = sinf(a.z * u); s.z = fmaf(iv.z, sn * sn, u);
    u = 2.f * acc.w; sn = sinf(a.w * u); s.w = fmaf(iv.w, sn * sn, u);
    ss[i] = s;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < T * kQ; i += blockDim.x) {
    const int row = i / kQ, q = i - row * kQ;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < kFilt; ++k) {                  // 2x sample 2 (l0 + row) + k - 5: staged 2 row + k
      const float w = fd[k];
      const float4 v = ss[(2 * row + k) * kQ + q];
      acc = make_float4(fmaf(w, v.x, acc.x), fmaf(w, v.y, acc.y), fmaf(w, v.z, acc.z), fmaf(w, v.w, acc.w));
    }
    emit(row, q, acc);
  }
}

// The producer of a GEMM operand [B * Lp][C] = Activation1d(x) (x [B * Lp][C], the operand's own window win: nullptr =
// the whole utterance) for t < len; +0 past it.  Grid: (B * tiles, C / 32), one CTA per 64 rows x 32 channels of one
// utterance.  Only rows exact_row(margin) are range-checked.
template <int OUT>
__global__ void __launch_bounds__(256) bigvgan_act_kernel(const float* __restrict__ x, const int64_t* __restrict__ lens,
                                                          const int64_t* __restrict__ win, int B, int Lp, int C, int tiles,
                                                          const float* __restrict__ prm, int margin, float* __restrict__ out32,
                                                          __half* __restrict__ outp, int* __restrict__ status) {
  __shared__ float4 xs[(kActTile + 2 * kAct) * kQ], ss[(2 * kActTile + 2 * kAct) * kQ];
  __shared__ float f[2 * kFilt];
  const int b = blockIdx.x / tiles, t0 = (blockIdx.x - b * tiles) * kActTile, c0 = blockIdx.y * kChunk;
  const Rows w = rows_of(win, lens, B, b);
  const long plane = (long)B * Lp * C;
  if (t0 >= w.len) {
    for (int i = threadIdx.x; i < kActTile * kQ; i += blockDim.x) {
      const int t = t0 + i / kQ;
      if (t < Lp) store_quad<OUT, RANGE_NEVER>(make_float4(0.f, 0.f, 0.f, 0.f), ((long)b * Lp + t) * C + c0 + 4 * (i % kQ), out32, outp,
                                               plane, nullptr, 0);
    }
    return;
  }
  if (threadIdx.x < 2 * kFilt) f[threadIdx.x] = prm[2L * C + threadIdx.x];
  __syncthreads();
  act_tile<kActTile>(x + (long)b * Lp * C, nullptr, 1, C, c0, t0, w.len, prm, C, f, xs, ss, [&](int i, int q, float4 v) {
    const int t = t0 + i;
    if (t >= Lp) return;
    if (t >= w.len) v = make_float4(0.f, 0.f, 0.f, 0.f);
    store_quad<OUT, RANGE_IF_STATUS>(v, ((long)b * Lp + t) * C + c0 + 4 * q, out32, outp, plane,
                                     t < w.len && (!win || exact_row(w, t, margin)) ? status : nullptr, FS2_BIGVGAN_RANGE);
  });
}

// audio[b, t] = final(bias + sum_c sum_j w[j][c] y[t + j - 3][c]) for t < n, else +0: y = Activation1d((S + R) / nk)
// (R nullable) of the last MRF's output, 0 outside [0, lens[b]) (conv_post's zero padding); final = tanh, or a clamp to
// [-1, 1].  w [7][C] (C = C'_U, zero columns for padded channels), bias nullable.  S and R have Lx rows per utterance in
// window win (nullptr: the whole utterance), audio Lout samples per row, rows ld apart; a window: audio row b holds
// samples [start, start + len) of awin, +0 past them.  One CTA per 64 samples of one utterance: per 32-channel chunk,
// the activation of the 70 rows they read, then thread (i, g) sums channels 8 g .. 8 g + 7 of sample i over the taps and
// the four partial sums are added in a fixed order.
__global__ void __launch_bounds__(256) bigvgan_post_kernel(const float* __restrict__ S, const float* __restrict__ R, int nk,
                                                           const int64_t* __restrict__ lens, const int64_t* __restrict__ win,
                                                           const int64_t* __restrict__ awin, int B, int Lx, int Lout, long ld, int C,
                                                           int tiles, const float* __restrict__ prm, const float* __restrict__ w,
                                                           const float* __restrict__ bias, int use_tanh, float* __restrict__ audio) {
  constexpr int TA = kPostTile + kPostTaps - 1;
  __shared__ float4 xs[(TA + 2 * kAct) * kQ], ss[(2 * TA + 2 * kAct) * kQ], ys[TA * kQ];
  __shared__ float f[2 * kFilt], wsm[kPostTaps * kChunk], part[4][kPostTile];
  const int b = blockIdx.x / tiles, t0 = (blockIdx.x - b * tiles) * kPostTile;
  const Rows r = rows_of(win, lens, B, b);
  const int a0 = awin ? (int)awin[b] : 0, n = awin ? (int)awin[B + b] : r.n;
  const int i = threadIdx.x & (kPostTile - 1), g = threadIdx.x / kPostTile;
  if (t0 >= n) {
    if (g == 0 && t0 + i < Lout) audio[(long)b * ld + t0 + i] = 0.f;
    return;
  }
  if (threadIdx.x < 2 * kFilt) f[threadIdx.x] = prm[2L * C + threadIdx.x];
  const int g0 = a0 + t0 - kPostTaps / 2;            // global row of y for sample t0, tap 0
  float acc = bias ? __ldg(bias) : 0.f;
  for (int c0 = 0; c0 < C; c0 += kChunk) {
    for (int k = threadIdx.x; k < kPostTaps * kChunk; k += blockDim.x) wsm[k] = w[(k / kChunk) * C + c0 + k % kChunk];
    __syncthreads();
    act_tile<TA>(S + (long)b * Lx * C, R ? R + (long)b * Lx * C : nullptr, nk, C, c0, g0 - r.start, r.len, prm, C, f, xs, ss,
                 [&](int k, int q, float4 v) { ys[k * kQ + q] = v; });
    __syncthreads();
    const float* y = reinterpret_cast<const float*>(ys);
    float p = 0.f;
#pragma unroll 1
    for (int j = 0; j < kPostTaps; ++j) {
      const int src = g0 + i + j;
      if (src < 0 || src >= r.n) continue;
#pragma unroll
      for (int c = 8 * g; c < 8 * g + 8; ++c) p = fmaf(wsm[j * kChunk + c], y[(i + j) * kChunk + c], p);
    }
    part[g][i] = p;
    __syncthreads();
    if (g == 0) acc += (part[0][i] + part[1][i]) + (part[2][i] + part[3][i]);
    __syncthreads();
  }
  if (g == 0 && t0 + i < Lout) audio[(long)b * ld + t0 + i] = t0 + i < n ? (use_tanh ? tanhf(acc) : fminf(fmaxf(acc, -1.f), 1.f)) : 0.f;
}

// prm (act_params(Cp) floats) of one activation: alpha' = exp(alpha) with logscale, inv = 1 / (beta' + 1e-9) with beta' =
// (exp(beta) or beta) for SnakeBeta, alpha' for Snake (beta == nullptr); 0 in the padded channels; then the two filters
__global__ void act_param_kernel(const float* __restrict__ alpha, const float* __restrict__ beta, const float* __restrict__ fu,
                                 const float* __restrict__ fd, int C, int Cp, int logscale, float* __restrict__ prm) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < Cp; c += gridDim.x * blockDim.x) {
    float a = 0.f, inv = 0.f;
    if (c < C) {
      a = logscale ? expf(alpha[c]) : alpha[c];
      const float be = beta ? (logscale ? expf(beta[c]) : beta[c]) : a;
      inv = 1.f / (be + kSnakeEps);
    }
    prm[c] = a;
    prm[Cp + c] = inv;
    if (c < kFilt) {
      prm[2L * Cp + c] = fu[c];
      prm[2L * Cp + kFilt + c] = fd[c];
    }
  }
}

}  // namespace

int bigvgan_act(int kind, const float* x, const float* prm, const int64_t* lens, const int64_t* win, int B, int Lp, int C, int margin,
                void* a, int* status, cudaStream_t st) {
  auto k = pick(kind, bigvgan_act_kernel<OUT_HILO>, bigvgan_act_kernel<OUT_HI>, bigvgan_act_kernel<OUT_F32>);
  const int tiles = (Lp + kActTile - 1) / kActTile;
  k<<<dim3((unsigned)((long)B * tiles), C / kChunk), 256, 0, st>>>(x, lens, win, B, Lp, C, tiles, prm, margin, (float*)a, (__half*)a, status);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int bigvgan_post(const float* S, const float* R, int nk, const int64_t* lens, const int64_t* win, const int64_t* awin, int B, int Lx,
                 int Lout, long ld, int C, const float* prm, const float* w, const float* bias, int use_tanh, float* audio, cudaStream_t st) {
  const int tiles = (Lout + kPostTile - 1) / kPostTile;
  bigvgan_post_kernel<<<(unsigned)((long)B * tiles), 256, 0, st>>>(S, R, nk, lens, win, awin, B, Lx, Lout, ld, C, tiles, prm, w, bias,
                                                                    use_tanh, audio);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int act_param(const float* const* t, int C, int logscale, int snakebeta, float* prm, cudaStream_t st) {
  const int Cp = ceil32(C);
  act_param_kernel<<<grid_for(Cp, 256), 256, 0, st>>>(t[0], snakebeta ? t[1] : nullptr, t[2], t[3], C, Cp, logscale, prm);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace fs2

using namespace fs2;

extern "C" {

// ---- a single activation on the vocoder's own code path (tests) -----------------------------------------------------
int fs2_op_bigvgan_act(int math_mode, int C, const float* x, const int64_t* lens, int B, int Lp, const float* const* tensors, int snakebeta,
                       int logscale, float* out, int* status, void* stream) {
  const char* who = "fs2_op_bigvgan_act";
  FS2_REQUIRE(math_mode >= FS2_MATH_FP32 && math_mode <= FS2_MATH_F16, "%s: bad math_mode %d", who, math_mode);
  FS2_REQUIRE(C >= 8 && C % 8 == 0 && C <= 2048, "%s: C must be a multiple of 8 in [8, 2048] (got %d)", who, C);
  FS2_REQUIRE(x && lens && tensors && tensors[0] && (tensors[1] || !snakebeta) && tensors[2] && tensors[3] && out && status,
              "%s: null argument", who);
  FS2_REQUIRE(B >= 1 && Lp >= 1, "%s: bad shape B=%d Lp=%d", who, B, Lp);
  const int Cp = ceil32(C), kind = out_kind(math_mode);
  const long rows = (long)B * Lp;
  FS2_REQUIRE(rows * Cp < (1L << 31), "%s: too many rows (%ld)", who, rows);
  cudaStream_t st = (cudaStream_t)stream;
  float *xp = nullptr, *prm = nullptr, *y = nullptr;
  void* a = nullptr;
  void* base = nullptr;
  int rc = temp_carve(&base, st, [&](Bump& b) {
    xp = b.floats((size_t)rows * Cp);
    prm = b.floats(act_params(Cp));
    a = b.floats((size_t)rows * Cp);
    y = b.floats((size_t)rows * Cp);
  });
  if (rc) return rc;
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  FS2_CUDA_CHECK(cudaMemsetAsync(a, 0, sizeof(float) * rows * Cp, st));
  if (!(rc = pad3(x, (int)rows, C, 1, xp, (int)rows, Cp, st)) && !(rc = act_param(tensors, C, logscale, snakebeta, prm, st)) &&
      !(rc = bigvgan_act(kind, xp, prm, lens, nullptr, B, Lp, Cp, 0, a, status, st))) {
    const float* rows32 = (const float*)a;
    if (kind != OUT_F32) rc = planes_to_rows((const __half*)a, rows * Cp, y, st), rows32 = y;
    if (!rc) rc = pad3(rows32, (int)rows, Cp, 1, out, (int)rows, C, st);
  }
  cudaFreeAsync(base, st);
  return rc;
}

}  // extern "C"
