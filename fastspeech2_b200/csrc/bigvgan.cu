// Batched BigVGAN vocoder (DESIGN.md section 18): log-mels [B, Lmax, 80] -> audio [B, Lmax * 256], each utterance
// NVIDIA BigVGAN's generator over its own olens[b] frames, on the library's tap-GEMM.
//
// The stage layout is HiFi-GAN's (hifigan.cu): stage s has Lp_s = Lmax * up_s rows per utterance of C'_s = ceil32(C0 / 2^s)
// channels, every GEMM of the stage runs with lens_s = olens * up_s, and every convolution zero-pads at the utterance's
// own edges through the rows-past-lens rule.  A width that is not a multiple of 32 (the 22 kHz large models end at 24) is
// zero-padded to C': its weights get zero rows and columns and its padded output channels a zero bias, so the padded
// channels stay exactly 0 through every layer (Snake(0) = 0).
//
//   mel operand   mel rows (0 past olens)                                  -> GEMM 7 taps, 80 -> C0     = conv_pre
//   per stage s:
//     rows        x = the previous MRF's (S + r) / nk, no activation       -> GEMM 3 taps, C'_s -> u C'_{s+1}: the
//                 ConvTranspose1d(k = 2u, stride u, pad u / 2) as hifigan.cu's polyphase GEMM, rows r C' + co
//     per AMP block j of the MRF, per conv step m (AMPBlock1: x = c2(a2(c1(a1(x)))) + x; AMPBlock2: x = c(a(x)) + x):
//                 act Activation1d(x) -> GEMM k taps at dilation d_m (-> act -> GEMM k taps, dilation 1), the residual
//                 add in the last GEMM's epilogue
//     add         S += r_j for the middle blocks (1 .. nk - 2)
//   post          Activation1d((S + r_last) / nk), conv C -> 1 (k = 7, zero padding, optional bias), tanh or clamp to
//                 [-1, 1], on CUDA cores, +0 past olens * 256
//
// Activation1d (alias-free torch's, per channel): up = 2 conv_transpose1d(replicate_pad(x, 5), f_up, stride 2)[15 : -15],
// s = Snake(up) = up + inv sin^2(alpha up) (inv = 1 / (alpha + 1e-9), or 1 / (beta + 1e-9) for SnakeBeta), out =
// conv1d(replicate_pad(s, (5, 6)), f_down, stride 2).  So 2x sample m of an utterance of n rows is u[m] = 2 sum_j
// x[clamp(j)] f_up[m + 5 - 2j] (six taps: j = m/2 - 3 .. m/2 + 2 for even m, (m-1)/2 - 2 .. (m-1)/2 + 3 for odd m), and
// out[t] = sum_k f_down[k] s[clamp(2t + k - 5)] with k = 0 .. 11, clamp to [0, 2n); out[t] reads rows t - 5 .. t + 5.
// Replicate padding is index clamping: to [0, len) of the buffer, which at an utterance edge is the utterance's edge and
// at a window side that is not one stays inside the buffer (those rows are wrong within the margin the plan absorbs).
//
// Launches per call: 4 + U * (2 + nk * G + max(nk - 2, 0)), G = 12 (AMPBlock1) or 4 (AMPBlock2), in every math mode.
// Buffers as HiFi-GAN's: five of [B * Lp_s][C'_s] at the current stage, A = max_s up_s C'_s floats per frame each.
//
// Every producer computes an element from its own utterance's rows below lens_s in a fixed arithmetic order that does not
// depend on where the row sits in its tile, so per-utterance results depend neither on the batch nor on the window.
//
// Windows (fs2_bigvgan_window): hifigan.cu's, on the chain plan of vocoder_window.cuh with R = the largest AMP block's
// reach including its activations (AMPBlock1 sum_m ((k-1)/2 (d_m + 1) + 2 a), AMPBlock2 sum_m ((k-1)/2 d_m + a), a = 5),
// level-0 margin 3 and a last-layer reach of 3 + a.  The range-check margins widen by a at every activation.
#include <math.h>

#include <algorithm>
#include <vector>

#include "vocoder_weights.cuh"
#include "vocoder_window.cuh"

namespace fs2 {
namespace {

constexpr int kMels = 80, kHop = 256, kPreTaps = 7, kPostTaps = 7;
constexpr int kAct = 5;                     // Activation1d's reach: output row t reads input rows t - 5 .. t + 5
constexpr int kFilt = 12;                   // taps of the up and down filters
constexpr int kChunk = 32, kQ = kChunk / 4; // channels per activation tile, and their float4 quads
constexpr int kActTile = 64;                // output rows per CTA of the activation producer
constexpr int kPostTile = 64;               // audio samples per CTA of the post kernel
constexpr float kSnakeEps = 1e-9f;          // Snake's no_div_by_zero

static_assert(FS2_BIGVGAN_BAD_LENGTH == FS2_HIFIGAN_BAD_LENGTH && FS2_BIGVGAN_BAD_START == FS2_HIFIGAN_BAD_START,
              "ups_prep writes the upsampling chains' common status bits");

inline int ceil32(int c) { return (c + 31) / 32 * 32; }

// One activation's parameters on the device, prm [2 C' + 24]: alpha' [C'] (exp(alpha) with snake_logscale), inv [C']
// (1 / (beta' + 1e-9), beta' = alpha' for Snake), f_up [12], f_down [12].  Padded channels have alpha' = inv = 0.
__host__ __device__ constexpr long act_params(int Cp) { return 2L * Cp + 2 * kFilt; }

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

// A GEMM operand [B * Lp][C] of plain rows: v = x, or the MRF combine (x + r) / nk (r nullable), for t < len; +0 past it.
// Local row t of utterance b reads x's row b * ldx + t + o, o = 0 for a whole call and, for a window (win), the window's
// start minus x's own (xwin; nullptr: x holds global rows, the mels).  conv_pre's operand (x = the mels, ldx = Lmax, C =
// 80) and every upsampling's (no activation before BigVGAN's upsamplings).  Every row it reads holds the whole call's
// values, so all are range-checked.
template <int OUT>
__global__ void bigvgan_rows_kernel(const float* __restrict__ x, const float* __restrict__ r, int nk, const int64_t* __restrict__ lens,
                                    const int64_t* __restrict__ xwin, int ldx, const int64_t* __restrict__ win, int B, int Lp, int C,
                                    float* __restrict__ out32, __half* __restrict__ outp, int* __restrict__ status) {
  const int Q = C / 4;
  const long rows = (long)B * Lp, total = rows * Q, plane = rows * C;
  const float fk = (float)nk;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / Q;
    const int b = (int)(row / Lp), t = (int)(row - (long)b * Lp);
    const int c = (int)(i - row * Q) * 4;
    const Rows w = rows_of(win, lens, B, b);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t < w.len) {
      const int o = win ? w.start - (xwin ? (int)xwin[b] : 0) : 0;
      const long src = ((long)b * ldx + t + o) * C + c;
      v = __ldg(reinterpret_cast<const float4*>(x + src));
      if (r) {
        const float4 u = __ldg(reinterpret_cast<const float4*>(r + src));
        v = make_float4(v.x + u.x, v.y + u.y, v.z + u.z, v.w + u.w);
      }
      if (nk != 1) v = make_float4(v.x / fk, v.y / fk, v.z / fk, v.w / fk);
    }
    store_quad<OUT, RANGE_IF_STATUS>(v, row * C + c, out32, outp, plane, status, FS2_BIGVGAN_RANGE);
  }
}

// s[i] += r[i] over n floats (n a multiple of 4): the MRF's running sum; rows past lens are +0 in both
__global__ void bigvgan_add_kernel(float* __restrict__ s, const float* __restrict__ r, long n) {
  for (long i = ((long)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < n; i += (long)gridDim.x * blockDim.x * 4) {
    float4 a = *reinterpret_cast<const float4*>(s + i);
    const float4 b = *reinterpret_cast<const float4*>(r + i);
    *reinterpret_cast<float4*>(s + i) = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
  }
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

int pad3(const float* src, int A, int Bn, int k, float* dst, int Ap, int Bp, cudaStream_t st) {
  pad3_kernel<<<grid_for((long)Ap * Bp * k, 256), 256, 0, st>>>(src, A, Bn, k, dst, Ap, Bp);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// ---- host side ------------------------------------------------------------------------------------------------------

struct Shape {
  int U, nk, type, steps, per, acts;   // upsamplings, blocks per MRF, block type, conv steps, convolutions and activations per block
  int C[kMaxUps + 1], Cp[kMaxUps + 1]; // stage widths C0 / 2^s and their padded widths ceil32
  UpsPlan ups;
  int layers, nact;                    // convolutions and activations in state_dict order
  long act;                            // floats per frame of the largest stage buffer, max_s up_s * C'_s
};

Shape shape_of(const fs2_bigvgan_config& cf) {
  const fs2_hifigan_config& c = cf.gen;
  Shape s;
  s.U = c.num_upsamples; s.nk = c.num_kernels; s.type = c.resblock;
  s.steps = s.type == 1 ? 3 : 2; s.per = s.type == 1 ? 6 : 2; s.acts = s.per;
  int R = 0;                                           // the MRF's reach: the largest block's, activations included
  for (int j = 0; j < s.nk; ++j) {
    int r = 0;
    for (int m = 0; m < s.steps; ++m)
      r += (c.resblock_kernel_sizes[j] - 1) / 2 * (c.resblock_dilation_sizes[j][m] + (s.type == 1)) + (s.type == 1 ? 2 : 1) * kAct;
    R = std::max(R, r);
  }
  // conv_pre's native taps leave its outer 3 rows wrong at a side that is not an utterance edge; conv_post reads 3 rows
  // of activation_post's output, which reads 5 more; no tail
  s.ups = ups_plan(s.U, c.upsample_rates, R, kPreTaps / 2, kPostTaps / 2 + kAct, 0);
  s.C[0] = c.upsample_initial_channel;
  s.Cp[0] = ceil32(s.C[0]);
  s.act = s.Cp[0];
  for (int i = 0; i < s.U; ++i) {
    s.C[i + 1] = s.C[i] / 2;
    s.Cp[i + 1] = ceil32(s.C[i + 1]);
    s.act = std::max(s.act, (long)s.ups.up[i + 1] * s.Cp[i + 1]);
  }
  s.layers = 2 + s.U + s.U * s.nk * s.per;
  s.nact = s.U * s.nk * s.acts + 1;
  return s;
}

int validate(const fs2_bigvgan_config* cf) {
  const char* who = "fs2_bigvgan_create";
  const fs2_hifigan_config* c = &cf->gen;
  FS2_REQUIRE(c->resblock == 1 || c->resblock == 2, "%s: resblock must be 1 or 2 (got %d)", who, c->resblock);
  FS2_REQUIRE(c->num_upsamples >= 1 && c->num_upsamples <= kMaxUps, "%s: num_upsamples must lie in [1, %d] (got %d)", who, kMaxUps,
              c->num_upsamples);
  long prod = 1;
  for (int i = 0; i < c->num_upsamples; ++i) {
    const int u = c->upsample_rates[i];
    FS2_REQUIRE(u >= 2 && u % 2 == 0 && u <= kHop, "%s: upsample_rates[%d] = %d must be even, in [2, 256]", who, i, u);
    FS2_REQUIRE(c->upsample_kernel_sizes[i] == 2 * u, "%s: upsample_kernel_sizes[%d] = %d must be twice the rate %d", who, i,
                c->upsample_kernel_sizes[i], u);
    prod *= u;
  }
  FS2_REQUIRE(prod == kHop, "%s: the product of upsample_rates is %ld, not the hop 256", who, prod);
  const int C0 = c->upsample_initial_channel;
  FS2_REQUIRE(C0 >= 8 && C0 <= 2048 && C0 % (8 << c->num_upsamples) == 0,
              "%s: upsample_initial_channel = %d must lie in [8, 2048] with every width C0 / 2^i a multiple of 8", who, C0);
  FS2_REQUIRE(c->num_kernels >= 1 && c->num_kernels <= FS2_HIFIGAN_MAX_KERNELS, "%s: num_kernels must lie in [1, %d] (got %d)", who,
              FS2_HIFIGAN_MAX_KERNELS, c->num_kernels);
  FS2_REQUIRE(c->num_dilations == (c->resblock == 1 ? 3 : 2), "%s: num_dilations must be %d for resblock %d (got %d)", who,
              c->resblock == 1 ? 3 : 2, c->resblock, c->num_dilations);
  for (int j = 0; j < c->num_kernels; ++j) {
    const int k = c->resblock_kernel_sizes[j];
    FS2_REQUIRE(k >= 1 && k <= 31 && k % 2 == 1, "%s: resblock_kernel_sizes[%d] = %d must be odd, in [1, 31]", who, j, k);
    for (int m = 0; m < c->num_dilations; ++m) {
      const int d = c->resblock_dilation_sizes[j][m];
      FS2_REQUIRE(d >= 1 && d <= 1024, "%s: resblock_dilation_sizes[%d][%d] = %d must lie in [1, 1024]", who, j, m, d);
    }
  }
  FS2_REQUIRE(cf->activation == FS2_BIGVGAN_SNAKE || cf->activation == FS2_BIGVGAN_SNAKEBETA,
              "%s: activation must be FS2_BIGVGAN_SNAKE or FS2_BIGVGAN_SNAKEBETA (got %d)", who, cf->activation);
  return FS2_OK;
}

// the activation producer (bigvgan_act_kernel) of x [B * Lp][C] into the operand a
int act(int kind, const float* x, const float* prm, const int64_t* lens, const int64_t* win, int B, int Lp, int C, int margin, void* a,
        int* status, cudaStream_t st) {
  auto k = pick(kind, bigvgan_act_kernel<OUT_HILO>, bigvgan_act_kernel<OUT_HI>, bigvgan_act_kernel<OUT_F32>);
  const int tiles = (Lp + kActTile - 1) / kActTile;
  k<<<dim3((unsigned)((long)B * tiles), C / kChunk), 256, 0, st>>>(x, lens, win, B, Lp, C, tiles, prm, margin, (float*)a, (__half*)a, status);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// the plain-rows producer (bigvgan_rows_kernel) into the operand a
int rows_op(int kind, const float* x, const float* r, int nk, const int64_t* lens, const int64_t* xwin, int ldx, const int64_t* win, int B,
            int Lp, int C, void* a, int* status, cudaStream_t st) {
  auto k = pick(kind, bigvgan_rows_kernel<OUT_HILO>, bigvgan_rows_kernel<OUT_HI>, bigvgan_rows_kernel<OUT_F32>);
  k<<<grid_for((long)B * Lp * (C / 4), 256), 256, 0, st>>>(x, r, nk, lens, xwin, ldx, win, B, Lp, C, (float*)a, (__half*)a, status);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// One AMP block x -> dest on rows [B * Lp][C]: w = its convolutions and prm its activations, both in state_dict order, dil
// its dilations.  Step m writes t[m & 1], the last one dest; dest must differ from x and from t[(steps - 2) & 1].  win
// (nullable): the rows' window; margin: its rows at a side that is not an utterance edge whose values differ from the
// whole call's on entry, widened here by a at each activation and by each convolution's reach.
int resblock(int mode, int type, const VWeight* w, const float* const* prm, const int* dil, const float* x, const int64_t* lens,
             const int64_t* win, int B, int Lp, int C, int margin, void* a, float* const* t, float* dest, int* status, cudaStream_t st) {
  const int steps = type == 1 ? 3 : 2, kind = out_kind(mode), half = (w[0].taps - 1) / 2;
  const float* X = x;
  int rc;
  for (int m = 0; m < steps; ++m) {
    float* out = m == steps - 1 ? dest : t[m & 1];
    margin += kAct;
    if ((rc = act(kind, X, prm[type == 1 ? 2 * m : m], lens, win, B, Lp, C, margin, a, status, st))) return rc;
    margin += half * dil[m];
    if (type == 1) {
      if ((rc = vweight_gemm(mode, w[m], a, B, Lp, ACT_NONE, lens, out, st, nullptr, dil[m]))) return rc;   // h = c1(a1(x))
      margin += kAct;
      if ((rc = act(kind, out, prm[2 * m + 1], lens, win, B, Lp, C, margin, a, status, st))) return rc;
      margin += half;
      if ((rc = vweight_gemm(mode, w[3 + m], a, B, Lp, ACT_NONE, lens, out, st, X, 1))) return rc;        // c2(a2(h)) + x
    } else {
      if ((rc = vweight_gemm(mode, w[m], a, B, Lp, ACT_NONE, lens, out, st, X, dil[m]))) return rc;       // c(a(x)) + x
    }
    X = out;
  }
  return FS2_OK;
}

struct BvPlan {
  int64_t* lens;      // [U + 1][B]; a window call: the n_wins(sh.ups) window descriptors [start | len | n][B]
  void* a;            // GEMM operand
  float* xu;          // the upsampling output of the current stage
  float* s;           // MRF sum
  float* t[2];        // chain buffers
};

BvPlan carve_plan(Bump& b, size_t lens_bytes, size_t n) {
  BvPlan p;
  p.lens = (int64_t*)b.bytes(lens_bytes);
  p.a = b.floats(n);
  p.xu = b.floats(n);
  p.s = b.floats(n);
  p.t[0] = b.floats(n);
  p.t[1] = b.floats(n);
  return p;
}

BvPlan plan(Bump& b, const Shape& sh, int B, int L) {
  return carve_plan(b, (size_t)(sh.U + 1) * B * sizeof(int64_t), (size_t)B * L * sh.act);
}

// A window call's workspace, from B and nf only: five buffers of the largest level buffer per utterance (rows x C' over
// every level; conv_pre's operand, 80 wide, and the upsamplings' operands, r_s <= h_s, fit in it)
BvPlan window_plan(Bump& b, const Shape& sh, int B, int nf) {
  long act = level_rows(sh.ups, 0, nf) * kMels;
  for (int s = 0; s <= sh.U; ++s) act = std::max(act, level_rows(sh.ups, s, nf) * sh.Cp[s]);
  return carve_plan(b, (size_t)3 * n_wins(sh.ups) * B * sizeof(int64_t), (size_t)B * act);
}

void set_conv(VWeight& w, int N, int K, int taps) { w.N = N; w.K = K; w.taps = taps; }

// w (K = C'in, N = C'out, or u C'out rows for a polyphase upsampling) from a torch-layout weight [A][Bn][k] and bias
// [Cout] of real widths Cin / Cout: zero-padded to w's widths in a stream-ordered temporary when they differ, then packed
// as hifigan.cu packs it
int pack_conv(const VWeight& w, const float* wt, const float* bias, int Cin, int Cout, int taps, int u, cudaStream_t st) {
  const int Cip = w.K, Cop = u ? w.N / u : w.N, kk = u ? 2 * u : taps;
  if (Cip == Cin && Cop == Cout) return vweight_pack_conv(w, wt, bias, Cin, Cout, taps, u, (long)w.N * w.K, st);
  const int A = u ? Cin : Cout, Bn = u ? Cout : Cin, Ap = u ? Cip : Cop, Bp = u ? Cop : Cip;
  void* base = nullptr;
  float *pw = nullptr, *pb = nullptr;
  int rc = temp_carve(&base, st, [&](Bump& b) {
    pw = b.floats((size_t)Ap * Bp * kk);
    pb = b.floats(Cop);
  });
  if (rc) return rc;
  if (!(rc = pad3(wt, A, Bn, kk, pw, Ap, Bp, st)) && !(rc = pad3(bias, Cout, 1, 1, pb, Cop, 1, st)))
    rc = vweight_pack_conv(w, pw, pb, Cip, Cop, taps, u, (long)w.N * w.K, st);
  cudaFreeAsync(base, st);
  return rc;
}

int check_size(int math_mode, int B, int L) {
  FS2_REQUIRE(B >= 1 && L >= 1, "fs2_bigvgan: need B >= 1 and Lmax >= 1 (got %d, %d)", B, L);
  return check_rows("fs2_bigvgan", "B * Lmax * 256", "sample", (long)B * L * kHop, math_mode);
}

int act_param(const float* const* t, int C, int logscale, int snakebeta, float* prm, cudaStream_t st) {
  const int Cp = ceil32(C);
  act_param_kernel<<<grid_for(Cp, 256), 256, 0, st>>>(t[0], snakebeta ? t[1] : nullptr, t[2], t[3], C, Cp, logscale, prm);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace
}  // namespace fs2

struct fs2_bigvgan_gen {
  int device = 0, math_mode = 0;
  fs2_bigvgan_config cfg;
  fs2::Shape sh;
  bool loaded = false;
  void* arena = nullptr; size_t arena_bytes = 0;
  fs2::VWeight pre, up[fs2::kMaxUps];
  std::vector<fs2::VWeight> blk;   // [U * nk][per]: the blocks' convolutions in state_dict order
  std::vector<float*> prm;         // [U * nk * acts + 1]: the activations' parameters in state_dict order, activation_post last
  float* post_w = nullptr;         // [7][C'_U]
  float* post_b = nullptr;         // nullptr without use_bias_at_final
};

namespace fs2 {
namespace {

// The generator on the plan p: whole utterances (starts == nullptr) or a window of nf frames from starts[b], as
// hifigan.cu's generate.  Lout audio samples per row, rows ld apart.  Both enqueue the same kernels.
int generate(const fs2_bigvgan_gen* m, const BvPlan& p, const float* mels, const int64_t* olens, const int64_t* starts, int B, int L,
             int nf, float* audio, long ld, int* status, cudaStream_t st) {
  const Shape& sh = m->sh;
  const bool w = starts != nullptr;
  const int mode = m->math_mode, kind = out_kind(mode), U = sh.U;
  auto desc = [&](int i) -> const int64_t* { return w ? p.lens + 3L * i * B : nullptr; };
  auto lens = [&](int i, int s) -> const int64_t* { return w ? p.lens + (3L * i + 1) * B : p.lens + (long)s * B; };   // window i / level s
  auto rows = [&](int s) { return w ? (int)level_rows(sh.ups, s, nf) : L * sh.ups.up[s]; };
  int rc = ups_prep(olens, starts, B, L, nf, sh.ups, p.lens, status, st);
  if (rc) return rc;
  if ((rc = rows_op(kind, mels, nullptr, 1, lens(win_level(0), 0), nullptr, L, desc(win_level(0)), B, rows(0), kMels, p.a, status, st)))
    return rc;
  if ((rc = vweight_gemm(mode, m->pre, p.a, B, rows(0), ACT_NONE, lens(win_level(0), 0), p.t[0], st))) return rc;
  const float* x = p.t[0];
  const float* r = nullptr;
  int nk_in = 1;
  for (int s = 0; s < U; ++s) {
    const int Lin = w ? (int)ups_rows(sh.ups, s, nf) : rows(s), Lp = rows(s + 1), C = sh.Cp[s + 1];
    const int uw = win_ups(sh.ups, s), lw = win_level(s + 1);
    if ((rc = rows_op(kind, x, r, nk_in, lens(uw, s), desc(win_level(s)), rows(s), desc(uw), B, Lin, sh.Cp[s], p.a, status, st))) return rc;
    if ((rc = vweight_gemm(mode, m->up[s], p.a, B, Lin, ACT_NONE, lens(uw, s), p.xu, st))) return rc;
    const int margin = m->cfg.gen.upsample_rates[s] / 2;   // the rows the edge phases leave wrong at a side that is not an edge
    float* last = p.s;
    for (int j = 0; j < sh.nk; ++j) {
      const int g = s * sh.nk + j;
      last = j == 0 ? p.s : p.t[(sh.steps - 1) & 1];
      if ((rc = resblock(mode, sh.type, &m->blk[(size_t)g * sh.per], &m->prm[(size_t)g * sh.acts], m->cfg.gen.resblock_dilation_sizes[j],
                         p.xu, lens(lw, s + 1), desc(lw), B, Lp, C, margin, p.a, p.t, last, status, st)))
        return rc;
      if (j >= 1 && j < sh.nk - 1) {
        bigvgan_add_kernel<<<grid_for((long)B * Lp * C / 4, 256), 256, 0, st>>>(p.s, last, (long)B * Lp * C);
        FS2_LAUNCH_CHECK();
      }
    }
    x = p.s;
    r = sh.nk > 1 ? last : nullptr;
    nk_in = sh.nk;
  }
  const int Lout = (w ? nf : L) * kHop, tiles = (Lout + kPostTile - 1) / kPostTile;
  bigvgan_post_kernel<<<(unsigned)((long)B * tiles), 256, 0, st>>>(x, r, nk_in, lens(win_level(U), U), desc(win_level(U)),
                                                                    desc(win_audio(sh.ups)), B, rows(U), Lout, ld, sh.Cp[U], tiles,
                                                                    m->prm.back(), m->post_w, m->post_b, m->cfg.use_tanh_at_final, audio);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace
}  // namespace fs2

using namespace fs2;

extern "C" {

int fs2_bigvgan_create(fs2_bigvgan_gen** out, int math_mode, const fs2_bigvgan_config* cfg) {
  FS2_REQUIRE(out && cfg, "fs2_bigvgan_create: null argument");
  FS2_REQUIRE(math_mode >= FS2_MATH_FP32 && math_mode <= FS2_MATH_F16, "fs2_bigvgan_create: bad math_mode %d", math_mode);
  int rc = validate(cfg);
  if (rc) return rc;
  int dev = 0;
  FS2_CUDA_CHECK(cudaGetDevice(&dev));
  fs2_bigvgan_gen* m = new fs2_bigvgan_gen();
  m->math_mode = math_mode;
  m->device = dev;
  m->cfg = *cfg;
  m->sh = shape_of(*cfg);
  const Shape& sh = m->sh;
  set_conv(m->pre, sh.Cp[0], kMels, kPreTaps);
  for (int s = 0; s < sh.U; ++s) set_conv(m->up[s], cfg->gen.upsample_rates[s] * sh.Cp[s + 1], sh.Cp[s], 3);
  m->blk.resize((size_t)sh.U * sh.nk * sh.per);
  for (int s = 0; s < sh.U; ++s)
    for (int j = 0; j < sh.nk; ++j)
      for (int i = 0; i < sh.per; ++i)
        set_conv(m->blk[((size_t)s * sh.nk + j) * sh.per + i], sh.Cp[s + 1], sh.Cp[s + 1], cfg->gen.resblock_kernel_sizes[j]);
  m->prm.assign(sh.nact, nullptr);
  *out = m;
  return FS2_OK;
}

void fs2_bigvgan_destroy(fs2_bigvgan_gen* m) {
  if (!m) return;
  if (m->arena) cudaFree(m->arena);
  delete m;
}

int fs2_bigvgan_load(fs2_bigvgan_gen* m, const float* const* weights, const float* const* biases, const float* const* acts, void* stream) {
  FS2_REQUIRE(m && weights && biases && acts, "fs2_bigvgan_load: null argument");
  const Shape& sh = m->sh;
  const int last = sh.layers - 1, beta = m->cfg.activation == FS2_BIGVGAN_SNAKEBETA;
  for (int i = 0; i < sh.layers; ++i)
    FS2_REQUIRE(weights[i] && (biases[i] || (i == last && !m->cfg.use_bias_at_final)), "fs2_bigvgan_load: layer %d: null tensor", i);
  for (int i = 0; i < sh.nact; ++i)
    FS2_REQUIRE(acts[4 * i] && (acts[4 * i + 1] || !beta) && acts[4 * i + 2] && acts[4 * i + 3], "fs2_bigvgan_load: activation %d: null tensor",
                i);
  cudaStream_t st = (cudaStream_t)stream;
  m->loaded = false;
  auto width = [&](int i) { return i == sh.nact - 1 ? sh.C[sh.U] : sh.C[i / (sh.nk * sh.acts) + 1]; };   // activation i's channels
  int rc = arena_carve(&m->arena, &m->arena_bytes, st, [&](Bump& b) {
    vweight_carve(b, m->pre, true);
    for (int s = 0; s < sh.U; ++s) vweight_carve(b, m->up[s], true);
    for (auto& w : m->blk) vweight_carve(b, w, true);
    for (int i = 0; i < sh.nact; ++i) m->prm[i] = b.floats(act_params(ceil32(width(i))));
    m->post_w = b.floats((size_t)kPostTaps * sh.Cp[sh.U]);
    m->post_b = m->cfg.use_bias_at_final ? b.floats(1) : nullptr;
    return FS2_OK;
  });
  if (rc) return rc;
  if ((rc = pack_conv(m->pre, weights[0], biases[0], kMels, sh.C[0], kPreTaps, 0, st))) return rc;
  for (int s = 0; s < sh.U; ++s)
    if ((rc = pack_conv(m->up[s], weights[1 + s], biases[1 + s], sh.C[s], sh.C[s + 1], 3, m->cfg.gen.upsample_rates[s], st))) return rc;
  for (size_t i = 0; i < m->blk.size(); ++i) {
    const int C = sh.C[i / ((size_t)sh.nk * sh.per) + 1];
    if ((rc = pack_conv(m->blk[i], weights[1 + sh.U + i], biases[1 + sh.U + i], C, C, m->blk[i].taps, 0, st))) return rc;
  }
  for (int i = 0; i < sh.nact; ++i)
    if ((rc = act_param(acts + 4 * i, width(i), m->cfg.snake_logscale, beta, m->prm[i], st))) return rc;
  const int C = sh.C[sh.U], Cp = sh.Cp[sh.U];
  FS2_CUDA_CHECK(cudaMemsetAsync(m->post_w, 0, sizeof(float) * kPostTaps * Cp, st));
  if ((rc = conv_pack(weights[last], 1, C, kPostTaps, 1, 0, Cp, C, m->post_w, st))) return rc;
  if (m->post_b) FS2_CUDA_CHECK(cudaMemcpyAsync(m->post_b, biases[last], sizeof(float), cudaMemcpyDeviceToDevice, st));
  m->loaded = true;
  return FS2_OK;
}

int fs2_bigvgan_workspace_bytes(fs2_bigvgan_gen* m, int B, int Lmax, size_t* bytes) {
  FS2_REQUIRE(m && bytes, "fs2_bigvgan_workspace_bytes: null argument");
  int rc = check_size(m->math_mode, B, Lmax);
  if (rc) return rc;
  Bump b(nullptr, 0);
  plan(b, m->sh, B, Lmax);
  *bytes = b.off + 256;
  return FS2_OK;
}

int fs2_bigvgan(fs2_bigvgan_gen* m, const float* mels, const int64_t* olens, int B, int Lmax, float* audio, int* status, void* ws,
                size_t ws_bytes, void* stream) {
  FS2_REQUIRE(m && mels && olens && audio && status && ws, "fs2_bigvgan: null argument");
  FS2_REQUIRE(m->loaded, "fs2_bigvgan: weights not loaded (fs2_bigvgan_load)");
  FS2_REQUIRE((reinterpret_cast<uintptr_t>(mels) & 15) == 0, "fs2_bigvgan: mels must be 16-byte aligned");
  int rc = check_size(m->math_mode, B, Lmax);
  if (rc) return rc;
  Bump b(ws, ws_bytes);
  BvPlan p = plan(b, m->sh, B, Lmax);
  if ((rc = b.check("fs2_bigvgan"))) return rc;
  return generate(m, p, mels, olens, nullptr, B, Lmax, 0, audio, (long)Lmax * kHop, status, (cudaStream_t)stream);
}

int fs2_bigvgan_window_workspace_bytes(fs2_bigvgan_gen* m, int B, int n_frames, size_t* bytes) {
  FS2_REQUIRE(m && bytes, "fs2_bigvgan_window_workspace_bytes: null argument");
  int rc = check_window_rows("fs2_bigvgan_window", m->sh.ups, B, n_frames, m->math_mode);
  if (rc) return rc;
  Bump b(nullptr, 0);
  window_plan(b, m->sh, B, n_frames);
  *bytes = b.off + 256;
  return FS2_OK;
}

int fs2_bigvgan_window(fs2_bigvgan_gen* m, const float* mels, const int64_t* olens, const int64_t* starts, int B, int Lmax, int n_frames,
                       float* audio, int64_t audio_ld, int* status, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(m && mels && olens && starts && audio && status && ws, "fs2_bigvgan_window: null argument");
  FS2_REQUIRE((reinterpret_cast<uintptr_t>(mels) & 15) == 0, "fs2_bigvgan_window: mels must be 16-byte aligned");
  int rc = check_window_rows("fs2_bigvgan_window", m->sh.ups, B, n_frames, m->math_mode);
  if (rc) return rc;
  if ((rc = check_window_extent("fs2_bigvgan_window", Lmax, 0, kHop, n_frames, audio_ld))) return rc;
  Bump b(ws, ws_bytes);
  BvPlan p = window_plan(b, m->sh, B, n_frames);
  if ((rc = b.check("fs2_bigvgan_window"))) return rc;
  FS2_REQUIRE(m->loaded, "fs2_bigvgan_window: weights not loaded (fs2_bigvgan_load)");
  return generate(m, p, mels, olens, starts, B, Lmax, n_frames, audio, audio_ld, status, (cudaStream_t)stream);
}

// ---- single layers on the vocoder's own code paths (tests) ----------------------------------------------------------
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
      !(rc = act(kind, xp, prm, lens, nullptr, B, Lp, Cp, 0, a, status, st))) {
    const float* rows32 = (const float*)a;
    if (kind != OUT_F32) rc = planes_to_rows((const __half*)a, rows * Cp, y, st), rows32 = y;
    if (!rc) rc = pad3(rows32, (int)rows, Cp, 1, out, (int)rows, C, st);
  }
  cudaFreeAsync(base, st);
  return rc;
}

int fs2_op_bigvgan_resblock(int math_mode, int type, int C, int k, int nd, const int* dils, const float* x, const int64_t* lens, int B,
                            int Lp, const float* const* weights, const float* const* biases, const float* const* acts, int snakebeta,
                            int logscale, float* out, int* status, void* stream) {
  const char* who = "fs2_op_bigvgan_resblock";
  FS2_REQUIRE(math_mode >= FS2_MATH_FP32 && math_mode <= FS2_MATH_F16, "%s: bad math_mode %d", who, math_mode);
  FS2_REQUIRE(type == 1 || type == 2, "%s: type must be 1 or 2 (got %d)", who, type);
  FS2_REQUIRE(C >= 32 && C % 32 == 0, "%s: C must be a multiple of 32 (got %d)", who, C);
  FS2_REQUIRE(k >= 1 && k <= 31 && k % 2 == 1, "%s: k must be odd, in [1, 31] (got %d)", who, k);
  FS2_REQUIRE(nd == (type == 1 ? 3 : 2), "%s: nd must be %d for type %d (got %d)", who, type == 1 ? 3 : 2, type, nd);
  FS2_REQUIRE(dils && x && lens && weights && biases && acts && out && status, "%s: null argument", who);
  for (int i = 0; i < nd; ++i) FS2_REQUIRE(dils[i] >= 1 && dils[i] <= 1024, "%s: dilation %d out of [1, 1024]", who, dils[i]);
  const int per = type == 1 ? 6 : 2;
  for (int i = 0; i < per; ++i)
    FS2_REQUIRE(weights[i] && biases[i] && acts[4 * i] && (acts[4 * i + 1] || !snakebeta) && acts[4 * i + 2] && acts[4 * i + 3],
                "%s: null argument", who);
  FS2_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 31) == 0,
              "%s: x must be 16-byte and out 32-byte aligned", who);
  FS2_REQUIRE(B >= 1 && Lp >= 1, "%s: bad shape B=%d Lp=%d", who, B, Lp);
  const long rows = (long)B * Lp;
  FS2_REQUIRE(rows * C < (1L << 31) && (math_mode != FS2_MATH_FP32 || rows <= kTapGemmFp32MaxRows), "%s: too many rows (%ld)", who, rows);
  cudaStream_t st = (cudaStream_t)stream;
  VWeight w[6];
  float* prm[6] = {};
  for (int i = 0; i < per; ++i) set_conv(w[i], C, C, k);
  void* a = nullptr;
  float* t[2] = {nullptr, nullptr};
  void* base = nullptr;
  int rc = temp_carve(&base, st, [&](Bump& b) {
    for (int i = 0; i < per; ++i) vweight_carve(b, w[i], true);
    for (int i = 0; i < per; ++i) prm[i] = b.floats(act_params(C));
    a = b.floats((size_t)rows * C);
    t[0] = b.floats((size_t)rows * C);
    t[1] = b.floats((size_t)rows * C);
  });
  if (rc) return rc;
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  for (int i = 0; i < per && !rc; ++i) rc = vweight_pack_conv(w[i], weights[i], biases[i], C, C, k, 0, (long)C * C, st);
  for (int i = 0; i < per && !rc; ++i) rc = act_param(acts + 4 * i, C, logscale, snakebeta, prm[i], st);
  if (!rc) rc = resblock(math_mode, type, w, prm, dils, x, lens, nullptr, B, Lp, C, 0, a, t, out, status, st);
  cudaFreeAsync(base, st);
  return rc;
}

}  // extern "C"
