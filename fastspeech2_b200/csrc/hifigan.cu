// Batched HiFi-GAN, iSTFTNet and BigVGAN vocoders (DESIGN.md sections 16, 18 and 19): log-mels [B, Lmax, 80] -> audio
// [B, Lmax * 256], each utterance the generator over its own olens[b] frames, on the library's tap-GEMM.  The three are
// one generator chain, driven here: conv_pre, U polyphase upsamplings, MRFs of ResBlock1 / ResBlock2 blocks, and a head.
// They differ in three places: the activation before each block convolution (lrelu(x, 0.1), or BigVGAN's
// Activation1d(Snake / SnakeBeta), bigvgan.cu), the producer before each upsampling (the lrelu of the MRF combine, or
// BigVGAN's plain combine), and the head (conv_post + tanh; iSTFTNet's inverse STFT, istftnet.cu; or BigVGAN's
// Activation1d + conv_post + tanh or clamp, bigvgan.cu).  This file holds the chain's kernels, its plan and weights, and
// the C entries of all three.
//
// Stage s (s = 0 .. U, U = num_upsamples) has Lp_s = Lmax * up_s rows per utterance (up_0 = 1, up_{s+1} = up_s * u_s) of
// C'_s = ceil32(C_s) channels, C_s = C0 / 2^s, and every GEMM of the stage runs with TapGemm::lens = lens_s = olens * up_s:
// row tiles wholly past an utterance are skipped and padded rows come out as exact zeros.  Every convolution is "same"
// with zero padding at the utterance's own edges, which is exactly what the tap GEMM's native taps give when the operand's
// rows past lens_s are zeros: the TMA unit zero-fills rows outside [0, Lp_s), and the producers below write every row, +0
// past lens_s.  HiFi-GAN's and iSTFTNet's widths are multiples of 32 (C' = C); a BigVGAN width that is not (the 22 kHz
// large models end at 24) runs zero-padded: its weights get zero rows and columns and its padded output channels a zero
// bias, so the padded channels stay exactly 0 through every layer (Snake(0) = 0).
//
//   mel operand   mel rows (0 past olens)                                       -> GEMM 7 taps, 80 -> C0    = conv_pre
//   per stage s:
//     rows        lrelu(x, 0.1) (BigVGAN: x), x = the previous MRF's ((r0 + r1) + ...) / nk -> GEMM 3 taps, C'_s -> u C'_{s+1}:
//                 the ConvTranspose1d(k = 2u, stride u, pad u / 2) as a polyphase GEMM.  Output row t's u phases, written
//                 row-major, are rows u t .. u t + u - 1 of the next stage; phase r < u/2 reads input rows {t-1, t}, r >= u/2
//                 reads {t, t+1}, and the third tap of each phase has zero weights.  Native taps rather than MelGAN's
//                 producer-stacked K = 3 Cin operand: the producer writes Cin values per row instead of 3 Cin.
//     per resblock j of the MRF, per conv step m (ResBlock1: x = c2(a(c1(a(x)))) + x; ResBlock2: x = c(a(x)) + x, a =
//                 lrelu(., 0.1) or an Activation1d): act a(x) -> GEMM k taps at dilation d_m (-> act -> GEMM k taps,
//                 dilation 1), the residual add in the last GEMM's epilogue (TapGemm::resid)
//     add         S += r_j for the middle resblocks (1 .. nk - 2): the MRF sum in hifi-gan's order
//   head          HiFi-GAN: lrelu((S + r_last) / nk, 0.01), conv C -> 1 (k = 7, zero padding), tanh, on CUDA cores, +0
//                 past olens * 256 (hifigan_post_kernel); iSTFTNet: istftnet_head; BigVGAN: bigvgan_post
//
// Launches per call: 4 + U * (2 + nk * G + max(nk - 2, 0)), G = 12 (ResBlock1: 3 steps of 2 producers + 2 GEMMs) or 4
// (ResBlock2: 2 steps of 1 + 1), in every math mode: 160 for HiFi-GAN V1 and BigVGAN base, 49 for V3, 82 for iSTFTNet
// C8C8I, 238 for BigVGAN's large models.
//
// Buffers, each [B * Lp_s][C'_s] at the current stage, so A floats per frame with A = max_s up_s * C'_s (8192 for V1 and
// V3): xu (the upsampling output every resblock of the MRF reads), S (r0, then the running sum), two chain buffers T0 / T1
// (a resblock's intermediate x and h; the last resblock ends in one of them, which the next producer combines with S), and
// the GEMM operand (fp32 rows, or hi + lo fp16 planes: the same bytes).  5 * 4 * A bytes per frame of B * Lmax: 163,840
// for V1 and V3.
//
// A GEMM row depends only on its own utterance's input rows, in a fixed K order, and every producer reads rows of its own
// utterance below lens_s only, so per-utterance results do not depend on the batch.
//
// Windows (fs2_<name>_window, DESIGN.md section 17): the same kernels and GEMMs on a window of each utterance's rows, on
// the chain plan of vocoder_window.cuh with R = the largest resblock's reach (BigVGAN's including its activations: AMPBlock1
// sum_m ((k-1)/2 (d_m + 1) + 2 a), AMPBlock2 sum_m ((k-1)/2 d_m + a), a = kAct = 5), level-0 margin 3 (conv_pre's native
// taps read level-0 rows outside the window), the head's reach (3; istft_reach; 3 + a) and no tail.  For the core frames
// [c0, c1), level s holds global rows [c0 up_s - h_s, c1 up_s + h_s) clipped to [0, olens up_s), in a buffer of n up_s +
// 2 h_s rows per utterance; upsampling s reads its input window [c0 up_s - r_s, c1 up_s + r_s) (clipped) out of level s.
// Every GEMM runs with lens = the clipped length, so the rows-past-lens and zero-fill rules above give each convolution
// its padding wherever a buffer side is an utterance edge.  A window descriptor [start | len | n] x B per buffer (nullptr
// = the whole utterance: start 0, len = n = lens[b]) maps local rows to global ones, and producers range-check only rows
// whose values equal the whole call's (exact_row): the margin widens by each convolution's reach and by a at each
// Activation1d.
#include <math.h>

#include <algorithm>
#include <vector>

#include "bigvgan.cuh"
#include "istftnet.cuh"
#include "vocoder_weights.cuh"
#include "vocoder_window.cuh"

namespace fs2 {
namespace {

constexpr int kMels = 80, kHop = 256, kPreTaps = 7, kPostTaps = 7;
constexpr float kSlope = 0.1f, kPostSlope = 0.01f;   // hifi-gan's LRELU_SLOPE, and F.leaky_relu's default before conv_post

__device__ __forceinline__ float lrelu(float v, float s) { return v > 0.f ? v : v * s; }

// A GEMM operand [B * Lp][C] = a(v) with v = x, or the MRF combine v = (x + r) / nk (r nullable: x / nk), and a =
// lrelu(., 0.1) (LRELU) or none, for t < lens[b]; +0 past it.  Every row is written: the next GEMM's taps read rows past
// lens[b] as its zero padding.  It writes conv_pre's operand (x = the mels, ldx = Lmax, C = 80), every upsampling's, and
// the lrelu before every HiFi-GAN block convolution.  A window (WINDOW, win != nullptr): the operand's rows are window
// win, and local row t of utterance b reads x's row b * ldx + t + start - xwin[b], x holding ldx rows per utterance of its
// own window xwin (nullptr: x holds global rows, the mels); only rows exact_row(margin) are range-checked (margin 0:
// every row, since exact_row(w, t, 0) holds for every t < len).
template <int OUT, bool LRELU, bool WINDOW>
__device__ __forceinline__ void act_loop(const float* __restrict__ x, const float* __restrict__ r, int nk, const int64_t* __restrict__ lens,
                                         const int64_t* __restrict__ xwin, int ldx, const int64_t* __restrict__ win, int B, int Lp, int C,
                                         int margin, float* __restrict__ out32, __half* __restrict__ outp, int* __restrict__ status) {
  const int Q = C / 4;
  const long rows = (long)B * Lp, total = rows * Q, plane = rows * C;
  const float fk = (float)nk;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / Q;
    const int b = (int)(row / Lp), t = (int)(row - (long)b * Lp);
    const int c = (int)(i - row * Q) * 4;
    const long off = row * C + c;
    const Rows w = rows_of(WINDOW ? win : nullptr, lens, B, b);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t < w.len) {
      const long src = WINDOW ? ((long)b * ldx + t + w.start - (xwin ? (int)xwin[b] : 0)) * C + c : off;
      v = *reinterpret_cast<const float4*>(x + src);
      if (r) {
        const float4 u = *reinterpret_cast<const float4*>(r + src);
        v = make_float4(v.x + u.x, v.y + u.y, v.z + u.z, v.w + u.w);
      }
      if (nk != 1) v = make_float4(v.x / fk, v.y / fk, v.z / fk, v.w / fk);
      if (LRELU) v = make_float4(lrelu(v.x, kSlope), lrelu(v.y, kSlope), lrelu(v.z, kSlope), lrelu(v.w, kSlope));
    }
    store_quad<OUT, RANGE_IF_STATUS>(v, off, out32, outp, plane, !WINDOW || exact_row(w, t, margin) ? status : nullptr,
                                     FS2_HIFIGAN_RANGE);
  }
}

template <int OUT, bool LRELU>
__global__ void hifigan_act_kernel(const float* __restrict__ x, const float* __restrict__ r, int nk, const int64_t* __restrict__ lens,
                                   const int64_t* __restrict__ xwin, int ldx, const int64_t* __restrict__ win, int B, int Lp, int C,
                                   int margin, float* __restrict__ out32, __half* __restrict__ outp, int* __restrict__ status) {
  if (win) act_loop<OUT, LRELU, true>(x, r, nk, lens, xwin, ldx, win, B, Lp, C, margin, out32, outp, status);
  else act_loop<OUT, LRELU, false>(x, r, nk, lens, xwin, ldx, win, B, Lp, C, margin, out32, outp, status);
}

// s[i] += r[i] over n floats (n a multiple of 4): the MRF's running sum; rows past lens are +0 in both
__global__ void hifigan_add_kernel(float* __restrict__ s, const float* __restrict__ r, long n) {
  for (long i = ((long)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < n; i += (long)gridDim.x * blockDim.x * 4) {
    float4 a = *reinterpret_cast<const float4*>(s + i);
    const float4 b = *reinterpret_cast<const float4*>(r + i);
    *reinterpret_cast<float4*>(s + i) = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
  }
}

// audio[b, t] = tanh(bias + sum_j sum_c w[j][c] lrelu(x[t + j - 3][c], 0.01)) for t < lens[b], else +0, where x = (S + R) / nk
// (R nullable) is the last MRF's output, 0 outside [0, lens[b]).  w: [7][C] in dynamic shared memory.  x has Lx rows per
// utterance in window win (nullptr: the whole utterance), audio Lout samples per row, rows ld apart.  A window: audio row b
// holds samples [start, start + len) of awin, +0 past them.
__global__ void __launch_bounds__(256) hifigan_post_kernel(const float* __restrict__ S, const float* __restrict__ R, int nk,
                                                           const int64_t* __restrict__ lens, const int64_t* __restrict__ win,
                                                           const int64_t* __restrict__ awin, int B, int Lx, int Lout, long ld, int C,
                                                           const float* __restrict__ w, const float* __restrict__ bias,
                                                           float* __restrict__ audio) {
  extern __shared__ __align__(16) float ws[];
  for (int i = threadIdx.x; i < kPostTaps * C; i += blockDim.x) ws[i] = w[i];
  __syncthreads();
  const float b0 = __ldg(bias), fk = (float)nk;
  const long total = (long)B * Lout;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int b = (int)(i / Lout), t = (int)(i - (long)b * Lout);
    const Rows r = rows_of(win, lens, B, b);
    const int a0 = awin ? (int)awin[b] : 0, n = awin ? (int)awin[B + b] : r.n;
    float y = 0.f;
    if (t < n) {
      float acc = b0;
#pragma unroll 1
      for (int j = 0; j < kPostTaps; ++j) {
        const int src = a0 + t + j - kPostTaps / 2;
        if (src < 0 || src >= r.n) continue;
        const long row = ((long)b * Lx + src - r.start) * C;
        for (int q = 0; q < C / 4; ++q) {
          float4 v = __ldg(reinterpret_cast<const float4*>(S + row) + q);
          if (R) {
            const float4 r = __ldg(reinterpret_cast<const float4*>(R + row) + q);
            v = make_float4(v.x + r.x, v.y + r.y, v.z + r.z, v.w + r.w);
          }
          if (nk != 1) v = make_float4(v.x / fk, v.y / fk, v.z / fk, v.w / fk);
          const float4 wv = *reinterpret_cast<const float4*>(ws + j * C + 4 * q);
          acc = fmaf(wv.x, lrelu(v.x, kPostSlope), acc);
          acc = fmaf(wv.y, lrelu(v.y, kPostSlope), acc);
          acc = fmaf(wv.z, lrelu(v.z, kPostSlope), acc);
          acc = fmaf(wv.w, lrelu(v.w, kPostSlope), acc);
        }
      }
      y = tanhf(acc);
    }
    audio[(long)b * ld + t] = y;
  }
}

// ---- host side ------------------------------------------------------------------------------------------------------

// what a config implies: widths, cumulative upsampling, convolutions and activations per resblock and in all
struct Shape {
  int U, nk, type, steps, per;         // upsamplings, resblocks per MRF, resblock type, conv steps and convolutions per resblock
  int C[kMaxUps + 1], Cp[kMaxUps + 1]; // stage widths C0 / 2^s and their operand widths ceil32
  UpsPlan ups;
  int layers, nact;                    // convolutions and Activation1d's (0 with lrelu) in state_dict order
  long act;                            // floats per frame of the largest stage buffer, max_s up_s * C'_s
};

// act_reach: an activation's reach, kAct for Activation1d and 0 for lrelu; post: the head's last-layer reach
Shape shape_of(const fs2_hifigan_config& c, int act_reach, int post) {
  Shape s;
  s.U = c.num_upsamples; s.nk = c.num_kernels; s.type = c.resblock;
  s.steps = s.type == 1 ? 3 : 2; s.per = s.type == 1 ? 6 : 2;
  int R = 0;                                           // the MRF's reach: the largest resblock's, activations included
  for (int j = 0; j < s.nk; ++j) {
    int r = 0;
    for (int m = 0; m < s.steps; ++m)
      r += (c.resblock_kernel_sizes[j] - 1) / 2 * (c.resblock_dilation_sizes[j][m] + (s.type == 1)) + (s.type == 1 ? 2 : 1) * act_reach;
    R = std::max(R, r);
  }
  // the window plan: conv_pre's native taps leave its outer 3 rows wrong at a side that is not an utterance edge; no tail
  s.ups = ups_plan(s.U, c.upsample_rates, R, kPreTaps / 2, post, 0);
  s.C[0] = c.upsample_initial_channel;
  s.Cp[0] = ceil32(s.C[0]);
  s.act = s.Cp[0];
  for (int i = 0; i < s.U; ++i) {
    s.C[i + 1] = s.C[i] / 2;
    s.Cp[i + 1] = ceil32(s.C[i + 1]);
    s.act = std::max(s.act, (long)s.ups.up[i + 1] * s.Cp[i + 1]);
  }
  s.layers = 2 + s.U + s.U * s.nk * s.per;
  s.nact = act_reach ? s.U * s.nk * s.per + 1 : 0;     // one per block convolution, then activation_post
  return s;
}

// multiple: what every width C0 / 2^i must be a multiple of (32; BigVGAN's padded widths 8); hop: the head's (1 for
// conv_post), so that the rates' product times hop is the frame hop 256
int validate(const fs2_hifigan_config* c, const char* who, int multiple, int hop) {
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
  if (hop == 1) FS2_REQUIRE(prod == kHop, "%s: the product of upsample_rates is %ld, not the hop 256", who, prod);
  else FS2_REQUIRE(prod * hop == kHop, "%s: the product of upsample_rates (%ld) times istft_hop (%d) is %ld, not the hop 256", who, prod, hop,
                   prod * hop);
  const int C0 = c->upsample_initial_channel;
  FS2_REQUIRE(C0 >= multiple && C0 <= 2048 && C0 % (multiple << c->num_upsamples) == 0,
              "%s: upsample_initial_channel = %d must lie in [%d, 2048] with every width C0 / 2^i a multiple of %d", who, C0, multiple,
              multiple);
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
  return FS2_OK;
}

// the rows producer (x, r, nk, xwin, ldx, win, margin as in hifigan_act_kernel), through lrelu or not, into the operand a
int act(int kind, bool lrelu, const float* x, const float* r, int nk, const int64_t* lens, const int64_t* xwin, int ldx, const int64_t* win,
        int B, int Lp, int C, int margin, void* a, int* status, cudaStream_t st) {
  auto k = lrelu ? pick(kind, hifigan_act_kernel<OUT_HILO, true>, hifigan_act_kernel<OUT_HI, true>, hifigan_act_kernel<OUT_F32, true>)
                 : pick(kind, hifigan_act_kernel<OUT_HILO, false>, hifigan_act_kernel<OUT_HI, false>, hifigan_act_kernel<OUT_F32, false>);
  k<<<grid_for((long)B * Lp * (C / 4), 256), 256, 0, st>>>(x, r, nk, lens, xwin, ldx, win, B, Lp, C, margin, (float*)a, (__half*)a, status);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// (lrelu +) ConvTranspose1d: x [B * Lin][Cin] (combined with r / nk) -> out [B * Lin][u Cout] = [B * Lin * u][Cout] through
// the operand a; rows >= lens[b] * u of out written as +0.  A window: the input window (win, lens; Lin rows per
// utterance) is read from x's own window xwin of ldx rows per utterance.  Every row it reads holds the whole call's
// values, so all are range-checked.
int upsample(int mode, bool lrelu, const VWeight& w, const float* x, const float* r, int nk, const int64_t* xwin, int ldx, const int64_t* lens,
             const int64_t* win, int B, int Lin, int Cin, void* a, float* out, int* status, cudaStream_t st) {
  int rc = act(out_kind(mode), lrelu, x, r, nk, lens, xwin, ldx, win, B, Lin, Cin, 0, a, status, st);
  return rc ? rc : vweight_gemm(mode, w, a, B, Lin, ACT_NONE, lens, out, st);
}

// One residual block x -> dest on rows [B * Lp][C]: w = its convolutions in state_dict order, prm its Activation1d's
// (nullptr: lrelu), dil its dilations.  Step m writes t[m & 1], the last one dest; dest must differ from x and from the
// buffer the last step reads (t[(steps - 2) & 1]).  win (nullable): the rows' window; margin: its rows at a side that is
// not an utterance edge whose values differ from the whole call's on entry, widened here by kAct at each Activation1d
// and by each convolution's reach.
int resblock(int mode, int type, const VWeight* w, const float* const* prm, const int* dil, const float* x, const int64_t* lens,
             const int64_t* win, int B, int Lp, int C, int margin, void* a, float* const* t, float* dest, int* status, cudaStream_t st) {
  const int steps = type == 1 ? 3 : 2, kind = out_kind(mode), half = (w[0].taps - 1) / 2, reach = prm ? kAct : 0;
  // activation i of the block on v, rows exact_row(margin) range-checked
  auto activate = [&](const float* v, int i) {
    margin += reach;
    return prm ? bigvgan_act(kind, v, prm[i], lens, win, B, Lp, C, margin, a, status, st)
               : act(kind, true, v, nullptr, 1, lens, win, Lp, win, B, Lp, C, margin, a, status, st);
  };
  const float* X = x;
  int rc;
  for (int m = 0; m < steps; ++m) {
    float* out = m == steps - 1 ? dest : t[m & 1];
    if ((rc = activate(X, type == 1 ? 2 * m : m))) return rc;
    margin += half * dil[m];
    if (type == 1) {
      if ((rc = vweight_gemm(mode, w[m], a, B, Lp, ACT_NONE, lens, out, st, nullptr, dil[m]))) return rc;   // h = c1(a1(x))
      if ((rc = activate(out, 2 * m + 1))) return rc;
      margin += half;
      if ((rc = vweight_gemm(mode, w[3 + m], a, B, Lp, ACT_NONE, lens, out, st, X, 1))) return rc;        // c2(a2(h)) + x
    } else {
      if ((rc = vweight_gemm(mode, w[m], a, B, Lp, ACT_NONE, lens, out, st, X, dil[m]))) return rc;       // c(a(x)) + x
    }
    X = out;
  }
  return FS2_OK;
}

struct HgPlan {
  int64_t* lens;      // [U + 1][B]; a window call: the n_wins(sh.ups) window descriptors [start | len | n][B]
  void* a;            // GEMM operand
  float* xu;          // the upsampling output of the current stage
  float* s;           // MRF sum
  float* t[2];        // chain buffers
};

HgPlan carve_plan(Bump& b, size_t lens_bytes, size_t n) {
  HgPlan p;
  p.lens = (int64_t*)b.bytes(lens_bytes);
  p.a = b.floats(n);
  p.xu = b.floats(n);
  p.s = b.floats(n);
  p.t[0] = b.floats(n);
  p.t[1] = b.floats(n);
  return p;
}

// a GEMM weight here is [taps][N][K] tap matrices with K = Cin, so vweight_pack_conv packs it at tap_stride = N K
void set_conv(VWeight& w, int N, int K, int taps) { w.N = N; w.K = K; w.taps = taps; }

// w (K = C'in, N = C'out, or u C'out rows for a polyphase upsampling) from a torch-layout weight [A][Bn][k] and bias
// [Cout] of real widths Cin / Cout: vweight_pack_conv, on a copy zero-padded to w's widths in a stream-ordered temporary
// when they differ
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

enum Head { kHeadPost, kHeadIstft, kHeadActPost };   // conv_post + tanh, iSTFTNet's inverse STFT, BigVGAN's activation_post + conv_post

}  // namespace
}  // namespace fs2

struct fs2_hifigan_gen {
  int device = 0, math_mode = 0;
  fs2_hifigan_config cfg;
  fs2::Shape sh;
  bool snake = false;              // Activation1d(Snake / SnakeBeta) before every block convolution and none before the
                                   // upsamplings (BigVGAN), else lrelu(x, 0.1) before both
  fs2::Head head = fs2::kHeadPost;
  int n_fft = 0, head_hop = 1;     // iSTFTNet's istft_n_fft, istft_hop; 0, 1 for the other heads
  int beta = 0, logscale = 0;      // BigVGAN: SnakeBeta, snake_logscale
  int use_tanh = 1, use_bias = 1;  // the head: tanh (else a clamp to [-1, 1]); conv_post has a bias
  bool loaded = false;
  void* arena = nullptr; size_t arena_bytes = 0;
  fs2::VWeight pre, up[fs2::kMaxUps];
  std::vector<fs2::VWeight> blk;   // [U * nk][per]: the resblocks' convolutions in state_dict order
  std::vector<float*> prm;         // [sh.nact]: the Activation1d's parameters in state_dict order, activation_post last
  float* post_w = nullptr;         // conv_post [7][O][C'_U], O = 1, or iSTFTNet's n_fft + 2
  float* post_b = nullptr;         // [O]; nullptr without use_bias
};

struct fs2_istftnet_gen : fs2_hifigan_gen {};
struct fs2_bigvgan_gen : fs2_hifigan_gen {};

namespace fs2 {
namespace {

// The generator on the plan p: whole utterances (starts == nullptr; level s has L up_s rows per utterance, lens [U + 1][B])
// or a window of nf frames from starts[b] (level_rows / ups_rows per utterance, the n_wins(sh.ups) window descriptors).  Lout
// audio samples per row, rows ld apart.  Both enqueue the same kernels.
int generate(const fs2_hifigan_gen* m, const HgPlan& p, const float* mels, const int64_t* olens, const int64_t* starts, int B, int L,
             int nf, float* audio, long ld, int* status, cudaStream_t st) {
  const Shape& sh = m->sh;
  const bool w = starts != nullptr;
  const int mode = m->math_mode, kind = out_kind(mode), U = sh.U;
  auto desc = [&](int i) -> const int64_t* { return w ? p.lens + 3L * i * B : nullptr; };
  auto lens = [&](int i, int s) -> const int64_t* { return w ? p.lens + (3L * i + 1) * B : p.lens + (long)s * B; };   // window i / level s
  auto rows = [&](int s) { return w ? (int)level_rows(sh.ups, s, nf) : L * sh.ups.up[s]; };
  int rc = ups_prep(olens, starts, B, 1, L, nf, sh.ups, p.lens, status, st);
  if (rc) return rc;
  if ((rc = act(kind, false, mels, nullptr, 1, lens(win_level(0), 0), nullptr, L, desc(win_level(0)), B, rows(0), kMels, 0, p.a, status, st)))
    return rc;
  if ((rc = vweight_gemm(mode, m->pre, p.a, B, rows(0), ACT_NONE, lens(win_level(0), 0), p.t[0], st))) return rc;
  // the stage input: conv_pre's output, then each MRF's (S + r) / nk
  const float* x = p.t[0];
  const float* r = nullptr;
  int nk_in = 1;
  for (int s = 0; s < U; ++s) {
    const int Lin = w ? (int)ups_rows(sh.ups, s, nf) : rows(s), Lp = rows(s + 1), C = sh.Cp[s + 1];
    const int uw = win_ups(sh.ups, s), lw = win_level(s + 1);
    if ((rc = upsample(mode, !m->snake, m->up[s], x, r, nk_in, desc(win_level(s)), rows(s), lens(uw, s), desc(uw), B, Lin, sh.Cp[s], p.a,
                       p.xu, status, st)))
      return rc;
    const int margin = m->cfg.upsample_rates[s] / 2;   // the rows the edge phases leave wrong at a side that is not an edge
    float* last = p.s;
    for (int j = 0; j < sh.nk; ++j) {
      const int g = s * sh.nk + j;
      last = j == 0 ? p.s : p.t[(sh.steps - 1) & 1];
      if ((rc = resblock(mode, sh.type, &m->blk[(size_t)g * sh.per], m->snake ? &m->prm[(size_t)g * sh.per] : nullptr,
                         m->cfg.resblock_dilation_sizes[j], p.xu, lens(lw, s + 1), desc(lw), B, Lp, C, margin, p.a, p.t, last, status, st)))
        return rc;
      if (j >= 1 && j < sh.nk - 1) {
        hifigan_add_kernel<<<grid_for((long)B * Lp * C / 4, 256), 256, 0, st>>>(p.s, last, (long)B * Lp * C);
        FS2_LAUNCH_CHECK();
      }
    }
    x = p.s;
    r = sh.nk > 1 ? last : nullptr;
    nk_in = sh.nk;
  }
  const int Lout = (w ? nf : L) * kHop, C = sh.Cp[U];
  const int64_t *lens_U = lens(win_level(U), U), *win_U = desc(win_level(U)), *awin = desc(win_audio(sh.ups));
  if (m->head == kHeadIstft)
    return istftnet_head(x, r, nk_in, lens_U, win_U, awin, B, rows(U), Lout, ld, C, m->n_fft, m->head_hop, m->post_w, m->post_b, audio, st);
  if (m->head == kHeadActPost)
    return bigvgan_post(x, r, nk_in, lens_U, win_U, awin, B, rows(U), Lout, ld, C, m->prm.back(), m->post_w, m->post_b, m->use_tanh, audio,
                        st);
  hifigan_post_kernel<<<grid_for((long)B * Lout, 256), 256, kPostTaps * C * sizeof(float), st>>>(
      x, r, nk_in, lens_U, win_U, awin, B, rows(U), Lout, ld, C, m->post_w, m->post_b, audio);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// the generator's side of the shared C entries (vocoder_window.cuh)
struct HgEntry {
  using Gen = fs2_hifigan_gen;
  static const UpsPlan& ups(const Gen* m) { return m->sh.ups; }
  static HgPlan plan(Bump& b, const Gen* m, int B, int L) {
    return carve_plan(b, (size_t)(m->sh.U + 1) * B * sizeof(int64_t), (size_t)B * L * m->sh.act);
  }
  // A window call's workspace, from B and nf only: five buffers of the largest level buffer per utterance (rows x C' over
  // every level; conv_pre's operand, 80 wide, and the upsamplings' operands, r_s <= h_s, fit in it)
  static HgPlan window_plan(Bump& b, const Gen* m, int B, int nf) {
    const Shape& sh = m->sh;
    long act = level_rows(sh.ups, 0, nf) * kMels;
    for (int s = 0; s <= sh.U; ++s) act = std::max(act, level_rows(sh.ups, s, nf) * sh.Cp[s]);
    return carve_plan(b, (size_t)3 * n_wins(sh.ups) * B * sizeof(int64_t), (size_t)B * act);
  }
  static constexpr auto generate = fs2::generate;
};

// A handle for a validated config with the given head (n_fft, hop: iSTFTNet's; 0, 1 otherwise) and activation
template <typename Gen>
int create_gen(Gen** out, int math_mode, const fs2_hifigan_config* cfg, Head head, int n_fft, int hop, bool snake) {
  int dev = 0;
  FS2_CUDA_CHECK(cudaGetDevice(&dev));
  Gen* m = new Gen();
  m->math_mode = math_mode;
  m->device = dev;
  m->cfg = *cfg;
  m->head = head;
  m->snake = snake;
  m->n_fft = n_fft;
  m->head_hop = hop;
  const int post = head == kHeadIstft ? istft_reach(n_fft, hop) : head == kHeadActPost ? kPostTaps / 2 + kAct : kPostTaps / 2;
  m->sh = shape_of(*cfg, snake ? kAct : 0, post);
  const Shape& sh = m->sh;
  set_conv(m->pre, sh.Cp[0], kMels, kPreTaps);
  for (int s = 0; s < sh.U; ++s) set_conv(m->up[s], cfg->upsample_rates[s] * sh.Cp[s + 1], sh.Cp[s], 3);
  m->blk.resize((size_t)sh.U * sh.nk * sh.per);
  for (int s = 0; s < sh.U; ++s)
    for (int j = 0; j < sh.nk; ++j)
      for (int i = 0; i < sh.per; ++i)
        set_conv(m->blk[((size_t)s * sh.nk + j) * sh.per + i], sh.Cp[s + 1], sh.Cp[s + 1], cfg->resblock_kernel_sizes[j]);
  m->prm.assign(sh.nact, nullptr);
  *out = m;
  return FS2_OK;
}

// acts: the Activation1d's tensors, 4 per activation (read with m->snake only); name: "fs2_<vocoder>", the prefix of every
// message
int load_gen(fs2_hifigan_gen* m, const float* const* weights, const float* const* biases, const float* const* acts, void* stream,
             const char* name) {
  FS2_REQUIRE(m && weights && biases && (acts || !m->snake), "%s_load: null argument", name);
  const Shape& sh = m->sh;
  const int last = sh.layers - 1;
  for (int i = 0; i < sh.layers; ++i)
    FS2_REQUIRE(weights[i] && (biases[i] || (i == last && !m->use_bias)), "%s_load: layer %d: null tensor", name, i);
  for (int i = 0; i < sh.nact; ++i)
    FS2_REQUIRE(acts[4 * i] && (acts[4 * i + 1] || !m->beta) && acts[4 * i + 2] && acts[4 * i + 3], "%s_load: activation %d: null tensor",
                name, i);
  cudaStream_t st = (cudaStream_t)stream;
  const int O = m->head == kHeadIstft ? m->n_fft + 2 : 1;   // conv_post's output channels
  m->loaded = false;
  auto width = [&](int i) { return i == sh.nact - 1 ? sh.C[sh.U] : sh.C[i / (sh.nk * sh.per) + 1]; };   // activation i's channels
  int rc = arena_carve(&m->arena, &m->arena_bytes, st, [&](Bump& b) {
    vweight_carve(b, m->pre, true);
    for (int s = 0; s < sh.U; ++s) vweight_carve(b, m->up[s], true);
    for (auto& w : m->blk) vweight_carve(b, w, true);
    for (int i = 0; i < sh.nact; ++i) m->prm[i] = b.floats(act_params(ceil32(width(i))));
    m->post_w = b.floats((size_t)kPostTaps * O * sh.Cp[sh.U]);
    m->post_b = m->use_bias ? b.floats(O) : nullptr;
    return FS2_OK;
  });
  if (rc) return rc;
  if ((rc = pack_conv(m->pre, weights[0], biases[0], kMels, sh.C[0], kPreTaps, 0, st))) return rc;
  for (int s = 0; s < sh.U; ++s)
    if ((rc = pack_conv(m->up[s], weights[1 + s], biases[1 + s], sh.C[s], sh.C[s + 1], 3, m->cfg.upsample_rates[s], st))) return rc;
  for (size_t i = 0; i < m->blk.size(); ++i) {
    const int C = sh.C[i / ((size_t)sh.nk * sh.per) + 1];
    if ((rc = pack_conv(m->blk[i], weights[1 + sh.U + i], biases[1 + sh.U + i], C, C, m->blk[i].taps, 0, st))) return rc;
  }
  for (int i = 0; i < sh.nact; ++i)
    if ((rc = act_param(acts + 4 * i, width(i), m->logscale, m->beta, m->prm[i], st))) return rc;
  const int C = sh.C[sh.U], Cp = sh.Cp[sh.U];
  if (Cp != C) FS2_CUDA_CHECK(cudaMemsetAsync(m->post_w, 0, sizeof(float) * kPostTaps * O * Cp, st));
  if ((rc = conv_pack(weights[last], O, C, kPostTaps, O, 0, (long)O * Cp, Cp, m->post_w, st))) return rc;
  if (m->post_b) FS2_CUDA_CHECK(cudaMemcpyAsync(m->post_b, biases[last], O * sizeof(float), cudaMemcpyDeviceToDevice, st));
  m->loaded = true;
  return FS2_OK;
}

// One residual block on rows [B * Lp][C] (fs2_op_hifigan_resblock; with acts, fs2_op_bigvgan_resblock's AMP block)
int op_resblock(const char* who, int math_mode, int type, int C, int k, int nd, const int* dils, const float* x, const int64_t* lens, int B,
                int Lp, const float* const* weights, const float* const* biases, bool snake, const float* const* acts, int snakebeta,
                int logscale, float* out, int* status, void* stream) {
  FS2_REQUIRE(math_mode >= FS2_MATH_FP32 && math_mode <= FS2_MATH_F16, "%s: bad math_mode %d", who, math_mode);
  FS2_REQUIRE(type == 1 || type == 2, "%s: type must be 1 or 2 (got %d)", who, type);
  FS2_REQUIRE(C >= 32 && C % 32 == 0, "%s: C must be a multiple of 32 (got %d)", who, C);
  FS2_REQUIRE(k >= 1 && k <= 31 && k % 2 == 1, "%s: k must be odd, in [1, 31] (got %d)", who, k);
  FS2_REQUIRE(nd == (type == 1 ? 3 : 2), "%s: nd must be %d for type %d (got %d)", who, type == 1 ? 3 : 2, type, nd);
  FS2_REQUIRE(dils && x && lens && weights && biases && (acts || !snake) && out && status, "%s: null argument", who);
  for (int i = 0; i < nd; ++i) FS2_REQUIRE(dils[i] >= 1 && dils[i] <= 1024, "%s: dilation %d out of [1, 1024]", who, dils[i]);
  const int per = type == 1 ? 6 : 2;
  for (int i = 0; i < per; ++i)
    FS2_REQUIRE(weights[i] && biases[i] &&
                    (!snake || (acts[4 * i] && (acts[4 * i + 1] || !snakebeta) && acts[4 * i + 2] && acts[4 * i + 3])),
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
    for (int i = 0; i < per && snake; ++i) prm[i] = b.floats(act_params(C));
    a = b.floats((size_t)rows * C);
    t[0] = b.floats((size_t)rows * C);
    t[1] = b.floats((size_t)rows * C);
  });
  if (rc) return rc;
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  for (int i = 0; i < per && !rc; ++i) rc = vweight_pack_conv(w[i], weights[i], biases[i], C, C, k, 0, (long)C * C, st);
  for (int i = 0; i < per && snake && !rc; ++i) rc = act_param(acts + 4 * i, C, logscale, snakebeta, prm[i], st);
  if (!rc) rc = resblock(math_mode, type, w, snake ? prm : nullptr, dils, x, lens, nullptr, B, Lp, C, 0, a, t, out, status, st);
  cudaFreeAsync(base, st);
  return rc;
}

static_assert(FS2_ISTFTNET_BAD_LENGTH == FS2_HIFIGAN_BAD_LENGTH && FS2_ISTFTNET_RANGE == FS2_HIFIGAN_RANGE &&
                  FS2_ISTFTNET_BAD_START == FS2_HIFIGAN_BAD_START,
              "iSTFTNet runs HiFi-GAN's kernels, which set HiFi-GAN's status bits");
static_assert(FS2_BIGVGAN_BAD_LENGTH == FS2_HIFIGAN_BAD_LENGTH && FS2_BIGVGAN_RANGE == FS2_HIFIGAN_RANGE &&
                  FS2_BIGVGAN_BAD_START == FS2_HIFIGAN_BAD_START,
              "BigVGAN runs HiFi-GAN's kernels, which set HiFi-GAN's status bits");

}  // namespace
}  // namespace fs2

using namespace fs2;

extern "C" {

int fs2_hifigan_create(fs2_hifigan_gen** out, int math_mode, const fs2_hifigan_config* cfg) {
  const char* who = "fs2_hifigan_create";
  FS2_REQUIRE(out && cfg, "%s: null argument", who);
  FS2_REQUIRE(math_mode >= FS2_MATH_FP32 && math_mode <= FS2_MATH_F16, "%s: bad math_mode %d", who, math_mode);
  int rc = validate(cfg, who, 32, 1);
  return rc ? rc : create_gen(out, math_mode, cfg, kHeadPost, 0, 1, false);
}

void fs2_hifigan_destroy(fs2_hifigan_gen* m) { destroy_gen(m); }

int fs2_hifigan_load(fs2_hifigan_gen* m, const float* const* weights, const float* const* biases, void* stream) {
  return load_gen(m, weights, biases, nullptr, stream, "fs2_hifigan");
}

int fs2_hifigan_workspace_bytes(fs2_hifigan_gen* m, int B, int Lmax, size_t* bytes) {
  return workspace_gen<HgEntry>(m, B, Lmax, bytes, "fs2_hifigan");
}

int fs2_hifigan(fs2_hifigan_gen* m, const float* mels, const int64_t* olens, int B, int Lmax, float* audio, int* status, void* ws,
                size_t ws_bytes, void* stream) {
  return call_gen<HgEntry>(m, mels, olens, B, Lmax, audio, status, ws, ws_bytes, stream, "fs2_hifigan");
}

int fs2_hifigan_window_workspace_bytes(fs2_hifigan_gen* m, int B, int n_frames, size_t* bytes) {
  return window_workspace_gen<HgEntry>(m, B, n_frames, bytes, "fs2_hifigan");
}

int fs2_hifigan_window(fs2_hifigan_gen* m, const float* mels, const int64_t* olens, const int64_t* starts, int B, int Lmax, int n_frames,
                       float* audio, int64_t audio_ld, int* status, void* ws, size_t ws_bytes, void* stream) {
  return window_gen<HgEntry>(m, mels, olens, starts, B, Lmax, n_frames, audio, audio_ld, status, ws, ws_bytes, stream, "fs2_hifigan");
}

int fs2_istftnet_create(fs2_istftnet_gen** out, int math_mode, const fs2_istftnet_config* cfg) {
  const char* who = "fs2_istftnet_create";
  FS2_REQUIRE(out && cfg, "%s: null argument", who);
  FS2_REQUIRE(math_mode >= FS2_MATH_FP32 && math_mode <= FS2_MATH_F16, "%s: bad math_mode %d", who, math_mode);
  const int n = cfg->istft_n_fft, hop = cfg->istft_hop;
  FS2_REQUIRE(n >= 2 && n % 2 == 0, "%s: istft_n_fft = %d must be even and at least 2", who, n);
  FS2_REQUIRE(n <= kIstftMaxNfft, "%s: istft_n_fft = %d is above %d, the most the head kernel's shared memory holds", who, n, kIstftMaxNfft);
  FS2_REQUIRE(hop >= 1 && n % hop == 0 && n / hop >= 2,
              "%s: istft_hop = %d must divide istft_n_fft = %d with istft_n_fft / istft_hop >= 2 (else the window envelope is 0)", who,
              hop, n);
  int rc = validate(&cfg->gen, who, 32, hop);
  return rc ? rc : create_gen(out, math_mode, &cfg->gen, kHeadIstft, n, hop, false);
}

void fs2_istftnet_destroy(fs2_istftnet_gen* m) { destroy_gen(m); }

int fs2_istftnet_load(fs2_istftnet_gen* m, const float* const* weights, const float* const* biases, void* stream) {
  return load_gen(m, weights, biases, nullptr, stream, "fs2_istftnet");
}

int fs2_istftnet_workspace_bytes(fs2_istftnet_gen* m, int B, int Lmax, size_t* bytes) {
  return workspace_gen<HgEntry>(m, B, Lmax, bytes, "fs2_istftnet");
}

int fs2_istftnet(fs2_istftnet_gen* m, const float* mels, const int64_t* olens, int B, int Lmax, float* audio, int* status, void* ws,
                 size_t ws_bytes, void* stream) {
  return call_gen<HgEntry>(m, mels, olens, B, Lmax, audio, status, ws, ws_bytes, stream, "fs2_istftnet");
}

int fs2_istftnet_window_workspace_bytes(fs2_istftnet_gen* m, int B, int n_frames, size_t* bytes) {
  return window_workspace_gen<HgEntry>(m, B, n_frames, bytes, "fs2_istftnet");
}

int fs2_istftnet_window(fs2_istftnet_gen* m, const float* mels, const int64_t* olens, const int64_t* starts, int B, int Lmax, int n_frames,
                        float* audio, int64_t audio_ld, int* status, void* ws, size_t ws_bytes, void* stream) {
  return window_gen<HgEntry>(m, mels, olens, starts, B, Lmax, n_frames, audio, audio_ld, status, ws, ws_bytes, stream, "fs2_istftnet");
}

int fs2_bigvgan_create(fs2_bigvgan_gen** out, int math_mode, const fs2_bigvgan_config* cfg) {
  const char* who = "fs2_bigvgan_create";
  FS2_REQUIRE(out && cfg, "%s: null argument", who);
  FS2_REQUIRE(math_mode >= FS2_MATH_FP32 && math_mode <= FS2_MATH_F16, "%s: bad math_mode %d", who, math_mode);
  int rc = validate(&cfg->gen, who, 8, 1);
  if (rc) return rc;
  FS2_REQUIRE(cfg->activation == FS2_BIGVGAN_SNAKE || cfg->activation == FS2_BIGVGAN_SNAKEBETA,
              "%s: activation must be FS2_BIGVGAN_SNAKE or FS2_BIGVGAN_SNAKEBETA (got %d)", who, cfg->activation);
  if ((rc = create_gen(out, math_mode, &cfg->gen, kHeadActPost, 0, 1, true))) return rc;
  fs2_bigvgan_gen* m = *out;
  m->beta = cfg->activation == FS2_BIGVGAN_SNAKEBETA;
  m->logscale = cfg->snake_logscale;
  m->use_tanh = cfg->use_tanh_at_final;
  m->use_bias = cfg->use_bias_at_final;
  return FS2_OK;
}

void fs2_bigvgan_destroy(fs2_bigvgan_gen* m) { destroy_gen(m); }

int fs2_bigvgan_load(fs2_bigvgan_gen* m, const float* const* weights, const float* const* biases, const float* const* acts, void* stream) {
  return load_gen(m, weights, biases, acts, stream, "fs2_bigvgan");
}

int fs2_bigvgan_workspace_bytes(fs2_bigvgan_gen* m, int B, int Lmax, size_t* bytes) {
  return workspace_gen<HgEntry>(m, B, Lmax, bytes, "fs2_bigvgan");
}

int fs2_bigvgan(fs2_bigvgan_gen* m, const float* mels, const int64_t* olens, int B, int Lmax, float* audio, int* status, void* ws,
                size_t ws_bytes, void* stream) {
  return call_gen<HgEntry>(m, mels, olens, B, Lmax, audio, status, ws, ws_bytes, stream, "fs2_bigvgan");
}

int fs2_bigvgan_window_workspace_bytes(fs2_bigvgan_gen* m, int B, int n_frames, size_t* bytes) {
  return window_workspace_gen<HgEntry>(m, B, n_frames, bytes, "fs2_bigvgan");
}

int fs2_bigvgan_window(fs2_bigvgan_gen* m, const float* mels, const int64_t* olens, const int64_t* starts, int B, int Lmax, int n_frames,
                       float* audio, int64_t audio_ld, int* status, void* ws, size_t ws_bytes, void* stream) {
  return window_gen<HgEntry>(m, mels, olens, starts, B, Lmax, n_frames, audio, audio_ld, status, ws, ws_bytes, stream, "fs2_bigvgan");
}

// ---- single layers on the vocoders' own code paths (tests) ----------------------------------------------------------
int fs2_op_hifigan_resblock(int math_mode, int type, int C, int k, int nd, const int* dils, const float* x, const int64_t* lens, int B,
                            int Lp, const float* const* weights, const float* const* biases, float* out, int* status, void* stream) {
  return op_resblock("fs2_op_hifigan_resblock", math_mode, type, C, k, nd, dils, x, lens, B, Lp, weights, biases, false, nullptr, 0, 0, out,
                     status, stream);
}

int fs2_op_bigvgan_resblock(int math_mode, int type, int C, int k, int nd, const int* dils, const float* x, const int64_t* lens, int B,
                            int Lp, const float* const* weights, const float* const* biases, const float* const* acts, int snakebeta,
                            int logscale, float* out, int* status, void* stream) {
  return op_resblock("fs2_op_bigvgan_resblock", math_mode, type, C, k, nd, dils, x, lens, B, Lp, weights, biases, true, acts, snakebeta,
                     logscale, out, status, stream);
}

int fs2_op_hifigan_upsample(int math_mode, int Cin, int Cout, int u, const float* x, const int64_t* lens, int B, int Lin, const float* w,
                            const float* b, float* out, int* status, void* stream) {
  const char* who = "fs2_op_hifigan_upsample";
  FS2_REQUIRE(math_mode >= FS2_MATH_FP32 && math_mode <= FS2_MATH_F16, "%s: bad math_mode %d", who, math_mode);
  FS2_REQUIRE(u >= 2 && u % 2 == 0 && u <= kHop, "%s: the rate u must be even, in [2, 256] (got %d)", who, u);
  FS2_REQUIRE(Cin >= 32 && Cin % 32 == 0 && Cout >= 32 && Cout % 32 == 0, "%s: Cin and Cout must be multiples of 32 (got %d, %d)", who,
              Cin, Cout);
  FS2_REQUIRE(x && lens && w && b && out && status, "%s: null argument", who);
  FS2_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 31) == 0,
              "%s: x must be 16-byte and out 32-byte aligned", who);
  FS2_REQUIRE(B >= 1 && Lin >= 1, "%s: bad shape B=%d Lin=%d", who, B, Lin);
  const long rows = (long)B * Lin;
  FS2_REQUIRE(rows * u * Cout < (1L << 31) && rows * Cin < (1L << 31) && (math_mode != FS2_MATH_FP32 || rows <= kTapGemmFp32MaxRows),
              "%s: too many rows (%ld)", who, rows);
  cudaStream_t st = (cudaStream_t)stream;
  VWeight wu;
  set_conv(wu, u * Cout, Cin, 3);
  void* a = nullptr;
  void* base = nullptr;
  int rc = temp_carve(&base, st, [&](Bump& bb) {
    vweight_carve(bb, wu, true);
    a = bb.floats((size_t)rows * Cin);
  });
  if (rc) return rc;
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  rc = vweight_pack_conv(wu, w, b, Cin, Cout, 3, u, (long)wu.N * Cin, st);
  if (!rc) rc = upsample(math_mode, true, wu, x, nullptr, 1, nullptr, Lin, lens, nullptr, B, Lin, Cin, a, out, status, st);
  cudaFreeAsync(base, st);
  return rc;
}

}  // extern "C"
