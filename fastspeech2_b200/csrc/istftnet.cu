// iSTFTNet's inverse-STFT head (DESIGN.md section 19), on CUDA cores in fp32 in every math mode.  The generator chain
// before it is HiFi-GAN's (hifigan.cu); this file holds only the head, so that hifigan.cu's kernels stay as they are.
//
// One CTA per (audio tile, utterance).  A tile of NS = hop (kF - n_fft / hop) samples is covered by at most kF frames
// (conv_post output rows); their x rows (kF + 6 with conv_post's taps and the reflected row) are staged in shared memory
// kC channels at a time with conv_post's weights for those channels, so each frame's n_fft + 2 values and its inverse DFT
// are computed once per tile.  Every value has a fixed arithmetic: conv_post sums bias, then channels ascending with taps
// ascending inside, in fmaf; full-precision expf / sinf / cosf; twiddles and the window rounded once from double; the
// overlap-add and the envelope sum frames ascending.  So a sample's bits do not depend on its tile, batch or window.
#include <math.h>

#include "istftnet.cuh"
#include "vocoder_weights.cuh"
#include "vocoder_window.cuh"

namespace fs2 {
namespace {

constexpr int kHeadThreads = 128;
constexpr int kF = 256;                    // frames per tile: 64 slots x 4 frames per thread
constexpr int kC = 16;                     // channels staged per pass
constexpr int kTaps = 7;
constexpr int kMaxO = kIstftMaxNfft + 2;
constexpr int kOH = (kMaxO + 1) / 2;       // outputs per thread: the two halves of the CTA take half of n_fft + 2 each
constexpr int kOHp = 12;                   // kOH padded to 3 float4
constexpr int kXRegion = (kF + 6) * (kC + 1) > kF * (kMaxO + kIstftMaxNfft) ? (kF + 6) * (kC + 1) : kF * (kMaxO + kIstftMaxNfft);
constexpr float kHeadSlope = 0.01f;        // F.leaky_relu's default before conv_post
static_assert(kOH <= kOHp && kOHp % 4 == 0, "a thread's outputs must fit its padded weight row");
static_assert(kHeadThreads == 2 * (kF / 4), "two halves of kF / 4 slots");

__global__ void __launch_bounds__(kHeadThreads) istftnet_head_kernel(const float* __restrict__ S, const float* __restrict__ R, int nk,
                                                                     const int64_t* __restrict__ lens, const int64_t* __restrict__ win,
                                                                     const int64_t* __restrict__ awin, int B, int Lx, int Lout, long ld,
                                                                     int C, int N, int hop, const float* __restrict__ w,
                                                                     const float* __restrict__ bias, float* __restrict__ audio) {
  __shared__ float xs[kXRegion];                              // staged x rows [kF + 6][kC + 1]; then y [kF][O] and frames [kF][N]
  __shared__ __align__(16) float wsm[kTaps * kC * 2 * kOHp];  // [tap][channel][half][kOHp]
  __shared__ float cs[kIstftMaxNfft], sn[kIstftMaxNfft], hw[kIstftMaxNfft], hw2[kIstftMaxNfft];
  const int b = blockIdx.y, tid = threadIdx.x;
  const Rows r = rows_of(win, lens, B, b);
  const long a0 = awin ? awin[b] * hop : 0, na = awin ? awin[B + b] * hop : (long)r.n * hop;
  const int NS = hop * (kF - N / hop);
  const long t0 = (long)blockIdx.x * NS, t1 = min(t0 + NS, (long)Lout), tv = min(t1, na);   // samples [t0, tv) are audio
  float* out = audio + (long)b * ld;
  if (t0 >= tv) {
    for (long t = t0 + tid; t < t1; t += kHeadThreads) out[t] = 0.f;
    return;
  }
  const int T = r.n, O = N + 2, M = N / 2 + 1, OH = (O + 1) / 2;
  // frames covering samples [n0, n1) (global, untrimmed position p = n + N / 2): hop f <= p < hop f + N, f in [0, T]
  const long n0 = a0 + t0, n1 = a0 + tv;
  const long plo = n0 + N / 2 - N + 1;
  const int f_lo = (int)(plo <= 0 ? 0 : (plo + hop - 1) / hop);
  const int f_hi = (int)min((n1 - 1 + N / 2) / hop, (long)T);
  const int nfr = f_hi - f_lo + 1, nrows = nfr + 6;
  if (tid < N) {
    const double th = 2.0 * (double)tid / (double)N;
    cs[tid] = (float)cospi(th);
    sn[tid] = (float)sinpi(th);
    const double h = 0.5 - 0.5 * cospi(th);                   // periodic Hann
    hw[tid] = (float)h;
    hw2[tid] = (float)(h * h);
  }
  const int half = tid / (kF / 4), slot = tid % (kF / 4);
  float acc[4][kOH];
#pragma unroll
  for (int q = 0; q < kOH; ++q) {
    const int o = half * OH + q;
    const float bq = q < OH && o < O ? __ldg(bias + o) : 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[i][q] = bq;
  }
  const float fk = (float)nk;
#pragma unroll 1
  for (int c0 = 0; c0 < C; c0 += kC) {
    __syncthreads();
    // x row g = f_lo - 4 + i: padded row g + 1 of ReflectionPad1d((1, 0)), i.e. x[1] for g = -1, 0 outside [0, T)
    for (int idx = tid; idx < nrows * (kC / 4); idx += kHeadThreads) {
      const int i = idx / (kC / 4), q = idx - i * (kC / 4);
      int g = f_lo - 4 + i;
      if (g == -1) g = 1;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (g >= 0 && g < T && g >= r.start && g < r.start + r.len) {
        const long off = ((long)b * Lx + g - r.start) * C + c0 + 4 * q;
        v = __ldg(reinterpret_cast<const float4*>(S + off));
        if (R) {
          const float4 u = __ldg(reinterpret_cast<const float4*>(R + off));
          v = make_float4(v.x + u.x, v.y + u.y, v.z + u.z, v.w + u.w);
        }
        if (nk != 1) v = make_float4(v.x / fk, v.y / fk, v.z / fk, v.w / fk);
      }
      float* d = xs + i * (kC + 1) + 4 * q;
      d[0] = v.x > 0.f ? v.x : v.x * kHeadSlope;
      d[1] = v.y > 0.f ? v.y : v.y * kHeadSlope;
      d[2] = v.z > 0.f ? v.z : v.z * kHeadSlope;
      d[3] = v.w > 0.f ? v.w : v.w * kHeadSlope;
    }
    for (int idx = tid; idx < kTaps * kC * 2 * kOHp; idx += kHeadThreads) {
      const int q = idx % kOHp, hh = (idx / kOHp) & 1, cc = (idx / (2 * kOHp)) % kC, j = idx / (2 * kOHp * kC);
      const int o = hh * OH + q;
      wsm[idx] = q < OH && o < O ? __ldg(w + ((long)j * O + o) * C + c0 + cc) : 0.f;
    }
    __syncthreads();
#pragma unroll 1
    for (int cc = 0; cc < kC; ++cc) {
#pragma unroll
      for (int j = 0; j < kTaps; ++j) {
        const float4* wp = reinterpret_cast<const float4*>(wsm + ((j * kC + cc) * 2 + half) * kOHp);
        const float4 w0 = wp[0], w1 = wp[1], w2 = wp[2];
        const float wq[12] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w, w2.x, w2.y, w2.z, w2.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float xv = xs[(slot + i * (kF / 4) + j) * (kC + 1) + cc];
#pragma unroll
          for (int q = 0; q < kOH; ++q) acc[i][q] = fmaf(wq[q], xv, acc[i][q]);
        }
      }
    }
  }
  __syncthreads();
  // y = conv_post's output: exp of the log-magnitudes (o < M), sin of the phases
  float* Y = xs;               // [kF][O]
  float* F = xs + kF * O;      // [kF][N]: windowed inverse DFT of each frame
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int f = slot + i * (kF / 4);
#pragma unroll
    for (int q = 0; q < kOH; ++q) {
      const int o = half * OH + q;
      if (f < nfr && q < OH && o < O) Y[f * O + o] = o < M ? expf(acc[i][q]) : sinf(acc[i][q]);
    }
  }
  __syncthreads();
  for (int idx = tid; idx < nfr * M; idx += kHeadThreads) {   // X_m = mag (cos ph + i sin ph)
    const int f = idx / M, m = idx - f * M;
    const float mag = Y[f * O + m], ph = Y[f * O + M + m];
    Y[f * O + m] = mag * cosf(ph);
    Y[f * O + M + m] = mag * sinf(ph);
  }
  __syncthreads();
  // c2r inverse DFT (the imaginary parts of bins 0 and N / 2 dropped), 1 / N, times the window
  for (int idx = tid; idx < nfr * N; idx += kHeadThreads) {
    const int f = idx / N, k = idx - f * N;
    const float* z = Y + f * O;
    float v = z[0];
    v += (k & 1) ? -z[N / 2] : z[N / 2];
    for (int m = 1; m < N / 2; ++m) {
      const int t = (m * k) % N;
      v = fmaf(2.f * z[m], cs[t], v);
      v = fmaf(-2.f * z[M + m], sn[t], v);
    }
    F[idx] = v / (float)N * hw[k];
  }
  __syncthreads();
  // overlap-add over the frames that exist, divided by their envelope sum_f w^2[p - hop f]; N / 2 trimmed at the front
  for (long t = t0 + tid; t < t1; t += kHeadThreads) {
    float y = 0.f;
    if (t < tv) {
      const long p = a0 + t + N / 2, lo = p - N + 1;
      const int fa = (int)(lo <= 0 ? 0 : (lo + hop - 1) / hop), fb = (int)min(p / hop, (long)T);
      float s = 0.f, env = 0.f;
      for (int f = fa; f <= fb; ++f) {
        const int k = (int)(p - (long)hop * f);
        s += F[(f - f_lo) * N + k];
        env += hw2[k];
      }
      y = s / env;
    }
    out[t] = y;
  }
}

}  // namespace

int istftnet_head(const float* S, const float* R, int nk, const int64_t* lens, const int64_t* win, const int64_t* awin, int B, int Lx,
                  int Lout, long ld, int C, int n_fft, int hop, const float* w, const float* bias, float* audio, cudaStream_t st) {
  const int NS = hop * (kF - n_fft / hop);
  const dim3 grid((unsigned)((Lout + NS - 1) / NS), (unsigned)B);
  istftnet_head_kernel<<<grid, kHeadThreads, 0, st>>>(S, R, nk, lens, win, awin, B, Lx, Lout, ld, C, n_fft, hop, w, bias, audio);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace fs2

using namespace fs2;

extern "C" {

// ---- the head alone on its own code path (tests) ------------------------------------------------------------------
int fs2_op_istftnet_head(int C, int n_fft, int hop, const float* x, const int64_t* lens, int B, int Lp, const float* w, const float* b,
                         float* audio, void* stream) {
  const char* who = "fs2_op_istftnet_head";
  FS2_REQUIRE(C >= 32 && C % 32 == 0 && C <= 2048, "%s: C must be a multiple of 32 in [32, 2048] (got %d)", who, C);
  FS2_REQUIRE(n_fft >= 2 && n_fft <= kIstftMaxNfft && n_fft % 2 == 0, "%s: n_fft must be even, in [2, %d] (got %d)", who, kIstftMaxNfft,
              n_fft);
  FS2_REQUIRE(hop >= 1 && n_fft % hop == 0 && n_fft / hop >= 2, "%s: hop must divide n_fft with n_fft / hop >= 2 (got %d, %d)", who, n_fft,
              hop);
  FS2_REQUIRE(x && lens && w && b && audio, "%s: null argument", who);
  FS2_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0, "%s: x must be 16-byte aligned", who);
  FS2_REQUIRE(B >= 1 && B <= 65535 && Lp >= 1, "%s: bad shape B=%d Lp=%d", who, B, Lp);
  FS2_REQUIRE((long)B * Lp * C < (1L << 31) && (long)Lp * hop < (1L << 31), "%s: too many rows (%ld)", who, (long)B * Lp);
  cudaStream_t st = (cudaStream_t)stream;
  const int O = n_fft + 2;
  float* wt = nullptr;
  void* base = nullptr;
  int rc = temp_carve(&base, st, [&](Bump& bb) { wt = bb.floats((size_t)kTaps * O * C); });
  if (rc) return rc;
  rc = conv_pack(w, O, C, kTaps, O, 0, (long)O * C, C, wt, st);
  if (!rc) rc = istftnet_head(x, nullptr, 1, lens, nullptr, nullptr, B, Lp, Lp * hop, (long)Lp * hop, C, n_fft, hop, wt, b, audio, st);
  cudaFreeAsync(base, st);
  return rc;
}

}  // extern "C"
