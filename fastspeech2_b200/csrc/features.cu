// Training features (DESIGN.md section 14): per-utterance log-mel, energy and WORLD DIO pitch of a ragged batch of wavs
// [B, Nmax] with lens [B], what the reference's nvidia_preprocessing.py computes one file at a time on the CPU.
//
// Mel and energy, rows = the B * Tmax frames, every GEMM with TapGemm::lens = T_b (rows past T_b come out as 0):
//   feat_frames      reflect-pad each utterance at its own edges and write the frames as the forward-DFT GEMM's operand
//                    (fp32 rows or fp16 planes); checks lens and |x| <= 1, writes T_b
//   GEMM             forward DFT (K = n_fft, N = cpad), the vocoder's packed Fourier basis
//   feat_magnitude   |Z| as the mel GEMM's operand (K = mpad, zero past cutoff) and energy = sqrt(sum_c |Z|^2), one warp
//                    per frame, each lane summing its columns in order, then a fixed butterfly
//   GEMM             mel filterbank (K = mpad, N = n_mels)
//   feat_log         log(max(., 1e-5)) into [B, Tmax, n_mels], +0 past T_b
//
// DIO, float64 on the CUDA cores (oracle/dio_oracle.py restates every step):
//   dio_prepare      per utterance: length / range check, mean of y (x then one zero) in a fixed tree, f0_length,
//                    fft_size, plens
//   dio_lowcut       z = low-cut FIR of y, circular modulo fft_size (the FFT product WORLD computes), stored for the
//                    index range every band filter reads
//   per band, one after another (the workspace holds one band's signal):
//     dio_band       s = Nuttall FIR of z, advanced by 2h: a tiled direct-form FIR from shared memory
//     dio_events     the four event series, each an order-preserving compaction of fine edges, one CTA per series
//     dio_frames     interp1 of the four series at each frame, candidate, score, running best band
//   dio_fix          FixF0Contour, one warp per utterance: steps 1-2 across the lanes, steps 3-4 as sequential walks
// Every sum has a fixed order and nothing depends on the batch, so utterance b is bit-identical to a B = 1 call.
#include <math.h>
#include <string.h>

#include <vector>

#include "vocoder_weights.cuh"

namespace fs2 {
namespace {

constexpr int kMaxBands = 16;
constexpr int FT = 256;              // FIR outputs per CTA
constexpr int EV_THREADS = 512;      // event compaction CTA
constexpr int EV_WARPS = EV_THREADS / 32;
constexpr double kLog2 = 0.69314718055994529;
constexpr double kMaxValue = 100000.0;
constexpr double kSafeGuard = 1e-12;

inline int grid_for(long n, int block, int cap = 132 * 8) {
  long g = (n + block - 1) / block;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

inline int matlab_round(double x) { return x > 0 ? (int)(x + 0.5) : (int)(x - 0.5); }

struct Bump {
  char* base; size_t off = 0, cap;
  Bump(void* b, size_t c) : base((char*)b), cap(c) {}
  void* bytes(size_t n) { size_t a = (off + 255) & ~(size_t)255; off = a + n; return base ? base + a : nullptr; }
  float* floats(size_t n) { return (float*)bytes(n * sizeof(float)); }
  double* doubles(size_t n) { return (double*)bytes(n * sizeof(double)); }
  bool ok() const { return base == nullptr || off <= cap; }
};

// ---- mel and energy ------------------------------------------------------------------------------------------------

// frames of utterance b; 0 for a length outside (n_fft/2, Nmax]
__device__ __forceinline__ int frames_of(const int64_t* __restrict__ lens, int b, int Nmax, int hop, int half) {
  const int64_t n = lens[b];
  return (n > half && n <= Nmax) ? (int)(n / hop) + 1 : 0;
}

// one pair of GEMM-operand values at element offset off (even) of a [rows][K] operand; plane = rows * K
template <int OUT>
__device__ __forceinline__ void store_operand(float v0, float v1, long off, float* __restrict__ out32, __half* __restrict__ outp, long plane) {
  if (OUT == OUT_F32) {
    *reinterpret_cast<float2*>(out32 + off) = make_float2(v0, v1);
  } else if (OUT == OUT_HILO) {
    uint32_t hi, lo;
    split_pair(v0, v1, hi, lo);
    *reinterpret_cast<uint32_t*>(outp + off) = hi;
    *reinterpret_cast<uint32_t*>(outp + plane + off) = lo;
  } else {
    *reinterpret_cast<uint32_t*>(outp + off) = hi_pair(v0, v1);
  }
}

// frames[row, k] = reflect_pad(x_b, n_fft/2)[t * hop + k] for t < T_b (rows past T_b are not written); flens[b] = T_b
template <int OUT>
__global__ void feat_frames_kernel(const float* __restrict__ wav, const int64_t* __restrict__ lens, int B, int Nmax, int T, int n_fft,
                                   int hop, float* __restrict__ out32, __half* __restrict__ outp, int64_t* __restrict__ flens,
                                   int* __restrict__ status) {
  const int half = n_fft / 2;
  const long total = (long)B * T * half, plane = (long)B * T * n_fft;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / half;
    const int k = (int)(i - row * half) * 2, b = (int)(row / T), t = (int)(row - (long)b * T);
    const int tb = frames_of(lens, b, Nmax, hop, half);
    if (t == 0 && k == 0) {
      flens[b] = tb;
      if (tb == 0) atomicOr(status, FS2_FEAT_BAD_LENGTH);
    }
    if (t >= tb) continue;
    const int n = (int)lens[b];
    float v[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      int s = t * hop + k + e - half;                 // reflect without repeating the edge sample (n > half)
      if (s < 0) s = -s;
      if (s >= n) s = 2 * (n - 1) - s;
      v[e] = wav[(long)b * Nmax + s];
    }
    if (!(fabsf(v[0]) <= 1.f && fabsf(v[1]) <= 1.f)) atomicOr(status, FS2_FEAT_RANGE);   // NaN included
    store_operand<OUT>(v[0], v[1], row * n_fft + k, out32, outp, plane);
  }
}

// one warp per frame: |Z| [row][mpad] (0 past cutoff) as the mel GEMM's operand, energy[row] = sqrt(sum_c |Z|^2)
template <int OUT>
__global__ void feat_magnitude_kernel(const float* __restrict__ z, int cpad, int cutoff, int mpad, const int64_t* __restrict__ flens,
                                      int B, int T, float* __restrict__ out32, __half* __restrict__ outp, float* __restrict__ energy) {
  const int lane = threadIdx.x & 31;
  const long rows = (long)B * T, plane = rows * mpad;
  const long stride = ((long)gridDim.x * blockDim.x) >> 5;
  for (long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += stride) {
    const int b = (int)(row / T), t = (int)(row - (long)b * T);
    if (t >= flens[b]) {
      if (lane == 0) energy[row] = 0.f;
      continue;
    }
    const float* zr = z + row * cpad;
    float acc = 0.f;
    for (int c = 2 * lane; c < mpad; c += 64) {
      float m[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        m[e] = 0.f;
        if (c + e < cutoff) {
          const float re = zr[c + e], im = zr[cutoff + c + e];
          m[e] = sqrtf(re * re + im * im);
          acc += m[e] * m[e];
        }
      }
      store_operand<OUT>(m[0], m[1], row * mpad + c, out32, outp, plane);
    }
    acc = warp_sum(acc);
    if (lane == 0) energy[row] = sqrtf(acc);
  }
}

__global__ void feat_log_kernel(const float* __restrict__ raw, const int64_t* __restrict__ flens, int B, int T, int n_mels,
                                float* __restrict__ mel) {
  const long total = (long)B * T * n_mels;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / n_mels;
    const int b = (int)(row / T), t = (int)(row - (long)b * T);
    mel[i] = t < flens[b] ? logf(fmaxf(raw[i], 1e-5f)) : 0.f;
  }
}

// ---- DIO -----------------------------------------------------------------------------------------------------------

struct DioMeta {
  int n;        // samples; 0 for an utterance that fails the length check (all its outputs are 0)
  int f0len;    // WORLD's f0_length
  int fft;      // WORLD's fft_size: the circular convolutions wrap modulo this
  double mean;  // mean of y[0:n+1]
};

// grid B: length / range check, mean of y in a fixed tree, f0_length, fft_size, plens
__global__ void __launch_bounds__(256) dio_prepare_kernel(const float* __restrict__ wav, const int64_t* __restrict__ lens, int Nmax,
                                                          int half, int hop, int fs, double fp, int fft_extra, int Tp,
                                                          DioMeta* __restrict__ meta, int64_t* __restrict__ plens, int* __restrict__ status) {
  __shared__ double part[256];
  __shared__ int bad;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int64_t n64 = lens[b];
  const bool ok = n64 > half && n64 <= Nmax;
  const int n = ok ? (int)n64 : 0;
  if (tid == 0) bad = 0;
  __syncthreads();
  double acc = 0.0;
  bool r = false;
  for (int i = tid; i < n; i += 256) {
    const float v = wav[(long)b * Nmax + i];
    r |= !(fabsf(v) <= 1.f);
    acc += (double)v;
  }
  part[tid] = acc;
  if (r) bad = 1;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (tid < s) part[tid] += part[tid + s];
    __syncthreads();
  }
  if (tid == 0) {
    if (!ok) atomicOr(status, FS2_FEAT_BAD_LENGTH);
    if (bad) atomicOr(status, FS2_FEAT_RANGE);
    DioMeta m;
    m.n = n;
    m.mean = n ? part[0] / (double)(n + 1) : 0.0;
    const int f0len = n ? (int)(1000.0 * n / fs / fp) + 1 : 0;     // GetSamplesForDIO, in this order
    m.f0len = f0len < Tp ? f0len : Tp;                               // f0_length <= T_b < Tp: a bound, never reached
    int F = 1;
    while (F <= n + 1 + fft_extra) F <<= 1;                          // smallest power of two above y_length + extra
    m.fft = F;
    meta[b] = m;
    const int tb = n ? n / hop + 1 : 0;
    plens[b] = m.f0len < tb ? m.f0len : tb;
  }
}

// z_ext[j] = z[(j - P) mod F] for j in [0, n + 1 + 2P), z = lc (*) y circular modulo F, lc taps at offsets -M..M
__global__ void __launch_bounds__(FT) dio_lowcut_kernel(const float* __restrict__ wav, int Nmax, const DioMeta* __restrict__ meta,
                                                        const double* __restrict__ lc, int M, int P, long zs, double* __restrict__ z) {
  extern __shared__ double sm[];
  double* taps = sm;
  double* yw = sm + 2 * M + 1;
  const int b = blockIdx.y, tid = threadIdx.x;
  const DioMeta m = meta[b];
  const int zlen = m.n + 1 + 2 * P, j0 = blockIdx.x * FT;
  if (m.n == 0 || j0 >= zlen) return;
  const int mask = m.fft - 1;
  for (int u = tid; u < 2 * M + 1; u += FT) taps[u] = lc[u];
  for (int u = tid; u < FT + 2 * M; u += FT) {
    const int r = (j0 - P - M + u) & mask;                           // y index modulo F (two's complement: negatives wrap)
    yw[u] = r < m.n ? (double)wav[(long)b * Nmax + r] - m.mean : (r == m.n ? -m.mean : 0.0);
  }
  __syncthreads();
  const int j = j0 + tid;
  if (j >= zlen) return;
  double acc = 0.0;
  for (int k = 0; k <= 2 * M; ++k) acc = fma(taps[k], yw[tid + 2 * M - k], acc);
  z[(long)b * zs + j] = acc;
}

// s[i] = sum_k nut[k] z[i + 2h - k], k = 0..4h-1, for i in [0, n + 1)
__global__ void __launch_bounds__(FT) dio_band_kernel(const DioMeta* __restrict__ meta, const double* __restrict__ z, long zs,
                                                      const double* __restrict__ nut, int h, int P, double* __restrict__ s, long ss) {
  extern __shared__ double sm[];
  const int L4 = 4 * h;
  double* taps = sm;
  double* zw = sm + L4;
  const int b = blockIdx.y, tid = threadIdx.x;
  const int n = meta[b].n, i0 = blockIdx.x * FT;
  if (n == 0 || i0 > n) return;
  const int zlen = n + 1 + 2 * P;
  for (int u = tid; u < L4; u += FT) taps[u] = nut[u];
  for (int u = tid; u < FT + L4 - 1; u += FT) {
    const int q = i0 - 2 * h + 1 + u + P;                            // z_ext index
    zw[u] = q < zlen ? z[(long)b * zs + q] : 0.0;                     // past zlen only outputs i > n read it
  }
  __syncthreads();
  const int i = i0 + tid;
  if (i > n) return;
  double acc = 0.0;
  for (int k = 0; k < L4; ++k) acc = fma(taps[k], zw[tid + L4 - 1 - k], acc);
  s[(long)b * ss + i] = acc;
}

// series 0: s, 1: -s, 2: d = (-s[i]) - (-s[i+1]) (peaks of s), 3: -d (dips)
__device__ __forceinline__ double ev_sig(const double* __restrict__ s, int series, int i) {
  if (series < 2) { const double v = s[i]; return series == 0 ? v : -v; }
  const double d = (-s[i]) - (-s[i + 1]);
  return series == 2 ? d : -d;
}

// grid (4, B): fine edges e - g[e-1] / (g[e] - g[e-1]) of the negative-going zero crossings (0 < g[e-1], g[e] <= 0) of
// one series, in order; count = their number
__global__ void __launch_bounds__(EV_THREADS) dio_events_kernel(const DioMeta* __restrict__ meta, const double* __restrict__ s, long ss,
                                                                double* __restrict__ fine, long es, int* __restrict__ count) {
  __shared__ int wsum[EV_WARPS];
  const int series = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n0 = meta[b].n;
  const int n = n0 == 0 ? 0 : (series < 2 ? n0 + 1 : n0);           // y_length, or y_length - 1 for the difference
  const double* sb = s + (long)b * ss;
  double* out = fine + ((long)b * 4 + series) * es;
  int base = 0;
  for (int i0 = 0; i0 < n - 1; i0 += EV_THREADS) {
    const int i = i0 + tid;
    double g0 = 0.0, g1 = 0.0;
    bool f = false;
    if (i < n - 1) {
      g0 = ev_sig(sb, series, i);
      g1 = ev_sig(sb, series, i + 1);
      f = 0.0 < g0 && g1 <= 0.0;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, f);
    if (lane == 0) wsum[warp] = __popc(bal);
    __syncthreads();
    if (warp == 0) {                                                  // inclusive scan of the warp counts
      int v = lane < EV_WARPS ? wsum[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
      }
      if (lane < EV_WARPS) wsum[lane] = v;
    }
    __syncthreads();
    if (f) out[base + (warp ? wsum[warp - 1] : 0) + __popc(bal & ((1u << lane) - 1u))] = (double)(i + 1) - g0 / (g1 - g0);
    base += wsum[EV_WARPS - 1];
    __syncthreads();
  }
  if (tid == 0) count[b * 4 + series] = base;
}

// interval locations x[j] = (fe[j] + fe[j+1]) / 2 / fs and intervals y[j] = fs / (fe[j+1] - fe[j]), j < n
__device__ __forceinline__ double ev_loc(const double* __restrict__ fe, int j, double fs) { return (fe[j] + fe[j + 1]) / 2.0 / fs; }
__device__ __forceinline__ double ev_val(const double* __restrict__ fe, int j, double fs) { return fs / (fe[j + 1] - fe[j]); }

// WORLD's interp1 + histc: segment k = min(1 + #{j >= 1: x[j] <= xi}, n - 1), linear, extrapolating at both ends
__device__ double interp_series(const double* __restrict__ fe, int n, double xi, double fs) {
  int lo = 1, hi = n;                                                 // first j in [1, n) with x[j] > xi, else n
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (ev_loc(fe, mid, fs) > xi) hi = mid; else lo = mid + 1;
  }
  const int k = lo < n - 1 ? lo : n - 1;
  const double x0 = ev_loc(fe, k - 1, fs), x1 = ev_loc(fe, k, fs), y0 = ev_val(fe, k - 1, fs), y1 = ev_val(fe, k, fs);
  const double sl = (xi - x0) / (x1 - x0);
  return __dadd_rn(y0, __dmul_rn(sl, y1 - y0));                      // unfused, as WORLD's C evaluates it
}

__device__ __forceinline__ double sq(double a) { return __dmul_rn(a, a); }

// grid (ceil(Tp / 128), B): the band's candidate and score at every frame < f0_length; the best band so far
__global__ void dio_frames_kernel(const DioMeta* __restrict__ meta, const double* __restrict__ fine, long es, const int* __restrict__ count,
                                  int B, int Tp, int band, double boundary, double f0_floor, double f0_ceil, double fs, double fp,
                                  double* __restrict__ cand, double* __restrict__ best_f0, double* __restrict__ best_score) {
  const int b = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= meta[b].f0len) return;
  int nint[4];
  bool ok = true;
#pragma unroll
  for (int q = 0; q < 4; ++q) { nint[q] = count[b * 4 + q] - 1; ok = ok && nint[q] >= 3; }
  double c = 0.0, sc = kMaxValue;
  if (ok) {
    const double xi = (double)i * fp / 1000.0;
    double v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) v[q] = interp_series(fine + ((long)b * 4 + q) * es, nint[q], xi, fs);
    c = (v[0] + v[1] + v[2] + v[3]) / 4.0;
    sc = sqrt(__dadd_rn(__dadd_rn(__dadd_rn(sq(v[0] - c), sq(v[1] - c)), sq(v[2] - c)), sq(v[3] - c)) / 3.0);
    if (c > boundary || c < boundary / 2.0 || c > f0_ceil || c < f0_floor) { c = 0.0; sc = kMaxValue; }
  }
  sc = sc / (c + kSafeGuard);
  const long o = (long)b * Tp + i;
  cand[(long)band * B * Tp + o] = c;
  if (band == 0 || best_score[o] > sc) { best_score[o] = sc; best_f0[o] = c; }   // the first minimum wins
}

// SelectBestF0: the candidate (over all bands) nearest (3 cur - past) / 2, 0 if it is off by more than allowed
__device__ double select_best(double cur, double past, const double* __restrict__ cand, long band_stride, int nb, long idx, double allowed) {
  const double ref = __dsub_rn(__dmul_rn(cur, 3.0), past) / 2.0;
  double best = cand[idx], err = fabs(ref - best);
  for (int j = 1; j < nb; ++j) {
    const double v = cand[j * band_stride + idx], e = fabs(ref - v);
    if (e < err) { err = e; best = v; }
  }
  return fabs(1.0 - best / ref) > allowed ? 0.0 : best;
}

// last frame i - 1 of the first voiced section ending at or after `from` - 1 (f[i] == 0, f[i-1] != 0), or -1
__device__ int next_section_end(const double* __restrict__ f, int n, int from) {
  for (int i = from; i < n; ++i) if (f[i] == 0.0 && f[i - 1] != 0.0) return i - 1;
  return -1;
}
// first frame i <= from of the last voiced section starting there (f[i-1] == 0, f[i] != 0), or -1
__device__ int prev_section_start(const double* __restrict__ f, int from) {
  for (int i = from; i >= 1; --i) if (f[i - 1] == 0.0 && f[i] != 0.0) return i;
  return -1;
}

// grid B, one warp: FixF0Contour on the best-band contour, then f0 [B, T] = contour truncated to plens[b], +0 after
__global__ void __launch_bounds__(32) dio_fix_kernel(const DioMeta* __restrict__ meta, const double* __restrict__ best,
                                                     const double* __restrict__ cand, int B, int Tp, int nb, int vrm, double allowed,
                                                     double* __restrict__ t1, double* __restrict__ t2, const int64_t* __restrict__ plens,
                                                     double* __restrict__ f0, int T) {
  const int b = blockIdx.x, lane = threadIdx.x;
  const int n = meta[b].f0len, pl = (int)plens[b];
  double* out = f0 + (long)b * T;
  if (n <= vrm) {
    for (int i = lane; i < T; i += 32) out[i] = 0.0;
    return;
  }
  const long o = (long)b * Tp;
  const double* bf = best + o;
  double* f = t1 + o;      // steps 1, then 3 and 4 in place
  double* s2 = t2 + o;     // step 2: the sections steps 3 and 4 start from
  for (int i = lane; i < n; i += 32) {                               // step 1: edges and jumps
    double v = 0.0;
    if (i >= vrm) {
      const double cur = i < n - vrm ? bf[i] : 0.0;
      const double prev = (i - 1 >= vrm && i - 1 < n - vrm) ? bf[i - 1] : 0.0;
      v = fabs((cur - prev) / (kSafeGuard + cur)) < allowed ? cur : 0.0;
    }
    f[i] = v;
  }
  __syncwarp();
  const int c = (vrm - 1) / 2;
  for (int i = lane; i < n; i += 32) {                               // step 2: a zero within +-c
    double v = f[i];
    if (i >= c && i < n - c)
      for (int j = -c; j <= c; ++j)
        if (f[i + j] == 0.0) { v = 0.0; break; }
    s2[i] = v;
  }
  __syncwarp();
  for (int i = lane; i < n; i += 32) f[i] = s2[i];
  __syncwarp();
  if (lane == 0) {
    const long bs = (long)B * Tp;
    for (int e = next_section_end(s2, n, 1); e >= 0;) {              // step 3: forward from each section's last frame
      const int nxt = next_section_end(s2, n, e + 2);
      const int limit = nxt < 0 ? n - 1 : nxt;
      for (int j = e; j < limit; ++j) {
        f[j + 1] = select_best(f[j], f[j - 1], cand, bs, nb, o + j + 1, allowed);
        if (f[j + 1] == 0.0) break;
      }
      e = nxt;
    }
    for (int p = prev_section_start(s2, n - 1); p >= 0;) {           // step 4: backwards, last section first
      const int prv = prev_section_start(s2, p - 1);
      const int limit = prv < 0 ? 1 : prv;
      for (int j = p; j > limit; --j) {
        f[j - 1] = select_best(f[j], f[j + 1], cand, bs, nb, o + j - 1, allowed);
        if (f[j - 1] == 0.0) break;
      }
      p = prv;
    }
  }
  __syncwarp();
  for (int i = lane; i < T; i += 32) out[i] = i < pl ? f[i] : 0.0;
}

}  // namespace
}  // namespace fs2

struct fs2_features {
  fs2_features_config cfg;
  int cutoff = 0, cpad = 0, mpad = 0;
  int n_bands = 0, lc_half = 0, pad = 0, vrm = 0, fft_extra = 0;
  double frame_period = 0;
  double boundary[fs2::kMaxBands];
  int h[fs2::kMaxBands], nut_off[fs2::kMaxBands];
  std::vector<double> taps_host;   // low-cut taps (2 M + 1), then each band's Nuttall window (4 h)
  bool loaded = false;
  int device = -1;
  void* arena = nullptr;
  fs2::VWeight fwd, mel;           // forward DFT [cpad][n_fft], mel filterbank [n_mels][mpad]
  double* taps = nullptr;
};

namespace fs2 {
namespace {

struct MelPlan {
  void* frames;      // forward-DFT operand [rows][n_fft]
  float* z;          // its output [rows][cpad]
  void* mag;         // mel operand [rows][mpad]
  float* raw;        // mel GEMM output [rows][n_mels]
  int64_t* flens;    // T_b [B]
};
// an operand takes rows * K * 4 bytes either way: fp32 rows, or hi + lo fp16 planes
MelPlan mel_plan(const fs2_features* f, Bump& bp, int B, int T) {
  const size_t rows = (size_t)B * T;
  MelPlan p;
  p.frames = bp.floats(rows * f->cfg.n_fft);
  p.z = bp.floats(rows * f->cpad);
  p.mag = bp.floats(rows * f->mpad);
  p.raw = bp.floats(rows * f->cfg.n_mels);
  p.flens = (int64_t*)bp.bytes((size_t)B * sizeof(int64_t));
  return p;
}

struct DioPlan {
  DioMeta* meta;
  double* z; long zs;          // low-cut output over the index range the bands read, [B][Nmax + 1 + 2P]
  double* s; long ss;          // one band's signal [B][Nmax + 2]
  double* fine; long es;       // fine edges [B][4][Nmax / 2 + 2]
  int* count;                  // [B][4]
  double *cand, *best_f0, *best_score, *t1, *t2;   // [n_bands][B][Tp], then [B][Tp] each
  int Tp;
};
DioPlan dio_plan(const fs2_features* f, Bump& bp, int B, int Nmax) {
  DioPlan p;
  p.Tp = Nmax / f->cfg.hop + 2;
  p.zs = (long)Nmax + 1 + 2 * f->pad;
  p.ss = (long)Nmax + 2;
  p.es = (long)Nmax / 2 + 2;       // negative-going crossings of n samples are at most ceil((n - 1) / 2)
  p.meta = (DioMeta*)bp.bytes((size_t)B * sizeof(DioMeta));
  p.z = bp.doubles((size_t)B * p.zs);
  p.s = bp.doubles((size_t)B * p.ss);
  p.fine = bp.doubles((size_t)B * 4 * p.es);
  p.count = (int*)bp.bytes((size_t)B * 4 * sizeof(int));
  const size_t fr = (size_t)B * p.Tp;
  p.cand = bp.doubles(fr * f->n_bands);
  p.best_f0 = bp.doubles(fr);
  p.best_score = bp.doubles(fr);
  p.t1 = bp.doubles(fr);
  p.t2 = bp.doubles(fr);
  return p;
}

int check_call(const fs2_features* f, const float* wav, const int64_t* lens, int B, int Nmax, const int* status, const void* ws, const char* who) {
  FS2_REQUIRE(f && wav && lens && status && ws, "%s: null argument", who);
  FS2_REQUIRE(f->loaded, "%s: weights not loaded (fs2_features_load)", who);
  FS2_REQUIRE(B >= 1 && B <= 65535 && Nmax > f->cfg.n_fft / 2, "%s: need 1 <= B <= 65535 and Nmax > n_fft/2 (got %d, %d)", who, B, Nmax);
  FS2_REQUIRE(Nmax < (1 << 30) && (long)B * (Nmax / f->cfg.hop + 1) * f->cpad < (1L << 40), "%s: batch too large", who);
  int dev = -1;
  FS2_CUDA_CHECK(cudaGetDevice(&dev));
  FS2_REQUIRE(dev == f->device, "%s: called on device %d, loaded on device %d", who, dev, f->device);
  return FS2_OK;
}

}  // namespace
}  // namespace fs2

using namespace fs2;

extern "C" {

int fs2_features_create(fs2_features** out, const fs2_features_config* cfg) {
  FS2_REQUIRE(out && cfg, "fs2_features_create: null argument");
  const fs2_features_config& c = *cfg;
  FS2_REQUIRE(c.sample_rate >= 1000 && c.sample_rate <= 96000, "fs2_features_create: sample_rate (%d) must lie in [1000, 96000]", c.sample_rate);
  FS2_REQUIRE(c.n_fft >= 16 && c.n_fft <= 4096 && c.n_fft % 16 == 0, "fs2_features_create: n_fft (%d) must be a multiple of 16 in [16, 4096]", c.n_fft);
  FS2_REQUIRE(c.hop >= 1 && c.hop <= c.n_fft / 2 && c.win_length >= 1 && c.win_length <= c.n_fft,
              "fs2_features_create: need 1 <= hop <= n_fft/2 and 1 <= win_length <= n_fft");
  FS2_REQUIRE(c.n_mels >= 16 && c.n_mels % 16 == 0, "fs2_features_create: n_mels (%d) must be a positive multiple of 16", c.n_mels);
  FS2_REQUIRE(c.math_mode >= FS2_MATH_FP32 && c.math_mode <= FS2_MATH_F16, "fs2_features_create: bad math_mode %d", c.math_mode);
  FS2_REQUIRE(c.f0_floor > 0 && c.f0_ceil > c.f0_floor && c.channels_in_octave > 0 && c.allowed_range > 0,
              "fs2_features_create: need 0 < f0_floor < f0_ceil, channels_in_octave > 0 and allowed_range > 0");
  const int n_bands = 1 + (int)(log(c.f0_ceil / c.f0_floor) / kLog2 * c.channels_in_octave);
  FS2_REQUIRE(n_bands <= kMaxBands, "fs2_features_create: %d DIO bands (at most %d)", n_bands, kMaxBands);
  fs2_features* f = new fs2_features();
  f->cfg = c;
  f->cutoff = c.n_fft / 2 + 1;
  f->cpad = (2 * f->cutoff + 63) / 64 * 64;
  f->mpad = (f->cutoff + 63) / 64 * 64;
  const double fs = (double)c.sample_rate;
  f->frame_period = (double)c.hop / fs * 1000.0;                    // the reference's hop / sample_rate * 1000
  f->n_bands = n_bands;
  for (int i = 0; i < n_bands; ++i) {
    f->boundary[i] = c.f0_floor * pow(2.0, (i + 1) / c.channels_in_octave);
    f->h[i] = matlab_round(fs / f->boundary[i] / 2.0);
  }
  f->pad = 2 * f->h[0];
  f->fft_extra = 4 * (int)(1.0 + fs / f->boundary[0] / 2.0);
  f->vrm = (int)(0.5 + 1000.0 / f->frame_period / c.f0_floor) * 2 + 1;
  // DesignLowCutFilter: delta minus the normalised Hann of N = 2M + 1 taps, centred; the normaliser summed in order
  const int M = matlab_round(fs / 50.0), N = 2 * M + 1;
  f->lc_half = M;
  const bool fits = (size_t)(4 * M + 1 + FT) * sizeof(double) <= 48 * 1024 && (size_t)(8 * f->h[0] + FT) * sizeof(double) <= 48 * 1024;
  if (!fits || f->h[n_bands - 1] < 1) {
    delete f;
    set_error("fs2_features_create: sample_rate / f0_floor give filters too long (or too short) for the FIR tiles");
    return FS2_ERR_INVALID;
  }
  std::vector<double>& t = f->taps_host;
  t.resize(N);
  double total = 0.0;
  for (int i = 1; i <= N; ++i) t[i - 1] = 0.5 - 0.5 * cos(i * 2.0 * 3.1415926535897932384 / (N + 1));
  for (int i = 0; i < N; ++i) total += t[i];
  for (int i = 0; i < N; ++i) t[i] = -t[i] / total;
  t[M] += 1.0;
  for (int j = 0; j < n_bands; ++j) {                                // NuttallWindow(4 h)
    const int L = 4 * f->h[j];
    f->nut_off[j] = (int)t.size();
    for (int i = 0; i < L; ++i) {
      const double x = i / (L - 1.0);
      t.push_back(0.355768 - 0.487396 * cos(2.0 * 3.1415926535897932384 * x) + 0.144232 * cos(4.0 * 3.1415926535897932384 * x) -
                  0.012604 * cos(6.0 * 3.1415926535897932384 * x));
    }
  }
  *out = f;
  return FS2_OK;
}

void fs2_features_destroy(fs2_features* f) {
  if (!f) return;
  if (f->arena) cudaFree(f->arena);
  delete f;
}

int fs2_features_load(fs2_features* f, const float* w_forward, const float* mel_basis, void* stream) {
  FS2_REQUIRE(f && w_forward && mel_basis, "fs2_features_load: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const int nf = f->cfg.n_fft;
  f->fwd.N = f->cpad; f->fwd.K = nf;
  f->mel.N = f->cfg.n_mels; f->mel.K = f->mpad;
  VWeight* ws[2] = {&f->fwd, &f->mel};
  for (int pass = 0; pass < 2; ++pass) {       // pass 0 sizes the arena, pass 1 carves it
    Bump b(pass ? f->arena : nullptr, pass ? (size_t)-1 : 0);
    for (VWeight* w : ws) {
      const size_t n = (size_t)w->N * w->K;
      w->w = b.floats(n); w->hi = (__half*)b.bytes(n * 2); w->lo = (__half*)b.bytes(n * 2); w->sc = b.floats(2);
    }
    f->taps = b.doubles(f->taps_host.size());
    if (pass == 0) {
      if (f->arena) { FS2_CUDA_CHECK(cudaStreamSynchronize(st)); FS2_CUDA_CHECK(cudaFree(f->arena)); f->arena = nullptr; }
      FS2_CUDA_CHECK(cudaMalloc(&f->arena, b.off + 256));
    }
  }
  FS2_CUDA_CHECK(cudaGetDevice(&f->device));
  int rc = vweight_pack(f->fwd, w_forward, 2 * f->cutoff, nf, 0, st); if (rc) return rc;
  rc = vweight_pack(f->mel, mel_basis, f->cfg.n_mels, f->cutoff, 0, st); if (rc) return rc;
  FS2_CUDA_CHECK(cudaMemcpyAsync(f->taps, f->taps_host.data(), f->taps_host.size() * sizeof(double), cudaMemcpyHostToDevice, st));
  FS2_CUDA_CHECK(cudaStreamSynchronize(st));   // the host taps must outlive the copy; loading is not on the hot path
  f->loaded = true;
  return FS2_OK;
}

int fs2_features_workspace_bytes(fs2_features* f, int B, int Nmax, size_t* bytes) {
  FS2_REQUIRE(f && bytes && B >= 0 && Nmax >= 0, "fs2_features_workspace_bytes: bad argument");
  Bump a(nullptr, 0), b(nullptr, 0);
  mel_plan(f, a, B, Nmax / f->cfg.hop + 1);
  dio_plan(f, b, B, Nmax);
  *bytes = (((a.off > b.off ? a.off : b.off) + 255) & ~(size_t)255) + 256;
  return FS2_OK;
}

int fs2_mel_energy(fs2_features* f, const float* wav, const int64_t* lens, int B, int Nmax, float* mel, float* energy, int* status,
                   void* ws, size_t ws_bytes, void* stream) {
  int rc = check_call(f, wav, lens, B, Nmax, status, ws, "fs2_mel_energy");
  if (rc) return rc;
  FS2_REQUIRE(mel && energy, "fs2_mel_energy: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const int T = Nmax / f->cfg.hop + 1, nf = f->cfg.n_fft, nm = f->cfg.n_mels, kind = out_kind(f->cfg.math_mode);
  Bump b(ws, ws_bytes);
  MelPlan p = mel_plan(f, b, B, T);
  if (!b.ok()) { set_error("fs2_mel_energy: workspace too small (%zu < %zu)", ws_bytes, b.off); return FS2_ERR_WORKSPACE; }
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  {
    auto k = pick(kind, feat_frames_kernel<OUT_HILO>, feat_frames_kernel<OUT_HI>, feat_frames_kernel<OUT_F32>);
    k<<<grid_for((long)B * T * (nf / 2), 256), 256, 0, st>>>(wav, lens, B, Nmax, T, nf, f->cfg.hop, (float*)p.frames, (__half*)p.frames,
                                                              p.flens, status);
    FS2_LAUNCH_CHECK();
  }
  if ((rc = vweight_gemm(f->cfg.math_mode, f->fwd, p.frames, B, T, ACT_NONE, p.flens, p.z, st))) return rc;
  {
    auto k = pick(kind, feat_magnitude_kernel<OUT_HILO>, feat_magnitude_kernel<OUT_HI>, feat_magnitude_kernel<OUT_F32>);
    k<<<grid_for((long)B * T * 32, 256), 256, 0, st>>>(p.z, f->cpad, f->cutoff, f->mpad, p.flens, B, T, (float*)p.mag, (__half*)p.mag, energy);
    FS2_LAUNCH_CHECK();
  }
  if ((rc = vweight_gemm(f->cfg.math_mode, f->mel, p.mag, B, T, ACT_NONE, p.flens, p.raw, st))) return rc;
  feat_log_kernel<<<grid_for((long)B * T * nm, 256), 256, 0, st>>>(p.raw, p.flens, B, T, nm, mel);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int fs2_dio(fs2_features* f, const float* wav, const int64_t* lens, int B, int Nmax, double* f0, int64_t* plens, int* status,
            void* ws, size_t ws_bytes, void* stream) {
  int rc = check_call(f, wav, lens, B, Nmax, status, ws, "fs2_dio");
  if (rc) return rc;
  FS2_REQUIRE(f0 && plens, "fs2_dio: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const int T = Nmax / f->cfg.hop + 1, M = f->lc_half, P = f->pad;
  const double fs = (double)f->cfg.sample_rate;
  Bump b(ws, ws_bytes);
  DioPlan p = dio_plan(f, b, B, Nmax);
  if (!b.ok()) { set_error("fs2_dio: workspace too small (%zu < %zu)", ws_bytes, b.off); return FS2_ERR_WORKSPACE; }
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  dio_prepare_kernel<<<B, 256, 0, st>>>(wav, lens, Nmax, f->cfg.n_fft / 2, f->cfg.hop, f->cfg.sample_rate, f->frame_period, f->fft_extra,
                                        p.Tp, p.meta, plens, status);
  FS2_LAUNCH_CHECK();
  {
    const dim3 grid((unsigned)((p.zs + FT - 1) / FT), B);
    dio_lowcut_kernel<<<grid, FT, (size_t)(4 * M + 1 + FT) * sizeof(double), st>>>(wav, Nmax, p.meta, f->taps, M, P, p.zs, p.z);
    FS2_LAUNCH_CHECK();
  }
  const dim3 band_grid((unsigned)((Nmax + 1 + FT - 1) / FT), B), frame_grid((unsigned)((p.Tp + 127) / 128), B);
  for (int j = 0; j < f->n_bands; ++j) {
    const int h = f->h[j];
    dio_band_kernel<<<band_grid, FT, (size_t)(8 * h - 1 + FT) * sizeof(double), st>>>(p.meta, p.z, p.zs, f->taps + f->nut_off[j], h, P, p.s, p.ss);
    FS2_LAUNCH_CHECK();
    dio_events_kernel<<<dim3(4, B), EV_THREADS, 0, st>>>(p.meta, p.s, p.ss, p.fine, p.es, p.count);
    FS2_LAUNCH_CHECK();
    dio_frames_kernel<<<frame_grid, 128, 0, st>>>(p.meta, p.fine, p.es, p.count, B, p.Tp, j, f->boundary[j], f->cfg.f0_floor, f->cfg.f0_ceil,
                                                  fs, f->frame_period, p.cand, p.best_f0, p.best_score);
    FS2_LAUNCH_CHECK();
  }
  dio_fix_kernel<<<B, 32, 0, st>>>(p.meta, p.best_f0, p.cand, B, p.Tp, f->n_bands, f->vrm, f->cfg.allowed_range, p.t1, p.t2, plens, f0, T);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // extern "C"
