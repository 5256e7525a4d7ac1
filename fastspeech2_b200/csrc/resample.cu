// Band-limited resampling (DESIGN.md section 22): what the reference's preprocessing gets from librosa.load(path, sr=...)
// for a file at another rate, i.e. resampy 0.2.x's kaiser_best `resample_f` followed by librosa's fix_length, for a
// ragged batch of mono utterances at one (sr_orig, sr_new) pair.
//
//   rs_clock_kernel  one CTA per utterance: lane 0 of warp 0 runs the time register, a running float64 sum (t = 0, 1,
//                    ... adds 1 / ratio each step, exactly resampy's dependent chain), into the workspace; warps 1.. check
//                    the utterance's samples for NaN / inf meanwhile
//   rs_taps_kernel   one thread per output sample walks the left wing, then the right wing, of the interpolated
//                    Kaiser-sinc table (win and delta interleaved as double2: one 16-byte load per tap), rounding the
//                    output to float32 after every tap as resampy's float32 output array does
// Every double product and sum is __dmul_rn / __dadd_rn, so nothing is contracted into an FMA: the output is bit-identical
// to the float64 restatement in oracle/resample_oracle.py, and an utterance's output does not depend on its batch mates.
#include <math.h>

#include "common.cuh"

namespace fs2 {
namespace {

constexpr int kRsTable = 512;                // table entries per zero crossing (resampy's precision 9)
constexpr int kClockThreads = 256;
constexpr int kTapThreads = 128;

struct RsParams {
  double ratio, time_increment, scale;       // sr_new / sr_orig, 1 / ratio (not sr_orig / sr_new), min(1, ratio)
  int index_step;                            // int(scale * 512), truncated as resampy does
};

// (n_out, M) of an utterance of N samples: int(N * ratio) and ceil(N * ratio); (0, 0) when N is outside [1, Nmax] or
// n_out < 1.
__device__ __forceinline__ void rs_lengths(int64_t N, int Nmax, double ratio, long long& n_out, long long& M) {
  n_out = M = 0;
  if (N < 1 || N > Nmax) return;
  const double p = __dmul_rn((double)N, ratio);
  if ((long long)p < 1) return;
  n_out = (long long)p;
  M = (long long)ceil(p);
}

__global__ void __launch_bounds__(kClockThreads) rs_clock_kernel(const float* __restrict__ x, const int64_t* __restrict__ lens, int Nmax,
                                                                  RsParams p, double* __restrict__ reg, long Mmax,
                                                                  int64_t* __restrict__ olens, int* __restrict__ status) {
  const int b = blockIdx.x;
  const int64_t N = lens[b];
  long long n_out, M;
  rs_lengths(N, Nmax, p.ratio, n_out, M);
  if (n_out == 0) {
    if (threadIdx.x == 0) {
      olens[b] = 0;
      atomicOr(status, FS2_RS_BAD_LENGTH);
    }
    return;
  }
  if (threadIdx.x < 32) {
    if (threadIdx.x == 0) {
      olens[b] = M;
      double* r = reg + (size_t)b * Mmax;
      double tr = 0.0;
      for (long long t = 0; t < n_out; ++t) {
        r[t] = tr;
        tr = __dadd_rn(tr, p.time_increment);
      }
    }
    return;
  }
  const float* xb = x + (size_t)b * Nmax;
  bool finite = true;
  for (int64_t i = threadIdx.x - 32; i < N; i += blockDim.x - 32) finite &= isfinite(__ldg(xb + i));
  if (__any_sync(0xffffffffu, !finite) && (threadIdx.x & 31) == 0) atomicOr(status, FS2_RS_NONFINITE);
}

// One wing of resampy's loop: count taps from sample src, stepping dir, at table offset int(frac * 512) + i * index_step.
__device__ __forceinline__ float rs_wing(float y, const double2* __restrict__ tab, const float* __restrict__ x, long long src, int dir,
                                         long long count, double frac, int step) {
  const double index_frac = __dmul_rn(frac, (double)kRsTable);
  const int offset = (int)index_frac;
  const double eta = __dsub_rn(index_frac, (double)offset);
  const long long lim = (FS2_RESAMPLE_TABLE - offset) / step;
  if (count > lim) count = lim;
  int j = offset;
  for (long long i = 0; i < count; ++i, j += step, src += dir) {
    const double2 e = __ldg(tab + j);
    const double w = __dadd_rn(e.x, __dmul_rn(eta, e.y));
    y = __double2float_rn(__dadd_rn((double)y, __dmul_rn(w, (double)__ldg(x + src))));
  }
  return y;
}

// y[b, t] for every t < Mmax: resampy's output for t < n_out, +0 past it and for a refused utterance.
__global__ void __launch_bounds__(kTapThreads) rs_taps_kernel(const float* __restrict__ x, const int64_t* __restrict__ lens, int B, int Nmax,
                                                               const double2* __restrict__ tab, RsParams p, const double* __restrict__ reg,
                                                               float* __restrict__ y, long Mmax) {
  const long total = (long)B * Mmax;
  for (long e = (long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
    const int b = (int)(e / Mmax);
    const long t = e - (long)b * Mmax;
    const int64_t N = lens[b];
    long long n_out, M;
    rs_lengths(N, Nmax, p.ratio, n_out, M);
    float out = 0.0f;
    if (t < n_out) {
      const double tr = reg[e];
      const long long n = (long long)tr;        // tr <= N - 1 + (rounding far below 1 / ratio): see the Mmax limit
      const double frac = __dmul_rn(p.scale, __dsub_rn(tr, (double)n));
      const float* xb = x + (size_t)b * Nmax;
      out = rs_wing(out, tab, xb, n, -1, n + 1, frac, p.index_step);
      out = rs_wing(out, tab, xb, n + 1, 1, N - n - 1, __dsub_rn(p.scale, frac), p.index_step);
    }
    y[e] = out;
  }
}

int check_sizes(int B, int Nmax, int sr_orig, int sr_new, int Mmax, RsParams* p, const char* who) {
  FS2_REQUIRE(B >= 1 && B <= (1 << 20), "%s: B (%d) must lie in [1, 2^20]", who, B);
  FS2_REQUIRE(Nmax >= 1, "%s: Nmax (%d) must be >= 1", who, Nmax);
  FS2_REQUIRE(sr_orig >= 1 && sr_new >= 1 && sr_orig <= (1 << 24) && sr_new <= (1 << 24),
              "%s: sample rates (%d, %d) must lie in [1, 2^24]", who, sr_orig, sr_new);
  FS2_REQUIRE(sr_orig != sr_new, "%s: equal sample rates (%d): the input is its own output, there is nothing to run", who, sr_orig);
  const double ratio = (double)sr_new / (double)sr_orig;
  const double scale = ratio < 1.0 ? ratio : 1.0;
  const int step = (int)(scale * kRsTable);
  FS2_REQUIRE(step >= 1, "%s: downsampling by more than 512 (%d -> %d Hz) leaves no tap step", who, sr_orig, sr_new);
  const double m = ceil((double)Nmax * ratio);
  FS2_REQUIRE(Mmax >= m && Mmax < (1 << 26), "%s: Mmax (%d) must lie in [ceil(Nmax * ratio) = %.0f, 2^26)", who, Mmax, m);
  if (p) *p = RsParams{ratio, 1.0 / ratio, scale, step};
  return FS2_OK;
}

}  // namespace
}  // namespace fs2

using namespace fs2;

extern "C" {

int fs2_resample_workspace_bytes(int B, int Nmax, int sr_orig, int sr_new, int Mmax, size_t* bytes) {
  FS2_REQUIRE(bytes, "fs2_resample_workspace_bytes: null argument");
  int rc = check_sizes(B, Nmax, sr_orig, sr_new, Mmax, nullptr, "fs2_resample_workspace_bytes");
  if (rc) return rc;
  *bytes = align256((size_t)B * Mmax * sizeof(double)) + 256;
  return FS2_OK;
}

int fs2_resample(const float* x, const int64_t* lens, int B, int Nmax, const double* table, int sr_orig, int sr_new, float* y,
                 int64_t* olens, int Mmax, int* status, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(x && lens && table && y && olens && status && ws, "fs2_resample: null argument");
  RsParams p;
  int rc = check_sizes(B, Nmax, sr_orig, sr_new, Mmax, &p, "fs2_resample");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Bump bump(ws, ws_bytes);
  double* reg = bump.doubles((size_t)B * Mmax);
  if ((rc = bump.check("fs2_resample"))) return rc;
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  rs_clock_kernel<<<B, kClockThreads, 0, st>>>(x, lens, Nmax, p, reg, Mmax, olens, status);
  FS2_LAUNCH_CHECK();
  rs_taps_kernel<<<grid_for((long)B * Mmax, kTapThreads, 132 * 16), kTapThreads, 0, st>>>(x, lens, B, Nmax, (const double2*)table, p, reg,
                                                                                          y, Mmax);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // extern "C"
