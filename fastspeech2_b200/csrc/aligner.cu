// Unsupervised duration aligner (DESIGN.md section 24): the hot path of Badlani et al.'s alignment module (FastPitch 1.1's
// AlignmentEncoder, forward-sum and binarization losses, mas_width1) for a ragged batch.  Queries q [B, L, 80] (frames),
// keys k [B, T, 80] (phonemes), lengths olens (frames) and ilens (phonemes) per utterance.
//
//   al_check_kernel       one CTA per utterance: length checks and NaN / inf in q[:olens], k[:ilens] -> flags[b], status
//   al_logprob_kernel     one warp per frame: sum-of-squares distances, log-softmax over the utterance's own phonemes, the
//                         beta-binomial prior in float64 (lgamma) -> logp
//   al_logprob_dq_kernel  one warp per frame: recomputed softmax, ds = dlogp - p * sum(dlogp) (to the workspace), dq
//   al_logprob_dk_kernel  one warp per phoneme: dk summed over frames in ascending order
//   al_forward_sum_kernel one CTA per utterance: CTC alpha (and beta + the gradient) in log space over 2 ilens + 1 states
//   al_mas_kernel         one CTA per utterance: mas_width1 on log softmax(logp), backtracked in 32-row windows
//   al_bin_loss_kernel    one CTA per utterance: -mean log soft[l, path(l)] and its gradient
//   al_mask_rows_kernel   rows t >= lens[b] of a [B, L, C] activation set to +0 (before every convolution)
// Float32 on the CUDA cores, no floating-point atomics: every sum has a fixed order that depends only on the utterance's
// own lengths, so an utterance's outputs are bit-identical to its B = 1 call.  The status word is OR-ed.
#include <math.h>

#include "common.cuh"

namespace fs2 {
namespace {

constexpr int kD = FS2_ALIGN_DIM;
constexpr int kMaxT = FS2_ALIGN_MAX_T;
constexpr float kTemp = 0.0005f;              // FastPitch's attention temperature
constexpr int kRowWarps = 8;                  // frames (or phonemes) per CTA of the logprob kernels, one warp each
constexpr int kLatThreads = 256;              // threads of the per-utterance kernels
constexpr int kDj = (kD + 31) / 32;           // channels per lane

__device__ __forceinline__ int utt_bits(int64_t N, int64_t M, int L, int T) {
  if (N < 1 || N > T || M < 1 || M > L) return FS2_ALIGN_BAD_LENGTH;
  return M < N ? FS2_ALIGN_INFEASIBLE : 0;
}

// log a + log b without overflow; -inf when both are -inf
__device__ __forceinline__ float lae(float a, float b) {
  const float m = fmaxf(a, b);
  if (m == -INFINITY) return -INFINITY;
  return m + log1pf(expf(fminf(a, b) - m));
}

__global__ void __launch_bounds__(kLatThreads) al_check_kernel(const float* __restrict__ q, const float* __restrict__ k,
                                                                const int64_t* __restrict__ ilens, const int64_t* __restrict__ olens,
                                                                int L, int T, int* __restrict__ flags, int* __restrict__ status) {
  const int b = blockIdx.x;
  int bits = utt_bits(ilens[b], olens[b], L, T);
  bool bad = false;
  if (!bits) {
    const long nq = olens[b] * kD, nk = ilens[b] * kD;
    const float* qb = q + (size_t)b * L * kD;
    const float* kb = k + (size_t)b * T * kD;
    for (long i = threadIdx.x; i < nq; i += blockDim.x) bad |= !isfinite(__ldg(qb + i));
    for (long i = threadIdx.x; i < nk; i += blockDim.x) bad |= !isfinite(__ldg(kb + i));
  }
  bad = __syncthreads_or(bad);
  if (threadIdx.x == 0) {
    if (bad) bits |= FS2_ALIGN_NONFINITE;
    flags[b] = bits;
    if (bits) atomicOr(status, bits);
  }
}

// -0.0005 * sum_c (q[c] - k[c])^2 of one (frame, phoneme) pair; lane j holds q[c] for c = j, j + 32, j + 64.  The xor
// butterfly leaves the same bits in every lane.
__device__ __forceinline__ float al_score(const float (&qv)[kDj], const float* __restrict__ kt, int lane) {
  float d = 0.f;
#pragma unroll
  for (int j = 0; j < kDj; ++j) {
    const int c = lane + 32 * j;
    if (c < kD) {
      const float e = qv[j] - __ldg(kt + c);
      d = fmaf(e, e, d);
    }
  }
  return -kTemp * warp_sum(d);
}

__device__ __forceinline__ void al_load_row(float (&v)[kDj], const float* __restrict__ row, int lane) {
#pragma unroll
  for (int j = 0; j < kDj; ++j) v[j] = lane + 32 * j < kD ? __ldg(row + lane + 32 * j) : 0.f;
}

// Scores of frame l against phonemes t < N into row[t] (lane t % 32 writes, and later reads, entry t); returns
// their log-sum-exp (all lanes).
__device__ float al_scores_lse(const float (&qv)[kDj], const float* __restrict__ kb, int N, float* row, int lane) {
  float m = -INFINITY;
  for (int t = 0; t < N; ++t) {
    const float s = al_score(qv, kb + (size_t)t * kD, lane);
    if (lane == (t & 31)) row[t] = s;
    m = fmaxf(m, s);
  }
  float sum = 0.f;
  for (int t = lane; t < N; t += 32) sum += expf(row[t] - m);
  return m + logf(warp_sum(sum));
}

__global__ void __launch_bounds__(kRowWarps * 32) al_logprob_kernel(const float* __restrict__ q, const float* __restrict__ k,
                                                                    const int64_t* __restrict__ ilens, const int64_t* __restrict__ olens,
                                                                    int L, int T, const int* __restrict__ flags, float* __restrict__ logp) {
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const int l = blockIdx.x * kRowWarps + (threadIdx.x >> 5);
  if (l >= L) return;
  float* out = logp + ((size_t)b * L + l) * T;
  const int N = flags[b] ? 0 : (int)ilens[b], M = flags[b] ? 0 : (int)olens[b];
  if (l >= M) {
    for (int t = lane; t < T; t += 32) out[t] = 0.f;
    return;
  }
  float qv[kDj];
  al_load_row(qv, q + ((size_t)b * L + l) * kD, lane);
  const float lse = al_scores_lse(qv, k + (size_t)b * T * kD, N, out, lane);
  // betabinom(N, a = l + 1, b = M - l).pmf(t) = C(N, t) B(t + a, N - t + b) / B(a, b), in float64
  const double a = l + 1.0, bb = (double)(M - l);
  const double rowc = lgamma(N + 1.0) - lgamma(N + a + bb) - lgamma(a) - lgamma(bb) + lgamma(a + bb);
  for (int t = lane; t < N; t += 32) {
    const double lpmf = rowc - lgamma(t + 1.0) - lgamma(N - t + 1.0) + lgamma(t + a) + lgamma(N - t + bb);
    out[t] = (out[t] - lse) + (float)log(exp(lpmf) + 1e-8);
  }
  for (int t = N + lane; t < T; t += 32) out[t] = 0.f;
}

__global__ void __launch_bounds__(kRowWarps * 32) al_logprob_dq_kernel(const float* __restrict__ q, const float* __restrict__ k,
                                                                       const int64_t* __restrict__ ilens, const int64_t* __restrict__ olens,
                                                                       int L, int T, const int* __restrict__ flags,
                                                                       const float* __restrict__ dlogp, float* __restrict__ ds,
                                                                       float* __restrict__ dq) {
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const int l = blockIdx.x * kRowWarps + (threadIdx.x >> 5);
  if (l >= L) return;
  float* dqr = dq + ((size_t)b * L + l) * kD;
  const int N = flags[b] ? 0 : (int)ilens[b], M = flags[b] ? 0 : (int)olens[b];
  if (l >= M) {
    for (int c = lane; c < kD; c += 32) dqr[c] = 0.f;
    return;
  }
  float qv[kDj];
  al_load_row(qv, q + ((size_t)b * L + l) * kD, lane);
  const float* kb = k + (size_t)b * T * kD;
  float* dsr = ds + ((size_t)b * L + l) * T;
  const float* dlr = dlogp + ((size_t)b * L + l) * T;
  const float lse = al_scores_lse(qv, kb, N, dsr, lane);
  float g = 0.f;
  for (int t = lane; t < N; t += 32) g += dlr[t];
  g = warp_sum(g);
  for (int t = lane; t < N; t += 32) dsr[t] = dlr[t] - expf(dsr[t] - lse) * g;
  __syncwarp();
  float acc[kDj] = {};
  for (int t = 0; t < N; ++t) {
    const float d = dsr[t];
    const float* kt = kb + (size_t)t * kD;
#pragma unroll
    for (int j = 0; j < kDj; ++j)
      if (lane + 32 * j < kD) acc[j] = fmaf(d, qv[j] - __ldg(kt + lane + 32 * j), acc[j]);
  }
#pragma unroll
  for (int j = 0; j < kDj; ++j)
    if (lane + 32 * j < kD) dqr[lane + 32 * j] = -2.f * kTemp * acc[j];
}

__global__ void __launch_bounds__(kRowWarps * 32) al_logprob_dk_kernel(const float* __restrict__ q, const float* __restrict__ k,
                                                                       const int64_t* __restrict__ ilens, const int64_t* __restrict__ olens,
                                                                       int L, int T, const int* __restrict__ flags,
                                                                       const float* __restrict__ ds, float* __restrict__ dk) {
  const int b = blockIdx.y, lane = threadIdx.x & 31;
  const int t = blockIdx.x * kRowWarps + (threadIdx.x >> 5);
  if (t >= T) return;
  float* dkr = dk + ((size_t)b * T + t) * kD;
  const int N = flags[b] ? 0 : (int)ilens[b], M = flags[b] ? 0 : (int)olens[b];
  if (t >= N) {
    for (int c = lane; c < kD; c += 32) dkr[c] = 0.f;
    return;
  }
  float kv[kDj];
  al_load_row(kv, k + ((size_t)b * T + t) * kD, lane);
  const float* qb = q + (size_t)b * L * kD;
  const float* dsc = ds + (size_t)b * L * T + t;
  float acc[kDj] = {};
#pragma unroll 4
  for (int l = 0; l < M; ++l) {
    const float d = dsc[(size_t)l * T];
    const float* qr = qb + (size_t)l * kD;
#pragma unroll
    for (int j = 0; j < kDj; ++j)
      if (lane + 32 * j < kD) acc[j] = fmaf(d, __ldg(qr + lane + 32 * j) - kv[j], acc[j]);
  }
#pragma unroll
  for (int j = 0; j < kDj; ++j)
    if (lane + 32 * j < kD) dkr[lane + 32 * j] = 2.f * kTemp * acc[j];
}

// Zeroes an utterance's [L, T] slice (a refused utterance's gradient).
__device__ __forceinline__ void al_zero_slice(float* p, int L, int T) {
  for (size_t i = threadIdx.x; i < (size_t)L * T; i += blockDim.x) p[i] = 0.f;
}

// Per-frame log-sum-exp of logp[l, :N] (with the blank's constant logit -1 when `blank`) into lse[l], one thread per frame,
// phonemes in ascending order; returns (block-wide) whether any logp[l < M, t < N] is NaN or inf.
__device__ bool al_row_lse(const float* __restrict__ lp, int M, int N, int T, bool blank, float* __restrict__ lse) {
  bool bad = false;
  for (int l = threadIdx.x; l < M; l += blockDim.x) {
    const float* r = lp + (size_t)l * T;
    float m = blank ? -1.f : -INFINITY;
    for (int t = 0; t < N; ++t) {
      const float v = r[t];
      bad |= !isfinite(v);
      m = fmaxf(m, v);
    }
    float s = blank ? expf(-1.f - m) : 0.f;
    for (int t = 0; t < N; ++t) s += expf(r[t] - m);
    lse[l] = m + logf(s);
  }
  return __syncthreads_or(bad);
}

__global__ void __launch_bounds__(kLatThreads) al_forward_sum_kernel(const float* __restrict__ logp, const int64_t* __restrict__ ilens,
                                                                      const int64_t* __restrict__ olens, int L, int T,
                                                                      const float* __restrict__ dloss, float* __restrict__ loss,
                                                                      float* __restrict__ dlogp, float* __restrict__ lse_ws,
                                                                      float* __restrict__ alpha_ws, int* __restrict__ status) {
  __shared__ float sa[2][2 * kMaxT + 1];
  const int b = blockIdx.x, tid = threadIdx.x;
  int bits = utt_bits(ilens[b], olens[b], L, T);
  const int N = bits ? 0 : (int)ilens[b], M = bits ? 0 : (int)olens[b];
  const float* lp = logp + (size_t)b * L * T;
  float* lse = lse_ws + (size_t)b * L;
  float* gout = dlogp ? dlogp + (size_t)b * L * T : nullptr;
  if (al_row_lse(lp, M, N, T, true, lse)) bits |= FS2_ALIGN_NONFINITE;
  if (bits) {
    if (tid == 0) {
      loss[b] = 0.f;
      atomicOr(status, bits);
    }
    if (gout) al_zero_slice(gout, L, T);
    return;
  }
  const int S = 2 * N + 1, ST = 2 * T + 1;
  float* A = alpha_ws + (size_t)b * L * ST;
  // log-softmax over [blank, labels] of frame l at state s: s even = blank, s = 2i + 1 = phoneme i
  auto emit = [&](int l, int s) { return ((s & 1) ? lp[(size_t)l * T + (s >> 1)] : -1.f) - lse[l]; };
  for (int s = tid; s < S; s += blockDim.x) {
    const float a = s < 2 ? emit(0, s) : -INFINITY;
    sa[0][s] = a;
    if (gout) A[s] = a;
  }
  __syncthreads();
  for (int l = 1; l < M; ++l) {
    const float* pv = sa[(l - 1) & 1];
    float* cv = sa[l & 1];
    for (int s = tid; s < S; s += blockDim.x) {
      float v = pv[s];
      if (s >= 1) v = lae(v, pv[s - 1]);
      if ((s & 1) && s >= 3) v = lae(v, pv[s - 2]);
      v += emit(l, s);
      cv[s] = v;
      if (gout) A[(size_t)l * ST + s] = v;
    }
    __syncthreads();
  }
  const float* fin = sa[(M - 1) & 1];
  const float nll = -lae(fin[S - 1], fin[S - 2]);
  const bool ok = isfinite(nll);
  if (tid == 0) loss[b] = ok ? nll / (float)N : 0.f;
  if (!gout) return;
  __syncthreads();                            // every thread has read fin before the beta pass reuses sa
  if (!ok) {
    al_zero_slice(gout, L, T);
    return;
  }
  const float scale = (dloss ? dloss[b] : 1.f) / (float)N;
  for (size_t i = tid; i < (size_t)(L - M) * T; i += blockDim.x) gout[(size_t)M * T + i] = 0.f;
  for (size_t i = tid; i < (size_t)M * (T - N); i += blockDim.x) gout[(i / (T - N)) * T + N + i % (T - N)] = 0.f;
  // beta (emission of frame l included), occupancy of phoneme i = exp(alpha + beta - emit + nll) at state 2i + 1
  for (int l = M - 1; l >= 0; --l) {
    const float* nv = sa[(l + 1) & 1];
    float* cv = sa[l & 1];
    for (int s = tid; s < S; s += blockDim.x) {
      const float e = emit(l, s);
      float v;
      if (l == M - 1) {
        v = s >= S - 2 ? e : -INFINITY;
      } else {
        v = nv[s];
        if (s + 1 < S) v = lae(v, nv[s + 1]);
        if ((s & 1) && s + 2 < S) v = lae(v, nv[s + 2]);
        v += e;
      }
      cv[s] = v;
      if (s & 1) {
        const float occ = expf(A[(size_t)l * ST + s] + v - e + nll);
        gout[(size_t)l * T + (s >> 1)] = scale * (expf(e) - occ);
      }
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kLatThreads) al_mas_kernel(const float* __restrict__ logp, const int64_t* __restrict__ ilens,
                                                              const int64_t* __restrict__ olens, int L, int T, int64_t* __restrict__ dur,
                                                              int32_t* __restrict__ path, float* __restrict__ lse_ws,
                                                              uint8_t* __restrict__ dir_ws, int* __restrict__ status) {
  __shared__ float sv[2][kMaxT];
  __shared__ int cnt[kMaxT];
  __shared__ uint8_t win[32][33];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
  int bits = utt_bits(ilens[b], olens[b], L, T);
  const int N = bits ? 0 : (int)ilens[b], M = bits ? 0 : (int)olens[b];
  const float* lp = logp + (size_t)b * L * T;
  float* lse = lse_ws + (size_t)b * L;
  uint8_t* dir = dir_ws + (size_t)b * L * T;
  // log-sum-exp of each frame in float64 (exp of the float32 differences, summed in phoneme order), rounded once: the
  // same operations as the numpy oracle, so log soft = logp - lse is the same float32 on both sides
  bool bad = false;
  for (int l = tid; l < M; l += blockDim.x) {
    const float* r = lp + (size_t)l * T;
    float m = -INFINITY;
    for (int t = 0; t < N; ++t) {
      bad |= !isfinite(r[t]);
      m = fmaxf(m, r[t]);
    }
    double s = 0.0;
    for (int t = 0; t < N; ++t) s += exp((double)r[t] - (double)m);
    lse[l] = (float)((double)m + log(s));
  }
  if (__syncthreads_or(bad)) bits |= FS2_ALIGN_NONFINITE;
  for (int t = tid; t < T; t += blockDim.x) cnt[t] = 0;
  int32_t* pb = path + (size_t)b * L;
  for (int l = (bits ? 0 : M) + tid; l < L; l += blockDim.x) pb[l] = -1;
  if (bits) {
    if (tid == 0) atomicOr(status, bits);
    for (int t = tid; t < T; t += blockDim.x) dur[(size_t)b * T + t] = 0;
    return;
  }
  // v[l, t] = log soft[l, t] + max(v[l-1, t], v[l-1, t-1]), the t-1 predecessor winning ties; row 0 starts at t = 0
  for (int t = tid; t < N; t += blockDim.x) sv[0][t] = t == 0 ? lp[0] - lse[0] : -INFINITY;
  __syncthreads();
  for (int l = 1; l < M; ++l) {
    const float* pv = sv[(l - 1) & 1];
    float* cv = sv[l & 1];
    const float lsel = lse[l];
    for (int t = tid; t < N; t += blockDim.x) {
      float p = pv[t];
      uint8_t d = 0;
      if (t >= 1 && pv[t - 1] >= p) {
        p = pv[t - 1];
        d = 1;
      }
      cv[t] = (lp[(size_t)l * T + t] - lsel) + p;
      dir[(size_t)l * T + t] = d;
    }
    __syncthreads();
  }
  // backtrack from (M - 1, N - 1): warp 0 stages the 32 x 32 window of decisions the next 32 rows can reach
  if (tid < 32) {
    int l = M - 1, t = N - 1;
    while (l >= 0) {
      for (int r = 0; r < 32; ++r) {
        const int ll = l - r, tt = t - lane;
        win[r][lane] = (ll >= 1 && tt >= 0) ? dir[(size_t)ll * T + tt] : 0;
      }
      __syncwarp();
      if (lane == 0) {
        const int top = t;
        for (int r = 0; r < 32 && l >= 0; ++r, --l) {
          pb[l] = t;
          ++cnt[t];
          t -= win[r][top - t];
        }
      }
      l = __shfl_sync(0xffffffffu, l, 0);
      t = __shfl_sync(0xffffffffu, t, 0);
      __syncwarp();
    }
  }
  __syncthreads();
  for (int t = tid; t < T; t += blockDim.x) dur[(size_t)b * T + t] = cnt[t];
}

__global__ void __launch_bounds__(kLatThreads) al_bin_loss_kernel(const float* __restrict__ logp, const int32_t* __restrict__ path,
                                                                   const int64_t* __restrict__ ilens, const int64_t* __restrict__ olens,
                                                                   int L, int T, const float* __restrict__ dloss, float* __restrict__ loss,
                                                                   float* __restrict__ dlogp, float* __restrict__ lse_ws,
                                                                   int* __restrict__ status) {
  __shared__ float part[kLatThreads / 32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int bits = utt_bits(ilens[b], olens[b], L, T);
  const int N = bits ? 0 : (int)ilens[b], M = bits ? 0 : (int)olens[b];
  const float* lp = logp + (size_t)b * L * T;
  const int32_t* pb = path + (size_t)b * L;
  float* gout = dlogp ? dlogp + (size_t)b * L * T : nullptr;
  bool badpath = false;
  for (int l = tid; l < M; l += blockDim.x) badpath |= pb[l] < 0 || pb[l] >= N;
  if (__syncthreads_or(badpath)) bits |= FS2_ALIGN_BAD_LENGTH;
  if (!bits && al_row_lse(lp, M, N, T, false, lse_ws + (size_t)b * L)) bits |= FS2_ALIGN_NONFINITE;
  if (bits) {
    if (tid == 0) {
      loss[b] = 0.f;
      atomicOr(status, bits);
    }
    if (gout) al_zero_slice(gout, L, T);
    return;
  }
  const float* lse = lse_ws + (size_t)b * L;
  const float scale = (dloss ? dloss[b] : 1.f) / (float)M;
  float acc = 0.f;                            // lane 0 of each warp: its frames in ascending order
  for (int l = warp; l < L; l += kLatThreads / 32) {
    float* g = gout ? gout + (size_t)l * T : nullptr;
    if (l >= M) {
      if (g)
        for (int t = lane; t < T; t += 32) g[t] = 0.f;
      continue;
    }
    const float* r = lp + (size_t)l * T;
    const int j = pb[l];
    const float p = expf(r[j] - lse[l]);
    acc += logf(fmaxf(p, 1e-12f));
    if (g) {
      const float s = p >= 1e-12f ? scale : 0.f;
      for (int t = lane; t < N; t += 32) g[t] = s * (expf(r[t] - lse[l]) - (t == j ? 1.f : 0.f));
      for (int t = N + lane; t < T; t += 32) g[t] = 0.f;
    }
  }
  if (lane == 0) part[warp] = acc;
  __syncthreads();
  if (tid == 0) {
    float s = 0.f;
    for (int w = 0; w < kLatThreads / 32; ++w) s += part[w];
    loss[b] = -s / (float)M;
  }
}

__global__ void al_mask_rows_kernel(const float* __restrict__ x, const int64_t* __restrict__ lens, int L, int C, long n,
                                    float* __restrict__ y) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long row = i / C;
    y[i] = (row % L) < lens[row / L] ? x[i] : 0.f;
  }
}

// The workspace carve every entry shares: per-utterance flags, per-frame log-sum-exp, and the [B, L, 2T + 1] float
// buffer (forward-sum alpha; logprob backward ds; MAS decisions use its first B L T bytes).
struct AlWs {
  int* flags; float* lse; float* big;
};

int al_carve(int B, int L, int T, void* ws, size_t ws_bytes, AlWs* w, size_t* need, const char* who) {
  FS2_REQUIRE(B >= 1 && B <= 65535, "%s: B (%d) must lie in [1, 65535]", who, B);
  FS2_REQUIRE(L >= 1 && L <= (1 << 20), "%s: L (%d) must lie in [1, 2^20]", who, L);
  FS2_REQUIRE(T >= 1 && T <= kMaxT, "%s: T (%d) must lie in [1, %d]", who, T, kMaxT);
  FS2_REQUIRE((double)B * L * (2.0 * T + 1) < 4e12 && (double)B * L * T < 2e12, "%s: B * L * T (%d * %d * %d) is too large", who, B, L, T);
  Bump bump(ws, ws_bytes);
  AlWs r;
  r.flags = (int*)bump.bytes((size_t)B * sizeof(int));
  r.lse = bump.floats((size_t)B * L);
  r.big = bump.floats((size_t)B * L * (2 * (size_t)T + 1));
  if (need) *need = bump.off;
  if (w) {
    FS2_REQUIRE(ws && ((uintptr_t)ws & 255) == 0, "%s: workspace must be non-null and 256-byte aligned", who);
    *w = r;
    return bump.check(who);
  }
  return FS2_OK;
}

inline dim3 rows_grid(int rows, int B) { return dim3((unsigned)((rows + kRowWarps - 1) / kRowWarps), (unsigned)B); }

}  // namespace
}  // namespace fs2

using namespace fs2;

extern "C" {

int fs2_align_workspace_bytes(int B, int L, int T, size_t* bytes) {
  FS2_REQUIRE(bytes, "fs2_align_workspace_bytes: null argument");
  return al_carve(B, L, T, nullptr, 0, nullptr, bytes, "fs2_align_workspace_bytes");
}

int fs2_align_logprob(const float* q, const float* k, const int64_t* ilens, const int64_t* olens, int B, int L, int T, float* logp,
                      int* status, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(q && k && ilens && olens && logp && status, "fs2_align_logprob: null argument");
  AlWs w;
  int rc = al_carve(B, L, T, ws, ws_bytes, &w, nullptr, "fs2_align_logprob");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  al_check_kernel<<<B, kLatThreads, 0, st>>>(q, k, ilens, olens, L, T, w.flags, status);
  FS2_LAUNCH_CHECK();
  al_logprob_kernel<<<rows_grid(L, B), kRowWarps * 32, 0, st>>>(q, k, ilens, olens, L, T, w.flags, logp);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int fs2_align_logprob_backward(const float* q, const float* k, const int64_t* ilens, const int64_t* olens, int B, int L, int T,
                               const float* dlogp, float* dq, float* dk, int* status, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(q && k && ilens && olens && dlogp && dq && dk && status, "fs2_align_logprob_backward: null argument");
  AlWs w;
  int rc = al_carve(B, L, T, ws, ws_bytes, &w, nullptr, "fs2_align_logprob_backward");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  al_check_kernel<<<B, kLatThreads, 0, st>>>(q, k, ilens, olens, L, T, w.flags, status);
  FS2_LAUNCH_CHECK();
  al_logprob_dq_kernel<<<rows_grid(L, B), kRowWarps * 32, 0, st>>>(q, k, ilens, olens, L, T, w.flags, dlogp, w.big, dq);
  FS2_LAUNCH_CHECK();
  al_logprob_dk_kernel<<<rows_grid(T, B), kRowWarps * 32, 0, st>>>(q, k, ilens, olens, L, T, w.flags, w.big, dk);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int fs2_align_forward_sum(const float* logp, const int64_t* ilens, const int64_t* olens, int B, int L, int T, const float* dloss,
                          float* loss, float* dlogp, int* status, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(logp && ilens && olens && loss && status, "fs2_align_forward_sum: null argument");
  AlWs w;
  int rc = al_carve(B, L, T, ws, ws_bytes, &w, nullptr, "fs2_align_forward_sum");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  al_forward_sum_kernel<<<B, kLatThreads, 0, st>>>(logp, ilens, olens, L, T, dloss, loss, dlogp, w.lse, w.big, status);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int fs2_align_mas(const float* logp, const int64_t* ilens, const int64_t* olens, int B, int L, int T, int64_t* durations,
                  int32_t* path, int* status, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(logp && ilens && olens && durations && path && status, "fs2_align_mas: null argument");
  AlWs w;
  int rc = al_carve(B, L, T, ws, ws_bytes, &w, nullptr, "fs2_align_mas");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  al_mas_kernel<<<B, kLatThreads, 0, st>>>(logp, ilens, olens, L, T, durations, path, w.lse, (uint8_t*)w.big, status);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int fs2_align_bin_loss(const float* logp, const int32_t* path, const int64_t* ilens, const int64_t* olens, int B, int L, int T,
                       const float* dloss, float* loss, float* dlogp, int* status, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(logp && path && ilens && olens && loss && status, "fs2_align_bin_loss: null argument");
  AlWs w;
  int rc = al_carve(B, L, T, ws, ws_bytes, &w, nullptr, "fs2_align_bin_loss");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  al_bin_loss_kernel<<<B, kLatThreads, 0, st>>>(logp, path, ilens, olens, L, T, dloss, loss, dlogp, w.lse, status);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int fs2_align_mask_rows(const float* x, const int64_t* lens, int B, int L, int C, float* y, void* stream) {
  FS2_REQUIRE(x && lens && y, "fs2_align_mask_rows: null argument");
  FS2_REQUIRE(B >= 1 && L >= 1 && C >= 1 && (double)B * L * C < 9e18, "fs2_align_mask_rows: bad shape [%d, %d, %d]", B, L, C);
  const long n = (long)B * L * C;
  al_mask_rows_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(x, lens, L, C, n, y);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // extern "C"
