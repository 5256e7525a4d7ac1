// Batched ECAPA-TDNN speaker encoder (DESIGN.md section 28): SpeechBrain's `spkrec-ecapa-voxceleb` front end and network on
// 16 kHz audio [B, Nmax] with sample counts lens [B] -> embeddings [B, D], each utterance over its own samples alone.
//
// Activations are rows [B * Tmax][C], utterance b at rows t < T_b = 1 + lens[b] / 160 (Tmax = 1 + Nmax / 160).  Every
// contraction except the per-utterance vectors is one tap-GEMM (vweight_gemm_args + tap_gemm) run with TapGemm::lens = T:
// row tiles wholly past an utterance are skipped and padded rows come out as exact zeros.  A producer writes each GEMM's A
// operand (fp32 rows, or hi / lo operand planes with their range check) and does what the GEMM does not:
//
//   taps        a convolution's k taps at dilation d side by side along K, reflected at the utterance's own edges, with the
//               BatchNorm affine of the rows it reads and the Res2Net sum x_i + y_(i-1)            block 0, Res2Net
//   rows        BatchNorm affine (per column, two sources split at a column), SE scale and residual     tdnn2, SE, MFA, ASP
//   att         tanh(BN(relu(W_h h + ctx_b)))                                                          ASP conv
//
// TDNNBlock is conv -> ReLU -> BatchNorm, so a GEMM writes relu(conv) and the BatchNorm affine is applied by whoever reads
// it.  The ASP's global context is folded: W [h; mu; sigma] = W_h h + (W_mu mu + W_sigma sigma + b), the second term a
// per-utterance vector ctx_b, so its GEMM has K = M and no [rows, 3M] tensor exists.
//
// The front end (Fbank + sentence mean norm) and every per-utterance reduction (SE means, ASP statistics, softmax over
// time, the small SE / context / fc matrix-vector products) run in fp32 on CUDA cores, each sum in an order that depends
// only on T_b (one thread per column walking t upwards, or one warp per output with a fixed butterfly), so an utterance's
// embedding does not depend on its batch mates.  No floating-point atomics.
#include <math.h>

#include <algorithm>
#include <vector>

#include "vocoder_weights.cuh"

namespace fs2 {
namespace {

constexpr int kFft = 400, kHop = 160, kBins = kFft / 2 + 1, kFpc = 16;   // frames per CTA of the DFT
constexpr float kTopDb = 80.f, kAmin = 1e-10f;
constexpr int kMatvecWarps = 8;

__device__ __forceinline__ int reflect(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return i;
}

// T[b] = frames of utterance b (samples: 1 + lens / 160; frames: lens itself), 0 when it lies outside [min_T, maxT]
// (FS2_ECAPA_BAD_LENGTH).  One block: it also writes the status word's first value.
__global__ void ecapa_prep_kernel(const int64_t* __restrict__ lens, int B, int samples, long maxv, int min_T, int64_t* __restrict__ T,
                                  int* __restrict__ status) {
  bool bad = false;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const int64_t n = lens[b];
    const int64_t t = samples ? 1 + n / kHop : n;
    const bool ok = n >= 0 && n <= maxv && t >= min_T;
    bad |= !ok;
    T[b] = ok ? t : 0;
  }
  bad = __syncthreads_or(bad);
  if (threadIdx.x == 0) *status = bad ? FS2_ECAPA_BAD_LENGTH : 0;
}

// log-mel power in dB of kFpc frames of utterance b (grid (ceil(Tmax / kFpc), B)): the hamming-windowed 400-point DFT of
// the centred, zero-padded frame (samples past lens[b] are never read), power, the filterbank, 10 log10(max(., 1e-10)).
// trig [400][2][201]: window * cos, -window * sin; fb [nm][201].
__global__ void __launch_bounds__(256) ecapa_fbank_kernel(const float* __restrict__ wav, const int64_t* __restrict__ lens,
                                                          const int64_t* __restrict__ T, int Nmax, int Tmax, const float* __restrict__ trig,
                                                          const float* __restrict__ fb, int nm, float* __restrict__ out) {
  __shared__ float xs[kFpc][kFft];
  __shared__ float ps[kFpc][kBins + 1];
  const int b = blockIdx.y, t0 = blockIdx.x * kFpc, Tb = (int)T[b];
  if (t0 >= Tb) return;
  const long N = lens[b];
  const int nf = min(kFpc, Tb - t0);
  for (int i = threadIdx.x; i < kFpc * kFft; i += blockDim.x) {
    const int f = i / kFft, n = i - f * kFft;
    const long s = (long)(t0 + f) * kHop - kFft / 2 + n;
    xs[f][n] = f < nf && s >= 0 && s < N ? wav[(long)b * Nmax + s] : 0.f;
  }
  __syncthreads();
  const int k = threadIdx.x;
  if (k < kBins) {
    float re[kFpc], im[kFpc];
#pragma unroll
    for (int f = 0; f < kFpc; ++f) re[f] = im[f] = 0.f;
#pragma unroll 2
    for (int n = 0; n < kFft; ++n) {
      const float c = __ldg(trig + n * 2 * kBins + k), s = __ldg(trig + n * 2 * kBins + kBins + k);
#pragma unroll
      for (int f = 0; f < kFpc; ++f) { re[f] = fmaf(xs[f][n], c, re[f]); im[f] = fmaf(xs[f][n], s, im[f]); }
    }
#pragma unroll
    for (int f = 0; f < kFpc; ++f) ps[f][k] = fmaf(re[f], re[f], im[f] * im[f]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nf * nm; i += blockDim.x) {
    const int f = i / nm, m = i - f * nm;
    float acc = 0.f;
    for (int q = 0; q < kBins; ++q) acc = fmaf(__ldg(fb + m * kBins + q), ps[f][q], acc);
    out[((long)b * Tmax + t0 + f) * nm + m] = 10.f * log10f(fmaxf(acc, kAmin));
  }
}

// in place on utterance b's rows [T_b][nm] (one block of 256 per utterance): clamp at (max - 80 dB), minus each band's
// mean over the T_b frames.  Band m's sum: G = 256 / nm partial sums over t = g, g + G, ..., then added in g order.
__global__ void __launch_bounds__(256) ecapa_fbank_norm_kernel(float* __restrict__ x, const int64_t* __restrict__ T, int Tmax, int nm) {
  __shared__ float red[256];
  const int b = blockIdx.x, Tb = (int)T[b];
  if (Tb == 0) return;
  float* xb = x + (long)b * Tmax * nm;
  const long n = (long)Tb * nm;
  float mx = -INFINITY;
  for (long i = threadIdx.x; i < n; i += blockDim.x) mx = fmaxf(mx, xb[i]);
  red[threadIdx.x] = mx;
  __syncthreads();
  for (int h = 128; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] = fmaxf(red[threadIdx.x], red[threadIdx.x + h]);
    __syncthreads();
  }
  const float floor_db = red[0] - kTopDb;
  __syncthreads();
  const int G = 256 / nm, g = threadIdx.x / nm, m = threadIdx.x - g * nm;
  if (g < G) {
    float s = 0.f;
    for (int t = g; t < Tb; t += G) s += fmaxf(xb[(long)t * nm + m], floor_db);
    red[threadIdx.x] = s;
  }
  __syncthreads();
  __shared__ float mean[256];
  if (threadIdx.x < nm) {
    float s = 0.f;
    for (int q = 0; q < G; ++q) s += red[q * nm + threadIdx.x];
    mean[threadIdx.x] = s / (float)Tb;
  }
  __syncthreads();
  for (long i = threadIdx.x; i < n; i += blockDim.x) {
    const int c = (int)(i % nm);
    xb[i] = fmaxf(xb[i], floor_db) - mean[c];
  }
}

__device__ __forceinline__ float4 affine4(float4 v, const float* __restrict__ s, const float* __restrict__ t, int c) {
  if (!s) return v;
  const float4 a = *reinterpret_cast<const float4*>(s + c), o = *reinterpret_cast<const float4*>(t + c);
  return make_float4(fmaf(v.x, a.x, o.x), fmaf(v.y, a.y, o.y), fmaf(v.z, a.z, o.z), fmaf(v.w, a.w, o.w));
}

// A [rows][taps * Cin]: tap j of row t = (x * xs + xt)[src] (+ (y * ys + yt)[src]), src = reflect(t + (j - taps / 2) d, T_b);
// x, y rows ldx / ldy floats apart (s / t nullable: no affine; y nullable: no second term).  Rows t >= T_b are not written.
template <int OUT>
__global__ void ecapa_taps_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ xs, const float* __restrict__ xt,
                                  const float* __restrict__ y, int ldy, const float* __restrict__ ys, const float* __restrict__ yt,
                                  const int64_t* __restrict__ T, int B, int L, int Cin, int taps, int d, float* __restrict__ out32,
                                  __half* __restrict__ outp, int* __restrict__ status) {
  const int K = taps * Cin, Q = K / 4;
  const long rows = (long)B * L, total = rows * Q, plane = rows * K;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / Q;
    const int k = (int)(i - row * Q) * 4, j = k / Cin, c = k - j * Cin;
    const int b = (int)(row / L), t = (int)(row - (long)b * L), Tb = (int)T[b];
    if (t >= Tb) continue;
    const long src = (long)b * L + reflect(t + (j - taps / 2) * d, Tb);
    float4 v = affine4(*reinterpret_cast<const float4*>(x + src * ldx + c), xs, xt, c);
    if (y) {
      const float4 w = affine4(*reinterpret_cast<const float4*>(y + src * ldy + c), ys, yt, c);
      v = make_float4(v.x + w.x, v.y + w.y, v.z + w.z, v.w + w.w);
    }
    store_quad<OUT, RANGE_ALWAYS>(v, row * K + k, out32, outp, plane, status, FS2_ECAPA_RANGE);
  }
}

// v = (src * s + t) * g[b] + res for rows t < T_b and C columns, src = x for columns < split, x2 beyond (both ldx apart);
// s / t, g [B][C], res (ldr apart), x2 nullable.  v goes to dst (ldd apart, nullable) and to the GEMM operand [rows][C]
// (a nullable: fp32 rows when OUT_F32, else planes with the range check).
template <int OUT>
__global__ void ecapa_rows_kernel(const float* __restrict__ x, const float* __restrict__ x2, int split, int ldx, const float* __restrict__ s,
                                  const float* __restrict__ t, const float* __restrict__ g, const float* __restrict__ res, int ldr,
                                  float* __restrict__ dst, int ldd, void* __restrict__ a, const int64_t* __restrict__ T, int B, int L, int C,
                                  int* __restrict__ status) {
  const int Q = C / 4;
  const long rows = (long)B * L, total = rows * Q, plane = rows * C;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / Q;
    const int c = (int)(i - row * Q) * 4;
    const int b = (int)(row / L), tt = (int)(row - (long)b * L);
    if (tt >= (int)T[b]) continue;
    const float* src = x2 && c >= split ? x2 : x;
    float4 v = affine4(*reinterpret_cast<const float4*>(src + row * ldx + c), s, t, c);
    if (g) {
      const float4 q = *reinterpret_cast<const float4*>(g + (long)b * C + c);
      v = make_float4(v.x * q.x, v.y * q.y, v.z * q.z, v.w * q.w);
    }
    if (res) {
      const float4 r = *reinterpret_cast<const float4*>(res + row * ldr + c);
      v = make_float4(v.x + r.x, v.y + r.y, v.z + r.z, v.w + r.w);
    }
    if (dst) *reinterpret_cast<float4*>(dst + row * ldd + c) = v;
    if (a) store_quad<OUT, RANGE_ALWAYS>(v, row * C + c, (float*)a, (__half*)a, plane, status, FS2_ECAPA_RANGE);
  }
}

// the ASP conv's operand [rows][Na]: tanh(relu(z + ctx[b]) * s + t), z = the tdnn GEMM's W_h h
template <int OUT>
__global__ void ecapa_att_kernel(const float* __restrict__ z, const float* __restrict__ ctx, const float* __restrict__ s, const float* __restrict__ t,
                                 const int64_t* __restrict__ T, int B, int L, int Na, float* __restrict__ out32, __half* __restrict__ outp,
                                 int* __restrict__ status) {
  const int Q = Na / 4;
  const long rows = (long)B * L, total = rows * Q, plane = rows * Na;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / Q;
    const int c = (int)(i - row * Q) * 4;
    const int b = (int)(row / L), tt = (int)(row - (long)b * L);
    if (tt >= (int)T[b]) continue;
    const float4 v = *reinterpret_cast<const float4*>(z + row * Na + c), q = *reinterpret_cast<const float4*>(ctx + (long)b * Na + c);
    const float4 r = affine4(make_float4(fmaxf(v.x + q.x, 0.f), fmaxf(v.y + q.y, 0.f), fmaxf(v.z + q.z, 0.f), fmaxf(v.w + q.w, 0.f)), s, t, c);
    store_quad<OUT, RANGE_ALWAYS>(make_float4(tanhf(r.x), tanhf(r.y), tanhf(r.z), tanhf(r.w)), row * Na + c, out32, outp, plane, status,
                                  FS2_ECAPA_RANGE);
  }
}

// out[b][c] = (1 / T_b) sum_{t < T_b} (x[b, t, c] * s[c] + t[c]), t ascending; grid (ceil(C / 128), B)
__global__ void ecapa_colmean_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ s, const float* __restrict__ sh,
                                     const int64_t* __restrict__ T, int L, int C, float* __restrict__ out) {
  const int b = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x, Tb = (int)T[b];
  if (c >= C) return;
  const float* xb = x + (long)b * L * ldx + c;
  float acc = 0.f;
  for (int t = 0; t < Tb; ++t) acc += s ? fmaf(xb[(long)t * ldx], s[c], sh[c]) : xb[(long)t * ldx];
  out[(long)b * C + c] = Tb ? acc / (float)Tb : 0.f;
}

// The ASP statistics of h [B * L][M] per (b, c), t ascending.  logits == nullptr: the global context with weights 1 / T_b;
// else the attention softmax over t < T_b of logits [B * L][M].  out[b] = [mu (M) | sqrt(max(var, 1e-12)) (M)].
__global__ void ecapa_stats_kernel(const float* __restrict__ h, const float* __restrict__ logits, const int64_t* __restrict__ T, int L, int M,
                                   float* __restrict__ out) {
  const int b = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x, Tb = (int)T[b];
  if (c >= M) return;
  const float* hb = h + (long)b * L * M + c;
  float* ob = out + (long)b * 2 * M;
  if (Tb == 0) { ob[c] = 0.f; ob[M + c] = 0.f; return; }
  float mu = 0.f, var = 0.f;
  if (!logits) {
    const float w = 1.f / (float)Tb;
    for (int t = 0; t < Tb; ++t) mu = fmaf(w, hb[(long)t * M], mu);
    for (int t = 0; t < Tb; ++t) { const float e = hb[(long)t * M] - mu; var = fmaf(w, e * e, var); }
  } else {
    const float* lb = logits + (long)b * L * M + c;
    float mx = -INFINITY, S = 0.f;
    for (int t = 0; t < Tb; ++t) mx = fmaxf(mx, lb[(long)t * M]);
    for (int t = 0; t < Tb; ++t) S += expf(lb[(long)t * M] - mx);
    for (int t = 0; t < Tb; ++t) mu = fmaf(expf(lb[(long)t * M] - mx) / S, hb[(long)t * M], mu);
    for (int t = 0; t < Tb; ++t) {
      const float e = hb[(long)t * M] - mu;
      var = fmaf(expf(lb[(long)t * M] - mx) / S, e * e, var);
    }
  }
  ob[c] = mu;
  ob[M + c] = sqrtf(fmaxf(var, 1e-12f));
}

// out[b][n] = act(sum_k W[n][k] (in[b][k] * s[k] + t[k]) + bias[n]) for n < N, 0 where T_b == 0; one warp per output,
// lane j summing k = j, j + 32, ... then the butterfly.  act: 0 none, 1 relu, 2 sigmoid.  grid (ceil(N / 8), B), dynamic
// shared memory K floats.
__global__ void __launch_bounds__(32 * kMatvecWarps) ecapa_matvec_kernel(const float* __restrict__ W, int ldw, int K, int N,
                                                                         const float* __restrict__ in, int ldin, const float* __restrict__ s,
                                                                         const float* __restrict__ sh, const float* __restrict__ bias, int act,
                                                                         const int64_t* __restrict__ T, float* __restrict__ out) {
  extern __shared__ float v[];
  const int b = blockIdx.y, lane = threadIdx.x & 31, n = blockIdx.x * kMatvecWarps + (threadIdx.x >> 5);
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float x = in[(long)b * ldin + k];
    v[k] = s ? fmaf(x, s[k], sh[k]) : x;
  }
  __syncthreads();
  if (n >= N) return;
  const float* w = W + (long)n * ldw;
  float acc = 0.f;
  for (int k = lane; k < K; k += 32) acc = fmaf(__ldg(w + k), v[k], acc);
  acc = warp_sum(acc) + bias[n];
  if (act == 1) acc = fmaxf(acc, 0.f);
  if (act == 2) acc = 1.f / (1.f + expf(-acc));
  if (lane == 0) out[(long)b * N + n] = T[b] ? acc : 0.f;
}

}  // namespace
}  // namespace fs2

struct fs2_ecapa_model {
  int device = 0, math_mode = 0;
  bool loaded = false;
  fs2_ecapa_config cfg;
  void* arena = nullptr; size_t arena_bytes = 0;
  float* trig = nullptr;       // [400][2][201]
  float* fb = nullptr;         // [n_mels][201]
  struct Bn { float* s = nullptr; float* t = nullptr; };
  fs2::VWeight b0; Bn b0n;
  struct Blk {
    fs2::VWeight t1, t2, r[FS2_ECAPA_MAX_SCALE];
    Bn t1n, t2n, rn[FS2_ECAPA_MAX_SCALE], t2in;   // t2in: the affine of tdnn2's input, [bn(tdnn1)[:C/s] | bn(r_1) | ... ]
    float *se1w = nullptr, *se1b = nullptr, *se2w = nullptr, *se2b = nullptr;
  } blk[FS2_ECAPA_MAX_BLOCKS];
  fs2::VWeight mfa; Bn mfan;
  fs2::VWeight atd; Bn atdn; float *atd_full = nullptr, *atd_b = nullptr;   // atd: W_h; atd_full: the whole [A][3M or M] weight
  fs2::VWeight aconv;
  Bn pooln; float *fc_w = nullptr, *fc_b = nullptr;
};

namespace fs2 {
namespace {

struct EcPlan {
  int64_t* T;        // [B] frames
  float* fbn;        // [rows][n_mels]
  void* a;           // GEMM operand, rows * Kmax
  float *x0, *xcat, *u, *r, *h, *z, *logits;
  float *sem, *sez, *seg, *gstat, *ctx, *pooled;
};

int k_max(const fs2_ecapa_config& c) {
  const int c8 = c.channels / c.scale;
  int k = std::max(c.kernel_sizes[0] * c.n_mels, c.n_blocks * c.channels);
  for (int i = 1; i <= c.n_blocks; ++i) k = std::max(k, c.kernel_sizes[i] * c8);
  return std::max(std::max(k, c.mfa_channels), c.attention_channels);
}

EcPlan plan_of(Bump& b, const fs2_ecapa_model* m, int B, int L) {
  const fs2_ecapa_config& c = m->cfg;
  const size_t rows = (size_t)B * L;
  const int M = c.mfa_channels;
  EcPlan p;
  p.T = (int64_t*)b.bytes(B * sizeof(int64_t));
  p.fbn = b.floats(rows * c.n_mels);
  p.a = b.floats(rows * k_max(c));
  p.x0 = b.floats(rows * c.channels);
  p.xcat = b.floats(rows * c.n_blocks * c.channels);
  p.u = b.floats(rows * c.channels);
  p.r = b.floats(rows * c.channels);
  p.h = b.floats(rows * M);
  p.z = b.floats(rows * c.attention_channels);
  p.logits = b.floats(rows * M);
  p.sem = b.floats((size_t)B * c.channels);
  p.sez = b.floats((size_t)B * c.se_channels);
  p.seg = b.floats((size_t)B * c.channels);
  p.gstat = b.floats((size_t)B * 2 * M);
  p.ctx = b.floats((size_t)B * c.attention_channels);
  p.pooled = b.floats((size_t)B * 2 * M);
  return p;
}

struct Run {
  const fs2_ecapa_model* m;
  const EcPlan& p;
  int B, L, mode, kind;
  int* status;
  cudaStream_t st;

  bool planes() const { return plane_mode(mode); }

  // out [rows][ldo] = act(a . w^T + bias) on the rows t < T_b; a: operand planes [rows][w.K] or fp32 rows ldx apart
  int gemm(const VWeight& w, const void* a, int ldx, int act, float* out, int ldo) const {
    TapGemm g = vweight_gemm_args(mode, w, a, B, L, act, p.T, out);
    if (!planes()) g.ldx = ldx;
    g.ldo = ldo;
    return tap_gemm(g, mode, st);
  }
  int taps(const float* x, int ldx, const fs2_ecapa_model::Bn* xn, int xoff, const float* y, const fs2_ecapa_model::Bn* yn, int yoff, int ldy, int Cin,
           int k, int d) const {
    auto kern = pick(kind, ecapa_taps_kernel<OUT_HILO>, ecapa_taps_kernel<OUT_HI>, ecapa_taps_kernel<OUT_F32>);
    kern<<<grid_for((long)B * L * (k * Cin / 4), 256), 256, 0, st>>>(
        x, ldx, xn ? xn->s + xoff : nullptr, xn ? xn->t + xoff : nullptr, y, ldy, yn ? yn->s + yoff : nullptr, yn ? yn->t + yoff : nullptr,
        p.T, B, L, Cin, k, d, (float*)p.a, (__half*)p.a, status);
    FS2_LAUNCH_CHECK();
    return FS2_OK;
  }
  int rows(const float* x, const float* x2, int split, int ldx, const fs2_ecapa_model::Bn* n, const float* g, const float* res, int ldr, float* dst,
           int ldd, bool operand, int C) const {
    auto kern = pick(kind, ecapa_rows_kernel<OUT_HILO>, ecapa_rows_kernel<OUT_HI>, ecapa_rows_kernel<OUT_F32>);
    kern<<<grid_for((long)B * L * (C / 4), 256), 256, 0, st>>>(x, x2, split, ldx, n ? n->s : nullptr, n ? n->t : nullptr, g, res, ldr, dst, ldd,
                                                              operand ? p.a : nullptr, p.T, B, L, C, status);
    FS2_LAUNCH_CHECK();
    return FS2_OK;
  }
  int matvec(const float* W, int ldw, int K, int N, const float* in, int ldin, const fs2_ecapa_model::Bn* n, const float* bias, int act,
             float* out) const {
    ecapa_matvec_kernel<<<dim3((N + kMatvecWarps - 1) / kMatvecWarps, B), 32 * kMatvecWarps, (size_t)std::max(K, 1) * sizeof(float), st>>>(
        W, ldw, K, N, in, ldin, n ? n->s : nullptr, n ? n->t : nullptr, bias, act, p.T, out);
    FS2_LAUNCH_CHECK();
    return FS2_OK;
  }

  // audio -> p.fbn (normalised features), p.T already set
  int front_end(const float* wav, const int64_t* lens, int Nmax) const {
    const fs2_ecapa_config& c = m->cfg;
    ecapa_fbank_kernel<<<dim3((L + kFpc - 1) / kFpc, B), 256, 0, st>>>(wav, lens, p.T, Nmax, L, m->trig, m->fb, c.n_mels, p.fbn);
    FS2_LAUNCH_CHECK();
    ecapa_fbank_norm_kernel<<<B, 256, 0, st>>>(p.fbn, p.T, L, c.n_mels);
    FS2_LAUNCH_CHECK();
    return FS2_OK;
  }
  // p.fbn -> p.x0 = bn(relu(conv(fbn))) (and, in the plane modes, its planes in p.a)
  int block0() const {
    const fs2_ecapa_config& c = m->cfg;
    int rc = taps(p.fbn, c.n_mels, nullptr, 0, nullptr, nullptr, 0, 0, c.n_mels, c.kernel_sizes[0], c.dilations[0]);
    if (rc || (rc = gemm(m->b0, p.a, m->b0.K, ACT_RELU, p.u, c.channels))) return rc;
    return rows(p.u, nullptr, 0, c.channels, &m->b0n, nullptr, nullptr, 0, p.x0, c.channels, planes(), c.channels);
  }
  // SE-Res2Net block i (1-based) on xin (fp32 rows ldin apart; in the plane modes its planes are in p.a) -> xcat slice i - 1
  // (and its planes in p.a)
  int block(int i, const float* xin, int ldin) const {
    const fs2_ecapa_config& c = m->cfg;
    const fs2_ecapa_model::Blk& k = m->blk[i - 1];
    const int C = c.channels, c8 = C / c.scale, ldc = c.n_blocks * C;
    int rc = gemm(k.t1, planes() ? p.a : (const void*)xin, ldin, ACT_RELU, p.u, C);
    for (int j = 1; !rc && j < c.scale; ++j) {
      rc = taps(p.u + j * c8, C, &k.t1n, j * c8, j >= 2 ? p.r + (j - 1) * c8 : nullptr, &k.rn[j - 1], 0, C, c8, c.kernel_sizes[i], c.dilations[i]);
      if (!rc) rc = gemm(k.r[j], p.a, k.r[j].K, ACT_RELU, p.r + j * c8, C);
    }
    if (rc || (rc = rows(p.u, p.r, c8, C, &k.t2in, nullptr, nullptr, 0, nullptr, 0, true, C))) return rc;
    if ((rc = gemm(k.t2, p.a, C, ACT_RELU, p.u, C))) return rc;
    // SE: v = bn(u); g = sigmoid(W2 relu(W1 mean_t(v) + b1) + b2); out = v * g + xin
    ecapa_colmean_kernel<<<dim3((C + 127) / 128, B), 128, 0, st>>>(p.u, C, k.t2n.s, k.t2n.t, p.T, L, C, p.sem);
    FS2_LAUNCH_CHECK();
    if ((rc = matvec(k.se1w, C, C, c.se_channels, p.sem, C, nullptr, k.se1b, 1, p.sez))) return rc;
    if ((rc = matvec(k.se2w, c.se_channels, c.se_channels, C, p.sez, c.se_channels, nullptr, k.se2b, 2, p.seg))) return rc;
    return rows(p.u, nullptr, 0, C, &k.t2n, p.seg, xin, ldin, p.xcat + (i - 1) * C, ldc, planes(), C);
  }
  // p.xcat -> p.h = bn(relu(mfa(xcat))) (and its planes in p.a)
  int mfa() const {
    const fs2_ecapa_config& c = m->cfg;
    const int ldc = c.n_blocks * c.channels, M = c.mfa_channels;
    int rc = FS2_OK;
    if (planes()) rc = rows(p.xcat, nullptr, 0, ldc, nullptr, nullptr, nullptr, 0, nullptr, 0, true, ldc);
    if (rc || (rc = gemm(m->mfa, planes() ? p.a : (const void*)p.xcat, ldc, ACT_RELU, p.h, M))) return rc;
    return rows(p.h, nullptr, 0, M, &m->mfan, nullptr, nullptr, 0, p.h, M, planes(), M);
  }
  // p.h (and its planes in p.a) -> p.pooled [B][2M]
  int asp() const {
    const fs2_ecapa_config& c = m->cfg;
    const int M = c.mfa_channels, A = c.attention_channels;
    int rc = FS2_OK;
    if (c.global_context) {
      ecapa_stats_kernel<<<dim3((M + 127) / 128, B), 128, 0, st>>>(p.h, nullptr, p.T, L, M, p.gstat);
      FS2_LAUNCH_CHECK();
    }
    const int ldw = c.global_context ? 3 * M : M;
    if ((rc = matvec(m->atd_full + M, ldw, c.global_context ? 2 * M : 0, A, p.gstat, 2 * M, nullptr, m->atd_b, 0, p.ctx))) return rc;
    if ((rc = gemm(m->atd, planes() ? p.a : (const void*)p.h, M, ACT_NONE, p.z, A))) return rc;
    auto kern = pick(kind, ecapa_att_kernel<OUT_HILO>, ecapa_att_kernel<OUT_HI>, ecapa_att_kernel<OUT_F32>);
    kern<<<grid_for((long)B * L * (A / 4), 256), 256, 0, st>>>(p.z, p.ctx, m->atdn.s, m->atdn.t, p.T, B, L, A, (float*)p.a, (__half*)p.a, status);
    FS2_LAUNCH_CHECK();
    if ((rc = gemm(m->aconv, p.a, A, ACT_NONE, p.logits, M))) return rc;
    ecapa_stats_kernel<<<dim3((M + 127) / 128, B), 128, 0, st>>>(p.h, p.logits, p.T, L, M, p.pooled);
    FS2_LAUNCH_CHECK();
    return FS2_OK;
  }
  int fc(float* emb) const {
    const fs2_ecapa_config& c = m->cfg;
    return matvec(m->fc_w, 2 * c.mfa_channels, 2 * c.mfa_channels, c.lin_neurons, p.pooled, 2 * c.mfa_channels, &m->pooln, m->fc_b, 0, emb);
  }
  int blocks() const {
    const fs2_ecapa_config& c = m->cfg;
    int rc = FS2_OK;
    for (int i = 1; !rc && i <= c.n_blocks; ++i)
      rc = i == 1 ? block(1, p.x0, c.channels) : block(i, p.xcat + (i - 2) * c.channels, c.n_blocks * c.channels);
    return rc;
  }
};

// frames the reflect padding needs: every "same" convolution pads d (k - 1) / 2 rows, and one reflection must reach them
int min_frames(const fs2_ecapa_config& c) {
  int pad = 0;
  for (int i = 0; i <= c.n_blocks; ++i) pad = std::max(pad, c.dilations[i] * (c.kernel_sizes[i] - 1) / 2);
  return pad + 1;
}

int check_config(const fs2_ecapa_config& c) {
  const char* who = "fs2_ecapa_create";
  FS2_REQUIRE(c.n_blocks >= 1 && c.n_blocks <= FS2_ECAPA_MAX_BLOCKS, "%s: n_blocks must lie in [1, %d] (got %d)", who, FS2_ECAPA_MAX_BLOCKS,
              c.n_blocks);
  FS2_REQUIRE(c.scale >= 2 && c.scale <= FS2_ECAPA_MAX_SCALE, "%s: res2net scale must lie in [2, %d] (got %d)", who, FS2_ECAPA_MAX_SCALE,
              c.scale);
  FS2_REQUIRE(c.channels >= 16 * c.scale && c.channels % (16 * c.scale) == 0 && c.channels <= 8192,
              "%s: channels (%d) must be a multiple of 16 * scale = %d, at most 8192", who, c.channels, 16 * c.scale);
  FS2_REQUIRE(c.n_mels >= 16 && c.n_mels % 16 == 0 && c.n_mels <= 256, "%s: n_mels (%d) must be a multiple of 16 in [16, 256]", who, c.n_mels);
  FS2_REQUIRE(c.mfa_channels >= 16 && c.mfa_channels % 16 == 0 && c.mfa_channels <= 8192, "%s: the MFA width (%d) must be a multiple of 16",
              who, c.mfa_channels);
  FS2_REQUIRE(c.attention_channels >= 16 && c.attention_channels % 16 == 0 && c.attention_channels <= 4096,
              "%s: attention_channels (%d) must be a multiple of 16", who, c.attention_channels);
  FS2_REQUIRE(c.se_channels >= 1 && c.se_channels <= 8192 && c.lin_neurons >= 1 && c.lin_neurons <= 8192,
              "%s: bad se_channels %d / lin_neurons %d", who, c.se_channels, c.lin_neurons);
  for (int i = 0; i <= c.n_blocks; ++i)
    FS2_REQUIRE(c.kernel_sizes[i] >= 1 && c.kernel_sizes[i] % 2 == 1 && c.kernel_sizes[i] <= 31 && c.dilations[i] >= 1 && c.dilations[i] <= 64,
                "%s: block %d: kernel size %d must be odd in [1, 31], dilation %d in [1, 64]", who, i, c.kernel_sizes[i], c.dilations[i]);
  FS2_REQUIRE(c.kernel_sizes[c.n_blocks + 1] == 1, "%s: the MFA kernel size must be 1 (got %d)", who, c.kernel_sizes[c.n_blocks + 1]);
  FS2_REQUIRE(2 * c.mfa_channels <= 12288 && c.channels <= 12288, "%s: widths exceed the matrix-vector kernel's shared memory", who);
  return FS2_OK;
}

// rows of a call over B utterances of Tmax frames: int32 row indices, fp32 mode's limit, and every operand's elements
int check_size(const fs2_ecapa_model* m, int B, long Tmax, const char* who) {
  FS2_REQUIRE(B >= 1 && Tmax >= 1, "%s: bad shape B=%d Tmax=%ld", who, B, Tmax);
  const long rows = (long)B * Tmax;
  int rc = check_rows(who, "B * Tmax", "frame", rows, m->math_mode);
  if (rc) return rc;
  const long widest = std::max<long>(k_max(m->cfg), (long)m->cfg.n_blocks * m->cfg.channels);
  FS2_REQUIRE(rows * widest < (1L << 31), "%s: B * Tmax * %ld = %ld operand elements reach 2^31", who, widest, rows * widest);
  return FS2_OK;
}

}  // namespace
}  // namespace fs2

using namespace fs2;

extern "C" {

int fs2_ecapa_create(fs2_ecapa_model** out, int math_mode, const fs2_ecapa_config* cfg) {
  FS2_REQUIRE(out && cfg, "fs2_ecapa_create: null argument");
  FS2_REQUIRE(math_mode >= FS2_MATH_FP32 && math_mode <= FS2_MATH_F16, "fs2_ecapa_create: bad math_mode %d", math_mode);
  int rc = check_config(*cfg);
  if (rc) return rc;
  fs2_ecapa_model* m = new fs2_ecapa_model();
  m->math_mode = math_mode;
  m->cfg = *cfg;
  cudaError_t e = cudaGetDevice(&m->device);
  if (e != cudaSuccess) { delete m; FS2_CUDA_CHECK(e); }
  *out = m;
  return FS2_OK;
}

void fs2_ecapa_destroy(fs2_ecapa_model* m) {
  if (!m) return;
  if (m->arena) cudaFree(m->arena);
  delete m;
}

int fs2_ecapa_n_tensors(const fs2_ecapa_config* c) {
  return c ? 4 + c->n_blocks * (4 + 4 * (c->scale - 1) + 4 + 4) + 4 + 4 + 2 + 2 + 2 : 0;
}

int fs2_ecapa_load(fs2_ecapa_model* m, const float* const* t, int n, void* stream) {
  FS2_REQUIRE(m && t, "fs2_ecapa_load: null argument");
  const fs2_ecapa_config& c = m->cfg;
  FS2_REQUIRE(n == fs2_ecapa_n_tensors(&c), "fs2_ecapa_load: %d tensors, the configuration takes %d", n, fs2_ecapa_n_tensors(&c));
  for (int i = 0; i < n; ++i) FS2_REQUIRE(t[i], "fs2_ecapa_load: tensor %d is null", i);
  cudaStream_t st = (cudaStream_t)stream;
  const int C = c.channels, c8 = C / c.scale, M = c.mfa_channels, A = c.attention_channels, se = c.se_channels, nm = c.n_mels;
  const int ctxK = c.global_context ? 3 * M : M;
  m->b0.N = C; m->b0.K = c.kernel_sizes[0] * nm;
  for (int i = 0; i < c.n_blocks; ++i) {
    fs2_ecapa_model::Blk& k = m->blk[i];
    k.t1.N = k.t1.K = k.t2.N = k.t2.K = C;
    for (int j = 1; j < c.scale; ++j) { k.r[j].N = c8; k.r[j].K = c.kernel_sizes[i + 1] * c8; }
  }
  m->mfa.N = M; m->mfa.K = c.n_blocks * C;
  m->atd.N = A; m->atd.K = M;
  m->aconv.N = M; m->aconv.K = A;
  m->loaded = false;
  auto bn = [](Bump& b, fs2_ecapa_model::Bn& x, int N) { x.s = b.floats(N); x.t = b.floats(N); };
  int rc = arena_carve(&m->arena, &m->arena_bytes, st, [&](Bump& b) {
    m->trig = b.floats(2 * kFft * kBins);
    m->fb = b.floats((size_t)nm * kBins);
    vweight_carve(b, m->b0, true); bn(b, m->b0n, C);
    for (int i = 0; i < c.n_blocks; ++i) {
      fs2_ecapa_model::Blk& k = m->blk[i];
      vweight_carve(b, k.t1, true); bn(b, k.t1n, C);
      for (int j = 1; j < c.scale; ++j) { vweight_carve(b, k.r[j], true); bn(b, k.rn[j], c8); }
      vweight_carve(b, k.t2, true); bn(b, k.t2n, C); bn(b, k.t2in, C);
      k.se1w = b.floats((size_t)se * C); k.se1b = b.floats(se); k.se2w = b.floats((size_t)C * se); k.se2b = b.floats(C);
    }
    vweight_carve(b, m->mfa, true); bn(b, m->mfan, M);
    vweight_carve(b, m->atd, false); bn(b, m->atdn, A); m->atd_full = b.floats((size_t)A * ctxK); m->atd_b = b.floats(A);
    vweight_carve(b, m->aconv, true);
    bn(b, m->pooln, 2 * M); m->fc_w = b.floats((size_t)c.lin_neurons * 2 * M); m->fc_b = b.floats(c.lin_neurons);
    return FS2_OK;
  });
  if (rc) return rc;
  // the front end's tables, in double on the host: periodic hamming window times the DFT's cos / -sin, and SpeechBrain's
  // triangular filterbank (DESIGN.md section 28)
  std::vector<float> trig(2 * kFft * kBins), fb((size_t)nm * kBins);
  for (int n = 0; n < kFft; ++n) {
    const double w = 0.54 - 0.46 * cos(2.0 * M_PI * n / kFft);
    for (int k = 0; k < kBins; ++k) {
      const double ph = 2.0 * M_PI * (double)((long)k * n % kFft) / kFft;
      trig[n * 2 * kBins + k] = (float)(w * cos(ph));
      trig[n * 2 * kBins + kBins + k] = (float)(-w * sin(ph));
    }
  }
  {
    auto mel = [](double f) { return 2595.0 * log10(1.0 + f / 700.0); };
    const double top = mel(8000.0);
    std::vector<double> hz(nm + 2);
    for (int i = 0; i < nm + 2; ++i) hz[i] = 700.0 * (pow(10.0, (top * i / (nm + 1)) / 2595.0) - 1.0);
    for (int mm = 0; mm < nm; ++mm) {
      const double fc = hz[mm + 1], band = hz[mm + 1] - hz[mm];
      for (int k = 0; k < kBins; ++k) {
        const double sl = (8000.0 * k / (kBins - 1) - fc) / band;
        fb[(size_t)mm * kBins + k] = (float)std::max(0.0, std::min(sl + 1.0, 1.0 - sl));
      }
    }
  }
  FS2_CUDA_CHECK(cudaMemcpyAsync(m->trig, trig.data(), trig.size() * sizeof(float), cudaMemcpyHostToDevice, st));
  FS2_CUDA_CHECK(cudaMemcpyAsync(m->fb, fb.data(), fb.size() * sizeof(float), cudaMemcpyHostToDevice, st));
  // host buffers must outlive the copies
  FS2_CUDA_CHECK(cudaStreamSynchronize(st));
  int q = 0;
  auto copy = [&](float* dst, size_t nfl) { return cudaMemcpyAsync(dst, t[q++], nfl * sizeof(float), cudaMemcpyDeviceToDevice, st); };
  auto conv = [&](const VWeight& w, int Cin, int Cout, int taps) {
    const int r = vweight_pack_conv(w, t[q], t[q + 1], Cin, Cout, taps, 0, Cin, st);
    q += 2;
    return r;
  };
  auto bnc = [&](fs2_ecapa_model::Bn& x, int N) {
    if (copy(x.s, N) != cudaSuccess || copy(x.t, N) != cudaSuccess) return (int)FS2_ERR_CUDA;
    return (int)FS2_OK;
  };
  if ((rc = conv(m->b0, nm, C, c.kernel_sizes[0])) || (rc = bnc(m->b0n, C))) return rc;
  for (int i = 0; i < c.n_blocks; ++i) {
    fs2_ecapa_model::Blk& k = m->blk[i];
    if ((rc = conv(k.t1, C, C, 1)) || (rc = bnc(k.t1n, C))) return rc;
    FS2_CUDA_CHECK(cudaMemcpyAsync(k.t2in.s, k.t1n.s, c8 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    FS2_CUDA_CHECK(cudaMemcpyAsync(k.t2in.t, k.t1n.t, c8 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    for (int j = 1; j < c.scale; ++j) {
      if ((rc = conv(k.r[j], c8, c8, c.kernel_sizes[i + 1])) || (rc = bnc(k.rn[j], c8))) return rc;
      FS2_CUDA_CHECK(cudaMemcpyAsync(k.t2in.s + j * c8, k.rn[j].s, c8 * sizeof(float), cudaMemcpyDeviceToDevice, st));
      FS2_CUDA_CHECK(cudaMemcpyAsync(k.t2in.t + j * c8, k.rn[j].t, c8 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    if ((rc = conv(k.t2, C, C, 1)) || (rc = bnc(k.t2n, C))) return rc;
    FS2_CUDA_CHECK(copy(k.se1w, (size_t)se * C)); FS2_CUDA_CHECK(copy(k.se1b, se));
    FS2_CUDA_CHECK(copy(k.se2w, (size_t)C * se)); FS2_CUDA_CHECK(copy(k.se2b, C));
  }
  if ((rc = conv(m->mfa, c.n_blocks * C, M, 1)) || (rc = bnc(m->mfan, M))) return rc;
  if ((rc = vweight_pack(m->atd, t[q], A, ctxK, 0, st))) return rc;   // W_h: the first M of the ctxK columns
  FS2_CUDA_CHECK(copy(m->atd_full, (size_t)A * ctxK)); FS2_CUDA_CHECK(copy(m->atd_b, A));
  if ((rc = bnc(m->atdn, A))) return rc;
  if ((rc = conv(m->aconv, A, M, 1))) return rc;
  if ((rc = bnc(m->pooln, 2 * M))) return rc;
  FS2_CUDA_CHECK(copy(m->fc_w, (size_t)c.lin_neurons * 2 * M)); FS2_CUDA_CHECK(copy(m->fc_b, c.lin_neurons));
  m->loaded = true;
  return FS2_OK;
}

int fs2_ecapa_workspace_bytes(fs2_ecapa_model* m, int B, int Nmax, size_t* bytes) {
  FS2_REQUIRE(m && bytes, "fs2_ecapa_workspace_bytes: null argument");
  FS2_REQUIRE(Nmax >= 1, "fs2_ecapa_workspace_bytes: bad Nmax %d", Nmax);
  const int L = 1 + Nmax / kHop;
  int rc = check_size(m, B, L, "fs2_ecapa");
  if (rc) return rc;
  Bump b(nullptr, 0);
  plan_of(b, m, B, L);
  *bytes = b.off + 256;
  return FS2_OK;
}

int fs2_ecapa(fs2_ecapa_model* m, const float* wavs, const int64_t* lens, int B, int Nmax, float* emb, int* status, void* ws, size_t ws_bytes,
              void* stream) {
  const char* who = "fs2_ecapa";
  FS2_REQUIRE(m && wavs && lens && emb && status && ws, "%s: null argument", who);
  FS2_REQUIRE(m->loaded, "%s: weights not loaded (fs2_ecapa_load)", who);
  FS2_REQUIRE(Nmax >= 1, "%s: bad Nmax %d", who, Nmax);
  const int L = 1 + Nmax / kHop;
  int rc = check_size(m, B, L, who);
  if (rc) return rc;
  Bump b(ws, ws_bytes);
  const EcPlan p = plan_of(b, m, B, L);
  if ((rc = b.check(who))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const Run run{m, p, B, L, m->math_mode, out_kind(m->math_mode), status, st};
  ecapa_prep_kernel<<<1, 256, 0, st>>>(lens, B, 1, Nmax, min_frames(m->cfg), p.T, status);
  FS2_LAUNCH_CHECK();
  if ((rc = run.front_end(wavs, lens, Nmax)) || (rc = run.block0()) || (rc = run.blocks()) || (rc = run.mfa()) || (rc = run.asp())) return rc;
  return run.fc(emb);
}

// One stage of fs2_ecapa on rows [B * L][Cin] with frame counts lens (test entry; the samples of stage 0).  Stages and
// their input -> output:
//   0  audio [B][L] (lens in samples)          -> normalised features [B][1 + L / 160][n_mels]
//   1  features [B * L][n_mels]                -> block 0's output [B * L][C]
//   1 + i (i = 1 .. n_blocks)  [B * L][C]      -> SE-Res2Net block i's output [B * L][C]
//   n_blocks + 2  [B * L][n_blocks * C]        -> the MFA's output [B * L][M]
//   n_blocks + 3  [B * L][M]                   -> the ASP's pooled statistics [B][2M]
// Every lens[b] (frames) must lie in [min_frames, L] (FS2_ECAPA_BAD_LENGTH in *status otherwise); rows past lens[b] of
// the input are never read; output rows past it are unspecified.  The workspace is fs2_ecapa_workspace_bytes(m, B, (L - 1) * 160).
int fs2_op_ecapa_stage(fs2_ecapa_model* m, int stage, const float* in, const int64_t* lens, int B, int L, float* out, int* status, void* ws,
                       size_t ws_bytes, void* stream) {
  const char* who = "fs2_op_ecapa_stage";
  FS2_REQUIRE(m && in && lens && out && status && ws, "%s: null argument", who);
  FS2_REQUIRE(m->loaded, "%s: weights not loaded (fs2_ecapa_load)", who);
  const fs2_ecapa_config& c = m->cfg;
  FS2_REQUIRE(stage >= 0 && stage <= c.n_blocks + 3, "%s: stage %d outside [0, %d]", who, stage, c.n_blocks + 3);
  FS2_REQUIRE(L >= 1, "%s: bad L %d", who, L);
  const int Lf = stage == 0 ? 1 + L / kHop : L;
  int rc = check_size(m, B, Lf, who);
  if (rc) return rc;
  Bump b(ws, ws_bytes);
  const EcPlan p = plan_of(b, m, B, Lf);
  if ((rc = b.check(who))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const Run run{m, p, B, Lf, m->math_mode, out_kind(m->math_mode), status, st};
  ecapa_prep_kernel<<<1, 256, 0, st>>>(lens, B, stage == 0, stage == 0 ? L : Lf, min_frames(c), p.T, status);
  FS2_LAUNCH_CHECK();
  const size_t rows = (size_t)B * Lf, f = sizeof(float);
  const int C = c.channels, M = c.mfa_channels;
  auto load = [&](float* dst, int width) { return cudaMemcpyAsync(dst, in, rows * width * f, cudaMemcpyDeviceToDevice, st); };
  if (stage == 0) {
    if ((rc = run.front_end(in, lens, L))) return rc;
    FS2_CUDA_CHECK(cudaMemcpyAsync(out, p.fbn, rows * c.n_mels * f, cudaMemcpyDeviceToDevice, st));
  } else if (stage == 1) {
    FS2_CUDA_CHECK(load(p.fbn, c.n_mels));
    if ((rc = run.block0())) return rc;
    FS2_CUDA_CHECK(cudaMemcpyAsync(out, p.x0, rows * C * f, cudaMemcpyDeviceToDevice, st));
  } else if (stage <= c.n_blocks + 1) {
    FS2_CUDA_CHECK(load(p.x0, C));
    if (run.planes() && (rc = run.rows(p.x0, nullptr, 0, C, nullptr, nullptr, nullptr, 0, nullptr, 0, true, C))) return rc;
    if ((rc = run.block(stage - 1, p.x0, C))) return rc;
    FS2_CUDA_CHECK(cudaMemcpy2DAsync(out, C * f, p.xcat + (stage - 2) * C, (size_t)c.n_blocks * C * f, C * f, rows, cudaMemcpyDeviceToDevice, st));
  } else if (stage == c.n_blocks + 2) {
    FS2_CUDA_CHECK(load(p.xcat, c.n_blocks * C));
    if ((rc = run.mfa())) return rc;
    FS2_CUDA_CHECK(cudaMemcpyAsync(out, p.h, rows * M * f, cudaMemcpyDeviceToDevice, st));
  } else {
    FS2_CUDA_CHECK(load(p.h, M));
    if (run.planes() && (rc = run.rows(p.h, nullptr, 0, M, nullptr, nullptr, nullptr, 0, nullptr, 0, true, M))) return rc;
    if ((rc = run.asp())) return rc;
    FS2_CUDA_CHECK(cudaMemcpyAsync(out, p.pooled, (size_t)B * 2 * M * f, cudaMemcpyDeviceToDevice, st));
  }
  return FS2_OK;
}

}  // extern "C"
