// Train-mode kernels (SURVEY.md section 8f-1): what `model.train(); loss, _ = model(...); loss.backward()` of
// train_fastspeech.py:100-123 needs beyond the eval path -- dropout, BatchNorm batch statistics, and the backward of every
// stage.  fp32 on CUDA cores, correctness first (the reference's training arithmetic is fp32): simple tiled kernels, each
// citing the reference op whose autograd formula it implements.  The Python side (fastspeech2_b200/train.py) chains them
// with torch.autograd.Function objects -- autograd is used for graph plumbing only, every number is produced here.
#include "vocoder_weights.cuh"

namespace fs2 {
namespace {

// ---- dropout (torch.nn.Dropout in train mode: keep with prob 1-p, scale by 1/(1-p)) ---------------------------------------
// Philox4x32-10 (common.cuh): mask byte i depends only on (seed, i), so the same mask is reproduced in backward without
// storing random state; tests inject masks instead (shared with the reference run).
__global__ void dropout_mask_kernel(uint8_t* __restrict__ mask, long n, float p, unsigned long long seed, unsigned long long offset) {
  const long quads = (n + 3) / 4;
  for (long q = (long)blockIdx.x * blockDim.x + threadIdx.x; q < quads; q += (long)gridDim.x * blockDim.x) {
    const unsigned long long c = offset + (unsigned long long)q;
    const uint4 r = philox4x32(make_uint4((unsigned)c, (unsigned)(c >> 32), 0u, 0u), make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
    const unsigned v[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (q * 4 + i < n) mask[q * 4 + i] = ((v[i] >> 8) * (1.0f / 16777216.0f)) >= p ? 1 : 0;
  }
}
// out = x * mask * scale (forward and backward are the same map)
__global__ void dropout_apply_kernel(const float* __restrict__ x, const uint8_t* __restrict__ mask, float scale, float* __restrict__ out, long n) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) out[i] = mask[i] ? x[i] * scale : 0.f;
}

// ---- activations' backward: dx = dy * f'(y) with the saved OUTPUT y (relu: y > 0; tanh: 1 - y^2) ---------------------------
__global__ void act_backward_kernel(const float* __restrict__ dy, const float* __restrict__ y, int act, float* __restrict__ dx, long n) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const float g = dy[i], v = y[i];
    dx[i] = act == ACT_RELU ? (v > 0.f ? g : 0.f) : act == ACT_TANH ? g * (1.f - v * v) : g;
  }
}
__global__ void relu_forward_kernel(const float* __restrict__ x, float* __restrict__ y, long n) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) y[i] = fmaxf(x[i], 0.f);
}
// y = a + b (residual add where no producing kernel can absorb it)
__global__ void add_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ y, long n) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) y[i] = a[i] + b[i];
}

// ---- column sums: out[c] (+)= sum_r x[r, c]  (bias gradients) ----------------------------------------------------------------
__global__ void colsum_kernel(const float* __restrict__ x, long rows, int C, float* __restrict__ out) {
  // block = 256 threads = 32 columns x 8 row-lanes; grid (C/32 ceil, row chunks)
  __shared__ float red[8][33];
  const int c = blockIdx.x * 32 + (threadIdx.x & 31), rl = threadIdx.x >> 5;
  float s = 0.f;
  if (c < C)
    for (long r = (long)blockIdx.y * 8 + rl; r < rows; r += (long)gridDim.y * 8) s += x[r * C + c];
  red[rl][threadIdx.x & 31] = s;
  __syncthreads();
  if (rl == 0 && c < C) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][threadIdx.x & 31];
    atomicAdd(out + c, t);
  }
}

// ---- Conv1d / Linear weight gradient ----------------------------------------------------------------------------------------
// dW[n][k][j] += sum_{b,t} dy[b,t,n] * x[b, t + j - pad, k]   (x zero outside [0,L)); output in the REFERENCE's layout
// [N][K][taps] (nn.Conv1d weight; taps == 1 is nn.Linear's [N][K]).  64 x 64 output tile per CTA, the reduction over the
// B*L rows is split over gridDim.z chunks and combined with atomicAdd (the gradient buffer is zero-initialised by autograd).
constexpr int WG_T = 64, WG_KM = 16;
__global__ void __launch_bounds__(256)
wgrad_kernel(const float* __restrict__ dy, int ldy, const float* __restrict__ x, int ldx, int B, int L, int N, int K, int taps,
             int chunks, float* __restrict__ dw) {
  __shared__ float sa[WG_KM][WG_T + 1];   // dy tile  [m][n]
  __shared__ float sb[WG_KM][WG_T + 1];   // x tile   [m][k]
  const int n0 = blockIdx.x * WG_T, k0 = blockIdx.y * WG_T;
  const int j = blockIdx.z / chunks, chunk = blockIdx.z - j * chunks;
  const int pad = (taps - 1) / 2, shift = j - pad;
  const long M = (long)B * L;
  const long per = (M + chunks - 1) / chunks;
  const long m_begin = (long)chunk * per, m_end = m_begin + per < M ? m_begin + per : M;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;   // 16 x 16 threads, 4 x 4 outputs each
  float acc[4][4] = {};
  for (long m0 = m_begin; m0 < m_end; m0 += WG_KM) {
    for (int i = threadIdx.x; i < WG_KM * WG_T; i += 256) {
      const int mm = i / WG_T, cc = i - mm * WG_T;
      const long m = m0 + mm;
      float a = 0.f, bv = 0.f;
      if (m < m_end) {
        if (n0 + cc < N) a = dy[m * ldy + n0 + cc];
        const long bb = m / L; const int t = (int)(m - bb * L) + shift;
        if (t >= 0 && t < L && k0 + cc < K) bv = x[(bb * L + t) * ldx + k0 + cc];
      }
      sa[mm][cc] = a; sb[mm][cc] = bv;
    }
    __syncthreads();
#pragma unroll
    for (int mm = 0; mm < WG_KM; ++mm) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = sa[mm][ty * 4 + i]; b[i] = sb[mm][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[i][q] = fmaf(a[i], b[q], acc[i][q]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int n = n0 + ty * 4 + i, k = k0 + tx * 4 + q;
      if (n < N && k < K) atomicAdd(dw + ((long)n * K + k) * taps + j, acc[i][q]);
    }
}
// reference layout [N][K][taps] -> dgrad operand in kernel layout [taps][K][N] with the taps reversed:
// dx[b,t,k] = sum_j sum_n dy[b, t + (taps-1-j) - pad', n] ... i.e. a "same" convolution of dy with W'[j'][k][n] = W[n][k][taps-1-j']
__global__ void pack_dgrad_weight_kernel(const float* __restrict__ w, int N, int K, int taps, float* __restrict__ out) {
  const long total = (long)N * K * taps;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int n = (int)(i % N); const long r = i / N; const int k = (int)(r % K); const int jp = (int)(r / K);
    out[i] = w[((long)n * K + k) * taps + (taps - 1 - jp)];
  }
}

// ---- LayerNorm backward (nn.LayerNorm over the last dim; encoder.py:37-38, modules.py:112-120) ---------------------------------
// x: the saved INPUT rows [rows, C]; dy, gamma -> dx; dgamma, dbeta accumulated with atomics (one partial sum per CTA).
template <int NV>
__global__ void __launch_bounds__(256)
layernorm_backward_kernel(const float* __restrict__ x, const float* __restrict__ dy, const float* __restrict__ gamma, float eps, long rows,
                          float* __restrict__ dx, float* __restrict__ dgamma, float* __restrict__ dbeta) {
  constexpr int C = NV * 128;
  __shared__ float sg[C], sb[C];
  for (int i = threadIdx.x; i < C; i += blockDim.x) { sg[i] = 0.f; sb[i] = 0.f; }
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float4 g4[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) g4[i] = __ldg(reinterpret_cast<const float4*>(gamma + i * 128 + lane * 4));
  float4 ag[NV], ab[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) { ag[i] = make_float4(0.f, 0.f, 0.f, 0.f); ab[i] = ag[i]; }
  for (long row = (long)blockIdx.x * 8 + wid; row < rows; row += (long)gridDim.x * 8) {
    float4 v[NV], d[NV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      v[i] = *reinterpret_cast<const float4*>(x + row * C + i * 128 + lane * 4);
      d[i] = *reinterpret_cast<const float4*>(dy + row * C + i * 128 + lane * 4);
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
    const float mean = warp_sum(s) * (1.0f / C);
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      v[i].x -= mean; v[i].y -= mean; v[i].z -= mean; v[i].w -= mean;
      ss += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
    }
    const float rstd = 1.0f / sqrtf(warp_sum(ss) * (1.0f / C) + eps);
    float sg1 = 0.f, sg2 = 0.f;   // sum(g), sum(g * xhat) with g = dy * gamma
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      v[i].x *= rstd; v[i].y *= rstd; v[i].z *= rstd; v[i].w *= rstd;           // xhat
      ag[i].x += d[i].x * v[i].x; ag[i].y += d[i].y * v[i].y; ag[i].z += d[i].z * v[i].z; ag[i].w += d[i].w * v[i].w;
      ab[i].x += d[i].x; ab[i].y += d[i].y; ab[i].z += d[i].z; ab[i].w += d[i].w;
      d[i].x *= g4[i].x; d[i].y *= g4[i].y; d[i].z *= g4[i].z; d[i].w *= g4[i].w;   // g
      sg1 += (d[i].x + d[i].y) + (d[i].z + d[i].w);
      sg2 += (d[i].x * v[i].x + d[i].y * v[i].y) + (d[i].z * v[i].z + d[i].w * v[i].w);
    }
    sg1 = warp_sum(sg1) * (1.0f / C); sg2 = warp_sum(sg2) * (1.0f / C);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      float4 o;
      o.x = rstd * (d[i].x - sg1 - v[i].x * sg2); o.y = rstd * (d[i].y - sg1 - v[i].y * sg2);
      o.z = rstd * (d[i].z - sg1 - v[i].z * sg2); o.w = rstd * (d[i].w - sg1 - v[i].w * sg2);
      *reinterpret_cast<float4*>(dx + row * C + i * 128 + lane * 4) = o;
    }
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = i * 128 + lane * 4;
    atomicAdd(&sg[c], ag[i].x); atomicAdd(&sg[c + 1], ag[i].y); atomicAdd(&sg[c + 2], ag[i].z); atomicAdd(&sg[c + 3], ag[i].w);
    atomicAdd(&sb[c], ab[i].x); atomicAdd(&sb[c + 1], ab[i].y); atomicAdd(&sb[c + 2], ab[i].z); atomicAdd(&sb[c + 3], ab[i].w);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < C; i += blockDim.x) { atomicAdd(dgamma + i, sg[i]); atomicAdd(dbeta + i, sb[i]); }
}

// ---- BatchNorm1d in train mode over rows of [rows, C] (modules.py:283-348: the Postnet's BatchNorm1d sees [B, C, L], i.e. its
// statistics run over all B*L frames of a channel, padded frames included) ----------------------------------------------------
// stats[0..C) = mean, stats[C..2C) = biased variance; also updates running_mean / running_var (momentum, unbiased variance)
__global__ void bn_stats_kernel(const float* __restrict__ x, long rows, int C, float* __restrict__ part /*[2][C] double-sum as float pairs*/) {
  // grid (C/32 ceil, chunks): partial sums and sums of squares in double
  __shared__ double r1[8][33], r2[8][33];
  const int c = blockIdx.x * 32 + (threadIdx.x & 31), rl = threadIdx.x >> 5;
  double s = 0.0, q = 0.0;
  if (c < C)
    for (long r = (long)blockIdx.y * 8 + rl; r < rows; r += (long)gridDim.y * 8) { const double v = x[r * C + c]; s += v; q += v * v; }
  r1[rl][threadIdx.x & 31] = s; r2[rl][threadIdx.x & 31] = q;
  __syncthreads();
  if (rl == 0 && c < C) {
    double a = 0.0, b = 0.0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { a += r1[i][threadIdx.x & 31]; b += r2[i][threadIdx.x & 31]; }
    atomicAdd(reinterpret_cast<double*>(part) + c, a);
    atomicAdd(reinterpret_cast<double*>(part) + C + c, b);
  }
}
__global__ void bn_finalize_kernel(const double* __restrict__ part, long rows, int C, float momentum, float* __restrict__ stats,
                                   float* __restrict__ running_mean, float* __restrict__ running_var) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double mean = part[c] / rows;
  double var = part[C + c] / rows - mean * mean;
  if (var < 0.0) var = 0.0;
  stats[c] = (float)mean; stats[C + c] = (float)var;
  if (running_mean) {
    const double unbiased = rows > 1 ? var * rows / (rows - 1) : var;
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)mean;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unbiased;
  }
}
// y = (x - mean) * rstd * gamma + beta, then optional tanh
__global__ void bn_apply_kernel(const float* __restrict__ x, const float* __restrict__ stats, const float* __restrict__ gamma,
                                const float* __restrict__ beta, float eps, long rows, int C, int act, float* __restrict__ y) {
  const long n = rows * C;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    float v = (x[i] - stats[c]) * (1.0f / sqrtf(stats[C + c] + eps)) * gamma[c] + beta[c];
    y[i] = act == ACT_TANH ? tanhf(v) : v;
  }
}
// backward: sums[0..C) = sum dy, sums[C..2C) = sum dy * xhat (double), then
// dx = gamma * rstd / M * (M dy - sum dy - xhat * sum(dy xhat)); dgamma = sum dy xhat; dbeta = sum dy
__global__ void bn_backward_sums_kernel(const float* __restrict__ x, const float* __restrict__ dy, const float* __restrict__ stats, float eps,
                                        long rows, int C, double* __restrict__ sums) {
  __shared__ double r1[8][33], r2[8][33];
  const int c = blockIdx.x * 32 + (threadIdx.x & 31), rl = threadIdx.x >> 5;
  double s = 0.0, q = 0.0;
  if (c < C) {
    const float mean = stats[c], rstd = 1.0f / sqrtf(stats[C + c] + eps);
    for (long r = (long)blockIdx.y * 8 + rl; r < rows; r += (long)gridDim.y * 8) {
      const float g = dy[r * C + c];
      s += g; q += (double)g * ((x[r * C + c] - mean) * rstd);
    }
  }
  r1[rl][threadIdx.x & 31] = s; r2[rl][threadIdx.x & 31] = q;
  __syncthreads();
  if (rl == 0 && c < C) {
    double a = 0.0, b = 0.0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { a += r1[i][threadIdx.x & 31]; b += r2[i][threadIdx.x & 31]; }
    atomicAdd(sums + c, a); atomicAdd(sums + C + c, b);
  }
}
__global__ void bn_backward_apply_kernel(const float* __restrict__ x, const float* __restrict__ dy, const float* __restrict__ stats,
                                         const float* __restrict__ gamma, float eps, long rows, int C, const double* __restrict__ sums,
                                         float* __restrict__ dx, float* __restrict__ dgamma, float* __restrict__ dbeta) {
  const long n = rows * C;
  const float invM = 1.0f / (float)rows;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const float rstd = 1.0f / sqrtf(stats[C + c] + eps), xh = (x[i] - stats[c]) * rstd;
    dx[i] = gamma[c] * rstd * (dy[i] - (float)sums[c] * invM - xh * (float)sums[C + c] * invM);
    if (i < C) { atomicAdd(dgamma + c, (float)sums[C + c]); atomicAdd(dbeta + c, (float)sums[c]); }
  }
}

// ---- batched fp32 GEMM for the attention products in train mode ------------------------------------------------------------------
// C[z][m][n] = alpha * sum_k A(z)[m][k] * B(z)[k][n], z = (b, h); element (m,k) of A at a + b*abs + h*ahs + m*ars + k*acs (strides in
// floats), same for B and C: every operand / transpose of attention.py:55-70 and of its backward is a choice of strides.
struct BgemmOperand { const float* p; long bs, hs, rs, cs; };
__global__ void __launch_bounds__(256)
bgemm_kernel(BgemmOperand A, BgemmOperand Bm, float* __restrict__ Cp, long cbs, long chs, long crs, long ccs, int heads, int M, int N, int K, float alpha) {
  __shared__ float sa[16][65], sb[16][65];
  const int z = blockIdx.z, b = z / heads, h = z - b * heads;
  const float* a = A.p + b * A.bs + h * A.hs; const float* bb = Bm.p + b * Bm.bs + h * Bm.hs;
  float* c = Cp + b * cbs + h * chs;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += 16) {
    for (int i = threadIdx.x; i < 16 * 64; i += 256) {
      // A tile [k][m]: pick the index order that keeps global reads contiguous for the contiguous stride
      int kk, mm;
      if (A.cs == 1) { kk = i & 15; mm = i >> 4; } else { mm = i & 63; kk = i >> 6; }
      sa[kk][mm] = (m0 + mm < M && k0 + kk < K) ? a[(long)(m0 + mm) * A.rs + (long)(k0 + kk) * A.cs] : 0.f;
      int k2, nn;
      if (Bm.rs == 1) { k2 = i & 15; nn = i >> 4; } else { nn = i & 63; k2 = i >> 6; }
      sb[k2][nn] = (n0 + nn < N && k0 + k2 < K) ? bb[(long)(k0 + k2) * Bm.rs + (long)(n0 + nn) * Bm.cs] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { av[i] = sa[kk][ty * 4 + i]; bv[i] = sb[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[i][q] = fmaf(av[i], bv[q], acc[i][q]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int m = m0 + ty * 4 + i, n = n0 + tx * 4 + q;
      if (m < M && n < N) c[(long)m * crs + (long)n * ccs] = alpha * acc[i][q];
    }
}
// attention.py:58-69 on materialised scores s [B*h, L, L]: mask (query AND key < len_b), softmax over keys, masked_fill(0),
// then dropout: p (pre-dropout probabilities, saved for backward) and pd = p * mask / (1 - rate).  One warp per row.
__global__ void attn_softmax_kernel(const float* __restrict__ s, const int64_t* __restrict__ lens, const uint8_t* __restrict__ dmask,
                                    float keep_scale, int heads, int L, long rows, float* __restrict__ p, float* __restrict__ pd) {
  const long row = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const long z = row / L; const int t = (int)(row - z * L);
  const int b = (int)(z / heads);
  const int len = lens ? (int)min((long)lens[b], (long)L) : L;
  const float* sr = s + row * L; float* pr = p + row * L; float* pdr = pd + row * L;
  const bool qvalid = t < len;
  float m = -INFINITY;
  if (qvalid) for (int u = lane; u < len; u += 32) m = fmaxf(m, sr[u]);
  m = warp_max(m);
  float sum = 0.f;
  if (qvalid) for (int u = lane; u < len; u += 32) sum += expf(sr[u] - m);
  sum = warp_sum(sum);
  const float inv = qvalid ? 1.0f / sum : 0.f;
  for (int u = lane; u < L; u += 32) {
    const float v = (qvalid && u < len) ? expf(sr[u] - m) * inv : 0.f;
    pr[u] = v;
    pdr[u] = dmask ? (dmask[row * L + u] ? v * keep_scale : 0.f) : v;
  }
}
// dS = P o (dP - rowsum(dP o P)) with dP = dPd * mask * keep_scale; masked positions have P = 0 -> dS = 0
__global__ void attn_softmax_backward_kernel(const float* __restrict__ p, const float* __restrict__ dpd, const uint8_t* __restrict__ dmask,
                                             float keep_scale, int L, long rows, float* __restrict__ ds) {
  const long row = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float* pr = p + row * L; const float* gr = dpd + row * L; float* dr = ds + row * L;
  float dot = 0.f;
  for (int u = lane; u < L; u += 32) {
    const float g = dmask ? (dmask[row * L + u] ? gr[u] * keep_scale : 0.f) : gr[u];
    dot += g * pr[u];
  }
  dot = warp_sum(dot);
  for (int u = lane; u < L; u += 32) {
    const float g = dmask ? (dmask[row * L + u] ? gr[u] * keep_scale : 0.f) : gr[u];
    dr[u] = pr[u] * (g - dot);
  }
}

// ---- embedding / positional encoding backward (fastspeech.py:65-67, embedding.py:105-120) ---------------------------------------
// dtable[id] += dy[row] (id != padding_idx 0: nn.Embedding(padding_idx=0) keeps that row's gradient at zero);
// dalpha += sum dy * pe[t]
__global__ void embed_backward_kernel(const int64_t* __restrict__ xs, const float* __restrict__ dy, const float* __restrict__ pe, long rows, int T,
                                      int C, int n_sym, float* __restrict__ dtable, float* __restrict__ dalpha) {
  const long row = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  float da = 0.f;
  if (row < rows) {
    const long id = xs ? xs[row] : 0; const int t = (int)(row % T);
    for (int c = lane; c < C; c += 32) {
      const float g = dy[row * C + c];
      if (dtable && id > 0 && id < n_sym) atomicAdd(dtable + id * C + c, g);
      da += g * pe[(long)t * C + c];
    }
  }
  da = warp_sum(da);
  if (lane == 0 && da != 0.f) atomicAdd(dalpha, da);
}
// y[row, :] = x[row, :] + alpha * pe[row % T, :]   (ScaledPositionalEncoding on the decoder input, embedding.py:105-120)
__global__ void posenc_add_kernel(const float* __restrict__ x, const float* __restrict__ pe, const float* __restrict__ alpha, long rows, int T, int C,
                                  float* __restrict__ y) {
  const long n = rows * C;
  const float a = alpha[0];
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long row = i / C; const int c = (int)(i - row * C);
    y[i] = __fadd_rn(x[i], __fmul_rn(a, pe[(row % T) * C + c]));
  }
}
// y[row, c] = x[row, c] + (W[c, id[row]] + b[c]): Linear(n_bins -> C) applied to a one-hot row, W in the reference's [C][n_bins] layout
__global__ void onehot_linear_forward_kernel(const float* __restrict__ x, const int64_t* __restrict__ ids, const float* __restrict__ W,
                                             const float* __restrict__ b, long rows, int C, int n_bins, float* __restrict__ y) {
  const long n = rows * C;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long row = i / C; const int c = (int)(i - row * C);
    y[i] = __fadd_rn(x[i], __fadd_rn(W[(long)c * n_bins + ids[row]], b[c]));
  }
}
// pitch / energy embedding (Linear on a one-hot, fastspeech.py:102,113,218-219): dW[c][id[row]] += dy[row][c], db[c] += dy[row][c]
// W in the reference's [C][n_bins] layout
__global__ void onehot_linear_backward_kernel(const int64_t* __restrict__ ids, const float* __restrict__ dy, long rows, int C, int n_bins,
                                              float* __restrict__ dW) {
  const long row = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const long id = ids[row];
  for (int c = lane; c < C; c += 32) atomicAdd(dW + (long)c * n_bins + id, dy[row * C + c]);
}

// ---- LengthRegulator backward (length_regulator.py:90-95: repeat): dhs[b,i,:] = sum of dout[b,j,:] over the frames j copied from i ---
__global__ void length_regulator_backward_kernel(const float* __restrict__ dout, const int32_t* __restrict__ cum, const int64_t* __restrict__ ilens,
                                                 int T, int C, int Lcap, float* __restrict__ dhs) {
  const int b = blockIdx.y, i = blockIdx.x;
  long il = ilens[b]; if (il > T) il = T;
  float* dst = dhs + ((long)b * T + i) * C;
  if (i >= il) { for (int c = threadIdx.x; c < C; c += blockDim.x) dst[c] = 0.f; return; }
  const int j0 = i ? cum[(long)b * T + i - 1] : 0, j1 = min(cum[(long)b * T + i], Lcap);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float s = 0.f;
    for (int j = j0; j < j1; ++j) s += dout[((long)b * Lcap + j) * C + c];
    dst[c] = s;
  }
}

// ---- predictor head: Linear(C -> 1) on rows, masked (duration_predictor.py:75,83-84; variance_predictor.py:51,75-78) -----------
__global__ void rowdot_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias, const int64_t* __restrict__ lens,
                              long rows, int L, int C, float* __restrict__ y) {
  const long row = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += x[row * C + c] * w[c];
  s = warp_sum(s) + bias[0];
  if (lane == 0) y[row] = (lens && (row % L) >= lens[row / L]) ? 0.f : s;
}
__global__ void rowdot_backward_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ dy, const int64_t* __restrict__ lens,
                                       long rows, int L, int C, float* __restrict__ dx, float* __restrict__ dw, float* __restrict__ dbias) {
  __shared__ float sw[384];
  for (int i = threadIdx.x; i < C; i += blockDim.x) sw[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float db = 0.f;
  for (long row = (long)blockIdx.x * 8 + wid; row < rows; row += (long)gridDim.x * 8) {
    const float g = (lens && (row % L) >= lens[row / L]) ? 0.f : dy[row];
    for (int c = lane; c < C; c += 32) {
      dx[row * C + c] = g * w[c];
      atomicAdd(&sw[c], g * x[row * C + c]);
    }
    if (lane == 0) db += g;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < C; i += blockDim.x) atomicAdd(dw + i, sw[i]);
  if (lane == 0 && db != 0.f) atomicAdd(dbias, db);
}

// ---- loss backward (fastspeech.py:277-324 with use_masking): upstream g = dL/dloss ----------------------------------------------
__global__ void loss_backward_kernel(const float* __restrict__ before, const float* __restrict__ after, const float* __restrict__ ys, int ld_ys_time,
                                     const float* __restrict__ d_out, const void* __restrict__ ds, int ds_dtype, const float* __restrict__ e_out,
                                     const float* __restrict__ p_out, const float* __restrict__ es, const float* __restrict__ ps,
                                     const int64_t* __restrict__ ilens, const int64_t* __restrict__ olens, int B, int T, int L, int odim,
                                     const float* __restrict__ gptr, float* __restrict__ g_before, float* __restrict__ g_after,
                                     float* __restrict__ g_d, float* __restrict__ g_e, float* __restrict__ g_p) {
  __shared__ float ni_s, no_s;
  if (threadIdx.x == 0) {
    double ni = 0, no = 0;
    for (int b = 0; b < B; ++b) { ni += (double)ilens[b]; no += (double)olens[b]; }
    ni_s = (float)ni; no_s = (float)no;
  }
  __syncthreads();
  const float g = gptr[0];
  const float cm = g / (no_s * odim), cd = 2.f * g / ni_s, ce = 2.f * g / no_s;
  const long n_mel = (long)B * L * odim, n_t = (long)B * T, n_l = (long)B * L;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n_mel; i += (long)gridDim.x * blockDim.x) {
    const long bl = i / odim; const int c = (int)(i - bl * odim);
    const long b = bl / L; const int t = (int)(bl - b * L);
    const bool valid = t < olens[b];
    const float y = valid ? ys[(b * ld_ys_time + t) * odim + c] : 0.f;
    const float d0 = before[i] - y, d1 = after[i] - y;
    g_before[i] = valid ? (d0 > 0.f ? cm : d0 < 0.f ? -cm : 0.f) : 0.f;
    g_after[i] = valid ? (d1 > 0.f ? cm : d1 < 0.f ? -cm : 0.f) : 0.f;
  }
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n_t; i += (long)gridDim.x * blockDim.x) {
    const long b = i / T; const int t = (int)(i - b * T);
    float v = 0.f;
    if (t < ilens[b]) {
      const float d = ds_dtype == FS2_DUR_F32 ? ((const float*)ds)[i] : ds_dtype == FS2_DUR_I32 ? (float)((const int32_t*)ds)[i] : (float)((const int64_t*)ds)[i];
      v = cd * (d_out[i] - logf(d + 1.0f));
    }
    g_d[i] = v;
  }
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n_l; i += (long)gridDim.x * blockDim.x) {
    const long b = i / L; const int t = (int)(i - b * L);
    const bool valid = t < olens[b];
    g_e[i] = valid ? ce * (e_out[i] - es[i]) : 0.f;
    g_p[i] = valid ? ce * (p_out[i] - ps[i]) : 0.f;
  }
}

// the bodies of fs2_conv_forward(_ex) and fs2_conv_dgrad(_ex) (see there); `who` names the entry in error messages
int conv_forward(const char* who, int math_mode, const float* x, int B, int L, int K, const float* w, const float* bias, int N,
                 int taps, int act, const float* resid, float* out, float* scratch, void* stream) {
  FS2_REQUIRE(x && w && out && scratch, "%s: null argument", who);
  cudaStream_t st = (cudaStream_t)stream;
  int rc = pack_conv_weight(w, N, K, taps, nullptr, scratch, st);
  if (rc) return rc;
  VWeight pw; pw.w = scratch; pw.bias = const_cast<float*>(bias); pw.N = N; pw.K = K; pw.taps = taps;
  return vweight_gemm(math_mode, pw, x, B, L, act, nullptr, out, st, resid);
}
int conv_dgrad(const char* who, int math_mode, const float* dy, int B, int L, int N, const float* w, int K, int taps, float* dx,
               float* scratch, void* stream) {
  FS2_REQUIRE(dy && w && dx && scratch, "%s: null argument", who);
  FS2_REQUIRE(taps > 0 && (taps & 1) == 1, "%s: taps must be odd (got %d)", who, taps);
  cudaStream_t st = (cudaStream_t)stream;
  pack_dgrad_weight_kernel<<<grid_for((long)N * K * taps, 256), 256, 0, st>>>(w, N, K, taps, scratch);
  FS2_LAUNCH_CHECK();
  VWeight pw; pw.w = scratch; pw.N = K; pw.K = N; pw.taps = taps;   // dx = conv(dy, w flipped / transposed): K outputs from N inputs
  return vweight_gemm(math_mode, pw, dy, B, L, ACT_NONE, nullptr, dx, st);
}

}  // namespace
}  // namespace fs2

using namespace fs2;

extern "C" {

int fs2_dropout_mask(uint8_t* mask, int64_t n, float p, uint64_t seed, uint64_t offset, void* stream) {
  FS2_REQUIRE(mask && n >= 0 && p >= 0.f && p < 1.f, "fs2_dropout_mask: bad argument");
  if (n == 0) return FS2_OK;
  dropout_mask_kernel<<<grid_for((n + 3) / 4, 256), 256, 0, (cudaStream_t)stream>>>(mask, n, p, seed, offset);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_dropout_apply(const float* x, const uint8_t* mask, float p, float* out, int64_t n, void* stream) {
  FS2_REQUIRE(x && mask && out && p >= 0.f && p < 1.f, "fs2_dropout_apply: bad argument");
  if (n == 0) return FS2_OK;
  dropout_apply_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(x, mask, 1.0f / (1.0f - p), out, n);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_act_backward(const float* dy, const float* y, int act, float* dx, int64_t n, void* stream) {
  FS2_REQUIRE(dy && y && dx, "fs2_act_backward: null argument");
  if (n == 0) return FS2_OK;
  act_backward_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(dy, y, act, dx, n);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_relu(const float* x, float* y, int64_t n, void* stream) {
  FS2_REQUIRE(x && y, "fs2_relu: null argument");
  if (n == 0) return FS2_OK;
  relu_forward_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(x, y, n);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_add(const float* a, const float* b, float* y, int64_t n, void* stream) {
  FS2_REQUIRE(a && b && y, "fs2_add: null argument");
  if (n == 0) return FS2_OK;
  add_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(a, b, y, n);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_colsum(const float* x, int64_t rows, int C, float* out, void* stream) {
  FS2_REQUIRE(x && out && C > 0, "fs2_colsum: bad argument");
  if (rows == 0) return FS2_OK;
  dim3 grid((C + 31) / 32, (unsigned)(rows / 512 + 1 > 64 ? 64 : rows / 512 + 1));
  colsum_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, rows, C, out);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
/* Conv1d / Linear in the reference's weight layout w [N][K][taps]:
 *   forward   out = act(conv(x, w) + bias) (+ resid)        (packs w into the kernel layout, then the fp32 tap-GEMM)
 *   dgrad     dx  = conv(dy, w flipped / transposed)
 *   wgrad     dw += dy^T x (per tap), accumulated into the caller's zero-initialised / running gradient
 * scratch: >= N*K*taps floats */
int fs2_conv_forward(const float* x, int B, int L, int K, const float* w, const float* bias, int N, int taps, int act, const float* resid,
                     float* out, float* scratch, void* stream) {
  return conv_forward("fs2_conv_forward", FS2_MATH_FP32, x, B, L, K, w, bias, N, taps, act, resid, out, scratch, stream);
}
int fs2_conv_dgrad(const float* dy, int B, int L, int N, const float* w, int K, int taps, float* dx, float* scratch, void* stream) {
  return conv_dgrad("fs2_conv_dgrad", FS2_MATH_FP32, dy, B, L, N, w, K, taps, dx, scratch, stream);
}
/* the same with a math mode: FS2_MATH_FP32 is exactly the calls above; FS2_MATH_TF32 runs the packed weights through the
 * tap GEMM's tf32 family (gemm_tc.cu) */
int fs2_conv_forward_ex(const float* x, int B, int L, int K, const float* w, const float* bias, int N, int taps, int act, const float* resid,
                        float* out, float* scratch, int math_mode, void* stream) {
  if (math_mode == FS2_MATH_FP32) return fs2_conv_forward(x, B, L, K, w, bias, N, taps, act, resid, out, scratch, stream);
  FS2_REQUIRE(math_mode == FS2_MATH_TF32, "fs2_conv_forward_ex: math_mode must be FS2_MATH_FP32 or FS2_MATH_TF32");
  return conv_forward("fs2_conv_forward_ex", math_mode, x, B, L, K, w, bias, N, taps, act, resid, out, scratch, stream);
}
int fs2_conv_dgrad_ex(const float* dy, int B, int L, int N, const float* w, int K, int taps, float* dx, float* scratch, int math_mode,
                      void* stream) {
  if (math_mode == FS2_MATH_FP32) return fs2_conv_dgrad(dy, B, L, N, w, K, taps, dx, scratch, stream);
  FS2_REQUIRE(math_mode == FS2_MATH_TF32, "fs2_conv_dgrad_ex: math_mode must be FS2_MATH_FP32 or FS2_MATH_TF32");
  return conv_dgrad("fs2_conv_dgrad_ex", math_mode, dy, B, L, N, w, K, taps, dx, scratch, stream);
}
int fs2_conv_wgrad(const float* dy, const float* x, int B, int L, int N, int K, int taps, float* dw, float* dbias, void* stream) {
  FS2_REQUIRE(dy && x && dw, "fs2_conv_wgrad: null argument");
  FS2_REQUIRE(B >= 0 && L >= 0 && N > 0 && K > 0 && taps > 0 && (taps & 1) == 1, "fs2_conv_wgrad: need B, L >= 0, N, K > 0 and odd taps");
  cudaStream_t st = (cudaStream_t)stream;
  const long M = (long)B * L;
  if (M == 0) return FS2_OK;
  const int tiles = ((N + WG_T - 1) / WG_T) * ((K + WG_T - 1) / WG_T) * taps;
  int chunks = (132 * 4 + tiles - 1) / tiles;
  const long max_chunks = (M + 255) / 256;
  if (chunks > max_chunks) chunks = (int)max_chunks;
  if (chunks < 1) chunks = 1;
  dim3 grid((N + WG_T - 1) / WG_T, (K + WG_T - 1) / WG_T, taps * chunks);
  wgrad_kernel<<<grid, 256, 0, st>>>(dy, N, x, K, B, L, N, K, taps, chunks, dw);
  FS2_LAUNCH_CHECK();
  if (dbias) return fs2_colsum(dy, M, N, dbias, stream);
  return FS2_OK;
}
int fs2_layernorm_backward(const float* x, const float* dy, const float* gamma, float eps, int64_t rows, int C, float* dx, float* dgamma,
                           float* dbeta, void* stream) {
  FS2_REQUIRE(x && dy && gamma && dx && dgamma && dbeta, "fs2_layernorm_backward: null argument");
  if (rows == 0) return FS2_OK;
  const int grid = (int)(rows / 8 + 1 > 132 * 4 ? 132 * 4 : rows / 8 + 1);
  if (C == 256) layernorm_backward_kernel<2><<<grid, 256, 0, (cudaStream_t)stream>>>(x, dy, gamma, eps, rows, dx, dgamma, dbeta);
  else if (C == 384) layernorm_backward_kernel<3><<<grid, 256, 0, (cudaStream_t)stream>>>(x, dy, gamma, eps, rows, dx, dgamma, dbeta);
  else { set_error("fs2_layernorm_backward: C=%d unsupported (256 or 384)", C); return FS2_ERR_INVALID; }
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
/* BatchNorm1d, training: stats [2*C] out (mean, biased var), running stats updated in place; scratch >= 4*C doubles, zeroed here */
int fs2_batchnorm_train(const float* x, int64_t rows, int C, const float* gamma, const float* beta, float eps, float momentum, int act,
                        float* running_mean, float* running_var, float* stats, float* y, void* scratch, void* stream) {
  FS2_REQUIRE(x && gamma && beta && stats && y && scratch && rows > 0, "fs2_batchnorm_train: bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  FS2_CUDA_CHECK(cudaMemsetAsync(scratch, 0, (size_t)2 * C * sizeof(double), st));
  dim3 grid((C + 31) / 32, (unsigned)(rows / 256 + 1 > 128 ? 128 : rows / 256 + 1));
  bn_stats_kernel<<<grid, 256, 0, st>>>(x, rows, C, reinterpret_cast<float*>(scratch));
  FS2_LAUNCH_CHECK();
  bn_finalize_kernel<<<(C + 127) / 128, 128, 0, st>>>(reinterpret_cast<const double*>(scratch), rows, C, momentum, stats, running_mean, running_var);
  FS2_LAUNCH_CHECK();
  bn_apply_kernel<<<grid_for(rows * C, 256), 256, 0, st>>>(x, stats, gamma, beta, eps, rows, C, act, y);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_batchnorm_backward(const float* x, const float* dy, const float* stats, const float* gamma, float eps, int64_t rows, int C, float* dx,
                           float* dgamma, float* dbeta, void* scratch, void* stream) {
  FS2_REQUIRE(x && dy && stats && gamma && dx && dgamma && dbeta && scratch && rows > 0, "fs2_batchnorm_backward: bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  FS2_CUDA_CHECK(cudaMemsetAsync(scratch, 0, (size_t)2 * C * sizeof(double), st));
  dim3 grid((C + 31) / 32, (unsigned)(rows / 256 + 1 > 128 ? 128 : rows / 256 + 1));
  bn_backward_sums_kernel<<<grid, 256, 0, st>>>(x, dy, stats, eps, rows, C, reinterpret_cast<double*>(scratch));
  FS2_LAUNCH_CHECK();
  bn_backward_apply_kernel<<<grid_for(rows * C, 256), 256, 0, st>>>(x, dy, stats, gamma, eps, rows, C, reinterpret_cast<const double*>(scratch), dx, dgamma, dbeta);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
/* strided batched fp32 GEMM over z = (b, h): C = alpha * A . B with every operand given by (pointer, batch stride, head stride,
 * row stride, column stride) in floats */
int fs2_bgemm(const float* a, int64_t abs_, int64_t ahs, int64_t ars, int64_t acs, const float* b, int64_t bbs, int64_t bhs, int64_t brs, int64_t bcs,
              float* c, int64_t cbs, int64_t chs, int64_t crs, int64_t ccs, int batch, int heads, int M, int N, int K, float alpha, void* stream) {
  FS2_REQUIRE(a && b && c && heads > 0, "fs2_bgemm: bad argument");
  if (batch == 0 || M == 0 || N == 0) return FS2_OK;
  BgemmOperand A{a, abs_, ahs, ars, acs}, Bm{b, bbs, bhs, brs, bcs};
  dim3 grid((N + 63) / 64, (M + 63) / 64, batch * heads);
  bgemm_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(A, Bm, c, cbs, chs, crs, ccs, heads, M, N, K, alpha);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_attn_softmax(const float* s, const int64_t* lens, const uint8_t* dmask, float p_drop, int B, int heads, int L, float* p, float* pd, void* stream) {
  FS2_REQUIRE(s && p && pd && p_drop >= 0.f && p_drop < 1.f, "fs2_attn_softmax: bad argument");
  const long rows = (long)B * heads * L;
  if (rows == 0) return FS2_OK;
  attn_softmax_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(s, lens, dmask, 1.0f / (1.0f - p_drop), heads, L, rows, p, pd);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_attn_softmax_backward(const float* p, const float* dpd, const uint8_t* dmask, float p_drop, int B, int heads, int L, float* ds, void* stream) {
  FS2_REQUIRE(p && dpd && ds, "fs2_attn_softmax_backward: null argument");
  const long rows = (long)B * heads * L;
  if (rows == 0) return FS2_OK;
  attn_softmax_backward_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(p, dpd, dmask, 1.0f / (1.0f - p_drop), L, rows, ds);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_embed_backward(const int64_t* xs, const float* dy, const float* pe, int B, int T, int C, int n_sym, float* dtable, float* dalpha, void* stream) {
  FS2_REQUIRE(dy && pe && dalpha && (xs || !dtable), "fs2_embed_backward: null argument");
  const long rows = (long)B * T;
  if (rows == 0) return FS2_OK;
  embed_backward_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(xs, dy, pe, rows, T, C, n_sym, dtable, dalpha);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_embed_posenc(const int64_t* xs, const float* table, int n_sym, const float* pe, const float* alpha, int B, int T, int C, float* out,
                     void* stream) {
  FS2_REQUIRE(xs && table && pe && alpha && out, "fs2_embed_posenc: null argument");
  return embed_posenc(xs, table, n_sym, pe, alpha, B, T, C, out, nullptr, nullptr, (cudaStream_t)stream);
}
int fs2_posenc_add(const float* x, const float* pe, const float* alpha, int B, int T, int C, float* y, void* stream) {
  FS2_REQUIRE(x && pe && alpha && y, "fs2_posenc_add: null argument");
  const long n = (long)B * T * C;
  if (n == 0) return FS2_OK;
  posenc_add_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(x, pe, alpha, (long)B * T, T, C, y);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_onehot_linear_forward(const float* x, const int64_t* ids, const float* W, const float* b, int64_t rows, int C, int n_bins, float* y,
                              void* stream) {
  FS2_REQUIRE(x && ids && W && b && y, "fs2_onehot_linear_forward: null argument");
  if (rows == 0) return FS2_OK;
  onehot_linear_forward_kernel<<<grid_for(rows * C, 256), 256, 0, (cudaStream_t)stream>>>(x, ids, W, b, rows, C, n_bins, y);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_onehot_linear_backward(const int64_t* ids, const float* dy, int64_t rows, int C, int n_bins, float* dW, float* dbias, void* stream) {
  FS2_REQUIRE(ids && dy && dW, "fs2_onehot_linear_backward: null argument");
  if (rows == 0) return FS2_OK;
  onehot_linear_backward_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(ids, dy, rows, C, n_bins, dW);
  FS2_LAUNCH_CHECK();
  if (dbias) return fs2_colsum(dy, rows, C, dbias, stream);
  return FS2_OK;
}
int fs2_length_regulator_backward(const float* dout, const int32_t* cum, const int64_t* ilens, int B, int T, int C, int Lcap, float* dhs, void* stream) {
  FS2_REQUIRE(dout && cum && ilens && dhs, "fs2_length_regulator_backward: null argument");
  if (B == 0 || T == 0) return FS2_OK;
  dim3 grid(T, B);
  length_regulator_backward_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(dout, cum, ilens, T, C, Lcap, dhs);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_rowdot(const float* x, const float* w, const float* bias, const int64_t* lens, int64_t rows, int L, int C, float* y, void* stream) {
  FS2_REQUIRE(x && w && bias && y && L > 0, "fs2_rowdot: bad argument");
  if (rows == 0) return FS2_OK;
  rowdot_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(x, w, bias, lens, rows, L, C, y);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_rowdot_backward(const float* x, const float* w, const float* dy, const int64_t* lens, int64_t rows, int L, int C, float* dx, float* dw,
                        float* dbias, void* stream) {
  FS2_REQUIRE(x && w && dy && dx && dw && dbias && L > 0 && C <= 384, "fs2_rowdot_backward: bad argument");
  if (rows == 0) return FS2_OK;
  const int grid = (int)(rows / 8 + 1 > 132 * 4 ? 132 * 4 : rows / 8 + 1);
  rowdot_backward_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, w, dy, lens, rows, L, C, dx, dw, dbias);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_loss_backward(const float* before, const float* after, const float* ys, int ld_ys_time, const float* d_out, const void* ds, int ds_dtype,
                      const float* e_out, const float* p_out, const float* es, const float* ps, const int64_t* ilens, const int64_t* olens,
                      int B, int T, int L, int odim, const float* grad_loss, float* g_before, float* g_after, float* g_d, float* g_e, float* g_p,
                      void* stream) {
  FS2_REQUIRE(before && after && ys && d_out && ds && e_out && p_out && es && ps && ilens && olens && grad_loss && g_before && g_after && g_d && g_e && g_p,
              "fs2_loss_backward: null argument");
  loss_backward_kernel<<<grid_for((long)B * L * odim, 256), 256, 0, (cudaStream_t)stream>>>(before, after, ys, ld_ys_time, d_out, ds, ds_dtype, e_out, p_out,
                                                                                           es, ps, ilens, olens, B, T, L, odim, grad_loss, g_before,
                                                                                           g_after, g_d, g_e, g_p);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // extern "C"
