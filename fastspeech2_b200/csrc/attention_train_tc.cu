// Fused tensor-core attention for the tf32 train step (DESIGN.md §13): forward and backward of core/attention.py:52-73 in
// train mode, the contract of train.py's AttentionFn (the materialized path), without any [B, h, L, L] tensor.
//
//   S = q.k^T / sqrt(dk), valid where query AND key < len_b; P = softmax over the valid keys (0 elsewhere; rows past len
//   are 0); Pd = P o M / (1 - p); O = Pd.V.   Backward with D = rowsum(dO o O):
//   dV = Pd^T.dO   dP = (dO.V^T) o M / (1 - p)   dS = P o (dP - D)   dQ = dS.K / sqrt(dk)   dK = dS^T.Q / sqrt(dk)
//
// Products are 1xTF32: warp-level mma.sync m16n8k8 with fp32 accumulation.  A prep pass copies q, k, v (and dO) rounded to
// tf32 with cvt.rna into the workspace, rows below len only; the tiles are loaded from there with cp.async, rows at or past
// len zero-filled, so nothing past len is ever read (NaN there changes no bit).  Loads overlap the MMAs: the forward and
// dQ kernels put their K and V tiles in separate cp.async groups and refill each as soon as its last reader is done;
// the dK/dV kernel double-buffers its Q / dO tiles.  The backward re-rounds q, k, v into its own workspace rather than
// keeping the forward's copies alive between the calls: that costs three B L C element passes per layer (a small
// fraction of the kernels' time) and keeps the saved state at q, k, v, O and the log-sum-exp.  P and dS are rounded in registers before
// they become A fragments.  Shared-memory rows are padded to dk + 4 floats, which makes every fragment load conflict free.
//
// Register-resident P: the accumulator fragment of S (thread holds keys 2t, 2t + 1 of rows g, g + 8) is used directly as
// the A fragment of P.V by reading A column t as key 2t and column t + 4 as key 2t + 1 of each 8-key slice; the B fragment
// of V (and of K in dQ += dS.K) is read from shared memory in the same order.  No permuted copy is written.
//
// Kernels (one CTA per 64-row tile of one (utterance, head); tiles wholly past len issue no MMA and write zeros):
//   attn_fwd_kernel    64 queries, 4 warps x 16 rows; key tiles of 64 up to len; online softmax in the exp2 domain.
//                      Writes O [B, L, C] and the row log-sum-exp lse [B*h, L] (natural log; 0 for rows past len).
//   attn_delta_kernel  D = rowsum(dO o O), one warp per row.
//   attn_dkdv_kernel   64 keys, 8 warps; query tiles of 32 up to len.  Warp (kg, qh) recomputes S^T and dP^T for its 16
//                      keys x 16 queries, stages Pd^T and dS^T (rounded) in shared memory; then warps qh = 0 accumulate
//                      dV = Pd^T.dO and warps qh = 1 dK = dS^T.Q over all 32 queries, each for its 16 keys x dk.  The
//                      split keeps one 16 x dk accumulator per warp (96 registers at dk = 192) and computes every
//                      product once.
//   attn_dq_kernel     64 queries, 4 warps; key tiles of 64; recomputes S and dP, accumulates dQ = dS.K.
// Every output element belongs to one CTA and is summed in a fixed order: no atomics, the same inputs give the same bits.
//
// Dropout: an explicit uint8 mask [B, h, L, L], or (seed, offset): keep bit of element e = ((b h + head) L + i) L + j is
// word e % 4 of Philox4x32-10 at counter offset + e / 4, kept if (word >> 8) 2^-24 >= p -- byte e of
// fs2_dropout_mask(mask, B h L L, p, seed, offset).  64-bit element indices throughout.
#include <math.h>

#include "tc_common.cuh"

namespace fs2 {
namespace {
using namespace tc;

constexpr int AT_TILE = 64;      // queries per forward / dQ CTA, keys per dK/dV CTA, keys per forward / dQ step
constexpr int AT_QSTEP = 32;     // queries per dK/dV step
constexpr int AT_PS = AT_QSTEP + 4;   // row pitch of the staged Pd^T / dS^T tiles
constexpr float AT_LOG2E = 1.4426950408889634f, AT_LN2 = 0.6931471805599453f;

struct Drop {
  const uint8_t* mask;           // explicit mask, or null: Philox (seed, offset)
  unsigned long long seed, offset;
  float p, keep_scale;
  int on;                        // p > 0
  int L;
};

struct AttnParams {
  const float *qr, *kr, *vr, *dor;   // tf32-rounded copies in the workspace, [B, L, C], rows below len only
  const float *o, *dout, *lse;       // backward inputs
  float* dvec;                       // D [B*h, L] (workspace)
  const int64_t* lens;
  int L, C, heads;
  float sl2, scale;                  // log2(e) / sqrt(dk), 1 / sqrt(dk)
  Drop drop;
  float *out, *lse_out, *dq, *dk, *dv;
};

__device__ __forceinline__ uint32_t u(float v) { return __float_as_uint(v); }
__device__ __forceinline__ void cp_async16(float* smem, const float* gmem, bool valid) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem), "r"(valid ? 16 : 0)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// all but the newest N committed groups have landed (this thread's copies; a __syncthreads makes them everyone's)
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ int clamp_len(const int64_t* lens, int b, int L) {
  const int64_t lb = lens[b];
  return lb < 0 ? 0 : (lb > L ? L : (int)lb);
}

// rows [r0, r0 + n) of one head (src = its column 0 in row 0, row pitch C) -> shared [n][DK + 4]; rows >= lim are zero
template <int DK>
__device__ __forceinline__ void load_rows(float* sm, const float* __restrict__ src, int C, int r0, int n, int lim, int tid, int nthr) {
  constexpr int V = DK / 4;
  for (int i = tid; i < n * V; i += nthr) {
    const int r = i / V, c = (i - r * V) * 4, row = r0 + r;
    const bool ok = row < lim;
    cp_async16(sm + r * (DK + 4) + c, src + (long)(ok ? row : 0) * C + c, ok);
  }
}

__device__ __forceinline__ unsigned word_of(uint4 r, int i) { return i == 0 ? r.x : i == 1 ? r.y : i == 2 ? r.z : r.w; }
__device__ __forceinline__ bool keep_word(unsigned w, float p) { return ((w >> 8) * (1.0f / 16777216.0f)) >= p; }
__device__ __forceinline__ uint4 philox_at(const Drop& d, unsigned long long c) {
  return philox4x32(make_uint4((unsigned)c, (unsigned)(c >> 32), 0u, 0u), make_uint2((unsigned)d.seed, (unsigned)(d.seed >> 32)));
}
// keep bits of elements e .. e + 3 (bit i = element e + i); `valid` bit i says element e + i exists (explicit mask reads)
__device__ __forceinline__ unsigned keep_four(const Drop& d, unsigned long long e, unsigned valid) {
  unsigned bits = 0;
  if (d.mask) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (((valid >> i) & 1) && d.mask[e + i]) bits |= 1u << i;
    return bits;
  }
  const int r = (int)(e & 3);
  const uint4 w0 = philox_at(d, d.offset + (e >> 2));
  uint4 w1 = w0;
  if (r) w1 = philox_at(d, d.offset + (e >> 2) + 1);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int k = r + i;
    if (keep_word(k < 4 ? word_of(w0, k) : word_of(w1, k - 4), d.p)) bits |= 1u << i;
  }
  return bits;
}

// Keep bits of the S-layout fragment of one 8-key slice: this thread holds keys c + 2t + {0,1} of rows g (row_e[0]) and
// g + 8 (row_e[1]).  Lanes t = 2s' and 2s' + 1 share keys c + 4s' .. + 3: the even lane draws them for row g, the odd lane
// for row g + 8, and they swap.  Returns bits {row g: key 2t, 2t+1; row g+8: key 2t, 2t+1} as bits 0..3.
__device__ __forceinline__ unsigned keep_frag(const Drop& d, const unsigned long long* row_e, const int* rows, int key4, int t, int len) {
  const int s = t & 1;
  unsigned valid = 0;
  const bool row_ok = (s ? rows[1] : rows[0]) < len;
#pragma unroll
  for (int i = 0; i < 4; ++i) valid |= (key4 + i < len && row_ok ? 1u : 0u) << i;
  const unsigned mine = keep_four(d, (s ? row_e[1] : row_e[0]) + key4, valid);
  const unsigned other = __shfl_xor_sync(0xffffffffu, mine, 1);
  const unsigned rg = s ? other : mine, rg8 = s ? mine : other;
  return ((rg >> (2 * s)) & 3u) | (((rg8 >> (2 * s)) & 3u) << 2);
}

// Keep bits of the S^T-layout fragment of one 8-query slice (dK/dV kernel): this thread holds queries c + 2t + {0,1} of
// key rows g and g + 8.  Keys run along lanes there (g = 4 a + r), so the four lanes r = 0..3 of a group share the keys
// 4a .. 4a + 3 (and 8 + 4a ..): lane r draws those four keys for query 2t + (r & 1) and key half r >> 1, then each lane
// gathers its key's bit from the four.  Returns bits {key g: query 2t, 2t+1; key g+8: query 2t, 2t+1} as bits 0..3.
__device__ __forceinline__ unsigned keep_frag_t(const Drop& d, unsigned long long bhL, int q, int key4, int lane, int len) {
  const int g = lane >> 2, t = lane & 3, r = g & 3, a4 = g & 4;
  const int qi = q + 2 * t + (r & 1), k4 = key4 + 8 * (r >> 1);
  unsigned valid = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) valid |= (qi < len && k4 + i < len ? 1u : 0u) << i;
  const unsigned mine = keep_four(d, (bhL + (unsigned long long)qi) * (unsigned long long)d.L + (unsigned long long)k4, valid);
  unsigned bits = 0;
#pragma unroll
  for (int rr = 0; rr < 4; ++rr) {           // rr = query parity + 2 x key half
    const unsigned w = __shfl_sync(0xffffffffu, mine, 4 * (a4 + rr) + t);
    bits |= ((w >> r) & 1u) << ((rr >> 1) * 2 + (rr & 1));
  }
  return bits;
}

// ---- prep: out = in rounded to tf32 on rows t < len of every utterance ----------------------------------------------------
__global__ void __launch_bounds__(256) attn_round_kernel(const float* __restrict__ in, const int64_t* __restrict__ lens, int L, int C, long n,
                                                         float* __restrict__ out) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long row = i / C;
    const int b = (int)(row / L), t = (int)(row - (long)b * L);
    if (t < clamp_len(lens, b, L)) out[i] = __uint_as_float(to_tf32(in[i]));
  }
}

// ---- forward ------------------------------------------------------------------------------------------------------------------
template <int DK>
__global__ void __launch_bounds__(128, 1) attn_fwd_kernel(const AttnParams a) {
  extern __shared__ float4 smem4[];
  constexpr int SS = DK + 4, NT = DK / 8;
  float* sQ = reinterpret_cast<float*>(smem4);
  float* sK = sQ + AT_TILE * SS;
  float* sV = sK + AT_TILE * SS;
  const int bh = blockIdx.x, b = bh / a.heads, hd = bh - b * a.heads;
  const int L = a.L, C = a.C, q0 = blockIdx.y * AT_TILE;
  const int len = clamp_len(a.lens, b, L);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const long ubase = (long)b * L * C + (long)hd * DK;
  float* out = a.out + ubase;
  float* lse = a.lse_out + (long)bh * L;
  const int rows[2] = {q0 + 16 * warp + g, q0 + 16 * warp + g + 8};
  if (q0 >= len) {
    for (int i = threadIdx.x; i < AT_TILE * DK; i += 128) {
      const int r = q0 + i / DK;
      if (r < L) out[(long)r * C + i % DK] = 0.f;
    }
    if (threadIdx.x < AT_TILE && q0 + (int)threadIdx.x < L) lse[q0 + threadIdx.x] = 0.f;
    return;
  }
  // K and V tiles are separate cp.async groups, each prefetched while the other is in use: K(k0 + 64) loads during the
  // softmax and P.V of step k0, V(k0 + 64) during the next step's S = Q K^T
  load_rows<DK>(sQ, a.qr + ubase, C, q0, AT_TILE, len, threadIdx.x, 128);
  load_rows<DK>(sK, a.kr + ubase, C, 0, AT_TILE, len, threadIdx.x, 128);
  cp_async_commit();
  load_rows<DK>(sV, a.vr + ubase, C, 0, AT_TILE, len, threadIdx.x, 128);
  cp_async_commit();
  float o[NT][4];
#pragma unroll
  for (int n = 0; n < NT; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  const unsigned long long row_e[2] = {((unsigned long long)bh * L + rows[0]) * L, ((unsigned long long)bh * L + rows[1]) * L};
  for (int k0 = 0; k0 < len; k0 += AT_TILE) {
    cp_async_wait<1>();                                 // K(k0) (and Q) landed; V(k0) may still be in flight
    __syncthreads();
    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll 4
    for (int kk = 0; kk < NT; ++kk) {
      const float* qa = sQ + (16 * warp + g) * SS + 8 * kk + t;
      const uint32_t a0 = u(qa[0]), a1 = u(qa[8 * SS]), a2 = u(qa[4]), a3 = u(qa[8 * SS + 4]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float* kb = sK + (8 * j + g) * SS + 8 * kk + t;
        mma_tf32(s[j], a0, a1, a2, a3, u(kb[0]), u(kb[4]));
      }
    }
    __syncthreads();                                    // every warp is done with sK: prefetch the next K tile
    if (k0 + AT_TILE < len) load_rows<DK>(sK, a.kr + ubase, C, k0 + AT_TILE, AT_TILE, len, threadIdx.x, 128);
    cp_async_commit();
    // mask and scale, tile row maxima
    float mt[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = k0 + 8 * j + 2 * t + (e & 1), h = e >> 1;
        const float v = (key < len && rows[h] < len) ? s[j][e] * a.sl2 : -INFINITY;
        s[j][e] = v;
        mt[h] = fmaxf(mt[h], v);
      }
    float alpha[2], mu[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mt[h] = fmaxf(mt[h], __shfl_xor_sync(0xffffffffu, mt[h], 1));
      mt[h] = fmaxf(mt[h], __shfl_xor_sync(0xffffffffu, mt[h], 2));
      const float mn = fmaxf(m[h], mt[h]);
      mu[h] = mn == -INFINITY ? 0.f : mn;
      alpha[h] = exp2f(m[h] - mu[h]);
      m[h] = mn;
      l[h] *= alpha[h];
    }
#pragma unroll
    for (int n = 0; n < NT; ++n) { o[n][0] *= alpha[0]; o[n][1] *= alpha[0]; o[n][2] *= alpha[1]; o[n][3] *= alpha[1]; }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      unsigned kb = 0xFu;
      if (a.drop.on) kb = keep_frag(a.drop, row_e, rows, k0 + 8 * j + 4 * (t >> 1), t, len);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float p = exp2f(s[j][e] - mu[e >> 1]);
        l[e >> 1] += p;
        const int bit = (e >> 1) * 2 + (e & 1);
        s[j][e] = __uint_as_float(to_tf32(a.drop.on ? (((kb >> bit) & 1) ? p * a.drop.keep_scale : 0.f) : p));
      }
    }
    cp_async_wait<1>();                                 // V(k0) landed; K(k0 + 64) may still be in flight
    __syncthreads();
    // O += Pd . V: A column t <-> key 2t, t + 4 <-> key 2t + 1
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t a0 = u(s[j][0]), a1 = u(s[j][2]), a2 = u(s[j][1]), a3 = u(s[j][3]);
      const float* vb = sV + (8 * j + 2 * t) * SS + g;
#pragma unroll
      for (int n = 0; n < NT; ++n) mma_tf32(o[n], a0, a1, a2, a3, u(vb[8 * n]), u(vb[SS + 8 * n]));
    }
    __syncthreads();                                    // every warp is done with sV: prefetch the next V tile
    if (k0 + AT_TILE < len) load_rows<DK>(sV, a.vr + ubase, C, k0 + AT_TILE, AT_TILE, len, threadIdx.x, 128);
    cp_async_commit();
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
    const int r = rows[h];
    if (r >= L) continue;
    const bool valid = r < len;
    const float inv = valid ? 1.0f / l[h] : 0.f;
    float* orow = out + (long)r * C + 2 * t;
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      orow[8 * n] = valid ? o[n][2 * h] * inv : 0.f;
      orow[8 * n + 1] = valid ? o[n][2 * h + 1] * inv : 0.f;
    }
    if (t == 0) lse[r] = valid ? (m[h] + log2f(l[h])) * AT_LN2 : 0.f;
  }
}

// ---- D = rowsum(dO o O), 0 past len: one warp per row --------------------------------------------------------------------
__global__ void __launch_bounds__(256) attn_delta_kernel(const AttnParams a, int dk, long rows_total) {
  const long row = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows_total) return;
  const int lane = threadIdx.x & 31;
  const long bh = row / a.L;
  const int i = (int)(row - bh * a.L), b = (int)(bh / a.heads), hd = (int)(bh - (long)b * a.heads);
  float s = 0.f;
  if (i < clamp_len(a.lens, b, a.L)) {
    const long off = ((long)b * a.L + i) * a.C + (long)hd * dk;
    for (int d = lane; d < dk; d += 32) s += a.dout[off + d] * a.o[off + d];
    s = warp_sum(s);
  }
  if (lane == 0) a.dvec[row] = s;
}

// ---- dK, dV ---------------------------------------------------------------------------------------------------------------------
template <int DK>
__global__ void __launch_bounds__(256, 1) attn_dkdv_kernel(const AttnParams a) {
  extern __shared__ float4 smem4[];
  constexpr int SS = DK + 4, NT = DK / 8;
  float* sK = reinterpret_cast<float*>(smem4);
  float* sV = sK + AT_TILE * SS;
  float* sQ2 = sV + AT_TILE * SS;                      // two stages of [Q rows | dO rows]
  float* sP = sQ2 + 4 * AT_QSTEP * SS;                 // Pd^T [64 keys][AT_PS]
  float* sS = sP + AT_TILE * AT_PS;                    // dS^T
  float* sL = sS + AT_TILE * AT_PS;                    // lse * log2(e) of the step's queries
  float* sD = sL + AT_QSTEP;
  const int bh = blockIdx.x, b = bh / a.heads, hd = bh - b * a.heads;
  const int L = a.L, C = a.C, k0 = blockIdx.y * AT_TILE;
  const int len = clamp_len(a.lens, b, L);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int kg = warp & 3, qh = warp >> 2;
  const long ubase = (long)b * L * C + (long)hd * DK;
  float* dst = (qh ? a.dk : a.dv) + ubase;
  if (k0 >= len) {
    for (int i = threadIdx.x; i < AT_TILE * DK; i += 256) {
      const int r = k0 + i / DK;
      if (r < L) { a.dk[ubase + (long)r * C + i % DK] = 0.f; a.dv[ubase + (long)r * C + i % DK] = 0.f; }
    }
    return;
  }
  // the Q / dO rows of query step n + 1 load into the other stage while step n computes
  load_rows<DK>(sK, a.kr + ubase, C, k0, AT_TILE, len, threadIdx.x, 256);
  load_rows<DK>(sV, a.vr + ubase, C, k0, AT_TILE, len, threadIdx.x, 256);
  load_rows<DK>(sQ2, a.qr + ubase, C, 0, AT_QSTEP, len, threadIdx.x, 256);
  load_rows<DK>(sQ2 + AT_QSTEP * SS, a.dor + ubase, C, 0, AT_QSTEP, len, threadIdx.x, 256);
  cp_async_commit();
  float acc[NT][4];
#pragma unroll
  for (int n = 0; n < NT; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;
  const int keys[2] = {k0 + 16 * kg + g, k0 + 16 * kg + g + 8};
  const float* lse = a.lse + (long)bh * L;
  const float* dvec = a.dvec + (long)bh * L;
  for (int i0 = 0, stage = 0; i0 < len; i0 += AT_QSTEP, stage ^= 1) {
    const float* sQ = sQ2 + stage * 2 * AT_QSTEP * SS;
    const float* sO = sQ + AT_QSTEP * SS;
    __syncthreads();                                   // the previous step's reads of the other stage, sP / sS, sL / sD are done
    if (i0 + AT_QSTEP < len) {
      float* nQ = sQ2 + (stage ^ 1) * 2 * AT_QSTEP * SS;
      load_rows<DK>(nQ, a.qr + ubase, C, i0 + AT_QSTEP, AT_QSTEP, len, threadIdx.x, 256);
      load_rows<DK>(nQ + AT_QSTEP * SS, a.dor + ubase, C, i0 + AT_QSTEP, AT_QSTEP, len, threadIdx.x, 256);
    }
    cp_async_commit();
    if (threadIdx.x < AT_QSTEP) {
      const int qi = i0 + threadIdx.x;
      sL[threadIdx.x] = qi < len ? lse[qi] * AT_LOG2E : 0.f;
      sD[threadIdx.x] = qi < len ? dvec[qi] : 0.f;
    }
    cp_async_wait<1>();                                // this step's stage landed; the next one may be in flight
    __syncthreads();
    // S^T and dPd^T for keys 16 kg.., queries 16 qh..
    float st[2][4], dp[2][4];
#pragma unroll
    for (int j = 0; j < 2; ++j) st[j][0] = st[j][1] = st[j][2] = st[j][3] = dp[j][0] = dp[j][1] = dp[j][2] = dp[j][3] = 0.f;
#pragma unroll 4
    for (int kk = 0; kk < NT; ++kk) {
      const float* ka = sK + (16 * kg + g) * SS + 8 * kk + t;
      const float* va = sV + (16 * kg + g) * SS + 8 * kk + t;
      const uint32_t k_0 = u(ka[0]), k_1 = u(ka[8 * SS]), k_2 = u(ka[4]), k_3 = u(ka[8 * SS + 4]);
      const uint32_t v_0 = u(va[0]), v_1 = u(va[8 * SS]), v_2 = u(va[4]), v_3 = u(va[8 * SS + 4]);
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const float* qb = sQ + (16 * qh + 8 * j + g) * SS + 8 * kk + t;
        const float* ob = sO + (16 * qh + 8 * j + g) * SS + 8 * kk + t;
        mma_tf32(st[j], k_0, k_1, k_2, k_3, u(qb[0]), u(qb[4]));
        mma_tf32(dp[j], v_0, v_1, v_2, v_3, u(ob[0]), u(ob[4]));
      }
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      unsigned kb = 0xFu;
      if (a.drop.on) kb = keep_frag_t(a.drop, (unsigned long long)bh * L, i0 + 16 * qh + 8 * j, k0 + 16 * kg + 4 * (g >> 2), lane, len);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int ql = 16 * qh + 8 * j + 2 * t + (e & 1), qi = i0 + ql, key = keys[e >> 1];
        const bool valid = qi < len && key < len;
        const float p = valid ? exp2f(st[j][e] * a.sl2 - sL[ql]) : 0.f;
        float pd = p, g_ = dp[j][e];
        if (a.drop.on) {
          const bool keep = valid && ((kb >> ((e >> 1) * 2 + (e & 1))) & 1);
          pd = keep ? p * a.drop.keep_scale : 0.f;
          g_ = keep ? g_ * a.drop.keep_scale : 0.f;
        }
        const int at = (16 * kg + g + 8 * (e >> 1)) * AT_PS + ql;
        sP[at] = __uint_as_float(to_tf32(pd));
        sS[at] = __uint_as_float(to_tf32(p * (g_ - sD[ql])));
      }
    }
    __syncthreads();
    // qh = 0: dV += Pd^T . dO;  qh = 1: dK += dS^T . Q   (16 keys x DK, over the step's 32 queries)
    const float* A = (qh ? sS : sP) + (16 * kg + g) * AT_PS + t;
    const float* Bm = (qh ? sQ : sO) + t * SS + g;
#pragma unroll
    for (int kq = 0; kq < AT_QSTEP / 8; ++kq) {
      const uint32_t a0 = u(A[8 * kq]), a1 = u(A[8 * AT_PS + 8 * kq]), a2 = u(A[8 * kq + 4]), a3 = u(A[8 * AT_PS + 8 * kq + 4]);
      const float* bb = Bm + 8 * kq * SS;
#pragma unroll
      for (int n = 0; n < NT; ++n) mma_tf32(acc[n], a0, a1, a2, a3, u(bb[8 * n]), u(bb[4 * SS + 8 * n]));
    }
  }
  const float mult = qh ? a.scale : 1.f;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = keys[h];
    if (r >= L) continue;
    const bool valid = r < len;
    float* row = dst + (long)r * C + 2 * t;
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      row[8 * n] = valid ? acc[n][2 * h] * mult : 0.f;
      row[8 * n + 1] = valid ? acc[n][2 * h + 1] * mult : 0.f;
    }
  }
}

// ---- dQ -------------------------------------------------------------------------------------------------------------------------
template <int DK>
__global__ void __launch_bounds__(128, 1) attn_dq_kernel(const AttnParams a) {
  extern __shared__ float4 smem4[];
  constexpr int SS = DK + 4, NT = DK / 8;
  float* sQ = reinterpret_cast<float*>(smem4);
  float* sO = sQ + AT_TILE * SS;
  float* sK = sO + AT_TILE * SS;
  float* sV = sK + AT_TILE * SS;
  const int bh = blockIdx.x, b = bh / a.heads, hd = bh - b * a.heads;
  const int L = a.L, C = a.C, q0 = blockIdx.y * AT_TILE;
  const int len = clamp_len(a.lens, b, L);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const long ubase = (long)b * L * C + (long)hd * DK;
  float* dq = a.dq + ubase;
  const int rows[2] = {q0 + 16 * warp + g, q0 + 16 * warp + g + 8};
  if (q0 >= len) {
    for (int i = threadIdx.x; i < AT_TILE * DK; i += 128) {
      const int r = q0 + i / DK;
      if (r < L) dq[(long)r * C + i % DK] = 0.f;
    }
    return;
  }
  // V and K tiles are separate cp.async groups: V(k0 + 64) loads during S and dQ += dS K of step k0, K(k0 + 64)
  // during the next step's dP = dO V^T
  load_rows<DK>(sQ, a.qr + ubase, C, q0, AT_TILE, len, threadIdx.x, 128);
  load_rows<DK>(sO, a.dor + ubase, C, q0, AT_TILE, len, threadIdx.x, 128);
  load_rows<DK>(sV, a.vr + ubase, C, 0, AT_TILE, len, threadIdx.x, 128);
  cp_async_commit();
  load_rows<DK>(sK, a.kr + ubase, C, 0, AT_TILE, len, threadIdx.x, 128);
  cp_async_commit();
  float lse2[2], dr[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const bool valid = rows[h] < len;
    lse2[h] = valid ? a.lse[(long)bh * L + rows[h]] * AT_LOG2E : 0.f;
    dr[h] = valid ? a.dvec[(long)bh * L + rows[h]] : 0.f;
  }
  const unsigned long long row_e[2] = {((unsigned long long)bh * L + rows[0]) * L, ((unsigned long long)bh * L + rows[1]) * L};
  float acc[NT][4];
#pragma unroll
  for (int n = 0; n < NT; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f;
  for (int k0 = 0; k0 < len; k0 += AT_TILE) {
    cp_async_wait<1>();                                 // V(k0) (and Q, dO) landed; K(k0) may still be in flight
    __syncthreads();
    float s[8][4], dp[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = dp[j][0] = dp[j][1] = dp[j][2] = dp[j][3] = 0.f;
#pragma unroll 2
    for (int kk = 0; kk < NT; ++kk) {
      const float* oa = sO + (16 * warp + g) * SS + 8 * kk + t;
      const uint32_t o_0 = u(oa[0]), o_1 = u(oa[8 * SS]), o_2 = u(oa[4]), o_3 = u(oa[8 * SS + 4]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float* vb = sV + (8 * j + g) * SS + 8 * kk + t;
        mma_tf32(dp[j], o_0, o_1, o_2, o_3, u(vb[0]), u(vb[4]));
      }
    }
    __syncthreads();                                    // every warp is done with sV: prefetch the next V tile
    if (k0 + AT_TILE < len) load_rows<DK>(sV, a.vr + ubase, C, k0 + AT_TILE, AT_TILE, len, threadIdx.x, 128);
    cp_async_commit();
    cp_async_wait<1>();                                 // K(k0) landed; V(k0 + 64) may still be in flight
    __syncthreads();
#pragma unroll 2
    for (int kk = 0; kk < NT; ++kk) {
      const float* qa = sQ + (16 * warp + g) * SS + 8 * kk + t;
      const uint32_t q_0 = u(qa[0]), q_1 = u(qa[8 * SS]), q_2 = u(qa[4]), q_3 = u(qa[8 * SS + 4]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float* kb = sK + (8 * j + g) * SS + 8 * kk + t;
        mma_tf32(s[j], q_0, q_1, q_2, q_3, u(kb[0]), u(kb[4]));
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      unsigned kb = 0xFu;
      if (a.drop.on) kb = keep_frag(a.drop, row_e, rows, k0 + 8 * j + 4 * (t >> 1), t, len);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = k0 + 8 * j + 2 * t + (e & 1), h = e >> 1;
        const bool valid = key < len && rows[h] < len;
        const float p = valid ? exp2f(s[j][e] * a.sl2 - lse2[h]) : 0.f;
        float g_ = dp[j][e];
        if (a.drop.on) g_ = ((kb >> (2 * h + (e & 1))) & 1) ? g_ * a.drop.keep_scale : 0.f;
        s[j][e] = __uint_as_float(to_tf32(p * (g_ - dr[h])));
      }
    }
    // dQ += dS . K, A column t <-> key 2t, t + 4 <-> key 2t + 1
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t a0 = u(s[j][0]), a1 = u(s[j][2]), a2 = u(s[j][1]), a3 = u(s[j][3]);
      const float* kb = sK + (8 * j + 2 * t) * SS + g;
#pragma unroll
      for (int n = 0; n < NT; ++n) mma_tf32(acc[n], a0, a1, a2, a3, u(kb[8 * n]), u(kb[SS + 8 * n]));
    }
    __syncthreads();                                    // every warp is done with sK: prefetch the next K tile
    if (k0 + AT_TILE < len) load_rows<DK>(sK, a.kr + ubase, C, k0 + AT_TILE, AT_TILE, len, threadIdx.x, 128);
    cp_async_commit();
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = rows[h];
    if (r >= L) continue;
    const bool valid = r < len;
    float* row = dq + (long)r * C + 2 * t;
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      row[8 * n] = valid ? acc[n][2 * h] * a.scale : 0.f;
      row[8 * n + 1] = valid ? acc[n][2 * h + 1] * a.scale : 0.f;
    }
  }
}

template <int DK>
struct AttnSmem {
  static constexpr size_t FWD = (size_t)3 * AT_TILE * (DK + 4) * 4;
  static constexpr size_t DQ = (size_t)4 * AT_TILE * (DK + 4) * 4;
  static constexpr size_t DKDV = ((size_t)(2 * AT_TILE + 4 * AT_QSTEP) * (DK + 4) + 2 * AT_TILE * AT_PS + 2 * AT_QSTEP) * 4;
};

struct AttnPlan {
  int dk, tiles;
  size_t plane, dvec_off, bytes;   // rounded copies at k * plane (k = 0..3: q, k, v, dO), D at dvec_off
};

int attn_plan(int B, int L, int C, int heads, AttnPlan* pl, const char* who) {
  FS2_REQUIRE(B >= 1 && L >= 1 && C >= 1 && heads >= 1, "%s: need B, L, C, heads >= 1", who);
  FS2_REQUIRE(C % heads == 0, "%s: C = %d is not divisible by heads = %d", who, C, heads);
  const int dk = C / heads;
  FS2_REQUIRE(dk == 128 || dk == 192, "%s: head width %d is not supported (128 or 192)", who, dk);
  uint64_t n, bhl, bhll;
  const bool ok = !__builtin_mul_overflow((uint64_t)B * (uint64_t)L, (uint64_t)C * 4, &n) &&
                  !__builtin_mul_overflow((uint64_t)B * (uint64_t)heads, (uint64_t)L * 4, &bhl) &&
                  !__builtin_mul_overflow((uint64_t)B * (uint64_t)heads * (uint64_t)L, (uint64_t)L, &bhll) &&
                  n < (1ull << 56) && bhll < (1ull << 62) && (uint64_t)B * heads < (1ull << 31);
  FS2_REQUIRE(ok, "%s: size too large", who);
  pl->dk = dk;
  pl->tiles = (L + AT_TILE - 1) / AT_TILE;
  FS2_REQUIRE(pl->tiles <= 65535, "%s: L = %d is too large", who, L);
  pl->plane = align256(n);
  pl->dvec_off = 4 * pl->plane;
  pl->bytes = pl->dvec_off + align256(bhl);
  return FS2_OK;
}

int attn_common(const AttnPlan& pl, float p_drop, const void* ws, size_t ws_bytes, const char* who) {
  FS2_REQUIRE(p_drop >= 0.f && p_drop < 1.f, "%s: p_drop must be in [0, 1)", who);
  FS2_REQUIRE(ws && (reinterpret_cast<uintptr_t>(ws) & 15) == 0, "%s: workspace missing or not 16-byte aligned", who);
  FS2_REQUIRE(ws_bytes >= pl.bytes, "%s: workspace of %zu bytes, %zu needed", who, ws_bytes, pl.bytes);
  return FS2_OK;
}

AttnParams make_params(const AttnPlan& pl, const int64_t* lens, int L, int C, int heads, float p_drop, const uint8_t* dmask, uint64_t seed,
                       uint64_t offset, void* ws) {
  AttnParams a = {};
  float* w = reinterpret_cast<float*>(ws);
  const size_t pf = pl.plane / 4;
  a.qr = w; a.kr = w + pf; a.vr = w + 2 * pf; a.dor = w + 3 * pf;
  a.dvec = w + pl.dvec_off / 4;
  a.lens = lens; a.L = L; a.C = C; a.heads = heads;
  a.scale = 1.0f / sqrtf((float)pl.dk);
  a.sl2 = AT_LOG2E / sqrtf((float)pl.dk);
  a.drop.mask = dmask; a.drop.seed = seed; a.drop.offset = offset; a.drop.p = p_drop;
  a.drop.keep_scale = 1.0f / (1.0f - p_drop);
  a.drop.on = p_drop > 0.f;
  a.drop.L = L;
  return a;
}

int round_rows(const float* in, const int64_t* lens, int B, int L, int C, float* out, cudaStream_t st) {
  const long n = (long)B * L * C;
  attn_round_kernel<<<grid_for(n, 256, 132 * 16), 256, 0, st>>>(in, lens, L, C, n, out);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

template <int DK>
int launch_forward(const AttnParams& a, int BH, int tiles, cudaStream_t st) {
  static unsigned long long configured = 0;
  int rc;
  if ((rc = tc::ensure_smem_attr(attn_fwd_kernel<DK>, AttnSmem<DK>::FWD, &configured))) return rc;
  attn_fwd_kernel<DK><<<dim3(BH, tiles), 128, AttnSmem<DK>::FWD, st>>>(a);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

template <int DK>
int launch_backward(const AttnParams& a, int BH, int tiles, cudaStream_t st) {
  static unsigned long long conf_kv = 0, conf_q = 0;
  int rc;
  if ((rc = tc::ensure_smem_attr(attn_dkdv_kernel<DK>, AttnSmem<DK>::DKDV, &conf_kv))) return rc;
  if ((rc = tc::ensure_smem_attr(attn_dq_kernel<DK>, AttnSmem<DK>::DQ, &conf_q))) return rc;
  attn_dkdv_kernel<DK><<<dim3(BH, tiles), 256, AttnSmem<DK>::DKDV, st>>>(a);
  FS2_LAUNCH_CHECK();
  attn_dq_kernel<DK><<<dim3(BH, tiles), 128, AttnSmem<DK>::DQ, st>>>(a);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace
}  // namespace fs2

using namespace fs2;

extern "C" {

int fs2_attn_train_ws_bytes(int B, int L, int C, int heads, size_t* bytes) {
  FS2_REQUIRE(bytes, "fs2_attn_train_ws_bytes: null argument");
  AttnPlan pl;
  int rc = attn_plan(B, L, C, heads, &pl, "fs2_attn_train_ws_bytes");
  if (rc) return rc;
  *bytes = pl.bytes;
  return FS2_OK;
}

int fs2_attn_train_forward(const float* q, const float* k, const float* v, const int64_t* lens, int B, int L, int C, int heads, float p_drop,
                           const uint8_t* dmask, uint64_t seed, uint64_t offset, float* out, float* lse, void* ws, size_t ws_bytes,
                           void* stream) {
  FS2_REQUIRE(q && k && v && lens && out && lse, "fs2_attn_train_forward: null argument");
  AttnPlan pl;
  int rc = attn_plan(B, L, C, heads, &pl, "fs2_attn_train_forward");
  if (rc || (rc = attn_common(pl, p_drop, ws, ws_bytes, "fs2_attn_train_forward"))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  AttnParams a = make_params(pl, lens, L, C, heads, p_drop, dmask, seed, offset, ws);
  a.out = out; a.lse_out = lse;
  if ((rc = round_rows(q, lens, B, L, C, const_cast<float*>(a.qr), st)) || (rc = round_rows(k, lens, B, L, C, const_cast<float*>(a.kr), st)) ||
      (rc = round_rows(v, lens, B, L, C, const_cast<float*>(a.vr), st)))
    return rc;
  return pl.dk == 128 ? launch_forward<128>(a, B * heads, pl.tiles, st) : launch_forward<192>(a, B * heads, pl.tiles, st);
}

int fs2_attn_train_backward(const float* q, const float* k, const float* v, const float* out, const float* lse, const float* dout,
                            const int64_t* lens, int B, int L, int C, int heads, float p_drop, const uint8_t* dmask, uint64_t seed,
                            uint64_t offset, float* dq, float* dk, float* dv, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(q && k && v && out && lse && dout && lens && dq && dk && dv, "fs2_attn_train_backward: null argument");
  AttnPlan pl;
  int rc = attn_plan(B, L, C, heads, &pl, "fs2_attn_train_backward");
  if (rc || (rc = attn_common(pl, p_drop, ws, ws_bytes, "fs2_attn_train_backward"))) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  AttnParams a = make_params(pl, lens, L, C, heads, p_drop, dmask, seed, offset, ws);
  a.o = out; a.dout = dout; a.lse = lse;
  a.dq = dq; a.dk = dk; a.dv = dv;
  if ((rc = round_rows(q, lens, B, L, C, const_cast<float*>(a.qr), st)) || (rc = round_rows(k, lens, B, L, C, const_cast<float*>(a.kr), st)) ||
      (rc = round_rows(v, lens, B, L, C, const_cast<float*>(a.vr), st)) || (rc = round_rows(dout, lens, B, L, C, const_cast<float*>(a.dor), st)))
    return rc;
  const long rows = (long)B * heads * L;
  attn_delta_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(a, pl.dk, rows);
  FS2_LAUNCH_CHECK();
  return pl.dk == 128 ? launch_backward<128>(a, B * heads, pl.tiles, st) : launch_backward<192>(a, B * heads, pl.tiles, st);
}

}  // extern "C"
