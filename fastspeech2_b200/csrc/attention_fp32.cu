// Exact-fp32 multi-head self-attention core (core/attention.py:52-73): streaming-softmax
// ("flash") formulation so the [B,h,L,L] score tensor the reference materialises (328 MB per
// decoder layer at B=64, L=800) never exists.
//
//   S = (q k^T) / sqrt(d_k);  S[:, u] = -inf for u >= len_b;  P = softmax_u(S);
//   P[t, :] = 0 for t >= len_b (the reference's second masked_fill turns those NaN rows into 0);
//   ctx = P v.    lens == nullptr reproduces the mask=None branch (attention.py:67).
//
// q, k, v live in one fused projection buffer qkv [B, L, 3C] (q | k | v, head h at columns
// h*d_k inside each third); ctx is written [B, L, C] with heads concatenated (attention.py:71-73).
//
// CTA = 64 queries x one (batch, head); 256 threads as a 16x16 grid.  Per 64-key tile:
// S (64x64) from shared-memory Q/K tiles with LDS.128 along d, online max/sum with 16-lane
// shuffles, P staged in shared memory, O (64 x d_k) accumulated in registers.
// Used for the encoder in every mode and for the decoder in FS2_MATH_FP32.
#include <math.h>

#include "tc_common.cuh"   // ensure_smem_attr

namespace fs2 {
namespace {

constexpr int BQ = 64, BKV = 64;

template <int DK>
struct AttnSmem {
  static constexpr int LDQ = DK + 4;  // float4-aligned rows, conflict-free for row-per-lane LDS.128
  static constexpr int LDP = BKV + 4;
  static constexpr size_t bytes = (size_t)(BQ * LDQ + BKV * LDQ + BKV * DK + BQ * LDP) * sizeof(float);
};

template <int DK>
__global__ void __launch_bounds__(256, 1)
attention_fp32_kernel(const float* __restrict__ qkv, const int64_t* __restrict__ lens, int L, int C,
                      float* __restrict__ ctx, float scale) {
  extern __shared__ __align__(16) float smem[];
  constexpr int LDQ = AttnSmem<DK>::LDQ, LDP = AttnSmem<DK>::LDP;
  float* Qs = smem;                  // [BQ][LDQ]
  float* Ks = Qs + BQ * LDQ;         // [BKV][LDQ]
  float* Vs = Ks + BKV * LDQ;        // [BKV][DK]
  float* Ps = Vs + BKV * DK;         // [BQ][LDP]

  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * BQ;
  const int ld = 3 * C;
  const float* base = qkv + (long)b * L * ld;
  const int len = lens ? (int)min((long)lens[b], (long)L) : L;  // keys >= len are masked
  constexpr int VPR = DK / 4;  // float4 per row

  // Q tile (rows beyond L are zero)
  for (int v = tid; v < BQ * VPR; v += 256) {
    int r = v / VPR, c = (v - r * VPR) * 4;
    float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q0 + r < L) val = __ldg(reinterpret_cast<const float4*>(base + (long)(q0 + r) * ld + h * DK + c));
    *reinterpret_cast<float4*>(&Qs[r * LDQ + c]) = val;
  }

  constexpr int NO = DK / 64;  // float4 output groups per thread: cols 4*tx + 64*g
  float4 o[4][NO];
  float m_run[4], l_run[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m_run[i] = -INFINITY; l_run[i] = 0.f;
#pragma unroll
    for (int g = 0; g < NO; ++g) o[i][g] = make_float4(0.f, 0.f, 0.f, 0.f);
  }

  for (int k0 = 0; k0 < len; k0 += BKV) {
    __syncthreads();  // previous tile fully consumed (also orders the Q stores on the first trip)
    for (int v = tid; v < BKV * VPR; v += 256) {
      int r = v / VPR, c = (v - r * VPR) * 4;
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
      if (k0 + r < len) {
        const float* p = base + (long)(k0 + r) * ld + h * DK + c;
        kv = __ldg(reinterpret_cast<const float4*>(p + C));
        vv = __ldg(reinterpret_cast<const float4*>(p + 2 * C));
      }
      *reinterpret_cast<float4*>(&Ks[r * LDQ + c]) = kv;
      *reinterpret_cast<float4*>(&Vs[r * DK + c]) = vv;
    }
    __syncthreads();

    // S[i][j] for rows ty + 16 i, cols tx + 16 j
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll 4
    for (int d = 0; d < DK; d += 4) {
      float4 qv[4], kv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) qv[i] = *reinterpret_cast<const float4*>(&Qs[(ty + 16 * i) * LDQ + d]);
#pragma unroll
      for (int j = 0; j < 4; ++j) kv[j] = *reinterpret_cast<const float4*>(&Ks[(tx + 16 * j) * LDQ + d]);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          s[i][j] = fmaf(qv[i].x, kv[j].x, s[i][j]); s[i][j] = fmaf(qv[i].y, kv[j].y, s[i][j]);
          s[i][j] = fmaf(qv[i].z, kv[j].z, s[i][j]); s[i][j] = fmaf(qv[i].w, kv[j].w, s[i][j]);
        }
    }
    // scale, mask, online softmax (row statistics shared by the 16 lanes with equal ty)
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        bool ok = (k0 + tx + 16 * j) < len;
        s[i][j] = ok ? s[i][j] * scale : -INFINITY;
        mx = fmaxf(mx, s[i][j]);
      }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
      float m_new = fmaxf(m_run[i], mx);          // finite: every tile has >= 1 valid key
      float corr = expf(m_run[i] - m_new);        // exp(-inf) = 0 on the first tile
      float rs = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float p = expf(s[i][j] - m_new);          // masked -> exp(-inf) = 0
        rs += p;
        Ps[(ty + 16 * i) * LDP + tx + 16 * j] = p;
      }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, off);
      l_run[i] = l_run[i] * corr + rs;
      m_run[i] = m_new;
#pragma unroll
      for (int g = 0; g < NO; ++g) { o[i][g].x *= corr; o[i][g].y *= corr; o[i][g].z *= corr; o[i][g].w *= corr; }
    }
    __syncthreads();
    // O += P V
#pragma unroll 2
    for (int c = 0; c < BKV; c += 4) {
      float4 pv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) pv[i] = *reinterpret_cast<const float4*>(&Ps[(ty + 16 * i) * LDP + c]);
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) {
#pragma unroll
        for (int g = 0; g < NO; ++g) {
          float4 vv = *reinterpret_cast<const float4*>(&Vs[(c + cc) * DK + 4 * tx + 64 * g]);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            float p = cc == 0 ? pv[i].x : cc == 1 ? pv[i].y : cc == 2 ? pv[i].z : pv[i].w;
            o[i][g].x = fmaf(p, vv.x, o[i][g].x); o[i][g].y = fmaf(p, vv.y, o[i][g].y);
            o[i][g].z = fmaf(p, vv.z, o[i][g].z); o[i][g].w = fmaf(p, vv.w, o[i][g].w);
          }
        }
      }
    }
  }

  // normalise and store; masked query rows (t >= len) are exactly 0 (attention.py:63-65)
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int t = q0 + ty + 16 * i;
    if (t >= L) continue;
    bool zero = (lens && t >= len) || l_run[i] == 0.f;
    float inv = zero ? 0.f : 1.0f / l_run[i];
#pragma unroll
    for (int g = 0; g < NO; ++g) {
      float4 r = make_float4(o[i][g].x * inv, o[i][g].y * inv, o[i][g].z * inv, o[i][g].w * inv);
      *reinterpret_cast<float4*>(ctx + ((long)b * L + t) * C + h * DK + 4 * tx + 64 * g) = r;
    }
  }
}

template <int DK>
int launch(const float* qkv, const int64_t* lens, int B, int L, int C, int heads, float* ctx, cudaStream_t st) {
  static unsigned long long configured = 0;   // per-device bit mask
  int rc;
  if ((rc = tc::ensure_smem_attr(attention_fp32_kernel<DK>, AttnSmem<DK>::bytes, &configured))) return rc;
  dim3 grid((L + BQ - 1) / BQ, heads, B);
  attention_fp32_kernel<DK><<<grid, 256, AttnSmem<DK>::bytes, st>>>(qkv, lens, L, C, ctx, 1.0f / sqrtf((float)DK));
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace

int attention_fp32(const float* qkv, const int64_t* lens, int B, int L, int C, int heads, float* ctx, cudaStream_t st) {
  FS2_REQUIRE(heads > 0 && C % heads == 0, "attention: C=%d not divisible by heads=%d", C, heads);
  if (B == 0 || L == 0) return FS2_OK;
  int dk = C / heads;
  if (dk == 128) return launch<128>(qkv, lens, B, L, C, heads, ctx, st);
  if (dk == 192) return launch<192>(qkv, lens, B, L, C, heads, ctx, st);
  set_error("attention_fp32: d_k=%d unsupported (128 or 192)", dk);
  return FS2_ERR_INVALID;
}

}  // namespace fs2
