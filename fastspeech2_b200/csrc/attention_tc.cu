// Tensor-core multi-head self-attention core (core/attention.py:52-73), two kernels:
//   attention_tc_kernel    (FS2_MATH_TF32): S = Q K^T and O = P V with tf32 operands (warp-level mma m16n8k8) on the
//                          fp32 q|k|v rows;
//   attention_wgmma_kernel (the operand-plane modes): warpgroup MMAs (wgmma) fed by TMA, either
//     F16 : fp16 operands on the hi planes (FS2_MATH_F16's decoder), or
//     X3  : the error-compensated form -- Q, K, V^T and P each as fp16 hi + lo, three products per term (lo.hi + hi.lo +
//           hi.hi), fp32 accumulation and softmax statistics: fp32-class scores and context (the encoder in every
//           tensor-core mode, the decoder in FS2_MATH_3XTF32).
// The [B,h,L,L] score tensor never touches HBM: S, P and O live in registers.
//
//   ctx[b,t,h*dk:(h+1)*dk] = softmax_u( q.k_u / sqrt(dk) | u < len_b ) . v ,  0 for t >= len_b
//   (lens == nullptr: no masking at all -- the reference's mask=None branch, attention.py:67)
//
// Operands:
//   TF32 : q, k rows of the fused projection buffer qkv [B, L, 3C]; V^T as vt [B*heads][dk][lpad] fp32
//   F16 / X3 : q|k planes qkp [P][B*L][2C] fp16, V^T planes vtp [P][B*heads][dk][lpad], all scaled by kPlaneScale
// V is stored transposed by the projection GEMM's epilogue (gemm_tc.cu), so that the B operand of P.V is contiguous along
// the keys just like K is along d_k.
//
// Both kernels walk the keys from 0 in tiles of 64 up to len, online softmax in the exp2 domain with the running maximum.
// A row's result therefore depends only on its utterance's len and on the q / k / v rows below len: not on L, the batch,
// the query tile or whether lens is given (the per-utterance contract, DESIGN.md section 5).  In F16 the row sum adds the
// *rounded* P values, so the weights the tensor core applies still sum to one.
#include <math.h>

#include "tc_common.cuh"

namespace fs2 {
namespace {
using namespace tc;

struct AParams {
  const void* q;   // TF32: qkv rows; else q|k planes
  const void* vt;  // TF32: vt fp32; else V^T planes
  int lpad;
  const int64_t* lens; int B, L, C, heads;
  float* ctx;      // [B,L,C] fp32 or null
  __half* ctxp;    // planes [P][B*L][C] or null (planes modes only)
  float scale_log2e;
};

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {   // a in the low half
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

__device__ __forceinline__ int utterance_len(const AParams& p, int b) {
  if (!p.lens) return p.L;
  const int64_t lb = p.lens[b];
  return lb < 0 ? 0 : (lb > p.L ? p.L : (int)lb);
}

// ---- tf32 -------------------------------------------------------------------------------------------------------
// CTA = 64 queries of one (batch, head), four warps of 16 query rows; 64 keys per step, K and V^T tiles staged in padded
// shared memory (row pitches chosen so that every fragment load is bank-conflict free).  The P fragments of S = Q K^T are,
// register for register, the A fragments of O += P V: the key order inside each 8-key slice is permuted to make that so
// (A column k <-> key 2k, k + 4 <-> key 2k + 1, and the V^T fragment follows the same order).
constexpr int BQ = 64, BKV = 64, ATT_THREADS = 128, PADE = 8;

template <int DK>
struct ACfg {
  static constexpr int LDQ = DK + PADE;                 // elements per Q / K row in shared memory
  static constexpr int LDV = BKV + PADE;                // elements per V^T row
  static constexpr size_t Q_ELEMS = (size_t)BQ * LDQ, K_ELEMS = (size_t)BKV * LDQ, V_ELEMS = (size_t)DK * LDV;
  static constexpr size_t SMEM = (Q_ELEMS + K_ELEMS + V_ELEMS) * sizeof(float);
};

// rows [r0, r0 + nrows) x cols [0, ncols) of a global matrix (row pitch ld elements) -> shared (pitch lds); rows >= valid
// and columns >= cvalid are zero (cvalid is a multiple of the vector width except at the very end of a row)
template <int NCOLS>
__device__ __forceinline__ void stage(float* __restrict__ dst, int lds, const float* __restrict__ src, long ld, int nrows, int rvalid, int cvalid) {
  constexpr int EPV = 4, VPR = NCOLS / EPV;
  for (int i = threadIdx.x; i < nrows * VPR; i += ATT_THREADS) {
    const int r = i / VPR, c = (i - r * VPR) * EPV;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r < rvalid) {
      if (c + EPV <= cvalid) {
        v = __ldg(reinterpret_cast<const uint4*>(src + (long)r * ld + c));
      } else if (c < cvalid) {
        float tmp[EPV];
#pragma unroll
        for (int e = 0; e < EPV; ++e) tmp[e] = c + e < cvalid ? src[(long)r * ld + c + e] : 0.f;
        v = *reinterpret_cast<const uint4*>(tmp);
      }
    }
    *reinterpret_cast<uint4*>(dst + r * lds + c) = v;
  }
}

template <int DK>
__global__ void __launch_bounds__(ATT_THREADS)
attention_tc_kernel(AParams p) {
  using A = ACfg<DK>;
  constexpr int LDQ = A::LDQ, LDV = A::LDV;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  float* Qs = reinterpret_cast<float*>(smem_raw);
  float* Ks = Qs + A::Q_ELEMS;
  float* Vs = Ks + A::K_ELEMS;

  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * BQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tq = lane & 3;
  const int L = p.L, C = p.C, dk = DK;
  pdl_wait();                                         // the lengths may come from the previous kernel
  const int len = utterance_len(p, b);

  // global views
  const long ldqk = 3L * C;
  const float* qg = reinterpret_cast<const float*>(p.q) + ((long)b * L) * ldqk + h * dk;
  const float* kg = qg + C;
  const float* vg = reinterpret_cast<const float*>(p.vt) + ((long)b * p.heads + h) * dk * (long)p.lpad;

  const int qvalid = min(BQ, max(len, 0) - q0);     // query rows of this CTA that produce output
  if (qvalid > 0) stage<DK>(Qs, LDQ, qg + (long)q0 * ldqk, ldqk, BQ, L - q0, DK);

  float o[DK / 8][4];
#pragma unroll
  for (int j = 0; j < DK / 8; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};
  const int kv_len = len;                             // keys u < len take part
  const float sl2 = p.scale_log2e;

  for (int k0 = 0; qvalid > 0 && k0 < kv_len; k0 += BKV) {
    const int kvalid = min(BKV, kv_len - k0);
    __syncthreads();                                  // previous tile fully consumed
    stage<DK>(Ks, LDQ, kg + (long)k0 * ldqk, ldqk, BKV, kvalid, DK);
    stage<BKV>(Vs, LDV, vg + k0, p.lpad, DK, DK, kvalid);
    __syncthreads();

    // ---- S = Q K^T for this warp's 16 rows x 64 keys ----
    float s[BKV / 8][4];
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
    const float* qw = Qs + (warp * 16) * LDQ;
#pragma unroll 4
    for (int kk = 0; kk < DK; kk += 8) {             // A column k <-> d = kk + 2k, k + 4 <-> kk + 2k + 1
      const float2 qa = *reinterpret_cast<const float2*>(qw + g * LDQ + kk + 2 * tq);
      const float2 qb = *reinterpret_cast<const float2*>(qw + (g + 8) * LDQ + kk + 2 * tq);
      const uint32_t a[4] = {to_tf32(qa.x), to_tf32(qb.x), to_tf32(qa.y), to_tf32(qb.y)};
#pragma unroll
      for (int n = 0; n < BKV / 8; ++n) {
        const float2 kb = *reinterpret_cast<const float2*>(Ks + (n * 8 + g) * LDQ + kk + 2 * tq);
        mma_tf32(s[n], a[0], a[1], a[2], a[3], to_tf32(kb.x), to_tf32(kb.y));
      }
    }

    // ---- online softmax (rows g and g + 8 of the warp; each row is spread over the 4 lanes of a quad) ----
    float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = n * 8 + 2 * tq + (e & 1);
        const float v = key < kvalid ? s[n][e] * sl2 : -INFINITY;
        s[n][e] = v;
        tmax[e >> 1] = fmaxf(tmax[e >> 1], v);
      }
    }
    float corr[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      tmax[r] = fmaxf(tmax[r], __shfl_xor_sync(0xffffffffu, tmax[r], 1));
      tmax[r] = fmaxf(tmax[r], __shfl_xor_sync(0xffffffffu, tmax[r], 2));
      const float mnew = fmaxf(mrow[r], tmax[r]);     // finite: every tile has at least one valid key
      corr[r] = exp2f(mrow[r] - mnew);
      mrow[r] = mnew;
      lrow[r] *= corr[r];
    }
#pragma unroll
    for (int j = 0; j < DK / 8; ++j) { o[j][0] *= corr[0]; o[j][1] *= corr[0]; o[j][2] *= corr[1]; o[j][3] *= corr[1]; }
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n) {
#pragma unroll
      for (int e = 0; e < 4; ++e) s[n][e] = exp2f(s[n][e] - mrow[e >> 1]);
    }

    // ---- O += P V, 8 keys per step: A column k <-> key 2k, k + 4 <-> key 2k + 1 ----
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n) {
      lrow[0] += s[n][0] + s[n][1]; lrow[1] += s[n][2] + s[n][3];
      const uint32_t a[4] = {to_tf32(s[n][0]), to_tf32(s[n][2]), to_tf32(s[n][1]), to_tf32(s[n][3])};
#pragma unroll
      for (int j = 0; j < DK / 8; ++j) {
        const float2 vb = *reinterpret_cast<const float2*>(Vs + (j * 8 + g) * LDV + n * 8 + 2 * tq);
        mma_tf32(o[j], a[0], a[1], a[2], a[3], to_tf32(vb.x), to_tf32(vb.y));
      }
    }
  }

  // ---- epilogue: O / l; rows past len are zero ----
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = lrow[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int t = q0 + warp * 16 + g + 8 * r;
    if (t >= L) continue;
    const bool valid = t < len;
    const float inv = valid && l > 0.f ? 1.f / l : 0.f;
    const long row = (long)b * L + t;
#pragma unroll
    for (int j = 0; j < DK / 8; ++j) {
      const long off = row * C + h * dk + j * 8 + 2 * tq;
      if (p.ctx) *reinterpret_cast<float2*>(p.ctx + off) = make_float2(o[j][2 * r] * inv, o[j][2 * r + 1] * inv);
    }
  }
  pdl_trigger();
}

// ---- operand planes: wgmma + TMA ---------------------------------------------------------------------------------
// CTA = 128 queries of one (batch, head), three warpgroups.  Warp 0 is the TMA producer: Q once, then per 64-key tile a
// K box and a V^T box into a ring of STAGES slots, K and V^T with their own full / empty mbarriers, so that K(j+1) loads
// while the consumers run softmax(j) and P.V(j), and V^T(j+1) while they run S(j+1).  Warpgroups 1 and 2 own 64 query
// rows each and are not synchronised with each other, so one's softmax overlaps the other's MMAs:
//   S = Q K^T  : wgmma m64n64k16, both operands in shared memory (128-byte swizzle, d_k / 64 atoms); X3: three products
//                per K step into one accumulator, small terms first (Q lo.K hi, Q hi.K lo, Q hi.K hi);
//   O += P V   : wgmma m64n{d_k}k16 with A = P from registers (the S accumulator packed to half2, tc_common.cuh) and
//                B = the V^T tile (d_k rows of 64 keys: K-major already); X3: P lo.V hi, P hi.V lo, P hi.V hi.
// Shared memory (d_k = 192, X3): Q 96 KB + one K stage 48 KB + one V^T stage 48 KB; the smaller variants get two stages.
// setmaxnreg moves registers from the producer warpgroup to the consumers (O alone is d_k / 2 registers per thread).
//
// Rows past len.  Per-utterance mode leaves q|k rows and V^T columns at and past len unwritten, and V^T columns in
// [L, lpad) are never written at all; TMA zero-fills only outside the tensor map.  Scores of keys >= len are *selected* to
// -inf (a NaN from a garbage K row does not survive), but P = 0 does not protect P.V from a NaN in V^T: in the last key
// tile, when it is partial, the producer zeroes the V^T columns >= len in shared memory before it releases the tile.
// Output rows in [len, L) are exact zeros; a consumer warpgroup whose rows all lie past len issues no MMA.
constexpr int FA_BQ = 128, FA_BKV = 64, FA_THREADS = 384;
constexpr int FA_PRODUCER_REGS = 40, FA_CONSUMER_REGS = 232;   // 128 * 40 + 256 * 232 <= 65536

template <int DK, bool X3>
struct FCfg {
  static constexpr int P = X3 ? 2 : 1;                        // operand planes
  static constexpr int ATOMS = DK / 64;                       // 128-byte swizzle atoms along d_k
  static constexpr int Q_ATOM = FA_BQ * 128, K_ATOM = FA_BKV * 128;   // bytes: [rows][64 halfs]
  static constexpr int Q_BYTES = P * ATOMS * Q_ATOM;          // [plane][atom][128 rows]
  static constexpr int K_BYTES = P * ATOMS * K_ATOM;          // one K stage: [plane][atom][64 keys]
  static constexpr int V_PLANE = DK * 128;                    // one V^T stage: [plane][d_k rows][64 keys]
  static constexpr int V_BYTES = P * V_PLANE;
  static constexpr int STAGE_BYTES = K_BYTES + V_BYTES;
  static constexpr int BUDGET = 227 * 1024 - 1024 /*align slack*/ - 256 /*barriers*/;
  static constexpr int FIT = (BUDGET - Q_BYTES) / STAGE_BYTES;
  static constexpr int STAGES = FIT > 2 ? 2 : FIT;
  static constexpr size_t SMEM = (size_t)Q_BYTES + (size_t)STAGES * STAGE_BYTES + 1024 + 256;
  static_assert(DK % 64 == 0 && DK <= 256, "d_k: whole swizzle atoms, one wgmma N");
  static_assert(STAGES >= 1, "resources");
};

template <int DK>
__device__ __forceinline__ void wgmma_pv(float* o, const uint32_t* a, uint64_t b) {
  if constexpr (DK == 192) wgmma_f16_rs_n192(o, a, b, 1); else wgmma_f16_rs_n128(o, a, b, 1);
}

template <int DK, bool X3>
__global__ void __launch_bounds__(FA_THREADS, 1)
attention_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                       const __grid_constant__ CUtensorMap tmap_v, AParams p) {
  using F = FCfg<DK, X3>;
  constexpr int P = F::P, ATOMS = F::ATOMS, S = F::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* qs = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // swizzle atoms need 1024-byte alignment
  uint8_t* ring = qs + F::Q_BYTES;                          // slot s: K at ring + s * STAGE_BYTES, V^T right after it
  uint64_t* q_full = reinterpret_cast<uint64_t*>(ring + (size_t)S * F::STAGE_BYTES);
  uint64_t* k_full = q_full + 1;
  uint64_t* k_empty = k_full + S;
  uint64_t* v_full = k_empty + S;
  uint64_t* v_empty = v_full + S;
  uint64_t* v_tail = v_empty + S;                           // the partial last V^T tile lands here first

  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * FA_BQ;
  const int warp = uniform_warp_idx(), lane = threadIdx.x & 31;
  pdl_wait();                                               // the lengths and operands may come from the previous kernel
  const int len = utterance_len(p, b);
  const int active = q0 >= len ? 0 : (q0 + 64 >= len ? 1 : 2);   // consumer warpgroups with a row below len

  if (threadIdx.x == 0) {
    const uint32_t consumers = 4 * (active > 0 ? active : 1);    // every warp of an active warpgroup releases a slot
    mbar_init(q_full, 1);
    for (int s = 0; s < S; ++s) {
      mbar_init(&k_full[s], 1); mbar_init(&k_empty[s], consumers);
      mbar_init(&v_full[s], 1); mbar_init(&v_empty[s], consumers);
    }
    mbar_init(v_tail, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<FA_PRODUCER_REGS>();
    if (warp != 0 || active == 0) { pdl_trigger(); return; }
    // ---- TMA producer (whole warp; one lane elected inside each asm) ----
    const uint32_t q_addr = smem_u32(qs), ring_addr = smem_u32(ring);
    const int kcol = p.C + h * DK, vrow = b * p.heads + h, vplane = p.B * p.heads;
    mbar_expect_tx_elect(smem_u32(q_full), F::Q_BYTES);
#pragma unroll
    for (int pl = 0; pl < P; ++pl)
#pragma unroll
      for (int a = 0; a < ATOMS; ++a)
        tma_load_3d_elect(q_addr + (pl * ATOMS + a) * F::Q_ATOM, &tmap_q, smem_u32(q_full), h * DK + a * 64, q0, b + pl * p.B);
    for (int j = 0, k0 = 0; k0 < len; ++j, k0 += FA_BKV) {
      const int s = j % S;
      const uint32_t parity = ((j / S) & 1) ^ 1;
      const uint32_t k_addr = ring_addr + (uint32_t)s * F::STAGE_BYTES, v_addr = k_addr + F::K_BYTES;
      const uint32_t kf = smem_u32(&k_full[s]);
      mbar_wait(&k_empty[s], parity);
      mbar_expect_tx_elect(kf, F::K_BYTES);
#pragma unroll
      for (int pl = 0; pl < P; ++pl)
#pragma unroll
        for (int a = 0; a < ATOMS; ++a)
          tma_load_3d_elect(k_addr + (pl * ATOMS + a) * F::K_ATOM, &tmap_k, kf, kcol + a * 64, k0, b + pl * p.B);
      const int kvalid = len - k0;
      const bool tail = kvalid < FA_BKV;
      const uint32_t vf = smem_u32(tail ? v_tail : &v_full[s]);
      mbar_wait(&v_empty[s], parity);
      mbar_expect_tx_elect(vf, F::V_BYTES);
#pragma unroll
      for (int pl = 0; pl < P; ++pl) tma_load_3d_elect(v_addr + pl * F::V_PLANE, &tmap_v, vf, k0, 0, vrow + pl * vplane);
      if (tail) {
        // zero keys >= len of every V^T row: 16-byte chunk c of row r holds keys 8c .. 8c + 7 at chunk c ^ (r % 8)
        mbar_wait(v_tail, 0);
        uint8_t* vt = ring + (size_t)s * F::STAGE_BYTES + F::K_BYTES;
        for (int i = lane; i < P * DK * 8; i += 32) {
          const int r = i >> 3, c = i & 7, keep = kvalid - 8 * c;
          if (keep >= 8) continue;
          uint4* q = reinterpret_cast<uint4*>(vt + r * 128 + ((c ^ (r & 7)) << 4));
          uint4 v = make_uint4(0, 0, 0, 0);
          if (keep > 0) {
            uint32_t w[4] = {q->x, q->y, q->z, q->w};
#pragma unroll
            for (int e = 0; e < 4; ++e) w[e] = 2 * e >= keep ? 0u : (2 * e + 1 >= keep ? (w[e] & 0xFFFFu) : w[e]);
            v = make_uint4(w[0], w[1], w[2], w[3]);
          }
          *q = v;
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) mbar_arrive(&v_full[s]);
      }
    }
    pdl_trigger();
    return;
  }

  // ---- consumers: warpgroup cg owns query rows q0 + 64 cg .. q0 + 64 cg + 63 ----
  setmaxnreg_inc<FA_CONSUMER_REGS>();
  const int cg = (warp >> 2) - 1, wq = warp & 3, g = lane >> 2, tq = lane & 3;
  float o[DK / 2];                                          // d[4 j + 2 r + {0,1}]: row r0 + 8 r, columns 8 j + 2 tq + {0,1}
#pragma unroll
  for (int i = 0; i < DK / 2; ++i) o[i] = 0.f;
  float mrow[2] = {-INFINITY, -INFINITY}, lrow[2] = {0.f, 0.f};
  const float sl2 = p.scale_log2e;

  if (cg < active) {
    const uint32_t q_addr = smem_u32(qs) + cg * (64 * 128), ring_addr = smem_u32(ring);
    mbar_wait(q_full, 0);
    for (int j = 0, k0 = 0; k0 < len; ++j, k0 += FA_BKV) {
      const int s = j % S;
      const uint32_t parity = (j / S) & 1;
      const uint32_t k_addr = ring_addr + (uint32_t)s * F::STAGE_BYTES, v_addr = k_addr + F::K_BYTES;

      // ---- S = Q K^T: 64 rows x 64 keys ----
      float sc[FA_BKV / 2];
      mbar_wait(&k_full[s], parity);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < DK / 16; ++kk) {                // +32 bytes along d_k inside the swizzle row = +2 in descriptor units
        const int a = kk >> 2, off = 2 * (kk & 3);
        const uint64_t qh = make_sw128_kmajor_desc(q_addr + a * F::Q_ATOM) + off;
        const uint64_t kh = make_sw128_kmajor_desc(k_addr + a * F::K_ATOM) + off;
        if constexpr (X3) {
          const uint64_t ql = make_sw128_kmajor_desc(q_addr + (ATOMS + a) * F::Q_ATOM) + off;
          const uint64_t kl = make_sw128_kmajor_desc(k_addr + (ATOMS + a) * F::K_ATOM) + off;
          wgmma_f16_n64(sc, ql, kh, kk != 0);
          wgmma_f16_n64(sc, qh, kl, 1);
          wgmma_f16_n64(sc, qh, kh, 1);
        } else {
          wgmma_f16_n64(sc, qh, kh, kk != 0);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      pin_regs<FA_BKV / 2>(sc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&k_empty[s]);

      // ---- online softmax: rows r0 (r = 0) and r0 + 8 (r = 1), each spread over the 4 lanes of a quad ----
      const int kvalid = len - k0;
      float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < FA_BKV / 2; ++i) {
        const int key = 8 * (i >> 2) + 2 * tq + (i & 1);
        const float v = key < kvalid ? sc[i] * sl2 : -INFINITY;
        sc[i] = v;
        tmax[(i >> 1) & 1] = fmaxf(tmax[(i >> 1) & 1], v);
      }
      float corr[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        tmax[r] = fmaxf(tmax[r], __shfl_xor_sync(0xffffffffu, tmax[r], 1));
        tmax[r] = fmaxf(tmax[r], __shfl_xor_sync(0xffffffffu, tmax[r], 2));
        const float mnew = fmaxf(mrow[r], tmax[r]);         // finite for a valid row: every tile has a key below len
        corr[r] = exp2f(mrow[r] - mnew);
        mrow[r] = mnew;
        lrow[r] *= corr[r];
      }
#pragma unroll
      for (int i = 0; i < DK / 2; ++i) o[i] *= corr[(i >> 1) & 1];
      uint32_t ph[FA_BKV / 4], plo[X3 ? FA_BKV / 4 : 1];   // P as the A fragments of the four 16-key steps
#pragma unroll
      for (int i = 0; i < FA_BKV / 4; ++i) {
        const float e0 = exp2f(sc[2 * i] - mrow[i & 1]), e1 = exp2f(sc[2 * i + 1] - mrow[i & 1]);
        ph[i] = pack_h2(e0, e1);
        const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&ph[i]));
        if constexpr (X3) {
          plo[i] = pack_h2(e0 - hf.x, e1 - hf.y);
          lrow[i & 1] += e0 + e1;
        } else {                                            // the row sum of the weights the tensor core actually applies
          lrow[i & 1] += hf.x + hf.y;
        }
      }

      // ---- O += P V ----
      mbar_wait(&v_full[s], parity);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < FA_BKV / 16; ++ks) {
        const uint64_t vh = make_sw128_kmajor_desc(v_addr) + 2 * ks;
        if constexpr (X3) {
          const uint64_t vl = make_sw128_kmajor_desc(v_addr + F::V_PLANE) + 2 * ks;
          wgmma_pv<DK>(o, plo + 4 * ks, vh);
          wgmma_pv<DK>(o, ph + 4 * ks, vl);
        }
        wgmma_pv<DK>(o, ph + 4 * ks, vh);
      }
      wgmma_commit();
      wgmma_wait<0>();
      pin_regs<DK / 2>(o);
      __syncwarp();
      if (lane == 0) mbar_arrive(&v_empty[s]);
    }
  }

  // ---- epilogue: O / l (V planes carry kPlaneScale); rows past len are exact zeros ----
  const int L = p.L, C = p.C;
  const long rows = (long)p.B * L;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    float l = lrow[r];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int t = q0 + 64 * cg + 16 * wq + g + 8 * r;
    if (t >= L) continue;
    const bool valid = t < len;
    const float inv = valid && l > 0.f ? kPlaneInv / l : 0.f;
    const long row = (long)b * L + t;
#pragma unroll
    for (int j = 0; j < DK / 8; ++j) {
      const float v0 = valid ? o[4 * j + 2 * r] * inv : 0.f, v1 = valid ? o[4 * j + 2 * r + 1] * inv : 0.f;
      const long off = row * C + h * DK + j * 8 + 2 * tq;
      if (p.ctx) *reinterpret_cast<float2*>(p.ctx + off) = make_float2(v0, v1);
      if (p.ctxp) {
        uint32_t hi, lo;
        split_pair(v0, v1, hi, lo);
        *reinterpret_cast<uint32_t*>(p.ctxp + off) = hi;
        if (X3) *reinterpret_cast<uint32_t*>(p.ctxp + rows * C + off) = lo;
      }
    }
  }
  pdl_trigger();
}

template <int DK>
int launch_tf32(const AParams& p, cudaStream_t st) {
  using A = ACfg<DK>;
  static unsigned long long configured = 0;   // per-device bit mask
  int rc;
  if ((rc = ensure_smem_attr(attention_tc_kernel<DK>, A::SMEM, &configured))) return rc;
  dim3 grid((p.L + BQ - 1) / BQ, p.heads, p.B);
  FS2_CUDA_CHECK(launch_pdl(attention_tc_kernel<DK>, grid, dim3(ATT_THREADS), A::SMEM, st, p));
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

template <int DK, bool X3>
int launch_wgmma(const AParams& p, cudaStream_t st) {
  using F = FCfg<DK, X3>;
  static unsigned long long configured = 0;   // per-device bit mask
  int rc;
  if ((rc = ensure_smem_attr(attention_wgmma_kernel<DK, X3>, F::SMEM, &configured))) return rc;
  // q|k planes as {2C, L, P * B} (rows past L zero-fill), V^T planes as {lpad, d_k, P * B * heads}
  CUtensorMap mq, mk, mv;
  const uint64_t qk_row = (uint64_t)2 * p.C * sizeof(__half), v_row = (uint64_t)p.lpad * sizeof(__half);
  const uint64_t qk_utt = (uint64_t)F::P * p.B, v_mats = (uint64_t)F::P * p.B * p.heads;
  if ((rc = make_map(&mq, p.q, 2 * (uint64_t)p.C, p.L, qk_utt, qk_row, qk_row * p.L, FA_BQ, true))) return rc;
  if ((rc = make_map(&mk, p.q, 2 * (uint64_t)p.C, p.L, qk_utt, qk_row, qk_row * p.L, FA_BKV, true))) return rc;
  if ((rc = make_map(&mv, p.vt, p.lpad, DK, v_mats, v_row, v_row * DK, DK, true))) return rc;
  dim3 grid((p.L + FA_BQ - 1) / FA_BQ, p.heads, p.B);
  FS2_CUDA_CHECK(launch_pdl(attention_wgmma_kernel<DK, X3>, grid, dim3(FA_THREADS), F::SMEM, st, mq, mk, mv, p));
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

__global__ void transpose_v_kernel(const float* __restrict__ qkv, int L, int C, float* __restrict__ vt, int lpad) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, t0 = blockIdx.x * 32, n0 = blockIdx.y * 32;   // n over the C columns of the V third
  int t = t0 + threadIdx.y, n = n0 + threadIdx.x;
  tile[threadIdx.y][threadIdx.x] = (t < L) ? qkv[((long)b * L + t) * 3 * C + 2 * C + n] : 0.f;
  __syncthreads();
  t = t0 + threadIdx.x; n = n0 + threadIdx.y;
  if (t < L) vt[((long)b * C + n) * lpad + t] = tile[threadIdx.x][threadIdx.y];   // (b*heads + h)*dk + d == b*C + n
}

// test helper (single-operator entry): qkv fp32 [B,L,3C] -> q|k planes [2][B*L][2C] and V^T planes [2][B*heads][dk][lpad]
__global__ void qkv_to_planes_kernel(const float* __restrict__ qkv, int B, int L, int C, __half* __restrict__ qkp,
                                     __half* __restrict__ vtp, int lpad) {
  const long rows = (long)B * L;
  const long total = rows * 3 * C;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long r = i / (3 * C); const int c = (int)(i - r * 3 * C);
    const float x = fminf(fmaxf(qkv[i] * kPlaneScale, -65504.f), 65504.f);
    const __half hi = __float2half_rn(x), lo = __float2half_rn(x - __half2float(hi));
    if (c < 2 * C) {
      qkp[r * 2 * C + c] = hi; qkp[(rows + r) * 2 * C + c] = lo;
    } else {
      const long bb = r / L; const int t = (int)(r - bb * L);
      const long o = (bb * C + (c - 2 * C)) * (long)lpad + t;           // (b*heads + h)*dk + d == b*C + n
      vtp[o] = hi; vtp[(long)B * C * lpad + o] = lo;
    }
  }
}

}  // namespace

int transpose_v(const float* qkv, int B, int L, int C, int heads, float* vt, int lpad, cudaStream_t st) {
  (void)heads;
  dim3 grid((L + 31) / 32, C / 32, B), block(32, 32);
  transpose_v_kernel<<<grid, block, 0, st>>>(qkv, L, C, vt, lpad);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int qkv_to_planes(const float* qkv, int B, int L, int C, int heads, __half* qkp, __half* vtp, int lpad, cudaStream_t st) {
  (void)heads;
  const long total = (long)B * L * 3 * C;
  if (total == 0) return FS2_OK;
  long blocks = (total + 255) / 256;
  qkv_to_planes_kernel<<<(int)(blocks > 132 * 16 ? 132 * 16 : blocks), 256, 0, st>>>(qkv, B, L, C, qkp, vtp, lpad);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int attention_tf32(const float* qkv, const float* vt, int lpad, const int64_t* lens, int B, int L, int C, int heads,
                   float* ctx, cudaStream_t st) {
  FS2_REQUIRE(heads > 0 && C % heads == 0, "attention: C=%d not divisible by heads=%d", C, heads);
  FS2_REQUIRE(vt && lpad >= L && lpad % 4 == 0, "attention_tf32: needs the transposed V buffer with a 16-byte aligned row pitch");
  if (B == 0 || L == 0) return FS2_OK;
  AParams p;
  p.q = qkv; p.vt = vt; p.lpad = lpad; p.lens = lens; p.B = B; p.L = L; p.C = C; p.heads = heads; p.ctx = ctx; p.ctxp = nullptr;
  p.scale_log2e = (1.0f / sqrtf((float)(C / heads))) * 1.4426950408889634f;
  const int dk = C / heads;
  if (dk == 192) return launch_tf32<192>(p, st);
  if (dk == 128) return launch_tf32<128>(p, st);
  set_error("attention: d_k=%d unsupported (128 or 192)", dk);
  return FS2_ERR_INVALID;
}

int attention_planes(const __half* qkp, const __half* vtp, int lpad, const int64_t* lens, int B, int L, int C, int heads, bool x3,
                     float* ctx, __half* ctxp, cudaStream_t st) {
  FS2_REQUIRE(heads > 0 && C % heads == 0, "attention: C=%d not divisible by heads=%d", C, heads);
  FS2_REQUIRE(qkp && vtp && lpad >= L && lpad % 8 == 0, "attention_planes: needs q|k planes and transposed V planes with a 16-byte aligned row pitch");
  FS2_REQUIRE((reinterpret_cast<uintptr_t>(qkp) & 15) == 0 && (reinterpret_cast<uintptr_t>(vtp) & 15) == 0,
              "attention_planes: operand planes must be 16-byte aligned");
  FS2_REQUIRE(ctx || ctxp, "attention_planes: no output");
  FS2_REQUIRE(!ctxp || ((reinterpret_cast<uintptr_t>(ctxp) & 31) == 0 && (((long)B * L * C) % 16) == 0), "attention_planes: context planes must be 32-byte aligned");
  if (B == 0 || L == 0) return FS2_OK;
  AParams p;
  p.q = qkp; p.vt = vtp; p.lpad = lpad; p.lens = lens; p.B = B; p.L = L; p.C = C; p.heads = heads; p.ctx = ctx; p.ctxp = ctxp;
  p.scale_log2e = (1.0f / sqrtf((float)(C / heads))) * 1.4426950408889634f * kPlaneInv * kPlaneInv;
  const int dk = C / heads;
  if (dk == 192) return x3 ? launch_wgmma<192, true>(p, st) : launch_wgmma<192, false>(p, st);
  if (dk == 128) return x3 ? launch_wgmma<128, true>(p, st) : launch_wgmma<128, false>(p, st);
  set_error("attention: d_k=%d unsupported (128 or 192)", dk);
  return FS2_ERR_INVALID;
}

}  // namespace fs2
