// Tensor-core "tap GEMM" for sm_90a: wgmma (warpgroup MMA, tf32 or f16 operands, fp32 accumulators in registers),
// operands staged in shared memory by TMA (cp.async.bulk.tensor, 128-byte swizzle), mbarrier pipelines, persistent CTAs.
//
//   out[b,t,n] = act( sum_{j<taps} sum_{k<K} x[b, t+(j-pad)*dil, k] * w[j][n][k] + bias[n] ) (+ resid[b,t,n])
//
// Same contract as gemm_fp32.cu (the CUDA-core family).  Three instantiation families:
//   <BN, false, false>  plain tf32 (one MMA per product) on the fp32 activations themselves: the decoder side in
//                       FS2_MATH_TF32;
//   <BN, false, true>   f16 on the hi planes of activations and weights (decoder side in FS2_MATH_F16);
//   <BN, true,  true>   error-compensated "3xF16" on hi + lo planes (encoder and predictors in every tensor-core mode,
//                       everything in FS2_MATH_3XTF32): fp32-class results; their outputs feed round() / bucketize(),
//                       where 10-bit-mantissa noise (~1e-3) would flip integers.  Three products per K step into one
//                       accumulator, small terms first: lo.hi + hi.lo + hi.hi.
// Operand planes (common.cuh): activations are pre-scaled by kPlaneScale, weights by a per-layer power of two; the
// epilogue multiplies the accumulator by the exact inverse (oscale) in the same FMA that adds the bias.  Results leave as
// fp32 rows and / or as the operand planes of the next contraction (no separate split / conversion pass).
//
// Why no im2col: activations are [B, time, channel] with channels innermost, which *is* the K-major A operand of a GEMM.
// Tap j of a 1-D convolution is the same matrix shifted by (j - pad) * dil rows (dil = 1 except in dilated convolutions), so
// the producer just issues the TMA box at row coordinate t0 + (j - pad) * dil of a 3-D tensor map {channel, time,
// utterance}; rows outside [0, L) of the utterance are
// zero-filled by the TMA unit (that is exactly Conv1d's "same" padding).  K loop = taps x ceil(K / 32) pipeline steps of
// 4 MMAs with K = 8 each (tf32; f16: ceil(K / 64) steps with K = 16 each: one 128-byte swizzle row either way).
//
// One persistent CTA per SM walks the 128 x BN output tiles (n fastest, so concurrently running CTAs share weight tiles
// in L2).  Warp roles (3 warpgroups): warp 0 is the TMA producer, filling one ordered ring of stages for the CTA's tiles
// in turn; warpgroups 1 and 2 "ping-pong": the CTA's k-th tile belongs wholly to warpgroup k & 1, which issues the wgmma
// chains of both 64-row halves on each of the tile's ring stages (BN accumulator registers per thread; setmaxnreg moves
// registers from the producer warpgroup), releases a stage as soon as the MMAs that read it have completed (one stage
// stays in flight), then runs the epilogue (bias / ReLU / tanh / residual, fp32 rows, operand planes, or the transposed
// V third) while the other warpgroup already issues the next tile's MMAs.  The epilogue goes through a small staging area
// in shared memory, 16 columns at a time (Cfg::SW), so that one rolled loop with tile-uniform choices stores whole row
// segments and V runs of up to 128 time steps; where the ring leaves no room for it, it runs from the registers.  An
// mbarrier pair makes the two main loops strictly alternate (see the consumer loop), so the tensor cores do not wait for
// an epilogue.  A row's K loop (the MMAs that accumulate it, and their order) depends neither on its tile nor on the
// warpgroup, so results do not depend on the schedule (per-utterance bit-identity, DESIGN.md §5).
// Convolutions tile each utterance separately so the shifted boxes never cross an utterance boundary: floor(L/128) full
// row tiles per utterance, and the tails (L % 128 rows, in 16-row granules loaded by separate small TMA boxes) of several
// utterances packed into shared tiles, so no tensor-core rows are spent on padding.  Plain GEMMs (taps == 1) tile the flat
// [B*L, K] matrix, except in per-utterance mode (TapGemm::lens), where they tile per utterance as well so that tiles
// wholly past an utterance's length can be skipped.  Every mbarrier wait is bounded: a pipeline bug traps instead of
// hanging the GPU.
// The 3xF16 lo planes are addressed through the same tensor map: plane stride = B*L rows, i.e. utterance index b + B.
#include <stdlib.h>

#include "tc_common.cuh"

namespace fs2 {
namespace {
using namespace tc;

constexpr int BM = 128;
constexpr int BK = 32;                 // fp32 elements per pipeline step = one 128-byte swizzle row (64 when the operands are fp16)
constexpr int A_BYTES = BM * BK * 4;   // 16 KB
constexpr int THREADS = 384;           // producer warpgroup + two consumer warpgroups
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;   // setmaxnreg: 128 * 40 + 256 * 232 <= 65536; a consumer holds BN accumulators
constexpr int RING_BUDGET = 227 * 1024 - 1024 /*align slack*/ - 256 /*barriers*/;

struct TcParams {
  int L, tiles_per_utt;          // tiles_per_utt == 0: flat tiling, L = B*L rows
  int m_tiles, n_tiles;
  // convolutions (tiles_per_utt > 0): every utterance has `full` 128-row tiles; its tail (L % 128 rows, `gn` granules
  // of 16 rows) shares a packed tile with the tails of upt - 1 other utterances, so no MMA rows are wasted on padding
  int B, full, gn, upt, full_tiles;
  int K, taps, pad, dil;         // tap j reads rows t + (j - pad) * dil
  const float* bias; const float* resid; int ldr; int act;
  float* out; int ldo;
  float a_inv; const float* w_inv;   // accumulator scale = a_inv * (w_inv ? *w_inv : 1): undoes the operand planes' pre-scaling
  __half* outp; __half* outp_lo; int ldo_p;   // result as operand planes (hi; lo when the consumer is 3xF16); out may then be null
  // optional: columns >= vt_col0 are the V third of a q|k|v projection and are stored transposed,
  // vt[(b*heads + h)*dk + d][t] with row pitch vt_lpad, for the attention kernel's P.V operand
  float* vt_out; __half* vtp; __half* vtp_lo; int vt_col0, vt_dk, vt_heads, vt_lpad, vt_L;
  // per-utterance mode (nullable; needs the per-utterance tiling): rows t >= lens[b] are written as exact zeros in every
  // non-V column, fp32 rows and planes alike, and an ordinary tile with t0 >= lens[b] is dead -- no TMA loads, no MMAs,
  // only those zero stores.  The transposed V third of those rows is not needed (the attention kernels read no key row
  // past len), so dead and live tiles alike skip its stores there.
  const int64_t* lens;
};

// Epilogue staging (per consumer warpgroup): one slice of SW columns of its 128-row tile, either row-major (SW floats per
// row, 16-byte chunks XOR-swizzled by row) or, for the transposed V third, column-major (VT_PITCH floats per column,
// rows XOR-swizzled in 4-row groups by row / 32).  Both patterns make the fragment writes and the read-back free of
// bank conflicts.
constexpr int VT_PITCH = BM + 4;
constexpr int stage_area(int sw) { return 2 * 4 * sw * VT_PITCH; }   // two warpgroups; the column-major form is the larger

template <int BN, bool PRECISE, bool HALF = false>
struct Cfg {
  static constexpr int B_BYTES = BN * BK * 4;
  static constexpr int STAGE_BYTES = (PRECISE ? 2 : 1) * (A_BYTES + B_BYTES);   // [A hi][A lo][B hi][B lo]
  static_assert(!PRECISE || HALF, "the error-compensated family is 3xF16");
  static constexpr int STAGES = (RING_BUDGET / STAGE_BYTES) > 8 ? 8 : (RING_BUDGET / STAGE_BYTES);
  static constexpr int RING = STAGES * STAGE_BYTES;
  // staging slice width in the shared memory the ring leaves over; 0: no room (f16 / tf32 at BN = 128), the epilogue
  // then runs straight from the accumulator registers
  static constexpr int SW = RING + stage_area(16) <= RING_BUDGET ? 16 : RING + stage_area(8) <= RING_BUDGET ? 8 : 0;
  static constexpr int STG_BYTES = SW ? stage_area(SW) : 0;
  static constexpr size_t SMEM = (size_t)RING + STG_BYTES + 1024 + 256;
  static_assert(SMEM <= 227 * 1024 && BN % (SW ? SW : 16) == 0, "staging must fit beside the ring and divide the tile");
  static constexpr int BKE = HALF ? 2 * BK : BK;           // K elements per pipeline step
  static constexpr int A_LO = A_BYTES;                      // offsets inside a stage
  static constexpr int B_HI = PRECISE ? 2 * A_BYTES : A_BYTES;
  static constexpr int B_LO = B_HI + B_BYTES;
  static constexpr uint32_t TX_BYTES = (PRECISE ? 2 : 1) * (A_BYTES + B_BYTES);
  static_assert(BN % 16 == 0 && BN >= 16 && BN <= 128, "tile width: sums of wgmma N = 128 / 64 / 16");
  static_assert(B_BYTES % 1024 == 0, "B stage must keep 1024-byte alignment");
  static_assert(STAGES >= 2, "resources");
};

// D[64 x BN] (+)= A . B^T for one 32-byte K slice, as wgmma instructions of N = 128, 64 and 16 (column offset c0 of the
// tile: B rows c0.., accumulator registers d[c0 / 2]..)
template <int BN, bool HALF, int C0 = 0>
__device__ __forceinline__ void mma_tile(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  if constexpr (BN - C0 >= 128) {
    if constexpr (HALF) wgmma_f16_n128(d + C0 / 2, a, b + (C0 * 128 >> 4), acc); else wgmma_tf32_n128(d + C0 / 2, a, b + (C0 * 128 >> 4), acc);
    mma_tile<BN, HALF, C0 + 128>(d, a, b, acc);
  } else if constexpr (BN - C0 >= 64) {
    if constexpr (HALF) wgmma_f16_n64(d + C0 / 2, a, b + (C0 * 128 >> 4), acc); else wgmma_tf32_n64(d + C0 / 2, a, b + (C0 * 128 >> 4), acc);
    mma_tile<BN, HALF, C0 + 64>(d, a, b, acc);
  } else if constexpr (BN - C0 >= 16) {
    if constexpr (HALF) wgmma_f16_n16(d + C0 / 2, a, b + (C0 * 128 >> 4), acc); else wgmma_tf32_n16(d + C0 / 2, a, b + (C0 * 128 >> 4), acc);
    mma_tile<BN, HALF, C0 + 16>(d, a, b, acc);
  }
}

__device__ __forceinline__ void named_bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }
// row-major staging: physical 16-byte chunk of logical chunk c in row r is c ^ row_swz(r); column-major: row r sits at
// r ^ col_swz(r)
template <int SW>
__device__ __forceinline__ int row_swz(int r) { return SW == 16 ? 3 * ((r >> 1) & 1) : (r >> 2) & 1; }
__device__ __forceinline__ int col_swz(int r) { return r ^ ((r >> 5) << 2); }

// Writes slice s (columns SW s .. SW s + SW - 1 of the warpgroup's 128 x BN accumulators) to its staging area.  The
// accumulators need constant register indices: one branch per slice.
template <int BN, int SW, int S = 0>
__device__ __forceinline__ void stage_slice(const float* d, int s, float* stg, bool col_major, int wq, int lane) {
  if constexpr (S < BN / SW) {
    if (s != S) { stage_slice<BN, SW, S + 1>(d, s, stg, col_major, wq, lane); return; }
#pragma unroll
    for (int hf = 0; hf < 2; ++hf) {
#pragma unroll
      for (int jj = 0; jj < SW / 8; ++jj) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float* v = d + hf * (BN / 2) + 4 * (S * (SW / 8) + jj) + 2 * h;
          const int row = 64 * hf + 16 * wq + (lane >> 2) + 8 * h, col = 8 * jj + 2 * (lane & 3);
          if (col_major) {
            stg[col * VT_PITCH + col_swz(row)] = v[0];
            stg[(col + 1) * VT_PITCH + col_swz(row)] = v[1];
          } else {
            *reinterpret_cast<float2*>(stg + row * SW + 4 * ((col >> 2) ^ row_swz<SW>(row)) + (col & 3)) = make_float2(v[0], v[1]);
          }
        }
      }
    }
  }
}

template <int BN, bool PRECISE, bool HALF>
__global__ void __launch_bounds__(THREADS, 1)
tap_gemm_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                   const __grid_constant__ CUtensorMap tmap_b_lo, const __grid_constant__ CUtensorMap tmap_a16, TcParams p) {
  using C = Cfg<BN, PRECISE, HALF>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* tiles = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // keeps the shared address space (no generic LD/ST)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(tiles + (size_t)C::STAGES * C::STAGE_BYTES);
  uint64_t* empty_bar = full_bar + C::STAGES;

  const int warp = uniform_warp_idx(), lane = threadIdx.x & 31;
  const int kchunks = (p.K + C::BKE - 1) / C::BKE;
  const int steps = p.taps * kchunks;
  const int total_tiles = p.m_tiles * p.n_tiles;

  uint64_t* order_bar = empty_bar + C::STAGES;             // [cg]: the other warpgroup has issued its previous tile's MMAs

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }   // the 4 warps of one consumer warpgroup release
    mbar_init(&order_bar[0], 4); mbar_init(&order_bar[1], 4);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();                                              // everything above overlapped the previous kernel's tail

  // packed < 0: ordinary tile (utterance b, rows t0 .. t0+127); packed >= 0: index of a packed tail tile.
  // Returns true for a dead tile (per-utterance mode: every row lies past lens[b]).
  auto tile_coords = [&](int tile, int& n0, int& b, int& t0, int& packed) -> bool {
    const int mt = tile / p.n_tiles;
    n0 = (tile - mt * p.n_tiles) * BN;
    packed = -1;
    if (p.tiles_per_utt == 0) { b = 0; t0 = mt * BM; }
    else if (mt < p.full_tiles) { b = mt / p.full; t0 = (mt - b * p.full) * BM; }
    else { packed = mt - p.full_tiles; b = packed * p.upt; t0 = p.full * BM; }
    return packed < 0 && p.lens != nullptr && t0 >= p.lens[b];
  };

  if (warp < 4) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp != 0) { pdl_trigger(); return; }
    // ---- TMA producer: the whole warp runs the loop, one lane is elected inside each asm; everything a stage's loads need
    // is computed before the wait for its slot, and the tap / K-chunk indices are carried as counters
    const uint32_t tiles_addr = smem_u32(tiles), full_addr = smem_u32(full_bar);
    int n = 0;      // ring position, runs across tiles
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      int n0, b, t0, packed;
      if (tile_coords(tile, n0, b, t0, packed)) continue;   // dead tile: the consumers take no stage from the ring either
      int j = 0, kc = 0;                        // tap, K chunk of step s
      for (int s = 0; s < steps; ++s, ++n) {
        const int slot = n % C::STAGES, round = n / C::STAGES;
        const int k0 = kc * C::BKE, row = t0 + (j - p.pad) * p.dil;
        const uint32_t st = tiles_addr + (uint32_t)slot * C::STAGE_BYTES, fb = full_addr + (uint32_t)slot * 8u;
        pin_before(st, fb, k0, row);
        mbar_wait(&empty_bar[slot], (round & 1) ^ 1);
        mbar_expect_tx_elect(fb, C::TX_BYTES);
        if (packed < 0) {
          tma_load_3d_elect(st, &tmap_a, fb, k0, row, b);
          if (PRECISE) tma_load_3d_elect(st + C::A_LO, &tmap_a, fb, k0, row, b + p.B);
        } else {
          // eight 16-row boxes: granule g belongs to utterance b + g / gn (zero-filled past the batch or past L)
          for (int g = 0; g < 8; ++g) {
            const int u = g / p.gn, gi = g - u * p.gn;
            const bool real = u < p.upt && b + u < p.B;
            const int oob = PRECISE ? 2 * p.B : p.B;  // out of bounds in dim 2 -> the box is all zeros
            tma_load_3d_elect(st + g * (16 * 128), &tmap_a16, fb, k0, row + gi * 16, real ? b + u : oob);
            if (PRECISE) tma_load_3d_elect(st + C::A_LO + g * (16 * 128), &tmap_a16, fb, k0, row + gi * 16, real ? b + u + p.B : oob);
          }
        }
        tma_load_3d_elect(st + C::B_HI, &tmap_b, fb, k0, n0, j);
        if (PRECISE) tma_load_3d_elect(st + C::B_LO, &tmap_b_lo, fb, k0, n0, j);
        if (++kc == kchunks) { kc = 0; ++j; }
      }
    }
  } else {
    // ---- consumers: warpgroup cg = 0 / 1 owns every other tile of the CTA (its k-th tile goes to k & 1), all 128 rows ----
    setmaxnreg_inc<CONSUMER_REGS>();
    const int cg = (warp >> 2) - 1, wq = warp & 3;
    const int r_lo = 16 * wq + (lane >> 2);      // rows 64 hf + r_lo + 8 h of the tile (hf, h = 0 / 1); columns 8 j + 2 (lane % 4)
    const int act = p.act, ldr = p.ldr, ldo = p.ldo;
    const float* __restrict__ resid = p.resid; float* __restrict__ out = p.out;
    const bool has_res = resid != nullptr;
    const float oscale = p.a_inv * (p.w_inv ? __ldg(p.w_inv) : 1.0f);   // exact power of two (1 in the tf32 family)
    float d[BN];                                  // [hf][BN / 2]: the accumulators of the tile's two 64-row halves
    constexpr int SW = C::SW, LPR = SW / 8;       // staged epilogue: slice width, threads per row (8 columns each)
    float* stg = reinterpret_cast<float*>(tiles + (size_t)C::RING + 256) + cg * (C::STG_BYTES / 8);
    const int tid = threadIdx.x - 128 * (cg + 1);
    int n = 0;                                    // ring position: advanced past the other warpgroup's tiles as well
    int k = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++k) {
      int n0, b, t0, packed;
      const int tile_steps = tile_coords(tile, n0, b, t0, packed) ? 0 : steps;
      if ((k & 1) != cg) { n += tile_steps; continue; }
      // row of the tile -> global row mm; ok: the row exists; zero: per-utterance mode, the row lies past lens;
      // *left: rows of the utterance from this one on that exist and lie before lens
      auto row_at = [&](int row, long& mm, bool& ok, bool& zero, int* left = nullptr) {
        int bb = b, t = t0 + row;
        ok = t < p.L;                            // flat mode: L == total rows
        if (packed >= 0) {                       // packed tail tile: 16-row granule g of the tile -> utterance b + g / gn
          const int g = row >> 4, u = g / p.gn, gi = g - u * p.gn;
          bb += u;
          t = t0 + gi * 16 + (row & 15);
          ok = u < p.upt && bb < p.B && t < p.L;
        }
        mm = (long)bb * p.L + t;
        zero = ok && p.lens != nullptr && t >= p.lens[bb];
        if (left) *left = ok && !zero ? (p.lens != nullptr && p.lens[bb] < p.L ? (int)p.lens[bb] : p.L) - t : 0;
      };
      const bool to_vt = (p.vt_out != nullptr || p.vtp != nullptr) && n0 >= p.vt_col0;   // tile-uniform (tile widths divide the V third)
      long m[4]; bool row_ok[4], row_zero[4];    // direct epilogue: the thread's accumulator rows 64 hf + r_lo + 8 h
      if constexpr (SW == 0) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {            // i = 2 hf + h
          row_at(64 * (i >> 1) + r_lo + 8 * (i & 1), m[i], row_ok[i], row_zero[i]);
          if (has_res && row_ok[i]) prefetch_l2(resid + m[i] * ldr + n0);   // residual rows -> L2 while the main loop runs
        }
      } else if (has_res) {
#pragma unroll
        for (int i = 0; i < LPR; ++i) {
          long mm; bool ok, zero;
          row_at(tid / LPR + (BM / LPR) * i, mm, ok, zero);
          if (ok) prefetch_l2(resid + mm * ldr + n0);   // residual rows -> L2 while the main loop runs
        }
      }
      // Main loops alternate between the warpgroups: this tile's starts once the other warpgroup has issued the MMAs of the
      // CTA's previous tile (it arrives even for a dead tile).  That keeps the tensor cores fed by one warpgroup while the
      // other runs its epilogue, and it is what makes the parity waits below sound: every ring position before this tile
      // has been filled, so the producer is never a whole ring round behind the position waited for.
      if (k > 0) mbar_wait(&order_bar[cg], ((k - 1) >> 1) & 1);
      int prev = -1;
      for (int s = 0; s < tile_steps; ++s, ++n) {
        const int slot = n % C::STAGES, round = n / C::STAGES;
        const uint32_t base = smem_u32(tiles + (size_t)slot * C::STAGE_BYTES);
        const uint64_t a_hi = make_sw128_kmajor_desc(base), b_hi = make_sw128_kmajor_desc(base + C::B_HI);
        const uint64_t a_lo = make_sw128_kmajor_desc(base + C::A_LO), b_lo = make_sw128_kmajor_desc(base + C::B_LO);
        constexpr uint64_t HALF_A = (A_BYTES / 2) >> 4;   // second 64-row half of the A tile, in descriptor units
        mbar_wait(&full_bar[slot], round & 1);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {         // +32 bytes along K inside the swizzle row = +2 in descriptor units
#pragma unroll
          for (int hf = 0; hf < 2; ++hf) {
            float* dh = d + hf * (BN / 2);
            if (PRECISE) {
              mma_tile<BN, true>(dh, a_lo + hf * HALF_A + 2 * kk, b_hi + 2 * kk, (s | kk) != 0);   // small terms first
              mma_tile<BN, true>(dh, a_hi + hf * HALF_A + 2 * kk, b_lo + 2 * kk, 1);
              mma_tile<BN, true>(dh, a_hi + hf * HALF_A + 2 * kk, b_hi + 2 * kk, 1);
            } else {
              mma_tile<BN, HALF>(dh, a_hi + hf * HALF_A + 2 * kk, b_hi + 2 * kk, (s | kk) != 0);
            }
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                         // the previous stage's MMAs are done: release its slot
        pin_regs<BN>(d);
        if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
        prev = slot;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&order_bar[cg ^ 1]);   // the other warpgroup's next main loop may start
      wgmma_wait<0>();
      pin_regs<BN>(d);
      if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
      if (tile_steps == 0) {
#pragma unroll
        for (int i = 0; i < BN; ++i) d[i] = 0.f;
      }

      if constexpr (SW > 0) {
        // ---- staged epilogue: per slice, the accumulators go to shared memory and come back as whole row segments
        // (8 columns per thread, LPR threads per row) or, for the V third, as column runs of 8 consecutive rows ----
        const bool res16 = (reinterpret_cast<uintptr_t>(resid) & 15) == 0;
        // V tiles: this thread's rows r8 .. r8 + 7 lie in one 16-row granule, so the rows to store (ok, not past lens) are
        // its first nv, with global rows mm0 + i; vrun: they form one aligned 16-byte run of a vt row
        const int r8 = 8 * (tid & 15);
        auto vt_row = [&](int mm) {              // vt[(ub * heads + h) * dk + d][ut] for h * dk + d = 0 (B * L < 2^31 rows)
          const int ub = mm / p.vt_L;
          return (long)ub * p.vt_heads * p.vt_dk * p.vt_lpad + (mm - ub * p.vt_L);
        };
        long mm0 = 0, vo = 0; int nv = 0; bool vrun = false;
        if (to_vt) {
          bool ok, zero;
          row_at(r8, mm0, ok, zero, &nv);
          nv = nv < 8 ? nv : 8;
          vo = vt_row(mm0);
          vrun = nv == 8 && (int)mm0 % p.vt_L + 8 <= p.vt_L && (vo & 7) == 0 && p.vtp != nullptr &&
                 (reinterpret_cast<uintptr_t>(p.vtp) & 15) == 0;
        }
#pragma unroll 1
        for (int s = 0; s < BN / SW; ++s) {
          named_bar_sync(1 + cg, 128);           // the warpgroup has read the previous slice
          stage_slice<BN, SW>(d, s, stg, to_vt, wq, lane);
          named_bar_sync(1 + cg, 128);
          if (to_vt) {
#pragma unroll
            for (int pass = 0; pass < SW / 8; ++pass) {
              const int cl = (tid >> 4) + 8 * pass, col = n0 + s * SW + cl;
              const float bias = p.bias ? __ldg(p.bias + col) : 0.f;
              const float4 x0 = *reinterpret_cast<const float4*>(stg + cl * VT_PITCH + col_swz(r8));
              const float4 x1 = *reinterpret_cast<const float4*>(stg + cl * VT_PITCH + col_swz(r8 + 4));
              float v[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
#pragma unroll
              for (int e = 0; e < 8; ++e) v[e] = fmaf(v[e], oscale, bias);
              const long oc = (long)(col - p.vt_col0) * p.vt_lpad;
              if (vrun) {                        // 16 consecutive threads: 128 time steps of one vt row
                uint4 hi, lo;
                split_pair(v[0], v[1], hi.x, lo.x); split_pair(v[2], v[3], hi.y, lo.y);
                split_pair(v[4], v[5], hi.z, lo.z); split_pair(v[6], v[7], hi.w, lo.w);
                *reinterpret_cast<uint4*>(p.vtp + vo + oc) = hi;
                if (p.vtp_lo != nullptr) *reinterpret_cast<uint4*>(p.vtp_lo + vo + oc) = lo;
                continue;
              }
#pragma unroll 1
              for (int i = 0; i < nv; ++i) {     // rows that cross an utterance or are not 16-byte aligned in vt
                const float x = fmaf(stg[cl * VT_PITCH + col_swz(r8 + i)], oscale, bias);
                const long o = vt_row(mm0 + i) + oc;
                if (p.vt_out != nullptr) { p.vt_out[o] = x; continue; }
                uint32_t hi, lo;
                split_pair(x, x, hi, lo);
                p.vtp[o] = __ushort_as_half((unsigned short)hi);
                if (p.vtp_lo != nullptr) p.vtp_lo[o] = __ushort_as_half((unsigned short)lo);
              }
            }
            continue;
          }
          const int h = tid % LPR, col = n0 + s * SW + 8 * h;
          float bv[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) bv[e] = p.bias ? __ldg(p.bias + col + e) : 0.f;
#pragma unroll 1
          for (int i = 0; i < LPR; ++i) {
            const int row = tid / LPR + (BM / LPR) * i;
            long mm; bool ok, zero;
            row_at(row, mm, ok, zero);
            if (!ok) continue;
            // every load of the row (residual) is issued before its stores: a caller's residual may be the output
            float rv[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            if (has_res) {
              const float* rp = resid + mm * ldr + col;
              if (res16) {
                const float4 a = __ldg(reinterpret_cast<const float4*>(rp)), c = __ldg(reinterpret_cast<const float4*>(rp + 4));
                rv[0] = a.x; rv[1] = a.y; rv[2] = a.z; rv[3] = a.w; rv[4] = c.x; rv[5] = c.y; rv[6] = c.z; rv[7] = c.w;
              } else {
#pragma unroll
                for (int e = 0; e < 8; e += 2) {
                  const float2 a = __ldg(reinterpret_cast<const float2*>(rp + e));
                  rv[e] = a.x; rv[e + 1] = a.y;
                }
              }
            }
            const float* sr = stg + row * SW;
            const float4 x0 = *reinterpret_cast<const float4*>(sr + 4 * ((2 * h) ^ row_swz<SW>(row)));
            const float4 x1 = *reinterpret_cast<const float4*>(sr + 4 * ((2 * h + 1) ^ row_swz<SW>(row)));
            float v[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              v[e] = fmaf(v[e], oscale, bv[e]);
              if (act == ACT_RELU) v[e] = fmaxf(v[e], 0.f);
              else if (act == ACT_TANH) v[e] = tanhf(v[e]);
              if (has_res) v[e] += rv[e];
              if (zero) v[e] = 0.f;
            }
            if (HALF && p.outp != nullptr) {     // operand planes of the next contraction
              const long off = mm * p.ldo_p + col;
              if (p.outp_lo != nullptr) {
                uint4 hi, lo;
                split_pair(v[0], v[1], hi.x, lo.x); split_pair(v[2], v[3], hi.y, lo.y);
                split_pair(v[4], v[5], hi.z, lo.z); split_pair(v[6], v[7], hi.w, lo.w);
                *reinterpret_cast<uint4*>(p.outp + off) = hi;
                *reinterpret_cast<uint4*>(p.outp_lo + off) = lo;
              } else {
                *reinterpret_cast<uint4*>(p.outp + off) = make_uint4(hi_pair(v[0], v[1]), hi_pair(v[2], v[3]), hi_pair(v[4], v[5]), hi_pair(v[6], v[7]));
              }
            }
            if (out != nullptr) {
              *reinterpret_cast<float4*>(out + mm * ldo + col) = make_float4(v[0], v[1], v[2], v[3]);
              *reinterpret_cast<float4*>(out + mm * ldo + col + 4) = make_float4(v[4], v[5], v[6], v[7]);
            }
          }
        }
        continue;
      }

      // ---- epilogue from registers: element pairs (row, columns c, c + 1) ----
      // Row by row, every load of a row (bias, residual) is issued before its first store: as far as the compiler knows,
      // the stores may alias the loads, so interleaving them would serialise one load latency per column pair.
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (!row_ok[i] || (to_vt && row_zero[i])) continue;
        const long mm = m[i];
        float* dr = d + (i >> 1) * (BN / 2) + 2 * (i & 1);   // this row's pairs: dr[4 jj], dr[4 jj + 1]
#pragma unroll
        for (int jj = 0; jj < BN / 8; ++jj) {
          const int col = n0 + 8 * jj + 2 * (lane & 3);
          float v0 = dr[4 * jj], v1 = dr[4 * jj + 1];
          const float b0 = p.bias ? __ldg(p.bias + col) : 0.f, b1 = p.bias ? __ldg(p.bias + col + 1) : 0.f;
          v0 = fmaf(v0, oscale, b0); v1 = fmaf(v1, oscale, b1);
          if (!to_vt) {
            if (act == ACT_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            else if (act == ACT_TANH) { v0 = tanhf(v0); v1 = tanhf(v1); }
            if (has_res) {
              const float2 r = __ldg(reinterpret_cast<const float2*>(resid + mm * ldr + col));
              v0 += r.x; v1 += r.y;
            }
            if (row_zero[i]) { v0 = 0.f; v1 = 0.f; }
          }
          dr[4 * jj] = v0; dr[4 * jj + 1] = v1;
        }
        if (to_vt) {
          // transposed store: for a fixed column the 8 row groups of a warp hold consecutive time steps.
          // vt[(ub * heads + h) * dk + d][ut] with h * dk + d = col - vt_col0
          const long ub = mm / p.vt_L;
          const long orow = ub * p.vt_heads * p.vt_dk * (long)p.vt_lpad + (mm - ub * p.vt_L);
#pragma unroll
          for (int jj = 0; jj < BN / 8; ++jj) {
            const int col = n0 + 8 * jj + 2 * (lane & 3);
            const float v0 = dr[4 * jj], v1 = dr[4 * jj + 1];
            const long o = orow + (long)(col - p.vt_col0) * p.vt_lpad;
            if (p.vt_out != nullptr) {
              p.vt_out[o] = v0; p.vt_out[o + p.vt_lpad] = v1;
            } else {
              uint32_t hi, lo;
              split_pair(v0, v1, hi, lo);
              const __half2 h2 = *reinterpret_cast<const __half2*>(&hi), l2 = *reinterpret_cast<const __half2*>(&lo);
              p.vtp[o] = __low2half(h2); p.vtp[o + p.vt_lpad] = __high2half(h2);
              if (p.vtp_lo != nullptr) { p.vtp_lo[o] = __low2half(l2); p.vtp_lo[o + p.vt_lpad] = __high2half(l2); }
            }
          }
          continue;
        }
#pragma unroll
        for (int jj = 0; jj < BN / 8; ++jj) {
          const int col = n0 + 8 * jj + 2 * (lane & 3);
          const float v0 = dr[4 * jj], v1 = dr[4 * jj + 1];
          if (HALF && p.outp != nullptr) {       // operand planes of the next contraction
            const long off = mm * p.ldo_p + col;
            if (p.outp_lo != nullptr) {
              uint32_t hi, lo;
              split_pair(v0, v1, hi, lo);
              *reinterpret_cast<uint32_t*>(p.outp + off) = hi;
              *reinterpret_cast<uint32_t*>(p.outp_lo + off) = lo;
            } else {
              *reinterpret_cast<uint32_t*>(p.outp + off) = hi_pair(v0, v1);
            }
          }
          if (out != nullptr) *reinterpret_cast<float2*>(out + mm * ldo + col) = make_float2(v0, v1);
        }
      }
    }
  }
  pdl_trigger();                               // this CTA's work is done: the next kernel may start launching (FS2_PDL)
}

// Pre-pass for tensors that enter the library as fp32 (LengthRegulator output, single-operator test entries):
// x [rows][ldx] fp32 -> S[0] = hi plane, S[1] = lo plane, each [rows][K] fp16, scaled by kPlaneScale.
// One float4 per thread and step, 8-byte stores.
__global__ void split_rows_f16_kernel(const float* __restrict__ x, int ldx, long rows, int K, __half* __restrict__ S) {
  pdl_trigger(); pdl_wait();
  const int kq = K >> 2;
  const long quads = rows * kq;
  __half* __restrict__ lo_plane = S + rows * K;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < quads; i += (long)gridDim.x * blockDim.x) {
    const long r = i / kq;
    const int c = (int)(i - r * kq) * 4;
    const float4 v = *reinterpret_cast<const float4*>(x + r * ldx + c);
    uint2 hv, lv;
    split_pair(v.x, v.y, hv.x, lv.x);
    split_pair(v.z, v.w, hv.y, lv.y);
    *reinterpret_cast<uint2*>(S + r * K + c) = hv;
    *reinterpret_cast<uint2*>(lo_plane + r * K + c) = lv;
  }
}

// ---- host side ----------------------------------------------------------------------------------
template <int BN, bool PRECISE, bool HALF = false>
int launch(const TapGemm& g, cudaStream_t st) {
  using C = Cfg<BN, PRECISE, HALF>;
  static unsigned long long configured = 0;   // per-device bit mask
  int rc;
  if ((rc = ensure_smem_attr(tap_gemm_tc_kernel<BN, PRECISE, HALF>, C::SMEM, &configured))) return rc;
  TcParams p;
  p.K = g.K; p.taps = g.taps; p.pad = (g.taps - 1) / 2; p.dil = g.dil > 1 ? g.dil : 1;
  p.bias = g.bias; p.resid = g.resid; p.ldr = g.ldr; p.act = g.act; p.out = g.out; p.ldo = g.ldo;
  const long rows = (long)g.B * g.L;
  p.a_inv = HALF ? g.a_inv : 1.0f; p.w_inv = HALF ? g.w_inv : nullptr;
  p.outp = HALF ? g.outp : nullptr; p.ldo_p = g.ldo_p;
  p.outp_lo = (HALF && g.outp && g.outp_lo) ? g.outp + rows * g.ldo_p : nullptr;
  p.vt_out = HALF ? nullptr : g.vt_out; p.vtp = HALF ? g.vtp : nullptr;
  p.vtp_lo = (HALF && g.vtp && g.outp_lo) ? g.vtp + (long)g.B * g.vt_heads * g.vt_dk * g.vt_lpad : nullptr;
  p.vt_col0 = g.vt_col0; p.vt_dk = g.vt_dk; p.vt_heads = g.vt_heads; p.vt_lpad = g.vt_lpad; p.vt_L = g.L;
  p.lens = g.lens;
  CUtensorMap ma, mb, mb_lo, ma16;
  const int esz = HALF ? 2 : 4;
  constexpr int planes = HALF && PRECISE ? 2 : 1;          // 3xF16: [hi plane][lo plane], each [B*L][K] fp16
  const void* xa = HALF ? (const void*)g.xp : (const void*)g.x;
  const uint64_t row_bytes = HALF ? (uint64_t)g.K * 2 : (uint64_t)g.ldx * 4;
  // with lens, plain GEMMs take the per-utterance tiling too, so that tiles past an utterance's length are dead; a row's
  // K loop is the same in either tiling, so its result does not depend on it
  if (g.taps == 1 && g.lens == nullptr) {  // flat [B*L, K]
    const uint64_t M = (uint64_t)g.B * g.L;
    p.L = (int)M; p.tiles_per_utt = 0;
    p.m_tiles = (int)((M + BM - 1) / BM);
    p.B = 1; p.full = 0; p.gn = 1; p.upt = 1; p.full_tiles = 0;
    if ((rc = make_map(&ma, xa, g.K, M, planes, row_bytes, row_bytes * M, BM, HALF))) return rc;
    ma16 = ma;
  } else {            // per-utterance tiles: shifted boxes zero-fill outside [0, L)
    p.L = g.L; p.tiles_per_utt = (g.L + BM - 1) / BM;
    p.B = g.B; p.full = g.L / BM;
    int tail = g.L % BM;
    p.gn = tail ? (tail + 15) / 16 : 1;
    p.upt = tail ? 8 / p.gn : 1;
    if (tail && p.upt == 1) { p.full += 1; tail = 0; p.gn = 1; }   // tail > 64 rows: nothing to share, keep one ordinary (partly empty) tile
    p.full_tiles = p.full * g.B;
    p.m_tiles = p.full_tiles + (tail ? (g.B + p.upt - 1) / p.upt : 0);
    if ((rc = make_map(&ma, xa, g.K, g.L, (uint64_t)g.B * planes, row_bytes, row_bytes * g.L, BM, HALF))) return rc;
    if ((rc = make_map(&ma16, xa, g.K, g.L, (uint64_t)g.B * planes, row_bytes, row_bytes * g.L, 16, HALF))) return rc;
  }
  p.n_tiles = g.N / BN;
  const void* w_hi = HALF ? (const void*)g.w_hi : (const void*)g.w;
  if ((rc = make_map(&mb, w_hi, g.K, g.N, g.taps, (uint64_t)g.K * esz, (uint64_t)g.K * esz * g.N, BN, HALF))) return rc;
  if ((rc = make_map(&mb_lo, PRECISE ? (const void*)g.w_lo : w_hi, g.K, g.N, g.taps, (uint64_t)g.K * esz, (uint64_t)g.K * esz * g.N, BN, HALF))) return rc;
  const int total = p.m_tiles * p.n_tiles;
  const int grid = total < sm_count_current() ? total : sm_count_current();
  FS2_CUDA_CHECK(launch_pdl(tap_gemm_tc_kernel<BN, PRECISE, HALF>, dim3(grid), dim3(THREADS), C::SMEM, st, ma, mb, mb_lo, ma16, p));
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// widest supported tile that divides N (wgmma N = 128, 64 + 16, 64, 16 + 16, 16)
int tile_width(int N) { return N % 128 == 0 ? 128 : N % 80 == 0 ? 80 : N % 64 == 0 ? 64 : N % 32 == 0 ? 32 : 16; }

template <bool PRECISE, bool HALF>
int launch_any(const TapGemm& g, cudaStream_t st) {
  switch (tile_width(g.N)) {
    case 128: return launch<128, PRECISE, HALF>(g, st);
    case 80: return launch<80, PRECISE, HALF>(g, st);
    case 64: return launch<64, PRECISE, HALF>(g, st);
    case 32: return launch<32, PRECISE, HALF>(g, st);
    default: return launch<16, PRECISE, HALF>(g, st);
  }
}

int check_output(const TapGemm& g, const char* who) {
  FS2_REQUIRE((g.taps & 1) == 1, "%s: taps must be odd", who);
  FS2_REQUIRE(g.N % 16 == 0, "%s: N (%d) must be a multiple of 16", who, g.N);
  FS2_REQUIRE(!g.resid || g.ldr % 4 == 0, "%s: row strides must be 16-byte multiples", who);
  FS2_REQUIRE(!g.out || (g.ldo % 8 == 0 && (reinterpret_cast<uintptr_t>(g.out) & 31) == 0), "%s: output rows must be 32-byte aligned", who);
  return FS2_OK;
}
int check_common(const TapGemm& g, const char* who) {
  FS2_REQUIRE(g.K % 4 == 0, "%s: K (%d) must be a multiple of 4", who, g.K);
  FS2_REQUIRE(g.ldx % 4 == 0, "%s: row strides must be 16-byte multiples", who);
  FS2_REQUIRE((reinterpret_cast<uintptr_t>(g.x) & 15) == 0 && (reinterpret_cast<uintptr_t>(g.w) & 15) == 0 && g.out != nullptr,
              "%s: operands must be 16-byte aligned", who);
  return check_output(g, who);
}

}  // namespace

int tap_gemm_tf32(const TapGemm& g, cudaStream_t st) {
  int rc = check_common(g, "tap_gemm_tf32");
  if (rc) return rc;
  FS2_REQUIRE(!g.vt_out || g.vt_col0 % tile_width(g.N) == 0, "tap_gemm_tf32: the transposed V third must start at a tile boundary");
  if ((long)g.B * g.L == 0) return FS2_OK;
  return launch_any<false, false>(g, st);
}

// f16 on the hi planes (g.precise == false) or 3xF16 on hi + lo planes
int tap_gemm_planes(const TapGemm& g, cudaStream_t st) {
  const char* who = g.precise ? "tap_gemm_planes(3xF16)" : "tap_gemm_planes(f16)";
  FS2_REQUIRE(g.xp && g.w_hi && (!g.precise || g.w_lo) && (g.out || g.outp || g.vtp), "%s: operand planes / an output missing", who);
  FS2_REQUIRE(g.K % 8 == 0, "%s: K (%d) must be a multiple of 8 (16-byte plane rows)", who, g.K);
  FS2_REQUIRE((reinterpret_cast<uintptr_t>(g.xp) & 15) == 0 && (reinterpret_cast<uintptr_t>(g.w_hi) & 15) == 0, "%s: operands must be 16-byte aligned", who);
  FS2_REQUIRE(!g.outp || (g.ldo_p % 16 == 0 && (reinterpret_cast<uintptr_t>(g.outp) & 31) == 0 && (((long)g.B * g.L * g.ldo_p) % 16) == 0),
              "%s: output plane rows must be 32-byte aligned", who);
  {
    const int bn = tile_width(g.N);
    FS2_REQUIRE(!g.vtp || (g.vt_lpad % 8 == 0 && g.N % bn == 0 && g.vt_col0 % bn == 0 && g.vt_dk % 32 == 0),
                "%s: transposed V planes need a 16-byte row pitch and tile-aligned thirds", who);
  }
  int rc = check_output(g, who);
  if (rc) return rc;
  if ((long)g.B * g.L == 0) return FS2_OK;
  return g.precise ? launch_any<true, true>(g, st) : launch_any<false, true>(g, st);
}

int split_rows(const float* x, int ldx, long rows, int K, __half* planes, cudaStream_t st) {
  if (rows == 0) return FS2_OK;
  FS2_REQUIRE(K % 4 == 0 && ldx % 4 == 0, "split_rows: K and the row stride must be multiples of 4");
  const long quads = rows * (K / 4);
  long blocks = (quads + 255) / 256;
  FS2_CUDA_CHECK(launch_pdl(split_rows_f16_kernel, dim3((unsigned)(blocks > 132 * 16 ? 132 * 16 : blocks)), dim3(256), 0, st, x, ldx, rows, K, planes));
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

namespace {
// weights: hi = rn(s w), lo = rn(s w - hi) with the layer's power-of-two scale s (device scalar; null = 1)
__global__ void split_f16_kernel(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo, long n,
                                 const float* __restrict__ scale) {
  const float s = scale ? __ldg(scale) : 1.0f;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const float x = fminf(fmaxf(src[i] * s, -65504.f), 65504.f);
    const __half h = __float2half_rn(x);
    hi[i] = h; lo[i] = __float2half_rn(x - __half2float(h));
  }
}
// one CTA: max |w| -> s = 2^k with s * max in [2^13, 2^14)  (fp16 max is 2^16: headroom for rounding, none of the
// weight's lo plane below ~2^-17 of the layer maximum is subnormal)
__global__ void weight_scale_kernel(const float* __restrict__ w, long n, float* __restrict__ scale, float* __restrict__ inv) {
  __shared__ float red[32];
  float m = 0.f;
  for (long i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, fabsf(w[i]));
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    m = warp_max(m);
    if (threadIdx.x == 0) {
      int k = 0;
      if (m > 0.f && isfinite(m)) {
        int e;
        frexpf(m, &e);          // m = f * 2^e, f in [0.5, 1)  ->  m * 2^(14 - e) in [2^13, 2^14)
        k = 14 - e;
        k = k > 60 ? 60 : (k < -60 ? -60 : k);
      }
      scale[0] = ldexpf(1.0f, k); inv[0] = ldexpf(1.0f, -k);
    }
  }
}
}  // namespace

namespace {
__global__ void planes_to_rows_kernel(const __half* __restrict__ planes, long n, float* __restrict__ out) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
    out[i] = (__half2float(planes[i]) + __half2float(planes[n + i])) * kPlaneInv;
}
}  // namespace

// test helper: planes [2][n] (hi, lo; scaled by kPlaneScale) -> fp32
int planes_to_rows(const __half* planes, long n, float* out, cudaStream_t st) {
  if (n == 0) return FS2_OK;
  long blocks = (n + 255) / 256;
  planes_to_rows_kernel<<<(int)(blocks > 1184 ? 1184 : blocks), 256, 0, st>>>(planes, n, out);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int split_f16(const float* src, __half* hi, __half* lo, long n, const float* scale, cudaStream_t st) {
  if (n == 0) return FS2_OK;
  long blocks = (n + 255) / 256;
  split_f16_kernel<<<(int)(blocks > 1184 ? 1184 : blocks), 256, 0, st>>>(src, hi, lo, n, scale);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int weight_scale(const float* w, long n, float* scale, float* inv, cudaStream_t st) {
  weight_scale_kernel<<<1, 1024, 0, st>>>(w, n, scale, inv);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace fs2
