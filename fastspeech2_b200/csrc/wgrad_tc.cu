// Tensor-core weight gradient of a Conv1d("same") / Linear for the tf32 train mode (sm_90a):
//
//   dW[n][k][j] += sum_{b, t < L} dy[b,t,n] * x[b, t+j-pad, k]      (x zero outside [0, L) of each utterance)
//
// the contract of train.cu's wgrad_kernel, output in the reference's layout [N][K][taps].  The contraction runs over time,
// and tf32 wgmma wants both operands K-major, so a producer pass writes the transposes dy^T [B][N][Lp] (Lp = L rounded up
// to 4: 16-byte TMA row strides) and x^T (phase copies, below), each value rounded to tf32 with cvt.rna.  The MMA truncates its
// operands to tf32, which is then exact: products are of round-to-nearest operands, so the result carries no truncation bias.
//
// Main kernel: one 128 x 128 output tile (dy channels n x x channels k) of one tap over one split of the (utterance, time)
// range is a work unit.  The range is the sequence of 32-step time chunks of utterance 0, then utterance 1, ...; split s
// covers chunks [s Q / S, (s+1) Q / S) of the Q = B ceil(L / 32) chunks, so a split may start or end inside an utterance.
// Per chunk the TMA producer loads the dy^T box {t0.., n0.., b} of a 3-D tensor map {time, channel, utterance} with time
// extent L, and the x^T box of tap j, which starts at time t0 + j - pad.  Every box starts at a non-negative multiple of
// 4 elements (16 bytes) in time: x^T is written in four phase copies, copy r holding x shifted right by P + r steps
// (P = pad rounded up to 4; explicit zeros in front, time extent L + P + r), and tap j reads the copy that puts its box
// start on 16 bytes.  (The first H100 run of the direct form, x^T boxes starting at any time step, stopped at a pipeline
// wait timeout at the first taps > 1 case; aligned starts are what the tap GEMM's loads use.)  A convolution (taps > 1)
// has four copies, a Linear one.  The unit zero-fills past each map's time extent (the convolution's padding, and the
// tail of the last chunk) and past N / K (edge tiles), and never reads the columns past that extent.
// A 32-step chunk is one 128-byte swizzle row.  Warp roles as in the tap GEMM (gemm_tc.cu): warp 0 is the producer filling
// an mbarrier ring, two consumer warpgroups each issue m64n128k8 wgmma chains on one 64-row half of every stage (setmaxnreg
// moves registers from the producer warpgroup), persistent CTAs walk the units.
// Each split writes its fp32 partial tile to the workspace; a reduce kernel adds the partials into dW in a fixed order
// (split 0 first).  No atomics: the same inputs always give the same bits.  The split count depends on the shape only, not
// on the device, so the bits do not change with the GPU's SM count either.
//
// A unit loads its dy tile once per tap: a unit covering all taps of an output tile would need taps x 64 accumulator
// registers per consumer thread (576 at k = 9), and the x boxes of neighbouring taps overlap, so they mostly hit in L2.
#include <math.h>

#include "tc_common.cuh"

namespace fs2 {
namespace {
using namespace tc;

constexpr int WT_BM = 128;                                   // dy channels per tile (two 64-row warpgroup halves)
constexpr int WT_BN = 128;                                   // x channels per tile
constexpr int WT_BT = 32;                                    // time steps per stage: one 128-byte swizzle row of fp32
constexpr int WT_A_BYTES = WT_BM * WT_BT * 4;                // 16 KB
constexpr int WT_STAGE_BYTES = (WT_BM + WT_BN) * WT_BT * 4;  // 32 KB
constexpr int WT_STAGES = 6;
constexpr size_t WT_SMEM = (size_t)WT_STAGES * WT_STAGE_BYTES + 1024 + 256;
constexpr int WT_THREADS = 384;                              // producer warpgroup + two consumer warpgroups
constexpr int WT_PRODUCER_REGS = 40, WT_CONSUMER_REGS = 232;
constexpr int WT_PLAN_CTAS = 132;                            // the split count aims at whole waves of this many CTAs
constexpr int WT_MAX_SPLITS = 64;
constexpr int WT_MIN_CHUNKS = 4;                             // chunks per split, at least (when there are that many)
constexpr int WT_PHASES = 4;                                 // x^T phase copies of a convolution: box starts on 16 bytes

struct WgradParams {
  int N, K, taps, pad, P;     // P: left shift of x^T copy 0 (pad rounded up to 4)
  int n_tiles, k_tiles, splits, units;
  long Q; int cpu;           // chunks in all, chunks per utterance
  float* part;               // [splits][taps][N][K]
};

__device__ __forceinline__ float tf32_rna(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return __uint_as_float(r);
}

// in [B][L][C] -> `copies` outputs [B][C][pitch] (copy stride cstride floats), rounded to tf32: copy r holds time t at
// column t + shift + r, and zeros in columns [0, shift + r); columns past L + shift + r are not written.
// One 32 x 32 tile per step.
__global__ void __launch_bounds__(256) transpose_tf32_kernel(const float* __restrict__ in, int B, int L, int C, int shift, int copies,
                                                             long pitch, long cstride, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int tt = (L + 31) / 32, ct = (C + 31) / 32;
  const long total = (long)B * tt * ct;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (long i = blockIdx.x; i < total; i += gridDim.x) {
    const int c0 = (int)(i % ct) * 32;
    const long r = i / ct;
    const int t0 = (int)(r % tt) * 32, b = (int)(r / tt);
    const float* src = in + (long)b * L * C;
    for (int y = ty; y < 32; y += 8) {
      const int t = t0 + y, c = c0 + tx;
      if (t < L && c < C) tile[y][tx] = tf32_rna(src[(long)t * C + c]);
    }
    __syncthreads();
    for (int r = 0; r < copies; ++r) {
      float* dst = out + r * cstride + (long)b * C * pitch + shift + r;
      for (int y = ty; y < 32; y += 8) {
        const int c = c0 + y, t = t0 + tx;
        if (c < C && t < L) dst[(long)c * pitch + t] = tile[tx][y];
        if (t0 == 0 && c < C)
          for (int z = tx; z < shift + r; z += 32) dst[(long)c * pitch - shift - r + z] = 0.f;
      }
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(WT_THREADS, 1)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap map_dy, const __grid_constant__ CUtensorMap map_x0, const __grid_constant__ CUtensorMap map_x1,
                const __grid_constant__ CUtensorMap map_x2, const __grid_constant__ CUtensorMap map_x3, WgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* tiles = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(tiles + (size_t)WT_STAGES * WT_STAGE_BYTES);
  uint64_t* empty_bar = full_bar + WT_STAGES;
  const int warp = uniform_warp_idx(), lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < WT_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }   // the 8 consumer warps release
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // unit = ((split * n_tiles + n tile) * taps + tap) * k_tiles + k tile: CTAs running together share a split's time range
  auto unit_coords = [&](int u, int& split, int& j, int& n0, int& k0, long& c0, long& c1) {
    const int kt = u % p.k_tiles;
    int r = u / p.k_tiles;
    j = r % p.taps; r /= p.taps;
    const int nt = r % p.n_tiles;
    split = r / p.n_tiles;
    n0 = nt * WT_BM; k0 = kt * WT_BN;
    c0 = (long)split * p.Q / p.splits; c1 = (long)(split + 1) * p.Q / p.splits;
  };

  if (warp < 4) {
    setmaxnreg_dec<WT_PRODUCER_REGS>();
    if (warp != 0) return;
    // ---- TMA producer: the whole warp runs the loop, one lane is elected inside each asm ----
    const uint32_t tiles_addr = smem_u32(tiles), full_addr = smem_u32(full_bar);
    int n = 0;                                 // ring position, runs across units
    for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
      int split, j, n0, k0; long c0, c1;
      unit_coords(u, split, j, n0, k0, c0, c1);
      int b = (int)(c0 / p.cpu), tc = (int)(c0 - (long)b * p.cpu);
      // tap j: x^T copy r at time t0 + s + P + r, a non-negative multiple of 4 (s = j - pad >= -P)
      const int sh = j - p.pad + p.P, r = (-sh) & 3;
      const CUtensorMap* map_x = r == 0 ? &map_x0 : r == 1 ? &map_x1 : r == 2 ? &map_x2 : &map_x3;
      for (long c = c0; c < c1; ++c, ++n) {
        const int slot = n % WT_STAGES, round = n / WT_STAGES;
        const int t0 = tc * WT_BT;
        const uint32_t st = tiles_addr + (uint32_t)slot * WT_STAGE_BYTES, fb = full_addr + (uint32_t)slot * 8u;
        pin_before(st, fb, t0, b);
        mbar_wait(&empty_bar[slot], (round & 1) ^ 1);
        mbar_expect_tx_elect(fb, WT_STAGE_BYTES);
        tma_load_3d_elect(st, &map_dy, fb, t0, n0, b);
        tma_load_3d_elect(st + WT_A_BYTES, map_x, fb, t0 + sh + r, k0, b);
        if (++tc == p.cpu) { tc = 0; ++b; }
      }
    }
  } else {
    // ---- consumers: warpgroup cg owns rows 64 cg .. 64 cg + 63 of every tile ----
    setmaxnreg_inc<WT_CONSUMER_REGS>();
    const int cg = (warp >> 2) - 1, wq = warp & 3;
    constexpr uint64_t HALF_A = (WT_A_BYTES / 2) >> 4;   // second 64-row half of the dy tile, in descriptor units
    float d[WT_BN / 2];
    int n = 0;
    for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
      int split, j, n0, k0; long c0, c1;
      unit_coords(u, split, j, n0, k0, c0, c1);
      const long steps = c1 - c0;
      int prev = -1;
      for (long s = 0; s < steps; ++s, ++n) {
        const int slot = n % WT_STAGES, round = n / WT_STAGES;
        const uint32_t base = smem_u32(tiles + (size_t)slot * WT_STAGE_BYTES);
        const uint64_t a = make_sw128_kmajor_desc(base) + cg * HALF_A, bd = make_sw128_kmajor_desc(base + WT_A_BYTES);
        mbar_wait(&full_bar[slot], round & 1);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)           // +32 bytes along time inside the swizzle row = +2 in descriptor units
          wgmma_tf32_n128(d, a + 2 * kk, bd + 2 * kk, (s | kk) != 0);
        wgmma_commit();
        wgmma_wait<1>();                         // the previous stage's MMAs are done: release its slot
        pin_regs<WT_BN / 2>(d);
        if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
        prev = slot;
      }
      wgmma_wait<0>();
      pin_regs<WT_BN / 2>(d);
      if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[prev]); }
      if (steps == 0) {
#pragma unroll
        for (int i = 0; i < WT_BN / 2; ++i) d[i] = 0.f;
      }
      // ---- epilogue: this split's partial tile; d[4 jj + 2 h + {0,1}] = row 16 wq + lane / 4 + 8 h, columns 8 jj + 2 (lane % 4) + {0,1}
      float* __restrict__ dst = p.part + (long)(split * p.taps + j) * p.N * p.K;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = n0 + 64 * cg + 16 * wq + (lane >> 2) + 8 * h;
        if (row >= p.N) continue;
        float* dr = dst + (long)row * p.K;
#pragma unroll
        for (int jj = 0; jj < WT_BN / 8; ++jj) {
          const int col = k0 + 8 * jj + 2 * (lane & 3);
          if (col < p.K) dr[col] = d[4 * jj + 2 * h];
          if (col + 1 < p.K) dr[col + 1] = d[4 * jj + 2 * h + 1];
        }
      }
      __syncwarp();                              // converged again before the next unit's waits and wgmma
    }
  }
}

// dw[n][k][j] += sum over splits, in split order, of part[split][j][n][k]
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, int splits, int taps, int N, int K, float* __restrict__ dw) {
  const long nk = (long)N * K, tnk = nk * taps;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < tnk; i += (long)gridDim.x * blockDim.x) {
    float s = part[i];
    for (int q = 1; q < splits; ++q) s += part[q * tnk + i];
    const long j = i / nk, r = i - j * nk;
    dw[r * taps + j] += s;
  }
}

struct WgradPlan {
  long Lp, Q; int cpu;
  int P, phases; long Lx;          // x^T: phase copies [phases][B][K][Lx], copy r shifted right by P + r
  int n_tiles, k_tiles, splits, units;
  size_t dyT_off, xT_off, bytes;   // partial sums at offset 0
};

bool mul_ok(uint64_t a, uint64_t b, uint64_t* r) { return !__builtin_mul_overflow(a, b, r); }
uint64_t align256(uint64_t v) { return (v + 255) & ~(uint64_t)255; }

// Shape -> decomposition and workspace layout; FS2_ERR_INVALID for a bad or overflowing size.  B * L == 0 plans nothing.
int wgrad_plan(int B, int L, int N, int K, int taps, WgradPlan* pl, const char* who) {
  FS2_REQUIRE(B >= 0 && L >= 0 && N > 0 && K > 0 && taps > 0 && (taps & 1) == 1, "%s: need B, L >= 0, N, K > 0 and odd taps", who);
  *pl = WgradPlan{};
  if ((long)B * L == 0) return FS2_OK;
  pl->Lp = ((long)L + 3) & ~3L;
  pl->P = ((taps - 1) / 2 + 3) & ~3;
  pl->phases = taps > 1 ? WT_PHASES : 1;
  pl->Lx = ((long)L + pl->P + pl->phases - 1 + 3) & ~3L;
  pl->cpu = (L + WT_BT - 1) / WT_BT;
  pl->Q = (long)B * pl->cpu;
  pl->n_tiles = (N + WT_BM - 1) / WT_BM;
  pl->k_tiles = (K + WT_BN - 1) / WT_BN;
  const uint64_t tiles = (uint64_t)pl->n_tiles * pl->k_tiles * (uint64_t)taps;
  // TMA limits: byte strides below 2^40, int32 coordinates (t0 + j - pad), int work-unit and chunk counts
  FS2_REQUIRE((long)L + 2L * taps < (1L << 30) && pl->Q < (1L << 31) && tiles * WT_MAX_SPLITS < (1ull << 31), "%s: size too large", who);
  FS2_REQUIRE((uint64_t)pl->Lx * 4 * (uint64_t)(N > K ? N : K) < (1ull << 40), "%s: size too large (TMA stride)", who);
  // splits: the fewest that bring the units' last wave clearly closer to full (5 points), with >= WT_MIN_CHUNKS chunks each
  long smax = pl->Q / WT_MIN_CHUNKS;
  smax = smax < 1 ? 1 : (smax > WT_MAX_SPLITS ? WT_MAX_SPLITS : smax);
  auto eff = [&](long s) { const double u = (double)tiles * s; return u / (ceil(u / WT_PLAN_CTAS) * WT_PLAN_CTAS); };
  int best = 1; double best_eff = eff(1);
  for (long s = 2; s <= smax; ++s) {
    const double e = eff(s);
    if (e > best_eff + 0.05) { best = (int)s; best_eff = e; }
  }
  pl->splits = best;
  pl->units = (int)(tiles * best);
  uint64_t part, dyT, xT, t;
  const bool ok = mul_ok((uint64_t)best * taps, (uint64_t)N * K, &t) && mul_ok(t, 4, &part) &&
                  mul_ok((uint64_t)B * N, (uint64_t)pl->Lp * 4, &dyT) && mul_ok((uint64_t)B * K * pl->phases, (uint64_t)pl->Lx * 4, &xT) &&
                  part < (1ull << 61) && dyT < (1ull << 61) && xT < (1ull << 61);
  FS2_REQUIRE(ok, "%s: size too large (workspace overflows)", who);
  pl->dyT_off = align256(part);
  pl->xT_off = pl->dyT_off + align256(dyT);
  pl->bytes = pl->xT_off + align256(xT);
  return FS2_OK;
}

}  // namespace
}  // namespace fs2

using namespace fs2;

extern "C" {

int fs2_conv_wgrad_tc_ws_bytes(int B, int L, int N, int K, int taps, size_t* bytes) {
  FS2_REQUIRE(bytes, "fs2_conv_wgrad_tc_ws_bytes: null argument");
  WgradPlan pl;
  int rc = wgrad_plan(B, L, N, K, taps, &pl, "fs2_conv_wgrad_tc_ws_bytes");
  if (rc) return rc;
  *bytes = pl.bytes;
  return FS2_OK;
}

int fs2_conv_wgrad_tc(const float* dy, const float* x, int B, int L, int N, int K, int taps, float* dw, float* dbias, void* ws,
                      size_t ws_bytes, void* stream) {
  FS2_REQUIRE(dy && x && dw, "fs2_conv_wgrad_tc: null argument");
  WgradPlan pl;
  int rc = wgrad_plan(B, L, N, K, taps, &pl, "fs2_conv_wgrad_tc");
  if (rc) return rc;
  if ((long)B * L == 0) return FS2_OK;
  FS2_REQUIRE(ws && (reinterpret_cast<uintptr_t>(ws) & 15) == 0, "fs2_conv_wgrad_tc: workspace missing or not 16-byte aligned");
  FS2_REQUIRE(ws_bytes >= pl.bytes, "fs2_conv_wgrad_tc: workspace of %zu bytes, %zu needed", ws_bytes, pl.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  static unsigned long long configured = 0;
  if ((rc = ensure_smem_attr(wgrad_tc_kernel, WT_SMEM, &configured))) return rc;
  float* part = reinterpret_cast<float*>(ws);
  float* dyT = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(ws) + pl.dyT_off);
  float* xT = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(ws) + pl.xT_off);
  const long xstride = (long)B * K * pl.Lx;      // floats between x^T phase copies
  auto transpose = [&](const float* in, int C_, int shift, int copies, long pitch, float* out) -> int {
    const long tiles = (long)B * pl.cpu * ((C_ + 31) / 32);
    transpose_tf32_kernel<<<(unsigned)(tiles < 132 * 16 ? tiles : 132 * 16), 256, 0, st>>>(in, B, L, C_, shift, copies, pitch, xstride, out);
    FS2_LAUNCH_CHECK();
    return FS2_OK;
  };
  if ((rc = transpose(dy, N, 0, 1, pl.Lp, dyT)) || (rc = transpose(x, K, pl.P, pl.phases, pl.Lx, xT))) return rc;
  CUtensorMap mdy, mx[WT_PHASES];
  if ((rc = make_map(&mdy, dyT, L, N, B, pl.Lp * 4, (uint64_t)N * pl.Lp * 4, WT_BM))) return rc;
  for (int r = 0; r < WT_PHASES; ++r) {          // a Linear has one copy: its map serves every (unused) phase
    const int c = r < pl.phases ? r : 0;
    if ((rc = make_map(&mx[r], xT + c * xstride, (uint64_t)L + pl.P + c, K, B, pl.Lx * 4, (uint64_t)K * pl.Lx * 4, WT_BN))) return rc;
  }
  WgradParams p;
  p.N = N; p.K = K; p.taps = taps; p.pad = (taps - 1) / 2; p.P = pl.P;
  p.n_tiles = pl.n_tiles; p.k_tiles = pl.k_tiles; p.splits = pl.splits; p.units = pl.units;
  p.Q = pl.Q; p.cpu = pl.cpu; p.part = part;
  const int grid = pl.units < sm_count_current() ? pl.units : sm_count_current();
  wgrad_tc_kernel<<<grid, WT_THREADS, WT_SMEM, st>>>(mdy, mx[0], mx[1], mx[2], mx[3], p);
  FS2_LAUNCH_CHECK();
  const long tnk = (long)taps * N * K;
  const long blocks = (tnk + 255) / 256;
  wgrad_reduce_kernel<<<(unsigned)(blocks < 132 * 8 ? blocks : 132 * 8), 256, 0, st>>>(part, pl.splits, taps, N, K, dw);
  FS2_LAUNCH_CHECK();
  if (dbias) return fs2_colsum(dy, (int64_t)B * L, N, dbias, stream);
  return FS2_OK;
}

}  // extern "C"
