// Objective evaluation (DESIGN.md section 20): mel-cepstral distortion under a full DTW alignment of synthesized and
// reference log-mels, and F0, voicing and energy errors along the alignment path, for a ragged batch of pairs.
//
//   eval_cepstra   c[t, k] = sum_m double(mel[t, m]) * D[m, k], one thread per (row, k), valid rows only, stored k-major
//                  [B][K][L] so that a warp's cells read consecutive doubles; checks the lengths and that every valid
//                  log-mel is finite
//   eval_dtw       one CTA per pair sweeps the anti-diagonals s = i + j of A(i, j) = d(i, j) + min(predecessors), with
//                  d computed on the fly from the two cepstra; three rolling diagonals of A and of the path length in
//                  shared memory (global workspace when the shorter side exceeds kDtwSmemCells); with a path, one
//                  direction byte per cell, stored diagonal-major so that each diagonal's writes are coalesced
//   eval_backtrack one thread per pair follows the direction bytes from the last cell and writes the path (0,0) first
//   eval_prosody   one thread per pair walks a path in order and accumulates the voicing, F0 and energy sums
// Every double sum and product is __dadd_rn / __dmul_rn, so nothing is contracted into an FMA: cepstra, costs, paths and
// MCD are bit-identical to a float64 restatement with the same operation order (oracle/eval_oracle.py), and a pair's
// results do not depend on its batch mates.
#include <math.h>
#include <math_constants.h>

#include "common.cuh"

namespace fs2 {
namespace {

constexpr int kDtwThreads = 1024;          // one cell per thread on diagonals of up to 1024 cells
constexpr int kDtwSmemCells = 1024;           // diagonal cells kept in shared memory: 3 * (8 + 4) * 1024 = 36 KiB
constexpr int kCepThreads = 256;

__device__ __forceinline__ bool len_ok(int64_t n, int L) { return n >= 1 && n <= L; }

// cep[b, k, t] for t < lens[b] (other columns are not written)
__global__ void eval_cepstra_kernel(const float* __restrict__ mel, const int64_t* __restrict__ lens, int B, int L, int M,
                                    const double* __restrict__ D, int K, double* __restrict__ cep, int* __restrict__ status) {
  const long total = (long)B * L * K;
  int bits = 0;
  for (long e = (long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
    const long bk = e / L;
    const int t = (int)(e - bk * L), b = (int)(bk / K), k = (int)(bk - (long)b * K);
    const long row = (long)b * L + t;
    const int64_t n = lens[b];
    if (!len_ok(n, L)) {
      if (t == 0 && k == 0) bits |= FS2_EVAL_BAD_LENGTH;
      continue;
    }
    if (t >= n) continue;
    const float* x = mel + row * M;
    double acc = 0.0;
    bool finite = true;
    for (int m = 0; m < M; ++m) {
      const float v = x[m];
      finite &= isfinite(v);
      acc = __dadd_rn(acc, __dmul_rn((double)v, D[(long)m * K + k]));
    }
    cep[e] = acc;
    if (!finite && k == 0) bits |= FS2_EVAL_NONFINITE;
  }
  if (bits) atomicOr(status, bits);
}

// a, b: column t of a k-major [K][L] cepstrum (row strides la, lb): a warp's cells read consecutive doubles of each row.
__device__ __forceinline__ double cep_distance(const double* __restrict__ a, int la, const double* __restrict__ b, int lb, int K) {
  double acc = 0.0;
#pragma unroll 8
  for (int k = 0; k < K; ++k) {
    const double d = __dsub_rn(__ldg(a + (size_t)k * la), __ldg(b + (size_t)k * lb));
    acc = __dadd_rn(acc, __dmul_rn(d, d));
  }
  return __dsqrt_rn(acc);
}

// First cell index i of anti-diagonal s of an Lx x Ly grid.
__device__ __forceinline__ int diag_lo(int s, int Ly) { return s - (Ly - 1) > 0 ? s - (Ly - 1) : 0; }

// One CTA per pair.  Diagonal s holds cells i in [lo(s), hi(s)], j = s - i, at index i - lo(s) of its rolling slot s % 3.
// dir (null without a path): byte at [b][s][i - lo(s)] of a [B][Lx_max + Ly_max - 1][W] array, 0 = (i-1, j-1),
// 1 = (i-1, j), 2 = (i, j-1).
__global__ void __launch_bounds__(kDtwThreads) eval_dtw_kernel(const double* __restrict__ cx, const int64_t* __restrict__ xlens, int Lx_max,
                                                                const double* __restrict__ cy, const int64_t* __restrict__ ylens, int Ly_max,
                                                                int K, int W, double scale, double* __restrict__ mcd, double* __restrict__ cost,
                                                                int64_t* __restrict__ plen, uint8_t* __restrict__ dir,
                                                                double* __restrict__ gA, int* __restrict__ gP) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int b = blockIdx.x;
  const int64_t nx = xlens[b], ny = ylens[b];
  if (!len_ok(nx, Lx_max) || !len_ok(ny, Ly_max)) {
    if (threadIdx.x == 0) { mcd[b] = CUDART_NAN; cost[b] = CUDART_NAN; plen[b] = 0; }
    return;
  }
  const int Lx = (int)nx, Ly = (int)ny;
  double* A;
  int* P;
  if (gA != nullptr) {
    A = gA + (size_t)b * 3 * W;
    P = gP + (size_t)b * 3 * W;
  } else {
    A = (double*)smem;
    P = (int*)(A + 3 * W);
  }
  const double* X = cx + (size_t)b * Lx_max * K;
  const double* Y = cy + (size_t)b * Ly_max * K;
  uint8_t* Db = dir ? dir + (size_t)b * (Lx_max + Ly_max - 1) * W : nullptr;
  const int S = Lx + Ly - 1;
  for (int s = 0; s < S; ++s) {
    const int lo = diag_lo(s, Ly), hi = s < Lx - 1 ? s : Lx - 1;
    const int lo1 = diag_lo(s - 1, Ly), lo2 = diag_lo(s - 2, Ly);
    double* A0 = A + (s % 3) * W;
    const double* A1 = A + ((s + 2) % 3) * W;
    const double* A2 = A + ((s + 1) % 3) * W;
    int* P0 = P + (s % 3) * W;
    const int* P1 = P + ((s + 2) % 3) * W;
    const int* P2 = P + ((s + 1) % 3) * W;
    for (int i = lo + threadIdx.x; i <= hi; i += blockDim.x) {
      const int j = s - i;
      const double d = cep_distance(X + i, Lx_max, Y + j, Ly_max, K);
      double best = 0.0;
      int bp = 0, dv = 0;
      bool have = false;
      if (i > 0 && j > 0) { best = A2[i - 1 - lo2]; bp = P2[i - 1 - lo2]; dv = 0; have = true; }
      if (i > 0) {
        const double v = A1[i - 1 - lo1];
        if (!have || v < best) { best = v; bp = P1[i - 1 - lo1]; dv = 1; have = true; }
      }
      if (j > 0) {
        const double v = A1[i - lo1];
        if (!have || v < best) { best = v; bp = P1[i - lo1]; dv = 2; have = true; }
      }
      const double a = have ? __dadd_rn(d, best) : d;
      const int p = bp + 1;
      A0[i - lo] = a;
      P0[i - lo] = p;
      if (Db) Db[(size_t)s * W + (i - lo)] = (uint8_t)dv;
      if (s == S - 1) {
        cost[b] = a;
        plen[b] = p;
        mcd[b] = __dmul_rn(__ddiv_rn(a, (double)p), scale);
      }
    }
    __syncthreads();
  }
}

// path[b, p] = (i, j) for p < plen[b], from (0, 0); the rest of path[b] is left as the caller set it (-1)
__global__ void eval_backtrack_kernel(const uint8_t* __restrict__ dir, const int64_t* __restrict__ xlens, int Lx_max,
                                      const int64_t* __restrict__ ylens, int Ly_max, int B, int W, const int64_t* __restrict__ plen,
                                      int32_t* __restrict__ path) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int64_t nx = xlens[b], ny = ylens[b];
  if (!len_ok(nx, Lx_max) || !len_ok(ny, Ly_max)) return;
  const int Ly = (int)ny;
  const uint8_t* Db = dir + (size_t)b * (Lx_max + Ly_max - 1) * W;
  int32_t* out = path + (size_t)b * (Lx_max + Ly_max - 1) * 2;
  int i = (int)nx - 1, j = Ly - 1;
  for (int p = (int)plen[b] - 1; p >= 0; --p) {
    out[2 * p] = i;
    out[2 * p + 1] = j;
    const int s = i + j;
    if (s == 0) break;
    const int dv = Db[(size_t)s * W + (i - diag_lo(s, Ly))];
    if (dv != 2) --i;
    if (dv != 1) --j;
  }
}

// counts[b] = (P, n_vuv, n_voiced, n_gross), sums[b] = (sq_cents, sq_energy), accumulated in path order
__global__ void eval_prosody_kernel(const int32_t* __restrict__ path, const int64_t* __restrict__ plen, int B, int P_max,
                                    const double* __restrict__ f0x, const int64_t* __restrict__ f0x_lens, int Fx,
                                    const double* __restrict__ f0y, const int64_t* __restrict__ f0y_lens, int Fy,
                                    const float* __restrict__ ex, int Ex, const float* __restrict__ ey, int Ey,
                                    int64_t* __restrict__ counts, double* __restrict__ sums, int* __restrict__ status) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const int64_t P = plen[b], nfx = f0x_lens[b], nfy = f0y_lens[b];
  int64_t n_vuv = 0, n_voiced = 0, n_gross = 0, n = 0;
  double sq_cents = 0.0, sq_energy = 0.0;
  int bits = 0;
  if (P < 0 || P > P_max || nfx < 0 || nfx > Fx || nfy < 0 || nfy > Fy) {
    bits = FS2_EVAL_BAD_LENGTH;
  } else {
    const int32_t* pb = path + (size_t)b * P_max * 2;
    for (int64_t p = 0; p < P; ++p) {
      const int i = pb[2 * p], j = pb[2 * p + 1];
      if (i < 0 || i >= Ex || j < 0 || j >= Ey) { bits = FS2_EVAL_BAD_LENGTH; break; }
      const double fx = i < nfx ? f0x[(size_t)b * Fx + i] : 0.0;
      const double fy = j < nfy ? f0y[(size_t)b * Fy + j] : 0.0;
      const bool vx = fx > 0.0, vy = fy > 0.0;
      n_vuv += vx != vy;
      if (vx && vy) {
        ++n_voiced;
        const double r = __ddiv_rn(fx, fy);
        const double c = __dmul_rn(1200.0, log2(r));
        sq_cents = __dadd_rn(sq_cents, __dmul_rn(c, c));
        n_gross += fabs(__dsub_rn(r, 1.0)) > 0.2;
      }
      const double e = __dsub_rn((double)ex[(size_t)b * Ex + i], (double)ey[(size_t)b * Ey + j]);
      sq_energy = __dadd_rn(sq_energy, __dmul_rn(e, e));
      ++n;
    }
  }
  counts[4 * b] = n;
  counts[4 * b + 1] = n_vuv;
  counts[4 * b + 2] = n_voiced;
  counts[4 * b + 3] = n_gross;
  sums[2 * b] = sq_cents;
  sums[2 * b + 1] = sq_energy;
  if (bits) atomicOr(status, bits);
}

struct DtwPlan {
  double* cx; double* cy;
  double* gA; int* gP;          // rolling diagonals in global memory (null: shared memory)
  uint8_t* dir;                 // direction bytes (null without a path)
  int W;
};

DtwPlan dtw_plan(Bump& b, int B, int Lx_max, int Ly_max, int K, bool with_path) {
  DtwPlan p{};
  p.W = Lx_max < Ly_max ? Lx_max : Ly_max;
  p.cx = b.doubles((size_t)B * Lx_max * K);
  p.cy = b.doubles((size_t)B * Ly_max * K);
  if (p.W > kDtwSmemCells) {
    p.gA = b.doubles((size_t)B * 3 * p.W);
    p.gP = (int*)b.bytes((size_t)B * 3 * p.W * sizeof(int));
  }
  if (with_path) p.dir = (uint8_t*)b.bytes((size_t)B * (Lx_max + Ly_max - 1) * p.W);
  return p;
}

int check_sizes(int B, int Lx_max, int Ly_max, int n_mels, int n_cep, const char* who) {
  FS2_REQUIRE(B >= 1 && B <= (1 << 20), "%s: B (%d) must lie in [1, 2^20]", who, B);
  FS2_REQUIRE(Lx_max >= 1 && Ly_max >= 1 && Lx_max < (1 << 24) && Ly_max < (1 << 24),
              "%s: Lx_max and Ly_max (%d, %d) must lie in [1, 2^24)", who, Lx_max, Ly_max);
  FS2_REQUIRE(n_mels >= 2 && n_mels <= 4096, "%s: n_mels (%d) must lie in [2, 4096]", who, n_mels);
  FS2_REQUIRE(n_cep >= 1 && n_cep <= n_mels - 1, "%s: n_cep (%d) must lie in [1, n_mels - 1 = %d]", who, n_cep, n_mels - 1);
  const long W = Lx_max < Ly_max ? Lx_max : Ly_max;
  FS2_REQUIRE((long)(Lx_max + Ly_max) * W < (1L << 40) && (long)B * (Lx_max + Ly_max) * n_mels < (1L << 40),
              "%s: batch too large", who);
  return FS2_OK;
}

}  // namespace
}  // namespace fs2

using namespace fs2;

extern "C" {

int fs2_dtw_workspace_bytes(int B, int Lx_max, int Ly_max, int n_mels, int n_cep, int with_path, size_t* bytes) {
  FS2_REQUIRE(bytes, "fs2_dtw_workspace_bytes: null argument");
  int rc = check_sizes(B, Lx_max, Ly_max, n_mels, n_cep, "fs2_dtw_workspace_bytes");
  if (rc) return rc;
  Bump b(nullptr, 0);
  dtw_plan(b, B, Lx_max, Ly_max, n_cep, with_path != 0);
  *bytes = align256(b.off) + 256;
  return FS2_OK;
}

int fs2_mcd_dtw(const float* x, const int64_t* xlens, int Lx_max, const float* y, const int64_t* ylens, int Ly_max, int B,
                int n_mels, const double* dct, int n_cep, double scale, double* mcd, double* cost, int64_t* plen, int32_t* path,
                int* status, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(x && xlens && y && ylens && dct && mcd && cost && plen && status && ws, "fs2_mcd_dtw: null argument");
  int rc = check_sizes(B, Lx_max, Ly_max, n_mels, n_cep, "fs2_mcd_dtw");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Bump b(ws, ws_bytes);
  DtwPlan p = dtw_plan(b, B, Lx_max, Ly_max, n_cep, path != nullptr);
  if ((rc = b.check("fs2_mcd_dtw"))) return rc;
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  eval_cepstra_kernel<<<grid_for((long)B * Lx_max * n_cep, kCepThreads), kCepThreads, 0, st>>>(x, xlens, B, Lx_max, n_mels, dct, n_cep,
                                                                                                 p.cx, status);
  FS2_LAUNCH_CHECK();
  eval_cepstra_kernel<<<grid_for((long)B * Ly_max * n_cep, kCepThreads), kCepThreads, 0, st>>>(y, ylens, B, Ly_max, n_mels, dct, n_cep,
                                                                                                 p.cy, status);
  FS2_LAUNCH_CHECK();
  const size_t smem = p.gA ? 0 : (size_t)3 * p.W * (sizeof(double) + sizeof(int));
  eval_dtw_kernel<<<B, kDtwThreads, smem, st>>>(p.cx, xlens, Lx_max, p.cy, ylens, Ly_max, n_cep, p.W, scale, mcd, cost, plen, p.dir,
                                                p.gA, p.gP);
  FS2_LAUNCH_CHECK();
  if (path) {
    FS2_CUDA_CHECK(cudaMemsetAsync(path, 0xff, (size_t)B * (Lx_max + Ly_max - 1) * 2 * sizeof(int32_t), st));
    eval_backtrack_kernel<<<(B + 63) / 64, 64, 0, st>>>(p.dir, xlens, Lx_max, ylens, Ly_max, B, p.W, plen, path);
    FS2_LAUNCH_CHECK();
  }
  return FS2_OK;
}

int fs2_path_prosody(const int32_t* path, const int64_t* plen, int B, int P_max, const double* f0x, const int64_t* f0x_lens, int Fx,
                     const double* f0y, const int64_t* f0y_lens, int Fy, const float* ex, int Ex, const float* ey, int Ey,
                     int64_t* counts, double* sums, int* status, void* stream) {
  FS2_REQUIRE(path && plen && f0x && f0x_lens && f0y && f0y_lens && ex && ey && counts && sums && status,
              "fs2_path_prosody: null argument");
  FS2_REQUIRE(B >= 1 && B <= (1 << 20) && P_max >= 1 && Fx >= 1 && Fy >= 1 && Ex >= 1 && Ey >= 1,
              "fs2_path_prosody: need 1 <= B <= 2^20 and P_max, Fx, Fy, Ex, Ey >= 1 (got %d, %d, %d, %d, %d, %d)", B, P_max, Fx, Fy, Ex,
              Ey);
  cudaStream_t st = (cudaStream_t)stream;
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  eval_prosody_kernel<<<(B + 63) / 64, 64, 0, st>>>(path, plen, B, P_max, f0x, f0x_lens, Fx, f0y, f0y_lens, Fy, ex, Ex, ey, Ey, counts, sums,
                                                     status);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // extern "C"
