// Batched MelGAN vocoder (DESIGN.md section 8): log-mels [B, Lmax, 80] -> audio [B, Lmax * 256], each utterance over its
// own olens[b] frames plus its 10 tail frames, on the library's tap-GEMM.
//
// Every layer is one GEMM over the rows of its stage, [B, Lp_s, C] with Lp_s = (Lmax + 10) * up_s (up = 1, 8, 64, 128,
// 256), run with TapGemm::lens = lens_s = (olens + 10) * up_s: row tiles wholly past an utterance are skipped and padded
// rows come out as exact zeros.  The GEMM's A operand is written by a producer kernel that does the index work the GEMM
// does not: reflection at each utterance's own edges, dilation, the leaky ReLU, and the taps laid side by side along K
// (operand planes in f16 / 3xF16, fp32 rows in fp32 / tf32):
//
//   pre_operand   (mel + 5) / 5 with the tail frames, reflect 3, 7 taps      -> GEMM 80*7 -> 512
//   taps (zero)   lrelu(x) at rows t-1, t, t+1                               -> GEMM 3 Cin -> s Cout: ConvTranspose1d
//                 (k = 2s, stride s, pad s/2) as a polyphase GEMM: output row t's s phases, written row-major, are rows
//                 s t .. s t + s - 1 of the next stage; phase r < s/2 reads rows {t-1, t}, r >= s/2 reads {t, t+1}, the
//                 third tap of each phase has zero weights
//   taps (reflect) lrelu(x) at rows t-d, t, t+d, reflected at the edges     -> GEMM 3C -> C        = h  (dilated conv)
//   concat        [lrelu(h) | x]                                             -> GEMM 2C -> C        = x' (1x1 conv + shortcut)
//   post          lrelu, reflect 3, conv 32 -> 1 (k = 7), tanh, trim to olens * 256 on CUDA cores, 0 past it
//
// A residual block runs either unfused (two producers and two tap-GEMMs: fp32, tf32, and the wide stages of f16 / 3xF16)
// or as one fused kernel (melgan_block_kernel: the narrow stages of f16 / 3xF16; fused_blocks() picks).  Launches per
// call: 3 + 4 * 2 + (stages unfused) * 12 + (stages fused) * 3 + 1: 60 in fp32 / tf32, 42 in 3xF16, 33 in f16.
// DESIGN.md section 8 gives the bounds and measured times of both routes.
//
// Rows past lens_s of a GEMM input are never written: a live tile reads them, but a GEMM output row depends only on its
// own input row and the epilogue stores 0 there.  Every producer reads rows of its own utterance below lens_s only, so
// per-utterance results do not depend on the batch.
//
// Windows (fs2_melgan_window, DESIGN.md section 11): the same kernels and GEMMs on a window of each utterance's rows.
// Every buffer then holds, per utterance, rows [start, start + len) of the utterance's n rows at its rate (a window
// descriptor [start | len | n] x B in the workspace; nullptr = the whole utterance, start 0 and len = n = lens[b]).
// Producers map a local row to its global row, reflect or zero-pad at the utterance's true edges, and read a source
// outside the window as 0: such rows lie in the halo and are discarded.  Only rows whose values equal the whole call's
// (all but `margin` rows at a window side that is not an utterance edge) are range-checked.
#include <math.h>
#include <string.h>

#include <algorithm>

#include "operand_planes.cuh"

namespace fs2 {
namespace {

constexpr int kMels = 80, kTail = 10, kPreTaps = 7, kPostTaps = 7, kPostC = 32, kStages = 4;
constexpr int kLayers = 42;                          // convolutions, in state_dict order
constexpr float kPadMel = -11.5129f;                 // value of the tail frames (seungwonpark/melgan `inference`)
constexpr int kCin[kStages] = {512, 256, 128, 64}, kCout[kStages] = {256, 128, 64, 32}, kStride[kStages] = {8, 8, 2, 2};


inline int grid_for(long n, int block, int cap = 132 * 8) {
  long g = (n + block - 1) / block;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

__host__ __device__ constexpr int upsampling(int s) { return s == 0 ? 1 : s == 1 ? 8 : s == 2 ? 64 : s == 3 ? 128 : 256; }
// ReflectionPad1d index map on [0, n) (edge sample not repeated); n exceeds every pad used here
__device__ __forceinline__ int reflect(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return i;
}
__device__ __forceinline__ float lrelu(float v) { return v > 0.f ? v : v * 0.2f; }
__device__ __forceinline__ float4 lrelu4(float4 v) { return make_float4(lrelu(v.x), lrelu(v.y), lrelu(v.z), lrelu(v.w)); }

// ---- window plan (DESIGN.md section 11) ----
// rows ConvTranspose s reads on each side of its core, at its input's rate: what the next ResStack (reach 13) and the
// layers after it need, divided by the stride, plus one row for the phases that read row t - 1 or t + 1
__host__ __device__ constexpr int reach(int s) { return s == 0 ? 3 : s == 1 ? 4 : s == 2 ? 12 : 9; }
__host__ __device__ constexpr int stride_of(int s) { return s < 2 ? 8 : 2; }        // kStride[s], usable on the device
constexpr int kResReach = 1 + 3 + 9, kPostReach = kPostTaps / 2;
// halo of buffer s on each side of its core: 3 first-conv rows (level 0), else stride * reach of the ConvTranspose that
// writes it; the ConvTranspose s input window is the level-s core +- reach(s)
__host__ __device__ constexpr int level_halo(int s) { return s == 0 ? reach(0) : stride_of(s - 1) * reach(s - 1); }
// rows per utterance of level s and of ConvTranspose s's input window, for n frames; level_rows(s + 1) = stride * convt_rows(s)
__host__ __device__ constexpr long level_rows(int s, long n) { return n * upsampling(s) + 2 * level_halo(s); }
__host__ __device__ constexpr long convt_rows(int s, long n) { return n * upsampling(s) + 2 * reach(s); }
// halo rows whose values differ from the whole call's at a window side that is not an utterance edge: ConvTranspose s's
// phases at its input window's edge read a row outside it, so level s + 1 starts with stride / 2 such rows; every residual
// block adds its dilation.  The next layer's input window must lie inside the exact rows:
__host__ __device__ constexpr int level_margin(int s) { return s == 0 ? 0 : stride_of(s - 1) / 2; }
constexpr bool plan_is_exact() {
  for (int s = 1; s <= kStages; ++s)
    if (level_margin(s) + kResReach > level_halo(s) - (s < kStages ? reach(s) : kPostReach)) return false;
  return level_margin(0) <= level_halo(0) - reach(0);
}
static_assert(plan_is_exact(), "a window's halo must cover every layer's reach");
// window descriptors of a window call: levels 0..4, ConvTranspose 1..3's input windows (ConvTranspose 0 reads all of
// level 0), and the audio samples [c0 * 256, c1 * 256)
constexpr int kWins = kStages + 1 + kStages - 1 + 1, kWinAudio = kWins - 1;
__host__ __device__ constexpr int convt_win(int s) { return s == 0 ? 0 : kStages + s; }

// rows of utterance b in a buffer (see the top of the file)
struct Rows { int start, len, n; };
__device__ __forceinline__ Rows rows_of(const int64_t* __restrict__ win, const int64_t* __restrict__ lens, int B, int b) {
  if (!win) {
    const int n = (int)lens[b];
    return {0, n, n};
  }
  return {(int)win[b], (int)win[B + b], (int)win[2 * B + b]};
}
// local row t holds the whole call's values: not within `margin` rows of a window side that is not an utterance edge
__device__ __forceinline__ bool exact_row(const Rows& r, int t, int margin) {
  return (r.start == 0 || t >= margin) && (r.start + r.len == r.n || t < r.len - margin);
}

// four GEMM-operand values at element offset off (a multiple of 4) of a [rows][K] operand; plane = rows * K; status ==
// nullptr: a halo row, not range-checked
template <int OUT>
__device__ __forceinline__ void store_quad(float4 v, long off, float* __restrict__ out32, __half* __restrict__ outp, long plane,
                                           int* __restrict__ status) {
  if (OUT == OUT_F32) {
    *reinterpret_cast<float4*>(out32 + off) = v;
    return;
  }
  if (status && !(fabsf(v.x) <= kPlaneMax && fabsf(v.y) <= kPlaneMax && fabsf(v.z) <= kPlaneMax && fabsf(v.w) <= kPlaneMax))
    atomicOr(status, FS2_MELGAN_RANGE);                 // saturation is reported, not hidden
  if (OUT == OUT_HILO) {
    uint2 hi, lo;
    split_pair(v.x, v.y, hi.x, lo.x);
    split_pair(v.z, v.w, hi.y, lo.y);
    *reinterpret_cast<uint2*>(outp + off) = hi;
    *reinterpret_cast<uint2*>(outp + plane + off) = lo;
  } else {
    *reinterpret_cast<uint2*>(outp + off) = make_uint2(hi_pair(v.x, v.y), hi_pair(v.z, v.w));
  }
}

// one CTA: lens[s][b] = (olens[b] + 10) * up_s for 1 <= olens[b] <= L, else 0 (the utterance is skipped); *status = 0 or
// FS2_MELGAN_BAD_LENGTH.  Runs first, so the producers' range bits land on a cleared word.
// starts != nullptr (a window of nf frames from starts[b]): lens = the kWins window descriptors instead, for the core
// frames [c0, c1) = [starts[b], min(starts[b] + nf, olens[b])); empty (len 0) when that is empty or the utterance is
// invalid, and FS2_MELGAN_BAD_START for starts[b] < 0.
__global__ void melgan_prep_kernel(const int64_t* __restrict__ olens, const int64_t* __restrict__ starts, int B, int L, int nf,
                                   int64_t* __restrict__ lens, int* __restrict__ status) {
  __shared__ int bad;
  if (threadIdx.x == 0) bad = 0;
  __syncthreads();
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const int64_t n = olens[b];
    const bool ok = n >= 1 && n <= L;
    if (!ok) atomicOr(&bad, FS2_MELGAN_BAD_LENGTH);
    if (!starts) {
      for (int s = 0; s <= kStages; ++s) lens[s * B + b] = ok ? (n + kTail) * upsampling(s) : 0;
      continue;
    }
    const int64_t c0 = starts[b];
    if (c0 < 0) atomicOr(&bad, FS2_MELGAN_BAD_START);
    const bool live = ok && c0 >= 0 && c0 < n;
    const int64_t c1 = live ? min(c0 + nf, n) : 0;
    auto put = [&](int w, int64_t lo, int64_t hi, int s) {
      int64_t* d = lens + 3L * w * B + b;
      d[0] = live ? lo : 0;
      d[B] = live ? hi - lo : 0;
      d[2 * B] = live ? (n + kTail) * upsampling(s) : 0;
    };
    put(0, max(c0 - reach(0), (int64_t)0), c1 + reach(0), 0);
    for (int s = 0; s < kStages; ++s) {
      const int64_t lo = max(c0 * upsampling(s) - reach(s), (int64_t)0), hi = c1 * upsampling(s) + reach(s);
      if (s > 0) put(convt_win(s), lo, hi, s);
      put(s + 1, lo * stride_of(s), hi * stride_of(s), s + 1);
    }
    put(kWinAudio, c0 * upsampling(kStages), c1 * upsampling(kStages), kStages);
  }
  __syncthreads();
  if (threadIdx.x == 0) *status = bad;
}

// first conv's operand [rows][7 * 80]: tap j of row t = (m + 5) / 5 at frame reflect(t + j - 3), m = the mel frame below
// olens[b] or the tail value.  Frames past olens[b] are never read (NaN there changes nothing).  A window (win) reads the
// frames its rows reach only.
template <int OUT>
__global__ void melgan_pre_operand_kernel(const float* __restrict__ mels, const int64_t* __restrict__ lens, const int64_t* __restrict__ win,
                                          int B, int L, int Lp, float* __restrict__ out32, __half* __restrict__ outp, int* __restrict__ status) {
  constexpr int K = kMels * kPreTaps, Q = K / 4;
  const long rows = (long)B * Lp, total = rows * Q, plane = rows * K;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / Q;
    const int k = (int)(i - row * Q) * 4, j = k / kMels, c = k - j * kMels;
    const int b = (int)(row / Lp), t = (int)(row - (long)b * Lp);
    const Rows r = rows_of(win, lens, B, b);
    if (t >= r.len) continue;
    const int src = reflect(r.start + t + j - kPreTaps / 2, r.n);
    float4 v = make_float4(kPadMel, kPadMel, kPadMel, kPadMel);
    if (src < r.n - kTail) v = *reinterpret_cast<const float4*>(mels + ((long)b * L + src) * kMels + c);
    v = make_float4((v.x + 5.f) / 5.f, (v.y + 5.f) / 5.f, (v.z + 5.f) / 5.f, (v.w + 5.f) / 5.f);
    store_quad<OUT>(v, row * K + k, out32, outp, plane, status);
  }
}

// three-tap operand [rows][3C]: tap j of row t = lrelu(x[t + (j - 1) d]); outside [0, n) the row is reflected (REFLECT:
// the dilated convolutions) or zero (the transposed convolutions, d = 1).  x has ldx rows per utterance in its own
// window xwin (nullptr: the operand's rows, ldx = Lp); a source outside it reads as 0.  The loop is bound by its index
// work, so whole utterances (win == nullptr) run a loop compiled without the window's (WINDOW = false).
template <int OUT, bool REFLECT, bool WINDOW>
__device__ __forceinline__ void taps_loop(const float* __restrict__ x, const int64_t* __restrict__ xwin, int ldx, const int64_t* __restrict__ lens,
                                          const int64_t* __restrict__ win, int B, int Lp, int C, int d, int margin, float* __restrict__ out32,
                                          __half* __restrict__ outp, int* __restrict__ status) {
  const int K = 3 * C, Q = K / 4;
  const long rows = (long)B * Lp, total = rows * Q, plane = rows * K;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / Q;
    const int k = (int)(i - row * Q) * 4, j = k / C, c = k - j * C;
    const int b = (int)(row / Lp), t = (int)(row - (long)b * Lp);
    const Rows r = rows_of(WINDOW ? win : nullptr, lens, B, b);
    if (t >= r.len) continue;
    int src = r.start + t + (j - 1) * d;
    if (REFLECT) src = reflect(src, r.n);
    bool in = src >= 0 && src < r.n;
    if (WINDOW) {
      const Rows xr = xwin ? rows_of(xwin, lens, B, b) : r;
      src -= xr.start;
      in = in && src >= 0 && src < xr.len;
    }
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (in) v = lrelu4(*reinterpret_cast<const float4*>(x + ((long)b * ldx + src) * C + c));
    store_quad<OUT>(v, row * K + k, out32, outp, plane, !WINDOW || exact_row(r, t, margin) ? status : nullptr);
  }
}

template <int OUT, bool REFLECT>
__global__ void melgan_taps_kernel(const float* __restrict__ x, const int64_t* __restrict__ xwin, int ldx, const int64_t* __restrict__ lens,
                                   const int64_t* __restrict__ win, int B, int Lp, int C, int d, int margin, float* __restrict__ out32,
                                   __half* __restrict__ outp, int* __restrict__ status) {
  if (win) taps_loop<OUT, REFLECT, true>(x, xwin, ldx, lens, win, B, Lp, C, d, margin, out32, outp, status);
  else taps_loop<OUT, REFLECT, false>(x, xwin, ldx, lens, win, B, Lp, C, d, margin, out32, outp, status);
}

// operand [rows][2C] = [lrelu(h) | x] of the fused 1x1 GEMM [W2 | Ws]
template <int OUT>
__global__ void melgan_concat_kernel(const float* __restrict__ h, const float* __restrict__ x, const int64_t* __restrict__ lens,
                                     const int64_t* __restrict__ win, int B, int Lp, int C, int margin, float* __restrict__ out32,
                                     __half* __restrict__ outp, int* __restrict__ status) {
  const int K = 2 * C, Q = K / 4;
  const long rows = (long)B * Lp, total = rows * Q, plane = rows * K;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / Q;
    const int k = (int)(i - row * Q) * 4;
    const int b = (int)(row / Lp), t = (int)(row - (long)b * Lp);
    const Rows r = rows_of(win, lens, B, b);
    if (t >= r.len) continue;
    const float4 v = k < C ? lrelu4(*reinterpret_cast<const float4*>(h + row * C + k)) : *reinterpret_cast<const float4*>(x + row * C + k - C);
    store_quad<OUT>(v, row * K + k, out32, outp, plane, exact_row(r, t, margin) ? status : nullptr);
  }
}

// ---- fused residual block (f16 / 3xF16): one kernel per block, h never leaves the registers ----------------------------
// mma.sync m16n8k16 (f16 operands, fp32 accumulators).  Fragment layout, g = lane / 4, q = lane % 4: A a0 (row g, cols
// 2q, 2q+1), a1 (row g+8, same cols), a2 / a3 (cols 2q+8, 2q+9); B b0 (k = 2q, 2q+1; n = g), b1 (k = 2q+8, 2q+9);
// D d0, d1 (row g, cols 2q, 2q+1), d2, d3 (row g+8).  So the D tiles n8 = 2kc, 2kc+1 of one GEMM are exactly the A
// fragment of K chunk kc of the next one.
__device__ __forceinline__ void mma_f16(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// two values -> hi (and lo) fp16 pairs of (v * kPlaneScale), with the plane range check
template <bool PRECISE>
__device__ __forceinline__ void to_planes(float a, float b, uint32_t& hi, uint32_t& lo, bool& bad) {
  bad |= !(fabsf(a) <= kPlaneMax && fabsf(b) <= kPlaneMax);
  if (PRECISE) split_pair(a, b, hi, lo);
  else hi = hi_pair(a, b);
}

// D (+)= A . B^T for one n8 tile: 3xF16 as lo.hi + hi.lo + hi.hi (small terms first), f16 as hi.hi
template <bool PRECISE>
__device__ __forceinline__ void mma_tile(float* d, const uint32_t* ah, const uint32_t* al, const __half* __restrict__ wh,
                                         const __half* __restrict__ wl, long off) {
  const uint32_t bh0 = __ldg(reinterpret_cast<const unsigned int*>(wh + off)), bh1 = __ldg(reinterpret_cast<const unsigned int*>(wh + off + 8));
  if (PRECISE) {
    const uint32_t bl0 = __ldg(reinterpret_cast<const unsigned int*>(wl + off)), bl1 = __ldg(reinterpret_cast<const unsigned int*>(wl + off + 8));
    mma_f16(d, al, bh0, bh1);
    mma_f16(d, ah, bl0, bl1);
  }
  mma_f16(d, ah, bh0, bh1);
}

// One residual block, x' = [W2 | Ws] . [lrelu(h) | x] + (b2 + bs) with h = W1 . taps(lrelu(x)) + b1 (dilation d, reflected
// at the utterance's edges).  A warp owns 16 rows: it builds the A fragments of the dilated conv straight from the fp32
// rows of x (reflect, lrelu, split into planes in registers), keeps h's accumulators in registers, turns them into the A
// fragments of the 1x1 GEMM (bias, lrelu, split), adds the shortcut's K half from x, and writes x' in fp32 (0 past the
// utterance).  Weights are the packed [N][K] planes of the unfused route, read through L1.  A row's result depends on its
// own utterance's rows only, in a fixed K order.  win / margin: as in melgan_taps_kernel; a row's range bits count only
// where exact_row holds.
template <int C, bool PRECISE>
__global__ void __launch_bounds__(C == 256 ? 64 : 128, 1) melgan_block_kernel(const float* __restrict__ x, const int64_t* __restrict__ lens,
                                                           const int64_t* __restrict__ win, int B, int Lp, int d, int margin,
                                                           const __half* __restrict__ w1h, const __half* __restrict__ w1l,
                                                           const float* __restrict__ w1inv, const float* __restrict__ b1,
                                                           const __half* __restrict__ w2h, const __half* __restrict__ w2l,
                                                           const float* __restrict__ w2inv, const float* __restrict__ b2,
                                                           float* __restrict__ out, int* __restrict__ status) {
  // C = 256: h's A fragments go to shared memory (in fragment order, each thread reads back what it wrote), so that h's
  // accumulators and the 1x1 GEMM's do not have to be live together; two warps per CTA keep that at 32 KB
  constexpr bool HS = C == 256;
  constexpr int WARPS = HS ? 2 : 4, NT = C / 8, K1 = 3 * C, K2 = 2 * C, NG = HS ? 32 : (C < 64 ? C : 64);
  __shared__ uint32_t hs[HS ? WARPS * (C / 16) * 8 * 32 : 1];
  const int lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3, warp = threadIdx.x >> 5;
  const long rows = (long)B * Lp, m0 = ((long)blockIdx.x * WARPS + warp) * 16;
  if (m0 >= rows) return;
  long base[2]; int t[2], o[2], n[2], len[2]; bool live[2], chk[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const long m = m0 + g + 8 * h;
    const bool in = m < rows;
    const int b = in ? (int)(m / Lp) : 0;
    const Rows r = in ? rows_of(win, lens, B, b) : Rows{0, 0, 0};
    t[h] = in ? (int)(m - (long)b * Lp) : 0;
    o[h] = r.start; n[h] = r.n; len[h] = r.len;
    base[h] = (long)b * Lp;
    live[h] = in && t[h] < r.len;
    chk[h] = live[h] && exact_row(r, t[h], margin);
  }
  const bool any = __any_sync(0xffffffffu, live[0] || live[1]);
  bool bad[2] = {false, false};     // per row half; counted where chk
  if (any) {
    const float s1 = kPlaneInv * __ldg(w1inv), s2 = kPlaneInv * __ldg(w2inv);
    float acc[NT][4];
#pragma unroll
    for (int i = 0; i < NT; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    // ---- h = W1 . [lrelu(x[t-d]) | lrelu(x[t]) | lrelu(x[t+d])] ----
#pragma unroll 1
    for (int kk = 0; kk < K1 / 16; ++kk) {
      const int k0 = kk * 16, j = k0 / C, c0 = k0 - j * C;
      uint32_t ah[4], al[4];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float2 v0 = make_float2(0.f, 0.f), v1 = v0;
        const int src = reflect(o[h] + t[h] + (j - 1) * d, n[h]) - o[h];
        if (live[h] && src >= 0 && src < len[h]) {
          const float* r = x + (base[h] + src) * C + c0 + 2 * q;
          v0 = *reinterpret_cast<const float2*>(r);
          v1 = *reinterpret_cast<const float2*>(r + 8);
        }
        to_planes<PRECISE>(lrelu(v0.x), lrelu(v0.y), ah[h], al[h], bad[h]);
        to_planes<PRECISE>(lrelu(v1.x), lrelu(v1.y), ah[h + 2], al[h + 2], bad[h]);
      }
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) mma_tile<PRECISE>(acc[nt], ah, al, w1h, w1l, (long)(nt * 8 + g) * K1 + k0 + 2 * q);
    }
    // lrelu(h + b1) as the A fragments of K chunk kc of the 1x1 GEMM: D tile 2kc + hf -> registers 2hf, 2hf + 1
    auto h_frags = [&](int kc, uint32_t* ah, uint32_t* al) {
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        const float* a = acc[2 * kc + hf];
        const int col = 16 * kc + 8 * hf + 2 * q;
        const float bb0 = __ldg(b1 + col), bb1 = __ldg(b1 + col + 1);
        to_planes<PRECISE>(lrelu(fmaf(a[0], s1, bb0)), lrelu(fmaf(a[1], s1, bb1)), ah[2 * hf], al[2 * hf], bad[0]);
        to_planes<PRECISE>(lrelu(fmaf(a[2], s1, bb0)), lrelu(fmaf(a[3], s1, bb1)), ah[2 * hf + 1], al[2 * hf + 1], bad[1]);
      }
    };
    uint32_t* hw = hs + warp * (C / 16) * 8 * 32 + lane;
    if (HS) {
#pragma unroll
      for (int kc = 0; kc < C / 16; ++kc) {
        uint32_t ah[4], al[4];
        h_frags(kc, ah, al);
#pragma unroll
        for (int r = 0; r < 4; ++r) { hw[(kc * 8 + r) * 32] = ah[r]; hw[(kc * 8 + 4 + r) * 32] = al[r]; }
      }
    }
    // ---- x' = [W2 | Ws] . [lrelu(h) | x] + bias, NG output columns at a time ----
#pragma unroll 1
    for (int n0 = 0; n0 < C; n0 += NG) {
      float o[NG / 8][4];
#pragma unroll
      for (int i = 0; i < NG / 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
#pragma unroll HS ? 1 : C / 16
      for (int kc = 0; kc < C / 16; ++kc) {
        uint32_t ah[4], al[4];
        if (HS) {
#pragma unroll
          for (int r = 0; r < 4; ++r) { ah[r] = hw[(kc * 8 + r) * 32]; al[r] = hw[(kc * 8 + 4 + r) * 32]; }
        } else {
          h_frags(kc, ah, al);
        }
#pragma unroll
        for (int nt = 0; nt < NG / 8; ++nt) mma_tile<PRECISE>(o[nt], ah, al, w2h, w2l, (long)(n0 + nt * 8 + g) * K2 + 16 * kc + 2 * q);
      }
#pragma unroll 1
      for (int kc = 0; kc < C / 16; ++kc) {
        uint32_t ah[4], al[4];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float2 v0 = make_float2(0.f, 0.f), v1 = v0;
          if (live[h]) {
            const float* r = x + (base[h] + t[h]) * C + 16 * kc + 2 * q;
            v0 = *reinterpret_cast<const float2*>(r);
            v1 = *reinterpret_cast<const float2*>(r + 8);
          }
          to_planes<PRECISE>(v0.x, v0.y, ah[h], al[h], bad[h]);
          to_planes<PRECISE>(v1.x, v1.y, ah[h + 2], al[h + 2], bad[h]);
        }
#pragma unroll
        for (int nt = 0; nt < NG / 8; ++nt) mma_tile<PRECISE>(o[nt], ah, al, w2h, w2l, (long)(n0 + nt * 8 + g) * K2 + C + 16 * kc + 2 * q);
      }
#pragma unroll
      for (int nt = 0; nt < NG / 8; ++nt) {
        const int col = n0 + nt * 8 + 2 * q;
        const float bb0 = __ldg(b2 + col), bb1 = __ldg(b2 + col + 1);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long m = m0 + g + 8 * h;
          if (m >= rows) continue;
          const float2 v = live[h] ? make_float2(fmaf(o[nt][2 * h], s2, bb0), fmaf(o[nt][2 * h + 1], s2, bb1)) : make_float2(0.f, 0.f);
          *reinterpret_cast<float2*>(out + m * C + col) = v;
        }
      }
    }
  } else {
    for (int h = 0; h < 2; ++h) {
      const long m = m0 + g + 8 * h;
      if (m >= rows) continue;
      for (int c = 2 * q; c < C; c += 8) *reinterpret_cast<float2*>(out + m * C + c) = make_float2(0.f, 0.f);
    }
  }
  const bool flag = (bad[0] && chk[0]) || (bad[1] && chk[1]);
  if (__any_sync(0xffffffffu, flag) && lane == 0) atomicOr(status, FS2_MELGAN_RANGE);   // saturation is reported, not hidden
}

// audio[b, t] = tanh(bias + sum_j sum_c w[j][c] lrelu(x[reflect(t + j - 3)][c])) for t < olens[b] * 256, else 0; rows of
// audio ld samples apart.  A window: x in window win, and audio row b holds samples [start, start + len) of awin (0 past them).
__global__ void __launch_bounds__(256) melgan_post_kernel(const float* __restrict__ x, const int64_t* __restrict__ lens,
                                                          const int64_t* __restrict__ win, const int64_t* __restrict__ awin, int B, int Lp,
                                                          int Lout, long ld, const float* __restrict__ w, const float* __restrict__ bias,
                                                          float* __restrict__ audio) {
  __shared__ __align__(16) float ws[kPostTaps * kPostC];
  for (int i = threadIdx.x; i < kPostTaps * kPostC; i += blockDim.x) ws[i] = w[i];
  __syncthreads();
  const float b0 = __ldg(bias);
  const long total = (long)B * Lout;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int b = (int)(i / Lout), t = (int)(i - (long)b * Lout);
    const Rows r = rows_of(win, lens, B, b);
    const int a0 = awin ? (int)awin[b] : 0, alen = awin ? (int)awin[B + b] : r.n - kTail * upsampling(kStages);
    float y = 0.f;
    if (t < alen) {
      float acc = b0;
#pragma unroll
      for (int j = 0; j < kPostTaps; ++j) {
        const float4* r4 = reinterpret_cast<const float4*>(x + ((long)b * Lp + reflect(a0 + t + j - kPostTaps / 2, r.n) - r.start) * kPostC);
#pragma unroll
        for (int q = 0; q < kPostC / 4; ++q) {
          const float4 v = lrelu4(__ldg(r4 + q));
          const float4 wv = *reinterpret_cast<const float4*>(ws + j * kPostC + 4 * q);
          acc = fmaf(wv.x, v.x, acc); acc = fmaf(wv.y, v.y, acc); acc = fmaf(wv.z, v.z, acc); acc = fmaf(wv.w, v.w, acc);
        }
      }
      y = tanhf(acc);
    }
    audio[(long)b * ld + t] = y;
  }
}

// GEMM weight [N][K] from a folded torch-layout weight:
//   kind 0  Conv1d w [N][Cin][taps]              -> dst[n][j Cin + c] = w[n][c][j]
//   kind 1  ConvTranspose1d w [Cin][Cout][2s]    -> dst[r Cout + co][j Cin + ci] = w[ci][co][k(r, j)] (0 where phase r
//           does not read input row t + j - 1): k = r + s/2 + s for j = 0, r + s/2 for j = 1 (r < s/2); r + s/2 - s for
//           j = 2, r + s/2 for j = 1 (r >= s/2)
//   kind 2  [W2 | Ws], both [N][Cin][1]           -> dst[n][c] = W2[n][c], dst[n][Cin + c] = Ws[n][c]
__global__ void melgan_pack_kernel(int kind, const float* __restrict__ w, const float* __restrict__ w2, int N, int K, int Cin, int Cout,
                                   int taps, int s, float* __restrict__ dst) {
  const long total = (long)N * K;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int n = (int)(i / K), k = (int)(i - (long)n * K);
    float v;
    if (kind == 0) {
      const int j = k / Cin, c = k - j * Cin;
      v = w[((long)n * Cin + c) * taps + j];
    } else if (kind == 1) {
      const int r = n / Cout, co = n - r * Cout, j = k / Cin, ci = k - j * Cin, p = s / 2;
      const int kk = r < p ? (j == 1 ? r + p : j == 0 ? r + p + s : -1) : (j == 2 ? r + p - s : j == 1 ? r + p : -1);
      v = kk >= 0 ? w[((long)ci * Cout + co) * (2 * s) + kk] : 0.f;
    } else {
      v = k < Cin ? w[(long)n * Cin + k] : w2[(long)n * Cin + k - Cin];
    }
    dst[i] = v;
  }
}

// dst[n] = b[n % Cout] (+ b2[n])
__global__ void melgan_bias_kernel(const float* __restrict__ b, const float* __restrict__ b2, int N, int Cout, float* __restrict__ dst) {
  for (int n = blockIdx.x * blockDim.x + threadIdx.x; n < N; n += gridDim.x * blockDim.x)
    dst[n] = b2 ? b[n] + b2[n] : b[n % Cout];
}

struct MWeight {               // one GEMM weight [N][K]: fp32 (fp32 / tf32 families) and scaled fp16 planes, bias [N]
  float* w = nullptr; __half* hi = nullptr; __half* lo = nullptr; float* sc = nullptr; float* bias = nullptr;   // sc = [scale, 1 / scale]
  int N = 0, K = 0;
};

struct Bump {
  char* base; size_t off = 0, cap;
  Bump(void* b, size_t c) : base((char*)b), cap(c) {}
  void* bytes(size_t n) { size_t a = (off + 255) & ~(size_t)255; off = a + n; return base ? base + a : nullptr; }
  float* floats(size_t n) { return (float*)bytes(n * sizeof(float)); }
  bool ok() const { return base == nullptr || off <= cap; }
};

}  // namespace
}  // namespace fs2

struct fs2_melgan_gen {
  int device = 0, math_mode = 0;
  bool loaded = false;
  void* arena = nullptr;
  fs2::MWeight pre, up[fs2::kStages], dil[fs2::kStages][3], pair[fs2::kStages][3];
  float* post_w = nullptr;     // [7][32]
  float* post_b = nullptr;
};

namespace fs2 {
namespace {

struct MgPlan {
  int64_t* lens;     // [5][B]; a window call: the kWins window descriptors [start | len | n][B]
  void* a;           // GEMM operand, up to rows * 3C of the widest stage
  float* x[2];       // activations [rows][C], ping-pong
  float* h;          // dilated conv output [rows][C] (unfused route only)
};

// A window call's workspace, from B and nf only: per utterance, the largest operand (rows x K over every producer) and
// the largest activation (rows x C over every level) of the window's buffers
MgPlan window_plan(Bump& b, int B, int nf) {
  long op = level_rows(0, nf) * kMels * kPreTaps, act = level_rows(0, nf) * 512;
  for (int s = 0; s < kStages; ++s) {
    op = std::max(op, std::max(convt_rows(s, nf) * 3 * kCin[s], level_rows(s + 1, nf) * 3 * kCout[s]));
    act = std::max(act, level_rows(s + 1, nf) * kCout[s]);
  }
  MgPlan p;
  p.lens = (int64_t*)b.bytes((size_t)3 * kWins * B * sizeof(int64_t));
  p.a = b.floats((size_t)B * op);
  p.x[0] = b.floats((size_t)B * act);
  p.x[1] = b.floats((size_t)B * act);
  p.h = b.floats((size_t)B * act);
  return p;
}

// per frame of Lp: values of the largest operand (3C at the three late stages, 24576) and activation (8192)
constexpr long kOperandPerFrame = 3L * 256 * 32, kActPerFrame = 256L * 32;

MgPlan plan(Bump& b, int B, int L, bool fused) {
  const size_t frames = (size_t)B * (L + kTail);
  MgPlan p;
  p.lens = (int64_t*)b.bytes((size_t)(kStages + 1) * B * sizeof(int64_t));
  p.a = b.floats(frames * kOperandPerFrame);
  p.x[0] = b.floats(frames * kActPerFrame);
  p.x[1] = b.floats(frames * kActPerFrame);
  p.h = fused ? nullptr : b.floats(frames * kActPerFrame);
  return p;
}



// one GEMM weight from its torch-layout tensors (melgan_pack_kernel's kind, Cin, Cout, taps, s): the packed fp32 [N][K],
// the bias [N], the power-of-two scale and the fp16 planes; w->N, w->K and the buffers are set by the caller
int pack_weight(MWeight* w, int kind, const float* wt, const float* wt2, const float* b, const float* b2, int Cin, int Cout, int taps,
                int s, cudaStream_t st) {
  const long n = (long)w->N * w->K;
  melgan_pack_kernel<<<grid_for(n, 256), 256, 0, st>>>(kind, wt, wt2, w->N, w->K, Cin, Cout, taps, s, w->w);
  FS2_LAUNCH_CHECK();
  melgan_bias_kernel<<<grid_for(w->N, 256), 256, 0, st>>>(b, b2, w->N, Cout, w->bias);
  FS2_LAUNCH_CHECK();
  int rc = weight_scale(w->w, n, w->sc, w->sc + 1, st); if (rc) return rc;
  return split_f16(w->w, w->hi, w->lo, n, w->sc, st);
}

// carves one MWeight of N x K out of a Bump
void carve(Bump& b, MWeight* w, int N, int K) {
  w->N = N; w->K = K;
  const size_t n = (size_t)N * K;
  w->w = b.floats(n); w->hi = (__half*)b.bytes(n * 2); w->lo = (__half*)b.bytes(n * 2); w->sc = b.floats(2); w->bias = b.floats(N);
}

// out [B * Lp][w.N] = a [B * Lp][w.K] . w^T + bias, rows t >= lens[b] written as 0 (and skipped by the tensor-core kernel)
int gemm(int mode, const MWeight& w, const void* a, int B, int Lp, const int64_t* lens, float* out, cudaStream_t st) {
  TapGemm g;
  memset(&g, 0, sizeof(g));
  g.B = B; g.L = Lp; g.K = w.K; g.N = w.N; g.taps = 1; g.act = ACT_NONE; g.out = out; g.ldo = w.N; g.lens = lens;
  g.w = w.w; g.bias = w.bias; g.a_inv = 1.0f; g.ldx = w.K;
  if (mode == FS2_MATH_FP32 || mode == FS2_MATH_TF32) {
    g.x = (const float*)a;
    return mode == FS2_MATH_FP32 ? tap_gemm_fp32(g, st) : tap_gemm_tf32(g, st);
  }
  g.xp = (const __half*)a; g.w_hi = w.hi; g.w_lo = w.lo; g.w_inv = w.sc + 1; g.a_inv = kPlaneInv;
  g.precise = mode == FS2_MATH_3XTF32;
  return tap_gemm_planes(g, st);
}

// the taps producer: operand rows [B * Lp] (window win, lens) from x, ldx rows per utterance in window xwin (nullptr: the
// operand's own rows, ldx = Lp); margin: see exact_row
int run_taps(int kind, bool reflect_edges, const float* x, const int64_t* xwin, int ldx, const int64_t* lens, const int64_t* win, int B,
             int Lp, int C, int d, int margin, void* out, int* status, cudaStream_t st) {
  auto k = reflect_edges ? pick(kind, melgan_taps_kernel<OUT_HILO, true>, melgan_taps_kernel<OUT_HI, true>, melgan_taps_kernel<OUT_F32, true>)
                         : pick(kind, melgan_taps_kernel<OUT_HILO, false>, melgan_taps_kernel<OUT_HI, false>, melgan_taps_kernel<OUT_F32, false>);
  k<<<grid_for((long)B * Lp * (3 * C / 4), 256), 256, 0, st>>>(x, xwin, ldx, lens, win, B, Lp, C, d, margin, (float*)out, (__half*)out, status);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// Which route a residual block of C channels takes.  fp32 / tf32: producers + tap-GEMMs.  f16 / 3xF16: the fused
// mma.sync kernel where it measured faster than producers + the wgmma tap-GEMM (H100, filelist64, DESIGN.md section 8):
// C <= 128 in f16, C <= 64 in 3xF16.  At C = 256 (and 128 in 3xF16) the fused kernel's per-warp weight fragments cost
// more than the unfused route's HBM round trips.
bool fused_blocks(int mode, int C) {
  return (mode == FS2_MATH_F16 && C <= 128) || (mode == FS2_MATH_3XTF32 && C <= 64);
}

template <int C>
int run_block(int mode, const MWeight& w1, const MWeight& w2, const float* x, const int64_t* lens, const int64_t* win, int B, int Lp, int d,
              int margin, float* out, int* status, cudaStream_t st) {
  constexpr int warps = C == 256 ? 2 : 4;          // as in melgan_block_kernel: 16 rows per warp
  const long rows = (long)B * Lp, ctas = (rows + 16 * warps - 1) / (16 * warps);
  FS2_REQUIRE(ctas < (1L << 31), "fs2_melgan: too many rows (%ld)", rows);
  auto k = mode == FS2_MATH_3XTF32 ? melgan_block_kernel<C, true> : melgan_block_kernel<C, false>;
  k<<<(unsigned)ctas, 32 * warps, 0, st>>>(x, lens, win, B, Lp, d, margin, w1.hi, w1.lo, w1.sc + 1, w1.bias, w2.hi, w2.lo, w2.sc + 1, w2.bias, out, status);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// One residual block x -> out on [B * Lp][C] rows (dilation d, w1 = the dilated conv, w2 = [W2 | Ws]): the fused kernel
// (f16 / 3xF16, C in {32, 64, 128, 256}), or producers + tap-GEMMs through the scratch operand a (rows * 3C floats) and h
// (rows * C floats).  win, margin: the rows' window and its halo rows after this block (see exact_row).
int res_block(int mode, bool fused, const MWeight& w1, const MWeight& w2, const float* x, const int64_t* lens, const int64_t* win, int B,
              int Lp, int C, int d, int margin, void* a, float* h, float* out, int* status, cudaStream_t st) {
  if (fused) {
    return C == 256 ? run_block<256>(mode, w1, w2, x, lens, win, B, Lp, d, margin, out, status, st)
         : C == 128 ? run_block<128>(mode, w1, w2, x, lens, win, B, Lp, d, margin, out, status, st)
         : C == 64  ? run_block<64>(mode, w1, w2, x, lens, win, B, Lp, d, margin, out, status, st)
                    : run_block<32>(mode, w1, w2, x, lens, win, B, Lp, d, margin, out, status, st);
  }
  const int kind = out_kind(mode);
  int rc = run_taps(kind, true, x, nullptr, Lp, lens, win, B, Lp, C, d, margin, a, status, st);
  if (rc || (rc = gemm(mode, w1, a, B, Lp, lens, h, st))) return rc;
  auto concat = pick(kind, melgan_concat_kernel<OUT_HILO>, melgan_concat_kernel<OUT_HI>, melgan_concat_kernel<OUT_F32>);
  concat<<<grid_for((long)B * Lp * (2 * C / 4), 256), 256, 0, st>>>(h, x, lens, win, B, Lp, C, margin, (float*)a, (__half*)a, status);
  FS2_LAUNCH_CHECK();
  return gemm(mode, w2, a, B, Lp, lens, out, st);
}

// lrelu + ConvTranspose1d (k = 2s, stride s, pad s/2) x [B * Lin][Cin] -> out [B * Lin][s Cout] = [B * Lin * s][Cout], through
// the scratch operand a (rows * 3 Cin floats): rows t < lens[b] of x in, rows >= lens[b] * s of out written as 0.  A window:
// the input window (win, lens; Lin rows per utterance) is read from x's own window xwin of ldx rows per utterance.
int upsample(int mode, const MWeight& w, const float* x, const int64_t* xwin, int ldx, const int64_t* lens, const int64_t* win, int B, int Lin,
             int Cin, void* a, float* out, int* status, cudaStream_t st) {
  int rc = run_taps(out_kind(mode), false, x, xwin, ldx, lens, win, B, Lin, Cin, 1, 1, a, status, st);
  return rc ? rc : gemm(mode, w, a, B, Lin, lens, out, st);
}

// The generator on the plan p: whole utterances (starts == nullptr; every buffer (Lmax + 10) * up_s rows per utterance,
// lens [5][B]) or a window of nf frames from starts[b] (level_rows / convt_rows per utterance, the kWins window
// descriptors).  Lout audio samples per row, rows ld apart.  Both enqueue the same kernels.
int generate(const fs2_melgan_gen* m, const MgPlan& p, const float* mels, const int64_t* olens, const int64_t* starts, int B, int Lmax,
             int nf, float* audio, long ld, int* status, cudaStream_t st) {
  const bool w = starts != nullptr;
  const int mode = m->math_mode, kind = out_kind(mode);
  auto desc = [&](int i) -> const int64_t* { return w ? p.lens + 3L * i * B : nullptr; };
  auto lens = [&](int i, int s) -> const int64_t* { return w ? p.lens + (3L * i + 1) * B : p.lens + (long)s * B; };   // window i / level s
  auto rows = [&](int s) { return w ? (int)level_rows(s, nf) : (Lmax + kTail) * upsampling(s); };
  int rc;
  melgan_prep_kernel<<<1, 256, 0, st>>>(olens, starts, B, Lmax, nf, p.lens, status);
  FS2_LAUNCH_CHECK();
  {
    auto k = pick(kind, melgan_pre_operand_kernel<OUT_HILO>, melgan_pre_operand_kernel<OUT_HI>, melgan_pre_operand_kernel<OUT_F32>);
    k<<<grid_for((long)B * rows(0) * (kMels * kPreTaps / 4), 256), 256, 0, st>>>(mels, lens(0, 0), desc(0), B, Lmax, rows(0), (float*)p.a,
                                                                                (__half*)p.a, status);
    FS2_LAUNCH_CHECK();
  }
  if ((rc = gemm(mode, m->pre, p.a, B, rows(0), lens(0, 0), p.x[0], st))) return rc;
  int cur = 0;
  for (int s = 0; s < kStages; ++s) {
    const int C = kCout[s], cw = convt_win(s), Lin = w ? (int)convt_rows(s, nf) : rows(s);
    // lrelu, ConvTranspose1d: [B * Lin][s Cout] row-major is [B * Lout][Cout]
    if ((rc = upsample(mode, m->up[s], p.x[cur], desc(s), rows(s), lens(cw, s), desc(cw), B, Lin, kCin[s], p.a, p.x[cur ^ 1], status, st)))
      return rc;
    cur ^= 1;
    int margin = level_margin(s + 1);
    for (int i = 0, d = 1; i < 3; ++i, d *= 3) {
      margin += d;
      if ((rc = res_block(mode, fused_blocks(mode, C), m->dil[s][i], m->pair[s][i], p.x[cur], lens(s + 1, s + 1), desc(s + 1), B, rows(s + 1),
                          C, d, margin, p.a, p.h, p.x[cur ^ 1], status, st)))
        return rc;
      cur ^= 1;
    }
  }
  const int Lout = (w ? nf : Lmax) * upsampling(kStages);
  melgan_post_kernel<<<grid_for((long)B * Lout, 256), 256, 0, st>>>(p.x[cur], lens(kStages, kStages), desc(kStages), desc(kWinAudio), B,
                                                                   rows(kStages), Lout, ld, m->post_w, m->post_b, audio);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int check_size(const fs2_melgan_gen* m, int B, int L) {
  FS2_REQUIRE(B >= 1 && L >= 1, "fs2_melgan: need B >= 1 and Lmax >= 1 (got %d, %d)", B, L);
  const long samples = (long)B * (L + kTail) * upsampling(kStages);
  FS2_REQUIRE(samples < (1L << 31), "fs2_melgan: B * (Lmax + 10) * 256 = %ld sample rows exceed the int32 row index", samples);
  // the CUDA-core GEMM puts row tiles of 128 on grid.y (at most 65535)
  FS2_REQUIRE(m->math_mode != FS2_MATH_FP32 || samples <= 65535L * 128,
              "fs2_melgan: B * (Lmax + 10) * 256 = %ld sample rows exceed fp32 mode's limit of %ld", samples, 65535L * 128);
  return FS2_OK;
}

// a window's limits apply to its rows: the largest buffer, level 4, has B * level_rows(4, nf) rows
int check_window(const fs2_melgan_gen* m, int B, int nf) {
  FS2_REQUIRE(B >= 1 && nf >= 1, "fs2_melgan_window: need B >= 1 and n_frames >= 1 (got %d, %d)", B, nf);
  const long rows = (long)B * level_rows(kStages, nf);
  FS2_REQUIRE(rows < (1L << 31), "fs2_melgan_window: B * (256 * n_frames + 36) = %ld window rows exceed the int32 row index", rows);
  FS2_REQUIRE(m->math_mode != FS2_MATH_FP32 || rows <= 65535L * 128,
              "fs2_melgan_window: B * (256 * n_frames + 36) = %ld window rows exceed fp32 mode's limit of %ld", rows, 65535L * 128);
  return FS2_OK;
}

}  // namespace
}  // namespace fs2

using namespace fs2;

extern "C" {

int fs2_melgan_create(fs2_melgan_gen** out, int math_mode) {
  FS2_REQUIRE(out, "fs2_melgan_create: null argument");
  FS2_REQUIRE(math_mode >= FS2_MATH_FP32 && math_mode <= FS2_MATH_F16, "fs2_melgan_create: bad math_mode %d", math_mode);
  fs2_melgan_gen* m = new fs2_melgan_gen();
  m->math_mode = math_mode;
  FS2_CUDA_CHECK(cudaGetDevice(&m->device));
  *out = m;
  return FS2_OK;
}

void fs2_melgan_destroy(fs2_melgan_gen* m) {
  if (!m) return;
  if (m->arena) cudaFree(m->arena);
  delete m;
}

int fs2_melgan_load(fs2_melgan_gen* m, const float* const* weights, const float* const* biases, void* stream) {
  FS2_REQUIRE(m && weights && biases, "fs2_melgan_load: null argument");
  for (int i = 0; i < kLayers; ++i) FS2_REQUIRE(weights[i] && biases[i], "fs2_melgan_load: layer %d: null tensor", i);
  cudaStream_t st = (cudaStream_t)stream;
  // layer index of the state_dict order: 0 = generator.1; stage s: 1 + 10 s = its ConvTranspose1d, then the ResStack's
  // blocks.i.2 (2 + 10 s + 2 i), blocks.i.4 (3 + 10 s + 2 i), shortcuts.i (8 + 10 s + i); 41 = generator.16
  struct Job { MWeight* w; int kind, N, K, Cin, Cout, taps, s; int l, l2; };
  Job jobs[1 + kStages * 7];
  int nj = 0;
  jobs[nj++] = {&m->pre, 0, 512, kMels * kPreTaps, kMels, 512, kPreTaps, 0, 0, -1};
  for (int s = 0; s < kStages; ++s) {
    const int ci = kCin[s], co = kCout[s], sd = kStride[s], base = 1 + 10 * s;
    jobs[nj++] = {&m->up[s], 1, sd * co, 3 * ci, ci, co, 0, sd, base, -1};
    for (int i = 0; i < 3; ++i) {
      jobs[nj++] = {&m->dil[s][i], 0, co, 3 * co, co, co, 3, 0, base + 1 + 2 * i, -1};
      jobs[nj++] = {&m->pair[s][i], 2, co, 2 * co, co, co, 1, 0, base + 2 + 2 * i, base + 7 + i};
    }
  }
  for (int pass = 0; pass < 2; ++pass) {       // pass 0 sizes the arena, pass 1 carves it
    Bump b(pass ? m->arena : nullptr, pass ? (size_t)-1 : 0);
    for (int j = 0; j < nj; ++j) carve(b, jobs[j].w, jobs[j].N, jobs[j].K);
    m->post_w = b.floats(kPostTaps * kPostC);
    m->post_b = b.floats(1);
    if (pass == 0) {
      if (m->arena) { FS2_CUDA_CHECK(cudaStreamSynchronize(st)); FS2_CUDA_CHECK(cudaFree(m->arena)); m->arena = nullptr; }
      m->loaded = false;
      FS2_CUDA_CHECK(cudaMalloc(&m->arena, b.off + 256));
    }
  }
  for (int j = 0; j < nj; ++j) {
    const Job& q = jobs[j];
    const int rc = pack_weight(q.w, q.kind, weights[q.l], q.l2 >= 0 ? weights[q.l2] : nullptr, biases[q.l], q.l2 >= 0 ? biases[q.l2] : nullptr,
                               q.Cin, q.Cout, q.taps, q.s, st);
    if (rc) return rc;
  }
  melgan_pack_kernel<<<1, 256, 0, st>>>(0, weights[kLayers - 1], nullptr, 1, kPostTaps * kPostC, kPostC, 1, kPostTaps, 0, m->post_w);
  FS2_LAUNCH_CHECK();
  FS2_CUDA_CHECK(cudaMemcpyAsync(m->post_b, biases[kLayers - 1], sizeof(float), cudaMemcpyDeviceToDevice, st));
  m->loaded = true;
  return FS2_OK;
}

int fs2_melgan_workspace_bytes(fs2_melgan_gen* m, int B, int Lmax, size_t* bytes) {
  FS2_REQUIRE(m && bytes, "fs2_melgan_workspace_bytes: null argument");
  int rc = check_size(m, B, Lmax);
  if (rc) return rc;
  Bump b(nullptr, 0);
  plan(b, B, Lmax, false);
  *bytes = b.off + 256;
  return FS2_OK;
}

int fs2_melgan(fs2_melgan_gen* m, const float* mels, const int64_t* olens, int B, int Lmax, float* audio, int* status, void* ws,
               size_t ws_bytes, void* stream) {
  FS2_REQUIRE(m && mels && olens && audio && status && ws, "fs2_melgan: null argument");
  FS2_REQUIRE(m->loaded, "fs2_melgan: weights not loaded (fs2_melgan_load)");
  FS2_REQUIRE((reinterpret_cast<uintptr_t>(mels) & 15) == 0, "fs2_melgan: mels must be 16-byte aligned");
  int rc = check_size(m, B, Lmax);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Bump b(ws, ws_bytes);
  MgPlan p = plan(b, B, Lmax, false);
  if (!b.ok()) { set_error("fs2_melgan: workspace too small (%zu < %zu)", ws_bytes, b.off); return FS2_ERR_WORKSPACE; }
  return generate(m, p, mels, olens, nullptr, B, Lmax, 0, audio, (long)Lmax * upsampling(kStages), status, st);
}

int fs2_melgan_window_workspace_bytes(fs2_melgan_gen* m, int B, int n_frames, size_t* bytes) {
  FS2_REQUIRE(m && bytes, "fs2_melgan_window_workspace_bytes: null argument");
  int rc = check_window(m, B, n_frames);
  if (rc) return rc;
  Bump b(nullptr, 0);
  window_plan(b, B, n_frames);
  *bytes = b.off + 256;
  return FS2_OK;
}

int fs2_melgan_window(fs2_melgan_gen* m, const float* mels, const int64_t* olens, const int64_t* starts, int B, int Lmax, int n_frames,
                      float* audio, int64_t audio_ld, int* status, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(m && mels && olens && starts && audio && status && ws, "fs2_melgan_window: null argument");
  FS2_REQUIRE((reinterpret_cast<uintptr_t>(mels) & 15) == 0, "fs2_melgan_window: mels must be 16-byte aligned");
  int rc = check_window(m, B, n_frames);
  if (rc) return rc;
  FS2_REQUIRE(Lmax >= 1 && ((long)Lmax + kTail) * upsampling(kStages) < (1L << 31),
              "fs2_melgan_window: need 1 <= Lmax and (Lmax + 10) * 256 below 2^31 (got Lmax = %d)", Lmax);
  FS2_REQUIRE(audio_ld >= (int64_t)n_frames * upsampling(kStages), "fs2_melgan_window: audio_ld = %lld below n_frames * 256 = %ld",
              (long long)audio_ld, (long)n_frames * upsampling(kStages));
  Bump b(ws, ws_bytes);
  MgPlan p = window_plan(b, B, n_frames);
  if (!b.ok()) { set_error("fs2_melgan_window: workspace too small (%zu < %zu)", ws_bytes, b.off); return FS2_ERR_WORKSPACE; }
  FS2_REQUIRE(m->loaded, "fs2_melgan_window: weights not loaded (fs2_melgan_load)");
  return generate(m, p, mels, olens, starts, B, Lmax, n_frames, audio, audio_ld, status, (cudaStream_t)stream);
}

// ---- single layers on the vocoder's own code paths (tests) ----------------------------------------------------------
// Both pack the caller's torch-layout weights into a stream-ordered temporary with the calls fs2_melgan_load makes, then
// run what fs2_melgan runs for that layer.
int fs2_op_melgan_block(int math_mode, int route, int C, const float* x, const int64_t* lens, int B, int Lp, int d, const float* w1,
                        const float* b1, const float* w2, const float* b2, const float* ws, const float* bs, float* out, int* status,
                        void* stream) {
  const char* who = "fs2_op_melgan_block";
  FS2_REQUIRE(math_mode >= FS2_MATH_FP32 && math_mode <= FS2_MATH_F16, "%s: bad math_mode %d", who, math_mode);
  FS2_REQUIRE(route >= 0 && route <= 2, "%s: route must be 0 (the vocoder's), 1 (unfused) or 2 (fused), got %d", who, route);
  FS2_REQUIRE(C == 32 || C == 64 || C == 128 || C == 256, "%s: C must be 32, 64, 128 or 256 (got %d)", who, C);
  const bool planes = math_mode == FS2_MATH_F16 || math_mode == FS2_MATH_3XTF32;
  FS2_REQUIRE(route != 2 || planes, "%s: the fused route runs in FS2_MATH_F16 / FS2_MATH_3XTF32 only", who);
  FS2_REQUIRE(x && lens && w1 && b1 && w2 && b2 && ws && bs && out && status, "%s: null argument", who);
  FS2_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 31) == 0,
              "%s: x must be 16-byte and out 32-byte aligned", who);
  FS2_REQUIRE(B >= 1 && Lp >= 1 && d >= 1 && (long)Lp + d < (1L << 30), "%s: bad shape B=%d Lp=%d d=%d", who, B, Lp, d);
  const long rows = (long)B * Lp;
  FS2_REQUIRE(rows * 3 * C < (1L << 31) && (math_mode != FS2_MATH_FP32 || rows <= 65535L * 128), "%s: too many rows (%ld)", who, rows);
  cudaStream_t st = (cudaStream_t)stream;
  const bool fused = route == 0 ? fused_blocks(math_mode, C) : route == 2;
  MWeight wd, wp;
  void* a = nullptr;
  float* h = nullptr;
  void* base = nullptr;
  for (int pass = 0; pass < 2; ++pass) {       // pass 0 sizes the temporary, pass 1 carves it
    Bump b(base, (size_t)-1);
    carve(b, &wd, C, 3 * C);
    carve(b, &wp, C, 2 * C);
    a = b.floats((size_t)rows * 3 * C);
    h = b.floats((size_t)rows * C);
    if (pass == 0) FS2_CUDA_CHECK(cudaMallocAsync(&base, b.off + 256, st));
  }
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  int rc = pack_weight(&wd, 0, w1, nullptr, b1, nullptr, C, C, 3, 0, st);
  if (!rc) rc = pack_weight(&wp, 2, w2, ws, b2, bs, C, C, 1, 0, st);
  if (!rc) rc = res_block(math_mode, fused, wd, wp, x, lens, nullptr, B, Lp, C, d, 0, a, h, out, status, st);
  cudaFreeAsync(base, st);
  return rc;
}

int fs2_op_melgan_upsample(int math_mode, int Cin, int Cout, int s, const float* x, const int64_t* lens, int B, int Lin, const float* w,
                           const float* b, float* out, int* status, void* stream) {
  const char* who = "fs2_op_melgan_upsample";
  FS2_REQUIRE(math_mode >= FS2_MATH_FP32 && math_mode <= FS2_MATH_F16, "%s: bad math_mode %d", who, math_mode);
  FS2_REQUIRE(s >= 2 && s % 2 == 0, "%s: the stride s must be even and >= 2 (got %d)", who, s);
  FS2_REQUIRE(Cin >= 16 && Cin % 16 == 0 && Cout >= 16 && Cout % 16 == 0, "%s: Cin and Cout must be multiples of 16 (got %d, %d)", who,
              Cin, Cout);
  FS2_REQUIRE(x && lens && w && b && out && status, "%s: null argument", who);
  FS2_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 31) == 0,
              "%s: x must be 16-byte and out 32-byte aligned", who);
  FS2_REQUIRE(B >= 1 && Lin >= 1, "%s: bad shape B=%d Lin=%d", who, B, Lin);
  const long rows = (long)B * Lin;
  FS2_REQUIRE(rows * s * Cout < (1L << 31) && rows * 3 * Cin < (1L << 31) && (math_mode != FS2_MATH_FP32 || rows <= 65535L * 128),
              "%s: too many rows (%ld)", who, rows);
  cudaStream_t st = (cudaStream_t)stream;
  MWeight wu;
  void* a = nullptr;
  void* base = nullptr;
  for (int pass = 0; pass < 2; ++pass) {
    Bump bb(base, (size_t)-1);
    carve(bb, &wu, s * Cout, 3 * Cin);
    a = bb.floats((size_t)rows * 3 * Cin);
    if (pass == 0) FS2_CUDA_CHECK(cudaMallocAsync(&base, bb.off + 256, st));
  }
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  int rc = pack_weight(&wu, 1, w, nullptr, b, nullptr, Cin, Cout, 0, s, st);
  if (!rc) rc = upsample(math_mode, wu, x, nullptr, Lin, lens, nullptr, B, Lin, Cin, a, out, status, st);
  cudaFreeAsync(base, st);
  return rc;
}

}  // extern "C"
