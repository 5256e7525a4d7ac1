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
// Windows (fs2_melgan_window, DESIGN.md section 11; vocoder_window.cuh): the same kernels and GEMMs on a window of each
// utterance's rows.  Every buffer then holds, per utterance, rows [start, start + len) of the utterance's n rows at its
// rate (a window descriptor [start | len | n] x B in the workspace; nullptr = the whole utterance).  Producers map a local
// row to its global row, reflect or zero-pad at the utterance's true edges, and read a source outside the window as 0:
// such rows lie in the halo and are discarded.  Only rows whose values equal the whole call's (all but `margin` rows at a
// window side that is not an utterance edge) are range-checked.
#include <math.h>

#include <algorithm>

#include "vocoder_weights.cuh"
#include "vocoder_window.cuh"

namespace fs2 {
namespace {

constexpr int kMels = 80, kTail = 10, kPreTaps = 7, kPostTaps = 7, kPostC = 32, kStages = 4;
constexpr int kLayers = 42;                          // convolutions, in state_dict order
constexpr float kPadMel = -11.5129f;                 // value of the tail frames (seungwonpark/melgan `inference`)
constexpr int kCin[kStages] = {512, 256, 128, 64}, kCout[kStages] = {256, 128, 64, 32}, kStride[kStages] = {8, 8, 2, 2};

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
// The chain plan with MelGAN's parameters: a ResStack reads 1 + 3 + 9 rows on each side, the first conv's producer stacks
// its taps from mel frames (so level 0 has no wrong rows), the last conv reads 3, and 10 tail frames.
constexpr int kResReach = 1 + 3 + 9, kPostReach = kPostTaps / 2;
constexpr UpsPlan kPlan = ups_plan(kStages, kStride, kResReach, 0, kPostReach, kTail);
static_assert(kPlan.reach[0] == 3 && kPlan.reach[1] == 4 && kPlan.reach[2] == 12 && kPlan.reach[3] == 9, "DESIGN.md section 11");
static_assert(kPlan.halo[0] == 3 && kPlan.halo[1] == 24 && kPlan.halo[2] == 32 && kPlan.halo[3] == 24 && kPlan.halo[4] == 18,
              "DESIGN.md section 11");
// rows at a window side that is not an utterance edge whose values differ from the whole call's, on entry to level s:
// ConvTranspose s-1's phases at its input window's edge read a row outside it; every residual block adds its dilation.
// The next layer's input window must lie inside the exact rows:
constexpr int level_margin(int s) { return s == 0 ? 0 : kStride[s - 1] / 2; }
constexpr bool plan_is_exact() {
  for (int s = 1; s <= kStages; ++s)
    if (level_margin(s) + kResReach > kPlan.halo[s] - (s < kStages ? kPlan.reach[s] : kPostReach)) return false;
  return level_margin(0) <= kPlan.halo[0] - kPlan.reach[0];
}
static_assert(plan_is_exact(), "a window's halo must cover every layer's reach");

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
    store_quad<OUT, RANGE_IF_STATUS>(v, row * K + k, out32, outp, plane, status, FS2_MELGAN_RANGE);
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
    store_quad<OUT, RANGE_IF_STATUS>(v, row * K + k, out32, outp, plane, !WINDOW || exact_row(r, t, margin) ? status : nullptr,
                                     FS2_MELGAN_RANGE);
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
    store_quad<OUT, RANGE_IF_STATUS>(v, row * K + k, out32, outp, plane, exact_row(r, t, margin) ? status : nullptr, FS2_MELGAN_RANGE);
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

}  // namespace
}  // namespace fs2

struct fs2_melgan_gen {
  int device = 0, math_mode = 0;
  bool loaded = false;
  void* arena = nullptr; size_t arena_bytes = 0;
  fs2::VWeight pre, up[fs2::kStages], dil[fs2::kStages][3], pair[fs2::kStages][3];
  float* post_w = nullptr;     // [7][32]
  float* post_b = nullptr;
};

namespace fs2 {
namespace {

struct MgPlan {
  int64_t* lens;     // [5][B]; a window call: the n_wins(kPlan) window descriptors [start | len | n][B]
  void* a;           // GEMM operand, up to rows * 3C of the widest stage
  float* x[2];       // activations [rows][C], ping-pong
  float* h;          // dilated conv output [rows][C] (unfused route only)
};

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
int run_block(int mode, const VWeight& w1, const VWeight& w2, const float* x, const int64_t* lens, const int64_t* win, int B, int Lp, int d,
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
int res_block(int mode, bool fused, const VWeight& w1, const VWeight& w2, const float* x, const int64_t* lens, const int64_t* win, int B,
              int Lp, int C, int d, int margin, void* a, float* h, float* out, int* status, cudaStream_t st) {
  if (fused) {
    return C == 256 ? run_block<256>(mode, w1, w2, x, lens, win, B, Lp, d, margin, out, status, st)
         : C == 128 ? run_block<128>(mode, w1, w2, x, lens, win, B, Lp, d, margin, out, status, st)
         : C == 64  ? run_block<64>(mode, w1, w2, x, lens, win, B, Lp, d, margin, out, status, st)
                    : run_block<32>(mode, w1, w2, x, lens, win, B, Lp, d, margin, out, status, st);
  }
  const int kind = out_kind(mode);
  int rc = run_taps(kind, true, x, nullptr, Lp, lens, win, B, Lp, C, d, margin, a, status, st);
  if (rc || (rc = vweight_gemm(mode, w1, a, B, Lp, ACT_NONE, lens, h, st))) return rc;
  auto concat = pick(kind, melgan_concat_kernel<OUT_HILO>, melgan_concat_kernel<OUT_HI>, melgan_concat_kernel<OUT_F32>);
  concat<<<grid_for((long)B * Lp * (2 * C / 4), 256), 256, 0, st>>>(h, x, lens, win, B, Lp, C, margin, (float*)a, (__half*)a, status);
  FS2_LAUNCH_CHECK();
  return vweight_gemm(mode, w2, a, B, Lp, ACT_NONE, lens, out, st);
}

// lrelu + ConvTranspose1d (k = 2s, stride s, pad s/2) x [B * Lin][Cin] -> out [B * Lin][s Cout] = [B * Lin * s][Cout], through
// the scratch operand a (rows * 3 Cin floats): rows t < lens[b] of x in, rows >= lens[b] * s of out written as 0.  A window:
// the input window (win, lens; Lin rows per utterance) is read from x's own window xwin of ldx rows per utterance.
int upsample(int mode, const VWeight& w, const float* x, const int64_t* xwin, int ldx, const int64_t* lens, const int64_t* win, int B, int Lin,
             int Cin, void* a, float* out, int* status, cudaStream_t st) {
  int rc = run_taps(out_kind(mode), false, x, xwin, ldx, lens, win, B, Lin, Cin, 1, 1, a, status, st);
  return rc ? rc : vweight_gemm(mode, w, a, B, Lin, ACT_NONE, lens, out, st);
}

// The generator on the plan p: whole utterances (starts == nullptr; every buffer (Lmax + 10) * up_s rows per utterance,
// lens [5][B]) or a window of nf frames from starts[b] (level_rows / ups_rows per utterance, the n_wins(kPlan) window
// descriptors).  Lout audio samples per row, rows ld apart.  Both enqueue the same kernels.
int generate(const fs2_melgan_gen* m, const MgPlan& p, const float* mels, const int64_t* olens, const int64_t* starts, int B, int Lmax,
             int nf, float* audio, long ld, int* status, cudaStream_t st) {
  const bool w = starts != nullptr;
  const int mode = m->math_mode, kind = out_kind(mode);
  auto desc = [&](int i) -> const int64_t* { return w ? p.lens + 3L * i * B : nullptr; };
  auto lens = [&](int i, int s) -> const int64_t* { return w ? p.lens + (3L * i + 1) * B : p.lens + (long)s * B; };   // window i / level s
  auto rows = [&](int s) { return w ? (int)level_rows(kPlan, s, nf) : (Lmax + kTail) * upsampling(s); };
  int rc = ups_prep(olens, starts, B, 1, Lmax, nf, kPlan, p.lens, status, st);
  if (rc) return rc;
  {
    auto k = pick(kind, melgan_pre_operand_kernel<OUT_HILO>, melgan_pre_operand_kernel<OUT_HI>, melgan_pre_operand_kernel<OUT_F32>);
    k<<<grid_for((long)B * rows(0) * (kMels * kPreTaps / 4), 256), 256, 0, st>>>(mels, lens(0, 0), desc(0), B, Lmax, rows(0), (float*)p.a,
                                                                                (__half*)p.a, status);
    FS2_LAUNCH_CHECK();
  }
  if ((rc = vweight_gemm(mode, m->pre, p.a, B, rows(0), ACT_NONE, lens(0, 0), p.x[0], st))) return rc;
  int cur = 0;
  for (int s = 0; s < kStages; ++s) {
    const int C = kCout[s], cw = win_ups(kPlan, s), Lin = w ? (int)ups_rows(kPlan, s, nf) : rows(s);
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
  melgan_post_kernel<<<grid_for((long)B * Lout, 256), 256, 0, st>>>(p.x[cur], lens(kStages, kStages), desc(kStages), desc(win_audio(kPlan)), B,
                                                                   rows(kStages), Lout, ld, m->post_w, m->post_b, audio);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// per frame of Lp: values of the largest operand (3C at the three late stages, 24576) and activation (8192)
constexpr long kOperandPerFrame = 3L * 256 * 32, kActPerFrame = 256L * 32;

// the generator's side of the shared C entries (vocoder_window.cuh)
struct MgEntry {
  using Gen = fs2_melgan_gen;
  static const UpsPlan& ups(const Gen*) { return kPlan; }
  static MgPlan plan(Bump& b, const Gen*, int B, int L) {
    const size_t frames = (size_t)B * (L + kTail);
    MgPlan p;
    p.lens = (int64_t*)b.bytes((size_t)(kStages + 1) * B * sizeof(int64_t));
    p.a = b.floats(frames * kOperandPerFrame);
    p.x[0] = b.floats(frames * kActPerFrame);
    p.x[1] = b.floats(frames * kActPerFrame);
    p.h = b.floats(frames * kActPerFrame);
    return p;
  }
  // A window call's workspace, from B and nf only: per utterance, the largest operand (rows x K over every producer) and
  // the largest activation (rows x C over every level) of the window's buffers
  static MgPlan window_plan(Bump& b, const Gen*, int B, int nf) {
    long op = level_rows(kPlan, 0, nf) * kMels * kPreTaps, act = level_rows(kPlan, 0, nf) * 512;
    for (int s = 0; s < kStages; ++s) {
      op = std::max(op, std::max(ups_rows(kPlan, s, nf) * 3 * kCin[s], level_rows(kPlan, s + 1, nf) * 3 * kCout[s]));
      act = std::max(act, level_rows(kPlan, s + 1, nf) * kCout[s]);
    }
    MgPlan p;
    p.lens = (int64_t*)b.bytes((size_t)3 * n_wins(kPlan) * B * sizeof(int64_t));
    p.a = b.floats((size_t)B * op);
    p.x[0] = b.floats((size_t)B * act);
    p.x[1] = b.floats((size_t)B * act);
    p.h = b.floats((size_t)B * act);
    return p;
  }
  static constexpr auto generate = fs2::generate;
};

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

void fs2_melgan_destroy(fs2_melgan_gen* m) { destroy_gen(m); }

int fs2_melgan_load(fs2_melgan_gen* m, const float* const* weights, const float* const* biases, void* stream) {
  FS2_REQUIRE(m && weights && biases, "fs2_melgan_load: null argument");
  for (int i = 0; i < kLayers; ++i) FS2_REQUIRE(weights[i] && biases[i], "fs2_melgan_load: layer %d: null tensor", i);
  cudaStream_t st = (cudaStream_t)stream;
  // layer index of the state_dict order: 0 = generator.1; stage s: 1 + 10 s = its ConvTranspose1d, then the ResStack's
  // blocks.i.2 (2 + 10 s + 2 i), blocks.i.4 (3 + 10 s + 2 i), shortcuts.i (8 + 10 s + i); 41 = generator.16
  // A GEMM weight here is [N][K] with a convolution's taps side by side along K (vweight_pack_conv at tap_stride = Cin); a
  // residual block's 1x1 convolution and its shortcut (l2) share one weight [W2 | Ws] over the operand [h | x]
  struct Job { VWeight* w; int N, K, Cin, Cout, taps, s; int l, l2; };
  Job jobs[1 + kStages * 7];
  int nj = 0;
  jobs[nj++] = {&m->pre, 512, kMels * kPreTaps, kMels, 512, kPreTaps, 0, 0, -1};
  for (int s = 0; s < kStages; ++s) {
    const int ci = kCin[s], co = kCout[s], sd = kStride[s], base = 1 + 10 * s;
    jobs[nj++] = {&m->up[s], sd * co, 3 * ci, ci, co, 3, sd, base, -1};
    for (int i = 0; i < 3; ++i) {
      jobs[nj++] = {&m->dil[s][i], co, 3 * co, co, co, 3, 0, base + 1 + 2 * i, -1};
      jobs[nj++] = {&m->pair[s][i], co, 2 * co, co, co, 1, 0, base + 2 + 2 * i, base + 7 + i};
    }
  }
  for (int j = 0; j < nj; ++j) { jobs[j].w->N = jobs[j].N; jobs[j].w->K = jobs[j].K; }
  m->loaded = false;
  int rc = arena_carve(&m->arena, &m->arena_bytes, st, [&](Bump& b) {
    for (int j = 0; j < nj; ++j) vweight_carve(b, *jobs[j].w, true);
    m->post_w = b.floats(kPostTaps * kPostC);
    m->post_b = b.floats(1);
    return FS2_OK;
  });
  if (rc) return rc;
  for (int j = 0; j < nj; ++j) {
    const Job& q = jobs[j];
    rc = vweight_pack_conv(*q.w, weights[q.l], biases[q.l], q.Cin, q.Cout, q.taps, q.s, q.Cin, st, q.l2 >= 0 ? weights[q.l2] : nullptr,
                           q.l2 >= 0 ? biases[q.l2] : nullptr);
    if (rc) return rc;
  }
  if ((rc = conv_pack(weights[kLayers - 1], 1, kPostC, kPostTaps, 1, 0, kPostC, kPostTaps * kPostC, m->post_w, st))) return rc;
  FS2_CUDA_CHECK(cudaMemcpyAsync(m->post_b, biases[kLayers - 1], sizeof(float), cudaMemcpyDeviceToDevice, st));
  m->loaded = true;
  return FS2_OK;
}

int fs2_melgan_workspace_bytes(fs2_melgan_gen* m, int B, int Lmax, size_t* bytes) {
  return workspace_gen<MgEntry>(m, B, Lmax, bytes, "fs2_melgan");
}

int fs2_melgan(fs2_melgan_gen* m, const float* mels, const int64_t* olens, int B, int Lmax, float* audio, int* status, void* ws,
               size_t ws_bytes, void* stream) {
  return call_gen<MgEntry>(m, mels, olens, B, Lmax, audio, status, ws, ws_bytes, stream, "fs2_melgan");
}

int fs2_melgan_window_workspace_bytes(fs2_melgan_gen* m, int B, int n_frames, size_t* bytes) {
  return window_workspace_gen<MgEntry>(m, B, n_frames, bytes, "fs2_melgan");
}

int fs2_melgan_window(fs2_melgan_gen* m, const float* mels, const int64_t* olens, const int64_t* starts, int B, int Lmax, int n_frames,
                      float* audio, int64_t audio_ld, int* status, void* ws, size_t ws_bytes, void* stream) {
  return window_gen<MgEntry>(m, mels, olens, starts, B, Lmax, n_frames, audio, audio_ld, status, ws, ws_bytes, stream, "fs2_melgan");
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
  FS2_REQUIRE(rows * 3 * C < (1L << 31) && (math_mode != FS2_MATH_FP32 || rows <= kTapGemmFp32MaxRows), "%s: too many rows (%ld)", who, rows);
  cudaStream_t st = (cudaStream_t)stream;
  const bool fused = route == 0 ? fused_blocks(math_mode, C) : route == 2;
  VWeight wd, wp;
  wd.N = C; wd.K = 3 * C;
  wp.N = C; wp.K = 2 * C;
  void* a = nullptr;
  float* h = nullptr;
  void* base = nullptr;
  int rc = temp_carve(&base, st, [&](Bump& b) {
    vweight_carve(b, wd, true);
    vweight_carve(b, wp, true);
    a = b.floats((size_t)rows * 3 * C);
    h = b.floats((size_t)rows * C);
  });
  if (rc) return rc;
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  rc = vweight_pack_conv(wd, w1, b1, C, C, 3, 0, C, st);
  if (!rc) rc = vweight_pack_conv(wp, w2, b2, C, C, 1, 0, C, st, ws, bs);
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
  FS2_REQUIRE(rows * s * Cout < (1L << 31) && rows * 3 * Cin < (1L << 31) && (math_mode != FS2_MATH_FP32 || rows <= kTapGemmFp32MaxRows),
              "%s: too many rows (%ld)", who, rows);
  cudaStream_t st = (cudaStream_t)stream;
  VWeight wu;
  wu.N = s * Cout; wu.K = 3 * Cin;
  void* a = nullptr;
  void* base = nullptr;
  int rc = temp_carve(&base, st, [&](Bump& bb) {
    vweight_carve(bb, wu, true);
    a = bb.floats((size_t)rows * 3 * Cin);
  });
  if (rc) return rc;
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  rc = vweight_pack_conv(wu, w, b, Cin, Cout, 3, s, Cin, st);
  if (!rc) rc = upsample(math_mode, wu, x, nullptr, Lin, lens, nullptr, B, Lin, Cin, a, out, status, st);
  cudaFreeAsync(base, st);
  return rc;
}

}  // extern "C"
