// Batched WaveGlow vocoder (DESIGN.md section 9): log-mels [B, Lmax, 80] -> audio [B, Lmax * 256], each utterance the
// inverse flow (`WaveGlow.infer`) over its own olens[b] frames, on the library's tap-GEMM.
//
// Audio is handled in groups of 8 samples: one "step" row per group, 32 steps per mel frame, so every per-step tensor is
// [B, Ls, .] with Ls = Lmax * 32 and every GEMM runs with TapGemm::lens = olens * 32 (olens for the frame-level
// upsampling): row tiles wholly past an utterance are skipped and padded rows come out as exact zeros, which is also the
// zero padding the dilated convolutions see at each utterance's own edges.
//
//   up operand     mel frames t-3 .. t side by side (0 outside [0, olens[b]))              -> GEMM 320 -> 80 * 256
//                  ConvTranspose1d(80, 80, 1024, stride 256) trimmed to olens * 256 samples, as a polyphase GEMM whose
//                  columns come out in (step-in-frame, c * 8 + g) order: the frame rows of the result *are* the step rows
//                  of the cond operand [B * Ls][640] (planes written by a separate pass with the range check)
//   per flow k = 11 .. 0 (c channels, n_half = c / 2):
//     start        x = W_start . audio_0 + b on CUDA cores (K = n_half), fp32 rows (+ planes)
//     layer i:     cond GEMM      640 -> 2C, both biases                                     = cd
//                  in-layer GEMM  C -> 2C, 3 taps at dilation 2^i, resid = cd                 = ia
//                  gate           tanh(ia[:C]) * sigmoid(ia[C:])                              = acts (GEMM operand)
//                  res GEMM       C -> C, resid = x (layers 0 .. 6)                           = x' (+ planes)
//                  skip GEMM      C -> C, resid = skip (layers 1 .. 7)                        = skip'
//     flow         end conv (C -> 2 n_half) on skip, affine coupling, inverse 1x1 conv, on CUDA cores
//
// The flow state [B * Ls][8] holds the audio channels in columns 8 - c .. 7, and starts as fp32(sigma * z) in all eight:
// z's channels 0-1 and 2-3 are exactly the early noise prepended after flows 4 and 8, so the concatenation costs nothing.
// After flow 0 the state is the audio itself ([B, Ls, 8] row-major = [B, Lmax * 256]), so the last flow writes `audio`.
// Launches per call: 4 + 12 * 41 = 496, plus 1 (the cond planes) in f16 / 3xF16; a window adds 1 (its audio copy).
// run() is upsample() then flow() per k; the per-stage test entries at the end of the file call the same two functions.
//
// A GEMM row depends only on its own input rows (the in-layer GEMM: rows t, t +- 2^i of its own utterance, zero outside
// [0, olens * 32)), in a fixed K order, so per-utterance results do not depend on the batch.
//
// Windows (fs2_waveglow_window, DESIGN.md section 12): the same kernels and GEMMs on one buffer per utterance that holds
// global frames [f0, f1) = [max(0, s - H), min(olens, s + n + H)) around the core [s, s + n), H = 96 frames, every buffer
// (n + 2H) * 32 step rows long.  The window layer (vocoder_window.cuh) describes it as a plan of two levels, the frames
// and their step rows, each with a halo of H frames: ups_prep writes a descriptor [start | len | n] x B for the frames,
// the step rows and the core's step rows (nullptr = the whole utterance).  A flow reaches 255 step rows on each side, so
// halo rows at a side that is not an utterance edge (f0 > 0, f1 < olens) differ from the whole call's by at most 255 more
// rows per flow, and the core is exact after all 12.  The noise, the upsampling operand and the cond planes are keyed by
// global frames and steps, so they are exact everywhere in the buffer; start and gate range-check only rows whose values
// equal the whole call's (exact_row).
#include <math.h>

#include "vocoder_weights.cuh"
#include "vocoder_window.cuh"

namespace fs2 {
namespace {

constexpr int kMels = 80, kHop = 256, kGroup = 8, kSteps = kHop / kGroup, kFlows = 12, kLayers = 8;
constexpr int kCond = kMels * kGroup;          // 640 cond channels per step
constexpr int kUpTaps = 4, kUpK = kUpTaps * kMels, kUpN = kMels * kHop, kUpKernel = kUpTaps * kHop;
constexpr int kPerFlow = 2 + 6 * kLayers + 3;  // tensors per flow in fs2_waveglow_load
constexpr int kTensors = 2 + kFlows * kPerFlow;
// ---- window plan (DESIGN.md section 12) ----
constexpr int kFlowReach = (1 << kLayers) - 1;                              // 8 k = 3 layers at dilation 2^i: 255 step rows
constexpr int kHalo = (kFlows * kFlowReach + kSteps - 1) / kSteps;          // 96 frames on each side of a window's core
// The window plan (vocoder_window.cuh): level 0 the frames, level 1 their step rows, each with a halo of kHalo frames;
// the upsampling reads level 0's rows (its reach is the halo, so its input window is level 0's); no tail frames.  The
// descriptors are level 0's, level 1's and the audio's, all three in the rows of their level (the audio: step rows).
constexpr UpsPlan kPlan{1, {1, kSteps}, {kHalo}, {kHalo, kSteps * kHalo}, 0};
static_assert(kPlan.halo[1] >= kFlows * kFlowReach, "the halo must cover the 12 flows' reach");
static_assert(n_wins(kPlan) == 3 && win_audio(kPlan) == 2, "descriptors of level 0, level 1 and the audio");
constexpr UpsPlan kStepPlan{0, {1}, {}, {}, 0};                             // fs2_op_waveglow_flow's lengths: step rows

__host__ __device__ inline int flow_channels(int k) { return k < 4 ? 8 : k < 8 ? 6 : 4; }

// Four standard normals for channels 4q .. 4q + 3 of step t of the utterance with seed s: Philox4x32-10 with key
// (s mod 2^32, s / 2^32) and counter (t, q, 0, 0), Box-Muller on two pairs of 23-bit uniforms in (0, 1).
__device__ __forceinline__ float4 normal4(uint64_t seed, uint32_t t, uint32_t q) {
  const uint4 r = philox4x32(make_uint4(t, q, 0u, 0u), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  const float u0 = ((float)(r.x >> 9) + 0.5f) * 0x1p-23f, u1 = ((float)(r.y >> 9) + 0.5f) * 0x1p-23f;
  const float u2 = ((float)(r.z >> 9) + 0.5f) * 0x1p-23f, u3 = ((float)(r.w >> 9) + 0.5f) * 0x1p-23f;
  const float r0 = sqrtf(-2.f * logf(u0)), r1 = sqrtf(-2.f * logf(u2));
  float s0, c0, s1, c1;
  sincospif(2.f * u1, &s0, &c0);
  sincospif(2.f * u3, &s1, &c1);
  return make_float4(r0 * c0, r0 * s0, r1 * c1, r1 * s1);
}

// The standard-normal draw z [B, 8, Ls] for the steps t < n_b = min(lens[b] * mult, Ls): from zin ([B, 8, ldz]) or from
// Philox keyed by seeds[b].  state [B * Ls][8] (nullable) = fp32(sigma * z), the product in double and rounded once;
// zout [B, 8, Ls] (nullable) = z; both 0 for t >= n_b.  zin is never read there.  win (a window's step rows): local step t
// is global step start + t, in zin and in the Philox counter alike.
__global__ void wg_noise_kernel(const float* __restrict__ zin, int ldz, const int64_t* __restrict__ seeds, const int64_t* __restrict__ lens,
                                const int64_t* __restrict__ win, int mult, int B, int Ls, double sigma, float* __restrict__ state,
                                float* __restrict__ zout) {
  const long total = (long)B * Ls * 2;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i >> 1;
    const int q = (int)(i & 1), b = (int)(row / Ls), t = (int)(row - (long)b * Ls);
    long n = lens[b] * mult;
    n = n < 0 ? 0 : (n > Ls ? Ls : n);
    float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t < n) {
      const long tg = (long)rows_of(win, lens, B, b).start + t;
      if (zin) {
        const float* zb = zin + ((long)b * kGroup + 4 * q) * ldz + tg;
        z = make_float4(zb[0], zb[ldz], zb[2L * ldz], zb[3L * ldz]);
      } else {
        z = normal4((uint64_t)seeds[b], (uint32_t)tg, (uint32_t)q);
      }
    }
    if (state)
      *reinterpret_cast<float4*>(state + row * kGroup + 4 * q) =
          make_float4((float)(sigma * z.x), (float)(sigma * z.y), (float)(sigma * z.z), (float)(sigma * z.w));
    if (zout) {
      float* zb = zout + ((long)b * kGroup + 4 * q) * Ls + t;
      zb[0] = z.x; zb[Ls] = z.y; zb[2L * Ls] = z.z; zb[3L * Ls] = z.w;
    }
  }
}

// upsampling operand [B * L][4 * 80]: tap j of frame row t = mel frame t - 3 + j of its utterance, 0 outside [0, n).
// Rows t >= len are not written (the GEMM writes 0 there); frames past olens[b] are never read.  mels has Lm frames per
// utterance.  win (a window's frames): row t is global frame start + t, and the source is 0 outside [0, n = olens[b]), so
// every row equals the whole call's.
template <int OUT>
__global__ void wg_up_operand_kernel(const float* __restrict__ mels, const int64_t* __restrict__ lensF, const int64_t* __restrict__ win,
                                     int B, int L, int Lm, float* __restrict__ out32, __half* __restrict__ outp, int* __restrict__ status) {
  constexpr int Q = kUpK / 4;
  const long rows = (long)B * L, total = rows * Q, plane = rows * kUpK;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / Q;
    const int k = (int)(i - row * Q) * 4, j = k / kMels, c = k - j * kMels;
    const int b = (int)(row / L), t = (int)(row - (long)b * L);
    const Rows r = rows_of(win, lensF, B, b);
    if (t >= r.len) continue;
    const int src = r.start + t - (kUpTaps - 1) + j;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (src >= 0 && src < r.n) v = *reinterpret_cast<const float4*>(mels + ((long)b * Lm + src) * kMels + c);
    store_quad<OUT, RANGE_IF_STATUS>(v, row * kUpK + k, out32, outp, plane, status, FS2_WAVEGLOW_RANGE);
  }
}

// operand planes of fp32 rows x [B * Ls][K] with the range check (rows t >= lens[b] are not written)
template <int OUT>
__global__ void wg_planes_kernel(const float* __restrict__ x, const int64_t* __restrict__ lens, int B, int Ls, int K,
                                 __half* __restrict__ outp, int* __restrict__ status) {
  const int Q = K / 4;
  const long rows = (long)B * Ls, total = rows * Q, plane = rows * K;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / Q;
    const int b = (int)(row / Ls), t = (int)(row - (long)b * Ls);
    if (t >= (int)lens[b]) continue;
    const long off = row * K + (i - row * Q) * 4;
    store_quad<OUT, RANGE_IF_STATUS>(*reinterpret_cast<const float4*>(x + off), off, nullptr, outp, plane, status, FS2_WAVEGLOW_RANGE);
  }
}

// WN start: x[r][n] = bias[n] + sum_{q < h} w[n][q] * state[r][o + q] for t < lens[b], else 0 -- fp32 rows (the residual
// stream) and, in the plane modes, the in-layer GEMM's operand planes.  Padded rows are written: the dilated taps read them.
// win / margin (a window's step rows): only exact rows are range-checked.
template <int OUT>
__global__ void wg_start_kernel(const float* __restrict__ state, const int64_t* __restrict__ lens, const int64_t* __restrict__ win,
                                int margin, int B, int Ls, int C, int o, int h, const float* __restrict__ w, const float* __restrict__ bias,
                                float* __restrict__ x, __half* __restrict__ xp, int* __restrict__ status) {
  const int Q = C / 4;
  const long rows = (long)B * Ls, total = rows * Q, plane = rows * C;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / Q;
    const int n = (int)(i - row * Q) * 4;
    const int b = (int)(row / Ls), t = (int)(row - (long)b * Ls);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t < (int)lens[b]) {
      v = *reinterpret_cast<const float4*>(bias + n);
      const float* a = state + row * kGroup + o;
      for (int q = 0; q < h; ++q) {
        const float aq = a[q];
        v.x = fmaf(__ldg(w + (n + 0) * h + q), aq, v.x);
        v.y = fmaf(__ldg(w + (n + 1) * h + q), aq, v.y);
        v.z = fmaf(__ldg(w + (n + 2) * h + q), aq, v.z);
        v.w = fmaf(__ldg(w + (n + 3) * h + q), aq, v.w);
      }
    }
    *reinterpret_cast<float4*>(x + row * C + n) = v;
    if (OUT != OUT_F32)
      store_quad<OUT, RANGE_IF_STATUS>(v, row * C + n, nullptr, xp, plane, exact_row(rows_of(win, lens, B, b), t, margin) ? status : nullptr,
                                       FS2_WAVEGLOW_RANGE);
  }
}

// gate: acts[r][c] = tanh(ia[r][c]) * sigmoid(ia[r][C + c]) as the res / skip GEMMs' operand (rows t >= lens[b] are not
// written).  xchk (nullable, plane modes): the layer's input rows x, written as planes by the previous res GEMM's
// epilogue, are range-checked here.  win (a window's step rows): acts only at rows exact at `margin`, x at `xmargin`.
template <int OUT>
__global__ void wg_gate_kernel(const float* __restrict__ ia, const float* __restrict__ xchk, const int64_t* __restrict__ lens,
                               const int64_t* __restrict__ win, int margin, int xmargin, int B, int Ls, int C, float* __restrict__ out32,
                               __half* __restrict__ outp, int* __restrict__ status) {
  const int Q = C / 4;
  const long rows = (long)B * Ls, total = rows * Q, plane = rows * C;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / Q;
    const int c = (int)(i - row * Q) * 4;
    const int b = (int)(row / Ls), t = (int)(row - (long)b * Ls);
    const Rows r = rows_of(win, lens, B, b);
    if (t >= r.len) continue;
    const float4 a = *reinterpret_cast<const float4*>(ia + row * 2 * C + c);
    const float4 g = *reinterpret_cast<const float4*>(ia + row * 2 * C + C + c);
    const float4 v = make_float4(tanhf(a.x) * (1.f / (1.f + expf(-g.x))), tanhf(a.y) * (1.f / (1.f + expf(-g.y))),
                                 tanhf(a.z) * (1.f / (1.f + expf(-g.z))), tanhf(a.w) * (1.f / (1.f + expf(-g.w))));
    store_quad<OUT, RANGE_IF_STATUS>(v, row * C + c, out32, outp, plane, exact_row(r, t, margin) ? status : nullptr, FS2_WAVEGLOW_RANGE);
    if (xchk && exact_row(r, t, xmargin)) {
      const float4 x = *reinterpret_cast<const float4*>(xchk + row * C + c);
      if (!(fabsf(x.x) <= kPlaneMax && fabsf(x.y) <= kPlaneMax && fabsf(x.z) <= kPlaneMax && fabsf(x.w) <= kPlaneMax))
        atomicOr(status, FS2_WAVEGLOW_RANGE);
    }
  }
}

// One flow's tail, a warp per step row: [b_shift | log_s] = W_end . skip + b_end (2H dot products of length C), then
// audio_1 = (audio_1 - b_shift) / exp(log_s) and the inverse 1x1 conv over the c = 2H channels in columns o .. 7 of the
// state.  out may alias in (the in-place update of the state) or be the audio; rows t >= lens[b] get zeros.
template <int H>
__global__ void __launch_bounds__(256) wg_flow_kernel(const float* __restrict__ skip, int C, const float* in, float* out,
                                                      const int64_t* __restrict__ lens, int B, int Ls, int o,
                                                      const float* __restrict__ we, const float* __restrict__ be,
                                                      const float* __restrict__ winv) {
  constexpr int c = 2 * H;
  extern __shared__ __align__(16) float sh[];
  float* swe = sh;                   // [2H][C]
  float* swi = sh + c * C;           // [c][c]
  float* sbe = swi + c * c;          // [2H]
  for (int i = threadIdx.x; i < c * C; i += blockDim.x) swe[i] = we[i];
  for (int i = threadIdx.x; i < c * c; i += blockDim.x) swi[i] = winv[i];
  if (threadIdx.x < c) sbe[threadIdx.x] = be[threadIdx.x];
  __syncthreads();
  const int lane = threadIdx.x & 31, warps = blockDim.x >> 5;
  const long rows = (long)B * Ls;
  for (long r = (long)blockIdx.x * warps + (threadIdx.x >> 5); r < rows; r += (long)gridDim.x * warps) {
    const int b = (int)(r / Ls), t = (int)(r - (long)b * Ls);
    float* dst = out + r * kGroup + o;
    if (t >= (int)lens[b]) {
      if (lane < c) dst[lane] = 0.f;
      continue;
    }
    float acc[c];
#pragma unroll
    for (int e = 0; e < c; ++e) acc[e] = 0.f;
    const float4* srow = reinterpret_cast<const float4*>(skip + r * C);
    for (int q = lane; q < C / 4; q += 32) {
      const float4 v = __ldg(srow + q);
#pragma unroll
      for (int e = 0; e < c; ++e) {
        const float4 w = reinterpret_cast<const float4*>(swe + e * C)[q];
        acc[e] = fmaf(w.x, v.x, fmaf(w.y, v.y, fmaf(w.z, v.z, fmaf(w.w, v.w, acc[e]))));
      }
    }
#pragma unroll
    for (int e = 0; e < c; ++e) acc[e] = warp_sum(acc[e]);
    const float* src = in + r * kGroup + o;
    float v[c];
#pragma unroll
    for (int q = 0; q < H; ++q) {
      v[q] = src[q];
      v[H + q] = (src[H + q] - (acc[q] + sbe[q])) / expf(acc[H + q] + sbe[H + q]);
    }
    __syncwarp();                   // every lane has read the row before any lane overwrites it
    if (lane < c) {
      float y = 0.f;
#pragma unroll
      for (int q = 0; q < c; ++q) y = fmaf(swi[lane * c + q], v[q], y);
      dst[lane] = y;
    }
  }
}

// a window's audio: row b (ld samples apart) = the samples of the core's step rows awin in the final state [B * Ls][8]
// (step rows win; utterance b's samples are contiguous there), then +0 up to nf * 256
__global__ void wg_win_audio_kernel(const float* __restrict__ state, const int64_t* __restrict__ win, const int64_t* __restrict__ awin,
                                    int B, int Ls, int nf, float* __restrict__ audio, long ld) {
  const int n = nf * kHop;
  const long total = (long)B * n;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int b = (int)(i / n), t = (int)(i - (long)b * n);
    const Rows r = rows_of(win, nullptr, B, b), a = rows_of(awin, nullptr, B, b);
    float v = 0.f;
    if (t < a.len * kGroup) v = state[((long)b * Ls + a.start - r.start) * kGroup + t];
    audio[(long)b * ld + t] = v;
  }
}

// in-layer weight, Conv1d [N][K][taps] -> the tap GEMM's [taps][N][K]
__global__ void wg_pack_taps_kernel(const float* __restrict__ w, int N, int K, int taps, float* __restrict__ dst) {
  const long total = (long)N * K * taps;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int j = (int)(i / ((long)N * K));
    const long nk = i - (long)j * N * K;
    dst[i] = w[nk * taps + j];
  }
}

// ConvTranspose1d(80, 80, 1024, stride 256) [ci][co][1024] -> polyphase GEMM weight [20480][320]: column n = s * 640 +
// co * 8 + g is output sample r = 8 s + g of a frame, K index j * 80 + ci reads frame t - 3 + j through kernel tap
// r + 256 (3 - j); bias[n] = b[co]
__global__ void wg_pack_up_kernel(const float* __restrict__ w, const float* __restrict__ b, float* __restrict__ dst, float* __restrict__ bias) {
  const long total = (long)kUpN * kUpK;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int n = (int)(i / kUpK), k = (int)(i - (long)n * kUpK);
    const int s = n / kCond, co = (n - s * kCond) / kGroup, g = n % kGroup, r = s * kGroup + g;
    const int j = k / kMels, ci = k - j * kMels;
    dst[i] = w[((long)ci * kMels + co) * kUpKernel + r + kHop * (kUpTaps - 1 - j)];
    if (k == 0) bias[n] = b[co];
  }
}

__global__ void wg_add_kernel(const float* __restrict__ a, const float* __restrict__ b, int n, float* __restrict__ dst) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = a[i] + b[i];
}

struct WFlow {
  float *start_w = nullptr, *start_b = nullptr;   // [C][h], [C]
  VWeight cond[kLayers], in[kLayers], res[kLayers - 1], skip[kLayers];
  float *end_w = nullptr, *end_b = nullptr;       // [2h][C], [2h]
  float* winv = nullptr;                          // [c][c]
};

}  // namespace
}  // namespace fs2

struct fs2_waveglow_net {
  int device = 0, math_mode = 0, C = 0;
  bool loaded = false;
  void* arena = nullptr; size_t arena_bytes = 0;
  fs2::VWeight up;
  fs2::WFlow flows[fs2::kFlows];
};

namespace fs2 {
namespace {

struct WgPlan {
  int64_t* lens;       // ups_prep's block: the whole call's lengths [2][B] of frames and step rows, or a window call's
                       // n_wins(kPlan) descriptors [start | len | n][B] of frames, step rows and the audio's step rows
  int64_t* lensF;      // [B] frame lengths in it (0 for a bad olens[b])
  int64_t* lensS;      // [B] step lengths = lensF * 32
  int64_t* winF;       // a window call: the descriptors of its frames and its step rows (nullptr: whole utterances)
  int64_t* winS;
  void* up_a;          // upsampling operand [B * L][320]
  float* cond;         // upsampled mels as fp32 step rows [B * Ls][640].  The plane modes need them only until the
                       // planes are written, before ia is first used, so there they alias ia when its rows hold 640
                       // floats (2C >= 640); otherwise they have a region of their own
  __half* condp;       // their planes [P][B * Ls][640] (plane modes)
  float* state;        // flow state [B * Ls][8]
  float* x[2];         // residual stream [B * Ls][C], ping-pong
  __half* xp;          // its planes [P][B * Ls][C] (plane modes)
  float* cd;           // cond GEMM output [B * Ls][2C]
  float* ia;           // in-layer GEMM output [B * Ls][2C]
  void* acts;          // gate output [B * Ls][C] (fp32 rows or planes)
  float* skip[2];      // skip accumulator [B * Ls][C], ping-pong
};

// a flow's buffers over `rows` step rows: x, xp, cd, ia, acts, skip and the cond planes (plane modes)
void plan_wn(Bump& b, WgPlan& p, bool planes, int C, size_t rows) {
  p.x[0] = b.floats(rows * C);
  p.x[1] = b.floats(rows * C);
  p.xp = planes ? (__half*)b.floats(rows * C) : nullptr;
  p.cd = b.floats(rows * 2 * C);
  p.ia = b.floats(rows * 2 * C);
  p.acts = b.floats(rows * C);
  p.skip[0] = b.floats(rows * C);
  p.skip[1] = b.floats(rows * C);
  p.condp = planes ? (__half*)b.floats(rows * kCond) : nullptr;
}

// buffers of L frames per utterance: the whole call's (L = Lmax) or a window's (window, L = n_frames + 2H)
WgPlan plan(Bump& b, int mode, int C, int B, int L, bool window = false) {
  const size_t frames = (size_t)B * L, rows = frames * kSteps;
  const bool planes = plane_mode(mode);
  WgPlan p;
  p.lens = (int64_t*)b.bytes((size_t)(window ? 3 * n_wins(kPlan) : kPlan.n + 1) * B * sizeof(int64_t));
  auto row = [&](int i) { return p.lens ? p.lens + (long)i * B : nullptr; };
  p.lensF = row(window ? 3 * win_level(0) + 1 : 0);
  p.lensS = row(window ? 3 * win_level(1) + 1 : 1);
  p.winF = window ? row(3 * win_level(0)) : nullptr;
  p.winS = window ? row(3 * win_level(1)) : nullptr;
  p.up_a = b.floats(frames * kUpK);                   // fp32 rows, or hi + lo planes: the same bytes
  p.state = b.floats(rows * kGroup);
  plan_wn(b, p, planes, C, rows);
  p.cond = planes && 2 * C >= kCond ? p.ia : b.floats(rows * kCond);    // ia holds rows * 2C floats
  return p;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }   // null counts as aligned

int check_size(const fs2_waveglow_net* m, int B, int L) {
  FS2_REQUIRE(B >= 1 && L >= 1, "fs2_waveglow: need B >= 1 and Lmax >= 1 (got %d, %d)", B, L);
  return check_rows("fs2_waveglow", "B * Lmax * 32", "step", (long)B * L * kSteps, m->math_mode);
}

// a window's limits apply to its rows: B buffers of (n_frames + 2H) * 32 step rows
int check_window(const fs2_waveglow_net* m, int B, int nf) {
  FS2_REQUIRE(B >= 1 && nf >= 1, "fs2_waveglow_window: need B >= 1 and n_frames >= 1 (got %d, %d)", B, nf);
  return check_rows("fs2_waveglow_window", "B * (n_frames + 192) * 32", "window", (long)B * ((long)nf + 2 * kHalo) * kSteps,
                    m->math_mode);
}

template <typename K>
int launch_flow(K kernel, int c, int C, const float* skip, const float* in, float* out, const int64_t* lens, int B, int Ls, int o,
                const WFlow& f, cudaStream_t st) {
  const size_t smem = (size_t)(c * C + c * c + c) * sizeof(float);
  kernel<<<grid_for((long)B * Ls, 8), 256, smem, st>>>(skip, C, in, out, lens, B, Ls, o, f.end_w, f.end_b, f.winv);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// flow k's tail (wg_flow_kernel) on the WN skip sum `skip`: columns 8 - c .. 7 of the state `in` into those of `out`
int flow_tail(const fs2_waveglow_net* m, int k, const float* skip, const float* in, float* out, const int64_t* lens, int B, int Ls,
              cudaStream_t st) {
  const WFlow& f = m->flows[k];
  const int c = flow_channels(k), h = c / 2, o = kGroup - c, C = m->C;
  return h == 4 ? launch_flow(wg_flow_kernel<4>, c, C, skip, in, out, lens, B, Ls, o, f, st)
       : h == 3 ? launch_flow(wg_flow_kernel<3>, c, C, skip, in, out, lens, B, Ls, o, f, st)
                : launch_flow(wg_flow_kernel<2>, c, C, skip, in, out, lens, B, Ls, o, f, st);
}

// The upsampling on the plan p (L frames per utterance, mels Lm frames apart): the operand of frames t - 3 .. t, the
// polyphase GEMM into the fp32 cond rows p.cond and, in the plane modes, their planes p.condp with the range check.
// *cond_a: the cond GEMMs' operand (p.condp or p.cond).
int upsample(const fs2_waveglow_net* m, const WgPlan& p, const float* mels, int B, int L, int Lm, int* status, cudaStream_t st,
             const void** cond_a) {
  const int kind = out_kind(m->math_mode);
  const bool planes = plane_mode(m->math_mode);
  const long rows = (long)B * L * kSteps;
  int rc;
  {
    auto k = pick(kind, wg_up_operand_kernel<OUT_HILO>, wg_up_operand_kernel<OUT_HI>, wg_up_operand_kernel<OUT_F32>);
    k<<<grid_for((long)B * L * (kUpK / 4), 256), 256, 0, st>>>(mels, p.lensF, p.winF, B, L, Lm, (float*)p.up_a, (__half*)p.up_a, status);
    FS2_LAUNCH_CHECK();
  }
  if ((rc = vweight_gemm(m->math_mode, m->up, p.up_a, B, L, ACT_NONE, p.lensF, p.cond, st))) return rc;
  if (planes) {
    auto k = kind == OUT_HILO ? wg_planes_kernel<OUT_HILO> : wg_planes_kernel<OUT_HI>;
    k<<<grid_for(rows * (kCond / 4), 256), 256, 0, st>>>(p.cond, p.lensS, B, L * kSteps, kCond, p.condp, status);
    FS2_LAUNCH_CHECK();
  }
  *cond_a = planes ? (const void*)p.condp : (const void*)p.cond;
  return FS2_OK;
}

// Flow k of the inverse on the plan p (Ls step rows per utterance, lengths p.lensS): WN k -- start on columns o .. o + h - 1
// of the state `in`, then per layer the cond and in-layer GEMMs, the gate and the res / skip GEMMs -- and flow_tail from
// `in` into `out` (which may be `in`).  *wn (nullable): the buffer that holds WN's skip sum (before `end`).
int flow(const fs2_waveglow_net* m, int k, const WgPlan& p, const void* cond_a, const float* in, float* out, int B, int Ls, int* status,
         cudaStream_t st, const float** wn = nullptr) {
  const int kind = out_kind(m->math_mode), C = m->C;
  const bool planes = plane_mode(m->math_mode);
  const long rows = (long)B * Ls;
  const int64_t* win = p.winS;
  const WFlow& f = m->flows[k];
  const int c = flow_channels(k), h = c / 2, o = kGroup - c;
  const int exact = (kFlows - 1 - k) * kFlowReach;          // a window's rows are exact this far from an interior side
  auto start = pick(kind, wg_start_kernel<OUT_HILO>, wg_start_kernel<OUT_HI>, wg_start_kernel<OUT_F32>);
  auto gate = pick(kind, wg_gate_kernel<OUT_HILO>, wg_gate_kernel<OUT_HI>, wg_gate_kernel<OUT_F32>);
  int rc;
  start<<<grid_for(rows * (C / 4), 256), 256, 0, st>>>(in, p.lensS, win, exact, B, Ls, C, o, h, f.start_w, f.start_b, p.x[0], p.xp, status);
  FS2_LAUNCH_CHECK();
  int cur = 0, sk = 0;
  for (int i = 0; i < kLayers; ++i) {
    if ((rc = vweight_gemm(m->math_mode, f.cond[i], cond_a, B, Ls, ACT_NONE, p.lensS, p.cd, st))) return rc;
    const void* xa = planes ? (const void*)p.xp : (const void*)p.x[cur];
    if ((rc = vweight_gemm(m->math_mode, f.in[i], xa, B, Ls, ACT_NONE, p.lensS, p.ia, st, p.cd, 1 << i))) return rc;
    // layer i's input x is exact at exact + 2^i - 1, its in-layer output (and so acts and the next x) at exact + 2^(i+1) - 1
    gate<<<grid_for(rows * (C / 4), 256), 256, 0, st>>>(p.ia, planes && i > 0 ? p.x[cur] : nullptr, p.lensS, win, exact + (2 << i) - 1,
                                                         exact + (1 << i) - 1, B, Ls, C, (float*)p.acts, (__half*)p.acts, status);
    FS2_LAUNCH_CHECK();
    if (i < kLayers - 1) {
      if ((rc = vweight_gemm(m->math_mode, f.res[i], p.acts, B, Ls, ACT_NONE, p.lensS, p.x[cur ^ 1], st, p.x[cur], 1, p.xp))) return rc;
      cur ^= 1;
    }
    if ((rc = vweight_gemm(m->math_mode, f.skip[i], p.acts, B, Ls, ACT_NONE, p.lensS, p.skip[sk ^ 1], st, i ? p.skip[sk] : nullptr))) return rc;
    sk ^= 1;
  }
  if (wn) *wn = p.skip[sk];
  return flow_tail(m, k, p.skip[sk], in, out, p.lensS, B, Ls, st);
}

// The inverse flow on the plan p: whole utterances (starts == nullptr; buffers of Lmax frames, audio written by the last
// flow) or a window of nf frames from starts[b] (buffers of nf + 2H frames, the window descriptors p.lens, the core copied
// out by wg_win_audio_kernel).  audio rows ld samples apart.  Both enqueue the same kernels but the first and the last.
int run(const fs2_waveglow_net* m, const WgPlan& p, const float* mels, const int64_t* olens, const int64_t* starts, int B, int Lmax,
        int nf, double sigma, const int64_t* seeds, const float* z, float* audio, long ld, int* status, cudaStream_t st) {
  const bool window = starts != nullptr;
  const int L = window ? nf + 2 * kHalo : Lmax;
  const int Ls = L * kSteps;
  const long rows = (long)B * Ls;
  int rc;

  if ((rc = ups_prep(olens, starts, B, 1, Lmax, nf, kPlan, p.lens, status, st))) return rc;
  wg_noise_kernel<<<grid_for(rows * 2, 256), 256, 0, st>>>(z, Lmax * kSteps, seeds, p.lensS, p.winS, 1, B, Ls, sigma, p.state, nullptr);
  FS2_LAUNCH_CHECK();
  const void* cond_a = nullptr;
  if ((rc = upsample(m, p, mels, B, L, Lmax, status, st, &cond_a))) return rc;
  for (int k = kFlows - 1; k >= 0; --k)
    if ((rc = flow(m, k, p, cond_a, p.state, k == 0 && !window ? audio : p.state, B, Ls, status, st))) return rc;
  if (window) {
    wg_win_audio_kernel<<<grid_for((long)B * nf * kHop, 256), 256, 0, st>>>(p.state, p.winS, p.lens + 3L * win_audio(kPlan) * B, B, Ls,
                                                                           nf, audio, ld);
    FS2_LAUNCH_CHECK();
  }
  return FS2_OK;
}

}  // namespace
}  // namespace fs2

using namespace fs2;

extern "C" {

int fs2_waveglow_create(fs2_waveglow_net** out, int math_mode, int n_channels) {
  FS2_REQUIRE(out, "fs2_waveglow_create: null argument");
  FS2_REQUIRE(math_mode >= FS2_MATH_FP32 && math_mode <= FS2_MATH_F16, "fs2_waveglow_create: bad math_mode %d", math_mode);
  FS2_REQUIRE(n_channels >= 64 && n_channels <= 1024 && n_channels % 64 == 0,
              "fs2_waveglow_create: n_channels must be a multiple of 64 in [64, 1024] (got %d)", n_channels);
  fs2_waveglow_net* m = new fs2_waveglow_net();
  m->math_mode = math_mode;
  m->C = n_channels;
  FS2_CUDA_CHECK(cudaGetDevice(&m->device));
  *out = m;
  return FS2_OK;
}

void fs2_waveglow_destroy(fs2_waveglow_net* m) { destroy_gen(m); }

int fs2_waveglow_load(fs2_waveglow_net* m, const float* const* t, int n, void* stream) {
  FS2_REQUIRE(m && t, "fs2_waveglow_load: null argument");
  FS2_REQUIRE(n == kTensors, "fs2_waveglow_load: expected %d tensors, got %d", kTensors, n);
  for (int i = 0; i < n; ++i) FS2_REQUIRE(t[i], "fs2_waveglow_load: tensor %d is null", i);
  cudaStream_t st = (cudaStream_t)stream;
  const int C = m->C;
  // GEMM weights in the order they are carved and packed: (weight, source tensor index, N row offset in it)
  struct Job { VWeight* w; int src, bsrc, bsrc2, row0; };
  Job jobs[1 + kFlows * (4 * kLayers - 1)];
  int nj = 0;
  m->up.N = kUpN; m->up.K = kUpK;
  jobs[nj++] = {&m->up, 0, 1, -1, 0};
  for (int k = 0; k < kFlows; ++k) {
    WFlow& f = m->flows[k];
    const int base = 2 + k * kPerFlow;        // start.w, start.b, in.{i}.(w, b), cond.{i}.(w, b), res_skip.{i}.(w, b), end.w, end.b, winv
    for (int i = 0; i < kLayers; ++i) {
      const int in_w = base + 2 + 2 * i, cond_w = base + 2 + 2 * kLayers + 2 * i, rs_w = base + 2 + 4 * kLayers + 2 * i;
      f.in[i].N = 2 * C; f.in[i].K = C; f.in[i].taps = 3;
      jobs[nj++] = {&f.in[i], in_w, -1, -1, 0};
      f.cond[i].N = 2 * C; f.cond[i].K = kCond;
      jobs[nj++] = {&f.cond[i], cond_w, cond_w + 1, in_w + 1, 0};          // bias = b_cond + b_in
      if (i < kLayers - 1) {
        f.res[i].N = C; f.res[i].K = C;
        jobs[nj++] = {&f.res[i], rs_w, rs_w + 1, -1, 0};
      }
      f.skip[i].N = C; f.skip[i].K = C;
      jobs[nj++] = {&f.skip[i], rs_w, rs_w + 1, -1, i < kLayers - 1 ? C : 0};
    }
  }
  m->loaded = false;
  int rc = arena_carve(&m->arena, &m->arena_bytes, st, [&](Bump& b) {
    for (int j = 0; j < nj; ++j) vweight_carve(b, *jobs[j].w, jobs[j].bsrc >= 0);
    for (int k = 0; k < kFlows; ++k) {
      WFlow& f = m->flows[k];
      const int c = flow_channels(k), h = c / 2;
      f.start_w = b.floats((size_t)C * h); f.start_b = b.floats(C);
      f.end_w = b.floats((size_t)c * C); f.end_b = b.floats(c); f.winv = b.floats((size_t)c * c);
    }
    return FS2_OK;
  });
  if (rc) return rc;
  for (int j = 0; j < nj; ++j) {
    const Job& q = jobs[j];
    VWeight* w = q.w;
    const long e = (long)w->taps * w->N * w->K;
    if (j == 0) {
      wg_pack_up_kernel<<<grid_for(e, 256), 256, 0, st>>>(t[0], t[1], w->w, w->bias);
      FS2_LAUNCH_CHECK();
    } else if (w->taps > 1) {
      wg_pack_taps_kernel<<<grid_for(e, 256), 256, 0, st>>>(t[q.src], w->N, w->K, w->taps, w->w);
      FS2_LAUNCH_CHECK();
    } else {
      FS2_CUDA_CHECK(cudaMemcpyAsync(w->w, t[q.src] + (long)q.row0 * w->K, e * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    if (j > 0 && q.bsrc >= 0) {
      if (q.bsrc2 >= 0) {
        wg_add_kernel<<<grid_for(w->N, 256), 256, 0, st>>>(t[q.bsrc], t[q.bsrc2], w->N, w->bias);
        FS2_LAUNCH_CHECK();
      } else {
        FS2_CUDA_CHECK(cudaMemcpyAsync(w->bias, t[q.bsrc] + q.row0, w->N * sizeof(float), cudaMemcpyDeviceToDevice, st));
      }
    }
    if ((rc = vweight_planes(*w, st))) return rc;
  }
  for (int k = 0; k < kFlows; ++k) {
    WFlow& f = m->flows[k];
    const int c = flow_channels(k), h = c / 2, base = 2 + k * kPerFlow, tail = base + 2 + 6 * kLayers;
    FS2_CUDA_CHECK(cudaMemcpyAsync(f.start_w, t[base], (size_t)C * h * sizeof(float), cudaMemcpyDeviceToDevice, st));
    FS2_CUDA_CHECK(cudaMemcpyAsync(f.start_b, t[base + 1], (size_t)C * sizeof(float), cudaMemcpyDeviceToDevice, st));
    FS2_CUDA_CHECK(cudaMemcpyAsync(f.end_w, t[tail], (size_t)c * C * sizeof(float), cudaMemcpyDeviceToDevice, st));
    FS2_CUDA_CHECK(cudaMemcpyAsync(f.end_b, t[tail + 1], (size_t)c * sizeof(float), cudaMemcpyDeviceToDevice, st));
    FS2_CUDA_CHECK(cudaMemcpyAsync(f.winv, t[tail + 2], (size_t)c * c * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  m->loaded = true;
  return FS2_OK;
}

int fs2_waveglow_workspace_bytes(fs2_waveglow_net* m, int B, int Lmax, size_t* bytes) {
  FS2_REQUIRE(m && bytes, "fs2_waveglow_workspace_bytes: null argument");
  int rc = check_size(m, B, Lmax);
  if (rc) return rc;
  Bump b(nullptr, 0);
  plan(b, m->math_mode, m->C, B, Lmax);
  *bytes = b.off + 256;
  return FS2_OK;
}

int fs2_waveglow_noise(const int64_t* seeds, const int64_t* olens, int B, int Lmax, float* z, void* stream) {
  FS2_REQUIRE(seeds && olens && z, "fs2_waveglow_noise: null argument");
  FS2_REQUIRE(B >= 1 && Lmax >= 1 && (long)B * Lmax * kSteps < (1L << 31), "fs2_waveglow_noise: bad shape B=%d Lmax=%d", B, Lmax);
  const int Ls = Lmax * kSteps;
  wg_noise_kernel<<<grid_for((long)B * Ls * 2, 256), 256, 0, (cudaStream_t)stream>>>(nullptr, Ls, seeds, olens, nullptr, kSteps, B, Ls, 1.0,
                                                                                   nullptr, z);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int fs2_waveglow(fs2_waveglow_net* m, const float* mels, const int64_t* olens, int B, int Lmax, double sigma, const int64_t* seeds,
                 const float* z, float* audio, int* status, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(m && mels && olens && audio && status && ws && (seeds || z), "fs2_waveglow: null argument");
  FS2_REQUIRE(m->loaded, "fs2_waveglow: weights not loaded (fs2_waveglow_load)");
  FS2_REQUIRE((reinterpret_cast<uintptr_t>(mels) & 15) == 0, "fs2_waveglow: mels must be 16-byte aligned");
  FS2_REQUIRE(isfinite(sigma) && sigma >= 0.0, "fs2_waveglow: sigma must be finite and >= 0");
  int rc = check_size(m, B, Lmax);
  if (rc) return rc;
  Bump b(ws, ws_bytes);
  WgPlan p = plan(b, m->math_mode, m->C, B, Lmax);
  if ((rc = b.check("fs2_waveglow"))) return rc;
  return run(m, p, mels, olens, nullptr, B, Lmax, 0, sigma, seeds, z, audio, (long)Lmax * kHop, status, (cudaStream_t)stream);
}

int fs2_waveglow_window_workspace_bytes(fs2_waveglow_net* m, int B, int n_frames, size_t* bytes) {
  FS2_REQUIRE(m && bytes, "fs2_waveglow_window_workspace_bytes: null argument");
  int rc = check_window(m, B, n_frames);
  if (rc) return rc;
  Bump b(nullptr, 0);
  plan(b, m->math_mode, m->C, B, n_frames + 2 * kHalo, true);
  *bytes = b.off + 256;
  return FS2_OK;
}

int fs2_waveglow_window(fs2_waveglow_net* m, const float* mels, const int64_t* olens, const int64_t* starts, int B, int Lmax,
                        int n_frames, double sigma, const int64_t* seeds, const float* z, float* audio, int64_t audio_ld,
                        int* status, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(m && mels && olens && starts && audio && status && ws && (seeds || z), "fs2_waveglow_window: null argument");
  FS2_REQUIRE((reinterpret_cast<uintptr_t>(mels) & 15) == 0, "fs2_waveglow_window: mels must be 16-byte aligned");
  FS2_REQUIRE(isfinite(sigma) && sigma >= 0.0, "fs2_waveglow_window: sigma must be finite and >= 0");
  int rc = check_window(m, B, n_frames);
  if (rc) return rc;
  if ((rc = check_window_extent("fs2_waveglow_window", Lmax, 0, kSteps, n_frames, audio_ld))) return rc;
  Bump b(ws, ws_bytes);
  WgPlan p = plan(b, m->math_mode, m->C, B, n_frames + 2 * kHalo, true);
  if ((rc = b.check("fs2_waveglow_window"))) return rc;
  FS2_REQUIRE(m->loaded, "fs2_waveglow_window: weights not loaded (fs2_waveglow_load)");
  return run(m, p, mels, olens, starts, B, Lmax, n_frames, sigma, seeds, z, audio, (long)audio_ld, status, (cudaStream_t)stream);
}

// ---- stages of the inverse on the vocoder's own code paths (tests) --------------------------------------------------
// Both run what fs2_waveglow runs for that stage, on a loaded handle's packed weights, with the buffers in a stream-ordered
// temporary.  The length pass is ups_prep's with 0 allowed: a length outside [0, L] is 0 and sets FS2_WAVEGLOW_BAD_LENGTH,
// so it never becomes an out-of-bounds row.
int fs2_op_waveglow_upsample(fs2_waveglow_net* m, const float* mels, const int64_t* olens, int B, int Lmax, float* cond,
                             float* cond_planes, int* status, void* stream) {
  const char* who = "fs2_op_waveglow_upsample";
  // the checks that need no handle first, so that each refusal names its own cause
  FS2_REQUIRE(mels && olens && cond && status, "%s: null argument", who);
  FS2_REQUIRE(B >= 1 && Lmax >= 1, "%s: need B >= 1 and Lmax >= 1 (got %d, %d)", who, B, Lmax);
  FS2_REQUIRE(aligned16(mels) && aligned16(cond) && aligned16(cond_planes), "%s: mels, cond and cond_planes must be 16-byte aligned", who);
  FS2_REQUIRE(m && m->loaded, "%s: null or unloaded handle (fs2_waveglow_load)", who);
  const bool planes = plane_mode(m->math_mode);
  FS2_REQUIRE(!cond_planes || planes, "%s: cond_planes needs FS2_MATH_F16 or FS2_MATH_3XTF32", who);
  int rc = check_rows(who, "B * Lmax * 32", "step", (long)B * Lmax * kSteps, m->math_mode);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const long rows = (long)B * Lmax * kSteps;
  WgPlan p{};
  void* base = nullptr;
  if ((rc = temp_carve(&base, st, [&](Bump& b) {
         p.lens = (int64_t*)b.bytes((size_t)(kPlan.n + 1) * B * sizeof(int64_t));
         p.up_a = b.floats((size_t)B * Lmax * kUpK);
         p.condp = planes ? (__half*)b.floats((size_t)rows * kCond) : nullptr;   // hi + lo planes
       })))
    return rc;
  p.lensF = p.lens;
  p.lensS = p.lens + B;
  p.cond = cond;
  auto enqueue = [&]() -> int {      // every error returns here, so that the temporary is released on every path
    if (int r = ups_prep(olens, nullptr, B, 0, Lmax, 0, kPlan, p.lens, status, st)) return r;
    // the planes of rows past lens are never written: zeros there (and in f16's unused lo plane) read back as +0
    if (planes) FS2_CUDA_CHECK(cudaMemsetAsync(p.condp, 0, (size_t)rows * kCond * sizeof(float), st));
    const void* cond_a = nullptr;
    int r = upsample(m, p, mels, B, Lmax, Lmax, status, st, &cond_a);
    if (!r && cond_planes) r = planes_to_rows(p.condp, rows * kCond, cond_planes, st);
    return r;
  };
  rc = enqueue();
  cudaFreeAsync(base, st);
  return rc;
}

int fs2_op_waveglow_flow(fs2_waveglow_net* m, int k, const float* cond, const float* skip_in, const float* state_in, float* state_out,
                         const int64_t* lens, int B, int Ls, float* wn_out, int* status, void* stream) {
  const char* who = "fs2_op_waveglow_flow";
  // the checks that need no handle first, so that each refusal names its own cause
  FS2_REQUIRE(state_in && state_out && lens && status && (skip_in || cond), "%s: null argument", who);
  FS2_REQUIRE(!(skip_in && wn_out), "%s: wn_out needs the WN to run (skip_in NULL)", who);
  FS2_REQUIRE(k >= 0 && k < kFlows, "%s: flow k must lie in [0, %d) (got %d)", who, kFlows, k);
  FS2_REQUIRE(B >= 1 && Ls >= 1, "%s: need B >= 1 and Ls >= 1 (got %d, %d)", who, B, Ls);
  FS2_REQUIRE(aligned16(cond) && aligned16(skip_in) && aligned16(state_in) && aligned16(state_out) && aligned16(wn_out),
              "%s: cond, skip_in, state_in, state_out and wn_out must be 16-byte aligned", who);
  FS2_REQUIRE(m && m->loaded, "%s: null or unloaded handle (fs2_waveglow_load)", who);
  int rc = check_rows(who, "B * Ls", "step", (long)B * Ls, m->math_mode);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const bool planes = plane_mode(m->math_mode);
  const long rows = (long)B * Ls;
  WgPlan p{};
  void* base = nullptr;
  if ((rc = temp_carve(&base, st, [&](Bump& b) {
         p.lensS = (int64_t*)b.bytes((size_t)B * sizeof(int64_t));      // ups_prep's block for kStepPlan
         if (!skip_in) plan_wn(b, p, planes, m->C, (size_t)rows);
       })))
    return rc;
  auto enqueue = [&]() -> int {      // every error returns here, so that the temporary is released on every path
    if (int r = ups_prep(lens, nullptr, B, 0, Ls, 0, kStepPlan, p.lensS, status, st)) return r;
    if (skip_in) return flow_tail(m, k, skip_in, state_in, state_out, p.lensS, B, Ls, st);
    const void* cond_a = cond;
    if (planes) {     // the cond planes with the range check, as the vocoder's upsampling writes them
      auto kp = out_kind(m->math_mode) == OUT_HILO ? wg_planes_kernel<OUT_HILO> : wg_planes_kernel<OUT_HI>;
      kp<<<grid_for(rows * (kCond / 4), 256), 256, 0, st>>>(cond, p.lensS, B, Ls, kCond, p.condp, status);
      FS2_LAUNCH_CHECK();
      cond_a = p.condp;
    }
    const float* wn = nullptr;
    int r = flow(m, k, p, cond_a, state_in, state_out, B, Ls, status, st, &wn);
    if (!r && wn_out) FS2_CUDA_CHECK(cudaMemcpyAsync(wn_out, wn, (size_t)rows * m->C * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return r;
  };
  rc = enqueue();
  cudaFreeAsync(base, st);
  return rc;
}

}  // extern "C"
