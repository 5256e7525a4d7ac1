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
// Launches per call: 4 + 12 * 41 = 496, plus 1 (the cond planes) in f16 / 3xF16.
//
// A GEMM row depends only on its own input rows (the in-layer GEMM: rows t, t +- 2^i of its own utterance, zero outside
// [0, olens * 32)), in a fixed K order, so per-utterance results do not depend on the batch.
#include <math.h>
#include <string.h>

#include "operand_planes.cuh"

namespace fs2 {
namespace {

constexpr int kMels = 80, kHop = 256, kGroup = 8, kSteps = kHop / kGroup, kFlows = 12, kLayers = 8;
constexpr int kCond = kMels * kGroup;          // 640 cond channels per step
constexpr int kUpTaps = 4, kUpK = kUpTaps * kMels, kUpN = kMels * kHop, kUpKernel = kUpTaps * kHop;
constexpr int kPerFlow = 2 + 6 * kLayers + 3;  // tensors per flow in fs2_waveglow_load
constexpr int kTensors = 2 + kFlows * kPerFlow;

__host__ __device__ inline int flow_channels(int k) { return k < 4 ? 8 : k < 8 ? 6 : 4; }

inline int grid_for(long n, int block, int cap = 132 * 8) {
  long g = (n + block - 1) / block;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// four GEMM-operand values at element offset off (a multiple of 4) of a [rows][K] operand; plane = rows * K
template <int OUT>
__device__ __forceinline__ void put_quad(float4 v, long off, float* __restrict__ out32, __half* __restrict__ outp, long plane,
                                         int* __restrict__ status) {
  if (OUT == OUT_F32) {
    *reinterpret_cast<float4*>(out32 + off) = v;
    return;
  }
  if (!(fabsf(v.x) <= kPlaneMax && fabsf(v.y) <= kPlaneMax && fabsf(v.z) <= kPlaneMax && fabsf(v.w) <= kPlaneMax))
    atomicOr(status, FS2_WAVEGLOW_RANGE);               // saturation is reported, not hidden
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

// one CTA: lensF[b] = olens[b], lensS[b] = olens[b] * 32 for 1 <= olens[b] <= L, else 0 (the utterance is skipped);
// *status = 0 or FS2_WAVEGLOW_BAD_LENGTH.  Runs first, so the producers' range bits land on a cleared word.
__global__ void wg_prep_kernel(const int64_t* __restrict__ olens, int B, int L, int64_t* __restrict__ lensF,
                               int64_t* __restrict__ lensS, int* __restrict__ status) {
  __shared__ int bad;
  if (threadIdx.x == 0) bad = 0;
  __syncthreads();
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const int64_t n = olens[b];
    const bool ok = n >= 1 && n <= L;
    if (!ok) atomicOr(&bad, 1);
    lensF[b] = ok ? n : 0;
    lensS[b] = ok ? n * kSteps : 0;
  }
  __syncthreads();
  if (threadIdx.x == 0) *status = bad ? FS2_WAVEGLOW_BAD_LENGTH : 0;
}

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

// The standard-normal draw z [B, 8, Ls] for the steps t < n_b = min(lens[b] * mult, Ls): from zin (same layout) or from
// Philox keyed by seeds[b].  state [B * Ls][8] (nullable) = fp32(sigma * z), the product in double and rounded once;
// zout [B, 8, Ls] (nullable) = z; both 0 for t >= n_b.  zin is never read there.
__global__ void wg_noise_kernel(const float* __restrict__ zin, const int64_t* __restrict__ seeds, const int64_t* __restrict__ lens,
                                int mult, int B, int Ls, double sigma, float* __restrict__ state, float* __restrict__ zout) {
  const long total = (long)B * Ls * 2;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i >> 1;
    const int q = (int)(i & 1), b = (int)(row / Ls), t = (int)(row - (long)b * Ls);
    long n = lens[b] * mult;
    n = n < 0 ? 0 : (n > Ls ? Ls : n);
    float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t < n) {
      if (zin) {
        const float* zb = zin + ((long)b * kGroup + 4 * q) * Ls + t;
        z = make_float4(zb[0], zb[Ls], zb[2L * Ls], zb[3L * Ls]);
      } else {
        z = normal4((uint64_t)seeds[b], (uint32_t)t, (uint32_t)q);
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
// Rows t >= n are not written (the GEMM writes 0 there); frames past olens[b] are never read.
template <int OUT>
__global__ void wg_up_operand_kernel(const float* __restrict__ mels, const int64_t* __restrict__ lensF, int B, int L,
                                     float* __restrict__ out32, __half* __restrict__ outp, int* __restrict__ status) {
  constexpr int Q = kUpK / 4;
  const long rows = (long)B * L, total = rows * Q, plane = rows * kUpK;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / Q;
    const int k = (int)(i - row * Q) * 4, j = k / kMels, c = k - j * kMels;
    const int b = (int)(row / L), t = (int)(row - (long)b * L), n = (int)lensF[b];
    if (t >= n) continue;
    const int src = t - (kUpTaps - 1) + j;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (src >= 0 && src < n) v = *reinterpret_cast<const float4*>(mels + ((long)b * L + src) * kMels + c);
    put_quad<OUT>(v, row * kUpK + k, out32, outp, plane, status);
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
    put_quad<OUT>(*reinterpret_cast<const float4*>(x + off), off, nullptr, outp, plane, status);
  }
}

// WN start: x[r][n] = bias[n] + sum_{q < h} w[n][q] * state[r][o + q] for t < lens[b], else 0 -- fp32 rows (the residual
// stream) and, in the plane modes, the in-layer GEMM's operand planes.  Padded rows are written: the dilated taps read them.
template <int OUT>
__global__ void wg_start_kernel(const float* __restrict__ state, const int64_t* __restrict__ lens, int B, int Ls, int C, int o, int h,
                                const float* __restrict__ w, const float* __restrict__ bias, float* __restrict__ x,
                                __half* __restrict__ xp, int* __restrict__ status) {
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
    if (OUT != OUT_F32) put_quad<OUT>(v, row * C + n, nullptr, xp, plane, status);
  }
}

// gate: acts[r][c] = tanh(ia[r][c]) * sigmoid(ia[r][C + c]) as the res / skip GEMMs' operand (rows t >= lens[b] are not
// written).  xchk (nullable, plane modes): the layer's input rows x, written as planes by the previous res GEMM's
// epilogue, are range-checked here.
template <int OUT>
__global__ void wg_gate_kernel(const float* __restrict__ ia, const float* __restrict__ xchk, const int64_t* __restrict__ lens, int B,
                               int Ls, int C, float* __restrict__ out32, __half* __restrict__ outp, int* __restrict__ status) {
  const int Q = C / 4;
  const long rows = (long)B * Ls, total = rows * Q, plane = rows * C;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / Q;
    const int c = (int)(i - row * Q) * 4;
    const int b = (int)(row / Ls), t = (int)(row - (long)b * Ls);
    if (t >= (int)lens[b]) continue;
    const float4 a = *reinterpret_cast<const float4*>(ia + row * 2 * C + c);
    const float4 g = *reinterpret_cast<const float4*>(ia + row * 2 * C + C + c);
    const float4 v = make_float4(tanhf(a.x) * (1.f / (1.f + expf(-g.x))), tanhf(a.y) * (1.f / (1.f + expf(-g.y))),
                                 tanhf(a.z) * (1.f / (1.f + expf(-g.z))), tanhf(a.w) * (1.f / (1.f + expf(-g.w))));
    put_quad<OUT>(v, row * C + c, out32, outp, plane, status);
    if (xchk) {
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

struct WWeight {               // one GEMM weight [taps][N][K]: fp32 (fp32 / tf32 families) and scaled fp16 planes, bias [N]
  float* w = nullptr; __half* hi = nullptr; __half* lo = nullptr; float* sc = nullptr; float* bias = nullptr;   // sc = [scale, 1 / scale]
  int N = 0, K = 0, taps = 1;
};

struct WFlow {
  float *start_w = nullptr, *start_b = nullptr;   // [C][h], [C]
  WWeight cond[kLayers], in[kLayers], res[kLayers - 1], skip[kLayers];
  float *end_w = nullptr, *end_b = nullptr;       // [2h][C], [2h]
  float* winv = nullptr;                          // [c][c]
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

struct fs2_waveglow_net {
  int device = 0, math_mode = 0, C = 0;
  bool loaded = false;
  void* arena = nullptr;
  fs2::WWeight up;
  fs2::WFlow flows[fs2::kFlows];
};

namespace fs2 {
namespace {

struct WgPlan {
  int64_t* lensF;      // [B] frame lengths (0 for a bad olens[b])
  int64_t* lensS;      // [B] step lengths = lensF * 32
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

bool plane_mode(int mode) { return mode == FS2_MATH_F16 || mode == FS2_MATH_3XTF32; }

WgPlan plan(Bump& b, int mode, int C, int B, int L) {
  const size_t frames = (size_t)B * L, rows = frames * kSteps;
  const bool planes = plane_mode(mode);
  WgPlan p;
  p.lensF = (int64_t*)b.bytes((size_t)B * sizeof(int64_t));
  p.lensS = (int64_t*)b.bytes((size_t)B * sizeof(int64_t));
  p.up_a = b.floats(frames * kUpK);                   // fp32 rows, or hi + lo planes: the same bytes
  p.state = b.floats(rows * kGroup);
  p.x[0] = b.floats(rows * C);
  p.x[1] = b.floats(rows * C);
  p.xp = planes ? (__half*)b.floats(rows * C) : nullptr;
  p.cd = b.floats(rows * 2 * C);
  p.ia = b.floats(rows * 2 * C);
  p.acts = b.floats(rows * C);
  p.skip[0] = b.floats(rows * C);
  p.skip[1] = b.floats(rows * C);
  p.condp = planes ? (__half*)b.floats(rows * kCond) : nullptr;
  p.cond = planes && 2 * C >= kCond ? p.ia : b.floats(rows * kCond);    // ia holds rows * 2C floats
  return p;
}

// out [B * L][w.N] = a [B * L][w.K] (taps at dilation dil) . w^T + bias (+ resid), rows t >= lens[b] written as 0 (and
// skipped by the tensor-core kernel); outp (plane modes, nullable): the result's operand planes as well
int gemm(const fs2_waveglow_net* m, const WWeight& w, const void* a, int B, int L, const int64_t* lens, int dil, const float* resid,
         float* out, __half* outp, cudaStream_t st) {
  TapGemm g;
  memset(&g, 0, sizeof(g));
  g.B = B; g.L = L; g.K = w.K; g.N = w.N; g.taps = w.taps; g.dil = dil; g.act = ACT_NONE; g.out = out; g.ldo = w.N; g.lens = lens;
  g.w = w.w; g.bias = w.bias; g.resid = resid; g.ldr = w.N; g.a_inv = 1.0f; g.ldx = w.K;
  if (!plane_mode(m->math_mode)) {
    g.x = (const float*)a;
    return m->math_mode == FS2_MATH_FP32 ? tap_gemm_fp32(g, st) : tap_gemm_tf32(g, st);
  }
  g.xp = (const __half*)a; g.w_hi = w.hi; g.w_lo = w.lo; g.w_inv = w.sc + 1; g.a_inv = kPlaneInv;
  g.precise = m->math_mode == FS2_MATH_3XTF32;
  if (outp) { g.outp = outp; g.ldo_p = w.N; g.outp_lo = g.precise; }
  return tap_gemm_planes(g, st);
}

int check_size(const fs2_waveglow_net* m, int B, int L) {
  FS2_REQUIRE(B >= 1 && L >= 1, "fs2_waveglow: need B >= 1 and Lmax >= 1 (got %d, %d)", B, L);
  const long rows = (long)B * L * kSteps;
  FS2_REQUIRE(rows < (1L << 31), "fs2_waveglow: B * Lmax * 32 = %ld step rows exceed the int32 row index", rows);
  // the CUDA-core GEMM puts row tiles of 128 on grid.y (at most 65535)
  FS2_REQUIRE(m->math_mode != FS2_MATH_FP32 || rows <= 65535L * 128,
              "fs2_waveglow: B * Lmax * 32 = %ld step rows exceed fp32 mode's limit of %ld", rows, 65535L * 128);
  return FS2_OK;
}

template <typename K>
int launch_flow(K kernel, int c, int C, const float* skip, const float* in, float* out, const int64_t* lens, int B, int Ls, int o,
                const WFlow& f, cudaStream_t st) {
  const size_t smem = (size_t)(c * C + c * c + c) * sizeof(float);
  kernel<<<grid_for((long)B * Ls, 8), 256, smem, st>>>(skip, C, in, out, lens, B, Ls, o, f.end_w, f.end_b, f.winv);
  FS2_LAUNCH_CHECK();
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

void fs2_waveglow_destroy(fs2_waveglow_net* m) {
  if (!m) return;
  if (m->arena) cudaFree(m->arena);
  delete m;
}

int fs2_waveglow_load(fs2_waveglow_net* m, const float* const* t, int n, void* stream) {
  FS2_REQUIRE(m && t, "fs2_waveglow_load: null argument");
  FS2_REQUIRE(n == kTensors, "fs2_waveglow_load: expected %d tensors, got %d", kTensors, n);
  for (int i = 0; i < n; ++i) FS2_REQUIRE(t[i], "fs2_waveglow_load: tensor %d is null", i);
  cudaStream_t st = (cudaStream_t)stream;
  const int C = m->C;
  // GEMM weights in the order they are carved and packed: (weight, source tensor index, N row offset in it)
  struct Job { WWeight* w; int src, bsrc, bsrc2, row0; };
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
  for (int pass = 0; pass < 2; ++pass) {       // pass 0 sizes the arena, pass 1 carves it
    Bump b(pass ? m->arena : nullptr, pass ? (size_t)-1 : 0);
    for (int j = 0; j < nj; ++j) {
      WWeight* w = jobs[j].w;
      const size_t e = (size_t)w->taps * w->N * w->K;
      w->w = b.floats(e); w->hi = (__half*)b.bytes(e * 2); w->lo = (__half*)b.bytes(e * 2); w->sc = b.floats(2);
      w->bias = jobs[j].bsrc >= 0 ? b.floats(w->N) : nullptr;
    }
    for (int k = 0; k < kFlows; ++k) {
      WFlow& f = m->flows[k];
      const int c = flow_channels(k), h = c / 2;
      f.start_w = b.floats((size_t)C * h); f.start_b = b.floats(C);
      f.end_w = b.floats((size_t)c * C); f.end_b = b.floats(c); f.winv = b.floats((size_t)c * c);
    }
    if (pass == 0) {
      if (m->arena) { FS2_CUDA_CHECK(cudaStreamSynchronize(st)); FS2_CUDA_CHECK(cudaFree(m->arena)); m->arena = nullptr; }
      m->loaded = false;
      FS2_CUDA_CHECK(cudaMalloc(&m->arena, b.off + 256));
    }
  }
  for (int j = 0; j < nj; ++j) {
    const Job& q = jobs[j];
    WWeight* w = q.w;
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
    int rc = weight_scale(w->w, e, w->sc, w->sc + 1, st); if (rc) return rc;
    rc = split_f16(w->w, w->hi, w->lo, e, w->sc, st); if (rc) return rc;
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
  wg_noise_kernel<<<grid_for((long)B * Ls * 2, 256), 256, 0, (cudaStream_t)stream>>>(nullptr, seeds, olens, kSteps, B, Ls, 1.0, nullptr, z);
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
  cudaStream_t st = (cudaStream_t)stream;
  Bump b(ws, ws_bytes);
  WgPlan p = plan(b, m->math_mode, m->C, B, Lmax);
  if (!b.ok()) { set_error("fs2_waveglow: workspace too small (%zu < %zu)", ws_bytes, b.off); return FS2_ERR_WORKSPACE; }
  const int kind = out_kind(m->math_mode), C = m->C, Ls = Lmax * kSteps;
  const bool planes = plane_mode(m->math_mode);
  const long rows = (long)B * Ls;

  wg_prep_kernel<<<1, 256, 0, st>>>(olens, B, Lmax, p.lensF, p.lensS, status);
  FS2_LAUNCH_CHECK();
  wg_noise_kernel<<<grid_for(rows * 2, 256), 256, 0, st>>>(z, seeds, p.lensS, 1, B, Ls, sigma, p.state, nullptr);
  FS2_LAUNCH_CHECK();
  {
    auto k = pick(kind, wg_up_operand_kernel<OUT_HILO>, wg_up_operand_kernel<OUT_HI>, wg_up_operand_kernel<OUT_F32>);
    k<<<grid_for((long)B * Lmax * (kUpK / 4), 256), 256, 0, st>>>(mels, p.lensF, B, Lmax, (float*)p.up_a, (__half*)p.up_a, status);
    FS2_LAUNCH_CHECK();
  }
  if ((rc = gemm(m, m->up, p.up_a, B, Lmax, p.lensF, 1, nullptr, p.cond, nullptr, st))) return rc;
  if (planes) {
    auto k = kind == OUT_HILO ? wg_planes_kernel<OUT_HILO> : wg_planes_kernel<OUT_HI>;
    k<<<grid_for(rows * (kCond / 4), 256), 256, 0, st>>>(p.cond, p.lensS, B, Ls, kCond, p.condp, status);
    FS2_LAUNCH_CHECK();
  }
  const void* cond_a = planes ? (const void*)p.condp : (const void*)p.cond;
  auto start = pick(kind, wg_start_kernel<OUT_HILO>, wg_start_kernel<OUT_HI>, wg_start_kernel<OUT_F32>);
  auto gate = pick(kind, wg_gate_kernel<OUT_HILO>, wg_gate_kernel<OUT_HI>, wg_gate_kernel<OUT_F32>);
  for (int k = kFlows - 1; k >= 0; --k) {
    const WFlow& f = m->flows[k];
    const int c = flow_channels(k), h = c / 2, o = kGroup - c;
    start<<<grid_for(rows * (C / 4), 256), 256, 0, st>>>(p.state, p.lensS, B, Ls, C, o, h, f.start_w, f.start_b, p.x[0], p.xp, status);
    FS2_LAUNCH_CHECK();
    int cur = 0, sk = 0;
    for (int i = 0; i < kLayers; ++i) {
      if ((rc = gemm(m, f.cond[i], cond_a, B, Ls, p.lensS, 1, nullptr, p.cd, nullptr, st))) return rc;
      const void* xa = planes ? (const void*)p.xp : (const void*)p.x[cur];
      if ((rc = gemm(m, f.in[i], xa, B, Ls, p.lensS, 1 << i, p.cd, p.ia, nullptr, st))) return rc;
      gate<<<grid_for(rows * (C / 4), 256), 256, 0, st>>>(p.ia, planes && i > 0 ? p.x[cur] : nullptr, p.lensS, B, Ls, C, (float*)p.acts,
                                                           (__half*)p.acts, status);
      FS2_LAUNCH_CHECK();
      if (i < kLayers - 1) {
        if ((rc = gemm(m, f.res[i], p.acts, B, Ls, p.lensS, 1, p.x[cur], p.x[cur ^ 1], p.xp, st))) return rc;
        cur ^= 1;
      }
      if ((rc = gemm(m, f.skip[i], p.acts, B, Ls, p.lensS, 1, i ? p.skip[sk] : nullptr, p.skip[sk ^ 1], nullptr, st))) return rc;
      sk ^= 1;
    }
    float* dst = k == 0 ? audio : p.state;
    rc = h == 4 ? launch_flow(wg_flow_kernel<4>, c, C, p.skip[sk], p.state, dst, p.lensS, B, Ls, o, f, st)
       : h == 3 ? launch_flow(wg_flow_kernel<3>, c, C, p.skip[sk], p.state, dst, p.lensS, B, Ls, o, f, st)
                : launch_flow(wg_flow_kernel<2>, c, C, p.skip[sk], p.state, dst, p.lensS, B, Ls, o, f, st);
    if (rc) return rc;
  }
  return FS2_OK;
}

}  // extern "C"
