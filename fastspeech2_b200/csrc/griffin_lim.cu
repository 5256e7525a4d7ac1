// Batched waveform synthesis (DESIGN.md section 7): log-mels [B, Lmax, n_mels] -> magnitudes by the mel filterbank's
// pseudo-inverse -> Griffin-Lim per utterance over its own olens[b] frames, on the library's tap-GEMM.
//
// Rows are the B*Lmax frames.  Every GEMM runs with TapGemm::lens = olens: row tiles wholly past an utterance are
// skipped and padded rows come out as zeros.  The kernels that produce GEMM inputs write the operand planes (f16 /
// 3xF16) or fp32 rows (fp32 / tf32) directly, so the loop has no split pass and no temporary:
//
//   mel_expand        exp(mel) rows                                   -> GEMM P (K = n_mels, N = mpad, ReLU) -> M fp32
//   gl_project        rec = M (.) u, u from seed / angles / Z (+ momentum) -> inverse GEMM (K = cpad, N = n_fft) -> frames
//   ola_frame         overlap-add, window sum, scale, trim, reflect-pad and re-frame -> forward GEMM (K = n_fft, N = cpad) -> Z
//   ola_audio         the same overlap-add on the last pass, written as audio (0 past (olens[b] - 1) * hop)
//
// Launches: 5 + 4 * n_iters.  OLA + reframe is one kernel: a CTA owns FPB consecutive output frames of one utterance,
// overlap-adds the (FPB - 1) * hop + n_fft signal samples they cover into shared memory (reflection at the utterance's
// edges is an index map), then writes the frames.  The signal never goes to HBM, at the price of recomputing
// (n_fft - hop) / (FPB * hop) of the samples (37 % at FPB = 8, hop = n_fft / 4) from L2-resident GEMM output.
//
// Rows past olens[b] of the GEMM inputs are never written: a live tile reads them, but a GEMM output row depends only on
// its own input row, and the epilogue stores 0 there whatever was read.  Per-utterance results therefore do not depend on
// the batch: the same rows see the same K loop, the same element-wise maps and the same overlap-add order.
#include <float.h>
#include <math.h>

#include "vocoder_weights.cuh"

struct fs2_vocoder;

namespace fs2 {
namespace {

constexpr int FPB = 8;                                 // output frames per ola_frame CTA

// frames of utterance b that are processed; 0 for a length that fails the contract (reported by mel_expand)
__device__ __forceinline__ int valid_len(const int64_t* __restrict__ olens, int b, int L, int hop, int half) {
  const int64_t n = olens[b];
  return (n >= 1 && n <= L && (n - 1) * hop > half) ? (int)n : 0;
}

// exp(mels) as the mel GEMM's operand (K = n_mels); zero rows past the utterance.  Also checks olens.
template <int OUT>
__global__ void mel_expand_kernel(const float* __restrict__ mels, const int64_t* __restrict__ olens, int B, int L, int n_mels,
                                  int hop, int half, float* __restrict__ out32, __half* __restrict__ outp, int* __restrict__ status) {
  const int pairs = n_mels / 2;
  const long total = (long)B * L * pairs, plane = (long)B * L * n_mels;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / pairs;
    const int k = (int)(i - row * pairs) * 2, b = (int)(row / L), t = (int)(row - (long)b * L);
    const int len = valid_len(olens, b, L, hop, half);
    if (t == 0 && k == 0 && len == 0) atomicOr(status, FS2_VOC_BAD_LENGTH);
    float v0 = 0.f, v1 = 0.f;
    if (t < len) {                                    // frames past olens[b] are never read (NaN there changes nothing)
      const float2 m = *reinterpret_cast<const float2*>(mels + row * n_mels + k);
      v0 = expf(m.x); v1 = expf(m.y);
    }
    store_pair<OUT, RANGE_ALWAYS>(v0, v1, row * n_mels + k, out32, outp, plane, status, FS2_VOC_RANGE);
  }
}

// rec[row, :] = M (.) u as the inverse GEMM's operand [rows][cpad]: columns [0, cutoff) real, [cutoff, 2 cutoff)
// imaginary, the rest 0.  SRC: 0 = Philox phases keyed by seeds[b], counter t * cutoff + c; 1 = angles [B, cutoff, L];
// 2 = u = Zh / |Zh| of the forward GEMM's output Z [rows][cpad] (Zh = Z - mom_k * Zprev when MOM), (1, 0) where Zh = 0.
template <int SRC, bool MOM>
__device__ __forceinline__ float2 phasor(int c, int b, int t, long row, int L, int cutoff, int ldz, const float* __restrict__ z,
                                         const float* __restrict__ zprev, float mom_k, const int64_t* __restrict__ seeds,
                                         const float* __restrict__ angles) {
  float s, co;
  if (SRC == 0) {
    const unsigned long long ctr = (unsigned long long)t * cutoff + c, key = (unsigned long long)seeds[b];
    const uint4 r = philox4x32(make_uint4((unsigned)ctr, (unsigned)(ctr >> 32), 0u, 0u), make_uint2((unsigned)key, (unsigned)(key >> 32)));
    sincospif((float)(r.x >> 8) * (2.0f / 16777216.0f), &s, &co);     // uniform phase 2 pi U, U in [0, 1) on 24 bits
    return make_float2(co, s);
  }
  if (SRC == 1) {
    sincosf(angles[((long)b * cutoff + c) * L + t], &s, &co);
    return make_float2(co, s);
  }
  float re = z[row * ldz + c], im = z[row * ldz + cutoff + c];
  if (MOM) { re = fmaf(-mom_k, zprev[row * ldz + c], re); im = fmaf(-mom_k, zprev[row * ldz + cutoff + c], im); }
  const float r = hypotf(re, im);
  return r > 0.f ? make_float2(re / r, im / r) : make_float2(1.f, 0.f);   // atan2(0, 0) = 0 in the reference
}

template <int OUT, int SRC, bool MOM>
__global__ void gl_project_kernel(const float* __restrict__ mag, int ldm, const float* __restrict__ z, const float* __restrict__ zprev,
                                  float mom_k, const int64_t* __restrict__ seeds, const float* __restrict__ angles,
                                  const int64_t* __restrict__ olens, int B, int L, int cutoff, int cpad, int hop, int half,
                                  float* __restrict__ out32, __half* __restrict__ outp, int* __restrict__ status) {
  const int pairs = cpad / 2;
  const long total = (long)B * L * pairs, plane = (long)B * L * cpad;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long row = i / pairs;
    const int j = (int)(i - row * pairs) * 2, b = (int)(row / L), t = (int)(row - (long)b * L);
    if (t >= valid_len(olens, b, L, hop, half)) continue;
    float v[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int col = j + e;
      v[e] = 0.f;
      if (col < 2 * cutoff) {
        const int c = col < cutoff ? col : col - cutoff;
        const float2 u = phasor<SRC, MOM>(c, b, t, row, L, cutoff, cpad, z, zprev, mom_k, seeds, angles);
        v[e] = mag[row * ldm + c] * (col < cutoff ? u.x : u.y);
      }
    }
    store_pair<OUT, RANGE_ALWAYS>(v[0], v[1], row * cpad + j, out32, outp, plane, status, FS2_VOC_RANGE);
  }
}

// sample s (trimmed coordinates, 0 <= s < (len - 1) * hop) of ISTFT: overlap-add of the inverse GEMM's frames
// fr [rows][n_fft] over f = f_lo..f_hi in increasing order, / window sum (same frames, from the win^2 table) where it
// exceeds FLT_MIN, * n_fft / hop (utils/stft.py:119-149 restated; window sum of dataset/audio_processing.py:169-221)
__device__ __forceinline__ float ola_sample(const float* __restrict__ fr, const float* __restrict__ win_sq, long row0, int len,
                                            int n_fft, int hop, int half, float scale, int s) {
  const int q = s + half;
  int f_hi = q / hop; if (f_hi > len - 1) f_hi = len - 1;
  int f_lo = q - n_fft + 1 <= 0 ? 0 : (q - n_fft + hop) / hop;
  float acc = 0.f, ws = 0.f;
  for (int f = f_lo; f <= f_hi; ++f) {
    const int k = q - f * hop;
    acc += fr[(row0 + f) * n_fft + k];
    ws += win_sq[k];
  }
  if (ws > FLT_MIN) acc /= ws;
  return acc * scale;
}

// grid (ceil(L / FPB), B): overlap-add the samples under frames f0 .. f0 + FPB - 1 into shared memory, then write those
// frames of reflect_pad(y, n_fft / 2) as the forward GEMM's operand [rows][n_fft]
template <int OUT>
__global__ void __launch_bounds__(256) ola_frame_kernel(const float* __restrict__ fr, const float* __restrict__ win_sq,
                                                        const int64_t* __restrict__ olens, int L, int n_fft, int hop, float scale,
                                                        float* __restrict__ out32, __half* __restrict__ outp, long plane,
                                                        int* __restrict__ status) {
  extern __shared__ float seg[];
  const int b = blockIdx.y, f0 = blockIdx.x * FPB, half = n_fft / 2;
  const int len = valid_len(olens, b, L, hop, half);
  if (f0 >= len) return;
  const int nf = len - f0 < FPB ? len - f0 : FPB, n = (len - 1) * hop, W = (nf - 1) * hop + n_fft;
  const long row0 = (long)b * L;
  for (int p = threadIdx.x; p < W; p += blockDim.x) {
    int s = f0 * hop + p - half;                   // reflect without repeating the edge sample (n > half by valid_len)
    if (s < 0) s = -s;
    if (s >= n) s = 2 * (n - 1) - s;
    seg[p] = ola_sample(fr, win_sq, row0, len, n_fft, hop, half, scale, s);
  }
  __syncthreads();
  const int hp = n_fft / 2;
  for (int i = threadIdx.x; i < nf * hp; i += blockDim.x) {
    const int f = i / hp, k = (i - f * hp) * 2;
    store_pair<OUT, RANGE_ALWAYS>(seg[f * hop + k], seg[f * hop + k + 1], (row0 + f0 + f) * n_fft + k, out32, outp, plane, status,
                                  FS2_VOC_RANGE);
  }
}

// audio [B, (L - 1) * hop]: the last ISTFT, 0 from (olens[b] - 1) * hop on
__global__ void ola_audio_kernel(const float* __restrict__ fr, const float* __restrict__ win_sq, const int64_t* __restrict__ olens,
                                 int B, int L, int n_fft, int hop, float scale, float* __restrict__ audio) {
  const int half = n_fft / 2, n_out = (L - 1) * hop;
  const long total = (long)B * n_out;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int b = (int)(i / n_out), s = (int)(i - (long)b * n_out);
    const int len = valid_len(olens, b, L, hop, half);
    audio[i] = s < (len - 1) * hop ? ola_sample(fr, win_sq, (long)b * L, len, n_fft, hop, half, scale, s) : 0.f;
  }
}

// mag_out [B, cutoff, L] = M [rows][ldm] transposed, 0 past the utterance (M rows there are already 0)
__global__ void mag_transpose_kernel(const float* __restrict__ m, int ldm, int B, int L, int cutoff, float* __restrict__ out) {
  const long total = (long)B * cutoff * L;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int t = (int)(i % L); const long r = i / L; const int c = (int)(r % cutoff); const long b = r / cutoff;
    out[i] = m[(b * L + t) * ldm + c];
  }
}

}  // namespace
}  // namespace fs2

struct fs2_vocoder {
  fs2_vocoder_config cfg;
  int device = 0, cutoff = 0, cpad = 0, mpad = 0;
  bool loaded = false;
  void* arena = nullptr; size_t arena_bytes = 0;
  fs2::VWeight fwd, inv, mel;   // forward DFT [cpad][n_fft], inverse DFT [n_fft][cpad], mel pseudo-inverse [mpad][n_mels]
  float* win_sq = nullptr;
};

namespace fs2 {
namespace {

struct GlPlan {
  void* melx;          // exp(mel) operand [rows][n_mels]
  float* mag;          // M [rows][mpad]
  void* rec;           // inverse GEMM operand [rows][cpad]
  float* fr;           // inverse GEMM output [rows][n_fft]
  void* frames;        // forward GEMM operand [rows][n_fft]
  float* z[2];         // forward GEMM output [rows][cpad], ping-pong (momentum reads the previous one)
};
// an operand takes rows * K * 4 bytes either way: fp32 rows, or hi + lo fp16 planes
GlPlan plan(const fs2_vocoder* v, Bump& b, int B, int L, bool momentum_state) {
  const size_t rows = (size_t)B * L;
  GlPlan p;
  p.melx = b.floats(rows * v->cfg.n_mels);
  p.mag = b.floats(rows * v->mpad);
  p.rec = b.floats(rows * v->cpad);
  p.fr = b.floats(rows * v->cfg.n_fft);
  p.frames = b.floats(rows * v->cfg.n_fft);
  p.z[0] = b.floats(rows * v->cpad);
  p.z[1] = momentum_state ? b.floats(rows * v->cpad) : p.z[0];
  return p;
}

int mel_stage(fs2_vocoder* v, const float* mels, const int64_t* olens, int B, int L, const GlPlan& p, int* status, cudaStream_t st) {
  const int kind = out_kind(v->cfg.math_mode), nm = v->cfg.n_mels;
  auto k = pick(kind, mel_expand_kernel<OUT_HILO>, mel_expand_kernel<OUT_HI>, mel_expand_kernel<OUT_F32>);
  const long total = (long)B * L * (nm / 2);
  k<<<grid_for(total, 256), 256, 0, st>>>(mels, olens, B, L, nm, v->cfg.hop, v->cfg.n_fft / 2, (float*)p.melx, (__half*)p.melx, status);
  FS2_LAUNCH_CHECK();
  return vweight_gemm(v->cfg.math_mode, v->mel, p.melx, B, L, ACT_RELU, olens, p.mag, st);
}

int check_call(fs2_vocoder* v, const float* mels, const int64_t* olens, int B, int L, const int* status, void* ws) {
  FS2_REQUIRE(v && mels && olens && status && ws, "fs2_vocoder: null argument");
  FS2_REQUIRE(v->loaded, "fs2_vocoder: bases not loaded (fs2_vocoder_load)");
  FS2_REQUIRE(B >= 1 && L >= 2, "fs2_vocoder: need B >= 1 and Lmax >= 2 (got %d, %d)", B, L);
  FS2_REQUIRE((long)L * v->cfg.hop < (1L << 31) && (long)B * L * v->cpad < (1L << 40), "fs2_vocoder: batch too large");
  return FS2_OK;
}

}  // namespace
}  // namespace fs2

using namespace fs2;

extern "C" {

int fs2_vocoder_create(fs2_vocoder** out, const fs2_vocoder_config* cfg) {
  FS2_REQUIRE(out && cfg, "fs2_vocoder_create: null argument");
  const fs2_vocoder_config& c = *cfg;
  FS2_REQUIRE(c.n_fft >= 16 && c.n_fft % 16 == 0, "fs2_vocoder_create: n_fft (%d) must be a positive multiple of 16", c.n_fft);
  FS2_REQUIRE(c.hop >= 1 && c.hop <= c.n_fft && c.win_length >= 1 && c.win_length <= c.n_fft, "fs2_vocoder_create: need 1 <= hop, win_length <= n_fft");
  FS2_REQUIRE(c.n_mels >= 16 && c.n_mels % 16 == 0, "fs2_vocoder_create: n_mels (%d) must be a positive multiple of 16", c.n_mels);
  FS2_REQUIRE(c.math_mode >= FS2_MATH_FP32 && c.math_mode <= FS2_MATH_F16, "fs2_vocoder_create: bad math_mode %d", c.math_mode);
  FS2_REQUIRE((size_t)((FPB - 1) * c.hop + c.n_fft) * sizeof(float) <= 48 * 1024, "fs2_vocoder_create: n_fft / hop too large for the overlap-add tile");
  fs2_vocoder* v = new fs2_vocoder();
  v->cfg = c;
  FS2_CUDA_CHECK(cudaGetDevice(&v->device));
  v->cutoff = c.n_fft / 2 + 1;
  v->cpad = (2 * v->cutoff + 63) / 64 * 64;   // K / N of the DFT GEMMs: whole 64-wide tiles
  v->mpad = (v->cutoff + 63) / 64 * 64;
  *out = v;
  return FS2_OK;
}

void fs2_vocoder_destroy(fs2_vocoder* v) {
  if (!v) return;
  if (v->arena) cudaFree(v->arena);
  delete v;
}

int fs2_vocoder_load(fs2_vocoder* v, const float* w_forward, const float* w_inverse, const float* mel_inverse, const float* window_sq,
                     void* stream) {
  FS2_REQUIRE(v && w_forward && w_inverse && mel_inverse && window_sq, "fs2_vocoder_load: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  const int nf = v->cfg.n_fft, c2 = 2 * v->cutoff;
  v->fwd.N = v->cpad; v->fwd.K = nf;
  v->inv.N = nf; v->inv.K = v->cpad;
  v->mel.N = v->mpad; v->mel.K = v->cfg.n_mels;
  int rc = arena_carve(&v->arena, &v->arena_bytes, st, [&](Bump& b) {
    for (VWeight* w : {&v->fwd, &v->inv, &v->mel}) vweight_carve(b, *w, false);
    v->win_sq = b.floats(nf);
    return FS2_OK;
  });
  if (rc) return rc;
  struct { const float* src; int sr, sc, tr; VWeight* w; } packs[3] = {
      {w_forward, c2, nf, 0, &v->fwd}, {w_inverse, c2, nf, 1, &v->inv}, {mel_inverse, v->cutoff, v->cfg.n_mels, 0, &v->mel}};
  for (auto& p : packs)
    if ((rc = vweight_pack(*p.w, p.src, p.sr, p.sc, p.tr, st))) return rc;
  FS2_CUDA_CHECK(cudaMemcpyAsync(v->win_sq, window_sq, nf * sizeof(float), cudaMemcpyDeviceToDevice, st));
  v->loaded = true;
  return FS2_OK;
}

int fs2_vocoder_workspace_bytes(fs2_vocoder* v, int B, int Lmax, size_t* bytes) {
  FS2_REQUIRE(v && bytes && B >= 0 && Lmax >= 0, "fs2_vocoder_workspace_bytes: bad argument");
  Bump b(nullptr, 0);
  plan(v, b, B, Lmax, true);
  *bytes = b.off + 256;
  return FS2_OK;
}

int fs2_mel_magnitude(fs2_vocoder* v, const float* mels, const int64_t* olens, int B, int Lmax, float* mag_out, int* status,
                      void* ws, size_t ws_bytes, void* stream) {
  int rc = check_call(v, mels, olens, B, Lmax, status, ws);
  if (rc) return rc;
  FS2_REQUIRE(mag_out, "fs2_mel_magnitude: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  Bump b(ws, ws_bytes);
  GlPlan p = plan(v, b, B, Lmax, false);
  if ((rc = b.check("fs2_mel_magnitude"))) return rc;
  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  if ((rc = mel_stage(v, mels, olens, B, Lmax, p, status, st))) return rc;
  const long total = (long)B * v->cutoff * Lmax;
  mag_transpose_kernel<<<grid_for(total, 256), 256, 0, st>>>(p.mag, v->mpad, B, Lmax, v->cutoff, mag_out);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int fs2_griffin_lim(fs2_vocoder* v, const float* mels, const int64_t* olens, int B, int Lmax, int n_iters, float momentum,
                    const int64_t* seeds, const float* angles, float* audio, int* status, void* ws, size_t ws_bytes, void* stream) {
  int rc = check_call(v, mels, olens, B, Lmax, status, ws);
  if (rc) return rc;
  FS2_REQUIRE(audio && (seeds || angles), "fs2_griffin_lim: null argument (audio, and seeds or angles, are required)");
  FS2_REQUIRE(n_iters >= 0, "fs2_griffin_lim: n_iters must be >= 0 (got %d)", n_iters);
  FS2_REQUIRE(momentum >= 0.f && momentum < 1.f, "fs2_griffin_lim: momentum must lie in [0, 1) (got %g)", (double)momentum);
  cudaStream_t st = (cudaStream_t)stream;
  const bool mom = momentum > 0.f;
  Bump b(ws, ws_bytes);
  GlPlan p = plan(v, b, B, Lmax, mom);
  if ((rc = b.check("fs2_griffin_lim"))) return rc;
  const int nf = v->cfg.n_fft, hop = v->cfg.hop, half = nf / 2, kind = out_kind(v->cfg.math_mode);
  const float mom_k = (float)((double)momentum / (1.0 + (double)momentum));
  const float scale = (float)nf / (float)hop;
  const long rows = (long)B * Lmax;
  float* rec32 = (float*)p.rec; __half* recp = (__half*)p.rec;
  float* frm32 = (float*)p.frames; __half* frmp = (__half*)p.frames;

  FS2_CUDA_CHECK(cudaMemsetAsync(status, 0, sizeof(int), st));
  if ((rc = mel_stage(v, mels, olens, B, Lmax, p, status, st))) return rc;
  const long proj_total = rows * (v->cpad / 2);
  const int proj_grid = grid_for(proj_total, 256);
  // rec from the initial phases, then the first ISTFT's frames
  {
    auto k = angles ? pick(kind, gl_project_kernel<OUT_HILO, 1, false>, gl_project_kernel<OUT_HI, 1, false>, gl_project_kernel<OUT_F32, 1, false>)
                    : pick(kind, gl_project_kernel<OUT_HILO, 0, false>, gl_project_kernel<OUT_HI, 0, false>, gl_project_kernel<OUT_F32, 0, false>);
    k<<<proj_grid, 256, 0, st>>>(p.mag, v->mpad, nullptr, nullptr, 0.f, seeds, angles, olens, B, Lmax, v->cutoff, v->cpad, hop, half,
                                 rec32, recp, status);
    FS2_LAUNCH_CHECK();
  }
  if ((rc = vweight_gemm(v->cfg.math_mode, v->inv, p.rec, B, Lmax, ACT_NONE, olens, p.fr, st))) return rc;
  const dim3 ola_grid((Lmax + FPB - 1) / FPB, B);
  const size_t ola_smem = (size_t)((FPB - 1) * hop + nf) * sizeof(float);
  auto ola = pick(kind, ola_frame_kernel<OUT_HILO>, ola_frame_kernel<OUT_HI>, ola_frame_kernel<OUT_F32>);
  auto proj = mom ? pick(kind, gl_project_kernel<OUT_HILO, 2, true>, gl_project_kernel<OUT_HI, 2, true>, gl_project_kernel<OUT_F32, 2, true>)
                  : pick(kind, gl_project_kernel<OUT_HILO, 2, false>, gl_project_kernel<OUT_HI, 2, false>, gl_project_kernel<OUT_F32, 2, false>);
  auto proj0 = pick(kind, gl_project_kernel<OUT_HILO, 2, false>, gl_project_kernel<OUT_HI, 2, false>, gl_project_kernel<OUT_F32, 2, false>);
  for (int it = 0; it < n_iters; ++it) {
    ola<<<ola_grid, 256, ola_smem, st>>>(p.fr, v->win_sq, olens, Lmax, nf, hop, scale, frm32, frmp, rows * nf, status);
    FS2_LAUNCH_CHECK();
    float* z = p.z[it & 1];
    if ((rc = vweight_gemm(v->cfg.math_mode, v->fwd, p.frames, B, Lmax, ACT_NONE, olens, z, st))) return rc;
    // Z_prev starts at 0: the first pass has no momentum term
    auto k = it == 0 ? proj0 : proj;
    k<<<proj_grid, 256, 0, st>>>(p.mag, v->mpad, z, p.z[(it + 1) & 1], mom_k, seeds, angles, olens, B, Lmax, v->cutoff, v->cpad, hop,
                                 half, rec32, recp, status);
    FS2_LAUNCH_CHECK();
    if ((rc = vweight_gemm(v->cfg.math_mode, v->inv, p.rec, B, Lmax, ACT_NONE, olens, p.fr, st))) return rc;
  }
  const long n_audio = (long)B * (Lmax - 1) * hop;
  ola_audio_kernel<<<grid_for(n_audio, 256), 256, 0, st>>>(p.fr, v->win_sq, olens, B, Lmax, nf, hop, scale, audio);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // extern "C"
