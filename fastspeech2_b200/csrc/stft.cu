// Vocoder hand-off kernels (SURVEY.md section 8f-2): the STFT / inverse-STFT pair Griffin-Lim iterates
// (utils/stft.py:41-156, dataset/audio_processing.py:224-240), cuFFT-free like the reference: the reference runs the
// transform as F.conv1d with a [2*cutoff, 1, n_fft] windowed Fourier basis at stride hop, and the inverse as
// F.conv_transpose1d with the pseudo-inverse basis -- both are GEMMs over a [frames, n_fft] matrix, so here
//   transform : reflect-pad + frame extraction (this file) -> tap-GEMM with the forward basis (library GEMM kernels)
//               -> magnitude / phase (this file)
//   inverse   : magnitude * (cos, sin)(phase) (this file) -> tap-GEMM with the inverse basis -> overlap-add, window-sum
//               normalisation, hop scaling and trimming in one pass (this file).
// All HBM-bound elementwise / gather kernels; the two GEMMs go through fs2_op_tap_gemm.
#include <math.h>

#include "common.cuh"

namespace fs2 {
namespace {

// frames[b, f, k] = xpad[b, f*hop + k], xpad = reflect-pad(x, n_fft/2) (utils/stft.py:89-95: F.pad(..., mode="reflect"))
__global__ void stft_frames_kernel(const float* __restrict__ x, int n, int n_fft, int hop, int frames, long total, float* __restrict__ out) {
  const int half = n_fft / 2;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int k = (int)(i % n_fft); const long r = i / n_fft; const int f = (int)(r % frames); const long b = r / frames;
    int s = f * hop + k - half;                       // index into the unpadded signal
    if (s < 0) s = -s;                                // reflect without repeating the edge sample
    if (s >= n) s = 2 * (n - 1) - s;
    out[i] = x[b * n + s];
  }
}
// spec[b, f, 0:cutoff] = real, [cutoff:2*cutoff] = imag  ->  magnitude, phase in the reference's [B, cutoff, frames] layout
__global__ void stft_magphase_kernel(const float* __restrict__ spec, int ld, int cutoff, int frames, long total, float* __restrict__ mag,
                                     float* __restrict__ phase) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int f = (int)(i % frames); const long r = i / frames; const int c = (int)(r % cutoff); const long b = r / cutoff;
    const float re = spec[(b * frames + f) * ld + c], im = spec[(b * frames + f) * ld + cutoff + c];
    mag[i] = sqrtf(re * re + im * im);
    phase[i] = atan2f(im, re);
  }
}
// rec[b, f, c] = mag * cos(phase), rec[b, f, cutoff + c] = mag * sin(phase); columns >= 2*cutoff (GEMM K padding) = 0
__global__ void istft_recombine_kernel(const float* __restrict__ mag, const float* __restrict__ phase, int cutoff, int frames, int ld, long total,
                                       float* __restrict__ rec) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % ld); const long r = i / ld; const int f = (int)(r % frames); const long b = r / frames;
    float v = 0.f;
    if (c < 2 * cutoff) {
      const int cc = c < cutoff ? c : c - cutoff;
      const long o = (b * cutoff + cc) * frames + f;
      float sn, cs;
      sincosf(phase[o], &sn, &cs);
      v = mag[o] * (c < cutoff ? cs : sn);
    }
    rec[i] = v;
  }
}
// conv_transpose1d(stride = hop) as a gather: y[b, s] = sum_f frames_out[b, f, s + half - f*hop], then / window_sum where it is
// > tiny, * n_fft / hop, with the first and last n_fft/2 samples already trimmed (utils/stft.py:121-149)
__global__ void istft_overlap_add_kernel(const float* __restrict__ fr, int n_fft, int hop, int frames, int n_out, const float* __restrict__ wsum,
                                         float tiny, float scale, long total, float* __restrict__ y) {
  const int half = n_fft / 2;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int s = (int)(i % n_out); const long b = i / n_out;
    const int p = s + half;                            // position in the untrimmed signal
    int f_hi = p / hop; if (f_hi > frames - 1) f_hi = frames - 1;
    int f_lo = (p - n_fft + hop) / hop; if (p - n_fft + 1 <= 0) f_lo = 0; if (f_lo < 0) f_lo = 0;
    float acc = 0.f;
    for (int f = f_lo; f <= f_hi; ++f) {
      const int k = p - f * hop;
      if (k >= 0 && k < n_fft) acc += fr[(b * frames + f) * n_fft + k];
    }
    const float w = wsum[p];
    if (w > tiny) acc /= w;
    y[i] = acc * scale;
  }
}

}  // namespace
}  // namespace fs2

using namespace fs2;

extern "C" {

int fs2_stft_frames(const float* x, int B, int n, int n_fft, int hop, int frames, float* out, void* stream) {
  FS2_REQUIRE(x && out && n > n_fft / 2 && hop > 0, "fs2_stft_frames: bad argument (the signal must be longer than n_fft/2 for reflect padding)");
  const long total = (long)B * frames * n_fft;
  if (total == 0) return FS2_OK;
  stft_frames_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(x, n, n_fft, hop, frames, total, out);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_stft_magphase(const float* spec, int ld, int B, int cutoff, int frames, float* mag, float* phase, void* stream) {
  FS2_REQUIRE(spec && mag && phase && ld >= 2 * cutoff, "fs2_stft_magphase: bad argument");
  const long total = (long)B * cutoff * frames;
  if (total == 0) return FS2_OK;
  stft_magphase_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(spec, ld, cutoff, frames, total, mag, phase);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_istft_recombine(const float* mag, const float* phase, int B, int cutoff, int frames, int ld, float* rec, void* stream) {
  FS2_REQUIRE(mag && phase && rec && ld >= 2 * cutoff, "fs2_istft_recombine: bad argument");
  const long total = (long)B * frames * ld;
  if (total == 0) return FS2_OK;
  istft_recombine_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(mag, phase, cutoff, frames, ld, total, rec);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fs2_istft_overlap_add(const float* frames_out, int B, int n_fft, int hop, int frames, const float* window_sum, float tiny, float* y, void* stream) {
  FS2_REQUIRE(frames_out && window_sum && y && frames > 0, "fs2_istft_overlap_add: bad argument");
  const int n_out = (frames - 1) * hop;               // n_fft + hop*(frames-1) minus n_fft/2 at both ends
  const long total = (long)B * n_out;
  if (total == 0) return FS2_OK;
  istft_overlap_add_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(frames_out, n_fft, hop, frames, n_out, window_sum, tiny,
                                                                                   (float)n_fft / (float)hop, total, y);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // extern "C"
