// The vocoders' window layer (vocoder_window.cuh).
#include "vocoder_window.cuh"

#include <algorithm>

#include "vocoder_weights.cuh"

namespace fs2 {
namespace {

constexpr int kBadLength = 1, kBadStart = 4;
static_assert(FS2_MELGAN_BAD_LENGTH == kBadLength && FS2_HIFIGAN_BAD_LENGTH == kBadLength && FS2_WAVEGLOW_BAD_LENGTH == kBadLength,
              "the vocoders' BAD_LENGTH bits differ");
static_assert(FS2_MELGAN_BAD_START == kBadStart && FS2_HIFIGAN_BAD_START == kBadStart && FS2_WAVEGLOW_BAD_START == kBadStart,
              "the vocoders' BAD_START bits differ");

__global__ void ups_prep_kernel(const int64_t* __restrict__ olens, const int64_t* __restrict__ starts, int B, int lo, int L, int nf, UpsPlan p,
                                int64_t* __restrict__ lens, int* __restrict__ status) {
  __shared__ int bad;
  if (threadIdx.x == 0) bad = 0;
  __syncthreads();
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    const int64_t n = olens[b];
    const bool ok = n >= lo && n <= L;
    if (!ok) atomicOr(&bad, kBadLength);
    if (!starts) {
      for (int s = 0; s <= p.n; ++s) lens[(long)s * B + b] = ok ? (n + p.tail) * p.up[s] : 0;
      continue;
    }
    const int64_t c0 = starts[b];
    if (c0 < 0) atomicOr(&bad, kBadStart);
    const bool live = ok && c0 >= 0 && c0 < n;
    const int64_t c1 = live ? min(c0 + nf, n) : 0;
    auto put = [&](int w, int64_t lo, int64_t hi, int64_t total) {
      int64_t* d = lens + 3L * w * B + b;
      d[0] = live ? lo : 0;
      d[B] = live ? hi - lo : 0;
      d[2 * B] = live ? total : 0;
    };
    for (int s = 0; s <= p.n; ++s) {
      const int64_t up = p.up[s], total = (n + p.tail) * up;
      put(win_level(s), max(c0 * up - p.halo[s], (int64_t)0), min(c1 * up + p.halo[s], total), total);
      if (s < p.n && p.reach[s] != p.halo[s])
        put(win_ups(p, s), max(c0 * up - p.reach[s], (int64_t)0), min(c1 * up + p.reach[s], total), total);
    }
    const int64_t up = p.up[p.n];
    put(win_audio(p), c0 * up, c1 * up, (n + p.tail) * up);
  }
  __syncthreads();
  if (threadIdx.x == 0) *status = bad;
}

}  // namespace

int ups_prep(const int64_t* olens, const int64_t* starts, int B, int lo, int L, int nf, const UpsPlan& p, int64_t* lens, int* status,
             cudaStream_t st) {
  ups_prep_kernel<<<1, 256, 0, st>>>(olens, starts, B, lo, L, nf, p, lens, status);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int check_size(const char* who, const UpsPlan& p, int B, int L, int math_mode) {
  FS2_REQUIRE(B >= 1 && L >= 1, "%s: need B >= 1 and Lmax >= 1 (got %d, %d)", who, B, L);
  const int up = p.up[p.n];
  char formula[48];
  if (p.tail) snprintf(formula, sizeof formula, "B * (Lmax + %d) * %d", p.tail, up);
  else snprintf(formula, sizeof formula, "B * Lmax * %d", up);
  return check_rows(who, formula, up == 256 ? "sample" : "row", (long)B * ((long)L + p.tail) * up, math_mode);
}

int check_window_rows(const char* who, const UpsPlan& p, int B, int nf, int math_mode) {
  FS2_REQUIRE(B >= 1 && nf >= 1, "%s: need B >= 1 and n_frames >= 1 (got %d, %d)", who, B, nf);
  int top = 0;
  for (int s = 1; s <= p.n; ++s)
    if (level_rows(p, s, nf) > level_rows(p, top, nf)) top = s;
  char formula[64];
  snprintf(formula, sizeof formula, "B * (%d * n_frames + %d)", p.up[top], 2 * p.halo[top]);
  return check_rows(who, formula, "window", (long)B * std::min(level_rows(p, top, nf), 1L << 31), math_mode);
}

int check_window_extent(const char* who, int Lmax, int tail, int rows_per_frame, int n_frames, int64_t audio_ld) {
  char lmax[32] = "Lmax";
  if (tail) snprintf(lmax, sizeof lmax, "(Lmax + %d)", tail);
  FS2_REQUIRE(Lmax >= 1 && ((long)Lmax + tail) * rows_per_frame < (1L << 31), "%s: need 1 <= Lmax and %s * %d below 2^31 (got Lmax = %d)",
              who, lmax, rows_per_frame, Lmax);
  FS2_REQUIRE(audio_ld >= (int64_t)n_frames * 256, "%s: audio_ld = %lld below n_frames * 256 = %ld", who, (long long)audio_ld,
              (long)n_frames * 256);
  return FS2_OK;
}

}  // namespace fs2
