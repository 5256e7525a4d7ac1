// The window layer of an upsampling chain, MelGAN (melgan.cu) and HiFi-GAN (hifigan.cu): a first conv (level 0, one row
// per frame), U polyphase ConvTranspose1d layers (k = 2u, stride u), each followed by a residual stack that reads R rows
// on each side, and a last conv.  The plan of which rows every buffer of a window holds (DESIGN.md section 11), the window
// descriptors a call's prep kernel writes, and the helpers the producers read them with.
#pragma once
#include "common.cuh"

namespace fs2 {

constexpr int kMaxUps = FS2_HIFIGAN_MAX_UPSAMPLES;

// n upsamplings; cumulative upsampling of levels 0 .. n; their input reaches; the level halos; tail frames
struct UpsPlan { int n; int up[kMaxUps + 1]; int reach[kMaxUps]; int halo[kMaxUps + 1]; int tail; };

// The plan of a chain with these rates, stack reach R, level-0 margin (rows of level 0 wrong at a window side that is not
// an utterance edge), last-conv reach and tail, walking back from the audio: upsampling s reads reach_s input rows on
// each side of its core, level s holds halo_s rows, halo_{s+1} = u_s reach_s and halo_0 = reach_0 + margin0.
constexpr UpsPlan ups_plan(int n, const int* rates, int R, int margin0, int post, int tail) {
  UpsPlan p{};
  p.n = n; p.tail = tail; p.up[0] = 1;
  for (int i = 0; i < n; ++i) p.up[i + 1] = p.up[i] * rates[i];
  int need = post;
  for (int i = n - 1; i >= 0; --i) {
    need += R;
    // output rows [-need, 0) of upsampling i's core: row o = u t + q reads input rows t - 1, t (q < u / 2) or t, t + 1
    const int u = rates[i], o = -need, t = (o - (u - 1)) / u, q = o - t * u;   // floor division of a negative o
    p.reach[i] = need = -(q < u / 2 ? t - 1 : t);
    p.halo[i + 1] = u * need;
  }
  p.halo[0] = need + margin0;
  return p;
}

// rows per utterance of level s's window buffer and of upsampling s's input window, for nf frames
constexpr long level_rows(const UpsPlan& p, int s, long nf) { return nf * p.up[s] + 2L * p.halo[s]; }
constexpr long ups_rows(const UpsPlan& p, int s, long nf) { return nf * p.up[s] + 2L * p.reach[s]; }

// Window descriptors of a window call, [start | len | n] x B each: levels 0 .. n, then the input window of every upsampling
// s whose reach differs from its level's halo (where they are equal, level s's descriptor is that window), then the audio
// samples.
constexpr int win_level(int s) { return s; }
constexpr int win_ups(const UpsPlan& p, int s) {
  if (p.reach[s] == p.halo[s]) return win_level(s);
  int w = p.n + 1;
  for (int i = 0; i < s; ++i) w += p.reach[i] != p.halo[i];
  return w;
}
constexpr int n_wins(const UpsPlan& p) {
  int w = p.n + 2;
  for (int i = 0; i < p.n; ++i) w += p.reach[i] != p.halo[i];
  return w;
}
constexpr int win_audio(const UpsPlan& p) { return n_wins(p) - 1; }

// rows of utterance b in a buffer: global rows [start, start + len) of the utterance's n rows at its rate (win == nullptr:
// the whole utterance, start 0 and len = n = lens[b])
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

// One CTA, enqueued first so that the producers' range bits land on a cleared word.  A whole call (starts == nullptr):
// lens[s][b] = (olens[b] + tail) * up_s, 0 for olens[b] outside [1, L].  A window of nf frames from starts[b]: the n_wins(p)
// descriptors of the core [starts[b], min(starts[b] + nf, olens[b])), clipped to the utterance, len 0 when it is empty.
// *status = BAD_LENGTH (1) for some olens[b] outside [1, L] | BAD_START (4) for some starts[b] < 0.
int ups_prep(const int64_t* olens, const int64_t* starts, int B, int L, int nf, const UpsPlan& p, int64_t* lens, int* status,
             cudaStream_t st);

// A window's size checks: B >= 1, n_frames >= 1, and check_rows on the rows of its largest level buffer, whose formula
// the error quotes as "B * (<up_s> * n_frames + <2 halo_s>)"
int check_window_rows(const char* who, const UpsPlan& p, int B, int n_frames, int math_mode);

// A window entry's extent checks, in this order: 1 <= Lmax with (Lmax + tail) * rows_per_frame (an utterance's rows at
// its finest rate) below 2^31, then audio_ld >= n_frames * 256
int check_window_extent(const char* who, int Lmax, int tail, int rows_per_frame, int n_frames, int64_t audio_ld);

}  // namespace fs2
