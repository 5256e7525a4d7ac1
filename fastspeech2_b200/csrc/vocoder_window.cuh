// The window layer of the vocoders whose window calls run a plan of levels: MelGAN (melgan.cu), HiFi-GAN, iSTFTNet and
// BigVGAN (hifigan.cu), and WaveGlow (waveglow.cu).  The plan of which rows every buffer of a window holds (DESIGN.md
// sections 11 and 12), the window descriptors a call's prep kernel writes, the helpers the producers read them with, and
// the C entries' one sequence of checks.
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
// lens[s][b] = (olens[b] + tail) * up_s, 0 for olens[b] outside [lo, L].  A window of nf frames from starts[b]: the
// n_wins(p) descriptors of the core [starts[b], min(starts[b] + nf, olens[b])), clipped to the utterance, all 0 when it is
// empty.  *status = BAD_LENGTH (1) for some olens[b] outside [lo, L] | BAD_START (4) for some starts[b] < 0.  lo = 1 for
// the vocoders' calls; WaveGlow's single-stage entries take lo = 0 (an empty utterance is valid there).
int ups_prep(const int64_t* olens, const int64_t* starts, int B, int lo, int L, int nf, const UpsPlan& p, int64_t* lens, int* status,
             cudaStream_t st);

// A whole call's size checks: B >= 1, Lmax >= 1, and check_rows on its largest GEMM, B * (Lmax + tail) * up_n rows
// ("sample" rows when up_n is the hop 256)
int check_size(const char* who, const UpsPlan& p, int B, int Lmax, int math_mode);

// A window's size checks: B >= 1, n_frames >= 1, and check_rows on the rows of its largest level buffer, whose formula
// the error quotes as "B * (<up_s> * n_frames + <2 halo_s>)"
int check_window_rows(const char* who, const UpsPlan& p, int B, int n_frames, int math_mode);

// A window entry's extent checks, in this order: 1 <= Lmax with (Lmax + tail) * rows_per_frame (an utterance's rows at
// its finest rate) below 2^31, then audio_ld >= n_frames * 256
int check_window_extent(const char* who, int Lmax, int tail, int rows_per_frame, int n_frames, int64_t audio_ld);

// ---- the C entries of MelGAN, HiFi-GAN, iSTFTNet and BigVGAN ----
// name: "fs2_<vocoder>", the prefix of every message.  The whole call checks, in this order, null arguments, weights
// loaded, 16-byte mels, the size limits and the workspace; a window null arguments, 16-byte mels, the window-row limits,
// the extent, the workspace and weights loaded.  V is the vocoder's side:
//   V::Gen                                  the handle (math_mode, loaded, arena)
//   V::ups(m)                               its UpsPlan
//   V::plan(b, m, B, Lmax)                  the whole call's workspace carve, and V::window_plan(b, m, B, n_frames) a window's
//   V::generate(m, p, mels, olens, starts, B, Lmax, n_frames, audio, ld, status, stream)
//                                           the call on a carve p: whole utterances (starts == nullptr) or a window
template <typename V>
int workspace_gen(typename V::Gen* m, int B, int Lmax, size_t* bytes, const char* name) {
  FS2_REQUIRE(m && bytes, "%s_workspace_bytes: null argument", name);
  int rc = check_size(name, V::ups(m), B, Lmax, m->math_mode);
  if (rc) return rc;
  Bump b(nullptr, 0);
  V::plan(b, m, B, Lmax);
  *bytes = b.off + 256;
  return FS2_OK;
}

template <typename V>
int call_gen(typename V::Gen* m, const float* mels, const int64_t* olens, int B, int Lmax, float* audio, int* status, void* ws,
             size_t ws_bytes, void* stream, const char* name) {
  FS2_REQUIRE(m && mels && olens && audio && status && ws, "%s: null argument", name);
  FS2_REQUIRE(m->loaded, "%s: weights not loaded (%s_load)", name, name);
  FS2_REQUIRE((reinterpret_cast<uintptr_t>(mels) & 15) == 0, "%s: mels must be 16-byte aligned", name);
  int rc = check_size(name, V::ups(m), B, Lmax, m->math_mode);
  if (rc) return rc;
  Bump b(ws, ws_bytes);
  const auto p = V::plan(b, m, B, Lmax);
  if ((rc = b.check(name))) return rc;
  return V::generate(m, p, mels, olens, nullptr, B, Lmax, 0, audio, (long)Lmax * 256, status, (cudaStream_t)stream);
}

template <typename V>
int window_workspace_gen(typename V::Gen* m, int B, int n_frames, size_t* bytes, const char* name) {
  char who[48];
  snprintf(who, sizeof who, "%s_window", name);
  FS2_REQUIRE(m && bytes, "%s_workspace_bytes: null argument", who);
  int rc = check_window_rows(who, V::ups(m), B, n_frames, m->math_mode);
  if (rc) return rc;
  Bump b(nullptr, 0);
  V::window_plan(b, m, B, n_frames);
  *bytes = b.off + 256;
  return FS2_OK;
}

template <typename V>
int window_gen(typename V::Gen* m, const float* mels, const int64_t* olens, const int64_t* starts, int B, int Lmax, int n_frames,
               float* audio, int64_t audio_ld, int* status, void* ws, size_t ws_bytes, void* stream, const char* name) {
  char who[48];
  snprintf(who, sizeof who, "%s_window", name);
  FS2_REQUIRE(m && mels && olens && starts && audio && status && ws, "%s: null argument", who);
  FS2_REQUIRE((reinterpret_cast<uintptr_t>(mels) & 15) == 0, "%s: mels must be 16-byte aligned", who);
  int rc = check_window_rows(who, V::ups(m), B, n_frames, m->math_mode);
  if (rc) return rc;
  if ((rc = check_window_extent(who, Lmax, V::ups(m).tail, 256, n_frames, audio_ld))) return rc;
  Bump b(ws, ws_bytes);
  const auto p = V::window_plan(b, m, B, n_frames);
  if ((rc = b.check(who))) return rc;
  FS2_REQUIRE(m->loaded, "%s: weights not loaded (%s_load)", who, name);
  return V::generate(m, p, mels, olens, starts, B, Lmax, n_frames, audio, audio_ld, status, (cudaStream_t)stream);
}

// every vocoder handle's destroy: its weight arena, then the handle
template <typename Gen>
void destroy_gen(Gen* m) {
  if (!m) return;
  if (m->arena) cudaFree(m->arena);
  delete m;
}

}  // namespace fs2
