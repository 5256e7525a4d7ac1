// iSTFTNet's head (istftnet.cu, DESIGN.md section 19): what replaces HiFi-GAN's conv_post + tanh after the last MRF of
// the shared generator chain (hifigan.cu).
#pragma once
#include "common.cuh"

namespace fs2 {

constexpr int kIstftMaxNfft = 16;   // the largest n_fft the head kernel's shared memory holds

// Last-level rows the head reads on each side of the rows of its audio samples: frame f reads rows f - 4 .. f + 2
// (conv_post's 3 taps and the reflected row), and the samples of rows [r0, r1) are covered by frames
// [r0 - e, r1 + e], e = (n_fft / 2 - 1) / hop.  5 for n_fft 16, hop 4.
constexpr int istft_reach(int n_fft, int hop) { return 4 + (n_fft / 2 - 1) / hop; }

// audio = istft(exp(y[:M]) * exp(i sin(y[M:]))), y = conv_post(ReflectionPad1d((1, 0))(lrelu(x, 0.01))), M = n_fft / 2 + 1,
// x = (S + R) / nk (R nullable) the last MRF's output: rows of utterance b in window win (nullptr: the whole utterance of
// lens[b] rows; x has Lx rows per utterance), 0 outside the utterance.  w: conv_post [7][n_fft + 2][C] (tap-major), bias
// [n_fft + 2].  Audio row b (Lout samples, rows ld apart) holds samples [hop start, hop (start + len)) of awin (nullptr:
// all hop lens[b]), +0 past them.
int istftnet_head(const float* S, const float* R, int nk, const int64_t* lens, const int64_t* win, const int64_t* awin, int B, int Lx,
                  int Lout, long ld, int C, int n_fft, int hop, const float* w, const float* bias, float* audio, cudaStream_t st);

}  // namespace fs2
