// BigVGAN's anti-aliased activation (bigvgan.cu, DESIGN.md section 18): the Activation1d(Snake / SnakeBeta) producer that
// replaces HiFi-GAN's lrelu in front of every block convolution of the shared generator chain (hifigan.cu), and the head
// that replaces its conv_post + tanh.
#pragma once
#include "common.cuh"

namespace fs2 {

constexpr int kAct = 5;                     // Activation1d's reach: output row t reads input rows t - 5 .. t + 5
constexpr int kFilt = 12;                   // taps of the up and down filters

// a width padded to the 32-channel tiles of the activation producer and the GEMMs
inline int ceil32(int c) { return (c + 31) / 32 * 32; }

// One activation's parameters on the device, prm [2 C' + 24]: alpha' [C'] (exp(alpha) with snake_logscale), inv [C']
// (1 / (beta' + 1e-9), beta' = alpha' for Snake), f_up [12], f_down [12].  Padded channels have alpha' = inv = 0.
__host__ __device__ constexpr long act_params(int Cp) { return 2L * Cp + 2 * kFilt; }

// prm (act_params(ceil32(C)) floats) from one activation's tensors t[0 .. 3]: alpha [C], beta [C] (read with snakebeta),
// upsample.filter [12], downsample.lowpass.filter [12]
int act_param(const float* const* t, int C, int logscale, int snakebeta, float* prm, cudaStream_t st);

// The GEMM operand a [B * Lp][C] = Activation1d(x) (x [B * Lp][C] in the operand's own window win, nullptr: the whole
// utterance of lens[b] rows) for t < len, +0 past it, on the operand kind `kind`; only rows exact_row(margin) are
// range-checked (FS2_HIFIGAN_RANGE).  C a multiple of 32.
int bigvgan_act(int kind, const float* x, const float* prm, const int64_t* lens, const int64_t* win, int B, int Lp, int C, int margin,
                void* a, int* status, cudaStream_t st);

// audio = final(conv_post(Activation1d((S + R) / nk))), final = tanh (use_tanh) or a clamp to [-1, 1]: S, R (nullable),
// lens, win, awin, B, Lx, Lout, ld as istftnet_head's; w [7][C] (C = C'_U), bias nullable; prm activation_post's
int bigvgan_post(const float* S, const float* R, int nk, const int64_t* lens, const int64_t* win, const int64_t* awin, int B, int Lx,
                 int Lout, long ld, int C, const float* prm, const float* w, const float* bias, int use_tanh, float* audio, cudaStream_t st);

}  // namespace fs2
