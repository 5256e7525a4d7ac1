// Helpers of the code that writes tap-GEMM operands directly (api.cu, griffin_lim.cu, melgan.cu, waveglow.cu, features.cu,
// through vocoder_weights.cuh): the operand's form by math mode, and the range an fp16 operand plane holds.
#pragma once
#include "common.cuh"

namespace fs2 {

constexpr float kPlaneMax = 65504.0f / kPlaneScale;   // largest |x| an operand plane holds without saturating

enum OutKind { OUT_F32 = 0, OUT_HI = 1, OUT_HILO = 2 };   // GEMM operand as fp32 rows / hi plane / hi + lo planes

inline int out_kind(int mode) { return mode == FS2_MATH_3XTF32 ? OUT_HILO : mode == FS2_MATH_F16 ? OUT_HI : OUT_F32; }
inline bool plane_mode(int mode) { return mode == FS2_MATH_F16 || mode == FS2_MATH_3XTF32; }

// the kernel instantiation for an operand kind: k3 (hi + lo planes), k2 (hi plane) or k1 (fp32 rows)
template <typename K3, typename K2, typename K1>
K1 pick(int kind, K3 k3, K2 k2, K1 k1) { return kind == OUT_HILO ? k3 : kind == OUT_HI ? k2 : k1; }

}  // namespace fs2
