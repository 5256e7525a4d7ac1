// Helpers of the code that writes tap-GEMM operands directly (api.cu, griffin_lim.cu, melgan.cu, waveglow.cu, features.cu,
// through vocoder_weights.cuh): the operand's form by math mode, the range an fp16 operand plane holds, and the stores
// that write an operand as fp32 rows or as planes.
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

// Whether a plane store checks its values against kPlaneMax (NaN fails) and sets range_bit in *status when one is out of
// range: never, always, or only when status != nullptr (the caller passes null for a halo row)
enum RangeCheck { RANGE_NEVER, RANGE_ALWAYS, RANGE_IF_STATUS };

// one pair of GEMM-operand values at element offset off (even) of a [rows][K] operand; plane = rows * K
template <int OUT, int CHECK>
__device__ __forceinline__ void store_pair(float v0, float v1, long off, float* __restrict__ out32, __half* __restrict__ outp,
                                           long plane, int* __restrict__ status, int range_bit) {
  if (OUT == OUT_F32) {
    *reinterpret_cast<float2*>(out32 + off) = make_float2(v0, v1);
    return;
  }
  if (CHECK != RANGE_NEVER && (CHECK == RANGE_ALWAYS || status) && !(fabsf(v0) <= kPlaneMax && fabsf(v1) <= kPlaneMax))
    atomicOr(status, range_bit);                        // saturation is reported, not hidden
  if (OUT == OUT_HILO) {
    uint32_t hi, lo;
    split_pair(v0, v1, hi, lo);
    *reinterpret_cast<uint32_t*>(outp + off) = hi;
    *reinterpret_cast<uint32_t*>(outp + plane + off) = lo;
  } else {
    *reinterpret_cast<uint32_t*>(outp + off) = hi_pair(v0, v1);
  }
}

// four GEMM-operand values at element offset off (a multiple of 4) of a [rows][K] operand; plane = rows * K
template <int OUT, int CHECK>
__device__ __forceinline__ void store_quad(float4 v, long off, float* __restrict__ out32, __half* __restrict__ outp, long plane,
                                           int* __restrict__ status, int range_bit) {
  if (OUT == OUT_F32) {
    *reinterpret_cast<float4*>(out32 + off) = v;
    return;
  }
  if (CHECK != RANGE_NEVER && (CHECK == RANGE_ALWAYS || status) &&
      !(fabsf(v.x) <= kPlaneMax && fabsf(v.y) <= kPlaneMax && fabsf(v.z) <= kPlaneMax && fabsf(v.w) <= kPlaneMax))
    atomicOr(status, range_bit);                        // saturation is reported, not hidden
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

}  // namespace fs2
