// External speaker embeddings (DESIGN.md section 27): ESPnet2's `spembs` with integration type "add".  One fixed-size
// embedding e_b per utterance (an x-vector, ECAPA or d-vector from any speaker-verification model) is L2-normalised and
// projected to adim,
//   v_b = W . (e_b / max(||e_b||_2, 1e-12)) + bias,        W [adim, D], bias [adim]
// and v_b is added to every encoder output row of utterance b.  The eval path adds it in the epilogue of the last encoder
// LayerNorm (rowwise.cu, RowNorm::spk_vec); the train step adds it with fs2_speaker_add (ids 0 .. B-1, table = v).
//
// Everything here is summed in an order fixed by D (and adim) alone, with no atomics on floats:
//   forward:  one CTA per utterance.  Thread i sums e[d]^2 for d = i, i + 256, ... in order, then a fixed shared-memory
//             tree over the 256 threads gives ||e||^2.  Each warp owns outputs a = warp, warp + 8, ...; lane j sums
//             W[a, d] * e_hat[d] for d = j, j + 32, ... in order, then the butterfly warp_sum.  So v_b depends only on e_b.
//   backward: one thread per element of dW (and of dbias): dW[a, d] += sum_b dv[b, a] * e_hat[b, d] with b ascending,
//             dbias[a] += sum_b dv[b, a] likewise.  The same dv always gives the same bits.
// It runs in fp32 in every math mode: B x adim x D multiply-adds are too few to be worth the tensor cores.
#include "common.cuh"

namespace fs2 {
namespace {

constexpr int SPE_THREADS = 256, SPE_WARPS = SPE_THREADS / 32;

// grid B, block 256, dynamic shared memory D floats (the normalised embedding)
__global__ void __launch_bounds__(SPE_THREADS) spemb_project_kernel(const float* __restrict__ W, const float* __restrict__ bias,
                                                                     const float* __restrict__ e, int D, int A,
                                                                     float* __restrict__ v, float* __restrict__ en,
                                                                     int32_t* __restrict__ bad, int32_t* __restrict__ status) {
  extern __shared__ float s_en[];
  __shared__ float s_red[SPE_THREADS];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* eb = e + (long)b * D;
  float ss = 0.f;
  bool finite = true;
  for (int d = tid; d < D; d += SPE_THREADS) {
    const float x = eb[d];
    finite = finite && isfinite(x);
    ss = __fmaf_rn(x, x, ss);
    s_en[d] = x;
  }
  s_red[tid] = ss;
  const int nonfinite = __syncthreads_or(!finite);
#pragma unroll
  for (int h = SPE_THREADS / 2; h > 0; h >>= 1) {
    if (tid < h) s_red[tid] = __fadd_rn(s_red[tid], s_red[tid + h]);
    __syncthreads();
  }
  // a finite embedding whose fp32 sum of squares overflows (elements above ~1.8e19) would normalise to 0 and silently
  // give v = bias: it is flagged like a non-finite one
  const bool flagged = nonfinite || !isfinite(s_red[0]);
  // F.normalize: x / max(||x||, eps), a correctly rounded sqrt and division
  const float nrm = fmaxf(__fsqrt_rn(s_red[0]), 1e-12f);
  for (int d = tid; d < D; d += SPE_THREADS) {
    const float x = __fdiv_rn(s_en[d], nrm);
    s_en[d] = x;
    if (en) en[(long)b * D + d] = x;
  }
  __syncthreads();
  for (int a = warp; a < A; a += SPE_WARPS) {
    const float* wa = W + (long)a * D;
    float acc = 0.f;
    for (int d = lane; d < D; d += 32) acc = __fmaf_rn(__ldg(wa + d), s_en[d], acc);
    acc = warp_sum(acc);
    if (lane == 0) v[(long)b * A + a] = __fadd_rn(acc, __ldg(bias + a));
  }
  if (tid == 0) {
    if (bad) bad[b] = flagged ? 1 : 0;
    if (status && flagged) atomicOr(status, FS2_SPEMB_NONFINITE);
  }
}

// one thread per element of dW [A, D] (i < A * D) and of dbias [A] (the A threads after them)
__global__ void spemb_project_backward_kernel(const float* __restrict__ dv, const float* __restrict__ en, int B, int D, int A,
                                              float* __restrict__ dW, float* __restrict__ dbias) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long nW = (long)A * D;
  if (i < nW) {
    const int a = (int)(i / D), d = (int)(i - (long)a * D);
    float acc = 0.f;
    for (int b = 0; b < B; ++b) acc = __fmaf_rn(dv[(long)b * A + a], en[(long)b * D + d], acc);
    dW[i] = __fadd_rn(dW[i], acc);
  } else if (i < nW + A) {
    const int a = (int)(i - nW);
    float acc = 0.f;
    for (int b = 0; b < B; ++b) acc = __fadd_rn(acc, dv[(long)b * A + a]);
    dbias[a] = __fadd_rn(dbias[a], acc);
  }
}

}  // namespace

int spemb_project(const float* W, const float* bias, const float* e, int B, int D, int A, float* v, float* en, int32_t* bad,
                  int32_t* status, cudaStream_t st) {
  FS2_REQUIRE(W && bias && e && v, "fs2_spemb_project: null argument");
  FS2_REQUIRE(B >= 0 && D >= 1 && D <= FS2_SPEMB_MAX_DIM && A >= 1,
              "fs2_spemb_project: bad shape B=%d D=%d adim=%d (D must lie in [1, %d])", B, D, A, FS2_SPEMB_MAX_DIM);
  if (B == 0) return FS2_OK;
  spemb_project_kernel<<<B, SPE_THREADS, (size_t)D * sizeof(float), st>>>(W, bias, e, D, A, v, en, bad, status);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace fs2

using namespace fs2;

extern "C" {

int fs2_spemb_project(const float* W, const float* bias, const float* spembs, int B, int D, int adim, float* v, float* en,
                      int32_t* bad, int32_t* status, void* stream) {
  return spemb_project(W, bias, spembs, B, D, adim, v, en, bad, status, (cudaStream_t)stream);
}

int fs2_spemb_project_backward(const float* dv, const float* en, int B, int D, int adim, float* dW, float* dbias, void* stream) {
  FS2_REQUIRE(dv && en && dW && dbias, "fs2_spemb_project_backward: null argument");
  FS2_REQUIRE(B >= 0 && D >= 1 && D <= FS2_SPEMB_MAX_DIM && adim >= 1,
              "fs2_spemb_project_backward: bad shape B=%d D=%d adim=%d (D must lie in [1, %d])", B, D, adim, FS2_SPEMB_MAX_DIM);
  if (B == 0) return FS2_OK;
  const long n = (long)adim * D + adim;
  spemb_project_backward_kernel<<<(int)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(dv, en, B, D, adim, dW, dbias);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // extern "C"
