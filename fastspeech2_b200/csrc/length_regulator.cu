// LengthRegulator as prefix-scan + gather (core/duration_modeling/length_regulator.py:38-95,
// utils/util.py:91-104).  The reference expands each phoneme with a Python-level
// `repeat` + `cat` (B*T host syncs on a GPU); here:
//
//   plan   : one CTA per utterance. Durations -> int (alpha scaling with round-half-even,
//            float truncation like int(d_)), all-zero -> all-one rule, block-wide inclusive
//            prefix sum built from warp shuffles, olens[b], max_b olens via atomicMax.
//   gather : out[b,j,:] = hs[b, upper_bound(cum[b,:], j), :]; a CTA owns 32 consecutive
//            frames of one utterance, 32 lanes binary-search their phoneme index (cum row in
//            shared memory), then all 256 threads stream 16-byte vectors: source rows come
//            from L2 (hs is read ~mean-duration times), destination rows are written once
//            with streaming stores.  Pure copy => bit-exact.
//
// HBM-bound: algorithmic bytes = B*T*C*4 (read) + B*T*8 (durations) + B*Lcap*C*4 (write).
#include "common.cuh"

namespace fs2 {
namespace {

constexpr int PLAN_THREADS = 256;

// rint(fp32(d) * fp32(a)), half to even: torch.round(ds.float() * alpha).long() (:58-59).  Clamped to 2^31 so that a sum
// of Tmax of them cannot wrap a long: any total past INT32_MAX reaches the caller through olens / stats[0] and is refused
// there (cum is int32)
__device__ __forceinline__ long scaled_duration(float d, float a) {
  const float s = __fmul_rn(d, a);
  return s >= 2147483648.0f ? 2147483648L : (long)rintf(s);
}

__device__ __forceinline__ long load_duration(const void* ds, int dtype, long idx, float alpha, bool scale) {
  if (dtype == FS2_DUR_F32) {
    float f = ((const float*)ds)[idx];
    if (scale) return scaled_duration(f, alpha);
    return (long)truncf(f);                    // int(d_)                               (:93)
  }
  long d = dtype == FS2_DUR_I32 ? (long)((const int32_t*)ds)[idx] : (long)((const int64_t*)ds)[idx];
  if (scale) return scaled_duration((float)d, alpha);
  return d;
}

__global__ void __launch_bounds__(PLAN_THREADS)
length_plan_kernel(void* ds, int dtype, const int64_t* __restrict__ ilens, float alpha, const float* __restrict__ alpha_v,
                   int T, int mutate, int32_t* __restrict__ cum, int64_t* __restrict__ olens,
                   unsigned long long* __restrict__ stats, int64_t* __restrict__ d_used) {
  __shared__ long warp_tot[PLAN_THREADS / 32];
  __shared__ long carry_s;
  __shared__ int any_nonzero, n_negative;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  long ilen = ilens[b];
  if (ilen > T) ilen = T;
  if (ilen < 0) ilen = 0;
  const bool scale = alpha_v || alpha != 1.0f;   // alpha_v: one factor per phoneme [B, T], in place of the scalar
  const long base = (long)b * T;
  if (tid == 0) { carry_s = 0; any_nonzero = 0; n_negative = 0; }
  __syncthreads();

  // pass 1: the reference tests `d.sum() == 0` on the truncated slice (:86).  For integer
  // durations that is "sum of the (possibly negative) values"; for float durations it is the
  // float sum *before* int().  Track the sum the same way.
  {
    double part = 0.0;
    for (long t = tid; t < ilen; t += PLAN_THREADS) {
      if (dtype == FS2_DUR_F32 && !scale) part += (double)((const float*)ds)[base + t];
      else part += (double)load_duration(ds, dtype, base + t, alpha_v ? alpha_v[base + t] : alpha, scale);
    }
    // any lane with a non-zero partial sum: exact for non-negative inputs (the only valid ones)
    if (part != 0.0) atomicOr(&any_nonzero, 1);
  }
  __syncthreads();
  const bool fill_one = (any_nonzero == 0) && ilen > 0;

  // pass 2: inclusive scan in chunks of PLAN_THREADS
  for (long t0 = 0; t0 < T; t0 += PLAN_THREADS) {
    long t = t0 + tid;
    long d = 0;
    if (t < ilen) {
      d = fill_one ? 1 : load_duration(ds, dtype, base + t, alpha_v ? alpha_v[base + t] : alpha, scale);
      if (d < 0) { atomicAdd(&n_negative, 1); d = 0; }
      if (fill_one && mutate) {  // d.fill_(1) on a view of the caller's tensor (:87)
        if (dtype == FS2_DUR_F32) ((float*)ds)[base + t] = 1.0f;
        else if (dtype == FS2_DUR_I32) ((int32_t*)ds)[base + t] = 1;
        else ((int64_t*)ds)[base + t] = 1;
      }
    }
    long v = d;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      long n = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += n;
    }
    if (lane == 31) warp_tot[wid] = v;
    __syncthreads();
    long prefix = carry_s;
    for (int w = 0; w < wid; ++w) prefix += warp_tot[w];
    v += prefix;
    if (t < T) {
      cum[base + t] = (int32_t)v;  // positions >= ilen repeat the total (d = 0 there)
      if (d_used) d_used[base + t] = d;   // the frame counts the gather expands: scaled, all-zero rule applied, 0 past ilen
    }
    __syncthreads();
    if (tid == PLAN_THREADS - 1) carry_s = v;
    __syncthreads();
  }
  if (tid == 0) {
    olens[b] = carry_s;
    atomicMax(&stats[0], (unsigned long long)carry_s);
    if (n_negative) atomicAdd(&stats[1], (unsigned long long)n_negative);
  }
}

constexpr int FRAMES_PER_CTA = 32;

template <int VEC_PER_ROW_MAX>
__global__ void __launch_bounds__(256)
length_gather_kernel(const float* __restrict__ hs, const int32_t* __restrict__ cum, const int64_t* __restrict__ ilens,
                     int T, int C, float* __restrict__ out, int Lcap, const float* __restrict__ fac_in,
                     float* __restrict__ fac_out) {
  pdl_trigger(); pdl_wait();
  extern __shared__ int32_t scum[];  // [T]
  __shared__ int src_row[FRAMES_PER_CTA];
  const int b = blockIdx.y;
  const int j0 = blockIdx.x * FRAMES_PER_CTA;
  const int tid = threadIdx.x;
  long ilen = ilens[b];
  if (ilen > T) ilen = T;
  if (ilen < 0) ilen = 0;
  const int32_t* crow = cum + (long)b * T;
  const int total = ilen > 0 ? crow[ilen - 1] : 0;
  if (j0 < total) {
    for (int t = tid; t < ilen; t += blockDim.x) scum[t] = crow[t];
  }
  __syncthreads();
  if (tid < FRAMES_PER_CTA) {
    int j = j0 + tid, idx = -1;
    if (j < total) {  // first i with cum[i] > j
      int lo = 0, hi = (int)ilen - 1;
      while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (scum[mid] > j) hi = mid; else lo = mid + 1;
      }
      idx = lo;
    }
    src_row[tid] = idx;
    if (fac_out && j < Lcap) {   // per-phoneme factors [2][B, T] -> per-frame [2][B, Lcap]; 1 where no phoneme is expanded
      const long B = gridDim.y, o = (long)b * Lcap + j, i = (long)b * T + idx;
      fac_out[o] = idx >= 0 ? fac_in[i] : 1.0f;
      fac_out[B * Lcap + o] = idx >= 0 ? fac_in[B * T + i] : 1.0f;
    }
  }
  __syncthreads();
  const int vec_per_row = C >> 2;
  const int nvec = FRAMES_PER_CTA * vec_per_row;
  const float4* src = reinterpret_cast<const float4*>(hs + (long)b * T * C);
  float4* dst = reinterpret_cast<float4*>(out + ((long)b * Lcap + j0) * C);
  for (int v = tid; v < nvec; v += blockDim.x) {
    int f = v / vec_per_row, c = v - f * vec_per_row;
    if (j0 + f >= Lcap) break;
    int r = src_row[f];
    float4 val = r >= 0 ? __ldg(src + (long)r * vec_per_row + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    __stcs(dst + (long)f * vec_per_row + c, val);
  }
}

}  // namespace

int length_plan(void* ds, int ds_dtype, const int64_t* ilens, float alpha, const float* alpha_v, int B, int T, int mutate,
                int32_t* cum, int64_t* olens, int64_t* stats, int64_t* d_used, cudaStream_t st) {
  FS2_REQUIRE(alpha > 0.f, "length_plan: alpha must be > 0 (length_regulator.py:57)");
  FS2_REQUIRE(!(alpha_v && mutate), "length_plan: per-phoneme factors scale a private copy, mutate_ds must be 0");
  FS2_REQUIRE(ds_dtype == FS2_DUR_I64 || ds_dtype == FS2_DUR_F32 || ds_dtype == FS2_DUR_I32, "length_plan: bad ds dtype %d", ds_dtype);
  FS2_CUDA_CHECK(cudaMemsetAsync(stats, 0, 2 * sizeof(int64_t), st));
  if (B == 0) return FS2_OK;
  length_plan_kernel<<<B, PLAN_THREADS, 0, st>>>(ds, ds_dtype, ilens, alpha, alpha_v, T, mutate, cum, olens,
                                                 reinterpret_cast<unsigned long long*>(stats), d_used);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int length_gather(const float* hs, const int32_t* cum, const int64_t* ilens, int B, int T, int C, float* out, int Lcap,
                  const float* fac_in, float* fac_out, cudaStream_t st) {
  FS2_REQUIRE(C % 4 == 0, "length_gather: C must be a multiple of 4");
  FS2_REQUIRE((fac_in == nullptr) == (fac_out == nullptr), "length_gather: factors in and out must both be given or both be NULL");
  if (B == 0 || Lcap == 0) return FS2_OK;
  size_t smem = (size_t)T * sizeof(int32_t);
  FS2_REQUIRE(smem <= 200 * 1024, "length_gather: Tmax=%d too large for the shared cum row", T);
  static unsigned long long attr_set = 0;   // per-device bit mask: the attribute is a per-device setting
  if (smem > 48 * 1024) {
    int dev = 0;
    FS2_CUDA_CHECK(cudaGetDevice(&dev));
    if (dev >= 64 || !((attr_set >> dev) & 1ull)) {
      FS2_CUDA_CHECK(cudaFuncSetAttribute(length_gather_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      if (dev < 64) attr_set |= 1ull << dev;
    }
  }
  dim3 grid((Lcap + FRAMES_PER_CTA - 1) / FRAMES_PER_CTA, B);
  FS2_CUDA_CHECK(launch_pdl(length_gather_kernel<0>, grid, dim3(256), smem, st, hs, cum, ilens, T, C, out, Lcap, fac_in, fac_out));
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace fs2
