// HBM-bound row kernels: embedding + positional encoding, LayerNorm with the fusions the
// path needs, bucketize + embedding-gather-add, one-hot, masked losses, weight repacking.
// One warp owns one [C]-row and keeps it in registers (C = 256 or 384 -> 2 or 3 float4 per
// lane), so every row is read once and written once with 16-byte coalesced accesses.
#include "common.cuh"

namespace fs2 {
namespace {

constexpr int ROWS_PER_CTA = 8;  // 8 warps

// ---- encoder input: Embedding(pad 0) + x + alpha * pe  (fastspeech.py:65-67, embedding.py:119) ----
template <int NV>  // float4 per lane
__global__ void embed_posenc_kernel(const int64_t* __restrict__ xs, const float* __restrict__ table, int n_sym,
                                    const float* __restrict__ pe, const float* __restrict__ alpha, long rows, int T,
                                    float* __restrict__ out, __half* __restrict__ planes, const int64_t* __restrict__ lens) {
  pdl_trigger(); pdl_wait();
  const int C = NV * 128;
  long row = (long)blockIdx.x * ROWS_PER_CTA + (threadIdx.x >> 5);
  if (row >= rows) return;
  int lane = threadIdx.x & 31;
  int t = (int)(row % T);
  const bool padded = lens && t >= lens[row / T];
  long id = xs[row];
  if (id < 0 || id >= n_sym) id = 0;  // out-of-range ids behave like padding instead of faulting
  const float a = __ldg(alpha);
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    int c = v * 128 + lane * 4;
    float4 e = __ldg(reinterpret_cast<const float4*>(table + id * C + c));
    float4 p = __ldg(reinterpret_cast<const float4*>(pe + (long)t * C + c));
    float4 o;  // x + (alpha * pe): two roundings like the reference's mul then add
    o.x = __fadd_rn(e.x, __fmul_rn(a, p.x)); o.y = __fadd_rn(e.y, __fmul_rn(a, p.y));
    o.z = __fadd_rn(e.z, __fmul_rn(a, p.z)); o.w = __fadd_rn(e.w, __fmul_rn(a, p.w));
    if (padded) o = make_float4(0.f, 0.f, 0.f, 0.f);
    *reinterpret_cast<float4*>(out + row * C + c) = o;
    if (planes) {   // operand planes of the first q|k|v projection (3xF16)
      uint2 hv, lv;
      split_pair(o.x, o.y, hv.x, lv.x); split_pair(o.z, o.w, hv.y, lv.y);
      *reinterpret_cast<uint2*>(planes + row * C + c) = hv;
      *reinterpret_cast<uint2*>(planes + (rows + row) * C + c) = lv;
    }
  }
}

// ---- LayerNorm over channels with optional residual / ReLU / pos-enc / scalar head ----------
// encoder.py:60-69 (eps 1e-5), encoder.py:119-125, modules.py:112-120 (eps 1e-12),
// duration_predictor.py:75-84, variance_predictor.py:50-51,75-78.
template <int NV>
__global__ void row_norm_kernel(RowNorm r) {
  pdl_trigger(); pdl_wait();
  long row = (long)blockIdx.x * ROWS_PER_CTA + (threadIdx.x >> 5);
  if (row >= r.rows) return;
  const int C = NV * 128;
  int lane = threadIdx.x & 31;
  float4 v[NV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int c = i * 128 + lane * 4;
    v[i] = *reinterpret_cast<const float4*>(r.x + row * r.ldx + c);
    if (r.resid) {
      float4 q = *reinterpret_cast<const float4*>(r.resid + row * r.ldr + c);
      v[i].x += q.x; v[i].y += q.y; v[i].z += q.z; v[i].w += q.w;
    }
    s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
  const float mean = warp_sum(s) * (1.0f / C);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    ss += (a * a + b * b) + (c * c + d * d);
  }
  const float rstd = 1.0f / sqrtf(warp_sum(ss) * (1.0f / C) + r.eps);
  int t = r.L > 0 ? (int)(row % r.L) : 0;
  long bidx = r.L > 0 ? row / r.L : 0;
  const bool padded = r.lens && (long)t >= r.lens[bidx];
  const float alpha = r.pe ? __ldg(r.alpha) : 0.f;
  float dot = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int c = i * 128 + lane * 4;
    float4 g = __ldg(reinterpret_cast<const float4*>(r.gamma + c));
    float4 b = __ldg(reinterpret_cast<const float4*>(r.beta + c));
    float4 y;
    y.x = (v[i].x - mean) * rstd * g.x + b.x; y.y = (v[i].y - mean) * rstd * g.y + b.y;
    y.z = (v[i].z - mean) * rstd * g.z + b.z; y.w = (v[i].w - mean) * rstd * g.w + b.w;
    if (r.relu_after) { y.x = fmaxf(y.x, 0.f); y.y = fmaxf(y.y, 0.f); y.z = fmaxf(y.z, 0.f); y.w = fmaxf(y.w, 0.f); }
    if (r.pe) {
      float4 p = __ldg(reinterpret_cast<const float4*>(r.pe + (long)t * C + c));
      y.x = __fadd_rn(y.x, __fmul_rn(alpha, p.x)); y.y = __fadd_rn(y.y, __fmul_rn(alpha, p.y));
      y.z = __fadd_rn(y.z, __fmul_rn(alpha, p.z)); y.w = __fadd_rn(y.w, __fmul_rn(alpha, p.w));
    }
    if (r.head_w) {
      float4 w = __ldg(reinterpret_cast<const float4*>(r.head_w + c));
      dot += (y.x * w.x + y.y * w.y) + (y.z * w.z + y.w * w.w);
    }
    if (padded) y = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r.out) *reinterpret_cast<float4*>(r.out + row * r.ldo + c) = y;
    if (r.split_out) {   // operand planes of the next contraction: hi = rn(s y), lo = rn(s y - hi), 8-byte stores
      uint2 hv, lv;
      split_pair(y.x, y.y, hv.x, lv.x); split_pair(y.z, y.w, hv.y, lv.y);
      *reinterpret_cast<uint2*>(r.split_out + row * C + c) = hv;
      if (r.split_lo) *reinterpret_cast<uint2*>(r.split_out + (r.rows + row) * C + c) = lv;
    }
  }
  if (r.head_w) {
    dot = warp_sum(dot) + __ldg(r.head_b);
    if (lane == 0) {
      if (r.head_out) r.head_out[row] = padded ? 0.f : (r.head_scale ? __fmul_rn(dot, __ldg(r.head_scale + row)) : dot);
      if (r.dur_out) {
        // clamp(round(exp(x) - 1), min=0).long(), round = half to even (duration_predictor.py:77-81)
        float d = fmaxf(rintf(expf(dot) - 1.0f), 0.f);
        r.dur_out[row] = padded ? 0 : (int64_t)d;
      }
    }
  }
}

// ---- bucketize (variance_predictor.py:158,231) ------------------------------------------------
__global__ void bucketize_kernel(const float* __restrict__ vals, const float* __restrict__ bins, int n_edges, int64_t n,
                                 int64_t* __restrict__ ids) {
  extern __shared__ float sbins[];
  for (int i = threadIdx.x; i < n_edges; i += blockDim.x) sbins[i] = bins[i];
  __syncthreads();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    ids[i] = bucket_of(vals[i], sbins, n_edges);
}

__global__ void one_hot_kernel(const int64_t* __restrict__ ids, int64_t n, int n_bins, float* __restrict__ out) {
  // one warp per row, float4 stores
  int64_t row = (int64_t)blockIdx.x * ROWS_PER_CTA + (threadIdx.x >> 5);
  if (row >= n) return;
  int lane = threadIdx.x & 31;
  int id = (int)ids[row];
  for (int c = lane * 4; c < n_bins; c += 128) {
    float4 o = make_float4(c == id ? 1.f : 0.f, c + 1 == id ? 1.f : 0.f, c + 2 == id ? 1.f : 0.f, c + 3 == id ? 1.f : 0.f);
    __stcs(reinterpret_cast<float4*>(out + row * n_bins + c), o);
  }
}

// ---- hs + pitch_embed(one_hot_pitch) + energy_embed(one_hot_energy)  (fastspeech.py:218-219) ---
// one_hot x Linear == W[:, id] + b exactly (all other products are +0), so this is a gather.
template <int NV>
__global__ void variance_embed_add_kernel(const float* __restrict__ hm, const float* __restrict__ e_val,
                                          const float* __restrict__ p_val, const float* __restrict__ e_bins,
                                          const float* __restrict__ p_bins, int n_edges, const float* __restrict__ e_tab,
                                          const float* __restrict__ e_bias, const float* __restrict__ p_tab,
                                          const float* __restrict__ p_bias, int64_t rows, float* __restrict__ out,
                                          __half* __restrict__ planes, int planes_lo,
                                          int64_t* __restrict__ e_ids, int64_t* __restrict__ p_ids,
                                          const int64_t* __restrict__ lens, int L) {
  pdl_trigger(); pdl_wait();
  const int C = NV * 128;
  int64_t row = (int64_t)blockIdx.x * ROWS_PER_CTA + (threadIdx.x >> 5);
  if (row >= rows) return;
  int lane = threadIdx.x & 31;
  const bool padded = lens && row % L >= lens[row / L];
  int ide = bucket_of(__ldg(e_val + row), e_bins, n_edges);
  int idp = bucket_of(__ldg(p_val + row), p_bins, n_edges);
  if (lane == 0) {
    if (e_ids) e_ids[row] = padded ? -1 : ide;
    if (p_ids) p_ids[row] = padded ? -1 : idp;
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int c = i * 128 + lane * 4;
    float4 h = *reinterpret_cast<const float4*>(hm + row * C + c);
    float4 pw = __ldg(reinterpret_cast<const float4*>(p_tab + (long)idp * C + c));
    float4 pb = __ldg(reinterpret_cast<const float4*>(p_bias + c));
    float4 ew = __ldg(reinterpret_cast<const float4*>(e_tab + (long)ide * C + c));
    float4 eb = __ldg(reinterpret_cast<const float4*>(e_bias + c));
    float4 o;  // pitch first, then energy (fastspeech.py:218-219)
    o.x = __fadd_rn(__fadd_rn(h.x, __fadd_rn(pw.x, pb.x)), __fadd_rn(ew.x, eb.x));
    o.y = __fadd_rn(__fadd_rn(h.y, __fadd_rn(pw.y, pb.y)), __fadd_rn(ew.y, eb.y));
    o.z = __fadd_rn(__fadd_rn(h.z, __fadd_rn(pw.z, pb.z)), __fadd_rn(ew.z, eb.z));
    o.w = __fadd_rn(__fadd_rn(h.w, __fadd_rn(pw.w, pb.w)), __fadd_rn(ew.w, eb.w));
    if (padded) o = make_float4(0.f, 0.f, 0.f, 0.f);
    if (out) *reinterpret_cast<float4*>(out + row * C + c) = o;
    if (planes) {   // operand planes of the decoder input Linear
      uint2 hv, lv;
      split_pair(o.x, o.y, hv.x, lv.x); split_pair(o.z, o.w, hv.y, lv.y);
      *reinterpret_cast<uint2*>(planes + row * C + c) = hv;
      if (planes_lo) *reinterpret_cast<uint2*>(planes + (rows + row) * C + c) = lv;
    }
  }
}

// ---- masked losses (fastspeech.py:277-333) ---------------------------------------------------
// acc[0..4] (double): sum|before-ys|, sum|after-ys|, sum(d-log(ds+1))^2, sum(e-es)^2, sum(p-ps)^2
__device__ __forceinline__ void block_accumulate(float v, double* dst) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0 && v != 0.f) atomicAdd(dst, (double)v);
}

__global__ void loss_mel_kernel(const float* __restrict__ before, const float* __restrict__ after,
                                const float* __restrict__ ys, int ld_ys_time, const int64_t* __restrict__ olens, int L,
                                int odim, double* acc) {
  // grid: (chunks, B).  The valid part of an utterance is one contiguous run of olens[b]*odim floats in all three
  // tensors (odim % 4 == 0), so the kernel streams 16-byte vectors: HBM-bound, 3 x 4 bytes per valid element.
  const int b = blockIdx.y;
  const long nvec = (long)olens[b] * odim / 4;
  const float4* pb = reinterpret_cast<const float4*>(before + (long)b * L * odim);
  const float4* pa = reinterpret_cast<const float4*>(after + (long)b * L * odim);
  const float4* py = reinterpret_cast<const float4*>(ys + (long)b * ld_ys_time * odim);
  float s0 = 0.f, s1 = 0.f;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long)gridDim.x * blockDim.x) {
    const float4 y = __ldg(py + i), x0 = __ldg(pb + i), x1 = __ldg(pa + i);
    s0 += (fabsf(x0.x - y.x) + fabsf(x0.y - y.y)) + (fabsf(x0.z - y.z) + fabsf(x0.w - y.w));
    s1 += (fabsf(x1.x - y.x) + fabsf(x1.y - y.y)) + (fabsf(x1.z - y.z) + fabsf(x1.w - y.w));
  }
  block_accumulate(s0, acc + 0);
  block_accumulate(s1, acc + 1);
}

__global__ void loss_seq_kernel(const float* __restrict__ d_out, const void* __restrict__ ds, int ds_dtype,
                                const float* __restrict__ e_out, const float* __restrict__ p_out,
                                const float* __restrict__ es, const float* __restrict__ ps,
                                const int64_t* __restrict__ ilens, const int64_t* __restrict__ olens, int T, int L,
                                double* acc) {
  int b = blockIdx.y;
  float sd = 0.f, se = 0.f, sp = 0.f;
  long il = ilens[b], ol = olens[b];
  for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < il; t += (long)gridDim.x * blockDim.x) {
    long o = (long)b * T + t;
    float d = ds_dtype == FS2_DUR_F32 ? ((const float*)ds)[o]
            : ds_dtype == FS2_DUR_I32 ? (float)((const int32_t*)ds)[o] : (float)((const int64_t*)ds)[o];
    float diff = d_out[o] - logf(d + 1.0f);  // duration_predictor.py:148
    sd += diff * diff;
  }
  for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < ol; t += (long)gridDim.x * blockDim.x) {
    long o = (long)b * L + t;
    float de = e_out[o] - es[o], dp = p_out[o] - ps[o];
    se += de * de; sp += dp * dp;
  }
  block_accumulate(sd, acc + 2);
  block_accumulate(se, acc + 3);
  block_accumulate(sp, acc + 4);
}

__global__ void loss_finalize_kernel(const double* acc, const int64_t* ilens, const int64_t* olens, int B, int odim,
                                     float* out7) {
  double ni = 0, no = 0;
  for (int b = 0; b < B; ++b) { ni += (double)ilens[b]; no += (double)olens[b]; }
  float before = (float)(acc[0] / (no * odim)), after = (float)(acc[1] / (no * odim));
  float dur = (float)(acc[2] / ni), en = (float)(acc[3] / no), pi = (float)(acc[4] / no);
  float l1 = before + after;
  out7[0] = l1; out7[1] = before; out7[2] = after; out7[3] = dur; out7[4] = en; out7[5] = pi;
  out7[6] = ((l1 + dur) + en) + pi;  // fastspeech.py:324
}

// ---- weight repacking -------------------------------------------------------------------------
__global__ void pack_conv_weight_kernel(const float* __restrict__ src, int N, int K, int taps,
                                        const float* __restrict__ scale, float* __restrict__ dst) {
  long total = (long)N * K * taps;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    // dst index i = (j*N + n)*K + k
    int k = (int)(i % K); long r = i / K; int n = (int)(r % N); int j = (int)(r / N);
    float v = src[((long)n * K + k) * taps + j];
    if (scale) v *= scale[n];
    dst[i] = v;
  }
}
__global__ void pack_transpose_kernel(const float* __restrict__ src, int rows, int cols, float* __restrict__ dst) {
  long total = (long)rows * cols;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    int r = (int)(i % rows); int c = (int)(i / rows);  // dst [cols][rows]
    dst[i] = src[(long)r * cols + c];
  }
}
__global__ void fold_batchnorm_kernel(const float* gamma, const float* beta, const float* mean, const float* var,
                                      float eps, int N, float* scale, float* shift) {
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float s = gamma[n] / sqrtf(var[n] + eps);  // BatchNorm1d eval (modules.py:296, eps 1e-5)
  scale[n] = s;
  shift[n] = beta[n] - mean[n] * s;
}

inline int grid_for(long n, int block, int cap = 132 * 8) {
  long g = (n + block - 1) / block;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace

int embed_posenc(const int64_t* xs, const float* table, int n_sym, const float* pe, const float* alpha, int B, int T,
                 int C, float* out, __half* planes, const int64_t* lens, cudaStream_t st) {
  long rows = (long)B * T;
  if (rows == 0) return FS2_OK;
  int grid = (int)((rows + ROWS_PER_CTA - 1) / ROWS_PER_CTA);
  if (C == 256) { FS2_CUDA_CHECK(launch_pdl(embed_posenc_kernel<2>, dim3(grid), dim3(256), 0, st, xs, table, n_sym, pe, alpha, rows, T, out, planes, lens)); }
  else if (C == 384) { FS2_CUDA_CHECK(launch_pdl(embed_posenc_kernel<3>, dim3(grid), dim3(256), 0, st, xs, table, n_sym, pe, alpha, rows, T, out, planes, lens)); }
  else { set_error("embed_posenc: C=%d unsupported (256 or 384)", C); return FS2_ERR_INVALID; }
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int row_norm(const RowNorm& r, cudaStream_t st) {
  if (r.rows == 0) return FS2_OK;
  FS2_REQUIRE(r.ldx % 4 == 0 && (!r.out || r.ldo % 4 == 0) && (!r.resid || r.ldr % 4 == 0), "row_norm: strides must be 16-byte multiples");
  FS2_REQUIRE(!r.split_out || (reinterpret_cast<uintptr_t>(r.split_out) & 7) == 0, "row_norm: operand planes must be 8-byte aligned");
  FS2_REQUIRE(!r.lens || r.L > 0, "row_norm: lens needs L > 0");
  int grid = (int)((r.rows + ROWS_PER_CTA - 1) / ROWS_PER_CTA);
  if (r.C == 256) { FS2_CUDA_CHECK(launch_pdl(row_norm_kernel<2>, dim3(grid), dim3(256), 0, st, r)); }
  else if (r.C == 384) { FS2_CUDA_CHECK(launch_pdl(row_norm_kernel<3>, dim3(grid), dim3(256), 0, st, r)); }
  else { set_error("row_norm: C=%d unsupported (256 or 384)", r.C); return FS2_ERR_INVALID; }
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int bucketize(const float* vals, const float* bins, int n_edges, int64_t n, int64_t* ids, cudaStream_t st) {
  if (n == 0) return FS2_OK;
  bucketize_kernel<<<grid_for(n, 256), 256, n_edges * sizeof(float), st>>>(vals, bins, n_edges, n, ids);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int one_hot(const int64_t* ids, int64_t n, int n_bins, float* out, cudaStream_t st) {
  if (n == 0) return FS2_OK;
  FS2_REQUIRE(n_bins % 4 == 0, "one_hot: n_bins must be a multiple of 4");
  one_hot_kernel<<<(int)((n + ROWS_PER_CTA - 1) / ROWS_PER_CTA), 256, 0, st>>>(ids, n, n_bins, out);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int variance_embed_add(const float* hm, const float* e_val, const float* p_val, const float* e_bins, const float* p_bins,
                       int n_edges, const float* e_tab, const float* e_bias, const float* p_tab, const float* p_bias,
                       int64_t rows, int C, float* out, __half* planes, int planes_lo, int64_t* e_ids, int64_t* p_ids,
                       const int64_t* lens, int L, cudaStream_t st) {
  if (rows == 0) return FS2_OK;
  FS2_REQUIRE(!lens || L > 0, "variance_embed_add: lens needs L > 0");
  int grid = (int)((rows + ROWS_PER_CTA - 1) / ROWS_PER_CTA);
  if (C == 256) {
    FS2_CUDA_CHECK(launch_pdl(variance_embed_add_kernel<2>, dim3(grid), dim3(256), 0, st, hm, e_val, p_val, e_bins, p_bins, n_edges, e_tab, e_bias, p_tab,
                              p_bias, rows, out, planes, planes_lo, e_ids, p_ids, lens, L));
  } else if (C == 384) {
    FS2_CUDA_CHECK(launch_pdl(variance_embed_add_kernel<3>, dim3(grid), dim3(256), 0, st, hm, e_val, p_val, e_bins, p_bins, n_edges, e_tab, e_bias, p_tab,
                              p_bias, rows, out, planes, planes_lo, e_ids, p_ids, lens, L));
  }
  else { set_error("variance_embed_add: C=%d unsupported", C); return FS2_ERR_INVALID; }
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int masked_losses(const float* before, const float* after, const float* ys, int ld_ys_time, const float* d_out,
                  const void* ds, int ds_dtype, const float* e_out, const float* p_out, const float* es, const float* ps,
                  const int64_t* ilens, const int64_t* olens, int B, int T, int L, int odim, float* out7, void* scratch,
                  cudaStream_t st) {
  double* acc = reinterpret_cast<double*>(scratch);
  FS2_REQUIRE(odim % 4 == 0 && (reinterpret_cast<uintptr_t>(ys) & 15) == 0, "masked_losses: odim must be a multiple of 4 and ys 16-byte aligned");
  FS2_CUDA_CHECK(cudaMemsetAsync(acc, 0, 8 * sizeof(double), st));
  if (B > 0) {
    dim3 g1(grid_for((long)L * odim / 4, 256, 32), B), g2(grid_for(L > T ? L : T, 256, 16), B);
    loss_mel_kernel<<<g1, 256, 0, st>>>(before, after, ys, ld_ys_time, olens, L, odim, acc);
    FS2_LAUNCH_CHECK();
    loss_seq_kernel<<<g2, 256, 0, st>>>(d_out, ds, ds_dtype, e_out, p_out, es, ps, ilens, olens, T, L, acc);
    FS2_LAUNCH_CHECK();
  }
  loss_finalize_kernel<<<1, 1, 0, st>>>(acc, ilens, olens, B, odim, out7);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

int pack_conv_weight(const float* src, int N, int K, int taps, const float* scale, float* dst, cudaStream_t st) {
  pack_conv_weight_kernel<<<grid_for((long)N * K * taps, 256), 256, 0, st>>>(src, N, K, taps, scale, dst);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int pack_transpose(const float* src, int rows, int cols, float* dst, cudaStream_t st) {
  pack_transpose_kernel<<<grid_for((long)rows * cols, 256), 256, 0, st>>>(src, rows, cols, dst);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}
int fold_batchnorm(const float* gamma, const float* beta, const float* mean, const float* var, float eps, int N,
                   float* scale, float* shift, cudaStream_t st) {
  fold_batchnorm_kernel<<<(N + 127) / 128, 128, 0, st>>>(gamma, beta, mean, var, eps, N, scale, shift);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace fs2
