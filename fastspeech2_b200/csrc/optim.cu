// Optimizer step of the train loop (DESIGN.md section 15): the reference's clip_grad_norm_ + NaN guard + NoamOpt.step()
// (Adam, betas (0.9, 0.98), eps 1e-9, no weight decay) as three launches over a multi-tensor table:
//   optim_sumsq_kernel   one CTA per chunk of FS2_OPTIM_CHUNK elements: fp64 sum of squares of the grads
//   optim_scalar_kernel  one CTA: fixed-order sum of the chunk sums -> norm, clip coefficient, skip flag; when the step
//                        runs, advances the Noam counter and every entry's Adam step and forms the per-entry scalars
//   optim_update_kernel  one CTA per chunk: g *= coefficient, then torch's foreach Adam arithmetic, one pass over p, g, m, v
// The reduction tree depends only on the table (chunk boundaries, 256 threads per chunk, fixed combine order), never on
// the SM count, the grid schedule or the stream.  Every fp32 operation is an explicit _rn intrinsic: torch evaluates
// lerp / mul / addcmul / sqrt / div / add / addcdiv as separate kernels, and its addcmul / addcdiv and lerp are fmas.
#include "common.cuh"

namespace fs2 {
namespace {

constexpr int kThreads = 256;
constexpr int64_t kChunk = FS2_OPTIM_CHUNK;

struct Scalars {          // workspace tail written by optim_scalar_kernel
  float norm, coef;
  int skip, pad;
};

// ---- double-double helpers for the per-step scalars ---------------------------------------------------------------------
__device__ __forceinline__ void dd_mul(double ah, double al, double bh, double bl, double& rh, double& rl) {
  const double p = __dmul_rn(ah, bh);
  double e = __fma_rn(ah, bh, -p);
  e = __dadd_rn(e, __dadd_rn(__dmul_rn(ah, bl), __dmul_rn(al, bh)));
  rh = __dadd_rn(p, e);
  rl = __dsub_rn(e, __dsub_rn(rh, p));
}

// beta ** n for integer n >= 1, squaring in double-double, rounded to double (tests/_optim_plan.py::pow_int)
__device__ double pow_int(double beta, int64_t n) {
  double rh = 1.0, rl = 0.0, bh = beta, bl = 0.0;
  while (n > 0) {
    if (n & 1) dd_mul(rh, rl, bh, bl, rh, rl);
    dd_mul(bh, bl, bh, bl, bh, bl);
    n >>= 1;
  }
  return __dadd_rn(rh, rl);
}

// correctly rounded s ** -0.5 (s >= 1): 1 / sqrt(s) and one Newton correction from the exact residual 1 - s r^2
__device__ double rsqrt_cr(double s) {
  const double r = __ddiv_rn(1.0, __dsqrt_rn(s));
  const double p = __dmul_rn(r, r), pe = __fma_rn(r, r, -p);
  const double a = __dmul_rn(s, p), ae = __fma_rn(s, p, -a);
  const double e = __dsub_rn(__dsub_rn(__dsub_rn(1.0, a), ae), __dmul_rn(s, pe));
  return __dadd_rn(r, __dmul_rn(__dmul_rn(r, 0.5), e));
}

// NoamOpt.rate(step): (factor * model_size ** -0.5) * min(step ** -0.5, step * warmup ** -1.5), in double
__device__ double noam_rate(int64_t step, const fs2_noam_adam_hp& hp) {
  const double s = (double)step;
  const double r = rsqrt_cr(s), sw = __dmul_rn(s, hp.warmup_pow);
  return __dmul_rn(hp.rate_scale, sw < r ? sw : r);
}

// torch Adam's per-tensor scalars, cast to fp32 as its foreach kernels receive them: -lr / (1 - beta1 ** t) and
// sqrt(1 - beta2 ** t).  t is the fp32 step count as torch keeps it (exact integers up to 2^24)
__device__ void adam_scalars(double lr, float t, const fs2_noam_adam_hp& hp, float& step_size, float& bc2_sqrt) {
  const int64_t n = t >= 1.0f ? (t < 1.0e18f ? (int64_t)t : (int64_t)1e18) : 1;
  const double bc1 = __dsub_rn(1.0, pow_int(hp.beta1, n));
  const double bc2 = __dsub_rn(1.0, pow_int(hp.beta2, n));
  step_size = __double2float_rn(-__ddiv_rn(lr, bc1));
  bc2_sqrt = __double2float_rn(__dsqrt_rn(bc2));
}

__device__ __forceinline__ int entry_of(const fs2_optim_entry* __restrict__ table, int n, int64_t chunk) {
  int lo = 0, hi = n - 1;                                // last entry with chunk0 <= chunk
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (table[mid].chunk0 <= chunk) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// fixed-order block sum: warp xor tree, then warp 0 adds the eight warp sums in order
__device__ double block_sum(double v) {
  __shared__ double warp[kThreads / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) warp[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kThreads / 32; ++w) s = __dadd_rn(s, warp[w]);
  return s;                                             // valid in thread 0
}

__device__ __forceinline__ bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

__global__ void __launch_bounds__(kThreads) optim_sumsq_kernel(const fs2_optim_entry* __restrict__ table, int n,
                                                                double* __restrict__ partial) {
  const int64_t c = blockIdx.x;
  const fs2_optim_entry e = table[entry_of(table, n, c)];
  const int64_t off = (c - e.chunk0) * kChunk;
  const int64_t len = min(kChunk, e.numel - off);
  const float* g = e.grad + off;
  double acc = 0.0;
  int64_t head = 0;
  if (((uintptr_t)g & 3) == 0) head = min(len, (int64_t)(((16 - ((uintptr_t)g & 15)) & 15) >> 2));
  else head = len;
  for (int64_t i = threadIdx.x; i < head; i += kThreads) { const double x = g[i]; acc = __fma_rn(x, x, acc); }
  const int64_t nv = (len - head) >> 2;
  const float4* g4 = reinterpret_cast<const float4*>(g + head);
  for (int64_t i = threadIdx.x; i < nv; i += kThreads) {
    const float4 x = __ldg(g4 + i);
    acc = __fma_rn((double)x.x, (double)x.x, acc);
    acc = __fma_rn((double)x.y, (double)x.y, acc);
    acc = __fma_rn((double)x.z, (double)x.z, acc);
    acc = __fma_rn((double)x.w, (double)x.w, acc);
  }
  for (int64_t i = head + nv * 4 + threadIdx.x; i < len; i += kThreads) { const double x = g[i]; acc = __fma_rn(x, x, acc); }
  const double s = block_sum(acc);
  if (threadIdx.x == 0) partial[c] = s;
}

// clip < 0: step() (coefficient 1, no norm)
__global__ void __launch_bounds__(kThreads) optim_scalar_kernel(const fs2_optim_entry* __restrict__ table, int n,
                                                                 int64_t n_chunks, const double* __restrict__ partial,
                                                                 float max_norm, int clip, fs2_noam_adam_hp hp,
                                                                 int64_t* noam_step, double* lr_out, float* norm_out,
                                                                 float2* __restrict__ per_entry, Scalars* sc) {
  __shared__ int s_skip;
  __shared__ double s_lr;
  if (clip) {
    double acc = 0.0;
    for (int64_t i = threadIdx.x; i < n_chunks; i += kThreads) acc = __dadd_rn(acc, partial[i]);
    const double total = block_sum(acc);
    if (threadIdx.x == 0) {
      const float norm = __double2float_rn(__dsqrt_rn(total));      // sqrt in double, then fp32: one correct rounding
      float coef = __fmul_rn(__frcp_rn(__fadd_rn(norm, 1e-6f)), max_norm);
      coef = isnan(coef) ? coef : fminf(coef, 1.0f);
      *norm_out = norm;
      s_skip = isnan(norm);
      sc->norm = norm; sc->coef = coef; sc->skip = s_skip;
    }
  } else if (threadIdx.x == 0) {
    s_skip = 0;
    sc->norm = 0.0f; sc->coef = 1.0f; sc->skip = 0;
  }
  if (threadIdx.x == 0 && !s_skip) {
    const int64_t step = *noam_step + 1;
    *noam_step = step;
    s_lr = noam_rate(step, hp);
    *lr_out = s_lr;
  }
  __syncthreads();
  if (s_skip) return;
  for (int t = threadIdx.x; t < n; t += kThreads) {
    float* sp = table[t].step;
    const float st = __fadd_rn(*sp, 1.0f);
    *sp = st;
    float ss, bc;
    adam_scalars(s_lr, st, hp, ss, bc);
    per_entry[t] = make_float2(ss, bc);
  }
}

struct AdamConst { float w1, b2, c2, eps; };

__device__ __forceinline__ void adam_one(float& p, float g, float& m, float& v, float coef, float ss, float bc, const AdamConst& k) {
  g = __fmul_rn(g, coef);                                                   // clip: torch._foreach_mul_(grads, coef)
  m = __fmaf_rn(k.w1, __fsub_rn(g, m), m);                                  // lerp_(m, g, 1 - beta1): m + w (g - m)
  v = __fmaf_rn(k.c2, __fmul_rn(g, g), __fmul_rn(v, k.b2));                 // mul_(v, beta2); addcmul_(v, g, g, 1 - beta2)
  const float den = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc), k.eps);         // sqrt; div_(bc2_sqrt); add_(eps)
  p = __fmaf_rn(ss, __fdiv_rn(m, den), p);                                  // addcdiv_(p, m, den, step_size)
}

__global__ void __launch_bounds__(kThreads) optim_update_kernel(const fs2_optim_entry* __restrict__ table, int n,
                                                                 const float2* __restrict__ per_entry,
                                                                 const Scalars* __restrict__ sc, AdamConst k) {
  if (sc->skip) return;
  const float coef = sc->coef;
  const int64_t c = blockIdx.x;
  const int t = entry_of(table, n, c);
  const fs2_optim_entry e = table[t];
  const float2 s = per_entry[t];
  const int64_t off = (c - e.chunk0) * kChunk;
  const int64_t len = min(kChunk, e.numel - off);
  float* p = e.param + off; const float* g = e.grad + off; float* m = e.exp_avg + off; float* v = e.exp_avg_sq + off;
  const uintptr_t mis = (uintptr_t)p & 15;
  const bool vec = ((uintptr_t)g & 15) == mis && ((uintptr_t)m & 15) == mis && ((uintptr_t)v & 15) == mis && (mis & 3) == 0;
  const int64_t head = vec ? min(len, (int64_t)(((16 - mis) & 15) >> 2)) : len;
  for (int64_t i = threadIdx.x; i < head; i += kThreads) {
    float pi = p[i], mi = m[i], vi = v[i];
    adam_one(pi, g[i], mi, vi, coef, s.x, s.y, k);
    p[i] = pi; m[i] = mi; v[i] = vi;
  }
  const int64_t nv = (len - head) >> 2;
  float4* p4 = reinterpret_cast<float4*>(p + head); const float4* g4 = reinterpret_cast<const float4*>(g + head);
  float4* m4 = reinterpret_cast<float4*>(m + head); float4* v4 = reinterpret_cast<float4*>(v + head);
  for (int64_t i = threadIdx.x; i < nv; i += kThreads) {
    float4 pp = p4[i], mm = m4[i], vv = v4[i];
    const float4 gg = __ldg(g4 + i);
    adam_one(pp.x, gg.x, mm.x, vv.x, coef, s.x, s.y, k);
    adam_one(pp.y, gg.y, mm.y, vv.y, coef, s.x, s.y, k);
    adam_one(pp.z, gg.z, mm.z, vv.z, coef, s.x, s.y, k);
    adam_one(pp.w, gg.w, mm.w, vv.w, coef, s.x, s.y, k);
    p4[i] = pp; m4[i] = mm; v4[i] = vv;
  }
  for (int64_t i = head + nv * 4 + threadIdx.x; i < len; i += kThreads) {
    float pi = p[i], mi = m[i], vi = v[i];
    adam_one(pi, g[i], mi, vi, coef, s.x, s.y, k);
    p[i] = pi; m[i] = mi; v[i] = vi;
  }
}

__global__ void optim_noam_scalars_kernel(int64_t step0, int count, fs2_noam_adam_hp hp, double* lr, float* step_size,
                                          float* bc2_sqrt) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
    const int64_t step = step0 + i;
    const double r = noam_rate(step, hp);
    float ss, bc;
    adam_scalars(r, (float)step, hp, ss, bc);
    lr[i] = r; step_size[i] = ss; bc2_sqrt[i] = bc;
  }
}

struct Plan {
  int64_t n_chunks = 0;
  size_t bytes = 0, off_entry = 0, off_scalars = 0;
};

int make_plan(const int64_t* numel, int n, Plan& pl, const char* who) {
  FS2_REQUIRE(numel != nullptr && n >= 1, "%s: empty parameter table", who);
  int64_t chunks = 0;
  for (int t = 0; t < n; ++t) {
    FS2_REQUIRE(numel[t] >= 1 && numel[t] <= ((int64_t)1 << 62), "%s: entry %d has numel %lld", who, t, (long long)numel[t]);
    chunks += (numel[t] + kChunk - 1) / kChunk;
    FS2_REQUIRE(chunks <= 0x7fffffffLL, "%s: more than 2^31 - 1 chunks of %d elements", who, (int)kChunk);
  }
  pl.n_chunks = chunks;
  pl.off_entry = align256(8 * (size_t)chunks);
  pl.off_scalars = pl.off_entry + align256(8 * (size_t)n);
  pl.bytes = pl.off_scalars + align256(sizeof(Scalars));
  return FS2_OK;
}

AdamConst adam_const(const fs2_noam_adam_hp& hp) {
  // the Python scalars torch passes, rounded to fp32 by its foreach kernels: 1 - beta1, beta2, 1 - beta2, eps
  return AdamConst{(float)(1.0 - hp.beta1), (float)hp.beta2, (float)(1.0 - hp.beta2), (float)hp.eps};
}

int run(const fs2_optim_entry* table, const int64_t* numel, int n, const fs2_noam_adam_hp* hp, int clip, float max_norm,
        int64_t* noam_step, double* lr, float* norm, void* ws, size_t ws_bytes, void* stream, const char* who) {
  Plan pl;
  if (int rc = make_plan(numel, n, pl, who)) return rc;
  FS2_REQUIRE(table && hp && noam_step && lr && ws && (norm || !clip), "%s: null pointer argument", who);
  FS2_REQUIRE(((uintptr_t)ws & 255) == 0, "%s: workspace is not 256-byte aligned", who);
  FS2_REQUIRE(ws_bytes >= pl.bytes, "%s: workspace of %zu bytes, %zu needed", who, ws_bytes, pl.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  char* w = (char*)ws;
  double* partial = (double*)w;
  float2* per_entry = (float2*)(w + pl.off_entry);
  Scalars* sc = (Scalars*)(w + pl.off_scalars);
  if (clip) {
    optim_sumsq_kernel<<<(unsigned)pl.n_chunks, kThreads, 0, st>>>(table, n, partial);
    FS2_LAUNCH_CHECK();
  }
  optim_scalar_kernel<<<1, kThreads, 0, st>>>(table, n, pl.n_chunks, partial, max_norm, clip, *hp, noam_step, lr, norm,
                                             per_entry, sc);
  FS2_LAUNCH_CHECK();
  optim_update_kernel<<<(unsigned)pl.n_chunks, kThreads, 0, st>>>(table, n, per_entry, sc, adam_const(*hp));
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace
}  // namespace fs2

extern "C" {

int fs2_optim_ws_bytes(const int64_t* numel, int n, size_t* bytes) {
  fs2::Plan pl;
  if (int rc = fs2::make_plan(numel, n, pl, "fs2_optim_ws_bytes")) return rc;
  FS2_REQUIRE(bytes != nullptr, "fs2_optim_ws_bytes: null output");
  *bytes = pl.bytes;
  return FS2_OK;
}

int fs2_optim_noam_adam(const fs2_optim_entry* table, const int64_t* numel, int n, const fs2_noam_adam_hp* hp,
                        int64_t* noam_step, double* lr, void* ws, size_t ws_bytes, void* stream) {
  return fs2::run(table, numel, n, hp, 0, 0.0f, noam_step, lr, nullptr, ws, ws_bytes, stream, "fs2_optim_noam_adam");
}

int fs2_optim_clip_noam_adam(const fs2_optim_entry* table, const int64_t* numel, int n, const fs2_noam_adam_hp* hp,
                             float max_norm, int64_t* noam_step, double* lr, float* norm, void* ws, size_t ws_bytes,
                             void* stream) {
  return fs2::run(table, numel, n, hp, 1, max_norm, noam_step, lr, norm, ws, ws_bytes, stream, "fs2_optim_clip_noam_adam");
}

int fs2_optim_noam_scalars(int64_t step0, int count, const fs2_noam_adam_hp* hp, double* lr, float* step_size,
                           float* bc2_sqrt, void* stream) {
  FS2_REQUIRE(hp && lr && step_size && bc2_sqrt && step0 >= 1 && count >= 1, "fs2_optim_noam_scalars: bad argument");
  fs2::optim_noam_scalars_kernel<<<fs2::grid_for(count, 256), 256, 0, (cudaStream_t)stream>>>(step0, count, *hp, lr,
                                                                                             step_size, bc2_sqrt);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // extern "C"
