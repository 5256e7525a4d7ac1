// Shared declarations of libfs2b200.so (internal; the public ABI is include/fs2_b200.h).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <atomic>

#include "../../include/fs2_b200.h"

namespace fs2 {

void set_error(const char* fmt, ...);
extern std::atomic<unsigned long long> g_kernel_launches;  // every kernel this library enqueues (fs2_kernel_launches())

#define FS2_CUDA_CHECK(expr)                                                                   \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      fs2::set_error("%s failed at %s:%d: %s", #expr, __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return FS2_ERR_CUDA;                                                                     \
    }                                                                                          \
  } while (0)

#define FS2_LAUNCH_CHECK()                 \
  do {                                     \
    ++fs2::g_kernel_launches;              \
    FS2_CUDA_CHECK(cudaGetLastError());    \
  } while (0)

#define FS2_REQUIRE(cond, ...)      \
  do {                              \
    if (!(cond)) {                  \
      fs2::set_error(__VA_ARGS__);  \
      return FS2_ERR_INVALID;       \
    }                               \
  } while (0)

// ---- operator launchers (one per kernel family) -------------------------------------------
// All of them enqueue on `st` and return FS2_OK / error code.

enum Act { ACT_NONE = 0, ACT_RELU = 1, ACT_TANH = 2 };

// fp16 operand planes: every activation that feeds a f16 / 3xF16 contraction lives in HBM as
//   hi = rn_fp16(clamp(x * kPlaneScale)),  lo = rn_fp16(x * kPlaneScale - hi)        (lo only where a 3xF16 consumer exists)
// laid out [plane][row][K] (hi plane first, same row pitch), written by the kernel that produces x.  The power-of-two
// pre-scale moves the fp16-subnormal threshold of `lo` from |x| < 2^-3 down to |x| < 2^-7 (full 22 mantissa bits above it)
// and is undone exactly in the consuming epilogue (oscale).  Weights carry their own per-layer power-of-two scale.
constexpr float kPlaneScale = 16.0f;
constexpr float kPlaneInv = 1.0f / 16.0f;

// out[m, n] = act( sum_{j<taps} sum_{k<K} x[b, t+(j-pad)*dil, k] * w[j][n][k] + bias[n] ) (+ resid[m, n])
// x rows have stride ldx floats, time extent L per utterance (zero outside [0,L)); m = b*L + t.
struct TapGemm {
  const float* x; int ldx;      // fp32 activations (fp32 FMA and tf32 families)
  int B, L, K;
  const float* w;      // [taps][N][K]
  const float* bias;   // [N] or nullptr
  int N, taps;
  int act;
  const float* resid; int ldr;  // nullptr => none
  float* out; int ldo;          // fp32 result (may be null in the plane families when only planes are wanted)
  // q|k|v projection: output columns >= vt_col0 (the V third) are stored transposed, [b*heads + h][d][t] with row pitch
  // vt_lpad, for the attention kernel's K-major P.V operand: vt_out fp32 (tf32 family) or vtp fp16 planes
  float* vt_out = nullptr; int vt_col0 = 0, vt_dk = 0, vt_heads = 0, vt_lpad = 0;
  __half* vtp = nullptr;        // planes [P][B*heads][dk][vt_lpad], scaled by kPlaneScale
  // plane families (f16 on the hi plane; 3xF16 on hi + lo):
  const __half* xp = nullptr;   // A operand planes [P][B*L][K], row pitch K halfs
  const __half* w_hi = nullptr; const __half* w_lo = nullptr;   // weight planes, [taps][N][K], scaled by 1 / *w_inv
  const float* w_inv = nullptr; // device scalar: inverse of the weight planes' power-of-two scale (null: 1)
  float a_inv = 1.0f;           // inverse of the A planes' scale (kPlaneInv for planes written by this library)
  __half* outp = nullptr; int ldo_p = 0; bool outp_lo = false;   // result as planes [P][B*L][ldo_p] (lo plane when outp_lo)
  bool precise = false;         // 3xF16 (hi + lo operands) instead of plain f16 on the hi planes
  // per-utterance mode (FS2_PER_UTTERANCE): rows t >= lens[b] are written as exact zeros (fp32 rows and planes; the
  // transposed V third is left unwritten there), and the tensor-core kernel skips row tiles that lie wholly past lens[b]
  const int64_t* lens = nullptr;
  int dil = 1;                  // tap spacing in rows (dilated convolution); 0 (a memset TapGemm) counts as 1
};
int tap_gemm_fp32(const TapGemm& g, cudaStream_t st);
constexpr long kTapGemmFp32MaxRows = 65535L * 128;     // tap_gemm_fp32 puts row tiles of 128 on grid.y (at most 65535)
int tap_gemm_tf32(const TapGemm& g, cudaStream_t st);   // wgmma + TMA, tf32 on fp32 data (gemm_tc.cu)
int tap_gemm_planes(const TapGemm& g, cudaStream_t st); // same kernel on fp16 operand planes: f16 or 3xF16 (g.precise)
int split_f16(const float* src, __half* hi, __half* lo, long n, const float* scale /*device scalar or null*/, cudaStream_t st);
// x [rows][ldx] fp32 -> planes [2][rows][K] scaled by kPlaneScale (the one pre-pass left: LengthRegulator output, test entries)
int split_rows(const float* x, int ldx, long rows, int K, __half* planes, cudaStream_t st);
int planes_to_rows(const __half* planes, long n, float* out, cudaStream_t st);   // test helper: (hi + lo) / kPlaneScale
// power-of-two scale of a weight tensor: inv[0] = 2^-k with max|w| * 2^k in [2^13, 2^14), scale[0] = 2^k (1 for all-zero)
int weight_scale(const float* w, long n, float* scale, float* inv, cudaStream_t st);
constexpr int MATH_3XTF32 = FS2_MATH_3XTF32;            // also what the other tensor-core modes use for the encoder + predictors

constexpr size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

// bump allocator over a caller-provided buffer (null: counting only, the size needed is `off`), 256-byte aligned carves
struct Bump {
  char* base; size_t off = 0, cap;
  Bump(void* b, size_t c) : base((char*)b), cap(c) {}
  void* bytes(size_t n) { size_t a = align256(off); off = a + n; return base ? base + a : nullptr; }
  float* floats(size_t n) { return (float*)bytes(n * sizeof(float)); }
  double* doubles(size_t n) { return (double*)bytes(n * sizeof(double)); }
  // FS2_ERR_WORKSPACE (error "<who>: workspace too small") when the carves overran the buffer
  int check(const char* who) const {
    if (base == nullptr || off <= cap) return FS2_OK;
    set_error("%s: workspace too small (%zu < %zu)", who, cap, off);
    return FS2_ERR_WORKSPACE;
  }
};

// blocks of a grid-stride launch over n items: ceil(n / block), at least 1 and at most cap
inline int grid_for(long n, int block, int cap = 132 * 8) {
  long g = (n + block - 1) / block;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// Row LayerNorm with the fusions the path needs.
struct RowNorm {
  const float* x; int ldx;        // [rows, C]
  const float* resid; int ldr;    // optional, added before the statistics
  const float* gamma; const float* beta; float eps;
  int64_t rows; int C;            // C in {256, 384}
  float* out; int ldo;            // optional (nullptr when only the head is wanted)
  int relu_after;                 // y = relu(LN(.))   (decoder input layer, core/encoder.py:118-125)
  const float* pe; const float* alpha; int L;  // optional: y += alpha * pe[t], t = row % L
  // optional scalar head (predictors): s = y . head_w + head_b, 0 where t >= lens[b]
  const float* head_w; const float* head_b; float* head_out; int64_t* dur_out;
  const float* head_scale;        // optional [rows]: head_out[row] = fp32(s * head_scale[row]), one rounding (prosody control)
  const int64_t* lens;            // optional mask (needs L > 0): rows t >= lens[b] write 0 to the head, out and split_out
  __half* split_out;              // optional operand planes of y (scaled by kPlaneScale): hi at [row][C], lo at [rows + row][C]
  int split_lo;                   // write the lo plane too (3xF16 consumer)
  // optional speaker table (the last encoder LayerNorm of a multi-speaker model): y += spk_table[spk[row / spk_L]], one
  // fp32 add after gamma / beta, before out, split_out and the head.  An id outside [0, n_spk) adds nothing; masked rows
  // (lens) still write 0
  const float* spk_table; const int64_t* spk; int n_spk; int spk_L;
  // optional per-utterance vector (projected external speaker embeddings, DESIGN.md section 27): y += spk_vec[row / spk_L],
  // one more fp32 add after the table's, so y = (LN + E[spk]) + v; needs spk_L > 0
  const float* spk_vec;
};
int row_norm(const RowNorm& r, cudaStream_t st);
// v [B, A] = W [A, D] . normalize(e [B, D]) + bias (spembs.cu); en [B, D] (nullable) receives the normalised embeddings,
// bad [B] (nullable) 1 where e_b holds a non-finite value or its sum of squares overflows fp32, else 0; status (nullable)
// |= FS2_SPEMB_NONFINITE then
int spemb_project(const float* W, const float* bias, const float* e, int B, int D, int A, float* v, float* en, int32_t* bad,
                  int32_t* status, cudaStream_t st);

// lens (nullable): rows t >= lens[b] are written as zeros (per-utterance mode)
int embed_posenc(const int64_t* xs, const float* table, int n_sym, const float* pe, const float* alpha, int B, int T,
                 int C, float* out, __half* planes /*nullable: hi + lo*/, const int64_t* lens, cudaStream_t st);

int bucketize(const float* vals, const float* bins, int n_edges, int64_t n, int64_t* ids, cudaStream_t st);
int one_hot(const int64_t* ids, int64_t n, int n_bins, float* out, cudaStream_t st);
// out[r,:] = (hm[r,:] + (p_tab[p_id[r]] + p_bias)) + (e_tab[e_id[r]] + e_bias); ids from values (nullable id outs).
// lens (nullable, rows = B * L): frames t >= lens[b] get zero rows and id -1 (an all-zero one-hot)
int variance_embed_add(const float* hm, const float* e_val, const float* p_val, const float* e_bins, const float* p_bins,
                       int n_edges, const float* e_tab, const float* e_bias, const float* p_tab, const float* p_bias,
                       int64_t rows, int C, float* out, __half* planes /*nullable: hi (+ lo)*/, int planes_lo, int64_t* e_ids,
                       int64_t* p_ids, const int64_t* lens, int L, cudaStream_t st);

int attention_fp32(const float* qkv, const int64_t* lens, int B, int L, int C, int heads, float* ctx, cudaStream_t st);
// tensor-core attention: q, k from qkv [B,L,3C]; v from the transposed buffer vt [B*heads, dk, lpad]
int attention_tf32(const float* qkv, const float* vt, int lpad, const int64_t* lens, int B, int L, int C, int heads,
                   float* ctx, cudaStream_t st);

// fp16-plane attention (attention_f16.cu): q, k from planes qkp [P][B*L][2C], v from vtp [P][B*heads][dk][lpad] (all scaled
// by kPlaneScale); x3 = error-compensated (hi + lo planes, three f16 products per term), else f16 on the hi planes.
// Result: ctx fp32 [B,L,C] (nullable) and / or ctxp planes [P][B*L][C] (nullable; lo plane when x3)
int attention_planes(const __half* qkp, const __half* vtp, int lpad, const int64_t* lens, int B, int L, int C, int heads, bool x3,
                     float* ctx, __half* ctxp, cudaStream_t st);
// test helper: qkv fp32 [B,L,3C] -> qkp / vtp planes
int qkv_to_planes(const float* qkv, int B, int L, int C, int heads, __half* qkp, __half* vtp, int lpad, cudaStream_t st);
// vt[(b*heads + h)*dk + d][t] = qkv[b, t, 2C + h*dk + d]   (test helper for the single-operator entry)
int transpose_v(const float* qkv, int B, int L, int C, int heads, float* vt, int lpad, cudaStream_t st);

// alpha_v (nullable): per-phoneme factors [B, T] in place of the scalar alpha; d_used (nullable): [B, T] frame counts expanded
int length_plan(void* ds, int ds_dtype, const int64_t* ilens, float alpha, const float* alpha_v, int B, int T, int mutate,
                int32_t* cum, int64_t* olens, int64_t* stats, int64_t* d_used, cudaStream_t st);
// spk (nullable) [B]: a non-empty slot whose id lies outside [0, n_spk) is emptied and sets FS2_PLAN_BAD_SPEAKER;
// spemb_bad (nullable) [B]: a non-empty slot with spemb_bad[b] != 0 is emptied and sets FS2_SPEMB_NONFINITE
int length_plan_cap(const void* ds, int ds_dtype, const int64_t* ilens, const float* alpha_v, const float* fac, const int64_t* spk,
                    int n_spk, const int32_t* spemb_bad, int B, int T, long Lc, int32_t* cum, int64_t* olens, int64_t* need, int64_t* d_used, int* status,
                    cudaStream_t st);
int synth_status(const int* plan, const int* voc, const int64_t* olens, int B, int hop, int* word, int64_t* alens, cudaStream_t st);
int length_gather(const float* hs, const int32_t* cum, const int64_t* ilens, int B, int T, int C, float* out, int Lcap,
                  const float* fac_in, float* fac_out, cudaStream_t st);

int masked_losses(const float* before, const float* after, const float* ys, int ld_ys_time, const float* d_out,
                  const void* ds, int ds_dtype, const float* e_out, const float* p_out, const float* es, const float* ps,
                  const int64_t* ilens, const int64_t* olens, int B, int T, int L, int odim, float* out7, void* scratch,
                  cudaStream_t st);

// ---- deterministic train mode (DESIGN.md section 26): ordered sums, no floating-point atomics ----
// dw[n][k][j] += sum over q < splits, in ascending q, of part[q][j][n][k] (wgrad_tc.cu); taps = N = 1 sums rows of [splits][K]
int ordered_reduce(const float* part, int splits, int taps, int N, int K, float* dw, cudaStream_t st);
// out[k] = sum_{i < n} part[k * sk + i * si], k < K, in double, in a fixed order (train.cu)
int ordered_sum_f64(const double* part, long n, long si, long sk, int K, double* out, cudaStream_t st);
// workspace of masked_losses_det and its carve (train.cu)
size_t loss_det_ws_bytes(int B, int T, int L, int odim);
int loss_det_carve(void* ws, int B, int T, int L, int odim, double** acc, double** mel, long* n_mel, double** seq, long* n_seq);
int masked_losses_det(const float* before, const float* after, const float* ys, int ld_ys_time, const float* d_out,
                      const void* ds, int ds_dtype, const float* e_out, const float* p_out, const float* es, const float* ps,
                      const int64_t* ilens, const int64_t* olens, int B, int T, int L, int odim, float* out7, void* ws,
                      cudaStream_t st);
// the bodies of the ordered train entries (train.cu); the C entries with their argument checks are in train_det.cu
size_t colsum_det_bytes(long rows, int C);
int colsum_det(const float* x, long rows, int C, float* out, void* ws, cudaStream_t st);
size_t conv_wgrad_det_bytes(int B, int L, int N, int K, int taps, bool bias);
int conv_wgrad_det(const float* dy, const float* x, int B, int L, int N, int K, int taps, float* dw, float* dbias, void* ws, cudaStream_t st);
size_t layernorm_backward_det_bytes(long rows, int C);
int layernorm_backward_det(const float* x, const float* dy, const float* gamma, float eps, long rows, int C, float* dx, float* dgamma,
                           float* dbeta, void* ws, cudaStream_t st);
size_t batchnorm_det_bytes(long rows, int C);
int batchnorm_train_det(const float* x, long rows, int C, const float* gamma, const float* beta, float eps, float momentum, int act,
                        float* running_mean, float* running_var, float* stats, float* y, void* ws, cudaStream_t st);
int batchnorm_backward_det(const float* x, const float* dy, const float* stats, const float* gamma, float eps, long rows, int C, float* dx,
                           float* dgamma, float* dbeta, void* ws, cudaStream_t st);
size_t embed_backward_det_bytes(long rows, int C, int n_sym, bool table);
int embed_backward_det(const int64_t* xs, const float* dy, const float* pe, int B, int T, int C, int n_sym, float* dtable, float* dalpha,
                       void* ws, cudaStream_t st);
size_t onehot_linear_backward_det_bytes(long rows, int C, int n_bins, bool bias);
int onehot_linear_backward_det(const int64_t* ids, const float* dy, long rows, int C, int n_bins, float* dW, float* dbias, void* ws,
                               cudaStream_t st);
size_t rowdot_backward_det_bytes(long rows, int C);
int rowdot_backward_det(const float* x, const float* w, const float* dy, const int64_t* lens, long rows, int L, int C, float* dx, float* dw,
                        float* dbias, void* ws, cudaStream_t st);
int scatter_max_ids();   // largest id range (n_sym, n_bins) of the ordered scatter

// weight repacking helpers (pack.cu)
int pack_conv_weight(const float* src, int N, int K, int taps, const float* scale /*[N] or null*/, float* dst,
                     cudaStream_t st);  // src [N][K][taps] -> dst [taps][N][K] * scale[n]
int pack_transpose(const float* src, int rows, int cols, float* dst, cudaStream_t st);  // [rows][cols] -> [cols][rows]
int fold_batchnorm(const float* gamma, const float* beta, const float* mean, const float* var, float eps, int N,
                   float* scale, float* shift, cudaStream_t st);

// ---- programmatic dependent launch (experiment, FS2_PDL=1; off by default) ---------------------
// Every kernel of the step calls pdl_wait() before its first global-memory access (= the previous grid has completed and its
// writes are visible) and pdl_trigger() once its work is done (the persistent tensor-core GEMM) or first thing (the short
// row-wise kernels), so that the launch latency, mbarrier init and tensor-map fetch of kernel k+1 overlap the
// tail of kernel k.  Correct (tools/pdl_check.py: 30 graph replays per mode bit-identical to the eager step; the whole GPU
// suite passes with it) but no gain inside the CUDA graph: with the trigger at kernel start 6.41 / 6.46 ms per c2 step against
// 6.30 / 6.22 without (alternating runs on one box, profiles/r02_bench_r2j_pdl*.json); with the trigger at the end 6.68 / 6.59
// against 6.83 / 6.55 (gpurun_out/bench_h2_pdl*.json) -- inside the noise.  Without the launch attribute the calls are no-ops.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
inline bool pdl_enabled() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("FS2_PDL"); v = e ? atoi(e) : 0; }
  return v != 0;
}
// kernel<<<grid, block, smem, st>>>(args...) with the programmatic-stream-serialization attribute; ONLY for kernels that call
// pdl_wait() before touching global memory
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// SMs of the current device (persistent grids: one CTA per SM)
inline int sm_count_current() {
  static int cached[64];
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (!cached[dev]) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

// ---- small device helpers -----------------------------------------------------------------
// two floats -> packed fp16 pair (a in the low half), round-to-nearest, saturating at +-65504 (F2FP.SATFINITE: one instruction
// instead of four FMNMX clamps + the pack; the epilogues that write operand planes are instruction-latency bound)
__device__ __forceinline__ uint32_t pack_f16x2_sat(float a, float b) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
// two fp32 values -> packed fp16 hi pair and lo pair of (v * kPlaneScale)
__device__ __forceinline__ void split_pair(float a, float b, uint32_t& hi, uint32_t& lo) {
  a *= kPlaneScale; b *= kPlaneScale;
  hi = pack_f16x2_sat(a, b);
  const float2 g = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  lo = pack_f16x2_sat(a - g.x, b - g.y);        // beyond the fp16 range hi saturates and lo carries (saturating) what it can of the rest
}
__device__ __forceinline__ uint32_t hi_pair(float a, float b) { return pack_f16x2_sat(a * kPlaneScale, b * kPlaneScale); }
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// Philox4x32-10 counter-based generator (dropout masks, Griffin-Lim initial phases): the output depends only on
// (counter, key), so any element can be redrawn without stored state
__device__ __forceinline__ uint4 philox4x32(uint4 ctr, uint2 key) {
  const unsigned M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const unsigned hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x, hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0; key.y += W1;
  }
  return ctr;
}
// torch.bucketize(right=False): first i with !(bins[i] < x) ... written as torch does so NaN -> n_edges
__device__ __forceinline__ int bucket_of(float x, const float* __restrict__ bins, int n_edges) {
  int lo = 0, hi = n_edges;
  while (lo < hi) {
    int mid = lo + ((hi - lo) >> 1);
    if (!(bins[mid] >= x)) lo = mid + 1; else hi = mid;
  }
  return lo;
}

}  // namespace fs2
