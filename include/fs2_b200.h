/*
 * fs2_b200.h -- C ABI of libfs2b200.so, the sm_90a FastSpeech2 mel-synthesis forward path.
 *
 * The reference (rishikksh20/FastSpeech2) has no FFI layer: its operator API for this
 * path is the Python class `FeedForwardTransformer` in fastspeech.py, whose stages call
 * torch.nn modules.  Each entry point below replaces one stage of
 * `FeedForwardTransformer._forward` (fastspeech.py:169-243) / `forward` (:245-337); the
 * reference lines a function replaces are cited at its declaration.  The Python class in
 * fastspeech2_b200/fastspeech.py binds these with ctypes (INTEGRATION.md shows the stub).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no torch / C++ types in signatures.
 *   - every function returns 0 on success or a negative FS2_ERR_* code;
 *     fs2_last_error() returns a thread-local message for the last failure.
 *   - all tensor pointers are DEVICE pointers (fp32 row-major [batch, time, channel],
 *     lengths / ids / durations int64) unless a parameter says "host".
 *   - the caller owns every input, output and workspace buffer; the library owns only the
 *     opaque handle (packed weights, TMA descriptors, launch plans).
 *   - all work is enqueued on the `stream` argument (a cudaStream_t passed as void*);
 *     no function synchronises the device.  fs2_length_plan writes its two result words to
 *     device memory; the caller reads them back (that is the path's single host sync).
 *   - a handle is bound to one device and is not thread-safe; entry points that take a handle select its device for
 *     the call and restore the caller's.  Handle-less entry points (LengthRegulator, losses, single operators, train /
 *     STFT / peer kernels) run on the CURRENT device like any CUDA library call: select the device your buffers live on.
 */
#ifndef FS2_H100_H_
#define FS2_H100_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FS2_OK 0
#define FS2_ERR_INVALID (-1)        /* bad argument / unsupported shape            */
#define FS2_ERR_CUDA (-2)           /* a CUDA runtime / driver call failed         */
#define FS2_ERR_MISSING_WEIGHT (-3) /* fs2_load_weights: a required key is absent  */
#define FS2_ERR_WORKSPACE (-4)      /* workspace too small                         */
#define FS2_ERR_NOT_LOADED (-5)     /* stage called before fs2_load_weights        */

/* duration dtypes accepted by the length regulator (tests/test_fastspeech2.py:17 feeds floats) */
#define FS2_DUR_I64 0
#define FS2_DUR_F32 1
#define FS2_DUR_I32 2

/* arithmetic of the dense contractions (accumulation is fp32 in registers everywhere).
 *   FS2_MATH_FP32: fp32 FMA on CUDA cores everywhere.
 *   FS2_MATH_3XTF32 ("3xf16", the reference-precision tensor-core mode and the Python class's default): every dense
 *     contraction -- projections, convolutions AND both attention products -- error-compensated on tensor-core: each operand
 *     is held as two fp16 planes hi = rn(s x), lo = rn(s x - hi) (s an exact power of two, undone in the epilogue), and
 *     a product is accumulated as hi.hi + hi.lo + lo.hi.  fp32-class results (max-abs ~1e-5 on the mels).
 *   FS2_MATH_F16: encoder + predictors as in FS2_MATH_3XTF32 (their outputs feed round() / bucketize()); the decoder
 *     side (input Linear, q|k|v, attention, out-projection, conv-FFN, mel Linear, Postnet) on f16 over the hi
 *     planes only: 10-bit-mantissa operands (like tf32, round-to-nearest), twice the tf32 MMA rate.
 *   FS2_MATH_TF32: encoder + predictors as above; decoder side on tf32 reading the fp32 rows directly.
 * Normalisation, softmax statistics, gathers and every integer kernel are fp32 / exact in all modes. */
#define FS2_MATH_FP32 0
#define FS2_MATH_TF32 1
#define FS2_MATH_3XTF32 2
#define FS2_MATH_F16 3

typedef struct fs2_handle fs2_handle;

/* Shapes of the network: the subset of `hp` read by FeedForwardTransformer.__init__
 * (fastspeech.py:37-160; values in configs/default.yaml:38-106). */
typedef struct fs2_config {
  int32_t idim, odim;               /* 68 symbols, 80 mel bins                            */
  int32_t adim, aheads, elayers, eunits;   /* encoder: 256, 2, 4, 1024                    */
  int32_t ddim, dlayers, dunits;           /* decoder: 384, 4, 1024 (heads shared)        */
  int32_t ffn_kernel;               /* positionwise_conv_kernel_size: 9                   */
  int32_t pred_layers, pred_chans, pred_kernel; /* 2, 256, 3                              */
  int32_t postnet_layers, postnet_chans, postnet_filts; /* 5, 256, 5                      */
  int32_t n_bins;                   /* 256 pitch / energy buckets                         */
  int32_t pe_len;                   /* informational: the positional tables' row counts are read off the tensors at load time */
  int32_t math_mode;                /* FS2_MATH_*                                         */
} fs2_config;

/* One checkpoint tensor, addressed by its reference state_dict key. */
typedef struct fs2_weight_desc {
  const char* name;     /* e.g. "decoder.encoders_.0.feed_forward.w_1.weight"  */
  const void* data;     /* device pointer, contiguous                           */
  int32_t ndim;
  int64_t shape[4];
  int32_t dtype;        /* 0 = float32, 1 = int64                               */
} fs2_weight_desc;

const char* fs2_last_error(void);
/* "fs2-b200 <ver> sm_90a" ; lets the binding check it loaded the right library */
const char* fs2_version(void);
/* number of kernels this library has enqueued in this process (bench.py reports the per-step delta) */
unsigned long long fs2_kernel_launches(void);

/* ---- handle --------------------------------------------------------------------------- */
/* replaces FeedForwardTransformer.__init__ shape plumbing (fastspeech.py:37-160) */
int fs2_create(fs2_handle** out, const fs2_config* cfg, int device);
void fs2_destroy(fs2_handle* h);
int fs2_set_math_mode(fs2_handle* h, int math_mode);

/* Repack the checkpoint into kernel layout: Conv1d [N,K,taps] -> [taps][N][K]; q/k/v Linear
 * concatenated; BatchNorm1d (eval) folded into the Postnet convolutions
 * (core/modules.py:283-348); pitch/energy embedding Linear transposed to a [bin][channel]
 * table.  Replaces load_state_dict -> module attribute reads of the reference. */
int fs2_load_weights(fs2_handle* h, const fs2_weight_desc* w, int n, void* stream);

/* Bytes of scratch the two big stages need (max of both) for a batch of B utterances,
 * Tmax phonemes and Lmax frames. */
int fs2_workspace_bytes(fs2_handle* h, int B, int Tmax, int Lmax, size_t* out);

/* ---- per-kernel-class CUDA-event profiler (used by bench.py for the roofline; off by default) -
 * While enabled, every kernel the stage functions enqueue is bracketed by two events on the
 * launch stream.  fs2_profile_read synchronises those events, sums elapsed ms / launches /
 * algorithmic FLOPs / algorithmic bytes per class into arrays of fs2_profile_classes()
 * entries, and clears the records. */
int fs2_profile_enable(fs2_handle* h, int on);
int fs2_profile_classes(void);
const char* fs2_profile_label(int cls);
int fs2_profile_read(fs2_handle* h, double* ms, int64_t* launches, double* flop, double* bytes);

/* ---- stage 1: phoneme encoder + duration predictor ------------------------------------- */
/* fastspeech.py:180-193,210: _source_mask, encoder (core/encoder.py:185-204 ->
 * attention.py:30-74, modules.py:237-248), duration_predictor (duration_predictor.py:64-86).
 *   xs [B,Tmax] i64 (0 = pad), ilens [B] i64
 *   hs [B,Tmax,adim] f32 out
 *   d_log [B,Tmax] f32 out (log-domain prediction, 0 at pads)           -- may be NULL
 *   d_int [B,Tmax] i64 out (clamp(round(exp(x)-1),0), 0 at pads)        -- may be NULL */
int fs2_encode(fs2_handle* h, const int64_t* xs, const int64_t* ilens, int B, int Tmax, float* hs, float* d_log,
               int64_t* d_int, void* ws, size_t ws_bytes, void* stream);

/* Per-utterance batching (flags of fs2_encode_ex / fs2_decode_ex).  Without it a batch reproduces the reference's
 * semantics, under which an utterance's result depends on its batch mates: the convolutions read the padded positions
 * (non-zero after the first block) and inference runs the decoder unmasked.  With it, every tensor a convolution reads
 * and every output holds exact zeros at rows t >= len_b (len = ilens in the encoder, olens in the decoder), so utterance b
 * of a batch is bit-identical to the same utterance run alone (B = 1, Tmax = ilens[b], L = olens[b]) in every math mode,
 * and row tiles wholly in padding are skipped. */
#define FS2_PER_UTTERANCE 1

/* fs2_encode with flags (0 or FS2_PER_UTTERANCE); fs2_encode is the flags = 0 case.  With FS2_PER_UTTERANCE,
 * hs[b, t >= ilens[b], :] == 0 (d_log / d_int are 0 there in either mode). */
int fs2_encode_ex(fs2_handle* h, const int64_t* xs, const int64_t* ilens, int B, int Tmax, float* hs, float* d_log,
                  int64_t* d_int, void* ws, size_t ws_bytes, int flags, void* stream);

/* ---- stage 2: LengthRegulator (needs no handle) ---------------------------------------- */
/* core/duration_modeling/length_regulator.py:38-95 + utils/util.py:91-104.
 * Plan: per utterance, optionally scale by alpha (round half to even, :58-59), truncate to
 * ilens (:60-61), apply the all-zero -> all-one rule (:86-88; written back into `ds` when
 * mutate_ds != 0, which mirrors the reference's in-place fill_ for alpha == 1), inclusive
 * prefix sum.
 *   ds [B,Tmax] of ds_dtype; cum [B,Tmax] i32 out; olens [B] i64 out
 *   stats [2] i64 out (device): stats[0] = max_b olens[b], stats[1] = #negative durations */
int fs2_length_plan(void* ds, int ds_dtype, const int64_t* ilens, float alpha, int B, int Tmax, int mutate_ds,
                    int32_t* cum, int64_t* olens, int64_t* stats, void* stream);
/* Gather: out[b,j,:] = hs[b, min{i: cum[b,i] > j}, :] for j < olens[b], 0 for the rest of
 * [0,Lcap).  Bit-exact copy.  hs [B,Tmax,C], out [B,Lcap,C]; C % 4 == 0. */
int fs2_length_gather(const float* hs, const int32_t* cum, const int64_t* ilens, int B, int Tmax, int C, float* out,
                      int Lcap, void* stream);

/* Prosody control (speed).  fs2_length_plan with one duration factor per phoneme; fs2_length_plan is the case
 * alpha_v = d_used = NULL.  The reference scales by one scalar, torch.round(ds.float() * alpha).long()
 * (length_regulator.py:57-59); here
 *   alpha_v [B,Tmax] f32 or NULL: d'[b,t] = rint_half_even(fp32(d) * alpha_v[b,t]) (one fp32 rounding before the
 *           rint), in place of the scalar alpha (which must then be 1).  The all-zero -> all-one rule (:86-88) is
 *           evaluated on the scaled slice.  Requires mutate_ds == 0: the caller's ds are never written.
 *   d_used  [B,Tmax] i64 out or NULL: the frame counts the gather expands (scaled, all-zero rule applied, 0 past ilens).
 * A total frame count that does not fit the int32 prefix sum is reported, not wrapped: olens[b] and stats[0] hold the
 * true total (at least 2^31), and the caller must refuse to gather from such a plan. */
int fs2_length_plan_ex(void* ds, int ds_dtype, const int64_t* ilens, float alpha, const float* alpha_v, int B, int Tmax,
                       int mutate_ds, int32_t* cum, int64_t* olens, int64_t* stats, int64_t* d_used, void* stream);
/* fs2_length_gather with a side output for the pitch / energy controls; fs2_length_gather is fac_in = fac_out = NULL.
 *   fac_in  [2][B,Tmax] f32: per-phoneme factors (plane 0 energy, plane 1 pitch, say; the kernel does not care)
 *   fac_out [2][B,Lcap] f32 out: fac_out[k][b,j] = fac_in[k][b, min{i: cum[b,i] > j}] for j < olens[b], 1.0 for the rest
 * Both or neither. */
int fs2_length_gather_ex(const float* hs, const int32_t* cum, const int64_t* ilens, int B, int Tmax, int C, float* out,
                         int Lcap, const float* fac_in, float* fac_out, void* stream);

/* Capacity plan (synthesis replayed from a CUDA graph at a fixed frame capacity Lc, DESIGN.md section 21): the scan of
 * fs2_length_plan_ex with mutate_ds = 0 and alpha = 1, sized by Lc instead of by a host read, and nothing read back.
 *   ds, ds_dtype, ilens, alpha_v, d_used: as in fs2_length_plan_ex (alpha_v may be NULL)
 *   fac     [2][B,Tmax] f32 or NULL: the pitch / energy factors (fs2_length_gather_ex's fac_in), checked like alpha_v
 *   need    [B] i64 out: the frames slot b plans, computed exactly as fs2_length_plan_ex's olens (speed, all-zero rule)
 *   olens   [B] i64 out: need[b] when 1 <= ilens[b] <= Tmax, need[b] <= Lc and the slot's factors are valid; else 0
 *   cum     [B,Tmax] i32 out: fs2_length_plan_ex's where olens[b] = need[b], all zeros where olens[b] = 0, so that
 *           fs2_length_gather_ex into Lc rows writes such a slot as zeros; d_used is likewise 0 there
 *   status  one i32 (device) out, zeroed by the call, then the OR of
 *     FS2_PLAN_BAD_ILENS    some ilens[b] outside [0, Tmax];
 *     FS2_PLAN_BAD_CONTROL  a factor of alpha_v or fac at t < ilens[b] is non-finite or <= 0;
 *     FS2_PLAN_OVERFLOW     some need[b] > Lc (informational: that slot is skipped, need says what would fit it).
 * ilens[b] == 0 marks an empty slot: need and olens 0, no bit.  Needs B, Tmax, Lc >= 1 and Lc <= INT32_MAX (cum is
 * int32). */
#define FS2_PLAN_BAD_ILENS 1
#define FS2_PLAN_BAD_CONTROL 2
#define FS2_PLAN_OVERFLOW 4
int fs2_length_plan_cap(const void* ds, int ds_dtype, const int64_t* ilens, const float* alpha_v, const float* fac, int B,
                        int Tmax, int64_t Lc, int32_t* cum, int64_t* olens, int64_t* need, int64_t* d_used, int32_t* status,
                        void* stream);
/* The status word of one graphed synthesis: *word = *plan_status | (vocoder bits << FS2_SYNTH_VOC_SHIFT), where the
 * vocoder's bits are *voc_status (NULL: none) without its BAD_LENGTH bit when some olens[b] is 0 (an empty, overflowed or
 * refused slot, which the vocoder reports as a bad length by design).  alens [B] i64 out or NULL: olens[b] * hop.
 * Every vocoder's status word has BAD_LENGTH = 1 and RANGE = 2. */
#define FS2_SYNTH_VOC_SHIFT 8
int fs2_synth_status(const int32_t* plan_status, const int32_t* voc_status, const int64_t* olens, int B, int hop,
                     int32_t* word, int64_t* alens, void* stream);

/* ---- stage 3: variance adaptor + mel decoder + Postnet --------------------------------- */
/* fastspeech.py:195-238.
 *   hm [B,L,adim] f32: length-regulated encoder states (read only)
 *   olens [B] i64 or NULL.  NULL reproduces is_inference=True: decoder unmasked
 *         (fastspeech.py:221-224) and e_out / p_out unmasked.
 *   es, ps [B,L] f32 or NULL.  NULL => bucketize the predictors' own outputs (:195-196),
 *         else bucketize the given values (:200-206).
 *   before, after [B,L,odim] f32 out; e_out, p_out [B,L] f32 out (predictor values)
 *   e_ids, p_ids [B,L] i64 out (bucket indices actually embedded) -- may be NULL */
int fs2_decode(fs2_handle* h, const float* hm, const int64_t* olens, const float* es, const float* ps, int B, int L,
               float* before, float* after, float* e_out, float* p_out, int64_t* e_ids, int64_t* p_ids, void* ws,
               size_t ws_bytes, void* stream);

/* fs2_decode with flags (0 or FS2_PER_UTTERANCE); fs2_decode is the flags = 0 case.  With FS2_PER_UTTERANCE, olens is
 * required also when es / ps are NULL (predict-and-bucketize: pass the lengths of the length plan), hm must be zero at
 * rows t >= olens[b] (fs2_length_gather writes it so), and at those rows before / after / e_out / p_out are 0 and
 * e_ids / p_ids are -1 (an all-zero one-hot). */
int fs2_decode_ex(fs2_handle* h, const float* hm, const int64_t* olens, const float* es, const float* ps, int B, int L,
                  float* before, float* after, float* e_out, float* p_out, int64_t* e_ids, int64_t* p_ids, void* ws,
                  size_t ws_bytes, int flags, void* stream);

/* Prosody control (pitch, energy).  fs2_decode_ex with per-frame factors on the predicted values; fs2_decode_ex is the
 * case e_scale = p_scale = NULL.  The reference's EnergyPredictor / PitchPredictor.inference(xs, alpha) return
 * `xs * alpha` before bucketize (variance_predictor.py:58,140-152,213-225); here
 *   e_scale, p_scale [B,L] f32 or NULL (each independently): e_out[b,t] = fp32(e[b,t] * e_scale[b,t]), one fp32
 *           rounding, no FMA; likewise p_out.  e_ids / p_ids and the decoder input bucketize the scaled values.
 * Predict mode only: a scale together with es / ps returns FS2_ERR_INVALID.  Valid with flags 0 and FS2_PER_UTTERANCE;
 * fs2_length_gather_ex expands per-phoneme factors into this layout. */
int fs2_decode_ctl(fs2_handle* h, const float* hm, const int64_t* olens, const float* es, const float* ps, int B, int L,
                   float* before, float* after, float* e_out, float* p_out, int64_t* e_ids, int64_t* p_ids,
                   const float* e_scale, const float* p_scale, void* ws, size_t ws_bytes, int flags, void* stream);

/* ---- stage 4: masked losses (fastspeech.py:277-333) ------------------------------------- */
/* out7 (device, f32): l1, before, after, duration, energy, pitch, total -- the order of
 * report_keys (fastspeech.py:325-333).  use_masking=True, use_weighted_masking=False.
 * scratch: >= 64 bytes of device memory (zeroed by the call). */
int fs2_masked_losses(const float* before, const float* after, const float* ys, int ld_ys_time, const float* d_out,
                      const void* ds, int ds_dtype, const float* e_out, const float* p_out, const float* es,
                      const float* ps, const int64_t* ilens, const int64_t* olens, int B, int Tmax, int L, int odim,
                      float* out7, void* scratch, void* stream);

/* ---- single operators (used by the per-kernel parity tests; same kernels as the stages) - */
/* variance_predictor.py:154-159,227-232 + fastspeech.py:218-219 */
int fs2_bucketize(const float* vals, const float* bins, int n_edges, int64_t n, int64_t* ids, void* stream);
/* F.one_hot(ids, n_bins).float(): the 4th/5th return value of _forward(is_inference=True) */
int fs2_one_hot(const int64_t* ids, int64_t n, int n_bins, float* out, void* stream);
/* out[b,t,:] = act(sum_j x[b,t+j-pad,:] . W[j] + bias) (+ resid); W [taps][N][K].
 * math_mode selects the kernel family: FS2_MATH_FP32 (CUDA cores), FS2_MATH_TF32 (tf32), FS2_MATH_3XTF32 (the
 * error-compensated tensor-core family) or FS2_MATH_F16 (f16); the last two run on fp16 operand planes of x and
 * w made on the fly here (inside a stage the producing kernel writes them).
 * act: 0 none, 1 relu, 2 tanh */
int fs2_op_tap_gemm(int math_mode, const float* x, int B, int L, int K, const float* w, const float* bias, int N, int taps,
                    int act, const float* resid, float* out, void* stream);
/* fs2_op_tap_gemm with the rest of the kernel's epilogue; fs2_op_tap_gemm is this call with every new argument NULL / 0.
 *   lens [B] i64 (device) or NULL: per-utterance mode, as in the FS2_PER_UTTERANCE stages.  Rows t >= lens[b] are written
 *        as exact zeros (out and planes), and the tensor-core families skip the MMAs of 128-row tiles wholly past
 *        lens[b].  Values lie in [0, L]; a convolution's (taps > 1) input must hold zeros at rows t >= lens[b].
 *   out  may be NULL in FS2_MATH_F16 / FS2_MATH_3XTF32 when out_planes or vt is given.
 *   out_planes (FS2_MATH_F16 / FS2_MATH_3XTF32 only) fp16 [P][B*L][N], P = 2 in FS2_MATH_3XTF32 (hi, lo) and 1 in
 *        FS2_MATH_F16 (hi): the result as the operand planes of a next contraction, scaled by 16.
 *   vt   (tensor-core families only) with vt_col0, vt_heads, vt_lpad: columns >= vt_col0 (the V third of a q|k|v
 *        projection) get the bias only and are stored transposed, vt[(b*vt_heads + h)*dk + d][t] with
 *        h*dk + d = n - vt_col0, dk = (N - vt_col0) / vt_heads and row pitch vt_lpad >= L, instead of in out /
 *        out_planes; entries at t >= lens[b] and t >= L are not written.  FS2_MATH_TF32: fp32 [B*vt_heads][dk][vt_lpad];
 *        the plane families: fp16 planes [P][B*vt_heads][dk][vt_lpad] scaled by 16 (vt_lpad % 8 == 0, dk % 32 == 0).
 *        vt_col0 must be a multiple of the kernel's tile width (the largest of 128, 80, 64, 32, 16 dividing N).
 * FS2_MATH_FP32 accepts lens and rejects out_planes and vt with FS2_ERR_INVALID. */
int fs2_op_tap_gemm_ex(int math_mode, const float* x, int B, int L, int K, const float* w, const float* bias, int N,
                       int taps, int act, const float* resid, const int64_t* lens, float* out, void* out_planes,
                       int vt_col0, int vt_heads, void* vt, int vt_lpad, void* stream);
/* fs2_op_tap_gemm_ex with dilated taps: tap j reads row t + (j - pad) * dil of the same utterance (zero outside [0, L)),
 * the layout of nn.Conv1d(dilation = dil, padding = pad * dil).  dil >= 1, and dil * pad + L < 2^30 when dil > 1
 * (FS2_ERR_INVALID otherwise); fs2_op_tap_gemm_ex is the case dil = 1. */
int fs2_op_tap_gemm_dil(int math_mode, const float* x, int B, int L, int K, const float* w, const float* bias, int N,
                        int taps, int act, const float* resid, const int64_t* lens, float* out, void* out_planes,
                        int vt_col0, int vt_heads, void* vt, int vt_lpad, int dil, void* stream);
/* out = LayerNorm_N(x . w^T + bias + resid) * gamma + beta as a tensor-core GEMM followed by the row LayerNorm kernel (x [rows,K], w [N,K]);
 * the form of core/encoder.py:60-62 / :67-69: FS2_MATH_TF32 (tf32 on the fp32 rows, N = 384),
 * FS2_MATH_F16 (f16) and FS2_MATH_3XTF32 (error-compensated 3xF16) on operand planes made on the fly here,
 * N in {256, 384}.
 * out_planes (nullable, plane families): the operand planes the kernel writes for the next contraction, returned
 * recombined as fp32 [rows,N] = (hi + lo) / scale (hi only in FS2_MATH_F16) */
int fs2_op_gemm_layernorm(int math_mode, const float* x, int64_t rows, int K, int N, const float* w, const float* bias,
                          const float* resid, const float* gamma, const float* beta, float eps, float* out,
                          float* out_planes, void* stream);
/* qkv [B,L,3C] (q | k | v, heads contiguous inside each) -> ctx [B,L,C]; lens NULL => no mask.  FS2_MATH_FP32: CUDA cores;
 * FS2_MATH_TF32: tensor-core tf32; FS2_MATH_F16 / FS2_MATH_3XTF32: tensor-core f16 / error-compensated 3xF16 on planes */
int fs2_op_attention(int math_mode, const float* qkv, const int64_t* lens, int B, int L, int C, int heads, float* ctx,
                     void* stream);
/* The operand-plane attention on the layouts the model's q|k|v projection writes, all fp16 scaled by 16:
 *   qkp  q|k planes [P][B*L][2C] (16-byte aligned), P = 2 in FS2_MATH_3XTF32 (hi, lo) and 1 in FS2_MATH_F16 (hi);
 *   vtp  V^T planes [P][B*heads][d_k][lpad], lpad >= L, lpad % 8 == 0 (16-byte aligned).
 * Outputs (at least one): ctx fp32 [B,L,C] and/or ctxp, the context as operand planes [P][B*L][C] (32-byte aligned,
 * B*L*C % 16 == 0).  lens as in fs2_op_attention; rows t >= lens[b] are written as +0.  Only q|k rows and V^T columns
 * below lens[b] (below L when lens is NULL) are read for their values.  Other math modes are rejected. */
int fs2_op_attention_planes(int math_mode, const void* qkp, const void* vtp, int lpad, const int64_t* lens, int B, int L,
                            int C, int heads, float* ctx, void* ctxp, void* stream);
/* y = LayerNorm_C(x (+resid)) * g + b over the last dim (C in {256,384}) */
int fs2_op_layernorm(const float* x, const float* resid, const float* g, const float* b, float eps, int64_t rows, int C,
                     float* out, void* stream);

/* ---- train mode (SURVEY.md section 8f-1): dropout, BatchNorm batch statistics and the backward of every stage ------- */
/* What `model.train(); loss, _ = model(...); loss.backward()` of train_fastspeech.py:100-123 needs; fp32 on CUDA cores
 * (csrc/train.cu).  fastspeech2_b200/train.py chains these with torch.autograd.Function objects (autograd = graph plumbing
 * only).  Weights are taken in the REFERENCE's layouts (nn.Conv1d [N,K,taps], nn.Linear [N,K]); gradients are accumulated
 * (+=) into caller-zeroed buffers of the same layouts.  Activations are [B, time, channel] fp32 like the eval path. */
/* nn.Dropout (train): mask[i] = 1 keep / 0 drop from a Philox4x32-10 stream keyed by (seed, offset + i/4); out = x * mask / (1-p) */
int fs2_dropout_mask(uint8_t* mask, int64_t n, float p, uint64_t seed, uint64_t offset, void* stream);
int fs2_dropout_apply(const float* x, const uint8_t* mask, float p, float* out, int64_t n, void* stream);
/* dx = dy * f'(y) from the saved output y: act 1 = relu, 2 = tanh */
int fs2_act_backward(const float* dy, const float* y, int act, float* dx, int64_t n, void* stream);
int fs2_relu(const float* x, float* y, int64_t n, void* stream);
int fs2_add(const float* a, const float* b, float* y, int64_t n, void* stream);
int fs2_colsum(const float* x, int64_t rows, int C, float* out /* += */, void* stream);
/* Conv1d("same") / Linear: forward (core/modules.py:247-248, attention.py:48-50,74, ...), input gradient, weight + bias
 * gradient.  scratch: N*K*taps floats.  taps must be odd: fs2_conv_dgrad and fs2_conv_wgrad return FS2_ERR_INVALID
 * for even or non-positive taps (and wgrad for N, K < 1 or B, L < 0) before launching anything */
int fs2_conv_forward(const float* x, int B, int L, int K, const float* w, const float* bias, int N, int taps, int act, const float* resid,
                     float* out, float* scratch, void* stream);
int fs2_conv_dgrad(const float* dy, int B, int L, int N, const float* w, int K, int taps, float* dx, float* scratch, void* stream);
int fs2_conv_wgrad(const float* dy, const float* x, int B, int L, int N, int K, int taps, float* dw /* += */, float* dbias /* += or NULL */, void* stream);
/* The tf32 train mode (DESIGN.md §10).  math_mode FS2_MATH_FP32 is exactly fs2_conv_forward / fs2_conv_dgrad; FS2_MATH_TF32
 * runs the same packed weights through the tensor-core tap GEMM's tf32 family (operands truncated to tf32 by the MMA, fp32
 * accumulation), which needs K % 4 == 0, N % 16 == 0 (forward; dgrad: the reverse) and 16-byte aligned rows.  Other modes:
 * FS2_ERR_INVALID. */
int fs2_conv_forward_ex(const float* x, int B, int L, int K, const float* w, const float* bias, int N, int taps, int act, const float* resid,
                        float* out, float* scratch, int math_mode, void* stream);
int fs2_conv_dgrad_ex(const float* dy, int B, int L, int N, const float* w, int K, int taps, float* dx, float* scratch, int math_mode,
                      void* stream);
/* Weight gradient on the tensor cores: dw[n][k][j] += sum_{b, t < L} dy[b,t,n] * x[b, t+j-pad, k] (x zero outside [0, L) of
 * each utterance; pad = (taps - 1) / 2, taps odd), dw in the reference layout [N][K][taps]; dy [B,L,N], x [B,L,K] fp32.
 * Operands are rounded to tf32 (round to nearest) and multiplied by tf32 wgmma with fp32 accumulation; split-K partial
 * sums are added into dw in a fixed order, without atomics, so the same inputs always give the same bits, on any H100.
 * dbias (+=, optional) is the column sum of dy (fs2_colsum, atomics).  ws: caller-owned device workspace of at least
 * fs2_conv_wgrad_tc_ws_bytes(...) bytes, 16-byte aligned; its contents on entry do not matter.  Any N, K >= 1; sizes whose
 * workspace or tensor strides would overflow, and a short workspace, are FS2_ERR_INVALID.  B * L == 0 adds nothing. */
int fs2_conv_wgrad_tc_ws_bytes(int B, int L, int N, int K, int taps, size_t* bytes);
int fs2_conv_wgrad_tc(const float* dy, const float* x, int B, int L, int N, int K, int taps, float* dw /* += */, float* dbias /* += or NULL */,
                      void* ws, size_t ws_bytes, void* stream);
/* nn.LayerNorm backward from the saved input rows (C in {256, 384}) */
int fs2_layernorm_backward(const float* x, const float* dy, const float* gamma, float eps, int64_t rows, int C, float* dx, float* dgamma /* += */,
                           float* dbeta /* += */, void* stream);
/* BatchNorm1d over the rows of [rows, C] with batch statistics (core/modules.py:296), optional tanh (act 2); updates the running
 * statistics in place (momentum, unbiased variance); stats [2C] = mean | biased variance; scratch: 2*C doubles */
int fs2_batchnorm_train(const float* x, int64_t rows, int C, const float* gamma, const float* beta, float eps, float momentum, int act,
                        float* running_mean, float* running_var, float* stats, float* y, void* scratch, void* stream);
int fs2_batchnorm_backward(const float* x, const float* dy, const float* stats, const float* gamma, float eps, int64_t rows, int C, float* dx,
                           float* dgamma /* += */, float* dbeta /* += */, void* scratch, void* stream);
/* strided batched fp32 GEMM over (batch, head): C = alpha * A . B, every operand as (pointer, batch stride, head stride, row
 * stride, column stride) in floats -- the attention products and their transposes in forward and backward */
int fs2_bgemm(const float* a, int64_t abs_, int64_t ahs, int64_t ars, int64_t acs, const float* b, int64_t bbs, int64_t bhs, int64_t brs, int64_t bcs,
              float* c, int64_t cbs, int64_t chs, int64_t crs, int64_t ccs, int batch, int heads, int M, int N, int K, float alpha, void* stream);
/* core/attention.py:58-69 on materialised scores [B*heads, L, L]: mask, softmax, masked_fill(0) -> p; dropout -> pd; and its backward */
int fs2_attn_softmax(const float* s, const int64_t* lens, const uint8_t* dmask, float p_drop, int B, int heads, int L, float* p, float* pd, void* stream);
int fs2_attn_softmax_backward(const float* p, const float* dpd, const uint8_t* dmask, float p_drop, int B, int heads, int L, float* ds, void* stream);
/* Fused attention of the tf32 train mode (DESIGN.md §13, csrc/attention_train_tc.cu): the forward and backward of
 * fs2_bgemm + fs2_attn_softmax[_backward] above (train.py's AttentionFn) on q, k, v [B, L, C] (heads contiguous, head width
 * C / heads = 128 or 192), without any [B, heads, L, L] tensor.  Products are 1xTF32 on the tensor cores (operands rounded
 * to tf32 with round-to-nearest, fp32 accumulation); no atomics, so the same inputs give the same bits.  A score is valid
 * where query and key are below lens[b] (clamped to [0, L]); rows of out / dq and of dk / dv past lens[b] are written as 0,
 * and nothing past lens[b] is read.  Dropout after the softmax (scale 1 / (1 - p_drop)): dmask [B, heads, L, L] uint8
 * (1 = keep) when non-NULL, else element e = ((b heads + h) L + i) L + j is kept where byte e of
 * fs2_dropout_mask(mask, B heads L L, p_drop, seed, offset) is 1 (regenerated, never stored).  lse [B * heads, L] is the row
 * log-sum-exp of the valid scores (0 for rows past lens[b]); the backward takes it and the forward's out.
 * ws: caller-owned device workspace, 16-byte aligned, of at least fs2_attn_train_ws_bytes(...) =
 *   4 * align256(B L C 4) + align256(B heads L 4) bytes;
 * its contents on entry do not matter.  B, L >= 1; a null pointer, another head width, C not divisible by heads, p_drop
 * outside [0, 1), a short or misaligned workspace and sizes that would overflow are FS2_ERR_INVALID. */
int fs2_attn_train_ws_bytes(int B, int L, int C, int heads, size_t* bytes);
int fs2_attn_train_forward(const float* q, const float* k, const float* v, const int64_t* lens, int B, int L, int C, int heads, float p_drop,
                           const uint8_t* dmask, uint64_t seed, uint64_t offset, float* out, float* lse, void* ws, size_t ws_bytes,
                           void* stream);
int fs2_attn_train_backward(const float* q, const float* k, const float* v, const float* out, const float* lse, const float* dout,
                            const int64_t* lens, int B, int L, int C, int heads, float p_drop, const uint8_t* dmask, uint64_t seed,
                            uint64_t offset, float* dq, float* dk, float* dv, void* ws, size_t ws_bytes, void* stream);
/* encoder input (fastspeech.py:65-67 + embedding.py:105-120 before its dropout) and its backward; decoder-side x + alpha*pe */
int fs2_embed_posenc(const int64_t* xs, const float* table, int n_sym, const float* pe, const float* alpha, int B, int T, int C, float* out,
                     void* stream);
int fs2_embed_backward(const int64_t* xs /* NULL: positional part only */, const float* dy, const float* pe, int B, int T, int C, int n_sym,
                       float* dtable /* += or NULL */, float* dalpha /* += */, void* stream);
int fs2_posenc_add(const float* x, const float* pe, const float* alpha, int B, int T, int C, float* y, void* stream);
/* pitch / energy embedding = Linear(n_bins -> C) on a one-hot (fastspeech.py:102,113,218-219), W [C, n_bins] */
int fs2_onehot_linear_forward(const float* x, const int64_t* ids, const float* W, const float* b, int64_t rows, int C, int n_bins, float* y,
                              void* stream);
int fs2_onehot_linear_backward(const int64_t* ids, const float* dy, int64_t rows, int C, int n_bins, float* dW /* += */, float* dbias /* += or NULL */,
                               void* stream);
/* LengthRegulator backward: dhs[b,i,:] = sum of dout[b,j,:] over the frames j expanded from phoneme i (cum from fs2_length_plan) */
int fs2_length_regulator_backward(const float* dout, const int32_t* cum, const int64_t* ilens, int B, int T, int C, int Lcap, float* dhs, void* stream);
/* predictor head Linear(C -> 1) + masked_fill(pad, 0) (duration_predictor.py:75,83-84) and its backward */
int fs2_rowdot(const float* x, const float* w, const float* bias, const int64_t* lens, int64_t rows, int L, int C, float* y, void* stream);
int fs2_rowdot_backward(const float* x, const float* w, const float* dy, const int64_t* lens, int64_t rows, int L, int C, float* dx, float* dw /* += */,
                        float* dbias /* += */, void* stream);
/* gradients of the total loss of fs2_masked_losses w.r.t. its five predicted inputs; grad_loss: device scalar dL/dloss */
int fs2_loss_backward(const float* before, const float* after, const float* ys, int ld_ys_time, const float* d_out, const void* ds, int ds_dtype,
                      const float* e_out, const float* p_out, const float* es, const float* ps, const int64_t* ilens, const int64_t* olens,
                      int B, int T, int L, int odim, const float* grad_loss, float* g_before, float* g_after, float* g_d, float* g_e, float* g_p,
                      void* stream);

/* ---- vocoder hand-off (SURVEY.md section 8f-2): the STFT / inverse STFT Griffin-Lim iterates ------------------------- */
/* utils/stft.py:82-151 without cuFFT, like the reference (which runs them as conv1d / conv_transpose1d with Fourier bases):
 * the two GEMMs go through fs2_op_tap_gemm, these are the kernels around them.  fastspeech2_b200/vocoder.py drives them.
 *   fs2_stft_frames       frames[b,f,k] = reflect_pad(x, n_fft/2)[b, f*hop + k]                       (:89-95)
 *   fs2_stft_magphase     spec [B*frames, ld] (real | imag) -> magnitude, phase [B, cutoff, frames]   (:105-112)
 *   fs2_istft_recombine   (magnitude, phase) -> [B*frames, ld] = mag*cos | mag*sin | 0-padding        (:115-117)
 *   fs2_istft_overlap_add overlap-add of [B, frames, n_fft] at stride hop, / window_sum where > tiny, * n_fft/hop, trimmed
 *                         by n_fft/2 at both ends -> y [B, (frames-1)*hop]                              (:119-149) */
int fs2_stft_frames(const float* x, int B, int n, int n_fft, int hop, int frames, float* out, void* stream);
int fs2_stft_magphase(const float* spec, int ld, int B, int cutoff, int frames, float* mag, float* phase, void* stream);
int fs2_istft_recombine(const float* mag, const float* phase, int B, int cutoff, int frames, int ld, float* rec, void* stream);
int fs2_istft_overlap_add(const float* frames_out, int B, int n_fft, int hop, int frames, const float* window_sum, float tiny, float* y, void* stream);

/* ---- batched waveform synthesis: mel inversion + per-utterance Griffin-Lim (DESIGN.md section 7) -------------------- */
/* From the model's log-mels [B, Lmax, n_mels] with frame counts olens [B] to audio [B, (Lmax-1)*hop]:
 *   M[b, f, :] = max(0, P . exp(mels[b, f, :])) for f < olens[b] (P = pinv(mel filterbank), [cutoff = n_fft/2+1, n_mels]);
 *   y = ISTFT(M (.) u), then n_iters x { Z = STFT(y); Zh = Z - momentum/(1+momentum) Z_prev; u = Zh/|Zh| ((1,0) where
 *   Zh == 0); Z_prev = Z; y = ISTFT(M (.) u) }, each utterance over its own olens[b] frames (reflect padding and window
 *   sum at its own edges).  u at the start: the phasors of `angles` [B, cutoff, Lmax] (radians), or drawn from
 *   Philox4x32-10 keyed by seeds[b] with counter f * cutoff + c.  audio[b, s] = 0 for s >= (olens[b]-1)*hop; utterance b
 *   is bit-identical to a B = 1 call on its own frames.  No allocation, no synchronisation: calls can be graph-captured.
 * Data-dependent checks run on the device and are reported in *status (device int, zeroed by the call):
 *   FS2_VOC_BAD_LENGTH  some olens[b] outside [1, Lmax] or with (olens[b]-1)*hop <= n_fft/2 (too short for reflect
 *                       padding); such an utterance's audio is 0;
 *   FS2_VOC_RANGE       an fp16 operand plane (f16 / 3xF16 modes) would saturate: some exp(mel), |M (.) u| or |y| above
 *                       65504 / kPlaneScale (4094).  Magnitudes of a signal within [-1, 1] are at most n_fft/2. */
#define FS2_VOC_BAD_LENGTH 1
#define FS2_VOC_RANGE 2
typedef struct fs2_vocoder fs2_vocoder;
typedef struct fs2_vocoder_config {
  int32_t n_fft, hop, win_length, n_mels;
  int32_t math_mode;   /* FS2_MATH_*: the three GEMMs (mel inversion, inverse and forward DFT) */
} fs2_vocoder_config;
/* on the current device */
int fs2_vocoder_create(fs2_vocoder** out, const fs2_vocoder_config* cfg);
void fs2_vocoder_destroy(fs2_vocoder* v);
/* device fp32: w_forward / w_inverse [2*cutoff, n_fft] (windowed Fourier basis and its scaled pseudo-inverse, the
 * reference STFT's forward_basis / inverse_basis), mel_inverse [cutoff, n_mels], window_sq [n_fft] (squared padded window) */
int fs2_vocoder_load(fs2_vocoder* v, const float* w_forward, const float* w_inverse, const float* mel_inverse, const float* window_sq,
                     void* stream);
int fs2_vocoder_workspace_bytes(fs2_vocoder* v, int B, int Lmax, size_t* bytes);
/* mag_out [B, cutoff, Lmax] = M (the reference's [B, freq, frames] layout), 0 at frames >= olens[b] */
int fs2_mel_magnitude(fs2_vocoder* v, const float* mels, const int64_t* olens, int B, int Lmax, float* mag_out, int* status,
                      void* ws, size_t ws_bytes, void* stream);
/* seeds [B] (used when angles == NULL) or angles [B, cutoff, Lmax]; momentum in [0, 1); audio [B, (Lmax-1)*hop] */
int fs2_griffin_lim(fs2_vocoder* v, const float* mels, const int64_t* olens, int B, int Lmax, int n_iters, float momentum,
                    const int64_t* seeds, const float* angles, float* audio, int* status, void* ws, size_t ws_bytes, void* stream);

/* ---- training features: mel, energy and DIO pitch per utterance (DESIGN.md section 14) ----------------------------- */
/* What the reference's nvidia_preprocessing.py computes per wav file, for a ragged batch: wav [B, Nmax] fp32 with lens [B]
 * (int64); utterance b is x_b = wav[b, :lens[b]] and samples past lens[b] are never read.  T_b = lens[b] / hop + 1,
 * Tmax = Nmax / hop + 1.
 *   fs2_mel_energy  mel [B, Tmax, n_mels] = log(max(mel_basis . |STFT(x_b)|, 1e-5)) (the layout synthesis returns) and
 *                   energy [B, Tmax] = sqrt(sum_c |STFT(x_b)|[c]^2); the STFT is the reference's (periodic Hann window,
 *                   reflect padding of n_fft/2 at the utterance's own edges, stride hop), on the tap GEMM in math_mode.
 *   fs2_dio         f0 [B, Tmax] float64 and plens [B] int64: WORLD's DIO (pyworld.dio with f0_floor, f0_ceil,
 *                   channels_in_octave, frame_period = hop / sample_rate * 1000, speed 1, allowed_range) truncated to
 *                   plens[b] = min(f0_length_b, T_b), f0_length = int(1000.0 * lens[b] / sample_rate / frame_period) + 1.
 *                   Float64 throughout; the filters run as direct-form circular FIRs.
 * Frames past T_b / plens[b] are +0.  Utterance b is bit-identical to a B = 1 call on x_b.  No allocation, no
 * synchronisation: calls can be graph-captured.  Data-dependent checks are reported in *status (device int, zeroed by the call):
 *   FS2_FEAT_BAD_LENGTH  some lens[b] outside (n_fft/2, Nmax] (reflect padding needs more than n_fft/2 samples); that
 *                        utterance's outputs are 0 and its plens 0;
 *   FS2_FEAT_RANGE       some |x| > 1 (or NaN) within lens (the reference asserts |y| <= 1; it also bounds the fp16
 *                        operand planes, |STFT| <= n_fft/2).
 * Workspace (one buffer serves both entries), with cutoff = n_fft/2 + 1, cpad = ceil(2 cutoff / 64) * 64,
 * mpad = ceil(cutoff / 64) * 64, Tp = Tmax + 1, P = 2 round(sample_rate / (f0_floor * 2^(1/channels_in_octave)) / 2),
 * every term rounded up to 256 bytes; the total is the larger sum plus 256:
 *   mel  = B Tmax (n_fft + cpad + mpad + n_mels) * 4 + B * 8
 *   dio  = B * 24 + B (Nmax + 1 + 2P) * 8 + B (Nmax + 2) * 8 + 4 B (Nmax / 2 + 2) * 8 + 4 B * 4 + (n_bands + 4) B Tp * 8
 *   that is at most 48 B Nmax + 16 KiB * B + 4 KiB at the default 22.05 kHz,
 *   n_fft 1024, hop 256, 80 mels. */
#define FS2_FEAT_BAD_LENGTH 1
#define FS2_FEAT_RANGE 2
typedef struct fs2_features fs2_features;
typedef struct fs2_features_config {
  int32_t sample_rate, n_fft, hop, win_length, n_mels;
  int32_t math_mode;    /* FS2_MATH_*: the two GEMMs (forward DFT, mel filterbank) */
  double f0_floor, f0_ceil, channels_in_octave, allowed_range;   /* DIO: 71, 800, 2, 0.1 in the reference */
} fs2_features_config;
/* create touches no device; load allocates the weights on the current device, and calls run on that device */
int fs2_features_create(fs2_features** out, const fs2_features_config* cfg);
void fs2_features_destroy(fs2_features* f);
/* device fp32: w_forward [2*cutoff, n_fft] (the reference STFT's windowed forward_basis), mel_basis [n_mels, cutoff] */
int fs2_features_load(fs2_features* f, const float* w_forward, const float* mel_basis, void* stream);
int fs2_features_workspace_bytes(fs2_features* f, int B, int Nmax, size_t* bytes);
int fs2_mel_energy(fs2_features* f, const float* wav, const int64_t* lens, int B, int Nmax, float* mel, float* energy, int* status,
                   void* ws, size_t ws_bytes, void* stream);
int fs2_dio(fs2_features* f, const float* wav, const int64_t* lens, int B, int Nmax, double* f0, int64_t* plens, int* status,
            void* ws, size_t ws_bytes, void* stream);

/* ---- objective evaluation: MCD under DTW, and F0, voicing and energy errors along its path (DESIGN.md section 20) ---- */
/* Synthesized log-mels x [B, Lx_max, n_mels] fp32 with xlens [B], reference log-mels y [B, Ly_max, n_mels] with ylens [B]
 * (the layout fs2_mel_energy writes); rows at or past a length are never read.  Pair b (Lx = xlens[b], Ly = ylens[b]):
 *   c[t, k]  = sum_{m < n_mels} double(mel[t, m]) * dct[m, k - 1], k = 1..n_cep   (dct: the orthonormal DCT-II basis
 *              without c0, float64 [n_mels, n_cep], built by the caller)
 *   d(i, j)  = sqrt(sum_k (cx[i, k] - cy[j, k])^2)
 *   A(0, 0)  = d(0, 0), A(i, j) = d(i, j) + min over (i-1, j-1), (i-1, j), (i, j-1) that exist, in that order, the first
 *              minimum winning; no band
 *   cost[b]  = A(Lx - 1, Ly - 1), plen[b] = P the number of cells on the chosen path, mcd[b] = cost / P * scale
 *              (scale = 10 sqrt(2) / ln 10 for dB)
 *   path     NULL, or int32 [B, Lx_max + Ly_max - 1, 2]: the path's (i, j) from (0, 0), -1 past plen[b]
 * Sums run over increasing m / k with every product and sum rounded (no FMA contraction): float64 restatements with the
 * same order match bit for bit, and pair b is bit-identical to a B = 1 call.  4 kernels (and a memset) with a path, 3
 * without; no allocation, no synchronisation.  Data-dependent checks are reported in *status (device int, zeroed):
 *   FS2_EVAL_BAD_LENGTH  some xlens[b] / ylens[b] outside [1, L_max]; that pair's mcd and cost are NaN, plen 0, path -1;
 *   FS2_EVAL_NONFINITE   a non-finite log-mel inside a valid region.
 * Workspace (fs2_dtw_workspace_bytes), with W = min(Lx_max, Ly_max) and every term rounded up to 256 bytes, plus 256:
 *   8 B (Lx_max + Ly_max) n_cep  +  (W > 1024 ? 36 B W : 0)  +  (with_path ? B (Lx_max + Ly_max - 1) W : 0)
 * so without a path it grows with Lx_max + Ly_max, not with their product.
 *
 * fs2_path_prosody walks each path[b, :plen[b]] ([B, P_max, 2], as fs2_mcd_dtw writes it) in order, with
 * fx = f0x[b, i] if i < f0x_lens[b] else 0 (f0x [B, Fx] float64), fy likewise, a frame voiced when its F0 > 0, and the
 * energies ex [B, Ex], ey [B, Ey] fp32:
 *   counts[b] = (P, cells whose voicing differs, cells voiced on both sides, voiced cells with |fx/fy - 1| > 0.2)  int64
 *   sums[b]   = (sum (1200 log2(fx/fy))^2 over cells voiced on both sides, sum (ex[i] - ey[j])^2)            float64
 * FS2_EVAL_BAD_LENGTH in *status: plen[b] outside [0, P_max], a F0 length outside [0, Fx] / [0, Fy], or a path cell
 * outside [0, Ex) x [0, Ey) (the pair's walk stops there).  One kernel, no workspace. */
#define FS2_EVAL_BAD_LENGTH 1
#define FS2_EVAL_NONFINITE 2
int fs2_dtw_workspace_bytes(int B, int Lx_max, int Ly_max, int n_mels, int n_cep, int with_path, size_t* bytes);
int fs2_mcd_dtw(const float* x, const int64_t* xlens, int Lx_max, const float* y, const int64_t* ylens, int Ly_max, int B,
                int n_mels, const double* dct, int n_cep, double scale, double* mcd, double* cost, int64_t* plen, int32_t* path,
                int* status, void* ws, size_t ws_bytes, void* stream);
int fs2_path_prosody(const int32_t* path, const int64_t* plen, int B, int P_max, const double* f0x, const int64_t* f0x_lens, int Fx,
                     const double* f0y, const int64_t* f0y_lens, int Fy, const float* ex, int Ex, const float* ey, int Ey,
                     int64_t* counts, double* sums, int* status, void* stream);

/* ---- band-limited resampling: librosa 0.7.0's resample (resampy kaiser_best) (DESIGN.md section 22) ---------------- */
/* Mono utterances x [B, Nmax] fp32 with sample counts lens [B] at sr_orig -> y [B, Mmax] fp32 at sr_new, with
 * ratio = double(sr_new) / sr_orig, scale = min(1, ratio), 1 / ratio per output step and index_step = int(scale * 512).
 * table: float64 [FS2_RESAMPLE_TABLE][2], (win[j], delta[j]) interleaved, the kaiser_best right wing (64 zero crossings,
 * 512 entries each, rolloff 0.9475937167399596, Kaiser beta 14.769656459379492) times ratio when ratio < 1, and its
 * forward difference (delta[last] = 0), built by the caller.  Utterance b (N = lens[b]):
 *   n_out    = int(N * ratio) samples computed, olens[b] = ceil(N * ratio), y[b, t] = +0 for t >= n_out
 *   y[b, t]  = resampy's resample_f: the time register, a running float64 sum of 1 / ratio from 0, gives n and frac; the
 *              left wing's taps x[n - i], then the right wing's x[n + 1 + k], each weight win[j] + eta * delta[j], each
 *              product and sum in float64 without FMA, y rounded to float32 after every tap
 * Samples at or past lens[b] are never read; y[b] is bit-identical to a B = 1 call.  Requires sr_orig != sr_new (equal
 * rates return the input unchanged, with no call), index_step >= 1, Mmax in [ceil(Nmax * ratio), 2^26) (which keeps the
 * running sum's rounding far below one input step, so n stays below N).  A memset and 2 kernels; no allocation, no
 * synchronisation.  Data-dependent checks are reported in *status (device int, zeroed):
 *   FS2_RS_BAD_LENGTH  some lens[b] outside [1, Nmax], or int(N * ratio) < 1; that row is 0 and olens[b] 0;
 *   FS2_RS_NONFINITE   a NaN or inf sample within lens[b].
 * Workspace (fs2_resample_workspace_bytes): the time register, 8 B Mmax rounded up to 256 bytes, plus 256. */
#define FS2_RS_BAD_LENGTH 1
#define FS2_RS_NONFINITE 2
#define FS2_RESAMPLE_TABLE 32769
int fs2_resample_workspace_bytes(int B, int Nmax, int sr_orig, int sr_new, int Mmax, size_t* bytes);
int fs2_resample(const float* x, const int64_t* lens, int B, int Nmax, const double* table, int sr_orig, int sr_new, float* y,
                 int64_t* olens, int Mmax, int* status, void* ws, size_t ws_bytes, void* stream);

/* ---- batched MelGAN vocoder (DESIGN.md section 8) ------------------------------------------------------------------- */
/* seungwonpark/melgan's Generator(mel_channel = 80) on log-mels [B, Lmax, 80] with frame counts olens [B]: utterance b is
 * the generator applied to its own frames mels[b, :olens[b]] followed by 10 frames of -11.5129, every reflection pad at its
 * own edges, trimmed to olens[b] * 256 samples.  audio [B, Lmax * 256] fp32, 0 from olens[b] * 256 on; audio[b] is
 * bit-identical to a B = 1 call on its own frames; mel frames past olens[b] are never read.  No allocation, no
 * synchronisation: a call can be graph-captured.  It enqueues 60 kernels.
 * Data-dependent checks run on the device and are reported in *status (device int, written by the call):
 *   FS2_MELGAN_BAD_LENGTH  some olens[b] outside [1, Lmax]; that utterance's audio is 0;
 *   FS2_MELGAN_RANGE       an fp16 operand plane (f16 / 3xF16 modes) would saturate: some GEMM input above 65504 /
 *                          kPlaneScale (4094) in magnitude. */
#define FS2_MELGAN_BAD_LENGTH 1
#define FS2_MELGAN_RANGE 2
typedef struct fs2_melgan_gen fs2_melgan_gen;
/* on the current device; math_mode FS2_MATH_*: every GEMM of the generator (the last conv runs on CUDA cores in fp32) */
int fs2_melgan_create(fs2_melgan_gen** out, int math_mode);
void fs2_melgan_destroy(fs2_melgan_gen* m);
/* weights[42], biases[42]: device fp32 tensors of the 42 convolutions in state_dict order (generator.1, generator.3,
 * generator.4.blocks.{0,1,2}.{2,4}, generator.4.shortcuts.{0,1,2}, generator.6, ... generator.16), weight norm already
 * folded (w = g * v / |v|), in torch's layouts: Conv1d [Cout, Cin, k], ConvTranspose1d [Cin, Cout, k].  Packed once into
 * the GEMM layouts; the tensors may be freed afterwards (stream order). */
int fs2_melgan_load(fs2_melgan_gen* m, const float* const* weights, const float* const* biases, void* stream);
/* fails (FS2_ERR_INVALID) when B * (Lmax + 10) * 256 reaches 2^31, or 65535 * 128 in FS2_MATH_FP32 */
int fs2_melgan_workspace_bytes(fs2_melgan_gen* m, int B, int Lmax, size_t* bytes);
int fs2_melgan(fs2_melgan_gen* m, const float* mels, const int64_t* olens, int B, int Lmax, float* audio, int* status, void* ws,
               size_t ws_bytes, void* stream);
/* A window of the same audio (DESIGN.md section 11): for every utterance b, audio row b (audio_ld >= n_frames * 256
 * samples apart, n_frames * 256 written) holds samples [starts[b] * 256, min(starts[b] + n_frames, olens[b]) * 256) of
 * utterance b, bit-identical to the same samples of fs2_melgan on the whole batch in every math mode, then +0.  A row
 * with starts[b] >= olens[b] is all +0.  starts [B] is a device array, so one captured call serves every step of a stream.
 * Only mel frames [starts[b] - 6, starts[b] + n_frames + 6) below olens[b] are read.  The workspace depends on B and
 * n_frames only; the limits apply to the window's B * (256 * n_frames + 36) rows (below 2^31, at most 65535 * 128 in
 * FS2_MATH_FP32), and (Lmax + 10) * 256 must stay below 2^31.  No allocation, no synchronisation; it enqueues the same
 * kernels as fs2_melgan.  *status: the bits of fs2_melgan (FS2_MELGAN_RANGE only for rows whose values equal the whole
 * call's) and
 *   FS2_MELGAN_BAD_START   some starts[b] < 0; that row is +0. */
#define FS2_MELGAN_BAD_START 4
int fs2_melgan_window_workspace_bytes(fs2_melgan_gen* m, int B, int n_frames, size_t* bytes);
int fs2_melgan_window(fs2_melgan_gen* m, const float* mels, const int64_t* olens, const int64_t* starts, int B, int Lmax,
                      int n_frames, float* audio, int64_t audio_ld, int* status, void* ws, size_t ws_bytes, void* stream);
/* Single MelGAN layers on fs2_melgan's code paths (used by the per-layer tests).  Weights come in torch's layouts and are
 * packed into a stream-ordered temporary as fs2_melgan_load packs them.  status (device int) is set to 0 or
 * FS2_MELGAN_RANGE.  x 16-byte and out 32-byte aligned.
 * fs2_op_melgan_block: one residual block on rows [B*Lp][C], utterance b at rows t < lens[b]:
 *   out = Ws . x + bs + W2 . lrelu(W1 (*)_d reflect_d(lrelu(x)) + b1) + b2, rows t >= lens[b] written as +0;
 *   w1 [C][C][3] (dilation d), w2 and ws [C][C][1].  Every lens[b] must be 0 or lie in [d + 1, Lp], so that one
 *   reflection reaches every tap (fs2_melgan's stages always meet this); rows t >= lens[b] of x are never read.
 *   route 0 = the route fs2_melgan takes at this C and math mode, 1 = producers + tap-GEMMs, 2 = the fused kernel
 *   (FS2_MATH_F16 / FS2_MATH_3XTF32 only).  C in {32, 64, 128, 256}.
 * fs2_op_melgan_upsample: lrelu + ConvTranspose1d(Cin -> Cout, k = 2s, stride s, padding s/2) on x [B*Lin][Cin], each
 *   utterance over its rows t < lens[b] (lens[b] in [0, Lin]) with zeros outside them; w [Cin][Cout][2s], b [Cout];
 *   out [B*Lin*s][Cout], rows at or past lens[b]*s written as +0.  s even, Cin and Cout multiples of 16. */
int fs2_op_melgan_block(int math_mode, int route, int C, const float* x, const int64_t* lens, int B, int Lp, int d, const float* w1,
                        const float* b1, const float* w2, const float* b2, const float* ws, const float* bs, float* out, int* status,
                        void* stream);
int fs2_op_melgan_upsample(int math_mode, int Cin, int Cout, int s, const float* x, const int64_t* lens, int B, int Lin, const float* w,
                           const float* b, float* out, int* status, void* stream);

/* ---- batched HiFi-GAN vocoder (DESIGN.md section 16) ---------------------------------------------------------------- */
/* jik876/hifi-gan's Generator on log-mels [B, Lmax, 80] with frame counts olens [B]: utterance b is the generator applied
 * to mels[b, :olens[b]] alone (every convolution zero-pads at its own edges; no tail frames, no normalisation), olens[b] *
 * 256 samples.  audio [B, Lmax * 256] fp32, +0 from olens[b] * 256 on; audio[b] is bit-identical to a B = 1 call on its
 * own frames; mel frames past olens[b] are never read.  No allocation, no synchronisation: a call can be graph-captured.
 * It enqueues 4 + U * (2 + K * G + max(K - 2, 0)) kernels, U = num_upsamples, K = num_kernels, G = 12 (resblock 1) or 4
 * (resblock 2): 160 for V1, 49 for V3, in every math mode.
 * Data-dependent checks run on the device and are reported in *status (device int, written by the call):
 *   FS2_HIFIGAN_BAD_LENGTH  some olens[b] outside [1, Lmax]; that utterance's audio is 0;
 *   FS2_HIFIGAN_RANGE       an fp16 operand plane (f16 / 3xF16 modes) would saturate: some GEMM input above 65504 /
 *                           kPlaneScale (4094) in magnitude. */
#define FS2_HIFIGAN_BAD_LENGTH 1
#define FS2_HIFIGAN_RANGE 2
#define FS2_HIFIGAN_MAX_UPSAMPLES 8
#define FS2_HIFIGAN_MAX_KERNELS 8
/* hifi-gan's config.json fields.  Accepted: resblock 1 or 2; the upsample rates even, their product 256, every kernel size
 * twice its rate; every width upsample_initial_channel / 2^i (i = 0 .. num_upsamples) a multiple of 32, at most 2048;
 * resblock kernel sizes odd in [1, 31]; num_dilations 3 (resblock 1) or 2 (resblock 2), dilations in [1, 1024]. */
typedef struct fs2_hifigan_config {
  int resblock;
  int num_upsamples;
  int upsample_rates[FS2_HIFIGAN_MAX_UPSAMPLES];
  int upsample_kernel_sizes[FS2_HIFIGAN_MAX_UPSAMPLES];
  int upsample_initial_channel;
  int num_kernels;
  int resblock_kernel_sizes[FS2_HIFIGAN_MAX_KERNELS];
  int num_dilations;
  int resblock_dilation_sizes[FS2_HIFIGAN_MAX_KERNELS][4];
} fs2_hifigan_config;
typedef struct fs2_hifigan_gen fs2_hifigan_gen;
/* on the current device; math_mode FS2_MATH_*: every GEMM of the generator (conv_post runs on CUDA cores in fp32).
 * FS2_ERR_INVALID for a config outside the accepted set. */
int fs2_hifigan_create(fs2_hifigan_gen** out, int math_mode, const fs2_hifigan_config* cfg);
void fs2_hifigan_destroy(fs2_hifigan_gen* m);
/* weights[n], biases[n]: device fp32 tensors of the n convolutions in state_dict order (conv_pre, ups.{0..U-1},
 * resblocks.{0..U*K-1} with convs1.{0,1,2} then convs2.{0,1,2} (resblock 1) or convs.{0,1} (resblock 2), conv_post), weight
 * norm already folded, in torch's layouts: Conv1d [Cout, Cin, k], ConvTranspose1d [Cin, Cout, k].  Packed once; the tensors
 * may be freed afterwards (stream order). */
int fs2_hifigan_load(fs2_hifigan_gen* m, const float* const* weights, const float* const* biases, void* stream);
/* fails (FS2_ERR_INVALID) when B * Lmax * 256 reaches 2^31, or exceeds 65535 * 128 in FS2_MATH_FP32 */
int fs2_hifigan_workspace_bytes(fs2_hifigan_gen* m, int B, int Lmax, size_t* bytes);
int fs2_hifigan(fs2_hifigan_gen* m, const float* mels, const int64_t* olens, int B, int Lmax, float* audio, int* status, void* ws,
                size_t ws_bytes, void* stream);
/* A window of the same audio (DESIGN.md section 17): for every utterance b, audio row b (audio_ld >= n_frames * 256
 * samples apart, n_frames * 256 written) holds samples [starts[b] * 256, min(starts[b] + n_frames, olens[b]) * 256) of
 * utterance b, bit-identical to the same samples of fs2_hifigan on the whole batch in every math mode, then +0.  A row
 * with starts[b] >= olens[b] is all +0.  starts [B] is a device array, so one captured call serves every step of a stream.
 * Only mel frames [starts[b] - h_0, starts[b] + n_frames + h_0) below olens[b] are read, h_0 the config's level-0 halo (13
 * for V1, 11 for V3).  The workspace depends on B and n_frames only; the limits apply to the window's largest buffer (V1
 * and V3: B * (256 * n_frames + 2 h_U) rows; below 2^31, at most 65535 * 128 in FS2_MATH_FP32), and Lmax * 256 must stay
 * below 2^31.  No allocation, no synchronisation; it enqueues the same kernels as fs2_hifigan.  *status: the bits of
 * fs2_hifigan (FS2_HIFIGAN_RANGE only for rows whose values equal the whole call's) and
 *   FS2_HIFIGAN_BAD_START  some starts[b] < 0; that row is +0. */
#define FS2_HIFIGAN_BAD_START 4
int fs2_hifigan_window_workspace_bytes(fs2_hifigan_gen* m, int B, int n_frames, size_t* bytes);
int fs2_hifigan_window(fs2_hifigan_gen* m, const float* mels, const int64_t* olens, const int64_t* starts, int B, int Lmax,
                       int n_frames, float* audio, int64_t audio_ld, int* status, void* ws, size_t ws_bytes, void* stream);
/* Single HiFi-GAN layers on fs2_hifigan's code paths (used by the per-layer tests).  Weights come in torch's layouts and are
 * packed into a stream-ordered temporary as fs2_hifigan_load packs them.  status (device int) is set to 0 or
 * FS2_HIFIGAN_RANGE.  x 16-byte and out 32-byte aligned; utterance b is rows t < lens[b] (lens[b] in [0, Lp]), zero outside
 * them; rows t >= lens[b] of x are never read and those of out are written as +0.
 * fs2_op_hifigan_resblock: one residual block (type 1 or 2) on rows [B*Lp][C], kernel size k, dilations dils[nd] (host;
 *   nd = 3 for type 1, 2 for type 2); weights / biases (host arrays of device pointers): the block's convolutions in
 *   state_dict order, each [C][C][k] / [C].  C a multiple of 32.
 * fs2_op_hifigan_upsample: lrelu(x, 0.1) then ConvTranspose1d(Cin -> Cout, k = 2u, stride u, padding u/2) on x [B*Lin][Cin];
 *   w [Cin][Cout][2u], b [Cout]; out [B*Lin*u][Cout].  u even, Cin and Cout multiples of 32. */
int fs2_op_hifigan_resblock(int math_mode, int type, int C, int k, int nd, const int* dils, const float* x, const int64_t* lens, int B,
                            int Lp, const float* const* weights, const float* const* biases, float* out, int* status, void* stream);
int fs2_op_hifigan_upsample(int math_mode, int Cin, int Cout, int u, const float* x, const int64_t* lens, int B, int Lin, const float* w,
                            const float* b, float* out, int* status, void* stream);

/* ---- batched BigVGAN vocoder (DESIGN.md section 18) ----------------------------------------------------------------- */
/* NVIDIA BigVGAN's generator on log-mels [B, Lmax, 80] with frame counts olens [B], with the call surface of fs2_hifigan:
 * utterance b is the generator applied to mels[b, :olens[b]] alone (every convolution zero-pads and every Activation1d
 * replicate-pads at its own edges), olens[b] * 256 samples, bit-identical to a B = 1 call, +0 past them; mel frames past
 * olens[b] are never read.  No allocation, no synchronisation.  It enqueues 4 + U * (2 + K * G + max(K - 2, 0)) kernels,
 * as fs2_hifigan: 160 for the 22 kHz base model, 238 for the large ones, in every math mode.  *status: FS2_BIGVGAN_BAD_LENGTH
 * and FS2_BIGVGAN_RANGE as fs2_hifigan's (and FS2_BIGVGAN_BAD_START for a window). */
#define FS2_BIGVGAN_BAD_LENGTH 1
#define FS2_BIGVGAN_RANGE 2
#define FS2_BIGVGAN_BAD_START 4
#define FS2_BIGVGAN_SNAKE 0
#define FS2_BIGVGAN_SNAKEBETA 1
/* BigVGAN's config.json fields.  gen: the fields it shares with hifi-gan, accepted as fs2_hifigan_create accepts them
 * except the widths: every upsample_initial_channel / 2^i a multiple of 8, at most 2048 (a width that is not a multiple of
 * 32 runs zero-padded to the next one).  activation FS2_BIGVGAN_SNAKE or FS2_BIGVGAN_SNAKEBETA; snake_logscale: the
 * parameters hold log alpha (and log beta); use_tanh_at_final: tanh, else a clamp to [-1, 1]; use_bias_at_final:
 * conv_post has a bias. */
typedef struct fs2_bigvgan_config {
  fs2_hifigan_config gen;
  int activation;
  int snake_logscale;
  int use_tanh_at_final;
  int use_bias_at_final;
} fs2_bigvgan_config;
typedef struct fs2_bigvgan_gen fs2_bigvgan_gen;
int fs2_bigvgan_create(fs2_bigvgan_gen** out, int math_mode, const fs2_bigvgan_config* cfg);
void fs2_bigvgan_destroy(fs2_bigvgan_gen* m);
/* weights[n], biases[n]: as fs2_hifigan_load's, in BigVGAN's state_dict order (conv_pre, ups.{i}.0, resblocks.{j}.convs1 /
 * convs2 or convs, conv_post); biases[n - 1] is ignored (may be NULL) without use_bias_at_final.  acts[4 a + 0 .. 3]: the
 * a-th Activation1d in state_dict order (resblocks.{j}.activations.{i}, then activation_post): alpha [C], beta [C] (NULL
 * for Snake), upsample.filter [12] and downsample.lowpass.filter [12], device fp32. */
int fs2_bigvgan_load(fs2_bigvgan_gen* m, const float* const* weights, const float* const* biases, const float* const* acts, void* stream);
int fs2_bigvgan_workspace_bytes(fs2_bigvgan_gen* m, int B, int Lmax, size_t* bytes);
int fs2_bigvgan(fs2_bigvgan_gen* m, const float* mels, const int64_t* olens, int B, int Lmax, float* audio, int* status, void* ws,
                size_t ws_bytes, void* stream);
/* A window of the same audio, as fs2_hifigan_window, on the window plan of the config (DESIGN.md section 18). */
int fs2_bigvgan_window_workspace_bytes(fs2_bigvgan_gen* m, int B, int n_frames, size_t* bytes);
int fs2_bigvgan_window(fs2_bigvgan_gen* m, const float* mels, const int64_t* olens, const int64_t* starts, int B, int Lmax,
                       int n_frames, float* audio, int64_t audio_ld, int* status, void* ws, size_t ws_bytes, void* stream);
/* Single BigVGAN layers on fs2_bigvgan's code paths (per-layer tests), packed into a stream-ordered temporary.  status is
 * set to 0 or FS2_BIGVGAN_RANGE; utterance b is rows t < lens[b] of Lp, rows past it are never read and written as +0.
 * fs2_op_bigvgan_act: one Activation1d on x [B*Lp][C] (C a multiple of 8, padded to 32 as the vocoder pads it), its four
 *   tensors as in fs2_bigvgan_load, into out [B*Lp][C]: the GEMM operand of math_mode read back as fp32 ((hi + lo) / 16 in
 *   the plane modes).
 * fs2_op_bigvgan_resblock: one AMP block (type 1 or 2) on rows [B*Lp][C] (C a multiple of 32), as fs2_op_hifigan_resblock,
 *   with acts[4 i + 0 .. 3] its activations in state_dict order. */
int fs2_op_bigvgan_act(int math_mode, int C, const float* x, const int64_t* lens, int B, int Lp, const float* const* tensors, int snakebeta,
                       int logscale, float* out, int* status, void* stream);
int fs2_op_bigvgan_resblock(int math_mode, int type, int C, int k, int nd, const int* dils, const float* x, const int64_t* lens, int B,
                            int Lp, const float* const* weights, const float* const* biases, const float* const* acts, int snakebeta,
                            int logscale, float* out, int* status, void* stream);

/* ---- batched iSTFTNet vocoder (DESIGN.md section 19) ---------------------------------------------------------------- */
/* rishikksh20/iSTFTNet-pytorch's Generator on log-mels [B, Lmax, 80] with frame counts olens [B], with the call surface of
 * fs2_hifigan: hifi-gan's generator up to its last MRF (the same kernels), then an inverse-STFT head in place of
 * conv_post + tanh: y = conv_post(ReflectionPad1d((1, 0))(lrelu(x, 0.01))) with n_fft + 2 channels, and
 * audio = istft(exp(y[:n_fft/2+1]) * exp(i sin(y[n_fft/2+1:])), n_fft, hop, periodic Hann, center=True).  Utterance b is
 * the generator applied to mels[b, :olens[b]] alone, olens[b] * 256 samples, bit-identical to a B = 1 call, +0 past them;
 * mel frames past olens[b] are never read.  The head runs on CUDA cores in fp32 in every math mode.  No allocation, no
 * synchronisation.  It enqueues 4 + U * (2 + K * G + max(K - 2, 0)) kernels, as fs2_hifigan: 82 for C8C8I.  *status:
 * FS2_ISTFTNET_BAD_LENGTH and FS2_ISTFTNET_RANGE as fs2_hifigan's (and FS2_ISTFTNET_BAD_START for a window). */
#define FS2_ISTFTNET_BAD_LENGTH 1
#define FS2_ISTFTNET_RANGE 2
#define FS2_ISTFTNET_BAD_START 4
/* iSTFTNet's config.json fields.  gen: hifi-gan's, accepted as fs2_hifigan_create accepts them except that the product
 * of the upsample rates times istft_hop must be 256.  istft_n_fft even, at most 16 (the head kernel's shared memory);
 * istft_hop divides it with istft_n_fft / istft_hop >= 2 (the window envelope is 0 somewhere otherwise). */
typedef struct fs2_istftnet_config {
  fs2_hifigan_config gen;
  int istft_n_fft;
  int istft_hop;
} fs2_istftnet_config;
typedef struct fs2_istftnet_gen fs2_istftnet_gen;
int fs2_istftnet_create(fs2_istftnet_gen** out, int math_mode, const fs2_istftnet_config* cfg);
void fs2_istftnet_destroy(fs2_istftnet_gen* m);
/* weights / biases as fs2_hifigan_load's, conv_post [n_fft + 2, C_U, 7] with its bias [n_fft + 2] */
int fs2_istftnet_load(fs2_istftnet_gen* m, const float* const* weights, const float* const* biases, void* stream);
/* fails (FS2_ERR_INVALID) when B * Lmax * (256 / istft_hop) (the last level's rows) reaches 2^31, or exceeds 65535 * 128
 * in FS2_MATH_FP32 */
int fs2_istftnet_workspace_bytes(fs2_istftnet_gen* m, int B, int Lmax, size_t* bytes);
int fs2_istftnet(fs2_istftnet_gen* m, const float* mels, const int64_t* olens, int B, int Lmax, float* audio, int* status, void* ws,
                 size_t ws_bytes, void* stream);
/* A window of the same audio, as fs2_hifigan_window, on the window plan of the config with the head's reach
 * (4 + (n_fft / 2 - 1) / hop last-level rows: 5 for C8C8I). */
int fs2_istftnet_window_workspace_bytes(fs2_istftnet_gen* m, int B, int n_frames, size_t* bytes);
int fs2_istftnet_window(fs2_istftnet_gen* m, const float* mels, const int64_t* olens, const int64_t* starts, int B, int Lmax,
                        int n_frames, float* audio, int64_t audio_ld, int* status, void* ws, size_t ws_bytes, void* stream);
/* The head alone on fs2_istftnet's code path (per-layer tests): x [B*Lp][C] the last MRF's output (C a multiple of 32),
 * utterance b its rows t < lens[b] (lens[b] in [0, Lp]; a reflected row past lens[b] is 0), conv_post w [n_fft + 2][C][7]
 * and b [n_fft + 2] (device, torch's layout), into audio [B][Lp * hop]: hop * lens[b] samples, +0 past them. */
int fs2_op_istftnet_head(int C, int n_fft, int hop, const float* x, const int64_t* lens, int B, int Lp, const float* w, const float* b,
                         float* audio, void* stream);

/* ---- batched WaveGlow vocoder (DESIGN.md section 9) ----------------------------------------------------------------- */
/* DeepLearningExamples' WaveGlow (n_mel_channels 80, n_flows 12, n_group 8, n_early_every 4, n_early_size 2, WN: 8 layers,
 * kernel 3, n_channels C) in its inverse direction, `infer`, on log-mels [B, Lmax, 80] with frame counts olens [B]:
 * utterance b is infer(mels[b, :olens[b]]) alone -- the upsampling sees only its frames below olens[b] and every dilated
 * convolution zero-pads at its own edges.  audio [B, Lmax * 256] fp32, 0 from olens[b] * 256 on; audio[b] is bit-identical
 * to a B = 1 call with the same noise; mel frames past olens[b] and z steps past olens[b] * 32 are never read.
 * Noise: z [B, 8, Lmax * 32] (device fp32, the layout WaveGlow.forward returns: channels 0-1 the early output of flow 4,
 * 2-3 that of flow 8, 4-7 the last four) or, when z is NULL, drawn per utterance from Philox4x32-10 keyed by seeds[b]
 * (fs2_waveglow_noise writes the same draw).  The flows receive fp32(sigma * z), the product taken in double and rounded
 * once.  No allocation, no synchronisation: a call
 * can be graph-captured.  It enqueues 496 kernels (497 in FS2_MATH_F16 / FS2_MATH_3XTF32).
 * Data-dependent checks run on the device and are reported in *status (device int, written by the call):
 *   FS2_WAVEGLOW_BAD_LENGTH  some olens[b] outside [1, Lmax]; that utterance's audio is 0;
 *   FS2_WAVEGLOW_RANGE       an fp16 operand plane (f16 / 3xF16 modes) would saturate: some GEMM input above 65504 /
 *                            kPlaneScale (4094) in magnitude. */
#define FS2_WAVEGLOW_BAD_LENGTH 1
#define FS2_WAVEGLOW_RANGE 2
typedef struct fs2_waveglow_net fs2_waveglow_net;
/* on the current device; math_mode FS2_MATH_*: every GEMM (start, end, coupling and the 1x1 inverses run on CUDA cores in
 * fp32); n_channels C: a multiple of 64 in [64, 1024] (the published models use 256 or 512) */
int fs2_waveglow_create(fs2_waveglow_net** out, int math_mode, int n_channels);
void fs2_waveglow_destroy(fs2_waveglow_net* m);
/* tensors[638]: device fp32, weight norm folded, torch layouts: upsample.weight [80, 80, 1024], upsample.bias [80], then per
 * flow k = 0 .. 11 (c = 8, 8, 8, 8, 6, 6, 6, 6, 4, 4, 4, 4 channels, h = c / 2): start.weight [C, h, 1], start.bias [C],
 * in_layers.{0..7}.(weight [2C, C, 3], bias [2C]), cond_layers.{0..7}.(weight [2C, 640, 1], bias [2C]),
 * res_skip_layers.{0..7}.(weight [2C or C (i = 7), C, 1], bias), end.weight [2h, C, 1], end.bias [2h], and the inverse of
 * convinv.k's weight [c, c].  Packed once; the tensors may be freed afterwards (stream order). */
int fs2_waveglow_load(fs2_waveglow_net* m, const float* const* tensors, int n, void* stream);
/* fails (FS2_ERR_INVALID) when B * Lmax * 32 reaches 2^31, or exceeds 65535 * 128 in FS2_MATH_FP32 */
int fs2_waveglow_workspace_bytes(fs2_waveglow_net* m, int B, int Lmax, size_t* bytes);
/* sigma finite and >= 0; seeds [B] i64 (device, used when z is NULL) or z [B, 8, Lmax * 32] */
int fs2_waveglow(fs2_waveglow_net* m, const float* mels, const int64_t* olens, int B, int Lmax, double sigma, const int64_t* seeds,
                 const float* z, float* audio, int* status, void* ws, size_t ws_bytes, void* stream);
/* A window of the same audio (DESIGN.md section 12): for every utterance b, audio row b (audio_ld >= n_frames * 256
 * samples apart, n_frames * 256 written) holds samples [starts[b] * 256, min(starts[b] + n_frames, olens[b]) * 256) of
 * utterance b, bit-identical to the same samples of fs2_waveglow on the whole batch with the same sigma and seeds / z in
 * every math mode, then +0.  A row with starts[b] >= olens[b] is all +0.  starts, olens and seeds [B] are device arrays,
 * so one captured call serves every step of a stream.  z keeps the whole call's layout [B, 8, Lmax * 32].  Only mel frames
 * [starts[b] - 99, starts[b] + n_frames + 96) below olens[b] and z steps [(starts[b] - 96) * 32, (starts[b] + n_frames +
 * 96) * 32) below olens[b] * 32 are read.  The workspace depends on B and n_frames only; the limits apply to the window's
 * B * (n_frames + 192) * 32 step rows (below 2^31, at most 65535 * 128 in FS2_MATH_FP32), and Lmax * 32 must stay below
 * 2^31.  No allocation, no synchronisation.  It enqueues 497 kernels (498 in FS2_MATH_F16 / FS2_MATH_3XTF32): those of
 * fs2_waveglow and a copy of the window's audio.  *status: the bits of fs2_waveglow (FS2_WAVEGLOW_RANGE only for values
 * the whole call also checks) and
 *   FS2_WAVEGLOW_BAD_START   some starts[b] < 0; that row is +0. */
#define FS2_WAVEGLOW_BAD_START 4
int fs2_waveglow_window_workspace_bytes(fs2_waveglow_net* m, int B, int n_frames, size_t* bytes);
int fs2_waveglow_window(fs2_waveglow_net* m, const float* mels, const int64_t* olens, const int64_t* starts, int B, int Lmax,
                        int n_frames, double sigma, const int64_t* seeds, const float* z, float* audio, int64_t audio_ld,
                        int* status, void* ws, size_t ws_bytes, void* stream);
/* the standard-normal draw a seeded fs2_waveglow call uses: z [B, 8, Lmax * 32], 0 at steps t >= olens[b] * 32.  Element
 * (b, ch, t) is Box-Muller on Philox4x32-10(counter (t, ch / 4, 0, 0), key (seeds[b] mod 2^32, seeds[b] / 2^32)). */
int fs2_waveglow_noise(const int64_t* seeds, const int64_t* olens, int B, int Lmax, float* z, void* stream);
/* Stages of the inverse on fs2_waveglow's code paths (per-stage tests), on a loaded handle's packed weights, buffers in a
 * stream-ordered temporary; no synchronisation.  Lengths (device int64 [B]) outside [0, L] count as 0 and set
 * FS2_WAVEGLOW_BAD_LENGTH in *status (device int, written by the call; FS2_WAVEGLOW_RANGE as fs2_waveglow's).  Float
 * pointers 16-byte aligned.  A null or unloaded handle, B or L < 1, misaligned pointers and fs2_waveglow's row limits on
 * B * L step rows are FS2_ERR_INVALID before anything is enqueued.
 * fs2_op_waveglow_upsample: the upsampling of mels [B, Lmax, 80] with frame counts olens into cond [B * Lmax * 32][640]
 *   fp32, the rows the cond GEMMs read (+0 at steps t >= olens[b] * 32; frames past olens[b] are never read).
 *   cond_planes (nullable, FS2_MATH_F16 / FS2_MATH_3XTF32 only): the same rows as the GEMMs' operand planes read back as
 *   fp32, (hi + lo) / 16 (hi / 16 in FS2_MATH_F16), +0 past the steps.
 * fs2_op_waveglow_flow: flow k (0 .. 11, c = 8, 8, 8, 8, 6, 6, 6, 6, 4, 4, 4, 4 channels) of the inverse on the state
 *   [B * Ls][8] (utterance b its rows t < lens[b], in steps; any Ls >= 1): WN k on cond [B * Ls][640] fp32 rows (their
 *   planes written with the range check in the plane modes), then end, the affine coupling and the inverse 1x1 conv from
 *   columns 8 - c .. 7 of state_in into those of state_out (== state_in, or disjoint from it).  Only those columns are
 *   written, +0 at rows t >= lens[b]; rows past lens[b] of state_in, cond and skip_in are never read.  wn_out [B * Ls][C]
 *   (nullable): WN's skip sum before end.  skip_in [B * Ls][C] (nullable): the WN is not run, and the flow's tail runs on
 *   skip_in in its place (cond is then not read and may be NULL; wn_out must be NULL). */
int fs2_op_waveglow_upsample(fs2_waveglow_net* m, const float* mels, const int64_t* olens, int B, int Lmax, float* cond,
                             float* cond_planes, int* status, void* stream);
int fs2_op_waveglow_flow(fs2_waveglow_net* m, int k, const float* cond, const float* skip_in, const float* state_in, float* state_out,
                         const int64_t* lens, int B, int Ls, float* wn_out, int* status, void* stream);

/* ---- multi-GPU exchange step: gather of the final mel shards on one rank over NVLink peer memory ----------------- */
/* Replaces what a reference user would write as torch.distributed.gather / all_gather of `after_outs` (the reference has
 * no multi-GPU path; SURVEY.md section 8e defines the step).  The root rank owns one receive buffer and exports it with
 * CUDA IPC; the other ranks map it and push their shard with a copy-engine transfer followed by a release-store of the
 * step number into a flag word; the root waits on the flags with a one-warp acquire-spin kernel.  No collective kernel
 * occupies SMs and nothing is sent to ranks that do not need it.  fastspeech2_b200/sharded.py::PeerGather drives these.
 *   fs2_peer_alloc  cudaMalloc + zero `bytes` on the current device, IPC handle (64 bytes) out
 *   fs2_peer_open   map a peer's allocation into this process (enables peer access lazily); fs2_peer_close unmaps
 *   fs2_peer_copy   asynchronous device-to-(peer-)device copy on `stream`
 *   fs2_flag_signal one-thread kernel: system-scope fence, *flag = value
 *   fs2_flag_wait   one-warp kernel: spin until flags[r] >= value for all r < n, r != skip (bounded: traps after ~10 s) */
int fs2_peer_alloc(size_t bytes, void** ptr, void* handle64);
int fs2_peer_free(void* ptr);
int fs2_peer_open(const void* handle64, void** ptr);
int fs2_peer_close(void* ptr);
int fs2_peer_copy(void* dst, const void* src, size_t bytes, void* stream);
int fs2_flag_signal(int64_t* flag, int64_t value, void* stream);
int fs2_flag_wait(const int64_t* flags, int n, int skip, int64_t value, void* stream);

/* ---- optimizer step: Noam-scheduled Adam, gradient-norm clipping and the NaN guard (DESIGN.md section 15) --------- */
/* Replaces the reference loop's `clip_grad_norm_(model.parameters(), grad_clip); if isnan(norm): skip; NoamOpt.step()`
 * (train_fastspeech.py:117-124, core/optimizer.py) with Adam(betas, eps, weight_decay=0) arithmetic bit-identical to
 * torch's foreach Adam.  fastspeech2_b200/optim.py::NoamAdam drives these.
 *
 * The parameter table is an array of entries in DEVICE memory, built by the caller: one per parameter that has a
 * gradient.  Entry t covers chunks [chunk0, chunk0 + ceil(numel / FS2_OPTIM_CHUNK)) with chunk0 the running sum of the
 * chunk counts of the entries before it; `numel` (HOST, n entries) repeats the sizes so that the call can check them and
 * size its grid.  Any numel >= 1 and any 4-byte aligned pointer are valid (16-byte vectors where the four arrays of an
 * entry share their alignment).  `step` is the entry's Adam step count (fp32, as torch keeps it).
 *
 * Workspace (caller-owned, 256-byte aligned, size from fs2_optim_ws_bytes):
 *   align256(8 n_chunks) + align256(8 n) + align256(16)  bytes  (fp64 chunk sums of squares; per-entry step size and
 *   bias-correction root; norm, coefficient, skip flag).
 * Device state (caller-owned): noam_step (int64, NoamOpt._step), lr (double, the lr of the last step that ran).
 *   fs2_optim_noam_adam       noam_step += 1, lr = rate(noam_step), every entry's step += 1, one Adam update
 *   fs2_optim_clip_noam_adam  total norm of the grads (fp64 chunk sums, fixed-order reduction, one rounding to fp32) into
 *                             *norm, coefficient min(max_norm * (1 / (norm + 1e-6)), 1); NaN norm: nothing else changes;
 *                             otherwise the update above on grad * coefficient (the grads themselves are not written)
 *   fs2_optim_noam_scalars    test entry: lr, fp32 step size and fp32 bias-correction root for steps step0 .. step0+count-1
 * Three (clip) or two kernels, no allocation, no synchronisation: graph-capturable.  An empty table, numel < 1, a
 * chunk count past 2^31 - 1, a null pointer or a short / misaligned workspace are FS2_ERR_INVALID. */
#define FS2_OPTIM_CHUNK 65536
typedef struct fs2_optim_entry {
  float* param; const float* grad; float* exp_avg; float* exp_avg_sq; float* step;
  int64_t numel; int64_t chunk0;
} fs2_optim_entry;
typedef struct fs2_noam_adam_hp {
  double rate_scale;   /* factor * model_size ** -0.5, computed by the caller as NoamOpt.rate groups it */
  double warmup_pow;   /* warmup ** -1.5 */
  double beta1, beta2, eps;
} fs2_noam_adam_hp;
int fs2_optim_ws_bytes(const int64_t* numel, int n, size_t* bytes);
int fs2_optim_noam_adam(const fs2_optim_entry* table, const int64_t* numel, int n, const fs2_noam_adam_hp* hp,
                        int64_t* noam_step, double* lr, void* ws, size_t ws_bytes, void* stream);
int fs2_optim_clip_noam_adam(const fs2_optim_entry* table, const int64_t* numel, int n, const fs2_noam_adam_hp* hp,
                             float max_norm, int64_t* noam_step, double* lr, float* norm, void* ws, size_t ws_bytes,
                             void* stream);
int fs2_optim_noam_scalars(int64_t step0, int count, const fs2_noam_adam_hp* hp, double* lr, float* step_size,
                           float* bc2_sqrt, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FS2_H100_H_ */
