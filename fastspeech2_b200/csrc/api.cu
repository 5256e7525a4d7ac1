// C ABI of libfs2b200.so (declared in include/fs2_b200.h): handle, checkpoint repacking and
// the host-side sequencing of the kernels for each stage of FeedForwardTransformer._forward
// (fastspeech.py:169-243).  No kernel lives here.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <string>
#include <unordered_map>
#include <vector>

#include "vocoder_weights.cuh"

namespace fs2 {

static thread_local char g_err[512] = "";
std::atomic<unsigned long long> g_kernel_launches{0};
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// every Linear / Conv1d is a VWeight (vocoder_weights.cuh) with a per-layer power-of-two scale chosen at load time
struct Norm { const float* g = nullptr; const float* b = nullptr; float eps = 1e-5f; };
struct Block { VWeight qkv, out, w1, w2; Norm ln1, ln2; };
struct Predictor { VWeight conv[4]; Norm ln[4]; const float* head_w = nullptr; const float* head_b = nullptr; int layers = 0; };


// ---- per-kernel-class CUDA-event profiler (bench.py roofline; off by default) -------------
enum ProfClass {
  P_EMBED, P_ENC_QKV, P_ENC_ATTN, P_ENC_OUT, P_ENC_W1, P_ENC_W2, P_PRED_GEMM, P_ROWNORM, P_VAR_EMBED, P_DEC_IN, P_DEC_QKV,
  P_DEC_ATTN, P_DEC_OUT, P_DEC_W1, P_DEC_W2, P_FEAT_OUT, P_POSTNET, P_COUNT
};
static const char* kProfLabels[P_COUNT] = {
  "embed_posenc", "enc.qkv_proj", "enc.attention", "enc.out_proj", "enc.ffn_w1_conv9", "enc.ffn_w2", "predictor.tap_gemm", "row_norm",
  "variance_embed_add", "dec.embed_linear", "dec.qkv_proj", "dec.attention", "dec.out_proj", "dec.ffn_w1_conv9", "dec.ffn_w2", "feat_out", "postnet.conv5"};
struct ProfRec { int cls; cudaEvent_t a, b; double flop, bytes; };
struct Profiler {
  bool on = false;
  std::vector<ProfRec> recs;
};
static thread_local Profiler* t_prof = nullptr;
struct ProfScope {
  ProfRec r; bool live; cudaStream_t st;
  ProfScope(int cls, double flop, double bytes, cudaStream_t s) : live(t_prof && t_prof->on), st(s) {
    if (!live) return;
    r.cls = cls; r.flop = flop; r.bytes = bytes;
    cudaEventCreate(&r.a); cudaEventCreate(&r.b);
    cudaEventRecord(r.a, st);
  }
  ~ProfScope() {
    if (!live) return;
    cudaEventRecord(r.b, st);
    t_prof->recs.push_back(r);
  }
};

}  // namespace fs2

struct fs2_handle {
  fs2::Profiler prof;
  int enc_pe_len = 0, dec_pe_len = 0;
  fs2_config cfg;
  int device = 0;
  bool loaded = false;
  void* arena = nullptr;      // packed weights (owned)
  size_t arena_bytes = 0;
  // encoder side
  const float* emb = nullptr; const float* enc_pe = nullptr; const float* enc_alpha = nullptr;
  std::vector<fs2::Block> enc, dec;
  fs2::Predictor dur, energy, pitch;
  const float* e_bins = nullptr; const float* p_bins = nullptr;
  const float* e_tab = nullptr; const float* e_tab_bias = nullptr;
  const float* p_tab = nullptr; const float* p_tab_bias = nullptr;
  const float* spk_table = nullptr; int n_speakers = 0;   // optional speaker_embed.weight [n_speakers, adim]
  const float* spemb_w = nullptr; const float* spemb_b = nullptr; int spemb_dim = 0;   // optional spk_embed_proj [adim, D], [adim]
  // decoder side
  fs2::VWeight dec_in; fs2::Norm dec_in_ln; const float* dec_pe = nullptr; const float* dec_alpha = nullptr;
  fs2::VWeight feat_out;
  std::vector<fs2::VWeight> postnet;
};

namespace fs2 {
namespace {

using Map = std::unordered_map<std::string, const fs2_weight_desc*>;

// selects the handle's device for the duration of an ABI call and restores the caller's (torch's) current device
struct DeviceGuard {
  int prev = -1; bool ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) { ok = false; return; }
    if (prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};
#define FS2_DEVICE_GUARD(h)                                                              \
  DeviceGuard _guard((h)->device);                                                       \
  if (!_guard.ok) { set_error("cannot select device %d", (h)->device); return FS2_ERR_CUDA; }

int dense(const TapGemm& g, int math_mode, cudaStream_t st, int cls) {
  const double M = (double)g.B * g.L;
  // algorithmic bytes: operands at the width this launch reads them (hi plane: 2 B; fp32, or hi + lo planes: 4 B),
  // the result at the width(s) it is written, the residual as fp32
  const double e_in = g.xp ? (g.precise ? 4.0 : 2.0) : 4.0;
  const double e_out = (g.out ? 4.0 : 0.0) + ((g.outp || g.vtp) ? (g.outp_lo ? 4.0 : 2.0) : 0.0);
  ProfScope prof_scope(cls, 2.0 * M * g.N * g.K * g.taps,
               e_in * (M * g.K + (double)g.taps * g.N * g.K) + M * g.N * (e_out + (g.resid ? 4.0 : 0.0)), st);
  return tap_gemm(g, math_mode, st);
}
int norm_rows(const RowNorm& r, cudaStream_t st) {
  ProfScope prof_scope(P_ROWNORM, 8.0 * r.rows * r.C,
                       4.0 * r.rows * r.C * (1 + (r.resid ? 1 : 0) + (r.out ? 1 : 0)) + (r.split_out ? (r.split_lo ? 4.0 : 2.0) * r.rows * r.C : 0.0), st);
  return row_norm(r, st);
}
inline int round4(int x) { return (x + 3) & ~3; }
inline int round8(int x) { return (x + 7) & ~7; }

// a GEMM's A operand in math_mode: the fp32 rows x, or the operand planes xp of the same tensor in the plane modes
inline const void* operand(int math_mode, const float* x, const __half* xp) { return plane_mode(math_mode) ? (const void*)xp : x; }

RowNorm make_norm(const Norm& n, const float* x, int ldx, int64_t rows, int C, float* out, int ldo) {
  RowNorm r;
  memset(&r, 0, sizeof(r));
  r.x = x; r.ldx = ldx; r.gamma = n.g; r.beta = n.b; r.eps = n.eps; r.rows = rows; r.C = C; r.out = out; r.ldo = ldo;
  return r;
}

// Per-utterance mode (FS2_PER_UTTERANCE): zlens != nullptr.  Every tensor a convolution reads or the caller receives then
// holds exact zeros at rows t >= zlens[b], so each convolution's "same" padding falls at the utterance's own length, as in
// a B = 1 run.  zlens == nullptr leaves the kernels exactly as in the reference-semantics path.
RowNorm masked(RowNorm r, const int64_t* zlens, int L) {
  if (zlens) { r.lens = zlens; r.L = L; }
  return r;
}

// the speaker adds of the last encoder LayerNorm (RowNorm::spk_table, RowNorm::spk_vec); nullptr: none
struct SpeakerAdd { const float* table = nullptr; const int64_t* ids = nullptr; int n = 0; const float* vec = nullptr; };

struct BlockBufs {
  float *x, *y;            // fp32 rows [rows, C]: block input / output ping-pong (the residual stream)
  float *qkv, *vt, *ctx, *hid;   // fp32 families: q|k|v rows, transposed V, context, conv-FFN hidden
  __half *xp, *qkp, *vtp, *ctxp, *hidp;   // plane families: the same tensors as operand planes (qkp..hidp alias the fp32 ones)
};

// FFT blocks in math mode `mode`; the result lands in *result.  fp32 / tf32: fp32 rows everywhere.  f16 / 3xF16: every
// contraction reads fp16 operand planes written by its producer and writes the planes its consumer reads; fp32 rows exist
// only for the residual stream (x, y), and residual + LayerNorm run as a row kernel after each projection.  On entry w.xp
// holds the planes of w.x; on exit it holds the planes of *result.
int run_blocks(const std::vector<Block>& blocks, const BlockBufs& w, const int64_t* lens, const int64_t* zlens, int B, int L,
               int C, int heads, int mode, bool is_dec, cudaStream_t st, float** result, const SpeakerAdd& spk = SpeakerAdd()) {
  const int64_t rows = (int64_t)B * L;
  const int c_qkv = is_dec ? P_DEC_QKV : P_ENC_QKV, c_att = is_dec ? P_DEC_ATTN : P_ENC_ATTN;
  const int c_out = is_dec ? P_DEC_OUT : P_ENC_OUT, c_w1 = is_dec ? P_DEC_W1 : P_ENC_W1, c_w2 = is_dec ? P_DEC_W2 : P_ENC_W2;
  const bool planes = plane_mode(mode), x3 = mode == FS2_MATH_3XTF32;
  const int lpad = planes ? round8(L) : round4(L);
  float *x = w.x, *y = w.y;
  for (const Block& k : blocks) {
    int rc;
    // q | k | v projection (attention.py:48-50), one GEMM with N = 3C.  tf32: the V third is also stored transposed for the
    // tensor-core attention (gemm_tc.cu epilogue).  Plane modes: q | k leave as planes [P][rows][2C], the V third as
    // transposed planes [P][B*heads][dk][lpad]; no fp32 copy exists
    TapGemm gq = vweight_gemm_args(mode, k.qkv, operand(mode, x, w.xp), B, L, ACT_NONE, zlens, planes ? nullptr : w.qkv,
                                   nullptr, 1, w.qkp);
    if (planes) { gq.ldo_p = 2 * C; gq.vtp = w.vtp; }
    else if (mode == FS2_MATH_TF32) gq.vt_out = w.vt;
    if (gq.vtp || gq.vt_out) { gq.vt_col0 = 2 * C; gq.vt_dk = C / heads; gq.vt_heads = heads; gq.vt_lpad = lpad; }
    if ((rc = dense(gq, mode, st, c_qkv))) return rc;
    {
      ProfScope prof_scope(c_att, 4.0 * B * (double)L * L * C, (planes && !x3 ? 2.0 : 4.0) * 4.0 * B * (double)L * C, st);
      rc = planes ? attention_planes(w.qkp, w.vtp, lpad, lens, B, L, C, heads, x3, nullptr, w.ctxp, st)
         : mode == FS2_MATH_TF32 ? attention_tf32(w.qkv, w.vt, lpad, lens, B, L, C, heads, w.ctx, st)
                                 : attention_fp32(w.qkv, lens, B, L, C, heads, w.ctx, st);
      if (rc) return rc;
    }
    // x = LN(x + linear_out(ctx)) (attention.py:74, encoder.py:60-62); plane modes: the LayerNorm also writes the conv-FFN's
    // operand planes.  Per-utterance mode: ctx rows past len are the attention kernels' output of those query rows times 0
    // (the q|k|v projection writes them as zeros, DESIGN.md section 5, so they are zeros of either sign); the out-projection
    // reads each ctx row only for its own output row, which it writes as 0 there
    if ((rc = dense(vweight_gemm_args(mode, k.out, operand(mode, w.ctx, w.ctxp), B, L, ACT_NONE, zlens, y, x), mode, st, c_out)))
      return rc;
    RowNorm r1 = masked(make_norm(k.ln1, y, C, rows, C, x, C), zlens, L);
    if (planes) { r1.split_out = w.xp; r1.split_lo = x3; }
    if ((rc = norm_rows(r1, st))) return rc;
    // conv-FFN: hid = relu(conv_k(x)); x = LN(x + conv_1(hid))  (modules.py:247-248, encoder.py:64-69); plane modes: the
    // hidden activations exist only as planes
    TapGemm g1 = vweight_gemm_args(mode, k.w1, operand(mode, x, w.xp), B, L, ACT_RELU, zlens, planes ? nullptr : w.hid, nullptr,
                                   1, w.hidp);
    if ((rc = dense(g1, mode, st, c_w1))) return rc;
    if ((rc = dense(vweight_gemm_args(mode, k.w2, operand(mode, w.hid, w.hidp), B, L, ACT_NONE, zlens, y, x), mode, st, c_w2)))
      return rc;
    RowNorm r2 = masked(make_norm(k.ln2, y, C, rows, C, x, C), zlens, L);
    if (planes) { r2.split_out = w.xp; r2.split_lo = x3; }   // planes of the block output: A operand of the next q|k|v / mel projection
    if (spk.table && &k == &blocks.back()) { r2.spk_table = spk.table; r2.spk = spk.ids; r2.n_spk = spk.n; r2.spk_L = L; }
    if (spk.vec && &k == &blocks.back()) { r2.spk_vec = spk.vec; r2.spk_L = L; }
    if ((rc = norm_rows(r2, st))) return rc;
  }
  *result = x;
  return FS2_OK;
}

// conv stack + scalar head (duration_predictor.py:64-86 / variance_predictor.py:39-60).  xp == nullptr: exact fp32 FMA on
// the rows x; else error-compensated 3xF16 on the planes xp (the LayerNorms write the next layer's planes into t2p).
// head_scale (nullable, [B*L]): the head's value times a per-row factor, one fp32 rounding (prosody control)
int run_predictor(const Predictor& p, const float* x, const __half* xp, int C, int B, int L, float* t1, float* t2, __half* t2p,
                  const int64_t* lens, const int64_t* zlens, float* head_out, int64_t* dur_out, const float* head_scale,
                  cudaStream_t st) {
  const int64_t rows = (int64_t)B * L;
  const int mode = xp ? MATH_3XTF32 : FS2_MATH_FP32;
  const float* cur = x; const __half* cur_p = xp;
  for (int i = 0; i < p.layers; ++i) {
    int rc;
    const int N = p.conv[i].N;
    if ((rc = dense(vweight_gemm_args(mode, p.conv[i], operand(mode, cur, cur_p), B, L, ACT_RELU, zlens, t1), mode, st, P_PRED_GEMM)))
      return rc;
    RowNorm r = masked(make_norm(p.ln[i], t1, N, rows, N, xp ? nullptr : t2, N), zlens, L);
    if (i == p.layers - 1) {  // last layer: only the scalar head leaves the kernel
      r.out = nullptr; r.head_w = p.head_w; r.head_b = p.head_b; r.head_out = head_out; r.dur_out = dur_out;
      r.head_scale = head_scale;
      r.lens = lens; r.L = L;
    } else if (xp) {
      r.split_out = t2p; r.split_lo = 1;
    }
    if ((rc = norm_rows(r, st))) return rc;
    cur = t2; cur_p = t2p;
  }
  return FS2_OK;
}

const fs2_weight_desc* find(const Map& m, const std::string& k) {
  auto it = m.find(k);
  return it == m.end() ? nullptr : it->second;
}

#define NEED(var, key)                                                        \
  const fs2_weight_desc* var = find(m, key);                                  \
  if (!var) { set_error("fs2_load_weights: missing key '%s'", std::string(key).c_str()); return FS2_ERR_MISSING_WEIGHT; }

// One pass over the checkpoint: on a counting Bump it checks every tensor and sizes the arena, on the arena it fills it
struct Packer {
  fs2_handle* h; const Map& m; cudaStream_t st; Bump& bump; bool counting;
  Packer(fs2_handle* h_, const Map& m_, cudaStream_t s, Bump& b) : h(h_), m(m_), st(s), bump(b), counting(b.base == nullptr) {}

  int copy_into(const std::string& key, int64_t n, float* dst) {
    NEED(d, key);
    int64_t have = 1; for (int i = 0; i < d->ndim; ++i) have *= d->shape[i];
    if (have != n) { set_error("fs2_load_weights: '%s' has %lld elements, expected %lld", key.c_str(), (long long)have, (long long)n); return FS2_ERR_INVALID; }
    if (!counting) FS2_CUDA_CHECK(cudaMemcpyAsync(dst, d->data, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return FS2_OK;
  }
  int copy(const std::string& key, int64_t n, const float** out) {
    float* dst = bump.floats(n);
    *out = dst;
    return copy_into(key, n, dst);
  }
  // a [taps][N][K] weight with a bias [N], carved from the arena
  VWeight carve(int N, int K, int taps) {
    VWeight w; w.N = N; w.K = K; w.taps = taps;
    vweight_carve(bump, w, true);
    return w;
  }
  // w's rows from the Linear [N,K] (taps=1) or Conv1d [N,K,taps] wkey, times scale[n] when given, and its planes
  int fill(const std::string& wkey, VWeight& w, const float* scale = nullptr) {
    NEED(d, wkey);
    int64_t have = 1; for (int i = 0; i < d->ndim; ++i) have *= d->shape[i];
    if (have != (int64_t)w.N * w.K * w.taps) { set_error("fs2_load_weights: '%s' has %lld elements, expected %dx%dx%d", wkey.c_str(), (long long)have, w.N, w.K, w.taps); return FS2_ERR_INVALID; }
    if (counting) return FS2_OK;
    int rc = pack_conv_weight((const float*)d->data, w.N, w.K, w.taps, scale, w.w, st);
    return rc ? rc : vweight_planes(w, st);
  }
  int dense(const std::string& wkey, const std::string& bkey, int N, int K, int taps, VWeight* out) {
    *out = carve(N, K, taps);
    int rc = fill(wkey, *out);
    return rc ? rc : copy_into(bkey, N, out->bias);
  }
  // positional table [1, rows, C]: as many rows as the checkpoint tensor holds (the reference regenerates a longer table
  // on demand, core/embedding.py:48-66; the Python class does the same and the repack picks the new length up here)
  int pos_table(const std::string& key, int C, const float** out, int* rows) {
    NEED(d, key);
    int64_t have = 1; for (int i = 0; i < d->ndim; ++i) have *= d->shape[i];
    if (have <= 0 || have % C != 0) { set_error("fs2_load_weights: '%s' has %lld elements, not a multiple of %d", key.c_str(), (long long)have, C); return FS2_ERR_INVALID; }
    *rows = (int)(have / C);
    return copy(key, have, out);
  }
  int norm(const std::string& prefix, int C, float eps, Norm* out) {
    int rc;
    if ((rc = copy(prefix + "weight", C, &out->g))) return rc;
    if ((rc = copy(prefix + "bias", C, &out->b))) return rc;
    out->eps = eps;
    return FS2_OK;
  }
  int blocks(const std::string& prefix, int n, int C, int H, int kffn, std::vector<Block>* out) {
    out->assign(n, Block());
    for (int i = 0; i < n; ++i) {
      std::string p = prefix + ".encoders_." + std::to_string(i) + ".";
      Block& b = (*out)[i];
      // fused q|k|v: three [C,C] Linear weights stacked along N
      b.qkv = carve(3 * C, C, 1);
      const char* nm[3] = {"q", "k", "v"};
      for (int j = 0; j < 3; ++j) {
        NEED(w, p + "self_attn.linear_" + nm[j] + ".weight");
        NEED(bb, p + "self_attn.linear_" + nm[j] + ".bias");
        if (!counting) {
          FS2_CUDA_CHECK(cudaMemcpyAsync(b.qkv.w + (size_t)j * C * C, w->data, (size_t)C * C * sizeof(float), cudaMemcpyDeviceToDevice, st));
          FS2_CUDA_CHECK(cudaMemcpyAsync(b.qkv.bias + (size_t)j * C, bb->data, (size_t)C * sizeof(float), cudaMemcpyDeviceToDevice, st));
        }
      }
      int rc;
      if (!counting && (rc = vweight_planes(b.qkv, st))) return rc;
      if ((rc = dense(p + "self_attn.linear_out.weight", p + "self_attn.linear_out.bias", C, C, 1, &b.out))) return rc;
      if ((rc = dense(p + "feed_forward.w_1.weight", p + "feed_forward.w_1.bias", H, C, kffn, &b.w1))) return rc;
      if ((rc = dense(p + "feed_forward.w_2.weight", p + "feed_forward.w_2.bias", C, H, 1, &b.w2))) return rc;
      if ((rc = norm(p + "norm1.", C, 1e-5f, &b.ln1))) return rc;   // encoder.py:37-38
      if ((rc = norm(p + "norm2.", C, 1e-5f, &b.ln2))) return rc;
    }
    return FS2_OK;
  }
  int predictor(const std::string& prefix, Predictor* out) {
    const fs2_config& c = h->cfg;
    out->layers = c.pred_layers;
    for (int i = 0; i < c.pred_layers; ++i) {
      std::string p = prefix + "conv." + std::to_string(i) + ".";
      int rc;
      if ((rc = dense(p + "0.weight", p + "0.bias", c.pred_chans, i == 0 ? c.adim : c.pred_chans, c.pred_kernel, &out->conv[i]))) return rc;
      if ((rc = norm(p + "2.layer_norm.", c.pred_chans, 1e-12f, &out->ln[i]))) return rc;  // modules.py:115
    }
    int rc;
    if ((rc = copy(prefix + "linear.weight", c.pred_chans, &out->head_w))) return rc;
    return copy(prefix + "linear.bias", 1, &out->head_b);
  }

  int run() {
    const fs2_config& c = h->cfg;
    int rc;
    // encoder (fastspeech.py:65-84)
    if ((rc = copy("encoder.embed.0.weight", (int64_t)c.idim * c.adim, &h->emb))) return rc;
    if ((rc = copy("encoder.embed.1.alpha", 1, &h->enc_alpha))) return rc;
    if ((rc = pos_table("encoder.embed.1.pe", c.adim, &h->enc_pe, &h->enc_pe_len))) return rc;
    if ((rc = blocks("encoder", c.elayers, c.adim, c.eunits, c.ffn_kernel, &h->enc))) return rc;
    if ((rc = predictor("duration_predictor.", &h->dur))) return rc;
    if ((rc = predictor("energy_predictor.predictor.", &h->energy))) return rc;
    if ((rc = predictor("pitch_predictor.predictor.", &h->pitch))) return rc;
    if ((rc = copy("energy_predictor.energy_bins", c.n_bins - 1, &h->e_bins))) return rc;
    if ((rc = copy("pitch_predictor.pitch_bins", c.n_bins - 1, &h->p_bins))) return rc;
    // energy_embed / pitch_embed: Linear(n_bins -> adim) applied to a one-hot == column gather;
    // store W^T as a [bin][channel] table (fastspeech.py:102,113,218-219)
    {
      NEED(we, "energy_embed.weight"); NEED(wp, "pitch_embed.weight");
      float* te = bump.floats((size_t)c.n_bins * c.adim);
      float* tp = bump.floats((size_t)c.n_bins * c.adim);
      if (!counting) {
        if ((rc = pack_transpose((const float*)we->data, c.adim, c.n_bins, te, st))) return rc;
        if ((rc = pack_transpose((const float*)wp->data, c.adim, c.n_bins, tp, st))) return rc;
      }
      h->e_tab = te; h->p_tab = tp;
      if ((rc = copy("energy_embed.bias", c.adim, &h->e_tab_bias))) return rc;
      if ((rc = copy("pitch_embed.bias", c.adim, &h->p_tab_bias))) return rc;
    }
    // optional speaker table (multi-speaker models): n read off the tensor
    h->spk_table = nullptr; h->n_speakers = 0;
    if (const fs2_weight_desc* sp = find(m, "speaker_embed.weight")) {
      if (sp->ndim != 2 || sp->shape[0] < 1 || sp->shape[0] > INT32_MAX || sp->shape[1] != c.adim || sp->dtype != 0) {
        set_error("fs2_load_weights: 'speaker_embed.weight' must be float32 [n >= 1, adim=%d]", c.adim);
        return FS2_ERR_INVALID;
      }
      if ((rc = copy("speaker_embed.weight", sp->shape[0] * c.adim, &h->spk_table))) return rc;
      h->n_speakers = (int)sp->shape[0];
    }
    // optional speaker-embedding projection (DESIGN.md section 27): D read off the weight, the bias must come with it
    h->spemb_w = h->spemb_b = nullptr; h->spemb_dim = 0;
    {
      const fs2_weight_desc* pw = find(m, "spk_embed_proj.weight");
      const fs2_weight_desc* pb = find(m, "spk_embed_proj.bias");
      if (pw || pb) {
        if (!pw || !pb || pw->ndim != 2 || pw->shape[0] != c.adim || pw->shape[1] < 1 || pw->shape[1] > FS2_SPEMB_MAX_DIM ||
            pw->dtype != 0 || pb->ndim != 1 || pb->shape[0] != c.adim || pb->dtype != 0) {
          set_error("fs2_load_weights: 'spk_embed_proj.weight' [adim=%d, D in [1, %d]] and 'spk_embed_proj.bias' [adim] must "
                    "both be float32", c.adim, FS2_SPEMB_MAX_DIM);
          return FS2_ERR_INVALID;
        }
        if ((rc = copy("spk_embed_proj.weight", pw->shape[1] * c.adim, &h->spemb_w))) return rc;
        if ((rc = copy("spk_embed_proj.bias", c.adim, &h->spemb_b))) return rc;
        h->spemb_dim = (int)pw->shape[1];
      }
    }
    // decoder (fastspeech.py:119-136; input layer core/encoder.py:118-125)
    if ((rc = dense("decoder.embed.0.weight", "decoder.embed.0.bias", c.ddim, c.adim, 1, &h->dec_in))) return rc;
    if ((rc = norm("decoder.embed.1.", c.ddim, 1e-5f, &h->dec_in_ln))) return rc;
    if ((rc = copy("decoder.embed.4.alpha", 1, &h->dec_alpha))) return rc;
    if ((rc = pos_table("decoder.embed.4.pe", c.ddim, &h->dec_pe, &h->dec_pe_len))) return rc;
    if ((rc = blocks("decoder", c.dlayers, c.ddim, c.dunits, c.ffn_kernel, &h->dec))) return rc;
    if ((rc = dense("feat_out.weight", "feat_out.bias", c.odim, c.ddim, 1, &h->feat_out))) return rc;
    // Postnet: Conv1d(no bias) + BatchNorm1d(eval) folded into weight scale + bias (modules.py:283-348)
    h->postnet.assign(c.postnet_layers, VWeight());
    for (int i = 0; i < c.postnet_layers; ++i) {
      std::string p = "postnet.postnet." + std::to_string(i) + ".";
      int cin = i == 0 ? c.odim : c.postnet_chans;
      int cout = i == c.postnet_layers - 1 ? c.odim : c.postnet_chans;
      VWeight& w = h->postnet[i];
      w = carve(cout, cin, c.postnet_filts);
      float* scale = bump.floats(cout);
      NEED(g, p + "1.weight"); NEED(b, p + "1.bias"); NEED(mu, p + "1.running_mean"); NEED(var, p + "1.running_var");
      if (!counting && (rc = fold_batchnorm((const float*)g->data, (const float*)b->data, (const float*)mu->data,
                                            (const float*)var->data, 1e-5f, cout, scale, w.bias, st))) return rc;
      if ((rc = fill(p + "0.weight", w, scale))) return rc;
    }
    return FS2_OK;
  }
};

// Workspace layouts.  A tensor exists either as fp32 rows (fp32 / tf32 families) or as fp16 operand planes [2][rows][K]
// (plane families) -- the same bytes, so the two views alias one allocation.
struct EncodePlan { BlockBufs w; float *t1, *t2; __half* t2p; float* v; };
// spemb: the handle has a speaker-embedding projection, whose per-utterance vectors v [B, adim] then live here too
EncodePlan plan_encode(const fs2_config& c, Bump& b, int B, int T, bool spemb) {
  const int64_t rows = (int64_t)B * T;
  EncodePlan p;
  p.w.x = b.floats(rows * c.adim); p.w.y = b.floats(rows * c.adim);
  p.w.xp = (__half*)b.floats(rows * c.adim);
  p.w.qkv = b.floats(rows * 3 * c.adim); p.w.qkp = (__half*)p.w.qkv;
  p.w.vt = b.floats((int64_t)B * c.adim * round8(T)); p.w.vtp = (__half*)p.w.vt;
  p.w.ctx = b.floats(rows * c.adim); p.w.ctxp = (__half*)p.w.ctx;
  p.w.hid = b.floats(rows * c.eunits); p.w.hidp = (__half*)p.w.hid;
  p.t1 = b.floats(rows * c.pred_chans); p.t2 = b.floats(rows * c.pred_chans); p.t2p = (__half*)p.t2;
  p.v = spemb ? b.floats((int64_t)B * c.adim) : nullptr;
  return p;
}
struct DecodePlan { BlockBufs w; float *hm2, *t1, *t2, *q1, *q2; __half *hmp, *hm2p, *t2p, *beforep; };
DecodePlan plan_decode(const fs2_config& c, Bump& b, int B, int L) {
  const int64_t rows = (int64_t)B * L;
  DecodePlan p;
  p.hmp = (__half*)b.floats(rows * c.adim);                          // planes of the length-regulated states (predictor input)
  p.hm2 = b.floats(rows * c.adim); p.hm2p = (__half*)p.hm2;
  p.w.x = b.floats(rows * c.ddim); p.w.y = b.floats(rows * c.ddim);
  p.w.xp = (__half*)b.floats(rows * c.ddim);
  p.w.qkv = b.floats(rows * 3 * c.ddim); p.w.qkp = (__half*)p.w.qkv;
  p.w.vt = b.floats((int64_t)B * c.ddim * round8(L)); p.w.vtp = (__half*)p.w.vt;
  p.w.ctx = b.floats(rows * c.ddim); p.w.ctxp = (__half*)p.w.ctx;
  p.w.hid = b.floats(rows * c.dunits); p.w.hidp = (__half*)p.w.hid;
  p.t1 = b.floats(rows * c.pred_chans); p.t2 = b.floats(rows * c.pred_chans); p.t2p = (__half*)p.t2;
  p.q1 = b.floats(rows * c.postnet_chans); p.q2 = b.floats(rows * c.postnet_chans);
  p.beforep = (__half*)b.floats(rows * c.odim);
  return p;
}

// the RowNorm of an fs2_row_norm_desc (the header's copy of its fields) plus a per-utterance vector
RowNorm row_norm_of(const fs2_row_norm_desc& d, const float* spk_vec) {
  RowNorm r;
  r.x = d.x; r.ldx = d.ldx; r.resid = d.resid; r.ldr = d.ldr; r.gamma = d.gamma; r.beta = d.beta; r.eps = d.eps;
  r.rows = d.rows; r.C = d.C; r.out = d.out; r.ldo = d.ldo; r.relu_after = d.relu_after;
  r.pe = d.pe; r.alpha = d.alpha; r.L = d.L;
  r.head_w = d.head_w; r.head_b = d.head_b; r.head_out = d.head_out; r.dur_out = d.dur_out; r.head_scale = d.head_scale;
  r.lens = d.lens; r.split_out = reinterpret_cast<__half*>(d.split_out); r.split_lo = d.split_lo;
  r.spk_table = d.spk_table; r.spk = d.spk; r.n_spk = d.n_spk; r.spk_L = d.spk_L;
  r.spk_vec = spk_vec;
  return r;
}

}  // namespace
}  // namespace fs2

using namespace fs2;

extern "C" {

const char* fs2_last_error(void) { return g_err; }
const char* fs2_version(void) { return "fs2-b200 0.3 sm_90a"; }
unsigned long long fs2_kernel_launches(void) { return g_kernel_launches.load(); }

int fs2_create(fs2_handle** out, const fs2_config* cfg, int device) {
  FS2_REQUIRE(out && cfg, "fs2_create: null argument");
  FS2_REQUIRE(cfg->aheads > 0 && cfg->adim % cfg->aheads == 0 && cfg->ddim % cfg->aheads == 0, "fs2_create: dims not divisible by heads");
  FS2_REQUIRE((cfg->adim == 256 || cfg->adim == 384) && (cfg->ddim == 256 || cfg->ddim == 384),
              "fs2_create: adim/ddim must be 256 or 384 (got %d/%d); kernels are specialised for configs/default.yaml", cfg->adim, cfg->ddim);
  FS2_REQUIRE(cfg->pred_chans == 256 || cfg->pred_chans == 384, "fs2_create: predictor channels must be 256 or 384");
  FS2_REQUIRE(cfg->pred_layers >= 1 && cfg->pred_layers <= 4, "fs2_create: 1..4 predictor layers");
  FS2_REQUIRE(cfg->eunits % 16 == 0 && cfg->dunits % 16 == 0 && cfg->odim % 16 == 0 && cfg->postnet_chans % 16 == 0, "fs2_create: channel counts must be multiples of 16");
  FS2_REQUIRE((cfg->ffn_kernel & 1) && (cfg->pred_kernel & 1) && (cfg->postnet_filts & 1), "fs2_create: kernel sizes must be odd");
  FS2_REQUIRE(cfg->postnet_layers >= 1, "fs2_create: postnet_layers == 0 is not supported");
  FS2_REQUIRE(cfg->n_bins % 4 == 0, "fs2_create: n_bins must be a multiple of 4");
  FS2_REQUIRE(cfg->math_mode >= FS2_MATH_FP32 && cfg->math_mode <= FS2_MATH_F16, "fs2_create: bad math_mode");
  int n_dev = 0;
  FS2_CUDA_CHECK(cudaGetDeviceCount(&n_dev));
  FS2_REQUIRE(device >= 0 && device < n_dev, "fs2_create: device %d out of range (%d visible)", device, n_dev);
  fs2_handle* h = new fs2_handle();
  h->cfg = *cfg;
  h->device = device;
  *out = h;
  return FS2_OK;
}

void fs2_destroy(fs2_handle* h) {
  if (!h) return;
  if (t_prof == &h->prof) t_prof = nullptr;   // the single-operator entries must not record into a destroyed handle's profiler
  {
    DeviceGuard guard(h->device);
    if (h->arena) cudaFree(h->arena);
  }
  delete h;
}

int fs2_profile_enable(fs2_handle* h, int on) {
  FS2_REQUIRE(h, "fs2_profile_enable: null handle");
  h->prof.on = on != 0;
  return FS2_OK;
}
int fs2_profile_classes(void) { return P_COUNT; }
const char* fs2_profile_label(int i) { return i >= 0 && i < P_COUNT ? kProfLabels[i] : ""; }
int fs2_profile_read(fs2_handle* h, double* ms, int64_t* launches, double* flop, double* bytes) {
  FS2_REQUIRE(h && ms && launches && flop && bytes, "fs2_profile_read: null argument");
  FS2_DEVICE_GUARD(h);
  for (int i = 0; i < P_COUNT; ++i) { ms[i] = 0; launches[i] = 0; flop[i] = 0; bytes[i] = 0; }
  for (ProfRec& r : h->prof.recs) {
    FS2_CUDA_CHECK(cudaEventSynchronize(r.b));
    float t = 0.f;
    FS2_CUDA_CHECK(cudaEventElapsedTime(&t, r.a, r.b));
    ms[r.cls] += t; launches[r.cls] += 1; flop[r.cls] += r.flop; bytes[r.cls] += r.bytes;
    cudaEventDestroy(r.a); cudaEventDestroy(r.b);
  }
  h->prof.recs.clear();
  return FS2_OK;
}

int fs2_set_math_mode(fs2_handle* h, int math_mode) {
  FS2_REQUIRE(h, "fs2_set_math_mode: null handle");
  FS2_REQUIRE(math_mode >= FS2_MATH_FP32 && math_mode <= FS2_MATH_F16, "fs2_set_math_mode: bad mode %d", math_mode);
  h->cfg.math_mode = math_mode;
  return FS2_OK;
}

int fs2_load_weights(fs2_handle* h, const fs2_weight_desc* w, int n, void* stream) {
  FS2_REQUIRE(h && w && n > 0, "fs2_load_weights: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  FS2_DEVICE_GUARD(h);
  Map m;
  for (int i = 0; i < n; ++i) {
    FS2_REQUIRE(w[i].name && w[i].data, "fs2_load_weights: entry %d has a null name/data", i);
    m[w[i].name] = &w[i];
  }
  h->loaded = false;
  int rc = arena_carve(&h->arena, &h->arena_bytes, st, [&](Bump& b) { return Packer(h, m, st, b).run(); });
  if (rc) return rc;
  h->loaded = true;
  return FS2_OK;
}

int fs2_workspace_bytes(fs2_handle* h, int B, int Tmax, int Lmax, size_t* out) {
  FS2_REQUIRE(h && out && B >= 0 && Tmax >= 0 && Lmax >= 0, "fs2_workspace_bytes: bad argument");
  Bump e(nullptr, 0), d(nullptr, 0);
  plan_encode(h->cfg, e, B, Tmax, h->spemb_w != nullptr);
  plan_decode(h->cfg, d, B, Lmax);
  *out = (e.off > d.off ? e.off : d.off) + 1024;
  return FS2_OK;
}

int fs2_encode(fs2_handle* h, const int64_t* xs, const int64_t* ilens, int B, int Tmax, float* hs, float* d_log,
               int64_t* d_int, void* ws, size_t ws_bytes, void* stream) {
  return fs2_encode_ex(h, xs, ilens, B, Tmax, hs, d_log, d_int, ws, ws_bytes, 0, stream);
}

int fs2_encode_ex(fs2_handle* h, const int64_t* xs, const int64_t* ilens, int B, int Tmax, float* hs, float* d_log,
                  int64_t* d_int, void* ws, size_t ws_bytes, int flags, void* stream) {
  return fs2_encode_spk(h, xs, ilens, nullptr, B, Tmax, hs, d_log, d_int, ws, ws_bytes, flags, stream);
}

int fs2_encode_spk(fs2_handle* h, const int64_t* xs, const int64_t* ilens, const int64_t* spk, int B, int Tmax, float* hs,
                   float* d_log, int64_t* d_int, void* ws, size_t ws_bytes, int flags, void* stream) {
  return fs2_encode_spemb(h, xs, ilens, spk, nullptr, 0, B, Tmax, hs, d_log, d_int, ws, ws_bytes, flags, nullptr, nullptr, stream);
}

int fs2_encode_spemb(fs2_handle* h, const int64_t* xs, const int64_t* ilens, const int64_t* spk, const float* spembs, int D, int B,
                     int Tmax, float* hs, float* d_log, int64_t* d_int, void* ws, size_t ws_bytes, int flags, int32_t* bad,
                     int32_t* status, void* stream) {
  FS2_REQUIRE(h && xs && ilens && hs && ws, "fs2_encode: null argument");
  FS2_REQUIRE((flags & ~FS2_PER_UTTERANCE) == 0, "fs2_encode_ex: unknown flags 0x%x", flags);
  if (!h->loaded) { set_error("fs2_encode: weights not loaded"); return FS2_ERR_NOT_LOADED; }
  FS2_REQUIRE(!h->spk_table || spk, "fs2_encode: the model has a speaker table (%d speakers): pass speaker ids (fs2_encode_spk)",
              h->n_speakers);
  FS2_REQUIRE(h->spk_table || !spk, "fs2_encode_spk: speaker ids given but the model has no speaker table");
  FS2_REQUIRE(!h->spemb_w || spembs, "fs2_encode: the model has a speaker-embedding projection (D=%d): pass spembs "
              "(fs2_encode_spemb)", h->spemb_dim);
  FS2_REQUIRE(h->spemb_w || !spembs, "fs2_encode_spemb: speaker embeddings given but the model has no projection "
              "(spk_embed_proj)");
  FS2_REQUIRE(!spembs || D == h->spemb_dim, "fs2_encode_spemb: D=%d but the loaded projection takes D=%d", D, h->spemb_dim);
  FS2_REQUIRE(Tmax <= h->enc_pe_len, "fs2_encode: Tmax=%d exceeds the positional table (%d rows)", Tmax, h->enc_pe_len);
  FS2_DEVICE_GUARD(h);
  cudaStream_t st = (cudaStream_t)stream;
  const fs2_config& c = h->cfg;
  t_prof = &h->prof;
  Bump b(ws, ws_bytes);
  EncodePlan p = plan_encode(c, b, B, Tmax, h->spemb_w != nullptr);
  int rc = b.check("fs2_encode");
  if (rc) return rc;
  // the encoder's output feeds round() in the duration predictor: exact fp32 FMA in FS2_MATH_FP32,
  // error-compensated 3xF16 on the tensor cores in every other mode (never a plain 10-bit-mantissa product)
  const bool planes = c.math_mode != FS2_MATH_FP32;
  const int64_t* zlens = (flags & FS2_PER_UTTERANCE) ? ilens : nullptr;
  { ProfScope prof_scope(P_EMBED, 0, (planes ? 12.0 : 8.0) * B * Tmax * c.adim, st);
    if ((rc = embed_posenc(xs, h->emb, c.idim, h->enc_pe, h->enc_alpha, B, Tmax, c.adim, p.w.x, planes ? p.w.xp : nullptr, zlens, st))) return rc; }
  float* enc_out = nullptr;
  SpeakerAdd sa;
  sa.table = h->spk_table; sa.ids = spk; sa.n = h->n_speakers;
  if (spembs) {
    if ((rc = spemb_project(h->spemb_w, h->spemb_b, spembs, B, D, c.adim, p.v, nullptr, bad, status, st))) return rc;
    sa.vec = p.v;
  }
  if ((rc = run_blocks(h->enc, p.w, ilens, zlens, B, Tmax, c.adim, c.aheads, planes ? MATH_3XTF32 : FS2_MATH_FP32, false, st,
                       &enc_out, sa))) return rc;
  FS2_CUDA_CHECK(cudaMemcpyAsync(hs, enc_out, (size_t)B * Tmax * c.adim * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if (d_log || d_int)
    if ((rc = run_predictor(h->dur, enc_out, planes ? p.w.xp : nullptr, c.adim, B, Tmax, p.t1, p.t2, p.t2p, ilens, zlens, d_log, d_int, nullptr, st))) return rc;
  return FS2_OK;
}

int fs2_length_plan(void* ds, int ds_dtype, const int64_t* ilens, float alpha, int B, int Tmax, int mutate_ds,
                    int32_t* cum, int64_t* olens, int64_t* stats, void* stream) {
  return fs2_length_plan_ex(ds, ds_dtype, ilens, alpha, nullptr, B, Tmax, mutate_ds, cum, olens, stats, nullptr, stream);
}

int fs2_length_plan_ex(void* ds, int ds_dtype, const int64_t* ilens, float alpha, const float* alpha_v, int B, int Tmax,
                       int mutate_ds, int32_t* cum, int64_t* olens, int64_t* stats, int64_t* d_used, void* stream) {
  FS2_REQUIRE(ds && ilens && cum && olens && stats, "fs2_length_plan: null argument");
  return length_plan(ds, ds_dtype, ilens, alpha, alpha_v, B, Tmax, mutate_ds, cum, olens, stats, d_used, (cudaStream_t)stream);
}

int fs2_length_gather(const float* hs, const int32_t* cum, const int64_t* ilens, int B, int Tmax, int C, float* out,
                      int Lcap, void* stream) {
  return fs2_length_gather_ex(hs, cum, ilens, B, Tmax, C, out, Lcap, nullptr, nullptr, stream);
}

int fs2_length_gather_ex(const float* hs, const int32_t* cum, const int64_t* ilens, int B, int Tmax, int C, float* out,
                         int Lcap, const float* fac_in, float* fac_out, void* stream) {
  FS2_REQUIRE(hs && cum && ilens && (out || Lcap == 0), "fs2_length_gather: null argument");
  return length_gather(hs, cum, ilens, B, Tmax, C, out, Lcap, fac_in, fac_out, (cudaStream_t)stream);
}

int fs2_length_plan_cap(const void* ds, int ds_dtype, const int64_t* ilens, const float* alpha_v, const float* fac, int B,
                        int Tmax, int64_t Lc, int32_t* cum, int64_t* olens, int64_t* need, int64_t* d_used, int32_t* status,
                        void* stream) {
  return fs2_length_plan_cap_spk(ds, ds_dtype, ilens, alpha_v, fac, nullptr, 0, B, Tmax, Lc, cum, olens, need, d_used, status,
                                 stream);
}

int fs2_length_plan_cap_spk(const void* ds, int ds_dtype, const int64_t* ilens, const float* alpha_v, const float* fac,
                            const int64_t* spk, int n_speakers, int B, int Tmax, int64_t Lc, int32_t* cum, int64_t* olens,
                            int64_t* need, int64_t* d_used, int32_t* status, void* stream) {
  return fs2_length_plan_cap_spemb(ds, ds_dtype, ilens, alpha_v, fac, spk, n_speakers, nullptr, B, Tmax, Lc, cum, olens, need,
                                   d_used, status, stream);
}

int fs2_length_plan_cap_spemb(const void* ds, int ds_dtype, const int64_t* ilens, const float* alpha_v, const float* fac,
                              const int64_t* spk, int n_speakers, const int32_t* spemb_bad, int B, int Tmax, int64_t Lc,
                              int32_t* cum, int64_t* olens, int64_t* need, int64_t* d_used, int32_t* status, void* stream) {
  FS2_REQUIRE(ds && ilens && cum && olens && need && status, "fs2_length_plan_cap: null argument");
  FS2_REQUIRE(!spk || n_speakers >= 1, "fs2_length_plan_cap_spk: speaker ids need n_speakers >= 1 (got %d)", n_speakers);
  FS2_REQUIRE(B >= 1 && Tmax >= 1, "fs2_length_plan_cap: B=%d and Tmax=%d must be >= 1", B, Tmax);
  FS2_REQUIRE(Lc >= 1 && Lc <= INT32_MAX, "fs2_length_plan_cap: capacity Lc=%lld must lie in [1, %d] (the prefix sum is int32)",
              (long long)Lc, INT32_MAX);
  return length_plan_cap(ds, ds_dtype, ilens, alpha_v, fac, spk, n_speakers, spemb_bad, B, Tmax, (long)Lc, cum, olens, need, d_used,
                         status, (cudaStream_t)stream);
}

int fs2_synth_status(const int32_t* plan_status, const int32_t* voc_status, const int64_t* olens, int B, int hop,
                     int32_t* word, int64_t* alens, void* stream) {
  FS2_REQUIRE(plan_status && olens && word, "fs2_synth_status: null argument");
  FS2_REQUIRE(B >= 1 && hop >= 1, "fs2_synth_status: B=%d and hop=%d must be >= 1", B, hop);
  return synth_status(plan_status, voc_status, olens, B, hop, word, alens, (cudaStream_t)stream);
}

int fs2_decode(fs2_handle* h, const float* hm, const int64_t* olens, const float* es, const float* ps, int B, int L,
               float* before, float* after, float* e_out, float* p_out, int64_t* e_ids, int64_t* p_ids, void* ws,
               size_t ws_bytes, void* stream) {
  return fs2_decode_ex(h, hm, olens, es, ps, B, L, before, after, e_out, p_out, e_ids, p_ids, ws, ws_bytes, 0, stream);
}

int fs2_decode_ex(fs2_handle* h, const float* hm, const int64_t* olens, const float* es, const float* ps, int B, int L,
                  float* before, float* after, float* e_out, float* p_out, int64_t* e_ids, int64_t* p_ids, void* ws,
                  size_t ws_bytes, int flags, void* stream) {
  return fs2_decode_ctl(h, hm, olens, es, ps, B, L, before, after, e_out, p_out, e_ids, p_ids, nullptr, nullptr, ws, ws_bytes,
                        flags, stream);
}

int fs2_decode_ctl(fs2_handle* h, const float* hm, const int64_t* olens, const float* es, const float* ps, int B, int L,
                   float* before, float* after, float* e_out, float* p_out, int64_t* e_ids, int64_t* p_ids,
                   const float* e_scale, const float* p_scale, void* ws, size_t ws_bytes, int flags, void* stream) {
  FS2_REQUIRE(h && hm && before && after && e_out && p_out && ws, "fs2_decode: null argument");
  FS2_REQUIRE((es == nullptr) == (ps == nullptr), "fs2_decode: es and ps must both be given or both be NULL");
  FS2_REQUIRE(!(e_scale || p_scale) || !es, "fs2_decode_ctl: e_scale / p_scale scale predicted values; with es / ps given there are none");
  FS2_REQUIRE((flags & ~FS2_PER_UTTERANCE) == 0, "fs2_decode_ex: unknown flags 0x%x", flags);
  FS2_REQUIRE(!(flags & FS2_PER_UTTERANCE) || olens, "fs2_decode_ex: FS2_PER_UTTERANCE needs olens");
  if (!h->loaded) { set_error("fs2_decode: weights not loaded"); return FS2_ERR_NOT_LOADED; }
  FS2_REQUIRE(L <= h->dec_pe_len, "fs2_decode: L=%d exceeds the positional table (%d rows)", L, h->dec_pe_len);
  FS2_DEVICE_GUARD(h);
  cudaStream_t st = (cudaStream_t)stream;
  const fs2_config& c = h->cfg;
  const int64_t rows = (int64_t)B * L;
  t_prof = &h->prof;
  Bump b(ws, ws_bytes);
  DecodePlan p = plan_decode(c, b, B, L);
  int rc = b.check("fs2_decode");
  if (rc) return rc;
  const int mode = c.math_mode;
  const bool pred_planes = mode != FS2_MATH_FP32;                              // predictors: 3xF16 in every tensor-core mode
  const bool dec_planes = plane_mode(mode);                                    // decoder side on operand planes
  const bool x3 = mode == FS2_MATH_3XTF32;
  const int64_t* zlens = (flags & FS2_PER_UTTERANCE) ? olens : nullptr;   // hm rows past olens are zero (length_gather)
  // energy / pitch predictors on the length-regulated states (fastspeech.py:195-196,214-216); fp32-class.  hm enters the
  // library as fp32 rows (the LengthRegulator is its own ABI stage), so this is the one operand pre-pass left in a step
  if (pred_planes) {
    ProfScope prof_scope(P_ROWNORM, 0, 8.0 * rows * c.adim, st);
    if ((rc = split_rows(hm, c.adim, rows, c.adim, p.hmp, st))) return rc;
  }
  if ((rc = run_predictor(h->energy, hm, pred_planes ? p.hmp : nullptr, c.adim, B, L, p.t1, p.t2, p.t2p, olens, zlens, e_out, nullptr, e_scale, st))) return rc;
  if ((rc = run_predictor(h->pitch, hm, pred_planes ? p.hmp : nullptr, c.adim, B, L, p.t1, p.t2, p.t2p, olens, zlens, p_out, nullptr, p_scale, st))) return rc;
  // hs + pitch_embed(one_hot) + energy_embed(one_hot) (fastspeech.py:218-219); plane families: straight to the decoder
  // input Linear's operand planes
  { ProfScope prof_scope(P_VAR_EMBED, 0, 4.0 * rows * c.adim * 4, st);
  if ((rc = variance_embed_add(hm, es ? es : e_out, ps ? ps : p_out, h->e_bins, h->p_bins, c.n_bins - 1, h->e_tab,
                               h->e_tab_bias, h->p_tab, h->p_tab_bias, rows, c.adim, dec_planes ? nullptr : p.hm2,
                               dec_planes ? p.hm2p : nullptr, x3, e_ids, p_ids, zlens, L, st))) return rc; }
  // decoder input layer: Linear -> LayerNorm -> ReLU -> x + alpha*pe (core/encoder.py:118-125)
  {
    if ((rc = dense(vweight_gemm_args(mode, h->dec_in, operand(mode, p.hm2, p.hm2p), B, L, ACT_NONE, zlens, p.w.y), mode, st,
                    P_DEC_IN))) return rc;
    RowNorm r = masked(make_norm(h->dec_in_ln, p.w.y, c.ddim, rows, c.ddim, p.w.x, c.ddim), zlens, L);
    r.relu_after = 1; r.pe = h->dec_pe; r.alpha = h->dec_alpha; r.L = L;
    if (dec_planes) { r.split_out = p.w.xp; r.split_lo = x3; }    // first block's q|k|v reads the planes
    if ((rc = norm_rows(r, st))) return rc;
  }
  float* dec_out = nullptr;
  if ((rc = run_blocks(h->dec, p.w, olens, zlens, B, L, c.ddim, c.aheads, mode, true, st, &dec_out))) return rc;
  // mel linear (fastspeech.py:228-230); plane families: from the planes of the last block's output, and the Postnet
  // chain stays in planes until the final residual layer
  if ((rc = dense(vweight_gemm_args(mode, h->feat_out, operand(mode, dec_out, p.w.xp), B, L, ACT_NONE, zlens, before, nullptr, 1,
                                    p.beforep), mode, st, P_FEAT_OUT))) return rc;
  // Postnet + residual (fastspeech.py:236-238, modules.py:350-359)
  const float* cur = before;
  const __half* cur_p = p.beforep;
  float* pp[2] = {p.q1, p.q2};
  for (int i = 0; i < c.postnet_layers; ++i) {
    const bool last = i == c.postnet_layers - 1;
    float* dst = last ? after : pp[i & 1];
    // plane families: the inner layers write only the planes the next one reads
    TapGemm g = vweight_gemm_args(mode, h->postnet[i], operand(mode, cur, cur_p), B, L, last ? ACT_NONE : ACT_TANH, zlens,
                                  dec_planes && !last ? nullptr : dst, last ? before : nullptr, 1,
                                  last ? nullptr : reinterpret_cast<__half*>(dst));
    if ((rc = dense(g, mode, st, P_POSTNET))) return rc;
    cur = dst; cur_p = reinterpret_cast<const __half*>(dst);
  }
  return FS2_OK;
}

int fs2_masked_losses(const float* before, const float* after, const float* ys, int ld_ys_time, const float* d_out,
                      const void* ds, int ds_dtype, const float* e_out, const float* p_out, const float* es,
                      const float* ps, const int64_t* ilens, const int64_t* olens, int B, int Tmax, int L, int odim,
                      float* out7, void* scratch, void* stream) {
  FS2_REQUIRE(before && after && ys && d_out && ds && e_out && p_out && es && ps && ilens && olens && out7 && scratch,
              "fs2_masked_losses: null argument");
  return masked_losses(before, after, ys, ld_ys_time, d_out, ds, ds_dtype, e_out, p_out, es, ps, ilens, olens, B, Tmax, L,
                       odim, out7, scratch, (cudaStream_t)stream);
}

int fs2_bucketize(const float* vals, const float* bins, int n_edges, int64_t n, int64_t* ids, void* stream) {
  FS2_REQUIRE(vals && bins && ids, "fs2_bucketize: null argument");
  return bucketize(vals, bins, n_edges, n, ids, (cudaStream_t)stream);
}
int fs2_one_hot(const int64_t* ids, int64_t n, int n_bins, float* out, void* stream) {
  FS2_REQUIRE(ids && out, "fs2_one_hot: null argument");
  return one_hot(ids, n, n_bins, out, (cudaStream_t)stream);
}

namespace {
// single-operator entries (tests): the weight [taps][N][K] at the caller's pointer; in the plane families the operand planes
// of x and the weight's scale and planes are made on the fly in a stream-ordered temporary, layout
// [x planes 2*nx][w hi nw][w lo nw][scale, inv]
struct TempPlanes {
  __half* base = nullptr; __half* xp = nullptr; VWeight w; cudaStream_t st;
  TempPlanes(const float* w_, const float* bias, int N, int K, int taps) {
    w.w = const_cast<float*>(w_); w.bias = const_cast<float*>(bias); w.N = N; w.K = K; w.taps = taps;
  }
  int make(const float* x, long rows, cudaStream_t s) {
    st = s;
    const size_t nx = (size_t)rows * w.K, nw = (size_t)w.taps * w.N * w.K;
    const size_t nx8 = (2 * nx + 15) & ~(size_t)15, nw8 = (nw + 15) & ~(size_t)15;
    FS2_CUDA_CHECK(cudaMallocAsync(&base, (nx8 + 2 * nw8) * sizeof(__half) + 64, st));
    xp = base; w.hi = base + nx8; w.lo = w.hi + nw8; w.sc = reinterpret_cast<float*>(w.lo + nw8);
    int rc = split_rows(x, w.K, rows, w.K, xp, st);
    return rc ? rc : vweight_planes(w, st);
  }
  ~TempPlanes() { if (base) cudaFreeAsync(base, st); }
};
}  // namespace

int fs2_op_tap_gemm(int math_mode, const float* x, int B, int L, int K, const float* w, const float* bias, int N, int taps,
                    int act, const float* resid, float* out, void* stream) {
  return fs2_op_tap_gemm_ex(math_mode, x, B, L, K, w, bias, N, taps, act, resid, nullptr, out, nullptr, 0, 0, nullptr, 0,
                            stream);
}
int fs2_op_tap_gemm_ex(int math_mode, const float* x, int B, int L, int K, const float* w, const float* bias, int N,
                       int taps, int act, const float* resid, const int64_t* lens, float* out, void* out_planes,
                       int vt_col0, int vt_heads, void* vt, int vt_lpad, void* stream) {
  return fs2_op_tap_gemm_dil(math_mode, x, B, L, K, w, bias, N, taps, act, resid, lens, out, out_planes, vt_col0, vt_heads, vt,
                             vt_lpad, 1, stream);
}
int fs2_op_tap_gemm_dil(int math_mode, const float* x, int B, int L, int K, const float* w, const float* bias, int N,
                        int taps, int act, const float* resid, const int64_t* lens, float* out, void* out_planes,
                        int vt_col0, int vt_heads, void* vt, int vt_lpad, int dil, void* stream) {
  const char* who = "fs2_op_tap_gemm";
  FS2_REQUIRE(math_mode == FS2_MATH_FP32 || math_mode == FS2_MATH_TF32 || math_mode == FS2_MATH_F16 || math_mode == FS2_MATH_3XTF32,
              "%s: unknown math mode %d", who, math_mode);
  const bool planes = plane_mode(math_mode);
  FS2_REQUIRE(x && w && (out || (planes && (out_planes || vt))), "%s: null argument", who);
  FS2_REQUIRE(B >= 0 && L >= 0 && K > 0 && N > 0 && taps > 0, "%s: bad shape B=%d L=%d K=%d N=%d taps=%d", who, B, L, K, N, taps);
  // tap rows t + (j - pad) * dil are int32 row coordinates: keep them in range (dil = 1 is the undilated call, as before)
  FS2_REQUIRE(dil == 1 || (dil > 1 && (long)dil * ((taps - 1) / 2) + L < (1L << 30)),
              "%s: need dil >= 1 and dil * (taps - 1) / 2 + L < 2^30 (got dil=%d taps=%d L=%d)", who, dil, taps, L);
  FS2_REQUIRE(!out_planes || planes, "%s: out_planes needs FS2_MATH_F16 or FS2_MATH_3XTF32", who);
  FS2_REQUIRE(!vt || math_mode != FS2_MATH_FP32, "%s: the fp32 family has no transposed V output", who);
  FS2_REQUIRE(!vt || (vt_heads > 0 && vt_col0 >= 0 && vt_col0 < N && (N - vt_col0) % vt_heads == 0 && vt_lpad >= L),
              "%s: transposed V needs 0 <= vt_col0 < N, heads dividing N - vt_col0 and vt_lpad >= L", who);
  cudaStream_t st = (cudaStream_t)stream;
  TempPlanes t(w, bias, N, K, taps);
  if (planes) { int rc = t.make(x, (long)B * L, st); if (rc) return rc; }
  TapGemm g = vweight_gemm_args(math_mode, t.w, operand(math_mode, x, t.xp), B, L, act, lens, out, resid, dil,
                                reinterpret_cast<__half*>(out_planes));
  if (vt) {
    g.vt_col0 = vt_col0; g.vt_heads = vt_heads; g.vt_dk = (N - vt_col0) / vt_heads; g.vt_lpad = vt_lpad;
    if (planes) g.vtp = reinterpret_cast<__half*>(vt); else g.vt_out = reinterpret_cast<float*>(vt);
    g.outp_lo = g.precise;   // the lo flag covers vt's lo plane too
  }
  return dense(g, math_mode, st, P_DEC_W1);
}
int fs2_op_gemm_layernorm(int math_mode, const float* x, int64_t rows, int K, int N, const float* w, const float* bias, const float* resid,
                          const float* gamma, const float* beta, float eps, float* out, float* out_planes, void* stream) {
  FS2_REQUIRE(x && w && gamma && beta && out, "fs2_op_gemm_layernorm: null argument");
  FS2_REQUIRE(rows < (1LL << 31), "fs2_op_gemm_layernorm: too many rows");
  FS2_REQUIRE(math_mode == FS2_MATH_TF32 || math_mode == FS2_MATH_F16 || math_mode == FS2_MATH_3XTF32,
              "fs2_op_gemm_layernorm: tensor-core modes only (FS2_MATH_TF32, FS2_MATH_F16, FS2_MATH_3XTF32)");
  FS2_REQUIRE(N == 384 || (N == 256 && math_mode != FS2_MATH_TF32), "fs2_op_gemm_layernorm: N must be 384 (or 256 in the plane families)");
  cudaStream_t st = (cudaStream_t)stream;
  FS2_REQUIRE(!out_planes || math_mode != FS2_MATH_TF32, "fs2_op_gemm_layernorm: the tf32 variant has no plane output in this entry");
  // y = x w^T + bias + resid on the tensor cores, then the row LayerNorm (which also writes the operand planes)
  float* y = nullptr;
  __half* op = nullptr;
  FS2_CUDA_CHECK(cudaMallocAsync(&y, (size_t)rows * N * sizeof(float) + 64, st));
  TempPlanes t(w, bias, N, K, 1);
  int rc = plane_mode(math_mode) ? t.make(x, (long)rows, st) : FS2_OK;
  if (!rc)
    rc = dense(vweight_gemm_args(math_mode, t.w, operand(math_mode, x, t.xp), 1, (int)rows, ACT_NONE, nullptr, y, resid), math_mode,
               st, P_DEC_OUT);
  Norm n; n.g = gamma; n.b = beta; n.eps = eps;
  RowNorm r = make_norm(n, y, N, rows, N, out, N);
  // optional: the result's operand planes (what the next contraction would read), returned as fp32 = (hi + lo) / kPlaneScale
  if (!rc && out_planes) {
    if (cudaMallocAsync(&op, (size_t)2 * rows * N * sizeof(__half) + 64, st) != cudaSuccess ||
        cudaMemsetAsync(op, 0, (size_t)2 * rows * N * sizeof(__half), st) != cudaSuccess) {
      set_error("fs2_op_gemm_layernorm: plane buffer allocation failed");
      rc = FS2_ERR_CUDA;
    }
    r.split_out = op; r.split_lo = math_mode == MATH_3XTF32;
  }
  if (!rc) rc = norm_rows(r, st);
  if (!rc && op) rc = planes_to_rows(op, (long)rows * N, out_planes, st);
  if (op) cudaFreeAsync(op, st);
  cudaFreeAsync(y, st);
  return rc;
}
int fs2_op_attention(int math_mode, const float* qkv, const int64_t* lens, int B, int L, int C, int heads, float* ctx,
                     void* stream) {
  FS2_REQUIRE(math_mode == FS2_MATH_FP32 || math_mode == FS2_MATH_TF32 || math_mode == FS2_MATH_F16 || math_mode == FS2_MATH_3XTF32,
              "fs2_op_attention: unknown math mode %d", math_mode);
  FS2_REQUIRE(qkv && ctx, "fs2_op_attention: null argument");
  FS2_REQUIRE(heads > 0 && C % heads == 0, "fs2_op_attention: C=%d not divisible by heads=%d", C, heads);
  cudaStream_t st = (cudaStream_t)stream;
  const double flop = 4.0 * B * (double)L * L * C, bytes = 4.0 * 4.0 * B * (double)L * C;
  if (math_mode == FS2_MATH_FP32) { ProfScope prof_scope(P_DEC_ATTN, flop, bytes, st); return attention_fp32(qkv, lens, B, L, C, heads, ctx, st); }
  if (math_mode == FS2_MATH_TF32) {
    // single-operator entry (tests): build the transposed V the projection epilogue normally provides
    float* vt = nullptr;
    const int lpad = round4(L);
    FS2_CUDA_CHECK(cudaMallocAsync(&vt, (size_t)B * C * lpad * sizeof(float) + 16, st));
    int rc = transpose_v(qkv, B, L, C, heads, vt, lpad, st);
    if (!rc) { ProfScope prof_scope(P_DEC_ATTN, flop, bytes, st); rc = attention_tf32(qkv, vt, lpad, lens, B, L, C, heads, ctx, st); }
    cudaFreeAsync(vt, st);
    return rc;
  }
  // plane families: q|k planes and transposed V planes made on the fly
  const int lpad = round8(L);
  const size_t nqk = (((size_t)2 * B * L * 2 * C) + 15) & ~(size_t)15, nvt = (size_t)2 * B * C * lpad;
  __half* tmp = nullptr;
  FS2_CUDA_CHECK(cudaMallocAsync(&tmp, (nqk + nvt) * sizeof(__half) + 64, st));
  int rc = qkv_to_planes(qkv, B, L, C, heads, tmp, tmp + nqk, lpad, st);
  if (!rc) { ProfScope prof_scope(P_DEC_ATTN, flop, bytes, st); rc = attention_planes(tmp, tmp + nqk, lpad, lens, B, L, C, heads, math_mode == MATH_3XTF32, ctx, nullptr, st); }
  cudaFreeAsync(tmp, st);
  return rc;
}
int fs2_op_attention_planes(int math_mode, const void* qkp, const void* vtp, int lpad, const int64_t* lens, int B, int L,
                            int C, int heads, float* ctx, void* ctxp, void* stream) {
  FS2_REQUIRE(math_mode == FS2_MATH_F16 || math_mode == FS2_MATH_3XTF32,
              "fs2_op_attention_planes: unknown math mode %d (operand planes exist in FS2_MATH_F16 and FS2_MATH_3XTF32)", math_mode);
  cudaStream_t st = (cudaStream_t)stream;
  const bool x3 = math_mode == FS2_MATH_3XTF32;
  ProfScope prof_scope(P_DEC_ATTN, 4.0 * B * (double)L * L * C, (x3 ? 4.0 : 2.0) * 4.0 * B * (double)L * C, st);
  return attention_planes(reinterpret_cast<const __half*>(qkp), reinterpret_cast<const __half*>(vtp), lpad, lens, B, L, C,
                          heads, x3, ctx, reinterpret_cast<__half*>(ctxp), st);
}
int fs2_op_layernorm(const float* x, const float* resid, const float* g, const float* b, float eps, int64_t rows, int C,
                     float* out, void* stream) {
  FS2_REQUIRE(x && g && b && out, "fs2_op_layernorm: null argument");
  Norm n; n.g = g; n.b = b; n.eps = eps;
  RowNorm r = make_norm(n, x, C, rows, C, out, C);
  r.resid = resid; r.ldr = C;
  return row_norm(r, (cudaStream_t)stream);
}
int fs2_op_row_norm(const fs2_row_norm_desc* d, void* stream) {
  FS2_REQUIRE(d, "fs2_op_row_norm: null descriptor");
  FS2_REQUIRE(d->out || d->split_out || d->head_w, "fs2_op_row_norm: no output (out, split_out or head_w)");
  return row_norm(row_norm_of(*d, nullptr), (cudaStream_t)stream);
}
int fs2_op_row_norm_spemb(const fs2_row_norm_desc* d, const float* spk_vec, void* stream) {
  FS2_REQUIRE(d, "fs2_op_row_norm_spemb: null descriptor");
  FS2_REQUIRE(d->out || d->split_out || d->head_w, "fs2_op_row_norm_spemb: no output (out, split_out or head_w)");
  return row_norm(row_norm_of(*d, spk_vec), (cudaStream_t)stream);
}
int fs2_op_variance_embed_add(const float* hm, const float* e_val, const float* p_val, const float* e_bins, const float* p_bins,
                              int n_edges, const float* e_tab, const float* e_bias, const float* p_tab, const float* p_bias,
                              int64_t rows, int C, float* out, void* planes, int planes_lo, int64_t* e_ids, int64_t* p_ids,
                              const int64_t* lens, int L, void* stream) {
  FS2_REQUIRE(hm && e_val && p_val && e_bins && p_bins && e_tab && e_bias && p_tab && p_bias && (out || planes),
              "fs2_op_variance_embed_add: null argument");
  return variance_embed_add(hm, e_val, p_val, e_bins, p_bins, n_edges, e_tab, e_bias, p_tab, p_bias, rows, C, out,
                            reinterpret_cast<__half*>(planes), planes_lo, e_ids, p_ids, lens, L, (cudaStream_t)stream);
}

}  // extern "C"
