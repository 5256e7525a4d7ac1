// C entries of the deterministic train mode (DESIGN.md section 26): the ordered twins of every train entry that sums with
// floating-point atomics.  Each takes a caller-owned workspace, sized by its _ws_bytes query, and checks every argument --
// the workspace included -- before anything is launched.  The kernels and the bodies are those of train.cu and rowwise.cu:
// the same math, instantiated with kOrdered, so partial sums land in the workspace and are added in a fixed order.
#include "common.cuh"

namespace fs2 {
namespace {

// present, 16-byte aligned and at least `need` bytes (a call that needs none may pass NULL)
int check_ws(const char* who, const void* ws, size_t ws_bytes, size_t need) {
  if (need == 0) return FS2_OK;
  FS2_REQUIRE(ws && (reinterpret_cast<uintptr_t>(ws) & 15) == 0, "%s: workspace missing or not 16-byte aligned", who);
  FS2_REQUIRE(ws_bytes >= need, "%s: workspace of %zu bytes, %zu needed", who, ws_bytes, need);
  return FS2_OK;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

constexpr long MAX_SCATTER_ROWS = (1L << 31) - 1;   // the sorted row list holds int32 row indices

}  // namespace
}  // namespace fs2

using namespace fs2;

#define FS2_WS_BYTES(expr)                                      \
  do {                                                          \
    FS2_REQUIRE(bytes, "%s: null argument", __func__);          \
    *bytes = (expr);                                            \
    return FS2_OK;                                              \
  } while (0)

extern "C" {

int fs2_colsum_det_ws_bytes(int64_t rows, int C, size_t* bytes) {
  FS2_REQUIRE(rows >= 0 && C > 0, "fs2_colsum_det_ws_bytes: need rows >= 0 and C > 0");
  FS2_WS_BYTES(colsum_det_bytes(rows, C));
}
int fs2_colsum_det(const float* x, int64_t rows, int C, float* out, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(x && out, "fs2_colsum_det: null argument");
  FS2_REQUIRE(rows >= 0 && C > 0, "fs2_colsum_det: need rows >= 0 and C > 0");
  int rc = check_ws("fs2_colsum_det", ws, ws_bytes, colsum_det_bytes(rows, C));
  if (rc) return rc;
  return colsum_det(x, rows, C, out, ws, (cudaStream_t)stream);
}

int fs2_conv_wgrad_det_ws_bytes(int B, int L, int N, int K, int taps, size_t* bytes) {
  FS2_REQUIRE(B >= 0 && L >= 0 && N > 0 && K > 0 && taps > 0 && (taps & 1) == 1,
              "fs2_conv_wgrad_det_ws_bytes: need B, L >= 0, N, K > 0 and odd taps");
  FS2_WS_BYTES(conv_wgrad_det_bytes(B, L, N, K, taps, true));
}
int fs2_conv_wgrad_det(const float* dy, const float* x, int B, int L, int N, int K, int taps, float* dw, float* dbias, void* ws,
                       size_t ws_bytes, void* stream) {
  FS2_REQUIRE(dy && x && dw, "fs2_conv_wgrad_det: null argument");
  FS2_REQUIRE(B >= 0 && L >= 0 && N > 0 && K > 0 && taps > 0 && (taps & 1) == 1, "fs2_conv_wgrad_det: need B, L >= 0, N, K > 0 and odd taps");
  int rc = check_ws("fs2_conv_wgrad_det", ws, ws_bytes, conv_wgrad_det_bytes(B, L, N, K, taps, dbias != nullptr));
  if (rc) return rc;
  return conv_wgrad_det(dy, x, B, L, N, K, taps, dw, dbias, ws, (cudaStream_t)stream);
}

int fs2_layernorm_backward_det_ws_bytes(int64_t rows, int C, size_t* bytes) {
  FS2_REQUIRE(rows >= 0 && (C == 256 || C == 384), "fs2_layernorm_backward_det_ws_bytes: need rows >= 0 and C in {256, 384}");
  FS2_WS_BYTES(layernorm_backward_det_bytes(rows, C));
}
int fs2_layernorm_backward_det(const float* x, const float* dy, const float* gamma, float eps, int64_t rows, int C, float* dx, float* dgamma,
                               float* dbeta, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(x && dy && gamma && dx && dgamma && dbeta, "fs2_layernorm_backward_det: null argument");
  FS2_REQUIRE(rows >= 0 && (C == 256 || C == 384), "fs2_layernorm_backward_det: need rows >= 0 and C in {256, 384} (got C=%d)", C);
  FS2_REQUIRE(aligned16(x) && aligned16(dy) && aligned16(gamma) && aligned16(dx), "fs2_layernorm_backward_det: x, dy, gamma and dx must be 16-byte aligned");
  int rc = check_ws("fs2_layernorm_backward_det", ws, ws_bytes, layernorm_backward_det_bytes(rows, C));
  if (rc) return rc;
  return layernorm_backward_det(x, dy, gamma, eps, rows, C, dx, dgamma, dbeta, ws, (cudaStream_t)stream);
}

int fs2_batchnorm_train_det_ws_bytes(int64_t rows, int C, size_t* bytes) {
  FS2_REQUIRE(rows > 0 && C > 0, "fs2_batchnorm_train_det_ws_bytes: need rows, C > 0");
  FS2_WS_BYTES(batchnorm_det_bytes(rows, C));
}
int fs2_batchnorm_train_det(const float* x, int64_t rows, int C, const float* gamma, const float* beta, float eps, float momentum, int act,
                            float* running_mean, float* running_var, float* stats, float* y, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(x && gamma && beta && stats && y, "fs2_batchnorm_train_det: null argument");
  FS2_REQUIRE(rows > 0 && C > 0, "fs2_batchnorm_train_det: need rows, C > 0");
  FS2_REQUIRE(!running_mean == !running_var, "fs2_batchnorm_train_det: running_mean and running_var go together");
  int rc = check_ws("fs2_batchnorm_train_det", ws, ws_bytes, batchnorm_det_bytes(rows, C));
  if (rc) return rc;
  return batchnorm_train_det(x, rows, C, gamma, beta, eps, momentum, act, running_mean, running_var, stats, y, ws, (cudaStream_t)stream);
}
int fs2_batchnorm_backward_det_ws_bytes(int64_t rows, int C, size_t* bytes) {
  FS2_REQUIRE(rows > 0 && C > 0, "fs2_batchnorm_backward_det_ws_bytes: need rows, C > 0");
  FS2_WS_BYTES(batchnorm_det_bytes(rows, C));
}
int fs2_batchnorm_backward_det(const float* x, const float* dy, const float* stats, const float* gamma, float eps, int64_t rows, int C, float* dx,
                               float* dgamma, float* dbeta, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(x && dy && stats && gamma && dx && dgamma && dbeta, "fs2_batchnorm_backward_det: null argument");
  FS2_REQUIRE(rows > 0 && C > 0, "fs2_batchnorm_backward_det: need rows, C > 0");
  int rc = check_ws("fs2_batchnorm_backward_det", ws, ws_bytes, batchnorm_det_bytes(rows, C));
  if (rc) return rc;
  return batchnorm_backward_det(x, dy, stats, gamma, eps, rows, C, dx, dgamma, dbeta, ws, (cudaStream_t)stream);
}

int fs2_embed_backward_det_ws_bytes(int B, int T, int C, int n_sym, size_t* bytes) {
  FS2_REQUIRE(B >= 0 && T >= 0 && C > 0 && n_sym >= 0 && n_sym <= scatter_max_ids() && (long)B * T <= MAX_SCATTER_ROWS,
              "fs2_embed_backward_det_ws_bytes: need B, T >= 0, B * T < 2^31, C > 0 and 0 <= n_sym <= %d", scatter_max_ids());
  FS2_WS_BYTES(embed_backward_det_bytes((long)B * T, C, n_sym, true));
}
int fs2_embed_backward_det(const int64_t* xs, const float* dy, const float* pe, int B, int T, int C, int n_sym, float* dtable, float* dalpha,
                           void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(dy && pe && dalpha && (xs || !dtable), "fs2_embed_backward_det: null argument");
  FS2_REQUIRE(B >= 0 && T >= 0 && C > 0 && (long)B * T <= MAX_SCATTER_ROWS, "fs2_embed_backward_det: need B, T >= 0, B * T < 2^31 and C > 0");
  FS2_REQUIRE(!dtable || (n_sym >= 1 && n_sym <= scatter_max_ids()), "fs2_embed_backward_det: a table needs 1 <= n_sym <= %d (got %d)",
              scatter_max_ids(), n_sym);
  int rc = check_ws("fs2_embed_backward_det", ws, ws_bytes, embed_backward_det_bytes((long)B * T, C, dtable ? n_sym : 0, dtable != nullptr));
  if (rc) return rc;
  return embed_backward_det(xs, dy, pe, B, T, C, n_sym, dtable, dalpha, ws, (cudaStream_t)stream);
}

int fs2_onehot_linear_backward_det_ws_bytes(int64_t rows, int C, int n_bins, size_t* bytes) {
  FS2_REQUIRE(rows >= 0 && rows <= MAX_SCATTER_ROWS && C > 0 && n_bins >= 1 && n_bins <= scatter_max_ids(),
              "fs2_onehot_linear_backward_det_ws_bytes: need 0 <= rows < 2^31, C > 0 and 1 <= n_bins <= %d", scatter_max_ids());
  FS2_WS_BYTES(onehot_linear_backward_det_bytes(rows, C, n_bins, true));
}
int fs2_onehot_linear_backward_det(const int64_t* ids, const float* dy, int64_t rows, int C, int n_bins, float* dW, float* dbias, void* ws,
                                   size_t ws_bytes, void* stream) {
  FS2_REQUIRE(ids && dy && dW, "fs2_onehot_linear_backward_det: null argument");
  FS2_REQUIRE(rows >= 0 && rows <= MAX_SCATTER_ROWS && C > 0 && n_bins >= 1 && n_bins <= scatter_max_ids(),
              "fs2_onehot_linear_backward_det: need 0 <= rows < 2^31, C > 0 and 1 <= n_bins <= %d", scatter_max_ids());
  int rc = check_ws("fs2_onehot_linear_backward_det", ws, ws_bytes, onehot_linear_backward_det_bytes(rows, C, n_bins, dbias != nullptr));
  if (rc) return rc;
  return onehot_linear_backward_det(ids, dy, rows, C, n_bins, dW, dbias, ws, (cudaStream_t)stream);
}

int fs2_rowdot_backward_det_ws_bytes(int64_t rows, int C, size_t* bytes) {
  FS2_REQUIRE(rows >= 0 && C > 0 && C <= 384, "fs2_rowdot_backward_det_ws_bytes: need rows >= 0 and 0 < C <= 384");
  FS2_WS_BYTES(rowdot_backward_det_bytes(rows, C));
}
int fs2_rowdot_backward_det(const float* x, const float* w, const float* dy, const int64_t* lens, int64_t rows, int L, int C, float* dx, float* dw,
                            float* dbias, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(x && w && dy && dx && dw && dbias, "fs2_rowdot_backward_det: null argument");
  FS2_REQUIRE(rows >= 0 && L > 0 && C > 0 && C <= 384, "fs2_rowdot_backward_det: need rows >= 0, L > 0 and 0 < C <= 384");
  int rc = check_ws("fs2_rowdot_backward_det", ws, ws_bytes, rowdot_backward_det_bytes(rows, C));
  if (rc) return rc;
  return rowdot_backward_det(x, w, dy, lens, rows, L, C, dx, dw, dbias, ws, (cudaStream_t)stream);
}

int fs2_masked_losses_det_ws_bytes(int B, int Tmax, int L, int odim, size_t* bytes) {
  FS2_REQUIRE(B >= 0 && Tmax >= 0 && L >= 0 && odim > 0, "fs2_masked_losses_det_ws_bytes: need B, Tmax, L >= 0 and odim > 0");
  FS2_WS_BYTES(loss_det_ws_bytes(B, Tmax, L, odim));
}
int fs2_masked_losses_det(const float* before, const float* after, const float* ys, int ld_ys_time, const float* d_out,
                          const void* ds, int ds_dtype, const float* e_out, const float* p_out, const float* es,
                          const float* ps, const int64_t* ilens, const int64_t* olens, int B, int Tmax, int L, int odim,
                          float* out7, void* ws, size_t ws_bytes, void* stream) {
  FS2_REQUIRE(before && after && ys && d_out && ds && e_out && p_out && es && ps && ilens && olens && out7,
              "fs2_masked_losses_det: null argument");
  FS2_REQUIRE(B >= 0 && Tmax >= 0 && L >= 0 && odim > 0 && odim % 4 == 0 && aligned16(ys) && aligned16(before) && aligned16(after),
              "fs2_masked_losses_det: need B, Tmax, L >= 0, odim a positive multiple of 4 and before, after, ys 16-byte aligned");
  int rc = check_ws("fs2_masked_losses_det", ws, ws_bytes, loss_det_ws_bytes(B, Tmax, L, odim));
  if (rc) return rc;
  return masked_losses_det(before, after, ys, ld_ys_time, d_out, ds, ds_dtype, e_out, p_out, es, ps, ilens, olens, B, Tmax, L, odim,
                           out7, ws, (cudaStream_t)stream);
}

}  // extern "C"
