// extern "C" entry points of libmpgcn_b200 (declared in include/mpgcn_b200.h).
#include "../../include/mpgcn_b200.h"

#include "kernels.h"

namespace mpgcn {
// precision 2 (bf16x3) serves whole layers only: its queries are those of bdgcn_forward_tc / bdgcn_backward_tc with bf = true
size_t bdgcn_saved_bytes(const BdgcnShape& s, int precision) {
  if (precision == PREC_BF16X3_TC) return s.whole() ? tc_saved_bytes(s, true) : 0;
  return precision == PREC_FP16_TC ? tc_saved_bytes(s) : simt_saved_bytes(s);
}
size_t bdgcn_fwd_workspace_bytes(const BdgcnShape& s, int precision) {
  if (precision == PREC_BF16X3_TC) return s.whole() ? tc_fwd_ws_bytes(s, true) : 0;
  return precision == PREC_FP16_TC ? tc_fwd_ws_bytes(s) : simt_fwd_ws_bytes(s);
}
size_t bdgcn_bwd_workspace_bytes(const BdgcnShape& s, int precision) {
  if (precision == PREC_BF16X3_TC) return s.whole() ? tc_bwd_ws_bytes(s, true) : 0;
  return precision == PREC_FP16_TC ? tc_bwd_ws_bytes(s) : simt_bwd_ws_bytes(s);
}
size_t bdgcn_sgrad_workspace_bytes(const BdgcnShape& s, int precision) {
  if (precision == PREC_BF16X3_TC) return 0;
  return precision == PREC_FP16_TC ? tc_sgrad_ws_bytes(s) : simt_sgrad_ws_bytes(s);
}
}  // namespace mpgcn

using namespace mpgcn;

static BdgcnShape mk(int B, int N, int K, int C, int H, int dynamic, int act) {
  BdgcnShape s;
  s.B = B; s.N = N; s.K = K; s.C = C; s.H = H; s.dynamic = dynamic; s.act = act;
  s.R = N; s.row0 = 0; s.Ko = K; s.Kd = K; s.partial = 0;      // the whole layer
  return s;
}

// a PART of the layer (include/mpgcn_b200.h: mpgcn_bdgcn_part)
static BdgcnShape mk_part(int B, int N, int C, int H, int dynamic, const mpgcn_bdgcn_part* part) {
  BdgcnShape s = mk(B, N, part ? (part->Ko > part->Kd ? part->Ko : part->Kd) : 1, C, H, dynamic, 0);
  if (part) { s.R = part->rows; s.row0 = part->row0; s.Ko = part->Ko; s.Kd = part->Kd; }
  s.partial = 1;
  return s;
}
static int check_part(const BdgcnShape& s, int precision) {
  MPGCN_CHECK(s.B >= 1 && s.N >= 1 && s.C >= 1 && s.H >= 1, "bad BDGCN shape B=%d N=%d C=%d H=%d", s.B, s.N, s.C, s.H);
  MPGCN_CHECK(s.Ko >= 1 && s.Kd >= 1 && s.R >= 1 && s.row0 >= 0 && s.row0 + s.R <= s.N,
              "bad layer part: rows [%d, %d) of N=%d, Ko=%d, Kd=%d", s.row0, s.row0 + s.R, s.N, s.Ko, s.Kd);
  MPGCN_CHECK(precision != PREC_BF16X3_TC, "layer parts: precision 2 (bf16x3) runs whole layers only");
  MPGCN_CHECK(precision == PREC_FP32_SIMT || precision == PREC_FP16_TC, "unknown precision %d", precision);
  if (precision == PREC_FP16_TC)
    MPGCN_CHECK(tc_supported(s), "precision 1 (tensor cores) needs C and H to be multiples of 32, from C == H == 32 up, H <= 1024 (got C=%d H=%d Ko=%d Kd=%d)", s.C, s.H, s.Ko, s.Kd);
  return 0;
}

// algorithmic flops of one layer call (SURVEY.md section 8(d)): F_f = 2KN^3(C+H) + 2K^2N^2CH, F_fb = 4KN^3(C+H) + 6K^2N^2CH
static double layer_flops(const BdgcnShape& s, bool backward) {
  const double n3 = 2.0 * s.K * (double)s.N * s.N * s.N * (s.C + s.H), mix = 2.0 * s.K * s.K * (double)s.N * s.N * s.C * s.H;
  return s.B * (backward ? n3 + 2.0 * mix : n3 + mix);
}

static int check_shape(const BdgcnShape& s, int precision) {
  MPGCN_CHECK(s.B >= 1 && s.N >= 1 && s.K >= 1 && s.C >= 1 && s.H >= 1, "bad BDGCN shape B=%d N=%d K=%d C=%d H=%d", s.B, s.N, s.K, s.C, s.H);
  MPGCN_CHECK(precision == PREC_FP32_SIMT || precision == PREC_FP16_TC || precision == PREC_BF16X3_TC, "unknown precision %d", precision);
  MPGCN_CHECK(s.act == 0 || s.act == 1, "unknown activation code %d", s.act);
  if (precision != PREC_FP32_SIMT)
    MPGCN_CHECK(tc_supported(s), "precision %d (tensor cores) needs C and H to be multiples of 32, from C == H == 32 up, H <= 1024 (got C=%d H=%d K=%d)", precision, s.C, s.H, s.K);
  return 0;
}

// precision 2 takes no fp16 copies of the activations
static int check_bf16x3_extras(const char* what, int precision, const mpgcn_bdgcn_extras* x) {
  if (precision == PREC_BF16X3_TC && x)
    MPGCN_CHECK(!x->x_f16 && !x->out_f16 && !x->d_pre_f16, "%s: precision 2 (bf16x3) takes no fp16 activation copies (x_f16 / out_f16 / d_pre_f16)", what);
  return 0;
}

extern "C" {

int mpgcn_abi_version(void) { return MPGCN_B200_ABI_VERSION; }
const char* mpgcn_last_error(void) { return last_error(); }

int mpgcn_set_deterministic(int on) { return det_set(on); }
int mpgcn_get_deterministic(void) { return det_mode(); }

int mpgcn_bdgcn_precision_supported(int B, int N, int K, int C, int H, int precision) {
  const BdgcnShape s = mk(B, N, K, C, H, 0, 0);
  if (precision == PREC_FP32_SIMT) return B >= 1 && N >= 1 && K >= 1 && C >= 1 && H >= 1;
  if (precision == PREC_FP16_TC || precision == PREC_BF16X3_TC) return tc_supported(s) ? 1 : 0;
  return 0;
}

size_t mpgcn_bdgcn_saved_bytes(int B, int N, int K, int C, int H, int precision) { return bdgcn_saved_bytes(mk(B, N, K, C, H, 0, 0), precision); }
size_t mpgcn_bdgcn_fwd_workspace_bytes(int B, int N, int K, int C, int H, int dynamic, int precision) {
  return bdgcn_fwd_workspace_bytes(mk(B, N, K, C, H, dynamic, 0), precision);
}
size_t mpgcn_bdgcn_bwd_workspace_bytes(int B, int N, int K, int C, int H, int dynamic, int precision) {
  return bdgcn_bwd_workspace_bytes(mk(B, N, K, C, H, dynamic, 0), precision);
}

static BdgcnExtras to_extras(const mpgcn_bdgcn_extras* x) {
  BdgcnExtras e;
  if (x) {
    e.go_prepared = x->go_prepared; e.gd_prepared = x->gd_prepared; e.x_f16 = x->x_f16; e.out_f16 = x->out_f16;
    e.d_out_absmax = x->d_out_absmax; e.dx_absmax = x->dX_absmax;
    e.d_pre_f16 = x->d_pre_f16; e.d_pre_scale2 = x->d_pre_scale2;
  }
  return e;
}

size_t mpgcn_bdgcn_supports_prepared_bytes(long long planes, int N) { return (planes >= 1 && N >= 1) ? bdgcn_supports_prepared_bytes(planes, N) : 0; }
size_t mpgcn_bdgcn_supports_prepared_bytes_ex(long long planes, int N, int precision) {
  if (precision != PREC_FP16_TC && precision != PREC_BF16X3_TC) return 0;
  return (planes >= 1 && N >= 1) ? bdgcn_supports_prepared_bytes(planes, N, precision == PREC_BF16X3_TC) : 0;
}

int mpgcn_bdgcn_prepare_supports(const float* G, void* prepared, size_t prepared_bytes, long long planes, int N, void* stream) {
  MPGCN_CHECK(G && prepared && planes >= 1 && N >= 1, "mpgcn_bdgcn_prepare_supports: bad argument");
  MPGCN_CHECK(prepared_bytes >= bdgcn_supports_prepared_bytes(planes, N), "mpgcn_bdgcn_prepare_supports: buffer too small (%zu < %zu)",
              prepared_bytes, bdgcn_supports_prepared_bytes(planes, N));
  return bdgcn_prepare_supports(G, prepared, planes, N, static_cast<cudaStream_t>(stream));
}

int mpgcn_bdgcn_prepare_supports_ex(const float* G, void* prepared, size_t prepared_bytes, long long planes, int N, int precision, void* stream) {
  MPGCN_CHECK(precision == PREC_FP16_TC || precision == PREC_BF16X3_TC, "mpgcn_bdgcn_prepare_supports_ex: precision %d has no prepared supports",
              precision);
  MPGCN_CHECK(G && prepared && planes >= 1 && N >= 1, "mpgcn_bdgcn_prepare_supports_ex: bad argument");
  const bool bf = precision == PREC_BF16X3_TC;
  MPGCN_CHECK(prepared_bytes >= bdgcn_supports_prepared_bytes(planes, N, bf), "mpgcn_bdgcn_prepare_supports_ex: buffer too small (%zu < %zu)",
              prepared_bytes, bdgcn_supports_prepared_bytes(planes, N, bf));
  return bdgcn_prepare_supports(G, prepared, planes, N, static_cast<cudaStream_t>(stream), bf);
}

int mpgcn_bdgcn_forward_x(const float* X, const float* G_o, const float* G_d, int dynamic, const float* W, const float* bias, int act,
                          float* out, void* saved, void* workspace, size_t workspace_bytes, int B, int N, int K, int C, int H,
                          int precision, const mpgcn_bdgcn_extras* extras, void* stream) {
  const BdgcnShape s = mk(B, N, K, C, H, dynamic ? 1 : 0, act);
  if (int e = check_shape(s, precision)) return e;
  if (int e = check_bf16x3_extras("mpgcn_bdgcn_forward", precision, extras)) return e;
  MPGCN_CHECK(X && G_o && G_d && W && out && workspace, "mpgcn_bdgcn_forward: null pointer argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfRegion region(PROF_LAYER_FWD, layer_flops(s, false), st);
  if (precision == PREC_FP16_TC) return bdgcn_forward_tc(s, X, G_o, G_d, W, bias, out, saved, workspace, workspace_bytes, to_extras(extras), st);
  if (precision == PREC_BF16X3_TC)
    return bdgcn_forward_tc(s, X, G_o, G_d, W, bias, out, saved, workspace, workspace_bytes, to_extras(extras), st, true);
  return bdgcn_forward_simt(s, X, G_o, G_d, W, bias, out, saved, workspace, workspace_bytes, st);      // exact path: extras unused
}

int mpgcn_bdgcn_forward(const float* X, const float* G_o, const float* G_d, int dynamic, const float* W, const float* bias, int act,
                        float* out, void* saved, void* workspace, size_t workspace_bytes, int B, int N, int K, int C, int H,
                        int precision, void* stream) {
  return mpgcn_bdgcn_forward_x(X, G_o, G_d, dynamic, W, bias, act, out, saved, workspace, workspace_bytes, B, N, K, C, H, precision,
                               nullptr, stream);
}

int mpgcn_bdgcn_backward_x(const float* d_out, const float* out, const float* G_o, const float* G_d, int dynamic, const float* W, int act,
                           const void* saved, float* dX, float* dW, float* db, void* workspace, size_t workspace_bytes, int B, int N,
                           int K, int C, int H, int precision, const mpgcn_bdgcn_extras* extras, void* stream) {
  const BdgcnShape s = mk(B, N, K, C, H, dynamic ? 1 : 0, act);
  if (int e = check_shape(s, precision)) return e;
  if (int e = check_bf16x3_extras("mpgcn_bdgcn_backward", precision, extras)) return e;
  const bool have_out16 = extras && extras->out_f16 && precision == PREC_FP16_TC;
  MPGCN_CHECK(d_out && (out || have_out16) && G_o && G_d && W && saved && dW && workspace, "mpgcn_bdgcn_backward: null pointer argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfRegion region(PROF_LAYER_BWD, layer_flops(s, true), st);
  if (precision == PREC_FP16_TC || precision == PREC_BF16X3_TC)
    return bdgcn_backward_tc(s, d_out, out, G_o, G_d, W, saved, dX, dW, db, workspace, workspace_bytes, to_extras(extras), st,
                             precision == PREC_BF16X3_TC);
  if (extras && extras->dX_absmax) MPGCN_CUDA(cudaMemsetAsync(extras->dX_absmax, 0, sizeof(float), st));      // "unknown"
  return bdgcn_backward_simt(s, d_out, out, G_o, G_d, W, saved, dX, dW, db, workspace, workspace_bytes, st);
}

size_t mpgcn_bdgcn_support_grad_workspace_bytes(int B, int N, int K, int C, int H, int dynamic, int precision) {
  const BdgcnShape s = mk(B, N, K, C, H, dynamic, 0);
  if (check_shape(s, precision)) return 0;
  return bdgcn_sgrad_workspace_bytes(s, precision);      // 0 for precision 2: no support gradient
}

int mpgcn_bdgcn_backward_supports(const float* d_out, const float* out, const float* G_o, const float* G_d, int dynamic, const float* W, int act,
                                  const void* saved, float* dX, float* dW, float* db, void* workspace, size_t workspace_bytes, int B, int N,
                                  int K, int C, int H, int precision, const mpgcn_bdgcn_extras* extras, const float* X, float* dG_o,
                                  float* dG_d, void* stream) {
  const BdgcnShape s = mk(B, N, K, C, H, dynamic ? 1 : 0, act);
  if (int e = check_shape(s, precision)) return e;
  MPGCN_CHECK(precision != PREC_BF16X3_TC, "mpgcn_bdgcn_backward_supports: precision 2 (bf16x3) has no support gradient");
  const bool have_out16 = extras && extras->out_f16 && precision == PREC_FP16_TC;
  MPGCN_CHECK(d_out && (out || have_out16) && X && G_o && G_d && W && saved && dW && workspace,
              "mpgcn_bdgcn_backward_supports: null pointer argument");
  MPGCN_CHECK(dynamic || (dG_o && !dG_d), "mpgcn_bdgcn_backward_supports: static supports take their gradient in dG_o; dG_d must be NULL");
  MPGCN_CHECK(!extras || !extras->d_pre_f16, "mpgcn_bdgcn_backward_supports: a prepared fp16 dPre belongs to a layer part");
  // the supports' own gradient adds 2 K B N^3 (C + H) to the backward's flops
  const double dg_flops = 2.0 * s.K * s.B * (double)s.N * s.N * s.N * (s.C + s.H);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfRegion region(PROF_LAYER_BWD, layer_flops(s, true) + dg_flops, st);
  if (precision == PREC_FP16_TC)
    return bdgcn_backward_supports_tc(s, d_out, out, X, G_o, G_d, W, saved, dX, dW, db, dG_o, dG_d, workspace, workspace_bytes,
                                      to_extras(extras), st);
  if (extras && extras->dX_absmax) MPGCN_CUDA(cudaMemsetAsync(extras->dX_absmax, 0, sizeof(float), st));      // "unknown"
  return bdgcn_backward_supports_simt(s, d_out, out, X, G_o, G_d, W, saved, dX, dW, db, dG_o, dG_d, workspace, workspace_bytes, st);
}

int mpgcn_bdgcn_backward_ex(const float* d_out, const float* out, const float* G_o, const float* G_d, int dynamic, const float* W, int act,
                            const void* saved, float* dX, float* dW, float* db, void* workspace, size_t workspace_bytes, int B, int N,
                            int K, int C, int H, int precision, const float* d_out_absmax, float* dX_absmax, void* stream) {
  mpgcn_bdgcn_extras x{};
  x.d_out_absmax = d_out_absmax; x.dX_absmax = dX_absmax;
  return mpgcn_bdgcn_backward_x(d_out, out, G_o, G_d, dynamic, W, act, saved, dX, dW, db, workspace, workspace_bytes, B, N, K, C, H,
                                precision, &x, stream);
}

int mpgcn_bdgcn_backward(const float* d_out, const float* out, const float* G_o, const float* G_d, int dynamic, const float* W, int act,
                         const void* saved, float* dX, float* dW, float* db, void* workspace, size_t workspace_bytes, int B, int N,
                         int K, int C, int H, int precision, void* stream) {
  return mpgcn_bdgcn_backward_x(d_out, out, G_o, G_d, dynamic, W, act, saved, dX, dW, db, workspace, workspace_bytes, B, N, K, C, H,
                                precision, nullptr, stream);
}

size_t mpgcn_bdgcn_part_saved_bytes(int B, int N, int C, int H, int precision, const mpgcn_bdgcn_part* part) {
  return bdgcn_saved_bytes(mk_part(B, N, C, H, 0, part), precision);
}
size_t mpgcn_bdgcn_part_fwd_workspace_bytes(int B, int N, int C, int H, int dynamic, int precision, const mpgcn_bdgcn_part* part) {
  return bdgcn_fwd_workspace_bytes(mk_part(B, N, C, H, dynamic, part), precision);
}
size_t mpgcn_bdgcn_part_bwd_workspace_bytes(int B, int N, int C, int H, int dynamic, int precision, const mpgcn_bdgcn_part* part) {
  return bdgcn_bwd_workspace_bytes(mk_part(B, N, C, H, dynamic, part), precision);
}

int mpgcn_bdgcn_forward_part(const float* X, const float* G_o, const float* G_d, int dynamic, const float* W, float* pre_partial, void* saved,
                             void* workspace, size_t workspace_bytes, int B, int N, int C, int H, int precision,
                             const mpgcn_bdgcn_part* part, const mpgcn_bdgcn_extras* extras, void* stream) {
  MPGCN_CHECK(part != nullptr, "mpgcn_bdgcn_forward_part: part descriptor is NULL");
  const BdgcnShape s = mk_part(B, N, C, H, dynamic ? 1 : 0, part);
  if (int e = check_part(s, precision)) return e;
  MPGCN_CHECK(X && G_o && G_d && W && pre_partial && workspace, "mpgcn_bdgcn_forward_part: null pointer argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfRegion region(PROF_LAYER_FWD, layer_flops(s, false) * s.R / s.N * (s.Ko + s.Kd) / (2.0 * s.K), st);
  if (precision == PREC_FP16_TC)
  {
    BdgcnExtras ex;                 // of the extras only the prepared supports apply to a part
    if (extras) { ex.go_prepared = extras->go_prepared; ex.gd_prepared = extras->gd_prepared; }
    return bdgcn_forward_tc(s, X, G_o, G_d, W, nullptr, pre_partial, saved, workspace, workspace_bytes, ex, st);
  }
  return bdgcn_forward_simt(s, X, G_o, G_d, W, nullptr, pre_partial, saved, workspace, workspace_bytes, st);
}

int mpgcn_bdgcn_backward_part(const float* d_pre, const float* G_o, const float* G_d, int dynamic, const float* W, const void* saved, float* dX,
                              float* dW, void* workspace, size_t workspace_bytes, int B, int N, int C, int H, int precision,
                              const mpgcn_bdgcn_part* part, const mpgcn_bdgcn_extras* extras, void* stream) {
  MPGCN_CHECK(part != nullptr, "mpgcn_bdgcn_backward_part: part descriptor is NULL");
  const BdgcnShape s = mk_part(B, N, C, H, dynamic ? 1 : 0, part);
  if (int e = check_part(s, precision)) return e;
  const bool have16 = extras && extras->d_pre_f16 && precision == PREC_FP16_TC;
  MPGCN_CHECK((d_pre || have16) && G_o && G_d && W && saved && dW && workspace, "mpgcn_bdgcn_backward_part: null pointer argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfRegion region(PROF_LAYER_BWD, layer_flops(s, true) * s.R / s.N * (s.Ko + s.Kd) / (2.0 * s.K), st);
  if (precision == PREC_FP16_TC) {
    BdgcnExtras ex = to_extras(extras);
    ex.x_f16 = nullptr; ex.out_f16 = nullptr; ex.dx_absmax = nullptr;
    return bdgcn_backward_tc(s, d_pre, nullptr, G_o, G_d, W, saved, dX, dW, nullptr, workspace, workspace_bytes, ex, st);
  }
  return bdgcn_backward_simt(s, d_pre, nullptr, G_o, G_d, W, saved, dX, dW, nullptr, workspace, workspace_bytes, st);
}

size_t mpgcn_sparse_supports_bytes(int K, int N, long long nnz) { return sparse_supports_bytes(K, N, nnz); }

int mpgcn_sparse_supports_build(const long long* indices, const float* values, long long nnz, int K, int N, void* supports,
                                size_t supports_bytes, void* stream) {
  MPGCN_CHECK(sparse_shape_ok(K, N, nnz), "mpgcn_sparse_supports_build: bad stack K=%d N=%d nnz=%lld (int32 indices: nnz < 2^31)", K, N, nnz);
  MPGCN_CHECK(supports && (nnz == 0 || (indices && values)), "mpgcn_sparse_supports_build: null pointer argument");
  MPGCN_CHECK(supports_bytes >= sparse_supports_bytes(K, N, nnz), "mpgcn_sparse_supports_build: buffer too small (%zu < %zu bytes)",
              supports_bytes, sparse_supports_bytes(K, N, nnz));
  return sparse_supports_build(indices, values, nnz, K, N, supports, static_cast<cudaStream_t>(stream));
}

static int check_sparse(const char* what, const BdgcnShape& s, const void* supports, size_t supports_bytes, long long nnz) {
  if (int e = check_shape(s, PREC_FP32_SIMT)) return e;
  MPGCN_CHECK(sparse_shape_ok(s.K, s.N, nnz), "%s: bad support stack K=%d N=%d nnz=%lld", what, s.K, s.N, nnz);
  MPGCN_CHECK(supports != nullptr, "%s: null pointer argument", what);
  MPGCN_CHECK(supports_bytes >= sparse_supports_bytes(s.K, s.N, nnz), "%s: support buffer too small (%zu < %zu bytes)", what,
              supports_bytes, sparse_supports_bytes(s.K, s.N, nnz));
  return 0;
}

int mpgcn_bdgcn_forward_sparse(const float* X, const void* supports, size_t supports_bytes, long long nnz, const float* W, const float* bias,
                               int act, float* out, void* saved, void* workspace, size_t workspace_bytes, int B, int N, int K, int C, int H,
                               void* stream) {
  const BdgcnShape s = mk(B, N, K, C, H, 0, act);
  if (int e = check_sparse("mpgcn_bdgcn_forward_sparse", s, supports, supports_bytes, nnz)) return e;
  MPGCN_CHECK(X && W && out && workspace, "mpgcn_bdgcn_forward_sparse: null pointer argument");
  const SparseSupports sp = sparse_supports_view(supports, K, N, nnz);
  return bdgcn_forward_simt(s, X, nullptr, nullptr, W, bias, out, saved, workspace, workspace_bytes, static_cast<cudaStream_t>(stream), &sp);
}

int mpgcn_bdgcn_backward_sparse(const float* d_out, const float* out, const void* supports, size_t supports_bytes, long long nnz,
                                const float* W, int act, const void* saved, float* dX, float* dW, float* db, void* workspace,
                                size_t workspace_bytes, int B, int N, int K, int C, int H, void* stream) {
  const BdgcnShape s = mk(B, N, K, C, H, 0, act);
  if (int e = check_sparse("mpgcn_bdgcn_backward_sparse", s, supports, supports_bytes, nnz)) return e;
  MPGCN_CHECK(d_out && out && W && saved && dW && workspace, "mpgcn_bdgcn_backward_sparse: null pointer argument");
  const SparseSupports sp = sparse_supports_view(supports, K, N, nnz);
  return bdgcn_backward_simt(s, d_out, out, nullptr, nullptr, W, saved, dX, dW, db, workspace, workspace_bytes,
                             static_cast<cudaStream_t>(stream), &sp);
}

int mpgcn_bias_act(float* x, const float* bias, int act, long long n, int H, void* stream) {
  MPGCN_CHECK(x && n >= 1 && (act == 0 || act == 1), "mpgcn_bias_act: bad argument");
  return bias_act_inplace(x, bias, act, (size_t)n, H, static_cast<cudaStream_t>(stream));
}

int mpgcn_rows_reduce_bias_act(float* out, const float* const* partials, int g, const float* bias, int act, int B, int N, int row0, int rows,
                               int H, void* stream) {
  MPGCN_CHECK(out && partials && B >= 1 && (act == 0 || act == 1), "mpgcn_rows_reduce_bias_act: bad argument");
  return rows_reduce_bias_act(out, partials, g, bias, act, B, N, row0, rows, H, static_cast<cudaStream_t>(stream));
}

int mpgcn_relu_backward_scatter(const float* d_out, const float* out, int act, float* const* dsts, int g, float* db, int B, int N, int row0,
                                int rows, int H, void* stream) {
  MPGCN_CHECK(!det_mode(), "mpgcn_relu_backward_scatter: no deterministic implementation (the mode of mpgcn_set_deterministic is on)");
  MPGCN_CHECK(d_out && dsts && B >= 1 && (act == 0 || (act == 1 && out)), "mpgcn_relu_backward_scatter: bad argument");
  return relu_backward_scatter(d_out, out, act, dsts, g, db, B, N, row0, rows, H, static_cast<cudaStream_t>(stream));
}

int mpgcn_relu_backward_scatter_f16(const float* d_out, const float* out, int act, void* const* dsts, int g, float* db, const float* absmax,
                                    float* scale2, int B, int N, int row0, int rows, int H, void* stream) {
  MPGCN_CHECK(!det_mode(), "mpgcn_relu_backward_scatter_f16: no deterministic implementation (the mode of mpgcn_set_deterministic is on)");
  MPGCN_CHECK(d_out && dsts && B >= 1 && (act == 0 || (act == 1 && out)), "mpgcn_relu_backward_scatter_f16: bad argument");
  return relu_backward_scatter_f16(d_out, out, act, reinterpret_cast<__half* const*>(dsts), g, db, absmax, scale2, B, N, row0, rows, H,
                                   static_cast<cudaStream_t>(stream));
}

int mpgcn_absmax(const float* x, long long n, float* out, void* stream) {
  MPGCN_CHECK(x && out && n >= 1, "mpgcn_absmax: bad argument");
  return absmax_f32(x, (size_t)n, out, static_cast<cudaStream_t>(stream));
}

int mpgcn_relu_backward(const float* d_out, const float* out, int act, float* d_pre, float* db, long long n, int H, void* stream) {
  MPGCN_CHECK(!det_mode(), "mpgcn_relu_backward: no deterministic implementation (the mode of mpgcn_set_deterministic is on)");
  MPGCN_CHECK(d_out && d_pre && n >= 1 && (act == 0 || (act == 1 && out)), "mpgcn_relu_backward: bad argument");
  return relu_bwd_prep(d_out, out, act, nullptr, d_pre, db, (size_t)n, H, nullptr, static_cast<cudaStream_t>(stream));
}

int mpgcn_adj_num_supports(int kernel_type, int K) { return adj_num_supports(kernel_type, K); }
size_t mpgcn_adj_workspace_bytes(int B, int N, int kernel_type, int K) { return adj_workspace_bytes(B, N); }
int mpgcn_adj_process(const float* flow, float* supports, int B, int N, int kernel_type, int K, void* workspace, size_t workspace_bytes,
                      void* stream) {
  MPGCN_CHECK(flow && supports, "mpgcn_adj_process: null pointer argument");
  return adj_process(flow, supports, B, N, kernel_type, K, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}
size_t mpgcn_adj_backward_workspace_bytes(int B, int N, int kernel_type, int K) {
  if (adj_num_supports(kernel_type, K) < 1 || B < 1 || N < 1 || K < 0) return 0;
  return adj_backward_workspace_bytes(B, N, kernel_type, K);
}
int mpgcn_adj_process_backward(const float* flow, const float* supports, const float* d_supports, float* d_flow, int B, int N, int kernel_type,
                               int K, void* workspace, size_t workspace_bytes, void* stream) {
  MPGCN_CHECK(flow && supports && d_supports && d_flow && workspace, "mpgcn_adj_process_backward: null pointer argument");
  return adj_process_backward(flow, supports, d_supports, d_flow, B, N, kernel_type, K, workspace, workspace_bytes,
                              static_cast<cudaStream_t>(stream));
}

int mpgcn_head_forward(const float* const* g, const float* w, const float* bias, float* y, float* pre, long long cells, int C, int M,
                       void* stream) {
  MPGCN_CHECK(g && w && bias && y && cells >= 1, "mpgcn_head_forward: null pointer or empty input");
  if (head_check("mpgcn_head_forward", g, w, nullptr, C, M)) return 1;
  ProfRegion region(PROF_HEAD, 2.0 * cells * C * M, static_cast<cudaStream_t>(stream));
  return head_forward(g, w, bias, y, pre, cells, C, M, static_cast<cudaStream_t>(stream));
}

int mpgcn_head_backward(const float* const* g, const float* w, const float* pre, const float* dy, float* const* dg, float* dw, float* db,
                        float* dg_absmax, long long cells, int C, int M, void* stream) {
  MPGCN_CHECK(!det_mode(), "mpgcn_head_backward: the deterministic mode needs a workspace: call mpgcn_head_backward_ex");
  return mpgcn_head_backward_ex(g, w, pre, dy, dg, dw, db, dg_absmax, cells, C, M, nullptr, 0, stream);
}

size_t mpgcn_head_backward_workspace_bytes(long long cells, int C, int M) {
  return det_mode() && cells >= 1 && C >= 1 && M >= 1 ? head_bwd_slot_bytes(cells, C, M) : 0;
}

int mpgcn_head_backward_ex(const float* const* g, const float* w, const float* pre, const float* dy, float* const* dg, float* dw, float* db,
                           float* dg_absmax, long long cells, int C, int M, void* workspace, size_t workspace_bytes, void* stream) {
  MPGCN_CHECK(g && w && pre && dy && dw && db && cells >= 1, "mpgcn_head_backward: null pointer or empty input");
  if (head_check("mpgcn_head_backward", g, w, dg, C, M)) return 1;
  const size_t need = mpgcn_head_backward_workspace_bytes(cells, C, M);
  MPGCN_CHECK(workspace_bytes >= need && (need == 0 || workspace != nullptr), "mpgcn_head_backward: workspace too small for the %s mode (%zu < %zu bytes)",
              det_mode() ? "deterministic" : "default", workspace_bytes, need);
  ProfRegion region(PROF_HEAD, 4.0 * cells * C * M, static_cast<cudaStream_t>(stream));
  return head_backward(g, w, pre, dy, dg, dw, db, dg_absmax, cells, C, M, static_cast<cudaStream_t>(stream),
                       det_mode() ? static_cast<float*>(workspace) : nullptr);
}

void mpgcn_profile_enable(int on) { prof_enable(on); }
void mpgcn_profile_reset(void) { prof_reset(); }
int mpgcn_profile_read(int tag, long long* launches, double* flops, double* ms) {
  MPGCN_CHECK(launches && flops && ms, "mpgcn_profile_read: null output pointer");
  MPGCN_CHECK(prof_read(tag, launches, flops, ms) == 0, "mpgcn_profile_read: unknown tag %d", tag);
  return 0;
}

long long mpgcn_debug_tc_workspace_offset(int which, int B, int N, int K, int dynamic) {
  return tc_debug_offset(mk(B, N, K, 32, 32, dynamic, 0), which);
}

size_t mpgcn_dyn_graph_workspace_bytes(int P, int N) { return (P >= 1 && N >= 1) ? dyn_graph_workspace_bytes(P, N) : 0; }

int mpgcn_dyn_graph_build(const float* od_history, int periods, float* o_graph, float* d_graph, int P, int N, void* workspace,
                          size_t workspace_bytes, void* stream) {
  MPGCN_CHECK(od_history && o_graph && d_graph, "mpgcn_dyn_graph_build: null pointer argument");
  return dyn_graph_build(od_history, periods, o_graph, d_graph, P, N, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

int mpgcn_lstm_precision_supported(int T, int C, int precision) {
  if (precision == PREC_FP32_SIMT) return lstm_bwd_cells_per_block(T, C) >= 1 ? 1 : 0;     // the backward bounds T (DESIGN.md 6.4)
  if (precision == PREC_FP16_TC) return lstm_tc_supported(T, C) ? 1 : 0;
  return 0;
}

// sizes for the width of the tensor-core kernel; a width it does not run keeps the hidden-32 size these always returned
static int lstm_tc_size_width(int C) { return lstm_tc_supported(1, C) ? C : 32; }

size_t mpgcn_lstm_bwd_workspace_bytes(int B, int T, long long NN, int C, int precision) {
  if (precision == PREC_FP16_TC) return lstm_tc_bwd_workspace_bytes(B, T, NN, lstm_tc_size_width(C));
  return lstm_bwd_workspace_bytes(C);
}

size_t mpgcn_lstm_saved_bytes(int B, int T, long long NN, int C, int precision) {
  return precision == PREC_FP16_TC ? lstm_tc_saved_bytes(B, T, NN, lstm_tc_size_width(C)) : 0;
}

int mpgcn_lstm_stack_supported(int T, int C, int L, int precision) {
  if (L == 1) return mpgcn_lstm_precision_supported(T, C, precision);
  return precision == PREC_FP16_TC && lstm_tc_stack_supported(T, C, L) ? 1 : 0;
}

size_t mpgcn_lstm_stack_saved_bytes(int B, int T, long long NN, int C, int L, int precision) {
  return mpgcn_lstm_stack_supported(T, C, L, precision) && L >= 2 ? lstm_tc_stack_saved_bytes(B, T, NN, C, L) : 0;
}
size_t mpgcn_lstm_stack_fwd_workspace_bytes(int B, int T, long long NN, int C, int L, int precision) {
  return mpgcn_lstm_stack_supported(T, C, L, precision) && L >= 2 ? lstm_tc_stack_fwd_workspace_bytes(B, T, NN, C, L) : 0;
}
size_t mpgcn_lstm_stack_bwd_workspace_bytes(int B, int T, long long NN, int C, int L, int precision) {
  return mpgcn_lstm_stack_supported(T, C, L, precision) && L >= 2 ? lstm_tc_stack_bwd_workspace_bytes(B, T, NN, C, L) : 0;
}

size_t mpgcn_lstm_recompute_bwd_workspace_bytes(int B, int T, long long NN, int C, int L, long long chunk_cells, int precision) {
  if (precision != PREC_FP16_TC || L < 1 || !mpgcn_lstm_stack_supported(T, C, L, precision) || B < 1 || NN < 1 || chunk_cells < 1) return 0;
  return lstm_tc_recompute_bwd_workspace_bytes(B, T, NN, C, L, chunk_cells);
}

// The argument checks of every LSTM entry, all before its first CUDA call: L layers (the stack entries take L >= 2), x_seq and
// h (h_T or d_hT), the L device pointers of each weight array w = {w_ih, w_hh, b_ih, b_hh} and, in a backward, of each gradient
// array g, a non-empty input, and kernels for (T, C, L) at the precision.  Precision 0 keeps no training state in the first
// place, so the recomputing backward runs the tensor-core kernels only.
enum LstmCall { LSTM_LAST, LSTM_STACK, LSTM_RECOMPUTE };
static int check_lstm(const char* what, LstmCall call, int L, const float* x_seq, const float* h, const float* const* const* w,
                      float* const* const* g, int B, int T, long long NN, int C, int precision) {
  MPGCN_CHECK(L >= (call == LSTM_STACK ? 2 : 1), "%s: L=%d%s", what, L, call == LSTM_STACK ? " (a single layer is mpgcn_lstm_last_*)" : "");
  MPGCN_CHECK(x_seq && h, "%s: null pointer argument", what);
  for (int k = 0; k < 4; ++k) {
    MPGCN_CHECK(w[k] && (!g || g[k]), "%s: null pointer argument", what);
    for (int l = 0; l < L; ++l) MPGCN_CHECK(w[k][l] && (!g || g[k][l]), "%s: null pointer argument (layer %d)", what, l);
  }
  MPGCN_CHECK(B >= 1 && T >= 1 && NN >= 1, "%s: empty input", what);
  MPGCN_CHECK((call != LSTM_RECOMPUTE || precision == PREC_FP16_TC) && mpgcn_lstm_stack_supported(T, C, L, precision),
              "%s: precision %d does not support T=%d, hidden=%d, L=%d", what, precision, T, C, L);
  return 0;
}

int mpgcn_lstm_last_forward_train(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, float* hT,
                                  void* saved, size_t saved_bytes, int B, int T, long long NN, int C, int precision, void* stream) {
  const float* const* w[4] = {&w_ih, &w_hh, &b_ih, &b_hh};
  if (int e = check_lstm("mpgcn_lstm_last_forward", LSTM_LAST, 1, x_seq, hT, w, nullptr, B, T, NN, C, precision)) return e;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (precision == PREC_FP16_TC) {
    MPGCN_CHECK(saved == nullptr || saved_bytes >= lstm_tc_saved_bytes(B, T, NN, C), "lstm forward: saved buffer too small (%zu < %zu)",
                saved_bytes, lstm_tc_saved_bytes(B, T, NN, C));
    return lstm_forward_tc(x_seq, 1, w[0], w[1], w[2], w[3], hT, saved, nullptr, 0, B, T, NN, C, st);
  }
  return lstm_last_forward(x_seq, w_ih, w_hh, b_ih, b_hh, hT, B, T, NN, C, st);
}

int mpgcn_lstm_last_forward(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, float* hT,
                            int B, int T, long long NN, int C, int precision, void* stream) {
  return mpgcn_lstm_last_forward_train(x_seq, w_ih, w_hh, b_ih, b_hh, hT, nullptr, 0, B, T, NN, C, precision, stream);
}

int mpgcn_lstm_last_backward_saved(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                                   const float* d_hT, float* d_w_ih, float* d_w_hh, float* d_b_ih, float* d_b_hh, float* d_x,
                                   const void* saved, size_t saved_bytes, void* workspace, size_t workspace_bytes, int B, int T,
                                   long long NN, int C, int precision, const float* d_hT_absmax, void* stream) {
  const float* const* w[4] = {&w_ih, &w_hh, &b_ih, &b_hh};
  float* const* g[4] = {&d_w_ih, &d_w_hh, &d_b_ih, &d_b_hh};
  if (int e = check_lstm("mpgcn_lstm_last_backward", LSTM_LAST, 1, x_seq, d_hT, w, g, B, T, NN, C, precision)) return e;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (precision == PREC_FP16_TC) {
    MPGCN_CHECK(saved == nullptr || saved_bytes >= lstm_tc_saved_bytes(B, T, NN, C), "lstm backward: saved buffer too small (%zu < %zu)",
                saved_bytes, lstm_tc_saved_bytes(B, T, NN, C));
    return lstm_last_backward_tc(x_seq, w_ih, w_hh, b_ih, b_hh, d_hT, d_w_ih, d_w_hh, d_b_ih, d_b_hh, d_x, saved, B, T, NN, C, workspace,
                                 workspace_bytes, d_hT_absmax, st);
  }
  return lstm_last_backward(x_seq, w_ih, w_hh, b_ih, b_hh, d_hT, d_w_ih, d_w_hh, d_b_ih, d_b_hh, d_x, B, T, NN, C, workspace,
                            workspace_bytes, st);
}

int mpgcn_lstm_last_backward(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                             const float* d_hT, float* d_w_ih, float* d_w_hh, float* d_b_ih, float* d_b_hh, float* d_x, void* workspace,
                             size_t workspace_bytes, int B, int T, long long NN, int C, int precision, void* stream) {
  return mpgcn_lstm_last_backward_saved(x_seq, w_ih, w_hh, b_ih, b_hh, d_hT, d_w_ih, d_w_hh, d_b_ih, d_b_hh, d_x, nullptr, 0, workspace,
                                        workspace_bytes, B, T, NN, C, precision, nullptr, stream);
}

int mpgcn_lstm_last_backward_ex(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                                const float* d_hT, float* d_w_ih, float* d_w_hh, float* d_b_ih, float* d_b_hh, float* d_x, void* workspace,
                                size_t workspace_bytes, int B, int T, long long NN, int C, int precision, const float* d_hT_absmax,
                                void* stream) {
  return mpgcn_lstm_last_backward_saved(x_seq, w_ih, w_hh, b_ih, b_hh, d_hT, d_w_ih, d_w_hh, d_b_ih, d_b_hh, d_x, nullptr, 0, workspace,
                                        workspace_bytes, B, T, NN, C, precision, d_hT_absmax, stream);
}

int mpgcn_lstm_stack_forward(const float* x_seq, int L, const float* const* w_ih, const float* const* w_hh, const float* const* b_ih,
                             const float* const* b_hh, float* hT, void* saved, size_t saved_bytes, void* workspace, size_t workspace_bytes,
                             int B, int T, long long NN, int C, int precision, void* stream) {
  const float* const* w[4] = {w_ih, w_hh, b_ih, b_hh};
  if (int e = check_lstm("mpgcn_lstm_stack_forward", LSTM_STACK, L, x_seq, hT, w, nullptr, B, T, NN, C, precision)) return e;
  MPGCN_CHECK(saved == nullptr || saved_bytes >= lstm_tc_stack_saved_bytes(B, T, NN, C, L),
              "lstm stack forward: saved buffer too small (%zu < %zu)", saved_bytes, lstm_tc_stack_saved_bytes(B, T, NN, C, L));
  return lstm_forward_tc(x_seq, L, w_ih, w_hh, b_ih, b_hh, hT, saved, workspace, workspace_bytes, B, T, NN, C,
                         static_cast<cudaStream_t>(stream));
}

int mpgcn_lstm_stack_backward(const float* x_seq, int L, const float* const* w_ih, const float* const* w_hh, const float* const* b_ih,
                              const float* const* b_hh, const float* d_hT, float* const* d_w_ih, float* const* d_w_hh, float* const* d_b_ih,
                              float* const* d_b_hh, float* d_x, const void* saved, size_t saved_bytes, void* workspace,
                              size_t workspace_bytes, int B, int T, long long NN, int C, int precision, const float* d_hT_absmax,
                              void* stream) {
  const float* const* w[4] = {w_ih, w_hh, b_ih, b_hh};
  float* const* g[4] = {d_w_ih, d_w_hh, d_b_ih, d_b_hh};
  if (int e = check_lstm("mpgcn_lstm_stack_backward", LSTM_STACK, L, x_seq, d_hT, w, g, B, T, NN, C, precision)) return e;
  MPGCN_CHECK(saved != nullptr, "mpgcn_lstm_stack_backward: null pointer argument");
  MPGCN_CHECK(saved_bytes >= lstm_tc_stack_saved_bytes(B, T, NN, C, L), "lstm stack backward: saved buffer too small (%zu < %zu)",
              saved_bytes, lstm_tc_stack_saved_bytes(B, T, NN, C, L));
  return lstm_stack_backward_tc(x_seq, L, w_ih, w_hh, b_ih, b_hh, d_hT, d_w_ih, d_w_hh, d_b_ih, d_b_hh, d_x, saved, workspace, workspace_bytes,
                                B, T, NN, C, d_hT_absmax, static_cast<cudaStream_t>(stream));
}

int mpgcn_lstm_backward_recompute(const float* x_seq, int L, const float* const* w_ih, const float* const* w_hh, const float* const* b_ih,
                                  const float* const* b_hh, const float* d_hT, float* const* d_w_ih, float* const* d_w_hh,
                                  float* const* d_b_ih, float* const* d_b_hh, float* d_x, long long chunk_cells, void* workspace,
                                  size_t workspace_bytes, int B, int T, long long NN, int C, int precision, const float* d_hT_absmax,
                                  void* stream) {
  const float* const* w[4] = {w_ih, w_hh, b_ih, b_hh};
  float* const* g[4] = {d_w_ih, d_w_hh, d_b_ih, d_b_hh};
  if (int e = check_lstm("mpgcn_lstm_backward_recompute", LSTM_RECOMPUTE, L, x_seq, d_hT, w, g, B, T, NN, C, precision)) return e;
  MPGCN_CHECK(chunk_cells >= 1, "mpgcn_lstm_backward_recompute: chunk_cells=%lld (at least 1)", chunk_cells);
  return lstm_recompute_backward_tc(x_seq, L, w_ih, w_hh, b_ih, b_hh, d_hT, d_w_ih, d_w_hh, d_b_ih, d_b_hh, d_x, chunk_cells, workspace,
                                    workspace_bytes, B, T, NN, C, d_hT_absmax, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
