// BDGCN layer, exact fp32 mode (precision 0): the factored evaluation order of
// SURVEY.md section 7.1 expressed as calls of the strided SIMT SGEMM.
//
//   forward  (reference: /root/reference/MPGCN.py:24-50)
//     Z[b,d,n,e,l] = sum_c X[b,n,c,l] G_d[c,e]
//     U[b,o,n,e,h] = sum_{d,l} Z[b,d,n,e,l] W[o,d,l,h]
//     out[b,m,e,h] = act( sum_{o,n} G_o[n,m] U[b,o,n,e,h] + bias[h] )
//   backward (what autograd derives from the same lines; supports never need grad)
//     dPre = dOut * act'(out) ; db = sum dPre
//     V[b,o,n,e,h] = sum_m G_o[n,m] dPre[b,m,e,h]
//     dW[o,d,l,h]  = sum_{b,n,e} Z[b,d,n,e,l] V[b,o,n,e,h]
//     Y[b,d,n,e,l] = sum_{o,h} V[b,o,n,e,h] W[o,d,l,h]
//     dX[b,n,c,l]  = sum_{d,e} Y[b,d,n,e,l] G_d[c,e]
//   support gradients (opt-in; U recomputed from the Z stash)
//     dG_o[n,m] = sum_{b,e,h} U_o[b,n,e,h] dPre[b,m,e,h]     dG_d[c,e] = sum_{b,n,l} X[b,n,c,l] Y_d[b,n,e,l]
// Sparse static supports (bdgcn_sparse.cu) replace the four N^3 stages (Z, out, V, dX) by gathers over their nonzeros; the mix
// stages, dW, Y, the layouts and the stash stay these.
#include "kernels.h"

namespace mpgcn {

// cells of an activation slab: R origin rows x N destinations (R = N for a whole layer)
static size_t rn(const BdgcnShape& s) { return (size_t)s.R * s.N; }

size_t simt_saved_bytes(const BdgcnShape& s) { return (size_t)s.B * s.Kd * rn(s) * s.C * sizeof(float); }

// forward workspace: U, then Z (used only when the caller passes no `saved` buffer)
struct SimtFwdLayout { size_t u, z, total; };
static SimtFwdLayout simt_fwd_layout(const BdgcnShape& s) {
  SimtFwdLayout L;
  size_t off = 0;
  L.u = take(off, (size_t)s.B * s.Ko * rn(s) * s.H * 4, 256);
  L.z = take(off, simt_saved_bytes(s), 256);
  L.total = align_up(off, 256) + 256;    // unused padding: the size this workspace has always had
  return L;
}
size_t simt_fwd_ws_bytes(const BdgcnShape& s) { return simt_fwd_layout(s).total; }

// dW = sum over R*N rows: split-K into up to 256 slices of >= 2048 rows
static int dw_ksplit(const BdgcnShape& s) {
  long long ks = (long long)rn(s) / 2048;
  return (int)(ks < 1 ? 1 : ks > 256 ? 256 : ks);
}
static int dw_mt(const BdgcnShape& s) { return (s.Kd * s.C + 127) / 128; }

// backward workspace: dPre (every origin row m, always), V, Y, Wq; `sgrad` (the support gradient) adds U, recomputed from the Z
// stash.  Deterministic mode's region follows: the bias-gradient slots and (ksplit > 1) the dW slices in the layout of
// reduce_dw_partials, [slice][MT * 128 rows d*C + c][Ko*H columns o*H + h], MT = ceil(Kd*C / 128); both empty with the mode off.
struct SimtBwdLayout { size_t dpre, v, y, wq, u, db_slots, dw_slices, total; };
static SimtBwdLayout simt_bwd_layout(const BdgcnShape& s, bool sgrad) {
  SimtBwdLayout L{};
  size_t off = 0;
  L.dpre = take(off, (size_t)s.B * s.N * s.N * s.H * 4, 256);
  L.v = take(off, (size_t)s.B * s.Ko * rn(s) * s.H * 4, 256);
  L.y = take(off, (size_t)s.B * s.Kd * rn(s) * s.C * 4, 256);
  L.wq = take(off, (size_t)s.Ko * s.Kd * s.C * s.H * 4, 256);
  if (sgrad) L.u = take(off, (size_t)s.B * s.Ko * rn(s) * s.H * 4, 256);
  off = align_up(off, 256) + (sgrad ? 1024 + 256 : 1024);     // unused padding: the sizes these workspaces have always had
  const int ks = dw_ksplit(s);
  L.db_slots = take(off, det_mode() ? bias_grad_slot_bytes(s.H) : 0, 256);
  L.dw_slices = take(off, det_mode() && ks > 1 ? (size_t)ks * dw_mt(s) * 128 * s.Ko * s.H * 4 : 0, 256);
  L.total = align_up(off, 256);
  return L;
}
size_t simt_bwd_ws_bytes(const BdgcnShape& s) { return simt_bwd_layout(s, false).total; }
size_t simt_sgrad_ws_bytes(const BdgcnShape& s) { return simt_bwd_layout(s, true).total; }

static void zero3(long long (&a)[3]) { a[0] = a[1] = a[2] = 0; }

// Activations are [B][*][R rows n][N][ch] slabs (rows [row0, row0 + R) of the N origins), G_d has Kd planes, G_o has Ko,
// W is the [Ko][Kd][C][H] slice; `partial`: the forward stops at the raw partial pre-activation, the backward starts from dPre.
int bdgcn_forward_simt(const BdgcnShape& s, const float* X, const float* Go, const float* Gd, const float* W, const float* bias,
                       float* out, void* saved, void* ws, size_t ws_bytes, cudaStream_t st, const SparseSupports* sp) {
  const long long N = s.N, R = s.R, RN = R * N, NN = N * N, C = s.C, H = s.H, Ko = s.Ko, Kd = s.Kd;
  const SimtFwdLayout L = simt_fwd_layout(s);
  MPGCN_CHECK(ws_bytes >= L.total, "bdgcn_forward: workspace too small (%zu < %zu bytes)", ws_bytes, L.total);
  uint8_t* wb = static_cast<uint8_t*>(ws);
  float* U = reinterpret_cast<float*>(wb + L.u);
  float* Z = saved ? static_cast<float*>(saved) : reinterpret_cast<float*>(wb + L.z);
  const long long go_sb = s.dynamic ? Ko * NN : 0, gd_sb = s.dynamic ? Kd * NN : 0;   // support batch strides

  if (sp) {
    if (int e = sparse_stage(SPARSE_FWD_A, s, *sp, X, Z, nullptr, st)) return e;
  } else {  // Z[b,d,n] (e x l) = G_d^T (e x c) * X[b,n] (c x l)
    SgemmParams p{};
    p.A = Gd; p.B = X; p.D = Z;
    p.M = (int)N; p.N = (int)C; p.K = (int)N;
    p.a_si = 1; p.a_sk = N; p.b_sk = C; p.b_sj = 1; p.d_si = C;
    p.nseg = 1; p.Z0 = s.B; p.Z1 = (int)Kd; p.Z2 = (int)R;
    p.a_sz[0] = gd_sb; p.a_sz[1] = NN; p.a_sz[2] = 0;
    p.b_sz[0] = RN * C; p.b_sz[1] = 0; p.b_sz[2] = N * C;
    p.d_sz[0] = Kd * RN * C; p.d_sz[1] = RN * C; p.d_sz[2] = N * C;
    p.ksplit = 1; p.alpha = 1.f;
    if (int e = simt_sgemm(p, st)) return e;
  }
  {  // U[b,o] (rows x h) = sum_d Z[b,d] (rows x l) * W[o,d] (l x h)
    SgemmParams p{};
    p.A = Z; p.B = W; p.D = U;
    p.M = (int)RN; p.N = (int)H; p.K = (int)C;
    p.a_si = C; p.a_sk = 1; p.b_sk = H; p.b_sj = 1; p.d_si = H;
    p.nseg = (int)Kd; p.a_sseg = RN * C; p.b_sseg = C * H;
    p.Z0 = s.B; p.Z1 = (int)Ko; p.Z2 = 1;
    zero3(p.a_sz); zero3(p.b_sz); zero3(p.d_sz);
    p.a_sz[0] = Kd * RN * C;
    p.b_sz[1] = Kd * C * H;
    p.d_sz[0] = Ko * RN * H; p.d_sz[1] = RN * H;
    p.ksplit = 1; p.alpha = 1.f;
    if (int e = simt_sgemm(p, st)) return e;
  }
  if (sp) {
    if (int e = sparse_stage(SPARSE_FWD_B, s, *sp, U, out, bias, st)) return e;
  } else {  // out[b] (m x (e,h)) = act( sum_o G_o[row0.., :]^T (m x n) * U[b,o] (n x (e,h)) + bias[h] ): one k-segment per support
    SgemmParams p{};
    p.A = Go + (long long)s.row0 * N; p.B = U; p.D = out;
    p.M = (int)N; p.N = (int)(N * H); p.K = (int)R;
    p.a_si = 1; p.a_sk = N; p.b_sk = N * H; p.b_sj = 1; p.d_si = N * H;
    p.nseg = (int)Ko; p.a_sseg = NN; p.b_sseg = RN * H;
    p.Z0 = s.B; p.Z1 = 1; p.Z2 = 1;
    zero3(p.a_sz); zero3(p.b_sz); zero3(p.d_sz);
    p.a_sz[0] = go_sb; p.b_sz[0] = Ko * RN * H; p.d_sz[0] = NN * H;
    p.ksplit = 1; p.alpha = 1.f;
    if (!s.partial) { p.bias = bias; p.bias_mod = (int)H; p.relu = s.act; }
    if (int e = simt_sgemm(p, st)) return e;
  }
  return 0;
}

// L: the layout, checked against the workspace; form_y: form Y even without dX (the support gradient reads it)
static int backward_simt_impl(const BdgcnShape& s, const float* d_out, const float* out, const float* Go, const float* Gd, const float* W,
                              const void* saved, float* dX, float* dW, float* db, void* ws, const SimtBwdLayout& L, bool form_y,
                              cudaStream_t st, const SparseSupports* sp) {
  const long long N = s.N, R = s.R, RN = R * N, NN = N * N, C = s.C, H = s.H, Ko = s.Ko, Kd = s.Kd;
  const float* Z = static_cast<const float*>(saved);
  MPGCN_CHECK(Z != nullptr, "bdgcn_backward: forward was run without a `saved` buffer");
  uint8_t* wb = static_cast<uint8_t*>(ws);
  float* dPre = reinterpret_cast<float*>(wb + L.dpre);
  float* V = reinterpret_cast<float*>(wb + L.v);
  float* Y = reinterpret_cast<float*>(wb + L.y);
  float* Wq = reinterpret_cast<float*>(wb + L.wq);
  const bool det = det_mode();     // fixed-order sums from the slots instead of atomics
  const long long go_sb = s.dynamic ? Ko * NN : 0, gd_sb = s.dynamic ? Kd * NN : 0;

  const float* dP = d_out;         // a partial call receives dPre itself (every origin row m, already masked)
  if (!s.partial) {
    if (int e = relu_bwd_prep(d_out, out, s.act, nullptr, dPre, db, (size_t)s.B * NN * H, (int)H, nullptr, st,
                              det ? reinterpret_cast<float*>(wb + L.db_slots) : nullptr))
      return e;
    dP = dPre;
  }

  if (sp) {
    if (int e = sparse_stage(SPARSE_BWD_V, s, *sp, dP, V, nullptr, st)) return e;
  } else {  // V[b,o] (n x (e,h)) = G_o[row0.., :] (n x m) * dPre[b] (m x (e,h))
    SgemmParams p{};
    p.A = Go + (long long)s.row0 * N; p.B = dP; p.D = V;
    p.M = (int)R; p.N = (int)(N * H); p.K = (int)N;
    p.a_si = N; p.a_sk = 1; p.b_sk = N * H; p.b_sj = 1; p.d_si = N * H;
    p.nseg = 1; p.Z0 = s.B; p.Z1 = (int)Ko; p.Z2 = 1;
    zero3(p.a_sz); zero3(p.b_sz); zero3(p.d_sz);
    p.a_sz[0] = go_sb; p.a_sz[1] = NN;
    p.b_sz[0] = NN * H;
    p.d_sz[0] = Ko * RN * H; p.d_sz[1] = RN * H;
    p.ksplit = 1; p.alpha = 1.f;
    if (int e = simt_sgemm(p, st)) return e;
  }
  {  // dW[o,d] (l x h) = sum_b Z[b,d]^T (l x rows) * V[b,o] (rows x h)
    const int ks = dw_ksplit(s);
    const bool slices = det && ks > 1;      // deterministic: every slice stores its partial, reduce_dw_partials adds them in order
    if (!slices) MPGCN_CUDA(cudaMemsetAsync(dW, 0, sizeof(float) * Ko * Kd * C * H, st));
    SgemmParams p{};
    p.A = Z; p.B = V; p.D = dW;
    p.M = (int)C; p.N = (int)H; p.K = (int)RN;
    p.a_si = 1; p.a_sk = C; p.b_sk = H; p.b_sj = 1; p.d_si = H;
    p.nseg = s.B; p.a_sseg = Kd * RN * C; p.b_sseg = Ko * RN * H;
    p.Z0 = (int)Ko; p.Z1 = (int)Kd; p.Z2 = 1;      // z0 = o, z1 = d
    zero3(p.a_sz); zero3(p.b_sz); zero3(p.d_sz);
    p.a_sz[1] = RN * C;
    p.b_sz[0] = RN * H;
    p.d_sz[0] = Kd * C * H; p.d_sz[1] = C * H;
    p.ksplit = ks; p.alpha = 1.f;
    float* P = slices ? reinterpret_cast<float*>(wb + L.dw_slices) : nullptr;
    if (slices) {
      p.D = P; p.d_si = Ko * H; p.d_sz[0] = H; p.d_sz[1] = C * Ko * H;
      p.d_sslice = (long long)dw_mt(s) * 128 * Ko * H;
    }
    if (int e = simt_sgemm(p, st)) return e;
    if (slices)
      if (int e = reduce_dw_partials(P, dW, ks, dw_mt(s), (int)Ko, (int)Kd, (int)C, (int)H, nullptr, st)) return e;
  }
  if (dX || form_y) {
    if (int e = permute_w_bwd(W, Wq, (int)Ko, (int)Kd, (int)C, (int)H, st)) return e;
    {  // Y[b,d] (rows x l) = sum_o V[b,o] (rows x h) * Wq[d,o] (h x l)
      SgemmParams p{};
      p.A = V; p.B = Wq; p.D = Y;
      p.M = (int)RN; p.N = (int)C; p.K = (int)H;
      p.a_si = H; p.a_sk = 1; p.b_sk = C; p.b_sj = 1; p.d_si = C;
      p.nseg = (int)Ko; p.a_sseg = RN * H; p.b_sseg = H * C;
      p.Z0 = s.B; p.Z1 = (int)Kd; p.Z2 = 1;
      zero3(p.a_sz); zero3(p.b_sz); zero3(p.d_sz);
      p.a_sz[0] = Ko * RN * H;
      p.b_sz[1] = Ko * H * C;
      p.d_sz[0] = Kd * RN * C; p.d_sz[1] = RN * C;
      p.ksplit = 1; p.alpha = 1.f;
      if (int e = simt_sgemm(p, st)) return e;
    }
    if (dX && sp) {
      if (int e = sparse_stage(SPARSE_BWD_DX, s, *sp, Y, dX, nullptr, st)) return e;
    } else if (dX) {  // dX[b,n] (c x l) = sum_d G_d (c x e) * Y[b,d,n] (e x l)
      SgemmParams p{};
      p.A = Gd; p.B = Y; p.D = dX;
      p.M = (int)N; p.N = (int)C; p.K = (int)N;
      p.a_si = N; p.a_sk = 1; p.b_sk = C; p.b_sj = 1; p.d_si = C;
      p.nseg = (int)Kd; p.a_sseg = NN; p.b_sseg = RN * C;
      p.Z0 = s.B; p.Z1 = (int)R; p.Z2 = 1;
      zero3(p.a_sz); zero3(p.b_sz); zero3(p.d_sz);
      p.a_sz[0] = gd_sb;
      p.b_sz[0] = Kd * RN * C; p.b_sz[1] = N * C;
      p.d_sz[0] = RN * C; p.d_sz[1] = N * C;
      p.ksplit = 1; p.alpha = 1.f;
      if (int e = simt_sgemm(p, st)) return e;
    }
  }
  return 0;
}

}  // namespace mpgcn

namespace mpgcn {

int bdgcn_backward_simt(const BdgcnShape& s, const float* d_out, const float* out, const float* Go, const float* Gd, const float* W,
                        const void* saved, float* dX, float* dW, float* db, void* ws, size_t ws_bytes, cudaStream_t st,
                        const SparseSupports* sp) {
  const SimtBwdLayout L = simt_bwd_layout(s, false);
  MPGCN_CHECK(ws_bytes >= L.total, "bdgcn_backward: workspace too small (%zu < %zu bytes)", ws_bytes, L.total);
  return backward_simt_impl(s, d_out, out, Go, Gd, W, saved, dX, dW, db, ws, L, false, st, sp);
}

int bdgcn_backward_supports_simt(const BdgcnShape& s, const float* d_out, const float* out, const float* X, const float* Go, const float* Gd,
                                 const float* W, const void* saved, float* dX, float* dW, float* db, float* dGo, float* dGd, void* ws,
                                 size_t ws_bytes, cudaStream_t st) {
  MPGCN_CHECK(s.whole(), "support gradients: whole layers only");
  const SimtBwdLayout L = simt_bwd_layout(s, true);
  MPGCN_CHECK(ws_bytes >= L.total, "bdgcn_backward_supports: workspace too small (%zu < %zu bytes)", ws_bytes, L.total);
  const bool want_d = dGd != nullptr || (!s.dynamic && dGo != nullptr);
  if (int e = backward_simt_impl(s, d_out, out, Go, Gd, W, saved, dX, dW, db, ws, L, want_d, st, nullptr)) return e;
  const long long N = s.N, NN = N * N, C = s.C, H = s.H, Ko = s.Ko, Kd = s.Kd;
  const float* Z = static_cast<const float*>(saved);
  uint8_t* wb = static_cast<uint8_t*>(ws);
  const float* dPre = reinterpret_cast<const float*>(wb + L.dpre);
  const float* Y = reinterpret_cast<const float*>(wb + L.y);
  float* U = reinterpret_cast<float*>(wb + L.u);
  if (dGo) {
    {  // U[b,o] (rows x h) = sum_d Z[b,d] (rows x l) * W[o,d] (l x h), as the forward
      SgemmParams p{};
      p.A = Z; p.B = W; p.D = U;
      p.M = (int)NN; p.N = (int)H; p.K = (int)C;
      p.a_si = C; p.a_sk = 1; p.b_sk = H; p.b_sj = 1; p.d_si = H;
      p.nseg = (int)Kd; p.a_sseg = NN * C; p.b_sseg = C * H;
      p.Z0 = s.B; p.Z1 = (int)Ko; p.Z2 = 1;
      p.a_sz[0] = Kd * NN * C;
      p.b_sz[1] = Kd * C * H;
      p.d_sz[0] = Ko * NN * H; p.d_sz[1] = NN * H;
      p.ksplit = 1; p.alpha = 1.f;
      if (int e = simt_sgemm(p, st)) return e;
    }
    {  // dG_o (n x m) = sum_b U[b,o] (n x (e,h)) * dPre[b]^T ((e,h) x m): one k-segment per sample when the supports are static
      SgemmParams p{};
      p.A = U; p.B = dPre; p.D = dGo;
      p.M = (int)N; p.N = (int)N; p.K = (int)(N * H);
      p.a_si = N * H; p.a_sk = 1; p.b_sk = 1; p.b_sj = N * H; p.d_si = N;
      if (s.dynamic) {
        p.nseg = 1; p.Z0 = s.B; p.Z1 = (int)Ko; p.Z2 = 1;
        p.a_sz[0] = Ko * NN * H; p.a_sz[1] = NN * H; p.b_sz[0] = NN * H; p.d_sz[0] = Ko * NN; p.d_sz[1] = NN;
      } else {
        p.nseg = s.B; p.a_sseg = Ko * NN * H; p.b_sseg = NN * H; p.Z0 = (int)Ko; p.Z1 = 1; p.Z2 = 1;
        p.a_sz[0] = NN * H; p.d_sz[0] = NN;
      }
      p.ksplit = 1; p.alpha = 1.f;
      if (int e = simt_sgemm(p, st)) return e;
    }
  }
  if (want_d) {
    // dG_d (c x e) = sum_n X[b,n] (c x l) * Y[b,d,n]^T (l x e): one k-segment per origin row n; static supports add every sample
    // (one launch each) into the dG_o result, the stack's one gradient
    SgemmParams p{};
    p.M = (int)N; p.N = (int)N; p.K = (int)C;
    p.a_si = C; p.a_sk = 1; p.b_sk = 1; p.b_sj = C; p.d_si = N;
    p.nseg = (int)N; p.a_sseg = N * C; p.b_sseg = N * C;
    p.ksplit = 1; p.alpha = 1.f;
    if (s.dynamic) {
      p.A = X; p.B = Y; p.D = dGd;
      p.Z0 = s.B; p.Z1 = (int)Kd; p.Z2 = 1;
      p.a_sz[0] = NN * C; p.b_sz[0] = Kd * NN * C; p.b_sz[1] = NN * C; p.d_sz[0] = Kd * NN; p.d_sz[1] = NN;
      if (int e = simt_sgemm(p, st)) return e;
    } else {
      p.Z0 = (int)Kd; p.Z1 = 1; p.Z2 = 1;
      p.b_sz[0] = NN * C; p.d_sz[0] = NN;
      p.D = dGo; p.Cin = dGo; p.beta = 1.f; p.c_sz[0] = NN;
      for (int b = 0; b < s.B; ++b) {
        p.A = X + (size_t)b * NN * C; p.B = Y + (size_t)b * Kd * NN * C;
          if (int e = simt_sgemm(p, st)) return e;
      }
    }
  }
  return 0;
}

}  // namespace mpgcn
