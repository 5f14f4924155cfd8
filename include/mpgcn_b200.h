/* mpgcn_b200 -- C ABI of the H100-native MPGCN hot path.
 *
 * The reference (underdoc-wang/MPGCN) has no FFI: its "plugin boundary" for this path is the
 * Python module surface `MPGCN.BDGCN` / `MPGCN.MPGCN` (reference MPGCN.py:6-50, 54-112), whose
 * arithmetic it delegates to torch.einsum / nn.LSTM.  These entry points are what a binding
 * for that surface calls instead; `mpgcn_b200/MPGCN.py` is that binding (ctypes), and
 * INTEGRATION.md shows the stub a reference maintainer would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer on the current CUDA device unless stated otherwise;
 *     tensors are dense, row-major (last index fastest), fp32 (`float`), in the reference's own
 *     layouts; nothing is mutated except the documented outputs;
 *   - `stream` is a cudaStream_t (0 = default stream); all work is enqueued on it and the
 *     calls return without synchronising;
 *   - return value 0 = success; non-zero = failure, message from mpgcn_last_error()
 *     (thread-local).  Nothing ever aborts the process;
 *   - `precision`: 0 = exact fp32 CUDA-core kernels; 1 = fp16-operand / fp32-accumulate
 *     wgmma tensor-core engine (requires C and H to be multiples of 32, H <= 1024, C != H allowed;
 *     any number of supports K);
 *   - tensors must be 16-byte aligned; the outputs of the precision-1 layer (`out`, `dX`, `out_f16`) 32-byte aligned
 *     (256-bit stores).  Allocator-returned buffers always are;
 *   - `workspace` is caller-owned scratch of at least the size the matching *_workspace_bytes
 *     query returns (256-byte aligned); `saved` is the activation stash forward fills for
 *     backward (size from mpgcn_bdgcn_saved_bytes, 64-byte aligned); pass NULL for inference.
 */
#ifndef MPGCN_B200_H_
#define MPGCN_B200_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MPGCN_B200_ABI_VERSION 4   /* 2: extras struct, prepared supports, LSTM training pair, dg_absmax, dyn graphs;
                                      3: layer parts (origin-row / support shards), bias_act, relu_backward, region tags;
                                      4: peer push removed: mpgcn_bdgcn_part loses peer_g / peer_rank / peer_out,
                                         mpgcn_rows_reduce_bias_act loses part_rows */

#if defined(__GNUC__)
#define MPGCN_API __attribute__((visibility("default")))
#else
#define MPGCN_API
#endif

MPGCN_API int mpgcn_abi_version(void);
MPGCN_API const char* mpgcn_last_error(void);

/* Deterministic mode of the CALLING HOST THREAD (thread-local, off by default; DESIGN.md section 11).  With it on, every sum that
 * the default kernels form across CTAs with floating-point atomics -- the LSTM weight and bias gradients, the BDGCN bias gradient,
 * the fp32 BDGCN dW, the head's dw / db, the column norms of mpgcn_dyn_graph_build -- is formed from per-CTA partials ("slots") in
 * the workspace, added by one kernel in a fixed order.  Results are then bitwise reproducible for a given shape on a given GPU model
 * and SM count (the promise cuBLAS makes), whatever runs concurrently.  The workspace queries of the affected calls read the same
 * mode (they grow by the slots; with the mode off they return what they always did), and every call checks before its first CUDA
 * call that its workspace is large enough for the current mode.  mpgcn_head_backward has no workspace: with the mode on it refuses,
 * and mpgcn_head_backward_ex takes one.  mpgcn_relu_backward and mpgcn_relu_backward_scatter[_f16] have no deterministic
 * implementation: with the mode on they return an error.  set returns the previous value. */
MPGCN_API int mpgcn_set_deterministic(int on);
MPGCN_API int mpgcn_get_deterministic(void);

/* 1 if `precision` can serve this layer shape, else 0 (replaces nothing in the reference; the
 * Python binding uses it to pick the kernel family). */
MPGCN_API int mpgcn_bdgcn_precision_supported(int B, int N, int K, int C, int H, int precision);

MPGCN_API size_t mpgcn_bdgcn_saved_bytes(int B, int N, int K, int C, int H, int precision);
MPGCN_API size_t mpgcn_bdgcn_fwd_workspace_bytes(int B, int N, int K, int C, int H, int dynamic, int precision);
MPGCN_API size_t mpgcn_bdgcn_bwd_workspace_bytes(int B, int N, int K, int C, int H, int dynamic, int precision);

/* BDGCN.forward  (reference MPGCN.py:24-50):
 *     out[b,m,e,h] = act( sum_{o,d,l} ( sum_{n,c} G_o[n,m] X[b,n,c,l] G_d[c,e] ) W[(o*K+d)*C+l, h] + bias[h] )
 *   X   [B,N,N,C]
 *   G_o, G_d : static graph  (dynamic == 0): both point to the same [K,N,N] support stack
 *                                             (MPGCN.py:26-32);
 *              dynamic graph (dynamic == 1): [B,K,N,N] origin / destination stacks, the two
 *                                             members of the reference's tuple (MPGCN.py:34-40)
 *   W   [K*K*C, H]   bias [H] or NULL (use_bias=False)   act: 0 = None, 1 = ReLU (MPGCN.py:13,49)
 *   out [B,N,N,H] */
MPGCN_API int mpgcn_bdgcn_forward(const float* X, const float* G_o, const float* G_d, int dynamic, const float* W, const float* bias, int act,
                        float* out, void* saved, void* workspace, size_t workspace_bytes, int B, int N, int K, int C, int H,
                        int precision, void* stream);

/* Gradients autograd derives through MPGCN.py:24-50 (loss.backward(), Model_Trainer.py:114).
 *   d_out [B,N,N,H], out = forward output (for the ReLU mask), saved = forward stash
 *   dX [B,N,N,C] or NULL (input needs no grad), dW [K*K*C,H], db [H] or NULL */
MPGCN_API int mpgcn_bdgcn_backward(const float* d_out, const float* out, const float* G_o, const float* G_d, int dynamic, const float* W, int act,
                         const void* saved, float* dX, float* dW, float* db, void* workspace, size_t workspace_bytes, int B, int N,
                         int K, int C, int H, int precision, void* stream);

/* Optional side inputs / outputs of the tensor-core layer (precision 1; ignored by precision 0).  They carry what a caller that
 * chains layers already has, so that the library does not redo it; every field is nullable and results do not depend on them:
 *   go_prepared, gd_prepared   supports converted once by mpgcn_bdgcn_prepare_supports (the same G_o / G_d serve every layer of a
 *                              branch, forward and backward -- "each support staged once and reused");
 *   x_f16                      forward: an fp16 copy of X (same layout), e.g. the out_f16 of the previous layer: skips the cast;
 *   out_f16                    forward: receives an fp16 copy of `out`;  backward: that copy, read for the ReLU mask instead of
 *                              the fp32 `out` (`out` may then be NULL);
 *   d_out_absmax, dX_absmax    backward: the gradient-magnitude hand-over described below. */
typedef struct mpgcn_bdgcn_extras {
  const void* go_prepared;
  const void* gd_prepared;
  const void* x_f16;
  void* out_f16;
  const float* d_out_absmax;
  float* dX_absmax;
  /* ABI 3, backward_part only: dPre [B,N,N,H] already masked, multiplied by d_pre_scale2[0] and cast to fp16, with its device
   * [S, 1/S] pair -- what mpgcn_relu_backward_scatter_f16 leaves in every rank's buffer; the fp32 d_pre argument may then be NULL */
  const void* d_pre_f16;
  const float* d_pre_scale2;
} mpgcn_bdgcn_extras;

/* planes = (dynamic ? B : 1) * K support matrices [N,N] -> fp16 padded copy + diagonal remainders (256-byte aligned buffer) */
MPGCN_API size_t mpgcn_bdgcn_supports_prepared_bytes(long long planes, int N);
MPGCN_API int mpgcn_bdgcn_prepare_supports(const float* G, void* prepared, size_t prepared_bytes, long long planes, int N, void* stream);
/* mpgcn_bdgcn_forward / mpgcn_bdgcn_backward with the optional extras (extras == NULL: identical to the plain calls) */
MPGCN_API int mpgcn_bdgcn_forward_x(const float* X, const float* G_o, const float* G_d, int dynamic, const float* W, const float* bias, int act,
                          float* out, void* saved, void* workspace, size_t workspace_bytes, int B, int N, int K, int C, int H,
                          int precision, const mpgcn_bdgcn_extras* extras, void* stream);
MPGCN_API int mpgcn_bdgcn_backward_x(const float* d_out, const float* out, const float* G_o, const float* G_d, int dynamic, const float* W, int act,
                           const void* saved, float* dX, float* dW, float* db, void* workspace, size_t workspace_bytes, int B, int N,
                           int K, int C, int H, int precision, const mpgcn_bdgcn_extras* extras, void* stream);

/* Same, with the gradient-magnitude hand-over used by the fp16 path: d_out_absmax (nullable) = device scalar already holding
 * max|d_out| (as written by the call that produced d_out; skips one pass over d_out); dX_absmax (nullable) receives max|dX|
 * (0 when unknown).  Pure optimisation: results are identical with or without the hints. */
MPGCN_API int mpgcn_bdgcn_backward_ex(const float* d_out, const float* out, const float* G_o, const float* G_d, int dynamic, const float* W, int act,
                            const void* saved, float* dX, float* dW, float* db, void* workspace, size_t workspace_bytes, int B, int N,
                            int K, int C, int H, int precision, const float* d_out_absmax, float* dX_absmax, void* stream);

/* Gradient with respect to the supports (learnable G): mpgcn_bdgcn_backward_x plus
 *     dG_o[n,m] = sum_{b,e,h} U_o[b,n,e,h] dPre[b,m,e,h]   (U_o = sum_d (G_d-transformed X)_d W[o,d], recomputed from `saved`)
 *     dG_d[c,e] = sum_{b,n,l} X[b,n,c,l] Y_d[b,n,e,l]      (Y_d = sum_o (G_o dPre)_o W[o,d]^T)
 * static supports (G_o == G_d == G [K,N,N]): dG_o receives dL/dG [K,N,N] = dG_o + dG_d summed over the batch; dG_d must be NULL.
 * dynamic supports: dG_o [B,K,N,N] and dG_d [B,K,N,N], either of them NULL when not wanted.  X [B,N,N,C] is the forward's input;
 * dX, dW and db are bitwise those of mpgcn_bdgcn_backward_x on the same arguments (the dG stages run after its stages).  Adds
 * 2 K B N^3 (C + H) flops.  workspace: mpgcn_bdgcn_support_grad_workspace_bytes (at least the backward's). */
MPGCN_API size_t mpgcn_bdgcn_support_grad_workspace_bytes(int B, int N, int K, int C, int H, int dynamic, int precision);
MPGCN_API int mpgcn_bdgcn_backward_supports(const float* d_out, const float* out, const float* G_o, const float* G_d, int dynamic, const float* W,
                                  int act, const void* saved, float* dX, float* dW, float* db, void* workspace, size_t workspace_bytes,
                                  int B, int N, int K, int C, int H, int precision, const mpgcn_bdgcn_extras* extras, const float* X,
                                  float* dG_o, float* dG_d, void* stream);

/* ---- Sparse static supports (DESIGN.md section 12) --------------------------------------------------------------------------------
 * A static [K,N,N] stack given by its nonzeros runs the precision-0 layer with its four N^3 contractions (Z = X x_2 G_d,
 * out = sum_o G_o^T x_1 U_o, V = G_o x_1 dPre, dX = sum_d Y_d x_2 G_d^T) replaced by gathers over the stored entries: 2 B N nnz ch
 * flops each instead of 2 B K N^3 ch.  Results are fp32, each output element summed in a fixed order (support, then ascending index),
 * so they do not depend on mpgcn_set_deterministic.  Only stored entries are multiplied: a non-finite X does not reach an output
 * through a zero of G (the dense layer's 0 * inf = NaN).
 *   mpgcn_sparse_supports_build: indices [3][nnz] int64 (support k, row, column; torch's COO `indices()`), values [nnz] fp32, in any
 *   order; duplicates are kept and add up; entries outside [0,K) x [0,N) x [0,N) are ignored.  Builds the CSR and CSC of every support
 *   (int32 indices) into `supports` (mpgcn_sparse_supports_bytes, 256-byte aligned; 0 for K < 1, N < 1, nnz < 0 or nnz >= 2^31)
 *   with a counting sort on the device, without synchronising.  The buffer must stay unmodified while layer calls use it.
 *   mpgcn_bdgcn_forward_sparse / _backward_sparse: mpgcn_bdgcn_forward / _backward (precision 0, static supports) with G_o, G_d and
 *   `dynamic` replaced by that buffer, its size and nnz.  saved, workspaces: the precision-0 queries (mpgcn_bdgcn_saved_bytes,
 *   mpgcn_bdgcn_fwd / _bwd_workspace_bytes with dynamic 0, precision 0).  Every argument is checked before the first CUDA call.
 *   Their gathers count as tag 7 (fp32 SIMT) launches with flops 2 B N nnz ch; they open no layer region (tags 11, 12). */
MPGCN_API size_t mpgcn_sparse_supports_bytes(int K, int N, long long nnz);
MPGCN_API int mpgcn_sparse_supports_build(const long long* indices, const float* values, long long nnz, int K, int N, void* supports,
                                          size_t supports_bytes, void* stream);
MPGCN_API int mpgcn_bdgcn_forward_sparse(const float* X, const void* supports, size_t supports_bytes, long long nnz, const float* W,
                                         const float* bias, int act, float* out, void* saved, void* workspace, size_t workspace_bytes,
                                         int B, int N, int K, int C, int H, void* stream);
MPGCN_API int mpgcn_bdgcn_backward_sparse(const float* d_out, const float* out, const void* supports, size_t supports_bytes, long long nnz,
                                          const float* W, int act, const void* saved, float* dX, float* dW, float* db, void* workspace,
                                          size_t workspace_bytes, int B, int N, int K, int C, int H, void* stream);

/* ---- PARTS of a layer: what one GPU evaluates when a layer is sharded (SURVEY.md section 8(e)) -----------------------------------
 * The reference has no multi-GPU code; these entry points are the engine's own addition behind the same BDGCN.forward math
 * (MPGCN.py:24-50).  A part is described by
 *     rows [row0, row0 + rows) of the N ORIGIN rows n that this call holds of X / dX (and of the internal Z, U, V, Y), and
 *     Ko origin supports in G_o ([Ko,N,N] or [B,Ko,N,N]), Kd destination supports in G_d, W = the [Ko*Kd*C, H] slice of the
 *     layer's weight in (o, d, l) row order.
 *   origin-row shard (8(e) row 1): rows = N / g, Ko = Kd = K, the same G for every rank;
 *   K shard          (8(e) row 2): rows = N, Ko = K, Kd = K / g, G_d = this rank's destination supports, W[:, D_j] its slice.
 * forward_part writes the RAW PARTIAL pre-activation for EVERY origin row m
 *     pre_partial[b,m,e,h] = sum_{o < Ko} sum_{n in rows} G_o[n,m] * ( sum_{d < Kd, l} (sum_c X[b,n,c,l] G_d[c,e]) W[o,d,l,h] )
 * -- no bias, no activation: the caller sums the partials over the ranks (reduce-scatter over m / all-reduce) and then applies
 * mpgcn_bias_act.  backward_part takes dPre [B,N,N,H] for every origin row m (the caller masks its own rows with
 * mpgcn_relu_backward and all-gathers them / has them replicated) and returns dX for its rows ([B,rows,N,C]; K shard: the
 * partial sum over its d, to be all-reduced) and dW for its slice (row shard: partial over its rows, to be all-reduced).
 *   X [B,rows,N,C]   pre_partial [B,N,N,H] (required)   saved: mpgcn_bdgcn_part_saved_bytes   d_pre [B,N,N,H]   dX [B,rows,N,C] or NULL
 *   extras (nullable): go_prepared / gd_prepared (supports converted once by mpgcn_bdgcn_prepare_supports), d_out_absmax (= max|d_pre|
 *   already known), d_pre_f16 + d_pre_scale2 (backward: the fp16 dPre produced by mpgcn_relu_backward_scatter_f16). */
typedef struct mpgcn_bdgcn_part {
  int row0, rows;
  int Ko, Kd;
} mpgcn_bdgcn_part;
MPGCN_API size_t mpgcn_bdgcn_part_saved_bytes(int B, int N, int C, int H, int precision, const mpgcn_bdgcn_part* part);
MPGCN_API size_t mpgcn_bdgcn_part_fwd_workspace_bytes(int B, int N, int C, int H, int dynamic, int precision, const mpgcn_bdgcn_part* part);
MPGCN_API size_t mpgcn_bdgcn_part_bwd_workspace_bytes(int B, int N, int C, int H, int dynamic, int precision, const mpgcn_bdgcn_part* part);
MPGCN_API int mpgcn_bdgcn_forward_part(const float* X, const float* G_o, const float* G_d, int dynamic, const float* W, float* pre_partial,
                             void* saved, void* workspace, size_t workspace_bytes, int B, int N, int C, int H, int precision,
                             const mpgcn_bdgcn_part* part, const mpgcn_bdgcn_extras* extras, void* stream);
MPGCN_API int mpgcn_bdgcn_backward_part(const float* d_pre, const float* G_o, const float* G_d, int dynamic, const float* W, const void* saved,
                              float* dX, float* dW, void* workspace, size_t workspace_bytes, int B, int N, int C, int H, int precision,
                              const mpgcn_bdgcn_part* part, const mpgcn_bdgcn_extras* extras, void* stream);
/* x[i] = act(x[i] + bias[i % H]) in place -- the `+= b`, activation of MPGCN.py:47-49, applied AFTER the exchange step */
MPGCN_API int mpgcn_bias_act(float* x, const float* bias, int act, long long n, int H, void* stream);
/* d_pre = d_out * [out > 0] (act 1) or d_out (act 0); db[h] = sum d_pre (nullable) -- the head of the backward, BEFORE the exchange */
MPGCN_API int mpgcn_relu_backward(const float* d_out, const float* out, int act, float* d_pre, float* db, long long n, int H, void* stream);

/* The two exchange steps of the origin-row shard, fused into this library's own kernels over PEER memory (NVLink P2P): no separate
 * collective.  `partials` / `dsts` are HOST arrays of g <= 8 DEVICE pointers to [B,N,N,H] fp32 buffers -- the rank's own and its peers'
 * buffers mapped into this process (symmetric memory / CUDA IPC); the caller places a barrier between the producers and these calls.
 *   rows_reduce_bias_act:  out[b,r,e,h] = act( sum_j partials[j][b, row0 + r, e, h] + bias[h] )   out [B,rows,N,H]
 *        = reduce-scatter of the partial pre-activations (each rank reads ITS rows from every rank) + MPGCN.py:47-49;
 *   relu_backward_scatter: d_pre = d_out * [out > 0] (d_out, out [B,rows,N,H]) stored to rows [row0, row0 + rows) of EVERY dsts[j];
 *        db[h] = sum d_pre (nullable)   = ReLU mask + all-gather of dPre.
 * rows_reduce_bias_act takes any H >= 1, relu_backward_scatter and its fp16 flavour any 1 <= H <= 1024. */
MPGCN_API int mpgcn_rows_reduce_bias_act(float* out, const float* const* partials, int g, const float* bias, int act, int B, int N, int row0,
                               int rows, int H, void* stream);
MPGCN_API int mpgcn_relu_backward_scatter(const float* d_out, const float* out, int act, float* const* dsts, int g, float* db, int B, int N,
                                int row0, int rows, int H, void* stream);
/* The same for the tensor-core path with its fp16 cast folded in: absmax = device scalar holding the GLOBAL max|d_out| (every rank's
 * mpgcn_absmax reduced with MAX), scale2 [2] receives [S, 1/S] (S = 2^k, S * absmax in [16, 32)); dsts[j] are fp16 [B,N,N,H] buffers
 * that receive fp16(S * d_pre): half the bytes on the wire, and no rank runs a cast or absmax pass over the gathered tensor. */
MPGCN_API int mpgcn_relu_backward_scatter_f16(const float* d_out, const float* out, int act, void* const* dsts, int g, float* db,
                                    const float* absmax, float* scale2, int B, int N, int row0, int rows, int H, void* stream);
MPGCN_API int mpgcn_absmax(const float* x, long long n, float* out, void* stream);

/* nn.LSTM(input_size=1, hidden=C, layers=1, batch_first) over the B*NN OD cells with zero initial
 * state, returning only the last hidden state (reference MPGCN.py:69,80-87,100-104).
 *   x_seq [B,T,NN] (= the model input [B,T,N,N,1] unchanged, NN = N*N)
 *   w_ih [4C,1], w_hh [4C,C], b_ih [4C], b_hh [4C]   (gate order i,f,g,o)
 *   hT   [B*NN, C]
 * precision 0: fp32 CUDA-core kernels (C <= 64, and T no longer than their backward's shared-memory stash holds: 15 steps at
 * C = 64, 224 at 32, 8041 at 1; mpgcn_lstm_precision_supported answers it); precision 1: tensor-core gate GEMM with the recurrent h rounded to
 * fp16 as MMA operand, state and activations in fp32 (C = 32, 96 or 128; 1 <= T <= 256); x enters that GEMM as an fp16
 * hi + lo pair, exact to ~22 bits for |x| < 65504 and saturating beyond. */
MPGCN_API int mpgcn_lstm_precision_supported(int T, int C, int precision);
MPGCN_API size_t mpgcn_lstm_bwd_workspace_bytes(int B, int T, long long NN, int C, int precision);
MPGCN_API int mpgcn_lstm_last_forward(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, float* hT,
                            int B, int T, long long NN, int C, int precision, void* stream);
/* BPTT for the above. d_hT [B*NN,C]; outputs d_w_ih [4C], d_w_hh [4C,C], d_b_ih [4C], d_b_hh [4C];
 * d_x [B,T,NN] or NULL; workspace from mpgcn_lstm_bwd_workspace_bytes (256-byte aligned). */
MPGCN_API int mpgcn_lstm_last_backward(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                             const float* d_hT, float* d_w_ih, float* d_w_hh, float* d_b_ih, float* d_b_hh, float* d_x, void* workspace,
                             size_t workspace_bytes, int B, int T, long long NN, int C, int precision, void* stream);

/* Support-matrix builder = Adj_Processor(kernel_type, K).process(flow) (reference GCN.py:56-138), batched on the device:
 *   flow [B,N,N] -> supports [B,Ks,N,N], Ks = mpgcn_adj_num_supports(kernel_type, K)
 *   kernel_type: 0 localpool (K ignored, Ks = 1), 1 chebyshev (Ks = K+1; lambda_max = 2, the branch the reference always
 *   takes on torch >= 2), 2 random_walk_diffusion (Ks = K+1), 3 dual_random_walk_diffusion (Ks = 2K+1); anything else is an
 *   error with the reference's message. */
MPGCN_API int mpgcn_adj_num_supports(int kernel_type, int K);
MPGCN_API size_t mpgcn_adj_workspace_bytes(int B, int N, int kernel_type, int K);
MPGCN_API int mpgcn_adj_process(const float* flow, float* supports, int B, int N, int kernel_type, int K, void* workspace, size_t workspace_bytes,
                      void* stream);
/* Its adjoint: d_flow [B,N,N] = dL/dflow from d_supports [B,Ks,N,N] = dL/dsupports, given the forward's flow and its output
 * supports (read, not recomputed).  All fp32 on CUDA cores: the Chebyshev recursion's adjoint is 2(K-1) N^3 SGEMMs per series per
 * batch element.  Where the forward masked 1/sum to 0 (random walk, both series) that row's or column's contribution is exactly 0;
 * the symmetric kernels give non-finite values where their forward does.  K = 0 (identity only): d_flow = 0.  No allocation, no
 * synchronisation; arguments are checked before any CUDA call.  workspace: mpgcn_adj_backward_workspace_bytes (0: bad arguments). */
MPGCN_API size_t mpgcn_adj_backward_workspace_bytes(int B, int N, int kernel_type, int K);
MPGCN_API int mpgcn_adj_process_backward(const float* flow, const float* supports, const float* d_supports, float* d_flow, int B, int N,
                               int kernel_type, int K, void* workspace, size_t workspace_bytes, void* stream);

MPGCN_API int mpgcn_lstm_last_backward_ex(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                                const float* d_hT, float* d_w_ih, float* d_w_hh, float* d_b_ih, float* d_b_hh, float* d_x, void* workspace,
                                size_t workspace_bytes, int B, int T, long long NN, int C, int precision, const float* d_hT_absmax,
                                void* stream);

/* Training pair for the LSTM (what autograd keeps between nn.LSTM's forward and backward, MPGCN.py:100-104 under
 * loss.backward(), Model_Trainer.py:114).  The forward additionally writes c_t and h_t of every step (fp16) into `saved`
 * (mpgcn_lstm_saved_bytes; 0 for precision 0, whose backward recomputes; 16-byte aligned; NULL = plain inference forward);
 * the backward walks that buffer once in reverse.  With saved == NULL the backward is mpgcn_lstm_last_backward_ex: it first
 * rebuilds that state in its workspace (mpgcn_lstm_bwd_workspace_bytes includes the saved size); with saved != NULL the
 * workspace needs mpgcn_lstm_bwd_workspace_bytes - mpgcn_lstm_saved_bytes bytes: 1024 at C = 32, and at C = 96, 128 also
 * the fp16 gate gradients of every cell and step (4C halves each), which a separate pass reduces to d_w_*.  The saved state
 * takes 2C halves per cell and step (C = 32: 128-cell tiles; 96: 64-cell; 128: 48-cell). */
MPGCN_API size_t mpgcn_lstm_saved_bytes(int B, int T, long long NN, int C, int precision);
MPGCN_API int mpgcn_lstm_last_forward_train(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                                  float* hT, void* saved, size_t saved_bytes, int B, int T, long long NN, int C, int precision,
                                  void* stream);
MPGCN_API int mpgcn_lstm_last_backward_saved(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                                   const float* d_hT, float* d_w_ih, float* d_w_hh, float* d_b_ih, float* d_b_hh, float* d_x,
                                   const void* saved, size_t saved_bytes, void* workspace, size_t workspace_bytes, int B, int T,
                                   long long NN, int C, int precision, const float* d_hT_absmax, void* stream);

/* Stacked LSTM: nn.LSTM(input_size=1, hidden=C, num_layers=L, batch_first) over the B*NN OD cells with zero initial state,
 * last hidden state of the top layer only (reference MPGCN.py:69,80-87,100-104 with lstm_num_layers = L).  Tensor cores
 * (precision 1) at C = 32 and 96, L >= 2, 1 <= T <= 256; mpgcn_lstm_stack_supported answers it (L = 1: the single-layer
 * query, whose entry points are mpgcn_lstm_last_*).  Per-layer parameters are HOST arrays of L device pointers in nn.LSTM's
 * layout: w_ih[0] [4C,1], w_ih[l > 0] [4C,C], w_hh[l] [4C,C], b_ih[l], b_hh[l] [4C]; the gradients likewise.
 * Forward: with saved != NULL (mpgcn_lstm_stack_saved_bytes, 256-byte aligned) the training state c_t, h_t of every layer
 * and step; with saved == NULL an inference forward that keeps only the h sequence of the layer below in the workspace
 * (mpgcn_lstm_stack_fwd_workspace_bytes; unused in training).  Backward from that saved state (there is no recomputing
 * flavour): workspace from mpgcn_lstm_stack_bwd_workspace_bytes, d_x [B,T,NN] or NULL, d_hT_absmax as in
 * mpgcn_lstm_last_backward_ex.  All buffers 256-byte aligned.  Backward workspace layout: [S, 1/S] (1024 B), the fp32 sequence
 * d(h^{l-1}_t) handed from walk to walk (C floats per cell and step, DESIGN.md 6.4), then the fp16 gate-gradient records of one layer, reused
 * by every layer; a workspace with L - 1 more record regions (each of the size the query counts) keeps every layer's records. */
MPGCN_API int mpgcn_lstm_stack_supported(int T, int C, int L, int precision);
MPGCN_API size_t mpgcn_lstm_stack_saved_bytes(int B, int T, long long NN, int C, int L, int precision);
MPGCN_API size_t mpgcn_lstm_stack_fwd_workspace_bytes(int B, int T, long long NN, int C, int L, int precision);
MPGCN_API size_t mpgcn_lstm_stack_bwd_workspace_bytes(int B, int T, long long NN, int C, int L, int precision);
MPGCN_API int mpgcn_lstm_stack_forward(const float* x_seq, int L, const float* const* w_ih, const float* const* w_hh,
                                       const float* const* b_ih, const float* const* b_hh, float* hT, void* saved, size_t saved_bytes,
                                       void* workspace, size_t workspace_bytes, int B, int T, long long NN, int C, int precision,
                                       void* stream);
MPGCN_API int mpgcn_lstm_stack_backward(const float* x_seq, int L, const float* const* w_ih, const float* const* w_hh,
                                        const float* const* b_ih, const float* const* b_hh, const float* d_hT, float* const* d_w_ih,
                                        float* const* d_w_hh, float* const* d_b_ih, float* const* d_b_hh, float* d_x, const void* saved,
                                        size_t saved_bytes, void* workspace, size_t workspace_bytes, int B, int T, long long NN, int C,
                                        int precision, const float* d_hT_absmax, void* stream);

/* Recomputing LSTM backward (L = 1 or a stack; precision 1 wherever mpgcn_lstm_stack_supported(T, C, L, 1) holds), for a
 * forward that kept no training state: mpgcn_lstm_last_forward, or mpgcn_lstm_stack_forward with saved == NULL.  The state
 * is rebuilt and walked back one chunk of cells at a time, so the workspace is O(chunk_cells), not O(B NN T C), at the cost of
 * one more forward.  A chunk is chunk_cells (>= 1) rounded up to whole tiles, at least one wave of the backward grid, at most
 * every cell.  d_x and the per-cell gradients are bitwise those of mpgcn_lstm_last_backward_saved / mpgcn_lstm_stack_backward;
 * the weight gradients differ in fp32 summation order only.  Parameters as mpgcn_lstm_stack_backward's (HOST arrays of L
 * device pointers).  Workspace (256-byte aligned) from mpgcn_lstm_recompute_bwd_workspace_bytes (0: arguments it does not
 * support): [S, 1/S] (1024 B), a stack's fp32 d(h^{l-1}_t) sequence of one chunk, deterministic mode's slots (one region per
 * layer), the chunk's saved state of every layer, and at C = 96, 128 or in a stack the chunk's gate-gradient records. */
MPGCN_API size_t mpgcn_lstm_recompute_bwd_workspace_bytes(int B, int T, long long NN, int C, int L, long long chunk_cells, int precision);
MPGCN_API int mpgcn_lstm_backward_recompute(const float* x_seq, int L, const float* const* w_ih, const float* const* w_hh,
                                            const float* const* b_ih, const float* const* b_hh, const float* d_hT, float* const* d_w_ih,
                                            float* const* d_w_hh, float* const* d_b_ih, float* const* d_b_hh, float* d_x,
                                            long long chunk_cells, void* workspace, size_t workspace_bytes, int B, int T, long long NN,
                                            int C, int precision, const float* d_hT_absmax, void* stream);

/* Dynamic origin / destination graphs from the OD history = DataInput.construct_dyn_G (reference Data_Container_OD.py:39-59).
 *   od_history [periods * P, N, N]  the first periods*P days of the (un-normalised) OD tensor, P = perceived period (7)
 *   o_graph, d_graph [P, N, N]      slot t: A_t = mean_k od_history[t + k P];
 *       o_graph[t][i][j] = cosine_distance(A_t[i,:], A_t[j,:])            (:50-52)
 *       d_graph[t][i][j] = cosine_distance(A_t[:,i], A_t[j,:])            (:54-56: column i against ROW j, as the reference does)
 *   cosine_distance = clip(1 - u.v / sqrt(u.u v.v), 0, 2) (scipy), NaN for a zero vector.  fp32 on the device (the reference
 *   is float64 on the host): absolute error ~1e-6.  The reference stacks the slots on the LAST axis ([N,N,P]); the Python
 *   mirror mpgcn_b200.dyn_graph.construct_dyn_G returns that layout. */
MPGCN_API size_t mpgcn_dyn_graph_workspace_bytes(int P, int N);
MPGCN_API int mpgcn_dyn_graph_build(const float* od_history, int periods, float* o_graph, float* d_graph, int P, int N, void* workspace,
                          size_t workspace_bytes, void* stream);

/* FC head + multi-perspective fusion (reference MPGCN.py:74-76,107,110,112), one pass:
 *     y[cell] = (1/M) * sum_m relu( g_m[cell,:] . w[m,:] + bias[m] )      (Linear(C -> 1) + ReLU per branch, mean over the M branches)
 *   g    HOST array of M device pointers, each [cells, C] (cells = B*N*N);  w [M,C], bias [M];  y [cells]
 *   pre  [M,cells] pre-activations kept for backward, or NULL (inference)
 * backward: dy [cells]; dg HOST array of M device pointers [cells, C] (or NULL / NULL entries), dw [M,C], db [M];
 * dg_absmax [M] (nullable) receives max|dg_m| per branch (see mpgcn_bdgcn_backward_ex).
 * 1 <= M <= 8, C a multiple of 4; w, every g[m] (never NULL) and every non-NULL dg[m] 16-byte aligned: checked before any CUDA call. */
MPGCN_API int mpgcn_head_forward(const float* const* g, const float* w, const float* bias, float* y, float* pre, long long cells, int C, int M,
                       void* stream);
MPGCN_API int mpgcn_head_backward(const float* const* g, const float* w, const float* pre, const float* dy, float* const* dg, float* dw, float* db,
                        float* dg_absmax, long long cells, int C, int M, void* stream);
/* The backward with a workspace (256-byte aligned) of mpgcn_head_backward_workspace_bytes: 0 with the deterministic mode off
 * (then identical to mpgcn_head_backward), else one [M*C + M] float slot per block of the kernel's grid. */
MPGCN_API size_t mpgcn_head_backward_workspace_bytes(long long cells, int C, int M);
MPGCN_API int mpgcn_head_backward_ex(const float* const* g, const float* w, const float* pre, const float* dy, float* const* dg, float* dw,
                                     float* db, float* dg_absmax, long long cells, int C, int M, void* workspace, size_t workspace_bytes,
                                     void* stream);

/* Launch accounting (bench.py evidence).  Every launch of a kernel of this library is counted per tag
 * (0 FWD_A, 1 FWD_MIX, 2 FWD_B, 3 BWD_V, 4 BWD_DW, 5 BWD_MIX, 6 BWD_DX: wgmma contractions; 7 fp32 SIMT GEMM;
 * 8 elementwise/layout; 9 LSTM forward; 10 LSTM backward).  With profiling enabled, tags 0-6, 9, 10 are also
 * bracketed by CUDA events on the launch stream; mpgcn_profile_read (HOST pointers; call after synchronising)
 * returns launches, algorithmic flops and summed device milliseconds since the last reset.
 * Tags 11 (mpgcn_bdgcn_forward*), 12 (mpgcn_bdgcn_backward*) and 13 (mpgcn_head_*) are REGIONS: whole C-ABI calls -- every
 * kernel of the call and the gaps between them -- with `launches` counting calls and `flops` the layer's algorithmic work
 * (per sample F_fwd = 2KN^3(C+H) + 2K^2N^2CH, F_bwd = 2KN^3(C+H) + 4K^2N^2CH; DESIGN.md section 2); bench.py's `roofline_layer`.
 * Tag 14: the peer-memory exchange kernels of the row shard (mpgcn_rows_reduce_bias_act, mpgcn_relu_backward_scatter[_f16]), timed.
 * Thread-safe: counters behind a mutex, the open bracket is per calling thread. */
MPGCN_API void mpgcn_profile_enable(int on);
MPGCN_API void mpgcn_profile_reset(void);
MPGCN_API int mpgcn_profile_read(int tag, long long* launches, double* flops, double* ms);

/* Test / diagnostics only: byte offset of an intermediate inside the precision-1 workspace
 * (which: 0 X16, 1 Gd16, 2 Go16, 3 W16, 4 U16 forward; 10 dP16, 11 Gd16, 12 Go16, 13 V16, 14 Y16, 15 Wq16,
 * 16 dW partials backward; 17 = number of dW split-K slices). */
MPGCN_API long long mpgcn_debug_tc_workspace_offset(int which, int B, int N, int K, int dynamic);

#ifdef __cplusplus
}
#endif
#endif /* MPGCN_B200_H_ */
