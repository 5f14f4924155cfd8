// Internal host-side declarations shared by the translation units of libmpgcn_b200.
#pragma once

#include "common.cuh"

namespace mpgcn {

const char* last_error();
void prof_enable(int on);
void prof_reset();
int prof_read(int tag, long long* launches, double* flops, double* ms);

// ---- generic fp32 SIMT strided/batched contraction (simt_kernels.cu) ---------------------
//   D[z](i,j) (+)= alpha * sum_seg sum_k A[z](i,k;seg) * B[z](k,j;seg)  (+ bias[j % bias_mod], ReLU)
struct SgemmParams {
  const float* A;
  const float* B;
  float* D;
  int M, N, K;                 // K per segment
  long long a_si, a_sk;        // element strides of A(i,k)
  long long b_sk, b_sj;        // element strides of B(k,j)
  long long d_si;              // D(i,j): j stride 1
  int nseg;
  long long a_sseg, b_sseg;
  int Z0, Z1, Z2;              // batch z = (z0*Z1 + z1)*Z2 + z2
  long long a_sz[3], b_sz[3], d_sz[3];
  int ksplit;                  // > 1: split each segment's K into slices, atomically add into D (D pre-zeroed) ...
  long long d_sslice;          // ... or, when non-zero, slice s stores its partial at D + s * d_sslice (deterministic mode)
  float alpha;
  const float* bias;
  int bias_mod;
  int relu;
  const float* Cin;            // optional: D = alpha*A*B + beta*Cin (Cin indexed like D); ksplit must be 1
  float beta;
  long long c_sz[3];
};
int simt_sgemm(const SgemmParams& p, cudaStream_t stream);

// ---- fixed-order reduction of per-CTA partials (deterministic mode; simt_kernels.cu) ------------------------------------
// A slot is one CTA's contribution laid out as an "image" of up to three outputs back to back: image[i] for i < end[0] goes to
// dst[0][i], end[0] <= i < end[1] to dst[1][i - end[0]], then dst[2].  For each row a < rows:
//     dst_k[a * width_k + j] = sum_{s < slots} P[a * a_stride + s * s_stride + start_k + j]
// summed in the same order on every run: 32 interleaved groups of slots, each in slot order, then the groups in order.
struct SlotImage {
  float* dst[3];
  long long end[3];
};
SlotImage slot_image(float* d0, long long n0, float* d1 = nullptr, long long n1 = 0, float* d2 = nullptr, long long n2 = 0);
int reduce_slots(const float* P, int slots, long long s_stride, int rows, long long a_stride, const SlotImage& img, cudaStream_t s);
// the slots of the bias gradient of relu_bwd_prep*: one [H] partial per block of its grid (at most 16 blocks per SM)
size_t bias_grad_slot_bytes(int H);

// ---- elementwise / layout helpers (simt_kernels.cu) ---------------------------------------
int cvt_f32_to_f16(const float* src, __half* dst, size_t n, cudaStream_t s);
// delta[p*N + i] = G[p][i][i] - float(fp16(G[p][i][i])) for `planes` N x N matrices
int support_diag_delta(const float* G, float* delta, size_t planes, int N, cudaStream_t s);
// [rows][cols] fp32 -> [rows][ld] fp16 (ld >= cols, padding zeroed)
int cvt_f32_to_f16_padded(const float* src, __half* dst, size_t rows, int cols, int ld, cudaStream_t s);
// bf16x3 (precision 2) operand pairs: [rows][cols] fp32 -> hi = bf16_rn(x) as [rows][ld] (padding zeroed), then lo = bf16_rn(x - hi)
// the same way right behind it (rows * ld elements on); ld = cols converts a plain array
int cvt_f32_to_bf16x3_padded(const float* src, __nv_bfloat16* dst, size_t rows, int cols, int ld, cudaStream_t s);
// d_pre = d_out * (out > 0) (relu) or d_out, 1 <= H <= 1024; exactly one output: fp32, or fp16(scale[0] * d_pre) (scale: device
// scalar); db[h] = sum d_pre (nullable); db_slots (bias_grad_slot_bytes, nullable): db from per-block partials in a fixed order
int relu_bwd_prep(const float* d_out, const float* out, int relu, __half* d_pre16, float* d_pre32, float* db, size_t n, int H,
                  const float* scale, cudaStream_t s, float* db_slots = nullptr);
// the same with the ReLU mask taken from an fp16 copy of the forward output (tensor-core path: fp16 d_pre only)
int relu_bwd_prep_f16mask(const float* d_out, const __half* out16, int relu, __half* d_pre16, float* db, size_t n, int H,
                          const float* scale, cudaStream_t s, float* db_slots = nullptr);
// the same as a bf16x3 pair of scale[0] * d_pre: hi d_pair[0, n), lo d_pair[n, 2n) (fp32 mask)
int relu_bwd_prep_bf16x3(const float* d_out, const float* out, int relu, __nv_bfloat16* d_pair, float* db, size_t n, int H, const float* scale,
                         cudaStream_t s, float* db_slots = nullptr);
// scale2[0] = S = 2^k with S*max|d_out| in [16,32), scale2[1] = 1/S (S = 1 for an all-zero or non-finite input).
// fp16 has 5 exponent bits: realistic gradients (MSE mean over B*N*N cells ~ 1e-7) must be rescaled before the cast.
// absmax_hint: optional device scalar already holding max|d_out| (produced by the epilogue that wrote d_out): skips the pass
int grad_scale_prepare(const float* d_out, size_t n, float* scale2, const float* absmax_hint, cudaStream_t s);
// W[o][d][l][h] fp32 (o < Ko, d < Kd) -> Wq[d][o][h][l] fp32
int permute_w_bwd(const float* W, float* wq32, int Ko, int Kd, int C, int H, cudaStream_t s);
// W[o][d][c][h] fp32 -> the fp16 W operand of a tensor-core channel mix (bdgcn_tc.cu), C and H multiples of 32, c = 32 lc + l,
// h = 32 hc + h':  lo != null: forward, hi / lo = fp16 split as [(hc,o)][(d,lc)][l][h'];  lo == null: backward, [(d,lc)][(o,hc)][h'][l]
int permute_w_mix(const float* W, __half* hi, __half* lo, int Ko, int Kd, int C, int H, cudaStream_t s);
// the same as a bf16x3 pair (fwd: the forward layout; else the backward one), hi pair[0, n), lo pair[n, 2n) for n = Ko*Kd*C*H
int permute_w_mix_bf16x3(const float* W, __nv_bfloat16* pair, int fwd, int Ko, int Kd, int C, int H, cudaStream_t s);
// dW[o][d][c][h] = sum_slices P[slice][d*C + c][o*H + h]   (P: [slice][MT*128 rows][Ko*H]; o < Ko, d < Kd)
int reduce_dw_partials(const float* P, float* dW, int slices, int MT, int Ko, int Kd, int C, int H, const float* inv_scale, cudaStream_t s);
// dG[n][m] (+)= inv_scale * sum_slices P[slice][n][m]   (P: [slice][N][ldp]; n, m < N; accumulate: add to dG)
int reduce_dg_partials(const float* P, float* dG, int slices, int N, int ldp, const float* inv_scale, int accumulate, cudaStream_t s);
// out[p][i] = (row0 <= i < row0 + rows) ? delta[p][i] : 0   (diagonal remainders restricted to an origin-row slab)
int mask_delta_rows(const float* delta, float* out, size_t planes, int N, int row0, int rows, cudaStream_t s);
// x[i] = act(x[i] + bias[i % H]) in place (bias nullable; act 0 none / 1 ReLU): the epilogue a partial layer call leaves out
int bias_act_inplace(float* x, const float* bias, int act, size_t n, int H, cudaStream_t s);
// exchange steps of the origin-row shard fused into elementwise kernels over peer memory (parts / dsts: HOST arrays of g <= 8 DEVICE
// pointers to [B][N][N][H] buffers, the rank's own and its peers' NVLink-mapped ones); rows_reduce_bias_act takes any H >= 1, the
// relu_backward_scatter pair any 1 <= H <= 1024
int rows_reduce_bias_act(float* out, const float* const* parts, int g, const float* bias, int act, int B, int N, int row0, int rows, int H,
                         cudaStream_t s);
// the same with the fp16 cast of the tensor-core path folded in: scale2 = [S, 1/S] from the GLOBAL max|d_out| (device scalar), values
// stored as fp16(S * d_pre) -- half the bytes on the wire and no cast / absmax pass over the gathered tensor on any rank
int relu_backward_scatter_f16(const float* d_out, const float* out, int act, __half* const* dsts, int g, float* db, const float* absmax,
                              float* scale2, int B, int N, int row0, int rows, int H, cudaStream_t s);
int absmax_f32(const float* x, size_t n, float* out, cudaStream_t s);
int relu_backward_scatter(const float* d_out, const float* out, int act, float* const* dsts, int g, float* db, int B, int N, int row0, int rows,
                          int H, cudaStream_t s);

// ---- per-cell LSTM, last hidden state (lstm_kernels.cu) ------------------------------------
int lstm_last_forward(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, float* hT,
                      int B, int T, long long NN, int C, cudaStream_t s);
int lstm_last_backward(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                       const float* d_hT, float* d_w_ih, float* d_w_hh, float* d_b_ih, float* d_b_hh, float* d_x, int B, int T,
                       long long NN, int C, void* ws, size_t ws_bytes, cudaStream_t s);
size_t lstm_bwd_workspace_bytes(int C);
// cells per block of the backward, which keeps every recomputed step of its cells in shared memory; 0 where not even one cell
// fits (T above 15 at hidden 64, 95 at 48, 224 at 32) or C is outside 1..64
int lstm_bwd_cells_per_block(int T, int C);
// d_b_hh = d_b_ih (n = 4C floats): the last step of both LSTM backwards, whose gate bias gradients are the same sum
int lstm_copy_bias_grad(const float* d_b_ih, float* d_b_hh, int n, cudaStream_t st);

// FC head + branch mean (head_kernels.cu); g / dg are HOST arrays of M device pointers
int head_check(const char* what, const float* const* g, const float* w, float* const* dg, int C, int M);
int head_forward(const float* const* g, const float* w, const float* bias, float* y, float* pre, long long cells, int C, int M,
                 cudaStream_t st);
int head_backward(const float* const* g, const float* w, const float* pre, const float* dy, float* const* dg, float* dw, float* db,
                  float* dg_absmax /*[M] or null*/, long long cells, int C, int M, cudaStream_t st, float* slots = nullptr);
// slots of head_backward in deterministic mode: one [M x C | M] partial per block of its grid
size_t head_bwd_slot_bytes(long long cells, int C, int M);

// support-matrix builder (adj_kernels.cu): reference GCN.Adj_Processor.process
enum AdjKernel { ADJ_LOCALPOOL = 0, ADJ_CHEBYSHEV = 1, ADJ_RANDOM_WALK = 2, ADJ_DUAL_RANDOM_WALK = 3 };
int adj_num_supports(int kernel_type, int K);
size_t adj_workspace_bytes(int B, int N);
int adj_process(const float* flow, float* supports, int B, int N, int kernel_type, int K, void* ws, size_t ws_bytes, cudaStream_t st);
// its adjoint: d_flow [B,N,N] from d_supports [B,Ks,N,N], reading the forward's supports (no allocation, no synchronisation)
size_t adj_backward_workspace_bytes(int B, int N, int kernel_type, int K);
int adj_process_backward(const float* flow, const float* supports, const float* d_supports, float* d_flow, int B, int N, int kernel_type,
                         int K, void* ws, size_t ws_bytes, cudaStream_t st);

// dynamic O / D graphs from the OD history (dyn_graph_kernels.cu)
size_t dyn_graph_workspace_bytes(int P, int N);
int dyn_graph_build(const float* od_hist, int periods, float* o_g, float* d_g, int P, int N, void* ws, size_t ws_bytes, cudaStream_t st);

// tensor-core LSTM (lstm_tc.cu): hidden size C = 32, 96, 128; per-layer weights as HOST arrays of L device pointers
bool lstm_tc_supported(int T, int C);
size_t lstm_tc_bwd_workspace_bytes(int B, int T, long long NN, int C);
size_t lstm_tc_saved_bytes(int B, int T, long long NN, int C);
// L = 1 or a stack.  saved (nullable): training state c_t, h_t of every layer written by the forward; the backward walks it
// instead of recomputing the forward.  ws: a stack's inference workspace (lstm_tc_stack_fwd_workspace_bytes), unused otherwise
int lstm_forward_tc(const float* x_seq, int L, const float* const* w_ih, const float* const* w_hh, const float* const* b_ih,
                    const float* const* b_hh, float* hT, void* saved, void* ws, size_t ws_bytes, int B, int T, long long NN, int C,
                    cudaStream_t s);
int lstm_last_backward_tc(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                          const float* d_hT, float* d_w_ih, float* d_w_hh, float* d_b_ih, float* d_b_hh, float* d_x, const void* saved,
                          int B, int T, long long NN, int C, void* ws, size_t ws_bytes, const float* d_hT_absmax, cudaStream_t s);
// stacked (L >= 2 layers) at hidden 32 and 96
bool lstm_tc_stack_supported(int T, int C, int L);
size_t lstm_tc_stack_saved_bytes(int B, int T, long long NN, int C, int L);
size_t lstm_tc_stack_fwd_workspace_bytes(int B, int T, long long NN, int C, int L);
size_t lstm_tc_stack_bwd_workspace_bytes(int B, int T, long long NN, int C, int L);
int lstm_stack_backward_tc(const float* x_seq, int L, const float* const* w_ih, const float* const* w_hh, const float* const* b_ih,
                           const float* const* b_hh, const float* d_hT, float* const* d_w_ih, float* const* d_w_hh, float* const* d_b_ih,
                           float* const* d_b_hh, float* d_x, const void* saved, void* ws, size_t ws_bytes, int B, int T, long long NN,
                           int C, const float* d_hT_absmax, cudaStream_t s);
// backward without training state (L = 1 or a stack): the state is rebuilt and walked back one chunk of chunk_cells cells at a time
size_t lstm_tc_recompute_bwd_workspace_bytes(int B, int T, long long NN, int C, int L, long long chunk_cells);
int lstm_recompute_backward_tc(const float* x_seq, int L, const float* const* w_ih, const float* const* w_hh, const float* const* b_ih,
                               const float* const* b_hh, const float* d_hT, float* const* d_w_ih, float* const* d_w_hh,
                               float* const* d_b_ih, float* const* d_b_hh, float* d_x, long long chunk_cells, void* ws, size_t ws_bytes,
                               int B, int T, long long NN, int C, const float* d_hT_absmax, cudaStream_t s);

// ---- BDGCN layer orchestration ---------------------------------------------------------------
struct BdgcnShape {
  int B, N, K, C, H;
  int dynamic;      // supports are per-sample [B,K,N,N] pairs
  int act;          // 0 none, 1 relu
  // Which PART of the layer this call evaluates (multi-GPU shards, SURVEY.md section 8(e)); a whole layer has
  // R = N, row0 = 0, Ko = Kd = K, partial = 0.
  int R, row0;      // origin rows n in [row0, row0 + R) are present: X / Z / U / V / Y / dX are [B, R, N, *] slabs
  int Ko, Kd;       // supports in G_o / in G_d; W is the [Ko*Kd*C, H] slice in (o, d, l) row order
  int partial;      // forward writes the raw partial pre-activation sum_{o, n in slab} ... (no bias, no activation);
                    // backward receives dPre (already masked) instead of dOut
  bool whole() const { return R == N && row0 == 0 && Ko == K && Kd == K && !partial; }
};
// PREC_BF16X3_TC: the tensor-core layer on bf16 pairs, three products per contraction (bdgcn_tc.cu; DESIGN.md section 3)
enum Precision { PREC_FP32_SIMT = 0, PREC_FP16_TC = 1, PREC_BF16X3_TC = 2 };

bool tc_supported(const BdgcnShape& s);
// buffer sizes of a layer call in either precision (api.cu), from those of each kernel family
size_t bdgcn_saved_bytes(const BdgcnShape& s, int precision);
size_t bdgcn_fwd_workspace_bytes(const BdgcnShape& s, int precision);
size_t bdgcn_bwd_workspace_bytes(const BdgcnShape& s, int precision);
size_t bdgcn_sgrad_workspace_bytes(const BdgcnShape& s, int precision);
size_t simt_saved_bytes(const BdgcnShape& s);
size_t simt_fwd_ws_bytes(const BdgcnShape& s);
size_t simt_bwd_ws_bytes(const BdgcnShape& s);
size_t simt_sgrad_ws_bytes(const BdgcnShape& s);
// bf: the bf16x3 layer (every 16-bit stash / workspace tensor a hi / lo pair)
size_t tc_saved_bytes(const BdgcnShape& s, bool bf = false);
size_t tc_fwd_ws_bytes(const BdgcnShape& s, bool bf = false);
size_t tc_bwd_ws_bytes(const BdgcnShape& s, bool bf = false);
size_t tc_sgrad_ws_bytes(const BdgcnShape& s);
long long tc_debug_offset(const BdgcnShape& s, int which);

// ---- sparse static supports (bdgcn_sparse.cu): CSR and CSC of a [K,N,N] stack in one device buffer ----------------------
struct SparseSupports {
  int K, N;
  long long nnz;
  const int* csr_ptr;          // [K][N + 1] offsets into csr_idx / csr_val (row r of support k: [ptr[k][r], ptr[k][r + 1]))
  const int* csr_idx;          // column of each nonzero, ascending within a row
  const float* csr_val;
  const int* csc_ptr;          // the same for G^T: column c of support k, its rows ascending
  const int* csc_idx;
  const float* csc_val;
};
// K >= 1, N >= 1, 0 <= nnz < 2^31 (int32 indices)
bool sparse_shape_ok(int K, int N, long long nnz);
size_t sparse_supports_bytes(int K, int N, long long nnz);
// indices [3][nnz] int64 (support, row, column), values [nnz]: any order, duplicates kept (they add up); entries outside the stack
// are ignored.  No host synchronisation.
int sparse_supports_build(const long long* indices, const float* values, long long nnz, int K, int N, void* buf, cudaStream_t st);
SparseSupports sparse_supports_view(const void* buf, int K, int N, long long nnz);
// the four N^3 stages of the fp32 layer as gathers over the nonzeros (whole static layers); bias / act: FWD_B's epilogue
enum SparseStage { SPARSE_FWD_A, SPARSE_FWD_B, SPARSE_BWD_V, SPARSE_BWD_DX };
int sparse_stage(SparseStage stage, const BdgcnShape& s, const SparseSupports& sp, const float* in, float* out, const float* bias,
                 cudaStream_t st);

// sp (nullable): sparse static supports, whose gathers replace the four N^3 SGEMMs (Go / Gd unused)
int bdgcn_forward_simt(const BdgcnShape& s, const float* X, const float* Go, const float* Gd, const float* W, const float* bias,
                       float* out, void* saved, void* ws, size_t ws_bytes, cudaStream_t st, const SparseSupports* sp = nullptr);
int bdgcn_backward_simt(const BdgcnShape& s, const float* d_out, const float* out, const float* Go, const float* Gd, const float* W,
                        const void* saved, float* dX, float* dW, float* db, void* ws, size_t ws_bytes, cudaStream_t st,
                        const SparseSupports* sp = nullptr);
// optional side inputs / outputs of the tensor-core layer (mirror of mpgcn_bdgcn_extras in include/mpgcn_b200.h); all nullable
struct BdgcnExtras {
  const void* go_prepared = nullptr;    // supports already converted by bdgcn_prepare_supports (fp16 padded + diagonal remainders)
  const void* gd_prepared = nullptr;
  const void* x_f16 = nullptr;          // forward: fp16 copy of X (skips the conversion pass)
  void* out_f16 = nullptr;              // forward: receives an fp16 copy of out;  backward: that copy (ReLU mask source instead of out)
  const float* d_out_absmax = nullptr;  // backward: max|d_out| already known
  float* dx_absmax = nullptr;           // backward: receives max|dX|
  const void* d_pre_f16 = nullptr;      // backward of a PART: dPre [B,N,N,H] already masked, scaled by scale2[0] and cast to fp16
  const float* d_pre_scale2 = nullptr;  //   ... with its device [S, 1/S] pair (mpgcn_relu_backward_scatter_f16 produces both)
};
// bf: the bf16x3 layer -- supports prepared as a bf16 pair, and whole layers without the fp16 side buffers (x_f16, out_f16, d_pre_f16)
size_t bdgcn_supports_prepared_bytes(long long planes, int N, bool bf = false);
int bdgcn_prepare_supports(const float* G, void* prepared, long long planes, int N, cudaStream_t st, bool bf = false);
int bdgcn_forward_tc(const BdgcnShape& s, const float* X, const float* Go, const float* Gd, const float* W, const float* bias,
                     float* out, void* saved, void* ws, size_t ws_bytes, const BdgcnExtras& ex, cudaStream_t st, bool bf = false);
int bdgcn_backward_tc(const BdgcnShape& s, const float* d_out, const float* out, const float* Go, const float* Gd, const float* W,
                      const void* saved, float* dX, float* dW, float* db, void* ws, size_t ws_bytes, const BdgcnExtras& ex,
                      cudaStream_t st, bool bf = false);
// the backward plus the support gradients (whole layer): static supports get dGo [K][N][N] = dG_o + dG_d summed over the batch
// (dGd unused), dynamic ones dGo [B][K][N][N] and dGd [B][K][N][N] (either nullable).  dX / dW / db are those of the backward.
int bdgcn_backward_supports_tc(const BdgcnShape& s, const float* d_out, const float* out, const float* X, const float* Go, const float* Gd,
                               const float* W, const void* saved, float* dX, float* dW, float* db, float* dGo, float* dGd, void* ws,
                               size_t ws_bytes, const BdgcnExtras& ex, cudaStream_t st);
int bdgcn_backward_supports_simt(const BdgcnShape& s, const float* d_out, const float* out, const float* X, const float* Go, const float* Gd,
                                 const float* W, const void* saved, float* dX, float* dW, float* db, float* dGo, float* dGd, void* ws,
                                 size_t ws_bytes, cudaStream_t st);

}  // namespace mpgcn
