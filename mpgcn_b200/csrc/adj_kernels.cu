// Support-matrix builder on the GPU: the arithmetic of the reference's Adj_Processor.process
// (/root/reference/GCN.py:56-138), batched over the whole [B,N,N] flow tensor instead of a Python loop over the batch on
// the CPU (the reference calls it twice per training step, Model_Trainer.py:84,106).  SURVEY.md section 8(f) rank 1.
//
//   localpool                   I + D^-1/2 A D^-1/2                                   (GCN.py:69-72, 111-114)
//   chebyshev                   x = (2/lambda_max) (I - D^-1/2 A D^-1/2) - I with lambda_max = 2, the branch the reference
//                               always takes on torch >= 2 (torch.eig was removed; bare except, GCN.py:117-126)
//   random_walk_diffusion       x = (D^-1 A)^T, 1/0 -> 0                               (GCN.py:79-82, 103-108)
//   dual_random_walk_diffusion  forward series of (D^-1 A)^T, backward series of (D_T^-1 A^T)^T   (GCN.py:84-91)
//   series: T_0 = I, T_1 = x, T_k = 2 x T_{k-1} - T_{k-2}                              (GCN.py:128-138)
// All fp32: the N^3 recursion runs on the exact CUDA-core SGEMM with a fused "2 A B - C" epilogue.
#include "kernels.h"

namespace mpgcn {

int adj_num_supports(int kernel_type, int K) {
  switch (kernel_type) {
    case ADJ_LOCALPOOL: return 1;
    case ADJ_CHEBYSHEV:
    case ADJ_RANDOM_WALK: return K + 1;
    case ADJ_DUAL_RANDOM_WALK: return 2 * K + 1;
    default: return -1;
  }
}

// forward workspace: row sums and column sums
struct AdjLayout { size_t rowsum, colsum, total; };
static AdjLayout adj_layout(int B, int N) {
  AdjLayout L;
  size_t off = 0;
  L.rowsum = take(off, (size_t)B * N * sizeof(float), 256);
  L.colsum = take(off, (size_t)B * N * sizeof(float), 256);
  L.total = align_up(off, 256) + 256;    // unused padding: the size this workspace has always had
  return L;
}
size_t adj_workspace_bytes(int B, int N) { return adj_layout(B, N).total; }

// sums[b][i] = sum_j A[b][i][j] (by_col = 0) or sum_j A[b][j][i] (by_col = 1); one warp per (b, i)
__global__ void adj_sums_kernel(const float* __restrict__ A, float* __restrict__ sums, int B, int N, int by_col) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= (long long)B * N) return;
  const int b = (int)(w / N), i = (int)(w % N);
  const float* base = A + (size_t)b * N * N;
  float s = 0.f;
  for (int j = lane; j < N; j += 32) s += by_col ? base[(size_t)j * N + i] : base[(size_t)i * N + j];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) sums[w] = s;
}

// mode 0: out = I + sym_norm(A)                      (localpool)
// mode 1: out = (1 * (I - sym_norm(A))) - I            (chebyshev x, lambda_max = 2: same operation order as the reference)
// mode 2: out = (D^-1 A)^T                            (random walk, forward)         out[i][j] = A[j][i] / rowsum[j]
// mode 3: out = (D_T^-1 A^T)^T                        (random walk, backward)        out[i][j] = A[i][j] / colsum[j]
// `out` is support k_out of a [B][Ks][N][N] stack; optionally the identity is written to support 0.
__global__ void adj_build_kernel(const float* __restrict__ A, const float* __restrict__ rowsum, const float* __restrict__ colsum,
                                 float* __restrict__ sup, int B, int N, int Ks, int k_out, int mode, int write_identity) {
  const size_t total = (size_t)B * N * N;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
    const int j = (int)(t % N);
    const int i = (int)((t / N) % N);
    const int b = (int)(t / ((size_t)N * N));
    const float* Ab = A + (size_t)b * N * N;
    float v;
    if (mode <= 1) {
      const float di = powf(rowsum[(size_t)b * N + i], -0.5f), dj = powf(rowsum[(size_t)b * N + j], -0.5f);
      const float an = (di * Ab[(size_t)i * N + j]) * dj;
      const float id = (i == j) ? 1.f : 0.f;
      v = (mode == 0) ? id + an : (1.0f * (id - an)) - id;
    } else if (mode == 2) {
      const float s = rowsum[(size_t)b * N + j];
      const float dinv = 1.f / s;
      v = (isinf(dinv) ? 0.f : dinv) * Ab[(size_t)j * N + i];
    } else {
      const float s = colsum[(size_t)b * N + j];
      const float dinv = 1.f / s;
      v = (isinf(dinv) ? 0.f : dinv) * Ab[(size_t)i * N + j];
    }
    float* Sb = sup + (size_t)b * Ks * N * N;
    Sb[(size_t)k_out * N * N + (size_t)i * N + j] = v;
    if (write_identity) Sb[(size_t)i * N + j] = (i == j) ? 1.f : 0.f;
  }
}

static unsigned adj_grid(size_t work, int threads) {
  size_t b = (work + threads - 1) / threads;
  const size_t cap = (size_t)device_sm_count() * 16;
  return (unsigned)(b < cap ? (b < 1 ? 1 : b) : cap);
}

// T_k = 2 * x * T_{k-1} - T_{k-2} for every batch element; x = support k_x, T's are supports of the same stack
static int cheb_step(float* sup, int B, int N, int Ks, int k_x, int k_prev, int k_prev2, int k_out, cudaStream_t st) {
  const long long NN = (long long)N * N;
  SgemmParams p{};
  p.A = sup + k_x * NN; p.B = sup + k_prev * NN; p.D = sup + k_out * NN; p.Cin = sup + k_prev2 * NN;
  p.M = N; p.N = N; p.K = N;
  p.a_si = N; p.a_sk = 1; p.b_sk = N; p.b_sj = 1; p.d_si = N;
  p.nseg = 1; p.Z0 = B; p.Z1 = 1; p.Z2 = 1;
  for (int i = 0; i < 3; ++i) { p.a_sz[i] = 0; p.b_sz[i] = 0; p.d_sz[i] = 0; p.c_sz[i] = 0; }
  p.a_sz[0] = p.b_sz[0] = p.d_sz[0] = p.c_sz[0] = (long long)Ks * NN;
  p.ksplit = 1; p.alpha = 2.f; p.beta = -1.f;
  return simt_sgemm(p, st);
}

int adj_process(const float* flow, float* supports, int B, int N, int kernel_type, int K, void* ws, size_t ws_bytes, cudaStream_t st) {
  const int Ks = adj_num_supports(kernel_type, K);
  MPGCN_CHECK(Ks >= 1, "Invalid kernel_type. Must be one of [chebyshev, localpool, random_walk_diffusion, dual_random_walk_diffusion].");
  MPGCN_CHECK(B >= 1 && N >= 1 && K >= 0, "adj_process: bad shape B=%d N=%d K=%d", B, N, K);
  const AdjLayout L = adj_layout(B, N);
  MPGCN_CHECK(ws != nullptr && ws_bytes >= L.total, "adj_process: workspace too small (%zu < %zu bytes)", ws_bytes, L.total);
  float* rowsum = reinterpret_cast<float*>(static_cast<uint8_t*>(ws) + L.rowsum);
  float* colsum = reinterpret_cast<float*>(static_cast<uint8_t*>(ws) + L.colsum);
  const size_t warps = (size_t)B * N;
  prof_count(PROF_ELEMENTWISE);
  adj_sums_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(flow, rowsum, B, N, 0);
  if (kernel_type == ADJ_DUAL_RANDOM_WALK) {
    prof_count(PROF_ELEMENTWISE);
    adj_sums_kernel<<<(unsigned)((warps * 32 + 255) / 256), 256, 0, st>>>(flow, colsum, B, N, 1);
  }
  const size_t total = (size_t)B * N * N;
  prof_count(PROF_ELEMENTWISE);
  if (kernel_type == ADJ_LOCALPOOL) {
    adj_build_kernel<<<adj_grid(total, 256), 256, 0, st>>>(flow, rowsum, colsum, supports, B, N, Ks, 0, 0, 0);
    MPGCN_CUDA(cudaGetLastError());
    return 0;
  }
  if (K == 0) {      // only T_0 = I: write x into a scratch-free way by building the identity alone
    adj_build_kernel<<<adj_grid(total, 256), 256, 0, st>>>(flow, rowsum, colsum, supports, B, N, Ks, 0, 2, 1);
    MPGCN_CUDA(cudaGetLastError());   // support 0 first receives x, then the identity (same thread, program order)
    return 0;
  }
  const int mode = (kernel_type == ADJ_CHEBYSHEV) ? 1 : 2;
  adj_build_kernel<<<adj_grid(total, 256), 256, 0, st>>>(flow, rowsum, colsum, supports, B, N, Ks, 1, mode, 1);   // T_0 = I, T_1 = x
  MPGCN_CUDA(cudaGetLastError());
  for (int k = 2; k <= K; ++k)
    if (int e = cheb_step(supports, B, N, Ks, 1, k - 1, k - 2, k, st)) return e;
  if (kernel_type == ADJ_DUAL_RANDOM_WALK) {     // backward series occupies supports K+1 .. 2K; its T_0 is the shared identity
    prof_count(PROF_ELEMENTWISE);
    adj_build_kernel<<<adj_grid(total, 256), 256, 0, st>>>(flow, rowsum, colsum, supports, B, N, Ks, K + 1, 3, 0);
    MPGCN_CUDA(cudaGetLastError());
    for (int k = 2; k <= K; ++k)
      if (int e = cheb_step(supports, B, N, Ks, K + 1, K + k - 1, k == 2 ? 0 : K + k - 2, K + k, st)) return e;
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------------
// Backward: d_flow from d_supports (the adjoint of adj_process, per batch element A = flow[b], G_k = dL/dT_k).
//
//   series adjoint, k = K .. 2:   gx += 2 G_k T_{k-1}^T,   G_{k-1} += 2 x^T G_k,   G_{k-2} -= G_k;   then gx += G_1
//     (gx is accumulated in G_1's plane, which no step reads as an operand; G_0 belongs to the identity and is discarded)
//   random walk   x_ij = A_ji dinv_j:   dA_ji += gx_ij dinv_j,   dA_j. += -dinv_j^2 sum_i gx_ij A_ji
//   dual, backward series x_ij = A_ij cinv_j:   dA_ij += gx_ij cinv_j,   dA_.j += -cinv_j^2 sum_i gx_ij A_ij
//   symmetric     An = D A D, d = r^-1/2, gAn = -gx (chebyshev) or d_supports[0] (localpool):
//                 dA_ij = d_i d_j gAn_ij + gr_i,   gr_i = -1/2 r_i^-3/2 (sum_j gAn_ij A_ij d_j + sum_j gAn_ji d_j A_ji)
// dinv / cinv are masked to 0 exactly where the forward masked them (isinf(1/s)), so such a row or column contributes exactly 0.
//
// Workspace: [B][Ks][N][N] working copy of d_supports (only when K >= 2), then row sums, column sums and two per-row reductions.
// ---------------------------------------------------------------------------------------------------------------------------
struct AdjBwdLayout { size_t grads, rowsum, colsum, red0, red1, total; };
static AdjBwdLayout adj_bwd_layout(int B, int N, int kernel_type, int K) {
  AdjBwdLayout L;
  size_t off = 0;
  const size_t vec = (size_t)B * N * sizeof(float);
  L.grads = take(off, kernel_type == ADJ_LOCALPOOL || K < 2 ? 0 : (size_t)B * adj_num_supports(kernel_type, K) * N * N * sizeof(float), 256);
  L.rowsum = take(off, vec, 256);
  L.colsum = take(off, vec, 256);
  L.red0 = take(off, vec, 256);
  L.red1 = take(off, vec, 256);
  L.total = align_up(off, 256) + 256;    // unused padding: the size this workspace has always had
  return L;
}

size_t adj_backward_workspace_bytes(int B, int N, int kernel_type, int K) { return adj_bwd_layout(B, N, kernel_type, K).total; }

__device__ __forceinline__ float masked_inv(float s) {
  const float v = 1.f / s;
  return isinf(v) ? 0.f : v;
}

// out[b][i] (+)= sum_j P(i,j) Q(i,j) w(j), P(i,j) = P[b*pz + i*pi + j*pj] (Q likewise), w(j) = rowsum[b][j]^-1/2 (sym_w) or 1;
// one warp per (b, i)
__global__ void adj_wsum_kernel(const float* __restrict__ P, long long pz, long long pi, long long pj, const float* __restrict__ Q,
                                long long qz, long long qi, long long qj, const float* __restrict__ rowsum, int sym_w,
                                float* __restrict__ out, int accumulate, int B, int N) {
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= (long long)B * N) return;
  const int b = (int)(w / N), i = (int)(w % N);
  const float* Pb = P + b * pz + i * pi;
  const float* Qb = Q + b * qz + i * qi;
  float s = 0.f;
  for (int j = lane; j < N; j += 32) {
    float v = Pb[j * pj] * Qb[j * qj];
    if (sym_w) v *= powf(rowsum[(size_t)b * N + j], -0.5f);
    s += v;
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) out[w] = accumulate ? out[w] + s : s;
}

// d_flow[b][a][c] for one kernel type (every element written).  gx: G_1 plane of the forward series, gy: of the backward series
// (dual only), both with batch stride gz; red0 / red1: the per-row reductions of adj_wsum_kernel.
//   mode 0 / 1 (localpool / chebyshev, sg = +1 / -1):  sg (d_a d_c gx[a][c] - 1/2 r_a^-3/2 red0[a])
//   mode 2 / 3 (random walk / dual):  gx[c][a] dinv_a - dinv_a^2 red0[a]   (+ gy[a][c] cinv_c - cinv_c^2 red1[c])
__global__ void adj_norm_grad_kernel(const float* __restrict__ A, const float* __restrict__ gx, const float* __restrict__ gy, long long gz,
                                     const float* __restrict__ rowsum, const float* __restrict__ colsum, const float* __restrict__ red0,
                                     const float* __restrict__ red1, float* __restrict__ dA, int B, int N, int mode) {
  const size_t total = (size_t)B * N * N;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
    const int c = (int)(t % N);
    const int a = (int)((t / N) % N);
    const int b = (int)(t / ((size_t)N * N));
    const float* gxb = gx + b * gz;
    const size_t ra = (size_t)b * N + a, rc = (size_t)b * N + c;
    float v;
    if (mode <= 1) {
      const float r = rowsum[ra];
      const float gan = gxb[(size_t)a * N + c];
      v = powf(r, -0.5f) * powf(rowsum[rc], -0.5f) * gan - 0.5f * powf(r, -1.5f) * red0[ra];
      if (mode == 1) v = -v;
    } else {
      const float di = masked_inv(rowsum[ra]);
      v = gxb[(size_t)c * N + a] * di - di * di * red0[ra];
      if (mode == 3) {
        const float ci = masked_inv(colsum[rc]);
        v += gy[b * gz + (size_t)a * N + c] * ci - ci * ci * red1[rc];
      }
    }
    dA[t] = v;
  }
}

// G_{k-2} -= G_k for every series (Z1 = nser, series stride sser) and batch element (stride bz)
__global__ void adj_sub_plane_kernel(float* __restrict__ G, long long bz, long long sser, int nser, int dst, int src, int B, long long NN) {
  const size_t total = (size_t)B * nser * NN;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
    const long long e = (long long)(t % NN);
    const int s = (int)((t / NN) % nser);
    const int b = (int)(t / ((size_t)NN * nser));
    float* base = G + b * bz + s * sser;
    base[(long long)dst * NN + e] -= base[(long long)src * NN + e];
  }
}

// D = 2 op(X) op(Y) + D over B batch elements and nser series; planes are indices into [B][Ks][N][N] stacks, the series differ by
// K planes.  tx / ty: take the operand transposed.
static int adj_bwd_gemm(const float* X, int px, int tx, const float* Y, int py, int ty, float* D, int pd, int B, int N, int Ks, int K,
                        int nser, cudaStream_t st) {
  const long long NN = (long long)N * N;
  SgemmParams p{};
  p.A = X + px * NN; p.B = Y + py * NN; p.D = D + pd * NN; p.Cin = p.D;
  p.M = N; p.N = N; p.K = N;
  p.a_si = tx ? 1 : N; p.a_sk = tx ? N : 1;
  p.b_sk = ty ? 1 : N; p.b_sj = ty ? N : 1;
  p.d_si = N;
  p.nseg = 1; p.Z0 = B; p.Z1 = nser; p.Z2 = 1;
  for (int i = 0; i < 3; ++i) { p.a_sz[i] = 0; p.b_sz[i] = 0; p.d_sz[i] = 0; p.c_sz[i] = 0; }
  p.a_sz[0] = p.b_sz[0] = p.d_sz[0] = p.c_sz[0] = (long long)Ks * NN;
  p.a_sz[1] = p.b_sz[1] = p.d_sz[1] = p.c_sz[1] = (long long)K * NN;
  p.ksplit = 1; p.alpha = 2.f; p.beta = 1.f;
  return simt_sgemm(p, st);
}

int adj_process_backward(const float* flow, const float* supports, const float* d_supports, float* d_flow, int B, int N, int kernel_type,
                         int K, void* ws, size_t ws_bytes, cudaStream_t st) {
  MPGCN_CHECK(adj_num_supports(kernel_type, 1) >= 1,
              "Invalid kernel_type. Must be one of [chebyshev, localpool, random_walk_diffusion, dual_random_walk_diffusion].");
  MPGCN_CHECK(B >= 1 && N >= 1 && K >= 0, "adj_process_backward: bad shape B=%d N=%d K=%d", B, N, K);
  const int Ks = adj_num_supports(kernel_type, K);
  const AdjBwdLayout L = adj_bwd_layout(B, N, kernel_type, K);
  MPGCN_CHECK(ws != nullptr && ws_bytes >= L.total, "adj_process_backward: workspace too small (%zu < %zu bytes)", ws_bytes, L.total);
  const size_t total = (size_t)B * N * N;
  if (kernel_type != ADJ_LOCALPOOL && K == 0) {       // only the identity: its gradient is not the flow's
    MPGCN_CUDA(cudaMemsetAsync(d_flow, 0, total * sizeof(float), st));
    return 0;
  }
  const long long NN = (long long)N * N;
  uint8_t* w8 = static_cast<uint8_t*>(ws);
  float* grads = reinterpret_cast<float*>(w8 + L.grads);
  float* rowsum = reinterpret_cast<float*>(w8 + L.rowsum);
  float* colsum = reinterpret_cast<float*>(w8 + L.colsum);
  float* red0 = reinterpret_cast<float*>(w8 + L.red0);
  float* red1 = reinterpret_cast<float*>(w8 + L.red1);
  const unsigned warp_blocks = (unsigned)(((size_t)B * N * 32 + 255) / 256);
  const bool dual = kernel_type == ADJ_DUAL_RANDOM_WALK;

  prof_count(PROF_ELEMENTWISE);
  adj_sums_kernel<<<warp_blocks, 256, 0, st>>>(flow, rowsum, B, N, 0);
  if (dual) {
    prof_count(PROF_ELEMENTWISE);
    adj_sums_kernel<<<warp_blocks, 256, 0, st>>>(flow, colsum, B, N, 1);
  }

  // gx of each series in plane 1 (forward series) and K + 1 (backward series) of a [B][Ks][N][N] stack
  const float* g = d_supports;
  if (kernel_type != ADJ_LOCALPOOL && K >= 2) {
    MPGCN_CUDA(cudaMemcpyAsync(grads, d_supports, (size_t)B * Ks * NN * sizeof(float), cudaMemcpyDeviceToDevice, st));
    const int nser = dual ? 2 : 1;
    for (int k = K; k >= 2; --k) {
      // gx += 2 G_k T_{k-1}^T;  G_{k-1} += 2 x^T G_k  (x = T_1);  G_{k-2} -= G_k
      if (int e = adj_bwd_gemm(grads, k, 0, supports, k - 1, 1, grads, 1, B, N, Ks, K, nser, st)) return e;
      if (int e = adj_bwd_gemm(supports, 1, 1, grads, k, 0, grads, k - 1, B, N, Ks, K, nser, st)) return e;
      if (k - 2 >= 1) {
        prof_count(PROF_ELEMENTWISE);
        adj_sub_plane_kernel<<<adj_grid((size_t)B * nser * NN, 256), 256, 0, st>>>(grads, (long long)Ks * NN, (long long)K * NN, nser,
                                                                                    k - 2, k, B, NN);
        MPGCN_CUDA(cudaGetLastError());
      }
    }
    g = grads;
  }
  const long long gz = (long long)Ks * NN;
  const float* gx = kernel_type == ADJ_LOCALPOOL ? g : g + NN;
  const float* gy = dual ? g + (long long)(K + 1) * NN : nullptr;

  // per-row reductions
  if (kernel_type <= ADJ_CHEBYSHEV) {           // red0[i] = sum_j g_ij A_ij d_j + sum_j g_ji A_ji d_j
    prof_count(PROF_ELEMENTWISE);
    adj_wsum_kernel<<<warp_blocks, 256, 0, st>>>(gx, gz, N, 1, flow, NN, N, 1, rowsum, 1, red0, 0, B, N);
    prof_count(PROF_ELEMENTWISE);
    adj_wsum_kernel<<<warp_blocks, 256, 0, st>>>(gx, gz, 1, N, flow, NN, 1, N, rowsum, 1, red0, 1, B, N);
  } else {                                      // red0[j] = sum_i gx_ij A_ji
    prof_count(PROF_ELEMENTWISE);
    adj_wsum_kernel<<<warp_blocks, 256, 0, st>>>(gx, gz, 1, N, flow, NN, N, 1, rowsum, 0, red0, 0, B, N);
    if (dual) {                                 // red1[j] = sum_i gy_ij A_ij
      prof_count(PROF_ELEMENTWISE);
      adj_wsum_kernel<<<warp_blocks, 256, 0, st>>>(gy, gz, 1, N, flow, NN, 1, N, rowsum, 0, red1, 0, B, N);
    }
  }
  prof_count(PROF_ELEMENTWISE);
  adj_norm_grad_kernel<<<adj_grid(total, 256), 256, 0, st>>>(flow, gx, gy, gz, rowsum, colsum, red0, red1, d_flow, B, N, kernel_type);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace mpgcn
