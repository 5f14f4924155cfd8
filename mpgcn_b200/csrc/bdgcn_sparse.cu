// Sparse static supports for the exact fp32 layer (precision 0): the four N^3 stages of bdgcn_simt.cu as gathers over the
// stored nonzeros of G (DESIGN.md section 12).
//
//   structure  one device buffer per [K,N,N] stack: CSR and CSC (the CSR of G^T) of every support, int32 indices, row pointers
//              as offsets into the stack's nonzero arrays ([K][N + 1]), built from COO by a counting sort on the device.
//   stages     out_slab[i, :] = sum_support sum_{j in nz(A_i)} a_ij in_slab[j, :] over [N, ch] slabs:
//                FWD_A  Z_d  = X x_2 G_d             CSC, one output per support, slabs X[b,n] (contiguous)
//                FWD_B  out  = act(sum_o G_o^T x_1 U_o + bias)  CSC, summed over supports, slabs U[b,o,:,e,:] (rows N*H apart)
//                BWD_V  V_o  = G_o x_1 dPre          CSR, one output per support, slabs dPre[b,:,e,:]
//                BWD_DX dX   = sum_d Y_d x_2 G_d^T   CSR, summed over supports, slabs Y[b,d,n]
// Every output element is one thread's sum in a fixed order (support, then nonzero order within the row), so the results do
// not depend on the launch or on the deterministic mode, and no floating-point atomic is involved.
#include "kernels.h"

#include <algorithm>

namespace mpgcn {

// ---------------------------------------------------------------------------------------------------------------------------
// structure
// ---------------------------------------------------------------------------------------------------------------------------
// CSR then CSC (pointers, indices, values), then the build's scratch: per-segment counters (CSR, CSC) and one (key, entry) pair
// per nonzero, reused by both formats.
struct SparseLayout { size_t csr_ptr, csr_idx, csr_val, csc_ptr, csc_idx, csc_val, cnt, key, orig, total; };
static SparseLayout sparse_layout(int K, int N, long long nnz) {
  SparseLayout L;
  size_t off = 0;
  const size_t P = (size_t)K * (N + 1) * 4, Z = (size_t)nnz * 4;
  L.csr_ptr = take(off, P, 256); L.csr_idx = take(off, Z, 256); L.csr_val = take(off, Z, 256);
  L.csc_ptr = take(off, P, 256); L.csc_idx = take(off, Z, 256); L.csc_val = take(off, Z, 256);
  L.cnt = take(off, (size_t)2 * K * N * 4, 256);
  L.key = take(off, Z, 256); L.orig = take(off, Z, 256);
  L.total = align_up(off, 256);
  return L;
}

bool sparse_shape_ok(int K, int N, long long nnz) {
  return K >= 1 && N >= 1 && nnz >= 0 && nnz < (1ll << 31) && (long long)K * (N + 1) < (1ll << 31);
}

size_t sparse_supports_bytes(int K, int N, long long nnz) { return sparse_shape_ok(K, N, nnz) ? sparse_layout(K, N, nnz).total : 0; }

SparseSupports sparse_supports_view(const void* buf, int K, int N, long long nnz) {
  const SparseLayout L = sparse_layout(K, N, nnz);
  const uint8_t* b = static_cast<const uint8_t*>(buf);
  SparseSupports sp;
  sp.K = K; sp.N = N; sp.nnz = nnz;
  sp.csr_ptr = reinterpret_cast<const int*>(b + L.csr_ptr); sp.csr_idx = reinterpret_cast<const int*>(b + L.csr_idx);
  sp.csr_val = reinterpret_cast<const float*>(b + L.csr_val);
  sp.csc_ptr = reinterpret_cast<const int*>(b + L.csc_ptr); sp.csc_idx = reinterpret_cast<const int*>(b + L.csc_idx);
  sp.csc_val = reinterpret_cast<const float*>(b + L.csc_val);
  return sp;
}

static __device__ __forceinline__ bool coo_entry(const long long* ix, long long nnz, long long e, int K, int N, int& k, int& r, int& c) {
  const long long kk = ix[e], rr = ix[nnz + e], cc = ix[2 * nnz + e];
  if (kk < 0 || kk >= K || rr < 0 || rr >= N || cc < 0 || cc >= N) return false;     // outside the stack: ignored
  k = (int)kk; r = (int)rr; c = (int)cc;
  return true;
}

// Integer counters only: the order in which threads take them decides no floating-point sum (sp_place_kernel fixes every
// position from the entries themselves).
__global__ void sp_count_kernel(const long long* __restrict__ ix, long long nnz, int K, int N, unsigned* cnt_r, unsigned* cnt_c) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < nnz; e += (long long)gridDim.x * blockDim.x) {
    int k, r, c;
    if (!coo_entry(ix, nnz, e, K, N, k, r, c)) continue;
    atomicInc(&cnt_r[(long long)k * N + r], 0xFFFFFFFFu);
    atomicInc(&cnt_c[(long long)k * N + c], 0xFFFFFFFFu);
  }
}

// exclusive scan of the K*N segment counts (one block): ptr[k][seg] = start of the segment, ptr[k][N] = end of support k; the
// counts become the segments' placement cursors
__global__ void __launch_bounds__(1024) sp_scan_kernel(unsigned* cnt, int* ptr, int K, int N) {
  __shared__ unsigned warp_sum[32];
  const long long n = (long long)K * N;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned carry = 0;
  for (long long base = 0; base < n; base += 1024) {
    const long long i = base + threadIdx.x;
    const unsigned v = i < n ? cnt[i] : 0u;
    unsigned x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned y = __shfl_up_sync(0xFFFFFFFFu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_sum[warp] = x;
    __syncthreads();
    if (warp == 0) {
      unsigned w = warp_sum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(0xFFFFFFFFu, w, o);
        if (lane >= o) w += y;
      }
      warp_sum[lane] = w;
    }
    __syncthreads();
    const unsigned excl = carry + (warp ? warp_sum[warp - 1] : 0u) + x - v;
    if (i < n) {
      ptr[(i / N) * (N + 1) + i % N] = (int)excl;
      cnt[i] = excl;
    }
    carry += warp_sum[31];
    __syncthreads();
  }
  for (int k = threadIdx.x; k < K; k += blockDim.x) ptr[(long long)k * (N + 1) + N] = k + 1 < K ? ptr[(long long)(k + 1) * (N + 1)] : (int)carry;
}

// every entry into its segment (row for CSR, column for CSC) at a cursor: (key = the other index, entry number)
__global__ void sp_scatter_kernel(const long long* __restrict__ ix, long long nnz, int K, int N, int by_col, unsigned* cursor, int* key,
                                  int* orig) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < nnz; e += (long long)gridDim.x * blockDim.x) {
    int k, r, c;
    if (!coo_entry(ix, nnz, e, K, N, k, r, c)) continue;
    const unsigned pos = atomicInc(&cursor[(long long)k * N + (by_col ? c : r)], 0xFFFFFFFFu);
    key[pos] = by_col ? r : c;
    orig[pos] = (int)e;
  }
}

// final position = segment start + rank of (key, entry number) within the segment: ascending index, duplicates in COO order
__global__ void sp_place_kernel(const long long* __restrict__ ix, const float* __restrict__ values, long long nnz, int K, int N, int by_col,
                                const int* __restrict__ ptr, const int* __restrict__ key, const int* __restrict__ orig, int* idx_out,
                                float* val_out) {
  const long long total = ptr[(long long)K * (N + 1) - 1];
  for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
    const int e = orig[p], kp = key[p];
    const long long seg = ix[e] * (N + 1) + (by_col ? ix[2 * nnz + e] : ix[nnz + e]);
    const int lo = ptr[seg], hi = ptr[seg + 1];
    int rank = 0;
    for (int q = lo; q < hi; ++q) {
      const int kq = key[q];
      rank += (kq < kp || (kq == kp && orig[q] < e)) ? 1 : 0;
    }
    idx_out[lo + rank] = kp;
    val_out[lo + rank] = values[e];
  }
}

static unsigned grid_1d(long long items, int threads) {
  long long b = (items + threads - 1) / threads;
  const long long cap = (long long)device_sm_count() * 8;
  return (unsigned)(b < 1 ? 1 : b > cap ? cap : b);
}

int sparse_supports_build(const long long* indices, const float* values, long long nnz, int K, int N, void* buf, cudaStream_t st) {
  const SparseLayout L = sparse_layout(K, N, nnz);
  uint8_t* b = static_cast<uint8_t*>(buf);
  unsigned* cnt_r = reinterpret_cast<unsigned*>(b + L.cnt);
  unsigned* cnt_c = cnt_r + (size_t)K * N;
  int* key = reinterpret_cast<int*>(b + L.key);
  int* orig = reinterpret_cast<int*>(b + L.orig);
  int* csr_ptr = reinterpret_cast<int*>(b + L.csr_ptr);
  int* csc_ptr = reinterpret_cast<int*>(b + L.csc_ptr);
  MPGCN_CUDA(cudaMemsetAsync(cnt_r, 0, (size_t)2 * K * N * 4, st));
  if (nnz > 0) {
    prof_count(PROF_ELEMENTWISE);
    sp_count_kernel<<<grid_1d(nnz, 256), 256, 0, st>>>(indices, nnz, K, N, cnt_r, cnt_c);
    MPGCN_CUDA(cudaGetLastError());
  }
  for (int f = 0; f < 2; ++f) {
    int* ptr = f ? csc_ptr : csr_ptr;
    unsigned* cnt = f ? cnt_c : cnt_r;
    prof_count(PROF_ELEMENTWISE);
    sp_scan_kernel<<<1, 1024, 0, st>>>(cnt, ptr, K, N);
    MPGCN_CUDA(cudaGetLastError());
    if (nnz == 0) continue;
    prof_count(PROF_ELEMENTWISE);
    sp_scatter_kernel<<<grid_1d(nnz, 256), 256, 0, st>>>(indices, nnz, K, N, f, cnt, key, orig);
    MPGCN_CUDA(cudaGetLastError());
    prof_count(PROF_ELEMENTWISE);
    sp_place_kernel<<<grid_1d(nnz, 256), 256, 0, st>>>(indices, values, nnz, K, N, f, ptr, key, orig,
                                                        reinterpret_cast<int*>(b + (f ? L.csc_idx : L.csr_idx)),
                                                        reinterpret_cast<float*>(b + (f ? L.csc_val : L.csr_val)));
    MPGCN_CUDA(cudaGetLastError());
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------------
// gather contraction
// ---------------------------------------------------------------------------------------------------------------------------
// Block (z0, z1, chunk) computes channels [c0, c0 + cw) of one output slab.  in_k = in + z0 in_s0 + z1 in_s1 + k in_sk holds
// rows j at in_row (sum: one input slab per support; otherwise one input slab shared by the K outputs out + k out_sk).
struct GatherArgs {
  const int* ptr;
  const int* idx;
  const float* val;
  const float* in;
  float* out;
  const float* bias;
  long long in_s0, in_s1, in_sk, in_row;
  long long out_s0, out_s1, out_sk, out_row;
  int N, K, ch, Z1, cw, nchunks;
  int sum, staged, relu;
};

constexpr int GATHER_THREADS = 512;
constexpr int GATHER_SMEM = 112 * 1024;       // two blocks per SM

__global__ void __launch_bounds__(GATHER_THREADS) sparse_gather_kernel(const GatherArgs a) {
  extern __shared__ float stage[];
  long long bid = blockIdx.x;
  const int chunk = (int)(bid % a.nchunks);
  bid /= a.nchunks;
  const long long z1 = bid % a.Z1, z0 = bid / a.Z1;
  const int c0 = chunk * a.cw, cw = min(a.cw, a.ch - c0);
  const float* in = a.in + z0 * a.in_s0 + z1 * a.in_s1 + c0;
  const float* src = in;
  long long s_row = a.in_row, s_k = a.in_sk;
  if (a.staged) {     // the slab's channel chunk (every support's, when summed) in shared memory: each input element read once
    const int per = a.N * cw;
    const long long n = (long long)(a.sum ? a.K : 1) * per;
    for (long long t = threadIdx.x; t < n; t += blockDim.x) {
      const int k = (int)(t / per), rem = (int)(t % per), j = rem / cw, c = rem % cw;
      stage[t] = in[k * a.in_sk + j * a.in_row + c];
    }
    __syncthreads();
    src = stage;
    s_row = cw;
    s_k = per;
  }
  float* out = a.out + z0 * a.out_s0 + z1 * a.out_s1 + c0;
  const long long np1 = a.N + 1;
  for (int t = threadIdx.x; t < a.N * cw; t += blockDim.x) {
    const int i = t / cw, c = t % cw;
    if (a.sum) {
      float acc = 0.f;
      for (int k = 0; k < a.K; ++k) {
        const float* sk = src + k * s_k + c;
        const int hi = a.ptr[k * np1 + i + 1];
        for (int p = a.ptr[k * np1 + i]; p < hi; ++p) acc = fmaf(a.val[p], sk[a.idx[p] * s_row], acc);
      }
      if (a.bias) acc += a.bias[c0 + c];
      if (a.relu) acc = fmaxf(acc, 0.f);
      out[i * a.out_row + c] = acc;
    } else {
      for (int k = 0; k < a.K; ++k) {
        float acc = 0.f;
        const int hi = a.ptr[k * np1 + i + 1];
        for (int p = a.ptr[k * np1 + i]; p < hi; ++p) acc = fmaf(a.val[p], src[a.idx[p] * s_row + c], acc);
        out[k * a.out_sk + i * a.out_row + c] = acc;
      }
    }
  }
}

int sparse_stage(SparseStage stage, const BdgcnShape& s, const SparseSupports& sp, const float* in, float* out, const float* bias,
                 cudaStream_t st) {
  MPGCN_CHECK(s.whole() && !s.dynamic && sp.K == s.K && sp.N == s.N, "sparse supports: whole static layers only");
  const long long N = s.N, NN = N * N, K = s.K, C = s.C, H = s.H;
  GatherArgs a{};
  const bool csc = stage == SPARSE_FWD_A || stage == SPARSE_FWD_B;
  a.ptr = csc ? sp.csc_ptr : sp.csr_ptr; a.idx = csc ? sp.csc_idx : sp.csr_idx; a.val = csc ? sp.csc_val : sp.csr_val;
  a.in = in; a.out = out; a.N = s.N; a.K = s.K; a.Z1 = s.N;
  switch (stage) {
    case SPARSE_FWD_A:      // X [B][n][c][l] -> Z [B][d][n][e][l], slab (b, n)
      a.ch = s.C; a.sum = 0;
      a.in_s0 = NN * C; a.in_s1 = N * C; a.in_row = C;
      a.out_s0 = K * NN * C; a.out_s1 = N * C; a.out_sk = NN * C; a.out_row = C;
      break;
    case SPARSE_FWD_B:      // U [B][o][n][e][h] -> out [B][m][e][h], slab (b, e)
      a.ch = s.H; a.sum = 1; a.bias = bias; a.relu = s.act;
      a.in_s0 = K * NN * H; a.in_s1 = H; a.in_sk = NN * H; a.in_row = N * H;
      a.out_s0 = NN * H; a.out_s1 = H; a.out_row = N * H;
      break;
    case SPARSE_BWD_V:      // dPre [B][m][e][h] -> V [B][o][n][e][h], slab (b, e)
      a.ch = s.H; a.sum = 0;
      a.in_s0 = NN * H; a.in_s1 = H; a.in_row = N * H;
      a.out_s0 = K * NN * H; a.out_s1 = H; a.out_sk = NN * H; a.out_row = N * H;
      break;
    case SPARSE_BWD_DX:     // Y [B][d][n][e][l] -> dX [B][n][c][l], slab (b, n)
      a.ch = s.C; a.sum = 1;
      a.in_s0 = K * NN * C; a.in_s1 = N * C; a.in_sk = NN * C; a.in_row = C;
      a.out_s0 = NN * C; a.out_s1 = N * C; a.out_row = C;
      break;
  }
  // channel chunk: as many channels as fit the staging budget; a slab whose single channel does not fit is gathered from global
  // memory (L2) instead, 32 channels at a time
  const long long per_channel = (a.sum ? K : 1) * N * 4;
  a.staged = per_channel <= GATHER_SMEM;
  a.cw = a.staged ? (int)std::min<long long>(a.ch, GATHER_SMEM / per_channel) : std::min(a.ch, 32);
  a.nchunks = (a.ch + a.cw - 1) / a.cw;
  const long long blocks = (long long)s.B * N * a.nchunks;
  MPGCN_CHECK(blocks < (1ll << 31), "sparse supports: grid too large (%lld blocks)", blocks);
  const int smem = a.staged ? (int)(per_channel * a.cw) : 0;
  static DynSmemAttr attr;
  if (int e = ensure_dyn_smem(sparse_gather_kernel, smem, attr)) return e;
  const long long work = (long long)N * a.cw;
  const int threads = work >= GATHER_THREADS ? GATHER_THREADS : (int)((work + 31) / 32 * 32);
  prof_begin(PROF_SIMT_GEMM, 2.0 * s.B * (double)N * sp.nnz * a.ch, st);
  sparse_gather_kernel<<<(unsigned)blocks, threads, smem, st>>>(a);
  prof_end(st);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace mpgcn
