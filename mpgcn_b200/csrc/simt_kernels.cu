// fp32 CUDA-core path: a strided / batched / segmented SGEMM that evaluates every
// contraction of the BDGCN layer exactly in fp32 (precision mode 0), plus the elementwise
// and layout kernels shared with the tensor-core path.
//
// This is the exact-arithmetic mode of the product (used for shapes the tensor-core engine
// does not cover -- channel counts other than 32 -- and as the on-device cross-check of
// the fp16 tensor path).  It is NOT a CPU fallback: everything here runs on the GPU.
#include "kernels.h"

#include <algorithm>
#include <type_traits>

namespace mpgcn {

// ---------------------------------------------------------------------------------------
// SGEMM: 64 x BN output tile, 16-deep k slab, 256 threads, 4 x (BN/16) micro-tile
// ---------------------------------------------------------------------------------------
template <int BN>
__global__ void __launch_bounds__(256) sgemm_kernel(const SgemmParams p, int tiles_m, int tiles_n) {
  constexpr int BM = 64, BKS = 16, TN = BN / 16;
  __shared__ float As[BKS][BM + 4];
  __shared__ float Bs[BKS][BN + 4];

  long long bid = blockIdx.x;
  const int tn = (int)(bid % tiles_n); bid /= tiles_n;
  const int tm = (int)(bid % tiles_m); bid /= tiles_m;
  const int slice = (int)(bid % p.ksplit); bid /= p.ksplit;
  const int z2 = (int)(bid % p.Z2); bid /= p.Z2;
  const int z1 = (int)(bid % p.Z1); bid /= p.Z1;
  const int z0 = (int)bid;

  const float* A = p.A + z0 * p.a_sz[0] + z1 * p.a_sz[1] + z2 * p.a_sz[2];
  const float* B = p.B + z0 * p.b_sz[0] + z1 * p.b_sz[1] + z2 * p.b_sz[2];
  float* D = p.D + z0 * p.d_sz[0] + z1 * p.d_sz[1] + z2 * p.d_sz[2] + slice * p.d_sslice;
  const float* Cin = p.Cin ? p.Cin + z0 * p.c_sz[0] + z1 * p.c_sz[1] + z2 * p.c_sz[2] : nullptr;

  const int tid = threadIdx.x;
  const int ty = tid / 16, tx = tid % 16;
  const int i0 = tm * BM, j0 = tn * BN;

  float acc[4][TN];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < TN; ++b) acc[a][b] = 0.f;

  const int k_per_slice = (p.K + p.ksplit - 1) / p.ksplit;
  const int k_lo = slice * k_per_slice;
  const int k_hi = min(p.K, k_lo + k_per_slice);
  const bool a_i_fast = (p.a_si == 1);
  const bool b_j_fast = (p.b_sj == 1);

  for (int seg = 0; seg < p.nseg; ++seg) {
    const float* As_g = A + seg * p.a_sseg;
    const float* Bs_g = B + seg * p.b_sseg;
    for (int k0 = k_lo; k0 < k_hi; k0 += BKS) {
#pragma unroll
      for (int q = 0; q < (BM * BKS) / 256; ++q) {
        const int idx = tid + q * 256;
        const int ii = a_i_fast ? idx % BM : idx / BKS;
        const int kk = a_i_fast ? idx / BM : idx % BKS;
        const int gi = i0 + ii, gk = k0 + kk;
        As[kk][ii] = (gi < p.M && gk < k_hi) ? As_g[gi * p.a_si + gk * p.a_sk] : 0.f;
      }
#pragma unroll
      for (int q = 0; q < (BN * BKS) / 256; ++q) {
        const int idx = tid + q * 256;
        const int jj = b_j_fast ? idx % BN : idx / BKS;
        const int kk = b_j_fast ? idx / BN : idx % BKS;
        const int gj = j0 + jj, gk = k0 + kk;
        Bs[kk][jj] = (gj < p.N && gk < k_hi) ? Bs_g[gk * p.b_sk + gj * p.b_sj] : 0.f;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < BKS; ++kk) {
        float a[4], b[TN];
#pragma unroll
        for (int x = 0; x < 4; ++x) a[x] = As[kk][ty * 4 + x];
#pragma unroll
        for (int y = 0; y < TN; ++y) b[y] = Bs[kk][tx * TN + y];
#pragma unroll
        for (int x = 0; x < 4; ++x)
#pragma unroll
          for (int y = 0; y < TN; ++y) acc[x][y] = fmaf(a[x], b[y], acc[x][y]);
      }
      __syncthreads();
    }
  }

#pragma unroll
  for (int x = 0; x < 4; ++x) {
    const int gi = i0 + ty * 4 + x;
    if (gi >= p.M) continue;
#pragma unroll
    for (int y = 0; y < TN; ++y) {
      const int gj = j0 + tx * TN + y;
      if (gj >= p.N) continue;
      float v = acc[x][y] * p.alpha;
      float* dst = D + gi * p.d_si + gj;
      if (p.ksplit > 1 && p.d_sslice == 0) {
        atomicAdd(dst, v);
      } else {
        if (Cin) v = fmaf(p.beta, Cin[gi * p.d_si + gj], v);
        if (p.bias) v += p.bias[gj % p.bias_mod];
        if (p.relu) v = fmaxf(v, 0.f);
        *dst = v;
      }
    }
  }
}

int simt_sgemm(const SgemmParams& p, cudaStream_t stream) {
  MPGCN_CHECK(p.M > 0 && p.N > 0 && p.K > 0 && p.nseg > 0 && p.ksplit > 0, "simt_sgemm: empty problem");
  MPGCN_CHECK(p.Cin == nullptr || p.ksplit == 1, "simt_sgemm: Cin needs ksplit == 1");
  MPGCN_CHECK(p.d_sslice == 0 || (p.bias == nullptr && !p.relu), "simt_sgemm: slice partials take no epilogue");
  const int bn = (p.N <= 32) ? 32 : 64;
  const int tiles_m = (p.M + 63) / 64;
  const int tiles_n = (p.N + bn - 1) / bn;
  const long long blocks = (long long)tiles_m * tiles_n * p.ksplit * p.Z0 * p.Z1 * p.Z2;
  MPGCN_CHECK(blocks > 0 && blocks < (1ll << 31), "simt_sgemm: grid too large (%lld blocks)", blocks);
  prof_count(PROF_SIMT_GEMM);
  if (bn == 32)
    sgemm_kernel<32><<<(unsigned)blocks, 256, 0, stream>>>(p, tiles_m, tiles_n);
  else
    sgemm_kernel<64><<<(unsigned)blocks, 256, 0, stream>>>(p, tiles_m, tiles_n);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------
// elementwise / layout kernels
// ---------------------------------------------------------------------------------------
__global__ void cvt_f16_kernel(const float* __restrict__ src, __half* __restrict__ dst, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const size_t n4 = n / 4;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = reinterpret_cast<const float4*>(src)[i];
    __half2 a = __halves2half2(f2h_sat(v.x), f2h_sat(v.y));
    __half2 b = __halves2half2(f2h_sat(v.z), f2h_sat(v.w));
    uint2 pk;
    pk.x = *reinterpret_cast<uint32_t*>(&a);
    pk.y = *reinterpret_cast<uint32_t*>(&b);
    reinterpret_cast<uint2*>(dst)[i] = pk;
  }
  for (size_t i = n4 * 4 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) dst[i] = f2h_sat(src[i]);
}

static inline unsigned grid_for(size_t work_items, int threads) {
  size_t b = (work_items + threads - 1) / threads;
  const size_t cap = (size_t)device_sm_count() * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (unsigned)b;
}

int cvt_f32_to_f16(const float* src, __half* dst, size_t n, cudaStream_t s) {
  if (n == 0) return 0;
  MPGCN_CHECK((reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 7) == 0, "cvt: misaligned pointers");
  prof_count(PROF_ELEMENTWISE);
  cvt_f16_kernel<<<grid_for(n / 4 + 1, 256), 256, 0, s>>>(src, dst, n);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

// delta[p][i] = G_p[i,i] - fp16(G_p[i,i]) where the diagonal entry DOMINATES its column (G_ii^2 > kDiagTau * sum_{c != i} G_ci^2),
// else 0.  The contraction epilogues add delta * (the diagonal operand row) back, which removes the one rounding error that
// matters when a support is close to the identity (Chebyshev / random-walk T_k of a sparse graph); for a dense support the
// diagonal is one of N comparable terms, the remainder is noise-level, and a zero delta lets the epilogue skip the re-read
// of the operand tensor altogether.
constexpr float kDiagTau = 0.0625f;
__global__ void diag_delta_kernel(const float* __restrict__ G, float* __restrict__ delta, size_t planes, int N) {
  // block = 32 columns x 32 row groups of one plane; blockIdx.x enumerates (plane, column block)
  __shared__ float s_sq[32][33];
  const int cblocks = (N + 31) / 32;
  const size_t p = blockIdx.x / cblocks;
  const int i = (int)(blockIdx.x % cblocks) * 32 + (threadIdx.x & 31);
  const int rg = threadIdx.x >> 5;
  const float* plane = G + p * (size_t)N * N;
  float sq = 0.f;
  if (i < N)
    for (int c = rg; c < N; c += 32) { const float v = plane[(size_t)c * N + i]; sq = fmaf(v, v, sq); }   // 128-byte rows per warp
  s_sq[rg][threadIdx.x & 31] = sq;
  __syncthreads();
  if (rg == 0 && i < N) {
    float col = 0.f;
#pragma unroll
    for (int r = 0; r < 32; ++r) col += s_sq[r][threadIdx.x];
    const float g = plane[(size_t)i * N + i];
    float d = g - __half2float(f2h_sat(g));
    if (!(g * g > kDiagTau * (col - g * g))) d = 0.f;
    delta[p * N + i] = d;
  }
}
int support_diag_delta(const float* G, float* delta, size_t planes, int N, cudaStream_t s) {
  prof_count(PROF_ELEMENTWISE);
  const size_t blocks = planes * (size_t)((N + 31) / 32);
  MPGCN_CHECK(blocks < (1ull << 31), "support_diag_delta: too many planes");
  diag_delta_kernel<<<(unsigned)blocks, 1024, 0, s>>>(G, delta, planes, N);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

__global__ void cvt_f16_padded_kernel(const float* __restrict__ src, __half* __restrict__ dst, size_t rows, int cols, int ld) {
  const size_t total = rows * (size_t)ld;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const size_t r = i / ld;
    const int c = (int)(i - r * ld);
    dst[i] = (c < cols) ? f2h_sat(src[r * cols + c]) : __float2half_rn(0.f);
  }
}

int cvt_f32_to_f16_padded(const float* src, __half* dst, size_t rows, int cols, int ld, cudaStream_t s) {
  if (rows == 0) return 0;
  prof_count(PROF_ELEMENTWISE);
  cvt_f16_padded_kernel<<<grid_for(rows * ld, 256), 256, 0, s>>>(src, dst, rows, cols, ld);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

// ---- bf16x3 operand pairs: hi = bf16_rn(x) at dst[i], lo = bf16_rn(x - hi) at dst[total + i] ----
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}

// [rows][cols] fp32 -> [rows][ld] pair planes (ld >= cols, padding zeroed); ld = cols is a plain conversion
__global__ void cvt_bf16x3_padded_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, size_t rows, int cols, int ld) {
  const size_t total = rows * (size_t)ld;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    __nv_bfloat16 hi = __float2bfloat16_rn(0.f), lo = hi;
    if (ld == cols) {               // unpadded: no index arithmetic
      split_bf16(src[i], hi, lo);
    } else {
      const size_t r = i / ld;
      const int c = (int)(i - r * ld);
      if (c < cols) split_bf16(src[r * cols + c], hi, lo);
    }
    dst[i] = hi;
    dst[total + i] = lo;
  }
}

int cvt_f32_to_bf16x3_padded(const float* src, __nv_bfloat16* dst, size_t rows, int cols, int ld, cudaStream_t s) {
  if (rows == 0) return 0;
  prof_count(PROF_ELEMENTWISE);
  cvt_bf16x3_padded_kernel<<<grid_for(rows * ld, 256), 256, 0, s>>>(src, dst, rows, cols, ld);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

// ---- ReLU backward: d_pre = d_out * [out > 0] (or d_out), stored as fp32 or as fp16(S * d_pre) into g <= 8 destinations, and the
// per-channel bias gradient db[h] = sum d_pre.  The local pass of a layer backward is one sample and one destination; the row
// shard's all-gather (relu_backward_scatter[_f16]) writes rows [row0, row0 + rows) of every rank's [B][N][N][H] buffer.
enum class Mask { None, F32, F16 };   // ReLU mask source: none (linear layer), the fp32 forward output, or its fp16 copy
template <class T>
struct PeerPtrs { T* p[8]; };
template <>
struct PeerPtrs<__nv_bfloat16> { __nv_bfloat16* p[8]; size_t lo_off; };   // bf16x3 pairs: the lo plane lo_off elements behind

// V consecutive values at p <-> V floats in registers; V = 4 is one 16-byte (fp32) or 8-byte (fp16) access
__device__ __forceinline__ void ld_v(const float* p, float (&v)[1]) { v[0] = *p; }
__device__ __forceinline__ void ld_v(const float* p, float (&v)[4]) {
  const float4 t = *reinterpret_cast<const float4*>(p);
  v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
__device__ __forceinline__ void ld_v(const __half* p, float (&v)[1]) { v[0] = __half2float(*p); }
__device__ __forceinline__ void ld_v(const __half* p, float (&v)[4]) {
  const uint2 t = *reinterpret_cast<const uint2*>(p);
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&t.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&t.y));
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}
// read once: streaming loads
__device__ __forceinline__ void ld_cs_v(const float* p, float (&v)[1]) { v[0] = __ldcs(p); }
__device__ __forceinline__ void ld_cs_v(const float* p, float (&v)[4]) {
  const float4 t = __ldcs(reinterpret_cast<const float4*>(p));
  v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
// fp32 stores the value, fp16 stores fp16(S * value) (saturating).  __stwb is the default store; a plain assignment through the
// cast pointer compiles to 4-byte stores here.
__device__ __forceinline__ void st_v(float* p, const float (&v)[1], float) { *p = v[0]; }
__device__ __forceinline__ void st_v(float* p, const float (&v)[4], float) { __stwb(reinterpret_cast<float4*>(p), make_float4(v[0], v[1], v[2], v[3])); }
__device__ __forceinline__ void st_v(__half* p, const float (&v)[1], float S) { *p = f2h_sat(v[0] * S); }
__device__ __forceinline__ void st_v(__half* p, const float (&v)[4], float S) {
  const __half2 a = __halves2half2(f2h_sat(v[0] * S), f2h_sat(v[1] * S)), b = __halves2half2(f2h_sat(v[2] * S), f2h_sat(v[3] * S));
  __stwb(reinterpret_cast<uint2*>(p), make_uint2(*reinterpret_cast<const unsigned int*>(&a), *reinterpret_cast<const unsigned int*>(&b)));
}
// a bf16x3 pair of S * value: hi at p, lo at p + lo_off
__device__ __forceinline__ void st_pair(__nv_bfloat16* p, size_t lo_off, const float (&v)[1], float S) { split_bf16(v[0] * S, p[0], p[lo_off]); }
__device__ __forceinline__ void st_pair(__nv_bfloat16* p, size_t lo_off, const float (&v)[4], float S) {
  uint32_t h0, l0, h1, l1;
  split_bf16x2(v[0] * S, v[1] * S, h0, l0);
  split_bf16x2(v[2] * S, v[3] * S, h1, l1);
  __stwb(reinterpret_cast<uint2*>(p), make_uint2(h0, h1));
  __stwb(reinterpret_cast<uint2*>(p + lo_off), make_uint2(l0, l1));
}

// db[c] += the block's partial sums of channel c.  The block is a multiple of H / V threads with at least H of them, so thread t
// owns channels V * (t % (H / V)) .. + V - 1 for its whole grid-stride loop; thread c < H adds the partials of channel c in thread order.
// With slots (deterministic mode) the block stores that sum in its own [H] slot instead, for reduce_slots to add in block order.
template <int V>
__device__ __forceinline__ void block_bias_grad(const float (&local)[V], float* db, float* slots, int H) {
  extern __shared__ float s_db[];   // [V][blockDim.x]
  const int nt = blockDim.x;
#pragma unroll
  for (int e = 0; e < V; ++e) s_db[e * nt + threadIdx.x] = local[e];
  __syncthreads();
  if ((int)threadIdx.x < H) {
    const int q = threadIdx.x / V, e = threadIdx.x % V;
    float sum = 0.f;
    for (int t = q; t < nt; t += H / V) sum += s_db[e * nt + t];
    if (slots) slots[((size_t)blockIdx.y * gridDim.x + blockIdx.x) * H + threadIdx.x] = sum;
    else atomicAdd(&db[threadIdx.x], sum);
  }
}

// grid.y = sample b: d_out[b * n + i] -> dst[j][b * full + off + i] for i < n; S = scale[0] for an fp16 destination.  At most
// 32 registers, so that 2048 threads fit on an SM: a streaming kernel needs every load in flight it can get.
template <int V, Mask M, class T>
__global__ void __launch_bounds__(1024, 2) relu_bwd_kernel(const float* __restrict__ d_out, const void* __restrict__ mask, PeerPtrs<T> dst, int g, float* __restrict__ db,
                                float* __restrict__ db_slots, const float* __restrict__ scale, size_t n, size_t full, size_t off, int H) {
  using MaskT = std::conditional_t<M == Mask::F16, __half, float>;
  const float S = std::is_same<T, float>::value ? 1.f : __ldg(scale);
  const size_t b = blockIdx.y;
  float local[V] = {};
  for (size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * V; i < n; i += (size_t)gridDim.x * blockDim.x * V) {
    float v[V];
    ld_v(d_out + b * n + i, v);
    if constexpr (M != Mask::None) {
      float o[V];
      ld_v(static_cast<const MaskT*>(mask) + b * n + i, o);
#pragma unroll
      for (int e = 0; e < V; ++e) v[e] = o[e] > 0.f ? v[e] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if constexpr (std::is_same<T, __nv_bfloat16>::value) {
        if (j < g) st_pair(dst.p[j] + b * full + off + i, dst.lo_off, v, S);
      } else {
        if (j < g) st_v(dst.p[j] + b * full + off + i, v, S);
      }
    }
#pragma unroll
    for (int e = 0; e < V; ++e) local[e] += v[e];
  }
  if (db) block_bias_grad<V>(local, db, db_slots, H);
}

static bool aligned(const void* p, size_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

// Block size of the elementwise kernels that keep a thread's channels fixed: a multiple of H / V threads (the grid stride then is
// one too), at least one thread per channel, 256 for every H / V that divides 256.
static int channel_block(int H, int V) {
  const int HV = H / V;
  return HV * std::max(256 / HV, V);
}

// One relu_bwd_kernel launch over B samples of n elements; V = 4 when H, n, full, off are multiples of 4 and every pointer is aligned
// for the vector access, else V = 1.  The exchange steps (PROF_EXCHANGE) are timed, the local pass is counted.
template <Mask M, class T>
static int relu_bwd_launch(const float* d_out, const void* mask, T* const* dsts, int g, float* db, const float* scale, int B, size_t n,
                           size_t full, size_t off, int H, ProfTag tag, cudaStream_t s, float* db_slots = nullptr, size_t lo_off = 0) {
  MPGCN_CHECK(H >= 1 && H <= 1024, "relu backward: H=%d unsupported (1..1024)", H);
  MPGCN_CHECK(g >= 1 && g <= 8, "relu backward: %d ranks unsupported (1..8)", g);
  constexpr bool f16 = !std::is_same<T, float>::value;
  MPGCN_CHECK(!f16 || scale != nullptr, "relu backward: an fp16 destination needs its scale");
  bool vec = H % 4 == 0 && (n | full | off) % 4 == 0 && aligned(d_out, 16) && (M == Mask::None || aligned(mask, M == Mask::F16 ? 8 : 16));
  PeerPtrs<T> pp{};
  if constexpr (std::is_same<T, __nv_bfloat16>::value) {
    pp.lo_off = lo_off;
    vec = vec && lo_off % 4 == 0;
  }
  for (int j = 0; j < g; ++j) {
    MPGCN_CHECK(dsts[j] != nullptr, "relu backward: destination %d is null", j);
    pp.p[j] = dsts[j];
    vec = vec && aligned(dsts[j], 4 * sizeof(T));
  }
  MPGCN_CHECK(!db_slots || B == 1, "relu backward: fixed-order bias gradient of one sample only");
  if (db && !db_slots) MPGCN_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * H, s));
  if (!db) db_slots = nullptr;
  const int V = vec ? 4 : 1, threads = channel_block(H, V);
  const dim3 grid(grid_for(n / V, threads), (unsigned)B);
  const size_t smem = (size_t)V * threads * sizeof(float);
  if (tag == PROF_EXCHANGE) prof_begin(tag, 0.0, s);
  else prof_count(tag);
  if (vec) relu_bwd_kernel<4, M, T><<<grid, threads, smem, s>>>(d_out, mask, pp, g, db, db_slots, scale, n, full, off, H);
  else relu_bwd_kernel<1, M, T><<<grid, threads, smem, s>>>(d_out, mask, pp, g, db, db_slots, scale, n, full, off, H);
  prof_end(s);
  MPGCN_CUDA(cudaGetLastError());
  if (db_slots) return reduce_slots(db_slots, (int)grid.x, H, 1, 0, slot_image(db, H), s);
  return 0;
}
// the same with the ReLU mask taken from the fp32 forward output (act 1) or no mask (act 0)
template <class T>
static int relu_bwd_launch(const float* d_out, const float* out, int act, T* const* dsts, int g, float* db, const float* scale, int B, size_t n,
                           size_t full, size_t off, int H, ProfTag tag, cudaStream_t s, float* db_slots = nullptr, size_t lo_off = 0) {
  return act ? relu_bwd_launch<Mask::F32>(d_out, out, dsts, g, db, scale, B, n, full, off, H, tag, s, db_slots, lo_off)
             : relu_bwd_launch<Mask::None>(d_out, nullptr, dsts, g, db, scale, B, n, full, off, H, tag, s, db_slots, lo_off);
}

int relu_bwd_prep_f16mask(const float* d_out, const __half* out16, int relu, __half* d16, float* db, size_t n, int H, const float* scale,
                          cudaStream_t s, float* db_slots) {
  if (n == 0) return 0;
  if (!relu) return relu_bwd_launch<Mask::None>(d_out, nullptr, &d16, 1, db, scale, 1, n, n, 0, H, PROF_ELEMENTWISE, s, db_slots);
  return relu_bwd_launch<Mask::F16>(d_out, out16, &d16, 1, db, scale, 1, n, n, 0, H, PROF_ELEMENTWISE, s, db_slots);
}

int relu_bwd_prep(const float* d_out, const float* out, int relu, __half* d16, float* d32, float* db, size_t n, int H,
                  const float* scale, cudaStream_t s, float* db_slots) {
  if (n == 0) return 0;
  MPGCN_CHECK((d16 == nullptr) != (d32 == nullptr), "relu_bwd_prep: exactly one of the fp16 and fp32 outputs");
  if (d16) return relu_bwd_launch(d_out, out, relu, &d16, 1, db, scale, 1, n, n, 0, H, PROF_ELEMENTWISE, s, db_slots);
  return relu_bwd_launch(d_out, out, relu, &d32, 1, db, nullptr, 1, n, n, 0, H, PROF_ELEMENTWISE, s, db_slots);
}

int relu_bwd_prep_bf16x3(const float* d_out, const float* out, int relu, __nv_bfloat16* d_pair, float* db, size_t n, int H, const float* scale,
                         cudaStream_t s, float* db_slots) {
  if (n == 0) return 0;
  return relu_bwd_launch(d_out, out, relu, &d_pair, 1, db, scale, 1, n, n, 0, H, PROF_ELEMENTWISE, s, db_slots, n);
}

size_t bias_grad_slot_bytes(int H) { return align_up((size_t)device_sm_count() * 16 * H * sizeof(float), 256); }

// max |x| over a tensor as the bit pattern of a non-negative float (monotone as unsigned int)
__global__ void absmax_kernel(const float* __restrict__ x, size_t n, unsigned int* __restrict__ amax_bits) {
  float m = 0.f;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) m = fmaxf(m, fabsf(x[i]));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(amax_bits, __float_as_uint(m));
}
__global__ void make_scale_kernel(float* scale2, const float* hint) {
  const float amax = hint ? *hint : __uint_as_float(*reinterpret_cast<unsigned int*>(scale2));
  float S = 1.f;
  if (amax > 0.f && amax < 3.0e38f) {
    int e;
    frexpf(amax, &e);            // amax = f * 2^e, f in [0.5, 1)
    int k = 5 - e;               // S * amax in [16, 32)
    k = max(-100, min(100, k));
    S = ldexpf(1.f, k);
  }
  scale2[0] = S;
  scale2[1] = 1.f / S;
}

int grad_scale_prepare(const float* d_out, size_t n, float* scale2, const float* absmax_hint, cudaStream_t s) {
  if (absmax_hint == nullptr) {
    MPGCN_CUDA(cudaMemsetAsync(scale2, 0, 2 * sizeof(float), s));
    prof_count(PROF_ELEMENTWISE);
    absmax_kernel<<<grid_for(n, 256), 256, 0, s>>>(d_out, n, reinterpret_cast<unsigned int*>(scale2));
  }
  prof_count(PROF_ELEMENTWISE);
  make_scale_kernel<<<1, 1, 0, s>>>(scale2, absmax_hint);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

__global__ void permute_w_bwd_kernel(const float* __restrict__ W, float* __restrict__ q32, int Ko, int Kd, int C, int H) {
  const int total = Ko * Kd * C * H;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    // destination index i = ((d*Ko + o)*H + h)*C + l
    const int l = i % C;
    const int h = (i / C) % H;
    const int o = (i / (C * H)) % Ko;
    const int d = i / (C * H * Ko);
    q32[i] = W[((size_t)(o * Kd + d) * C + l) * H + h];
  }
}

int permute_w_bwd(const float* W, float* wq32, int Ko, int Kd, int C, int H, cudaStream_t s) {
  prof_count(PROF_ELEMENTWISE);
  permute_w_bwd_kernel<<<grid_for((size_t)Ko * Kd * C * H, 256), 256, 0, s>>>(W, wq32, Ko, Kd, C, H);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

// W[o][d][32 lc + l][32 hc + h] -> one [32][32] block per (output plane, input plane) of a channel mix, see kernels.h: the W
// element that lands at index i of the forward (fwd) or backward operand
__device__ __forceinline__ float w_mix_src(const float* __restrict__ W, int i, bool fwd, int Ko, int Kd, int C, int H) {
  const int cC = C / 32, cH = H / 32;
  const int e0 = i % 32, e1 = (i / 32) % 32, blk = i / 1024;
  int o, d, lc, hc, l, h;
  if (fwd) {     // forward: i = ((hc*Ko + o)*Kd*cC + d*cC + lc)*1024 + l*32 + h
    h = e0; l = e1;
    const int sp = blk % (Kd * cC), r = blk / (Kd * cC);
    d = sp / cC; lc = sp % cC; o = r % Ko; hc = r / Ko;
  } else {       // backward: i = ((d*cC + lc)*Ko*cH + o*cH + hc)*1024 + h*32 + l
    l = e0; h = e1;
    const int sp = blk % (Ko * cH), r = blk / (Ko * cH);
    o = sp / cH; hc = sp % cH; d = r / cC; lc = r % cC;
  }
  return W[((size_t)(o * Kd + d) * C + lc * 32 + l) * H + hc * 32 + h];
}
__global__ void permute_w_mix_kernel(const float* __restrict__ W, __half* __restrict__ hi, __half* __restrict__ lo, int Ko, int Kd, int C,
                                     int H) {
  const int total = Ko * Kd * C * H;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const float v = w_mix_src(W, i, lo != nullptr, Ko, Kd, C, H);
    const __half x = f2h_sat(v);
    hi[i] = x;
    if (lo) lo[i] = f2h_sat(v - __half2float(x));
  }
}

// bf16x3: the pair of W, hi at pair[i], lo at pair[total + i]
__global__ void permute_w_mix_bf16x3_kernel(const float* __restrict__ W, __nv_bfloat16* __restrict__ pair, int fwd, int Ko, int Kd, int C, int H) {
  const int total = Ko * Kd * C * H;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x)
    split_bf16(w_mix_src(W, i, fwd != 0, Ko, Kd, C, H), pair[i], pair[total + i]);
}

int permute_w_mix_bf16x3(const float* W, __nv_bfloat16* pair, int fwd, int Ko, int Kd, int C, int H, cudaStream_t s) {
  MPGCN_CHECK(C % 32 == 0 && H % 32 == 0, "permute_w_mix: C=%d H=%d are not multiples of 32", C, H);
  prof_count(PROF_ELEMENTWISE);
  permute_w_mix_bf16x3_kernel<<<grid_for((size_t)Ko * Kd * C * H, 256), 256, 0, s>>>(W, pair, fwd, Ko, Kd, C, H);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

int permute_w_mix(const float* W, __half* hi, __half* lo, int Ko, int Kd, int C, int H, cudaStream_t s) {
  MPGCN_CHECK(C % 32 == 0 && H % 32 == 0, "permute_w_mix: C=%d H=%d are not multiples of 32", C, H);
  prof_count(PROF_ELEMENTWISE);
  permute_w_mix_kernel<<<grid_for((size_t)Ko * Kd * C * H, 256), 256, 0, s>>>(W, hi, lo, Ko, Kd, C, H);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

__global__ void reduce_dw_kernel(const float* __restrict__ P, float* __restrict__ dW, int slices, int MT, int Ko, int Kd, int C, int H,
                                 const float* __restrict__ inv_scale) {
  const float a = inv_scale ? __ldg(inv_scale) : 1.f;
  // dW index i = ((o*Kd + d)*C + c)*H + h ; partial row d*C + c (= m-tile (d*C + c) / 128), column o*H + h
  const int total = Ko * Kd * C * H;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int h = i % H;
    const int c = (i / H) % C;
    const int d = (i / (H * C)) % Kd;
    const int o = i / (H * C * Kd);
    const size_t row = (size_t)d * C + c;
    float sum = 0.f;
    for (int s = 0; s < slices; ++s) sum += P[((size_t)s * MT * 128 + row) * Ko * H + (size_t)o * H + h];
    dW[i] = sum * a;
  }
}

int reduce_dw_partials(const float* P, float* dW, int slices, int MT, int Ko, int Kd, int C, int H, const float* inv_scale, cudaStream_t s) {
  prof_count(PROF_ELEMENTWISE);
  reduce_dw_kernel<<<grid_for((size_t)Ko * Kd * C * H, 256), 256, 0, s>>>(P, dW, slices, MT, Ko, Kd, C, H, inv_scale);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

__global__ void reduce_dg_kernel(const float* __restrict__ P, float* __restrict__ dG, int slices, int N, int ldp,
                                 const float* __restrict__ inv_scale, int accumulate) {
  const float a = inv_scale ? __ldg(inv_scale) : 1.f;
  const size_t total = (size_t)N * N, slice = (size_t)N * ldp;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t r = i / N, c = i % N;
    float sum = 0.f;
    for (int s = 0; s < slices; ++s) sum += P[s * slice + r * ldp + c];
    dG[i] = accumulate ? fmaf(sum, a, dG[i]) : sum * a;
  }
}

int reduce_dg_partials(const float* P, float* dG, int slices, int N, int ldp, const float* inv_scale, int accumulate, cudaStream_t s) {
  prof_count(PROF_BWD_DG);
  reduce_dg_kernel<<<grid_for((size_t)N * N, 256), 256, 0, s>>>(P, dG, slices, N, ldp, inv_scale, accumulate);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

// Block (32, 32): lane x owns image element blockIdx.x * 32 + x (coalesced across the slot), warp y adds slots y, y + 32, ... in
// slot order, and warp 0 adds the 32 group sums in group order.  The order depends on the slot count only, never on timing.
__global__ void __launch_bounds__(1024) reduce_slots_kernel(const float* __restrict__ P, int slots, long long s_stride,
                                                            long long a_stride, SlotImage img) {
  __shared__ float part[32][33];
  const long long i = (long long)blockIdx.x * 32 + threadIdx.x;
  const float* src = P + (long long)blockIdx.y * a_stride + i;
  float acc = 0.f;
  if (i < img.end[2])
    for (int t = threadIdx.y; t < slots; t += 32) acc += src[(long long)t * s_stride];
  part[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && i < img.end[2]) {
    float sum = 0.f;
#pragma unroll
    for (int w = 0; w < 32; ++w) sum += part[w][threadIdx.x];
    const int k = i < img.end[0] ? 0 : i < img.end[1] ? 1 : 2;
    const long long start = k == 0 ? 0 : img.end[k - 1];
    img.dst[k][(long long)blockIdx.y * (img.end[k] - start) + (i - start)] = sum;
  }
}

SlotImage slot_image(float* d0, long long n0, float* d1, long long n1, float* d2, long long n2) {
  SlotImage m;
  m.dst[0] = d0; m.dst[1] = d1; m.dst[2] = d2;
  m.end[0] = n0; m.end[1] = n0 + n1; m.end[2] = n0 + n1 + n2;
  return m;
}

int reduce_slots(const float* P, int slots, long long s_stride, int rows, long long a_stride, const SlotImage& img, cudaStream_t s) {
  MPGCN_CHECK(slots >= 1 && rows >= 1 && img.end[2] >= 1, "reduce_slots: empty reduction");
  prof_count(PROF_ELEMENTWISE);
  reduce_slots_kernel<<<dim3((unsigned)((img.end[2] + 31) / 32), (unsigned)rows), dim3(32, 32), 0, s>>>(P, slots, s_stride, a_stride, img);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

__global__ void mask_delta_rows_kernel(const float* __restrict__ delta, float* __restrict__ out, size_t total, int N, int row0, int rows) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i % N) - row0;
    out[i] = (r >= 0 && r < rows) ? delta[i] : 0.f;
  }
}
int mask_delta_rows(const float* delta, float* out, size_t planes, int N, int row0, int rows, cudaStream_t s) {
  prof_count(PROF_ELEMENTWISE);
  mask_delta_rows_kernel<<<grid_for(planes * N, 256), 256, 0, s>>>(delta, out, planes * N, N, row0, rows);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

// ---- exchange steps of the origin-row shard, fused into elementwise kernels over PEER memory (NVLink P2P loads / stores) ----
// out[b][i] = act( sum_j parts[j][b * full + off + i] + bias[i % H] ) for i < n; grid.y = sample b.  For the row shard's reduce-scatter
// of the partial pre-activations, every rank reads ITS rows out of all g partial buffers (its own and, over NVLink, the peers') and
// applies the bias / activation epilogue (reference MPGCN.py:47-49).  bias_act_inplace is g = 1, parts[0] == out: out and parts
// alias, hence no __restrict__ on them.
template <int V>
__global__ void reduce_bias_act_kernel(float* out, PeerPtrs<const float> parts, int g, const float* __restrict__ bias, int act, size_t n,
                                       size_t full, size_t off, int H) {
  const size_t b = blockIdx.y;
  for (size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * V; i < n; i += (size_t)gridDim.x * blockDim.x * V) {
    float acc[V];
    ld_cs_v(parts.p[0] + b * full + off + i, acc);
#pragma unroll
    for (int j = 1; j < 8; ++j) {
      if (j < g) {
        float v[V];
        ld_cs_v(parts.p[j] + b * full + off + i, v);
#pragma unroll
        for (int e = 0; e < V; ++e) acc[e] += v[e];
      }
    }
    if (bias) {
      float bb[V];
      ld_v(bias + i % H, bb);
#pragma unroll
      for (int e = 0; e < V; ++e) acc[e] += bb[e];
    }
    if (act)
#pragma unroll
      for (int e = 0; e < V; ++e) acc[e] = fmaxf(acc[e], 0.f);
    st_v(out + b * n + i, acc, 1.f);
  }
}
// B samples of n outputs, 256 threads; V = 4 when H, n, full, off are multiples of 4 and every pointer is 16-byte aligned
static int reduce_bias_act(float* out, const float* const* parts, int g, const float* bias, int act, int B, size_t n, size_t full, size_t off,
                           int H, ProfTag tag, cudaStream_t s) {
  MPGCN_CHECK(g >= 1 && g <= 8, "rows_reduce: %d ranks unsupported (1..8)", g);
  MPGCN_CHECK(H >= 1, "bias_act: H=%d", H);
  bool vec = H % 4 == 0 && (n | full | off) % 4 == 0 && aligned(out, 16) && aligned(bias, 16);
  PeerPtrs<const float> pp{};
  for (int j = 0; j < g; ++j) {
    MPGCN_CHECK(parts[j] != nullptr, "rows_reduce: partial buffer %d is null", j);
    pp.p[j] = parts[j];
    vec = vec && aligned(parts[j], 16);
  }
  const dim3 grid(grid_for(vec ? n / 4 : n, 256), (unsigned)B);
  if (tag == PROF_EXCHANGE) prof_begin(tag, 0.0, s);
  else prof_count(tag);
  if (vec) reduce_bias_act_kernel<4><<<grid, 256, 0, s>>>(out, pp, g, bias, act, n, full, off, H);
  else reduce_bias_act_kernel<1><<<grid, 256, 0, s>>>(out, pp, g, bias, act, n, full, off, H);
  prof_end(s);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

int bias_act_inplace(float* x, const float* bias, int act, size_t n, int H, cudaStream_t s) {
  return reduce_bias_act(x, &x, 1, bias, act, 1, n, n, 0, H, PROF_ELEMENTWISE, s);
}

int rows_reduce_bias_act(float* out, const float* const* parts, int g, const float* bias, int act, int B, int N, int row0, int rows, int H,
                         cudaStream_t s) {
  MPGCN_CHECK(H >= 1 && row0 >= 0 && rows >= 1 && row0 + rows <= N, "rows_reduce: bad slab rows [%d, %d) of %d, H=%d", row0, row0 + rows, N, H);
  return reduce_bias_act(out, parts, g, bias, act, B, (size_t)rows * N * H, (size_t)N * N * H, (size_t)row0 * N * H, H, PROF_EXCHANGE, s);
}

// d_pre = d_out * [out > 0] (or d_out), written to rows [row0, row0 + rows) of EVERY destination buffer [B][N][N][H] -- the rank's own
// and, over NVLink, the peers': the all-gather of dPre fused with the ReLU mask; db[h] = sum d_pre.
int relu_backward_scatter(const float* d_out, const float* out, int act, float* const* dsts, int g, float* db, int B, int N, int row0, int rows,
                          int H, cudaStream_t s) {
  MPGCN_CHECK(row0 >= 0 && rows >= 1 && row0 + rows <= N, "relu_backward_scatter: bad slab rows [%d, %d) of %d", row0, row0 + rows, N);
  return relu_bwd_launch(d_out, out, act, dsts, g, db, nullptr, B, (size_t)rows * N * H, (size_t)N * N * H, (size_t)row0 * N * H, H,
                         PROF_EXCHANGE, s);
}
// the same storing fp16(S * d_pre), S from the global max|d_out|
int relu_backward_scatter_f16(const float* d_out, const float* out, int act, __half* const* dsts, int g, float* db, const float* absmax,
                              float* scale2, int B, int N, int row0, int rows, int H, cudaStream_t s) {
  MPGCN_CHECK(row0 >= 0 && rows >= 1 && row0 + rows <= N, "relu_backward_scatter_f16: bad slab rows [%d, %d) of %d", row0, row0 + rows, N);
  MPGCN_CHECK(absmax != nullptr && scale2 != nullptr, "relu_backward_scatter_f16: absmax / scale2 are required");
  prof_count(PROF_ELEMENTWISE);
  make_scale_kernel<<<1, 1, 0, s>>>(scale2, absmax);
  return relu_bwd_launch(d_out, out, act, dsts, g, db, scale2, B, (size_t)rows * N * H, (size_t)N * N * H, (size_t)row0 * N * H, H,
                         PROF_EXCHANGE, s);
}
int absmax_f32(const float* x, size_t n, float* out, cudaStream_t s) {
  MPGCN_CUDA(cudaMemsetAsync(out, 0, sizeof(float), s));
  prof_count(PROF_ELEMENTWISE);
  absmax_kernel<<<grid_for(n, 256), 256, 0, s>>>(x, n, reinterpret_cast<unsigned int*>(out));
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace mpgcn
