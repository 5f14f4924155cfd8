// fp32 CUDA-core path: a strided / batched / segmented SGEMM that evaluates every
// contraction of the BDGCN layer exactly in fp32 (precision mode 0), plus the elementwise
// and layout kernels shared with the tensor-core path.
//
// This is the exact-arithmetic mode of the product (used for shapes the tensor-core engine
// does not cover -- channel counts other than 32 -- and as the on-device cross-check of
// the fp16 tensor path).  It is NOT a CPU fallback: everything here runs on the GPU.
#include "kernels.h"

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
  float* D = p.D + z0 * p.d_sz[0] + z1 * p.d_sz[1] + z2 * p.d_sz[2];
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
      if (p.ksplit > 1) {
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

__global__ void cvt_f16_hilo_kernel(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float x = src[i];
    const __half h = f2h_sat(x);
    hi[i] = h;
    lo[i] = f2h_sat(x - __half2float(h));
  }
}
int cvt_f32_to_f16_hilo(const float* src, __half* hi, __half* lo, size_t n, cudaStream_t s) {
  if (n == 0) return 0;
  prof_count(PROF_ELEMENTWISE);
  cvt_f16_hilo_kernel<<<grid_for(n, 256), 256, 0, s>>>(src, hi, lo, n);
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

// d_pre = d_out * [out > 0];  db[h] += sum over cells.  Thread's channel is fixed because the
// grid stride is a multiple of H.
__global__ void relu_bwd_prep_kernel(const float* __restrict__ d_out, const float* __restrict__ out, int relu,
                                     __half* __restrict__ d16, float* __restrict__ d32, float* __restrict__ db, size_t n, int H,
                                     const float* __restrict__ scale) {
  const float S = scale ? __ldg(scale) : 1.f;
  extern __shared__ float s_db[];   // [blockDim.x]
  const size_t stride = (size_t)gridDim.x * blockDim.x;   // multiple of H by construction
  float local = 0.f;
  const size_t first = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (size_t i = first; i < n; i += stride) {
    float g = d_out[i];
    if (relu && !(out[i] > 0.f)) g = 0.f;
    if (d16) d16[i] = f2h_sat(g * S);
    if (d32) d32[i] = g;
    local += g;
  }
  if (db) {
    s_db[threadIdx.x] = local;
    __syncthreads();
    if ((int)threadIdx.x < H) {
      // threads t, t+H, t+2H, ... of this block share channel (first % H)
      float sum = 0.f;
      for (int t = threadIdx.x; t < (int)blockDim.x; t += H) sum += s_db[t];
      const int ch = (int)(((size_t)blockIdx.x * blockDim.x + threadIdx.x) % H);
      atomicAdd(&db[ch], sum);
    }
  }
}

// Same, four channels per thread (float4 loads, one 8-byte fp16 store): H % 4 == 0, H / 4 divides the block size, so a
// thread keeps its four channels across the grid-stride loop.
__global__ void relu_bwd_prep_vec4_kernel(const float4* __restrict__ d_out, const float4* __restrict__ out, int relu,
                                          uint2* __restrict__ d16, float4* __restrict__ d32, float* __restrict__ db, size_t n4, int H4,
                                          const float* __restrict__ scale) {
  const float S = scale ? __ldg(scale) : 1.f;
  extern __shared__ float s_db[];   // [4][blockDim.x]
  const size_t stride = (size_t)gridDim.x * blockDim.x;   // multiple of H4 by construction
  float l0 = 0.f, l1 = 0.f, l2 = 0.f, l3 = 0.f;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 g = d_out[i];
    if (relu) {
      const float4 o = out[i];
      g.x = o.x > 0.f ? g.x : 0.f; g.y = o.y > 0.f ? g.y : 0.f;
      g.z = o.z > 0.f ? g.z : 0.f; g.w = o.w > 0.f ? g.w : 0.f;
    }
    if (d16) {
      const __half2 a = __halves2half2(f2h_sat(g.x * S), f2h_sat(g.y * S)), b = __halves2half2(f2h_sat(g.z * S), f2h_sat(g.w * S));
      d16[i] = make_uint2(*reinterpret_cast<const unsigned int*>(&a), *reinterpret_cast<const unsigned int*>(&b));
    }
    if (d32) d32[i] = g;
    l0 += g.x; l1 += g.y; l2 += g.z; l3 += g.w;
  }
  if (db) {
    const int nt = blockDim.x;
    s_db[threadIdx.x] = l0; s_db[nt + threadIdx.x] = l1; s_db[2 * nt + threadIdx.x] = l2; s_db[3 * nt + threadIdx.x] = l3;
    __syncthreads();
    if ((int)threadIdx.x < 4 * H4) {       // one thread per channel: quad q = channel / 4, component e = channel % 4
      const int q = threadIdx.x >> 2, e = threadIdx.x & 3;
      float sum = 0.f;
      for (int t = q; t < nt; t += H4) sum += s_db[e * nt + t];
      const int quad0 = (int)(((size_t)blockIdx.x * blockDim.x) % H4);      // channel quad of thread 0 of this block
      atomicAdd(&db[((q + quad0) % H4) * 4 + e], sum);
    }
  }
}

__global__ void relu_bwd_prep_f16mask_kernel(const float4* __restrict__ d_out, const uint2* __restrict__ out16, int relu,
                                             uint2* __restrict__ d16, float* __restrict__ db, size_t n4, int H4,
                                             const float* __restrict__ scale) {
  const float S = scale ? __ldg(scale) : 1.f;
  extern __shared__ float s_db[];   // [4][blockDim.x]
  const size_t stride = (size_t)gridDim.x * blockDim.x;   // multiple of H4 by construction
  float l0 = 0.f, l1 = 0.f, l2 = 0.f, l3 = 0.f;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 g = d_out[i];
    if (relu) {
      const uint2 o = out16[i];
      const float2 o01 = __half22float2(*reinterpret_cast<const __half2*>(&o.x)), o23 = __half22float2(*reinterpret_cast<const __half2*>(&o.y));
      g.x = o01.x > 0.f ? g.x : 0.f; g.y = o01.y > 0.f ? g.y : 0.f;
      g.z = o23.x > 0.f ? g.z : 0.f; g.w = o23.y > 0.f ? g.w : 0.f;
    }
    const __half2 a = __halves2half2(f2h_sat(g.x * S), f2h_sat(g.y * S)), b = __halves2half2(f2h_sat(g.z * S), f2h_sat(g.w * S));
    d16[i] = make_uint2(*reinterpret_cast<const unsigned int*>(&a), *reinterpret_cast<const unsigned int*>(&b));
    l0 += g.x; l1 += g.y; l2 += g.z; l3 += g.w;
  }
  if (db) {
    const int nt = blockDim.x;
    s_db[threadIdx.x] = l0; s_db[nt + threadIdx.x] = l1; s_db[2 * nt + threadIdx.x] = l2; s_db[3 * nt + threadIdx.x] = l3;
    __syncthreads();
    if ((int)threadIdx.x < 4 * H4) {
      const int q = threadIdx.x >> 2, e = threadIdx.x & 3;
      float sum = 0.f;
      for (int t = q; t < nt; t += H4) sum += s_db[e * nt + t];
      const int quad0 = (int)(((size_t)blockIdx.x * blockDim.x) % H4);
      atomicAdd(&db[((q + quad0) % H4) * 4 + e], sum);
    }
  }
}

// block size of the four-channel kernels: a multiple of H / 4 (a thread keeps its channel quad across the grid-stride loop) with
// at least one thread per channel for the bias-gradient reduction; 256 for every H <= 256 whose quad count divides 256
static int quad_block(int H) {
  const int H4 = H / 4;
  return H4 * (256 / H4 > 4 ? 256 / H4 : 4);
}

int relu_bwd_prep_f16mask(const float* d_out, const __half* out16, int relu, __half* d16, float* db, size_t n, int H, const float* scale,
                          cudaStream_t s) {
  if (n == 0) return 0;
  MPGCN_CHECK(H % 4 == 0 && H >= 4 && H <= 1024 && n % 4 == 0, "relu_bwd_prep_f16mask: H=%d / n=%zu unsupported", H, n);
  MPGCN_CHECK(((reinterpret_cast<uintptr_t>(d_out) & 15) | (reinterpret_cast<uintptr_t>(out16) & 7) | (reinterpret_cast<uintptr_t>(d16) & 7)) == 0,
              "relu_bwd_prep_f16mask: misaligned pointer");
  const int threads = quad_block(H);
  prof_count(PROF_ELEMENTWISE);
  relu_bwd_prep_f16mask_kernel<<<grid_for(n / 4, threads), threads, 4 * threads * sizeof(float), s>>>(
      reinterpret_cast<const float4*>(d_out), reinterpret_cast<const uint2*>(out16), relu, reinterpret_cast<uint2*>(d16), db, n / 4, H / 4, scale);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

int relu_bwd_prep(const float* d_out, const float* out, int relu, __half* d16, float* d32, float* db, size_t n, int H,
                  const float* scale, cudaStream_t s) {
  if (n == 0) return 0;
  MPGCN_CHECK(H >= 1 && H <= 1024, "relu_bwd_prep: H=%d unsupported", H);
  const bool aligned = ((reinterpret_cast<uintptr_t>(d_out) | reinterpret_cast<uintptr_t>(out) | reinterpret_cast<uintptr_t>(d32)) & 15) == 0 &&
                       (reinterpret_cast<uintptr_t>(d16) & 7) == 0;
  if (H % 4 == 0 && 256 % (H / 4) == 0 && n % 4 == 0 && aligned) {
    const int threads = quad_block(H);
    unsigned blocks = grid_for(n / 4, threads);
    prof_count(PROF_ELEMENTWISE);
    relu_bwd_prep_vec4_kernel<<<blocks, threads, 4 * threads * sizeof(float), s>>>(
        reinterpret_cast<const float4*>(d_out), reinterpret_cast<const float4*>(out), relu, reinterpret_cast<uint2*>(d16),
        reinterpret_cast<float4*>(d32), db, n / 4, H / 4, scale);
    MPGCN_CUDA(cudaGetLastError());
    return 0;
  }
  int threads = (256 / H) * H;          // multiple of H so each thread keeps one channel
  if (threads == 0) threads = H;
  unsigned blocks = grid_for(n, threads);
  prof_count(PROF_ELEMENTWISE);
  relu_bwd_prep_kernel<<<blocks, threads, threads * sizeof(float), s>>>(d_out, out, relu, d16, d32, db, n, H, scale);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

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

__global__ void permute_w_bwd_kernel(const float* __restrict__ W, __half* __restrict__ q16, float* __restrict__ q32, int Ko, int Kd, int C,
                                     int H) {
  const int total = Ko * Kd * C * H;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    // destination index i = ((d*Ko + o)*H + h)*C + l
    const int l = i % C;
    const int h = (i / C) % H;
    const int o = (i / (C * H)) % Ko;
    const int d = i / (C * H * Ko);
    const float v = W[((size_t)(o * Kd + d) * C + l) * H + h];
    if (q16) q16[i] = f2h_sat(v);
    if (q32) q32[i] = v;
  }
}

int permute_w_bwd(const float* W, __half* wq16, float* wq32, int Ko, int Kd, int C, int H, cudaStream_t s) {
  prof_count(PROF_ELEMENTWISE);
  permute_w_bwd_kernel<<<grid_for((size_t)Ko * Kd * C * H, 256), 256, 0, s>>>(W, wq16, wq32, Ko, Kd, C, H);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

// W[o][d][32 lc + l][32 hc + h] -> one [32][32] block per (output plane, input plane) of a channel mix, see kernels.h
__global__ void permute_w_mix_kernel(const float* __restrict__ W, __half* __restrict__ hi, __half* __restrict__ lo, int Ko, int Kd, int C,
                                     int H) {
  const int cC = C / 32, cH = H / 32;
  const int total = Ko * Kd * C * H;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int e0 = i % 32, e1 = (i / 32) % 32, blk = i / 1024;
    int o, d, lc, hc, l, h;
    if (lo) {      // forward: i = ((hc*Ko + o)*Kd*cC + d*cC + lc)*1024 + l*32 + h
      h = e0; l = e1;
      const int sp = blk % (Kd * cC), r = blk / (Kd * cC);
      d = sp / cC; lc = sp % cC; o = r % Ko; hc = r / Ko;
    } else {       // backward: i = ((d*cC + lc)*Ko*cH + o*cH + hc)*1024 + h*32 + l
      l = e0; h = e1;
      const int sp = blk % (Ko * cH), r = blk / (Ko * cH);
      o = sp / cH; hc = sp % cH; d = r / cC; lc = r % cC;
    }
    const float v = W[((size_t)(o * Kd + d) * C + lc * 32 + l) * H + hc * 32 + h];
    const __half x = f2h_sat(v);
    hi[i] = x;
    if (lo) lo[i] = f2h_sat(v - __half2float(x));
  }
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

// in place: x = act(x + bias[channel]); H % 4 == 0 and 16-byte alignment take the float4 path
__global__ void bias_act_vec4_kernel(float4* __restrict__ x, const float* __restrict__ bias, int act, size_t n4, int H4) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    float4 v = x[i];
    if (bias) {
      const float4 b = reinterpret_cast<const float4*>(bias)[i % H4];
      v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w;
    }
    if (act) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    x[i] = v;
  }
}
__global__ void bias_act_kernel(float* __restrict__ x, const float* __restrict__ bias, int act, size_t n, int H) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float v = x[i] + (bias ? bias[i % H] : 0.f);
    x[i] = act ? fmaxf(v, 0.f) : v;
  }
}
// ---- exchange steps of the origin-row shard, fused into elementwise kernels over PEER memory (NVLink P2P loads / stores) ----
struct PeerPtrs { float* p[8]; };

// out[b][r][e][h] = act( sum_j part[j][b][row0 + r][e][h] + bias[h] ): the reduce-scatter of the partial pre-activations -- every rank
// reads ITS rows out of all g partial buffers (its own and, over NVLink, the peers') -- fused with the bias / activation epilogue
// (reference MPGCN.py:47-49).  grid.y = sample; x4 = float4 index inside the sample's slab.
__global__ void rows_reduce_bias_act_kernel(float4* __restrict__ out, PeerPtrs parts, int g, const float* __restrict__ bias, int act,
                                            size_t slab4 /*rows*N*H/4*/, size_t full4 /*N*N*H/4*/, size_t off4 /*row0*N*H/4*/, int H4) {
  const size_t b = blockIdx.y;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < slab4; i += (size_t)gridDim.x * blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (j < g) {
        const float4 v = __ldcs(reinterpret_cast<const float4*>(parts.p[j]) + b * full4 + off4 + i);      // read once: streaming
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
    }
    if (bias) {
      const float4 bb = reinterpret_cast<const float4*>(bias)[i % H4];
      acc.x += bb.x; acc.y += bb.y; acc.z += bb.z; acc.w += bb.w;
    }
    if (act) { acc.x = fmaxf(acc.x, 0.f); acc.y = fmaxf(acc.y, 0.f); acc.z = fmaxf(acc.z, 0.f); acc.w = fmaxf(acc.w, 0.f); }
    out[b * slab4 + i] = acc;
  }
}
int rows_reduce_bias_act(float* out, const float* const* parts, int g, const float* bias, int act, int B, int N, int row0, int rows, int H,
                         cudaStream_t s) {
  MPGCN_CHECK(g >= 1 && g <= 8, "rows_reduce: %d ranks unsupported (1..8)", g);
  MPGCN_CHECK(H % 4 == 0 && row0 >= 0 && rows >= 1 && row0 + rows <= N, "rows_reduce: bad slab rows [%d, %d) of %d, H=%d", row0, row0 + rows, N, H);
  PeerPtrs pp{};
  for (int j = 0; j < g; ++j) {
    MPGCN_CHECK(parts[j] != nullptr && (reinterpret_cast<uintptr_t>(parts[j]) & 15) == 0, "rows_reduce: partial buffer %d null or misaligned", j);
    pp.p[j] = const_cast<float*>(parts[j]);
  }
  const size_t slab4 = (size_t)rows * N * H / 4, full4 = (size_t)N * N * H / 4, off4 = (size_t)row0 * N * H / 4;
  dim3 grid(grid_for(slab4, 256), (unsigned)B);
  prof_begin(PROF_EXCHANGE, 0.0, s);
  rows_reduce_bias_act_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<float4*>(out), pp, g, bias, act, slab4, full4, off4, H / 4);
  prof_end(s);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

// d_pre = d_out * [out > 0] (or d_out), written to rows [row0, row0 + rows) of EVERY destination buffer [B][N][N][H] -- the rank's own
// and, over NVLink, the peers': the all-gather of dPre fused with the ReLU mask; db[h] += sum d_pre.  H4 divides the block size,
// so a thread keeps its four channels.
__global__ void relu_backward_scatter_kernel(const float4* __restrict__ d_out, const float4* __restrict__ out, int act, PeerPtrs dst, int g,
                                             float* __restrict__ db, size_t slab4, size_t full4, size_t off4, int H4) {
  extern __shared__ float s_db[];   // [4][blockDim.x]
  const size_t b = blockIdx.y;
  float l0 = 0.f, l1 = 0.f, l2 = 0.f, l3 = 0.f;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < slab4; i += (size_t)gridDim.x * blockDim.x) {
    float4 gq = d_out[b * slab4 + i];
    if (act) {
      const float4 o = out[b * slab4 + i];
      gq.x = o.x > 0.f ? gq.x : 0.f; gq.y = o.y > 0.f ? gq.y : 0.f; gq.z = o.z > 0.f ? gq.z : 0.f; gq.w = o.w > 0.f ? gq.w : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (j < g) reinterpret_cast<float4*>(dst.p[j])[b * full4 + off4 + i] = gq;
    l0 += gq.x; l1 += gq.y; l2 += gq.z; l3 += gq.w;
  }
  if (db) {
    const int nt = blockDim.x;
    s_db[threadIdx.x] = l0; s_db[nt + threadIdx.x] = l1; s_db[2 * nt + threadIdx.x] = l2; s_db[3 * nt + threadIdx.x] = l3;
    __syncthreads();
    if ((int)threadIdx.x < 4 * H4) {       // one thread per channel: quad q = channel / 4, component e = channel % 4
      const int q = threadIdx.x >> 2, e = threadIdx.x & 3;
      float sum = 0.f;
      for (int t = q; t < nt; t += H4) sum += s_db[e * nt + t];      // threads t = q (mod H4) own quad q (the grid stride is a multiple of H4)
      atomicAdd(&db[q * 4 + e], sum);
    }
  }
}
int relu_backward_scatter(const float* d_out, const float* out, int act, float* const* dsts, int g, float* db, int B, int N, int row0, int rows,
                          int H, cudaStream_t s) {
  MPGCN_CHECK(g >= 1 && g <= 8, "relu_backward_scatter: %d ranks unsupported (1..8)", g);
  MPGCN_CHECK(H % 4 == 0 && 256 % (H / 4) == 0 && 4 * (H / 4) <= 256, "relu_backward_scatter: H=%d unsupported", H);
  MPGCN_CHECK(row0 >= 0 && rows >= 1 && row0 + rows <= N, "relu_backward_scatter: bad slab rows [%d, %d) of %d", row0, row0 + rows, N);
  PeerPtrs pp{};
  for (int j = 0; j < g; ++j) {
    MPGCN_CHECK(dsts[j] != nullptr && (reinterpret_cast<uintptr_t>(dsts[j]) & 15) == 0, "relu_backward_scatter: destination %d null or misaligned", j);
    pp.p[j] = dsts[j];
  }
  if (db) MPGCN_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * H, s));
  const size_t slab4 = (size_t)rows * N * H / 4, full4 = (size_t)N * N * H / 4, off4 = (size_t)row0 * N * H / 4;
  dim3 grid(grid_for(slab4, 256), (unsigned)B);
  prof_begin(PROF_EXCHANGE, 0.0, s);
  relu_backward_scatter_kernel<<<grid, 256, 4 * 256 * sizeof(float), s>>>(reinterpret_cast<const float4*>(d_out), reinterpret_cast<const float4*>(out),
                                                                         act, pp, g, db, slab4, full4, off4, H / 4);
  prof_end(s);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

struct PeerPtrs16 { __half* p[8]; };
__global__ void relu_backward_scatter_f16_kernel(const float4* __restrict__ d_out, const float4* __restrict__ out, int act, PeerPtrs16 dst, int g,
                                                 float* __restrict__ db, const float* __restrict__ scale2, size_t slab4, size_t full4, size_t off4,
                                                 int H4) {
  extern __shared__ float s_db[];   // [4][blockDim.x]
  const float S = __ldg(scale2);
  const size_t b = blockIdx.y;
  float l0 = 0.f, l1 = 0.f, l2 = 0.f, l3 = 0.f;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < slab4; i += (size_t)gridDim.x * blockDim.x) {
    float4 gq = d_out[b * slab4 + i];
    if (act) {
      const float4 o = out[b * slab4 + i];
      gq.x = o.x > 0.f ? gq.x : 0.f; gq.y = o.y > 0.f ? gq.y : 0.f; gq.z = o.z > 0.f ? gq.z : 0.f; gq.w = o.w > 0.f ? gq.w : 0.f;
    }
    const __half2 lo = __halves2half2(f2h_sat(gq.x * S), f2h_sat(gq.y * S)), hi = __halves2half2(f2h_sat(gq.z * S), f2h_sat(gq.w * S));
    const uint2 pk = make_uint2(*reinterpret_cast<const unsigned int*>(&lo), *reinterpret_cast<const unsigned int*>(&hi));
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (j < g) reinterpret_cast<uint2*>(dst.p[j])[b * full4 + off4 + i] = pk;
    l0 += gq.x; l1 += gq.y; l2 += gq.z; l3 += gq.w;
  }
  if (db) {
    const int nt = blockDim.x;
    s_db[threadIdx.x] = l0; s_db[nt + threadIdx.x] = l1; s_db[2 * nt + threadIdx.x] = l2; s_db[3 * nt + threadIdx.x] = l3;
    __syncthreads();
    if ((int)threadIdx.x < 4 * H4) {
      const int q = threadIdx.x >> 2, e = threadIdx.x & 3;
      float sum = 0.f;
      for (int t = q; t < nt; t += H4) sum += s_db[e * nt + t];
      atomicAdd(&db[q * 4 + e], sum);
    }
  }
}
int relu_backward_scatter_f16(const float* d_out, const float* out, int act, __half* const* dsts, int g, float* db, const float* absmax,
                              float* scale2, int B, int N, int row0, int rows, int H, cudaStream_t s) {
  MPGCN_CHECK(g >= 1 && g <= 8, "relu_backward_scatter_f16: %d ranks unsupported (1..8)", g);
  MPGCN_CHECK(H % 4 == 0 && 256 % (H / 4) == 0 && 4 * (H / 4) <= 256, "relu_backward_scatter_f16: H=%d unsupported", H);
  MPGCN_CHECK(row0 >= 0 && rows >= 1 && row0 + rows <= N, "relu_backward_scatter_f16: bad slab rows [%d, %d) of %d", row0, row0 + rows, N);
  MPGCN_CHECK(absmax != nullptr && scale2 != nullptr, "relu_backward_scatter_f16: absmax / scale2 are required");
  PeerPtrs16 pp{};
  for (int j = 0; j < g; ++j) {
    MPGCN_CHECK(dsts[j] != nullptr && (reinterpret_cast<uintptr_t>(dsts[j]) & 7) == 0, "relu_backward_scatter_f16: destination %d null or misaligned", j);
    pp.p[j] = dsts[j];
  }
  if (db) MPGCN_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * H, s));
  prof_count(PROF_ELEMENTWISE);
  make_scale_kernel<<<1, 1, 0, s>>>(scale2, absmax);
  const size_t slab4 = (size_t)rows * N * H / 4, full4 = (size_t)N * N * H / 4, off4 = (size_t)row0 * N * H / 4;
  dim3 grid(grid_for(slab4, 256), (unsigned)B);
  prof_begin(PROF_EXCHANGE, 0.0, s);
  relu_backward_scatter_f16_kernel<<<grid, 256, 4 * 256 * sizeof(float), s>>>(reinterpret_cast<const float4*>(d_out), reinterpret_cast<const float4*>(out),
                                                                             act, pp, g, db, scale2, slab4, full4, off4, H / 4);
  prof_end(s);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}
int absmax_f32(const float* x, size_t n, float* out, cudaStream_t s) {
  MPGCN_CUDA(cudaMemsetAsync(out, 0, sizeof(float), s));
  prof_count(PROF_ELEMENTWISE);
  absmax_kernel<<<grid_for(n, 256), 256, 0, s>>>(x, n, reinterpret_cast<unsigned int*>(out));
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

int bias_act_inplace(float* x, const float* bias, int act, size_t n, int H, cudaStream_t s) {
  MPGCN_CHECK(H >= 1, "bias_act: H=%d", H);
  prof_count(PROF_ELEMENTWISE);
  const bool vec = (H % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(bias)) & 15) == 0;
  if (vec) bias_act_vec4_kernel<<<grid_for(n / 4, 256), 256, 0, s>>>(reinterpret_cast<float4*>(x), bias, act, n / 4, H / 4);
  else bias_act_kernel<<<grid_for(n, 256), 256, 0, s>>>(x, bias, act, n, H);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace mpgcn
