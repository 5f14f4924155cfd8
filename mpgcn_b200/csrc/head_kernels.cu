// FC head + branch fusion of the MPGCN model in one pass (reference: /root/reference/MPGCN.py:74-76,107,110,112):
//     y[b,n,c] = (1/M) * sum_m relu( g_m[b,n,c,:] . w_m + bias_m )          (Linear(C -> 1) + ReLU per branch, mean over branches)
// HBM-bound elementwise work: each cell reads M x C floats and writes one.  Eight threads share a cell (a float4 each for
// C = 32; generally C/8 strided elements), so a warp reads four consecutive cells = 512 contiguous bytes per branch.
#include "kernels.h"

namespace mpgcn {

constexpr int kMaxBranches = 8;

struct HeadPtrs {
  const float* g[kMaxBranches];      // [cells][C] per branch
  float* dg[kMaxBranches];           // backward: [cells][C] per branch
};

// MT = compile-time branch count (1..4; the branch loop is unrolled, so HeadPtrs stays in the constant bank: with a run-time
// index the whole struct was copied to local memory and every p.g[m] became a local load) or 0 = run-time M
template <int MT>
__global__ void head_fwd_kernel(HeadPtrs p, const float* __restrict__ w /*[M][C]*/, const float* __restrict__ bias /*[M]*/,
                                float* __restrict__ y, float* __restrict__ pre /*[M][cells] or null*/, long long cells, int C, int Mrt) {
  const int M = MT ? MT : Mrt;
  const int sub = threadIdx.x & 7;
  const long long stride = (long long)gridDim.x * (blockDim.x >> 3);
  constexpr int U = 4;               // cells per thread and iteration: U x M independent 16-byte loads in flight
  // The eight lanes of a cell shuffle among themselves only: the four 8-lane groups of a warp own different cells, so near
  // the end of the range (cells % 4 != 0, e.g. N = 47 with an odd batch) some groups have left the loop while others reduce.
  const unsigned gmask = 0xFFu << (threadIdx.x & 24);
  for (long long cell0 = (long long)blockIdx.x * (blockDim.x >> 3) + (threadIdx.x >> 3); cell0 < cells; cell0 += U * stride) {
    float acc[U];
#pragma unroll
    for (int u = 0; u < U; ++u) acc[u] = 0.f;
#pragma unroll
    for (int m = 0; m < (MT ? MT : kMaxBranches); ++m) {
      if (!MT && m >= M) break;
      float s[U];
      float4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {          // issue every load of the iteration first (C <= 32: one float4 per thread and cell)
        const long long cell = cell0 + u * stride;
        v[u] = (cell < cells && sub * 4 < C) ? *reinterpret_cast<const float4*>(p.g[m] + cell * C + sub * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      const float4 w0 = (sub * 4 < C) ? *reinterpret_cast<const float4*>(w + m * C + sub * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        s[u] = v[u].x * w0.x + v[u].y * w0.y + v[u].z * w0.z + v[u].w * w0.w;
        const long long cell = cell0 + u * stride;
        if (C > 32 && cell < cells) {
          const float* g = p.g[m] + cell * C;
          for (int l = sub * 4 + 32; l < C; l += 32) {
            const float4 vv = *reinterpret_cast<const float4*>(g + l);
            const float4 ww = *reinterpret_cast<const float4*>(w + m * C + l);
            s[u] += vv.x * ww.x + vv.y * ww.y + vv.z * ww.z + vv.w * ww.w;
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        s[u] += __shfl_xor_sync(gmask, s[u], 1);
        s[u] += __shfl_xor_sync(gmask, s[u], 2);
        s[u] += __shfl_xor_sync(gmask, s[u], 4);
        s[u] += bias[m];
        const long long cell = cell0 + u * stride;
        if (pre != nullptr && sub == 0 && cell < cells) pre[(long long)m * cells + cell] = s[u];
        acc[u] += fmaxf(s[u], 0.f);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long cell = cell0 + u * stride;
      if (sub == 0 && cell < cells) y[cell] = acc[u] / (float)M;
    }
  }
}

// d g_m[cell,:] = dy[cell]/M * [pre_m > 0] * w_m ;  dw_m += sum_cell d_pre * g_m[cell,:] ;  db_m += sum_cell d_pre
template <int MT>
__global__ void head_bwd_kernel(HeadPtrs p, const float* __restrict__ w, const float* __restrict__ pre, const float* __restrict__ dy,
                                float* __restrict__ dw /*[M][C]*/, float* __restrict__ db /*[M]*/, float* __restrict__ dg_absmax /*[M] or null*/,
                                long long cells, int C, int Mrt) {
  const int M = MT ? MT : Mrt;
  extern __shared__ float s_acc[];     // [M][C + 1] block-level accumulators
  for (int i = threadIdx.x; i < M * (C + 1); i += blockDim.x) s_acc[i] = 0.f;
  __syncthreads();
  const int sub = threadIdx.x & 7;
  const long long stride = (long long)gridDim.x * (blockDim.x >> 3);
  const float inv_m = 1.f / (float)M;
  // per-thread partial sums for the (few) weight elements this thread touches: C/8 per branch, kept in registers for C = 32
#pragma unroll
  for (int m = 0; m < (MT ? MT : kMaxBranches); ++m) {
    if (!MT && m >= M) break;
    float wacc[4] = {0.f, 0.f, 0.f, 0.f}, bacc = 0.f;     // C <= 32 fast path; larger C falls through to smem atomics below
    float amax = 0.f;
    constexpr int U = 4;             // cells per thread and iteration
    for (long long cell0 = (long long)blockIdx.x * (blockDim.x >> 3) + (threadIdx.x >> 3); cell0 < cells; cell0 += U * stride) {
      float d[U];
      float4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {          // issue every load of the iteration first (C <= 32: one float4 per thread and cell)
        const long long cell = cell0 + u * stride;
        const bool ok = cell < cells;
        d[u] = (ok && pre[(long long)m * cells + cell] > 0.f) ? dy[cell] * inv_m : 0.f;
        v[u] = (ok && sub * 4 < C) ? *reinterpret_cast<const float4*>(p.g[m] + cell * C + sub * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long cell = cell0 + u * stride;
        if (cell >= cells) continue;
        const float* g = p.g[m] + cell * C;
        float* dg = p.dg[m] ? p.dg[m] + cell * C : nullptr;
        for (int l = sub * 4; l < C; l += 32) {
          const float4 vv = (l < 32) ? v[u] : *reinterpret_cast<const float4*>(g + l);
          const float4 ww = *reinterpret_cast<const float4*>(w + m * C + l);
          if (dg) {
            const float4 o = make_float4(d[u] * ww.x, d[u] * ww.y, d[u] * ww.z, d[u] * ww.w);
            *reinterpret_cast<float4*>(dg + l) = o;
            amax = fmaxf(amax, fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fmaxf(fabsf(o.z), fabsf(o.w))));
          }
          if (l < 32) {
            wacc[0] += d[u] * vv.x; wacc[1] += d[u] * vv.y; wacc[2] += d[u] * vv.z; wacc[3] += d[u] * vv.w;
          } else {
            atomicAdd(&s_acc[m * (C + 1) + l], d[u] * vv.x); atomicAdd(&s_acc[m * (C + 1) + l + 1], d[u] * vv.y);
            atomicAdd(&s_acc[m * (C + 1) + l + 2], d[u] * vv.z); atomicAdd(&s_acc[m * (C + 1) + l + 3], d[u] * vv.w);
          }
        }
        if (sub == 0) bacc += d[u];
      }
    }
    if (sub * 4 < C) {
#pragma unroll
      for (int e = 0; e < 4; ++e) atomicAdd(&s_acc[m * (C + 1) + sub * 4 + e], wacc[e]);
    }
    if (sub == 0) atomicAdd(&s_acc[m * (C + 1) + C], bacc);
    if (dg_absmax) {
      for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
      if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<unsigned int*>(dg_absmax + m), __float_as_uint(amax));
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < M * (C + 1); i += blockDim.x) {
    const int m = i / (C + 1), l = i % (C + 1);
    if (l < C) atomicAdd(&dw[m * C + l], s_acc[i]);
    else atomicAdd(&db[m], s_acc[i]);
  }
}

// The same gradients in a fixed order (deterministic mode): a block's cells and the cells of each thread are those of
// head_bwd_kernel, but the weight sums never meet an atomic.  Channels go in chunks of 32: in chunk l0 thread (cell lane
// c = threadIdx.x / 8, sub) keeps channels l0 + 4 sub .. + 3 of its cells in registers, then thread t < 32 adds channel l0 + t over the
// 32 cell lanes in lane order; the bias sum is formed the same way in chunk 0.  The block stores [dw M x C | db M] to its slot,
// which reduce_slots adds over the blocks in block order.
template <int MT>
__global__ void head_bwd_det_kernel(HeadPtrs p, const float* __restrict__ w, const float* __restrict__ pre, const float* __restrict__ dy,
                                    float* __restrict__ slots, float* __restrict__ dg_absmax, long long cells, int C, int Mrt) {
  const int M = MT ? MT : Mrt;
  __shared__ float s_red[5][257];      // [4 channels | bias][thread]
  const int sub = threadIdx.x & 7, lane = threadIdx.x >> 3;
  const long long stride = (long long)gridDim.x * (blockDim.x >> 3);
  const float inv_m = 1.f / (float)M;
  float* slot = slots + (size_t)blockIdx.x * M * (C + 1);
#pragma unroll
  for (int m = 0; m < (MT ? MT : kMaxBranches); ++m) {
    if (!MT && m >= M) break;
    float amax = 0.f;
    for (int l0 = 0; l0 < C; l0 += 32) {
      const int l = l0 + sub * 4;
      const bool mine = l < C;
      const float4 ww = mine ? *reinterpret_cast<const float4*>(w + m * C + l) : make_float4(0.f, 0.f, 0.f, 0.f);
      float wacc[4] = {0.f, 0.f, 0.f, 0.f}, bacc = 0.f;
      for (long long cell = (long long)blockIdx.x * (blockDim.x >> 3) + lane; cell < cells; cell += stride) {
        const float d = pre[(long long)m * cells + cell] > 0.f ? dy[cell] * inv_m : 0.f;
        if (mine) {
          const float4 vv = *reinterpret_cast<const float4*>(p.g[m] + cell * C + l);
          wacc[0] += d * vv.x; wacc[1] += d * vv.y; wacc[2] += d * vv.z; wacc[3] += d * vv.w;
          if (p.dg[m]) {
            const float4 o = make_float4(d * ww.x, d * ww.y, d * ww.z, d * ww.w);
            *reinterpret_cast<float4*>(p.dg[m] + cell * C + l) = o;
            amax = fmaxf(amax, fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fmaxf(fabsf(o.z), fabsf(o.w))));
          }
        }
        bacc += d;
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) s_red[e][threadIdx.x] = wacc[e];
      s_red[4][threadIdx.x] = bacc;
      __syncthreads();
      if (threadIdx.x < 32 && l0 + (int)threadIdx.x < C) {
        const int sb = threadIdx.x >> 2, e = threadIdx.x & 3;
        float sum = 0.f;
        for (int c = 0; c < 32; ++c) sum += s_red[e][c * 8 + sb];
        slot[m * C + l0 + threadIdx.x] = sum;
      }
      if (l0 == 0 && threadIdx.x == 32) {
        float sum = 0.f;
        for (int c = 0; c < 32; ++c) sum += s_red[4][c * 8];
        slot[M * C + m] = sum;
      }
      __syncthreads();
    }
    if (dg_absmax) {
      for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
      if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<unsigned int*>(dg_absmax + m), __float_as_uint(amax));
    }
  }
}

static int head_grid(long long cells) {
  long long b = (cells + 31) / 32;
  const long long cap = (long long)device_sm_count() * 8;
  return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Everything the kernels dereference without a bounds check, refused on the host before any CUDA call: w and each g[m] are read
// and each dg[m] written as float4, so all must be 16-byte aligned; every g[m] is read; a dg[m] may be null (no gradient).
int head_check(const char* what, const float* const* g, const float* w, float* const* dg, int C, int M) {
  MPGCN_CHECK(M >= 1 && M <= kMaxBranches, "%s: %d branches unsupported (1..%d)", what, M, kMaxBranches);
  MPGCN_CHECK(C >= 4 && C % 4 == 0, "%s: C=%d must be a multiple of 4", what, C);
  MPGCN_CHECK(aligned16(w), "%s: w must be 16-byte aligned", what);
  for (int m = 0; m < M; ++m) {
    MPGCN_CHECK(g[m] != nullptr, "%s: branch %d input is a null pointer", what, m);
    MPGCN_CHECK(aligned16(g[m]), "%s: branch %d input must be 16-byte aligned", what, m);
    MPGCN_CHECK(dg == nullptr || aligned16(dg[m]), "%s: branch %d gradient must be 16-byte aligned", what, m);
  }
  return 0;
}

// head_forward / head_backward: arguments already passed head_check (api.cu)
int head_forward(const float* const* g, const float* w, const float* bias, float* y, float* pre, long long cells, int C, int M,
                 cudaStream_t st) {
  HeadPtrs p{};
  for (int m = 0; m < M; ++m) p.g[m] = g[m];
  prof_count(PROF_ELEMENTWISE);
  switch (M) {
    case 1: head_fwd_kernel<1><<<head_grid(cells), 256, 0, st>>>(p, w, bias, y, pre, cells, C, M); break;
    case 2: head_fwd_kernel<2><<<head_grid(cells), 256, 0, st>>>(p, w, bias, y, pre, cells, C, M); break;
    case 3: head_fwd_kernel<3><<<head_grid(cells), 256, 0, st>>>(p, w, bias, y, pre, cells, C, M); break;
    case 4: head_fwd_kernel<4><<<head_grid(cells), 256, 0, st>>>(p, w, bias, y, pre, cells, C, M); break;
    default: head_fwd_kernel<0><<<head_grid(cells), 256, 0, st>>>(p, w, bias, y, pre, cells, C, M); break;
  }
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

size_t head_bwd_slot_bytes(long long cells, int C, int M) { return align_up((size_t)head_grid(cells) * M * (C + 1) * sizeof(float), 256); }

int head_backward(const float* const* g, const float* w, const float* pre, const float* dy, float* const* dg, float* dw, float* db,
                  float* dg_absmax, long long cells, int C, int M, cudaStream_t st, float* slots) {
  HeadPtrs p{};
  for (int m = 0; m < M; ++m) {
    p.g[m] = g[m];
    p.dg[m] = dg ? dg[m] : nullptr;
  }
  if (slots) {
    if (dg_absmax) MPGCN_CUDA(cudaMemsetAsync(dg_absmax, 0, sizeof(float) * M, st));
    const int grid = head_grid(cells);
    prof_count(PROF_ELEMENTWISE);
    switch (M) {
      case 1: head_bwd_det_kernel<1><<<grid, 256, 0, st>>>(p, w, pre, dy, slots, dg_absmax, cells, C, M); break;
      case 2: head_bwd_det_kernel<2><<<grid, 256, 0, st>>>(p, w, pre, dy, slots, dg_absmax, cells, C, M); break;
      case 3: head_bwd_det_kernel<3><<<grid, 256, 0, st>>>(p, w, pre, dy, slots, dg_absmax, cells, C, M); break;
      case 4: head_bwd_det_kernel<4><<<grid, 256, 0, st>>>(p, w, pre, dy, slots, dg_absmax, cells, C, M); break;
      default: head_bwd_det_kernel<0><<<grid, 256, 0, st>>>(p, w, pre, dy, slots, dg_absmax, cells, C, M); break;
    }
    MPGCN_CUDA(cudaGetLastError());
    return reduce_slots(slots, grid, (long long)M * (C + 1), 1, 0, slot_image(dw, (long long)M * C, db, M), st);
  }
  MPGCN_CUDA(cudaMemsetAsync(dw, 0, sizeof(float) * M * C, st));
  MPGCN_CUDA(cudaMemsetAsync(db, 0, sizeof(float) * M, st));
  if (dg_absmax) MPGCN_CUDA(cudaMemsetAsync(dg_absmax, 0, sizeof(float) * M, st));
  prof_count(PROF_ELEMENTWISE);
  const size_t sm = sizeof(float) * M * (C + 1);
  switch (M) {
    case 1: head_bwd_kernel<1><<<head_grid(cells), 256, sm, st>>>(p, w, pre, dy, dw, db, dg_absmax, cells, C, M); break;
    case 2: head_bwd_kernel<2><<<head_grid(cells), 256, sm, st>>>(p, w, pre, dy, dw, db, dg_absmax, cells, C, M); break;
    case 3: head_bwd_kernel<3><<<head_grid(cells), 256, sm, st>>>(p, w, pre, dy, dw, db, dg_absmax, cells, C, M); break;
    case 4: head_bwd_kernel<4><<<head_grid(cells), 256, sm, st>>>(p, w, pre, dy, dw, db, dg_absmax, cells, C, M); break;
    default: head_bwd_kernel<0><<<head_grid(cells), 256, sm, st>>>(p, w, pre, dy, dw, db, dg_absmax, cells, C, M); break;
  }
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace mpgcn
