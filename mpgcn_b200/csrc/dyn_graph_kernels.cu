// Dynamic O / D graphs from the OD history = DataInput.construct_dyn_G (reference: /root/reference/Data_Container_OD.py:39-59).
//
// For each slot t of the perceived period P (7 weekdays):   A_t = mean over periods of OD[t + k P]          (:45)
//     O_G[t][i][j] = cosine_distance(A_t[i, :], A_t[j, :])                                                  (:50-52, eq. 6)
//     D_G[t][i][j] = cosine_distance(A_t[:, i], A_t[j, :])    -- column i against ROW j, exactly as the reference
//                                                                 does at :56 (its eq. 7 quirk is kept, not fixed)
// with scipy's cosine distance 1 - u.v / sqrt(u.u v.v), clipped to [0, 2]; a zero vector gives NaN (0/0) as in scipy.
// The reference makes 2 P N^2 Python-level scipy calls (14 M at N = 1000); here it is two batched N x N x N products of the
// row-normalised / column-normalised average on the exact fp32 SGEMM:  O = 1 - R R^T,  D = 1 - C R^T.
#include "kernels.h"

namespace mpgcn {

// avg[t][e] = (1 / periods) * sum_k od[(t + k P)][e]
__global__ void period_mean_kernel(const float* __restrict__ od, float* __restrict__ avg, int P, int periods, size_t NN) {
  const size_t total = (size_t)P * NN;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const float inv = 1.f / (float)periods;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const size_t t = i / NN, e = i - t * NN;
    float s = 0.f;
    for (int k = 0; k < periods; ++k) s += od[((size_t)k * P + t) * NN + e];
    avg[i] = s * inv;
  }
}

// one warp per (t, i): rn2 = |A_t[i, :]|^2 (coalesced);  COLS: cn2 = |A_t[:, i]|^2 is accumulated by the same pass with atomics
// on a pre-zeroed buffer (each lane owns column j of the row it reads).  Deterministic mode runs COLS = false and col_norms_kernel.
template <bool COLS = true>
__global__ void norms_kernel(const float* __restrict__ avg, float* __restrict__ rn2, float* __restrict__ cn2, int P, int N) {
  const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= (size_t)P * N) return;
  const size_t t = warp / N;
  const float* row = avg + warp * (size_t)N;
  float s = 0.f;
  for (int j = lane; j < N; j += 32) {
    const float v = row[j];
    s = fmaf(v, v, s);
    if (COLS) atomicAdd(&cn2[t * N + j], v * v);
  }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) rn2[warp] = s;
}

// cn2[t][j] = |A_t[:, j]|^2 in row order: one thread per (t, j), consecutive threads read consecutive columns of a row
__global__ void col_norms_kernel(const float* __restrict__ avg, float* __restrict__ cn2, int P, int N) {
  const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= (size_t)P * N) return;
  const size_t t = k / N, j = k % N;
  const float* col = avg + t * (size_t)N * N + j;
  float s = 0.f;
  for (int i = 0; i < N; ++i) {
    const float v = col[(size_t)i * N];
    s += v * v;
  }
  cn2[k] = s;
}

// R[t][i][k] = A[i][k] / |A[i,:]| ;  C[t][i][k] = A[k][i] / |A[:,i]|   (32 x 32 smem tile transpose for C)
__global__ void normalize_kernel(const float* __restrict__ avg, const float* __restrict__ rn2, const float* __restrict__ cn2,
                                 float* __restrict__ R, float* __restrict__ Cm, int N) {
  __shared__ float tile[32][33];
  const size_t t = blockIdx.z;
  const float* A = avg + t * (size_t)N * N;
  const int i0 = blockIdx.y * 32, k0 = blockIdx.x * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int i = i0 + r, k = k0 + threadIdx.x;
    float v = 0.f;
    if (i < N && k < N) {
      v = A[(size_t)i * N + k];
      R[t * (size_t)N * N + (size_t)i * N + k] = v / sqrtf(rn2[t * N + i]);
    }
    tile[r][threadIdx.x] = v;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int c = k0 + r, i = i0 + threadIdx.x;      // C row = column index c of A, C column = row index i of A
    if (c < N && i < N) Cm[t * (size_t)N * N + (size_t)c * N + i] = tile[threadIdx.x][r] / sqrtf(cn2[t * N + c]);
  }
}

__global__ void clip02_kernel(float* __restrict__ x, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float v = x[i];
    x[i] = (v != v) ? v : fminf(fmaxf(v, 0.f), 2.f);      // np.clip keeps NaN
  }
}

__global__ void fill_kernel(float* x, float v, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] = v;
}

// workspace: the period mean, the row- and column-normalised planes, the squared row and column norms, and a vector of ones
struct DynGraphLayout { size_t avg, R, Cm, rn2, cn2, ones, total; };
static DynGraphLayout dyn_graph_layout(int P, int N) {
  DynGraphLayout L;
  size_t off = 0;
  const size_t plane = (size_t)P * N * N * sizeof(float), vec = (size_t)P * N * sizeof(float);
  L.avg = take(off, plane, 256);
  L.R = take(off, plane, 256);
  L.Cm = take(off, plane, 256);
  L.rn2 = take(off, vec, 256);
  L.cn2 = take(off, vec, 256);
  L.ones = take(off, (size_t)N * sizeof(float), 256);
  L.total = align_up(off, 256);
  return L;
}
size_t dyn_graph_workspace_bytes(int P, int N) { return dyn_graph_layout(P, N).total; }

static unsigned dg_grid(size_t work, int threads) {
  size_t b = (work + threads - 1) / threads;
  const size_t cap = (size_t)device_sm_count() * 16;
  return (unsigned)(b < cap ? (b < 1 ? 1 : b) : cap);
}

int dyn_graph_build(const float* od_hist, int periods, float* o_g, float* d_g, int P, int N, void* ws, size_t ws_bytes, cudaStream_t st) {
  MPGCN_CHECK(P >= 1 && N >= 1 && periods >= 1, "dyn_graph: bad shape P=%d N=%d periods=%d", P, N, periods);
  const DynGraphLayout L = dyn_graph_layout(P, N);
  MPGCN_CHECK(ws != nullptr && ws_bytes >= L.total, "dyn_graph: workspace too small (%zu < %zu bytes)", ws_bytes, L.total);
  const size_t NN = (size_t)N * N;
  uint8_t* w = static_cast<uint8_t*>(ws);
  float* avg = reinterpret_cast<float*>(w + L.avg);
  float* R = reinterpret_cast<float*>(w + L.R);
  float* Cm = reinterpret_cast<float*>(w + L.Cm);
  float* rn2 = reinterpret_cast<float*>(w + L.rn2);
  float* cn2 = reinterpret_cast<float*>(w + L.cn2);
  float* ones = reinterpret_cast<float*>(w + L.ones);

  prof_count(PROF_ELEMENTWISE);
  period_mean_kernel<<<dg_grid((size_t)P * NN, 256), 256, 0, st>>>(od_hist, avg, P, periods, NN);
  if (det_mode()) {      // column norms in a fixed order: no atomics (DESIGN.md section 11), no extra workspace
    prof_count(PROF_ELEMENTWISE);
    norms_kernel<false><<<(unsigned)(((size_t)P * N * 32 + 255) / 256), 256, 0, st>>>(avg, rn2, cn2, P, N);
    prof_count(PROF_ELEMENTWISE);
    col_norms_kernel<<<(unsigned)(((size_t)P * N + 255) / 256), 256, 0, st>>>(avg, cn2, P, N);
  } else {
    MPGCN_CUDA(cudaMemsetAsync(cn2, 0, (size_t)P * N * sizeof(float), st));
    prof_count(PROF_ELEMENTWISE);
    norms_kernel<true><<<(unsigned)(((size_t)P * N * 32 + 255) / 256), 256, 0, st>>>(avg, rn2, cn2, P, N);
  }
  prof_count(PROF_ELEMENTWISE);
  normalize_kernel<<<dim3((N + 31) / 32, (N + 31) / 32, P), dim3(32, 8), 0, st>>>(avg, rn2, cn2, R, Cm, N);
  fill_kernel<<<(N + 255) / 256, 256, 0, st>>>(ones, 1.f, N);
  MPGCN_CUDA(cudaGetLastError());

  // D(i,j) = 1 - sum_k A(i,k) * R(j,k), batched over the P slots:  A = R -> O graph,  A = C -> D graph
  for (int which = 0; which < 2; ++which) {
    SgemmParams p{};
    p.A = which == 0 ? R : Cm; p.B = R; p.D = which == 0 ? o_g : d_g;
    p.M = N; p.N = N; p.K = N;
    p.a_si = N; p.a_sk = 1; p.b_sk = 1; p.b_sj = N; p.d_si = N;
    p.nseg = 1; p.Z0 = P; p.Z1 = 1; p.Z2 = 1;
    for (int i = 0; i < 3; ++i) { p.a_sz[i] = 0; p.b_sz[i] = 0; p.d_sz[i] = 0; p.c_sz[i] = 0; }
    p.a_sz[0] = p.b_sz[0] = p.d_sz[0] = (long long)NN;
    p.ksplit = 1; p.alpha = -1.f; p.beta = 0.f;
    p.bias = ones; p.bias_mod = N;
    if (int e = simt_sgemm(p, st)) return e;
    prof_count(PROF_ELEMENTWISE);
    clip02_kernel<<<dg_grid((size_t)P * NN, 256), 256, 0, st>>>(p.D, (size_t)P * NN);
  }
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace mpgcn
