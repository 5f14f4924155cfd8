// Per-OD-cell LSTM, last hidden state only (forward + BPTT backward).
//
// Reference semantics: nn.LSTM(input_size=1, hidden_size=C, num_layers=1, batch_first=True)
// applied to B*N*N independent sequences with a zero initial state, of which the model
// only uses lstm_out[:, -1, :]  (/root/reference/MPGCN.py:69, 80-87, 100-104).  Gate order
// i, f, g, o (PyTorch).  The kernels read x_seq in its native [B, T, N, N, 1] layout
// (coalesced over the cell index), never materialise the zero (h0, c0) tensors nor the
// [B*N*N, T, C] output sequence, and write only h_T.
//
// v1: fp32 CUDA-core kernels.  One block works on a tile of CELLS cells with one thread
// per (cell, hidden unit); W_hh lives transposed in shared memory.  Backward recomputes the
// forward pass of the tile into shared memory (gates, c, h per step) and then walks back in
// time, accumulating weight gradients in shared memory and flushing them once per block.
#include "kernels.h"

namespace mpgcn {

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + __expf(-x)); }
__device__ __forceinline__ float tanhf_(float x) {
  // 2*sigmoid(2x) - 1 with exp computed in fp32; abs error ~1e-7
  const float e = __expf(-2.f * fabsf(x));
  const float t = (1.f - e) / (1.f + e);
  return copysignf(t, x);
}

// x_seq element for cell `cell` (global index over B*NN) at step t
__device__ __forceinline__ size_t x_index(long long cell, int t, int T, long long NN) {
  const long long b = cell / NN;
  const long long r = cell - b * NN;
  return (size_t)((b * T + t) * NN + r);
}

// ---------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------
__global__ void lstm_fwd_kernel(const float* __restrict__ x_seq, const float* __restrict__ w_ih, const float* __restrict__ w_hh,
                                const float* __restrict__ b_ih, const float* __restrict__ b_hh, float* __restrict__ hT,
                                long long cells, int T, long long NN, int C, int CELLS) {
  extern __shared__ float sm[];
  float* Wt = sm;                       // [C][4C]   Wt[k][j] = w_hh[j][k]
  float* bias = Wt + (size_t)C * 4 * C; // [4C]      b_ih + b_hh
  float* wih = bias + 4 * C;            // [4C]
  float* hbuf = wih + 4 * C;            // [2][CELLS][C]

  const int tid = threadIdx.x;
  for (int e = tid; e < 4 * C * C; e += blockDim.x) {
    const int j = e / C, k = e % C;
    Wt[(size_t)k * 4 * C + j] = w_hh[e];
  }
  for (int j = tid; j < 4 * C; j += blockDim.x) {
    bias[j] = b_ih[j] + b_hh[j];
    wih[j] = w_ih[j];
  }
  __syncthreads();

  const int s = tid / C, u = tid % C;
  const long long tiles = (cells + CELLS - 1) / CELLS;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long cell = tile * CELLS + s;
    const bool live = cell < cells;
    float c_state = 0.f;
    hbuf[(size_t)s * C + u] = 0.f;
    __syncthreads();
    int cur = 0;
    for (int t = 0; t < T; ++t) {
      const float xv = live ? x_seq[x_index(cell, t, T, NN)] : 0.f;
      float ai = fmaf(wih[u], xv, bias[u]);
      float af = fmaf(wih[C + u], xv, bias[C + u]);
      float ag = fmaf(wih[2 * C + u], xv, bias[2 * C + u]);
      float ao = fmaf(wih[3 * C + u], xv, bias[3 * C + u]);
      const float* hrow = hbuf + ((size_t)cur * CELLS + s) * C;
      for (int k = 0; k < C; ++k) {
        const float hk = hrow[k];
        const float* w = Wt + (size_t)k * 4 * C;
        ai = fmaf(w[u], hk, ai);
        af = fmaf(w[C + u], hk, af);
        ag = fmaf(w[2 * C + u], hk, ag);
        ao = fmaf(w[3 * C + u], hk, ao);
      }
      const float ig = sigmoidf_(ai), fg = sigmoidf_(af), gg = tanhf_(ag), og = sigmoidf_(ao);
      c_state = fmaf(fg, c_state, ig * gg);
      const float h = og * tanhf_(c_state);
      hbuf[((size_t)(cur ^ 1) * CELLS + s) * C + u] = h;
      cur ^= 1;
      __syncthreads();
    }
    if (live) hT[(size_t)cell * C + u] = hbuf[((size_t)cur * CELLS + s) * C + u];
    __syncthreads();
  }
}

int lstm_last_forward(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, float* hT,
                      int B, int T, long long NN, int C, cudaStream_t st) {
  MPGCN_CHECK(B > 0 && T > 0 && NN > 0, "lstm: empty input");
  MPGCN_CHECK(C >= 1 && C <= 128, "lstm: hidden size %d unsupported (1..128)", C);
  const long long cells = (long long)B * NN;
  int CELLS = 256 / C;
  if (CELLS < 1) CELLS = 1;
  if (CELLS > 32) CELLS = 32;
  const int threads = CELLS * C;
  const size_t smem = ((size_t)4 * C * C + 8 * C + 2 * (size_t)CELLS * C) * sizeof(float);
  static DynSmemAttr attr = {};
  if (smem > 48 * 1024) { if (int e = ensure_dyn_smem(lstm_fwd_kernel, (int)smem, attr)) return e; }
  const long long tiles = (cells + CELLS - 1) / CELLS;
  long long grid = (long long)device_sm_count() * 8;
  if (grid > tiles) grid = tiles;
  prof_begin(PROF_LSTM_FWD, 8.0 * C * (C + 1) * (double)cells * T, st);
  lstm_fwd_kernel<<<(unsigned)grid, threads, smem, st>>>(x_seq, w_ih, w_hh, b_ih, b_hh, hT, cells, T, NN, C, CELLS);
  prof_end(st);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------
// backward (BPTT with in-kernel recomputation)
// ---------------------------------------------------------------------------------------
// DET (deterministic mode): instead of adding its accumulators to the gradients with atomics, a block stores them, in their shared-
// memory order [4C x C w_hh | 4C w_ih | 4C b], to its slot d_w_hh + blockIdx.x * (4C x C + 8C); reduce_slots adds the blocks in order.
template <bool DET>
__global__ void lstm_bwd_kernel(const float* __restrict__ x_seq, const float* __restrict__ w_ih, const float* __restrict__ w_hh,
                                const float* __restrict__ b_ih, const float* __restrict__ b_hh, const float* __restrict__ d_hT,
                                float* __restrict__ d_w_ih, float* __restrict__ d_w_hh, float* __restrict__ d_b, float* __restrict__ d_x,
                                long long cells, int T, long long NN, int C, int CELLS) {
  extern __shared__ float sm[];
  const int G = 4 * C;
  float* Wt = sm;                               // [C][4C] transposed w_hh (forward recompute)
  float* Wn = Wt + (size_t)C * G;               // [4C][C] natural w_hh (dh = da * W)
  float* bias = Wn + (size_t)G * C;             // [4C]
  float* wih = bias + G;                        // [4C]
  float* acc_whh = wih + G;                     // [4C][C] gradient accumulators
  float* acc_wih = acc_whh + (size_t)G * C;     // [4C]
  float* acc_b = acc_wih + G;                   // [4C]
  float* xs = acc_b + G;                        // [T][CELLS]
  float* da = xs + (size_t)T * CELLS;           // [CELLS][4C]
  float* dh = da + (size_t)CELLS * G;           // [CELLS][C]
  float* stash = dh + (size_t)CELLS * C;        // [T][CELLS][6C]: i f g o c h

  const int tid = threadIdx.x;
  const int nthr = blockDim.x;
  for (int e = tid; e < G * C; e += nthr) {
    const int j = e / C, k = e % C;
    const float w = w_hh[e];
    Wn[e] = w;
    Wt[(size_t)k * G + j] = w;
    acc_whh[e] = 0.f;
  }
  for (int j = tid; j < G; j += nthr) {
    bias[j] = b_ih[j] + b_hh[j];
    wih[j] = w_ih[j];
    acc_wih[j] = 0.f;
    acc_b[j] = 0.f;
  }
  __syncthreads();

  const int s = tid / C, u = tid % C;
  const long long tiles = (cells + CELLS - 1) / CELLS;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long cell = tile * CELLS + s;
    const bool live = cell < cells;
    // ---- recompute forward, stash gates / c / h per step ----
    float c_state = 0.f;
    for (int t = 0; t < T; ++t) {
      const float xv = live ? x_seq[x_index(cell, t, T, NN)] : 0.f;
      if (u == 0) xs[(size_t)t * CELLS + s] = xv;
      float ai = fmaf(wih[u], xv, bias[u]);
      float af = fmaf(wih[C + u], xv, bias[C + u]);
      float ag = fmaf(wih[2 * C + u], xv, bias[2 * C + u]);
      float ao = fmaf(wih[3 * C + u], xv, bias[3 * C + u]);
      if (t > 0) {
        const float* hrow = stash + (((size_t)(t - 1) * CELLS + s) * 6 + 5) * C;
        for (int k = 0; k < C; ++k) {
          const float hk = hrow[k];
          const float* w = Wt + (size_t)k * G;
          ai = fmaf(w[u], hk, ai);
          af = fmaf(w[C + u], hk, af);
          ag = fmaf(w[2 * C + u], hk, ag);
          ao = fmaf(w[3 * C + u], hk, ao);
        }
      }
      const float ig = sigmoidf_(ai), fg = sigmoidf_(af), gg = tanhf_(ag), og = sigmoidf_(ao);
      c_state = fmaf(fg, c_state, ig * gg);
      const float h = og * tanhf_(c_state);
      float* st = stash + ((size_t)t * CELLS + s) * 6 * C;
      st[0 * C + u] = ig;
      st[1 * C + u] = fg;
      st[2 * C + u] = gg;
      st[3 * C + u] = og;
      st[4 * C + u] = c_state;
      st[5 * C + u] = h;
      __syncthreads();
    }
    // ---- backward through time ----
    dh[(size_t)s * C + u] = live ? d_hT[(size_t)cell * C + u] : 0.f;
    float dc = 0.f;
    __syncthreads();
    for (int t = T - 1; t >= 0; --t) {
      const float* st = stash + ((size_t)t * CELLS + s) * 6 * C;
      const float ig = st[u], fg = st[C + u], gg = st[2 * C + u], og = st[3 * C + u];
      const float c_t = st[4 * C + u];
      const float c_prev = (t > 0) ? stash[(((size_t)(t - 1) * CELLS + s) * 6 + 4) * C + u] : 0.f;
      const float tc = tanhf_(c_t);
      const float dhv = dh[(size_t)s * C + u];
      const float d_o = dhv * tc;
      dc = fmaf(dhv * og, 1.f - tc * tc, dc);
      const float d_i = dc * gg, d_f = dc * c_prev, d_g = dc * ig;
      float* dar = da + (size_t)s * G;
      dar[u] = d_i * ig * (1.f - ig);
      dar[C + u] = d_f * fg * (1.f - fg);
      dar[2 * C + u] = d_g * (1.f - gg * gg);
      dar[3 * C + u] = d_o * og * (1.f - og);
      dc *= fg;
      __syncthreads();
      // dh_{t-1}[s][u] = sum_j da[s][j] * w_hh[j][u]
      float acc = 0.f;
      for (int j = 0; j < G; ++j) acc = fmaf(dar[j], Wn[(size_t)j * C + u], acc);
      // weight-gradient accumulators owned by this thread
      for (int e = tid; e < G * C; e += nthr) {
        const int j = e / C, k = e % C;
        float sum = 0.f;
        if (t > 0) {
          for (int ss = 0; ss < CELLS; ++ss)
            sum = fmaf(da[(size_t)ss * G + j], stash[(((size_t)(t - 1) * CELLS + ss) * 6 + 5) * C + k], sum);
        }
        acc_whh[e] += sum;
      }
      for (int j = tid; j < G; j += nthr) {
        float sb = 0.f, sx = 0.f;
        for (int ss = 0; ss < CELLS; ++ss) {
          const float d = da[(size_t)ss * G + j];
          sb += d;
          sx = fmaf(d, xs[(size_t)t * CELLS + ss], sx);
        }
        acc_b[j] += sb;
        acc_wih[j] += sx;
      }
      if (d_x != nullptr && u == 0 && live) {
        float sx = 0.f;
        for (int j = 0; j < G; ++j) sx = fmaf(dar[j], wih[j], sx);
        d_x[x_index(cell, t, T, NN)] = sx;
      }
      __syncthreads();
      dh[(size_t)s * C + u] = acc;
      __syncthreads();
    }
  }
  if constexpr (DET) {
    __syncthreads();
    float* slot = d_w_hh + (size_t)blockIdx.x * (G * C + 2 * G);
    for (int e = tid; e < G * C + 2 * G; e += nthr) slot[e] = acc_whh[e];
  } else {
    for (int e = tid; e < G * C; e += nthr) atomicAdd(&d_w_hh[e], acc_whh[e]);
    for (int j = tid; j < G; j += nthr) {
      atomicAdd(&d_w_ih[j], acc_wih[j]);
      atomicAdd(&d_b[j], acc_b[j]);
    }
  }
}

__global__ void copy_kernel(const float* src, float* dst, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[i];
}
int lstm_copy_bias_grad(const float* d_b_ih, float* d_b_hh, int n, cudaStream_t st) {
  prof_count(PROF_ELEMENTWISE);
  copy_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_b_ih, d_b_hh, n);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

static constexpr size_t kBwdSmemBudget = 220 * 1024;

// shared memory of lstm_bwd_kernel: weights and their gradient accumulators, then per cell T*(6C + 1) stash/x + 4C da + C dh
static size_t lstm_bwd_fixed_bytes(int C) { return ((size_t)3 * 4 * C * C + 4 * 4 * (size_t)C) * sizeof(float); }
static size_t lstm_bwd_per_cell_bytes(int T, int C) { return ((size_t)T * (6 * C + 1) + 5 * (size_t)C) * sizeof(float); }

int lstm_bwd_cells_per_block(int T, int C) {
  if (T < 1 || C < 1 || C > 64) return 0;
  const size_t fixed = lstm_bwd_fixed_bytes(C);
  if (fixed >= kBwdSmemBudget) return 0;
  const size_t cells = (kBwdSmemBudget - fixed) / lstm_bwd_per_cell_bytes(T, C);
  const size_t cap = 1024 / C < 16 ? 1024 / C : 16;
  return (int)(cells < cap ? cells : cap);
}

// workspace of the backward: 256 bytes it does not use (the size it has always had), then deterministic mode's slots: one
// [4C x C | 4C | 4C] partial per block (<= SMs blocks), empty with the mode off or at a hidden size the backward does not run
struct LstmBwdLayout { size_t slots, total; };
static LstmBwdLayout lstm_bwd_layout(int C) {
  LstmBwdLayout L;
  size_t off = 256;
  L.slots = take(off, det_mode() && C >= 1 && C <= 64 ? (size_t)device_sm_count() * (4 * C * C + 8 * C) * sizeof(float) : 0, 256);
  L.total = align_up(off, 256);
  return L;
}
size_t lstm_bwd_workspace_bytes(int C) { return lstm_bwd_layout(C).total; }

int lstm_last_backward(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                       const float* d_hT, float* d_w_ih, float* d_w_hh, float* d_b_ih, float* d_b_hh, float* d_x, int B, int T,
                       long long NN, int C, void* ws, size_t ws_bytes, cudaStream_t st) {
  MPGCN_CHECK(B > 0 && T > 0 && NN > 0, "lstm: empty input");
  MPGCN_CHECK(C >= 1 && C <= 64, "lstm backward: hidden size %d unsupported (1..64)", C);
  const LstmBwdLayout L = lstm_bwd_layout(C);
  MPGCN_CHECK(ws != nullptr && ws_bytes >= L.total, "lstm backward: workspace too small (%zu < %zu)", ws_bytes, L.total);
  float* slots = det_mode() ? reinterpret_cast<float*>(static_cast<uint8_t*>(ws) + L.slots) : nullptr;   // fixed-order flush
  MPGCN_CHECK(!slots || (reinterpret_cast<uintptr_t>(ws) & 255) == 0, "lstm backward: workspace must be 256-byte aligned");
  const long long cells = (long long)B * NN;
  const int G = 4 * C;
  const int CELLS = lstm_bwd_cells_per_block(T, C);
  MPGCN_CHECK(CELLS >= 1, "lstm backward: sequence length %d too long for the shared-memory stash", T);
  const int threads = CELLS * C;
  const size_t smem = lstm_bwd_fixed_bytes(C) + (size_t)CELLS * lstm_bwd_per_cell_bytes(T, C);
  static DynSmemAttr attr = {}, attr_det = {};
  if (slots) {
    if (int e = ensure_dyn_smem(lstm_bwd_kernel<true>, (int)(kBwdSmemBudget + 4096), attr_det)) return e;
  } else {
    if (int e = ensure_dyn_smem(lstm_bwd_kernel<false>, (int)(kBwdSmemBudget + 4096), attr)) return e;
    MPGCN_CUDA(cudaMemsetAsync(d_w_ih, 0, sizeof(float) * G, st));
    MPGCN_CUDA(cudaMemsetAsync(d_w_hh, 0, sizeof(float) * G * C, st));
    MPGCN_CUDA(cudaMemsetAsync(d_b_ih, 0, sizeof(float) * G, st));
  }
  const long long tiles = (cells + CELLS - 1) / CELLS;
  long long grid = device_sm_count();
  if (grid > tiles) grid = tiles;
  prof_begin(PROF_LSTM_BWD, 16.0 * C * (C + 1) * (double)cells * T, st);
  if (slots)
    lstm_bwd_kernel<true><<<(unsigned)grid, threads, smem, st>>>(x_seq, w_ih, w_hh, b_ih, b_hh, d_hT, nullptr, slots, nullptr, d_x, cells, T,
                                                                 NN, C, CELLS);
  else
    lstm_bwd_kernel<false><<<(unsigned)grid, threads, smem, st>>>(x_seq, w_ih, w_hh, b_ih, b_hh, d_hT, d_w_ih, d_w_hh, d_b_ih, d_x, cells, T,
                                                                  NN, C, CELLS);
  prof_end(st);
  MPGCN_CUDA(cudaGetLastError());
  if (slots)
    if (int e = reduce_slots(slots, (int)grid, (long long)G * C + 2 * G, 1, 0, slot_image(d_w_hh, (long long)G * C, d_w_ih, G, d_b_ih, G), st))
      return e;
  return lstm_copy_bias_grad(d_b_ih, d_b_hh, G, st);
}

}  // namespace mpgcn
