// Per-OD-cell LSTM on tensor cores at hidden sizes H = 32 CH (CH = 1, 3, 4: H = 32, 96, 128), forward and BPTT backward.
//
// Reference semantics: nn.LSTM(1, H, 1, batch_first=True) over B*N*N independent cells with zero initial state, last hidden
// state only (reference MPGCN.py: LSTM branch of MPGCN.forward); gate order i,f,g,o.
//
// One kernel family with three instances.  What they share is written once below: the tile geometry (Dims), the gate-weight
// tile (load_wx), the gate GEMM of a step (gate_mma), the cell update (cell_update), the cell gradient (cell_grad) and the
// saved-state layout (save_off).  A warp owns 16 cells x one 32-unit slice of all four gates; a tile is CG such 16-cell groups
// of CH warps each.  The gate GEMM of a step, affine part and ex2 scaling included, is [16 cells x (H + 16)] . [(H + 16) x 128
// gate columns] of warp-level mma.sync m16n8k16 (fp16 operands, fp32 accumulators) whose accumulator is the exponent argument
// of the activation.  In the m16n8 accumulator fragment a thread holds, for two cells, the same 8 hidden units of all four
// gates, so the whole cell update is thread-local.  h is rounded to fp16 only as MMA operand; c, the gate arguments and the
// returned h_T stay fp32.  Activations cost 7 SFU operations per hidden unit and step.  The training forward (SAVE) also
// stores c_t, h_t (fp16) of every step; a backward call that comes without that state first re-runs the SAVE forward into its
// workspace.  The instances differ in how h_t and the weight gradient move between warps (details at each kernel):
//   H = 32    lstm_fwd_tc_kernel<SAVE>, lstm_bwd_saved_tc_kernel<DX>.  A warp holds all 4H gate columns, so the new h_t is
//             already the A fragment of the next step's MMA: the recurrence never leaves registers and a step needs no
//             barrier.  128-cell tiles, 8 warps, 2 CTAs per SM in the forward.  The backward is one reverse walk that keeps
//             dWext [128 x 48] in registers across every step and tile of the CTA and reads W_hh^T from its own shared copy;
//             its warps share only the dWext operands, through a ring of shared tiles guarded by mbarriers.
//   H = 96,   lstm_fwd_tcw_kernel<CH, SAVE>, lstm_bwd_walk_tcw_kernel<CH>, lstm_dw_tcw_kernel<CH>.  The CH warps of a group
//   H = 128   exchange h_t through shared memory, one named barrier per group and step; one CTA per SM.  dWext fits neither
//             in registers nor in shared memory, so the walk writes its gate gradients to the workspace and a separate pass
//             reduces them.
//
// mma.sync m16n8k16 fragments (lane = 4 g + q): accumulator element (row g + 8 h, column 2 q + e) of an n8 tile is d[2 h + e];
// A element (row g + 8 h, k 2 q + e + 8 kh) is half e of a[h + 2 kh]; B element (k 2 q + e + 8 kh, column g) is half e of b[kh].
// Per thread: cell rows g, g + 8 of the warp's 16 (index h), units u = 32 js + 8 jn + 2 q + e of the warp's slice js (slot
// s = 2 jn + e, jn < 4).
#include "kernels.h"

namespace mpgcn {
namespace lstm_tc {

template <int CH, bool UP = false>
struct Dims {
  // 16-cell groups per tile: 8 at H = 32 (8 warps; h stays in registers, so 2 CTAs fit an SM in the forward), 4 at H = 96 (12
  // warps, <= 168 registers per thread), 3 at H = 128 (12 warps; 16 warps would cap a thread at 128 registers, which the
  // backward walk exceeds)
  static constexpr int CG = CH == 1 ? 8 : CH == 3 ? 4 : 3;
  static constexpr int CELLS = 16 * CG;
  static constexpr int H = 32 * CH;
  static constexpr int G4 = 4 * H;
  // operand row of a cell: h_{t-1} (H) | x columns (16, see load_wx); UP, a stacked layer above the first:
  // h_{t-1} (H) | h^{l-1}_t (H) | bias columns (16)
  static constexpr int KX = (UP ? 2 * H : H) + 16;
  static constexpr int WX_LD = KX + 8;         // padded so that 8 consecutive rows fall in distinct 16-byte bank groups
  static constexpr int HX_LD = KX + 8;         // staged operand rows of the weight-gradient GEMM
  static constexpr int H_LD = H + 8;           // h exchange tile row stride
  static constexpr int DA_LD = G4 + 8;         // da tile row stride
  static constexpr int NW = CG * CH;           // warps per CTA
  static constexpr int THREADS = 32 * NW;
  static constexpr int FWD_CTAS_PER_SM = CH == 1 ? 2 : 1;
  static constexpr int BWD_CTAS_PER_SM = 1;
  static constexpr int TILE_HALVES = CELLS * H * 2;     // saved c_t | h_t per (tile, step)
};

constexpr int WT_LD = 136;      // H = 32 backward: W_hh^T row stride (128 gates + padding)
constexpr float kLn2 = 0.69314718055994531f;

// SFU primitives (2 ulp each); ex2 saturates to 0 / +inf and rcp(inf) = 0, which are the limits the activations need.
__device__ __forceinline__ float ex2_(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// x enters the gate MMA as fp16 hi + lo (exact to ~22 bits for |x| < 65504); both parts saturate instead of overflowing to inf,
// so larger inputs give finite (saturated-gate) results rather than NaN
__device__ __forceinline__ float x_split_hi(float x) { return __half2float(__float2half_rn(fminf(fmaxf(x, -65504.f), 65504.f))); }
__device__ __forceinline__ float x_split_lo(float x, float hi) { return fminf(fmaxf(x - hi, -65504.f), 65504.f); }

// x_seq is [B][T][NN]: element (cell, t) = x_base(cell) + t * NN; the 64-bit division is done once per tile
__device__ __forceinline__ size_t x_base(long long cell, int T, long long NN) {
  const long long b = cell / NN;
  return (size_t)(b * T * NN + (cell - b * NN));
}
__device__ __forceinline__ uint32_t pack2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ uint4 pack8(const float* v) {
  return make_uint4(pack2(v[0], v[1]), pack2(v[2], v[3]), pack2(v[4], v[5]), pack2(v[6], v[7]));
}
__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
  const __half2* h2 = reinterpret_cast<const __half2*>(&v);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 t = __half22float2(h2[e]);
    f[2 * e] = t.x;
    f[2 * e + 1] = t.y;
  }
}

// Wx rows are kept in slice order r = 128 js + 32 gate + u (gate row j = gate H + 32 js + u), so a warp's B operand is one
// contiguous block of 128 rows; at H = 32 the order is the natural one.
template <int CH>
__device__ __forceinline__ int gate_row(int r) { return (r & 127) / 32 * (32 * CH) + 32 * (r >> 7) + (r & 31); }
__device__ __forceinline__ float row_scale(int r) { return ((r & 127) >> 5) == 2 ? -2.8853900817779268f : -1.4426950408889634f; }

// Wx[r][k] = s_j * [ W_hh[j,:] | wih_hi  b_hi  wih_hi  wih_lo  b_lo  0 0 0 | 0 .. ]  (j = gate_row(r), k < H + 16; s_j = -log2 e
// for i, f, o and -2 log2 e for g): with the operand row of a cell  hx_t = [ h_{t-1} (H) | x_hi  1  x_lo  x_hi  1  0 0 0 | 0 .. ]
// the product hx_t . Wx[r] is s_j * (W_hh h_{t-1} + w_ih x_t + b)_j; x, w_ih and b are split into fp16 hi + lo parts, so the
// affine part keeps ~22 bits.
// UP (a stacked layer l > 0, w_ih [4H][H]): Wx[r] = s_j * [ W_hh[j,:] | W_ih[j,:] | b_hi  b_lo  0 .. ] against the operand row
// [ h_{t-1} | h^{l-1}_t | 1  1  0 .. ]: W_ih is a single fp16 like W_hh, since its operand h^{l-1}_t is one too.
template <int CH, bool UP = false>
__device__ void load_wx(__half* sWx, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh) {
  using D = Dims<CH, UP>;
  constexpr int NCH = D::KX / 8;
  for (int e = threadIdx.x; e < D::G4 * NCH; e += blockDim.x) {
    const int r = e / NCH, ch = e % NCH, j = gate_row<CH>(r);
    const float sc = row_scale(r);
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (ch < D::H / 8) {
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = sc * w_hh[(size_t)j * D::H + ch * 8 + i];
    } else if constexpr (UP) {
      if (ch < 2 * D::H / 8) {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = sc * w_ih[(size_t)j * D::H + ch * 8 - D::H + i];
      } else if (ch == 2 * D::H / 8) {
        const float bb = sc * (b_ih[j] + b_hh[j]), b_hi = __half2float(__float2half_rn(bb));
        v[0] = b_hi; v[1] = bb - b_hi;
      }
    } else if (ch == D::H / 8) {
      const float wi = sc * w_ih[j], bb = sc * (b_ih[j] + b_hh[j]);
      const float wi_hi = __half2float(__float2half_rn(wi)), b_hi = __half2float(__float2half_rn(bb));
      v[0] = wi_hi; v[1] = b_hi; v[2] = wi_hi; v[3] = wi - wi_hi; v[4] = bb - b_hi;
    }
    *reinterpret_cast<uint4*>(sWx + r * D::WX_LD + ch * 8) = pack8(v);
  }
}

// the x / 1 columns H + 2 q, H + 1 + 2 q of a cell's operand row (see load_wx)
__device__ __forceinline__ uint32_t x_cols(float x, int q) {
  const float x_hi = x_split_hi(x);
  return q == 0 ? pack2(x_hi, 1.f) : q == 1 ? pack2(x_split_lo(x, x_hi), x_hi) : q == 2 ? pack2(1.f, 0.f) : 0u;
}
// UP: the bias columns 2 H + 2 q, 2 H + 1 + 2 q
__device__ __forceinline__ uint32_t bias_cols(int q) { return q == 0 ? pack2(1.f, 1.f) : 0u; }

// acc[nt] (nt = gate * 4 + jn) = hx_t . Wx^T for the warp's 16 cells and 128 gate columns.  a_h(kb, a) supplies the A fragment
// of h-block kb < 2 CH (UP: kb < 4 CH, h^{l-1}_t from kb = 2 CH); xw[h] are the x columns H .. H + 7 of row h (UP: the bias
// columns 2 H .. 2 H + 7), the only nonzero columns of the last k-block, which therefore runs as m16n8k8 (its upper 8 columns
// would add exact zeros).  wx_addr: first of the warp's 128 Wx rows.
template <int CH, bool UP = false, class AH>
__device__ __forceinline__ void gate_mma(float (&acc)[16][4], AH&& a_h, const uint32_t (&xw)[2], uint32_t wx_addr) {
  using D = Dims<CH, UP>;
  const int lane = threadIdx.x & 31, mi = lane >> 3;
#pragma unroll
  for (int nt = 0; nt < 16; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
#pragma unroll
  for (int kb = 0; kb < (D::KX - 16) / 16; ++kb) {
    uint32_t a[4];
    a_h(kb, a);
#pragma unroll
    for (int pr = 0; pr < 8; ++pr) {
      uint32_t b0, b1, b2, b3;
      ldmatrix_x4(wx_addr + (uint32_t)(((16 * pr + 8 * (mi >> 1) + (lane & 7)) * D::WX_LD + 16 * kb + 8 * (mi & 1)) * 2), b0, b1, b2, b3);
      mma_16816(acc[2 * pr], a, b0, b1);
      mma_16816(acc[2 * pr + 1], a, b2, b3);
    }
  }
#pragma unroll
  for (int pr = 0; pr < 8; ++pr) {   // x columns: the k-half H .. H + 7 of n8 tiles 2 pr, 2 pr + 1
    uint32_t b0, b1;
    ldmatrix_x2(wx_addr + (uint32_t)(((16 * pr + 8 * (mi & 1) + (lane & 7)) * D::WX_LD + D::KX - 16) * 2), b0, b1);
    mma_1688(acc[2 * pr], xw[0], xw[1], b0);
    mma_1688(acc[2 * pr + 1], xw[0], xw[1], b1);
  }
}

// One step of the thread's 2 x 8 units: c (c_{t-1} -> c_t) in place and h_t into hv, from the gate accumulators.
// Seven SFU operations per hidden unit (5 ex2 + 2 rcp): i, g, f share one reciprocal of the product of their three (1 + 2^arg)
// terms, o and tanh(c) share another.  The accumulators are -log2e * pre (i, f, o) and -2 log2e * pre (g); arguments are
// clamped from above at 40 (ex2(-big) = 0 is fine), so a triple product stays below 1.4e36; the clamp moves sigmoid / tanh by
// < 1e-12.
__device__ __forceinline__ void cell_update(const float (&acc)[16][4], float (&c)[2][8], float (&hv)[2][8]) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int s = 0; s < 8; ++s) {
      const int jn = s >> 1, k = 2 * h + (s & 1);
      const float ai = 1.f + ex2_(fminf(acc[jn][k], 40.f));
      const float af = 1.f + ex2_(fminf(acc[4 + jn][k], 40.f));
      const float ag = 1.f + ex2_(fminf(acc[8 + jn][k], 40.f));
      const float p = 1.f + ex2_(fminf(acc[12 + jn][k], 40.f));
      const float pig = ai * ag;
      const float r = rcp_(pig * af);
      const float gi = r * (ag * af);                    // sigmoid(i)
      const float gg = fmaf(r + r, ai * af, -1.f);       // tanh(g)
      const float gf = r * pig;                          // sigmoid(f)
      c[h][s] = fmaf(gf, c[h][s], gi * gg);
      const float ac = 1.f + ex2_(fminf(-2.8853900817779268f * c[h][s], 40.f));
      const float r2 = rcp_(p * ac);
      hv[h][s] = (r2 * ac) * fmaf(r2 + r2, p, -1.f);     // sigmoid(o) * tanh(c)
    }
  }
}

// The gate gradients of cell row h at one step of the reverse walk, from the gate accumulators recomputed from the saved
// h_{t-1}, the saved c_t, c_{t-1} (vc, vcp) and the incoming dh, dc of the row's 8 units (dc becomes dc_{t-1} in place):
// d[gate][s] for gates i, f, g, o.  With DX, returns the thread's part of the row's dx = sum over its units u of
// d[.][s] w_ih[. H + u] (s_wih: w_ih by gate row; js: the warp's unit slice); without, 0.  The 7 SFU operations of cell_update.
template <int CH, bool DX>
__device__ __forceinline__ float cell_grad(const float (&acc)[16][4], int h, const uint4& vc, const uint4& vcp, const float (&dh)[8],
                                           float (&dc)[8], const float* s_wih, int js, int q, float (&d)[4][8]) {
  constexpr int H = Dims<CH>::H;
  float fc[8], fcp[8];
  unpack8(vc, fc);
  unpack8(vcp, fcp);
  float dx = 0.f;
#pragma unroll
  for (int s = 0; s < 8; ++s) {
    const int jn = s >> 1, k = 2 * h + (s & 1);
    const float ai = 1.f + ex2_(fminf(acc[jn][k], 40.f));
    const float af = 1.f + ex2_(fminf(acc[4 + jn][k], 40.f));
    const float ag = 1.f + ex2_(fminf(acc[8 + jn][k], 40.f));
    const float ao = 1.f + ex2_(fminf(acc[12 + jn][k], 40.f));
    const float ac = 1.f + ex2_(fminf(-2.8853900817779268f * fc[s], 40.f));
    const float pig = ai * ag;
    const float r1 = rcp_(pig * af), r2 = rcp_(ao * ac);
    const float gi = r1 * (ag * af), gg = fmaf(r1 + r1, ai * af, -1.f), gf = r1 * pig;
    const float go = r2 * ac, tcv = fmaf(r2 + r2, ao, -1.f);
    const float dhv = dh[s];
    const float dcv = fmaf(dhv * go, fmaf(-tcv, tcv, 1.f), dc[s]);
    d[3][s] = (dhv * tcv) * fmaf(-go, go, go);
    d[0][s] = (dcv * gg) * fmaf(-gi, gi, gi);
    d[1][s] = (dcv * fcp[s]) * fmaf(-gf, gf, gf);
    d[2][s] = (dcv * gi) * fmaf(-gg, gg, 1.f);
    dc[s] = dcv * gf;
    if (DX) {
      const int u = 32 * js + 8 * jn + 2 * q + (s & 1);
      dx += d[0][s] * s_wih[u] + d[1][s] * s_wih[H + u] + d[2][s] * s_wih[2 * H + u] + d[3][s] * s_wih[3 * H + u];
    }
  }
  return dx;
}

// Every kernel runs the tiles tile0 .. tile0 + tiles - 1 of the `cells` cells.  x_seq, h_T, d_hT and d_x are addressed by the
// global cell, (tile0 + tile) CELLS + ..; the training state, the da records, h_seq and d_seq by the tile within the range, so a
// range's region of them has the layout the full-size buffer has for those tiles (tile0 = 0 and all tiles: the whole call).
// Training state written by the forward kernels and read by the backward ones: per (tile, step) NW x 1024 halves,
// [warp][c | h][lane][16 halves], the 16 halves of a thread in slot order h * 8 + s (its register fragment, stored as is);
// warp = cg CH + js.
template <int CH>
__device__ __forceinline__ size_t save_off(long long tile, int T, int t, int warp, int kind, int lane) {
  return ((size_t)tile * T + t) * Dims<CH>::TILE_HALVES + (size_t)warp * 1024 + (size_t)kind * 512 + (size_t)lane * 16;
}

// A stacked layer reads the h_t of the layer below from a sequence whose warp blocks lie `ld` halves apart: the training state
// (base saved + 512, ld 1024: the h half of save_off) or the h-only sequence an inference forward hands up (ld 512).  The tiles
// of every layer of one width are the same, so a lane's fragment there is its own A fragment.
template <int CH>
__device__ __forceinline__ size_t h_off(long long tile, int T, int t, int warp, int lane, int ld) {
  return (((size_t)tile * T + t) * Dims<CH>::NW + warp) * (size_t)ld + (size_t)lane * 16;
}
// A fragment of h k-block kb < 2 CH of a 16-cell group from its first warp's fragment hp: slice kb / 2 is the same lane's
// fragment of warp kb / 2 of the group; k-block kb = 2 sl + kk takes its words (h, 2 kk) and (h, 2 kk + 1), i.e. the uint2
// number 2 h + kk of the 16 halves
__device__ __forceinline__ void a_from_seq(const __half* hp, int ld, int kb, uint32_t (&a)[4]) {
  const uint2* p = reinterpret_cast<const uint2*>(hp + (kb >> 1) * ld);
  const uint2 r0 = __ldg(p + (kb & 1)), r1 = __ldg(p + 2 + (kb & 1));
  a[0] = r0.x; a[1] = r1.x; a[2] = r0.y; a[3] = r1.y;
}
// gradient sequence between the walks of a stack, fp32 in the walk's register fragment: per (tile, step, warp, lane) the 16
// values dh[h][s] of the thread (scaled by S); the walk of layer l writes d(h^{l-1}_t) there, the walk of layer l - 1 adds it
template <int CH>
__device__ __forceinline__ size_t dseq_off(long long tile, int T, int t, int warp, int lane) {
  return (((size_t)tile * T + t) * Dims<CH>::NW + warp) * 512 + (size_t)lane * 16;
}

// =======================================================================================
// H = 32
// =======================================================================================
// forward: the thread's h_t, packed to fp16 pairs, is its A fragment of the next step's h k-blocks.
// RANGE: runs the tiles tile0 .. tile0 + tiles - 1; without, every tile of `cells` (tile0 and tiles are not read), which keeps the
// code of the headline's whole-call launches as it was before tile ranges (the same holds for lstm_bwd_saved_tc_kernel)
template <bool SAVE, bool RANGE = false>
__global__ void __launch_bounds__(Dims<1>::THREADS, Dims<1>::FWD_CTAS_PER_SM)
lstm_fwd_tc_kernel(const float* __restrict__ x_seq, const float* __restrict__ w_ih, const float* __restrict__ w_hh,
                   const float* __restrict__ b_ih, const float* __restrict__ b_hh, float* __restrict__ hT, __half* __restrict__ saved,
                   long long cells, long long tile0, long long tiles, int T, long long NN) {
  using D = Dims<1>;
  __shared__ __align__(16) __half sWx[D::G4 * D::WX_LD];
  load_wx<1>(sWx, w_ih, w_hh, b_ih, b_hh);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const uint32_t wx_addr = smem_u32(sWx);
  const long long t0 = RANGE ? tile0 : 0, ntiles = RANGE ? tiles : (cells + D::CELLS - 1) / D::CELLS;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    long long cell[2];
    bool live[2];
    size_t xb[2];
    float xv[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      cell[h] = (t0 + tile) * D::CELLS + warp * 16 + g + 8 * h;
      live[h] = cell[h] < cells;
      xb[h] = live[h] ? x_base(cell[h], T, NN) : 0;
      xv[h] = live[h] ? x_seq[xb[h]] : 0.f;
    }
    float c[2][8], hv[2][8];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int s = 0; s < 8; ++s) { c[h][s] = 0.f; hv[h][s] = 0.f; }
    for (int t = 0; t < T; ++t) {
      uint32_t hw[8], xw[2];          // word h * 4 + jn: units 8 jn + 2 q, +1 of cell row h
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int jn = 0; jn < 4; ++jn) hw[4 * h + jn] = pack2(hv[h][2 * jn], hv[h][2 * jn + 1]);
        xw[h] = x_cols(xv[h], q);
      }
      float acc[16][4];
      gate_mma<1>(acc, [&](int kb, uint32_t (&a)[4]) {
        a[0] = hw[2 * kb]; a[1] = hw[4 + 2 * kb]; a[2] = hw[2 * kb + 1]; a[3] = hw[4 + 2 * kb + 1];
      }, xw, wx_addr);
#pragma unroll
      for (int h = 0; h < 2; ++h) xv[h] = (live[h] && t + 1 < T) ? x_seq[xb[h] + (size_t)(t + 1) * NN] : 0.f;
      cell_update(acc, c, hv);
      if (SAVE) {                     // training: c_t and h_t (fp16) for the backward kernel, see save_off()
        uint4* dc = reinterpret_cast<uint4*>(saved + save_off<1>(tile, T, t, warp, 0, lane));
        uint4* dh = reinterpret_cast<uint4*>(saved + save_off<1>(tile, T, t, warp, 1, lane));
        dc[0] = pack8(c[0]); dc[1] = pack8(c[1]);
        dh[0] = pack8(hv[0]); dh[1] = pack8(hv[1]);
      }
    }
    if (hT != nullptr) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (live[h]) {
#pragma unroll
          for (int jn = 0; jn < 4; ++jn)
            *reinterpret_cast<float2*>(hT + (size_t)cell[h] * D::H + 8 * jn + 2 * q) = make_float2(hv[h][2 * jn], hv[h][2 * jn + 1]);
        }
    }
  }
}

// backward from the forward kernel's saved c_t / h_t (training path)
// One reverse walk, no forward recompute: the gate pre-activations of step t depend only on the SAVED h_{t-1} and on x_t.
// Per step and warp (16 cells), all on mma.sync:
//     gates_t  = hx_t x Wx^T                (as in the forward; A = saved h_{t-1} fragment + x columns)
//     dh_{t-1} = da_t x W_hh                (A = da_t straight from the gate-gradient registers, B = W_hh^T in shared memory)
// and per step over the CTA's 128 cells:
//     dWext   += da_t^T x hx_t              (128 gates x 40 nonzero columns; warp w owns gates 16 w .. 16 w + 15;
//                                            columns 0..31 dW_hh, 32 + 34 dW_ih, 33 db)
// The warps meet only in that last product, so no step waits for the whole CTA.  Its operands go through a ring of kBwdRing
// da / hx tiles in shared memory: a warp waits on the slot's empty barrier, writes its 16 rows, arrives on the full barrier,
// and then takes its product of the PREVIOUS step (waiting for that slot to be full, arriving on its empty barrier once read).
// A warp can so run up to two steps ahead of the slowest, and one warp's product can overlap another's cell gradient.
// The saved state and x of the walk stream in by cp.async, two steps ahead, into a per-warp ring of the same depth: entry k is
// the (tile, t) of the walk's k-th step, a warp's own 2 KB c_t | h_t block of it (each thread copies, and later reads, exactly
// its own 64 bytes, so its cp.async wait is the only synchronisation) and the x_t of the thread's two cells.  Step k reads
// c_{t-1}, h_{t-1} from entry k + 1 and keeps c_{t-1} in registers as the c_t of the next step.
// DX: the instance that also writes d_x (the host picks it from d_x != nullptr).
constexpr int kBwdRing = 3;
constexpr size_t kBwdSavedSmem =
    (size_t)(Dims<1>::G4 * Dims<1>::WX_LD + Dims<1>::H * WT_LD + kBwdRing * Dims<1>::CELLS * (Dims<1>::DA_LD + Dims<1>::HX_LD)) * sizeof(__half) +
    (size_t)kBwdRing * Dims<1>::NW * 2048 +                      // saved-state ring: [slot][warp][c h0, c h1, h h0, h h1][lane] uint4
    (size_t)kBwdRing * Dims<1>::THREADS * 2 * sizeof(float) +    // x ring: [slot][thread][row h]
    Dims<1>::G4 * sizeof(float) + 2 * kBwdRing * sizeof(uint64_t);

// DET (deterministic mode): the flush stores the CTA's dWext to its slot d_w_hh + blockIdx.x * 4352, laid out as the outputs
// [128 x 32 w_hh | 128 w_ih | 128 b] (the two x columns of w_ih added in the CTA first), instead of adding it with atomics; with
// acc it adds to the slot instead (a later chunk of lstm_recompute_backward_tc: the CTA owns the slot, the stream orders the chunks).
template <bool DX, bool DET = false, bool RANGE = false>
__global__ void __launch_bounds__(Dims<1>::THREADS, Dims<1>::BWD_CTAS_PER_SM)
lstm_bwd_saved_tc_kernel(const float* __restrict__ x_seq, const float* __restrict__ w_ih, const float* __restrict__ w_hh,
                         const float* __restrict__ b_ih, const float* __restrict__ b_hh, const float* __restrict__ d_hT,
                         float* __restrict__ d_w_ih, float* __restrict__ d_w_hh, float* __restrict__ d_b, float* __restrict__ d_x,
                         const __half* __restrict__ saved, const float* __restrict__ scale2, long long cells, long long tile0, long long tiles,
                         int T, long long NN, bool acc) {
  using D = Dims<1>;
  constexpr int C = D::H, CELLS = D::CELLS;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __half* sWx = reinterpret_cast<__half*>(smem_raw);       // [128][WX_LD]
  __half* sWT = sWx + D::G4 * D::WX_LD;                    // [32 units][WT_LD]: W_hh^T
  __half* sDA = sWT + C * WT_LD;                           // kBwdRing x [128 cells][DA_LD]
  __half* sHX = sDA + kBwdRing * CELLS * D::DA_LD;         // kBwdRing x [128 cells][HX_LD]
  uint4* sST = reinterpret_cast<uint4*>(sHX + kBwdRing * CELLS * D::HX_LD);
  float* sX = reinterpret_cast<float*>(sST + kBwdRing * D::NW * 128);
  float* s_wih = sX + kBwdRing * D::THREADS * 2;
  uint64_t* full = reinterpret_cast<uint64_t*>(s_wih + D::G4);     // da / hx slot written by all 8 warps
  uint64_t* empty = full + kBwdRing;                               // da / hx slot read by all 8 warps

  load_wx<1>(sWx, w_ih, w_hh, b_ih, b_hh);
  for (int e = threadIdx.x; e < D::G4 * C; e += blockDim.x) {
    const int j = e / C, u = e % C;
    sWT[u * WT_LD + j] = __float2half_rn(w_hh[e]);
  }
  for (int j = threadIdx.x; j < D::G4; j += blockDim.x) s_wih[j] = w_ih[j];
  if (threadIdx.x == 0)
    for (int s = 0; s < kBwdRing; ++s) { mbar_init(&full[s], D::NW); mbar_init(&empty[s], D::NW); }
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3, mi = lane >> 3;
  const uint32_t wx_addr = smem_u32(sWx), wt_addr = smem_u32(sWT), da_addr = smem_u32(sDA), hx_addr = smem_u32(sHX);
  const long long t0 = RANGE ? tile0 : 0, ntiles = RANGE ? tiles : (cells + CELLS - 1) / CELLS;
  const float S = scale2[0], invS = scale2[1];
  float dw[5][4];                     // dWext: gate 16 warp + g + 8 (i >> 1), column 8 nt + 2 q + (i & 1); columns 40..47 are 0
#pragma unroll
  for (int nt = 0; nt < 5; ++nt) dw[nt][0] = dw[nt][1] = dw[nt][2] = dw[nt][3] = 0.f;

  // ---- the saved-state / x stream: entry (pf_tile, pf_t) is fetched next ----
  long long pf_tile = blockIdx.x;
  int pf_t = T - 1;
  size_t pf_xb[2];
  auto pf_cells = [&]() {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long cell = (t0 + pf_tile) * CELLS + warp * 16 + g + 8 * h;
      pf_xb[h] = pf_tile < ntiles && cell < cells ? x_base(cell, T, NN) : ~(size_t)0;
    }
  };
  auto fetch = [&](int slot) {
    if (pf_tile < ntiles) {
      const uint4* pc = reinterpret_cast<const uint4*>(saved + save_off<1>(pf_tile, T, pf_t, warp, 0, lane));
      const uint4* ph = reinterpret_cast<const uint4*>(saved + save_off<1>(pf_tile, T, pf_t, warp, 1, lane));
      uint4* dst = sST + (slot * D::NW + warp) * 128 + lane;
      cp_async16(dst, pc); cp_async16(dst + 32, pc + 1); cp_async16(dst + 64, ph); cp_async16(dst + 96, ph + 1);
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (pf_xb[h] != ~(size_t)0) cp_async4(sX + (slot * D::THREADS + threadIdx.x) * 2 + h, x_seq + pf_xb[h] + (size_t)pf_t * NN);
    }
    cp_async_commit();
    if (--pf_t < 0) { pf_t = T - 1; pf_tile += gridDim.x; pf_cells(); }
  };
  // ---- dWext[16 warp .. +15][0..47] += da^T x hx over the 128 cells of the step held in da / hx slot `slot` ----
  auto dwext = [&](int slot, uint32_t phase) {
    mbar_wait_inline(&full[slot], phase);
    const uint32_t da_b = da_addr + (uint32_t)(slot * CELLS * D::DA_LD * 2), hx_b = hx_addr + (uint32_t)(slot * CELLS * D::HX_LD * 2);
#pragma unroll
    for (int kc = 0; kc < 8; ++kc) {
      uint32_t a[4];
      ldmatrix_x4_trans(da_b + (uint32_t)(((16 * kc + 8 * (mi >> 1) + (lane & 7)) * D::DA_LD + 16 * warp + 8 * (mi & 1)) * 2), a[0], a[1], a[2], a[3]);
#pragma unroll
      for (int pr = 0; pr < 2; ++pr) {
        uint32_t b0, b1, b2, b3;
        ldmatrix_x4_trans(hx_b + (uint32_t)(((16 * kc + 8 * (mi & 1) + (lane & 7)) * D::HX_LD + 16 * pr + 8 * (mi >> 1)) * 2), b0, b1, b2, b3);
        mma_16816(dw[2 * pr], a, b0, b1);
        mma_16816(dw[2 * pr + 1], a, b2, b3);
      }
      uint32_t b0, b1;                // columns 32..39; 40..47 are zero and never flushed
      ldmatrix_x2_trans(hx_b + (uint32_t)(((16 * kc + 8 * (mi & 1) + (lane & 7)) * D::HX_LD + 32) * 2), b0, b1);
      mma_16816(dw[4], a, b0, b1);
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[slot]);
  };

  pf_cells();
  fetch(0);
  fetch(1);
  int slot = 0, prev_slot = 0;        // ring slot of this step (k mod kBwdRing) and of the previous one
  uint32_t phase = 0, prev_phase = 0; // (k / kBwdRing) & 1: the barrier phase of the slot's current use
  bool have_prev = false;

  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    long long cell[2];
    bool live[2];
    size_t xb[2];
    float dh[2][8], dc[2][8];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      cell[h] = (t0 + tile) * CELLS + warp * 16 + g + 8 * h;
      live[h] = cell[h] < cells;
      xb[h] = DX && live[h] ? x_base(cell[h], T, NN) : 0;
#pragma unroll
      for (int s = 0; s < 8; ++s) {
        dh[h][s] = live[h] ? d_hT[(size_t)cell[h] * C + 8 * (s >> 1) + 2 * q + (s & 1)] * S : 0.f;
        dc[h][s] = 0.f;
      }
    }
    uint4 vc[2];                      // c_t: read from the stream at the tile's first step, then carried from c_{t-1}
    for (int t = T - 1; t >= 0; --t) {
      fetch(slot == 0 ? kBwdRing - 1 : slot - 1);   // entry k + 2 into the slot of entry k - 1, last read in the previous step
      cp_async_wait<1>();                           // entries k and k + 1 have landed
      const uint4* st0 = sST + (slot * D::NW + warp) * 128 + lane;
      const uint4* st1 = sST + ((slot + 1 == kBwdRing ? 0 : slot + 1) * D::NW + warp) * 128 + lane;
      if (t == T - 1) { vc[0] = st0[0]; vc[1] = st0[32]; }
      // saved state: c_{t-1}, h_{t-1} (zero before the first step)
      uint4 vcp[2], vhp[2];
      if (t > 0) {
        vcp[0] = st1[0]; vcp[1] = st1[32]; vhp[0] = st1[64]; vhp[1] = st1[96];
      } else {
        vcp[0] = vcp[1] = vhp[0] = vhp[1] = make_uint4(0u, 0u, 0u, 0u);
      }
      const uint32_t hw[8] = {vhp[0].x, vhp[0].y, vhp[0].z, vhp[0].w, vhp[1].x, vhp[1].y, vhp[1].z, vhp[1].w};
      uint32_t xw[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) xw[h] = x_cols(live[h] ? sX[(slot * D::THREADS + threadIdx.x) * 2 + h] : 0.f, q);
      float acc[16][4];
      gate_mma<1>(acc, [&](int kb, uint32_t (&a)[4]) {
        a[0] = hw[2 * kb]; a[1] = hw[4 + 2 * kb]; a[2] = hw[2 * kb + 1]; a[3] = hw[4 + 2 * kb + 1];
      }, xw, wx_addr);

      uint32_t da[16][2];             // fp16 pairs: gate column 8 nt + 2 q, +1 of row h, nt = gate * 4 + jn
      float dx[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float d[4][8];
        dx[h] = cell_grad<1, DX>(acc, h, vc[h], vcp[h], dh[h], dc[h], s_wih, 0, q, d);
#pragma unroll
        for (int jn = 0; jn < 4; ++jn)
#pragma unroll
          for (int gt = 0; gt < 4; ++gt) da[4 * gt + jn][h] = pack2(d[gt][2 * jn], d[gt][2 * jn + 1]);
      }
      if (DX) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float v = dx[h];
          v += __shfl_xor_sync(0xffffffffu, v, 1);
          v += __shfl_xor_sync(0xffffffffu, v, 2);
          if (q == 0 && live[h]) d_x[xb[h] + (size_t)t * NN] = v * invS;
        }
      }
      if (t > 0) {                    // dh_{t-1} = da_t x W_hh
        float adh[4][4];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) adh[nt][0] = adh[nt][1] = adh[nt][2] = adh[nt][3] = 0.f;
#pragma unroll
        for (int kb = 0; kb < 8; ++kb) {
          const uint32_t a[4] = {da[2 * kb][0], da[2 * kb][1], da[2 * kb + 1][0], da[2 * kb + 1][1]};
#pragma unroll
          for (int pr = 0; pr < 2; ++pr) {
            uint32_t b0, b1, b2, b3;
            ldmatrix_x4(wt_addr + (uint32_t)(((16 * pr + 8 * (mi >> 1) + (lane & 7)) * WT_LD + 16 * kb + 8 * (mi & 1)) * 2), b0, b1, b2, b3);
            mma_16816(adh[2 * pr], a, b0, b1);
            mma_16816(adh[2 * pr + 1], a, b2, b3);
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int s = 0; s < 8; ++s) dh[h][s] = adh[s >> 1][2 * h + (s & 1)];
      }
      // da_t and hx_t of the warp's cells into this step's slot, once every warp has read the step that last used it
      mbar_wait_inline(&empty[slot], phase ^ 1u);
      __half* sda = sDA + slot * CELLS * D::DA_LD;
      __half* shx = sHX + slot * CELLS * D::HX_LD;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = warp * 16 + g + 8 * h;
#pragma unroll
        for (int nt = 0; nt < 16; ++nt) *reinterpret_cast<uint32_t*>(sda + row * D::DA_LD + 8 * nt + 2 * q) = da[nt][h];
#pragma unroll
        for (int jn = 0; jn < 4; ++jn) *reinterpret_cast<uint32_t*>(shx + row * D::HX_LD + 8 * jn + 2 * q) = hw[4 * h + jn];
        *reinterpret_cast<uint32_t*>(shx + row * D::HX_LD + 32 + 2 * q) = xw[h];
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&full[slot]);
      if (have_prev) dwext(prev_slot, prev_phase);  // the previous step's product, in step order
      have_prev = true;
      prev_slot = slot;
      prev_phase = phase;
      if (++slot == kBwdRing) { slot = 0; phase ^= 1u; }
      vc[0] = vcp[0];
      vc[1] = vcp[1];
    }
  }
  if (have_prev) dwext(prev_slot, prev_phase);
  // ---- flush the weight-gradient accumulator ----
  if constexpr (DET) {
    float* slot = d_w_hh + (size_t)blockIdx.x * (D::G4 * C + 2 * D::G4);
    auto put = [&](int i, float v) { slot[i] = acc ? slot[i] + v : v; };
#pragma unroll
    for (int nt = 0; nt < 5; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int j = 16 * warp + g + 8 * (i >> 1), col = 8 * nt + 2 * q + (i & 1);
        const float v = dw[nt][i] * invS;
        const float next = __shfl_down_sync(0xffffffffu, v, 1);     // lane q + 1: column col + 2
        if (col < C) put(j * C + col, v);
        else if (col == 32) put(D::G4 * C + j, v + next);            // columns 32 and 34: the x hi / lo pair of w_ih
        else if (col == 33) put(D::G4 * C + D::G4 + j, v);
      }
  } else {
#pragma unroll
    for (int nt = 0; nt < 5; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int j = 16 * warp + g + 8 * (i >> 1), col = 8 * nt + 2 * q + (i & 1);
        const float v = dw[nt][i] * invS;
        if (col < C) atomicAdd(&d_w_hh[j * C + col], v);
        else if (col == 32 || col == 34) atomicAdd(&d_w_ih[j], v);
        else if (col == 33) atomicAdd(&d_b[j], v);
      }
  }
}

// =======================================================================================
// H = 96, 128
// =======================================================================================
// A warp owns one 32-unit slice js of all four gates (128 of the 4H gate columns), and the CH warps of a 16-cell group cg
// exchange h_t through shared memory once per step (one named barrier per group and step).  One CTA per SM: the gate weights
// take 4H x (H + 24) halves of shared memory, 152 KB at H = 128.
// Backward: dWext [4H x (H + 16)] no longer fits a CTA's registers (74 K fp32 at H = 128).  The reverse walk writes the scaled
// fp16 gate gradients of every (tile, step) to the workspace and a separate tensor-core pass reduces dWext = sum da^T hx over
// cells and steps, reading h_{t-1} from the saved state.  The workspace is as large as twice the saved state; tiling the
// reduction inside the walk would need either 74 K fp32 of shared memory or a read-modify-write of a per-CTA fp32 partial every
// step.  dh_{t-1} = da_t W_hh reads W_hh from the same shared Wx block (ldmatrix.trans), since a transposed copy does not fit
// beside it; da_t is divided by the row scale s_j before it is rounded to fp16 and the weight-gradient pass multiplies s_j back.

// ---------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------
template <int CH, bool UP = false>
constexpr size_t kFwdWideSmem = (size_t)(Dims<CH, UP>::G4 * Dims<CH, UP>::WX_LD + 2 * Dims<CH>::CELLS * Dims<CH>::H_LD) * sizeof(__half);

// Layers of a stack (lstm_stack_forward_tc) run this kernel at every width, hidden 32 as CH = 1:
//   UP     the input is h^{l-1}_t of the layer below from h_in (see h_off) instead of x_seq: in training its saved state + 512
//          (ld 1024), in inference its h-only sequence (ld 512);
//   HSEQ   an inference layer below the top also writes h_t of every step to h_seq (h_off, ld 512) for the layer above.
template <int CH, bool SAVE, bool UP = false, bool HSEQ = false>
__global__ void __launch_bounds__(Dims<CH>::THREADS, Dims<CH>::FWD_CTAS_PER_SM)
lstm_fwd_tcw_kernel(const float* __restrict__ x_seq, const float* __restrict__ w_ih, const float* __restrict__ w_hh,
                    const float* __restrict__ b_ih, const float* __restrict__ b_hh, float* __restrict__ hT, __half* __restrict__ saved,
                    long long cells, long long tile0, long long tiles, int T, long long NN, const __half* __restrict__ h_in,
                    __half* __restrict__ h_seq) {
  using D = Dims<CH, UP>;
  constexpr int CELLS = D::CELLS;
  constexpr int IN_LD = SAVE ? 1024 : 512;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __half* sWx = reinterpret_cast<__half*>(smem_raw);       // [G4][WX_LD], slice order
  __half* sH = sWx + D::G4 * D::WX_LD;                     // 2 x [CELLS][H_LD]: h_t of the tile, double-buffered by step
  load_wx<CH, UP>(sWx, w_ih, w_hh, b_ih, b_hh);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const int cg = warp / CH, js = warp % CH;
  const uint32_t wx_addr = smem_u32(sWx + js * 128 * D::WX_LD);
  // this lane's ldmatrix row address in the h tile: row 16 cg + (lane & 15), column 8 (lane >> 4)
  const uint32_t h_addr = smem_u32(sH + (cg * 16 + (lane & 15)) * D::H_LD + 8 * (lane >> 4));
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    long long cell[2];
    bool live[2];
    size_t xb[2];
    float xv[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      cell[h] = (tile0 + tile) * CELLS + cg * 16 + g + 8 * h;
      live[h] = cell[h] < cells;
      xb[h] = !UP && live[h] ? x_base(cell[h], T, NN) : 0;
      xv[h] = !UP && live[h] ? x_seq[xb[h]] : 0.f;
    }
    float c[2][8];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int s = 0; s < 8; ++s) c[h][s] = 0.f;
    for (int t = 0; t < T; ++t) {
      uint32_t xw[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) xw[h] = UP ? bias_cols(q) : x_cols(xv[h], q);
      // h_{t-1} was written to buffer t & 1 before the previous step's barrier; zero before the first step
      const uint32_t hb = h_addr + (uint32_t)((t & 1) * CELLS * D::H_LD * 2);
      const __half* hin = UP ? h_in + h_off<CH>(tile, T, t, cg * CH, lane, IN_LD) : nullptr;
      float acc[16][4];
      gate_mma<CH, UP>(acc, [&](int kb, uint32_t (&a)[4]) {
        if (UP && kb >= 2 * CH) a_from_seq(hin, IN_LD, kb - 2 * CH, a);
        else if (t == 0) { a[0] = a[1] = a[2] = a[3] = 0u; }
        else ldmatrix_x4(hb + 32 * kb, a[0], a[1], a[2], a[3]);
      }, xw, wx_addr);
      if (!UP) {
#pragma unroll
        for (int h = 0; h < 2; ++h) xv[h] = (live[h] && t + 1 < T) ? x_seq[xb[h] + (size_t)(t + 1) * NN] : 0.f;
      }
      float hv[2][8];
      cell_update(acc, c, hv);
      if (SAVE) {
        uint4* dc = reinterpret_cast<uint4*>(saved + save_off<CH>(tile, T, t, warp, 0, lane));
        uint4* dh = reinterpret_cast<uint4*>(saved + save_off<CH>(tile, T, t, warp, 1, lane));
        dc[0] = pack8(c[0]); dc[1] = pack8(c[1]);
        dh[0] = pack8(hv[0]); dh[1] = pack8(hv[1]);
      }
      if (HSEQ) {
        uint4* dh = reinterpret_cast<uint4*>(h_seq + h_off<CH>(tile, T, t, warp, lane, 512));
        dh[0] = pack8(hv[0]); dh[1] = pack8(hv[1]);
      }
      if (t + 1 < T) {
        __half* sh = sH + ((t + 1) & 1) * CELLS * D::H_LD;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int jn = 0; jn < 4; ++jn)
            *reinterpret_cast<uint32_t*>(sh + (cg * 16 + g + 8 * h) * D::H_LD + 32 * js + 8 * jn + 2 * q) = pack2(hv[h][2 * jn], hv[h][2 * jn + 1]);
      } else if (hT != nullptr) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (live[h]) {
#pragma unroll
            for (int jn = 0; jn < 4; ++jn)
              *reinterpret_cast<float2*>(hT + (size_t)cell[h] * D::H + 32 * js + 8 * jn + 2 * q) = make_float2(hv[h][2 * jn], hv[h][2 * jn + 1]);
          }
      }
      // h_t is complete for the group; buffer (t + 1) & 1 is not written again before every warp has passed the next barrier
      named_bar_sync(1 + cg, 32 * CH);
    }
  }
}

// ---------------------------------------------------------------------------------------
// backward from the saved c_t / h_t: reverse walk (dh, dc, dx and the gate gradients) ...
// ---------------------------------------------------------------------------------------
// Per step and warp: gates_t = hx_t x Wx^T (A = the group's saved h_{t-1}, read per k-block from global memory, + x columns);
// the thread-local cell gradient; da'_t = da_t / s_j of the warp's 128 gate columns into the group's rows of the shared da
// tile and into the workspace record of (tile, t) (rows = cells, 4H columns in slice order); after the group barrier
// dh_{t-1}[slice] = da'_t x (s W_hh) over all 4H gates, and dx = sum of the CH slice partials in a fixed order.
// In a stack (hidden 32 as CH = 1):
//   DHIN   a layer below the top: dh_t = the recurrent part + d(h_t) of the layer above, read from d_seq (dseq_off) at step t;
//          d_hT is not read;
//   UP     a layer above the first: the input columns are h^{l-1}_t from h_in (the lower layer's saved state + 512) and the
//          walk also writes d(h^{l-1}_t) = da'_t x (s W_ih) to d_seq -- the dh_{t-1} product over the W_ih columns of Wx; no dx.
//          A middle layer reads and writes d_seq in place: each thread reads its own 16 values of a step before it writes them.
template <int CH, bool UP = false>
constexpr size_t kWalkSmem = (size_t)(Dims<CH, UP>::G4 * Dims<CH, UP>::WX_LD + Dims<CH>::CELLS * Dims<CH>::DA_LD) * sizeof(__half) +
                             (size_t)(Dims<CH>::CELLS * CH + Dims<CH>::G4) * sizeof(float);

// dh[slice js] of the warp's 16 cells = da'_t x (s W) with W the 4H x H block of Wx columns col0 .. col0 + H - 1 (W_hh at 0,
// W_ih at H in a stacked layer): B from Wx rows (k = gate row r), columns col0 + 32 js ..
template <int CH, bool UP>
__device__ __forceinline__ void da_times_w(uint32_t da_addr, uint32_t wx_all, int col0, int lane, int mi, int js, float (&dh)[2][8]) {
  using D = Dims<CH, UP>;
  float adh[4][4];
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) adh[nt][0] = adh[nt][1] = adh[nt][2] = adh[nt][3] = 0.f;
#pragma unroll (UP ? 2 : 4)
  for (int kb = 0; kb < D::G4 / 16; ++kb) {
    uint32_t a[4];
    ldmatrix_x4(da_addr + 32 * kb, a[0], a[1], a[2], a[3]);
#pragma unroll
    for (int pr = 0; pr < 2; ++pr) {
      uint32_t b0, b1, b2, b3;
      ldmatrix_x4_trans(wx_all + (uint32_t)(((16 * kb + 8 * (mi & 1) + (lane & 7)) * D::WX_LD + col0 + 32 * js + 16 * pr + 8 * (mi >> 1)) * 2),
                        b0, b1, b2, b3);
      mma_16816(adh[2 * pr], a, b0, b1);
      mma_16816(adh[2 * pr + 1], a, b2, b3);
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int s = 0; s < 8; ++s) dh[h][s] = adh[s >> 1][2 * h + (s & 1)];
}

template <int CH, bool UP = false, bool DHIN = false>
__global__ void __launch_bounds__(Dims<CH>::THREADS, Dims<CH>::BWD_CTAS_PER_SM)
lstm_bwd_walk_tcw_kernel(const float* __restrict__ x_seq, const float* __restrict__ w_ih, const float* __restrict__ w_hh,
                         const float* __restrict__ b_ih, const float* __restrict__ b_hh, const float* __restrict__ d_hT,
                         float* __restrict__ d_x, const __half* __restrict__ saved, __half* __restrict__ da_rec,
                         const float* __restrict__ scale2, long long cells, long long tile0, long long tiles, int T, long long NN,
                         const __half* __restrict__ h_in, float* __restrict__ d_seq) {
  using D = Dims<CH, UP>;
  constexpr int CELLS = D::CELLS;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __half* sWx = reinterpret_cast<__half*>(smem_raw);       // [G4][WX_LD], slice order
  __half* sDA = sWx + D::G4 * D::WX_LD;                    // [CELLS][DA_LD]: da'_t, columns in slice order
  float* sDX = reinterpret_cast<float*>(sDA + CELLS * D::DA_LD);   // [CELLS][CH]: dx partial of each slice
  float* s_wih = sDX + CELLS * CH;                         // [G4] by gate row j
  load_wx<CH, UP>(sWx, w_ih, w_hh, b_ih, b_hh);
  if (!UP)
    for (int j = threadIdx.x; j < D::G4; j += blockDim.x) s_wih[j] = w_ih[j];
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3, mi = lane >> 3;
  const int cg = warp / CH, js = warp % CH;
  const uint32_t wx_all = smem_u32(sWx), wx_addr = wx_all + (uint32_t)(js * 128 * D::WX_LD * 2);
  const uint32_t da_addr = smem_u32(sDA + (cg * 16 + (lane & 15)) * D::DA_LD + 8 * (lane >> 4));
  const float S = scale2[0], invS = scale2[1];

  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    long long cell[2];
    bool live[2];
    size_t xb[2];
    float dh[2][8], dc[2][8];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      cell[h] = (tile0 + tile) * CELLS + cg * 16 + g + 8 * h;
      live[h] = cell[h] < cells;
      xb[h] = live[h] ? x_base(cell[h], T, NN) : 0;
#pragma unroll
      for (int s = 0; s < 8; ++s) {
        // (a top layer reads S here rather than keep it in a register across tiles: it has none to spare)
        dh[h][s] = !DHIN && live[h] ? d_hT[(size_t)cell[h] * D::H + 32 * js + 8 * (s >> 1) + 2 * q + (s & 1)] * (UP ? __ldg(scale2) : S) : 0.f;
        dc[h][s] = 0.f;
      }
    }
    // the dx writer of the group (lanes 0..15 of slice 0) owns row 16 cg + lane
    const long long dx_cell = (tile0 + tile) * CELLS + cg * 16 + (lane & 15);
    const bool dx_live = !UP && d_x != nullptr && js == 0 && lane < 16 && dx_cell < cells;
    const size_t dx_base = dx_live ? x_base(dx_cell, T, NN) : 0;

    for (int t = T - 1; t >= 0; --t) {
      if (DHIN) {                     // d(h_t) from the layer above
        const float4* p = reinterpret_cast<const float4*>(d_seq + dseq_off<CH>(tile, T, t, warp, lane));
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float4 v = p[i];
          dh[i >> 1][4 * (i & 1)] += v.x; dh[i >> 1][4 * (i & 1) + 1] += v.y;
          dh[i >> 1][4 * (i & 1) + 2] += v.z; dh[i >> 1][4 * (i & 1) + 3] += v.w;
        }
      }
      uint32_t xw[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) xw[h] = UP ? bias_cols(q) : x_cols(live[h] ? x_seq[xb[h] + (size_t)t * NN] : 0.f, q);
      // h_{t-1} of the group from the saved state (a_from_seq); UP: then h^{l-1}_t of the layer below
      const __half* hp = saved + (t > 0 ? save_off<CH>(tile, T, t - 1, cg * CH, 1, lane) : 0);
      const __half* hin = UP ? h_in + h_off<CH>(tile, T, t, cg * CH, lane, 1024) : nullptr;
      float acc[16][4];
      gate_mma<CH, UP>(acc, [&](int kb, uint32_t (&a)[4]) {
        if (UP && kb >= 2 * CH) { a_from_seq(hin, 1024, kb - 2 * CH, a); return; }
        if (t == 0) { a[0] = a[1] = a[2] = a[3] = 0u; return; }
        const uint2* p = reinterpret_cast<const uint2*>(hp + (kb >> 1) * 1024);
        const uint2 r0 = __ldg(p + (kb & 1)), r1 = __ldg(p + 2 + (kb & 1));
        a[0] = r0.x; a[1] = r1.x; a[2] = r0.y; a[3] = r1.y;
      }, xw, wx_addr);

      uint4 vc[2], vcp[2];
      {
        const uint4* pc = reinterpret_cast<const uint4*>(saved + save_off<CH>(tile, T, t, warp, 0, lane));
        vc[0] = pc[0]; vc[1] = pc[1];
        if (t > 0) {
          const uint4* pcp = reinterpret_cast<const uint4*>(saved + save_off<CH>(tile, T, t - 1, warp, 0, lane));
          vcp[0] = pcp[0]; vcp[1] = pcp[1];
        } else {
          vcp[0] = vcp[1] = make_uint4(0u, 0u, 0u, 0u);
        }
      }
      uint32_t da[16][2];             // fp16 pairs of da' = da / s_j: gate column 8 nt + 2 q, +1 of row h, nt = gate * 4 + jn
      float dx[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float d[4][8];
        dx[h] = cell_grad<CH, !UP>(acc, h, vc[h], vcp[h], dh[h], dc[h], s_wih, js, q, d);
#pragma unroll
        for (int jn = 0; jn < 4; ++jn)
#pragma unroll
          for (int gt = 0; gt < 4; ++gt) {
            const float inv_s = gt == 2 ? -0.5f * kLn2 : -kLn2;     // 1 / s_j: -ln 2 for i, f, o and -ln 2 / 2 for g
            da[4 * gt + jn][h] = pack2(inv_s * d[gt][2 * jn], inv_s * d[gt][2 * jn + 1]);
          }
        if (!UP) {
          dx[h] += __shfl_xor_sync(0xffffffffu, dx[h], 1);
          dx[h] += __shfl_xor_sync(0xffffffffu, dx[h], 2);
        }
      }
      // every warp of the group has finished reading the previous step's da tile and dx partials
      named_bar_sync(1 + cg, 32 * CH);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = cg * 16 + g + 8 * h;
#pragma unroll
        for (int nt = 0; nt < 16; ++nt) *reinterpret_cast<uint32_t*>(sDA + row * D::DA_LD + 128 * js + 8 * nt + 2 * q) = da[nt][h];
        if (!UP && q == 0) sDX[row * CH + js] = dx[h];
      }
      named_bar_sync(1 + cg, 32 * CH);
      if (dx_live) {
        float v = 0.f;
#pragma unroll
        for (int sl = 0; sl < CH; ++sl) v += sDX[(cg * 16 + lane) * CH + sl];
        d_x[dx_base + (size_t)t * NN] = v * invS;
      }
      {                                // the warp's 16 x 128 block of the da tile -> the (tile, t) record
        __half* rec = da_rec + (((size_t)tile * T + t) * CELLS + cg * 16) * D::G4 + 128 * js;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int idx = 32 * i + lane, row = idx >> 4, ch = idx & 15;
          *reinterpret_cast<uint4*>(rec + (size_t)row * D::G4 + 8 * ch) =
              *reinterpret_cast<const uint4*>(sDA + (cg * 16 + row) * D::DA_LD + 128 * js + 8 * ch);
        }
      }
      if (UP) {                       // d(h^{l-1}_t) into d_seq, while dh (consumed by cell_grad) holds nothing
        da_times_w<CH, UP>(da_addr, wx_all, D::H, lane, mi, js, dh);
        float4* p = reinterpret_cast<float4*>(d_seq + dseq_off<CH>(tile, T, t, warp, lane));
#pragma unroll
        for (int i = 0; i < 4; ++i)
          p[i] = make_float4(dh[i >> 1][4 * (i & 1)], dh[i >> 1][4 * (i & 1) + 1], dh[i >> 1][4 * (i & 1) + 2], dh[i >> 1][4 * (i & 1) + 3]);
      }
      if (t > 0) {                    // dh_{t-1}[slice js] = da'_t x (s W_hh): B from Wx rows (k = gate row r), columns 32 js ..
        float adh[4][4];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) adh[nt][0] = adh[nt][1] = adh[nt][2] = adh[nt][3] = 0.f;
#pragma unroll (UP ? 2 : 4)
        for (int kb = 0; kb < D::G4 / 16; ++kb) {
          uint32_t a[4];
          ldmatrix_x4(da_addr + 32 * kb, a[0], a[1], a[2], a[3]);
#pragma unroll
          for (int pr = 0; pr < 2; ++pr) {
            uint32_t b0, b1, b2, b3;
            ldmatrix_x4_trans(wx_all + (uint32_t)(((16 * kb + 8 * (mi & 1) + (lane & 7)) * D::WX_LD + 32 * js + 16 * pr + 8 * (mi >> 1)) * 2),
                              b0, b1, b2, b3);
            mma_16816(adh[2 * pr], a, b0, b1);
            mma_16816(adh[2 * pr + 1], a, b2, b3);
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int s = 0; s < 8; ++s) dh[h][s] = adh[s >> 1][2 * h + (s & 1)];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------
// ... and the weight-gradient pass: dWext[r][k] = s_j * sum over (tile, t, cell) of da'[cell][r] hx_t[cell][k]
// ---------------------------------------------------------------------------------------
// CTA (js, split): the 128 gate rows of slice js, all KX columns, over a contiguous range of (tile, t) records.  Per record
// the da block and hx (h_{t-1} from the saved state, x columns; UP: h_{t-1}, h^{l-1}_t from h_in = the lower layer's saved
// state + 512, bias columns) are staged in shared memory; warp w owns gate rows 16 w .. +15.
constexpr int DW_THREADS = 256;
constexpr int DW_DA_LD = 136;
// the staged tiles; above the 48 KB of static shared memory (hidden 32 in a stack) they are dynamic
template <int CH, bool UP = false>
constexpr size_t kDwSmem = (size_t)Dims<CH>::CELLS * (DW_DA_LD + Dims<CH, UP>::HX_LD) * sizeof(__half);

// DET (deterministic mode): CTA (js, split) stores its rows to the split's slot d_w_hh + split * (4H x H + 4H x KI + 4H), laid out as
// the outputs [4H x H w_hh | 4H x KI w_ih | 4H b] (KI = H for UP, else 1 with the x hi / lo columns added first), without atomics;
// with acc it adds them to the slot (a later chunk of lstm_recompute_backward_tc).
template <int CH, bool UP = false, bool DET = false>
__global__ void __launch_bounds__(DW_THREADS)
lstm_dw_tcw_kernel(const float* __restrict__ x_seq, const __half* __restrict__ saved, const __half* __restrict__ da_rec,
                   float* __restrict__ d_w_ih, float* __restrict__ d_w_hh, float* __restrict__ d_b, const float* __restrict__ scale2,
                   long long cells, long long tile0, long long tiles, int T, long long NN, const __half* __restrict__ h_in, bool acc) {
  using D = Dims<CH, UP>;
  constexpr int CELLS = D::CELLS;
  constexpr int HX_LD = D::HX_LD;
  constexpr int NX = D::KX / 8;                 // n8 tiles of columns
  __half* sDA;
  __half* sHX;
  if constexpr (kDwSmem<CH, UP> <= 48 * 1024) {
    __shared__ __align__(16) __half s_da[CELLS * DW_DA_LD];
    __shared__ __align__(16) __half s_hx[CELLS * HX_LD];
    sDA = s_da;
    sHX = s_hx;
  } else {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    sDA = reinterpret_cast<__half*>(smem_raw);
    sHX = sDA + CELLS * DW_DA_LD;
  }
  const int js = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3, mi = lane >> 3;
  const long long records = tiles * T;
  const long long per = (records + gridDim.y - 1) / gridDim.y;
  const long long r0 = blockIdx.y * per, r1 = r0 + per < records ? r0 + per : records;
  for (int e = threadIdx.x; e < CELLS; e += blockDim.x)          // constant zero columns KX - 8 .. KX - 1
    *reinterpret_cast<uint4*>(sHX + e * HX_LD + D::KX - 8) = make_uint4(0u, 0u, 0u, 0u);
  if (UP)
    for (int e = threadIdx.x; e < CELLS * 4; e += blockDim.x)     // constant bias columns 2 H .. 2 H + 7
      *reinterpret_cast<uint32_t*>(sHX + (e >> 2) * HX_LD + 2 * D::H + 2 * (e & 3)) = bias_cols(e & 3);
  const uint32_t da_addr = smem_u32(sDA), hx_addr = smem_u32(sHX);
  float dw[NX][4];
#pragma unroll
  for (int nt = 0; nt < NX; ++nt) dw[nt][0] = dw[nt][1] = dw[nt][2] = dw[nt][3] = 0.f;

  for (long long rec = r0; rec < r1; ++rec) {
    const long long tile = rec / T;
    const int t = (int)(rec - tile * T);
    __syncthreads();                              // the previous record's tiles are no longer read
    for (int e = threadIdx.x; e < CELLS * 16; e += blockDim.x) {
      const int row = e >> 4, ch = e & 15;
      *reinterpret_cast<uint4*>(sDA + row * DW_DA_LD + 8 * ch) =
          __ldg(reinterpret_cast<const uint4*>(da_rec + ((size_t)rec * CELLS + row) * D::G4 + 128 * js + 8 * ch));
    }
    for (int e = threadIdx.x; e < D::NW * 64; e += blockDim.x) {    // saved h_{t-1}: (warp, lane, row half) -> 4 words
      const int w = e >> 6, l = (e >> 1) & 31, h = e & 1;
      const int row = (w / CH) * 16 + (l >> 2) + 8 * h, col = 32 * (w % CH) + 2 * (l & 3);
      const uint4 v = t > 0 ? __ldg(reinterpret_cast<const uint4*>(saved + save_off<CH>(tile, T, t - 1, w, 1, l)) + h)
                            : make_uint4(0u, 0u, 0u, 0u);
      uint32_t* d = reinterpret_cast<uint32_t*>(sHX + row * HX_LD + col);
      d[0] = v.x; d[4] = v.y; d[8] = v.z; d[12] = v.w;
    }
    if (UP) {
      for (int e = threadIdx.x; e < D::NW * 64; e += blockDim.x) {  // h^{l-1}_t, the same way into columns H ..
        const int w = e >> 6, l = (e >> 1) & 31, h = e & 1;
        const int row = (w / CH) * 16 + (l >> 2) + 8 * h, col = D::H + 32 * (w % CH) + 2 * (l & 3);
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(h_in + h_off<CH>(tile, T, t, w, l, 1024)) + h);
        uint32_t* d = reinterpret_cast<uint32_t*>(sHX + row * HX_LD + col);
        d[0] = v.x; d[4] = v.y; d[8] = v.z; d[12] = v.w;
      }
    } else {
      for (int e = threadIdx.x; e < CELLS * 4; e += blockDim.x) {     // x columns H .. H + 7
        const int row = e >> 2, qq = e & 3;
        const long long cell = (tile0 + tile) * CELLS + row;
        const float x = cell < cells ? x_seq[x_base(cell, T, NN) + (size_t)t * NN] : 0.f;
        *reinterpret_cast<uint32_t*>(sHX + row * HX_LD + D::H + 2 * qq) = x_cols(x, qq);
      }
    }
    __syncthreads();
#pragma unroll
    for (int kc = 0; kc < CELLS / 16; ++kc) {
      uint32_t a[4];
      ldmatrix_x4_trans(da_addr + (uint32_t)(((16 * kc + 8 * (mi >> 1) + (lane & 7)) * DW_DA_LD + 16 * warp + 8 * (mi & 1)) * 2), a[0], a[1], a[2], a[3]);
#pragma unroll
      for (int pr = 0; pr < NX / 2; ++pr) {
        uint32_t b0, b1, b2, b3;
        ldmatrix_x4_trans(hx_addr + (uint32_t)(((16 * kc + 8 * (mi & 1) + (lane & 7)) * HX_LD + 16 * pr + 8 * (mi >> 1)) * 2), b0, b1, b2, b3);
        mma_16816(dw[2 * pr], a, b0, b1);
        mma_16816(dw[2 * pr + 1], a, b2, b3);
      }
    }
  }
  const float invS = scale2[1];
  if constexpr (DET) {
    constexpr int KI = UP ? D::H : 1;
    float* slot = d_w_hh + (size_t)blockIdx.y * (D::G4 * D::H + D::G4 * KI + D::G4);
    float* s_ih = slot + D::G4 * D::H;
    float* s_b = s_ih + D::G4 * KI;
    auto put = [&](float* p, float v) { *p = acc ? *p + v : v; };
#pragma unroll
    for (int nt = 0; nt < NX; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = 128 * js + 16 * warp + g + 8 * (i >> 1), col = 8 * nt + 2 * q + (i & 1), j = gate_row<CH>(r);
        const float v = dw[nt][i] * row_scale(r) * invS;
        const float next = __shfl_down_sync(0xffffffffu, v, 1);     // lane q + 1: column col + 2
        if (col < D::H) put(slot + (size_t)j * D::H + col, v);
        else if (UP) {
          if (col < 2 * D::H) put(s_ih + (size_t)j * D::H + col - D::H, v);
          else if (col == 2 * D::H) put(s_b + j, v);
        }
        else if (col == D::H) put(s_ih + j, v + next);
        else if (col == D::H + 1) put(s_b + j, v);
      }
  } else {
#pragma unroll
    for (int nt = 0; nt < NX; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int r = 128 * js + 16 * warp + g + 8 * (i >> 1), col = 8 * nt + 2 * q + (i & 1), j = gate_row<CH>(r);
        const float v = dw[nt][i] * row_scale(r) * invS;
        if (col < D::H) atomicAdd(&d_w_hh[(size_t)j * D::H + col], v);
        else if (UP) {
          if (col < 2 * D::H) atomicAdd(&d_w_ih[(size_t)j * D::H + col - D::H], v);
          else if (col == 2 * D::H) atomicAdd(&d_b[j], v);     // (column 2 H + 1, against b_lo, is the same sum)
        }
        else if (col == D::H || col == D::H + 2) atomicAdd(&d_w_ih[j], v);
        else if (col == D::H + 1) atomicAdd(&d_b[j], v);
      }
  }
}

}  // namespace lstm_tc

// ---------------------------------------------------------------------------------------
// host
// ---------------------------------------------------------------------------------------
using lstm_tc::Dims;

bool lstm_tc_supported(int T, int C) { return (C == 32 || C == 96 || C == 128) && T >= 1 && T <= 256; }

static long long lstm_tc_tile_cells(int C) { return C == 32 ? Dims<1>::CELLS : C == 96 ? Dims<3>::CELLS : Dims<4>::CELLS; }

// cells of B NN rounded up to whole tiles of the width's kernels
static long long lstm_tc_padded_cells(int B, long long NN, int C) {
  const long long tc = lstm_tc_tile_cells(C);
  return ((long long)B * NN + tc - 1) / tc * tc;
}

// the tiles [tile0, tile0 + n) of a launch (see lstm_tc::save_off): every tile of a call, or one chunk of the recomputing backward
struct TileRange { long long tile0, n; };
static TileRange all_tiles(long long cells, int C) { return {0, (cells + lstm_tc_tile_cells(C) - 1) / lstm_tc_tile_cells(C)}; }
// the cells of a range that exist (the last tile of a call may be part padding)
static long long range_cells(long long cells, TileRange r, int C) {
  const long long end = (r.tile0 + r.n) * lstm_tc_tile_cells(C);
  return (end < cells ? end : cells) - r.tile0 * lstm_tc_tile_cells(C);
}

static int lstm_grid(long long tiles, int ctas_per_sm) {
  long long g = (long long)ctas_per_sm * device_sm_count();
  return (int)(g < tiles ? g : tiles);
}
// CTAs per slice of the wide dW pass over `tiles` tiles: up to 4 per SM in all, each a contiguous range of (tile, step) records
template <int CH>
static int lstm_dw_splits(long long tiles, int T) {
  const long long records = tiles * T, s = 4LL * device_sm_count() / CH;
  return (int)(s < records ? s : records);
}

// Deterministic mode's weight-gradient flush (DESIGN.md section 11); slots == nullptr: atomics.  Each CTA of the hidden-32 walk,
// or each split of a dW pass, writes its own slot image (acc: adds to it, a later chunk of the recomputing backward), and with
// reduce_tiles > 0 the slots that a launch over that many tiles writes are then reduced into the outputs in a fixed order (0: a
// chunk before the last; the recomputing backward reduces after its last chunk the slots its first, largest, chunk wrote).
struct DetFlush { float* slots; bool acc; long long reduce_tiles; };

// c_t | h_t of every cell (tiles padded) and step: 2 C halves, see lstm_tc::save_off
size_t lstm_tc_saved_bytes(int B, int T, long long NN, int C) {
  return (size_t)lstm_tc_padded_cells(B, NN, C) * T * 2 * C * sizeof(__half);
}

// wide widths: the gate-gradient records of the reverse walk, 4 C halves per cell and step (lstm_tc::lstm_bwd_walk_tcw_kernel)
static size_t lstm_tcw_da_bytes(int B, int T, long long NN, int C) {
  return (size_t)lstm_tc_padded_cells(B, NN, C) * T * 4 * C * sizeof(__half);
}

// Deterministic mode: the slots of the weight-gradient flush, one image [4C x C w_hh | 4C x KI w_ih | 4C b] (KI = C in an upper
// stack layer, else 1) per CTA of the single-layer hidden-32 walk, or per split of the wide dW pass (every stack layer included)
static size_t lstm_tc_slot_bytes(int C, bool up) {
  const size_t G4 = 4 * (size_t)C, image = G4 * C + G4 * (up ? C : 1) + G4;
  const size_t n = C == 32 && !up ? (size_t)Dims<1>::BWD_CTAS_PER_SM * device_sm_count() : (size_t)4 * device_sm_count() / (C / 32);
  return align_up(n * image * sizeof(float), 256);
}

// workspace of the backward: the grad scale (1 KB), at the wide widths the da records, deterministic mode's slots (empty with the
// mode off) and, for a call without a saved buffer from the forward (`rebuild`), room to re-run the (training) forward into
struct LstmTcBwdLayout { size_t scale, da, slots, saved, total; };
static LstmTcBwdLayout lstm_tc_bwd_layout(int B, int T, long long NN, int C, bool rebuild) {
  LstmTcBwdLayout L;
  size_t off = 0;
  L.scale = take(off, 1024, 256);
  L.da = take(off, C == 32 ? 0 : lstm_tcw_da_bytes(B, T, NN, C), 256);
  L.slots = take(off, det_mode() ? lstm_tc_slot_bytes(C, false) : 0, 256);
  L.saved = take(off, rebuild ? lstm_tc_saved_bytes(B, T, NN, C) : 0, 256);
  L.total = align_up(off, 256);
  return L;
}
size_t lstm_tc_bwd_workspace_bytes(int B, int T, long long NN, int C) { return lstm_tc_bwd_layout(B, T, NN, C, true).total; }

template <int CH>
static int lstm_forward_tcw(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, float* hT,
                            void* saved, long long cells, TileRange r, int T, long long NN, cudaStream_t st) {
  using D = Dims<CH>;
  auto kern = saved ? lstm_tc::lstm_fwd_tcw_kernel<CH, true> : lstm_tc::lstm_fwd_tcw_kernel<CH, false>;
  constexpr size_t smem = lstm_tc::kFwdWideSmem<CH>;
  static DynSmemAttr attr_t = {}, attr_f = {};
  if (int e = ensure_dyn_smem(kern, (int)smem, saved ? attr_t : attr_f)) return e;
  prof_begin(PROF_LSTM_FWD, 8.0 * D::H * (D::H + 1) * (double)range_cells(cells, r, D::H) * T, st);
  kern<<<lstm_grid(r.n, D::FWD_CTAS_PER_SM), D::THREADS, smem, st>>>(x_seq, w_ih, w_hh, b_ih, b_hh, hT, static_cast<__half*>(saved), cells,
                                                                     r.tile0, r.n, T, NN, nullptr, nullptr);
  prof_end(st);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

// lstm_backward_h32 and lstm_backward_tcw<CH>: the kernels of one width's backward over the tiles r, run once the grad scale and
// the zeroed weight gradients are in place.  da_rec: the gate-gradient records of the wide walk (the hidden-32 walk keeps them on
// chip).  f.slots: deterministic mode's flush slots (lstm_tc_slot_bytes), null for the atomic flush
static int lstm_backward_h32(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                             const float* d_hT, float* d_w_ih, float* d_w_hh, float* d_b, float* d_x, const void* saved,
                             void* /*da_rec*/, DetFlush f, const float* scale2, long long cells, TileRange r, int T, long long NN,
                             cudaStream_t st) {
  using D = Dims<1>;
  float* slots = f.slots;
  using K = decltype(&lstm_tc::lstm_bwd_saved_tc_kernel<false>);
  static const K kerns[2][2][2] = {     // [RANGE][DET][DX]
      {{lstm_tc::lstm_bwd_saved_tc_kernel<false>, lstm_tc::lstm_bwd_saved_tc_kernel<true>},
       {lstm_tc::lstm_bwd_saved_tc_kernel<false, true>, lstm_tc::lstm_bwd_saved_tc_kernel<true, true>}},
      {{lstm_tc::lstm_bwd_saved_tc_kernel<false, false, true>, lstm_tc::lstm_bwd_saved_tc_kernel<true, false, true>},
       {lstm_tc::lstm_bwd_saved_tc_kernel<false, true, true>, lstm_tc::lstm_bwd_saved_tc_kernel<true, true, true>}}};
  static DynSmemAttr attrs[2][2][2] = {};
  const bool range = r.tile0 != 0 || r.n != all_tiles(cells, D::H).n;
  const K kern = kerns[range][slots != nullptr][d_x != nullptr];
  if (int e = ensure_dyn_smem(kern, (int)lstm_tc::kBwdSavedSmem, attrs[range][slots != nullptr][d_x != nullptr])) return e;
  prof_begin(PROF_LSTM_BWD, 12.0 * D::H * (D::H + 1) * (double)range_cells(cells, r, D::H) * T, st);
  kern<<<lstm_grid(r.n, D::BWD_CTAS_PER_SM), D::THREADS, lstm_tc::kBwdSavedSmem, st>>>(
      x_seq, w_ih, w_hh, b_ih, b_hh, d_hT, d_w_ih, slots ? slots : d_w_hh, d_b, d_x, static_cast<const __half*>(saved), scale2, cells,
      r.tile0, r.n, T, NN, f.acc);
  prof_end(st);
  MPGCN_CUDA(cudaGetLastError());
  if (slots && f.reduce_tiles)
    return reduce_slots(slots, lstm_grid(f.reduce_tiles, D::BWD_CTAS_PER_SM), (long long)D::G4 * D::H + 2 * D::G4, 1, 0,
                        slot_image(d_w_hh, (long long)D::G4 * D::H, d_w_ih, D::G4, d_b, D::G4), st);
  return 0;
}

// the wide dW pass of one layer (KI = H for an upper stack layer, else 1), then in deterministic mode the reduction of its slots
template <int CH, bool UP>
static int lstm_dw_pass(const float* x_seq, const void* saved, const void* da_rec, float* d_w_ih, float* d_w_hh, float* d_b, DetFlush f,
                        const float* scale2, long long cells, TileRange r, int T, long long NN, const void* h_in, double flops, cudaStream_t st) {
  using D = Dims<CH>;
  constexpr int KI = UP ? D::H : 1;
  float* slots = f.slots;
  auto dw = slots ? lstm_tc::lstm_dw_tcw_kernel<CH, UP, true> : lstm_tc::lstm_dw_tcw_kernel<CH, UP>;
  constexpr size_t dw_smem = lstm_tc::kDwSmem<CH, UP> <= 48 * 1024 ? 0 : lstm_tc::kDwSmem<CH, UP>;
  static DynSmemAttr attr_d = {}, attr_dd = {};
  if (dw_smem)
    if (int e = ensure_dyn_smem(dw, (int)dw_smem, slots ? attr_dd : attr_d)) return e;
  prof_begin(PROF_LSTM_BWD, flops, st);
  dw<<<dim3(CH, (unsigned)lstm_dw_splits<CH>(r.n, T)), lstm_tc::DW_THREADS, dw_smem, st>>>(
      x_seq, static_cast<const __half*>(saved), static_cast<const __half*>(da_rec), d_w_ih, slots ? slots : d_w_hh, d_b, scale2, cells,
      r.tile0, r.n, T, NN, static_cast<const __half*>(h_in), f.acc);
  prof_end(st);
  MPGCN_CUDA(cudaGetLastError());
  if (slots && f.reduce_tiles)
    return reduce_slots(slots, lstm_dw_splits<CH>(f.reduce_tiles, T), (long long)D::G4 * (D::H + KI + 1), 1, 0,
                        slot_image(d_w_hh, (long long)D::G4 * D::H, d_w_ih, (long long)D::G4 * KI, d_b, D::G4), st);
  return 0;
}

template <int CH>
static int lstm_backward_tcw(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                             const float* d_hT, float* d_w_ih, float* d_w_hh, float* d_b, float* d_x, const void* saved, void* da_rec,
                             DetFlush f, const float* scale2, long long cells, TileRange r, int T, long long NN, cudaStream_t st) {
  using D = Dims<CH>;
  constexpr size_t smem = lstm_tc::kWalkSmem<CH>;
  const double rc = (double)range_cells(cells, r, D::H);
  static DynSmemAttr attr_b = {};
  if (int e = ensure_dyn_smem(lstm_tc::lstm_bwd_walk_tcw_kernel<CH>, (int)smem, attr_b)) return e;
  // walk: the gate recompute and dh_{t-1} (2 x 8 H (H + 1) per cell and step, as the hidden-32 count splits it) ...
  prof_begin(PROF_LSTM_BWD, 8.0 * D::H * (D::H + 1) * rc * T, st);
  lstm_tc::lstm_bwd_walk_tcw_kernel<CH><<<lstm_grid(r.n, D::BWD_CTAS_PER_SM), D::THREADS, smem, st>>>(
      x_seq, w_ih, w_hh, b_ih, b_hh, d_hT, d_x, static_cast<const __half*>(saved), static_cast<__half*>(da_rec), scale2, cells, r.tile0,
      r.n, T, NN, nullptr, nullptr);
  prof_end(st);
  MPGCN_CUDA(cudaGetLastError());
  // ... and the weight gradient (8 H (H + 1) / 2 more: 12 H (H + 1) in all)
  return lstm_dw_pass<CH, false>(x_seq, saved, da_rec, d_w_ih, d_w_hh, d_b, f, scale2, cells, r, T, NN, nullptr,
                                 4.0 * D::H * (D::H + 1) * rc * T, st);
}

// the single-layer forward over the tiles r (saved: their training state, or null)
static int lstm_forward_range(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, float* hT,
                              void* saved, long long cells, TileRange r, int T, long long NN, int C, cudaStream_t st) {
  using D = Dims<1>;
  if (C == 96) return lstm_forward_tcw<3>(x_seq, w_ih, w_hh, b_ih, b_hh, hT, saved, cells, r, T, NN, st);
  if (C == 128) return lstm_forward_tcw<4>(x_seq, w_ih, w_hh, b_ih, b_hh, hT, saved, cells, r, T, NN, st);
  MPGCN_CHECK(C == D::H, "lstm forward: no tensor-core kernel for hidden=%d", C);
  const bool range = r.tile0 != 0 || r.n != all_tiles(cells, C).n;
  auto kern = range ? (saved ? lstm_tc::lstm_fwd_tc_kernel<true, true> : lstm_tc::lstm_fwd_tc_kernel<false, true>)
                    : (saved ? lstm_tc::lstm_fwd_tc_kernel<true> : lstm_tc::lstm_fwd_tc_kernel<false>);
  prof_begin(PROF_LSTM_FWD, 8.0 * C * (C + 1) * (double)range_cells(cells, r, C) * T, st);
  kern<<<lstm_grid(r.n, D::FWD_CTAS_PER_SM), D::THREADS, 0, st>>>(x_seq, w_ih, w_hh, b_ih, b_hh, hT, static_cast<__half*>(saved), cells,
                                                                  r.tile0, r.n, T, NN);
  prof_end(st);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

int lstm_last_forward_tc(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, float* hT,
                         void* saved, int B, int T, long long NN, int C, cudaStream_t st) {
  const long long cells = (long long)B * NN;
  MPGCN_CHECK(saved == nullptr || (reinterpret_cast<uintptr_t>(saved) & 15) == 0, "lstm forward: saved buffer must be 16-byte aligned");
  return lstm_forward_range(x_seq, w_ih, w_hh, b_ih, b_hh, hT, saved, cells, all_tiles(cells, C), T, NN, C, st);
}

int lstm_last_backward_tc(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                          const float* d_hT, float* d_w_ih, float* d_w_hh, float* d_b_ih, float* d_b_hh, float* d_x, const void* saved,
                          int B, int T, long long NN, int C, void* ws, size_t ws_bytes, const float* d_hT_absmax, cudaStream_t st) {
  const long long cells = (long long)B * NN;
  const LstmTcBwdLayout L = lstm_tc_bwd_layout(B, T, NN, C, saved == nullptr);
  MPGCN_CHECK(ws != nullptr && ws_bytes >= L.total, "lstm backward: workspace too small (%zu < %zu)", ws_bytes, L.total);
  MPGCN_CHECK(saved == nullptr || (reinterpret_cast<uintptr_t>(saved) & 15) == 0, "lstm backward: saved buffer must be 16-byte aligned");
  MPGCN_CHECK((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "lstm backward: workspace must be 256-byte aligned");
  MPGCN_CHECK(C == 32 || C == 96 || C == 128, "lstm backward: no tensor-core kernel for hidden=%d", C);
  uint8_t* wb = static_cast<uint8_t*>(ws);
  float* scale2 = reinterpret_cast<float*>(wb + L.scale);
  void* da_rec = wb + L.da;
  float* slots = det_mode() ? reinterpret_cast<float*>(wb + L.slots) : nullptr;     // fixed-order flush instead of atomics
  if (saved == nullptr) {          // the caller kept no forward state: rebuild it (same kernel, same bits as the training forward)
    void* tmp = wb + L.saved;
    if (int e = lstm_last_forward_tc(x_seq, w_ih, w_hh, b_ih, b_hh, nullptr, tmp, B, T, NN, C, st)) return e;
    saved = tmp;
  }
  const int G4 = 4 * C;
  if (int e = grad_scale_prepare(d_hT, (size_t)cells * C, scale2, d_hT_absmax, st)) return e;
  MPGCN_CUDA(cudaMemsetAsync(d_w_ih, 0, sizeof(float) * G4, st));
  MPGCN_CUDA(cudaMemsetAsync(d_w_hh, 0, sizeof(float) * G4 * C, st));
  MPGCN_CUDA(cudaMemsetAsync(d_b_ih, 0, sizeof(float) * G4, st));
  if (C == 32 && d_x) MPGCN_CUDA(cudaMemsetAsync(d_x, 0, sizeof(float) * (size_t)cells * T, st));
  const TileRange r = all_tiles(cells, C);
  auto backward = C == 32 ? lstm_backward_h32 : C == 96 ? lstm_backward_tcw<3> : lstm_backward_tcw<4>;
  if (int e = backward(x_seq, w_ih, w_hh, b_ih, b_hh, d_hT, d_w_ih, d_w_hh, d_b_ih, d_x, saved, da_rec, DetFlush{slots, false, r.n}, scale2,
                       cells, r, T, NN, st))
    return e;
  return lstm_copy_bias_grad(d_b_ih, d_b_hh, G4, st);
}

// ---------------------------------------------------------------------------------------
// stacked LSTM (L >= 2 layers): every layer on the wide kernels, hidden 32 as CH = 1
// ---------------------------------------------------------------------------------------
// Hidden 32 and 96 only: an upper layer's gate weights, 4H x (2H + 24) halves, take 22 KB and 162 KB of shared memory; at 128
// they would take 280 KB, more than a CTA has.
bool lstm_tc_stack_supported(int T, int C, int L) { return L >= 2 && (C == 32 || C == 96) && T >= 1 && T <= 256; }

// training state of the stack: one lstm_tc_saved_bytes block per layer (multiples of 256 bytes)
size_t lstm_tc_stack_saved_bytes(int B, int T, long long NN, int C, int L) { return (size_t)L * lstm_tc_saved_bytes(B, T, NN, C); }

// inference forward: the h-only sequences (C halves per cell and step) that an inference layer hands to the layer above, of two
// consecutive layers (layer l writes h[l & 1]; one sequence for L = 2)
struct StackFwdLayout { size_t h[2], total; };
static StackFwdLayout stack_fwd_layout(int B, int T, long long NN, int C, int L) {
  StackFwdLayout Y;
  size_t off = 0;
  const size_t hseq = (size_t)lstm_tc_padded_cells(B, NN, C) * T * C * sizeof(__half);
  Y.h[0] = take(off, hseq, 256);
  Y.h[1] = L >= 3 ? take(off, hseq, 256) : Y.h[0];
  Y.total = align_up(off, 256);
  return Y;
}
size_t lstm_tc_stack_fwd_workspace_bytes(int B, int T, long long NN, int C, int L) { return stack_fwd_layout(B, T, NN, C, L).total; }

// backward: the grad scale (1 KB), the fp32 gradient sequence d(h^{l-1}_t) between consecutive walks (lstm_tc::dseq_off),
// deterministic mode's slots of the dW passes (lstm_tc_slot_bytes of an upper layer, the largest; empty with the mode off) and
// the da records of one layer (the layers run one after another).  A workspace of `every_layer` bytes keeps every layer's
// records (layer l at da + l * da_stride) instead of reusing one region, so that they can be read back after the call.
struct StackBwdLayout { size_t scale, d_seq, slots, da, da_stride, total, every_layer; };
static StackBwdLayout stack_bwd_layout(int B, int T, long long NN, int C, int L) {
  StackBwdLayout Y;
  size_t off = 0;
  Y.scale = take(off, 1024, 256);
  Y.d_seq = take(off, (size_t)lstm_tc_padded_cells(B, NN, C) * T * C * sizeof(float), 256);
  Y.slots = take(off, det_mode() ? lstm_tc_slot_bytes(C, true) : 0, 256);
  Y.da_stride = align_up(lstm_tcw_da_bytes(B, T, NN, C), 256);
  Y.da = take(off, Y.da_stride, 256);
  Y.total = off;
  Y.every_layer = off + (size_t)(L - 1) * Y.da_stride;
  return Y;
}
size_t lstm_tc_stack_bwd_workspace_bytes(int B, int T, long long NN, int C, int L) { return stack_bwd_layout(B, T, NN, C, L).total; }

template <int CH, bool SAVE, bool UP, bool HSEQ>
static int stack_fwd_layer(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, float* hT,
                           void* saved, const void* h_in, void* h_seq, long long cells, TileRange r, int T, long long NN, cudaStream_t st) {
  using D = Dims<CH>;
  auto kern = lstm_tc::lstm_fwd_tcw_kernel<CH, SAVE, UP, HSEQ>;
  constexpr size_t smem = lstm_tc::kFwdWideSmem<CH, UP>;
  static DynSmemAttr attr = {};
  if (int e = ensure_dyn_smem(kern, (int)smem, attr)) return e;
  prof_begin(PROF_LSTM_FWD, 8.0 * D::H * ((UP ? 2 : 1) * D::H + 1) * (double)range_cells(cells, r, D::H) * T, st);
  kern<<<lstm_grid(r.n, D::FWD_CTAS_PER_SM), D::THREADS, smem, st>>>(x_seq, w_ih, w_hh, b_ih, b_hh, hT, static_cast<__half*>(saved), cells,
                                                                     r.tile0, r.n, T, NN, static_cast<const __half*>(h_in),
                                                                     static_cast<__half*>(h_seq));
  prof_end(st);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

// the stack over the tiles r; training (saved != null): layer l's state at saved + l * layer_bytes
template <int CH>
static int stack_forward(const float* x_seq, int L, const float* const* w_ih, const float* const* w_hh, const float* const* b_ih,
                         const float* const* b_hh, float* hT, void* saved, size_t layer_bytes, void* ws, const StackFwdLayout& Y,
                         long long cells, TileRange r, int T, long long NN, cudaStream_t st) {
  auto lsaved = [&](int l) { return static_cast<uint8_t*>(saved) + (size_t)l * layer_bytes; };
  auto hbuf = [&](int l) { return static_cast<uint8_t*>(ws) + Y.h[l & 1]; };   // inference: h of layer l
  for (int l = 0; l < L; ++l) {
    const bool top = l == L - 1;
    float* out = top ? hT : nullptr;
    int e;
    if (saved) {       // training: every layer keeps c_t | h_t; the layer above reads the h half
      if (l == 0) e = stack_fwd_layer<CH, true, false, false>(x_seq, w_ih[0], w_hh[0], b_ih[0], b_hh[0], out, lsaved(0), nullptr, nullptr,
                                                           cells, r, T, NN, st);
      else e = stack_fwd_layer<CH, true, true, false>(nullptr, w_ih[l], w_hh[l], b_ih[l], b_hh[l], out, lsaved(l), lsaved(l - 1) + 1024, nullptr, cells, r, T, NN, st);
    } else if (l == 0) {
      e = stack_fwd_layer<CH, false, false, true>(x_seq, w_ih[0], w_hh[0], b_ih[0], b_hh[0], nullptr, nullptr, nullptr, hbuf(0), cells, r, T,
                                                  NN, st);
    } else if (!top) {
      e = stack_fwd_layer<CH, false, true, true>(nullptr, w_ih[l], w_hh[l], b_ih[l], b_hh[l], nullptr, nullptr, hbuf(l - 1), hbuf(l),
                                                 cells, r, T, NN, st);
    } else {
      e = stack_fwd_layer<CH, false, true, false>(nullptr, w_ih[l], w_hh[l], b_ih[l], b_hh[l], hT, nullptr, hbuf(l - 1), nullptr, cells,
                                                  r, T, NN, st);
    }
    if (e) return e;
  }
  return 0;
}

template <int CH, bool UP, bool DHIN>
static int stack_bwd_layer(const float* x_seq, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, const float* d_hT,
                           float* d_w_ih, float* d_w_hh, float* d_b, float* d_x, const void* saved, const void* h_in, void* da_rec,
                           float* d_seq, DetFlush f, const float* scale2, long long cells, TileRange r, int T, long long NN, cudaStream_t st) {
  using D = Dims<CH>;
  const double rc = (double)range_cells(cells, r, D::H);
  constexpr int KH = UP ? 2 * D::H : D::H;     // the input and recurrent columns of the gate GEMM
  auto walk = lstm_tc::lstm_bwd_walk_tcw_kernel<CH, UP, DHIN>;
  constexpr size_t smem = lstm_tc::kWalkSmem<CH, UP>;
  static DynSmemAttr attr_w = {};
  if (int e = ensure_dyn_smem(walk, (int)smem, attr_w)) return e;
  // the walk and the weight gradient, counted as the single layer's are, with the gate GEMM KH + 1 deep: 8 H (KH + 1) ...
  prof_begin(PROF_LSTM_BWD, 8.0 * D::H * (KH + 1) * rc * T, st);
  walk<<<lstm_grid(r.n, D::BWD_CTAS_PER_SM), D::THREADS, smem, st>>>(x_seq, w_ih, w_hh, b_ih, b_hh, d_hT, d_x,
                                                                     static_cast<const __half*>(saved), static_cast<__half*>(da_rec), scale2,
                                                                     cells, r.tile0, r.n, T, NN, static_cast<const __half*>(h_in), d_seq);
  prof_end(st);
  MPGCN_CUDA(cudaGetLastError());
  // ... and the weight gradient, 4 H (KH + 1)
  return lstm_dw_pass<CH, UP>(x_seq, saved, da_rec, d_w_ih, d_w_hh, d_b, f, scale2, cells, r, T, NN, h_in, 4.0 * D::H * (KH + 1) * rc * T, st);
}

template <int CH>
static int stack_backward(const float* x_seq, int L, const float* const* w_ih, const float* const* w_hh, const float* const* b_ih,
                          const float* const* b_hh, const float* d_hT, float* const* d_w_ih, float* const* d_w_hh, float* const* d_b,
                          float* d_x, const void* saved, size_t layer_bytes, uint8_t* da_rec, size_t da_stride, float* d_seq, DetFlush f,
                          size_t slot_stride, const float* scale2, long long cells, TileRange r, int T, long long NN, cudaStream_t st) {
  auto lsaved = [&](int l) { return static_cast<const uint8_t*>(saved) + (size_t)l * layer_bytes; };
  for (int l = L - 1; l >= 0; --l) {    // top-down: the walk of layer l leaves d(h^{l-1}_t) in d_seq for layer l - 1
    const bool top = l == L - 1;
    uint8_t* rec = da_rec + (size_t)l * da_stride;
    // slot_stride floats apart, each layer's slots (0: the layers share one region, each reducing its own before the next)
    const DetFlush fl = {f.slots ? f.slots + (size_t)l * slot_stride : nullptr, f.acc, f.reduce_tiles};
    int e;
    if (l == 0)
      e = stack_bwd_layer<CH, false, true>(x_seq, w_ih[0], w_hh[0], b_ih[0], b_hh[0], nullptr, d_w_ih[0], d_w_hh[0], d_b[0], d_x, lsaved(0),
                                           nullptr, rec, d_seq, fl, scale2, cells, r, T, NN, st);
    else if (top)
      e = stack_bwd_layer<CH, true, false>(nullptr, w_ih[l], w_hh[l], b_ih[l], b_hh[l], d_hT, d_w_ih[l], d_w_hh[l], d_b[l], nullptr,
                                           lsaved(l), lsaved(l - 1) + 1024, rec, d_seq, fl, scale2, cells, r, T, NN, st);
    else
      e = stack_bwd_layer<CH, true, true>(nullptr, w_ih[l], w_hh[l], b_ih[l], b_hh[l], nullptr, d_w_ih[l], d_w_hh[l], d_b[l], nullptr,
                                          lsaved(l), lsaved(l - 1) + 1024, rec, d_seq, fl, scale2, cells, r, T, NN, st);
    if (e) return e;
  }
  return 0;
}

int lstm_stack_forward_tc(const float* x_seq, int L, const float* const* w_ih, const float* const* w_hh, const float* const* b_ih,
                          const float* const* b_hh, float* hT, void* saved, void* ws, size_t ws_bytes, int B, int T, long long NN, int C,
                          cudaStream_t st) {
  MPGCN_CHECK(lstm_tc_stack_supported(T, C, L), "lstm stack: no tensor-core kernels for L=%d, hidden=%d, T=%d", L, C, T);
  MPGCN_CHECK(saved == nullptr || (reinterpret_cast<uintptr_t>(saved) & 255) == 0, "lstm stack forward: saved buffer must be 256-byte aligned");
  const StackFwdLayout Y = stack_fwd_layout(B, T, NN, C, L);
  if (saved == nullptr) {      // inference: the h sequences live in the workspace
    MPGCN_CHECK(ws != nullptr && ws_bytes >= Y.total, "lstm stack forward: workspace too small (%zu < %zu)", ws_bytes, Y.total);
    MPGCN_CHECK((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "lstm stack forward: workspace must be 256-byte aligned");
  }
  const long long cells = (long long)B * NN;
  const size_t layer_bytes = lstm_tc_saved_bytes(B, T, NN, C);
  return C == 32 ? stack_forward<1>(x_seq, L, w_ih, w_hh, b_ih, b_hh, hT, saved, layer_bytes, ws, Y, cells, all_tiles(cells, C), T, NN, st)
                 : stack_forward<3>(x_seq, L, w_ih, w_hh, b_ih, b_hh, hT, saved, layer_bytes, ws, Y, cells, all_tiles(cells, C), T, NN, st);
}

int lstm_stack_backward_tc(const float* x_seq, int L, const float* const* w_ih, const float* const* w_hh, const float* const* b_ih,
                           const float* const* b_hh, const float* d_hT, float* const* d_w_ih, float* const* d_w_hh, float* const* d_b_ih,
                           float* const* d_b_hh, float* d_x, const void* saved, void* ws, size_t ws_bytes, int B, int T, long long NN,
                           int C, const float* d_hT_absmax, cudaStream_t st) {
  MPGCN_CHECK(lstm_tc_stack_supported(T, C, L), "lstm stack: no tensor-core kernels for L=%d, hidden=%d, T=%d", L, C, T);
  const StackBwdLayout Y = stack_bwd_layout(B, T, NN, C, L);
  MPGCN_CHECK(ws != nullptr && ws_bytes >= Y.total, "lstm stack backward: workspace too small (%zu < %zu)", ws_bytes, Y.total);
  MPGCN_CHECK((reinterpret_cast<uintptr_t>(saved) & 255) == 0, "lstm stack backward: saved buffer must be 256-byte aligned");
  MPGCN_CHECK((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "lstm stack backward: workspace must be 256-byte aligned");
  const long long cells = (long long)B * NN;
  uint8_t* wb = static_cast<uint8_t*>(ws);
  float* scale2 = reinterpret_cast<float*>(wb + Y.scale);
  float* d_seq = reinterpret_cast<float*>(wb + Y.d_seq);
  float* slots = det_mode() ? reinterpret_cast<float*>(wb + Y.slots) : nullptr;     // fixed-order flush instead of atomics
  uint8_t* da_rec = wb + Y.da;
  const size_t da_stride = ws_bytes >= Y.every_layer ? Y.da_stride : 0;     // every layer's records, or one region
  // one gradient scale S for the whole stack, from max|d_hT|: every walk keeps dh, dc and d_seq in units of S
  if (int e = grad_scale_prepare(d_hT, (size_t)cells * C, scale2, d_hT_absmax, st)) return e;
  const int G4 = 4 * C;
  for (int l = 0; l < L; ++l) {
    MPGCN_CUDA(cudaMemsetAsync(d_w_ih[l], 0, sizeof(float) * G4 * (l == 0 ? 1 : C), st));
    MPGCN_CUDA(cudaMemsetAsync(d_w_hh[l], 0, sizeof(float) * G4 * C, st));
    MPGCN_CUDA(cudaMemsetAsync(d_b_ih[l], 0, sizeof(float) * G4, st));
  }
  const TileRange r = all_tiles(cells, C);
  const DetFlush f = {slots, false, r.n};
  const size_t layer_bytes = lstm_tc_saved_bytes(B, T, NN, C);
  const int e = C == 32 ? stack_backward<1>(x_seq, L, w_ih, w_hh, b_ih, b_hh, d_hT, d_w_ih, d_w_hh, d_b_ih, d_x, saved, layer_bytes, da_rec,
                                            da_stride, d_seq, f, 0, scale2, cells, r, T, NN, st)
                        : stack_backward<3>(x_seq, L, w_ih, w_hh, b_ih, b_hh, d_hT, d_w_ih, d_w_hh, d_b_ih, d_x, saved, layer_bytes, da_rec,
                                            da_stride, d_seq, f, 0, scale2, cells, r, T, NN, st);
  if (e) return e;
  for (int l = 0; l < L; ++l)
    if (int e2 = lstm_copy_bias_grad(d_b_ih[l], d_b_hh[l], G4, st)) return e2;
  return 0;
}

// ---------------------------------------------------------------------------------------
// recomputing backward: the forward kept no state; it is rebuilt and walked back one chunk of tiles at a time
// ---------------------------------------------------------------------------------------
// Per chunk: the SAVE forward of every layer over the chunk into the chunk's state region (layer l reads layer l - 1's, as in
// the training forward), the walks top-down, the dW passes over the chunk's records.  The kernels are those of the stored-state
// path, so every cell sees the same state bits and the same S (one grad scale over all cells): h_T, dx and the per-cell gate
// gradients are bitwise those of mpgcn_lstm_last_backward_saved / mpgcn_lstm_stack_backward; the weight gradients differ only
// in fp32 summation order.  Memory: O(chunk) instead of O(B NN T C); cost: one more forward.

// tiles of a chunk: chunk_cells rounded up to whole tiles, raised to one wave of the backward grid (one CTA per SM at every
// width) so that no chunk leaves SMs idle, and capped at every tile
static long long recompute_chunk_tiles(long long cells, int C, long long chunk_cells) {
  const long long tc = lstm_tc_tile_cells(C), all = all_tiles(cells, C).n;
  const long long wave = (long long)Dims<1>::BWD_CTAS_PER_SM * device_sm_count();
  long long n = chunk_cells / tc + (chunk_cells % tc != 0);
  if (n < wave) n = wave;
  return n < all ? n : all;
}

// workspace: the grad scale (1 KB); a stack's fp32 sequence d(h^{l-1}_t) of one chunk; deterministic mode's slots, one
// lstm_tc_slot_bytes region per layer that accumulates across chunks (empty with the mode off); the chunk's training state of
// every layer (lstm_tc_saved_bytes of the chunk's cells); the chunk's da records at the wide widths and in stacks, one region
// reused by every layer
struct RecomputeLayout { long long chunk_tiles; size_t scale, d_seq, slots, slot_stride, saved, saved_stride, da, total; };
static RecomputeLayout recompute_layout(int B, int T, long long NN, int C, int L, long long chunk_cells) {
  RecomputeLayout Y;
  Y.chunk_tiles = recompute_chunk_tiles((long long)B * NN, C, chunk_cells);
  const long long cc = Y.chunk_tiles * lstm_tc_tile_cells(C);
  size_t off = 0;
  Y.scale = take(off, 1024, 256);
  Y.d_seq = take(off, L >= 2 ? (size_t)cc * T * C * sizeof(float) : 0, 256);
  Y.slot_stride = det_mode() ? lstm_tc_slot_bytes(C, L >= 2) : 0;
  Y.slots = take(off, (size_t)L * Y.slot_stride, 256);
  Y.saved_stride = align_up(lstm_tc_saved_bytes(1, T, cc, C), 256);
  Y.saved = take(off, (size_t)L * Y.saved_stride, 256);
  Y.da = take(off, C == 32 && L == 1 ? 0 : lstm_tcw_da_bytes(1, T, cc, C), 256);
  Y.total = align_up(off, 256);
  return Y;
}
size_t lstm_tc_recompute_bwd_workspace_bytes(int B, int T, long long NN, int C, int L, long long chunk_cells) {
  return recompute_layout(B, T, NN, C, L, chunk_cells).total;
}

int lstm_recompute_backward_tc(const float* x_seq, int L, const float* const* w_ih, const float* const* w_hh, const float* const* b_ih,
                               const float* const* b_hh, const float* d_hT, float* const* d_w_ih, float* const* d_w_hh,
                               float* const* d_b_ih, float* const* d_b_hh, float* d_x, long long chunk_cells, void* ws, size_t ws_bytes,
                               int B, int T, long long NN, int C, const float* d_hT_absmax, cudaStream_t st) {
  MPGCN_CHECK(L == 1 ? lstm_tc_supported(T, C) : lstm_tc_stack_supported(T, C, L), "lstm recompute: no tensor-core kernels for L=%d, hidden=%d, T=%d",
              L, C, T);
  MPGCN_CHECK(chunk_cells >= 1, "lstm recompute: chunk_cells=%lld (at least 1)", chunk_cells);
  const RecomputeLayout Y = recompute_layout(B, T, NN, C, L, chunk_cells);
  MPGCN_CHECK(ws != nullptr && ws_bytes >= Y.total, "lstm recompute: workspace too small (%zu < %zu)", ws_bytes, Y.total);
  MPGCN_CHECK((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "lstm recompute: workspace must be 256-byte aligned");
  const long long cells = (long long)B * NN, all = all_tiles(cells, C).n;
  uint8_t* wb = static_cast<uint8_t*>(ws);
  float* scale2 = reinterpret_cast<float*>(wb + Y.scale);
  float* d_seq = reinterpret_cast<float*>(wb + Y.d_seq);
  float* slots = det_mode() ? reinterpret_cast<float*>(wb + Y.slots) : nullptr;
  void* saved = wb + Y.saved;
  uint8_t* da_rec = wb + Y.da;
  if (int e = grad_scale_prepare(d_hT, (size_t)cells * C, scale2, d_hT_absmax, st)) return e;
  const int G4 = 4 * C;
  for (int l = 0; l < L; ++l) {
    MPGCN_CUDA(cudaMemsetAsync(d_w_ih[l], 0, sizeof(float) * G4 * (l == 0 ? 1 : C), st));
    MPGCN_CUDA(cudaMemsetAsync(d_w_hh[l], 0, sizeof(float) * G4 * C, st));
    MPGCN_CUDA(cudaMemsetAsync(d_b_ih[l], 0, sizeof(float) * G4, st));
  }
  // every launch below writes d_x of its chunk's cells in full, so d_x needs no clearing
  for (long long t0 = 0; t0 < all; t0 += Y.chunk_tiles) {
    const TileRange r = {t0, Y.chunk_tiles < all - t0 ? Y.chunk_tiles : all - t0};
    const DetFlush f = {slots, t0 > 0, t0 + r.n == all ? Y.chunk_tiles : 0};
    int e;
    if (L == 1) {
      e = lstm_forward_range(x_seq, w_ih[0], w_hh[0], b_ih[0], b_hh[0], nullptr, saved, cells, r, T, NN, C, st);
      if (e == 0) {
        auto backward = C == 32 ? lstm_backward_h32 : C == 96 ? lstm_backward_tcw<3> : lstm_backward_tcw<4>;
        e = backward(x_seq, w_ih[0], w_hh[0], b_ih[0], b_hh[0], d_hT, d_w_ih[0], d_w_hh[0], d_b_ih[0], d_x, saved, da_rec, f, scale2, cells,
                     r, T, NN, st);
      }
    } else {
      const StackFwdLayout none = {};      // (a training forward keeps no h sequence in a workspace)
      const size_t slot_floats = Y.slot_stride / sizeof(float);
      e = C == 32 ? stack_forward<1>(x_seq, L, w_ih, w_hh, b_ih, b_hh, nullptr, saved, Y.saved_stride, nullptr, none, cells, r, T, NN, st)
                  : stack_forward<3>(x_seq, L, w_ih, w_hh, b_ih, b_hh, nullptr, saved, Y.saved_stride, nullptr, none, cells, r, T, NN, st);
      if (e == 0)
        e = C == 32 ? stack_backward<1>(x_seq, L, w_ih, w_hh, b_ih, b_hh, d_hT, d_w_ih, d_w_hh, d_b_ih, d_x, saved, Y.saved_stride, da_rec, 0,
                                        d_seq, f, slot_floats, scale2, cells, r, T, NN, st)
                    : stack_backward<3>(x_seq, L, w_ih, w_hh, b_ih, b_hh, d_hT, d_w_ih, d_w_hh, d_b_ih, d_x, saved, Y.saved_stride, da_rec, 0,
                                        d_seq, f, slot_floats, scale2, cells, r, T, NN, st);
    }
    if (e) return e;
  }
  for (int l = 0; l < L; ++l)
    if (int e = lstm_copy_bias_grad(d_b_ih[l], d_b_hh[l], G4, st)) return e;
  return 0;
}

}  // namespace mpgcn
