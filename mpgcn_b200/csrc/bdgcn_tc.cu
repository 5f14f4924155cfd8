// BDGCN layer on the wgmma contraction engine (precision 1: fp16 operands, fp32 accumulate; precision 2, bf16x3: every operand a
// pair of bf16 planes hi = bf16(a), lo = bf16(a - hi), each product hi*hi + hi*lo + lo*hi, fp32 accumulate).
//
// Same factored algebra as bdgcn_simt.cu (reference: BDGCN.forward of MPGCN.py; factoring:
// SURVEY.md section 7.1); each contraction is one launch of tc::contract_kernel with operands
// described by TMA tensor maps over fp16 copies living in the caller's workspace.
//
// Channel widths C = 32 cC and H = 32 cH.  The copies of the caller's tensors (X16, dP16) keep their channel-last layout; the
// engine's intermediates hold 32-channel "chunk planes" [..][rows][e][32] (lc < cC indexes an input chunk, hc < cH an output
// chunk; at C = H = 32 every chunk index is 0 and the layouts are the single-chunk ones):
//
//   forward   X16 [B][n][c][C]      G16 [zg][K][N][Np]  (Np = N rounded up to 8, rows padded)
//             Z16 [B][d][lc][n][e][32]  (saved for backward)   U16 [B][hc][o][n][e][32]
//     FWD_A   Z = X x2 G_d          A_MN128 (G_d [c][e])     B = X16 chunk lc (ch, c, n, b)        one launch per lc
//     FWD_MIX U = sum_d Z_d W[o,d]  A_K64   (Z plane)        B = W16  [(hc,o)][(d,lc,l)][32]       Kd cC -> Ko cH planes
//     FWD_B   out = act(sum_o G_o^T x1 U_o + b)   A_MN128 (G flat [(o,n)][m])  B = U16 chunk hc flat  one launch per hc
//   backward  dP16 [B][m][e][H]   V16 [B][o][hc][n][e][32]   Y16 [B][d][lc][n][e][32]   Wq16 [(d,lc)][(o,hc,h)][32]
//     BWD_V   V = G_o x1 dPre       A_K128  (G_o [n][m])     B = dP16 chunk hc flat                one launch per hc
//     BWD_DW  dW = Z^T V            A_MN64  (Z, Kd cC chunks)  B = V16 (Ko cH chunks)   split-K
//     BWD_MIX Y = sum_o V_o W[o,d]^T  A_K64 (V plane)        B = Wq16                              Ko cH -> Kd cC planes
//     BWD_DX  dX = sum_d Y_d x2 G_d^T A_K128 (G_d [c][e])    B = Y16 chunk lc (l, e, n, (b,d))     one launch per lc
//   support gradients (opt-in, after the stages above; X16 [B][n][c][C] cast again, U16 recomputed from the Z stash by FWD_MIX)
//     BWD_DGO dG_o[n][m] = sum_{b,e,h} U_o[b,n,e,h] dPre[b,m,e,h]   A_K64 (U16 plane, k = (e, 32))   B K-major = dP16 [m][(e, 32 hc)]
//     BWD_DGD dG_d[c][e] = sum_{b,n,l} X[b,n,c,l] Y_d[b,n,e,l]     A_K64 (X16 [c][(lc, 32)])        B K-major = Y16 [e][32] per (b,d,lc,n)
//             one split-K launch per output plane into fp32 partials [slice][N][32 ceil(N/32)], each reduced (x 1/S) into dG
// The N^3 contractions act on each channel on its own, so a chunk is a 32-channel layer to them; the chunk planes are laid out
// so that the per-chunk launch addresses them through a base offset and strides (plane index (b*K + d)*cC + lc of Z16 / Y16
// and (b*Ko + o)*cH + hc of V16 are affine in the launch's z = b*K + d; U16 keeps FWD_B's flat (o, n) contraction per chunk).
// bf16x3 (DESIGN.md section 3): each 16-bit tensor above (X16, G16, Z16, U16, dP16, V16, Y16, W16 / Wq16) holds bf16 instead and is
// followed by its lo plane, a copy of its layout right behind it, so the lo plane of TMA plane z is plane z + (the tensor's plane
// count): the engine runs each contraction as three passes over k (two for the mixes, whose resident W pair already is the
// b_res_reps = 2 halves) and the epilogues write the 16-bit results as pairs.  No diagonal-remainder correction (a pair carries
// 16 significant bits), no support gradients, no layer parts.
#include "kernels.h"
#include "tc_engine.cuh"

#include <string.h>

namespace mpgcn {

using tc::GemmParams;

namespace {
inline int ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }
inline int pad8(int n) { return (n + 7) / 8 * 8; }
const int kBig = 1 << 30;

tc::OperandMap omap(int z_div, int z_mod, int z_mul, int seg_mul, int k_seg, int seg_mod = 1 << 30, int seg_hi_mul = 0) {
  tc::OperandMap m;
  m.z_div = z_div; m.z_mod = z_mod; m.z_mul = z_mul; m.seg_mul = seg_mul; m.k_seg = k_seg;
  m.seg_mod = seg_mod; m.seg_hi_mul = seg_hi_mul;
  return m;
}

void init_params(GemmParams& p) {
  memset(&p, 0, sizeof(p));
  p.am = omap(1, 1, 0, 0, 0);
  p.bm = omap(1, 1, 0, 0, 0);
  p.kb_per_slice = 1;
  p.ep.alpha = 1.f;
}

// one contraction in the precision of the call: fp16, or bf16x3 in `passes` passes of p.kb_total k-blocks over plane pairs whose lo
// planes lie a_plane_z / b_plane_z TMA z coordinates after the hi ones (tc_engine.cuh, GemmParams::kb_pass)
int launch(bool bf, int ak, int bk, GemmParams& p, int passes, int a_plane_z, int b_plane_z, cudaStream_t st) {
  if (!bf) return tc::launch_contract(ak, bk, p, st);
  p.kb_pass = p.kb_total;
  p.kb_total *= passes;
  p.a_plane_z = a_plane_z;
  p.b_plane_z = b_plane_z;
  p.ep.corr_src = nullptr;
  return tc::launch_contract_bf16x3(ak, bk, p, st);
}

// support stack G16 [zg*K][N rows][Np]: as A_MN128 (dims m, k-rows, z) or A_K128 (dims k, m-rows, z)
int map_support_mn(CUtensorMap* m, const __half* g16, int N, int Np, long long rows_per_z, long long nz) {
  const uint64_t dims[4] = {(uint64_t)N, (uint64_t)rows_per_z, (uint64_t)nz, 1};
  const uint64_t str[3] = {(uint64_t)Np * 2, (uint64_t)rows_per_z * Np * 2, (uint64_t)rows_per_z * Np * 2 * (uint64_t)nz};
  const uint32_t box[4] = {64, 64, 1, 1};
  return make_tmap_f16(m, g16, 4, dims, str, box, TMAP_SW128);
}
int map_support_k(CUtensorMap* m, const __half* g16, int N, int Np, long long nz) {
  const uint64_t dims[4] = {(uint64_t)N, (uint64_t)N, (uint64_t)nz, 1};
  const uint64_t str[3] = {(uint64_t)Np * 2, (uint64_t)N * Np * 2, (uint64_t)N * Np * 2 * (uint64_t)nz};
  const uint32_t box[4] = {64, 128, 1, 1};
  return make_tmap_f16(m, g16, 4, dims, str, box, TMAP_SW128);
}
// channel-chunk tensor T[z][r][k][32]: dims (ch, k, r, z)
int map_chunks(CUtensorMap* m, const __half* t, long long k_rows, long long k_stride_el, long long r_count, long long r_stride_el,
               long long z_count, long long z_stride_el, int box_k, int box_r) {
  const uint64_t dims[4] = {32, (uint64_t)k_rows, (uint64_t)r_count, (uint64_t)z_count};
  const uint64_t str[3] = {(uint64_t)k_stride_el * 2, (uint64_t)r_stride_el * 2, (uint64_t)z_stride_el * 2};
  const uint32_t box[4] = {32, (uint32_t)box_k, (uint32_t)box_r, 1};
  return make_tmap_f16(m, t, 4, dims, str, box, TMAP_SW64);
}
// K-major plane tensor T[plane][rows][32]: dims (k=32, row, plane, 1), box (32, 128)
int map_planes(CUtensorMap* m, const __half* t, long long rows, long long planes, int box_planes = 1) {
  const uint64_t dims[4] = {32, (uint64_t)rows, (uint64_t)planes, 1};
  const uint64_t str[3] = {64, (uint64_t)rows * 64, (uint64_t)rows * 64 * (uint64_t)planes};
  const uint32_t box[4] = {32, 128, (uint32_t)box_planes, 1};
  return make_tmap_f16(m, t, 4, dims, str, box, TMAP_SW64);
}
}  // namespace

// Any number of supports: the N^3 contractions index supports through z and k-segments, the channel mixes and BWD_DW split
// more than 8 output planes into column groups, and the FWD_B epilogue walks its remainders 8 segments at a time.  Any
// channel widths that are multiples of 32 up to 1024: a layer of width 32 c is c chunk planes to the mixes and BWD_DW and c
// launches of the N^3 contractions (the ReLU / bias-gradient pass keeps one channel per thread of a block: H <= 1024).
bool tc_supported(const BdgcnShape& s) {
  return s.C >= 32 && s.C % 32 == 0 && s.H >= 32 && s.H % 32 == 0 && s.H <= 1024 && s.Ko >= 1 && s.Kd >= 1 && s.N >= 1 && s.B >= 1 &&
         s.R >= 1 && s.row0 >= 0 && s.row0 + s.R <= s.N;
}

// The int indices that grow with the number of supports and chunks: the plane index b*Kd*cC + .. / b*Ko*cH + .. (TMA plane
// coordinates of every contraction, p.Z of FWD_A / BWD_V), the k coordinate o*N + n of FWD_B's support map, and the
// Ko*Kd*C*H weight elements of the weight permutations / reduce_dw_partials.  (Tile counts are checked at launch; byte sizes
// are size_t.)
static int check_index_range(const BdgcnShape& s) {
  const long long K = s.Ko > s.Kd ? s.Ko : s.Kd;
  const long long in_planes = (long long)s.Kd * (s.C / 32), out_planes = (long long)s.Ko * (s.H / 32);
  const long long planes = in_planes > out_planes ? in_planes : out_planes;
  MPGCN_CHECK((long long)s.B * planes < (1ll << 31) && K * s.N + 128 < (1ll << 31) && (long long)s.Ko * s.Kd * s.C * s.H < (1ll << 31),
              "tensor-core path: B=%d N=%d Ko=%d Kd=%d C=%d H=%d overflows the engine's 32-bit plane and row indices", s.B, s.N, s.Ko,
              s.Kd, s.C, s.H);
  return 0;
}

// cells of an activation slab: R origin rows x N destinations
static size_t rn(const BdgcnShape& s) { return (size_t)s.R * s.N; }
static size_t g16_elems(const BdgcnShape& s, int K) { return (size_t)(s.dynamic ? s.B : 1) * K * s.N * pad8(s.N); }
static size_t g_planes(const BdgcnShape& s, int K) { return (size_t)(s.dynamic ? s.B : 1) * K; }

// a bf16x3 pair is two planes of 16-bit elements
size_t tc_saved_bytes(const BdgcnShape& s, bool bf) { return (size_t)(bf ? 2 : 1) * s.B * s.Kd * rn(s) * s.C * sizeof(__half); }

// workspace layouts (byte offsets); also served to tests by mpgcn_debug_tc_workspace_offset()
struct FwdLayout { size_t x16, gd16, go16, w16, u16, z16, dd, dgo, dgo_masked, total; };
static FwdLayout fwd_layout(const BdgcnShape& s, bool bf) {
  FwdLayout L;
  size_t off = 0;
  const size_t pl = bf ? 2 : 1;                          // bf16x3: hi and lo planes
  L.x16 = take(off, pl * s.B * rn(s) * s.C * 2, 1024);
  L.gd16 = take(off, pl * g16_elems(s, s.Kd) * 2, 1024);
  L.go16 = take(off, pl * g16_elems(s, s.Ko) * 2, 1024);
  L.w16 = take(off, (size_t)2 * s.Ko * s.Kd * s.C * s.H * 2, 1024);    // [hi | lo]
  L.u16 = take(off, pl * s.B * s.Ko * rn(s) * s.H * 2, 1024);
  L.dd = take(off, g_planes(s, s.Kd) * s.N * 4, 1024);   // support-diagonal fp16 remainders (destination / origin)
  L.dgo = take(off, g_planes(s, s.Ko) * s.N * 4, 1024);
  L.dgo_masked = take(off, g_planes(s, s.Ko) * s.N * 4, 1024);   // origin remainders restricted to the row slab
  L.z16 = take(off, tc_saved_bytes(s, bf), 1024);        // used only when the caller passes no `saved` buffer
  L.total = align_up(off, 1024);
  return L;
}
size_t tc_fwd_ws_bytes(const BdgcnShape& s, bool bf) { return fwd_layout(s, bf).total; }
// BWD_DW: rows are the Kd*cC chunks of Z16, 4 per m-tile; columns are the Ko*cH chunks of V16, all in one tile up to 8,
// else ceil(n / 8) column tiles of dw_chunks(n) chunks each (the last one partly past n: TMA zero-fills those chunks and the
// epilogue skips them)
static int dw_row_chunks(const BdgcnShape& s) { return s.Kd * (s.C / 32); }
static int dw_col_chunks(const BdgcnShape& s) { return s.Ko * (s.H / 32); }
static int dw_col_tiles(int n) { return ceil_div(n, 8); }
static int dw_chunks(int n) { return ceil_div(n, dw_col_tiles(n)); }
static int dw_slices(const BdgcnShape& s, int* kb_per_slice, int* kb_total, int passes = 1) {
  const int kbps = ceil_div((long long)rn(s), 64);
  const int total = s.B * kbps * passes;
  const int tiles = ceil_div(dw_row_chunks(s), 4) * dw_col_tiles(dw_col_chunks(s));     // tiles per slice
  int want = device_sm_count() / tiles;
  if (want < 1) want = 1;
  int per = ceil_div(total, want);
  if (per < 1) per = 1;
  *kb_per_slice = per;
  *kb_total = total;
  return ceil_div(total, per);
}
// support gradients: the dG partials
static int dg_chunks(const BdgcnShape& s) { return ceil_div(s.N, 32); }                 // 32-column chunks of a dG row
static int dg_r(const BdgcnShape& s) { return dg_chunks(s) < 8 ? dg_chunks(s) : 8; }   // chunks per tile
static int dg_max_slices(const BdgcnShape& s) {
  const int tiles = ceil_div(s.N, 128) * ceil_div(dg_chunks(s), dg_r(s));
  const int want = device_sm_count() / tiles;
  return want < 1 ? 1 : want;
}
// backward workspace; `sgrad` (the support gradient) appends X16, U16, the forward's fp16 W split and the dG partials.  Last,
// deterministic mode's bias-gradient slots (relu_bwd_prep), empty with the mode off; dW and dG already reduce their split-K
// partials in a fixed order.
struct BwdLayout { size_t dp16, gd16, go16, v16, y16, wq16, partials, scale, x16, u16, w16, dg_partials, db_slots, total; };
static BwdLayout bwd_layout(const BdgcnShape& s, bool sgrad, bool bf = false) {
  BwdLayout L{};
  size_t off = 0;
  const size_t pl = bf ? 2 : 1;                                      // bf16x3: hi and lo planes (Wq: both halves)
  L.dp16 = take(off, pl * s.B * s.N * s.N * s.H * 2, 1024);          // dPre: every origin row m, always
  L.gd16 = take(off, pl * g16_elems(s, s.Kd) * 2, 1024);
  L.go16 = take(off, pl * g16_elems(s, s.Ko) * 2, 1024);
  L.v16 = take(off, pl * s.B * s.Ko * rn(s) * s.H * 2, 1024);
  L.y16 = take(off, pl * s.B * s.Kd * rn(s) * s.C * 2, 1024);
  L.wq16 = take(off, pl * s.Ko * s.Kd * s.C * s.H * 2, 1024);
  int per = 1, total = 1;
  const int slices = dw_slices(s, &per, &total, bf ? 3 : 1);
  L.partials = take(off, (size_t)slices * ceil_div(dw_row_chunks(s), 4) * 128 * s.Ko * s.H * 4, 1024);
  L.scale = take(off, 64, 1024);
  if (sgrad) {
    L.x16 = take(off, (size_t)s.B * rn(s) * s.C * 2, 1024);
    L.u16 = take(off, (size_t)s.B * s.Ko * rn(s) * s.H * 2, 1024);
    L.w16 = take(off, (size_t)2 * s.Ko * s.Kd * s.C * s.H * 2, 1024);
    L.dg_partials = take(off, (size_t)dg_max_slices(s) * s.N * 32 * dg_chunks(s) * 4, 1024);
  }
  L.db_slots = take(off, det_mode() ? bias_grad_slot_bytes(s.H) : 0, 1024);
  L.total = off;     // the slots end the workspace unpadded
  return L;
}
size_t tc_bwd_ws_bytes(const BdgcnShape& s, bool bf) { return bwd_layout(s, false, bf).total; }
size_t tc_sgrad_ws_bytes(const BdgcnShape& s) { return bwd_layout(s, true).total; }

// which: 0 x16, 1 gd16, 2 go16, 3 w16, 4 u16 (forward); 10 dp16, 11 gd16, 12 go16, 13 v16, 14 y16, 15 wq16, 16 partials,
// 17 number of dW slices (not an offset)
long long tc_debug_offset(const BdgcnShape& s, int which) {
  const FwdLayout F = fwd_layout(s, false);
  const BwdLayout Bw = bwd_layout(s, false);
  int per = 1, total = 1;
  switch (which) {
    case 0: return (long long)F.x16;
    case 1: return (long long)F.gd16;
    case 2: return (long long)F.go16;
    case 3: return (long long)F.w16;
    case 4: return (long long)F.u16;
    case 5: return (long long)F.dd;
    case 6: return (long long)F.dgo;
    case 10: return (long long)Bw.dp16;
    case 11: return (long long)Bw.gd16;
    case 12: return (long long)Bw.go16;
    case 13: return (long long)Bw.v16;
    case 14: return (long long)Bw.y16;
    case 15: return (long long)Bw.wq16;
    case 16: return (long long)Bw.partials;
    case 17: return dw_slices(s, &per, &total);
    case 18: return (long long)Bw.scale;
    default: return -1;
  }
}

// ---------------------------------------------------------------------------------------
// individual contractions.  Activations are [B][*][R rows n][N][32] slabs (R = N for a whole layer); supports G_d has Kd
// planes per sample, G_o has Ko.
// ---------------------------------------------------------------------------------------
// FWD_A:  Z16[b][d][lc][n][e][l] = sum_c G_d[c][e] X16[b][n][c][32 lc + l]      one launch per input chunk lc
// bf: bf16x3 pairs (every pointer then addresses the hi plane of a pair, see the head of this file)
static int run_fwd_a(const BdgcnShape& s, const __half* gd16, const __half* x16, __half* z16, const float* delta_d, cudaStream_t st,
                     bool bf = false) {
  const int N = s.N, R = s.R, K = s.Kd, Np = pad8(N), C = s.C, cC = s.C / 32, pl = bf ? 2 : 1;
  const long long NN = (long long)rn(s);
  for (int lc = 0; lc < cC; ++lc) {
    const __half* xc = x16 + lc * 32;
    GemmParams p;
    init_params(p);
    if (int e = map_support_mn(&p.a_map, gd16, N, Np, N, (long long)g_planes(s, K) * pl)) return e;
    if (int e = map_chunks(&p.b_map, xc, N, C, R, (long long)N * C, (long long)s.B * pl, (long long)R * N * C, 64, 8)) return e;
    p.am = omap(1, s.dynamic ? kBig : K, 1, 0, 0);        // z = b*K + d -> support index
    p.bm = omap(K, kBig, 1, 0, 0);                        // -> b
    p.MT = ceil_div(N, 128); p.NT = ceil_div(R, 8); p.Z = s.B * K; p.R = 8;
    p.z_inner = K;                                        // the K supports of one (sample, row block) run back to back: X16 block from L2
    p.kb_total = p.kb_per_seg = ceil_div(N, 64);
    p.ep.out = z16 + lc * NN * 32; p.ep.out_f16 = 1;      // plane (b*K + d)*cC + lc
    p.ep.sZ = cC * NN * 32; p.ep.sI = 32; p.ep.sR = (long long)N * 32;
    p.ep.m_valid = N; p.ep.r_valid = R;
    // Z[b,d,n,e,:] += (G_d[e,e] - fp16(G_d[e,e])) * X16[b,n,e,:]
    p.ep.corr_src = xc; p.ep.corr_delta = delta_d; p.ep.corr_nseg = 1;
    p.ep.cZ = (long long)R * N * C; p.ep.cI = C; p.ep.cR = (long long)N * C; p.ep.cSeg = 0;
    if (bf) p.ep.out16 = z16 + lc * NN * 32 + (size_t)s.B * K * cC * NN * 32;     // the lo plane of Z
    prof_set_next(PROF_FWD_A, 2.0 * s.B * K * (double)R * N * N * 32);
    if (int e = launch(bf, tc::A_MN128, 64, p, 3, (int)g_planes(s, K), s.B, st)) return e;
  }
  return 0;
}

// MIX: D16[b][r][row][32] = sum_{seg < Kin} A16[b][seg][row][32] * Wm16[r][(seg,32)][32], r < Kout   (both channel mixes)
// One tile emits all the output planes of its rows as Kout chunks of 32 columns, so one launch covers Kout <= 8 (the widest
// wgmma, N = 256).  More output planes go in ceil(Kout / 8) groups of balanced size, one launch each: group [r0, r0 + Rg) sees
// W from its first output plane on and writes from output plane r0 on, with the same plane stride.  Each group re-reads A.
// bf16x3 (bf, w_halves = 2: W's hi / lo pair): the A pair runs in two passes with W resident, hi meeting both halves and lo W hi
// only, or in three passes with W streaming (one half per pass); the output is written as a pair
static int run_mix_group(const BdgcnShape& s, const __half* a16, const __half* w16, int w_halves, __half* d16, int tag, int Kin,
                         int Kout, int r0, int Rg, cudaStream_t st, bool bf) {
  const long long NN = (long long)rn(s);
  const int pl = bf ? 2 : 1;
  GemmParams p;
  init_params(p);
  w16 += (size_t)r0 * Kin * 32 * 32;                                  // W rows of output plane r0, every half
  if (bf) p.ep.out16 = d16 + (size_t)s.B * Kout * NN * 32 + (size_t)r0 * NN * 32;   // the lo plane of the output
  d16 += (size_t)r0 * NN * 32;
  const size_t w_bytes = (size_t)Rg * w_halves * Kin * 32 * 64;        // Kin * w_halves tiles of Rg chunks x [32 k][64 B]
  int bk = 32;
  if (Kin == 2 || Kin == 3) {
    // One k-block per tile: a single TMA box brings the Kin planes of a 128-cell tile (the single-thread producer / MMA loops
    // cost ~0.3 us per k-block, which bounded the per-plane version at a third of the HBM rate), W resident in shared memory
    bk = 32 * Kin;
    if (int e = map_planes(&p.a_map, a16, NN, (long long)s.B * Kin * pl, Kin)) return e;
    if (int e = map_chunks(&p.b_map, w16, (long long)Kin * 32, 32, Rg, (long long)Kin * 32 * 32, w_halves, (long long)Kout * Kin * 32 * 32, bk, Rg)) return e;
    p.am = omap(1, kBig, Kin, 0, 0);               // z = b -> first plane b*Kin
    p.bm = omap(1, 1, 0, 1, 0);                    // resident tile index = weight half
    p.kb_total = 1; p.kb_per_seg = 1; p.b_res_reps = w_halves;
  } else {
    if (int e = map_planes(&p.a_map, a16, NN, (long long)s.B * Kin * pl)) return e;
    if (int e = map_chunks(&p.b_map, w16, (long long)Kin * 32, 32, Rg, (long long)Kin * 32 * 32, w_halves, (long long)Kout * Kin * 32 * 32, 32, Rg)) return e;
    // segment s: plane = b*Kin + (s % Kin); weight rows (s % Kin)*32 of half s / Kin  (half 0 = fp16(W), half 1 = fp16(W - half 0))
    p.am = omap(1, kBig, Kin, 1, 0, Kin, 0);
    p.bm = omap(1, 1, 0, 0, 32, Kin, 1);
    if (w_bytes > 160 * 1024) { p.kb_total = bf ? Kin : Kin * w_halves; p.kb_per_seg = 1; }   // large K: W streams with A
    else { p.kb_total = Kin; p.kb_per_seg = 1; p.b_res_reps = w_halves; }              // W resident, A plane by plane
  }
  const int passes = p.b_res_reps ? 2 : 3;
  p.MT = ceil_div(NN, 128); p.NT = 1; p.Z = s.B; p.R = Rg;
  p.ep.out = d16; p.ep.out_f16 = 1;
  p.ep.sZ = (long long)Kout * NN * 32; p.ep.sI = 32; p.ep.sR = NN * 32;
  p.ep.m_valid = (int)NN; p.ep.r_valid = Rg;
  prof_set_next(tag, 2.0 * s.B * (double)Kin * Rg * NN * 32 * 32);   // algorithmic flops (the fp16 hi/lo weight split doubles the executed MMAs)
  return launch(bf, tc::A_K64, bk, p, passes, (int)(s.B * Kin), 1, st);   // lo planes: B*Kin A planes, one W half on
}
static int run_mix(const BdgcnShape& s, const __half* a16, const __half* w16, int w_halves, __half* d16, int tag, int Kin, int Kout,
                   cudaStream_t st, bool bf = false) {
  const int groups = ceil_div(Kout, 8);
  for (int g = 0, r0 = 0; g < groups; ++g) {
    const int Rg = Kout / groups + (g < Kout % groups ? 1 : 0);     // 9 -> 5 + 4, 17 -> 6 + 6 + 5
    if (int e = run_mix_group(s, a16, w16, w_halves, d16, tag, Kin, Kout, r0, Rg, st, bf)) return e;
    r0 += Rg;
  }
  return 0;
}

// FWD_B: out[b][m][e][32 hc + h] = act( sum_{(o,n)} G_o[row0 + n][m] U16[b][hc][o][n][e][h] + bias[32 hc + h] )
//        n < R, every m < N; one launch per output chunk hc
static int run_fwd_b(const BdgcnShape& s, const __half* go16, const __half* u16_all, const float* bias, float* out, __half* out16,
                     const float* delta_o, cudaStream_t st, bool bf = false) {
  const int N = s.N, R = s.R, K = s.Ko, Np = pad8(N), H = s.H, cH = s.H / 32, pl = bf ? 2 : 1;
  const bool slab = !(R == N && s.row0 == 0);
  const int gplanes = s.dynamic ? s.B : 1;
  int a_lo = 0, b_lo = 0;                 // bf16x3: TMA z distance of the lo planes
  for (int hc = 0; hc < cH; ++hc) {
    const __half* u16 = u16_all + (size_t)hc * K * rn(s) * 32;
    GemmParams p;
    init_params(p);
    if (!slab) {
      // whole layer: the contraction index (o, n) is a plain row index of the flat [K*N][N] support stack and of U16
      if (int e = map_support_mn(&p.a_map, go16, N, Np, (long long)K * N, gplanes * pl)) return e;
      // U16 [b][hc][(o,n)][e][h] read as (h, k = (o,n) rows, r = e, b): dims listed with non-monotonic strides (the r stride,
      // 64 B, is smaller than the k stride) so that ONE box (32 ch, 64 k, 4|8 r) lands in the canonical [r][k][64 B] layout
      if (int e = map_chunks(&p.b_map, u16, (long long)K * N, (long long)N * 32, N, 32, (long long)s.B * pl, (long long)cH * K * N * N * 32, 64, 8)) return e;
      p.am = omap(1, s.dynamic ? kBig : 1, 1, 0, 0);
      p.bm = omap(1, kBig, 1, 0, 0);
      p.kb_total = p.kb_per_seg = ceil_div((long long)K * N, 64);
      a_lo = gplanes; b_lo = s.B;
    } else {
      // origin-row slab: one k-segment per support o.  A = rows [row0, row0 + R) of G_o (k coordinate o*N + kk inside the flat
      // stack, base pointer moved to row0); B = U16 [b][hc][o][n < R]: TMA zero-fills rows >= R, which also cancels the rows of
      // the NEXT slab that the last k-block of a segment reads from G.
      {
        const uint64_t dims[4] = {(uint64_t)N, (uint64_t)((long long)K * N - s.row0), (uint64_t)(gplanes * pl), 1};
        const uint64_t str[3] = {(uint64_t)Np * 2, (uint64_t)K * N * Np * 2, (uint64_t)K * N * Np * 2 * (uint64_t)gplanes};
        const uint32_t box[4] = {64, 64, 1, 1};
        if (int e = make_tmap_f16(&p.a_map, go16 + (size_t)s.row0 * Np, 4, dims, str, box, TMAP_SW128)) return e;
      }
      if (int e = map_chunks(&p.b_map, u16, R, (long long)N * 32, N, 32, (long long)s.B * cH * K * pl - (long long)hc * K, (long long)R * N * 32, 64, 8)) return e;
      p.am = omap(1, s.dynamic ? kBig : 1, 1, 0, N);          // k coordinate += o * N
      p.bm = omap(1, kBig, cH * K, 1, 0);                     // plane = (b*cH + hc)*K + o, from this chunk's base
      p.kb_per_seg = ceil_div(R, 64);
      p.kb_total = K * p.kb_per_seg;
      a_lo = gplanes; b_lo = s.B * cH * K;
    }
    p.MT = ceil_div(N, 128); p.NT = ceil_div(N, 8); p.Z = s.B; p.R = 8;
    p.ep.out = out + hc * 32; p.ep.out_f16 = 0; p.ep.out16 = out16 ? out16 + hc * 32 : nullptr;
    p.ep.sZ = (long long)N * N * H; p.ep.sI = (long long)N * H; p.ep.sR = H;
    p.ep.m_valid = N; p.ep.r_valid = N;
    p.ep.bias = (s.partial || !bias) ? nullptr : bias + hc * 32; p.ep.relu = s.partial ? 0 : s.act;
    // pre[b,m,e,:] += sum_o (G_o[m,m] - fp16(G_o[m,m])) * U16[b,hc,o,m,e,:]   (delta_o is zero outside the slab: the row n = m of
    // U exists only for row0 <= m < row0 + R; corr_src is moved so that row index m addresses slab row m - row0)
    p.ep.corr_src = u16 - (long long)s.row0 * N * 32; p.ep.corr_delta = delta_o; p.ep.corr_nseg = K;
    // (the epilogue forms the sample offset as zB * cZ with zB = b in the flat mode and b*cH*K in the slab mode)
    p.ep.cZ = slab ? (long long)R * N * 32 : (long long)cH * K * R * N * 32;
    p.ep.cSeg = (long long)R * N * 32; p.ep.cI = (long long)N * 32; p.ep.cR = 32;
    prof_set_next(PROF_FWD_B, 2.0 * s.B * K * (double)R * N * N * 32);
    if (int e = launch(bf, tc::A_MN128, 64, p, 3, a_lo, b_lo, st)) return e;
  }
  return 0;
}

// BWD_V: V16[b][o][hc][n][e][h] = sum_m G_o[row0 + n][m] dP16[b][m][e][32 hc + h]       n < R; one launch per output chunk hc
static int run_bwd_v(const BdgcnShape& s, const __half* go16, const __half* dp16, __half* v16, cudaStream_t st, bool bf = false) {
  const int N = s.N, R = s.R, K = s.Ko, Np = pad8(N), H = s.H, cH = s.H / 32, pl = bf ? 2 : 1;
  const long long NN = (long long)rn(s);
  for (int hc = 0; hc < cH; ++hc) {
    GemmParams p;
    init_params(p);
    {   // rows [row0, row0 + R) of every support plane, K-major
      const long long nz = (long long)g_planes(s, K);
      const uint64_t dims[4] = {(uint64_t)N, (uint64_t)R, (uint64_t)(nz * pl), 1};
      const uint64_t str[3] = {(uint64_t)Np * 2, (uint64_t)N * Np * 2, (uint64_t)N * Np * 2 * (uint64_t)nz};
      const uint32_t box[4] = {64, 128, 1, 1};
      if (int e = make_tmap_f16(&p.a_map, go16 + (size_t)s.row0 * Np, 4, dims, str, box, TMAP_SW128)) return e;
    }
    // dP16 [b][m][e][H] chunk hc read as (h, k = m, r = e, b), see run_fwd_b
    if (int e = map_chunks(&p.b_map, dp16 + hc * 32, N, (long long)N * H, N, H, (long long)s.B * pl, (long long)N * N * H, 64, 8)) return e;
    p.am = omap(1, s.dynamic ? kBig : K, 1, 0, 0);        // z = b*K + o
    p.bm = omap(K, kBig, 1, 0, 0);
    p.MT = ceil_div(R, 128); p.NT = ceil_div(N, 8); p.Z = s.B * K; p.R = 8;
    p.z_inner = K;                                        // dP16 block of one (sample, e block) serves the K supports back to back
    p.kb_total = p.kb_per_seg = ceil_div(N, 64);
    p.ep.out = v16 + hc * NN * 32; p.ep.out_f16 = 1;      // plane (b*K + o)*cH + hc
    p.ep.sZ = cH * NN * 32; p.ep.sI = (long long)N * 32; p.ep.sR = 32;
    p.ep.m_valid = R; p.ep.r_valid = N;
    if (bf) p.ep.out16 = v16 + hc * NN * 32 + (size_t)s.B * K * cH * NN * 32;     // the lo plane of V
    prof_set_next(PROF_BWD_V, 2.0 * s.B * K * (double)R * N * N * 32);
    if (int e = launch(bf, tc::A_K128, 64, p, 3, (int)g_planes(s, K), s.B, st)) return e;
  }
  return 0;
}

// BWD_DW: P[slice][a*32 + l][(o*cH + hc)*32 + h] = sum over the slice's (b,row) range of Z16 chunk a = d*cC + lc [b][row][l] times
// V16 chunk (o, hc) [b][row][h]; that is P[slice][d*C + c][o*H + h'] in W's channel numbering
static int run_bwd_dw(const BdgcnShape& s, const __half* z16, const __half* v16, float* partials, int* slices_out, int* mt_out,
                      cudaStream_t st, bool bf = false) {
  const int rows = dw_row_chunks(s), cols = dw_col_chunks(s), pl = bf ? 2 : 1, passes = bf ? 3 : 1;
  const long long NN = (long long)rn(s);
  GemmParams p;
  init_params(p);
  if (int e = map_chunks(&p.a_map, z16, NN, 32, rows, NN * 32, (long long)s.B * pl, (long long)rows * NN * 32, 64, 4)) return e;
  if (int e = map_chunks(&p.b_map, v16, NN, 32, cols, NN * 32, (long long)s.B * pl, (long long)cols * NN * 32, 64, dw_chunks(cols))) return e;
  p.am = omap(1, 1, 0, 1, 0);           // z (slice) ignored; batch element = segment
  p.bm = omap(1, 1, 0, 1, 0);
  int per = 1, total = 1;
  const int slices = dw_slices(s, &per, &total, passes);      // split-K over every pass
  p.MT = ceil_div(rows, 4); p.NT = dw_col_tiles(cols); p.Z = slices; p.R = dw_chunks(cols);   // output chunk r = nt * R + j
  p.kb_total = total / passes; p.kb_per_seg = ceil_div(NN, 64);
  p.split_k = 1; p.kb_per_slice = per;
  p.ep.out = partials; p.ep.out_f16 = 0;
  p.ep.sZ = (long long)p.MT * 128 * cols * 32; p.ep.sI = (long long)cols * 32; p.ep.sR = 32;
  p.ep.m_valid = p.MT * 128; p.ep.r_valid = cols;
  *slices_out = slices;
  *mt_out = p.MT;
  prof_set_next(PROF_BWD_DW, 2.0 * s.B * (double)s.Ko * s.Kd * NN * s.C * s.H);
  return launch(bf, tc::A_MN64, 64, p, passes, s.B, s.B, st);
}

// BWD_DX: dX[b][n][c][32 lc + l] = sum_{d,e} G_d[c][e] Y16[b][d][lc][n][e][l]       n < R; one launch per input chunk lc
static int run_bwd_dx(const BdgcnShape& s, const __half* gd16, const __half* y16, float* dX, const float* inv_scale, float* dx_absmax,
                      cudaStream_t st, bool bf = false) {
  const int N = s.N, R = s.R, K = s.Kd, Np = pad8(N), C = s.C, cC = s.C / 32, pl = bf ? 2 : 1;
  const long long NN = (long long)rn(s);
  for (int lc = 0; lc < cC; ++lc) {
    GemmParams p;
    init_params(p);
    if (int e = map_support_k(&p.a_map, gd16, N, Np, (long long)g_planes(s, K) * pl)) return e;
    if (int e = map_chunks(&p.b_map, y16 + lc * NN * 32, N, 32, R, (long long)N * 32, (long long)s.B * K * cC * pl - lc, NN * 32, 64, 8)) return e;
    p.am = omap(1, s.dynamic ? kBig : 1, s.dynamic ? K : 0, 1, 0);   // support index = (b*K) + d
    p.bm = omap(1, kBig, K * cC, cC, 0);                              // plane = (b*K + d)*cC, from this chunk's base
    p.MT = ceil_div(N, 128); p.NT = ceil_div(R, 8); p.Z = s.B; p.R = 8;
    p.kb_per_seg = ceil_div(N, 64); p.kb_total = K * p.kb_per_seg;
    p.ep.out = dX + lc * 32; p.ep.out_f16 = 0; p.ep.alpha_dev = inv_scale; p.ep.absmax_out = dx_absmax;   // max over every chunk
    p.ep.sZ = (long long)R * N * C; p.ep.sI = C; p.ep.sR = (long long)N * C;
    p.ep.m_valid = N; p.ep.r_valid = R;
    prof_set_next(PROF_BWD_DX, 2.0 * s.B * K * (double)R * N * N * 32);
    if (int e = launch(bf, tc::A_K128, 64, p, 3, (int)g_planes(s, K), s.B * K * cC, st)) return e;
  }
  return 0;
}

// Prepared supports: [planes][N][Np] fp16 (padding zeroed) followed, 256-byte aligned, by the [planes][N] diagonal remainders.
// A caller that uses the same supports for several layers / for forward and backward converts them once.
// bf16x3: the [hi | lo] pair of [planes][N][Np] bf16 planes, no remainders.
static size_t prep_g16_bytes(long long planes, int N) { return align_up((size_t)planes * N * pad8(N) * sizeof(__half), 256); }
size_t bdgcn_supports_prepared_bytes(long long planes, int N, bool bf) {
  if (bf) return align_up((size_t)2 * planes * N * pad8(N) * sizeof(__half), 256);
  return prep_g16_bytes(planes, N) + align_up((size_t)planes * N * sizeof(float), 256);
}
int bdgcn_prepare_supports(const float* G, void* prepared, long long planes, int N, cudaStream_t st, bool bf) {
  MPGCN_CHECK((reinterpret_cast<uintptr_t>(prepared) & 255) == 0, "prepared-supports buffer must be 256-byte aligned");
  if (bf) return cvt_f32_to_bf16x3_padded(G, static_cast<__nv_bfloat16*>(prepared), (size_t)planes * N, N, pad8(N), st);
  __half* g16 = static_cast<__half*>(prepared);
  float* delta = reinterpret_cast<float*>(static_cast<uint8_t*>(prepared) + prep_g16_bytes(planes, N));
  if (int e = cvt_f32_to_f16_padded(G, g16, (size_t)planes * N, N, pad8(N), st)) return e;
  return support_diag_delta(G, delta, (size_t)planes, N, st);
}

// resolves the fp16 supports (and, for the forward, the diagonal remainders) of one side: prepared by the caller, shared
// with the other side (static graph: Go == Gd), or converted here into the workspace
struct SideG { const __half* g16; const float* delta; };
static int resolve_side(const BdgcnShape& s, int K, const float* G, const void* prepared, __half* ws16, float* ws_delta, bool want_delta,
                        SideG* out, cudaStream_t st, bool bf = false) {
  const long long planes = (long long)g_planes(s, K);
  if (bf) {         // a bf16x3 pair, no remainders
    MPGCN_CHECK((reinterpret_cast<uintptr_t>(prepared) & 255) == 0, "prepared-supports buffer must be 256-byte aligned");
    out->delta = nullptr;
    out->g16 = prepared ? static_cast<const __half*>(prepared) : ws16;
    if (prepared) return 0;
    return cvt_f32_to_bf16x3_padded(G, reinterpret_cast<__nv_bfloat16*>(ws16), (size_t)planes * s.N, s.N, pad8(s.N), st);
  }
  if (prepared) {
    MPGCN_CHECK((reinterpret_cast<uintptr_t>(prepared) & 255) == 0, "prepared-supports buffer must be 256-byte aligned");
    out->g16 = static_cast<const __half*>(prepared);
    out->delta = reinterpret_cast<const float*>(static_cast<const uint8_t*>(prepared) + prep_g16_bytes(planes, s.N));
    return 0;
  }
  if (int e = cvt_f32_to_f16_padded(G, ws16, (size_t)planes * s.N, s.N, pad8(s.N), st)) return e;
  if (want_delta) { if (int e = support_diag_delta(G, ws_delta, (size_t)planes, s.N, st)) return e; }
  out->g16 = ws16;
  out->delta = ws_delta;
  return 0;
}

// ---------------------------------------------------------------------------------------
// layer forward / backward
// ---------------------------------------------------------------------------------------
int bdgcn_forward_tc(const BdgcnShape& s, const float* X, const float* Go, const float* Gd, const float* W, const float* bias,
                     float* out, void* saved, void* ws, size_t ws_bytes, const BdgcnExtras& ex, cudaStream_t st, bool bf) {
  MPGCN_CHECK(tc_supported(s), "tensor-core path needs C and H to be multiples of 32 (H <= 1024) and Ko, Kd >= 1 (got C=%d H=%d Ko=%d Kd=%d)",
              s.C, s.H, s.Ko, s.Kd);
  MPGCN_CHECK(!bf || (s.whole() && ex.x_f16 == nullptr && ex.out_f16 == nullptr), "bf16x3: whole layers only, without fp16 side buffers");
  if (int e = check_index_range(s)) return e;
  const size_t NN = rn(s);
  const FwdLayout L = fwd_layout(s, bf);
  MPGCN_CHECK(ws_bytes >= L.total, "bdgcn_forward: workspace too small (%zu < %zu bytes)", ws_bytes, L.total);
  MPGCN_CHECK((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "workspace must be 256-byte aligned");
  uint8_t* wb = static_cast<uint8_t*>(ws);
  __half* x16_ws = reinterpret_cast<__half*>(wb + L.x16);
  __half* w16 = reinterpret_cast<__half*>(wb + L.w16);
  __half* u16 = reinterpret_cast<__half*>(wb + L.u16);
  __half* z16 = saved ? static_cast<__half*>(saved) : reinterpret_cast<__half*>(wb + L.z16);
  MPGCN_CHECK((reinterpret_cast<uintptr_t>(z16) & 63) == 0, "`saved` buffer must be 64-byte aligned");
  MPGCN_CHECK(((reinterpret_cast<uintptr_t>(ex.x_f16) | reinterpret_cast<uintptr_t>(ex.out_f16) | reinterpret_cast<uintptr_t>(out)) & 31) == 0,
              "bdgcn_forward: `out` and the fp16 side buffers must be 32-byte aligned (256-bit stores)");
  MPGCN_CHECK((reinterpret_cast<uintptr_t>(X) & 15) == 0, "bdgcn_forward: X must be 16-byte aligned");

  if (bf) {
    SideG gd{}, go{};
    if (int e = cvt_f32_to_bf16x3_padded(X, reinterpret_cast<__nv_bfloat16*>(x16_ws), (size_t)s.B * NN, s.C, s.C, st)) return e;
    if (int e = resolve_side(s, s.Kd, Gd, ex.gd_prepared, reinterpret_cast<__half*>(wb + L.gd16), nullptr, false, &gd, st, true)) return e;
    if (Go == Gd && ex.go_prepared == nullptr) go = gd;
    else if (int e = resolve_side(s, s.Ko, Go, ex.go_prepared, reinterpret_cast<__half*>(wb + L.go16), nullptr, false, &go, st, true)) return e;
    if (int e = permute_w_mix_bf16x3(W, reinterpret_cast<__nv_bfloat16*>(w16), 1, s.Ko, s.Kd, s.C, s.H, st)) return e;
    if (int e = run_fwd_a(s, gd.g16, x16_ws, z16, nullptr, st, true)) return e;
    if (int e = run_mix(s, z16, w16, 2, u16, PROF_FWD_MIX, s.Kd * (s.C / 32), s.Ko * (s.H / 32), st, true)) return e;
    return run_fwd_b(s, go.g16, u16, bias, out, nullptr, nullptr, st, true);
  }
  const __half* x16 = static_cast<const __half*>(ex.x_f16);
  if (x16 == nullptr) {
    if (int e = cvt_f32_to_f16(X, x16_ws, (size_t)s.B * NN * s.C, st)) return e;
    x16 = x16_ws;
  }
  SideG gd{}, go{};
  if (int e = resolve_side(s, s.Kd, Gd, ex.gd_prepared, reinterpret_cast<__half*>(wb + L.gd16), reinterpret_cast<float*>(wb + L.dd), true, &gd, st)) return e;
  if (Go == Gd && ex.go_prepared == nullptr && s.Ko == s.Kd) go = gd;
  else if (int e = resolve_side(s, s.Ko, Go, ex.go_prepared, reinterpret_cast<__half*>(wb + L.go16), reinterpret_cast<float*>(wb + L.dgo), true, &go, st)) return e;
  const float* delta_o = go.delta;
  if (!(s.R == s.N && s.row0 == 0)) {     // the origin-side remainder applies to the rows n = m of this slab only
    float* masked = reinterpret_cast<float*>(wb + L.dgo_masked);
    if (int e = mask_delta_rows(go.delta, masked, g_planes(s, s.Ko), s.N, s.row0, s.R, st)) return e;
    delta_o = masked;
  }
  if (int e = permute_w_mix(W, w16, w16 + (size_t)s.Ko * s.Kd * s.C * s.H, s.Ko, s.Kd, s.C, s.H, st)) return e;
  if (int e = run_fwd_a(s, gd.g16, x16, z16, gd.delta, st)) return e;
  if (int e = run_mix(s, z16, w16, 2, u16, PROF_FWD_MIX, s.Kd * (s.C / 32), s.Ko * (s.H / 32), st)) return e;
  if (int e = run_fwd_b(s, go.g16, u16, bias, out, static_cast<__half*>(ex.out_f16), delta_o, st)) return e;
  return 0;
}

// L: the layout, checked against the workspace; form_y: run BWD_MIX (Y16) even without dX (the support gradient reads it)
static int backward_tc_impl(const BdgcnShape& s, const float* d_out, const float* out, const float* Go, const float* Gd, const float* W,
                            const void* saved, float* dX, float* dW, float* db, void* ws, const BwdLayout& L, const BdgcnExtras& ex,
                            bool form_y, cudaStream_t st, bool bf = false) {
  MPGCN_CHECK(tc_supported(s), "tensor-core path needs C and H to be multiples of 32 (H <= 1024) and Ko, Kd >= 1 (got C=%d H=%d Ko=%d Kd=%d)",
              s.C, s.H, s.Ko, s.Kd);
  if (int e = check_index_range(s)) return e;
  MPGCN_CHECK(saved != nullptr, "bdgcn_backward: forward was run without a `saved` buffer");
  const int act = s.partial ? 0 : s.act;       // a partial call receives dPre: the mask was applied by the caller, after the exchange
  MPGCN_CHECK(out != nullptr || ex.out_f16 != nullptr || !act, "bdgcn_backward: the ReLU mask needs `out` or its fp16 copy");
  MPGCN_CHECK((reinterpret_cast<uintptr_t>(dX) & 31) == 0, "bdgcn_backward: dX must be 32-byte aligned (256-bit stores)");
  MPGCN_CHECK(((reinterpret_cast<uintptr_t>(d_out) | reinterpret_cast<uintptr_t>(out)) & 15) == 0, "bdgcn_backward: d_out / out must be 16-byte aligned");
  const size_t NNfull = (size_t)s.N * s.N;
  const __half* z16 = static_cast<const __half*>(saved);
  MPGCN_CHECK((reinterpret_cast<uintptr_t>(ws) & 255) == 0, "workspace must be 256-byte aligned");
  uint8_t* wb = static_cast<uint8_t*>(ws);
  float* db_slots = det_mode() ? reinterpret_cast<float*>(wb + L.db_slots) : nullptr;    // fixed-order bias gradient
  const __half* dp16 = reinterpret_cast<__half*>(wb + L.dp16);
  __half* v16 = reinterpret_cast<__half*>(wb + L.v16);
  __half* y16 = reinterpret_cast<__half*>(wb + L.y16);
  __half* wq16 = reinterpret_cast<__half*>(wb + L.wq16);
  float* partials = reinterpret_cast<float*>(wb + L.partials);
  const float* scale2 = reinterpret_cast<float*>(wb + L.scale);   // [S, 1/S]: power-of-two gradient scale (fp16 range)

  if (bf) {
    // bf16x3 keeps the power-of-two scale S of the fp16 path: exact in both directions, and harmless in bf16's range
    MPGCN_CHECK(s.whole() && ex.d_pre_f16 == nullptr && ex.out_f16 == nullptr, "bf16x3: whole layers only, without fp16 side buffers");
    MPGCN_CHECK(out != nullptr || !act, "bdgcn_backward: the ReLU mask needs `out`");
    float* scale2_ws = reinterpret_cast<float*>(wb + L.scale);
    if (int e = grad_scale_prepare(d_out, (size_t)s.B * NNfull * s.H, scale2_ws, ex.d_out_absmax, st)) return e;
    if (int e = relu_bwd_prep_bf16x3(d_out, out, act, reinterpret_cast<__nv_bfloat16*>(wb + L.dp16), db, (size_t)s.B * NNfull * s.H, s.H,
                                     scale2_ws, st, db_slots))
      return e;
    SideG gd{}, go{};
    const bool shared = Go == Gd && s.Ko == s.Kd;
    if (dX || shared) {
      if (int e = resolve_side(s, s.Kd, Gd, ex.gd_prepared, reinterpret_cast<__half*>(wb + L.gd16), nullptr, false, &gd, st, true)) return e;
    }
    if (shared && ex.go_prepared == nullptr) go = gd;
    else if (int e = resolve_side(s, s.Ko, Go, ex.go_prepared, reinterpret_cast<__half*>(wb + L.go16), nullptr, false, &go, st, true)) return e;
    if (int e = run_bwd_v(s, go.g16, dp16, v16, st, true)) return e;
    int slices = 0, mt = 0;
    if (int e = run_bwd_dw(s, z16, v16, partials, &slices, &mt, st, true)) return e;
    if (int e = reduce_dw_partials(partials, dW, slices, mt, s.Ko, s.Kd, s.C, s.H, scale2 + 1, st)) return e;
    if (dX) {
      if (ex.dx_absmax) MPGCN_CUDA(cudaMemsetAsync(ex.dx_absmax, 0, sizeof(float), st));
      if (int e = permute_w_mix_bf16x3(W, reinterpret_cast<__nv_bfloat16*>(wq16), 0, s.Ko, s.Kd, s.C, s.H, st)) return e;
      if (int e = run_mix(s, v16, wq16, 2, y16, PROF_BWD_MIX, s.Ko * (s.H / 32), s.Kd * (s.C / 32), st, true)) return e;
      if (int e = run_bwd_dx(s, gd.g16, y16, dX, scale2 + 1, ex.dx_absmax, st, true)) return e;
    }
    return 0;
  }
  if (ex.d_pre_f16 != nullptr) {
    // dPre arrives masked, scaled and cast (mpgcn_relu_backward_scatter_f16 wrote it into every rank's buffer): no pass over it here
    MPGCN_CHECK(s.partial && ex.d_pre_scale2 != nullptr, "bdgcn_backward: a prepared fp16 dPre needs a part call and its scale pair");
    MPGCN_CHECK((reinterpret_cast<uintptr_t>(ex.d_pre_f16) & 15) == 0, "bdgcn_backward: prepared fp16 dPre must be 16-byte aligned");
    dp16 = static_cast<const __half*>(ex.d_pre_f16);
    scale2 = ex.d_pre_scale2;
  } else {
    __half* dp16_ws = reinterpret_cast<__half*>(wb + L.dp16);
    float* scale2_ws = reinterpret_cast<float*>(wb + L.scale);
    if (int e = grad_scale_prepare(d_out, (size_t)s.B * NNfull * s.H, scale2_ws, ex.d_out_absmax, st)) return e;
    if (ex.out_f16 != nullptr && act) {
      if (int e = relu_bwd_prep_f16mask(d_out, static_cast<const __half*>(ex.out_f16), act, dp16_ws, db, (size_t)s.B * NNfull * s.H, s.H, scale2_ws, st,
                                        db_slots))
        return e;
    } else {
      if (int e = relu_bwd_prep(d_out, out, act, dp16_ws, nullptr, db, (size_t)s.B * NNfull * s.H, s.H, scale2_ws, st, db_slots)) return e;
    }
  }
  SideG gd{}, go{};
  const bool shared = Go == Gd && s.Ko == s.Kd;
  if (dX || shared) {
    if (int e = resolve_side(s, s.Kd, Gd, ex.gd_prepared, reinterpret_cast<__half*>(wb + L.gd16), nullptr, false, &gd, st)) return e;
  }
  if (shared && ex.go_prepared == nullptr) go = gd;
  else if (int e = resolve_side(s, s.Ko, Go, ex.go_prepared, reinterpret_cast<__half*>(wb + L.go16), nullptr, false, &go, st)) return e;
  if (int e = run_bwd_v(s, go.g16, dp16, v16, st)) return e;
  int slices = 0, mt = 0;
  if (int e = run_bwd_dw(s, z16, v16, partials, &slices, &mt, st)) return e;
  if (int e = reduce_dw_partials(partials, dW, slices, mt, s.Ko, s.Kd, s.C, s.H, scale2 + 1, st)) return e;
  if (dX || form_y) {
    if (dX && ex.dx_absmax) MPGCN_CUDA(cudaMemsetAsync(ex.dx_absmax, 0, sizeof(float), st));
    if (int e = permute_w_mix(W, wq16, nullptr, s.Ko, s.Kd, s.C, s.H, st)) return e;
    if (int e = run_mix(s, v16, wq16, 1, y16, PROF_BWD_MIX, s.Ko * (s.H / 32), s.Kd * (s.C / 32), st)) return e;
    if (dX) { if (int e = run_bwd_dx(s, gd.g16, y16, dX, scale2 + 1, ex.dx_absmax, st)) return e; }
  }
  return 0;
}

int bdgcn_backward_tc(const BdgcnShape& s, const float* d_out, const float* out, const float* Go, const float* Gd, const float* W,
                      const void* saved, float* dX, float* dW, float* db, void* ws, size_t ws_bytes, const BdgcnExtras& ex,
                      cudaStream_t st, bool bf) {
  const BwdLayout L = bwd_layout(s, false, bf);
  MPGCN_CHECK(ws_bytes >= L.total, "bdgcn_backward: workspace too small (%zu < %zu bytes)", ws_bytes, L.total);
  return backward_tc_impl(s, d_out, out, Go, Gd, W, saved, dX, dW, db, ws, L, ex, false, st, bf);
}

// One support-gradient contraction into the partials [slice][N][ldp] (ldp = 32 ceil(N/32): a 32-column chunk never runs into
// the next row), then reduced into dG [N][N].  A is K-major SW64 (one 32-wide k block per k-block), B K-major.
static int run_dg(const BdgcnShape& s, GemmParams& p, int kb_total, int kb_per_seg, double flops, float* partials, float* dG,
                  const float* inv_scale, int accumulate, cudaStream_t st) {
  const int N = s.N, ldp = 32 * dg_chunks(s);
  int per = ceil_div(kb_total, dg_max_slices(s));
  if (per < 1) per = 1;
  const int slices = ceil_div(kb_total, per);
  p.R = dg_r(s); p.MT = ceil_div(N, 128); p.NT = ceil_div(dg_chunks(s), p.R); p.Z = slices;
  p.kb_total = kb_total; p.kb_per_seg = kb_per_seg;
  p.split_k = 1; p.kb_per_slice = per;
  p.ep.out = partials; p.ep.out_f16 = 0;
  p.ep.sZ = (long long)N * ldp; p.ep.sI = ldp; p.ep.sR = 32;
  p.ep.m_valid = N; p.ep.r_valid = dg_chunks(s);
  prof_set_next(PROF_BWD_DG, flops);
  if (int e = tc::launch_contract_bkm(p, st)) return e;
  return reduce_dg_partials(partials, dG, slices, N, ldp, inv_scale, accumulate, st);
}

// BWD_DGO, output plane o (sample b, or every sample summed when b < 0):
//   dG_o[n][m] = sum_{(b,) hc, e, h} U16[b][hc][o][n][e][h] dP16[b][m][e][32 hc + h]      k-block = (segment (b,) hc; e), 32 h
static int run_bwd_dgo(const BdgcnShape& s, const __half* u16, const __half* dp16, int b, int o, float* partials, float* dG,
                       const float* inv_scale, cudaStream_t st) {
  const int N = s.N, H = s.H, cH = s.H / 32, Ko = s.Ko;
  const long long NN = (long long)N * N;
  const long long plane0 = (long long)(b < 0 ? 0 : b) * cH * Ko + o;           // U16 plane (b*cH + hc)*Ko + o
  GemmParams p;
  init_params(p);
  {   // U16 planes [n][(e, h)] from plane0 on: dims ((e,h), n, plane)
    const uint64_t dims[4] = {(uint64_t)N * 32, (uint64_t)N, (uint64_t)((long long)s.B * cH * Ko - plane0), 1};
    const uint64_t str[3] = {(uint64_t)N * 64, (uint64_t)NN * 64, (uint64_t)NN * 64 * (uint64_t)((long long)s.B * cH * Ko - plane0)};
    const uint32_t box[4] = {32, 128, 1, 1};
    if (int e = make_tmap_f16(&p.a_map, u16 + plane0 * NN * 32, 4, dims, str, box, TMAP_SW64)) return e;
  }
  {   // dP16 [b][m][e][H]: dims (h, m, e, b), a box of 32 h x 32 R rows m
    const long long nb = b < 0 ? s.B : 1;
    const uint64_t dims[4] = {(uint64_t)H, (uint64_t)N, (uint64_t)N, (uint64_t)nb};
    const uint64_t str[3] = {(uint64_t)N * H * 2, (uint64_t)H * 2, (uint64_t)NN * H * 2};
    const uint32_t box[4] = {32, (uint32_t)(32 * dg_r(s)), 1, 1};
    if (int e = make_tmap_f16(&p.b_map, dp16 + (b < 0 ? 0 : (long long)b * NN * H), 4, dims, str, box, TMAP_SW64)) return e;
  }
  const int nseg = (b < 0 ? s.B : 1) * cH;              // segment = (b,) hc
  p.am = omap(1, 1, 0, Ko, 0);                           // plane0 + seg * Ko; k = e * 32
  p.bm = omap(1, 1, 0, 0, 32, cH, 1);                    // h = 32 (seg % cH); b = seg / cH; e = k-block in the segment
  const double flops = 2.0 * (b < 0 ? s.B : 1) * (double)NN * N * H;
  return run_dg(s, p, nseg * N, N, flops, partials, dG, inv_scale, 0, st);
}

// BWD_DGD, output plane d (sample b, or every sample summed when b < 0), added to dG when `accumulate`:
//   dG_d[c][e] = sum_{(b,) n, l} X16[b][n][c][l] Y16[b][d][lc][n][e][l - 32 lc]      k-block = (segment (b,) n; lc), 32 l
static int run_bwd_dgd(const BdgcnShape& s, const __half* x16, const __half* y16, int b, int d, float* partials, float* dG,
                       const float* inv_scale, int accumulate, cudaStream_t st) {
  const int N = s.N, C = s.C, cC = s.C / 32, Kd = s.Kd;
  const long long NN = (long long)N * N;
  GemmParams p;
  init_params(p);
  {   // X16 [(b,) n][c][C]: dims (C, c, (b,n))
    const long long planes = (long long)(b < 0 ? s.B : 1) * N;
    const uint64_t dims[4] = {(uint64_t)C, (uint64_t)N, (uint64_t)planes, 1};
    const uint64_t str[3] = {(uint64_t)C * 2, (uint64_t)N * C * 2, (uint64_t)N * C * 2 * (uint64_t)planes};
    const uint32_t box[4] = {32, 128, 1, 1};
    if (int e = make_tmap_f16(&p.a_map, x16 + (b < 0 ? 0 : (long long)b * NN * C), 4, dims, str, box, TMAP_SW64)) return e;
  }
  {   // Y16 [b][d][lc][n][e][32] from plane (b*Kd + d)*cC on: dims (l, e, lc, flat (b, n) = b*Kd*cC*N + n), a box of 32 l x 32 R rows e
    const long long plane0 = ((long long)(b < 0 ? 0 : b) * Kd + d) * cC;
    const uint64_t flat = (uint64_t)(((long long)s.B * Kd * cC - plane0) * N);
    const uint64_t dims[4] = {32, (uint64_t)N, (uint64_t)cC, flat};
    const uint64_t str[3] = {64, (uint64_t)NN * 64, (uint64_t)N * 64};
    const uint32_t box[4] = {32, (uint32_t)(32 * dg_r(s)), 1, 1};
    if (int e = make_tmap_f16(&p.b_map, y16 + plane0 * NN * 32, 4, dims, str, box, TMAP_SW64)) return e;
  }
  const int nseg = (b < 0 ? s.B : 1) * N;                // segment = (b,) n
  p.am = omap(1, 1, 0, 1, 0);                            // X plane b*N + n = seg; k = lc * 32
  p.bm = omap(1, 1, 0, 1, 0, N, Kd * cC * N);            // flat n + b*Kd*cC*N; lc = k-block in the segment
  const double flops = 2.0 * (b < 0 ? s.B : 1) * (double)NN * N * C;
  return run_dg(s, p, nseg * cC, cC, flops, partials, dG, inv_scale, accumulate, st);
}

int bdgcn_backward_supports_tc(const BdgcnShape& s, const float* d_out, const float* out, const float* X, const float* Go, const float* Gd,
                               const float* W, const void* saved, float* dX, float* dW, float* db, float* dGo, float* dGd, void* ws,
                               size_t ws_bytes, const BdgcnExtras& ex, cudaStream_t st) {
  MPGCN_CHECK(s.whole(), "support gradients: whole layers only");
  MPGCN_CHECK(ex.d_pre_f16 == nullptr, "support gradients: a prepared fp16 dPre belongs to a layer part");
  const BwdLayout L = bwd_layout(s, true);
  MPGCN_CHECK(ws_bytes >= L.total, "bdgcn_backward_supports: workspace too small (%zu < %zu bytes)", ws_bytes, L.total);
  MPGCN_CHECK((reinterpret_cast<uintptr_t>(X) & 15) == 0, "bdgcn_backward_supports: X must be 16-byte aligned");
  const bool want_d = dGd != nullptr || (!s.dynamic && dGo != nullptr);
  if (int e = backward_tc_impl(s, d_out, out, Go, Gd, W, saved, dX, dW, db, ws, L, ex, want_d, st)) return e;
  uint8_t* wb = static_cast<uint8_t*>(ws);
  const __half* z16 = static_cast<const __half*>(saved);
  const __half* dp16 = reinterpret_cast<const __half*>(wb + L.dp16);
  const __half* y16 = reinterpret_cast<const __half*>(wb + L.y16);
  const float* inv_scale = reinterpret_cast<const float*>(wb + L.scale) + 1;
  __half* x16 = reinterpret_cast<__half*>(wb + L.x16);
  __half* u16 = reinterpret_cast<__half*>(wb + L.u16);
  __half* w16 = reinterpret_cast<__half*>(wb + L.w16);
  float* partials = reinterpret_cast<float*>(wb + L.dg_partials);
  const size_t NN = (size_t)s.N * s.N;
  if (dGo) {   // U16 again, as the forward formed it (FWD_MIX of the saved Z16)
    if (int e = permute_w_mix(W, w16, w16 + (size_t)s.Ko * s.Kd * s.C * s.H, s.Ko, s.Kd, s.C, s.H, st)) return e;
    if (int e = run_mix(s, z16, w16, 2, u16, PROF_BWD_DG, s.Kd * (s.C / 32), s.Ko * (s.H / 32), st)) return e;
    for (int b = s.dynamic ? 0 : -1; b < (s.dynamic ? s.B : 0); ++b)
      for (int o = 0; o < s.Ko; ++o) {
        float* dst = dGo + ((size_t)(b < 0 ? 0 : b) * s.Ko + o) * NN;
        if (int e = run_bwd_dgo(s, u16, dp16, b, o, partials, dst, inv_scale, st)) return e;
      }
  }
  if (want_d) {
    if (int e = cvt_f32_to_f16(X, x16, (size_t)s.B * NN * s.C, st)) return e;
    float* base = s.dynamic ? dGd : dGo;                   // static supports: G_d is G_o, one gradient
    for (int b = s.dynamic ? 0 : -1; b < (s.dynamic ? s.B : 0); ++b)
      for (int d = 0; d < s.Kd; ++d) {
        float* dst = base + ((size_t)(b < 0 ? 0 : b) * s.Kd + d) * NN;
        if (int e = run_bwd_dgd(s, x16, y16, b, d, partials, dst, inv_scale, s.dynamic ? 0 : 1, st)) return e;
      }
  }
  return 0;
}

}  // namespace mpgcn
