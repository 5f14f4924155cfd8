// wgmma / TMA contraction engine: one persistent, warp-specialised kernel template that
// evaluates every tensor-core contraction of the BDGCN layer (forward and backward).
//
//   D[z][i][(r,ch)] = alpha * sum_k A_z[k or i major] * B_z[k][(r,ch)]   (+ bias[ch], ReLU)
//
// * fp16 operands (or bf16 pairs in three passes: bf16x3, precision 2), fp32 accumulation in registers, M = 128 rows per tile (two consumer warpgroups of
//   64 rows each), N = 32*R columns per tile (R <= 8 "channel chunks" of 32 = one 64-byte swizzle row).
// * operands are staged by TMA into a multi-stage shared-memory ring in exactly the
//   canonical wgmma layouts, so no thread ever touches operand bytes:
//     A_MN128 : A is [k][m], m contiguous      (G_d for  Z = X x2 G_d ; G_o flat for  pre = sum G_o^T U)
//     A_K128  : A is [m][k], k contiguous      (G_o for  V = G_o x1 dPre ; G_d for dX)
//     A_K64   : A is [m][32], one 32-wide k block per plane (channel mixes Z->U, V->Y)
//     A_MN64  : A is [k][chunk][32]            (Z for the weight gradient dW = Z^T V)
//     B       : [k][chunk r][32 ch], 64-byte rows, SWIZZLE_64B, MN-major; or, with BKM (A_K64, BK = 32 only), K-major
//               [32 r rows][32 k], 64-byte rows, SWIZZLE_64B (the support-gradient products dG = U dPre^T and X Y^T, whose
//               reduction runs over the channels: both operands have it contiguous)
// * warpgroups 0 and 1 = MMA + epilogue of rows 0..63 / 64..127 of the tile.  Thread 0 also issues the TMA loads: it fills
//   the ring, then refills each stage as soon as both warpgroups released it, so loads run up to `stages` k-blocks (into the
//   next tile as well) ahead of the MMAs.  (A separate producer warp takes the CTA past 256 threads, which caps registers at
//   168 per thread unless setmaxnreg hands the consumers up to 232; that split has not been tried.)
// * the epilogue writes each 64-row x 32-channel chunk of the result, converted, into one of two shared-memory store buffers
//   per warpgroup and stores it by TMA (cp.async.bulk.tensor, bulk-group completion): the stores drain while the next tile's
//   MMAs run, and partial tiles are clipped by the output tensor map.
//
// Reference math being evaluated: BDGCN.forward of the reference MPGCN.py, in the factored order of SURVEY.md section 7.1.
#pragma once

#include "common.cuh"
#include "wgmma.cuh"

#include <type_traits>

namespace mpgcn {
namespace tc {

enum AKind : int { A_MN128 = 0, A_K128 = 1, A_K64 = 2, A_MN64 = 3 };

// tile/k-block -> TMA coordinate map of one operand
struct OperandMap {
  int z_div, z_mod, z_mul;   // z' = ((z / z_div) % z_mod) * z_mul + (seg % seg_mod) * seg_mul + (seg / seg_mod) * seg_hi_mul
  int seg_mod, seg_mul, seg_hi_mul;
  int k_seg;                 // k coordinate (elements) += (seg % seg_mod) * k_seg
};

struct Epilogue {
  void* out;                 // float* or __half*
  __half* out16;             // optional fp16 shadow of a float output (same strides), may be null
  long long sZ, sI, sR;      // element strides of z, row i, chunk r (channel stride is 1)
  int m_valid, r_valid;      // bounds on i and r
  int out_f16;               // 1: out is __half
  int relu;
  const float* bias;         // [32] or null
  float alpha;
  const float* alpha_dev;    // optional device scalar multiplied into alpha (gradient un-scaling), may be null
  float* absmax_out;         // optional device scalar (pre-zeroed): receives max |stored value| (bit pattern, atomicMax)
  // optional diagonal correction (forward only): out[z][i][r][:] += sum_seg delta[(zA*corr_nseg + seg)*m_valid + i] *
  // corr_src[zB*cZ + seg*cSeg + i*cI + r*cR + :], the exact remainder of the support diagonal lost by its fp16 rounding
  const __half* corr_src;
  const float* corr_delta;
  long long cZ, cI, cR, cSeg;
  int corr_nseg;             // any count: the epilogue walks the segments 8 at a time
};

struct alignas(64) GemmParams {
  CUtensorMap a_map;
  CUtensorMap b_map;
  // the output as (32 ch, m_valid rows, r_valid chunks, Z) with the strides of `ep`, box one chunk of 64 rows; and its fp16
  // shadow.  Set by launch_contract from `ep`.
  CUtensorMap out_map;
  CUtensorMap out16_map;
  OperandMap am, bm;
  int MT, NT, Z;             // tile grid: tile id = (z * NT + nt) * MT + mt
  int R;                     // 32-column chunks per tile
  int kb_total, kb_per_seg;  // k-blocks over all segments / per segment
  int split_k, kb_per_slice; // split-K: z is a k-slice [z*kb_per_slice, ...)
  int stages;
  int st_bytes;              // one store buffer: a chunk of 64 rows in the output type (+ 4 KB fp16 shadow); set by launch_contract
  // resident B (channel mixes): the whole B operand -- b_res_reps * kb_total tiles, index rep * kb_total + kb -- is loaded
  // once per CTA and every A k-block is multiplied by its b_res_reps tiles (the fp16 hi / lo halves of W); 0 = B streams
  // through the ring with A.  Needs NT == 1, kb_per_seg == 1, no split-K, a z-independent B map.
  int b_res_reps;
  int z_inner;               // > 1: z = zo * z_inner + zi and zi varies right after the m-tiles (before the n-tiles): the z_inner
                             // contractions that share one B block (the K supports applied to one X16 / dP16 row block) run back to
                             // back, so that block is fetched from HBM once and then served from L2
  Epilogue ep;
  // bf16x3 (contract_kernel with T = __nv_bfloat16): every operand is a pair of bf16 planes, the lo plane a_plane_z / b_plane_z
  // TMA z coordinates after the hi one, and the k-blocks run in passes of kb_pass (kb_total = passes * kb_pass), pass p reading
  // A plane {hi, hi, lo}[p] and B plane {hi, lo, hi}[p].  With a resident B (the hi / lo halves of W as b_res_reps = 2) there
  // are two passes over A: hi meets both halves, lo meets W hi only.  Unused by the fp16 instances.
  int kb_pass;
  int a_plane_z, b_plane_z;
};

constexpr int kConsumerWGs = 2;                        // 64 tile rows each
constexpr int kThreads1 = 128 * kConsumerWGs;          // 256 threads: the 128 x 256 fp32 accumulator tile needs ~250 registers

template <int AK, int BK>
struct Cfg {
  // A_K64 with BK = 32 P: P planes per k-block, one [128 m][64 B] slab each (a single TMA box over the plane dimension)
  static constexpr int A_STAGE = (AK == A_MN128) ? BK * 256 : (AK == A_K128) ? 128 * 128 : (AK == A_K64) ? 128 * 64 * (BK / 32) : 4 * BK * 64;
  static constexpr bool A_MN = (AK == A_MN128) || (AK == A_MN64);
  // byte advance of the A descriptor start address per MMA (K = 16)
  static constexpr uint32_t A_KSTEP = (AK == A_MN128) ? 16 * 128 : (AK == A_MN64) ? 16 * 64 : 32;
  static constexpr uint32_t A_LBO = (AK == A_MN128) ? BK * 128 : (AK == A_MN64) ? BK * 64 : 16;
  static constexpr uint32_t A_SBO = (AK == A_MN128 || AK == A_K128) ? 1024 : 512;
  static constexpr uint32_t A_LAYOUT = (AK == A_MN128 || AK == A_K128) ? GMMA_SW128 : GMMA_SW64;
  static constexpr uint32_t B_KSTEP = 16 * 64;
  static constexpr uint32_t B_LBO = BK * 64;
  static constexpr uint32_t B_SBO = 512;
  static_assert(AK != A_K128 || BK == 64, "K-major SW128 rows hold exactly 64 halves");
  static_assert(AK != A_K64 || BK % 32 == 0, "K-major SW64 rows hold exactly 32 halves: BK counts whole planes");
  // byte offset of the rows [64 wg, 64 wg + 64) of the tile inside an A stage (the A operand of consumer warpgroup wg)
  static constexpr uint32_t A_WG = (AK == A_MN128) ? BK * 128 : (AK == A_K128) ? 64 * 128 : (AK == A_K64) ? 64 * 64 : 2 * BK * 64;
  // byte offset of the A descriptor for the k-th MMA (K = 16) of a k-block
  __host__ __device__ static constexpr uint32_t a_koff(int k) {
    return (AK == A_K64) ? (uint32_t)(k >> 1) * 8192u + (uint32_t)(k & 1) * 32u : (uint32_t)k * A_KSTEP;
  }
  static_assert(BK % 16 == 0, "wgmma K is 16 for fp16");
};

// shared memory of one CTA: the operand ring (or A ring + resident B), two store buffers of st_bytes per consumer warpgroup
__host__ __device__ inline size_t smem_bytes(int a_stage, int R, int BK, int stages, int b_resident_tiles, int st_bytes) {
  const size_t b_stage = (size_t)R * BK * 64;
  return 1024 /*align slack*/ + (size_t)stages * a_stage + (size_t)(b_resident_tiles ? b_resident_tiles : stages) * b_stage +
         (size_t)2 * kConsumerWGs * st_bytes + 512 /*barriers, bias*/;
}

#ifdef __CUDACC__
// tile id -> (m tile, n tile, z); see GemmParams::z_inner
__device__ __forceinline__ void decode_tile(const GemmParams& p, int t, int& mt, int& nt, int& z) {
  if (p.z_inner > 1) {
    mt = t % p.MT;
    int rest = t / p.MT;
    const int zi = rest % p.z_inner;
    rest /= p.z_inner;
    nt = rest % p.NT;
    z = (rest / p.NT) * p.z_inner + zi;
  } else {
    mt = t % p.MT;
    const int rest = t / p.MT;
    nt = rest % p.NT;
    z = rest / p.NT;
  }
}

__device__ __forceinline__ uint32_t pack_h2(float a, float b) { return f2h2_sat_bits(a, b); }   // an fp16 operand never holds inf

// T: the operand element type, __half (precision 1) or __nv_bfloat16 (precision 2, bf16x3: see GemmParams::kb_pass; a 16-bit
// output is written as a bf16 hi plane to out_map and a lo plane to out16_map)
template <int AK, int BK, bool BKM = false, class T = __half>
__global__ void __launch_bounds__(kThreads1, 1) contract_kernel(const __grid_constant__ GemmParams p) {
  using C = Cfg<AK, BK>;
  constexpr bool BF = std::is_same<T, __nv_bfloat16>::value;
  static_assert(!BF || !BKM, "bf16x3 has no K-major B contraction");
  static_assert(!BKM || (AK == A_K64 && BK == 32), "a K-major B tile is one 32-wide k block, paired with a K-major SW64 A");
  constexpr int A_STAGE = C::A_STAGE;
  const int R = p.R;
  const int B_STAGE = R * BK * 64;
  const int S = p.stages;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int kb_res = BF ? p.kb_pass : p.kb_total;   // k-blocks per resident B rep
  const int NRES = p.b_res_reps * kb_res;           // resident B tiles (0: B goes through the ring)
  uint8_t* sA = smem;
  uint8_t* sB = sA + (size_t)S * A_STAGE;
  uint8_t* sStore = sB + (size_t)(NRES ? NRES : S) * B_STAGE;     // 2 store buffers per consumer warpgroup
  uint64_t* full = reinterpret_cast<uint64_t*>(sStore + (size_t)2 * kConsumerWGs * p.st_bytes);
  uint64_t* empty = full + S;
  uint64_t* bres_full = empty + S;
  float* sbias = reinterpret_cast<float*>(bres_full + 1);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.a_map);
    tma_prefetch_desc(&p.b_map);
    tma_prefetch_desc(&p.out_map);
    for (int s = 0; s < S; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 4 * kConsumerWGs);     // one arrival per warp
    }
    mbar_init(bres_full, 1);
    fence_barrier_init();
  }
  if (warp == 0) sbias[lane] = p.ep.bias ? p.ep.bias[lane] : 0.f;
  __syncthreads();

  const int num_tiles = p.MT * p.NT * p.Z;

  // ------------------------------ TMA producer state (thread 0) ------------------------------
  // cursor over the (tile, k-block) sequence of this CTA; segment / k-block counters are advanced incrementally: the
  // channel-mix contractions spend only ~100 clk of MMA per k-block, so integer divisions per load would bound the kernel
  int p_t = blockIdx.x, p_kb = 0, p_kb1 = 0, p_kk = 0, p_sa_lo = 0, p_sa_hi = 0, p_sb_lo = 0, p_sb_hi = 0, p_zA0 = 0, p_zB0 = 0, p_mt = 0, p_nt = 0;
  int p_stage = 0;
  uint32_t p_phase = 0;
  int p_pass = 0, p_pass_end = 0;   // bf16x3: pass of k-block p_kb, and the k-block that starts the next one
  auto p_start_tile = [&]() {
    int z;
    decode_tile(p, p_t, p_mt, p_nt, z);
    p_kb = p.split_k ? z * p.kb_per_slice : 0;
    p_kb1 = p.split_k ? min(p_kb + p.kb_per_slice, p.kb_total) : p.kb_total;
    p_zA0 = ((z / p.am.z_div) % p.am.z_mod) * p.am.z_mul;
    p_zB0 = ((z / p.bm.z_div) % p.bm.z_mod) * p.bm.z_mul;
    int kin = p_kb;                 // k-block within the pass
    if constexpr (BF) {
      p_pass = p_kb / p.kb_pass;
      p_pass_end = (p_pass + 1) * p.kb_pass;
      kin = p_kb - p_pass * p.kb_pass;
    }
    const int seg = kin / p.kb_per_seg;
    p_kk = kin - seg * p.kb_per_seg;
    p_sa_lo = seg % p.am.seg_mod; p_sa_hi = seg / p.am.seg_mod;
    p_sb_lo = seg % p.bm.seg_mod; p_sb_hi = seg / p.bm.seg_mod;
  };
  // issue the loads of the next k-block into the next ring stage (waits until both warpgroups released that stage)
  auto produce = [&]() {
    if (p_t >= num_tiles) return;
    mbar_wait_inline(&empty[p_stage], p_phase ^ 1u);
    mbar_arrive_expect_tx(&full[p_stage], (uint32_t)(A_STAGE + (NRES ? 0 : B_STAGE)));
    int zA = p_zA0 + p_sa_lo * p.am.seg_mul + p_sa_hi * p.am.seg_hi_mul;
    int zB = p_zB0 + p_sb_lo * p.bm.seg_mul + p_sb_hi * p.bm.seg_hi_mul;
    if constexpr (BF) {             // the pass's planes: A {hi, hi, lo}, B {hi, lo, hi} (resident B: A {hi, lo})
      zA += (NRES ? p_pass : p_pass >> 1) * p.a_plane_z;
      zB += (p_pass & 1) * p.b_plane_z;
    }
    const int kA = p_kk * BK + p_sa_lo * p.am.k_seg;
    const int kB = p_kk * BK + p_sb_lo * p.bm.k_seg;
    uint8_t* a_dst = sA + (size_t)p_stage * A_STAGE;
    uint8_t* b_dst = sB + (size_t)p_stage * B_STAGE;
    if (AK == A_MN128) {          // dims (m, k, z, 1), two 64-wide m boxes
      tma_load_4d(a_dst, &p.a_map, &full[p_stage], p_mt * 128, kA, zA, 0);
      tma_load_4d(a_dst + BK * 128, &p.a_map, &full[p_stage], p_mt * 128 + 64, kA, zA, 0);
    } else if (AK == A_K128 || AK == A_K64) {   // dims (k, m, z, 1)
      tma_load_4d(a_dst, &p.a_map, &full[p_stage], kA, p_mt * 128, zA, 0);
    } else {                      // A_MN64: dims (ch, k, chunk, z), 4 chunks per tile
      tma_load_4d(a_dst, &p.a_map, &full[p_stage], 0, kA, p_mt * 4, zA);
    }
    if constexpr (BKM)            // dims (k within the block, n row, k-block, z): the segment's k offset selects a 32-wide chunk
      tma_load_4d(b_dst, &p.b_map, &full[p_stage], p_sb_lo * p.bm.k_seg, p_nt * R * 32, p_kk, zB);
    else if (!NRES)               // dims (ch, k, r, z); a resident B was loaded once up front
      tma_load_4d(b_dst, &p.b_map, &full[p_stage], 0, kB, p_nt * R, zB);
    if (++p_stage == S) { p_stage = 0; p_phase ^= 1u; }
    if (++p_kk == p.kb_per_seg) {
      p_kk = 0;
      if (++p_sa_lo == p.am.seg_mod) { p_sa_lo = 0; ++p_sa_hi; }
      if (++p_sb_lo == p.bm.seg_mod) { p_sb_lo = 0; ++p_sb_hi; }
    }
    if constexpr (BF) {
      if (p_kb + 1 == p_pass_end) {    // the next pass starts again at segment 0
        ++p_pass;
        p_pass_end += p.kb_pass;
        p_kk = p_sa_lo = p_sa_hi = p_sb_lo = p_sb_hi = 0;
      }
    }
    if (++p_kb == p_kb1) {
      p_t += gridDim.x;
      if (p_t < num_tiles) p_start_tile();
    }
  };
  if (threadIdx.x == 0 && (int)blockIdx.x < num_tiles) {
    if (NRES) {                   // the whole B operand, once
      mbar_arrive_expect_tx(bres_full, (uint32_t)(NRES * B_STAGE));
      for (int sg = 0; sg < NRES; ++sg) {
        const int lo = sg % p.bm.seg_mod, hi = sg / p.bm.seg_mod;
        tma_load_4d(sB + (size_t)sg * B_STAGE, &p.b_map, bres_full, 0, lo * p.bm.k_seg, 0, lo * p.bm.seg_mul + hi * p.bm.seg_hi_mul);
      }
    }
    p_start_tile();
    for (int s = 0; s < S; ++s) produce();
  }
  __syncwarp();

  {
    // ------------------------------ MMA + epilogue (warpgroup wg: tile rows 64 wg .. 64 wg + 63) ------------------------------
    const int wg = warp >> 2;
    const int tw = threadIdx.x & 127;   // thread within the warpgroup
    const int wq = warp & 3, g = lane >> 2, q = lane & 3;
    const float alpha = p.ep.alpha_dev ? p.ep.alpha * __ldg(p.ep.alpha_dev) : p.ep.alpha;
    const uint64_t a_hi = gmma_desc_hi(C::A_SBO, C::A_LAYOUT);
    const uint64_t b_hi = gmma_desc_hi(C::B_SBO, GMMA_SW64);
    uint32_t st_seq = 0;                // store buffers used so far by this warpgroup: buffer st_seq & 1 is next
    float amax = 0.f;
    float acc[128];
    int stage = 0;
    uint32_t phase = 0;
    if (NRES && (int)blockIdx.x < num_tiles) mbar_wait_inline(bres_full, 0);
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      int mt, nt, z;
      decode_tile(p, t, mt, nt, z);
      const int kb0 = p.split_k ? z * p.kb_per_slice : 0;
      const int kb1 = p.split_k ? min(kb0 + p.kb_per_slice, p.kb_total) : p.kb_total;
      // one k-block of MMAs stays in flight: a stage is released (and refilled by thread 0) once the MMAs of the NEXT k-block
      // are issued and wgmma.wait_group 1 has retired the ones that read it
      int prev = -1;
      int c_pass = 0, c_pass_end = 0;       // bf16x3: the pass of kb (a resident B is indexed by the k-block within it)
      if constexpr (BF) {
        c_pass = kb0 / p.kb_pass;
        c_pass_end = (c_pass + 1) * p.kb_pass;
      }
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait_inline(&full[stage], phase);
        const uint32_t a_addr = smem_u32(sA + (size_t)stage * A_STAGE) + C::A_WG * (uint32_t)wg;
        int reps = NRES ? p.b_res_reps : 1;
        int kin = kb;
        if constexpr (BF) {
          if (kb == c_pass_end) { ++c_pass; c_pass_end += p.kb_pass; }
          kin = kb - c_pass * p.kb_pass;
          if (c_pass > 0) reps = 1;         // the lo plane of A meets W hi only
        }
        wgmma_fence();
        for (int rep = 0; rep < reps; ++rep) {
          const uint32_t b_addr = smem_u32(sB + (size_t)(NRES ? rep * kb_res + kin : stage) * B_STAGE);
          const int first = (kb == kb0 && rep == 0) ? 1 : 0;
          // one dispatch on the tile width per k-block: the BK / 16 MMAs of a case then chain on the same registers
          auto kblock = [&](auto width) {
            constexpr int RW = decltype(width)::value;
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) {
              const uint64_t ad = gmma_desc(a_hi, a_addr + C::a_koff(k), C::A_LBO);
              // K-major B: the k-th 16 halves of each 64-byte row (8-row core matrices 512 B apart, as the K-major A_K64 tile)
              const uint64_t bd = BKM ? gmma_desc(b_hi, b_addr + k * 32, 16) : gmma_desc(b_hi, b_addr + k * C::B_KSTEP, C::B_LBO);
              wgmma_n<RW, C::A_MN ? 1 : 0, BKM ? 0 : 1, T>(acc, ad, bd, (first && k == 0) ? 0 : 1);
            }
          };
          switch (R) {
            case 1: kblock(std::integral_constant<int, 1>()); break;
            case 2: kblock(std::integral_constant<int, 2>()); break;
            case 3: kblock(std::integral_constant<int, 3>()); break;
            case 4: kblock(std::integral_constant<int, 4>()); break;
            case 5: kblock(std::integral_constant<int, 5>()); break;
            case 6: kblock(std::integral_constant<int, 6>()); break;
            case 7: kblock(std::integral_constant<int, 7>()); break;
            default: kblock(std::integral_constant<int, 8>()); break;
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty[prev]);    // this warp's reads of that stage are complete
          if (threadIdx.x == 0) produce();              // refill it with the k-block S ahead
          __syncwarp();
        }
        prev = stage;
        if (++stage == S) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev]);
        if (threadIdx.x == 0) produce();
        __syncwarp();
      }
      // ---- epilogue: chunk by chunk straight from the accumulator fragment into a store buffer in the output's layout, which
      // one thread then writes out by TMA.  The MMAs of the next tile start while that store is in flight.  Per element the
      // same operations as a row-wise pass, in the same order: correction FMAs by segment, * alpha, + bias, ReLU, conversion.
      const int row0 = mt * 128 + wg * 64;     // first output row of this warpgroup; the tensor maps clip rows >= m_valid
      int ii[2];
      long long cbase[2] = {0, 0};
      const float* dsrc[2] = {nullptr, nullptr};   // delta of segment 0 of row ii[h]: segment sg at dsrc[h][sg * m_valid]
      // the remainders of the first 8 segments stay in registers for the whole tile; those of segments 8.. (more than 8
      // supports) are re-read per chunk, 8 at a time
      float dl[2][8];
      bool any_corr[2] = {false, false};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        ii[h] = row0 + 16 * wq + g + 8 * h;
        if (p.ep.corr_src != nullptr) {
          const int zA = ((z / p.am.z_div) % p.am.z_mod) * p.am.z_mul;
          const int zB = ((z / p.bm.z_div) % p.bm.z_mod) * p.bm.z_mul;
          cbase[h] = (long long)zB * p.ep.cZ + (long long)ii[h] * p.ep.cI;
          dsrc[h] = p.ep.corr_delta + (long long)zA * p.ep.corr_nseg * p.ep.m_valid + ii[h];
#pragma unroll
          for (int sgi = 0; sgi < 8; ++sgi) {
            dl[h][sgi] = (sgi < p.ep.corr_nseg && ii[h] < p.ep.m_valid) ? __ldg(dsrc[h] + (long long)sgi * p.ep.m_valid) : 0.f;
            any_corr[h] |= (dl[h][sgi] != 0.f);
          }
          for (int sg = 8; sg < p.ep.corr_nseg && !any_corr[h] && ii[h] < p.ep.m_valid; ++sg)
            any_corr[h] = __ldg(dsrc[h] + (long long)sg * p.ep.m_valid) != 0.f;
        } else {
#pragma unroll
          for (int sgi = 0; sgi < 8; ++sgi) dl[h][sgi] = 0.f;
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (j < R) {
          const int r = nt * R + j;
          // accumulator fragment: acc[16 j + 4 jj + 2 h + e] = D[row 16 wq + g + 8 h][column 32 j + 8 jj + 2 q + e]
          float v[16];
#pragma unroll
          for (int c = 0; c < 16; ++c) v[c] = acc[16 * j + c];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if (!any_corr[h] || ii[h] >= p.ep.m_valid || r >= p.ep.r_valid) continue;
            // segments in groups of 8 (one group for <= 8 supports), in segment order
            for (int sg0 = 0; sg0 < p.ep.corr_nseg; sg0 += 8) {
              float dg[8];
#pragma unroll
              for (int sgi = 0; sgi < 8; ++sgi)
                dg[sgi] = sg0 == 0 ? dl[h][sgi] : (sg0 + sgi < p.ep.corr_nseg ? __ldg(dsrc[h] + (long long)(sg0 + sgi) * p.ep.m_valid) : 0.f);
#pragma unroll
              for (int sgi = 0; sgi < 8; ++sgi) {
                if (sg0 + sgi < p.ep.corr_nseg && dg[sgi] != 0.f) {
                  const __half2* src = reinterpret_cast<const __half2*>(p.ep.corr_src + cbase[h] + (long long)(sg0 + sgi) * p.ep.cSeg +
                                                                        (long long)r * p.ep.cR) + q;
#pragma unroll
                  for (int jj = 0; jj < 4; ++jj) {
                    const float2 f = __half22float2(__ldg(src + 4 * jj));
                    v[4 * jj + 2 * h] = fmaf(dg[sgi], f.x, v[4 * jj + 2 * h]);
                    v[4 * jj + 2 * h + 1] = fmaf(dg[sgi], f.y, v[4 * jj + 2 * h + 1]);
                  }
                }
              }
            }
          }
#pragma unroll
          for (int c = 0; c < 16; ++c) {
            float x = v[c] * alpha;
            if (p.ep.bias) x += sbias[8 * (c >> 2) + 2 * q + (c & 1)];
            if (p.ep.relu) x = fmaxf(x, 0.f);
            v[c] = x;
          }
          if (p.ep.absmax_out && r < p.ep.r_valid) {
#pragma unroll
            for (int c = 0; c < 16; ++c)
              if (ii[(c >> 1) & 1] < p.ep.m_valid) amax = fmaxf(amax, fabsf(v[c]));
          }
          // store buffer of this chunk: [64 rows][32 channels], 128-byte rows SWIZZLE_128B (fp32) or 64-byte rows SWIZZLE_64B
          // (fp16), the fp16 shadow of an fp32 output 8 KB behind; conflict-free fragment writes
          uint8_t* buf = sStore + (size_t)(wg * 2 + (st_seq & 1)) * p.st_bytes;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint32_t rho = 16 * wq + g + 8 * h;
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const uint32_t o16 = (rho * 64 + 16 * jj + 4 * q) ^ (((rho >> 1) & 3) << 4);
              if constexpr (BF) {         // a 16-bit output is a bf16 pair: hi plane, and 4 KB behind it the lo plane
                if (p.ep.out_f16) {
                  uint32_t hi2, lo2;
                  split_bf16x2(v[4 * jj + 2 * h], v[4 * jj + 2 * h + 1], hi2, lo2);
                  *reinterpret_cast<uint32_t*>(buf + o16) = hi2;
                  *reinterpret_cast<uint32_t*>(buf + 4096 + o16) = lo2;
                } else {
                  const uint32_t o32 = (rho * 128 + 32 * jj + 8 * q) ^ ((rho & 7) << 4);
                  *reinterpret_cast<float2*>(buf + o32) = make_float2(v[4 * jj + 2 * h], v[4 * jj + 2 * h + 1]);
                }
                continue;
              }
              const uint32_t h2 = pack_h2(v[4 * jj + 2 * h], v[4 * jj + 2 * h + 1]);
              if (p.ep.out_f16) {
                *reinterpret_cast<uint32_t*>(buf + o16) = h2;
              } else {
                const uint32_t o32 = (rho * 128 + 32 * jj + 8 * q) ^ ((rho & 7) << 4);
                *reinterpret_cast<float2*>(buf + o32) = make_float2(v[4 * jj + 2 * h], v[4 * jj + 2 * h + 1]);
                if (p.ep.out16) *reinterpret_cast<uint32_t*>(buf + 8192 + o16) = h2;
              }
            }
          }
          fence_proxy_async_smem();                 // the generic-proxy writes above, before the TMA engine reads them
          if (tw == 0) bulk_wait_read<0>();         // the other buffer's store has read it: it may be rewritten after the barrier
          named_bar_sync(1 + wg, 128);
          if (tw == 0) {
            tma_store_4d(&p.out_map, buf, 0, row0, r, z);
            if constexpr (BF) {
              if (p.ep.out_f16) tma_store_4d(&p.out16_map, buf + 4096, 0, row0, r, z);
            } else if (!p.ep.out_f16 && p.ep.out16) {
              tma_store_4d(&p.out16_map, buf + 8192, 0, row0, r, z);
            }
            bulk_commit();
          }
          ++st_seq;
        }
      }
    }
    if (tw == 0) bulk_wait_all();                   // shared memory must outlive the last stores
    if (p.ep.absmax_out) {
      for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
      if (lane == 0) atomicMax(reinterpret_cast<unsigned int*>(p.ep.absmax_out), __float_as_uint(amax));
    }
  }
}
#endif  // __CUDACC__

// Launch one contraction (implemented in tc_engine.cu).  ak/bk select the instantiation.
int launch_contract(int ak, int bk, GemmParams& p, cudaStream_t stream);
// the same with a K-major B operand (A_K64, BK = 32; no resident B)
int launch_contract_bkm(GemmParams& p, cudaStream_t stream);
// bf16x3 (precision 2): bf16 pair operands in passes, see GemmParams::kb_pass; the A kinds / BKs of launch_contract
int launch_contract_bf16x3(int ak, int bk, GemmParams& p, cudaStream_t stream);

}  // namespace tc
}  // namespace mpgcn
