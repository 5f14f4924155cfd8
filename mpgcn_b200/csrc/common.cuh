// Shared device/host helpers for the mpgcn_b200 CUDA library (sm_90a only).
//
// PTX wrappers for the Hopper primitives the kernels use: mbarrier, TMA
// (cp.async.bulk.tensor), wgmma (warpgroup MMA), mma.sync / ldmatrix.  Nothing here is
// reference code; the reference (underdoc-wang/MPGCN) has no native code at all.
#pragma once

#include <cuda.h>            // CUtensorMap (types only; libcuda is resolved at run time)
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#if defined(__CUDA_ARCH__) && !defined(__CUDA_ARCH_FEAT_SM90_ALL)
#error "mpgcn_b200 must be compiled for sm_90a (-gencode arch=compute_90a,code=sm_90a)"
#endif

namespace mpgcn {

// ----------------------------------------------------------------------------------------
// host-side error plumbing (C-ABI functions return int, message via mpgcn_last_error())
// ----------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
#define MPGCN_CHECK(cond, ...)                                                     \
  do {                                                                             \
    if (!(cond)) {                                                                 \
      ::mpgcn::set_error(__VA_ARGS__);                                             \
      return 1;                                                                    \
    }                                                                              \
  } while (0)
#define MPGCN_CUDA(call)                                                           \
  do {                                                                             \
    cudaError_t e__ = (call);                                                      \
    if (e__ != cudaSuccess) {                                                      \
      ::mpgcn::set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
      return 2;                                                                    \
    }                                                                              \
  } while (0)

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Each workspace has one layout function: a struct of region offsets plus `total`, read by its size query and by its call.
// take() places a region of `bytes` at the first multiple of `align` at or after `off` and moves `off` to its end.
static inline size_t take(size_t& off, size_t bytes, size_t align) {
  off = align_up(off, align);
  const size_t r = off;
  off += bytes;
  return r;
}

// ----------------------------------------------------------------------------------------
// device: shared-memory addresses, mbarrier
// ----------------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must trap (-> cudaErrorLaunchFailure), never hang the GPU.  The slow path is kept out
// of line so that the many call sites do not bloat the kernels past the instruction cache.
static __device__ __noinline__ void mbar_wait_slow(uint64_t* bar, uint32_t parity) {
  const long long t0 = clock64();
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (((++spins) & 0xFFFu) == 0 && (clock64() - t0) > 6000000000LL) {   // ~3 s
      printf("mpgcn_b200: mbarrier wait timed out (block %d thread %d)\n", blockIdx.x, threadIdx.x);
      __trap();
    }
  }
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  mbar_wait_slow(bar, parity);
}
// The same bounded wait without any function call (no printf): for code between wgmma instructions, where a call forces
// ptxas to serialise the wgmma pipeline.  A timeout traps without a message.
__device__ __forceinline__ void mbar_wait_inline(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > 6000000000LL) __trap();   // ~3 s
}

// ----------------------------------------------------------------------------------------
// device: cp.async (per-thread asynchronous copies global -> shared).  After cp_async_wait<N> every group of the thread but
// the newest N has landed and is visible to that thread; other threads need a barrier before they read it.
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ----------------------------------------------------------------------------------------
// device: TMA (bulk tensor copies global -> shared, completion on an mbarrier)
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar,
                                            int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// shared -> global tile store (bulk-group completion); the smem writes it reads must precede it behind fence_proxy_async_smem
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* smem_src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(map), "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// every committed store of this thread but the newest N has finished READING its shared-memory source
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// every committed store of this thread is complete
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ----------------------------------------------------------------------------------------
// device: wgmma (warpgroup MMA, operands in shared memory, fp32 accumulators in registers)
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// barrier over `count` threads (whole warps) under id 1..15 (0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// wgmma shared-memory matrix descriptor (PTX ISA, "Matrix Descriptor Format" of wgmma):
//   [0,14) start address >> 4 | [16,30) leading byte offset >> 4 | [32,46) stride byte offset >> 4
//   [62,64) swizzle mode (1 = 128B, 2 = 64B)
// K-major: SBO = byte stride between 8-row groups (LBO unused).  MN-major: LBO = byte stride between swizzle-atom columns
// along M / N, SBO = byte stride between 8-row groups along K.
constexpr uint32_t GMMA_SW128 = 1u, GMMA_SW64 = 2u;
__device__ __forceinline__ uint64_t gmma_desc_hi(uint32_t sbo_bytes, uint32_t swizzle) {
  return (static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) | (static_cast<uint64_t>(swizzle) << 30)) << 32;
}
__device__ __forceinline__ uint64_t gmma_desc(uint64_t hi, uint32_t smem_addr, uint32_t lbo_bytes) {
  return hi | static_cast<uint64_t>((smem_addr >> 4) & 0x3FFFu) | (static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16);
}

// mma.sync m16n8k16, fp16 x fp16 -> fp32 (warp-level tensor-core MMA; register fragments as in the PTX ISA)
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// m16n8k8: the same with one k-half (A: a0 row g, a1 row g + 8; B: b0)
__device__ __forceinline__ void mma_1688(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t b0) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5}, {%6}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a0), "r"(a1), "r"(b0));
}
__device__ __forceinline__ void ldmatrix_x2(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x2_trans(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];" : "=r"(r0), "=r"(r1) : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}

// fp32 -> fp16 round-to-nearest-even, saturating at +-65504 instead of producing inf; NaN stays NaN (a clamp with
// fminf / fmaxf would turn it into a finite number).  Every in-range value converts exactly as __float2half_rn does.
__device__ __forceinline__ __half f2h_sat(float x) { return __float2half_rn(fabsf(x) > 65504.f ? copysignf(65504.f, x) : x); }
// the same for a pair, in one instruction (F2FP.SATFINITE): low half = a, high half = b, as __floats2half2_rn(a, b)
__device__ __forceinline__ uint32_t f2h2_sat_bits(float a, float b) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
// fp32 pair (a, b) -> bf16 pairs hi = bf16_rn(x), lo = bf16_rn(x - hi) (bf16x3 operands), packed low half = a as above.  bf16
// has fp32's exponent range: no saturation, and hi + lo carries 16 significant bits.
__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(b), "f"(a));
  const float ha = __uint_as_float(hi << 16), hb = __uint_as_float(hi & 0xffff0000u);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(b - hb), "f"(a - ha));
}
#endif  // __CUDACC__

// ----------------------------------------------------------------------------------------
// host: tensor-map encoding through the driver entry point (no link-time libcuda dependency)
// ----------------------------------------------------------------------------------------
enum TmapSwizzle { TMAP_SW64 = 0, TMAP_SW128 = 1 };
// fp16 tensor, up to 4 dims (innermost first); strides_bytes[i] is the stride of dim i+1.
int make_tmap_f16(CUtensorMap* out, const void* gptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box, TmapSwizzle swz);

int device_sm_count();

// Deterministic mode of the calling host thread (mpgcn_set_deterministic, DESIGN.md section 11): every cross-CTA floating-point
// sum writes per-CTA partials ("slots") to the workspace and one fixed-order kernel adds them, instead of atomics.
int det_mode();
int det_set(int on);

// Function attributes (the > 48 KB dynamic shared-memory opt-in) belong to a device / context, not to the process: a
// kernel that already ran on cuda:0 still needs the opt-in on cuda:1.  One cache per kernel, indexed by device ordinal.
struct DynSmemAttr { int bytes[64]; };
int ensure_dyn_smem_impl(const void* kernel, int bytes, DynSmemAttr& cache);
template <class Kernel>
inline int ensure_dyn_smem(Kernel kernel, int bytes, DynSmemAttr& cache) {
  return ensure_dyn_smem_impl(reinterpret_cast<const void*>(kernel), bytes, cache);
}

// ----------------------------------------------------------------------------------------
// host: launch accounting / per-launch CUDA-event timing (bench.py's roofline evidence)
// ----------------------------------------------------------------------------------------
enum ProfTag {
  PROF_FWD_A = 0, PROF_FWD_MIX, PROF_FWD_B, PROF_BWD_V, PROF_BWD_DW, PROF_BWD_MIX, PROF_BWD_DX,   // wgmma contractions
  PROF_SIMT_GEMM, PROF_ELEMENTWISE, PROF_LSTM_FWD, PROF_LSTM_BWD,
  // regions, not kernels: a whole C-ABI call (every kernel of it, the gaps between them included); they count calls, not launches
  PROF_LAYER_FWD, PROF_LAYER_BWD, PROF_HEAD,
  PROF_EXCHANGE,      // kernels: the peer-memory exchange steps of the row shard (rows_reduce_bias_act, relu_backward_scatter[_f16])
  PROF_BWD_DG,        // kernels: the support gradient of the tensor-core path (U16 recompute, BWD_DGO / BWD_DGD, their reductions)
  PROF_NUM_TAGS
};
constexpr int PROF_FIRST_REGION_TAG = PROF_LAYER_FWD;
// All of these may be called from several host threads (one stream each): the counters sit behind a mutex, the
// "next launch" annotation and the open begin/end bracket are thread-local.
void prof_set_next(int tag, double flops);             // annotate the next contraction launch (this thread's)
void prof_take_next(int* tag, double* flops);          // fetch and clear this thread's annotation
void prof_count(int tag);                              // count one launch of our own kernels
void prof_begin(int tag, double flops, cudaStream_t s);   // event before launch (no-op unless enabled)
void prof_end(cudaStream_t s);                            // event after launch
// whole-call bracket (nests around the per-launch brackets): event pair recorded only while profiling is enabled
struct ProfRegion {
  void* a = nullptr;
  int tag;
  cudaStream_t s;
  ProfRegion(int tag, double flops, cudaStream_t s);
  ~ProfRegion();
};

}  // namespace mpgcn
