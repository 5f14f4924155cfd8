// Host side of the wgmma contraction engine: kernel instantiations, launch, tensor maps.
#include "tc_engine.cuh"

#include <mutex>
#include <vector>
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

namespace mpgcn {

// ---------------------------------------------------------------------------------------
// error string (thread local), device attributes
// ---------------------------------------------------------------------------------------
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }

// deterministic mode, per host thread like the error string: one thread's setting never changes another's launches
static thread_local int g_det = 0;
int det_mode() { return g_det; }
int det_set(int on) {
  const int prev = g_det;
  g_det = on ? 1 : 0;
  return prev;
}

int ensure_dyn_smem_impl(const void* kernel, int bytes, DynSmemAttr& cache) {
  static std::mutex mu;
  int dev = 0;
  MPGCN_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  const bool known = dev >= 0 && dev < 64;
  if (!known || cache.bytes[dev] < bytes) {
    MPGCN_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    if (known) cache.bytes[dev] = bytes;
  }
  return 0;
}

int device_sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

// ---------------------------------------------------------------------------------------
// launch accounting and optional per-launch event timing
// ---------------------------------------------------------------------------------------
namespace {
struct ProfState {
  bool enabled = false;
  long long launches[PROF_NUM_TAGS] = {0};
  double flops[PROF_NUM_TAGS] = {0};
  double ms[PROF_NUM_TAGS] = {0};
  struct Pending { cudaEvent_t a, b; int tag; };
  std::vector<Pending> pending;
  std::vector<cudaEvent_t> pool;
  std::mutex mu;
} g_prof;
thread_local int t_cur_tag = -1;
thread_local cudaEvent_t t_cur_a = nullptr;
thread_local int t_next_tag = -1;
thread_local double t_next_flops = 0;
cudaEvent_t prof_event() {          // caller holds g_prof.mu
  if (!g_prof.pool.empty()) { cudaEvent_t e = g_prof.pool.back(); g_prof.pool.pop_back(); return e; }
  cudaEvent_t e = nullptr;
  cudaEventCreate(&e);
  return e;
}
}  // namespace

void prof_set_next(int tag, double flops) { t_next_tag = tag; t_next_flops = flops; }
void prof_take_next(int* tag, double* flops) {
  *tag = t_next_tag;
  *flops = t_next_flops;
  t_next_tag = -1;
  t_next_flops = 0;
}
void prof_count(int tag) {
  std::lock_guard<std::mutex> lock(g_prof.mu);
  if (tag >= 0 && tag < PROF_NUM_TAGS) g_prof.launches[tag]++;
}
void prof_begin(int tag, double flops, cudaStream_t s) {
  std::lock_guard<std::mutex> lock(g_prof.mu);
  if (tag >= 0 && tag < PROF_NUM_TAGS) { g_prof.launches[tag]++; g_prof.flops[tag] += flops; }
  if (!g_prof.enabled) return;
  t_cur_tag = tag;
  t_cur_a = prof_event();
  cudaEventRecord(t_cur_a, s);
}
void prof_end(cudaStream_t s) {
  if (t_cur_a == nullptr) return;
  std::lock_guard<std::mutex> lock(g_prof.mu);
  cudaEvent_t b = prof_event();
  cudaEventRecord(b, s);
  g_prof.pending.push_back({t_cur_a, b, t_cur_tag});
  t_cur_a = nullptr;
}
ProfRegion::ProfRegion(int tag_, double flops, cudaStream_t s_) : tag(tag_), s(s_) {
  std::lock_guard<std::mutex> lock(g_prof.mu);
  if (tag >= 0 && tag < PROF_NUM_TAGS) { g_prof.launches[tag]++; g_prof.flops[tag] += flops; }
  if (!g_prof.enabled) return;
  cudaEvent_t e = prof_event();
  cudaEventRecord(e, s);
  a = e;
}
ProfRegion::~ProfRegion() {
  if (a == nullptr) return;
  std::lock_guard<std::mutex> lock(g_prof.mu);
  cudaEvent_t b = prof_event();
  cudaEventRecord(b, s);
  g_prof.pending.push_back({static_cast<cudaEvent_t>(a), b, tag});
}
void prof_enable(int on) {
  std::lock_guard<std::mutex> lock(g_prof.mu);
  g_prof.enabled = on != 0;
}
void prof_reset() {
  std::lock_guard<std::mutex> lock(g_prof.mu);
  for (int i = 0; i < PROF_NUM_TAGS; ++i) { g_prof.launches[i] = 0; g_prof.flops[i] = 0; g_prof.ms[i] = 0; }
  for (auto& p : g_prof.pending) { g_prof.pool.push_back(p.a); g_prof.pool.push_back(p.b); }
  g_prof.pending.clear();
}
// resolves pending event pairs (caller must have synchronised the stream)
int prof_read(int tag, long long* launches, double* flops, double* ms) {
  std::lock_guard<std::mutex> lock(g_prof.mu);
  for (auto& p : g_prof.pending) {
    float t = 0.f;
    if (cudaEventElapsedTime(&t, p.a, p.b) == cudaSuccess && p.tag >= 0 && p.tag < PROF_NUM_TAGS) g_prof.ms[p.tag] += t;
    g_prof.pool.push_back(p.a);
    g_prof.pool.push_back(p.b);
  }
  g_prof.pending.clear();
  if (tag < 0 || tag >= PROF_NUM_TAGS) return 1;
  *launches = g_prof.launches[tag];
  *flops = g_prof.flops[tag];
  *ms = g_prof.ms[tag];
  return 0;
}

// ---------------------------------------------------------------------------------------
// tensor maps: cuTensorMapEncodeTiled resolved through the runtime (no -lcuda at link time,
// so the library loads -- and its symbols can be checked -- on a machine without a driver)
// ---------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

int make_tmap_f16(CUtensorMap* out, const void* gptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box, TmapSwizzle swz) {
  EncodeTiledFn fn = get_encode_fn();
  MPGCN_CHECK(fn != nullptr, "cuTensorMapEncodeTiled is not available (no CUDA driver?)");
  MPGCN_CHECK(rank >= 1 && rank <= 4, "tensor map rank %d unsupported", rank);
  cuuint64_t gdim[4] = {1, 1, 1, 1};
  cuuint64_t gstr[3] = {0, 0, 0};
  cuuint32_t bx[4] = {1, 1, 1, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
  }
  // always encode rank 4 (the kernel issues 4-d copies); pad with unit dims whose stride
  // continues the outermost real stride
  uint64_t last = (rank >= 2) ? strides_bytes[rank - 2] * dims[rank - 1] : dims[0] * 2;
  for (int i = 0; i < 3; ++i) {
    if (i < rank - 1) gstr[i] = strides_bytes[i];
    else { gstr[i] = align_up(last, 16); }
  }
  for (int i = 0; i < 3; ++i)
    MPGCN_CHECK(gstr[i] % 16 == 0 && gstr[i] < (1ull << 40), "tensor map stride %llu of dim %d is not a multiple of 16",
                (unsigned long long)gstr[i], i + 1);
  MPGCN_CHECK((reinterpret_cast<uintptr_t>(gptr) & 15) == 0, "tensor map base pointer must be 16-byte aligned");
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(gptr), gdim, gstr, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz == TMAP_SW128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  MPGCN_CHECK(r == CUDA_SUCCESS,
              "cuTensorMapEncodeTiled failed (%d): dims=(%llu,%llu,%llu,%llu) strides=(%llu,%llu,%llu) box=(%u,%u,%u,%u)", (int)r,
              (unsigned long long)gdim[0], (unsigned long long)gdim[1], (unsigned long long)gdim[2], (unsigned long long)gdim[3],
              (unsigned long long)gstr[0], (unsigned long long)gstr[1], (unsigned long long)gstr[2], bx[0], bx[1], bx[2], bx[3]);
  return 0;
}

namespace tc {

static const int kMaxSmem = 232448;   // 227 KB opt-in limit per CTA on sm_90

// Store map of a contraction output: element (ch, i, r, z) at base + z*sZ + i*sI + r*sR + ch, dims (32, m_valid, r_valid, Z),
// box one chunk of 64 rows, in the swizzle the epilogue writes its store buffer with (a 64- or 128-byte row).  TMA clips every
// box at these dims, which is what bounds a partial tile.
static int make_out_map(CUtensorMap* m, const void* base, bool f16, const Epilogue& ep, int Z) {
  EncodeTiledFn fn = get_encode_fn();
  MPGCN_CHECK(fn != nullptr, "cuTensorMapEncodeTiled is not available (no CUDA driver?)");
  const uint64_t es = f16 ? 2 : 4;
  cuuint64_t dims[4] = {32, (cuuint64_t)ep.m_valid, (cuuint64_t)ep.r_valid, (cuuint64_t)Z};
  cuuint64_t str[3] = {(cuuint64_t)ep.sI * es, (cuuint64_t)ep.sR * es, (cuuint64_t)ep.sZ * es};
  cuuint32_t box[4] = {32, 64, 1, 1};
  cuuint32_t one[4] = {1, 1, 1, 1};
  for (int i = 0; i < 3; ++i)
    MPGCN_CHECK(str[i] % 16 == 0 && str[i] < (1ull << 40), "output stride %llu of dim %d is not a multiple of 16 bytes",
                (unsigned long long)str[i], i + 1);
  MPGCN_CHECK((reinterpret_cast<uintptr_t>(base) & 15) == 0, "output pointer must be 16-byte aligned");
  CUresult r = fn(m, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<void*>(base), dims, str, box,
                  one, CU_TENSOR_MAP_INTERLEAVE_NONE, f16 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  MPGCN_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (output) failed (%d): dims=(32,%d,%d,%d) strides=(%llu,%llu,%llu)", (int)r,
              ep.m_valid, ep.r_valid, Z, (unsigned long long)str[0], (unsigned long long)str[1], (unsigned long long)str[2]);
  return 0;
}

template <int AK, int BK, bool BKM = false, class T = __half>
static int launch_impl(GemmParams& p, cudaStream_t stream) {
  using C = Cfg<AK, BK>;
  constexpr bool BF = std::is_same<T, __nv_bfloat16>::value;
  static DynSmemAttr attr = {};
  if (int e = ensure_dyn_smem(contract_kernel<AK, BK, BKM, T>, kMaxSmem, attr)) return e;
  MPGCN_CHECK(p.R >= 1 && p.R <= 8, "R=%d out of range", p.R);
  const size_t b_stage = (size_t)p.R * BK * 64;
  if (BF)
    MPGCN_CHECK(p.kb_pass > 0 && p.kb_total % p.kb_pass == 0 && p.kb_pass % p.kb_per_seg == 0 && p.ep.corr_src == nullptr &&
                    (p.ep.out_f16 ? p.ep.out16 != nullptr : p.ep.out16 == nullptr),
                "bf16x3 contraction: kb_total=%d is not whole passes of %d k-blocks, or an fp16-only epilogue option is set", p.kb_total,
                p.kb_pass);
  const int nres = p.b_res_reps * (BF ? p.kb_pass : p.kb_total);
  MPGCN_CHECK(!BKM || nres == 0, "a K-major B operand streams through the ring");
  MPGCN_CHECK(p.ep.out != nullptr && p.ep.m_valid > 0 && p.ep.r_valid > 0, "contraction without an output");
  if (int e = make_out_map(&p.out_map, p.ep.out, p.ep.out_f16 != 0, p.ep, p.Z)) return e;
  const bool shadow = !p.ep.out_f16 && p.ep.out16 != nullptr;
  if (shadow || (BF && p.ep.out_f16))         // the fp16 shadow, or the lo plane of a bf16 pair
    if (int e = make_out_map(&p.out16_map, p.ep.out16, true, p.ep, p.Z)) return e;
  p.st_bytes = p.ep.out_f16 ? (BF ? 2 * 64 * 64 : 64 * 64) : shadow ? 64 * 128 + 64 * 64 : 64 * 128;
  const size_t fixed = smem_bytes(0, p.R, BK, 0, 0, p.st_bytes);      // everything but the ring
  int stages;
  if (nres) {
    MPGCN_CHECK(p.NT == 1 && p.kb_per_seg == 1 && !p.split_k && p.bm.z_mul == 0, "resident B needs a tile-independent B operand");
    MPGCN_CHECK(fixed + (size_t)nres * b_stage + 2 * (size_t)C::A_STAGE <= (size_t)kMaxSmem, "resident B operand does not fit in shared memory");
    stages = (int)((kMaxSmem - fixed - (size_t)nres * b_stage) / (size_t)C::A_STAGE);
  } else {
    stages = (int)((kMaxSmem - fixed) / ((size_t)C::A_STAGE + b_stage));
  }
  // small stages (channel mixes, 8 KB of A per k-block) are HBM-latency bound: keep >= 128 KB of loads in flight per SM
  const int max_stages = ((size_t)C::A_STAGE + (nres ? 0 : b_stage) <= 16384) ? 16 : 8;
  if (stages > max_stages) stages = max_stages;
  MPGCN_CHECK(stages >= 2, "tile does not fit in shared memory");
  p.stages = stages;
  // always request the full opt-in budget: exactly one CTA per SM
  const size_t smem = kMaxSmem;
  MPGCN_CHECK(smem_bytes(C::A_STAGE, p.R, BK, stages, nres, p.st_bytes) <= smem, "internal: smem budget");
  const long long tiles = (long long)p.MT * p.NT * p.Z;
  MPGCN_CHECK(tiles > 0 && tiles < (1ll << 31), "bad tile count %lld", tiles);
  MPGCN_CHECK(p.kb_total > 0 && p.kb_per_seg > 0, "empty contraction");
  int grid = (int)(tiles < device_sm_count() ? tiles : device_sm_count());
  int tag = -1;
  double fl = 0;
  prof_take_next(&tag, &fl);
  prof_begin(tag, fl, stream);
  contract_kernel<AK, BK, BKM, T><<<grid, kThreads1, smem, stream>>>(p);
  prof_end(stream);
  MPGCN_CUDA(cudaGetLastError());
  return 0;
}

int launch_contract(int ak, int bk, GemmParams& p, cudaStream_t stream) {
  if (ak == A_MN128 && bk == 64) return launch_impl<A_MN128, 64>(p, stream);
  if (ak == A_K128 && bk == 64) return launch_impl<A_K128, 64>(p, stream);
  if (ak == A_K64 && bk == 32) return launch_impl<A_K64, 32>(p, stream);
  if (ak == A_K64 && bk == 64) return launch_impl<A_K64, 64>(p, stream);
  if (ak == A_K64 && bk == 96) return launch_impl<A_K64, 96>(p, stream);
  if (ak == A_MN64 && bk == 64) return launch_impl<A_MN64, 64>(p, stream);
  set_error("no contraction kernel for A kind %d, BK %d", ak, bk);
  return 1;
}

int launch_contract_bkm(GemmParams& p, cudaStream_t stream) { return launch_impl<A_K64, 32, true>(p, stream); }

int launch_contract_bf16x3(int ak, int bk, GemmParams& p, cudaStream_t stream) {
  using BF = __nv_bfloat16;
  if (ak == A_MN128 && bk == 64) return launch_impl<A_MN128, 64, false, BF>(p, stream);
  if (ak == A_K128 && bk == 64) return launch_impl<A_K128, 64, false, BF>(p, stream);
  if (ak == A_K64 && bk == 32) return launch_impl<A_K64, 32, false, BF>(p, stream);
  if (ak == A_K64 && bk == 64) return launch_impl<A_K64, 64, false, BF>(p, stream);
  if (ak == A_K64 && bk == 96) return launch_impl<A_K64, 96, false, BF>(p, stream);
  if (ak == A_MN64 && bk == 64) return launch_impl<A_MN64, 64, false, BF>(p, stream);
  set_error("no bf16x3 contraction kernel for A kind %d, BK %d", ak, bk);
  return 1;
}

}  // namespace tc
}  // namespace mpgcn
