// Host launcher for the wgmma split-plane GEMM: builds the TMA tensor maps and picks the stage count.
#include <atomic>
#include <cstdlib>
#include <mutex>
#include <unordered_map>
#include <vector>

#include "gemm_sm90.cuh"

namespace oob {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

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

// 3-D map over [planes][rows][ld] bf16; box = {64 elements, box_rows, box_planes}, SWIZZLE_128B (one smem row is
// exactly one swizzle span).
static int make_map(CUtensorMap* m, const PlaneMat& a, int box_rows, int box_planes) {
  EncodeTiledFn enc = get_encode_fn();
  OOB_CHECK(enc != nullptr, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  OOB_CHECK((a.ld % 8) == 0 && (a.plane_stride % 8) == 0, "split-plane operand strides must be multiples of 8");
  OOB_CHECK((reinterpret_cast<uintptr_t>(a.base) & 15) == 0, "split-plane operand must be 16 B aligned");
  OOB_CHECK(box_planes <= a.nplanes, "GEMM asks for %d planes, operand has %d", box_planes, a.nplanes);
  cuuint64_t dims[3] = {(cuuint64_t)a.cols, (cuuint64_t)a.rows, (cuuint64_t)a.nplanes};
  cuuint64_t strides[2] = {(cuuint64_t)a.ld * 2, (cuuint64_t)a.plane_stride * 2};
  cuuint32_t box[3] = {(cuuint32_t)GEMM_BK, (cuuint32_t)box_rows, (cuuint32_t)box_planes};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<bf16*>(a.base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  OOB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d): rows=%ld cols=%ld ld=%ld", (int)r, a.rows, a.cols,
            a.ld);
  return 0;
}

// Descriptor cache.  A training step launches the same few hundred (buffer, shape, box) combinations every micro-batch
// (encoding two maps per GEMM on the host costs tens of thousands of cuTensorMapEncodeTiled calls per GPT-2-XL step); a map depends
// only on the key below, never on the buffer's contents, so entries stay valid for as long as the address is reused
// for the same shape.  Per host thread (no lock); bounded.
struct MapKey {
  const void* base; long rows, cols, ld, plane_stride; int nplanes, box_rows, box_planes;
  bool operator==(const MapKey& o) const {
    return base == o.base && rows == o.rows && cols == o.cols && ld == o.ld && plane_stride == o.plane_stride &&
           nplanes == o.nplanes && box_rows == o.box_rows && box_planes == o.box_planes;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.base) * 0x9E3779B97F4A7C15ull;
    auto mix = [&h](size_t v) { h ^= v + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2); };
    mix((size_t)k.rows); mix((size_t)k.cols); mix((size_t)k.ld); mix((size_t)k.plane_stride);
    mix((size_t)k.nplanes * 1000003u + (size_t)k.box_rows * 10007u + (size_t)k.box_planes * 101u);
    return h;
  }
};
static std::atomic<long> g_map_encodes{0};
long tensor_map_encodes() { return g_map_encodes.load(); }

int tensor_map_3d(const CUtensorMap** out, const PlaneMat& a, int box_rows, int box_planes) {
  thread_local std::unordered_map<MapKey, CUtensorMap, MapKeyHash> cache;
  const MapKey key{a.base, a.rows, a.cols, a.ld, a.plane_stride, a.nplanes, box_rows, box_planes};
  auto it = cache.find(key);
  if (it == cache.end()) {
    if (cache.size() >= 16384) cache.clear();
    CUtensorMap m;
    if (int rc = make_map(&m, a, box_rows, box_planes)) return rc;
    g_map_encodes.fetch_add(1, std::memory_order_relaxed);
    it = cache.emplace(key, m).first;
  }
  *out = &it->second;
  return 0;
}

// ---- optional CUDA-event timing of every launch (roofline measurement) ----------------------------------------
struct TimedLaunch { cudaEvent_t a, b; double flops; double executed; };
static bool g_timing = false;
static std::vector<TimedLaunch> g_timed;
static std::vector<cudaEvent_t> g_event_pool;
static cudaEvent_t get_event() {
  if (!g_event_pool.empty()) { cudaEvent_t e = g_event_pool.back(); g_event_pool.pop_back(); return e; }
  cudaEvent_t e; cudaEventCreate(&e); return e;
}
int gemm_timing_begin() { g_timed.clear(); g_timing = true; return 0; }
int gemm_timing_end(double* total_ms, double* total_flops, double* executed_flops, long* launches) {
  g_timing = false;
  double ms = 0, fl = 0, ex = 0;
  for (auto& t : g_timed) {
    OOB_CUDA_OK(cudaEventSynchronize(t.b));
    float x = 0;
    OOB_CUDA_OK(cudaEventElapsedTime(&x, t.a, t.b));
    ms += x; fl += t.flops; ex += t.executed;
    g_event_pool.push_back(t.a); g_event_pool.push_back(t.b);
  }
  if (total_ms) *total_ms = ms;
  if (total_flops) *total_flops = fl;
  if (executed_flops) *executed_flops = ex;
  if (launches) *launches = (long)g_timed.size();
  g_timed.clear();
  return 0;
}

template <bool A_MN, bool B_MN, bool F16>
static int launch_t(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream) {
  static int max_smem = -1;
  if (max_smem < 0) {
    int dev = 0;
    OOB_CUDA_OK(cudaGetDevice(&dev));
    OOB_CUDA_OK(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  }
  static bool attr_set = false;
  auto kern = gemm_planes_sm90_kernel<A_MN, B_MN, F16>;
  if (!attr_set) {
    OOB_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    attr_set = true;
  }
  const int stage = gemm_stage_bytes(p.nsplit);
  const int overhead = 1024 + 256;   // alignment slack, barriers
  int stages = (max_smem - overhead) / stage;
  if (stages > 8) stages = 8;
  OOB_CHECK(stages >= 2, "GEMM tile does not fit %d B of shared memory", max_smem);
  OOB_CHECK((size_t)stages * stage >= sizeof(float) * GEMM_BM * GEMM_STAGE_LD, "GEMM epilogue staging does not fit");
  const dim3 grid((p.M + GEMM_BM - 1) / GEMM_BM, (p.N + GEMM_BN - 1) / GEMM_BN);
  OOB_CHECK(grid.y <= 65535, "GEMM N = %d too large", p.N);
  const size_t smem = (size_t)stages * stage + overhead;
  TimedLaunch tl{};
  if (g_timing) { tl.a = get_event(); tl.b = get_event(); tl.flops = 2.0 * p.M * p.N * p.K;
    tl.executed = tl.flops * (p.nsplit == 1 ? 1 : (p.nsplit == 2 ? 3 : 6)); cudaEventRecord(tl.a, stream); }
  kern<<<grid, GEMM_THREADS, smem, stream>>>(ta, tb, p, stages);
  OOB_CUDA_OK(cudaGetLastError());
  if (g_timing) { cudaEventRecord(tl.b, stream); g_timed.push_back(tl); }
  count_launch();
  return 0;
}

int gemm_launch(const PlaneMat& A, int a_mn, const PlaneMat& B, int b_mn, const GemmParams& p_in, cudaStream_t stream) {
  GemmParams p = p_in;
  OOB_CHECK(p.nsplit >= 1 && p.nsplit <= 3, "nsplit must be 1..3");
  OOB_CHECK(p.M > 0 && p.N > 0 && p.K > 0, "empty GEMM %d x %d x %d", p.M, p.N, p.K);
  // operand formats: bf16 x (1..3) planes, or fp16 x (1..2) planes with the second plane pre-scaled by 2^11.  wgmma
  // takes one element type for both operands, so the two must agree.
  OOB_CHECK(A.fp16 == B.fp16, "mixed fp16 / bf16 operands are not supported");
  p.corr_scale = 1.0f;
  if (A.fp16) {
    OOB_CHECK(p.nsplit <= 2, "fp16 planes come in pairs: nsplit must be 1 or 2");
    if (p.nsplit == 2) p.corr_scale = 1.0f / 2048.0f;
  }
  OOB_CHECK(A.nplanes >= p.nsplit && B.nplanes >= p.nsplit, "operands carry fewer planes than nsplit");
  {
    GemmEpilogue& e = p.epi;
    auto ok16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    e.vec4 = (!e.d || (ok16(e.d) && (e.ldd & 3) == 0)) && (!e.bias || ok16(e.bias)) &&
             (!e.resid || (ok16(e.resid) && (e.ldr & 3) == 0)) && (!e.aux || (ok16(e.aux) && (e.ldaux & 3) == 0)) &&
             (!e.planes || ((reinterpret_cast<uintptr_t>(e.planes) & 7) == 0 && (e.ldp & 3) == 0 &&
                            (e.plane_stride & 3) == 0));
  }
  const CUtensorMap *pta = nullptr, *ptb = nullptr;
  int rc;
  // K-major operand: stored [MN][K] -> box {64 k, tile rows, planes}; MN-major: stored [K][MN] -> box {64 mn, 64 k rows}
  if (!a_mn) {
    OOB_CHECK(A.rows >= p.M && A.cols >= p.K, "A (K-major) is %ld x %ld, need %d x %d", A.rows, A.cols, p.M, p.K);
    rc = tensor_map_3d(&pta, PlaneMat{A.base, (long)p.M, (long)p.K, A.ld, A.plane_stride, A.nplanes}, GEMM_BM, p.nsplit);
  } else {
    OOB_CHECK(A.rows >= p.K && A.cols >= p.M, "A (M-major) is %ld x %ld, need %d x %d", A.rows, A.cols, p.K, p.M);
    rc = tensor_map_3d(&pta, PlaneMat{A.base, (long)p.K, (long)p.M, A.ld, A.plane_stride, A.nplanes}, GEMM_BK, p.nsplit);
  }
  if (rc) return rc;
  if (!b_mn) {
    OOB_CHECK(B.rows >= p.N && B.cols >= p.K, "B (K-major) is %ld x %ld, need %d x %d", B.rows, B.cols, p.N, p.K);
    rc = tensor_map_3d(&ptb, PlaneMat{B.base, (long)p.N, (long)p.K, B.ld, B.plane_stride, B.nplanes}, GEMM_BN, p.nsplit);
  } else {
    OOB_CHECK(B.rows >= p.K && B.cols >= p.N, "B (N-major) is %ld x %ld, need %d x %d", B.rows, B.cols, p.K, p.N);
    rc = tensor_map_3d(&ptb, PlaneMat{B.base, (long)p.K, (long)p.N, B.ld, B.plane_stride, B.nplanes}, GEMM_BK, p.nsplit);
  }
  if (rc) return rc;
  const CUtensorMap& ta = *pta;
  const CUtensorMap& tb = *ptb;
#define OOB_DISPATCH_MAJORS(F16)                                                  \
  do {                                                                            \
    if (!a_mn && !b_mn) return launch_t<false, false, F16>(ta, tb, p, stream);    \
    if (!a_mn && b_mn) return launch_t<false, true, F16>(ta, tb, p, stream);      \
    if (a_mn && !b_mn) return launch_t<true, false, F16>(ta, tb, p, stream);      \
    return launch_t<true, true, F16>(ta, tb, p, stream);                          \
  } while (0)
  if (A.fp16) OOB_DISPATCH_MAJORS(true);
  OOB_DISPATCH_MAJORS(false);
#undef OOB_DISPATCH_MAJORS
}

}  // namespace oob
