// Host-side runtime helpers: error string, TMA descriptor encoding (driver entry point fetched through the runtime,
// so the library has no link-time dependency on libcuda), device properties.
#include <stdarg.h>
#include <string.h>

#include <mutex>

#include "common.cuh"
#include "kernels.h"

namespace vs {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
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

int make_tmap_f16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                  const uint32_t* box, int swizzle) {
  EncodeTiledFn enc = get_encode();
  VS_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled entry point unavailable (no CUDA driver?)");
  VS_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base address must be 16-byte aligned");
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) {
      gstr[i - 1] = strides_bytes[i - 1];
      VS_REQUIRE(gstr[i - 1] % 16 == 0, "TMA stride %d (%llu bytes) must be a multiple of 16", i,
                 (unsigned long long)gstr[i - 1]);
    }
    VS_REQUIRE(bx[i] >= 1 && bx[i] <= 256, "TMA box dim %d = %u out of range", i, bx[i]);
  }
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle == 1 ? CU_TENSOR_MAP_SWIZZLE_128B : swizzle == 2 ? CU_TENSOR_MAP_SWIZZLE_64B
                   : swizzle == 3 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  VS_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu,%llu box %u,%u)",
             (int)r, rank, (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
  return 0;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

}  // namespace vs

// ---------------------------------------------------------------------------------------------------------------
// Lightweight per-launch profiler (CUDA events on the launching stream) and launch counter, used by bench.py for the
// live roofline numbers.  Disabled by default; when enabled every launcher brackets its kernel(s) with two events.
#include <atomic>
#include <vector>

namespace vs {

static std::atomic<long long> g_launches{0};
static bool g_prof_on = false;
struct ProfEntry { cudaEvent_t a, b; int cat; double work; long long m; int n, k; };
static std::vector<ProfEntry> g_prof;
static std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_pool;

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
long long launch_count() { return g_launches.load(); }

ProfScope::ProfScope(cudaStream_t st, int cat, double work, int nlaunch, long long m, int n, int k) : st_(st), idx_(-1) {
  count_launch(nlaunch);
  if (!g_prof_on) return;
  ProfEntry e;
  if (!g_pool.empty()) { e.a = g_pool.back().first; e.b = g_pool.back().second; g_pool.pop_back(); }
  else { cudaEventCreate(&e.a); cudaEventCreate(&e.b); }
  e.cat = cat; e.work = work; e.m = m; e.n = n; e.k = k;
  cudaEventRecord(e.a, st);
  idx_ = (int)g_prof.size();
  g_prof.push_back(e);
}
ProfScope::~ProfScope() {
  if (idx_ >= 0) cudaEventRecord(g_prof[idx_].b, st_);
}

// A/B switches of the kernels (name, value).  Defaults are the shipped configuration.
struct Option { const char* name; int value; };
static Option g_options[] = {
    {"attn_tc", 1},        // wgmma attention for d = 40 / 80 (0 = mma.sync kernel)
    {"gemm_stages", 0},    // smem ring depth limit (0 = all)
    {"gemm_ctas", 0},
    {"gemm_epi_slot", 1},  // short-K linears and GEGLUs read their epilogue operands from shared-memory slots (0 = from global memory)      // persistent GEMM grid cap (0 = one CTA per SM); tests run other tile schedules with it
    {"ln_fold", 1},        // LayerNorms folded into the GEMM that consumes them (0 = stand-alone LayerNorm kernel)
    {"ln_fuse", 1},        // row statistics of folded LayerNorms come from the producing GEMM's epilogue (0 = ln_stats_kernel pass)
    {"tattn_vst", 1},      // temporal attention: outputs staged in shared memory and written with 16-byte stores (0 = 4-byte)
    {"gn_fused", 1},       // per-frame GroupNorms as one cluster-resident pass (0 = statistics kernel + apply kernel)
    {"gn_stats_v2", 0},    // GroupNorm statistics with per-position accumulators (no per-element group select); A/B
    {"subpixel", 1},       // nearest-2x + 3x3 conv as four 2x2 sub-pixel convs on the low-resolution input (0 = materialise)
    {"pdl", 1},            // programmatic dependent launch between the hot kernels (0 = plain stream order)
};
int set_option(const char* name, int value) {
  for (Option& o : g_options)
    if (strcmp(name, o.name) == 0) { o.value = value; return 0; }
  set_error("unknown option '%s'", name);
  return 2;
}
int get_option(const char* name) {
  for (const Option& o : g_options)
    if (strcmp(name, o.name) == 0) return o.value;
  return 0;
}

int prof_dump(const char* path) {
  struct Agg { int cat; long long m; int n, k; double work, ms; long long count; };
  std::vector<Agg> aggs;
  for (auto& e : g_prof) {
    if (cudaEventSynchronize(e.b) != cudaSuccess) { set_error("profile: event sync failed"); return 1; }
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e.a, e.b);
    Agg* hit = nullptr;
    for (auto& a : aggs)
      if (a.cat == e.cat && a.m == e.m && a.n == e.n && a.k == e.k && a.work == e.work) { hit = &a; break; }
    if (!hit) { aggs.push_back(Agg{e.cat, e.m, e.n, e.k, e.work, 0.0, 0}); hit = &aggs.back(); }
    hit->ms += ms;
    hit->count += 1;
  }
  FILE* f = fopen(path, "w");
  if (!f) { set_error("cannot open %s", path); return 2; }
  fprintf(f, "category,m,n,k,work_per_launch,launches,total_ms\n");
  for (auto& a : aggs) fprintf(f, "%d,%lld,%d,%d,%.6g,%lld,%.4f\n", a.cat, a.m, a.n, a.k, a.work, a.count, a.ms);
  fclose(f);
  return 0;
}

void prof_enable(bool on) { g_prof_on = on; }
void prof_reset() {
  for (auto& e : g_prof) g_pool.push_back({e.a, e.b});
  g_prof.clear();
}
int prof_collect(int cat, double* ms, double* work, long long* count) {
  double t = 0, w = 0; long long n = 0;
  for (auto& e : g_prof) {
    if (e.cat != cat) continue;
    if (cudaEventSynchronize(e.b) != cudaSuccess) { set_error("profile: event sync failed"); return 1; }
    float m = 0.f;
    cudaEventElapsedTime(&m, e.a, e.b);
    t += m; w += e.work; ++n;
  }
  *ms = t; *work = w; *count = n;
  return 0;
}

}  // namespace vs
