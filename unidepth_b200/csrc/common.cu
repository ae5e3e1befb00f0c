#include "common.h"

#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

namespace udb {

static thread_local char g_err[512] = "";
std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// ---- per-launch profile (off unless udb_profile_begin was called)
struct ProfEntry {
  const char* name;
  cudaEvent_t ev;
  double flops, bytes;
};
static std::vector<ProfEntry> g_prof;
static bool g_prof_on = false;
static cudaStream_t g_prof_stream = nullptr;
static cudaEvent_t g_prof_start = nullptr;
static thread_local double g_flops = 0.0, g_bytes = 0.0;

void note_work(double flops, double bytes) {
  g_flops = flops;
  g_bytes = bytes;
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return 1;
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  if (g_prof_on) {
    ProfEntry pe{what, nullptr, g_flops, g_bytes};
    if (cudaEventCreate(&pe.ev) == cudaSuccess && cudaEventRecord(pe.ev, g_prof_stream) == cudaSuccess) g_prof.push_back(pe);
  }
  g_flops = g_bytes = 0.0;
  return 0;
}

int num_sms() {
  static std::atomic<int> per_dev[64];
  int dev = 0;
  cudaGetDevice(&dev);
  int n = per_dev[dev & 63].load(std::memory_order_relaxed);
  if (n == 0) {
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
    per_dev[dev & 63].store(n, std::memory_order_relaxed);
  }
  return n;
}

int check_dims(const char* fn, std::initializer_list<NamedDim> dims) {
  for (const auto& d : dims)
    if (d.v < 1) { set_error("%s: %s=%d must be >= 1", fn, d.name, d.v); return 1; }
  return 0;
}

int check_ptrs(const char* fn, std::initializer_list<NamedPtr> ptrs, int align, const char* noun) {
  for (const auto& a : ptrs) {
    if (align > 0 && (!a.p || reinterpret_cast<uintptr_t>(a.p) % align)) {
      set_error("%s: `%s` must be a non-null, %d-byte aligned %s", fn, a.name, align, noun);
      return 1;
    }
    if (!a.p) { set_error("%s: `%s` must be non-null", fn, a.name); return 1; }
  }
  return 0;
}

bool pdl_enabled() {
  static const bool on = [] {
    const char* e = getenv("UDB_PDL");
    return e ? atoi(e) != 0 : true;
  }();
  return on;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) {
      set_error("cuTensorMapEncodeTiled entry point unavailable (%s)", cudaGetErrorString(e));
      return nullptr;
    }
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int make_tmap(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
              const uint32_t* box, CUtensorMapDataType dtype, CUtensorMapSwizzle swizzle) {
  EncodeTiledFn fn = get_encode();
  if (!fn) return 1;
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) gstr[i - 1] = strides_bytes[i - 1];
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) {
    set_error("TMA base pointer %p is not 16-byte aligned", base);
    return 1;
  }
  for (int i = 0; i + 1 < rank; ++i) {
    if (gstr[i] % 16 != 0) {
      set_error("TMA stride %d = %llu bytes is not a multiple of 16", i, (unsigned long long)gstr[i]);
      return 1;
    }
  }
  CUresult r = fn(map, dtype, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed: CUresult %d (rank %d dims %llu,%llu box %u,%u)", (int)r,
              rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0), box[0],
              rank > 1 ? box[1] : 0);
    return 1;
  }
  return 0;
}

}  // namespace udb

extern "C" {
int udb_version(void) { return UDB_VERSION; }
const char* udb_last_error(void) { return udb::g_err; }
int64_t udb_launch_count(void) { return udb::g_launches.load(); }

int udb_profile_begin(void* stream) {
  using namespace udb;
  if (g_prof_on) { set_error("udb_profile_begin: already profiling"); return 1; }
  g_prof.clear();
  g_prof_stream = reinterpret_cast<cudaStream_t>(stream);
  if (cudaEventCreate(&g_prof_start) != cudaSuccess || cudaEventRecord(g_prof_start, g_prof_stream) != cudaSuccess) {
    set_error("udb_profile_begin: event creation failed");
    return 1;
  }
  g_prof_on = true;
  return 0;
}

int udb_profile_end(udb_profile_entry_t* out, int32_t cap) {
  using namespace udb;
  if (!g_prof_on) { set_error("udb_profile_end: not profiling"); return -1; }
  g_prof_on = false;
  cudaStreamSynchronize(g_prof_stream);
  cudaEvent_t prev = g_prof_start;
  int n = 0;
  for (auto& pe : g_prof) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, prev, pe.ev);
    if (out && n < cap) {
      strncpy(out[n].name, pe.name, sizeof(out[n].name) - 1);
      out[n].name[sizeof(out[n].name) - 1] = 0;
      out[n].ms = ms;
      out[n].flops = pe.flops;
      out[n].bytes = pe.bytes;
    }
    ++n;
    if (prev != g_prof_start) cudaEventDestroy(prev);
    prev = pe.ev;
  }
  if (prev != g_prof_start) cudaEventDestroy(prev);
  cudaEventDestroy(g_prof_start);
  g_prof.clear();
  return n;
}
}
