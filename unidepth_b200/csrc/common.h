// Host-side helpers shared by the .cu files: error reporting, launch counting, TMA tensor maps.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <initializer_list>

#include "../../include/udb.h"

namespace udb {

void set_error(const char* fmt, ...);
extern std::atomic<int64_t> g_launches;

// Called after every kernel launch of this library: error check, launch counting and -- between udb_profile_begin /
// udb_profile_end -- a CUDA event per launch so that per-kernel durations can be read back (bench.py's rooflines).
int check_launch(const char* what);
// Algorithmic work of the launch that follows (consumed by its check_launch): flops and bytes moved, for the profile.
void note_work(double flops, double bytes);

int num_sms();   // of the CURRENT device (cached per device)

#define ST(s) reinterpret_cast<cudaStream_t>(s)

// Blocks of 256 threads for a grid-stride loop over `total` items: at least 1, at most per_sm per SM.
inline int grid_1d(long long total, int per_sm) {
  const long long g = (total + 255) / 256, cap = (long long)num_sms() * per_sm;
  return (int)(g > cap ? cap : (g < 1 ? 1 : g));
}

// Argument checks of the launchers: 0 when they hold, else 1 with the error "<fn>: <name>=<v> must be >= 1",
// "<fn>: `<name>` must be non-null" or, with align > 0, "<fn>: `<name>` must be a non-null, <align>-byte aligned <noun>".
struct NamedDim { int v; const char* name; };
struct NamedPtr { const void* p; const char* name; };
int check_dims(const char* fn, std::initializer_list<NamedDim> dims);
int check_ptrs(const char* fn, std::initializer_list<NamedPtr> ptrs, int align = 0, const char* noun = "pointer");

// Shape bounds of udb_cross_attn_small(_f32): 0, or 1 with the error set under the name `fn`.  The V1 engine checks its
// camera head's context length with it before anything is enqueued, so that its dry run names the bound.
int cross_attn_small_check(const char* fn, int nq, int nk, int D);

// true the first time it is called on the current device for this mask (per-device one-time setup such as
// cudaFuncSetAttribute: function attributes are per device / context, not per process)
inline bool first_on_device(std::atomic<uint64_t>& mask) {
  int d = 0;
  cudaGetDevice(&d);
  const uint64_t bit = 1ull << (d & 63);
  return !(mask.fetch_or(bit) & bit);
}

// UDB_PDL=0 disables programmatic dependent launch (default on)
bool pdl_enabled();

// Launch with optional cluster dimension and the programmatic-stream-serialization attribute.
template <typename Kernel, typename... Args>
inline cudaError_t launch_ex(Kernel kernel, dim3 grid, dim3 block, size_t smem, cudaStream_t st, int cluster_x,
                             Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  if (pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time libcuda).
// dims/strides innermost first; strides_bytes has rank-1 entries (stride of dim 1..rank-1).
int make_tmap(CUtensorMap* map, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
              const uint32_t* box, CUtensorMapDataType dtype, CUtensorMapSwizzle swizzle);
inline int make_tmap_f16(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                         const uint64_t* strides_bytes, const uint32_t* box, bool swizzle128) {
  return make_tmap(map, base, rank, dims, strides_bytes, box, CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                   swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE);
}

}  // namespace udb
