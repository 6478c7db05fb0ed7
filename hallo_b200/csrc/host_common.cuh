// Host-side helpers shared by the C-ABI translation units: error string, launch counter,
// and cuTensorMapEncodeTiled obtained through the runtime (no link-time libcuda dependency).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>

#include "../../include/hallo_b200.h"

namespace hb {

extern char g_last_error[512];
extern std::atomic<int64_t> g_launch_count;

// run-time kernel-selection switches (hallo_b200_set_option); initial value from HALLO_B200_<NAME>
enum Option { OPT_XATTN_TC = 0, OPT_TATTN_MMA, OPT_GN_FUSED, OPT_GEMM_SPLITK, OPT_PDL, OPT_COUNT };
int option(Option o);

inline int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
  return code;
}

#define HB_CUDA_CHECK(expr)                                                              \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess)                                                               \
      return hb::fail(HB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                      __FILE__, __LINE__);                                               \
  } while (0)

#define HB_LAUNCH_CHECK()                                                                   \
  do {                                                                                      \
    hb::g_launch_count.fetch_add(1, std::memory_order_relaxed);                             \
    cudaError_t _e = cudaGetLastError();                                                    \
    if (_e != cudaSuccess)                                                                  \
      return hb::fail(HB_ERR_CUDA, "kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), \
                      __FILE__, __LINE__);                                                  \
  } while (0)

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode_tiled();

// rank-R tiled tensor map over 16-bit elements, 128B (or 64B / 32B) swizzle, zero OOB fill.
// dims/strides innermost first; strides_bytes has rank-1 entries (dims 1..R-1).
int make_tmap_16b(CUtensorMap* out, int dtype, const void* base, int rank, const uint64_t* dims,
                  const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes = 128);

inline int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// Every kernel launch of the library goes through here.  `cluster` > 1 sets the cluster dimension; with option "pdl"
// the launch carries programmatic stream serialization, i.e. the kernel may become resident while its predecessor
// drains -- every kernel launched this way calls pdl_wait() (ptx.cuh) before it touches global memory.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel_cluster(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                         int cluster, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (cluster > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  if (option(OPT_PDL) != 0) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                 Args&&... args) {
  return launch_kernel_cluster(kern, grid, block, smem, stream, 1, static_cast<Args&&>(args)...);
}

}  // namespace hb
