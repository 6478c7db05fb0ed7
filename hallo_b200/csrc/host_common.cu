#include "host_common.cuh"

#include <cctype>
#include <cstdlib>
#include <cstring>
#include <mutex>

namespace hb {

char g_last_error[512] = "";
std::atomic<int64_t> g_launch_count{0};

static const char* const kOptionNames[OPT_COUNT] = {"xattn_tc", "tattn_mma", "gn_fused", "gemm_splitk", "pdl"};
// defaults: the tensor-core / fused kernels are ON; setting an option to 0 selects the CUDA-core or unfused kernel
// (A/B measurements).  pdl (programmatic dependent launch) is opt-in.
static const int kOptionDefaults[OPT_COUNT] = {1, 1, 1, 1, 0};
static std::atomic<int> g_options[OPT_COUNT];
static std::atomic<bool> g_options_init{false};

static void init_options() {
  if (g_options_init.load(std::memory_order_acquire)) return;
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  if (g_options_init.load(std::memory_order_relaxed)) return;
  for (int i = 0; i < OPT_COUNT; ++i) {
    char env[64] = "HALLO_B200_";
    size_t n = strlen(env);
    for (const char* c = kOptionNames[i]; *c && n + 1 < sizeof(env); ++c) env[n++] = (char)toupper((unsigned char)*c);
    env[n] = 0;
    const char* v = getenv(env);
    // a variable that is set but empty or non-numeric counts as 1 (the historical "defined = on" switches)
    int val = kOptionDefaults[i];
    if (v != nullptr) val = (*v >= '0' && *v <= '9') ? atoi(v) : 1;
    g_options[i].store(val, std::memory_order_relaxed);
  }
  g_options_init.store(true, std::memory_order_release);
}

int option(Option o) {
  init_options();
  return g_options[o].load(std::memory_order_relaxed);
}
static int find_option(const char* name) {
  if (name == nullptr) return -1;
  for (int i = 0; i < OPT_COUNT; ++i)
    if (strcmp(name, kOptionNames[i]) == 0) return i;
  return -1;
}

PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || p == nullptr) return nullptr;
  fn = reinterpret_cast<PFN_encodeTiled>(p);
  return fn;
}

int make_tmap_16b(CUtensorMap* out, int dtype, const void* base, int rank, const uint64_t* dims,
                  const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return fail(HB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0)
    return fail(HB_ERR_BAD_SHAPE, "tensor map base %p not 16B aligned", base);
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (box[i] == 0 || box[i] > 256) return fail(HB_ERR_BAD_SHAPE, "tmap box[%d]=%u", i, box[i]);
  }
  for (int i = 0; i + 1 < rank; ++i) {
    gstr[i] = strides_bytes[i];
    if (gstr[i] % 16 != 0)
      return fail(HB_ERR_BAD_SHAPE, "tmap stride[%d]=%llu not a multiple of 16 B", i,
                  (unsigned long long)gstr[i]);
  }
  CUtensorMapDataType dt =
      dtype == HB_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  if (swizzle_bytes != 128 && swizzle_bytes != 64) return fail(HB_ERR_BAD_SHAPE, "tmap swizzle %d", swizzle_bytes);
  if ((uint64_t)box[0] * 2 > (uint64_t)swizzle_bytes)
    return fail(HB_ERR_BAD_SHAPE, "tmap inner box %u x 2 B exceeds the %d B swizzle span", box[0], swizzle_bytes);
  CUresult r = enc(out, dt, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    return fail(HB_ERR_CUDA,
                "cuTensorMapEncodeTiled failed (%d): rank %d dims [%llu %llu %llu %llu] box [%u %u %u %u]",
                (int)r, rank, (unsigned long long)gdim[0], (unsigned long long)(rank > 1 ? gdim[1] : 0),
                (unsigned long long)(rank > 2 ? gdim[2] : 0), (unsigned long long)(rank > 3 ? gdim[3] : 0),
                bx[0], rank > 1 ? bx[1] : 0, rank > 2 ? bx[2] : 0, rank > 3 ? bx[3] : 0);
  }
  return HB_OK;
}

}  // namespace hb

extern "C" {

int hallo_b200_abi_version(void) { return 3; }
int hallo_b200_sizeof_gemm_params(void) { return (int)sizeof(hb_gemm_params); }
int hallo_b200_sizeof_attention_params(void) { return (int)sizeof(hb_attention_params); }

const char* hallo_b200_last_error(void) { return hb::g_last_error; }

int hallo_b200_set_option(const char* name, int value) {
  hb::init_options();
  const int i = hb::find_option(name);
  if (i < 0) return hb::fail(HB_ERR_BAD_SHAPE, "hallo_b200_set_option: unknown option '%s'", name ? name : "(null)");
  hb::g_options[i].store(value, std::memory_order_relaxed);
  return HB_OK;
}
int hallo_b200_get_option(const char* name) {
  hb::init_options();
  const int i = hb::find_option(name);
  return i < 0 ? -1 : hb::g_options[i].load(std::memory_order_relaxed);
}

int64_t hallo_b200_launch_count(int reset) {
  int64_t v = hb::g_launch_count.load();
  if (reset) hb::g_launch_count.store(0);
  return v;
}

}  // extern "C"
