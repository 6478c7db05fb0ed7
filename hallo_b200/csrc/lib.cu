// Unity translation unit: the whole C-ABI library is one TU so that the device error word and
// the launch counter have exactly one definition (no -rdc needed).
#include "host_common.cu"
#include "gemm_tc.cu"
#include "attn_tc.cu"
#include "attn_api.cu"
#include "tattn_mma.cu"
#include "aux.cu"
#include "peer.cu"

extern "C" int hallo_b200_device_error(unsigned int* code_out) {
  unsigned int v = 0;
  cudaError_t e = cudaMemcpyFromSymbol(&v, hb::g_hb_error, sizeof(v));
  if (e != cudaSuccess) return hb::fail(HB_ERR_CUDA, "device error word unreadable: %s", cudaGetErrorString(e));
  if (v != 0) {
    unsigned int z = 0;
    cudaMemcpyToSymbol(hb::g_hb_error, &z, sizeof(z));
  }
  if (code_out) *code_out = v;
  return v != 0 ? HB_ERR_DEVICE_TRAP : HB_OK;
}
