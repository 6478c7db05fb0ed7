// C entry point of hallo_b200_attention: picks the kernel instance per head dim.
#include "host_common.cuh"
#include <cstdlib>

namespace hb {

template <typename T>
static int dispatch_attn(const hb_attention_params* p, cudaStream_t s) {
  // template arguments: head dim, K / V ring depth, CTAs per SM (registers: O grows with the head dim)
  switch (p->head_dim) {
    case 40: return launch_attn<T, 40, 3, 2>(p, s);
    case 80: return launch_attn<T, 80, 2, 1>(p, s);
    case 160: return launch_attn<T, 160, 2, 1>(p, s);
    default: return fail(HB_ERR_BAD_SHAPE, "attention: head_dim %d not in {40, 80, 160}", p->head_dim);
  }
}

}  // namespace hb

extern "C" int hallo_b200_attention(const hb_attention_params* p, hb_stream_t stream) {
  using namespace hb;
  if (p == nullptr || p->Q == nullptr || p->K == nullptr || p->V == nullptr || p->O == nullptr)
    return fail(HB_ERR_NULL, "hallo_b200_attention: null pointer");
  if (p->L <= 0 || p->frames <= 0 || p->heads <= 0 || p->heads > 256)
    return fail(HB_ERR_BAD_SHAPE, "hallo_b200_attention: L=%d frames=%d heads=%d", p->L, p->frames, p->heads);
  if (p->ldq % 8 || p->ldk % 8 || p->ldv % 8 || p->ldo % 8)
    return fail(HB_ERR_BAD_SHAPE, "hallo_b200_attention: leading dims must be multiples of 8");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (p->dtype == HB_F16) return dispatch_attn<__half>(p, s);
  if (p->dtype == HB_BF16) return dispatch_attn<__nv_bfloat16>(p, s);
  return fail(HB_ERR_BAD_DTYPE, "hallo_b200_attention: dtype %d", p->dtype);
}
