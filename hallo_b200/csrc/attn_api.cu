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
    case 512: return launch_attn_wide<T>(p, s);     // one head, V / O columns split over 4 CTAs
    default: return fail(HB_ERR_BAD_SHAPE, "attention: head_dim %d not in {40, 80, 160, 512}", p->head_dim);
  }
}

}  // namespace hb

extern "C" int hallo_b200_attention(const hb_attention_params* p, hb_stream_t stream) {
  using namespace hb;
  // Every argument check happens here, before any driver call or launch, so a bad call fails the same way with or
  // without a device.
  if (p == nullptr || p->Q == nullptr || p->K == nullptr || p->V == nullptr || p->O == nullptr)
    return fail(HB_ERR_NULL, "hallo_b200_attention: null pointer");
  const bool has_ref = p->ref_index != nullptr;
  if (has_ref && (p->Kref == nullptr || p->Vref == nullptr || p->ref_frames <= 0))
    return fail(HB_ERR_NULL, "hallo_b200_attention: ref_index given without Kref/Vref (ref_frames=%d)", p->ref_frames);
  if (p->L <= 0 || p->frames <= 0 || p->heads <= 0 || p->heads > 256)
    return fail(HB_ERR_BAD_SHAPE, "hallo_b200_attention: L=%d frames=%d heads=%d", p->L, p->frames, p->heads);
  if (p->ldq % 8 || p->ldk % 8 || p->ldv % 8 || p->ldo % 8 || (has_ref && (p->ldkref % 8 || p->ldvref % 8)))
    return fail(HB_ERR_BAD_SHAPE, "hallo_b200_attention: leading dims must be multiples of 8");
  // Q / K / V (and Kref / Vref) are read by TMA: 16-byte aligned bases.  Both kernels store O two elements at a time
  // as one 32-bit word, so O must be 4-byte aligned (an O view at an odd element offset would fault).
  const auto misaligned = [](const void* a, uintptr_t n) { return (reinterpret_cast<uintptr_t>(a) & (n - 1)) != 0; };
  if (misaligned(p->Q, 16) || misaligned(p->K, 16) || misaligned(p->V, 16) ||
      (has_ref && (misaligned(p->Kref, 16) || misaligned(p->Vref, 16))))
    return fail(HB_ERR_BAD_SHAPE, "hallo_b200_attention: Q/K/V/Kref/Vref must be 16-byte aligned");
  if (misaligned(p->O, 4))
    return fail(HB_ERR_BAD_SHAPE, "hallo_b200_attention: O %p must be 4-byte aligned", p->O);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (p->dtype == HB_F16) return dispatch_attn<__half>(p, s);
  if (p->dtype == HB_BF16) return dispatch_attn<__nv_bfloat16>(p, s);
  return fail(HB_ERR_BAD_DTYPE, "hallo_b200_attention: dtype %d", p->dtype);
}
