// Thin inline-PTX wrappers for the sm_90a features the kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), the wgmma shared-memory descriptor and fences, and the
// warp-level mma.sync / ldmatrix / cp.async path.
//
// The descriptor bit layout follows the PTX ISA "matrix descriptor" table of wgmma (the same fields
// CUTLASS names GmmaDescriptor).
#pragma once
#include <cstdint>
#include <cuda_fp16.h>
#include <cuda_bf16.h>

namespace hb {

// ------------------------------------------------------------------------------------------
// misc
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// Device-side error word: kernels that time out on a barrier write a code here and trap,
// so a wrong descriptor cannot hang the GPU.
static __device__ unsigned int g_hb_error = 0;

// ------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: ~2 s at 2 GHz, then record an error code and trap (kills the context, not the GPU).
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, uint32_t code = 1) {
  if (mbar_try_wait(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) {
      atomicExch(&g_hb_error, code | (blockIdx.x << 8));
      __trap();
    }
  }
}

// ------------------------------------------------------------------------------------------
// TMA tiled loads (tensor maps are passed as __grid_constant__ kernel parameters)
// ------------------------------------------------------------------------------------------
// Programmatic dependent launch (option "pdl"): a kernel launched with programmatic stream serialization may start
// while its predecessor in the stream is still draining.  pdl_wait() blocks until the predecessor grid has completed
// and its memory is visible (a no-op without the launch attribute) and must precede every global access; pdl_launch()
// lets the successor's CTAs be scheduled.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;\n" ::: "memory"); }
__device__ __forceinline__ void pdl_launch() { asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory"); }

__device__ __forceinline__ void prefetch_l1(const void* p) {
  asm volatile("prefetch.global.L1 [%0];\n" ::"l"(p));
}
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];\n" ::"l"(tmap) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const void* tmap, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];\n" ::"r"(smem_u32(dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const void* tmap, uint64_t* bar, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];\n" ::"r"(smem_u32(dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const void* tmap, uint64_t* bar, int c0,
                                            int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];\n" ::"r"(smem_u32(dst)),
      "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// TMA tiled stores (shared -> global, bulk-group completion).  The box is clipped against the tensor bounds, so
// ragged row / column tails need no masking.  Generic-proxy writes to the source buffer must be followed by
// fence_proxy_async_smem() + a barrier before the elected thread issues the store.
__device__ __forceinline__ void tma_store_2d(const void* tmap, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];\n" ::"l"(tmap),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_4d(const void* tmap, const void* src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];\n" ::"l"(tmap),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void sts128(uint32_t saddr, const uint4& v) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};\n" ::"r"(saddr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t saddr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];\n" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(saddr)
               : "memory");
  return v;
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
// wait until at most N of this thread's bulk groups still READ their shared-memory source (buffer reusable)
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;\n" ::"n"(N) : "memory");
}
// wait until at most N bulk groups are incomplete (global writes performed)
template <int N>
__device__ __forceinline__ void bulk_wait_group() {
  asm volatile("cp.async.bulk.wait_group %0;\n" ::"n"(N) : "memory");
}

// ------------------------------------------------------------------------------------------
// wgmma: shared-memory matrix descriptors and the warpgroup fences (the MMAs themselves: wgmma.cuh)
// ------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor, 128-byte swizzle, tile base 1024-byte aligned.
//   bits [0,14)  start address >> 4        bits [16,30) leading byte offset >> 4
//   bits [32,46) stride byte offset >> 4   bits [62,64) layout type (1 = SWIZZLE_128B)
// K-major operand  : rows of 128 B (64 halfs), 8-row groups 1024 B apart -> SBO = 1024, LBO unused.
// MN-major operand : 64 MN-elements contiguous (128 B) per k-row, 8 k-rows = 1024 B (SBO),
//                    next 64-wide MN panel LBO bytes away.
// Advancing 16 elements along K inside a 128 B swizzle row adds 32 B, i.e. +2 to the descriptor.
__device__ __forceinline__ uint64_t make_desc_sw128(uint32_t saddr, uint32_t lbo_bytes,
                                                    uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
// orders this thread's register writes of accumulators / A fragments before the next wgmma reads them
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
// wait until at most N committed wgmma groups of this warpgroup are still pending
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across an asynchronous wgmma
template <int R>
__device__ __forceinline__ void wgmma_pin(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ------------------------------------------------------------------------------------------
// small numeric helpers shared by the kernels
// ------------------------------------------------------------------------------------------
template <typename T>
struct Cvt;
template <>
struct Cvt<__half> {
  __device__ static __forceinline__ float to_f(__half v) { return __half2float(v); }
  __device__ static __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
  __device__ static __forceinline__ uint32_t pack2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
  __device__ static __forceinline__ float2 unpack2(uint32_t u) {
    __half2 h = *reinterpret_cast<__half2*>(&u);
    return __half22float2(h);
  }
};
template <>
struct Cvt<__nv_bfloat16> {
  __device__ static __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
  __device__ static __forceinline__ __nv_bfloat16 from_f(float v) {
    return __float2bfloat16_rn(v);
  }
  __device__ static __forceinline__ uint32_t pack2(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
  }
  __device__ static __forceinline__ float2 unpack2(uint32_t u) {
    __nv_bfloat162 h = *reinterpret_cast<__nv_bfloat162*>(&u);
    return __bfloat1622float2(h);
  }
};

// named barriers (ids 1..15; 0 is __syncthreads): sub-CTA producer/consumer hand-offs
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ float max3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// exp2 on the FMA / ALU pipes (no MUFU): round-to-nearest split x = n + f, degree-3 minimax 2^f on [-0.5, 0.5]
// (max rel. error 7.5e-5, far below half precision), exponent inserted with an integer add.  x <= ~2^22.
__device__ __forceinline__ float exp2_poly(float x) {
  x = fmaxf(x, -126.0f);
  const float t = x + 12582912.0f;                    // 1.5 * 2^23: the low mantissa bits of t hold rint(x)
  const float f = x - (t - 12582912.0f);
  float p = fmaf(f, 0.0551716481f, 0.242611121f);
  p = fmaf(p, f, 0.693260989f);
  p = fmaf(p, f, 0.999928074f);
  return __int_as_float(__float_as_int(p) + (__float_as_int(t) << 23));
}
// volatile variant: keeps its place in the instruction stream (used to batch MUFU issue)
__device__ __forceinline__ float fast_exp2_v(float x) {
  float y;
  asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float gelu_erf(float x) {
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f));
}
// erf-GELU with the Abramowitz-Stegun 7.1.26 erf (|abs err| < 1.5e-7): one rcp + one ex2 instead of erff()
__device__ __forceinline__ float gelu_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));   // MUFU.RCP, not the IEEE sequence
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  poly *= t;
  const float e = poly * fast_exp2(-z * z * 1.4426950408889634f);   // 1 - erf(z)
  const float erf_abs = 1.0f - e;
  const float erfx = copysignf(erf_abs, x);
  return 0.5f * x * (1.0f + erfx);
}
// x * sigmoid(x) with one ex2.approx and one rcp.approx (the IEEE division of `x / (1 + exp(-x))` costs ~8 extra
// instructions per element, which matters in the HBM-bound GroupNorm-apply + SiLU)
__device__ __forceinline__ float silu_f(float x) {
  const float e = fast_exp2(-1.4426950408889634f * x);
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return x * r;
}

// ------------------------------------------------------------------------------------------
// warp-level tensor-core path (mma.sync m16n8k16, ldmatrix, cp.async): the small-problem kernels
// ------------------------------------------------------------------------------------------
template <typename T>
struct WarpMma;
template <>
struct WarpMma<__half> {
  static __device__ __forceinline__ void mma(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
        "{%0, %1, %2, %3};\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
  }
};
template <>
struct WarpMma<__nv_bfloat16> {
  static __device__ __forceinline__ void mma(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
        "{%0, %1, %2, %3};\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
  }
};

__device__ __forceinline__ void ldsm_x4(uint32_t saddr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];\n"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(saddr)
               : "memory");
}
__device__ __forceinline__ void ldsm_x2(uint32_t saddr, uint32_t (&r)[2]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];\n" : "=r"(r[0]), "=r"(r[1]) : "r"(saddr) : "memory");
}
__device__ __forceinline__ void ldsm_x2_trans(uint32_t saddr, uint32_t (&r)[2]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];\n"
               : "=r"(r[0]), "=r"(r[1])
               : "r"(saddr)
               : "memory");
}
__device__ __forceinline__ void cp_async16(uint32_t saddr, const void* gptr) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(saddr), "l"(gptr) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

}  // namespace hb
