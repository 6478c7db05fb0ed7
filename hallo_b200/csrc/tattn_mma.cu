// Temporal self-attention (motion_module.py:553-609) on warp-level tensor-core MMAs.
//
// The op is a batch of tiny attentions -- per (pixel, head): Q [Fq x d] against K, V [Fk x d], Fk <= 32 frames --
// whose rows lie L*ld elements apart in the token matrices.  wgmma (M = 64 tiles, operands through
// descriptors) has nothing to grab here, and the job is HBM-bound anyway (q/k/v read once, o written once), so the
// kernel uses mma.sync m16n8k16 -- enough to take the ~5000 scalar FMA/convert instructions per thread of the
// CUDA-core kernel off the critical path:
//   1. the CTA copies the Q, K, V rows of PIX pixels (all frames, all heads) into shared memory with 16-byte
//      cp.async; rows are padded so that the 8 frame-rows of an ldmatrix fall into different bank groups;
//   2. each warp takes (pixel, head) tasks: S = Q K^T (A, B via ldmatrix), masked softmax on the accumulator
//      fragments (quad shuffles), O = P V (P re-packed from the S fragments, V via ldmatrix.trans), O written over
//      the task's own Q slice in shared memory;
//   3. the CTA copies the O rows out with coalesced 16-byte stores.
// Option "tattn_mma" (default on); 0 selects the CUDA-core kernel in aux.cu.
#include "host_common.cuh"
#include "ptx.cuh"

namespace hb {

constexpr int kTattnThreads = 256;

// D: head dim (multiple of 8); MT: 16-row query tiles (Fq <= 16 MT); NT: 8-key tiles (Fk <= 8 NT)
template <typename T, int D, int MT, int NT>
__global__ void __launch_bounds__(kTattnThreads)
tattn_mma_kernel(const T* __restrict__ Q, long long ldq, const T* __restrict__ K, const T* __restrict__ V,
                 long long ldkv, T* __restrict__ O, long long ldo, int Fq, int Fk, int L, int heads, int pix_per_cta,
                 int ps, int fs, float scale_log2) {
  pdl_wait();
  pdl_launch();
  extern __shared__ uint4 tattn_smem[];
  constexpr int KS = (D + 15) / 16;           // k-steps of Q K^T
  constexpr bool kHalfStep = (D % 16) == 8;   // the last k-step only holds 8 real dims
  constexpr int KK = (NT + 1) / 2;            // k-steps (16 keys) of P V
  constexpr int NJ = D / 8;                   // 8-dim output tiles
  const int C = heads * D;
  const int cvec = C >> 3;
  const int b = blockIdx.y;
  const int pix0 = blockIdx.x * pix_per_cta;
  const int npix = min(pix_per_cta, L - pix0);
  const uint32_t s0 = smem_u32(tattn_smem);
  const uint32_t sQ = s0, sK = s0 + (uint32_t)Fq * fs, sV = sK + (uint32_t)Fk * fs;

  // ---- 1. global -> shared (row (f, p) of a matrix at f*fs + p*ps) ----
  {
    const int rows_q = Fq * npix, rows_kv = Fk * npix;
    const int total = (rows_q + 2 * rows_kv) * cvec;
    for (int i = threadIdx.x; i < total; i += kTattnThreads) {
      const int v = i % cvec;
      int r = i / cvec;
      const T* src;
      uint32_t dst;
      if (r < rows_q) {
        const int f = r / npix, p = r - f * npix;
        src = Q + (((long long)b * Fq + f) * L + pix0 + p) * ldq + v * 8;
        dst = sQ + f * fs + p * ps + v * 16;
      } else {
        r -= rows_q;
        const bool isv = r >= rows_kv;
        if (isv) r -= rows_kv;
        const int f = r / npix, p = r - f * npix;
        src = (isv ? V : K) + (((long long)b * Fk + f) * L + pix0 + p) * ldkv + v * 8;
        dst = (isv ? sV : sK) + f * fs + p * ps + v * 16;
      }
      cp_async16(dst, src);
    }
    cp_async_wait_all();
  }
  __syncthreads();

  // ---- 2. per-warp (pixel, head) attention on fragments ----
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  for (int task = warp; task < npix * heads; task += kTattnThreads / 32) {
    const int p = task / heads, h = task - p * heads;
    const uint32_t toff = (uint32_t)p * ps + (uint32_t)h * (D * 2);
    float s[MT][NT][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) s[mt][nt][e] = 0.f;

#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      uint32_t a[MT][4];
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        const int row = min(mt * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, Fq - 1);   // rows past Fq: any valid row
        ldsm_x4(sQ + toff + row * fs + (2 * ks + (lane >> 4)) * 16, a[mt]);
        if (kHalfStep && ks == KS - 1) a[mt][2] = a[mt][3] = 0u;                    // dims d .. d+7 belong to the next head
      }
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        uint32_t bk[2];
        const int key = min(nt * 8 + (lane & 7), Fk - 1);                            // keys past Fk are masked below
        ldsm_x2(sK + toff + key * fs + (2 * ks + ((lane >> 3) & 1)) * 16, bk);
        if (kHalfStep && ks == KS - 1) bk[1] = 0u;
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) WarpMma<T>::mma(s[mt][nt], a[mt], bk);
      }
    }

    // masked softmax over the keys; C fragment: [0], [1] = row g, keys 8 nt + 2t, +1;  [2], [3] = row g + 8
    float inv[MT][2];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float mx = -INFINITY;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float v = s[mt][nt][hh * 2 + e];
            if (nt * 8 + 2 * t + e >= Fk) v = -INFINITY;
            s[mt][nt][hh * 2 + e] = v;
            mx = fmaxf(mx, v);
          }
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        float sum = 0.f;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float pe = fast_exp2((s[mt][nt][hh * 2 + e] - mx) * scale_log2);   // exp2(-inf) = 0 for masked keys
            s[mt][nt][hh * 2 + e] = pe;
            sum += pe;
          }
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
        inv[mt][hh] = 1.0f / sum;
      }

    // P as A fragments: two adjacent key tiles of S make one 16-key k-step
    uint32_t pa[MT][KK][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int kk = 0; kk < KK; ++kk) {
        pa[mt][kk][0] = Cvt<T>::pack2(s[mt][2 * kk][0], s[mt][2 * kk][1]);
        pa[mt][kk][1] = Cvt<T>::pack2(s[mt][2 * kk][2], s[mt][2 * kk][3]);
        if (2 * kk + 1 < NT) {
          pa[mt][kk][2] = Cvt<T>::pack2(s[mt][2 * kk + 1][0], s[mt][2 * kk + 1][1]);
          pa[mt][kk][3] = Cvt<T>::pack2(s[mt][2 * kk + 1][2], s[mt][2 * kk + 1][3]);
        } else {
          pa[mt][kk][2] = pa[mt][kk][3] = 0u;
        }
      }

    // O = P V, 8 output dims at a time; results replace this task's Q slice (only this warp reads it, and all of
    // its ldmatrix reads of Q are behind us)
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      float o[MT][4];
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int e = 0; e < 4; ++e) o[mt][e] = 0.f;
#pragma unroll
      for (int kk = 0; kk < KK; ++kk) {
        uint32_t bv[2];
        const int key = min(kk * 16 + (lane & 15), Fk - 1);                          // P is 0 for keys past Fk
        ldsm_x2_trans(sV + toff + key * fs + j * 16, bv);
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) WarpMma<T>::mma(o[mt], pa[mt][kk], bv);
      }
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int frame = mt * 16 + g + hh * 8;
          if (frame < Fq) {
            const uint32_t val = Cvt<T>::pack2(o[mt][hh * 2] * inv[mt][hh], o[mt][hh * 2 + 1] * inv[mt][hh]);
            asm volatile("st.shared.b32 [%0], %1;\n" ::"r"(sQ + toff + frame * fs + (8 * j + 2 * t) * 2), "r"(val) : "memory");
          }
        }
    }
    __syncwarp();
  }
  __syncthreads();

  // ---- 3. shared -> global, coalesced rows ----
  {
    const int total = Fq * npix * cvec;
    for (int i = threadIdx.x; i < total; i += kTattnThreads) {
      const int v = i % cvec;
      const int r = i / cvec;
      const int f = r / npix, p = r - f * npix;
      const uint4 val = lds128(sQ + f * fs + p * ps + v * 16);
      *reinterpret_cast<uint4*>(O + (((long long)b * Fq + f) * L + pix0 + p) * ldo + v * 8) = val;
    }
  }
}

template <typename T, int D, int MT, int NT>
static int launch_tattn_mma(const void* Q, long long ldq, const void* K, const void* V, long long ldkv, void* O,
                            long long ldo, int batch, int Fq, int Fk, int L, int heads, cudaStream_t s) {
  const int C = heads * D;
  const int ps = C * 2 + 16;                                   // row pitch: 16-byte pad
  const int rows = Fq + 2 * Fk;
  int pix = (72 * 1024) / (rows * ps);                         // ~72 KB per CTA: three CTAs per SM at C = 320
  if (pix < 1) pix = 1;
  if (pix > 4) pix = 4;
  if (pix > L) pix = L;
  int fs = pix * ps;
  if (((fs >> 4) & 1) == 0) fs += 16;                          // frame stride = odd multiple of 16 B: the 8 rows of an
                                                               // ldmatrix land in 8 different bank groups
  const size_t smem = (size_t)rows * fs;
  if (smem > 220 * 1024) return 1;
  auto kern = tattn_mma_kernel<T, D, MT, NT>;
  static bool attr_set = false;
  if (!attr_set) {
    HB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    attr_set = true;
  }
  dim3 grid((L + pix - 1) / pix, batch);
  const float sc = (float)(1.4426950408889634 / sqrt((double)D));
  launch_kernel(kern, grid, kTattnThreads, smem, s, (const T*)Q, ldq, (const T*)K, (const T*)V, ldkv, (T*)O, ldo, Fq, Fk, L, heads,
                                         pix, ps, fs, sc);
  HB_LAUNCH_CHECK();
  return HB_OK;
}

template <typename T, int D>
static int dispatch_tattn_mma(const void* Q, long long ldq, const void* K, const void* V, long long ldkv, void* O,
                              long long ldo, int batch, int Fq, int Fk, int L, int heads, cudaStream_t s) {
#define HB_TM(MT_, NT_) return launch_tattn_mma<T, D, MT_, NT_>(Q, ldq, K, V, ldkv, O, ldo, batch, Fq, Fk, L, heads, s)
  if (Fq <= 16) {
    if (Fk <= 8) HB_TM(1, 1);
    if (Fk <= 24) HB_TM(1, 3);
    HB_TM(1, 4);
  }
  if (Fk <= 8) HB_TM(2, 1);
  if (Fk <= 24) HB_TM(2, 3);
  HB_TM(2, 4);
#undef HB_TM
}

// returns HB_OK if handled, 1 if the shape is left to the CUDA-core kernels, < 0 on error
int tattn_mma_try(int dtype, const void* Q, long long ldq, const void* K, const void* V, long long ldkv, void* O,
                  long long ldo, int batch, int Fq, int Fk, int L, int heads, int head_dim, cudaStream_t s) {
  if (option(OPT_TATTN_MMA) == 0) return 1;
  if (Fq < 1 || Fq > 32 || Fk < 1 || Fk > 32) return 1;
  if (((reinterpret_cast<uintptr_t>(Q) | reinterpret_cast<uintptr_t>(K) | reinterpret_cast<uintptr_t>(V) |
        reinterpret_cast<uintptr_t>(O)) & 15) != 0)
    return 1;
#define HB_TD(T_)                                                                                                    \
  switch (head_dim) {                                                                                                \
    case 40: return dispatch_tattn_mma<T_, 40>(Q, ldq, K, V, ldkv, O, ldo, batch, Fq, Fk, L, heads, s);              \
    case 80: return dispatch_tattn_mma<T_, 80>(Q, ldq, K, V, ldkv, O, ldo, batch, Fq, Fk, L, heads, s);              \
    case 160: return dispatch_tattn_mma<T_, 160>(Q, ldq, K, V, ldkv, O, ldo, batch, Fq, Fk, L, heads, s);            \
    default: return 1;                                                                                               \
  }
  if (dtype == HB_F16) { HB_TD(__half) }
  if (dtype == HB_BF16) { HB_TD(__nv_bfloat16) }
#undef HB_TD
  return 1;
}

}  // namespace hb
