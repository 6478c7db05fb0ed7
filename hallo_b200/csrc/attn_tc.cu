// hallo_b200_attention and the tensor-core path of hallo_b200_cross_attention: fused softmax(Q K^T / sqrt(d)) V on
// sm_90a warpgroup MMAs (wgmma), flash-attention style.
//
// One CTA = one (frame, query column group, 128-query tile).  Keys come in up to two SEGMENTS that are
// concatenated in-kernel: segment 0 = the frame's own tokens, segment 1 (optional, per frame) =
// the ReferenceNet tokens of CFG half ref_index[frame] -- this is the `torch.cat([norm_hidden_states,
// bank])` of mutual_self_attention.py:253-263, without ever materialising the 2L-key tensor, and
// without recomputing the uncond half (mutual_self_attention.py:264-284): uncond frames simply have
// ref_index = -1.
//
//   warps 0-3, 4-7  two consumer warpgroups, 64 query rows each: S = Q K_j^T (wgmma, Q and K from shared memory,
//                   fp32 in registers), online max / sum in fp32 registers, O += P_j V_j (wgmma, A = P_j packed
//                   to fp16/bf16 in registers, V MN-major in shared memory).
//   warp 8          TMA producer: Q tile once, then K / V tiles of BN keys through a STAGES-deep ring.
//
// Cross-attention (hallo_b200_cross_attention, <= 32 image / audio keys per frame) runs the same kernel with one
// key tile: the key frame is frame / kv_frame_div, and each mask region has its own query and key column groups.
//
// Head dim 512 (the VAE) has its own kernel, attn_wide_kernel, at the end of this file.
//
// Head dims 40 / 80 / 160 are not multiples of the 64-element swizzle span: TMA boxes of 64 columns
// over a (d, head, token, frame) tensor map zero-fill the columns >= d, so Q/K/V stay unpadded in HBM.
#include "host_common.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace hb {

constexpr int kAttnThreads = 288;     // two consumer warpgroups + the TMA warp
constexpr int kAttnConsumers = 256;

struct AttnDev {
  int L;                 // queries per frame
  int Lk;                // keys per segment
  int frames;
  int heads;             // query column groups per region
  int kv_region_groups;  // K / V column group of (region r, head h) = r * kv_region_groups + h
  int kv_frame_div;      // key frame = frame / kv_frame_div
  const int* ref_index;  // [frames] or nullptr
  void* O;
  long long ldo;
  int o_region_stride;
  float scale_log2;      // d^-0.5 * log2(e)
};

template <int D, int BN, int STAGES>
struct AttnCfg {
  static constexpr int kChunks = (D + 63) / 64;          // 64-column swizzle chunks per row
  static constexpr int kKSteps = (D + 15) / 16;          // MMA K steps for Q K^T
  static constexpr int kDv = ((D + 15) / 16) * 16;       // N of the P V MMA (48 / 80 / 160)
  static constexpr int kQBytes = kChunks * 128 * 128;
  static constexpr int kKVBytes = kChunks * BN * 128;    // one K (or V) tile
  static constexpr int kOffK = kQBytes;
  static constexpr int kOffV = kOffK + STAGES * kKVBytes;
  static constexpr int kOffBar = kOffV + STAGES * kKVBytes;
  static constexpr int kTotal = kOffBar + 256 + 1024;
  static_assert((BN * 128) % 1024 == 0, "K / V chunks must keep the 1024 B swizzle alignment");
};

template <typename T, int D, int BN, int STAGES, int MINB>
__global__ void __launch_bounds__(kAttnThreads, MINB)
attn_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK0,
               const __grid_constant__ CUtensorMap tmV0, const __grid_constant__ CUtensorMap tmK1,
               const __grid_constant__ CUtensorMap tmV1, const AttnDev p) {
  using CF = AttnCfg<D, BN, STAGES>;
  constexpr int RS = BN / 2;         // S registers per thread
  constexpr int RO = CF::kDv / 2;    // O registers per thread
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + CF::kOffBar);
  uint64_t* q_full = bars;                 // 1
  uint64_t* k_full = bars + 1;             // STAGES
  uint64_t* v_full = k_full + STAGES;      // STAGES
  uint64_t* kv_empty = v_full + STAGES;    // STAGES

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int qt = blockIdx.x;
  const int qg = blockIdx.y;                           // query column group = region * heads + head
  const int region = qg / p.heads;
  const int head = qg - region * p.heads;
  const int kg = region * p.kv_region_groups + head;
  const int frame = p.frames - 1 - (int)blockIdx.z;   // cond (two-segment) frames are scheduled first
  const int kvf = frame / p.kv_frame_div;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&k_full[s], 1);
      mbar_init(&v_full[s], 1);
      mbar_init(&kv_empty[s], kAttnConsumers);
    }
    fence_barrier_init();
  }
  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK0);
    tma_prefetch_desc(&tmV0);
  }
  __syncthreads();
  pdl_wait();
  pdl_launch();
  const int ref = (p.ref_index != nullptr) ? p.ref_index[frame] : -1;
  const int tiles_per_seg = (p.Lk + BN - 1) / BN;
  const int ntiles = tiles_per_seg * (ref >= 0 ? 2 : 1);

  if (warp == 8) {
    // ============================ TMA producer ============================
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, CF::kQBytes);
#pragma unroll
      for (int c = 0; c < CF::kChunks; ++c)
        tma_load_4d(smem + c * (128 * 128), &tmQ, q_full, c * 64, qg, qt * 128, frame);
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < ntiles; ++j) {
        const int seg = j / tiles_per_seg;
        const int kt = j - seg * tiles_per_seg;
        const CUtensorMap* mk = seg == 0 ? &tmK0 : &tmK1;
        const CUtensorMap* mv = seg == 0 ? &tmV0 : &tmV1;
        const int fr = seg == 0 ? kvf : ref;
        mbar_wait(&kv_empty[stage], phase ^ 1, 0x41);
        mbar_arrive_expect_tx(&k_full[stage], CF::kKVBytes);
#pragma unroll
        for (int c = 0; c < CF::kChunks; ++c)
          tma_load_4d(smem + CF::kOffK + stage * CF::kKVBytes + c * (BN * 128), mk, &k_full[stage],
                      c * 64, kg, kt * BN, fr);
        mbar_arrive_expect_tx(&v_full[stage], CF::kKVBytes);
#pragma unroll
        for (int c = 0; c < CF::kChunks; ++c)
          tma_load_4d(smem + CF::kOffV + stage * CF::kKVBytes + c * (BN * 128), mv, &v_full[stage],
                      c * 64, kg, kt * BN, fr);
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
    return;
  }

  // ============================ consumer warpgroups ============================
  const int wg = threadIdx.x >> 7;
  const int r0 = (warp & 3) * 16 + (lane >> 2);      // rows r0, r0 + 8 of this warpgroup's 64
  const int cq = 2 * (lane & 3);
  const uint32_t sQ = smem_u32(smem) + wg * (64 * 128);
  const uint32_t sK = smem_u32(smem + CF::kOffK);
  const uint32_t sV = smem_u32(smem + CF::kOffV);
  float o[RO];
#pragma unroll
  for (int i = 0; i < RO; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_sum[2] = {0.f, 0.f};                       // partial sums over this thread's columns
  mbar_wait(q_full, 0, 0x51);

  int stage = 0;
  uint32_t phase = 0;
  for (int j = 0; j < ntiles; ++j) {
    const int key0 = (j % tiles_per_seg) * BN;
    float s[RS];
    mbar_wait(&k_full[stage], phase, 0x52);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < CF::kKSteps; ++k) {
      const uint32_t off_q = (k >> 2) * (128 * 128) + (k & 3) * 32;
      const uint32_t off_k = stage * CF::kKVBytes + (k >> 2) * (BN * 128) + (k & 3) * 32;
      Wgmma<BN, T>::ss(s, make_desc_sw128(sQ + off_q, 16, 1024), make_desc_sw128(sK + off_k, 16, 1024), k != 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_pin(s);

    if (key0 + BN > p.Lk) {
#pragma unroll
      for (int i = 0; i < BN / 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (key0 + 8 * i + cq + e >= p.Lk) {
            s[4 * i + e] = -INFINITY;
            s[4 * i + 2 + e] = -INFINITY;
          }
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      mx[0] = max3(mx[0], s[4 * i], s[4 * i + 1]);
      mx[1] = max3(mx[1], s[4 * i + 2], s[4 * i + 3]);
    }
    float f[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));   // the four lanes of a quad share a row
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      const float m_new = fmaxf(m_run[h], mx[h] * p.scale_log2);     // every key tile has at least one valid key
      f[h] = fast_exp2(m_run[h] - m_new);
      m_run[h] = m_new;
      l_sum[h] *= f[h];
    }
#pragma unroll
    for (int i = 0; i < RO / 4; ++i) {
      o[4 * i] *= f[0];
      o[4 * i + 1] *= f[0];
      o[4 * i + 2] *= f[1];
      o[4 * i + 3] *= f[1];
    }
    // P = exp2(S * scale - m), packed as the A fragments of the P V MMA (16 keys per K step)
    uint32_t pa[BN / 16][4];
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      const float e0 = fast_exp2(fmaf(s[4 * i], p.scale_log2, -m_run[0]));
      const float e1 = fast_exp2(fmaf(s[4 * i + 1], p.scale_log2, -m_run[0]));
      const float e2 = fast_exp2(fmaf(s[4 * i + 2], p.scale_log2, -m_run[1]));
      const float e3 = fast_exp2(fmaf(s[4 * i + 3], p.scale_log2, -m_run[1]));
      l_sum[0] += e0 + e1;
      l_sum[1] += e2 + e3;
      pa[i >> 1][(i & 1) * 2] = Cvt<T>::pack2(e0, e1);
      pa[i >> 1][(i & 1) * 2 + 1] = Cvt<T>::pack2(e2, e3);
    }
    mbar_wait(&v_full[stage], phase, 0x53);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BN / 16; ++k)
      Wgmma<CF::kDv, T>::rs(o, pa[k], make_desc_sw128(sV + stage * CF::kKVBytes + k * 2048, BN * 128, 1024), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_pin(o);
    mbar_arrive(&kv_empty[stage]);
    if (++stage == STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }

  // ---- epilogue: O / l -> global ----
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_sum[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.0f / l;
    const int qrow = qt * 128 + wg * 64 + r0 + 8 * h;
    if (qrow >= p.L) continue;
    T* out = reinterpret_cast<T*>(p.O) + ((long long)frame * p.L + qrow) * p.ldo + region * p.o_region_stride + head * D;
#pragma unroll
    for (int i = 0; i < RO / 4; ++i) {
      const int col = 8 * i + cq;
      if (col < D) *reinterpret_cast<uint32_t*>(out + col) = Cvt<T>::pack2(o[4 * i + 2 * h] * inv, o[4 * i + 2 * h + 1] * inv);
    }
  }
}

// (d, group, token, frame) tensor map over a [frames*rows, ld] token matrix whose columns are groups of D
static int make_qkv_map(CUtensorMap* m, int dtype, const void* base, int D, int groups, int rows, int frames,
                        long long ld, int box_rows) {
  uint64_t dims[4] = {(uint64_t)D, (uint64_t)groups, (uint64_t)rows, (uint64_t)frames};
  uint64_t str[3] = {(uint64_t)D * 2, (uint64_t)ld * 2, (uint64_t)ld * 2 * rows};
  uint32_t box[4] = {64, 1, (uint32_t)box_rows, 1};
  return make_tmap_16b(m, dtype, base, 4, dims, str, box);
}

template <typename T, int D, int BN, int STAGES, int MINB>
static int launch_attn_kernel(const CUtensorMap& tmQ, const CUtensorMap& tmK0, const CUtensorMap& tmV0,
                              const CUtensorMap& tmK1, const CUtensorMap& tmV1, const AttnDev& d, int query_groups,
                              cudaStream_t stream) {
  using CF = AttnCfg<D, BN, STAGES>;
  static_assert(CF::kTotal * MINB <= 232448, "attention smem budget");
  auto kern = attn_tc_kernel<T, D, BN, STAGES, MINB>;
  static bool attr_set = false;
  if (!attr_set) {
    HB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, CF::kTotal));
    attr_set = true;
  }
  dim3 grid((d.L + 127) / 128, query_groups, d.frames);
  HB_CUDA_CHECK(launch_kernel(kern, grid, kAttnThreads, CF::kTotal, stream, tmQ, tmK0, tmV0, tmK1, tmV1, d));
  HB_LAUNCH_CHECK();
  return HB_OK;
}

// self-attention over the frame's tokens (+ the reference tokens of ref_index[frame]): 64-key steps
template <typename T, int D, int STAGES, int MINB>
static int launch_attn(const hb_attention_params* q, cudaStream_t stream) {
  constexpr int BN = 64;
  CUtensorMap tmQ, tmK0, tmV0, tmK1, tmV1;
  int rc;
  if ((rc = make_qkv_map(&tmQ, q->dtype, q->Q, D, q->heads, q->L, q->frames, q->ldq, 128))) return rc;
  if ((rc = make_qkv_map(&tmK0, q->dtype, q->K, D, q->heads, q->L, q->frames, q->ldk, BN))) return rc;
  if ((rc = make_qkv_map(&tmV0, q->dtype, q->V, D, q->heads, q->L, q->frames, q->ldv, BN))) return rc;
  if (q->ref_index != nullptr) {     // Kref / Vref / ref_frames checked by hallo_b200_attention
    if ((rc = make_qkv_map(&tmK1, q->dtype, q->Kref, D, q->heads, q->L, q->ref_frames, q->ldkref, BN))) return rc;
    if ((rc = make_qkv_map(&tmV1, q->dtype, q->Vref, D, q->heads, q->L, q->ref_frames, q->ldvref, BN))) return rc;
  } else {
    tmK1 = tmK0;
    tmV1 = tmV0;
  }
  AttnDev d{};
  d.L = q->L;
  d.Lk = q->L;
  d.frames = q->frames;
  d.heads = q->heads;
  d.kv_region_groups = 0;
  d.kv_frame_div = 1;
  d.ref_index = q->ref_index;
  d.O = q->O;
  d.ldo = q->ldo;
  d.o_region_stride = 0;
  d.scale_log2 = (float)(1.4426950408889634 / sqrt((double)D));
  return launch_attn_kernel<T, D, BN, STAGES, MINB>(tmQ, tmK0, tmV0, tmK1, tmV1, d, q->heads, stream);
}

// cross-attention against n_keys <= NK keys of frame / kv_frame_div; Q columns: region r, head h at r*heads*D + h*D;
// K / V: [K_r | V_r] pairs of heads*D columns
template <typename T, int D, int NK>
static int launch_xattn(int dtype, const void* Q, long long ldq, const void* K, const void* V, long long ldkv,
                        void* O, long long ldo, int o_region_stride, int frames, int L, int heads, int n_keys,
                        int kv_frame_div, int regions, cudaStream_t stream) {
  CUtensorMap tmQ, tmK, tmV;
  int rc;
  const int kv_frames = (frames + kv_frame_div - 1) / kv_frame_div;
  if ((rc = make_qkv_map(&tmQ, dtype, Q, D, regions * heads, L, frames, ldq, 128))) return rc;
  if ((rc = make_qkv_map(&tmK, dtype, K, D, 2 * regions * heads, n_keys, kv_frames, ldkv, NK))) return rc;
  if ((rc = make_qkv_map(&tmV, dtype, V, D, 2 * regions * heads, n_keys, kv_frames, ldkv, NK))) return rc;
  AttnDev d{};
  d.L = L;
  d.Lk = n_keys;
  d.frames = frames;
  d.heads = heads;
  d.kv_region_groups = 2 * heads;
  d.kv_frame_div = kv_frame_div;
  d.ref_index = nullptr;
  d.O = O;
  d.ldo = ldo;
  d.o_region_stride = o_region_stride;
  d.scale_log2 = (float)(1.4426950408889634 / sqrt((double)D));
  return launch_attn_kernel<T, D, NK, 1, (D > 80 ? 1 : 2)>(tmQ, tmK, tmV, tmK, tmV, d, heads * regions, stream);
}

template <typename T>
static int dispatch_xattn(int dtype, const void* Q, long long ldq, const void* K, const void* V, long long ldkv, void* O,
                          long long ldo, int o_region_stride, int frames, int L, int heads, int head_dim, int n_keys,
                          int kv_frame_div, int regions, cudaStream_t s) {
#define HB_X(D_, NK_) \
  return launch_xattn<T, D_, NK_>(dtype, Q, ldq, K, V, ldkv, O, ldo, o_region_stride, frames, L, heads, n_keys, kv_frame_div, regions, s)
  if (n_keys > 16) {
    if (head_dim == 40) HB_X(40, 32);
    if (head_dim == 80) HB_X(80, 32);
    if (head_dim == 160) HB_X(160, 32);
  } else {
    if (head_dim == 40) HB_X(40, 16);
    if (head_dim == 80) HB_X(80, 16);
    if (head_dim == 160) HB_X(160, 16);
  }
#undef HB_X
  return fail(HB_ERR_BAD_SHAPE, "cross_attention (tensor cores): head_dim %d", head_dim);
}

// returns HB_OK if handled, 1 if the shape is left to the CUDA-core kernel
int xattn_tc_try(int dtype, const void* Q, long long ldq, int q_region_stride, const void* K, const void* V,
                 long long ldkv, int kv_region_stride, void* O, long long ldo, int o_region_stride, int frames, int L,
                 int heads, int head_dim, int n_keys, int kv_frame_div, int regions, cudaStream_t s) {
  const bool off = option(OPT_XATTN_TC) == 0;
  const int C = heads * head_dim;
  // layout contract of this path: Q regions C apart, [K_r | V_r] pairs 2C apart with V = K + C columns, n_keys <= 32
  if (off || (head_dim != 40 && head_dim != 80 && head_dim != 160) || n_keys > 32 || n_keys < 1 || L < 128) return 1;
  if (regions > 1 && (q_region_stride != C || kv_region_stride != 2 * C)) return 1;
  if (reinterpret_cast<const char*>(V) - reinterpret_cast<const char*>(K) != (long long)C * 2) return 1;
  if (dtype == HB_F16)
    return dispatch_xattn<__half>(dtype, Q, ldq, K, V, ldkv, O, ldo, o_region_stride, frames, L, heads, head_dim, n_keys,
                                  kv_frame_div, regions, s);
  if (dtype == HB_BF16)
    return dispatch_xattn<__nv_bfloat16>(dtype, Q, ldq, K, V, ldkv, O, ldo, o_region_stride, frames, L, heads, head_dim,
                                         n_keys, kv_frame_div, regions, s);
  return 1;
}

// ------------------------------------------------------------------------------------------------------------------
// Head dim 512, one head: the VAE mid-block attention (diffusers Attention(heads=1, bias=True) over the (h/8)(w/8)
// tokens of a frame).  A 64 x 512 fp32 O accumulator does not fit in a warpgroup's registers, and a 128 x 512 Q tile
// leaves too little shared memory for a whole-row K ring.  So the V / O columns are split over kWideSplit CTAs of
// kWideDv columns each (blockIdx.y); every CTA computes the full 512-wide Q K^T of its 128 queries (the recomputation
// is (kWideSplit - 1) / kWideSplit of the Q K^T work, ~2 % of a VAE decode) and keeps scores and softmax in fp32.
//
//   shared memory: Q tile 128 x 512 (8 swizzle chunks of 64 columns, loaded once)         128 KB
//                  K ring of kWideKStages chunks, each 64 keys x 64 columns                  64 KB
//                  V ring of kWideVStages tiles, each 64 keys x kWideDv columns              32 KB
//   warps 0-7: two consumer warpgroups (64 query rows each); S = sum over the 8 chunks of Q_c K_c^T, each chunk slot
//              handed back to the producer as soon as its MMAs have retired; then the same online softmax and
//              O += P V as attn_tc_kernel.
//   warp 8:    TMA producer.
constexpr int kWideD = 512;
constexpr int kWideDv = 128;
constexpr int kWideSplit = kWideD / kWideDv;
constexpr int kWideBN = 64;
constexpr int kWideKStages = 8;
constexpr int kWideVStages = 2;
constexpr int kWideQBytes = (kWideD / 64) * 128 * 128;
constexpr int kWideKBytes = kWideBN * 128;                     // one 64-column chunk of a key tile
constexpr int kWideVBytes = (kWideDv / 64) * kWideBN * 128;    // kWideDv columns of a key tile
constexpr int kWideOffK = kWideQBytes;
constexpr int kWideOffV = kWideOffK + kWideKStages * kWideKBytes;
constexpr int kWideOffBar = kWideOffV + kWideVStages * kWideVBytes;
constexpr int kWideSmem = kWideOffBar + 256 + 1024;
static_assert(kWideSmem <= 232448, "wide attention smem budget");

template <typename T>
__global__ void __launch_bounds__(kAttnThreads, 1)
attn_wide_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                 const __grid_constant__ CUtensorMap tmV, const AttnDev p) {
  constexpr int BN = kWideBN;
  constexpr int RS = BN / 2;
  constexpr int RO = kWideDv / 2;
  constexpr int kChunks = kWideD / 64;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kWideOffBar);
  uint64_t* q_full = bars;
  uint64_t* k_full = bars + 1;
  uint64_t* k_empty = k_full + kWideKStages;
  uint64_t* v_full = k_empty + kWideKStages;
  uint64_t* v_empty = v_full + kWideVStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int qt = blockIdx.x;
  const int vcol0 = blockIdx.y * kWideDv;
  const int frame = blockIdx.z;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < kWideKStages; ++s) {
      mbar_init(&k_full[s], 1);
      mbar_init(&k_empty[s], kAttnConsumers);
    }
    for (int s = 0; s < kWideVStages; ++s) {
      mbar_init(&v_full[s], 1);
      mbar_init(&v_empty[s], kAttnConsumers);
    }
    fence_barrier_init();
  }
  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
  }
  __syncthreads();
  pdl_wait();
  pdl_launch();
  const int ntiles = (p.Lk + BN - 1) / BN;

  if (warp == 8) {
    // ============================ TMA producer ============================
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, kWideQBytes);
#pragma unroll
      for (int c = 0; c < kChunks; ++c) tma_load_4d(smem + c * (128 * 128), &tmQ, q_full, c * 64, 0, qt * 128, frame);
      int ks = 0, vs = 0;
      uint32_t kph = 0, vph = 0;
      for (int j = 0; j < ntiles; ++j) {
        for (int c = 0; c < kChunks; ++c) {
          mbar_wait(&k_empty[ks], kph ^ 1, 0x61);
          mbar_arrive_expect_tx(&k_full[ks], kWideKBytes);
          tma_load_4d(smem + kWideOffK + ks * kWideKBytes, &tmK, &k_full[ks], c * 64, 0, j * BN, frame);
          if (++ks == kWideKStages) {
            ks = 0;
            kph ^= 1;
          }
        }
        mbar_wait(&v_empty[vs], vph ^ 1, 0x62);
        mbar_arrive_expect_tx(&v_full[vs], kWideVBytes);
#pragma unroll
        for (int c = 0; c < kWideDv / 64; ++c)
          tma_load_4d(smem + kWideOffV + vs * kWideVBytes + c * (BN * 128), &tmV, &v_full[vs], vcol0 + c * 64, 0,
                      j * BN, frame);
        if (++vs == kWideVStages) {
          vs = 0;
          vph ^= 1;
        }
      }
    }
    return;
  }

  // ============================ consumer warpgroups ============================
  const int wg = threadIdx.x >> 7;
  const int r0 = (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const uint32_t sQ = smem_u32(smem) + wg * (64 * 128);
  const uint32_t sK = smem_u32(smem + kWideOffK);
  const uint32_t sV = smem_u32(smem + kWideOffV);
  float o[RO];
#pragma unroll
  for (int i = 0; i < RO; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};
  float l_sum[2] = {0.f, 0.f};
  mbar_wait(q_full, 0, 0x71);

  int ks = 0, vs = 0;
  uint32_t kph = 0, vph = 0;
  for (int j = 0; j < ntiles; ++j) {
    const int key0 = j * BN;
    float s[RS];
    int prev = -1;
#pragma unroll 1
    for (int c = 0; c < kChunks; ++c) {
      mbar_wait(&k_full[ks], kph, 0x72);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        Wgmma<BN, T>::ss(s, make_desc_sw128(sQ + c * (128 * 128) + k * 32, 16, 1024),
                         make_desc_sw128(sK + ks * kWideKBytes + k * 32, 16, 1024), (c | k) != 0);
      wgmma_commit();
      wgmma_wait<1>();                       // the MMAs of chunk c - 1 have retired: its slot goes back
      if (prev >= 0) mbar_arrive(&k_empty[prev]);
      prev = ks;
      if (++ks == kWideKStages) {
        ks = 0;
        kph ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_pin(s);
    mbar_arrive(&k_empty[prev]);

    if (key0 + BN > p.Lk) {
#pragma unroll
      for (int i = 0; i < BN / 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (key0 + 8 * i + cq + e >= p.Lk) {
            s[4 * i + e] = -INFINITY;
            s[4 * i + 2 + e] = -INFINITY;
          }
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      mx[0] = max3(mx[0], s[4 * i], s[4 * i + 1]);
      mx[1] = max3(mx[1], s[4 * i + 2], s[4 * i + 3]);
    }
    float f[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      const float m_new = fmaxf(m_run[h], mx[h] * p.scale_log2);     // every key tile has at least one valid key
      f[h] = fast_exp2(m_run[h] - m_new);
      m_run[h] = m_new;
      l_sum[h] *= f[h];
    }
#pragma unroll
    for (int i = 0; i < RO / 4; ++i) {
      o[4 * i] *= f[0];
      o[4 * i + 1] *= f[0];
      o[4 * i + 2] *= f[1];
      o[4 * i + 3] *= f[1];
    }
    uint32_t pa[BN / 16][4];
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      const float e0 = fast_exp2(fmaf(s[4 * i], p.scale_log2, -m_run[0]));
      const float e1 = fast_exp2(fmaf(s[4 * i + 1], p.scale_log2, -m_run[0]));
      const float e2 = fast_exp2(fmaf(s[4 * i + 2], p.scale_log2, -m_run[1]));
      const float e3 = fast_exp2(fmaf(s[4 * i + 3], p.scale_log2, -m_run[1]));
      l_sum[0] += e0 + e1;
      l_sum[1] += e2 + e3;
      pa[i >> 1][(i & 1) * 2] = Cvt<T>::pack2(e0, e1);
      pa[i >> 1][(i & 1) * 2 + 1] = Cvt<T>::pack2(e2, e3);
    }
    mbar_wait(&v_full[vs], vph, 0x73);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BN / 16; ++k)
      Wgmma<kWideDv, T>::rs(o, pa[k], make_desc_sw128(sV + vs * kWideVBytes + k * 2048, BN * 128, 1024), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_pin(o);
    mbar_arrive(&v_empty[vs]);
    if (++vs == kWideVStages) {
      vs = 0;
      vph ^= 1;
    }
  }

#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_sum[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.0f / l;
    const int qrow = qt * 128 + wg * 64 + r0 + 8 * h;
    if (qrow >= p.L) continue;
    T* out = reinterpret_cast<T*>(p.O) + ((long long)frame * p.L + qrow) * p.ldo + vcol0;
#pragma unroll
    for (int i = 0; i < RO / 4; ++i) {
      const int col = 8 * i + cq;
      *reinterpret_cast<uint32_t*>(out + col) = Cvt<T>::pack2(o[4 * i + 2 * h] * inv, o[4 * i + 2 * h + 1] * inv);
    }
  }
}

// hallo_b200_attention with head_dim 512 (heads == 1, no reference keys)
template <typename T>
static int launch_attn_wide(const hb_attention_params* q, cudaStream_t stream) {
  if (q->heads != 1 || q->ref_index != nullptr)
    return fail(HB_ERR_BAD_SHAPE, "attention: head_dim 512 takes one head and no reference keys");
  CUtensorMap tmQ, tmK, tmV;
  int rc;
  if ((rc = make_qkv_map(&tmQ, q->dtype, q->Q, kWideD, 1, q->L, q->frames, q->ldq, 128))) return rc;
  if ((rc = make_qkv_map(&tmK, q->dtype, q->K, kWideD, 1, q->L, q->frames, q->ldk, kWideBN))) return rc;
  if ((rc = make_qkv_map(&tmV, q->dtype, q->V, kWideD, 1, q->L, q->frames, q->ldv, kWideBN))) return rc;
  AttnDev d{};
  d.L = q->L;
  d.Lk = q->L;
  d.frames = q->frames;
  d.heads = 1;
  d.kv_frame_div = 1;
  d.O = q->O;
  d.ldo = q->ldo;
  d.scale_log2 = (float)(1.4426950408889634 / sqrt((double)kWideD));
  auto kern = attn_wide_kernel<T>;
  static bool attr_set = false;
  if (!attr_set) {
    HB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kWideSmem));
    attr_set = true;
  }
  dim3 grid((d.L + 127) / 128, kWideSplit, d.frames);
  HB_CUDA_CHECK(launch_kernel(kern, grid, kAttnThreads, kWideSmem, stream, tmQ, tmK, tmV, d));
  HB_LAUNCH_CHECK();
  return HB_OK;
}

}  // namespace hb
