// hallo_b200_gemm: persistent warp-specialised wgmma GEMM / implicit-GEMM conv3x3 (sm_90a).
//
//   warps 0-3, 4-7 : two consumer warpgroups.  Warpgroup g owns rows [64g, 64g + 64) of the 128 x BN tile: one
//                    wgmma m64nBNk16 per 16-wide K step (fp32 accumulators in registers), then the epilogue.
//   warp 8         : TMA producer (A tile 128x64, W tile BNx64 per stage, 128B-swizzled; the residual tile), one
//                    elected lane.
//
// Each warpgroup keeps one wgmma group in flight: the stage of K step i is handed back to the producer once the
// MMAs of step i + 1 have been issued and those of step i have completed.
//
// Staged epilogue (bias / group bias / row scale / GEGLU / residual): every warpgroup owns a 64 x BN staging tile in
// shared memory, stored as CW-column chunks (CW = 32 or 16, swizzled over CW * 2 bytes, so the accumulator-layout
// accesses are free of bank conflicts).  The producer loads the tile's residual into it with TMA during the K loop;
// the warpgroup adds the epilogue terms in place and one thread stores the chunks with TMA, whose clipping at the
// tensor bounds replaces the M-tail and overhanging-conv-box masks.  The warpgroup then goes straight on to the next
// tile: its store drains while that tile's MMAs run, and the staging tile is handed back to the producer (barrier
// stg_free) after the first k-block of the next tile, once the store has read it.
// Row scatter to peer buffers, the EPI_FULL options (activation, LayerNorm fold, row statistics) and output or
// residual pointers that are not 16-byte aligned keep the register epilogue, which stores straight to global memory.
//
// Split-K (p.splits = S > 1, chosen by the host when the tiles cover less than half of the SMs): the grid holds one
// CTA per (tile, split); split s runs k-blocks [s*kper, (s+1)*kper).  Splits 1.. store their raw fp32 accumulators to
// the workspace ([tile][split-1][register][thread]: coalesced) and bump one counter per (tile, warpgroup); split 0
// waits for S-1 arrivals on the counter of each of its warpgroups, adds the partials in split order and runs the
// usual epilogue.  All CTAs of such a grid are co-resident (<= 1 per SM), so the wait cannot deadlock; the
// summation order is fixed, so results do not depend on timing.
// Tiles are walked n-fastest so the CTAs running concurrently share the same A rows in L2.
//
// Implicit conv: the A operand of tap (kh,kw) is the NHWC box shifted by (kh-1, kw-1); TMA's
// out-of-bounds zero fill supplies the padding, so no im2col buffer exists anywhere.
#include <cstdlib>

#include "host_common.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace hb {

constexpr int kBM = 128;
constexpr int kBK = 64;
constexpr int kBN = 160;              // divides every channel count of the UNet (320, 640, 1280, ...)
constexpr int kBN2 = 128;             // power-of-two widths (the VAE's 128 / 256 / 512 / 1536): no wasted columns
constexpr int kGemmStages = 5;        // BN = 160: 5 x 36 KB of operand stages + 40 KB of staging tiles
constexpr int kGemmStages2 = 6;       // BN = 128: 6 x 32 KB + 32 KB
constexpr int kGemmThreads = 288;     // two consumer warpgroups + the TMA warp
constexpr int kGemmConsumers = 256;

struct GemmDev {
  int M, N, K, K1;
  int tiles_m, tiles_n;
  void* C;
  long long ldc;
  const void* bias;
  const void* group_bias;
  long long ld_group_bias;
  int rows_per_group;
  const void* row_scale;
  const void* residual;
  long long ldr;
  float alpha;
  int flags;
  const float* ln_stats;
  const float* ln_colsum;
  float ln_eps;
  float* stats_out;
  hb_row_scatter sc;   // sc.seg > 0: output rows go to peer buffers
  int splits;          // split-K factor S (1 = off); S > 1 => gridDim.x == tiles * S
  float* ws;           // S > 1: fp32 partial tiles
  int* cnt;            // S > 1: arrival counters, [tile][warpgroup], zero between launches
  // conv geometry
  int cin, img_n, img_h, img_w, box_w, box_h, box_n, tiles_w, tiles_h;
  int stride2;         // 0: stride 1, pad 1; 1: stride 2, pad 1 (conv3x3 == 2); 2: stride 2, pad (0, 1) (conv3x3 == 3)
  int staged;          // epilogue through the staging tiles and TMA stores (tmC; tmR when residual != nullptr)
  int wg_dw, wg_dh, wg_dn;   // conv: origin of warpgroup 1's half box within the tile's box
};

// split-K: wait until `need` partial tiles have been published on *cnt, then re-arm the counter for the next launch
__device__ __forceinline__ void splitk_wait(int* cnt, int need) {
  const long long t0 = clock64();
  for (;;) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];\n" : "=r"(v) : "l"(cnt) : "memory");
    if (v >= need) break;
    if (clock64() - t0 > 4000000000LL) {
      atomicExch(&g_hb_error, 0x36u | (blockIdx.x << 8));
      __trap();
    }
    __nanosleep(64);
  }
  *cnt = 0;
}

template <int BN, int STAGES>
struct GemmSmem {
  static constexpr int kABytes = kBM * kBK * 2;
  static constexpr int kBBytes = BN * kBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStgOffset = STAGES * kStageBytes;
  static constexpr int kStgBytes = 64 * BN * 2;            // one warpgroup's staging tile
  static constexpr int kBarOffset = kStgOffset + 2 * kStgBytes;
  static constexpr int kTotal = kBarOffset + 256 + 1024;  // + barriers + alignment slack
  static_assert(kStageBytes % 1024 == 0 && kStgBytes % 1024 == 0, "stage alignment");
  static_assert(2 * STAGES * 8 + 4 * 8 <= 256, "barrier space");
};

// Staging-tile geometry of an epilogue that writes NOUT columns per tile: CW-column chunks of 64 rows, swizzled over
// the chunk's row width (Swizzle<log2(CW * 2 / 16), 4, 3>, what the tensor map's CU_TENSOR_MAP_SWIZZLE_{64,32}B does).
template <int NOUT>
struct Staging {
  static constexpr int kCW = NOUT % 32 == 0 ? 32 : 16;
  static constexpr int kChunks = NOUT / kCW;
  static constexpr int kChunkBytes = 64 * kCW * 2;
  static constexpr int kSwizzle = kCW * 2;
  static_assert(NOUT % 16 == 0, "staging width");
  // byte offset of element (r, c) of the 64 x NOUT tile
  __device__ static __forceinline__ uint32_t offset(int r, int c) {
    const uint32_t o = (uint32_t)((c / kCW) * kChunkBytes + r * (kCW * 2) + (c % kCW) * 2);
    return o ^ (((o >> 7) & (kSwizzle / 16 - 1)) << 4);
  }
};

// EPI fixes the epilogue at compile time: EPI_PLAIN = bias / group bias / row scale / residual, EPI_GEGLU = the same
// with the (value, gate) GEGLU pairing, EPI_FULL = every option decided at run time (activation, folded LayerNorm,
// row statistics).  The common cases then carry no dead branches in their epilogue.
enum { EPI_PLAIN = 0, EPI_GEGLU = 1, EPI_FULL = 2 };

template <typename T, int BN, int STAGES, bool CONV, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
               const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmC,
               const __grid_constant__ CUtensorMap tmR, const GemmDev p) {
  using SM = GemmSmem<BN, STAGES>;
  static_assert(BN % 16 == 0 && BN <= 256, "BN");
  constexpr int R = BN / 2;             // accumulator registers per consumer thread
  constexpr int NOUT = EPI == EPI_GEGLU ? BN / 2 : BN;   // output columns per tile (staged epilogue)
  using STG = Staging<NOUT>;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + SM::kBarOffset);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* res_full = empty_bar + STAGES;   // [warpgroup]: residual tile landed in the staging tile
  uint64_t* stg_free = res_full + 2;         // [warpgroup]: the previous tile's store has read the staging tile

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const bool staged = EPI != EPI_FULL && p.staged != 0;
  const bool stage_resid = staged && p.residual != nullptr;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kGemmConsumers);
    }
    for (int g = 0; g < 2; ++g) {
      mbar_init(&res_full[g], 1);
      mbar_init(&stg_free[g], 1);
    }
    fence_barrier_init();
  }
  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (p.K1 < p.K) tma_prefetch_desc(&tmA2);
    if (staged) tma_prefetch_desc(&tmC);
    if (stage_resid) tma_prefetch_desc(&tmR);
  }
  __syncthreads();
  pdl_wait();        // everything above (barriers, tensor-map prefetch) may overlap the predecessor's tail
  pdl_launch();

  const int num_tiles = p.tiles_m * p.tiles_n;
  const int kblocks = p.K / kBK;
  const int cin_blocks = CONV ? p.cin / kBK : 1;
  // split-K: CTA c owns unit (tile c / S, split c % S) and nothing else -> every tile loop below runs once
  const int S = p.splits;
  const int split = S > 1 ? (int)blockIdx.x % S : 0;
  const int first = S > 1 ? (int)blockIdx.x / S : (int)blockIdx.x;
  const int stride = S > 1 ? num_tiles : (int)gridDim.x;
  const int kper = (kblocks + S - 1) / S;
  const int kb0 = split * kper;
  const int kb1 = (kb0 + kper < kblocks) ? kb0 + kper : kblocks;

  auto tile_origin = [&](int t, int& tm, int& tn, int& n0, int& h0, int& w0) {
    tm = t / p.tiles_n;
    tn = t % p.tiles_n;
    n0 = h0 = w0 = 0;
    if (CONV) {
      const int per_img = p.tiles_w * p.tiles_h;
      const int nb = tm / per_img;
      const int rem = tm - nb * per_img;
      const int hb_ = rem / p.tiles_w;
      n0 = nb * p.box_n;
      h0 = hb_ * p.box_h;
      w0 = (rem - hb_ * p.tiles_w) * p.box_w;
    }
  };
  // staging tile of warpgroup g <-> global memory (output through tmC, residual through tmR): chunk ch of the tile
  auto stg_copy = [&](bool store, int g, int ch, int tm, int tn, int n0, int h0, int w0) {
    uint8_t* st = smem + SM::kStgOffset + g * SM::kStgBytes + ch * STG::kChunkBytes;
    const int c = tn * NOUT + ch * STG::kCW;
    if (CONV) {
      const int cw = w0 + g * p.wg_dw, chh = h0 + g * p.wg_dh, cn = n0 + g * p.wg_dn;
      if (store) tma_store_4d(&tmC, st, c, cw, chh, cn);
      else tma_load_4d(st, &tmR, &res_full[g], c, cw, chh, cn);
    } else {
      if (store) tma_store_2d(&tmC, st, c, tm * kBM + 64 * g);
      else tma_load_2d(st, &tmR, &res_full[g], c, tm * kBM + 64 * g);
    }
  };
  // chunks of tile column tn that hold output columns (N = 8 heads: one of five)
  auto live_chunks = [&](int tn) {
    const int left = ((EPI == EPI_GEGLU) ? p.N / 2 : p.N) - tn * NOUT;
    const int n = (left + STG::kCW - 1) / STG::kCW;
    return n < STG::kChunks ? n : STG::kChunks;
  };

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      int it = 0;
      for (int t = first; t < num_tiles; t += stride, ++it) {
        int tm, tn, n0, h0, w0;
        tile_origin(t, tm, tn, n0, h0, w0);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1, 0x11);
          uint8_t* sa = smem + stage * SM::kStageBytes;
          uint8_t* sb = sa + SM::kABytes;
          mbar_arrive_expect_tx(&full_bar[stage], SM::kStageBytes);
          if (CONV) {
            const int tap = kb / cin_blocks;
            const int cb = kb - tap * cin_blocks;
            const int kh = tap / 3, kw = tap - kh * 3;
            if (p.stride2 == 1) {
              // input is stored as 4 phase planes [(p*2+q)*img_n + n][h/2][w/2][C] (x[2i+p][2j+q]);
              // output o reads input rows 2o-1 .. 2o+1: tap kh reads phase (kh==1 ? 0 : 1) at row offset (kh==0 ? -1 : 0)
              const int ph = (kh == 1) ? 0 : 1, pw = (kw == 1) ? 0 : 1;
              tma_load_4d(sa, &tmA, &full_bar[stage], cb * kBK, w0 - (kw == 0), h0 - (kh == 0),
                          (ph * 2 + pw) * p.img_n + n0);
            } else if (p.stride2 == 2) {
              // zero pad (0, 1) (diffusers Downsample2D(padding=0)): output o reads input rows 2o .. 2o+2, so tap kh
              // reads phase (kh==1 ? 1 : 0) at row offset (kh==2 ? 1 : 0); the last row / column of the padded input
              // lies past the plane and comes from the TMA out-of-bounds zero fill
              const int ph = (kh == 1) ? 1 : 0, pw = (kw == 1) ? 1 : 0;
              tma_load_4d(sa, &tmA, &full_bar[stage], cb * kBK, w0 + (kw == 2), h0 + (kh == 2),
                          (ph * 2 + pw) * p.img_n + n0);
            } else {
              tma_load_4d(sa, &tmA, &full_bar[stage], cb * kBK, w0 + kw - 1, h0 + kh - 1, n0);
            }
          } else {
            const int k = kb * kBK;
            const CUtensorMap* ma = (k < p.K1) ? &tmA : &tmA2;
            tma_load_2d(sa, ma, &full_bar[stage], (k < p.K1) ? k : k - p.K1, tm * kBM);
          }
          tma_load_2d(sb, &tmB, &full_bar[stage], kb * kBK, tn * BN);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
        // the tile's residual, once each warpgroup's store of the previous tile has left its staging tile
        if (stage_resid && split == 0) {
          for (int g = 0; g < 2; ++g) {
            if (it > 0) mbar_wait(&stg_free[g], (it - 1) & 1, 0x13);
            const int nch = live_chunks(tn);
            mbar_arrive_expect_tx(&res_full[g], nch * STG::kChunkBytes);
            for (int ch = 0; ch < nch; ++ch) stg_copy(false, g, ch, tm, tn, n0, h0, w0);
          }
        }
      }
    }
    return;
  }

  // ===================== consumer warpgroups: MMA + epilogue =====================
  const int wg = threadIdx.x >> 7;
  const int ct = threadIdx.x;                            // 0..255
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // tile rows r0 and r0 + 8 of this thread
  const int cq = 2 * (lane & 3);                         // column pair within each 8-column block
  const T* bias = reinterpret_cast<const T*>(p.bias);
  const T* gbias = reinterpret_cast<const T*>(p.group_bias);
  const T* rscale = reinterpret_cast<const T*>(p.row_scale);
  const T* resid = reinterpret_cast<const T*>(p.residual);
  T* C = reinterpret_cast<T*>(p.C);
  const bool geglu = (EPI == EPI_GEGLU) || (EPI == EPI_FULL && (p.flags & HB_EPI_GEGLU) != 0);
  const int n_out = geglu ? (p.N >> 1) : p.N;

  const bool stg_leader = (ct & 127) == 0;                // issues this warpgroup's TMA stores
  int stage = 0;
  uint32_t phase = 0;
  float acc[R];
  int it = 0;
  for (int t = first; t < num_tiles; t += stride, ++it) {
    int tm, tn, n0, h0, w0;
    tile_origin(t, tm, tn, n0, h0, w0);
    int prev = -1;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full_bar[stage], phase, 0x22);
      const uint32_t sa = smem_u32(smem + stage * SM::kStageBytes) + wg * (64 * 128);
      const uint32_t sb = smem_u32(smem + stage * SM::kStageBytes + SM::kABytes);
      const uint64_t adesc = make_desc_sw128(sa, 16, 1024);
      const uint64_t bdesc = make_desc_sw128(sb, 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBK / 16; ++k) Wgmma<BN, T>::ss(acc, adesc + 2 * k, bdesc + 2 * k, ((kb - kb0) | k) != 0);
      wgmma_commit();
      // the previous tile's store has had the first k-block's MMAs to read the staging tile: hand it back
      if (staged && it > 0 && kb == kb0 && stg_leader) {
        bulk_wait_group_read<0>();
        mbar_arrive(&stg_free[wg]);
      }
      wgmma_wait<1>();
      if (prev >= 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == STAGES) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    wgmma_pin(acc);
    if (prev >= 0) mbar_arrive(&empty_bar[prev]);

    if (split != 0) {
      // ===================== split-K partial: raw fp32 accumulators -> workspace =====================
      float* ws = p.ws + ((size_t)t * (S - 1) + (split - 1)) * (size_t)(BN * kBM) + ct;
#pragma unroll
      for (int j = 0; j < R; ++j) __stcg(ws + j * kGemmConsumers, acc[j]);
      __threadfence();
      named_bar_sync(1 + wg, 128);
      if ((ct & 127) == 0) atomicAdd(p.cnt + 2 * t + wg, 1);
      continue;
    }
    if (S > 1) {
      if ((ct & 127) == 0) splitk_wait(p.cnt + 2 * t + wg, S - 1);
      named_bar_sync(1 + wg, 128);
      __threadfence();
#pragma unroll 1
      for (int s2 = 0; s2 < S - 1; ++s2) {
        const float* w = p.ws + ((size_t)t * (S - 1) + s2) * (size_t)(BN * kBM) + ct;
#pragma unroll
        for (int j = 0; j < R; ++j) acc[j] += __ldcg(w + j * kGemmConsumers);
      }
    }

    if (staged) {
      // ===================== staged epilogue: registers -> staging tile (+ residual) -> TMA store =====================
      if (stage_resid) mbar_wait(&res_full[wg], it & 1, 0x23);
      else if (it > 0) mbar_wait(&stg_free[wg], (it - 1) & 1, 0x24);
      uint8_t* stg = smem + SM::kStgOffset + wg * SM::kStgBytes;
      const int rl0 = r0 - 64 * wg;                       // rows rl0, rl0 + 8 of the warpgroup's 64-row half
      float rs[2];
      const T* gb_row[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r_in_tile = r0 + 8 * h;
        long long row;
        bool row_ok;
        if (CONV) {
          const int dn = r_in_tile / (p.box_h * p.box_w);
          const int r2 = r_in_tile - dn * (p.box_h * p.box_w);
          const int dh = r2 / p.box_w;
          const int dw = r2 - dh * p.box_w;
          const int in_ = n0 + dn, ih = h0 + dh, iw = w0 + dw;
          row = ((long long)in_ * p.img_h + ih) * p.img_w + iw;
          row_ok = in_ < p.img_n && ih < p.img_h && iw < p.img_w;
        } else {
          row = (long long)tm * kBM + r_in_tile;
          row_ok = row < p.M;
        }
        // rows outside the output are computed from zero-filled operands and clipped by the store
        rs[h] = p.alpha;
        if (rscale != nullptr && row_ok) rs[h] *= Cvt<T>::to_f(rscale[row]);
        gb_row[h] = (gbias != nullptr && row_ok) ? gbias + (row / p.rows_per_group) * p.ld_group_bias : nullptr;
      }
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const int col = tn * BN + 8 * i + cq;
        if (col >= p.N) continue;
        float2 b2 = make_float2(0.f, 0.f);
        if (bias != nullptr) b2 = Cvt<T>::unpack2(*reinterpret_cast<const uint32_t*>(bias + col));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
          v0 += b2.x;
          v1 += b2.y;
          if (gb_row[h] != nullptr) {
            const float2 g2 = Cvt<T>::unpack2(*reinterpret_cast<const uint32_t*>(gb_row[h] + col));
            v0 += g2.x;
            v1 += g2.y;
          }
          if (geglu) {
            T* s = reinterpret_cast<T*>(stg + STG::offset(rl0 + 8 * h, 4 * i + (cq >> 1)));
            float o = v0 * gelu_fast(v1) * rs[h];
            if (resid != nullptr) o += Cvt<T>::to_f(*s);
            *s = Cvt<T>::from_f(o);
          } else {
            uint32_t* s = reinterpret_cast<uint32_t*>(stg + STG::offset(rl0 + 8 * h, 8 * i + cq));
            float w0_ = v0 * rs[h], w1_ = v1 * rs[h];
            if (resid != nullptr) {
              const float2 r2 = Cvt<T>::unpack2(*s);
              w0_ += r2.x;
              w1_ += r2.y;
            }
            *s = Cvt<T>::pack2(w0_, w1_);
          }
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(1 + wg, 128);
      if (stg_leader) {
        for (int ch = 0; ch < live_chunks(tn); ++ch) stg_copy(true, wg, ch, tm, tn, n0, h0, w0);
        bulk_commit_group();
      }
      continue;
    }

    // ===================== epilogue: this thread's two rows, BN/4 columns each =====================
    long long row[2];
    bool row_ok[2];
    float rs[2], ln_mu[2], ln_rstd[2], osum[2], osq[2];
    const T* gb_row[2];
    T* crow[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r_in_tile = r0 + 8 * h;
      if (CONV) {
        const int dn = r_in_tile / (p.box_h * p.box_w);
        const int r2 = r_in_tile - dn * (p.box_h * p.box_w);
        const int dh = r2 / p.box_w;
        const int dw = r2 - dh * p.box_w;
        const int in_ = n0 + dn, ih = h0 + dh, iw = w0 + dw;
        row[h] = ((long long)in_ * p.img_h + ih) * p.img_w + iw;
        row_ok[h] = in_ < p.img_n && ih < p.img_h && iw < p.img_w;   // boxes may overhang the image batch
      } else {
        row[h] = (long long)tm * kBM + r_in_tile;
        row_ok[h] = row[h] < p.M;
      }
      rs[h] = p.alpha;
      if (rscale != nullptr && row_ok[h]) rs[h] *= Cvt<T>::to_f(rscale[row[h]]);
      gb_row[h] = (gbias != nullptr && row_ok[h]) ? gbias + (row[h] / p.rows_per_group) * p.ld_group_bias : nullptr;
      // folded LayerNorm of the A rows: v = rstd * (acc - mu * colsum[n])
      ln_mu[h] = 0.f;
      ln_rstd[h] = 1.f;
      if (EPI == EPI_FULL && p.ln_stats != nullptr && row_ok[h]) {
        const float2 st = *reinterpret_cast<const float2*>(p.ln_stats + 2 * row[h]);
        ln_mu[h] = st.x / (float)p.K;
        const float var = fmaxf(st.y / (float)p.K - ln_mu[h] * ln_mu[h], 0.f);
        ln_rstd[h] = rsqrtf(var + p.ln_eps);
      }
      osum[h] = osq[h] = 0.f;
      // destination of this row: local C, or (frame-sharded motion module) the owner rank's buffer
      crow[h] = C + row[h] * p.ldc;
      if (p.sc.seg > 0 && row_ok[h]) {
        const long long sg = row[h] / p.sc.seg;
        const long long qq = row[h] - sg * p.sc.seg;
        const long long dd = sg / p.sc.segs_per_dest;
        const long long ii = sg - dd * p.sc.segs_per_dest;
        crow[h] = reinterpret_cast<T*>(p.sc.base[dd]) + (ii * p.sc.seg_stride + p.sc.row0 + qq) * p.ldc;
      }
    }
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
      const int col = tn * BN + 8 * i + cq;         // accumulator (= weight row) column of acc[4i], acc[4i + 1]
      if (col >= p.N) continue;                     // N % 8 == 0: col + 1 < N as well
      float2 b2 = make_float2(0.f, 0.f), cs = make_float2(0.f, 0.f);
      if (bias != nullptr) b2 = Cvt<T>::unpack2(*reinterpret_cast<const uint32_t*>(bias + col));
      if (EPI == EPI_FULL && p.ln_stats != nullptr) cs = *reinterpret_cast<const float2*>(p.ln_colsum + col);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!row_ok[h]) continue;
        float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
        if (EPI == EPI_FULL && p.ln_stats != nullptr) {
          v0 = ln_rstd[h] * (v0 - ln_mu[h] * cs.x);
          v1 = ln_rstd[h] * (v1 - ln_mu[h] * cs.y);
        }
        v0 += b2.x;
        v1 += b2.y;
        if (gb_row[h] != nullptr) {
          const float2 g2 = Cvt<T>::unpack2(*reinterpret_cast<const uint32_t*>(gb_row[h] + col));
          v0 += g2.x;
          v1 += g2.y;
        }
        if (EPI == EPI_FULL) {
          if (p.flags & HB_EPI_SILU) {
            v0 = silu_f(v0);
            v1 = silu_f(v1);
          } else if (p.flags & HB_EPI_RELU) {
            v0 = fmaxf(v0, 0.f);
            v1 = fmaxf(v1, 0.f);
          }
        }
        if (geglu) {
          // (value, gate) pair -> one output column
          const int oc = col >> 1;
          float o = v0 * gelu_fast(v1) * rs[h];
          if (resid != nullptr) o += Cvt<T>::to_f(resid[row[h] * p.ldr + oc]);
          crow[h][oc] = Cvt<T>::from_f(o);
        } else if (col < n_out) {
          float w0 = v0 * rs[h], w1 = v1 * rs[h];
          if (resid != nullptr) {
            const float2 r2 = Cvt<T>::unpack2(*reinterpret_cast<const uint32_t*>(resid + row[h] * p.ldr + col));
            w0 += r2.x;
            w1 += r2.y;
          }
          const uint32_t o2 = Cvt<T>::pack2(w0, w1);
          *reinterpret_cast<uint32_t*>(crow[h] + col) = o2;
          if (EPI == EPI_FULL && p.stats_out != nullptr) {
            // statistics of the values as the next LayerNorm will read them (rounded to the storage type)
            const float2 q = Cvt<T>::unpack2(o2);
            osum[h] += q.x + q.y;
            osq[h] += q.x * q.x + q.y * q.y;
          }
        }
      }
    }
    if (EPI == EPI_FULL && p.stats_out != nullptr) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        // the four lanes of a quad hold the same row
        osum[h] += __shfl_xor_sync(0xffffffffu, osum[h], 1);
        osum[h] += __shfl_xor_sync(0xffffffffu, osum[h], 2);
        osq[h] += __shfl_xor_sync(0xffffffffu, osq[h], 1);
        osq[h] += __shfl_xor_sync(0xffffffffu, osq[h], 2);
        if ((lane & 3) == 0 && row_ok[h]) {
          atomicAdd(p.stats_out + 2 * row[h], osum[h]);
          atomicAdd(p.stats_out + 2 * row[h] + 1, osq[h]);
        }
      }
    }
  }
  if (staged && stg_leader) bulk_wait_group<0>();   // the staging tiles must outlive the last stores
}

constexpr long long kSplitKCounterBytes = 8192;     // head of the split-K workspace: arrival counters
constexpr int kSplitKMinBlocks = 32;                // shortest K loop (64-wide k-blocks) that is split
static int g_last_splits = 1;                       // split factor of the most recent launch (tests / diagnostics)

// Split factor of a launch of `tiles` tiles (of cta-group `cg`) on `max_ctas` SMs; pure host arithmetic, also exported
// as hallo_b200_gemm_choose_splits for the CPU tests.  1 = unsplit.
static int choose_splits(int tiles, int max_ctas, int kblocks, int cg, int bn, long long workspace_bytes, int splitk_opt) {
  const int min_blocks = splitk_opt > 1 ? splitk_opt : kSplitKMinBlocks;
  if (splitk_opt == 0 || workspace_bytes <= kSplitKCounterBytes || tiles <= 0 || tiles * 2 > max_ctas || kblocks < min_blocks ||
      (long long)tiles * cg * 8 * (long long)sizeof(int) > kSplitKCounterBytes)
    return 1;
  int S = (int)(sqrtf((float)kblocks / 4.0f) + 0.5f);
  if (S > max_ctas / tiles) S = max_ctas / tiles;
  if (S > 16) S = 16;
  const long long tile_bytes = (long long)cg * bn * kBM * (long long)sizeof(float);
  const long long room = (workspace_bytes - kSplitKCounterBytes) / tile_bytes;      // partial tiles that fit
  while (S > 1 && (long long)tiles * (S - 1) > room) --S;
  while (S > 1 && (S - 1) * ((kblocks + S - 1) / S) >= kblocks) --S;                // no empty split
  return S > 1 ? S : 1;
}

// pick the NHWC box (box_w, box_h, box_n), box_w*box_h*box_n == 128, that covers the image batch with the
// fewest tiles; boxes may overhang (TMA zero-fills, the epilogue masks), so any image size works.
static void pick_conv_box(int n, int h, int w, int* bw, int* bh, int* bn) {
  long long best = -1;
  for (int cw = 1; cw <= 128; cw <<= 1)
    for (int ch = 1; cw * ch <= 128; ch <<= 1) {
      const int cn = 128 / (cw * ch);
      const long long tiles = (long long)((w + cw - 1) / cw) * ((h + ch - 1) / ch) * ((n + cn - 1) / cn);
      // prefer wider boxes on ties (longer contiguous TMA rows)
      if (best < 0 || tiles < best || (tiles == best && cw > *bw)) {
        best = tiles;
        *bw = cw;
        *bh = ch;
        *bn = cn;
      }
    }
}

template <typename T, int BN, int STAGES, int EPI>
static int launch_gemm(const hb_gemm_params* q, cudaStream_t stream) {
  using SM = GemmSmem<BN, STAGES>;
  static_assert(SM::kTotal <= 232448, "gemm smem budget");
  GemmDev d{};
  d.M = q->M;
  d.N = q->N;
  d.K = q->K;
  d.K1 = (q->A2 != nullptr) ? q->K1 : q->K;
  d.C = q->C;
  d.ldc = q->ldc;
  d.bias = q->bias;
  d.group_bias = q->group_bias;
  d.ld_group_bias = q->ld_group_bias;
  d.rows_per_group = q->rows_per_group > 0 ? q->rows_per_group : 1;
  d.row_scale = q->row_scale;
  d.residual = q->residual;
  d.ldr = q->ldr;
  d.alpha = q->alpha;
  d.flags = q->flags;
  d.ln_stats = q->ln_stats;
  d.ln_colsum = q->ln_colsum;
  d.ln_eps = q->ln_eps;
  d.stats_out = q->stats_out;
  if (q->scatter != nullptr) d.sc = *q->scatter;
  d.tiles_n = (q->N + BN - 1) / BN;

  CUtensorMap tmA, tmA2, tmB;
  int rc;
  {
    uint64_t dims[2] = {(uint64_t)q->K, (uint64_t)q->N};
    uint64_t str[1] = {(uint64_t)q->ldw * 2};
    uint32_t box[2] = {kBK, (uint32_t)BN};
    if ((rc = make_tmap_16b(&tmB, q->dtype, q->W, 2, dims, str, box)) != HB_OK) return rc;
  }
  if (q->conv3x3) {
    const int cin = q->K / 9;
    if (q->K % 9 != 0 || cin % kBK != 0)
      return fail(HB_ERR_BAD_SHAPE, "conv3x3 needs Cin %% 64 == 0 (K=%d)", q->K);
    if ((long long)q->img_n * q->img_h * q->img_w != q->M)
      return fail(HB_ERR_BAD_SHAPE, "conv3x3 M=%d != n*h*w", q->M);
    int bw = 1, bh = 1, bn = 128;
    pick_conv_box(q->img_n, q->img_h, q->img_w, &bw, &bh, &bn);
    d.cin = cin;
    d.img_n = q->img_n;
    d.stride2 = q->conv3x3 - 1;
    d.img_h = q->img_h;
    d.img_w = q->img_w;
    d.box_w = bw;
    d.box_h = bh;
    d.box_n = bn;
    d.tiles_w = (q->img_w + bw - 1) / bw;
    d.tiles_h = (q->img_h + bh - 1) / bh;
    d.tiles_m = d.tiles_w * d.tiles_h * ((q->img_n + bn - 1) / bn);
    uint64_t dims[4] = {(uint64_t)cin, (uint64_t)q->img_w, (uint64_t)q->img_h,
                        (uint64_t)q->img_n * (q->conv3x3 >= 2 ? 4 : 1)};
    uint64_t str[3] = {(uint64_t)q->lda * 2, (uint64_t)q->lda * 2 * q->img_w,
                       (uint64_t)q->lda * 2 * q->img_w * q->img_h};
    uint32_t box[4] = {kBK, (uint32_t)bw, (uint32_t)bh, (uint32_t)bn};
    if ((rc = make_tmap_16b(&tmA, q->dtype, q->A, 4, dims, str, box)) != HB_OK) return rc;
    tmA2 = tmA;
  } else {
    d.tiles_m = (q->M + kBM - 1) / kBM;
    uint64_t dims[2] = {(uint64_t)d.K1, (uint64_t)q->M};
    uint64_t str[1] = {(uint64_t)q->lda * 2};
    uint32_t box[2] = {kBK, kBM};
    if ((rc = make_tmap_16b(&tmA, q->dtype, q->A, 2, dims, str, box)) != HB_OK) return rc;
    if (q->A2 != nullptr) {
      uint64_t dims2[2] = {(uint64_t)(q->K - q->K1), (uint64_t)q->M};
      uint64_t str2[1] = {(uint64_t)q->lda2 * 2};
      if ((rc = make_tmap_16b(&tmA2, q->dtype, q->A2, 2, dims2, str2, box)) != HB_OK) return rc;
    } else {
      tmA2 = tmA;
    }
  }

  // staged epilogue: output / residual maps with the box of one warpgroup's half tile, CW columns wide
  constexpr int NOUT = EPI == EPI_GEGLU ? BN / 2 : BN;
  using STG = Staging<NOUT>;
  auto aligned16 = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
  d.staged = EPI != EPI_FULL && q->scatter == nullptr && aligned16(q->C) &&
             (q->residual == nullptr || aligned16(q->residual));
  CUtensorMap tmC = tmA, tmR = tmA;
  if (d.staged) {
    const uint64_t n_out = (EPI == EPI_GEGLU) ? q->N / 2 : q->N;
    auto make_out_map = [&](CUtensorMap* m, const void* base, long long ld) {
      if (q->conv3x3) {
        // half box: split the tile's (w, h, n) box along its outermost dimension that is larger than 1
        const int hn = d.box_n > 1 ? d.box_n / 2 : 1;
        const int hh = d.box_n > 1 ? d.box_h : (d.box_h > 1 ? d.box_h / 2 : 1);
        const int hw = d.box_n > 1 || d.box_h > 1 ? d.box_w : d.box_w / 2;
        d.wg_dn = d.box_n > 1 ? hn : 0;
        d.wg_dh = d.box_n == 1 && d.box_h > 1 ? hh : 0;
        d.wg_dw = d.box_n == 1 && d.box_h == 1 ? hw : 0;
        uint64_t dims[4] = {n_out, (uint64_t)q->img_w, (uint64_t)q->img_h, (uint64_t)q->img_n};
        uint64_t str[3] = {(uint64_t)ld * 2, (uint64_t)ld * 2 * q->img_w, (uint64_t)ld * 2 * q->img_w * q->img_h};
        uint32_t box[4] = {(uint32_t)STG::kCW, (uint32_t)hw, (uint32_t)hh, (uint32_t)hn};
        return make_tmap_16b(m, q->dtype, base, 4, dims, str, box, STG::kSwizzle);
      }
      uint64_t dims[2] = {n_out, (uint64_t)q->M};
      uint64_t str[1] = {(uint64_t)ld * 2};
      uint32_t box[2] = {(uint32_t)STG::kCW, 64};
      return make_tmap_16b(m, q->dtype, base, 2, dims, str, box, STG::kSwizzle);
    };
    if ((rc = make_out_map(&tmC, q->C, q->ldc)) != HB_OK) return rc;
    if (q->residual != nullptr && (rc = make_out_map(&tmR, q->residual, q->ldr)) != HB_OK) return rc;
  }

  const int tiles = d.tiles_m * d.tiles_n;
  if (tiles <= 0) return HB_OK;
  const int max_ctas = num_sms();
  // split-K: a CTA streams kblocks/S operand stages and the reducing CTA reads S-1 partial tiles (128 x BN fp32)
  // back, so the per-CTA traffic is smallest near S = sqrt(kblocks / 4).  The hand-over (partial store, fence,
  // counter, read-back) costs a few microseconds, which a K loop below kSplitKMinBlocks k-blocks does not win back;
  // an option value > 1 overrides that threshold (A/B runs).
  d.splits = choose_splits(tiles, max_ctas, q->K / kBK, 1, BN, q->workspace != nullptr ? q->workspace_bytes : 0,
                           option(OPT_GEMM_SPLITK));
  if (d.splits > 1) {
    d.cnt = reinterpret_cast<int*>(q->workspace);
    d.ws = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(q->workspace) + kSplitKCounterBytes);
  }
  g_last_splits = d.splits;
  const int grid = d.splits > 1 ? tiles * d.splits : (tiles < max_ctas ? tiles : max_ctas);
  // instantiated: GEMM with every epilogue; conv3x3 with PLAIN only (hallo_b200_gemm rejects an activation /
  // LayerNorm fold / GEGLU on a conv)
  auto kern = gemm_tc_kernel<T, BN, STAGES, false, EPI>;
  if constexpr (EPI == EPI_PLAIN) {
    if (q->conv3x3) kern = gemm_tc_kernel<T, BN, STAGES, true, EPI>;
  } else {
    if (q->conv3x3) return fail(HB_ERR_BAD_SHAPE, "internal: conv3x3 routed to a GEMM-only epilogue");
  }
  static bool attr_set[2] = {false, false};
  if (!attr_set[q->conv3x3 ? 1 : 0]) {
    HB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::kTotal));
    attr_set[q->conv3x3 ? 1 : 0] = true;
  }
  HB_CUDA_CHECK(launch_kernel(kern, dim3(grid), dim3(kGemmThreads), SM::kTotal, stream, tmA, tmA2, tmB, tmC, tmR, d));
  HB_LAUNCH_CHECK();
  return HB_OK;
}

template <typename T>
static int dispatch_gemm(const hb_gemm_params* p, cudaStream_t s) {
  // anything beyond bias / group bias / row scale / residual: the epilogue with every option decided at run time
  const bool geglu = (p->flags & HB_EPI_GEGLU) != 0;
  const bool full = (p->flags & (HB_EPI_SILU | HB_EPI_RELU)) != 0 || p->ln_stats != nullptr || p->stats_out != nullptr;
  // tile width: 160 unless N is a multiple of 128 but not of 160 (every UNet / ReferenceNet N is a multiple of 160;
  // a 160-wide tile would leave 20-37.5 % of the MMA columns of N = 128 / 256 / 512 / 1536 empty)
  if (p->N % kBN != 0 && p->N % kBN2 == 0) {
    if (full) return launch_gemm<T, kBN2, kGemmStages2, EPI_FULL>(p, s);
    if (geglu) return launch_gemm<T, kBN2, kGemmStages2, EPI_GEGLU>(p, s);
    return launch_gemm<T, kBN2, kGemmStages2, EPI_PLAIN>(p, s);
  }
  if (full) return launch_gemm<T, kBN, kGemmStages, EPI_FULL>(p, s);
  if (geglu) return launch_gemm<T, kBN, kGemmStages, EPI_GEGLU>(p, s);
  return launch_gemm<T, kBN, kGemmStages, EPI_PLAIN>(p, s);
}

}  // namespace hb

extern "C" long long hallo_b200_gemm_workspace_bytes(void) {
  // counters + 256 partial tiles of 128 x 160 fp32 (a split grid has at most one CTA per SM)
  return hb::kSplitKCounterBytes + 160LL * 256 * hb::kBM * (long long)sizeof(float);
}

extern "C" int hallo_b200_gemm_last_splits(void) { return hb::g_last_splits; }
extern "C" int hallo_b200_gemm_choose_splits(int tiles, int sm_units, int K, int cta_group, int bn, long long workspace_bytes,
                                             int option_value) {
  return hb::choose_splits(tiles, sm_units, K / hb::kBK, cta_group, bn, workspace_bytes, option_value);
}

extern "C" int hallo_b200_gemm(const hb_gemm_params* p, hb_stream_t stream) {
  using namespace hb;
  if (p == nullptr || p->A == nullptr || p->W == nullptr || p->C == nullptr)
    return fail(HB_ERR_NULL, "hallo_b200_gemm: null pointer");
  if (p->M <= 0 || p->N <= 0 || p->K <= 0 || p->K % kBK != 0)
    return fail(HB_ERR_BAD_SHAPE, "hallo_b200_gemm: M=%d N=%d K=%d (K %% 64 != 0?)", p->M, p->N, p->K);
  if (p->N % 8 != 0 || p->lda % 8 != 0 || p->ldw % 8 != 0 || p->ldc % 8 != 0 ||
      (p->residual && p->ldr % 8 != 0) || ((p->flags & HB_EPI_GEGLU) && p->N % 16 != 0))
    return fail(HB_ERR_BAD_SHAPE, "hallo_b200_gemm: leading dims / N must be multiples of 8");
  if ((p->ln_stats != nullptr) != (p->ln_colsum != nullptr) || (p->ln_stats != nullptr && (p->conv3x3 || p->N % 4 != 0)))
    return fail(HB_ERR_BAD_SHAPE, "hallo_b200_gemm: ln_stats and ln_colsum go together (plain GEMM only)");
  if (p->conv3x3 && ((p->flags & (HB_EPI_SILU | HB_EPI_RELU | HB_EPI_GEGLU)) != 0 || p->stats_out != nullptr))
    return fail(HB_ERR_BAD_SHAPE, "hallo_b200_gemm: conv3x3 takes bias / group bias / row scale / residual only");
  if (p->stats_out != nullptr && (p->flags & HB_EPI_GEGLU))
    return fail(HB_ERR_BAD_SHAPE, "hallo_b200_gemm: stats_out is not defined for the GEGLU epilogue");
  if (p->scatter != nullptr && (p->residual != nullptr || p->conv3x3 || p->scatter->seg <= 0 ||
                               p->scatter->segs_per_dest <= 0 ||
                               (p->M + p->scatter->seg - 1) / p->scatter->seg > (long long)HB_MAX_PEERS * p->scatter->segs_per_dest))
    return fail(HB_ERR_BAD_SHAPE, "hallo_b200_gemm: row scatter needs a plain GEMM without residual and <= %d destinations",
                HB_MAX_PEERS);
  if (p->workspace != nullptr && ((reinterpret_cast<uintptr_t>(p->workspace) & 15) != 0 || p->workspace_bytes < 0))
    return fail(HB_ERR_BAD_SHAPE, "hallo_b200_gemm: workspace must be 16-byte aligned");
  if (p->conv3x3 < 0 || p->conv3x3 > 3)
    return fail(HB_ERR_BAD_SHAPE, "hallo_b200_gemm: conv3x3 mode %d not in 0..3", p->conv3x3);
  if (p->A2 != nullptr && (p->K1 % kBK != 0 || p->K1 <= 0 || p->K1 >= p->K || p->conv3x3))
    return fail(HB_ERR_BAD_SHAPE, "hallo_b200_gemm: bad K split %d of %d", p->K1, p->K);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (p->dtype == HB_F16) return dispatch_gemm<__half>(p, s);
  if (p->dtype == HB_BF16) return dispatch_gemm<__nv_bfloat16>(p, s);
  return fail(HB_ERR_BAD_DTYPE, "hallo_b200_gemm: dtype %d", p->dtype);
}
