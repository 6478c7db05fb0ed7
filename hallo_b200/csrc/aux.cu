// HBM-bound helper kernels of the denoising path: LayerNorm(+PE), GroupNorm(+SiLU), the two
// small-key attentions (image/audio cross-attention, temporal attention), layout helpers and the
// CFG + DDIM update.  All use 128-bit global accesses on channels-last token matrices.
#include "host_common.cuh"
#include "ptx.cuh"

namespace hb {

template <typename T>
__device__ __forceinline__ void load8(const T* p, float (&v)[8]) {
  uint4 u = *reinterpret_cast<const uint4*>(p);
  float2 a = Cvt<T>::unpack2(u.x), b = Cvt<T>::unpack2(u.y), c = Cvt<T>::unpack2(u.z),
         d = Cvt<T>::unpack2(u.w);
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y; v[4] = c.x; v[5] = c.y; v[6] = d.x; v[7] = d.y;
}
template <typename T>
__device__ __forceinline__ void store8(T* p, const float (&v)[8]) {
  uint4 u;
  u.x = Cvt<T>::pack2(v[0], v[1]);
  u.y = Cvt<T>::pack2(v[2], v[3]);
  u.z = Cvt<T>::pack2(v[4], v[5]);
  u.w = Cvt<T>::pack2(v[6], v[7]);
  *reinterpret_cast<uint4*>(p) = u;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------------
// LayerNorm over C (one warp per row), optional sinusoidal positional-encoding add after the norm
// (motion_module.py:585-586: PE is added to LN(x) before q/k/v).
// ------------------------------------------------------------------------------------------------
template <typename T, int LPR, int VPL>
__global__ void __launch_bounds__(256) layernorm_kernel(const T* __restrict__ x, long long ldx,
                                                        T* __restrict__ out, long long ldo,
                                                        const T* __restrict__ gamma,
                                                        const T* __restrict__ beta, int rows, int C,
                                                        float eps, const float* __restrict__ pe,
                                                        const int* __restrict__ pe_index, int L,
                                                        int frames) {
  pdl_wait();
  pdl_launch();
  // LPR lanes cooperate on one row (C = LPR * VPL * 8 channels); a warp handles 32 / LPR rows.
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPR;
  const long long row = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * RPW + lane / LPR;
  const bool ok = row < rows;
  float v[VPL][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    if (ok) {
      load8(x + row * ldx + (sub + i * LPR) * 8, v[i]);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[i][j] = 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) s += v[i][j];
  }
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / C;
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float d = v[i][j] - mean;
      ss += d * d;
    }
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float rstd = rsqrtf(ss / C + eps);
  if (!ok) return;
  const float* perow = nullptr;
  if (pe != nullptr) {
    int f = (int)((row / L) % frames);
    if (pe_index != nullptr) f = pe_index[f];
    perow = pe + (long long)f * C;
  }
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int c0 = (sub + i * LPR) * 8;
    float g[8], b[8], o[8];
    load8(gamma + c0, g);
    load8(beta + c0, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float y = (v[i][j] - mean) * rstd * g[j] + b[j];
      if (perow != nullptr) {
        // the reference adds PE to the (already rounded) LN output in the model dtype
        y = Cvt<T>::to_f(Cvt<T>::from_f(y)) + perow[c0 + j];
      }
      o[j] = y;
    }
    store8(out + row * ldo + c0, o);
  }
}

// ------------------------------------------------------------------------------------------------
// GroupNorm over (C/G channels x HW pixels) per frame, channels-last, optional two-source channel
// concat (UNet skip connection), optional SiLU, optional frame re-indexing on output.
//   pass 1: per-(frame, group) sum / sum-of-squares of x - pivot   pass 2: normalise (+SiLU)
// The pivot is one element of the group (its first channel at pixel 0 of the frame).  Shifting by it keeps
// E[d^2] - E[d]^2 well conditioned when the group's mean is large against its spread: unshifted, an fp32
// E[x^2] - mean^2 loses about 2 log10(mean / std) digits (rstd off by ~4e-2 at mean / std = 100, HW = 512^2).
// ------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float gn_pivot(const T* __restrict__ x1, int C1, const T* __restrict__ x2, int C2, int HW,
                                          int n, int c) {
  return Cvt<T>::to_f(c < C1 ? x1[(long long)n * HW * C1 + c] : x2[(long long)n * HW * C2 + (c - C1)]);
}

template <typename T>
__global__ void __launch_bounds__(512) gn_stats_kernel(const T* __restrict__ x1, int C1,
                                                       const T* __restrict__ x2, int C2, int HW,
                                                       int pix_per_cta, int G,
                                                       float* __restrict__ stats) {
  pdl_wait();
  pdl_launch();
  extern __shared__ float sm[];   // [PY][C] sums, then [PY][C] sumsq
  const int C = C1 + C2;
  const int nvec = C >> 3;
  const int PY = blockDim.x / nvec;
  const int cv = threadIdx.x % nvec;
  const int py = threadIdx.x / nvec;
  const int n = blockIdx.y;
  const int p0 = blockIdx.x * pix_per_cta;
  const int p1 = min(HW, p0 + pix_per_cta);
  const int cpg = C / G;
  // pivots of the groups of this thread's 8 channels: cached loads with no dependence on the pixel loads below, so
  // both are in flight together (one division; the group index steps at each multiple of cpg)
  float s[8], q[8], pv[8];
  int next = (cv * 8 / cpg + 1) * cpg;                // first channel of the next group
  float piv = gn_pivot(x1, C1, x2, C2, HW, n, next - cpg);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    if (cv * 8 + j == next) {
      piv = gn_pivot(x1, C1, x2, C2, HW, n, next);
      next += cpg;
    }
    s[j] = q[j] = 0.f;
    pv[j] = piv;
  }
  if (py < PY) {
    const bool first = cv * 8 < C1;
    const T* base = first ? x1 + (long long)n * HW * C1 + cv * 8
                          : x2 + (long long)n * HW * C2 + (cv * 8 - C1);
    const int ld = first ? C1 : C2;
    int p = p0 + py;
    for (; p + 3 * PY < p1; p += 4 * PY) {          // 4 independent 16-byte loads in flight per thread
      float v[4][8];
#pragma unroll
      for (int u = 0; u < 4; ++u) load8(base + (long long)(p + u * PY) * ld, v[u]);
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[u][j] - pv[j];
          s[j] += d;
          q[j] += d * d;
        }
    }
    for (; p < p1; p += PY) {
      float v[8];
      load8(base + (long long)p * ld, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = v[j] - pv[j];
        s[j] += d;
        q[j] += d * d;
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      sm[py * C + cv * 8 + j] = s[j];
      sm[(PY + py) * C + cv * 8 + j] = q[j];
    }
  }
  __syncthreads();
  // reduce over PY and over the channels of each group: one thread per group
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    float a = 0.f, b = 0.f;
    for (int y = 0; y < PY; ++y)
      for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
        a += sm[y * C + c];
        b += sm[(PY + y) * C + c];
      }
    // partial sums of this pixel chunk: summed in a fixed order by gn_finalize_kernel (no atomics -> bitwise
    // reproducible, and no memset launch)
    float* dst = stats + (((long long)n * gridDim.x + blockIdx.x) * G + g) * 2;
    dst[0] = a;
    dst[1] = b;
  }
}

// per-(frame, channel) scale / shift from the group sums:  y = x * sc + sh.  The sums are of x - pivot; the pivot is
// read again from x (the same element gn_stats_kernel read), so the workspace holds nothing but the sums.
template <typename T>
__global__ void gn_finalize_kernel(const float* __restrict__ stats, int nchunks, const T* __restrict__ x1, int C1,
                                   const T* __restrict__ x2, int C2, const T* __restrict__ gamma,
                                   const T* __restrict__ beta, float eps, int G, int HW, float* __restrict__ scsh) {
  pdl_wait();
  pdl_launch();
  __shared__ float gsum[64][3];
  const int n = blockIdx.x;
  const int C = C1 + C2;
  const int cpg = C / G;
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    float a = 0.f, b = 0.f;
    for (int k = 0; k < nchunks; ++k) {
      const float* src = stats + (((long long)n * nchunks + k) * G + g) * 2;
      a += src[0];
      b += src[1];
    }
    gsum[g][0] = a;
    gsum[g][1] = b;
    gsum[g][2] = gn_pivot(x1, C1, x2, C2, HW, n, g * cpg);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const int grp = c / cpg;
    const float cnt = (float)cpg * HW;
    const float md = gsum[grp][0] / cnt;                 // mean of x - pivot
    const float m = gsum[grp][2] + md;
    const float var = fmaxf(gsum[grp][1] / cnt - md * md, 0.f);
    const float r = rsqrtf(var + eps);
    const float g = Cvt<T>::to_f(gamma[c]);
    scsh[((long long)n * 2) * C + c] = r * g;
    scsh[((long long)n * 2 + 1) * C + c] = Cvt<T>::to_f(beta[c]) - m * r * g;
  }
}

// One-launch GroupNorm for slabs that fit shared memory: CTA (frame n, group g) reads its [HW x C/G] slab once
// (kept in shared memory as raw 16-bit pairs), reduces its statistics in the CTA, then normalises (+SiLU) out of
// shared memory.  x is read once instead of twice and the stats / finalize / apply launches collapse into one.  The
// sums are of x - pivot, as in gn_stats_kernel (same pivot).  A two-pass over the slab (mean, then the sum of
// (x - mean)^2 out of shared memory) is as accurate but was measured ~5% slower at the UNet's 16x16 level.
// On by default; option "gn_fused" = 0 selects the three-launch path.
template <int V>
struct GnVec;                                     // V channel pairs = 4V bytes per access
template <>
struct GnVec<1> { using type = uint32_t; };
template <>
struct GnVec<2> { using type = uint2; };
template <>
struct GnVec<4> { using type = uint4; };

template <typename T, int V>
__global__ void __launch_bounds__(256) gn_fused_kernel(const T* __restrict__ x1, int C1, const T* __restrict__ x2, int C2,
                                                        int HW, int G, const T* __restrict__ gamma,
                                                        const T* __restrict__ beta, float eps, int silu,
                                                        T* __restrict__ out, int fpb_in, int fpb_out, int frame_off) {
  pdl_wait();
  pdl_launch();
  using Vec = typename GnVec<V>::type;
  extern __shared__ uint4 gn_slab_raw[];           // [HW][cpg / (2V)] vectors of V channel pairs
  Vec* slab = reinterpret_cast<Vec*>(gn_slab_raw);
  __shared__ float red[2][8];
  __shared__ float stat[2];
  const int C = C1 + C2;
  const int cpg = C / G;
  const int vpp = cpg / (2 * V);                   // vectors per pixel in this group
  const int n = blockIdx.y, g = blockIdx.x;
  const int c_base = g * cpg;
  const int total = HW * vpp;
  auto src_of = [&](int i) -> const Vec* {
    const int p = i / vpp;
    const int c = c_base + 2 * V * (i - p * vpp);
    const T* src = (c < C1) ? x1 + ((long long)n * HW + p) * C1 + c : x2 + ((long long)n * HW + p) * C2 + (c - C1);
    return reinterpret_cast<const Vec*>(src);
  };
  // pivot: the group's first channel at pixel 0 (a cached load, in flight with the slab loads)
  const float pv = gn_pivot(x1, C1, x2, C2, HW, n, c_base);
  float s = 0.f, q = 0.f;
  auto accum = [&](const Vec& u) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(&u);
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const float2 v = Cvt<T>::unpack2(w[k]);
      const float d0 = v.x - pv, d1 = v.y - pv;
      s += d0 + d1;
      q += d0 * d0 + d1 * d1;
    }
  };
  int i = threadIdx.x;
  for (; i + 768 < total; i += 1024) {             // 4 independent loads in flight per thread
    Vec u[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) u[k] = *src_of(i + k * 256);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      slab[i + k * 256] = u[k];
      accum(u[k]);
    }
  }
  for (; i < total; i += 256) {
    const Vec u = *src_of(i);
    slab[i] = u;
    accum(u);
  }
  // CTA sums in a fixed order (warp shuffles, then warps 0..7 by thread 0): bitwise reproducible
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = s;
    red[1][threadIdx.x >> 5] = q;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
      a += red[0][w];
      b += red[1][w];
    }
    const float cnt = (float)cpg * HW;
    const float md = a / cnt;                      // mean of x - pivot
    stat[0] = pv + md;
    stat[1] = rsqrtf(fmaxf(b / cnt - md * md, 0.f) + eps);
  }
  __syncthreads();
  const float m = stat[0], r = stat[1];
  const int n_out = (n / fpb_in) * fpb_out + frame_off + (n % fpb_in);
  for (int j = threadIdx.x; j < total; j += 256) {
    const int p = j / vpp;
    const int c = c_base + 2 * V * (j - p * vpp);
    Vec u = slab[j];
    uint32_t* w = reinterpret_cast<uint32_t*>(&u);
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const float2 v = Cvt<T>::unpack2(w[k]);
      const float g0 = Cvt<T>::to_f(gamma[c + 2 * k]) * r, g1 = Cvt<T>::to_f(gamma[c + 2 * k + 1]) * r;
      float y0 = fmaf(v.x, g0, Cvt<T>::to_f(beta[c + 2 * k]) - m * g0);
      float y1 = fmaf(v.y, g1, Cvt<T>::to_f(beta[c + 2 * k + 1]) - m * g1);
      if (silu) {
        y0 = silu_f(Cvt<T>::to_f(Cvt<T>::from_f(y0)));   // reference rounds the GN output before SiLU
        y1 = silu_f(Cvt<T>::to_f(Cvt<T>::from_f(y1)));
      }
      w[k] = Cvt<T>::pack2(y0, y1);
    }
    *reinterpret_cast<Vec*>(out + ((long long)n_out * HW + p) * C + c) = u;
  }
}

// seg > 0: rows are scattered by pixel slice -- pixel p of output frame n_out goes to base[p / seg] at row
// n_out * seg + p % seg (the frame -> pixel ownership swap in front of a motion module; base[] are peer-mapped buffers)
struct GnScatter {
  void* base[HB_MAX_PEERS];
  int seg;
};

template <typename T>
__global__ void __launch_bounds__(512) gn_apply_kernel(const T* __restrict__ x1, int C1,
                                                       const T* __restrict__ x2, int C2, int HW,
                                                       int pix_per_cta, const float* __restrict__ scsh,
                                                       int silu, T* __restrict__ out, int fpb_in,
                                                       int fpb_out, int frame_off, const GnScatter scat) {
  pdl_wait();
  pdl_launch();
  // thread (cv, py): fixed 8 channels, strided pixels -> per-channel scale/shift live in registers
  const int C = C1 + C2;
  const int nvec = C >> 3;
  const int PY = blockDim.x / nvec;
  const int cv = threadIdx.x % nvec;
  const int py = threadIdx.x / nvec;
  if (py >= PY) return;
  const int n = blockIdx.y;
  const int c0 = cv * 8;
  float sc[8], sh[8];
  {
    const float4* a = reinterpret_cast<const float4*>(scsh + ((long long)n * 2) * C + c0);
    const float4* b = reinterpret_cast<const float4*>(scsh + ((long long)n * 2 + 1) * C + c0);
    const float4 a0 = a[0], a1 = a[1], b0 = b[0], b1 = b[1];
    sc[0] = a0.x; sc[1] = a0.y; sc[2] = a0.z; sc[3] = a0.w; sc[4] = a1.x; sc[5] = a1.y; sc[6] = a1.z; sc[7] = a1.w;
    sh[0] = b0.x; sh[1] = b0.y; sh[2] = b0.z; sh[3] = b0.w; sh[4] = b1.x; sh[5] = b1.y; sh[6] = b1.z; sh[7] = b1.w;
  }
  const int n_out = (n / fpb_in) * fpb_out + frame_off + (n % fpb_in);
  const bool first = c0 < C1;
  const T* src = first ? x1 + (long long)n * HW * C1 + c0 : x2 + (long long)n * HW * C2 + (c0 - C1);
  const int ld = first ? C1 : C2;
  T* dst = out + (long long)n_out * HW * C + c0;
  const int p0 = blockIdx.x * pix_per_cta;
  const int p1 = min(HW, p0 + pix_per_cta);
  for (int p = p0 + py; p < p1; p += PY) {
    float v[8], o[8];
    load8(src + (long long)p * ld, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float y = fmaf(v[j], sc[j], sh[j]);
      if (silu) {
        y = Cvt<T>::to_f(Cvt<T>::from_f(y));   // reference rounds the GN output before SiLU
        y = silu_f(y);
      }
      o[j] = y;
    }
    if (scat.seg > 0) {
      const int d = p / scat.seg;
      store8(reinterpret_cast<T*>(scat.base[d]) + ((long long)n_out * scat.seg + (p - d * scat.seg)) * C + c0, o);
    } else {
      store8(dst + (long long)p * C, o);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Cross-attention against a handful of keys (4 image tokens / 32 audio tokens), CUDA cores.
// One thread per (query row, head); K/V of the (kv-frame, head, region) live in shared memory.
// ------------------------------------------------------------------------------------------------
template <typename T, int NK>
__global__ void __launch_bounds__(128) xattn_kernel(
    const T* __restrict__ Q, long long ldq, int q_region_stride, const T* __restrict__ K,
    const T* __restrict__ V, long long ldkv, int kv_region_stride, T* __restrict__ O, long long ldo,
    int o_region_stride, int L, int heads, int d, int kv_frame_div, float scale_log2) {
  pdl_wait();
  pdl_launch();
  extern __shared__ float smf[];   // K [NK][d] then V [NK][d] as float
  const int frame = blockIdx.y;
  const int head = blockIdx.z % heads;
  const int region = blockIdx.z / heads;
  const int kvf = frame / kv_frame_div;
  float* sK = smf;
  float* sV = smf + NK * d;
  for (int i = threadIdx.x; i < NK * d; i += blockDim.x) {
    const int k = i / d, c = i - k * d;
    const long long r = (long long)kvf * NK + k;
    sK[i] = Cvt<T>::to_f(K[r * ldkv + region * kv_region_stride + head * d + c]);
    sV[i] = Cvt<T>::to_f(V[r * ldkv + region * kv_region_stride + head * d + c]);
  }
  __syncthreads();
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= L) return;
  const long long row = (long long)frame * L + pix;
  const T* q = Q + row * ldq + region * q_region_stride + head * d;
  float s[NK];
#pragma unroll
  for (int k = 0; k < NK; ++k) s[k] = 0.f;
  for (int c = 0; c < d; c += 8) {
    float qv[8];
    load8(q + c, qv);
#pragma unroll
    for (int k = 0; k < NK; ++k) {
      const float4 k0 = *reinterpret_cast<const float4*>(sK + k * d + c);
      const float4 k1 = *reinterpret_cast<const float4*>(sK + k * d + c + 4);
      s[k] += qv[0] * k0.x + qv[1] * k0.y + qv[2] * k0.z + qv[3] * k0.w + qv[4] * k1.x +
              qv[5] * k1.y + qv[6] * k1.z + qv[7] * k1.w;
    }
  }
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < NK; ++k) mx = fmaxf(mx, s[k]);
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < NK; ++k) {
    s[k] = fast_exp2((s[k] - mx) * scale_log2);
    sum += s[k];
  }
  const float inv = 1.f / sum;
  T* o = O + row * ldo + region * o_region_stride + head * d;
  for (int c = 0; c < d; c += 8) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int k = 0; k < NK; ++k) {
      const float4 v0 = *reinterpret_cast<const float4*>(sV + k * d + c);
      const float4 v1 = *reinterpret_cast<const float4*>(sV + k * d + c + 4);
      acc[0] += s[k] * v0.x; acc[1] += s[k] * v0.y; acc[2] += s[k] * v0.z; acc[3] += s[k] * v0.w;
      acc[4] += s[k] * v1.x; acc[5] += s[k] * v1.y; acc[6] += s[k] * v1.z; acc[7] += s[k] * v1.w;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] *= inv;
    store8(o + c, acc);
  }
}

// ------------------------------------------------------------------------------------------------
// Temporal self-attention over the frame axis at each pixel (motion_module.py:579-609).
// Tokens are stored (batch, frame, pixel, channel); no transposes are materialised.
// One thread per (batch, query frame, pixel, head); keys / values stream through L1.
// ------------------------------------------------------------------------------------------------
template <typename T, int MAXF>
__global__ void __launch_bounds__(288) tattn_kernel(const T* __restrict__ Q, long long ldq,
                                                    const T* __restrict__ K,
                                                    const T* __restrict__ V, long long ldkv,
                                                    T* __restrict__ O, long long ldo, int batch,
                                                    int Fq, int Fk, int L, int heads, int d,
                                                    float scale_log2) {
  pdl_wait();
  pdl_launch();
  // thread order (head, query frame, pixel, batch): the Fq query frames of a pixel sit next to each other,
  // so the 2*Fk K/V rows of that pixel are fetched from L2 once and re-read by the other frames through L1.
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)batch * Fq * L * heads;
  if (idx >= total) return;
  const int head = (int)(idx % heads);
  long long t = idx / heads;
  const int fq = (int)(t % Fq);
  t /= Fq;
  const int pix = (int)(t % L);
  const int b = (int)(t / L);
  const T* q = Q + (((long long)b * Fq + fq) * L + pix) * ldq + head * d;
  const T* kbase = K + ((long long)b * Fk * L + pix) * ldkv + head * d;
  const T* vbase = V + ((long long)b * Fk * L + pix) * ldkv + head * d;
  const long long fstride = (long long)L * ldkv;
  float s[MAXF];
#pragma unroll
  for (int k = 0; k < MAXF; ++k) s[k] = 0.f;
  for (int c = 0; c < d; c += 8) {
    float qv[8];
    load8(q + c, qv);
#pragma unroll
    for (int k = 0; k < MAXF; ++k) {
      if (k < Fk) {
        float kv[8];
        load8(kbase + k * fstride + c, kv);
#pragma unroll
        for (int j = 0; j < 8; ++j) s[k] += qv[j] * kv[j];
      }
    }
  }
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < MAXF; ++k)
    if (k < Fk) mx = fmaxf(mx, s[k]);
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < MAXF; ++k) {
    s[k] = (k < Fk) ? fast_exp2((s[k] - mx) * scale_log2) : 0.f;
    sum += s[k];
  }
  const float inv = 1.f / sum;
  T* o = O + (((long long)b * Fq + fq) * L + pix) * ldo + head * d;
  for (int c = 0; c < d; c += 8) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int k = 0; k < MAXF; ++k) {
      if (k < Fk) {
        float vv[8];
        load8(vbase + k * fstride + c, vv);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += s[k] * vv[j];
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] *= inv;
    store8(o + c, acc);
  }
}

// Shared-memory variant: a CTA stages the K / V rows of PIX pixels (all Fk frames, all heads) with coalesced
// 128-bit loads, then one thread per (pixel, head, query frame) runs the Fk-key softmax out of shared memory
// (the lanes of a warp differ only in head / frame, so the 16-byte smem reads are conflict-free broadcasts).
template <typename T, int MAXF>
__global__ void __launch_bounds__(576) tattn_smem_kernel(const T* __restrict__ Q, long long ldq,
                                                         const T* __restrict__ K,
                                                         const T* __restrict__ V, long long ldkv,
                                                         T* __restrict__ O, long long ldo, int Fq, int Fk,
                                                         int L, int heads, int d, int pix_per_cta,
                                                         float scale_log2) {
  pdl_wait();
  pdl_launch();
  extern __shared__ uint4 sm4[];
  const int C = heads * d;
  const int cvec = C >> 3;                       // 16-byte vectors per row
  const int b = blockIdx.y;
  const int pix0 = blockIdx.x * pix_per_cta;
  const int npix = min(pix_per_cta, L - pix0);
  uint4* sK = sm4;                               // [Fk][pix_per_cta][cvec]
  uint4* sV = sm4 + (size_t)Fk * pix_per_cta * cvec;
  const int rows = Fk * npix;
  for (int i = threadIdx.x; i < rows * cvec; i += blockDim.x) {
    const int v = i % cvec;
    const int r = i / cvec;
    const int f = r / npix, p = r - f * npix;
    const long long grow = ((long long)b * Fk + f) * L + pix0 + p;
    sK[((size_t)f * pix_per_cta + p) * cvec + v] = *reinterpret_cast<const uint4*>(K + grow * ldkv + v * 8);
    sV[((size_t)f * pix_per_cta + p) * cvec + v] = *reinterpret_cast<const uint4*>(V + grow * ldkv + v * 8);
  }
  __syncthreads();
  const int per_pix = heads * Fq;
  const int p = threadIdx.x / per_pix;
  if (p >= npix) return;
  const int rem = threadIdx.x - p * per_pix;
  const int fq = rem / heads;
  const int head = rem - fq * heads;
  const int dvec = d >> 3;
  const T* q = Q + (((long long)b * Fq + fq) * L + pix0 + p) * ldq + head * d;
  float s[MAXF];
#pragma unroll
  for (int k = 0; k < MAXF; ++k) s[k] = 0.f;
  for (int c = 0; c < dvec; ++c) {
    float qv[8];
    load8(q + c * 8, qv);
#pragma unroll
    for (int k = 0; k < MAXF; ++k) {
      if (k < Fk) {
        const uint4 u = sK[((size_t)k * pix_per_cta + p) * cvec + head * dvec + c];
        const float2 a0 = Cvt<T>::unpack2(u.x), a1 = Cvt<T>::unpack2(u.y), a2 = Cvt<T>::unpack2(u.z),
                     a3 = Cvt<T>::unpack2(u.w);
        s[k] += qv[0] * a0.x + qv[1] * a0.y + qv[2] * a1.x + qv[3] * a1.y + qv[4] * a2.x + qv[5] * a2.y +
                qv[6] * a3.x + qv[7] * a3.y;
      }
    }
  }
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < MAXF; ++k)
    if (k < Fk) mx = fmaxf(mx, s[k]);
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < MAXF; ++k) {
    s[k] = (k < Fk) ? fast_exp2((s[k] - mx) * scale_log2) : 0.f;
    sum += s[k];
  }
  const float inv = 1.f / sum;
  T* o = O + (((long long)b * Fq + fq) * L + pix0 + p) * ldo + head * d;
  for (int c = 0; c < dvec; ++c) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int k = 0; k < MAXF; ++k) {
      if (k < Fk) {
        const uint4 u = sV[((size_t)k * pix_per_cta + p) * cvec + head * dvec + c];
        const float2 a0 = Cvt<T>::unpack2(u.x), a1 = Cvt<T>::unpack2(u.y), a2 = Cvt<T>::unpack2(u.z),
                     a3 = Cvt<T>::unpack2(u.w);
        acc[0] += s[k] * a0.x; acc[1] += s[k] * a0.y; acc[2] += s[k] * a1.x; acc[3] += s[k] * a1.y;
        acc[4] += s[k] * a2.x; acc[5] += s[k] * a2.y; acc[6] += s[k] * a3.x; acc[7] += s[k] * a3.y;
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] *= inv;
    store8(o + c * 8, acc);
  }
}

// ------------------------------------------------------------------------------------------------
// layout helpers
// ------------------------------------------------------------------------------------------------
// nearest 2x upsample, NHWC (resnet.py:166-183 F.interpolate(scale 2, nearest))
template <typename T>
__global__ void upsample2x_kernel(const T* __restrict__ x, T* __restrict__ out, int N, int H, int W,
                                  int C) {
  pdl_wait();
  pdl_launch();
  const int nvec = C >> 3;
  const long long total = (long long)N * (2 * H) * (2 * W) * nvec;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % nvec);
    long long t = i / nvec;
    const int ow = (int)(t % (2 * W));
    t /= (2 * W);
    const int oh = (int)(t % (2 * H));
    const int n = (int)(t / (2 * H));
    const uint4 v = *reinterpret_cast<const uint4*>(
        x + (((long long)n * H + (oh >> 1)) * W + (ow >> 1)) * C + cv * 8);
    *reinterpret_cast<uint4*>(out + i * 8) = v;
  }
}

// space-to-depth phase planes for the stride-2 conv: out[(p*2+q)*N + n, i, j, :] = x[n, 2i+p, 2j+q, :]
template <typename T>
__global__ void phase_split_kernel(const T* __restrict__ x, T* __restrict__ out, int N, int H, int W,
                                   int C) {
  pdl_wait();
  pdl_launch();
  const int nvec = C >> 3;
  const int H2 = H >> 1, W2 = W >> 1;
  const long long total = (long long)N * H * W * nvec;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int cv = (int)(i % nvec);
    long long t = i / nvec;
    const int w = (int)(t % W);
    t /= W;
    const int h = (int)(t % H);
    const int n = (int)(t / H);
    const uint4 v = *reinterpret_cast<const uint4*>(x + i * 8);
    const int pq = (h & 1) * 2 + (w & 1);
    *reinterpret_cast<uint4*>(out + ((((long long)pq * N + n) * H2 + (h >> 1)) * W2 + (w >> 1)) * C +
                              cv * 8) = v;
  }
}

// im2col of the 4-channel latent for conv_in: rows = (b, f, h, w), 64 columns = 9 taps x 4 ch (+ zero pad).
// latents: fp32 [1, Cl, F, H, W]; both CFG halves see the same latents (face_animate.py:398).
template <typename T>
__global__ void im2col_latent_kernel(const float* __restrict__ lat, T* __restrict__ out, int batch,
                                     int Cl, int F, int H, int W, long long batch_stride) {
  pdl_wait();
  pdl_launch();
  const long long total = (long long)batch * F * H * W;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int w = (int)(i % W);
  long long t = i / W;
  const int h = (int)(t % H);
  t /= H;
  const int f = (int)(t % F);
  lat += (t / F) * batch_stride;
  float v[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) v[j] = 0.f;
  for (int kh = 0; kh < 3; ++kh)
    for (int kw = 0; kw < 3; ++kw) {
      const int hh = h + kh - 1, ww = w + kw - 1;
      if (hh < 0 || hh >= H || ww < 0 || ww >= W) continue;
      for (int c = 0; c < Cl; ++c)
        v[(kh * 3 + kw) * Cl + c] = lat[(((long long)c * F + f) * H + hh) * W + ww];
    }
  T* o = out + i * 64;
#pragma unroll
  for (int j = 0; j < 64; j += 8) {
    float vv[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) vv[q] = v[j + q];
    store8(o + j, vv);
  }
}

// im2col of a small-channel fp32 NCHW image for a 3x3 stem conv, with a per-pixel affine map applied BEFORE the zero
// padding: column (kh*3 + kw)*Cl + c of row (n, h, w) = y_c(n, h + kh - 1, w + kw - 1), y = mat (scale x) + bias, and 0
// outside the image.  The VAE decoder's post_quant_conv (1x1, with bias) followed by the padded conv_in cannot be
// folded into one conv exactly (the border taps would see the bias), so it is applied here, per gathered pixel.
template <typename T>
__global__ void im2col_affine_kernel(const float* __restrict__ x, T* __restrict__ out, int N, int Cl, int H, int W,
                                     const float* __restrict__ mat, const float* __restrict__ bias, float scale) {
  pdl_wait();
  pdl_launch();
  const long long total = (long long)N * H * W;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int w = (int)(i % W);
  long long t = i / W;
  const int h = (int)(t % H);
  const int n = (int)(t / H);
  const long long plane = (long long)H * W;
  const float* xn = x + (long long)n * Cl * plane;
  float v[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) v[j] = 0.f;
  for (int kh = 0; kh < 3; ++kh)
    for (int kw = 0; kw < 3; ++kw) {
      const int hh = h + kh - 1, ww = w + kw - 1;
      if (hh < 0 || hh >= H || ww < 0 || ww >= W) continue;
      float xin[7];
      for (int c = 0; c < Cl; ++c) xin[c] = scale * xn[c * plane + (long long)hh * W + ww];
      for (int c = 0; c < Cl; ++c) {
        float y = xin[c];
        if (mat != nullptr) {
          y = 0.f;
          for (int c2 = 0; c2 < Cl; ++c2) y = fmaf(mat[c * Cl + c2], xin[c2], y);
        }
        if (bias != nullptr) y += bias[c];
        v[(kh * 3 + kw) * Cl + c] = y;
      }
    }
  T* o = out + i * 64;
#pragma unroll
  for (int j = 0; j < 64; j += 8) {
    float vv[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) vv[q] = v[j + q];
    store8(o + j, vv);
  }
}

// sinusoidal timestep embedding [cos | sin] (diffusers Timesteps(flip_sin_to_cos=True, shift 0)),
// one row per CFG half; t comes from the per-step table indexed by the device step counter.
template <typename T>
__global__ void timestep_embed_kernel(const float* __restrict__ t_table, const int* __restrict__ step,
                                      T* __restrict__ out, int rows, int dim) {
  pdl_wait();
  pdl_launch();
  const int half = dim >> 1;
  const float t = t_table[*step];
  for (int i = threadIdx.x; i < rows * dim; i += blockDim.x) {
    const int c = i % dim;
    const int k = c < half ? c : c - half;
    const float freq = expf(-9.210340371976184f * (float)k / (float)half);
    const float a = t * freq;
    out[i] = Cvt<T>::from_f(c < half ? cosf(a) : sinf(a));
  }
}

// CFG combine + DDIM v-prediction update (face_animate.py:415-420; diffusers DDIMScheduler.step, eta 0)
//   v = v_u + s (v_c - v_u);  x0 = sqrt(a_t) x - sqrt(1-a_t) v;  eps = sqrt(a_t) v + sqrt(1-a_t) x
//   x <- sqrt(a_p) x0 + sqrt(1-a_p) eps
// model_out: [2*F*H*W, ldm] channels-last (first Cl columns valid), rows [uncond | cond].
template <typename T>
__global__ void cfg_ddim_kernel(const T* __restrict__ model_out, long long ldm,
                                float* __restrict__ lat, const float* __restrict__ coef,
                                const int* __restrict__ step, float guidance, int Cl, int F, int HW,
                                float* __restrict__ v_out) {
  pdl_wait();
  pdl_launch();
  const long long total = (long long)F * HW;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float* cf = coef + 4 * (*step);
  const float sa = cf[0], sb = cf[1], sap = cf[2], sbp = cf[3];
  const int f = (int)(i / HW);
  const int p = (int)(i - (long long)f * HW);
  for (int c = 0; c < Cl; ++c) {
    const float vu = Cvt<T>::to_f(model_out[i * ldm + c]);
    const float vc = Cvt<T>::to_f(model_out[(total + i) * ldm + c]);
    const float v = vu + guidance * (vc - vu);
    float* xp = lat + ((long long)c * F + f) * HW + p;
    const float x = *xp;
    const float x0 = sa * x - sb * v;
    const float eps = sa * v + sb * x;
    *xp = sap * x0 + sbp * eps;
    if (v_out != nullptr) v_out[((long long)c * F + f) * HW + p] = v;
  }
}

// CFG combine + DPM-Solver++ (order 1 or 2, data prediction) update, one table row per step:
//   v = v_u + s (v_c - v_u);  x0 = alpha x - sigma v;  x <- a x + b x0 + c x0_prev;  x0_prev <- x0
// coef row = [alpha, sigma, a, b, c].  Rows with c == 0 (first-order steps, among them step 0 of every window) never
// read x0_hist: it is uninitialised there, and 0 * NaN would be NaN.  Same layouts and grid as cfg_ddim_kernel.
template <typename T>
__global__ void cfg_multistep_kernel(const T* __restrict__ model_out, long long ldm,
                                     float* __restrict__ lat, float* __restrict__ x0_hist,
                                     const float* __restrict__ coef, const int* __restrict__ step, float guidance,
                                     int Cl, int F, int HW) {
  pdl_wait();
  pdl_launch();
  const long long total = (long long)F * HW;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float* cf = coef + 5 * (*step);
  const float sa = cf[0], sb = cf[1], ca = cf[2], cb = cf[3], cc = cf[4];
  const int f = (int)(i / HW);
  const int p = (int)(i - (long long)f * HW);
  for (int c = 0; c < Cl; ++c) {
    const float vu = Cvt<T>::to_f(model_out[i * ldm + c]);
    const float vc = Cvt<T>::to_f(model_out[(total + i) * ldm + c]);
    const float v = vu + guidance * (vc - vu);
    const long long o = ((long long)c * F + f) * HW + p;
    const float x = lat[o];
    const float x0 = sa * x - sb * v;
    float xn = ca * x + cb * x0;
    if (cc != 0.f) xn += cc * x0_hist[o];
    lat[o] = xn;
    x0_hist[o] = x0;
  }
}

// CFG combine + ancestral (Euler-a) update in the VP form, one table row per step:
//   v = v_u + s (v_c - v_u);  x0 = alpha y - sigma v;  y <- a y + b x0 + d z
// coef row = [alpha, sigma, a, b, d]; z = noise[step][c, f, p], the step's Gaussian draw in the model dtype, laid out
// like the latents ([n_steps, Cl, F, HW]).  Same layouts and grid as cfg_ddim_kernel.
template <typename T>
__global__ void cfg_ancestral_kernel(const T* __restrict__ model_out, long long ldm, float* __restrict__ lat,
                                     const T* __restrict__ noise, const float* __restrict__ coef,
                                     const int* __restrict__ step, float guidance, int Cl, int F, int HW) {
  pdl_wait();
  pdl_launch();
  const long long total = (long long)F * HW;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int st = *step;
  const float* cf = coef + 5 * st;
  const float sa = cf[0], sb = cf[1], ca = cf[2], cb = cf[3], cd = cf[4];
  const T* z = noise + (long long)st * Cl * total;
  const int f = (int)(i / HW);
  const int p = (int)(i - (long long)f * HW);
  for (int c = 0; c < Cl; ++c) {
    const float vu = Cvt<T>::to_f(model_out[i * ldm + c]);
    const float vc = Cvt<T>::to_f(model_out[(total + i) * ldm + c]);
    const float v = vu + guidance * (vc - vu);
    const long long o = ((long long)c * F + f) * HW + p;
    const float y = lat[o];
    const float x0 = sa * y - sb * v;
    lat[o] = ca * y + cb * x0 + cd * Cvt<T>::to_f(z[o]);
  }
}

// CFG combine + UniPC (bh1 / bh2, order 1 or 2, data prediction) update, one table row per step:
//   v = v_u + s (v_c - v_u);  m = alpha x - sigma v             (data estimate at the sample the UNet saw)
//   c = kx x + kL L + k0 m + k1 m1 + k2 m2                      (UniC corrector; kx = 1 and the rest 0 on rows without it)
//   x <- pc c + p0 m + p1 m1;  L <- c;  m2 <- m1;  m1 <- m      (UniP predictor, then the history moves one step)
// coef row = [alpha, sigma, kx, kL, k0, k1, k2, pc, p0, p1].  A term with a zero coefficient never reads its buffer:
// L, m1 and m2 are uninitialised on the first rows of a window, and 0 * NaN would be NaN.  m1 is always read, since it
// moves into m2, but only enters the arithmetic when k1 or p1 is nonzero.  Same layouts and grid as cfg_ddim_kernel.
template <typename T>
__global__ void cfg_unipc_kernel(const T* __restrict__ model_out, long long ldm, float* __restrict__ lat,
                                 float* __restrict__ last, float* __restrict__ m1_hist, float* __restrict__ m2_hist,
                                 const float* __restrict__ coef, const int* __restrict__ step, float guidance,
                                 int Cl, int F, int HW) {
  pdl_wait();
  pdl_launch();
  const long long total = (long long)F * HW;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float* cf = coef + 10 * (*step);
  const float sa = cf[0], sb = cf[1], kx = cf[2], kl = cf[3], k0 = cf[4], k1 = cf[5], k2 = cf[6];
  const float pc = cf[7], p0 = cf[8], p1 = cf[9];
  const int f = (int)(i / HW);
  const int p = (int)(i - (long long)f * HW);
  for (int c = 0; c < Cl; ++c) {
    const float vu = Cvt<T>::to_f(model_out[i * ldm + c]);
    const float vc = Cvt<T>::to_f(model_out[(total + i) * ldm + c]);
    const float v = vu + guidance * (vc - vu);
    const long long o = ((long long)c * F + f) * HW + p;
    const float x = lat[o];
    const float m = sa * x - sb * v;
    const float m1 = m1_hist[o];
    float cr = k0 * m;
    if (kx != 0.f) cr += kx * x;
    if (kl != 0.f) cr += kl * last[o];
    if (k1 != 0.f) cr += k1 * m1;
    if (k2 != 0.f) cr += k2 * m2_hist[o];
    float xn = pc * cr + p0 * m;
    if (p1 != 0.f) xn += p1 * m1;
    lat[o] = xn;
    last[o] = cr;
    m2_hist[o] = m1;
    m1_hist[o] = m;
  }
}

// Three-branch CFG combine with a separate audio guidance scale (dual guidance), in place:
//   v = v_u + s (v_r - v_u) + s_a (v_c - v_r)
// model_out: [3*F*H*W, ldm] channels-last (first Cl columns valid), rows [uncond | cond | cond without audio].  v is
// computed in fp32 and written back as [0 | v] over the first two halves, so any of the two-branch step kernels above,
// run on the same buffer with guidance = 1, sees v_u + 1 (v_c - v_u) = 0 + (v - 0) = v exactly.  The one rounding this
// adds to the step is v to the model dtype; the reference's CFG combine runs in the model dtype as well.  The third
// half is not written.  Same grid as cfg_ddim_kernel; every element is owned by one thread (no atomics).
template <typename T>
__global__ void cfg_guide3_kernel(T* __restrict__ model_out, long long ldm, float guidance, float audio_guidance,
                                  int Cl, long long total) {
  pdl_wait();
  pdl_launch();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  T* u = model_out + i * ldm;
  T* c = model_out + (total + i) * ldm;
  const T* r = model_out + (2 * total + i) * ldm;
  for (int k = 0; k < Cl; ++k) {
    const float vu = Cvt<T>::to_f(u[k]);
    const float vc = Cvt<T>::to_f(c[k]);
    const float vr = Cvt<T>::to_f(r[k]);
    const float v = vu + guidance * (vr - vu) + audio_guidance * (vc - vr);
    u[k] = Cvt<T>::from_f(0.f);
    c[k] = Cvt<T>::from_f(v);
  }
}

// Guidance rescale (Lin et al. 2023, diffusers rescale_noise_cfg), in three kernels so the window-wide statistics stay
// deterministic without atomics and can be shared across frame-sharded ranks:
//   stats : v_cfg (the two- or three-branch combine above, fp32) per element; each of the HB_RESCALE_PARTIALS CTAs
//           writes (sum v_c, sum v_c^2, sum v_cfg, sum v_cfg^2), accumulated in fp64, to partials[cta]
//   reduce: one CTA sums the partials in fixed order and stores the 4 totals to every destination (this rank's slot
//           of each rank's totals table)
//   apply : every CTA forms k = phi std(v_c) / std(v_cfg) + (1 - phi) from the per-rank totals, summed in rank
//           order, and writes [0 | k v_cfg] over halves 0 and 1 in the model dtype, ready for any cfg_*_step with
//           guidance = 1 (as cfg_guide3_kernel does).  std is the unbiased one, over the n = ranks * Cl * F * HW
//           elements of the window.
// The grid of the stats kernel is fixed, the element-to-thread map depends on the shape alone, and every sum runs in
// a fixed order: the same inputs give bitwise-equal factors on every run and on every rank.
template <typename T>
__device__ __forceinline__ float cfg_combine(const T* __restrict__ mo, long long ldm, int nb, float guidance,
                                             float audio_guidance, long long total, long long i, int k, float& vc) {
  const float vu = Cvt<T>::to_f(mo[i * ldm + k]);
  vc = Cvt<T>::to_f(mo[(total + i) * ldm + k]);
  if (nb == 3) {
    const float vr = Cvt<T>::to_f(mo[(2 * total + i) * ldm + k]);
    return vu + guidance * (vr - vu) + audio_guidance * (vc - vr);
  }
  return vu + guidance * (vc - vu);
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

constexpr int kRescaleThreads = 256;

template <typename T>
__global__ void __launch_bounds__(kRescaleThreads) cfg_rescale_stats_kernel(
    const T* __restrict__ model_out, long long ldm, int nb, float guidance, float audio_guidance, int Cl,
    long long total, double* __restrict__ partials) {
  pdl_wait();
  pdl_launch();
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    for (int k = 0; k < Cl; ++k) {
      float vc;
      const float v = cfg_combine(model_out, ldm, nb, guidance, audio_guidance, total, i, k, vc);
      s[0] += vc;
      s[1] += (double)vc * vc;                     // exact: a product of two floats fits a double
      s[2] += v;
      s[3] += (double)v * v;
    }
  }
  __shared__ double red[4][kRescaleThreads / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const double w = warp_sum_d(s[q]);
    if (lane == 0) red[q][warp] = w;
  }
  __syncthreads();
  if (threadIdx.x < 4) {
    double t = 0.0;
    for (int w = 0; w < kRescaleThreads / 32; ++w) t += red[threadIdx.x][w];
    partials[blockIdx.x * 4 + threadIdx.x] = t;
  }
}

struct RescaleDst {
  double* p[HB_MAX_PEERS];
  int n;
};

// 4 warps: warp q sums quantity q over the partials (lane l takes l, l + 32, ...), then stores it to every destination.
__global__ void __launch_bounds__(128) cfg_rescale_reduce_kernel(const double* __restrict__ partials, RescaleDst dst) {
  pdl_wait();
  pdl_launch();
  const int q = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double s = 0.0;
  for (int j = lane; j < HB_RESCALE_PARTIALS; j += 32) s += partials[j * 4 + q];
  s = warp_sum_d(s);
  if (lane == 0)
    for (int d = 0; d < dst.n; ++d) dst.p[d][q] = s;
}

template <typename T>
__global__ void cfg_rescale_apply_kernel(T* __restrict__ model_out, long long ldm, int nb, float guidance,
                                         float audio_guidance, float rescale, const double* __restrict__ totals,
                                         int n_ranks, int Cl, long long total) {
  pdl_wait();
  pdl_launch();
  __shared__ float factor;
  if (threadIdx.x == 0) {
    double s[4] = {0.0, 0.0, 0.0, 0.0};
    for (int r = 0; r < n_ranks; ++r)
      for (int q = 0; q < 4; ++q) s[q] += totals[r * 4 + q];
    const double n = (double)n_ranks * Cl * total;
    double k = 1.0;
    // one-pass variances; var(v_cfg) at or below the rounding of the fp64 sums counts as std = 0: v is kept as is
    const double var_t = (s[1] - s[0] * s[0] / n) / (n - 1.0);
    const double var_g = (s[3] - s[2] * s[2] / n) / (n - 1.0);
    if (n > 1.0 && var_g > 1e-12 * (s[3] / n)) k = rescale * sqrt(fmax(var_t, 0.0) / var_g) + (1.0 - rescale);
    factor = (float)k;
  }
  __syncthreads();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float k = factor;
  for (int c = 0; c < Cl; ++c) {
    float vc;
    const float v = cfg_combine(model_out, ldm, nb, guidance, audio_guidance, total, i, c, vc);
    model_out[i * ldm + c] = Cvt<T>::from_f(0.f);
    model_out[(total + i) * ldm + c] = Cvt<T>::from_f(k * v);
  }
}

__global__ void advance_step_kernel(int* step, int n_steps) {
  pdl_wait();
  pdl_launch();
  if (threadIdx.x == 0 && blockIdx.x == 0) *step = (*step + 1) % n_steps;
}

// channels-last fp16/bf16 [rows, ld] (first C columns) -> reference layout fp32 [b, C, F, H*W]
template <typename T>
__global__ void nhwc_to_bcfhw_kernel(const T* __restrict__ x, long long ld, float* __restrict__ out,
                                     int B, int C, int F, int HW) {
  pdl_wait();
  pdl_launch();
  const long long total = (long long)B * F * HW;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int p = (int)(i % HW);
  long long t = i / HW;
  const int f = (int)(t % F);
  const int b = (int)(t / F);
  for (int c = 0; c < C; ++c)
    out[(((long long)b * C + c) * F + f) * HW + p] = Cvt<T>::to_f(x[i * ld + c]);
}

template <typename T>
__global__ void add_rows_kernel(T* __restrict__ x, const T* __restrict__ y, long long nvec) {
  pdl_wait();
  pdl_launch();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * blockDim.x) {
    float a[8], b[8];
    load8(x + i * 8, a);
    load8(y + i * 8, b);
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] += b[j];
    store8(x + i * 8, a);
  }
}

static inline int grid_for(long long total, int block, int cap_mult = 8) {
  long long g = (total + block - 1) / block;
  long long cap = (long long)num_sms() * cap_mult;
  return (int)(g < cap ? (g > 0 ? g : 1) : cap);
}

}  // namespace hb

using namespace hb;

#define HB_DISPATCH_T(dtype, ...)                                       \
  if ((dtype) == HB_F16) {                                              \
    using T = __half;                                                   \
    __VA_ARGS__                                                         \
  } else if ((dtype) == HB_BF16) {                                      \
    using T = __nv_bfloat16;                                            \
    __VA_ARGS__                                                         \
  } else {                                                              \
    return fail(HB_ERR_BAD_DTYPE, "dtype %d", (int)(dtype));            \
  }

extern "C" int hallo_b200_layernorm(int dtype, const void* x, int64_t ldx, void* out, int64_t ldo,
                                    const void* gamma, const void* beta, int rows, int C, float eps,
                                    const float* pe, const int32_t* pe_index, int L, int frames,
                                    hb_stream_t stream) {
  if (!x || !out || !gamma || !beta) return fail(HB_ERR_NULL, "layernorm: null pointer");
  if (C % 8 != 0 || ldx % 8 || ldo % 8) return fail(HB_ERR_BAD_SHAPE, "layernorm: C=%d", C);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int wpb = 8;
#define HB_LN_LAUNCH(LPR, VPL)                                                                          \
  {                                                                                                     \
    const int rpb = wpb * (32 / LPR);                                                                   \
    const int grid = (rows + rpb - 1) / rpb;                                                            \
    launch_kernel(layernorm_kernel<T, LPR, VPL>, grid, wpb * 32, 0, s, (const T*)x, ldx, (T*)out, ldo,             \
                                                             (const T*)gamma, (const T*)beta, rows, C,  \
                                                             eps, pe, pe_index, L > 0 ? L : 1,          \
                                                             frames > 0 ? frames : 1);                  \
  }
  HB_DISPATCH_T(dtype, {
    switch (C) {
      case 320: HB_LN_LAUNCH(8, 5) break;
      case 640: HB_LN_LAUNCH(16, 5) break;
      case 1280: HB_LN_LAUNCH(32, 5) break;
      case 2560: HB_LN_LAUNCH(32, 10) break;
      case 768: HB_LN_LAUNCH(32, 3) break;
      default: return fail(HB_ERR_BAD_SHAPE, "layernorm: C=%d not in {320, 640, 768, 1280, 2560}", C);
    }
  })
#undef HB_LN_LAUNCH
  HB_LAUNCH_CHECK();
  return HB_OK;
}

static int groupnorm_impl(int dtype, const void* x1, int C1, const void* x2, int C2, int N, int HW, int G,
                          const void* gamma, const void* beta, float eps, int silu, void* out, float* stats_ws,
                          int fpb_in, int fpb_out, int frame_off, const GnScatter& sc, hb_stream_t stream);

extern "C" int hallo_b200_groupnorm(int dtype, const void* x1, int C1, const void* x2, int C2, int N,
                                    int HW, int G, const void* gamma, const void* beta, float eps,
                                    int silu, void* out, float* stats_ws, int fpb_in, int fpb_out,
                                    int frame_off, hb_stream_t stream) {
  GnScatter none{};
  return groupnorm_impl(dtype, x1, C1, x2, C2, N, HW, G, gamma, beta, eps, silu, out, stats_ws, fpb_in, fpb_out,
                        frame_off, none, stream);
}

extern "C" int hallo_b200_groupnorm_scatter(int dtype, const void* x1, int C1, int N, int HW, int G,
                                            const void* gamma, const void* beta, float eps,
                                            void* const* out_peers, int n_dest, float* stats_ws, int fpb_in,
                                            int fpb_out, int frame_off, hb_stream_t stream) {
  if (!out_peers || n_dest < 1 || n_dest > HB_MAX_PEERS || HW % n_dest != 0)
    return fail(HB_ERR_BAD_SHAPE, "groupnorm_scatter: %d destinations for %d pixels", n_dest, HW);
  GnScatter sc{};
  for (int i = 0; i < n_dest; ++i) {
    if (!out_peers[i]) return fail(HB_ERR_NULL, "groupnorm_scatter: null destination %d", i);
    sc.base[i] = out_peers[i];
  }
  sc.seg = HW / n_dest;
  return groupnorm_impl(dtype, x1, C1, nullptr, 0, N, HW, G, gamma, beta, eps, 0, out_peers[0], stats_ws, fpb_in,
                        fpb_out, frame_off, sc, stream);
}

static int groupnorm_impl(int dtype, const void* x1, int C1, const void* x2, int C2, int N, int HW, int G,
                          const void* gamma, const void* beta, float eps, int silu, void* out, float* stats_ws,
                          int fpb_in, int fpb_out, int frame_off, const GnScatter& sc, hb_stream_t stream) {
  if (!x1 || !out || !gamma || !beta || !stats_ws) return fail(HB_ERR_NULL, "groupnorm: null pointer");
  const int C = C1 + C2;
  if (C1 % 8 || C2 % 8 || C % G || G > 64 || (C2 > 0 && !x2))
    return fail(HB_ERR_BAD_SHAPE, "groupnorm: C1=%d C2=%d G=%d", C1, C2, G);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  {
    // one-launch path for slabs (HW x C/G halfs) that fit shared memory (option "gn_fused", see gn_fused_kernel)
    const int cpg = C / G;
    const size_t slab = (size_t)HW * cpg * 2;
    // A CTA of the one-launch kernel reads a C/G-channel sliver of every pixel, so it wins where the slivers are wide
    // or the three launches are mostly latency.  Measured on an H100 SXM (80 GB, 400 W power limit), fp16, SiLU,
    // three launches vs one, in us: HW <= 256 (levels 2-3): 60 vs 14 (N 32, HW 64, C 1280) up to 103 vs 51 (HW 256,
    // C 2560); C/G = 40: 127 vs 104 (N 32, HW 1024, C 1280), 62 vs 23 at N 4; C/G = 20: 32 vs 20 at 5 MB (N 4, HW 1024,
    // C 640) but 66 vs 97 at 40 MB; C/G = 10 (level 0, C 320): the one-launch kernel is slower at every size measured
    // (5-80 MB, e.g. 30 vs 46 at N 4).
    const bool small = HW <= 256 || cpg >= 40 || (cpg >= 20 && (size_t)N * HW * C * 2 <= ((size_t)12 << 20));
    if (hb::option(hb::OPT_GN_FUSED) != 0 && cpg % 2 == 0 && slab <= 96 * 1024 && sc.seg == 0 && small) {
      if (fpb_in <= 0) { fpb_in = N; fpb_out = N; frame_off = 0; }
      const int vw = (cpg % 8 == 0) ? 4 : ((cpg % 4 == 0) ? 2 : 1);     // channel pairs per access (16 / 8 / 4 bytes)
      HB_DISPATCH_T(dtype, {
        auto kern = vw == 4 ? gn_fused_kernel<T, 4> : (vw == 2 ? gn_fused_kernel<T, 2> : gn_fused_kernel<T, 1>);
        HB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        launch_kernel(kern, dim3(G, N), 256, slab, s, (const T*)x1, C1, (const T*)x2, C2, HW, G, (const T*)gamma, (const T*)beta,
                                           eps, silu, (T*)out, fpb_in, fpb_out, frame_off);
      })
      HB_LAUNCH_CHECK();
      return HB_OK;
    }
  }
  // workspace: [N][chunks][G][2] partial sums, then [N][2][C] scale / shift
  const int nvec = C / 8;
  if (nvec > 512) return fail(HB_ERR_BAD_SHAPE, "groupnorm: C=%d too wide", C);
  int PY = 256 / nvec;
  if (PY < 1) PY = 1;
  const int threads = nvec * PY;
  int pix_per_cta = 64;                              // >= 2048 CTAs at 64x64x32 frames: enough loads in flight
  if (HW < pix_per_cta) pix_per_cta = HW;
  dim3 g1((HW + pix_per_cta - 1) / pix_per_cta, N);
  float* scsh = stats_ws + 2 * (size_t)N * G * g1.x;
  const size_t smem = sizeof(float) * 2 * PY * C;
  if (fpb_in <= 0) { fpb_in = N; fpb_out = N; frame_off = 0; }
  HB_DISPATCH_T(dtype, {
    launch_kernel(gn_stats_kernel<T>, g1, threads, smem, s, (const T*)x1, C1, (const T*)x2, C2, HW, pix_per_cta, G,
                                                 stats_ws);
    HB_LAUNCH_CHECK();
    launch_kernel(gn_finalize_kernel<T>, N, 256, 0, s, stats_ws, (int)g1.x, (const T*)x1, C1, (const T*)x2, C2,
                  (const T*)gamma, (const T*)beta, eps, G, HW, scsh);
    HB_LAUNCH_CHECK();
    int ppc = 64;                                     // pixels per CTA of the apply pass
    if (HW < ppc) ppc = HW;
    dim3 g2((HW + ppc - 1) / ppc, N);
    launch_kernel(gn_apply_kernel<T>, g2, threads, 0, s, (const T*)x1, C1, (const T*)x2, C2, HW, ppc, scsh, silu, (T*)out,
                                              fpb_in, fpb_out, frame_off, sc);
  })
  HB_LAUNCH_CHECK();
  return HB_OK;
}

extern "C" int hallo_b200_cross_attention(int dtype, const void* Q, int64_t ldq, int q_region_stride,
                                          const void* K, const void* V, int64_t ldkv,
                                          int kv_region_stride, void* O, int64_t ldo,
                                          int o_region_stride, int frames, int L, int heads,
                                          int head_dim, int n_keys, int kv_frame_div, int regions,
                                          hb_stream_t stream) {
  if (!Q || !K || !V || !O) return fail(HB_ERR_NULL, "cross_attention: null pointer");
  if (head_dim % 8 || (n_keys != 4 && n_keys != 32) || ldq % 8 || ldkv % 8 || ldo % 8 ||
      q_region_stride % 8 || kv_region_stride % 8 || o_region_stride % 8)
    return fail(HB_ERR_BAD_SHAPE, "cross_attention: head_dim=%d n_keys=%d", head_dim, n_keys);
  // The CUDA-core kernel reads Q and stores O 8 elements at a time (16 bytes), the tensor-core kernel stores O as
  // 32-bit pairs.  Misaligned Q / O are rejected rather than sent to either path, so that the "xattn_tc" option never
  // decides whether a call works.
  if ((reinterpret_cast<uintptr_t>(Q) | reinterpret_cast<uintptr_t>(O)) & 15)
    return fail(HB_ERR_BAD_SHAPE, "cross_attention: Q %p and O %p must be 16-byte aligned", Q, O);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  {
    // tensor-core path (csrc/attn_tc.cu) for the layouts the engine produces; CUDA cores otherwise
    const int r = hb::xattn_tc_try(dtype, Q, ldq, q_region_stride, K, V, ldkv, kv_region_stride, O, ldo, o_region_stride,
                                   frames, L, heads, head_dim, n_keys, kv_frame_div, regions, s);
    if (r <= 0) return r;
  }
  dim3 grid((L + 127) / 128, frames, heads * regions);
  const float sc = (float)(1.4426950408889634 / sqrt((double)head_dim));
  const size_t smem = sizeof(float) * 2 * n_keys * head_dim;
  HB_DISPATCH_T(dtype, {
    if (n_keys == 4)
      launch_kernel(xattn_kernel<T, 4>, grid, 128, smem, s, (const T*)Q, ldq, q_region_stride, (const T*)K,
                                                 (const T*)V, ldkv, kv_region_stride, (T*)O, ldo,
                                                 o_region_stride, L, heads, head_dim, kv_frame_div, sc);
    else
      launch_kernel(xattn_kernel<T, 32>, grid, 128, smem, s, (const T*)Q, ldq, q_region_stride, (const T*)K,
                                                  (const T*)V, ldkv, kv_region_stride, (T*)O, ldo,
                                                  o_region_stride, L, heads, head_dim, kv_frame_div, sc);
  })
  HB_LAUNCH_CHECK();
  return HB_OK;
}

extern "C" int hallo_b200_temporal_attention(int dtype, const void* Q, int64_t ldq, const void* K,
                                             const void* V, int64_t ldkv, void* O, int64_t ldo,
                                             int batch, int Fq, int Fk, int L, int heads,
                                             int head_dim, hb_stream_t stream) {
  if (!Q || !K || !V || !O) return fail(HB_ERR_NULL, "temporal_attention: null pointer");
  if (head_dim % 8 || Fk > 32 || Fk < 1 || ldq % 8 || ldkv % 8 || ldo % 8)
    return fail(HB_ERR_BAD_SHAPE, "temporal_attention: head_dim=%d Fk=%d", head_dim, Fk);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  {
    const int rc = hb::tattn_mma_try(dtype, Q, ldq, K, V, ldkv, O, ldo, batch, Fq, Fk, L, heads, head_dim, s);
    if (rc != 1) return rc;      // handled (or failed) by the tensor-core kernel; 1 = not enabled / not eligible
  }
  {
    // shared-memory variant when one pixel's threads fit a CTA and its K/V rows fit shared memory
    const int C = heads * head_dim;
    const int per_pix = heads * Fq;
    int ppc = 576 / per_pix;
    const size_t row_bytes = (size_t)2 * Fk * C * 2;                 // K + V bytes of one pixel
    while (ppc > 1 && ppc * row_bytes > 56 * 1024) --ppc;            // small CTAs: several resident per SM so the
                                                                     // K/V fill of one overlaps the math of others
    if (ppc >= 1 && ppc * row_bytes <= 200 * 1024 && Fk <= 32 && C % 8 == 0) {
      const size_t smem = ppc * row_bytes;
      dim3 grid2((L + ppc - 1) / ppc, batch);
      const float sc2 = (float)(1.4426950408889634 / sqrt((double)head_dim));
      HB_DISPATCH_T(dtype, {
        auto kern = Fk <= 18 ? tattn_smem_kernel<T, 18> : tattn_smem_kernel<T, 32>;
        HB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        launch_kernel(kern, grid2, ppc * per_pix, smem, s, (const T*)Q, ldq, (const T*)K, (const T*)V, ldkv, (T*)O, ldo, Fq,
                                               Fk, L, heads, head_dim, ppc, sc2);
      })
      HB_LAUNCH_CHECK();
      return HB_OK;
    }
  }
  const long long total = (long long)batch * Fq * L * heads;
  const int block = (heads * Fq <= 288 && (288 % (heads * Fq)) == 0) ? 288 : 256;   // whole pixels per CTA when possible
  const int grid = (int)((total + block - 1) / block);
  const float sc = (float)(1.4426950408889634 / sqrt((double)head_dim));
  HB_DISPATCH_T(dtype, {
    if (Fk <= 18)
      launch_kernel(tattn_kernel<T, 18>, grid, block, 0, s, (const T*)Q, ldq, (const T*)K, (const T*)V, ldkv, (T*)O,
                                               ldo, batch, Fq, Fk, L, heads, head_dim, sc);
    else
      launch_kernel(tattn_kernel<T, 32>, grid, block, 0, s, (const T*)Q, ldq, (const T*)K, (const T*)V, ldkv, (T*)O,
                                               ldo, batch, Fq, Fk, L, heads, head_dim, sc);
  })
  HB_LAUNCH_CHECK();
  return HB_OK;
}

extern "C" int hallo_b200_upsample2x(int dtype, const void* x, void* out, int N, int H, int W, int C,
                                     hb_stream_t stream) {
  if (!x || !out) return fail(HB_ERR_NULL, "upsample2x: null pointer");
  if (C % 8) return fail(HB_ERR_BAD_SHAPE, "upsample2x: C=%d", C);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long total = (long long)N * 4 * H * W * (C / 8);
  HB_DISPATCH_T(dtype, {
    launch_kernel(upsample2x_kernel<T>, grid_for(total, 256), 256, 0, s, (const T*)x, (T*)out, N, H, W, C);
  })
  HB_LAUNCH_CHECK();
  return HB_OK;
}

extern "C" int hallo_b200_phase_split(int dtype, const void* x, void* out, int N, int H, int W, int C,
                                      hb_stream_t stream) {
  if (!x || !out) return fail(HB_ERR_NULL, "phase_split: null pointer");
  if (C % 8 || H % 2 || W % 2) return fail(HB_ERR_BAD_SHAPE, "phase_split: C=%d H=%d W=%d", C, H, W);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long total = (long long)N * H * W * (C / 8);
  HB_DISPATCH_T(dtype, {
    launch_kernel(phase_split_kernel<T>, grid_for(total, 256), 256, 0, s, (const T*)x, (T*)out, N, H, W, C);
  })
  HB_LAUNCH_CHECK();
  return HB_OK;
}

extern "C" int hallo_b200_im2col_latent(int dtype, const float* latents, void* out, int batch, int Cl,
                                        int F, int H, int W, int per_half_latents, hb_stream_t stream) {
  if (!latents || !out) return fail(HB_ERR_NULL, "im2col_latent: null pointer");
  if (Cl * 9 > 64) return fail(HB_ERR_BAD_SHAPE, "im2col_latent: Cl=%d", Cl);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long total = (long long)batch * F * H * W;
  HB_DISPATCH_T(dtype, {
    launch_kernel(im2col_latent_kernel<T>, (int)((total + 127) / 128), 128, 0, s, 
        latents, (T*)out, batch, Cl, F, H, W, per_half_latents ? (long long)Cl * F * H * W : 0LL);
  })
  HB_LAUNCH_CHECK();
  return HB_OK;
}

extern "C" int hallo_b200_im2col_affine(int dtype, const float* x, void* out, int N, int Cl, int H, int W,
                                        const float* mat, const float* bias, float scale, hb_stream_t stream) {
  if (!x || !out) return fail(HB_ERR_NULL, "im2col_affine: null pointer");
  if (Cl < 1 || Cl * 9 > 64 || N < 0 || H <= 0 || W <= 0)
    return fail(HB_ERR_BAD_SHAPE, "im2col_affine: N=%d Cl=%d H=%d W=%d", N, Cl, H, W);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long total = (long long)N * H * W;
  if (total == 0) return HB_OK;
  HB_DISPATCH_T(dtype, {
    launch_kernel(im2col_affine_kernel<T>, (int)((total + 127) / 128), 128, 0, s, x, (T*)out, N, Cl, H, W, mat, bias,
                  scale);
  })
  HB_LAUNCH_CHECK();
  return HB_OK;
}

extern "C" int hallo_b200_timestep_embed(int dtype, const float* t_table, const int32_t* step, void* out,
                                         int rows, int dim, hb_stream_t stream) {
  if (!t_table || !step || !out) return fail(HB_ERR_NULL, "timestep_embed: null pointer");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  HB_DISPATCH_T(dtype, { launch_kernel(timestep_embed_kernel<T>, 1, 256, 0, s, t_table, step, (T*)out, rows, dim); })
  HB_LAUNCH_CHECK();
  return HB_OK;
}

extern "C" int hallo_b200_cfg_ddim_step(int dtype, const void* model_out, int64_t ldm, float* latents,
                                        const float* coef, const int32_t* step, float guidance, int Cl,
                                        int F, int HW, float* v_out, hb_stream_t stream) {
  if (!model_out || !latents || !coef || !step) return fail(HB_ERR_NULL, "cfg_ddim_step: null pointer");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long total = (long long)F * HW;
  HB_DISPATCH_T(dtype, {
    launch_kernel(cfg_ddim_kernel<T>, (int)((total + 127) / 128), 128, 0, s, (const T*)model_out, ldm, latents, coef,
                                                                  step, guidance, Cl, F, HW, v_out);
  })
  HB_LAUNCH_CHECK();
  return HB_OK;
}

extern "C" int hallo_b200_cfg_multistep_step(int dtype, const void* model_out, int64_t ldm, float* latents,
                                             float* x0_hist, const float* coef, const int32_t* step, float guidance,
                                             int Cl, int F, int HW, hb_stream_t stream) {
  if (!model_out || !latents || !x0_hist || !coef || !step)
    return fail(HB_ERR_NULL, "cfg_multistep_step: null pointer");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long total = (long long)F * HW;
  HB_DISPATCH_T(dtype, {
    launch_kernel(cfg_multistep_kernel<T>, (int)((total + 127) / 128), 128, 0, s, (const T*)model_out, ldm, latents,
                  x0_hist, coef, step, guidance, Cl, F, HW);
  })
  HB_LAUNCH_CHECK();
  return HB_OK;
}

extern "C" int hallo_b200_cfg_ancestral_step(int dtype, const void* model_out, int64_t ldm, float* latents,
                                             const void* noise, const float* coef, const int32_t* step,
                                             float guidance, int Cl, int F, int HW, hb_stream_t stream) {
  if (!model_out || !latents || !noise || !coef || !step)
    return fail(HB_ERR_NULL, "cfg_ancestral_step: null pointer");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long total = (long long)F * HW;
  HB_DISPATCH_T(dtype, {
    launch_kernel(cfg_ancestral_kernel<T>, (int)((total + 127) / 128), 128, 0, s, (const T*)model_out, ldm, latents,
                  (const T*)noise, coef, step, guidance, Cl, F, HW);
  })
  HB_LAUNCH_CHECK();
  return HB_OK;
}

extern "C" int hallo_b200_cfg_unipc_step(int dtype, const void* model_out, int64_t ldm, float* latents,
                                         float* last_sample, float* x0_hist, float* x0_hist2, const float* coef,
                                         const int32_t* step, float guidance, int Cl, int F, int HW,
                                         hb_stream_t stream) {
  if (!model_out || !latents || !last_sample || !x0_hist || !x0_hist2 || !coef || !step)
    return fail(HB_ERR_NULL, "cfg_unipc_step: null pointer");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long total = (long long)F * HW;
  HB_DISPATCH_T(dtype, {
    launch_kernel(cfg_unipc_kernel<T>, (int)((total + 127) / 128), 128, 0, s, (const T*)model_out, ldm, latents,
                  last_sample, x0_hist, x0_hist2, coef, step, guidance, Cl, F, HW);
  })
  HB_LAUNCH_CHECK();
  return HB_OK;
}

extern "C" int hallo_b200_cfg_guide3_step(int dtype, void* model_out, int64_t ldm, float guidance,
                                          float audio_guidance, int Cl, int F, int HW, hb_stream_t stream) {
  if (!model_out) return fail(HB_ERR_NULL, "cfg_guide3_step: null pointer");
  if (dtype != HB_F16 && dtype != HB_BF16) return fail(HB_ERR_BAD_DTYPE, "cfg_guide3_step: dtype %d", dtype);
  if (Cl < 1 || ldm < Cl || F < 1 || HW < 1)
    return fail(HB_ERR_BAD_SHAPE, "cfg_guide3_step: Cl=%d ldm=%lld F=%d HW=%d", Cl, (long long)ldm, F, HW);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long total = (long long)F * HW;
  HB_DISPATCH_T(dtype, {
    launch_kernel(cfg_guide3_kernel<T>, (int)((total + 127) / 128), 128, 0, s, (T*)model_out, ldm, guidance,
                  audio_guidance, Cl, total);
  })
  HB_LAUNCH_CHECK();
  return HB_OK;
}

static int check_rescale_args(const char* what, int dtype, int64_t ldm, int nb, int Cl, int F, int HW) {
  if (dtype != HB_F16 && dtype != HB_BF16) return fail(HB_ERR_BAD_DTYPE, "%s: dtype %d", what, dtype);
  if ((nb != 2 && nb != 3) || Cl < 1 || ldm < Cl || F < 1 || HW < 1)
    return fail(HB_ERR_BAD_SHAPE, "%s: nb=%d Cl=%d ldm=%lld F=%d HW=%d", what, nb, Cl, (long long)ldm, F, HW);
  return HB_OK;
}

extern "C" int hallo_b200_cfg_rescale_stats(int dtype, const void* model_out, int64_t ldm, int nb, float guidance,
                                            float audio_guidance, int Cl, int F, int HW, double* partials,
                                            hb_stream_t stream) {
  if (!model_out || !partials) return fail(HB_ERR_NULL, "cfg_rescale_stats: null pointer");
  if (int e = check_rescale_args("cfg_rescale_stats", dtype, ldm, nb, Cl, F, HW)) return e;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long total = (long long)F * HW;
  HB_DISPATCH_T(dtype, {
    launch_kernel(cfg_rescale_stats_kernel<T>, HB_RESCALE_PARTIALS, kRescaleThreads, 0, s, (const T*)model_out, ldm,
                  nb, guidance, audio_guidance, Cl, total, partials);
  })
  HB_LAUNCH_CHECK();
  return HB_OK;
}

extern "C" int hallo_b200_cfg_rescale_reduce(const double* partials, double* const* dst, int n_dst,
                                             hb_stream_t stream) {
  if (!partials || !dst) return fail(HB_ERR_NULL, "cfg_rescale_reduce: null pointer");
  if (n_dst < 1 || n_dst > HB_MAX_PEERS) return fail(HB_ERR_BAD_SHAPE, "cfg_rescale_reduce: %d destinations", n_dst);
  RescaleDst d{};
  for (int i = 0; i < n_dst; ++i) {
    if (!dst[i]) return fail(HB_ERR_NULL, "cfg_rescale_reduce: null destination %d", i);
    d.p[i] = dst[i];
  }
  d.n = n_dst;
  launch_kernel(cfg_rescale_reduce_kernel, 1, 128, 0, reinterpret_cast<cudaStream_t>(stream), partials, d);
  HB_LAUNCH_CHECK();
  return HB_OK;
}

extern "C" int hallo_b200_cfg_rescale_apply(int dtype, void* model_out, int64_t ldm, int nb, float guidance,
                                            float audio_guidance, float rescale, const double* totals, int n_ranks,
                                            int Cl, int F, int HW, hb_stream_t stream) {
  if (!model_out || !totals) return fail(HB_ERR_NULL, "cfg_rescale_apply: null pointer");
  if (int e = check_rescale_args("cfg_rescale_apply", dtype, ldm, nb, Cl, F, HW)) return e;
  if (n_ranks < 1 || n_ranks > HB_MAX_PEERS || !(rescale >= 0.f && rescale <= 1.f))
    return fail(HB_ERR_BAD_SHAPE, "cfg_rescale_apply: n_ranks=%d rescale=%g", n_ranks, (double)rescale);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long total = (long long)F * HW;
  HB_DISPATCH_T(dtype, {
    launch_kernel(cfg_rescale_apply_kernel<T>, (int)((total + 127) / 128), 128, 0, s, (T*)model_out, ldm, nb,
                  guidance, audio_guidance, rescale, totals, n_ranks, Cl, total);
  })
  HB_LAUNCH_CHECK();
  return HB_OK;
}

extern "C" int hallo_b200_advance_step(int32_t* step, int n_steps, hb_stream_t stream) {
  if (!step) return fail(HB_ERR_NULL, "advance_step: null pointer");
  launch_kernel(advance_step_kernel, 1, 32, 0, reinterpret_cast<cudaStream_t>(stream), step, n_steps);
  HB_LAUNCH_CHECK();
  return HB_OK;
}

extern "C" int hallo_b200_tokens_to_bcfhw(int dtype, const void* x, int64_t ld, float* out, int B, int C,
                                          int F, int HW, hb_stream_t stream) {
  if (!x || !out) return fail(HB_ERR_NULL, "tokens_to_bcfhw: null pointer");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long total = (long long)B * F * HW;
  HB_DISPATCH_T(dtype, {
    launch_kernel(nhwc_to_bcfhw_kernel<T>, (int)((total + 127) / 128), 128, 0, s, (const T*)x, ld, out, B, C, F, HW);
  })
  HB_LAUNCH_CHECK();
  return HB_OK;
}
