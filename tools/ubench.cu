// Micro-benchmarks of instruction throughput that drive kernel design decisions (not on the product path).
// Built by __graft_entry__.build() into tools/libhb_ubench.so -- a design-evidence tool, NOT part of libhallo_b200.so
// nor of include/hallo_b200.h.
#include "../hallo_b200/csrc/host_common.cuh"
#include "../hallo_b200/csrc/ptx.cuh"

namespace hb {   // this standalone library carries its own copies of the two host globals it touches
char g_last_error[512] = "";
std::atomic<int64_t> g_launch_count{0};
}

namespace hb {

template <int MODE>
__global__ void __launch_bounds__(256) ubench_exp_kernel(float* out, int iters, float seed) {
  // 8 independent dependency chains per thread
  float a[8];
  uint32_t h[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    a[i] = seed * (float)(threadIdx.x + i + 1) * 1e-3f;
    __half2 t = __floats2half2_rn(a[i], -a[i]);
    h[i] = *reinterpret_cast<uint32_t*>(&t);
  }
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (MODE == 0) {
        asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(a[i]) : "f"(a[i]));
      } else if (MODE == 1) {
        asm volatile("ex2.approx.f16x2 %0, %1;" : "=r"(h[i]) : "r"(h[i]));
      } else if (MODE == 2) {
        asm volatile("ex2.approx.ftz.bf16x2 %0, %1;" : "=r"(h[i]) : "r"(h[i]));
      } else if (MODE == 3) {
        asm volatile("fma.rn.f32 %0, %1, %1, %0;" : "+f"(a[i]) : "f"(seed));
      } else if (MODE == 4) {
        asm volatile("max.f32 %0, %0, %1;" : "+f"(a[i]) : "f"(seed));
      } else if (MODE == 5) {
        asm volatile("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(h[i]) : "f"(a[i]), "f"(seed));
      } else if (MODE == 6) {
        asm volatile("add.f32 %0, %0, %1;" : "+f"(a[i]) : "f"(seed));
      }
    }
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += a[i] + __uint_as_float(h[i]);
  if (s == 123.456f) out[0] = s;
}

// mma.sync m16n8k16 (f16 in, f32 accumulate): 8 independent accumulator chains per warp
__global__ void __launch_bounds__(256) ubench_mma_sync_kernel(float* out, int iters) {
  float d[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) d[i][e] = 0.f;
  const uint32_t a0 = 0x3c003c00u + threadIdx.x, b0 = 0x38003800u;     // (1.0, 1.0)-ish / (0.5, 0.5)
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      asm volatile(
          "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
          "{%0, %1, %2, %3};\n"
          : "+f"(d[i][0]), "+f"(d[i][1]), "+f"(d[i][2]), "+f"(d[i][3])
          : "r"(a0), "r"(a0), "r"(a0), "r"(a0), "r"(b0), "r"(b0));
    }
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += d[i][0] + d[i][1] + d[i][2] + d[i][3];
  if (s == 123.456f) out[0] = s;
}

}  // namespace hb

// returns ops (thread-level instructions) executed per launch; caller times it
extern "C" int hb_ubench_exp(int mode, int iters, float* scratch, hb_stream_t stream) {
  using namespace hb;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int grid = num_sms() * 8;
  switch (mode) {
    case 0: ubench_exp_kernel<0><<<grid, 256, 0, s>>>(scratch, iters, 0.5f); break;
    case 1: ubench_exp_kernel<1><<<grid, 256, 0, s>>>(scratch, iters, 0.5f); break;
    case 2: ubench_exp_kernel<2><<<grid, 256, 0, s>>>(scratch, iters, 0.5f); break;
    case 3: ubench_exp_kernel<3><<<grid, 256, 0, s>>>(scratch, iters, 0.5f); break;
    case 4: ubench_exp_kernel<4><<<grid, 256, 0, s>>>(scratch, iters, 0.5f); break;
    case 5: ubench_exp_kernel<5><<<grid, 256, 0, s>>>(scratch, iters, 0.5f); break;
    case 6: ubench_exp_kernel<6><<<grid, 256, 0, s>>>(scratch, iters, 0.5f); break;
    case 7: ubench_mma_sync_kernel<<<grid, 256, 0, s>>>(scratch, iters); break;
    default: return fail(HB_ERR_BAD_SHAPE, "ubench mode %d", mode);
  }
  HB_LAUNCH_CHECK();
  return grid * 256;
}
