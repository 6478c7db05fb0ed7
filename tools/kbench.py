"""Micro-benchmarks of individual kernels (CUDA-event timed, L2 flushed between reps).

Usage (on an H100):  python tools/kbench.py gemm conv attn ...
Prints one line per case: name, time, TFLOP/s (algorithmic) and fraction of the H100 SXM data-sheet dense fp16/bf16
rate (989 TFLOP/s at 700 W; a power-limited card reaches less).  gemm / conv run the denoising step's shapes with their
epilogues and print each one's data-sheet lower bound (FLOPs or HBM bytes), which of the two sets it, and the fraction
of it reached.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hallo_b200 import ops  # noqa: E402

PEAK = 989.0

_flush = None


def timeit(fn, reps=10, warm=3):
    global _flush
    if _flush is None:
        _flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        _flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def report(name, ms, flops):
    tf = flops / ms / 1e9
    print(f"{name:48s} {ms:9.4f} ms {tf:9.1f} TFLOP/s  {tf / PEAK:6.3f} of measured peak", flush=True)


# H100 SXM data-sheet rates (700 W): dense fp16/bf16 tensor FLOP/s and HBM3 bandwidth
PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35


def report_bound(name, ms, flops, nbytes):
    """time, the least time at data-sheet rates (larger of FLOPs / peak and bytes / bandwidth), what sets it, and
    the fraction of that bound reached."""
    t_tc, t_hbm = flops / PEAK_TFLOPS / 1e9, nbytes / PEAK_TBS / 1e9
    bound = max(t_tc, t_hbm)
    print(f"{name:44s} {ms * 1e3:9.1f} us  bound {bound * 1e3:8.1f} us ({'tensor' if t_tc >= t_hbm else 'hbm':6s})"
          f"  {bound / ms:6.3f} of bound  {flops / ms / 1e9:6.1f} TFLOP/s  {nbytes / ms / 1e9:6.2f} TB/s", flush=True)


# The denoising step's GEMMs (512x512, 16 frames, CFG batch 2): shape, epilogue, launches per step.  "res" = bias +
# residual (to_out, proj_out, FF2, audio zero-conv, conv2 of a ResNet), "geglu" = FF1 with its GEGLU epilogue.
STEP_GEMMS = [(131072, 320, 320, "res", 25), (131072, 320, 320, "", 25), (131072, 320, 1280, "res", 10),
              (147456, 320, 1280, "res", 5), (147456, 320, 320, "res", 10), (32768, 640, 640, "res", 17),
              (131072, 320, 960, "res", 5), (32768, 640, 2560, "res", 6), (8192, 1280, 5120, "res", 6),
              (131072, 2560, 320, "geglu", 10), (147456, 2560, 320, "geglu", 5), (32768, 5120, 640, "geglu", 6),
              (8192, 10240, 1280, "geglu", 6), (131072, 960, 320, "", 15), (147456, 960, 320, "", 10),
              (8192, 1280, 1280, "res", 31), (36864, 1920, 640, "", 10)]
# (n, h, cin, cout, residual): conv1 / conv2 of the ResNets at each level, and the 8-channel conv_out head
STEP_CONVS = [(32, 64, 320, 320, True), (32, 32, 640, 640, True), (32, 16, 1280, 1280, True),
              (32, 16, 2560, 1280, False), (32, 8, 1280, 1280, True), (32, 64, 960, 320, False),
              (32, 64, 640, 320, False), (32, 64, 320, 8, False)]


def bench_gemm():
    dev = "cuda"
    for (M, N, K, epi, count) in STEP_GEMMS:
        geglu, res = epi == "geglu", epi == "res"
        n_out = N // 2 if geglu else N
        a = torch.randn(M, K, device=dev, dtype=torch.float16)
        w = torch.randn(N, K, device=dev, dtype=torch.float16) * 0.02
        bias = torch.randn(N, device=dev, dtype=torch.float16)
        out = torch.empty(M, n_out, device=dev, dtype=torch.float16)
        r = torch.randn(M, n_out, device=dev, dtype=torch.float16) if res else None
        ms = timeit(lambda: ops.gemm(a, w, out, bias=bias, residual=r, geglu=geglu))
        nbytes = 2 * (M * K + N * K + M * n_out * (2 if res else 1))
        report_bound(f"gemm M{M} N{N} K{K} {epi or 'bias'} x{count}", ms, 2.0 * M * N * K, nbytes)


def bench_conv():
    dev = "cuda"
    for (n, h, cin, cout, res) in STEP_CONVS:
        x = torch.randn(n, h, h, cin, device=dev, dtype=torch.float16)
        w = torch.randn(cout, 9 * cin, device=dev, dtype=torch.float16) * 0.01
        bias = torch.randn(cout, device=dev, dtype=torch.float16)
        out = torch.empty(n * h * h, cout, device=dev, dtype=torch.float16)
        r = torch.randn(n * h * h, cout, device=dev, dtype=torch.float16) if res else None
        ms = timeit(lambda: ops.conv3x3(x, w, out, bias=bias, residual=r))
        M = n * h * h
        nbytes = 2 * (M * cin + 9 * cin * cout + M * cout * (2 if res else 1))
        report_bound(f"conv3x3 n{n} {h}x{h} {cin}->{cout}{' res' if res else ''}", ms, 2.0 * M * 9 * cin * cout,
                     nbytes)


def bench_attn():
    dev = "cuda"
    for (C, L, frames, with_ref) in [(320, 4096, 32, True), (320, 4096, 32, False), (640, 1024, 32, True),
                                     (1280, 256, 32, True), (1280, 64, 32, True)]:
        qkv = torch.randn(frames * L, 3 * C, device=dev, dtype=torch.float16)
        q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
        kvref = torch.randn(2 * L, 2 * C, device=dev, dtype=torch.float16)
        out = torch.empty(frames * L, C, device=dev, dtype=torch.float16)
        ridx = torch.tensor([-1] * (frames // 2) + [n % 2 for n in range(frames // 2)], dtype=torch.int32, device=dev)
        if with_ref:
            fn = lambda: ops.attention(q, k, v, out, heads=8, L=L, kref=kvref[:, :C], vref=kvref[:, C:], ref_index=ridx)
            flops = 4.0 * (frames // 2) * L * (2 * L) * C + 4.0 * (frames // 2) * L * L * C
        else:
            fn = lambda: ops.attention(q, k, v, out, heads=8, L=L)
            flops = 4.0 * frames * L * L * C
        ms = timeit(fn)
        report(f"attn C{C} L{L} f{frames} ref={with_ref}", ms, flops)
        if not with_ref:
            qh = q.reshape(frames, L, 8, C // 8).transpose(1, 2)
            kh = k.reshape(frames, L, 8, C // 8).transpose(1, 2)
            vh = v.reshape(frames, L, 8, C // 8).transpose(1, 2)
            ms = timeit(lambda: torch.nn.functional.scaled_dot_product_attention(qh, kh, vh))
            report("  torch sdpa same shape", ms, flops)


if __name__ == "__main__":
    which = sys.argv[1:] or ["gemm", "conv"]
    for wname in which:
        globals()["bench_" + wname]()
