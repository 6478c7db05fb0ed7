"""Micro-benchmarks of individual kernels (CUDA-event timed, L2 flushed between reps).

Usage (on an H100):  python tools/kbench.py gemm conv attn ...
Prints one line per case: name, ms, TFLOP/s (algorithmic) and fraction of the H100 SXM data-sheet dense fp16/bf16
rate (989 TFLOP/s at 700 W; a power-limited card reaches less).
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


def bench_gemm():
    dev = "cuda"
    for (M, N, K, geglu) in [(131072, 320, 320, False), (131072, 2560, 320, True), (131072, 320, 1280, False),
                             (32768, 640, 640, False), (32768, 5120, 640, True), (8192, 1280, 1280, False),
                             (8192, 10240, 1280, True), (8192, 1280, 5120, False), (147456, 320, 320, False)]:
        a = torch.randn(M, K, device=dev, dtype=torch.float16)
        w = torch.randn(N, K, device=dev, dtype=torch.float16) * 0.02
        out = torch.empty(M, N // 2 if geglu else N, device=dev, dtype=torch.float16)
        ms = timeit(lambda: ops.gemm(a, w, out, geglu=geglu))
        report(f"gemm M{M} N{N} K{K}{' geglu' if geglu else ''}", ms, 2.0 * M * N * K)
        if not geglu and N <= 1280:
            res = torch.randn(M, N, device=dev, dtype=torch.float16)
            bias = torch.randn(N, device=dev, dtype=torch.float16)
            ms = timeit(lambda: ops.gemm(a, w, out, bias=bias, residual=res))
            report(f"gemm M{M} N{N} K{K} +bias+residual", ms, 2.0 * M * N * K)
        ms = timeit(lambda: torch.matmul(a, w.t()))
        report(f"  cublas same shape", ms, 2.0 * M * N * K)


def bench_conv():
    dev = "cuda"
    for (n, h, cin, cout) in [(32, 64, 320, 320), (32, 32, 640, 640), (32, 16, 1280, 1280), (32, 8, 1280, 1280),
                              (32, 64, 960, 320), (32, 16, 2560, 1280)]:
        x = torch.randn(n, h, h, cin, device=dev, dtype=torch.float16)
        w = torch.randn(cout, 9 * cin, device=dev, dtype=torch.float16) * 0.01
        out = torch.empty(n * h * h, cout, device=dev, dtype=torch.float16)
        ms = timeit(lambda: ops.conv3x3(x, w, out))
        report(f"conv3x3 n{n} {h}x{h} {cin}->{cout}", ms, 2.0 * n * h * h * 9 * cin * cout)




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
