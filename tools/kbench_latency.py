"""GPU-side latency of SMALL kernels (the regime of levels 2-3 and of a sharded rank): N identical launches captured in
one CUDA graph (stream-ordered, so they serialise), total time / N.  Compares the GEMM run-time options, against a
trivial kernel as the floor.
    python tools/kbench_latency.py            (on an H100)"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hallo_b200 import lib, ops  # noqa: E402

dev = "cuda"
REPS = 200


def graph_time(fn, reps=REPS):
    fn()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = 1e9
    for _ in range(3):
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best / reps * 1e3          # us per launch


def main():
    x = torch.randn(256, 320, device=dev, dtype=torch.float16)
    g_, b_ = torch.ones(320, device=dev, dtype=torch.float16), torch.zeros(320, device=dev, dtype=torch.float16)
    o = torch.empty_like(x)
    print(f"floor: layernorm 256x320                          {graph_time(lambda: ops.layernorm(x, g_, b_, o)):7.2f} us", flush=True)
    shapes = [(256, 1280, 1280), (1024, 1280, 1280), (4096, 640, 640), (16384, 320, 320), (1024, 640, 640), (256, 320, 320),
              (8192, 1280, 1280), (32768, 640, 640)]
    variants = [("default", {}), ("pdl=1 (prologue under the predecessor's tail)", {"pdl": 1}), ("gemm_splitk=0", {"gemm_splitk": 0})]
    for (M, N, K) in shapes:
        a = torch.randn(M, K, device=dev, dtype=torch.float16)
        w = torch.randn(N, K, device=dev, dtype=torch.float16) * 0.02
        out = torch.empty(M, N, device=dev, dtype=torch.float16)
        bias = torch.randn(N, device=dev, dtype=torch.float16)
        res = torch.randn(M, N, device=dev, dtype=torch.float16)
        for name, opts in variants:
            saved = {k: lib.get_option(k) for k in opts}
            for k, v in opts.items():
                lib.set_option(k, v)
            t_plain = graph_time(lambda: ops.gemm(a, w, out))
            t_res = graph_time(lambda: ops.gemm(a, w, out, bias=bias, residual=res))
            for k, v in saved.items():
                lib.set_option(k, v)
            print(f"gemm M{M:<6d} N{N:<5d} K{K:<5d} {name:40s} {t_plain:7.2f} us   +bias+residual {t_res:7.2f} us", flush=True)
        t = graph_time(lambda: torch.matmul(a, w.t()))
        print(f"gemm M{M:<6d} N{N:<5d} K{K:<5d} {'cuBLAS (torch.matmul)':40s} {t:7.2f} us", flush=True)


if __name__ == "__main__":
    main()
