"""Time hallo_b200_groupnorm (both paths) on the UNet and VAE shapes, with F.group_norm on the same data as a yardstick
for the run-to-run spread.

Each round times `--launches` back-to-back launches between two CUDA events, after `--warmup` launches of every
shape; rounds alternate between the libraries given with --lib (several builds of the same sources can be compared in
one process) and the paths (option gn_fused on / off).  Prints the card's name and power limit, then one line per
(shape, library, path): median, min and max microseconds per launch over the rounds.

    python tools/time_groupnorm.py [--lib path/to/libhallo_b200.so ...] [--rounds 7] [--launches 200]
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (name, frames, hw, channels, silu)
SHAPES = [
    ("unet_L0 32x4096x320 silu", 32, 4096, 320, True),
    ("unet_L2 32x256x1280 silu", 32, 256, 1280, True),
    ("vae_512 2x262144x128", 2, 262144, 128, False),
    ("vae_256 2x65536x256", 2, 65536, 256, False),
    ("vae_256 2x65536x512", 2, 65536, 512, False),
]
GROUPS = 32


def card():
    """Name, power limit and max SM clock as nvidia-smi reports them (read-only query)."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30)
        name, power, clock = [s.strip() for s in q.stdout.strip().split(",")]
        return f"{name}, power limit {power}, max SM clock {clock}"
    except Exception as e:                       # noqa: BLE001 -- reported, not fatal
        return f"{torch.cuda.get_device_name()}, power limit unknown ({e})"


class Lib:
    """One build of the library, called through its C ABI."""

    def __init__(self, path):
        self.path = path
        self.h = C.CDLL(path)
        self.h.hallo_b200_set_option.argtypes = [C.c_char_p, C.c_int]
        self.h.hallo_b200_last_error.restype = C.c_char_p

    def set_fused(self, on):
        assert self.h.hallo_b200_set_option(b"gn_fused", 1 if on else 0) == 0

    def groupnorm(self, x, gamma, beta, out, ws, n, hw, silu):
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        rc = self.h.hallo_b200_groupnorm(
            C.c_int(0 if x.dtype == torch.float16 else 1), C.c_void_p(x.data_ptr()), C.c_int(x.shape[1]), None,
            C.c_int(0), C.c_int(n), C.c_int(hw), C.c_int(GROUPS), C.c_void_p(gamma.data_ptr()),
            C.c_void_p(beta.data_ptr()), C.c_float(1e-5), C.c_int(1 if silu else 0), C.c_void_p(out.data_ptr()),
            C.c_void_p(ws.data_ptr()), C.c_int(0), C.c_int(0), C.c_int(0), stream)
        if rc != 0:
            raise RuntimeError(f"{self.path}: groupnorm failed: {self.h.hallo_b200_last_error().decode()}")


def time_us(fn, launches):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], help="library build to time (repeatable); default: in-tree")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--dtype", default="f16", choices=["f16", "bf16"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_groupnorm.py needs a CUDA device")
    if not args.lib:
        import __graft_entry__ as g
        g.build()
        args.lib = [os.path.join(ROOT, "hallo_b200", "libhallo_b200.so")]
    libs = [Lib(os.path.abspath(p)) for p in args.lib]
    dt = torch.float16 if args.dtype == "f16" else torch.bfloat16
    dev = torch.device("cuda:0")
    print(f"# {card()}; {args.dtype}; {args.rounds} rounds x {args.launches} launches", flush=True)
    gen = torch.Generator(device=dev).manual_seed(0)
    for name, n, hw, c, silu in SHAPES:
        x = torch.randn(n * hw, c, generator=gen, device=dev).to(dt)
        gamma = (1 + 0.1 * torch.randn(c, generator=gen, device=dev)).to(dt)
        beta = (0.1 * torch.randn(c, generator=gen, device=dev)).to(dt)
        out = torch.empty_like(x)
        ws = torch.empty(2 * n * (GROUPS * ((hw + 63) // 64) + c), device=dev, dtype=torch.float32)
        x_nchw = x.view(n, hw, c).permute(0, 2, 1).contiguous()

        def yardstick():
            y = F.group_norm(x_nchw, GROUPS, gamma, beta, 1e-5)
            return F.silu(y) if silu else y

        runs = {(lib.path, fused): [] for lib in libs for fused in (True, False)}
        runs[("F.group_norm", None)] = []

        def call(lib, fused):
            lib.set_fused(fused)
            return lambda: lib.groupnorm(x, gamma, beta, out, ws, n, hw, silu)

        for (path, fused) in runs:
            fn = yardstick if fused is None else call(next(l for l in libs if l.path == path), fused)
            for _ in range(args.warmup):
                fn()
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for (path, fused), ts in runs.items():
                fn = yardstick if fused is None else call(next(l for l in libs if l.path == path), fused)
                ts.append(time_us(fn, args.launches))
        for (path, fused), ts in runs.items():
            label = path if fused is None else f"{os.path.relpath(path, ROOT)} gn_fused={int(fused)}"
            print(f"{name:28s} {label:52s} median {statistics.median(ts):8.1f} us  "
                  f"min {min(ts):8.1f}  max {max(ts):8.1f}", flush=True)
    for lib in libs:
        lib.set_fused(True)


if __name__ == "__main__":
    main()
