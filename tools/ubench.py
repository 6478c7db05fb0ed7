"""Instruction-throughput micro-benchmarks on the SM (per-SM per-clock rates) -- evidence for softmax design."""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hallo_b200 import lib  # noqa: E402

NAMES = {0: "ex2.approx.ftz.f32", 1: "ex2.approx.ftz.f16x2", 2: "ex2.approx.ftz.bf16x2", 3: "fma.rn.f32 (3-reg)",
         4: "max.f32", 5: "cvt.rn.f16x2.f32", 6: "add.f32", 7: "mma.sync.m16n8k16.f16 (per-thread count)"}
h = C.CDLL(os.path.join(os.path.dirname(os.path.abspath(__file__)), "libhb_ubench.so"))
scratch = torch.zeros(16, device="cuda")
iters = 4096
sms = torch.cuda.get_device_properties(0).multi_processor_count
clk = 1.98e9       # H100 SXM maximum SM clock
for mode, name in NAMES.items():
    for _ in range(2):
        n = h.hb_ubench_exp(C.c_int(mode), C.c_int(iters), C.c_void_p(scratch.data_ptr()), lib.current_stream())
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    n = h.hb_ubench_exp(C.c_int(mode), C.c_int(iters), C.c_void_p(scratch.data_ptr()), lib.current_stream())
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    ops = n * iters * 8
    per_sm_clk = ops / (ms * 1e-3) / sms / clk
    extra = ""
    if mode == 7:     # one warp-level MMA = 16 x 8 x 16 x 2 flop
        extra = f"  = {per_sm_clk / 32 * 4096:8.0f} FLOP/clk/SM = {per_sm_clk / 32 * 4096 * sms * clk / 1e12:7.1f} TFLOP/s"
    print(f"{name:26s} {ms:8.3f} ms  {per_sm_clk:7.1f} thread-instr / clk / SM (at 1980 MHz){extra}", flush=True)
