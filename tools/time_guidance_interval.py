"""Cost of guided and unguided steps under guidance limited to an interval: the bench workload (random-init weights,
512x512 = latent 64x64, 16 frames, CFG 3.5, DDIM, 40-step schedule).  A guided step replays the two-branch engine's CUDA
graph; an unguided step replays its cond-only companion's graph (the UNet on the cond rows alone, then the same DDIM
step on v = v_c).  Rounds of each are alternated in one process so both see the same card state.

Prints one JSON line: ms per guided and per unguided step (median over the repetitions) and their ratio, peak device
memory after the two-branch engine is captured and again after the companion is captured too, one whole 40-step window
with an example interval (its guided-step count, its time, and the rel L2 of its final latents against a window guided
at every step), the card name, its power limit and the median SM clock sampled while timing.

    python tools/time_guidance_interval.py [--size 64] [--frames 16] [--steps 10] [--reps 5] [--warmup 3]
                                           [--interval 200,800] [--json FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=64, help="latent side (64 = 512x512)")
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--steps", type=int, default=10, help="timed steps per repetition")
    ap.add_argument("--reps", type=int, default=5, help="repetitions per kind of step, alternated")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--interval", default="200,800", help="t_lo,t_hi of the example window")
    ap.add_argument("--json", default="", help="also write the result line to this file")
    args = ap.parse_args()

    import torch
    from bench import ClockSampler
    from time_audio_guidance import card
    from hallo_b200.dist import window_inputs_to_device
    from hallo_b200.engine import DenoiseEngine, PackedWeights, guided_steps
    from hallo_b200.scheduler import DDIMScheduler
    from hallo_b200.spec import UNetConfig
    from hallo_b200.synth import synth_inputs, synth_state_dict_device

    if not torch.cuda.is_available():
        raise SystemExit("time_guidance_interval.py measures on a CUDA device; none is available")
    dev, dt = torch.device("cuda:0"), torch.float16
    cfg = UNetConfig()
    W = PackedWeights(synth_state_dict_device(cfg, dev, seed=0), cfg, dev, dt)
    inp = synth_inputs(cfg, args.size, args.size, args.frames, seed=42)
    win = window_inputs_to_device(inp, dev, dt)
    sch = DDIMScheduler()
    sch.set_timesteps(40)
    ts, coef = sch.timesteps.tolist(), sch.coef_table()
    n = len(ts)
    lat0 = inp["sample"][:1].float().to(dev)
    interval = tuple(float(x) for x in args.interval.split(","))

    eng = DenoiseEngine(W, args.size, args.size, args.frames)
    eng.begin_window(**win)
    eng.set_schedule(ts, coef, 3.5)
    eng.latents.copy_(lat0)
    eng.capture()
    for _ in range(args.warmup):
        eng.step()
    torch.cuda.synchronize()
    peak_main = torch.cuda.max_memory_allocated(dev)
    main_graph = eng.graph
    eng.set_schedule(ts, coef, 3.5, guided=[False] * n)            # every step unguided: the companion's graph
    assert eng.graph is main_graph
    cond = eng.cond_engine()
    cond.capture()
    for _ in range(args.warmup):
        eng.step()
    torch.cuda.synchronize()
    peak_both = torch.cuda.max_memory_allocated(dev)

    masks = {"guided": None, "unguided": [False] * n}
    ms = {k: [] for k in masks}
    clocks = ClockSampler(0)
    clocks.start()
    for _ in range(args.reps):
        for k, m in masks.items():
            eng.set_schedule(ts, coef, 3.5, guided=m)
            eng.latents.copy_(lat0)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                eng.step()
            e1.record()
            torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1) / args.steps)
    clk = clocks.stop()
    assert eng.graph is main_graph and cond.graph is not None

    # one whole window with the example interval, and one guided at every step
    window = {}
    for k, m in (("interval", guided_steps(ts, interval)), ("every_step", None)):
        eng.set_schedule(ts, coef, 3.5, guided=m)
        eng.latents.copy_(lat0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            eng.step()
        e1.record()
        torch.cuda.synchronize()
        window[k] = (e0.elapsed_time(e1), eng.latents.clone(), n if m is None else sum(m))
    moved = float((window["interval"][1] - window["every_step"][1]).norm() / window["every_step"][1].norm())

    med = {k: statistics.median(v) for k, v in ms.items()}
    res = {"workload": f"latent {args.size}x{args.size}, {args.frames} frames, fp16, DDIM 40 steps, CFG 3.5, CUDA graph",
           "ms_per_step": med, "unguided_over_guided": med["unguided"] / med["guided"], "ms_per_step_all": ms,
           "peak_mib": {"two_branch_engine": peak_main / 2 ** 20, "with_cond_only_companion": peak_both / 2 ** 20},
           "example_window": {"interval": interval, "guided_steps": window["interval"][2], "steps": n,
                              "ms": window["interval"][0], "ms_every_step_guided": window["every_step"][0],
                              "final_latents_rel_l2_vs_every_step_guided": moved,
                              "finite": bool(torch.isfinite(window["interval"][1]).all())},
           "card": card(), "sm_mhz_median": clk.get("sm_mhz"), "clock_reasons": clk.get("reasons")}
    line = json.dumps(res)
    print(line, flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
