"""Cost and effect of guidance rescale: the bench workload (random-init weights, 512x512 = latent 64x64, 16 frames,
CFG 3.5, DDIM, 40-step schedule) stepped through its CUDA graph with guidance_rescale = 0 and = 0.7, alternated in one
process so both see the same card state.

Prints one JSON line: ms per step (median over the repetitions) for each phi and their difference, the time of the
rescale pre-pass alone (stats + reduce + apply on the step's model output, CUDA events over many launches), the rel L2
between the final latents of a whole 40-step window at phi = 0.7 and at phi = 0, the card name, its power limit and the
median SM clock sampled while timing.

    python tools/time_guidance_rescale.py [--size 64] [--frames 16] [--steps 10] [--reps 5] [--warmup 3] [--json FILE]
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
    ap.add_argument("--reps", type=int, default=5, help="repetitions per phi, alternated")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--phi", type=float, default=0.7)
    ap.add_argument("--json", default="", help="also write the result line to this file")
    args = ap.parse_args()

    import torch
    from bench import ClockSampler
    from time_audio_guidance import card
    from hallo_b200.dist import window_inputs_to_device
    from hallo_b200.engine import DenoiseEngine, PackedWeights
    from hallo_b200.scheduler import DDIMScheduler
    from hallo_b200.spec import UNetConfig
    from hallo_b200.synth import synth_inputs, synth_state_dict_device

    if not torch.cuda.is_available():
        raise SystemExit("time_guidance_rescale.py measures on a CUDA device; none is available")
    dev, dt = torch.device("cuda:0"), torch.float16
    cfg = UNetConfig()
    W = PackedWeights(synth_state_dict_device(cfg, dev, seed=0), cfg, dev, dt)
    inp = synth_inputs(cfg, args.size, args.size, args.frames, seed=42)
    win = window_inputs_to_device(inp, dev, dt)
    sch = DDIMScheduler()
    sch.set_timesteps(40)
    lat0 = inp["sample"][:1].float().to(dev)
    phis = (0.0, args.phi)

    def make(phi):
        eng = DenoiseEngine(W, args.size, args.size, args.frames)
        eng.begin_window(**win)
        eng.set_schedule(sch.timesteps.tolist(), sch.coef_table(), 3.5, guidance_rescale=phi)
        eng.latents.copy_(lat0)
        eng.capture()
        for _ in range(args.warmup):
            eng.step()
        torch.cuda.synchronize()
        return eng

    engines = {p: make(p) for p in phis}

    ms = {p: [] for p in phis}
    clocks = ClockSampler(0)
    clocks.start()
    for _ in range(args.reps):
        for p in phis:
            eng = engines[p]
            eng.latents.copy_(lat0)
            eng.step_idx.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                eng.step()
            e1.record()
            torch.cuda.synchronize()
            ms[p].append(e0.elapsed_time(e1) / args.steps)
    # the pre-pass alone, on the step's own model output (its rows are rewritten, so this runs on a copy)
    eng = engines[args.phi]
    saved = eng.model_out.clone()
    n_pre = 200
    eng._cfg_rescale(eng.model_out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n_pre):
        eng._cfg_rescale(eng.model_out)
    e1.record()
    torch.cuda.synchronize()
    pre_us = e0.elapsed_time(e1) / n_pre * 1e3
    eng.model_out.copy_(saved)
    clk = clocks.stop()

    # effect: a whole window at each phi
    final = {}
    for p in phis:
        e = engines[p]
        e.latents.copy_(lat0)
        e.step_idx.zero_()
        for _ in range(40):
            e.step()
        torch.cuda.synchronize()
        final[p] = e.latents.clone()
    moved = float((final[args.phi] - final[0.0]).norm() / final[0.0].norm())

    med = {p: statistics.median(v) for p, v in ms.items()}
    res = {"workload": f"latent {args.size}x{args.size}, {args.frames} frames, fp16, DDIM 40 steps, CFG 3.5, CUDA graph",
           "ms_per_step": {"phi=0": med[0.0], f"phi={args.phi}": med[args.phi]},
           "delta_ms_per_step": med[args.phi] - med[0.0],
           "ms_per_step_all": {"phi=0": ms[0.0], f"phi={args.phi}": ms[args.phi]},
           "rescale_prepass_us": pre_us,
           "final_latents_rel_l2_phi_vs_0": moved, "finite": bool(torch.isfinite(final[args.phi]).all()),
           "card": card(), "sm_mhz_median": clk.get("sm_mhz"), "clock_reasons": clk.get("reasons")}
    line = json.dumps(res)
    print(line, flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
