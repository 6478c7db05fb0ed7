"""How accurately DDIM, DPM-Solver++ 2M and UniPC (bh2, order 2) integrate the denoising ODE at a given step count,
and what a step costs.

The workload is bench.py's: random-init weights (seed 0, drawn on the device), synthetic inputs (seed 42), one
16-frame window at 512 x 512 (latent 64 x 64), CFG 3.5, fp16.  The reference solution is the mean of a 500-step DDIM
run and a 500-step DPM-Solver++ 2M run; their mutual rel-L2 distance is printed as the floor below which no
difference means anything.  Each row is the rel-L2 of the final latents against that reference and against the same
sampler's 500-step run (UniPC has none: "-"), and ms per step from CUDA events around the graph replays of that
run.  A last line gives the sensitivity of the solution to its start: the rel-L2 change of 40-step DDIM's final
latents when the initial latents move by 1e-3 (rel L2).  When that is large, this network's ODE amplifies any
perturbation, discretisation error included, and step-count differences say little.  DDIM steps from t to t - 1000 // n (diffusers' rule), which
matches the trailing timesteps only when n divides 1000: at 400 steps each step covers 2 of the 2.5 timesteps between
evaluations, so a 400-step DDIM run is not a converged solution (measured: 0.18 rel L2 from 400-step DPM-Solver++
2M, against 2.7e-3 at 500 steps).  The card's name, power limit and the median SM clock sampled during the timed
replays are printed with the table.

The weights are random-init, so this measures how accurately each sampler integrates this network's probability-flow
ODE.  It says nothing about how videos from trained weights look: perceptual quality is not measured.

    python tools/sampler_convergence.py [--ddim 10,20,25,40] [--dpm 10,15,20,25,40] [--unipc 10,15,20,25]
                                        [--ref-steps 500] [--json FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    """Name, power limit and max SM clock as nvidia-smi reports them (read-only query)."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30)
        name, power, clock = [s.strip() for s in q.stdout.strip().split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                       # noqa: BLE001 -- reported, not fatal
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unknown ({e})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ddim", default="10,20,25,40")
    ap.add_argument("--dpm", default="10,15,20,25,40")
    ap.add_argument("--unipc", default="10,15,20,25")
    ap.add_argument("--ref-steps", type=int, default=500,
                    help="reference step count; DDIM needs one that divides 1000")
    ap.add_argument("--size", type=int, default=64, help="latent side (64 = 512x512)")
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--json", default="", metavar="FILE", help="also write the results to FILE")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sampler_convergence.py needs a CUDA device (hallo_b200 has no CPU path)")

    from bench import ClockSampler
    from hallo_b200.dist import window_inputs_to_device
    from hallo_b200.engine import DenoiseEngine, PackedWeights
    from hallo_b200.scheduler import (DDIMScheduler, DPMSolverMultistepScheduler, UniPCMultistepScheduler,
                                      sampler_table_of)
    from hallo_b200.spec import UNetConfig
    from hallo_b200.synth import host_threads, synth_inputs, synth_state_dict_device
    torch.set_num_threads(host_threads())
    dev, dt, guidance = torch.device("cuda:0"), torch.float16, 3.5
    cfg = UNetConfig()
    W = PackedWeights(synth_state_dict_device(cfg, dev, seed=0), cfg, dev, dt)
    inp = synth_inputs(cfg, args.size, args.size, args.frames, seed=42)
    eng = DenoiseEngine(W, args.size, args.size, args.frames)
    eng.begin_window(**window_inputs_to_device(inp, dev, dt))
    lat0 = inp["sample"][:1].float().to(dev)
    clocks = ClockSampler(torch.cuda.current_device())

    def run(sched, n, start=lat0):
        """n graph replays from the bench's initial latents: (final latents, ms per step)."""
        sched.set_timesteps(n)
        kind, table = sampler_table_of(sched)
        eng.set_schedule(sched.timesteps.tolist(), table, guidance, kind)
        eng.latents.copy_(start)
        if eng.graph is None:
            eng.capture()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            eng.step()
        e1.record()
        torch.cuda.synchronize()
        return eng.latents.clone(), e0.elapsed_time(e1) / n

    samplers = {"DDIM": DDIMScheduler, "DPM-Solver++ 2M": DPMSolverMultistepScheduler,
                "UniPC bh2": UniPCMultistepScheduler}
    clocks.start()
    ref_ddim, ms_ref_ddim = run(DDIMScheduler(), args.ref_steps)
    ref_dpm, ms_ref_dpm = run(DPMSolverMultistepScheduler(), args.ref_steps)
    ref = 0.5 * (ref_ddim + ref_dpm)
    own_ref = {"DDIM": ref_ddim, "DPM-Solver++ 2M": ref_dpm}

    def rel(a, b):
        return float((a - b).norm() / b.norm())

    floor = rel(ref_ddim, ref_dpm)
    rows = []
    for name, steps in (("DDIM", args.ddim), ("DPM-Solver++ 2M", args.dpm), ("UniPC bh2", args.unipc)):
        for n in [int(s) for s in steps.split(",") if s]:
            lat, ms = run(samplers[name](), n)
            rows.append({"sampler": name, "steps": n, "rel_l2_vs_ref": rel(lat, ref),
                         f"rel_l2_vs_own_{args.ref_steps}": rel(lat, own_ref[name]) if name in own_ref else None,
                         "ms_per_step": ms,
                         "finite": bool(torch.isfinite(lat).all())})
    clk = clocks.stop()
    g = torch.Generator(device=dev).manual_seed(1)
    noise = torch.randn(lat0.shape, generator=g, device=dev)
    base, _ = run(DDIMScheduler(), 40)
    moved, _ = run(DDIMScheduler(), 40, lat0 + 1e-3 * lat0.norm() / noise.norm() * noise)
    sensitivity = rel(moved, base)
    res = {"card": card(), "sm_clock_during_runs": clk, "workload": f"{args.size * 8}x{args.size * 8}, {args.frames} "
           f"frames, CFG {guidance}, fp16, weights seed 0 (random init), inputs seed 42",
           "reference": f"mean of {args.ref_steps}-step DDIM and {args.ref_steps}-step DPM-Solver++ 2M",
           "floor_rel_l2": floor, "sensitivity_40_step_ddim_to_1e-3_start": sensitivity,
           "ref_ms_per_step": {"DDIM": ms_ref_ddim, "DPM-Solver++ 2M": ms_ref_dpm}, "rows": rows}
    c = res["card"]
    print(f"# {c['gpu']}, power limit {c.get('power_limit')}, median SM clock during the runs {clk.get('sm_mhz')} MHz "
          f"(max {c.get('max_sm_clock')}); {res['workload']}")
    print(f"# reference: {res['reference']}; their distance (floor) = {floor:.3e} rel L2")
    print(f"| sampler | steps | rel L2 vs reference | rel L2 vs same sampler at {args.ref_steps} | ms / step |")
    print("|---|---|---|---|---|")
    for r in rows:
        own = r[f"rel_l2_vs_own_{args.ref_steps}"]
        print(f"| {r['sampler']} | {r['steps']} | {r['rel_l2_vs_ref']:.3e} | {'-' if own is None else f'{own:.3e}'} "
              f"| {r['ms_per_step']:.1f} |")
    print(f"# sensitivity: 40-step DDIM final latents move by {sensitivity:.3e} rel L2 when the start moves by 1e-3")
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
