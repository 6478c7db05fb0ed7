"""SD-1.5 VAE on the library's kernels (hallo_b200.vae_engine) against the same module called as it is (cuDNN
convolutions, PyTorch SDPA), on one GPU, alternated in the same process.

Workloads (seeded random-init AutoencoderKL): the pipeline's per-window decode of 16 frames in chunks of 8, and an
encode of 3 frames (source image + 2 motion frames), at 512 x 512 in fp16 and at 768 x 768 in bf16.  For each it prints
one JSON line: ms per call of both paths (median over the timed rounds, CUDA events), TFLOP/s from hallo_b200.flops,
the rel-L2 distance between the two paths' outputs, and the card's name and power limit.

    python tools/prof_vae.py [--rounds 5] [--warmup 2] [--only decode512]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
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
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", default=None, help="run one workload: decode512, encode512, decode768, encode768")
    args = ap.parse_args()

    import __graft_entry__ as g
    g.build()
    from hallo_b200.flops import vae_decode_flops, vae_encode_flops
    from hallo_b200.models.vae import AutoencoderKL
    from hallo_b200.vae_engine import EngineVAE
    torch.backends.cudnn.benchmark = True
    dev = torch.device("cuda:0")
    info = card()
    torch.manual_seed(0)
    base = AutoencoderKL().eval()
    workloads = [("decode512", "decode", 512, torch.float16, 16), ("encode512", "encode", 512, torch.float16, 3),
                 ("decode768", "decode", 768, torch.bfloat16, 16), ("encode768", "encode", 768, torch.bfloat16, 3)]
    for name, kind, size, dtype, frames in workloads:
        if args.only and args.only != name:
            continue
        m = AutoencoderKL().eval()
        m.load_state_dict(base.state_dict())
        m = m.to(dev, dtype)
        eng = EngineVAE(m)
        gen = torch.Generator().manual_seed(size)
        if kind == "decode":
            x = torch.randn(frames, 4, size // 8, size // 8, generator=gen).to(dev, dtype)
            flops = frames * vae_decode_flops(size, size)

            def run(vae):                        # the pipeline's decode_latents: chunks of 8 frames
                return torch.cat([vae.decode(x[i:i + 8]).sample for i in range(0, frames, 8)])
        else:
            x = (torch.rand(frames, 3, size, size, generator=gen) * 2 - 1).to(dev, dtype)
            flops = frames * vae_encode_flops(size, size)

            def run(vae):
                return vae.encode(x).latent_dist.mean
        paths = {"engine": eng, "module": m}
        times = {k: [] for k in paths}
        with torch.no_grad():
            for _ in range(args.warmup):
                for v in paths.values():
                    run(v)
            torch.cuda.synchronize()
            for _ in range(args.rounds):
                for k, v in paths.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    run(v)
                    e1.record()
                    torch.cuda.synchronize()
                    times[k].append(e0.elapsed_time(e1))
            a, b = run(eng).float(), run(m).float()
        err = float((a - b).norm() / b.norm().clamp_min(1e-20))
        res = {"workload": name, "frames": frames, "size": size, "dtype": str(dtype).replace("torch.", ""),
               "gflop": round(flops / 1e9, 1)}
        for k in paths:
            ms = statistics.median(times[k])
            res[f"{k}_ms"] = round(ms, 2)
            res[f"{k}_tflops"] = round(flops / ms / 1e9, 1)
            res[f"{k}_ms_spread"] = [round(min(times[k]), 2), round(max(times[k]), 2)]
        res["speedup"] = round(res["module_ms"] / res["engine_ms"], 3)
        res["rel_l2_engine_vs_module"] = float(f"{err:.3e}")
        res.update(info)
        print(json.dumps(res), flush=True)
        del eng, m, paths
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
