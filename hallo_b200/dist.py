"""Frame-window sharding of one denoising window over the GPUs of a box (SURVEY.md 8e).

Everything on the path except temporal attention is independent per (CFG half, frame).  A rank owns a contiguous
frame group of EVERY CFG half (two, or three with a separate audio guidance scale):
  * spatial / audio attention, convolutions, norms, feed-forwards: rank-local, identical work on every rank (the cond
    half's 2L-key attention and the uncond half's L-key attention are split evenly -- no idle half);
  * CFG combine + DDIM update: rank-local (all halves of a frame live on the same rank) -- no exchange;
  * motion modules: frame <-> pixel ownership swap fused into the producing kernels (engine.DenoiseEngine._motion_px).
R = 1: everything local.  R in {2, 4, 8, 16}: f / R frames per rank; the token count of every level must divide by R.
"""
from __future__ import annotations

import os
from typing import List, Tuple

from .engine import Shard


# "peer": the frame <-> pixel swap is fused into the producing kernels' stores over NVLink peer memory (the product path);
# "nccl": the same swap as two all_to_all_single calls per motion module (A/B baseline and safe fallback).
# "peer" is the default: it needs no collective inside the captured graph; tests/test_multigpu_gpu.py checks both
# exchanges against the unsharded engine.
DEFAULT_EXCHANGE = "peer"


def frame_groups(n_frames: int, groups: int) -> List[Tuple[int, ...]]:
    if groups < 1 or n_frames % groups != 0:
        raise ValueError(f"{n_frames} frames do not split into {groups} equal groups")
    per = n_frames // groups
    return [tuple(range(g * per, (g + 1) * per)) for g in range(groups)]


def shard_layout(world: int, n_frames: int, branches: int = 2):
    """[(halves, frames)] per rank: every CFG half (branches = 2: uncond, cond; 3: also cond without audio), a
    contiguous frame group."""
    if branches not in (2, 3):
        raise ValueError(f"a window has 2 or 3 CFG branches, got {branches}")
    return [(tuple(range(branches)), fr) for fr in frame_groups(n_frames, world)]


def plan_shard(rank: int, world: int, n_frames: int, exchange: str = None, branches: int = 2) -> Shard:
    halves, frames = shard_layout(world, n_frames, branches)[rank]
    if world == 1:
        return Shard(halves=halves, frames=frames)
    import torch.distributed as dist
    exchange = exchange or os.environ.get("HALLO_B200_EXCHANGE", DEFAULT_EXCHANGE)
    if exchange not in ("peer", "nccl"):
        raise ValueError(f"HALLO_B200_EXCHANGE must be 'peer' or 'nccl', got {exchange!r}")
    return Shard(halves=halves, frames=frames, group=dist.group.WORLD, group_size=world, rank_in_group=rank,
                 exchange=exchange)


# ---- reference formulation of the two swaps on plain tensors (what the fused kernels / the NCCL variant implement);
# ---- exercised with gloo on CPU (tests/test_host_cpu.py) so the index algebra is checked without GPUs
def frames_to_pixels(gn_local, nb: int, fl: int, R: int, group):
    """[nb, fl, L, C] rows of this rank's frames -> [nb, R*fl, L/R, C]: this rank's pixel slice of ALL frames of the
    window, global frame order (chunk s of the all-to-all result comes from rank s)."""
    import torch
    import torch.distributed as dist
    _, _, L, C = gn_local.shape
    Lg = L // R
    send = gn_local.reshape(nb, fl, R, Lg, C).permute(2, 0, 1, 3, 4).contiguous()       # chunk d = my frames, slice d
    recv = torch.empty_like(send)
    dist.all_to_all_single(recv, send, group=group)
    return recv.permute(1, 0, 2, 3, 4).reshape(nb, R * fl, Lg, C)


def pixels_to_frames(y, nb: int, fl: int, R: int, group):
    """[nb, R*fl, L/R, C] (all frames, my pixel slice) -> [nb, fl, L, C] (my frames, all pixels)."""
    import torch
    import torch.distributed as dist
    Lg, C = y.shape[2], y.shape[3]
    send = y.reshape(nb, R, fl, Lg, C).permute(1, 0, 2, 3, 4).contiguous()               # chunk d = frames of rank d
    recv = torch.empty_like(send)
    dist.all_to_all_single(recv, send, group=group)                                      # chunk s = my frames, slice s
    return recv.permute(1, 2, 0, 3, 4).reshape(nb, fl, R * Lg, C)


def scatter_row_destination(r: int, seg: int, segs_per_dest: int, seg_stride: int, row0: int):
    """hb_row_scatter (include/hallo_b200.h) restated: (destination rank, destination row) of GEMM output row r."""
    s, q = divmod(r, seg)
    d, i = divmod(s, segs_per_dest)
    return d, i * seg_stride + row0 + q


def window_inputs_to_device(inp: dict, dev, dtype):
    """synth/bench helper: the begin_window keyword arguments of a full (unsharded) input dict, on the device."""
    return dict(encoder_hidden_states=inp["encoder_hidden_states"].to(dev, dtype),
                audio_embedding=inp["audio_embedding"].to(dev, dtype), mask_cond_fea=inp["mask_cond_fea"].to(dev, dtype),
                full_mask=[m.to(dev, dtype) for m in inp["full_mask"]], face_mask=[m.to(dev, dtype) for m in inp["face_mask"]],
                lip_mask=[m.to(dev, dtype) for m in inp["lip_mask"]], motion_scale=inp["motion_scale"],
                banks={k: v.to(dev) for k, v in inp["banks"].items()})


def sharded_vs_unsharded(eng, inp: dict, steps: int = 2, use_graph: bool = False):
    """Correctness of a sharded run (collective; call on every rank): `steps` denoising steps of the sharded engine
    from inp["sample"], the final latents gathered on rank 0 and compared with the SAME steps of an unsharded engine
    built on rank 0 from the same packed weights.  Returns rel-L2 on rank 0, None elsewhere.  The engine's window must
    already be set up (begin_window + set_schedule)."""
    import torch
    import torch.distributed as dist
    from .engine import DenoiseEngine, Shard
    sh = eng.shard
    rank, world = sh.rank_in_group, sh.group_size
    lat0 = inp["sample"][:1].float()
    eng.latents.copy_(lat0[:, :, list(sh.frames)].to(eng.dev))
    eng.reset_steps()
    cond = eng.cond_engine()                                              # guidance interval: the unguided steps' engine
    saved = eng.graph, None if cond is None else cond.graph
    if not use_graph:
        eng.graph = None
        if cond is not None:
            cond.graph = None
    for _ in range(steps):
        eng.step()
    torch.cuda.synchronize()
    eng.graph = saved[0]
    if cond is not None:
        cond.graph = saved[1]
    parts = [torch.empty_like(eng.latents) for _ in range(world)]
    dist.all_gather(parts, eng.latents.contiguous(), group=sh.group)
    noise = None
    if eng.sampler == "ancestral":                                        # each rank holds its frames' draws
        nparts = [torch.empty_like(eng.noise) for _ in range(world)]
        dist.all_gather(nparts, eng.noise, group=sh.group)
        noise = torch.cat(nparts, dim=2)
    eng.reset_steps()
    if rank != 0:
        dist.barrier(group=sh.group)
        return None
    full = torch.cat(parts, dim=2)                                        # frame groups in rank order
    ref = DenoiseEngine(eng.W, eng.h, eng.w, eng.f, Shard(halves=tuple(sh.halves), frames=tuple(range(eng.f))))
    ref.begin_window(**window_inputs_to_device(inp, eng.dev, eng.dtype))
    ref.n_steps, ref.guidance, ref.sampler = eng.n_steps, eng.guidance, eng.sampler
    ref.audio_guidance = eng.audio_guidance
    ref.guidance_rescale = eng.guidance_rescale
    ref.guided = eng.guided
    ref.t_table.copy_(eng.t_table)
    ref.coef.copy_(eng.coef)
    ref.coef_ms.copy_(eng.coef_ms)
    ref.coef_uni.copy_(eng.coef_uni)
    if noise is not None:
        ref.set_noise(noise)
    ref.latents.copy_(lat0.to(eng.dev))
    for _ in range(steps):
        ref.step()
    torch.cuda.synchronize()
    err = float((full - ref.latents).norm() / ref.latents.norm())
    ref.release()
    del ref
    torch.cuda.empty_cache()
    dist.barrier(group=sh.group)
    return err
