"""Deterministic synthetic weights and inputs for the denoising hot path (SURVEY.md 8d).

There is no network, so neither SD-1.5 / AnimateDiff / net.pth weights nor real audio/image
features exist here.  Everything is drawn from seeded CPU generators so that the oracle, the
golden-fixture script, the parity tests and bench.py all see bit-identical tensors.

Weight init (not torch's default): every tensor gets its own generator seeded from a hash of its
key, so any subset can be regenerated independently.
  weights  ~ N(0, 1/fan_in)        (keeps q.k/sqrt(d) ~ N(0,1): softmaxes are not near-uniform)
  zero_w   ~ N(0, 1/fan_in) * 0.5  (the reference zero-initialises these; de-zeroed so the audio and
                                    temporal branches are visible to parity, SURVEY.md 8c)
  biases   ~ N(0, 0.05);  norm weight ~ 1 + N(0, 0.1);  norm bias ~ N(0, 0.1)
  pe       = the sinusoid table of motion_module.py:435-445
"""
from __future__ import annotations

import hashlib
from typing import Dict, List, Optional

import torch

from .spec import UNetConfig, param_spec, param_spec_2d, reader_bank_order, sinusoid_pe


def _gen(seed: int, key: str) -> torch.Generator:
    h = hashlib.sha256(f"{seed}:{key}".encode()).digest()
    return torch.Generator(device="cpu").manual_seed(int.from_bytes(h[:7], "little"))


def synth_state_dict(cfg: UNetConfig, seed: int = 0, dtype=torch.float32,
                     only_prefix: Optional[str] = None, spec=None) -> Dict[str, torch.Tensor]:
    sd: Dict[str, torch.Tensor] = {}
    for key, shape, kind in (param_spec(cfg) if spec is None else spec):
        if only_prefix is not None and not key.startswith(only_prefix):
            continue
        g = _gen(seed, key)
        if kind == "pe":
            t = sinusoid_pe(shape[1], shape[2])
        elif kind in ("w", "zero_w"):
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            t = torch.randn(shape, generator=g) * (fan_in ** -0.5)
            if kind == "zero_w":
                t = t * 0.5
        elif kind == "b":
            t = torch.randn(shape, generator=g) * 0.05
        elif kind == "norm_w":
            t = 1.0 + torch.randn(shape, generator=g) * 0.1
        elif kind == "norm_b":
            t = torch.randn(shape, generator=g) * 0.1
        else:
            raise ValueError(kind)
        sd[key] = t.to(dtype)
    return sd


def synth_state_dict_device(cfg: UNetConfig, device, seed: int = 0, spec=None) -> Dict[str, torch.Tensor]:
    """Same distributions as synth_state_dict but drawn directly on `device` from one seeded stream (about a
    second instead of ~15 s per process on the host).  Used by bench.py, where only "random-init weights of the
    architecture" matters; the parity tests keep the per-key CPU streams so that the oracle sees identical values."""
    torch.manual_seed(seed)
    sd: Dict[str, torch.Tensor] = {}
    for key, shape, kind in (param_spec(cfg) if spec is None else spec):
        if kind == "pe":
            sd[key] = sinusoid_pe(shape[1], shape[2]).to(device)
        elif kind in ("w", "zero_w"):
            fan_in = 1
            for s_ in shape[1:]:
                fan_in *= s_
            t = torch.randn(shape, device=device) * (fan_in ** -0.5)
            sd[key] = t * 0.5 if kind == "zero_w" else t
        elif kind == "b":
            sd[key] = torch.randn(shape, device=device) * 0.05
        elif kind == "norm_w":
            sd[key] = 1.0 + torch.randn(shape, device=device) * 0.1
        elif kind == "norm_b":
            sd[key] = torch.randn(shape, device=device) * 0.1
        else:
            raise ValueError(kind)
    return sd


def synth_state_dict_2d(cfg: UNetConfig, seed: int = 1, dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """Random-init weights of the ReferenceNet (SD-1.5 UNet2D, hallo/models/unet_2d_condition.py): same per-key streams
    and distributions as the denoising UNet, its own seed."""
    return synth_state_dict(cfg, seed=seed, dtype=dtype, spec=param_spec_2d(cfg))


def synth_refnet_inputs(cfg: UNetConfig, h: int, w: int, seed: int = 7, dtype=torch.float32) -> dict:
    """What FaceAnimatePipeline feeds the ReferenceNet (face_animate.py:386-395): the VAE latents of the reference image
    and the nm motion frames, repeated for the two CFG halves -> (2*(1+nm), 4, h, w); timestep 0; the (2, 4, 768)
    image tokens [uncond, cond]."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    lat = torch.randn(1 + cfg.n_motion_frames, cfg.in_channels, h, w, generator=g)
    ehs = torch.randn(2, 4, cfg.cross_attention_dim, generator=g)
    return dict(sample=lat.repeat(2, 1, 1, 1).to(dtype), timestep=0, encoder_hidden_states=ehs.to(dtype))


def synth_audio_proj_state_dict(seed: int = 2, seq_len=5, blocks=12, channels=768, intermediate_dim=512, output_dim=768,
                                context_tokens=32) -> Dict[str, torch.Tensor]:
    """Random-init weights of AudioProjModel (hallo/models/audio_proj.py:62-94), per-key seeded like the UNets."""
    din = seq_len * blocks * channels
    shapes = {"proj1.weight": (intermediate_dim, din), "proj1.bias": (intermediate_dim,),
              "proj2.weight": (intermediate_dim, intermediate_dim), "proj2.bias": (intermediate_dim,),
              "proj3.weight": (context_tokens * output_dim, intermediate_dim), "proj3.bias": (context_tokens * output_dim,),
              "norm.weight": (output_dim,), "norm.bias": (output_dim,)}
    sd = {}
    for k, shp in shapes.items():
        g = _gen(seed, "audio_proj." + k)
        if k.endswith("proj1.weight") or k.endswith("proj2.weight") or k.endswith("proj3.weight"):
            sd[k] = torch.randn(shp, generator=g) * (2.0 / shp[1]) ** 0.5          # He: ReLU layers keep unit scale
        elif k == "norm.weight":
            sd[k] = 1.0 + 0.1 * torch.randn(shp, generator=g)
        else:
            sd[k] = 0.1 * torch.randn(shp, generator=g)
    return sd


def mask_levels(h: int, w: int):
    """Token counts of the 4 mask scales (image_processor.py:156-180): latent /1,/2,/4,/8."""
    return [(h // s) * (w // s) for s in (1, 2, 4, 8)]


def synth_inputs(cfg: UNetConfig, h: int, w: int, f: int, seed: int = 42, dtype=torch.float32,
                 timestep: int = 999, motion_scale=(1.0, 1.0, 1.0)) -> dict:
    """Inputs of UNet3DConditionModel.forward exactly as FaceAnimatePipeline assembles them for CFG
    (face_animate.py:345-412): batch row 0 = uncond, row 1 = cond."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    nm = cfg.n_motion_frames
    lat = torch.randn(1, cfg.in_channels, f, h, w, generator=g)
    sample = torch.cat([lat, lat], 0)                                   # face_animate.py:398
    ehs = torch.randn(2, 4, cfg.cross_attention_dim, generator=g)       # [uncond tokens, cond tokens]
    audio_c = torch.randn(1, f, 32, cfg.audio_attention_dim, generator=g)
    audio = torch.cat([torch.zeros_like(audio_c), audio_c], 0)          # face_animate.py:377-378
    mcf_c = torch.randn(1, cfg.block_out_channels[0], f, h, w, generator=g) * 0.5
    mask_cond_fea = torch.cat([torch.zeros_like(mcf_c), mcf_c], 0)      # face_animate.py:343
    masks = {}
    for name in ("full", "face", "lip"):
        lv = []
        for L in mask_levels(h, w):
            m = torch.rand(f, L, generator=g)
            lv.append(torch.cat([m, m], 0))                             # face_animate.py:345-360
        masks[name] = lv
    # ReferenceNet bank per spatial block: rows [ref, m1..m_nm | ref, m1..m_nm] (face_animate.py:388-390)
    banks = {}
    nblk = len(cfg.block_out_channels)
    for name, C in reader_bank_order(cfg):
        if name.startswith("mid_block"):
            s = 2 ** (nblk - 1)
        elif name.startswith("down_blocks"):
            s = 2 ** int(name.split(".")[1])
        else:
            s = 2 ** (nblk - 1 - int(name.split(".")[1]))
        L = (h // s) * (w // s)
        # the two CFG halves see different ReferenceNet conditioning, so their banks differ in general
        bank = torch.randn(2 * (1 + nm), L, C, generator=_gen(seed, "bank:" + name))
        banks[name] = bank.to(torch.float16)                            # update() casts to fp16 (Q4)
    out = dict(sample=sample.to(dtype), timestep=timestep, encoder_hidden_states=ehs.to(dtype),
               audio_embedding=audio.to(dtype), mask_cond_fea=mask_cond_fea.to(dtype),
               full_mask=[m.to(dtype) for m in masks["full"]], face_mask=[m.to(dtype) for m in masks["face"]],
               lip_mask=[m.to(dtype) for m in masks["lip"]], motion_scale=list(motion_scale), banks=banks)
    return out


def host_threads() -> int:
    """Usable host cores: the scheduler affinity mask (cgroup-limited boxes report the whole host in cpu_count)."""
    import os
    try:
        n = len(os.sched_getaffinity(0))
    except Exception:
        n = os.cpu_count() or 1
    try:
        q = open("/sys/fs/cgroup/cpu.max").read().split()
        if q[0] != "max":
            n = min(n, max(1, int(int(q[0]) / int(q[1]))))
    except Exception:
        pass
    return max(1, n)


def golden_sample_index(numel: int) -> torch.Tensor:
    """Fixed, seeded half of the element indices of a flattened output: golden vectors too large to store whole keep
    these elements only (tests/golden, written by oracle/make_golden.py)."""
    g = torch.Generator().manual_seed(0)
    return torch.randperm(numel, generator=g)[: numel // 2].sort().values
