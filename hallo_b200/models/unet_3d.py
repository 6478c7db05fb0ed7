"""UNet3DConditionModel -- the reference's class surface over the sm_90a engine.

Mirrors hallo/models/unet_3d.py (UNet3DConditionModel.__init__ :121-361, .forward :510-715,
.from_pretrained_2d :717-839): same constructor keywords, the same 1946-entry state dict (so the
released net.pth loads with strict=True, scripts/inference.py:244-250), the same forward signature
and outputs.  There are no sub-module forwards: forward() hands the tensors to
hallo_b200.engine.DenoiseEngine, which runs the pre-planned CUDA kernels.  CUDA only -- calling
forward() without a GPU / without the built extension raises (north_star: no CPU fallback).
"""
from __future__ import annotations

import json
from dataclasses import dataclass
from pathlib import Path
from types import SimpleNamespace
from typing import Dict, Optional, Tuple, Union

import torch
from torch import nn

from ..engine import DenoiseEngine, PackedWeights, Shard
from ..spec import HALLO_UNET_KWARGS, SD15_UNET_CONFIG, UNetConfig, param_spec, reader_bank_order, sinusoid_pe


@dataclass
class UNet3DConditionOutput:
    sample: torch.FloatTensor


class _Node(nn.Module):
    """Pure parameter container; the tree only exists to reproduce the reference's state-dict keys."""


# Construction target of the parameter tensors.  Default: initialised fp32 tensors on the host (what `from_config` of the
# reference produces).  `with empty_weights(device, dtype):` creates them uninitialised, directly on the device, for callers
# that load a state dict right after (bench.py: 8 ranks x 1.5 G parameters would otherwise be drawn and held on the host).
_INIT = {"device": None, "dtype": None, "empty": False}


class empty_weights:
    def __init__(self, device, dtype):
        self.new = {"device": device, "dtype": dtype, "empty": True}

    def __enter__(self):
        self.old = dict(_INIT)
        _INIT.update(self.new)

    def __exit__(self, *exc):
        _INIT.update(self.old)
        return False


def _new_param(shape, kind, g):
    """One parameter tensor of the given kind (param_spec): reference-like default initialisation, or uninitialised
    device storage inside `empty_weights`."""
    if _INIT["empty"]:
        return torch.empty(shape, device=_INIT["device"], dtype=_INIT["dtype"])
    if kind == "w":
        fan_in = 1
        for s_ in shape[1:]:
            fan_in *= s_
        return torch.empty(shape).uniform_(-1, 1, generator=g) * (fan_in ** -0.5)
    if kind == "norm_w":
        return torch.ones(shape)
    return torch.zeros(shape)          # zero_w (reference zero-initialises), biases, norm biases


def _attach(root: nn.Module, key: str, tensor: torch.Tensor, buffer: bool):
    parts = key.split(".")
    m = root
    for p in parts[:-1]:
        if p not in m._modules:
            m.add_module(p, _Node())
        m = m._modules[p]
    if buffer:
        m.register_buffer(parts[-1], tensor)
    else:
        m.register_parameter(parts[-1], nn.Parameter(tensor, requires_grad=False))


class UNet3DConditionModel(nn.Module):
    _supports_gradient_checkpointing = True

    def __init__(self, sample_size=None, in_channels=4, out_channels=4, flip_sin_to_cos=True, freq_shift=0,
                 down_block_types=("CrossAttnDownBlock3D", "CrossAttnDownBlock3D", "CrossAttnDownBlock3D", "DownBlock3D"),
                 mid_block_type="UNetMidBlock3DCrossAttn",
                 up_block_types=("UpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D", "CrossAttnUpBlock3D"),
                 only_cross_attention=False, block_out_channels=(320, 640, 1280, 1280), layers_per_block=2,
                 downsample_padding=1, mid_block_scale_factor=1, act_fn="silu", norm_num_groups=32, norm_eps=1e-5,
                 cross_attention_dim=768, attention_head_dim=8, dual_cross_attention=False,
                 use_linear_projection=False, class_embed_type=None, num_class_embeds=None, upcast_attention=False,
                 resnet_time_scale_shift="default", use_inflated_groupnorm=True, use_motion_module=True,
                 motion_module_resolutions=(1, 2, 4, 8), motion_module_mid_block=True,
                 motion_module_decoder_only=False, motion_module_type="Vanilla", motion_module_kwargs=None,
                 unet_use_cross_frame_attention=False, unet_use_temporal_attention=False, use_audio_module=True,
                 audio_attention_dim=768, stack_enable_blocks_name=("up", "down", "mid"),
                 stack_enable_blocks_depth=(0, 1, 2, 3), **extra_config):
        super().__init__()
        cfg_kwargs = dict(locals())
        for k in ("self", "__class__", "extra_config", "cfg_kwargs"):
            cfg_kwargs.pop(k, None)
        unsupported = []
        if tuple(down_block_types) != ("CrossAttnDownBlock3D",) * 3 + ("DownBlock3D",):
            unsupported.append("down_block_types")
        if tuple(up_block_types) != ("UpBlock3D",) + ("CrossAttnUpBlock3D",) * 3:
            unsupported.append("up_block_types")
        if not (use_motion_module and use_audio_module and motion_module_mid_block) or motion_module_decoder_only:
            unsupported.append("motion/audio module switches")
        if use_linear_projection or dual_cross_attention or class_embed_type or num_class_embeds or \
                unet_use_temporal_attention or unet_use_cross_frame_attention or act_fn != "silu" or \
                resnet_time_scale_shift != "default" or not flip_sin_to_cos or freq_shift != 0:
            unsupported.append("non-Hallo variant switches")
        if unsupported:
            raise NotImplementedError(f"hallo_b200 implements the shipped Hallo configuration only: {unsupported}")
        mm = dict(HALLO_UNET_KWARGS["motion_module_kwargs"])
        mm.update(motion_module_kwargs or {})
        self.config = SimpleNamespace(**cfg_kwargs, **extra_config)
        self.config.center_input_sample = extra_config.get("center_input_sample", False)   # Q6
        self.sample_size = sample_size
        self.in_channels = in_channels
        self.arch = UNetConfig(in_channels=in_channels, out_channels=out_channels,
                               block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
                               heads=attention_head_dim if isinstance(attention_head_dim, int) else attention_head_dim[0],
                               cross_attention_dim=cross_attention_dim, audio_attention_dim=audio_attention_dim,
                               norm_num_groups=norm_num_groups, norm_eps=norm_eps,
                               pe_max_len=mm.get("temporal_position_encoding_max_len", 32))
        g = torch.Generator().manual_seed(0)
        for key, shape, kind in param_spec(self.arch):
            if kind == "pe":
                _attach(self, key, sinusoid_pe(shape[1], shape[2]), buffer=True)
                continue
            t = _new_param(shape, kind, g)
            _attach(self, key, t, buffer=False)
        self.gradient_checkpointing = False
        self._banks: Dict[str, torch.Tensor] = {}
        self._reader = None
        self._packed: Optional[PackedWeights] = None
        self._packed_version = None
        self._engines: Dict[Tuple, DenoiseEngine] = {}
        self._window_key = None

    # ------------------------------------------------------------------ diffusers-style helpers
    @property
    def device(self):
        return next(self.parameters()).device

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    def enable_gradient_checkpointing(self):
        """Kept for API parity (scripts/inference.py:234).  On the reference this flag selects the branch
        that inference actually runs (SURVEY Q1); that branch is the only one implemented here."""
        self.gradient_checkpointing = True

    @classmethod
    def from_config(cls, config: dict, **kwargs):
        cfg = {k: v for k, v in dict(config).items() if not k.startswith("_")}
        cfg.update(kwargs)
        return cls(**cfg)

    @classmethod
    def from_pretrained_2d(cls, pretrained_model_path, motion_module_path, subfolder=None,
                           unet_additional_kwargs=None, mm_zero_proj_out=False, use_landmark=True):
        """hallo/models/unet_3d.py:717-839: SD-1.5 2D weights + AnimateDiff motion module, non-strict,
        shape-mismatched tensors keep this model's own initialisation."""
        p = Path(pretrained_model_path)
        if subfolder is not None:
            p = p / subfolder
        config_file = p / "config.json"
        if not config_file.is_file():
            raise RuntimeError(f"{config_file} does not exist or is not a file")
        cfg = json.load(open(config_file))
        for k in ("_class_name", "_diffusers_version", "down_block_types", "up_block_types", "mid_block_type"):
            cfg.pop(k, None)
        if use_landmark:
            cfg["in_channels"] = 8
            cfg["out_channels"] = 8
        model = cls.from_config(cfg, **(unet_additional_kwargs or {}))
        st = p / "diffusion_pytorch_model.safetensors"
        if st.exists():
            from safetensors.torch import load_file
            sd = load_file(str(st), device="cpu")
        elif (p / "diffusion_pytorch_model.bin").exists():
            sd = torch.load(p / "diffusion_pytorch_model.bin", map_location="cpu", weights_only=True)
        else:
            raise FileNotFoundError(f"no weights file found in {p}")
        mp = Path(motion_module_path)
        if mp.exists() and mp.is_file():
            if mp.suffix.lower() in (".pth", ".pt", ".ckpt"):
                msd = torch.load(mp, map_location="cpu", weights_only=True)
            elif mp.suffix.lower() == ".safetensors":
                from safetensors.torch import load_file
                msd = load_file(str(mp), device="cpu")
            else:
                raise RuntimeError(f"unknown file format for motion module weights: {mp.suffix}")
            if mm_zero_proj_out:
                msd = {k: v for k, v in msd.items() if "proj_out" not in k}
            sd.update(msd)
        own = model.state_dict()
        for k in list(sd):
            if k in own and sd[k].shape != own[k].shape:
                sd[k] = own[k]
        model.load_state_dict(sd, strict=False)
        return model

    # ------------------------------------------------------------------ engine plumbing
    def _weights(self) -> PackedWeights:
        ver = (self.device, self.dtype, tuple(p._version for p in self.parameters()))
        if self._packed is None or self._packed_version != ver:
            if self.device.type != "cuda":
                raise RuntimeError("hallo_b200.UNet3DConditionModel runs on CUDA (sm_90a) only; there is no CPU path")
            self._packed = PackedWeights(self.state_dict(), self.arch, self.device, self.dtype)
            self._packed_version = ver
            self._engines.clear()
        return self._packed

    def engine(self, h: int, w: int, n_frames: int, shard=None, branches: int = 2) -> DenoiseEngine:
        """The denoising engine of this window geometry.  branches = 3 (no shard given) builds an engine with the CFG
        halves (0, 1, 2) for a separate audio guidance scale; a shard brings its own halves.  Engines of the same
        geometry and frames that differ only in their halves replace each other: switching between two and three
        branches keeps one set of activation buffers alive (the three-branch set is about 1.5x the two-branch one).
        The cond-only companion that runs the unguided steps of a guidance interval belongs to its engine
        (DenoiseEngine.cond_engine), not to this cache: it lives and goes with that engine."""
        if shard is None and branches == 3:
            shard = Shard(halves=(0, 1, 2), frames=tuple(range(n_frames)))
        elif branches not in (2, 3) or (shard is not None and len(shard.halves) != branches):
            raise ValueError(f"{branches} CFG branches with shard halves {None if shard is None else shard.halves}")
        frames = tuple(range(n_frames)) if shard is None else tuple(shard.frames)
        key = (h, w, n_frames, None if shard is None else (shard.halves, shard.frames))
        W = self._weights()
        eng = self._engines.get(key)
        if eng is None:
            for k in [k for k, e in self._engines.items()
                      if k[:3] == (h, w, n_frames) and tuple(e.shard.frames) == frames and e.nb != branches]:
                old = self._engines.pop(k)
                old.release()                    # its cond-only companion (guidance_interval) goes with it
                del old
            eng = DenoiseEngine(W, h, w, n_frames, shard)
            self._engines[key] = eng
            self._window_key = None
        return eng

    def set_banks(self, banks: Dict[str, torch.Tensor]):
        """ReferenceNet features per spatial block, [(b*(1+nm)), L, C] (mutual_self_attention.py:404-453)."""
        self._banks = dict(banks)
        self._window_key = None

    def forward(self, sample, timestep, encoder_hidden_states, audio_embedding=None, class_labels=None,
                mask_cond_fea=None, attention_mask=None, full_mask=None, face_mask=None, lip_mask=None,
                motion_scale=None, down_block_additional_residuals=None, mid_block_additional_residual=None,
                return_dict: bool = True):
        if attention_mask is not None or class_labels is not None or down_block_additional_residuals is not None \
                or mid_block_additional_residual is not None:
            raise NotImplementedError("not used by the Hallo pipeline; not implemented")
        if not self._banks:
            # Q2: the reference's Transformer3DModel only works after ReferenceAttentionControl(read) is attached
            raise RuntimeError("no reference banks: attach ReferenceAttentionControl(mode='read') and update() first")
        if sample.shape[0] != 2:
            raise NotImplementedError("classifier-free-guidance batch of 2 expected (uncond, cond)")
        b, c, f, h, w = sample.shape
        if self.config.center_input_sample:
            sample = 2 * sample - 1.0
        eng = self.engine(h, w, f)
        ms = None if motion_scale is None else tuple(float(x) for x in motion_scale)
        # window constants are re-hoisted unless every input is the SAME live object at the same version: the key holds
        # strong references (an id() alone can be recycled by a new tensor after the old one is collected)
        wins = [encoder_hidden_states, audio_embedding, mask_cond_fea] + list(full_mask) + list(face_mask) + list(lip_mask)
        wkey = (wins, [None if t is None else t._version for t in wins], ms, self._banks)
        old = self._window_key
        same = old is not None and len(old[0]) == len(wins) and all(a is b for a, b in zip(old[0], wins)) \
            and old[1] == wkey[1] and old[2] == ms and old[3] is self._banks
        if not same:
            if mask_cond_fea is None:
                mask_cond_fea = torch.zeros(b, self.arch.block_out_channels[0], f, h, w, device=sample.device,
                                            dtype=sample.dtype)
            eng.begin_window(encoder_hidden_states=encoder_hidden_states, audio_embedding=audio_embedding,
                             mask_cond_fea=mask_cond_fea, full_mask=full_mask, face_mask=face_mask, lip_mask=lip_mask,
                             motion_scale=ms, banks=self._banks)
            self._window_key = wkey
        t = float(timestep) if not torch.is_tensor(timestep) else float(timestep.reshape(-1)[0])
        eng.set_timestep(t)
        out = eng.forward_only(sample.float(), step=0).to(sample.dtype)
        if not return_dict:
            return (out,)
        return UNet3DConditionOutput(sample=out)
