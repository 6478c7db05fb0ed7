"""UNet2DConditionModel -- the ReferenceNet's class surface over hallo_b200.refnet.ReferenceNetEngine.

Mirrors what scripts/inference.py and FaceAnimatePipeline touch of hallo/models/unet_2d_condition.py:
`from_pretrained(path, subfolder="unet")` (:196-199 of the script), `.to()`, `.requires_grad_()`,
`.enable_gradient_checkpointing()`, the 682-entry state dict (so `net.load_state_dict(...)` stays strict-clean), and
`forward(sample, timestep, encoder_hidden_states=, return_dict=False)` (face_animate.py:386-393).  The write-mode
ReferenceAttentionControl reads the banks straight from the engine (no module hooks, no clones).  CUDA only.
"""
from __future__ import annotations

import json
from dataclasses import dataclass
from pathlib import Path
from types import SimpleNamespace
from typing import Dict, Optional, Tuple

import torch
from torch import nn

from ..refnet import ReferenceNetEngine, ReferenceNetWeights
from ..spec import SD15_UNET_CONFIG, UNetConfig, param_spec_2d
from .unet_3d import _attach, _new_param


@dataclass
class UNet2DConditionOutput:
    sample: torch.FloatTensor


class UNet2DConditionModel(nn.Module):
    _supports_gradient_checkpointing = True

    def __init__(self, sample_size=None, in_channels=4, out_channels=4, center_input_sample=False, flip_sin_to_cos=True,
                 freq_shift=0, down_block_types=("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",),
                 mid_block_type="UNetMidBlock2DCrossAttn", up_block_types=("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3,
                 only_cross_attention=False, block_out_channels=(320, 640, 1280, 1280), layers_per_block=2,
                 downsample_padding=1, mid_block_scale_factor=1, act_fn="silu", norm_num_groups=32, norm_eps=1e-5,
                 cross_attention_dim=768, attention_head_dim=8, use_linear_projection=False, **extra_config):
        super().__init__()
        cfg_kwargs = dict(locals())
        for k in ("self", "__class__", "extra_config", "cfg_kwargs"):
            cfg_kwargs.pop(k, None)
        if tuple(down_block_types) != ("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",) or \
                tuple(up_block_types) != ("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3 or \
                mid_block_type != "UNetMidBlock2DCrossAttn" or use_linear_projection or only_cross_attention or \
                act_fn != "silu" or not flip_sin_to_cos or freq_shift != 0 or in_channels != 4:
            raise NotImplementedError("hallo_b200 implements the SD-1.5 ReferenceNet configuration the reference ships")
        self.config = SimpleNamespace(**cfg_kwargs, **extra_config)
        self.in_channels = in_channels
        self.arch = UNetConfig(in_channels=in_channels, out_channels=out_channels,
                               block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
                               heads=attention_head_dim if isinstance(attention_head_dim, int) else attention_head_dim[0],
                               cross_attention_dim=cross_attention_dim, norm_num_groups=norm_num_groups, norm_eps=norm_eps)
        g = torch.Generator().manual_seed(1)
        for key, shape, kind in param_spec_2d(self.arch):
            t = _new_param(shape, kind, g)
            _attach(self, key, t, buffer=False)
        self.gradient_checkpointing = False
        self._packed: Optional[ReferenceNetWeights] = None
        self._packed_version = None
        self._engines: Dict[Tuple, ReferenceNetEngine] = {}
        self.banks: Dict[str, torch.Tensor] = {}          # written by forward(): {attn block name: (n, L, C)}

    @property
    def device(self):
        return next(self.parameters()).device

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    def enable_gradient_checkpointing(self):
        self.gradient_checkpointing = True                 # API parity (scripts/inference.py:233); no effect at inference

    @classmethod
    def from_config(cls, config: dict, **kwargs):
        cfg = {k: v for k, v in dict(config).items() if not k.startswith("_")}
        cfg.update(kwargs)
        return cls(**cfg)

    @classmethod
    def from_pretrained(cls, pretrained_model_path, subfolder=None, **kwargs):
        """diffusers-style loader used at scripts/inference.py:196-199: <path>/<subfolder>/config.json + weights."""
        p = Path(pretrained_model_path)
        if subfolder is not None:
            p = p / subfolder
        cfg = json.load(open(p / "config.json"))
        for k in ("_class_name", "_diffusers_version"):
            cfg.pop(k, None)
        model = cls.from_config(cfg)
        st = p / "diffusion_pytorch_model.safetensors"
        if st.exists():
            from safetensors.torch import load_file
            sd = load_file(str(st), device="cpu")
        elif (p / "diffusion_pytorch_model.bin").exists():
            sd = torch.load(p / "diffusion_pytorch_model.bin", map_location="cpu", weights_only=True)
        else:
            raise FileNotFoundError(f"no weights file found in {p}")
        # the SD-1.5 checkpoint carries conv_norm_out / conv_out; the reference's class drops them (:683-686)
        sd = {k: v for k, v in sd.items() if not k.startswith(("conv_norm_out.", "conv_out."))}
        model.load_state_dict(sd, strict=True)
        return model

    def _weights(self) -> ReferenceNetWeights:
        ver = (self.device, self.dtype, tuple(p._version for p in self.parameters()))
        if self._packed is None or self._packed_version != ver:
            if self.device.type != "cuda":
                raise RuntimeError("hallo_b200.UNet2DConditionModel runs on CUDA (sm_90a) only; there is no CPU path")
            self._packed = ReferenceNetWeights(self.state_dict(), self.arch, self.device, self.dtype)
            self._packed_version = ver
            self._engines.clear()
        return self._packed

    def forward(self, sample, timestep, encoder_hidden_states, cond_tensor=None, return_dict: bool = True,
                post_process: bool = False, **unused):
        if cond_tensor is not None or post_process:
            raise NotImplementedError("the pipeline calls the ReferenceNet without cond_tensor / post_process")
        if any(v is not None for v in unused.values()):
            raise NotImplementedError(f"not used by the Hallo pipeline: {sorted(k for k, v in unused.items() if v is not None)}")
        n, _, h, w = sample.shape
        W = self._weights()
        eng = self._engines.get((n, h, w))
        if eng is None:
            eng = self._engines[(n, h, w)] = ReferenceNetEngine(W, h, w, n)
        out, banks = eng.run(sample, timestep, encoder_hidden_states)
        self.banks = banks
        out = out.to(sample.dtype)
        if not return_dict:
            return (out,)
        return UNet2DConditionOutput(sample=out)
