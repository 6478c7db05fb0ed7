"""AutoencoderKL (SD-1.5 VAE) -- the window-turnaround component of SURVEY.md 8f row 2.

The reference takes it from diffusers (`AutoencoderKL.from_pretrained`, scripts/inference.py:195; used at
hallo/animate/face_animate.py:222-246 `decode_latents` and :332-336 `vae.encode(ref).latent_dist.mean`).  diffusers
is absent from this image, so this is a restatement of the published architecture (diffusers 0.27.2
models/autoencoders/{autoencoder_kl,vae}.py, SD-1.5 config: block_out_channels (128, 256, 512, 512), 2 layers per
block, 32 norm groups, eps 1e-6, single-head mid-block attention, latent channels 4) with diffusers' state-dict key
names, so `sd-vae-ft-mse` checkpoints load with strict=True.  This module is plain PyTorch (cuDNN convolutions,
channels_last): the CPU path, and the parity reference of hallo_b200/vae_engine.py, which runs the same state dict on
the library's kernels -- FaceAnimatePipeline routes an SD-1.5 VAE on CUDA in fp16 / bf16 there, and calls this module
otherwise.  Parity: unpinned against upstream (no diffusers here); the architecture test checks the key grammar,
shapes and the encode/decode contract.
"""
from __future__ import annotations

from types import SimpleNamespace

import torch
import torch.nn.functional as F
from torch import nn


class _Resnet(nn.Module):
    def __init__(self, cin, cout, groups=32, eps=1e-6):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, cin, eps=eps)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.norm2 = nn.GroupNorm(groups, cout, eps=eps)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(cin, cout, 1) if cin != cout else None

    def forward(self, x):
        h = self.conv1(F.silu(self.norm1(x)))
        h = self.conv2(F.silu(self.norm2(h)))
        return (x if self.conv_shortcut is None else self.conv_shortcut(x)) + h


class _MidAttention(nn.Module):
    """diffusers Attention(heads=1, residual_connection=True, bias=True) with its own GroupNorm."""

    def __init__(self, c, groups=32, eps=1e-6):
        super().__init__()
        self.group_norm = nn.GroupNorm(groups, c, eps=eps)
        self.to_q, self.to_k, self.to_v = nn.Linear(c, c), nn.Linear(c, c), nn.Linear(c, c)
        self.to_out = nn.ModuleList([nn.Linear(c, c), nn.Dropout(0.0)])

    def forward(self, x):
        b, c, h, w = x.shape
        t = self.group_norm(x.reshape(b, c, h * w)).transpose(1, 2)
        q, k, v = self.to_q(t), self.to_k(t), self.to_v(t)
        o = F.scaled_dot_product_attention(q.unsqueeze(1), k.unsqueeze(1), v.unsqueeze(1)).squeeze(1)
        o = self.to_out[0](o).transpose(1, 2).reshape(b, c, h, w)
        return o + x


class _Mid(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.attentions = nn.ModuleList([_MidAttention(c)])
        self.resnets = nn.ModuleList([_Resnet(c, c), _Resnet(c, c)])

    def forward(self, x):
        return self.resnets[1](self.attentions[0](self.resnets[0](x)))


class _Sampler(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, stride=1, padding=1)


class _Down(_Sampler):
    def __init__(self, c):
        super().__init__(c)
        self.conv = nn.Conv2d(c, c, 3, stride=2, padding=0)

    def forward(self, x):
        return self.conv(F.pad(x, (0, 1, 0, 1)))          # Downsample2D(padding=0): asymmetric zero pad, stride 2


class _Up(_Sampler):
    def forward(self, x):
        return self.conv(F.interpolate(x, scale_factor=2.0, mode="nearest"))


class _Block(nn.Module):
    def __init__(self, cin, cout, n, down=False, up=False):
        super().__init__()
        self.resnets = nn.ModuleList([_Resnet(cin if i == 0 else cout, cout) for i in range(n)])
        if down:
            self.downsamplers = nn.ModuleList([_Down(cout)])
        if up:
            self.upsamplers = nn.ModuleList([_Up(cout)])

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        for s in getattr(self, "downsamplers", []):
            x = s(x)
        for s in getattr(self, "upsamplers", []):
            x = s(x)
        return x


class Encoder(nn.Module):
    def __init__(self, cin, latent, boc, layers):
        super().__init__()
        self.conv_in = nn.Conv2d(cin, boc[0], 3, padding=1)
        self.down_blocks = nn.ModuleList([_Block(boc[max(i - 1, 0)], boc[i], layers, down=i < len(boc) - 1)
                                          for i in range(len(boc))])
        self.mid_block = _Mid(boc[-1])
        self.conv_norm_out = nn.GroupNorm(32, boc[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(boc[-1], 2 * latent, 3, padding=1)

    def forward(self, x):
        x = self.conv_in(x)
        for b in self.down_blocks:
            x = b(x)
        return self.conv_out(F.silu(self.conv_norm_out(self.mid_block(x))))


class Decoder(nn.Module):
    def __init__(self, latent, cout, boc, layers):
        super().__init__()
        rev = list(reversed(boc))
        self.conv_in = nn.Conv2d(latent, rev[0], 3, padding=1)
        self.mid_block = _Mid(rev[0])
        self.up_blocks = nn.ModuleList([_Block(rev[max(i - 1, 0)], rev[i], layers + 1, up=i < len(boc) - 1)
                                        for i in range(len(boc))])
        self.conv_norm_out = nn.GroupNorm(32, rev[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(rev[-1], cout, 3, padding=1)

    def forward(self, z):
        x = self.mid_block(self.conv_in(z))
        for b in self.up_blocks:
            x = b(x)
        return self.conv_out(F.silu(self.conv_norm_out(x)))


class _Posterior:
    """DiagonalGaussianDistribution: the pipeline only reads `.mean` (face_animate.py:335)."""

    def __init__(self, moments):
        self.mean, self.logvar = moments.chunk(2, dim=1)

    def mode(self):
        return self.mean


class AutoencoderKL(nn.Module):
    def __init__(self, in_channels=3, out_channels=3, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                 latent_channels=4, scaling_factor=0.18215, **unused):
        super().__init__()
        self.config = SimpleNamespace(in_channels=in_channels, out_channels=out_channels,
                                      block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
                                      latent_channels=latent_channels, scaling_factor=scaling_factor)
        self.encoder = Encoder(in_channels, latent_channels, tuple(block_out_channels), layers_per_block)
        self.decoder = Decoder(latent_channels, out_channels, tuple(block_out_channels), layers_per_block)
        self.quant_conv = nn.Conv2d(2 * latent_channels, 2 * latent_channels, 1)
        self.post_quant_conv = nn.Conv2d(latent_channels, latent_channels, 1)

    @property
    def device(self):
        return next(self.parameters()).device

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    @classmethod
    def from_pretrained(cls, path, **kwargs):
        import json
        from pathlib import Path
        p = Path(path)
        cfg = json.load(open(p / "config.json"))
        model = cls(**{k: v for k, v in cfg.items() if not k.startswith("_")})
        st = p / "diffusion_pytorch_model.safetensors"
        if st.exists():
            from safetensors.torch import load_file
            sd = load_file(str(st), device="cpu")
        else:
            sd = torch.load(p / "diffusion_pytorch_model.bin", map_location="cpu", weights_only=True)
        model.load_state_dict(sd, strict=True)
        return model

    @torch.no_grad()
    def encode(self, x):
        x = x.contiguous(memory_format=torch.channels_last)
        return SimpleNamespace(latent_dist=_Posterior(self.quant_conv(self.encoder(x))))

    @torch.no_grad()
    def decode(self, z):
        z = z.contiguous(memory_format=torch.channels_last)
        return SimpleNamespace(sample=self.decoder(self.post_quant_conv(z)))
