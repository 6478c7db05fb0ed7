"""AudioProjModel (hallo/models/audio_proj.py:40-124): wav2vec window (bz, f, 5, 12, 768) -> 32 context tokens
of 768 per frame (SURVEY.md A10).  36 M parameters, M = 16 rows per window -- or all windows of a clip in one call
(hallo_b200.driver, SURVEY.md 8f row 4).  Everything runs in the sm_90a kernels: three wgmma GEMMs with the ReLU
fused into the epilogue (HB_EPI_RELU) and the final LayerNorm in hallo_b200_layernorm."""
from __future__ import annotations

import torch
from torch import nn

from .. import ops


class AudioProjModel(nn.Module):
    def __init__(self, seq_len=5, blocks=12, channels=768, intermediate_dim=512, output_dim=768, context_tokens=32):
        super().__init__()
        self.seq_len, self.blocks, self.channels = seq_len, blocks, channels
        self.input_dim = seq_len * blocks * channels
        self.intermediate_dim, self.context_tokens, self.output_dim = intermediate_dim, context_tokens, output_dim
        self.proj1 = nn.Linear(self.input_dim, intermediate_dim)
        self.proj2 = nn.Linear(intermediate_dim, intermediate_dim)
        self.proj3 = nn.Linear(intermediate_dim, context_tokens * output_dim)
        self.norm = nn.LayerNorm(output_dim)

    @property
    def device(self):
        return next(self.parameters()).device

    @property
    def dtype(self):
        return next(self.parameters()).dtype

    def _linear(self, x, lin, relu=False):
        out = torch.empty(x.shape[0], lin.out_features, device=x.device, dtype=x.dtype)
        return ops.gemm(x.contiguous(), lin.weight, out, bias=lin.bias, relu=relu)

    @torch.no_grad()
    def forward(self, audio_embeds):
        bz, f = audio_embeds.shape[:2]
        x = audio_embeds.reshape(bz * f, self.input_dim)
        if x.dtype not in (torch.float16, torch.bfloat16) or not x.is_cuda:
            raise RuntimeError("hallo_b200.AudioProjModel runs in fp16/bf16 on CUDA only (no CPU path)")
        x = self._linear(x, self.proj1, relu=True)
        x = self._linear(x, self.proj2, relu=True)
        x = self._linear(x, self.proj3).reshape(bz * f * self.context_tokens, self.output_dim)
        out = torch.empty_like(x)
        ops.layernorm(x, self.norm.weight, self.norm.bias, out, eps=self.norm.eps)
        return out.reshape(bz, f, self.context_tokens, self.output_dim)
