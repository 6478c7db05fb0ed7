"""ReferenceAttentionControl (hallo/models/mutual_self_attention.py:39-496) for the H100 engine.

read  mode: attaches to hallo_b200's UNet3DConditionModel; update(writer) pairs the writer's banks with the 16
            spatial transformer blocks in the reference's order (stable sort by -norm1 width over module DFS order,
            :404-453) and hands them to the engine, cast to fp16 first exactly like the reference (Q4).  The
            read-side arithmetic (KV concat, CFG handling, motion-frame hand-off; :233-327) lives in the kernels.
write mode: with hallo_b200's engine-backed ReferenceNet (models/unet_2d_condition.py) the banks are the engine's
            norm1 buffers, read directly; with any other (reference, PyTorch) ReferenceNet, `norm1(hidden_states)` of
            every BasicTransformerBlock-like module is banked through forward pre-hooks.
"""
from __future__ import annotations

from typing import Dict, List

import torch

from ..spec import reader_bank_order


def _dfs(module: torch.nn.Module) -> List[torch.nn.Module]:
    out = [module]
    for c in module.children():
        out += _dfs(c)
    return out


def _is_writer_block(m) -> bool:
    return type(m).__name__ == "BasicTransformerBlock" and hasattr(m, "norm1") and hasattr(m, "attn1")


class ReferenceAttentionControl:
    def __init__(self, unet, mode="write", do_classifier_free_guidance=False,
                 attention_auto_machine_weight=float("inf"), gn_auto_machine_weight=1.0, style_fidelity=1.0,
                 reference_attn=True, reference_adain=False, fusion_blocks="midup", batch_size=1):
        assert mode in ("read", "write")
        assert fusion_blocks in ("midup", "full")
        if mode == "read" and fusion_blocks != "full":
            raise NotImplementedError("the Hallo pipeline uses fusion_blocks='full' (face_animate.py:300-313)")
        self.unet = unet
        self.mode = mode
        self.reference_attn = reference_attn
        self.fusion_blocks = fusion_blocks
        self.do_classifier_free_guidance = do_classifier_free_guidance
        self._hooks = []
        self._writer_blocks: List[torch.nn.Module] = []
        self._engine_writer = mode == "write" and hasattr(unet, "banks") and hasattr(unet, "arch")
        if self._engine_writer:
            pass      # hallo_b200's own ReferenceNet: forward() leaves the banks in unet.banks, nothing to hook
        elif mode == "write" and reference_attn:
            blocks = [m for m in _dfs(unet) if _is_writer_block(m)]
            blocks = sorted(blocks, key=lambda x: -x.norm1.normalized_shape[0])
            for m in blocks:
                m.bank = []

                def pre(mod, args, kwargs=None):
                    hs = args[0] if args else kwargs["hidden_states"]
                    mod.bank.append(mod.norm1(hs).clone())

                self._hooks.append(m.register_forward_pre_hook(pre))
            self._writer_blocks = blocks
        if mode == "read":
            if not hasattr(unet, "set_banks"):
                raise TypeError("read mode expects hallo_b200.models.unet_3d.UNet3DConditionModel")
            unet._reader = self

    # writer-side view used by update()
    def banks_in_pairing_order(self) -> List[torch.Tensor]:
        if self._engine_writer:
            return [self.unet.banks[name] for name, _ in reader_bank_order(self.unet.arch)] if self.unet.banks else []
        return [m.bank[0] for m in self._writer_blocks if len(m.bank) > 0]

    def update(self, writer, dtype=torch.float16):
        """Copy the writer's banks into the reader, cast to `dtype` (fp16 by default, regardless of model dtype: Q4)."""
        if not self.reference_attn:
            return
        if isinstance(writer, dict):
            banks = {k: v.clone().to(dtype) for k, v in writer.items()}
        else:
            feats = writer.banks_in_pairing_order()
            order = reader_bank_order(self.unet.arch)
            assert len(feats) == len(order), (len(feats), len(order))
            banks = {}
            for (name, C), t in zip(order, feats):
                assert t.shape[-1] == C, (name, tuple(t.shape), C)
                banks[name] = t.clone().to(dtype)
        self.unet.set_banks(banks)

    def clear(self):
        if self.mode == "read":
            self.unet.set_banks({})
        elif self._engine_writer:
            self.unet.banks = {}
        else:
            # the pipeline builds a new writer per window (face_animate.py:300-313): drop this writer's pre-hooks with
            # its banks, or every window would leave 16 more hooks (and norm1 + clone calls) on the ReferenceNet
            for m in self._writer_blocks:
                m.bank.clear()
            self.remove_hooks()

    def remove_hooks(self):
        for h in self._hooks:
            h.remove()
        self._hooks = []

    def __del__(self):
        try:
            self.remove_hooks()
        except Exception:
            pass
