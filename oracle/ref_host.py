"""ORACLE / test infrastructure -- never imported by hallo_b200/.

Hosts the UNMODIFIED reference hot-path files from a reference checkout (named by $HALLO_REFERENCE_ROOT) on CPU
through the compat shim in oracle/compat (diffusers==0.27.2 / xformers are not dependencies; SURVEY.md 8c).
oracle/make_golden.py uses it to write the fixtures under tests/golden/; the tests compare with those fixtures
and with the self-contained restatement in oracle/port.py.
"""
from __future__ import annotations

import os
import sys

import torch

REFERENCE_ROOT = os.environ.get("HALLO_REFERENCE_ROOT", "")
_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)


def available() -> bool:
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "hallo", "models"))


def _activate():
    compat = os.path.join(_HERE, "compat")
    for p in (REFERENCE_ROOT, compat):
        if p in sys.path:
            sys.path.remove(p)
    # compat first (provides `diffusers`, `xformers`), then the reference tree (provides `hallo`)
    sys.path.insert(0, REFERENCE_ROOT)
    sys.path.insert(0, compat)
    if _ROOT not in sys.path:
        sys.path.append(_ROOT)


def build_reference_unet(base_cfg=None, extra=None):
    """UNet3DConditionModel.from_config(...) on the SHIPPED branch: module left in train() mode and
    enable_gradient_checkpointing() called, exactly like scripts/inference.py:198-205, 233-234 (Q1)."""
    assert available(), "reference tree not present"
    _activate()
    from hallo.models.unet_3d import UNet3DConditionModel  # unmodified reference file
    from hallo_b200.spec import HALLO_UNET_KWARGS, SD15_UNET_CONFIG
    base = dict(SD15_UNET_CONFIG if base_cfg is None else base_cfg)
    extra = dict(HALLO_UNET_KWARGS if extra is None else extra)
    unet = UNet3DConditionModel.from_config(base, **extra)
    unet.requires_grad_(False)
    unet.enable_gradient_checkpointing()
    return unet


def attach_reader(unet, banks: dict):
    """ReferenceAttentionControl in read mode + synthetic banks (mutual_self_attention.py:300-313 usage)."""
    _activate()
    from hallo.models.attention import TemporalBasicTransformerBlock
    from hallo.models.mutual_self_attention import ReferenceAttentionControl
    reader = ReferenceAttentionControl(unet, do_classifier_free_guidance=True, mode="read", batch_size=1,
                                       fusion_blocks="full")
    n = 0
    for name, blk in unet.named_modules():
        if isinstance(blk, TemporalBasicTransformerBlock):
            attn_name = name.rsplit(".transformer_blocks", 1)[0]
            blk.bank = [banks[attn_name].clone()]
            n += 1
    assert n == len(banks), (n, len(banks))
    return reader


@torch.no_grad()
def run_reference_unet(unet, inp: dict):
    return unet(inp["sample"], torch.tensor(inp["timestep"]), encoder_hidden_states=inp["encoder_hidden_states"],
                audio_embedding=inp["audio_embedding"], mask_cond_fea=inp["mask_cond_fea"],
                full_mask=inp["full_mask"], face_mask=inp["face_mask"], lip_mask=inp["lip_mask"],
                motion_scale=inp["motion_scale"], return_dict=False)[0]


# ----------------------------------------------------------------------------- ReferenceNet (unmodified reference UNet2D)
def build_reference_unet2d(base_cfg=None):
    """hallo.models.unet_2d_condition.UNet2DConditionModel from the SD-1.5 config (scripts/inference.py:196-199 uses
    from_pretrained, which returns an eval() module; there is no dropout, so mode does not change the arithmetic)."""
    assert available(), "reference tree not present"
    _activate()
    from hallo.models.unet_2d_condition import UNet2DConditionModel  # unmodified reference file
    from hallo_b200.spec import SD15_UNET_CONFIG
    unet = UNet2DConditionModel.from_config(dict(SD15_UNET_CONFIG if base_cfg is None else base_cfg))
    unet.requires_grad_(False)
    unet.eval()
    return unet


@torch.no_grad()
def run_reference_net(unet2d, inp: dict):
    """ReferenceNet forward with the reference's own ReferenceAttentionControl(mode="write") attached
    (face_animate.py:300-306, 386-393).  Returns (sample, [bank per writer block in the control's pairing order],
    [module name per bank])."""
    _activate()
    from hallo.models.mutual_self_attention import ReferenceAttentionControl
    writer = ReferenceAttentionControl(unet2d, do_classifier_free_guidance=True, mode="write", batch_size=1,
                                       fusion_blocks="full")
    out = unet2d(inp["sample"], torch.tensor(inp["timestep"]), encoder_hidden_states=inp["encoder_hidden_states"],
                 return_dict=False)[0]
    from hallo.models.attention import BasicTransformerBlock
    mods = [(n, m) for n, m in unet2d.named_modules() if isinstance(m, BasicTransformerBlock)]
    # the control's own order: torch_dfs order (down, up, mid) stably sorted by -norm1 width (mutual_self_attention.py:371-385)
    mods = sorted(mods, key=lambda nm: -nm[1].norm1.normalized_shape[0])
    banks = [m.bank[0].clone() for _, m in mods]
    names = [n.rsplit(".transformer_blocks", 1)[0] for n, _ in mods]
    writer.clear()
    return out, banks, names
