"""ORACLE / test infrastructure -- never imported by hallo_b200/ (the product has no CPU path).

Self-contained plain-PyTorch restatement of the reference's denoising hot path:
  UNet3DConditionModel.forward on the SHIPPED branch (train()-mode + gradient checkpointing, SURVEY Q1)
  with ReferenceAttentionControl in read mode (CFG), + the CFG combine + DDIM v-prediction update.

It exists because neither the reference checkout nor diffusers is a dependency of this project.  It is pinned
against the unmodified reference files run through oracle/compat
(tests/test_oracle_cpu.py::test_port_matches_reference_host, and the committed fixtures made by
oracle/make_golden.py).  The reference itself ships no tests / golden vectors for this path
(SURVEY.md section 4), so beyond that cross-check parity is "unpinned" by the upstream project.

Each function cites the reference lines it restates.  Layout follows the reference (b c f h w).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from hallo_b200.spec import BlockSpec, LayerSpec, ResnetSpec, UNetConfig, build_blocks

SD = Dict[str, torch.Tensor]


# ----------------------------------------------------------------------------- primitives
def linear(sd: SD, name: str, x):
    return F.linear(x, sd[f"{name}.weight"], sd.get(f"{name}.bias"))


def conv2d(sd: SD, name: str, x, stride=1, padding=1):
    return F.conv2d(x, sd[f"{name}.weight"], sd.get(f"{name}.bias"), stride=stride, padding=padding)


def inflated_conv(sd: SD, name: str, x, stride=1, padding=1):
    """InflatedConv3d: 2-D conv applied per frame (hallo/models/resnet.py:50-66)."""
    b, c, f, h, w = x.shape
    y = conv2d(sd, name, x.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w), stride, padding)
    return y.reshape(b, f, *y.shape[1:]).permute(0, 2, 1, 3, 4)


def inflated_gn(sd: SD, name: str, x, groups, eps):
    """InflatedGroupNorm: GroupNorm per frame (hallo/models/resnet.py:88-101)."""
    b, c, f, h, w = x.shape
    y = F.group_norm(x.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w), groups, sd[f"{name}.weight"],
                     sd[f"{name}.bias"], eps)
    return y.reshape(b, f, c, h, w).permute(0, 2, 1, 3, 4)


def layer_norm(sd: SD, name: str, x):
    return F.layer_norm(x, (x.shape[-1],), sd[f"{name}.weight"], sd[f"{name}.bias"], 1e-5)


USE_SDPA = False   # bench.py's CPU baseline flips this: same math through torch's fused CPU kernel, like the reference


def attention(sd: SD, name: str, x, ctx, heads):
    """diffusers Attention + AttnProcessor2_0 (SURVEY.md Appendix A): bias-free q/k/v, softmax(qk^T/sqrt d)v,
    to_out[0] with bias.  Explicit softmax form (independent of F.scaled_dot_product_attention) unless USE_SDPA."""
    q = F.linear(x, sd[f"{name}.to_q.weight"])
    k = F.linear(ctx, sd[f"{name}.to_k.weight"])
    v = F.linear(ctx, sd[f"{name}.to_v.weight"])
    B, Lq, Cq = q.shape
    d = Cq // heads

    def split(t):
        return t.reshape(t.shape[0], t.shape[1], heads, d).permute(0, 2, 1, 3)

    q, k, v = split(q), split(k), split(v)
    if USE_SDPA:
        o = F.scaled_dot_product_attention(q, k, v).permute(0, 2, 1, 3).reshape(B, Lq, Cq)
    else:
        p = torch.softmax((q @ k.transpose(-1, -2)) * (d ** -0.5), dim=-1)
        o = (p @ v).permute(0, 2, 1, 3).reshape(B, Lq, Cq)
    return linear(sd, f"{name}.to_out.0", o)


def feed_forward(sd: SD, name: str, x):
    """diffusers FeedForward(geglu): Linear(C->8C), value*gelu_erf(gate), Linear(4C->C)."""
    h = linear(sd, f"{name}.net.0.proj", x)
    a, g = h.chunk(2, dim=-1)
    return linear(sd, f"{name}.net.2", a * F.gelu(g))


def timestep_embedding(sd: SD, t: torch.Tensor, dim: int, dtype):
    """Timesteps(dim, flip_sin_to_cos=True, shift=0) + TimestepEmbedding (unet_3d.py:565-588)."""
    half = dim // 2
    freq = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
    ang = t[:, None].float() * freq[None]
    emb = torch.cat([torch.cos(ang), torch.sin(ang)], dim=-1).to(dtype)
    return linear(sd, "time_embedding.linear_2", F.silu(linear(sd, "time_embedding.linear_1", emb)))


# ----------------------------------------------------------------------------- modules
def resnet_block(sd: SD, rs: ResnetSpec, x, temb, cfg: UNetConfig):
    """ResnetBlock3D.forward (hallo/models/resnet.py:372-412)."""
    n = rs.name
    h = F.silu(inflated_gn(sd, f"{n}.norm1", x, cfg.norm_num_groups, cfg.norm_eps))
    h = inflated_conv(sd, f"{n}.conv1", h)
    h = h + linear(sd, f"{n}.time_emb_proj", F.silu(temb))[:, :, None, None, None]
    h = F.silu(inflated_gn(sd, f"{n}.norm2", h, cfg.norm_num_groups, cfg.norm_eps))
    h = inflated_conv(sd, f"{n}.conv2", h)
    if rs.has_shortcut:
        x = inflated_conv(sd, f"{n}.conv_shortcut", x, padding=0)
    return x + h


def _tokens_in(sd: SD, name: str, x, groups):
    """GN(eps 1e-6) -> 1x1 proj_in -> (b f) (h w) c   (transformer_3d.py:180-203)."""
    b, c, f, h, w = x.shape
    xf = x.permute(0, 2, 1, 3, 4).reshape(b * f, c, h, w)
    t = F.group_norm(xf, groups, sd[f"{name}.norm.weight"], sd[f"{name}.norm.bias"], 1e-6)
    t = conv2d(sd, f"{name}.proj_in", t, padding=0)
    return xf, t.permute(0, 2, 3, 1).reshape(b * f, h * w, t.shape[1])


def _tokens_out(sd: SD, name: str, t, resid, b, f, h, w):
    """(b f) L c -> NCHW -> 1x1 proj_out -> + residual -> b c f h w   (transformer_3d.py:236-253)."""
    y = t.reshape(b * f, h, w, t.shape[-1]).permute(0, 3, 1, 2)
    y = conv2d(sd, f"{name}.proj_out", y, padding=0) + resid
    return y.reshape(b, f, y.shape[1], h, w).permute(0, 2, 1, 3, 4)


def spatial_transformer(sd: SD, name: str, x, ehs, bank, cfg: UNetConfig):
    """Transformer3DModel (spatial) + hacked TemporalBasicTransformerBlock.forward in read mode with CFG
    (transformer_3d.py:147-257, mutual_self_attention.py:233-327).  Returns (x, motion_frame_features)."""
    b, c, f, h, w = x.shape
    H = cfg.heads
    resid, t = _tokens_in(sd, name, x, cfg.norm_num_groups)
    ctx = ehs.repeat_interleave(f, dim=0)                      # "b n c -> (b f) n c" (transformer_3d.py:189-192)
    tb = f"{name}.transformer_blocks.0"
    n1 = layer_norm(sd, f"{tb}.norm1", t)
    L, C = t.shape[1], t.shape[2]
    bank4 = bank.to(n1.dtype).reshape(b, -1, L, C)             # "(b s) l c -> b s l c"  (:235-252)
    # Quirk (SURVEY Q9, found by running the reference): `[:, 0].repeat(1, video_length, 1, 1)` acts on a
    # 3-D tensor (the `.unsqueeze(1)` at :241 is commented out), so it TILES over the batch axis:
    # row n of the (b f) batch gets the reference features of CFG half n % b, not n // f.
    ref = bank4[:, 0].repeat(f, 1, 1)
    motion = bank4[:, 1:]                                      # (b, nm, L, C)
    out = attention(sd, f"{tb}.attn1", n1, torch.cat([n1, ref], dim=1), H) + t      # (:253-263)
    half = (b * f) // 2                                        # uc_mask: first half = uncond rows (:158-166,264-284)
    out_uc = attention(sd, f"{tb}.attn1", n1[:half], n1[:half], H) + t[:half]
    t = torch.cat([out_uc, out[half:]], dim=0)
    t = attention(sd, f"{tb}.attn2", layer_norm(sd, f"{tb}.norm2", t), ctx, H) + t   # (:289-303)
    t = feed_forward(sd, f"{tb}.ff", layer_norm(sd, f"{tb}.norm3", t)) + t           # (:306-307)
    return _tokens_out(sd, name, t, resid, b, f, h, w), motion


def audio_transformer(sd: SD, name: str, x, audio, masks, level, motion_scale, cfg: UNetConfig):
    """Transformer3DModel (audio) + AudioTemporalBasicTransformerBlock.forward
    (transformer_3d.py:184-187, attention.py:784-907)."""
    b, c, f, h, w = x.shape
    H = cfg.heads
    resid, t = _tokens_in(sd, name, x, cfg.norm_num_groups)
    ctx = audio.reshape(b * f, audio.shape[2], audio.shape[3])     # "(bs f) margin dim"
    tb = f"{name}.transformer_blocks.0"
    t = attention(sd, f"{tb}.attn1", layer_norm(sd, f"{tb}.norm1", t), layer_norm(sd, f"{tb}.norm1", t), H) + t
    n2 = layer_norm(sd, f"{tb}.norm2", t)
    Ci = t.shape[-1]
    acc = None
    for r, (rname, mask) in enumerate(zip(("full", "face", "lip"), masks)):
        br = attention(sd, f"{tb}.attn2_{r}", n2, ctx, H) * mask[level][:, :, None]    # (:854-860)
        br = br.reshape(b * f, h, w, Ci).permute(0, 3, 1, 2)
        br = conv2d(sd, f"{tb}.zero_conv_{rname}", br, padding=0).permute(0, 2, 3, 1).reshape(b * f, h * w, Ci)
        br = motion_scale[r] * br                                                      # (:892-897)
        acc = br if acc is None else acc + br
    t = acc + t
    t = feed_forward(sd, f"{tb}.ff", layer_norm(sd, f"{tb}.norm3", t)) + t             # (:905)
    return _tokens_out(sd, name, t, resid, b, f, h, w)


def motion_module(sd: SD, name: str, x, cfg: UNetConfig):
    """VanillaTemporalModule -> TemporalTransformer3DModel -> TemporalTransformerBlock -> VersatileAttention
    (motion_module.py:174-197, 270-316, 387-423, 553-609).  x: (b, C, F, h, w), F includes motion frames."""
    b, c, Fr, h, w = x.shape
    H = cfg.heads
    tt = f"{name}.temporal_transformer"
    xf = x.permute(0, 2, 1, 3, 4).reshape(b * Fr, c, h, w)
    t = F.group_norm(xf, cfg.norm_num_groups, sd[f"{tt}.norm.weight"], sd[f"{tt}.norm.bias"], 1e-6)
    t = t.permute(0, 2, 3, 1).reshape(b * Fr, h * w, c)
    t = linear(sd, f"{tt}.proj_in", t)
    tb = f"{tt}.transformer_blocks.0"
    d = h * w
    for a in range(2):
        n = layer_norm(sd, f"{tb}.norms.{a}", t)
        n = n.reshape(b, Fr, d, c).permute(0, 2, 1, 3).reshape(b * d, Fr, c)       # "(b f) d c -> (b d) f c"
        n = n + sd[f"{tb}.attention_blocks.{a}.pos_encoder.pe"][:, :Fr].to(n.dtype)  # PE after LN (:585-586)
        o = attention(sd, f"{tb}.attention_blocks.{a}", n, n, H)
        o = o.reshape(b, d, Fr, c).permute(0, 2, 1, 3).reshape(b * Fr, d, c)
        t = o + t
    t = feed_forward(sd, f"{tb}.ff", layer_norm(sd, f"{tb}.ff_norm", t)) + t
    t = linear(sd, f"{tt}.proj_out", t)
    y = t.reshape(b * Fr, h, w, c).permute(0, 3, 1, 2) + xf
    return y.reshape(b, Fr, c, h, w).permute(0, 2, 1, 3, 4)


def cross_layer(sd: SD, l: LayerSpec, x, temb, inp, depth, cfg: UNetConfig):
    """One `resnet -> attn -> audio -> motion` layer on the shipped branch
    (unet_3d_blocks.py:692-748 / 1148-1202 / mid 436-494)."""
    x = resnet_block(sd, l.resnet, x, temb, cfg)
    x, motion = spatial_transformer(sd, l.attn, x, inp["encoder_hidden_states"], inp["banks"][l.attn], cfg)
    b, c, f, h, w = x.shape
    mf = motion.reshape(b, motion.shape[1], h, w, c).permute(0, 4, 1, 2, 3)      # "b f (d1 d2) c -> b c f d1 d2"
    nm = mf.shape[2]
    x = audio_transformer(sd, l.audio, x, inp["audio_embedding"],
                          (inp["full_mask"], inp["face_mask"], inp["lip_mask"]), depth, inp["motion_scale"], cfg)
    x = motion_module(sd, l.motion, torch.cat([mf.to(x.dtype), x], dim=2), cfg)[:, :, nm:]
    return x


@torch.no_grad()
def unet_forward(sd: SD, cfg: UNetConfig, inp: dict, taps: Optional[dict] = None) -> torch.Tensor:
    """UNet3DConditionModel.forward (hallo/models/unet_3d.py:510-715), shipped branch."""
    x = inp["sample"]
    dtype = x.dtype
    t = torch.as_tensor(inp["timestep"]).reshape(-1).expand(x.shape[0])
    temb = timestep_embedding(sd, t, cfg.block_out_channels[0], dtype)
    x = inflated_conv(sd, "conv_in", x)
    if inp.get("mask_cond_fea") is not None:
        x = x + inp["mask_cond_fea"]
    skips = [x]
    blocks = build_blocks(cfg)
    for b in blocks:
        if b.kind in ("down_x", "down"):
            for l in b.layers:
                if b.kind == "down_x":
                    x = cross_layer(sd, l, x, temb, inp, b.depth, cfg)
                else:
                    x = resnet_block(sd, l.resnet, x, temb, cfg)   # Q1b: motion module skipped (:905-915)
                skips.append(x)
            if b.downsampler:
                x = inflated_conv(sd, f"{b.downsampler}.conv", x, stride=2, padding=1)
                skips.append(x)
        elif b.kind == "mid":
            x = resnet_block(sd, b.extra_resnet, x, temb, cfg)
            l = b.layers[0]
            # mid: attn -> audio -> motion -> resnet  (unet_3d_blocks.py:436-494)
            x, motion = spatial_transformer(sd, l.attn, x, inp["encoder_hidden_states"], inp["banks"][l.attn], cfg)
            bb, c, f, h, w = x.shape
            mf = motion.reshape(bb, motion.shape[1], h, w, c).permute(0, 4, 1, 2, 3)
            nm = mf.shape[2]
            x = audio_transformer(sd, l.audio, x, inp["audio_embedding"],
                                  (inp["full_mask"], inp["face_mask"], inp["lip_mask"]), b.depth,
                                  inp["motion_scale"], cfg)
            x = motion_module(sd, l.motion, torch.cat([mf.to(x.dtype), x], dim=2), cfg)[:, :, nm:]
            x = resnet_block(sd, l.resnet, x, temb, cfg)
        else:
            for l in b.layers:
                x = torch.cat([x, skips.pop()], dim=1)
                if b.kind == "up_x":
                    x = cross_layer(sd, l, x, temb, inp, b.depth, cfg)
                else:
                    x = resnet_block(sd, l.resnet, x, temb, cfg)   # Q1b (:1376-1386)
            if b.upsampler:
                bb, c, f, h, w = x.shape
                xu = F.interpolate(x, scale_factor=[1.0, 2.0, 2.0], mode="nearest")     # resnet.py:166-183
                x = inflated_conv(sd, f"{b.upsampler}.conv", xu)
        if taps is not None:
            taps[b.name] = x.clone()
    x = F.silu(inflated_gn(sd, "conv_norm_out", x, cfg.norm_num_groups, cfg.norm_eps))
    return inflated_conv(sd, "conv_out", x)


# ----------------------------------------------------------------------------- scheduler + loop
class DDIM:
    """DDIMScheduler as configured by the reference (SURVEY.md Q7 / Appendix A): linear betas
    0.00085->0.012 over 1000 steps, zero-terminal-SNR rescale, trailing spacing, v-prediction, eta 0.
    diffusers itself is absent from the image, so this part of the oracle is restated from the published
    algorithm and is NOT cross-checked against diffusers ("parity unpinned" for the scheduler constants)."""

    def __init__(self, num_train=1000, beta_start=0.00085, beta_end=0.012):
        betas = torch.linspace(beta_start, beta_end, num_train, dtype=torch.float32)
        alphas_bar_sqrt = torch.cumprod(1.0 - betas, 0).sqrt()
        s0, sT = alphas_bar_sqrt[0].clone(), alphas_bar_sqrt[-1].clone()
        alphas_bar_sqrt = (alphas_bar_sqrt - sT) * s0 / (s0 - sT)
        alphas_bar = alphas_bar_sqrt ** 2
        alphas = torch.cat([alphas_bar[0:1], alphas_bar[1:] / alphas_bar[:-1]])
        self.alphas_cumprod = torch.cumprod(alphas, 0)         # same round trip diffusers does
        self.num_train = num_train
        self.final_alpha_cumprod = torch.tensor(1.0)

    def timesteps(self, n):
        import numpy as np
        return (np.round(np.arange(self.num_train, 0, -self.num_train / n)) - 1).astype("int64").tolist()

    def step(self, v, t, x, n_steps):
        prev = t - self.num_train // n_steps
        a_t = self.alphas_cumprod[t]
        a_p = self.alphas_cumprod[prev] if prev >= 0 else self.final_alpha_cumprod
        b_t = 1 - a_t
        x0 = (a_t ** 0.5) * x - (b_t ** 0.5) * v
        eps = (a_t ** 0.5) * v + (b_t ** 0.5) * x
        return (a_p ** 0.5) * x0 + ((1 - a_p) ** 0.5) * eps


@torch.no_grad()
def denoise_loop(sd: SD, cfg: UNetConfig, inp: dict, latents: torch.Tensor, n_steps: int, guidance: float,
                 max_steps: Optional[int] = None) -> torch.Tensor:
    """FaceAnimatePipeline.__call__ loop body (hallo/animate/face_animate.py:384-427)."""
    sch = DDIM()
    ts = sch.timesteps(n_steps)
    for i, t in enumerate(ts if max_steps is None else ts[:max_steps]):
        cur = dict(inp)
        cur["sample"] = torch.cat([latents, latents], 0)
        cur["timestep"] = t
        v = unet_forward(sd, cfg, cur)
        vu, vc = v.chunk(2)
        v = vu + guidance * (vc - vu)
        latents = sch.step(v, t, latents, n_steps).to(latents.dtype)
    return latents


# ----------------------------------------------------------------------------- ReferenceNet (SD-1.5 UNet2D, write mode)
def _resnet2d(sd: SD, rs: ResnetSpec, x, temb, cfg: UNetConfig):
    """diffusers ResnetBlock2D as used by hallo/models/unet_2d_blocks.py (time_embedding_norm="default")."""
    n = rs.name
    h = F.silu(F.group_norm(x, cfg.norm_num_groups, sd[f"{n}.norm1.weight"], sd[f"{n}.norm1.bias"], cfg.norm_eps))
    h = conv2d(sd, f"{n}.conv1", h)
    h = h + linear(sd, f"{n}.time_emb_proj", F.silu(temb))[:, :, None, None]
    h = F.silu(F.group_norm(h, cfg.norm_num_groups, sd[f"{n}.norm2.weight"], sd[f"{n}.norm2.bias"], cfg.norm_eps))
    h = conv2d(sd, f"{n}.conv2", h)
    if rs.has_shortcut:
        x = conv2d(sd, f"{n}.conv_shortcut", x, padding=0)
    return x + h


def _transformer2d_write(sd: SD, name: str, x, ehs, banks: dict, cfg: UNetConfig):
    """Transformer2DModel.forward (transformer_2d.py:245-420: GN eps 1e-6, 1x1 proj_in, NLC) around the hacked
    BasicTransformerBlock forward in WRITE mode (mutual_self_attention.py:223-232, 329-366): bank norm1(x), plain
    self-attention, image cross-attention with the tokens TILED over the batch (`.repeat(tmp, 1, 1)`, :340-346), FF."""
    n, c, h, w = x.shape
    H = cfg.heads
    t = F.group_norm(x, cfg.norm_num_groups, sd[f"{name}.norm.weight"], sd[f"{name}.norm.bias"], 1e-6)
    t = conv2d(sd, f"{name}.proj_in", t, padding=0).permute(0, 2, 3, 1).reshape(n, h * w, c)
    tb = f"{name}.transformer_blocks.0"
    n1 = layer_norm(sd, f"{tb}.norm1", t)
    banks[name] = n1.clone()
    t = attention(sd, f"{tb}.attn1", n1, n1, H) + t
    ctx = ehs.repeat(n // ehs.shape[0], 1, 1)
    t = attention(sd, f"{tb}.attn2", layer_norm(sd, f"{tb}.norm2", t), ctx, H) + t
    t = feed_forward(sd, f"{tb}.ff", layer_norm(sd, f"{tb}.norm3", t)) + t
    y = t.reshape(n, h, w, c).permute(0, 3, 1, 2)
    return conv2d(sd, f"{name}.proj_out", y, padding=0) + x


@torch.no_grad()
def reference_net_forward(sd: SD, cfg: UNetConfig, inp: dict):
    """UNet2DConditionModel.forward of the ReferenceNet (hallo/models/unet_2d_condition.py:905-1356, post_process=False)
    with ReferenceAttentionControl(mode="write") attached.  inp: sample (n, 4, h, w), timestep, encoder_hidden_states
    (2, tokens, 768).  Returns (features of the last up block, {attention block name: bank (n, L, C)})."""
    x = inp["sample"]
    t = torch.as_tensor(inp["timestep"]).reshape(-1).expand(x.shape[0])
    temb = timestep_embedding(sd, t, cfg.block_out_channels[0], x.dtype)
    ehs = inp["encoder_hidden_states"]
    banks: dict = {}
    x = conv2d(sd, "conv_in", x)
    skips = [x]
    for b in build_blocks(cfg):
        if b.kind in ("down_x", "down"):
            for l in b.layers:
                x = _resnet2d(sd, l.resnet, x, temb, cfg)
                if l.attn:
                    x = _transformer2d_write(sd, l.attn, x, ehs, banks, cfg)
                skips.append(x)
            if b.downsampler:
                x = conv2d(sd, f"{b.downsampler}.conv", x, stride=2, padding=1)
                skips.append(x)
        elif b.kind == "mid":
            x = _resnet2d(sd, b.extra_resnet, x, temb, cfg)
            x = _transformer2d_write(sd, b.layers[0].attn, x, ehs, banks, cfg)
            x = _resnet2d(sd, b.layers[0].resnet, x, temb, cfg)
        else:
            for l in b.layers:
                x = torch.cat([x, skips.pop()], dim=1)
                x = _resnet2d(sd, l.resnet, x, temb, cfg)
                if l.attn:
                    x = _transformer2d_write(sd, l.attn, x, ehs, banks, cfg)
            if b.upsampler:
                x = conv2d(sd, f"{b.upsampler}.conv", F.interpolate(x, scale_factor=2.0, mode="nearest"))
    return x, banks
