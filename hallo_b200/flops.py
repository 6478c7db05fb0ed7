"""Algorithmic FLOPs of one UNet3D forward (the figure roofline.achieved uses) -- SURVEY.md 8d "formula card".

2*M*N*K per GEMM / conv, 4*Lq*Lk*C per attention (QK^T + PV, true head_dim), cond half attends 2L keys and
uncond half L keys, step-invariant K/V projections counted once per forward, elementwise / norm / softmax not
counted, skipped motion modules (Q1b) not counted.  `python -m hallo_b200.flops` prints the table."""
from __future__ import annotations

from typing import Dict

from .spec import UNetConfig, build_blocks


def unet_forward_flops(cfg: UNetConfig, h: int, w: int, f: int, b: int = 2) -> Dict[str, float]:
    nm = cfg.n_motion_frames
    B, F = b * f, f + nm
    out: Dict[str, float] = {}

    def add(k, v):
        out[k] = out.get(k, 0.0) + float(v)

    blocks = build_blocks(cfg)
    nblk = len(cfg.block_out_channels)

    def level_of(bk):
        if bk.name.startswith("mid"):
            return nblk - 1
        i = int(bk.name.split(".")[1])
        return i if bk.name.startswith("down") else nblk - 1 - i

    def resnet(rs, side):
        add("resnet convs", 2 * B * side * side * 9 * (rs.cin * rs.cout + rs.cout * rs.cout))
        if rs.has_shortcut:
            add("resnet convs", 2 * B * side * side * rs.cin * rs.cout)

    for bk in blocks:
        lv = level_of(bk)
        hh, ww = h >> lv, w >> lv
        L = hh * ww
        C = bk.channels
        if bk.extra_resnet is not None:
            resnet(bk.extra_resnet, hh)
        for l in bk.layers:
            resnet(l.resnet, hh)
            if l.attn:
                add("spatial proj in/out", 2 * (2 * B * L * C * C))
                add("spatial Q/K/V/O", 4 * (2 * B * L * C * C) + 2 * (2 * b * L * C * C))
                add("spatial self-attn SDPA", 4 * (B / 2) * L * (2 * L) * C + 4 * (B / 2) * L * L * C)
                add("image cross-attn", 2 * (2 * B * L * C * C) + 2 * (2 * b * 4 * cfg.cross_attention_dim * C) + 4 * B * L * 4 * C)
                add("spatial FF", 2 * B * L * C * 8 * C + 2 * B * L * 4 * C * C)
            if l.audio:
                Ci = l.audio_inner
                add("audio proj in/out", 2 * (2 * B * L * C * Ci))
                add("audio self Q/K/V/O", 4 * (2 * B * L * Ci * Ci))
                add("audio self-attn SDPA", 4 * B * L * L * Ci)
                add("audio 3x cross-attn", 3 * (2 * (2 * B * L * Ci * Ci) + 2 * (2 * B * 32 * cfg.audio_attention_dim * Ci)
                                              + 4 * B * L * 32 * Ci + 2 * B * L * Ci * Ci))
                add("audio FF", 2 * B * L * Ci * 8 * Ci + 2 * B * L * 4 * Ci * Ci)
            if l.motion and l.motion_executed:
                n = b * F * L
                add("motion proj in/out", 2 * (2 * n * C * C))
                add("temporal Q/K/V/O", 2 * 4 * (2 * n * C * C))
                add("temporal SDPA", 2 * 4 * b * L * F * F * C)
                add("motion FF", 2 * n * C * 8 * C + 2 * n * 4 * C * C)
        if bk.downsampler:
            add("down/up-sample convs", 2 * B * (hh // 2) * (ww // 2) * 9 * C * C)
        if bk.upsampler:
            add("down/up-sample convs", 2 * B * (2 * hh) * (2 * ww) * 9 * C * C)
    c0 = cfg.block_out_channels[0]
    add("conv_in/out", 2 * B * h * w * 9 * cfg.in_channels * c0 + 2 * B * h * w * 9 * c0 * cfg.out_channels)
    out["total"] = sum(out.values())
    return out


def _vae_resnet(hw: int, cin: int, cout: int) -> float:
    return 2.0 * hw * 9 * (cin * cout + cout * cout) + (2.0 * hw * cin * cout if cin != cout else 0.0)


def _vae_mid(hw: int, c: int) -> float:
    # two ResNet blocks + single-head attention: Q, K, V, out projections and 4 L^2 C for Q K^T + P V
    return 2 * _vae_resnet(hw, c, c) + 4 * (2.0 * hw * c * c) + 4.0 * hw * hw * c


def vae_decode_flops(h: int, w: int) -> float:
    """FLOPs of one SD-1.5 VAE decode (post_quant_conv ... conv_out) of an h x w frame: 2 M N K per conv / linear,
    4 L^2 512 for the mid-block attention.  2514.5 GFLOP at 512 x 512."""
    boc = (512, 512, 256, 128)
    hh, ww = h // 8, w // 8
    f = 2.0 * hh * ww * 4 * 4 + 2.0 * hh * ww * 9 * 4 * boc[0]
    f += _vae_mid(hh * ww, boc[0])
    cin = boc[0]
    for i, c in enumerate(boc):
        for j in range(3):
            f += _vae_resnet(hh * ww, cin if j == 0 else c, c)
        cin = c
        if i < len(boc) - 1:
            hh, ww = 2 * hh, 2 * ww
            f += 2.0 * hh * ww * 9 * c * c
    return f + 2.0 * hh * ww * 9 * boc[-1] * 3


def vae_encode_flops(h: int, w: int) -> float:
    """FLOPs of one SD-1.5 VAE encode (conv_in ... quant_conv, both moments) of an h x w frame, counted as
    vae_decode_flops counts.  1116.7 GFLOP at 512 x 512."""
    boc = (128, 256, 512, 512)
    hh, ww = h, w
    f = 2.0 * hh * ww * 9 * 3 * boc[0]
    cin = boc[0]
    for i, c in enumerate(boc):
        for j in range(2):
            f += _vae_resnet(hh * ww, cin if j == 0 else c, c)
        cin = c
        if i < len(boc) - 1:
            hh, ww = hh // 2, ww // 2
            f += 2.0 * hh * ww * 9 * c * c
    f += _vae_mid(hh * ww, boc[-1])
    return f + 2.0 * hh * ww * 9 * boc[-1] * 8 + 2.0 * hh * ww * 8 * 8


def spatial_attention_flops(L: int, C: int, frames_cond: int, frames_uncond: int) -> float:
    """K1: cond frames attend [self, ref] = 2L keys, uncond frames L keys."""
    return 4.0 * frames_cond * L * (2 * L) * C + 4.0 * frames_uncond * L * L * C


if __name__ == "__main__":
    for hw in (64, 96):
        t = unet_forward_flops(UNetConfig(), hw, hw, 16)
        print(f"latent {hw}x{hw}, b=2, f=16")
        for k, v in sorted(t.items(), key=lambda kv: -kv[1]):
            print(f"  {k:28s} {v / 1e12:8.3f} TFLOP  {100 * v / t['total']:5.1f} %")
