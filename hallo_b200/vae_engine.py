"""Kernel-plan executor for the SD-1.5 VAE (AutoencoderKL): encode and decode on the library's sm_90a kernels.

The pipeline runs the VAE in every window (face_animate.py `decode_latents` on all frames, the motion-frame encode in
`__call__`, the source-image encode in `prepare_static`); at 512 x 512 a 16-frame decode is 40 TFLOP, the size of most
of a UNet forward.  This executes the module of hallo_b200/models/vae.py -- diffusers' AutoencoderKL, the same state
dict -- as a flat sequence of kernels over channels-last token matrices [n*H*W, C]:

  ResNet block   GroupNorm+SiLU -> 3x3 conv -> GroupNorm+SiLU -> 3x3 conv with the input (or its 1x1 shortcut
                 GEMM) as the fused residual (DenoiseEngine._resnet without the time-embedding bias)
  mid attention  GroupNorm -> fused QKV GEMM (N = 1536) -> single-head attention, head_dim 512 -> to_out GEMM with
                 the residual
  downsampler    phase split -> stride-2 conv with the (0, 1) zero pad (conv3x3 mode 3)
  upsampler      nearest 2x -> 3x3 conv
  stems          im2col_affine -> GEMM: the encoder's RGB conv_in, and the decoder's conv_in with post_quant_conv
                 applied per gathered pixel (it cannot be folded into conv_in: the zero pad comes after its bias)
  heads          GroupNorm+SiLU -> 3x3 conv padded to 8 output rows -> tokens_to_bcfhw.  The encoder's conv_out and
                 quant_conv fold exactly into one conv that yields the 4 mean channels (the pipeline never reads the
                 log-variance).

Frames are independent, so a call of any length runs in chunks of `n` frames.  No GEMM or conv of the plan splits its
K loop (split_k=False): a frame's output is then bitwise the same whatever the chunk size or the number of frames in
the call (every other kernel of the plan already works frame by frame in a fixed order).  Buffers are reused by tag;
each tag holds the largest view it has served.  Device memory at n = 8 frames (fp16 / bf16): the largest buffers are
the decoder's 256-channel stage at full resolution, 2 * 256 * H * W * n bytes each (1.07 GB at 512 x 512); three
buffers reach that size and three more half of it, about 4.8 GB in all at 512 x 512 and 10.9 GB at 768 x 768 (sum of
the buffer sizes).  A smaller n lowers it proportionally.
"""
from __future__ import annotations

import functools
from types import SimpleNamespace
from typing import Dict, Optional

import torch

from . import ops

GROUPS = 32
EPS = 1e-6
LATENT = 4
BLOCK_OUT = (128, 256, 512, 512)
LAYERS = 2


@functools.lru_cache(maxsize=1)
def sd15_vae_shapes() -> Dict[str, tuple]:
    """Key -> shape of the SD-1.5 AutoencoderKL state dict (hallo_b200.models.vae, diffusers' key grammar)."""
    from .models.vae import AutoencoderKL
    with torch.device("meta"):
        m = AutoencoderKL()
    return {k: tuple(v.shape) for k, v in m.state_dict().items()}


def has_sd15_grammar(module) -> bool:
    """True when `module` is an nn.Module whose state dict has exactly the SD-1.5 VAE keys and shapes."""
    if not isinstance(module, torch.nn.Module):
        return False
    sd = module.state_dict()
    ref = sd15_vae_shapes()
    return sd.keys() == ref.keys() and all(tuple(sd[k].shape) == s for k, s in ref.items())


def fold_quant_conv(w_out: torch.Tensor, b_out: torch.Tensor, w_q: torch.Tensor, b_q: torch.Tensor, keep: int):
    """Encoder conv_out (3x3, C -> 2*latent) followed by quant_conv (1x1, 2*latent -> 2*latent): quant_conv acts per
    pixel on the conv's output, bias included, so rows [0, keep) of their composition are one 3x3 conv
        W' = Wq[:keep] . Wout,  b' = Wq[:keep] . bout + bq[:keep]
    exactly.  Computed in the inputs' dtype (float64 in the exactness test)."""
    wq = w_q.reshape(w_q.shape[0], w_q.shape[1])[:keep]
    w = torch.einsum("oc,cikl->oikl", wq, w_out)
    b = wq @ b_out + b_q[:keep]
    return w, b


class VAEWeights:
    """Device-resident, kernel-ready copies of an SD-1.5 AutoencoderKL state dict (packed once per model load)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device, dtype):
        ref = sd15_vae_shapes()
        got = {k: tuple(v.shape) for k, v in state_dict.items()}
        if got != ref:
            missing, extra = sorted(ref.keys() - got.keys()), sorted(got.keys() - ref.keys())
            bad = sorted(k for k in ref.keys() & got.keys() if ref[k] != got[k])
            raise ValueError(f"not an SD-1.5 AutoencoderKL state dict: missing {missing[:4]}, unexpected {extra[:4]}, "
                             f"wrong shape {bad[:4]}")
        sd = state_dict
        self.device, self.dtype = device, dtype
        self.t: Dict[str, torch.Tensor] = {}

        def put(name, x, dt=None):
            self.t[name] = x.detach().to(device=device, dtype=dt or dtype).contiguous()

        def norm(name):
            put(f"{name}.w", sd[f"{name}.weight"])
            put(f"{name}.b", sd[f"{name}.bias"])

        def conv3(name):
            put(f"{name}.w", ops.pack_conv3x3_weight(sd[f"{name}.weight"]))
            put(f"{name}.b", sd[f"{name}.bias"])

        def resnet(name):
            norm(f"{name}.norm1")
            conv3(f"{name}.conv1")
            norm(f"{name}.norm2")
            conv3(f"{name}.conv2")
            if f"{name}.conv_shortcut.weight" in sd:
                w = sd[f"{name}.conv_shortcut.weight"]
                put(f"{name}.conv_shortcut.w", w.reshape(w.shape[0], -1))
                put(f"{name}.conv_shortcut.b", sd[f"{name}.conv_shortcut.bias"])

        def mid(name):
            resnet(f"{name}.resnets.0")
            a = f"{name}.attentions.0"
            norm(f"{a}.group_norm")
            put(f"{a}.qkv.w", torch.cat([sd[f"{a}.to_{x}.weight"] for x in "qkv"], 0))
            put(f"{a}.qkv.b", torch.cat([sd[f"{a}.to_{x}.bias"] for x in "qkv"], 0))
            put(f"{a}.to_out.w", sd[f"{a}.to_out.0.weight"])
            put(f"{a}.to_out.b", sd[f"{a}.to_out.0.bias"])
            resnet(f"{name}.resnets.1")

        # encoder
        put("encoder.conv_in.w", ops.pack_stem_weight(sd["encoder.conv_in.weight"]))
        put("encoder.conv_in.b", sd["encoder.conv_in.bias"])
        for i in range(len(BLOCK_OUT)):
            for j in range(LAYERS):
                resnet(f"encoder.down_blocks.{i}.resnets.{j}")
            if i < len(BLOCK_OUT) - 1:
                conv3(f"encoder.down_blocks.{i}.downsamplers.0.conv")
        mid("encoder.mid_block")
        norm("encoder.conv_norm_out")
        w, b = fold_quant_conv(sd["encoder.conv_out.weight"].double(), sd["encoder.conv_out.bias"].double(),
                               sd["quant_conv.weight"].double(), sd["quant_conv.bias"].double(), LATENT)
        put("encoder.conv_out.w", ops.pad_rows(ops.pack_conv3x3_weight(w), 8))
        put("encoder.conv_out.b", ops.pad_rows(b, 8))
        # decoder
        put("post_quant_conv.w", sd["post_quant_conv.weight"].reshape(LATENT, LATENT), torch.float32)
        put("post_quant_conv.b", sd["post_quant_conv.bias"], torch.float32)
        put("decoder.conv_in.w", ops.pack_stem_weight(sd["decoder.conv_in.weight"]))
        put("decoder.conv_in.b", sd["decoder.conv_in.bias"])
        mid("decoder.mid_block")
        for i in range(len(BLOCK_OUT)):
            for j in range(LAYERS + 1):
                resnet(f"decoder.up_blocks.{i}.resnets.{j}")
            if i < len(BLOCK_OUT) - 1:
                conv3(f"decoder.up_blocks.{i}.upsamplers.0.conv")
        norm("decoder.conv_norm_out")
        put("decoder.conv_out.w", ops.pad_rows(ops.pack_conv3x3_weight(sd["decoder.conv_out.weight"]), 8))
        put("decoder.conv_out.b", ops.pad_rows(sd["decoder.conv_out.bias"], 8))

    def __getitem__(self, k):
        return self.t[k]

    def __contains__(self, k):
        return k in self.t


class VAEEngine:
    """encode / decode of an SD-1.5 VAE for images of h x w pixels (multiples of 16), in chunks of n frames.

    Call surface of the module the pipeline uses: `encode(x).latent_dist.mean` (x [N, 3, h, w] in [-1, 1]) and
    `decode(z).sample` (z [N, 4, h/8, w/8], already divided by the scaling factor); outputs in the weights' dtype."""

    def __init__(self, weights: VAEWeights, h: int, w: int, n: int = 8):
        assert h % 16 == 0 and w % 16 == 0, "the encoder halves the image three times into even phase planes"
        self.W = weights
        self.dtype, self.dev = weights.dtype, weights.device
        self.h, self.w, self.n = h, w, n
        self._bufs: Dict[str, torch.Tensor] = {}

    # ------------------------------------------------------------------ buffers
    def buf(self, tag: str, rows: int, cols: int, dtype=None) -> torch.Tensor:
        """[rows, cols] view of the buffer `tag` (grown on demand; a tag never holds two live tensors)."""
        dtype = dtype or self.dtype
        need = rows * cols
        t = self._bufs.get(tag)
        if t is None or t.numel() < need or t.dtype != dtype:
            t = torch.empty(need, device=self.dev, dtype=dtype)
            self._bufs[tag] = t
        return t[:need].view(rows, cols)

    def _gn(self, x, name, out, n, hw, silu):
        C = x.shape[1]
        ws = self.buf("gn.ws", 1, ops.gn_workspace_floats(n, hw, GROUPS, C), torch.float32)
        return ops.groupnorm(x, self.W[f"{name}.w"], self.W[f"{name}.b"], out, ws, n_frames=n, hw=hw, groups=GROUPS,
                             eps=EPS, silu=silu)

    # ------------------------------------------------------------------ modules
    def _resnet(self, name, x, n, hh, ww, out_tag):
        W = self.W
        M, cin = x.shape
        cout = W[f"{name}.conv1.b"].shape[0]
        t1 = self.buf("rs.gn", M, cin)
        self._gn(x, f"{name}.norm1", t1, n, hh * ww, True)
        t2 = self.buf("rs.c1", M, cout)
        ops.conv3x3(t1.view(n, hh, ww, cin), W[f"{name}.conv1.w"], t2, bias=W[f"{name}.conv1.b"], split_k=False)
        t3 = self.buf("rs.gn", M, cout)
        self._gn(t2, f"{name}.norm2", t3, n, hh * ww, True)
        if f"{name}.conv_shortcut.w" in W:
            sc = self.buf("rs.sc", M, cout)
            ops.gemm(x, W[f"{name}.conv_shortcut.w"], sc, bias=W[f"{name}.conv_shortcut.b"], split_k=False)
        else:
            sc = x
        out = self.buf(out_tag, M, cout)
        ops.conv3x3(t3.view(n, hh, ww, cout), W[f"{name}.conv2.w"], out, bias=W[f"{name}.conv2.b"], residual=sc,
                    split_k=False)
        return out

    def _attention(self, name, x, n, L, out_tag):
        W = self.W
        M, C = x.shape
        t = self.buf("at.gn", M, C)
        self._gn(x, f"{name}.group_norm", t, n, L, False)
        qkv = self.buf("at.qkv", M, 3 * C)
        ops.gemm(t, W[f"{name}.qkv.w"], qkv, bias=W[f"{name}.qkv.b"], split_k=False)
        a = self.buf("at.o", M, C)
        ops.attention(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], a, heads=1, L=L)
        out = self.buf(out_tag, M, C)
        ops.gemm(a, W[f"{name}.to_out.w"], out, bias=W[f"{name}.to_out.b"], residual=x, split_k=False)
        return out

    def _mid(self, name, x, n, hh, ww):
        x = self._resnet(f"{name}.resnets.0", x, n, hh, ww, "x.b")
        x = self._attention(f"{name}.attentions.0", x, n, hh * ww, "x.a")
        return self._resnet(f"{name}.resnets.1", x, n, hh, ww, "x.b")

    def _head(self, prefix, x, n, hh, ww, channels):
        """GroupNorm+SiLU -> conv_out (8 padded rows) -> fp32 [n, channels, hh, ww]."""
        C = x.shape[1]
        t = self.buf("rs.gn", x.shape[0], C)
        self._gn(x, f"{prefix}.conv_norm_out", t, n, hh * ww, True)
        o = self.buf("head", x.shape[0], 8)
        ops.conv3x3(t.view(n, hh, ww, C), self.W[f"{prefix}.conv_out.w"], o, bias=self.W[f"{prefix}.conv_out.b"],
                    split_k=False)
        out = torch.empty(n, channels, 1, hh, ww, device=self.dev, dtype=torch.float32)
        ops.tokens_to_bcfhw(o, out)
        return out.view(n, channels, hh, ww)

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def _encode(self, x: torch.Tensor) -> torch.Tensor:
        W = self.W
        n, _, hh, ww = x.shape
        cols = self.buf("im2col", n * hh * ww, 64)
        ops.im2col_affine(x.to(device=self.dev, dtype=torch.float32).contiguous(), cols)
        h = self.buf("x.a", n * hh * ww, BLOCK_OUT[0])
        ops.gemm(cols, W["encoder.conv_in.w"], h, bias=W["encoder.conv_in.b"], split_k=False)
        for i in range(len(BLOCK_OUT)):
            for j in range(LAYERS):
                h = self._resnet(f"encoder.down_blocks.{i}.resnets.{j}", h, n, hh, ww, "x.b" if j % 2 == 0 else "x.a")
            if i < len(BLOCK_OUT) - 1:
                C = h.shape[1]
                planes = self.buf("ds.planes", n * hh * ww, C)
                ops.phase_split(h.view(n, hh, ww, C), planes.view(4 * n, hh // 2, ww // 2, C))
                hh, ww = hh // 2, ww // 2
                h = self.buf("x.a", n * hh * ww, C)
                ops.conv3x3_stride2(planes.view(4 * n, hh, ww, C), W[f"encoder.down_blocks.{i}.downsamplers.0.conv.w"],
                                    h, n=n, ho=hh, wo=ww, bias=W[f"encoder.down_blocks.{i}.downsamplers.0.conv.b"],
                                    pad_end=True, split_k=False)
        h = self._mid("encoder.mid_block", h, n, hh, ww)
        return self._head("encoder", h, n, hh, ww, LATENT)

    @torch.no_grad()
    def _decode(self, z: torch.Tensor) -> torch.Tensor:
        W = self.W
        n, _, hh, ww = z.shape
        cols = self.buf("im2col", n * hh * ww, 64)
        ops.im2col_affine(z.to(device=self.dev, dtype=torch.float32).contiguous(), cols, mat=W["post_quant_conv.w"],
                          bias=W["post_quant_conv.b"])
        h = self.buf("x.a", n * hh * ww, BLOCK_OUT[-1])
        ops.gemm(cols, W["decoder.conv_in.w"], h, bias=W["decoder.conv_in.b"], split_k=False)
        h = self._mid("decoder.mid_block", h, n, hh, ww)
        for i in range(len(BLOCK_OUT)):
            for j in range(LAYERS + 1):
                h = self._resnet(f"decoder.up_blocks.{i}.resnets.{j}", h, n, hh, ww, "x.a" if j % 2 == 0 else "x.b")
            if i < len(BLOCK_OUT) - 1:
                C = h.shape[1]
                up = self.buf("us.up", 4 * n * hh * ww, C)
                ops.upsample2x(h.view(n, hh, ww, C), up.view(n, 2 * hh, 2 * ww, C))
                hh, ww = 2 * hh, 2 * ww
                h = self.buf("x.b", n * hh * ww, C)            # the block's output is in x.a (j = 2)
                ops.conv3x3(up.view(n, hh, ww, C), W[f"decoder.up_blocks.{i}.upsamplers.0.conv.w"], h,
                            bias=W[f"decoder.up_blocks.{i}.upsamplers.0.conv.b"], split_k=False)
        return self._head("decoder", h, n, hh, ww, 3)

    def _chunked(self, fn, x):
        outs = [fn(x[i:i + self.n]) for i in range(0, x.shape[0], self.n)]
        out = outs[0] if len(outs) == 1 else torch.cat(outs)
        return out.to(self.dtype)

    # ------------------------------------------------------------------ public
    @torch.no_grad()
    def encode(self, x: torch.Tensor):
        """x [N, 3, h, w] -> SimpleNamespace(latent_dist=SimpleNamespace(mean=[N, 4, h/8, w/8])) in the weights' dtype."""
        assert x.dim() == 4 and x.shape[1] == 3 and tuple(x.shape[2:]) == (self.h, self.w), tuple(x.shape)
        mean = self._chunked(self._encode, x)
        return SimpleNamespace(latent_dist=SimpleNamespace(mean=mean))

    @torch.no_grad()
    def decode(self, z: torch.Tensor):
        """z [N, 4, h/8, w/8] -> SimpleNamespace(sample=[N, 3, h, w]) in the weights' dtype."""
        assert z.dim() == 4 and z.shape[1] == LATENT and tuple(z.shape[2:]) == (self.h // 8, self.w // 8), tuple(z.shape)
        return SimpleNamespace(sample=self._chunked(self._decode, z))


class EngineVAE:
    """The VAE call surface (`encode`, `decode`, `dtype`, `device`) over VAEWeights packed from `module`, with one
    VAEEngine per image size."""

    def __init__(self, module: torch.nn.Module, n: int = 8):
        p = next(module.parameters())
        self.device, self.dtype = p.device, p.dtype
        self.weights = VAEWeights(module.state_dict(), self.device, self.dtype)
        self.n = n
        self._engines: Dict[tuple, VAEEngine] = {}

    def engine(self, h: int, w: int) -> VAEEngine:
        eng = self._engines.get((h, w))
        if eng is None:
            eng = self._engines[(h, w)] = VAEEngine(self.weights, h, w, self.n)
        return eng

    def encode(self, x):
        return self.engine(x.shape[-2], x.shape[-1]).encode(x)

    def decode(self, z):
        return self.engine(8 * z.shape[-2], 8 * z.shape[-1]).decode(z)


def runs_on_engine(module) -> bool:
    """The pipeline's routing rule: an nn.Module with the SD-1.5 grammar, on CUDA, in fp16 or bf16."""
    if not isinstance(module, torch.nn.Module):
        return False
    p = next(module.parameters(), None)
    if p is None or p.device.type != "cuda" or p.dtype not in (torch.float16, torch.bfloat16):
        return False
    return has_sd15_grammar(module)


def version_key(module) -> Optional[tuple]:
    """Changes whenever the module's parameters are modified in place, moved or cast (cf. UNet3DConditionModel)."""
    return (id(module), tuple((p.device, p.dtype, p.data_ptr(), p._version) for p in module.parameters()))
