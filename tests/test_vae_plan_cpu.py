"""The VAE engine's host plan (hallo_b200/vae_engine.py) without a GPU: the ops wrappers are replaced by the PyTorch
stand-ins of tests/cpu_ops.py plus the stand-ins below for the entry points the VAE adds (im2col_affine, the (0, 1)
padded stride-2 conv), and the engine runs in fp32 against the module of hallo_b200/models/vae.py.  Also: the
quant_conv fold, the SD-1.5 grammar predicate and the FLOP formulas."""
import pytest
import torch
import torch.nn.functional as F

import cpu_ops
from conftest import rel_l2
from hallo_b200.synth import host_threads


def op_im2col_affine(x, out, *, mat=None, bias=None, scale=1.0):
    n, cl, h, w = x.shape
    y = scale * x.float()
    if mat is not None:
        y = torch.einsum("oc,nchw->nohw", mat.float(), y)
    if bias is not None:
        y = y + bias.float()[None, :, None, None]
    cols = F.unfold(y, 3, padding=1).view(n, cl, 9, h * w)                  # zero pad AFTER the affine map
    out.zero_()
    out[:, :9 * cl].copy_(cols.permute(0, 3, 2, 1).reshape(n * h * w, 9 * cl).to(out.dtype))
    return out


def op_conv3x3_stride2(x_planes, w_packed, out, *, n, ho, wo, bias=None, pad_end=False):
    cin = x_planes.shape[-1]
    pl = x_planes.view(4, n, ho, wo, cin)
    x = torch.empty(n, 2 * ho, 2 * wo, cin, dtype=x_planes.dtype)
    for p in range(2):
        for q in range(2):
            x[:, p::2, q::2] = pl[p * 2 + q]
    xc = x.float().permute(0, 3, 1, 2)
    w = w_packed.float().reshape(w_packed.shape[0], 3, 3, cin).permute(0, 3, 1, 2)
    y = F.conv2d(F.pad(xc, (0, 1, 0, 1)), w, stride=2) if pad_end else F.conv2d(xc, w, stride=2, padding=1)
    v = y.permute(0, 2, 3, 1).reshape(n * ho * wo, -1)
    if bias is not None:
        v = v + bias.float()
    out.copy_(v.to(out.dtype))
    return out


def _no_split(fn):
    """split_k only changes the GPU's summation order: the stand-ins ignore it."""
    return lambda *a, split_k=True, **kw: fn(*a, **kw)


def _install(monkeypatch):
    from hallo_b200 import ops
    cpu_ops.install(monkeypatch)
    monkeypatch.setattr(ops, "gemm", _no_split(cpu_ops.op_gemm))
    monkeypatch.setattr(ops, "conv3x3", _no_split(cpu_ops.op_conv3x3))
    monkeypatch.setattr(ops, "conv3x3_stride2", _no_split(op_conv3x3_stride2))
    monkeypatch.setattr(ops, "im2col_affine", op_im2col_affine)


@pytest.fixture(scope="module")
def vae():
    from hallo_b200.models.vae import AutoencoderKL
    torch.set_num_threads(host_threads())
    torch.manual_seed(0)
    m = AutoencoderKL().eval()
    with torch.no_grad():                       # non-trivial norm affines and post_quant_conv bias
        for k, p in m.named_parameters():
            if "norm" in k:
                p.add_(0.1 * torch.randn_like(p))
            if k.startswith("post_quant_conv") or k.startswith("quant_conv"):
                p.add_(0.2 * torch.randn_like(p))
    return m


@pytest.fixture(scope="module")
def weights(vae):
    from hallo_b200.vae_engine import VAEWeights
    return VAEWeights(vae.state_dict(), torch.device("cpu"), torch.float32)


@pytest.mark.parametrize("lh,lw", [(8, 8), (6, 10)])
def test_vae_decode_plan_matches_module(monkeypatch, vae, weights, lh, lw):
    from hallo_b200.vae_engine import VAEEngine
    _install(monkeypatch)
    z = torch.randn(2, 4, lh, lw, generator=torch.Generator().manual_seed(lh * lw))
    ref = vae.decode(z).sample
    out = VAEEngine(weights, 8 * lh, 8 * lw, n=2).decode(z).sample
    assert out.shape == ref.shape and out.dtype == ref.dtype
    assert rel_l2(out, ref) < 2e-4


@pytest.mark.parametrize("h,w", [(64, 64), (48, 80)])
def test_vae_encode_plan_matches_module(monkeypatch, vae, weights, h, w):
    from hallo_b200.vae_engine import VAEEngine
    _install(monkeypatch)
    x = torch.rand(3, 3, h, w, generator=torch.Generator().manual_seed(h + w)) * 2 - 1
    ref = vae.encode(x).latent_dist.mean
    out = VAEEngine(weights, h, w, n=2).encode(x).latent_dist.mean           # 3 frames in chunks of 2
    assert out.shape == ref.shape == (3, 4, h // 8, w // 8)
    assert rel_l2(out, ref) < 2e-4


def test_quant_conv_fold_is_exact_in_fp64():
    from hallo_b200.vae_engine import fold_quant_conv
    g = torch.Generator().manual_seed(1)
    w_out, b_out = torch.randn(8, 16, 3, 3, generator=g, dtype=torch.float64), torch.randn(8, generator=g, dtype=torch.float64)
    w_q, b_q = torch.randn(8, 8, 1, 1, generator=g, dtype=torch.float64), torch.randn(8, generator=g, dtype=torch.float64)
    x = torch.randn(2, 16, 7, 5, generator=g, dtype=torch.float64)
    ref = F.conv2d(F.conv2d(x, w_out, b_out, padding=1), w_q, b_q)[:, :4]
    w, b = fold_quant_conv(w_out, b_out, w_q, b_q, 4)
    got = F.conv2d(x, w, b, padding=1)
    assert float((got - ref).abs().max()) < 1e-12 * float(ref.abs().max())


def test_sd15_grammar_predicate():
    from hallo_b200.models.vae import AutoencoderKL
    from hallo_b200.vae_engine import has_sd15_grammar, runs_on_engine

    class Stub(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.enc = torch.nn.Conv2d(3, 4, 8, stride=8)

    with torch.device("meta"):
        m = AutoencoderKL()
        small = AutoencoderKL(block_out_channels=(64, 64, 64, 64))
    assert has_sd15_grammar(m)
    assert not has_sd15_grammar(Stub()) and not has_sd15_grammar(small) and not has_sd15_grammar(object())
    assert not runs_on_engine(m)                 # not on CUDA: the module is called as it is


def test_vae_weights_reject_other_state_dicts(vae):
    from hallo_b200.vae_engine import VAEWeights
    sd = dict(vae.state_dict())
    sd.pop("quant_conv.bias")
    with pytest.raises(ValueError):
        VAEWeights(sd, torch.device("cpu"), torch.float32)


@pytest.mark.parametrize("h,w", [(512, 512), (384, 640)])
def test_vae_flops_match_flop_counter(h, w):
    from torch.utils.flop_counter import FlopCounterMode
    from hallo_b200.flops import vae_decode_flops, vae_encode_flops
    from hallo_b200.models.vae import AutoencoderKL
    with torch.device("meta"):
        m = AutoencoderKL()
        x = torch.empty(1, 3, h, w)
        z = torch.empty(1, 4, h // 8, w // 8)
    with FlopCounterMode(display=False) as fc:
        m.decode(z)
    assert fc.get_total_flops() == vae_decode_flops(h, w)
    with FlopCounterMode(display=False) as fc:
        m.encode(x)
    assert fc.get_total_flops() == vae_encode_flops(h, w)
    if (h, w) == (512, 512):
        assert round(vae_decode_flops(h, w) / 1e9, 1) == 2514.5 and round(vae_encode_flops(h, w) / 1e9, 1) == 1116.7
