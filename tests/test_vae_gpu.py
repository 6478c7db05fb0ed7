"""The SD-1.5 VAE on the sm_90a kernels: head_dim-512 attention, the (0, 1)-padded stride-2 conv, the 128-wide GEMM
tile, im2col_affine, and whole encodes / decodes of hallo_b200/vae_engine.py against the module of
hallo_b200/models/vae.py in fp32 on the CPU (the oracle).  Attention inputs are scaled so that the softmax is peaked
(a near-uniform softmax would hide a key-order bug); each test asserts it."""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0") if torch.cuda.is_available() else None
TOL = {torch.float16: 1e-2, torch.bfloat16: 2e-2}


@pytest.fixture(scope="module", autouse=True)
def _lib():
    import __graft_entry__ as g
    from hallo_b200.synth import host_threads
    g.build()
    torch.set_num_threads(host_threads())
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _peak(q, k):
    """Mean over queries of the largest softmax probability: q [L, d], k [L, d] (fp32)."""
    s = (q.float() @ k.float().t()) * q.shape[1] ** -0.5
    return float(torch.softmax(s, dim=-1).max(dim=-1).values.mean())


# ----------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("L,frames", [(4096, 2), (120, 3)])
def test_attention_head_dim_512(dtype, L, frames):
    from hallo_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(L + frames)
    qkv = torch.randn(frames * L, 3 * 512, generator=g)
    qkv[:, :1024] *= 1.8                                     # q, k: score std ~ 3, a peaked softmax
    qkv = qkv.to(DEV, dtype)
    q, k, v = qkv[:, :512], qkv[:, 512:1024], qkv[:, 1024:]
    out = torch.empty(frames * L, 512, device=DEV, dtype=dtype)
    ops.attention(q, k, v, out, heads=1, L=L)
    q3, k3, v3 = (t.float().reshape(frames, 1, L, 512) for t in (q, k, v))
    ref = F.scaled_dot_product_attention(q3, k3, v3).reshape(frames * L, 512)
    peak = _peak(q[:L], k[:L])
    err = rel_l2(out, ref)
    print(f"attention d512 L{L} x{frames} {dtype}: rel L2 {err:.2e}, mean row-max probability {peak:.3f}")
    assert peak > 0.05
    assert err < TOL[dtype]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_stride2_conv_end_pad(dtype):
    from hallo_b200 import ops
    n, H, W, cin, cout = 2, 34, 20, 128, 256
    g = torch.Generator(device="cpu").manual_seed(5)
    x = torch.randn(n, H, W, cin, generator=g).to(DEV, dtype)
    w = (torch.randn(cout, cin, 3, 3, generator=g) * 0.05).to(DEV, dtype)
    b = torch.randn(cout, generator=g).to(DEV, dtype)
    planes = torch.empty(4 * n, H // 2, W // 2, cin, device=DEV, dtype=dtype)
    ops.phase_split(x, planes)
    out = torch.empty(n * (H // 2) * (W // 2), cout, device=DEV, dtype=dtype)
    ops.conv3x3_stride2(planes, ops.pack_conv3x3_weight(w), out, n=n, ho=H // 2, wo=W // 2, bias=b, pad_end=True)
    ref = F.conv2d(F.pad(x.float().permute(0, 3, 1, 2), (0, 1, 0, 1)), w.float(), b.float(), stride=2)
    assert rel_l2(out, ref.permute(0, 2, 3, 1).reshape(-1, cout)) < TOL[dtype]


@pytest.mark.parametrize("N", [128, 256, 512, 1536])
@pytest.mark.parametrize("M,K", [(1000, 512), (256, 4608)])
def test_gemm_tile_128(N, M, K):
    from hallo_b200 import ops
    dtype = torch.float16
    g = torch.Generator(device="cpu").manual_seed(N + M)
    a = torch.randn(M, K, generator=g).to(DEV, dtype)
    w = (torch.randn(N, K, generator=g) * K ** -0.5).to(DEV, dtype)
    b = torch.randn(N, generator=g).to(DEV, dtype)
    r = torch.randn(M, N, generator=g).to(DEV, dtype)
    out = torch.empty(M, N, device=DEV, dtype=dtype)
    ops.gemm(a, w, out, bias=b, residual=r)
    ref = a.float() @ w.float().t() + b.float() + r.float()
    assert rel_l2(out, ref) < 5e-3


def test_im2col_affine():
    from hallo_b200 import ops
    from test_vae_plan_cpu import op_im2col_affine
    g = torch.Generator(device="cpu").manual_seed(7)
    x = torch.randn(3, 4, 6, 10, generator=g)
    mat, bias = torch.randn(4, 4, generator=g), torch.randn(4, generator=g)
    ref = op_im2col_affine(x, torch.empty(180, 64), mat=mat, bias=bias, scale=1.5)
    out = torch.empty(180, 64, device=DEV, dtype=torch.bfloat16)
    ops.im2col_affine(x.to(DEV), out, mat=mat.to(DEV), bias=bias.to(DEV), scale=1.5)
    assert rel_l2(out, ref) < 5e-3
    rgb = torch.randn(2, 3, 5, 7, generator=g)
    out = torch.empty(70, 64, device=DEV, dtype=torch.float16)
    ops.im2col_affine(rgb.to(DEV), out)
    assert rel_l2(out, op_im2col_affine(rgb, torch.empty(70, 64))) < 1e-3


# ----------------------------------------------------------------------------------------------- whole VAE
@pytest.fixture(scope="module")
def vae_cpu():
    """Seeded AutoencoderKL in fp32 on the CPU, mid-block to_q / to_k scaled so the attention is peaked."""
    from hallo_b200.models.vae import AutoencoderKL
    torch.manual_seed(0)
    m = AutoencoderKL().eval()
    with torch.no_grad():
        for part in (m.encoder, m.decoder):
            a = part.mid_block.attentions[0]
            for lin in (a.to_q, a.to_k):
                lin.weight.mul_(3.0)
                lin.bias.mul_(3.0)
    return m


def _mid_peak(module, part, run):
    """Mean row-max softmax probability of the mid-block attention of module.<part> during run()."""
    a = getattr(module, part).mid_block.attentions[0]
    seen = []

    def hook(mod, args):
        x = args[0][:1].float()
        b, c, h, w = x.shape
        t = mod.group_norm(x.reshape(b, c, h * w).to(mod.group_norm.weight.dtype)).transpose(1, 2)[0].float()
        seen.append(_peak(F.linear(t, mod.to_q.weight.float(), mod.to_q.bias.float()),
                          F.linear(t, mod.to_k.weight.float(), mod.to_k.bias.float())))
    hnd = a.register_forward_pre_hook(hook)
    try:
        out = run()
    finally:
        hnd.remove()
    return out, seen[0]


def _gpu_vae(vae_cpu, dtype):
    import copy
    return copy.deepcopy(vae_cpu).to(DEV, dtype)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("lh,lw,n", [(8, 8, 3), (12, 20, 3), (64, 64, 1)])
def test_vae_decode(vae_cpu, dtype, lh, lw, n):
    from hallo_b200 import lib
    from hallo_b200.vae_engine import EngineVAE
    z = torch.randn(n, 4, lh, lw, generator=torch.Generator().manual_seed(lh * lw + n))
    ref, peak = _mid_peak(vae_cpu, "decoder", lambda: vae_cpu.decode(z).sample)
    m = _gpu_vae(vae_cpu, dtype)
    lib.launch_count(reset=True)
    out = EngineVAE(m).decode(z.to(DEV, dtype)).sample
    torch.cuda.synchronize()
    assert lib.launch_count() > 0 and out.dtype == dtype and out.shape == ref.shape
    err = rel_l2(out, ref)
    own = rel_l2(m.decode(z.to(DEV, dtype)).sample, ref)
    print(f"decode {lh}x{lw} n{n} {dtype}: engine rel L2 {err:.2e}, module on GPU {own:.2e}, peak {peak:.3f}")
    assert peak > 0.05
    # bf16 storage: this random-init decoder amplifies rounding to ~2.5e-2 on either path (the module itself on the
    # GPU: ~3e-2), so the bound there is the module's own distance
    assert err < max(TOL[dtype], own)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("h,w", [(64, 64), (96, 160), (512, 512)])
def test_vae_encode(vae_cpu, dtype, h, w):
    from hallo_b200.vae_engine import EngineVAE
    n = 1 if h == 512 else 2
    x = torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(h + w)) * 2 - 1
    ref, peak = _mid_peak(vae_cpu, "encoder", lambda: vae_cpu.encode(x).latent_dist.mean)
    m = _gpu_vae(vae_cpu, dtype)
    out = EngineVAE(m).encode(x.to(DEV, dtype)).latent_dist.mean
    assert out.dtype == dtype and out.shape == ref.shape
    err = rel_l2(out, ref)
    own = rel_l2(m.encode(x.to(DEV, dtype)).latent_dist.mean, ref)
    print(f"encode {h}x{w} n{n} {dtype}: engine rel L2 {err:.2e}, module on GPU {own:.2e}, peak {peak:.3f}")
    assert peak > 0.05
    assert err < TOL[dtype]


def test_vae_decode_deterministic_and_chunk_invariant(vae_cpu):
    from hallo_b200.vae_engine import VAEWeights, VAEEngine
    m = _gpu_vae(vae_cpu, torch.float16)
    W = VAEWeights(m.state_dict(), DEV, torch.float16)
    z = torch.randn(8, 4, 16, 24, generator=torch.Generator().manual_seed(3)).to(DEV, torch.float16)
    e8 = VAEEngine(W, 128, 192, n=8)
    a = e8.decode(z).sample.clone()
    b = e8.decode(z).sample
    assert torch.equal(a, b)
    c = VAEEngine(W, 128, 192, n=1).decode(z).sample
    assert rel_l2(c, a) < 1e-3
    assert torch.equal(c, a)                     # no split K loops: per-frame results do not depend on the chunk


def test_pipeline_routes_sd_vae_to_the_engine(vae_cpu):
    from hallo_b200 import lib
    from hallo_b200.animate.face_animate import FaceAnimatePipeline
    from test_pipeline_gpu import StubVAE

    def pipe(vae):
        return FaceAnimatePipeline(vae=vae, reference_unet=None, denoising_unet=None, face_locator=None,
                                   image_proj=None, scheduler=None)

    lat = torch.randn(1, 4, 10, 12, 16, generator=torch.Generator().manual_seed(11)).to(DEV) * 0.18215
    p16 = pipe(_gpu_vae(vae_cpu, torch.float16))
    lib.launch_count(reset=True)
    got = p16.decode_latents(lat, to_numpy=False)
    torch.cuda.synchronize()
    n_engine = lib.launch_count()
    lib.launch_count(reset=True)
    ref = pipe(_gpu_vae(vae_cpu, torch.float32)).decode_latents(lat, to_numpy=False)          # fp32: module path
    torch.cuda.synchronize()
    n_module = lib.launch_count()
    assert n_engine > 0 and n_module == 0
    assert got.shape == ref.shape == (1, 3, 10, 96, 128) and got.dtype == torch.float32 and got.device == lat.device
    assert rel_l2(got, ref) < 1e-2
    # a parameter changed in place: repacked, and the output follows
    with torch.no_grad():
        p16.vae.decoder.conv_out.bias.add_(0.5)
    moved = p16.decode_latents(lat, to_numpy=False)
    assert float((moved - got).abs().max()) > 0.05
    stub = pipe(StubVAE().to(DEV, torch.float16))
    lib.launch_count(reset=True)
    stub.decode_latents(lat, to_numpy=False)
    torch.cuda.synchronize()
    assert lib.launch_count() == 0


def test_no_device_error():
    from hallo_b200 import lib
    torch.cuda.synchronize()
    assert lib.device_error() == 0
