"""GPU parity of hallo_b200_attention (wgmma flash attention with in-kernel reference-KV concat)
against a plain PyTorch fp32 softmax(QK^T/sqrt d)V of the same op."""
import pytest
import torch

from conftest import rel_l2

pytestmark = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _ref_attn(q, k, v, heads):
    # q [F, Lq, C], k/v [F, Lk, C]
    F_, Lq, C = q.shape
    d = C // heads
    qh = q.float().view(F_, Lq, heads, d).transpose(1, 2)
    kh = k.float().view(F_, -1, heads, d).transpose(1, 2)
    vh = v.float().view(F_, -1, heads, d).transpose(1, 2)
    p = torch.softmax(qh @ kh.transpose(-1, -2) * d ** -0.5, dim=-1)
    return (p @ vh).transpose(1, 2).reshape(F_, Lq, C)


@pytest.mark.parametrize("C,L,frames", [(320, 256, 4), (320, 1024, 2), (640, 256, 4), (640, 64, 6), (1280, 64, 4),
                                        (1280, 256, 2), (320, 144, 3), (1280, 144, 2)])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_self_attention(C, L, frames, dtype):
    from hallo_b200 import ops
    dev = _dev()
    g = torch.Generator().manual_seed(C + L)
    qkv = torch.randn(frames * L, 3 * C, generator=g).to(dev, dtype)     # fused projection buffer
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    out = torch.full((frames * L, C), float("nan"), device=dev, dtype=dtype)
    ops.attention(q, k, v, out, heads=8, L=L)
    torch.cuda.synchronize()
    ref = _ref_attn(q.reshape(frames, L, C), k.reshape(frames, L, C), v.reshape(frames, L, C), 8)
    assert rel_l2(out.view(frames, L, C), ref) < (4e-3 if dtype == torch.float16 else 2e-2)


@pytest.mark.parametrize("C,L", [(320, 512), (640, 256), (1280, 64)])
def test_reference_kv_concat(C, L):
    """cond frames attend to [self, ref[n % 2]]; uncond frames to self only (Q3 + Q9)."""
    from hallo_b200 import ops
    dev = _dev()
    dtype = torch.float16
    frames = 8
    g = torch.Generator().manual_seed(L)
    # peaked softmax: scale q up so key ordering / segment bugs cannot average out
    q = (torch.randn(frames * L, C, generator=g) * 2).to(dev, dtype)
    k = torch.randn(frames * L, C, generator=g).to(dev, dtype)
    v = torch.randn(frames * L, C, generator=g).to(dev, dtype)
    kvref = torch.randn(2 * L, 2 * C, generator=g).to(dev, dtype)
    kref, vref = kvref[:, :C], kvref[:, C:]
    ridx = torch.tensor([-1, -1, -1, -1, 0, 1, 0, 1], dtype=torch.int32, device=dev)
    out = torch.empty(frames * L, C, device=dev, dtype=dtype)
    ops.attention(q, k, v, out, heads=8, L=L, kref=kref, vref=vref, ref_index=ridx)
    torch.cuda.synchronize()
    q3, k3, v3 = (t.reshape(frames, L, C) for t in (q, k, v))
    kr, vr = kref.reshape(2, L, C), vref.reshape(2, L, C)
    refs = []
    for n in range(frames):
        r = int(ridx[n])
        kk = k3[n:n + 1] if r < 0 else torch.cat([k3[n:n + 1], kr[r:r + 1]], 1)
        vv = v3[n:n + 1] if r < 0 else torch.cat([v3[n:n + 1], vr[r:r + 1]], 1)
        refs.append(_ref_attn(q3[n:n + 1], kk, vv, 8))
    ref = torch.cat(refs, 0)
    assert rel_l2(out.view(frames, L, C), ref) < 4e-3


def test_large_scores_lazy_rescale():
    """Scores spanning a wide range exercise the lazy O-rescale path."""
    from hallo_b200 import ops
    dev = _dev()
    C, L, frames = 320, 1024, 2
    g = torch.Generator().manual_seed(3)
    q = (torch.randn(frames * L, C, generator=g) * 4).to(dev, torch.float16)
    k = torch.randn(frames * L, C, generator=g)
    k[L // 2:] *= 3.0   # later keys produce much larger logits -> running max keeps growing
    k = k.to(dev, torch.float16)
    v = torch.randn(frames * L, C, generator=g).to(dev, torch.float16)
    out = torch.empty(frames * L, C, device=dev, dtype=torch.float16)
    ops.attention(q, k, v, out, heads=8, L=L)
    torch.cuda.synchronize()
    ref = _ref_attn(q.reshape(frames, L, C), k.reshape(frames, L, C), v.reshape(frames, L, C), 8)
    assert rel_l2(out.view(frames, L, C), ref) < 4e-3


def _ref_attn_cuda(q, k, v, heads):
    """fp32 softmax(QK^T/sqrt d)V on the device, one frame at a time (the 4096 x 8192 score matrices of the headline
    shape are 1 GB per frame in fp32 -- too slow for the host, fine for torch on the GPU as a plain fp32 checker)."""
    assert not torch.backends.cuda.matmul.allow_tf32
    return torch.cat([_ref_attn(q[n:n + 1], k[n:n + 1], v[n:n + 1], heads) for n in range(q.shape[0])], 0)


@pytest.mark.parametrize("C,L,dtype", [(320, 4096, torch.float16), (640, 1024, torch.float16), (1280, 256, torch.float16),
                                       (320, 4096, torch.bfloat16), (320, 9216, torch.bfloat16)])
def test_reference_kv_concat_headline_shapes(C, L, dtype):
    """The shapes bench.py times: L0 = 4096 queries against 8192 keys (self + in-kernel reference concat) at head_dim 40,
    and the L1 / L2 launches (d = 80 / 160); config-4's L0 = 9216 in bf16.  Peaked softmax (q scaled up) so that a wrong
    key segment / ordering cannot average out.  mutual_self_attention.py:233-286 (Q3, Q9)."""
    from hallo_b200 import ops
    dev = _dev()
    frames = 4
    g = torch.Generator().manual_seed(L + C)
    q = (torch.randn(frames * L, C, generator=g) * 2).to(dev, dtype)
    k = torch.randn(frames * L, C, generator=g).to(dev, dtype)
    v = torch.randn(frames * L, C, generator=g).to(dev, dtype)
    kvref = torch.randn(2 * L, 2 * C, generator=g).to(dev, dtype)
    kref, vref = kvref[:, :C], kvref[:, C:]
    ridx = torch.tensor([-1, -1, 1, 0], dtype=torch.int32, device=dev)
    out = torch.full((frames * L, C), float("nan"), device=dev, dtype=dtype)
    ops.attention(q, k, v, out, heads=8, L=L, kref=kref, vref=vref, ref_index=ridx)
    torch.cuda.synchronize()
    q3, k3, v3 = (t.reshape(frames, L, C) for t in (q, k, v))
    kr, vr = kref.reshape(2, L, C), vref.reshape(2, L, C)
    worst = 0.0
    for n in range(frames):
        r = int(ridx[n])
        kk = k3[n:n + 1] if r < 0 else torch.cat([k3[n:n + 1], kr[r:r + 1]], 1)
        vv = v3[n:n + 1] if r < 0 else torch.cat([v3[n:n + 1], vr[r:r + 1]], 1)
        ref = _ref_attn_cuda(q3[n:n + 1], kk, vv, 8)
        worst = max(worst, rel_l2(out.view(frames, L, C)[n:n + 1], ref))
    print(f"C{C} L{L} {dtype}: worst per-frame rel L2 = {worst:.3e}")
    assert worst < (4e-3 if dtype == torch.float16 else 2e-2)
