"""GPU parity of hallo_b200_gemm (wgmma) against a plain PyTorch fp32 reference of the same op."""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2

pytestmark = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


TOL = {torch.float16: 2e-3, torch.bfloat16: 1.2e-2}


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K", [(128, 160, 64), (256, 320, 320), (2048, 1280, 1280), (1000, 328, 192),
                                   (8, 640, 768), (4096, 2560, 320), (512, 960, 320), (384, 1920, 640),
                                   (300, 320, 64), (131072, 320, 320)])
def test_gemm_plain(M, N, K, dtype):
    from hallo_b200 import ops
    dev = _dev()
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K, generator=g).to(dev, dtype)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev, dtype)
    out = torch.full((M, N), float("nan"), device=dev, dtype=dtype)
    ops.gemm(a, w, out)
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t()
    assert rel_l2(out, ref) < TOL[dtype]


def test_gemm_epilogue_all():
    from hallo_b200 import ops
    dev = _dev()
    dtype = torch.float16
    M, N, K = 1536, 640, 384
    g = torch.Generator(device="cpu").manual_seed(1)
    a = torch.randn(M, K, generator=g).to(dev, dtype)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev, dtype)
    bias = torch.randn(N, generator=g).to(dev, dtype)
    res = torch.randn(M, N, generator=g).to(dev, dtype)
    rs = torch.rand(M, generator=g).to(dev, dtype)
    gb = torch.randn(3, N, generator=g).to(dev, dtype)
    out = torch.empty(M, N, device=dev, dtype=dtype)
    ops.gemm(a, w, out, bias=bias, residual=res, row_scale=rs, group_bias=gb, rows_per_group=512, alpha=0.7)
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t() + bias.float() + gb.float().repeat_interleave(512, 0)
    ref = ref * rs.float()[:, None] * 0.7 + res.float()
    assert rel_l2(out, ref) < 2e-3


def test_gemm_geglu_and_split_k():
    from hallo_b200 import ops
    dev = _dev()
    dtype = torch.float16
    M, C = 1024, 320
    g = torch.Generator(device="cpu").manual_seed(2)
    x = torch.randn(M, C, generator=g).to(dev, dtype)
    w = (torch.randn(8 * C, C, generator=g) / C ** 0.5).to(dev, dtype)
    b = torch.randn(8 * C, generator=g).to(dev, dtype)
    wi, bi = ops.pack_geglu_weight(w, b)
    out = torch.empty(M, 4 * C, device=dev, dtype=dtype)
    ops.gemm(x, wi, out, bias=bi, geglu=True)
    torch.cuda.synchronize()
    h = x.float() @ w.float().t() + b.float()
    ref = h[:, :4 * C] * F.gelu(h[:, 4 * C:])
    assert rel_l2(out, ref) < 2e-3
    # K split over two sources, output written into a column slice of a wider buffer
    a1 = torch.randn(M, 640, generator=g).to(dev, dtype)
    a2 = torch.randn(M, 320, generator=g).to(dev, dtype)
    w2 = (torch.randn(320, 960, generator=g) / 30).to(dev, dtype)
    wide = torch.zeros(M, 640, device=dev, dtype=dtype)
    ops.gemm(a1, w2, wide[:, 320:], a2=a2)
    torch.cuda.synchronize()
    ref2 = torch.cat([a1, a2], 1).float() @ w2.float().t()
    assert rel_l2(wide[:, 320:], ref2) < 2e-3
    assert float(wide[:, :320].abs().max()) == 0.0


@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 64, 64, 320, 320), (4, 32, 32, 640, 320), (4, 16, 16, 1280, 640),
                                            (4, 8, 8, 1280, 1280), (2, 24, 24, 128, 160), (8, 12, 12, 64, 160),
                                            (4, 1, 1, 320, 320), (6, 2, 2, 640, 160), (3, 20, 12, 64, 320)])
def test_conv3x3(n, h, w, cin, cout):
    from hallo_b200 import ops
    dev = _dev()
    dtype = torch.float16
    g = torch.Generator(device="cpu").manual_seed(n + h + cin)
    x = torch.randn(n, cin, h, w, generator=g).to(dev, dtype)
    wt = (torch.randn(cout, cin, 3, 3, generator=g) / (3 * cin ** 0.5)).to(dev, dtype)
    b = torch.randn(cout, generator=g).to(dev, dtype)
    x_nhwc = x.permute(0, 2, 3, 1).contiguous()
    out = torch.empty(n * h * w, cout, device=dev, dtype=dtype)
    ops.conv3x3(x_nhwc, ops.pack_conv3x3_weight(wt), out, bias=b)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float(), wt.float(), b.float(), padding=1).permute(0, 2, 3, 1).reshape(n * h * w, cout)
    assert rel_l2(out, ref) < 2e-3


@pytest.mark.parametrize("M,C,N,geglu", [(2048, 320, 960, False), (1024, 640, 5120, True), (777, 1280, 1280, False)])
def test_layernorm_folded_into_gemm(M, C, N, geglu):
    """producer GEMM accumulates row (sum, sumsq) through stats_out; consumer GEMM applies LayerNorm in its epilogue."""
    from hallo_b200 import ops
    dev = _dev()
    dtype = torch.float16
    g = torch.Generator(device="cpu").manual_seed(M + N)
    a0 = torch.randn(M, 320, generator=g).to(dev, dtype)
    w0 = (torch.randn(C, 320, generator=g) / 320 ** 0.5).to(dev, dtype)
    res = (torch.randn(M, C, generator=g) * 2 + 0.7).to(dev, dtype)
    x = torch.empty(M, C, device=dev, dtype=dtype)
    stats = torch.zeros(M, 2, device=dev, dtype=torch.float32)
    ops.gemm(a0, w0, x, residual=res, stats_out=stats)                 # x = a0 w0^T + res, plus row statistics
    torch.cuda.synchronize()
    xf = x.float()
    assert torch.allclose(stats[:, 0], xf.sum(1), rtol=1e-4, atol=1e-2)
    assert torch.allclose(stats[:, 1], (xf * xf).sum(1), rtol=1e-4, atol=1e-2)
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).to(dev, dtype)
    beta = (0.2 * torch.randn(C, generator=g)).to(dev, dtype)
    w = (torch.randn(N, C, generator=g) / C ** 0.5).to(dev, dtype)
    b = torch.randn(N, generator=g).to(dev, dtype)
    ref = F.layer_norm(xf, (C,), gamma.float(), beta.float(), 1e-5) @ w.float().t() + b.float()
    if geglu:
        wi, bi = ops.pack_geglu_weight(w, b)
        ref = ref[:, :N // 2] * F.gelu(ref[:, N // 2:])
    else:
        wi, bi = w, b
    wg, colsum, bb = ops.fold_layernorm(wi, bi, gamma, beta, dtype)
    out = torch.empty(M, N // 2 if geglu else N, device=dev, dtype=dtype)
    ops.gemm(x, wg, out, bias=bb, geglu=geglu, ln_stats=stats, ln_colsum=colsum, ln_eps=1e-5)
    torch.cuda.synchronize()
    assert rel_l2(out, ref) < 3e-3


def _with_splitk(fn):
    """fn() with option gemm_splitk on, then off; returns (split result, split factor used, unsplit result)."""
    from hallo_b200 import lib
    was = int(lib.load().hallo_b200_get_option(b"gemm_splitk"))
    lib.set_option("gemm_splitk", 16)                      # > 1: split from 16 k-blocks on (the default needs 32)
    try:
        a = fn().clone()
        torch.cuda.synchronize()
        splits = int(lib.load().hallo_b200_gemm_last_splits())
        b = fn().clone()                                   # second launch: counters must have been re-armed
        torch.cuda.synchronize()
        lib.set_option("gemm_splitk", 0)
        c = fn().clone()
        torch.cuda.synchronize()
        assert int(lib.load().hallo_b200_gemm_last_splits()) == 1
    finally:
        lib.set_option("gemm_splitk", was)
    assert torch.equal(a, b), "split-K summation order must not depend on timing"
    return a, splits, c


@pytest.mark.parametrize("pdl", [1, 0])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K,geglu", [(256, 1280, 1280, False), (256, 1280, 5120, False), (1024, 1280, 5120, False),
                                         (200, 960, 2560, False), (256, 320, 1024, False), (8, 1280, 1280, False),
                                         (64, 640, 2048, False), (256, 5120, 1280, True), (512, 2560, 1024, True)])
def test_gemm_split_k_option(M, N, K, geglu, dtype, pdl):
    """Option gemm_splitk (include/hallo_b200.h): K loop of a few-tile GEMM divided over several CTAs, fp32 partials
    reduced by split 0 in fixed order -- plain and GEGLU epilogues with bias, residual and row scale, launched with and
    without programmatic dependent launch (option pdl: a launch may start while its predecessor drains)."""
    from hallo_b200 import lib, ops
    dev = _dev()
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g).to(dev, dtype)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev, dtype)
    b = torch.randn(N, generator=g).to(dev, dtype)
    n_out = N // 2 if geglu else N
    res = torch.randn(M, n_out, generator=g).to(dev, dtype)
    rs = torch.rand(M, generator=g).to(dev, dtype)
    if geglu:
        w, b = ops.pack_geglu_weight(w, b)
    out = torch.empty(M, n_out, device=dev, dtype=dtype)
    was_pdl = lib.get_option("pdl")
    lib.set_option("pdl", pdl)
    try:
        got, splits, unsplit = _with_splitk(lambda: ops.gemm(a, w, out, bias=b, residual=res, row_scale=rs, geglu=geglu))
    finally:
        lib.set_option("pdl", was_pdl)
    assert splits > 1, "shape chosen to split"
    h = a.float() @ (w.float().t())
    h = h + b.float()
    if geglu:
        h = h[:, 0::2] * F.gelu(h[:, 1::2])
    ref = h * rs.float()[:, None] + res.float()
    print(f"M{M} N{N} K{K} geglu={geglu} pdl={pdl}: S={splits}, rel L2 vs fp32 {rel_l2(got, ref):.2e}, vs unsplit {rel_l2(got, unsplit):.2e}")
    assert rel_l2(got, ref) < TOL[dtype]
    assert rel_l2(got, unsplit) < TOL[dtype]


@pytest.mark.parametrize("n,h,w,cin,cout", [(4, 8, 8, 1280, 1280), (4, 16, 16, 1280, 640), (4, 8, 8, 2560, 1280),
                                            (2, 16, 16, 640, 320), (4, 4, 4, 1280, 1280)])
def test_conv3x3_split_k_option(n, h, w, cin, cout):
    from hallo_b200 import ops
    dev = _dev()
    dtype = torch.float16
    g = torch.Generator(device="cpu").manual_seed(n + h + cin)
    x = torch.randn(n, cin, h, w, generator=g).to(dev, dtype)
    wt = (torch.randn(cout, cin, 3, 3, generator=g) / (3 * cin ** 0.5)).to(dev, dtype)
    b = torch.randn(cout, generator=g).to(dev, dtype)
    res = torch.randn(n * h * w, cout, generator=g).to(dev, dtype)
    x_nhwc = x.permute(0, 2, 3, 1).contiguous()
    wp = ops.pack_conv3x3_weight(wt)
    out = torch.empty(n * h * w, cout, device=dev, dtype=dtype)
    got, splits, unsplit = _with_splitk(lambda: ops.conv3x3(x_nhwc, wp, out, bias=b, residual=res))
    assert splits > 1
    ref = F.conv2d(x.float(), wt.float(), b.float(), padding=1).permute(0, 2, 3, 1).reshape(n * h * w, cout) + res.float()
    print(f"conv n{n} {h}x{w} {cin}->{cout}: S={splits}, rel L2 vs fp32 {rel_l2(got, ref):.2e}")
    assert rel_l2(got, ref) < 2e-3
    assert rel_l2(got, unsplit) < 2e-3


def test_split_k_interleaved_shapes_reuse_the_workspace():
    """Back-to-back split GEMMs of different shapes share one workspace and one set of counters: each launch must
    leave the counters at zero for the next (stream order), whatever its tile count."""
    from hallo_b200 import lib, ops
    dev = _dev()
    dtype = torch.float16
    g = torch.Generator(device="cpu").manual_seed(99)
    shapes = [(256, 1280, 5120), (1024, 1280, 1280), (128, 640, 2560), (256, 1280, 5120), (512, 960, 1920)]
    cases = []
    for M, N, K in shapes:
        a = torch.randn(M, K, generator=g).to(dev, dtype)
        w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev, dtype)
        cases.append((a, w, torch.empty(M, N, device=dev, dtype=dtype)))
    was = int(lib.load().hallo_b200_get_option(b"gemm_splitk"))
    lib.set_option("gemm_splitk", 16)
    try:
        for _ in range(5):
            for a, w, out in cases:
                ops.gemm(a, w, out)
        torch.cuda.synchronize()
    finally:
        lib.set_option("gemm_splitk", was)
    for a, w, out in cases:
        assert rel_l2(out, a.float() @ w.float().t()) < 2e-3
