"""GPU parity of the GEMM / conv3x3 epilogue that stages the output tile in shared memory and stores it with TMA.

The store is clipped at the tensor bounds instead of masked per row, so next to the fp32 PyTorch reference every case
checks that nothing outside the output was written: outputs and residuals are views into larger buffers whose other
elements hold a sentinel (rows past M, columns beyond a column slice, images past the batch)."""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2

pytestmark = pytest.mark.gpu

TOL = {torch.float16: 2e-3, torch.bfloat16: 1.2e-2}
DTYPES = [torch.float16, torch.bfloat16]
SENTINEL = -7.0


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _slice(rows, cols, dev, dtype, extra_rows=5, col0=16, extra_cols=24):
    """[rows, cols] view at column col0 of a sentinel-filled buffer with spare rows and columns around it."""
    buf = torch.full((rows + extra_rows, col0 + cols + extra_cols), SENTINEL, device=dev, dtype=dtype)
    return buf, buf[:rows, col0:col0 + cols]


def _untouched(buf, view):
    mask = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    r0 = (view.data_ptr() - buf.data_ptr()) // buf.element_size() // buf.stride(0)
    c0 = (view.data_ptr() - buf.data_ptr()) // buf.element_size() % buf.stride(0)
    mask[r0:r0 + view.shape[0], c0:c0 + view.shape[1]] = False
    return bool((buf[mask] == SENTINEL).all())


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M,N,K", [(1000, 320, 320), (130, 640, 640), (300, 1280, 192), (77, 328, 64),
                                   (2, 320, 1280), (333, 256, 128), (40000, 320, 320)])
def test_staged_gemm_column_slices_and_row_tails(M, N, K, dtype):
    """bias + group bias + row scale + residual; output and residual are column slices (ldc, ldr != N) and M is not a
    multiple of the 128-row tile."""
    from hallo_b200 import ops
    dev = _dev()
    g = torch.Generator(device="cpu").manual_seed(M + 3 * N + 7 * K)
    a = torch.randn(M, K, generator=g).to(dev, dtype)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev, dtype)
    bias = torch.randn(N, generator=g).to(dev, dtype)
    rs = torch.rand(M, generator=g).to(dev, dtype)
    rpg = max(M // 3, 1)
    gb = torch.randn((M + rpg - 1) // rpg, N, generator=g).to(dev, dtype)
    rbuf, res = _slice(M, N, dev, dtype, col0=40)
    res.copy_(torch.randn(M, N, generator=g).to(dev, dtype))
    obuf, out = _slice(M, N, dev, dtype)
    ops.gemm(a, w, out, bias=bias, residual=res, row_scale=rs, group_bias=gb, rows_per_group=rpg, alpha=0.7)
    torch.cuda.synchronize()
    ref = a.float() @ w.float().t() + bias.float() + gb.float().repeat_interleave(rpg, 0)[:M]
    ref = ref * rs.float()[:, None] * 0.7 + res.float()
    assert rel_l2(out, ref) < TOL[dtype]
    assert _untouched(obuf, out)
    # no residual: the staging tile is handed from tile to tile without the residual load
    ops.gemm(a, w, out, bias=bias)
    torch.cuda.synchronize()
    assert rel_l2(out, a.float() @ w.float().t() + bias.float()) < TOL[dtype]
    assert _untouched(obuf, out)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M,C,mult", [(5000, 320, 8), (300, 640, 8), (515, 256, 4)])
def test_staged_geglu_with_residual(M, C, mult, dtype):
    """GEGLU stages BN/2 output columns per tile (80 of a 160-wide tile, 64 of a 128-wide one)."""
    from hallo_b200 import ops
    dev = _dev()
    g = torch.Generator(device="cpu").manual_seed(M + C)
    N = mult * C
    x = torch.randn(M, C, generator=g).to(dev, dtype)
    w = (torch.randn(N, C, generator=g) / C ** 0.5).to(dev, dtype)
    b = torch.randn(N, generator=g).to(dev, dtype)
    wi, bi = ops.pack_geglu_weight(w, b)
    rbuf, res = _slice(M, N // 2, dev, dtype, col0=40)
    res.copy_(torch.randn(M, N // 2, generator=g).to(dev, dtype))
    obuf, out = _slice(M, N // 2, dev, dtype)
    ops.gemm(x, wi, out, bias=bi, residual=res, geglu=True)
    torch.cuda.synchronize()
    h = x.float() @ w.float().t() + b.float()
    ref = h[:, :N // 2] * F.gelu(h[:, N // 2:]) + res.float()
    assert rel_l2(out, ref) < TOL[dtype]
    assert _untouched(obuf, out)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n,h,cin,cout", [(3, 96, 64, 320), (5, 12, 128, 160), (32, 12, 64, 320), (2, 12, 64, 8),
                                          (3, 96, 128, 8)])
def test_staged_conv_overhanging_boxes(n, h, cin, cout, dtype):
    """conv3x3 + bias + residual at 96x96 and 12x12, whose 128-pixel boxes overhang the image batch, and the 8-channel
    output head; the output is followed by sentinel rows that an overhanging box must not reach."""
    from hallo_b200 import ops
    dev = _dev()
    g = torch.Generator(device="cpu").manual_seed(n * h + cin + cout)
    x = torch.randn(n, cin, h, h, generator=g).to(dev, dtype)
    wt = (torch.randn(cout, cin, 3, 3, generator=g) / (3 * cin ** 0.5)).to(dev, dtype)
    b = torch.randn(cout, generator=g).to(dev, dtype)
    M = n * h * h
    res = torch.randn(M, cout, generator=g).to(dev, dtype)
    obuf = torch.full((M + 4 * h * h, cout), SENTINEL, device=dev, dtype=dtype)
    out = obuf[:M]
    ops.conv3x3(x.permute(0, 2, 3, 1).contiguous(), ops.pack_conv3x3_weight(wt), out, bias=b, residual=res)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float(), wt.float(), b.float(), padding=1).permute(0, 2, 3, 1).reshape(M, cout) + res.float()
    assert rel_l2(out, ref) < TOL[dtype]
    assert bool((obuf[M:] == SENTINEL).all())


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M,N,K,geglu", [(256, 320, 2560, False), (200, 1280, 2048, False), (256, 2560, 2048, True)])
def test_staged_split_k_reduction(M, N, K, geglu, dtype):
    """split 0 adds the fp32 partial tiles and runs the staged epilogue (bias + residual)."""
    from hallo_b200 import lib, ops
    dev = _dev()
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g).to(dev, dtype)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev, dtype)
    b = torch.randn(N, generator=g).to(dev, dtype)
    n_out = N // 2 if geglu else N
    if geglu:
        w, b = ops.pack_geglu_weight(w, b)
    res = torch.randn(M, n_out, generator=g).to(dev, dtype)
    obuf, out = _slice(M, n_out, dev, dtype)
    ops.gemm(a, w, out, bias=b, residual=res, geglu=geglu)
    torch.cuda.synchronize()
    assert int(lib.load().hallo_b200_gemm_last_splits()) > 1
    h = a.float() @ w.float().t() + b.float()
    ref = (h[:, 0::2] * F.gelu(h[:, 1::2]) if geglu else h) + res.float()
    assert rel_l2(out, ref) < TOL[dtype]
    assert _untouched(obuf, out)
    split_out = out.clone()
    ops.gemm(a, w, out, bias=b, residual=res, geglu=geglu, split_k=False)
    torch.cuda.synchronize()
    assert rel_l2(split_out, out) < TOL[dtype]


@pytest.mark.parametrize("dtype", DTYPES)
def test_unaligned_output_keeps_register_epilogue(dtype):
    """An output or residual view that is not 16-byte aligned cannot be a TMA tensor: same result through the
    register epilogue."""
    from hallo_b200 import ops
    dev = _dev()
    g = torch.Generator(device="cpu").manual_seed(5)
    M, N, K = 700, 320, 320
    a = torch.randn(M, K, generator=g).to(dev, dtype)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev, dtype)
    res_buf = torch.randn(M, N + 16, generator=g).to(dev, dtype)
    res = res_buf[:, 4:4 + N]                                       # 8-byte aligned
    obuf, out = _slice(M, N, dev, dtype, col0=4, extra_cols=28)
    ops.gemm(a, w, out, residual=res)
    torch.cuda.synchronize()
    assert rel_l2(out, a.float() @ w.float().t() + res.float()) < TOL[dtype]
    assert _untouched(obuf, out)
