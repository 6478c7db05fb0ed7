"""Every kernel path of the helper ops (csrc/aux.cu, csrc/tattn_mma.cu, the cross-attention in csrc/attn_tc.cu) and
the LayerNorm fold of the GEMM, in fp16 and bf16, against float64 references computed from the same rounded inputs.

Each case forces a path with the kernel-selection options (include/hallo_b200.h) and asserts, from a torch.profiler
trace, that the kernel it targets is the one that ran, so a shape that quietly lands on another path fails.  Outputs
are views into NaN-filled buffers with guard rows / columns: every output element must be written and nothing around
it.  Errors are checked globally and per (frame, head) / (frame, group) slice, so one wrong head, frame or tail pixel
cannot hide in the average."""
import contextlib
import math
import re

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["f16", "bf16"]
# attention: global / per-slice relative L2 bounds (fp16: 11-bit, bf16: 8-bit significand; P is rounded to the storage
# type before the P V product on the tensor-core paths)
ATTN_TOL = {torch.float16: (2e-3, 4e-3), torch.bfloat16: (1.2e-2, 2.4e-2)}


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@contextlib.contextmanager
def _option(name, value):
    """Set a kernel-selection option for the duration of the block, then restore the old value."""
    from hallo_b200 import lib
    was = lib.get_option(name)
    lib.set_option(name, value)
    try:
        yield
    finally:
        lib.set_option(name, was)


def _kernels(fn, expect, tries=3):
    """Names of the CUDA kernels fn() launched (torch.profiler, CUDA activity).  The profiler now and then drops the
    records of some kernels of a short session (seen on an H100: a GroupNorm trace with its finalize and apply kernels
    but not its stats kernel), so a trace without a kernel named like `expect` is taken again, up to `tries` times; fn
    must be safe to repeat.  A path that is not taken still fails: every trace then lacks its kernel."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(tries):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        if any(expect in n for n in names):
            break
    return names


def _ran(names, kernel, not_kernels=()):
    assert any(kernel in n for n in names), f"{kernel} did not run; kernels launched: {names}"
    for other in not_kernels:
        assert not any(other in n for n in names), f"{other} ran as well as {kernel}: {names}"


def _trace(fn, kernel):
    """fn() under the profiler; asserts that `kernel` ran."""
    _ran(_kernels(fn, kernel), kernel)


def _randn(shape, gen, dtype, mean=0.0, std=1.0):
    return (torch.randn(shape, generator=gen, device="cuda", dtype=torch.float32) * std + mean).to(dtype)


class _Guarded:
    """A NaN-filled buffer with `gr` guard rows above and below and `gc` guard columns left and right of the
    [rows, cols] output view (gc = 0: a contiguous view, for ops that need one)."""

    def __init__(self, rows, cols, dtype, gr=3, gc=8):
        self.big = torch.full((rows + 2 * gr, cols + 2 * gc), float("nan"), device="cuda", dtype=dtype)
        self.view = self.big[gr:gr + rows, gc:gc + cols]
        self.mask = torch.zeros(self.big.shape, dtype=torch.bool, device="cuda")
        self.mask[gr:gr + rows, gc:gc + cols] = True

    def check(self, written=None):
        """Guard region bit-identical (still NaN); every element of the output view (or of `written`, a bool mask
        over the view) finite."""
        mask = self.mask.clone()
        if written is not None:
            mask[self.mask] = written.reshape(-1)
        _assert_all_nan_bits(self.big[~mask])
        assert torch.isfinite(self.big[mask].float()).all(), "output element left unwritten (still NaN)"


def _assert_all_nan_bits(t):
    nan = torch.full((1,), float("nan"), dtype=t.dtype, device=t.device).view(torch.int16)
    bits = t.reshape(-1).view(torch.int16)
    assert torch.equal(bits, nan.expand_as(bits)), "a kernel wrote outside its output"


def _errs(out, ref, slices):
    """(global rel L2, worst rel L2 over `slices` equal slices of the leading dim) in float64."""
    o = out.double().reshape(slices, -1)
    r = ref.double().reshape(slices, -1)
    d = o - r
    glob = float(d.norm() / r.norm().clamp_min(1e-300))
    worst = float((d.norm(dim=1) / r.norm(dim=1).clamp_min(1e-300)).max())
    return glob, worst


def _floor(ref, dtype):
    """Relative L2 of rounding the exact output to the storage type: the best any kernel can do."""
    return float((ref.to(dtype).double() - ref).norm() / ref.norm())


# ------------------------------------------------------------------------------------------------ temporal attention
def _mma_tiles(fq, fk):
    """(MT, NT) instantiation of tattn_mma_kernel that dispatch_tattn_mma picks."""
    return (1 if fq <= 16 else 2), (1 if fk <= 8 else (3 if fk <= 24 else 4))


def _mma_fits(heads, d, fq, fk, L):
    """launch_tattn_mma's shared-memory rule: the Q, K, V rows of at least one pixel must fit 220 KB."""
    ps = heads * d * 2 + 16
    rows = fq + 2 * fk
    pix = max(1, min(4, (72 * 1024) // (rows * ps), L))
    fs = pix * ps
    if ((fs >> 4) & 1) == 0:
        fs += 16
    return rows * fs <= 220 * 1024


def _run_tattn(heads, d, fq, fk, L, dtype, seed, expect, b=2):
    """Q, K, V are column slices of one fused [rows, 3C] buffer; O a view with guard rows / columns."""
    C = heads * d
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = _randn((b * max(fq, fk) * L, 3 * C), g, dtype)
    q, k, v = qkv[:b * fq * L, :C], qkv[:b * fk * L, C:2 * C], qkv[:b * fk * L, 2 * C:]
    out = _Guarded(b * fq * L, C, dtype)
    from hallo_b200 import ops
    names = _kernels(lambda: ops.temporal_attention(q, k, v, out.view, batch=b, fq=fq, fk=fk, tokens=L, heads=heads),
                     expect)
    qd = q.double().view(b, fq, L, heads, d).permute(0, 2, 3, 1, 4)
    kd = k.double().view(b, fk, L, heads, d).permute(0, 2, 3, 1, 4)
    vd = v.double().view(b, fk, L, heads, d).permute(0, 2, 3, 1, 4)
    ref = torch.softmax(qd @ kd.transpose(-1, -2) / math.sqrt(d), -1) @ vd        # [b, L, H, fq, d]
    ref = ref.permute(0, 3, 2, 1, 4)                                              # slices (b, fq, H) x (L, d)
    got = out.view.view(b, fq, L, heads, d).permute(0, 1, 3, 2, 4)
    out.check()
    return names, _errs(got, ref, b * fq * heads)


def _tattn_cases():
    """(Fq, Fk) pairs over Fk in {1, 8, 9, 24, 25, 32} and Fq in {1, 16, 17, 32}, Fq != Fk both ways, reaching all six
    (MT, NT) instantiations; d = 160 with Fq = Fk = 32 (96 rows of 2.5 KB) does not fit the tensor-core kernel's shared
    memory and is covered by test_temporal_attention_mma_falls_back_when_rows_do_not_fit."""
    cases = []
    for path in ("tattn_mma_kernel", "tattn_smem_kernel"):
        for d in (40, 80, 160):
            for fq, fk in [(1, 1), (16, 8), (17, 8), (1, 9), (32, 24), (16, 25), (17, 32), (32, 32)]:
                if path == "tattn_mma_kernel" and not _mma_fits(8, d, fq, fk, 64):
                    continue
                cases.append(pytest.param(path, d, fq, fk, id=f"{path}-d{d}-Fq{fq}-Fk{fk}"))
    return cases


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("L", [64, 67])
@pytest.mark.parametrize("path,d,fq,fk", _tattn_cases())
def test_temporal_attention_path(path, d, fq, fk, L, dtype):
    """tattn_mma on: all six (MT, NT) instantiations, ragged Fq / Fk, a last CTA with fewer pixels (L = 67).
    tattn_mma off: the shared-memory CUDA-core kernel on the same shapes."""
    _dev()
    with _option("tattn_mma", 1 if path == "tattn_mma_kernel" else 0):
        names, (glob, worst) = _run_tattn(8, d, fq, fk, L, dtype, seed=d * 1000 + fq * 37 + fk + L, expect=path)
    if path == "tattn_mma_kernel":
        mt, nt = _mma_tiles(fq, fk)
        hit = [n for n in names if "tattn_mma_kernel" in n]
        assert len(hit) == 1, names
        m = re.search(r"tattn_mma_kernel<[^,]+,\s*(\d+),\s*(\d+),\s*(\d+)\s*>", hit[0])
        assert m is not None, hit[0]
        assert tuple(int(v) for v in m.groups()) == (d, mt, nt), hit[0]
    else:
        _ran(names, "tattn_smem_kernel", ("tattn_mma_kernel", "tattn_kernel<"))
    tol, stol = ATTN_TOL[dtype]
    assert glob < tol and worst < stol, (glob, worst)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("L", [64, 67])
def test_temporal_attention_mma_falls_back_when_rows_do_not_fit(L, dtype):
    """tattn_mma on, d = 160 (C = 1280), Fq = Fk = 32: one pixel's Q, K, V rows exceed 220 KB, so the shared-memory
    CUDA-core kernel takes the call."""
    _dev()
    assert not _mma_fits(8, 160, 32, 32, L)
    with _option("tattn_mma", 1):
        names, (glob, worst) = _run_tattn(8, 160, 32, 32, L, dtype, seed=L + 5, expect="tattn_smem_kernel")
    _ran(names, "tattn_smem_kernel", ("tattn_mma_kernel", "tattn_kernel<"))
    tol, stol = ATTN_TOL[dtype]
    assert glob < tol and worst < stol, (glob, worst)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("heads,d,fq,fk", [(8, 320, 16, 32), (8, 320, 1, 25), (8, 400, 17, 17)])
def test_temporal_attention_l1_kernel(heads, d, fq, fk, dtype):
    """Rows too wide for the shared-memory variant (Fk * C * 4 bytes > 200 KB): the L1 kernel, both MAXF
    instantiations (Fk <= 18 and Fk <= 32)."""
    _dev()
    with _option("tattn_mma", 0):
        names, (glob, worst) = _run_tattn(heads, d, fq, fk, 67, dtype, seed=d + fq + fk, expect="tattn_kernel<", b=1)
    _ran(names, "tattn_kernel<", ("tattn_smem_kernel", "tattn_mma_kernel"))
    maxf = [re.search(r"tattn_kernel<[^,]+,\s*(\d+)\s*>", n) for n in names if "tattn_kernel<" in n]
    assert maxf and maxf[0] is not None and int(maxf[0].group(1)) == (18 if fk <= 18 else 32), names
    tol, stol = ATTN_TOL[dtype]
    assert glob < tol and worst < stol, (glob, worst)


# ------------------------------------------------------------------------------------------------ cross-attention
def _run_xattn(d, nk, L, regions, div, dtype, layout, seed, expect, heads=8, frames=4):
    """layout "adjacent": [K_r | V_r] pairs 2C apart (the tensor-core layout); "v_gap": V = K + 2C columns;
    "region_stride": [K_r | V_r] pairs 3C apart."""
    from hallo_b200 import ops
    C = heads * d
    kvf = frames // div
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = _randn((frames * L, regions * C), g, dtype)
    if layout == "adjacent":
        rs, voff = 2 * C, C
    elif layout == "v_gap":
        rs, voff = 3 * C, 2 * C
    else:
        rs, voff = 3 * C, C
    kv = _randn((kvf * nk, regions * rs), g, dtype)
    k, v = kv[:, :C], kv[:, voff:voff + C]
    out = _Guarded(frames * L, regions * C, dtype)
    names = _kernels(lambda: ops.cross_attention(q, k, v, out.view, frames=frames, tokens=L, heads=heads, head_dim=d,
                                                 n_keys=nk, kv_frame_div=div, regions=regions, q_region_stride=C,
                                                 kv_region_stride=rs, o_region_stride=C), expect)
    qd = q.double().view(frames, L, regions, heads, d).permute(0, 2, 3, 1, 4)               # [f, r, H, L, d]
    kvd = kv.double().view(kvf, nk, regions, rs)
    kd = kvd[..., :C].reshape(kvf, nk, regions, heads, d).permute(0, 2, 3, 1, 4).repeat_interleave(div, 0)
    vd = kvd[..., voff:voff + C].reshape(kvf, nk, regions, heads, d).permute(0, 2, 3, 1, 4).repeat_interleave(div, 0)
    ref = torch.softmax(qd @ kd.transpose(-1, -2) / math.sqrt(d), -1) @ vd                  # [f, r, H, L, d]
    got = out.view.view(frames, L, regions, heads, d).permute(0, 2, 3, 1, 4)
    out.check()
    return names, _errs(got, ref, frames * regions * heads)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("regions,div", [(1, 2), (3, 1)])
@pytest.mark.parametrize("L", [64, 127, 128, 129, 200, 1024])
@pytest.mark.parametrize("nk", [4, 32])
@pytest.mark.parametrize("d", [40, 80, 160])
@pytest.mark.parametrize("tc", [1, 0], ids=["xattn_tc1", "xattn_tc0"])
def test_cross_attention_path(tc, d, nk, L, regions, div, dtype):
    """xattn_tc on: the wgmma kernel from L = 128 on (L not a multiple of 128 included), the CUDA-core kernel below;
    off: the CUDA-core kernel everywhere."""
    _dev()
    expect, other = ("attn_tc_kernel", "xattn_kernel") if tc and L >= 128 else ("xattn_kernel", "attn_tc_kernel")
    with _option("xattn_tc", tc):
        names, (glob, worst) = _run_xattn(d, nk, L, regions, div, dtype, "adjacent", seed=d * 100 + nk + L + regions,
                                          expect=expect)
    _ran(names, expect, (other,))
    tol, stol = ATTN_TOL[dtype]
    assert glob < tol and worst < stol, (glob, worst)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("nk", [4, 32])
@pytest.mark.parametrize("d", [40, 80, 160])
@pytest.mark.parametrize("layout,regions", [("v_gap", 1), ("region_stride", 2)])
def test_cross_attention_layout_fallback(layout, regions, d, nk, dtype):
    """K / V layouts outside the tensor-core path's contract fall back to the CUDA-core kernel and stay right."""
    _dev()
    with _option("xattn_tc", 1):
        names, (glob, worst) = _run_xattn(d, nk, 200, regions, 1, dtype, layout, seed=d + nk + regions,
                                          expect="xattn_kernel")
    _ran(names, "xattn_kernel", ("attn_tc_kernel",))
    tol, stol = ATTN_TOL[dtype]
    assert glob < tol and worst < stol, (glob, worst)


# ------------------------------------------------------------------------------------------------ GroupNorm
G = 32


def _gn_fused_chosen(C, hw, n):
    """The size rule of groupnorm_impl (csrc/aux.cu) with option gn_fused on."""
    cpg = C // G
    small = hw <= 256 or cpg >= 40 or (cpg >= 20 and n * hw * C * 2 <= (12 << 20))
    return cpg % 2 == 0 and hw * cpg * 2 <= 96 * 1024 and small


def _gn_ref(xc, gamma, beta, n, hw, eps, silu, dtype):
    """float64 GroupNorm of the rounded input; with SiLU, as the kernels define it: SiLU of the GN output rounded to
    the storage type."""
    C = xc.shape[1]
    x = xc.double().view(n, hw, G, C // G)
    mean = x.mean(dim=(1, 3), keepdim=True)
    var = (x - mean).square().mean(dim=(1, 3), keepdim=True)
    y = ((x - mean) / torch.sqrt(var + eps)).view(n, hw, C) * gamma.double() + beta.double()
    if silu:
        y = F.silu(y.to(dtype).double())
    return y


def _gn_check(got, ref, n, hw, C, dtype):
    """err <= 2 x the rounding floor of the exact output + 1e-5, per (frame, group) slice <= 4 x that."""
    bound = 2 * _floor(ref, dtype) + 1e-5
    g4 = got.reshape(n, hw, G, C // G).permute(0, 2, 1, 3)
    r4 = ref.reshape(n, hw, G, C // G).permute(0, 2, 1, 3)
    glob, worst = _errs(g4, r4, n * G)
    print(f"groupnorm rel L2 {glob:.3e}, worst (frame, group) {worst:.3e}, bound {bound:.3e}")
    assert glob <= bound and worst <= 4 * bound, (glob, worst, bound)


def _gn_inputs(C1, C2, n, hw, offset, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x1 = _randn((n * hw, C1), g, dtype, mean=offset)
    x2 = _randn((n * hw, C2), g, dtype, mean=offset * 0.5) if C2 else None
    C = C1 + C2
    gam = _randn((C,), g, dtype, mean=1.0, std=0.1)
    bet = _randn((C,), g, dtype, std=0.1)
    return x1, x2, gam, bet


# (C1, C2): the UNet's skip concats, including groups that straddle the two sources (960 = 640 + 320 at 30 channels
# per group, 1920 = 1280 + 640 at 60)
_GN_SPLIT = {640: (320, 320), 960: (640, 320), 1920: (1280, 640), 2560: (1280, 1280)}


def _gn_cases():
    cases = []
    for i, C in enumerate([128, 256, 512, 320, 640, 960, 1280, 1920, 2560]):
        for j, hw in enumerate([64, 100, 256, 4096] + ([1024] if C in (640, 1280) else [])):
            k = i + j
            C1, C2 = _GN_SPLIT[C] if (C in _GN_SPLIT and k % 2 == 1) else (C, 0)
            silu = k % 2 == 0
            eps = 1e-5 if (k // 2) % 2 == 0 else 1e-6
            for path in ("gn_fused_kernel", "gn_stats_kernel"):
                if path == "gn_fused_kernel" and not _gn_fused_chosen(C, hw, 2):
                    continue
                cases.append(pytest.param(path, C1, C2, hw, silu, eps,
                                          id=f"{path}-C{C1}+{C2}-hw{hw}-{'silu' if silu else 'nosilu'}-eps{eps:g}"))
    cases.append(pytest.param("gn_stats_kernel", 128, 0, 262144, False, 1e-6, id="gn_stats_kernel-vae512-C128"))
    return cases


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("offset", [0.0, 10.0, 100.0])
@pytest.mark.parametrize("path,C1,C2,hw,silu,eps", _gn_cases())
def test_groupnorm_path(path, C1, C2, hw, silu, eps, offset, dtype):
    """Both GroupNorm paths over channels-per-group 4..80 (and the odd 10 / 30), with inputs N(offset, 1): the
    statistics must not lose precision to a large per-group mean."""
    from hallo_b200 import ops
    _dev()
    n = 1 if hw > 100000 else 2
    C = C1 + C2
    x1, x2, gam, bet = _gn_inputs(C1, C2, n, hw, offset, dtype, seed=C * 7 + hw + int(offset))
    out = _Guarded(n * hw, C, dtype, gr=5, gc=0)
    ws = torch.empty(ops.gn_workspace_floats(n, hw, G, C), device="cuda", dtype=torch.float32)
    with _option("gn_fused", 1 if path == "gn_fused_kernel" else 0):
        names = _kernels(lambda: ops.groupnorm(x1, gam, bet, out.view, ws, n_frames=n, hw=hw, eps=eps, silu=silu, x2=x2),
                         path)
    _ran(names, path, ("gn_stats_kernel" if path == "gn_fused_kernel" else "gn_fused_kernel",))
    out.check()
    xc = x1 if x2 is None else torch.cat([x1, x2], 1)
    ref = _gn_ref(xc, gam, bet, n, hw, eps, silu, dtype)
    _gn_check(out.view, ref, n, hw, C, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("offset", [0.0, 100.0])
@pytest.mark.parametrize("path", ["gn_fused_kernel", "gn_stats_kernel"])
def test_groupnorm_frame_remap_path(path, offset, dtype):
    """fpb_in / fpb_out / frame_off: frame n goes to (n / fpb_in) * fpb_out + frame_off + n % fpb_in; the frames
    between stay untouched."""
    from hallo_b200 import ops
    _dev()
    b, f, hw, C = 2, 4, 64, 320
    x, _, gam, bet = _gn_inputs(C, 0, b * f, hw, offset, dtype, seed=int(offset) + 3)
    out = _Guarded(b * (f + 2) * hw, C, dtype, gr=5, gc=0)
    ws = torch.empty(ops.gn_workspace_floats(b * f, hw, G, C), device="cuda", dtype=torch.float32)
    with _option("gn_fused", 1 if path == "gn_fused_kernel" else 0):
        names = _kernels(lambda: ops.groupnorm(x, gam, bet, out.view, ws, n_frames=b * f, hw=hw, eps=1e-6,
                                               silu=True, fpb_in=f, fpb_out=f + 2, frame_off=2), path)
    _ran(names, path)
    written = torch.zeros(b, f + 2, hw, C, dtype=torch.bool, device="cuda")
    written[:, 2:] = True
    out.check(written)
    ref = _gn_ref(x, gam, bet, b * f, hw, 1e-6, True, dtype)
    _gn_check(out.view.view(b, f + 2, hw, C)[:, 2:], ref, b * f, hw, C, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("offset", [0.0, 100.0])
def test_groupnorm_scatter_path(offset, dtype):
    """hallo_b200_groupnorm_scatter (always the three-launch path): pixel slice d of output frame n_out goes to
    destination d; everything else in the destinations stays untouched."""
    from hallo_b200 import ops
    _dev()
    nb, fl, hw, C, R, nm, me = 2, 2, 256, 640, 4, 2, 1
    seg, F18 = hw // R, nm + fl * R
    x, _, gam, bet = _gn_inputs(C, 0, nb * fl, hw, offset, dtype, seed=int(offset) + 4)
    dest = [_Guarded(nb * F18 * seg, C, dtype, gr=5, gc=0) for _ in range(R)]
    ws = torch.empty(ops.gn_workspace_floats(nb * fl, hw, G, C), device="cuda", dtype=torch.float32)
    names = _kernels(lambda: ops.groupnorm_scatter(x, gam, bet, [t.view.data_ptr() for t in dest], ws,
                                                   n_frames=nb * fl, hw=hw, eps=1e-5, fpb_in=fl, fpb_out=F18,
                                                   frame_off=nm + me * fl), "gn_stats_kernel")
    _ran(names, "gn_stats_kernel", ("gn_fused_kernel",))
    written = torch.zeros(nb, F18, seg, C, dtype=torch.bool, device="cuda")
    written[:, nm + me * fl: nm + (me + 1) * fl] = True
    for t in dest:
        t.check(written)
    got = torch.stack([t.view.view(nb, F18, seg, C)[:, nm + me * fl: nm + (me + 1) * fl] for t in dest], 2)
    ref = _gn_ref(x, gam, bet, nb * fl, hw, 1e-5, False, dtype)
    _gn_check(got.reshape(nb * fl * hw, C), ref, nb * fl, hw, C, dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("path,C,hw", [("gn_fused_kernel", 640, 256), ("gn_stats_kernel", 640, 256),
                                       ("gn_stats_kernel", 128, 65536)])
def test_groupnorm_bitwise_reproducible(path, C, hw, dtype):
    """Fixed summation order on both paths: the same call twice gives the same bits."""
    from hallo_b200 import ops
    _dev()
    n = 2
    x, _, gam, bet = _gn_inputs(C, 0, n, hw, 100.0, dtype, seed=C + hw)
    ws = torch.empty(ops.gn_workspace_floats(n, hw, G, C), device="cuda", dtype=torch.float32)
    outs = []
    with _option("gn_fused", 1 if path == "gn_fused_kernel" else 0):
        for _ in range(2):
            out = torch.empty(n * hw, C, device="cuda", dtype=dtype)
            names = _kernels(lambda: ops.groupnorm(x, gam, bet, out, ws, n_frames=n, hw=hw, eps=1e-5, silu=True), path)
            _ran(names, path)
            outs.append(out)
    assert torch.equal(outs[0], outs[1])


# ------------------------------------------------------------------------------------------------ LayerNorm
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("offset", [0.0, 100.0])
@pytest.mark.parametrize("pe", ["nope", "pe", "pe_index"])
@pytest.mark.parametrize("C", [320, 640, 768, 1280, 2560])
def test_layernorm_path(C, pe, offset, dtype):
    """999 rows (a partial last CTA), strided input and output views, PE with and without a frame remap, inputs
    N(offset, 1)."""
    from hallo_b200 import ops
    from hallo_b200.spec import sinusoid_pe
    _dev()
    b, frames, L = 3, 9, 37
    rows = b * frames * L
    g = torch.Generator(device="cuda").manual_seed(C + int(offset))
    xb = _randn((rows, C + 24), g, dtype, mean=offset)
    x = xb[:, 8:8 + C]
    gam = _randn((C,), g, dtype, mean=1.0, std=0.1)
    bet = _randn((C,), g, dtype, std=0.1)
    out = _Guarded(rows, C, dtype)
    kw = {}
    fidx = torch.arange(frames, device="cuda")
    if pe != "nope":
        table = sinusoid_pe(32, C)[0].to("cuda")
        kw = dict(pe=table, tokens_per_frame=L, frames=frames)
        if pe == "pe_index":
            idx = torch.tensor([0, 1, 6, 7, 8, 9, 30, 31, 2], dtype=torch.int32, device="cuda")
            kw["pe_index"] = idx
            fidx = idx.long()
    names = _kernels(lambda: ops.layernorm(x, gam, bet, out.view, eps=1e-5, **kw), "layernorm_kernel")
    _ran(names, "layernorm_kernel")
    out.check()
    ref = F.layer_norm(x.double(), (C,), gam.double(), bet.double(), 1e-5)
    if pe != "nope":
        # the reference adds PE to the LayerNorm output rounded to the model dtype
        ref = ref.to(dtype).double().view(b, frames, L, C) + table.double()[fidx].view(1, frames, 1, C)
    bound = 2 * _floor(ref, dtype) + 1e-5
    glob, worst = _errs(out.view, ref.reshape(rows, C), b * frames)
    assert glob <= bound and worst <= 4 * bound, (glob, worst, bound)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("M,C,N,geglu", [(2048, 320, 960, False), (1024, 640, 5120, True), (777, 1280, 1280, False)])
def test_layernorm_folded_gemm_offset_rows(M, C, N, geglu, dtype):
    """stats_out (row sum / sum of squares by fp32 atomics in the producing GEMM) + the ln_stats epilogue of the
    consuming GEMM, on rows whose mean is ~10x their spread."""
    from hallo_b200 import ops
    _dev()
    g = torch.Generator(device="cuda").manual_seed(M + N + C)
    a0 = _randn((M, 320), g, dtype)
    w0 = _randn((C, 320), g, dtype, std=320 ** -0.5)
    res = _randn((M, C), g, dtype, mean=15.0, std=1.0)          # x = a0 w0^T + res: mean 15, std ~1.4
    x = torch.empty(M, C, device="cuda", dtype=dtype)
    stats = torch.zeros(M, 2, device="cuda", dtype=torch.float32)
    ops.gemm(a0, w0, x, residual=res, stats_out=stats)
    torch.cuda.synchronize()
    xd = x.double()
    assert float(xd.mean(1).min()) > 8 * float(xd.std(1).max())
    assert torch.allclose(stats[:, 0].double(), xd.sum(1), rtol=1e-4, atol=1e-2)
    assert torch.allclose(stats[:, 1].double(), (xd * xd).sum(1), rtol=1e-4, atol=1e-2)
    gamma = _randn((C,), g, dtype, mean=1.0, std=0.2)
    beta = _randn((C,), g, dtype, std=0.2)
    w = _randn((N, C), g, dtype, std=C ** -0.5)
    b = _randn((N,), g, dtype)
    ref = F.layer_norm(xd, (C,), gamma.double(), beta.double(), 1e-5) @ w.double().t() + b.double()
    if geglu:
        wi, bi = ops.pack_geglu_weight(w, b)
        ref = ref[:, :N // 2] * F.gelu(ref[:, N // 2:])
    else:
        wi, bi = w, b
    wg, colsum, bb = ops.fold_layernorm(wi, bi, gamma, beta, dtype)
    out = _Guarded(M, N // 2 if geglu else N, dtype)
    ops.gemm(x, wg, out.view, bias=bb, geglu=geglu, ln_stats=stats, ln_colsum=colsum, ln_eps=1e-5)
    torch.cuda.synchronize()
    out.check()
    glob, _ = _errs(out.view, ref, 1)
    assert glob < (3e-3 if dtype == torch.float16 else 1.2e-2), glob


# ------------------------------------------------------------------------------------------------ layout / step kernels
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_upsample_and_phase_split_exact(dtype):
    from hallo_b200 import ops
    _dev()
    n, h, w, C = 3, 10, 14, 136
    g = torch.Generator(device="cuda").manual_seed(31)
    x = _randn((n, h, w, C), g, dtype)
    up = _Guarded(n * 4 * h * w, C, dtype, gr=5, gc=0)
    _trace(lambda: ops.upsample2x(x, up.view.view(n, 2 * h, 2 * w, C)), "upsample2x_kernel")
    up.check()
    assert torch.equal(up.view.view(n, 2 * h, 2 * w, C), x.repeat_interleave(2, 1).repeat_interleave(2, 2))
    planes = _Guarded(n * h * w, C, dtype, gr=5, gc=0)
    _trace(lambda: ops.phase_split(x, planes.view.view(4 * n, h // 2, w // 2, C)), "phase_split_kernel")
    planes.check()
    ref = torch.cat([x[:, p::2, q::2] for p in range(2) for q in range(2)], 0)
    assert torch.equal(planes.view.view(4 * n, h // 2, w // 2, C), ref)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("per_half", [False, True])
def test_im2col_latent_exact(per_half, dtype):
    """Both CFG halves from one latent (per_half_latents = 0) or one latent each (1); the gather is a copy, so the
    result equals the latents rounded to the storage type, and the pad columns are zero."""
    from hallo_b200 import ops
    _dev()
    Cl, Fr, H, W, batch = 4, 3, 9, 7, 2
    g = torch.Generator(device="cuda").manual_seed(32)
    lat = torch.randn((batch if per_half else 1, Cl, Fr, H, W), generator=g, device="cuda")
    cols = _Guarded(batch * Fr * H * W, 64, dtype, gr=5, gc=0)
    _trace(lambda: ops.im2col_latent(lat, cols.view, batch=batch), "im2col_latent_kernel")
    cols.check()
    for bi in range(batch):
        lb = lat[bi if per_half else 0]
        unf = F.unfold(lb.permute(1, 0, 2, 3), 3, padding=1)                        # [F, Cl*9, HW], index c*9 + tap
        unf = unf.view(Fr, Cl, 9, H * W).permute(0, 3, 2, 1).reshape(Fr * H * W, 9 * Cl)
        blk = cols.view[bi * Fr * H * W:(bi + 1) * Fr * H * W]
        assert torch.equal(blk[:, :9 * Cl], unf.to(dtype))
        assert float(blk[:, 9 * Cl:].float().abs().max()) == 0.0


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_cfg_ddim_step_and_tokens_to_bcfhw(dtype):
    from hallo_b200 import ops
    _dev()
    Cl, Fr, H, W = 4, 5, 6, 10
    g = torch.Generator(device="cuda").manual_seed(33)
    lat = torch.randn((1, Cl, Fr, H, W), generator=g, device="cuda")
    mo_big = _randn((2 * Fr * H * W, 24), g, dtype)
    mo = mo_big[:, 8:16]                                                     # ld 24, first Cl columns used
    coef = torch.tensor([[0.0, 1.0, 0.3, 0.95], [0.6, 0.8, 0.9, 0.43]], device="cuda")
    step = torch.tensor([1], dtype=torch.int32, device="cuda")
    lat0 = lat.clone()
    v_out = torch.full_like(lat, float("nan"))
    _trace(lambda: (lat.copy_(lat0), ops.cfg_ddim_step(mo, lat, coef, step, guidance=3.5, v_out=v_out)),
           "cfg_ddim_kernel")
    half = Fr * H * W
    vu = mo[:half, :Cl].double().view(Fr, H, W, Cl).permute(3, 0, 1, 2)[None]
    vc = mo[half:, :Cl].double().view(Fr, H, W, Cl).permute(3, 0, 1, 2)[None]
    v = vu + 3.5 * (vc - vu)
    sa, sb, sap, sbp = (float(c) for c in coef[1].double())
    x0d = lat0.double()
    ref = sap * (sa * x0d - sb * v) + sbp * (sa * v + sb * x0d)
    assert _errs(lat, ref, 1)[0] < 1e-5 and _errs(v_out, v, 1)[0] < 1e-5
    out = torch.full((2, Cl, Fr, H, W), float("nan"), device="cuda")
    _trace(lambda: ops.tokens_to_bcfhw(mo, out), "nhwc_to_bcfhw_kernel")
    assert torch.equal(out, mo[:, :Cl].float().view(2, Fr, H, W, Cl).permute(0, 4, 1, 2, 3))
