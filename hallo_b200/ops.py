"""Python call wrappers over the C ABI: torch tensors in, raw pointers + sizes out.

Every function launches asynchronously on torch's current CUDA stream (so the calls can be
captured into a CUDA graph) and writes into caller-provided output tensors.
"""
from __future__ import annotations

import ctypes as C
import threading
from typing import Optional

import torch

from . import lib


# Optional per-op timing (bench.py / tools): set PROFILE = [] to collect (name, start_event, end_event).
PROFILE = None


def _timed(name_fn):
    def deco(fn):
        import functools

        @functools.wraps(fn)
        def wrapper(*args, **kwargs):
            if PROFILE is None:
                return fn(*args, **kwargs)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn(*args, **kwargs)
            e1.record()
            PROFILE.append((name_fn(*args, **kwargs), e0, e1))
            return out
        return wrapper
    return deco


class timed_region:
    """`with ops.timed_region("name"):` -- same (name, start, end) record as the decorated ops, for engine-level steps
    such as the NCCL exchanges; free when PROFILE is None."""

    def __init__(self, name: str):
        self.name = name

    def __enter__(self):
        if PROFILE is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if PROFILE is not None and hasattr(self, "e0"):
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            PROFILE.append((self.name, self.e0, e1))
        return False


def _rowmajor_ld(t: torch.Tensor) -> int:
    assert t.dim() == 2 and t.stride(1) == 1, f"need row-major 2-D view, got {tuple(t.shape)} {t.stride()}"
    return t.stride(0)


_tls = threading.local()


def gemm_workspace_bytes() -> int:
    return int(lib.load().hallo_b200_gemm_workspace_bytes())


def _bind_workspace(p, device) -> None:
    """Split-K scratch (hb_gemm_params.workspace): one zero-filled buffer per (host thread, device), allocated at the
    first eager GEMM.  Every GEMM a thread launches goes to that thread's current stream, so no two GEMMs that may run
    concurrently share it (thread-rank tests: one buffer per rank thread).  Never allocated inside a graph capture: a
    GEMM captured before any eager one simply runs unsplit."""
    pool = getattr(_tls, "gemm_ws", None)
    if pool is None:
        pool = _tls.gemm_ws = {}
    ws = pool.get(device.index)
    if ws is None:
        if torch.cuda.is_current_stream_capturing():
            return
        ws = pool[device.index] = torch.zeros(gemm_workspace_bytes(), dtype=torch.uint8, device=device)
    p.workspace, p.workspace_bytes = ws.data_ptr(), ws.numel()


@_timed(lambda a, w, out, **kw: f"gemm M{a.shape[0]} N{w.shape[0]} K{w.shape[1]}" + (" geglu" if kw.get("geglu") else ""))
def gemm(a: torch.Tensor, w: torch.Tensor, out: torch.Tensor, *, bias: Optional[torch.Tensor] = None,
         residual: Optional[torch.Tensor] = None, row_scale: Optional[torch.Tensor] = None,
         group_bias: Optional[torch.Tensor] = None, rows_per_group: int = 0, alpha: float = 1.0,
         geglu: bool = False, silu: bool = False, relu: bool = False, a2: Optional[torch.Tensor] = None,
         ln_stats: Optional[torch.Tensor] = None, ln_colsum: Optional[torch.Tensor] = None, ln_eps: float = 1e-5,
         stats_out: Optional[torch.Tensor] = None, scatter: Optional["lib.RowScatter"] = None,
         split_k: bool = True) -> torch.Tensor:
    """out[M, N(/2)] = epilogue(cat([a, a2], 1) @ w.T); see include/hallo_b200.h.  With `scatter` (row_scatter()) the
    rows go to the per-destination buffers instead of `out` (which then only supplies ldc / the shape check).
    split_k=False: no split-K workspace, so the K loop is never split and a row's result does not depend on how many
    rows share the launch (the split is only chosen for launches whose tiles fill less than half of the SMs)."""
    p = lib.GemmParams()
    p.dtype = lib.dtype_code(a.dtype)
    M, K1 = a.shape
    N, K = w.shape
    p.M, p.N, p.K = M, N, K
    p.A, p.lda = lib.ptr(a), _rowmajor_ld(a)
    if a2 is not None:
        assert a2.shape[0] == M and K1 + a2.shape[1] == K
        p.A2, p.lda2, p.K1 = lib.ptr(a2), _rowmajor_ld(a2), K1
    else:
        assert K1 == K, (K1, K)
    p.W, p.ldw = lib.ptr(w), _rowmajor_ld(w)
    p.C, p.ldc = lib.ptr(out), _rowmajor_ld(out)
    assert out.shape[0] == M and out.shape[1] == (N // 2 if geglu else N), (out.shape, M, N)
    p.bias = lib.ptr(bias)
    if group_bias is not None:
        p.group_bias, p.ld_group_bias, p.rows_per_group = lib.ptr(group_bias), _rowmajor_ld(group_bias), rows_per_group
    p.row_scale = lib.ptr(row_scale)
    if residual is not None:
        p.residual, p.ldr = lib.ptr(residual), _rowmajor_ld(residual)
    p.alpha = alpha
    p.flags = (lib.HB_EPI_GEGLU if geglu else 0) | (lib.HB_EPI_SILU if silu else 0) | (lib.HB_EPI_RELU if relu else 0)
    if ln_stats is not None:
        assert ln_stats.dtype == torch.float32 and ln_stats.numel() >= 2 * M and ln_colsum.dtype == torch.float32
        assert ln_colsum.numel() == N and ln_stats.is_contiguous() and ln_colsum.is_contiguous()
        p.ln_stats, p.ln_colsum, p.ln_eps = lib.ptr(ln_stats), lib.ptr(ln_colsum), ln_eps
    if stats_out is not None:
        assert stats_out.dtype == torch.float32 and stats_out.numel() >= 2 * M and stats_out.is_contiguous()
        p.stats_out = lib.ptr(stats_out)
    if scatter is not None:
        assert residual is None
        p.scatter = C.addressof(scatter)
    if split_k:
        _bind_workspace(p, a.device)
    lib.check(lib.load().hallo_b200_gemm(C.byref(p), lib.current_stream()), "gemm")
    return out


def row_scatter(bases, seg: int, segs_per_dest: int, seg_stride: int, row0: int) -> "lib.RowScatter":
    """hb_row_scatter: GEMM output row r -> bases[(r // seg) // segs_per_dest] at row
    ((r // seg) % segs_per_dest) * seg_stride + row0 + r % seg."""
    sc = lib.RowScatter()
    assert 1 <= len(bases) <= 16
    for i, b in enumerate(bases):
        sc.base[i] = int(b)
    sc.seg, sc.segs_per_dest, sc.seg_stride, sc.row0 = int(seg), int(segs_per_dest), int(seg_stride), int(row0)
    return sc


@_timed(lambda x, w, out, **kw: f"conv3x3 n{x.shape[0]} {x.shape[1]}x{x.shape[2]} {x.shape[3]}->{w.shape[0]}")
def conv3x3(x: torch.Tensor, w_packed: torch.Tensor, out: torch.Tensor, *, bias: Optional[torch.Tensor] = None,
            residual: Optional[torch.Tensor] = None, group_bias: Optional[torch.Tensor] = None,
            rows_per_group: int = 0, split_k: bool = True) -> torch.Tensor:
    """x: NHWC [n, h, w, cin]; w_packed: [cout, 9*cin] ([cout][kh][kw][cin]); out: [n*h*w, cout].  split_k: see gemm."""
    n, h, w_, cin = x.shape
    assert x.is_contiguous() or (x.stride(3) == 1 and x.stride(1) == w_ * x.stride(2) and x.stride(0) == h * x.stride(1))
    p = lib.GemmParams()
    p.dtype = lib.dtype_code(x.dtype)
    p.M, p.N, p.K = n * h * w_, w_packed.shape[0], w_packed.shape[1]
    assert p.K == 9 * cin
    p.A, p.lda = lib.ptr(x), (cin if x.is_contiguous() else x.stride(2))
    p.W, p.ldw = lib.ptr(w_packed), _rowmajor_ld(w_packed)
    p.C, p.ldc = lib.ptr(out), _rowmajor_ld(out)
    p.bias = lib.ptr(bias)
    if group_bias is not None:
        p.group_bias, p.ld_group_bias, p.rows_per_group = lib.ptr(group_bias), _rowmajor_ld(group_bias), rows_per_group
    if residual is not None:
        p.residual, p.ldr = lib.ptr(residual), _rowmajor_ld(residual)
    p.alpha = 1.0
    p.conv3x3 = 1
    p.img_n, p.img_h, p.img_w = n, h, w_
    if split_k:
        _bind_workspace(p, x.device)
    lib.check(lib.load().hallo_b200_gemm(C.byref(p), lib.current_stream()), "conv3x3")
    return out


def pack_conv3x3_weight(w: torch.Tensor) -> torch.Tensor:
    """torch conv weight [cout, cin, 3, 3] -> [cout, 9*cin] with k = (kh*3 + kw)*cin + c."""
    cout, cin, kh, kw = w.shape
    assert kh == 3 and kw == 3
    return w.permute(0, 2, 3, 1).reshape(cout, 9 * cin).contiguous()


def pack_stem_weight(w: torch.Tensor) -> torch.Tensor:
    """3x3 conv weight over a few input channels [cout, cl, 3, 3] -> [cout, 64] (k = tap*cl + c, zero columns from
    9*cl on): the weight of the GEMM that follows im2col_latent / im2col_affine."""
    cout, cl = w.shape[0], w.shape[1]
    assert 9 * cl <= 64 and w.shape[2:] == (3, 3)
    wi = torch.zeros(cout, 64, dtype=w.dtype, device=w.device)
    wi[:, :9 * cl] = w.permute(0, 2, 3, 1).reshape(cout, 9 * cl)
    return wi


def pad_rows(x: torch.Tensor, rows: int) -> torch.Tensor:
    """x [r, ...] -> [rows, ...] with zero rows appended (a narrow output head padded to the GEMM's N % 8 == 0)."""
    out = torch.zeros((rows,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    out[:x.shape[0]] = x
    return out


def pack_geglu_weight(w: torch.Tensor, b: Optional[torch.Tensor]):
    """FeedForward.net[0].proj ([8C, C]: value rows then gate rows) -> rows interleaved (v0,g0,v1,g1..)."""
    n2, k = w.shape
    half = n2 // 2
    wi = torch.stack([w[:half], w[half:]], dim=1).reshape(n2, k).contiguous()
    bi = None if b is None else torch.stack([b[:half], b[half:]], dim=1).reshape(n2).contiguous()
    return wi, bi


@_timed(lambda q, k, v, out, **kw: f"attention C{q.shape[1]} L{kw['L']} rows{q.shape[0]}" + (" +ref" if kw.get("ref_index") is not None else ""))
def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, *, heads: int, L: int,
              kref: Optional[torch.Tensor] = None, vref: Optional[torch.Tensor] = None,
              ref_index: Optional[torch.Tensor] = None) -> torch.Tensor:
    """q/k/v/out: [frames*L, C] row-major views (column slices of a fused buffer are fine).
    kref/vref: [ref_frames*L, C]; ref_index: int32 [frames] device tensor (-1 = no reference keys)."""
    p = lib.AttentionParams()
    p.dtype = lib.dtype_code(q.dtype)
    rows, Cq = q.shape
    assert rows % L == 0 and Cq % heads == 0
    p.head_dim, p.heads, p.L, p.frames = Cq // heads, heads, L, rows // L
    p.Q, p.ldq = lib.ptr(q), _rowmajor_ld(q)
    p.K, p.ldk = lib.ptr(k), _rowmajor_ld(k)
    p.V, p.ldv = lib.ptr(v), _rowmajor_ld(v)
    p.O, p.ldo = lib.ptr(out), _rowmajor_ld(out)
    if ref_index is not None:
        assert ref_index.dtype == torch.int32 and ref_index.numel() == p.frames and ref_index.is_cuda
        p.Kref, p.ldkref = lib.ptr(kref), _rowmajor_ld(kref)
        p.Vref, p.ldvref = lib.ptr(vref), _rowmajor_ld(vref)
        p.ref_frames = kref.shape[0] // L
        p.ref_index = lib.ptr(ref_index)
    lib.check(lib.load().hallo_b200_attention(C.byref(p), lib.current_stream()), "attention")
    return out


# ----------------------------------------------------------------------------- aux kernels (csrc/aux.cu)
def _i(v) -> C.c_int:
    return C.c_int(int(v))


@_timed(lambda x, *a, **kw: f"layernorm C{x.shape[1]} rows{x.shape[0]}")
def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, out: torch.Tensor, *, eps: float = 1e-5,
              pe: Optional[torch.Tensor] = None, pe_index: Optional[torch.Tensor] = None, tokens_per_frame: int = 0,
              frames: int = 0) -> torch.Tensor:
    rows, Cc = x.shape
    if pe is not None:
        assert pe.dtype == torch.float32 and pe.is_contiguous() and pe.shape[-1] == Cc
    lib.check(lib.load().hallo_b200_layernorm(
        _i(lib.dtype_code(x.dtype)), C.c_void_p(lib.ptr(x)), C.c_int64(_rowmajor_ld(x)), C.c_void_p(lib.ptr(out)),
        C.c_int64(_rowmajor_ld(out)), C.c_void_p(lib.ptr(gamma)), C.c_void_p(lib.ptr(beta)), _i(rows), _i(Cc),
        C.c_float(eps), C.c_void_p(lib.ptr(pe)), C.c_void_p(lib.ptr(pe_index)), _i(tokens_per_frame), _i(frames),
        lib.current_stream()), "layernorm")
    return out


def gn_workspace_floats(n_frames: int, hw: int, groups: int, channels: int) -> int:
    """fp32 elements hallo_b200_groupnorm needs: per-chunk (64 pixels) group sums + per-channel scale / shift."""
    return 2 * n_frames * (groups * ((hw + 63) // 64) + channels)


@_timed(lambda x1, *a, **kw: f"groupnorm C{x1.shape[1] + (0 if kw.get('x2') is None else kw['x2'].shape[1])} rows{x1.shape[0]}")
def groupnorm(x1: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, out: torch.Tensor, stats_ws: torch.Tensor, *,
              n_frames: int, hw: int, groups: int = 32, eps: float = 1e-5, silu: bool = False,
              x2: Optional[torch.Tensor] = None, fpb_in: int = 0, fpb_out: int = 0, frame_off: int = 0) -> torch.Tensor:
    """x1: [n_frames*hw, C1] contiguous, x2: optional [n_frames*hw, C2]; out: [*, C1+C2] contiguous."""
    assert x1.is_contiguous() and (x2 is None or x2.is_contiguous()) and out.is_contiguous()
    C1 = x1.shape[1]
    C2 = 0 if x2 is None else x2.shape[1]
    assert stats_ws.dtype == torch.float32 and stats_ws.numel() >= gn_workspace_floats(n_frames, hw, groups, C1 + C2)
    lib.check(lib.load().hallo_b200_groupnorm(
        _i(lib.dtype_code(x1.dtype)), C.c_void_p(lib.ptr(x1)), _i(C1), C.c_void_p(lib.ptr(x2)), _i(C2), _i(n_frames),
        _i(hw), _i(groups), C.c_void_p(lib.ptr(gamma)), C.c_void_p(lib.ptr(beta)), C.c_float(eps), _i(1 if silu else 0),
        C.c_void_p(lib.ptr(out)), C.c_void_p(lib.ptr(stats_ws)), _i(fpb_in), _i(fpb_out), _i(frame_off),
        lib.current_stream()), "groupnorm")
    return out


@_timed(lambda x1, *a, **kw: f"groupnorm_scatter C{x1.shape[1]} rows{x1.shape[0]}")
def groupnorm_scatter(x1: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, out_addrs, stats_ws: torch.Tensor, *,
                      n_frames: int, hw: int, groups: int = 32, eps: float = 1e-5, fpb_in: int = 0, fpb_out: int = 0,
                      frame_off: int = 0) -> None:
    """GroupNorm whose rows are stored by pixel slice into `out_addrs` (one device address per destination rank):
    pixel p of output frame n_out -> out_addrs[p // seg] + ((n_out * seg + p % seg) * C), seg = hw // len(out_addrs)."""
    assert x1.is_contiguous() and hw % len(out_addrs) == 0
    C1 = x1.shape[1]
    assert stats_ws.dtype == torch.float32 and stats_ws.numel() >= gn_workspace_floats(n_frames, hw, groups, C1)
    arr = (C.c_void_p * len(out_addrs))(*[C.c_void_p(int(a)) for a in out_addrs])
    lib.check(lib.load().hallo_b200_groupnorm_scatter(
        _i(lib.dtype_code(x1.dtype)), C.c_void_p(lib.ptr(x1)), _i(C1), _i(n_frames), _i(hw), _i(groups),
        C.c_void_p(lib.ptr(gamma)), C.c_void_p(lib.ptr(beta)), C.c_float(eps), arr, _i(len(out_addrs)),
        C.c_void_p(lib.ptr(stats_ws)), _i(fpb_in), _i(fpb_out), _i(frame_off), lib.current_stream()), "groupnorm_scatter")


@_timed(lambda a, *r, **kw: f"add n{a.numel()}")
def add(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    assert a.is_contiguous() and b.is_contiguous() and out.is_contiguous() and a.numel() == b.numel() == out.numel()
    lib.check(lib.load().hallo_b200_add(_i(lib.dtype_code(a.dtype)), C.c_void_p(lib.ptr(a)), C.c_void_p(lib.ptr(b)),
                                        C.c_void_p(lib.ptr(out)), C.c_int64(a.numel()), lib.current_stream()), "add")
    return out


@_timed(lambda q, *a, **kw: f"cross_attention keys{kw['n_keys']} d{kw['head_dim']} rows{q.shape[0]}")
def cross_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, *, frames: int, tokens: int,
                    heads: int, head_dim: int, n_keys: int, kv_frame_div: int = 1, regions: int = 1,
                    q_region_stride: int = 0, kv_region_stride: int = 0, o_region_stride: int = 0) -> torch.Tensor:
    """q/out: [frames*tokens, ld]; k/v: [kv_frames*n_keys, ldkv] (same ld for both)."""
    assert _rowmajor_ld(k) == _rowmajor_ld(v)
    lib.check(lib.load().hallo_b200_cross_attention(
        _i(lib.dtype_code(q.dtype)), C.c_void_p(lib.ptr(q)), C.c_int64(_rowmajor_ld(q)), _i(q_region_stride),
        C.c_void_p(lib.ptr(k)), C.c_void_p(lib.ptr(v)), C.c_int64(_rowmajor_ld(k)), _i(kv_region_stride),
        C.c_void_p(lib.ptr(out)), C.c_int64(_rowmajor_ld(out)), _i(o_region_stride), _i(frames), _i(tokens), _i(heads),
        _i(head_dim), _i(n_keys), _i(kv_frame_div), _i(regions), lib.current_stream()), "cross_attention")
    return out


@_timed(lambda q, k, v, out, **kw: f"temporal_attention C{out.shape[1]} rows{q.shape[0]} fk{kw.get('fk')}")
def temporal_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, *, batch: int, fq: int,
                       fk: int, tokens: int, heads: int) -> torch.Tensor:
    """q/out: [batch*fq*tokens, ld]; k/v: [batch*fk*tokens, ldkv]."""
    assert _rowmajor_ld(k) == _rowmajor_ld(v)
    head_dim = out.shape[1] // heads
    lib.check(lib.load().hallo_b200_temporal_attention(
        _i(lib.dtype_code(q.dtype)), C.c_void_p(lib.ptr(q)), C.c_int64(_rowmajor_ld(q)), C.c_void_p(lib.ptr(k)),
        C.c_void_p(lib.ptr(v)), C.c_int64(_rowmajor_ld(k)), C.c_void_p(lib.ptr(out)), C.c_int64(_rowmajor_ld(out)),
        _i(batch), _i(fq), _i(fk), _i(tokens), _i(heads), _i(head_dim), lib.current_stream()), "temporal_attention")
    return out


@_timed(lambda x, *a, **kw: f"upsample2x C{x.shape[3]} {x.shape[1]}")
def upsample2x(x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    n, h, w, c = x.shape
    assert x.is_contiguous() and out.is_contiguous() and out.numel() == 4 * x.numel()
    lib.check(lib.load().hallo_b200_upsample2x(_i(lib.dtype_code(x.dtype)), C.c_void_p(lib.ptr(x)),
                                               C.c_void_p(lib.ptr(out)), _i(n), _i(h), _i(w), _i(c),
                                               lib.current_stream()), "upsample2x")
    return out


@_timed(lambda x, *a, **kw: f"phase_split C{x.shape[3]} {x.shape[1]}")
def phase_split(x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    n, h, w, c = x.shape
    assert x.is_contiguous() and out.is_contiguous() and out.numel() == x.numel()
    lib.check(lib.load().hallo_b200_phase_split(_i(lib.dtype_code(x.dtype)), C.c_void_p(lib.ptr(x)),
                                                C.c_void_p(lib.ptr(out)), _i(n), _i(h), _i(w), _i(c),
                                                lib.current_stream()), "phase_split")
    return out


@_timed(lambda x, w, *a, **kw: f"conv3x3s2 {x.shape[3]}->{w.shape[0]} {kw['ho']}")
def conv3x3_stride2(x_planes: torch.Tensor, w_packed: torch.Tensor, out: torch.Tensor, *, n: int, ho: int, wo: int,
                    bias: Optional[torch.Tensor] = None, pad_end: bool = False, split_k: bool = True) -> torch.Tensor:
    """x_planes: phase planes [4*n, ho, wo, cin] from phase_split; out: [n*ho*wo, cout].
    pad_end=False: zero padding 1 on every side (Downsample3D); True: zero padding (0, 1) on each axis, i.e. only after
    the last row / column (diffusers Downsample2D(padding=0), the VAE encoder).  split_k: see gemm."""
    cin = x_planes.shape[-1]
    assert x_planes.is_contiguous() and x_planes.shape[0] == 4 * n
    p = lib.GemmParams()
    p.dtype = lib.dtype_code(x_planes.dtype)
    p.M, p.N, p.K = n * ho * wo, w_packed.shape[0], w_packed.shape[1]
    assert p.K == 9 * cin
    p.A, p.lda = lib.ptr(x_planes), cin
    p.W, p.ldw = lib.ptr(w_packed), _rowmajor_ld(w_packed)
    p.C, p.ldc = lib.ptr(out), _rowmajor_ld(out)
    p.bias = lib.ptr(bias)
    p.alpha = 1.0
    p.conv3x3 = 3 if pad_end else 2
    p.img_n, p.img_h, p.img_w = n, ho, wo
    if split_k:
        _bind_workspace(p, x_planes.device)
    lib.check(lib.load().hallo_b200_gemm(C.byref(p), lib.current_stream()), "conv3x3_stride2")
    return out


@_timed(lambda *a, **kw: "im2col_latent")
def im2col_latent(latents: torch.Tensor, out: torch.Tensor, *, batch: int) -> torch.Tensor:
    """latents: fp32 [1 or batch, Cl, F, H, W] contiguous; out: [batch*F*H*W, 64]."""
    lb, cl, f, h, w = latents.shape
    assert latents.dtype == torch.float32 and latents.is_contiguous() and out.is_contiguous()
    assert lb in (1, batch)
    lib.check(lib.load().hallo_b200_im2col_latent(_i(lib.dtype_code(out.dtype)), C.c_void_p(lib.ptr(latents)),
                                                  C.c_void_p(lib.ptr(out)), _i(batch), _i(cl), _i(f), _i(h), _i(w),
                                                  _i(1 if (lb == batch and batch > 1) else 0),
                                                  lib.current_stream()), "im2col_latent")
    return out


@_timed(lambda x, out, **kw: f"im2col_affine Cl{x.shape[1]} rows{out.shape[0]}")
def im2col_affine(x: torch.Tensor, out: torch.Tensor, *, mat: Optional[torch.Tensor] = None,
                  bias: Optional[torch.Tensor] = None, scale: float = 1.0) -> torch.Tensor:
    """x: fp32 NCHW [n, cl, h, w] contiguous, 9*cl <= 64; out: [n*h*w, 64].  Column (kh*3 + kw)*cl + c of row (n, y, x)
    holds (mat @ (scale * pixel) + bias)[c] of pixel (y + kh - 1, x + kw - 1), 0 outside the image.  mat: fp32 [cl, cl]
    or None (identity); bias: fp32 [cl] or None."""
    n, cl, h, w = x.shape
    assert x.dtype == torch.float32 and x.is_contiguous() and out.is_contiguous() and out.shape == (n * h * w, 64)
    for t, shape in ((mat, (cl, cl)), (bias, (cl,))):
        assert t is None or (t.dtype == torch.float32 and t.is_contiguous() and tuple(t.shape) == shape)
    lib.check(lib.load().hallo_b200_im2col_affine(_i(lib.dtype_code(out.dtype)), C.c_void_p(lib.ptr(x)),
                                                  C.c_void_p(lib.ptr(out)), _i(n), _i(cl), _i(h), _i(w),
                                                  C.c_void_p(lib.ptr(mat)), C.c_void_p(lib.ptr(bias)),
                                                  C.c_float(scale), lib.current_stream()), "im2col_affine")
    return out


@_timed(lambda *a, **kw: "timestep_embed")
def timestep_embed(t_table: torch.Tensor, step: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    rows, dim = out.shape
    assert t_table.dtype == torch.float32 and step.dtype == torch.int32 and out.is_contiguous()
    lib.check(lib.load().hallo_b200_timestep_embed(_i(lib.dtype_code(out.dtype)), C.c_void_p(lib.ptr(t_table)),
                                                   C.c_void_p(lib.ptr(step)), C.c_void_p(lib.ptr(out)), _i(rows),
                                                   _i(dim), lib.current_stream()), "timestep_embed")
    return out


@_timed(lambda *a, **kw: "cfg_ddim_step")
def cfg_ddim_step(model_out: torch.Tensor, latents: torch.Tensor, coef: torch.Tensor, step: torch.Tensor, *,
                  guidance: float, v_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """model_out: [2*F*HW, ld] tokens (uncond rows then cond rows); latents: fp32 [1, Cl, F, H, W] updated in place."""
    _, cl, f, h, w = latents.shape
    assert latents.dtype == torch.float32 and latents.is_contiguous() and coef.dtype == torch.float32
    lib.check(lib.load().hallo_b200_cfg_ddim_step(
        _i(lib.dtype_code(model_out.dtype)), C.c_void_p(lib.ptr(model_out)), C.c_int64(_rowmajor_ld(model_out)),
        C.c_void_p(lib.ptr(latents)), C.c_void_p(lib.ptr(coef)), C.c_void_p(lib.ptr(step)), C.c_float(guidance), _i(cl),
        _i(f), _i(h * w), C.c_void_p(lib.ptr(v_out)), lib.current_stream()), "cfg_ddim_step")
    return latents


def advance_step(step: torch.Tensor, n_steps: int) -> None:
    lib.check(lib.load().hallo_b200_advance_step(C.c_void_p(lib.ptr(step)), _i(n_steps), lib.current_stream()),
              "advance_step")


@_timed(lambda *a, **kw: "tokens_to_bcfhw")
def tokens_to_bcfhw(x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """x: [B*F*HW, ld] tokens (first C columns used); out: fp32 [B, C, F, H, W]."""
    b, c, f, h, w = out.shape
    assert out.dtype == torch.float32 and out.is_contiguous()
    lib.check(lib.load().hallo_b200_tokens_to_bcfhw(_i(lib.dtype_code(x.dtype)), C.c_void_p(lib.ptr(x)),
                                                    C.c_int64(_rowmajor_ld(x)), C.c_void_p(lib.ptr(out)), _i(b), _i(c),
                                                    _i(f), _i(h * w), lib.current_stream()), "tokens_to_bcfhw")
    return out


def fold_layernorm(w: torch.Tensor, b: Optional[torch.Tensor], gamma: torch.Tensor, beta: torch.Tensor, dtype):
    """nn.LayerNorm(gamma, beta) -> nn.Linear(w, b) folded for hallo_b200_gemm's ln_* epilogue.
    Returns (W*diag(gamma) in `dtype`, fp32 row sums of that packed matrix, W beta + b in `dtype`)."""
    wf = w.float()
    wg = (wf * gamma.float()[None, :]).to(dtype)
    colsum = wg.float().sum(dim=1).contiguous()
    bb = wf @ beta.float()
    if b is not None:
        bb = bb + b.float()
    return wg.contiguous(), colsum, bb.to(dtype).contiguous()
