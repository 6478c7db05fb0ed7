"""hallo_b200_attention (attn_tc_kernel at head dims 40 / 80 / 160, attn_wide_kernel at 512) over the shape matrix of
tests/attn_cases.py: L from 1 to 9216, one or eight heads, up to 32 frames, every reference-key layout.

- Routing: inputs built so that every query has exactly one winning key (tests/attn_cases.py); O must equal V[target]
  bit for bit.  A tail mask, a segment or frame read from the wrong place, or a running max rescaled inconsistently
  moves whole rows and shows up exactly, whatever the tolerance.
- Temperature: each query sees a winner and a runner-up G log2 units below it; O / V[runner-up] must be the softmax
  weight 2^-G / (1 + 2^-G) to within the rounding of P and O.  Catches a wrong softmax scale.
- Numerics: random inputs in five regimes against a float64 softmax of the rounded inputs, per (frame, head,
  128-query tile) and globally, with the rounding floor of the exact output printed beside them.
- Guards: Q / K / V (and Kref / Vref) are column slices of one buffer [pad | Q | pad | K | pad | V | pad] whose pads
  and rows past the last frame are NaN; O is a view into a NaN buffer with guard rows and columns.
- Invariance: a repeated call, pdl on / off, and each frame run alone give the same bits.
- Path: a torch.profiler trace, taken in a child process, shows the kernel instantiation that was expected."""
import contextlib
import math
import re

import pytest
import torch

import attn_cases as ac

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["f16", "bf16"]
# global relative L2 bounds the kernels met before these tests; a (frame, head, 128-query tile) may reach twice that
TOL = {torch.float16: 4e-3, torch.bfloat16: 2e-2}
PAD = 64          # NaN columns around each of Q / K / V in the fused input buffer: a whole 64-column TMA box
TAIL_ROWS = 80    # NaN rows past the last frame


@pytest.fixture(scope="module", autouse=True)
def _release_cached_memory():
    """Hand the allocator's cached blocks back once this module is done, so its large reference buffers do not stay
    reserved for the rest of the suite."""
    yield
    if torch.cuda.is_available():
        torch.cuda.synchronize()
        torch.cuda.empty_cache()


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@contextlib.contextmanager
def _option(name, value):
    from hallo_b200 import lib
    was = lib.get_option(name)
    lib.set_option(name, value)
    try:
        yield
    finally:
        lib.set_option(name, was)


def _kernels(fn, expect, tries=3):
    """Names of the CUDA kernels fn() launched (torch.profiler); retried when a short trace dropped `expect`."""
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


class _Guarded:
    """A NaN-filled buffer with `gr` guard rows above and below and `gc` guard columns left and right of the
    [rows, cols] output view."""

    def __init__(self, rows, cols, dtype, gr=3, gc=8):
        self.big = torch.full((rows + 2 * gr, cols + 2 * gc), float("nan"), device="cuda", dtype=dtype)
        self.view = self.big[gr:gr + rows, gc:gc + cols]
        self.mask = torch.zeros(self.big.shape, dtype=torch.bool, device="cuda")
        self.mask[gr:gr + rows, gc:gc + cols] = True

    def check(self):
        """Guard region bit-identical (still NaN); every element of the output view finite."""
        _assert_all_nan_bits(self.big[~self.mask])
        assert torch.isfinite(self.big[self.mask].float()).all(), "output element left unwritten (still NaN)"


def _assert_all_nan_bits(t):
    nan = torch.full((1,), float("nan"), dtype=t.dtype, device=t.device).view(torch.int16)
    bits = t.reshape(-1).view(torch.int16)
    assert torch.equal(bits, nan.expand_as(bits)), "a kernel wrote outside its output"


def _fused(parts, dtype):
    """Column slices of one buffer [pad | parts[0] | pad | parts[1] | ... | pad], NaN in the pads and in TAIL_ROWS
    rows past the last frame."""
    rows, C = parts[0].shape
    big = torch.full((rows + TAIL_ROWS, len(parts) * (C + PAD) + PAD), float("nan"), device="cuda", dtype=dtype)
    views = []
    for i, t in enumerate(parts):
        c0 = PAD + i * (C + PAD)
        big[:rows, c0:c0 + C] = t.to(device="cuda", dtype=dtype)
        views.append(big[:rows, c0:c0 + C])
    return views


def _inputs(c, dtype, q, k, v, kref, vref):
    qv, kv, vv = _fused([q, k, v], dtype)
    kr = vr = ridx = None
    if c.ridx is not None:
        kr, vr = _fused([kref, vref], dtype)
        ridx = torch.tensor(c.ridx, dtype=torch.int32, device="cuda")
    return qv, kv, vv, kr, vr, ridx


def _attend(c, q, k, v, kr, vr, ridx, out):
    from hallo_b200 import ops
    ops.attention(q, k, v, out, heads=c.heads, L=c.L, kref=kr, vref=vr, ref_index=ridx)


def _run_guarded(c, dtype, ins):
    out = _Guarded(c.frames * c.L, c.heads * c.d, dtype)
    _attend(c, *ins, out.view)
    torch.cuda.synchronize()
    out.check()
    return out.view.clone()


# ------------------------------------------------------------------------------------------------------ routing
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("c", ac.routing_cases(), ids=ac.case_id)
def test_routing_exact(c, dtype):
    _dev()
    inp = ac.routing_inputs(c)
    got = _run_guarded(c, dtype, _inputs(c, dtype, inp["q"], inp["k"], inp["v"], inp["kref"], inp["vref"]))
    want = inp["expect"].to("cuda", dtype)
    bad = (got.view(torch.int16) != want.view(torch.int16)).view(c.frames, c.L, c.heads, c.d).any(-1)
    if bad.any():
        f, i, h = (int(x) for x in bad.nonzero()[0])
        t = int(inp["target"][f, h, i])
        pytest.fail(f"{int(bad.sum())} of {bad.numel()} (frame, query, head) rows differ from V[target]; first: frame "
                    f"{f} query {i} head {h} target key {t} ({'reference' if t >= c.L else 'own'} segment)")


# -------------------------------------------------------------------------------------------------- temperature
_PAIRS = [(0, 1), (63, 64), (64, 63), (199, 0), (127, 128), (198, 199), (5, 192), (192, 5)]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("d", [40, 80, 160, 512])
def test_softmax_temperature(d, dtype):
    """Each (frame, head) has a winner key j0 (raw score 0), a runner-up j1 (raw score -a) and 198 keys at -64 a; the
    query row sets a so that the gap is G = a d^-0.5 log2 e, swept over [0.25, 13] in fp16 (P stays a normal fp16)
    and [0.25, 60] in bf16.  V is 0 except at j1, so O / V[j1] = 2^-G / (1 + 2^-G + 198 * 2^-64G).  The pairs put j1
    before and after j0, across a tile boundary and in the last partial tile.  A 0.1 % error in the softmax scale moves
    the largest-G rows by G ln 2 / 1000: 0.9 % (fp16) and 4 % (bf16), several times the tolerance."""
    _dev()
    L, H = 200, (8 if d < 512 else 1)
    F = len(_PAIRS) // H
    C = H * d
    scale = ac.LOG2E / math.sqrt(d)
    gmax = 13.0 if dtype == torch.float16 else 60.0
    G = torch.linspace(0.25, gmax, L, dtype=torch.float64)
    a = (G / scale).to(dtype).double()                       # the query value as stored
    G = a * scale
    q = torch.zeros(F, L, H, d, dtype=torch.float64)
    k = torch.zeros(F, L, H, d, dtype=torch.float64)
    v = torch.zeros(F, L, H, d, dtype=torch.float64)
    vals = (64 + torch.arange(d, dtype=torch.float64) % 64) / 64          # [1, 2), exact
    for f in range(F):
        for h in range(H):
            j0, j1 = _PAIRS[f * H + h]
            col = (7 * h + 3) % d
            q[f, :, h, col] = a if f % 2 == 0 else a.flip(0)
            k[f, :, h, col] = -64.0
            k[f, j0, h, col] = 0.0
            k[f, j1, h, col] = -1.0
            v[f, j1, h] = vals.roll(h)
    c = ac.Case(d, H, L, F, 0, None)
    ins = _inputs(c, dtype, *(t.reshape(F * L, C) for t in (q, k, v)), None, None)
    got = _run_guarded(c, dtype, ins).double().view(F, L, H, d)
    w = torch.exp2(-G) / (1 + torch.exp2(-G) + (L - 2) * torch.exp2(-64 * G))
    worst, where = 0.0, None
    for f in range(F):
        wf = (w if f % 2 == 0 else w.flip(0)).to("cuda")
        for h in range(H):
            j1 = _PAIRS[f * H + h][1]
            ratio = got[f, :, h] / (v[f, j1, h].to("cuda") * wf[:, None])
            err = (ratio - 1).abs().max(1).values
            i = int(err.argmax())
            if float(err[i]) > worst:
                worst, where = float(err[i]), (f, h, i)
    # P is rounded to the storage type, O is rounded again: 3 units of roundoff leave room for ex2.approx
    tol = 3 * (2.0 ** -11 if dtype == torch.float16 else 2.0 ** -8)
    print(f"ATTN-TEMP d{d} {DT_IDS[DTYPES.index(dtype)]}: worst |O / (w V) - 1| = {worst:.2e} (tol {tol:.2e}) at "
          f"(frame, head, row) {where}")
    assert worst <= tol, (worst, where)


# ----------------------------------------------------------------------------------------------------- numerics
def _regime(i, c):
    regimes = ["normal", "peaked", "offset"] + (["ref_hi", "ref_lo"] if c.ridx is not None else [])
    return regimes[i % len(regimes)]


def _numeric_inputs(c, regime, seed):
    """float32 inputs on the device: N(0, 1); peaked (q x 4); a shared column adding 64 * 64 = 4096 to every raw score
    (offset); reference keys x 2 or x 0.25 (ref_hi / ref_lo)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = c.heads * c.d
    R = c.ref_frames
    q, k, v = (torch.randn(c.frames * c.L, C, generator=g, device="cuda") for _ in range(3))
    kref = vref = None
    if R:
        kref, vref = (torch.randn(R * c.L, C, generator=g, device="cuda") for _ in range(2))
    if regime == "peaked":
        q *= 4
    elif regime == "offset":
        for t in (q, k, kref):
            if t is not None:
                t.view(t.shape[0], c.heads, c.d)[:, :, 0] = 64.0
    elif regime == "ref_hi":
        kref *= 2
    elif regime == "ref_lo":
        kref *= 0.25
    return q, k, v, kref, vref


def _reference(c, ins, rows):
    """float64 softmax(Q K^T / sqrt d) V of the rounded inputs for query rows `rows` of every frame:
    [frames, n, heads, d]."""
    q, k, v, kr, vr, _ = ins
    F, L, H, d = c.frames, c.L, c.heads, c.d
    out = torch.empty(F, len(rows), H, d, dtype=torch.float64, device="cuda")
    for f in range(F):
        qf = q.view(F, L, H, d)[f, rows].double()
        kf, vf = k.view(F, L, H, d)[f].double(), v.view(F, L, H, d)[f].double()
        r = -1 if c.ridx is None else c.ridx[f]
        if r >= 0:
            kf = torch.cat([kf, kr.view(c.ref_frames, L, H, d)[r].double()])
            vf = torch.cat([vf, vr.view(c.ref_frames, L, H, d)[r].double()])
        p = torch.softmax(torch.einsum("nhd,khd->hnk", qf, kf) / math.sqrt(d), -1)
        out[f] = torch.einsum("hnk,khd->nhd", p, vf)
    return out


def _tile_errors(got, ref, rows):
    """(global rel L2, worst rel L2 over (frame, head, 128-query tile)) of got against ref, both [F, n, H, d]."""
    e2 = (got - ref).pow(2).sum(-1)
    r2 = ref.pow(2).sum(-1)
    tiles = torch.as_tensor(rows // ac.QT, device=got.device)
    T = int(tiles.max()) + 1
    E = torch.zeros(got.shape[0], T, got.shape[2], dtype=torch.float64, device=got.device).index_add_(1, tiles, e2)
    Rr = torch.zeros_like(E).index_add_(1, tiles, r2)
    has = Rr > 0
    worst = float((E[has] / Rr[has]).sqrt().max())
    return float((e2.sum() / r2.sum()).sqrt()), worst


_NUM_CASES = [pytest.param(i, c, id=ac.case_id(c)) for i, c in enumerate(ac.self_attention_cases())]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("i,c", _NUM_CASES)
def test_numerics_per_tile(i, c, dtype):
    _dev()
    regime = _regime(i, c)
    ins = _inputs(c, dtype, *_numeric_inputs(c, regime, seed=1000 * i + c.d))
    got = _run_guarded(c, dtype, ins)
    rows = ac.sample_rows(c.L, seed=i)
    rows_t = torch.as_tensor(rows, device="cuda")
    ref = _reference(c, ins, rows_t)
    got = got.view(c.frames, c.L, c.heads, c.d)[:, rows_t].double()
    glob, worst = _tile_errors(got, ref, rows)
    fglob, fworst = _tile_errors(ref.to(dtype).double(), ref, rows)
    bound = TOL[dtype]
    print(f"ATTN-NUM {ac.case_id(c)} {DT_IDS[DTYPES.index(dtype)]} {regime}: global {glob:.2e} worst tile {worst:.2e} "
          f"| floor global {fglob:.2e} worst tile {fworst:.2e}")
    assert glob < bound and worst < 2 * bound, (glob, worst)


# --------------------------------------------------------------------------------------------------- invariance
_INV_CASES = [ac.Case(40, 8, 200, 6, 3, [2, 0, 1, -1, 2, 0]), ac.Case(80, 8, 65, 5, 2, [-1, -1, 0, 1, 0]),
              ac.Case(160, 1, 1024, 2, 1, [-1, 0]), ac.Case(512, 1, 65, 3, 0, None)]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("c", _INV_CASES, ids=ac.case_id)
def test_bitwise_invariance(c, dtype):
    """A repeated call, the same call with programmatic dependent launch, and every frame run alone with its own
    ref_index entry all give the bits of the first call."""
    _dev()
    ins = _inputs(c, dtype, *_numeric_inputs(c, "normal", seed=7 + c.L))
    q, k, v, kr, vr, ridx = ins
    first = _run_guarded(c, dtype, ins)
    assert torch.equal(first.view(torch.int16), _run_guarded(c, dtype, ins).view(torch.int16)), "repeat"
    with _option("pdl", 1):
        pdl = _run_guarded(c, dtype, ins)
    assert torch.equal(first.view(torch.int16), pdl.view(torch.int16)), "pdl"
    L = c.L
    one = c._replace(frames=1, ridx=None if c.ridx is None else [c.ridx[0]])
    for n in range(c.frames):
        sl = slice(n * L, (n + 1) * L)
        r1 = None if ridx is None else ridx[n:n + 1].clone()
        got = _run_guarded(one, dtype, (q[sl], k[sl], v[sl], kr, vr, r1))
        assert torch.equal(first[sl].view(torch.int16), got.view(torch.int16)), f"frame {n} alone"


# --------------------------------------------------------------------------------------------------------- path
def _trace_paths():
    """{"<d>-<dtype>": names of the CUDA kernels one hallo_b200_attention call launched}, d in 40 / 80 / 160 / 512."""
    out = {}
    for d in (40, 80, 160, 512):
        heads = 8 if d < 512 else 1
        c = ac.Case(d, heads, 130, 2, 2 if d < 512 else 0, [-1, 1] if d < 512 else None)
        for dtype, dt in zip(DTYPES, DT_IDS):
            ins = _inputs(c, dtype, *_numeric_inputs(c, "normal", seed=d))
            o = torch.empty(c.frames * c.L, heads * d, device="cuda", dtype=dtype)
            out[f"{d}-{dt}"] = _kernels(lambda: _attend(c, *ins, o), "attn_")
    return out


@pytest.fixture(scope="module")
def path_traces():
    """_trace_paths() run in a child process.  A torch.profiler session in the test process left the later sessions of
    tests/test_kernel_paths_gpu.py without any CUDA kernel record (seen on an H100 with CUDA-graph tests run in
    between), so the profiler is kept out of the process the rest of the suite runs in."""
    import json
    import os
    import subprocess
    import sys
    _dev()
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import json, sys; sys.path[:0] = [{here!r}, {os.path.dirname(here)!r}]; "
            "import test_attention_paths_gpu as t; print(json.dumps(t._trace_paths()))")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("d", [40, 80, 160, 512])
def test_kernel_path(d, dtype, path_traces):
    _dev()
    names = path_traces[f"{d}-{DT_IDS[DTYPES.index(dtype)]}"]
    tname = "__half" if dtype == torch.float16 else "__nv_bfloat16"
    if d < 512:
        pat = re.compile(rf"attn_tc_kernel<{tname}, {d}, 64,")
        assert not any("attn_wide_kernel" in n for n in names), names
    else:
        pat = re.compile(rf"attn_wide_kernel<{tname}>")
        assert not any("attn_tc_kernel" in n for n in names), names
    assert sum(bool(pat.search(n)) for n in names) == 1, (pat.pattern, names)
