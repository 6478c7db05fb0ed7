"""TEST INFRASTRUCTURE shared by tests/test_attention_paths_gpu.py and tests/test_attention_routing_cpu.py: the shape
matrix of hallo_b200_attention, the exact key-routing inputs, and a float64 restatement of the kernels' 64-key tile
loop.  Nothing under hallo_b200/ imports this file.

Routing inputs.  Every key of every source (the frame's own tokens, each reference frame) gets a distinct +-1 code in
a few columns of its head; the code is made from the key's id (source * L + key), a per-head mask and per-head code
columns.  The other K columns hold small noise that Q multiplies by 0.  Each query is ALPHA[d] x the code of its
target key, so the target's score beats every other key's by at least 2 alpha (one code bit), which is >= 40 in log2
units after d^-0.5 log2 e.  V holds odd multiples of 2^-6 in (-2, 2) that encode (source, key, head, column); they are
exact in fp16 and bf16.  With these inputs every other key's weight is below 2^-40, P of the target rounds to 1.0
and O[q] must equal V[target(q)] bit for bit."""
import math
from collections import namedtuple

import numpy as np
import torch

LOG2E = 1.4426950408889634
BN = 64        # keys per tile: attn_tc_kernel<T, D, 64, ...> and attn_wide_kernel
QT = 128       # queries per CTA
# smallest power of two with 2 * alpha * d^-0.5 * log2(e) >= 40
ALPHA = {40: 128, 80: 128, 160: 256, 512: 512}
for _d, _a in ALPHA.items():
    assert 2 * _a * LOG2E / math.sqrt(_d) >= 40 and _a * LOG2E / math.sqrt(_d) < 40

Case = namedtuple("Case", "d heads L frames ref_frames ridx")


def case_id(c):
    if c.ridx is None:
        ref = "noref"
    else:
        ref = f"ref{c.ref_frames}[{','.join(map(str, c.ridx[:6]))}{',..' if len(c.ridx) > 6 else ''}]"
    return f"d{c.d}-h{c.heads}-L{c.L}-F{c.frames}-{ref}"


def _ref_mode(i, frames):
    """(ref_frames, ref_index) layouts: none; the two-half layout (uncond -1, cond (g % 2)); the cond-only companion
    (every frame >= 0); one reference frame; three reference frames with every index and -1."""
    h = frames // 2
    modes = [
        (0, None),
        (2, [-1] * h + [g % 2 for g in range(frames - h)]),
        (2, [g % 2 for g in range(frames)]),
        (1, [-1 if g % 3 == 0 else 0 for g in range(frames)]),
        (3, [[2, 0, 1, -1][g % 4] for g in range(frames)]),
    ]
    return modes[i % len(modes)]


def self_attention_cases():
    """The shape matrix: head dims 40 / 80 / 160 over L in {1, 4, 16, 36, 63, 64, 65, 144, 200, 576, 1024} (+ 4096 at
    d = 40), heads 8 or 1, up to 32 frames, cycling through the reference layouts; head dim 512 with one head and no
    reference over L in {1, 4, 63, 64, 65, 120, 4096}."""
    out = []
    for d in (40, 80, 160):
        Ls = [1, 4, 16, 36, 63, 64, 65, 144, 200, 576, 1024] + ([4096] if d == 40 else [])
        for i, L in enumerate(Ls):
            frames = max(2, min(32, 2048 // L))
            rf, ridx = _ref_mode(i + d // 40, frames)
            out.append(Case(d, 1 if i % 3 == 2 else 8, L, frames, rf, ridx))
    for L in (1, 4, 63, 64, 65, 120, 4096):
        out.append(Case(512, 1, L, max(2, min(4, 4096 // L)), 0, None))
    return out


def routing_cases():
    """self_attention_cases() plus the config-4 headline length: L = 9216 at d = 40 with reference keys."""
    return self_attention_cases() + [Case(40, 1, 9216, 2, 2, [-1, 1])]


def sample_rows(L, seed=0):
    """Query rows a reference is computed for: all of them up to L = 2048; beyond, the first and last 128-query tile
    of the frame plus 256 seeded rows."""
    if L < 2048:
        return np.arange(L)
    last = QT * ((L - 1) // QT)
    rng = np.random.default_rng(seed + L)
    return np.unique(np.concatenate([np.arange(QT), np.arange(last, L), rng.choice(L, 256, replace=False)]))


def _code_columns(d, m, head, rng):
    if d == 512:
        # spread over all eight 64-column chunks (bit b -> chunk b % 8), shifted per head
        return np.array([(b % 8) * 64 + 8 * (b // 8) + (3 * head + b) % 8 for b in range(m)])
    return rng.permutation(d)[:m]


def _targets(L, nk, rng, rot):
    """L target keys out of nk (own keys 0..L-1, reference keys L..2L-1): first the edges -- key 0, key L - 1, both
    sides of every 64-key tile boundary, the start of the last (partial) tile, in both segments -- rotated by `rot`,
    then a random permutation."""
    special = set()
    for base in range(0, nk, L):
        special |= {base, base + L - 1, base + BN * ((L - 1) // BN)}
        for t in range(BN, L, BN):
            special |= {base + t - 1, base + t}
    special = np.array(sorted(special))
    special = np.roll(special, rot % len(special))
    order = np.concatenate([special, rng.permutation(nk)])
    _, first = np.unique(order, return_index=True)
    return order[np.sort(first)][:L]


def _v_values(nsrc, L, H, d):
    """odd multiples of 2^-6 in (-2, 2), a hash of (source, key, head, column)"""
    s = np.arange(nsrc, dtype=np.uint64)[:, None, None, None]
    j = np.arange(L, dtype=np.uint64)[None, :, None, None]
    h = np.arange(H, dtype=np.uint64)[None, None, :, None]
    c = np.arange(d, dtype=np.uint64)[None, None, None, :]
    x = s * np.uint64(7919) + j * np.uint64(104729) + h * np.uint64(1299709) + c * np.uint64(15485863)
    x = (x * np.uint64(2654435761)) % np.uint64(1 << 32)
    x = (x ^ (x >> np.uint64(15))) * np.uint64(2246822519) % np.uint64(1 << 32)
    return ((2.0 * ((x >> np.uint64(9)) % np.uint64(128)).astype(np.float64) - 127.0) / 64.0).astype(np.float32)


def routing_inputs(c, seed=0):
    """float32 CPU tensors q, k, v [frames*L, heads*d], kref, vref [ref_frames*L, heads*d] (None without reference
    keys), the target key of every query [frames, heads, L] (own keys 0..L-1, reference keys L..2L-1) and the exact
    output `expect` = V[target] [frames*L, heads*d].  All values are exact in fp16 and bf16."""
    d, H, L, F, R = c.d, c.heads, c.L, c.frames, c.ref_frames
    rng = np.random.default_rng(seed + 7 * L + d)
    nsrc = F + R                                   # sources: own tokens of frames 0..F-1, then reference frames
    m = max(1, math.ceil(math.log2(nsrc * L)))     # code bits: key id = source * L + key
    assert m <= d
    ids = np.arange(nsrc * L, dtype=np.int64).reshape(nsrc, L)
    K = rng.choice(np.array([-0.5, -0.25, 0.25, 0.5], np.float32), size=(nsrc, L, H, d))
    V = _v_values(nsrc, L, H, d)
    Q = np.zeros((F, L, H, d), np.float32)
    E = np.empty((F, L, H, d), np.float32)
    tgt = np.empty((F, H, L), np.int64)
    for h in range(H):
        cols = _code_columns(d, m, h, rng)
        mask = int(rng.integers(0, 1 << m))
        code = (2 * (((ids ^ mask)[..., None] >> np.arange(m)) & 1) - 1).astype(np.float32)   # [nsrc, L, m]
        K[:, :, h, cols] = code
        for f in range(F):
            r = -1 if c.ridx is None else c.ridx[f]
            nk = L * (2 if r >= 0 else 1)
            t = _targets(L, nk, rng, f * H + h)
            tgt[f, h] = t
            src = np.where(t < L, f, F + max(r, 0))
            Q[f, :, h][:, cols] = ALPHA[d] * code[src, t % L]
            E[f, :, h] = V[src, t % L, h]
    C = H * d
    q, e = torch.from_numpy(Q.reshape(F * L, C)), torch.from_numpy(E.reshape(F * L, C))
    k, v = torch.from_numpy(K[:F].reshape(F * L, C)), torch.from_numpy(V[:F].reshape(F * L, C))
    kref = vref = None
    if R:
        kref, vref = torch.from_numpy(K[F:].reshape(R * L, C)), torch.from_numpy(V[F:].reshape(R * L, C))
    return dict(q=q, k=k, v=v, kref=kref, vref=vref, target=tgt, expect=e)


def _round(x, dtype):
    return x.to(torch.float32).to(dtype).to(torch.float64)


def tile_loop(q, segs, d, dtype):
    """float64 restatement of the kernels' loop for one (frame, head): q [n, d]; segs = [(K, V), ...] key segments in
    kernel order (own, then reference), each [Lk, d].  64-key tiles with the tail masked, running max in log2 units,
    l rescaled with O, P = exp2(s * scale - m) rounded to the storage dtype for the P V product while l sums the
    unrounded P, then O / l.  Returns O [n, d] in float64 (before the output rounding)."""
    scale = float(np.float32(LOG2E / math.sqrt(d)))
    n = q.shape[0]
    m = torch.full((n,), -math.inf, dtype=torch.float64)
    l = torch.zeros(n, dtype=torch.float64)
    o = torch.zeros(n, d, dtype=torch.float64)
    for ks, vs in segs:
        for t0 in range(0, ks.shape[0], BN):
            s = (q @ ks[t0:t0 + BN].T) * scale
            m_new = torch.maximum(m, s.max(1).values)
            f = torch.exp2(m - m_new)
            l, o, m = l * f, o * f[:, None], m_new
            e = torch.exp2(s - m[:, None])
            l = l + e.sum(1)
            o = o + _round(e, dtype) @ vs[t0:t0 + BN]
    return o / l[:, None]


def tile_loop_all(inp, c, dtype, rows):
    """tile_loop over every (frame, head) for the query rows `rows` of each frame: [frames, len(rows), heads * d],
    rounded to dtype and back to float64."""
    d, H, L, F = c.d, c.heads, c.L, c.frames
    q = _round(inp["q"], dtype).view(F, L, H, d)
    k, v = _round(inp["k"], dtype).view(F, L, H, d), _round(inp["v"], dtype).view(F, L, H, d)
    if c.ref_frames:
        kr = _round(inp["kref"], dtype).view(c.ref_frames, L, H, d)
        vr = _round(inp["vref"], dtype).view(c.ref_frames, L, H, d)
    rows_t = torch.as_tensor(rows)
    out = torch.empty(F, len(rows), H, d, dtype=torch.float64)
    for f in range(F):
        r = -1 if c.ridx is None else c.ridx[f]
        for h in range(H):
            segs = [(k[f, :, h], v[f, :, h])] + ([(kr[r, :, h], vr[r, :, h])] if r >= 0 else [])
            out[f, :, h] = tile_loop(q[f, rows_t, h], segs, d, dtype)
    return _round(out, dtype).view(F, len(rows), H * d)
