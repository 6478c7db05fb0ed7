"""CPU checks of kernel-side index / algorithm logic that can be restated without a GPU:
 * the lane-level fragment arithmetic of hallo_b200/csrc/tattn_mma.cu (ldmatrix / mma.sync m16n8k16 layouts per the
   PTX ISA) reproduces softmax(Q K^T / sqrt(d)) V for every (pixel, head) task, including ragged frame counts, the
   half-filled last k-step of head_dim 40 and the uninitialised row padding;
 * the panel assignment and 64B-swizzle addressing of the GEMM's TMA-store epilogue (gemm_tc.cu, TEPI);
 * the float32 summation order of the three-launch GroupNorm statistics (aux.cu, gn_stats + gn_finalize).
These are restatements of the kernels' control flow in numpy, not the kernels themselves; the GPU parity tests
remain the gate."""
import numpy as np
import pytest


# ------------------------------------------------------------------------------------------------ PTX fragment model
def _ldsm(smem, addrs, n, trans=False):
    """ldmatrix.m8n8.x{n}[.trans].b16: matrix i takes its 8 row addresses from lanes 8i..8i+7."""
    regs = [[None] * n for _ in range(32)]
    for i in range(n):
        M = np.stack([smem[addrs[8 * i + r] // 2: addrs[8 * i + r] // 2 + 8] for r in range(8)])
        for l in range(32):
            g, t = l >> 2, l & 3
            regs[l][i] = (M[g, 2 * t], M[g, 2 * t + 1]) if not trans else (M[2 * t, g], M[2 * t + 1, g])
    return regs


def _mma(d, a, b):
    """mma.sync.m16n8k16.row.col: d (16x8, C layout) += A (16x16) B (16x8) from per-lane fragments."""
    A = np.zeros((16, 16))
    B = np.zeros((16, 8))
    for l in range(32):
        g, t = l >> 2, l & 3
        A[g, 2 * t], A[g, 2 * t + 1] = a[l][0]
        A[g + 8, 2 * t], A[g + 8, 2 * t + 1] = a[l][1]
        A[g, 2 * t + 8], A[g, 2 * t + 9] = a[l][2]
        A[g + 8, 2 * t + 8], A[g + 8, 2 * t + 9] = a[l][3]
        B[2 * t, g], B[2 * t + 1, g] = b[l][0]
        B[2 * t + 8, g], B[2 * t + 9, g] = b[l][1]
    Cm = A @ B
    for l in range(32):
        g, t = l >> 2, l & 3
        d[l][0] += Cm[g, 2 * t]
        d[l][1] += Cm[g, 2 * t + 1]
        d[l][2] += Cm[g + 8, 2 * t]
        d[l][3] += Cm[g + 8, 2 * t + 1]


def _tattn_mma_model(D, Fq, Fk, heads, pix, seed=0):
    rng = np.random.default_rng(seed)
    MT = 1 if Fq <= 16 else 2
    NT = 1 if Fk <= 8 else (3 if Fk <= 24 else 4)
    KS, half_step, KK, NJ = (D + 15) // 16, (D % 16) == 8, (NT + 1) // 2, D // 8
    C = heads * D
    ps = C * 2 + 16
    fs = pix * ps
    if ((fs >> 4) & 1) == 0:
        fs += 16
    smem = np.full((Fq + 2 * Fk) * fs // 2 + 64, np.nan)          # NaN = never-written padding
    sQ, sK, sV = 0, Fq * fs, (Fq + Fk) * fs
    Q, K, V = (rng.standard_normal((F, pix, C)) for F in (Fq, Fk, Fk))
    for base, X in ((sQ, Q), (sK, K), (sV, V)):
        for f in range(X.shape[0]):
            for p in range(pix):
                a = (base + f * fs + p * ps) // 2
                smem[a:a + C] = X[f, p]
    scale = 1.0 / np.sqrt(D)
    worst = 0.0
    for task in range(pix * heads):
        p, h = task // heads, task % heads
        toff = p * ps + h * D * 2
        s = [[[[0.0] * 4 for _ in range(32)] for _ in range(NT)] for _ in range(MT)]
        for ks in range(KS):
            a = []
            for mt in range(MT):
                r = _ldsm(smem, [sQ + toff + min(mt * 16 + (l & 7) + ((l >> 3) & 1) * 8, Fq - 1) * fs +
                                 (2 * ks + (l >> 4)) * 16 for l in range(32)], 4)
                if half_step and ks == KS - 1:
                    for l in range(32):
                        r[l][2] = r[l][3] = (0.0, 0.0)
                a.append(r)
            for nt in range(NT):
                bk = _ldsm(smem, [sK + toff + min(nt * 8 + (l & 7), Fk - 1) * fs + (2 * ks + ((l >> 3) & 1)) * 16
                                  for l in range(32)], 2)
                if half_step and ks == KS - 1:
                    for l in range(32):
                        bk[l][1] = (0.0, 0.0)
                for mt in range(MT):
                    _mma(s[mt][nt], a[mt], bk)
        inv = [[[0.0, 0.0] for _ in range(32)] for _ in range(MT)]
        for mt in range(MT):
            for hh in range(2):
                mx = [-np.inf] * 32
                for l in range(32):
                    for nt in range(NT):
                        for e in range(2):
                            if nt * 8 + 2 * (l & 3) + e >= Fk:
                                s[mt][nt][l][hh * 2 + e] = -np.inf
                            mx[l] = max(mx[l], s[mt][nt][l][hh * 2 + e])
                mx = [max(mx[l], mx[l ^ 1]) for l in range(32)]
                mx = [max(mx[l], mx[l ^ 2]) for l in range(32)]
                sm = [0.0] * 32
                for l in range(32):
                    for nt in range(NT):
                        for e in range(2):
                            pe = np.exp((s[mt][nt][l][hh * 2 + e] - mx[l]) * scale)
                            s[mt][nt][l][hh * 2 + e] = pe
                            sm[l] += pe
                sm = [sm[l] + sm[l ^ 1] for l in range(32)]
                sm = [sm[l] + sm[l ^ 2] for l in range(32)]
                for l in range(32):
                    inv[mt][l][hh] = 1.0 / sm[l]
        pa = [[[[None] * 4 for _ in range(32)] for _ in range(KK)] for _ in range(MT)]
        for mt in range(MT):
            for kk in range(KK):
                for l in range(32):
                    pa[mt][kk][l][0] = (s[mt][2 * kk][l][0], s[mt][2 * kk][l][1])
                    pa[mt][kk][l][1] = (s[mt][2 * kk][l][2], s[mt][2 * kk][l][3])
                    if 2 * kk + 1 < NT:
                        pa[mt][kk][l][2] = (s[mt][2 * kk + 1][l][0], s[mt][2 * kk + 1][l][1])
                        pa[mt][kk][l][3] = (s[mt][2 * kk + 1][l][2], s[mt][2 * kk + 1][l][3])
                    else:
                        pa[mt][kk][l][2] = pa[mt][kk][l][3] = (0.0, 0.0)
        out = np.full((Fq, D), np.nan)
        for j in range(NJ):
            o = [[[0.0] * 4 for _ in range(32)] for _ in range(MT)]
            for kk in range(KK):
                bv = _ldsm(smem, [sV + toff + min(kk * 16 + (l & 15), Fk - 1) * fs + j * 16 for l in range(32)], 2, trans=True)
                for mt in range(MT):
                    _mma(o[mt], pa[mt][kk], bv)
            for mt in range(MT):
                for hh in range(2):
                    for l in range(32):
                        g, t = l >> 2, l & 3
                        frame = mt * 16 + g + hh * 8
                        if frame < Fq:
                            out[frame, 8 * j + 2 * t] = o[mt][l][hh * 2] * inv[mt][l][hh]
                            out[frame, 8 * j + 2 * t + 1] = o[mt][l][hh * 2 + 1] * inv[mt][l][hh]
        q, k, v = (X[:, p, h * D:(h + 1) * D] for X in (Q, K, V))
        sc = q @ k.T * scale
        pr = np.exp(sc - sc.max(1, keepdims=True))
        ref = (pr / pr.sum(1, keepdims=True)) @ v
        assert not np.isnan(out).any()
        worst = max(worst, float(np.abs(out - ref).max()))
    return worst


@pytest.mark.parametrize("D,Fq,Fk,heads,pix", [(40, 18, 18, 8, 2), (80, 18, 18, 2, 1), (160, 18, 18, 2, 1), (40, 6, 18, 4, 2),
                                               (40, 3, 3, 8, 3), (40, 32, 32, 2, 1), (80, 17, 25, 2, 1)])
def test_tattn_mma_fragment_logic(D, Fq, Fk, heads, pix):
    assert _tattn_mma_model(D, Fq, Fk, heads, pix) < 1e-12


# ------------------------------------------------------------------------------------------------ streamed softmax
def _tepi_cover(BN, geglu):
    """Panel / unit assignment of gemm_tc_kernel<TEPI> (hallo_b200/csrc/gemm_tc.cu): returns, per output column of a
    tile, how many times it is written, and per accumulator column how many times it is read."""
    out_bn = BN // 2 if geglu else BN
    panels = BN // 64 if geglu else BN // 32
    written = np.zeros(out_bn, int)
    read = np.zeros(BN, int)
    max_units = 2 * ((BN // 64 + 1) // 2) if BN % 64 == 0 else (BN // 32 + 1) // 2
    for grp in (0, 1):
        my_panels = (panels - grp + 1) // 2
        my_units = 2 * my_panels if geglu else my_panels
        assert my_units <= max_units
        for u in range(my_units):
            col = (grp + 2 * (u >> 1)) * 64 + (u & 1) * 32 if geglu else (grp + 2 * u) * 32
            read[col:col + 32] += 1
            if geglu:
                panel, chunks = grp + 2 * (u >> 1), [(u & 1) * 2, (u & 1) * 2 + 1]
            else:
                panel, chunks = grp + 2 * u, [0, 1, 2, 3]
            for c in chunks:
                written[panel * 32 + c * 8: panel * 32 + c * 8 + 8] += 1
            # value/gate pairing of the GEGLU weight packing: accumulator column 2j, 2j+1 -> output column j
            if geglu:
                assert (col >> 1) == panel * 32 + chunks[0] * 8
    return written, read


@pytest.mark.parametrize("BN,geglu", [(256, False), (192, False), (160, False), (128, False), (256, True), (192, True)])
def test_tepi_panel_assignment_covers_each_column_once(BN, geglu):
    written, read = _tepi_cover(BN, geglu)
    assert (written == 1).all() and (read == 1).all()


def test_tepi_swizzle64_is_bank_conflict_free_and_bijective():
    """Panel buffer: 128 rows x 64 B, chunk c of row r at r*64 + ((c ^ ((r >> 1) & 3)) << 4) (CU_TENSOR_MAP_SWIZZLE_64B:
    address bits [4:5] ^= bits [7:8]).  A 128-bit shared access is served per quarter-warp: the 8 lanes (= 8 consecutive
    rows, same logical chunk) must touch 8 different 16-byte bank groups."""
    seen = set()
    for r in range(128):
        for c in range(4):
            off = r * 64 + ((c ^ ((r >> 1) & 3)) << 4)
            assert off == (r * 64 + c * 16) ^ ((((r * 64 + c * 16) >> 7) & 3) << 4)     # the hardware's address form
            seen.add(off)
    assert len(seen) == 512 and max(seen) < 8192
    for r0 in range(0, 128, 8):
        for c in range(4):
            groups = {((r * 64 + ((c ^ ((r >> 1) & 3)) << 4)) % 128) // 16 for r in range(r0, r0 + 8)}
            assert len(groups) == 8


# ------------------------------------------------------------------------------------------------ attn3 (register S)


# ------------------------------------------------------------------------------------------------ GroupNorm statistics
def _gn_stats_model(x, G, pivot, eps=1e-6):
    """float32 restatement of gn_stats_kernel + gn_finalize_kernel (hallo_b200/csrc/aux.cu) for one frame, in the
    kernels' summation order.  x: [HW, C] values of the storage type, as float32.
    pivot=True (the kernels): sums of d = x - pivot, pivot = the group's first channel at pixel 0; mean = pivot + A/cnt,
    var = B/cnt - (A/cnt)^2.  pivot=False: the one-pass form on x itself, var = E[x^2] - mean^2.
    Returns (mean, rstd) per group."""
    f32 = np.float32
    HW, C = x.shape
    cpg, nvec = C // G, C // 8
    PY = max(1, 256 // nvec)                     # pixel rows of a stats CTA (threads = nvec * PY)
    ppc = 64                                     # pixels per stats CTA
    assert HW % ppc == 0 and ppc % PY == 0
    nch = HW // ppc
    piv = x[0, ::cpg].copy() if pivot else np.zeros(G, f32)
    d = (x - np.repeat(piv, cpg)[None, :]).astype(f32)
    # thread (cv, py) of chunk k accumulates pixels k*64 + py, + PY, + 2 PY, ... in that order, per channel
    dk = d.reshape(nch, ppc // PY, PY, C)
    s = np.zeros((nch, PY, C), f32)
    q = np.zeros((nch, PY, C), f32)
    for u in range(ppc // PY):
        s = s + dk[:, u]
        q = q + dk[:, u] * dk[:, u]
    # one thread per group: rows py = 0..PY-1 outer, the group's channels inner
    s4, q4 = s.reshape(nch, PY, G, cpg), q.reshape(nch, PY, G, cpg)
    a = np.zeros((nch, G), f32)
    b = np.zeros((nch, G), f32)
    for y in range(PY):
        for c in range(cpg):
            a = a + s4[:, y, :, c]
            b = b + q4[:, y, :, c]
    # gn_finalize_kernel: the chunk partials in chunk order
    A = np.zeros(G, f32)
    B = np.zeros(G, f32)
    for k in range(nch):
        A = A + a[k]
        B = B + b[k]
    cnt = f32(cpg * HW)
    md = A / cnt
    mean = piv + md
    var = np.maximum(B / cnt - md * md, f32(0))
    return mean, f32(1) / np.sqrt(var + f32(eps))


@pytest.mark.parametrize("hw,offset", [(4096, 100.0), (262144, 100.0)])
def test_groupnorm_pivoted_statistics(hw, offset):
    """At the VAE's 512^2 top level (HW = 262144, C = 128, 4 channels per group) with N(100, 1) fp16 input the
    pivoted sums keep rstd within 1e-5 of float64; the one-pass E[x^2] - mean^2 they replaced is off by more than
    1e-2 there (about 2 log10(mean / std) digits lost to cancellation)."""
    rng = np.random.default_rng(7)
    C, G = 128, 32
    x = (rng.standard_normal((hw, C)) + offset).astype(np.float16).astype(np.float32)
    xd = x.astype(np.float64).reshape(hw, G, C // G)
    rstd_ref = 1.0 / np.sqrt(xd.var(axis=(0, 2)) + 1e-6)
    mean_ref = xd.mean(axis=(0, 2))
    mean, rstd = _gn_stats_model(x, G, pivot=True)
    err = float(np.abs(rstd / rstd_ref - 1).max())
    assert err < 1e-5, err
    assert float(np.abs(mean - mean_ref).max()) < 1e-5 * offset
    if hw == 262144:
        _, rstd_old = _gn_stats_model(x, G, pivot=False)
        err_old = float(np.abs(rstd_old / rstd_ref - 1).max())
        assert err_old > 1e-2, err_old
