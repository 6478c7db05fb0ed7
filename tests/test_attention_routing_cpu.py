"""CPU side of the self-attention tests.

1. The exact key-routing inputs of tests/test_attention_paths_gpu.py, run through a float64 restatement of the
   kernels' 64-key tile loop (tests/attn_cases.py), must give V[target] bit for bit in fp16 and bf16.  A GPU routing
   failure then points at the kernel, not at the construction.
2. hallo_b200_attention rejects bad arguments before any driver call or launch: on a host without a CUDA device every
   case below returns its documented hb_status and names the problem in hallo_b200_last_error()."""
import ctypes as C

import numpy as np
import pytest
import torch

import attn_cases as ac

DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["f16", "bf16"]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("c", ac.routing_cases(), ids=ac.case_id)
def test_tile_loop_routes_every_query_to_its_target(c, dtype):
    inp = ac.routing_inputs(c)
    rows = ac.sample_rows(c.L)
    got = ac.tile_loop_all(inp, c, dtype, rows)
    want = inp["expect"].view(c.frames, c.L, -1)[:, torch.as_tensor(rows)].double()
    assert torch.equal(want, ac._round(want, dtype)), "routing V values are not exact in the storage dtype"
    bad = (got != want).any(-1)
    assert not bad.any(), f"{int(bad.sum())} query rows do not return V[target]"


def test_routing_targets_cover_the_tile_edges():
    """Across the heads and frames of one case the targets include key 0, key L - 1, both sides of every 64-key
    boundary and the last partial tile, in the own and the reference segment."""
    c = ac.Case(40, 8, 200, 4, 2, [0, 1, -1, 1])
    t = ac.routing_inputs(c)["target"]
    seen = set(np.unique(t[[0, 1, 3]]).tolist())
    for base in (0, 200):
        for key in (0, 63, 64, 127, 128, 191, 192, 199):
            assert base + key in seen, base + key
    assert set(np.unique(t[2]).tolist()) <= set(range(200))
    # a different target permutation per head
    assert len({tuple(t[0, h]) for h in range(8)}) == 8


# ------------------------------------------------------------------------------------------ entry-point validation
HB_ERR_BAD_SHAPE, HB_ERR_NULL = -1, -4
_A = 0x100000          # 16-byte aligned stand-in device addresses, never dereferenced: each call must fail first


def _params(**kw):
    from hallo_b200 import lib
    p = lib.AttentionParams()
    p.dtype, p.head_dim, p.heads, p.L, p.frames = lib.HB_F16, 40, 8, 64, 2
    p.Q, p.K, p.V, p.O = _A, _A + 0x10000, _A + 0x20000, _A + 0x30000
    p.ldq = p.ldk = p.ldv = p.ldo = p.ldkref = p.ldvref = 320
    for k, v in kw.items():
        setattr(p, k, v)
    return p


_REF = dict(Kref=_A + 0x40000, Vref=_A + 0x50000, ref_frames=2, ref_index=_A + 0x60000)

_BAD = [
    ("null-Q", dict(Q=None), HB_ERR_NULL, "null pointer"),
    ("null-K", dict(K=None), HB_ERR_NULL, "null pointer"),
    ("null-V", dict(V=None), HB_ERR_NULL, "null pointer"),
    ("null-O", dict(O=None), HB_ERR_NULL, "null pointer"),
    ("head-dim-64", dict(head_dim=64), HB_ERR_BAD_SHAPE, "head_dim 64"),
    ("heads-0", dict(heads=0), HB_ERR_BAD_SHAPE, "heads=0"),
    ("heads-257", dict(heads=257), HB_ERR_BAD_SHAPE, "heads=257"),
    ("ldq", dict(ldq=324), HB_ERR_BAD_SHAPE, "multiples of 8"),
    ("ldk", dict(ldk=324), HB_ERR_BAD_SHAPE, "multiples of 8"),
    ("ldv", dict(ldv=324), HB_ERR_BAD_SHAPE, "multiples of 8"),
    ("ldo", dict(ldo=324), HB_ERR_BAD_SHAPE, "multiples of 8"),
    ("ldkref", dict(_REF, ldkref=324), HB_ERR_BAD_SHAPE, "multiples of 8"),
    ("ldvref", dict(_REF, ldvref=324), HB_ERR_BAD_SHAPE, "multiples of 8"),
    ("d512-heads-2", dict(head_dim=512, heads=2, ldq=1024, ldk=1024, ldv=1024, ldo=1024), HB_ERR_BAD_SHAPE,
     "one head and no reference"),
    ("d512-ref", dict(_REF, head_dim=512, heads=1, ldq=512, ldk=512, ldv=512, ldo=512, ldkref=512, ldvref=512),
     HB_ERR_BAD_SHAPE, "one head and no reference"),
    ("ref-without-Kref", dict(_REF, Kref=None), HB_ERR_NULL, "without Kref/Vref"),
    ("ref-without-Vref", dict(_REF, Vref=None), HB_ERR_NULL, "without Kref/Vref"),
    ("ref-frames-0", dict(_REF, ref_frames=0), HB_ERR_NULL, "without Kref/Vref"),
    ("O-odd-element", dict(O=_A + 0x30000 + 2), HB_ERR_BAD_SHAPE, "4-byte aligned"),
    ("Q-misaligned", dict(Q=_A + 8), HB_ERR_BAD_SHAPE, "16-byte aligned"),
    ("Kref-misaligned", dict(_REF, Kref=_A + 0x40000 + 8), HB_ERR_BAD_SHAPE, "16-byte aligned"),
]


@pytest.mark.parametrize("kw,status,msg", [pytest.param(*b[1:], id=b[0]) for b in _BAD])
def test_attention_rejects_bad_arguments_before_any_launch(kw, status, msg):
    """Runs only without a device: these calls pass stand-in pointers that are safe only because they are rejected
    before a driver call or launch.  A check that moved behind a driver call returns HB_ERR_CUDA here instead."""
    if torch.cuda.is_available():
        pytest.skip("passes stand-in device pointers; only safe on a host without a CUDA device")
    from hallo_b200 import lib
    h = lib.load()
    p = _params(**kw)
    rc = h.hallo_b200_attention(C.byref(p), None)
    err = h.hallo_b200_last_error().decode()
    assert rc == status, (rc, err)
    assert msg in err, err


def test_attention_null_params_struct():
    if torch.cuda.is_available():
        pytest.skip("only run on a host without a CUDA device")
    from hallo_b200 import lib
    h = lib.load()
    assert h.hallo_b200_attention(None, None) == HB_ERR_NULL
    assert "null pointer" in h.hallo_b200_last_error().decode()


def test_cross_attention_rejects_misaligned_q_and_o():
    """Both cross-attention kernels need O aligned (the CUDA-core one moves 16 bytes per access), so the entry point
    rejects a misaligned Q or O up front instead of letting the "xattn_tc" option decide whether the call works."""
    if torch.cuda.is_available():
        pytest.skip("passes stand-in device pointers; only safe on a host without a CUDA device")
    from hallo_b200 import lib
    h = lib.load()
    for q, o in ((_A, _A + 0x1000 + 4), (_A + 8, _A + 0x1000)):
        rc = h.hallo_b200_cross_attention(
            lib.HB_F16, C.c_void_p(q), C.c_int64(320), 0, C.c_void_p(_A + 0x2000), C.c_void_p(_A + 0x2000 + 640),
            C.c_int64(640), 0, C.c_void_p(o), C.c_int64(320), 0, 2, 128, 8, 40, 32, 1, 1, None)
        assert rc == HB_ERR_BAD_SHAPE
        assert "16-byte aligned" in h.hallo_b200_last_error().decode()
