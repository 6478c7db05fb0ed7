"""GPU parity of the HBM-bound helper kernels (csrc/aux.cu) against plain PyTorch fp32 references."""
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2

pytestmark = pytest.mark.gpu
DT = torch.float16


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.mark.parametrize("C", [320, 640, 1280, 2560])
def test_layernorm(C):
    from hallo_b200 import ops
    dev = _dev()
    g = torch.Generator().manual_seed(C)
    rows = 1000
    x = (torch.randn(rows, C, generator=g) * 3 + 0.5).to(dev, DT)
    gam = (1 + 0.1 * torch.randn(C, generator=g)).to(dev, DT)
    bet = (0.1 * torch.randn(C, generator=g)).to(dev, DT)
    out = torch.empty_like(x)
    ops.layernorm(x, gam, bet, out)
    torch.cuda.synchronize()
    ref = F.layer_norm(x.float(), (C,), gam.float(), bet.float(), 1e-5)
    assert rel_l2(out, ref) < 1e-3


def test_layernorm_pe():
    from hallo_b200 import ops
    from hallo_b200.spec import sinusoid_pe
    dev = _dev()
    C, L, Fr, b = 320, 16, 18, 2
    g = torch.Generator().manual_seed(5)
    x = torch.randn(b * Fr * L, C, generator=g).to(dev, DT)
    gam = (1 + 0.1 * torch.randn(C, generator=g)).to(dev, DT)
    bet = (0.1 * torch.randn(C, generator=g)).to(dev, DT)
    pe = sinusoid_pe(32, C)[0].to(dev)
    out = torch.empty_like(x)
    ops.layernorm(x, gam, bet, out, pe=pe, tokens_per_frame=L, frames=Fr)
    torch.cuda.synchronize()
    ref = F.layer_norm(x.float(), (C,), gam.float(), bet.float(), 1e-5).view(b, Fr, L, C) + pe[:Fr].view(1, Fr, 1, C)
    assert rel_l2(out.view(b, Fr, L, C), ref) < 1.5e-3
    # remapped frame positions (sharded ranks hold a subset of frames)
    idx = torch.tensor([0, 1, 6, 7, 8, 9] + [0] * 12, dtype=torch.int32, device=dev)
    ops.layernorm(x, gam, bet, out, pe=pe, pe_index=idx, tokens_per_frame=L, frames=Fr)
    torch.cuda.synchronize()
    ref2 = F.layer_norm(x.float(), (C,), gam.float(), bet.float(), 1e-5).view(b, Fr, L, C) + pe[idx.long()].view(1, Fr, 1, C)
    assert rel_l2(out.view(b, Fr, L, C), ref2) < 1.5e-3


@pytest.mark.parametrize("C1,C2,hw,silu", [(320, 0, 4096, True), (640, 0, 1024, False), (1280, 640, 256, True),
                                           (640, 320, 1024, True), (1280, 1280, 64, True), (320, 0, 100, False)])
def test_groupnorm(C1, C2, hw, silu):
    from hallo_b200 import ops
    dev = _dev()
    n = 3
    g = torch.Generator().manual_seed(C1 + hw)
    x1 = (torch.randn(n * hw, C1, generator=g) * 2 + 0.3).to(dev, DT)
    x2 = (torch.randn(n * hw, C2, generator=g) - 0.2).to(dev, DT) if C2 else None
    C = C1 + C2
    gam = (1 + 0.1 * torch.randn(C, generator=g)).to(dev, DT)
    bet = (0.1 * torch.randn(C, generator=g)).to(dev, DT)
    out = torch.empty(n * hw, C, device=dev, dtype=DT)
    ws = torch.empty(ops.gn_workspace_floats(n, hw, 32, C), device=dev, dtype=torch.float32)
    ops.groupnorm(x1, gam, bet, out, ws, n_frames=n, hw=hw, eps=1e-5, silu=silu, x2=x2)
    torch.cuda.synchronize()
    xc = x1 if x2 is None else torch.cat([x1, x2], 1)
    xr = xc.float().view(n, hw, C).permute(0, 2, 1)
    ref = F.group_norm(xr, 32, gam.float(), bet.float(), 1e-5)
    if silu:
        ref = F.silu(ref)
    ref = ref.permute(0, 2, 1).reshape(n * hw, C)
    assert rel_l2(out, ref) < 2e-3


def test_groupnorm_scatter_single_destination_and_slices():
    """hallo_b200_groupnorm_scatter (the frame -> pixel swap in front of a motion module, fused into the GroupNorm's
    store): with every destination pointing into ONE local buffer at different offsets the result must be the plain
    GroupNorm rearranged as [dest][frame_out][pixel slice] -- the addressing the peer-memory path relies on."""
    from hallo_b200 import ops
    dev = _dev()
    nb, fl, hw, C, R, nm, me = 2, 2, 64, 320, 4, 2, 1
    f, seg = fl * R, hw // R
    F18 = nm + f
    g = torch.Generator().manual_seed(21)
    x = torch.randn(nb * fl * hw, C, generator=g).to(dev, DT)
    gam = (1 + 0.1 * torch.randn(C, generator=g)).to(dev, DT)
    bet = (0.1 * torch.randn(C, generator=g)).to(dev, DT)
    dest = torch.zeros(R, nb * F18 * seg, C, device=dev, dtype=DT)        # "rank d's x18 buffer"
    ws = torch.empty(ops.gn_workspace_floats(nb * fl, hw, 32, C), device=dev, dtype=torch.float32)
    ops.groupnorm_scatter(x, gam, bet, [dest[d].data_ptr() for d in range(R)], ws, n_frames=nb * fl, hw=hw, eps=1e-6,
                          fpb_in=fl, fpb_out=F18, frame_off=nm + me * fl)
    torch.cuda.synchronize()
    ref = F.group_norm(x.float().view(nb * fl, hw, C).permute(0, 2, 1), 32, gam.float(), bet.float(), 1e-6).permute(0, 2, 1)
    ref = ref.reshape(nb, fl, R, seg, C)
    d5 = dest.view(R, nb, F18, seg, C)
    got = d5[:, :, nm + me * fl: nm + (me + 1) * fl].permute(1, 2, 0, 3, 4)          # [nb, fl, R, seg, C]
    assert rel_l2(got, ref) < 2e-3
    untouched = torch.cat([d5[:, :, :nm + me * fl].reshape(-1), d5[:, :, nm + (me + 1) * fl:].reshape(-1)])
    assert float(untouched.abs().max()) == 0.0


def test_gemm_row_scatter_and_add():
    """hb_row_scatter epilogue (a motion module's proj_out storing rows into the frame owners' buffers) and
    hallo_b200_add, on one device: destinations are slices of a local buffer."""
    from hallo_b200 import ops
    dev = _dev()
    nb, fl, R, Lg, C, me = 2, 2, 4, 32, 320, 2
    f, L = fl * R, Lg * R
    g = torch.Generator().manual_seed(22)
    a = torch.randn(f * Lg, C, generator=g).to(dev, DT)                    # rows (global frame g, pixel p of my slice)
    w = (torch.randn(C, C, generator=g) * 0.05).to(dev, DT)
    bias = torch.randn(C, generator=g).to(dev, DT)
    recv = torch.zeros(R, nb * fl * L, C, device=dev, dtype=DT)            # "rank d's recv buffer"
    b = 1
    sc = ops.row_scatter([recv[d].data_ptr() for d in range(R)], seg=Lg, segs_per_dest=fl, seg_stride=L,
                         row0=b * fl * L + me * Lg)
    ops.gemm(a, w, recv[0][:f * Lg], bias=bias, scatter=sc)
    torch.cuda.synchronize()
    ref = (a.float() @ w.float().t() + bias.float()).view(R, fl, Lg, C)   # [dest, local frame, pixel, C]
    got = recv.view(R, nb, fl, R, Lg, C)[:, b, :, me]
    assert rel_l2(got, ref) < 2e-3
    mask = torch.ones_like(recv.view(R, nb, fl, R, Lg, C), dtype=torch.bool)
    mask[:, b, :, me] = False
    assert float(recv.view(R, nb, fl, R, Lg, C)[mask].abs().max()) == 0.0
    x = torch.randn(nb * fl * L, C, generator=g).to(dev, DT)
    out = torch.empty_like(x)
    ops.add(recv[0], x, out)
    torch.cuda.synchronize()
    assert torch.equal(out, (recv[0].float() + x.float()).to(DT))


def test_groupnorm_frame_remap():
    from hallo_b200 import ops
    dev = _dev()
    b, f, hw, C = 2, 4, 64, 320
    g = torch.Generator().manual_seed(9)
    x = torch.randn(b * f * hw, C, generator=g).to(dev, DT)
    gam = torch.ones(C, device=dev, dtype=DT)
    bet = torch.zeros(C, device=dev, dtype=DT)
    out = torch.zeros(b * (f + 2) * hw, C, device=dev, dtype=DT)
    ws = torch.empty(ops.gn_workspace_floats(b * f, hw, 32, C), device=dev, dtype=torch.float32)
    ops.groupnorm(x, gam, bet, out, ws, n_frames=b * f, hw=hw, eps=1e-6, fpb_in=f, fpb_out=f + 2, frame_off=2)
    torch.cuda.synchronize()
    ref = F.group_norm(x.float().view(b * f, hw, C).permute(0, 2, 1), 32, None, None, 1e-6).permute(0, 2, 1)
    o = out.view(b, f + 2, hw, C)
    assert float(o[:, :2].abs().max()) == 0.0
    assert rel_l2(o[:, 2:].reshape(b * f, hw, C), ref) < 2e-3


def _sdpa(q, k, v):
    d = q.shape[-1]
    p = torch.softmax(q @ k.transpose(-1, -2) * d ** -0.5, -1)
    return p @ v


@pytest.mark.parametrize("C,nk,L", [(320, 4, 200), (1280, 4, 200), (320, 32, 200), (640, 32, 200), (1280, 32, 200),
                                    (320, 32, 1024), (320, 4, 1024), (640, 32, 64)])
def test_cross_attention(C, nk, L):
    """L >= 128 runs the wgmma kernel (csrc/attn_tc.cu), smaller L the CUDA-core kernel."""
    from hallo_b200 import ops
    dev = _dev()
    H, frames, f = 8, 4, 2
    d = C // H
    regions = 3 if nk == 32 else 1
    div = f if nk == 4 else 1
    kvf = frames // div
    g = torch.Generator().manual_seed(C + nk)
    q = torch.randn(frames * L, regions * C, generator=g).to(dev, DT)
    kv = torch.randn(kvf * nk, regions * 2 * C, generator=g).to(dev, DT)
    out = torch.empty(frames * L, regions * C, device=dev, dtype=DT)
    k, v = kv[:, :C], kv[:, C:]
    ops.cross_attention(q, k, v, out, frames=frames, tokens=L, heads=H, head_dim=d, n_keys=nk, kv_frame_div=div,
                        regions=regions, q_region_stride=C, kv_region_stride=2 * C, o_region_stride=C)
    torch.cuda.synchronize()
    for r in range(regions):
        qr = q[:, r * C:(r + 1) * C].float().view(frames, L, H, d).transpose(1, 2)
        kr = kv[:, r * 2 * C:r * 2 * C + C].float().view(kvf, nk, H, d).transpose(1, 2).repeat_interleave(div, 0)
        vr = kv[:, r * 2 * C + C:(r + 1) * 2 * C].float().view(kvf, nk, H, d).transpose(1, 2).repeat_interleave(div, 0)
        ref = _sdpa(qr, kr, vr).transpose(1, 2).reshape(frames * L, C)
        assert rel_l2(out[:, r * C:(r + 1) * C], ref) < 2e-3, r


@pytest.mark.parametrize("C,fq,fk", [(320, 18, 18), (1280, 18, 18), (640, 6, 18), (320, 3, 3)])
def test_temporal_attention(C, fq, fk):
    from hallo_b200 import ops
    dev = _dev()
    H, b, L = 8, 2, 64
    d = C // H
    g = torch.Generator().manual_seed(C + fq)
    qkv = torch.randn(b * fk * L, 3 * C, generator=g).to(dev, DT)
    qq = torch.randn(b * fq * L, C, generator=g).to(dev, DT)
    out = torch.empty(b * fq * L, C, device=dev, dtype=DT)
    ops.temporal_attention(qq, qkv[:, C:2 * C], qkv[:, 2 * C:], out, batch=b, fq=fq, fk=fk, tokens=L, heads=H)
    torch.cuda.synchronize()
    q4 = qq.float().view(b, fq, L, H, d).permute(0, 2, 3, 1, 4)
    k4 = qkv[:, C:2 * C].float().view(b, fk, L, H, d).permute(0, 2, 3, 1, 4)
    v4 = qkv[:, 2 * C:].float().view(b, fk, L, H, d).permute(0, 2, 3, 1, 4)
    ref = _sdpa(q4, k4, v4).permute(0, 3, 1, 2, 4).reshape(b * fq * L, C)
    assert rel_l2(out, ref) < 2e-3


def test_resample_and_stride2_conv():
    from hallo_b200 import ops
    dev = _dev()
    n, h, w, C, Co = 4, 16, 16, 320, 320
    g = torch.Generator().manual_seed(11)
    x = torch.randn(n, h, w, C, generator=g).to(dev, DT)
    up = torch.empty(n, 2 * h, 2 * w, C, device=dev, dtype=DT)
    ops.upsample2x(x, up)
    ref_up = F.interpolate(x.permute(0, 3, 1, 2).float(), scale_factor=2.0, mode="nearest").permute(0, 2, 3, 1)
    torch.cuda.synchronize()
    assert torch.equal(up.float(), ref_up)
    wt = (torch.randn(Co, C, 3, 3, generator=g) / (3 * C ** 0.5)).to(dev, DT)
    bias = torch.randn(Co, generator=g).to(dev, DT)
    planes = torch.empty(4 * n, h // 2, w // 2, C, device=dev, dtype=DT)
    ops.phase_split(x, planes)
    out = torch.empty(n * (h // 2) * (w // 2), Co, device=dev, dtype=DT)
    ops.conv3x3_stride2(planes, ops.pack_conv3x3_weight(wt), out, n=n, ho=h // 2, wo=w // 2, bias=bias)
    torch.cuda.synchronize()
    ref = F.conv2d(x.permute(0, 3, 1, 2).float(), wt.float(), bias.float(), stride=2, padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(-1, Co)
    assert rel_l2(out, ref) < 2e-3


def test_silu_epilogue_and_timestep_embedding():
    from hallo_b200 import ops
    dev = _dev()
    g = torch.Generator().manual_seed(12)
    t_table = torch.tensor([999.0, 974.0, 24.0], device=dev)
    step = torch.tensor([1], dtype=torch.int32, device=dev)
    emb = torch.empty(2, 320, device=dev, dtype=DT)
    ops.timestep_embed(t_table, step, emb)
    torch.cuda.synchronize()
    half = 160
    freq = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / half)
    ref = torch.cat([torch.cos(974.0 * freq), torch.sin(974.0 * freq)])
    assert rel_l2(emb[0], ref) < 2e-3 and torch.equal(emb[0], emb[1])
    w = (torch.randn(1280, 320, generator=g) / 18).to(dev, DT)
    b = torch.randn(1280, generator=g).to(dev, DT)
    out = torch.empty(2, 1280, device=dev, dtype=DT)
    ops.gemm(emb, w, out, bias=b, silu=True)
    torch.cuda.synchronize()
    assert rel_l2(out, F.silu(emb.float() @ w.float().t() + b.float())) < 2e-3
    ops.advance_step(step, 3)
    ops.advance_step(step, 3)
    torch.cuda.synchronize()
    assert int(step) == 0


def test_im2col_cfg_ddim_and_layout():
    from hallo_b200 import ops
    dev = _dev()
    g = torch.Generator().manual_seed(13)
    Cl, Fr, H, W = 4, 3, 8, 8
    lat = torch.randn(1, Cl, Fr, H, W, generator=g).to(dev)
    cols = torch.empty(2 * Fr * H * W, 64, device=dev, dtype=DT)
    ops.im2col_latent(lat, cols, batch=2)
    torch.cuda.synchronize()
    unf = F.unfold(lat[0].permute(1, 0, 2, 3), 3, padding=1)          # [F, Cl*9, HW] with index c*9 + tap
    unf = unf.view(Fr, Cl, 9, H * W).permute(0, 3, 2, 1).reshape(Fr * H * W, 36)   # tap*Cl + c
    assert rel_l2(cols[:Fr * H * W, :36], unf) < 1e-3
    assert torch.equal(cols[:Fr * H * W], cols[Fr * H * W:]) and float(cols[:, 36:].abs().max()) == 0.0
    # CFG + DDIM
    mo = torch.randn(2 * Fr * H * W, 8, generator=g).to(dev, DT)
    coef = torch.tensor([[0.0, 1.0, 0.3, 0.95], [0.6, 0.8, 0.9, 0.43]], device=dev)
    step = torch.tensor([1], dtype=torch.int32, device=dev)
    lat0 = lat.clone()
    v_out = torch.empty_like(lat)
    ops.cfg_ddim_step(mo, lat, coef, step, guidance=3.5, v_out=v_out)
    torch.cuda.synchronize()
    vu = mo[:Fr * H * W, :Cl].float().view(Fr, H, W, Cl).permute(3, 0, 1, 2)[None]
    vc = mo[Fr * H * W:, :Cl].float().view(Fr, H, W, Cl).permute(3, 0, 1, 2)[None]
    v = vu + 3.5 * (vc - vu)
    sa, sb, sap, sbp = coef[1].tolist()
    x0 = sa * lat0 - sb * v
    eps = sa * v + sb * lat0
    assert rel_l2(lat, sap * x0 + sbp * eps) < 1e-5 and rel_l2(v_out, v) < 1e-5
    out = torch.empty(2, Cl, Fr, H, W, device=dev)
    ops.tokens_to_bcfhw(mo, out)
    torch.cuda.synchronize()
    ref = mo[:, :Cl].float().view(2, Fr, H, W, Cl).permute(0, 4, 1, 2, 3)
    assert torch.equal(out, ref)
