"""CPU tests of guidance rescale (`guidance_rescale`, diffusers rescale_noise_cfg): a float64 restatement of diffusers'
function against PyTorch stand-ins for the three new ops (stats, reduce, apply), properties that rest on no
restatement, the engine's step tail for all five samplers against forward_only + float64 rescale + the sampler's table
row, a frame-sharded window over two thread-ranks, argument validation and the captured-graph key."""
import math

import pytest
import torch

from conftest import rel_l2
from test_audio_guidance_cpu import (SAMPLERS, _engine, _inputs, _install_step_stand_ins, _table, _window, guide3_f64,
                                     op_cfg_guide3_step)
from hallo_b200.scheduler import DDIMScheduler

RESCALE_PARTIALS, RESCALE_THREADS = 256, 256          # HB_RESCALE_PARTIALS CTAs of 256 threads (hallo_b200/csrc/aux.cu)


# ---------------------------------------------------------------- restatement and stand-ins
def rescale_noise_cfg_f64(noise_cfg, noise_pred_text, guidance_rescale):
    """diffusers 0.27.2 rescale_noise_cfg, in float64: std over every dimension but the batch, torch.std's default
    (unbiased) correction."""
    noise_cfg, noise_pred_text = noise_cfg.double(), noise_pred_text.double()
    dims = list(range(1, noise_pred_text.ndim))
    std_text = noise_pred_text.std(dim=dims, keepdim=True)
    std_cfg = noise_cfg.std(dim=dims, keepdim=True)
    noise_pred_rescaled = noise_cfg * (std_text / std_cfg)
    return guidance_rescale * noise_pred_rescaled + (1 - guidance_rescale) * noise_cfg


def combine_f64(mo, nb, s, sa):
    """The engine's CFG combine of per-half predictions mo [nb, ...]: two branches, or guide3's three."""
    vu, vc, vr = mo[0:1].double(), mo[1:2].double(), mo[2:3].double()
    return vu + s * (vc - vu) if nb == 2 else guide3_f64(vu, vc, vr, s, sa)


def _halves(model_out, nb, cl, n):
    mo = model_out[:nb * n, :cl].float()
    return [mo[b * n:(b + 1) * n] for b in range(nb)]


def _v_cfg(model_out, nb, cl, n, guidance, audio_guidance):
    h = _halves(model_out, nb, cl, n)
    if nb == 3:
        return h[1], h[0] + guidance * (h[2] - h[0]) + audio_guidance * (h[1] - h[2])
    return h[1], h[0] + guidance * (h[1] - h[0])


def op_cfg_rescale_stats(model_out, partials, *, nb, cl, frames, hw, guidance, audio_guidance=0.0):
    """Stand-in for hallo_b200_cfg_rescale_stats (include/hallo_b200.h): row i of a half belongs to CTA
    (i mod 256*256) // 256; per-CTA sums of v_c, v_c^2, v_cfg, v_cfg^2 in float64, v_cfg in fp32."""
    n = frames * hw
    vc, v = (t.double() for t in _v_cfg(model_out, nb, cl, n, guidance, audio_guidance))
    cta = (torch.arange(n) % (RESCALE_PARTIALS * RESCALE_THREADS)) // RESCALE_THREADS
    q = torch.stack([vc.sum(1), (vc * vc).sum(1), v.sum(1), (v * v).sum(1)], 1)          # [n, 4]
    partials.view(RESCALE_PARTIALS, 4).zero_().index_add_(0, cta, q)
    return partials


def op_cfg_rescale_reduce(partials, dst):
    """Stand-in for hallo_b200_cfg_rescale_reduce: the 4 totals of the partials stored to every destination."""
    tot = partials.view(RESCALE_PARTIALS, 4).sum(0)
    for d in dst:
        d.copy_(tot)


def rescale_factor(totals, n_local, phi):
    """k = phi std_t / std_g + (1 - phi) from totals [ranks, 4] summed in rank order; 1 where std_g is 0 (up to the
    rounding of the float64 sums)."""
    s = [0.0] * 4
    for r in range(totals.shape[0]):
        for q in range(4):
            s[q] += float(totals[r, q])
    n = float(totals.shape[0] * n_local)
    var_t = (s[1] - s[0] * s[0] / n) / (n - 1.0)
    var_g = (s[3] - s[2] * s[2] / n) / (n - 1.0)
    if n > 1.0 and var_g > 1e-12 * (s[3] / n):
        return phi * math.sqrt(max(var_t, 0.0) / var_g) + (1.0 - phi)
    return 1.0


def op_cfg_rescale_apply(model_out, totals, *, nb, cl, frames, hw, guidance, audio_guidance=0.0, rescale):
    """Stand-in for hallo_b200_cfg_rescale_apply: [0 | k v_cfg] over the first two halves in the model dtype."""
    n = frames * hw
    _, v = _v_cfg(model_out, nb, cl, n, guidance, audio_guidance)
    k = torch.tensor(rescale_factor(totals, cl * n, rescale), dtype=torch.float32)
    model_out[:n, :cl] = 0
    model_out[n:2 * n, :cl] = (k * v).to(model_out.dtype)
    return model_out


RESCALE_OPS = (op_cfg_rescale_stats, op_cfg_rescale_reduce, op_cfg_rescale_apply)


def install_rescale_stand_ins(monkeypatch):
    from hallo_b200 import ops
    for fn in RESCALE_OPS:
        monkeypatch.setattr(ops, fn.__name__[3:], fn)


def run_rescale(ops, mo, *, nb, cl, frames, hw, guidance, audio_guidance, rescale):
    """stats -> reduce -> apply on one rank (the engine's R = 1 sequence), through `ops` (hallo_b200.ops or this
    module's stand-ins, by name)."""
    dev = mo.device
    part = torch.zeros(RESCALE_PARTIALS, 4, dtype=torch.float64, device=dev)
    tot = torch.zeros(1, 4, dtype=torch.float64, device=dev)
    kw = dict(nb=nb, cl=cl, frames=frames, hw=hw, guidance=guidance, audio_guidance=audio_guidance)
    ops.cfg_rescale_stats(mo, part, **kw)
    ops.cfg_rescale_reduce(part, [tot[0]])
    ops.cfg_rescale_apply(mo, tot, rescale=rescale, **kw)
    return tot


class StandIns:
    cfg_rescale_stats = staticmethod(op_cfg_rescale_stats)
    cfg_rescale_reduce = staticmethod(op_cfg_rescale_reduce)
    cfg_rescale_apply = staticmethod(op_cfg_rescale_apply)
    cfg_guide3_step = staticmethod(op_cfg_guide3_step)


def make_model_out(nb, cl, frames, hw, ldm, dtype, scale=1.0, seed=3, device="cpu"):
    """[nb*frames*hw, ldm] with NaN past column cl; the halves get different spreads so the factor is not 1."""
    g = torch.Generator().manual_seed(seed)
    n = frames * hw
    mo = torch.full((nb * n, ldm), float("nan"))
    for b in range(nb):
        mo[b * n:(b + 1) * n, :cl] = torch.randn(n, cl, generator=g) * scale * (1.0 + 0.5 * b) + 0.1 * b
    return mo.to(device, dtype)


def to_bcfhw(rows, cl, frames, h, w):
    """[frames*h*w, cl] rows -> [1, cl, frames, h, w] (the engine's (frame, pixel) row order)."""
    return rows.reshape(frames, h, w, cl).permute(3, 0, 1, 2).unsqueeze(0)


def check_properties(ops, dtype, device="cpu"):
    """Properties of stats -> reduce -> apply that rest on no restatement: phi = 1 gives v with the std of v_c;
    phi = 0 writes v_cfg itself; a constant v_cfg (std 0) is kept as it is, without NaN.  Returns the phi = 1 error."""
    cl, frames, hw, ldm, s = 4, 3, 63, 8, 3.5
    n = frames * hw
    eps = torch.finfo(dtype).eps
    for nb in (2, 3):
        mo = make_model_out(nb, cl, frames, hw, ldm, dtype, device=device)
        ref = mo.clone()
        run_rescale(ops, mo, nb=nb, cl=cl, frames=frames, hw=hw, guidance=s, audio_guidance=6.0, rescale=1.0)
        v = mo[n:2 * n, :cl].double().cpu()
        std_c = ref[n:2 * n, :cl].double().cpu().std()
        err1 = float(abs(v.std() - std_c) / std_c)
        assert err1 <= 2 * eps, (nb, err1)
        mo0 = ref.clone()
        run_rescale(ops, mo0, nb=nb, cl=cl, frames=frames, hw=hw, guidance=s, audio_guidance=6.0, rescale=0.0)
        _, vcfg = _v_cfg(ref.cpu(), nb, cl, n, s, 6.0)
        got0 = mo0[n:2 * n, :cl].cpu().float()
        assert float((got0 - vcfg).abs().max()) <= eps * float(vcfg.abs().max()), nb    # k = 1: v_cfg, rounded once
        if nb == 3:                                           # the same [0 | v] as the three-branch combine alone
            g3 = ops.cfg_guide3_step(ref.clone(), cl=cl, frames=frames, hw=hw, guidance=s, audio_guidance=6.0)
            assert torch.equal(mo0[:2 * n, :cl], g3[:2 * n, :cl])
        assert torch.equal(mo0[:n, :cl].float().cpu(), torch.zeros(n, cl))
        assert torch.equal(mo0[nb * n:].cpu().isnan(), ref[nb * n:].cpu().isnan())
        assert mo0[:, cl:].isnan().all() and mo[:, cl:].isnan().all()            # columns past Cl untouched
        if nb == 3:
            assert torch.equal(mo0[2 * n:, :cl], ref[2 * n:, :cl])                   # third half untouched
    # v_u = v_c = constant: v_cfg is the constant, std_g = 0 -> kept, not NaN
    for c in (0.0, 0.3):
        mo = torch.full((2 * n, ldm), float("nan"))
        mo[:, :cl] = c
        mo = mo.to(device, dtype)
        run_rescale(ops, mo, nb=2, cl=cl, frames=frames, hw=hw, guidance=s, audio_guidance=0.0, rescale=0.7)
        assert torch.equal(mo[n:, :cl].float().cpu(), torch.full((n, cl), float(torch.tensor(c).to(dtype)))), c
    return err1


# ---------------------------------------------------------------- the ops against the restatement
@pytest.mark.parametrize("nb", [2, 3])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_stand_ins_match_rescale_noise_cfg(nb, dtype):
    cl, f, h, w, ldm, s, sa, phi = 4, 3, 7, 9, 8, 3.5, 6.0, 0.7
    n = f * h * w
    mo = make_model_out(nb, cl, f, h * w, ldm, dtype, scale=300.0)               # |v| up to ~1e3
    ref = mo.clone()
    run_rescale(StandIns, mo, nb=nb, cl=cl, frames=f, hw=h * w, guidance=s, audio_guidance=sa, rescale=phi)
    halves = [to_bcfhw(x, cl, f, h, w) for x in _halves(ref, nb, cl, n)]
    vcfg = combine_f64(torch.cat(halves), nb, s, sa)
    want = rescale_noise_cfg_f64(vcfg, halves[1], phi)
    got = to_bcfhw(mo[n:2 * n, :cl], cl, f, h, w).double()
    err = float((got - want).abs().max() / want.abs().max())
    print(f"stand-ins nb={nb} {dtype}: max error / max |v| = {err:.2e}")
    assert err <= torch.finfo(dtype).eps / 2 + 8 * torch.finfo(torch.float32).eps       # one rounding to the dtype
    assert torch.equal(mo[:n, :cl].float(), torch.zeros(n, cl)) and mo[:, cl:].isnan().all()
    moved = float((want - vcfg).abs().max() / vcfg.abs().max())
    assert moved > 1e-2                                                           # the factor is not 1 here


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_properties_of_stand_ins(dtype):
    check_properties(StandIns, dtype)


def test_restatement_properties():
    """rescale_noise_cfg itself: phi = 1 gives std(v_c), phi = 0 gives v_cfg (no restatement of the ops involved)."""
    g = torch.Generator().manual_seed(1)
    vc, vcfg = torch.randn(1, 4, 3, 5, 5, generator=g, dtype=torch.float64), torch.randn(1, 4, 3, 5, 5, generator=g,
                                                                                     dtype=torch.float64) * 4
    assert abs(float(rescale_noise_cfg_f64(vcfg, vc, 1.0).std() - vc.std())) < 1e-12
    assert torch.equal(rescale_noise_cfg_f64(vcfg, vc, 0.0), vcfg)


# ---------------------------------------------------------------- the engine on CPU stand-ins
@pytest.fixture(scope="module")
def weights():
    from hallo_b200.engine import PackedWeights
    from hallo_b200.spec import UNetConfig
    from hallo_b200.synth import host_threads, synth_state_dict
    torch.set_num_threads(host_threads())
    cfg = UNetConfig()
    return PackedWeights(synth_state_dict(cfg, seed=0), cfg, torch.device("cpu"), torch.float32)


def host_update(kind, row, x, v, state, z=None):
    """One scheduler update from the sampler's table row in float64 (include/hallo_b200.h, cfg_*_step with v given)."""
    r = [float(c) for c in row]
    if kind == "ddim":
        sa, sb, pa, pb = r
        return pa * (sa * x - sb * v) + pb * (sa * v + sb * x)
    if kind in ("multistep", "ancestral"):
        al, sg, a, b, c = r
        x0 = al * x - sg * v
        if kind == "ancestral":
            return a * x + b * x0 + c * z
        xn = a * x + b * x0 + (c * state["m1"] if c != 0.0 else 0.0)
        state["m1"] = x0
        return xn
    al, sg, kx, kl, k0, k1, k2, pc, p0, p1 = r
    m = al * x - sg * v
    m1 = state.get("m1")
    cr = k0 * m
    if kx != 0.0:
        cr = cr + kx * x
    if kl != 0.0:
        cr = cr + kl * state["last"]
    if k1 != 0.0:
        cr = cr + k1 * m1
    if k2 != 0.0:
        cr = cr + k2 * state["m2"]
    xn = pc * cr + p0 * m + (p1 * m1 if p1 != 0.0 else 0.0)
    state.update(last=cr, m2=m1, m1=m)
    return xn


@pytest.mark.parametrize("nb", [2, 3])
def test_engine_step_tail_matches_host(monkeypatch, weights, nb):
    """phi = 0.7, two eager steps of every sampler against forward_only + float64 combine + float64 rescale_noise_cfg
    + the sampler's table row; phi = 0 issues no rescale op."""
    from hallo_b200 import ops
    _install_step_stand_ins(monkeypatch)
    install_rescale_stand_ins(monkeypatch)
    calls = []
    for name in ("cfg_rescale_stats", "cfg_rescale_reduce", "cfg_rescale_apply", "cfg_guide3_step"):
        fn = getattr(ops, name)
        monkeypatch.setattr(ops, name, lambda *a, _n=name, _f=fn, **kw: (calls.append(_n), _f(*a, **kw))[1])
    f = 2
    inp = _inputs(f, seed=11)
    eng = _engine(weights, f, halves=tuple(range(nb)))
    eng.begin_window(**_window(inp))
    lat0 = inp["sample"][:1].float()
    sa = 6.0 if nb == 3 else None
    for cls in SAMPLERS:
        ts, kind, table = _table(cls, 10)
        noise = torch.randn(10, 4, f, 8, 8, generator=torch.Generator().manual_seed(2)) if kind == "ancestral" else None
        eng.set_schedule(ts, table, 3.5, kind, noise=noise, audio_guidance=sa, guidance_rescale=0.7)
        x, state = lat0.double(), {}
        for i in range(2):
            mo = eng.forward_only(x.float(), step=i).double()
            v = rescale_noise_cfg_f64(combine_f64(mo, nb, 3.5, sa or 0.0), mo[1:2], 0.7)
            x = host_update(kind, table[i], x, v, state, None if noise is None else noise[i].double().unsqueeze(0))
        out = {}
        for phi in (0.7, 0.0):
            eng.set_schedule(ts, table, 3.5, kind, noise=noise, audio_guidance=sa, guidance_rescale=phi)
            eng.latents.copy_(lat0)
            calls.clear()
            eng.step()
            eng.step()
            out[phi] = (eng.latents.clone(), list(calls))
        err, moved = rel_l2(out[0.7][0], x), rel_l2(out[0.0][0], x)
        print(f"{cls.__name__}, nb = {nb}: engine vs host, 2 steps at phi = 0.7: rel L2 = {err:.2e} "
              f"(phi = 0 vs the host's phi = 0.7: {moved:.2e})")
        assert err < 1e-5 and moved > 100 * err, cls.__name__
        assert out[0.7][1] == ["cfg_rescale_stats", "cfg_rescale_reduce", "cfg_rescale_apply"] * 2
        # phi = 0: the path without the rescale (guide3 for three branches, nothing for two)
        assert out[0.0][1] == (["cfg_guide3_step"] * 2 if nb == 3 else [])


def test_frame_sharded_window_shares_the_factor(monkeypatch, weights):
    """Two thread-ranks (conftest.ThreadGroup, exchange="nccl") with phi = 0.7: every rank holds bitwise-equal totals
    of both ranks (so applies a bitwise-equal factor), and the gathered latents equal the unsharded window's."""
    from conftest import ThreadGroup
    from hallo_b200.dist import shard_layout
    _install_step_stand_ins(monkeypatch)
    install_rescale_stand_ins(monkeypatch)
    f, R, size = 4, 2, 16
    inp = _inputs(f, size=size, seed=31)
    d = DDIMScheduler()
    d.set_timesteps(10)
    ts, coef = d.timesteps.tolist(), d.coef_table()
    lat = inp["sample"][:1].float()
    full = _engine(weights, f, size=size)
    full.begin_window(**_window(inp))
    full.set_schedule(ts, coef, 3.5, guidance_rescale=0.7)
    full.latents.copy_(lat)
    full.step()
    full.step()
    ref = full.latents.clone()
    ref_tot = full._bufs[("rescale.totals", 1, 4, torch.float64)].clone()
    grp = ThreadGroup(R, monkeypatch)
    layout = shard_layout(R, f)

    def rank_fn(r):
        halves, frames = layout[r]
        eng = _engine(weights, f, halves=halves, frames=frames, size=size, group=grp, group_size=R, rank_in_group=r,
                      exchange="nccl")
        eng.begin_window(**_window(inp))
        eng.set_schedule(ts, coef, 3.5, guidance_rescale=0.7)
        eng.latents.copy_(lat[:, :, list(frames)])
        eng.step()
        eng.step()
        return eng.latents.clone(), eng._bufs[("rescale.totals", R, 4, torch.float64)].clone()

    res = grp.run(rank_fn)
    got = torch.cat([x for x, _ in res], dim=2)
    tots = [t for _, t in res]
    n_local = 4 * (f // R) * size * size
    factors = [rescale_factor(t, n_local, 0.7) for t in tots]
    err = rel_l2(got, ref)
    print(f"2 thread-ranks vs unsharded, 2 DDIM steps at phi = 0.7: rel L2 = {err:.2e}; factors {factors} "
          f"(unsharded {rescale_factor(ref_tot, 4 * f * size * size, 0.7)})")
    assert torch.equal(tots[0], tots[1]) and factors[0] == factors[1] and factors[0] != 1.0
    assert torch.allclose(tots[0].sum(0), ref_tot[0], rtol=1e-4, atol=1e-4 * float(ref_tot.abs().max()))
    assert err < 1e-4


# ---------------------------------------------------------------- arguments and the graph key
BAD = (math.nan, math.inf, -math.inf, -0.1, 1.1)


def test_argument_validation(weights):
    from types import SimpleNamespace
    from hallo_b200.animate.face_animate import FaceAnimatePipeline
    from hallo_b200.driver import ClipAnimator
    two = _engine(weights, 2)
    ts, kind, table = _table(DDIMScheduler, 10)
    for bad in BAD:
        with pytest.raises(ValueError, match="guidance_rescale"):
            two.set_schedule(ts, table, 3.5, guidance_rescale=bad)
    for ok in (0.0, -0.0, 0.7, 1.0, 1):
        two.set_schedule(ts, table, 3.5, guidance_rescale=ok)
        assert two.guidance_rescale == float(ok) and math.copysign(1.0, two.guidance_rescale) == 1.0
    # the pipeline checks the keyword before any work, after the guidance_scale check
    unet = SimpleNamespace(device=torch.device("cpu"), config=SimpleNamespace(sample_size=8))
    pipe = FaceAnimatePipeline(vae=SimpleNamespace(config=SimpleNamespace(block_out_channels=(1, 2, 3, 4))),
                               reference_unet=None, denoising_unet=unet, face_locator=None, image_proj=None,
                               scheduler=None)
    args = dict(ref_image=None, face_emb=None, audio_tensor=None, face_mask=None, pixel_values_full_mask=None,
                pixel_values_face_mask=None, pixel_values_lip_mask=None, width=64, height=64, video_length=2,
                num_inference_steps=10)
    for bad in BAD:
        with pytest.raises(ValueError, match="guidance_rescale"):
            pipe(guidance_scale=3.5, guidance_rescale=bad, **args)
        with pytest.raises(NotImplementedError):                          # guidance off is refused first, as before
            pipe(guidance_scale=1.0, guidance_rescale=bad, **args)
        with pytest.raises(ValueError, match="guidance_rescale"):
            ClipAnimator(pipeline=None, audio_proj=None)(None, None, None, None, None, None, None,
                                                          guidance_rescale=bad)


def test_graph_key_changes_with_phi(weights):
    three = _engine(weights, 2, halves=(0, 1, 2))
    ts, kind, table = _table(DDIMScheduler, 10)
    three.set_schedule(ts, table, 3.5, audio_guidance=7.0)
    k0 = three._schedule_key()
    three.set_schedule(ts, table, 3.5, audio_guidance=7.0, guidance_rescale=0.7)
    k1 = three._schedule_key()
    assert k0 != k1 and k0[-1] == k1[-1] == 7.0 and 0.7 in k1
    # a captured graph is dropped when phi changes and kept when it does not
    three.graph, three._captured_with = object(), k1
    three.set_schedule(ts, table, 3.5, audio_guidance=7.0, guidance_rescale=0.7)
    assert three.graph is not None
    three.set_schedule(ts, table, 3.5, audio_guidance=7.0, guidance_rescale=0.5)
    assert three.graph is None
