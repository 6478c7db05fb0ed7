"""CPU tests of guidance limited to an interval (`guidance_interval`): argument validation and its order against the
guidance_scale check, the per-step mask for all five samplers, the cond-only companion engine's window and shared state,
the engine loop (guided and unguided steps mixed) against a host loop for every sampler with 2 and 3 branches and with
and without guidance rescale, the op sequence of an interval that covers every step, and a frame-sharded window over two
thread-ranks.  Everything runs on the PyTorch stand-ins of tests/cpu_ops.py."""
import math

import pytest
import torch

from conftest import rel_l2
from test_audio_guidance_cpu import (SAMPLERS, _engine, _inputs, _install_step_stand_ins, _table, _window, _sig,
                                     guide3_f64)
from test_guidance_rescale_cpu import host_update, install_rescale_stand_ins, rescale_noise_cfg_f64
from hallo_b200.engine import check_guidance_interval, guided_steps
from hallo_b200.scheduler import DDIMScheduler, EulerDiscreteScheduler


@pytest.fixture(scope="module")
def weights():
    from hallo_b200.engine import PackedWeights
    from hallo_b200.spec import UNetConfig
    from hallo_b200.synth import host_threads, synth_state_dict
    torch.set_num_threads(host_threads())
    cfg = UNetConfig()
    return PackedWeights(synth_state_dict(cfg, seed=0), cfg, torch.device("cpu"), torch.float32)


# ---------------------------------------------------------------- arguments
BAD = (5.0, (1.0,), (1.0, 2.0, 3.0), "ab", (None, 3.0), (math.nan, 500.0), (100.0, math.inf), (-math.inf, 0.0),
       (900.0, 100.0))


def test_argument_validation(weights):
    from types import SimpleNamespace
    from hallo_b200.animate.face_animate import FaceAnimatePipeline
    from hallo_b200.driver import ClipAnimator
    for bad in BAD:
        with pytest.raises(ValueError, match="guidance_interval"):
            check_guidance_interval(bad)
    assert check_guidance_interval(None) is None
    assert check_guidance_interval((100, 900)) == (100.0, 900.0)
    assert check_guidance_interval([500.0, 500.0]) == (500.0, 500.0)
    assert check_guidance_interval(torch.tensor([1.5, 2.5])) == (1.5, 2.5)
    unet = SimpleNamespace(device=torch.device("cpu"), config=SimpleNamespace(sample_size=8))
    pipe = FaceAnimatePipeline(vae=SimpleNamespace(config=SimpleNamespace(block_out_channels=(1, 2, 3, 4))),
                               reference_unet=None, denoising_unet=unet, face_locator=None, image_proj=None,
                               scheduler=None)
    args = dict(ref_image=None, face_emb=None, audio_tensor=None, face_mask=None, pixel_values_full_mask=None,
                pixel_values_face_mask=None, pixel_values_lip_mask=None, width=64, height=64, video_length=2,
                num_inference_steps=10)
    for bad in BAD:
        with pytest.raises(ValueError, match="guidance_interval"):
            pipe(guidance_scale=3.5, guidance_interval=bad, **args)
        with pytest.raises(NotImplementedError):                          # guidance off is refused first, as before
            pipe(guidance_scale=1.0, guidance_interval=bad, **args)
        with pytest.raises(ValueError, match="guidance_interval"):
            ClipAnimator(pipeline=None, audio_proj=None)(None, None, None, None, None, None, None,
                                                          guidance_interval=bad)
    two = _engine(weights, 2)
    ts, kind, table = _table(DDIMScheduler, 10)
    with pytest.raises(ValueError, match="guided"):
        two.set_schedule(ts, table, 3.5, guided=[True] * 9)


# ---------------------------------------------------------------- the per-step mask
@pytest.mark.parametrize("cls", SAMPLERS, ids=lambda c: c.__name__)
def test_guided_mask(cls):
    """Step i is guided iff t_lo <= timesteps[i] <= t_hi, both ends closed, in the scheduler's own units (floats for
    the Euler classes)."""
    ts, _, _ = _table(cls, 10)
    assert len(ts) == 10 and all(a > b for a, b in zip(ts, ts[1:]))
    assert guided_steps(ts, None) is None
    # closed ends: an interval whose ends are timesteps 6 and 3 guides steps 3..6
    m = guided_steps(ts, (ts[6], ts[3]))
    assert m == [3 <= i <= 6 for i in range(10)], (ts, m)
    # an end just inside the next step leaves that step out
    lo, hi = math.nextafter(float(ts[6]), math.inf), math.nextafter(float(ts[3]), -math.inf)
    assert guided_steps(ts, (lo, hi)) == [4 <= i <= 5 for i in range(10)]
    assert guided_steps(ts, (ts[4], ts[4])) == [i == 4 for i in range(10)]
    assert guided_steps(ts, (-1e9, 1e9)) == [True] * 10
    assert guided_steps(ts, (ts[0] + 1, ts[0] + 2)) == [False] * 10              # no step: the window runs unguided
    if cls is EulerDiscreteScheduler:
        # linspace spacing gives fractional float timesteps: they are compared as they are, not rounded
        e = EulerDiscreteScheduler(timestep_spacing="linspace")
        e.set_timesteps(7)                                   # 999 / 6 apart: 832.5, 666.0, 499.5, ...
        ts = e.timesteps.tolist()
        t1 = ts[1]
        assert t1 != int(t1)
        assert guided_steps(ts, (t1, t1)) == [i == 1 for i in range(7)]
        assert guided_steps(ts, (math.floor(t1), math.floor(t1))) == [False] * 7
        assert guided_steps(e.timesteps, (math.floor(t1), math.ceil(t1))) == [i == 1 for i in range(7)]


def test_set_schedule_keeps_the_main_graph(weights):
    """The mask is not part of the main engine's graph key; an all-guided mask is the path without an interval and
    builds no companion; a mixed mask builds the cond-only companion over the main engine's state."""
    eng = _engine(weights, 2)
    ts, kind, table = _table(DDIMScheduler, 10)
    eng.set_schedule(ts, table, 3.5)
    eng.graph, eng._captured_with = object(), eng._schedule_key()
    g = eng.graph
    eng.set_schedule(ts, table, 3.5, guided=[True] * 10)
    assert eng.guided is None and eng._cond is None and eng.cond_engine() is None and eng.graph is g
    eng.set_schedule(ts, table, 3.5, guided=[False] * 10)               # no window yet: the companion waits for one
    assert eng._cond is None and eng.graph is g
    with pytest.raises(RuntimeError, match="begin_window"):
        eng.step()


def test_companion_window_and_shared_state(monkeypatch, weights):
    """The companion has shard halves (1,) over the same frames, the cond half's window inputs (ref_index (f + g) % 2,
    bank half 1, cond masks) and the main engine's state tensors at the same addresses; a new window of the main
    engine reaches it; changing the mask re-captures neither engine."""
    from hallo_b200.engine import Shard
    _install_step_stand_ins(monkeypatch)
    f = 4
    inp = _inputs(f)
    fr = (2, 3)
    eng = _engine(weights, f, halves=(0, 1, 2), frames=fr)
    eng.begin_window(**_window(inp))
    ts, kind, table = _table(DDIMScheduler, 10)
    eng.set_schedule(ts, table, 3.5, audio_guidance=6.0, guided=[i % 2 == 0 for i in range(10)])
    c = eng.cond_engine()
    assert c is eng._cond and c.nb == 1 and tuple(c.shard.halves) == (1,) and tuple(c.shard.frames) == fr
    for name in ("latents", "x0_hist", "last_sample", "x0_hist2", "step_idx", "t_table", "coef", "coef_ms", "coef_uni"):
        assert getattr(c, name) is getattr(eng, name), name
    assert c.window["ref_index"].tolist() == [(f + g) % 2 for g in fr]
    ref = _engine(weights, f, halves=(1,), frames=fr)
    ref.begin_window(**_window(inp))
    w1 = eng.window
    for k, v in ref.window.items():
        if isinstance(v, torch.Tensor):
            assert torch.equal(c.window[k], v), k
    for lv, L in enumerate((64, 16, 4, 1)):                              # the cond half of the main engine's masks
        assert torch.equal(c.window[f"mask.lip.{lv}"], w1[f"mask.lip.{lv}"].view(3, -1)[1])
    assert c.guidance == 1.0 and c.guidance_rescale == 0.0 and c.audio_guidance is None
    # a new window of the main engine is set up on the companion before its next step
    inp2 = _inputs(f, seed=9)
    eng.begin_window(**_window(inp2))
    assert eng.cond_engine() is c
    ref.begin_window(**_window(inp2))
    assert torch.equal(c.window["mask_cond"], ref.window["mask_cond"])
    # the mask is not in either graph key
    eng.graph, eng._captured_with = object(), eng._schedule_key()
    c.graph, c._captured_with = object(), c._schedule_key()
    g, gc = eng.graph, c.graph
    eng.set_schedule(ts, table, 3.5, audio_guidance=6.0, guided=[i < 3 for i in range(10)])
    assert eng.graph is g and eng.cond_engine() is c and c.graph is gc
    eng.set_schedule(ts, table, 3.5, audio_guidance=6.0)
    assert eng.graph is g and eng.cond_engine() is None and eng._cond is c
    assert Shard().halves == (0, 1)


# ---------------------------------------------------------------- the engine loop against the host loop
def _host_v(mo, nb, s, sa, phi, guided):
    """v of one step from a forward of every half mo [nb, ...] (float64): the combine (+ rescale) when guided, v_c
    when not."""
    if not guided:
        return mo[1:2]
    v = mo[0:1] + s * (mo[1:2] - mo[0:1]) if nb == 2 else guide3_f64(mo[0:1], mo[1:2], mo[2:3], s, sa)
    return rescale_noise_cfg_f64(v, mo[1:2], phi) if phi > 0 else v


@pytest.mark.parametrize("phi", [0.0, 0.7])
@pytest.mark.parametrize("nb", [2, 3])
def test_engine_loop_matches_host(monkeypatch, weights, nb, phi):
    """Every sampler, 3 steps unguided / guided / unguided (the interval holds step 1 alone): the engine
    against a host loop of the main engine's forward_only, whose guided steps take the float64 combine (and rescale)
    and whose unguided steps take the cond half v_c alone, then the sampler's table row.  Histories carry across the
    switches.  Unguided steps issue no combine or rescale op and run the companion's forward on the cond rows only."""
    from hallo_b200 import ops
    _install_step_stand_ins(monkeypatch)
    install_rescale_stand_ins(monkeypatch)
    calls = []
    for name in ("cfg_rescale_stats", "cfg_rescale_apply", "cfg_guide3_step", "conv3x3"):
        fn = getattr(ops, name)
        monkeypatch.setattr(ops, name, lambda *a, _n=name, _f=fn, **kw: (calls.append((_n, a[0].shape[0])),
                                                                          _f(*a, **kw))[1])
    f, steps, s = 2, 3, 3.5
    sa = 6.0 if nb == 3 else None
    inp = _inputs(f, seed=13)
    eng = _engine(weights, f, halves=tuple(range(nb)))
    eng.begin_window(**_window(inp))
    lat0 = inp["sample"][:1].float()
    for cls in SAMPLERS:
        ts, kind, table = _table(cls, 10)
        mask = guided_steps(ts, (ts[1], ts[1]))
        assert mask[:steps] == [False, True, False]
        noise = torch.randn(10, 4, f, 8, 8, generator=torch.Generator().manual_seed(2)) if kind == "ancestral" else None
        eng.set_schedule(ts, table, s, kind, noise=noise, audio_guidance=sa, guidance_rescale=phi)
        x, state = lat0.double(), {}
        for i in range(steps):
            mo = eng.forward_only(x.float(), step=i).double()
            v = _host_v(mo, nb, s, sa or 0.0, phi, mask[i])
            x = host_update(kind, table[i], x, v, state, None if noise is None else noise[i].double().unsqueeze(0))
        eng.set_schedule(ts, table, s, kind, noise=noise, audio_guidance=sa, guidance_rescale=phi, guided=mask)
        eng.latents.copy_(lat0)
        calls.clear()
        per_step = []
        for i in range(steps):
            n0 = len(calls)
            eng.step()
            per_step.append(calls[n0:])
        got = eng.latents.clone()
        err = rel_l2(got, x)
        print(f"{cls.__name__}, nb = {nb}, phi = {phi}: engine vs host, {steps} steps with 2 unguided: rel L2 = "
              f"{err:.2e}")
        assert err < 1e-5, cls.__name__
        assert int(eng.step_idx) == steps
        for i, cs in enumerate(per_step):
            names = {n for n, _ in cs}
            frames = {r for n, r in cs if n == "conv3x3"}                # the frame batch of every 3x3 conv
            if mask[i]:
                assert frames == {nb * f}, (i, frames)
                assert ("cfg_guide3_step" in names) == (nb == 3 and phi == 0.0)
                assert ("cfg_rescale_apply" in names) == (phi > 0)
            else:
                assert frames == {f} and not names & {"cfg_guide3_step", "cfg_rescale_stats", "cfg_rescale_apply"}
    c = eng._cond
    assert torch.equal(c.model_pair[:8 * 8 * f], torch.zeros(8 * 8 * f, 8))        # the [0 | v_c] pair's zero half


def test_interval_over_every_step_issues_the_same_ops_as_none(monkeypatch, weights):
    """An interval that holds every step gives the op sequence of no interval (names, shapes, views, arguments), for
    every sampler, and builds no companion."""
    from hallo_b200 import ops
    _install_step_stand_ins(monkeypatch)
    names = [n for n in dir(ops) if not n.startswith("_") and callable(getattr(ops, n))]
    calls = []
    for name in names:
        fn = getattr(ops, name)
        if not getattr(fn, "__module__", "").startswith(("hallo_b200.ops", "cpu_ops", "test_")):
            continue
        monkeypatch.setattr(ops, name, lambda *a, _n=name, _f=fn, **kw: (
            calls.append((_n, _sig(a), tuple(sorted((k, _sig(v)) for k, v in kw.items())))), _f(*a, **kw))[1])
    f = 2
    inp = _inputs(f, seed=3)
    eng = _engine(weights, f)
    eng.begin_window(**_window(inp))
    lat0 = inp["sample"][:1].float()
    for cls in SAMPLERS:
        ts, kind, table = _table(cls, 10)
        noise = torch.zeros(10, 4, f, 8, 8) if kind == "ancestral" else None
        out = []
        for iv in (None, (min(ts) - 0.5, max(ts))):
            eng.set_schedule(ts, table, 3.5, kind, noise=noise, guided=guided_steps(ts, iv))
            eng.latents.copy_(lat0)
            calls.clear()
            eng.step()
            eng.step()
            out.append((list(calls), eng.latents.clone()))
        assert out[0][0] == out[1][0] and len(out[0][0]) > 100, cls.__name__
        assert torch.equal(out[0][1], out[1][1])
        assert eng._cond is None


def test_frame_sharded_window_matches_unsharded(monkeypatch, weights):
    """Two thread-ranks (conftest.ThreadGroup, exchange="nccl"), DPM-Solver++ with steps unguided / guided / unguided:
    the gathered latents equal the unsharded window's; each rank's companion shares that rank's group and frames."""
    from conftest import ThreadGroup
    from hallo_b200.dist import shard_layout
    _install_step_stand_ins(monkeypatch)
    f, R, size, steps = 4, 2, 16, 3
    inp = _inputs(f, size=size, seed=31)
    ts, kind, table = _table(SAMPLERS[1], 10)
    mask = [i == 1 for i in range(10)]
    lat = inp["sample"][:1].float()
    full = _engine(weights, f, size=size)
    full.begin_window(**_window(inp))
    full.set_schedule(ts, table, 3.5, kind, guided=mask)
    full.latents.copy_(lat)
    for _ in range(steps):
        full.step()
    ref = full.latents.clone()
    full.set_schedule(ts, table, 3.5, kind)
    full.latents.copy_(lat)
    for _ in range(steps):
        full.step()
    guided_all = full.latents.clone()
    grp = ThreadGroup(R, monkeypatch)
    layout = shard_layout(R, f)

    def rank_fn(r):
        halves, frames = layout[r]
        eng = _engine(weights, f, halves=halves, frames=frames, size=size, group=grp, group_size=R, rank_in_group=r,
                      exchange="nccl")
        eng.begin_window(**_window(inp))
        eng.set_schedule(ts, table, 3.5, kind, guided=mask)
        c = eng.cond_engine()
        assert c.shard.group is grp and c.shard.rank_in_group == r and c.px and tuple(c.shard.frames) == frames
        eng.latents.copy_(lat[:, :, list(frames)])
        for _ in range(steps):
            eng.step()
        return eng.latents.clone()

    got = torch.cat(grp.run(rank_fn), dim=2)
    err, moved = rel_l2(got, ref), rel_l2(guided_all, ref)
    print(f"2 thread-ranks vs unsharded, {steps} DPM-Solver++ steps (unguided, guided, unguided): rel L2 = {err:.2e} "
          f"(every step guided: {moved:.2e})")
    assert err < 1e-4 and moved > 100 * err
