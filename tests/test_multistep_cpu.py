"""DPM-Solver++ (order 1 / 2, data prediction) without a GPU: the stand-in scheduler's timesteps and [n, 5] table
against a float64 restatement of the update written here, the stateful host step() against the table, the order-1
table against the DDIM path, diffusers-style scheduler objects read through their attributes, and the engine's
multistep step tail on the CPU stand-ins of tests/cpu_ops.py."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import cpu_ops
from conftest import rel_l2
from hallo_b200.scheduler import (DDIMScheduler, DPMSolverMultistepScheduler, coef_table_of, dpm_solver_table,
                                  sampler_table_of)


def _points(ac, timesteps, final_abar):
    """alpha, sigma (float64) at the step points, then the final point."""
    abar = [float(ac[t]) for t in timesteps] + [final_abar]
    return [math.sqrt(a) for a in abar], [math.sqrt(1.0 - a) for a in abar]


def _lam(al, sg):
    return -math.inf if al == 0.0 else (math.inf if sg == 0.0 else math.log(al) - math.log(sg))


def _restated_step(al, sg, i, x, x0, x0_prev, second, solver_type):
    """x_{i+1} from the update as written (float64): E = alpha_{i+1} (1 - e^{-h}), order 1 = (sigma_{i+1} / sigma_i) x + E x0,
    order 2 adds E D1 / 2 (midpoint) or alpha_{i+1} (1 - (1 - e^{-h}) / h) D1 (heun), D1 = (x0 - x0_prev) h_i / h_{i-1}."""
    h = _lam(al[i + 1], sg[i + 1]) - _lam(al[i], sg[i])
    one_m = 1.0 - math.exp(-h)
    e = al[i + 1] * one_m
    out = (sg[i + 1] / sg[i]) * x + e * x0
    if second:
        h_prev = _lam(al[i], sg[i]) - _lam(al[i - 1], sg[i - 1])
        d1 = (x0 - x0_prev) * (0.0 if math.isinf(h_prev) else h / h_prev)
        out = out + (0.5 * e * d1 if solver_type == "midpoint" else al[i + 1] * (1.0 - one_m / h) * d1)
    return out


def _second_flags(n, order, lower_order_final, final_sigmas_type, euler_at_final=False):
    flags = []
    for i in range(n):
        last_first = i == n - 1 and (euler_at_final or (lower_order_final and n < 15) or final_sigmas_type == "zero")
        flags.append(order == 2 and i > 0 and not last_first)
    return flags


@pytest.mark.parametrize("n", [10, 20, 25, 40])
def test_standin_timesteps_and_finite_table(n):
    s = DPMSolverMultistepScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="linear", clip_sample=False,
                                    steps_offset=1, prediction_type="v_prediction", rescale_betas_zero_snr=True,
                                    timestep_spacing="trailing")
    s.set_timesteps(n)
    d = DDIMScheduler()
    d.set_timesteps(n)
    assert s.timesteps.tolist() == d.timesteps.tolist() and s.timesteps[0] == 999
    if n == 40:
        assert s.timesteps.tolist() == list(range(999, 0, -25))
    assert s.order == 1 and s.init_noise_sigma == 1.0
    assert len(s.sigmas) == n + 1 and float(s.sigmas[-1]) == 0.0
    assert float(s.alphas_cumprod[-1]) == 2.0 ** -24                 # diffusers' stand-in for zero terminal SNR
    t = s.coef_table()
    assert tuple(t.shape) == (n, 5) and torch.isfinite(t).all()
    assert float(t[0, 4]) == 0.0                                     # step 0 never reads the history
    assert float(t[-1, 2]) == 0.0 and float(t[-1, 3]) == 1.0          # sigma_n = 0: x_n = x0


@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("solver_type", ["midpoint", "heun"])
@pytest.mark.parametrize("final_sigmas_type", ["zero", "sigma_min"])
@pytest.mark.parametrize("lower_order_final", [True, False])
@pytest.mark.parametrize("n", [10, 20])
def test_table_matches_float64_restatement(order, solver_type, final_sigmas_type, lower_order_final, n):
    s = DPMSolverMultistepScheduler(solver_order=order, solver_type=solver_type, final_sigmas_type=final_sigmas_type,
                                    lower_order_final=lower_order_final)
    s.set_timesteps(n)
    ac = s.alphas_cumprod.double()
    al, sg = _points(ac, s.timesteps.tolist(), 1.0 if final_sigmas_type == "zero" else float(ac[0]))
    flags = _second_flags(n, order, lower_order_final, final_sigmas_type)
    table = s.coef_table().double()
    g = torch.Generator().manual_seed(n + 7 * order)
    x = torch.randn(4, 3, 8, 8, generator=g, dtype=torch.float64)
    x0_prev = torch.full_like(x, float("nan"))
    for i in range(n):
        v = torch.randn(x.shape, generator=g, dtype=torch.float64)
        x0 = al[i] * x - sg[i] * v
        want = _restated_step(al, sg, i, x, x0, x0_prev, flags[i], solver_type)
        ta, ts, a, b, c = table[i].tolist()
        assert abs(ta - al[i]) <= 1e-6 * al[i] + 1e-12 and abs(ts - sg[i]) <= 1e-6
        assert (c == 0.0) == (not flags[i])
        got = a * x + b * x0 + (c * x0_prev if c != 0.0 else 0.0)
        assert torch.isfinite(want).all()
        assert float((got - want).abs().max()) <= 1e-6 * max(1.0, float(want.abs().max())), i
        x, x0_prev = want, x0


@pytest.mark.parametrize("solver_type", ["midpoint", "heun"])
@pytest.mark.parametrize("n", [10, 20])
def test_stateful_step_equals_table_chain(solver_type, n):
    s = DPMSolverMultistepScheduler(solver_type=solver_type, final_sigmas_type="sigma_min", lower_order_final=False)
    s.set_timesteps(n)
    table = s.coef_table().double()
    g = torch.Generator().manual_seed(3)
    x_host = x_tab = torch.randn(1, 4, 3, 8, 8, generator=g, dtype=torch.float64)
    hist = torch.full_like(x_tab, float("nan"))
    for i, t in enumerate(s.timesteps.tolist()):
        v = torch.randn(x_tab.shape, generator=g, dtype=torch.float64)
        out = s.step(v, t, x_host)
        x_host = out.prev_sample
        al, sg, a, b, c = table[i].tolist()
        x0 = al * x_tab - sg * v
        x_tab = a * x_tab + b * x0 + (c * hist if c != 0.0 else 0.0)
        hist = x0
        assert torch.allclose(out.pred_original_sample, x0, rtol=1e-5, atol=1e-5)
    assert rel_l2(x_host, x_tab) < 1e-6
    # a fresh set_timesteps restarts the step index and drops the history
    s.set_timesteps(n)
    v = torch.randn(x_tab.shape, generator=g, dtype=torch.float64)
    al, sg, a, b, _ = table[0].tolist()
    assert torch.allclose(s.step(v, 999, x_tab, return_dict=False)[0], a * x_tab + b * (al * x_tab - sg * v), atol=1e-6)


def test_order1_table_from_ddim_alphas_reproduces_ddim():
    """DPM-Solver++ of order 1 IS the DDIM (eta 0) update.  Built from the DDIM scheduler's own alpha_cumprod, which is
    exactly 0 at t = 999 (lambda_0 = -inf), the table must reproduce DDIM's coef_table update over the whole schedule."""
    d = DDIMScheduler()
    d.set_timesteps(40)
    ac = d.alphas_cumprod.double()
    assert float(ac[999]) == 0.0
    al, sg = _points(ac, d.timesteps.tolist(), float(d.final_alpha_cumprod))
    table = dpm_solver_table(al, sg, [False] * 40).double()
    assert torch.isfinite(table).all()
    ddim = coef_table_of(d).double()
    g = torch.Generator().manual_seed(11)
    x_ddim = x_dpm = torch.randn(1, 4, 3, 8, 8, generator=g, dtype=torch.float64)
    for i in range(40):
        v = torch.randn(x_dpm.shape, generator=g, dtype=torch.float64)
        sa, sb, pa, pb = ddim[i].tolist()
        x_ddim = pa * (sa * x_ddim - sb * v) + pb * (sa * v + sb * x_ddim)
        al_i, sg_i, a, b, c = table[i].tolist()
        assert c == 0.0
        x_dpm = a * x_dpm + b * (al_i * x_dpm - sg_i * v)
        assert float((x_dpm - x_ddim).abs().max()) <= 1e-6 * max(1.0, float(x_ddim.abs().max())), i


def _diffusers_like(s, **cfg):
    base = dict(num_train_timesteps=1000, solver_order=s.solver_order, algorithm_type="dpmsolver++",
                solver_type=s.solver_type, lower_order_final=s.lower_order_final, euler_at_final=s.euler_at_final,
                final_sigmas_type=s.final_sigmas_type, thresholding=False, variance_type=None,
                prediction_type="v_prediction")
    base.update(cfg)
    return SimpleNamespace(config=SimpleNamespace(**base), timesteps=s.timesteps, sigmas=s.sigmas,
                           alphas_cumprod=s.alphas_cumprod)


def test_diffusers_style_object_through_sampler_table_of():
    s = DPMSolverMultistepScheduler()
    s.set_timesteps(25)
    kind, table = sampler_table_of(s)
    assert kind == "multistep" and torch.equal(table, s.coef_table())
    fake = _diffusers_like(s)
    kind, got = sampler_table_of(fake)
    assert kind == "multistep" and tuple(got.shape) == (25, 5)
    assert torch.allclose(got, table, rtol=2e-6, atol=1e-7)            # the object's fp32 sigmas vs our float64 points
    fake.config = vars(fake.config)                                     # diffusers' FrozenDict config: a mapping
    assert torch.allclose(sampler_table_of(fake)[1], table, rtol=2e-6, atol=1e-7)
    # euler_at_final / final point sigma_min: the last row's order follows the object's config
    s2 = DPMSolverMultistepScheduler(final_sigmas_type="sigma_min", lower_order_final=False)
    s2.set_timesteps(25)
    assert float(s2.coef_table()[-1, 4]) != 0.0
    assert float(sampler_table_of(_diffusers_like(s2, euler_at_final=True))[1][-1, 4]) == 0.0
    # a sigma = inf first point (alpha_cumprod exactly 0) takes the limit alpha = 0, sigma = 1
    d = DDIMScheduler()
    d.set_timesteps(25)
    ac = d.alphas_cumprod.double()
    sig = torch.tensor([math.sqrt((1 - float(ac[t])) / float(ac[t])) if float(ac[t]) > 0 else math.inf
                        for t in d.timesteps.tolist()] + [0.0], dtype=torch.float64)
    _, t_inf = sampler_table_of(SimpleNamespace(config=_diffusers_like(s).config, timesteps=d.timesteps, sigmas=sig))
    al, sg = _points(ac, d.timesteps.tolist(), 1.0)
    assert torch.isfinite(t_inf).all() and float(t_inf[0, 0]) == 0.0 and float(t_inf[0, 1]) == 1.0
    assert torch.allclose(t_inf, dpm_solver_table(al, sg, _second_flags(25, 2, True, "zero")), rtol=1e-6, atol=1e-7)
    # a scheduler without solver_order stays on the DDIM path, unchanged
    ddim_fake = SimpleNamespace(config=SimpleNamespace(num_train_timesteps=1000, prediction_type="v_prediction"),
                                num_inference_steps=25, timesteps=d.timesteps, alphas_cumprod=d.alphas_cumprod,
                                final_alpha_cumprod=d.final_alpha_cumprod)
    kind, t4 = sampler_table_of(ddim_fake)
    assert kind == "ddim" and torch.equal(t4, coef_table_of(d))
    assert sampler_table_of(d)[0] == "ddim" and torch.equal(sampler_table_of(d)[1], d.coef_table())


@pytest.mark.parametrize("setting,value", [("solver_order", 3), ("algorithm_type", "sde-dpmsolver++"),
                                           ("thresholding", True), ("variance_type", "learned_range"),
                                           ("prediction_type", "epsilon")])
def test_unsupported_settings_raise(setting, value):
    s = DPMSolverMultistepScheduler()
    s.set_timesteps(10)
    with pytest.raises(NotImplementedError, match=setting):
        sampler_table_of(_diffusers_like(s, **{setting: value}))
    with pytest.raises(NotImplementedError, match=setting):
        DPMSolverMultistepScheduler(**{setting: value})


# ---------------------------------------------------------------- engine plan (CPU stand-ins)
def op_cfg_multistep_step(model_out, latents, x0_hist, coef, step, *, guidance):
    """PyTorch stand-in for hallo_b200_cfg_multistep_step (include/hallo_b200.h)."""
    _, cl, f, h, w = latents.shape
    n = f * h * w
    mo = model_out.float()[:, :cl]
    vu, vc = mo[:n], mo[n:2 * n]
    v = (vu + guidance * (vc - vu)).reshape(f, h, w, cl).permute(3, 0, 1, 2).unsqueeze(0)
    al, sg, a, b, c = [float(z) for z in coef[int(step[0])]]
    x0 = al * latents - sg * v
    new = a * latents + b * x0
    if c != 0.0:
        new = new + c * x0_hist
    latents.copy_(new)
    x0_hist.copy_(x0)
    return latents


def test_engine_multistep_plan_matches_host_loop(monkeypatch):
    from hallo_b200 import ops
    from hallo_b200.engine import DenoiseEngine, PackedWeights
    from hallo_b200.spec import UNetConfig
    from hallo_b200.synth import host_threads, synth_inputs, synth_state_dict
    torch.set_num_threads(host_threads())
    cpu_ops.install(monkeypatch)
    monkeypatch.setattr(ops, "cfg_multistep_step", op_cfg_multistep_step)
    cfg = UNetConfig()
    W = PackedWeights(synth_state_dict(cfg, seed=0), cfg, torch.device("cpu"), torch.float32)
    inp = synth_inputs(cfg, 8, 8, 2, seed=4)
    for k in inp["banks"]:
        inp["banks"][k] = inp["banks"][k].float()
    lat0 = inp["sample"][:1].clone()
    eng = DenoiseEngine(W, 8, 8, 2)
    eng.begin_window(encoder_hidden_states=inp["encoder_hidden_states"], audio_embedding=inp["audio_embedding"],
                     mask_cond_fea=inp["mask_cond_fea"], full_mask=inp["full_mask"], face_mask=inp["face_mask"],
                     lip_mask=inp["lip_mask"], motion_scale=inp["motion_scale"], banks=inp["banks"])
    ddim = DDIMScheduler()
    ddim.set_timesteps(40)

    def run_ddim():
        eng.set_schedule(ddim.timesteps.tolist(), ddim.coef_table(), 3.5)
        eng.latents.copy_(lat0)
        eng.step()
        eng.step()
        return eng.latents.clone()

    ddim_first = run_ddim()
    s = DPMSolverMultistepScheduler()
    s.set_timesteps(10)
    x = lat0.clone()
    for i, t in enumerate(s.timesteps.tolist()[:3]):           # host loop: forward_only + CFG + the scheduler's step()
        eng.set_schedule(s.timesteps.tolist(), s.coef_table(), 3.5, "multistep")
        mo = eng.forward_only(x, step=i)
        x = s.step(mo[:1] + 3.5 * (mo[1:] - mo[:1]), t, x).prev_sample
    kind, table = sampler_table_of(s)
    eng.set_schedule(s.timesteps.tolist(), table, 3.5, kind)
    eng.latents.copy_(lat0)
    eng.x0_hist.fill_(float("nan"))                             # step 0 must not read the history
    for _ in range(3):
        eng.step()
    assert int(eng.step_idx) == 3 and torch.isfinite(eng.latents).all()
    assert float(table[1, 4]) != 0.0 and rel_l2(eng.latents, x) < 2e-4
    assert torch.equal(run_ddim(), ddim_first)                  # back to DDIM on the same engine
    with pytest.raises(ValueError):
        eng.set_schedule(s.timesteps.tolist(), table, 3.5)      # a [n, 5] table is not a DDIM table
