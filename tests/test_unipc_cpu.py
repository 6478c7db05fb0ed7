"""UniPC (bh1 / bh2, order 1 / 2, data prediction) without a GPU: the stand-in scheduler's stateful step() against an
independent float64 restatement of diffusers' UniPCMultistepScheduler.step / multistep_uni_c_bh_update /
multistep_uni_p_bh_update written here, the [n, 10] table chained against step(), finiteness at zero terminal SNR,
the order-1 corrector-free table against DPM-Solver++ of order 1, diffusers-style objects read through their
attributes, the unsupported settings, and the engine's UniPC step tail on the CPU stand-ins of tests/cpu_ops.py."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import cpu_ops
from conftest import rel_l2
from hallo_b200 import scheduler as sch
from hallo_b200.scheduler import (DDIMScheduler, DPMSolverMultistepScheduler, UniPCMultistepScheduler,
                                  dpm_solver_table, latent_scales_of, sampler_table_of, unipc_table)


class DiffusersUniPC:
    """The update of diffusers.UniPCMultistepScheduler (predict_x0=True, v-prediction), restated line by line in
    float64 torch: sigmas are the scheduler's own n + 1 sigma / alpha values."""

    def __init__(self, sigmas, timesteps, solver_order, solver_type, lower_order_final, disable_corrector):
        self.sigmas = torch.as_tensor(sigmas, dtype=torch.float64)
        self.timesteps = list(timesteps)
        self.solver_order, self.solver_type = solver_order, solver_type
        self.lower_order_final, self.disable_corrector = lower_order_final, list(disable_corrector)
        self.model_outputs = [None] * solver_order
        self.timestep_list = [None] * solver_order
        self.lower_order_nums = 0
        self.last_sample = None
        self.step_index = None
        self.this_order = None

    @staticmethod
    def _sigma_to_alpha_sigma_t(sigma):
        alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
        return alpha_t, sigma * alpha_t

    def convert_model_output(self, model_output, sample):
        alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(self.sigmas[self.step_index])
        return alpha_t * sample - sigma_t * model_output

    def _b_and_r(self, rks, hh, order):
        h_phi_1 = torch.expm1(hh)
        h_phi_k = h_phi_1 / hh - 1
        factorial_i = 1
        B_h = hh if self.solver_type == "bh1" else torch.expm1(hh)
        R, b = [], []
        for i in range(1, order + 1):
            R.append(torch.pow(rks, i - 1))
            b.append(h_phi_k * factorial_i / B_h)
            factorial_i *= i + 1
            h_phi_k = h_phi_k / hh - 1 / factorial_i
        return h_phi_1, B_h, torch.stack(R), torch.stack(b)

    def multistep_uni_p_bh_update(self, sample, order):
        m0 = self.model_outputs[-1]
        x = sample
        sigma_t, sigma_s0 = self.sigmas[self.step_index + 1], self.sigmas[self.step_index]
        alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(sigma_t)
        alpha_s0, sigma_s0 = self._sigma_to_alpha_sigma_t(sigma_s0)
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
        h = lambda_t - lambda_s0
        rks, D1s = [], []
        for i in range(1, order):
            si = self.step_index - i
            mi = self.model_outputs[-(i + 1)]
            alpha_si, sigma_si = self._sigma_to_alpha_sigma_t(self.sigmas[si])
            lambda_si = torch.log(alpha_si) - torch.log(sigma_si)
            rk = (lambda_si - lambda_s0) / h
            rks.append(rk)
            D1s.append((mi - m0) / rk)
        rks.append(torch.tensor(1.0, dtype=torch.float64))
        h_phi_1, B_h, R, b = self._b_and_r(torch.stack(rks), -h, order)
        if len(D1s) > 0:
            D1s = torch.stack(D1s, dim=1)
            rhos_p = torch.tensor([0.5], dtype=x.dtype) if order == 2 else torch.linalg.solve(R[:-1, :-1], b[:-1])
        else:
            D1s = None
        x_t_ = sigma_t / sigma_s0 * x - alpha_t * h_phi_1 * m0
        if D1s is None:
            # diffusers computes x_t_ - alpha_t * B_h * 0 here, which is NaN for bh1 onto sigma = 0 (B_h = -inf); the
            # stand-in and the engine take the first-order step's limit, x_t_
            return x_t_
        pred_res = torch.einsum("k,bkc...->bc...", rhos_p, D1s)
        return x_t_ - alpha_t * B_h * pred_res

    def multistep_uni_c_bh_update(self, this_model_output, last_sample, this_sample, order):
        m0 = self.model_outputs[-1]
        x = last_sample
        model_t = this_model_output
        sigma_t, sigma_s0 = self.sigmas[self.step_index], self.sigmas[self.step_index - 1]
        alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(sigma_t)
        alpha_s0, sigma_s0 = self._sigma_to_alpha_sigma_t(sigma_s0)
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
        h = lambda_t - lambda_s0
        rks, D1s = [], []
        for i in range(1, order):
            si = self.step_index - (i + 1)
            mi = self.model_outputs[-(i + 1)]
            alpha_si, sigma_si = self._sigma_to_alpha_sigma_t(self.sigmas[si])
            lambda_si = torch.log(alpha_si) - torch.log(sigma_si)
            rk = (lambda_si - lambda_s0) / h
            rks.append(rk)
            D1s.append((mi - m0) / rk)
        rks.append(torch.tensor(1.0, dtype=torch.float64))
        h_phi_1, B_h, R, b = self._b_and_r(torch.stack(rks), -h, order)
        D1s = torch.stack(D1s, dim=1) if len(D1s) > 0 else None
        rhos_c = torch.tensor([0.5], dtype=x.dtype) if order == 1 else torch.linalg.solve(R, b)
        x_t_ = sigma_t / sigma_s0 * x - alpha_t * h_phi_1 * m0
        corr_res = torch.einsum("k,bkc...->bc...", rhos_c[:-1], D1s) if D1s is not None else 0
        D1_t = model_t - m0
        return x_t_ - alpha_t * B_h * (corr_res + rhos_c[-1] * D1_t)

    def step(self, model_output, timestep, sample):
        if self.step_index is None:
            self.step_index = self.timesteps.index(timestep)
        use_corrector = (self.step_index > 0 and self.step_index - 1 not in self.disable_corrector
                         and self.last_sample is not None)
        model_output_convert = self.convert_model_output(model_output, sample)
        if use_corrector:
            sample = self.multistep_uni_c_bh_update(model_output_convert, self.last_sample, sample, self.this_order)
        for i in range(self.solver_order - 1):
            self.model_outputs[i] = self.model_outputs[i + 1]
            self.timestep_list[i] = self.timestep_list[i + 1]
        self.model_outputs[-1] = model_output_convert
        self.timestep_list[-1] = timestep
        if self.lower_order_final:
            this_order = min(self.solver_order, len(self.timesteps) - self.step_index)
        else:
            this_order = self.solver_order
        self.this_order = min(this_order, self.lower_order_nums + 1)
        self.last_sample = sample
        prev_sample = self.multistep_uni_p_bh_update(sample, self.this_order)
        if self.lower_order_nums < self.solver_order:
            self.lower_order_nums += 1
        self.step_index += 1
        return prev_sample


def _expected_timesteps(n, spacing, T=1000, steps_offset=1):
    if spacing == "trailing":
        return [int(round(T - k * T / n)) - 1 for k in range(n)]
    if spacing == "leading":
        r = T // (n + 1)
        return [k * r + steps_offset for k in range(n, 0, -1)]
    return [int(np.round(k * (T - 1) / n)) for k in range(n, 0, -1)]


def _sigmas64(s):
    """float64 sigma / alpha at the stand-in's timesteps from its alpha_cumprod, then the final point."""
    ac = s.alphas_cumprod.double()
    pts = [math.sqrt((1 - float(ac[t])) / float(ac[t])) for t in s.timesteps.tolist()]
    return pts + [0.0 if s.final_sigmas_type == "zero" else math.sqrt((1 - float(ac[0])) / float(ac[0]))]


def _disable(kind, n):
    return {"none": [], "first": [0], "all": list(range(n))}[kind]


def _chain_table(table, vs, x):
    """The kernel's arithmetic in float64 over the rows, with NaN-initialised state and zero terms skipped."""
    last = torch.full_like(x, float("nan"))
    m1 = torch.full_like(x, float("nan"))
    m2 = torch.full_like(x, float("nan"))
    for row, v in zip(table.double().tolist(), vs):
        al, sg, kx, kl, k0, k1, k2, pc, p0, p1 = row
        m = al * x - sg * v
        c = k0 * m
        for k, t in ((kx, x), (kl, last), (k1, m1), (k2, m2)):
            if k != 0.0:
                c = c + k * t
        x = pc * c + p0 * m + (p1 * m1 if p1 != 0.0 else 0.0)
        last, m2, m1 = c, m1, m
    return x


@pytest.mark.parametrize("n", [5, 10, 20, 40])
@pytest.mark.parametrize("spacing", ["trailing", "leading", "linspace"])
@pytest.mark.parametrize("disable", ["none", "first", "all"])
@pytest.mark.parametrize("lower_order_final", [True, False])
@pytest.mark.parametrize("solver_type", ["bh1", "bh2"])
@pytest.mark.parametrize("order", [1, 2])
def test_standin_step_matches_diffusers_restatement(order, solver_type, lower_order_final, disable, spacing, n):
    """Stateful step() and the chained table against the restatement, to 1e-6.  lower_order_final=False runs with
    final_sigmas_type="sigma_min" (onto sigma = 0 it raises, see test_unsupported_settings_raise)."""
    final = "zero" if lower_order_final else "sigma_min"
    dc = _disable(disable, n)
    s = UniPCMultistepScheduler(solver_order=order, solver_type=solver_type, lower_order_final=lower_order_final,
                                disable_corrector=dc, timestep_spacing=spacing, final_sigmas_type=final)
    s.set_timesteps(n)
    assert s.timesteps.tolist() == _expected_timesteps(n, spacing)
    ref = DiffusersUniPC(_sigmas64(s), s.timesteps.tolist(), order, solver_type, lower_order_final, dc)
    g = torch.Generator().manual_seed(1000 * n + 10 * order + len(dc))
    x0 = torch.randn(1, 4, 2, 4, 4, generator=g, dtype=torch.float64)
    vs = [torch.randn(x0.shape, generator=g, dtype=torch.float64) for _ in range(n)]
    x_ref = x_s = x0
    for t, v in zip(s.timesteps.tolist(), vs):
        x_ref = ref.step(v, t, x_ref)
        x_s = s.step(v, t, x_s).prev_sample
        assert torch.isfinite(x_ref).all()
        assert float((x_s - x_ref).abs().max()) <= 1e-6 * max(1.0, float(x_ref.abs().max())), t
    table = s.coef_table()
    assert tuple(table.shape) == (n, 10) and torch.isfinite(table).all()
    x_tab = _chain_table(table, vs, x0)
    assert float((x_tab - x_ref).abs().max()) <= 1e-6 * max(1.0, float(x_ref.abs().max()))
    if final == "zero":
        assert table[-1, 7].item() == 0.0 and table[-1, 8].item() == 1.0 and table[-1, 9].item() == 0.0


def test_row_kinds():
    """Row 0: no corrector and first order; row 1: order-1 corrector; row 2 on: order-2 corrector; last row first
    order (lower_order_final, even at n >= 15); disable_corrector drops exactly the rows after the listed steps."""
    for n in (10, 20):
        s = UniPCMultistepScheduler()
        s.set_timesteps(n)
        t = s.coef_table()
        assert t[0, 2:7].tolist() == [1.0, 0.0, 0.0, 0.0, 0.0] and t[0, 9].item() == 0.0
        assert t[1, 2].item() == 0.0 and t[1, 6].item() == 0.0 and t[1, 9].item() != 0.0
        assert (t[2:, 6] != 0).all() and (t[1:-1, 9] != 0).all() and t[-1, 9].item() == 0.0
    s = UniPCMultistepScheduler(disable_corrector=[0, 3])
    s.set_timesteps(10)
    t = s.coef_table()
    assert [i for i in range(10) if t[i, 2].item() == 1.0] == [0, 1, 4]
    assert sch.unipc_orders(5, 2, True) == [1, 2, 2, 2, 1] and sch.unipc_orders(5, 2, False) == [1, 2, 2, 2, 2]


@pytest.mark.parametrize("solver_type", ["bh1", "bh2"])
@pytest.mark.parametrize("n", [1, 2, 5, 10, 25, 40, 100])
def test_rows_finite_at_zero_terminal_snr(solver_type, n):
    for kw in ({}, {"final_sigmas_type": "sigma_min", "lower_order_final": False}, {"solver_order": 1}):
        s = UniPCMultistepScheduler(solver_type=solver_type, rescale_betas_zero_snr=True, **kw)
        s.set_timesteps(n)
        assert float(s.alphas_cumprod[-1]) == 2.0 ** -24 and s.timesteps[0] == 999
        assert torch.isfinite(s.coef_table()).all()
    # alpha_cumprod exactly 0 at t = 999 (DDIM's own): lambda_0 = -inf.  bh2 takes the limits; bh1's corrector after
    # point 0 has B(h) = -inf and raises, unless that corrector is disabled
    d = DDIMScheduler()
    d.set_timesteps(n)
    ac = d.alphas_cumprod.double()
    assert float(ac[999]) == 0.0
    al = [math.sqrt(float(ac[t])) for t in d.timesteps.tolist()] + [1.0]
    sg = [math.sqrt(1 - float(ac[t])) for t in d.timesteps.tolist()] + [0.0]
    if solver_type == "bh2" or n == 1:
        t = unipc_table(al, sg, solver_type=solver_type)
        assert torch.isfinite(t).all() and t[0, 0].item() == 0.0 and t[0, 8].item() == pytest.approx(al[1], rel=1e-6)
        if n > 2:
            assert t[1, 9].item() == 0.0 and t[2, 6].item() == 0.0       # differences against point 0 vanish
    else:
        with pytest.raises(NotImplementedError, match="bh1"):
            unipc_table(al, sg, solver_type=solver_type)
        assert torch.isfinite(unipc_table(al, sg, [0], solver_type=solver_type)).all()


@pytest.mark.parametrize("n", [10, 40])
def test_order1_without_corrector_is_dpm_solver_order1(n):
    """UniP of order 1 is DPM-Solver++ of order 1: on the same sigmas the rows must agree, with the corrector off."""
    s = UniPCMultistepScheduler(solver_order=1, disable_corrector=list(range(n)))
    s.set_timesteps(n)
    d = DPMSolverMultistepScheduler(solver_order=1)
    d.set_timesteps(n)
    assert s.timesteps.tolist() == d.timesteps.tolist() and torch.equal(s.sigmas, d.sigmas)
    u, m = s.coef_table(), d.coef_table()
    assert (u[:, 2] == 1).all() and (u[:, 3:7] == 0).all() and (u[:, 9] == 0).all() and (m[:, 4] == 0).all()
    assert torch.equal(u[:, :2], m[:, :2]) and torch.allclose(u[:, 7:9], m[:, 2:4], rtol=1e-6, atol=1e-7)
    # and on DDIM's own alpha_cumprod, exactly 0 at t = 999
    dd = DDIMScheduler()
    dd.set_timesteps(n)
    ac = dd.alphas_cumprod.double()
    al = [math.sqrt(float(ac[t])) for t in dd.timesteps.tolist()] + [1.0]
    sg = [math.sqrt(1 - float(ac[t])) for t in dd.timesteps.tolist()] + [0.0]
    u0 = unipc_table(al, sg, list(range(n)), solver_order=1)
    assert torch.allclose(u0[:, 7:9], dpm_solver_table(al, sg, [False] * n)[:, 2:4], rtol=1e-6, atol=1e-7)


def _diffusers_like(s, **cfg):
    """An object with diffusers' class name and attributes only (config, timesteps, sigmas)."""
    base = dict(num_train_timesteps=1000, solver_order=s.solver_order, solver_type=s.solver_type, predict_x0=True,
                lower_order_final=s.lower_order_final, disable_corrector=list(s.disable_corrector), thresholding=False,
                prediction_type="v_prediction", use_karras_sigmas=False, solver_p=None,
                final_sigmas_type=s.final_sigmas_type, timestep_spacing=s.timestep_spacing)
    base.update(cfg)
    obj = type("UniPCMultistepScheduler", (), {})()
    obj.config, obj.timesteps, obj.sigmas = SimpleNamespace(**base), s.timesteps, s.sigmas
    return obj


@pytest.mark.parametrize("kw", [{}, {"solver_type": "bh1"}, {"disable_corrector": [0, 4]},
                                {"final_sigmas_type": "sigma_min", "lower_order_final": False}, {"solver_order": 1}])
def test_diffusers_style_object_through_sampler_table_of(kw):
    s = UniPCMultistepScheduler(**kw)
    s.set_timesteps(25)
    kind, table = sampler_table_of(s)
    assert kind == "unipc" and torch.equal(table, s.coef_table())
    fake = _diffusers_like(s)
    kind, got = sampler_table_of(fake)
    assert kind == "unipc" and tuple(got.shape) == (25, 10)
    assert torch.allclose(got, table, rtol=1e-5, atol=1e-6)          # the object's fp32 sigmas vs our float64 points
    fake.config = vars(fake.config)                                   # diffusers' FrozenDict config: a mapping
    assert torch.allclose(sampler_table_of(fake)[1], table, rtol=1e-5, atol=1e-6)
    assert (latent_scales_of(fake) == 1.0).all() and (latent_scales_of(s) == 1.0).all()


def test_unipc_object_never_reaches_the_dpm_branch(monkeypatch):
    def no(*a, **k):
        raise AssertionError("DPM-Solver++ code reached")
    monkeypatch.setattr(sch, "_check_dpm_config", no)
    monkeypatch.setattr(sch, "dpm_solver_table", no)
    monkeypatch.setattr(sch, "dpm_second_order_steps", no)
    s = UniPCMultistepScheduler()
    s.set_timesteps(10)
    assert sampler_table_of(_diffusers_like(s))[0] == "unipc"
    assert sampler_table_of(s)[0] == "unipc"


@pytest.mark.parametrize("setting,value", [("predict_x0", False), ("solver_order", 3), ("thresholding", True),
                                           ("prediction_type", "epsilon"), ("use_karras_sigmas", True),
                                           ("use_exponential_sigmas", True), ("use_beta_sigmas", True),
                                           ("solver_type", "bh3"), ("solver_p", object())])
def test_unsupported_settings_raise(setting, value):
    s = UniPCMultistepScheduler()
    s.set_timesteps(10)
    with pytest.raises(NotImplementedError, match=setting):
        sampler_table_of(_diffusers_like(s, **{setting: value}))
    with pytest.raises(NotImplementedError, match=setting):
        UniPCMultistepScheduler(**{setting: value})


def test_second_order_last_step_onto_sigma_zero_raises():
    with pytest.raises(NotImplementedError, match="lower_order_final"):
        UniPCMultistepScheduler(lower_order_final=False, final_sigmas_type="zero")
    s = UniPCMultistepScheduler(lower_order_final=False, final_sigmas_type="sigma_min")
    s.set_timesteps(10)
    s.final_sigmas_type = "zero"
    s.sigmas = torch.cat([s.sigmas[:-1], torch.zeros(1)])
    with pytest.raises(NotImplementedError, match="lower_order_final"):
        sampler_table_of(_diffusers_like(s))
    assert torch.isfinite(sampler_table_of(_diffusers_like(s, lower_order_final=True))[1]).all()


# ---------------------------------------------------------------- engine plan (CPU stand-ins)
def op_cfg_unipc_step(model_out, latents, last_sample, x0_hist, x0_hist2, coef, step, *, guidance):
    """PyTorch stand-in for hallo_b200_cfg_unipc_step (include/hallo_b200.h)."""
    _, cl, f, h, w = latents.shape
    n = f * h * w
    mo = model_out.float()[:, :cl]
    vu, vc = mo[:n], mo[n:2 * n]
    v = (vu + guidance * (vc - vu)).reshape(f, h, w, cl).permute(3, 0, 1, 2).unsqueeze(0)
    al, sg, kx, kl, k0, k1, k2, pc, p0, p1 = [float(z) for z in coef[int(step[0])]]
    m = al * latents - sg * v
    c = k0 * m
    for k, t in ((kx, latents), (kl, last_sample), (k1, x0_hist), (k2, x0_hist2)):
        if k != 0.0:
            c = c + k * t
    new = pc * c + p0 * m + (p1 * x0_hist if p1 != 0.0 else 0.0)
    latents.copy_(new)
    last_sample.copy_(c)
    x0_hist2.copy_(x0_hist)
    x0_hist.copy_(m)
    return latents


def test_engine_unipc_plan_matches_host_loop(monkeypatch):
    from hallo_b200 import ops
    from hallo_b200.engine import DenoiseEngine, PackedWeights
    from hallo_b200.spec import UNetConfig
    from hallo_b200.synth import host_threads, synth_inputs, synth_state_dict
    torch.set_num_threads(host_threads())
    cpu_ops.install(monkeypatch)
    monkeypatch.setattr(ops, "cfg_unipc_step", op_cfg_unipc_step)
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
    s = UniPCMultistepScheduler()
    s.set_timesteps(10)
    kind, table = sampler_table_of(s)
    x = lat0.clone()
    for i, t in enumerate(s.timesteps.tolist()[:4]):           # host loop: forward_only + CFG + the scheduler's step()
        eng.set_schedule(s.timesteps.tolist(), table, 3.5, kind)
        mo = eng.forward_only(x, step=i)
        x = s.step(mo[:1] + 3.5 * (mo[1:] - mo[:1]), t, x).prev_sample
    eng.set_schedule(s.timesteps.tolist(), table, 3.5, kind)
    eng.latents.copy_(lat0)
    for buf in (eng.last_sample, eng.x0_hist, eng.x0_hist2):   # row 0 must read no state
        buf.fill_(float("nan"))
    for _ in range(4):
        eng.step()
    assert int(eng.step_idx) == 4 and torch.isfinite(eng.latents).all()
    assert rel_l2(eng.latents, x) < 2e-4
    assert torch.equal(run_ddim(), ddim_first)                  # back to DDIM on the same engine
    with pytest.raises(ValueError):
        eng.set_schedule(s.timesteps.tolist(), table, 3.5, "multistep")    # a [n, 10] table is not a [n, 5] one
