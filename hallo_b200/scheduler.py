"""DDIM schedule as the reference configures it (SURVEY.md Q7): linear betas 0.00085 -> 0.012, zero-terminal-SNR
rescale, trailing timestep spacing, v-prediction, eta 0, final_alpha_cumprod = 1
(configs/inference/default.yaml:79-88, scripts/inference.py:186-193, hallo/animate/face_animate.py:285-286, 420).

Only the per-step scalar tables live here (host side, fp64 -> fp32); the update itself is the
`hallo_b200_cfg_ddim_step` kernel.  Mirrors the constructor keywords of diffusers.DDIMScheduler that the
reference passes, so `DDIMScheduler(**sched_kwargs)` keeps working at the call site.

DPMSolverMultistepScheduler is the second sampler the engine runs: DPM-Solver++ of order 1 or 2 ("2M") in the
data-prediction form, restated from the algorithm diffusers.DPMSolverMultistepScheduler documents (Lu et al. 2022,
arXiv:2211.01095), with the same constructor keywords.  Its update is the `hallo_b200_cfg_multistep_step` kernel.
`sampler_table_of` gives the engine the sampler kind and table of either class, ours or diffusers'.

EulerDiscreteScheduler and EulerAncestralDiscreteScheduler ("Euler", "Euler a") restate diffusers' classes of the same
names (release 0.27.2).  They work on x = y / alpha; the engine keeps y, so their tables are in the VP form (see
euler_table) and `latent_scales_of` converts between the two.  Euler runs on the multistep kernel; Euler-a on
`hallo_b200_cfg_ancestral_step`, with its per-step noise drawn on the host from the caller's generator.

UniPCMultistepScheduler is UniPC (bh1 / bh2, order 1 or 2, data prediction), diffusers' usual few-step sampler for
SD-family models.  Its corrector reuses the UNet evaluation the next step needs, so a step is still one forward; the
corrector and predictor together are one [n, 10] table row (unipc_table) for `hallo_b200_cfg_unipc_step`.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch


class DDIMSchedulerOutput:
    def __init__(self, prev_sample, pred_original_sample=None):
        self.prev_sample = prev_sample
        self.pred_original_sample = pred_original_sample


class DDIMScheduler:
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012,
                 beta_schedule: str = "linear", clip_sample: bool = False, set_alpha_to_one: bool = True,
                 steps_offset: int = 1, prediction_type: str = "v_prediction", rescale_betas_zero_snr: bool = True,
                 timestep_spacing: str = "trailing", **unused):
        if beta_schedule == "linear":
            betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
        elif beta_schedule == "scaled_linear":
            betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        else:
            raise NotImplementedError(beta_schedule)
        if prediction_type != "v_prediction" or clip_sample:
            raise NotImplementedError("the Hallo pipeline uses v_prediction without clipping")
        if rescale_betas_zero_snr:
            abar_sqrt = torch.cumprod(1.0 - betas, 0).sqrt()
            s0, sT = abar_sqrt[0].clone(), abar_sqrt[-1].clone()
            abar_sqrt = (abar_sqrt - sT) * s0 / (s0 - sT)
            abar = abar_sqrt ** 2
            alphas = torch.cat([abar[0:1], abar[1:] / abar[:-1]])
            betas = 1 - alphas
        self.alphas_cumprod = torch.cumprod(1.0 - betas, 0)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.num_train_timesteps = num_train_timesteps
        self.timestep_spacing = timestep_spacing
        self.steps_offset = steps_offset
        self.num_inference_steps: Optional[int] = None
        self.timesteps = torch.arange(num_train_timesteps - 1, -1, -1)

    def set_timesteps(self, num_inference_steps: int, device=None):
        self.num_inference_steps = num_inference_steps
        n, T = num_inference_steps, self.num_train_timesteps
        if self.timestep_spacing == "trailing":
            ts = np.round(np.arange(T, 0, -T / n)) - 1
        elif self.timestep_spacing == "leading":
            ts = (np.arange(0, n) * (T // n)).round()[::-1].copy() + self.steps_offset
        else:
            raise NotImplementedError(self.timestep_spacing)
        self.timesteps = torch.from_numpy(ts.astype(np.int64)).to(device)

    def scale_model_input(self, sample, timestep=None):
        return sample

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, eta: float = 0.0,
             use_clipped_model_output: bool = False, generator=None, variance_noise=None, return_dict: bool = True):
        """diffusers DDIMScheduler.step as the reference calls it (face_animate.py:420: v-prediction, eta 0):
        x0 = sqrt(a_t) x - sqrt(1-a_t) v;  eps = sqrt(a_t) v + sqrt(1-a_t) x;  prev = sqrt(a_prev) x0 + sqrt(1-a_prev) eps.
        Host/PyTorch form of what `hallo_b200_cfg_ddim_step` does on the device -- kept so the scheduler object is a
        complete stand-in at the call site (callbacks, custom loops); the engine's loop does not call it."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the scheduler")
        if eta != 0.0:
            raise NotImplementedError("eta != 0 (stochastic DDIM) is not part of the reference configuration")
        t = int(timestep)
        prev = t - self.num_train_timesteps // self.num_inference_steps
        a_t = self.alphas_cumprod[t].to(torch.float64)
        a_p = (self.alphas_cumprod[prev] if prev >= 0 else self.final_alpha_cumprod).to(torch.float64)
        sa, sb = float(a_t.sqrt()), float((1 - a_t).sqrt())
        x0 = sa * sample - sb * model_output
        eps = sa * model_output + sb * sample
        prev_sample = float(a_p.sqrt()) * x0 + float((1 - a_p).sqrt()) * eps
        if not return_dict:
            return (prev_sample,)
        return DDIMSchedulerOutput(prev_sample=prev_sample, pred_original_sample=x0)

    def coef_table(self) -> torch.Tensor:
        """[n_steps, 4] = sqrt(a_t), sqrt(1 - a_t), sqrt(a_prev), sqrt(1 - a_prev) per inference step."""
        n = self.num_inference_steps
        rows: List[List[float]] = []
        for t in self.timesteps.tolist():
            prev = t - self.num_train_timesteps // n
            a_t = self.alphas_cumprod[t].double()
            a_p = self.alphas_cumprod[prev].double() if prev >= 0 else self.final_alpha_cumprod.double()
            rows.append([float(a_t.sqrt()), float((1 - a_t).sqrt()), float(a_p.sqrt()), float((1 - a_p).sqrt())])
        return torch.tensor(rows, dtype=torch.float32)


def coef_table_of(sched) -> torch.Tensor:
    """The [n_steps, 4] table for ANY DDIM-style scheduler object that has run set_timesteps: hallo_b200's own class,
    or diffusers.DDIMScheduler as the unmodified scripts/inference.py constructs it (:186-193) -- read through the
    attributes diffusers exposes (alphas_cumprod, final_alpha_cumprod, timesteps, config.num_train_timesteps,
    config.prediction_type)."""
    if hasattr(sched, "coef_table"):
        return sched.coef_table()
    cfg = getattr(sched, "config", None)
    pred = getattr(cfg, "prediction_type", None) if cfg is not None else None
    if pred is None and isinstance(cfg, dict):
        pred = cfg.get("prediction_type")
    if pred not in (None, "v_prediction"):
        raise NotImplementedError(f"the engine's DDIM update is the v-prediction form the reference ships, got {pred!r}")
    T = int(cfg["num_train_timesteps"] if isinstance(cfg, dict) else getattr(cfg, "num_train_timesteps"))
    n = int(sched.num_inference_steps)
    rows = []
    for t in [int(x) for x in sched.timesteps]:
        prev = t - T // n
        a_t = sched.alphas_cumprod[t].double()
        a_p = sched.alphas_cumprod[prev].double() if prev >= 0 else torch.as_tensor(sched.final_alpha_cumprod).double()
        rows.append([float(a_t.sqrt()), float((1 - a_t).sqrt()), float(a_p.sqrt()), float((1 - a_p).sqrt())])
    return torch.tensor(rows, dtype=torch.float32)


def dpm_second_order_steps(n: int, solver_order: int, lower_order_final: bool = True, euler_at_final: bool = False,
                           final_sigmas_type: str = "zero") -> List[bool]:
    """Which of n steps take the second-order update, by diffusers' rule: step 0 has no history; the last step drops to
    first order with euler_at_final, with lower_order_final below 15 steps, or when the final point is sigma = 0."""
    last_first = euler_at_final or (lower_order_final and n < 15) or final_sigmas_type == "zero"
    return [solver_order == 2 and i > 0 and not (i == n - 1 and last_first) for i in range(n)]


def dpm_solver_table(alpha: Sequence[float], sigma: Sequence[float], second_order: Sequence[bool],
                     solver_type: str = "midpoint") -> torch.Tensor:
    """[n, 5] rows [alpha_i, sigma_i, a_i, b_i, c_i] of DPM-Solver++ in data prediction, x_{i+1} = a x_i + b x0_i +
    c x0_{i-1} with x0_i = alpha_i x_i - sigma_i v_i.  alpha, sigma: the n step points, then the final point.
    With lambda = log alpha - log sigma, h_i = lambda_{i+1} - lambda_i and E = alpha_{i+1} (1 - e^{-h_i}):
    a = sigma_{i+1} / sigma_i, b = E, c = 0 at first order; second order adds K (h_i / h_{i-1}) (x0_i - x0_{i-1}), K = E/2
    (midpoint) or alpha_{i+1} (1 - (1 - e^{-h_i}) / h_i) (heun).  Computed in float64 and stored as fp32.  The limits
    are taken where they are reached: alpha_0 = 0 (zero terminal SNR, lambda_0 = -inf) gives e^{-h_0} = 0 and
    h_1 / h_0 = 0; sigma_n = 0 (the final point is x0) gives a = 0 and E = alpha_n."""
    al, sg = np.asarray(alpha, np.float64), np.asarray(sigma, np.float64)
    n = len(al) - 1
    if len(sg) != n + 1 or len(second_order) != n:
        raise ValueError(f"{n + 1} alphas, {len(sg)} sigmas and {len(second_order)} order flags do not describe {n} steps")
    if solver_type not in ("midpoint", "heun"):
        raise NotImplementedError(f"solver_type {solver_type!r}: the engine implements 'midpoint' and 'heun'")
    with np.errstate(divide="ignore"):
        lam = np.log(al) - np.log(sg)
    rows = np.zeros((n, 5), np.float64)
    for i in range(n):
        a = sg[i + 1] / sg[i]
        e = al[i + 1] - a * al[i]                          # = alpha_{i+1} (1 - e^{-h_i}), finite at both limits
        b, c = e, 0.0
        if second_order[i] and i > 0:
            h, h_prev = lam[i + 1] - lam[i], lam[i] - lam[i - 1]
            rho = 0.0 if np.isinf(h_prev) else h / h_prev
            k = 0.5 * e if solver_type == "midpoint" else al[i + 1] * (1.0 + np.expm1(-h) / h)
            b, c = e + k * rho, -k * rho
        rows[i] = (al[i], sg[i], a, b, c)
    return torch.from_numpy(rows).to(torch.float32)


def _solver_alphas_cumprod(num_train_timesteps: int, beta_start: float, beta_end: float, beta_schedule: str,
                           rescale_betas_zero_snr: bool) -> torch.Tensor:
    """alpha_cumprod of the training schedule for the multistep solvers (DPM-Solver++, UniPC): DDIM's, with the
    zero-terminal-SNR value alpha_cumprod[-1] = 0 replaced by 2^-24, as diffusers does, so lambda stays finite."""
    ac = DDIMScheduler(num_train_timesteps, beta_start, beta_end, beta_schedule,
                       rescale_betas_zero_snr=rescale_betas_zero_snr).alphas_cumprod.clone()
    if rescale_betas_zero_snr:
        ac[-1] = 2.0 ** -24
    return ac


def _solver_timesteps(n: int, T: int, spacing: str, steps_offset: int) -> np.ndarray:
    """int64 [n] timesteps of the multistep solvers for "trailing", "leading" or "linspace" spacing (diffusers'
    DPMSolverMultistepScheduler / UniPCMultistepScheduler rule, which differs from DDIM's for "leading")."""
    if spacing == "trailing":
        ts = np.round(np.arange(T, 0, -T / n)) - 1
    elif spacing == "leading":
        ts = (np.arange(0, n + 1) * (T // (n + 1))).round()[::-1][:-1] + steps_offset
    else:
        ts = np.linspace(0, T - 1, n + 1).round()[::-1][:-1]
    return ts.astype(np.int64).copy()


def _solver_points(alphas_cumprod: torch.Tensor, ts: np.ndarray, final_sigmas_type: str):
    """float64 alpha, sigma at the n step points, then the final point: abar = 1 ("zero") or alpha_cumprod[0]
    ("sigma_min")."""
    ac = alphas_cumprod.double().numpy()
    abar = np.append(ac[ts], 1.0 if final_sigmas_type == "zero" else ac[0])
    return np.sqrt(abar), np.sqrt(1.0 - abar)


def _points_from_sigmas(sched, what: str):
    """float64 alpha, sigma of a diffusers-style solver object from its own n + 1 sigmas = sigma / alpha."""
    n = len(sched.timesteps)
    s = torch.as_tensor(sched.sigmas).detach().cpu().double().numpy()
    if len(s) != n + 1:
        raise ValueError(f"a {n}-step {what} schedule needs {n + 1} sigmas, got {len(s)}")
    al = 1.0 / np.sqrt(1.0 + s * s)
    with np.errstate(invalid="ignore"):
        sg = np.where(np.isinf(s), 1.0, s * al)                   # sigma / alpha = inf: alpha = 0, sigma = 1
    return al, sg


def _check_dpm_config(get) -> None:
    """NotImplementedError, naming the setting, for DPMSolverMultistepScheduler settings the engine does not run."""
    order = int(get("solver_order", 2))
    if order not in (1, 2):
        raise NotImplementedError(f"solver_order {order}: the engine runs DPM-Solver++ of order 1 or 2")
    algo = get("algorithm_type", "dpmsolver++")
    if algo != "dpmsolver++":
        raise NotImplementedError(f"algorithm_type {algo!r}: the engine runs the deterministic 'dpmsolver++'")
    if get("thresholding", False):
        raise NotImplementedError("thresholding: dynamic thresholding of x0 is not implemented")
    if get("variance_type", None) is not None:
        raise NotImplementedError(f"variance_type {get('variance_type')!r}: learned variances are not implemented")
    pred = get("prediction_type", None)
    if pred not in (None, "v_prediction"):
        raise NotImplementedError(f"prediction_type {pred!r}: the engine's update is the v-prediction form")
    st = get("solver_type", "midpoint")
    if st not in ("midpoint", "heun"):
        raise NotImplementedError(f"solver_type {st!r}: the engine implements 'midpoint' and 'heun'")


class DPMSolverMultistepScheduler:
    """DPM-Solver++ (data prediction, v-prediction model) of order 1 or 2 with the constructor keywords of
    diffusers.DPMSolverMultistepScheduler and the DDIM keywords the reference passes.  Zero-terminal-SNR rescaling
    replaces alpha_cumprod = 0 at the last training timestep by 2^-24, as diffusers does."""
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012,
                 beta_schedule: str = "linear", solver_order: int = 2, prediction_type: str = "v_prediction",
                 thresholding: bool = False, algorithm_type: str = "dpmsolver++", solver_type: str = "midpoint",
                 lower_order_final: bool = True, euler_at_final: bool = False, final_sigmas_type: str = "zero",
                 variance_type: Optional[str] = None, rescale_betas_zero_snr: bool = True,
                 timestep_spacing: str = "trailing", steps_offset: int = 1, **unused):
        kw = dict(solver_order=solver_order, prediction_type=prediction_type, thresholding=thresholding,
                  algorithm_type=algorithm_type, solver_type=solver_type, variance_type=variance_type)
        _check_dpm_config(lambda k, d=None: kw.get(k, d))
        for k in ("use_karras_sigmas", "use_exponential_sigmas", "use_beta_sigmas", "use_lu_lambdas"):
            if unused.get(k):
                raise NotImplementedError(f"{k}: only the training sigmas at the chosen timesteps are implemented")
        if final_sigmas_type not in ("zero", "sigma_min"):
            raise NotImplementedError(f"final_sigmas_type {final_sigmas_type!r}")
        if timestep_spacing not in ("trailing", "leading", "linspace"):
            raise NotImplementedError(timestep_spacing)
        self.alphas_cumprod = _solver_alphas_cumprod(num_train_timesteps, beta_start, beta_end, beta_schedule,
                                                     rescale_betas_zero_snr)
        self.num_train_timesteps = num_train_timesteps
        self.solver_order, self.solver_type = int(solver_order), solver_type
        self.lower_order_final, self.euler_at_final = lower_order_final, euler_at_final
        self.final_sigmas_type = final_sigmas_type
        self.timestep_spacing, self.steps_offset = timestep_spacing, steps_offset
        self.num_inference_steps: Optional[int] = None
        self.timesteps = torch.arange(num_train_timesteps - 1, -1, -1)
        self.sigmas = None
        self._step_index: Optional[int] = None
        self._x0_prev: Optional[torch.Tensor] = None

    def set_timesteps(self, num_inference_steps: int, device=None):
        n = num_inference_steps
        ts = _solver_timesteps(n, self.num_train_timesteps, self.timestep_spacing, self.steps_offset)
        self.num_inference_steps = n
        self.timesteps = torch.from_numpy(ts).to(device)
        self._alpha, self._sigma = _solver_points(self.alphas_cumprod, ts, self.final_sigmas_type)
        self.sigmas = torch.from_numpy(self._sigma / self._alpha).to(torch.float32)
        self._second = dpm_second_order_steps(n, self.solver_order, self.lower_order_final, self.euler_at_final,
                                              self.final_sigmas_type)
        self._step_index = None
        self._x0_prev = None

    def scale_model_input(self, sample, timestep=None):
        return sample

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, generator=None, variance_noise=None,
             return_dict: bool = True):
        """One DPM-Solver++ step in diffusers' form (dpm_solver_first_order_update /
        multistep_dpm_solver_second_order_update), float64 on the host.  Stateful like diffusers: the step index
        comes from the first timestep seen after set_timesteps, the previous data estimate is kept between calls.
        Host form of what `hallo_b200_cfg_multistep_step` does on the device; the engine's loop does not call it."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the scheduler")
        if self._step_index is None:
            self._step_index = self.timesteps.tolist().index(int(timestep))
        i = self._step_index
        al, sg = self._alpha, self._sigma
        with np.errstate(divide="ignore"):
            lam = np.log(al) - np.log(sg)
        x, v = sample.double(), model_output.double()
        x0 = al[i] * x - sg[i] * v
        h = lam[i + 1] - lam[i]
        em1 = float(np.expm1(-h))                                   # e^{-h} - 1
        prev = (sg[i + 1] / sg[i]) * x - (al[i + 1] * em1) * x0
        if self._second[i] and self._x0_prev is not None:
            r0 = (lam[i] - lam[i - 1]) / h
            d1 = (1.0 / r0) * (x0 - self._x0_prev)
            if self.solver_type == "midpoint":
                prev = prev - 0.5 * (al[i + 1] * em1) * d1
            else:
                prev = prev + (al[i + 1] * (em1 / h + 1.0)) * d1
        self._x0_prev = x0
        self._step_index = i + 1
        prev_sample = prev.to(sample.dtype)
        if not return_dict:
            return (prev_sample,)
        return DDIMSchedulerOutput(prev_sample=prev_sample, pred_original_sample=x0.to(sample.dtype))

    def coef_table(self) -> torch.Tensor:
        """[n_steps, 5] rows [alpha, sigma, a, b, c] for `hallo_b200_cfg_multistep_step` (see dpm_solver_table)."""
        if self.num_inference_steps is None:
            raise ValueError("run set_timesteps first")
        return dpm_solver_table(self._alpha, self._sigma, self._second, self.solver_type)


# ---------------------------------------------------------------------------------------------------- Euler, Euler-a
# diffusers' Euler classes keep x in the "VE" form x = y / alpha, sigma = sqrt((1 - abar) / abar), and feed the UNet
# scale_model_input(x) = x / sqrt(sigma^2 + 1) = alpha x = y, the VP latent the engine stores.  So the engine keeps y,
# and every step is one [alpha, sigma_vp, a, b, d] row: y' = a y + b x0 + d z with x0 = alpha y - sigma_vp v, which is
# diffusers' v-prediction pred_original_sample -sigma / sqrt(sigma^2 + 1) v + x / (sigma^2 + 1).
EULER_KINDS = {"EulerDiscreteScheduler": "multistep", "EulerAncestralDiscreteScheduler": "ancestral"}


def euler_table(sigmas: Sequence[float], ancestral: bool) -> torch.Tensor:
    """[n, 5] rows [alpha_i, sigma_vp_i, a_i, b_i, d_i] of Euler (ancestral=False, d = 0) or Euler-a in the VP form,
    from the n + 1 VE sigmas (the step points, then the final sigma_n = 0).  With alpha_i = 1 / sqrt(1 + sigma_i^2) and
    sigma_vp_i = sigma_i alpha_i: Euler-a's sigma_up = sqrt(sigma_{i+1}^2 (sigma_i^2 - sigma_{i+1}^2) / sigma_i^2) and
    sigma_down = sqrt(sigma_{i+1}^2 - sigma_up^2) (Euler: sigma_up = 0, sigma_down = sigma_{i+1}), then
    a = alpha_{i+1} sigma_down / (sigma_i alpha_i), b = alpha_{i+1} (1 - sigma_down / sigma_i), d = alpha_{i+1} sigma_up.
    Computed in float64 and stored as fp32.  sigma_i alpha_i stays finite (about 1) where sigma_i is large (about 4096
    at step 0 of a zero-terminal-SNR schedule), and sigma_i = inf takes its limit (alpha = 0, sigma_vp = 1)."""
    s = np.asarray(sigmas, np.float64)
    n = len(s) - 1
    if n < 1 or s[-1] != 0.0:
        raise ValueError(f"an Euler schedule needs n + 1 sigmas ending in 0, got {len(s)} ending in {s[-1] if n >= 0 else None}")
    al = 1.0 / np.sqrt(1.0 + s * s)
    with np.errstate(invalid="ignore"):
        sv = np.where(np.isinf(s), 1.0, s * al)
    rows = np.zeros((n, 5), np.float64)
    for i in range(n):
        s0, s1 = s[i], s[i + 1]
        if not ancestral:
            up, down = 0.0, s1
        elif np.isinf(s0):
            up, down = s1, 0.0
        else:
            up = np.sqrt(s1 * s1 * (s0 * s0 - s1 * s1) / (s0 * s0))
            down = np.sqrt(max(s1 * s1 - up * up, 0.0))
        ratio = 0.0 if np.isinf(s0) else down / s0
        rows[i] = (al[i], sv[i], al[i + 1] * down / sv[i], al[i + 1] * (1.0 - ratio), al[i + 1] * up)
    return torch.from_numpy(rows).to(torch.float32)


def _check_euler_config(get) -> None:
    """NotImplementedError, naming the setting, for Euler / Euler-a settings the engine does not run."""
    pred = get("prediction_type", None)
    if pred not in (None, "v_prediction"):
        raise NotImplementedError(f"prediction_type {pred!r}: the engine's update is the v-prediction form")
    for k in ("use_karras_sigmas", "use_exponential_sigmas", "use_beta_sigmas"):
        if get(k, False):
            raise NotImplementedError(f"{k}: only the training sigmas at the chosen timesteps are implemented")
    interp = get("interpolation_type", "linear")
    if interp != "linear":
        raise NotImplementedError(f"interpolation_type {interp!r}: the engine's sigmas are interpolated linearly")
    tt = get("timestep_type", "discrete")
    if tt != "discrete":
        raise NotImplementedError(f"timestep_type {tt!r}: the UNet is conditioned on discrete training timesteps")
    fst = get("final_sigmas_type", "zero")
    if fst != "zero":
        raise NotImplementedError(f"final_sigmas_type {fst!r}: the engine's last step lands on sigma = 0")
    if get("trained_betas", None) is not None:
        raise NotImplementedError("trained_betas: the engine's stand-ins build betas from beta_schedule")


def randn_tensor(shape, generator=None, device=None, dtype=None) -> torch.Tensor:
    """diffusers.utils.torch_utils.randn_tensor for one generator: a CPU generator draws on the CPU, then moves."""
    if isinstance(generator, list):
        if len(generator) != 1:
            raise NotImplementedError("one generator per batch element: the engine runs a batch of one")
        generator = generator[0]
    device = torch.device(device) if device is not None else torch.device("cpu")
    rand_device = device
    if generator is not None and generator.device.type != device.type:
        if generator.device.type != "cpu":
            raise ValueError(f"cannot draw {device} noise from a {generator.device} generator")
        rand_device = torch.device("cpu")
    return torch.randn(shape, generator=generator, device=rand_device, dtype=dtype).to(device)


class EulerDiscreteScheduler:
    """Euler (Karras et al. 2022, arXiv:2206.00364, Algorithm 2 without churn) on the VE sigmas of the training schedule,
    with the constructor keywords of diffusers.EulerDiscreteScheduler and the reference's DDIM configuration as the
    defaults.  Restates the diffusers 0.27.2 release: fp32 timesteps and sigmas (np.interp of the training sigmas at the
    timesteps, then a final 0), init_noise_sigma = max sigma for "linspace" / "trailing" spacing and sqrt(max^2 + 1)
    otherwise, and a step() that draws one noise tensor from the generator on every call.  Zero-terminal-SNR rescaling
    replaces alpha_cumprod = 0 at the last training timestep by 2^-24, as diffusers does."""
    order = 1
    _ancestral = False

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012,
                 beta_schedule: str = "linear", trained_betas=None, prediction_type: str = "v_prediction",
                 interpolation_type: str = "linear", use_karras_sigmas: bool = False, timestep_spacing: str = "trailing",
                 timestep_type: str = "discrete", steps_offset: int = 1, rescale_betas_zero_snr: bool = True,
                 **unused):
        kw = dict(prediction_type=prediction_type, interpolation_type=interpolation_type, trained_betas=trained_betas,
                  use_karras_sigmas=use_karras_sigmas, timestep_type=timestep_type, **unused)
        _check_euler_config(lambda k, d=None: kw.get(k, d))
        if timestep_spacing not in ("trailing", "leading", "linspace"):
            raise NotImplementedError(f"timestep_spacing {timestep_spacing!r}")
        ac = DDIMScheduler(num_train_timesteps, beta_start, beta_end, beta_schedule,
                           rescale_betas_zero_snr=rescale_betas_zero_snr).alphas_cumprod.clone()
        if rescale_betas_zero_snr:
            ac[-1] = 2.0 ** -24
        self.alphas_cumprod = ac
        self.num_train_timesteps = num_train_timesteps
        self.timestep_spacing, self.steps_offset = timestep_spacing, steps_offset
        self.num_inference_steps: Optional[int] = None
        self.timesteps = torch.from_numpy(np.linspace(0, num_train_timesteps - 1, num_train_timesteps)[::-1].copy()
                                          ).to(torch.float32)
        self.sigmas = torch.cat([(((1 - ac) / ac) ** 0.5).flip(0), torch.zeros(1)])
        self._step_index: Optional[int] = None

    @property
    def init_noise_sigma(self):
        m = self.sigmas.max()
        return m if self.timestep_spacing in ("linspace", "trailing") else (m ** 2 + 1) ** 0.5

    def set_timesteps(self, num_inference_steps: int, device=None):
        n, T = num_inference_steps, self.num_train_timesteps
        if self.timestep_spacing == "linspace":
            ts = np.linspace(0, T - 1, n, dtype=np.float32)[::-1].copy()
        elif self.timestep_spacing == "leading":
            ts = (np.arange(0, n) * (T // n)).round()[::-1].copy().astype(np.float32)
            ts += self.steps_offset
        else:
            ts = np.arange(T, 0, -T / n).round().copy().astype(np.float32)
            ts -= 1
        train = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()        # fp32, as diffusers
        sig = np.interp(ts, np.arange(0, len(train)), train)
        self.num_inference_steps = n
        self.timesteps = torch.from_numpy(ts.astype(np.float32)).to(device)
        self.sigmas = torch.cat([torch.from_numpy(sig).to(torch.float32), torch.zeros(1)])
        self._step_index = None

    def _init_step_index(self, timestep):
        cand = (self.timesteps.cpu() == float(timestep)).nonzero()
        self._step_index = int(cand[1 if len(cand) > 1 else 0])

    def scale_model_input(self, sample, timestep=None):
        if self._step_index is None:
            self._init_step_index(timestep)
        sigma = self.sigmas[self._step_index]
        return sample / ((sigma ** 2 + 1) ** 0.5)

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, s_churn: float = 0.0,
             s_tmin: float = 0.0, s_tmax: float = float("inf"), s_noise: float = 1.0, generator=None,
             return_dict: bool = True):
        """One step in diffusers' VE form, float64 on the host; Euler-a adds sigma_up times the step's noise draw.
        Stateful like diffusers: the step index comes from the first timestep seen after set_timesteps.  Host form of
        what the engine's step kernels do on y = alpha x; the engine's loop does not call it."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the scheduler")
        if s_churn != 0.0:
            raise NotImplementedError("s_churn: stochastic churn is not implemented (the engine runs s_churn = 0)")
        if self._step_index is None:
            self._init_step_index(timestep)
        i = self._step_index
        s0, s1 = float(self.sigmas[i]), float(self.sigmas[i + 1])
        x, v = sample.double(), model_output.double()
        x0 = v * (-s0 / (s0 ** 2 + 1) ** 0.5) + x / (s0 ** 2 + 1)
        noise = randn_tensor(model_output.shape, generator=generator, device=model_output.device,
                             dtype=model_output.dtype)
        if self._ancestral:
            up = (s1 ** 2 * (s0 ** 2 - s1 ** 2) / s0 ** 2) ** 0.5
            down = (s1 ** 2 - up ** 2) ** 0.5
            prev = x + (x - x0) / s0 * (down - s0) + noise.double() * up
        else:
            prev = x + (x - x0) / s0 * (s1 - s0)
        self._step_index = i + 1
        prev_sample = prev.to(model_output.dtype)
        if not return_dict:
            return (prev_sample,)
        return DDIMSchedulerOutput(prev_sample=prev_sample, pred_original_sample=x0.to(model_output.dtype))

    def coef_table(self) -> torch.Tensor:
        """[n_steps, 5] rows [alpha, sigma_vp, a, b, d] in the VP form (see euler_table): read by
        `hallo_b200_cfg_multistep_step` for Euler (d = c = 0) and `hallo_b200_cfg_ancestral_step` for Euler-a."""
        if self.num_inference_steps is None:
            raise ValueError("run set_timesteps first")
        return euler_table(self.sigmas.double().numpy(), self._ancestral)


class EulerAncestralDiscreteScheduler(EulerDiscreteScheduler):
    """Euler-a: Euler to sigma_down, then fresh noise of standard deviation sigma_up (Karras et al. 2022), with the
    constructor keywords of diffusers.EulerAncestralDiscreteScheduler.  step() draws randn_tensor(model_output.shape,
    dtype=model_output.dtype) from the generator on every call, the last one (sigma_up = 0) included, as diffusers
    0.27.2 does; the engine reads the same draws from a per-window noise table."""
    _ancestral = True


# ----------------------------------------------------------------------------------------------------------- UniPC
# UniPC (Zhao et al. 2023, arXiv:2302.04867) in data prediction: step i sees the sample s_i the UNet ran on, forms
# m_i = alpha_i s_i - sigma_i v_i, corrects the sample with the new m_i (UniC, reusing the evaluation the next step
# needs anyway), then predicts s_{i+1} from the corrected sample (UniP).  Both are linear in the sample, the previous
# corrected sample L and the data estimates m_i, m_{i-1}, m_{i-2}, so each step is one table row.
def unipc_orders(n: int, solver_order: int, lower_order_final: bool = True) -> List[int]:
    """The order of each of n steps by diffusers' rule: min(solver_order, i + 1), and with lower_order_final also at
    most n - i, so the last step is first order whatever n is (unlike DPM-Solver++, which lowers it below 15 steps)."""
    return [min(solver_order, n - i if lower_order_final else solver_order, i + 1) for i in range(n)]


def _unipc_bh(h: float, solver_type: str) -> float:
    """B(h) of the bh1 / bh2 variants, with hh = -h (data prediction)."""
    return -h if solver_type == "bh1" else float(np.expm1(-h))


def unipc_table(alpha: Sequence[float], sigma: Sequence[float], disable_corrector: Sequence[int] = (),
                solver_order: int = 2, solver_type: str = "bh2", lower_order_final: bool = True) -> torch.Tensor:
    """[n, 10] rows [alpha_i, sigma_i, kx, kL, k0, k1, k2, pc, p0, p1] of UniPC (data prediction, order 1 or 2, bh1
    or bh2), for the engine's step s -> s' with m_i = alpha_i s - sigma_i v:
      corrector  c = kx s + kL L + k0 m_i + k1 m_{i-1} + k2 m_{i-2}  (kx = 1, the rest 0 at i = 0, where i - 1 is in
                 disable_corrector; otherwise kx = 0 and L is the previous step's corrected sample)
      predictor  s' = pc c + p0 m_i + p1 m_{i-1}
    alpha, sigma: the n step points, then the final point.  With lambda = log alpha - log sigma, the update from point
    a to point b (h = lambda_b - lambda_a) is (sigma_b / sigma_a) x + E m_a - alpha_b B(h) sum rho_k D_k, where
    E = alpha_b (1 - e^{-h}), B(h) = -h (bh1) or e^{-h} - 1 (bh2), and D_k the scaled differences of diffusers'
    multistep_uni_p_bh_update / multistep_uni_c_bh_update.  The predictor of order 2 uses rho = 0.5, as diffusers
    hard-codes; the corrector uses rho = 0.5 at order 1 and solves diffusers' 2 x 2 system R rho = b at order 2.  The
    corrector at step i has the order of step i - 1's predictor.  Computed in float64 and stored as fp32.
    The limits are taken where they are reached: alpha_0 = 0 (lambda_0 = -inf) gives E = alpha_1 and drops every
    difference against point 0 (its r_k is infinite); sigma_n = 0 gives pc = 0 and p0 = alpha_n at first order.  A
    second-order last step onto sigma = 0 (r_k -> 0) and bh1's corrector after alpha_0 = 0 (B = -inf) have no finite
    limit and raise NotImplementedError."""
    al, sg = np.asarray(alpha, np.float64), np.asarray(sigma, np.float64)
    n = len(al) - 1
    if len(sg) != n + 1 or n < 1:
        raise ValueError(f"{len(al)} alphas and {len(sg)} sigmas do not describe a UniPC schedule")
    if solver_type not in ("bh1", "bh2"):
        raise NotImplementedError(f"solver_type {solver_type!r}: the engine runs UniPC 'bh1' and 'bh2'")
    if solver_order not in (1, 2):
        raise NotImplementedError(f"solver_order {solver_order}: the engine runs UniPC of order 1 or 2")
    orders = unipc_orders(n, solver_order, lower_order_final)
    if orders[-1] == 2 and sg[n] == 0.0:
        raise NotImplementedError("lower_order_final=False with a final sigma of 0 (final_sigmas_type='zero'): a "
                                  "second-order UniPC step onto sigma = 0 diverges; keep lower_order_final=True")
    with np.errstate(divide="ignore"):
        lam = np.log(al) - np.log(sg)
    skip = {int(k) for k in disable_corrector}

    def base(a, b):
        """sigma_b / sigma_a and E = alpha_b (1 - e^{-h}) = alpha_b - (sigma_b / sigma_a) alpha_a (finite at both ends)."""
        r = sg[b] / sg[a]
        return r, al[b] - r * al[a]

    def inv_rk(prev, a, h):
        """1 / r_k, r_k = (lambda_prev - lambda_a) / h; 0 where lambda_prev = -inf."""
        return 0.0 if np.isinf(lam[prev]) else h / (lam[prev] - lam[a])

    rows = np.zeros((n, 10), np.float64)
    for i in range(n):
        kx, kl, k0, k1, k2 = 1.0, 0.0, 0.0, 0.0, 0.0
        if i > 0 and (i - 1) not in skip:                          # UniC: from point i - 1 to i, with m_i
            kx = 0.0
            kl, e = base(i - 1, i)
            h = lam[i] - lam[i - 1]
            bh = _unipc_bh(h, solver_type)
            if not np.isfinite(bh):
                raise NotImplementedError(f"solver_type {solver_type!r} with alpha = 0 at step point {i - 1}: the "
                                          "corrector's B(h) is infinite; use 'bh2' or an alpha_cumprod above 0")
            if orders[i - 1] == 1:
                rho_t, rho_p_rk = 0.5, 0.0
            else:
                hh = -h
                phi = np.expm1(hh) / hh - 1.0                      # h_phi_k at k = 1, then k = 2
                b1 = phi / bh
                b2 = (phi / hh - 0.5) * 2.0 / bh
                q = inv_rk(i - 2, i - 1, h)
                if q == 0.0:                                       # r_k = -inf: rho_0 -> 0, rho_t -> b1
                    rho_t, rho_p_rk = b1, 0.0
                else:                                              # solve [[1, 1], [r_k, 1]] rho = [b1, b2]
                    rk = 1.0 / q
                    rho0 = (b2 - b1) / (rk - 1.0)
                    rho_t, rho_p_rk = b1 - rho0, rho0 * q
            k0 = -al[i] * bh * rho_t
            k2 = -al[i] * bh * rho_p_rk
            k1 = e - k0 - k2
        pc, e = base(i, i + 1)                                     # UniP: from point i to i + 1, with the corrected c
        p0, p1 = e, 0.0
        if orders[i] == 2:
            h = lam[i + 1] - lam[i]
            p1 = -al[i + 1] * _unipc_bh(h, solver_type) * 0.5 * inv_rk(i - 1, i, h)
            p0 = e - p1
        rows[i] = (al[i], sg[i], kx, kl, k0, k1, k2, pc, p0, p1)
    if not np.isfinite(rows).all():
        raise ValueError(f"UniPC rows {sorted(set(np.nonzero(~np.isfinite(rows))[0].tolist()))} are not finite: "
                         "the schedule repeats a point or ends above its start")
    return torch.from_numpy(rows).to(torch.float32)


def _check_unipc_config(get) -> None:
    """NotImplementedError, naming the setting, for UniPCMultistepScheduler settings the engine does not run."""
    if not get("predict_x0", True):
        raise NotImplementedError("predict_x0=False: the engine runs UniPC in data prediction (predict_x0=True)")
    order = int(get("solver_order", 2))
    if order not in (1, 2):
        raise NotImplementedError(f"solver_order {order}: the engine runs UniPC of order 1 or 2")
    st = get("solver_type", "bh2")
    if st not in ("bh1", "bh2"):
        raise NotImplementedError(f"solver_type {st!r}: the engine runs UniPC 'bh1' and 'bh2'")
    if get("thresholding", False):
        raise NotImplementedError("thresholding: dynamic thresholding of x0 is not implemented")
    pred = get("prediction_type", None)
    if pred not in (None, "v_prediction"):
        raise NotImplementedError(f"prediction_type {pred!r}: the engine's update is the v-prediction form")
    for k in ("use_karras_sigmas", "use_exponential_sigmas", "use_beta_sigmas", "use_flow_sigmas"):
        if get(k, False):
            raise NotImplementedError(f"{k}: only the training sigmas at the chosen timesteps are implemented")
    if get("solver_p", None) is not None:
        raise NotImplementedError("solver_p: an external predictor scheduler is not implemented")


class UniPCMultistepScheduler:
    """UniPC (bh1 / bh2, order 1 or 2, data prediction, v-prediction model) with the constructor keywords of
    diffusers.UniPCMultistepScheduler and the DDIM keywords the reference passes.  step() restates the update of
    diffusers 0.27.2, the release the reference pins (step / multistep_uni_c_bh_update / multistep_uni_p_bh_update,
    order-2 predictor with rho = 0.5), with two keywords of later releases, chosen as for DPMSolverMultistepScheduler:
      - final_sigmas_type, default "zero" (the last step lands on sigma = 0, x = m).  diffusers 0.27.2 has no such
        keyword and always ends on the smallest training sigma, which final_sigmas_type="sigma_min" reproduces.
      - rescale_betas_zero_snr, default True, the reference's setting; alpha_cumprod = 0 at the last training timestep
        is replaced by 2^-24, as diffusers does.
    One deliberate difference: diffusers' first-order predictor still adds -alpha_t B(h) * 0, which is NaN for bh1
    onto a final sigma of 0 (B(h) = -inf); here that step is its limit, the data estimate m.
    The timestep spacing and alpha_cumprod are DPMSolverMultistepScheduler's.  Its update is the
    `hallo_b200_cfg_unipc_step` kernel; step() is the float64 host form, which the engine's loop does not call."""
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012,
                 beta_schedule: str = "linear", trained_betas=None, solver_order: int = 2,
                 prediction_type: str = "v_prediction", thresholding: bool = False,
                 dynamic_thresholding_ratio: float = 0.995, sample_max_value: float = 1.0, predict_x0: bool = True,
                 solver_type: str = "bh2", lower_order_final: bool = True, disable_corrector: Sequence[int] = (),
                 solver_p=None, use_karras_sigmas: bool = False, timestep_spacing: str = "trailing",
                 steps_offset: int = 1, final_sigmas_type: str = "zero", rescale_betas_zero_snr: bool = True,
                 **unused):
        kw = dict(predict_x0=predict_x0, solver_order=solver_order, solver_type=solver_type, thresholding=thresholding,
                  prediction_type=prediction_type, use_karras_sigmas=use_karras_sigmas, solver_p=solver_p, **unused)
        _check_unipc_config(lambda k, d=None: kw.get(k, d))
        if trained_betas is not None:
            raise NotImplementedError("trained_betas: the engine's stand-ins build betas from beta_schedule")
        if final_sigmas_type not in ("zero", "sigma_min"):
            raise NotImplementedError(f"final_sigmas_type {final_sigmas_type!r}")
        if final_sigmas_type == "zero" and not lower_order_final and solver_order == 2:
            raise NotImplementedError("lower_order_final=False with final_sigmas_type='zero': a second-order UniPC "
                                      "step onto sigma = 0 diverges; keep lower_order_final=True")
        if timestep_spacing not in ("trailing", "leading", "linspace"):
            raise NotImplementedError(f"timestep_spacing {timestep_spacing!r}")
        self.alphas_cumprod = _solver_alphas_cumprod(num_train_timesteps, beta_start, beta_end, beta_schedule,
                                                     rescale_betas_zero_snr)
        self.num_train_timesteps = num_train_timesteps
        self.solver_order, self.solver_type = int(solver_order), solver_type
        self.lower_order_final = bool(lower_order_final)
        self.disable_corrector = [int(k) for k in disable_corrector]
        self.final_sigmas_type = final_sigmas_type
        self.timestep_spacing, self.steps_offset = timestep_spacing, steps_offset
        self.num_inference_steps: Optional[int] = None
        self.timesteps = torch.arange(num_train_timesteps - 1, -1, -1)
        self.sigmas = None
        self._step_index: Optional[int] = None

    def set_timesteps(self, num_inference_steps: int, device=None):
        n = num_inference_steps
        ts = _solver_timesteps(n, self.num_train_timesteps, self.timestep_spacing, self.steps_offset)
        self.num_inference_steps = n
        self.timesteps = torch.from_numpy(ts).to(device)
        self._alpha, self._sigma = _solver_points(self.alphas_cumprod, ts, self.final_sigmas_type)
        self.sigmas = torch.from_numpy(self._sigma / self._alpha).to(torch.float32)
        with np.errstate(divide="ignore"):
            self._lambda = np.log(self._alpha) - np.log(self._sigma)
        self._step_index = None
        self.model_outputs: List[Optional[torch.Tensor]] = [None] * self.solver_order
        self.lower_order_nums = 0
        self.last_sample: Optional[torch.Tensor] = None
        self.this_order = 1

    def scale_model_input(self, sample, timestep=None):
        return sample

    def _bh_update(self, a: int, b: int, x, m_a, m_k, k: Optional[int], model_t, rhos):
        """diffusers' bh update from point a to point b in data prediction, float64:
        x_b = (sigma_b / sigma_a) x - alpha_b h_phi_1 m_a - alpha_b B(h) (rho_0 D_1 [+ rho_t (model_t - m_a)]), with
        D_1 = (m_k - m_a) / r_k from the earlier point k (order 2; k = None at order 1).  rhos = None solves diffusers'
        system R rho = b (the order-2 corrector)."""
        al, sg, lam = self._alpha, self._sigma, self._lambda
        h = lam[b] - lam[a]
        hh = -h
        h_phi_1 = float(np.expm1(hh))
        out = (sg[b] / sg[a]) * x - (al[b] * h_phi_1) * m_a
        if k is None and model_t is None:
            return out
        bh = _unipc_bh(h, self.solver_type)
        rks = ([(lam[k] - lam[a]) / h] if k is not None else []) + [1.0]
        if rhos is None:
            R, bv, h_phi_k, fact = [], [], h_phi_1 / hh - 1.0, 1
            for j in range(1, len(rks) + 1):
                R.append([r ** (j - 1) for r in rks])
                bv.append(h_phi_k * fact / bh)
                fact *= j + 1
                h_phi_k = h_phi_k / hh - 1.0 / fact
            rhos = np.linalg.solve(np.array(R), np.array(bv)).tolist()
        res = torch.zeros_like(x)
        if k is not None:
            res = res + rhos[0] * ((m_k - m_a) / rks[0])
        if model_t is not None:
            res = res + rhos[-1] * (model_t - m_a)
        return out - (al[b] * bh) * res

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, return_dict: bool = True):
        """One UniPC step in diffusers' form, float64 on the host: the data estimate at the given sample, the corrector
        (when i > 0 and i - 1 is not in disable_corrector) with the previous step's order, then the predictor.
        Stateful like diffusers: the step index comes from the first timestep seen after set_timesteps; the data
        estimates and the last corrected sample are kept between calls.  Returns the predicted next sample."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the scheduler")
        if self._step_index is None:
            self._step_index = self.timesteps.tolist().index(int(timestep))
        i = self._step_index
        x, v = sample.double(), model_output.double()
        m = self._alpha[i] * x - self._sigma[i] * v                             # convert_model_output, at the UNet's input
        if i > 0 and (i - 1) not in self.disable_corrector and self.last_sample is not None:
            # multistep_uni_c_bh_update, from point i - 1 to i with the previous step's order: m_{i-1} is
            # model_outputs[-1], m_{i-2} is model_outputs[-2]; rho = [0.5] at order 1, solve(R, b) at order 2
            two = self.this_order == 2
            x = self._bh_update(i - 1, i, self.last_sample, self.model_outputs[-1],
                                self.model_outputs[-2] if two else None, i - 2 if two else None, m,
                                None if two else [0.5])
        self.model_outputs = self.model_outputs[1:] + [m]
        n = len(self.timesteps)
        this_order = min(self.solver_order, n - i) if self.lower_order_final else self.solver_order
        self.this_order = min(this_order, self.lower_order_nums + 1)
        self.last_sample = x
        # multistep_uni_p_bh_update, from point i to i + 1: at order 2 diffusers fixes rho_p = [0.5]
        two = self.this_order == 2
        prev = self._bh_update(i, i + 1, x, m, self.model_outputs[-2] if two else None, i - 1 if two else None, None,
                               [0.5])
        if self.lower_order_nums < self.solver_order:
            self.lower_order_nums += 1
        self._step_index = i + 1
        prev_sample = prev.to(sample.dtype)
        if not return_dict:
            return (prev_sample,)
        return DDIMSchedulerOutput(prev_sample=prev_sample, pred_original_sample=m.to(sample.dtype))

    def coef_table(self) -> torch.Tensor:
        """[n_steps, 10] rows [alpha, sigma, kx, kL, k0, k1, k2, pc, p0, p1] for `hallo_b200_cfg_unipc_step` (see
        unipc_table)."""
        if self.num_inference_steps is None:
            raise ValueError("run set_timesteps first")
        return unipc_table(self._alpha, self._sigma, self.disable_corrector, self.solver_order, self.solver_type,
                           self.lower_order_final)


def latent_scales_of(sched) -> np.ndarray:
    """float64 [n + 1]: the factor between the scheduler's own latents and the engine's y at each step point, then the
    final point.  1 / alpha_i = sqrt(1 + sigma_i^2) for the Euler classes (x = y / alpha), ones for DDIM / DPM-Solver++
    / UniPC (whose latents are y).  The final scale is 1 for all of them."""
    n = len(sched.timesteps)
    if type(sched).__name__ not in EULER_KINDS:
        return np.ones(n + 1)
    s = torch.as_tensor(sched.sigmas).detach().cpu().double().numpy()
    if len(s) != n + 1:
        raise ValueError(f"a {n}-step Euler schedule needs {n + 1} sigmas, got {len(s)}")
    return np.sqrt(1.0 + s * s)


def sampler_table_of(sched) -> Tuple[str, torch.Tensor]:
    """(kind, table) of a scheduler object that has run set_timesteps, for DenoiseEngine.set_schedule:
    ("multistep", [n, 5]) for DPMSolverMultistepScheduler -- ours, or diffusers' read through its attributes
    (config.solver_order / algorithm_type / solver_type / lower_order_final / euler_at_final / final_sigmas_type /
    thresholding / variance_type / prediction_type, timesteps, and its own sigmas = sigma / alpha, n + 1 of them) --
    ("multistep", [n, 5]) for EulerDiscreteScheduler and ("ancestral", [n, 5]) for EulerAncestralDiscreteScheduler,
    ours or diffusers' (recognised by class name, read through timesteps, sigmas and config.prediction_type /
    use_karras_sigmas / interpolation_type / timestep_type / final_sigmas_type), ("unipc", [n, 10]) for
    UniPCMultistepScheduler, ours or diffusers' (recognised by class name, read through timesteps, its own n + 1
    sigmas and config.solver_order / solver_type / predict_x0 / lower_order_final / disable_corrector /
    prediction_type / thresholding / use_karras_sigmas / solver_p), and ("ddim", [n, 4]) from coef_table_of for any
    other, DDIM-style, scheduler."""
    if isinstance(sched, DPMSolverMultistepScheduler):
        return "multistep", sched.coef_table()
    cfg = getattr(sched, "config", None)

    def get(k, d=None):
        if cfg is None:
            return d
        v = cfg.get(k, d) if isinstance(cfg, dict) else getattr(cfg, k, d)
        return d if v is None and d is not None else v

    if type(sched).__name__ == "UniPCMultistepScheduler":               # before the DPM branch: it has solver_order too
        if isinstance(sched, UniPCMultistepScheduler):
            return "unipc", sched.coef_table()
        _check_unipc_config(get)
        al, sg = _points_from_sigmas(sched, "UniPC")
        return "unipc", unipc_table(al, sg, get("disable_corrector", []) or [], int(get("solver_order", 2)),
                                    get("solver_type", "bh2"), bool(get("lower_order_final", True)))
    euler = EULER_KINDS.get(type(sched).__name__)
    if euler is not None:
        _check_euler_config(get)
        n = len(sched.timesteps)
        s = torch.as_tensor(sched.sigmas).detach().cpu().double().numpy()
        if len(s) != n + 1:
            raise ValueError(f"a {n}-step Euler schedule needs {n + 1} sigmas, got {len(s)}")
        return euler, euler_table(s, euler == "ancestral")
    if cfg is None or get("solver_order") is None:
        return "ddim", coef_table_of(sched)
    _check_dpm_config(get)
    n = len(sched.timesteps)
    al, sg = _points_from_sigmas(sched, "DPM-Solver++")
    second = dpm_second_order_steps(n, int(get("solver_order")), bool(get("lower_order_final", True)),
                                    bool(get("euler_at_final", False)), get("final_sigmas_type", "zero"))
    return "multistep", dpm_solver_table(al, sg, second, get("solver_type", "midpoint"))
