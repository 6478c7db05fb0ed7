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
        ac = DDIMScheduler(num_train_timesteps, beta_start, beta_end, beta_schedule,
                           rescale_betas_zero_snr=rescale_betas_zero_snr).alphas_cumprod.clone()
        if rescale_betas_zero_snr:
            ac[-1] = 2.0 ** -24
        self.alphas_cumprod = ac
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
        n, T = num_inference_steps, self.num_train_timesteps
        if self.timestep_spacing == "trailing":
            ts = np.round(np.arange(T, 0, -T / n)) - 1
        elif self.timestep_spacing == "leading":
            ts = (np.arange(0, n + 1) * (T // (n + 1))).round()[::-1][:-1] + self.steps_offset
        else:
            ts = np.linspace(0, T - 1, n + 1).round()[::-1][:-1]
        ts = ts.astype(np.int64)
        self.num_inference_steps = n
        self.timesteps = torch.from_numpy(ts.copy()).to(device)
        ac = self.alphas_cumprod.double().numpy()
        abar = np.append(ac[ts], 1.0 if self.final_sigmas_type == "zero" else ac[0])
        self._alpha, self._sigma = np.sqrt(abar), np.sqrt(1.0 - abar)       # step points, then the final point
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


def sampler_table_of(sched) -> Tuple[str, torch.Tensor]:
    """(kind, table) of a scheduler object that has run set_timesteps, for DenoiseEngine.set_schedule:
    ("multistep", [n, 5]) for DPMSolverMultistepScheduler -- ours, or diffusers' read through its attributes
    (config.solver_order / algorithm_type / solver_type / lower_order_final / euler_at_final / final_sigmas_type /
    thresholding / variance_type / prediction_type, timesteps, and its own sigmas = sigma / alpha, n + 1 of them) --
    and ("ddim", [n, 4]) from coef_table_of for any other, DDIM-style, scheduler."""
    if isinstance(sched, DPMSolverMultistepScheduler):
        return "multistep", sched.coef_table()
    cfg = getattr(sched, "config", None)

    def get(k, d=None):
        v = cfg.get(k, d) if isinstance(cfg, dict) else getattr(cfg, k, d)
        return d if v is None and d is not None else v

    if cfg is None or get("solver_order") is None:
        return "ddim", coef_table_of(sched)
    _check_dpm_config(get)
    n = len(sched.timesteps)
    s = torch.as_tensor(sched.sigmas).detach().cpu().double().numpy()
    if len(s) != n + 1:
        raise ValueError(f"a {n}-step DPM-Solver++ schedule needs {n + 1} sigmas, got {len(s)}")
    al = 1.0 / np.sqrt(1.0 + s * s)
    with np.errstate(invalid="ignore"):
        sg = np.where(np.isinf(s), 1.0, s * al)                   # sigma / alpha = inf: alpha = 0, sigma = 1
    second = dpm_second_order_steps(n, int(get("solver_order")), bool(get("lower_order_final", True)),
                                    bool(get("euler_at_final", False)), get("final_sigmas_type", "zero"))
    return "multistep", dpm_solver_table(al, sg, second, get("solver_type", "midpoint"))
