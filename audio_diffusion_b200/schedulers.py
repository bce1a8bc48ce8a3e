"""`DDPMScheduler` / `DDIMScheduler` — drop-ins for the diffusers classes at the call sites of the reference:
`set_timesteps`, `timesteps`, `step(...)["prev_sample"]`, `add_noise`, `alphas_cumprod`,
`final_alpha_cumprod`, `num_inference_steps`, `config.num_train_timesteps`
(audiodiffusion/pipeline_audio_diffusion.py:115,150,157,159,165-179,221-234; scripts/train_unet.py:161-164,250).

Coefficients are computed exactly as diffusers does (fp32 0-d torch tensors on the host).  `step()` is the
reference-compatible elementwise path (torch ops on whatever device the tensors live on); `step_coef()` hands
the same scalars to the fused U-Net output kernel (`UNet2DModel.forward_step`), which is what
`AudioDiffusionPipeline` uses so that no separate elementwise launch runs per step.  `DPMSolverMultistepScheduler` (the
sampler diffusers recommends for these ε-prediction models, 15-25 steps) does the same with `MultistepCoefC` and history
buffers on the device.
"""
from __future__ import annotations

import json
import math
import os
from typing import Optional

import numpy as np
import torch

from ._lib import MultistepCoefC, StepCoefC


class _Cfg(dict):
    __getattr__ = dict.__getitem__


class SchedulerOutput(dict):
    def __init__(self, prev_sample, pred_original_sample=None):
        super().__init__(prev_sample=prev_sample, pred_original_sample=pred_original_sample)
        self.prev_sample = prev_sample
        self.pred_original_sample = pred_original_sample


def randn_tensor(shape, generator, device, dtype=torch.float32) -> torch.Tensor:
    """diffusers.utils.torch_utils.randn_tensor as the schedulers use it ([3P-recall] 0.24): a CPU generator with a CUDA
    target draws on the CPU and moves the result (so CPU-seeded runs reproduce across devices)."""
    device = torch.device(device)
    if generator is not None and generator.device.type != device.type and generator.device.type == "cpu":
        return torch.randn(shape, generator=generator, device="cpu", dtype=dtype).to(device)
    return torch.randn(shape, generator=generator, device=device, dtype=dtype)


class _SchedulerBase:
    config_name = "scheduler_config.json"
    _class_name = "SchedulerBase"

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 1e-4, beta_end: float = 0.02,
                 beta_schedule: str = "linear", clip_sample: bool = True, clip_sample_range: float = 1.0,
                 prediction_type: str = "epsilon", timestep_spacing: str = "leading", steps_offset: int = 0, **extra):
        if beta_schedule != "linear" or prediction_type != "epsilon" or timestep_spacing != "leading":
            raise ValueError("b200 schedulers implement the reference defaults: linear betas, epsilon, leading")
        self.config = _Cfg(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                           beta_schedule=beta_schedule, clip_sample=clip_sample, clip_sample_range=clip_sample_range,
                           prediction_type=prediction_type, timestep_spacing=timestep_spacing,
                           steps_offset=steps_offset, _class_name=self._class_name, **extra)
        self.betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.one = torch.tensor(1.0)
        self.init_noise_sigma = 1.0
        self.num_inference_steps: Optional[int] = None
        self.timesteps = torch.from_numpy(np.arange(0, num_train_timesteps)[::-1].copy())

    # -- diffusers-compatible API ----------------------------------------------------------------
    def set_timesteps(self, num_inference_steps: int, device=None):
        T = self.config.num_train_timesteps
        if num_inference_steps > T:
            raise ValueError("num_inference_steps cannot exceed num_train_timesteps")
        self.num_inference_steps = num_inference_steps
        ratio = T // num_inference_steps
        ts = (np.arange(0, num_inference_steps) * ratio).round()[::-1].copy().astype(np.int64)
        ts += self.config.steps_offset
        self.timesteps = torch.from_numpy(ts).to(device) if device is not None else torch.from_numpy(ts)

    def scale_model_input(self, sample, timestep=None):
        return sample

    def add_noise(self, original_samples: torch.Tensor, noise: torch.Tensor, timesteps) -> torch.Tensor:
        ac = self.alphas_cumprod.to(device=original_samples.device, dtype=original_samples.dtype)
        timesteps = torch.as_tensor(timesteps).to(original_samples.device)
        sa = (ac[timesteps] ** 0.5).flatten()
        sb = ((1 - ac[timesteps]) ** 0.5).flatten()
        while sa.ndim < original_samples.ndim:
            sa = sa.unsqueeze(-1)
            sb = sb.unsqueeze(-1)
        return sa * original_samples + sb * noise

    def __len__(self):
        return self.config.num_train_timesteps

    # -- persistence (diffusers directory layout: scheduler/scheduler_config.json) -------------------
    def save_pretrained(self, path: str):
        os.makedirs(path, exist_ok=True)
        with open(os.path.join(path, self.config_name), "w") as f:
            json.dump(dict(self.config), f, indent=2)

    @classmethod
    def from_pretrained(cls, path: str, **kw):
        with open(os.path.join(path, cls.config_name)) as f:
            cfg = json.load(f)
        cfg = {k: v for k, v in cfg.items() if not k.startswith("_")}
        cfg.update(kw)
        known = {"num_train_timesteps", "beta_start", "beta_end", "beta_schedule", "clip_sample", "clip_sample_range",
                 "prediction_type", "timestep_spacing", "steps_offset", "set_alpha_to_one", "variance_type"}
        return cls(**{k: v for k, v in cfg.items() if k in known})

    def _noise(self, like: torch.Tensor, generator):
        return randn_tensor(like.shape, generator, like.device, like.dtype)


class DDPMScheduler(_SchedulerBase):
    _class_name = "DDPMScheduler"

    def __init__(self, num_train_timesteps: int = 1000, variance_type: str = "fixed_small", **kw):
        if variance_type != "fixed_small":
            raise ValueError("only variance_type='fixed_small' (the reference default) is implemented")
        super().__init__(num_train_timesteps, variance_type=variance_type, **kw)

    def _scalars(self, t: int):
        n = self.num_inference_steps or self.config.num_train_timesteps
        prev_t = t - self.config.num_train_timesteps // n
        a_t = self.alphas_cumprod[t]
        a_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.one
        b_t = 1 - a_t
        b_prev = 1 - a_prev
        cur_a = a_t / a_prev
        cur_b = 1 - cur_a
        c_x0 = (a_prev ** 0.5 * cur_b) / b_t
        c_xt = cur_a ** 0.5 * b_prev / b_t
        var = torch.clamp((1 - a_prev) / (1 - a_t) * cur_b, min=1e-20)
        return a_t, b_t, c_x0, c_xt, var

    def step(self, model_output, timestep, sample, generator=None, return_dict: bool = True):
        t = int(timestep)
        a_t, b_t, c_x0, c_xt, var = self._scalars(t)
        x0 = (sample - b_t ** 0.5 * model_output) / a_t ** 0.5
        if self.config.clip_sample:
            x0 = x0.clamp(-self.config.clip_sample_range, self.config.clip_sample_range)
        prev = c_x0 * x0 + c_xt * sample
        if t > 0:
            prev = prev + (var ** 0.5) * self._noise(model_output, generator)
        return SchedulerOutput(prev, x0) if return_dict else (prev,)

    def needs_noise(self, timestep, eta: float = 0.0) -> bool:
        return int(timestep) > 0

    def step_coef(self, timestep, eta: float = 0.0) -> StepCoefC:
        t = int(timestep)
        a_t, b_t, c_x0, c_xt, var = self._scalars(t)
        c = StepCoefC()
        c.sqrt_1m_at = float(b_t ** 0.5)
        c.inv_sqrt_at = float(1.0 / a_t ** 0.5)
        c.clip = float(self.config.clip_sample_range)
        c.do_clip = 1 if self.config.clip_sample else 0
        c.c_x0, c.c_xt, c.c_eps = float(c_x0), float(c_xt), 0.0
        c.c_z = float(var ** 0.5) if t > 0 else 0.0
        return c


class DDIMScheduler(_SchedulerBase):
    _class_name = "DDIMScheduler"

    def __init__(self, num_train_timesteps: int = 1000, set_alpha_to_one: bool = True, **kw):
        super().__init__(num_train_timesteps, set_alpha_to_one=set_alpha_to_one, **kw)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]

    def _scalars(self, t: int, eta: float):
        prev_t = t - self.config.num_train_timesteps // self.num_inference_steps
        a_t = self.alphas_cumprod[t]
        a_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
        b_t = 1 - a_t
        var = ((1 - a_prev) / (1 - a_t)) * (1 - a_t / a_prev)
        std = eta * var ** 0.5
        return a_t, a_prev, b_t, std

    def step(self, model_output, timestep, sample, eta: float = 0.0, use_clipped_model_output: bool = False,
             generator=None, variance_noise=None, return_dict: bool = True):
        if use_clipped_model_output:
            raise ValueError("use_clipped_model_output=True is not used by the reference and is not implemented")
        t = int(timestep)
        a_t, a_prev, b_t, std = self._scalars(t, eta)
        x0 = (sample - b_t ** 0.5 * model_output) / a_t ** 0.5
        if self.config.clip_sample:
            x0 = x0.clamp(-self.config.clip_sample_range, self.config.clip_sample_range)
        direction = (1 - a_prev - std ** 2) ** 0.5 * model_output
        prev = a_prev ** 0.5 * x0 + direction
        if eta > 0:
            z = variance_noise if variance_noise is not None else self._noise(model_output, generator)
            prev = prev + std * z
        return SchedulerOutput(prev, x0) if return_dict else (prev,)

    def needs_noise(self, timestep, eta: float = 0.0) -> bool:
        return eta > 0

    def invert_step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor) -> torch.Tensor:
        """One step of deterministic DDIM inversion, x_{t-Δ} -> x_t (audiodiffusion/pipeline_audio_diffusion.py:229-240):
        remove the ε-direction at the lower noise level, rescale to x0, then re-noise to level t with the same ε."""
        t = int(timestep)
        prev_t = t - self.config.num_train_timesteps // self.num_inference_steps
        a_t = self.alphas_cumprod[t]
        a_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
        x0 = (sample - (1 - a_prev) ** 0.5 * model_output) * a_prev ** (-0.5)
        return x0 * a_t ** 0.5 + (1 - a_t) ** 0.5 * model_output

    def step_coef(self, timestep, eta: float = 0.0) -> StepCoefC:
        t = int(timestep)
        a_t, a_prev, b_t, std = self._scalars(t, eta)
        c = StepCoefC()
        c.sqrt_1m_at = float(b_t ** 0.5)
        c.inv_sqrt_at = float(1.0 / a_t ** 0.5)
        c.clip = float(self.config.clip_sample_range)
        c.do_clip = 1 if self.config.clip_sample else 0
        c.c_x0 = float(a_prev ** 0.5)
        c.c_xt = 0.0
        c.c_eps = float((1 - a_prev - std ** 2) ** 0.5)
        c.c_z = float(std) if eta > 0 else 0.0
        return c


class DPMSolverMultistepScheduler(_SchedulerBase):
    """DPM-Solver++ (Lu et al. 2022) as diffusers 0.24's `DPMSolverMultistepScheduler` runs it on an ε-prediction model
    with linear betas: 15-25 steps instead of DDPM's 1000.  Every statement about diffusers here is [3P-recall] 0.24.

    Each step converts ε to the data prediction x0 = (x - σ_t ε) / α_t and extrapolates along the probability-flow ODE
    (`dpmsolver++`) or the SDE (`sde-dpmsolver++`, one `randn_tensor` draw per step) from this step's x0 and, past the
    warm-up, the x0 of up to two earlier steps.  Every update is linear in x, x0, x0_{-1}, x0_{-2} and the noise, so
    `step_coef` hands the fused output kernel five scalars (`MultistepCoefC`) and the two earlier x0 live in history
    buffers on the device (`UNet2DModel.forward_step(..., history=)`).  `step()` and `step_coef()` advance the same
    multistep state (step index, warm-up count), so a run may use either per step but not both for one step."""
    _class_name = "DPMSolverMultistepScheduler"
    _SPACINGS = ("linspace", "leading", "trailing")

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 1e-4, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, solver_order: int = 2,
                 prediction_type: str = "epsilon", thresholding: bool = False, dynamic_thresholding_ratio: float = 0.995,
                 sample_max_value: float = 1.0, algorithm_type: str = "dpmsolver++", solver_type: str = "midpoint",
                 lower_order_final: bool = True, euler_at_final: bool = False, use_karras_sigmas: bool = False,
                 use_lu_lambdas: bool = False, lambda_min_clipped: float = -float("inf"), variance_type=None,
                 timestep_spacing: str = "linspace", steps_offset: int = 0):
        bad = []
        if beta_schedule != "linear" or trained_betas is not None:
            bad.append(f"beta_schedule={beta_schedule!r}" if beta_schedule != "linear" else "trained_betas")
        if prediction_type != "epsilon": bad.append(f"prediction_type={prediction_type!r}")
        if thresholding: bad.append("thresholding=True")
        if algorithm_type not in ("dpmsolver++", "sde-dpmsolver++"): bad.append(f"algorithm_type={algorithm_type!r}")
        elif solver_order not in ((1, 2, 3) if algorithm_type == "dpmsolver++" else (1, 2)):
            bad.append(f"solver_order={solver_order!r} with {algorithm_type}")
        if solver_type not in ("midpoint", "heun"): bad.append(f"solver_type={solver_type!r}")
        if use_karras_sigmas: bad.append("use_karras_sigmas=True")
        if use_lu_lambdas: bad.append("use_lu_lambdas=True")
        if lambda_min_clipped != -float("inf"): bad.append(f"lambda_min_clipped={lambda_min_clipped!r}")
        if variance_type is not None: bad.append(f"variance_type={variance_type!r}")
        if timestep_spacing not in self._SPACINGS: bad.append(f"timestep_spacing={timestep_spacing!r}")
        if bad:
            raise ValueError(f"DPMSolverMultistepScheduler(b200): unsupported configuration: {bad} (implemented: linear "
                             "betas, epsilon, dpmsolver++ order 1-3 / sde-dpmsolver++ order 1-2, midpoint / heun, "
                             f"timestep_spacing in {self._SPACINGS})")
        self.config = _Cfg(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                           beta_schedule=beta_schedule, trained_betas=None, solver_order=solver_order,
                           prediction_type=prediction_type, thresholding=False,
                           dynamic_thresholding_ratio=dynamic_thresholding_ratio, sample_max_value=sample_max_value,
                           algorithm_type=algorithm_type, solver_type=solver_type, lower_order_final=lower_order_final,
                           euler_at_final=euler_at_final, use_karras_sigmas=False, use_lu_lambdas=False,
                           lambda_min_clipped=lambda_min_clipped, variance_type=None, timestep_spacing=timestep_spacing,
                           steps_offset=steps_offset, _class_name=self._class_name)
        self.betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.sigmas = ((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5
        self.init_noise_sigma = 1.0
        self.num_inference_steps: Optional[int] = None
        self.timesteps = torch.from_numpy(np.linspace(0, num_train_timesteps - 1, num_train_timesteps,
                                                      dtype=np.float32)[::-1].copy())
        self.model_outputs = [None] * solver_order
        self.lower_order_nums = 0
        self._step_index: Optional[int] = None

    @property
    def step_index(self) -> Optional[int]:
        return self._step_index

    @classmethod
    def from_pretrained(cls, path: str, **kw):
        import inspect
        with open(os.path.join(path, cls.config_name)) as f:
            cfg = json.load(f)
        cfg.update(kw)
        known = set(inspect.signature(cls.__init__).parameters) - {"self"}
        return cls(**{k: v for k, v in cfg.items() if k in known})

    def set_timesteps(self, num_inference_steps: int, device=None):
        T = self.config.num_train_timesteps
        if not 1 <= num_inference_steps <= T:
            raise ValueError(f"num_inference_steps must be in [1, {T}], got {num_inference_steps}")
        last = T                                 # lambda_min_clipped = -inf clips nothing
        spacing = self.config.timestep_spacing
        if spacing == "linspace":
            ts = np.linspace(0, last - 1, num_inference_steps + 1).round()[::-1][:-1].copy().astype(np.int64)
        elif spacing == "leading":
            ratio = last // (num_inference_steps + 1)
            if ratio == 0:                       # every timestep would be 0 and the step index would run off the end
                raise ValueError(f"timestep_spacing='leading' needs num_inference_steps < {T}, got {num_inference_steps}")
            ts = (np.arange(0, num_inference_steps + 1) * ratio).round()[::-1][:-1].copy().astype(np.int64)
            ts += self.config.steps_offset
        else:
            ratio = T / num_inference_steps
            ts = np.arange(last, 0, -ratio).round().copy().astype(np.int64)
            ts -= 1
        sig = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()
        sig = np.interp(ts, np.arange(0, len(sig)), sig)
        sigma_last = ((1 - self.alphas_cumprod[0]) / self.alphas_cumprod[0]) ** 0.5
        self.sigmas = torch.from_numpy(np.concatenate([sig, [float(sigma_last)]]).astype(np.float32))
        self.timesteps = torch.from_numpy(ts).to(device=device, dtype=torch.int64)
        self.num_inference_steps = len(ts)
        self.model_outputs = [None] * self.config.solver_order
        self.lower_order_nums = 0
        self._step_index = None

    # -- multistep bookkeeping, shared by step() and step_coef() -----------------------------------------
    def _init_step_index(self, timestep) -> None:
        t = timestep.to(self.timesteps.device) if torch.is_tensor(timestep) else timestep
        cand = (self.timesteps == t).nonzero()
        if len(cand) == 0:
            self._step_index = len(self.timesteps) - 1
        else:
            self._step_index = cand[1 if len(cand) > 1 else 0].item()

    def _begin(self, timestep):
        """(step index, solver order of this step)."""
        if self.num_inference_steps is None:
            raise ValueError("call set_timesteps before step")
        if self._step_index is None:
            self._init_step_index(timestep)
        i, n, cfg = self._step_index, len(self.timesteps), self.config
        final = i == n - 1 and (cfg.euler_at_final or (cfg.lower_order_final and n < 15))
        second = i == n - 2 and cfg.lower_order_final and n < 15
        if cfg.solver_order == 1 or self.lower_order_nums < 1 or final:
            return i, 1
        if cfg.solver_order == 2 or self.lower_order_nums < 2 or second:
            return i, 2
        return i, 3

    def _end(self) -> None:
        if self.lower_order_nums < self.config.solver_order:
            self.lower_order_nums += 1
        self._step_index += 1

    @staticmethod
    def _alpha_sigma(sigma):
        alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
        return alpha_t, sigma * alpha_t

    def _lam(self, j: int):
        """(α, σ, λ) at sigmas[j], fp32 as the torch path computes them."""
        a, s = self._alpha_sigma(self.sigmas[j])
        return a, s, torch.log(a) - torch.log(s)

    # -- diffusers-compatible API ----------------------------------------------------------------
    def convert_model_output(self, model_output: torch.Tensor, sample: torch.Tensor) -> torch.Tensor:
        alpha_t, sigma_t = self._alpha_sigma(self.sigmas[self._step_index])
        return (sample - sigma_t * model_output) / alpha_t

    def step(self, model_output, timestep, sample, generator=None, return_dict: bool = True):
        i, order = self._begin(timestep)
        x0 = self.convert_model_output(model_output, sample)
        for k in range(self.config.solver_order - 1):
            self.model_outputs[k] = self.model_outputs[k + 1]
        self.model_outputs[-1] = x0
        sde = self.config.algorithm_type == "sde-dpmsolver++"
        noise = self._noise(model_output, generator) if sde else None
        alpha_t, sigma_t, lambda_t = self._lam(i + 1)
        _, sigma_s0, lambda_s0 = self._lam(i)
        h = lambda_t - lambda_s0
        heun = self.config.solver_type == "heun"
        m = self.model_outputs
        if order == 1:
            D0 = x0
        elif order == 2:
            _, _, lambda_s1 = self._lam(i - 1)
            r0 = (lambda_s0 - lambda_s1) / h
            D0, D1 = m[-1], (1.0 / r0) * (m[-1] - m[-2])
        else:
            _, _, lambda_s1 = self._lam(i - 1)
            _, _, lambda_s2 = self._lam(i - 2)
            r0, r1 = (lambda_s0 - lambda_s1) / h, (lambda_s1 - lambda_s2) / h
            D1_0, D1_1 = (1.0 / r0) * (m[-1] - m[-2]), (1.0 / r1) * (m[-2] - m[-3])
            D0 = m[-1]
            D1 = D1_0 + (r0 / (r0 + r1)) * (D1_0 - D1_1)
            D2 = (1.0 / (r0 + r1)) * (D1_0 - D1_1)
        if not sde:
            prev = (sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * D0
            if order == 2:
                if heun:
                    prev = prev + (alpha_t * ((torch.exp(-h) - 1.0) / h + 1.0)) * D1
                else:
                    prev = prev - 0.5 * (alpha_t * (torch.exp(-h) - 1.0)) * D1
            elif order == 3:
                prev = (prev + (alpha_t * ((torch.exp(-h) - 1.0) / h + 1.0)) * D1
                        - (alpha_t * ((torch.exp(-h) - 1.0 + h) / h ** 2 - 0.5)) * D2)
        else:
            prev = (sigma_t / sigma_s0 * torch.exp(-h)) * sample + (alpha_t * (1 - torch.exp(-2.0 * h))) * D0
            if order == 2:
                if heun:
                    prev = prev + (alpha_t * ((1.0 - torch.exp(-2.0 * h)) / (-2.0 * h) + 1.0)) * D1
                else:
                    prev = prev + 0.5 * (alpha_t * (1 - torch.exp(-2.0 * h))) * D1
            prev = prev + sigma_t * torch.sqrt(1.0 - torch.exp(-2.0 * h)) * noise
        self._end()
        return SchedulerOutput(prev, x0) if return_dict else (prev,)

    def needs_noise(self, timestep, eta: float = 0.0) -> bool:
        return self.config.algorithm_type == "sde-dpmsolver++"

    def fold(self, i: int, order: int):
        """The update of step i at `order` folded into x_out = c_xt x + c_x0 x0 + c_h1 x0_{-1} + c_h2 x0_{-2} + c_z z, and
        the conversion x0 = (x - sigma_s * eps) * inv_alpha_s: fp64 from the fp32 sigmas.  Returns a dict of floats."""
        def asl(j):
            s = float(self.sigmas[j])
            a = 1.0 / math.sqrt(s * s + 1.0)
            return a, s * a, math.log(a) - math.log(s * a)
        alpha_t, sigma_t, lam_t = asl(i + 1)
        alpha_s0, sigma_s0, lam_s0 = asl(i)
        h = lam_t - lam_s0
        c = dict(sqrt_1m_at=sigma_s0, inv_sqrt_at=1.0 / alpha_s0, c_h1=0.0, c_h2=0.0, c_z=0.0)
        if self.config.algorithm_type == "dpmsolver++":
            A = alpha_t * math.expm1(-h)                                 # x_t = c_xt x - A D0 + ...
            B = alpha_t * (math.expm1(-h) / h + 1.0) if order > 1 else 0.0
            c["c_xt"], c["c_x0"] = sigma_t / sigma_s0, -A
            if order == 2:
                r0 = (lam_s0 - asl(i - 1)[2]) / h
                k = B if self.config.solver_type == "heun" else -0.5 * A     # coefficient of D1 = (x0 - x0_{-1}) / r0
                c["c_x0"] += k / r0
                c["c_h1"] = -k / r0
            elif order == 3:
                lam_s1, lam_s2 = asl(i - 1)[2], asl(i - 2)[2]
                r0, r1 = (lam_s0 - lam_s1) / h, (lam_s1 - lam_s2) / h
                C_ = alpha_t * ((math.expm1(-h) + h) / h ** 2 - 0.5)
                a0, a1, q, kr = 1.0 / r0, 1.0 / r1, 1.0 / (r0 + r1), r0 / (r0 + r1)
                # D1 = D1_0 + kr (D1_0 - D1_1), D2 = q (D1_0 - D1_1); D1_0 = a0 (m0 - m1), D1_1 = a1 (m1 - m2)
                c["c_x0"] += B * a0 * (1 + kr) - C_ * q * a0
                c["c_h1"] = -B * (a0 + kr * (a0 + a1)) + C_ * q * (a0 + a1)
                c["c_h2"] = B * kr * a1 - C_ * q * a1
        else:
            E2 = -math.expm1(-2.0 * h)                                   # 1 - e^{-2h}
            A = alpha_t * E2
            c["c_xt"], c["c_x0"] = sigma_t / sigma_s0 * math.exp(-h), A
            c["c_z"] = sigma_t * math.sqrt(E2)
            if order == 2:
                r0 = (lam_s0 - asl(i - 1)[2]) / h
                k = alpha_t * (E2 / (-2.0 * h) + 1.0) if self.config.solver_type == "heun" else 0.5 * A
                c["c_x0"] += k / r0
                c["c_h1"] = -k / r0
        return c

    def step_coef(self, timestep, eta: float = 0.0) -> MultistepCoefC:
        """This step's scalars for the fused kernel (`UNet2DModel.forward_step`); advances the multistep state as `step()`
        does.  The kernel reads the two earlier x0 from the history buffers and writes this step's x0 there."""
        i, order = self._begin(timestep)
        f = self.fold(i, order)
        self._end()
        c = MultistepCoefC()
        s = c.step
        s.sqrt_1m_at, s.inv_sqrt_at, s.clip, s.do_clip = f["sqrt_1m_at"], f["inv_sqrt_at"], 1.0, 0
        s.c_x0, s.c_xt, s.c_eps, s.c_z = f["c_x0"], f["c_xt"], 0.0, f["c_z"]
        c.c_h1, c.c_h2 = f["c_h1"], f["c_h2"]
        return c

    @property
    def history_len(self) -> int:
        """History buffers the fused step needs: the x0 of the solver_order - 1 previous steps."""
        return self.config.solver_order - 1
