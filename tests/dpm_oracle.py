"""Restatement of diffusers==0.24.0 DPMSolverMultistepScheduler in plain fp32 torch, for the configurations the engine
implements: linear betas, epsilon prediction, algorithm_type dpmsolver++ / sde-dpmsolver++, solver_type midpoint / heun,
no thresholding, no Karras sigmas.

TEST INFRASTRUCTURE, kept apart from the product's scheduler (audio_diffusion_b200/schedulers.py) as oracle/ keeps DDPM
and DDIM.  PARITY UNPINNED: diffusers cannot be imported here; every line is [3P-recall] of the 0.24 source
(set_timesteps, _sigma_to_alpha_sigma_t, convert_model_output, dpm_solver_first_order_update,
multistep_dpm_solver_second_order_update, multistep_dpm_solver_third_order_update, _init_step_index, step).
"""
from __future__ import annotations

import numpy as np
import torch


class OracleDPM:
    def __init__(self, num_train_timesteps=1000, beta_start=1e-4, beta_end=0.02, solver_order=2,
                 algorithm_type="dpmsolver++", solver_type="midpoint", lower_order_final=True, euler_at_final=False,
                 timestep_spacing="linspace", steps_offset=0):
        self.T = num_train_timesteps
        self.solver_order, self.algorithm_type, self.solver_type = solver_order, algorithm_type, solver_type
        self.lower_order_final, self.euler_at_final = lower_order_final, euler_at_final
        self.timestep_spacing, self.steps_offset = timestep_spacing, steps_offset
        self.betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.alpha_t = torch.sqrt(self.alphas_cumprod)
        self.sigma_t = torch.sqrt(1 - self.alphas_cumprod)
        self.lambda_t = torch.log(self.alpha_t) - torch.log(self.sigma_t)
        self.sigmas = ((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5
        self.num_inference_steps = None
        self.model_outputs = [None] * solver_order
        self.lower_order_nums = 0
        self._step_index = None

    def set_timesteps(self, num_inference_steps):
        clipped_idx = torch.searchsorted(torch.flip(self.lambda_t, [0]), -float("inf"))     # lambda_min_clipped = -inf
        last_timestep = ((self.T - clipped_idx).numpy()).item()
        if self.timestep_spacing == "linspace":
            timesteps = np.linspace(0, last_timestep - 1, num_inference_steps + 1).round()[::-1][:-1].copy().astype(np.int64)
        elif self.timestep_spacing == "leading":
            step_ratio = last_timestep // (num_inference_steps + 1)
            timesteps = (np.arange(0, num_inference_steps + 1) * step_ratio).round()[::-1][:-1].copy().astype(np.int64)
            timesteps += self.steps_offset
        elif self.timestep_spacing == "trailing":
            step_ratio = self.T / num_inference_steps
            timesteps = np.arange(last_timestep, 0, -step_ratio).round().copy().astype(np.int64)
            timesteps -= 1
        else:
            raise ValueError(self.timestep_spacing)
        sigmas = np.array(((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5)
        sigmas = np.interp(timesteps, np.arange(0, len(sigmas)), sigmas)
        sigma_last = ((1 - self.alphas_cumprod[0]) / self.alphas_cumprod[0]) ** 0.5
        sigmas = np.concatenate([sigmas, [sigma_last]]).astype(np.float32)
        self.sigmas = torch.from_numpy(sigmas)
        self.timesteps = torch.from_numpy(timesteps).to(dtype=torch.int64)
        self.num_inference_steps = len(timesteps)
        self.model_outputs = [None] * self.solver_order
        self.lower_order_nums = 0
        self._step_index = None

    def _sigma_to_alpha_sigma_t(self, sigma):
        alpha_t = 1 / ((sigma**2 + 1) ** 0.5)
        sigma_t = sigma * alpha_t
        return alpha_t, sigma_t

    def convert_model_output(self, model_output, sample):
        sigma = self.sigmas[self._step_index]
        alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(sigma)
        return (sample - sigma_t * model_output) / alpha_t

    def dpm_solver_first_order_update(self, model_output, sample, noise=None):
        sigma_t, sigma_s = self.sigmas[self._step_index + 1], self.sigmas[self._step_index]
        alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(sigma_t)
        alpha_s, sigma_s = self._sigma_to_alpha_sigma_t(sigma_s)
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s = torch.log(alpha_s) - torch.log(sigma_s)
        h = lambda_t - lambda_s
        if self.algorithm_type == "dpmsolver++":
            x_t = (sigma_t / sigma_s) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * model_output
        else:
            x_t = ((sigma_t / sigma_s * torch.exp(-h)) * sample
                   + (alpha_t * (1 - torch.exp(-2.0 * h))) * model_output
                   + sigma_t * torch.sqrt(1.0 - torch.exp(-2 * h)) * noise)
        return x_t

    def multistep_dpm_solver_second_order_update(self, model_output_list, sample, noise=None):
        sigma_t, sigma_s0, sigma_s1 = (self.sigmas[self._step_index + 1], self.sigmas[self._step_index],
                                       self.sigmas[self._step_index - 1])
        alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(sigma_t)
        alpha_s0, sigma_s0 = self._sigma_to_alpha_sigma_t(sigma_s0)
        alpha_s1, sigma_s1 = self._sigma_to_alpha_sigma_t(sigma_s1)
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
        lambda_s1 = torch.log(alpha_s1) - torch.log(sigma_s1)
        m0, m1 = model_output_list[-1], model_output_list[-2]
        h, h_0 = lambda_t - lambda_s0, lambda_s0 - lambda_s1
        r0 = h_0 / h
        D0, D1 = m0, (1.0 / r0) * (m0 - m1)
        if self.algorithm_type == "dpmsolver++":
            if self.solver_type == "midpoint":
                x_t = ((sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * D0
                       - 0.5 * (alpha_t * (torch.exp(-h) - 1.0)) * D1)
            else:
                x_t = ((sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * D0
                       + (alpha_t * ((torch.exp(-h) - 1.0) / h + 1.0)) * D1)
        else:
            if self.solver_type == "midpoint":
                x_t = ((sigma_t / sigma_s0 * torch.exp(-h)) * sample + (alpha_t * (1 - torch.exp(-2.0 * h))) * D0
                       + 0.5 * (alpha_t * (1 - torch.exp(-2.0 * h))) * D1
                       + sigma_t * torch.sqrt(1.0 - torch.exp(-2.0 * h)) * noise)
            else:
                x_t = ((sigma_t / sigma_s0 * torch.exp(-h)) * sample + (alpha_t * (1 - torch.exp(-2.0 * h))) * D0
                       + (alpha_t * ((1.0 - torch.exp(-2.0 * h)) / (-2.0 * h) + 1.0)) * D1
                       + sigma_t * torch.sqrt(1.0 - torch.exp(-2.0 * h)) * noise)
        return x_t

    def multistep_dpm_solver_third_order_update(self, model_output_list, sample):
        sigma_t, sigma_s0, sigma_s1, sigma_s2 = (self.sigmas[self._step_index + 1], self.sigmas[self._step_index],
                                                 self.sigmas[self._step_index - 1], self.sigmas[self._step_index - 2])
        alpha_t, sigma_t = self._sigma_to_alpha_sigma_t(sigma_t)
        alpha_s0, sigma_s0 = self._sigma_to_alpha_sigma_t(sigma_s0)
        alpha_s1, sigma_s1 = self._sigma_to_alpha_sigma_t(sigma_s1)
        alpha_s2, sigma_s2 = self._sigma_to_alpha_sigma_t(sigma_s2)
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
        lambda_s1 = torch.log(alpha_s1) - torch.log(sigma_s1)
        lambda_s2 = torch.log(alpha_s2) - torch.log(sigma_s2)
        m0, m1, m2 = model_output_list[-1], model_output_list[-2], model_output_list[-3]
        h, h_0, h_1 = lambda_t - lambda_s0, lambda_s0 - lambda_s1, lambda_s1 - lambda_s2
        r0, r1 = h_0 / h, h_1 / h
        D0 = m0
        D1_0, D1_1 = (1.0 / r0) * (m0 - m1), (1.0 / r1) * (m1 - m2)
        D1 = D1_0 + (r0 / (r0 + r1)) * (D1_0 - D1_1)
        D2 = (1.0 / (r0 + r1)) * (D1_0 - D1_1)
        return ((sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * D0
                + (alpha_t * ((torch.exp(-h) - 1.0) / h + 1.0)) * D1
                - (alpha_t * ((torch.exp(-h) - 1.0 + h) / h**2 - 0.5)) * D2)

    def _init_step_index(self, timestep):
        index_candidates = (self.timesteps == timestep).nonzero()
        if len(index_candidates) == 0:
            step_index = len(self.timesteps) - 1
        elif len(index_candidates) > 1:
            step_index = index_candidates[1].item()
        else:
            step_index = index_candidates[0].item()
        self._step_index = step_index

    def step(self, model_output, timestep, sample, generator=None):
        if self._step_index is None:
            self._init_step_index(timestep)
        lower_order_final = (self._step_index == len(self.timesteps) - 1) and (
            self.euler_at_final or (self.lower_order_final and len(self.timesteps) < 15))
        lower_order_second = ((self._step_index == len(self.timesteps) - 2) and self.lower_order_final
                              and len(self.timesteps) < 15)
        model_output = self.convert_model_output(model_output, sample=sample)
        for i in range(self.solver_order - 1):
            self.model_outputs[i] = self.model_outputs[i + 1]
        self.model_outputs[-1] = model_output
        if self.algorithm_type == "sde-dpmsolver++":
            noise = torch.randn(model_output.shape, generator=generator, device=model_output.device,
                                dtype=model_output.dtype)
        else:
            noise = None
        if self.solver_order == 1 or self.lower_order_nums < 1 or lower_order_final:
            prev_sample = self.dpm_solver_first_order_update(model_output, sample=sample, noise=noise)
        elif self.solver_order == 2 or self.lower_order_nums < 2 or lower_order_second:
            prev_sample = self.multistep_dpm_solver_second_order_update(self.model_outputs, sample=sample, noise=noise)
        else:
            prev_sample = self.multistep_dpm_solver_third_order_update(self.model_outputs, sample=sample)
        if self.lower_order_nums < self.solver_order:
            self.lower_order_nums += 1
        self._step_index += 1
        return {"prev_sample": prev_sample}
