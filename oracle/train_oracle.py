"""CPU restatement of one training step of scripts/train_unet.py:227-267 (SURVEY §3.4, §8 row T-step).

TEST INFRASTRUCTURE (see oracle/__init__.py).  PARITY UNPINNED for the diffusers pieces (EMAModel, get_scheduler —
[3P-recall] diffusers==0.24.0); the optimizer is pinned against torch.optim.AdamW, which IS available here
(tests/test_cpu_oracle.py::test_train_oracle_adamw_matches_torch).

    noise  = randn; t = randint(0, T, (B,))                                  train_unet.py:238-247
    noisy  = noise_scheduler.add_noise(clean, noise, t)                      :250
    pred   = model(noisy, t)["sample"]; loss = F.mse_loss(pred, noise)       :257-258
    loss.backward(); clip_grad_norm_(params, 1.0)                            :259-262
    AdamW(lr, betas=(0.95, 0.999), weight_decay=1e-6, eps=1e-8).step()       :166-172, :263
    lr = cosine-with-warmup(step)                                            :174-179, :264
    EMAModel(inv_gamma=1, power=3/4, max_value=0.9999).step(model)           :185-190, :265-266
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, Optional

import torch

from .schedulers_oracle import OracleDDPM
from .unet_cond_oracle import CondUNetConfig, unet_cond_forward
from .unet_oracle import UNetConfig, unet_forward


def cosine_with_warmup(step: int, warmup: int, total: int) -> float:
    """LR multiplier of diffusers.optimization.get_cosine_schedule_with_warmup (num_cycles = 0.5)."""
    if step < warmup:
        return float(step) / float(max(1, warmup))
    p = float(step - warmup) / float(max(1, total - warmup))
    return max(0.0, 0.5 * (1.0 + math.cos(math.pi * 2.0 * 0.5 * p)))


def ema_decay(optimization_step: int, inv_gamma: float = 1.0, power: float = 0.75, max_value: float = 0.9999,
              min_value: float = 0.0, update_after_step: int = 0) -> float:
    """EMAModel.get_decay with the warm-up schedule (inv_gamma / power given => use_ema_warmup)."""
    step = max(0, optimization_step - update_after_step - 1)
    if step <= 0:
        return 0.0
    cur = 1.0 - (1.0 + step / inv_gamma) ** -power
    return max(min_value, min(cur, max_value))


@dataclass
class TrainState:
    step: int = 0                       # optimizer steps taken
    exp_avg: Dict[str, torch.Tensor] = field(default_factory=dict)
    exp_avg_sq: Dict[str, torch.Tensor] = field(default_factory=dict)
    ema: Dict[str, torch.Tensor] = field(default_factory=dict)


def clip_grad_norm(grads: Dict[str, torch.Tensor], max_norm: float = 1.0):
    """torch.nn.utils.clip_grad_norm_: total 2-norm over all tensors, coefficient max_norm / (norm + 1e-6) clamped to 1."""
    total = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).float()
    coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
    return {k: g * coef for k, g in grads.items()}, total


def adamw_update(p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, step: int, lr: float,
                 beta1: float = 0.95, beta2: float = 0.999, eps: float = 1e-8, weight_decay: float = 1e-6):
    """One torch.optim.AdamW update (decoupled decay, bias-corrected), in place; `step` is 1-based."""
    p.mul_(1.0 - lr * weight_decay)
    m.mul_(beta1).add_(g, alpha=1.0 - beta1)
    v.mul_(beta2).addcmul_(g, g, value=1.0 - beta2)
    bc1 = 1.0 - beta1 ** step
    bc2 = 1.0 - beta2 ** step
    denom = (v.sqrt() / math.sqrt(bc2)).add_(eps)
    p.addcdiv_(m, denom, value=-lr / bc1)


def loss_and_grads(w: Dict[str, torch.Tensor], cfg: UNetConfig, clean: torch.Tensor, noise: torch.Tensor,
                   t: torch.Tensor, sched: Optional[OracleDDPM] = None):
    """MSE(ε̂, ε) and its gradients w.r.t. every parameter, by autograd over the oracle forward (fp32)."""
    sched = sched or OracleDDPM()
    noisy = sched.add_noise(clean, noise, t)
    wl = {k: v.detach().clone().requires_grad_(True) for k, v in w.items()}
    pred = unet_forward(wl, cfg, noisy, t)
    loss = torch.mean((pred - noise) ** 2)
    grads = torch.autograd.grad(loss, list(wl.values()))
    return loss.detach(), dict(zip(wl.keys(), grads)), pred.detach()


def cond_loss_and_grads(w: Dict[str, torch.Tensor], cfg: CondUNetConfig, clean: torch.Tensor, noise: torch.Tensor,
                        t: torch.Tensor, enc: torch.Tensor):
    """MSE(ε̂, ε) of one conditional training step (scripts/train_unet.py:250-258) and its parameter gradients, by
    autograd over the conditional oracle forward."""
    noisy = OracleDDPM().add_noise(clean, noise, t)
    wl = {k: v.detach().clone().requires_grad_(True) for k, v in w.items()}
    pred = unet_cond_forward(wl, cfg, noisy, t, enc)
    loss = torch.mean((pred - noise) ** 2)
    grads = torch.autograd.grad(loss, list(wl.values()))
    return loss.detach(), dict(zip(wl.keys(), grads))


def train_step(w: Dict[str, torch.Tensor], cfg: UNetConfig, state: TrainState, clean: torch.Tensor, noise: torch.Tensor,
               t: torch.Tensor, base_lr: float = 1e-4, warmup: int = 500, total_steps: int = 10000,
               use_ema: bool = True):
    """One optimisation step, updating `w` and `state` in place. Returns (loss, grad_norm, lr used, ema decay)."""
    if use_ema and not state.ema:          # EMAModel clones the parameters when it is constructed (before any step)
        state.ema = {k: v.detach().clone() for k, v in w.items()}
    loss, grads, _ = loss_and_grads(w, cfg, clean, noise, t)
    grads, gnorm = clip_grad_norm(grads, 1.0)
    lr = base_lr * cosine_with_warmup(state.step, warmup, total_steps)   # LambdaLR: lr of step k uses lambda(k)
    state.step += 1
    for k in w:
        if k not in state.exp_avg:
            state.exp_avg[k] = torch.zeros_like(w[k])
            state.exp_avg_sq[k] = torch.zeros_like(w[k])
        adamw_update(w[k], grads[k], state.exp_avg[k], state.exp_avg_sq[k], state.step, lr)
    decay = 0.0
    if use_ema:
        decay = ema_decay(state.step)        # EMAModel.step increments its counter, then evaluates the decay
        for k in w:
            state.ema[k].sub_((1.0 - decay) * (state.ema[k] - w[k]))
    return loss, gnorm, lr, decay
