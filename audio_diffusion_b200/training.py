"""Optimizer side of `scripts/train_unet.py`'s training step on the H100 engine (SURVEY §8 row T-step).

`FusedAdamW` has the `torch.optim.AdamW` constructor the reference uses (train_unet.py:166-172) and folds
`accelerator.clip_grad_norm_(model.parameters(), 1.0)` (:262), the AdamW update (:263) and `EMAModel.step` (:265-266)
into one pass over all parameters (`b200ad_optim_step`, two launches).  `EMAModel` keeps diffusers==0.24's surface
(`step`, `copy_to`, `decay`, `get_decay`).  `mse_loss` is `F.mse_loss` + dL/dpred in one kernel.

`train_step` is the loop body of train_unet.py:238-267 on the engine (forward and backward in libb200ad.so through
`UNet2DModel`'s autograd node); the unchanged reference script itself runs on `compat/accelerate`.

`vae_loss` / `vae_train_step` are the autoencoder's objective and loop body (scripts/train_vae.py with
config/ldm_autoencoder_kl.yaml): L1 reconstruction + kl_weight * KL, the generator loss of ldm's LPIPSWithDiscriminator
before its discriminator starts, without the LPIPS term.  Encoder and decoder backward run in libb200ad.so through
`AutoencoderKL`'s autograd nodes, so a perceptual term added in torch also reaches the decoder.
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, Optional

import torch

from . import _lib
from ._lib import OptimHParamsC


def ema_decay(optimization_step: int, inv_gamma: float = 1.0, power: float = 2 / 3, max_value: float = 0.9999,
              min_value: float = 0.0, update_after_step: int = 0) -> float:
    """EMAModel.get_decay with the warm-up schedule ([3P-recall] diffusers 0.24 training_utils.EMAModel)."""
    step = max(0, optimization_step - update_after_step - 1)
    if step <= 0:
        return 0.0
    cur = 1.0 - (1.0 + step / inv_gamma) ** -power
    return max(min_value, min(cur, max_value))


class EMAModel:
    """Shadow copy of the parameters. With a `FusedAdamW` attached (`optimizer.attach_ema(ema)`) the shadow update happens
    inside the optimizer kernel and `step()` only advances the schedule."""

    def __init__(self, parameters, decay: float = 0.9999, min_decay: float = 0.0, update_after_step: int = 0,
                 use_ema_warmup: bool = False, inv_gamma: float = 1.0, power: float = 2 / 3, **kwargs):
        if isinstance(parameters, torch.nn.Module):
            parameters = parameters.parameters()
        if kwargs.get("max_value") is not None:      # deprecated spellings the reference still uses (train_unet.py:185-190)
            decay = kwargs["max_value"]
            use_ema_warmup = True
        if kwargs.get("min_value") is not None:
            min_decay = kwargs["min_value"]
        if "inv_gamma" in kwargs or inv_gamma != 1.0 or power != 2 / 3:
            use_ema_warmup = True
        self.shadow_params = [p.detach().clone() for p in parameters]
        self.decay, self.min_decay = decay, min_decay
        self.update_after_step, self.use_ema_warmup = update_after_step, use_ema_warmup
        self.inv_gamma, self.power = inv_gamma, power
        self.optimization_step = 0
        self.cur_decay_value = 0.0
        self._fused = False

    def get_decay(self, optimization_step: int) -> float:
        step = max(0, optimization_step - self.update_after_step - 1)
        if step <= 0:
            return 0.0
        cur = 1 - (1 + step / self.inv_gamma) ** -self.power if self.use_ema_warmup else (1 + step) / (10 + step)
        return max(min(cur, self.decay), self.min_decay)

    def next_decay(self) -> float:
        """Decay the coming `step()` will use (what FusedAdamW passes to the kernel)."""
        return self.get_decay(self.optimization_step + 1)

    @torch.no_grad()
    def step(self, parameters) -> None:
        if isinstance(parameters, torch.nn.Module):
            parameters = parameters.parameters()
        self.optimization_step += 1
        decay = self.get_decay(self.optimization_step)
        self.cur_decay_value = decay
        if self._fused:
            return                                   # the optimizer kernel already moved the shadows with this decay
        for s, p in zip(self.shadow_params, parameters):
            if p.requires_grad:
                s.sub_((1 - decay) * (s - p.to(s.device)))
            else:
                s.copy_(p)

    @torch.no_grad()
    def copy_to(self, parameters: Iterable[torch.nn.Parameter]) -> None:
        for s, p in zip(self.shadow_params, parameters):
            p.copy_(s.to(p.device))     # in-place on the parameter itself: bumps its version (the U-Net re-packs its weights)

    def to(self, device=None, dtype=None):
        self.shadow_params = [s.to(device=device, dtype=dtype) if s.is_floating_point() else s.to(device=device)
                              for s in self.shadow_params]
        return self


class FusedAdamW(torch.optim.Optimizer):
    """`torch.optim.AdamW(params, lr, betas, weight_decay, eps)` on one fused kernel pass; `max_grad_norm` adds
    `clip_grad_norm_` semantics, `attach_ema` the EMA shadow update. One param group; fp32 contiguous CUDA parameters."""

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 1e-2,
                 max_grad_norm: Optional[float] = None):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        if len(self.param_groups) != 1:
            raise ValueError("FusedAdamW supports a single parameter group")
        self.max_grad_norm = max_grad_norm
        self._h = None
        self._bound_key = None
        self._ema: Optional[EMAModel] = None
        self.param_groups[0].setdefault("step", 0)     # lives in the param group so state_dict() / resume keeps it
        self.grad_norm: Optional[torch.Tensor] = None

    def attach_ema(self, ema: EMAModel) -> None:
        self._ema = ema
        ema._fused = True
        self._release()

    def _release(self):
        if self._h is not None:
            _lib.lib().b200ad_optim_destroy(self._h)
            self._h = None
        self._bound_key = None

    def load_state_dict(self, state_dict):
        """Resume: the moments are replaced by the loaded tensors, so the raw pointers held by the kernel handle are stale."""
        super().load_state_dict(state_dict)
        self.param_groups[0].setdefault("step", 0)
        self._release()

    def _pointer_key(self):
        """Every device pointer the kernel handle holds: parameters, both moments and (if attached) the EMA shadows."""
        g = self.param_groups[0]["params"]
        key = []
        for i, p in enumerate(g):
            if not p.requires_grad:
                continue
            st = self.state.get(p, {})
            key.append((p.data_ptr(), st["exp_avg"].data_ptr() if "exp_avg" in st else 0,
                        st["exp_avg_sq"].data_ptr() if "exp_avg_sq" in st else 0,
                        self._ema.shadow_params[i].data_ptr() if self._ema is not None else 0))
        return tuple(key)

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass

    def _bind(self):
        _lib.require_cuda()
        ps = [p for p in self.param_groups[0]["params"] if p.requires_grad]
        for p in ps:
            if p.device.type != "cuda" or p.dtype != torch.float32 or not p.is_contiguous():
                raise _lib.B200ADError("FusedAdamW: parameters must be contiguous fp32 CUDA tensors (no CPU fallback)")
            st = self.state[p]
            if "exp_avg" not in st:
                st["exp_avg"] = torch.zeros_like(p)
                st["exp_avg_sq"] = torch.zeros_like(p)
        self._ps = ps
        n = len(ps)
        arr = lambda ts: (C.c_void_p * n)(*[t.data_ptr() for t in ts])
        sizes = (C.c_int64 * n)(*[p.numel() for p in ps])
        ema = None
        if self._ema is not None:
            idx = [i for i, p in enumerate(self.param_groups[0]["params"]) if p.requires_grad]
            shadows = [self._ema.shadow_params[i] for i in idx]
            for s, p in zip(shadows, ps):
                if s.device != p.device or s.dtype != torch.float32 or not s.is_contiguous():
                    raise _lib.B200ADError("FusedAdamW: EMA shadows must be contiguous fp32 on the parameters' device")
            ema = arr(shadows)
        h = C.c_void_p()
        with torch.cuda.device(ps[0].device):
            _lib.check(_lib.lib().b200ad_optim_create(n, sizes, arr(ps), arr([self.state[p]["exp_avg"] for p in ps]),
                                                      arr([self.state[p]["exp_avg_sq"] for p in ps]), ema, C.byref(h)))
        self._h = h
        self._bound_key = self._pointer_key()

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        # module.to(), optimizer.load_state_dict() and EMAModel.to() all replace tensors: rebind when any pointer moved
        if self._h is not None and self._pointer_key() != self._bound_key:
            self._release()
        if self._h is None:
            self._bind()
        g = self.param_groups[0]
        ps = self._ps
        grads = []
        for p in ps:
            if p.grad is None:
                raise _lib.B200ADError("FusedAdamW.step: every parameter needs a gradient")
            gr = p.grad
            if gr.dtype != torch.float32 or not gr.is_contiguous():
                gr = gr.to(torch.float32).contiguous()
            grads.append(gr)
        g["step"] = int(g.get("step", 0)) + 1
        hp = OptimHParamsC(g["lr"], g["betas"][0], g["betas"][1], g["eps"], g["weight_decay"],
                           self.max_grad_norm if self.max_grad_norm else -1.0,
                           self._ema.next_decay() if self._ema is not None else -1.0, g["step"])
        if self.grad_norm is None:
            self.grad_norm = torch.zeros(1, dtype=torch.float32, device=ps[0].device)
        arr = (C.c_void_p * len(grads))(*[t.data_ptr() for t in grads])
        with torch.cuda.device(ps[0].device):
            _lib.check(_lib.lib().b200ad_optim_step(self._h, arr, C.byref(hp), self.grad_norm.data_ptr(), _lib.stream_ptr()))
        for p in ps:      # the kernel wrote through raw pointers: tell autograd (and the U-Net's weight-packing cache) so
            torch.autograd.graph.increment_version(p)
        return loss


def train_step(model, optimizer: "FusedAdamW", noise_scheduler, clean_images: torch.Tensor, ema: Optional[EMAModel] = None,
               lr_scheduler=None, generator: Optional[torch.Generator] = None, noise: Optional[torch.Tensor] = None,
               timesteps: Optional[torch.Tensor] = None, encoder_hidden_states: Optional[torch.Tensor] = None):
    """One iteration of the training loop body, scripts/train_unet.py:238-267, on the engine: noise + per-sample timesteps,
    `add_noise`, U-Net forward, MSE, backward (CUDA), clip + AdamW + EMA (one fused kernel pass), LR scheduler step.
    Returns the loss tensor (detached).  `noise` / `timesteps` may be given for reproducible tests.
    `encoder_hidden_states`: the batch's audio encodings for a `UNet2DConditionModel` (train_unet.py --encodings, :255)."""
    x = clean_images
    if noise is None:
        noise = torch.randn(x.shape, generator=generator, device=x.device if generator is None else generator.device).to(x.device)
    if timesteps is None:
        timesteps = torch.randint(0, noise_scheduler.config.num_train_timesteps, (x.shape[0],), generator=generator,
                                  device=x.device if generator is None else generator.device).long().to(x.device)
    noisy = noise_scheduler.add_noise(x, noise, timesteps)
    if encoder_hidden_states is None:
        pred = model(noisy, timesteps)["sample"]
    else:
        pred = model(noisy, timesteps, encoder_hidden_states)["sample"]
    loss = torch.nn.functional.mse_loss(pred, noise)
    loss.backward()
    optimizer.step()
    if lr_scheduler is not None:
        lr_scheduler.step()
    if ema is not None:
        ema.step(model.parameters())
    optimizer.zero_grad(set_to_none=True)
    return loss.detach()


def mse_loss(pred: torch.Tensor, target: torch.Tensor, want_grad: bool = True):
    """(`F.mse_loss(pred, target)`, dL/dpred) — train_unet.py:258 and the seed of the backward pass."""
    _lib.require_cuda()
    if pred.device.type != "cuda":
        raise _lib.B200ADError("mse_loss: CUDA tensors required (no CPU fallback)")
    p = pred.detach().to(torch.float32).contiguous()
    t = target.detach().to(device=p.device, dtype=torch.float32).contiguous()
    loss = torch.empty(1, dtype=torch.float32, device=p.device)
    grad = torch.empty_like(p) if want_grad else None
    scratch = torch.empty(1, dtype=torch.float64, device=p.device)
    with torch.cuda.device(p.device):
        _lib.check(_lib.lib().b200ad_mse_loss_grad(p.data_ptr(), t.data_ptr(), p.numel(), loss.data_ptr(),
                                                   grad.data_ptr() if grad is not None else None, scratch.data_ptr(),
                                                   _lib.stream_ptr()))
    return loss[0], grad


def vae_loss(x: torch.Tensor, x_hat: torch.Tensor, posterior, kl_weight: float = 1e-6):
    """(loss, rec, kl) of ldm's LPIPSWithDiscriminator before the discriminator starts, perceptual weight 0 and the
    learned logvar at its initial 0 ([3P-recall] ldm.modules.losses.contperceptual):
        nll  = sum(|x - x_hat| / exp(logvar) + logvar) / N,   kl = sum(posterior.kl()) / N,   loss = nll + kl_weight * kl.
    `rec` is mean |x - x_hat| (what ldm logs as rec_loss)."""
    rec = torch.abs(x.to(x_hat.dtype) - x_hat)
    n = x_hat.shape[0]
    nll = rec.sum() / n
    kl = posterior.kl().sum() / n
    return nll + kl_weight * kl, rec.mean(), kl


def vae_train_step(vae, optimizer, images: torch.Tensor, generator: Optional[torch.Generator] = None,
                   kl_weight: float = 1e-6):
    """One iteration of the autoencoder's training loop: encode, sample the posterior, decode, `vae_loss`, backward
    (CUDA), optimizer step, zero_grad.  ldm's optimizer is `FusedAdamW(vae.parameters(), lr=4.5e-6, betas=(0.5, 0.9),
    weight_decay=0.0)`.  Returns (loss, rec, kl), detached."""
    posterior = vae.encode(images).latent_dist
    z = posterior.sample(generator=generator)
    x_hat = vae.decode(z).sample
    loss, rec, kl = vae_loss(images, x_hat, posterior, kl_weight)
    loss.backward()
    optimizer.step()
    optimizer.zero_grad(set_to_none=True)
    return loss.detach(), rec.detach(), kl.detach()
