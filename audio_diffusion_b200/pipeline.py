"""`AudioDiffusionPipeline` — same call surface as audiodiffusion/pipeline_audio_diffusion.py:39-258
(`__call__`, `encode`, `slerp`, `get_default_steps`) plus the minimal `DiffusionPipeline` base the reference
relies on (`register_modules`, `device`, `progress_bar`, `to`, `save_pretrained`, `from_pretrained`).

The reference's own file runs unchanged on `audio_diffusion_b200/compat` (tests/test_cpu_dropin.py); this module is
the engine's pipeline, organised as four stages with the reference's observable behaviour:

  1. `_start_state`      initial noise, drawn with the caller's generator exactly as :120-130 does;
  2. `_condition`        optional audio conditioning / in-painting columns (:134-157);
  3. `_denoise`          the loop (:159-185) on `UNet2DModel.forward_step` — U-Net forward with the DDPM/DDIM/DPM-Solver++
                         update fused into the output kernel (the reference makes two calls, :163 and :165-179);
  4. `_deliver`          optional VAE decode (:187-190), float -> uint8 on the GPU, bit-exact with :192-194, PIL images,
                         and `Mel.images_to_audio` batched on the GPU instead of one image at a time on the CPU (:201).

RNG stays in PyTorch: initial noise and per-step noise are drawn from the caller's `torch.Generator` with the same
calls, shapes and order as the reference, so seeds reproduce the reference stream (:120-130, :171, :178).
"""
from __future__ import annotations

import json
import math
import os
from typing import List, Optional, Union

import numpy as np
import torch
from PIL import Image

from . import _lib
from .hub_io import DIFFUSERS_VERSION, save_model
from .mel import Mel
from .schedulers import DDIMScheduler, DDPMScheduler, DPMSolverMultistepScheduler, randn_tensor
from .unet import UNet2DModel
from .vae import AutoencoderKL

LATENT_SCALE = 0.18215            # training-time scaling of the VAE latents (:147, :189)
GRAPH_MAX_BATCH = 8               # batches up to this size run the denoising step as a CUDA-graph replay

# model_index.json entries: [library, class] as upstream diffusers resolves them, so directories written here load in the
# reference / in diffusers, and directories pushed by the reference's train_unet.py load here.
_UPSTREAM = {
    "UNet2DModel": "diffusers", "UNet2DConditionModel": "diffusers", "AutoencoderKL": "diffusers",
    "DDPMScheduler": "diffusers", "DDIMScheduler": "diffusers", "DPMSolverMultistepScheduler": "diffusers",
    "Mel": "audio_diffusion",
}


class BaseOutput(dict):
    def __init__(self, **kw):
        super().__init__(**kw)
        for k, v in kw.items():
            setattr(self, k, v)


class AudioPipelineOutput(BaseOutput):
    def __init__(self, audios):
        super().__init__(audios=audios)


class ImagePipelineOutput(BaseOutput):
    def __init__(self, images):
        super().__init__(images=images)


class DiffusionPipeline:
    config_name = "model_index.json"
    _optional_components: List[str] = []

    def __init__(self):
        self._modules_ = {}
        self._progress = None

    def register_modules(self, **kwargs):
        for k, v in kwargs.items():
            self._modules_[k] = v
            setattr(self, k, v)

    @property
    def device(self) -> torch.device:
        for m in self._modules_.values():
            if isinstance(m, torch.nn.Module):
                return next(m.parameters()).device
        return torch.device("cpu")

    def to(self, device):
        for k, m in self._modules_.items():
            if isinstance(m, torch.nn.Module):
                m.to(device)
        return self

    def set_progress_bar_config(self, **kw):
        self._progress_kw = kw

    def progress_bar(self, iterable):
        kw = getattr(self, "_progress_kw", {})
        if kw.get("disable"):
            return iterable
        try:
            from tqdm.auto import tqdm
            return tqdm(iterable, **kw)
        except Exception:
            return iterable

    # -- diffusers directory layout: model_index.json + one sub-directory per module -----------------------
    def save_pretrained(self, path: str, safe_serialization: bool = True, **_unused):
        os.makedirs(path, exist_ok=True)
        index = {"_class_name": type(self).__name__, "_diffusers_version": DIFFUSERS_VERSION}
        for k, m in self._modules_.items():
            if m is None:
                index[k] = [None, None]
                continue
            cname = type(m).__name__
            index[k] = [_UPSTREAM.get(cname, "diffusers"), cname]
            sub = os.path.join(path, k)
            if isinstance(m, torch.nn.Module) and hasattr(m, "config"):
                save_model(m, sub, safe_serialization=safe_serialization)
            else:
                m.save_pretrained(sub)
        with open(os.path.join(path, self.config_name), "w") as f:
            json.dump(index, f, indent=2)

    @classmethod
    def from_pretrained(cls, path: str, **kw):
        """`model_index.json` maps every component to [library, class].  The class is looked up the way diffusers does it —
        in the named library if that is importable (`diffusers` here is the engine's import surface, compat/diffusers) —
        and otherwise in the engine's own table; the component directory is loaded by the class's `from_pretrained`."""
        import importlib
        with open(os.path.join(path, cls.config_name)) as f:
            index = json.load(f)
        own = {"UNet2DModel": UNet2DModel, "AutoencoderKL": AutoencoderKL, "DDPMScheduler": DDPMScheduler,
               "DDIMScheduler": DDIMScheduler, "DPMSolverMultistepScheduler": DPMSolverMultistepScheduler, "Mel": Mel}
        mods = {}
        for k, v in index.items():
            if k.startswith("_") or not isinstance(v, list):
                continue
            sub = os.path.join(path, k)
            lib, cname = v[0], v[1]
            if cname is None or not os.path.isdir(sub):
                mods[k] = None
                continue
            klass = None
            try:
                klass = getattr(importlib.import_module(lib), cname, None) if lib else None
            except ImportError:
                klass = None
            if klass is None and cname == "UNet2DConditionModel":
                from .unet_cond import UNet2DConditionModel as klass
            klass = klass or own.get(cname)
            if klass is None or not hasattr(klass, "from_pretrained"):
                raise ValueError(f"from_pretrained: component {k} of class {cname} is not supported by the b200 engine")
            mods[k] = klass.from_pretrained(sub)
        mods.setdefault("vqvae", None)
        return cls(**mods)


def load_unet(sub: str) -> UNet2DModel:
    return UNet2DModel.from_pretrained(sub)


def load_vae(sub: str) -> AutoencoderKL:
    """`vqvae/` component of a latent pipeline (diffusers AutoencoderKL layout)."""
    return AutoencoderKL.from_pretrained(sub)


def image_to_unit_range(image) -> np.ndarray:
    """8-bit greyscale PIL image (or array) -> float64 array in [-1, 1]: byte / 255 * 2 - 1 (:137-140, :225-228)."""
    px = np.asarray(image, dtype=np.uint8)
    return (px / 255) * 2 - 1


class AudioDiffusionPipeline(DiffusionPipeline):
    _optional_components = ["vqvae"]

    def __init__(self, vqvae, unet, mel: Mel, scheduler: Union[DDIMScheduler, DDPMScheduler, DPMSolverMultistepScheduler]):
        super().__init__()
        self.register_modules(unet=unet, scheduler=scheduler, mel=mel, vqvae=vqvae)

    def get_default_steps(self) -> int:
        return 50 if isinstance(self.scheduler, DDIMScheduler) else 1000

    # ------------------------------------------------------------------------------------------------ stage 1
    def _start_state(self, batch_size: int, generator, noise) -> torch.Tensor:
        size = self.unet.sample_size
        if isinstance(size, int):                     # older checkpoints store an int (:118-119)
            size = self.unet.sample_size = (size, size)
        if noise is None:
            noise = torch.randn((batch_size, self.unet.in_channels, size[0], size[1]), generator=generator,
                                device=self.device)
        return noise.to(device=self.device, dtype=torch.float32).clone()

    # ------------------------------------------------------------------------------------------------ stage 2
    def _condition(self, images, audio_file, raw_audio, slice_index, start_step, generator, mask_start_secs, mask_end_secs):
        """Audio-conditioned start (:134-157).  Returns (frames, left, right): `frames[:, k]` is the conditioning image
        noised to the level of loop step k, `left` / `right` the number of columns kept from it at either edge."""
        self.mel.load_audio(audio_file, raw_audio)
        ref = torch.tensor(image_to_unit_range(self.mel.audio_slice_to_image(slice_index))[np.newaxis],
                           dtype=torch.float).to(self.device)                                  # (1, H, W)
        if self.vqvae is not None:                    # latent audio diffusion: condition in latent space (:143-147)
            ref = LATENT_SCALE * self.vqvae.encode(ref.unsqueeze(0)).latent_dist.sample(generator=generator)[0]
        steps_left = self.scheduler.timesteps[start_step:]
        if start_step > 0:                            # start from the conditioning image noised to the previous level
            images[0, 0] = self.scheduler.add_noise(ref, images, self.scheduler.timesteps[start_step - 1])
        cols_per_sec = self.unet.sample_size[1] * self.mel.get_sample_rate() / self.mel.x_res / self.mel.hop_length
        # In the reference `images` and `noise` are one tensor (:131), so the in-painting frames are built from the noise
        # AFTER the assignment above rewrote its [0, 0] plane; `images` holds exactly those values here.
        frames = self.scheduler.add_noise(ref, images, torch.as_tensor(steps_left))
        return frames, int(mask_start_secs * cols_per_sec), int(mask_end_secs * cols_per_sec)

    # ------------------------------------------------------------------------------------------------ stage 3
    def _denoise(self, images, start_step, eta, step_generator, encoding, inpaint):
        sch, unet = self.scheduler, self.unet
        fused = hasattr(unet, "forward_step") and hasattr(sch, "step_coef")
        extra = {"eta": eta} if isinstance(sch, DDIMScheduler) else {}
        cond = () if encoding is None else (encoding,)
        # A multistep scheduler's fused step keeps the x0 of its previous steps in history planes on the device, zeroed
        # here so that a coefficient of 0 (the warm-up steps) never meets a stale value.
        nhist = sch.history_len if fused and isinstance(sch, DPMSolverMultistepScheduler) else None
        hist = None
        # Small batches (the facade's batch_size=1, audiodiffusion/__init__.py:59) are bound by the host enqueueing ~120
        # launches per step: replay the step as one CUDA graph (same kernels, bit-identical results).
        stepper = None
        if (fused and encoding is None and inpaint is None and images.shape[0] <= GRAPH_MAX_BATCH
                and hasattr(unet, "graph_stepper") and not getattr(unet, "is_conditional", False)
                and os.environ.get("B200AD_CUDA_GRAPH", "1") != "0"):
            stepper = unet.graph_stepper(images, history=nhist)
            images = stepper.x                    # the stepper's own buffer, initialised from the start state
        elif nhist:
            hist = torch.zeros((nhist,) + tuple(images.shape), dtype=torch.float32, device=images.device)
        for k, t in enumerate(self.progress_bar(sch.timesteps[start_step:])):
            if fused:
                z = None
                if sch.needs_noise(t, eta):           # drawn as scheduler.step would draw it (:171, :178)
                    z = randn_tensor(images.shape, step_generator, images.device, images.dtype)
                if stepper is not None:
                    images = stepper.step(t, sch.step_coef(t, eta), z)
                    continue
                images = unet.forward_step(images, t, sch.step_coef(t, eta), *cond, noise=z, out=images, history=hist)
            else:                                     # any model / scheduler pair with the reference's duck type
                eps = unet(images, t, *cond)["sample"]
                images = sch.step(model_output=eps, timestep=t, sample=images, generator=step_generator,
                                  **extra)["prev_sample"]
            if inpaint is not None:
                frames, left, right = inpaint
                if left > 0:
                    images[..., :left] = frames[:, k, :, :left]
                if right > 0:
                    images[..., -right:] = frames[:, k, :, -right:]
        return images

    # ------------------------------------------------------------------------------------------------ stage 4
    def _deliver(self, images, return_dict: bool, return_audio: bool):
        if self.vqvae is not None:
            images = self.vqvae.decode(1 / LATENT_SCALE * images)["sample"]        # undo the training-time scaling (:187-190)
        u8 = self.images_to_u8(images)                # (B, C, H, W) uint8, still on the device
        host = u8.permute(0, 2, 3, 1).cpu().numpy()
        if host.shape[3] == 1:
            pil = [Image.fromarray(a[:, :, 0]) for a in host]
        else:                                         # RGB VAEs from the hub (:198)
            pil = [Image.fromarray(a, mode="RGB").convert("L") for a in host]
        if not return_audio:
            return pil
        if host.shape[3] == 1 and hasattr(self.mel, "images_to_audio"):
            audios = list(self.mel.images_to_audio(u8[:, 0]))          # batched Griffin-Lim (the engine's Mel)
        else:                                                          # any object with the reference Mel's surface (:201)
            audios = [self.mel.image_to_audio(im) for im in pil]
        if not return_dict:
            return pil, (self.mel.get_sample_rate(), audios)
        return BaseOutput(audios=np.array(audios)[:, np.newaxis, :], images=pil)

    @torch.no_grad()
    def __call__(
        self,
        batch_size: int = 1,
        audio_file: str = None,
        raw_audio: np.ndarray = None,
        slice: int = 0,
        start_step: int = 0,
        steps: int = None,
        generator: torch.Generator = None,
        mask_start_secs: float = 0,
        mask_end_secs: float = 0,
        step_generator: torch.Generator = None,
        eta: float = 0,
        noise: torch.Tensor = None,
        encoding: torch.Tensor = None,
        return_dict=True,
        return_audio: bool = True,
    ):
        """Same arguments and results as the reference's `__call__` (:62-205); `return_audio=False` (an addition) skips the
        Griffin-Lim tail and returns the PIL images only."""
        if encoding is not None and not getattr(self.unet, "is_conditional", False):
            raise ValueError("`encoding` needs a UNet2DConditionModel (scripts/train_unet.py:139-159)")
        self.scheduler.set_timesteps(steps or self.get_default_steps())
        images = self._start_state(batch_size, generator, noise)
        inpaint = None
        if audio_file is not None or raw_audio is not None:
            inpaint = self._condition(images, audio_file, raw_audio, slice, start_step, generator, mask_start_secs,
                                      mask_end_secs)
        images = self._denoise(images, start_step, eta, step_generator or generator, encoding, inpaint)
        return self._deliver(images, return_dict, return_audio)

    @staticmethod
    def images_to_u8(images: torch.Tensor) -> torch.Tensor:
        """`(images/2+0.5).clamp(0,1)*255 -> round -> uint8` (:192-194), bit-exact, on the device."""
        x = images.to(torch.float32).contiguous()
        out = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().b200ad_sample_to_u8(x.data_ptr(), out.data_ptr(), x.numel(), _lib.stream_ptr()))
        return out

    @torch.no_grad()
    def encode(self, images: List[Image.Image], steps: int = 50) -> torch.Tensor:
        """DDIM inversion (:207-242): walk the timesteps upwards and recover the noise that generates `images`."""
        if not isinstance(self.scheduler, DDIMScheduler):
            raise AssertionError("encode() is deterministic inversion and needs a DDIMScheduler")
        self.scheduler.set_timesteps(steps)
        batch = np.stack([image_to_unit_range(im)[np.newaxis] for im in images])
        sample = torch.Tensor(batch).to(self.device)
        for t in self.progress_bar(torch.flip(self.scheduler.timesteps, (0,))):
            eps = self.unet(sample, t)["sample"]
            sample = self.scheduler.invert_step(eps, t, sample)
        return sample

    @staticmethod
    def slerp(x0: torch.Tensor, x1: torch.Tensor, alpha: float) -> torch.Tensor:
        """Spherical interpolation between two noise tensors (:244-258): weights sin((1-a)θ)/sin θ and sin(aθ)/sin θ with
        θ the angle between the flattened tensors."""
        cos_theta = torch.dot(torch.flatten(x0), torch.flatten(x1)) / torch.norm(x0) / torch.norm(x1)
        theta = math.acos(cos_theta)
        return math.sin((1 - alpha) * theta) * x0 / math.sin(theta) + math.sin(alpha * theta) * x1 / math.sin(theta)
