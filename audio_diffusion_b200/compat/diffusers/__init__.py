"""Minimal `diffusers` import surface for the unchanged teticio/audio-diffusion sources, backed by audio_diffusion_b200.

Only the names the reference imports exist (pipeline_audio_diffusion.py:24-33, mel.py:22-23, train_unet.py:17-20,
audio_encoder.py:3, audio_to_images.py:10)."""
import torch

from audio_diffusion_b200.hub_io import model_from_dir, save_model
from audio_diffusion_b200.mel import Mel
from audio_diffusion_b200.pipeline import (AudioPipelineOutput, BaseOutput, DiffusionPipeline, ImagePipelineOutput)
from audio_diffusion_b200.schedulers import DDIMScheduler, DDPMScheduler, DPMSolverMultistepScheduler
from audio_diffusion_b200.unet import UNet2DModel
from audio_diffusion_b200.unet_cond import UNet2DConditionModel
from audio_diffusion_b200.vae import AutoencoderKL

from .configuration_utils import ConfigMixin, register_to_config  # noqa: F401

__version__ = "0.24.0+b200shim"


class ModelMixin(torch.nn.Module):
    """`diffusers.ModelMixin` as audiodiffusion/audio_encoder.py:62 uses it: an nn.Module with the hub directory layout
    (`config.json` + `diffusion_pytorch_model.safetensors`).  The reference's AudioEncoder (a small separable-conv CNN that
    runs once per audio file, outside the denoising loop) executes on it unchanged, as plain PyTorch layers."""
    config_name = "config.json"

    @classmethod
    def from_pretrained(cls, path, subfolder=None, **_unused):
        import os
        sub = os.path.join(path, subfolder) if subfolder else path
        if not hasattr(cls, "config") and not os.path.exists(os.path.join(sub, "config.json")):
            model = cls()
            from audio_diffusion_b200.hub_io import load_weights
            model.load_state_dict(load_weights(sub))
            return model
        return model_from_dir(cls, sub)

    def save_pretrained(self, path, safe_serialization=True, **_unused):
        if not hasattr(self, "config"):
            self.config = {}
        save_model(self, path, safe_serialization=safe_serialization)

    @property
    def device(self):
        return next(self.parameters()).device
