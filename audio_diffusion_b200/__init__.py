"""audio_diffusion_b200 — H100-native (sm_90a) engine for the teticio/audio-diffusion hot path.

Public surface mirrors the reference objects the unchanged `AudioDiffusionPipeline` drives:
`UNet2DModel`, `AutoencoderKL`, `DDPMScheduler`, `DDIMScheduler`, `DPMSolverMultistepScheduler`, `Mel`,
`AudioDiffusionPipeline`.
"""
__version__ = "0.1.0"

from . import _lib  # noqa: F401


def __getattr__(name):
    # lazy imports keep `import audio_diffusion_b200` cheap and side-effect free
    if name == "UNet2DModel":
        from .unet import UNet2DModel
        return UNet2DModel
    if name == "AutoencoderKL":
        from .vae import AutoencoderKL
        return AutoencoderKL
    if name in ("DDPMScheduler", "DDIMScheduler", "DPMSolverMultistepScheduler"):
        from . import schedulers
        return getattr(schedulers, name)
    if name == "Mel":
        from .mel import Mel
        return Mel
    if name in ("AudioDiffusionPipeline", "DiffusionPipeline"):
        from . import pipeline
        return getattr(pipeline, name)
    if name in ("FusedAdamW", "EMAModel", "mse_loss"):
        from . import training
        return getattr(training, name)
    raise AttributeError(name)
