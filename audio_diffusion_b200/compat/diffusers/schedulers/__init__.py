from audio_diffusion_b200.schedulers import DDIMScheduler, DDPMScheduler, DPMSolverMultistepScheduler  # noqa: F401
