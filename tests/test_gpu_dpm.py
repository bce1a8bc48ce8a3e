"""GPU tests of DPM-Solver++ on the fused U-Net output kernel: every step of a 20-step run against the scheduler's torch
`step()` on the same model output, whole pipeline loops against the generic branch (`unet(...)["sample"]` + `step()`), the
CUDA-graph stepper against the eager loop, and the DDPM / DDIM launches unchanged.

Bars: a fused step differs from `step()` only by how its update is rounded: five fp32 coefficients folded from fp64 (the
torch path forms D1 / D2 differences of x0 first) and x0 formed with 1 / alpha instead of a division.  The per-step bar is
therefore relative to the largest term of the linear combination, 1e-5 of it.  Whole loops run 20 steps through the bf16
U-Net, where those last-bit differences feed back into the next model input; their bar is 1 % of the sample's range."""
import os

import numpy as np
import pytest
import torch

from cases import PUBLISHED, TWO_LEVEL, TWO_LEVEL_COND

pytestmark = pytest.mark.gpu

STEP_CONFIGS = [dict(solver_order=o, solver_type=st, algorithm_type=alg)
                for alg, orders in (("dpmsolver++", (1, 2, 3)), ("sde-dpmsolver++", (1, 2)))
                for o in orders for st in ("midpoint", "heun") if not (o == 1 and st == "heun")]


def _unet(cuda, size, arch=TWO_LEVEL, seed=3):
    from audio_diffusion_b200.unet import UNet2DModel
    return UNet2DModel(sample_size=(size, size), seed=seed, **arch).to(cuda)


@pytest.mark.parametrize("size,batch", [(64, 4), (256, 2)])   # 256 x 256: the published layout (attention at 16 x 16)
@pytest.mark.parametrize("kw", STEP_CONFIGS, ids=lambda k: "-".join(str(v) for v in k.values()))
def test_each_fused_step_matches_step(cuda, size, batch, kw):
    from audio_diffusion_b200.schedulers import DPMSolverMultistepScheduler, randn_tensor
    model = _unet(cuda, size, PUBLISHED if size == 256 else TWO_LEVEL)
    a, b = DPMSolverMultistepScheduler(**kw), DPMSolverMultistepScheduler(**kw)
    a.set_timesteps(20)
    b.set_timesteps(20)
    x = torch.randn(batch, 1, size, size, generator=torch.Generator().manual_seed(1)).to(cuda)
    hist = torch.zeros((max(b.history_len, 1),) + tuple(x.shape), device=cuda)
    g1, g2 = torch.Generator(device=cuda).manual_seed(5), torch.Generator(device=cuda).manual_seed(5)
    worst = 0.0
    with torch.no_grad():
        for t in a.timesteps:
            z = randn_tensor(x.shape, g1, x.device) if b.needs_noise(t) else None
            h_prev = hist.clone()
            c = b.step_coef(t)
            fused, eps = model.forward_step(x, t, c, noise=z, want_eps=True, history=hist if b.history_len else None)
            ref = a.step(eps, t, x, generator=g2)["prev_sample"]
            s = c.step
            x0 = (x.double() - s.sqrt_1m_at * eps.double()) * s.inv_sqrt_at
            terms = [abs(s.c_xt) * x.double().abs(), abs(s.c_x0) * x0.abs(), abs(c.c_h1) * h_prev[0].double().abs()]
            if b.history_len == 2:
                terms.append(abs(c.c_h2) * h_prev[1].double().abs())
            if z is not None:
                terms.append(abs(s.c_z) * z.double().abs())
            scale = torch.stack(terms).amax().item()
            err = (fused.double() - ref.double()).abs().max().item()
            worst = max(worst, err / scale)
            assert err <= 1e-5 * scale, (int(t), err, scale)
            if b.history_len:
                torch.testing.assert_close(hist[0], a.model_outputs[-1], rtol=1e-5, atol=1e-5 * x0.abs().max().item())
            x = ref
    print(f"worst step error / largest term: {worst:.2e}")


class _Generic:
    """The model without `forward_step`: the pipeline takes the reference's generic branch (`unet(...)["sample"]` +
    `scheduler.step(..., generator=)`)."""

    def __init__(self, m):
        self.m = m
        self.sample_size, self.in_channels = m.sample_size, m.in_channels
        self.is_conditional = getattr(m, "is_conditional", False)

    def __call__(self, *a):
        return self.m(*a)


def _loop_pair(pipe, **call):
    """(fused, generic) final samples of the same seeded call (eager: no CUDA graph), before any VAE decode."""
    from audio_diffusion_b200.schedulers import DPMSolverMultistepScheduler
    pipe._deliver = lambda images, return_dict, return_audio: images.clone()
    pipe.scheduler = DPMSolverMultistepScheduler(solver_order=2)
    model = pipe.unet
    os.environ["B200AD_CUDA_GRAPH"] = "0"
    try:
        outs = []
        for unet in (model, _Generic(model)):
            pipe.unet = unet
            outs.append(pipe(generator=torch.Generator(device=pipe.device).manual_seed(11), steps=20, **call))
    finally:
        pipe.unet = model
        os.environ.pop("B200AD_CUDA_GRAPH", None)
    return outs


def _pipe(cuda, unet, vqvae=None, res=32):
    from audio_diffusion_b200.mel import Mel
    from audio_diffusion_b200.pipeline import AudioDiffusionPipeline
    from audio_diffusion_b200.schedulers import DPMSolverMultistepScheduler
    pipe = AudioDiffusionPipeline(vqvae=vqvae, unet=unet, mel=Mel(x_res=res, y_res=res, hop_length=256),
                                  scheduler=DPMSolverMultistepScheduler(solver_order=2))
    pipe.set_progress_bar_config(disable=True)
    return pipe


def _close(fused, generic, what):
    span = generic.abs().max().item()
    err = (fused - generic).abs().max().item()
    print(f"{what}: max |fused - generic| = {err:.3e} of {span:.3e}")
    assert torch.isfinite(fused).all() and err <= 1e-2 * span, (what, err, span)


@pytest.mark.parametrize("case", ["plain", "start_step", "inpaint", "latent4"])
def test_pipeline_loop_matches_generic_branch(cuda, case):
    from audio_diffusion_b200.unet import UNet2DModel
    if case == "latent4":
        unet = UNet2DModel(sample_size=(16, 16), seed=6, **dict(TWO_LEVEL, in_channels=4, out_channels=4)).to(cuda)
        pipe, call = _pipe(cuda, unet, res=16), dict(batch_size=3)
    else:
        pipe, call = _pipe(cuda, _unet(cuda, 32)), dict(batch_size=2)
    if case == "start_step":
        call["start_step"] = 7
    if case == "inpaint":       # audio-conditioned from step 5 with in-painted edges (pipeline_audio_diffusion.py:133-185)
        call = dict(batch_size=1, raw_audio=np.random.default_rng(2).standard_normal(32 * 256 * 2).astype(np.float32),
                    start_step=5, mask_start_secs=0.05, mask_end_secs=0.05)
    fused, generic = _loop_pair(pipe, **call)
    _close(fused, generic, case)


@pytest.mark.parametrize("seq", [1, 8])
def test_conditional_pipeline_loop_matches_generic_branch(cuda, seq):
    from audio_diffusion_b200.unet_cond import UNet2DConditionModel
    unet = UNet2DConditionModel(sample_size=(32, 32), seed=7, **TWO_LEVEL_COND).to(cuda)
    enc = torch.randn(2, seq, 100, generator=torch.Generator().manual_seed(seq)).to(cuda)
    fused, generic = _loop_pair(_pipe(cuda, unet), batch_size=2, encoding=enc)
    _close(fused, generic, f"conditional S={seq}")


@pytest.mark.parametrize("batch", [1, 8])
def test_graph_stepper_equals_eager(cuda, batch):
    """The pipeline's CUDA-graph path (history buffers captured with the graph) gives the eager fused loop's samples bit for
    bit, for orders 2 and 3; and two consecutive seeded calls agree, so the history is zeroed between calls."""
    from audio_diffusion_b200.schedulers import DPMSolverMultistepScheduler
    pipe = _pipe(cuda, _unet(cuda, 32))
    pipe._deliver = lambda images, return_dict, return_audio: images.clone()
    for order in (2, 3):
        pipe.scheduler = DPMSolverMultistepScheduler(solver_order=order)
        outs = []
        for flag in ("0", "1", "1"):
            os.environ["B200AD_CUDA_GRAPH"] = flag
            try:
                outs.append(pipe(batch_size=batch, steps=20, generator=torch.Generator(device=cuda).manual_seed(3)))
            finally:
                os.environ.pop("B200AD_CUDA_GRAPH", None)
        assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2]), order
        steppers = pipe.unet.__dict__["_steppers"]
        assert ((batch, 1, 32, 32), torch.device(cuda), order - 1) in steppers


def test_graph_stepper_refuses_other_coefficients(cuda):
    from audio_diffusion_b200.schedulers import DDIMScheduler, DPMSolverMultistepScheduler
    model = _unet(cuda, 32)
    x = torch.randn(1, 1, 32, 32, device=cuda)
    ddim, dpm = DDIMScheduler(), DPMSolverMultistepScheduler()
    ddim.set_timesteps(10)
    dpm.set_timesteps(10)
    t = dpm.timesteps[0]
    with pytest.raises(ValueError, match="MultistepCoefC"):
        model.graph_stepper(x, history=1).step(t, ddim.step_coef(ddim.timesteps[0]))
    with pytest.raises(ValueError, match="StepCoefC"):
        model.graph_stepper(x).step(t, dpm.step_coef(t))
    with pytest.raises(ValueError, match="history"):
        model.forward_step(x, t, ddim.step_coef(ddim.timesteps[0]), history=torch.zeros((1,) + x.shape, device=cuda))


def test_ddpm_ddim_launches_unchanged(cuda):
    """A DPM step launches exactly what a DDPM or DDIM step launches (the update is the output kernel's epilogue), and the
    multistep entry point with no history gives the DDIM step's result bit for bit."""
    from audio_diffusion_b200._lib import MultistepCoefC
    from audio_diffusion_b200.schedulers import DDIMScheduler, DDPMScheduler, DPMSolverMultistepScheduler
    model = _unet(cuda, 32)
    x = torch.randn(2, 1, 32, 32, generator=torch.Generator().manual_seed(0)).to(cuda)
    counts = {}
    with torch.no_grad():
        model(x, 500)
        counts["forward"] = model.last_launch_count
        for name, sch in (("ddpm", DDPMScheduler()), ("ddim", DDIMScheduler()), ("dpm", DPMSolverMultistepScheduler())):
            sch.set_timesteps(20)
            hist = torch.zeros((1,) + x.shape, device=cuda) if name == "dpm" else None
            for t in sch.timesteps[:3]:
                model.forward_step(x, t, sch.step_coef(t), noise=torch.zeros_like(x), history=hist)
            counts[name] = model.last_launch_count
        ddim = DDIMScheduler()
        ddim.set_timesteps(20)
        t = ddim.timesteps[3]
        c = ddim.step_coef(t)
        plain = model.forward_step(x, t, c)
        multi = model.forward_step(x, t, MultistepCoefC(c, 0.0, 0.0))
    print(counts)
    assert counts["ddpm"] == counts["ddim"] == counts["dpm"] == counts["forward"], counts
    assert torch.equal(plain, multi)
