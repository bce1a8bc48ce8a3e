"""GPU parity of the pipeline path (AudioDiffusionPipeline mirror + fused U-Net/scheduler step) vs the oracle.

Tolerance (stated): a few-step trajectory through the bf16 U-Net; final samples must agree with the fp32 oracle
to rms 3 % and the uint8 images on >= 90 % of pixels within 2 grey levels (error compounds over steps and is
bounded by the per-step clamp of x0)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SMALL = dict(
    in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256),
    down_block_types=("DownBlock2D", "AttnDownBlock2D"), up_block_types=("AttnUpBlock2D", "UpBlock2D"))


def _models(cuda, seed=0):
    from audio_diffusion_b200.unet import UNet2DModel
    from oracle.unet_oracle import UNetConfig, init_weights
    ocfg = UNetConfig(sample_size=(32, 32), **SMALL)
    w = init_weights(ocfg, seed=seed)
    m = UNet2DModel(sample_size=(32, 32), **SMALL)
    m.load_state_dict(w)
    return m.to(cuda), ocfg, w


def _oracle_loop(w, ocfg, sch, noise, steps, gen, eta=None):
    from oracle.unet_oracle import unet_forward
    sch.set_timesteps(steps)
    x = noise.clone()
    for t in sch.timesteps:
        eps = unet_forward(w, ocfg, x, t)
        x = (sch.step(eps, t, x, eta=eta, generator=gen) if eta is not None else sch.step(eps, t, x, generator=gen))["prev_sample"]
    return x


@pytest.mark.parametrize("kind", ["ddpm", "ddim", "ddim_eta"])
def test_fused_step_loop_matches_oracle(cuda, kind):
    from audio_diffusion_b200.mel import Mel
    from audio_diffusion_b200.pipeline import AudioDiffusionPipeline
    from audio_diffusion_b200.schedulers import DDIMScheduler, DDPMScheduler
    from oracle.schedulers_oracle import OracleDDIM, OracleDDPM
    model, ocfg, w = _models(cuda)
    steps = 8
    eta = {"ddpm": None, "ddim": 0.0, "ddim_eta": 0.7}[kind]
    sch = DDPMScheduler() if kind == "ddpm" else DDIMScheduler()
    osch = OracleDDPM() if kind == "ddpm" else OracleDDIM()
    pipe = AudioDiffusionPipeline(vqvae=None, unet=model, mel=Mel(x_res=32, y_res=32, hop_length=512), scheduler=sch)
    pipe.set_progress_bar_config(disable=True)
    # same RNG stream on both sides: CPU generators (device noise would differ between cpu and cuda Philox)
    noise = torch.randn(2, 1, 32, 32, generator=torch.Generator().manual_seed(42))
    # oracle draws per-step noise from a CPU generator; the pipeline draws on the device, so feed identical noise
    # through eta=0 / compare DDPM with the noise stream replayed on the CPU
    if kind == "ddim":
        # eta = 0 has no shared noise to damp the 1/sqrt(alpha_bar) amplification of the bf16 U-Net error, and a
        # random-weight U-Net is not a contractive denoiser, so a free-running trajectory is not a meaningful
        # parity target.  Teacher-force instead: every step starts from the oracle's x and must match its x_prev.
        from oracle.unet_oracle import unet_forward
        sch.set_timesteps(steps)
        osch.set_timesteps(steps)
        x = noise.clone()
        for t in osch.timesteps:
            nxt = osch.step(unet_forward(w, ocfg, x, t), t, x, eta=0.0)["prev_sample"]
            got = model.forward_step(x.to(cuda), t, sch.step_coef(t, 0.0)).cpu()
            rel = ((got - nxt).pow(2).mean().sqrt() / nxt.pow(2).mean().sqrt()).item()
            assert rel < 3e-2, f"ddim step t={int(t)}: rms-rel {rel:.4f}"
            x = nxt
        return
    else:
        # replay: generate the device noise stream first, then hand the same tensors to the oracle
        gdev = torch.Generator(device=cuda).manual_seed(7)
        zs = [torch.randn(noise.shape, generator=gdev, device=cuda).cpu() for _ in range(steps)]

        class Replay:
            def __init__(self): self.i = 0
        rp = Replay()
        import oracle.schedulers_oracle as so
        real_randn = torch.randn

        def fake_randn(shape, generator=None, device=None, dtype=None):
            z = zs[rp.i]; rp.i += 1
            return z
        so.torch.randn = fake_randn
        try:
            ref = _oracle_loop(w, ocfg, osch, noise, steps, None, eta=eta)
        finally:
            so.torch.randn = real_randn
        imgs = pipe(batch_size=2, steps=steps, noise=noise.to(cuda), eta=eta if eta is not None else 0,
                    step_generator=torch.Generator(device=cuda).manual_seed(7), return_audio=False)
    ref_u8 = ((ref / 2 + 0.5).clamp(0, 1).permute(0, 2, 3, 1).numpy() * 255).round().astype("uint8")[..., 0]
    got_u8 = np.stack([np.asarray(im) for im in imgs])
    d = np.abs(got_u8.astype(int) - ref_u8.astype(int))
    assert (d <= 2).mean() >= 0.90, f"{kind}: only {(d <= 2).mean():.3f} of pixels within 2 grey levels (max {d.max()})"


def test_unfused_reference_path_equals_fused(cuda):
    """unet(x,t)['sample'] + scheduler.step (the reference's two calls) == fused forward_step."""
    from audio_diffusion_b200.schedulers import DDPMScheduler
    model, ocfg, w = _models(cuda, seed=2)
    sch = DDPMScheduler()
    sch.set_timesteps(1000)
    x = torch.randn(2, 1, 32, 32, generator=torch.Generator().manual_seed(1)).to(cuda)
    z = torch.randn(2, 1, 32, 32, generator=torch.Generator().manual_seed(2)).to(cuda)
    t = sch.timesteps[100]
    with torch.no_grad():
        eps = model(x, t)["sample"]
        fused, eps2 = model.forward_step(x, t, sch.step_coef(t), noise=z, want_eps=True)

    class G:  # scheduler.step draws noise via torch.randn(generator=...): replay z
        pass
    import audio_diffusion_b200.schedulers as ps
    real = ps._SchedulerBase._noise
    ps._SchedulerBase._noise = lambda self, like, gen: z
    try:
        unfused = sch.step(model_output=eps, timestep=t, sample=x)["prev_sample"]
    finally:
        ps._SchedulerBase._noise = real
    assert torch.equal(eps, eps2) or (eps - eps2).abs().max() < 2e-3 * eps.abs().max()
    assert (fused - unfused).abs().max() < 3e-3 * unfused.abs().max() + 1e-5


def test_pipeline_call_end_to_end_with_audio(cuda):
    """Whole __call__: noise -> images (PIL) -> audio, shapes per pipeline_audio_diffusion.py:192-205."""
    from PIL import Image
    from audio_diffusion_b200.mel import Mel
    from audio_diffusion_b200.pipeline import AudioDiffusionPipeline
    from audio_diffusion_b200.schedulers import DDIMScheduler
    model, ocfg, w = _models(cuda, seed=3)
    pipe = AudioDiffusionPipeline(vqvae=None, unet=model, mel=Mel(x_res=32, y_res=32, hop_length=512, n_iter=4),
                                  scheduler=DDIMScheduler())
    pipe.set_progress_bar_config(disable=True)
    out = pipe(batch_size=3, steps=4, generator=torch.Generator(device=cuda).manual_seed(0))
    assert len(out.images) == 3 and isinstance(out.images[0], Image.Image) and out.images[0].size == (32, 32)
    assert out.audios.shape == (3, 1, (32 - 1) * 512)
    imgs, (sr, audios) = pipe(batch_size=1, steps=2, generator=torch.Generator(device=cuda).manual_seed(0), return_dict=False)
    assert sr == 22050 and len(audios) == 1 and audios[0].shape == ((32 - 1) * 512,)


def test_shard_invariance_single_gpu(cuda):
    """SURVEY §8c(6): a batch computed at once equals the concatenation of its shards (no cross-sample op)."""
    from audio_diffusion_b200.schedulers import DDIMScheduler
    model, ocfg, w = _models(cuda, seed=4)
    sch = DDIMScheduler()
    sch.set_timesteps(50)
    x = torch.randn(4, 1, 32, 32, generator=torch.Generator().manual_seed(9)).to(cuda)
    t = sch.timesteps[3]
    with torch.no_grad():
        full = model.forward_step(x, t, sch.step_coef(t)).clone()
        a = model.forward_step(x[:2].contiguous(), t, sch.step_coef(t)).clone()
        b = model.forward_step(x[2:].contiguous(), t, sch.step_coef(t)).clone()
    both = torch.cat([a, b])
    assert (full - both).abs().max() <= 2e-3 * full.abs().max()


def _latent_pipe(cuda, sch):
    """Latent audio diffusion (config C4 shape scaled down): 64x64 mel image <-> 8x8 latent, small U-Net on latents."""
    from audio_diffusion_b200.mel import Mel
    from audio_diffusion_b200.pipeline import AudioDiffusionPipeline
    from audio_diffusion_b200.unet import UNet2DModel
    from audio_diffusion_b200.vae import AutoencoderKL
    from oracle.unet_oracle import UNetConfig, init_weights
    from oracle.vae_oracle import VAEConfig
    from oracle.vae_oracle import init_weights as vae_init
    ocfg = UNetConfig(sample_size=(8, 8), **SMALL)
    w = init_weights(ocfg, seed=5)
    unet = UNet2DModel(sample_size=(8, 8), **SMALL)
    unet.load_state_dict(w)
    vcfg = VAEConfig()
    vw = vae_init(vcfg, seed=6)
    vae = AutoencoderKL(in_channels=1, out_channels=1, down_block_types=("DownEncoderBlock2D",) * 4,
                        up_block_types=("UpDecoderBlock2D",) * 4, block_out_channels=vcfg.block_out_channels,
                        layers_per_block=2, latent_channels=1)
    vae.load_state_dict(vw)
    pipe = AudioDiffusionPipeline(vqvae=vae.to(cuda), unet=unet.to(cuda), mel=Mel(x_res=64, y_res=64, hop_length=256),
                                  scheduler=sch)
    pipe.set_progress_bar_config(disable=True)
    return pipe, (ocfg, w), (vcfg, vw)


def test_latent_pipeline_decodes_through_vae(cuda):
    """pipeline_audio_diffusion.py:187-190 — with a `vqvae`, the denoised latents are rescaled by 1/0.18215 and decoded.
    The pipeline's images must equal decode(latents / 0.18215) of the same (seeded) latent loop, and the decoded
    image must match the oracle VAE applied to those latents (bf16 tolerance, >= 90 % of pixels within 2 levels)."""
    from audio_diffusion_b200.schedulers import DDIMScheduler
    from oracle.vae_oracle import decode
    sch = DDIMScheduler()
    pipe, _, (vcfg, vw) = _latent_pipe(cuda, sch)
    noise = torch.randn(2, 1, 8, 8, generator=torch.Generator().manual_seed(1)).to(cuda)
    out = pipe(batch_size=2, steps=4, noise=noise.clone(), return_audio=True)
    imgs = np.stack([np.asarray(im) for im in out.images])
    assert imgs.shape == (2, 64, 64) and imgs.dtype == np.uint8
    assert out.audios.shape[0] == 2 and out.audios.shape[2] == (64 - 1) * 256
    # replay the latent loop by hand
    sch.set_timesteps(4)
    x = noise.clone()
    for t in sch.timesteps:
        x = pipe.unet.forward_step(x, t, sch.step_coef(t, 0.0), out=x)
    lat = (1 / 0.18215 * x)
    dec = pipe.vqvae.decode(lat)["sample"]
    u8 = pipe.images_to_u8(dec)[:, 0].cpu().numpy()
    assert (np.abs(u8.astype(int) - imgs.astype(int)) <= 1).mean() > 0.999
    ref = decode(vw, vcfg, lat.cpu())
    ref_u8 = ((ref / 2 + 0.5).clamp(0, 1) * 255).round().to(torch.uint8)[:, 0].numpy()
    assert (np.abs(ref_u8.astype(int) - imgs.astype(int)) <= 2).mean() >= 0.9


def test_latent_pipeline_audio_conditioning(cuda):
    """pipeline_audio_diffusion.py:133-158 with a vqvae: the input slice is encoded to latents (sampled posterior, scaled by
    0.18215) before noising / masking; runs end to end and returns decoded images of the mel resolution."""
    from audio_diffusion_b200.schedulers import DDIMScheduler
    sch = DDIMScheduler()
    pipe, _, _ = _latent_pipe(cuda, sch)
    rng = np.random.default_rng(0)
    audio = (0.1 * rng.standard_normal(64 * 256 * 2)).astype(np.float32)
    g = torch.Generator(device=cuda).manual_seed(3)
    out = pipe(batch_size=1, raw_audio=audio, slice=0, start_step=2, steps=4, generator=g, mask_start_secs=0.1)
    assert np.asarray(out.images[0]).shape == (64, 64)
    assert np.isfinite(out.audios).all()


def test_golden_reference_driven_images(cuda):
    """tests/golden/pipeline_ddpm_small.npz: uint8 images returned by the REFERENCE's own pipeline file (driving the fp32
    oracle U-Net, tests/golden/make_golden.py). The product pipeline on the same noise, weights and CPU step generator reproduces
    them to the stated trajectory tolerance (>= 90 % of pixels within 2 grey levels)."""
    import os
    from audio_diffusion_b200.mel import Mel
    from audio_diffusion_b200.pipeline import AudioDiffusionPipeline
    from audio_diffusion_b200.schedulers import DDPMScheduler
    from audio_diffusion_b200.unet import UNet2DModel
    from oracle.unet_oracle import UNetConfig, init_weights
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pipeline_ddpm_small.npz"))
    w = init_weights(UNetConfig(sample_size=(32, 32), **SMALL), seed=int(z["weight_seed"]))
    m = UNet2DModel(sample_size=(32, 32), **SMALL)
    m.load_state_dict(w)
    pipe = AudioDiffusionPipeline(vqvae=None, unet=m.to(cuda), mel=Mel(x_res=32, y_res=32, hop_length=512, n_iter=2),
                                  scheduler=DDPMScheduler())
    pipe.set_progress_bar_config(disable=True)
    imgs = pipe(batch_size=2, steps=int(z["steps"]), noise=torch.from_numpy(z["noise"]).to(cuda),
                step_generator=torch.Generator().manual_seed(int(z["step_seed"])), return_audio=False)
    got = np.stack([np.asarray(im) for im in imgs]).astype(int)
    frac = (np.abs(got - z["images"].astype(int)) <= 2).mean()
    assert frac >= 0.9, frac


def test_graph_stepper_equals_eager(cuda):
    """CUDA-graph replay of the fused step (`UNet2DModel.graph_stepper`, b200ad_unet_forward_step_dev) is the same launch
    sequence as the eager `forward_step`: bit-identical samples over a few DDPM steps, batch 1 and 2; and the pipeline takes
    that path for small batches with the same images as with B200AD_CUDA_GRAPH=0."""
    import os
    from audio_diffusion_b200.mel import Mel
    from audio_diffusion_b200.pipeline import AudioDiffusionPipeline
    from audio_diffusion_b200.schedulers import DDPMScheduler
    from audio_diffusion_b200.unet import UNet2DModel
    arch = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256),
                down_block_types=("DownBlock2D", "AttnDownBlock2D"), up_block_types=("AttnUpBlock2D", "UpBlock2D"))
    model = UNet2DModel(sample_size=(32, 32), seed=4, **arch).to(cuda)
    sch = DDPMScheduler()
    sch.set_timesteps(1000)
    for n in (1, 2):
        g = torch.Generator().manual_seed(n)
        x0 = torch.randn(n, 1, 32, 32, generator=g).to(cuda)
        zs = [torch.randn(n, 1, 32, 32, generator=g).to(cuda) for _ in range(4)]
        xe = x0.clone()
        with torch.no_grad():
            for i in range(4):
                t = sch.timesteps[100 + i]
                xe = model.forward_step(xe, t, sch.step_coef(t), noise=zs[i], out=xe)
            st = model.graph_stepper(x0)
            for i in range(4):
                t = sch.timesteps[100 + i]
                st.step(t, sch.step_coef(t), zs[i])
            assert torch.equal(xe, st.x), (xe - st.x).abs().max().item()
            st2 = model.graph_stepper(x0)          # same shape, model still bound the same way: the cached graph, reset to x0
            assert st2 is st and torch.equal(st2.x, x0)
            for i in range(4):
                t = sch.timesteps[100 + i]
                st2.step(t, sch.step_coef(t), zs[i])
            assert torch.equal(xe, st2.x)
    pipe = AudioDiffusionPipeline(vqvae=None, unet=model, mel=Mel(x_res=32, y_res=32), scheduler=DDPMScheduler())
    pipe.set_progress_bar_config(disable=True)
    outs = []
    for flag in ("1", "0"):
        os.environ["B200AD_CUDA_GRAPH"] = flag
        try:
            gen = torch.Generator(device=cuda).manual_seed(7)
            imgs = pipe(batch_size=2, steps=6, generator=gen, return_audio=False)
        finally:
            os.environ.pop("B200AD_CUDA_GRAPH", None)
        outs.append([__import__("numpy").asarray(im) for im in imgs])
    for a, b in zip(*outs):
        assert (a == b).all()
