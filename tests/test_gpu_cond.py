"""GPU parity of the conditional path (SURVEY §8 f3): `UNet2DConditionModel` as scripts/train_unet.py:139-159 builds it,
called with the (B, 1, 100) audio encodings (audiodiffusion/pipeline_audio_diffusion.py:160-161), against the fp32 oracle
(oracle/unet_cond_oracle.py).  Tolerances as for the unconditional U-Net: per layer max <= 6 % / rms <= 2.5 %, epsilon
max <= 6 % / rms <= 1.5 % (bf16 activations and GEMM operands, fp32 accumulation, fp32 softmax)."""
import numpy as np
import pytest
import torch

from cases import PUBLISHED_COND

pytestmark = pytest.mark.gpu


def _build(cuda, size, seed=0):
    from audio_diffusion_b200.unet_cond import UNet2DConditionModel
    from oracle.unet_cond_oracle import CondUNetConfig, init_weights
    ocfg = CondUNetConfig(sample_size=size)
    w = init_weights(ocfg, seed=seed)
    model = UNet2DConditionModel(sample_size=size, **PUBLISHED_COND)
    assert set(model.state_dict().keys()) == set(w.keys())
    model.load_state_dict(w)
    return model.to(cuda).eval(), ocfg, w


def _rel(got, ref):
    err = got - ref
    return (err.abs().max().item() / (ref.abs().max().item() + 1e-12),
            (err.pow(2).mean().sqrt() / (ref.pow(2).mean().sqrt() + 1e-12)).item())


@pytest.mark.parametrize("size", [(32, 32), (64, 64)])
def test_cond_unet_layers_and_eps(cuda, monkeypatch, size):
    from oracle.unet_cond_oracle import unet_cond_forward
    monkeypatch.setenv("B200AD_DEBUG_NOPOOL", "1")
    model, ocfg, w = _build(cuda, size)
    assert sum(p.numel() for p in model.parameters()) == 135_559_809
    g = torch.Generator().manual_seed(42)
    x = torch.randn(2, 1, *size, generator=g)
    enc = torch.randn(2, 1, 100, generator=g)
    t = torch.tensor([17, 801])
    taps = {}
    with torch.no_grad():
        ref = unet_cond_forward(w, ocfg, x, t, enc, taps)
        out = model(x.to(cuda), t.to(cuda), enc.to(cuda))["sample"]
    torch.cuda.synchronize()
    names = ["conv_in", "down_blocks.0.resnets.0", "down_blocks.0.attentions.0.attn2", "down_blocks.0.attentions.0",
             "down_blocks.0.attentions.1", "down_blocks.0.downsamplers.0.conv", "down_blocks.1.attentions.1",
             "down_blocks.2.attentions.0.attn2", "down_blocks.2.attentions.1", "down_blocks.3.resnets.1",
             "mid_block.attentions.0", "mid_block.resnets.1", "up_blocks.0.resnets.2", "up_blocks.0.upsamplers.0.conv",
             "up_blocks.1.attentions.0", "up_blocks.1.attentions.2", "up_blocks.2.attentions.2", "up_blocks.3.attentions.0",
             "up_blocks.3.attentions.2"]
    worst = (0.0, 0.0)
    for name in names:
        mx, rms = _rel(model.debug_tensor(name).cpu(), taps[name])
        print("%-44s max-rel %.4f rms-rel %.4f" % (name, mx, rms))
        worst = (max(worst[0], mx), max(worst[1], rms))
    mx, rms = _rel(out.cpu(), ref)
    print("eps max-rel %.4f rms-rel %.4f | worst layer %.4f / %.4f" % (mx, rms, worst[0], worst[1]))
    assert worst[0] <= 6e-2 and worst[1] <= 2.5e-2
    assert mx <= 6e-2 and rms <= 1.5e-2


def test_cond_encoding_matters_and_2d_encoding(cuda):
    """A (B, 100) encoding is accepted like (B, 1, 100); different encodings give different outputs; missing -> error."""
    model, ocfg, w = _build(cuda, (32, 32), seed=1)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 1, 32, 32, generator=g).to(cuda)
    e = torch.randn(2, 100, generator=g).to(cuda)
    with torch.no_grad():
        a = model(x, 500, e)["sample"]
        b = model(x, 500, e[:, None, :])["sample"]
        c = model(x, 500, torch.flip(e, (0,)))["sample"]
    assert torch.equal(a, b)
    assert (a - c).abs().max() > 1e-3 * a.abs().max()
    with pytest.raises(ValueError):
        model(x, 500)


def test_cond_pipeline_fused_matches_oracle_loop(cuda):
    """`pipe(..., encoding=enc)` (fused scheduler step) vs the oracle loop, DDPM, 6 steps, shared CPU noise streams."""
    from audio_diffusion_b200.mel import Mel
    from audio_diffusion_b200.pipeline import AudioDiffusionPipeline
    from audio_diffusion_b200.schedulers import DDPMScheduler
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_cond_oracle import unet_cond_forward
    model, ocfg, w = _build(cuda, (32, 32), seed=2)
    pipe = AudioDiffusionPipeline(vqvae=None, unet=model, mel=Mel(x_res=32, y_res=32, hop_length=512), scheduler=DDPMScheduler())
    pipe.set_progress_bar_config(disable=True)
    g = torch.Generator().manual_seed(9)
    noise = torch.randn(2, 1, 32, 32, generator=g)
    enc = torch.randn(2, 1, 100, generator=g)
    steps = 6
    imgs = pipe(batch_size=2, steps=steps, noise=noise.to(cuda), step_generator=torch.Generator().manual_seed(5),
                encoding=enc.to(cuda), return_audio=False)
    osch = OracleDDPM()
    osch.set_timesteps(steps)
    x, gen = noise.clone(), torch.Generator().manual_seed(5)
    with torch.no_grad():
        for t in osch.timesteps:
            x = osch.step(unet_cond_forward(w, ocfg, x, t, enc), t, x, generator=gen)["prev_sample"]
    ref = ((x / 2 + 0.5).clamp(0, 1).permute(0, 2, 3, 1).numpy() * 255).round().astype("uint8")[..., 0]
    got = np.stack([np.asarray(im) for im in imgs])
    d = np.abs(got.astype(int) - ref.astype(int))
    print(f"conditional pipeline: mean |d| {d.mean():.3f}, within 2: {(d <= 2).mean():.3f}, max {d.max()}")
    assert (d <= 2).mean() >= 0.90
