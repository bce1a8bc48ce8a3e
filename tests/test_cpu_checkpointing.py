"""Gradient checkpointing without a device: the training-memory size query (`b200ad_*_training_bytes`: training workspace
plus backward arena) gives the sizes it gave before checkpointing existed when it is off, and strictly less when it is on;
and the diffusers toggles round-trip on all three model classes."""
import pytest

PUBLISHED = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 128, 256, 256, 512, 512),
                 down_block_types=("DownBlock2D",) * 4 + ("AttnDownBlock2D", "DownBlock2D"),
                 up_block_types=("UpBlock2D", "AttnUpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D"))
COND = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256, 512, 512),
            down_block_types=("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",),
            up_block_types=("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3, cross_attention_dim=100)
LDM = dict(in_channels=1, out_channels=1, latent_channels=1, layers_per_block=2, block_out_channels=(128, 256, 512, 512),
           down_block_types=("DownEncoderBlock2D",) * 4, up_block_types=("UpDecoderBlock2D",) * 4)

# Training workspace + backward arena in bytes before gradient checkpointing was added (every activation kept).
PLAIN_BYTES = {
    "published": 17092031744,   # UNet2DModel 256x256, batch 16
    "cond": 93601632512,        # UNet2DConditionModel 256x256, batch 16, S = 1
    "ldm": 9459353856,          # AutoencoderKL 256x256, batch 8
}


def _model(which):
    if which == "published":
        from audio_diffusion_b200.unet import UNet2DModel
        return UNet2DModel(sample_size=(256, 256), **PUBLISHED)
    if which == "cond":
        from audio_diffusion_b200.unet_cond import UNet2DConditionModel
        return UNet2DConditionModel(sample_size=(256, 256), **COND)
    from audio_diffusion_b200.vae import AutoencoderKL
    return AutoencoderKL(**LDM)


def _training_bytes(m, which):
    from audio_diffusion_b200 import _lib
    L = _lib.lib()
    if which == "ldm":
        return L.b200ad_vae_training_bytes(m._h, 8, 256, 256)
    return L.b200ad_unet_training_bytes(m._h, 16, 256, 256, 1)


@pytest.mark.parametrize("which", ["published", "cond", "ldm"])
def test_training_bytes_off_unchanged_and_on_smaller(which):
    m = _model(which)
    off = _training_bytes(m, which)
    assert off == PLAIN_BYTES[which]
    m.enable_gradient_checkpointing()
    on = _training_bytes(m, which)
    print(f"{which}: {off / 2**30:.2f} GiB -> {on / 2**30:.2f} GiB with checkpointing (ratio {on / off:.3f})")
    assert 0 < on < off
    m.disable_gradient_checkpointing()
    assert _training_bytes(m, which) == off


def test_training_bytes_errors():
    from audio_diffusion_b200 import _lib
    L = _lib.lib()
    m = _model("published")
    assert L.b200ad_unet_training_bytes(m._h, 16, 250, 256, 1) == 0
    assert b"multiples of 32" in L.b200ad_last_error()
    assert L.b200ad_unet_training_bytes(m._h, 16, 256, 256, 2) == 0
    assert b"unconditional" in L.b200ad_last_error()
    c = _model("cond")
    assert L.b200ad_unet_training_bytes(c._h, 2, 64, 64, 77) > L.b200ad_unet_training_bytes(c._h, 2, 64, 64, 1) > 0
    assert L.b200ad_unet_training_bytes(c._h, 2, 64, 64, 257) == 0


@pytest.mark.parametrize("which", ["published", "cond", "ldm"])
def test_gradient_checkpointing_toggles(which):
    m = _model(which)
    assert type(m)._supports_gradient_checkpointing
    assert m.is_gradient_checkpointing is False
    m.enable_gradient_checkpointing()
    assert m.is_gradient_checkpointing is True
    m.enable_gradient_checkpointing()
    assert m.is_gradient_checkpointing is True
    m.disable_gradient_checkpointing()
    assert m.is_gradient_checkpointing is False
