"""Gradient checkpointing without a device: the training-memory size query (`b200ad_*_training_bytes`: training workspace
plus backward arena) gives the sizes it gave before checkpointing existed when it is off, and strictly less when it is on;
and the diffusers toggles round-trip on all three model classes."""
import pytest

from cases import PLAIN_BYTES, model_256, training_bytes


@pytest.mark.parametrize("which", ["published", "cond", "ldm"])
def test_training_bytes_off_unchanged_and_on_smaller(which):
    m = model_256(which)
    off = training_bytes(m, which)
    assert off == PLAIN_BYTES[which]
    m.enable_gradient_checkpointing()
    on = training_bytes(m, which)
    print(f"{which}: {off / 2**30:.2f} GiB -> {on / 2**30:.2f} GiB with checkpointing (ratio {on / off:.3f})")
    assert 0 < on < off
    m.disable_gradient_checkpointing()
    assert training_bytes(m, which) == off


def test_training_bytes_errors():
    from audio_diffusion_b200 import _lib
    L = _lib.lib()
    m = model_256("published")
    assert L.b200ad_unet_training_bytes(m._h, 16, 250, 256, 1) == 0
    assert b"multiples of 32" in L.b200ad_last_error()
    assert L.b200ad_unet_training_bytes(m._h, 16, 256, 256, 2) == 0
    assert b"unconditional" in L.b200ad_last_error()
    c = model_256("cond")
    assert L.b200ad_unet_training_bytes(c._h, 2, 64, 64, 77) > L.b200ad_unet_training_bytes(c._h, 2, 64, 64, 1) > 0
    assert L.b200ad_unet_training_bytes(c._h, 2, 64, 64, 257) == 0


@pytest.mark.parametrize("which", ["published", "cond", "ldm"])
def test_gradient_checkpointing_toggles(which):
    m = model_256(which)
    assert type(m)._supports_gradient_checkpointing
    assert m.is_gradient_checkpointing is False
    m.enable_gradient_checkpointing()
    assert m.is_gradient_checkpointing is True
    m.enable_gradient_checkpointing()
    assert m.is_gradient_checkpointing is True
    m.disable_gradient_checkpointing()
    assert m.is_gradient_checkpointing is False
