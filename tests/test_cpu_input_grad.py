"""Gradients with respect to the models' inputs, without a device.

* The library exports the data-gradient-only mode and the input-gradient backward calls.
* The training-memory query (`b200ad_*_training_bytes`) is unchanged with parameter gradients on (the default) and
  smaller with them off: that plan has no weight-gradient temporaries, bias-gradient sums or timestep-MLP scratch.
* The bf16 floor of dL/dx through the whole model, at the shapes and seeds of tests/test_gpu_input_grad.py: fp64
  autograd with bf16 storage (block_grads.bf16_storage: every conv / linear operand, output and gradient rounded where
  the engine stores it) against exact.  The GPU bars are stated from these floors.
"""
import pytest
import torch

from cases import PLAIN_BYTES, T3, TWO_LEVEL, TWO_LEVEL_COND, draw, model_256, oracle_config, training_bytes
from oracle import block_grads as bg


def test_symbols_exported():
    from audio_diffusion_b200 import _lib
    L = _lib.lib()
    for name in ("b200ad_unet_set_param_grads", "b200ad_vae_set_param_grads", "b200ad_unet_backward_input",
                 "b200ad_vae_encoder_backward_input"):
        assert hasattr(L, name), name


@pytest.mark.parametrize("which", ["published", "ldm"])
def test_training_bytes_data_only_smaller(which):
    from audio_diffusion_b200 import _lib
    m = model_256(which)
    set_pg = getattr(_lib.lib(), f"b200ad_{'vae' if which == 'ldm' else 'unet'}_set_param_grads")
    full = training_bytes(m, which)
    assert full == PLAIN_BYTES[which]
    assert set_pg(m._h, 0) == 0
    data = training_bytes(m, which)
    print(f"{which}: {full / 2**30:.2f} GiB -> {data / 2**30:.2f} GiB without parameter gradients")
    assert 0 < data < full
    assert set_pg(m._h, 1) == 0
    assert training_bytes(m, which) == full


def _floor(f, x, g_out):
    """errors() of dL/dx under bf16 storage against exact fp64 autograd of f (L = <f(x), g_out>)."""
    def grad(rounded):
        xl = x.clone().requires_grad_(True)
        with bg.bf16_storage() if rounded else torch.enable_grad():
            (g,) = torch.autograd.grad(f(xl), xl, g_out)
        return g
    e = bg.errors(grad(True), grad(False), act=True)
    print("floor (a, b, c):", tuple(round(v, 4) for v in e))
    return e


def test_unet_sample_grad_floor():
    """UNet2DModel TWO_LEVEL, 32x32, batch 3, T3: the MSE loss of tests/test_gpu_input_grad.py."""
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_oracle import init_weights, unet_forward
    cfg = oracle_config(TWO_LEVEL, (32, 32))
    w = {k: v.double() for k, v in init_weights(cfg, seed=2).items()}
    clean, noise, _ = draw(3, (32, 32), 2)
    t = torch.tensor(T3)
    noisy = OracleDDPM().add_noise(clean, noise, t).double()
    pred = unet_forward(w, cfg, noisy, t)
    g_eps = 2 * (pred - noise.double()) / pred.numel()
    a, b, c = _floor(lambda x: unet_forward(w, cfg, x, t), noisy, g_eps)
    assert max(a, b, c) < 0.05


@pytest.mark.parametrize("seq", [1, 8])
def test_cond_unet_sample_grad_floor(seq):
    """UNet2DConditionModel TWO_LEVEL_COND, 32x32, batch 3, T3, an encoding of `seq` tokens."""
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_cond_oracle import init_weights, unet_cond_forward
    cfg = oracle_config(TWO_LEVEL_COND, (32, 32))
    w = {k: v.double() for k, v in init_weights(cfg, seed=3).items()}
    clean, noise, enc = draw(3, (32, 32), 3, seq)
    enc = enc.double()
    t = torch.tensor(T3)
    noisy = OracleDDPM().add_noise(clean, noise, t).double()
    pred = unet_cond_forward(w, cfg, noisy, t, enc)
    g_eps = 2 * (pred - noise.double()) / pred.numel()
    a, b, c = _floor(lambda x: unet_cond_forward(w, cfg, x, t, enc), noisy, g_eps)
    assert max(a, b, c) < 0.05


def test_vae_image_grad_floor():
    """The ldm AutoencoderKL encoder at 64x64, batch 2, from seeded moment gradients."""
    from oracle import vae_oracle as vo
    cfg = vo.VAEConfig()
    w = {k: v.double() for k, v in vo.init_weights(cfg, seed=0).items()}
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 1, 64, 64, generator=g).clamp(-1, 1).double()
    gm = torch.randn(2, 2, 8, 8, generator=g).double()
    a, b, c = _floor(lambda xx: vo.encode_moments(w, cfg, xx), x, gm)
    assert max(a, b, c) < 0.05
