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

from oracle import block_grads as bg

from test_cpu_checkpointing import PLAIN_BYTES, _model, _training_bytes

TRAIN_CFG = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256),
                 down_block_types=("DownBlock2D", "AttnDownBlock2D"), up_block_types=("AttnUpBlock2D", "UpBlock2D"))
COND_CFG = dict(block_out_channels=(128, 256), down_block_types=("CrossAttnDownBlock2D", "DownBlock2D"),
                up_block_types=("UpBlock2D", "CrossAttnUpBlock2D"))
T3 = torch.tensor([37, 412, 903])


def test_symbols_exported():
    from audio_diffusion_b200 import _lib
    L = _lib.lib()
    for name in ("b200ad_unet_set_param_grads", "b200ad_vae_set_param_grads", "b200ad_unet_backward_input",
                 "b200ad_vae_encoder_backward_input"):
        assert hasattr(L, name), name


@pytest.mark.parametrize("which", ["published", "ldm"])
def test_training_bytes_data_only_smaller(which):
    from audio_diffusion_b200 import _lib
    m = _model(which)
    set_pg = getattr(_lib.lib(), f"b200ad_{'vae' if which == 'ldm' else 'unet'}_set_param_grads")
    full = _training_bytes(m, which)
    assert full == PLAIN_BYTES[which]
    assert set_pg(m._h, 0) == 0
    data = _training_bytes(m, which)
    print(f"{which}: {full / 2**30:.2f} GiB -> {data / 2**30:.2f} GiB without parameter gradients")
    assert 0 < data < full
    assert set_pg(m._h, 1) == 0
    assert _training_bytes(m, which) == full


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
    """UNet2DModel TRAIN_CFG, 32x32, batch 3, T3: the MSE loss of tests/test_gpu_input_grad.py."""
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_oracle import UNetConfig, init_weights, unet_forward
    cfg = UNetConfig(sample_size=(32, 32), **TRAIN_CFG)
    w = {k: v.double() for k, v in init_weights(cfg, seed=2).items()}
    g = torch.Generator().manual_seed(3)
    clean = torch.rand(3, 1, 32, 32, generator=g) * 2 - 1
    noise = torch.randn(3, 1, 32, 32, generator=g)
    noisy = OracleDDPM().add_noise(clean, noise, T3).double()
    pred = unet_forward(w, cfg, noisy, T3)
    g_eps = 2 * (pred - noise.double()) / pred.numel()
    a, b, c = _floor(lambda x: unet_forward(w, cfg, x, T3), noisy, g_eps)
    assert max(a, b, c) < 0.05


@pytest.mark.parametrize("seq", [1, 8])
def test_cond_unet_sample_grad_floor(seq):
    """UNet2DConditionModel COND_CFG, 32x32, batch 3, T3, an encoding of `seq` tokens."""
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_cond_oracle import CondUNetConfig, init_weights, unet_cond_forward
    cfg = CondUNetConfig(sample_size=(32, 32), **COND_CFG)
    w = {k: v.double() for k, v in init_weights(cfg, seed=3).items()}
    g = torch.Generator().manual_seed(4)
    clean = torch.rand(3, 1, 32, 32, generator=g) * 2 - 1
    noise = torch.randn(3, 1, 32, 32, generator=g)
    enc = torch.randn(3, seq, 100, generator=g).double()
    noisy = OracleDDPM().add_noise(clean, noise, T3).double()
    pred = unet_cond_forward(w, cfg, noisy, T3, enc)
    g_eps = 2 * (pred - noise.double()) / pred.numel()
    a, b, c = _floor(lambda x: unet_cond_forward(w, cfg, x, T3, enc), noisy, g_eps)
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
