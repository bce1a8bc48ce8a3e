"""Gradients with respect to the models' inputs on the GPU: the U-Nets' sample, the autoencoder's image and latents.

1. Head: the engine's input gradient against fp64 conv_transpose2d of its own gradient of conv_in's output (debug_grad)
   with the conv_in weights: only the fp32 accumulation differs, so the bars are 1e-4.
2. End to end: sample.grad / the image gradient from loss.backward() against fp64 autograd through the oracle model, with
   bars of at most 3x the bf16 floor tests/test_cpu_input_grad.py measures at these shapes and seeds (floor in the
   comments as (a, b, c), block_grads.errors' three measures).
3. The data-gradient-only backward of a frozen eval() model against the full backward: the same input gradient within a
   few times the run-to-run spread of the full backward (its GroupNorm / LayerNorm reductions accumulate with float
   atomics), no p.grad, no flat gradient buffer, no all-reduce, fewer launches.
4. Asking for the input gradient changes nothing else: the parameter gradients within the spread, one launch more.
5. Checkpointing: the input gradient with it equals the one without, within the spread.
6. A frozen decoder's latent gradient equals the training decoder's.
7. Guards: one forward per backward, no double backward, no encoding gradient, no backward past max_batch.
"""
import pytest
import torch
import torch.nn.functional as F

from cases import LDM, T3, TWO_LEVEL, TWO_LEVEL_COND, build, draw, w64
from oracle import block_grads as bg

pytestmark = pytest.mark.gpu

HEAD_BAR = 1e-4
K_SPREAD = 4.0
# end to end, (a, b, c)
UNET_BAR = (0.042, 0.0552, 0.042)        # floor (0.014, 0.0184, 0.014)
COND_BARS = {1: (0.045, 0.0522, 0.045),  # floor (0.015, 0.0174, 0.015)
             8: (0.048, 0.0486, 0.048)}  # floor (0.016, 0.0162, 0.016)
VAE_BAR = (0.0708, 0.0558, 0.0708)       # floor (0.0236, 0.0186, 0.0236)


def _unet_case(cuda, seq=None, size=(32, 32)):
    """(model in train(), fp64 weights on the device, oracle forward f(x), noisy sample, timesteps, encoding, noise) with
    the seeds of tests/test_cpu_input_grad.py."""
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_cond_oracle import unet_cond_forward
    from oracle.unet_oracle import unet_forward
    arch, seed = (TWO_LEVEL, 2) if seq is None else (TWO_LEVEL_COND, 3)
    model, cfg, w = build(arch, seed, cuda, size)
    clean, noise, enc = draw(3, size, seed, seq)
    t = torch.tensor(T3)
    noisy = OracleDDPM().add_noise(clean, noise, t).to(cuda)
    wd, tc = w64(w, cuda), t.to(cuda)
    if seq is None:
        f = lambda x: unet_forward(wd, cfg, x, tc)
    else:
        enc = enc.to(cuda)
        f = lambda x: unet_cond_forward(wd, cfg, x, tc, enc.double())
    return model, wd, f, noisy, tc, enc, noise.to(cuda)


def _call(model, x, t, enc):
    return model(x, t)["sample"] if enc is None else model(x, t, enc)["sample"]


def _sample_grad(model, x, t, enc, noise):
    """(dL/dx, the loss's output gradient) of the MSE loss, from zeroed parameter gradients."""
    for p in model.parameters():
        p.grad = None
    xl = x.clone().requires_grad_(True)
    pred = _call(model, xl, t, enc)
    F.mse_loss(pred, noise).backward()
    torch.cuda.synchronize()
    return xl.grad, 2 * (pred.detach() - noise) / pred.numel()


def _vae(cuda, max_batch=2):
    model, cfg, w = build(LDM, 0, cuda, max_batch=max_batch)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 1, 64, 64, generator=g).clamp(-1, 1).to(cuda)
    gm = torch.randn(2, 2, 8, 8, generator=g).to(cuda)
    return model, w64(w, cuda), cfg, x, gm


def _image_grad(vae, x, gm):
    for p in vae.parameters():
        p.grad = None
    xl = x.clone().requires_grad_(True)
    vae.encode(xl).latent_dist.parameters.backward(gm)
    torch.cuda.synchronize()
    return xl.grad


def _check(got, ref, bar, what):
    e = bg.errors(got, ref, act=True)
    print(f"{what}: (a, b, c) = ({e[0]:.2e}, {e[1]:.2e}, {e[2]:.2e})  bars {bar}")
    assert all(v <= b for v, b in zip(e, bar)), (what, e, bar)


def _check_spread(got, ref, ref2, what):
    spread = (ref2 - ref).norm().item()
    err = (got - ref).norm().item()
    print(f"{what}: |g| {ref.norm().item():.4e}  spread {spread:.3e}  err {err:.3e}")
    assert err <= K_SPREAD * spread + 1e-6 * ref.norm().item(), (what, err, spread)


def _freeze(model):
    model.eval()
    model.requires_grad_(False)
    return model


# ---------------------------------------------------------------------------------------------------------- 1 + 2
@pytest.mark.parametrize("seq", [None, 1, 8])
def test_unet_sample_grad(cuda, seq):
    """UNet2DModel (seq None) and UNet2DConditionModel (seq tokens), 32x32, batch 3, T3: the head against
    conv_transpose2d of the engine's own G(conv_in), and the whole sample gradient against fp64 autograd."""
    model, w64, f, noisy, t, enc, noise = _unet_case(cuda, seq)
    gx, g_eps = _sample_grad(model, noisy, t, enc, noise)
    head = F.conv_transpose2d(model.debug_grad("conv_in").double(), w64["conv_in.weight"], padding=1)
    _check(gx, head, (HEAD_BAR,) * 3, f"head (seq {seq})")
    xl = noisy.double().requires_grad_(True)
    (ref,) = torch.autograd.grad(f(xl), xl, g_eps.double())
    _check(gx, ref, UNET_BAR if seq is None else COND_BARS[seq], f"end to end (seq {seq})")


def test_vae_image_grad(cuda):
    """The ldm AutoencoderKL encoder at 64x64, batch 2: the head against conv_transpose2d of G(encoder.conv_in), and the
    image gradient against fp64 autograd of the oracle encoder."""
    from oracle import vae_oracle as vo
    vae, w64, cfg, x, gm = _vae(cuda)
    gx = _image_grad(vae, x, gm)
    head = F.conv_transpose2d(vae.debug_grad("encoder.conv_in").double(), w64["encoder.conv_in.weight"], padding=1)
    _check(gx, head, (HEAD_BAR,) * 3, "encoder head")
    xl = x.double().requires_grad_(True)
    (ref,) = torch.autograd.grad(vo.encode_moments(w64, cfg, xl), xl, gm.double())
    _check(gx, ref, VAE_BAR, "encoder end to end")


# ---------------------------------------------------------------------------------------------------------- 3 + 4 + 5
@pytest.mark.parametrize("seq", [None, 8])
def test_unet_data_only_and_full(cuda, monkeypatch, seq):
    """Frozen eval() model (data-only backward) against the full backward of the same weights; the full backward with and
    without the sample gradient; checkpointing on against off."""
    model, _, _, noisy, t, enc, noise = _unet_case(cuda, seq)
    # full mode: no sample gradient, twice (the spread), then with it
    flats, launches = [], []
    for _ in range(2):
        for p in model.parameters():
            p.grad = None
        F.mse_loss(_call(model, noisy, t, enc), noise).backward()
        torch.cuda.synchronize()
        flats.append(model._grad_flat.clone())
        launches.append(model.last_backward_launch_count)
    g_full, _ = _sample_grad(model, noisy, t, enc, noise)
    flat_x = model._grad_flat.clone()
    launches_x = model.last_backward_launch_count
    g_full2, _ = _sample_grad(model, noisy, t, enc, noise)
    assert launches[0] == launches[1] and launches_x == launches[0] + 1, (launches, launches_x)
    _check_spread(flat_x, flats[0], flats[1], "parameter gradients with / without the sample gradient")
    # checkpointing
    model.enable_gradient_checkpointing()
    g_ckpt, _ = _sample_grad(model, noisy, t, enc, noise)
    model.disable_gradient_checkpointing()
    _check_spread(g_ckpt, g_full, g_full2, "sample gradient, checkpointed")
    # data only, on a fresh model with the same weights
    fresh, _, _, _, _, _, _ = _unet_case(cuda, seq)
    _freeze(fresh)
    calls = []
    monkeypatch.setattr(fresh, "_allreduce_gradients", lambda: calls.append(1))
    g_data, _ = _sample_grad(fresh, noisy, t, enc, noise)
    _check_spread(g_data, g_full, g_full2, "sample gradient, data only")
    assert fresh._grad_flat is None and not calls
    assert all(p.grad is None for p in fresh.parameters())
    print("launches: full", launches[0], "full + g_x", launches_x, "data only", fresh.last_backward_launch_count)
    assert fresh.last_backward_launch_count < launches[0]
    # the same model back in training: parameter gradients as before
    fresh.requires_grad_(True)
    fresh.train()
    for p in fresh.parameters():
        p.grad = None
    F.mse_loss(_call(fresh, noisy, t, enc), noise).backward()
    torch.cuda.synchronize()
    _check_spread(fresh._grad_flat, flats[0], flats[1], "parameter gradients after the data-only phase")


def test_vae_data_only_and_full(cuda, monkeypatch):
    """The encoder's image gradient data-only against full, full with and without it, checkpointed; the frozen decoder's
    latent gradient against the training decoder's."""
    vae, _, _, x, gm = _vae(cuda)
    flats, launches = [], []
    for _ in range(2):
        for p in vae.parameters():
            p.grad = None
        vae.encode(x).latent_dist.parameters.backward(gm)
        torch.cuda.synchronize()
        flats.append(vae._grad_flat.clone())
        launches.append(vae.last_backward_launch_count)
    g_full = _image_grad(vae, x, gm)
    flat_x = vae._grad_flat.clone()
    assert vae.last_backward_launch_count == launches[0] + 1, (launches, vae.last_backward_launch_count)
    g_full2 = _image_grad(vae, x, gm)
    _check_spread(flat_x, flats[0], flats[1], "encoder parameter gradients with / without the image gradient")
    vae.enable_gradient_checkpointing()
    g_ckpt = _image_grad(vae, x, gm)
    vae.disable_gradient_checkpointing()
    _check_spread(g_ckpt, g_full, g_full2, "image gradient, checkpointed")
    # decoder, training mode: the latent gradient (twice, the spread)
    g = torch.Generator().manual_seed(5)
    z = torch.randn(2, 1, 8, 8, generator=g).to(cuda)
    gimg = torch.randn(2, 1, 64, 64, generator=g).to(cuda)
    gz = []
    for _ in range(2):
        for p in vae.parameters():
            p.grad = None
        zl = z.clone().requires_grad_(True)
        vae.decode(zl).sample.backward(gimg)
        torch.cuda.synchronize()
        gz.append(zl.grad)
    dec_full = vae.last_backward_launch_count
    # data only on a fresh model
    fresh, _, _, _, _ = _vae(cuda)
    _freeze(fresh)
    g_data = _image_grad(fresh, x, gm)
    _check_spread(g_data, g_full, g_full2, "image gradient, data only")
    zl = z.clone().requires_grad_(True)
    fresh.decode(zl).sample.backward(gimg)
    torch.cuda.synchronize()
    _check_spread(zl.grad, gz[0], gz[1], "latent gradient, frozen decoder")
    assert fresh._grad_flat is None and all(p.grad is None for p in fresh.parameters())
    print("decoder launches: full", dec_full, "data only", fresh.last_backward_launch_count)


# ---------------------------------------------------------------------------------------------------------- 7
def test_input_grad_guards(cuda):
    from audio_diffusion_b200 import _lib
    model, _, _, noisy, t, _, _ = _unet_case(cuda)
    _freeze(model)
    x = noisy.clone().requires_grad_(True)
    out = _call(model, x, t, None)
    _call(model, x, t, None)                 # another forward before the first one's backward
    with pytest.raises(_lib.B200ADError, match="another forward"):
        out.sum().backward()
    out = _call(model, x, t, None)
    (gx,) = torch.autograd.grad(out.square().sum(), x, create_graph=True)
    with pytest.raises(RuntimeError):        # the engine's backward is not differentiable again
        gx.sum().backward()
    # an encoding that requires grad is refused whenever the call has a backward, in eval() and in train()
    cond, _, _, cx, ct, enc, _ = _unet_case(cuda, 1)
    enc_g = enc.clone().requires_grad_(True)
    for train in (False, True):
        cond.train(train)
        with pytest.raises(NotImplementedError):
            cond(cx.clone().requires_grad_(True), ct, enc_g)
    # an autoencoder batch over max_batch: forward values, but the backward refuses
    vae, _, _, vx, _ = _vae(cuda, max_batch=1)
    _freeze(vae)
    xl = vx.clone().requires_grad_(True)
    m = vae.encode(xl).latent_dist.mode()
    with pytest.raises(_lib.B200ADError, match="max_batch"):
        m.sum().backward()
    zl = torch.zeros(2, 1, 8, 8, device=cuda, requires_grad=True)
    with pytest.raises(_lib.B200ADError, match="max_batch"):
        vae.decode(zl).sample.sum().backward()
