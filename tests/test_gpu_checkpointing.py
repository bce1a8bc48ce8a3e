"""Gradient checkpointing (`enable_gradient_checkpointing()`) on the GPU: the training forward keeps only the block outputs and
the backward recomputes every block's internals with the same forward kernels.  The forward output must not change, the
gradients must agree with the plain backward's within a few times the run-to-run spread of the plain backward itself
(its GroupNorm / LayerNorm / bias and split-K weight-gradient reductions accumulate with float atomics, so two plain
backward passes differ in the last bits, tests/test_gpu_cond_seq.py), the recompute must write no kept tensor, and one
training iteration must need less memory."""
import gc

import pytest
import torch

from cases import LDM, PUBLISHED, PUBLISHED_COND

pytestmark = pytest.mark.gpu

K_SPREAD = 4.0     # checkpointed gradient error allowed, in units of the plain backward's run-to-run difference


def _unet(cuda, s, seed=0):
    from audio_diffusion_b200.unet import UNet2DModel
    from audio_diffusion_b200.unet_cond import UNet2DConditionModel
    if s is None:
        return UNet2DModel(sample_size=(64, 64), seed=seed, **PUBLISHED).to(cuda).train()
    return UNet2DConditionModel(sample_size=(64, 64), seed=seed, **PUBLISHED_COND).to(cuda).train()


def _inputs(cuda, s, n=4, size=64, seed=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 1, size, size, generator=g).to(cuda)
    tgt = torch.randn(n, 1, size, size, generator=g).to(cuda)
    t = torch.randint(0, 1000, (n,), generator=g).to(cuda)
    enc = None if s is None else torch.randn(n, s, 100, generator=g).to(cuda)
    return x, tgt, t, enc


def _call(model, x, t, enc):
    return model(x, t)["sample"] if enc is None else model(x, t, enc)["sample"]


def _iteration(model, x, tgt, t, enc):
    """(output, flat gradient) of one forward + MSE + backward from zeroed gradients."""
    for p in model.parameters():
        p.grad = None
    out = _call(model, x, t, enc)
    torch.nn.functional.mse_loss(out, tgt).backward()
    torch.cuda.synchronize()
    return out.detach().clone(), model._grad_flat.clone()


def _check_out(got, ref):
    if not torch.equal(got, ref):
        rel = ((got - ref).abs().max() / ref.abs().max()).item()
        assert rel <= 2e-3, rel


def _check_grad(got, ref, ref2, what=""):
    spread = (ref2 - ref).norm().item()
    err = (got - ref).norm().item()
    print(f"{what} |g| {ref.norm().item():.4e}  plain spread {spread:.3e}  checkpointed err {err:.3e}")
    assert err <= K_SPREAD * spread + 1e-6 * ref.norm().item(), (err, spread)


def _block_outputs(model):
    """Names of the U-Net's block-output taps (each block's output, conv_in and the upsamplers)."""
    nb = len(model.config.block_out_channels)
    lp = model.config.layers_per_block
    names = ["conv_in", "mid_block.resnets.0", "mid_block.attentions.0", "mid_block.resnets.1"]
    for i in range(nb):
        for j in range(lp):
            names += [f"down_blocks.{i}.resnets.{j}", f"down_blocks.{i}.attentions.{j}"]
        names.append(f"down_blocks.{i}.downsamplers.0.conv")
        for j in range(lp + 1):
            names += [f"up_blocks.{i}.resnets.{j}", f"up_blocks.{i}.attentions.{j}"]
        names.append(f"up_blocks.{i}.upsamplers.0.conv")
    got = {}
    for n in names:
        try:
            got[n] = model.debug_tensor(n)
        except Exception as e:   # blocks the architecture does not have
            assert "unknown tap" in str(e), (n, e)
    return got


@pytest.mark.parametrize("s", [None, 1, 8], ids=["published", "cond_s1", "cond_s8"])
def test_checkpointed_training_matches_plain(cuda, s):
    """64x64, batch 4: the forward output equal to the plain one's, the flat gradient within K_SPREAD times the spread of two
    plain backward passes, every block output bit-identical before and after the checkpointed backward, an internal tap
    refused by name, and the recompute launches counted."""
    from audio_diffusion_b200 import _lib
    model = _unet(cuda, s)
    x, tgt, t, enc = _inputs(cuda, s)
    out_a, g_a = _iteration(model, x, tgt, t, enc)
    launches_plain = model.last_backward_launch_count
    out_b, g_b = _iteration(model, x, tgt, t, enc)
    assert torch.equal(out_a, out_b)
    model.enable_gradient_checkpointing()
    assert model.is_gradient_checkpointing
    for p in model.parameters():
        p.grad = None
    out_c = _call(model, x, t, enc)
    before = _block_outputs(model)
    assert len(before) > 20
    with pytest.raises(_lib.B200ADError, match="checkpointing"):
        model.debug_tensor("down_blocks.0.resnets.0.h1")
    torch.nn.functional.mse_loss(out_c, tgt).backward()
    torch.cuda.synchronize()
    after = _block_outputs(model)
    assert all(torch.equal(before[k], after[k]) for k in before), [k for k in before if not torch.equal(before[k], after[k])]
    _check_out(out_c.detach(), out_a)
    _check_grad(model._grad_flat, g_a, g_b, f"S={s}")
    print("backward launches", launches_plain, "->", model.last_backward_launch_count)
    assert model.last_backward_launch_count > launches_plain


def _vae_iteration(vae, x, noise):
    from audio_diffusion_b200.training import vae_loss
    for p in vae.parameters():
        p.grad = None
    post = vae.encode(x).latent_dist
    z = post.mean + post.std * noise
    x_hat = vae.decode(z).sample
    vae_loss(x, x_hat, post)[0].backward()
    torch.cuda.synchronize()
    parts = {"encoder": [], "decoder": []}
    for k, p in vae.named_parameters():
        parts["decoder" if k.startswith(("decoder.", "post_quant_conv.")) else "encoder"].append(p.grad.flatten())
    return x_hat.detach().clone(), {k: torch.cat(v).clone() for k, v in parts.items()}


def test_checkpointed_autoencoder_matches_plain(cuda):
    """The ldm autoencoder at 64x64, batch 2: the decoded image as without checkpointing, the decoder's and the encoder's
    gradients within K_SPREAD times the plain spread, block outputs untouched by the backward."""
    from audio_diffusion_b200.vae import AutoencoderKL
    vae = AutoencoderKL(seed=0, **LDM).to(cuda).train()
    g = torch.Generator().manual_seed(3)
    x = (torch.rand(2, 1, 64, 64, generator=g) * 2 - 1).to(cuda)
    noise = torch.randn(2, 1, 8, 8, generator=g).to(cuda)
    xa, ga = _vae_iteration(vae, x, noise)
    xb, gb = _vae_iteration(vae, x, noise)
    vae.enable_gradient_checkpointing()
    assert vae.is_gradient_checkpointing
    names = ["decoder.mid_block.attentions.0", "decoder.up_blocks.1.resnets.2", "encoder.down_blocks.0.downsamplers.0.conv",
             "encoder.mid_block.resnets.1"]
    from audio_diffusion_b200.training import vae_loss
    for p in vae.parameters():
        p.grad = None
    post = vae.encode(x).latent_dist
    x_hat = vae.decode(post.mean + post.std * noise).sample
    before = {n: vae.debug_tensor(n) for n in names}
    vae_loss(x, x_hat, post)[0].backward()
    torch.cuda.synchronize()
    assert all(torch.equal(before[n], vae.debug_tensor(n)) for n in names)
    _check_out(x_hat.detach(), xa)
    gc_ = {"encoder": [], "decoder": []}
    for k, p in vae.named_parameters():
        gc_["decoder" if k.startswith(("decoder.", "post_quant_conv.")) else "encoder"].append(p.grad.flatten())
    for part in ("decoder", "encoder"):
        _check_grad(torch.cat(gc_[part]), ga[part], gb[part], part)


def test_checkpointed_accumulation_and_train_step(cuda):
    """Two micro-batches accumulated under no_sync, then training.train_step on the whole batch, with and without
    checkpointing from the same weights: the accumulated gradient within K_SPREAD times the plain spread, the train_step
    loss within 1e-4, and the AdamW update of every parameter within a tenth of the learning rate for 99.9 % of them."""
    from audio_diffusion_b200.schedulers import DDPMScheduler
    from audio_diffusion_b200.training import FusedAdamW, train_step
    x, tgt, t, enc = _inputs(cuda, 8, seed=5)
    lr = 1e-4

    def run(ckpt):
        model = _unet(cuda, 8, seed=2)
        if ckpt:
            model.enable_gradient_checkpointing()
        opt = FusedAdamW(model.parameters(), lr=lr)
        with model.no_sync():
            (torch.nn.functional.mse_loss(_call(model, x[:2], t[:2], enc[:2]), tgt[:2]) / 2).backward()
        (torch.nn.functional.mse_loss(_call(model, x[2:], t[2:], enc[2:]), tgt[2:]) / 2).backward()
        g = model._grad_flat.clone()
        opt.step()
        opt.zero_grad(set_to_none=True)
        sch = DDPMScheduler(num_train_timesteps=1000)
        loss = train_step(model, opt, sch, x, noise=tgt, timesteps=t, encoder_hidden_states=enc)
        torch.cuda.synchronize()
        return g, loss.item(), torch.cat([p.detach().flatten() for p in model.parameters()])

    g_a, loss_a, p_a = run(False)
    g_b, _, _ = run(False)
    g_c, loss_c, p_c = run(True)
    _check_grad(g_c, g_a, g_b, "accumulated")
    assert abs(loss_c - loss_a) <= 1e-4 * abs(loss_a), (loss_c, loss_a)
    d = (p_c - p_a).abs()
    print("max parameter difference / lr", (d.max() / lr).item())
    assert (d > 0.1 * lr).float().mean().item() < 1e-3


def test_toggling_matches_fresh_models(cuda):
    """off -> on -> off between iterations of one model gives what a model bound fresh in each mode gives."""
    x, tgt, t, enc = _inputs(cuda, 8, seed=7)
    fresh = {}
    for mode in (False, True):
        m = _unet(cuda, 8, seed=4)
        if mode:
            m.enable_gradient_checkpointing()
        fresh[mode] = (_iteration(m, x, tgt, t, enc), _iteration(m, x, tgt, t, enc))
        del m
    model = _unet(cuda, 8, seed=4)
    for mode in (False, True, False):
        (model.enable_gradient_checkpointing if mode else model.disable_gradient_checkpointing)()
        assert model.is_gradient_checkpointing == mode
        out, g = _iteration(model, x, tgt, t, enc)
        (ref_out, ref_g), (_, ref_g2) = fresh[mode]
        _check_out(out, ref_out)
        _check_grad(g, ref_g, ref_g2, f"checkpointing={mode}")


def _peak_iteration_bytes(cuda, ckpt):
    from audio_diffusion_b200.unet import UNet2DModel
    model = UNet2DModel(sample_size=(256, 256), seed=0, **PUBLISHED).to(cuda).train()
    if ckpt:
        model.enable_gradient_checkpointing()
    x, tgt, t, _ = _inputs(cuda, None, n=2, size=256)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    torch.nn.functional.mse_loss(model(x, t)["sample"], tgt).backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del model
    gc.collect()
    torch.cuda.empty_cache()
    return peak


def test_checkpointing_lowers_peak_memory(cuda):
    """One training iteration of the published U-Net at 256x256, batch 2: the peak memory it allocates on top of the
    parameters is lower with checkpointing."""
    off = _peak_iteration_bytes(cuda, False)
    on = _peak_iteration_bytes(cuda, True)
    print(f"peak allocated by one iteration: off {off / 2**30:.3f} GiB, on {on / 2**30:.3f} GiB ({on / off:.3f})")
    assert on < off
