"""GPU parity of the optimizer side of the training step (b200ad_optim_step, b200ad_mse_loss_grad) against
oracle/train_oracle.py (itself pinned against torch.optim.AdamW on the CPU).  fp32 elementwise math: tolerance 2e-6
relative (fused multiply-adds and the order of the gradient-norm reduction differ from torch's)."""
import pytest
import torch

from cases import TWO_LEVEL

pytestmark = pytest.mark.gpu


def test_fused_adamw_clip_ema_matches_oracle(cuda):
    from audio_diffusion_b200.training import EMAModel, FusedAdamW
    from oracle.train_oracle import adamw_update, clip_grad_norm, ema_decay
    g = torch.Generator().manual_seed(0)
    shapes = [(128, 1, 3, 3), (128,), (517,), (256, 128, 3, 3), (70001,)]   # odd sizes straddle the 16384-element chunks
    ref = [torch.randn(s, generator=g) for s in shapes]
    params = [torch.nn.Parameter(r.clone().to(cuda)) for r in ref]
    opt = FusedAdamW(params, lr=1e-4, betas=(0.95, 0.999), weight_decay=1e-6, eps=1e-8, max_grad_norm=1.0)
    ema = EMAModel(params, inv_gamma=1.0, power=0.75, max_value=0.9999)
    opt.attach_ema(ema)
    m = [torch.zeros_like(r) for r in ref]
    v = [torch.zeros_like(r) for r in ref]
    sh = [r.clone() for r in ref]
    for step in range(1, 5):
        scale = 10.0 if step != 3 else 1e-3     # step 3: total norm < 1 -> no clipping
        grads = [torch.randn(s, generator=g) * scale for s in shapes]
        for p, gr in zip(params, grads):
            p.grad = gr.to(cuda)
        lr = 1e-4 * step
        opt.param_groups[0]["lr"] = lr          # what LambdaLR does between steps
        opt.step()
        ema.step(params)
        clipped, total = clip_grad_norm({str(i): gr for i, gr in enumerate(grads)}, 1.0)
        d = ema_decay(step, 1.0, 0.75, 0.9999)
        assert abs(ema.cur_decay_value - d) < 1e-12
        assert abs(opt.grad_norm.item() - total.item()) <= 2e-6 * total.item()
        for i in range(len(ref)):
            adamw_update(ref[i], clipped[str(i)], m[i], v[i], step, lr)
            sh[i].sub_((1.0 - d) * (sh[i] - ref[i]))
            assert torch.allclose(params[i].detach().cpu(), ref[i], rtol=2e-6, atol=1e-7), (step, i)
            assert torch.allclose(opt.state[params[i]]["exp_avg_sq"].cpu(), v[i], rtol=2e-6, atol=1e-12), (step, i)
            assert torch.allclose(ema.shadow_params[i].cpu(), sh[i], rtol=2e-6, atol=1e-7), (step, i)
    # copy_to (train_unet.py:292-301)
    ema.copy_to(params)
    assert torch.equal(params[0].detach(), ema.shadow_params[0])


def test_mse_loss_grad(cuda):
    from audio_diffusion_b200.training import mse_loss
    g = torch.Generator().manual_seed(1)
    pred = torch.randn(3, 1, 64, 48, generator=g)
    tgt = torch.randn(3, 1, 64, 48, generator=g)
    p = pred.clone().requires_grad_(True)
    ref = torch.nn.functional.mse_loss(p, tgt)
    ref.backward()
    loss, grad = mse_loss(pred.to(cuda), tgt.to(cuda))
    assert abs(loss.item() - ref.item()) <= 1e-6 * abs(ref.item())
    assert torch.allclose(grad.cpu(), p.grad, rtol=1e-6, atol=1e-9)


def _grad_report(model, grads_ref):
    rows = []
    num = den = 0.0
    for k, p in model.named_parameters():
        g, r = p.grad.detach().cpu().double(), grads_ref[k].double()
        e = (g - r).norm().item()
        s = r.norm().item()
        rows.append((e / (s + 1e-30), k, s, g.norm().item()))
        num += e * e
        den += s * s
    rows.sort(reverse=True)
    return rows, (num / den) ** 0.5


def test_unet_backward_matches_autograd(cuda):
    """All 300+ parameter gradients of one training step's loss (scripts/train_unet.py:250-259: add_noise, U-Net forward with
    per-sample timesteps, MSE, backward) from `b200ad_unet_backward` against torch autograd over the fp32 oracle.
    Tolerance (stated): activations and their gradients are bf16 on the GPU (what bf16 autocast gives the reference) —
    the concatenated gradient must agree to 3 % relative L2, every tensor with a non-negligible gradient to 10 %."""
    from audio_diffusion_b200.training import mse_loss
    from audio_diffusion_b200.unet import UNet2DModel
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.train_oracle import loss_and_grads
    from oracle.unet_oracle import UNetConfig, init_weights
    ocfg = UNetConfig(sample_size=(32, 32), **TWO_LEVEL)
    w = init_weights(ocfg, seed=2)
    model = UNet2DModel(sample_size=(32, 32), **TWO_LEVEL)
    model.load_state_dict(w)
    model = model.to(cuda).train()
    g = torch.Generator().manual_seed(3)
    clean = torch.rand(2, 1, 32, 32, generator=g) * 2 - 1
    noise = torch.randn(2, 1, 32, 32, generator=g)
    t = torch.tensor([37, 712])
    loss_ref, grads_ref, pred_ref = loss_and_grads(w, ocfg, clean, noise, t)
    noisy = OracleDDPM().add_noise(clean, noise, t).to(cuda)
    pred = model(noisy, t.to(cuda))["sample"]
    loss = torch.nn.functional.mse_loss(pred, noise.to(cuda))
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - loss_ref.item()) <= 2e-2 * loss_ref.item()
    rows, total = _grad_report(model, grads_ref)
    for e, k, s, gn in rows[:30]:
        print(f"{e:9.4f}  |ref| {s:10.3e}  |got| {gn:10.3e}  {k}")
    print("total relative L2 error", total, "backward launches", model.last_backward_launch_count)
    gmax = max(r[2] for r in rows)
    bad = [(e, k) for e, k, s, _ in rows if e > 0.10 and s > 1e-3 * gmax]
    assert total <= 3e-2 and not bad, (total, bad[:10])
    # inference after training mode still works (workspace is re-planned with pooling)
    with torch.no_grad():
        out = model(noisy, t.to(cuda))["sample"]
    assert (out - pred.detach()).abs().max() <= 2e-3 * pred.detach().abs().max() + 1e-5


def test_two_training_steps_match_oracle(cuda):
    """Two full iterations of scripts/train_unet.py:238-267 (add_noise, forward, MSE, backward, clip 1.0, AdamW, cosine LR
    with warm-up, EMA) on the engine vs oracle/train_oracle.py::train_step: loss to 2 %, updated parameters and EMA shadows
    to 2e-3 of the parameter update scale after two steps (Adam normalises the update, so bf16 gradient noise shows up
    only where |g| is comparable to its own error)."""
    import sys, os
    from audio_diffusion_b200.schedulers import DDPMScheduler
    from audio_diffusion_b200.training import EMAModel, FusedAdamW, train_step
    from audio_diffusion_b200.unet import UNet2DModel
    from oracle.train_oracle import TrainState
    from oracle.train_oracle import train_step as oracle_step
    from oracle.unet_oracle import UNetConfig, init_weights
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "audio_diffusion_b200", "compat"))
    try:
        from diffusers.optimization import get_scheduler
    finally:
        sys.path.pop(0)
    ocfg = UNetConfig(sample_size=(32, 32), **TWO_LEVEL)
    w = init_weights(ocfg, seed=4)
    w0 = {k: v.clone() for k, v in w.items()}
    model = UNet2DModel(sample_size=(32, 32), **TWO_LEVEL)
    model.load_state_dict(w)
    model = model.to(cuda).train()
    opt = FusedAdamW(model.parameters(), lr=1e-4, betas=(0.95, 0.999), weight_decay=1e-6, eps=1e-8, max_grad_norm=1.0)
    ema = EMAModel(model.parameters(), inv_gamma=1.0, power=0.75, max_value=0.9999)
    opt.attach_ema(ema)
    lrs = get_scheduler("cosine", optimizer=opt, num_warmup_steps=1, num_training_steps=10)
    sch = DDPMScheduler()
    st = TrainState()
    g = torch.Generator().manual_seed(5)
    for it in range(2):
        clean = torch.rand(2, 1, 32, 32, generator=g) * 2 - 1
        noise = torch.randn(2, 1, 32, 32, generator=g)
        t = torch.randint(0, 1000, (2,), generator=g)
        if it == 0:
            # LambdaLR starts at lambda(0) = 0 with one warm-up step: the oracle mirrors that
            pass
        loss_ref, gnorm_ref, lr_ref, decay_ref = oracle_step(w, ocfg, st, clean, noise, t, base_lr=1e-4, warmup=1,
                                                             total_steps=10)
        assert abs(opt.param_groups[0]["lr"] - lr_ref) < 1e-12
        loss = train_step(model, opt, sch, clean.to(cuda), ema=ema, lr_scheduler=lrs, noise=noise.to(cuda), timesteps=t.to(cuda))
        assert abs(loss.item() - loss_ref.item()) <= 2e-2 * loss_ref.item(), (it, loss.item(), loss_ref.item())
        assert abs(opt.grad_norm.item() - gnorm_ref.item()) <= 2e-2 * gnorm_ref.item()
        assert abs(ema.cur_decay_value - decay_ref) < 1e-12
    upd = max((w[k] - w0[k]).abs().max().item() for k in w)
    assert upd > 0
    sd = {k: v.detach().cpu() for k, v in model.named_parameters()}
    worst = max((sd[k] - w[k]).abs().max().item() for k in w)
    names = [k for k, _ in model.named_parameters()]
    worst_ema = max((s.cpu() - st.ema[k]).abs().max().item() for s, k in zip(ema.shadow_params, names))
    print("max update", upd, "worst param diff", worst, "worst ema diff", worst_ema)
    # Adam normalises the step: where the true gradient is (numerically) zero — e.g. the softmax-invariant to_k.bias — the
    # update direction is rounding noise on BOTH sides, so the bar is on the fraction of elements, not the worst one
    total = sum(v.numel() for v in w.values())
    frac = sum(((sd[k] - w[k]).abs() <= 0.1 * upd).float().sum().item() for k in w) / total
    frac_ema = sum(((s.cpu() - st.ema[k]).abs() <= 0.1 * upd).float().sum().item()
                   for s, k in zip(ema.shadow_params, names)) / total
    print("fraction within 10% of the update scale:", frac, frac_ema)
    assert frac >= 0.99 and frac_ema >= 0.99, (frac, frac_ema)


@pytest.mark.timeout(900)
def test_unet_backward_reference_architecture(cuda):
    """Same gradient parity on the architecture the reference trains (scripts/train_unet.py:115-137: six levels, attention in
    down block 4 / up block 1, 113.67 M parameters) at 64x64, batch 1 — every block type at every depth, 2x2 bottleneck."""
    from audio_diffusion_b200.unet import UNet2DModel
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.train_oracle import loss_and_grads
    from oracle.unet_oracle import UNetConfig, init_weights
    full = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 128, 256, 256, 512, 512),
                down_block_types=("DownBlock2D",) * 4 + ("AttnDownBlock2D", "DownBlock2D"),
                up_block_types=("UpBlock2D", "AttnUpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D"))
    ocfg = UNetConfig(sample_size=(64, 64), **full)
    w = init_weights(ocfg, seed=7)
    model = UNet2DModel(sample_size=(64, 64), **full)
    model.load_state_dict(w)
    model = model.to(cuda).train()
    g = torch.Generator().manual_seed(8)
    clean = torch.rand(1, 1, 64, 64, generator=g) * 2 - 1
    noise = torch.randn(1, 1, 64, 64, generator=g)
    t = torch.tensor([500])
    loss_ref, grads_ref, _ = loss_and_grads(w, ocfg, clean, noise, t)
    noisy = OracleDDPM().add_noise(clean, noise, t).to(cuda)
    pred = model(noisy, t.to(cuda))["sample"]
    torch.nn.functional.mse_loss(pred, noise.to(cuda)).backward()
    torch.cuda.synchronize()
    rows, total = _grad_report(model, grads_ref)
    for e, k, s, gn in rows[:12]:
        print(f"{e:9.4f}  |ref| {s:10.3e}  |got| {gn:10.3e}  {k}")
    print("total relative L2 error", total)
    gmax = max(r[2] for r in rows)
    bad = [(e, k) for e, k, s, _ in rows if e > 0.10 and s > 1e-3 * gmax]
    assert total <= 3e-2 and not bad, (total, bad[:10])


def test_ema_copy_to_refreshes_packed_weights(cuda):
    """scripts/train_unet.py:292-301: `ema_model.copy_to(unet.parameters())` right before sampling — the engine must notice
    that the parameters changed (its bf16-packed copy is keyed on parameter versions)."""
    from audio_diffusion_b200.training import EMAModel
    from audio_diffusion_b200.unet import UNet2DModel
    m = UNet2DModel(sample_size=(32, 32), seed=1, **TWO_LEVEL).to(cuda)
    x = torch.randn(1, 1, 32, 32, generator=torch.Generator().manual_seed(0)).to(cuda)
    with torch.no_grad():
        a = m(x, 10)["sample"].clone()
        ema = EMAModel(m.parameters())
        for s in ema.shadow_params:
            s.mul_(0.5)
        ema.copy_to(m.parameters())
        b = m(x, 10)["sample"].clone()
    assert (a - b).abs().max() > 1e-3 * a.abs().max()


def test_gradient_accumulation_equals_full_batch(cuda):
    """`accelerator.accumulate(model)` (scripts/train_unet.py:252): two micro-batches with loss / 2 each, gradients left in
    place between the backward calls, give the gradient of the full batch (GroupNorm is per sample)."""
    from audio_diffusion_b200.unet import UNet2DModel
    model = UNet2DModel(sample_size=(32, 32), seed=3, **TWO_LEVEL).to(cuda).train()
    g = torch.Generator().manual_seed(6)
    x = torch.randn(2, 1, 32, 32, generator=g).to(cuda)
    tgt = torch.randn(2, 1, 32, 32, generator=g).to(cuda)
    t = torch.tensor([100, 650]).to(cuda)
    torch.nn.functional.mse_loss(model(x, t)["sample"], tgt).backward()
    full = model._grad_flat.clone()
    for p in model.parameters():
        p.grad = None
    with model.no_sync():
        (torch.nn.functional.mse_loss(model(x[:1], t[:1])["sample"], tgt[:1]) / 2).backward()
    (torch.nn.functional.mse_loss(model(x[1:], t[1:])["sample"], tgt[1:]) / 2).backward()
    acc = model._grad_flat
    rel = ((acc - full).norm() / full.norm()).item()
    assert rel < 2e-3, rel


def test_backward_after_second_forward_is_refused(cuda):
    """The training forward keeps its activations in the model's single workspace: a second forward before backward()
    would silently give wrong gradients, so the engine refuses (ADVICE r1)."""
    from audio_diffusion_b200._lib import B200ADError
    from audio_diffusion_b200.unet import UNet2DModel
    model = UNet2DModel(sample_size=(32, 32), seed=3, **TWO_LEVEL).to(cuda).train()
    x = torch.randn(2, 1, 32, 32, generator=torch.Generator().manual_seed(1)).to(cuda)
    t = torch.tensor([10, 500]).to(cuda)
    first = model(x, t)["sample"]
    with torch.no_grad():
        model(x, t)                       # e.g. an evaluation call in between
    with pytest.raises(B200ADError):
        first.sum().backward()
    model(x, t)["sample"].sum().backward()      # the latest forward is fine
    assert all(p.grad is not None for p in model.parameters())
