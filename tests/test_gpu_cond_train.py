"""GPU parity of conditional training (scripts/train_unet.py --encodings: `model(noisy, t, enc)["sample"]`, MSE, backward,
clip, AdamW, EMA) on the architecture train_unet.py:139-159 builds, against torch autograd over the fp32 oracle
(oracle/unet_cond_oracle.py).  The bars are those of tests/test_gpu_train.py: activations and their gradients are bf16 on
the GPU (what bf16 autocast gives the reference), so the concatenated gradient must agree to 3 % relative L2 and every
tensor with a non-negligible gradient to 10 %; the attention backward alone to 2 % relative L2 per output."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

ARCH = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256, 512, 512),
            down_block_types=("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",),
            up_block_types=("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3, cross_attention_dim=100)
ZERO_GRAD = ("attn2.to_q.weight", "attn2.to_k.weight", "norm2.weight", "norm2.bias")


def cond_loss_and_grads(w, cfg, clean, noise, t, enc):
    """MSE(ε̂, ε) of one conditional training step (scripts/train_unet.py:250-258) and its parameter gradients, by fp32
    autograd over the oracle."""
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_cond_oracle import unet_cond_forward
    noisy = OracleDDPM().add_noise(clean, noise, t)
    wl = {k: v.detach().clone().requires_grad_(True) for k, v in w.items()}
    pred = unet_cond_forward(wl, cfg, noisy, t, enc)
    loss = torch.mean((pred - noise) ** 2)
    grads = torch.autograd.grad(loss, list(wl.values()))
    return loss.detach(), dict(zip(wl.keys(), grads))


def _rel_l2(got, ref):
    return ((got.double() - ref.double()).norm() / (ref.double().norm() + 1e-30)).item()


@pytest.mark.parametrize("d,hh,ww", [(16, 4, 4), (32, 4, 4), (64, 4, 4), (16, 20, 20), (32, 20, 20), (64, 20, 20),
                                     (16, 64, 64)])
def test_mha_forward_backward_matches_autograd(cuda, d, hh, ww):
    """b200ad_mha_forward_backward (8 heads of dim d, seq = hh * ww; 400 is not a multiple of the 64-row tiles) against CPU
    fp32 autograd of oracle.unet_cond_oracle._mha: O, dQ, dK, dV each within 2 % relative L2."""
    from audio_diffusion_b200 import _lib
    from oracle.unet_cond_oracle import _mha
    heads, n = 8, 2
    c = heads * d
    g = torch.Generator().manual_seed(d * 1000 + hh)
    q, k, v, do = (torch.randn(n, c, hh, ww, generator=g) for _ in range(4))
    tok = lambda a: a.flatten(2).transpose(1, 2)                  # [N, C, H, W] -> (N, seq, C)
    ql, kl, vl = (a.clone().requires_grad_(True) for a in (q, k, v))
    o_ref = _mha(tok(ql), tok(kl), tok(vl), heads)
    o_ref.backward(tok(do))
    L = _lib.lib()
    qd, kd, vd, dod = (a.to(cuda).contiguous() for a in (q, k, v, do))
    out, dq, dk, dv = (torch.empty_like(qd) for _ in range(4))
    nb = L.b200ad_mha_scratch_bytes(n, c, heads, hh, ww)
    scratch = torch.empty(nb, dtype=torch.uint8, device=cuda)
    _lib.check(L.b200ad_mha_forward_backward(qd.data_ptr(), kd.data_ptr(), vd.data_ptr(), dod.data_ptr(), out.data_ptr(),
                                             dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), n, c, heads, hh, ww,
                                             scratch.data_ptr(), nb, _lib.stream_ptr()))
    torch.cuda.synchronize()
    errs = {"O": _rel_l2(tok(out.cpu()), o_ref.detach()), "dQ": _rel_l2(dq.cpu(), ql.grad),
            "dK": _rel_l2(dk.cpu(), kl.grad), "dV": _rel_l2(dv.cpu(), vl.grad)}
    print(d, hh, ww, errs)
    assert all(e <= 2e-2 for e in errs.values()), errs


# two levels, transformers at 32x32 (head_dim 16) in the down and the up block: the scale of test_gpu_train.py's TRAIN_CFG
SMALL = dict(ARCH, block_out_channels=(128, 256), down_block_types=("CrossAttnDownBlock2D", "DownBlock2D"),
             up_block_types=("UpBlock2D", "CrossAttnUpBlock2D"))


def _build(cuda, size, seed, arch=ARCH):
    from audio_diffusion_b200.unet_cond import UNet2DConditionModel
    from oracle.unet_cond_oracle import CondUNetConfig, init_weights
    ocfg = CondUNetConfig(sample_size=size, block_out_channels=arch["block_out_channels"],
                          down_block_types=arch["down_block_types"], up_block_types=arch["up_block_types"])
    w = init_weights(ocfg, seed=seed)
    model = UNet2DConditionModel(sample_size=size, **arch)
    model.load_state_dict(w)
    return model.to(cuda).train(), ocfg, w


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


def _check_grads(cuda, size, n, seed):
    from oracle.schedulers_oracle import OracleDDPM
    model, ocfg, w = _build(cuda, size, seed)
    g = torch.Generator().manual_seed(seed + 1)
    clean = torch.rand(n, 1, *size, generator=g) * 2 - 1
    noise = torch.randn(n, 1, *size, generator=g)
    enc = torch.randn(n, 1, 100, generator=g)
    t = torch.tensor([37, 712][:n])
    loss_ref, grads_ref = cond_loss_and_grads(w, ocfg, clean, noise, t, enc)
    noisy = OracleDDPM().add_noise(clean, noise, t).to(cuda)
    pred = model(noisy, t.to(cuda), enc.to(cuda))["sample"]
    loss = torch.nn.functional.mse_loss(pred, noise.to(cuda))
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - loss_ref.item()) <= 2e-2 * loss_ref.item(), (loss.item(), loss_ref.item())
    rows, total = _grad_report(model, grads_ref)
    for e, k, s, gn in rows[:20]:
        print(f"{e:9.4f}  |ref| {s:10.3e}  |got| {gn:10.3e}  {k}")
    print("total relative L2 error", total, "backward launches", model.last_backward_launch_count)
    gmax = max(r[2] for r in rows)
    bad = [(e, k) for e, k, s, _ in rows if e > 0.10 and s > 1e-3 * gmax]
    assert total <= 3e-2 and not bad, (total, bad[:10])
    named = dict(model.named_parameters())
    zero = [k for k in named if any(k.endswith(".transformer_blocks.0." + z) for z in ZERO_GRAD)]
    assert len(zero) == 16 * 4
    assert all(torch.count_nonzero(named[k].grad) == 0 for k in zero)
    return model, noisy, t, enc, pred


def test_cond_unet_backward_matches_autograd(cuda):
    """Every parameter gradient of one conditional training loss at 32x32, batch 2, per-sample timesteps; then an eval
    forward after training mode must give the training forward's epsilon (inference is re-planned with pooling)."""
    model, noisy, t, enc, pred = _check_grads(cuda, (32, 32), 2, seed=2)
    with torch.no_grad():
        out = model.eval()(noisy, t.to(cuda), enc.to(cuda))["sample"]
    rel = ((out - pred.detach()).abs().max() / pred.detach().abs().max()).item()
    assert rel <= 2e-3, rel


@pytest.mark.timeout(900)
def test_cond_unet_backward_matches_autograd_64(cuda):
    """The same at the published model's 64x64 latent, batch 1: attention over 4096 pixels at head_dim 16."""
    _check_grads(cuda, (64, 64), 1, seed=5)


def _oracle_train_step(w, ocfg, st, clean, noise, t, enc, base_lr, warmup, total_steps):
    """oracle.train_oracle.train_step with the conditional loss: clip 1.0, AdamW, cosine LR with warm-up, EMA."""
    from oracle.train_oracle import adamw_update, clip_grad_norm, cosine_with_warmup, ema_decay
    if not st.ema:
        st.ema = {k: v.detach().clone() for k, v in w.items()}
    loss, grads = cond_loss_and_grads(w, ocfg, clean, noise, t, enc)
    grads, gnorm = clip_grad_norm(grads, 1.0)
    lr = base_lr * cosine_with_warmup(st.step, warmup, total_steps)
    st.step += 1
    for k in w:
        if k not in st.exp_avg:
            st.exp_avg[k] = torch.zeros_like(w[k])
            st.exp_avg_sq[k] = torch.zeros_like(w[k])
        adamw_update(w[k], grads[k], st.exp_avg[k], st.exp_avg_sq[k], st.step, lr)
    decay = ema_decay(st.step)
    for k in w:
        st.ema[k].sub_((1.0 - decay) * (st.ema[k] - w[k]))
    return loss, gnorm, lr, decay


def test_cond_two_training_steps_match_oracle(cuda):
    """training.train_step(..., encoder_hidden_states=enc) with FusedAdamW, EMA and cosine LR, twice, against the oracle step:
    loss and gradient norm to 2 %, parameters and EMA shadows within 10 % of the update scale for 99 % of the elements.
    Like test_two_training_steps_match_oracle it runs a two-level model: Adam turns every element's gradient into a step of
    about lr, so elements whose true gradient is below the bf16 gradient noise flip sides, and the deep bottleneck resnets of
    the full architecture hold more of those (measured there: 97.8 % of the parameters within the bar, the misses spread
    over all layer kinds, resnet convolutions most; the gradient bars themselves are checked on the full architecture)."""
    import os
    import sys
    from audio_diffusion_b200.schedulers import DDPMScheduler
    from audio_diffusion_b200.training import EMAModel, FusedAdamW, train_step
    from oracle.train_oracle import TrainState
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "audio_diffusion_b200", "compat"))
    try:
        from diffusers.optimization import get_scheduler
    finally:
        sys.path.pop(0)
    model, ocfg, w = _build(cuda, (32, 32), seed=4, arch=SMALL)
    w0 = {k: v.clone() for k, v in w.items()}
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
        enc = torch.randn(2, 1, 100, generator=g)
        t = torch.randint(0, 1000, (2,), generator=g)
        loss_ref, gnorm_ref, lr_ref, decay_ref = _oracle_train_step(w, ocfg, st, clean, noise, t, enc, 1e-4, 1, 10)
        assert abs(opt.param_groups[0]["lr"] - lr_ref) < 1e-12
        loss = train_step(model, opt, sch, clean.to(cuda), ema=ema, lr_scheduler=lrs, noise=noise.to(cuda),
                          timesteps=t.to(cuda), encoder_hidden_states=enc.to(cuda))
        assert abs(loss.item() - loss_ref.item()) <= 2e-2 * loss_ref.item(), (it, loss.item(), loss_ref.item())
        assert abs(opt.grad_norm.item() - gnorm_ref.item()) <= 2e-2 * gnorm_ref.item()
        assert abs(ema.cur_decay_value - decay_ref) < 1e-12
    upd = max((w[k] - w0[k]).abs().max().item() for k in w)
    assert upd > 0
    sd = {k: v.detach().cpu() for k, v in model.named_parameters()}
    names = [k for k, _ in model.named_parameters()]
    total = sum(v.numel() for v in w.values())
    frac = sum(((sd[k] - w[k]).abs() <= 0.1 * upd).float().sum().item() for k in w) / total
    frac_ema = sum(((s.cpu() - st.ema[k]).abs() <= 0.1 * upd).float().sum().item()
                   for s, k in zip(ema.shadow_params, names)) / total
    print("max update", upd, "fraction within 10% of the update scale:", frac, frac_ema)
    assert frac >= 0.99 and frac_ema >= 0.99, (frac, frac_ema)


def test_cond_reference_loop_body_on_engine_gradients(cuda):
    """scripts/train_unet.py:252-267 as written: model(noisy, t, enc)["sample"], F.mse_loss, backward, clip_grad_norm_, stock
    torch.optim.AdamW on the engine's p.grad views; on a fixed batch the loss goes down."""
    import torch.nn.functional as F
    from audio_diffusion_b200.schedulers import DDPMScheduler
    model, _, _ = _build(cuda, (32, 32), seed=6)
    optimizer = torch.optim.AdamW(model.parameters(), lr=3e-4, betas=(0.95, 0.999), weight_decay=1e-6, eps=1e-8)
    noise_scheduler = DDPMScheduler()
    g = torch.Generator().manual_seed(7)
    clean_images = (torch.rand(4, 1, 32, 32, generator=g) * 2 - 1).to(cuda)
    noise = torch.randn(4, 1, 32, 32, generator=g).to(cuda)
    encoding = torch.randn(4, 1, 100, generator=g).to(cuda)
    timesteps = torch.tensor([50, 300, 600, 900]).to(cuda)
    noisy_images = noise_scheduler.add_noise(clean_images, noise, timesteps)
    losses = []
    for _ in range(6):
        noise_pred = model(noisy_images, timesteps, encoding)["sample"]
        loss = F.mse_loss(noise_pred, noise)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 1.0)
        optimizer.step()
        optimizer.zero_grad()
        losses.append(loss.item())
    print("losses", losses)
    assert all(math.isfinite(v) for v in losses)
    assert losses[-1] < losses[0], losses


def test_cond_gradient_accumulation_equals_full_batch(cuda):
    """Two half-batches (loss / 2 each, the first under no_sync) give the full batch's gradient."""
    model, _, _ = _build(cuda, (32, 32), seed=3)
    g = torch.Generator().manual_seed(6)
    x = torch.randn(2, 1, 32, 32, generator=g).to(cuda)
    tgt = torch.randn(2, 1, 32, 32, generator=g).to(cuda)
    enc = torch.randn(2, 1, 100, generator=g).to(cuda)
    t = torch.tensor([100, 650]).to(cuda)
    torch.nn.functional.mse_loss(model(x, t, enc)["sample"], tgt).backward()
    full = model._grad_flat.clone()
    for p in model.parameters():
        p.grad = None
    with model.no_sync():
        (torch.nn.functional.mse_loss(model(x[:1], t[:1], enc[:1])["sample"], tgt[:1]) / 2).backward()
    (torch.nn.functional.mse_loss(model(x[1:], t[1:], enc[1:])["sample"], tgt[1:]) / 2).backward()
    rel = ((model._grad_flat - full).norm() / full.norm()).item()
    assert rel < 2e-3, rel


def test_cond_training_errors(cuda):
    """An encoding that requires grad, or none at all, is refused in training."""
    model, _, _ = _build(cuda, (32, 32), seed=1)
    x = torch.randn(2, 1, 32, 32).to(cuda)
    t = torch.tensor([10, 500]).to(cuda)
    with pytest.raises(NotImplementedError):
        model(x, t, torch.randn(2, 1, 100, device=cuda, requires_grad=True))
    with pytest.raises(ValueError):
        model(x, t)
