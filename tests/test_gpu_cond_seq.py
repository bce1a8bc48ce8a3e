"""GPU parity of the conditional U-Net against encodings of S > 1 tokens (`AudioEncoder.encode(files, pool=None)` gives one
100-d token per 5-second slice, (B, S, 100)): the cross-attention kernels against fp32 autograd, the model forward,
sampling and training against the fp32 oracle (oracle/unet_cond_oracle.py, which attends over any number of tokens), and
the S = 1 path left as it was.  Bars: those of tests/test_gpu_cond.py and tests/test_gpu_cond_train.py."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ARCH = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256, 512, 512),
            down_block_types=("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",),
            up_block_types=("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3, cross_attention_dim=100)
# two levels, transformers at head_dim 16 in the down and the up block (tests/test_gpu_cond_train.py's SMALL)
SMALL = dict(ARCH, block_out_channels=(128, 256), down_block_types=("CrossAttnDownBlock2D", "DownBlock2D"),
             up_block_types=("UpBlock2D", "CrossAttnUpBlock2D"))
ONE_TOKEN_ZERO = ("attn2.to_q.weight", "attn2.to_k.weight", "norm2.weight", "norm2.bias")


def _build(cuda, size, seed, arch=ARCH, train=False):
    from audio_diffusion_b200.unet_cond import UNet2DConditionModel
    from oracle.unet_cond_oracle import CondUNetConfig, init_weights
    ocfg = CondUNetConfig(sample_size=size, block_out_channels=arch["block_out_channels"],
                          down_block_types=arch["down_block_types"], up_block_types=arch["up_block_types"])
    w = init_weights(ocfg, seed=seed)
    model = UNet2DConditionModel(sample_size=size, **arch)
    model.load_state_dict(w)
    model = model.to(cuda)
    return (model.train() if train else model.eval()), ocfg, w


def _rel(got, ref):
    err = got - ref
    return (err.abs().max().item() / (ref.abs().max().item() + 1e-12),
            (err.pow(2).mean().sqrt() / (ref.pow(2).mean().sqrt() + 1e-12)).item())


def _rel_l2(got, ref):
    return ((got.double() - ref.double()).norm() / (ref.double().norm() + 1e-30)).item()


# ---------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("hh,ww", [(4, 4), (20, 20), (64, 64)])
@pytest.mark.parametrize("s", [2, 5, 16, 37, 256])
@pytest.mark.parametrize("d", [16, 32, 64])
def test_xattn_forward_backward_matches_autograd(cuda, d, s, hh, ww):
    """b200ad_xattn_forward_backward (8 heads of dim d, H*W queries against s keys) against CPU fp32 autograd of
    oracle.unet_cond_oracle._mha: O, dQ, dK, dV each within 2 % relative L2."""
    from audio_diffusion_b200 import _lib
    from oracle.unet_cond_oracle import _mha
    heads, n = 8, 2
    c = heads * d
    g = torch.Generator().manual_seed(d * 100000 + s * 100 + hh)
    q, do = (torch.randn(n, c, hh, ww, generator=g) for _ in range(2))
    k, v = (torch.randn(n, s, c, generator=g) for _ in range(2))
    tok = lambda a: a.flatten(2).transpose(1, 2)                  # [N, C, H, W] -> (N, seq, C)
    ql, kl, vl = q.clone().requires_grad_(True), k.clone().requires_grad_(True), v.clone().requires_grad_(True)
    o_ref = _mha(tok(ql), kl, vl, heads)
    o_ref.backward(tok(do))
    L = _lib.lib()
    qd, kd, vd, dod = (a.to(cuda).contiguous() for a in (q, k, v, do))
    out, dq = torch.empty_like(qd), torch.empty_like(qd)
    dk, dv = torch.empty_like(kd), torch.empty_like(vd)
    nb = L.b200ad_xattn_scratch_bytes(n, c, heads, hh, ww, s)
    scratch = torch.empty(nb, dtype=torch.uint8, device=cuda)
    _lib.check(L.b200ad_xattn_forward_backward(qd.data_ptr(), kd.data_ptr(), vd.data_ptr(), dod.data_ptr(), out.data_ptr(),
                                               dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), n, c, heads, hh, ww, s,
                                               scratch.data_ptr(), nb, _lib.stream_ptr()))
    torch.cuda.synchronize()
    errs = {"O": _rel_l2(tok(out.cpu()), o_ref.detach()), "dQ": _rel_l2(dq.cpu(), ql.grad),
            "dK": _rel_l2(dk.cpu(), kl.grad), "dV": _rel_l2(dv.cpu(), vl.grad)}
    print(d, s, hh, ww, errs)
    assert all(e <= 2e-2 for e in errs.values()), errs


# ---------------------------------------------------------------------------------------------------- forward
@pytest.mark.parametrize("s", [2, 37])
@pytest.mark.parametrize("size", [(32, 32), (64, 64)])
def test_cond_seq_layers_and_eps(cuda, monkeypatch, size, s):
    """The reference architecture with an (2, s, 100) encoding: per-layer taps (attn1 = h1, attn2 = h2 of a transformer
    block) and epsilon against unet_cond_forward, with test_gpu_cond.py's bars."""
    from oracle.unet_cond_oracle import unet_cond_forward
    monkeypatch.setenv("B200AD_DEBUG_NOPOOL", "1")
    model, ocfg, w = _build(cuda, size, seed=s)
    g = torch.Generator().manual_seed(42 + s)
    x = torch.randn(2, 1, *size, generator=g)
    enc = torch.randn(2, s, 100, generator=g)
    t = torch.tensor([17, 801])
    taps = {}
    with torch.no_grad():
        ref = unet_cond_forward(w, ocfg, x, t, enc, taps)
        out = model(x.to(cuda), t.to(cuda), enc.to(cuda))["sample"]
    torch.cuda.synchronize()
    names = ["down_blocks.0.attentions.0.attn1", "down_blocks.0.attentions.0.attn2", "down_blocks.0.attentions.0",
             "down_blocks.1.attentions.1.attn1", "down_blocks.1.attentions.1.attn2", "down_blocks.2.attentions.0.attn2",
             "down_blocks.2.attentions.1", "mid_block.attentions.0.attn1", "mid_block.attentions.0",
             "up_blocks.1.attentions.0.attn2", "up_blocks.1.attentions.2", "up_blocks.2.attentions.2.attn1",
             "up_blocks.3.attentions.0.attn2", "up_blocks.3.attentions.2"]
    worst = (0.0, 0.0)
    for name in names:
        mx, rms = _rel(model.debug_tensor(name).cpu(), taps[name])
        print("%-44s max-rel %.4f rms-rel %.4f" % (name, mx, rms))
        worst = (max(worst[0], mx), max(worst[1], rms))
    mx, rms = _rel(out.cpu(), ref)
    print("eps max-rel %.4f rms-rel %.4f | worst layer %.4f / %.4f" % (mx, rms, worst[0], worst[1]))
    assert worst[0] <= 6e-2 and worst[1] <= 2.5e-2
    assert mx <= 6e-2 and rms <= 1.5e-2


def test_one_token_path_unchanged_after_longer_encoding(cuda):
    """S = 1 keeps its own plan: after a model has run with S = 2, its S = 1 output equals a fresh model's bit for bit, and
    the S = 1 launch count is the fresh model's."""
    a, _, _ = _build(cuda, (32, 32), seed=7)
    b, _, _ = _build(cuda, (32, 32), seed=7)
    g = torch.Generator().manual_seed(8)
    x = torch.randn(2, 1, 32, 32, generator=g).to(cuda)
    e2 = torch.randn(2, 2, 100, generator=g).to(cuda)
    e1 = e2[:, :1].contiguous()
    with torch.no_grad():
        a(x, 300, e2)
        got = a(x, 300, e1)["sample"]
        n_a = a.last_launch_count
        ref = b(x, 300, e1)["sample"]
    assert torch.equal(got, ref)
    assert n_a == b.last_launch_count


def test_identical_tokens_match_one_token(cuda):
    """Two identical tokens attend exactly like one (softmax splits evenly over equal keys): the S = 2 path (K / V
    projections, cross-attention kernel) and the S = 1 path (per-sample vector) differ only by bf16 rounding."""
    model, _, _ = _build(cuda, (32, 32), seed=9)
    g = torch.Generator().manual_seed(10)
    x = torch.randn(2, 1, 32, 32, generator=g).to(cuda)
    e1 = torch.randn(2, 1, 100, generator=g).to(cuda)
    with torch.no_grad():
        one = model(x, 420, e1)["sample"]
        two = model(x, 420, e1.repeat(1, 2, 1))["sample"]
    mx, rms = _rel(two.cpu(), one.cpu())
    print(f"identical tokens: max-rel {mx:.4f} rms-rel {rms:.4f}")
    assert mx <= 6e-2 and rms <= 1.5e-2


@pytest.mark.parametrize("s", [5])
def test_cond_seq_pipeline_matches_oracle_loop(cuda, s):
    """`pipe(batch_size=2, steps=6, encoding=(2, s, 100))` (fused scheduler step) against the oracle DDPM loop: at least
    90 % of the pixels within 2 grey levels, as for one token."""
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
    enc = torch.randn(2, s, 100, generator=g)
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
    print(f"conditional pipeline, {s} tokens: mean |d| {d.mean():.3f}, within 2: {(d <= 2).mean():.3f}, max {d.max()}")
    assert (d <= 2).mean() >= 0.90


# ---------------------------------------------------------------------------------------------------- training
def cond_loss_and_grads(w, cfg, clean, noise, t, enc):
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_cond_oracle import unet_cond_forward
    noisy = OracleDDPM().add_noise(clean, noise, t)
    wl = {k: v.detach().clone().requires_grad_(True) for k, v in w.items()}
    pred = unet_cond_forward(wl, cfg, noisy, t, enc)
    loss = torch.mean((pred - noise) ** 2)
    grads = torch.autograd.grad(loss, list(wl.values()))
    return loss.detach(), dict(zip(wl.keys(), grads))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("s", [2, 77])
@pytest.mark.parametrize("arch,size", [("full", (32, 32)), ("small", (64, 64))])
def test_cond_seq_backward_matches_autograd(cuda, arch, size, s):
    """Every parameter gradient of one conditional training loss, batch 2, against autograd over the oracle: loss within
    2 %, concatenated gradient within 3 % relative L2, every tensor with a non-negligible gradient within 10 %.  The
    parameters that get exactly zero gradients with one token (attn2.to_q, attn2.to_k, norm2) are non-zero and inside
    those bars."""
    from oracle.schedulers_oracle import OracleDDPM
    model, ocfg, w = _build(cuda, size, seed=20 + s, arch=ARCH if arch == "full" else SMALL, train=True)
    g = torch.Generator().manual_seed(s)
    clean = torch.rand(2, 1, *size, generator=g) * 2 - 1
    noise = torch.randn(2, 1, *size, generator=g)
    enc = torch.randn(2, s, 100, generator=g)
    t = torch.tensor([37, 712])
    loss_ref, grads_ref = cond_loss_and_grads(w, ocfg, clean, noise, t, enc)
    noisy = OracleDDPM().add_noise(clean, noise, t).to(cuda)
    pred = model(noisy, t.to(cuda), enc.to(cuda))["sample"]
    loss = torch.nn.functional.mse_loss(pred, noise.to(cuda))
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - loss_ref.item()) <= 2e-2 * loss_ref.item(), (loss.item(), loss_ref.item())
    rows, num, den = [], 0.0, 0.0
    for k, p in model.named_parameters():
        gd, r = p.grad.detach().cpu().double(), grads_ref[k].double()
        e, sn = (gd - r).norm().item(), r.norm().item()
        rows.append((e / (sn + 1e-30), k, sn, gd.norm().item()))
        num += e * e
        den += sn * sn
    rows.sort(reverse=True)
    total = (num / den) ** 0.5
    for e, k, sn, gn in rows[:15]:
        print(f"{e:9.4f}  |ref| {sn:10.3e}  |got| {gn:10.3e}  {k}")
    print("total relative L2 error", total, "backward launches", model.last_backward_launch_count)
    gmax = max(r[2] for r in rows)
    bad = [(e, k) for e, k, sn, _ in rows if e > 0.10 and sn > 1e-3 * gmax]
    assert total <= 3e-2 and not bad, (total, bad[:10])
    by = {k: (e, sn, gn) for e, k, sn, gn in rows}
    named = [k for k in by if any(k.endswith(".transformer_blocks.0." + z) for z in ONE_TOKEN_ZERO)]
    assert named
    for k in named:
        e, sn, gn = by[k]
        assert gn > 0 and sn > 0, k
        assert e <= 0.10 or sn <= 1e-3 * gmax, (k, e)


@pytest.mark.parametrize("d,s,hh", [(16, 77, 64), (64, 256, 20), (32, 5, 64)])
def test_xattn_backward_deterministic(cuda, d, s, hh):
    """Two runs of the cross-attention forward and backward on the same inputs give bit-identical O, dQ, dK and dV: no float
    atomics, the per-split dK / dV partials are added in a fixed order (64 x 64 queries against 77 keys: several splits).
    (The model's flat gradient as a whole is not bitwise reproducible: the GroupNorm / LayerNorm / bias reductions and
    the split-K weight gradients of the rest of the backward accumulate with atomics.)"""
    from audio_diffusion_b200 import _lib
    heads, n = 8, 2
    c = heads * d
    g = torch.Generator().manual_seed(s)
    q, do = (torch.randn(n, c, hh, hh, generator=g).to(cuda) for _ in range(2))
    k, v = (torch.randn(n, s, c, generator=g).to(cuda) for _ in range(2))
    L = _lib.lib()
    nb = L.b200ad_xattn_scratch_bytes(n, c, heads, hh, hh, s)
    scratch = torch.empty(nb, dtype=torch.uint8, device=cuda)
    runs = []
    for _ in range(2):
        out, dq, dk, dv = torch.empty_like(q), torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        _lib.check(L.b200ad_xattn_forward_backward(q.data_ptr(), k.data_ptr(), v.data_ptr(), do.data_ptr(), out.data_ptr(),
                                                   dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), n, c, heads, hh, hh, s,
                                                   scratch.data_ptr(), nb, _lib.stream_ptr()))
        runs.append((out, dq, dk, dv))
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(*runs))


def test_cond_seq_gradient_accumulation_equals_full_batch(cuda):
    """Two half-batches (loss / 2 each, the first under no_sync) give the full batch's gradient, with 9 tokens."""
    model, _, _ = _build(cuda, (32, 32), seed=3, train=True)
    g = torch.Generator().manual_seed(6)
    x = torch.randn(2, 1, 32, 32, generator=g).to(cuda)
    tgt = torch.randn(2, 1, 32, 32, generator=g).to(cuda)
    enc = torch.randn(2, 9, 100, generator=g).to(cuda)
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


def test_cond_seq_two_training_steps_match_oracle(cuda):
    """training.train_step(..., encoder_hidden_states=(2, 6, 100)) with FusedAdamW, EMA and cosine LR, twice, against the
    oracle step on the two-level model, with the bars of test_cond_two_training_steps_match_oracle."""
    import os
    import sys
    from audio_diffusion_b200.schedulers import DDPMScheduler
    from audio_diffusion_b200.training import EMAModel, FusedAdamW, train_step
    from oracle.train_oracle import TrainState, adamw_update, clip_grad_norm, cosine_with_warmup, ema_decay
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "audio_diffusion_b200", "compat"))
    try:
        from diffusers.optimization import get_scheduler
    finally:
        sys.path.pop(0)
    model, ocfg, w = _build(cuda, (32, 32), seed=4, arch=SMALL, train=True)
    w0 = {k: v.clone() for k, v in w.items()}
    opt = FusedAdamW(model.parameters(), lr=1e-4, betas=(0.95, 0.999), weight_decay=1e-6, eps=1e-8, max_grad_norm=1.0)
    ema = EMAModel(model.parameters(), inv_gamma=1.0, power=0.75, max_value=0.9999)
    opt.attach_ema(ema)
    lrs = get_scheduler("cosine", optimizer=opt, num_warmup_steps=1, num_training_steps=10)
    sch = DDPMScheduler()
    st = TrainState()
    st.ema = {k: v.detach().clone() for k, v in w.items()}
    g = torch.Generator().manual_seed(5)
    for it in range(2):
        clean = torch.rand(2, 1, 32, 32, generator=g) * 2 - 1
        noise = torch.randn(2, 1, 32, 32, generator=g)
        enc = torch.randn(2, 6, 100, generator=g)
        t = torch.randint(0, 1000, (2,), generator=g)
        loss_ref, grads = cond_loss_and_grads(w, ocfg, clean, noise, t, enc)
        grads, gnorm_ref = clip_grad_norm(grads, 1.0)
        lr_ref = 1e-4 * cosine_with_warmup(st.step, 1, 10)
        st.step += 1
        for k in w:
            if k not in st.exp_avg:
                st.exp_avg[k] = torch.zeros_like(w[k])
                st.exp_avg_sq[k] = torch.zeros_like(w[k])
            adamw_update(w[k], grads[k], st.exp_avg[k], st.exp_avg_sq[k], st.step, lr_ref)
        decay_ref = ema_decay(st.step)
        for k in w:
            st.ema[k].sub_((1.0 - decay_ref) * (st.ema[k] - w[k]))
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


# ---------------------------------------------------------------------------------------------------- per block
# The two-level UNet2DConditionModel of the per-block tests (transformers at 32x32 in the down and the up block, 16x16 in
# the mid block), batch 3, against fp64 on the engine's own activations (oracle/block_grads.py) with the bars of
# tests/test_gpu_block_forward.py / tests/test_gpu_block_backward.py: 3 x the bf16 floor of each block kind, measured at
# these shapes, seeds and token counts; each test recomputes the floors and asserts every bar within (floor, 3.3 x floor].
# S -> key -> (a, b, c): 3 x the bf16 floor of tests/test_gpu_block_forward.py's _floors at this test's shapes and seeds
COND_SEQ_FWD_BARS = {
    3: {
        "down": (0.00681, 0.00885, 0.00696),   # floor (0.00227, 0.00295, 0.00232)
        "head": (0.00498, 0.00708, 0.00468),   # floor (0.00166, 0.00236, 0.00156)
        "resnet": (0.01209, 0.01737, 0.01251),   # floor (0.00403, 0.00579, 0.00417)
        "resnet.h1": (0.01017, 0.01794, 0.01089),   # floor (0.00339, 0.00598, 0.00363)
        "resnet.h1:mean": (0.01152, 0.01152, 0.01152),   # floor (0.00384, 0.00384, 0.00384)
        "resnet.out": (0.00975, 0.01794, 0.01014),   # floor (0.00325, 0.00598, 0.00338)
        "tail": (0.00819, 0.01197, 0.00819),   # floor (0.00273, 0.00399, 0.00273)
        "transformer": (0.00996, 0.01449, 0.01125),   # floor (0.00332, 0.00483, 0.00375)
        "transformer.attn2": (0.01089, 0.01644, 0.0126),   # floor (0.00363, 0.00548, 0.0042)
        "transformer.out": (0.00795, 0.0129, 0.00822),   # floor (0.00265, 0.0043, 0.00274)
        "up": (0.00729, 0.0102, 0.00786),   # floor (0.00243, 0.0034, 0.00262)
    },
    77: {
        "down": (0.00678, 0.00948, 0.00687),   # floor (0.00226, 0.00316, 0.00229)
        "head": (0.00498, 0.00708, 0.00468),   # floor (0.00166, 0.00236, 0.00156)
        "resnet": (0.01215, 0.01743, 0.01242),   # floor (0.00405, 0.00581, 0.00414)
        "resnet.h1": (0.01017, 0.01794, 0.01077),   # floor (0.00339, 0.00598, 0.00359)
        "resnet.h1:mean": (0.01311, 0.01311, 0.01311),   # floor (0.00437, 0.00437, 0.00437)
        "resnet.out": (0.00975, 0.01692, 0.01014),   # floor (0.00325, 0.00564, 0.00338)
        "tail": (0.00813, 0.0108, 0.00813),   # floor (0.00271, 0.0036, 0.00271)
        "transformer": (0.00966, 0.01242, 0.01008),   # floor (0.00322, 0.00414, 0.00336)
        "transformer.attn2": (0.01044, 0.01695, 0.01161),   # floor (0.00348, 0.00565, 0.00387)
        "transformer.out": (0.00789, 0.01197, 0.00807),   # floor (0.00263, 0.00399, 0.00269)
        "up": (0.00732, 0.01071, 0.00762),   # floor (0.00244, 0.00357, 0.00254)
    },
}
# S -> the transformer's (activation a, b, c), (parameter a, b, c): 3 x the bf16 floor (at least 0.5 %)
COND_SEQ_BWD_TRANSFORMER_BARS = {
    3: ((0.009, 0.0147, 0.0096), (0.0225, 0.0282, 0.0855)),   # floor (0.003, 0.0049, 0.0032) | (0.0075, 0.0094, 0.0285)
    77: ((0.009, 0.0111, 0.0093), (0.0216, 0.0204, 0.0948)),   # floor (0.003, 0.0037, 0.0031) | (0.0072, 0.0068, 0.0316)
}


@pytest.mark.timeout(600)
@pytest.mark.parametrize("s", [3, 77])
def test_cond_seq_forward_per_block(cuda, monkeypatch, s):
    """Every block, and every transformer's h2 (.attn2, after the LN2 / to_q / K-V / cross-attention / to_out steps), of
    the eval forward with an (3, s, 100) encoding, from the engine's own inputs."""
    import time
    from audio_diffusion_b200.unet_cond import UNet2DConditionModel
    from oracle import block_grads as bg
    from oracle.unet_cond_oracle import CondUNetConfig, init_weights, unet_cond_forward
    from test_gpu_block_backward import COND_ARCH, _w64
    from test_gpu_block_forward import _floors, check_against_floors, forward_checks
    monkeypatch.setenv("B200AD_DEBUG_NOPOOL", "1")
    cfg = CondUNetConfig(sample_size=(32, 32), **{k: COND_ARCH[k] for k in ("block_out_channels", "down_block_types",
                                                                              "up_block_types")})
    w = init_weights(cfg, seed=17)
    model = UNet2DConditionModel(sample_size=(32, 32), **COND_ARCH)
    model.load_state_dict(w)
    model = model.to(cuda).eval()
    g = torch.Generator().manual_seed(18)
    x = torch.randn(3, 1, 32, 32, generator=g).to(cuda)
    enc = torch.randn(3, s, 100, generator=g).to(cuda)
    t = torch.tensor([37, 412, 903], device=cuda)
    with torch.no_grad():
        eps = model(x, t, enc)["sample"]
    w64 = _w64(w, cuda)
    blocks = bg.unet_blocks(cfg)
    t0 = time.perf_counter()
    temb = bg.temb_act(w64, cfg, t)
    e64 = enc.double()
    rows = forward_checks(model.debug_tensor, blocks, x.double(), eps, w64, cfg, temb, e64)
    otaps = {}
    with torch.no_grad():
        unet_cond_forward(w64, cfg, x.double(), t, e64, otaps)
    floors = _floors(blocks, otaps, x.double(), w64, cfg, temb, e64)
    check_against_floors(f"UNet2DConditionModel 32x32 batch 3, {s} tokens", rows, floors, COND_SEQ_FWD_BARS[s], t0)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("s", [3, 77])
def test_cond_seq_backward_per_block(cuda, s):
    """After one training forward and backward with an (3, s, 100) encoding: every block's input gradient(s) and parameter
    gradients against fp64 autograd of that block from the engine's own input activations and output gradient.  The
    transformers' walk covers attn2.to_out, the cross-attention backward (dQ, the split dK / dV partial sums), the K / V
    weight gradients, to_q, LN2 with its residual and the two to_out biases; attn2.to_q, attn2.to_k and norm2 get non-zero
    gradients inside the bars.  The other block kinds keep test_gpu_block_backward.py's COND_BARS."""
    from audio_diffusion_b200.unet_cond import UNet2DConditionModel
    from oracle import block_grads as bg
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_cond_oracle import CondUNetConfig, init_weights, unet_cond_forward
    from test_cpu_block_backward import _floors
    from test_gpu_block_backward import COND_ARCH, COND_BARS, T3, _run_checks, _w64
    cfg = CondUNetConfig(sample_size=(32, 32), block_out_channels=COND_ARCH["block_out_channels"],
                         down_block_types=COND_ARCH["down_block_types"], up_block_types=COND_ARCH["up_block_types"])
    w = init_weights(cfg, seed=3)
    model = UNet2DConditionModel(sample_size=(32, 32), **COND_ARCH)
    model.load_state_dict(w)
    model = model.to(cuda).train()
    g = torch.Generator().manual_seed(4)
    clean = torch.rand(3, 1, 32, 32, generator=g) * 2 - 1
    noise = torch.randn(3, 1, 32, 32, generator=g)
    enc = torch.randn(3, s, 100, generator=g).to(cuda)
    t = torch.tensor(T3)
    noisy = OracleDDPM().add_noise(clean, noise, t).to(cuda)
    pred = model(noisy, t.to(cuda), enc)["sample"]
    noise = noise.to(cuda)
    torch.nn.functional.mse_loss(pred, noise).backward()
    g_eps = 2 * (pred.detach() - noise) / pred.numel()
    named = dict(model.named_parameters())
    once = [k for k in named if k.endswith(ONE_TOKEN_ZERO) and ".transformer_blocks." in k]
    assert len(once) == 6 * 4 and all(torch.count_nonzero(named[k].grad) > 0 for k in once)
    w64 = _w64(w, cuda)
    bars = dict(COND_BARS, transformer=COND_SEQ_BWD_TRANSFORMER_BARS[s])
    blocks = bg.unet_blocks(cfg)
    temb = bg.temb_act(w64, cfg, t.to(cuda))
    fails = _run_checks(model, blocks, noisy, g_eps, w64, cfg, bars, temb=temb, enc=enc)
    assert not fails, fails
    # the transformer bars against the floor at these inputs (oracle activations, fp64 on the device)
    taps = {}
    x64, n64, e64 = noisy.double(), noise.double(), enc.double()
    with torch.no_grad():
        ref = unet_cond_forward(w64, cfg, x64, t.to(cuda), e64, taps)
    fl = _floors(blocks, taps, x64, 2 * (ref - n64) / ref.numel(), w64, cfg, temb, e64)["transformer"]
    for f, b in zip(fl[0] + fl[1], bars["transformer"][0] + bars["transformer"][1]):
        assert f < b <= max(3.3 * round(f, 4), 5e-3) + 1e-9, (fl, bars["transformer"])


# ---------------------------------------------------------------------------------------------------- errors
def test_cond_seq_errors(cuda):
    """257 tokens: ValueError naming 256.  A raw set_encoding with a token count other than the planned one: the forward
    and the backward return an error status naming both counts; so does a backward whose plan predates a workspace
    re-planned for another count.  Training with an encoding that requires grad: refused."""
    from audio_diffusion_b200 import _lib
    model, _, _ = _build(cuda, (32, 32), seed=1)
    x = torch.randn(2, 1, 32, 32).to(cuda)
    t = torch.tensor([10, 500]).to(cuda)
    with pytest.raises(ValueError, match="256"):
        with torch.no_grad():
            model(x, t, torch.randn(2, 257, 100, device=cuda))
    e2 = torch.randn(2, 2, 100, device=cuda)
    e3 = torch.randn(2, 3, 100, device=cuda)
    with torch.no_grad():
        model(x, t, e2)                                            # planned for 2 tokens
    L = _lib.lib()
    out = torch.empty_like(x)
    tt = t.to(torch.float32)
    assert L.b200ad_unet_set_encoding(model._h, e3.data_ptr(), 3) == 0
    st = L.b200ad_unet_forward(model._h, x.data_ptr(), tt.data_ptr(), out.data_ptr(), _lib.stream_ptr())
    msg = L.b200ad_last_error().decode()
    assert st != 0 and "3" in msg and "2" in msg, msg
    assert L.b200ad_unet_set_encoder_len(model._h, 257) != 0
    assert L.b200ad_unet_set_encoder_len(model._h, 0) != 0
    torch.cuda.synchronize()
    with torch.no_grad():
        assert torch.isfinite(model(x, t, e2)["sample"]).all()    # the handle is still usable
    tm, _, _ = _build(cuda, (32, 32), seed=1, train=True)
    tm(x, t, e2)["sample"].sum().backward()
    assert tm._fn("set_encoding")(tm._h, e3.data_ptr(), 3) == 0
    g = torch.ones_like(x)
    st = tm._fn("backward")(tm._h, x.data_ptr(), g.data_ptr(), 0, _lib.stream_ptr())
    msg = L.b200ad_last_error().decode()
    assert st != 0 and "3" in msg and "2" in msg, msg
    # a workspace re-planned for 3 tokens without a new backward plan: the backward refuses, naming both counts
    assert tm._fn("set_encoder_len")(tm._h, 3) == 0
    need = tm._fn("workspace_bytes")(tm._h, 2, 32, 32)
    ws = torch.empty(need, dtype=torch.uint8, device=cuda)
    _lib.check(tm._fn("bind_workspace")(tm._h, ws.data_ptr(), need, 2, 32, 32, _lib.stream_ptr()))
    st = tm._fn("backward")(tm._h, x.data_ptr(), g.data_ptr(), 0, _lib.stream_ptr())
    msg = L.b200ad_last_error().decode()
    assert st != 0 and "3" in msg and "2" in msg, msg
    torch.cuda.synchronize()
    tm._ws_key = None                                          # the Python side re-binds what it owns
    with pytest.raises(NotImplementedError):
        tm(x, t, torch.randn(2, 2, 100, device=cuda, requires_grad=True))
