"""CPU checks of oracle/block_grads.py, the per-block references of tests/test_gpu_block_backward.py.

* Composition: the block references chained in reverse over the oracle's own fp64 activations, from the gradient of the
  model's output, reproduce fp64 autograd through the whole model (U-Net, conditional U-Net, both autoencoder parts),
  the U-Net's timestep MLP included: the block lists, the skip bookkeeping and each block's decomposition are right
  before any GPU number is trusted.
* Coverage: the blocks and the timestep MLP claim every parameter exactly once.
* Floor (block_grads.backward_floors): each block kind's gradients with bf16 storage (bf16_storage()) against exact, at
  the GPU test's shapes, over the oracle's activations and upstream gradients rounded to bf16 as the engine stores
  them, and the timestep MLP's gradients from the resnets' rounded temb_act gradients.  These are the floors the GPU
  bars (tests/cases.py) are stated from.
"""
import pytest
import torch

from blockcheck import bar_in_range
from cases import (COND_BARS, LDM, PUBLISHED, PUBLISHED4, PUBLISHED_ATTN, PUBLISHED_COND, T3, TWO_LEVEL, TWO_LEVEL_COND,
                   UNET_BARS, VAE_BARS, draw, oracle_config)
from oracle import block_grads as bg


def _d(w):
    return {k: v.double() for k, v in w.items()}


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def _check_params(grads, ref, expect):
    assert set(grads) == set(expect), sorted(set(expect) ^ set(grads))[:10]
    scale = max(r.norm().item() for r in ref.values())
    worst = max(((g - ref[k]).norm().item() / max(ref[k].norm().item(), 1e-9 * scale), k) for k, g in grads.items())
    print("composition: worst parameter relative error", worst)
    assert worst[0] < 1e-9      # fp64 rounding; a wrong decomposition or skip share is off by O(1)


def _unet_case(size, n, seed, arch=TWO_LEVEL):
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_oracle import init_weights, unet_forward
    cfg = oracle_config(arch, size)
    w = _d(init_weights(cfg, seed=seed))
    clean, noise, _ = draw(n, size, seed, c=arch["in_channels"])
    clean, noise = clean.double(), noise.double()
    t = torch.tensor(T3[:n])
    noisy = OracleDDPM().add_noise(clean, noise, t)
    taps = {}
    pred = unet_forward(w, cfg, noisy, t, taps)
    return cfg, w, clean, noise, t, noisy, taps, 2 * (pred - noise) / pred.numel()


def test_unet_block_chain_reproduces_autograd():
    from oracle.train_oracle import loss_and_grads
    cfg, w, clean, noise, t, noisy, taps, g_eps = _unet_case((16, 16), 3, 2)
    _, ref, _ = loss_and_grads(w, cfg, clean, noise, t)
    blocks = bg.unet_blocks(cfg)
    assert any(b.skip and taps[b.inp].shape[1] + taps[b.skip].shape[1] == 384 for b in blocks)   # cpg 12 straddles
    _, grads, _ = bg.chain(blocks, taps, noisy, g_eps, w, cfg, taps["temb_act"], t=t)
    _check_params(grads, ref, list(w))


def _cond_chain(arch, size, n, transformers):
    """The conditional U-Net's block references chained over the oracle's activations against whole-model autograd."""
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_cond_oracle import init_weights, unet_cond_forward
    cfg = oracle_config(arch, size)
    w = _d(init_weights(cfg, seed=3))
    clean, noise, enc = (v.double() for v in draw(n, size, 3, 1))
    t = torch.tensor(T3[:n])
    noisy = OracleDDPM().add_noise(clean, noise, t)
    wl = {k: v.clone().requires_grad_(True) for k, v in w.items()}
    pred = unet_cond_forward(wl, cfg, noisy, t, enc)
    ref = dict(zip(wl, torch.autograd.grad(((pred - noise) ** 2).mean(), list(wl.values()), allow_unused=True)))
    taps = {}
    pred = unet_cond_forward(w, cfg, noisy, t, enc, taps)
    blocks = bg.unet_blocks(cfg)
    assert sum(b.kind == "transformer" for b in blocks) == transformers
    _, grads, _ = bg.chain(blocks, taps, noisy, 2 * (pred - noise) / pred.numel(), w, cfg, bg.temb_act(w, cfg, t), enc, t)
    for k in grads:      # attn2.to_q / to_k and norm2 do not reach the output: exactly zero
        if ref[k] is None:
            ref[k] = torch.zeros_like(w[k])
            assert torch.count_nonzero(grads[k]) == 0, k
    _check_params(grads, ref, list(w))


def test_cond_unet_block_chain_reproduces_autograd():
    _cond_chain(TWO_LEVEL_COND, (16, 16), 3, 6)


@pytest.mark.timeout(300)
def test_published_unet_block_chain_reproduces_autograd():
    """The six-level UNet2DModel the GPU tests train at 64x64 and 256x256: attention at down block 4 and up block 1, skip
    connections across six levels, at 64x64 so that the last level is 2x2."""
    from oracle.train_oracle import loss_and_grads
    cfg, w, clean, noise, t, noisy, taps, g_eps = _unet_case((64, 64), 2, 2, PUBLISHED)
    _, ref, _ = loss_and_grads(w, cfg, clean, noise, t)
    blocks = bg.unet_blocks(cfg)
    assert [b.name for b in blocks if b.kind == "attn"] == PUBLISHED_ATTN
    assert sum(b.skip is not None for b in blocks) == 6 * 3
    _, grads, _ = bg.chain(blocks, taps, noisy, g_eps, w, cfg, taps["temb_act"], t=t)
    _check_params(grads, ref, list(w))


# the attention parameters whose gradients are exactly zero over one token: the softmax over one key is 1 whatever the
# scores, so no gradient reaches q or k (to_k.bias never gets one: the softmax is invariant to it)
ONE_TOKEN_ATTN_ZERO = ("to_q.weight", "to_q.bias", "to_k.weight")


@pytest.mark.timeout(300)
@pytest.mark.parametrize("arch", [PUBLISHED, PUBLISHED4], ids=["1ch", "4ch"])
def test_published_unet_32_block_chain_reproduces_autograd(arch):
    """The six-level UNet2DModel at its 32x32 latent, with 1 and with 4 latent channels: the 1x1 bottom level (down block
    5, the mid block, up block 0), the stride-2 conv from 2x2 to 1x1 and the upsample from 1x1 to 2x2.  The mid block
    attends over one token, so its q and k gradients are exactly zero in fp64, in autograd and in the block chain; the
    2x2 attention blocks' are not."""
    from oracle.train_oracle import loss_and_grads
    cfg, w, clean, noise, t, noisy, taps, g_eps = _unet_case((32, 32), 2, 2, arch)
    _, ref, _ = loss_and_grads(w, cfg, clean, noise, t)
    blocks = bg.unet_blocks(cfg)
    assert [b.name for b in blocks if b.kind == "attn"] == PUBLISHED_ATTN
    assert taps["mid_block.attentions.0"].shape[2:] == (1, 1)
    _, grads, _ = bg.chain(blocks, taps, noisy, g_eps, w, cfg, taps["temb_act"], t=t)
    _check_params(grads, ref, list(w))
    for blk in PUBLISHED_ATTN:
        for k in ONE_TOKEN_ATTN_ZERO:
            zero = blk == "mid_block.attentions.0"
            for g in (ref[f"{blk}.{k}"], grads[f"{blk}.{k}"]):
                assert (torch.count_nonzero(g) == 0) == zero, (blk, k)


@pytest.mark.timeout(300)
def test_published_cond_unet_block_chain_reproduces_autograd():
    """The four-level UNet2DConditionModel the GPU tests train at 64x64 (transformers in three down and three up blocks
    and the mid block), at 32x32."""
    _cond_chain(PUBLISHED_COND, (32, 32), 2, 16)


def test_vae_block_chain_reproduces_autograd():
    from oracle import vae_oracle as vo
    cfg = vo.VAEConfig()
    w = _d(vo.init_weights(cfg, seed=5))
    g = torch.Generator().manual_seed(6)
    x = torch.randn(2, 1, 32, 32, generator=g).clamp(-1, 1).double()
    z = torch.randn(2, 1, 4, 4, generator=g).double()
    gx = torch.randn(2, 1, 32, 32, generator=g).double()
    gm = torch.randn(2, 2, 4, 4, generator=g).double()
    for part, inp, gout, fwd in (("decoder", z, gx, vo.decode), ("encoder", x, gm, vo.encode_moments)):
        wl = {k: v.clone().requires_grad_(True) for k, v in w.items()}
        xi = inp.clone().requires_grad_(True)
        (fwd(wl, cfg, xi) * gout).sum().backward()
        ref = {k: v.grad for k, v in wl.items() if v.grad is not None}
        taps = {}
        fwd(w, cfg, inp, taps)
        _, grads, g_in = bg.chain(bg.vae_blocks(cfg, part), taps, inp, gout, w, cfg)
        _check_params(grads, ref, list(ref))
        if part == "decoder":
            assert _rel(g_in, xi.grad) < 1e-10


def _claims(names, blocks, extra=()):
    """{parameter name: the blocks (or the timestep MLP, "temb") whose prefixes claim it}."""
    owners = [(b.name or b.kind, b.prefixes) for b in blocks] + [("temb", p) for p in extra]
    return {k: [o for o, pre in owners if k.startswith(pre)] for k in names}


@pytest.mark.parametrize("model", ["published", "train", "cond_small", "cond_published", "vae"])
def test_every_parameter_claimed_once(model):
    """Every parameter of the oracle's init_weights is claimed by exactly one block of the per-block references or by the
    timestep MLP (temb_backward): a parameter outside them would have no per-tensor fp64 check in the GPU per-block
    tests, as time_embedding.* had none before the MLP was checked.  The conditional U-Net's parameters and block list
    do not depend on the encoder's token count, so one case covers S = 1 and S > 1.  The autoencoder: encoder and
    decoder block lists together."""
    from oracle import unet_cond_oracle as uco
    from oracle import unet_oracle as uo
    from oracle import vae_oracle as vo
    if model == "vae":
        cfg = oracle_config(LDM)
        names = list(vo.init_weights(cfg, seed=0))
        claims = _claims(names, bg.vae_blocks(cfg, "encoder") + bg.vae_blocks(cfg, "decoder"))
    else:
        arch = {"published": PUBLISHED, "train": TWO_LEVEL, "cond_small": TWO_LEVEL_COND, "cond_published": PUBLISHED_COND}
        cfg = oracle_config(arch[model], (32, 32))
        names = list((uco if model.startswith("cond") else uo).init_weights(cfg, seed=0))
        claims = _claims(names, bg.unet_blocks(cfg), bg.TEMB_PREFIXES)
        assert len([k for k, o in claims.items() if o == ["temb"]]) == 4
    bad = {k: o for k, o in claims.items() if len(o) != 1}
    assert names and not bad, bad


def _assert_floors(fl, bars):
    """Every bar of the GPU test lies above the floor and at most at three times the floor, or at 0.5 %: the engine forms
    a block's bias gradients from fp32 sums of its output gradient before it stores that gradient in bf16, while the
    reference sums the stored bf16 values; that difference (0.1 - 0.3 % measured) is the floor of the gradients no bf16
    rounding reaches (downsample / upsample weights, the scalar-kernel heads and tails)."""
    for kind, (a, p) in fl.items():
        for f, b in zip(a + p, bars[kind][0] + bars[kind][1]):
            assert bar_in_range(f, b, 3, 4, 5e-3), (kind, a, p, bars[kind])   # floors as printed


@pytest.mark.timeout(600)
def test_unet_block_floors():
    cfg, w, clean, noise, t, noisy, taps, g_eps = _unet_case((32, 32), 3, 2)
    _assert_floors(bg.backward_floors(bg.unet_blocks(cfg), taps, noisy, g_eps, w, cfg, taps["temb_act"], t=t), UNET_BARS)


@pytest.mark.timeout(600)
def test_cond_unet_block_floors():
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_cond_oracle import init_weights, unet_cond_forward
    cfg = oracle_config(TWO_LEVEL_COND, (32, 32))
    w = _d(init_weights(cfg, seed=3))
    clean, noise, enc = (v.double() for v in draw(3, (32, 32), 3, 1))
    t = torch.tensor(T3)
    noisy = OracleDDPM().add_noise(clean, noise, t)
    taps = {}
    pred = unet_cond_forward(w, cfg, noisy, t, enc, taps)
    blocks = bg.unet_blocks(cfg)
    _assert_floors(bg.backward_floors(blocks, taps, noisy, 2 * (pred - noise) / pred.numel(), w, cfg,
                                      bg.temb_act(w, cfg, t), enc, t), COND_BARS)


@pytest.mark.timeout(900)
def test_vae_block_floors():
    from oracle import vae_oracle as vo
    cfg = vo.VAEConfig()
    w = _d(vo.init_weights(cfg, seed=0))
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 1, 64, 64, generator=g).clamp(-1, 1).double()
    z = torch.randn(2, 1, 8, 8, generator=g).double()
    gx = torch.randn(2, 1, 64, 64, generator=g).double()
    gm = torch.randn(2, 2, 8, 8, generator=g).double()
    fl = {}
    for part, inp, gout, fwd in (("decoder", z, gx, vo.decode), ("encoder", x, gm, vo.encode_moments)):
        taps = {}
        fwd(w, cfg, inp, taps)
        for k, v in bg.backward_floors(bg.vae_blocks(cfg, part), taps, inp, gout, w, cfg).items():
            fl[part + ":" + k] = v
    _assert_floors(fl, VAE_BARS)
