"""CPU checks of oracle/block_grads.py, the per-block references of tests/test_gpu_block_backward.py.

* Composition: the block references chained in reverse over the oracle's own fp64 activations, from the gradient of the
  model's output, reproduce fp64 autograd through the whole model (U-Net, conditional U-Net, both autoencoder parts):
  the block lists, the skip bookkeeping and each block's decomposition are right before any GPU number is trusted.
* Floor: each block kind's gradients with bf16 storage (bf16_storage()) against exact, at the GPU test's shapes, over the
  oracle's activations and upstream gradients rounded to bf16 as the engine stores them.  These are the floors the GPU
  bars are stated from.
"""
import pytest
import torch

from oracle import block_grads as bg

TRAIN_CFG = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256),
                 down_block_types=("DownBlock2D", "AttnDownBlock2D"), up_block_types=("AttnUpBlock2D", "UpBlock2D"))
COND_CFG = dict(block_out_channels=(128, 256), down_block_types=("CrossAttnDownBlock2D", "DownBlock2D"),
                up_block_types=("UpBlock2D", "CrossAttnUpBlock2D"))
T3 = torch.tensor([37, 412, 903])


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


def _unet_case(size, n, seed, arch=TRAIN_CFG):
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_oracle import UNetConfig, init_weights, unet_forward
    cfg = UNetConfig(sample_size=size, **arch)
    w = _d(init_weights(cfg, seed=seed))
    g = torch.Generator().manual_seed(seed + 1)
    clean = (torch.rand(n, 1, *size, generator=g) * 2 - 1).double()
    noise = torch.randn(n, 1, *size, generator=g).double()
    t = T3[:n]
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
    _, grads, _ = bg.chain(blocks, taps, noisy, g_eps, w, cfg, taps["temb_act"])
    _check_params(grads, ref, [k for k in w if not k.startswith("time_embedding.")])


def _cond_chain(cfg_kw, size, n, transformers):
    """The conditional U-Net's block references chained over the oracle's activations against whole-model autograd."""
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_cond_oracle import CondUNetConfig, init_weights, unet_cond_forward
    cfg = CondUNetConfig(sample_size=size, **cfg_kw)
    w = _d(init_weights(cfg, seed=3))
    g = torch.Generator().manual_seed(4)
    clean = (torch.rand(n, 1, *size, generator=g) * 2 - 1).double()
    noise = torch.randn(n, 1, *size, generator=g).double()
    enc = torch.randn(n, 1, 100, generator=g).double()
    t = T3[:n]
    noisy = OracleDDPM().add_noise(clean, noise, t)
    wl = {k: v.clone().requires_grad_(True) for k, v in w.items()}
    pred = unet_cond_forward(wl, cfg, noisy, t, enc)
    ref = dict(zip(wl, torch.autograd.grad(((pred - noise) ** 2).mean(), list(wl.values()), allow_unused=True)))
    taps = {}
    pred = unet_cond_forward(w, cfg, noisy, t, enc, taps)
    blocks = bg.unet_blocks(cfg)
    assert sum(b.kind == "transformer" for b in blocks) == transformers
    _, grads, _ = bg.chain(blocks, taps, noisy, 2 * (pred - noise) / pred.numel(), w, cfg, bg.temb_act(w, cfg, t), enc)
    for k in grads:      # attn2.to_q / to_k and norm2 do not reach the output: exactly zero
        if ref[k] is None:
            ref[k] = torch.zeros_like(w[k])
            assert torch.count_nonzero(grads[k]) == 0, k
    _check_params(grads, ref, [k for k in w if not k.startswith("time_embedding.")])


def test_cond_unet_block_chain_reproduces_autograd():
    _cond_chain(COND_CFG, (16, 16), 3, 6)


@pytest.mark.timeout(300)
def test_published_unet_block_chain_reproduces_autograd():
    """The six-level UNet2DModel the GPU tests train at 64x64 and 256x256: attention at down block 4 and up block 1, skip
    connections across six levels, at 64x64 so that the last level is 2x2."""
    from oracle.train_oracle import loss_and_grads
    from test_gpu_fullconfig import REF_ARCH
    cfg, w, clean, noise, t, noisy, taps, g_eps = _unet_case((64, 64), 2, 2, REF_ARCH)
    _, ref, _ = loss_and_grads(w, cfg, clean, noise, t)
    blocks = bg.unet_blocks(cfg)
    assert [b.name for b in blocks if b.kind == "attn"] == (
        ["down_blocks.4.attentions.0", "down_blocks.4.attentions.1", "mid_block.attentions.0"]
        + [f"up_blocks.1.attentions.{j}" for j in range(3)])
    assert sum(b.skip is not None for b in blocks) == 6 * 3
    _, grads, _ = bg.chain(blocks, taps, noisy, g_eps, w, cfg, taps["temb_act"])
    _check_params(grads, ref, [k for k in w if not k.startswith("time_embedding.")])


@pytest.mark.timeout(300)
def test_published_cond_unet_block_chain_reproduces_autograd():
    """The four-level UNet2DConditionModel the GPU tests train at 64x64 (transformers in three down and three up blocks
    and the mid block), at 32x32."""
    from test_gpu_cond_train import ARCH
    _cond_chain({k: ARCH[k] for k in ("block_out_channels", "down_block_types", "up_block_types")}, (32, 32), 2, 16)


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


def _floors(blocks, taps, model_in, g_out, w, cfg, temb=None, enc=None):
    """bf16 floor of every block (rounded storage against exact, over bf16 inputs and upstream gradients), worst per
    kind: {kind: (activation (a, b, c), parameter (a, b, c))}."""
    G, _, _ = bg.chain(blocks, taps, model_in, g_out, w, cfg, temb, enc)
    out = {}
    for blk in blocks:
        xs = [model_in if blk.inp is None else bg.bf16(taps[blk.inp])] + ([bg.bf16(taps[blk.skip])] if blk.skip else [])
        gout = g_out if blk.out is None else bg.bf16(G[blk.out])
        ei, ep = bg.block_backward(blk, w, xs, gout, cfg, temb, enc)
        ri, rp = bg.block_backward(blk, w, xs, gout, cfg, temb, enc, rounded=True)
        acts = {} if blk.inp is None else {"in": (ri[0], ei[0])}
        if blk.skip:
            acts["skip"] = (ri[1], ei[1])
        rows, _ = bg.compare_block(acts, {k: (rp[k], ep[k]) for k in ep})
        wa, wp = bg.worst(rows, True), bg.worst(rows, False)
        pa, pp = out.get(blk.kind, ((0.0,) * 3, (0.0,) * 3))
        out[blk.kind] = (tuple(map(max, pa, wa)), tuple(map(max, pp, wp)))
    for k, (a, p) in out.items():
        print(f"floor {k:12s} act L2 {a[0]:.4f} max {a[1]:.4f} row {a[2]:.4f} | param L2 {p[0]:.4f} max {p[1]:.4f} "
              f"row {p[2]:.4f}")
    return out


def _assert_floors(fl, bars):
    """Every bar of the GPU test lies above the floor and at most at three times the floor, or at 0.5 %: the engine forms
    a block's bias gradients from fp32 sums of its output gradient before it stores that gradient in bf16, while the
    reference sums the stored bf16 values; that difference (0.1 - 0.3 % measured) is the floor of the gradients no bf16
    rounding reaches (downsample / upsample weights, the scalar-kernel heads and tails)."""
    for kind, (a, p) in fl.items():
        for f, b in zip(a + p, bars[kind][0] + bars[kind][1]):
            assert f < b <= max(3 * round(f, 4), 5e-3) + 1e-9, (kind, a, p, bars[kind])   # floors as printed


@pytest.mark.timeout(600)
def test_unet_block_floors():
    from test_gpu_block_backward import UNET_BARS
    cfg, w, clean, noise, t, noisy, taps, g_eps = _unet_case((32, 32), 3, 2)
    _assert_floors(_floors(bg.unet_blocks(cfg), taps, noisy, g_eps, w, cfg, taps["temb_act"]), UNET_BARS)


@pytest.mark.timeout(600)
def test_cond_unet_block_floors():
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_cond_oracle import CondUNetConfig, init_weights, unet_cond_forward
    from test_gpu_block_backward import COND_BARS
    cfg = CondUNetConfig(sample_size=(32, 32), **COND_CFG)
    w = _d(init_weights(cfg, seed=3))
    g = torch.Generator().manual_seed(4)
    clean = (torch.rand(3, 1, 32, 32, generator=g) * 2 - 1).double()
    noise = torch.randn(3, 1, 32, 32, generator=g).double()
    enc = torch.randn(3, 1, 100, generator=g).double()
    noisy = OracleDDPM().add_noise(clean, noise, T3)
    taps = {}
    pred = unet_cond_forward(w, cfg, noisy, T3, enc, taps)
    blocks = bg.unet_blocks(cfg)
    _assert_floors(_floors(blocks, taps, noisy, 2 * (pred - noise) / pred.numel(), w, cfg, bg.temb_act(w, cfg, T3), enc),
                   COND_BARS)


@pytest.mark.timeout(900)
def test_vae_block_floors():
    from oracle import vae_oracle as vo
    from test_gpu_block_backward import VAE_BARS
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
        for k, v in _floors(bg.vae_blocks(cfg, part), taps, inp, gout, w, cfg).items():
            fl[part + ":" + k] = v
    _assert_floors(fl, VAE_BARS)
