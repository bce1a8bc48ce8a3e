"""The U-Net and autoencoder backward block by block: after one real training forward and backward through the public
models, every block's input gradient(s) and parameter gradients, read from the engine (`debug_grad`, `p.grad`), against
fp64 autograd of that one block (oracle/block_grads.py) recomputed from the engine's own stored input activations
(`debug_tensor`) and the engine's own gradient of the block's output.  Errors do not compound across blocks, so the bars
are about one block's bf16 floor, not the whole backward's.

Each tensor is compared three ways (block_grads.errors): (a) relative L2; (b) max |err| / max |ref|, which sees an error
confined to borders, pad columns or single pixels; (c) the worst relative L2 of one output channel (weight gradients) or
one (sample, channel group) (activation gradients), which sees an error in one channel group, channel view or sample.

Bars, per block kind, for activation gradients and parameter gradients, are at most 3x the bf16 floor that
tests/test_cpu_block_backward.py measures at these shapes and seeds (bf16 storage of every conv / linear operand, output
and gradient against exact), and no lower than 0.5 %: the engine forms bias gradients from fp32 sums of a block's output
gradient before it stores that gradient in bf16, while the reference sums the stored values (0.1 - 0.3 % measured), and
that is the floor of the gradients no bf16 rounding reaches.  The floors are in the comments as (a, b, c).  Parameters
whose exact gradient is zero (softmax-invariant key biases) are listed, not compared.
"""
import pytest
import torch

from oracle import block_grads as bg

pytestmark = pytest.mark.gpu

TRAIN_CFG = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256),
                 down_block_types=("DownBlock2D", "AttnDownBlock2D"), up_block_types=("AttnUpBlock2D", "UpBlock2D"))
COND_ARCH = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256),
                 down_block_types=("CrossAttnDownBlock2D", "DownBlock2D"),
                 up_block_types=("UpBlock2D", "CrossAttnUpBlock2D"), cross_attention_dim=100)
T3 = [37, 412, 903]           # three distinct timesteps: batch 3, so per-sample sums must pick the right (odd) sample

# kind -> ((activation a, b, c), (parameter a, b, c))
UNET_BARS = {
    "head": ((0.005, 0.005, 0.005), (0.005, 0.005, 0.005)),   # floor (0.0, 0.0, 0.0) | (0.0, 0.0, 0.0)
    "resnet": ((0.0126, 0.0213, 0.0126), (0.0105, 0.0114, 0.0948)),   # floor (0.0042, 0.0071, 0.0042) | (0.0035, 0.0038, 0.0316)
    "down": ((0.0069, 0.0072, 0.0066), (0.005, 0.005, 0.005)),   # floor (0.0023, 0.0024, 0.0022) | (0.0, 0.0, 0.0)
    "attn": ((0.005, 0.009, 0.005), (0.0123, 0.0153, 0.0906)),   # floor (0.0017, 0.003, 0.0017) | (0.0041, 0.0051, 0.0302)
    "up": ((0.0087, 0.0116, 0.0084), (0.005, 0.005, 0.005)),   # floor (0.0029, 0.0039, 0.0028) | (0.0, 0.0, 0.0)
    "tail": ((0.0072, 0.0134, 0.0069), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.0045, 0.0023) | (0.0002, 0.0003, 0.0002)
}
COND_BARS = {
    "head": ((0.005, 0.005, 0.005), (0.005, 0.005, 0.005)),   # floor (0.0, 0.0, 0.0) | (0.0, 0.0, 0.0)
    "resnet": ((0.0126, 0.0269, 0.0126), (0.0123, 0.0141, 0.0714)),   # floor (0.0042, 0.009, 0.0042) | (0.0041, 0.0047, 0.0238)
    "transformer": ((0.009, 0.0098, 0.0096), (0.0222, 0.0213, 0.1023)),   # floor (0.003, 0.0033, 0.0032) | (0.0074, 0.0071, 0.0341)
    "down": ((0.0069, 0.0096, 0.0066), (0.005, 0.005, 0.005)),   # floor (0.0023, 0.0032, 0.0022) | (0.0, 0.0, 0.0)
    "up": ((0.0087, 0.0114, 0.0084), (0.005, 0.005, 0.005)),   # floor (0.0029, 0.0038, 0.0028) | (0.0, 0.0, 0.0)
    "tail": ((0.0072, 0.0141, 0.0072), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.0047, 0.0024) | (0.0002, 0.0003, 0.0002)
}
VAE_BARS = {
    "decoder:dec_head": ((0.005, 0.005, 0.005), (0.005, 0.005, 0.005)),   # floor (0.0, 0.0, 0.0) | (0.0, 0.0, 0.0)
    "decoder:resnet_vae": ((0.0126, 0.0183, 0.0123), (0.0213, 0.0309, 0.0849)),   # floor (0.0042, 0.0061, 0.0041) | (0.0071, 0.0103, 0.0283)
    "decoder:attn1": ((0.005, 0.0087, 0.005), (0.0165, 0.0174, 0.144)),   # floor (0.0017, 0.0029, 0.0017) | (0.0055, 0.0058, 0.048)
    "decoder:up": ((0.009, 0.0123, 0.0087), (0.005, 0.005, 0.005)),   # floor (0.003, 0.0041, 0.0029) | (0.0, 0.0, 0.0)
    "decoder:tail": ((0.0069, 0.0087, 0.0066), (0.0054, 0.0081, 0.0054)),   # floor (0.0023, 0.0029, 0.0022) | (0.0018, 0.0027, 0.0018)
    "encoder:head": ((0.005, 0.005, 0.005), (0.005, 0.005, 0.005)),   # floor (0.0, 0.0, 0.0) | (0.0, 0.0, 0.0)
    "encoder:resnet_vae": ((0.0126, 0.0165, 0.0123), (0.0147, 0.0207, 0.0276)),   # floor (0.0042, 0.0055, 0.0041) | (0.0049, 0.0069, 0.0092)
    "encoder:down_asym": ((0.0072, 0.0098, 0.0069), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.0033, 0.0023) | (0.0, 0.0, 0.0)
    "encoder:attn1": ((0.005, 0.0087, 0.005), (0.0174, 0.0171, 0.0956)),   # floor (0.0017, 0.0029, 0.0017) | (0.0058, 0.0057, 0.0319)
    "encoder:enc_tail": ((0.0072, 0.0153, 0.0075), (0.0098, 0.0101, 0.0098)),   # floor (0.0024, 0.0051, 0.0025) | (0.0033, 0.0034, 0.0033)
}


def _run_checks(model, blocks, model_in, g_out, w, cfg, bars, prefix="", temb=None, enc=None, g_in=None):
    """Compares every block; prints one table row per block; returns the blocks over their bars."""
    named = dict(model.named_parameters())
    skip_taps = {b.skip for b in blocks if b.skip}
    fails, worst_kind = [], {}
    print(f"\n{'block':44s} {'kind':12s} {'act L2':>7s} {'max':>7s} {'row':>7s} | {'par L2':>7s} {'max':>7s} {'row':>7s}")
    for blk in reversed(blocks):
        xs = [model_in if blk.inp is None else model.debug_tensor(blk.inp)]
        if blk.skip:
            xs.append(model.debug_tensor(blk.skip))
        gout = g_out if blk.out is None else model.debug_grad(blk.out)
        gi, gp = bg.block_backward(blk, w, xs, gout, cfg, temb, enc)
        acts = {}
        if blk.inp is not None:
            ref = gi[0]
            if blk.inp in skip_taps:            # the skip connection's share, checked at the block that consumes it
                ref = ref + model.debug_grad(blk.inp, skip=True).double()
            acts[f"G({blk.inp})"] = (model.debug_grad(blk.inp), ref)
        elif g_in is not None:
            acts["g_z"] = (g_in, gi[0])
        if blk.skip:
            acts[f"skip G({blk.skip})"] = (model.debug_grad(blk.skip, skip=True), gi[1])
        rows, skipped = bg.compare_block(acts, {k: (named[k].grad, gp[k]) for k in gp})
        wa, wp = bg.worst(rows, True), bg.worst(rows, False)
        kind = prefix + blk.kind
        ba, bp = bars[kind]
        over = [r for r in rows if any(e > b for e, b in zip(r[2:], ba if r[1] else bp))]
        print(f"{blk.name or 'conv_out':44s} {kind:12s} {wa[0]:7.4f} {wa[1]:7.4f} {wa[2]:7.4f} | {wp[0]:7.4f} {wp[1]:7.4f} "
              f"{wp[2]:7.4f}{'  OVER' if over else ''}{'  (zero ref: ' + ', '.join(skipped) + ')' if skipped else ''}")
        for r in over:
            print(f"    {r[0]}: {r[2]:.4f} {r[3]:.4f} {r[4]:.4f}")
        if over:
            fails.append((blk.name, [(r[0], round(r[2], 4), round(r[3], 4), round(r[4], 4)) for r in over]))
        pa, pp = worst_kind.get(kind, ((0.0,) * 3, (0.0,) * 3))
        worst_kind[kind] = (tuple(map(max, pa, wa)), tuple(map(max, pp, wp)))
    print("worst per kind (activation a, b, c | parameter a, b, c) against the bars:")
    for kind, (a, p) in worst_kind.items():
        print(f"  {kind:20s} {a[0]:.4f} {a[1]:.4f} {a[2]:.4f} | {p[0]:.4f} {p[1]:.4f} {p[2]:.4f}   bars {bars[kind]}")
    return fails


def _w64(w, dev):
    return {k: v.to(device=dev, dtype=torch.float64) for k, v in w.items()}


@pytest.mark.parametrize("size", [(32, 32), (32, 64)])
def test_unet_backward_per_block(cuda, size):
    """UNet2DModel (128, 256; DownBlock2D, AttnDownBlock2D), batch 3: every resnet (with and without conv_shortcut, over
    cat(input, skip), including up_blocks.0.resnets.2 whose 256 + 128 = 384 channels put a GroupNorm group of 12
    channels across the two sources), every head_dim-8 attention, the downsampler, the folded upsampler, conv_in and the
    conv_norm_out + conv_out tail."""
    from audio_diffusion_b200.unet import UNet2DModel
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_oracle import UNetConfig, init_weights
    cfg = UNetConfig(sample_size=size, **TRAIN_CFG)
    w = init_weights(cfg, seed=2)
    model = UNet2DModel(sample_size=size, **TRAIN_CFG)
    model.load_state_dict(w)
    model = model.to(cuda).train()
    g = torch.Generator().manual_seed(3)
    clean = torch.rand(3, 1, *size, generator=g) * 2 - 1
    noise = torch.randn(3, 1, *size, generator=g)
    t = torch.tensor(T3)
    noisy = OracleDDPM().add_noise(clean, noise, t).to(cuda)
    pred = model(noisy, t.to(cuda))["sample"]
    noise = noise.to(cuda)
    torch.nn.functional.mse_loss(pred, noise).backward()
    g_eps = 2 * (pred.detach() - noise) / pred.numel()
    w64 = _w64(w, cuda)
    blocks = bg.unet_blocks(cfg)
    fails = _run_checks(model, blocks, noisy, g_eps, w64, cfg, UNET_BARS, temb=bg.temb_act(w64, cfg, t.to(cuda)))
    assert not fails, fails


def test_cond_unet_backward_per_block(cuda):
    """UNet2DConditionModel (transformer blocks at 32x32 in the down and the up block, 16x16 in the mid block), batch 3:
    every block as above, the transformers included; attn2.to_q, attn2.to_k and norm2 get exactly zero gradients."""
    from audio_diffusion_b200.unet_cond import UNet2DConditionModel
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_cond_oracle import CondUNetConfig, init_weights
    cfg = CondUNetConfig(sample_size=(32, 32), block_out_channels=COND_ARCH["block_out_channels"],
                         down_block_types=COND_ARCH["down_block_types"], up_block_types=COND_ARCH["up_block_types"])
    w = init_weights(cfg, seed=3)
    model = UNet2DConditionModel(sample_size=(32, 32), **COND_ARCH)
    model.load_state_dict(w)
    model = model.to(cuda).train()
    g = torch.Generator().manual_seed(4)
    clean = torch.rand(3, 1, 32, 32, generator=g) * 2 - 1
    noise = torch.randn(3, 1, 32, 32, generator=g)
    enc = torch.randn(3, 1, 100, generator=g).to(cuda)
    t = torch.tensor(T3)
    noisy = OracleDDPM().add_noise(clean, noise, t).to(cuda)
    pred = model(noisy, t.to(cuda), enc)["sample"]
    noise = noise.to(cuda)
    torch.nn.functional.mse_loss(pred, noise).backward()
    g_eps = 2 * (pred.detach() - noise) / pred.numel()
    named = dict(model.named_parameters())
    zero = [k for k in named if k.endswith(("attn2.to_q.weight", "attn2.to_k.weight", "norm2.weight", "norm2.bias"))
            and ".transformer_blocks." in k]
    assert len(zero) == 6 * 4 and all(torch.count_nonzero(named[k].grad) == 0 for k in zero)
    w64 = _w64(w, cuda)
    fails = _run_checks(model, bg.unet_blocks(cfg), noisy, g_eps, w64, cfg, COND_BARS,
                        temb=bg.temb_act(w64, cfg, t.to(cuda)), enc=enc)
    assert not fails, fails


def test_vae_backward_per_block(cuda):
    """AutoencoderKL (ldm: 128, 256, 512, 512; 2 resnets per block) at 64x64, batch 2 (an 8x8 = 64-token latent):
    decoder backward from a seeded image gradient and encoder backward from seeded moment gradients.  Every resnet, the
    single-head attentions, the (0, 1, 0, 1)-padded downsamplers, the folded upsamplers, the encoder tail (conv_norm_out
    + conv_out + quant_conv, from g_moments), the decoder head (post_quant_conv + conv_in, to g_z) and the conv_out tail."""
    from audio_diffusion_b200.vae import AutoencoderKL
    from oracle import vae_oracle as vo
    cfg = vo.VAEConfig()
    w = vo.init_weights(cfg, seed=0)
    nb = len(cfg.block_out_channels)
    model = AutoencoderKL(in_channels=1, out_channels=1, down_block_types=("DownEncoderBlock2D",) * nb,
                          up_block_types=("UpDecoderBlock2D",) * nb, block_out_channels=cfg.block_out_channels,
                          layers_per_block=cfg.layers_per_block, latent_channels=1, max_batch=2)
    model.load_state_dict(w)
    model = model.to(cuda).train()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 1, 64, 64, generator=g).clamp(-1, 1).to(cuda)
    z = torch.randn(2, 1, 8, 8, generator=g).to(cuda)
    gx = torch.randn(2, 1, 64, 64, generator=g).to(cuda)
    gm = torch.randn(2, 2, 8, 8, generator=g).to(cuda)
    model.encode(x).latent_dist.parameters.backward(gm)
    zz = z.clone().requires_grad_(True)
    model.decode(zz).sample.backward(gx)
    w64 = _w64(w, cuda)
    fails = _run_checks(model, bg.vae_blocks(cfg, "decoder"), z, gx, w64, cfg, VAE_BARS, "decoder:", g_in=zz.grad)
    fails += _run_checks(model, bg.vae_blocks(cfg, "encoder"), x, gm, w64, cfg, VAE_BARS, "encoder:")
    assert not fails, fails
