"""CPU checks of the forward references in oracle/block_grads.py, the per-block references of
tests/test_gpu_block_forward.py.

* Composition: the block lists run forward from the model's input through `block_forward`, each block reading the outputs
  of the blocks before it (skip connections included), reproduce every oracle tap and the model output to 1e-12; inside
  every block, the sub-block steps of `sub_forward` chained over their own values reproduce the block's output and the
  oracle's sub-taps (a resnet's `.h1`, a transformer's `.attn2`) to 1e-12.  The block lists, the skip order and the
  sub-block splits restate the model before any GPU number is trusted (the backward twin: test_cpu_block_backward.py).
* The forward rounding model: which attention cores round their probabilities, and that the rounded references stay
  within a bf16 floor of the exact ones while differing from them.
"""
import pytest
import torch

from oracle import block_grads as bg

T3 = torch.tensor([37, 412, 903])


def _d(w):
    return {k: v.double() for k, v in w.items()}


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max()).item()


def _chain(blocks, model_in, w, cfg, taps, model_out, temb=None, enc=None):
    """block_forward over the block list from the model's input; every block's output against the oracle's tap, every
    block's sub-block chain against its output and the oracle's sub-taps."""
    acts, out, worst = {}, None, 0.0
    for blk in blocks:
        xs = [model_in if blk.inp is None else acts[blk.inp]] + ([acts[blk.skip]] if blk.skip else [])
        y = bg.block_forward(blk, w, xs, cfg, temb, enc)
        subs = bg.sub_forward(blk, w, xs, cfg, temb, enc, taps="all")
        worst = max(worst, _rel(subs["out"], y))
        for k, v in subs.items():
            if k != "out" and blk.name + k in taps:
                worst = max(worst, _rel(v, taps[blk.name + k]))
        if blk.out is None:
            out = y
        else:
            worst = max(worst, _rel(y, taps[blk.out]))
            acts[blk.out] = y
    worst = max(worst, _rel(out, model_out))
    print("composition: worst max-relative difference", worst)
    assert worst < 1e-12
    return acts


@pytest.mark.timeout(300)
def test_published_unet_block_forward_chain():
    """The six-level UNet2DModel at 64x64 (the last level 2x2), per-sample timesteps."""
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_oracle import UNetConfig, init_weights, unet_forward
    from test_gpu_fullconfig import REF_ARCH
    cfg = UNetConfig(sample_size=(64, 64), **REF_ARCH)
    w = _d(init_weights(cfg, seed=2))
    g = torch.Generator().manual_seed(3)
    x = OracleDDPM().add_noise((torch.rand(2, 1, 64, 64, generator=g) * 2 - 1).double(),
                               torch.randn(2, 1, 64, 64, generator=g).double(), T3[:2])
    taps = {}
    eps = unet_forward(w, cfg, x, T3[:2], taps)
    blocks = bg.unet_blocks(cfg)
    assert sum(blk.kind == "attn" for blk in blocks) == 6
    _chain(blocks, x, w, cfg, taps, eps, taps["temb_act"])


@pytest.mark.timeout(300)
def test_published_cond_unet_block_forward_chain():
    """The four-level UNet2DConditionModel at 32x32: sixteen transformers, distinct encodings."""
    from oracle.unet_cond_oracle import CondUNetConfig, init_weights, unet_cond_forward
    from test_gpu_cond_train import ARCH
    cfg = CondUNetConfig(sample_size=(32, 32), **{k: ARCH[k] for k in ("block_out_channels", "down_block_types",
                                                                         "up_block_types")})
    w = _d(init_weights(cfg, seed=3))
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 1, 32, 32, generator=g).double()
    enc = torch.randn(2, 1, 100, generator=g).double()
    taps = {}
    eps = unet_cond_forward(w, cfg, x, T3[:2], enc, taps)
    blocks = bg.unet_blocks(cfg)
    assert sum(blk.kind == "transformer" for blk in blocks) == 16
    _chain(blocks, x, w, cfg, taps, eps, bg.temb_act(w, cfg, T3[:2]), enc)


@pytest.mark.timeout(300)
def test_vae_block_forward_chain():
    """Both AutoencoderKL parts at 64x64 (an 8x8 latent)."""
    from oracle import vae_oracle as vo
    cfg = vo.VAEConfig()
    w = _d(vo.init_weights(cfg, seed=5))
    g = torch.Generator().manual_seed(6)
    x = torch.randn(2, 1, 64, 64, generator=g).clamp(-1, 1).double()
    z = torch.randn(2, 1, 8, 8, generator=g).double()
    for part, inp, fwd in (("decoder", z, vo.decode), ("encoder", x, vo.encode_moments)):
        taps = {}
        out = fwd(w, cfg, inp, taps)
        _chain(bg.vae_blocks(cfg, part), inp, w, cfg, taps, out)


def test_forward_rounding_model():
    """The probabilities are rounded where the engine packs them to bf16 (attention_mma_kernel: seq % 16 == 0 and
    seq <= 1536; mha_flash_kernel: always) and nowhere else (attention_kernel, the single-head attention).  A rounded
    reference differs from the exact one by a bf16 floor: more than 1e-4, less than 2 % relative L2."""
    from oracle.unet_oracle import UNetConfig, init_weights
    from test_gpu_fullconfig import REF_ARCH
    blk = bg.Block("attn", "mid_block.attentions.0", "x", None, "y", ("mid_block.attentions.0.",))
    for hw, rounds in (((6, 10), False), ((4, 4), True), ((16, 16), True), ((40, 40), False)):
        assert bg._probs_rounded(blk, torch.zeros(1, 8, *hw)) == rounds, hw
    assert bg._probs_rounded(bg.Block("transformer", "t", "x", None, "y", ()), torch.zeros(1, 8, 6, 10))
    assert not bg._probs_rounded(bg.Block("attn1", "a", "x", None, "y", ()), torch.zeros(1, 8, 32, 32))
    cfg = UNetConfig(sample_size=(64, 64), **REF_ARCH)
    w = _d(init_weights(cfg, seed=2))
    g = torch.Generator().manual_seed(7)
    for hw in ((4, 4), (6, 10)):
        x = bg.bf16(torch.randn(2, 512, *hw, generator=g).double())
        ex = bg.sub_forward(blk, w, [x], cfg)
        rd = bg.sub_forward(blk, w, [x], cfg, get=lambda k: bg.bf16(ex[k]), rounded=True)
        ex = bg.sub_forward(blk, w, [x], cfg, get=lambda k: bg.bf16(ex[k]))
        for k in (".qkv", ".ao", "out"):
            e = ((rd[k] - ex[k]).norm() / ex[k].norm()).item()
            assert 1e-4 < e < 2e-2, (hw, k, e)
        assert bg.block_forward(blk, w, [x], cfg, rounded=True).dtype == torch.float64
