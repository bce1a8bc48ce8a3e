"""CPU facts the conditional U-Net's backward relies on (oracle/unet_cond_oracle.py, fp32 autograd): with ONE encoder token
the cross-attention's softmax is constant, so attn2.to_q, attn2.to_k and norm2 get exactly zero gradients, while attn2.to_v
and attn2.to_out (the per-sample vector Wo (Wv enc) + bo) get real ones.  The engine launches nothing for the former."""
import torch

from oracle.schedulers_oracle import OracleDDPM
from oracle.unet_cond_oracle import CondUNetConfig, init_weights, unet_cond_forward

SMALL = dict(sample_size=(8, 8), block_out_channels=(32, 64), down_block_types=("CrossAttnDownBlock2D", "DownBlock2D"),
             up_block_types=("UpBlock2D", "CrossAttnUpBlock2D"))


def cond_loss_and_grads(w, cfg, clean, noise, t, enc):
    """MSE(ε̂, ε) of one conditional training step (scripts/train_unet.py:250-258) and its parameter gradients."""
    noisy = OracleDDPM().add_noise(clean, noise, t)
    wl = {k: v.detach().clone().requires_grad_(True) for k, v in w.items()}
    pred = unet_cond_forward(wl, cfg, noisy, t, enc)
    loss = torch.mean((pred - noise) ** 2)
    grads = torch.autograd.grad(loss, list(wl.values()))
    return loss.detach(), dict(zip(wl.keys(), grads))


def test_cond_cross_attention_gradients():
    cfg = CondUNetConfig(**SMALL)
    w = init_weights(cfg, seed=0)
    g = torch.Generator().manual_seed(1)
    clean = torch.rand(2, 1, 8, 8, generator=g) * 2 - 1
    noise = torch.randn(2, 1, 8, 8, generator=g)
    enc = torch.randn(2, 1, 100, generator=g)
    loss, grads = cond_loss_and_grads(w, cfg, clean, noise, torch.tensor([3, 900]), enc)
    assert torch.isfinite(loss)
    blocks = sorted({k.split(".transformer_blocks.0.")[0] for k in grads if ".transformer_blocks.0." in k})
    assert len(blocks) == 6            # 2 down, 1 mid, 3 up
    for b in blocks:
        t = b + ".transformer_blocks.0."
        for k in ("attn2.to_q.weight", "attn2.to_k.weight", "norm2.weight", "norm2.bias"):
            assert torch.count_nonzero(grads[t + k]) == 0, t + k
        for k in ("attn2.to_v.weight", "attn2.to_out.0.weight", "attn2.to_out.0.bias"):
            assert grads[t + k].abs().max() > 0, t + k
        # both output-projection biases are added once per pixel of the same tensor: equal gradients
        assert torch.allclose(grads[t + "attn2.to_out.0.bias"], grads[t + "attn1.to_out.0.bias"], rtol=1e-5, atol=1e-9)
