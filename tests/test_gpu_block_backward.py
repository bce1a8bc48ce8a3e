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

The U-Net's timestep MLP (time_embedding.linear_1 / linear_2) belongs to no block: after the walk, the engine's gradients
of its four tensors are compared with fp64 autograd of the MLP (block_grads.temb_backward) from the sum of every resnet's
fp64 gradient w.r.t. the temb_act it reads, as the "temb" row.  That checks, past the per-resnet time_emb_proj gradients,
the engine's gradient w.r.t. temb_act (its per-resnet rows scattered into one [N][rows] array and multiplied by the
concatenated time_emb_proj weights) and the MLP backward after it.  Its floor is the MLP's gradients from the resnets'
rounded-storage temb_act gradients against the exact ones (block_grads.backward_floors).

The bars are in tests/cases.py: tests/test_cpu_block_backward.py asserts them against the floors it measures.
"""
import pytest

from blockcheck import unet_backward_case, vae_backward_case
from cases import COND_BARS, T3, TWO_LEVEL, TWO_LEVEL_COND, UNET_BARS, VAE_BARS

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("size", [(32, 32), (32, 64)])
def test_unet_backward_per_block(cuda, size):
    """UNet2DModel (128, 256; DownBlock2D, AttnDownBlock2D), batch 3: every resnet (with and without conv_shortcut, over
    cat(input, skip), including up_blocks.0.resnets.2 whose 256 + 128 = 384 channels put a GroupNorm group of 12
    channels across the two sources), every head_dim-8 attention, the downsampler, the folded upsampler, conv_in and the
    conv_norm_out + conv_out tail."""
    unet_backward_case(cuda, TWO_LEVEL, size, 3, 2, T3, UNET_BARS)


def test_cond_unet_backward_per_block(cuda):
    """UNet2DConditionModel (transformer blocks at 32x32 in the down and the up block, 16x16 in the mid block), batch 3:
    every block as above, the transformers included; attn2.to_q, attn2.to_k and norm2 get exactly zero gradients."""
    unet_backward_case(cuda, TWO_LEVEL_COND, (32, 32), 3, 3, T3, COND_BARS, s=1, one_token_grads=True)


def test_vae_backward_per_block(cuda):
    """AutoencoderKL (ldm: 128, 256, 512, 512; 2 resnets per block) at 64x64, batch 2 (an 8x8 = 64-token latent):
    decoder backward from a seeded image gradient and encoder backward from seeded moment gradients.  Every resnet, the
    single-head attentions, the (0, 1, 0, 1)-padded downsamplers, the folded upsamplers, the encoder tail (conv_norm_out
    + conv_out + quant_conv, from g_moments), the decoder head (post_quant_conv + conv_in, to g_z) and the conv_out tail."""
    vae_backward_case(cuda, (64, 64), 0, VAE_BARS)
