"""The checkpointed backward block by block: with `enable_gradient_checkpointing()` the training forward keeps only the
block outputs, and the backward re-runs each block's forward ops into buffers shared between blocks before that block's
backward.  A recompute that reads or leaves a stale shared buffer (GroupNorm statistics accumulated twice, another block's
softmax probabilities or log-sum-exp, the parity planes of another level) corrupts one block's gradients; when that block
is small against the whole model, tests/test_gpu_checkpointing.py's bound on the flat gradient does not see it.

So the per-block comparison of tests/test_gpu_block_backward_trained.py and tests/test_gpu_cond_seq.py runs here on
checkpointed models: the same architectures, shapes and seeds, every block's input and parameter gradients and the
timestep MLP's against fp64 autograd of that block over the engine's own block inputs (`debug_tensor`, kept under
checkpointing) and output gradient (`debug_grad`, the backward's own arena, which the recompute never writes).  The
bf16 floors depend on the seeds alone, so the bars are the plain tests' own, measured and checked there.  The training
forward's intra-block taps are not kept under checkpointing, so its per-tap checks are not repeated.

Each test prints the fp64 time and the peak device memory; the docstrings give what an H100 80GB HBM3 at a 700 W power
limit measured.
"""
import pytest

from blockcheck import unet_backward_case, vae_backward_case
from cases import (COND64_BARS, COND_BARS, COND_SEQ_BWD_TRANSFORMER_BARS, PUBLISHED, PUBLISHED_ATTN, PUBLISHED_COND, T3, T5,
                   TWO_LEVEL_COND, UNET64_BARS, VAE256_BARS)

pytestmark = pytest.mark.gpu


@pytest.mark.timeout(600)
def test_unet_64_packed_backward_per_block_checkpointed(cuda):
    """The published UNet2DModel at 64x64, batch 5 (packed 8x8 / 4x4 / 2x2 levels, a one-image last item), checkpointed:
    the bars of test_unet_64_packed_backward_per_block.  fp64 work: 0.5 s, 3.4 GiB peak."""
    _, blocks = unet_backward_case(cuda, PUBLISHED, (64, 64), 5, 9, T5, UNET64_BARS, checkpointing=True)
    assert [b.name for b in blocks if b.kind == "attn"] == PUBLISHED_ATTN


@pytest.mark.timeout(600)
def test_cond_unet_64_backward_per_block_checkpointed(cuda):
    """The published UNet2DConditionModel at 64x64, batch 2, one-token encodings, checkpointed: the transformers' recompute
    of their flash-attention log-sum-exp at seq 4096 / 1024 / 256 / 64.  The bars of test_cond_unet_64_backward_per_block.
    fp64 work: 0.7 s, 11.4 GiB peak."""
    _, blocks = unet_backward_case(cuda, PUBLISHED_COND, (64, 64), 2, 6, [211, 650], COND64_BARS, s=1, checkpointing=True)
    assert sum(b.kind == "transformer" for b in blocks) == 16


@pytest.mark.timeout(600)
def test_cond_seq_77_backward_per_block_checkpointed(cuda):
    """The two-level UNet2DConditionModel at 32x32, batch 3, with a 77-token encoding, checkpointed: the recompute of the
    cross-attention's K / V projections and log-sum-exp as well.  The bars of test_cond_seq_backward_per_block[77].
    fp64 work: 0.3 s, 1.5 GiB peak."""
    bars = dict(COND_BARS, transformer=COND_SEQ_BWD_TRANSFORMER_BARS[77])
    unet_backward_case(cuda, TWO_LEVEL_COND, (32, 32), 3, 3, T3, bars, s=77, checkpointing=True, one_token_grads=True)


@pytest.mark.timeout(600)
def test_vae_256_backward_per_block_checkpointed(cuda):
    """The ldm autoencoder at 256x256, batch 2, checkpointed: the single-head attention's probabilities over 1024 tokens
    and the asymmetric downsampler's parity planes recomputed.  The bars of test_vae_256_backward_per_block.
    fp64 work: 0.8 s, 5.7 GiB peak."""
    vae_backward_case(cuda, (256, 256), 4, VAE256_BARS, checkpointing=True)
