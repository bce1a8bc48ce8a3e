"""The U-Net and autoencoder backward block by block at the shapes they are trained at, as tests/test_gpu_block_backward.py
does at small shapes: after one real training forward and backward through the public model, every block's input and
parameter gradients from the engine against fp64 autograd of that one block over the engine's own input activations and
output gradient, three metrics per tensor (block_grads.errors: relative L2, max |err| / max |ref|, worst row).

These shapes reach code the small models never run: the 8x32 and 16x16 conv tiles and the flat parity-scatter items of
the data-gradient convs at 64 - 256 pixel widths (the autoencoder's asymmetric 256 -> 128 downsampler included), the
packed 8x8 / 4x4 / 2x2 levels with a partly filled last item (batch 5), per-sample sums over an odd batch, the
autoencoder's single-head attention backward over S = 1024 tokens (16x16 tiles, 32 k-steps), the conditional model's
multi-head flash attention backward at seq 4096 (head_dim 16) and at the 16x16 / 8x8 levels (head_dim 64), and a
non-square image (96x160: odd 3x5 / 6x10 levels, the SIMT attention backward over 60 tokens).  Every U-Net case also
checks the timestep MLP's gradients (the "temb" row, tests/test_gpu_block_backward.py).  The same cases run with
gradient checkpointing in tests/test_gpu_block_backward_checkpointed.py, at the bars tests/cases.py keeps for both.

Bars.  The fp64 oracle of the whole model at these shapes is too slow for the CPU, so each block's bf16 floor is measured
here, in the same run, as tests/test_cpu_block_backward.py measures it at small shapes (block_grads.backward_floors):
the fp64 oracle's own forward on the GPU gives every block's input activations, block_grads.chain every block's output
gradient, and each block's reference under bf16_storage() on those rounded to bf16 is compared with the exact one, worst
per block kind.
The oracle's activations make the floor a function of the seeds alone.  The engine's own inputs would not: they move
between runs with the order of its fp32 atomics, and that moves the max and worst-row floors of some parameter gradients
by up to 2x, because each is one extreme of a different rounding pattern.  The bars below are three times the floor and
no lower than 0.5 % (the rule of tests/test_gpu_block_backward.py); every run asserts that the engine is within them and
that each bar lies in (floor, max(3.3 x floor, 0.5 %)] of the floors it measures.  The floors are in the comments as
(a, b, c).

The fp64 work (the oracle forward, and the exact and rounded reference of every block) is cheap on the GPU; each test
prints its time and the peak device memory, and its docstring gives what an H100 (80 GB SXM) measured.
"""
import contextlib

import pytest
import torch

from blockcheck import unet_backward_case, vae_backward_case
from cases import COND64_BARS, PUBLISHED, PUBLISHED_ATTN, PUBLISHED_COND, T5, UNET64_BARS, VAE256_BARS

pytestmark = pytest.mark.gpu

# kind -> ((activation a, b, c), (parameter a, b, c))
UNET256_BARS = {
    "head": ((0.005, 0.005, 0.005), (0.005, 0.005, 0.005)),   # floor (0.0, 0.0, 0.0) | (0.0, 0.0, 0.0)
    "resnet": ((0.0129, 0.0201, 0.0129), (0.0144, 0.0183, 0.0846)),   # floor (0.0043, 0.0067, 0.0043) | (0.0048, 0.0061, 0.0282)
    "down": ((0.0072, 0.0099, 0.0069), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.0033, 0.0023) | (0.0, 0.0, 0.0)
    "attn": ((0.0051, 0.0099, 0.0051), (0.0168, 0.0201, 0.0894)),   # floor (0.0017, 0.0033, 0.0017) | (0.0056, 0.0067, 0.0298)
    "up": ((0.0087, 0.0129, 0.0084), (0.005, 0.005, 0.005)),   # floor (0.0029, 0.0043, 0.0028) | (0.0, 0.0, 0.0)
    "tail": ((0.0072, 0.0186, 0.0066), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.0062, 0.0022) | (0.0001, 0.0002, 0.0001)
    "temb": ((0.005, 0.005, 0.005), (0.0057, 0.0066, 0.0717)),   # floor (0.0, 0.0, 0.0) | (0.0019, 0.0022, 0.0239)
}
UNET96x160_BARS = {
    "head": ((0.005, 0.005, 0.005), (0.005, 0.005, 0.005)),   # floor (0.0, 0.0, 0.0) | (0.0, 0.0, 0.0)
    "resnet": ((0.0129, 0.0222, 0.0135), (0.0144, 0.0195, 0.105)),   # floor (0.0043, 0.0074, 0.0045) | (0.0048, 0.0065, 0.035)
    "down": ((0.0072, 0.0117, 0.0069), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.0039, 0.0023) | (0.0, 0.0, 0.0)
    "attn": ((0.0054, 0.0078, 0.0057), (0.0171, 0.021, 0.1215)),   # floor (0.0018, 0.0026, 0.0019) | (0.0057, 0.007, 0.0405)
    "up": ((0.0087, 0.015, 0.0093), (0.005, 0.005, 0.005)),   # floor (0.0029, 0.005, 0.0031) | (0.0, 0.0, 0.0)
    "tail": ((0.0072, 0.0123, 0.0066), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.0041, 0.0022) | (0.0001, 0.0002, 0.0001)
    "temb": ((0.005, 0.005, 0.005), (0.0057, 0.0081, 0.0873)),   # floor (0.0, 0.0, 0.0) | (0.0019, 0.0027, 0.0291)
}

# the training forward (no timestep dedupe; every transformer tap kept: .h0, .n1, .qkv, .ao, .attn2, .n3, .ff1, .gg, .h3),
# block by block on the same run's activations as tests/test_gpu_block_forward.py checks the eval forward, bars by its
# rule: key -> (a, b, c), three times the floor printed beside it.  The fp64 times in the docstrings below include this
# work (measured with it: 256x256 11.3 s, 64x64 1.9 s, autoencoder 3.9 s, conditional 2.8 s; peak memory unchanged).
UNET256_FWD_BARS = {
    "attn": (0.00735, 0.01269, 0.00768),   # floor (0.00245, 0.00423, 0.00256)
    "attn.ao": (0.0051, 0.01056, 0.00561),   # floor (0.0017, 0.00352, 0.00187)
    "attn.out": (0.00636, 0.01224, 0.00678),   # floor (0.00212, 0.00408, 0.00226)
    "attn.qkv": (0.00882, 0.01251, 0.00873),   # floor (0.00294, 0.00417, 0.00291)
    "down": (0.00732, 0.01041, 0.00777),   # floor (0.00244, 0.00347, 0.00259)
    "head": (0.00498, 0.00606, 0.00462),   # floor (0.00166, 0.00202, 0.00154)
    "resnet": (0.01299, 0.01983, 0.01371),   # floor (0.00433, 0.00661, 0.00457)
    "resnet.h1": (0.0102, 0.02118, 0.01125),   # floor (0.0034, 0.00706, 0.00375)
    "resnet.out": (0.01017, 0.01722, 0.01053),   # floor (0.00339, 0.00574, 0.00351)
    "tail": (0.00924, 0.01008, 0.00885),   # floor (0.00308, 0.00336, 0.00295)
    "up": (0.00732, 0.01131, 0.00795),   # floor (0.00244, 0.00377, 0.00265)
    "resnet.h1:mean": (0.01971, 0.01971, 0.01971),   # floor (0.00657, 0.00657, 0.00657)
}
UNET64_FWD_BARS = {
    "attn": (0.00726, 0.01038, 0.00825),   # floor (0.00242, 0.00346, 0.00275)
    "attn.ao": (0.00549, 0.01044, 0.00612),   # floor (0.00183, 0.00348, 0.00204)
    "attn.out": (0.00621, 0.00981, 0.00699),   # floor (0.00207, 0.00327, 0.00233)
    "attn.qkv": (0.00876, 0.01242, 0.00939),   # floor (0.00292, 0.00414, 0.00313)
    "down": (0.00729, 0.01041, 0.00864),   # floor (0.00243, 0.00347, 0.00288)
    "head": (0.00498, 0.00738, 0.00468),   # floor (0.00166, 0.00246, 0.00156)
    "resnet": (0.01287, 0.018, 0.01503),   # floor (0.00429, 0.006, 0.00501)
    "resnet.h1": (0.01032, 0.01965, 0.01197),   # floor (0.00344, 0.00655, 0.00399)
    "resnet.out": (0.01002, 0.01725, 0.01098),   # floor (0.00334, 0.00575, 0.00366)
    "tail": (0.0084, 0.01176, 0.00771),   # floor (0.0028, 0.00392, 0.00257)
    "up": (0.00723, 0.01044, 0.00846),   # floor (0.00241, 0.00348, 0.00282)
    "resnet.h1:mean": (0.02574, 0.02574, 0.02574),   # floor (0.00858, 0.00858, 0.00858)
}
UNET96x160_FWD_BARS = {
    "attn": (0.00708, 0.01197, 0.00765),   # floor (0.00236, 0.00399, 0.00255)
    "attn.ao": (0.00498, 0.01053, 0.00534),   # floor (0.00166, 0.00351, 0.00178)
    "attn.out": (0.00618, 0.01098, 0.00648),   # floor (0.00206, 0.00366, 0.00216)
    "attn.qkv": (0.00879, 0.01416, 0.00876),   # floor (0.00293, 0.00472, 0.00292)
    "down": (0.00735, 0.01065, 0.00756),   # floor (0.00245, 0.00355, 0.00252)
    "head": (0.00498, 0.00684, 0.00465),   # floor (0.00166, 0.00228, 0.00155)
    "resnet": (0.01284, 0.01794, 0.01431),   # floor (0.00428, 0.00598, 0.00477)
    "resnet.h1": (0.01023, 0.01914, 0.01119),   # floor (0.00341, 0.00638, 0.00373)
    "resnet.h1:mean": (0.01767, 0.01767, 0.01767),   # floor (0.00589, 0.00589, 0.00589)
    "resnet.out": (0.01002, 0.01788, 0.01101),   # floor (0.00334, 0.00596, 0.00367)
    "tail": (0.00837, 0.00837, 0.00837),   # floor (0.00279, 0.00279, 0.00279)
    "up": (0.00723, 0.01023, 0.00753),   # floor (0.00241, 0.00341, 0.00251)
}
VAE256_FWD_BARS = {
    "decoder:attn1": (0.00579, 0.00942, 0.00579),   # floor (0.00193, 0.00314, 0.00193)
    "decoder:attn1.ao": (0.00495, 0.00906, 0.00531),   # floor (0.00165, 0.00302, 0.00177)
    "decoder:attn1.out": (0.00549, 0.00954, 0.00528),   # floor (0.00183, 0.00318, 0.00176)
    "decoder:attn1.qkv": (0.00876, 0.00993, 0.0087),   # floor (0.00292, 0.00331, 0.0029)
    "decoder:dec_head": (0.00498, 0.00594, 0.00462),   # floor (0.00166, 0.00198, 0.00154)
    "decoder:resnet_vae": (0.01233, 0.01788, 0.0135),   # floor (0.00411, 0.00596, 0.0045)
    "decoder:resnet_vae.h1": (0.00888, 0.01377, 0.00966),   # floor (0.00296, 0.00459, 0.00322)
    "decoder:resnet_vae.out": (0.00993, 0.01434, 0.01068),   # floor (0.00331, 0.00478, 0.00356)
    "decoder:tail": (0.00711, 0.00951, 0.00711),   # floor (0.00237, 0.00317, 0.00237)
    "decoder:up": (0.00711, 0.01098, 0.00729),   # floor (0.00237, 0.00366, 0.00243)
    "encoder:attn1": (0.00588, 0.0084, 0.00591),   # floor (0.00196, 0.0028, 0.00197)
    "encoder:attn1.ao": (0.00504, 0.00975, 0.00513),   # floor (0.00168, 0.00325, 0.00171)
    "encoder:attn1.out": (0.00555, 0.00861, 0.00528),   # floor (0.00185, 0.00287, 0.00176)
    "encoder:attn1.qkv": (0.00879, 0.01089, 0.00843),   # floor (0.00293, 0.00363, 0.00281)
    "encoder:down_asym": (0.00714, 0.00951, 0.00798),   # floor (0.00238, 0.00317, 0.00266)
    "encoder:enc_tail": (0.00501, 0.00756, 0.00501),   # floor (0.00167, 0.00252, 0.00167)
    "encoder:head": (0.00498, 0.01062, 0.00459),   # floor (0.00166, 0.00354, 0.00153)
    "encoder:resnet_vae": (0.01287, 0.01719, 0.01281),   # floor (0.00429, 0.00573, 0.00427)
    "encoder:resnet_vae.h1": (0.00885, 0.01176, 0.00915),   # floor (0.00295, 0.00392, 0.00305)
    "encoder:resnet_vae.out": (0.0099, 0.01554, 0.00963),   # floor (0.0033, 0.00518, 0.00321)
    "decoder:resnet_vae.h1:mean": (0.01281, 0.01281, 0.01281),   # floor (0.00427, 0.00427, 0.00427)
    "encoder:resnet_vae.h1:mean": (0.01101, 0.01101, 0.01101),   # floor (0.00367, 0.00367, 0.00367)
}
COND64_FWD_BARS = {
    "down": (0.00714, 0.01077, 0.00771),   # floor (0.00238, 0.00359, 0.00257)
    "head": (0.00498, 0.0069, 0.00465),   # floor (0.00166, 0.0023, 0.00155)
    "resnet": (0.0123, 0.01875, 0.01332),   # floor (0.0041, 0.00625, 0.00444)
    "resnet.h1": (0.01023, 0.02082, 0.01131),   # floor (0.00341, 0.00694, 0.00377)
    "resnet.out": (0.00987, 0.01749, 0.01062),   # floor (0.00329, 0.00583, 0.00354)
    "tail": (0.00915, 0.01083, 0.00915),   # floor (0.00305, 0.00361, 0.00305)
    "transformer": (0.01047, 0.01485, 0.01155),   # floor (0.00349, 0.00495, 0.00385)
    "transformer.ao": (0.00507, 0.01125, 0.00564),   # floor (0.00169, 0.00375, 0.00188)
    "transformer.attn2": (0.00702, 0.01137, 0.01086),   # floor (0.00234, 0.00379, 0.00362)
    "transformer.ff1": (0.00726, 0.01233, 0.00765),   # floor (0.00242, 0.00411, 0.00255)
    "transformer.gg": (0.00495, 0.009, 0.00498),   # floor (0.00165, 0.003, 0.00166)
    "transformer.h0": (0.00885, 0.01302, 0.00993),   # floor (0.00295, 0.00434, 0.00331)
    "transformer.h3": (0.00522, 0.00831, 0.00516),   # floor (0.00174, 0.00277, 0.00172)
    "transformer.n1": (0.00501, 0.01014, 0.00483),   # floor (0.00167, 0.00338, 0.00161)
    "transformer.n3": (0.00501, 0.01062, 0.00477),   # floor (0.00167, 0.00354, 0.00159)
    "transformer.out": (0.00738, 0.01272, 0.00768),   # floor (0.00246, 0.00424, 0.00256)
    "transformer.qkv": (0.00732, 0.01146, 0.00747),   # floor (0.00244, 0.00382, 0.00249)
    "up": (0.00708, 0.00939, 0.00789),   # floor (0.00236, 0.00313, 0.00263)
    "resnet.h1:mean": (0.01806, 0.01806, 0.01806),   # floor (0.00602, 0.00602, 0.00602)
}


def _unet_case(cuda, size, n, seed, bars, fwd_bars):
    """The published UNet2DModel at `size`, batch n: one training forward and backward, every block and the timestep MLP
    against fp64, the floors of the bars measured in the same run, and the training forward block by block."""
    model, blocks = unet_backward_case(cuda, PUBLISHED, size, n, seed, T5[:n], bars, floors=True, fwd_bars=fwd_bars)
    assert [b.name for b in blocks if b.kind == "attn"] == PUBLISHED_ATTN
    return model


@pytest.mark.timeout(900)
def test_unet_256_backward_per_block(cuda):
    """The published UNet2DModel (128, 128, 256, 256, 512, 512; attention at 16x16 with C = 512) at 256x256, batch 5:
    every level from 256x256 to 8x8, the 8x32 and 16x16 data-gradient tiles, the parity-scatter data gradient of every
    downsampler, the folded upsamplers' data gradients, and per-sample bias / time-embedding sums over an odd batch.
    fp64 work: 10 s, 28.6 GiB peak."""
    _unet_case(cuda, (256, 256), 5, 7, UNET256_BARS, UNET256_FWD_BARS)


@pytest.mark.timeout(600)
def test_unet_64_packed_backward_per_block(cuda):
    """The published UNet2DModel at 64x64, batch 5: the 8x8, 4x4 and 2x2 levels pack up to four images per conv work
    item, so the last item holds one image; a gradient leaking across the halo between packed images shows here and not
    at batch 1.  Attention at 4x4.  fp64 work: 1.2 s, 4.9 GiB peak."""
    _unet_case(cuda, (64, 64), 5, 9, UNET64_BARS, UNET64_FWD_BARS)


@pytest.mark.timeout(600)
def test_unet_96x160_backward_per_block(cuda):
    """The published UNet2DModel at 96x160, batch 3 (the shape of the forward's non-square per-block test): the levels are
    96x160, 48x80, 24x40, 12x20, 6x10 and 3x5.  The attention level is 6x10 = 60 tokens, not a multiple of 16, so the
    forward runs the SIMT attention_kernel and the backward attention_bwd_kernel at 60 tokens; the data- and weight-
    gradient convs run over 5-, 10-, 20- ... pixel rows whose pad columns differ from the square levels', wgrad_tc's
    flat pixel blocks straddle the end of an odd-sized image, and the 6x10 and 3x5 levels are packed work items of
    non-square images.  fp64 work: 2.3 s, 6.3 GiB peak."""
    levels = [(96 >> i, 160 >> i) for i in range(6)]
    assert levels[4] == (6, 10) and 6 * 10 % 16 != 0
    model = _unet_case(cuda, (96, 160), 3, 15, UNET96x160_BARS, UNET96x160_FWD_BARS)
    got = [tuple(model.debug_tensor(f"down_blocks.{i}.resnets.0").shape[2:]) for i in range(len(levels))]
    assert got == levels, got


@pytest.mark.timeout(600)
def test_vae_256_backward_per_block(cuda):
    """AutoencoderKL (ldm: 128, 256, 512, 512) at 256x256, batch 2 (a 32x32 latent): the mid blocks' single-head attention
    backward over S = 1024 tokens, the asymmetric (0, 1, 0, 1)-padded downsampler's data gradient from 256 to 128, and
    every 256x256 / 128x128 resnet; decoder backward from a seeded image gradient, encoder backward from seeded moment
    gradients.  fp64 work: 2.9 s, 12.0 GiB peak."""
    vae_backward_case(cuda, (256, 256), 4, VAE256_BARS, floors=True, fwd_bars=VAE256_FWD_BARS)


@pytest.mark.timeout(600)
def test_cond_unet_64_backward_per_block(cuda):
    """The published UNet2DConditionModel (128, 256, 512, 512; cross-attention transformers at 64x64, 32x32 and 16x16, the
    mid block at 8x8) at its 64x64 latent, batch 2 with distinct encodings: the flash attention backward inside the model
    at seq 4096 (head_dim 16) and at 16x16 / 8x8 (head_dim 64), on real activations.  fp64 work: 1.8 s, 18.0 GiB
    peak."""
    _, blocks = unet_backward_case(cuda, PUBLISHED_COND, (64, 64), 2, 6, [211, 650], COND64_BARS, s=1, floors=True,
                                   fwd_bars=COND64_FWD_BARS)
    assert sum(b.kind == "transformer" for b in blocks) == 16


@pytest.mark.timeout(600)
def test_batch16_gradient_equals_four_accumulated_micro_batches(cuda):
    """The published UNet2DModel at 256x256 (the benchmarked shape): the gradient of one batch-16 MSE step against four
    micro-batches of 4 with loss / 4, accumulated in place (`no_sync()` on the first three), as
    `accelerator.accumulate` runs them.  GroupNorm is per sample, so the two agree up to the order of the backward's fp32
    sums; anything sized or indexed by the batch (per-sample sums, weight-gradient split caps, offsets) that breaks at 16
    shows here.  Bars: each micro-batch's output equals its slice of the full batch's to 0.1 % of the largest value; 0.2 %
    relative L2 over all gradients; for every tensor with a non-negligible gradient (the key biases, whose true gradient
    is zero, left out) 1 %, or twice what the same tensor differs by between two identical batch-16 backward passes.
    Measured on an H100: outputs bit-identical, 0.018 % over all gradients; the worst tensors (deep conv weights whose
    gradient norm is 1e-3 of the largest) differ by 1.5 % between the accumulated and the full batch and by the same
    1.5 % between two runs of the full batch, from fp32 summation order alone."""
    from audio_diffusion_b200.unet import UNet2DModel
    model = UNet2DModel(sample_size=(256, 256), seed=3, **PUBLISHED).to(cuda).train()
    g = torch.Generator().manual_seed(8)
    x = torch.randn(16, 1, 256, 256, generator=g).to(cuda)
    tgt = torch.randn(16, 1, 256, 256, generator=g).to(cuda)
    t = torch.randint(0, 1000, (16,), generator=g).to(cuda)
    mse = torch.nn.functional.mse_loss
    runs = []
    for _ in range(2):
        for p in model.parameters():
            p.grad = None
        pred = model(x, t)["sample"]
        mse(pred, tgt).backward()
        runs.append({k: p.grad.clone() for k, p in model.named_parameters()})
    full_flat = model._grad_flat.clone()
    full, again = runs
    for p in model.parameters():
        p.grad = None
    out_err = 0.0
    for i in range(4):
        s = slice(4 * i, 4 * i + 4)
        with model.no_sync() if i < 3 else contextlib.nullcontext():
            pm = model(x[s], t[s])["sample"]
            out_err = max(out_err, (pm.detach() - pred[s].detach()).abs().max().item())
            (mse(pm, tgt[s]) / 4).backward()
    out_err /= pred.detach().abs().max().item()
    total = ((model._grad_flat - full_flat).norm() / full_flat.norm()).item()
    rel = lambda a, b: ((a - b).norm() / b.norm()).item()
    gmax = max(v.norm().item() for v in full.values())
    rows = sorted((rel(p.grad, full[k]), rel(again[k], full[k]), k) for k, p in model.named_parameters()
                  if not k.endswith("to_k.bias") and full[k].norm().item() > 1e-3 * gmax)
    print(f"\n{'tensor':48s} {'accumulated':>12s} {'run to run':>12s}")
    for e, r, k in rows[-8:]:
        print(f"{k:48s} {e:12.5f} {r:12.5f}")
    print(f"batch 16 vs 4 x 4 accumulated: outputs {out_err:.2e}, relative L2 {total:.5f} over all gradients, worst "
          f"tensor {rows[-1][0]:.5f} ({rows[-1][2]}), {len(rows)} tensors compared")
    assert out_err <= 1e-3, out_err
    assert total <= 2e-3, total
    bad = [(k, e, r) for e, r, k in rows if e > max(1e-2, 2 * r)]
    assert not bad, bad
