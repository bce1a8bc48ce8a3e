"""The U-Net and autoencoder backward block by block at the shapes they are trained at, as tests/test_gpu_block_backward.py
does at small shapes: after one real training forward and backward through the public model, every block's input and
parameter gradients from the engine against fp64 autograd of that one block over the engine's own input activations and
output gradient, three metrics per tensor (block_grads.errors: relative L2, max |err| / max |ref|, worst row).

These shapes reach code the small models never run: the 8x32 and 16x16 conv tiles and the flat parity-scatter items of
the data-gradient convs at 64 - 256 pixel widths (the autoencoder's asymmetric 256 -> 128 downsampler included), the
packed 8x8 / 4x4 / 2x2 levels with a partly filled last item (batch 5), per-sample sums over an odd batch, the
autoencoder's single-head attention backward over S = 1024 tokens (16x16 tiles, 32 k-steps), and the conditional model's
multi-head flash attention backward at seq 4096 (head_dim 16) and at the 16x16 / 8x8 levels (head_dim 64).

Bars.  The fp64 oracle of the whole model at these shapes is too slow for the CPU, so each block's bf16 floor is measured
here, in the same run, as tests/test_cpu_block_backward.py measures it at small shapes (`_floors`): the fp64 oracle's own
forward on the GPU gives every block's input activations, block_grads.chain every block's output gradient, and each
block's reference under bf16_storage() on those rounded to bf16 is compared with the exact one, worst per block kind.
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
import time

import pytest
import torch

from oracle import block_grads as bg
from test_cpu_block_backward import _floors
from test_gpu_block_backward import _run_checks, _w64
from test_gpu_block_forward import _floors as _fwd_floors
from test_gpu_block_forward import check_against_floors, forward_checks
from test_gpu_cond_train import ARCH as COND_ARCH
from test_gpu_fullconfig import REF_ARCH

pytestmark = pytest.mark.gpu

T5 = [37, 211, 412, 650, 903]    # five distinct timesteps: per-sample sums over an odd batch with a one-image last item

# kind -> ((activation a, b, c), (parameter a, b, c))
UNET256_BARS = {
    "head": ((0.005, 0.005, 0.005), (0.005, 0.005, 0.005)),   # floor (0.0, 0.0, 0.0) | (0.0, 0.0, 0.0)
    "resnet": ((0.0129, 0.0201, 0.0129), (0.0144, 0.0183, 0.0846)),   # floor (0.0043, 0.0067, 0.0043) | (0.0048, 0.0061, 0.0282)
    "down": ((0.0072, 0.0099, 0.0069), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.0033, 0.0023) | (0.0, 0.0, 0.0)
    "attn": ((0.0051, 0.0099, 0.0051), (0.0168, 0.0201, 0.0894)),   # floor (0.0017, 0.0033, 0.0017) | (0.0056, 0.0067, 0.0298)
    "up": ((0.0087, 0.0129, 0.0084), (0.005, 0.005, 0.005)),   # floor (0.0029, 0.0043, 0.0028) | (0.0, 0.0, 0.0)
    "tail": ((0.0072, 0.0186, 0.0066), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.0062, 0.0022) | (0.0001, 0.0002, 0.0001)
}
UNET64_BARS = {
    "head": ((0.005, 0.005, 0.005), (0.005, 0.005, 0.005)),   # floor (0.0, 0.0, 0.0) | (0.0, 0.0, 0.0)
    "resnet": ((0.0132, 0.0204, 0.0171), (0.015, 0.0201, 0.0651)),   # floor (0.0044, 0.0068, 0.0057) | (0.005, 0.0067, 0.0217)
    "down": ((0.0072, 0.009, 0.0072), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.003, 0.0024) | (0.0, 0.0, 0.0)
    "attn": ((0.0066, 0.0093, 0.0078), (0.0174, 0.0201, 0.0615)),   # floor (0.0022, 0.0031, 0.0026) | (0.0058, 0.0067, 0.0205)
    "up": ((0.0087, 0.0132, 0.0096), (0.005, 0.005, 0.005)),   # floor (0.0029, 0.0044, 0.0032) | (0.0, 0.0, 0.0)
    "tail": ((0.0069, 0.0123, 0.0069), (0.005, 0.005, 0.005)),   # floor (0.0023, 0.0041, 0.0023) | (0.0001, 0.0002, 0.0001)
}
VAE256_BARS = {
    "decoder:dec_head": ((0.005, 0.005, 0.005), (0.005, 0.005, 0.005)),   # floor (0.0, 0.0, 0.0) | (0.0, 0.0, 0.0)
    "decoder:resnet_vae": ((0.0123, 0.0156, 0.0117), (0.0159, 0.0243, 0.0372)),   # floor (0.0041, 0.0052, 0.0039) | (0.0053, 0.0081, 0.0124)
    "decoder:attn1": ((0.0051, 0.0084, 0.005), (0.012, 0.0159, 0.0939)),   # floor (0.0017, 0.0028, 0.0015) | (0.004, 0.0053, 0.0313)
    "decoder:up": ((0.0087, 0.015, 0.0081), (0.005, 0.005, 0.005)),   # floor (0.0029, 0.005, 0.0027) | (0.0, 0.0, 0.0)
    "decoder:tail": ((0.0069, 0.0183, 0.0066), (0.0066, 0.0072, 0.0066)),   # floor (0.0023, 0.0061, 0.0022) | (0.0022, 0.0024, 0.0022)
    "encoder:head": ((0.005, 0.005, 0.005), (0.005, 0.005, 0.005)),   # floor (0.0, 0.0, 0.0) | (0.0, 0.0, 0.0)
    "encoder:resnet_vae": ((0.0123, 0.0183, 0.0117), (0.0147, 0.0192, 0.0336)),   # floor (0.0041, 0.0061, 0.0039) | (0.0049, 0.0064, 0.0112)
    "encoder:down_asym": ((0.0072, 0.0105, 0.0066), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.0035, 0.0022) | (0.0, 0.0, 0.0)
    "encoder:attn1": ((0.0051, 0.0066, 0.005), (0.0198, 0.0168, 0.0903)),   # floor (0.0017, 0.0022, 0.0016) | (0.0066, 0.0056, 0.0301)
    "encoder:enc_tail": ((0.0069, 0.0135, 0.0066), (0.0066, 0.0078, 0.0066)),   # floor (0.0023, 0.0045, 0.0022) | (0.0022, 0.0026, 0.0022)
}
COND64_BARS = {
    "head": ((0.005, 0.005, 0.005), (0.005, 0.005, 0.005)),   # floor (0.0, 0.0, 0.0) | (0.0, 0.0, 0.0)
    "resnet": ((0.0126, 0.0183, 0.0123), (0.0135, 0.0192, 0.132)),   # floor (0.0042, 0.0061, 0.0041) | (0.0045, 0.0064, 0.044)
    "transformer": ((0.009, 0.0141, 0.0096), (0.0237, 0.0279, 0.1374)),   # floor (0.003, 0.0047, 0.0032) | (0.0079, 0.0093, 0.0458)
    "down": ((0.0072, 0.0108, 0.0069), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.0036, 0.0023) | (0.0, 0.0, 0.0)
    "up": ((0.009, 0.015, 0.0084), (0.005, 0.005, 0.005)),   # floor (0.003, 0.005, 0.0028) | (0.0, 0.0, 0.0)
    "tail": ((0.0072, 0.0117, 0.0066), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.0039, 0.0022) | (0.0002, 0.0003, 0.0002)
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


def _report(name, floors, bars, t0):
    """Prints the floors as a bar table (three times the floor, no lower than 0.5 %), the time and the peak memory of the
    reference work; returns the bars outside (floor, max(3.3 x floor, 0.5 %)]."""
    torch.cuda.synchronize()
    print(f"\n{name}: fp64 time {time.perf_counter() - t0:.1f} s, peak device memory "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
    print("floors as bars (3 x floor, >= 0.005):")
    bad = []
    for kind, (a, p) in floors.items():
        fl = tuple(round(f, 4) for f in a + p)
        sug = tuple(round(max(3 * f, 0.005), 4) for f in fl)
        print(f'    "{kind}": ({sug[:3]}, {sug[3:]}),   # floor {fl[:3]} | {fl[3:]}')
        for f, b in zip(a + p, bars[kind][0] + bars[kind][1]):
            if not f < b <= max(3.3 * round(f, 4), 5e-3) + 1e-9:
                bad.append((kind, round(f, 4), b))
    return bad


def _unet_case(cuda, size, n, seed, bars, fwd_bars):
    from audio_diffusion_b200.unet import UNet2DModel
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_oracle import UNetConfig, init_weights, unet_forward
    cfg = UNetConfig(sample_size=size, **REF_ARCH)
    w = init_weights(cfg, seed=seed)
    model = UNet2DModel(sample_size=size, **REF_ARCH)
    model.load_state_dict(w)
    model = model.to(cuda).train()
    g = torch.Generator().manual_seed(seed + 1)
    clean = torch.rand(n, 1, *size, generator=g) * 2 - 1
    noise = torch.randn(n, 1, *size, generator=g)
    t = torch.tensor(T5[:n])
    noisy = OracleDDPM().add_noise(clean, noise, t).to(cuda)
    pred = model(noisy, t.to(cuda))["sample"]
    noise = noise.to(cuda)
    torch.nn.functional.mse_loss(pred, noise).backward()
    g_eps = 2 * (pred.detach() - noise) / pred.numel()
    eps = pred.detach()
    del pred
    blocks = bg.unet_blocks(cfg)
    assert [b.name for b in blocks if b.kind == "attn"] == (
        ["down_blocks.4.attentions.0", "down_blocks.4.attentions.1", "mid_block.attentions.0"]
        + [f"up_blocks.1.attentions.{j}" for j in range(3)])
    w64 = _w64(w, cuda)
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    fails = _run_checks(model, blocks, noisy, g_eps, w64, cfg, bars, temb=bg.temb_act(w64, cfg, t.to(cuda)))
    taps = {}
    with torch.no_grad():
        pred = unet_forward(w64, cfg, noisy.double(), t.to(cuda), taps)
    floors = _floors(blocks, taps, noisy.double(), 2 * (pred - noise.double()) / pred.numel(), w64, cfg, taps["temb_act"])
    bad = _report(f"UNet2DModel {size[0]}x{size[1]} batch {n}", floors, bars, t0)
    temb = bg.temb_act(w64, cfg, t.to(cuda))
    frows = forward_checks(model.debug_tensor, blocks, noisy, eps, w64, cfg, temb, taps="all")
    ffl = _fwd_floors(blocks, taps, noisy.double(), w64, cfg, temb, taps="all")
    assert not fails, fails
    assert not bad, bad
    check_against_floors(f"UNet2DModel {size[0]}x{size[1]} batch {n}, training forward", frows, ffl, fwd_bars, t0)


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
def test_vae_256_backward_per_block(cuda):
    """AutoencoderKL (ldm: 128, 256, 512, 512) at 256x256, batch 2 (a 32x32 latent): the mid blocks' single-head attention
    backward over S = 1024 tokens, the asymmetric (0, 1, 0, 1)-padded downsampler's data gradient from 256 to 128, and
    every 256x256 / 128x128 resnet; decoder backward from a seeded image gradient, encoder backward from seeded moment
    gradients.  fp64 work: 2.9 s, 12.0 GiB peak."""
    from audio_diffusion_b200.vae import AutoencoderKL
    from oracle import vae_oracle as vo
    cfg = vo.VAEConfig()
    w = vo.init_weights(cfg, seed=4)
    nb = len(cfg.block_out_channels)
    model = AutoencoderKL(in_channels=1, out_channels=1, down_block_types=("DownEncoderBlock2D",) * nb,
                          up_block_types=("UpDecoderBlock2D",) * nb, block_out_channels=cfg.block_out_channels,
                          layers_per_block=cfg.layers_per_block, latent_channels=1, max_batch=2)
    model.load_state_dict(w)
    model = model.to(cuda).train()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 1, 256, 256, generator=g).clamp(-1, 1).to(cuda)
    z = torch.randn(2, 1, 32, 32, generator=g).to(cuda)
    gx = torch.randn(2, 1, 256, 256, generator=g).to(cuda)
    gm = torch.randn(2, 2, 32, 32, generator=g).to(cuda)
    mom = model.encode(x).latent_dist.parameters
    mom.backward(gm)
    zz = z.clone().requires_grad_(True)
    img = model.decode(zz).sample
    img.backward(gx)
    w64 = _w64(w, cuda)
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    fails = _run_checks(model, bg.vae_blocks(cfg, "decoder"), z, gx, w64, cfg, VAE256_BARS, "decoder:", g_in=zz.grad)
    fails += _run_checks(model, bg.vae_blocks(cfg, "encoder"), x, gm, w64, cfg, VAE256_BARS, "encoder:")
    floors, frows, ffl = {}, [], {}
    for part, inp, gout, fwd, out in (("decoder", z, gx, vo.decode, img.detach()),
                                      ("encoder", x, gm, vo.encode_moments, mom.detach())):
        taps = {}
        with torch.no_grad():
            fwd(w64, cfg, inp.double(), taps)
        blocks = bg.vae_blocks(cfg, part)
        for k, v in _floors(blocks, taps, inp.double(), gout.double(), w64, cfg).items():
            floors[part + ":" + k] = v
        frows += forward_checks(model.debug_tensor, blocks, inp.double(), out, w64, cfg, prefix=part + ":", taps="all")
        ffl.update(_fwd_floors(blocks, taps, inp.double(), w64, cfg, prefix=part + ":", taps="all"))
    bad = _report("AutoencoderKL 256x256 batch 2", floors, VAE256_BARS, t0)
    assert not fails, fails
    assert not bad, bad
    check_against_floors("AutoencoderKL 256x256 batch 2, training forward", frows, ffl, VAE256_FWD_BARS, t0)


@pytest.mark.timeout(600)
def test_cond_unet_64_backward_per_block(cuda):
    """The published UNet2DConditionModel (128, 256, 512, 512; cross-attention transformers at 64x64, 32x32 and 16x16, the
    mid block at 8x8) at its 64x64 latent, batch 2 with distinct encodings: the flash attention backward inside the model
    at seq 4096 (head_dim 16) and at 16x16 / 8x8 (head_dim 64), on real activations.  fp64 work: 1.8 s, 18.0 GiB
    peak."""
    from audio_diffusion_b200.unet_cond import UNet2DConditionModel
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_cond_oracle import CondUNetConfig, init_weights, unet_cond_forward
    cfg = CondUNetConfig(sample_size=(64, 64), block_out_channels=COND_ARCH["block_out_channels"],
                         down_block_types=COND_ARCH["down_block_types"], up_block_types=COND_ARCH["up_block_types"])
    w = init_weights(cfg, seed=6)
    model = UNet2DConditionModel(sample_size=(64, 64), **COND_ARCH)
    model.load_state_dict(w)
    model = model.to(cuda).train()
    g = torch.Generator().manual_seed(7)
    clean = torch.rand(2, 1, 64, 64, generator=g) * 2 - 1
    noise = torch.randn(2, 1, 64, 64, generator=g)
    enc = torch.randn(2, 1, 100, generator=g).to(cuda)
    t = torch.tensor([211, 650])
    noisy = OracleDDPM().add_noise(clean, noise, t).to(cuda)
    pred = model(noisy, t.to(cuda), enc)["sample"]
    noise = noise.to(cuda)
    torch.nn.functional.mse_loss(pred, noise).backward()
    g_eps = 2 * (pred.detach() - noise) / pred.numel()
    eps = pred.detach()
    del pred
    blocks = bg.unet_blocks(cfg)
    assert sum(b.kind == "transformer" for b in blocks) == 16
    w64 = _w64(w, cuda)
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    temb = bg.temb_act(w64, cfg, t.to(cuda))
    fails = _run_checks(model, blocks, noisy, g_eps, w64, cfg, COND64_BARS, temb=temb, enc=enc)
    taps = {}
    with torch.no_grad():
        pred = unet_cond_forward(w64, cfg, noisy.double(), t.to(cuda), enc.double(), taps)
    floors = _floors(blocks, taps, noisy.double(), 2 * (pred - noise.double()) / pred.numel(), w64, cfg, temb,
                     enc.double())
    bad = _report("UNet2DConditionModel 64x64 batch 2", floors, COND64_BARS, t0)
    frows = forward_checks(model.debug_tensor, blocks, noisy, eps, w64, cfg, temb, enc.double(), taps="all")
    ffl = _fwd_floors(blocks, taps, noisy.double(), w64, cfg, temb, enc.double(), taps="all")
    assert not fails, fails
    assert not bad, bad
    check_against_floors("UNet2DConditionModel 64x64 batch 2, training forward", frows, ffl, COND64_FWD_BARS, t0)


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
    model = UNet2DModel(sample_size=(256, 256), seed=3, **REF_ARCH).to(cuda).train()
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
