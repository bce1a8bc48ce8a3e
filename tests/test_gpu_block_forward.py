"""The U-Net and autoencoder forward block by block on the sampling path: the public models in eval mode (every activation
in its own buffer, B200AD_DEBUG_NOPOOL=1), every block's output and every sub-block tap the engine keeps, read from the
engine (`debug_tensor`), against the fp64 reference of that one block or step (oracle/block_grads.py: `block_forward`,
`sub_forward`) computed from the engine's own inputs of it.  Errors do not compound across blocks or steps, so a 1 - 2 %
error confined to one GroupNorm group, one sample's time-embedding row, one folded-upsample parity, a tile border or
the last packed work item shows here, where the end-to-end tests against the fp32 oracle (6 % max / 1.5 - 3 % rms per
layer) let it pass.

Keys: `<kind>` is the whole block from its inputs; `<kind>.h1` a resnet's GroupNorm + SiLU + conv1 + time projection
over cat(input, skip); `<kind>.out` its output from the engine's own `.h1` and input; `<kind>.qkv` an attention's
GroupNorm + q|k|v projection, `<kind>.ao` its core from the engine's own `.qkv`, `<kind>.out` the output projection +
residual from the engine's own `.ao`; `transformer.attn2` the transformer's h2 (proj_in, attn1, the one-key cross
attention) and `transformer.out` its output from the engine's own h2.  A Downsample2D's `.parity` tap must equal the
parity split of its input bit for bit.  Three metrics per tensor (block_grads.errors with act=True): relative L2,
max |err| / max |ref|, worst (sample, channel group) row; for `.h1` also `.h1:mean`, the largest pixel mean of the error
of one (sample, channel) over the reference's RMS, which sees a wrong time-embedding row that the row metric, diluted
by the rounding noise of the whole row, does not.

Bars.  The floor is measured in the same run (block_grads.forward_floors): the fp64 oracle's forward on the compared samples gives every
block's inputs; each block's reference and each step's reference under the forward rounding model
(bf16_storage(forward=True): bf16 conv / linear operands, weights and outputs, the bf16 probability numerators of the
tensor-core attention kernels, conv_out's bf16 weights, every tap stored in bf16) on those inputs rounded to bf16,
against the exact one; worst per key.  Each bar is 3x its floor; every run asserts that the engine is within its bars
and that each bar lies in (floor, 3.3 x floor].
"""
import pytest
import torch

from blockcheck import check_fused_step, forward_case, pooled_eps
from cases import LDM, PUBLISHED, PUBLISHED_COND
from oracle import block_grads as bg

pytestmark = pytest.mark.gpu

# key -> (a, b, c), three times the floor printed beside it
UNET256_BARS = {
    "attn": (0.00732, 0.01254, 0.00813),   # floor (0.00244, 0.00418, 0.00271)
    "attn.ao": (0.0051, 0.01158, 0.00561),   # floor (0.0017, 0.00386, 0.00187)
    "attn.out": (0.00636, 0.01251, 0.00654),   # floor (0.00212, 0.00417, 0.00218)
    "attn.qkv": (0.00882, 0.01248, 0.00885),   # floor (0.00294, 0.00416, 0.00295)
    "down": (0.00729, 0.01062, 0.00774),   # floor (0.00243, 0.00354, 0.00258)
    "head": (0.00498, 0.00591, 0.00456),   # floor (0.00166, 0.00197, 0.00152)
    "resnet": (0.01284, 0.02073, 0.0138),   # floor (0.00428, 0.00691, 0.0046)
    "resnet.h1": (0.0102, 0.01848, 0.01104),   # floor (0.0034, 0.00616, 0.00368)
    "resnet.out": (0.01005, 0.01881, 0.01143),   # floor (0.00335, 0.00627, 0.00381)
    "tail": (0.00879, 0.0105, 0.00807),   # floor (0.00293, 0.0035, 0.00269)
    "up": (0.00726, 0.0117, 0.00795),   # floor (0.00242, 0.0039, 0.00265)
    "resnet.h1:mean": (0.01608, 0.01608, 0.01608),   # floor (0.00536, 0.00536, 0.00536)
}
UNET64_BARS = {
    "attn": (0.00729, 0.00993, 0.00861),   # floor (0.00243, 0.00331, 0.00287)
    "attn.ao": (0.00543, 0.01164, 0.0063),   # floor (0.00181, 0.00388, 0.0021)
    "attn.out": (0.00624, 0.01164, 0.00705),   # floor (0.00208, 0.00388, 0.00235)
    "attn.qkv": (0.00885, 0.01239, 0.00984),   # floor (0.00295, 0.00413, 0.00328)
    "down": (0.00729, 0.01125, 0.009),   # floor (0.00243, 0.00375, 0.003)
    "head": (0.00498, 0.00693, 0.00462),   # floor (0.00166, 0.00231, 0.00154)
    "resnet": (0.01278, 0.02316, 0.01521),   # floor (0.00426, 0.00772, 0.00507)
    "resnet.h1": (0.01026, 0.01821, 0.01245),   # floor (0.00342, 0.00607, 0.00415)
    "resnet.out": (0.01005, 0.01881, 0.01104),   # floor (0.00335, 0.00627, 0.00368)
    "tail": (0.00897, 0.0084, 0.00834),   # floor (0.00299, 0.0028, 0.00278)
    "up": (0.00729, 0.01131, 0.00798),   # floor (0.00243, 0.00377, 0.00266)
    "resnet.h1:mean": (0.02289, 0.02289, 0.02289),   # floor (0.00763, 0.00763, 0.00763)
}
UNET96x160_BARS = {
    "attn": (0.00702, 0.01056, 0.00765),   # floor (0.00234, 0.00352, 0.00255)
    "attn.ao": (0.00504, 0.01026, 0.00552),   # floor (0.00168, 0.00342, 0.00184)
    "attn.out": (0.00618, 0.01065, 0.00642),   # floor (0.00206, 0.00355, 0.00214)
    "attn.qkv": (0.00876, 0.01281, 0.009),   # floor (0.00292, 0.00427, 0.003)
    "down": (0.00732, 0.01056, 0.00759),   # floor (0.00244, 0.00352, 0.00253)
    "head": (0.00498, 0.00633, 0.00459),   # floor (0.00166, 0.00211, 0.00153)
    "resnet": (0.01287, 0.01965, 0.01404),   # floor (0.00429, 0.00655, 0.00468)
    "resnet.h1": (0.01023, 0.01956, 0.0111),   # floor (0.00341, 0.00652, 0.0037)
    "resnet.out": (0.01002, 0.01788, 0.01086),   # floor (0.00334, 0.00596, 0.00362)
    "tail": (0.00846, 0.01032, 0.00846),   # floor (0.00282, 0.00344, 0.00282)
    "up": (0.0072, 0.0105, 0.00753),   # floor (0.0024, 0.0035, 0.00251)
    "resnet.h1:mean": (0.01605, 0.01605, 0.01605),   # floor (0.00535, 0.00535, 0.00535)
}
COND64_BARS = {
    "down": (0.00723, 0.0099, 0.00786),   # floor (0.00241, 0.0033, 0.00262)
    "head": (0.00498, 0.00705, 0.00462),   # floor (0.00166, 0.00235, 0.00154)
    "resnet": (0.01215, 0.01725, 0.01308),   # floor (0.00405, 0.00575, 0.00436)
    "resnet.h1": (0.0102, 0.01758, 0.01137),   # floor (0.0034, 0.00586, 0.00379)
    "resnet.out": (0.00966, 0.01869, 0.01056),   # floor (0.00322, 0.00623, 0.00352)
    "tail": (0.00906, 0.00957, 0.00906),   # floor (0.00302, 0.00319, 0.00302)
    "transformer": (0.01029, 0.01545, 0.01128),   # floor (0.00343, 0.00515, 0.00376)
    "transformer.attn2": (0.01053, 0.01716, 0.01341),   # floor (0.00351, 0.00572, 0.00447)
    "transformer.out": (0.00822, 0.01314, 0.00894),   # floor (0.00274, 0.00438, 0.00298)
    "up": (0.00726, 0.01167, 0.00822),   # floor (0.00242, 0.00389, 0.00274)
    "resnet.h1:mean": (0.01791, 0.01791, 0.01791),   # floor (0.00597, 0.00597, 0.00597)
}
VAE256_BARS = {
    "decoder:attn1": (0.00705, 0.00948, 0.0072),   # floor (0.00235, 0.00316, 0.0024)
    "decoder:attn1.ao": (0.00501, 0.00756, 0.00552),   # floor (0.00167, 0.00252, 0.00184)
    "decoder:attn1.out": (0.00621, 0.00909, 0.00609),   # floor (0.00207, 0.00303, 0.00203)
    "decoder:attn1.qkv": (0.00876, 0.01017, 0.00855),   # floor (0.00292, 0.00339, 0.00285)
    "decoder:dec_head": (0.00498, 0.0081, 0.00465),   # floor (0.00166, 0.0027, 0.00155)
    "decoder:resnet_vae": (0.01263, 0.01779, 0.01371),   # floor (0.00421, 0.00593, 0.00457)
    "decoder:resnet_vae.h1": (0.00882, 0.01209, 0.00978),   # floor (0.00294, 0.00403, 0.00326)
    "decoder:resnet_vae.out": (0.00966, 0.0153, 0.01077),   # floor (0.00322, 0.0051, 0.00359)
    "decoder:tail": (0.00762, 0.01077, 0.00762),   # floor (0.00254, 0.00359, 0.00254)
    "decoder:up": (0.00741, 0.01047, 0.00795),   # floor (0.00247, 0.00349, 0.00265)
    "encoder:attn1": (0.00588, 0.00867, 0.00594),   # floor (0.00196, 0.00289, 0.00198)
    "encoder:attn1.ao": (0.00504, 0.00903, 0.00513),   # floor (0.00168, 0.00301, 0.00171)
    "encoder:attn1.out": (0.00552, 0.00867, 0.00528),   # floor (0.00184, 0.00289, 0.00176)
    "encoder:attn1.qkv": (0.00882, 0.01023, 0.00879),   # floor (0.00294, 0.00341, 0.00293)
    "encoder:down_asym": (0.00717, 0.01068, 0.00762),   # floor (0.00239, 0.00356, 0.00254)
    "encoder:enc_tail": (0.00177, 0.00738, 0.00177),   # floor (0.00059, 0.00246, 0.00059)
    "encoder:head": (0.00498, 0.00996, 0.00462),   # floor (0.00166, 0.00332, 0.00154)
    "encoder:resnet_vae": (0.01284, 0.01767, 0.01272),   # floor (0.00428, 0.00589, 0.00424)
    "encoder:resnet_vae.h1": (0.00888, 0.0123, 0.00912),   # floor (0.00296, 0.0041, 0.00304)
    "encoder:resnet_vae.out": (0.00984, 0.018, 0.00966),   # floor (0.00328, 0.006, 0.00322)
    "decoder:resnet_vae.h1:mean": (0.01218, 0.01218, 0.01218),   # floor (0.00406, 0.00406, 0.00406)
    "encoder:resnet_vae.h1:mean": (0.01125, 0.01125, 0.01125),   # floor (0.00375, 0.00375, 0.00375)
}


@pytest.mark.timeout(1200)
def test_unet_256_batch64_forward_per_block(cuda, monkeypatch):
    """The published UNet2DModel at 256x256, batch 64 (the benchmarked shape: the conv planner's 8x32 and 16x16 tiles and
    the 8x8 level packed two images per item), per-sample timesteps t_i = 999 - 7 (i mod 13), so that samples 13 .. 63
    read the time embedding of an earlier sample with the same timestep (`temb_lead`).  Compared samples 0, 1, 13, 27,
    62, 63: the first and the last two; 0 and 1, and 62 and 63 (the last item), share a packed 8x8 work item; 13 repeats
    sample 0's timestep, 27 sample 1's, 62 and 63 samples 10 and 11's.
    The same input through the pooled buffers (no NOPOOL) gives the same eps: measured bit-identical (and two pooled runs
    bit-identical too).  The unpooled batch-64 workspace fits beside the fp64 work: on an H100 80GB HBM3 at a 700 W
    power limit, fp64 work 3 s, 32.1 GiB peak device memory."""
    sel = [0, 1, 13, 27, 62, 63]
    t = [999 - 7 * (i % 13) for i in range(64)]
    x, tt, w, eps = forward_case(cuda, monkeypatch, PUBLISHED, (256, 256), 64, 11, UNET256_BARS, t=t, sel=sel)
    monkeypatch.delenv("B200AD_DEBUG_NOPOOL")
    torch.cuda.empty_cache()
    e1, e2 = pooled_eps(cuda, PUBLISHED, w, (256, 256), x, tt)
    spread = (e1 - e2).abs().max().item()
    diff = (e1 - eps).abs().max().item()
    print(f"pooled vs unpooled eps: max |diff| {diff:.3e}; two pooled runs: {spread:.3e}")
    assert diff <= spread, (diff, spread)


@pytest.mark.timeout(600)
def test_unet_64_batch5_forward_per_block(cuda, monkeypatch):
    """The published UNet2DModel at 64x64, batch 5: the 8x8, 4x4 and 2x2 levels are packed, the last item holds one
    image (sample 4).  Attention at 4x4 (16 tokens: attention_mma_kernel) and, in the mid block, 2x2 (attention_kernel).
    All samples compared.  H100 80GB HBM3, 700 W: fp64 work 0.8 s, 2.1 GiB peak."""
    forward_case(cuda, monkeypatch, PUBLISHED, (64, 64), 5, 13, UNET64_BARS, t=[37, 211, 412, 650, 903],
                 sel=list(range(5)))


@pytest.mark.timeout(600)
def test_unet_96x160_forward_per_block(cuda, monkeypatch):
    """The published UNet2DModel at 96x160, batch 3: the attention level is 6x10 = 60 tokens (not a multiple of 16), so
    launch_attention runs the SIMT attention_kernel (its `.ao` rows in the table); the levels 3x5, 6x10, 12x20 ... 96x160
    are odd and non-square.  H100 80GB HBM3, 700 W: fp64 work 0.9 s, 2.9 GiB peak."""
    from oracle.unet_oracle import UNetConfig
    blocks = bg.unet_blocks(UNetConfig(sample_size=(96, 160), **PUBLISHED))
    assert [b.name for b in blocks if b.kind == "attn"][0] == "down_blocks.4.attentions.0"   # 96 / 16 x 160 / 16
    assert (96 // 16) * (160 // 16) % 16 != 0
    forward_case(cuda, monkeypatch, PUBLISHED, (96, 160), 3, 15, UNET96x160_BARS, t=[999, 500, 999], sel=[0, 1, 2])


@pytest.mark.timeout(600)
def test_cond_unet_64_forward_per_block(cuda, monkeypatch):
    """The published UNet2DConditionModel at its 64x64 latent, batch 3, distinct encodings: every transformer's eval path
    (mha_flash_kernel at seq 4096 / 1024 / 256 / 64 and the one-key cross attention folded into a per-sample vector).
    H100 80GB HBM3, 700 W: fp64 work 1.4 s, 15.8 GiB peak."""
    forward_case(cuda, monkeypatch, PUBLISHED_COND, (64, 64), 3, 17, COND64_BARS, t=[37, 412, 903], s=1)


@pytest.mark.timeout(600)
def test_vae_256_forward_per_block(cuda, monkeypatch):
    """AutoencoderKL (ldm: 128, 256, 512, 512) at 256x256, batch 3: encode from a seeded image (the single-head attention
    over S = 1024 tokens, the asymmetric 256 -> 128 downsampler; compared output: the moments), decode from seeded
    latents (teacher-forced: the decoder's blocks read the engine's own activations).  H100 80GB HBM3, 700 W: fp64 work
    1.8 s, 6.6 GiB peak."""
    forward_case(cuda, monkeypatch, LDM, (256, 256), 3, 19, VAE256_BARS)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("kind", ["ddpm", "ddim"])
def test_fused_step_256_batch64(cuda, kind):
    """The fused scheduler update of conv_out at the benchmarked shape (256x256, batch 64, pooled buffers): one DDPM step
    with noise at t = 999, where the x0 clip is active, and one DDIM step (eta = 0, 50 steps, t = 980).
    x_out against the fp64 update on the engine's own eps and the same z, within 8 fp32 roundings of the sum of its
    terms' magnitudes (blockcheck.check_fused_step).  eps of the fused step against model(x, t) on the same input: equal,
    or within what two identical model(x, t) calls differ by.  Measured on an H100 80GB HBM3 at 700 W: x0 clipped for
    99.6 % (DDPM) and 99.5 % (DDIM) of the elements; the largest error 0.24 and 0.16 of its bar; eps bit-identical to
    model(x, t), and two model(x, t) calls bit-identical."""
    from audio_diffusion_b200.schedulers import DDIMScheduler, DDPMScheduler
    from audio_diffusion_b200.unet import UNet2DModel
    model = UNet2DModel(sample_size=(256, 256), seed=21, **PUBLISHED).to(cuda).eval()
    g = torch.Generator().manual_seed(22)
    x = torch.randn(64, 1, 256, 256, generator=g).to(cuda)
    z = torch.randn(64, 1, 256, 256, generator=g).to(cuda) if kind == "ddpm" else None
    sch = DDPMScheduler() if kind == "ddpm" else DDIMScheduler()
    sch.set_timesteps(1000 if kind == "ddpm" else 50)
    t = int(sch.timesteps[0])
    c = sch.step_coef(t)
    assert (c.c_z != 0) == (kind == "ddpm")
    with torch.no_grad():
        x_out, eps = model.forward_step(x, t, c, noise=z, want_eps=True)
        e1, e2 = model(x, t)["sample"], model(x, t)["sample"]
    ratio, clipped = check_fused_step(c, x, eps, x_out, z)
    spread = (e1 - e2).abs().max().item()
    diff = (eps - e1).abs().max().item()
    print(f"\n{kind} t={t}: x0 clipped for {clipped:.1%} of the elements; max |x_out - ref| / bar {ratio[0]:.3f}; "
          f"eps vs model(x, t) {diff:.3e}, two model(x, t) calls {spread:.3e}")
    if kind == "ddpm":
        assert clipped > 0.05
    assert diff <= spread, (diff, spread)
