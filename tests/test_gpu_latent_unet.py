"""The published UNet2DModel at its 32x32 latent, as latent audio diffusion runs it (scripts/train_unet.py --vae builds it
with sample_size = latent_resolution and in = out = the autoencoder's latent channels; bench.py's C4 samples it at batch
128), checked block by block against fp64 as tests/test_gpu_block_forward.py and tests/test_gpu_block_backward_trained.py
check the pixel shapes, and the autoencoder's chunked decode of C4's 128 latents.

At 32x32 the six levels are 32, 16, 8, 4, 2 and 1, which reaches code the pixel shapes do not:
* a 1x1 bottom level (down block 5, the mid block, up block 0): every 3x3 conv reads eight pad taps and one real one,
  each GroupNorm group is 16 channels of one pixel;
* the stride-2 conv from 2x2 to 1x1 and the folded upsample from 1x1 to 2x2;
* attention over 4 tokens (down block 4, up block 1) and over 1 token (the mid block), both on the SIMT attention_kernel
  and attention_bwd_kernel.  Over one token the softmax is identically 1: the attention output is V bit for bit, and
  the to_q / to_k gradients are exactly zero;
* batch 128: the 8x8 .. 1x1 levels pack up to four images per conv work item over 128 samples, and the time embeddings
  of repeated timesteps are shared (temb_lead);
* four latent channels (a hub VAE's): the generic conv_in_kernel instead of the 1-channel one, and conv_out_kernel
  writing 4 planes of eps and of the fused scheduler update.
The single kernels of these levels (the 2x2 -> 1x1 stride-2 conv, the folded upsamples from 1x1 and 2x2, GroupNorm at
1x1, at batch 128 and at an odd batch) are checked through the C ABI in tests/test_gpu_ops.py.

Bars: the rule of the neighbouring tests.  The floors are measured in the same run on the fp64 oracle's own activations
(block_grads.forward_floors / backward_floors) and every bar lies in (floor, 3.3 x floor] (backward: or at 0.5 %); the
floors are in the comments beside the bars.
"""
import pytest
import torch

from blockcheck import check_fused_step, forward_case, pooled_eps, unet_backward_case
from cases import LDM, PUBLISHED, PUBLISHED4, PUBLISHED_ATTN, T5, TWO_LEVEL_COND, build

pytestmark = pytest.mark.gpu

LATENT = (32, 32)
LEVELS = [(32 >> i, 32 >> i) for i in range(6)]
MID_ATTN = "mid_block.attentions.0"
# over one token no gradient reaches q or k (to_k.bias never gets one)
ONE_TOKEN_ATTN_ZERO = ("to_q.weight", "to_q.bias", "to_k.weight")

# key -> (a, b, c), three times the floor printed beside it
FWD128_BARS = {
    "attn": (0.00912, 0.01395, 0.01233),   # floor (0.00304, 0.00465, 0.00411)
    "attn.ao": (0.00498, 0.00867, 0.00648),   # floor (0.00166, 0.00289, 0.00216)
    "attn.out": (0.00786, 0.01254, 0.01254),   # floor (0.00262, 0.00418, 0.00418)
    "attn.qkv": (0.00879, 0.01137, 0.01254),   # floor (0.00293, 0.00379, 0.00418)
    "down": (0.00726, 0.01083, 0.00954),   # floor (0.00242, 0.00361, 0.00318)
    "head": (0.00498, 0.00738, 0.00468),   # floor (0.00166, 0.00246, 0.00156)
    "resnet": (0.01266, 0.02025, 0.02445),   # floor (0.00422, 0.00675, 0.00815)
    "resnet.h1": (0.01029, 0.02061, 0.01707),   # floor (0.00343, 0.00687, 0.00569)
    "resnet.h1:mean": (0.05706, 0.05706, 0.05706),   # floor (0.01902, 0.01902, 0.01902)
    "resnet.out": (0.00996, 0.01731, 0.01608),   # floor (0.00332, 0.00577, 0.00536)
    "tail": (0.00702, 0.00849, 0.00669),   # floor (0.00234, 0.00283, 0.00223)
    "up": (0.00729, 0.01011, 0.0084),   # floor (0.00243, 0.00337, 0.0028)
}
FWD4_BARS = {
    "attn": (0.009, 0.01326, 0.01119),   # floor (0.003, 0.00442, 0.00373)
    "attn.ao": (0.00504, 0.00879, 0.00657),   # floor (0.00168, 0.00293, 0.00219)
    "attn.out": (0.00759, 0.01218, 0.01092),   # floor (0.00253, 0.00406, 0.00364)
    "attn.qkv": (0.00885, 0.01182, 0.01119),   # floor (0.00295, 0.00394, 0.00373)
    "down": (0.00729, 0.01119, 0.01047),   # floor (0.00243, 0.00373, 0.00349)
    "head": (0.00498, 0.00783, 0.00465),   # floor (0.00166, 0.00261, 0.00155)
    "resnet": (0.01284, 0.01986, 0.01926),   # floor (0.00428, 0.00662, 0.00642)
    "resnet.h1": (0.0102, 0.01659, 0.01647),   # floor (0.0034, 0.00553, 0.00549)
    "resnet.h1:mean": (0.05559, 0.05559, 0.05559),   # floor (0.01853, 0.01853, 0.01853)
    "resnet.out": (0.01005, 0.01722, 0.01428),   # floor (0.00335, 0.00574, 0.00476)
    "tail": (0.00762, 0.01092, 0.00714),   # floor (0.00254, 0.00364, 0.00238)
    "up": (0.00717, 0.01002, 0.0081),   # floor (0.00239, 0.00334, 0.0027)
}
# kind -> ((activation a, b, c), (parameter a, b, c)), and the training forward key -> (a, b, c)
BWD_BARS = {
    "head": ((0.005, 0.005, 0.005), (0.005, 0.005, 0.005)),   # floor (0.0, 0.0, 0.0) | (0.0, 0.0, 0.0)
    "resnet": ((0.0132, 0.021, 0.0273), (0.0147, 0.0183, 0.0801)),   # floor (0.0044, 0.007, 0.0091) | (0.0049, 0.0061, 0.0267)
    "down": ((0.0072, 0.0099, 0.0087), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.0033, 0.0029) | (0.0, 0.0, 0.0)
    "attn": ((0.0093, 0.0114, 0.0204), (0.0177, 0.0228, 0.0468)),   # floor (0.0031, 0.0038, 0.0068) | (0.0059, 0.0076, 0.0156)
    "up": ((0.009, 0.0117, 0.015), (0.005, 0.005, 0.005)),   # floor (0.003, 0.0039, 0.005) | (0.0, 0.0, 0.0)
    "tail": ((0.0072, 0.0138, 0.0072), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.0046, 0.0024) | (0.0001, 0.0001, 0.0001)
    "temb": ((0.005, 0.005, 0.005), (0.0066, 0.0069, 0.078)),   # floor (0.0, 0.0, 0.0) | (0.0022, 0.0023, 0.026)
}
BWD_FWD_BARS = {
    "attn": (0.00906, 0.01482, 0.01257),   # floor (0.00302, 0.00494, 0.00419)
    "attn.ao": (0.00498, 0.00816, 0.00657),   # floor (0.00166, 0.00272, 0.00219)
    "attn.out": (0.00777, 0.01287, 0.01188),   # floor (0.00259, 0.00429, 0.00396)
    "attn.qkv": (0.00888, 0.01188, 0.01092),   # floor (0.00296, 0.00396, 0.00364)
    "down": (0.00729, 0.01131, 0.01098),   # floor (0.00243, 0.00377, 0.00366)
    "head": (0.00498, 0.00732, 0.00474),   # floor (0.00166, 0.00244, 0.00158)
    "resnet": (0.01287, 0.02085, 0.01983),   # floor (0.00429, 0.00695, 0.00661)
    "resnet.h1": (0.0102, 0.01887, 0.01692),   # floor (0.0034, 0.00629, 0.00564)
    "resnet.h1:mean": (0.05739, 0.05739, 0.05739),   # floor (0.01913, 0.01913, 0.01913)
    "resnet.out": (0.01002, 0.01863, 0.01719),   # floor (0.00334, 0.00621, 0.00573)
    "tail": (0.00939, 0.01101, 0.00963),   # floor (0.00313, 0.00367, 0.00321)
    "up": (0.00726, 0.01074, 0.0084),   # floor (0.00242, 0.00358, 0.0028)
}


def _levels(model):
    return [tuple(model.debug_tensor(f"down_blocks.{i}.resnets.0").shape[2:]) for i in range(len(LEVELS))]


@pytest.mark.timeout(900)
def test_latent_unet_batch128_forward_per_block(cuda, monkeypatch):
    """C4's latent U-Net step, batch 128, t_i = 999 - 7 (i mod 13): samples 0 and 1 (the first packed item), 13 (sample
    0's timestep again) and 124 - 127 (the last packed item of the 1x1 level) compared block by block.  The same input
    through the pooled buffers gives the same eps as two pooled runs give each other; over one token the mid block's
    attention output (`.ao`) is the V third of its `.qkv` bit for bit.  Measured on an H100 80GB HBM3 at 700 W:
    pooled and unpooled eps bit-identical; fp64 work 1.3 s, 8.5 GiB peak device memory."""
    sel = [0, 1, 13, 124, 125, 126, 127]
    t = [999 - 7 * (i % 13) for i in range(128)]
    x, tt, w, eps = forward_case(cuda, monkeypatch, PUBLISHED, LATENT, 128, 23, FWD128_BARS, t=t, sel=sel)
    model = build(PUBLISHED, 23, cuda, LATENT, train=False)[0]       # still unpooled: every tap in its own buffer
    with torch.no_grad():
        again = model(x, tt)["sample"]
    assert _levels(model) == LEVELS
    assert model.debug_tensor(MID_ATTN).shape[2:] == (1, 1)
    ao, qkv = model.debug_tensor(MID_ATTN + ".ao"), model.debug_tensor(MID_ATTN + ".qkv")
    c = ao.shape[1]
    assert qkv.shape[1] == 3 * c
    assert torch.equal(ao, qkv[:, 2 * c:]), (ao - qkv[:, 2 * c:]).abs().max().item()
    del model
    monkeypatch.delenv("B200AD_DEBUG_NOPOOL")
    torch.cuda.empty_cache()
    e1, e2 = pooled_eps(cuda, PUBLISHED, w, LATENT, x, tt)
    spread = (e1 - e2).abs().max().item()
    diff = max((e1 - eps).abs().max().item(), (again - eps).abs().max().item())
    print(f"pooled vs unpooled eps: max |diff| {diff:.3e}; two pooled runs: {spread:.3e}")
    assert diff <= spread, (diff, spread)


@pytest.mark.timeout(600)
@pytest.mark.parametrize("kind", ["ddpm", "ddim"])
def test_latent_fused_step_batch128(cuda, kind):
    """The fused scheduler update at C4's shape (32x32, batch 128, pooled buffers): one DDPM step with noise at t = 999,
    where the x0 clip is active, and one DDIM step (eta = 0, 50 steps), x_out against the fp64 update
    (blockcheck.check_fused_step); eps of the fused step equal to model(x, t), or within what two model(x, t) calls
    differ by.  Measured on an H100 80GB HBM3 at 700 W: x0 clipped for 99.5 % (DDPM) and 99.4 % (DDIM) of the elements;
    the largest error 0.22 and 0.09 of its bar; eps bit-identical to model(x, t)."""
    from audio_diffusion_b200.schedulers import DDIMScheduler, DDPMScheduler
    from audio_diffusion_b200.unet import UNet2DModel
    model = UNet2DModel(sample_size=LATENT, seed=29, **PUBLISHED).to(cuda).eval()
    g = torch.Generator().manual_seed(30)
    x = torch.randn(128, 1, *LATENT, generator=g).to(cuda)
    z = torch.randn(128, 1, *LATENT, generator=g).to(cuda) if kind == "ddpm" else None
    sch = DDPMScheduler() if kind == "ddpm" else DDIMScheduler()
    sch.set_timesteps(1000 if kind == "ddpm" else 50)
    t = int(sch.timesteps[0])
    c = sch.step_coef(t)
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


@pytest.mark.timeout(900)
def test_latent_unet_backward_per_block(cuda):
    """The latent training step: batch 16 (train_unet.py's train_batch_size) at 16 distinct timesteps, every block's
    input and parameter gradients and the timestep MLP's against fp64, and the training forward block by block.  The
    mid block attends over one token: its to_q.weight, to_q.bias and to_k.weight gradients are exactly zero, while the
    2x2 attention blocks' are not.  H100 80GB HBM3, 700 W: fp64 work 5.4 s for the backward and 6.7 s with the
    training forward, 5.8 GiB peak."""
    t = [37 + 61 * i for i in range(16)]
    model, blocks = unet_backward_case(cuda, PUBLISHED, LATENT, 16, 27, t, BWD_BARS, floors=True, fwd_bars=BWD_FWD_BARS)
    assert [b.name for b in blocks if b.kind == "attn"] == PUBLISHED_ATTN
    assert _levels(model) == LEVELS
    named = dict(model.named_parameters())
    for blk in PUBLISHED_ATTN:
        for k in ONE_TOKEN_ATTN_ZERO:
            nz = torch.count_nonzero(named[f"{blk}.{k}"].grad).item()
            assert (nz == 0) == (blk == MID_ATTN), (blk, k, nz)


@pytest.mark.timeout(900)
def test_latent_unet_4ch(cuda, monkeypatch):
    """The published U-Net over four latent channels at 32x32, batch 5 (the last packed item part-full): the forward
    block by block (the head on the generic conv_in_kernel, the tail writing 4 planes), a fused DDPM step with 4-plane
    noise against the fp64 update on every plane, eps of forward_step(want_eps=True) equal to model(x, t) on all planes,
    and the training forward refused (the backward is 1-channel only).  H100 80GB HBM3, 700 W: fp64 work 0.7 s, 1.9 GiB
    peak; x_out within 0.20 - 0.21 of its bar on every plane, eps bit-identical to model(x, t)."""
    from audio_diffusion_b200 import _lib
    from audio_diffusion_b200.schedulers import DDPMScheduler
    from audio_diffusion_b200.unet import UNet2DModel
    x, tt, w, eps = forward_case(cuda, monkeypatch, PUBLISHED4, LATENT, 5, 25, FWD4_BARS, t=T5, sel=list(range(5)))
    assert x.shape[1] == eps.shape[1] == 4
    monkeypatch.delenv("B200AD_DEBUG_NOPOOL")
    torch.cuda.empty_cache()
    model = UNet2DModel(sample_size=LATENT, **PUBLISHED4)
    model.load_state_dict(w)
    model = model.to(cuda).eval()
    sch = DDPMScheduler()
    sch.set_timesteps(1000)
    t = int(sch.timesteps[0])
    c = sch.step_coef(t)
    z = torch.randn(5, 4, *LATENT, generator=torch.Generator().manual_seed(26)).to(cuda)
    with torch.no_grad():
        x_out, e_step = model.forward_step(x, t, c, noise=z, want_eps=True)
        e1, e2 = model(x, t)["sample"], model(x, t)["sample"]
    ratio, clipped = check_fused_step(c, x, e_step, x_out, z)
    spread = (e1 - e2).abs().max().item()
    diff = [(e_step[:, p] - e1[:, p]).abs().max().item() for p in range(4)]
    print(f"\n4 channels, ddpm t={t}: x0 clipped for {clipped:.1%}; max |x_out - ref| / bar per plane "
          f"{[round(r, 3) for r in ratio]}; eps vs model(x, t) per plane {diff}, two model(x, t) calls {spread:.3e}")
    assert len(ratio) == 4 and clipped > 0.05
    assert max(diff) <= spread, (diff, spread)
    assert all(e1[:, p].abs().max() > 0 for p in range(4))
    model.train()
    with pytest.raises(_lib.B200ADError, match="channels != 1 is not implemented"):
        model(x, tt)["sample"].sum().backward()


@pytest.mark.timeout(600)
def test_mismatched_shapes_refused(cuda):
    """A sample whose channels differ from in_channels, and noise or an output of another shape than the sample, are
    refused with ValueError before anything is bound or launched (conv_in would read planes past the sample, and the
    fused step would write eps planes past `out`), by every entry point: forward, forward_step, graph_stepper and its
    step, and the conditional model's forward.  The model still gives the same answer afterwards."""
    from audio_diffusion_b200.schedulers import DDPMScheduler
    from audio_diffusion_b200.unet import UNet2DModel
    from audio_diffusion_b200.unet_cond import UNet2DConditionModel
    model = UNet2DModel(sample_size=LATENT, seed=31, **PUBLISHED4).to(cuda).eval()
    g = torch.Generator().manual_seed(32)
    x = torch.randn(3, 4, *LATENT, generator=g).to(cuda)
    z = torch.randn(3, 4, *LATENT, generator=g).to(cuda)
    sch = DDPMScheduler()
    sch.set_timesteps(1000)
    c = sch.step_coef(999)
    with torch.no_grad():
        ref = model(x, 999)["sample"]
        ref_step = model.forward_step(x, 999, c, noise=z)
        x1, z1 = x[:, :1].contiguous(), z[:, :1].contiguous()
        with pytest.raises(ValueError, match="sample must be"):
            model(x1, 999)
        with pytest.raises(ValueError, match="sample must be"):
            model.forward_step(x1, 999, c)
        with pytest.raises(ValueError, match="sample must be"):
            model.graph_stepper(x1)
        with pytest.raises(ValueError, match="noise must be"):
            model.forward_step(x, 999, c, noise=z1)
        with pytest.raises(ValueError, match="noise must be"):
            model.forward_step(x, 999, c, noise=z[:2])
        with pytest.raises(ValueError, match="out must be"):
            model.forward_step(x, 999, c, out=torch.empty_like(x1))
        with pytest.raises(ValueError, match="out must be"):
            model.forward_step(x, 999, c, out=torch.empty(3, 4, 32, 16, device=cuda))
        st = model.graph_stepper(x)
        with pytest.raises(ValueError, match="noise must have"):
            st.step(999, c, z1)
        assert torch.equal(st.x, x)
        assert torch.equal(model(x, 999)["sample"], ref)
        assert torch.equal(model.forward_step(x, 999, c, noise=z), ref_step)
        assert torch.equal(st.step(999, c, z), ref_step)
        cond = UNet2DConditionModel(sample_size=LATENT, seed=33, **TWO_LEVEL_COND).to(cuda).eval()
        enc = torch.randn(3, 1, 100, generator=g).to(cuda)
        with pytest.raises(ValueError, match="sample must be"):
            cond(x, 999, enc)
        with pytest.raises(ValueError, match="sample must be"):
            cond.forward_step(x, 999, c, enc)
        assert cond(x1, 999, enc)["sample"].shape == x1.shape


@pytest.mark.timeout(600)
def test_latent_decode_chunks(cuda):
    """C4's decode: AutoencoderKL.decode of 128 latents (32x32) runs in chunks of max_batch = 16; each image is bitwise
    equal to decoding its chunk alone.  Then 20 latents, whose last chunk holds 4."""
    model = build(LDM, 35, cuda, train=False, max_batch=16)[0]
    g = torch.Generator().manual_seed(36)
    for n in (128, 20):
        z = torch.randn(n, 1, *LATENT, generator=g).to(cuda)
        with torch.no_grad():
            img = model.decode(z).sample
            assert img.shape == (n, 1, 256, 256)
            for s in range(0, n, 16):
                alone = model.decode(z[s:s + 16]).sample
                assert torch.equal(img[s:s + 16], alone), (n, s, (img[s:s + 16] - alone).abs().max().item())
