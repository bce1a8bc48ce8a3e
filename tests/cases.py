"""What the tests run: the architectures, the timesteps, the engine models built from the oracle's weights, the seeded
inputs of a training step, and the constants more than one test module reads (the recorded training-memory sizes and the
bars of the per-block fp64 checks that tests/test_cpu_block_backward.py states from its floors)."""
import torch

# scripts/train_unet.py's UNet2DModel: six levels, attention at the fifth
PUBLISHED = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 128, 256, 256, 512, 512),
                 down_block_types=("DownBlock2D",) * 4 + ("AttnDownBlock2D", "DownBlock2D"),
                 up_block_types=("UpBlock2D", "AttnUpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D"))
# the same U-Net over a hub VAE's four latent channels (scripts/train_unet.py --vae: in = out = latent_channels)
PUBLISHED4 = dict(PUBLISHED, in_channels=4, out_channels=4)
# scripts/train_unet.py's UNet2DConditionModel (--encodings): transformers in three down and three up blocks
PUBLISHED_COND = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256, 512, 512),
                      down_block_types=("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",),
                      up_block_types=("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3, cross_attention_dim=100)
# two levels (128, 256), attention at the second: every block kind of the published U-Net at a small scale
TWO_LEVEL = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256),
                 down_block_types=("DownBlock2D", "AttnDownBlock2D"), up_block_types=("AttnUpBlock2D", "UpBlock2D"))
# two levels, transformers (head_dim 16) in the first down and the last up block
TWO_LEVEL_COND = dict(PUBLISHED_COND, block_out_channels=(128, 256),
                      down_block_types=("CrossAttnDownBlock2D", "DownBlock2D"),
                      up_block_types=("UpBlock2D", "CrossAttnUpBlock2D"))
# config/ldm_autoencoder_kl.yaml as an AutoencoderKL: 1-channel image, 1-channel latent, /8 (oracle.vae_oracle.VAEConfig)
LDM = dict(in_channels=1, out_channels=1, latent_channels=1, layers_per_block=2, block_out_channels=(128, 256, 512, 512),
           down_block_types=("DownEncoderBlock2D",) * 4, up_block_types=("UpDecoderBlock2D",) * 4)

T3 = [37, 412, 903]              # three distinct timesteps: batch 3, so per-sample sums must pick the right (odd) sample
T5 = [37, 211, 412, 650, 903]    # five distinct timesteps: per-sample sums over an odd batch with a one-image last item

# the conditional U-Net's transformer parameters whose gradients are exactly zero with a one-token encoding: the softmax
# over one key is constant
ONE_TOKEN_ZERO = ("attn2.to_q.weight", "attn2.to_k.weight", "norm2.weight", "norm2.bias")
# the published U-Net's attention blocks
PUBLISHED_ATTN = (["down_blocks.4.attentions.0", "down_blocks.4.attentions.1", "mid_block.attentions.0"]
                  + [f"up_blocks.1.attentions.{j}" for j in range(3)])


def oracle_config(arch, size=None):
    """The oracle's config of `arch` at sample size `size` (the autoencoder: VAEConfig, which is LDM)."""
    if "latent_channels" in arch:
        from oracle.vae_oracle import VAEConfig
        return VAEConfig()
    if "cross_attention_dim" in arch:
        from oracle.unet_cond_oracle import CondUNetConfig
        return CondUNetConfig(sample_size=size, **arch)
    from oracle.unet_oracle import UNetConfig
    return UNetConfig(sample_size=size, **arch)


def build(arch, seed, dev, size=None, train=True, max_batch=16):
    """The engine model of `arch` with the oracle's init_weights(seed) loaded, on dev, in train() or eval():
    (model, oracle config, w).  A U-Net at sample size `size` (UNet2DConditionModel when `arch` has
    cross_attention_dim); LDM: the autoencoder, its activations bound for up to max_batch images."""
    cfg = oracle_config(arch, size)
    if "latent_channels" in arch:
        from audio_diffusion_b200.vae import AutoencoderKL
        from oracle.vae_oracle import init_weights
        model = AutoencoderKL(max_batch=max_batch, **arch)
    elif "cross_attention_dim" in arch:
        from audio_diffusion_b200.unet_cond import UNet2DConditionModel
        from oracle.unet_cond_oracle import init_weights
        model = UNet2DConditionModel(sample_size=size, **arch)
    else:
        from audio_diffusion_b200.unet import UNet2DModel
        from oracle.unet_oracle import init_weights
        model = UNet2DModel(sample_size=size, **arch)
    w = init_weights(cfg, seed=seed)
    model.load_state_dict(w)
    return model.to(dev).train(train), cfg, w


def w64(w, dev):
    return {k: v.to(device=dev, dtype=torch.float64) for k, v in w.items()}


def draw(n, size, seed, s=None, c=1):
    """The seeded inputs of a training step on weights of `seed`: clean c-channel images in [-1, 1), the noise and (s
    tokens) an encoding, drawn in that order from Generator(seed + 1)."""
    g = torch.Generator().manual_seed(seed + 1)
    clean = torch.rand(n, c, *size, generator=g) * 2 - 1
    noise = torch.randn(n, c, *size, generator=g)
    enc = None if s is None else torch.randn(n, s, 100, generator=g)
    return clean, noise, enc


def train_step(model, size, n, seed, t, s=None):
    """One seeded training step of an engine U-Net: draw()'s inputs noised by the oracle's DDPM at the timesteps t, the
    forward and the MSE backward.  Returns (noisy, t, enc, noise, eps, g_eps) on the model's device: eps the prediction,
    g_eps = dL/deps."""
    from oracle.schedulers_oracle import OracleDDPM
    dev = next(model.parameters()).device
    clean, noise, enc = draw(n, size, seed, s)
    t = torch.tensor(t)
    noisy = OracleDDPM().add_noise(clean, noise, t).to(dev)
    t, noise = t.to(dev), noise.to(dev)
    if enc is None:
        pred = model(noisy, t)["sample"]
    else:
        enc = enc.to(dev)
        pred = model(noisy, t, enc)["sample"]
    torch.nn.functional.mse_loss(pred, noise).backward()
    eps = pred.detach()
    return noisy, t, enc, noise, eps, 2 * (eps - noise) / eps.numel()


# Training workspace + backward arena in bytes before gradient checkpointing was added (every activation kept).
PLAIN_BYTES = {
    "published": 17092031744,   # UNet2DModel 256x256, batch 16
    "cond": 93601632512,        # UNet2DConditionModel 256x256, batch 16, S = 1
    "ldm": 9459353856,          # AutoencoderKL 256x256, batch 8
}


def model_256(which):
    if which == "published":
        from audio_diffusion_b200.unet import UNet2DModel
        return UNet2DModel(sample_size=(256, 256), **PUBLISHED)
    if which == "cond":
        from audio_diffusion_b200.unet_cond import UNet2DConditionModel
        return UNet2DConditionModel(sample_size=(256, 256), **PUBLISHED_COND)
    from audio_diffusion_b200.vae import AutoencoderKL
    return AutoencoderKL(**LDM)


def training_bytes(m, which):
    from audio_diffusion_b200 import _lib
    L = _lib.lib()
    if which == "ldm":
        return L.b200ad_vae_training_bytes(m._h, 8, 256, 256)
    return L.b200ad_unet_training_bytes(m._h, 16, 256, 256, 1)


# Per-block backward bars, kind -> ((activation a, b, c), (parameter a, b, c)), of tests/test_gpu_block_backward.py:
# the two-level U-Net and conditional U-Net at 32x32, batch 3, and the ldm autoencoder at 64x64, batch 2.
UNET_BARS = {
    "head": ((0.005, 0.005, 0.005), (0.005, 0.005, 0.005)),   # floor (0.0, 0.0, 0.0) | (0.0, 0.0, 0.0)
    "resnet": ((0.0126, 0.0213, 0.0126), (0.0105, 0.0114, 0.0948)),   # floor (0.0042, 0.0071, 0.0042) | (0.0035, 0.0038, 0.0316)
    "down": ((0.0069, 0.0072, 0.0066), (0.005, 0.005, 0.005)),   # floor (0.0023, 0.0024, 0.0022) | (0.0, 0.0, 0.0)
    "attn": ((0.005, 0.009, 0.005), (0.0123, 0.0153, 0.0906)),   # floor (0.0017, 0.003, 0.0017) | (0.0041, 0.0051, 0.0302)
    "up": ((0.0087, 0.0116, 0.0084), (0.005, 0.005, 0.005)),   # floor (0.0029, 0.0039, 0.0028) | (0.0, 0.0, 0.0)
    "tail": ((0.0072, 0.0134, 0.0069), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.0045, 0.0023) | (0.0002, 0.0003, 0.0002)
    "temb": ((0.005, 0.005, 0.005), (0.006, 0.0066, 0.0843)),   # floor (0.0, 0.0, 0.0) | (0.002, 0.0022, 0.0281)
}
COND_BARS = {
    "head": ((0.005, 0.005, 0.005), (0.005, 0.005, 0.005)),   # floor (0.0, 0.0, 0.0) | (0.0, 0.0, 0.0)
    "resnet": ((0.0126, 0.0269, 0.0126), (0.0123, 0.0141, 0.0714)),   # floor (0.0042, 0.009, 0.0042) | (0.0041, 0.0047, 0.0238)
    "transformer": ((0.009, 0.0098, 0.0096), (0.0222, 0.0213, 0.1023)),   # floor (0.003, 0.0033, 0.0032) | (0.0074, 0.0071, 0.0341)
    "down": ((0.0069, 0.0096, 0.0066), (0.005, 0.005, 0.005)),   # floor (0.0023, 0.0032, 0.0022) | (0.0, 0.0, 0.0)
    "up": ((0.0087, 0.0114, 0.0084), (0.005, 0.005, 0.005)),   # floor (0.0029, 0.0038, 0.0028) | (0.0, 0.0, 0.0)
    "tail": ((0.0072, 0.0141, 0.0072), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.0047, 0.0024) | (0.0002, 0.0003, 0.0002)
    "temb": ((0.005, 0.005, 0.005), (0.0069, 0.0087, 0.0672)),   # floor (0.0, 0.0, 0.0) | (0.0023, 0.0029, 0.0224)
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
# ... and of tests/test_gpu_block_backward_trained.py, which tests/test_gpu_block_backward_checkpointed.py holds the
# checkpointed backward to: the published U-Net at 64x64, batch 5, the ldm autoencoder at 256x256, batch 2, and the
# published conditional U-Net at 64x64, batch 2
UNET64_BARS = {
    "head": ((0.005, 0.005, 0.005), (0.005, 0.005, 0.005)),   # floor (0.0, 0.0, 0.0) | (0.0, 0.0, 0.0)
    "resnet": ((0.0132, 0.0204, 0.0171), (0.015, 0.0201, 0.0651)),   # floor (0.0044, 0.0068, 0.0057) | (0.005, 0.0067, 0.0217)
    "down": ((0.0072, 0.009, 0.0072), (0.005, 0.005, 0.005)),   # floor (0.0024, 0.003, 0.0024) | (0.0, 0.0, 0.0)
    "attn": ((0.0066, 0.0093, 0.0078), (0.0174, 0.0201, 0.0615)),   # floor (0.0022, 0.0031, 0.0026) | (0.0058, 0.0067, 0.0205)
    "up": ((0.0087, 0.0132, 0.0096), (0.005, 0.005, 0.005)),   # floor (0.0029, 0.0044, 0.0032) | (0.0, 0.0, 0.0)
    "tail": ((0.0069, 0.0123, 0.0069), (0.005, 0.005, 0.005)),   # floor (0.0023, 0.0041, 0.0023) | (0.0001, 0.0002, 0.0001)
    "temb": ((0.005, 0.005, 0.005), (0.006, 0.0063, 0.0618)),   # floor (0.0, 0.0, 0.0) | (0.002, 0.0021, 0.0206)
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
    "temb": ((0.005, 0.005, 0.005), (0.006, 0.006, 0.0765)),   # floor (0.0, 0.0, 0.0) | (0.002, 0.002, 0.0255)
}
# the two-level conditional U-Net's transformers with an S-token encoding (tests/test_gpu_cond_seq.py)
# S -> the transformer's (activation a, b, c), (parameter a, b, c): 3 x the bf16 floor (at least 0.5 %)
COND_SEQ_BWD_TRANSFORMER_BARS = {
    3: ((0.009, 0.0147, 0.0096), (0.0225, 0.0282, 0.0855)),   # floor (0.003, 0.0049, 0.0032) | (0.0075, 0.0094, 0.0285)
    77: ((0.009, 0.0111, 0.0093), (0.0216, 0.0204, 0.0948)),   # floor (0.003, 0.0037, 0.0031) | (0.0072, 0.0068, 0.0316)
}
