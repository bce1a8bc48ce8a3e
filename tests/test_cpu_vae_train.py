"""CPU checks of the autoencoder training objective (audio_diffusion_b200.training.vae_loss, the posterior's kl()) and the
derivation of the gradient tolerances of tests/test_gpu_vae_train.py."""
import math

import pytest
import torch


class _Post:
    """The training posterior's torch expressions on given moments (DiagonalGaussianDistribution with train=True)."""

    def __init__(self, moments):
        from audio_diffusion_b200.vae import DiagonalGaussianDistribution
        self.d = DiagonalGaussianDistribution(None, None, train=True)
        self.d._moments = moments

    def __getattr__(self, k):
        return getattr(self.d, k)


def test_vae_loss_matches_ldm_formula():
    """L1 + 1e-6 KL against a literal restatement of ldm's LPIPSWithDiscriminator generator loss before disc_start
    (perceptual weight 0, logvar 0)."""
    from audio_diffusion_b200.training import vae_loss
    g = torch.Generator().manual_seed(0)
    x = torch.rand(3, 1, 16, 16, generator=g) * 2 - 1
    xh = torch.randn(3, 1, 16, 16, generator=g)
    m = torch.randn(3, 2, 2, 2, generator=g) * 3
    post = _Post(m)
    loss, rec, kl = vae_loss(x, xh, post, kl_weight=1e-6)
    logvar0 = torch.zeros(())
    rec_ref = torch.abs(x - xh)
    nll = rec_ref / torch.exp(logvar0) + logvar0
    nll = torch.sum(nll) / nll.shape[0]
    mean, lv = m[:, :1], torch.clamp(m[:, 1:], -30.0, 20.0)
    kl_ref = 0.5 * torch.sum(mean ** 2 + torch.exp(lv) - 1.0 - lv, dim=[1, 2, 3])
    kl_ref = torch.sum(kl_ref) / kl_ref.shape[0]
    assert torch.allclose(loss, nll + 1e-6 * kl_ref, rtol=1e-6)
    assert torch.allclose(rec, rec_ref.mean(), rtol=1e-6)
    assert torch.allclose(kl, kl_ref, rtol=1e-6)


def test_posterior_kl_closed_form_and_clamp():
    """kl() is KL(N(mu, sigma^2) || N(0, 1)) summed over the latent, with logvar clamped to [-30, 20]: clamped entries
    get no gradient."""
    m = torch.tensor([[[[0.5, -1.0]], [[0.3, 40.0]]], [[[2.0, 0.0]], [[-35.0, -2.0]]]], requires_grad=True)
    post = _Post(m)
    kl = post.kl()
    mu, lv = m.detach()[:, 0], m.detach()[:, 1].clamp(-30, 20)
    sig2 = torch.exp(lv)
    ref = 0.5 * (mu ** 2 + sig2 - 1.0 - torch.log(sig2)).flatten(1).sum(1)
    assert torch.allclose(kl, ref, rtol=1e-5)
    kl.sum().backward()
    assert m.grad[0, 1, 0, 1] == 0 and m.grad[1, 1, 0, 0] == 0
    assert m.grad[0, 1, 0, 0] != 0
    assert torch.allclose(post.std, torch.exp(0.5 * post.logvar)) and torch.allclose(post.var, post.std ** 2, rtol=1e-6)
    assert torch.equal(post.mode(), post.mean)


def _floor(fn, w, keep=lambda k: True):
    """Relative L2 of the oracle's gradients with every conv / linear operand and output rounded to bf16, against fp32:
    total over all tensors, and the worst tensor among those with a non-negligible gradient."""
    import torch.nn.functional as F

    from oracle import vae_oracle as vo

    def grads():
        wl = {k: v.clone().requires_grad_(True) for k, v in w.items()}
        out = fn(wl)
        keys = [k for k in wl if wl[k].grad is not None and keep(k)]
        return {k: wl[k].grad for k in keys}, out

    g32, o32 = grads()
    oc, ol = F.conv2d, F.linear
    bf = lambda t: t.to(torch.bfloat16).to(torch.float32)
    vo.F.conv2d = lambda a, ww, b=None, **k: bf(oc(bf(a), bf(ww), b, **k))
    vo.F.linear = lambda a, ww, b=None: bf(ol(bf(a), bf(ww), b))
    try:
        g16, o16 = grads()
    finally:
        vo.F.conv2d, vo.F.linear = oc, ol
    num = den = 0.0
    gmax = max(g.norm().item() for g in g32.values())
    worst = 0.0
    for k in g32:
        e, s = (g16[k] - g32[k]).norm().item(), g32[k].norm().item()
        num += e * e
        den += s * s
        if s > 1e-3 * gmax:
            worst = max(worst, e / s)
    return math.sqrt(num / den), worst, o32, o16


def test_vae_backward_bf16_gradient_floor():
    """The floor the GPU gradient bars are stated from (tests/test_gpu_vae_train.py), at those tests' shapes (full ldm
    architecture, 64x64, batch 2): decoder backward from a seeded image gradient, encoder backward from seeded moment
    gradients.  Printed: total relative L2 and the worst non-negligible tensor."""
    from oracle import vae_oracle as vo
    cfg = vo.VAEConfig()
    w = vo.init_weights(cfg, seed=0)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 1, 64, 64, generator=g).clamp(-1, 1)
    z = torch.randn(2, 1, 8, 8, generator=g)
    gx = torch.randn(2, 1, 64, 64, generator=g)
    gm = torch.randn(2, 2, 8, 8, generator=g)

    def dec(wl):
        zz = z.clone().requires_grad_(True)
        (vo.decode(wl, cfg, zz) * gx).sum().backward()
        return zz.grad

    def enc(wl):
        (vo.encode_moments(wl, cfg, x) * gm).sum().backward()
        return None

    td, wd, gz32, gz16 = _floor(dec, w)
    te, we, _, _ = _floor(enc, w)
    rz = ((gz16 - gz32).norm() / gz32.norm()).item()
    print(f"bf16 floor: decoder total {td:.4f} worst {wd:.4f} g_z {rz:.4f}; encoder total {te:.4f} worst {we:.4f}")
    # measured: decoder total 3.5 %, worst 8.8 %, g_z 3.5 %; encoder total 2.4 %, worst 3.1 %.  The GPU bars are about
    # twice that (the engine's activation gradients are bf16 too, which this floor does not round): decoder and g_z 8 %,
    # encoder 6 %, every non-negligible tensor 25 %.
    assert td < 4e-2 and rz < 4e-2 and te < 3e-2
    assert wd < 0.125 and we < 0.125


def test_vae_loss_bf16_gradient_floor_256():
    """The same floor for the whole objective (L1 + 1e-6 KL through the sampled posterior) at 256x256, batch 1, the shape
    of tests/test_gpu_vae_train.py::test_vae_loss_step_matches_oracle_256.  The L1 gradient is sign(x_hat - x): bf16
    error in x_hat flips it wherever the reconstruction is close, and the encoder receives all of that through g_z."""
    from oracle import vae_oracle as vo
    cfg = vo.VAEConfig()
    w = vo.init_weights(cfg, seed=3)
    x = torch.rand(1, 1, 256, 256, generator=torch.Generator().manual_seed(4)) * 2 - 1
    noise = torch.randn(1, 1, 32, 32, generator=torch.Generator().manual_seed(5))

    def full(wl):
        mean, lv = torch.chunk(vo.encode_moments(wl, cfg, x), 2, dim=1)
        lv = lv.clamp(-30.0, 20.0)
        y = vo.decode(wl, cfg, mean + torch.exp(0.5 * lv) * noise)
        (torch.abs(x - y).sum() + 1e-6 * 0.5 * torch.sum(mean ** 2 + torch.exp(lv) - 1.0 - lv)).backward()
        return None

    enc = lambda k: k.startswith(("encoder.", "quant_conv."))
    te, we, _, _ = _floor(full, w, keep=enc)
    td, wd, _, _ = _floor(full, w, keep=lambda k: not enc(k))
    print(f"bf16 floor, whole objective at 256x256: decoder total {td:.4f} worst {wd:.4f}; encoder total {te:.4f} "
          f"worst {we:.4f}")
    # measured: decoder 1.9 % (worst 6.1 %), encoder 7.0 % (worst 8.5 %).  GPU bars: decoder 8 %, encoder 14 %, every
    # non-negligible tensor 30 % (bias gradients are sums over pixels of signed, partly cancelling terms).
    assert td < 4e-2 and te < 8e-2
