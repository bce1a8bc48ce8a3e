"""2-D tiled work items of conv_tc_kernel (8 columns x 32 rows of output pixels) against PyTorch and against the flat items.

Launches with W % 8 == 0 and H % 32 == 0 whose tile windows are smaller than the flat ones (W >= 64 for a 3x3 conv) take
the tiles; B200AD_CONV_DBG=4096 forces flat items, the reference path here.  Each output element sums the same products
in the same order in both shapes, so single-conv outputs must be bitwise identical; the GroupNorm partial sums are grouped
differently, so statistics agree to fp32 rounding, and a full model (whose GroupNorms read those statistics) as closely as a
change of accumulation order in the flat path alone lets it.
"""
import contextlib
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

FLAT = "4096"


@contextlib.contextmanager
def _dbg(value):
    old = os.environ.get("B200AD_CONV_DBG")
    if value is None:
        os.environ.pop("B200AD_CONV_DBG", None)
    else:
        os.environ["B200AD_CONV_DBG"] = value
    try:
        yield
    finally:
        if old is None:
            os.environ.pop("B200AD_CONV_DBG", None)
        else:
            os.environ["B200AD_CONV_DBG"] = old


def _bf(x):
    return x.to(torch.bfloat16).to(torch.float32)


def _run_conv(cuda, x, w, b, te, r, stride):
    from audio_diffusion_b200 import _lib
    L = _lib.lib()
    N, cin, H, W = x.shape
    cout, K = w.shape[0], w.shape[2]
    Ho, Wo = H // stride, W // stride
    d = lambda t: t.to(cuda).contiguous() if t is not None else None
    p = lambda t: t.data_ptr() if t is not None else None
    xd, wd, bd, ted, rd = d(x), d(w), d(b), d(te), d(r)
    y = torch.empty(N, cout, Ho, Wo, device=cuda)
    stats = torch.empty(N, cout // 4, 2, device=cuda)
    nb = L.b200ad_conv2d_scratch_bytes(N, cin, cout, H, W, K, stride)
    scratch = torch.empty(nb, dtype=torch.uint8, device=cuda)
    _lib.check(L.b200ad_conv2d(p(xd), p(wd), p(bd), p(ted), p(rd), p(y), p(stats), N, cin, cout, H, W, K, stride,
                               p(scratch), nb, _lib.stream_ptr()))
    torch.cuda.synchronize()
    return y.cpu(), stats.cpu()


@pytest.mark.parametrize("N,cin,cout,H,W,K,stride,temb,res", [
    (1, 128, 128, 256, 256, 3, 1, True, True),
    (2, 256, 128, 128, 128, 3, 1, True, True),
    (2, 384, 256, 64, 64, 3, 1, False, True),
    (2, 256, 256, 64, 128, 3, 1, True, False),
    (2, 256, 128, 128, 128, 1, 1, False, True),
    (1, 128, 128, 256, 256, 3, 2, False, False),
    (2, 128, 256, 128, 128, 3, 2, False, False),
])
def test_conv_tiles_match_torch_and_flat(cuda, N, cin, cout, H, W, K, stride, temb, res):
    g = torch.Generator().manual_seed(N * 1000 + H + cin)
    x = _bf(torch.randn(N, cin, H, W, generator=g))
    w = _bf(torch.randn(cout, cin, K, K, generator=g) / (cin * K * K) ** 0.5)
    b = torch.randn(cout, generator=g)
    te = torch.randn(N, cout, generator=g) if temb else None
    Ho, Wo = H // stride, W // stride
    r = _bf(torch.randn(N, cout, Ho, Wo, generator=g)) if res else None
    ref = F.conv2d(x, w, b, stride=stride, padding=K // 2)
    if temb:
        ref = ref + te[:, :, None, None]
    if res:
        ref = ref + r
    with _dbg(None):
        y, s = _run_conv(cuda, x, w, b, te, r, stride)
    with _dbg(FLAT):
        y_flat, s_flat = _run_conv(cuda, x, w, b, te, r, stride)
    scale = ref.abs().max().item()
    assert (y - ref).abs().max().item() <= 1.5e-2 * scale
    assert torch.equal(y, y_flat), f"max diff vs flat items {(y - y_flat).abs().max().item()}"
    q = ref.view(N, cout // 4, 4, Ho * Wo)
    s_ref = torch.stack([q.sum(dim=(2, 3)), (q * q).sum(dim=(2, 3))], dim=-1)
    assert (s - s_ref).abs().max().item() <= 2e-2 * s_ref[..., 1].abs().max().item() + 1e-3 * Ho * Wo
    # statistics: the same fp32 values summed in another grouping
    assert torch.allclose(s, s_flat, rtol=1e-4, atol=1e-4 * s_flat[..., 1].abs().max().item())


@pytest.mark.parametrize("silu,N,cin,cout,H,W", [(1, 2, 128, 128, 256, 256), (1, 2, 256, 256, 64, 64),
                                                 (0, 1, 384, 128, 128, 128)])
def test_fused_groupnorm_conv_tiles(cuda, silu, N, cin, cout, H, W):
    """GroupNorm(+SiLU) applied by the transform warps to a 2-D tile's window: zeros outside the image, the affine inside."""
    from audio_diffusion_b200 import _lib
    L = _lib.lib()
    g = torch.Generator().manual_seed(31 + H)
    x = _bf(torch.randn(N, cin, H, W, generator=g) * 1.7 + 0.3)
    gamma = 1 + 0.2 * torch.randn(cin, generator=g)
    beta = 0.2 * torch.randn(cin, generator=g)
    w = _bf(torch.randn(cout, cin, 3, 3, generator=g) / (cin * 9) ** 0.5)
    b = torch.randn(cout, generator=g)
    a = F.group_norm(x, 32, gamma, beta, 1e-5)
    if silu:
        a = F.silu(a)
    ref = F.conv2d(a, w, b, padding=1)
    d = lambda t: t.to(cuda).contiguous()
    xd, gd, bd, wd, biasd = d(x), d(gamma), d(beta), d(w), d(b)
    nb = L.b200ad_conv2d_scratch_bytes(N, cin, cout, H, W, 3, 1)
    scratch = torch.empty(nb, dtype=torch.uint8, device=cuda)
    outs = []
    for mode in (None, FLAT):
        y = torch.empty(N, cout, H, W, device=cuda)
        with _dbg(mode):
            _lib.check(L.b200ad_gn_conv2d(xd.data_ptr(), gd.data_ptr(), bd.data_ptr(), 32, 1e-5, silu, wd.data_ptr(),
                                          biasd.data_ptr(), y.data_ptr(), N, cin, cout, H, W, 3, scratch.data_ptr(), nb,
                                          _lib.stream_ptr()))
            torch.cuda.synchronize()
        outs.append(y.cpu())
    assert (outs[0] - ref).abs().max().item() <= 2.5e-2 * ref.abs().max().item()
    assert torch.equal(outs[0], outs[1]), f"max diff vs flat items {(outs[0] - outs[1]).abs().max().item()}"


@pytest.mark.parametrize("N,cin,cout,H,W,K", [(2, 128, 256, 64, 64, 3), (1, 256, 128, 128, 128, 3)])
def test_conv_dgrad_tiles(cuda, N, cin, cout, H, W, K):
    from audio_diffusion_b200 import _lib
    L = _lib.lib()
    g = torch.Generator().manual_seed(77 + H)
    w = _bf(torch.randn(cout, cin, K, K, generator=g) / (cout * K * K) ** 0.5)
    gy = _bf(torch.randn(N, cout, H, W, generator=g))
    x = torch.zeros(N, cin, H, W, requires_grad=True)
    F.conv2d(x, w, padding=K // 2).backward(gy)
    ref = x.grad
    gyd, wd = gy.to(cuda).contiguous(), w.to(cuda).contiguous()
    nb = L.b200ad_conv2d_scratch_bytes(N, cout, cin, H, W, K, 1)
    scratch = torch.empty(nb, dtype=torch.uint8, device=cuda)
    outs = []
    for mode in (None, FLAT):
        gx = torch.empty(N, cin, H, W, device=cuda)
        with _dbg(mode):
            _lib.check(L.b200ad_conv2d_dgrad(gyd.data_ptr(), wd.data_ptr(), gx.data_ptr(), N, cin, cout, H, W, K,
                                             scratch.data_ptr(), nb, _lib.stream_ptr()))
            torch.cuda.synchronize()
        outs.append(gx.cpu())
    assert (outs[0] - ref).abs().max().item() <= 1.5e-2 * ref.abs().max().item()
    assert torch.equal(outs[0], outs[1])


def _rel(a, b):
    err = a - b
    return (err.abs().max() / b.abs().max()).item(), (err.pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item()


# Bars (rms-rel, max-rel) of tiles against flat items, set by the flat path's own order noise: the flat items with the
# 1-tap k-steps of each conv interleaved between its 3x3 k-steps (a last-bit change of the same kind as regrouped GroupNorm
# partial sums) moved each output by (rms0, mx0) against the flat items; the bar is (max(1.5 rms0, 2e-3), max(2 mx0, 2e-2)).
# Measured on an NVIDIA H100 80GB HBM3 (700 W power limit) with the inputs of the tests below.
BARS_UNET_EPS = (0.01159, 0.02)          # rms0 0.00772, mx0 0.00919
BARS_VAE_MEAN = (0.009258, 0.02122)      # rms0 0.00617, mx0 0.01061
BARS_VAE_DECODE = (0.03208, 0.04575)     # rms0 0.02138, mx0 0.02287


def _check_against_order_noise(run, bars):
    """Tiles against flat items, within the spread that reordering the flat path's accumulation alone produces: through a
    deep net of bf16 activations a last-bit change grows to about 0.75 % rms for the published U-Net at 256 x 256, so the
    tiles must not move the result further than that.  A non-zero pad or guard would add errors along the image borders."""
    tiled = run(None)
    flat = run(FLAT)
    for t, f, (rms_bar, mx_bar) in zip(tiled, flat, bars):
        mx, rms = _rel(t, f)
        assert rms <= rms_bar and mx <= mx_bar, \
            f"tiles vs flat max-rel {mx:.5f} rms-rel {rms:.5f}; bars {mx_bar:.5f} / {rms_bar:.5f}"
        d = (t - f).pow(2).mean(dim=(0, 1)).sqrt()
        H, W = d.shape
        border = torch.zeros(H, W, dtype=torch.bool)
        border[0, :] = border[-1, :] = border[:, 0] = border[:, -1] = True
        assert d[border].pow(2).mean().sqrt() <= 2 * d[~border].pow(2).mean().sqrt() + 1e-6


def test_denoising_step_tiles_vs_flat(cuda):
    """The published U-Net at batch 64, 256 x 256: epsilon with 2-D tiles against forced-flat items."""
    from audio_diffusion_b200.unet import UNet2DModel
    arch = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 128, 256, 256, 512, 512),
                down_block_types=("DownBlock2D",) * 4 + ("AttnDownBlock2D", "DownBlock2D"),
                up_block_types=("UpBlock2D", "AttnUpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D"))
    model = UNet2DModel(sample_size=(256, 256), seed=0, **arch).to(cuda)
    g = torch.Generator(device=cuda).manual_seed(5)
    x = torch.randn(64, 1, 256, 256, generator=g, device=cuda)

    def run(mode):
        with torch.no_grad(), _dbg(mode):
            return (model(x, 500)["sample"].float().cpu(),)
    _check_against_order_noise(run, [BARS_UNET_EPS])


def test_vae_encode_decode_tiles_vs_flat(cuda):
    """The autoencoder at 256 x 256: its asymmetric stride-2 downsample (taps at dh, dw in {0, 1}) and the decoder's convs
    take 2-D tiles at the wide levels."""
    from audio_diffusion_b200.vae import AutoencoderKL
    model = AutoencoderKL(in_channels=1, out_channels=1, latent_channels=1, layers_per_block=2,
                          block_out_channels=(128, 256, 512, 512), down_block_types=("DownEncoderBlock2D",) * 4,
                          up_block_types=("UpDecoderBlock2D",) * 4, seed=0).to(cuda)
    g = torch.Generator(device=cuda).manual_seed(6)
    x = torch.randn(2, 1, 256, 256, generator=g, device=cuda)
    z = torch.randn(2, 1, 32, 32, generator=g, device=cuda)

    def run(mode):
        with torch.no_grad(), _dbg(mode):
            return model.encode(x).latent_dist.mean.float().cpu(), model.decode(z)["sample"].float().cpu()
    _check_against_order_noise(run, [BARS_VAE_MEAN, BARS_VAE_DECODE])
