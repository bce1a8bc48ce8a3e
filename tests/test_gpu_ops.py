"""GPU parity of single kernels (through the C ABI) against plain PyTorch on the CPU (fp64 for the conv, folded-upsample
and GroupNorm kernels, fp32 for the others).

Tolerances: operands are rounded to bf16 on both sides, accumulation is fp32, the kernel stores bf16
(relative rounding 2^-9), so |err| <= 1.5e-2 * max|ref| is the stated per-op bound.
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _bf(x):
    return x.to(torch.bfloat16).to(torch.float32)


def _conv(cuda, N, cin, cout, H, W, K, stride, temb=False, res=False, seed=0):
    from audio_diffusion_b200 import _lib
    L = _lib.lib()
    g = torch.Generator().manual_seed(seed)
    x = _bf(torch.randn(N, cin, H, W, generator=g))
    w = _bf(torch.randn(cout, cin, K, K, generator=g) / (cin * K * K) ** 0.5)
    b = torch.randn(cout, generator=g)
    te = torch.randn(N, cout, generator=g) if temb else None
    Ho, Wo = H // stride, W // stride
    r = _bf(torch.randn(N, cout, Ho, Wo, generator=g)) if res else None
    ref = F.conv2d(x.double(), w.double(), b.double(), stride=stride, padding=K // 2)
    if temb:
        ref = ref + te[:, :, None, None].double()
    if res:
        ref = ref + r.double()
    d = lambda t: t.to(cuda).contiguous() if t is not None else None
    xd, wd, bd, ted, rd = d(x), d(w), d(b), d(te), d(r)
    y = torch.empty(N, cout, Ho, Wo, device=cuda)
    stats = torch.empty(N, cout // 4, 2, device=cuda)
    nb = L.b200ad_conv2d_scratch_bytes(N, cin, cout, H, W, K, stride)
    scratch = torch.empty(nb, dtype=torch.uint8, device=cuda)
    p = lambda t: t.data_ptr() if t is not None else None
    _lib.check(L.b200ad_conv2d(p(xd), p(wd), p(bd), p(ted), p(rd), p(y), p(stats), N, cin, cout, H, W, K, stride,
                               p(scratch), nb, _lib.stream_ptr()))
    torch.cuda.synchronize()
    y = y.cpu()
    err = (y - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= 1.5e-2 * scale, f"conv err {err} vs scale {scale}"
    # GroupNorm partial statistics of the stored output, per (sample, 4-channel quad)
    q = ref.view(N, cout // 4, 4, Ho * Wo)
    s_ref = torch.stack([q.sum(dim=(2, 3)), (q * q).sum(dim=(2, 3))], dim=-1)
    s = stats.cpu()
    tol = 2e-2 * s_ref[..., 1].abs().max().item()
    assert (s - s_ref).abs().max().item() <= tol + 1e-3 * Ho * Wo


@pytest.mark.parametrize("H,W", [(32, 32), (16, 16), (8, 8), (64, 64)])
def test_conv3x3_flat(cuda, H, W):
    _conv(cuda, 2, 128, 128, H, W, 3, 1)


@pytest.mark.parametrize("N,H,W", [(5, 8, 8), (6, 4, 4), (9, 2, 2), (3, 1, 1), (7, 8, 12)])
def test_conv3x3_packed_small_images(cuda, N, H, W):
    """Small images (image + bottom halo inside one 128-pixel tile) are packed up to four per work item: batches that fill
    items completely and partially, time-embedding bias and residual per SAMPLE, statistics per sample."""
    _conv(cuda, N, 256, 256, H, W, 3, 1, temb=True, res=True, seed=N)
    _conv(cuda, N, 128, 128, H, W, 1, 1, seed=N + 1)


def test_conv3x3_stride2_to_small_images(cuda):
    _conv(cuda, 5, 128, 256, 16, 16, 3, 2, seed=9)     # 16x16 -> 8x8: the output (and the parity planes) are packed
    _conv(cuda, 6, 128, 128, 8, 8, 3, 2, seed=10)


@pytest.mark.parametrize("N", [128, 5])
def test_conv3x3_stride2_2x2_to_1x1(cuda, N):
    """The latent U-Net's last downsampler (32x32 latent: 2x2 -> 1x1, 512 channels): one real tap per output pixel."""
    _conv(cuda, N, 512, 512, 2, 2, 3, 2, seed=N)


def test_conv3x3_wide(cuda):
    _conv(cuda, 2, 128, 128, 8, 128, 3, 1)
    _conv(cuda, 1, 64, 128, 12, 256, 3, 1, seed=3)


def test_conv3x3_channels(cuda):
    _conv(cuda, 1, 384, 256, 16, 16, 3, 1, temb=True, res=True)


def test_conv1x1(cuda):
    _conv(cuda, 2, 256, 128, 16, 16, 1, 1, res=True)
    _conv(cuda, 1, 128, 384, 4, 128, 1, 1)


def test_conv3x3_stride2(cuda):
    _conv(cuda, 2, 128, 128, 32, 32, 3, 2)
    _conv(cuda, 1, 128, 128, 16, 256, 3, 2, seed=5)


@pytest.mark.parametrize("silu", [0, 1])
def test_group_norm(cuda, silu):
    _group_norm(cuda, 2, 384, 16, 16, silu)


@pytest.mark.parametrize("N", [128, 5])
def test_group_norm_1x1(cuda, N):
    """The latent U-Net's 1x1 bottom level: each group is 16 channels of one pixel."""
    _group_norm(cuda, N, 512, 1, 1, 1)


def _group_norm(cuda, N, Cc, H, W, silu):
    from audio_diffusion_b200 import _lib
    L = _lib.lib()
    g = torch.Generator().manual_seed(1)
    x = _bf(torch.randn(N, Cc, H, W, generator=g) * 2 + 0.5)
    gamma = torch.randn(Cc, generator=g)
    beta = torch.randn(Cc, generator=g)
    ref = F.group_norm(x.double(), 32, gamma.double(), beta.double(), 1e-5)
    if silu:
        ref = F.silu(ref)
    xd, gd, bd = x.to(cuda), gamma.to(cuda), beta.to(cuda)
    y = torch.empty_like(xd)
    nb = 1 << 28     # the padded planes of 128 1x1 images need 134 MiB
    scratch = torch.empty(nb, dtype=torch.uint8, device=cuda)
    _lib.check(L.b200ad_group_norm(xd.data_ptr(), gd.data_ptr(), bd.data_ptr(), y.data_ptr(), N, Cc, H, W, 32, 1e-5,
                                   silu, scratch.data_ptr(), nb, _lib.stream_ptr()))
    torch.cuda.synchronize()
    err = (y.cpu() - ref).abs().max().item()
    assert err <= 1.5e-2 * ref.abs().max().item(), err


def test_sample_to_u8_bit_exact(cuda):
    """pipeline_audio_diffusion.py:192-194 integer boundary — bit-exact vs numpy."""
    from audio_diffusion_b200 import _lib
    L = _lib.lib()
    g = torch.Generator().manual_seed(2)
    x = torch.randn(1 << 16, generator=g) * 1.2
    # include exact .5 ties: (k + 0.5) / 255 * 2 - 1
    ties = ((torch.arange(0, 255, dtype=torch.float32) + 0.5) / 255.0) * 2 - 1
    x = torch.cat([x, ties])
    ref = ((x / 2 + 0.5).clamp(0, 1).numpy() * 255).round().astype("uint8")
    xd = x.to(cuda)
    out = torch.empty(x.numel(), dtype=torch.uint8, device=cuda)
    _lib.check(L.b200ad_sample_to_u8(xd.data_ptr(), out.data_ptr(), x.numel(), _lib.stream_ptr()))
    torch.cuda.synchronize()
    assert (out.cpu().numpy() == ref).all()


@pytest.mark.parametrize("silu,N,cin,cout,H,W,K", [(1, 2, 128, 128, 32, 32, 3), (0, 1, 256, 128, 16, 16, 1),
                                                   (1, 1, 128, 256, 8, 128, 3), (1, 2, 384, 128, 16, 16, 3),
                                                   (1, 6, 256, 128, 8, 8, 3), (0, 5, 128, 128, 4, 4, 1)])
def test_fused_groupnorm_conv(cuda, silu, N, cin, cout, H, W, K):
    """conv2d(silu(GroupNorm(x))) with the normalisation applied in the conv kernel's operand staging (transform warps).
    Reference keeps the normalised tensor in fp32; ours rounds it to bf16 before the MMA: tolerance 2.5e-2 * max|ref|."""
    from audio_diffusion_b200 import _lib
    L = _lib.lib()
    g = torch.Generator().manual_seed(11)
    x = _bf(torch.randn(N, cin, H, W, generator=g) * 1.7 + 0.3)
    gamma = 1 + 0.2 * torch.randn(cin, generator=g)
    beta = 0.2 * torch.randn(cin, generator=g)
    w = _bf(torch.randn(cout, cin, K, K, generator=g) / (cin * K * K) ** 0.5)
    b = torch.randn(cout, generator=g)
    a = F.group_norm(x, 32, gamma, beta, 1e-5)
    if silu:
        a = F.silu(a)
    ref = F.conv2d(a, w, b, padding=K // 2)
    d = lambda t: t.to(cuda).contiguous()
    xd, gd, bd, wd, biasd = d(x), d(gamma), d(beta), d(w), d(b)
    y = torch.empty(N, cout, H, W, device=cuda)
    nb = L.b200ad_conv2d_scratch_bytes(N, cin, cout, H, W, K, 1)
    scratch = torch.empty(nb, dtype=torch.uint8, device=cuda)
    _lib.check(L.b200ad_gn_conv2d(xd.data_ptr(), gd.data_ptr(), bd.data_ptr(), 32, 1e-5, silu, wd.data_ptr(),
                                  biasd.data_ptr(), y.data_ptr(), N, cin, cout, H, W, K, scratch.data_ptr(), nb,
                                  _lib.stream_ptr()))
    torch.cuda.synchronize()
    err = (y.cpu() - ref).abs().max().item()
    assert err <= 2.5e-2 * ref.abs().max().item(), f"err {err} scale {ref.abs().max().item()}"


@pytest.mark.parametrize("N,C,cout,H,W", [(2, 128, 128, 16, 16), (1, 128, 256, 8, 64), (1, 256, 128, 4, 128),
                                          (5, 128, 128, 8, 8), (6, 256, 128, 4, 4), (128, 512, 512, 1, 1),
                                          (5, 512, 512, 1, 1), (128, 512, 512, 2, 2), (5, 512, 512, 2, 2)])
def test_upsample_conv_folded(cuda, N, C, cout, H, W):
    """conv3x3(nearest_2x(x)) computed as four 2x2 convs with pre-summed weights on the low-res tensor (b200ad_conv2d with
    stride = -2). The weight sums are rounded to bf16 once, so compare against the fp64 reference with 2e-2 * max|ref|."""
    from audio_diffusion_b200 import _lib
    L = _lib.lib()
    g = torch.Generator().manual_seed(21)
    x = _bf(torch.randn(N, C, H, W, generator=g))
    w = _bf(torch.randn(cout, C, 3, 3, generator=g) / (C * 9) ** 0.5)
    b = torch.randn(cout, generator=g)
    ref = F.conv2d(F.interpolate(x.double(), scale_factor=2.0, mode="nearest"), w.double(), b.double(), padding=1)
    xd, wd, bd = x.to(cuda), w.to(cuda), b.to(cuda)
    y = torch.empty(N, cout, 2 * H, 2 * W, device=cuda)
    stats = torch.empty(N, cout // 4, 2, device=cuda)
    nb = L.b200ad_conv2d_scratch_bytes(N, C, cout, H, W, 3, -2)
    scratch = torch.empty(nb, dtype=torch.uint8, device=cuda)
    _lib.check(L.b200ad_conv2d(xd.data_ptr(), wd.data_ptr(), bd.data_ptr(), None, None, y.data_ptr(), stats.data_ptr(),
                               N, C, cout, H, W, 3, -2, scratch.data_ptr(), nb, _lib.stream_ptr()))
    torch.cuda.synchronize()
    err = (y.cpu() - ref).abs().max().item()
    assert err <= 2e-2 * ref.abs().max().item(), err
    q = ref.view(N, cout // 4, 4, 4 * H * W)
    s_ref = torch.stack([q.sum(dim=(2, 3)), (q * q).sum(dim=(2, 3))], dim=-1)
    assert (stats.cpu() - s_ref).abs().max().item() <= 3e-2 * s_ref[..., 1].abs().max().item() + 1e-3 * 4 * H * W


@pytest.mark.parametrize("N,cin,cout,H,W,K", [(2, 128, 256, 16, 16, 3), (1, 256, 128, 8, 24, 3), (2, 128, 128, 32, 32, 1),
                                              (7, 256, 128, 8, 8, 3)])
def test_conv_dgrad_matches_autograd(cuda, N, cin, cout, H, W, K):
    """b200ad_conv2d_dgrad (forward kernel + transposed / mirrored weight packing) == torch autograd's input gradient of
    F.conv2d(x, w, padding=K//2) for the same upstream gradient (bf16-rounded operands, fp32 reference)."""
    from audio_diffusion_b200 import _lib
    L = _lib.lib()
    g = torch.Generator().manual_seed(7)
    w = _bf(torch.randn(cout, cin, K, K, generator=g) / (cout * K * K) ** 0.5)
    gy = _bf(torch.randn(N, cout, H, W, generator=g))
    x = torch.zeros(N, cin, H, W, requires_grad=True)
    F.conv2d(x, w, padding=K // 2).backward(gy)
    ref = x.grad
    gyd, wd = gy.to(cuda).contiguous(), w.to(cuda).contiguous()
    gx = torch.empty(N, cin, H, W, device=cuda)
    nb = L.b200ad_conv2d_scratch_bytes(N, cout, cin, H, W, K, 1)
    scratch = torch.empty(nb, dtype=torch.uint8, device=cuda)
    _lib.check(L.b200ad_conv2d_dgrad(gyd.data_ptr(), wd.data_ptr(), gx.data_ptr(), N, cin, cout, H, W, K,
                                     scratch.data_ptr(), nb, _lib.stream_ptr()))
    torch.cuda.synchronize()
    err = (gx.cpu() - ref).abs().max().item()
    assert err <= 1.5e-2 * ref.abs().max().item(), f"dgrad err {err} vs {ref.abs().max().item()}"
