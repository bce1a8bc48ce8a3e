"""wgmma weight-gradient kernel (b200ad_conv2d_wgrad) against torch autograd (bf16-rounded operands, fp32 reference).
Tolerance: products of bf16 values accumulated in fp32 in a different order: 2e-3 of max|ref|."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("N,cin,cout,H,W,K", [(1, 32, 128, 8, 8, 1), (2, 64, 128, 16, 16, 3), (1, 128, 256, 8, 24, 3),
                                              (2, 128, 128, 32, 32, 3)])
def test_conv_wgrad_matches_autograd(cuda, N, cin, cout, H, W, K):
    from audio_diffusion_b200 import _lib
    L = _lib.lib()
    bf = lambda t: t.to(torch.bfloat16).to(torch.float32)
    g = torch.Generator().manual_seed(5)
    a = bf(torch.randn(N, cin, H, W, generator=g))
    gy = bf(torch.randn(N, cout, H, W, generator=g))
    w = torch.zeros(cout, cin, K, K, requires_grad=True)
    F.conv2d(a, w, padding=K // 2).backward(gy)
    ref = w.grad
    ad, gyd = a.to(cuda).contiguous(), gy.to(cuda).contiguous()      # keep the device copies alive across the async call
    dw = torch.full((cout, cin, K, K), float("nan"), device=cuda)
    nb = L.b200ad_conv2d_wgrad_scratch_bytes(N, cin, cout, H, W)
    scratch = torch.empty(nb, dtype=torch.uint8, device=cuda)
    _lib.check(L.b200ad_conv2d_wgrad(gyd.data_ptr(), ad.data_ptr(), dw.data_ptr(), N, cin, cout, H, W, K,
                                     scratch.data_ptr(), nb, _lib.stream_ptr()))
    torch.cuda.synchronize()
    err = (dw.cpu() - ref).abs().max().item()
    assert err <= 2e-3 * ref.abs().max().item(), (err, ref.abs().max().item())
