"""CPU tests (-m "not gpu"): the oracle's own known-answer tests (SURVEY §8c — the reference ships no tests or
fixtures, so these replace them), host-side logic, and the C-ABI library's load/export check."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------- U-Net oracle
def test_unet_param_count_and_keys():
    from oracle.unet_oracle import UNetConfig, param_shapes
    sh = param_shapes(UNetConfig())
    assert sum(math.prod(s) for s in sh.values()) == 113_668_609  # SURVEY §8
    assert "down_blocks.4.attentions.1.to_out.0.weight" in sh and "up_blocks.1.attentions.2.to_q.bias" in sh
    assert "mid_block.attentions.0.group_norm.weight" in sh and "up_blocks.5.upsamplers.0.conv.weight" not in sh
    assert sh["up_blocks.5.resnets.0.conv1.weight"] == (128, 256, 3, 3)
    assert sh["up_blocks.2.resnets.2.conv_shortcut.weight"] == (256, 512, 1, 1)


def test_unet_flops_match_survey():
    from oracle.unet_oracle import UNetConfig, unet_flops
    assert abs(unet_flops(UNetConfig(), 256, 256) / 1e9 - 496.42) < 0.01
    assert abs(unet_flops(UNetConfig(), 64, 64) / 1e9 - 31.00) < 0.01
    assert abs(unet_flops(UNetConfig(), 32, 32) / 1e9 - 7.76) < 0.01


def test_unet_forward_shape_and_groupnorm_invariant():
    from oracle.unet_oracle import UNetConfig, init_weights, unet_forward
    cfg = UNetConfig(sample_size=(32, 32), block_out_channels=(128, 256),
                     down_block_types=("DownBlock2D", "AttnDownBlock2D"), up_block_types=("AttnUpBlock2D", "UpBlock2D"))
    w = init_weights(cfg, seed=0)
    x = torch.randn(2, 1, 32, 32, generator=torch.Generator().manual_seed(0))
    taps = {}
    y = unet_forward(w, cfg, x, torch.tensor([3, 700]), taps)
    assert y.shape == x.shape
    # per-sample timestep == scalar timestep on each sample
    y0 = unet_forward(w, cfg, x[:1], 3)
    assert torch.allclose(y[:1], y0, atol=1e-5)
    a = taps["down_blocks.0.resnets.0.act1"]  # silu(GN(x)); check GN via fresh computation
    h = taps["conv_in"]
    gn = torch.nn.functional.group_norm(h, 32)
    g = gn.view(2, 32, -1)
    assert g.mean(-1).abs().max() < 1e-4 and (g.var(-1, unbiased=False) - 1).abs().max() < 1e-3
    assert a.shape == h.shape


def test_timestep_embedding_layout():
    from oracle.unet_oracle import timestep_embedding
    e = timestep_embedding(torch.tensor([0, 10]), 128)
    assert torch.allclose(e[0, :64], torch.ones(64)) and torch.allclose(e[0, 64:], torch.zeros(64))  # [cos | sin]
    assert abs(e[1, 0].item() - math.cos(10.0)) < 1e-6 and abs(e[1, 64].item() - math.sin(10.0)) < 1e-6


# ------------------------------------------------------------------------------------------- schedulers
def test_scheduler_known_answers():
    from oracle.schedulers_oracle import OracleDDIM, OracleDDPM
    s = OracleDDPM()
    assert abs(s.alphas_cumprod[0].item() - (1 - 1e-4)) < 1e-7
    assert abs(s.alphas_cumprod[999].item() - 4.04e-5) < 2e-6
    s.set_timesteps(1000)
    assert s.timesteps[0].item() == 999 and s.timesteps[-1].item() == 0
    d = OracleDDIM()
    d.set_timesteps(50)
    assert d.timesteps[:3].tolist() == [980, 960, 940] and d.timesteps[-1].item() == 0
    x = torch.randn(1, 1, 8, 8, generator=torch.Generator().manual_seed(1))
    eps = torch.randn(1, 1, 8, 8, generator=torch.Generator().manual_seed(2))
    g = torch.Generator().manual_seed(3)
    a = s.step(eps, 0, x, generator=g)["prev_sample"]   # t == 0 adds no noise and consumes no RNG
    b = s.step(eps, 0, x, generator=torch.Generator().manual_seed(99))["prev_sample"]
    assert torch.equal(a, b)
    n = torch.randn(4, 1, 8, 8)
    noisy = s.add_noise(torch.zeros(4, 1, 8, 8), n, torch.tensor([999, 999, 0, 0]))
    assert torch.allclose(noisy[:2], n[:2] * (1 - s.alphas_cumprod[999]) ** 0.5)
    assert noisy[2:].abs().max() <= n[2:].abs().max() * 0.011


def test_product_schedulers_equal_oracle():
    """Host logic of the product schedulers (torch ops, CPU-runnable) against the oracle, incl. fused coefficients."""
    from audio_diffusion_b200.schedulers import DDIMScheduler, DDPMScheduler
    from oracle.schedulers_oracle import OracleDDIM, OracleDDPM
    x = torch.randn(2, 1, 16, 16, generator=torch.Generator().manual_seed(1))
    eps = torch.randn(2, 1, 16, 16, generator=torch.Generator().manual_seed(2))
    for P, O, n, kw in ((DDPMScheduler, OracleDDPM, 1000, {}), (DDIMScheduler, OracleDDIM, 50, {"eta": 0.0}),
                        (DDIMScheduler, OracleDDIM, 50, {"eta": 0.5})):
        p, o = P(), O()
        p.set_timesteps(n)
        o.set_timesteps(n)
        assert torch.equal(p.timesteps, o.timesteps) and torch.equal(p.alphas_cumprod, o.alphas_cumprod)
        for t in (p.timesteps[0], p.timesteps[n // 2], p.timesteps[-1]):
            a = p.step(model_output=eps, timestep=t, sample=x, generator=torch.Generator().manual_seed(5), **kw)["prev_sample"]
            b = o.step(eps, t, x, generator=torch.Generator().manual_seed(5), **kw)["prev_sample"]
            assert torch.equal(a, b)
            # fused-kernel form: x0 = clamp((x - c0 eps) * c1); out = c_x0 x0 + c_xt x + c_eps eps + c_z z
            c = p.step_coef(t, kw.get("eta", 0.0))
            z = torch.randn(eps.shape, generator=torch.Generator().manual_seed(5))
            x0 = ((x - c.sqrt_1m_at * eps) * c.inv_sqrt_at).clamp(-c.clip, c.clip)
            f = c.c_x0 * x0 + c.c_xt * x + c.c_eps * eps + (c.c_z * z if p.needs_noise(t, kw.get("eta", 0.0)) else 0)
            assert torch.allclose(f, b, atol=2e-5, rtol=1e-5)
        assert torch.equal(p.add_noise(x, eps, torch.tensor([10, 900])), o.add_noise(x, eps, torch.tensor([10, 900])))


def test_ddim_inversion_roundtrip():
    """pipeline_audio_diffusion.py:219-242: DDIM eta=0 encode -> sample round-trips for a fixed epsilon model."""
    from oracle.schedulers_oracle import OracleDDIM
    d = OracleDDIM()
    d.set_timesteps(50)
    x = torch.randn(1, 1, 8, 8, generator=torch.Generator().manual_seed(1)) * 0.3
    model = lambda s, t: 0.1 * torch.ones_like(s)  # noqa: E731
    s = x.clone()
    for t in torch.flip(d.timesteps, (0,)):
        prev = t - 1000 // 50
        a_t = d.alphas_cumprod[t]
        a_prev = d.alphas_cumprod[prev] if prev >= 0 else d.final_alpha_cumprod
        e = model(s, t)
        s = (s - (1 - a_prev) ** 0.5 * e) * a_prev ** (-0.5)
        s = s * a_t ** 0.5 + (1 - a_t) ** 0.5 * e
    for t in d.timesteps:
        s = d.step(model(s, t), t, s, eta=0.0)["prev_sample"]
    assert (s - x).abs().max() < 1e-3


# ------------------------------------------------------------------------------------------- mel oracle
def _tone(sr=22050, n=131071, f=440.0, noise=0.05, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    return (rng.standard_normal(n) * noise + 0.5 * np.sin(2 * np.pi * f * t)).astype(np.float32)


def test_mel_known_answers():
    from oracle import mel_oracle as mo
    assert mo.stft(np.zeros(131071, np.float32), 2048, 512).shape == (1025, 256)   # exactly 256 frames
    silent = mo.audio_slice_to_bytes(np.zeros(131071, np.float32))
    assert silent.shape == (256, 256) and silent.dtype == np.uint8 and (silent == 255).all()  # audio_to_images.py:46
    b = mo.audio_slice_to_bytes(_tone(f=440.0, noise=0.0))
    A = mo.mel_filterbank(22050, 2048, 256)
    expect = int(np.argmax(A[:, int(round(440.0 * 2048 / 22050))]))
    assert abs(int(np.argmax(b.astype(int).sum(1))) - expect) <= 1    # tone lights the Slaney row of 440 Hz
    assert b.max() == 255 and b.min() >= 0


def test_mel_u8_boundaries_bit_exact():
    from oracle import mel_oracle as mo
    ls = np.array([-80.0, -79.999, -40.0, -0.157, -0.156, 0.0, 5.0, -200.0], dtype=np.float32)
    out = mo.db_to_u8(ls, 80)
    assert out.tolist() == [0, 0, 128, 254, 255, 255, 255, 0]
    p = mo.u8_to_power(np.array([0, 255, 128], dtype=np.uint8))
    assert abs(p[0] - 1e-8) < 1e-20 and p[1] == 1.0 and abs(10 * np.log10(p[2]) - (128 * 80 / 255 - 80)) < 1e-12


def test_mel_nnls_is_initial_point_on_image_domain():
    """librosa.util.nnls's L-BFGS-B stops at iteration 0 for image-domain spectrograms (S <= 1), so the
    inverse mel transform is exactly clip(pinv(A) @ S, 0) — which is what the CUDA path computes."""
    import scipy.optimize
    from oracle import mel_oracle as mo
    b = mo.audio_slice_to_bytes(_tone(noise=0.2, seed=3), n_mels=64)[:, :32]
    S = mo.u8_to_power(b)
    A = mo.mel_filterbank(22050, 2048, 64, dtype=S.dtype)
    x0 = np.clip(np.linalg.pinv(A) @ S, 0, None)
    x, f, d = scipy.optimize.fmin_l_bfgs_b(mo._nnls_obj, x0, args=(x0.shape, A, S), bounds=[(0, None)] * x0.size)
    assert d["nit"] == 0 and np.array_equal(x.reshape(x0.shape), x0)


@pytest.mark.parametrize("kind", ["zeros", "ones", "random", "checker", "tone"])
def test_mel_nnls_initial_point_256x256_per_librosa_block(kind):
    """The same pin at the benchmarked size: 256 mels x 256 frames, split into librosa's column blocks
    (MAX_MEM_BLOCK 2**18 bytes / (256 mels * 8 B) = 128 columns), on degenerate and arbitrary byte images.
    L-BFGS-B returns at iteration 0 with x == clip(pinv(A) @ S, 0) for every block: the objective carries a 1/size
    factor, so on the image domain (S <= 1) the projected-gradient test (pgtol 1e-5) passes at the initial point."""
    import scipy.optimize
    from oracle import mel_oracle as mo
    rng = np.random.default_rng(0)
    b = {"zeros": lambda: np.zeros((256, 256), np.uint8), "ones": lambda: np.full((256, 256), 255, np.uint8),
         "random": lambda: rng.integers(0, 256, (256, 256), dtype=np.uint8),
         "checker": lambda: ((np.indices((256, 256)).sum(0) % 2) * 255).astype(np.uint8),
         "tone": lambda: mo.audio_slice_to_bytes(_tone(noise=0.2, seed=5), n_mels=256)}[kind]()
    S = mo.u8_to_power(b)
    A = mo.mel_filterbank(22050, 2048, 256, dtype=S.dtype)
    pinv = np.linalg.pinv(A)
    ncol = int((2 ** 8 * 2 ** 10) // (256 * A.itemsize))
    assert ncol == 128
    for s0 in range(0, 256, ncol):
        B = S[:, s0:s0 + ncol]
        x0 = np.clip(pinv @ B, 0, None)
        x, f, d = scipy.optimize.fmin_l_bfgs_b(mo._nnls_obj, x0, args=(x0.shape, A, B), bounds=[(0, None)] * x0.size)
        assert d["nit"] == 0 and d["funcalls"] == 1 and np.array_equal(x.reshape(x0.shape), x0), (kind, s0, d)
    # and the oracle's own nnls (which runs the optimiser) returns exactly that closed form
    assert np.array_equal(mo.nnls(A, S), np.clip(pinv @ S, 0, None))


def test_mel_roundtrip_in_mel_domain():
    from oracle import mel_oracle as mo
    cfg = dict(sr=22050, n_fft=2048, hop=512)
    y = _tone(n=64 * 512 - 1, noise=0.1)
    b = mo.audio_slice_to_bytes(y, n_mels=64, **cfg)
    a = mo.bytes_to_audio(b, n_iter=32, rng=np.random.default_rng(0), **cfg)
    assert a.shape == ((64 - 1) * 512,) and a.dtype == np.float32       # mel.py:165-167 output length
    b2 = mo.audio_slice_to_bytes(np.concatenate([a, np.zeros(64 * 512 - 1 - len(a), np.float32)]), n_mels=64, **cfg)
    assert np.abs(b2.astype(int) - b.astype(int)).mean() < 12.0


def test_product_mel_constants_equal_oracle():
    from audio_diffusion_b200.mel import Mel, slaney_mel_basis
    from oracle import mel_oracle as mo
    for dt in (np.float32, np.float64):
        assert np.array_equal(slaney_mel_basis(22050, 2048, 256, dt), mo.mel_filterbank(22050, 2048, 256, dtype=dt))
    m = Mel(x_res=64, y_res=64, hop_length=1024)
    assert m.slice_size == 64 * 1024 - 1 and m.n_mels == 64
    m.load_audio(raw_audio=np.ones(10, dtype=np.float32))
    assert len(m.audio) == 64 * 1024 and m.get_number_of_slices() == 1 and m.get_sample_rate() == 22050


# ------------------------------------------------------------------------------------------- C ABI
def test_library_loads_and_exports_every_declared_symbol():
    from audio_diffusion_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    L = ctypes.CDLL(_lib.LIB_PATH)
    hdr = open(os.path.join(ROOT, "include", "b200ad.h")).read()
    declared = set(re.findall(r"\b(b200ad_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"b200ad_unet_config", "b200ad_step_coef", "b200ad_mel_config"}
    assert declared, "no declarations parsed"
    for name in sorted(declared):
        assert hasattr(L, name), f"libb200ad.so does not export {name}"
    assert set(_lib.SYMBOLS) == declared
    assert _lib.lib().b200ad_version() >= 1


def test_unet_handle_param_table_matches_oracle_without_gpu():
    from audio_diffusion_b200.unet import UNet2DModel
    from oracle.unet_oracle import UNetConfig, param_shapes
    kw = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 128, 256, 256, 512, 512),
              down_block_types=("DownBlock2D",) * 4 + ("AttnDownBlock2D", "DownBlock2D"),
              up_block_types=("UpBlock2D", "AttnUpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D"))
    m = UNet2DModel(sample_size=(256, 256), **kw)
    sd = m.state_dict()
    ref = param_shapes(UNetConfig())
    assert set(sd.keys()) == set(ref.keys()) and len(sd) == len(ref)
    assert all(tuple(sd[k].shape) == ref[k] for k in ref)
    from audio_diffusion_b200 import _lib
    need = _lib.lib().b200ad_unet_workspace_bytes(m._h, 64, 256, 256)
    assert 5e9 < need < 60e9  # activations for config C2 fit an 80 GB H100


def test_product_fails_loudly_without_cuda():
    from audio_diffusion_b200 import _lib
    from audio_diffusion_b200.unet import UNet2DModel
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    m = UNet2DModel(sample_size=(32, 32), in_channels=1, out_channels=1, block_out_channels=(128, 128),
                    down_block_types=("DownBlock2D", "DownBlock2D"), up_block_types=("UpBlock2D", "UpBlock2D"))
    with pytest.raises(_lib.B200ADError):
        with torch.no_grad():
            m(torch.zeros(1, 1, 32, 32), 0)


def test_vae_oracle_shapes_and_param_table():
    """AutoencoderKL oracle: SURVEY §3.4 parameter counts (34.1 M encoder side, 49.5 M decoder side), latent geometry,
    and the library's parameter table (names, order, shapes) equal to the oracle's state-dict layout."""
    import ctypes as C

    from audio_diffusion_b200 import _lib
    from oracle import vae_oracle as vo

    cfg = vo.VAEConfig()
    sh = vo.param_shapes(cfg)
    cnt = lambda pre: sum(int(np.prod(s)) for k, s in sh.items() if k.startswith(pre))
    enc = cnt("encoder.") + cnt("quant_conv")
    dec = cnt("decoder.") + cnt("post_quant_conv")
    assert abs(enc / 1e6 - 34.1) < 0.1 and abs(dec / 1e6 - 49.5) < 0.1
    w = vo.init_weights(cfg, seed=0)
    x = torch.randn(1, 1, 32, 64, generator=torch.Generator().manual_seed(0))
    m = vo.encode_moments(w, cfg, x)
    assert m.shape == (1, 2, 4, 8)
    z = vo.posterior_sample(m, torch.zeros(1, 1, 4, 8))
    assert torch.equal(z, m[:, :1])
    assert vo.decode(w, cfg, z).shape == (1, 1, 32, 64)

    L = _lib.lib()
    c = _lib.VAEConfigC(1, 1, 1, 2, 4, (C.c_int * 8)(128, 256, 512, 512), 32, 1e-6)
    h = C.c_void_p()
    assert L.b200ad_vae_create(C.byref(c), C.byref(h)) == 0
    try:
        names = [L.b200ad_vae_param_name(h, i).decode() for i in range(L.b200ad_vae_num_params(h))]
        assert names == list(sh.keys())
        d = (C.c_int64 * 4)()
        for i, nm in enumerate(names):
            k = L.b200ad_vae_param_shape(h, i, d)
            assert tuple(d[:k]) == tuple(sh[nm]), nm
    finally:
        L.b200ad_vae_destroy(h)


def test_vae_bf16_rounding_floor():
    """Derivation of the decoder tolerance in tests/test_gpu_vae.py: the fp32 oracle with every conv / linear operand and
    output rounded to bf16 (what any bf16-storage engine does) against itself in fp32.  The encoder stays below 1.5% rms;
    the skip-free decoder chain compounds to a few percent."""
    import torch.nn.functional as F

    from oracle import vae_oracle as vo

    cfg = vo.VAEConfig()
    w = vo.init_weights(cfg, seed=0)
    x = torch.randn(2, 1, 64, 64, generator=torch.Generator().manual_seed(5)).clamp(-1, 1)
    m = vo.encode_moments(w, cfg, x)
    z = m[:, :1].contiguous()
    y = vo.decode(w, cfg, z)
    oc, ol = F.conv2d, F.linear
    bf = lambda t: t.to(torch.bfloat16).to(torch.float32)
    vo.F.conv2d = lambda a, ww, b=None, **k: bf(oc(bf(a), bf(ww), b, **k))
    vo.F.linear = lambda a, ww, b=None: bf(ol(bf(a), bf(ww), b))
    try:
        m2 = vo.encode_moments(w, cfg, x)
        y2 = vo.decode(w, cfg, z)
    finally:
        vo.F.conv2d, vo.F.linear = oc, ol
    rel = lambda a, b: ((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt()).item()
    assert rel(m2, m) < 1.5e-2
    assert 1e-2 < rel(y2, y) < 5e-2


def test_train_oracle_adamw_matches_torch():
    """The training oracle's optimizer / clipping restatement against torch itself (available here): AdamW(betas .95/.999,
    wd 1e-6, eps 1e-8) over three steps and clip_grad_norm_(1.0) — scripts/train_unet.py:166-172, :261-263."""
    from oracle.train_oracle import adamw_update, clip_grad_norm

    g = torch.Generator().manual_seed(0)
    p0 = torch.randn(37, 5, generator=g)
    p_ref = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([p_ref], lr=3e-4, betas=(0.95, 0.999), weight_decay=1e-6, eps=1e-8)
    p, m, v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
    for step in range(1, 4):
        grad = torch.randn(37, 5, generator=g) * 3
        p_ref.grad = grad.clone()
        total_ref = torch.nn.utils.clip_grad_norm_([p_ref], 1.0)
        clipped, total = clip_grad_norm({"p": grad}, 1.0)
        assert torch.allclose(total, total_ref, rtol=1e-6)
        assert torch.allclose(clipped["p"], p_ref.grad, rtol=1e-6, atol=1e-8)
        opt.step()
        adamw_update(p, clipped["p"], m, v, step, 3e-4)
        assert torch.allclose(p, p_ref.detach(), rtol=1e-6, atol=1e-7), step


def test_train_oracle_schedules_and_step():
    """Cosine-with-warmup multipliers, EMA decay schedule (inv_gamma 1, power 3/4, max .9999) and one full training step
    on a small U-Net: loss is finite, the clipped gradient norm is <= 1, parameters move, EMA follows with decay 0 first."""
    from oracle.train_oracle import TrainState, cosine_with_warmup, ema_decay, loss_and_grads, train_step
    from oracle.unet_oracle import UNetConfig, init_weights

    assert cosine_with_warmup(0, 500, 10000) == 0.0 and cosine_with_warmup(250, 500, 10000) == 0.5
    assert cosine_with_warmup(500, 500, 10000) == 1.0 and abs(cosine_with_warmup(5250, 500, 10000) - 0.5) < 1e-12
    assert cosine_with_warmup(10000, 500, 10000) < 1e-12
    assert ema_decay(0) == 0.0 and ema_decay(1) == 0.0
    assert abs(ema_decay(2) - (1 - 2 ** -0.75)) < 1e-12 and ema_decay(10 ** 9) == 0.9999
    # the shim's LambdaLR agrees with the oracle's multiplier
    import sys
    sys.path.insert(0, os.path.join(ROOT, "audio_diffusion_b200", "compat"))
    try:
        from diffusers.optimization import get_scheduler
    finally:
        sys.path.pop(0)
    q = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.AdamW([q], lr=1.0)
    sch = get_scheduler("cosine", optimizer=opt, num_warmup_steps=5, num_training_steps=50)
    for k in range(12):
        assert abs(sch.get_last_lr()[0] - cosine_with_warmup(k, 5, 50)) < 1e-12
        opt.step(); sch.step()

    cfg = UNetConfig(sample_size=(16, 16), in_channels=1, out_channels=1, layers_per_block=1, block_out_channels=(128, 128),
                     down_block_types=("DownBlock2D", "AttnDownBlock2D"), up_block_types=("AttnUpBlock2D", "UpBlock2D"))
    w = init_weights(cfg, seed=0)
    g = torch.Generator().manual_seed(1)
    clean = torch.rand(2, 1, 16, 16, generator=g) * 2 - 1
    noise = torch.randn(2, 1, 16, 16, generator=g)
    t = torch.tensor([10, 900])
    loss, grads, pred = loss_and_grads(w, cfg, clean, noise, t)
    assert torch.isfinite(loss) and set(grads) == set(w) and pred.shape == noise.shape
    st = TrainState()
    w0 = {k: v.clone() for k, v in w.items()}
    loss2, gnorm, lr, decay = train_step(w, cfg, st, clean, noise, t, base_lr=1e-4, warmup=0, total_steps=100)
    assert abs(loss2 - loss) < 1e-6 and lr == 1e-4 and decay == 0.0 and st.step == 1
    assert any(not torch.equal(w[k], w0[k]) for k in w)
    assert all(torch.equal(st.ema[k], w[k]) for k in w)          # decay 0: shadow == parameters after step 1


GOLDEN = os.path.join(ROOT, "tests", "golden")


def test_golden_vae_key_map_matches_library_table():
    """tests/golden/vae_key_map.json (written by the reference's own converter, tests/golden/make_golden.py) == libb200ad's
    AutoencoderKL parameter table after diffusers' deprecated-attention renames (names AND shapes)."""
    import ctypes as C
    import json

    from audio_diffusion_b200 import _lib
    with open(os.path.join(GOLDEN, "vae_key_map.json")) as f:
        gold = json.load(f)["keys"]
    ren = {".query.": ".to_q.", ".key.": ".to_k.", ".value.": ".to_v.", ".proj_attn.": ".to_out.0."}
    want = {}
    for k, shape in gold:
        for a, b in ren.items():
            k = k.replace(a, b)
        want[k] = tuple(shape)
    L = _lib.lib()
    c = _lib.VAEConfigC(1, 1, 1, 2, 4, (C.c_int * 8)(128, 256, 512, 512), 32, 1e-6)
    h = C.c_void_p()
    assert L.b200ad_vae_create(C.byref(c), C.byref(h)) == 0
    try:
        got = {}
        d = (C.c_int64 * 4)()
        for i in range(L.b200ad_vae_num_params(h)):
            k = L.b200ad_vae_param_shape(h, i, d)
            got[L.b200ad_vae_param_name(h, i).decode()] = tuple(d[:k])
    finally:
        L.b200ad_vae_destroy(h)
    assert got == want


def test_golden_pipeline_images_match_oracle_loop():
    """tests/golden/pipeline_ddpm_small.npz was produced by the reference's unchanged AudioDiffusionPipeline.__call__
    (tests/golden/make_golden.py); the oracle's own loop (oracle U-Net + OracleDDPM, same noise draws) gives the same bytes."""
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_oracle import UNetConfig, init_weights, unet_forward
    z = np.load(os.path.join(GOLDEN, "pipeline_ddpm_small.npz"))
    cfg = UNetConfig(sample_size=(32, 32), in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256),
                     down_block_types=("DownBlock2D", "AttnDownBlock2D"), up_block_types=("AttnUpBlock2D", "UpBlock2D"))
    w = init_weights(cfg, seed=int(z["weight_seed"]))
    sch = OracleDDPM()
    sch.set_timesteps(int(z["steps"]))
    gen = torch.Generator().manual_seed(int(z["step_seed"]))
    x = torch.from_numpy(z["noise"]).clone()
    for t in sch.timesteps:
        x = sch.step(unet_forward(w, cfg, x, t), t, x, generator=gen)["prev_sample"]
    img = ((x / 2 + 0.5).clamp(0, 1).permute(0, 2, 3, 1).numpy() * 255).round().astype("uint8")[:, :, :, 0]
    assert np.array_equal(img, z["images"])


def test_training_host_logic_without_gpu():
    """EMAModel's schedule and CPU shadow update (diffusers 0.24 surface: step / copy_to / get_decay, deprecated max_value /
    inv_gamma / power kwargs as scripts/train_unet.py:185-190 passes them), and the product's refusal to run without CUDA."""
    from audio_diffusion_b200._lib import B200ADError
    from audio_diffusion_b200.training import EMAModel, FusedAdamW, mse_loss
    from oracle.train_oracle import ema_decay

    lin = torch.nn.Linear(4, 3)
    ema = EMAModel(lin, inv_gamma=1.0, power=0.75, max_value=0.9999)
    ref = [p.detach().clone() for p in lin.parameters()]
    for step in range(1, 6):
        with torch.no_grad():
            for p in lin.parameters():
                p.add_(0.1 * step)
        ema.step(lin)                      # accepts a module or an iterable of parameters
        d = ema_decay(step, 1.0, 0.75, 0.9999)
        assert abs(ema.cur_decay_value - d) < 1e-12 and abs(ema.get_decay(step) - d) < 1e-12
        for r, p in zip(ref, lin.parameters()):
            r.sub_((1 - d) * (r - p.detach()))
    for s, r in zip(ema.shadow_params, ref):
        assert torch.allclose(s, r, rtol=1e-6, atol=1e-7)
    before = [p._version for p in lin.parameters()]
    ema.copy_to(lin.parameters())
    assert all(torch.equal(p.detach(), s) for p, s in zip(lin.parameters(), ema.shadow_params))
    assert all(p._version > v for p, v in zip(lin.parameters(), before))     # the engine keys its packed weights on this
    if not torch.cuda.is_available():
        opt = FusedAdamW(lin.parameters(), lr=1e-3)
        for p in lin.parameters():
            p.grad = torch.zeros_like(p)
        with pytest.raises(B200ADError):
            opt.step()
        with pytest.raises(B200ADError):
            mse_loss(torch.zeros(2), torch.zeros(2))
