"""The Mel codec (libb200ad: b200ad_mel_encode_ref / b200ad_mel_decode) against float64 references of the same
operations, at every n_fft the codec accepts and at the edges of its kernels: the radix-2 Stockham pass (log2(n_fft / 2)
odd: 64, 256, 1024, 4096), more than 48 KB of dynamic shared memory (4096), hop = n_fft (the window sum-square is 0 at
every frame start), a hop that does not divide n_fft, y_res not a multiple of 16 and x_res not a multiple of 64 (the
tails of the inverse-mel GEMM), y_res > n_fft / 2 + 1 (empty mel filters), and a decode batch of four distinct images
(the seeded phase is indexed by image).  The slices: noise plus two tones, one silent in its first half (all-zero frames
and frames across the edge), one silent throughout.  Decode gets the oracle's encodings of the three and one random
byte image, so every decode reference depends on numpy and the seeds alone.

E1 (`test_mel_power`): the mel power before quantisation against `mel_power64`, element by element, within
(k_m + 16) 2^-24 ref, k_m the non-zero weights of mel row m.  Derivation (u = 2^-24, the float32 unit roundoff):
the kernel computes X in float64 (its error, ~ 2^-53 log2(n_fft) ||frame|| absolute, is below 1e-12 of every bin that
contributes here, negligible) and rounds it to complex64: |re|^2 + |im|^2 moves by <= 2u relative; hypotf has a
maximum error of 3 ulp (CUDA C Programming Guide), <= 6u relative, 12u once squared; the fp32 square rounds once, u:
each term b_f |X_f|^2 is within 15u of exact.  The sequential fmaf sum of k_m non-negative terms rounds k_m times, each
by <= u of a partial sum <= the total: k_m u.  15u + k_m u, plus the second-order terms, is within (k_m + 16) u.  The
basis is the float32 constant the kernel multiplies by, promoted exactly.  Silent frames and empty filters must give
exactly 0.

E2 (`test_db_u8`): every pixel recomputed in float64 from the engine's own mel power (power_to_db with ref = max or a
scalar, amin 1e-10, top_db 80, then mel.py:149).  Pixels must be equal except where the float64 value before the
truncating cast lies within 1e-3 of an integer (the float32 chain is ~1e-4 grey levels off it); those may differ by
exactly 1.  The silent slice is all 255.

D1 (`test_decode_istft`): n_iter = 0, against `griffinlim(rounded=True)` from the engine's seeded spectrum
(`initial_spectrum`).  Per output sample p, with T_p the windowed frame terms overlapping at p and w_p the float32 window
sum-square: both sides round nearly equal float64 frame terms to float32 (<= 1 ulp apart, 2u |t| each), cast nearly
equal sums to float32 (2u sum |t|), use float32 window sum-squares <= 1 ulp apart (2u |y / w|) and round the quotient
(2u |y / w|); |y| <= sum |t|, so |engine - model| <= 8u sum |T_p| / w_p, plus the float64 differences of the two
transforms and of the pinv GEMM order, bounded generously by 2^-42 sum_f w max|irfft_f| / w_p.  Where w_p <= FLT_MIN
(hop = n_fft, every frame start) both leave the sum unnormalised and the same bar applies without the division: every
term there carries a window value of exactly 0, so the output must be exactly 0.

D2 (`test_griffinlim`): n_iter in {1, 4, 32}: the engine's audio against exact float64 Griffin-Lim from the same seeded
spectrum, relative L2 over the batch and max |err| / max |ref|.  The floor is `rounded` against exact on the same
inputs, measured in the same run; each bar is 3x the floor printed beside it (3 significant digits), and every run
asserts the engine within its bars and every bar in (floor, 3.3 x floor].

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit: E1 worst error 0.19 - 0.26 of its bar per config; E2
6 - 364 exempt pixels per config (364 of 393216 at 2048 / 512), 3 pixels differing by one in all, every one exempt;
D1 the engine equal to the rounded model at every sample; D2 the engine exactly at its floor (one third of each bar)
at every config and n_iter, at most 1.6e-7 relative L2 from the rounded model.  The whole file and
tests/test_gpu_mel.py ran in 45 s.  Each of three deliberate errors in the oracle failed the checks that can see it,
at 64 / 16, 512 / 128 and 4096 / 1024: one window sample scaled by 1 + 1e-3 (E1, D1, D2), one sign flipped in the
radix-2 pass of a numpy copy of the kernels' FFT schedule (E1, D1, D2 at the two sizes with that pass), the phase
index off by one image (D1, D2).
"""
import ctypes as C
import time

import numpy as np
import pytest
import scipy.fft
import torch

from blockcheck import power_limit
from oracle import mel_oracle as mo

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SEED = 0x5EED_1234_ABCD      # non-zero phase seed
TOP_DB = 80

# n_fft, hop, x_res, y_res
CONFIGS = [
    (64, 16, 64, 48),        # smallest size; radix-2 pass; y_res > F = 33: 14 empty filters
    (128, 128, 32, 32),      # hop = n_fft
    (256, 100, 64, 40),      # hop does not divide n_fft; radix-2 pass; y_res not a multiple of 16
    (512, 128, 96, 64),      # x_res not a multiple of 64
    (1024, 256, 128, 80),    # radix-2 pass
    (2048, 512, 256, 256),   # the product default (benchmarked)
    (2048, 2048, 64, 128),   # hop = n_fft at the default size
    (4096, 1024, 128, 128),  # radix-2 pass; > 48 KB of dynamic shared memory
]
CFG_IDS = [f"{n}-{h}-{x}x{y}" for n, h, x, y in CONFIGS]

# (n_fft, hop) -> {n_iter: (relative L2, max |err| / max |ref|)}, three times the floor printed beside it
GL_BARS = {
    (64, 16): {1: (2.08e-07, 2.9e-07), 4: (5.97e-07, 1.21e-06), 32: (1.21e-05, 3.12e-05)},
    # floor 1: (6.95e-08, 9.67e-08), 4: (1.99e-07, 4.04e-07), 32: (4.04e-06, 1.04e-05)
    (128, 128): {1: (1.41e-07, 1.56e-07), 4: (7.14e-07, 6.36e-07), 32: (0.000105, 0.000217)},
    # floor 1: (4.7e-08, 5.19e-08), 4: (2.38e-07, 2.12e-07), 32: (3.51e-05, 7.23e-05)
    (256, 100): {1: (2.96e-07, 3.78e-07), 4: (7.41e-07, 8.1e-07), 32: (5.85e-05, 0.000149)},
    # floor 1: (9.86e-08, 1.26e-07), 4: (2.47e-07, 2.7e-07), 32: (1.95e-05, 4.97e-05)
    (512, 128): {1: (2.19e-07, 3.51e-07), 4: (1.17e-06, 2.29e-06), 32: (3.45e-05, 4.14e-05)},
    # floor 1: (7.3e-08, 1.17e-07), 4: (3.9e-07, 7.62e-07), 32: (1.15e-05, 1.38e-05)
    (1024, 256): {1: (2.17e-07, 3.9e-07), 4: (1.51e-06, 3.06e-06), 32: (9.48e-05, 0.000259)},
    # floor 1: (7.24e-08, 1.3e-07), 4: (5.03e-07, 1.02e-06), 32: (3.16e-05, 8.64e-05)
    (2048, 512): {1: (2.28e-07, 4.89e-07), 4: (8.67e-07, 1.59e-06), 32: (8.97e-05, 0.000127)},
    # floor 1: (7.6e-08, 1.63e-07), 4: (2.89e-07, 5.3e-07), 32: (2.99e-05, 4.23e-05)
    (2048, 2048): {1: (1.84e-07, 3.09e-07), 4: (7.53e-07, 8.55e-07), 32: (2.67e-05, 2.65e-05)},
    # floor 1: (6.13e-08, 1.03e-07), 4: (2.51e-07, 2.85e-07), 32: (8.9e-06, 8.83e-06)
    (4096, 1024): {1: (2.41e-07, 4.86e-07), 4: (8.19e-07, 1.27e-06), 32: (5.64e-05, 9.36e-05)},
    # floor 1: (8.04e-08, 1.62e-07), 4: (2.73e-07, 4.24e-07), 32: (1.88e-05, 3.12e-05)
}


def slices(n_fft, hop, x_res):
    """(3, x_res * hop - 1) float32: noise + two tones; silent first half, then noise + two other tones; silence."""
    L = x_res * hop - 1
    rng = np.random.default_rng(n_fft + hop)
    t = np.arange(L) / 22050
    a = 0.05 * rng.standard_normal(L) + 0.5 * np.sin(2 * np.pi * 330.0 * t) + 0.2 * np.sin(2 * np.pi * 2900.0 * t)
    b = 0.05 * rng.standard_normal(L) + 0.4 * np.sin(2 * np.pi * 520.0 * t) + 0.3 * np.sin(2 * np.pi * 4700.0 * t)
    b[: L // 2] = 0.0
    return np.stack([a, b, np.zeros(L)]).astype(np.float32)


def decode_images(n_fft, hop, x_res, y_res):
    """(4, y_res, x_res) uint8: the oracle's encodings of `slices` and one random byte image."""
    enc = [mo.audio_slice_to_bytes(y, n_fft=n_fft, hop=hop, n_mels=y_res) for y in slices(n_fft, hop, x_res)]
    rnd = np.random.default_rng(7 * n_fft + hop).integers(0, 256, (y_res, x_res), dtype=np.uint8)
    return np.stack(enc + [rnd])


def gl_metrics(got, ref):
    err = got.astype(np.float64) - ref
    return float(np.linalg.norm(err) / np.linalg.norm(ref)), float(np.abs(err).max() / np.abs(ref).max())


def gl_batch(A0, n_iter, n_fft, hop, rounded):
    """Griffin-Lim of every image of the batch from its initial spectrum A0[i]: exact float64, or the rounded model."""
    mag = np.abs(A0)
    dt = np.float32 if rounded else np.float64
    return np.stack([mo.griffinlim(mag[i], n_iter, hop, n_fft, dtype=dt, angles0=A0[i], rounded=rounded)
                     for i in range(len(A0))])


def gl_floors(A0, n_fft, hop, iters=(1, 4, 32)):
    """{n_iter: (floor L2, floor max)}: the rounded model against exact float64 Griffin-Lim, and both references."""
    out = {}
    for k in iters:
        ex, rd = gl_batch(A0, k, n_fft, hop, False), gl_batch(A0, k, n_fft, hop, True)
        out[k] = (gl_metrics(rd, ex), ex, rd)
    return out


def _sig(x):
    return float(f"{x:.3g}")


def _mel(n_fft, hop, x_res, y_res, n_iter=32):
    from audio_diffusion_b200.mel import Mel
    return Mel(x_res=x_res, y_res=y_res, n_fft=n_fft, hop_length=hop, top_db=TOP_DB, n_iter=n_iter)


def _encode(mel, ys, dev, refs=None):
    """One b200ad_mel_encode_ref call: the uint8 images and the mel power they were quantised from."""
    from audio_diffusion_b200 import _lib
    basis_t, _ = mel._constants(dev)
    a = torch.from_numpy(ys).to(dev)
    n = a.shape[0]
    img = torch.empty((n, mel.y_res, mel.x_res), dtype=torch.uint8, device=dev)
    power = torch.empty((n, mel.y_res, mel.x_res), dtype=torch.float32, device=dev)
    r = None if refs is None else torch.tensor(refs, dtype=torch.float32, device=dev)
    scratch = mel._scratch(n, dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().b200ad_mel_encode_ref(C.byref(mel._cfg_c()), basis_t.data_ptr(), a.data_ptr(), img.data_ptr(),
                                                    n, None if r is None else r.data_ptr(), power.data_ptr(),
                                                    scratch.data_ptr(), scratch.numel(), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return img.cpu().numpy(), power.cpu().numpy()


def _decode(cfg, images, dev, n_iter):
    mel = _mel(*cfg, n_iter=n_iter)
    mel.phase_seed = SEED
    audio = mel.images_to_audio(images, device=dev)
    return audio, mel._constants(dev)[1].cpu().numpy()


def _header(name):
    print(f"\n{name} on {torch.cuda.get_device_properties(0).name} ({power_limit()})")


@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
def test_mel_power(cuda, cfg):
    n_fft, hop, x_res, y_res = cfg
    mel = _mel(*cfg)
    ys = slices(*cfg[:3])
    _, power = _encode(mel, ys, cuda)
    basis = mel._constants(cuda)[0].cpu().numpy().T            # (y_res, F) float32, the constant the kernel gets
    km = (basis != 0).sum(1)
    _header(f"E1 mel power {n_fft}/{hop} {x_res}x{y_res}")
    print(f"{'slice':>6s} {'worst err/bar':>14s} {'zeros':>7s} {'empty rows':>11s}")
    for i, y in enumerate(ys):
        ref = mo.mel_power64(y, basis, n_fft, hop)
        got = power[i].astype(np.float64)
        bar = (km[:, None] + 16) * U * ref
        zero = ref == 0
        worst = float((np.abs(got - ref)[~zero] / bar[~zero]).max()) if (~zero).any() else 0.0
        print(f"{i:6d} {worst:14.4f} {int(zero.sum()):7d} {int((km == 0).sum()):11d}")
        assert np.array_equal(got[zero], ref[zero]), f"slice {i}: non-zero power where the reference is exactly 0"
        assert worst <= 1.0, f"slice {i}: mel power off by {worst:.3f} x its bar"
        if i == 2:
            assert zero.all()
        if (km == 0).any():
            assert (got[km == 0] == 0).all()


def _u8_exact(power, ref, top_db=TOP_DB):
    """Pixels recomputed in float64 from the engine's mel power; returns (pixels, value before the truncating cast)."""
    ls = mo.power_to_db(power.astype(np.float64), ref=ref, top_db=top_db)
    v = ((ls + top_db) * 255 / top_db).clip(0, 255) + 0.5
    px = mo.db_to_u8(ls, top_db)
    assert np.array_equal(px, np.floor(v).astype(np.uint8))
    return px, v


@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
def test_db_u8(cuda, cfg):
    n_fft, hop, x_res, y_res = cfg
    mel = _mel(*cfg)
    ys = slices(*cfg[:3])
    _header(f"E2 dB / uint8 {n_fft}/{hop} {x_res}x{y_res}")
    print(f"{'ref':>8s} {'slice':>6s} {'pixels':>7s} {'exempt':>7s} {'differ':>7s}")
    for ref in ("max", 2.5):
        img, power = _encode(mel, ys, cuda, refs=None if ref == "max" else [ref] * len(ys))
        for i in range(len(ys)):
            want, v = _u8_exact(power[i], np.max if ref == "max" else np.float32(ref))
            exempt = np.abs(v - np.round(v)) < 1e-3
            d = img[i].astype(int) - want.astype(int)
            print(f"{ref!s:>8s} {i:6d} {d.size:7d} {int(exempt.sum()):7d} {int((d != 0).sum()):7d}")
            assert (d[~exempt] == 0).all(), f"ref {ref}, slice {i}: {int((d[~exempt] != 0).sum())} pixels differ"
            assert (np.abs(d[exempt]) <= 1).all()
        if ref == "max":
            assert (img[2] == 255).all()


def _ola_abs(A0, n_fft, hop):
    """Per trimmed output sample: sum |windowed frame term|, the float64-difference allowance, the float32 window
    sum-square."""
    frames = scipy.fft.irfft(A0, n=n_fft, axis=0)
    win = mo._hann(n_fft)
    T = A0.shape[-1]
    n = n_fft + hop * (T - 1)
    s, d, w = np.zeros(n), np.zeros(n), np.zeros(n)
    fmax = np.abs(frames).max(0)
    for f in range(T):
        s[f * hop: f * hop + n_fft] += np.abs(frames[:, f] * win)
        d[f * hop: f * hop + n_fft] += win * fmax[f]
        w[f * hop: f * hop + n_fft] += win ** 2
    cut = slice(n_fft // 2, n - n_fft // 2)
    return s[cut], d[cut], w[cut].astype(np.float32)


@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
def test_decode_istft(cuda, cfg):
    n_fft, hop, x_res, y_res = cfg
    imgs = decode_images(*cfg)
    audio, pinv = _decode(cfg, imgs, cuda, 0)
    A0 = mo.initial_spectrum(imgs, pinv, SEED, TOP_DB)
    _header(f"D1 n_iter 0 {n_fft}/{hop} {x_res}x{y_res}")
    print(f"{'image':>6s} {'worst err/bar':>14s} {'wss<=tiny':>10s} {'rel L2':>10s}")
    tiny = np.finfo(np.float32).tiny
    for i in range(len(imgs)):
        want = mo.griffinlim(np.abs(A0[i]), 0, hop, n_fft, dtype=np.float32, angles0=A0[i], rounded=True)
        s, dlt, wss = _ola_abs(A0[i], n_fft, hop)
        big = wss > tiny
        bar = 8 * U * s + 2.0 ** -42 * dlt
        bar[big] /= wss[big]
        err = np.abs(audio[i].astype(np.float64) - want)
        zero = bar == 0
        worst = float((err[~zero] / bar[~zero]).max())
        rel = float(np.linalg.norm(err) / np.linalg.norm(want))
        print(f"{i:6d} {worst:14.4f} {int((~big).sum()):10d} {rel:10.3e}")
        assert (~big).any() == (hop == n_fft)
        assert np.array_equal(audio[i][zero], want[zero]) and (want[~big] == 0).all()
        assert worst <= 1.0, f"image {i}: off by {worst:.3f} x its bar"


@pytest.mark.parametrize("cfg", CONFIGS, ids=CFG_IDS)
def test_griffinlim(cuda, cfg):
    n_fft, hop, x_res, y_res = cfg
    imgs = decode_images(*cfg)
    _header(f"D2 Griffin-Lim {n_fft}/{hop} {x_res}x{y_res}, batch {len(imgs)}")
    t0 = time.perf_counter()
    got = {k: _decode(cfg, imgs, cuda, k) for k in (1, 4, 32)}
    A0 = mo.initial_spectrum(imgs, got[1][1], SEED, TOP_DB)
    floors = gl_floors(A0, n_fft, hop)
    print(f"float64 references {time.perf_counter() - t0:.1f} s")
    bars = GL_BARS.get((n_fft, hop), {})
    print(f"{'n_iter':>6s} {'L2':>10s} {'bar':>10s} {'floor':>10s} {'max':>10s} {'bar':>10s} {'floor':>10s} "
          f"{'L2 vs rounded':>14s} {'max vs rounded':>15s}")
    over, bad = [], []
    for k, ((fl2, fmx), ex, rd) in floors.items():
        e = gl_metrics(got[k][0], ex)
        r = gl_metrics(got[k][0], rd.astype(np.float64))
        b = bars.get(k, (float("nan"),) * 2)
        print(f"{k:6d} {e[0]:10.3e} {b[0]:10.3e} {fl2:10.3e} {e[1]:10.3e} {b[1]:10.3e} {fmx:10.3e} {r[0]:14.3e} {r[1]:15.3e}")
        print(f"    bars as stated: {k}: ({_sig(3 * _sig(fl2))}, {_sig(3 * _sig(fmx))}),   # floor ({_sig(fl2)}, {_sig(fmx)})")
        if not all(v <= bb for v, bb in zip(e, b)):
            over.append((k, e, b))
        if not all(f < bb <= 3.3 * _sig(f) * (1 + 1e-9) for f, bb in zip((fl2, fmx), b)):
            bad.append((k, (fl2, fmx), b))
    assert not over, f"engine over its bars: {over}"
    assert not bad, f"bars not in (floor, 3.3 x floor]: {bad}"
