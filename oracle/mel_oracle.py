"""numpy/scipy restatement of the librosa==0.10.2.post1 calls made by audiodiffusion/mel.py.

TEST INFRASTRUCTURE (see oracle/__init__.py).  PARITY UNPINNED (librosa absent).
Reference call sites: mel.py:145-149 (`audio_slice_to_image`: feature.melspectrogram ->
power_to_db -> uint8) and mel.py:162-167 (`image_to_audio`: db_to_power ->
feature.inverse.mel_to_audio = filters.mel + util.nnls + griffinlim).
"""
from __future__ import annotations

import numpy as np
import scipy.fft
import scipy.optimize
import scipy.signal


# --------------------------------------------------------------------------- filters.mel
def hz_to_mel(f):
    """librosa.hz_to_mel(htk=False) — Slaney's Auditory-Toolbox scale."""
    f = np.asanyarray(f, dtype=float)
    f_sp = 200.0 / 3
    mels = f / f_sp
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    if f.ndim:
        big = f >= min_log_hz
        mels[big] = min_log_mel + np.log(f[big] / min_log_hz) / logstep
    elif f >= min_log_hz:
        mels = min_log_mel + np.log(f / min_log_hz) / logstep
    return mels


def mel_to_hz(m):
    m = np.asanyarray(m, dtype=float)
    f_sp = 200.0 / 3
    freqs = f_sp * m
    min_log_hz = 1000.0
    min_log_mel = min_log_hz / f_sp
    logstep = np.log(6.4) / 27.0
    if m.ndim:
        big = m >= min_log_mel
        freqs[big] = min_log_hz * np.exp(logstep * (m[big] - min_log_mel))
    elif m >= min_log_mel:
        freqs = min_log_hz * np.exp(logstep * (m - min_log_mel))
    return freqs


def mel_filterbank(sr: int, n_fft: int, n_mels: int, dtype=np.float32) -> np.ndarray:
    """librosa.filters.mel(sr, n_fft, n_mels, fmin=0, fmax=sr/2, htk=False, norm='slaney')."""
    fmax = float(sr) / 2
    weights = np.zeros((n_mels, 1 + n_fft // 2), dtype=dtype)
    fftfreqs = np.fft.rfftfreq(n=n_fft, d=1.0 / sr)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(0.0), hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = np.subtract.outer(mel_f, fftfreqs)
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        weights[i] = np.maximum(0, np.minimum(lower, upper))
    enorm = 2.0 / (mel_f[2: n_mels + 2] - mel_f[:n_mels])
    weights *= enorm[:, np.newaxis]
    return weights


# --------------------------------------------------------------------------- stft / istft
def _hann(n_fft: int) -> np.ndarray:
    return scipy.signal.get_window("hann", n_fft, fftbins=True)


def stft(y: np.ndarray, n_fft: int, hop: int) -> np.ndarray:
    """librosa.stft(center=True, pad_mode='constant', window='hann', win_length=n_fft).

    librosa multiplies the frames by the float64 scipy window (no cast), so the FFT itself runs in float64
    and only the stored matrix is complex64 for float32 input (util.dtype_r2c)."""
    cdtype = np.complex64 if y.dtype == np.float32 else np.complex128
    win = _hann(n_fft)
    yp = np.pad(y, (n_fft // 2, n_fft // 2), mode="constant")
    n_frames = 1 + (len(yp) - n_fft) // hop
    idx = np.arange(n_fft)[:, None] + hop * np.arange(n_frames)[None, :]
    frames = win[:, None] * yp[idx]
    return scipy.fft.rfft(frames, axis=0).astype(cdtype, copy=False)


def istft(S: np.ndarray, n_fft: int, hop: int, dtype=np.float32, rounded: bool = False) -> np.ndarray:
    """librosa.istft(center=True, length=None, window='hann'): overlap-add / window-sumsquare.

    rounded=True applies the storage roundings of the CUDA decode (mel.cu gl_istft_kernel / ola_sample) and only those:
    the windowed frames are stored as float32, summed in float64, the sum is cast to float32 and divided in float32 by
    the float32 window sum-square where that is above FLT_MIN (left unnormalised elsewhere).  Returns float32."""
    n_frames = S.shape[-1]
    win = _hann(n_fft)
    expected = n_fft + hop * (n_frames - 1)
    ytmp = scipy.fft.irfft(S, n=n_fft, axis=0) * win[:, None]
    if rounded:
        ytmp = ytmp.astype(np.float32).astype(np.float64)
    y = np.zeros(expected, dtype=np.float64)
    wss = np.zeros(expected, dtype=np.float64)
    wsq = win ** 2
    for f in range(n_frames):
        y[f * hop: f * hop + n_fft] += ytmp[:, f]
        wss[f * hop: f * hop + n_fft] += wsq
    if rounded:
        y32, w32 = y.astype(np.float32), wss.astype(np.float32)
        nz = w32 > np.finfo(np.float32).tiny
        y32[nz] /= w32[nz]
        return y32[n_fft // 2: expected - n_fft // 2]
    tiny = np.finfo(np.float32 if dtype == np.float32 else np.float64).tiny
    nz = wss > tiny
    y[nz] /= wss[nz]
    y = y[n_fft // 2: expected - n_fft // 2]
    return y.astype(dtype)


# --------------------------------------------------------------------------- forward codec
def melspectrogram(y: np.ndarray, sr: int, n_fft: int, hop: int, n_mels: int) -> np.ndarray:
    """librosa.feature.melspectrogram(power=2.0) — mel.py:145-147."""
    S = np.abs(stft(y, n_fft, hop)) ** 2
    M = mel_filterbank(sr, n_fft, n_mels)
    return np.einsum("ft,mf->mt", S, M, optimize=True)


def mel_power64(y: np.ndarray, basis: np.ndarray, n_fft: int, hop: int) -> np.ndarray:
    """The mel power spectrogram (n_mels, frames) in float64: the float64 STFT power of `y` times `basis` promoted to
    float64.  Given the float32 basis the CUDA encode multiplies by, this is the exact value of what that kernel
    computes, with no rounding of the basis in between."""
    S = np.abs(stft(np.asarray(y, dtype=np.float64), n_fft, hop)) ** 2
    return basis.astype(np.float64) @ S


def power_to_db(S: np.ndarray, ref=np.max, amin: float = 1e-10, top_db: float = 80.0) -> np.ndarray:
    """librosa.power_to_db — mel.py:148."""
    S = np.asarray(S)
    ref_value = ref(S) if callable(ref) else np.abs(ref)
    log_spec = 10.0 * np.log10(np.maximum(amin, S))
    log_spec -= 10.0 * np.log10(np.maximum(amin, ref_value))
    if top_db is not None:
        log_spec = np.maximum(log_spec, log_spec.max() - top_db)
    return log_spec


def db_to_u8(log_S: np.ndarray, top_db: float) -> np.ndarray:
    """mel.py:149 — integer boundary, must be bit-exact."""
    return (((log_S + top_db) * 255 / top_db).clip(0, 255) + 0.5).astype(np.uint8)


def audio_slice_to_bytes(y: np.ndarray, sr=22050, n_fft=2048, hop=512, n_mels=256, top_db=80) -> np.ndarray:
    """Mel.audio_slice_to_image minus PIL: returns the (n_mels, frames) uint8 array (mel.py:135-151)."""
    S = melspectrogram(y, sr, n_fft, hop, n_mels)
    return db_to_u8(power_to_db(S, ref=np.max, top_db=top_db), top_db)


# --------------------------------------------------------------------------- inverse codec
def u8_to_power(b: np.ndarray, top_db: float = 80.0) -> np.ndarray:
    """mel.py:162-164: bytes -> float64 dB -> librosa.db_to_power."""
    log_S = b.astype("float") * top_db / 255 - top_db
    return np.power(10.0, 0.1 * log_S)


def _nnls_obj(x, shape, A, B):
    x = x.reshape(shape)
    diff = np.einsum("mf,...ft->...mt", A, x, optimize=True) - B
    value = (1 / B.size) * 0.5 * np.sum(diff ** 2)
    grad = (1 / B.size) * np.einsum("mf,...mt->...ft", A, diff, optimize=True)
    return value, grad.flatten()


def _nnls_lbfgs_block(A, B):
    x_init = np.einsum("fm,...mt->...ft", np.linalg.pinv(A), B, optimize=True)
    np.clip(x_init, 0, None, out=x_init)
    shape = x_init.shape
    bounds = [(0, None)] * x_init.size
    x, _, _ = scipy.optimize.fmin_l_bfgs_b(_nnls_obj, x_init, args=(shape, A, B), bounds=bounds)
    return x.reshape(shape)


def nnls(A: np.ndarray, B: np.ndarray) -> np.ndarray:
    """librosa.util.nnls: column-blocked L-BFGS-B (MAX_MEM_BLOCK = 2**18 bytes)."""
    n_columns = int((2 ** 8 * 2 ** 10) // (np.prod(B.shape[:-1]) * A.itemsize))
    n_columns = max(n_columns, 1)
    if B.shape[-1] <= n_columns:
        return _nnls_lbfgs_block(A, B).astype(A.dtype)
    x = np.einsum("fm,...mt->...ft", np.linalg.pinv(A), B, optimize=True)
    np.clip(x, 0, None, out=x)
    for bl_s in range(0, x.shape[-1], n_columns):
        bl_t = min(bl_s + n_columns, B.shape[-1])
        x[..., bl_s:bl_t] = _nnls_lbfgs_block(A, B[..., bl_s:bl_t])
    return x


def mel_to_stft(M: np.ndarray, sr: int, n_fft: int) -> np.ndarray:
    A = mel_filterbank(sr, n_fft, M.shape[-2], dtype=M.dtype)
    inv = nnls(A, M)
    return np.power(inv, 0.5, out=inv)


def griffinlim(S: np.ndarray, n_iter: int, hop: int, n_fft: int, momentum: float = 0.99,
               rng: np.random.Generator | None = None, dtype=np.float32, angles0: np.ndarray | None = None,
               rounded: bool = False) -> np.ndarray:
    """librosa.griffinlim(init='random', random_state=None).  The reference leaves the RNG unseeded
    (non-deterministic); pass `rng` to make the oracle reproducible, or `angles0`, the initial complex spectrum
    (magnitude included), to start where another implementation starts.

    With S float64 and dtype=float64 every step runs in float64 (the exact Griffin-Lim).  rounded=True (S float64)
    applies the storage roundings of the CUDA decode and only those: the float32 frames and overlap-add of
    istft(rounded=True), `rebuilt` and `tprev` stored as complex64, the momentum step and the phase normalisation in
    float64, the latter only where |angles| > 0."""
    cdtype = np.complex64 if S.dtype == np.float32 else np.complex128
    eps = np.finfo(S.dtype).tiny
    if angles0 is None:
        rng = rng or np.random.default_rng()
        angles = np.exp(2j * np.pi * rng.random(size=S.shape)).astype(cdtype)
        angles *= S
    else:
        angles = np.array(angles0, dtype=cdtype)
    tprev = None
    for _ in range(n_iter):
        inverse = istft(angles, n_fft, hop, dtype=dtype, rounded=rounded)
        rebuilt = stft(inverse, n_fft, hop)
        if rounded:
            angles = rebuilt.astype(np.complex128)
            if tprev is not None:
                angles -= (momentum / (1 + momentum)) * tprev.astype(np.complex128)
            a = np.abs(angles)
            nz = a > 0
            angles[nz] *= S[nz] / a[nz]
        else:
            angles = rebuilt.astype(cdtype, copy=True)
            if tprev is not None:
                angles -= (momentum / (1 + momentum)) * tprev
            angles /= np.abs(angles) + eps
            angles *= S
        tprev = rebuilt
    return istft(angles, n_fft, hop, dtype=dtype, rounded=rounded)


def phase_u01(seed: int, idx) -> np.ndarray:
    """mel.cu `u01`: splitmix64 of state seed + (idx + 1) * 0x9E3779B97F4A7C15, top 53 bits scaled to [0, 1)."""
    idx = np.asarray(idx, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + np.uint64(0x9E3779B97F4A7C15) * (idx + np.uint64(1))
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return (z >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def initial_spectrum(images: np.ndarray, pinv: np.ndarray, seed: int, top_db: float = 80.0) -> np.ndarray:
    """The CUDA decode's Griffin-Lim starting point for a batch of (n, n_mels, frames) uint8 images, as (n, bins,
    frames) complex128: sqrt(max(pinv @ db_to_power(image), 0)) (the inverse mel transform, see
    test_mel_nnls_is_initial_point_on_image_domain) times exp(2 pi i u), u = phase_u01(seed, (n * frames + t) * bins + f)."""
    n, _, T = images.shape
    F = pinv.shape[0]
    mag = np.sqrt(np.maximum(pinv @ u8_to_power(images, top_db), 0.0))
    o = (np.arange(n)[:, None, None] * T + np.arange(T)[None, None, :]) * F + np.arange(F)[None, :, None]
    return mag * np.exp(2j * np.pi * phase_u01(seed, o))


def bytes_to_audio(b: np.ndarray, sr=22050, n_fft=2048, hop=512, top_db=80, n_iter=32,
                   rng: np.random.Generator | None = None) -> np.ndarray:
    """Mel.image_to_audio minus PIL (mel.py:153-168). Output length (x_res-1)*hop."""
    S = u8_to_power(b, top_db)
    mag = mel_to_stft(S, sr, n_fft)
    return griffinlim(mag, n_iter, hop, n_fft, rng=rng, dtype=np.float32)
