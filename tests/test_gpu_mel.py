"""GPU parity of the Mel codec kernels (C ABI b200ad_mel_encode / b200ad_mel_decode) against the numpy/scipy
oracle of the librosa calls in audiodiffusion/mel.py.

Tolerances (stated): encode — the uint8 image must equal the oracle's on >= 99.5 % of pixels and never differ by
more than one grey level (fp64 FFT vs pocketfft and float32 log10 rounding can move a value across a truncation
boundary).  decode — Griffin-Lim starts from a random phase (unseeded in the reference), so audio is compared
in the mel domain: re-encoding our audio must be as close to the source image as re-encoding the oracle's audio
(mean abs grey-level difference within 1.0 of the oracle's own round-trip error)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _audio(n, seed=0, f=440.0):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 22050
    y = rng.standard_normal(n) * 0.05 + 0.5 * np.sin(2 * np.pi * f * t) + 0.2 * np.sin(2 * np.pi * 3.1 * f * t)
    return (y * np.linspace(0.2, 1.0, n)).astype(np.float32)


# every n_fft the codec accepts and the edges of tests/test_gpu_mel_fp64.py's table, plus the 64 x 64 default-size case
@pytest.mark.parametrize("n_fft,hop,x_res,y_res", [(64, 16, 64, 48), (128, 128, 32, 32), (256, 100, 64, 40),
                                                   (512, 128, 96, 64), (1024, 256, 128, 80), (2048, 512, 256, 256),
                                                   (2048, 1024, 64, 64), (2048, 2048, 64, 128), (4096, 1024, 128, 128)])
def test_encode_matches_oracle(cuda, n_fft, hop, x_res, y_res):
    from audio_diffusion_b200.mel import Mel
    from oracle import mel_oracle as mo
    mel = Mel(x_res=x_res, y_res=y_res, n_fft=n_fft, hop_length=hop)
    L = mel.slice_size
    ys = np.stack([_audio(L, seed=s, f=220.0 * (s + 1)) for s in range(3)] + [np.zeros(L, np.float32)])
    got = mel.audio_slices_to_images(ys, device=cuda).cpu().numpy()
    for i in range(len(ys)):
        ref = mo.audio_slice_to_bytes(ys[i], n_fft=n_fft, hop=hop, n_mels=y_res)
        diff = np.abs(got[i].astype(int) - ref.astype(int))
        assert diff.max() <= 1, f"slice {i}: max grey diff {diff.max()}"
        assert (diff == 0).mean() >= 0.995, f"slice {i}: only {(diff == 0).mean():.4f} identical"
    assert (got[-1] == 255).all()  # silent slice -> all 255 (audio_to_images.py:46)


def test_mel_api_single_slice_and_pil(cuda):
    from PIL import Image
    from audio_diffusion_b200.mel import Mel
    from oracle import mel_oracle as mo
    mel = Mel(x_res=64, y_res=64, hop_length=1024)
    y = _audio(3 * mel.slice_size + 100, seed=5)
    mel.load_audio(raw_audio=y)
    assert mel.get_number_of_slices() == 3
    img = mel.audio_slice_to_image(1)
    assert isinstance(img, Image.Image) and img.size == (64, 64) and img.mode == "L"
    ref = mo.audio_slice_to_bytes(mel.get_audio_slice(1), hop=1024, n_mels=64)
    assert np.abs(np.asarray(img).astype(int) - ref.astype(int)).max() <= 1


def test_decode_mel_domain(cuda):
    from audio_diffusion_b200.mel import Mel
    from oracle import mel_oracle as mo
    mel = Mel(x_res=64, y_res=64, hop_length=512)
    L = mel.slice_size
    y = _audio(L, seed=1)
    img = mo.audio_slice_to_bytes(y, hop=512, n_mels=64)
    audio = mel.images_to_audio(np.stack([img, img]))
    assert audio.shape == (2, (64 - 1) * 512) and audio.dtype == np.float32   # mel.py:165-167
    assert not np.array_equal(audio[0], audio[1])                             # independent random phases
    ref_audio = mo.bytes_to_audio(img, hop=512, rng=np.random.default_rng(0))
    pad = lambda a: np.concatenate([a, np.zeros(L - len(a), np.float32)])     # noqa: E731
    err_ref = np.abs(mo.audio_slice_to_bytes(pad(ref_audio), hop=512, n_mels=64).astype(int) - img.astype(int)).mean()
    for k in range(2):
        back = mo.audio_slice_to_bytes(pad(audio[k]), hop=512, n_mels=64)
        err = np.abs(back.astype(int) - img.astype(int)).mean()
        assert err <= err_ref + 1.0, f"round trip {err:.2f} vs oracle {err_ref:.2f}"
    # signal level agrees with the oracle's reconstruction
    assert abs(np.sqrt((audio[0] ** 2).mean()) / np.sqrt((ref_audio ** 2).mean()) - 1) < 0.1


def test_decode_one_iteration_deterministic_part(cuda):
    """With n_iter = 0 the decode is istft(mag * exp(i phi)): its spectrum magnitude must reproduce
    sqrt(max(pinv(A) S, 0)) — checks the inverse-mel GEMM and the iSTFT independently of Griffin-Lim."""
    from audio_diffusion_b200.mel import Mel
    from oracle import mel_oracle as mo
    mel = Mel(x_res=64, y_res=64, hop_length=512, n_iter=0)
    img = mo.audio_slice_to_bytes(_audio(mel.slice_size, seed=2), hop=512, n_mels=64)
    a0 = mel.images_to_audio(img[None])[0]
    mag = mo.mel_to_stft(mo.u8_to_power(img), 22050, 2048)
    # energy of istft(random phase) concentrates where mag does: compare band energies of re-analysis
    S = np.abs(mo.stft(np.concatenate([a0, np.zeros(mel.slice_size - len(a0), np.float32)]), 2048, 512)) ** 2
    e_ref = (mag ** 2).sum(1)
    e_got = S.sum(1)
    top = np.argsort(e_ref)[-20:]
    ratio = e_got[top].sum() / e_ref[top].sum()
    assert 0.2 < ratio < 1.5, ratio


@pytest.mark.parametrize("ref", [1.0, 25.0, "median"])
def test_encode_with_other_ref(cuda, ref):
    """`Mel.audio_slice_to_image(slice, ref=...)` (mel.py:135) accepts any scalar or callable for librosa.power_to_db's
    reference power; the default np.max is the fast path, everything else goes through b200ad_mel_encode_ref."""
    from audio_diffusion_b200.mel import Mel
    from oracle import mel_oracle as mo
    mel = Mel(x_res=64, y_res=64, hop_length=1024)
    y = _audio(mel.slice_size, seed=3, f=330.0)
    r = np.median if ref == "median" else ref
    mel.load_audio(raw_audio=y)
    got = np.asarray(mel.audio_slice_to_image(0, ref=r))
    S = mo.melspectrogram(y, 22050, 2048, 1024, 64)
    want = mo.db_to_u8(mo.power_to_db(S, ref=r, top_db=80), 80)
    diff = np.abs(got.astype(int) - want.astype(int))
    assert diff.max() <= 1 and (diff == 0).mean() >= 0.995, (diff.max(), (diff == 0).mean())
