"""Generates tests/golden/* by running the reference's OWN Python files (read unchanged from a checkout of
teticio/audio-diffusion).  Run from the repo root:  python tests/golden/make_golden.py <reference checkout>

 * vae_key_map.json — output of audiodiffusion/utils.py::convert_ldm_vae_checkpoint on an ldm-format checkpoint of the
   config/ldm_autoencoder_kl.yaml shape: [hf key, shape] in the order the reference writes them.  Pins the parameter
   table of libb200ad's AutoencoderKL (b200ad_vae_param_name / _shape).
 * pipeline_ddpm_small.npz — audiodiffusion/pipeline_audio_diffusion.py::AudioDiffusionPipeline.__call__ (the reference
   file, on the import shim) driving the fp32 CPU oracle U-Net (seeded synthetic weights, oracle/unet_oracle.py) and the
   ORACLE's DDPM scheduler (oracle/schedulers_oracle.py - nothing of the product computes a number in this fixture; the
   product's own scheduler gives bit-identical images, which the generator asserts) for 6 steps from a given noise tensor
   with a CPU step generator: the uint8 images it returns.
   The GPU pipeline must reproduce them within the stated tolerance (tests/test_gpu_pipeline.py).
 * dropin_ref.npz — what tests/test_cpu_dropin.py compares the product against: the reference pipeline's images on the
   import shim, its audio-conditioned / in-painting images, DDIM inversion and slerp, the ldm -> diffusers VAE key mapping
   of its converter, and its Mel class's slicing bookkeeping (SHA-256 of the audio and of the slices).
The numerical content is the oracle's (diffusers cannot be imported here); what the fixtures pin is the reference
files' own logic: key mapping, loop order, noise draws, float->uint8 conversion.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF = sys.argv[1] if len(sys.argv) > 1 else sys.exit("usage: make_golden.py <reference checkout>")
sys.path[:0] = [ROOT, os.path.join(ROOT, "audio_diffusion_b200", "compat"), REF, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

SMALL = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256),
             down_block_types=("DownBlock2D", "AttnDownBlock2D"), up_block_types=("AttnUpBlock2D", "UpBlock2D"))


def vae_key_map():
    from audiodiffusion.utils import convert_ldm_vae_checkpoint
    from oracle.vae_oracle import VAEConfig, init_weights
    from test_cpu_dropin import _hf_to_ldm_vae
    w = init_weights(VAEConfig(), seed=0)
    conv = convert_ldm_vae_checkpoint(_hf_to_ldm_vae(w), None)
    out = [[k, list(v.shape)] for k, v in conv.items()]
    with open(os.path.join(ROOT, "tests", "golden", "vae_key_map.json"), "w") as f:
        json.dump({"source": "audiodiffusion/utils.py:156-291 convert_ldm_vae_checkpoint", "keys": out}, f, indent=0)
    print("vae_key_map.json", len(out))


def pipeline_small():
    from audiodiffusion.pipeline_audio_diffusion import AudioDiffusionPipeline as RefPipe
    from diffusers import DDPMScheduler as ProductDDPM      # the import shim = the product's scheduler (cross-check only)
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_oracle import UNetConfig, init_weights, unet_forward

    class OracleUNet:
        def __init__(self):
            self.cfg = UNetConfig(sample_size=(32, 32), **SMALL)
            self.w = init_weights(self.cfg, seed=11)
            self.sample_size = (32, 32)
            self.in_channels = 1

        def __call__(self, x, t):
            return {"sample": unet_forward(self.w, self.cfg, x, t)}

    class FakeMel:
        x_res, y_res, hop_length = 32, 32, 512

        def get_sample_rate(self):
            return 22050

        def image_to_audio(self, image):
            return np.zeros((self.x_res - 1) * self.hop_length, dtype=np.float32)

    noise = torch.randn(2, 1, 32, 32, generator=torch.Generator().manual_seed(42))

    def run(scheduler):
        pipe = RefPipe(vqvae=None, unet=OracleUNet(), mel=FakeMel(), scheduler=scheduler)
        pipe.set_progress_bar_config(disable=True)
        images, _ = pipe(batch_size=2, steps=6, noise=noise.clone(), step_generator=torch.Generator().manual_seed(7),
                         return_dict=False)
        return np.stack([np.asarray(im) for im in images]).astype(np.uint8)
    arr = run(OracleDDPM())
    assert np.array_equal(arr, run(ProductDDPM())), "the product's DDPMScheduler disagrees with the oracle's"

    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "pipeline_ddpm_small.npz"), noise=noise.numpy(), images=arr,
                        steps=6, weight_seed=11, step_seed=7)
    print("pipeline_ddpm_small.npz", arr.shape, arr.mean())


def dropin():
    import hashlib

    from audiodiffusion.mel import Mel as RefMel
    from audiodiffusion.pipeline_audio_diffusion import AudioDiffusionPipeline as RefPipe
    from audiodiffusion.utils import convert_ldm_vae_checkpoint
    from diffusers import DDIMScheduler, DDPMScheduler
    from oracle.vae_oracle import VAEConfig, init_weights
    from PIL import Image
    from test_cpu_dropin import FakeMel, OracleUNet, ScriptedMel, _hf_to_ldm_vae
    out = {}
    for sched in ("ddpm", "ddim"):
        is_ddim = sched == "ddim"
        pipe = RefPipe(vqvae=None, unet=OracleUNet(), mel=FakeMel(), scheduler=DDIMScheduler() if is_ddim else DDPMScheduler())
        pipe.set_progress_bar_config(disable=True)
        assert pipe.get_default_steps() == (50 if is_ddim else 1000)
        r = pipe(batch_size=2, steps=4, generator=torch.Generator().manual_seed(42))
        assert len(r.images) == 2 and r.audios.shape == (2, 1, 15 * 512)
        out[f"shim_{sched}"] = np.stack([np.asarray(im) for im in r.images])
        pipe = RefPipe(vqvae=None, unet=OracleUNet(), mel=ScriptedMel(), scheduler=DDIMScheduler() if is_ddim else DDPMScheduler())
        pipe.set_progress_bar_config(disable=True)
        images, (sr, audios) = pipe(**mirror_kwargs(is_ddim))
        assert sr == 22050 and len(audios) == 1
        out[f"mirror_{sched}"] = np.stack([np.asarray(im) for im in images])
    rng = np.random.default_rng(9)
    pil = [Image.fromarray(rng.integers(0, 256, (16, 16), dtype=np.uint8)) for _ in range(2)]
    pipe = RefPipe(vqvae=None, unet=OracleUNet(), mel=ScriptedMel(), scheduler=DDIMScheduler())
    pipe.set_progress_bar_config(disable=True)
    out["encode_ddim"] = pipe.encode(pil, steps=5).numpy()
    a, b = torch.randn(4, 4, generator=torch.Generator().manual_seed(1)), torch.randn(4, 4, generator=torch.Generator().manual_seed(2))
    out["slerp"] = RefPipe.slerp(a, b, 0.3).numpy()
    ldm = _hf_to_ldm_vae(init_weights(VAEConfig(), seed=3))
    tagged = {k: torch.tensor([float(i)]) for i, k in enumerate(ldm)}        # which ldm tensor lands under which key
    for k, v in ldm.items():
        if v.dim() == 4 and v.shape[2:] == (1, 1) and ".attn_1." in k:
            tagged[k] = tagged[k].reshape(1, 1, 1, 1).expand(v.shape[0], v.shape[1], 1, 1)
    conv = convert_ldm_vae_checkpoint(dict(tagged), None)
    out["vae_ldm_keys"] = np.array([list(ldm)[int(v.flatten()[0])] for v in conv.values()])
    out["vae_hf_keys"] = np.array(list(conv))
    out["vae_squeezed"] = np.array([v.dim() == 2 for v in conv.values()])
    mel = []
    rng = np.random.default_rng(0)
    for (x_res, y_res, hop) in MEL_CASES:
        for n in (10, x_res * hop - 1, x_res * hop, 3 * x_res * hop + 17):
            m = RefMel(x_res=x_res, y_res=y_res, hop_length=hop)
            m.load_audio(raw_audio=rng.standard_normal(n).astype(np.float32))
            h = hashlib.sha256(m.audio.tobytes())
            for i in range(m.get_number_of_slices()):
                h.update(m.get_audio_slice(i).tobytes())
            mel.append([m.slice_size, m.n_mels, m.get_sample_rate(), m.get_number_of_slices(), len(m.audio), str(m.audio.dtype),
                        h.hexdigest()])
        m.set_resolution(32, 16)
        mel.append([m.x_res, m.y_res, m.n_mels, m.slice_size])
    out["mel"] = np.array(json.dumps(mel))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "dropin_ref.npz"), **out)
    print("dropin_ref.npz", sorted(out))


if __name__ == "__main__":
    from test_cpu_dropin import MEL_CASES, mirror_kwargs
    vae_key_map()
    pipeline_small()
    dropin()
