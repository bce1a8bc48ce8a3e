"""CPU tests of the drop-in boundary: the product's pipeline, schedulers, VAE parameter table and Mel bookkeeping against
what the UNCHANGED reference files computed on top of the import shim (`audio_diffusion_b200/compat`), stored in
tests/golden/dropin_ref.npz by tests/golden/make_golden.py; and the N>1 path's host logic (weight broadcast + batch
sharding) over gloo with world_size 2.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MEL_CASES = [(256, 256, 512), (64, 64, 1024), (96, 32, 256)]


def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "dropin_ref.npz"))


def mirror_kwargs(is_ddim):
    """Arguments of the audio-conditioned / in-painting call (`raw_audio`, `start_step`, `mask_start_secs`,
    `mask_end_secs`, pipeline_audio_diffusion.py:133-185); the reference's start_step path is batch-1 only (:150)."""
    noise = torch.randn(1, 1, 16, 16, generator=torch.Generator().manual_seed(3))
    kw = dict(batch_size=1, raw_audio=np.zeros(16 * 512 * 2, dtype=np.float32), slice=0, start_step=2, steps=6, noise=noise,
              step_generator=torch.Generator().manual_seed(4), mask_start_secs=0.05, mask_end_secs=0.05, return_dict=False)
    if is_ddim:
        kw["eta"] = 0.5
    return kw


class OracleUNet:
    """Stand-in with the duck type the reference pipeline needs (callable, sample_size, in_channels), CPU oracle inside."""

    def __init__(self):
        from oracle.unet_oracle import UNetConfig, init_weights
        self.cfg = UNetConfig(sample_size=(16, 16), block_out_channels=(128, 128),
                              down_block_types=("DownBlock2D", "DownBlock2D"), up_block_types=("UpBlock2D", "UpBlock2D"),
                              layers_per_block=1)
        self.w = init_weights(self.cfg, seed=0)
        self.sample_size = 16
        self.in_channels = 1

    def __call__(self, x, t):
        from oracle.unet_oracle import unet_forward
        return {"sample": unet_forward(self.w, self.cfg, x, t)}


class FakeMel:
    x_res, y_res, hop_length = 16, 16, 512

    def get_sample_rate(self):
        return 22050

    def image_to_audio(self, image):
        return np.zeros((self.x_res - 1) * self.hop_length, dtype=np.float32)


@pytest.mark.parametrize("sched", ["ddpm", "ddim"])
def test_unchanged_reference_pipeline_runs_on_the_shim(sched):
    """The reference pipeline file on the shim's schedulers (stored uint8 images) == the same loop by hand with the oracle
    schedulers and the oracle U-Net."""
    from oracle.schedulers_oracle import OracleDDIM, OracleDDPM
    from oracle.unet_oracle import unet_forward
    is_ddim = sched == "ddim"
    unet = OracleUNet()
    g = torch.Generator().manual_seed(42)
    x = torch.randn((2, 1, 16, 16), generator=g)
    o = OracleDDIM() if is_ddim else OracleDDPM()
    o.set_timesteps(4)
    for t in o.timesteps:
        eps = unet_forward(unet.w, unet.cfg, x, t)
        x = (o.step(eps, t, x, eta=0, generator=g) if is_ddim else o.step(eps, t, x, generator=g))["prev_sample"]
    ref = ((x / 2 + 0.5).clamp(0, 1).permute(0, 2, 3, 1).numpy() * 255).round().astype("uint8")[..., 0]
    got = golden()[f"shim_{sched}"]
    assert np.array_equal(got, ref), np.abs(got.astype(int) - ref.astype(int)).max()


def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from audio_diffusion_b200.parallel import broadcast_parameters, shard_noise
    torch.manual_seed(100 + rank)                       # ranks start with different weights
    params = [torch.nn.Parameter(torch.randn(5, 3)), torch.nn.Parameter(torch.randn(7))]
    broadcast_parameters(params, src=0)
    full = torch.randn(8, 1, 4, 4, generator=torch.Generator().manual_seed(42))
    mine = shard_noise((8, 1, 4, 4), torch.Generator().manual_seed(42), rank, world, device="cpu")
    # numpy, not tensors: a tensor sent through the queue is fetched from this process, which may have exited by then
    q.put((rank, [p.detach().numpy().copy() for p in params], mine.numpy(), full.numpy()))
    dist.barrier()
    dist.destroy_process_group()


def test_weight_broadcast_and_noise_sharding_gloo_world2():
    """⑤ multi-GPU host logic: one broadcast of the weights, batch rows sliced from ONE global RNG stream so that
    results are shard-count invariant (SURVEY §8e)."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=120) for _ in procs], key=lambda r: r[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (r0, p0, m0, full), (r1, p1, m1, _) = [(r, [torch.from_numpy(a) for a in p], torch.from_numpy(m), torch.from_numpy(f))
                                          for r, p, m, f in res]
    assert all(torch.equal(a, b) for a, b in zip(p0, p1))            # weights identical after the broadcast
    assert torch.equal(torch.cat([m0, m1]), full)                    # shards tile the global noise stream


def _hf_to_ldm_vae(w, num_blocks=4):
    """Inverse of the reference's key mapping: an `ldm` AutoencoderKL state dict (CompVis naming: down.{i}.block.{j},
    mid.block_1 / attn_1 / block_2, up.{i} counted from the LOW-resolution end, 1x1-conv attention projections)."""
    out = {}
    for k, v in w.items():
        n = k
        n = n.replace("conv_norm_out", "norm_out")
        for i in range(num_blocks):
            n = n.replace(f"encoder.down_blocks.{i}.resnets.", f"encoder.down.{i}.block.")
            n = n.replace(f"encoder.down_blocks.{i}.downsamplers.0.", f"encoder.down.{i}.downsample.")
        if n.startswith("decoder.up_blocks."):
            i = int(n.split(".")[2])
            n = n.replace(f"decoder.up_blocks.{i}.resnets.", f"decoder.up.{num_blocks - 1 - i}.block.")
            n = n.replace(f"decoder.up_blocks.{i}.upsamplers.0.", f"decoder.up.{num_blocks - 1 - i}.upsample.")
        n = n.replace("mid_block.resnets.0", "mid.block_1").replace("mid_block.resnets.1", "mid.block_2")
        if "mid_block.attentions.0" in n:
            n = n.replace("mid_block.attentions.0", "mid.attn_1")
            n = (n.replace("group_norm", "norm").replace("to_q", "q").replace("to_k", "k").replace("to_v", "v")
                  .replace("to_out.0", "proj_out"))
            if n.endswith(".weight") and v.dim() == 2:
                v = v[:, :, None, None]
        n = n.replace("conv_shortcut", "nin_shortcut")
        out[n] = v.clone()
    return out


def test_reference_vae_converter_feeds_the_b200_autoencoder():
    """audiodiffusion/utils.py:156-291 (`convert_ldm_vae_checkpoint`, its stored key mapping) turns an ldm-format
    checkpoint into exactly the state dict the product's `AutoencoderKL` loads: the library's parameter table (names and
    shapes) is pinned against the reference's own converter."""
    from audio_diffusion_b200.vae import AutoencoderKL
    from oracle.vae_oracle import VAEConfig, init_weights
    w = init_weights(VAEConfig(), seed=3)
    ldm = _hf_to_ldm_vae(w)
    assert any(k.startswith("encoder.down.0.block.0.") for k in ldm) and "decoder.mid.attn_1.q.weight" in ldm
    assert ldm["decoder.mid.attn_1.q.weight"].dim() == 4
    z = golden()
    conv = {}
    for hf, lk, sq in zip(z["vae_hf_keys"], z["vae_ldm_keys"], z["vae_squeezed"]):
        conv[str(hf)] = ldm[str(lk)][:, :, 0, 0] if sq and ldm[str(lk)].dim() == 4 else ldm[str(lk)]
    vae = AutoencoderKL(in_channels=1, out_channels=1, down_block_types=("DownEncoderBlock2D",) * 4,
                        up_block_types=("UpDecoderBlock2D",) * 4, block_out_channels=(128, 256, 512, 512),
                        layers_per_block=2, latent_channels=1)
    vae.load_state_dict(conv)                                               # strict: every key must land
    sd = vae.state_dict()
    assert set(sd) == set(w) and len(sd) == 248
    for k in w:
        assert torch.equal(sd[k], w[k]), k


def test_gradient_allreduce_gloo_world2():
    """Data-parallel training's host logic (scripts/train_unet.py:181,259 via accelerate DDP): one all-reduce of the flat
    gradient buffer, mean over ranks — over gloo with world_size 2 (NCCL on the GPU box)."""
    code = f"""
import os, sys
sys.path.insert(0, {ROOT!r})
import torch, torch.distributed as dist
from audio_diffusion_b200.parallel import allreduce_mean_
rank = int(os.environ['RANK'])
dist.init_process_group('gloo', rank=rank, world_size=2)
flat = torch.arange(1000, dtype=torch.float32) * (rank + 1)
allreduce_mean_(flat)
assert torch.equal(flat, torch.arange(1000, dtype=torch.float32) * 1.5), flat[:4]
dist.destroy_process_group()
print('OK', rank)
"""
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT="29617", WORLD_SIZE="2")
    procs = [subprocess.Popen([sys.executable, "-c", code], env=dict(env, RANK=str(r)), stdout=subprocess.PIPE,
                              stderr=subprocess.PIPE, text=True) for r in range(2)]
    outs = [p.communicate(timeout=300) for p in procs]
    for p, (o, e) in zip(procs, outs):
        assert p.returncode == 0 and "OK" in o, o + e


def test_pipeline_directory_round_trip(tmp_path):
    """`pipeline.save_pretrained(dir)` / `AudioDiffusionPipeline.from_pretrained(dir)` (scripts/train_unet.py:106-111,
    :302-303; audiodiffusion/__init__.py:30-32) in the diffusers directory layout — model_index.json, unet/, vqvae/,
    scheduler/, mel/ — including a latent pipeline's AutoencoderKL and the deprecated attention key names of old hub files.
    Host logic only (no kernels run)."""
    import json

    from safetensors.torch import load_file, save_file

    from audio_diffusion_b200.mel import Mel
    from audio_diffusion_b200.pipeline import AudioDiffusionPipeline
    from audio_diffusion_b200.schedulers import DDIMScheduler
    from audio_diffusion_b200.unet import UNet2DModel
    from audio_diffusion_b200.vae import AutoencoderKL

    unet = UNet2DModel(sample_size=(8, 8), in_channels=1, out_channels=1, layers_per_block=1, block_out_channels=(128, 128),
                       down_block_types=("DownBlock2D", "AttnDownBlock2D"), up_block_types=("AttnUpBlock2D", "UpBlock2D"),
                       seed=1)
    vae = AutoencoderKL(in_channels=1, out_channels=1, down_block_types=("DownEncoderBlock2D",) * 2,
                        up_block_types=("UpDecoderBlock2D",) * 2, block_out_channels=(128, 128), layers_per_block=1,
                        latent_channels=1, seed=2)
    pipe = AudioDiffusionPipeline(vqvae=vae, unet=unet, mel=Mel(x_res=16, y_res=16, hop_length=256), scheduler=DDIMScheduler())
    d = str(tmp_path / "pipe")
    pipe.save_pretrained(d)
    idx = json.load(open(os.path.join(d, "model_index.json")))
    assert idx["unet"][1] == "UNet2DModel" and idx["vqvae"][1] == "AutoencoderKL" and idx["scheduler"][1] == "DDIMScheduler"
    # rewrite the U-Net weights with the deprecated attention names of older hub checkpoints
    f = os.path.join(d, "unet", "diffusion_pytorch_model.safetensors")
    sd = load_file(f)
    ren = {".to_q.": ".query.", ".to_k.": ".key.", ".to_v.": ".value.", ".to_out.0.": ".proj_attn."}
    old = {}
    for k, v in sd.items():
        for a, b in ren.items():
            k = k.replace(a, b)
        old[k] = v
    assert any(".query." in k for k in old)
    save_file(old, f)
    back = AudioDiffusionPipeline.from_pretrained(d)
    assert isinstance(back.scheduler, DDIMScheduler) and back.mel.x_res == 16 and back.mel.hop_length == 256
    for k, v in unet.state_dict().items():
        assert torch.equal(back.unet.state_dict()[k], v), k
    for k, v in vae.state_dict().items():
        assert torch.equal(back.vqvae.state_dict()[k], v), k
    assert back.unet.sample_size in ((8, 8), [8, 8]) and back.vqvae.config["latent_channels"] == 1


class ScriptedMel(FakeMel):
    """FakeMel plus the audio-conditioning surface (`load_audio`, `audio_slice_to_image`) with a fixed image."""

    def load_audio(self, audio_file=None, raw_audio=None):
        self.loaded = True

    def audio_slice_to_image(self, slice):
        from PIL import Image
        rng = np.random.default_rng(5)
        return Image.fromarray(rng.integers(0, 256, (self.y_res, self.x_res), dtype=np.uint8))


@pytest.mark.parametrize("sched", ["ddpm", "ddim"])
def test_mirrored_pipeline_equals_reference_pipeline_on_cpu(sched):
    """The product's own `AudioDiffusionPipeline.__call__` (audio_diffusion_b200/pipeline.py) against the reference's
    unchanged file for the audio-conditioned / in-painting path: identical uint8 images; for DDIM also inversion (`encode`,
    :207-242) and `slerp` (:244-263). Both drove the CPU oracle U-Net (the mirror then takes its unfused branch); only the
    mirror's float->uint8 CUDA kernel is replaced by the same torch expression."""
    from PIL import Image

    from audio_diffusion_b200.pipeline import AudioDiffusionPipeline as Mirror
    from audio_diffusion_b200.schedulers import DDIMScheduler, DDPMScheduler
    is_ddim = sched == "ddim"
    z = golden()
    u8 = Mirror.__dict__["images_to_u8"]
    Mirror.images_to_u8 = staticmethod(lambda x: ((x / 2 + 0.5).clamp(0, 1) * 255).round().to(torch.uint8))
    try:
        pipe = Mirror(vqvae=None, unet=OracleUNet(), mel=ScriptedMel(), scheduler=(DDIMScheduler() if is_ddim else DDPMScheduler()))
        pipe.set_progress_bar_config(disable=True)
        images, (sr, audios) = pipe(**mirror_kwargs(is_ddim))
        got = np.stack([np.asarray(im) for im in images])
        assert sr == 22050 and len(audios) == 1
        ref = z[f"mirror_{sched}"]
        assert ref.shape == (1, 16, 16) and np.array_equal(got, ref), np.abs(got.astype(int) - ref.astype(int)).max()
        if is_ddim:
            rng = np.random.default_rng(9)
            pil = [Image.fromarray(rng.integers(0, 256, (16, 16), dtype=np.uint8)) for _ in range(2)]
            pipe = Mirror(vqvae=None, unet=OracleUNet(), mel=ScriptedMel(), scheduler=DDIMScheduler())
            pipe.set_progress_bar_config(disable=True)
            enc = pipe.encode(pil, steps=5)
            assert enc.shape == (2, 1, 16, 16) and torch.equal(enc, torch.from_numpy(z["encode_ddim"]))
            a = torch.randn(4, 4, generator=torch.Generator().manual_seed(1))
            b = torch.randn(4, 4, generator=torch.Generator().manual_seed(2))
            assert torch.equal(Mirror.slerp(a, b, 0.3), torch.from_numpy(z["slerp"]))
    finally:
        Mirror.images_to_u8 = u8


def test_mel_host_logic_equals_reference_mel():
    """Slicing / padding / resolution bookkeeping of the engine's `Mel` against the reference's own `audiodiffusion/mel.py`
    class (stored sizes and SHA-256 of the audio and its slices; its librosa-backed transforms are not called): mel.py:80-133."""
    import hashlib
    import json

    from audio_diffusion_b200.mel import Mel
    ref = json.loads(str(golden()["mel"]))
    got = []
    rng = np.random.default_rng(0)
    for (x_res, y_res, hop) in MEL_CASES:
        for n in (10, x_res * hop - 1, x_res * hop, 3 * x_res * hop + 17):
            m = Mel(x_res=x_res, y_res=y_res, hop_length=hop)
            m.load_audio(raw_audio=rng.standard_normal(n).astype(np.float32))
            h = hashlib.sha256(m.audio.tobytes())
            for i in range(m.get_number_of_slices()):
                h.update(m.get_audio_slice(i).tobytes())
            got.append([m.slice_size, m.n_mels, m.get_sample_rate(), m.get_number_of_slices(), len(m.audio), str(m.audio.dtype),
                        h.hexdigest()])
        m.set_resolution(32, 16)
        got.append([m.x_res, m.y_res, m.n_mels, m.slice_size])
    assert got == ref


def test_conditional_unet_surface():
    """SURVEY §8 f3 boundary: `diffusers.UNet2DConditionModel` of the import shim resolves to the engine's class with
    exactly the diffusers state-dict keys / shapes of the architecture scripts/train_unet.py:139-159 builds."""
    code = f"""
import sys
sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'audio_diffusion_b200', 'compat')!r}]
from diffusers import UNet2DConditionModel
from audio_diffusion_b200.unet_cond import UNet2DConditionModel as engine_cls
assert UNet2DConditionModel is engine_cls
u = UNet2DConditionModel(sample_size=(32, 32), in_channels=1, out_channels=1, layers_per_block=2,
                         block_out_channels=(128, 256, 512, 512),
                         down_block_types=("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",),
                         up_block_types=("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3, cross_attention_dim=100)
from oracle.unet_cond_oracle import CondUNetConfig, param_shapes
sh = param_shapes(CondUNetConfig(sample_size=(32, 32)))
sd = u.state_dict()
assert set(sh) == set(sd) and all(tuple(sd[k].shape) == tuple(sh[k]) for k in sh)
assert sum(v.numel() for v in sd.values()) == 135559809
print('ok')
"""
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-2000:]


def test_grad_bucket_bounds_are_parameter_boundaries():
    """Buckets of the (opt-in) overlapped gradient all-reduce: ascending, start at 0, end at the buffer size, every inner
    boundary on a parameter's start offset (b200ad_unet_set_grad_buckets requires it)."""
    from audio_diffusion_b200.parallel import grad_bucket_bounds
    sizes = [1152, 128, 147456, 128, 65536, 512, 589824, 256, 36864, 128]
    offs, tot = [], 0
    for n in sizes:
        offs.append(tot)
        tot += n
    b = grad_bucket_bounds(offs, tot, nbuckets=4)
    assert b[0] == 0 and b[-1] == tot and all(x < y for x, y in zip(b, b[1:]))
    assert all(x in offs for x in b[1:-1])
    assert grad_bucket_bounds([0], 100, nbuckets=4) == [0, 100]          # a single tensor: one bucket


def test_bench_extras_formatting():
    """bench.py's `configs` object (C3 / C4 / B1 / C5 / Mel) is assembled on the host from a flat {name: seconds} dict that
    travelled through a max-over-ranks all-reduce: every sub-object and the rates derived from it."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(os.path.dirname(__file__), "..", "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    ex = {"c3_step_s": 0.035, "c3_tail_s": 0.07, "c3_call50_s": 1.82, "mel_encode_s": 0.0013, "mel_decode_s": 0.034,
          "c4_step_s": 0.0081, "c4_tail_s": 0.18, "c4_vae_decode_s": 0.078, "b1_step_s": 0.0046, "b1_host_enqueue_s": 0.0044,
          "b1_launches": 123.0, "b1_graph_step_s": 0.0044, "c5_step_s": 0.051, "c5_step_nosync_s": 0.050, "c5_launches": 830.0}
    out = bench.format_extras(ex, 2, 1439.1, 6572.5)
    assert set(out) == {"C3_ddim50", "C4_latent", "B1_latency", "C5_train", "mel_codec"}
    assert abs(out["C3_ddim50"]["value"] - 128 / (50 * 0.035 + 0.07)) < 1e-9
    assert abs(out["C5_train"]["value"] - 32 / 0.051) < 1e-9 and abs(out["C5_train"]["exposed_allreduce_ms"] - 1.0) < 1e-6
    assert out["B1_latency"]["ms_per_step"] == 4.4 and out["mel_codec"]["decode_frac"] < 1
