"""The launch sequence of the engine's plans, for checking that a host-side change leaves it alone.

For each workload it records every kernel, memset and copy the step puts on the GPU, in order, with grid and block dims
(torch.profiler with CUDA activities), the library's launch counts and plan sizes, and for the U-Net forward the op kinds
and FLOPs b200ad_unet_profile_step reports.  Run it once per library build (B200AD_LIB selects one) and compare the JSON
files: they must be equal.  With --tensors it also saves each workload's outputs and flat gradient buffer (`<name>.pt`)
for a numerical comparison.  Needs a CUDA device.

    B200AD_LIB=/path/to/libb200ad_old.so python tools/launch_trace.py --out trace_old --tensors
    python tools/launch_trace.py --out trace_new --tensors
"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from audio_diffusion_b200 import _lib  # noqa: E402
from audio_diffusion_b200.schedulers import DDPMScheduler  # noqa: E402
from audio_diffusion_b200.training import vae_loss  # noqa: E402
from audio_diffusion_b200.unet import UNet2DModel  # noqa: E402
from audio_diffusion_b200.unet_cond import UNet2DConditionModel  # noqa: E402
from audio_diffusion_b200.vae import AutoencoderKL  # noqa: E402

# the published model (teticio/audio-diffusion-256), as bench.py runs it
UNET_ARCH = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 128, 256, 256, 512, 512),
                 down_block_types=("DownBlock2D",) * 4 + ("AttnDownBlock2D", "DownBlock2D"),
                 up_block_types=("UpBlock2D", "AttnUpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D"))
# the conditional model train_unet.py --encodings builds (tests/test_gpu_cond_train.py)
COND_ARCH = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256, 512, 512),
                 down_block_types=("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",),
                 up_block_types=("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3, cross_attention_dim=100)
# ldm's autoencoder (config/ldm_autoencoder_kl.yaml)
VAE_ARCH = dict(in_channels=1, out_channels=1, down_block_types=("DownEncoderBlock2D",) * 4,
                up_block_types=("UpDecoderBlock2D",) * 4, block_out_channels=(128, 256, 512, 512), layers_per_block=2,
                latent_channels=1)


def traced(fn):
    """fn()'s result and the GPU work it enqueued: [name, grid, block] per kernel / memset / copy, in stream order."""
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    gpu = [e for e in events if e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")]
    gpu.sort(key=lambda e: e["ts"])
    return out, [[e["name"], e.get("args", {}).get("grid"), e.get("args", {}).get("block")] for e in gpu]


def seeded(seed, *shape, dev):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(dev)


def unet_forward(dev):
    """One fused denoising step of the published U-Net, batch 4, 256 x 256, then profile_step's op kinds and FLOPs."""
    model = UNet2DModel(sample_size=(256, 256), seed=0, **UNET_ARCH).to(dev).eval()
    sch = DDPMScheduler()
    sch.set_timesteps(1000)
    t = sch.timesteps[10]
    coef = sch.step_coef(t)
    x, z = seeded(1, 4, 1, 256, 256, dev=dev), seeded(2, 4, 1, 256, 256, dev=dev)
    with torch.no_grad():
        out, seq = traced(lambda: model.forward_step(x, t, coef, noise=z))
    rec = {"launches": seq, "last_launch_count": model.last_launch_count,
           "workspace_bytes": _lib.lib().b200ad_unet_workspace_bytes(model._h, 4, 256, 256)}
    L = _lib.lib()
    maxops = 1024
    op_ms, op_kind, op_fl = (C.c_float * maxops)(), (C.c_int * maxops)(), (C.c_double * maxops)()
    tt = model._timesteps(t, 4, dev)
    xo = torch.empty_like(x)
    n = L.b200ad_unet_profile_step(model._h, x.data_ptr(), tt.data_ptr(), z.data_ptr(), C.byref(coef), xo.data_ptr(),
                                   op_ms, op_kind, op_fl, maxops, _lib.stream_ptr())
    _lib.check(min(n, 0))
    rec["profile_op_kind"] = [op_kind[i] for i in range(n)]
    rec["profile_op_flops"] = [op_fl[i] for i in range(n)]
    return rec, {"sample": out}


def _unet_train(model, dev, n, hw, enc=None):
    sch = DDPMScheduler()
    clean = seeded(3, n, 1, hw, hw, dev=dev).clamp(-1, 1)
    noise = seeded(4, n, 1, hw, hw, dev=dev)
    t = torch.tensor([37, 712][:n], device=dev)
    noisy = sch.add_noise(clean, noise, t)

    def step():
        pred = model(noisy, t)["sample"] if enc is None else model(noisy, t, enc)["sample"]
        torch.nn.functional.mse_loss(pred, noise).backward()
        return pred.detach()
    pred, seq = traced(step)
    L = _lib.lib()
    rec = {"launches": seq, "last_launch_count": model.last_launch_count,
           "last_backward_launch_count": model.last_backward_launch_count,
           "workspace_bytes": L.b200ad_unet_workspace_bytes(model._h, n, hw, hw),
           "backward_bytes": L.b200ad_unet_backward_bytes(model._h)}
    return rec, {"sample": pred, "grad_flat": model._grad_flat.clone()}


def unet_train(dev):
    """One training step (forward + MSE + backward) of the published U-Net, batch 2, 256 x 256."""
    return _unet_train(UNet2DModel(sample_size=(256, 256), seed=0, **UNET_ARCH).to(dev).train(), dev, 2, 256)


def cond_train(dev):
    """One training step of the conditional U-Net at its 64 x 64 latent, batch 1, encoder sequence length 1."""
    model = UNet2DConditionModel(sample_size=(64, 64), seed=0, **COND_ARCH).to(dev).train()
    return _unet_train(model, dev, 1, 64, enc=seeded(5, 1, 1, 100, dev=dev))


def vae_infer(dev):
    """Encode and decode with the autoencoder, batch 2, 256 x 256."""
    vae = AutoencoderKL(seed=0, **VAE_ARCH).to(dev).eval()
    x = seeded(6, 2, 1, 256, 256, dev=dev).clamp(-1, 1)
    noise = torch.Generator().manual_seed(7)
    with torch.no_grad():
        z, enc_seq = traced(lambda: vae.encode(x).latent_dist.sample(generator=noise))
        enc_launches = vae.last_launch_count
        y, dec_seq = traced(lambda: vae.decode(z).sample)
    rec = {"encode": enc_seq, "encode_launch_count": enc_launches, "decode": dec_seq,
           "decode_launch_count": vae.last_launch_count,
           "workspace_bytes": _lib.lib().b200ad_vae_workspace_bytes(vae._h, 2, 256, 256)}
    return rec, {"z": z, "image": y}


def vae_train(dev):
    """One training step of the autoencoder (encode, sample, decode, L1 + KL, backward), batch 2, 64 x 64."""
    vae = AutoencoderKL(seed=0, max_batch=2, **VAE_ARCH).to(dev).train()
    x = seeded(8, 2, 1, 64, 64, dev=dev).clamp(-1, 1)
    noise = torch.Generator().manual_seed(9)

    def step():
        posterior = vae.encode(x).latent_dist
        y = vae.decode(posterior.sample(generator=noise)).sample
        vae_loss(x, y, posterior)[0].backward()
        return y.detach()
    y, seq = traced(step)
    rec = {"launches": seq, "last_launch_count": vae.last_launch_count, "backward_launch_count": vae.last_backward_launch_count,
           "backward_bytes": _lib.lib().b200ad_vae_backward_bytes(vae._h)}
    return rec, {"image": y, "grad_flat": vae._grad_flat.clone()}


WORKLOADS = {"unet_forward": unet_forward, "unet_train": unet_train, "cond_train": cond_train, "vae_infer": vae_infer,
             "vae_train": vae_train}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True, help="output directory (launch_trace.json, <workload>.pt)")
    ap.add_argument("--tensors", action="store_true", help="also save each workload's outputs and gradients")
    ap.add_argument("--only", nargs="*", choices=sorted(WORKLOADS), help="run these workloads only")
    args = ap.parse_args()
    _lib.require_cuda()
    dev = torch.device("cuda:0")
    os.makedirs(args.out, exist_ok=True)
    result = {}
    for name, fn in WORKLOADS.items():
        if args.only and name not in args.only:
            continue
        rec, tensors = fn(dev)
        result[name] = rec
        if args.tensors:
            torch.save({k: v.cpu() for k, v in tensors.items()}, os.path.join(args.out, name + ".pt"))
        torch.cuda.empty_cache()
    with open(os.path.join(args.out, "launch_trace.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps({k: {kk: (len(vv) if isinstance(vv, list) else vv) for kk, vv in v.items()} for k, v in result.items()}))


if __name__ == "__main__":
    main()
