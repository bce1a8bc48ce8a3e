"""Autoencoder training throughput (scripts/train_vae.py's iteration: encode, sample, decode, L1 + 1e-6 KL, backward,
Adam(lr 4.5e-6, betas (0.5, 0.9))) at 256x256, batch 1, 4 and 8, on the engine and as eager PyTorch on the same GPU
(torch autograd over oracle/vae_oracle.py under bf16 autocast, torch.optim.Adam).  Prints the GPU name and power limit,
images/s, the backward launches per step and, per batch, the forward's FLOP rate (894 GFLOP per image: encode 272 +
decode 622, SURVEY §8a; the backward's FLOPs are not counted).

usage (on a GPU machine): python tools/vae_train_bench.py [--steps K] [--no-baseline]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FWD_GFLOP = 894.0


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "unknown"
    return name, out


def _timed(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps


def engine(batch: int, steps: int, warmup: int = 2):
    from audio_diffusion_b200.training import FusedAdamW
    from audio_diffusion_b200.vae import AutoencoderKL
    from oracle.vae_oracle import VAEConfig, init_weights
    cfg = VAEConfig()
    n = len(cfg.block_out_channels)
    model = AutoencoderKL(in_channels=1, out_channels=1, down_block_types=("DownEncoderBlock2D",) * n,
                          up_block_types=("UpDecoderBlock2D",) * n, block_out_channels=cfg.block_out_channels,
                          layers_per_block=2, latent_channels=1, max_batch=batch)
    model.load_state_dict(init_weights(cfg, seed=0))
    model = model.cuda().train()
    opt = FusedAdamW(model.parameters(), lr=4.5e-6, betas=(0.5, 0.9), weight_decay=0.0)
    x = torch.rand(batch, 1, 256, 256, device="cuda") * 2 - 1
    launches = []

    def step():
        post = model.encode(x).latent_dist
        y = model.decode(post.sample()).sample
        loss = torch.abs(x - y).sum() / batch + 1e-6 * post.kl().sum() / batch
        loss.backward()
        launches.append(model.last_backward_launch_count)
        opt.step()
        opt.zero_grad(set_to_none=True)

    s = _timed(step, steps, warmup)
    return dict(batch=batch, ms_per_step=s * 1e3, images_per_s=batch / s,
                fwd_tflops=FWD_GFLOP * batch / s / 1e3, backward_launches=launches[-1])


def baseline(batch: int, steps: int, warmup: int = 2):
    """torch autograd over the oracle under bf16 autocast, torch.optim.Adam: the eager iteration."""
    from oracle.vae_oracle import VAEConfig, decode, encode_moments, init_weights
    cfg = VAEConfig()
    w = {k: v.cuda().requires_grad_(True) for k, v in init_weights(cfg, seed=0).items()}
    opt = torch.optim.Adam(list(w.values()), lr=4.5e-6, betas=(0.5, 0.9))
    x = torch.rand(batch, 1, 256, 256, device="cuda") * 2 - 1

    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            m = encode_moments(w, cfg, x).float()
            mean, logvar = torch.chunk(m, 2, dim=1)
            logvar = torch.clamp(logvar, -30.0, 20.0)
            z = mean + torch.exp(0.5 * logvar) * torch.randn_like(mean)
            y = decode(w, cfg, z).float()
        kl = 0.5 * torch.sum(mean ** 2 + torch.exp(logvar) - 1.0 - logvar)
        loss = torch.abs(x - y).sum() / batch + 1e-6 * kl / batch
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)

    s = _timed(step, steps, warmup)
    return dict(batch=batch, ms_per_step=s * 1e3, images_per_s=batch / s)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--no-baseline", action="store_true")
    args = ap.parse_args()
    name, plimit = gpu_info()
    print(json.dumps({"gpu": name, "power_limit": plimit}), flush=True)
    for b in (1, 4, 8):
        r = {"engine": engine(b, args.steps)}
        torch.cuda.empty_cache()
        if not args.no_baseline:
            r["eager_bf16_autocast"] = baseline(b, args.steps)
            r["speedup"] = r["eager_bf16_autocast"]["ms_per_step"] / r["engine"]["ms_per_step"]
            torch.cuda.empty_cache()
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
