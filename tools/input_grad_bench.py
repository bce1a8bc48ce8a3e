"""Cost of the gradient with respect to the input, on cuda:0.

Modes, each on a fresh model (so no buffer of another mode is still held), run twice before it is timed with CUDA events:
  (a) forward + backward with parameter gradients (train(): a training iteration without the optimizer step);
  (b) (a) with the input also requiring grad, so the backward writes its gradient too;
  (c) eval() with every parameter frozen, the input requiring grad: forward + data-gradient-only backward.
Workloads:
  * UNet2DModel as scripts/train_unet.py builds it, 256x256, batch 16 (the gradient w.r.t. the sample);
  * UNet2DConditionModel (train_unet.py --encodings), 64x64, batch 64, S = 1;
  * AutoencoderKL in the ldm config, 256x256, batch 8: the encoder's image gradient (loss on the moments), and the
    decoder's latent gradient (loss on the image; the decoder always returns dL/dz, so (b) is (a) there).
Reports per workload and mode: ms per iteration, last_backward_launch_count and torch.cuda.max_memory_allocated over the
timed iterations (parameters, packed weights and gradients included), with the GPU name and power limit; one JSON line.
usage: python tools/input_grad_bench.py [--steps K] [--only unet,cond,vae_enc,vae_dec]"""
import argparse, gc, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import torch.nn.functional as F

PUBLISHED = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 128, 256, 256, 512, 512),
                 down_block_types=("DownBlock2D",) * 4 + ("AttnDownBlock2D", "DownBlock2D"),
                 up_block_types=("UpBlock2D", "AttnUpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D"))
COND = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256, 512, 512),
            down_block_types=("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",),
            up_block_types=("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3, cross_attention_dim=100)
LDM = dict(in_channels=1, out_channels=1, latent_channels=1, layers_per_block=2, block_out_channels=(128, 256, 512, 512),
           down_block_types=("DownEncoderBlock2D",) * 4, up_block_types=("UpDecoderBlock2D",) * 4)
WORKLOADS = {"unet": (16, 256), "cond": (64, 64), "vae_enc": (8, 256), "vae_dec": (8, 256)}


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
    return torch.cuda.get_device_name(0), out


def make(kind, mode, dev):
    if kind == "unet":
        from audio_diffusion_b200.unet import UNet2DModel
        m = UNet2DModel(sample_size=(256, 256), seed=0, **PUBLISHED)
    elif kind == "cond":
        from audio_diffusion_b200.unet_cond import UNet2DConditionModel
        m = UNet2DConditionModel(sample_size=(64, 64), seed=0, **COND)
    else:
        from audio_diffusion_b200.vae import AutoencoderKL
        m = AutoencoderKL(max_batch=8, seed=0, **LDM)
    m = m.to(dev)
    if mode == "c":
        m.eval()
        m.requires_grad_(False)
    else:
        m.train()
    return m


def step_fn(kind, model, mode, dev):
    n, res = WORKLOADS[kind]
    g = torch.Generator().manual_seed(0)
    want_x = mode in ("b", "c")
    if kind in ("unet", "cond"):
        x = torch.randn(n, 1, res, res, generator=g).to(dev)
        tgt = torch.randn(n, 1, res, res, generator=g).to(dev)
        t = torch.randint(0, 1000, (n,), generator=g).to(dev)
        enc = torch.randn(n, 1, 100, generator=g).to(dev) if kind == "cond" else None

        def step():
            for p in model.parameters():
                p.grad = None
            xl = x.detach().requires_grad_(want_x)
            out = model(xl, t)["sample"] if enc is None else model(xl, t, enc)["sample"]
            F.mse_loss(out, tgt).backward()
        return step
    if kind == "vae_enc":
        x = torch.randn(n, 1, res, res, generator=g).clamp(-1, 1).to(dev)
        gm = torch.randn(n, 2, res // 8, res // 8, generator=g).to(dev)

        def step():
            for p in model.parameters():
                p.grad = None
            xl = x.detach().requires_grad_(want_x)
            model.encode(xl).latent_dist.parameters.backward(gm)
        return step
    z = torch.randn(n, 1, res // 8, res // 8, generator=g).to(dev)
    gimg = torch.randn(n, 1, res, res, generator=g).to(dev)

    def step():
        for p in model.parameters():
            p.grad = None
        zl = z.detach().requires_grad_(True)
        model.decode(zl).sample.backward(gimg)
    return step


def measure(kind, mode, steps, dev):
    model = make(kind, mode, dev)
    step = step_fn(kind, model, mode, dev)
    for _ in range(2):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        step()
    e.record()
    e.synchronize()
    r = dict(ms=s.elapsed_time(e) / steps, launches=model.last_backward_launch_count,
             peak_gib=torch.cuda.max_memory_allocated() / 2**30)
    del model, step
    gc.collect()
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--only", default=",".join(WORKLOADS))
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    name, limits = gpu_info()
    print(f"GPU: {name}; power limit, max SM clock: {limits}")
    res = {"gpu": name, "power_limit_and_max_sm_clock": limits, "steps": a.steps}
    for kind in a.only.split(","):
        modes = ("a", "c") if kind == "vae_dec" else ("a", "b", "c")
        rows = {m: measure(kind, m, a.steps, dev) for m in modes}
        res[kind] = rows
        n, r = WORKLOADS[kind]
        for m, v in rows.items():
            print(f"{kind:8s} {r}x{r} batch {n:3d} ({m}): {v['ms']:9.2f} ms/iter  launches {v['launches']:5d}  "
                  f"peak {v['peak_gib']:6.2f} GiB")
        if "b" in rows:
            print(f"{kind:8s} (b) / (a) = {rows['b']['ms'] / rows['a']['ms']:.4f}")
        print(f"{kind:8s} (c) / (a) = {rows['c']['ms'] / rows['a']['ms']:.4f} time, "
              f"{rows['c']['peak_gib'] / rows['a']['peak_gib']:.4f} memory")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
