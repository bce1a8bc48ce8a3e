"""Time and peak memory of one training iteration with gradient checkpointing off and on, on cuda:0.

Workloads (all 256x256):
  * UNet2DModel as scripts/train_unet.py builds it, batch 16, and the largest batch that fits each way: starting from
    the largest batch whose planned training memory (b200ad_unet_training_bytes) fits in the free device memory, one
    sample less until an iteration runs (the plan leaves out the allocator's and the model's own tensors);
  * UNet2DConditionModel (train_unet.py --encodings), batch 16, with S = 1 and S = 77 encoder tokens;
  * AutoencoderKL in the ldm config, batch 8 and 16 (encode, sample, decode, L1 + KL, backward).
An iteration is forward + loss + backward (no optimizer step).  Each workload and mode gets a fresh model, so no buffer of
another mode is still held; every shape is run twice before it is timed with CUDA events.  Peak memory is
torch.cuda.max_memory_allocated over the timed iterations (parameters, packed weights and gradients included).  Prints the
GPU name, power limit and SM clock limit, one line per workload and mode, and one JSON line.
usage: python tools/checkpoint_bench.py [--steps K] [--only unet,cond,vae]"""
import argparse, gc, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

PUBLISHED = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 128, 256, 256, 512, 512),
                 down_block_types=("DownBlock2D",) * 4 + ("AttnDownBlock2D", "DownBlock2D"),
                 up_block_types=("UpBlock2D", "AttnUpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D"))
COND = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256, 512, 512),
            down_block_types=("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",),
            up_block_types=("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3, cross_attention_dim=100)
LDM = dict(in_channels=1, out_channels=1, latent_channels=1, layers_per_block=2, block_out_channels=(128, 256, 512, 512),
           down_block_types=("DownEncoderBlock2D",) * 4, up_block_types=("UpDecoderBlock2D",) * 4)
RES = 256


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "unknown"
    return torch.cuda.get_device_name(0), out


def make(kind, ckpt):
    from audio_diffusion_b200.unet import UNet2DModel
    from audio_diffusion_b200.unet_cond import UNet2DConditionModel
    from audio_diffusion_b200.vae import AutoencoderKL
    if kind == "unet":
        m = UNet2DModel(sample_size=(RES, RES), seed=0, **PUBLISHED)
    elif kind == "cond":
        m = UNet2DConditionModel(sample_size=(RES, RES), seed=0, **COND)
    else:
        m = AutoencoderKL(seed=0, max_batch=64, **LDM)
    m = m.to("cuda:0").train()
    if ckpt:
        m.enable_gradient_checkpointing()
    return m


def iteration_fn(kind, m, n, s):
    from audio_diffusion_b200.training import vae_loss
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(n)
    x = torch.randn(n, 1, RES, RES, device=dev, generator=g)
    tgt = torch.randn_like(x)
    t = torch.randint(0, 1000, (n,), device=dev, generator=g)
    enc = torch.randn(n, s, 100, device=dev, generator=g) if kind == "cond" else None
    noise = torch.randn(n, 1, RES // 8, RES // 8, device=dev, generator=g)

    def fn():
        for p in m.parameters():
            p.grad = None
        if kind == "vae":
            post = m.encode(x.clamp(-1, 1)).latent_dist
            loss = vae_loss(x, m.decode(post.mean + post.std * noise).sample, post)[0]
        else:
            out = m(x, t)["sample"] if enc is None else m(x, t, enc)["sample"]
            loss = torch.nn.functional.mse_loss(out, tgt)
        loss.backward()
    return fn


def measure(kind, ckpt, n, s, steps):
    """(ms per iteration, peak GiB), or None if the iteration does not fit in device memory."""
    m = make(kind, ckpt)
    fn = None
    try:
        fn = iteration_fn(kind, m, n, s)
        fn(); fn()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            fn()
        b.record()
        torch.cuda.synchronize()
        res = (a.elapsed_time(b) / steps, torch.cuda.max_memory_allocated() / 2**30)
    except torch.cuda.OutOfMemoryError:
        res = None
    fn = None
    del m
    gc.collect()
    torch.cuda.empty_cache()
    return res


def planned_batch(ckpt):
    """The largest U-Net batch whose planned training memory fits in the free memory, less the model's own tensors."""
    from audio_diffusion_b200 import _lib
    m = make("unet", ckpt)
    L = _lib.lib()
    fixed = sum(p.numel() for p in m.parameters()) * 4 * 3 + (1 << 30)   # parameters, gradients, packed weights + margin
    free = torch.cuda.mem_get_info()[0] - fixed
    n = 16
    while L.b200ad_unet_training_bytes(m._h, n + 1, RES, RES, 1) <= free:
        n += 1
    del m
    gc.collect()
    torch.cuda.empty_cache()
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--only", default="unet,cond,vae")
    a = ap.parse_args()
    name, info = gpu_info()
    print(f"GPU {name}, power limit / max SM clock: {info}", flush=True)
    only = a.only.split(",")
    work = []
    planned = {}
    if "unet" in only:
        planned = {ckpt: planned_batch(ckpt) for ckpt in (False, True)}
        work += [("unet", 16, 1), ("unet", None, 1)]
    if "cond" in only:
        work += [("cond", 16, 1), ("cond", 16, 77)]
    if "vae" in only:
        work += [("vae", 8, 1), ("vae", 16, 1)]
    res = {}
    for kind, n, s in dict.fromkeys(work):
        row = {}
        for ckpt in (False, True):
            if n is None:     # the largest batch of this mode only
                m = planned[ckpt]
                while (r := measure(kind, ckpt, m, s, a.steps)) is None and m > 16:
                    m -= 1
                row["on" if ckpt else "off"] = None if r is None else {"batch": m, "ms": round(r[0], 1),
                                                                      "peak_gib": round(r[1], 2)}
                continue
            r = measure(kind, ckpt, n, s, a.steps)
            row["on" if ckpt else "off"] = None if r is None else {"ms": round(r[0], 1), "peak_gib": round(r[1], 2)}
        key = f"{kind} {RES}x{RES} b{'largest' if n is None else n}" + (f" S={s}" if kind == "cond" else "")
        res[key] = row
        fmt = lambda r: ("does not fit" if r is None else
                         (f"b{r['batch']} " if "batch" in r else "") + f"{r['ms']:9.1f} ms  {r['peak_gib']:6.2f} GiB")
        ratio = ""
        if row["off"] and row["on"]:
            ratio = f"  time x{row['on']['ms'] / row['off']['ms']:.3f}, memory x{row['on']['peak_gib'] / row['off']['peak_gib']:.3f}"
        print(f"{key:28s} off: {fmt(row['off'])} | on: {fmt(row['on'])}{ratio}", flush=True)
    print(json.dumps({"gpu": name, "limits": info, "results": res}))


if __name__ == "__main__":
    main()
