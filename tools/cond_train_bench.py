"""Times the conditional training iteration (scripts/train_unet.py --encodings, :238-267: add_noise, UNet2DConditionModel
forward + backward with the (B, 1, 100) encodings, clip + AdamW + EMA) on cuda:0 with CUDA events, at the published model's
64x64 latent (batch 16) and at 256x256 (batch 2).  Prints the GPU name and power limit, images/s, the per-kind backward
time (B200AD_BWD_PROFILE=1, one extra profiled step in a child process) and the achieved TFLOP/s of the attention backward,
counted from shapes as 10 * seq^2 * head_dim * heads per transformer block.  At 64x64 only it also times the baseline the
reference runs (diffusers + accelerate): torch autograd over oracle/unet_cond_oracle.py under bf16 autocast with
torch.optim.AdamW; at 256x256 its explicit softmax would need ~137 GB for one attention matrix.
usage: python tools/cond_train_bench.py [--steps K] [--no-baseline]"""
import argparse, json, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

ARCH = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256, 512, 512),
            down_block_types=("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",),
            up_block_types=("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3, cross_attention_dim=100)
SHAPES = {64: 16, 256: 2}    # resolution -> batch


def attn_bwd_flops(res: int, batch: int) -> float:
    """10 * seq^2 * C per transformer block (C = heads * head_dim), summed over the architecture's blocks."""
    boc, lpb = ARCH["block_out_channels"], ARCH["layers_per_block"]
    tot = 0.0
    for i, typ in enumerate(ARCH["down_block_types"]):
        if typ.startswith("CrossAttn"):
            tot += lpb * 10.0 * (res >> i) ** 4 * boc[i]
    tot += 10.0 * (res >> (len(boc) - 1)) ** 4 * boc[-1]                # mid block
    for i, typ in enumerate(ARCH["up_block_types"]):
        lvl = len(boc) - 1 - i
        if typ.startswith("CrossAttn"):
            tot += (lpb + 1) * 10.0 * (res >> lvl) ** 4 * boc[lvl]
    return tot * batch


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "unknown"
    return name, out


def engine(res: int, batch: int, steps: int, warmup: int = 2):
    from audio_diffusion_b200.schedulers import DDPMScheduler
    from audio_diffusion_b200.training import EMAModel, FusedAdamW, train_step
    from audio_diffusion_b200.unet_cond import UNet2DConditionModel
    dev = torch.device("cuda:0")
    model = UNet2DConditionModel(sample_size=(res, res), seed=0, **ARCH).to(dev).train()
    opt = FusedAdamW(model.parameters(), lr=1e-4, betas=(0.95, 0.999), weight_decay=1e-6, eps=1e-8, max_grad_norm=1.0)
    ema = EMAModel(model.parameters(), inv_gamma=1.0, power=0.75, max_value=0.9999)
    opt.attach_ema(ema)
    sch = DDPMScheduler()
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.rand(batch, 1, res, res, device=dev, generator=g) * 2 - 1
    enc = torch.randn(batch, 1, 100, device=dev, generator=g)
    losses = []
    step = lambda: losses.append(train_step(model, opt, sch, x, ema=ema, generator=g, encoder_hidden_states=enc))
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        step()
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / steps
    return {"ms_per_train_step": ms, "images_per_s": batch / ms * 1e3, "loss": [float(l) for l in losses],
            "backward_launches": model.last_backward_launch_count, "max_mem_GB": torch.cuda.max_memory_allocated() / 2**30}


def baseline(res: int, batch: int, steps: int, warmup: int = 2):
    """torch autograd over the oracle under bf16 autocast, stock AdamW + clip: what diffusers + accelerate run."""
    from oracle.schedulers_oracle import OracleDDPM
    from oracle.unet_cond_oracle import CondUNetConfig, init_weights, unet_cond_forward
    dev = torch.device("cuda:0")
    cfg = CondUNetConfig(sample_size=(res, res))
    w = {k: v.to(dev).requires_grad_(True) for k, v in init_weights(cfg, seed=0).items()}
    opt = torch.optim.AdamW(w.values(), lr=1e-4, betas=(0.95, 0.999), weight_decay=1e-6, eps=1e-8)
    sch = OracleDDPM()
    sch.alphas_cumprod = sch.alphas_cumprod.to(dev)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.rand(batch, 1, res, res, device=dev, generator=g) * 2 - 1
    enc = torch.randn(batch, 1, 100, device=dev, generator=g)

    def step():
        noise = torch.randn(x.shape, device=dev, generator=g)
        with torch.device(dev):     # the oracle creates its timestep tensors with default placement
            _step(noise)

    def _step(noise):
        t = torch.randint(0, 1000, (batch,), device=dev, generator=g)
        noisy = sch.add_noise(x, noise, t)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            pred = unet_cond_forward(w, cfg, noisy, t, enc)
        loss = torch.nn.functional.mse_loss(pred.float(), noise)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(w.values(), 1.0)
        opt.step()
        opt.zero_grad(set_to_none=True)
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        step()
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / steps
    return {"ms_per_train_step": ms, "images_per_s": batch / ms * 1e3, "max_mem_GB": torch.cuda.max_memory_allocated() / 2**30}


def profile(res: int, batch: int):
    """One profiled step in a child process (the library reads B200AD_BWD_PROFILE once)."""
    env = dict(os.environ, B200AD_BWD_PROFILE="1")
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--profile-child", str(res)], env=env,
                       capture_output=True, text=True, timeout=1200)
    lines = [l for l in r.stderr.splitlines() if l.startswith('{"backward_profile_ms"')]
    if not lines:
        return None
    return json.loads(lines[-1])["backward_profile_ms"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--no-baseline", action="store_true")
    ap.add_argument("--profile-child", type=int, default=0)
    args = ap.parse_args()
    if args.profile_child:
        engine(args.profile_child, SHAPES[args.profile_child], steps=1, warmup=2)
        return
    name, plimit = gpu_info()
    print(json.dumps({"gpu": name, "power_limit": plimit}), flush=True)
    for res, batch in SHAPES.items():
        torch.cuda.reset_peak_memory_stats()
        r = {"res": res, "batch": batch, "engine": engine(res, batch, args.steps)}
        torch.cuda.empty_cache()
        prof = profile(res, batch)
        if prof:
            r["backward_profile_ms"] = prof
            ms = sum(v for k, v in prof.items() if re.match(r"mha_bwd x\d+", k))
            fl = attn_bwd_flops(res, batch)
            r["attention_bwd"] = {"ms": ms, "gflop": fl / 1e9, "tflops": fl / (ms * 1e-3) / 1e12 if ms else None}
        if res == 64 and not args.no_baseline:
            torch.cuda.reset_peak_memory_stats()
            bb = batch          # the eager baseline keeps every attention matrix: halve the batch until it fits
            while bb >= 1:
                try:
                    r["baseline_bf16_autocast"] = dict(baseline(res, bb, args.steps), batch=bb)
                    break
                except torch.cuda.OutOfMemoryError:
                    r.setdefault("baseline_out_of_memory_at_batch", []).append(bb)
                    torch.cuda.empty_cache()
                    bb //= 2
            torch.cuda.empty_cache()
            bl = r.get("baseline_bf16_autocast")
            if bl:
                r["speedup_vs_baseline_images_per_s"] = r["engine"]["images_per_s"] / bl["images_per_s"]
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
