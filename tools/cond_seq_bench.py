"""Times UNet2DConditionModel as scripts/train_unet.py:140-159 builds it against encodings of S tokens, S in {1, 8, 77,
256}, on cuda:0 with CUDA events: one fused denoising step (`forward_step`, eval) and one training iteration (forward with
the encoding, MSE, backward), at the published 64x64 latent (batch 64) and at 256x256 (batch 16; the training iteration
also at batch 2, since batch 16 keeps more activations than 80 GB hold).  S = 1 is the per-sample
vector path; S > 1 runs the K / V projections, the cross-attention kernels and the two extra 1x1 projections per
transformer block.  Every shape is warmed up before it is timed.  Prints the GPU name and power limit, the times and each
time's ratio to S = 1, and one JSON line.  A shape that does not fit in device memory is reported as such.
usage: python tools/cond_seq_bench.py [--steps K] [--tokens 1,8,77,256]"""
import argparse, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

ARCH = dict(in_channels=1, out_channels=1, layers_per_block=2, block_out_channels=(128, 256, 512, 512),
            down_block_types=("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",),
            up_block_types=("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3, cross_attention_dim=100)
SHAPES = ((64, 64, (64,)), (256, 16, (16, 2)))    # (resolution, forward_step batch, training batches)


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "unknown"
    return name, out


def timed(fn, steps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(steps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--tokens", default="1,8,77,256")
    a = ap.parse_args()
    from audio_diffusion_b200.schedulers import DDPMScheduler
    from audio_diffusion_b200.unet_cond import UNet2DConditionModel
    dev = torch.device("cuda:0")
    name, plim = gpu_info()
    print(f"GPU {name}, power limit {plim}")
    tokens = [int(v) for v in a.tokens.split(",")]
    sch = DDPMScheduler()
    sch.set_timesteps(50)
    t_step = sch.timesteps[10]
    coef = sch.step_coef(t_step)
    res = {}
    for size, fbatch, tbatches in SHAPES:
        model = UNet2DConditionModel(sample_size=size, seed=0, **ARCH).to(dev)
        g = torch.Generator(device=dev).manual_seed(0)
        for mode, batch in [("forward_step", fbatch)] + [("train_iter", b) for b in tbatches]:
            x = torch.randn(batch, 1, size, size, device=dev, generator=g)
            z = torch.randn_like(x)
            tgt = torch.randn_like(x)
            tt = torch.randint(0, 1000, (batch,), device=dev, generator=g)
            for s in tokens:
                enc = torch.randn(batch, s, 100, device=dev, generator=g)
                if mode == "forward_step":
                    model.eval()

                    def fn():
                        with torch.no_grad():
                            model.forward_step(x, t_step, coef, encoder_hidden_states=enc, noise=z)
                else:
                    model.train()

                    def fn():
                        for p in model.parameters():
                            p.grad = None
                        torch.nn.functional.mse_loss(model(x, tt, enc)["sample"], tgt).backward()
                key = f"{mode} {size}x{size} b{batch} S={s}"
                try:
                    fn(); fn()                                    # warm-up: binding, module loading
                    ms = timed(fn, a.steps)
                except torch.cuda.OutOfMemoryError:
                    print(f"{key}: does not fit in device memory")
                    res[key] = None
                    for p in model.parameters():
                        p.grad = None
                    torch.cuda.empty_cache()
                    continue
                res[key] = ms
                base = res.get(f"{mode} {size}x{size} b{batch} S=1")
                ratio = f"  x{ms / base:.3f} of S=1" if base else ""
                print(f"{key:36s} {ms:9.2f} ms{ratio}", flush=True)
            del x, z, tgt
        del model
        torch.cuda.empty_cache()
    print(json.dumps({"gpu": name, "power_limit": plim, "ms": res}))


if __name__ == "__main__":
    main()
