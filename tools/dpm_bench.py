"""Whole-call time of AudioDiffusionPipeline for DDPM-1000, DDIM-50 and DPM-Solver++ 2M with 20 steps, on one GPU.

    python tools/dpm_bench.py --batch 64 --res 256       # eager fused loop
    python tools/dpm_bench.py --batch 1 --res 256        # the CUDA-graph path (batches <= 8)

Each call is `pipe(batch_size=, steps=, return_audio=False)` on the published U-Net layout (seeded synthetic weights) timed
with CUDA events after a warm-up call of the same configuration; the card's name and power limit are read in the same run.
It also times the fused step itself with and without the history traffic of the multistep update (DDIM coefficients vs
DPM-Solver++ order 2 and 3 on the same sample), over `--step-reps` back-to-back steps."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from audio_diffusion_b200.mel import Mel
from audio_diffusion_b200.pipeline import AudioDiffusionPipeline
from audio_diffusion_b200.schedulers import DDIMScheduler, DDPMScheduler, DPMSolverMultistepScheduler
from audio_diffusion_b200.unet import UNet2DModel
from bench import REF_ARCH


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def time_call(pipe, batch, steps, reps):
    gen = torch.Generator(device="cuda").manual_seed(0)
    pipe(batch_size=batch, steps=steps, generator=gen, return_audio=False)           # warm-up: binds, packs, captures
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        pipe(batch_size=batch, steps=steps, generator=gen, return_audio=False)
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return sorted(ms)[len(ms) // 2]


def time_steps(unet, batch, res, reps):
    """Median ms per fused step over `reps` eager steps: DDIM (no history) vs DPM-Solver++ order 2 / 3 (1 / 2 planes)."""
    x = torch.randn(batch, 1, res, res, device="cuda")
    out = {}
    for name, sch in (("ddim", DDIMScheduler()), ("dpm2", DPMSolverMultistepScheduler(solver_order=2)),
                      ("dpm3", DPMSolverMultistepScheduler(solver_order=3))):
        k = getattr(sch, "history_len", 0)
        hist = torch.zeros((k,) + tuple(x.shape), device="cuda") if k else None
        times = []
        for rep in range(3):
            sch.set_timesteps(reps)
            coefs = [(t, sch.step_coef(t)) for t in sch.timesteps]
            y = x.clone()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            for t, c in coefs:
                unet.forward_step(y, t, c, out=y, history=hist)
            b.record()
            torch.cuda.synchronize()
            if rep:                                                  # the first pass is the warm-up
                times.append(a.elapsed_time(b) / reps)
        out[name] = min(times)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ddpm-reps", type=int, default=1)
    ap.add_argument("--step-reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dpm_bench.py needs a CUDA device")
    unet = UNet2DModel(sample_size=(args.res, args.res), seed=0, **REF_ARCH).cuda()
    res = {"gpu": card(), "batch": args.batch, "res": args.res,
           "graph_path": args.batch <= 8 and os.environ.get("B200AD_CUDA_GRAPH", "1") != "0"}
    for name, sch, steps, reps in (("ddpm_1000", DDPMScheduler(), 1000, args.ddpm_reps),
                                   ("ddim_50", DDIMScheduler(), 50, args.reps),
                                   ("dpm2m_20", DPMSolverMultistepScheduler(solver_order=2), 20, args.reps)):
        pipe = AudioDiffusionPipeline(vqvae=None, unet=unet, mel=Mel(x_res=args.res, y_res=args.res), scheduler=sch)
        pipe.set_progress_bar_config(disable=True)
        ms = time_call(pipe, args.batch, steps, reps)
        res[name] = {"call_ms": round(ms, 2), "ms_per_step": round(ms / steps, 3),
                     "images_per_s": round(1e3 * args.batch / ms, 3)}
    with torch.no_grad():
        st = time_steps(unet, args.batch, args.res, args.step_reps)
    plane_mb = args.batch * args.res * args.res * 4 / 1e6
    res["eager_step_ms"] = {k: round(v, 4) for k, v in st.items()}
    res["history_overhead_ms"] = {"order2": round(st["dpm2"] - st["ddim"], 4), "order3": round(st["dpm3"] - st["ddim"], 4)}
    res["history_bytes_mb"] = {"order2": round(2 * plane_mb, 2), "order3": round(4 * plane_mb, 2)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
