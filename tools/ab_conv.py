"""A/B timing of conv_tc_kernel variants inside ONE process (same thermal / power state): the settings of
B200AD_CONV_DBG given on the command line are applied round-robin, `--steps` fused denoise steps each, `--reps` times;
prints mean / min / max ms per step per setting.

    python tools/ab_conv.py 0 8 64 4096 [--steps 5] [--reps 6] [--batch 64] [--res 256]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from bench import REF_ARCH
from audio_diffusion_b200.schedulers import DDPMScheduler
from audio_diffusion_b200.unet import UNet2DModel

ap = argparse.ArgumentParser()
ap.add_argument("cfgs", nargs="+")
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--reps", type=int, default=6)
ap.add_argument("--batch", type=int, default=64)
ap.add_argument("--res", type=int, default=256)
ap.add_argument("--tag", default="")
a = ap.parse_args()
dev = torch.device("cuda:0")
model = UNet2DModel(sample_size=(a.res, a.res), seed=0, **REF_ARCH).to(dev)
sch = DDPMScheduler()
sch.set_timesteps(1000)
g = torch.Generator(device=dev).manual_seed(42)
x = torch.randn(a.batch, 1, a.res, a.res, generator=g, device=dev)
z = torch.randn(a.batch, 1, a.res, a.res, generator=g, device=dev)
ts = sch.timesteps
res = {c: [] for c in a.cfgs}
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
with torch.no_grad():
    for i in range(5):
        model.forward_step(x, ts[i], sch.step_coef(ts[i]), noise=z, out=x)
    for rep in range(a.reps):
        for c in a.cfgs:
            os.environ["B200AD_CONV_DBG"] = c
            model.forward_step(x, ts[7], sch.step_coef(ts[7]), noise=z, out=x)
            torch.cuda.synchronize()
            e0.record()
            for i in range(a.steps):
                model.forward_step(x, ts[10 + i], sch.step_coef(ts[10 + i]), noise=z, out=x)
            e1.record()
            torch.cuda.synchronize()
            res[c].append(e0.elapsed_time(e1) / a.steps)
lines = []
for c, v in res.items():
    lines.append(f"{a.tag} dbg={c:>4s}  mean {sum(v) / len(v):7.3f}  min {min(v):7.3f}  max {max(v):7.3f} ms/step  (batch {a.batch}, {a.res}x{a.res}, {a.reps} x {a.steps} steps)")
print("\n".join(lines))
os.makedirs("gpurun_out", exist_ok=True)
with open("gpurun_out/ab_conv.txt", "a") as f:
    f.write("\n".join(lines) + "\n")
