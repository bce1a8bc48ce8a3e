"""Generates tests/golden/dpm_ref.npz by running the reference's OWN pipeline file (read unchanged from a checkout of
teticio/audio-diffusion) on the import shim with `DPMSolverMultistepScheduler`.  Run from the repo root:
    python tests/golden/make_golden_dpm.py <reference checkout>

The pipeline sends any scheduler other than DDIM through its generic branch (pipeline_audio_diffusion.py:174-179:
`scheduler.step(model_output=, timestep=, sample=, generator=)["prev_sample"]`).  Here it drives the fp32 CPU oracle U-Net
of tests/test_cpu_dropin.py with the shim's (the product's) scheduler, for 20 steps of DPM-Solver++ 2M and 8 steps of
SDE-DPM-Solver++ 2M (its noise drawn from the pipeline's generator inside `step`).  tests/test_cpu_dpm.py recomputes the
images with the oracle scheduler (tests/dpm_oracle.py) and the same U-Net.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF = sys.argv[1] if len(sys.argv) > 1 else sys.exit("usage: make_golden_dpm.py <reference checkout>")
sys.path[:0] = [ROOT, os.path.join(ROOT, "audio_diffusion_b200", "compat"), REF, os.path.join(ROOT, "tests")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

CASES = {"dpm2m_20": (dict(solver_order=2), 20), "sde2m_8": (dict(solver_order=2, algorithm_type="sde-dpmsolver++"), 8)}


def main():
    from audiodiffusion.pipeline_audio_diffusion import AudioDiffusionPipeline as RefPipe
    from diffusers import DPMSolverMultistepScheduler
    from test_cpu_dropin import FakeMel, OracleUNet
    out = {}
    for name, (kw, steps) in CASES.items():
        pipe = RefPipe(vqvae=None, unet=OracleUNet(), mel=FakeMel(), scheduler=DPMSolverMultistepScheduler(**kw))
        pipe.set_progress_bar_config(disable=True)
        r = pipe(batch_size=2, steps=steps, generator=torch.Generator().manual_seed(42))
        assert len(r.images) == 2 and r.audios.shape == (2, 1, 15 * 512)
        out[name] = np.stack([np.asarray(im) for im in r.images])
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "dpm_ref.npz"), **out)
    print("dpm_ref.npz", {k: (v.shape, float(v.mean())) for k, v in out.items()})


if __name__ == "__main__":
    main()
