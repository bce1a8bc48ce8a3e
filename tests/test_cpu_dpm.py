"""CPU tests of `DPMSolverMultistepScheduler` (DPM-Solver++): the product's torch `step()` against the fp32 restatement of
diffusers 0.24 (tests/dpm_oracle.py), timestep known answers, the first-order step against closed-form DDIM, convergence
on Gaussian data where the probability-flow ODE has an exact solution, the fused-kernel coefficients (`step_coef`) against
`step()`, the reference pipeline file on the import shim, the pipeline directory round trip and the refused options."""
import itertools
import json
import math
import os

import numpy as np
import pytest
import torch

from audio_diffusion_b200.schedulers import DPMSolverMultistepScheduler
from dpm_oracle import OracleDPM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def configs():
    """Every supported configuration (algorithm, order, solver type, lower_order_final, euler_at_final, spacing)."""
    out = []
    for alg, order, st, lof, eaf, sp in itertools.product(("dpmsolver++", "sde-dpmsolver++"), (1, 2, 3), ("midpoint", "heun"),
                                                          (True, False), (False, True), ("linspace", "leading", "trailing")):
        if alg == "sde-dpmsolver++" and order == 3:
            continue
        out.append(dict(algorithm_type=alg, solver_order=order, solver_type=st, lower_order_final=lof, euler_at_final=eaf,
                        timestep_spacing=sp))
    return out


def _id(kw):
    return "-".join(str(v) for v in kw.values())


@pytest.mark.parametrize("kw", configs(), ids=_id)
def test_step_equals_oracle_bit_for_bit(kw):
    """step() == the 0.24 restatement, bit for bit, over whole runs with seeded model outputs, from step 0 and from a later
    start (which warms up from first order again).  N = 1000 includes the steps diffusers 0.24 itself turns into inf / NaN
    (linspace repeats a timestep there, and trailing ends at t = 0 = sigma_last: h = 0); they must agree too."""
    for n in (10, 20, 25, 50, 1000):
        if kw["timestep_spacing"] == "leading" and n == 1000:
            continue                            # refused: every timestep would be 0 (test_refused_configurations)
        for start in (0, 3):
            s, o = DPMSolverMultistepScheduler(**kw), OracleDPM(**kw)
            s.set_timesteps(n)
            o.set_timesteps(n)
            assert torch.equal(s.timesteps, o.timesteps) and torch.equal(s.sigmas, o.sigmas)
            g = torch.Generator().manual_seed(n + start)
            x = torch.randn(2, 1, 4, 4, generator=g)
            y = x.clone()
            g1, g2 = torch.Generator().manual_seed(1), torch.Generator().manual_seed(1)
            for t in s.timesteps[start:]:
                eps = torch.randn(2, 1, 4, 4, generator=g)
                x = s.step(model_output=eps, timestep=t, sample=x, generator=g1)["prev_sample"]
                y = o.step(eps, t, y, generator=g2)["prev_sample"]
                torch.testing.assert_close(x, y, rtol=0, atol=0, equal_nan=True, msg=f"N={n} start={start} t={int(t)}")
            if n < 1000:
                assert torch.isfinite(x).all()


def test_timestep_known_answers():
    s = DPMSolverMultistepScheduler()
    s.set_timesteps(10)
    assert s.timesteps.tolist() == [999, 899, 799, 699, 599, 500, 400, 300, 200, 100]
    s.set_timesteps(20)
    assert s.timesteps.tolist() == [999] + list(range(949, 548, -50)) + list(range(500, 49, -50))
    s.set_timesteps(25)
    assert s.timesteps.tolist() == [999] + list(range(959, 518, -40)) + list(range(480, 39, -40))
    assert s.num_inference_steps == 25 and s.sigmas.shape == (26,) and s.sigmas.dtype == torch.float32
    ac = s.alphas_cumprod
    assert s.sigmas[-1] == ((1 - ac[0]) / ac[0]) ** 0.5                   # sigma_last = sigma(t = 0), not 0
    assert torch.equal(s.sigmas[:-1], (((1 - ac) / ac) ** 0.5)[s.timesteps])
    lead = DPMSolverMultistepScheduler(timestep_spacing="leading", steps_offset=1)
    lead.set_timesteps(10)
    assert lead.timesteps.tolist() == [90 * k + 1 for k in range(10, 0, -1)]
    trail = DPMSolverMultistepScheduler(timestep_spacing="trailing")
    trail.set_timesteps(10)
    assert trail.timesteps.tolist() == [999, 899, 799, 699, 599, 499, 399, 299, 199, 99]


@pytest.mark.parametrize("n", [10, 20, 50])
def test_first_order_step_is_closed_form_ddim(n):
    """A first-order dpmsolver++ step from t to s is DDIM with eta = 0 and no clipping: sqrt(a_s) x0 + sqrt(1 - a_s) eps
    (fp64 here), with a_s = 1 / (1 + sigma_s^2) at the scheduler's fp32 sigmas."""
    s = DPMSolverMultistepScheduler(solver_order=1)
    s.set_timesteps(n)
    g = torch.Generator().manual_seed(n)
    x = torch.randn(3, 1, 8, 8, generator=g)
    for i, t in enumerate(s.timesteps):
        eps = torch.randn(3, 1, 8, 8, generator=g)
        sig_t, sig_s = s.sigmas[i].double(), s.sigmas[i + 1].double()
        a_t, a_s = 1 / (1 + sig_t ** 2), 1 / (1 + sig_s ** 2)
        x0 = (x.double() - (1 - a_t).sqrt() * eps.double()) / a_t.sqrt()
        want = a_s.sqrt() * x0 + (1 - a_s).sqrt() * eps.double()
        x = s.step(eps, t, x)["prev_sample"]
        scale = max(want.abs().max().item(), 1.0)
        assert (x.double() - want).abs().max().item() <= 2e-6 * scale * max(1.0, float(sig_t)), (i, int(t))


def _gaussian_error(n, s_data=0.5, **kw):
    """Max error at sigma_last of a whole run on data ~ N(0, s^2) with the exact predictor eps*(x, t) = sigma x / (alpha^2 s^2
    + sigma^2), against the ODE's exact solution x_s = x_t sqrt(alpha_s^2 s^2 + sigma_s^2) / sqrt(alpha_t^2 s^2 + sigma_t^2)."""
    sch = DPMSolverMultistepScheduler(**kw)
    sch.set_timesteps(n)
    ac = sch.alphas_cumprod.double()
    t0 = int(sch.timesteps[0])
    v0 = ac[t0] * s_data ** 2 + (1 - ac[t0])
    x = torch.linspace(-3, 3, 13, dtype=torch.float64) * v0.sqrt()
    start = x.clone()
    for t in sch.timesteps:
        a, sg = ac[int(t)].sqrt(), (1 - ac[int(t)]).sqrt()
        x = sch.step(sg * x / (a * a * s_data ** 2 + sg * sg), t, x)["prev_sample"]
    exact = start * (ac[0] * s_data ** 2 + (1 - ac[0])).sqrt() / v0.sqrt()
    return (x - exact).abs().max().item()


# Measured slopes of log(error) against log(N), N = 16, 32, 64, 128 (fit over all four / last pair):
#   order 1: 0.97 / 0.98;  order 2 midpoint: 1.71 / 1.99;  order 2 heun: 1.82 / 2.08;  order 3: 1.33 / 2.64
# The error is dominated by the last step into sigma_last = sigma(0), the largest step in lambda; order 3 only reaches its
# asymptotic rate past N = 32 (its N = 16 error is below its N = 32 one), hence the last-pair bar.
@pytest.mark.parametrize("kw,fit_bar,pair_bar", [
    (dict(solver_order=1), (0.9, 1.1), (0.9, 1.1)),
    (dict(solver_order=2), (1.6, 2.4), (1.9, 2.4)),
    (dict(solver_order=2, solver_type="heun"), (1.7, 2.4), (1.9, 2.4)),
    (dict(solver_order=3), (1.2, 3.5), (2.4, 3.5)),
], ids=["order1", "order2-midpoint", "order2-heun", "order3"])
def test_convergence_on_gaussian_data(kw, fit_bar, pair_bar):
    ns = [16, 32, 64, 128]
    err = [_gaussian_error(n, **kw) for n in ns]
    fit = -np.polyfit(np.log(ns), np.log(err), 1)[0]
    pair = math.log2(err[-2] / err[-1])
    assert fit_bar[0] <= fit <= fit_bar[1] and pair_bar[0] <= pair <= pair_bar[1], (err, fit, pair)


@pytest.mark.parametrize("kw", [k for k in configs() if k["timestep_spacing"] == "linspace"], ids=_id)
def test_step_coef_folds_step(kw):
    """step_coef's five scalars, applied in fp64 (x0 from the sample and eps as the kernel forms it, history planes rotated
    as the kernel rotates them), reproduce step() within fp32 rounding; the two paths advance the same state."""
    for n in (10, 20, 25):
        a, b = DPMSolverMultistepScheduler(**kw), DPMSolverMultistepScheduler(**kw)
        a.set_timesteps(n)
        b.set_timesteps(n)
        g = torch.Generator().manual_seed(n)
        x = torch.randn(2, 1, 8, 8, generator=g)
        y = x.double()
        hist = torch.zeros((2,) + tuple(x.shape), dtype=torch.float64)
        for t in a.timesteps:
            eps = torch.randn(2, 1, 8, 8, generator=g)
            z = torch.randn(2, 1, 8, 8, generator=g)
            c = b.step_coef(t)
            s = c.step
            x0 = (y - s.sqrt_1m_at * eps.double()) * s.inv_sqrt_at
            y = s.c_xt * y + s.c_x0 * x0 + c.c_h1 * hist[0] + c.c_h2 * hist[1] + s.c_z * z.double()
            hist[1], hist[0] = hist[0].clone(), x0
            assert s.do_clip == 0 and s.c_eps == 0.0 and b.needs_noise(t) == (kw["algorithm_type"] == "sde-dpmsolver++")
            x = a.step(eps, t, x, generator=_fixed(z))["prev_sample"]
            assert a.step_index == b.step_index and a.lower_order_nums == b.lower_order_nums
            scale = max(1.0, x.abs().max().item())
            assert (x.double() - y).abs().max().item() <= 1e-5 * scale, (n, int(t))
            y = x.double()                      # both continue from step()'s sample: per-step comparison


class _fixed:
    """A CPU generator stand-in whose draw is `z` (randn_tensor calls torch.randn(shape, generator=...))."""
    device = torch.device("cpu")

    def __init__(self, z):
        self.z = z


@pytest.fixture(autouse=True)
def _randn_from_fixed(monkeypatch):
    real = torch.randn

    def randn(*a, generator=None, **k):
        if isinstance(generator, _fixed):
            return generator.z.clone()
        return real(*a, generator=generator, **k)
    monkeypatch.setattr(torch, "randn", randn)


def test_step_and_step_coef_choose_the_same_orders():
    """The order of every step, with start_step > 0, lower_order_final and euler_at_final, is the one step() uses: the fused
    coefficients of a first-order step carry no history term, of a second-order step no second history term."""
    for kw, n, start in [(dict(solver_order=3), 10, 0), (dict(solver_order=3), 20, 4), (dict(solver_order=2), 10, 5),
                         (dict(solver_order=2, euler_at_final=True, lower_order_final=False), 20, 0)]:
        s = DPMSolverMultistepScheduler(**kw)
        s.set_timesteps(n)
        orders = []
        for t in s.timesteps[start:]:
            c = s.step_coef(t)
            orders.append(1 if c.c_h1 == 0 else 2 if c.c_h2 == 0 else 3)
        o = OracleDPM(**kw)
        o.set_timesteps(n)
        want = []
        for i in range(start, n):
            final = i == n - 1 and (kw.get("euler_at_final", False) or (kw.get("lower_order_final", True) and n < 15))
            second = i == n - 2 and kw.get("lower_order_final", True) and n < 15
            k = i - start
            want.append(1 if kw["solver_order"] == 1 or k < 1 or final else
                        2 if kw["solver_order"] == 2 or k < 2 or second else 3)
        assert orders == want, (kw, n, start)


def _golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "dpm_ref.npz"))


@pytest.mark.parametrize("name,kw,steps", [("dpm2m_20", dict(solver_order=2), 20),
                                           ("sde2m_8", dict(solver_order=2, algorithm_type="sde-dpmsolver++"), 8)])
def test_unchanged_reference_pipeline_runs_on_the_shim(name, kw, steps):
    """The reference pipeline file with the shim's DPMSolverMultistepScheduler (stored uint8 images, its generic
    `scheduler.step(..., generator=)` branch) == the same loop by hand with the oracle scheduler and the oracle U-Net; and
    the engine's own pipeline (its unfused branch: the oracle U-Net has no forward_step) gives the same images."""
    from audio_diffusion_b200.pipeline import AudioDiffusionPipeline as Mirror
    from oracle.unet_oracle import unet_forward
    from test_cpu_dropin import FakeMel, OracleUNet
    unet = OracleUNet()
    g = torch.Generator().manual_seed(42)
    x = torch.randn((2, 1, 16, 16), generator=g)
    o = OracleDPM(**kw)
    o.set_timesteps(steps)
    for t in o.timesteps:
        x = o.step(unet_forward(unet.w, unet.cfg, x, t), t, x, generator=g)["prev_sample"]
    ref = ((x / 2 + 0.5).clamp(0, 1).permute(0, 2, 3, 1).numpy() * 255).round().astype("uint8")[..., 0]
    got = _golden()[name]
    assert np.array_equal(got, ref), np.abs(got.astype(int) - ref.astype(int)).max()
    u8 = Mirror.__dict__["images_to_u8"]
    Mirror.images_to_u8 = staticmethod(lambda v: ((v / 2 + 0.5).clamp(0, 1) * 255).round().to(torch.uint8))
    try:
        pipe = Mirror(vqvae=None, unet=OracleUNet(), mel=FakeMel(), scheduler=DPMSolverMultistepScheduler(**kw))
        pipe.set_progress_bar_config(disable=True)
        r = pipe(batch_size=2, steps=steps, generator=torch.Generator().manual_seed(42))
        assert pipe.get_default_steps() == 1000
        assert np.array_equal(np.stack([np.asarray(im) for im in r.images]), ref)
    finally:
        Mirror.images_to_u8 = u8


def test_directory_round_trip(tmp_path):
    """A pipeline directory whose scheduler/scheduler_config.json names DPMSolverMultistepScheduler loads back with the same
    configuration, through the pipeline's class map and through the shim."""
    import subprocess
    import sys

    from audio_diffusion_b200 import DPMSolverMultistepScheduler as Exported
    from audio_diffusion_b200.mel import Mel
    from audio_diffusion_b200.pipeline import AudioDiffusionPipeline
    from audio_diffusion_b200.unet import UNet2DModel
    assert Exported is DPMSolverMultistepScheduler
    code = (f"import sys; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'audio_diffusion_b200', 'compat')!r}]\n"
            "from diffusers import DPMSolverMultistepScheduler as a\n"
            "from diffusers.schedulers import DPMSolverMultistepScheduler as b\n"
            "from audio_diffusion_b200.schedulers import DPMSolverMultistepScheduler as c\n"
            "assert a is c and b is c\nprint('ok')")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-2000:]
    unet = UNet2DModel(sample_size=(8, 8), in_channels=1, out_channels=1, layers_per_block=1, block_out_channels=(128, 128),
                       down_block_types=("DownBlock2D", "DownBlock2D"), up_block_types=("UpBlock2D", "UpBlock2D"), seed=1)
    sch = DPMSolverMultistepScheduler(solver_order=3, solver_type="heun", timestep_spacing="trailing", euler_at_final=True)
    pipe = AudioDiffusionPipeline(vqvae=None, unet=unet, mel=Mel(x_res=16, y_res=16, hop_length=256), scheduler=sch)
    d = str(tmp_path / "pipe")
    pipe.save_pretrained(d)
    idx = json.load(open(os.path.join(d, "model_index.json")))
    assert idx["scheduler"] == ["diffusers", "DPMSolverMultistepScheduler"]
    cfg = json.load(open(os.path.join(d, "scheduler", "scheduler_config.json")))
    assert cfg["_class_name"] == "DPMSolverMultistepScheduler" and cfg["solver_order"] == 3
    back = AudioDiffusionPipeline.from_pretrained(d)
    assert isinstance(back.scheduler, DPMSolverMultistepScheduler)
    assert dict(back.scheduler.config) == dict(sch.config)
    back.scheduler.set_timesteps(12)
    sch.set_timesteps(12)
    assert torch.equal(back.scheduler.timesteps, sch.timesteps) and torch.equal(back.scheduler.sigmas, sch.sigmas)


@pytest.mark.parametrize("bad,word", [
    (dict(use_karras_sigmas=True), "use_karras_sigmas"), (dict(thresholding=True), "thresholding"),
    (dict(algorithm_type="dpmsolver"), "dpmsolver"), (dict(algorithm_type="sde-dpmsolver"), "sde-dpmsolver"),
    (dict(prediction_type="v_prediction"), "v_prediction"), (dict(beta_schedule="scaled_linear"), "scaled_linear"),
    (dict(solver_order=4), "solver_order"), (dict(algorithm_type="sde-dpmsolver++", solver_order=3), "solver_order"),
    (dict(solver_type="bh2"), "bh2"), (dict(timestep_spacing="karras"), "karras"),
    (dict(lambda_min_clipped=-5.1), "lambda_min_clipped"), (dict(variance_type="learned_range"), "variance_type"),
])
def test_refused_configurations(bad, word):
    with pytest.raises(ValueError, match=word):
        DPMSolverMultistepScheduler(**bad)


def test_refused_step_counts():
    with pytest.raises(ValueError, match="leading"):
        DPMSolverMultistepScheduler(timestep_spacing="leading").set_timesteps(1000)
    with pytest.raises(ValueError, match="num_inference_steps"):
        DPMSolverMultistepScheduler().set_timesteps(1001)
    with pytest.raises(ValueError, match="set_timesteps"):
        DPMSolverMultistepScheduler().step(torch.zeros(1), 999, torch.zeros(1))
