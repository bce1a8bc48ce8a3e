"""How the per-block fp64 checks compare: every block of the engine's forward or backward against the fp64 reference of
that one block (oracle/block_grads.py) on the engine's own inputs, one table row per block, the bars against the bf16
floors measured from the oracle's activations, and the fp64 time and peak device memory of the comparison.  The drivers
run one case of tests/test_gpu_block_backward*.py, tests/test_gpu_block_forward.py, tests/test_gpu_latent_unet.py and
tests/test_gpu_cond_seq.py each, with the architectures, builders and seeded inputs of tests/cases.py; check_fused_step
is the fused scheduler update's fp64 check."""
import time

import torch

import cases
from oracle import block_grads as bg


def bar_in_range(floor, bar, k, digits, least=0.0):
    """A bar stated from a floor printed to `digits` digits lies in (floor, max(k x floor, least)]."""
    return floor < bar <= max(k * round(floor, digits), least) + 1e-9


def power_limit():
    import subprocess
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # the card name is printed by report_time in any case
        return f"power limit not read: {e}"


def report_time(name, t0):
    """Prints the fp64 time since t0 and the peak device memory since the last reset."""
    torch.cuda.synchronize()
    print(f"\n{name}: fp64 time {time.perf_counter() - t0:.1f} s, peak device memory "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB on {torch.cuda.get_device_properties(0).name}")


# ---------------------------------------------------------------------------------------------------- backward
def run_backward_checks(model, blocks, model_in, g_out, w, cfg, bars, prefix="", temb=None, enc=None, g_in=None, t=None):
    """Compares every block; prints one table row per block; returns the blocks over their bars.  A U-Net (temb given)
    also needs its timesteps t: after the walk, the engine's time_embedding.* gradients against temb_backward of the sum
    of every resnet's fp64 temb_act gradient, as the "temb" row."""
    assert (temb is None) == (t is None), "a U-Net's checks need both temb and t"
    named = dict(model.named_parameters())
    skip_taps = {b.skip for b in blocks if b.skip}
    fails, worst_kind = [], {}
    g_temb = None
    print(f"\n{'block':44s} {'kind':12s} {'act L2':>7s} {'max':>7s} {'row':>7s} | {'par L2':>7s} {'max':>7s} {'row':>7s}")

    def row(name, kind, rows, skipped):
        wa, wp = bg.worst(rows, True), bg.worst(rows, False)
        ba, bp = bars[kind]
        over = [r for r in rows if any(e > b for e, b in zip(r[2:], ba if r[1] else bp))]
        print(f"{name:44s} {kind:12s} {wa[0]:7.4f} {wa[1]:7.4f} {wa[2]:7.4f} | {wp[0]:7.4f} {wp[1]:7.4f} "
              f"{wp[2]:7.4f}{'  OVER' if over else ''}{'  (zero ref: ' + ', '.join(skipped) + ')' if skipped else ''}")
        for r in over:
            print(f"    {r[0]}: {r[2]:.4f} {r[3]:.4f} {r[4]:.4f}")
        if over:
            fails.append((name, [(r[0], round(r[2], 4), round(r[3], 4), round(r[4], 4)) for r in over]))
        pa, pp = worst_kind.get(kind, ((0.0,) * 3, (0.0,) * 3))
        worst_kind[kind] = (tuple(map(max, pa, wa)), tuple(map(max, pp, wp)))

    for blk in reversed(blocks):
        xs = [model_in if blk.inp is None else model.debug_tensor(blk.inp)]
        if blk.skip:
            xs.append(model.debug_tensor(blk.skip))
        gout = g_out if blk.out is None else model.debug_grad(blk.out)
        gi, gp, gt = bg.block_backward(blk, w, xs, gout, cfg, temb, enc, temb_grad=True)
        if gt is not None:
            g_temb = gt if g_temb is None else g_temb + gt
        acts = {}
        if blk.inp is not None:
            ref = gi[0]
            if blk.inp in skip_taps:            # the skip connection's share, checked at the block that consumes it
                ref = ref + model.debug_grad(blk.inp, skip=True).double()
            acts[f"G({blk.inp})"] = (model.debug_grad(blk.inp), ref)
        elif g_in is not None:
            acts["g_z"] = (g_in, gi[0])
        if blk.skip:
            acts[f"skip G({blk.skip})"] = (model.debug_grad(blk.skip, skip=True), gi[1])
        rows, skipped = bg.compare_block(acts, {k: (named[k].grad, gp[k]) for k in gp})
        row(blk.name or "conv_out", prefix + blk.kind, rows, skipped)
    if t is not None:    # the timestep MLP, from the resnets' temb_act gradients (engine: gproj -> time_emb_proj^T -> MLP)
        ref = bg.temb_backward(w, cfg, t, g_temb)
        rows, skipped = bg.compare_block({}, {k: (named[k].grad, ref[k]) for k in ref})
        row("time_embedding", prefix + "temb", rows, skipped)
    print("worst per kind (activation a, b, c | parameter a, b, c) against the bars:")
    for kind, (a, p) in worst_kind.items():
        print(f"  {kind:20s} {a[0]:.4f} {a[1]:.4f} {a[2]:.4f} | {p[0]:.4f} {p[1]:.4f} {p[2]:.4f}   bars {bars[kind]}")
    return fails


def report_backward_floors(floors, bars, kinds=None):
    """Prints the floors as a bar table (three times the floor, no lower than 0.5 %); returns the bars (of `kinds`, None:
    all) outside (floor, max(3.3 x floor, 0.5 %)]."""
    print("floors as bars (3 x floor, >= 0.005):")
    bad = []
    for kind, (a, p) in floors.items():
        fl = tuple(round(f, 4) for f in a + p)
        sug = tuple(round(max(3 * f, 0.005), 4) for f in fl)
        print(f'    "{kind}": ({sug[:3]}, {sug[3:]}),   # floor {fl[:3]} | {fl[3:]}')
        if kinds is None or kind in kinds:
            bad += [(kind, round(f, 4), b) for f, b in zip(a + p, bars[kind][0] + bars[kind][1])
                    if not bar_in_range(f, b, 3.3, 4, 5e-3)]
    return bad


def unet_backward_case(cuda, arch, size, n, seed, t, bars, s=None, checkpointing=False, one_token_grads=False,
                       floors=False, floor_kinds=None, fwd_bars=None):
    """The U-Net `arch` at `size`, batch n, timesteps t (s: an s-token encoding): one seeded training forward and backward
    (cases.train_step), every block and the timestep MLP against fp64 (run_backward_checks).
    floors: the bf16 floors of the bars measured in the same run on the fp64 oracle's own activations, which make them a
    function of the seeds alone; the bars of floor_kinds (None: all) must lie in the rule's range of them.  fwd_bars
    (with floors): the training forward block by block as well, every tap kept.
    checkpointing: under enable_gradient_checkpointing(), whose backward recomputes each block's internals; the block
    outputs and their gradients, all the comparison reads, are kept, so it is held to the same bars.
    one_token_grads: every transformer's cases.ONE_TOKEN_ZERO gradients are exactly zero with one token and nonzero with
    more.  Returns (model, blocks) for the caller's own checks."""
    from oracle.unet_cond_oracle import unet_cond_forward
    from oracle.unet_oracle import unet_forward
    model, cfg, w = cases.build(arch, seed, cuda, size)
    if checkpointing:
        model.enable_gradient_checkpointing()
    noisy, t, enc, noise, eps, g_eps = cases.train_step(model, size, n, seed, t, s)
    blocks = bg.unet_blocks(cfg)
    if one_token_grads:
        named = dict(model.named_parameters())
        once = [k for k in named if k.endswith(cases.ONE_TOKEN_ZERO) and ".transformer_blocks." in k]
        assert len(once) == 4 * sum(b.kind == "transformer" for b in blocks)
        assert all((torch.count_nonzero(named[k].grad) > 0) == (s > 1) for k in once), s
    w64 = cases.w64(w, cuda)
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    temb = bg.temb_act(w64, cfg, t)
    fails = run_backward_checks(model, blocks, noisy, g_eps, w64, cfg, bars, temb=temb, enc=enc, t=t)
    name = (f"{type(model).__name__} {size[0]}x{size[1]} batch {n}" + (f", {s} tokens" if s and s > 1 else "")
            + (", checkpointed" if checkpointing else ""))
    report_time(name, t0)
    bad = []
    if floors:
        taps, x64, e64 = {}, noisy.double(), None if enc is None else enc.double()
        with torch.no_grad():
            if enc is None:
                ref = unet_forward(w64, cfg, x64, t, taps)
            else:
                ref = unet_cond_forward(w64, cfg, x64, t, e64, taps)
        g_ref = 2 * (ref - noise.double()) / ref.numel()
        # the plain oracle's own temb_act tap; the conditional oracle keeps none, so temb_act() of the same timesteps
        fl = bg.backward_floors(blocks, taps, x64, g_ref, w64, cfg, taps.get("temb_act", temb), e64, t)
        bad = report_backward_floors(fl, bars, floor_kinds)
    assert not fails, fails
    assert not bad, bad
    if fwd_bars is not None:
        frows = forward_checks(model.debug_tensor, blocks, noisy, eps, w64, cfg, temb, e64, taps="all")
        ffl = bg.forward_floors(blocks, taps, x64, w64, cfg, temb, e64, taps="all")
        check_against_floors(name + ", training forward", frows, ffl, fwd_bars, t0)
    return model, blocks


def vae_backward_case(cuda, size, seed, bars, checkpointing=False, floors=False, fwd_bars=None):
    """The ldm autoencoder at `size`, batch 2: encoder backward from seeded moment gradients and decoder backward from a
    seeded image gradient, every block of the decoder then the encoder against fp64; floors, fwd_bars and checkpointing
    as unet_backward_case."""
    from oracle import vae_oracle as vo
    model, cfg, w = cases.build(cases.LDM, seed, cuda, max_batch=2)
    if checkpointing:
        model.enable_gradient_checkpointing()
    lat = (size[0] // 8, size[1] // 8)
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(2, 1, *size, generator=g).clamp(-1, 1).to(cuda)
    z = torch.randn(2, 1, *lat, generator=g).to(cuda)
    gx = torch.randn(2, 1, *size, generator=g).to(cuda)
    gm = torch.randn(2, 2, *lat, generator=g).to(cuda)
    mom = model.encode(x).latent_dist.parameters
    mom.backward(gm)
    zz = z.clone().requires_grad_(True)
    img = model.decode(zz).sample
    img.backward(gx)
    w64 = cases.w64(w, cuda)
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    fails = run_backward_checks(model, bg.vae_blocks(cfg, "decoder"), z, gx, w64, cfg, bars, "decoder:", g_in=zz.grad)
    fails += run_backward_checks(model, bg.vae_blocks(cfg, "encoder"), x, gm, w64, cfg, bars, "encoder:")
    name = f"AutoencoderKL {size[0]}x{size[1]} batch 2" + (", checkpointed" if checkpointing else "")
    report_time(name, t0)
    bad, fl, frows, ffl = [], {}, [], {}
    if floors:
        for part, inp, gout, fwd, out in (("decoder", z, gx, vo.decode, img.detach()),
                                          ("encoder", x, gm, vo.encode_moments, mom.detach())):
            taps = {}
            with torch.no_grad():
                fwd(w64, cfg, inp.double(), taps)
            blocks = bg.vae_blocks(cfg, part)
            for k, v in bg.backward_floors(blocks, taps, inp.double(), gout.double(), w64, cfg).items():
                fl[part + ":" + k] = v
            if fwd_bars is not None:
                frows += forward_checks(model.debug_tensor, blocks, inp.double(), out, w64, cfg, prefix=part + ":",
                                        taps="all")
                ffl.update(bg.forward_floors(blocks, taps, inp.double(), w64, cfg, prefix=part + ":", taps="all"))
        bad = report_backward_floors(fl, bars)
    assert not fails, fails
    assert not bad, bad
    if fwd_bars is not None:
        check_against_floors(name + ", training forward", frows, ffl, fwd_bars, t0)


# ---------------------------------------------------------------------------------------------------- forward
def _keyed_errors(rows, key, got, ref):
    rows.append((key,) + bg.errors(got, ref, act=True))
    if key.endswith(".h1"):
        rows.append((key + ":mean",) + (bg.mean_offset(got, ref),) * 3)


def forward_checks(read, blocks, model_in, model_out, w, cfg, temb=None, enc=None, prefix="", taps=None, sel=None):
    """Compares every block and sub-block tap of the engine's forward with its fp64 reference on the engine's own inputs;
    read(name) reads an engine activation (debug_tensor), sel: the compared samples (None: all), model_in / model_out are
    the model's input and output on them; taps: the sub-taps to read (None: those kept in eval mode, "all": every one).
    Returns [(block, key, a, b, c)] and prints one table row per block and key."""
    si = None if sel is None else torch.tensor(sel, device=model_out.device)
    tap = lambda name: (read(name) if si is None else read(name).index_select(0, si)).double()
    out = []
    print(f"\n{'block':44s} {'key':22s} {'L2':>8s} {'max':>8s} {'row':>8s}")
    for blk in blocks:
        xs = [model_in if blk.inp is None else tap(blk.inp)] + ([tap(blk.skip)] if blk.skip else [])
        got = model_out if blk.out is None else tap(blk.out)
        rows = []
        _keyed_errors(rows, prefix + blk.kind, got, bg.block_forward(blk, w, xs, cfg, temb, enc))
        if blk.kind in bg.EVAL_SUBTAPS:
            subs = bg.sub_forward(blk, w, xs, cfg, temb, enc, get=lambda s: tap(blk.name + s), taps=taps)
            for s, ref in subs.items():
                _keyed_errors(rows, prefix + blk.kind + (".out" if s == "out" else s),
                              got if s == "out" else tap(blk.name + s), ref)
        if blk.kind in ("down", "down_asym"):
            par = read(blk.name + ".parity")        # the batch's four parity tensors viewed as one of 4C channels
            n, c4, hh, ww = par.shape
            par = par.reshape(n, c4 // 8, 8, hh, ww).reshape(4, n, c4 // 4, hh, ww)   # four tensors back to back
            x = read(blk.inp)
            split = torch.stack([x[:, :, a::2, b::2] for a in (0, 1) for b in (0, 1)]).to(par.dtype)
            same = torch.equal(par, split)
            rows.append((prefix + blk.kind + ".parity", 0.0 if same else 1.0, 0.0 if same else 1.0, 0.0 if same else 1.0))
        for key, a, b, c in rows:
            print(f"{blk.name or 'conv_out':44s} {key:22s} {a:8.5f} {b:8.5f} {c:8.5f}")
            out.append((blk.name, key, a, b, c))
    return out


def check_against_floors(name, rows, floors, bars, t0):
    """Prints the floors as a bar table and the fp64 time and peak memory; asserts the engine within its bars and every
    bar in (floor, 3.3 x floor]."""
    report_time(name, t0)
    print("floors as bars (3 x floor):")
    for key, f in sorted(floors.items()):
        f = tuple(round(v, 5) for v in f)
        print(f'    "{key}": ({round(3 * f[0], 5)}, {round(3 * f[1], 5)}, {round(3 * f[2], 5)}),   # floor {f}')
    use = bars or {k: tuple(3 * round(v, 5) for v in f) for k, f in floors.items()}
    over = [r for r in rows if r[1].endswith(".parity") and r[2] != 0.0]
    over += [r for r in rows if not r[1].endswith(".parity") and any(e > b for e, b in zip(r[2:], use[r[1]]))]
    for r in over:
        print("OVER", r, use.get(r[1]))
    assert bars, f"{name}: no bars stated"
    bad = [(k, f, bars.get(k)) for k, f in floors.items()
           if k not in bars or not all(bar_in_range(v, b, 3.3, 5) for v, b in zip(f, bars[k]))]
    assert not over, over
    assert not bad, bad


def forward_case(cuda, monkeypatch, arch, size, n, seed, bars, t=None, s=None, sel=None):
    """The eval forward of `arch` at `size`, batch n, block by block (forward_checks) with every activation in its own
    buffer (B200AD_DEBUG_NOPOOL=1), the bars against the floors measured in the same run (check_against_floors).  A U-Net:
    seeded samples at the timesteps t (s: with a seeded s-token encoding), the samples sel (None: all) compared; returns
    (x, t, w, eps) of the whole batch for the caller's further checks.  LDM: encode from a seeded image (compared output:
    the moments), then decode from seeded latents."""
    from oracle import vae_oracle as vo
    from oracle.unet_cond_oracle import unet_cond_forward
    from oracle.unet_oracle import unet_forward
    monkeypatch.setenv("B200AD_DEBUG_NOPOOL", "1")
    model, cfg, w = cases.build(arch, seed, cuda, size, train=False, max_batch=n)
    g = torch.Generator().manual_seed(seed + 1)
    if "latent_channels" in arch:
        x = torch.randn(n, 1, *size, generator=g).clamp(-1, 1).to(cuda)
        z = torch.randn(n, 1, size[0] // 8, size[1] // 8, generator=g).to(cuda)
        print(f"\n{power_limit()}")
        w64 = cases.w64(w, cuda)
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        rows, floors = [], {}
        for part, inp, fwd in (("encoder", x, vo.encode_moments), ("decoder", z, vo.decode)):
            with torch.no_grad():
                out = model.encode(inp).latent_dist.parameters if part == "encoder" else model.decode(inp).sample
            blocks = bg.vae_blocks(cfg, part)
            rows += forward_checks(model.debug_tensor, blocks, inp.double(), out, w64, cfg, prefix=part + ":")
            otaps = {}
            with torch.no_grad():
                fwd(w64, cfg, inp.double(), otaps)
            floors.update(bg.forward_floors(blocks, otaps, inp.double(), w64, cfg, prefix=part + ":"))
        check_against_floors(f"AutoencoderKL {size[0]}x{size[1]} batch {n}", rows, floors, bars, t0)
        return None
    x = torch.randn(n, arch.get("in_channels", 1), *size, generator=g).to(cuda)
    enc = None if s is None else torch.randn(n, s, 100, generator=g).to(cuda)
    t = torch.tensor(t, dtype=torch.float32, device=cuda)
    with torch.no_grad():
        eps = model(x, t)["sample"] if enc is None else model(x, t, enc)["sample"]
    print(f"\n{power_limit()}")
    si = torch.arange(n, device=cuda) if sel is None else torch.tensor(sel, device=cuda)
    w64 = cases.w64(w, cuda)
    blocks = bg.unet_blocks(cfg)
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    ts = t.long().index_select(0, si)
    temb = bg.temb_act(w64, cfg, ts)
    xin = x.index_select(0, si).double()
    e64 = None if enc is None else enc.index_select(0, si).double()
    rows = forward_checks(model.debug_tensor, blocks, xin, eps.index_select(0, si), w64, cfg, temb, e64, sel=sel)
    del model
    torch.cuda.empty_cache()
    otaps = {}
    with torch.no_grad():
        if enc is None:
            unet_forward(w64, cfg, xin, ts, otaps)
        else:
            unet_cond_forward(w64, cfg, xin, ts, e64, otaps)
    floors = bg.forward_floors(blocks, otaps, xin, w64, cfg, temb, e64)
    del otaps
    name = (f"{'UNet2DModel' if enc is None else 'UNet2DConditionModel'} {size[0]}x{size[1]} batch {n}"
            + (f", {s} tokens" if s and s > 1 else "") + ("" if sel is None else f", samples {sel}"))
    check_against_floors(name, rows, floors, bars, t0)
    return x, t, w, eps


def pooled_eps(cuda, arch, w, size, x, t):
    """eps of the same input through a UNet2DModel of `arch` with pooled activation buffers (the default), twice."""
    from audio_diffusion_b200.unet import UNet2DModel
    model = UNet2DModel(sample_size=size, **arch)
    model.load_state_dict(w)
    model = model.to(cuda).eval()
    with torch.no_grad():
        return model(x, t)["sample"], model(x, t)["sample"]


# ---------------------------------------------------------------------------------------------------- fused step
def check_fused_step(c, x, eps, x_out, z=None):
    """x_out of a fused scheduler step against the fp64 update of b200ad_step_coef's formula (include/b200ad.h) on the
    engine's own eps and the same noise z: the kernel evaluates it in six fp32 operations, so each element may differ by
    at most 8 fp32 roundings (8 * 2^-24) of the sum of its terms' magnitudes.  Asserts that bar on every channel plane;
    returns (the largest error over its bar per plane, the fraction of elements whose x0 the clip reaches)."""
    xd, ed = x.double(), eps.double()
    x0 = (xd - c.sqrt_1m_at * ed) * c.inv_sqrt_at
    clipped = (x0.abs() > c.clip).double().mean().item()
    if c.do_clip:
        x0 = x0.clamp(-c.clip, c.clip)
    ref = c.c_x0 * x0 + c.c_xt * xd + c.c_eps * ed
    mag = abs(c.c_x0) * c.inv_sqrt_at * (xd.abs() + c.sqrt_1m_at * ed.abs()) + abs(c.c_xt) * xd.abs() + abs(c.c_eps) * ed.abs()
    if z is not None:
        ref = ref + c.c_z * z.double()
        mag = mag + abs(c.c_z) * z.double().abs()
    ratio = ((x_out.double() - ref).abs() / (8 * 2.0 ** -24 * mag + 1e-30)).amax(dim=(0, 2, 3)).tolist()
    assert max(ratio) <= 1.0, ratio
    return ratio, clipped
