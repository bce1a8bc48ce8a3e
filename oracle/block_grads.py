"""Per-block fp64 references of the U-Net and autoencoder backward (TEST INFRASTRUCTURE, see oracle/__init__.py).

The engine's backward walks the forward's block list in reverse (csrc/backward.cu).  Each block there turns the gradient
of its output into the gradients of its input(s) and of its own parameters.  `block_backward` does the same for one block
by fp64 autograd over the oracle's pieces (`unet_oracle._resnet` / `_attention`, `unet_cond_oracle._transformer`,
`vae_oracle._resnet` / `_attn`, and the oracles' inline down- / upsample, head and tail code), from whatever input
activations and output gradient it is given: the engine's own, so that a per-block comparison does not compound the
error of the blocks after it.

`unet_blocks` / `vae_blocks` restate the engine's block lists (input, skip connection, output tap, parameters);
`chain` runs the references in reverse over given activations, which is how tests/test_cpu_block_backward.py shows that
the decomposition reproduces autograd through the whole model.  The U-Net's timestep MLP (time_embedding.*) belongs to no
block: every resnet's reference also returns the gradient of the temb_act it reads (block_backward(temb_grad=True)), and
`temb_backward` takes their sum through the MLP, so that the blocks and the MLP together claim every parameter.

`bf16_storage()` rounds, inside a reference, every conv / linear operand, weight and output to bf16 and every gradient
that flows back through those operands and outputs: the points where the engine stores a tensor or a gradient in bf16.
Comparing a reference run under it with the exact one gives the bf16 floor of a block's gradients: `backward_floors`,
worst per block kind over a model's blocks.

The forward: `block_forward` is the same `_forward` evaluated in fp64 without autograd; `sub_forward` splits a resnet, an
attention block and a transformer into the steps whose outputs the engine keeps as taps (`.h1`; `.qkv`, `.ao`; `.h0` ..
`.h3`), each step computed from the given values of the steps before it, so that a per-step comparison on the engine's
own taps pins an error to one step.  tests/test_cpu_block_forward.py shows that both restate the model.  Their rounded
forms add the bf16 points only the forward has (bf16_storage(forward=True), the stored outputs), which give the forward
floors (`forward_floors`); the backward floors do not use them.
"""
from __future__ import annotations

import contextlib
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from . import unet_cond_oracle as uco
from . import unet_oracle as uo
from . import vae_oracle as vo


@dataclass(frozen=True)
class Block:
    kind: str                      # head, resnet, attn, transformer, down, up, tail (U-Net); dec_head, enc_tail,
                                   # resnet_vae, attn1, down_asym (autoencoder)
    name: str                      # diffusers name prefix of the block
    inp: Optional[str]             # forward tap of the main input (None: the model's input)
    skip: Optional[str]            # forward tap of the skip connection concatenated after the input
    out: Optional[str]             # forward tap of the output (None: the model's output)
    prefixes: Tuple[str, ...]      # the block's parameters: every name starting with one of these


def unet_blocks(cfg) -> List[Block]:
    """UNet2DModel / UNet2DConditionModel as the engine's block list (csrc/unet.cu: unet_blocks)."""
    boc = cfg.block_out_channels
    nb = len(boc)

    def attn_kind(t):
        return "transformer" if t.startswith("CrossAttn") else "attn" if t.startswith("Attn") else None

    bl = [Block("head", "conv_in", None, None, "conv_in", ("conv_in.",))]
    cur = "conv_in"
    skips = [cur]

    def add(kind, n, skip=None):
        nonlocal cur
        bl.append(Block(kind, n, cur, skip, n, (n + ".",)))
        cur = n

    for i, t in enumerate(cfg.down_block_types):
        for j in range(cfg.layers_per_block):
            add("resnet", f"down_blocks.{i}.resnets.{j}")
            if attn_kind(t):
                add(attn_kind(t), f"down_blocks.{i}.attentions.{j}")
            skips.append(cur)
        if i != nb - 1:
            add("down", f"down_blocks.{i}.downsamplers.0.conv")
            skips.append(cur)
    add("resnet", "mid_block.resnets.0")
    add("transformer" if hasattr(cfg, "cross_attention_dim") else "attn", "mid_block.attentions.0")
    add("resnet", "mid_block.resnets.1")
    for i, t in enumerate(cfg.up_block_types):
        for j in range(cfg.layers_per_block + 1):
            add("resnet", f"up_blocks.{i}.resnets.{j}", skips.pop())
            if attn_kind(t):
                add(attn_kind(t), f"up_blocks.{i}.attentions.{j}")
        if i != nb - 1:
            add("up", f"up_blocks.{i}.upsamplers.0.conv")
    assert not skips
    bl.append(Block("tail", "", cur, None, None, ("conv_norm_out.", "conv_out.")))
    return bl


def vae_blocks(cfg: vo.VAEConfig, part: str) -> List[Block]:
    """One part ("encoder" or "decoder") of AutoencoderKL as the engine's block list (csrc/vae.cu: vae_blocks)."""
    boc = cfg.block_out_channels
    nb = len(boc)
    if part == "encoder":
        bl = [Block("head", "encoder.conv_in", None, None, "encoder.conv_in", ("encoder.conv_in.",))]
    else:
        bl = [Block("dec_head", "decoder.conv_in", None, None, "decoder.conv_in", ("post_quant_conv.", "decoder.conv_in."))]
    cur = bl[0].out

    def add(kind, n):
        nonlocal cur
        bl.append(Block(kind, n, cur, None, n, (n + ".",)))
        cur = n

    def mid():
        add("resnet_vae", f"{part}.mid_block.resnets.0")
        add("attn1", f"{part}.mid_block.attentions.0")
        add("resnet_vae", f"{part}.mid_block.resnets.1")

    if part == "encoder":
        for i in range(nb):
            for j in range(cfg.layers_per_block):
                add("resnet_vae", f"encoder.down_blocks.{i}.resnets.{j}")
            if i != nb - 1:
                add("down_asym", f"encoder.down_blocks.{i}.downsamplers.0.conv")
        mid()
        bl.append(Block("enc_tail", "encoder.", cur, None, None,
                        ("encoder.conv_norm_out.", "encoder.conv_out.", "quant_conv.")))
    else:
        mid()
        for i in range(nb):
            for j in range(cfg.layers_per_block + 1):
                add("resnet_vae", f"decoder.up_blocks.{i}.resnets.{j}")
            if i != nb - 1:
                add("up", f"decoder.up_blocks.{i}.upsamplers.0.conv")
        bl.append(Block("tail", "decoder.", cur, None, None, ("decoder.conv_norm_out.", "decoder.conv_out.")))
    return bl


TEMB_PREFIXES = ("time_embedding.",)   # the timestep MLP's parameters: no block's; temb_backward checks them


def temb_act(w, cfg, t: torch.Tensor) -> torch.Tensor:
    """silu(time_embedding(t)): what every resnet's time_emb_proj reads (unet_oracle.unet_forward), in w's dtype."""
    dt = w["time_embedding.linear_1.weight"].dtype
    emb = uo.timestep_embedding(t, cfg.block_out_channels[0]).to(dt)
    emb = F.silu(F.linear(emb, w["time_embedding.linear_1.weight"], w["time_embedding.linear_1.bias"]))
    return F.silu(F.linear(emb, w["time_embedding.linear_2.weight"], w["time_embedding.linear_2.bias"]))


def temb_backward(w, cfg, t: torch.Tensor, g_temb: torch.Tensor) -> Dict[str, torch.Tensor]:
    """fp64 autograd of temb_act(w, cfg, t) from the gradient g_temb of its output (the sum of every resnet's, from
    block_backward): {parameter name: gradient} of the four time_embedding.* tensors."""
    dev = g_temb.device
    pw = {k: w[k].detach().to(device=dev, dtype=torch.float64).requires_grad_(True) for k in w
          if k.startswith(TEMB_PREFIXES)}
    out = temb_act(pw, cfg, t.to(dev))
    return dict(zip(pw.keys(), torch.autograd.grad(out, list(pw.values()), g_temb.to(torch.float64))))


def _forward(blk: Block, w, xs: Sequence[torch.Tensor], cfg, temb_act, enc):
    """The block's forward over the oracle pieces; xs = [input] or [input, skip]."""
    n = blk.name
    x = torch.cat(list(xs), dim=1) if len(xs) > 1 else xs[0]
    k = blk.kind
    if k == "resnet":
        return uo._resnet(w, n, x, temb_act, cfg.norm_num_groups, cfg.norm_eps)
    if k == "attn":
        return uo._attention(w, n, x, cfg.norm_num_groups, cfg.norm_eps, cfg.attention_head_dim)
    if k == "transformer":
        return uco._transformer(w, n, x, enc, cfg)
    if k == "resnet_vae":
        return vo._resnet(w, n, x, cfg.norm_num_groups)
    if k == "attn1":
        return vo._attn(w, n, x, cfg.norm_num_groups)
    if k == "down":
        return F.conv2d(x, w[n + ".weight"], w[n + ".bias"], stride=2, padding=1)
    if k == "down_asym":
        return F.conv2d(F.pad(x, (0, 1, 0, 1), mode="constant", value=0), w[n + ".weight"], w[n + ".bias"], stride=2)
    if k == "up":
        return F.conv2d(F.interpolate(x, scale_factor=2.0, mode="nearest"), w[n + ".weight"], w[n + ".bias"], padding=1)
    if k == "head":
        return F.conv2d(x, w[n + ".weight"], w[n + ".bias"], padding=1)
    if k == "dec_head":
        h = F.conv2d(x, w["post_quant_conv.weight"], w["post_quant_conv.bias"])
        return F.conv2d(h, w[n + ".weight"], w[n + ".bias"], padding=1)
    if k in ("tail", "enc_tail"):
        eps = vo.EPS if n else cfg.norm_eps
        h = F.silu(F.group_norm(x, cfg.norm_num_groups, w[n + "conv_norm_out.weight"], w[n + "conv_norm_out.bias"], eps))
        h = F.conv2d(h, w[n + "conv_out.weight"], w[n + "conv_out.bias"], padding=1)
        return F.conv2d(h, w["quant_conv.weight"], w["quant_conv.bias"]) if k == "enc_tail" else h
    raise ValueError(f"unknown block kind {k}")


def bf16(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.bfloat16).to(t.dtype)


class _Store(torch.autograd.Function):
    """Identity that rounds the value (fwd) and the gradient flowing back through it (bwd) to bf16."""

    @staticmethod
    def forward(ctx, x, fwd, bwd):
        ctx.bwd = bwd
        return bf16(x) if fwd else x.clone()

    @staticmethod
    def backward(ctx, g):
        return (bf16(g) if ctx.bwd else g), None, None


def _softmax_bf16_probs(x, dim=-1, **_):
    """softmax whose numerators exp(s - max) are rounded to bf16 while the denominator sums them exact: the P.V MMA of
    attention_mma_kernel (csrc/small_ops.cu) and mha_flash_kernel (csrc/cond_ops.cu) reads the unnormalised exp(S) packed
    to bf16 and divides by the fp32 row sum afterwards."""
    e = torch.exp(x - x.amax(dim, keepdim=True))
    return bf16(e) / e.sum(dim, keepdim=True)


@contextlib.contextmanager
def bf16_storage(forward: bool = False, bf16_probs: bool = False):
    """Inside: conv / linear operands and outputs are stored in bf16 both ways, weights are bf16 (their gradients are not
    rounded: the engine accumulates them in fp32).  Linear layers over [N, D] vectors (the time embedding) stay exact.

    forward: also the bf16 roundings only the forward makes (the forward floors; the backward floors leave it off):
    conv_out's weights over a wide input are bf16 (conv_out_kernel in csrc/elementwise.cu builds bf16 MMA fragments from
    them; the autoencoder's encoder conv_out runs on conv_tc_kernel with packed bf16 weights).  bf16_probs: the attention
    probabilities' numerators are bf16 (_softmax_bf16_probs); the SIMT attention_kernel and the single-head attention keep
    fp32 probabilities."""
    conv, lin, smax = F.conv2d, F.linear, torch.softmax
    st = lambda t: _Store.apply(t, True, True)
    wq = lambda t: _Store.apply(t, True, False)

    def c(a, wt, b=None, *args, **kw):
        # convs with at most 4 channels on a side (conv_in, conv_out, quant_conv, post_quant_conv) run their backward in
        # fp32 scalar kernels: that side's gradient and the weight stay exact; conv_out's output over a wide input is
        # stored in bf16 (the autoencoder's encoder tail reads it back for quant_conv's weight gradient)
        if min(wt.shape[:2]) <= 4:
            a = a if wt.shape[1] <= 4 else st(a)
            if forward and wt.shape[1] > 4:
                wt = wq(wt)
            y = conv(a, wt, b, *args, **kw)
            return st(y) if wt.shape[0] > 4 else y if wt.shape[1] <= 4 else _Store.apply(y, True, False)
        return st(conv(st(a), wq(wt), b, *args, **kw))

    def l(a, wt, b=None):
        # forward: the cross-attention over a one-token encoding is a per-sample vector in fp32 (cross_attn_vec_kernel)
        if a.dim() == 2 or (forward and a.shape[-2] == 1):
            return lin(a, wt, b)
        return st(lin(st(a), wq(wt), b))

    F.conv2d, F.linear = c, l
    if bf16_probs:
        torch.softmax = _softmax_bf16_probs
    try:
        yield
    finally:
        F.conv2d, F.linear, torch.softmax = conv, lin, smax


def block_backward(blk: Block, w: Dict[str, torch.Tensor], xs: Sequence[torch.Tensor], gout: torch.Tensor, cfg,
                   temb_act: Optional[torch.Tensor] = None, enc: Optional[torch.Tensor] = None, rounded: bool = False,
                   temb_grad: bool = False):
    """fp64 autograd of one block from its inputs xs and output gradient gout.  Returns (gradients w.r.t. xs, {parameter
    name: gradient} for the block's own parameters); temb_grad: also, third, the gradient w.r.t. temb_act, or None for a
    block that does not read it (only the U-Net's resnets do, through time_emb_proj).  rounded: under bf16_storage(),
    with the input gradients rounded to bf16 as the engine stores them (the temb_act gradient stays fp32 there: the
    engine sums it from fp32 channel sums)."""
    dev = gout.device
    d = lambda t: t.detach().to(device=dev, dtype=torch.float64)
    pw = {k: d(v).requires_grad_(True) for k, v in w.items() if k.startswith(blk.prefixes)}
    xl = [d(x).requires_grad_(True) for x in xs]
    reads_temb = (temb_grad and temb_act is not None and blk.kind == "resnet"
                  and blk.name + ".time_emb_proj.weight" in pw)
    ta = d(temb_act).requires_grad_(reads_temb) if temb_act is not None else None
    en = d(enc) if enc is not None else None
    with bf16_storage() if rounded else contextlib.nullcontext():
        out = _forward(blk, pw, xl, cfg, ta, en)
        leaves = xl + list(pw.values()) + ([ta] if reads_temb else [])
        gr = torch.autograd.grad(out, leaves, d(gout), allow_unused=True)
    gr = [torch.zeros_like(t) if g is None else g for t, g in zip(leaves, gr)]
    gi = gr[:len(xl)]
    if rounded:
        gi = [bf16(g) for g in gi]
    gp = dict(zip(pw.keys(), gr[len(xl):len(xl) + len(pw)]))
    return (gi, gp, gr[-1] if reads_temb else None) if temb_grad else (gi, gp)


def _probs_rounded(blk: Block, x: torch.Tensor) -> bool:
    """Whether the block's attention core packs its probabilities to bf16 (launch_attention picks attention_mma_kernel
    for seq % 16 == 0 and seq <= 1536; the transformers always run mha_flash_kernel)."""
    seq = x.shape[2] * x.shape[3]
    return blk.kind == "transformer" or (blk.kind == "attn" and seq % 16 == 0 and seq * 32 <= 48 * 1024)


def _stored(blk: Block, t: torch.Tensor) -> torch.Tensor:
    """The value as the engine stores the block's output: bf16, except the model outputs (eps, image, moments: fp32)."""
    return t if blk.kind in ("tail", "enc_tail") else bf16(t)


@torch.no_grad()
def block_forward(blk: Block, w: Dict[str, torch.Tensor], xs: Sequence[torch.Tensor], cfg,
                  temb_act: Optional[torch.Tensor] = None, enc: Optional[torch.Tensor] = None, rounded: bool = False):
    """fp64 forward of one block from its inputs xs ([input] or [input, skip]): the `_forward` that block_backward
    differentiates.  rounded: under bf16_storage(forward=True) with the forward's own bf16 points, output stored as the
    engine stores it."""
    dev = xs[0].device
    d = lambda t: None if t is None else t.detach().to(device=dev, dtype=torch.float64)
    pw = {k: d(v) for k, v in w.items() if k.startswith(blk.prefixes)}
    xl = [d(x) for x in xs]
    if not rounded:
        return _forward(blk, pw, xl, cfg, d(temb_act), d(enc))
    with bf16_storage(forward=True, bf16_probs=_probs_rounded(blk, xl[0])):
        return _stored(blk, _forward(blk, pw, xl, cfg, d(temb_act), d(enc)))


def _lnc(x, w, p, eps=1e-5):
    """LayerNorm over the channels of an NCHW tensor."""
    return F.layer_norm(x.permute(0, 2, 3, 1), (x.shape[1],), w[p + ".weight"], w[p + ".bias"], eps).permute(0, 3, 1, 2)


def _c1(x, wt, b=None):
    """A linear layer over the pixel tokens of an NCHW tensor (the engine's 1-tap conv)."""
    return F.conv2d(x, wt[:, :, None, None] if wt.dim() == 2 else wt, b)


def _attn_core(qkv, heads, bf16_probs):
    """softmax(q k^T / sqrt(d)) v per head over the pixel tokens of the q | k | v tensor [N, 3C, H, W] -> [N, C, H, W]."""
    n, c3, hh, ww = qkv.shape
    c = c3 // 3
    q, k, v = (t.reshape(n, heads, c // heads, hh * ww).transpose(-1, -2) for t in qkv.split(c, dim=1))
    s = (q @ k.transpose(-1, -2)) * (c // heads) ** -0.5
    p = _softmax_bf16_probs(s) if bf16_probs else torch.softmax(s, dim=-1)
    return (p @ v).transpose(-1, -2).reshape(n, c, hh, ww)


def _stages(blk: Block, w, x, cfg, temb_act, enc, bf16_probs):
    """The sub-block steps of a block as (tap suffix, step) pairs in order; a step maps the values so far (by suffix; ""
    is the block input, "out" the output) to its own value.  Sub-taps the engine exposes are exactly these suffixes."""
    n = blk.name
    G = cfg.norm_num_groups
    if blk.kind in ("resnet", "resnet_vae"):
        eps = cfg.norm_eps if blk.kind == "resnet" else vo.EPS

        def h1(v):
            h = F.conv2d(F.silu(F.group_norm(v[""], G, w[n + ".norm1.weight"], w[n + ".norm1.bias"], eps)),
                         w[n + ".conv1.weight"], w[n + ".conv1.bias"], padding=1)
            if temb_act is not None and n + ".time_emb_proj.weight" in w:
                h = h + F.linear(temb_act, w[n + ".time_emb_proj.weight"], w[n + ".time_emb_proj.bias"])[:, :, None, None]
            return h

        def out(v):
            h = F.silu(F.group_norm(v[".h1"], G, w[n + ".norm2.weight"], w[n + ".norm2.bias"], eps))
            h = F.conv2d(h, w[n + ".conv2.weight"], w[n + ".conv2.bias"], padding=1)
            sc = v[""]
            if n + ".conv_shortcut.weight" in w:
                sc = F.conv2d(sc, w[n + ".conv_shortcut.weight"], w[n + ".conv_shortcut.bias"])
            return sc + h
        return [(".h1", h1), ("out", out)]
    if blk.kind in ("attn", "attn1"):
        eps = cfg.norm_eps if blk.kind == "attn" else vo.EPS
        heads = x.shape[1] // cfg.attention_head_dim if blk.kind == "attn" else 1

        def qkv(v):
            h = F.group_norm(v[""], G, w[n + ".group_norm.weight"], w[n + ".group_norm.bias"], eps)
            wt = torch.cat([w[n + ".to_q.weight"], w[n + ".to_k.weight"], w[n + ".to_v.weight"]])
            return _c1(h, wt, torch.cat([w[n + ".to_q.bias"], w[n + ".to_k.bias"], w[n + ".to_v.bias"]]))
        return [(".qkv", qkv), (".ao", lambda v: _attn_core(v[".qkv"], heads, bf16_probs)),
                ("out", lambda v: _c1(v[".ao"], w[n + ".to_out.0.weight"], w[n + ".to_out.0.bias"]) + v[""])]
    if blk.kind == "transformer":
        t = n + ".transformer_blocks.0"
        heads = cfg.attention_head_dim

        def attn2(v):
            h = _c1(v[".ao"], w[t + ".attn1.to_out.0.weight"], w[t + ".attn1.to_out.0.bias"]) + v[".h0"]
            b, c, hh, ww = h.shape
            tok = h.permute(0, 2, 3, 1).reshape(b, hh * ww, c)
            n2 = F.layer_norm(tok, (c,), w[t + ".norm2.weight"], w[t + ".norm2.bias"], 1e-5)
            a = uco._mha(F.linear(n2, w[t + ".attn2.to_q.weight"]), F.linear(enc, w[t + ".attn2.to_k.weight"]),
                         F.linear(enc, w[t + ".attn2.to_v.weight"]), heads)
            a = F.linear(a, w[t + ".attn2.to_out.0.weight"], w[t + ".attn2.to_out.0.bias"])
            return h + a.reshape(b, hh, ww, c).permute(0, 3, 1, 2)

        def gg(v):
            u, gate = v[".ff1"].chunk(2, dim=1)
            return u * F.gelu(gate)
        return [
            (".h0", lambda v: _c1(F.group_norm(v[""], G, w[n + ".norm.weight"], w[n + ".norm.bias"], 1e-6),
                                  w[n + ".proj_in.weight"], w[n + ".proj_in.bias"])),
            (".n1", lambda v: _lnc(v[".h0"], w, t + ".norm1")),
            (".qkv", lambda v: _c1(v[".n1"], torch.cat([w[t + f".attn1.to_{p}.weight"] for p in "qkv"]))),
            (".ao", lambda v: _attn_core(v[".qkv"], heads, bf16_probs)),
            (".attn2", attn2),
            (".n3", lambda v: _lnc(v[".attn2"], w, t + ".norm3")),
            (".ff1", lambda v: _c1(v[".n3"], w[t + ".ff.net.0.proj.weight"], w[t + ".ff.net.0.proj.bias"])),
            (".gg", gg),
            (".h3", lambda v: _c1(v[".gg"], w[t + ".ff.net.2.weight"], w[t + ".ff.net.2.bias"]) + v[".attn2"]),
            ("out", lambda v: _c1(v[".h3"], w[n + ".proj_out.weight"], w[n + ".proj_out.bias"]) + v[""]),
        ]
    return [("out", lambda v: _forward(blk, w, [v[""]], cfg, temb_act, enc))]


# the sub-taps the engine keeps in eval mode (training keeps every one of a transformer's)
EVAL_SUBTAPS = {"resnet": (".h1",), "resnet_vae": (".h1",), "attn": (".qkv", ".ao"), "attn1": (".qkv", ".ao"),
                "transformer": (".attn2",)}


@torch.no_grad()
def sub_forward(blk: Block, w: Dict[str, torch.Tensor], xs: Sequence[torch.Tensor], cfg,
                temb_act: Optional[torch.Tensor] = None, enc: Optional[torch.Tensor] = None, get=None,
                taps: Optional[Sequence[str]] = None, rounded: bool = False) -> Dict[str, torch.Tensor]:
    """fp64 references of a block's sub-taps and output, each step computed from the given values of the steps before it:
    get(suffix) for the suffixes in `taps` (the engine's own sub-taps, so that an error is pinned to one step; default:
    those the engine keeps in eval mode, "all": every step), the reference's own value of the steps the engine does not
    expose.  Returns {suffix: reference} for the suffixes in taps
    and "out".  rounded: every step under bf16_storage(forward=True) and stored in bf16, as the engine stores them."""
    dev = xs[0].device
    d = lambda t: None if t is None else t.detach().to(device=dev, dtype=torch.float64)
    pw = {k: d(v) for k, v in w.items() if k.startswith(blk.prefixes)}
    xl = [d(x) for x in xs]
    x = torch.cat(xl, dim=1) if len(xl) > 1 else xl[0]
    probs = _probs_rounded(blk, x)
    vals = {"": x}
    res = {}
    with bf16_storage(forward=True, bf16_probs=probs) if rounded else contextlib.nullcontext():
        steps = _stages(blk, pw, x, cfg, d(temb_act), d(enc), probs and rounded)
        if taps is None:
            taps = EVAL_SUBTAPS.get(blk.kind, ())
        elif taps == "all":
            taps = [s for s, _ in steps[:-1]]
        for name, fn in steps:
            y = fn(vals)
            if rounded:
                y = _stored(blk, y) if name == "out" else bf16(y)
            if name in taps or name == "out":
                res[name] = y
            vals[name] = d(get(name)) if get is not None and name in taps else y
    return res


def chain(blocks: Sequence[Block], acts: Dict[str, torch.Tensor], model_in: torch.Tensor, g_out: torch.Tensor, w, cfg,
          temb_act=None, enc=None, t=None):
    """Runs block_backward over `blocks` in reverse from the gradient of the model's output, over the activations `acts`
    (by tap name): the gradient of every tap (skip shares added where the skip connection is consumed), every block
    parameter's gradient, and the gradient w.r.t. the model's input.  With the timesteps t (U-Net), the resnets'
    temb_act gradients summed and taken through the timestep MLP (temb_backward) give its parameters' gradients too."""
    G: Dict[str, torch.Tensor] = {}
    grads: Dict[str, torch.Tensor] = {}
    g_in = g_temb = None
    for blk in reversed(blocks):
        gout = g_out if blk.out is None else G[blk.out]
        xs = [model_in if blk.inp is None else acts[blk.inp]] + ([acts[blk.skip]] if blk.skip else [])
        gi, gp, gt = block_backward(blk, w, xs, gout, cfg, temb_act, enc, temb_grad=True)
        grads.update(gp)
        if gt is not None:
            g_temb = gt if g_temb is None else g_temb + gt
        if blk.inp is None:
            g_in = gi[0]
        else:
            G[blk.inp] = G[blk.inp] + gi[0] if blk.inp in G else gi[0]
        if blk.skip:
            G[blk.skip] = G[blk.skip] + gi[1] if blk.skip in G else gi[1]
    if t is not None:
        grads.update(temb_backward(w, cfg, t, g_temb))
    return G, grads, g_in


def errors(got: torch.Tensor, ref: torch.Tensor, act: bool = False, groups: int = 32):
    """(a) relative L2; (b) max |err| / max |ref|; (c) worst relative L2 of one row: per output channel for a weight
    gradient, per (sample, channel group) for an activation gradient (act), each against its row norm plus a tenth of
    the RMS row norm (rows whose reference is near zero do not dominate).  Vectors (biases, norm affines) and tensors of
    at most 4 rows (quant_conv, conv_out with 1-2 outputs), where a row is most of the tensor: (c) = (a)."""
    got, ref = got.double(), ref.double().to(got.device)
    err = got - ref
    rn = ref.norm().item()
    a = err.norm().item() / (rn + 1e-300)
    b = err.abs().max().item() / (ref.abs().max().item() + 1e-300)
    if ref.dim() < 2:
        return a, b, a
    rows = ref.shape[0] * (groups if act and ref.shape[1] % groups == 0 else 1)
    if rows <= 4:
        return a, b, a
    rows_e, rows_r = err.reshape(rows, -1), ref.reshape(rows, -1)
    rr = rows_r.norm(dim=1)
    floor = 0.1 * rn / rows_r.shape[0] ** 0.5
    c = (rows_e.norm(dim=1) / (rr + floor + 1e-300)).max().item()
    return a, b, c


def compare_block(acts: Dict[str, Tuple[torch.Tensor, torch.Tensor]], params: Dict[str, Tuple[torch.Tensor, torch.Tensor]]):
    """errors() of a block's activation gradients and parameter gradients, each given as label -> (got, ref).  Returns
    (rows, skipped): rows = [(label, is_activation, a, b, c)]; skipped = the parameters whose reference gradient is zero
    up to fp64 rounding (softmax-invariant biases), below 1e-9 of the block's largest."""
    rows = [(k, True) + errors(g, r, act=True) for k, (g, r) in acts.items()]
    scale = max((r.double().norm().item() for _, r in params.values()), default=0.0)
    skipped = []
    for k, (g, r) in params.items():
        if r.double().norm().item() <= 1e-9 * scale:
            skipped.append(k)
            continue
        rows.append((k, False) + errors(g, r))
    return rows, skipped


def worst(rows, is_act: bool):
    """Largest (a), (b), (c) over the rows of one class (activation or parameter gradients)."""
    sel = [r[2:] for r in rows if r[1] == is_act]
    return tuple(max((s[i] for s in sel), default=0.0) for i in range(3))


def backward_floors(blocks, taps, model_in, g_out, w, cfg, temb=None, enc=None, t=None):
    """bf16 floor of every block (rounded storage against exact, over bf16 inputs and upstream gradients), worst per
    kind: {kind: (activation (a, b, c), parameter (a, b, c))}.  With the timesteps t (U-Net), also "temb": the timestep
    MLP's parameter gradients from the sum of the resnets' rounded-storage temb_act gradients against the exact sum."""
    G, _, _ = chain(blocks, taps, model_in, g_out, w, cfg, temb, enc)
    out = {}
    gt_exact = gt_round = 0.0
    for blk in blocks:
        xs = [model_in if blk.inp is None else bf16(taps[blk.inp])] + ([bf16(taps[blk.skip])] if blk.skip else [])
        gout = g_out if blk.out is None else bf16(G[blk.out])
        ei, ep, et = block_backward(blk, w, xs, gout, cfg, temb, enc, temb_grad=True)
        ri, rp, rt = block_backward(blk, w, xs, gout, cfg, temb, enc, True, temb_grad=True)
        if et is not None:
            gt_exact, gt_round = gt_exact + et, gt_round + rt
        acts = {} if blk.inp is None else {"in": (ri[0], ei[0])}
        if blk.skip:
            acts["skip"] = (ri[1], ei[1])
        rows, _ = compare_block(acts, {k: (rp[k], ep[k]) for k in ep})
        wa, wp = worst(rows, True), worst(rows, False)
        pa, pp = out.get(blk.kind, ((0.0,) * 3, (0.0,) * 3))
        out[blk.kind] = (tuple(map(max, pa, wa)), tuple(map(max, pp, wp)))
    if t is not None:
        ep, rp = temb_backward(w, cfg, t, gt_exact), temb_backward(w, cfg, t, gt_round)
        rows, _ = compare_block({}, {k: (rp[k], ep[k]) for k in ep})
        out["temb"] = ((0.0,) * 3, worst(rows, False))
    for k, (a, p) in out.items():
        print(f"floor {k:12s} act L2 {a[0]:.4f} max {a[1]:.4f} row {a[2]:.4f} | param L2 {p[0]:.4f} max {p[1]:.4f} "
              f"row {p[2]:.4f}")
    return out


def mean_offset(got, ref):
    """Largest |mean over the pixels of the error| of one (sample, channel), over the RMS of the reference: what a wrong
    per-sample time-embedding row or bias adds to a resnet's h1 is constant over the pixels, while rounding errors
    average out there."""
    err = (got.double() - ref.double()).mean(dim=(2, 3))
    return (err.abs().max() / ref.double().pow(2).mean().sqrt()).item()


def forward_floors(blocks, otaps, model_in, w, cfg, temb=None, enc=None, prefix="", taps=None):
    """bf16 floor of every block and step, worst per key: {key: (a, b, c)}."""
    fl = {}

    def put(key, got, ref):
        e = errors(got, ref, act=True)
        fl[key] = tuple(map(max, fl.get(key, (0.0,) * 3), e))
        if key.endswith(".h1"):
            fl[key + ":mean"] = tuple(map(max, fl.get(key + ":mean", (0.0,) * 3), (mean_offset(got, ref),) * 3))

    for blk in blocks:
        xs = [model_in if blk.inp is None else bf16(otaps[blk.inp])] + ([bf16(otaps[blk.skip])] if blk.skip else [])
        put(prefix + blk.kind, block_forward(blk, w, xs, cfg, temb, enc, rounded=True),
            block_forward(blk, w, xs, cfg, temb, enc))
        if blk.kind in EVAL_SUBTAPS:
            exact = sub_forward(blk, w, xs, cfg, temb, enc, taps=taps)
            get = lambda s: bf16(exact[s])
            ex = sub_forward(blk, w, xs, cfg, temb, enc, get=get, taps=taps)
            rd = sub_forward(blk, w, xs, cfg, temb, enc, get=get, taps=taps, rounded=True)
            for s in ex:
                put(prefix + blk.kind + (".out" if s == "out" else s), rd[s], ex[s])
    return fl
