"""Plain-PyTorch fp32 restatement of diffusers==0.24.0 `UNet2DConditionModel.forward(sample, timestep,
encoder_hidden_states)` for exactly the configuration the reference constructs at scripts/train_unet.py:139-159
(CrossAttnDownBlock2D x3 + DownBlock2D, UpBlock2D + CrossAttnUpBlock2D x3, block_out_channels (128, 256, 512, 512),
cross_attention_dim = width of the audio encodings = 100, audiodiffusion/audio_encoder.py:75) and calls at
audiodiffusion/pipeline_audio_diffusion.py:160-161 and scripts/train_unet.py:255.

TEST INFRASTRUCTURE (see oracle/__init__.py).  PARITY UNPINNED: diffusers is not available in this environment; this
follows the published 0.24.0 module graph ([3P-recall]):
  * `attention_head_dim=8` is, in UNet2DConditionModel, the NUMBER of heads (num_attention_heads defaults to it);
    head_dim = channels / 8;
  * Transformer2DModel (continuous input, use_linear_projection=False): GroupNorm(32, eps 1e-6) -> 1x1 conv proj_in ->
    BasicTransformerBlock -> 1x1 conv proj_out -> + residual;
  * BasicTransformerBlock: x += attn1(LayerNorm(x)); x += attn2(LayerNorm(x), encoder_hidden_states);
    x += ff(LayerNorm(x)); attention projections without bias (attention_bias=False), `to_out.0` with bias;
    ff = GEGLU(dim -> 4 dim) -> Linear(4 dim -> dim), exact (erf) GELU;
  * mid block = ResnetBlock2D, Transformer2DModel, ResnetBlock2D; resnets / samplers as in UNet2DModel.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Tuple

import torch
import torch.nn.functional as F

from .unet_oracle import _resnet, timestep_embedding


@dataclass
class CondUNetConfig:
    """Mirror of the UNet2DConditionModel ctor kwargs used at scripts/train_unet.py:139-159."""

    sample_size: Tuple[int, int] = (64, 64)
    in_channels: int = 1
    out_channels: int = 1
    layers_per_block: int = 2
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    down_block_types: Tuple[str, ...] = ("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D")
    up_block_types: Tuple[str, ...] = ("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D")
    cross_attention_dim: int = 100
    attention_head_dim: int = 8          # = number of heads (see module docstring)
    norm_num_groups: int = 32
    norm_eps: float = 1e-5


def param_shapes(cfg: CondUNetConfig) -> Dict[str, Tuple[int, ...]]:
    """State-dict key -> shape, diffusers 0.24 layout."""
    sh: Dict[str, Tuple[int, ...]] = {}
    boc = cfg.block_out_channels
    temb = boc[0] * 4
    X = cfg.cross_attention_dim

    def conv(name, cin, cout, k):
        sh[name + ".weight"] = (cout, cin, k, k)
        sh[name + ".bias"] = (cout,)

    def lin(name, cin, cout, bias=True):
        sh[name + ".weight"] = (cout, cin)
        if bias:
            sh[name + ".bias"] = (cout,)

    def norm(name, c):
        sh[name + ".weight"] = (c,)
        sh[name + ".bias"] = (c,)

    def resnet(name, cin, cout):
        norm(name + ".norm1", cin)
        conv(name + ".conv1", cin, cout, 3)
        lin(name + ".time_emb_proj", temb, cout)
        norm(name + ".norm2", cout)
        conv(name + ".conv2", cout, cout, 3)
        if cin != cout:
            conv(name + ".conv_shortcut", cin, cout, 1)

    def transformer(name, c):
        norm(name + ".norm", c)
        conv(name + ".proj_in", c, c, 1)
        b = name + ".transformer_blocks.0"
        norm(b + ".norm1", c)
        for p in ("to_q", "to_k", "to_v"):
            lin(f"{b}.attn1.{p}", c, c, bias=False)
        lin(b + ".attn1.to_out.0", c, c)
        norm(b + ".norm2", c)
        lin(b + ".attn2.to_q", c, c, bias=False)
        lin(b + ".attn2.to_k", X, c, bias=False)
        lin(b + ".attn2.to_v", X, c, bias=False)
        lin(b + ".attn2.to_out.0", c, c)
        norm(b + ".norm3", c)
        lin(b + ".ff.net.0.proj", c, 8 * c)
        lin(b + ".ff.net.2", 4 * c, c)
        conv(name + ".proj_out", c, c, 1)

    conv("conv_in", cfg.in_channels, boc[0], 3)
    lin("time_embedding.linear_1", boc[0], temb)
    lin("time_embedding.linear_2", temb, temb)
    out_c = boc[0]
    for i, typ in enumerate(cfg.down_block_types):
        in_c, out_c = out_c, boc[i]
        for j in range(cfg.layers_per_block):
            resnet(f"down_blocks.{i}.resnets.{j}", in_c if j == 0 else out_c, out_c)
            if typ == "CrossAttnDownBlock2D":
                transformer(f"down_blocks.{i}.attentions.{j}", out_c)
        if i != len(boc) - 1:
            conv(f"down_blocks.{i}.downsamplers.0.conv", out_c, out_c, 3)
    mid = boc[-1]
    resnet("mid_block.resnets.0", mid, mid)
    transformer("mid_block.attentions.0", mid)
    resnet("mid_block.resnets.1", mid, mid)
    rev = list(reversed(boc))
    out_c = rev[0]
    for i, typ in enumerate(cfg.up_block_types):
        prev_c = out_c
        out_c = rev[i]
        in_c = rev[min(i + 1, len(boc) - 1)]
        n = cfg.layers_per_block + 1
        for j in range(n):
            skip_c = in_c if j == n - 1 else out_c
            res_in = prev_c if j == 0 else out_c
            resnet(f"up_blocks.{i}.resnets.{j}", res_in + skip_c, out_c)
            if typ == "CrossAttnUpBlock2D":
                transformer(f"up_blocks.{i}.attentions.{j}", out_c)
        if i != len(boc) - 1:
            conv(f"up_blocks.{i}.upsamplers.0.conv", out_c, out_c, 3)
    norm("conv_norm_out", boc[0])
    conv("conv_out", boc[0], cfg.out_channels, 3)
    return sh


def init_weights(cfg: CondUNetConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded synthetic weights: PyTorch default init; norm affine parameters perturbed so that tests exercise them."""
    g = torch.Generator().manual_seed(seed)
    shapes = param_shapes(cfg)
    w: Dict[str, torch.Tensor] = {}
    for name, shape in shapes.items():
        leaf = name.rsplit(".", 2)[-2]
        if leaf.startswith("norm") or leaf == "conv_norm_out":
            w[name] = (1.0 if name.endswith(".weight") else 0.0) + 0.1 * torch.randn(shape, generator=g)
            continue
        wshape = shape if name.endswith(".weight") else shapes[name[:-5] + ".weight"]
        bound = 1.0 / math.sqrt(int(math.prod(wshape[1:])))
        w[name] = (torch.rand(shape, generator=g) * 2 - 1) * bound
    return w


def _mha(q, k, v, heads):
    b, nq, c = q.shape
    d = c // heads
    q = q.view(b, nq, heads, d).transpose(1, 2)
    k = k.view(b, -1, heads, d).transpose(1, 2)
    v = v.view(b, -1, heads, d).transpose(1, 2)
    s = torch.softmax((q @ k.transpose(-1, -2)) * (d ** -0.5), dim=-1)
    return (s @ v).transpose(1, 2).reshape(b, nq, c)


def _transformer(w, p, x, enc, cfg: CondUNetConfig, taps=None):
    b, c, hh, ww = x.shape
    heads = cfg.attention_head_dim
    res = x
    h = F.group_norm(x, cfg.norm_num_groups, w[p + ".norm.weight"], w[p + ".norm.bias"], 1e-6)
    h = F.conv2d(h, w[p + ".proj_in.weight"], w[p + ".proj_in.bias"])
    h = h.permute(0, 2, 3, 1).reshape(b, hh * ww, c)
    t = p + ".transformer_blocks.0"
    n1 = F.layer_norm(h, (c,), w[t + ".norm1.weight"], w[t + ".norm1.bias"], 1e-5)
    a = _mha(F.linear(n1, w[t + ".attn1.to_q.weight"]), F.linear(n1, w[t + ".attn1.to_k.weight"]),
             F.linear(n1, w[t + ".attn1.to_v.weight"]), heads)
    h = F.linear(a, w[t + ".attn1.to_out.0.weight"], w[t + ".attn1.to_out.0.bias"]) + h
    if taps is not None:
        taps[p + ".attn1"] = h.transpose(1, 2).reshape(b, c, hh, ww)
    n2 = F.layer_norm(h, (c,), w[t + ".norm2.weight"], w[t + ".norm2.bias"], 1e-5)
    a = _mha(F.linear(n2, w[t + ".attn2.to_q.weight"]), F.linear(enc, w[t + ".attn2.to_k.weight"]),
             F.linear(enc, w[t + ".attn2.to_v.weight"]), heads)
    h = F.linear(a, w[t + ".attn2.to_out.0.weight"], w[t + ".attn2.to_out.0.bias"]) + h
    if taps is not None:
        taps[p + ".attn2"] = h.transpose(1, 2).reshape(b, c, hh, ww)
    n3 = F.layer_norm(h, (c,), w[t + ".norm3.weight"], w[t + ".norm3.bias"], 1e-5)
    u, gate = F.linear(n3, w[t + ".ff.net.0.proj.weight"], w[t + ".ff.net.0.proj.bias"]).chunk(2, dim=-1)
    h = F.linear(u * F.gelu(gate), w[t + ".ff.net.2.weight"], w[t + ".ff.net.2.bias"]) + h
    h = h.reshape(b, hh, ww, c).permute(0, 3, 1, 2)
    out = F.conv2d(h, w[p + ".proj_out.weight"], w[p + ".proj_out.bias"]) + res
    if taps is not None:
        taps[p] = out
    return out


def unet_cond_forward(w: Dict[str, torch.Tensor], cfg: CondUNetConfig, sample: torch.Tensor, timestep,
                      encoder_hidden_states: torch.Tensor, taps: Dict[str, torch.Tensor] | None = None) -> torch.Tensor:
    """UNet2DConditionModel.forward(sample, timestep, encoder_hidden_states).sample (pipeline_audio_diffusion.py:161).
    `encoder_hidden_states`: (B, S, cross_attention_dim)."""
    boc = cfg.block_out_channels
    g, eps = cfg.norm_num_groups, cfg.norm_eps
    t = timestep
    if not torch.is_tensor(t):
        t = torch.tensor([t], dtype=torch.long, device=sample.device)
    elif t.ndim == 0:
        t = t[None]
    t = t * torch.ones(sample.shape[0], dtype=t.dtype, device=t.device)
    emb = timestep_embedding(t, boc[0]).to(sample.dtype)
    emb = F.linear(F.silu(F.linear(emb, w["time_embedding.linear_1.weight"], w["time_embedding.linear_1.bias"])),
                   w["time_embedding.linear_2.weight"], w["time_embedding.linear_2.bias"])
    temb_act = F.silu(emb)
    enc = encoder_hidden_states.to(sample.dtype)

    h = F.conv2d(sample, w["conv_in.weight"], w["conv_in.bias"], padding=1)
    if taps is not None:
        taps["conv_in"] = h
    skips: List[torch.Tensor] = [h]
    for i, typ in enumerate(cfg.down_block_types):
        for j in range(cfg.layers_per_block):
            h = _resnet(w, f"down_blocks.{i}.resnets.{j}", h, temb_act, g, eps, taps)
            if typ == "CrossAttnDownBlock2D":
                h = _transformer(w, f"down_blocks.{i}.attentions.{j}", h, enc, cfg, taps)
            skips.append(h)
        if i != len(boc) - 1:
            p = f"down_blocks.{i}.downsamplers.0.conv"
            h = F.conv2d(h, w[p + ".weight"], w[p + ".bias"], stride=2, padding=1)
            if taps is not None:
                taps[p] = h
            skips.append(h)
    h = _resnet(w, "mid_block.resnets.0", h, temb_act, g, eps, taps)
    h = _transformer(w, "mid_block.attentions.0", h, enc, cfg, taps)
    h = _resnet(w, "mid_block.resnets.1", h, temb_act, g, eps, taps)
    for i, typ in enumerate(cfg.up_block_types):
        for j in range(cfg.layers_per_block + 1):
            h = torch.cat([h, skips.pop()], dim=1)
            h = _resnet(w, f"up_blocks.{i}.resnets.{j}", h, temb_act, g, eps, taps)
            if typ == "CrossAttnUpBlock2D":
                h = _transformer(w, f"up_blocks.{i}.attentions.{j}", h, enc, cfg, taps)
        if i != len(boc) - 1:
            p = f"up_blocks.{i}.upsamplers.0.conv"
            h = F.interpolate(h, scale_factor=2.0, mode="nearest")
            h = F.conv2d(h, w[p + ".weight"], w[p + ".bias"], padding=1)
            if taps is not None:
                taps[p] = h
    assert not skips
    h = F.silu(F.group_norm(h, g, w["conv_norm_out.weight"], w["conv_norm_out.bias"], eps))
    return F.conv2d(h, w["conv_out.weight"], w["conv_out.bias"], padding=1)
