"""`UNet2DConditionModel` — drop-in for `diffusers.UNet2DConditionModel` as the reference constructs it
(scripts/train_unet.py:139-159) and calls it (`unet(sample, t, encoding)["sample"]`,
audiodiffusion/pipeline_audio_diffusion.py:160-161; scripts/train_unet.py:255): the conditional audio-diffusion model whose
cross-attention reads the 100-d audio encodings of `audiodiffusion/audio_encoder.py:62-107`.

Same constructor kwargs and diffusers state-dict keys (`down_blocks.i.attentions.j.transformer_blocks.0.attn1.to_q.weight`, ...).
Inference and training run in libb200ad.so: every projection / linear of the transformer blocks on the wgmma conv kernel
(and, in the backward, its data- and weight-gradient forms), self-attention (8 heads, head_dim = channels / 8) on flash-style
tensor-core kernels (the backward recomputes the attention matrix from the forward's row log-sum-exp).  Cross-attention:
an encoding of ONE token (the pooled AudioEncoder output, (B, 1, 100)) is a per-sample vector folded into the attn1 output
projection (softmax over one key is 1); an encoding of S > 1 tokens (e.g. `AudioEncoder.encode(files, pool=None)`: one token
per 5-second slice) runs the cross-attention kernels: the K / V projections of the encoding, flash-style attention of the
pixels against the S tokens and, in training, its backward down to the to_q / to_k / to_v weight gradients.

Training (`scripts/train_unet.py --encodings`: `model(noisy, t, enc)["sample"]`, MSE, `loss.backward()`) goes through the
same autograd node as `UNet2DModel`: parameter gradients only, as `p.grad` views of one flat buffer.  Limits: encoder
sequence length 1 <= S <= 256 (256 slices of 5 seconds: about 21 minutes of audio; a change of S re-plans the workspace);
no gradient w.r.t. the encoding (the reference's encodings are precomputed data), so an encoding with `requires_grad` is
refused in training.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple, Union

import torch

from ._lib import MAX_BLOCKS, StepCoefC
from .engine import _Cfg
from .unet import UNet2DModel, _unet_config

MAX_ENCODER_LEN = 256   # tokens of an encoding (the cross-attention kernels stage all of them in shared memory)


class UNet2DConditionModel(UNet2DModel):
    is_conditional = True

    def __init__(
        self,
        sample_size: Optional[Union[int, Tuple[int, int]]] = None,
        in_channels: int = 4,
        out_channels: int = 4,
        center_input_sample: bool = False,
        flip_sin_to_cos: bool = True,
        freq_shift: int = 0,
        down_block_types: Sequence[str] = ("CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"),
        mid_block_type: Optional[str] = "UNetMidBlock2DCrossAttn",
        up_block_types: Sequence[str] = ("UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"),
        only_cross_attention: bool = False,
        block_out_channels: Sequence[int] = (320, 640, 1280, 1280),
        layers_per_block: int = 2,
        downsample_padding: int = 1,
        mid_block_scale_factor: float = 1,
        dropout: float = 0.0,
        act_fn: str = "silu",
        norm_num_groups: int = 32,
        norm_eps: float = 1e-5,
        cross_attention_dim: int = 1280,
        transformer_layers_per_block: int = 1,
        attention_head_dim: int = 8,
        num_attention_heads: Optional[int] = None,
        dual_cross_attention: bool = False,
        use_linear_projection: bool = False,
        class_embed_type: Optional[str] = None,
        upcast_attention: bool = False,
        resnet_time_scale_shift: str = "default",
        time_embedding_type: str = "positional",
        seed: Optional[int] = None,
    ):
        torch.nn.Module.__init__(self)
        bad = []
        if center_input_sample or not flip_sin_to_cos or freq_shift != 0: bad.append("input / timestep embedding options")
        if mid_block_type != "UNetMidBlock2DCrossAttn": bad.append("mid_block_type")
        if only_cross_attention or dual_cross_attention or use_linear_projection or upcast_attention: bad.append("attention options")
        if downsample_padding != 1 or mid_block_scale_factor != 1 or dropout: bad.append("padding / scale / dropout")
        if act_fn != "silu" or resnet_time_scale_shift != "default" or time_embedding_type != "positional": bad.append("act / shift / time")
        if transformer_layers_per_block != 1 or class_embed_type is not None: bad.append("transformer depth / class embedding")
        heads = num_attention_heads if num_attention_heads is not None else attention_head_dim   # diffusers 0.24 naming quirk
        if heads != 8: bad.append("number of attention heads != 8")
        if len(block_out_channels) > MAX_BLOCKS or len(down_block_types) != len(block_out_channels): bad.append("blocks")
        for t in down_block_types:
            if t not in ("DownBlock2D", "CrossAttnDownBlock2D"): bad.append(t)
        for t in up_block_types:
            if t not in ("UpBlock2D", "CrossAttnUpBlock2D"): bad.append(t)
        if bad:
            raise ValueError(f"UNet2DConditionModel(b200): unsupported configuration: {bad}")
        self.sample_size = sample_size
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.config = _Cfg(
            sample_size=sample_size, in_channels=in_channels, out_channels=out_channels,
            down_block_types=tuple(down_block_types), mid_block_type=mid_block_type, up_block_types=tuple(up_block_types),
            block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
            cross_attention_dim=cross_attention_dim, attention_head_dim=attention_head_dim,
            norm_num_groups=norm_num_groups, norm_eps=norm_eps, _class_name="UNet2DConditionModel")
        self._init_engine(_unet_config(in_channels, out_channels, layers_per_block, block_out_channels, down_block_types,
                                       up_block_types, norm_num_groups, norm_eps, heads, cross_attention_dim), seed)

    def _encoding(self, enc: torch.Tensor, n: int, dev) -> torch.Tensor:
        if enc is None:
            raise ValueError("UNet2DConditionModel needs encoder_hidden_states (B, seq, cross_attention_dim)")
        e = enc.to(device=dev, dtype=torch.float32)
        if e.ndim == 2:
            e = e[:, None, :]
        if e.ndim != 3 or e.shape[0] != n or e.shape[2] != self.config.cross_attention_dim:
            raise ValueError(f"encoder_hidden_states must be ({n}, seq, {self.config.cross_attention_dim}), got {tuple(enc.shape)}")
        if not 1 <= e.shape[1] <= MAX_ENCODER_LEN:
            raise ValueError(f"UNet2DConditionModel(b200): encoder sequence length {e.shape[1]} outside [1, {MAX_ENCODER_LEN}]")
        return e.contiguous()

    def forward(self, sample: torch.Tensor, timestep, encoder_hidden_states: torch.Tensor = None, return_dict: bool = True):
        """ε = unet(sample, timestep, encoding)["sample"] — pipeline_audio_diffusion.py:161 (inference) and
        scripts/train_unet.py:255 (training: in train mode with grad enabled, backward() fills the parameter gradients)."""
        if self._needs_grad():
            if sample.requires_grad:
                raise NotImplementedError("UNet2DConditionModel(b200): gradients w.r.t. the input sample are not computed")
            if torch.is_tensor(encoder_hidden_states) and encoder_hidden_states.requires_grad:
                raise NotImplementedError("UNet2DConditionModel(b200): gradients w.r.t. encoder_hidden_states are not computed "
                                          "(pass precomputed encodings, e.g. .detach())")
        return self._forward(sample, timestep, encoder_hidden_states, return_dict)

    def forward_step(self, sample: torch.Tensor, timestep, coef: StepCoefC, encoder_hidden_states: torch.Tensor = None,
                     noise: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None, want_eps: bool = False):
        """Fused `scheduler.step(unet(sample, t, encoding), t, sample)["prev_sample"]` (pipeline_audio_diffusion.py:161-179)."""
        return self._forward_step(sample, timestep, coef, encoder_hidden_states, noise, out, want_eps)


def load_cond_unet(sub: str) -> UNet2DConditionModel:
    return UNet2DConditionModel.from_pretrained(sub)
