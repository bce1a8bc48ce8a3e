"""`AutoencoderKL` — drop-in for `diffusers.AutoencoderKL` on the two calls the reference makes
(audiodiffusion/pipeline_audio_diffusion.py:143-147 `vqvae.encode(x).latent_dist.sample(generator=...)`,
:187-190 `vqvae.decode(z)["sample"]`; scripts/train_unet.py:99-104, :230-235), in the architecture of
config/ldm_autoencoder_kl.yaml:18-28 and with the state-dict keys audiodiffusion/utils.py:156-303
(`convert_ldm_to_hf_vae`) produces.

Encoder, decoder, quant/post-quant convs and the posterior sampling run in libb200ad.so (vae.cu); PyTorch owns the
parameters (fp32 `nn.Parameter`s), the packed bf16 weights and the activation workspace (engine.py).  No CPU fallback.

Training (scripts/train_vae.py): with grad enabled, the module in train() mode and a parameter requiring grad, `encode`
and `decode` are autograd nodes whose backward passes run in libb200ad.so (backward.cu); the posterior is then a torch
expression on the differentiable moments, so autograd carries the reparameterisation, the logvar clamp and `kl()`.
An image (encode) or latents (decode) that require grad get their gradient in train() or eval(): a frozen or eval()
autoencoder runs the backward without parameter gradients (a loss in pixel space behind a frozen decoder, latents
optimised against a target), and moving between that and parameter training re-plans the workspace.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import torch
from torch.autograd.function import once_differentiable

from . import _lib
from ._lib import MAX_BLOCKS, VAEConfigC
from .engine import EngineModel, _Cfg
from .hub_io import _OLD_ATTENTION_KEYS


class DecoderOutput(dict):
    def __init__(self, sample):
        super().__init__(sample=sample)
        self.sample = sample


def _run_part(vae, part: int, param_grads: bool, launch) -> None:
    """A part's backward: with parameter gradients through _backward_part (p.grad views), otherwise launch(0) alone."""
    if param_grads:
        vae._backward_part(part, launch)
    else:
        with torch.cuda.device(vae._bwd_arena.device):
            launch(0)


class _VAEEncodeFunction(torch.autograd.Function):
    """Autograd node of the encoder with a backward: x -> moments; the backward pass is
    `b200ad_vae_encoder_backward_input`: the encoder's and quant_conv's parameter gradients (param_grads; the params are
    the node's inputs) and, when x requires grad, the gradient w.r.t. the image."""

    @staticmethod
    def forward(ctx, vae, param_grads, x, *params):
        m = vae._encode_train(x, param_grads)
        ctx.vae = vae
        ctx.param_grads = param_grads
        ctx.nparams = len(params)
        ctx.gen = vae._fwd_gen[0]
        ctx.save_for_backward(x)
        return m

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        vae = ctx.vae
        vae._check_gen(0, ctx.gen)
        g = g.to(torch.float32).contiguous()
        gx = torch.empty_like(x) if ctx.needs_input_grad[2] else None
        _run_part(vae, 0, ctx.param_grads, lambda accumulate: _lib.check(vae._fn("encoder_backward_input")(
            vae._h, x.data_ptr(), g.data_ptr(), gx.data_ptr() if gx is not None else None, accumulate,
            _lib.stream_ptr())))
        return (None, None, gx) + (None,) * ctx.nparams


class _VAEDecodeFunction(torch.autograd.Function):
    """Autograd node of the decoder with a backward: z -> image; the backward pass is `b200ad_vae_decoder_backward`:
    the gradient w.r.t. z and (param_grads; the params are the node's inputs) the decoder's and post_quant_conv's
    parameter gradients."""

    @staticmethod
    def forward(ctx, vae, param_grads, z, *params):
        out = vae._decode_train(z, param_grads)
        ctx.vae = vae
        ctx.param_grads = param_grads
        ctx.nparams = len(params)
        ctx.gen = vae._fwd_gen[1]
        ctx.zshape = z.shape
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        vae = ctx.vae
        vae._check_gen(1, ctx.gen)
        g = g.to(torch.float32).contiguous()
        gz = torch.empty(ctx.zshape, dtype=torch.float32, device=g.device)
        _run_part(vae, 1, ctx.param_grads, lambda accumulate: _lib.check(vae._fn("decoder_backward")(
            vae._h, g.data_ptr(), gz.data_ptr(), accumulate, _lib.stream_ptr())))
        return (None, None, gz) + (None,) * ctx.nparams


class _NoBackward(torch.autograd.Function):
    """Marks an inference result computed while gradients were requested but training is not possible (the batch exceeds
    max_batch, or a configuration without a backward): the forward values are today's, and backward() raises."""

    @staticmethod
    def forward(ctx, reason, t, *params):
        ctx.reason = reason
        return t.clone()

    @staticmethod
    def backward(ctx, g):
        raise _lib.B200ADError(f"AutoencoderKL(b200): no backward for this call: {ctx.reason}")


class DiagonalGaussianDistribution:
    """Posterior returned by `encode(x).latent_dist`: `.sample(generator)`, `.mode()`, `.mean`, `.logvar`, `.std`, `.var`,
    `.kl()`.

    `sample()` draws its noise exactly as diffusers does (`randn_tensor(mean.shape, generator, device)`).  Inference: then
    mean + std * noise is evaluated by the encoder's tail kernel (vae_sample_kernel) — the moments never leave the device.
    Training: the moments are the encoder node's differentiable output and every method is a torch expression on them.
    """

    def __init__(self, vae: "AutoencoderKL", x: torch.Tensor, train: bool = False, refuse: Optional[str] = None,
                 param_grads: bool = True):
        self._vae = vae
        self._x = x
        self._train = train
        self._param_grads = param_grads
        self._refuse = refuse
        self._moments: Optional[torch.Tensor] = None

    def _run(self, noise: Optional[torch.Tensor]) -> torch.Tensor:
        z, m = self._vae._encode(self._x, noise)
        if self._refuse:
            z, m = self._vae._no_backward(self._refuse, z, self._x), self._vae._no_backward(self._refuse, m, self._x)
        self._moments = m
        return z

    @property
    def parameters(self) -> torch.Tensor:
        if self._moments is None:
            if self._train:
                pg = self._param_grads
                self._moments = _VAEEncodeFunction.apply(self._vae, pg, self._x, *(self._vae._plist if pg else ()))
            else:
                self._run(None)
        return self._moments

    @property
    def mean(self) -> torch.Tensor:
        return torch.chunk(self.parameters, 2, dim=1)[0]

    @property
    def logvar(self) -> torch.Tensor:
        return torch.clamp(torch.chunk(self.parameters, 2, dim=1)[1], -30.0, 20.0)

    @property
    def std(self) -> torch.Tensor:
        return torch.exp(0.5 * self.logvar)

    @property
    def var(self) -> torch.Tensor:
        return torch.exp(self.logvar)

    def sample(self, generator: Optional[torch.Generator] = None) -> torch.Tensor:
        x = self._x
        shape = self._vae.latent_shape(x.shape)
        gdev = generator.device if generator is not None else x.device
        noise = torch.randn(shape, generator=generator, device=gdev, dtype=torch.float32).to(x.device)
        if self._train:
            return self.mean + self.std * noise
        return self._run(noise)

    def mode(self) -> torch.Tensor:
        if self._train:
            return self.mean
        return self._run(None)

    def kl(self) -> torch.Tensor:
        """KL(q(z|x) || N(0, I)) per sample, summed over the latent ([3P-recall] diffusers 0.24 / ldm `posterior.kl()`)."""
        return 0.5 * torch.sum(torch.pow(self.mean, 2) + self.var - 1.0 - self.logvar, dim=[1, 2, 3])


class AutoencoderKLOutput(dict):
    def __init__(self, latent_dist):
        super().__init__(latent_dist=latent_dist)
        self.latent_dist = latent_dist


class AutoencoderKL(EngineModel):
    _prefix = "vae"
    _parts = (("encoder", ("encoder.", "quant_conv.")), ("decoder", ("decoder.", "post_quant_conv.")))
    # config.json keys handed to the constructor: a diffusers autoencoder's others (force_upcast, ...) are ignored
    _config_keys = ("in_channels", "out_channels", "down_block_types", "up_block_types", "block_out_channels",
                    "layers_per_block", "act_fn", "latent_channels", "norm_num_groups", "sample_size", "scaling_factor")

    def __init__(
        self,
        in_channels: int = 3,
        out_channels: int = 3,
        down_block_types: Sequence[str] = ("DownEncoderBlock2D",),
        up_block_types: Sequence[str] = ("UpDecoderBlock2D",),
        block_out_channels: Sequence[int] = (64,),
        layers_per_block: int = 1,
        act_fn: str = "silu",
        latent_channels: int = 4,
        norm_num_groups: int = 32,
        sample_size: int = 32,
        scaling_factor: float = 0.18215,
        max_batch: int = 16,
        seed: Optional[int] = None,
    ):
        super().__init__()
        bad = []
        if act_fn != "silu": bad.append("act_fn")
        if any(t != "DownEncoderBlock2D" for t in down_block_types): bad.append("down_block_types")
        if any(t != "UpDecoderBlock2D" for t in up_block_types): bad.append("up_block_types")
        if len(block_out_channels) > MAX_BLOCKS or len(down_block_types) != len(block_out_channels): bad.append("blocks")
        if bad:
            raise ValueError(f"AutoencoderKL(b200): unsupported configuration: {bad}")
        self.config = _Cfg(
            in_channels=in_channels, out_channels=out_channels, down_block_types=tuple(down_block_types),
            up_block_types=tuple(up_block_types), block_out_channels=tuple(block_out_channels),
            layers_per_block=layers_per_block, act_fn=act_fn, latent_channels=latent_channels,
            norm_num_groups=norm_num_groups, sample_size=sample_size, scaling_factor=scaling_factor,
            _class_name="AutoencoderKL")
        self.max_batch = int(max_batch)  # activations are bound for at most this many images; larger batches are chunked
        c = VAEConfigC()
        c.in_channels, c.out_channels, c.latent_channels = in_channels, out_channels, latent_channels
        c.layers_per_block, c.num_blocks = layers_per_block, len(block_out_channels)
        for i, v in enumerate(block_out_channels):
            c.block_out_channels[i] = int(v)
        c.norm_num_groups, c.norm_eps = norm_num_groups, 1e-6
        self._init_engine(c, seed)
        self._factor = 1 << (len(block_out_channels) - 1)

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        """Accepts the deprecated attention key names (`query/key/value/proj_attn`, possibly conv-shaped) that
        audiodiffusion/utils.py:33-60,120-129 still writes — diffusers converts them on load
        ([3P-recall] `_convert_deprecated_attention_blocks`)."""
        fixed = {}
        for k, v in state_dict.items():
            for a, b in _OLD_ATTENTION_KEYS.items():
                k = k.replace(a, b)
            if ".attentions." in k and k.endswith(".weight") and v.dim() > 2:
                v = v.reshape(v.shape[0], v.shape[1])
            fixed[k] = v
        return super().load_state_dict(fixed, strict=strict, **kw)

    def latent_shape(self, image_shape) -> Tuple[int, int, int, int]:
        n, _, hh, ww = image_shape
        return (n, self.config.latent_channels, hh // self._factor, ww // self._factor)

    def _check(self, x: torch.Tensor, channels: int, what: str) -> torch.Tensor:
        _lib.require_cuda()
        if x.device.type != "cuda":
            raise _lib.B200ADError(f"AutoencoderKL(b200): {what} must be a CUDA tensor (no CPU fallback)")
        if x.dim() != 4 or x.shape[1] != channels:
            raise ValueError(f"AutoencoderKL(b200): {what} must be (N, {channels}, H, W), got {tuple(x.shape)}")
        return x.to(torch.float32).contiguous()

    @torch.no_grad()
    def _encode(self, x: torch.Tensor, noise: Optional[torch.Tensor]):
        x = self._check(x, self.config.in_channels, "encode input")
        n, _, hh, ww = x.shape
        if hh % self._factor or ww % self._factor:
            raise ValueError(f"AutoencoderKL(b200): H and W must be multiples of {self._factor}")
        lshape = self.latent_shape(x.shape)
        z = torch.empty(lshape, dtype=torch.float32, device=x.device)
        m = torch.empty((n, 2 * lshape[1], lshape[2], lshape[3]), dtype=torch.float32, device=x.device)
        if noise is not None:
            noise = noise.to(device=x.device, dtype=torch.float32).contiguous()
            if tuple(noise.shape) != tuple(lshape):
                raise ValueError("noise must have the latent shape")
        with torch.cuda.device(x.device):
            for s in range(0, n, self.max_batch):
                e = min(n, s + self.max_batch)
                self._bind(e - s, hh, ww, False, x.device)
                _lib.check(self._fn("encode")(self._h, x[s:e].data_ptr(), noise[s:e].data_ptr() if noise is not None else None,
                                              z[s:e].data_ptr(), m[s:e].data_ptr(), _lib.stream_ptr()))
        return z, m

    # ------------------------------------------------------------------ training (backward in libb200ad)
    def _train_refusal(self, n: int) -> Optional[str]:
        """Why a call that requests gradients cannot train (it then runs the inference path and its backward raises)."""
        c = self.config
        if (c.in_channels, c.out_channels, c.latent_channels) != (1, 1, 1):
            return "the backward is implemented for in_channels = out_channels = latent_channels = 1"
        if n > self.max_batch:
            return (f"a training batch of {n} exceeds max_batch={self.max_batch} (training keeps the whole batch's "
                    "activations; raise max_batch)")
        return None

    def _no_backward(self, reason: str, t: torch.Tensor, inp: torch.Tensor) -> torch.Tensor:
        """t, marked as having no backward: it requires grad when the call's input `inp` or a parameter does."""
        return _NoBackward.apply(reason, t, inp, *self._plist)

    def _encode_train(self, x: torch.Tensor, param_grads: bool) -> torch.Tensor:
        n, _, hh, ww = x.shape
        if hh % self._factor or ww % self._factor:
            raise ValueError(f"AutoencoderKL(b200): H and W must be multiples of {self._factor}")
        lshape = self.latent_shape(x.shape)
        with torch.cuda.device(x.device):
            self._bind(n, hh, ww, True, x.device, param_grads=param_grads)
            self._fwd_gen[0] += 1
            z = torch.empty(lshape, dtype=torch.float32, device=x.device)
            m = torch.empty((n, 2 * lshape[1], lshape[2], lshape[3]), dtype=torch.float32, device=x.device)
            _lib.check(self._fn("encode")(self._h, x.data_ptr(), None, z.data_ptr(), m.data_ptr(), _lib.stream_ptr()))
        return m

    def _decode_train(self, z: torch.Tensor, param_grads: bool) -> torch.Tensor:
        z = z.detach().to(torch.float32).contiguous()
        n, _, lh, lw = z.shape
        hh, ww = lh * self._factor, lw * self._factor
        with torch.cuda.device(z.device):
            self._bind(n, hh, ww, True, z.device, param_grads=param_grads)
            self._fwd_gen[1] += 1
            out = torch.empty((n, self.config.out_channels, hh, ww), dtype=torch.float32, device=z.device)
            _lib.check(self._fn("decode")(self._h, z.data_ptr(), out.data_ptr(), _lib.stream_ptr()))
        return out

    @property
    def backward_launch_count(self) -> int:
        """The autoencoder's earlier name of `last_backward_launch_count`, kept for existing callers."""
        return self.last_backward_launch_count

    # ------------------------------------------------------------------ public calls
    def encode(self, x: torch.Tensor, return_dict: bool = True):
        """`vqvae.encode(x).latent_dist` — the encoder runs when the distribution is sampled / inspected.  Differentiable
        w.r.t. the parameters (train() mode) and w.r.t. an image that requires grad (train() or eval())."""
        x = self._check(x, self.config.in_channels, "encode input")
        param_grads = self._needs_grad()
        grad = param_grads or self._input_grad(x)
        refuse = self._train_refusal(x.shape[0]) if grad else None
        dist = DiagonalGaussianDistribution(self, x, train=grad and not refuse, refuse=refuse, param_grads=param_grads)
        if not return_dict:
            return (dist,)
        return AutoencoderKLOutput(dist)

    def decode(self, z: torch.Tensor, return_dict: bool = True):
        """`vqvae.decode(z)["sample"]` (pipeline_audio_diffusion.py:190).  Differentiable w.r.t. the parameters (train()
        mode) and w.r.t. latents that require grad (train() or eval())."""
        param_grads = self._needs_grad()
        grad = param_grads or self._input_grad(z)
        refuse = self._train_refusal(z.shape[0]) if grad else None
        if grad and not refuse:
            self._check(z, self.config.latent_channels, "latents")
            out = _VAEDecodeFunction.apply(self, param_grads, z, *(self._plist if param_grads else ()))
            return (out,) if not return_dict else DecoderOutput(out)
        with torch.no_grad():
            res = self._decode_infer(z, return_dict)
        if refuse:
            out = self._no_backward(refuse, res[0] if not return_dict else res.sample, z)
            return (out,) if not return_dict else DecoderOutput(out)
        return res

    def _decode_infer(self, z: torch.Tensor, return_dict: bool):
        z = self._check(z, self.config.latent_channels, "latents")
        n, _, lh, lw = z.shape
        hh, ww = lh * self._factor, lw * self._factor
        out = torch.empty((n, self.config.out_channels, hh, ww), dtype=torch.float32, device=z.device)
        with torch.cuda.device(z.device):
            for s in range(0, n, self.max_batch):
                e = min(n, s + self.max_batch)
                self._bind(e - s, hh, ww, False, z.device)
                _lib.check(self._fn("decode")(self._h, z[s:e].data_ptr(), out[s:e].data_ptr(), _lib.stream_ptr()))
        if not return_dict:
            return (out,)
        return DecoderOutput(out)

    def forward(self, sample: torch.Tensor, sample_posterior: bool = False, return_dict: bool = True,
                generator: Optional[torch.Generator] = None):
        post = self.encode(sample).latent_dist
        z = post.sample(generator=generator) if sample_posterior else post.mode()
        return self.decode(z, return_dict=return_dict)
