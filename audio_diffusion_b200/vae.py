"""`AutoencoderKL` — drop-in for `diffusers.AutoencoderKL` on the two calls the reference makes
(audiodiffusion/pipeline_audio_diffusion.py:143-147 `vqvae.encode(x).latent_dist.sample(generator=...)`,
:187-190 `vqvae.decode(z)["sample"]`; scripts/train_unet.py:99-104, :230-235), in the architecture of
config/ldm_autoencoder_kl.yaml:18-28 and with the state-dict keys audiodiffusion/utils.py:156-303
(`convert_ldm_to_hf_vae`) produces.

Encoder, decoder, quant/post-quant convs and the posterior sampling run in libb200ad.so (vae.cu); PyTorch owns the
parameters (fp32 `nn.Parameter`s), the packed bf16 weights and the activation workspace.  No CPU fallback.

Training (scripts/train_vae.py): with grad enabled, the module in train() mode and a parameter requiring grad, `encode`
and `decode` are autograd nodes whose backward passes run in libb200ad.so (unet_bwd.cu); the posterior is then a torch
expression on the differentiable moments, so autograd carries the reparameterisation, the logvar clamp and `kl()`.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, Optional, Sequence, Tuple

import torch
from torch import nn

from . import _lib
from ._lib import MAX_BLOCKS, VAEConfigC
from .unet import _Cfg, _set_deep


class DecoderOutput(dict):
    def __init__(self, sample):
        super().__init__(sample=sample)
        self.sample = sample


class _VAEEncodeFunction(torch.autograd.Function):
    """Autograd node of the training encoder: x -> moments; the backward pass is `b200ad_vae_encoder_backward` (the
    encoder's and quant_conv's parameter gradients).  No gradient w.r.t. the image is produced."""

    @staticmethod
    def forward(ctx, vae, x, *params):
        m = vae._encode_train(x)
        ctx.vae = vae
        ctx.gen = vae._fwd_gen[0]
        ctx.save_for_backward(x)
        return m

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        ctx.vae._check_gen(0, ctx.gen)
        ctx.vae._backward_part(0, x, g)
        return (None, None) + (None,) * len(ctx.vae._pnames)


class _VAEDecodeFunction(torch.autograd.Function):
    """Autograd node of the training decoder: z -> image; the backward pass is `b200ad_vae_decoder_backward` (the
    decoder's and post_quant_conv's parameter gradients, and the gradient w.r.t. z)."""

    @staticmethod
    def forward(ctx, vae, z, *params):
        out = vae._decode_train(z)
        ctx.vae = vae
        ctx.gen = vae._fwd_gen[1]
        ctx.zshape = z.shape
        return out

    @staticmethod
    def backward(ctx, g):
        ctx.vae._check_gen(1, ctx.gen)
        gz = ctx.vae._backward_part(1, None, g, ctx.zshape)
        return (None, gz) + (None,) * len(ctx.vae._pnames)


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

    def __init__(self, vae: "AutoencoderKL", x: torch.Tensor, train: bool = False, refuse: Optional[str] = None):
        self._vae = vae
        self._x = x
        self._train = train
        self._refuse = refuse
        self._moments: Optional[torch.Tensor] = None

    def _run(self, noise: Optional[torch.Tensor]) -> torch.Tensor:
        z, m = self._vae._encode(self._x, noise)
        if self._refuse:
            z, m = self._vae._no_backward(self._refuse, z), self._vae._no_backward(self._refuse, m)
        self._moments = m
        return z

    @property
    def parameters(self) -> torch.Tensor:
        if self._moments is None:
            if self._train:
                named = self._vae._named()
                self._moments = _VAEEncodeFunction.apply(self._vae, self._x, *[named[k] for k in self._vae._pnames])
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


class AutoencoderKL(nn.Module):
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
        self._c = c
        L = _lib.lib()
        h = C.c_void_p()
        _lib.check(L.b200ad_vae_create(C.byref(c), C.byref(h)))
        self._h = h
        self._factor = 1 << (len(block_out_channels) - 1)
        g = torch.Generator().manual_seed(seed) if seed is not None else None
        self._pnames = []
        dims = (C.c_int64 * 4)()
        shapes: Dict[str, Tuple[int, ...]] = {}
        for i in range(L.b200ad_vae_num_params(h)):
            name = L.b200ad_vae_param_name(h, i).decode()
            nd = L.b200ad_vae_param_shape(h, i, dims)
            shapes[name] = tuple(int(dims[k]) for k in range(nd))
            self._pnames.append(name)
        for name in self._pnames:
            shape = shapes[name]
            is_norm = (".norm" in name) or ("group_norm" in name) or ("conv_norm_out" in name)
            if is_norm:
                t = torch.ones(shape) if name.endswith(".weight") else torch.zeros(shape)
            else:
                wshape = shapes[name[: name.rfind(".")] + ".weight"]
                bound = 1.0 / math.sqrt(int(math.prod(wshape[1:])))
                t = (torch.rand(shape, generator=g) * 2 - 1) * bound
            _set_deep(self, name, nn.Parameter(t))
        self._packed = None
        self._packed_key = None
        self._ws = None
        self._ws_key = None
        self._train_mode = False
        self._fwd_gen = [0, 0]        # forwards run per part (encoder, decoder): a backward must see its own forward's
        self._bwd_key = None
        self._grad_flat = None
        self._bwd_arena = None
        self._grad_views = {}
        self._grad_views_key = None

    # ------------------------------------------------------------------ diffusers directory layout
    _KEEP = ("in_channels", "out_channels", "down_block_types", "up_block_types", "block_out_channels",
             "layers_per_block", "act_fn", "latent_channels", "norm_num_groups", "sample_size", "scaling_factor")

    @classmethod
    def from_pretrained(cls, path: str, subfolder: Optional[str] = None, **kw) -> "AutoencoderKL":
        """`AutoencoderKL.from_pretrained(dir)` (scripts/train_unet.py:99-104): config.json + diffusion_pytorch_model.*;
        raises EnvironmentError when the directory holds no model, which the reference catches to fall back to the
        pipeline's `vqvae` component."""
        import json
        import os
        sub = os.path.join(path, subfolder) if subfolder else path
        cfgp = os.path.join(sub, "config.json")
        if not os.path.exists(cfgp):
            raise EnvironmentError(f"{sub} does not contain an AutoencoderKL (config.json missing)")
        with open(cfgp) as f:
            cfg = json.load(f)
        model = cls(**{k: cfg[k] for k in cls._KEEP if k in cfg})
        st = os.path.join(sub, "diffusion_pytorch_model.safetensors")
        if os.path.exists(st):
            from safetensors.torch import load_file
            sd = load_file(st)
        else:
            sd = torch.load(os.path.join(sub, "diffusion_pytorch_model.bin"), map_location="cpu")
        ren = {".query.": ".to_q.", ".key.": ".to_k.", ".value.": ".to_v.", ".proj_attn.": ".to_out.0."}
        fixed = {}
        for k, v in sd.items():
            for a, b in ren.items():
                k = k.replace(a, b)
            if v.dim() == 4 and k.endswith(".weight") and (".to_" in k) and v.shape[2:] == (1, 1):
                v = v[:, :, 0, 0]  # ldm-converted attention projections are 1x1 convs (utils.py:285-303)
            fixed[k] = v.to(torch.float32)
        model.load_state_dict(fixed)
        return model

    _DEPRECATED = {".query.": ".to_q.", ".key.": ".to_k.", ".value.": ".to_v.", ".proj_attn.": ".to_out.0."}

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        """Accepts the deprecated attention key names (`query/key/value/proj_attn`, possibly conv-shaped) that
        audiodiffusion/utils.py:33-60,120-129 still writes — diffusers converts them on load
        ([3P-recall] `_convert_deprecated_attention_blocks`)."""
        fixed = {}
        for k, v in state_dict.items():
            for a, b in self._DEPRECATED.items():
                k = k.replace(a, b)
            if ".attentions." in k and k.endswith(".weight") and v.dim() > 2:
                v = v.reshape(v.shape[0], v.shape[1])
            fixed[k] = v
        return super().load_state_dict(fixed, strict=strict, **kw)

    def save_pretrained(self, path: str) -> None:
        import json
        import os
        os.makedirs(path, exist_ok=True)
        with open(os.path.join(path, "config.json"), "w") as f:
            json.dump({k: v for k, v in self.config.items()}, f, indent=2)
        from safetensors.torch import save_file
        save_file({k: v.detach().cpu().contiguous() for k, v in self.state_dict().items()},
                  os.path.join(path, "diffusion_pytorch_model.safetensors"))

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                _lib.lib().b200ad_vae_destroy(self._h)
                self._h = None
        except Exception:
            pass

    @property
    def device(self) -> torch.device:
        return next(self.parameters()).device

    def latent_shape(self, image_shape) -> Tuple[int, int, int, int]:
        n, _, hh, ww = image_shape
        return (n, self.config.latent_channels, hh // self._factor, ww // self._factor)

    # ------------------------------------------------------------------ engine plumbing
    def _ensure_bound(self, n: int, hh: int, ww: int) -> None:
        _lib.require_cuda()
        L = _lib.lib()
        named = dict(self.named_parameters())
        params = [named[k] for k in self._pnames]
        dev = params[0].device
        if dev.type != "cuda":
            raise _lib.B200ADError("AutoencoderKL(b200): parameters must live on a CUDA device (call .to('cuda'))")
        for p in params:
            if p.dtype != torch.float32 or not p.is_contiguous():
                raise _lib.B200ADError("AutoencoderKL(b200): parameters must be contiguous fp32")
        key = tuple((p.data_ptr(), p._version) for p in params)
        if self._packed is None or self._packed.device != dev:
            self._packed = torch.empty(L.b200ad_vae_packed_bytes(self._h), dtype=torch.uint8, device=dev)
            self._packed_key = None
            self._ws_key = None
        if key != self._packed_key:
            arr = (C.c_void_p * len(params))(*[p.data_ptr() for p in params])
            _lib.check(L.b200ad_vae_set_params(self._h, arr, self._packed.data_ptr(), self._packed.numel(),
                                               _lib.stream_ptr()))
            self._packed_key = key
            self._ws_key = None
        wkey = (n, hh, ww, dev)
        if wkey != self._ws_key:
            self._fwd_gen = [g + 1 for g in self._fwd_gen]     # the activations of both parts are gone
            need = L.b200ad_vae_workspace_bytes(self._h, n, hh, ww)
            if self._ws is None or self._ws.numel() < need or self._ws.device != dev:
                self._ws = None
                self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
            _lib.check(L.b200ad_vae_bind_workspace(self._h, self._ws.data_ptr(), self._ws.numel(), n, hh, ww,
                                                   _lib.stream_ptr()))
            self._ws_key = wkey

    def _check(self, x: torch.Tensor, channels: int, what: str) -> torch.Tensor:
        _lib.require_cuda()
        if x.device.type != "cuda":
            raise _lib.B200ADError(f"AutoencoderKL(b200): {what} must be a CUDA tensor (no CPU fallback)")
        if x.dim() != 4 or x.shape[1] != channels:
            raise ValueError(f"AutoencoderKL(b200): {what} must be (N, {channels}, H, W), got {tuple(x.shape)}")
        return x.to(torch.float32).contiguous()

    @torch.no_grad()
    def _encode(self, x: torch.Tensor, noise: Optional[torch.Tensor]):
        self._set_training_mode(False)
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
        L = _lib.lib()
        with torch.cuda.device(x.device):
            for s in range(0, n, self.max_batch):
                e = min(n, s + self.max_batch)
                self._ensure_bound(e - s, hh, ww)
                _lib.check(L.b200ad_vae_encode(self._h, x[s:e].data_ptr(),
                                               noise[s:e].data_ptr() if noise is not None else None,
                                               z[s:e].data_ptr(), m[s:e].data_ptr(), _lib.stream_ptr()))
        return z, m

    # ------------------------------------------------------------------ training (backward in libb200ad)
    def _needs_grad(self) -> bool:
        return torch.is_grad_enabled() and self.training and any(p.requires_grad for p in self.parameters())

    def _train_refusal(self, n: int) -> Optional[str]:
        """Why a call that requests gradients cannot train (it then runs the inference path and its backward raises)."""
        c = self.config
        if (c.in_channels, c.out_channels, c.latent_channels) != (1, 1, 1):
            return "the backward is implemented for in_channels = out_channels = latent_channels = 1"
        if n > self.max_batch:
            return (f"a training batch of {n} exceeds max_batch={self.max_batch} (training keeps the whole batch's "
                    "activations; raise max_batch)")
        return None

    def _no_backward(self, reason: str, t: torch.Tensor) -> torch.Tensor:
        named = self._named()
        return _NoBackward.apply(reason, t, *[named[k] for k in self._pnames])

    def _named(self) -> Dict[str, nn.Parameter]:
        return dict(self.named_parameters())

    def _set_training_mode(self, on: bool) -> None:
        if self._train_mode != on:
            _lib.check(_lib.lib().b200ad_vae_set_training(self._h, 1 if on else 0))
            self._train_mode = on
            self._ws_key = None        # the workspace layout differs (no buffer pooling when training)
            self._bwd_key = None

    def _check_gen(self, part: int, gen: int) -> None:
        if gen != self._fwd_gen[part]:
            what = ("encoder", "decoder")[part]
            raise _lib.B200ADError(f"AutoencoderKL(b200): another forward ran on the {what} before backward(); the saved "
                                   "activations of this graph were overwritten (one forward per backward)")

    def _bind_train(self, n: int, hh: int, ww: int, dev) -> None:
        if n > self.max_batch:
            raise ValueError(f"AutoencoderKL(b200): a training batch of {n} exceeds max_batch={self.max_batch} (training "
                             "keeps the whole batch's activations; raise max_batch)")
        L = _lib.lib()
        self._set_training_mode(True)
        self._ensure_bound(n, hh, ww)
        if self._bwd_key != self._ws_key:
            nfl = L.b200ad_vae_grad_floats(self._h)
            if self._grad_flat is None or self._grad_flat.numel() != nfl or self._grad_flat.device != dev:
                self._grad_flat = torch.zeros(nfl, dtype=torch.float32, device=dev)
            need = L.b200ad_vae_backward_bytes(self._h)
            if need == 0:
                _lib.check(-1)
            if self._bwd_arena is None or self._bwd_arena.numel() < need or self._bwd_arena.device != dev:
                self._bwd_arena = None
                self._bwd_arena = torch.empty(need, dtype=torch.uint8, device=dev)
            _lib.check(L.b200ad_vae_bind_backward(self._h, self._bwd_arena.data_ptr(), self._bwd_arena.numel(),
                                                  self._grad_flat.data_ptr(), _lib.stream_ptr()))
            self._bwd_key = self._ws_key

    def _encode_train(self, x: torch.Tensor) -> torch.Tensor:
        n, _, hh, ww = x.shape
        if hh % self._factor or ww % self._factor:
            raise ValueError(f"AutoencoderKL(b200): H and W must be multiples of {self._factor}")
        lshape = self.latent_shape(x.shape)
        with torch.cuda.device(x.device):
            self._bind_train(n, hh, ww, x.device)
            self._fwd_gen[0] += 1
            z = torch.empty(lshape, dtype=torch.float32, device=x.device)
            m = torch.empty((n, 2 * lshape[1], lshape[2], lshape[3]), dtype=torch.float32, device=x.device)
            _lib.check(_lib.lib().b200ad_vae_encode(self._h, x.data_ptr(), None, z.data_ptr(), m.data_ptr(),
                                                    _lib.stream_ptr()))
        return m

    def _decode_train(self, z: torch.Tensor) -> torch.Tensor:
        z = z.detach().to(torch.float32).contiguous()
        n, _, lh, lw = z.shape
        hh, ww = lh * self._factor, lw * self._factor
        with torch.cuda.device(z.device):
            self._bind_train(n, hh, ww, z.device)
            self._fwd_gen[1] += 1
            out = torch.empty((n, self.config.out_channels, hh, ww), dtype=torch.float32, device=z.device)
            _lib.check(_lib.lib().b200ad_vae_decode(self._h, z.data_ptr(), out.data_ptr(), _lib.stream_ptr()))
        return out

    def _backward_part(self, part: int, x: Optional[torch.Tensor], g: torch.Tensor, zshape=None):
        """Backward of the encoder (part 0, from dL/dmoments) or the decoder (part 1, from dL/dimage; returns dL/dz)."""
        L = _lib.lib()
        g = g.to(torch.float32).contiguous()
        named = self._named()
        if self._grad_views_key != self._grad_flat.data_ptr():
            self._grad_views = {0: [], 1: []}
            for i, k in enumerate(self._pnames):
                off = L.b200ad_vae_grad_offset(self._h, i)
                p = named[k]
                enc = k.startswith("encoder.") or k.startswith("quant_conv.")
                self._grad_views[0 if enc else 1].append((p, self._grad_flat[off:off + p.numel()].view(p.shape)))
            self._grad_views_key = self._grad_flat.data_ptr()
        views = self._grad_views[part]
        # torch semantics, per part: p.grad None -> start from zero; p.grad still our view -> add to what is there
        have = [p.grad is not None for p, _ in views if p.requires_grad]
        accumulate = bool(have) and all(have)
        if any(have) and not accumulate:
            raise _lib.B200ADError("AutoencoderKL(b200): either all of a part's parameter gradients are set (accumulate) "
                                   "or none")
        gz = None
        with torch.cuda.device(g.device):
            if part == 0:
                _lib.check(L.b200ad_vae_encoder_backward(self._h, x.data_ptr(), g.data_ptr(), 1 if accumulate else 0,
                                                         _lib.stream_ptr()))
            else:
                gz = torch.empty(zshape, dtype=torch.float32, device=g.device)
                _lib.check(L.b200ad_vae_decoder_backward(self._h, g.data_ptr(), gz.data_ptr(), 1 if accumulate else 0,
                                                         _lib.stream_ptr()))
        for p, gv in views:
            if p.grad is not None and p.grad.data_ptr() != gv.data_ptr():
                raise _lib.B200ADError("AutoencoderKL(b200): p.grad must be None or the engine's own gradient view")
            p.grad = gv
        return gz

    @property
    def backward_launch_count(self) -> int:
        """Kernel launches of the last decoder backward plus those of the last encoder backward."""
        return _lib.lib().b200ad_vae_backward_launch_count(self._h)

    # ------------------------------------------------------------------ public calls
    def encode(self, x: torch.Tensor, return_dict: bool = True):
        """`vqvae.encode(x).latent_dist` — the encoder runs when the distribution is sampled / inspected."""
        x = self._check(x, self.config.in_channels, "encode input")
        grad = self._needs_grad()
        refuse = self._train_refusal(x.shape[0]) if grad else None
        dist = DiagonalGaussianDistribution(self, x, train=grad and not refuse, refuse=refuse)
        if not return_dict:
            return (dist,)
        return AutoencoderKLOutput(dist)

    def decode(self, z: torch.Tensor, return_dict: bool = True):
        """`vqvae.decode(z)["sample"]` (pipeline_audio_diffusion.py:190)."""
        grad = self._needs_grad()
        refuse = self._train_refusal(z.shape[0]) if grad else None
        if grad and not refuse:
            self._check(z, self.config.latent_channels, "latents")
            named = self._named()
            out = _VAEDecodeFunction.apply(self, z, *[named[k] for k in self._pnames])
            return (out,) if not return_dict else DecoderOutput(out)
        with torch.no_grad():
            res = self._decode_infer(z, return_dict)
        if refuse:
            out = self._no_backward(refuse, res[0] if not return_dict else res.sample)
            return (out,) if not return_dict else DecoderOutput(out)
        return res

    def _decode_infer(self, z: torch.Tensor, return_dict: bool):
        self._set_training_mode(False)
        z = self._check(z, self.config.latent_channels, "latents")
        n, _, lh, lw = z.shape
        hh, ww = lh * self._factor, lw * self._factor
        out = torch.empty((n, self.config.out_channels, hh, ww), dtype=torch.float32, device=z.device)
        L = _lib.lib()
        with torch.cuda.device(z.device):
            for s in range(0, n, self.max_batch):
                e = min(n, s + self.max_batch)
                self._ensure_bound(e - s, hh, ww)
                _lib.check(L.b200ad_vae_decode(self._h, z[s:e].data_ptr(), out[s:e].data_ptr(), _lib.stream_ptr()))
        if not return_dict:
            return (out,)
        return DecoderOutput(out)

    def forward(self, sample: torch.Tensor, sample_posterior: bool = False, return_dict: bool = True,
                generator: Optional[torch.Generator] = None):
        post = self.encode(sample).latent_dist
        z = post.sample(generator=generator) if sample_posterior else post.mode()
        return self.decode(z, return_dict=return_dict)

    def debug_tensor(self, name: str) -> torch.Tensor:
        L = _lib.lib()
        dims = (C.c_int * 3)()
        _lib.check(min(0, L.b200ad_vae_debug_tensor(self._h, name.encode(), None, dims, _lib.stream_ptr())))
        n = self._ws_key[0]
        out = torch.empty((n, dims[0], dims[1], dims[2]), dtype=torch.float32, device=self.device)
        _lib.check(min(0, L.b200ad_vae_debug_tensor(self._h, name.encode(), out.data_ptr(), dims, _lib.stream_ptr())))
        return out

    def debug_grad(self, name: str, skip: bool = False) -> torch.Tensor:
        """fp32 NCHW copy of the last decoder / encoder backward's gradient w.r.t. the activation `debug_tensor(name)`
        (skip=True: the share of it a skip connection brought; the autoencoder has none) (per-block backward tests)."""
        L = _lib.lib()
        dims = (C.c_int * 3)()
        _lib.check(min(0, L.b200ad_vae_debug_grad(self._h, name.encode(), int(skip), None, dims, _lib.stream_ptr())))
        n = self._ws_key[0]
        out = torch.empty((n, dims[0], dims[1], dims[2]), dtype=torch.float32, device=self.device)
        _lib.check(min(0, L.b200ad_vae_debug_grad(self._h, name.encode(), int(skip), out.data_ptr(), dims,
                                                  _lib.stream_ptr())))
        return out

    @property
    def last_launch_count(self) -> int:
        return _lib.lib().b200ad_vae_last_launch_count(self._h)
