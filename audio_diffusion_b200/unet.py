"""`UNet2DModel` — drop-in for `diffusers.UNet2DModel` as the reference constructs and calls it
(scripts/train_unet.py:115-137; audiodiffusion/pipeline_audio_diffusion.py:118-126,160-163,237).

Same constructor kwargs, same state-dict key layout (SURVEY §8b) and the same call convention
`unet(sample, timestep)["sample"]`; the forward runs entirely in libb200ad.so (tcgen05 implicit-GEMM
convs, fused GroupNorm statistics, fused scheduler step).  PyTorch owns every tensor: parameters are
ordinary fp32 `nn.Parameter`s, the packed bf16 weights and the activation workspace are torch byte tensors.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, Optional, Sequence, Tuple, Union

import torch
from torch import nn

from . import _lib
from ._lib import MAX_BLOCKS, StepCoefC, UNetConfigC


class UNet2DOutput(dict):
    """Indexable by ["sample"] and attribute `.sample`, like diffusers' BaseOutput."""

    def __init__(self, sample):
        super().__init__(sample=sample)
        self.sample = sample


class _Cfg(dict):
    __getattr__ = dict.__getitem__


def _set_deep(root: nn.Module, dotted: str, p: nn.Parameter) -> None:
    parts = dotted.split(".")
    m = root
    for name in parts[:-1]:
        if name not in m._modules:
            m.add_module(name, nn.Module())
        m = m._modules[name]
    m.register_parameter(parts[-1], p)


class _UNetFunction(torch.autograd.Function):
    """Autograd node of the training forward: the backward pass is `b200ad_unet_backward` (all parameter gradients in one
    call); the gradient w.r.t. the input sample is not produced (the reference never needs it).  `enc` is the conditional
    model's encoding (None for UNet2DModel): the node keeps it alive and the backward binds it again, since the library
    reads it for the cross-attention weight gradients; no gradient w.r.t. it is produced."""

    @staticmethod
    def forward(ctx, model, x, t, enc, *params):
        out = model._forward_train(x, t, enc)
        ctx.model = model
        ctx.gen = model._fwd_gen         # the activations live in the model's single workspace: backward must see THIS forward
        ctx.save_for_backward(x, enc)
        return out

    @staticmethod
    def backward(ctx, g):
        x, enc = ctx.saved_tensors
        if ctx.gen != ctx.model._fwd_gen:
            raise _lib.B200ADError("UNet2DModel(b200): another forward ran on this model before backward(); the saved "
                                   "activations of this graph were overwritten (one forward per backward)")
        ctx.model._backward_train(x, g, enc)     # fills p.grad (views of the flat gradient buffer)
        return (None, None, None, None) + (None,) * len(ctx.model._pnames)


class UNet2DModel(nn.Module):
    def __init__(
        self,
        sample_size: Optional[Union[int, Tuple[int, int]]] = None,
        in_channels: int = 3,
        out_channels: int = 3,
        center_input_sample: bool = False,
        time_embedding_type: str = "positional",
        freq_shift: int = 0,
        flip_sin_to_cos: bool = True,
        down_block_types: Sequence[str] = ("DownBlock2D", "AttnDownBlock2D", "AttnDownBlock2D", "AttnDownBlock2D"),
        up_block_types: Sequence[str] = ("AttnUpBlock2D", "AttnUpBlock2D", "AttnUpBlock2D", "UpBlock2D"),
        block_out_channels: Sequence[int] = (224, 448, 672, 896),
        layers_per_block: int = 2,
        mid_block_scale_factor: float = 1,
        downsample_padding: int = 1,
        act_fn: str = "silu",
        attention_head_dim: Optional[int] = 8,
        norm_num_groups: int = 32,
        norm_eps: float = 1e-5,
        resnet_time_scale_shift: str = "default",
        add_attention: bool = True,
        downsample_type: str = "conv",
        upsample_type: str = "conv",
        dropout: float = 0.0,
        attn_norm_num_groups: Optional[int] = None,
        class_embed_type: Optional[str] = None,
        num_class_embeds: Optional[int] = None,
        num_train_timesteps: Optional[int] = None,
        seed: Optional[int] = None,
    ):
        super().__init__()
        unsupported = []
        if downsample_type != "conv" or upsample_type != "conv": unsupported.append("downsample_type/upsample_type")
        if dropout: unsupported.append("dropout")
        if attn_norm_num_groups is not None and attn_norm_num_groups != norm_num_groups: unsupported.append("attn_norm_num_groups")
        if class_embed_type is not None or num_class_embeds is not None: unsupported.append("class embedding")
        for ch in block_out_channels:     # GroupNorm statistics are accumulated per 4-channel quad (csrc/conv_tc.cu)
            if ch % norm_num_groups or (ch // norm_num_groups) % 4:
                unsupported.append(f"norm_num_groups={norm_num_groups} with {ch} channels (channels per group must be a multiple of 4)")
                break
        if center_input_sample: unsupported.append("center_input_sample")
        if time_embedding_type != "positional": unsupported.append("time_embedding_type")
        if freq_shift != 0 or not flip_sin_to_cos: unsupported.append("freq_shift/flip_sin_to_cos")
        if mid_block_scale_factor != 1 or downsample_padding != 1: unsupported.append("scale/padding")
        if act_fn != "silu" or resnet_time_scale_shift != "default" or not add_attention: unsupported.append("act/shift/attn")
        if len(block_out_channels) > MAX_BLOCKS: unsupported.append("too many blocks")
        for t in down_block_types:
            if t not in ("DownBlock2D", "AttnDownBlock2D"): unsupported.append(t)
        for t in up_block_types:
            if t not in ("UpBlock2D", "AttnUpBlock2D"): unsupported.append(t)
        if unsupported:
            raise ValueError(f"UNet2DModel(b200): unsupported configuration: {unsupported}")
        self.sample_size = sample_size
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.config = _Cfg(
            sample_size=sample_size, in_channels=in_channels, out_channels=out_channels,
            down_block_types=tuple(down_block_types), up_block_types=tuple(up_block_types),
            block_out_channels=tuple(block_out_channels), layers_per_block=layers_per_block,
            attention_head_dim=attention_head_dim, norm_num_groups=norm_num_groups, norm_eps=norm_eps,
            center_input_sample=center_input_sample, time_embedding_type=time_embedding_type, freq_shift=freq_shift,
            flip_sin_to_cos=flip_sin_to_cos, mid_block_scale_factor=mid_block_scale_factor,
            downsample_padding=downsample_padding, act_fn=act_fn, resnet_time_scale_shift=resnet_time_scale_shift,
            add_attention=add_attention, downsample_type=downsample_type, upsample_type=upsample_type, dropout=dropout,
            attn_norm_num_groups=attn_norm_num_groups, class_embed_type=class_embed_type,
            num_class_embeds=num_class_embeds, num_train_timesteps=num_train_timesteps, _class_name="UNet2DModel")

        c = UNetConfigC()
        c.in_channels, c.out_channels = in_channels, out_channels
        c.layers_per_block, c.num_blocks = layers_per_block, len(block_out_channels)
        for i, v in enumerate(block_out_channels):
            c.block_out_channels[i] = int(v)
            c.down_attn[i] = 1 if down_block_types[i] == "AttnDownBlock2D" else 0
            c.up_attn[i] = 1 if up_block_types[i] == "AttnUpBlock2D" else 0
        c.norm_num_groups, c.norm_eps = norm_num_groups, norm_eps
        c.attention_head_dim = attention_head_dim if attention_head_dim is not None else -1
        self._init_engine(c, seed)

    def _init_engine(self, c: UNetConfigC, seed: Optional[int]) -> None:
        """Create the library handle and the fp32 master parameters (table and naming come from the library)."""
        self._c = c
        L = _lib.lib()
        h = C.c_void_p()
        _lib.check(L.b200ad_unet_create(C.byref(c), C.byref(h)))
        self._h = h
        # parameter table comes from the library (diffusers naming); PyTorch default init
        g = torch.Generator().manual_seed(seed) if seed is not None else None
        self._pnames = []
        dims = (C.c_int64 * 4)()
        shapes: Dict[str, Tuple[int, ...]] = {}
        for i in range(L.b200ad_unet_num_params(h)):
            name = L.b200ad_unet_param_name(h, i).decode()
            nd = L.b200ad_unet_param_shape(h, i, dims)
            shapes[name] = tuple(int(dims[k]) for k in range(nd))
            self._pnames.append(name)
        for name in self._pnames:
            shape = shapes[name]
            leaf = name.rsplit(".", 2)[-2]
            is_norm = leaf.startswith("norm") or leaf == "group_norm" or leaf == "conv_norm_out"
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
        self._plist = None
        self._fwd_gen = 0                # bumped by every forward that writes the workspace

    # ------------------------------------------------------------------ diffusers ModelMixin persistence
    @classmethod
    def from_pretrained(cls, path: str, subfolder: Optional[str] = None, **_unused) -> "UNet2DModel":
        """`<path>/config.json` + `diffusion_pytorch_model.{safetensors,bin}`; older hub files' attention key names
        (query/key/value/proj_attn) are renamed on the way in."""
        import os
        from .hub_io import model_from_dir
        return model_from_dir(cls, os.path.join(path, subfolder) if subfolder else path)

    def save_pretrained(self, path: str, safe_serialization: bool = True, **_unused) -> None:
        from .hub_io import save_model
        save_model(self, path, safe_serialization=safe_serialization)

    # ------------------------------------------------------------------ engine plumbing
    def __del__(self):
        try:
            if getattr(self, "_h", None):
                _lib.lib().b200ad_unet_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def _named(self) -> Dict[str, nn.Parameter]:
        return dict(self.named_parameters())

    @property
    def device(self) -> torch.device:
        return next(self.parameters()).device

    def _ensure_bound(self, n: int, hh: int, ww: int) -> None:
        _lib.require_cuda()
        L = _lib.lib()
        if self._plist is None:            # Parameter objects are stable (module.to() swaps .data); resolve the names once
            named = self._named()
            self._plist = [named[k] for k in self._pnames]
        params = self._plist
        dev = params[0].device
        if dev.type != "cuda":
            raise _lib.B200ADError("UNet2DModel(b200): parameters must live on a CUDA device (call .to('cuda'))")
        for p in params:
            if p.dtype != torch.float32 or not p.is_contiguous():
                raise _lib.B200ADError("UNet2DModel(b200): parameters must be contiguous fp32 (master weights)")
        key = tuple((p.data_ptr(), p._version) for p in params)
        if self._packed is None or self._packed.device != dev:
            self._packed = torch.empty(L.b200ad_unet_packed_bytes(self._h), dtype=torch.uint8, device=dev)
            self._packed_key = None
            self._ws_key = None
        if key != self._packed_key:
            arr = (C.c_void_p * len(params))(*[p.data_ptr() for p in params])
            _lib.check(L.b200ad_unet_set_params(self._h, arr, self._packed.data_ptr(), self._packed.numel(),
                                                _lib.stream_ptr()))
            self._packed_key = key
            self._ws_key = None  # plan holds parameter pointers
        wkey = (n, hh, ww, dev)
        if wkey != self._ws_key:
            need = L.b200ad_unet_workspace_bytes(self._h, n, hh, ww)
            if self._ws is None or self._ws.numel() < need or self._ws.device != dev:
                self._ws = None
                self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
            _lib.check(L.b200ad_unet_bind_workspace(self._h, self._ws.data_ptr(), self._ws.numel(), n, hh, ww,
                                                    _lib.stream_ptr()))
            self._ws_key = wkey

    def _timesteps(self, timestep, n: int, dev) -> torch.Tensor:
        t = timestep
        if not torch.is_tensor(t):
            t = torch.tensor([t], dtype=torch.float32, device=dev)
        t = t.to(device=dev, dtype=torch.float32).reshape(-1)
        if t.numel() == 1:
            t = t.expand(n)
        if t.numel() != n:
            raise ValueError("timestep must be a scalar or have one entry per sample")
        return t.contiguous()

    def _check_input(self, sample: torch.Tensor) -> torch.Tensor:
        _lib.require_cuda()
        if sample.device.type != "cuda":
            raise _lib.B200ADError("UNet2DModel(b200): input must be a CUDA tensor (no CPU fallback)")
        return sample.to(torch.float32).contiguous()

    # ------------------------------------------------------------------ public call
    def forward(self, sample: torch.Tensor, timestep, return_dict: bool = True):
        """ε = unet(sample, timestep)["sample"] — pipeline_audio_diffusion.py:163."""
        if sample.requires_grad:
            raise NotImplementedError("UNet2DModel(b200): gradients w.r.t. the input sample are not computed")
        needs_grad = torch.is_grad_enabled() and self.training and any(p.requires_grad for p in self.parameters())
        x = self._check_input(sample)
        n, _, hh, ww = x.shape
        if needs_grad:      # training step (scripts/train_unet.py:257-259): forward keeps every activation, backward in CUDA
            t = self._timesteps(timestep, n, x.device)
            named = self._named()
            out = _UNetFunction.apply(self, x, t, None, *[named[k] for k in self._pnames])
            return UNet2DOutput(out) if return_dict else (out,)
        with torch.cuda.device(x.device):
            self._fwd_gen += 1
            self._set_training_mode(False)
            self._ensure_bound(n, hh, ww)
            t = self._timesteps(timestep, n, x.device)
            out = torch.empty((n, self.out_channels, hh, ww), dtype=torch.float32, device=x.device)
            _lib.check(_lib.lib().b200ad_unet_forward(self._h, x.data_ptr(), t.data_ptr(), out.data_ptr(),
                                                      _lib.stream_ptr()))
        if not return_dict:
            return (out,)
        return UNet2DOutput(out)

    # ------------------------------------------------------------------ training (backward in libb200ad)
    def _set_training_mode(self, on: bool) -> None:
        if getattr(self, "_train_mode", False) != on:
            _lib.check(_lib.lib().b200ad_unet_set_training(self._h, 1 if on else 0))
            self._train_mode = on
            self._ws_key = None        # the workspace layout differs (no buffer pooling when training)
            self._bwd_key = None

    def _forward_train(self, x: torch.Tensor, t: torch.Tensor, enc: Optional[torch.Tensor] = None) -> torch.Tensor:
        L = _lib.lib()
        n, _, hh, ww = x.shape
        with torch.cuda.device(x.device):
            self._fwd_gen += 1
            self._set_training_mode(True)
            self._ensure_bound(n, hh, ww)
            if getattr(self, "_bwd_key", None) != self._ws_key:
                nfl = L.b200ad_unet_grad_floats(self._h)
                if getattr(self, "_grad_flat", None) is None or self._grad_flat.numel() != nfl or self._grad_flat.device != x.device:
                    self._grad_flat = torch.zeros(nfl, dtype=torch.float32, device=x.device)
                need = L.b200ad_unet_backward_bytes(self._h)
                if need == 0:
                    _lib.check(-1)
                if getattr(self, "_bwd_arena", None) is None or self._bwd_arena.numel() < need or self._bwd_arena.device != x.device:
                    self._bwd_arena = None
                    self._bwd_arena = torch.empty(need, dtype=torch.uint8, device=x.device)
                _lib.check(L.b200ad_unet_bind_backward(self._h, self._bwd_arena.data_ptr(), self._bwd_arena.numel(),
                                                       self._grad_flat.data_ptr(), _lib.stream_ptr()))
                self._bwd_key = self._ws_key
            out = torch.empty((n, self.out_channels, hh, ww), dtype=torch.float32, device=x.device)
            if enc is not None:
                _lib.check(L.b200ad_unet_set_encoding(self._h, enc.data_ptr(), enc.shape[1]))
            _lib.check(L.b200ad_unet_forward(self._h, x.data_ptr(), t.data_ptr(), out.data_ptr(), _lib.stream_ptr()))
        return out

    def _backward_train(self, x: torch.Tensor, g: torch.Tensor, enc: Optional[torch.Tensor] = None):
        L = _lib.lib()
        g = g.to(torch.float32).contiguous()
        # torch semantics: gradients accumulate until they are zeroed. p.grad is None (zero_grad(set_to_none=True), the
        # default) -> start from zero; p.grad still our view (not zeroed, or zeroed in place) -> add to what is there.
        views = getattr(self, "_grad_views", None)
        params = [p for p in self.parameters() if p.requires_grad]
        have = [p.grad is not None for p in params]
        accumulate = bool(views) and all(have)
        if any(have) and not accumulate:
            raise _lib.B200ADError("UNet2DModel(b200): either all parameter gradients are set (accumulate) or none")
        with torch.cuda.device(x.device):
            if enc is not None:          # another call may have bound a different encoding since the forward
                _lib.check(L.b200ad_unet_set_encoding(self._h, enc.data_ptr(), enc.shape[1]))
            _lib.check(L.b200ad_unet_backward(self._h, x.data_ptr(), g.data_ptr(), 1 if accumulate else 0, _lib.stream_ptr()))
        if not getattr(self, "_no_sync", False):
            self._allreduce_gradients()
        # Parameter gradients are VIEWS of the flat buffer, assigned directly (no 700-tensor clone / accumulate pass).
        if getattr(self, "_grad_views_key", None) != self._grad_flat.data_ptr():
            named = self._named()
            self._grad_views = []
            for i, k in enumerate(self._pnames):
                off = L.b200ad_unet_grad_offset(self._h, i)
                p = named[k]
                self._grad_views.append((p, self._grad_flat[off:off + p.numel()].view(p.shape)))
            self._grad_views_key = self._grad_flat.data_ptr()
        for p, gv in self._grad_views:
            if p.grad is not None and p.grad.data_ptr() != gv.data_ptr():
                raise _lib.B200ADError("UNet2DModel(b200): p.grad must be None or the engine's own gradient view")
            p.grad = gv

    def _allreduce_gradients(self) -> None:
        """Data parallel (accelerate's DDP, scripts/train_unet.py:181): mean of the flat gradient buffer over the ranks, ONE
        collective after the backward pass.  It is not overlapped with the backward pass: an all-reduce in four buckets,
        each started as soon as the backward pass had written it, measured 53.1 ms per iteration at 2 GPUs (B200, before
        the port to H100) with or without the overlap - the backward kernels are persistent CTAs that fill every SM, so
        NCCL's CTAs only get SMs at kernel boundaries and the time they hold them is taken from the next kernel."""
        from .parallel import allreduce_mean_
        allreduce_mean_(self._grad_flat)

    def no_sync(self):
        """Like `DistributedDataParallel.no_sync()`: backward passes inside the context skip the gradient all-reduce, so
        micro-batches accumulate locally and the first backward outside it reduces the sum (`accelerator.accumulate`)."""
        import contextlib

        @contextlib.contextmanager
        def ctx():
            old = getattr(self, "_no_sync", False)
            self._no_sync = True
            try:
                yield
            finally:
                self._no_sync = old
        return ctx()

    @property
    def last_backward_launch_count(self) -> int:
        return _lib.lib().b200ad_unet_backward_launch_count(self._h)

    @torch.no_grad()
    def forward_step(self, sample: torch.Tensor, timestep, coef: StepCoefC, noise: Optional[torch.Tensor] = None,
                     out: Optional[torch.Tensor] = None, want_eps: bool = False):
        """Fused `scheduler.step(unet(sample, t), t, sample)["prev_sample"]` (pipeline_audio_diffusion.py:163-179)."""
        x = self._check_input(sample)
        n, _, hh, ww = x.shape
        with torch.cuda.device(x.device):
            self._fwd_gen += 1
            self._set_training_mode(False)
            self._ensure_bound(n, hh, ww)
            t = self._timesteps(timestep, n, x.device)
            if out is None:
                out = torch.empty_like(x)
            eps = torch.empty_like(x) if want_eps else None
            z = noise.to(torch.float32).contiguous() if noise is not None else None
            _lib.check(_lib.lib().b200ad_unet_forward_step(
                self._h, x.data_ptr(), t.data_ptr(), z.data_ptr() if z is not None else None, C.byref(coef),
                out.data_ptr(), eps.data_ptr() if eps is not None else None, _lib.stream_ptr()))
        return (out, eps) if want_eps else out

    def graph_stepper(self, sample: torch.Tensor) -> "GraphStepper":
        """CUDA-graph replay of `forward_step`: see `GraphStepper`.  The stepper owns its sample buffer (`stepper.x`, initialised
        from `sample`) and is cached per shape, so repeated pipeline calls re-use one captured graph as long as the model
        stays bound the same way (weights, batch, mode)."""
        x = self._check_input(sample)
        n, _, hh, ww = x.shape
        cache = self.__dict__.setdefault("_steppers", {})
        key = (tuple(x.shape), x.device)
        st = cache.get(key)
        if st is not None:
            with torch.cuda.device(x.device):
                self._set_training_mode(False)
                self._ensure_bound(n, hh, ww)
            if st._bound == (self._packed_key, self._ws_key):
                st.x.copy_(x)
                return st
        st = GraphStepper(self, x.clone())
        cache[key] = st
        return st

    def debug_tensor(self, name: str) -> torch.Tensor:
        """fp32 NCHW copy of a named internal activation of the last forward (parity tests)."""
        L = _lib.lib()
        dims = (C.c_int * 3)()
        _lib.check(min(0, L.b200ad_unet_debug_tensor(self._h, name.encode(), None, dims, _lib.stream_ptr())))
        n = self._ws_key[0]
        out = torch.empty((n, dims[0], dims[1], dims[2]), dtype=torch.float32, device=self.device)
        _lib.check(min(0, L.b200ad_unet_debug_tensor(self._h, name.encode(), out.data_ptr(), dims, _lib.stream_ptr())))
        return out

    def debug_grad(self, name: str, skip: bool = False) -> torch.Tensor:
        """fp32 NCHW copy of the last backward's gradient w.r.t. the activation `debug_tensor(name)` (skip=True: the share
        of it that the skip connection brought) (per-block backward tests)."""
        L = _lib.lib()
        dims = (C.c_int * 3)()
        _lib.check(min(0, L.b200ad_unet_debug_grad(self._h, name.encode(), int(skip), None, dims, _lib.stream_ptr())))
        n = self._ws_key[0]
        out = torch.empty((n, dims[0], dims[1], dims[2]), dtype=torch.float32, device=self.device)
        _lib.check(min(0, L.b200ad_unet_debug_grad(self._h, name.encode(), int(skip), out.data_ptr(), dims,
                                                   _lib.stream_ptr())))
        return out

    @property
    def last_launch_count(self) -> int:
        return _lib.lib().b200ad_unet_last_launch_count(self._h)


class GraphStepper:
    """The denoising loop's step as ONE `cudaGraphLaunch`: `x <- scheduler.step(unet(x, t), t, x)` with everything that changes
    from step to step (timestep, scheduler coefficients, noise) in fixed device buffers (`b200ad_unet_forward_step_dev`).

    Small batches are bound by the host, not by the GPU: at batch 1 and 256x256 the ~120 launches of a step take longer to
    enqueue than to execute (bench.py `configs.B1_latency`), which is the path the reference facade takes
    (audiodiffusion/__init__.py:59 hard-codes batch_size=1).  The kernels and their order are those of `forward_step`, so the
    results are bit-identical to the eager path (tests/test_gpu_pipeline.py::test_graph_stepper_equals_eager)."""

    def __init__(self, model: UNet2DModel, sample: torch.Tensor):
        if getattr(model, "is_conditional", False):
            raise NotImplementedError("GraphStepper: unconditional U-Net only")
        if sample.dtype != torch.float32 or not sample.is_contiguous() or sample.device.type != "cuda":
            raise ValueError("GraphStepper: the sample buffer must be a contiguous fp32 CUDA tensor (it is updated in place)")
        self.model, self.x = model, sample
        n, _, hh, ww = sample.shape
        dev = sample.device
        self.t = torch.zeros(n, dtype=torch.float32, device=dev)
        self.z = torch.zeros_like(sample)
        self.coef = torch.zeros(32, dtype=torch.uint8, device=dev)          # one b200ad_step_coef
        L = _lib.lib()
        with torch.cuda.device(dev), torch.no_grad():
            model._fwd_gen += 1
            model._set_training_mode(False)
            model._ensure_bound(n, hh, ww)
            scratch = torch.empty_like(sample)

            def enqueue(out):
                _lib.check(L.b200ad_unet_forward_step_dev(model._h, self.x.data_ptr(), self.t.data_ptr(), self.z.data_ptr(),
                                                          self.coef.data_ptr(), out.data_ptr(), _lib.stream_ptr()))
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                enqueue(scratch)             # warm-up outside the capture (function attributes, lazy module loading);
                enqueue(scratch)             # writes to a scratch tensor: the sample is untouched
            torch.cuda.current_stream(dev).wait_stream(side)
            torch.cuda.synchronize(dev)
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                enqueue(self.x)
            del scratch
        self._bound = (model._packed_key, model._ws_key)

    def step(self, timestep, coef: StepCoefC, noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        m = self.model
        if (m._packed_key, m._ws_key) != self._bound:
            raise _lib.B200ADError("GraphStepper: the model was re-bound (weights, batch or mode changed) after the capture")
        c = StepCoefC(coef.sqrt_1m_at, coef.inv_sqrt_at, coef.clip, coef.c_x0, coef.c_xt, coef.c_eps,
                      coef.c_z if noise is not None else 0.0, coef.do_clip)
        with torch.cuda.device(self.x.device):
            _lib.check(_lib.lib().b200ad_step_scalars_upload(C.byref(c), float(timestep), self.coef.data_ptr(), self.t.data_ptr(),
                                                             self.t.numel(), _lib.stream_ptr()))
        if noise is not None:
            self.z.copy_(noise)
        m._fwd_gen += 1
        self.graph.replay()
        return self.x
