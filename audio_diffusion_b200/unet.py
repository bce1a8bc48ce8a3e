"""`UNet2DModel` — drop-in for `diffusers.UNet2DModel` as the reference constructs and calls it
(scripts/train_unet.py:115-137; audiodiffusion/pipeline_audio_diffusion.py:118-126,160-163,237).

Same constructor kwargs, same state-dict key layout (SURVEY §8b) and the same call convention
`unet(sample, timestep)["sample"]`; the forward runs entirely in libb200ad.so (wgmma implicit-GEMM convs, fused GroupNorm
statistics, fused scheduler step).  Training: with grad enabled and the module in train() mode, the forward is an autograd
node whose backward runs in libb200ad.so too (backward.cu).  A `sample` that requires grad gets its gradient in train()
or eval() (guidance, saliency); a frozen or eval() model then runs a backward without parameter gradients, and moving
between that and parameter training re-plans the workspace.  The engine plumbing is `EngineModel`'s (engine.py).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence, Tuple, Union

import torch
from torch.autograd.function import once_differentiable

from . import _lib
from ._lib import MAX_BLOCKS, MultistepCoefC, StepCoefC, UNetConfigC
from .engine import EngineModel, _Cfg


class UNet2DOutput(dict):
    """Indexable by ["sample"] and attribute `.sample`, like diffusers' BaseOutput."""

    def __init__(self, sample):
        super().__init__(sample=sample)
        self.sample = sample


def _unet_config(in_channels: int, out_channels: int, layers_per_block: int, block_out_channels: Sequence[int],
                 down_block_types: Sequence[str], up_block_types: Sequence[str], norm_num_groups: int, norm_eps: float,
                 attention_head_dim: int, cross_attention_dim: int = 0) -> UNetConfigC:
    c = UNetConfigC()
    c.in_channels, c.out_channels = in_channels, out_channels
    c.layers_per_block, c.num_blocks = layers_per_block, len(block_out_channels)
    for i, v in enumerate(block_out_channels):
        c.block_out_channels[i] = int(v)
        c.down_attn[i] = 1 if down_block_types[i] == "AttnDownBlock2D" else 0
        c.up_attn[i] = 1 if up_block_types[i] == "AttnUpBlock2D" else 0
        c.down_cross[i] = 1 if down_block_types[i] == "CrossAttnDownBlock2D" else 0
        c.up_cross[i] = 1 if up_block_types[i] == "CrossAttnUpBlock2D" else 0
    c.norm_num_groups, c.norm_eps = norm_num_groups, norm_eps
    c.attention_head_dim = attention_head_dim
    c.cross_attention_dim = cross_attention_dim
    return c


class _UNetFunction(torch.autograd.Function):
    """Autograd node of the forward with a backward: `b200ad_unet_backward_input`, which writes the gradient w.r.t. the
    sample when x requires grad.  param_grads: all parameter gradients in the same call (the params are the node's
    inputs); otherwise the data-gradient-only backward (no params, no flat buffer, no all-reduce).  `enc` is the
    conditional model's encoding (None for UNet2DModel): the node keeps it alive and the backward binds it again, since
    the library reads it for the cross-attention weight gradients; no gradient w.r.t. it is produced."""

    @staticmethod
    def forward(ctx, model, param_grads, x, t, enc, *params):
        out = model._run(x, t, enc, train=True, param_grads=param_grads)
        ctx.model = model
        ctx.param_grads = param_grads
        ctx.nparams = len(params)
        ctx.gen = model._fwd_gen[0]     # the activations live in the model's single workspace: backward must see THIS forward
        ctx.save_for_backward(x, enc)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, enc = ctx.saved_tensors
        m = ctx.model
        m._check_gen(0, ctx.gen)
        g = g.to(torch.float32).contiguous()
        gx = torch.empty_like(x) if ctx.needs_input_grad[2] else None

        def launch(accumulate):
            m._set_encoding(enc)      # another call may have bound a different encoding since the forward
            _lib.check(m._fn("backward_input")(m._h, x.data_ptr(), g.data_ptr(), gx.data_ptr() if gx is not None else None,
                                               accumulate, _lib.stream_ptr()))
            if ctx.param_grads and not m._no_sync:
                m._allreduce_gradients()
        if ctx.param_grads:
            m._backward_part(0, launch)     # fills p.grad (views of the flat gradient buffer)
        else:
            with torch.cuda.device(x.device):
                launch(0)
        return (None, None, gx, None, None) + (None,) * ctx.nparams


class UNet2DModel(EngineModel):
    _prefix = "unet"
    _no_sync = False

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
        self._init_engine(_unet_config(in_channels, out_channels, layers_per_block, block_out_channels, down_block_types,
                                       up_block_types, norm_num_groups, norm_eps,
                                       attention_head_dim if attention_head_dim is not None else -1), seed)

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
        """The sample as the library reads it; refuses one that is not (N, in_channels, H, W), whose planes conv_in
        would read past."""
        _lib.require_cuda()
        if sample.device.type != "cuda":
            raise self._err("input must be a CUDA tensor (no CPU fallback)")
        if sample.dim() != 4 or sample.shape[1] != self.in_channels:
            raise ValueError(f"{type(self).__name__}(b200): sample must be (N, {self.in_channels}, H, W), "
                             f"got {tuple(sample.shape)}")
        return sample.to(torch.float32).contiguous()

    def _check_step(self, x: torch.Tensor, name: str, t: Optional[torch.Tensor]) -> None:
        """Refuses a fused step the scheduler update cannot write in place of the sample: eps with other planes than the
        sample, or a noise / output tensor `t` (None: not given) of another shape, dtype, layout or device than x."""
        if self.out_channels != self.in_channels:
            raise ValueError(f"{type(self).__name__}(b200): a fused scheduler step needs out_channels == in_channels, "
                             f"got {self.out_channels} and {self.in_channels}")
        if t is not None and (t.shape != x.shape or t.device != x.device
                              or (name == "out" and (t.dtype != torch.float32 or not t.is_contiguous()))):
            raise ValueError(f"{type(self).__name__}(b200): {name} must be a {'contiguous fp32 ' if name == 'out' else ''}"
                             f"tensor of the sample's shape {tuple(x.shape)} on {x.device}, got {tuple(t.shape)} "
                             f"{t.dtype} on {t.device}")

    def _encoding(self, enc, n: int, dev) -> Optional[torch.Tensor]:
        """The conditional model's validated encoding; None here."""
        return None

    @staticmethod
    def _seq(enc: Optional[torch.Tensor]) -> Optional[int]:
        """The encoder sequence length the workspace is planned for (None: no encoding)."""
        return None if enc is None else int(enc.shape[1])

    def _set_encoding(self, enc: Optional[torch.Tensor]) -> None:
        if enc is not None:
            _lib.check(self._fn("set_encoding")(self._h, enc.data_ptr(), enc.shape[1]))

    # ------------------------------------------------------------------ public call
    def forward(self, sample: torch.Tensor, timestep, return_dict: bool = True):
        """ε = unet(sample, timestep)["sample"] — pipeline_audio_diffusion.py:163.  Differentiable w.r.t. the parameters
        (train() mode) and w.r.t. a `sample` that requires grad (train() or eval())."""
        return self._forward(sample, timestep, None, return_dict)

    def _forward(self, sample: torch.Tensor, timestep, enc, return_dict: bool):
        x = self._check_input(sample)
        param_grads = self._needs_grad()
        if param_grads or self._input_grad(x):    # a training step (scripts/train_unet.py:257-259) and / or a sample
            n = x.shape[0]                          # gradient: the forward keeps every activation
            t, e = self._timesteps(timestep, n, x.device), self._encoding(enc, n, x.device)
            out = _UNetFunction.apply(self, param_grads, x, t, e, *(self._plist if param_grads else ()))
        else:
            out = self._run(x, timestep, enc, train=False)
        return UNet2DOutput(out) if return_dict else (out,)

    def _run(self, x: torch.Tensor, timestep, enc, train: bool, param_grads: bool = True) -> torch.Tensor:
        """One forward into a new output tensor; timestep and encoding are converted after binding (already converted
        ones, as the training node passes them, are left as they are)."""
        n, _, hh, ww = x.shape
        with torch.cuda.device(x.device):
            self._fwd_gen[0] += 1
            e = self._encoding(enc, n, x.device)
            self._bind(n, hh, ww, train, x.device, self._seq(e), param_grads)
            t = self._timesteps(timestep, n, x.device)
            out = torch.empty((n, self.out_channels, hh, ww), dtype=torch.float32, device=x.device)
            self._set_encoding(e)
            _lib.check(self._fn("forward")(self._h, x.data_ptr(), t.data_ptr(), out.data_ptr(), _lib.stream_ptr()))
        return out

    # ------------------------------------------------------------------ data parallel
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
            old = self._no_sync
            self._no_sync = True
            try:
                yield
            finally:
                self._no_sync = old
        return ctx()

    # ------------------------------------------------------------------ sampling
    def forward_step(self, sample: torch.Tensor, timestep, coef: Union[StepCoefC, MultistepCoefC],
                     noise: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None, want_eps: bool = False,
                     history: Optional[torch.Tensor] = None):
        """Fused `scheduler.step(unet(sample, t), t, sample)["prev_sample"]` (pipeline_audio_diffusion.py:163-179).  A multistep
        scheduler (`DPMSolverMultistepScheduler.step_coef` gives `MultistepCoefC`) also passes `history`: fp32 (k, *sample.shape),
        k = 1 or 2, the x0 of the previous k steps, which the step reads and rotates in place (zero-filled at the start)."""
        return self._forward_step(sample, timestep, coef, None, noise, out, want_eps, history)

    def _check_history(self, x: torch.Tensor, coef, history: Optional[torch.Tensor]) -> int:
        """Number of history planes the step reads; refuses a history the coefficients do not match."""
        multi = isinstance(coef, MultistepCoefC)
        if history is None:
            if multi and (coef.c_h1 != 0.0 or coef.c_h2 != 0.0):
                raise ValueError(f"{type(self).__name__}(b200): multistep coefficients need a history tensor")
            return 0
        if not multi:
            raise ValueError(f"{type(self).__name__}(b200): a history tensor needs multistep coefficients (MultistepCoefC)")
        if (history.dim() != 5 or history.shape[0] not in (1, 2) or history.shape[1:] != x.shape
                or history.dtype != torch.float32 or not history.is_contiguous() or history.device != x.device):
            raise ValueError(f"{type(self).__name__}(b200): history must be a contiguous fp32 tensor (k, "
                             f"{', '.join(map(str, x.shape))}) with k in (1, 2) on {x.device}, got {tuple(history.shape)} "
                             f"{history.dtype} on {history.device}")
        if history.shape[0] == 1 and coef.c_h2 != 0.0:
            raise ValueError(f"{type(self).__name__}(b200): a third-order step needs two history planes")
        return history.shape[0]

    @torch.no_grad()
    def _forward_step(self, sample: torch.Tensor, timestep, coef, enc, noise: Optional[torch.Tensor],
                      out: Optional[torch.Tensor], want_eps: bool, history: Optional[torch.Tensor] = None):
        x = self._check_input(sample)
        self._check_step(x, "noise", noise)
        self._check_step(x, "out", out)
        k = self._check_history(x, coef, history)
        n, _, hh, ww = x.shape
        with torch.cuda.device(x.device):
            self._fwd_gen[0] += 1
            e = self._encoding(enc, n, x.device)
            self._bind(n, hh, ww, False, x.device, self._seq(e))
            t = self._timesteps(timestep, n, x.device)
            if out is None:
                out = torch.empty_like(x)
            eps = torch.empty_like(x) if want_eps else None
            z = noise.to(torch.float32).contiguous() if noise is not None else None
            self._set_encoding(e)
            zp, ep = z.data_ptr() if z is not None else None, eps.data_ptr() if eps is not None else None
            if isinstance(coef, MultistepCoefC):
                h1 = history[0].data_ptr() if k >= 1 else None
                h2 = history[1].data_ptr() if k == 2 else None
                _lib.check(self._fn("forward_multistep")(self._h, x.data_ptr(), t.data_ptr(), zp, C.byref(coef), h1, h2, out.data_ptr(),
                                                         ep, _lib.stream_ptr()))
            else:
                _lib.check(self._fn("forward_step")(self._h, x.data_ptr(), t.data_ptr(), zp, C.byref(coef), out.data_ptr(),
                                                    ep, _lib.stream_ptr()))
        return (out, eps) if want_eps else out

    def graph_stepper(self, sample: torch.Tensor, history: Optional[int] = None) -> "GraphStepper":
        """CUDA-graph replay of `forward_step`: see `GraphStepper`.  The stepper owns its sample buffer (`stepper.x`, initialised
        from `sample`) and is cached per shape and kind, so repeated pipeline calls re-use one captured graph as long as the
        model stays bound the same way (weights, batch, mode).  `history`: None for DDPM / DDIM coefficients (`StepCoefC`),
        else the number of history planes (0-2) of a multistep scheduler's steps (`MultistepCoefC`); they start zeroed."""
        x = self._check_input(sample)
        self._check_step(x, "sample", None)
        if history not in (None, 0, 1, 2):
            raise ValueError(f"graph_stepper: history must be None, 0, 1 or 2, got {history!r}")
        n, _, hh, ww = x.shape
        cache = self.__dict__.setdefault("_steppers", {})
        key = (tuple(x.shape), x.device, history)
        st = cache.get(key)
        if st is not None:
            with torch.cuda.device(x.device):
                self._bind(n, hh, ww, False, x.device)
            if st._bound == (self._packed_key, self._ws_key):
                st.x.copy_(x)
                if st.hist is not None:
                    st.hist.zero_()
                return st
        st = GraphStepper(self, x.clone(), history)
        cache[key] = st
        return st


class GraphStepper:
    """The denoising loop's step as ONE `cudaGraphLaunch`: `x <- scheduler.step(unet(x, t), t, x)` with everything that changes
    from step to step (timestep, scheduler coefficients, noise) in fixed device buffers (`b200ad_unet_forward_step_dev`, or
    `b200ad_unet_forward_multistep_dev` with the history buffers `hist` of a multistep scheduler).

    Small batches are bound by the host, not by the GPU: at batch 1 and 256x256 the ~120 launches of a step take longer to
    enqueue than to execute (bench.py `configs.B1_latency`), which is the path the reference facade takes
    (audiodiffusion/__init__.py:59 hard-codes batch_size=1).  The kernels and their order are those of `forward_step`, so the
    results are bit-identical to the eager path (tests/test_gpu_pipeline.py::test_graph_stepper_equals_eager)."""

    def __init__(self, model: UNet2DModel, sample: torch.Tensor, history: Optional[int] = None):
        if getattr(model, "is_conditional", False):
            raise NotImplementedError("GraphStepper: unconditional U-Net only")
        if sample.dtype != torch.float32 or not sample.is_contiguous() or sample.device.type != "cuda":
            raise ValueError("GraphStepper: the sample buffer must be a contiguous fp32 CUDA tensor (it is updated in place)")
        self.model, self.x = model, sample
        self.multistep = history is not None
        n, _, hh, ww = sample.shape
        dev = sample.device
        self.t = torch.zeros(n, dtype=torch.float32, device=dev)
        self.z = torch.zeros_like(sample)
        ctype = MultistepCoefC if self.multistep else StepCoefC
        self.coef = torch.zeros(C.sizeof(ctype), dtype=torch.uint8, device=dev)    # one b200ad_(multi)step_coef
        self.hist = torch.zeros((history,) + tuple(sample.shape), dtype=torch.float32, device=dev) if history else None
        h1 = self.hist[0].data_ptr() if history else None
        h2 = self.hist[1].data_ptr() if history == 2 else None
        L = _lib.lib()
        with torch.cuda.device(dev), torch.no_grad():
            model._fwd_gen[0] += 1
            model._bind(n, hh, ww, False, dev)
            scratch = torch.empty_like(sample)
            scratch_hist = torch.zeros_like(self.hist) if history else None

            def enqueue(out, hist1, hist2):
                if self.multistep:
                    _lib.check(L.b200ad_unet_forward_multistep_dev(model._h, self.x.data_ptr(), self.t.data_ptr(),
                                                                   self.z.data_ptr(), self.coef.data_ptr(), hist1, hist2,
                                                                   out.data_ptr(), _lib.stream_ptr()))
                else:
                    _lib.check(L.b200ad_unet_forward_step_dev(model._h, self.x.data_ptr(), self.t.data_ptr(), self.z.data_ptr(),
                                                              self.coef.data_ptr(), out.data_ptr(), _lib.stream_ptr()))
            sh1 = scratch_hist[0].data_ptr() if history else None
            sh2 = scratch_hist[1].data_ptr() if history == 2 else None
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                enqueue(scratch, sh1, sh2)   # warm-up outside the capture (function attributes, lazy module loading);
                enqueue(scratch, sh1, sh2)   # writes to scratch tensors: the sample and the history are untouched
            torch.cuda.current_stream(dev).wait_stream(side)
            torch.cuda.synchronize(dev)
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                enqueue(self.x, h1, h2)
            del scratch, scratch_hist
        self._bound = (model._packed_key, model._ws_key)

    def step(self, timestep, coef: Union[StepCoefC, MultistepCoefC], noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        m = self.model
        if (m._packed_key, m._ws_key) != self._bound:
            raise _lib.B200ADError("GraphStepper: the model was re-bound (weights, batch or mode changed) after the capture")
        if isinstance(coef, MultistepCoefC) != self.multistep:
            raise ValueError(f"GraphStepper: captured for {'MultistepCoefC' if self.multistep else 'StepCoefC'} coefficients, "
                             f"got {type(coef).__name__}")
        if noise is not None and noise.shape != self.x.shape:     # copy_ would broadcast it
            raise ValueError(f"GraphStepper: noise must have the sample's shape {tuple(self.x.shape)}, "
                             f"got {tuple(noise.shape)}")
        if self.multistep:
            k = 0 if self.hist is None else self.hist.shape[0]
            if (k < 1 and coef.c_h1 != 0.0) or (k < 2 and coef.c_h2 != 0.0):
                raise ValueError(f"GraphStepper: captured with {k} history planes, the coefficients need more")
            s = coef.step
            c = MultistepCoefC(StepCoefC(s.sqrt_1m_at, s.inv_sqrt_at, s.clip, s.c_x0, s.c_xt, s.c_eps,
                                         s.c_z if noise is not None else 0.0, s.do_clip), coef.c_h1, coef.c_h2)
            upload = _lib.lib().b200ad_multistep_scalars_upload
        else:
            c = StepCoefC(coef.sqrt_1m_at, coef.inv_sqrt_at, coef.clip, coef.c_x0, coef.c_xt, coef.c_eps,
                          coef.c_z if noise is not None else 0.0, coef.do_clip)
            upload = _lib.lib().b200ad_step_scalars_upload
        with torch.cuda.device(self.x.device):
            _lib.check(upload(C.byref(c), float(timestep), self.coef.data_ptr(), self.t.data_ptr(), self.t.numel(),
                              _lib.stream_ptr()))
        if noise is not None:
            self.z.copy_(noise)
        m._fwd_gen[0] += 1
        self.graph.replay()
        return self.x
