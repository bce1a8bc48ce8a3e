"""`EngineModel` — the `nn.Module` base of the models whose forward and backward run in libb200ad.so (`UNet2DModel`,
`AutoencoderKL`).  It drives a library handle `b200ad_<prefix>_*` through the protocol both models share: the parameter
table and its default initialisation, weight packing, the activation workspace, training mode, the backward arena with one
flat gradient buffer handed out as `p.grad` views, the one-forward-per-backward guard, debug read-outs and the diffusers
hub directory layout.  PyTorch owns every tensor: parameters are ordinary fp32 `nn.Parameter`s, the packed bf16 weights,
the workspace and the backward arena are torch byte tensors.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from typing import Callable, Dict, Optional, Sequence, Tuple, Union

import torch
from torch import nn

from . import _lib
from .hub_io import model_from_dir, save_model


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


def _is_norm(name: str) -> bool:
    """GroupNorm / LayerNorm affine parameters (`...norm1.weight`, `...group_norm.bias`, `conv_norm_out.weight`, ...)."""
    leaf = name.rsplit(".", 2)[-2]
    return leaf.startswith("norm") or leaf == "group_norm" or leaf == "conv_norm_out"


class EngineModel(nn.Module):
    _prefix = ""         # library symbols: b200ad_<prefix>_<fn>
    # backward parts: (name, parameter-name prefixes); each part's backward fills the gradients of its own parameters
    _parts: Tuple[Tuple[str, Union[str, Tuple[str, ...]]], ...] = (("model", ""),)
    _config_keys: Optional[Sequence[str]] = None    # config.json keys from_pretrained hands to the constructor (None: all)

    def _fn(self, name: str):
        return getattr(_lib.lib(), f"b200ad_{self._prefix}_{name}")

    def _init_engine(self, c: C.Structure, seed: Optional[int]) -> None:
        """Create the library handle and the fp32 master parameters (table and naming come from the library; PyTorch's
        default initialisation: norms 1 / 0, everything else uniform in +-1/sqrt(fan_in) of its layer's weight)."""
        self._c = c
        h = C.c_void_p()
        _lib.check(self._fn("create")(C.byref(c), C.byref(h)))
        self._h = h
        g = torch.Generator().manual_seed(seed) if seed is not None else None
        dims = (C.c_int64 * 4)()
        shapes: Dict[str, Tuple[int, ...]] = {}
        for i in range(self._fn("num_params")(h)):
            name = self._fn("param_name")(h, i).decode()
            nd = self._fn("param_shape")(h, i, dims)
            shapes[name] = tuple(int(dims[k]) for k in range(nd))
        self._pnames = list(shapes)
        for name, shape in shapes.items():
            if _is_norm(name):
                t = torch.ones(shape) if name.endswith(".weight") else torch.zeros(shape)
            else:
                wshape = shapes[name[: name.rfind(".")] + ".weight"]
                bound = 1.0 / math.sqrt(int(math.prod(wshape[1:])))
                t = (torch.rand(shape, generator=g) * 2 - 1) * bound
            _set_deep(self, name, nn.Parameter(t))
        named = dict(self.named_parameters())
        self._plist = [named[k] for k in self._pnames]   # Parameter objects are stable (module.to() swaps .data)
        self._packed = self._packed_key = None
        self._ws = self._ws_key = None
        self._train_mode = False
        self._fwd_gen = [0] * len(self._parts)   # forwards per part: a backward must see its own forward's activations
        self._bwd_key = None
        self._grad_flat = self._bwd_arena = None
        self._grad_views, self._grad_views_key = None, None

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self._fn("destroy")(self._h)
                self._h = None
        except Exception:
            pass

    # ------------------------------------------------------------------ diffusers ModelMixin persistence
    @classmethod
    def from_pretrained(cls, path: str, subfolder: Optional[str] = None, **_unused):
        """`<path>/config.json` + `diffusion_pytorch_model.{safetensors,bin}`; older hub files' attention key names
        (query/key/value/proj_attn) are renamed on the way in.  Raises EnvironmentError when the directory holds no
        config.json."""
        return model_from_dir(cls, os.path.join(path, subfolder) if subfolder else path, keep=cls._config_keys)

    def save_pretrained(self, path: str, safe_serialization: bool = True, **_unused) -> None:
        save_model(self, path, safe_serialization=safe_serialization)

    # ------------------------------------------------------------------ engine plumbing
    @property
    def device(self) -> torch.device:
        return next(self.parameters()).device

    def _err(self, msg: str) -> _lib.B200ADError:
        return _lib.B200ADError(f"{type(self).__name__}(b200): {msg}")

    def _needs_grad(self) -> bool:
        return torch.is_grad_enabled() and self.training and any(p.requires_grad for p in self.parameters())

    def _ensure_bound(self, n: int, hh: int, ww: int, seq: Optional[int] = None) -> None:
        """Packs the weights when a parameter's pointer or version changed, and binds the workspace for (n, hh, ww) and,
        for a conditional U-Net, the encoder sequence length `seq` (None: a model without an encoding)."""
        _lib.require_cuda()
        params = self._plist
        dev = params[0].device
        if dev.type != "cuda":
            raise self._err("parameters must live on a CUDA device (call .to('cuda'))")
        for p in params:
            if p.dtype != torch.float32 or not p.is_contiguous():
                raise self._err("parameters must be contiguous fp32 (master weights)")
        key = tuple((p.data_ptr(), p._version) for p in params)
        if self._packed is None or self._packed.device != dev:
            self._packed = torch.empty(self._fn("packed_bytes")(self._h), dtype=torch.uint8, device=dev)
            self._packed_key = None
            self._ws_key = None
        if key != self._packed_key:
            arr = (C.c_void_p * len(params))(*[p.data_ptr() for p in params])
            _lib.check(self._fn("set_params")(self._h, arr, self._packed.data_ptr(), self._packed.numel(),
                                              _lib.stream_ptr()))
            self._packed_key = key
            self._ws_key = None  # the plan holds parameter pointers
        wkey = (n, hh, ww, dev) if seq is None else (n, hh, ww, dev, seq)
        if wkey != self._ws_key:
            self._fwd_gen = [g + 1 for g in self._fwd_gen]     # the activations of every part are gone
            if seq is not None:
                _lib.check(self._fn("set_encoder_len")(self._h, seq))
            need = self._fn("workspace_bytes")(self._h, n, hh, ww)
            if self._ws is None or self._ws.numel() < need or self._ws.device != dev:
                self._ws = None
                self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
            _lib.check(self._fn("bind_workspace")(self._h, self._ws.data_ptr(), self._ws.numel(), n, hh, ww,
                                                  _lib.stream_ptr()))
            self._ws_key = wkey

    def _set_training_mode(self, on: bool) -> None:
        if self._train_mode != on:
            _lib.check(self._fn("set_training")(self._h, 1 if on else 0))
            self._train_mode = on
            self._ws_key = None        # the workspace layout differs (no buffer pooling when training)
            self._bwd_key = None

    def _bind_backward(self, dev: torch.device) -> None:
        """The backward arena and the flat gradient buffer, (re)bound whenever the workspace was."""
        if self._bwd_key == self._ws_key:
            return
        nfl = self._fn("grad_floats")(self._h)
        if self._grad_flat is None or self._grad_flat.numel() != nfl or self._grad_flat.device != dev:
            self._grad_flat = torch.zeros(nfl, dtype=torch.float32, device=dev)
        need = self._fn("backward_bytes")(self._h)
        if need == 0:
            _lib.check(-1)
        if self._bwd_arena is None or self._bwd_arena.numel() < need or self._bwd_arena.device != dev:
            self._bwd_arena = None
            self._bwd_arena = torch.empty(need, dtype=torch.uint8, device=dev)
        _lib.check(self._fn("bind_backward")(self._h, self._bwd_arena.data_ptr(), self._bwd_arena.numel(),
                                             self._grad_flat.data_ptr(), _lib.stream_ptr()))
        self._bwd_key = self._ws_key

    def _bind(self, n: int, hh: int, ww: int, train: bool, dev: torch.device, seq: Optional[int] = None) -> None:
        """Everything a forward of (n, hh, ww) (and `seq` encoder tokens) needs bound: mode, weights, workspace and, when
        training, the backward."""
        self._set_training_mode(train)
        self._ensure_bound(n, hh, ww, seq)
        if train:
            self._bind_backward(dev)

    # ------------------------------------------------------------------ backward parts
    def _check_gen(self, part: int, gen: int) -> None:
        if gen != self._fwd_gen[part]:
            raise self._err(f"another forward ran on the {self._parts[part][0]} before backward(); the saved activations "
                            "of this graph were overwritten (one forward per backward)")

    def _part_views(self, part: int):
        """(parameter, view of its slot in the flat gradient buffer) for every parameter of `part`."""
        if self._grad_views_key != self._grad_flat.data_ptr():
            offset = self._fn("grad_offset")
            self._grad_views = [[] for _ in self._parts]
            for i, (k, p) in enumerate(zip(self._pnames, self._plist)):
                j = next(j for j, (_, prefixes) in enumerate(self._parts) if k.startswith(prefixes))
                off = offset(self._h, i)
                self._grad_views[j].append((p, self._grad_flat[off:off + p.numel()].view(p.shape)))
            self._grad_views_key = self._grad_flat.data_ptr()
        return self._grad_views[part]

    def _backward_part(self, part: int, launch: Callable[[int], None]) -> None:
        """Runs `launch(accumulate)` (the part's backward in the library), then hands out the part's gradients as views of
        the flat buffer (no per-parameter copy).  torch semantics: every p.grad None (zero_grad(set_to_none=True), the
        default) -> start from zero; every p.grad still our view (not zeroed, or zeroed in place) -> add to what is there."""
        views = self._part_views(part)
        have = [p.grad is not None for p, _ in views if p.requires_grad]
        accumulate = bool(have) and all(have)
        if any(have) and not accumulate:
            raise self._err("either all of a part's parameter gradients are set (accumulate) or none")
        for p, gv in views:
            if p.grad is not None and p.grad.data_ptr() != gv.data_ptr():
                raise self._err("p.grad must be None or the engine's own gradient view")
        with torch.cuda.device(self._grad_flat.device):
            launch(1 if accumulate else 0)
        for p, gv in views:
            p.grad = gv

    # ------------------------------------------------------------------ read-outs
    def _debug_copy(self, fn, *args) -> torch.Tensor:
        dims = (C.c_int * 3)()
        _lib.check(min(0, fn(self._h, *args, None, dims, _lib.stream_ptr())))
        out = torch.empty((self._ws_key[0], *dims), dtype=torch.float32, device=self.device)
        _lib.check(min(0, fn(self._h, *args, out.data_ptr(), dims, _lib.stream_ptr())))
        return out

    def debug_tensor(self, name: str) -> torch.Tensor:
        """fp32 NCHW copy of a named internal activation of the last forward (parity tests)."""
        return self._debug_copy(self._fn("debug_tensor"), name.encode())

    def debug_grad(self, name: str, skip: bool = False) -> torch.Tensor:
        """fp32 NCHW copy of the last backward's gradient w.r.t. the activation `debug_tensor(name)` (skip=True: the share
        of it that a skip connection brought) (per-block backward tests)."""
        return self._debug_copy(self._fn("debug_grad"), name.encode(), int(skip))

    @property
    def last_launch_count(self) -> int:
        return self._fn("last_launch_count")(self._h)

    @property
    def last_backward_launch_count(self) -> int:
        """Kernel launches of the last backward of every part, summed."""
        return self._fn("backward_launch_count")(self._h)
