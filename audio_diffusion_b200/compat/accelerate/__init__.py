"""Minimal `accelerate` surface for the UNCHANGED scripts/train_unet.py (imports :13-15; calls :45-50, :181, :199-201,
:252-283, :285-346), on the H100 engine.

What HF accelerate 0.34 does for that script, restated here ([3P-recall] accelerate==0.34.2, requirements-lock.txt:2):
  * one process per GPU (torchrun env: RANK / LOCAL_RANK / WORLD_SIZE), NCCL process group, `accelerator.device`;
  * `prepare(model, optimizer, dataloader, lr_scheduler)`: the model goes to the device and is wrapped for data
    parallelism; the dataloader is sharded batch-wise across the processes (process r sees batches r, r+N, ...; the
    tail is completed from the first batches so every process runs the same number of steps, `even_batches=True`) and
    moves every batch to the device; the optimizer skips `step()` / `zero_grad()` while gradients are being
    accumulated; the LR scheduler is stepped only with the optimizer and `num_processes` times per call
    (`split_batches=False`), because the schedule was sized on the unsharded dataloader (train_unet.py:178);
  * `accumulate(model)`: gradients are synchronised on every `gradient_accumulation_steps`-th call and on the last
    batch of the dataloader; in between the backward runs under `no_sync()`;
  * `backward(loss)` divides the loss by `gradient_accumulation_steps`;
  * mixed precision "bf16": autocast around the model's forward.  The engine's U-Net already computes with bf16
    operands / fp32 accumulation and fp32 master weights (what autocast gives the reference), so this is a no-op here.
Data parallelism itself: `UNet2DModel`'s backward all-reduces its flat gradient buffer (parallel.allreduce_mean_), which
replaces the DDP wrapper; `unwrap_model` therefore returns the model itself and `model.module` does not exist
(train_unet.py:186,226 use getattr(model, "module", model)).
"""
from __future__ import annotations

import contextlib
import os
from typing import List

import torch

from . import logging, utils  # noqa: F401
from .utils import ProjectConfiguration


class _ShardedLoader:
    """DataLoaderShard + BatchSamplerShard(split_batches=False, even_batches=True): batches r, r+N, ... of the wrapped
    loader, each moved to the device; `end_of_dataloader` is raised on the last one (accumulate() syncs there)."""

    def __init__(self, loader, accelerator):
        self.loader, self.acc = loader, accelerator
        self.dataset = getattr(loader, "dataset", None)
        self.batch_size = getattr(loader, "batch_size", None)
        self.end_of_dataloader = False

    def __len__(self):
        n, w = len(self.loader), self.acc.num_processes
        return (n + w - 1) // w

    def _to_device(self, b):
        dev = self.acc.device
        if torch.is_tensor(b):
            return b.to(dev, non_blocking=True)
        if isinstance(b, dict):
            return {k: self._to_device(v) for k, v in b.items()}
        if isinstance(b, (list, tuple)):
            return type(b)(self._to_device(v) for v in b)
        return b

    def __iter__(self):
        w, r = self.acc.num_processes, self.acc.process_index
        self.end_of_dataloader = False
        self.acc._active_loader = self
        mine: List = []
        head: List = []                     # the first batches complete the last round when len(loader) % N != 0
        total = len(self)
        served = 0
        for i, batch in enumerate(self.loader):
            if i < w:
                head.append(batch)
            if i % w == r:
                served += 1
                self.end_of_dataloader = served == total
                yield self._to_device(batch)
        if served < total:                  # this rank's slot in the last round is empty: reuse an early batch
            self.end_of_dataloader = True
            yield self._to_device(head[(served * w + r) % max(len(head), 1)])


class _Optimizer:
    """AcceleratedOptimizer: step / zero_grad only when gradients are synchronised (i.e. not mid-accumulation)."""

    def __init__(self, opt, accelerator):
        self.optimizer, self.acc = opt, accelerator

    def step(self, closure=None):
        if self.acc.sync_gradients:
            self.optimizer.step(closure) if closure is not None else self.optimizer.step()

    def zero_grad(self, set_to_none=None):
        if self.acc.sync_gradients:
            self.optimizer.zero_grad() if set_to_none is None else self.optimizer.zero_grad(set_to_none=set_to_none)

    def __getattr__(self, name):
        return getattr(self.optimizer, name)


class _Scheduler:
    """AcceleratedScheduler(step_with_optimizer=True, split_batches=False)."""

    def __init__(self, sched, accelerator):
        self.scheduler, self.acc = sched, accelerator

    def step(self, *a, **k):
        if not self.acc.sync_gradients:
            return
        for _ in range(self.acc.num_processes):
            self.scheduler.step(*a, **k)

    def __getattr__(self, name):
        return getattr(self.scheduler, name)


class _TensorBoardTracker:
    name = "tensorboard"

    def __init__(self, run_name: str, logging_dir: str):
        from torch.utils.tensorboard import SummaryWriter
        self.writer = SummaryWriter(os.path.join(logging_dir, run_name))

    def log(self, values: dict, step=None):
        for k, v in values.items():
            if isinstance(v, (int, float)):
                self.writer.add_scalar(k, v, global_step=step)
        self.writer.flush()

    def finish(self):
        self.writer.close()


class Accelerator:
    def __init__(self, gradient_accumulation_steps: int = 1, mixed_precision: str = "no", log_with=None,
                 project_config: ProjectConfiguration = None, **_ignored):
        self.gradient_accumulation_steps = int(gradient_accumulation_steps)
        self.mixed_precision = mixed_precision
        self.log_with = log_with
        self.project_config = project_config or ProjectConfiguration()
        self.process_index = int(os.environ.get("RANK", "0"))
        self.local_process_index = int(os.environ.get("LOCAL_RANK", "0"))
        self.num_processes = int(os.environ.get("WORLD_SIZE", "1"))
        if torch.cuda.is_available():
            torch.cuda.set_device(self.local_process_index)
            self.device = torch.device("cuda", self.local_process_index)
        else:
            self.device = torch.device("cpu")
        if self.num_processes > 1:
            import torch.distributed as dist
            if not dist.is_initialized():
                os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
                if self.device.type == "cuda":
                    dist.init_process_group("nccl", device_id=self.device)
                else:
                    dist.init_process_group("gloo")
        self.sync_gradients = True
        self.step = 0
        self.trackers: list = []
        self._active_loader = None
        self._models: list = []

    # ---- process topology
    @property
    def is_main_process(self) -> bool:
        return self.process_index == 0

    @property
    def is_local_main_process(self) -> bool:
        return self.local_process_index == 0

    def wait_for_everyone(self):
        if self.num_processes > 1:
            import torch.distributed as dist
            dist.barrier()

    # ---- prepare
    def prepare(self, *objs):
        out = []
        for o in objs:
            if isinstance(o, torch.nn.Module):
                o = o.to(self.device)
                if self.num_processes > 1:      # what DDP does at construction: every rank starts from rank 0's weights
                    from audio_diffusion_b200.parallel import broadcast_parameters
                    broadcast_parameters(o.parameters(), src=0)
                self._models.append(o)
                out.append(o)
            elif isinstance(o, torch.optim.Optimizer):
                out.append(_Optimizer(o, self))
            elif isinstance(o, torch.utils.data.DataLoader):
                out.append(_ShardedLoader(o, self))
            elif hasattr(o, "step") and hasattr(o, "get_last_lr"):
                out.append(_Scheduler(o, self))
            else:
                out.append(o)
        return out[0] if len(out) == 1 else tuple(out)

    def unwrap_model(self, model):
        return getattr(model, "module", model)

    # ---- gradient accumulation / backward / clipping
    @contextlib.contextmanager
    def accumulate(self, *models):
        self.step += 1
        end = self._active_loader is not None and self._active_loader.end_of_dataloader
        self.sync_gradients = end or (self.step % self.gradient_accumulation_steps == 0)
        if end:
            self.step = 0
        with contextlib.ExitStack() as stack:
            if not self.sync_gradients:
                for m in models:
                    if hasattr(m, "no_sync"):
                        stack.enter_context(m.no_sync())
            yield

    def backward(self, loss, **kw):
        if self.gradient_accumulation_steps > 1:
            loss = loss / self.gradient_accumulation_steps
        loss.backward(**kw)

    def clip_grad_norm_(self, parameters, max_norm, norm_type=2):
        return torch.nn.utils.clip_grad_norm_(parameters, max_norm, norm_type=norm_type)

    # ---- tracking
    def init_trackers(self, project_name: str, config=None, init_kwargs=None):
        if self.is_main_process and self.log_with in ("tensorboard", ["tensorboard"], "all"):
            self.trackers = [_TensorBoardTracker(project_name, self.project_config.logging_dir or ".")]

    def log(self, values: dict, step=None):
        for t in self.trackers:
            t.log(values, step=step)

    def end_training(self):
        for t in self.trackers:
            t.finish()
        self.wait_for_everyone()
