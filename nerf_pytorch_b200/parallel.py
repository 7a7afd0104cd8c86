"""Data-parallel plumbing for the ray-sharded path (SURVEY.md section 8e).

Rays are independent units: each rank renders its own contiguous shard of the global batch
(weak scaling: 4096 rays per GPU) with replicated weights, and the ONLY collective of a step is
one all-reduce (NCCL over NVLink / NVSwitch on GPUs, gloo in the CPU tests) of the flat
gradient vector that the backward kernels write for BOTH networks (train_utils._RenderChunk).
A fused Adam over the flat parameter buffer follows on every rank, so replicas stay identical."""
from __future__ import annotations

import os
from typing import Iterable, Optional

import torch
import torch.distributed as dist

from . import ops, train_utils


def init_distributed(backend: Optional[str] = None):
    """One process per GPU, launched by torchrun (RANK / LOCAL_RANK / WORLD_SIZE / MASTER_* in env)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
            dist.init_process_group(backend, device_id=torch.device("cuda", local))
        else:
            dist.init_process_group(backend)
    return rank, local, world


def enable_gradient_sync(group=None):
    """Average parameter gradients across ranks: inside the render backward when the step renders ONE chunk of rays
    (two halves of one all-reduce, the fine network's overlapped with the coarse backward); for multi-chunk steps the
    chunks' gradients are summed first and ``sync_gradients`` / ``FusedAdam.step`` all-reduce them once."""
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        train_utils._GRAD_SYNC = (group, dist.get_world_size(group))
    else:
        train_utils._GRAD_SYNC = None


def disable_gradient_sync():
    train_utils._GRAD_SYNC = None
    train_utils._PENDING_SYNC = False


def sync_gradients(params) -> bool:
    """All-reduce (average) the ``.grad`` of ``params`` once if a multi-chunk backward left them unsynchronised.
    Optimizers other than FusedAdam call this between ``loss.backward()`` and ``optimizer.step()``."""
    if not train_utils._PENDING_SYNC or train_utils._GRAD_SYNC is None:
        train_utils._PENDING_SYNC = False
        return False
    group, world = train_utils._GRAD_SYNC
    grads = [p.grad for p in params if p.grad is not None]
    flat = torch.cat([g.reshape(-1) for g in grads])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    flat.mul_(1.0 / world)
    off = 0
    for g in grads:
        g.copy_(flat[off:off + g.numel()].view_as(g))
        off += g.numel()
    train_utils._PENDING_SYNC = False
    return True


def shard_bounds(n_total: int, rank: int, world: int):
    """Contiguous, near-equal shards (equal when world divides n_total, which keeps
    mean-of-local-means == global mean, SURVEY.md section 8e)."""
    base, rem = divmod(n_total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_rays(rank: int, world: int, *tensors: torch.Tensor):
    lo, hi = shard_bounds(tensors[0].shape[0], rank, world)
    return tuple(t[lo:hi] for t in tensors)


def allreduce_flat_(flat: torch.Tensor, world: int, group=None):
    """Sum-all-reduce and average a flat buffer in place (used by the gloo CPU tests and by callers
    that keep their own flat gradient buffer)."""
    if world > 1:
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
        flat.mul_(1.0 / world)
    return flat


def flatten_parameters(model, arch: ops.ArchSpec) -> torch.Tensor:
    """Re-home a model's parameters as views of ONE flat fp32 buffer in the library's canonical
    order, so that (a) the render path reads the flat vector without a gather, (b) FusedAdam
    updates everything with one kernel.  ``state_dict()`` keeps the reference's names/shapes."""
    params = train_utils._ordered_params(model, arch)
    dev = params[0].device
    flat = torch.empty(sum(p.numel() for p in params), dtype=torch.float32, device=dev)
    off = 0
    with torch.no_grad():
        for p in params:
            n = p.numel()
            flat[off:off + n].copy_(p.detach().reshape(-1))
            p.data = flat[off:off + n].view(p.shape)
            off += n
    params[0]._nerfb200_flat = flat
    return flat


class FusedAdam:
    """torch.optim.Adam semantics (train_nerf.py:136-141) over flat buffers, one kernel per model,
    with the reference's exponential LR schedule folded in (train_nerf.py:264-270).  The reference sets
    lr = lr0 * decay_factor ** (i / (lr_decay * 1000)) AFTER optimizer.step() of iteration i, so the step of iteration
    i runs with the rate computed at iteration i - 1 (iterations 0 and 1 both use lr0): reproduced here."""

    def __init__(self, models_and_archs: Iterable, lr=5e-3, betas=(0.9, 0.999), eps=1e-8, lr_decay: Optional[float] = None,
                 lr_decay_factor: float = 0.1):
        self.items = []
        for model, arch in models_and_archs:
            flat = flatten_parameters(model, arch)
            params = train_utils._ordered_params(model, arch)
            self.items.append(dict(model=model, arch=arch, flat=flat, params=params,
                                   m=torch.zeros_like(flat), v=torch.zeros_like(flat)))
        self.lr0, self.betas, self.eps = lr, betas, eps
        self.lr_decay, self.lr_decay_factor = lr_decay, lr_decay_factor
        self.step_count = 0

    def current_lr(self):
        if self.lr_decay is None:
            return self.lr0
        return self.lr0 * (self.lr_decay_factor ** (max(self.step_count - 1, 0) / (self.lr_decay * 1000.0)))

    def zero_grad(self):
        for it in self.items:
            for p in it["params"]:
                p.grad = None

    @torch.no_grad()
    def step(self, grad_scale: float = 1.0):
        lr = self.current_lr()
        self.step_count += 1
        if train_utils._PENDING_SYNC:  # multi-chunk step: one all-reduce over everything, now
            sync_gradients([p for it in self.items for p in it["params"]])
        for it in self.items:
            params = it["params"]
            g0 = params[0].grad
            if g0 is None:
                continue
            # gradients returned by the render backward are views of one flat buffer, in order
            base = g0.data_ptr()
            off, contiguous = 0, True
            for p in params:
                if p.grad is None or p.grad.data_ptr() != base + 4 * off or not p.grad.is_contiguous():
                    contiguous = False
                    break
                off += p.numel()
            if contiguous:
                gflat = g0.reshape(-1).as_strided((off,), (1,))
            else:
                gflat = torch.cat([p.grad.reshape(-1) for p in params])
            ops.adam_step(it["flat"], gflat.contiguous(), it["m"], it["v"], self.step_count, lr, self.betas[0],
                          self.betas[1], self.eps, grad_scale)
            model = it["model"]
            model._nerfb200_epoch = getattr(model, "_nerfb200_epoch", 0) + 1
