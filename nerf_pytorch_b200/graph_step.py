"""One training step of the reference's loop (train_nerf.py:175-270) as ONE CUDA graph launch, with no host
synchronisation: pixel draw, rays, render, loss, backward and Adam all run on the device.

A captured graph freezes its kernel arguments, so the only value that changes between replays is an int64 step counter
in device memory; every kernel that depends on the step reads it there (include/nerfb200.h, "a training step with no
host work").  The render path is the existing one: the step's four random inputs are written as tensors by
``random_fill_dev`` and passed to ``render_fwd`` / ``render_bwd``, which makes the step equal, bit for bit, to one
rendered with ``SeededRandoms(seed, step)`` (DESIGN §1)."""
from __future__ import annotations

from typing import Optional

import torch

from . import ops, train_utils
from .cache_pool import CachedRayPool

__all__ = ["CapturedTrainStep"]


def _cuda(t: torch.Tensor, what: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise NotImplementedError(f"CapturedTrainStep: {what} must be a CUDA tensor (there is no CPU path)")
    return t


class CapturedTrainStep:
    """``step()`` = one iteration of the reference's training loop at ``options.nerf.train.num_random_rays`` rays:

    * draw one training image uniformly and that many distinct pixels of it, from (``seed``, step);
    * the rays of those pixels (NDC, near / far and view directions as ``options.dataset`` says) and their targets;
    * ``run_one_iter_of_nerf`` in one chunk with the seeded randoms of that step, ``mse(rgb_coarse, t) +
      mse(rgb_fine, t)`` (the coarse term alone without a fine network) and its backward;
    * ``FusedAdam.step`` of both networks at the reference's one-step-late learning-rate schedule.

    The step is the optimizer's ``step_count``; it advances on the device and on the host.  A step equals, bit for bit,
    ``run_one_iter_of_nerf_from_pose(..., randoms=SeededRandoms(seed, step))`` at the same image and pixels, torch's
    ``mse_loss`` and ``backward`` and ``optimizer.step()`` (on impl 0 up to the fp32 CUDA-core weight gradients, which
    are summed with atomics).

    ``source``: ``(images, poses, focal)`` with images (N, H, W, 3) and poses (N, 3 | 4, 4) fp32 on the device (the
    reference's uncached loop), or a ``CachedRayPool`` whose images share (H, W, focal) and their ray count.
    ``optimizer``: the ``parallel.FusedAdam`` over both models; its parameters, moments and ``step_count`` are used in
    place, so a step built on an optimizer at step k continues its run.  Its ``lr`` / ``lr_decay`` /
    ``lr_decay_factor`` are the schedule; ``options.optimizer.lr`` and ``options.scheduler.*``, when present, must agree.
    ``impl``: None picks the kernels as ``run_one_iter_of_nerf`` does; 0 or 1 force one.
    ``capture=False`` runs the same launches eagerly on every ``step()`` (debugging, tests).

    Parameters updated by a captured step are written behind torch's back: ``step()`` tells the render path's weight
    cache (``train_utils.invalidate``), so eager calls in between see them.  Re-homing a parameter's storage after
    construction is not seen by the graph."""

    def __init__(self, model_coarse, model_fine, encode_position_fn, encode_direction_fn, options, optimizer, seed: int,
                 source, *, impl: Optional[int] = None, capture: bool = True):
        # ---- every refusal comes before the first launch
        o = options.nerf.train
        n = int(o.num_random_rays)
        if int(o.chunksize) < n:
            raise ValueError(f"CapturedTrainStep: chunksize {o.chunksize} < num_random_rays {n}: a step renders one chunk")
        if train_utils._GRAD_SYNC is not None:
            raise NotImplementedError("CapturedTrainStep: gradient sync across ranks is not captured; one GPU only")
        impl = train_utils.DEFAULT_IMPL if impl is None else int(impl)
        if impl == ops.IMPL_TC_FAST:
            raise NotImplementedError("CapturedTrainStep: impl=3 (single-pass fp16 wgmma forward) is inference only")
        if impl not in (None, ops.IMPL_SIMT, ops.IMPL_TC):
            raise ValueError(f"CapturedTrainStep: impl must be None, 0 or 1, got {impl}")
        if not 0 <= int(seed) < 2 ** 64:
            raise ValueError("CapturedTrainStep: seed must be in [0, 2^64)")
        nc, nf = int(o.num_coarse), int(o.num_fine)
        fine = nf > 0
        if fine and not model_fine:
            raise RuntimeError("CapturedTrainStep: num_fine > 0 but model_fine is None")
        models = [model_coarse] + ([model_fine] if fine else [])
        self._check_schedule(options, optimizer)
        items = []
        for m in models:
            it = next((it for it in optimizer.items if it["model"] is m), None)
            if it is None:
                raise ValueError("CapturedTrainStep: the optimizer does not hold this model")
            items.append(it)

        if isinstance(source, CachedRayPool):
            pool = source
            rows = {b - a for a, b in zip(pool.offsets[:-1], pool.offsets[1:])}
            if len(set(pool.meta)) != 1 or len(rows) != 1:
                raise ValueError("CapturedTrainStep: the pool's images differ in (H, W, focal) or in their ray count")
            (height, width, focal), n_pixels, n_images = pool.meta[0], rows.pop(), pool.num_images
            tensors = {"the ray pool": pool.ray_origins}
            self._pool, self._images, self._poses = pool, None, None
        else:
            images, poses, focal = source
            if images.dim() != 4 or images.shape[-1] != 3 or images.dtype != torch.float32:
                raise ValueError(f"CapturedTrainStep: images must be fp32 (N, H, W, 3), got {tuple(images.shape)}")
            if (poses.dim() != 3 or poses.shape[0] != images.shape[0] or poses.shape[1] not in (3, 4)
                    or poses.shape[2] != 4 or poses.dtype != torch.float32):
                raise ValueError(f"CapturedTrainStep: poses must be fp32 (N, 3 | 4, 4), got {tuple(poses.shape)}")
            n_images, height, width = images.shape[:3]
            n_pixels = height * width
            tensors = {"images": images, "poses": poses}
            self._pool, self._images, self._poses = None, images.contiguous(), poses.contiguous()
        if n > n_pixels:
            raise ValueError(f"CapturedTrainStep: cannot draw {n} distinct rays from an image of {n_pixels}")
        for what, t in tensors.items():
            _cuda(t, what)
        for m in models:
            for p in m.parameters():
                _cuda(p, "every parameter")

        enc_xyz = train_utils._probe_encoder(encode_position_fn, None)
        if enc_xyz is None:
            raise RuntimeError("CapturedTrainStep: encode_position_fn is required")
        use_viewdirs = bool(options.nerf.use_viewdirs)
        enc_dir = train_utils._probe_encoder(encode_direction_fn if use_viewdirs else None, None)
        self.arch_c = train_utils._arch_of(model_coarse, enc_xyz, enc_dir)
        self.arch_f = train_utils._arch_of(model_fine, enc_xyz, enc_dir) if fine else None
        if impl is None:
            impl = train_utils._auto_impl(self.arch_c, self.arch_f, nc, nf, training=True)
        for a, s in ((self.arch_c, nc), (self.arch_f, nc + nf)):
            if a is not None and not ops.impl_supported(a, s, impl):
                raise NotImplementedError(f"CapturedTrainStep: impl={impl} does not train this network "
                                          f"({ops._lib.load().nerfb200_last_error().decode()})")

        self.models, self.optimizer, self.seed, self.impl, self.n = models, optimizer, int(seed), impl, n
        self.height, self.width, self.focal, self.n_images, self.n_pixels = height, width, float(focal), n_images, n_pixels
        self.opts = ops.make_opts(nc, nf, o.perturb, o.lindisp, o.white_background, o.radiance_field_noise_std)
        self.ndc = options.dataset.no_ndc is False
        self.near, self.far, self.use_viewdirs = float(options.dataset.near), float(options.dataset.far), use_viewdirs
        self._items = items

        # ---- buffers: every pointer the step uses is fixed here
        dev = items[0]["flat"].device
        e = lambda *shape, dtype=torch.float32: torch.empty(*shape, dtype=dtype, device=dev)
        self.step_dev = torch.full((1,), optimizer.step_count, dtype=torch.int64, device=dev)
        self.image, self.pixel_ids = e(1, dtype=torch.int64), e(n, dtype=torch.int64)
        self._draw_ws = e(ops.draw_workspace_bytes(n_pixels), dtype=torch.uint8)
        self.target = e(n, 3)
        if self._pool is None:
            self.rays = e(n, 11 if use_viewdirs else 8)
        else:  # pack_rays writes the rows anew on each run
            self._ro, self._rd = e(n, 3), e(n, 3)
        perturb, noise = bool(o.perturb), float(o.radiance_field_noise_std) > 0.0
        sizes = {"t_rand": (perturb, nc), "noise_c": (noise, nc), "u": (perturb and fine, nf),
                 "noise_f": (noise and fine, nc + nf)}
        self.randoms = {k: e(n, s) for k, (used, s) in sizes.items() if used}
        self.blobs = [e(a.blob_floats()) for a in (self.arch_c, self.arch_f) if a is not None]
        self._ws = e(ops.render_workspace_bytes(self.arch_c, self.arch_f, self.opts, n, True), dtype=torch.uint8)
        self.loss = e(())
        self.g = [e(n, 8) for _ in models]
        self.flat_grad = e(sum(it["flat"].numel() for it in items))
        self.count = optimizer.step_count

        self._graph = None
        if capture:
            self._capture()

    @staticmethod
    def _check_schedule(options, opt):
        lr = getattr(getattr(options, "optimizer", None), "lr", None)
        sch = getattr(options, "scheduler", None)
        mine = (opt.lr0, opt.lr_decay, opt.lr_decay_factor)
        theirs = (lr if lr is not None else opt.lr0, getattr(sch, "lr_decay", opt.lr_decay),
                  getattr(sch, "lr_decay_factor", opt.lr_decay_factor))
        if tuple(map(lambda x: None if x is None else float(x), mine)) != tuple(
                map(lambda x: None if x is None else float(x), theirs)):
            raise ValueError(f"CapturedTrainStep: the optimizer's schedule (lr, lr_decay, lr_decay_factor) = {mine} "
                             f"disagrees with the options' {theirs}")
        if opt.lr_decay is not None and not float(opt.lr_decay) > 0.0:
            raise ValueError("CapturedTrainStep: lr_decay must be > 0 (or None for a constant rate)")

    # ---------------------------------------------------------------------------------------------
    def _launch(self):
        """Every launch of one step, in order; the same list is captured and run eagerly."""
        n, step = self.n, self.step_dev
        ops.draw_pixels(self.seed, step, self.n_images, self.n_pixels, n, self.image, self.pixel_ids, self._draw_ws)
        if self._pool is None:
            ops.gen_rays_posed(self._poses, self.image, self.height, self.width, self.focal, self.pixel_ids, self.ndc,
                               self.near, self.far, self.use_viewdirs, out=self.rays)
            ops.gather_rows(self._images, self.n_pixels, self.image, self.pixel_ids, out=self.target)
        else:
            p = self._pool
            ops.gather_rows(p.ray_origins, self.n_pixels, self.image, self.pixel_ids, out=self._ro)
            ops.gather_rows(p.ray_directions, self.n_pixels, self.image, self.pixel_ids, out=self._rd)
            ops.gather_rows(p.targets, self.n_pixels, self.image, self.pixel_ids, out=self.target)
            self.rays = ops.pack_rays(self._ro, self._rd, self.height, self.width, self.focal, self.ndc, self.near,
                                      self.far, self.use_viewdirs)
        for name, t in self.randoms.items():
            ops.random_fill_dev(self.seed, step, name, n, t.shape[1], out=t)
        for arch, it, blob in zip((self.arch_c, self.arch_f), self._items, self.blobs):
            ops.pack_weights(arch, it["flat"], blob)
        blob_f = self.blobs[1] if self.arch_f is not None else None
        out_c, out_f, _ = ops.render_fwd(self.arch_c, self.arch_f, self.opts, self.blobs[0], blob_f, self.rays,
                                         self.randoms, training=True, impl=self.impl, workspace=self._ws)
        g_f = self.g[1] if out_f is not None else None
        ops.mse_loss(out_c, out_f, self.target, self.loss, self.g[0], g_f)
        self.flat_grad.zero_()
        nc = self._items[0]["flat"].numel()
        ops.render_bwd(self.arch_c, self.arch_f, self.opts, self.blobs[0], blob_f, self.rays, self.randoms, self.g[0],
                       g_f, self._ws, self.flat_grad[:nc], self.flat_grad[nc:] if g_f is not None else None,
                       impl=self.impl)
        opt, off = self.optimizer, 0
        for it in self._items:
            k = it["flat"].numel()
            ops.adam_step_dev(it["flat"], self.flat_grad[off:off + k], it["m"], it["v"], step, opt.lr0, opt.lr_decay,
                              opt.lr_decay_factor, opt.betas[0], opt.betas[1], opt.eps)
            off += k
        ops.step_advance(step)
        self._out = (out_c, out_f)  # keeps the graph's outputs alive with it

    def _capture(self):
        # a warm-up step on a side stream loads every module and fills the allocator; it is undone, so the graph's first
        # replay is the optimizer's next step
        saved = [(it["flat"].clone(), it["m"].clone(), it["v"].clone()) for it in self._items]
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            self._launch()
            for it, (p, m, v) in zip(self._items, saved):
                it["flat"].copy_(p)
                it["m"].copy_(m)
                it["v"].copy_(v)
            self.step_dev.fill_(self.count)
        torch.cuda.current_stream().wait_stream(side)
        self._graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self._graph):
            self._launch()

    def step(self) -> torch.Tensor:
        """Run one training step; returns its loss as a 0-dim CUDA tensor, without synchronising."""
        if self.optimizer.step_count != self.count:  # stepped elsewhere in between (an eager FusedAdam.step)
            self.count = self.optimizer.step_count
            self.step_dev.fill_(self.count)
        if self.count >= 2 ** 30:
            raise ValueError("CapturedTrainStep: step must be < 2^30 (the seeded randoms' range)")
        if self._graph is not None:
            self._graph.replay()
        else:
            self._launch()
        self.count += 1
        self.optimizer.step_count = self.count
        for m in self.models:
            m._nerfb200_epoch = getattr(m, "_nerfb200_epoch", 0) + 1
        return self.loss.clone()
