"""Drop-in replacements for the reference's render driver (nerf/train_utils.py):

    run_one_iter_of_nerf            nerf/train_utils.py:130-202
    predict_and_render_radiance     nerf/train_utils.py:28-127

Same positional signatures, same option keys (``options.nerf.<mode>.*``, ``options.dataset.*``),
same 6-tuple result, differentiable w.r.t. the parameters of both models.  Everything per-ray
(stratified sampling, encoding, both MLPs, compositing, hierarchical resampling, their backward)
runs in libnerfb200.so; this file only moves pointers: it reads the options, draws the random
tensors in the reference's order (so a shared torch seed gives the reference-on-GPU's random
stream) or hands the kernels a seed instead (``ops.SeededRandoms``), flattens the parameters and
calls the C ABI through ``ops``.

There is no PyTorch fallback: an unsupported model / device / dtype raises.
"""
from __future__ import annotations

import math
import numbers
import weakref
from typing import Optional, Union

import torch

from . import ops
from .ops import SeededRandoms
from .nerf_helpers import Embedder, get_minibatches

# The reference does not forward ``mode`` to predict_and_render_radiance (train_utils.py:171-181),
# so validation renders use options.nerf.train.* for sampling/noise.  True reproduces that.
COMPAT_MODE_QUIRK = True

# None: wgmma tensor cores (three-term split-precision products) wherever the kernels support the configuration (training: hidden
# 128; inference: hidden 128 or 256; encodings <= 64 wide, >= 15 samples per ray), fp32 CUDA cores otherwise; 0 / 1 force one.
# 3 (ops.IMPL_TC_FAST, single-pass fp16 products) is for renders only: a call that would train with it raises.
DEFAULT_IMPL = None


def _auto_impl(arch_c, arch_f, n_coarse, n_fine, training=True):
    # inference only needs the wgmma forward (hidden 128 and 256); training needs the fused backward too (hidden 128)
    what = ops.IMPL_TC if training else ops.IMPL_TC_FWD
    ok = all(a is None or ops.impl_supported(a, n_coarse, what) for a in (arch_c, arch_f))
    return ops.IMPL_TC if ok else ops.IMPL_SIMT

# gradient synchronisation across ranks: (process_group, world_size) or None; see parallel.py
_GRAD_SYNC = None
# set when a step rendered its rays in several chunks: their gradients are summed by autograd first and
# all-reduced ONCE afterwards (parallel.sync_gradients / FusedAdam.step), never once per chunk
_PENDING_SYNC = False


def _trains(params) -> bool:
    """A call trains when autograd is on and one of its parameters requires grad."""
    return torch.is_grad_enabled() and any(p.requires_grad for p in params)


def _requested_impl(impl, *models):
    """The kernels a call asks for: ``impl``, else ``DEFAULT_IMPL``; None leaves the choice to ``_auto_impl``.
    ops.IMPL_TC_FAST renders only (no stash, no backward): a call that would train with it raises here, before
    anything is launched."""
    impl = DEFAULT_IMPL if impl is None else int(impl)
    if impl == ops.IMPL_TC_FAST and _trains(p for m in models if m is not None for p in m.parameters()):
        raise NotImplementedError("nerfb200: impl=3 (single-pass fp16 wgmma forward) is inference only; train with "
                                  "impl=0 or impl=1, or render under torch.no_grad()")
    return impl


def set_default_impl(impl):
    global DEFAULT_IMPL
    DEFAULT_IMPL = None if impl is None else int(impl)


# --------------------------------------------------------------------------------------------------
# model / encoder introspection
# --------------------------------------------------------------------------------------------------
_PROBED: dict = {}   # id(callable) -> (weakref or None, result): an opaque encoder is probed once, not on every chunk


def _probe_encoder(fn, dim_expected: Optional[int]):
    """(L, include_input, log_sampling) of an encoder.  ``Embedder`` objects carry their parameters;
    an opaque callable (the reference's own lambda, nerf_helpers.py:160-167) is identified by
    evaluating it once on a CPU probe and matching the stock encoding (memoised per callable)."""
    if fn is None:
        return None
    if isinstance(fn, Embedder) or all(hasattr(fn, a) for a in ("num_encoding_functions", "include_input", "log_sampling")):
        return int(fn.num_encoding_functions), bool(fn.include_input), bool(fn.log_sampling)
    hit = _PROBED.get(id(fn))
    if hit is not None and (hit[0] is None or hit[0]() is fn):
        return hit[1]
    res = _probe_encoder_uncached(fn)
    try:
        ref = weakref.ref(fn)
    except TypeError:   # not weak-referenceable: keep it alive through the key's lifetime instead
        ref = (lambda f: (lambda: f))(fn)
    _PROBED[id(fn)] = (ref, res)
    return res


def _probe_encoder_uncached(fn):
    probe = torch.tensor([[0.3, -0.7, 1.1]], dtype=torch.float32)
    try:
        got = fn(probe)
    except Exception as e:  # pragma: no cover - user callables
        raise NotImplementedError(f"nerfb200: cannot introspect encoder {fn!r}: {e}")
    dim = got.shape[-1]
    for include in (True, False):
        rest = dim - (3 if include else 0)
        if rest < 0 or rest % 6:
            continue
        L = rest // 6
        for log_sampling in (True, False):
            bands = ops.frequency_bands(L, log_sampling)
            parts = [probe] if include else []
            for f in bands:
                parts += [torch.sin(probe * f), torch.cos(probe * f)]
            ref = torch.cat(parts, -1) if len(parts) > 1 else parts[0]
            if ref.shape == got.shape and torch.allclose(ref, got.cpu().float(), atol=1e-6):
                return L, include, log_sampling
    raise NotImplementedError("nerfb200: encoder is not the stock positional_encoding; no fused path for it")


def _arch_of(model, enc_xyz, enc_dir) -> ops.ArchSpec:
    need = ("layer1", "layers_xyz")
    if not all(hasattr(model, a) for a in need):
        raise NotImplementedError(
            f"nerfb200: {type(model).__name__} is not a FlexibleNeRFModel (nerf/models.py:185); only that family is fused")
    use_viewdirs = hasattr(model, "fc_rgb")
    hidden = model.layer1.out_features
    n_xyz = len(model.layers_xyz)
    wide = [i for i, l in enumerate(model.layers_xyz) if l.in_features != l.out_features]
    skip = int(getattr(model, "skip_connect_every", 0)) or (wide[0] if wide else n_xyz + 1)
    rule = [i for i in range(n_xyz) if i % skip == 0 and i > 0]
    if rule != wide:
        raise NotImplementedError(f"nerfb200: skip layers {wide} do not follow skip_connect_every={skip}")
    Lx, incx, logx = enc_xyz
    if use_viewdirs:
        if enc_dir is None:
            raise RuntimeError("nerfb200: model uses view directions but no direction encoder was given")
        Ld, incd, logd = enc_dir
    else:
        Ld, incd, logd = 0, True, True
    arch = ops.ArchSpec(num_layers=n_xyz + 1, hidden=hidden, skip_every=skip, use_viewdirs=use_viewdirs,
                        n_freq_xyz=Lx, n_freq_dir=Ld, include_input_xyz=incx, include_input_dir=incd,
                        log_sampling_xyz=logx, log_sampling_dir=logd)
    if model.layer1.in_features != arch.dim_xyz:
        raise RuntimeError(f"nerfb200: layer1 expects {model.layer1.in_features} inputs, encoder produces {arch.dim_xyz}")
    if use_viewdirs and model.layers_dir[0].in_features != hidden + arch.dim_dir:
        raise RuntimeError("nerfb200: layers_dir[0] width does not match the direction encoder")
    return arch


def _ordered_params(model, arch: ops.ArchSpec):
    mods = [model.layer1] + list(model.layers_xyz)
    if arch.use_viewdirs:
        mods += [model.fc_feat, model.fc_alpha, model.layers_dir[0], model.fc_rgb]
    else:
        mods += [model.fc_out]
    out = []
    for m in mods:
        out += [m.weight, m.bias]
    return out


class _Packed:
    """Per-model cache: flat parameter vector + kernel blob, refreshed when any parameter changes
    (torch bumps ``_version`` on every in-place optimizer update)."""

    __slots__ = ("arch", "key", "flat", "blob")

    def __init__(self):
        self.arch = None
        self.key = None
        self.flat = None
        self.blob = None


_CACHE: "weakref.WeakKeyDictionary" = weakref.WeakKeyDictionary()


def _flat_view_if_contiguous(params):
    """If the parameters already live back-to-back in one storage (parallel.flatten_parameters),
    return that storage slice without copying."""
    p0 = params[0]
    base = p0.data_ptr()
    off = 0
    for p in params:
        if p.data_ptr() != base + 4 * off or not p.is_contiguous():
            return None
        off += p.numel()
    flat = getattr(p0, "_nerfb200_flat", None)
    if flat is not None and flat.data_ptr() == base and flat.numel() == off:
        return flat
    return None


def invalidate(model) -> None:
    """Drop the cached kernel blob of ``model``.  The cache key follows torch's parameter version counters and data
    pointers, so every update made through torch ops (optimizers, ``copy_``, ``load_state_dict``) and through
    ``FusedAdam`` is seen; call this after writing parameter memory behind torch's back (raw pointers, external kernels,
    ``p.data`` views mutated by foreign code)."""
    model._nerfb200_epoch = getattr(model, "_nerfb200_epoch", 0) + 1
    _CACHE.pop(model, None)


def _packed(model, arch: ops.ArchSpec):
    params = _ordered_params(model, arch)
    for p in params:
        if not p.is_cuda or p.dtype != torch.float32:
            raise NotImplementedError("nerfb200: parameters must be fp32 CUDA tensors (no CPU / half path)")
    ent = _CACHE.get(model)
    if ent is None:
        ent = _CACHE[model] = _Packed()
    key = (arch, tuple(p._version for p in params), tuple(p.data_ptr() for p in params),
           getattr(model, "_nerfb200_epoch", 0))
    if ent.key != key:
        with torch.no_grad():
            flat = _flat_view_if_contiguous(params)
            if flat is None:
                flat = torch.cat([p.detach().reshape(-1) for p in params])
            ent.flat = flat
            ent.blob = ops.pack_weights(arch, flat, None)  # fresh blob: an in-flight backward may still hold the old one
        ent.arch, ent.key = arch, key
    return params, ent.blob


# --------------------------------------------------------------------------------------------------
# autograd bridge for one ray chunk
# --------------------------------------------------------------------------------------------------
class _RenderChunk(torch.autograd.Function):
    @staticmethod
    def forward(ctx, cfg, rays, randoms, *params):
        arch_c, arch_f, opts, blob_c, blob_f, training, impl, n_chunks = cfg
        out_c, out_f, ws = ops.render_fwd(arch_c, arch_f, opts, blob_c, blob_f, rays, randoms, training=training,
                                          impl=impl)
        if training:
            ctx.cfg = cfg
            ctx.ws = ws
            # the backward needs the noise again: a SeededRandoms regenerates it in-kernel, drawn tensors are kept
            ctx.rng = randoms if isinstance(randoms, SeededRandoms) else None
            noise = (None, None) if ctx.rng is not None else (randoms.get("noise_c"), randoms.get("noise_f"))
            ctx.save_for_backward(rays, *noise)
        ctx.set_materialize_grads(False)
        if out_f is None:
            return out_c, None
        return out_c, out_f

    @staticmethod
    def backward(ctx, g_c, g_f):
        arch_c, arch_f, opts, blob_c, blob_f, training, impl, n_chunks = ctx.cfg
        rays, noise_c, noise_f = ctx.saved_tensors
        fine = opts.n_fine > 0
        n = rays.shape[0]
        if g_c is None:
            g_c = torch.zeros(n, 8, dtype=torch.float32, device=rays.device)
        if fine and g_f is None:
            g_f = torch.zeros(n, 8, dtype=torch.float32, device=rays.device)
        nc = arch_c.flat_param_count()
        nf = arch_f.flat_param_count() if fine else 0
        flat_grad = torch.zeros(nc + nf, dtype=torch.float32, device=rays.device)
        g_c = g_c.contiguous()
        g_f = g_f.contiguous() if fine else None
        randoms = ctx.rng if ctx.rng is not None else dict(noise_c=noise_c, noise_f=noise_f)
        args = (arch_c, arch_f, opts, blob_c, blob_f, rays, randoms, g_c, g_f, ctx.ws, flat_grad[:nc],
                flat_grad[nc:] if fine else None)
        sync = _GRAD_SYNC
        if sync is not None and n_chunks != 1:
            # several chunks per step: no collective here (ranks may even differ in their chunk counts); the summed
            # gradients are all-reduced once by parallel.sync_gradients / FusedAdam.step
            global _PENDING_SYNC
            _PENDING_SYNC = True
            sync = None
        if sync is None:
            ops.render_bwd(*args, impl=impl)
        else:
            # the ONE collective of a data-parallel step, split in two so that the fine network's half (final as soon
            # as its backward is done) crosses NVLink while the coarse network's backward is still running
            import torch.distributed as dist

            group, world = sync
            works = []
            if fine:
                ops.render_bwd(*args, impl=impl, parts=1)
                works.append(dist.all_reduce(flat_grad[nc:], op=dist.ReduceOp.SUM, group=group, async_op=True))
            ops.render_bwd(*args, impl=impl, parts=2 if fine else 3)
            works.append(dist.all_reduce(flat_grad[:nc], op=dist.ReduceOp.SUM, group=group, async_op=True))
            for w in works:
                w.wait()
            flat_grad.mul_(1.0 / world)
        ctx.ws = None
        grads = []
        for arch, base in ((arch_c, 0),) + (((arch_f, nc),) if fine else ()):
            for _, w_off, b_off, fin, fout in arch.flat_layout():
                grads.append(flat_grad[base + w_off: base + w_off + fin * fout].view(fout, fin))
                grads.append(flat_grad[base + b_off: base + b_off + fout])
        return (None,) * 3 + tuple(grads)


class _RunNetwork(torch.autograd.Function):
    """The MLP at caller-given points (ops.mlp_fwd_pts) and its parameter backward."""

    @staticmethod
    def forward(ctx, cfg, pts, dirs, *params):
        arch, blob, training, impl = cfg
        if not training:
            return ops.mlp_fwd_pts(arch, blob, pts, dirs, impl=impl)
        raw, stash = ops.mlp_fwd_pts(arch, blob, pts, dirs, impl=impl, want_stash=True)
        ctx.cfg, ctx.stash, ctx.dirs = cfg, stash, dirs
        return raw

    @staticmethod
    def backward(ctx, g):
        arch, blob, training, impl = ctx.cfg
        flat_grad = ops.mlp_bwd_pts(arch, blob, ctx.dirs, g.contiguous(), ctx.stash, impl=impl)
        ctx.stash = ctx.dirs = None
        # a step may query the network any number of times: its gradients are summed by autograd and reduced once by
        # parallel.sync_gradients / FusedAdam.step (which only clear the flag when gradient sync is off)
        global _PENDING_SYNC
        _PENDING_SYNC = True
        grads = []
        for _, w_off, b_off, fin, fout in arch.flat_layout():
            grads.append(flat_grad[w_off: w_off + fin * fout].view(fout, fin))
            grads.append(flat_grad[b_off: b_off + fout])
        return (None,) * 3 + tuple(grads)


# --------------------------------------------------------------------------------------------------
# public API
# --------------------------------------------------------------------------------------------------
def run_network(network_fn, pts, ray_batch, chunksize, embed_fn, embeddirs_fn, *, impl: Optional[int] = None):
    """nerf/train_utils.py:8-25: ``network_fn`` (a FlexibleNeRFModel) on the positional encodings of caller-chosen
    points, fused in one kernel.  ``pts`` (*B, S, 3); with ``embeddirs_fn`` every point of row b takes the view
    direction ``ray_batch[b, -3:]`` (``ray_batch`` (*B, C), C >= 3, read in place).  Without view directions ``pts``
    may have any leading shape.  Returns ``pts.shape[:-1] + (4,)`` fp32, differentiable w.r.t. the parameters of
    ``network_fn`` (not w.r.t. ``pts``).  ``chunksize`` is accepted; the result does not depend on it.

    ``impl``: as in ``predict_and_render_radiance``, with S samples per row."""
    impl = _requested_impl(impl, network_fn)
    if not pts.is_cuda or (embeddirs_fn is not None and not ray_batch.is_cuda):
        raise NotImplementedError("nerfb200: points and rays must be on a CUDA device (there is no CPU path)")
    if torch.is_grad_enabled() and pts.requires_grad:
        raise NotImplementedError("nerfb200: run_network gives no gradient w.r.t. the points; detach them")
    if pts.dim() < 1 or pts.shape[-1] != 3:
        raise ValueError(f"nerfb200: pts must be (..., 3), got shape {tuple(pts.shape)}")
    enc_xyz = _probe_encoder(embed_fn, None)
    if enc_xyz is None:
        raise RuntimeError("nerfb200: embed_fn is required (the reference crashes without it too)")
    arch = _arch_of(network_fn, enc_xyz, _probe_encoder(embeddirs_fn, None))
    out_shape = tuple(pts.shape[:-1]) + (4,)
    dirs = None
    if embeddirs_fn is not None:
        # the reference expands ray_batch[..., None, -3:] to pts.shape
        lead = tuple(pts.shape[:-2])
        if pts.dim() < 2 or tuple(ray_batch.shape[:-1]) != lead or ray_batch.shape[-1] < 3:
            raise ValueError(f"nerfb200: ray_batch {tuple(ray_batch.shape)} does not match pts {tuple(pts.shape)}: "
                             "need pts (*B, S, 3) and ray_batch (*B, C >= 3)")
        n_rays, n_samples = math.prod(lead), pts.shape[-2]
        if arch.use_viewdirs:
            d = ray_batch.detach()[..., -3:].float()
            try:
                dirs = d.view(n_rays, 3)
            except RuntimeError:  # rows not evenly spaced in memory
                dirs = d.reshape(n_rays, 3)
            if dirs.stride(1) != 1:
                dirs = dirs.contiguous()
    else:
        # no direction per row: the grouping into rows is free, so one row of all the points
        n_rays, n_samples = 1, pts.numel() // 3
    if n_rays * n_samples == 0:
        raise ValueError("nerfb200: run_network on an empty point set")
    params, blob = _packed(network_fn, arch)
    training = _trains(params)
    if impl is None:
        impl = _auto_impl(arch, None, n_samples, 0, training)
    p = pts.detach().float().contiguous().view(n_rays, n_samples, 3)
    raw = _RunNetwork.apply((arch, blob, training, impl), p, dirs, *params)
    return raw.view(out_shape)



def check_grid_call(grid, device, *models):
    """The refusals of an occupancy-grid render that precede any launch: not an OccupancyGrid, a call that would train,
    a grid on another device than ``device`` (None: not known yet) or whose bits are not the int32 words its resolution
    needs."""
    from .occupancy import OccupancyGrid

    if not isinstance(grid, OccupancyGrid):
        raise TypeError(f"nerfb200: grid must be an OccupancyGrid, got {type(grid).__name__}")
    if _trains(p for m in models if m is not None for p in m.parameters()):
        raise NotImplementedError("nerfb200: an occupancy grid renders only (inference); render under torch.no_grad() "
                                  "or with parameters that do not require grad")
    bits = grid.bits
    if device is not None and bits.device != torch.device(device):
        raise RuntimeError(f"nerfb200: the occupancy grid is on {bits.device}, the rays on {device}")
    want = ops.grid_words(grid.c_struct())
    if bits.dtype != torch.int32 or bits.dim() != 1 or bits.numel() != want or not bits.is_contiguous():
        raise RuntimeError(f"nerfb200: the occupancy grid's bits must be contiguous int32[{want}], got {bits.dtype}"
                           f"{list(bits.shape)}")


def _inference_impl(feature, render, impl, arch_c, arch_f, nc, nf):
    """The impl a grid or early-stopping render runs on, after the refusals that precede a launch: impl 0 and an
    architecture the wgmma inference forward refuses (the library's reason).  ``feature`` names the option in the impl 0
    refusal ("an occupancy grid"), ``render`` the render in the library's ("grid render")."""
    if impl is None:
        impl = _auto_impl(arch_c, arch_f, nc, nf, training=False)
    if impl == ops.IMPL_SIMT:
        raise NotImplementedError(f"nerfb200: {feature} runs on the wgmma inference forward (impl 1 or 3), not "
                                  "impl 0 (fp32 CUDA cores)" + "".join(
                                      f"; {why}" for a, n in ((arch_c, nc), (arch_f, nc + nf)) if a is not None
                                      for why in [ops.impl_refusal(a, n, ops.IMPL_TC_FWD)] if why))
    for a, n in ((arch_c, nc), (arch_f, nc + nf)):
        why = ops.impl_refusal(a, n, ops.IMPL_TC_FWD if impl == ops.IMPL_TC else impl) if a is not None else None
        if why:
            raise NotImplementedError(f"nerfb200 {render}: {why}")
    return impl


def check_early_stop_call(early_stop, *models):
    """The refusals of an early-stopping render that precede any launch: a threshold that is not a number in [0, 1), a
    call that would train."""
    if isinstance(early_stop, bool) or not isinstance(early_stop, numbers.Real) or not 0.0 <= float(early_stop) < 1.0:
        raise ValueError(f"nerfb200: early_stop must be a transmittance threshold in [0, 1), got {early_stop!r}")
    if _trains(p for m in models if m is not None for p in m.parameters()):
        raise NotImplementedError("nerfb200: early ray termination renders only (inference); render under "
                                  "torch.no_grad() or with parameters that do not require grad")


def check_normals_call(impl, *models):
    """The refusals of a normal-map render that need no architecture: a call that would train, impl 0 or 3."""
    if _trains(p for m in models if m is not None for p in m.parameters()):
        raise NotImplementedError("nerfb200: normal maps render only (inference); render under torch.no_grad() or with "
                                  "parameters that do not require grad")
    if impl is not None and int(impl) != ops.IMPL_TC:
        raise NotImplementedError(f"nerfb200: normal maps run on the wgmma kernels (impl 1), not impl={int(impl)}: the "
                                  "density gradient is built for impl 1 alone")


def normals_mode(normals):
    """The ``normals=`` of the render entry points: "world", or its truth value (ValueError for any other string)."""
    if isinstance(normals, str):
        if normals != "world":
            raise ValueError(f"nerfb200: normals must be False, True or \"world\", got {normals!r}")
        return normals
    return bool(normals)


def _world_ndc(normals, options, ndc):
    """The NDC camera of a ``normals="world"`` render of NDC ``options`` (None otherwise: the MLP's frame is world
    space already); ValueError when such a render has no (H, W, focal) to map with."""
    if normals != "world" or getattr(getattr(options, "dataset", None), "no_ndc", True) is not False:
        return None
    if ndc is None:
        raise ValueError("nerfb200: normals=\"world\" on an NDC scene needs the image's H, W and focal, which "
                         "predict_and_render_radiance's packed rays do not carry; call run_one_iter_of_nerf or "
                         "render_image")
    from .density import ndc_camera

    return ndc_camera(ndc)


def _normals_impl(impl, arch_c, arch_f, nc, nf):
    """impl 1, after the library's refusal of the last pass's density gradient (the render's own come from the library
    before its first launch)."""
    impl = ops.IMPL_TC if impl is None else int(impl)
    last = arch_f if nf > 0 else arch_c
    why = ops.density_grad_refusal(last, impl)
    if why:
        raise NotImplementedError(f"nerfb200 normal-map render: {why}")
    return impl


def predict_and_render_radiance(
    ray_batch,
    model_coarse,
    model_fine,
    options,
    mode="train",
    encode_position_fn=None,
    encode_direction_fn=None,
    *,
    randoms: Union[dict, SeededRandoms, None] = None,
    impl: Optional[int] = None,
    grid=None,
    early_stop: Optional[float] = None,
    normals: Union[bool, str] = False,
    _n_chunks: int = 1,
    _ndc=None,
):
    """nerf/train_utils.py:28-127 for one chunk of packed rays ``[o d near far (viewdir)]``.

    ``randoms`` (keyword-only, optional) injects the four random tensors the reference would draw
    (t_rand, noise_c, u, noise_f); by default they are drawn here with torch.rand/randn in the
    reference's order.  A ``SeededRandoms`` instead has the kernels generate them from its seed, step and
    ``ray_offset`` (the global index of ``ray_batch[0]``): no torch random number is drawn.

    ``impl``: None picks the kernels (``DEFAULT_IMPL``, else the automatic choice); ``ops.IMPL_TC_FAST`` renders with
    the single-pass fp16 forward and raises ``NotImplementedError`` if the call would train.

    ``grid``: an ``OccupancyGrid`` on the rays' device (inference only, impl 1 or 3): samples in its empty cells skip
    the MLP and get zero density.  None is the path without a grid.

    ``early_stop``: a transmittance threshold t in [0, 1) (inference only, impl 1 or 3, with or without ``grid``): the
    last pass stops a ray once its transmittance falls below t, so its rgb and acc move by at most t
    (include/nerfb200.h "early ray termination").  None is the path without it.

    ``normals``: also return the last pass's normal map N (n_rays, 3) as a seventh output (inference only, impl 1,
    with or without ``grid`` / ``early_stop``): the sum of the compositing weights times the outward unit normals
    -grad sigma / |grad sigma| at the pass's samples (include/nerfb200.h "normal maps"); not renormalised, so |N| <=
    acc.  False returns exactly the six outputs.  ``normals="world"`` is the normal map in world space: for a Blender
    scene the same as True; for an NDC scene (``options.dataset.no_ndc`` false) it needs the image's H, W and focal,
    which packed rays do not carry, so it is refused here (ValueError): ``run_one_iter_of_nerf`` and ``render_image``
    provide it."""
    normals = normals_mode(normals)
    cam = _world_ndc(normals, options, _ndc)
    impl = _requested_impl(impl, model_coarse, model_fine)
    if normals:
        check_normals_call(impl, model_coarse, model_fine)
    if grid is not None:
        check_grid_call(grid, ray_batch.device, model_coarse, model_fine)
    if early_stop is not None:
        check_early_stop_call(early_stop, model_coarse, model_fine)
    o = getattr(options.nerf, mode)
    if not ray_batch.is_cuda:
        raise NotImplementedError("nerfb200: rays must be on a CUDA device (there is no CPU path)")
    rays = ray_batch.detach().float().contiguous()
    n, dev = rays.shape[0], rays.device
    enc_xyz = _probe_encoder(encode_position_fn, None)
    if enc_xyz is None:
        raise RuntimeError("nerfb200: encode_position_fn is required (the reference crashes without it too)")
    enc_dir = _probe_encoder(encode_direction_fn, None)
    nc, nf = int(o.num_coarse), int(o.num_fine)
    fine = nf > 0
    arch_c = _arch_of(model_coarse, enc_xyz, enc_dir)
    if fine and not model_fine:
        raise RuntimeError("nerfb200: num_fine > 0 but model_fine is None (the reference fails here as well)")
    arch_f = _arch_of(model_fine, enc_xyz, enc_dir) if fine else None
    if grid is not None:
        impl = _inference_impl("an occupancy grid", "grid render", impl, arch_c, arch_f, nc, nf)
    elif early_stop is not None:
        impl = _inference_impl("early ray termination", "early-stopping render", impl, arch_c, arch_f, nc, nf)
    if normals:
        impl = _normals_impl(impl, arch_c, arch_f, nc, nf)
    params_c, blob_c = _packed(model_coarse, arch_c)
    params_f, blob_f = _packed(model_fine, arch_f) if fine else ([], None)
    noise_std = float(o.radiance_field_noise_std)
    perturb = bool(o.perturb)
    opts = ops.make_opts(nc, nf, perturb, o.lindisp, o.white_background, noise_std)

    rnd = randoms
    if not isinstance(randoms, SeededRandoms):  # seeded: the kernels generate all four
        given = randoms or {}

        def take(name, shape, fn):
            t = given.get(name)
            if t is None:
                return fn(shape, dtype=torch.float32, device=dev)
            return t.to(device=dev, dtype=torch.float32).contiguous()

        # reference draw order: rand(N,Nc) -> randn(N,Nc) -> rand(N,Nf) -> randn(N,Nc+Nf)  (SURVEY section 5); with
        # perturb off the fine pass resamples at the det=True linspace, which the kernel builds (nerf_helpers.py:272-276)
        rnd = {}
        if perturb:
            rnd["t_rand"] = take("t_rand", (n, nc), torch.rand)
        if noise_std > 0.0:
            rnd["noise_c"] = take("noise_c", (n, nc), torch.randn)
        if fine and perturb:
            rnd["u"] = take("u", (n, nf), torch.rand)
        if fine and noise_std > 0.0:
            rnd["noise_f"] = take("noise_f", (n, nc + nf), torch.randn)

    all_params = list(params_c) + list(params_f)
    training = _trains(all_params)
    if impl is None:
        impl = _auto_impl(arch_c, arch_f, nc, nf, training)
    nrm = None
    if normals:
        out_c, out_f, nrm, _ = ops.render_fwd_normals(arch_c, arch_f, opts, blob_c, blob_f, rays, rnd, grid,
                                                   None if early_stop is None else float(early_stop), impl=impl,
                                                   ndc=cam)
    elif early_stop is not None:
        out_c, out_f, _ = ops.render_fwd_early_stop(arch_c, arch_f, opts, blob_c, blob_f, rays, rnd, grid,
                                                    float(early_stop), impl=impl)
    elif grid is not None:
        out_c, out_f, _ = ops.render_fwd_grid(arch_c, arch_f, opts, blob_c, blob_f, rays, rnd, grid, impl=impl)
    else:
        cfg = (arch_c, arch_f, opts, blob_c, blob_f, training, impl, int(_n_chunks))
        out_c, out_f = _RenderChunk.apply(cfg, rays, rnd, *all_params)
    rgb_c, disp_c, acc_c = out_c[:, :3], out_c[:, 3], out_c[:, 4]
    six = (rgb_c, disp_c, acc_c) + ((None, None, None) if out_f is None else (out_f[:, :3], out_f[:, 3], out_f[:, 4]))
    return six + (nrm,) if normals else six


def run_one_iter_of_nerf(
    height,
    width,
    focal_length,
    model_coarse,
    model_fine,
    ray_origins,
    ray_directions,
    options,
    mode="train",
    encode_position_fn=None,
    encode_direction_fn=None,
    *,
    randoms: Union[dict, SeededRandoms, None] = None,
    impl: Optional[int] = None,
    grid=None,
    early_stop: Optional[float] = None,
    normals: Union[bool, str] = False,
):
    """nerf/train_utils.py:130-202: ray packing (viewdirs, optional NDC, near/far), chunking by
    ``options.nerf.<mode>.chunksize``, per-chunk render, concatenation and -- in "validation" mode --
    the reshape back to image shape.  ``normals=True`` appends the normal map of the last pass (see
    ``predict_and_render_radiance``) as a seventh output; ``normals="world"`` gives it in world space, for an NDC
    scene through the NDC map of ``height``, ``width`` and ``focal_length`` (include/nerfb200.h "NDC scenes")."""
    normals = normals_mode(normals)
    ndc = (height, width, focal_length) if normals == "world" else None
    if ndc is not None:
        _world_ndc(normals, options, ndc)  # a malformed camera is refused before any launch
    impl = _requested_impl(impl, model_coarse, model_fine)
    if normals:
        check_normals_call(impl, model_coarse, model_fine)
    if grid is not None:
        check_grid_call(grid, ray_directions.device, model_coarse, model_fine)
    if early_stop is not None:
        check_early_stop_call(early_stop, model_coarse, model_fine)
    use_viewdirs = bool(options.nerf.use_viewdirs)
    restore_shapes = [ray_directions.shape, ray_directions.shape[:-1], ray_directions.shape[:-1]]
    if model_fine:
        restore_shapes += restore_shapes
    if not ray_directions.is_cuda:
        raise NotImplementedError("nerfb200: rays must be on a CUDA device (there is no CPU path)")
    # view directions (from the pre-NDC directions), optional NDC warp, near / far columns and the row layout
    # [o d near far viewdir]: one kernel (csrc/raygen.cu), same op order as the reference's chain of torch ops
    rays = ops.pack_rays(ray_origins.reshape(-1, 3).float().contiguous(), ray_directions.reshape(-1, 3).float().contiguous(),
                         height, width, focal_length, options.dataset.no_ndc is False, options.dataset.near,
                         options.dataset.far, use_viewdirs)

    return _render_packed(rays, restore_shapes, model_coarse, model_fine, options, mode, encode_position_fn,
                          encode_direction_fn, randoms, impl, grid, early_stop, normals, ndc)


def run_one_iter_of_nerf_from_pose(
    height,
    width,
    focal_length,
    model_coarse,
    model_fine,
    tform_cam2world,
    pixel_ids,
    options,
    mode="train",
    encode_position_fn=None,
    encode_direction_fn=None,
    *,
    randoms: Union[dict, SeededRandoms, None] = None,
    impl: Optional[int] = None,
    grid=None,
    early_stop: Optional[float] = None,
):
    """``run_one_iter_of_nerf`` for callers that hold a pose and pixel ids instead of ray tensors (SURVEY.md section 8f-2):
    the reference's training loop builds ALL H*W rays of the image with get_ray_bundle and then indexes the few
    thousand it samples (train_nerf.py:196-226); here the rays of exactly those pixels are generated on the device
    (csrc/raygen.cu) in the packed layout the render kernels read.  ``pixel_ids``: int64, ``j * width + i``, on the
    target device (None = the whole image, returned image-shaped in "validation" mode)."""
    impl = _requested_impl(impl, model_coarse, model_fine)
    dev = pixel_ids.device if pixel_ids is not None else next(model_coarse.parameters()).device
    if grid is not None:
        check_grid_call(grid, dev, model_coarse, model_fine)
    if early_stop is not None:
        check_early_stop_call(early_stop, model_coarse, model_fine)
    use_viewdirs = bool(options.nerf.use_viewdirs)
    rays = ops.gen_rays(tform_cam2world, height, width, focal_length, pixel_ids, dev, ndc=options.dataset.no_ndc is False,
                        near=options.dataset.near, far=options.dataset.far, use_viewdirs=use_viewdirs)
    lead = (height, width) if pixel_ids is None else tuple(pixel_ids.shape)
    restore_shapes = [lead + (3,), lead, lead] * (2 if model_fine else 1)
    return _render_packed(rays, restore_shapes, model_coarse, model_fine, options, mode, encode_position_fn,
                          encode_direction_fn, randoms, impl, grid, early_stop)


def _render_packed(rays, restore_shapes, model_coarse, model_fine, options, mode, encode_position_fn, encode_direction_fn,
                   randoms, impl, grid=None, early_stop=None, normals=False, ndc=None):
    """Chunking, per-chunk render, concatenation and the validation reshape of train_utils.py:170-202.
    Seeded randoms follow each ray: chunk i starts at ``ray_offset`` + the index of its first ray."""
    chunksize = getattr(options.nerf, mode).chunksize
    batches = get_minibatches(rays, chunksize=chunksize)
    seeded = isinstance(randoms, SeededRandoms)
    if randoms is not None and not seeded and len(batches) != 1:
        raise ValueError("injected randoms require a single ray chunk")
    inner_mode = "train" if COMPAT_MODE_QUIRK else mode
    pred = [
        predict_and_render_radiance(
            batch, model_coarse, model_fine, options, mode=inner_mode,
            encode_position_fn=encode_position_fn,
            encode_direction_fn=encode_direction_fn if options.nerf.use_viewdirs else None,
            randoms=randoms.shifted(i * chunksize) if seeded else randoms, impl=impl, grid=grid,
            early_stop=early_stop, normals=normals, _n_chunks=len(batches), _ndc=ndc,
        )
        for i, batch in enumerate(batches)
    ]
    nrm = None
    if normals:
        nrm = torch.cat([p[6] for p in pred], dim=0)
        if mode == "validation":
            nrm = nrm.view(restore_shapes[0])
        pred = [p[:6] for p in pred]
    synthesized_images = list(zip(*pred))
    synthesized_images = [
        torch.cat(image, dim=0) if image[0] is not None else None for image in synthesized_images
    ]
    if mode == "validation":
        synthesized_images = [
            image.view(shape) if image is not None else None
            for (image, shape) in zip(synthesized_images, restore_shapes)
        ]
        if not model_fine:
            synthesized_images = synthesized_images + [None, None, None]
    return tuple(synthesized_images) + ((nrm,) if normals else ())
