"""Baked fields: a trained FlexibleNeRFModel evaluated once on the lattice points of the bricks an occupancy grid calls
occupied -- raw density plus degree-2 spherical-harmonic coefficients of its rgb logits over 64 view directions -- and
rendered by trilinear interpolation of those values, without the MLP (PlenOctrees- / SNeRG-style baking).

The bricks are the sparse meshes' (include/nerfb200.h "sparse meshes"), the values and the renderer are defined in
include/nerfb200.h "baked fields"; the bake is one fused wgmma kernel (csrc/mlp_tc.cu, bake_tc_kernel) and the renderer
one warp per ray (csrc/baked.cu).  A baked field can be fine-tuned against images through that renderer
(render_baked_rays, BakedFieldTrainer; include/nerfb200.h "baked fields: gradients and fine-tuning"), and pruned to the
bricks its renders use (baked_transparent_bricks, baked_brick_weights, prune_baked, BakedFieldTrainer.prune;
include/nerfb200.h "baked fields: pruning"), with total-variation and sparsity regularisers over the lattice
(baked_regularizer, BakedFieldTrainer's tv_sigma / tv_sh / sparsity; include/nerfb200.h "baked fields: regularisers").  This file validates arguments, sizes buffers and moves
pointers; the bake reads the active brick count back once to size its values.  A field can also start without a network
(``BakedField.full``) and be trained coarse to fine: train, prune, then subdivide to twice the resolution holding the
same trilinear function (subdivide_baked, BakedFieldTrainer.subdivide; include/nerfb200.h "baked fields:
subdivision").  A field kept, saved, rendered or pruned
may store its values in fp16 (``bake(dtype=torch.float16)``, ``BakedField.half``; include/nerfb200.h "baked fields: half
precision") or as 8-bit codes with a per-channel scale and offset (``BakedField.quantize``; include/nerfb200.h "baked
fields: 8-bit values"); fine-tuning, the regularisers and subdivision take fp32 fields only (``BakedField.float``).  Any
field, fp32, fp16 or 8-bit, can be meshed without a network (extract_baked_mesh; include/nerfb200.h "baked fields:
meshes"), rendered as a normal map (render_baked(normals=), render_baked_rays(normals=)) and probed point by point
(baked_raw, baked_density_gradient; include/nerfb200.h "baked fields: normal maps and point queries")."""
from __future__ import annotations

import math

import torch

from . import ops

_LOSSY = {torch.float16: ("an fp16 field", "convert it back with .half()"),
          torch.uint8: ("an 8-bit field", "quantise it again with .quantize()")}


def _lossy_refusal(what, dtype, lacks, fix="fine-tune field.float() and {back}"):
    """The ValueError of ``what`` for a ``dtype`` field, which has no ``lacks``; ``fix`` may name its way ``{back}``."""
    name, back = _LOSSY[dtype]
    return ValueError(f"{what}: {name} has no {lacks}; {fix.format(back=back)}")


def _widened(field, rows, ch):
    """fp32 channels ``ch`` of slots ``rows``, 8-bit codes dequantised as the kernels read them: q.float() * s + o."""
    v = field.values.detach()[rows, :, ch].float()
    return v * field.dequant[0, ch] + field.dequant[1, ch] if field.dtype == torch.uint8 else v


class BakedField:
    """A baked field on the device: ``bounds`` ((lo), (hi)) and ``resolution`` (three ints) of the lattice box,
    ``brick_map`` int32[bricks] (slot or -1), ``bricks`` int32[n_active] (slot -> brick), ``values``
    fp32[n_active, 729, 32], fp16 of that shape (include/nerfb200.h "baked fields: half precision") or uint8 codes of
    that shape, ``use_viewdirs`` (whether the network had view directions) and ``dequant``: for uint8 codes the fp32
    (2, 28) table of per-channel scales and offsets on the values' device (include/nerfb200.h "baked fields: 8-bit
    values"), None otherwise."""

    def __init__(self, bounds, resolution, brick_map, bricks, values, use_viewdirs: bool, *, dequant=None):
        self.bounds = (tuple(float(v) for v in bounds[0]), tuple(float(v) for v in bounds[1]))
        self.resolution = tuple(int(r) for r in resolution)
        self.brick_map = brick_map
        self.bricks = bricks
        self.values = values
        self.use_viewdirs = bool(use_viewdirs)
        self.dequant = dequant

    @classmethod
    def full(cls, bounds, resolution, *, sigma_raw=0.1, use_viewdirs=True, device="cuda") -> "BakedField":
        """A field on every brick of the lattice box ``bounds`` / ``resolution`` (checked as ``bake`` checks them),
        ``brick_map`` and ``bricks`` the identity, ``sigma_raw`` at every lattice point and every SH coefficient 0 (grey:
        sigmoid(0) = 0.5).  fp32.  The networkless starting point of a coarse-to-fine fit, as ``OccupancyGrid.full`` is
        of a grid.  The renderer's density is relu(sigma_raw), whose gradient is 0 at sigma_raw <= 0, so a start that can
        learn density is positive.  A non-finite ``sigma_raw`` raises ValueError."""
        from .mesh import _box

        lo, hi, res = _box(bounds, resolution, dense=False)
        sigma = float(sigma_raw)
        if not math.isfinite(sigma):
            raise ValueError(f"BakedField.full: sigma_raw must be finite, got {sigma_raw!r}")
        n = math.prod(-(-r // 8) for r in res)
        ids = torch.arange(n, dtype=torch.int32, device=device)
        values = torch.zeros(n, 729, 32, dtype=torch.float32, device=device)
        values[..., 0] = sigma
        return cls((lo, hi), res, ids, ids.clone(), values, use_viewdirs)

    @property
    def n_active(self) -> int:
        return int(self.values.shape[0])

    @property
    def dtype(self) -> torch.dtype:
        """The values' dtype: torch.float32, torch.float16 or torch.uint8."""
        return self.values.dtype

    def box(self):
        return ops.grid_struct(self.bounds, self.resolution)

    def half(self, chunk: int = 1024) -> "BakedField":
        """A new field with fp16 values under the conversion rule (include/nerfb200.h "baked fields: half precision"): a
        finite value saturates to +-65504 and rounds to nearest even, +-inf and NaN stay.  Converted ``chunk`` slots at a
        time, so the peak is both fields plus one chunk's temporaries; ``brick_map`` and ``bricks`` are shared.  Renders
        and peak weights of the result are bit for bit those of ``result.float()``.  Works on a CPU field too."""
        chunk = int(chunk)
        if chunk < 1:
            raise ValueError(f"BakedField.half: chunk must be >= 1, got {chunk}")
        if self.dtype == torch.uint8:
            raise _lossy_refusal("BakedField.half", self.dtype, "fp16 conversion", "dequantise it with .float() first")
        v = self.values.detach()
        out = torch.empty(v.shape, dtype=torch.float16, device=v.device)
        for s in range(0, self.n_active, chunk):
            c = v[s:s + chunk]
            out[s:s + chunk] = torch.where(c.isfinite(), c.clamp(-65504.0, 65504.0), c)  # the copy rounds to nearest even
        return BakedField(self.bounds, self.resolution, self.brick_map, self.bricks, out, self.use_viewdirs)

    def quantize(self, chunk: int = 1024) -> "BakedField":
        """A new 8-bit field under the quantisation rule (include/nerfb200.h "baked fields: 8-bit values"): per channel
        c = 0 .. 27 the range [min(0, min v), max(0, max v)] over every stored value, scale s_c = range / 255 (1 for an
        empty range), zero point z_c = clamp(rint(-lo_c / s_c), 0, 255) (an integer: 0 is +0), offset o_c = -(z_c s_c)
        and codes clamp(rint((v - o_c) / s_c), 0, 255), each op rounded to fp32; channels 28 .. 31 hold 0.  A CUDA field
        and its CPU copy give the same codes and dequant bits.  An fp16 field is widened exactly first, so its codes are
        those of ``field.float().quantize()``.  Two passes of ``chunk`` slots (the range, then
        the codes), so the peak is both fields plus one chunk's temporaries; ``brick_map`` and ``bricks`` are shared.
        Renders, peak weights and meshes of the result are bit for bit those of ``result.float()``.  Reads the range
        back once.  ValueError for a non-finite value in channels 0 .. 27, a range that overflows fp32, or an 8-bit
        field.  Works on a CPU field too."""
        chunk = int(chunk)
        if chunk < 1:
            raise ValueError(f"BakedField.quantize: chunk must be >= 1, got {chunk}")
        if self.dtype == torch.uint8:
            raise _lossy_refusal("BakedField.quantize", self.dtype, "requantisation",
                                 "dequantise it with .float() first")
        v = self.values.detach()
        lo = torch.zeros(28, dtype=torch.float32, device=v.device)
        hi = torch.zeros(28, dtype=torch.float32, device=v.device)
        for s in range(0, self.n_active, chunk):
            c = v[s:s + chunk, :, :28].float().reshape(-1, 28)
            lo = torch.minimum(lo, c.amin(0))  # NaN propagates, so the finiteness check below sees it
            hi = torch.maximum(hi, c.amax(0))
        # a tensor divisor: torch's CUDA division by a Python scalar multiplies by its rounded reciprocal, which is not
        # the rule's correctly rounded (hi - lo) / 255
        scale = (hi - lo) / torch.full_like(hi, 255.0)
        if not bool(torch.isfinite(torch.cat([lo, hi, scale])).all()):
            raise ValueError("BakedField.quantize: channels 0 .. 27 must be finite and their range must fit in fp32")
        scale = torch.where(scale == 0, torch.ones_like(scale), scale)
        zero = torch.round(-lo / scale).clamp(0, 255)
        zero = torch.where(zero == 0, torch.zeros_like(zero), zero)  # the integer 0 as +0 (clamp may keep a -0)
        offset = -(zero * scale)
        out = torch.zeros(v.shape, dtype=torch.uint8, device=v.device)
        for s in range(0, self.n_active, chunk):
            c = v[s:s + chunk, :, :28].float()
            out[s:s + chunk, :, :28] = torch.round((c - offset) / scale).clamp(0, 255).to(torch.uint8)
        return BakedField(self.bounds, self.resolution, self.brick_map, self.bricks, out, self.use_viewdirs,
                          dequant=torch.stack([scale, offset]))

    def float(self, chunk: int = 1024) -> "BakedField":
        """A field with fp32 values: an fp16 field widened exactly (a new tensor), an 8-bit field dequantised exactly
        under its rule, q.float() * s + o, ``chunk`` slots at a time (a new tensor, channels 28 .. 31 zero), an fp32
        field's own values tensor.  ``brick_map`` and ``bricks`` are shared.  Fine-tune ``field.float()``, then convert
        back with ``half()`` or ``quantize()``."""
        if self.values.dtype == torch.uint8:
            chunk = int(chunk)
            if chunk < 1:
                raise ValueError(f"BakedField.float: chunk must be >= 1, got {chunk}")
            v = torch.zeros(self.values.shape, dtype=torch.float32, device=self.values.device)
            for s in range(0, self.n_active, chunk):
                v[s:s + chunk, :, :28] = _widened(self, slice(s, s + chunk), slice(0, 28))
        else:
            v = self.values if self.values.dtype == torch.float32 else self.values.detach().float()
        return BakedField(self.bounds, self.resolution, self.brick_map, self.bricks, v, self.use_viewdirs)

    def __repr__(self):
        return (f"BakedField({self.n_active} bricks of {ops.mesh_sparse_brick_count(self.box())}, "
                f"{self.values.numel() * self.values.element_size() / 2 ** 20:.1f} MiB"
                f"{' fp16' if self.dtype == torch.float16 else ' 8-bit' if self.dtype == torch.uint8 else ''}, "
                f"resolution {self.resolution}"
                f"{', view directions' if self.use_viewdirs else ''})")

    def save(self, path) -> None:
        """Writes the field with torch.save; the values keep their dtype, an 8-bit field its ``dequant``."""
        torch.save({"bounds": self.bounds, "resolution": self.resolution, "brick_map": self.brick_map.cpu(),
                    "bricks": self.bricks.cpu(), "values": self.values.cpu(), "use_viewdirs": self.use_viewdirs,
                    "dequant": None if self.dequant is None else self.dequant.cpu()}, path)

    @classmethod
    def load(cls, path, device="cuda") -> "BakedField":
        """A field written by ``save``; a file without ``dequant`` (written before 8-bit fields) loads with None."""
        d = torch.load(path, map_location="cpu", weights_only=True)
        dq = d.get("dequant")
        return cls(d["bounds"], d["resolution"], d["brick_map"].to(device), d["bricks"].to(device),
                   d["values"].to(device), d["use_viewdirs"], dequant=None if dq is None else dq.to(device))


def bake(model, encode_position_fn, encode_direction_fn=None, *, bounds, resolution, grid,
         dtype=torch.float32) -> BakedField:
    """Bake ``model`` (the network that renders the final image: pass ``model_fine``) over the lattice box ``bounds``
    / ``resolution`` (as ``extract_mesh``; up to 4096 cubes per axis) on the bricks ``grid`` (an ``nb.OccupancyGrid`` on
    the model's device) calls occupied, under the sparse meshes' activity rule.  The field lives in the coordinates the
    MLP encodes: world space for Blender scenes, NDC for LLFF scenes.  ``dtype`` torch.float16 stores the values in
    half precision straight from the kernel (the conversion rule of ``BakedField.half`` at the store: the bits of
    ``bake(...).half()``, at half the memory and without an fp32 copy).  Argument errors raise ValueError, an
    architecture the wgmma inference forward refuses NotImplementedError, before any launch."""
    from . import train_utils
    from .mesh import _box, _check_grid, _network

    if dtype not in (torch.float32, torch.float16):
        raise ValueError(f"bake: dtype must be torch.float32 or torch.float16, got {dtype!r}")
    lo, hi, res = _box(bounds, resolution, dense=False)
    arch = _network(model, encode_position_fn, encode_direction_fn)
    dev = next(model.parameters()).device
    _check_grid(grid, dev)
    why = ops.bake_refusal(arch)
    if why is not None:
        raise NotImplementedError(f"nerfb200 bake: {why}")
    _, blob = train_utils._packed(model, arch)
    box = ops.grid_struct((lo, hi), res)
    brick_map, bricks, n_dev = ops.mesh_sparse_bricks(box, grid)
    n_active = int(n_dev.item())
    values = torch.empty(n_active, 729, 32, dtype=dtype, device=dev)
    if n_active:
        with torch.no_grad():
            ops.bake(arch, blob, box, bricks, 0, n_active, values)
    return BakedField((lo, hi), res, brick_map, bricks[:n_active].clone(), values, arch.use_viewdirs)


def render_baked(field: BakedField, height, width, focal_length, tform_cam2world, options, mode="validation", *,
                 early_stop=None, normals=False):
    """(rgb (H, W, 3), disp (H, W), acc (H, W)) of ``field`` seen from the pose ``tform_cam2world``.  The rays are
    ``render_image``'s: ``ops.gen_rays`` with ``options.dataset`` near / far / no_ndc and ``options.nerf.use_viewdirs``
    (which must match the baked network), and the white background of ``options.nerf.<mode>`` (``options.nerf.train``
    while ``train_utils.COMPAT_MODE_QUIRK`` holds, as ``render_image``).  Samples are spaced half the smallest cube side
    apart along each ray inside the box.  ``early_stop`` t in [0, 1) stops a ray once its transmittance falls below t
    (checked every 32 samples); a ray that never stops is bit for bit the render without it.

    ``normals=True`` appends the normal map (H, W, 3) in the field's frame: per pixel the sum over its samples of
    w (-g / |g|), g the gradient of the trilinear sigma_raw (include/nerfb200.h "baked fields: normal maps and point
    queries"); the first three outputs stay bit for bit those without it.  ``normals="world"`` gives it in world space:
    for an NDC field (``options.dataset.no_ndc`` false) through the NDC map of this call's ``height``, ``width`` and
    ``focal_length``, for a Blender field the same as True.  ``cast_to_normal_image`` turns it into an image."""
    from . import train_utils

    if not isinstance(field, BakedField):
        raise ValueError(f"render_baked: field must be an nb.BakedField, got {type(field).__name__}")
    normals = train_utils.normals_mode(normals)
    cam = train_utils._world_ndc(normals, options, (height, width, focal_length))
    if not field.values.is_cuda:
        raise NotImplementedError("nerfb200: the baked field must be on a CUDA device (there is no CPU path)")
    _check_viewdirs(field, options, "render_baked")
    stop = 0.0
    if early_stop is not None:
        stop = float(early_stop)
        if not 0.0 <= stop < 1.0:
            raise ValueError(f"render_baked: early_stop must lie in [0, 1), got {early_stop!r}")
    white = getattr(options.nerf, "train" if train_utils.COMPAT_MODE_QUIRK else mode).white_background
    rays = _pose_rays(field, height, width, focal_length, tform_cam2world, options)
    values = field.values if field.n_active else field.values.new_zeros(1, 729, 32)
    if normals:
        out, nrm = ops.baked_render_normals(field.box(), field.brick_map, values, field.use_viewdirs, rays, bool(white),
                                            stop, cam, dequant=field.dequant)
    else:
        out = ops.baked_render(field.box(), field.brick_map, values, field.use_viewdirs, rays, bool(white), stop,
                               dequant=field.dequant)
    img = out[:, :3].view(height, width, 3), out[:, 3].view(height, width), out[:, 4].view(height, width)
    return img + (nrm.view(height, width, 3),) if normals else img


def _check_viewdirs(field, options, what):
    use_viewdirs = bool(options.nerf.use_viewdirs)
    if use_viewdirs != field.use_viewdirs:
        raise ValueError(f"{what}: options.nerf.use_viewdirs is {use_viewdirs}, the baked network "
                         f"{'had' if field.use_viewdirs else 'had no'} view directions")


def _pose_rays(field, height, width, focal_length, tform_cam2world, options):
    """``render_image``'s rays of every pixel of one pose on the field's device (``_check_viewdirs`` first)."""
    return ops.gen_rays(tform_cam2world, height, width, focal_length, None, field.values.device,
                        ndc=options.dataset.no_ndc is False, near=options.dataset.near, far=options.dataset.far,
                        use_viewdirs=field.use_viewdirs)


def _check_values(field, what, stored=False):
    """A CUDA fp32 field, or one in any storage format where ``stored`` (renders, peak weights); fine-tuning is fp32."""
    if not isinstance(field, BakedField):
        raise ValueError(f"{what}: field must be an nb.BakedField, got {type(field).__name__}")
    if not stored and getattr(field.values, "dtype", None) in _LOSSY:
        raise _lossy_refusal(what, field.values.dtype, "gradient or fine-tuning path")
    if not (isinstance(field.values, torch.Tensor) and field.values.is_cuda
            and field.values.dtype in (torch.float32, torch.float16, torch.uint8)):
        raise ValueError(f"{what}: field.values must be an fp32, fp16 or uint8 CUDA tensor (there is no CPU path)")


class _BakedRender(torch.autograd.Function):
    """Rows (n, 8) of ``ops.baked_render`` (stop 0); the backward is ``baked_render_bwd`` then ``baked_tie``."""

    @staticmethod
    def forward(ctx, values, field, rays, white):
        vals = values if values.shape[0] else values.new_zeros(1, 729, 32)
        out = ops.baked_render(field.box(), field.brick_map, vals.detach(), field.use_viewdirs, rays, white, 0.0)
        ctx.save_for_backward(values, rays, out)
        ctx.field, ctx.white = field, white
        return out

    @staticmethod
    def backward(ctx, g):
        values, rays, out = ctx.saved_tensors
        if values.shape[0] == 0:
            return torch.zeros_like(values), None, None, None
        f = ctx.field
        box = f.box()
        d = torch.zeros_like(values)
        ops.baked_render_bwd(box, f.brick_map, values.detach(), f.use_viewdirs, rays, ctx.white, out, g.contiguous(), d)
        return ops.baked_tie(box, f.brick_map, f.bricks, d), None, None, None


def render_baked_rays(field: BakedField, rays, *, white_background=False, early_stop=None, normals=False, ndc=None):
    """(rgb (N, 3), disp (N,), acc (N,), depth (N,)) of the packed ``rays`` (N, 11) with view directions or (N, 8)
    without (``ops.gen_rays`` / ``ops.gen_rays_posed``) through ``field``.  Differentiable with respect to
    ``field.values`` when it requires grad: the gradient is the baked renderer's backward summed over every stored copy
    of each lattice point (include/nerfb200.h "baked fields: gradients and fine-tuning"), so copies that start equal stay
    equal under any elementwise optimiser.  ``early_stop`` as in ``render_baked``, for renders without a gradient.

    An fp16 or 8-bit field renders bit for bit like ``field.float()`` and has no gradient.  This is the differentiable
    render, which refuses such a field in grad mode as it did before fp16 fields could be rendered at all; under
    ``torch.no_grad()`` (or inference mode) it renders one whose values do not require grad.  Anything else raises
    ValueError (fine-tune ``field.float()``).  ``render_baked`` renders fp16 and 8-bit fields in any grad mode.

    ``normals=True`` (or "world") appends the normal map (N, 3) of ``render_baked(normals=)``, in the field's frame, or
    with ``ndc=(H, W, focal)`` (the camera NDC ``rays`` were generated with) in world space, as
    ``extract_baked_mesh(ndc=)`` maps its meshes.  Packed rays do not say whether the field lives in NDC, so "world"
    alone is the field's frame: pass ``ndc`` for an NDC field.  Normals are inference only: with a gradient (values that
    require grad, in grad mode) they raise ValueError, as ``early_stop`` does."""
    from . import density, train_utils

    normals = train_utils.normals_mode(normals)
    cam = density.ndc_camera(ndc) if ndc is not None else None
    if cam is not None and not normals:
        raise ValueError("render_baked_rays: ndc= maps the normal map to world space; pass normals=True with it")
    if normals and isinstance(field, BakedField) and isinstance(field.values, torch.Tensor) \
            and field.values.requires_grad and torch.is_grad_enabled():
        raise ValueError("render_baked_rays: normals have no gradient; render under torch.no_grad()")
    _check_values(field, "render_baked_rays", stored=True)
    # grad mode alone keeps the refusal every fp16 field met here before half precision (pinned by the fine-tuning tests)
    if field.dtype in _LOSSY and (field.values.requires_grad or torch.is_grad_enabled()):
        raise _lossy_refusal("render_baked_rays", field.dtype, "gradient",
                             "render it under torch.no_grad(), or fine-tune field.float() and {back}")
    stride = 11 if field.use_viewdirs else 8
    if not (isinstance(rays, torch.Tensor) and rays.dim() == 2 and rays.shape[1] == stride):
        raise ValueError(f"render_baked_rays: rays must be (N, {stride}) for a field "
                         f"{'with' if field.use_viewdirs else 'without'} view directions")
    grad = field.values.requires_grad and torch.is_grad_enabled()
    stop = 0.0
    if early_stop is not None:
        if grad:
            raise ValueError("render_baked_rays: early_stop has no gradient; render under torch.no_grad()")
        stop = float(early_stop)
        if not 0.0 <= stop < 1.0:
            raise ValueError(f"render_baked_rays: early_stop must lie in [0, 1), got {early_stop!r}")
    white = bool(white_background)
    if grad:
        out = _BakedRender.apply(field.values, field, rays, white)
    else:
        values = field.values.detach() if field.n_active else field.values.new_zeros(1, 729, 32)
        if normals:
            out, nrm = ops.baked_render_normals(field.box(), field.brick_map, values, field.use_viewdirs, rays, white,
                                                stop, cam, dequant=field.dequant)
            return out[:, :3], out[:, 3], out[:, 4], out[:, 5], nrm
        out = ops.baked_render(field.box(), field.brick_map, values, field.use_viewdirs, rays, white, stop,
                               dequant=field.dequant)
    return out[:, :3], out[:, 3], out[:, 4], out[:, 5]


def _check_weights(what, tv_sigma, tv_sh, sparsity):
    """The three regulariser weights as floats, each finite and >= 0 (ValueError otherwise)."""
    lam = (float(tv_sigma), float(tv_sh), float(sparsity))
    if not all(0.0 <= x < float("inf") for x in lam):
        raise ValueError(f"{what}: tv_sigma, tv_sh and sparsity must be finite and >= 0, got {lam}")
    return lam


class _BakedRegularizer(torch.autograd.Function):
    """The 0-dim fp32 loss of ``baked_regularizer``; the backward is the kernel's gradient times the upstream scalar."""

    @staticmethod
    def forward(ctx, values, field, lam):
        loss, count = _regularizer_value(field, values.detach(), lam)
        ctx.save_for_backward(values, count)
        ctx.field, ctx.lam = field, lam
        return loss

    @staticmethod
    def backward(ctx, g):
        values, count = ctx.saved_tensors
        f = ctx.field
        d = torch.zeros_like(values)
        ops.baked_regularizer(f.box(), f.brick_map, f.bricks, values.detach(), count, *ctx.lam, d=d)
        return d * g, None, None


def baked_regularizer(field: BakedField, *, tv_sigma=0.0, tv_sh=0.0, sparsity=0.0) -> torch.Tensor:
    """The 0-dim fp32 loss L = (1 / P) [tv_sigma sum_edges (d sigma_raw)^2 + tv_sh sum_edges sum over the 27 SH
    coefficients of (d coef)^2 + sparsity sum_points log(1 + 2 max(sigma_raw, 0)^2)] over the field's lattice points
    (P of them) and lattice edges (include/nerfb200.h "baked fields: regularisers"): the fp64 sum of the kernel's
    per-slot partials, rounded once.  Differentiable with respect to ``field.values``: the gradient is written at every
    stored copy of each lattice point and is the same bits at all of them, so ``mse + baked_regularizer(...)`` under
    ``torch.optim.Adam`` keeps the copies bit-equal, as ``render_baked_rays`` does.  Each call counts P (one memset and
    one launch) and forms the value (one launch); the backward is one more launch."""
    _check_values(field, "baked_regularizer")
    lam = _check_weights("baked_regularizer", tv_sigma, tv_sh, sparsity)
    if field.n_active == 0:
        raise ValueError("baked_regularizer: the field has no active brick")
    if field.values.requires_grad and torch.is_grad_enabled():
        return _BakedRegularizer.apply(field.values, field, lam)
    return _regularizer_value(field, field.values.detach(), lam)[0]


def _regularizer_value(field, values, lam):
    """(the fp32 loss, the device count P) of ``field``'s lattice at ``values``."""
    box = field.box()
    count = ops.baked_lattice_count(box, field.brick_map, field.bricks)
    partials = torch.empty(field.n_active, dtype=torch.float64, device=values.device)
    ops.baked_regularizer(box, field.brick_map, field.bricks, values, count, *lam, partials=partials)
    return partials.sum().float(), count


# default rates of BakedFieldTrainer: the best held-out PSNR of a sweep on lego A0 at 256^3 (DESIGN §4)
DEFAULT_LR_SIGMA = 1.0
DEFAULT_LR_SH = 1e-2


class BakedFieldTrainer:
    """Fine-tunes ``field.values`` in place through the baked renderer against images.  Each ``step()``, with no host
    synchronisation: draw one image and ``rays_per_step`` distinct pixels from (``seed``, step) (``ops.draw_pixels``),
    their rays (``gen_rays_posed``: NDC, near / far from ``options.dataset``, view directions as the field) and targets,
    ``baked_render`` (stop 0, the white background of ``options.nerf.train``), ``mse(rgb, target)``, the backward and the
    tie into a gradient buffer, and one Adam step (``ops.baked_adam_step_dev``: sigma_raw at ``lr_sigma``, the SH
    coefficients at ``lr_sh``, both times ``0.1 ** (step / (lr_decay * 1000))`` when ``lr_decay`` is given).

    ``images`` (n, H, W, 3) and ``poses`` (n, 3 | 4, 4) are fp32 on the field's device.  The trainer owns the Adam
    moments and the step counter (``step_dev``); ``loss`` is the last step's loss, a device tensor.  Memory: four
    buffers the size of ``field.values`` (gradient, tied gradient, m, v): 3.9 GiB for lego at 256^3 and 22.5 GiB at
    512^3 over the grid of both lego networks, 2.1 and 11.0 GiB over the fine network's grid (DESIGN §4).
    ``rays_per_step`` pixels are drawn from one image per step, so it cannot exceed H * W.  The backward's vector reductions run in hardware order, so two runs agree to fp32 rounding, not bitwise;
    every stored copy of a lattice point stays bit-equal to the others.

    ``tv_sigma``, ``tv_sh`` and ``sparsity`` (finite, >= 0; all 0 by default) add ``baked_regularizer``'s gradient at
    those weights into the tied gradient before the Adam step: one more launch per step when any is nonzero, none when
    all are 0, which leaves the step exactly the unregularised one.  P is counted on the device at construction and
    again by ``prune``.  ``loss`` stays the MSE alone (the regulariser's value would cost a reduction per step; call
    ``baked_regularizer`` for it)."""

    def __init__(self, field, images, poses, focal, options, *, lr_sigma=DEFAULT_LR_SIGMA, lr_sh=DEFAULT_LR_SH,
                 lr_decay=None, rays_per_step=4096, seed=0, tv_sigma=0.0, tv_sh=0.0, sparsity=0.0):
        _check_values(field, "BakedFieldTrainer")
        if field.n_active == 0:
            raise ValueError("BakedFieldTrainer: the field has no active brick")
        dev = field.values.device
        for name, t in (("images", images), ("poses", poses)):
            if not (isinstance(t, torch.Tensor) and t.device == dev and t.dtype == torch.float32):
                raise ValueError(f"BakedFieldTrainer: {name} must be fp32 on the field's device {dev}")
        if images.dim() != 4 or images.shape[3] != 3 or poses.dim() != 3 or poses.shape[1] not in (3, 4) \
                or poses.shape[2] != 4 or poses.shape[0] != images.shape[0]:
            raise ValueError("BakedFieldTrainer: need images (n, H, W, 3) and poses (n, 3 | 4, 4)")
        use_viewdirs = bool(options.nerf.use_viewdirs)
        if use_viewdirs != field.use_viewdirs:
            raise ValueError(f"BakedFieldTrainer: options.nerf.use_viewdirs is {use_viewdirs}, the baked network "
                             f"{'had' if field.use_viewdirs else 'had no'} view directions")
        n_img, H, W = images.shape[:3]
        n = int(rays_per_step)
        if not 0 < n <= H * W:
            raise ValueError(f"BakedFieldTrainer: rays_per_step must lie in 1 .. {H * W}, got {rays_per_step}")
        if not (float(lr_sigma) >= 0 and float(lr_sh) >= 0) or (lr_decay is not None and not float(lr_decay) > 0):
            raise ValueError("BakedFieldTrainer: need lr_sigma, lr_sh >= 0 and lr_decay None or > 0")
        if not 0 <= int(seed) < 2 ** 64:
            raise ValueError("BakedFieldTrainer: seed must be in [0, 2^64)")
        self.reg = _check_weights("BakedFieldTrainer", tv_sigma, tv_sh, sparsity)
        self.field, self.seed = field, int(seed)
        self.images, self.poses = images.contiguous(), poses.contiguous()
        self.focal, self.H, self.W, self.n_images, self.n = float(focal), int(H), int(W), int(n_img), n
        self.lr_sigma, self.lr_sh, self.lr_decay = float(lr_sigma), float(lr_sh), lr_decay
        self.ndc = options.dataset.no_ndc is False
        self.near, self.far = float(options.dataset.near), float(options.dataset.far)
        self.white = bool(options.nerf.train.white_background)
        self._box = field.box()
        v = field.values
        self.d_values, self.d_tied = torch.zeros_like(v), torch.zeros_like(v)
        self.m, self.v = torch.zeros_like(v), torch.zeros_like(v)
        self.step_dev = torch.zeros(1, dtype=torch.int64, device=dev)
        self._image = torch.empty(1, dtype=torch.int64, device=dev)
        self._ids = torch.empty(n, dtype=torch.int64, device=dev)
        self._ws = torch.empty(ops.draw_workspace_bytes(H * W), dtype=torch.uint8, device=dev)
        self._rays = torch.empty(n, 11 if use_viewdirs else 8, dtype=torch.float32, device=dev)
        self._target = torch.empty(n, 3, dtype=torch.float32, device=dev)
        self._out = torch.empty(n, 8, dtype=torch.float32, device=dev)
        self._g = torch.empty(n, 8, dtype=torch.float32, device=dev)
        self.loss = torch.zeros((), dtype=torch.float32, device=dev)
        self._count = ops.baked_lattice_count(self._box, field.brick_map, field.bricks)

    def step(self, n: int = 1):
        """Runs ``n`` steps; returns the last step's loss (a device tensor)."""
        f = self.field
        with torch.no_grad():
            for _ in range(int(n)):
                ops.draw_pixels(self.seed, self.step_dev, self.n_images, self.H * self.W, self.n, self._image,
                                self._ids, self._ws)
                ops.gen_rays_posed(self.poses, self._image, self.H, self.W, self.focal, self._ids, self.ndc, self.near,
                                   self.far, f.use_viewdirs, out=self._rays)
                ops.gather_rows(self.images.view(-1, 3), self.H * self.W, self._image, self._ids, out=self._target)
                ops.baked_render(self._box, f.brick_map, f.values, f.use_viewdirs, self._rays, self.white, 0.0,
                                 out=self._out)
                ops.mse_loss(self._out, None, self._target, self.loss, self._g)
                self.d_values.zero_()
                ops.baked_render_bwd(self._box, f.brick_map, f.values, f.use_viewdirs, self._rays, self.white,
                                     self._out, self._g, self.d_values)
                ops.baked_tie(self._box, f.brick_map, f.bricks, self.d_values, self.d_tied)
                if any(self.reg):
                    ops.baked_regularizer(self._box, f.brick_map, f.bricks, f.values, self._count, *self.reg,
                                          d=self.d_tied)
                ops.baked_adam_step_dev(f.values, self.d_tied, self.m, self.v, self.step_dev, self.lr_sigma,
                                        self.lr_sh, self.lr_decay)
                ops.step_advance(self.step_dev)
        return self.loss

    def prune(self, keep) -> None:
        """Compacts the trainer's field in place to the bricks where ``keep`` (bool[n_active] on the field's device) is
        true, as ``prune_baked`` does: the ``BakedField`` passed to the constructor then holds the pruned ``brick_map``,
        ``bricks`` and ``values``, the Adam moments ``m`` and ``v`` go through the same row gather, and the gradient
        buffers are reallocated at the new size (the old ones are freed first).  ``step_dev``, the seed, the rates and
        the schedule carry on, and the regularisers' P is counted again over the kept bricks.  A pruned brick never comes
        back: its samples become misses, and the tie no longer carries gradient into it.  Keeping no brick raises
        ValueError, as the constructor does.  Reads the kept count back once."""
        f = self.field
        _check_keep(f, keep, "BakedFieldTrainer.prune")
        idx = torch.nonzero(keep).reshape(-1)
        if idx.numel() == 0:
            raise ValueError("BakedFieldTrainer.prune: keep selects no brick (the field would have no active brick)")
        self.d_values = self.d_tied = None
        with torch.no_grad():
            f.brick_map, f.bricks, f.values = _pruned(f, idx)
            self.m, self.v = self.m.index_select(0, idx), self.v.index_select(0, idx)
        self.d_values, self.d_tied = torch.zeros_like(f.values), torch.zeros_like(f.values)
        ops.baked_lattice_count(self._box, f.brick_map, f.bricks, self._count)

    def subdivide(self) -> None:
        """Replaces the trainer's field in place by ``subdivide_baked`` of it: the ``BakedField`` passed to the
        constructor then holds twice the ``resolution`` and the child ``brick_map``, ``bricks`` and ``values``, and the
        Adam moments ``m`` and ``v`` go through the same kernel.  The gradient buffers are freed first and reallocated at
        the new size; while the child's values, m and v are formed the parent's are still held, so the peak is those
        six arrays, below the trainer's five buffers at the new size.  ``step_dev``, the seed, the rates and the schedule carry on, and the
        regularisers' P is counted again.  The refusals are ``subdivide_baked``'s, checked before anything changes.
        Reads the child brick count back once."""
        f = self.field
        res = _check_subdivide(f, "BakedFieldTrainer.subdivide")
        self.d_values = self.d_tied = None
        with torch.no_grad():
            brick_map, bricks = _child_bricks(f, res)
            box = f.box()
            values, m, v = (_subdivided(box, f.brick_map, x, bricks) for x in (f.values, self.m, self.v))
        f.resolution, f.brick_map, f.bricks, f.values = res, brick_map, bricks, values
        self.m, self.v = m, v
        self._box = f.box()
        self.d_values, self.d_tied = torch.zeros_like(f.values), torch.zeros_like(f.values)
        ops.baked_lattice_count(self._box, f.brick_map, f.bricks, self._count)


# ------------------------------------------------------------------------------------------------------------------------
# pruning (include/nerfb200.h "baked fields: pruning")
# ------------------------------------------------------------------------------------------------------------------------
def _check_keep(field, keep, what):
    if not isinstance(field, BakedField):
        raise ValueError(f"{what}: field must be an nb.BakedField, got {type(field).__name__}")
    if not (isinstance(keep, torch.Tensor) and keep.dtype == torch.bool and keep.shape == (field.n_active,)
            and keep.device == field.values.device):
        raise ValueError(f"{what}: keep must be a bool tensor of shape ({field.n_active},) on {field.values.device}")


def _pruned(field, idx):
    """(brick_map, bricks, values) of ``field`` restricted to the slots ``idx`` (ascending int64)."""
    bricks = field.bricks.index_select(0, idx)
    brick_map = torch.full_like(field.brick_map, -1)
    brick_map[bricks.long()] = torch.arange(idx.numel(), dtype=brick_map.dtype, device=brick_map.device)
    return brick_map, bricks, field.values.detach().index_select(0, idx)


def prune_baked(field: BakedField, keep) -> BakedField:
    """A new ``BakedField`` holding the bricks of ``field`` where ``keep`` (bool[n_active] on the field's device) is
    true.  Slots stay in ascending order (so ``bricks`` stays sorted), ``brick_map`` is rebuilt with -1 for the dropped
    bricks, and the kept rows of ``values`` are copied unchanged; ``field`` is not touched.  The copy needs the kept
    values' size again while both fields are alive.  Plain torch indexing: it works on a CPU field too.  Keeping no brick
    gives a field with ``n_active == 0``, which ``render_baked`` renders as empty.

    Lossless criteria (include/nerfb200.h "baked fields: pruning"): ``~baked_transparent_bricks(field)`` leaves every
    render the same bits; ``baked_brick_weights(...) > 0`` leaves the renders of the rays it was measured over the same
    bits.  An 8-bit field's codes are copied and its ``dequant`` shared, not formed again."""
    _check_keep(field, keep, "prune_baked")
    with torch.no_grad():
        brick_map, bricks, values = _pruned(field, torch.nonzero(keep).reshape(-1))
    return BakedField(field.bounds, field.resolution, brick_map, bricks, values, field.use_viewdirs,
                      dequant=field.dequant)


def baked_transparent_bricks(field: BakedField, chunk: int = 1024) -> torch.Tensor:
    """bool[n_active]: the bricks every stored sigma_raw of which is <= 0 and whose channels 0 .. 27 are all finite
    (an 8-bit field's dequantised sigma_raw; its values are always finite).  Dropping them leaves every render of the
    field the same bits (include/nerfb200.h "baked fields: pruning").  Torch over ``chunk`` slots at a time; works on a
    CPU field too."""
    if not isinstance(field, BakedField):
        raise ValueError(f"baked_transparent_bricks: field must be an nb.BakedField, got {type(field).__name__}")
    v = field.values.detach()
    out = torch.empty(field.n_active, dtype=torch.bool, device=v.device)
    for s in range(0, field.n_active, chunk):
        out[s:s + chunk] = (_widened(field, slice(s, s + chunk), 0) <= 0).all(1)
        if v.dtype != torch.uint8:  # codes dequantise to finite values
            out[s:s + chunk] &= torch.isfinite(v[s:s + chunk, :, :28]).flatten(1).all(1)
    return out


def baked_brick_weights_rays(field: BakedField, rays, out=None) -> torch.Tensor:
    """fp32[n_active]: each brick slot's peak rendering weight w = alpha T over the packed ``rays`` (N, 11) with view
    directions or (N, 8) without, laid out as ``render_baked_rays`` takes them: ``baked_render``'s weights at stop 0, a
    NaN weight as +inf (include/nerfb200.h "baked fields: pruning").  With ``out`` (fp32[n_active] on the field's
    device) the peaks are max-accumulated into it, so chunks of rays give the bits of one call.  A field without active
    bricks returns an empty tensor without a launch."""
    if not isinstance(field, BakedField):
        raise ValueError(f"baked_brick_weights_rays: field must be an nb.BakedField, got {type(field).__name__}")
    stride = 11 if field.use_viewdirs else 8
    if not (isinstance(rays, torch.Tensor) and rays.dim() == 2 and rays.shape[1] == stride
            and rays.dtype == torch.float32):
        raise ValueError(f"baked_brick_weights_rays: rays must be fp32 (N, {stride}) for a field "
                         f"{'with' if field.use_viewdirs else 'without'} view directions")
    if out is not None and not (isinstance(out, torch.Tensor) and out.dtype == torch.float32
                                and out.shape == (field.n_active,) and out.is_contiguous()):
        raise ValueError(f"baked_brick_weights_rays: out must be a contiguous fp32 tensor of shape ({field.n_active},)")
    _check_values(field, "baked_brick_weights_rays", stored=True)
    dev = field.values.device
    if rays.device != dev or (out is not None and out.device != dev):
        raise ValueError(f"baked_brick_weights_rays: rays and out must be on the field's device {dev}")
    if out is None:
        out = torch.zeros(field.n_active, dtype=torch.float32, device=dev)
    if field.n_active and rays.shape[0]:
        ops.baked_max_weights(field.box(), field.brick_map, field.values.detach(), field.use_viewdirs,
                              rays.contiguous(), out, dequant=field.dequant)
    return out


def baked_brick_weights(field: BakedField, poses, height, width, focal_length, options) -> torch.Tensor:
    """fp32[n_active]: each brick slot's peak rendering weight over every pixel of every pose in ``poses`` (n, 3 | 4,
    4), the rays formed as ``render_baked`` forms them (``options.dataset`` near / far / no_ndc, view directions as the
    field, which must match ``options.nerf.use_viewdirs``).  One launch per view, with no host synchronisation between
    them (the poses are copied to the host once).  ``weights > tau`` is the PlenOctrees pruning mask; ``weights > 0``
    prunes without changing those views' renders."""
    if not isinstance(field, BakedField):
        raise ValueError(f"baked_brick_weights: field must be an nb.BakedField, got {type(field).__name__}")
    if not (isinstance(poses, torch.Tensor) and poses.dim() == 3 and poses.shape[0] > 0 and poses.shape[1] in (3, 4)
            and poses.shape[2] == 4 and poses.is_floating_point()):
        raise ValueError("baked_brick_weights: poses must be a float tensor (n, 3 | 4, 4) with n >= 1")
    if not (int(height) > 0 and int(width) > 0):
        raise ValueError(f"baked_brick_weights: need height, width > 0, got {height}, {width}")
    _check_values(field, "baked_brick_weights", stored=True)
    _check_viewdirs(field, options, "baked_brick_weights")
    out = torch.zeros(field.n_active, dtype=torch.float32, device=field.values.device)
    if field.n_active == 0:
        return out
    host = poses.detach().to("cpu", torch.float32)
    values, box = field.values.detach(), field.box()
    for p in host:
        rays = _pose_rays(field, height, width, focal_length, p, options)
        ops.baked_max_weights(box, field.brick_map, values, field.use_viewdirs, rays, out, dequant=field.dequant)
    return out


# ------------------------------------------------------------------------------------------------------------------------
# subdivision (include/nerfb200.h "baked fields: subdivision")
# ------------------------------------------------------------------------------------------------------------------------
def _check_subdivide(field, what):
    """The child resolution of a CUDA fp32 ``field`` whose resolution is at most 2048 per axis (ValueError
    otherwise)."""
    if not isinstance(field, BakedField):
        raise ValueError(f"{what}: field must be an nb.BakedField, got {type(field).__name__}")
    if field.dtype in _LOSSY:
        raise _lossy_refusal(what, field.dtype, "subdivision", "subdivide field.float() and {back}")
    if not all(r <= 2048 for r in field.resolution):
        raise ValueError(f"{what}: resolution {field.resolution} is past 2048 on an axis (the child would pass 4096)")
    if not (field.values.is_cuda and field.values.dtype == torch.float32):
        raise ValueError(f"{what}: field.values must be an fp32 CUDA tensor (there is no CPU path)")
    return tuple(2 * r for r in field.resolution)


def _child_bricks(field, res):
    """(brick_map, bricks) int32 of the child box at ``res`` (twice the field's resolution): the children 2 pb + delta
    of every active parent brick pb that exist in the child box, ascending, and their rank.  Plain torch on the field's
    device; reads the child count back once."""
    dev = field.bricks.device
    nbp = [-(-r // 8) for r in field.resolution]
    nbc = [-(-r // 8) for r in res]
    br = field.bricks.long()
    b = torch.stack([br % nbp[0], br // nbp[0] % nbp[1], br // (nbp[0] * nbp[1])], -1)  # [n, 3]
    k = torch.arange(8, device=dev)
    c = 2 * b[:, None] + torch.stack([k & 1, k >> 1 & 1, k >> 2], -1)[None]  # [n, 8, 3]
    exists = (c < torch.tensor(nbc, device=dev)).all(-1)
    bricks = torch.sort(((c[..., 2] * nbc[1] + c[..., 1]) * nbc[0] + c[..., 0])[exists]).values.int()
    brick_map = torch.full((nbc[0] * nbc[1] * nbc[2],), -1, dtype=torch.int32, device=dev)
    brick_map[bricks.long()] = torch.arange(bricks.numel(), dtype=torch.int32, device=dev)
    return brick_map, bricks


def _subdivided(box, brick_map, values, child_bricks):
    """fp32 (n_child, 729, 32): ``values`` (of the parent ``box`` / ``brick_map``) subdivided onto ``child_bricks``."""
    out = torch.empty(child_bricks.numel(), 729, 32, dtype=torch.float32, device=values.device)
    if child_bricks.numel():
        ops.baked_subdivide(box, brick_map, values.detach(), child_bricks, out)
    return out


def subdivide_baked(field: BakedField) -> BakedField:
    """A new ``BakedField`` at twice ``field``'s resolution over the same bounds, holding the same trilinear function
    (include/nerfb200.h "baked fields: subdivision"): its active bricks are the children of ``field``'s, in ascending
    order, and every child lattice point is the parent's value there (a copy where it coincides with a parent point,
    the mean of 2, 4 or 8 parent points otherwise, each op rounded in fp32).  It renders the parent's continuous field
    with samples half as far apart.  ``field`` is not touched; the child needs up to 8 times the parent's values.  Prune
    first (``prune_baked``) to subdivide only the bricks worth keeping.  A field without active bricks gives an empty
    child without a launch.  ValueError for an fp16 field (subdivide ``field.float()``), a CPU field, or a resolution
    past 2048 on an axis, and for an 8-bit field.  Reads the child brick count back once."""
    res = _check_subdivide(field, "subdivide_baked")
    with torch.no_grad():
        brick_map, bricks = _child_bricks(field, res)
        values = _subdivided(field.box(), field.brick_map, field.values, bricks)
    return BakedField(field.bounds, res, brick_map, bricks, values, field.use_viewdirs)


# ------------------------------------------------------------------------------------------------------------------------
# meshes (include/nerfb200.h "baked fields: meshes")
# ------------------------------------------------------------------------------------------------------------------------
def extract_baked_mesh(field: BakedField, level: float = 50.0, *, colors: bool = False, normals: bool = False,
                       ndc=None):
    """The level set sigma = ``level`` of a baked field's own density as an ``nb.Mesh``, by sparse marching cubes over
    the field's active bricks on the GPU (include/nerfb200.h "baked fields: meshes").  No network is needed, so this
    meshes a fine-tuned, pruned, subdivided or from-scratch field as it renders.

    Marching cubes runs over sigma_raw (channel 0, an fp16 field's widened exactly, an 8-bit field's dequantised): for ``level`` >= 0 the crossing of
    the renderer's density relu(sigma_raw) along a lattice edge is the crossing of sigma_raw, so the faces and vertex
    numbering are those of ``extract_mesh`` on the baked network over the same grid, and the vertices lie on the
    renderer's surface.  ``normals=True`` sets ``Mesh.normals``: the outward unit normal from central differences of
    sigma_raw (a lattice point no active brick holds reads 0), (0, 0, 0) where the gradient vanishes.  ``colors=True``
    gives each vertex the renderer's colour of that point seen head-on from outside.

    ``ndc=(H, W, focal)`` is for a field baked from a forward-facing scene, which lives in NDC: the mesh is extracted in
    NDC and returned in world space, as ``extract_mesh(ndc=)`` does; the colours are seen along world directions.  A
    field that is not a ``BakedField``, a non-finite or negative ``level``, a malformed ``ndc`` or one whose box reaches
    z = 1 raises ValueError, a CPU field NotImplementedError, before any launch.  A field without active bricks or a
    level with no crossing gives an empty mesh.  Reads the mesh's two totals back once."""
    from . import density
    from .mesh import Mesh, _level

    if not isinstance(field, BakedField):
        raise ValueError(f"extract_baked_mesh: field must be an nb.BakedField, got {type(field).__name__}")
    level = _level(level)
    if level < 0.0:
        raise ValueError(f"extract_baked_mesh: level must be >= 0 (the density relu(sigma_raw) is never negative), got "
                         f"{level}")
    cam = density.ndc_camera(ndc) if ndc is not None else None
    if cam is not None and not field.bounds[1][2] < 1.0:
        raise ValueError(f"extract_baked_mesh: with ndc=, the field's NDC box needs hi_z < 1 (z = 1 is the far plane at "
                         f"infinity), got {field.bounds!r}")
    values = field.values
    if not (isinstance(values, torch.Tensor) and values.is_cuda):
        raise NotImplementedError("nerfb200: the baked field must be on a CUDA device (there is no CPU path)")
    if values.dtype not in (torch.float32, torch.float16, torch.uint8):
        raise ValueError(f"extract_baked_mesh: field.values must be fp32, fp16 or uint8, got {values.dtype}")
    dev = values.device

    def empty():
        z = torch.zeros(0, 3, dtype=torch.float32, device=dev)
        return Mesh(z, torch.zeros(0, 3, dtype=torch.int32, device=dev), z.clone() if colors else None,
                    z.clone() if normals else None)

    if field.n_active == 0:
        return empty()
    box = field.box()
    values = values.detach()
    with torch.no_grad():
        sigma = _widened(field, slice(None), 0).contiguous()  # (n_active, 729): the halo-0 sparse layout
        totals, ws = ops.mesh_sparse_count(box, field.brick_map, field.bricks, field.n_active, sigma, False, level)
        n_v, n_f = (int(t) for t in totals.tolist())  # the one host sync: the outputs' sizes
        if n_v == 0:
            return empty()
        want_dirs = normals or (colors and field.use_viewdirs)
        verts, faces, _, keys = ops.mesh_sparse_emit(box, field.brick_map, field.bricks, field.n_active, sigma, False,
                                                     level, ws, n_v, n_f, want_keys=colors or normals)
        dirs = nrm = None
        if want_dirs:
            dirs, nrm = ops.baked_mesh_dirs(box, field.brick_map, values, level, keys, want_normals=normals,
                                            dequant=field.dequant)
        if cam is not None:
            verts, faces, dirs = ops.ndc_mesh_to_world(cam, verts, faces, dirs)
            if normals:  # -(world dir), 0 where the NDC direction fell back (its normal is 0 there)
                nrm = torch.where((nrm == 0).all(-1, keepdim=True), torch.zeros_like(dirs), -dirs)
        rgb = None
        if colors:
            rgb = ops.baked_mesh_colors(box, field.brick_map, values, field.use_viewdirs, level, keys,
                                        dirs if field.use_viewdirs else None, dequant=field.dequant)
    return Mesh(verts, faces, rgb, nrm)


# ------------------------------------------------------------------------------------------------------------------------
# point queries (include/nerfb200.h "baked fields: normal maps and point queries")
# ------------------------------------------------------------------------------------------------------------------------
def _query_field(field, what):
    """The refusals every point query shares: not a ``BakedField`` or values that require grad in grad mode
    (ValueError), a CPU field (NotImplementedError)."""
    if not isinstance(field, BakedField):
        raise ValueError(f"{what}: field must be an nb.BakedField, got {type(field).__name__}")
    if isinstance(field.values, torch.Tensor) and field.values.requires_grad and torch.is_grad_enabled():
        raise ValueError(f"{what}: point queries are inference only (no gradient with respect to the values); call it "
                         "under torch.no_grad() or on values that do not require grad")
    if not (isinstance(field.values, torch.Tensor) and field.values.is_cuda):
        raise NotImplementedError("nerfb200: the baked field must be on a CUDA device (there is no CPU path)")
    if field.values.dtype not in (torch.float32, torch.float16, torch.uint8):
        raise ValueError(f"{what}: field.values must be fp32, fp16 or uint8, got {field.values.dtype}")


def _query(field, pts, dirs, want_raw, want_grad, use_viewdirs):
    """``ops.baked_query`` at flat points (P, 3) on the field's device; P may be 0."""
    if pts.device != field.values.device:
        raise ValueError(f"nerfb200: the points are on {pts.device}, the baked field on {field.values.device}")
    n = pts.shape[0]
    if n == 0 or field.n_active == 0:  # nothing to read: every point misses
        return (pts.new_zeros(n, 4) if want_raw else None), (pts.new_zeros(n, 3) if want_grad else None)
    return ops.baked_query(field.box(), field.brick_map, field.values.detach(), use_viewdirs, pts.contiguous(), dirs,
                           want_raw, want_grad, dequant=field.dequant)


def baked_density_gradient(field: BakedField, pts: torch.Tensor, *, ndc=None):
    """``(sigma_raw (...), grad (..., 3))`` of a baked field at ``pts`` (..., 3) fp32 CUDA on the field's device, as
    ``nb.density_gradient`` gives them for a network: sigma_raw is the renderer's trilinear interp at the point and grad
    its exact gradient inside the cube the renderer's lookup picks (one-sided on a cube face; include/nerfb200.h "baked
    fields: normal maps and point queries").  A point outside the box or in an inactive brick gives 0 and 0.  Any
    storage format; an fp16 or 8-bit field gives the bits of ``field.float()``.

    ``ndc=(H, W, focal)`` takes an NDC field's ``pts`` in world space (every z < 0, in front of the camera; ValueError
    otherwise): sigma_raw is read at the NDC point N(p) and grad is the world gradient J^T grad_q (include/nerfb200.h
    "NDC scenes"), exactly as ``density_gradient(ndc=)`` maps a network's.  Inference only: values that require grad in
    grad mode are refused (ValueError), as is a CPU field (NotImplementedError), before any launch."""
    from . import density

    cam = density.ndc_camera(ndc) if ndc is not None else None
    _query_field(field, "baked_density_gradient")
    pts = density._checked_points(pts, world_ndc=cam is not None)
    flat = pts.reshape(-1, 3)
    with torch.no_grad():
        if cam is not None:
            if flat.device != field.values.device:
                raise ValueError(f"nerfb200: the points are on {flat.device}, the baked field on "
                                 f"{field.values.device}")
            flat = ops.ndc_from_world(cam, flat.contiguous())
        raw, grad = _query(field, flat, None, True, True, False)  # sigma reads no view direction
        if cam is not None and flat.shape[0]:
            rows = torch.cat([raw[:, 3:], grad], 1)
            ops.ndc_grad_to_world(cam, flat, rows, out=rows)
            grad = rows[:, 1:]
        sigma = raw[:, 3]
    return sigma.reshape(pts.shape[:-1]), grad.reshape(pts.shape)


def baked_raw(field: BakedField, pts: torch.Tensor, viewdirs=None) -> torch.Tensor:
    """raw (..., 4) = (s_r, s_g, s_b, sigma_raw) of a baked field at ``pts`` (..., 3) in the field's own frame (world
    space for Blender scenes, NDC for LLFF scenes, as ``run_network`` takes its points): ``run_network``'s raw layout,
    the pre-sigmoid colour logits and the raw density, each the renderer's trilinear interp at the point, the logits seen
    along ``viewdirs`` (..., 3) as given (not normalised).  ``viewdirs`` is required for a field with view directions and
    refused for one without (the logits are then Y_0 coef_c0).  A point outside the box or in an inactive brick reads 0
    in every channel; at a lattice point the cell rule puts at fractions 0 the channels are the stored values bit for
    bit.  Any storage format, CUDA tensors on the field's device; inference only, as ``baked_density_gradient``."""
    from . import density

    _query_field(field, "baked_raw")
    if field.use_viewdirs != (viewdirs is not None):
        raise ValueError(f"baked_raw: the field {'has' if field.use_viewdirs else 'has no'} view directions; "
                         f"{'pass' if field.use_viewdirs else 'do not pass'} viewdirs")
    pts = density._checked_points(pts)
    dirs = None
    if viewdirs is not None:
        if not (isinstance(viewdirs, torch.Tensor) and viewdirs.dtype == torch.float32
                and viewdirs.shape == pts.shape and viewdirs.device == pts.device):
            raise ValueError(f"baked_raw: viewdirs must be an fp32 tensor of the points' shape {list(pts.shape)} on "
                             f"{pts.device}")
        dirs = viewdirs.reshape(-1, 3).contiguous()
    with torch.no_grad():
        raw, _ = _query(field, pts.reshape(-1, 3), dirs, True, False, field.use_viewdirs)
    return raw.reshape(*pts.shape[:-1], 4)
