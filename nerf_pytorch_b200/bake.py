"""Baked fields: a trained FlexibleNeRFModel evaluated once on the lattice points of the bricks an occupancy grid calls
occupied -- raw density plus degree-2 spherical-harmonic coefficients of its rgb logits over 64 view directions -- and
rendered by trilinear interpolation of those values, without the MLP (PlenOctrees- / SNeRG-style baking).

The bricks are the sparse meshes' (include/nerfb200.h "sparse meshes"), the values and the renderer are defined in
include/nerfb200.h "baked fields"; the bake is one fused wgmma kernel (csrc/mlp_tc.cu, bake_tc_kernel) and the renderer
one warp per ray (csrc/baked.cu).  This file validates arguments, sizes buffers and moves pointers; the bake reads the
active brick count back once to size its values."""
from __future__ import annotations

import torch

from . import ops


class BakedField:
    """A baked field on the device: ``bounds`` ((lo), (hi)) and ``resolution`` (three ints) of the lattice box,
    ``brick_map`` int32[bricks] (slot or -1), ``bricks`` int32[n_active] (slot -> brick), ``values``
    fp32[n_active, 729, 32] and ``use_viewdirs`` (whether the network had view directions)."""

    def __init__(self, bounds, resolution, brick_map, bricks, values, use_viewdirs: bool):
        self.bounds = (tuple(float(v) for v in bounds[0]), tuple(float(v) for v in bounds[1]))
        self.resolution = tuple(int(r) for r in resolution)
        self.brick_map = brick_map
        self.bricks = bricks
        self.values = values
        self.use_viewdirs = bool(use_viewdirs)

    @property
    def n_active(self) -> int:
        return int(self.values.shape[0])

    def box(self):
        return ops.grid_struct(self.bounds, self.resolution)

    def __repr__(self):
        return (f"BakedField({self.n_active} bricks of {ops.mesh_sparse_brick_count(self.box())}, "
                f"{self.values.numel() * 4 / 2 ** 20:.1f} MiB, resolution {self.resolution}"
                f"{', view directions' if self.use_viewdirs else ''})")

    def save(self, path) -> None:
        torch.save({"bounds": self.bounds, "resolution": self.resolution, "brick_map": self.brick_map.cpu(),
                    "bricks": self.bricks.cpu(), "values": self.values.cpu(), "use_viewdirs": self.use_viewdirs}, path)

    @classmethod
    def load(cls, path, device="cuda") -> "BakedField":
        d = torch.load(path, map_location="cpu", weights_only=True)
        return cls(d["bounds"], d["resolution"], d["brick_map"].to(device), d["bricks"].to(device),
                   d["values"].to(device), d["use_viewdirs"])


def bake(model, encode_position_fn, encode_direction_fn=None, *, bounds, resolution, grid) -> BakedField:
    """Bake ``model`` (the network that renders the final image: pass ``model_fine``) over the lattice box ``bounds``
    / ``resolution`` (as ``extract_mesh``; up to 4096 cubes per axis) on the bricks ``grid`` (an ``nb.OccupancyGrid`` on
    the model's device) calls occupied, under the sparse meshes' activity rule.  The field lives in the coordinates the
    MLP encodes: world space for Blender scenes, NDC for LLFF scenes.  Argument errors raise ValueError, an
    architecture the wgmma inference forward refuses NotImplementedError, before any launch."""
    from . import train_utils
    from .mesh import _box, _check_grid, _network

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
    values = torch.empty(n_active, 729, 32, dtype=torch.float32, device=dev)
    if n_active:
        with torch.no_grad():
            ops.bake(arch, blob, box, bricks, 0, n_active, values)
    return BakedField((lo, hi), res, brick_map, bricks[:n_active].clone(), values, arch.use_viewdirs)


def render_baked(field: BakedField, height, width, focal_length, tform_cam2world, options, mode="validation", *,
                 early_stop=None):
    """(rgb (H, W, 3), disp (H, W), acc (H, W)) of ``field`` seen from the pose ``tform_cam2world``.  The rays are
    ``render_image``'s: ``ops.gen_rays`` with ``options.dataset`` near / far / no_ndc and ``options.nerf.use_viewdirs``
    (which must match the baked network), and the white background of ``options.nerf.<mode>`` (``options.nerf.train``
    while ``train_utils.COMPAT_MODE_QUIRK`` holds, as ``render_image``).  Samples are spaced half the smallest cube side
    apart along each ray inside the box.  ``early_stop`` t in [0, 1) stops a ray once its transmittance falls below t
    (checked every 32 samples); a ray that never stops is bit for bit the render without it."""
    from . import train_utils

    if not isinstance(field, BakedField):
        raise ValueError(f"render_baked: field must be an nb.BakedField, got {type(field).__name__}")
    if not field.values.is_cuda:
        raise NotImplementedError("nerfb200: the baked field must be on a CUDA device (there is no CPU path)")
    use_viewdirs = bool(options.nerf.use_viewdirs)
    if use_viewdirs != field.use_viewdirs:
        raise ValueError(f"render_baked: options.nerf.use_viewdirs is {use_viewdirs}, the baked network "
                         f"{'had' if field.use_viewdirs else 'had no'} view directions")
    stop = 0.0
    if early_stop is not None:
        stop = float(early_stop)
        if not 0.0 <= stop < 1.0:
            raise ValueError(f"render_baked: early_stop must lie in [0, 1), got {early_stop!r}")
    white = getattr(options.nerf, "train" if train_utils.COMPAT_MODE_QUIRK else mode).white_background
    dev = field.values.device
    rays = ops.gen_rays(tform_cam2world, height, width, focal_length, None, dev, ndc=options.dataset.no_ndc is False,
                        near=options.dataset.near, far=options.dataset.far, use_viewdirs=use_viewdirs)
    values = field.values if field.n_active else field.values.new_zeros(1, 729, 32)
    out = ops.baked_render(field.box(), field.brick_map, values, use_viewdirs, rays, bool(white), stop)
    return out[:, :3].view(height, width, 3), out[:, 3].view(height, width), out[:, 4].view(height, width)
