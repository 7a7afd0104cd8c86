"""Meshes from trained networks: the density of a FlexibleNeRFModel on a lattice over a box, queried through the fused
MLP forward (``ops.mlp_fwd_pts``), and marching cubes over it on the GPU (csrc/mesh.cu).

The lattice, the vertex rule, the case table and the face order are defined once, in include/nerfb200.h ("meshes"; the
sparse path over an occupancy grid's bricks in "sparse meshes", csrc/mesh_sparse.cu); this file validates arguments,
sizes buffers and moves pointers.  The surface step reads its two totals back once to allocate the outputs: that is its
only host synchronisation, besides the sparse path's read of its active brick count."""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch

from . import ops

# lattice points per MLP call when the caller does not choose: 4 M points keep the query's buffers near 112 MB
_SLAB_POINTS = 1 << 22


def _box(bounds, resolution, dense=True):
    """(lo, hi, res) after the refusals that need no device: ValueError for a malformed box or lattice (and, for the
    dense path, one past 2^31 points)."""
    try:
        lo, hi = bounds
        lo, hi = tuple(float(v) for v in lo), tuple(float(v) for v in hi)
    except (TypeError, ValueError):
        raise ValueError(f"mesh: bounds must be ((x0, y0, z0), (x1, y1, z1)), got {bounds!r}") from None
    if len(lo) != 3 or len(hi) != 3:
        raise ValueError(f"mesh: bounds must be ((x0, y0, z0), (x1, y1, z1)), got {bounds!r}")
    if not all(math.isfinite(v) for v in lo + hi) or not all(h > l for l, h in zip(lo, hi)):
        raise ValueError(f"mesh: bounds must be finite with hi > lo on every axis, got {bounds!r}")
    res = (resolution,) * 3 if isinstance(resolution, int) else tuple(resolution)
    if len(res) != 3 or not all(isinstance(r, int) for r in res):
        raise ValueError(f"mesh: resolution must be an int or three ints, got {resolution!r}")
    if not all(2 <= r <= 4096 for r in res):
        raise ValueError(f"mesh: resolution must be 2 .. 4096 cubes per axis, got {resolution!r}")
    if dense and math.prod(r + 1 for r in res) > 2 ** 31:
        raise ValueError(f"mesh: a lattice of {' x '.join(str(r + 1) for r in res)} points is past 2^31")
    return lo, hi, res


def _level(level):
    level = float(level)
    if not math.isfinite(level):
        raise ValueError(f"mesh: level must be finite, got {level}")
    return level


class Mesh:
    """A triangle mesh on the device: ``vertices`` (V, 3) fp32, ``faces`` (F, 3) int32 vertex ids, counter-clockwise
    seen from outside (where density <= level), ``colors`` (V, 3) fp32 in [0, 1] or None, and ``normals`` (V, 3) fp32
    outward unit normals or None."""

    def __init__(self, vertices: torch.Tensor, faces: torch.Tensor, colors: Optional[torch.Tensor] = None,
                 normals: Optional[torch.Tensor] = None):
        self.vertices = vertices
        self.faces = faces
        self.colors = colors
        self.normals = normals

    def __repr__(self):
        return (f"Mesh({self.vertices.shape[0]} vertices, {self.faces.shape[0]} faces"
                f"{', colors' if self.colors is not None else ''}{', normals' if self.normals is not None else ''})")

    def save_ply(self, path) -> None:
        """Binary little-endian PLY: float x y z (then float nx ny nz with normals, and uchar red green blue when
        colored), faces as uchar-counted int lists.  Written on the host with numpy."""
        v = self.vertices.detach().cpu().numpy().astype("<f4")
        f = self.faces.detach().cpu().numpy().astype("<i4")
        fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
        if self.normals is not None:
            fields += [("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")]
        if self.colors is not None:
            fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
        vrec = np.empty(v.shape[0], dtype=fields)
        vrec["x"], vrec["y"], vrec["z"] = v[:, 0], v[:, 1], v[:, 2]
        if self.normals is not None:
            n = self.normals.detach().cpu().numpy().astype("<f4")
            vrec["nx"], vrec["ny"], vrec["nz"] = n[:, 0], n[:, 1], n[:, 2]
        if self.colors is not None:
            c = np.clip(np.rint(self.colors.detach().cpu().numpy() * 255.0), 0, 255).astype("u1")
            vrec["red"], vrec["green"], vrec["blue"] = c[:, 0], c[:, 1], c[:, 2]
        frec = np.empty(f.shape[0], dtype=[("n", "u1"), ("v", "<i4", (3,))])
        frec["n"] = 3
        frec["v"] = f
        head = ["ply", "format binary_little_endian 1.0", f"element vertex {v.shape[0]}",
                "property float x", "property float y", "property float z"]
        if self.normals is not None:
            head += ["property float nx", "property float ny", "property float nz"]
        if self.colors is not None:
            head += ["property uchar red", "property uchar green", "property uchar blue"]
        head += [f"element face {f.shape[0]}", "property list uchar int vertex_indices", "end_header"]
        with open(path, "wb") as fh:
            fh.write(("\n".join(head) + "\n").encode("ascii"))
            fh.write(vrec.tobytes())
            fh.write(frec.tobytes())


def _surface(volume: torch.Tensor, box, level: float, want_dirs: bool):
    totals, ws = ops.mesh_count(box, volume, level)
    n_v, n_f = (int(t) for t in totals.tolist())  # the one host sync: the outputs' sizes
    return ops.mesh_emit(box, volume, level, ws, n_v, n_f, want_dirs=want_dirs)


def extract_mesh_from_volume(volume: torch.Tensor, bounds, level: float) -> Mesh:
    """Marching cubes over a caller-given field: ``volume`` (n_z, n_y, n_x) fp32 CUDA, each side >= 3, holds the value
    at lattice point (x_i, y_j, z_k) in ``volume[k, j, i]``, the lattice spanning ``bounds`` with n - 1 cubes per axis
    (point i at lo + (hi - lo) * i / (n - 1), include/nerfb200.h).  Inside is value > ``level``."""
    if not isinstance(volume, torch.Tensor) or not volume.is_cuda:
        raise NotImplementedError("nerfb200: the volume must be a CUDA tensor (there is no CPU path)")
    if volume.dtype != torch.float32 or volume.dim() != 3:
        raise ValueError(f"mesh: volume must be a 3-d fp32 tensor, got {volume.dtype}{list(volume.shape)}")
    nz, ny, nx = volume.shape
    lo, hi, res = _box(bounds, (nx - 1, ny - 1, nz - 1))
    level = _level(level)
    v, f, _ = _surface(volume.contiguous(), ops.grid_struct((lo, hi), res), level, False)
    return Mesh(v, f)


def _network(model, encode_position_fn, encode_direction_fn):
    """(arch, blob) of a FlexibleNeRFModel on the device; the refusals precede any launch."""
    from . import train_utils
    from .nerf_helpers import get_embedding_function

    params = list(model.parameters()) if hasattr(model, "parameters") else []
    enc_xyz = train_utils._probe_encoder(encode_position_fn, None)
    if enc_xyz is None:
        raise ValueError("mesh: encode_position_fn is required")
    enc_dir = None
    if hasattr(model, "fc_rgb") and hasattr(model, "layers_dir"):
        if encode_direction_fn is not None:
            enc_dir = train_utils._probe_encoder(encode_direction_fn, None)
        else:
            dim = model.layers_dir[0].in_features - model.layer1.out_features
            enc_dir = train_utils._probe_encoder(get_embedding_function((dim - 3) // 6), None)
    arch = train_utils._arch_of(model, enc_xyz, enc_dir)
    if not params or not all(p.is_cuda and p.dtype == torch.float32 for p in params):
        raise NotImplementedError("nerfb200: parameters must be fp32 CUDA tensors (no CPU / half path)")
    return arch


def _query_impl(arch, impl):
    """The MLP kernels of the lattice query: None picks the wgmma inference forward where the architecture allows it,
    else the fp32 kernels; an explicit impl the architecture refuses raises NotImplementedError."""
    from . import train_utils

    if impl is None:
        return train_utils._auto_impl(arch, None, 64, 0, training=False)
    use = int(impl)
    why = ops.impl_refusal(arch, 64, ops.IMPL_TC_FWD if use == ops.IMPL_TC else use)
    if why is not None:
        raise NotImplementedError(f"nerfb200 mesh: impl {use}: {why}")
    return use


def density_volume(model, encode_position_fn, bounds=((-1.5,) * 3, (1.5,) * 3), resolution=256, *,
                   encode_direction_fn=None, impl: Optional[int] = None,
                   planes_per_slab: Optional[int] = None) -> torch.Tensor:
    """sigma = relu(raw sigma) of ``model`` at the (R + 1)^3 lattice points of ``bounds`` (``resolution`` R cubes per
    axis, an int or three ints), as an (n_z, n_y, n_x) fp32 tensor on the model's device, laid out as
    ``extract_mesh_from_volume`` reads it.  sigma reads the trunk alone, so the view direction of the query is
    irrelevant; ``encode_direction_fn`` defaults to the stock encoder of the width the model's layers_dir[0] expects.
    ``impl``: the MLP kernels (None: the wgmma inference forward where the architecture allows it, else fp32 CUDA
    cores).  The lattice is queried ``planes_per_slab`` z planes at a time (default: about 4 M points per call); each
    point depends on its lattice index alone, so the volume does not depend on the slab size."""
    from . import train_utils

    lo, hi, res = _box(bounds, resolution)
    arch = _network(model, encode_position_fn, encode_direction_fn)
    use = _query_impl(arch, impl)
    n0, n1, n2 = (r + 1 for r in res)
    plane = n0 * n1
    slab = int(planes_per_slab) if planes_per_slab is not None else max(1, _SLAB_POINTS // plane)
    if slab < 1:
        raise ValueError(f"mesh: planes_per_slab must be >= 1, got {planes_per_slab}")
    slab = min(slab, n2)
    _, blob = train_utils._packed(model, arch)
    dev = blob.device
    box = ops.grid_struct((lo, hi), res)
    rows_max = -(-slab * plane // 64)
    pts = torch.zeros(rows_max * 64, 3, dtype=torch.float32, device=dev)
    direction = torch.tensor([[0.0, 0.0, 1.0]], dtype=torch.float32, device=dev)
    vol = torch.empty(n2, plane, dtype=torch.float32, device=dev)
    with torch.no_grad():
        for z0 in range(0, n2, slab):
            nz = min(slab, n2 - z0)
            n = nz * plane
            rows = -(-n // 64)  # rows of 64 samples; the tail past n holds earlier points and is discarded
            ops.mesh_lattice_points(box, z0, nz, pts)
            dirs = direction.expand(rows, 3) if arch.use_viewdirs else None
            raw = ops.mlp_fwd_pts(arch, blob, pts[:rows * 64].view(rows, 64, 3), dirs, impl=use)
            vol[z0:z0 + nz].view(-1).copy_(torch.relu(raw.view(-1, 4)[:n, 3]))
    return vol.view(n2, n1, n0)


def _check_grid(grid, device):
    """The refusals of a sparse extraction's grid: ValueError for anything but an OccupancyGrid with well-formed bits
    on ``device``, NotImplementedError for bits on the CPU."""
    from .occupancy import OccupancyGrid

    if not isinstance(grid, OccupancyGrid):
        raise ValueError(f"mesh: grid must be an nb.OccupancyGrid, got {type(grid).__name__}")
    bits = grid.bits
    if not isinstance(bits, torch.Tensor) or not bits.is_cuda:
        raise NotImplementedError("nerfb200: the grid's bits must be a CUDA tensor (there is no CPU path)")
    if bits.device != device:
        raise ValueError(f"mesh: the grid is on {bits.device}, the model on {device}")
    if bits.dtype != torch.int32 or bits.dim() != 1 or not bits.is_contiguous() or \
            bits.numel() != ops.grid_words(grid.c_struct()):
        raise ValueError(f"mesh: the grid's bits must be contiguous int32[{ops.grid_words(grid.c_struct())}], got "
                         f"{bits.dtype}{list(bits.shape)}")


def _sparse_surface(arch, blob, use, box, grid, level: float, want_dirs: bool, bricks_per_call, want_keys=False):
    """The sparse path (include/nerfb200.h "sparse meshes"): the grid's active bricks, the MLP at their lattice points
    (with the one-point halo when view directions are wanted), then classify, scan and emit over them.  Two host reads:
    the active brick count, which sizes the query, and the mesh's two totals."""
    halo = bool(want_dirs)
    brick_map, bricks, n_dev = ops.mesh_sparse_bricks(box, grid)
    n_active = int(n_dev.item())
    per_brick = (ops.mesh_brick() + 1 + 2 * halo) ** 3
    chunk = max(1, min(n_active, int(bricks_per_call) if bricks_per_call is not None else _SLAB_POINTS // per_brick))
    dev = blob.device
    values = torch.empty(n_active * per_brick, dtype=torch.float32, device=dev)
    if n_active:
        rows_max = -(-chunk * per_brick // 64)
        pts = torch.zeros(rows_max * 64, 3, dtype=torch.float32, device=dev)
        direction = torch.tensor([[0.0, 0.0, 1.0]], dtype=torch.float32, device=dev)
        with torch.no_grad():
            for first in range(0, n_active, chunk):
                n = min(chunk, n_active - first) * per_brick
                rows = -(-n // 64)  # the tail past n holds earlier points and is discarded
                ops.mesh_sparse_points(box, bricks, first, min(chunk, n_active - first), halo, pts)
                dirs = direction.expand(rows, 3) if arch.use_viewdirs else None
                raw = ops.mlp_fwd_pts(arch, blob, pts[:rows * 64].view(rows, 64, 3), dirs, impl=use)
                values[first * per_brick:first * per_brick + n].copy_(torch.relu(raw.view(-1, 4)[:n, 3]))
    totals, ws = ops.mesh_sparse_count(box, brick_map, bricks, n_active, values, halo, level)
    n_v, n_f = (int(t) for t in totals.tolist())
    return ops.mesh_sparse_emit(box, brick_map, bricks, n_active, values, halo, level, ws, n_v, n_f,
                                want_dirs=want_dirs, want_keys=want_keys)


def extract_mesh(model, encode_position_fn, bounds=((-1.5,) * 3, (1.5,) * 3), resolution=256, level: float = 50.0,
                 encode_direction_fn=None, colors: bool = False, impl: Optional[int] = None, *,
                 planes_per_slab: Optional[int] = None, normals: bool = False, grid=None,
                 bricks_per_call: Optional[int] = None) -> Mesh:
    """The level set sigma = ``level`` of a trained FlexibleNeRFModel over ``bounds``, by marching cubes on the GPU.

    The density is ``density_volume(model, ...)`` (the fused MLP at the (R + 1)^3 lattice points); inside is
    sigma > ``level``.  Faces are counter-clockwise seen from outside, and the mesh is closed wherever the surface stays
    inside the box.  ``colors=True`` gives each vertex sigmoid(rgb) of the same network at the vertex, seen along the
    direction of a ray reaching it head-on from outside: the normalised density gradient (-n for the outward normal n;
    +z where the gradient vanishes), from central differences of the volume at the edge's two lattice points,
    interpolated along the edge.  That query has one sample per vertex, below the wgmma forward's minimum, so it runs on
    the fp32 kernels.  ``normals=True`` sets ``Mesh.normals``: the outward unit normal -grad / |grad| of the density at
    each vertex, from the analytic gradient of ``density_gradient`` (impl 1 whatever ``impl`` the lattice query ran
    on; (0, 0, 0) where the gradient vanishes).  Argument errors raise ValueError, an unsupported model or device
    NotImplementedError, before any launch.

    ``grid`` (an ``nb.OccupancyGrid`` on the model's device) makes the extraction sparse: the lattice is cut into bricks
    of ``ops.mesh_brick()``^3 cubes, and only the bricks with a corner point in an occupied cell or outside the grid's
    box have their points queried and their cubes marched, ``bricks_per_call`` bricks per MLP call (default: about 4 M
    points).  Each lattice point gets the same value as in the dense path, so the faces are those of the dense mesh in
    the active bricks and the vertices (colors and normals too) are bit-identical, numbered brick by brick
    (include/nerfb200.h "sparse meshes").  Nothing is allocated at (R + 1)^3, so the lattice may pass 2^31 points (up to
    4096 cubes per axis).  Build the grid with ``OccupancyGrid.from_models(..., threshold=t)`` for some t below
    ``level`` (the default t = 0 is conservative): a surface in a brick the grid calls empty is missing from the mesh.
    ``planes_per_slab`` belongs to the dense path and is refused with a grid."""
    return _extract_mesh(model, encode_position_fn, bounds, resolution, level, encode_direction_fn, colors, impl,
                         planes_per_slab, normals, grid, bricks_per_call)[0]


def _extract_mesh(model, encode_position_fn, bounds, resolution, level, encode_direction_fn, colors, impl,
                  planes_per_slab, normals, grid, bricks_per_call, edge_keys=False):
    """extract_mesh, and with ``edge_keys`` on the sparse path also each vertex's lattice edge q * 3 + a (a test
    hook: the dense mesh numbers its vertices in that key's order)."""
    from . import train_utils
    from . import density

    lo, hi, res = _box(bounds, resolution, dense=grid is None)
    level = _level(level)
    if grid is not None:
        if planes_per_slab is not None:
            raise ValueError("mesh: planes_per_slab applies to the dense path; it cannot be given with grid=")
        if bricks_per_call is not None and int(bricks_per_call) < 1:
            raise ValueError(f"mesh: bricks_per_call must be >= 1, got {bricks_per_call}")
    arch = _network(model, encode_position_fn, encode_direction_fn)
    grad_impl = density.refusal(arch, None) if normals else None
    box = ops.grid_struct((lo, hi), res)
    want_dirs = colors and arch.use_viewdirs
    keys = None
    if grid is None:
        vol = density_volume(model, encode_position_fn, (lo, hi), res, encode_direction_fn=encode_direction_fn,
                             impl=impl, planes_per_slab=planes_per_slab)
        verts, faces, dirs = _surface(vol, box, level, want_dirs=want_dirs)
    else:
        _check_grid(grid, next(model.parameters()).device)
        use = _query_impl(arch, impl)
        _, blob = train_utils._packed(model, arch)
        verts, faces, dirs, keys = _sparse_surface(arch, blob, use, box, grid, level, want_dirs, bricks_per_call,
                                                   want_keys=edge_keys)
    rgb = None
    if colors:
        if verts.shape[0] == 0:
            rgb = verts.new_zeros(0, 3)
        else:
            _, blob = train_utils._packed(model, arch)
            use = train_utils._auto_impl(arch, None, 1, 0, training=False)
            with torch.no_grad():
                raw = ops.mlp_fwd_pts(arch, blob, verts.view(-1, 1, 3), dirs, impl=use)
            rgb = torch.sigmoid(raw.view(-1, 4)[:, :3])
    nrm = None
    if normals:
        _, blob = train_utils._packed(model, arch)
        _, g = density.density_grad_points(arch, blob, verts, grad_impl)
        norm = torch.linalg.vector_norm(g, dim=-1, keepdim=True)
        nrm = torch.where(norm > 0, -g / norm, torch.zeros_like(g))
    return Mesh(verts, faces, rgb, nrm), keys
