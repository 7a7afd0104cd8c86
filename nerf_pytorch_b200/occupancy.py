"""Occupancy grids for inference renders: a bitfield over a box that says which cells the network's density leaves empty,
so that ``render_image(..., grid=...)`` (and the other render entry points) run the MLP only on samples in occupied cells
or outside the box.  A skipped sample gets exactly zero density.

The layout -- the box, the cell rule and the bit order -- is defined once, in include/nerfb200.h (``nerfb200_grid_t``);
this file packs bits in that order and builds grids from models.  Building runs once per scene, so it uses torch ops
around the library's MLP forward."""
from __future__ import annotations

from typing import Optional, Sequence

import torch

from . import ops


def _resolution(resolution):
    if isinstance(resolution, int):
        resolution = (resolution,) * 3
    res = tuple(int(r) for r in resolution)
    if len(res) != 3:
        raise ValueError(f"OccupancyGrid: resolution must be an int or three ints, got {resolution!r}")
    return res


def _bounds(bounds):
    lo, hi = bounds
    lo, hi = tuple(float(v) for v in lo), tuple(float(v) for v in hi)
    if len(lo) != 3 or len(hi) != 3:
        raise ValueError(f"OccupancyGrid: bounds must be ((x0, y0, z0), (x1, y1, z1)), got {bounds!r}")
    return lo, hi


def pack_bits(occupied: torch.Tensor) -> torch.Tensor:
    """(res_z, res_y, res_x) bool -> int32 words: cell (i_z * res_y + i_y) * res_x + i_x at bit (idx & 31) of word
    idx >> 5, least significant bit first (include/nerfb200.h)."""
    flat = occupied.reshape(-1).to(torch.int64)
    pad = (-flat.numel()) % 32
    if pad:
        flat = torch.cat((flat, flat.new_zeros(pad)))
    words = (flat.view(-1, 32) << torch.arange(32, device=flat.device)).sum(1)
    return torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)


def unpack_bits(bits: torch.Tensor, resolution) -> torch.Tensor:
    """Inverse of pack_bits: (res_z, res_y, res_x) bool."""
    rx, ry, rz = resolution
    w = bits.to(torch.int64) & 0xFFFFFFFF
    flat = ((w[:, None] >> torch.arange(32, device=bits.device)) & 1).reshape(-1)[: rx * ry * rz]
    return flat.bool().view(rz, ry, rx)


class OccupancyGrid:
    """A bitfield of ``resolution`` cells (an int or (res_x, res_y, res_z)) over the box ``bounds`` = ((x0, y0, z0),
    (x1, y1, z1)) in the coordinates the MLP encodes: world space for Blender scenes, NDC for forward-facing (LLFF) ones.
    ``bits`` are int32 words on the device the render runs on.  A sample inside the box whose cell is clear is skipped;
    a sample outside the box is always evaluated."""

    def __init__(self, bounds, resolution, bits: torch.Tensor):
        self.bounds = _bounds(bounds)
        self.resolution = _resolution(resolution)
        self.bits = bits
        n = ops.grid_words(self.c_struct())
        if bits.dtype != torch.int32 or bits.dim() != 1 or bits.numel() != n:
            raise ValueError(f"OccupancyGrid: bits must be int32[{n}], got {bits.dtype}{list(bits.shape)}")

    def c_struct(self):
        return ops.grid_struct(self.bounds, self.resolution)

    @property
    def device(self):
        return self.bits.device

    def to(self, device) -> "OccupancyGrid":
        return OccupancyGrid(self.bounds, self.resolution, self.bits.to(device))

    @classmethod
    def from_occupancy(cls, bounds, occupied: torch.Tensor) -> "OccupancyGrid":
        """From a (res_z, res_y, res_x) bool tensor."""
        rz, ry, rx = occupied.shape
        return cls(bounds, (rx, ry, rz), pack_bits(occupied))

    @classmethod
    def full(cls, bounds, resolution=128, device=None) -> "OccupancyGrid":
        rx, ry, rz = _resolution(resolution)
        return cls.from_occupancy(bounds, torch.ones(rz, ry, rx, dtype=torch.bool, device=device or "cuda"))

    @classmethod
    def empty(cls, bounds, resolution=128, device=None) -> "OccupancyGrid":
        rx, ry, rz = _resolution(resolution)
        return cls.from_occupancy(bounds, torch.zeros(rz, ry, rx, dtype=torch.bool, device=device or "cuda"))

    def occupancy(self) -> torch.Tensor:
        """(res_z, res_y, res_x) bool."""
        return unpack_bits(self.bits, self.resolution)

    @property
    def occupied_fraction(self) -> float:
        rx, ry, rz = self.resolution
        return self.occupancy().sum().item() / (rx * ry * rz)

    def cell_of(self, xyz: torch.Tensor) -> torch.Tensor:
        """The cell rule of include/nerfb200.h in torch fp32 ops: int64 cell index of each point of (..., 3), -1 outside
        the box."""
        lo = torch.tensor(self.bounds[0], dtype=torch.float32, device=xyz.device)
        hi = torch.tensor(self.bounds[1], dtype=torch.float32, device=xyz.device)
        res = torch.tensor(self.resolution, dtype=torch.float32, device=xyz.device)
        scale = res / (hi - lo)
        t = (xyz.float() - lo) * scale
        inside = ((t >= 0) & (t < res)).all(-1)
        i = torch.where(inside[..., None], t, torch.zeros_like(t)).to(torch.int64)
        idx = (i[..., 2] * self.resolution[1] + i[..., 1]) * self.resolution[0] + i[..., 0]
        return torch.where(inside, idx, torch.full_like(idx, -1))

    @classmethod
    def from_models(cls, models: Sequence, encode_position_fn, bounds, resolution=128, threshold: float = 0.0,
                    probes_per_cell: int = 8, seed: int = 0, *, encode_direction_fn=None, impl: Optional[int] = None,
                    cells_per_batch: int = 1 << 18) -> "OccupancyGrid":
        """Probe every cell of the box at ``probes_per_cell`` seeded uniform points through each network's fused MLP
        (``ops.mlp_fwd_pts``): a cell is occupied when max over its probes of relu(sigma) exceeds ``threshold`` for any
        of ``models``; the occupied set is then dilated by one cell.  sigma reads the trunk alone (fc_alpha), so the view
        direction of the probes is irrelevant; ``encode_direction_fn`` defaults to the stock encoder of the width the
        model's layers_dir[0] expects."""
        from . import train_utils
        from .nerf_helpers import get_embedding_function

        lo, hi = _bounds(bounds)
        rx, ry, rz = _resolution(resolution)
        models = [m for m in models if m is not None]
        if not models:
            raise ValueError("OccupancyGrid.from_models: no model given")
        dev = next(models[0].parameters()).device
        enc_xyz = train_utils._probe_encoder(encode_position_fn, None)
        nets = []
        for m in models:
            enc_dir = None
            if hasattr(m, "fc_rgb"):
                if encode_direction_fn is not None:
                    enc_dir = train_utils._probe_encoder(encode_direction_fn, None)
                else:
                    dim = m.layers_dir[0].in_features - m.layer1.out_features
                    enc_dir = train_utils._probe_encoder(get_embedding_function((dim - 3) // 6), None)
            arch = train_utils._arch_of(m, enc_xyz, enc_dir)
            _, blob = train_utils._packed(m, arch)
            use = train_utils._auto_impl(arch, None, 64, 0, training=False) if impl is None else int(impl)
            nets.append((arch, blob, use))

        n_cells = rx * ry * rz
        lo_t = torch.tensor(lo, dtype=torch.float32, device=dev)
        size = (torch.tensor(hi, dtype=torch.float32, device=dev) - lo_t) / torch.tensor((rx, ry, rz),
                                                                                        dtype=torch.float32, device=dev)
        gen = torch.Generator(device=dev).manual_seed(int(seed))
        occ = torch.zeros(n_cells, dtype=torch.bool, device=dev)
        direction = torch.tensor([[0.0, 0.0, 1.0]], device=dev)
        with torch.no_grad():
            for c0 in range(0, n_cells, cells_per_batch):
                idx = torch.arange(c0, min(c0 + cells_per_batch, n_cells), device=dev)
                cell = torch.stack((idx % rx, (idx // rx) % ry, idx // (rx * ry)), -1).float()
                u = torch.rand(idx.numel(), probes_per_cell, 3, generator=gen, device=dev)
                pts = lo_t + (cell[:, None, :] + u) * size
                pts = pts.reshape(-1, 64, 3) if pts.numel() % 192 == 0 else pts.reshape(1, -1, 3)
                for arch, blob, use in nets:
                    dirs = direction.expand(pts.shape[0], 3) if arch.use_viewdirs else None
                    raw = ops.mlp_fwd_pts(arch, blob, pts, dirs, impl=use)
                    sigma = torch.relu(raw[..., 3]).reshape(idx.numel(), probes_per_cell).amax(1)
                    occ[c0:c0 + idx.numel()] |= sigma > threshold
        occ3 = occ.view(rz, ry, rx)
        dil = torch.nn.functional.max_pool3d(occ3[None, None].float(), 3, stride=1, padding=1)[0, 0] > 0
        return cls.from_occupancy((lo, hi), dil)
