"""CPU: the occupancy grid's layout and the refusals of grid renders that need no GPU.
  1. the header's cell rule: the library's host restatement (nerfb200_grid_locate) and OccupancyGrid.cell_of give the same
     cell for every point, on cell boundaries, at the box's faces and for NaN;
  2. the bit order: pack_bits / unpack_bits round-trip, and cell idx is bit idx & 31 of word idx >> 5;
  3. descriptor checks and workspace queries;
  4. a training call with a grid raises before it touches the rays (CPU tensors reach the check)."""
import ctypes as C

import pytest
import torch


def _grid_struct(bounds, res):
    from nerf_pytorch_b200 import ops

    return ops.grid_struct(bounds, res)


def test_cell_rule_matches_the_library_host_restatement():
    from nerf_pytorch_b200 import ops
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    bounds = ((-1.5, -1.25, -0.3), (1.5, 1.75, 2.1))
    res = (37, 64, 5)
    g = OccupancyGrid(bounds, res, torch.zeros(ops.grid_words(_grid_struct(bounds, res)), dtype=torch.int32))
    gen = torch.Generator().manual_seed(0)
    lo, hi = torch.tensor(bounds[0]), torch.tensor(bounds[1])
    pts = lo + (hi - lo) * (torch.rand(20000, 3, generator=gen) * 1.2 - 0.1)
    # exact cell boundaries and faces, their fp32 neighbours, and NaN
    edges = lo + (hi - lo) * torch.stack([torch.arange(r + 1).float() / r for r in res[:1]] * 3, -1)[:, :3]
    faces = torch.stack((torch.nextafter(edges, edges - 1), edges, torch.nextafter(edges, edges + 1)), 0).reshape(-1, 3)
    nan = torch.tensor([[float("nan"), 0.0, 0.5]])
    pts = torch.cat((pts, faces, nan))
    want = ops.grid_locate(g.c_struct(), pts)
    got = g.cell_of(pts)
    assert torch.equal(got, want)
    assert (want == -1).any() and (want >= 0).any() and want[-1] == -1
    assert want.max() < res[0] * res[1] * res[2]


def test_bits_follow_the_header_order():
    from nerf_pytorch_b200.occupancy import pack_bits, unpack_bits

    gen = torch.Generator().manual_seed(1)
    occ = torch.rand(5, 7, 9, generator=gen) < 0.4
    bits = pack_bits(occ)
    assert bits.dtype == torch.int32 and bits.numel() == (5 * 7 * 9 + 31) // 32
    assert torch.equal(unpack_bits(bits, (9, 7, 5)), occ)
    flat = occ.reshape(-1)
    w = bits.to(torch.int64) & 0xFFFFFFFF
    for idx in range(flat.numel()):
        assert bool((w[idx >> 5] >> (idx & 31)) & 1) == bool(flat[idx])
    iz, iy, ix = 3, 2, 8
    assert flat[(iz * 7 + iy) * 9 + ix] == occ[iz, iy, ix]


def test_descriptor_checks_and_queries():
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    assert ops.grid_words(_grid_struct(((0, 0, 0), (1, 1, 1)), (128, 128, 128))) == 128 ** 3 // 32
    for bad in ((((0, 0, 0), (1, 1, 1)), (0, 4, 4)), (((0, 0, 0), (1, 1, 1)), (4, 4, 4097)),
                (((0, 0, 0), (1, 0, 1)), (4, 4, 4)), (((0, 0, float("nan")), (1, 1, 1)), (4, 4, 4))):
        assert lib.nerfb200_grid_words(C.byref(_grid_struct(*bad))) == -1
        assert "invalid grid" in lib.nerfb200_last_error().decode()
    assert lib.nerfb200_grid_max_blocks(25, 64) == 3 * 10
    assert lib.nerfb200_grid_max_blocks(1, 15) == 3
    assert lib.nerfb200_grid_scratch_ints(25, 64) == 25 * 64 + 6
    arch = ops.ArchSpec(num_layers=4, hidden=128, n_freq_xyz=10)
    opts = ops.make_opts(64, 128, True, False, False, 1.0)
    base = ops.render_workspace_bytes(arch, arch, opts, 4096, False)
    assert ops.render_grid_workspace_bytes(arch, arch, opts, 4096) > base


def test_training_call_with_a_grid_raises_before_touching_the_rays():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200.occupancy import OccupancyGrid
    from oracle import nerf_oracle as O

    mc, mf = nb.FlexibleNeRFModel(), nb.FlexibleNeRFModel()
    opts = O.make_options()
    epf, edf = nb.get_embedding_function(6), nb.get_embedding_function(4)
    grid = OccupancyGrid.full(((-2, -2, -2), (2, 2, 2)), 8, device="cpu")
    with pytest.raises(NotImplementedError, match="inference"):
        nb.predict_and_render_radiance(torch.zeros(4, 11), mc, mf, opts, encode_position_fn=epf,
                                       encode_direction_fn=edf, grid=grid)
    with pytest.raises(TypeError, match="OccupancyGrid"):
        with torch.no_grad():
            nb.predict_and_render_radiance(torch.zeros(4, 11), mc, mf, opts, encode_position_fn=epf,
                                           encode_direction_fn=edf, grid=object())
