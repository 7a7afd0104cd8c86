"""CPU: the sparse meshes' brick activity, sizes and refusals (include/nerfb200.h "sparse meshes").
  1. the library's activity test (its host statement, the same function the device runs) against a numpy statement of
     the point rule: a brick is active when one of its corner lattice points lies outside the grid's box or in an
     occupied cell -- for random grids, boxes partly outside the grid, anisotropic lattices and partial bricks;
  2. the workspace and scratch sizes, and the brick count;
  3. the C symbols, and every C and Python refusal, before anything touches a device."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from nerf_pytorch_b200 import _lib, ops

FAKE = C.c_void_p(256)  # never dereferenced: every call below is refused first


def _coords(lo, hi, res):
    """p_c(i) = lo + ((hi - lo) * i) / res, fp32 with each op rounded."""
    return [np.float32(lo[c]) + (np.float32(hi[c]) - np.float32(lo[c])) * np.arange(res[c] + 1, dtype=np.float32)
            / np.float32(res[c]) for c in range(3)]


def _axis_cells(x, lo, hi, res):
    """The cell rule of "occupancy grid" along one axis: the cell of each coordinate, -1 outside [lo, hi)."""
    scale = np.float32(res) / (np.float32(hi) - np.float32(lo))
    t = (x.astype(np.float32) - np.float32(lo)) * scale
    inside = (t >= 0) & (t < np.float32(res))
    return np.where(inside, np.floor(np.where(inside, t, 0)).astype(np.int64), -1)


def _active_by_points(box_lo, box_hi, res, g_lo, g_hi, g_res, occ):
    """bool[bricks]: the point rule, corner point by corner point."""
    B = ops.mesh_brick()
    X = _coords(box_lo, box_hi, res)
    cells = [_axis_cells(X[c], g_lo[c], g_hi[c], g_res[c]) for c in range(3)]
    nb = [-(-r // B) for r in res]
    out = np.zeros(nb[0] * nb[1] * nb[2], bool)
    for b2 in range(nb[2]):
        for b1 in range(nb[1]):
            for b0 in range(nb[0]):
                idx = [np.arange(b * B, min(b * B + B, r) + 1) for b, r in zip((b0, b1, b2), res)]
                c0, c1, c2 = np.meshgrid(cells[0][idx[0]], cells[1][idx[1]], cells[2][idx[2]], indexing="ij")
                outside = (c0 < 0) | (c1 < 0) | (c2 < 0)
                occupied = occ[np.where(outside, 0, c2), np.where(outside, 0, c1), np.where(outside, 0, c0)]
                out[(b2 * nb[1] + b1) * nb[0] + b0] = bool((outside | occupied).any())
    return out


CASES = [
    # (box lo, box hi, lattice res), (grid lo, grid hi, grid res), occupancy
    ((-1, -1, -1), (1, 1, 1), (64, 64, 64), (-1, -1, -1), (1, 1, 1), (16, 16, 16), 0.1),
    ((-1, -1, -1), (1, 1, 1), (37, 21, 50), (-1, -1, -1), (1, 1, 1), (32, 8, 20), 0.5),
    ((-1.5, -1.5, -1.5), (1.5, 1.5, 1.5), (40, 40, 40), (-1, -1.2, -0.5), (1, 1, 1.7), (12, 30, 9), 0.2),
    ((0, 0, 0), (1, 2, 3), (17, 33, 9), (0.25, -1, 0.5), (3, 1.5, 2.0), (7, 7, 7), 0.9),
    ((-1, -1, -1), (1, 1, 1), (24, 24, 24), (-1, -1, -1), (1, 1, 1), (100, 100, 100), 0.01),  # finer grid than lattice
    ((-1, -1, -1), (1, 1, 1), (30, 30, 30), (-1, -1, -1), (1, 1, 1), (5, 5, 5), 0.0),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_activity_is_the_point_rule(case):
    box_lo, box_hi, res, g_lo, g_hi, g_res, frac = CASES[case]
    rng = np.random.default_rng(case)
    occ = rng.random((g_res[2], g_res[1], g_res[0])) < frac
    from nerf_pytorch_b200.occupancy import pack_bits

    bits = pack_bits(torch.from_numpy(occ))
    got = ops.mesh_sparse_bricks_host(ops.grid_struct((box_lo, box_hi), res), ops.grid_struct((g_lo, g_hi), g_res),
                                      bits).numpy()
    want = _active_by_points(box_lo, box_hi, res, g_lo, g_hi, g_res, occ)
    print(f"[mesh_sparse] case {case}: {int(want.sum())} of {want.size} bricks active")
    assert got.shape == want.shape and np.array_equal(got, want)


def test_sizes():
    B = ops.mesh_brick()
    assert B == 8
    box = ops.grid_struct(((-1,) * 3, (1,) * 3), (100, 17, 4096))
    nb = (-(-100 // B)) * (-(-17 // B)) * (4096 // B)
    assert ops.mesh_sparse_brick_count(box) == nb
    a16 = lambda b: (b + 15) // 16 * 16  # noqa: E731
    groups = -(-(B + 1) ** 3 // 32)
    for n in (0, 1, 5, 1000):
        want = a16(n * groups * 16) + 2 * a16(4 * n) + 2 * a16(8 * n)
        assert ops.mesh_sparse_workspace_bytes(box, n) == want
    tiles = -(-nb // 256)
    assert ops.mesh_sparse_scratch_bytes(box) == a16(3 * 4097 * 4) + a16(4 * tiles) + 2 * a16(8 * tiles) + 16
    big = ops.grid_struct(((-1,) * 3, (1,) * 3), (4096, 4096, 4096))  # past the dense path's 2^31 points
    assert ops.mesh_sparse_brick_count(big) == 512 ** 3


def test_symbols_and_c_refusals():
    lib = _lib.load()
    names = ("nerfb200_mesh_brick", "nerfb200_mesh_sparse_brick_count", "nerfb200_mesh_sparse_scratch_bytes",
             "nerfb200_mesh_sparse_workspace_bytes", "nerfb200_mesh_sparse_bricks", "nerfb200_mesh_sparse_bricks_host",
             "nerfb200_mesh_sparse_points", "nerfb200_mesh_sparse_count", "nerfb200_mesh_sparse_emit")
    for name in names:
        assert name in _lib.SIGNATURES and hasattr(lib, name)
    ok = ops.grid_struct(((-1,) * 3, (1,) * 3), (64, 64, 64))
    bad_boxes = [ops.grid_struct(((-1,) * 3, (1,) * 3), (0, 64, 64)),
                 ops.grid_struct(((-1,) * 3, (1,) * 3), (64, 64, 4097)),
                 ops.grid_struct(((1, -1, -1), (-1, 1, 1)), (64, 64, 64)),
                 ops.grid_struct(((-1, -1, math.nan), (1, 1, 1)), (64, 64, 64))]
    before = ops.launch_count()
    for bad in bad_boxes:
        assert lib.nerfb200_mesh_sparse_brick_count(C.byref(bad)) == -1
        assert lib.nerfb200_mesh_sparse_scratch_bytes(C.byref(bad)) == -1
        assert lib.nerfb200_mesh_sparse_workspace_bytes(C.byref(bad), 1) == -1
        for box, grid in ((bad, ok), (ok, bad)):
            assert lib.nerfb200_mesh_sparse_bricks(C.byref(box), C.byref(grid), FAKE, FAKE, FAKE, FAKE, FAKE,
                                                   None) == _lib.ERR_INVALID
            assert lib.nerfb200_mesh_sparse_bricks_host(C.byref(box), C.byref(grid), FAKE, FAKE) == _lib.ERR_INVALID
        assert lib.nerfb200_mesh_sparse_points(C.byref(bad), FAKE, 0, 1, 0, FAKE, None) == _lib.ERR_INVALID
        assert lib.nerfb200_mesh_sparse_count(C.byref(bad), FAKE, FAKE, 1, FAKE, 0, 0.5, FAKE, FAKE,
                                              None) == _lib.ERR_INVALID
        assert lib.nerfb200_mesh_sparse_emit(C.byref(bad), FAKE, FAKE, 1, FAKE, 0, 0.5, FAKE, 1, 1, FAKE, FAKE, None,
                                             None, None) == _lib.ERR_INVALID
    nb = ops.mesh_sparse_brick_count(ok)
    assert lib.nerfb200_mesh_sparse_workspace_bytes(C.byref(ok), nb + 1) == -1
    assert lib.nerfb200_mesh_sparse_workspace_bytes(C.byref(ok), -1) == -1
    # null pointers
    for i in range(5):
        ptrs = [FAKE] * 5
        ptrs[i] = None
        assert lib.nerfb200_mesh_sparse_bricks(C.byref(ok), C.byref(ok), *ptrs, None) == _lib.ERR_INVALID
    assert lib.nerfb200_mesh_sparse_bricks_host(C.byref(ok), C.byref(ok), None, FAKE) == _lib.ERR_INVALID
    # points: null, halo, brick range
    for args in ((None, 0, 1, 0, FAKE), (FAKE, 0, 1, 0, None), (FAKE, 0, 1, 2, FAKE), (FAKE, -1, 1, 0, FAKE),
                 (FAKE, 0, 0, 0, FAKE), (FAKE, nb - 1, 2, 0, FAKE)):
        assert lib.nerfb200_mesh_sparse_points(C.byref(ok), *args, None) == _lib.ERR_INVALID
    # count / emit: level, halo, active count, null pointers, view directions without the halo
    for level, halo, n, vals, ws in ((math.nan, 0, 1, FAKE, FAKE), (math.inf, 0, 1, FAKE, FAKE),
                                     (0.5, 2, 1, FAKE, FAKE), (0.5, 0, -1, FAKE, FAKE), (0.5, 0, nb + 1, FAKE, FAKE),
                                     (0.5, 0, 1, None, FAKE), (0.5, 0, 1, FAKE, None)):
        assert lib.nerfb200_mesh_sparse_count(C.byref(ok), FAKE, FAKE, n, vals, halo, level, ws, FAKE,
                                              None) == _lib.ERR_INVALID
        assert lib.nerfb200_mesh_sparse_emit(C.byref(ok), FAKE, FAKE, n, vals, halo, level, ws, 1, 1, FAKE, FAKE,
                                             None, None, None) == _lib.ERR_INVALID
    assert lib.nerfb200_mesh_sparse_count(C.byref(ok), None, FAKE, 1, FAKE, 0, 0.5, FAKE, FAKE,
                                          None) == _lib.ERR_INVALID
    assert lib.nerfb200_mesh_sparse_count(C.byref(ok), FAKE, FAKE, 1, FAKE, 0, 0.5, FAKE, None,
                                          None) == _lib.ERR_INVALID
    assert lib.nerfb200_mesh_sparse_emit(C.byref(ok), FAKE, FAKE, 1, FAKE, 0, 0.5, FAKE, 1, 1, FAKE, FAKE, FAKE,
                                         None, None) == _lib.ERR_INVALID  # view directions need the halo
    assert lib.nerfb200_mesh_sparse_emit(C.byref(ok), FAKE, FAKE, 1, FAKE, 1, 0.5, FAKE, 1, 1, None, FAKE, None,
                                         None, None) == _lib.ERR_INVALID
    assert lib.nerfb200_mesh_sparse_emit(C.byref(ok), FAKE, FAKE, 1, FAKE, 1, 0.5, FAKE, 2 ** 31 + 1, 1, FAKE, FAKE,
                                         None, None, None) == _lib.ERR_UNSUPPORTED
    assert ops.launch_count() == before


def test_python_refusals_fire_before_any_launch():
    import nerf_pytorch_b200 as nb

    model = nb.FlexibleNeRFModel()  # on the CPU
    epf = nb.get_embedding_function(6)
    box = ((-1.0,) * 3, (1.0,) * 3)
    grid = nb.OccupancyGrid(box, 8, torch.zeros(16, dtype=torch.int32))  # bits on the CPU
    before = ops.launch_count()
    for kw, err in ((dict(grid=grid, planes_per_slab=4), ValueError), (dict(grid=grid, bricks_per_call=0), ValueError),
                    (dict(grid=grid, resolution=4097), ValueError), (dict(grid=grid, resolution=1), ValueError),
                    (dict(grid=grid, level=math.nan), ValueError), (dict(grid=grid), NotImplementedError),
                    (dict(grid="full"), NotImplementedError)):
        args = dict(bounds=box, resolution=16, level=1.0)
        args.update(kw)
        with pytest.raises(err):
            nb.extract_mesh(model, epf, **args)
    # a 2048^3 lattice is past the dense path's limit, but not the sparse path's: it fails here on the CPU model only
    with pytest.raises(ValueError):
        nb.extract_mesh(model, epf, box, 2048)
    with pytest.raises(NotImplementedError, match="CUDA"):
        nb.extract_mesh(model, epf, box, 2048, grid=grid)
    assert ops.launch_count() == before
