"""Host: subdividing baked fields (include/nerfb200.h "baked fields: subdivision"): the ABI symbol, its signature and
the Python exports, every C-level refusal before any launch, the Python refusals of nb.subdivide_baked,
BakedFieldTrainer.subdivide and nb.BakedField.full, and the child-brick list restated in numpy against a brute force
over the child box's bricks.  No GPU."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "nerfb200_baked_subdivide"


def test_abi_symbol_signature_and_exports():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import _lib, ops

    with open(os.path.join(ROOT, "include", "nerfb200.h")) as f:
        header = f.read()
    assert re.search(r"int32_t\s+" + NAME + r"\(", header)
    assert "baked fields: subdivision" in header
    lib = _lib.load()
    assert hasattr(lib, NAME)
    P, I32, I64 = C.c_void_p, C.c_int32, C.c_int64
    assert _lib.SIGNATURES[NAME] == (I32, [C.POINTER(_lib.Grid), P, I64, P, P, I64, P, P])
    assert "subdivide_baked" in nb.__all__ and callable(nb.subdivide_baked)
    assert callable(nb.BakedField.full) and callable(nb.BakedFieldTrainer.subdivide) and callable(ops.baked_subdivide)


def test_entry_point_refuses_before_any_launch():
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    f = lib.nerfb200_baked_subdivide
    before = ops.launch_count()
    box = ops.grid_struct(((-1.0,) * 3, (1.0,) * 3), (16, 16, 16))  # 8 parent bricks, 64 child bricks
    per = 729 * 32 * 4
    a, b = C.c_void_p(1 << 20), C.c_void_p(1 << 30)  # far apart: no overlap
    # an invalid box; a child resolution past 4096 on one axis (2049 -> 4098); 2048 is accepted by the checks
    for lo, hi, res in (((1.0,) * 3, (-1.0,) * 3, (16,) * 3), ((-1.0,) * 3, (1.0,) * 3, (0, 16, 16)),
                        ((-1.0,) * 3, (1.0,) * 3, (16, 2049, 16)), ((-1.0,) * 3, (1.0,) * 3, (16, 16, 4096))):
        bad = ops.grid_struct((lo, hi), res)
        assert f(C.byref(bad), a, 1, a, b, 1, b, None) == _lib.ERR_INVALID, res
    assert f(None, a, 1, a, b, 1, b, None) == _lib.ERR_INVALID
    # every null pointer
    for i in range(4):
        ptrs = [a, a, b, b]
        ptrs[i] = None
        bm, vals, cb, cv = ptrs
        assert f(C.byref(box), bm, 1, vals, cb, 1, cv, None) == _lib.ERR_INVALID, i
    # counts: n_active outside 0 .. 8, n_child outside 0 .. 64
    for n_active, n_child in ((-1, 1), (9, 1), (1, -1), (1, 65)):
        assert f(C.byref(box), a, n_active, a, b, n_child, b, None) == _lib.ERR_INVALID, (n_active, n_child)
    # child_values overlapping values: equal, inside, straddling either end
    base = 1 << 24
    for cv in (base, base + 16, base + 3 * per - 16, base - per + 16):
        assert f(C.byref(box), a, 3, C.c_void_p(base), b, 2, C.c_void_p(cv), None) == _lib.ERR_INVALID, cv
    assert "baked_subdivide" in lib.nerfb200_last_error().decode()
    # a count of 0 with disjoint buffers is accepted and launches nothing; so is a child that just touches values
    assert f(C.byref(box), a, 3, C.c_void_p(base), b, 0, C.c_void_p(base + 3 * per), None) == _lib.OK
    assert f(C.byref(box), a, 0, C.c_void_p(base), b, 0, C.c_void_p(base), None) == _lib.OK
    assert ops.launch_count() == before


def _cpu_field(res, active=0.6, seed=0, viewdirs=True):
    import nerf_pytorch_b200 as nb

    g = torch.Generator().manual_seed(seed)
    nb_ = [-(-r // 8) for r in res]
    act = torch.rand(nb_[0] * nb_[1] * nb_[2], generator=g) < active
    act[0] = True
    brick_map = torch.where(act, torch.cumsum(act.int(), 0) - 1, -1).int()
    bricks = torch.nonzero(act).reshape(-1).int()
    return nb.BakedField(((-1.0,) * 3, (1.0,) * 3), res, brick_map, bricks, torch.zeros(bricks.numel(), 1, 1),
                         viewdirs)


def test_python_refusals_precede_any_launch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    before = ops.launch_count()
    f = _cpu_field((16, 16, 16))
    f.values = torch.zeros(f.n_active, 729, 32)
    with pytest.raises(ValueError, match="BakedField"):
        nb.subdivide_baked(object())
    with pytest.raises(ValueError, match="CUDA"):  # a CPU field
        nb.subdivide_baked(f)
    h = nb.BakedField(f.bounds, f.resolution, f.brick_map, f.bricks, f.values.half(), True)
    with pytest.raises(ValueError, match=r"subdivide field\.float\(\)"):
        nb.subdivide_baked(h)
    big = nb.BakedField(f.bounds, (16, 2049, 16), f.brick_map, f.bricks, torch.zeros(1, 729, 32, device="meta"), True)
    with pytest.raises(ValueError, match="2048"):
        nb.subdivide_baked(big)
    # BakedFieldTrainer.subdivide: the same refusals, before the field or the buffers change
    for field, match in ((h, "float"), (f, "CUDA"), (big, "2048")):
        t = nb.BakedFieldTrainer.__new__(nb.BakedFieldTrainer)
        t.field, t.d_values, t.m = field, "grad", "m"
        snap = (field.resolution, field.brick_map, field.bricks, field.values)
        with pytest.raises(ValueError, match=match):
            t.subdivide()
        assert (field.resolution, field.brick_map, field.bricks, field.values) == snap
        assert t.d_values == "grad" and t.m == "m"
    # BakedField.full: the bake's box checks and a finite sigma_raw
    for bounds, res in ((((1.0,) * 3, (-1.0,) * 3), 16), ((((-1.0,) * 3, (1.0,) * 3)), 1),
                        ((((-1.0,) * 3, (1.0,) * 3)), 4097), ((((-1.0,) * 3, (1.0,) * 3)), (16, 16)),
                        ((((-1.0,) * 3, (float("inf"),) * 3)), 16)):
        with pytest.raises(ValueError, match="mesh"):
            nb.BakedField.full(bounds, res, device="cpu")
    for s in (float("nan"), float("inf"), -float("inf")):
        with pytest.raises(ValueError, match="sigma_raw"):
            nb.BakedField.full(((-1.0,) * 3, (1.0,) * 3), 16, sigma_raw=s, device="cpu")
    assert ops.launch_count() == before


def test_full_field_on_the_cpu():
    import nerf_pytorch_b200 as nb

    f = nb.BakedField.full(((-1.0, -2.0, -0.5), (1.0, 2.0, 0.5)), (20, 13, 37), sigma_raw=0.25, use_viewdirs=False,
                           device="cpu")
    n = 3 * 2 * 5
    assert f.n_active == n and f.resolution == (20, 13, 37) and not f.use_viewdirs and f.dtype == torch.float32
    assert f.bounds == ((-1.0, -2.0, -0.5), (1.0, 2.0, 0.5))
    assert torch.equal(f.brick_map, torch.arange(n, dtype=torch.int32))
    assert torch.equal(f.bricks, torch.arange(n, dtype=torch.int32))
    assert f.values.shape == (n, 729, 32)
    assert bool((f.values[..., 0] == 0.25).all()) and bool((f.values[..., 1:] == 0).all())


def _brute_children(res, bricks):
    """The child box's bricks (ascending) whose parent brick (each coordinate halved) is in ``bricks``, by a pass over
    every child brick in numpy."""
    nbp = [-(-r // 8) for r in res]
    nbc = [-(-2 * r // 8) for r in res]
    active = np.zeros(nbp[0] * nbp[1] * nbp[2], dtype=bool)
    active[np.asarray(bricks, dtype=np.int64)] = True
    cid = np.arange(nbc[0] * nbc[1] * nbc[2])
    cx, cy, cz = cid % nbc[0], cid // nbc[0] % nbc[1], cid // (nbc[0] * nbc[1])
    # a child brick exists in the child box by construction (8 c < 2 res); its parent is floor(c / 2)
    assert bool(((8 * cx < 2 * res[0]) & (8 * cy < 2 * res[1]) & (8 * cz < 2 * res[2])).all())
    parent = ((cz // 2) * nbp[1] + cy // 2) * nbp[0] + cx // 2
    return cid[active[parent]], nbc


@pytest.mark.parametrize("res,active,seed", [
    ((16, 16, 16), 1.0, 0), ((16, 16, 16), 0.4, 1), ((20, 13, 37), 0.5, 2), ((20, 13, 37), 1.0, 3),
    ((9, 8, 7), 1.0, 4), ((17, 33, 2), 0.7, 5), ((2048, 12, 20), 0.3, 6), ((24, 2048, 9), 0.05, 7)])
def test_child_bricks_against_a_brute_force(res, active, seed):
    from nerf_pytorch_b200.bake import _child_bricks

    f = _cpu_field(res, active, seed)
    child = tuple(2 * r for r in res)
    brick_map, bricks = _child_bricks(f, child)
    want, nbc = _brute_children(res, f.bricks.numpy())
    assert bricks.dtype == torch.int32 and brick_map.dtype == torch.int32
    assert brick_map.shape == (nbc[0] * nbc[1] * nbc[2],)
    np.testing.assert_array_equal(bricks.numpy(), want)
    # brick_map is the rank of bricks, -1 elsewhere
    rank = np.full(brick_map.numel(), -1, dtype=np.int32)
    rank[want] = np.arange(want.size, dtype=np.int32)
    np.testing.assert_array_equal(brick_map.numpy(), rank)
    # per axis a parent brick has 2 children, or 1 when it is a partial brick on the upper face holding <= 4 cubes
    nbp = [-(-r // 8) for r in res]
    per_axis = [np.where((np.arange(nbp[c]) == nbp[c] - 1) & (res[c] - 8 * (nbp[c] - 1) <= 4), 1, 2) for c in range(3)]
    b = f.bricks.numpy().astype(np.int64)
    n = per_axis[0][b % nbp[0]] * per_axis[1][b // nbp[0] % nbp[1]] * per_axis[2][b // (nbp[0] * nbp[1])]
    assert int(n.sum()) == want.size


def test_child_bricks_of_an_empty_field():
    from nerf_pytorch_b200.bake import _child_bricks

    f = _cpu_field((20, 13, 37))
    f.bricks = f.bricks[:0]
    brick_map, bricks = _child_bricks(f, (40, 26, 74))
    assert bricks.numel() == 0 and brick_map.numel() == 5 * 4 * 10 and bool((brick_map == -1).all())
