"""Host: the baked-field regularisers' entry points (include/nerfb200.h "baked fields: regularisers"): ABI symbols and
signatures, every C-level refusal before any launch, the Python refusals of nb.baked_regularizer and the trainer's
weights, and the lattice's points and edges restated in numpy (restated here) against a brute force over the
cubes of the active bricks, with P from the restatement.  No GPU."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

from helpers import baked_lattice

NAMES = ("nerfb200_baked_lattice_count", "nerfb200_baked_regularizer")


def test_abi_symbols_and_signatures():
    from nerf_pytorch_b200 import _lib

    lib = _lib.load()
    P, I32, I64, F64 = C.c_void_p, C.c_int32, C.c_int64, C.c_double
    GP = C.POINTER(_lib.Grid)
    want = {
        "nerfb200_baked_lattice_count": (I32, [GP, P, P, I64, P, P]),
        "nerfb200_baked_regularizer": (I32, [GP, P, P, I64, P, P, F64, F64, F64, P, P, P]),
    }
    for name in NAMES:
        assert hasattr(lib, name)
        assert _lib.SIGNATURES[name] == want[name], name


def test_entry_points_refuse_before_any_launch():
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    before = ops.launch_count()
    box = ops.grid_struct(((-1.0,) * 3, (1.0,) * 3), (16, 16, 16))  # 8 bricks
    bad_box = ops.grid_struct(((1.0,) * 3, (-1.0,) * 3), (16, 16, 16))
    fake, other = C.c_void_p(256), C.c_void_p(1 << 40)
    # baked_lattice_count: box, pointers, n_active
    k = lib.nerfb200_baked_lattice_count
    assert k(C.byref(bad_box), fake, fake, 1, fake, None) == _lib.ERR_INVALID
    for i in range(3):
        ptrs = [fake] * 3
        ptrs[i] = None
        assert k(C.byref(box), ptrs[0], ptrs[1], 1, ptrs[2], None) == _lib.ERR_INVALID, i
    assert k(C.byref(box), fake, fake, 0, fake, None) == _lib.ERR_INVALID
    assert k(C.byref(box), fake, fake, 9, fake, None) == _lib.ERR_INVALID
    # baked_regularizer: box, pointers, n_active, weights, aliasing
    r = lib.nerfb200_baked_regularizer

    def reg(box_=box, bm=fake, br=fake, n=1, vals=fake, cnt=fake, lam=(1.0, 1.0, 1.0), d=other, part=other):
        return r(C.byref(box_), bm, br, n, vals, cnt, *lam, d, part, None)

    assert reg(box_=bad_box) == _lib.ERR_INVALID
    assert reg(bm=None) == _lib.ERR_INVALID
    assert reg(br=None) == _lib.ERR_INVALID
    assert reg(vals=None) == _lib.ERR_INVALID
    assert reg(cnt=None) == _lib.ERR_INVALID
    assert reg(d=None, part=None) == _lib.ERR_INVALID
    assert reg(n=0) == _lib.ERR_INVALID
    assert reg(n=-1) == _lib.ERR_INVALID
    assert reg(n=9) == _lib.ERR_INVALID
    for bad in (-1.0, float("nan"), float("inf"), -0.5e-30):
        for i in range(3):
            lam = [0.0, 0.0, 0.0]
            lam[i] = bad
            assert reg(lam=tuple(lam)) == _lib.ERR_INVALID, (bad, i)
    assert reg(d=fake) == _lib.ERR_INVALID  # d is values
    base = 1 << 20
    assert reg(n=2, vals=C.c_void_p(base), d=C.c_void_p(base + 729 * 128)) == _lib.ERR_INVALID  # d inside values
    assert reg(n=2, vals=C.c_void_p(base + 729 * 128), d=C.c_void_p(base)) == _lib.ERR_INVALID  # values inside d
    assert ops.launch_count() == before


def test_python_refusals_precede_any_launch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    before = ops.launch_count()
    bm = torch.zeros(8, dtype=torch.int32)
    cpu = nb.BakedField(((-1.0,) * 3, (1.0,) * 3), (16, 16, 16), bm, torch.zeros(1, dtype=torch.int32),
                        torch.zeros(1, 729, 32), True)
    with pytest.raises(ValueError):
        nb.baked_regularizer(object(), tv_sigma=1.0)
    with pytest.raises(ValueError):  # CPU values
        nb.baked_regularizer(cpu, tv_sigma=1.0)
    if torch.cuda.is_available():  # the remaining refusals need CUDA values; without a device they are the one above
        f16 = nb.BakedField(cpu.bounds, cpu.resolution, bm.cuda(), cpu.bricks.cuda(),
                            torch.zeros(1, 729, 32, dtype=torch.float16, device="cuda"), True)
        with pytest.raises(ValueError):
            nb.baked_regularizer(f16, tv_sigma=1.0)
        ok = nb.BakedField(cpu.bounds, cpu.resolution, bm.cuda(), cpu.bricks.cuda(),
                           torch.zeros(1, 729, 32, device="cuda"), True)
        for kw in ({"tv_sigma": -1.0}, {"tv_sh": float("nan")}, {"sparsity": float("inf")}):
            with pytest.raises(ValueError):
                nb.baked_regularizer(ok, **kw)
        empty = nb.BakedField(cpu.bounds, cpu.resolution, torch.full_like(bm, -1).cuda(), cpu.bricks[:0].cuda(),
                              torch.zeros(0, 729, 32, device="cuda"), True)
        with pytest.raises(ValueError):
            nb.baked_regularizer(empty, sparsity=1.0)
    opts = O.make_options()
    imgs, poses = torch.zeros(2, 8, 8, 3), torch.zeros(2, 4, 4)
    with pytest.raises(ValueError):
        nb.BakedFieldTrainer(cpu, imgs, poses, 10.0, opts, tv_sigma=1.0)
    with pytest.raises(ValueError):  # the weights are checked too (CPU values fail first without a device)
        nb.BakedFieldTrainer(cpu, imgs, poses, 10.0, opts, sparsity=-1.0)
    assert ops.launch_count() == before


def test_trainer_weights_are_checked_before_any_launch():
    from nerf_pytorch_b200.bake import _check_weights

    assert _check_weights("t", 0, 1e-3, 2) == (0.0, 1e-3, 2.0)
    for lam in ((-1.0, 0.0, 0.0), (0.0, float("nan"), 0.0), (0.0, 0.0, float("inf"))):
        with pytest.raises(ValueError):
            _check_weights("t", *lam)


# ------------------------------------------------------------------------------------------------------------------------
# the lattice's points and edges (header, "Lattice points", "Edges"): the restatement against a brute force
# ------------------------------------------------------------------------------------------------------------------------


def _brute_force(res, active):
    """(points, edges) from the cubes of the active bricks: brick b holds the lattice points 8 b_a .. min(8 b_a + 8,
    res_a) on each axis, and (q, q + e_c) is an edge when one brick holds both."""
    shape = (res[2] + 1, res[1] + 1, res[0] + 1)
    points = np.zeros(shape, dtype=bool)
    edges = [np.zeros(shape, dtype=bool) for _ in range(3)]
    for bz, by, bx in zip(*np.nonzero(active)):
        b = (bx, by, bz)
        lo = [8 * b[a] for a in range(3)]
        hi = [min(8 * b[a] + 8, res[a]) for a in range(3)]
        points[lo[2]:hi[2] + 1, lo[1]:hi[1] + 1, lo[0]:hi[0] + 1] = True
        for c in range(3):
            h = list(hi)
            h[c] -= 1  # the edge's lower point q needs q_c + 1 inside the brick
            edges[c][lo[2]:h[2] + 1, lo[1]:h[1] + 1, lo[0]:h[0] + 1] = True
    return points, edges


def _active(res, kind, seed=0):
    nb = [-(-r // 8) for r in res]
    shape = (nb[2], nb[1], nb[0])
    if kind == "random":
        a = np.random.default_rng(seed).random(shape) < 0.5
        a.flat[0] = True
        return a
    a = np.zeros(shape, dtype=bool)
    if kind == "edge":  # two bricks sharing one brick edge (no face)
        a[0, 0, 0] = a[0, 1, 1] = True
    elif kind == "corner":  # two bricks sharing one corner point
        a[0, 0, 0] = a[1, 1, 1] = True
    elif kind == "isolated":  # one brick with no active neighbour, one on the upper corner of the box
        a[0, 0, 0] = a[-1, -1, -1] = True
    elif kind == "full":
        a[:] = True
    return a


CASES = [((16, 16, 16), "full"), ((13, 9, 17), "full"), ((13, 9, 17), "random"), ((24, 20, 28), "random"),
         ((20, 17, 33), "random"), ((16, 16, 16), "edge"), ((13, 21, 11), "edge"), ((16, 16, 16), "corner"),
         ((13, 21, 11), "corner"), ((40, 40, 40), "isolated"), ((29, 18, 35), "isolated"), ((1, 25, 7), "random"),
         ((8, 8, 8), "full")]


@pytest.mark.parametrize("res,kind", CASES)
def test_restated_lattice_matches_brute_force(res, kind):
    active = _active(res, kind, seed=sum(res))
    points, edges = baked_lattice(res, active)
    want_points, want_edges = _brute_force(res, active)
    assert np.array_equal(points, want_points)
    for c in range(3):
        assert np.array_equal(edges[c], want_edges[c]), c
        # an edge's two points are lattice points, and no edge leaves the box (clamped repeats are one point)
        up = np.roll(edges[c], 1, axis=2 - c)
        assert not edges[c].take(-1, axis=2 - c).any()
        assert (points[edges[c]]).all() and (points[up]).all()
    if kind == "edge" and res == (16, 16, 16):  # the shared brick edge's 9 points are held by both bricks
        assert int(points.sum()) == 2 * 729 - 9
    if kind == "corner" and res == (16, 16, 16):  # one shared corner point
        assert int(points.sum()) == 2 * 729 - 1
        assert sum(int(e.sum()) for e in edges) == 2 * 3 * 8 * 81  # each brick's own 3 x 8 x 9 x 9 edges


@pytest.mark.parametrize("res,kind", CASES)
def test_lattice_point_count_is_the_canonical_copies(res, kind):
    """P from the restatement equals the number of stored copies that are their point's first copy in the tie's order
    (the counting kernel's rule), enumerated from the stored copies directly."""
    active = _active(res, kind, seed=sum(res))
    points, _ = baked_lattice(res, active)
    nb = [-(-r // 8) for r in res]
    first = {}
    for bz, by, bx in zip(*np.nonzero(active)):  # bricks in ascending order give the stored copies' points
        for l in itertools.product(range(9), repeat=3):  # (l_2, l_1, l_0)
            q = (min(bz * 8 + l[0], res[2]), min(by * 8 + l[1], res[1]), min(bx * 8 + l[2], res[0]))
            first.setdefault(q, (bz, by, bx, l))
    assert int(points.sum()) == len(first)
    if kind == "full":
        assert int(points.sum()) == (res[0] + 1) * (res[1] + 1) * (res[2] + 1)
    if kind == "isolated":  # a whole brick and the box's last brick, which the box may cut
        last = [res[c] - 8 * (nb[c] - 1) + 1 for c in range(3)]
        assert int(points.sum()) == 729 + last[0] * last[1] * last[2]
