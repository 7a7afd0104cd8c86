"""Host: pruning baked fields (include/nerfb200.h "baked fields: pruning"): the ABI symbol, its signature and the
Python exports, every C-level refusal before any launch, the Python refusals of nb.baked_brick_weights_rays,
nb.baked_brick_weights, nb.prune_baked and BakedFieldTrainer.prune, prune_baked's bookkeeping on a CPU field, and
nb.baked_transparent_bricks on hand-made values.  No GPU."""
import ctypes as C
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "nerfb200_baked_max_weights"
PUBLIC = ("baked_brick_weights", "baked_brick_weights_rays", "baked_transparent_bricks", "prune_baked")


def test_abi_symbol_signature_and_exports():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import _lib

    with open(os.path.join(ROOT, "include", "nerfb200.h")) as f:
        header = f.read()
    assert re.search(r"int32_t\s+" + NAME + r"\(", header)
    lib = _lib.load()
    assert hasattr(lib, NAME)
    P, I32, I64 = C.c_void_p, C.c_int32, C.c_int64
    assert _lib.SIGNATURES[NAME] == (I32, [C.POINTER(_lib.Grid), P, P, I32, P, I32, I64, P, P])
    assert lib.nerfb200_version() == 101
    for name in PUBLIC:
        assert name in nb.__all__ and callable(getattr(nb, name)), name
    assert callable(nb.BakedFieldTrainer.prune)


def test_entry_point_refuses_before_any_launch():
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    before = ops.launch_count()
    box = ops.grid_struct(((-1.0,) * 3, (1.0,) * 3), (16, 16, 16))
    bad_box = ops.grid_struct(((1.0,) * 3, (-1.0,) * 3), (16, 16, 16))
    fake = C.c_void_p(256)
    f = lib.nerfb200_baked_max_weights
    assert f(C.byref(bad_box), fake, fake, 0, fake, 8, 4, fake, None) == _lib.ERR_INVALID
    for i in range(4):
        ptrs = [fake] * 4
        ptrs[i] = None
        bm, vals, rays, mw = ptrs
        assert f(C.byref(box), bm, vals, 0, rays, 8, 4, mw, None) == _lib.ERR_INVALID, i
    assert f(C.byref(box), fake, fake, 0, fake, 8, 0, fake, None) == _lib.ERR_INVALID
    assert f(C.byref(box), fake, fake, 0, fake, 8, -5, fake, None) == _lib.ERR_INVALID
    assert f(C.byref(box), fake, fake, 1, fake, 10, 4, fake, None) == _lib.ERR_INVALID  # view directions need 11
    assert f(C.byref(box), fake, fake, 0, fake, 7, 4, fake, None) == _lib.ERR_INVALID
    assert "baked_max_weights" in lib.nerfb200_last_error().decode()
    assert ops.launch_count() == before


def _cpu_field(res=(20, 17, 12), active=0.6, seed=0, viewdirs=True):
    """A CPU field on a random subset of bricks; every value distinct, so moved rows are recognisable."""
    import nerf_pytorch_b200 as nb

    g = torch.Generator().manual_seed(seed)
    nb_ = [-(-r // 8) for r in res]
    n_bricks = nb_[0] * nb_[1] * nb_[2]
    act = torch.rand(n_bricks, generator=g) < active
    act[0] = True
    brick_map = torch.where(act, torch.cumsum(act.int(), 0) - 1, -1).int()
    bricks = torch.nonzero(act).reshape(-1).int()
    values = torch.randn(bricks.numel(), 729, 32, generator=g)
    return nb.BakedField(((-1.0,) * 3, (1.0,) * 3), res, brick_map, bricks, values, viewdirs)


def test_python_refusals_precede_any_launch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    before = ops.launch_count()
    f = _cpu_field()
    n = f.n_active
    ok = torch.ones(n, dtype=torch.bool)
    # prune_baked: keep of the wrong dtype, length or device; not a field
    for keep in (ok.to(torch.uint8), ok.int(), torch.ones(n + 1, dtype=torch.bool), torch.ones(n - 1, dtype=torch.bool),
                 ok.view(1, n), torch.ones(n, dtype=torch.bool, device="meta"), [True] * n):
        with pytest.raises(ValueError, match="keep"):
            nb.prune_baked(f, keep)
    with pytest.raises(ValueError, match="BakedField"):
        nb.prune_baked(object(), ok)
    # baked_brick_weights_rays: rays of the wrong shape or dtype, out of the wrong shape or dtype, a CPU field
    with pytest.raises(ValueError, match="BakedField"):
        nb.baked_brick_weights_rays(object(), torch.zeros(4, 11))
    for rays in (torch.zeros(4, 8), torch.zeros(4, 12), torch.zeros(44), torch.zeros(4, 11, dtype=torch.float64),
                 torch.zeros(1, 4, 11)):
        with pytest.raises(ValueError, match="rays"):
            nb.baked_brick_weights_rays(f, rays)
    for out in (torch.zeros(n + 1), torch.zeros(n, dtype=torch.float64), torch.zeros(n, 1), torch.zeros(2 * n)[::2]):
        with pytest.raises(ValueError, match="out"):
            nb.baked_brick_weights_rays(f, torch.zeros(4, 11), out=out)
    with pytest.raises(ValueError, match="CUDA"):
        nb.baked_brick_weights_rays(f, torch.zeros(4, 11))
    noview = _cpu_field(viewdirs=False)
    with pytest.raises(ValueError, match="rays"):  # stride 11 for a field without view directions
        nb.baked_brick_weights_rays(noview, torch.zeros(4, 11))
    # baked_brick_weights: malformed poses and sizes, a CPU field
    opts = O.make_options()
    for poses in (torch.zeros(4, 4), torch.zeros(0, 4, 4), torch.zeros(2, 2, 4), torch.zeros(2, 4, 3),
                  torch.zeros(2, 4, 4, dtype=torch.int64), [torch.eye(4)]):
        with pytest.raises(ValueError, match="poses"):
            nb.baked_brick_weights(f, poses, 8, 8, 10.0, opts)
    with pytest.raises(ValueError, match="height"):
        nb.baked_brick_weights(f, torch.zeros(2, 4, 4), 0, 8, 10.0, opts)
    with pytest.raises(ValueError, match="CUDA"):
        nb.baked_brick_weights(f, torch.zeros(2, 4, 4), 8, 8, 10.0, opts)
    # BakedFieldTrainer.prune keeping nothing: refused before the field or the buffers change
    t = nb.BakedFieldTrainer.__new__(nb.BakedFieldTrainer)
    t.field = f
    values, bm = f.values, f.brick_map
    with pytest.raises(ValueError, match="no brick"):
        t.prune(torch.zeros(n, dtype=torch.bool))
    with pytest.raises(ValueError, match="keep"):
        t.prune(ok[:-1])
    assert f.values is values and f.brick_map is bm and f.n_active == n
    assert ops.launch_count() == before


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_prune_baked_bookkeeping_on_a_cpu_field(seed):
    import nerf_pytorch_b200 as nb

    f = _cpu_field((20, 17, 33), active=0.7, seed=seed)
    snap = [x.clone() for x in (f.brick_map, f.bricks, f.values)]
    keep = torch.rand(f.n_active, generator=torch.Generator().manual_seed(seed + 10)) < 0.5
    keep[-1] = True
    p = nb.prune_baked(f, keep)
    # the argument is untouched
    for a, b in zip(snap, (f.brick_map, f.bricks, f.values)):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    kept = torch.nonzero(keep).reshape(-1)
    assert p.n_active == int(keep.sum()) and p.bounds == f.bounds and p.resolution == f.resolution
    assert p.use_viewdirs == f.use_viewdirs
    assert p.brick_map.dtype == torch.int32 and p.bricks.dtype == torch.int32 and p.values.dtype == torch.float32
    assert p.brick_map.shape == f.brick_map.shape
    # brick_map[bricks[s]] == s for every new slot, slots in ascending order (bricks sorted), dropped bricks -> -1
    s = torch.arange(p.n_active, dtype=torch.int32)
    assert torch.equal(p.brick_map[p.bricks.long()], s)
    assert bool((p.bricks[1:] > p.bricks[:-1]).all())
    assert torch.equal(p.bricks, f.bricks[kept])
    dropped = f.bricks[~keep].long()
    assert bool((p.brick_map[dropped] == -1).all())
    never = f.brick_map < 0
    assert bool((p.brick_map[never] == -1).all())
    assert int((p.brick_map >= 0).sum()) == p.n_active
    # rows moved bit for bit
    assert torch.equal(p.values.view(torch.int32), f.values[kept].view(torch.int32))
    assert p.values.data_ptr() != f.values.data_ptr()
    # keep-all gives equal tensors; keep-none gives an empty field
    a = nb.prune_baked(f, torch.ones(f.n_active, dtype=torch.bool))
    for x, y in ((a.brick_map, f.brick_map), (a.bricks, f.bricks), (a.values, f.values)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    e = nb.prune_baked(f, torch.zeros(f.n_active, dtype=torch.bool))
    assert e.n_active == 0 and e.values.shape == (0, 729, 32) and e.bricks.numel() == 0
    assert bool((e.brick_map == -1).all())
    # pruning a pruned field composes
    keep2 = torch.arange(p.n_active) % 2 == 0
    q = nb.prune_baked(p, keep2)
    assert torch.equal(q.bricks, f.bricks[kept[keep2]])
    assert torch.equal(q.values.view(torch.int32), f.values[kept[keep2]].view(torch.int32))


def test_transparent_bricks_on_hand_made_values():
    import nerf_pytorch_b200 as nb

    nan, inf = float("nan"), float("inf")
    f = _cpu_field((24, 16, 8), active=1.0)  # 6 bricks
    assert f.n_active == 6
    v = torch.randn(6, 729, 32, generator=torch.Generator().manual_seed(5))
    v[..., 0] = -v[..., 0].abs()  # every brick transparent to start with
    v[0, :, 0] = -0.0  # sigma_raw -0 everywhere: transparent
    v[0, :, 28:] = nan  # channels 28 .. 31 are not read by the renderer
    v[1, :, 0] = 0.0  # +0 everywhere: transparent
    v[1, 100, 0] = -0.0
    v[2, 400, 0] = 1e-30  # one positive sigma_raw: not transparent
    v[3, 7, 0] = nan  # a NaN sigma_raw: not transparent
    v[4, 3, 17] = nan  # a NaN coefficient in an otherwise transparent brick: kept
    v[5, 728, 27] = -inf  # an infinite coefficient: kept
    f.values = v
    got = nb.baked_transparent_bricks(f)
    assert got.dtype == torch.bool and got.shape == (6,)
    assert got.tolist() == [True, True, False, False, False, False]
    for chunk in (1, 4, 6, 100):  # chunking does not change the answer
        assert nb.baked_transparent_bricks(f, chunk=chunk).tolist() == got.tolist()
    v[5, 728, 27] = 0.0
    v[4, 3, 17] = inf
    assert nb.baked_transparent_bricks(f).tolist() == [True, True, False, False, False, True]
    v[0, 0, 0] = -inf  # a non-finite sigma_raw: kept
    assert nb.baked_transparent_bricks(f).tolist() == [False, True, False, False, False, True]
    empty = nb.prune_baked(f, torch.zeros(6, dtype=torch.bool))
    assert nb.baked_transparent_bricks(empty).shape == (0,)
