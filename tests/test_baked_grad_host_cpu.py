"""Host: the baked-field gradient entry points (include/nerfb200.h "baked fields: gradients and fine-tuning"): ABI
symbols and signatures, every C-level refusal before any launch, the Python refusals of nb.render_baked_rays and
nb.BakedFieldTrainer, and the tie's copy enumeration restated in numpy against a brute force over the stored copies.
No GPU."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

NAMES = ("nerfb200_baked_render_bwd", "nerfb200_baked_tie", "nerfb200_baked_adam_step_dev")


def test_abi_symbols_and_signatures():
    from nerf_pytorch_b200 import _lib

    lib = _lib.load()
    P, I32, I64, F32, F64 = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_double
    GP = C.POINTER(_lib.Grid)
    want = {
        "nerfb200_baked_render_bwd": (I32, [GP, P, P, I32, P, I32, I64, I32, P, P, P, P]),
        "nerfb200_baked_tie": (I32, [GP, P, P, I64, P, P, P]),
        "nerfb200_baked_adam_step_dev": (I32, [P, P, P, P, I64, P, F64, F64, F64, F64, F32, F32, F32, P]),
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
    # baked_render_bwd: box, pointers, n_rays, stride
    b = lib.nerfb200_baked_render_bwd
    assert b(C.byref(bad_box), fake, fake, 0, fake, 8, 4, 0, fake, fake, fake, None) == _lib.ERR_INVALID
    for i in range(6):
        ptrs = [fake] * 6
        ptrs[i] = None
        bm, vals, rays, out, g, d = ptrs
        assert b(C.byref(box), bm, vals, 0, rays, 8, 4, 0, out, g, d, None) == _lib.ERR_INVALID, i
    assert b(C.byref(box), fake, fake, 0, fake, 8, 0, 0, fake, fake, fake, None) == _lib.ERR_INVALID
    assert b(C.byref(box), fake, fake, 0, fake, 8, -3, 0, fake, fake, fake, None) == _lib.ERR_INVALID
    assert b(C.byref(box), fake, fake, 1, fake, 10, 4, 0, fake, fake, fake, None) == _lib.ERR_INVALID
    assert b(C.byref(box), fake, fake, 0, fake, 7, 4, 0, fake, fake, fake, None) == _lib.ERR_INVALID
    # baked_tie: box, pointers, n_active, aliasing
    t = lib.nerfb200_baked_tie
    assert t(C.byref(bad_box), fake, fake, 1, fake, other, None) == _lib.ERR_INVALID
    for i in range(4):
        ptrs = [fake, fake, fake, other]
        ptrs[i] = None
        assert t(C.byref(box), ptrs[0], ptrs[1], 1, ptrs[2], ptrs[3], None) == _lib.ERR_INVALID, i
    assert t(C.byref(box), fake, fake, 0, fake, other, None) == _lib.ERR_INVALID
    assert t(C.byref(box), fake, fake, 9, fake, other, None) == _lib.ERR_INVALID
    assert t(C.byref(box), fake, fake, 1, fake, fake, None) == _lib.ERR_INVALID
    assert t(C.byref(box), fake, fake, 2, C.c_void_p(1 << 20), C.c_void_p((1 << 20) + 729 * 128), None) \
        == _lib.ERR_INVALID  # d_tied starts inside d_values
    assert t(C.byref(box), fake, fake, 2, C.c_void_p((1 << 20) + 729 * 128), C.c_void_p(1 << 20), None) \
        == _lib.ERR_INVALID  # d_values starts inside d_tied
    # baked_adam_step_dev: pointers, n_active, rates and schedule
    a = lib.nerfb200_baked_adam_step_dev
    for i in range(5):
        ptrs = [fake] * 5
        ptrs[i] = None
        p, g, m, v, s = ptrs
        assert a(p, g, m, v, 1, s, 1.0, 1e-2, 0.0, 0.1, 0.9, 0.999, 1e-8, None) == _lib.ERR_INVALID, i
    assert a(fake, fake, fake, fake, 0, fake, 1.0, 1e-2, 0.0, 0.1, 0.9, 0.999, 1e-8, None) == _lib.ERR_INVALID
    assert a(fake, fake, fake, fake, 1, fake, -1.0, 1e-2, 0.0, 0.1, 0.9, 0.999, 1e-8, None) == _lib.ERR_INVALID
    assert a(fake, fake, fake, fake, 1, fake, 1.0, float("nan"), 0.0, 0.1, 0.9, 0.999, 1e-8, None) == _lib.ERR_INVALID
    assert a(fake, fake, fake, fake, 1, fake, 1.0, 1e-2, -1.0, 0.1, 0.9, 0.999, 1e-8, None) == _lib.ERR_INVALID
    assert a(fake, fake, fake, fake, 1, fake, 1.0, 1e-2, 0.0, 0.0, 0.9, 0.999, 1e-8, None) == _lib.ERR_INVALID
    assert ops.launch_count() == before


def test_python_refusals_precede_any_launch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    before = ops.launch_count()
    bm = torch.zeros(8, dtype=torch.int32)
    cpu = nb.BakedField(((-1.0,) * 3, (1.0,) * 3), (16, 16, 16), bm, torch.zeros(0, dtype=torch.int32),
                        torch.zeros(0, 729, 32), True)
    rays = torch.zeros(4, 11)
    with pytest.raises(ValueError):
        nb.render_baked_rays(object(), rays)
    with pytest.raises(ValueError):  # CPU values
        nb.render_baked_rays(cpu, rays)
    if torch.cuda.is_available():  # the remaining refusals need CUDA values; without a device they are the one above
        f16 = nb.BakedField(cpu.bounds, cpu.resolution, bm.cuda(), cpu.bricks.cuda(),
                            torch.zeros(0, 729, 32, dtype=torch.float16, device="cuda"), True)
        with pytest.raises(ValueError):
            nb.render_baked_rays(f16, rays.cuda())
        ok = nb.BakedField(cpu.bounds, cpu.resolution, bm.cuda(), cpu.bricks.cuda(),
                           torch.zeros(1, 729, 32, device="cuda", requires_grad=True), True)
        with pytest.raises(ValueError):  # stride 8 for a field with view directions
            nb.render_baked_rays(ok, torch.zeros(4, 8, device="cuda"))
        with pytest.raises(ValueError):  # early stopping has no gradient
            nb.render_baked_rays(ok, torch.zeros(4, 11, device="cuda"), early_stop=0.1)
    opts = O.make_options()
    imgs, poses = torch.zeros(2, 8, 8, 3), torch.zeros(2, 4, 4)
    with pytest.raises(ValueError):
        nb.BakedFieldTrainer(object(), imgs, poses, 10.0, opts, lr_sigma=1.0, lr_sh=1e-2)
    with pytest.raises(ValueError):
        nb.BakedFieldTrainer(cpu, imgs, poses, 10.0, opts, lr_sigma=1.0, lr_sh=1e-2)
    assert ops.launch_count() == before


# ------------------------------------------------------------------------------------------------------------------------
# the tie's copy enumeration (header, "Tie"): a numpy restatement against a brute force
# ------------------------------------------------------------------------------------------------------------------------
def _axis_copies(q, res):
    """The header's copies of lattice index q along one axis: (brick, point) pairs in ascending brick order."""
    nb = -(-res // 8)
    if q == res:
        return [(nb - 1, l) for l in range(res - 8 * (nb - 1), 9)]
    if q > 0 and q % 8 == 0:
        return [(q // 8 - 1, 8), (q // 8, 0)]
    return [(q // 8, q % 8)]


@pytest.mark.parametrize("res", [(16, 16, 16), (9, 9, 9), (13, 8, 17), (1, 25, 7), (24, 3, 10)])
def test_copy_enumeration_lists_exactly_the_stored_copies(res):
    rng = np.random.default_rng(sum(res))
    nb = [-(-r // 8) for r in res]
    n_bricks = nb[0] * nb[1] * nb[2]
    active = rng.random(n_bricks) < 0.7
    active[0] = True
    slot_of = np.where(active, np.cumsum(active) - 1, -1)
    # brute force: every stored (slot, l) and the lattice point it holds (b B + l clamped onto 0 .. res)
    stored = {}
    for brick in np.nonzero(active)[0]:
        b = (brick % nb[0], brick // nb[0] % nb[1], brick // (nb[0] * nb[1]))
        for l in itertools.product(range(9), repeat=3):  # (l_0, l_1, l_2)
            q = tuple(min(b[c] * 8 + l[c], res[c]) for c in range(3))
            stored.setdefault(q, set()).add((int(slot_of[brick]), l[2] * 81 + l[1] * 9 + l[0]))
    listed_total = 0
    for q, copies in stored.items():
        lists = [_axis_copies(q[c], res[c]) for c in range(3)]
        listed = []
        for (bz, lz), (by, ly), (bx, lx) in itertools.product(lists[2], lists[1], lists[0]):
            s = slot_of[(bz * nb[1] + by) * nb[0] + bx]
            if s >= 0:
                listed.append((int(s), lz * 81 + ly * 9 + lx))
        assert len(listed) == len(set(listed)), q  # no copy listed twice
        assert set(listed) == copies, q  # every listed copy holds q, and every copy of q is listed
        listed_total += len(listed)
    assert listed_total == int(active.sum()) * 729  # each stored value belongs to exactly one lattice point
