"""Host: the bake's directions, SH basis and projection (nerfb200_bake_basis, include/nerfb200.h "baked fields"), the
argument refusals of nb.bake / nb.render_baked and the bake entry points, and the new ABI symbols.  No GPU."""
import ctypes as C
import math

import numpy as np
import pytest
import scipy.special
import torch

# the real SH of the header, in basis order j = 0 .. 8: (l, m)
LM = [(0, 0), (1, -1), (1, 0), (1, 1), (2, -2), (2, -1), (2, 0), (2, 1), (2, 2)]


def _basis():
    from nerf_pytorch_b200 import ops

    d, m = ops.bake_basis()
    return d.numpy(), m.numpy()


def _sh64(d):
    """Y[i][j] in fp64 from the header's constants."""
    x, y, z = (d[:, c].astype(np.float64) for c in range(3))
    return np.stack([np.full_like(x, 0.28209479177387814), -0.4886025119029199 * y, 0.4886025119029199 * z,
                     -0.4886025119029199 * x, 1.0925484305920792 * x * y, -1.0925484305920792 * y * z,
                     0.31539156525252005 * (2 * z * z - x * x - y * y), -1.0925484305920792 * x * z,
                     0.5462742152960396 * (x * x - y * y)], -1)


def test_directions_are_the_spherical_fibonacci_lattice():
    d, _ = _basis()
    i = np.arange(64, dtype=np.float64)
    z = 1 - (2 * i + 1) / 64
    r = np.sqrt(1 - z * z)
    phi = i * math.pi * (3 - math.sqrt(5))
    want = np.stack([r * np.cos(phi), r * np.sin(phi), z], -1).astype(np.float32)
    assert np.array_equal(d, want)


def test_sh_constants_are_scipys_real_harmonics():
    """Real Y_lm = sqrt 2 Re Y_l^m (m > 0), sqrt 2 Im Y_l^|m| (m < 0), Y_l^0, from scipy's complex harmonics with the
    Condon-Shortley phase: the header's signs.  scipy sees the angles of the fp32 directions, which are unit length only
    to fp32 rounding, so the two agree to ~1e-7."""
    d, _ = _basis()
    x, y, z = (d[:, c].astype(np.float64) for c in range(3))
    polar, azim = np.arccos(np.clip(z, -1, 1)), np.arctan2(y, x)
    got = _sh64(d)
    for j, (l, m) in enumerate(LM):
        c = scipy.special.sph_harm_y(l, abs(m), polar, azim)
        want = c.real if m == 0 else math.sqrt(2) * (c.real if m > 0 else c.imag)
        assert np.allclose(got[:, j], want, rtol=0, atol=1e-6), (l, m)


def test_projection_is_the_pseudo_inverse_within_fp32_rounding():
    d, M = _basis()
    pinv = np.linalg.pinv(_sh64(d))
    assert M.shape == (9, 64)
    err = np.abs(M.astype(np.float64) - pinv)
    assert (err <= 2.0 ** -24 * np.abs(pinv) + 1e-12).all(), err.max()


def test_projection_reproduces_a_degree_2_field():
    d, M = _basis()
    Y = _sh64(d)
    rng = np.random.default_rng(3)
    for _ in range(8):
        c = rng.standard_normal(9)
        f = Y @ c
        got = M.astype(np.float64) @ f
        assert np.allclose(got, c, rtol=0, atol=1e-6 * np.abs(c).max()), (got, c)


def test_abi_symbols_are_present():
    from nerf_pytorch_b200 import _lib

    lib = _lib.load()
    for name in ("nerfb200_bake_basis", "nerfb200_bake_supported", "nerfb200_bake", "nerfb200_baked_render"):
        assert hasattr(lib, name) and name in _lib.SIGNATURES


def test_entry_points_refuse_before_any_launch():
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    before = ops.launch_count()
    box = ops.grid_struct(((-1.0,) * 3, (1.0,) * 3), (16, 16, 16))
    bad_box = ops.grid_struct(((1.0,) * 3, (-1.0,) * 3), (16, 16, 16))
    arch = ops.ArchSpec().c_struct()
    fake = C.c_void_p(256)
    # bake: null pointers, slot ranges, box, architecture
    assert lib.nerfb200_bake(C.byref(arch), None, C.byref(box), fake, 0, 1, fake, None, None) == _lib.ERR_INVALID
    assert lib.nerfb200_bake(C.byref(arch), fake, C.byref(box), fake, 0, 9, fake, None, None) == _lib.ERR_INVALID
    assert lib.nerfb200_bake(C.byref(arch), fake, C.byref(box), fake, -1, 1, fake, None, None) == _lib.ERR_INVALID
    assert lib.nerfb200_bake(C.byref(arch), fake, C.byref(box), fake, 0, 0, fake, None, None) == _lib.ERR_INVALID
    assert lib.nerfb200_bake(C.byref(arch), fake, C.byref(bad_box), fake, 0, 1, fake, None, None) == _lib.ERR_INVALID
    a64 = ops.ArchSpec(hidden=64).c_struct()
    assert lib.nerfb200_bake(C.byref(a64), fake, C.byref(box), fake, 0, 1, fake, None, None) != _lib.OK
    wide = ops.ArchSpec(n_freq_xyz=16).c_struct()  # a 99-wide encoding: the wgmma forward refuses it
    assert lib.nerfb200_bake_supported(C.byref(wide)) == _lib.ERR_UNSUPPORTED
    assert lib.nerfb200_bake(C.byref(wide), fake, C.byref(box), fake, 0, 1, fake, None, None) == _lib.ERR_UNSUPPORTED
    assert lib.nerfb200_bake_supported(C.byref(arch)) == _lib.OK
    assert lib.nerfb200_bake_supported(C.byref(ops.ArchSpec(hidden=256, skip_every=4).c_struct())) == _lib.OK
    assert lib.nerfb200_bake_supported(C.byref(ops.ArchSpec(use_viewdirs=False).c_struct())) == _lib.OK
    # baked_render: stride, threshold, pointers, box
    r = lib.nerfb200_baked_render
    assert r(C.byref(box), fake, fake, 1, fake, 8, 4, 0, 0.0, fake, None) == _lib.ERR_INVALID
    assert r(C.byref(box), fake, fake, 0, fake, 8, 4, 0, 1.0, fake, None) == _lib.ERR_INVALID
    assert r(C.byref(box), fake, fake, 0, fake, 8, 4, 0, float("nan"), fake, None) == _lib.ERR_INVALID
    assert r(C.byref(box), fake, fake, 0, fake, 8, 4, 0, -0.1, fake, None) == _lib.ERR_INVALID
    assert r(C.byref(box), None, fake, 0, fake, 8, 4, 0, 0.0, fake, None) == _lib.ERR_INVALID
    assert r(C.byref(box), fake, fake, 0, fake, 8, 0, 0, 0.0, fake, None) == _lib.ERR_INVALID
    assert r(C.byref(bad_box), fake, fake, 0, fake, 8, 4, 0, 0.0, fake, None) == _lib.ERR_INVALID
    assert ops.launch_count() == before


def test_python_refusals_precede_any_launch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    before = ops.launch_count()
    m = nb.FlexibleNeRFModel()
    epf = nb.get_embedding_function(6)
    for bounds, res in ((((-1.0,) * 3, (1.0,) * 3), 1), ((((1.0,) * 3), (-1.0,) * 3), 16), (((-1.0,) * 2, (1.0,) * 2), 16),
                        (((-1.0,) * 3, (1.0,) * 3), 5000), (((-1.0,) * 3, (1.0,) * 3), (16, 16))):
        with pytest.raises(ValueError):
            nb.bake(m, epf, bounds=bounds, resolution=res, grid=None)
    with pytest.raises(NotImplementedError):  # CPU parameters: there is no CPU path
        nb.bake(m, epf, bounds=((-1.0,) * 3, (1.0,) * 3), resolution=16, grid=None)
    opts = O.make_options()
    with pytest.raises(ValueError):
        nb.render_baked(object(), 8, 8, 10.0, torch.eye(4), opts)
    f = nb.BakedField(((-1.0,) * 3, (1.0,) * 3), (16, 16, 16), torch.zeros(8, dtype=torch.int32),
                      torch.zeros(0, dtype=torch.int32), torch.zeros(0, 729, 32), True)
    with pytest.raises(NotImplementedError):
        nb.render_baked(f, 8, 8, 10.0, torch.eye(4), opts)
    assert ops.launch_count() == before


# encodings of the support sweep: (n_freq_xyz, n_freq_dir) 10/4 as shipped, 10/5 without the raw direction input (30
# channels), none, and no view directions
SUPPORT_ENCODINGS = {
    "10/4": dict(n_freq_xyz=10, n_freq_dir=4),
    "10/5_noinput_dir": dict(n_freq_xyz=10, n_freq_dir=5, include_input_dir=False),
    "0/0": dict(n_freq_xyz=0, n_freq_dir=0),
    "noview": dict(n_freq_xyz=10, use_viewdirs=False),
}


@pytest.mark.parametrize("hidden", [128, 256])
def test_bake_takes_exactly_what_the_wgmma_forward_takes(hidden):
    """Over 1 .. 16 layers, skip 1 .. 5 and SUPPORT_ENCODINGS, bake_refusal is None exactly when the wgmma inference
    forward takes the architecture.  The bake's own "too deep for its shared-memory budget" refusal is unreachable
    there: a layout change that makes it reachable shows up here first."""
    from nerf_pytorch_b200 import ops

    taken = 0
    for layers in range(1, 17):
        for skip in range(1, 6):
            for enc, kw in SUPPORT_ENCODINGS.items():
                arch = ops.ArchSpec(num_layers=layers, hidden=hidden, skip_every=skip, **kw)
                why = ops.bake_refusal(arch)
                fwd = ops.impl_supported(arch, 64, ops.IMPL_TC_FWD)
                assert (why is None) == fwd, (layers, skip, enc, why)
                assert why is None or "too deep" not in why, (layers, skip, enc, why)
                taken += why is None
    assert taken > 0
