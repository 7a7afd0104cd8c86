"""The density gradient's host side, without a GPU: the new C ABI symbols are declared, bound and exported; every
refusal fires before a device is touched; Mesh.save_ply adds the normal properties only when the mesh has normals."""
import ctypes as C
import os
import re
import struct

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("nerfb200_density_grad", "nerfb200_density_grad_supported")


def test_symbols_declared_bound_exported():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import _lib

    header = open(os.path.join(ROOT, "include", "nerfb200.h")).read()
    lib = _lib.load()
    for name in NEW:
        assert re.search(r"\b" + name + r"\(", header), name
        assert name in _lib.SIGNATURES
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1]
    assert "density_gradient" in nb.__all__ and callable(nb.density_gradient)
    assert "normals" in nb.extract_mesh.__code__.co_varnames


def _arch(**kw):
    from nerf_pytorch_b200 import ops

    base = dict(num_layers=8, hidden=128, skip_every=3, n_freq_xyz=10, n_freq_dir=4)
    base.update(kw)
    return ops.ArchSpec(**base)


def test_library_accepts_impl1_at_128_and_256_and_refuses_the_rest():
    from nerf_pytorch_b200 import ops

    assert ops.density_grad_refusal(_arch(), ops.IMPL_TC) is None
    assert ops.density_grad_refusal(_arch(hidden=256, skip_every=4), ops.IMPL_TC) is None
    assert ops.density_grad_refusal(_arch(use_viewdirs=False), ops.IMPL_TC) is None
    for impl in (ops.IMPL_SIMT, ops.IMPL_TC_FAST):
        assert "impl=1" in ops.density_grad_refusal(_arch(), impl)
    assert "unknown impl" in ops.density_grad_refusal(_arch(), 7)
    assert "hidden_size" in ops.density_grad_refusal(_arch(hidden=64), ops.IMPL_TC)
    assert "encodings wider" in ops.density_grad_refusal(_arch(n_freq_xyz=12), ops.IMPL_TC)


def test_c_abi_refuses_before_any_launch():
    """Fake device pointers: every refusal returns before the pointers are read or a kernel is launched."""
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    fake = C.c_void_p(0x1000)
    a = C.byref(_arch().c_struct())
    n0 = ops.launch_count()
    assert lib.nerfb200_density_grad(a, fake, fake, 10, fake, ops.IMPL_SIMT, None) == _lib.ERR_UNSUPPORTED
    assert lib.nerfb200_density_grad(a, fake, fake, 10, fake, ops.IMPL_TC_FAST, None) == _lib.ERR_UNSUPPORTED
    assert lib.nerfb200_density_grad(a, fake, fake, 0, fake, ops.IMPL_TC, None) == _lib.ERR_INVALID
    assert lib.nerfb200_density_grad(a, None, fake, 10, fake, ops.IMPL_TC, None) == _lib.ERR_INVALID
    assert lib.nerfb200_density_grad(a, fake, fake, 1 << 31, fake, ops.IMPL_TC, None) == _lib.ERR_UNSUPPORTED
    a64 = C.byref(_arch(hidden=64).c_struct())
    assert lib.nerfb200_density_grad(a64, fake, fake, 10, fake, ops.IMPL_TC, None) == _lib.ERR_UNSUPPORTED
    assert ops.launch_count() == n0


def _model(hidden=128, requires_grad=True):
    import nerf_pytorch_b200 as nb

    m = nb.FlexibleNeRFModel(num_layers=4, hidden_size=hidden, skip_connect_every=4, num_encoding_fn_xyz=10,
                             num_encoding_fn_dir=4)
    for p in m.parameters():
        p.requires_grad_(requires_grad)
    return m, nb.get_embedding_function(10)


def test_python_refusals_need_no_device():
    import nerf_pytorch_b200 as nb

    m, epf = _model()
    pts = torch.zeros(5, 3)
    with pytest.raises(NotImplementedError, match="inference only"):
        nb.density_gradient(m, epf, pts)  # would train: autograd on and parameters that require grad
    with torch.no_grad():
        with pytest.raises(ValueError, match=r"\(\.\.\., 3\)"):
            nb.density_gradient(m, epf, torch.zeros(5, 2))
        with pytest.raises(ValueError, match="fp32"):
            nb.density_gradient(m, epf, torch.zeros(5, 3, dtype=torch.float64))
        with pytest.raises(NotImplementedError, match="CUDA"):
            nb.density_gradient(m, epf, pts)
        with pytest.raises(TypeError):
            nb.density_gradient(m, epf, np.zeros((5, 3), np.float32))


def _cpu_mesh():
    from nerf_pytorch_b200 import Mesh

    v = torch.tensor([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.5]], dtype=torch.float32)
    f = torch.tensor([[0, 1, 2]], dtype=torch.int32)
    return v, f, Mesh


def test_ply_without_normals_is_unchanged(tmp_path):
    v, f, Mesh = _cpu_mesh()
    path = tmp_path / "m.ply"
    Mesh(v, f).save_ply(path)
    # the fixture: the format as written before vertex normals existed
    want = (b"ply\nformat binary_little_endian 1.0\nelement vertex 3\nproperty float x\nproperty float y\n"
            b"property float z\nelement face 1\nproperty list uchar int vertex_indices\nend_header\n")
    want += b"".join(struct.pack("<3f", *row) for row in v.tolist())
    want += struct.pack("<B3i", 3, 0, 1, 2)
    assert path.read_bytes() == want
    colored = tmp_path / "c.ply"
    Mesh(v, f, torch.tensor([[1.0, 0.0, 0.5]] * 3)).save_ply(colored)
    head = colored.read_bytes().split(b"end_header\n")[0]
    assert b"nx" not in head and b"property uchar red" in head


def test_ply_with_normals_adds_three_float_properties(tmp_path):
    v, f, Mesh = _cpu_mesh()
    n = torch.tensor([[0.0, 0.0, 1.0], [0.0, 1.0, 0.0], [1.0, 0.0, 0.0]])
    col = torch.tensor([[1.0, 0.0, 0.5]] * 3)
    path = tmp_path / "n.ply"
    Mesh(v, f, col, n).save_ply(path)
    head, body = path.read_bytes().split(b"end_header\n")
    assert (b"property float x\nproperty float y\nproperty float z\nproperty float nx\nproperty float ny\n"
            b"property float nz\nproperty uchar red\nproperty uchar green\nproperty uchar blue\n") in head + b"\n"
    rec = np.frombuffer(body[:3 * 27], dtype=[("p", "<f4", 6), ("c", "u1", 3)])
    assert np.array_equal(rec["p"][:, :3], v.numpy()) and np.array_equal(rec["p"][:, 3:], n.numpy())
    assert rec["c"].tolist() == [[255, 0, 128]] * 3
