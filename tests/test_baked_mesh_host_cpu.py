"""Host: meshes of baked fields (include/nerfb200.h "baked fields: meshes"): the four ABI symbols, their signatures and
the Python exports, every C-level refusal before any launch, and every refusal of nb.extract_baked_mesh before any
launch.  No GPU."""
import ctypes as C
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("nerfb200_baked_mesh_dirs", "nerfb200_baked_mesh_dirs_f16", "nerfb200_baked_mesh_colors",
         "nerfb200_baked_mesh_colors_f16")


def test_abi_symbols_signatures_and_exports():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import _lib, ops

    with open(os.path.join(ROOT, "include", "nerfb200.h")) as f:
        header = f.read()
    assert "baked fields: meshes" in header
    lib = _lib.load()
    P, I32, I64, F32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
    GP = C.POINTER(_lib.Grid)
    want = {"dirs": (I32, [GP, P, P, F32, P, I64, P, P, P]), "colors": (I32, [GP, P, P, I32, F32, P, P, I64, P, P])}
    for name in NAMES:
        assert re.search(r"int32_t\s+" + name + r"\(", header), name
        assert hasattr(lib, name)
        assert _lib.SIGNATURES[name] == want["dirs" if "dirs" in name else "colors"], name
    assert "extract_baked_mesh" in nb.__all__ and callable(nb.extract_baked_mesh)
    assert callable(ops.baked_mesh_dirs) and callable(ops.baked_mesh_colors)


def _box():
    from nerf_pytorch_b200 import ops

    return ops.grid_struct(((-1.0,) * 3, (1.0,) * 3), (16, 16, 16))


def test_entry_points_refuse_before_any_launch():
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    before = ops.launch_count()
    box = _box()
    a = C.c_void_p(1 << 20)  # 16-B aligned stand-ins: never dereferenced by a refused call
    bad_boxes = [ops.grid_struct(((1.0,) * 3, (-1.0,) * 3), (16,) * 3),
                 ops.grid_struct(((-1.0,) * 3, (1.0,) * 3), (0, 16, 16))]
    for name in NAMES:
        f = getattr(lib, name)
        colors = "colors" in name

        def call(bx=C.byref(box), bm=a, vals=a, level=50.0, keys=a, n=4, dirs=a, out=a, viewdirs=1):
            if colors:
                return f(bx, bm, vals, viewdirs, level, keys, dirs, n, out, None)
            return f(bx, bm, vals, level, keys, n, out, None, None)

        for bx in bad_boxes:
            assert call(bx=C.byref(bx)) == _lib.ERR_INVALID, name
        assert call(bx=None) == _lib.ERR_INVALID, name
        for k in ("bm", "vals", "keys", "out"):
            assert call(**{k: None}) == _lib.ERR_INVALID, (name, k)
            assert name.split("nerfb200_")[1] in lib.nerfb200_last_error().decode()
        if colors:  # dirs are needed with view directions alone
            assert call(dirs=None) == _lib.ERR_INVALID, name
            assert "dirs" in lib.nerfb200_last_error().decode()
        assert call(n=-1) == _lib.ERR_INVALID, name
        for level in (float("nan"), float("inf"), -float("inf")):
            assert call(level=level) == _lib.ERR_INVALID, (name, level)
            assert "level" in lib.nerfb200_last_error().decode()
        if name.endswith("_f16"):
            for off in (2, 8):
                assert call(vals=C.c_void_p((1 << 20) + off)) == _lib.ERR_INVALID, (name, off)
                assert "16-B aligned" in lib.nerfb200_last_error().decode()
        # n_vertices 0 is accepted and launches nothing (a negative level is the Python interface's refusal)
        assert call(n=0) == _lib.OK, name
        assert call(n=0, level=-1.0) == _lib.OK, name
        if colors:
            assert call(n=0, dirs=None, viewdirs=0) == _lib.OK, name
    assert ops.launch_count() == before


def _cpu_field(dtype=torch.float32, bounds=((-1.0,) * 3, (1.0,) * 3)):
    import nerf_pytorch_b200 as nb

    n = 8
    ids = torch.arange(n, dtype=torch.int32)
    return nb.BakedField(bounds, (16, 16, 16), ids, ids.clone(), torch.zeros(n, 729, 32, dtype=dtype), True)


def test_python_refusals_precede_any_launch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    before = ops.launch_count()
    f = _cpu_field()
    for bad in (object(), None, f.values):
        with pytest.raises(ValueError, match="BakedField"):
            nb.extract_baked_mesh(bad)
    for level in (float("nan"), float("inf"), -float("inf")):
        with pytest.raises(ValueError, match="level"):
            nb.extract_baked_mesh(f, level)
    for level in (-1.0, -1e-30):
        with pytest.raises(ValueError, match=">= 0"):
            nb.extract_baked_mesh(f, level, colors=True, normals=True)
    for ndc in ((42, 56), (42, 56, -1.0), (0, 56, 45.3), (42.5, 56, 45.3), (42, 56, float("nan")), "fern", (True, 5, 1.0)):
        with pytest.raises(ValueError, match="ndc"):
            nb.extract_baked_mesh(f, ndc=ndc)
    for hi_z in (1.0, 1.5):  # the NDC box reaching z = 1
        g = _cpu_field(bounds=((-1.0,) * 3, (1.0, 1.0, hi_z)))
        with pytest.raises(ValueError, match="hi_z < 1"):
            nb.extract_baked_mesh(g, ndc=(42, 56, 45.3))
    # a CPU field, fp32 or fp16, with or without attributes
    for dtype in (torch.float32, torch.float16):
        with pytest.raises(NotImplementedError, match="CUDA"):
            nb.extract_baked_mesh(_cpu_field(dtype), 0.0, colors=True, normals=True)
    with pytest.raises(NotImplementedError, match="CUDA"):
        nb.extract_baked_mesh(_cpu_field(bounds=((-1.0,) * 3, (1.0, 1.0, 0.98))), ndc=(42, 56, 45.3))
    assert ops.launch_count() == before
