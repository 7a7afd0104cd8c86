"""Host: normal maps and point queries of baked fields (include/nerfb200.h "baked fields: normal maps and point
queries").  The six entry points' ABI and the library's refusals, checked before any launch, and the Python refusals of
render_baked(normals=), render_baked_rays(normals=, ndc=), nb.baked_raw and nb.baked_density_gradient.  No GPU."""
import ctypes as C

import pytest
import torch

BOX = ((-1.0,) * 3, (1.0,) * 3)
FAKE, ODD = C.c_void_p(256), C.c_void_p(256 + 8)  # device-looking pointers, 16-B aligned and not


def _field(viewdirs=True, requires_grad=False, dtype=torch.float32):
    import nerf_pytorch_b200 as nb

    ids = torch.arange(8, dtype=torch.int32)
    values = torch.zeros(8, 729, 32, dtype=dtype, requires_grad=requires_grad and dtype == torch.float32)
    return nb.BakedField(BOX, (16, 16, 16), ids, ids.clone(), values, viewdirs)


def test_the_six_entry_points_exist_with_their_signatures():
    from nerf_pytorch_b200 import _lib

    GP, NP, P = C.POINTER(_lib.Grid), C.POINTER(_lib.Ndc), C.c_void_p
    I32, I64, F32 = C.c_int32, C.c_int64, C.c_float
    sig = _lib.SIGNATURES
    render = [GP, P, P, I32, P, I32, I64, I32, F32, NP, P, P, P]
    query = [GP, P, P, I32, P, P, I64, P, P, P]
    assert sig["nerfb200_baked_render_normals"] == (I32, render)
    assert sig["nerfb200_baked_render_normals_f16"] == (I32, render)
    assert sig["nerfb200_baked_render_normals_u8"] == (I32, render[:3] + [P] + render[3:])
    assert sig["nerfb200_baked_query"] == (I32, query)
    assert sig["nerfb200_baked_query_f16"] == (I32, query)
    assert sig["nerfb200_baked_query_u8"] == (I32, query[:3] + [P] + query[3:])
    lib = _lib.load()
    for name in ("render_normals", "query"):
        for sfx in ("", "_f16", "_u8"):
            assert hasattr(lib, f"nerfb200_baked_{name}{sfx}")
    # baked_render's own argument list is untouched: the normals render is its arguments plus ndc and normals
    assert sig["nerfb200_baked_render"] == (I32, render[:9] + [P, P])


def test_the_library_refuses_before_any_launch():
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    before = ops.launch_count()
    box = ops.grid_struct(BOX, (16, 16, 16))
    bad_box = ops.grid_struct(((1.0,) * 3, (-1.0,) * 3), (16, 16, 16))
    good_cam = ops.ndc_struct(42, 56, 45.3)
    bad_cams = (ops.ndc_struct(0, 56, 45.3), ops.ndc_struct(42, -1, 45.3), ops.ndc_struct(42, 56, 0.0),
                ops.ndc_struct(42, 56, float("inf")), ops.ndc_struct(42, 56, float("nan")))
    r = lib.nerfb200_baked_render_normals

    def render(b=box, bm=FAKE, vals=FAKE, vd=1, rays=FAKE, stride=11, n=4, t=0.0, cam=None, out=FAKE, nrm=FAKE):
        return r(C.byref(b), bm, vals, vd, rays, stride, n, 0, t, None if cam is None else C.byref(cam), out, nrm, None)

    for kw in (dict(b=bad_box), dict(bm=None), dict(vals=None), dict(rays=None), dict(out=None), dict(nrm=None),
               dict(n=0), dict(n=-1), dict(stride=10), dict(vd=0, stride=7), dict(t=1.0), dict(t=-0.1),
               dict(t=float("nan"))):
        assert render(**kw) == _lib.ERR_INVALID, kw
    for cam in bad_cams:
        assert render(cam=cam) == _lib.ERR_INVALID
        assert "NDC camera" in lib.nerfb200_last_error().decode()
    f16 = lib.nerfb200_baked_render_normals_f16
    assert f16(C.byref(box), FAKE, ODD, 1, FAKE, 11, 4, 0, 0.0, None, FAKE, FAKE, None) == _lib.ERR_INVALID
    assert "aligned" in lib.nerfb200_last_error().decode()
    u8 = lib.nerfb200_baked_render_normals_u8
    assert u8(C.byref(box), FAKE, FAKE, None, 1, FAKE, 11, 4, 0, 0.0, C.byref(good_cam), FAKE, FAKE, None) \
        == _lib.ERR_INVALID
    assert "dequant" in lib.nerfb200_last_error().decode()
    assert u8(C.byref(box), FAKE, ODD, FAKE, 1, FAKE, 11, 4, 0, 0.0, None, FAKE, FAKE, None) == _lib.ERR_INVALID

    q = lib.nerfb200_baked_query

    def query(b=box, bm=FAKE, vals=FAKE, vd=1, pts=FAKE, dirs=FAKE, n=4, raw=FAKE, grad=FAKE):
        return q(C.byref(b), bm, vals, vd, pts, dirs, n, raw, grad, None)

    for kw in (dict(b=bad_box), dict(bm=None), dict(vals=None), dict(pts=None), dict(n=-1), dict(raw=None, grad=None),
               dict(dirs=None)):
        assert query(**kw) == _lib.ERR_INVALID, kw
    assert query(dirs=None) == _lib.ERR_INVALID and "view directions need dirs" in lib.nerfb200_last_error().decode()
    assert query(n=-1) == _lib.ERR_INVALID and "n_points" in lib.nerfb200_last_error().decode()
    assert query(raw=None, grad=None) == _lib.ERR_INVALID and "both null" in lib.nerfb200_last_error().decode()
    qf = lib.nerfb200_baked_query_f16
    assert qf(C.byref(box), FAKE, ODD, 1, FAKE, FAKE, 4, FAKE, FAKE, None) == _lib.ERR_INVALID
    qu = lib.nerfb200_baked_query_u8
    assert qu(C.byref(box), FAKE, FAKE, None, 1, FAKE, FAKE, 4, FAKE, FAKE, None) == _lib.ERR_INVALID
    assert ops.launch_count() == before
    # accepted without a launch: no point, and dirs not needed for the gradient alone or without view directions
    assert query(n=0) == _lib.OK
    assert query(n=0, dirs=None, raw=None) == _lib.OK
    assert query(n=0, vd=0, dirs=None) == _lib.OK
    assert qu(C.byref(box), FAKE, FAKE, FAKE, 1, FAKE, FAKE, 0, FAKE, None, None) == _lib.OK
    assert ops.launch_count() == before


def test_render_refusals():
    import nerf_pytorch_b200 as nb
    from oracle import nerf_oracle as O

    opts = O.make_options(no_ndc=True, near=2.0, far=6.0)
    ndc_opts = O.make_options(no_ndc=False, near=0.0, far=1.0)
    f = _field()
    pose = torch.eye(4)
    with pytest.raises(ValueError, match="normals must be"):
        nb.render_baked(f, 8, 8, 10.0, pose, opts, normals="ndc")
    with pytest.raises(ValueError, match="ndc must be"):  # an NDC scene's world map from a malformed camera
        nb.render_baked(f, 0, 8, 10.0, pose, ndc_opts, normals="world")
    with pytest.raises(NotImplementedError, match="CUDA"):  # a CPU field, after the arguments
        nb.render_baked(f, 8, 8, 10.0, pose, opts, normals=True)
    rays = torch.zeros(4, 11)
    with pytest.raises(ValueError, match="normals must be"):
        nb.render_baked_rays(f, rays, normals="Normals")
    for bad in ((8, 8), (0, 8, 10.0), (8, 8, -1.0), (8.5, 8, 10.0), (8, 8, float("nan")), "8,8,10"):
        with pytest.raises(ValueError, match="ndc must be"):
            nb.render_baked_rays(f, rays, normals=True, ndc=bad)
    with pytest.raises(ValueError, match="normals=True"):  # ndc= without normals
        nb.render_baked_rays(f, rays, ndc=(8, 8, 10.0))
    g = _field(requires_grad=True)
    with pytest.raises(ValueError, match="no gradient"):
        nb.render_baked_rays(g, rays, normals=True)
    with torch.no_grad(), pytest.raises(ValueError, match="CUDA"):  # no gradient: the CPU refusal
        nb.render_baked_rays(g, rays, normals=True)
    with pytest.raises(ValueError, match="CUDA"):  # without normals the CPU refusal comes first, as before
        nb.render_baked_rays(f, rays)


def test_query_refusals():
    import nerf_pytorch_b200 as nb

    pts = torch.zeros(5, 3)
    with pytest.raises(ValueError, match="nb.BakedField"):
        nb.baked_raw(object(), pts)
    with pytest.raises(ValueError, match="nb.BakedField"):
        nb.baked_density_gradient(object(), pts)
    for fn in (nb.baked_density_gradient, lambda f, p: nb.baked_raw(f, p, torch.zeros(5, 3))):
        with pytest.raises(NotImplementedError, match="CUDA"):  # a CPU field
            fn(_field(), pts)
        with pytest.raises(ValueError, match="inference only"):  # values that require grad, in grad mode
            fn(_field(requires_grad=True), pts)
    for bad in ((8, 8), (8, 0, 10.0), (8, 8, 0.0)):
        with pytest.raises(ValueError, match="ndc must be"):
            nb.baked_density_gradient(_field(), pts, ndc=bad)


def test_point_checks_on_a_cuda_looking_field(monkeypatch):
    """The point, view-direction and z checks run after the field's: they are reached with the field's CUDA check
    stubbed out (nothing is launched: every refusal precedes the query)."""
    import importlib

    import nerf_pytorch_b200 as nb

    bake = importlib.import_module("nerf_pytorch_b200.bake")  # the package's name bake is the function
    monkeypatch.setattr(bake, "_query_field", lambda field, what: None)
    f = _field()
    no_view = _field(viewdirs=False)
    with pytest.raises(ValueError, match=r"\(\.\.\., 3\)"):
        nb.baked_raw(f, torch.zeros(5, 2), torch.zeros(5, 2))
    with pytest.raises(ValueError, match=r"\(\.\.\., 3\)"):
        nb.baked_density_gradient(f, torch.zeros(5, 3, dtype=torch.float64))
    with pytest.raises(TypeError):
        nb.baked_density_gradient(f, [[0.0, 0.0, 0.0]])
    with pytest.raises(ValueError, match="z must be < 0"):  # world points with z >= 0
        nb.baked_density_gradient(f, torch.tensor([[0.0, 0.0, -1.0], [0.0, 0.0, 0.0]]), ndc=(8, 8, 10.0))
    with pytest.raises(ValueError, match="pass viewdirs"):  # missing
        nb.baked_raw(f, torch.zeros(5, 3))
    with pytest.raises(ValueError, match="do not pass viewdirs"):  # extra
        nb.baked_raw(no_view, torch.zeros(5, 3), torch.zeros(5, 3))
    with pytest.raises(NotImplementedError, match="CUDA"):  # CPU points reach _checked_points' device refusal
        nb.baked_raw(f, torch.zeros(5, 3), torch.zeros(5, 3))
