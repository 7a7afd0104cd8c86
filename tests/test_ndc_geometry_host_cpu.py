"""World-space geometry of NDC scenes (include/nerfb200.h "NDC scenes"), without a GPU:
  * an fp64 numpy statement of the map N of ndc_rays, its inverse and J^T, against finite differences and against the
    oracle's ndc_rays; the sign of s = 1 / p_z and of det J, and that N keeps straight lines straight;
  * the new C ABI symbols are declared, bound and exported, and refuse a malformed camera or arguments before any launch;
  * every Python refusal of ndc= and normals="world" fires before a device is touched."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from oracle import nerf_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("nerfb200_ndc_mesh_to_world", "nerfb200_ndc_from_world", "nerfb200_ndc_grad_to_world",
       "nerfb200_render_fwd_normals_ndc")
# the fern scene of the shipped weights (tests/test_normals_render_gpu.py)
H, W, FOCAL = 42, 56, 45.3


def _swh(h=H, w=W, f=FOCAL):
    return -1.0 / (w / (2.0 * f)), -1.0 / (h / (2.0 * f))


def N(p, sw, sh):
    return np.stack([sw * p[..., 0] / p[..., 2], sh * p[..., 1] / p[..., 2], 1.0 + 2.0 / p[..., 2]], -1)


def N_inv(q, sw, sh):
    pz = 2.0 / (q[..., 2] - 1.0)
    return np.stack([q[..., 0] * pz / sw, q[..., 1] * pz / sh, pz], -1)


def JT(q, g, sw, sh):
    """The header's J^T(q) g."""
    s = (q[..., 2] - 1.0) * 0.5
    return np.stack([s * sw * g[..., 0], s * sh * g[..., 1],
                     s * (-(q[..., 0] * g[..., 0] + q[..., 1] * g[..., 1]) - (q[..., 2] - 1.0) * g[..., 2])], -1)


def _frustum_points(n, seed):
    rng = np.random.default_rng(seed)
    z = -rng.uniform(1.0, 50.0, n)
    x = rng.uniform(-0.6, 0.6, n) * -z
    y = rng.uniform(-0.4, 0.4, n) * -z
    return np.stack([x, y, z], -1)


def test_inverse_and_jacobian_against_finite_differences():
    sw, sh = _swh()
    p = _frustum_points(2000, 1)
    q = N(p, sw, sh)
    assert np.allclose(N_inv(q, sw, sh), p, rtol=1e-12, atol=1e-12)
    assert (q[:, 2] < 1.0).all() and (q[:, 2] >= -1.0).all()
    # J by central differences, then J^T g for random g against the header's closed form
    h = 1e-6 * np.abs(p[:, 2:3])  # a step relative to the depth
    J = np.empty((p.shape[0], 3, 3))
    for c in range(3):
        e = np.eye(3)[c]
        J[:, :, c] = (N(p + h * e, sw, sh) - N(p - h * e, sw, sh)) / (2 * h)
    g = np.random.default_rng(2).normal(size=p.shape)
    fd = np.einsum("nij,ni->nj", J, g)
    closed = JT(q, g, sw, sh)
    scale = np.abs(fd).max(-1, keepdims=True)
    assert np.abs(closed - fd).max() / scale.min() < 1e-5
    # s = 1 / p_z is negative in the frustum, and N reverses orientation
    s = (q[:, 2] - 1.0) * 0.5
    assert np.allclose(s, 1.0 / p[:, 2]) and (s < 0).all()
    det = np.linalg.det(J)
    assert np.allclose(det, -2.0 * sw * sh / p[:, 2] ** 4, rtol=1e-5) and (det < 0).all()


def test_map_is_ndc_rays_and_keeps_lines_straight():
    sw, sh = _swh()
    rng = np.random.default_rng(3)
    o = rng.normal(size=(500, 3)) * 0.1
    d = np.concatenate([rng.uniform(-0.5, 0.5, (500, 2)), -np.ones((500, 1))], -1)
    ro, rd = O.ndc_rays(H, W, FOCAL, 1.0, torch.from_numpy(o), torch.from_numpy(d))
    ro, rd = ro.numpy(), rd.numpy()
    t_near = -(1.0 + o[:, 2]) / d[:, 2]
    for t in (0.0, 0.5, 3.0, 40.0):
        p = o + (t_near + t)[:, None] * d
        q = N(p, sw, sh)
        # q lies on the NDC ray: q - ro is parallel to rd
        assert np.abs(np.cross(q - ro, rd)).max() < 1e-9 * max(1.0, np.abs(q - ro).max())
    assert np.allclose(N(o + t_near[:, None] * d, sw, sh), ro, atol=1e-12)


def test_sw_sh_are_those_of_ray_generation():
    """fp32(-1 / (W / (2 f))) in double, rounded once, with the fp32 focal: what ops.pack_rays' NDC rows use."""
    f32 = float(np.float32(FOCAL))
    sw = float(np.float32(-1.0 / (float(W) / (2.0 * f32))))
    assert sw == float(np.float32(_swh(f=f32)[0]))


def test_symbols_declared_bound_exported():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import _lib

    header = open(os.path.join(ROOT, "include", "nerfb200.h")).read()
    lib = _lib.load()
    for name in NEW:
        assert re.search(r"\b" + name + r"\(", header), name
        assert name in _lib.SIGNATURES
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1]
    assert "ndc" in nb.extract_mesh.__code__.co_varnames
    assert "ndc" in nb.density_gradient.__code__.co_varnames


def test_c_abi_refuses_before_any_launch():
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    fake = C.c_void_p(0x1000)
    good = ops.ndc_struct(H, W, FOCAL)
    n0 = ops.launch_count()
    for cam in (None, ops.ndc_struct(0, W, FOCAL), ops.ndc_struct(H, -1, FOCAL), ops.ndc_struct(H, W, 0.0),
                ops.ndc_struct(H, W, float("nan")), ops.ndc_struct(H, W, float("inf"))):
        ref = C.byref(cam) if cam is not None else None
        assert lib.nerfb200_ndc_from_world(ref, fake, 4, fake, None) == _lib.ERR_INVALID
        assert lib.nerfb200_ndc_grad_to_world(ref, fake, fake, 4, fake, None) == _lib.ERR_INVALID
        assert lib.nerfb200_ndc_mesh_to_world(ref, fake, fake, None, 4, 4, fake, fake, None, None) == _lib.ERR_INVALID
        assert "NDC camera" in lib.nerfb200_last_error().decode()
    g = C.byref(good)
    assert lib.nerfb200_ndc_from_world(g, fake, -1, fake, None) == _lib.ERR_INVALID
    assert lib.nerfb200_ndc_from_world(g, None, 4, fake, None) == _lib.ERR_INVALID
    assert lib.nerfb200_ndc_grad_to_world(g, fake, None, 4, fake, None) == _lib.ERR_INVALID
    assert lib.nerfb200_ndc_mesh_to_world(g, fake, fake, fake, 4, 4, fake, fake, None, None) == _lib.ERR_INVALID
    assert lib.nerfb200_ndc_mesh_to_world(g, None, fake, None, 4, 4, fake, fake, None, None) == _lib.ERR_INVALID
    assert lib.nerfb200_ndc_mesh_to_world(g, fake, fake, None, 4, -1, fake, fake, None, None) == _lib.ERR_INVALID
    # empty inputs launch nothing and succeed
    assert lib.nerfb200_ndc_from_world(g, None, 0, None, None) == _lib.OK
    assert lib.nerfb200_ndc_mesh_to_world(g, None, None, None, 0, 0, None, None, None, None) == _lib.OK
    a = C.byref(ops.ArchSpec(num_layers=4, hidden=128, skip_every=4, n_freq_xyz=6, n_freq_dir=4).c_struct())
    o = C.byref(ops.make_opts(64, 0, False, False, False, 0.0))
    args = [a, None, o, fake, None, fake, 11, 8, None, None, None, None, None, None, None, -1.0]
    assert lib.nerfb200_render_fwd_normals_ndc(*args, None, fake, None, fake, fake, 1, None) == _lib.ERR_INVALID
    assert lib.nerfb200_render_fwd_normals_ndc(*args, g, fake, None, fake, fake, 0, None) == _lib.ERR_UNSUPPORTED
    assert ops.launch_count() == n0


def _models():
    import nerf_pytorch_b200 as nb

    out = []
    for _ in range(2):
        m = nb.FlexibleNeRFModel(num_layers=4, hidden_size=128, skip_connect_every=4, num_encoding_fn_xyz=6,
                                 num_encoding_fn_dir=4)
        for p in m.parameters():
            p.requires_grad_(False)
        out.append(m)
    return out, nb.get_embedding_function(6), nb.get_embedding_function(4)


BAD_NDC = [(H, W), (H, W, FOCAL, 1), "fern", 3.0, (0, W, FOCAL), (H, -2, FOCAL), (H, W, 0.0),
           (H, W, -1.0), (H, W, float("nan")), (H, W, float("inf")), (42.5, W, FOCAL), (True, W, FOCAL),
           (H, W, "45")]


@pytest.mark.parametrize("bad", BAD_NDC, ids=range(len(BAD_NDC)))
def test_malformed_ndc_is_refused_before_any_device_use(bad):
    """CPU models and points would be refused with NotImplementedError on first use: a ValueError proves the check ran
    first."""
    import nerf_pytorch_b200 as nb

    (m, _), epf, edf = _models()
    box = ((-1.0, -1.0, -1.0), (1.0, 1.0, 0.9))
    with pytest.raises(ValueError, match="ndc"):
        nb.extract_mesh(m, epf, box, 32, encode_direction_fn=edf, ndc=bad)
    with pytest.raises(ValueError, match="ndc"):
        nb.density_gradient(m, epf, -torch.ones(4, 3), ndc=bad)


def test_other_refusals_fire_before_any_device_use():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    (mc, mf), epf, edf = _models()
    n0 = ops.launch_count()
    cam = (H, W, FOCAL)
    for hi_z in (1.0, 1.5, float("inf")):
        with pytest.raises(ValueError, match="hi_z < 1|finite"):
            nb.extract_mesh(mc, epf, ((-1.0, -1.0, -1.0), (1.0, 1.0, hi_z)), 32, encode_direction_fn=edf, ndc=cam)
    with pytest.raises(NotImplementedError, match="CUDA"):  # a well-formed call gets as far as the device check
        nb.extract_mesh(mc, epf, ((-1.0, -1.0, -1.0), (1.0, 1.0, 0.99)), 32, encode_direction_fn=edf, ndc=cam)
    for z in (0.0, 1.0, float("nan")):
        pts = -torch.ones(5, 3)
        pts[3, 2] = z
        with pytest.raises(ValueError, match="z must be < 0"):
            nb.density_gradient(mc, epf, pts, ndc=cam)
    with pytest.raises(NotImplementedError, match="CUDA"):
        nb.density_gradient(mc, epf, -torch.ones(5, 3), ndc=cam)
    fern = O.make_options(no_ndc=False, near=0.0, far=1.0, num_coarse=64, num_fine=64, perturb=False,
                          radiance_field_noise_std=0.0)
    rays = torch.zeros(8, 11)
    kw = dict(encode_position_fn=epf, encode_direction_fn=edf)
    with torch.no_grad():
        with pytest.raises(ValueError, match="H, W and focal"):
            nb.predict_and_render_radiance(rays, mc, mf, fern, normals="world", **kw)
        for bad in ("World", "ndc", ""):
            with pytest.raises(ValueError, match="normals must be"):
                nb.predict_and_render_radiance(rays, mc, mf, fern, normals=bad, **kw)
            with pytest.raises(ValueError, match="normals must be"):
                nb.render_image(H, W, FOCAL, torch.eye(4), mc, mf, fern, normals=bad, device="cpu", **kw)
        with pytest.raises(ValueError, match="ndc must be"):
            nb.render_image(H, W, -1.0, torch.eye(4), mc, mf, fern, normals="world", device="cpu", **kw)
        with pytest.raises(ValueError, match="ndc must be"):
            nb.run_one_iter_of_nerf(0, W, FOCAL, mc, mf, rays[:, :3], rays[:, 3:6], fern, normals="world", **kw)
    assert ops.launch_count() == n0
