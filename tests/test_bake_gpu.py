"""GPU: baked fields (nb.bake / nb.render_baked; csrc/mlp_tc.cu bake_tc_kernel, csrc/baked.cu; include/nerfb200.h
"baked fields").

  1. the bake against the network: sigma_raw and the logits hook at all 64 directions bit-equal mlp_fwd_pts(impl=1) at
     the same points; the SH coefficients match an fp64 projection of those logits.  Lego A0 (shipped), A1 and A2 at
     init, a coarse-only network without view directions, fern A0 in NDC; 1 brick and a count that ends mid-tile;
  2. the bricks are mesh_sparse_bricks'; an empty grid renders acc = 0 and the background;
  3. the renderer against an fp64 restatement that gathers from the kernel's own values: Blender and NDC rays, with and
     without view directions and a white background, rays that miss the box; early stopping;
  4. reproducibility, save / load;
  5. quality: PSNR of render_baked against render_image's fine output on lego (256^3, 512^3) and fern."""
import numpy as np
import pytest
import torch

from helpers import (COEF_REL, FERN_BOX, FERN_CAM, LEGO_BOX, LEGO_CAM, OUT_ABS, baked_render64, bits_equal, net_at,
                     psnr32, scene_pose, shipped_models)

pytestmark = pytest.mark.gpu


def report(what, ctx, value):
    print(f"[bake] {what} {ctx}: {value}")


def _model(kind):
    """(model, encode_position_fn, encode_direction_fn, camera (H, W, focal, pose, no_ndc, near, far), box): the shipped
    scenes' fine network (helpers.shipped_models), or "a1", "a2" and "noview" (coarse-only, no view directions) at
    torch's init under seed 7 on the lego camera."""
    import nerf_pytorch_b200 as nb

    lego_cam = (*LEGO_CAM, "spherical", True, 2.0, 6.0)
    if kind in ("lego", "fern"):
        _, m, epf, edf = shipped_models(kind)
        cam = lego_cam if kind == "lego" else (*FERN_CAM, "eye", False, 0.0, 1.0)
        return m, epf, edf, cam, LEGO_BOX if kind == "lego" else FERN_BOX
    torch.manual_seed(7)
    if kind == "a1":
        m = nb.FlexibleNeRFModel(num_layers=8, hidden_size=128, skip_connect_every=3, num_encoding_fn_xyz=10)
    elif kind == "a2":
        m = nb.FlexibleNeRFModel(num_layers=8, hidden_size=256, skip_connect_every=4, num_encoding_fn_xyz=10)
    else:  # "noview": coarse-only, no view directions
        m = nb.FlexibleNeRFModel(num_layers=4, hidden_size=128, skip_connect_every=4, num_encoding_fn_xyz=10,
                                 use_viewdirs=False)
    return m.cuda(), nb.get_embedding_function(10), nb.get_embedding_function(4), lego_cam, ((-1.0,) * 3, (1.0,) * 3)


def _arch_blob(m, epf, edf):
    from nerf_pytorch_b200 import mesh, train_utils

    arch = mesh._network(m, epf, edf)
    return arch, train_utils._packed(m, arch)[1]


def _field(kind, res=16, grid=None):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    m, epf, edf, cam, box = _model(kind)
    grid = OccupancyGrid.full(box, 8) if grid is None else grid
    return nb.bake(m, epf, edf if m.use_viewdirs else None, bounds=box, resolution=res, grid=grid), m, epf, edf, cam


# ------------------------------------------------------------------------------------------------------------------------
# 1. the bake against the network
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("count", [1, 3])
@pytest.mark.parametrize("kind", ["lego", "a1", "a2", "noview", "fern"])
def test_bake_matches_the_network(kind, count):
    from nerf_pytorch_b200 import ops

    m, epf, edf, _, box = _model(kind)
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    arch, blob = _arch_blob(m, epf, edf if m.use_viewdirs else None)
    g = ops.grid_struct(box, (24, 24, 24))
    brick_map, bricks, n = ops.mesh_sparse_bricks(g, OccupancyGrid.full(box, 8))
    first = 5
    P = count * 729
    values = torch.full((int(n.item()), 729, 32), float("nan"), device="cuda")
    logits = torch.empty(P, 64, 3, device="cuda")
    ops.bake(arch, blob, g, bricks, first, count, values, logits)
    pts = torch.empty(P, 3, device="cuda")
    ops.mesh_sparse_points(g, bricks, first, count, False, pts)
    dirs, proj = ops.bake_basis()
    got = values[first:first + count].reshape(P, 32)
    want_sigma = net_at(arch, blob, pts, None if not arch.use_viewdirs else dirs[0].cuda())[:, 3]
    assert bits_equal(got[:, 0], want_sigma), kind
    if arch.use_viewdirs:
        for d in range(64):
            raw = net_at(arch, blob, pts, dirs[d].cuda())
            assert bits_equal(logits[:, d], raw[:, :3]), (kind, d)
        coef64 = torch.einsum("jd,pdc->pcj", proj.double().cuda(), logits.double())
    else:
        raw = net_at(arch, blob, pts, None)
        assert bits_equal(logits, raw[:, None, :3].expand(P, 64, 3)), kind
        coef64 = torch.zeros(P, 3, 9, dtype=torch.float64, device="cuda")
        coef64[:, :, 0] = raw[:, :3].double() / np.float32(0.28209479177387814)
    scale = logits.abs().amax(dim=(1, 2)).double()[:, None]
    err = ((got[:, 1:28].double().view(P, 3, 9) - coef64).abs().view(P, 27) / scale.clamp_min(1e-30)).max().item()
    report("coefficient error / max |logit|", (kind, count), err)
    assert err <= COEF_REL, (kind, err)
    assert (got[:, 28:] == 0).all()
    untouched = torch.ones(values.shape[0], dtype=torch.bool)
    untouched[first:first + count] = False
    assert torch.isnan(values[untouched.cuda()]).all()


# ------------------------------------------------------------------------------------------------------------------------
# 2. bricks; an empty grid
# ------------------------------------------------------------------------------------------------------------------------
def test_bricks_are_the_sparse_meshes_and_an_empty_grid_renders_the_background():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops
    from nerf_pytorch_b200.occupancy import OccupancyGrid
    from oracle import nerf_oracle as O

    m, epf, edf, cam, box = _model("lego")
    grid = OccupancyGrid.from_models([m], epf, box, 32, encode_direction_fn=edf)
    f = nb.bake(m, epf, edf, bounds=box, resolution=40, grid=grid)
    bm, br, n = ops.mesh_sparse_bricks(ops.grid_struct(box, (40,) * 3), grid)
    assert bits_equal(f.brick_map, bm) and bits_equal(f.bricks, br[:int(n.item())])
    assert 0 < f.n_active < bm.numel()
    H, W, focal, pose, no_ndc, near, far = cam
    # a lattice point outside the grid's box makes its brick active: the empty grid covers the whole lattice
    empty = OccupancyGrid.empty(((-2.0,) * 3, (2.0,) * 3), 32)
    for white in (False, True):
        e = nb.bake(m, epf, edf, bounds=box, resolution=40, grid=empty)
        assert e.n_active == 0
        opts = O.make_options(no_ndc=no_ndc, near=near, far=far, white_background=white)
        rgb, disp, acc = nb.render_baked(e, H, W, focal, scene_pose(pose), opts)
        assert (acc == 0).all() and (rgb == (1.0 if white else 0.0)).all() and torch.isnan(disp).all()


# ------------------------------------------------------------------------------------------------------------------------
# 3. the renderer against fp64
# ------------------------------------------------------------------------------------------------------------------------
def _rays(cam, use_viewdirs):
    from nerf_pytorch_b200 import ops

    H, W, focal, pose, no_ndc, near, far = cam
    return ops.gen_rays(scene_pose(pose), H, W, focal, None, "cuda", ndc=not no_ndc, near=near, far=far,
                        use_viewdirs=use_viewdirs)


@pytest.mark.parametrize("white", [False, True])
@pytest.mark.parametrize("kind", ["lego", "noview", "fern"])
def test_renderer_matches_fp64(kind, white):
    from nerf_pytorch_b200 import ops

    field, m, *_, cam = _field(kind, res=(24, 20, 28))
    rays = _rays(cam, field.use_viewdirs)
    if kind == "lego":  # rays that miss the box: turned away from it
        rays[::7, 3:6] = -rays[::7, 3:6]
    out = ops.baked_render(field.box(), field.brick_map, field.values, field.use_viewdirs, rays, white)
    rgb, acc, depth, disp = baked_render64(field, rays, white)
    far = float(rays[:, 7].max())
    e_rgb = (out[:, :3].double() - rgb).abs().max().item()
    e_acc = (out[:, 4].double() - acc).abs().max().item()
    e_depth = (out[:, 5].double() - depth).abs().max().item() / far
    report("rgb / acc / depth error", (kind, white), (e_rgb, e_acc, e_depth))
    assert e_rgb <= OUT_ABS and e_acc <= OUT_ABS and e_depth <= OUT_ABS
    empty = acc == 0
    assert torch.isnan(out[empty, 3]).all()
    ok = acc > 1e-3
    assert torch.allclose(out[ok, 3].double(), disp[ok], rtol=1e-3)
    if kind == "lego":
        assert bool(empty.any()) and bool((acc > 0.5).any())


def test_early_stop_guarantee():
    from nerf_pytorch_b200 import ops

    field, *_, cam = _field("lego", res=32)
    rays = _rays(cam, True)
    base = ops.baked_render(field.box(), field.brick_map, field.values, True, rays, False)
    for t in (1e-3, 0.1, 0.5):
        e = ops.baked_render(field.box(), field.brick_map, field.values, True, rays, False, t)
        same = (e == base).all(-1) | ((e[:, 3] != e[:, 3]) & (base[:, 3] != base[:, 3]))
        stopped = ~same
        report("rays stopped", t, int(stopped.sum()))
        assert bool(stopped.any()) and bool(same.any())
        d = e[stopped] - base[stopped]
        assert ((d[:, :3] <= 1e-6) & (d[:, :3] >= -t - 1e-6)).all() and ((d[:, 4] <= 1e-6) & (d[:, 4] >= -t - 1e-6)).all()
        assert (base[stopped, 4] >= 1 - t - 1e-5).all()  # a ray stops only once it is nearly opaque


# ------------------------------------------------------------------------------------------------------------------------
# 4. reproducibility
# ------------------------------------------------------------------------------------------------------------------------
def test_bake_and_render_are_reproducible_and_survive_save_load(tmp_path):
    import nerf_pytorch_b200 as nb
    from oracle import nerf_oracle as O

    f1, m, epf, edf, cam = _field("a2", res=24)
    f2, *_ = _field("a2", res=24)
    assert bits_equal(f1.values, f2.values)
    H, W, focal, pose, no_ndc, near, far = cam
    opts = O.make_options(no_ndc=no_ndc, near=near, far=far)
    a = nb.render_baked(f1, H, W, focal, scene_pose(pose), opts)
    b = nb.render_baked(f1, H, W, focal, scene_pose(pose), opts)
    f1.save(tmp_path / "field.pt")
    g = nb.BakedField.load(tmp_path / "field.pt")
    c = nb.render_baked(g, H, W, focal, scene_pose(pose), opts)
    for x, y, z in zip(a, b, c):
        assert bits_equal(x, y) and bits_equal(x, z)


# ------------------------------------------------------------------------------------------------------------------------
# 5. quality against the network's render
# ------------------------------------------------------------------------------------------------------------------------
# PSNR (dB) of render_baked against render_image's fine output, measured on an H100 80GB HBM3 at 700 W; the test allows
# PSNR_MARGIN below each
PSNR_MEASURED = {("lego", 256): 29.38, ("lego", 512): 35.39, ("fern", 256): 27.53}
PSNR_MARGIN = 1.0


@pytest.mark.parametrize("kind,res", list(PSNR_MEASURED))
def test_quality_against_the_network(kind, res):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200.occupancy import OccupancyGrid
    from oracle import nerf_oracle as O

    m, epf, edf, cam, box = _model(kind)
    H, W, focal, pose, no_ndc, near, far = cam
    grid = OccupancyGrid.from_models([m], epf, box, 128, encode_direction_fn=edf)
    field = nb.bake(m, epf, edf, bounds=box, resolution=res, grid=grid)
    opts = O.make_options(no_ndc=no_ndc, near=near, far=far, num_coarse=64, num_fine=128, perturb=False,
                          radiance_field_noise_std=0.0)
    mc = shipped_models(kind)[0]
    ref = nb.render_image(H, W, focal, scene_pose(pose), mc, m, opts, encode_position_fn=epf, encode_direction_fn=edf,
                          impl=1)[3]
    rgb, _, _ = nb.render_baked(field, H, W, focal, scene_pose(pose), opts)
    psnr = psnr32(rgb, ref)
    report("PSNR vs render_image", (kind, res, field.n_active), psnr)
    assert psnr >= PSNR_MEASURED[(kind, res)] - PSNR_MARGIN
