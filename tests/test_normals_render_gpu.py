"""Normal maps of renders (include/nerfb200.h, "normal maps"; csrc/normals.cu and density_grad_tc_kernel) on the GPU:
  * with normals=True the six render outputs are bit for bit those of the same call without it: the default render,
    with an occupancy grid, with early stopping, and with both;
  * N against an fp64 restatement from the render's own workspace (mlp_checks.normals64): the last pass's depths and
    raw outputs, the fp64 compositing weights of that raw (with the seeded noise the render used), and grad sigma by fp64
    autograd at o + d z, summed in sample order -- lego A0 (Blender), fern A0 (NDC), a coarse-only network, a seeded
    perturb + noise render, 8 x 256 networks (A2) and A1 / A2 mixed across the two passes, with and without a grid and
    early stopping, and a last pass of 1024 samples;
  * |N| <= acc + eps, N = 0 exactly where acc = 0;
  * cast_to_normal_image, and the refusals (a call that would train, impl 0, impl 3) before any launch."""
import pytest
import torch

import mlp_checks as M
from helpers import bits_equal, scene_pose
from mlp_checks import ACC_EPS, G_ERR, N_FLOOR
from oracle import nerf_oracle as O

pytestmark = pytest.mark.gpu

# (shipped weights or None, H, W, focal, pose, no_ndc, near, far, L_xyz, (coarse, fine) networks, bounds of a grid):
# mlp_checks.H256_SCENES' format.  The bars on N (G_ERR, N_FLOOR, ACC_EPS) are mlp_checks'.
A0 = (4, 128, 4, "shipped")
SCENES = {
    "lego": ("lego_lowres", 48, 48, 66.7, "spherical", True, 2.0, 6.0, 10, (A0, A0), ((-1.5,) * 3, (1.5,) * 3)),
    "fern": ("fern_lowres", 42, 56, 45.3, "eye", False, 0.0, 1.0, 6, (A0, A0), ((-1.2, -1.2, -1.0), (1.2, 1.2, 1.0))),
    **M.H256_SCENES,
}
H256 = list(M.H256_SCENES)


def report(what, ctx, value):
    print(f"measured {what} {ctx}: {value}")


def _options(scene, perturb=False, noise=0.0, num_fine=128):
    _, H, W, focal, pose, no_ndc, near, far, *_ = SCENES[scene]
    return O.make_options(no_ndc=no_ndc, near=near, far=far, num_coarse=64, num_fine=num_fine, perturb=perturb,
                          radiance_field_noise_std=noise)


def _grid(scene, models, encoders):
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    return OccupancyGrid.from_models(models, encoders[0], SCENES[scene][-1], 128, encode_direction_fn=encoders[1])


def _image(scene, normals, grid=None, early_stop=None, randoms=None, perturb=False, noise=0.0):
    import nerf_pytorch_b200 as nb

    _, H, W, focal, pose, _, _, _, l_xyz, *_ = SCENES[scene]
    mc, mf = M.scene_models(SCENES[scene])
    return nb.render_image(H, W, focal, scene_pose(pose), mc, mf, _options(scene, perturb, noise), mode="validation",
                           encode_position_fn=nb.get_embedding_function(l_xyz),
                           encode_direction_fn=nb.get_embedding_function(4), impl=1, grid=grid,
                           early_stop=early_stop, randoms=randoms, normals=normals)


VARIANTS = ["default", "grid", "early_stop", "grid+early_stop"]


@pytest.mark.parametrize("variant", VARIANTS)
def test_six_outputs_are_those_of_the_render_without_normals(variant):
    _six_outputs_are_those_of_the_render_without_normals("lego", variant)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("scene", H256)
def test_six_outputs_are_those_of_the_render_without_normals_at_hidden_256(scene, variant):
    _six_outputs_are_those_of_the_render_without_normals(scene, variant)


def _six_outputs_are_those_of_the_render_without_normals(scene, variant):
    import nerf_pytorch_b200 as nb

    grid = None
    if "grid" in variant:
        mc, mf = M.scene_models(SCENES[scene])
        grid = _grid(scene, [mc, mf], (nb.get_embedding_function(SCENES[scene][8]), nb.get_embedding_function(4)))
    stop = 1e-3 if "early_stop" in variant else None
    rng = nb.SeededRandoms(5, 2)
    plain = _image(scene, False, grid, stop, rng, perturb=True, noise=0.2)
    with_n = _image(scene, True, grid, stop, rng, perturb=True, noise=0.2)
    assert len(plain) == 6 and len(with_n) == 7
    assert all(bits_equal(a, b) for a, b in zip(plain, with_n[:6])), (scene, variant)
    n, acc = with_n[6], with_n[5]
    assert n.shape == (*SCENES[scene][1:3], 3) and torch.isfinite(n).all()
    norm = n.norm(dim=-1)
    report("max |N| - acc", (scene, variant), f"{(norm - acc).max().item():.3e}")
    assert (norm <= acc + ACC_EPS).all()
    assert (n[acc == 0] == 0).all()
    img = nb.cast_to_normal_image(n)
    assert img.dtype == torch.uint8 and img.shape == n.shape


def _render(scene, perturb, noise, coarse_only, seed, grid_kind=None, stop=None, counts=(64, 128)):
    """(arch of the last pass, its state dict, rays, z, raw, noise of the last pass or None, noise_std, normals, acc)
    of one render_fwd_normals call at (n_coarse, n_fine) `counts` (with a grid of the networks' density for grid_kind
    "model", early stopping at `stop`), read back from its workspace."""
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops, train_utils

    _, H, W, focal, pose, no_ndc, near, far, l_xyz, *_ = SCENES[scene]
    mc, mf = M.scene_models(SCENES[scene])
    epf, edf = nb.get_embedding_function(l_xyz), nb.get_embedding_function(4)
    archs = [train_utils._arch_of(m, train_utils._probe_encoder(epf, None), train_utils._probe_encoder(edf, None))
             for m in (mc, mf)]
    blobs = [train_utils._packed(m, a)[1] for m, a in zip((mc, mf), archs)]
    sd_last = {k: v.detach().cpu() for k, v in (mc if coarse_only else mf).state_dict().items()}
    grid = _grid(scene, [mc, mf], (epf, edf)) if grid_kind == "model" else None
    nc, nf = counts[0], 0 if coarse_only else counts[1]
    opts = ops.make_opts(nc, nf, perturb, False, False, noise)
    rays = ops.gen_rays(scene_pose(pose), H, W, focal, None, "cuda", ndc=not no_ndc, near=near, far=far)
    rng = nb.SeededRandoms(seed, 0)
    arch, arch_f = archs[0], None if coarse_only else archs[1]
    with torch.no_grad():
        out_c, out_f, normals, ws = ops.render_fwd_normals(arch, arch_f, opts, blobs[0], blobs[1] if nf else None, rays,
                                                           rng, grid, stop, impl=1)
    n, s = rays.shape[0], nc + nf
    lay = ops.render_workspace_layout(arch, arch_f, opts, n, False)
    zname, rname = ("z_coarse", "raw_coarse") if coarse_only else ("z_fine", "raw_fine")
    f = ws.view(torch.float32)
    z = f[lay[zname] // 4: lay[zname] // 4 + n * s].view(n, s)
    raw = f[lay[rname] // 4: lay[rname] // 4 + n * s * 4].view(n, s, 4)
    nz = ops.random_fill(rng, "noise_c" if coarse_only else "noise_f", n, s) if noise > 0 else None
    acc = (out_c if coarse_only else out_f)[:, 4]
    return arch_f or arch, sd_last, rays, z.clone(), raw.clone(), nz, noise, normals, acc


@pytest.mark.parametrize("scene,perturb,noise,coarse_only", [
    ("lego", False, 0.0, False), ("fern", False, 0.0, False), ("lego", False, 0.0, True), ("lego", True, 0.2, False),
    ("a2", False, 0.0, False), ("mixed", False, 0.0, False), ("mixed_rev", True, 0.2, False)])
def test_normals_match_an_fp64_restatement(scene, perturb, noise, coarse_only):
    _normals_match_an_fp64_restatement(scene, perturb, noise, coarse_only, None, None)


@pytest.mark.parametrize("scene,perturb,noise,coarse_only,grid_kind,stop", [
    ("lego", True, 0.2, False, "model", 1e-2), ("a2", True, 0.2, False, "model", 1e-2),
    ("a2", False, 0.0, True, None, 1e-2), ("mixed", False, 0.0, False, "model", None),
    ("mixed_rev", True, 0.2, False, None, 1e-2)])
def test_normals_with_a_grid_or_early_stopping_match_an_fp64_restatement(scene, perturb, noise, coarse_only, grid_kind,
                                                                          stop):
    _normals_match_an_fp64_restatement(scene, perturb, noise, coarse_only, grid_kind, stop)


def test_normals_at_1024_samples_match_an_fp64_restatement():
    """The largest pass the library takes: the density gradient runs over n_rays x 1024 compacted points."""
    _normals_match_an_fp64_restatement("lego", True, 0.2, False, None, None, (64, 960))


def _normals_match_an_fp64_restatement(scene, perturb, noise, coarse_only, grid_kind, stop, counts=(64, 128)):
    ctx = (scene, perturb, noise, coarse_only, grid_kind, stop, counts)
    arch, sd, rays, z, raw, nz, std, normals, acc = _render(scene, perturb, noise, coarse_only, 3, grid_kind, stop,
                                                            counts)
    N64, bound, n_live, n_tie = M.normals64(arch, sd, rays, z, raw, std, nz)
    err = (normals.double() - N64).abs().max(-1).values
    report("max |N - N64|", ctx, f"{err.max().item():.3e}, max err / bound {(err / bound).max().item():.3f} (rays "
                                 f"{rays.shape[0]}, live samples {n_live}, tie samples {n_tie})")
    assert (err <= bound).all(), ctx
    assert (normals.norm(dim=-1) <= acc + ACC_EPS).all(), ctx
    assert (normals[acc == 0] == 0).all(), ctx


def test_normals_refusals_fire_before_any_launch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    mc, mf = M.scene_models(SCENES["lego"])
    kw = dict(encode_position_fn=nb.get_embedding_function(10), encode_direction_fn=nb.get_embedding_function(4))
    o = _options("lego", num_fine=64)
    rays = ops.gen_rays(torch.eye(4), 8, 8, 10.0, None, "cuda", ndc=False, near=2.0, far=6.0)
    with torch.no_grad():  # pack both models once, so that nothing below is a first use
        nb.predict_and_render_radiance(rays, mc, mf, o, normals=True, **kw)
    torch.cuda.synchronize()
    before = ops.launch_count()
    with pytest.raises(NotImplementedError, match="inference"):
        nb.predict_and_render_radiance(rays, mc, mf, o, normals=True, **kw)
    with pytest.raises(NotImplementedError, match="inference"):
        nb.run_one_iter_of_nerf(8, 8, 10.0, mc, mf, rays[:, :3], rays[:, 3:6], o, normals=True, **kw)
    with torch.no_grad():
        for bad in (ops.IMPL_SIMT, ops.IMPL_TC_FAST):
            with pytest.raises(NotImplementedError, match="impl"):
                nb.predict_and_render_radiance(rays, mc, mf, o, normals=True, impl=bad, **kw)
            with pytest.raises(NotImplementedError, match="impl=1"):
                ops.render_fwd_normals(ops.ArchSpec(num_layers=4, hidden=128, skip_every=4, n_freq_xyz=10,
                                                    n_freq_dir=4), None, ops.make_opts(64, 0, False, False, False, 0.0),
                                       torch.zeros(1, device="cuda"), None, rays, {}, impl=bad)
        # 8x256 with L_dir 6: 39 direction channels, wider than the wgmma forward's 32
        ldir6 = [nb.FlexibleNeRFModel(num_layers=8, hidden_size=256, num_encoding_fn_xyz=10, num_encoding_fn_dir=6).cuda()
                 for _ in range(2)]
        kw6 = dict(encode_position_fn=kw["encode_position_fn"], encode_direction_fn=nb.get_embedding_function(6))
        grid = OccupancyGrid.full(SCENES["lego"][-1], 16)
        for g, stop in ((None, None), (grid, None), (None, 1e-2), (grid, 1e-2)):
            with pytest.raises(NotImplementedError, match="32"):
                nb.predict_and_render_radiance(rays, *ldir6, o, normals=True, grid=g, early_stop=stop, **kw6)
        a6 = ops.ArchSpec(num_layers=8, hidden=256, n_freq_xyz=10, n_freq_dir=6)
        assert "32" in ops.density_grad_refusal(a6)
        with pytest.raises(NotImplementedError, match="32"):
            ops.render_fwd_normals(a6, a6, ops.make_opts(64, 64, False, False, False, 0.0),
                                   torch.zeros(a6.blob_floats(), device="cuda"), torch.zeros(a6.blob_floats(), device="cuda"),
                                   rays, {}, impl=ops.IMPL_TC)
    assert ops.launch_count() == before
    with torch.no_grad(), pytest.raises(NotImplementedError, match="32"):  # after generating the image's rays
        nb.render_image(8, 8, 10.0, torch.eye(4), *ldir6, o, normals=True, **kw6)
