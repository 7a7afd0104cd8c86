"""GPU: occupancy-grid inference renders (nb.OccupancyGrid, ops.render_fwd_grid, render_image(grid=...)).
  1. a full grid gives render_fwd's six outputs bit for bit, every sample evaluated, also at the sample counts where
     compaction and the wgmma tiles change shape (COUNTS);
  2. an empty grid evaluates nothing: every ray composites zero density;
  3. per ray: a ray none of whose skipped samples (either pass) has positive density in the default render's raw is
     bit-identical to the default render; every evaluated point's raw equals the default raw at that point;
  4. the compaction's map, padding and blocks against a torch restatement, and its determinism;
  5. chunking invariance of grid renders with seeded randoms;
  6. the refusals, before any launch;
  7. PSNR of renders with grids built from the shipped lego and fern weights, against the default render.
Run with -s to print the measured figures."""
import math

import pytest
import torch

import mlp_checks as M
from helpers import OUT_NAMES, bits_equal, compaction_reference, psnr64, scene_pose, skipped_samples, ws_view

pytestmark = pytest.mark.gpu

# (shipped weights or None, H, W, focal, pose, no_ndc, near, far, L_xyz, (coarse, fine) networks, bounds of the grid):
# mlp_checks.H256_SCENES' format
A0, A1 = (4, 128, 4, "shipped"), (8, 128, 3, "init")
SCENES = {
    "lego": ("lego_lowres", 48, 48, 66.7, "spherical", True, 2.0, 6.0, 10, (A0, A0), ((-1.5,) * 3, (1.5,) * 3)),
    "a1": (None, 40, 40, 55.0, "spherical", True, 2.0, 6.0, 10, (A1, A1), ((-1.5,) * 3, (1.5,) * 3)),
    "fern": ("fern_lowres", 42, 56, 45.3, "eye", False, 0.0, 1.0, 6, (A0, A0), ((-1.2, -1.2, -1.0), (1.2, 1.2, 1.0))),
    **M.H256_SCENES,
}
# the scenes whose networks run hidden 256 in some pass
H256 = list(M.H256_SCENES)
VARIANTS = {  # (perturb, noise_std, white_bkgd)
    "det": (False, 0.0, False),
    "perturb_noise": (True, 1.0, False),
    "white_perturb": (True, 0.0, True),
}
IMPLS = {"impl1": 1, "impl3": 3}


def report(what, ctx, value):
    print(f"[occupancy] {what} {ctx}: {value}")


def _setup(scene, variant="det", n_fine=128, n_coarse=64):
    """((arch_c, arch_f), blobs, opts, rays, models, encoders) of a scene at the ops level."""
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops, train_utils

    _, H, W, focal, pose, no_ndc, near, far, l_xyz, *_ = SCENES[scene]
    mc, mf = M.scene_models(SCENES[scene])
    epf, edf = nb.get_embedding_function(l_xyz), nb.get_embedding_function(4)
    archs = tuple(train_utils._arch_of(m, train_utils._probe_encoder(epf, None), train_utils._probe_encoder(edf, None))
                  for m in (mc, mf))
    blobs = [train_utils._packed(m, a)[1] for m, a in zip((mc, mf), archs)]
    perturb, noise, white = VARIANTS[variant]
    opts = ops.make_opts(n_coarse, n_fine, perturb, False, white, noise)
    rays = ops.gen_rays(scene_pose(pose), H, W, focal, None, "cuda", ndc=not no_ndc, near=near, far=far)
    return archs, blobs, opts, rays, (mc, mf), (epf, edf)


def _grid_random(scene, frac, seed, res=32):
    """A seeded grid with a fraction ``frac`` of its cells occupied.  In NDC (fern) a ray through the camera centre keeps
    its (x, y), and the scene has density along nearly every ray, so the cells are (x, y) columns one cell deep: a ray
    whose column is occupied skips nothing."""
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    g = torch.Generator(device="cuda").manual_seed(seed)
    rz = 1 if scene == "fern" else res
    occ = torch.rand(rz, res, res, generator=g, device="cuda") < frac
    return OccupancyGrid.from_occupancy(SCENES[scene][-1], occ)


def _grid_model(scene, models, encoders, res=64):
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    return OccupancyGrid.from_models(models, encoders[0], SCENES[scene][-1], res, encode_direction_fn=encoders[1])


def _render_both(archs, blobs, opts, rays, grid, impl, rng):
    from nerf_pytorch_b200 import ops

    oc, of, ws = ops.render_fwd(*archs, opts, blobs[0], blobs[1], rays, rng, training=False, impl=impl)
    ne = torch.zeros(2, dtype=torch.int64, device="cuda")
    gc, gf, gws = ops.render_fwd_grid(*archs, opts, blobs[0], blobs[1], rays, rng, grid, impl=impl, n_evaluated=ne)
    torch.cuda.synchronize()
    return (oc, of, ws), (gc, gf, gws), ne


# ------------------------------------------------------------------------------------------------------------------------
# 1. full grid
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("scene", list(SCENES))
@pytest.mark.parametrize("impl", list(IMPLS))
def test_full_grid_is_the_default_render_bit_for_bit(impl, scene, variant):
    _full_grid_is_the_default_render_bit_for_bit(impl, scene, variant)


# (n_coarse, n_fine) where compaction changes shape: each group of 10 rays holds 10 S rows, no multiple of the 64-row
# blocks here; the wgmma kernels' smallest pass (15 samples, 10 rays per tile); the early-stopping counts of
# test_early_stop_gpu.py (one partial round of 32, a last round of one, exactly one round, 32 rounds)
COUNTS = [(15, 0), (33, 0), (15, 17), (15, 1009)]


@pytest.mark.parametrize("counts", COUNTS, ids=[f"{nc}+{nf}" for nc, nf in COUNTS])
@pytest.mark.parametrize("scene", ["lego", "a2"])
@pytest.mark.parametrize("impl", list(IMPLS))
def test_full_grid_is_the_default_render_bit_for_bit_at_boundary_counts(impl, scene, counts):
    _full_grid_is_the_default_render_bit_for_bit(impl, scene, "perturb_noise", *counts)


def _full_grid_is_the_default_render_bit_for_bit(impl, scene, variant, nc=64, nf=128):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    archs, blobs, opts, rays, _, _ = _setup(scene, variant, nf, nc)
    if not nf:
        archs, blobs = (archs[0], None), [blobs[0], None]
    grid = OccupancyGrid.full(SCENES[scene][-1], 32)
    (oc, of, _), (gc, gf, _), ne = _render_both(archs, blobs, opts, rays, grid, IMPLS[impl], nb.SeededRandoms(5, 2))
    n = rays.shape[0]
    assert bits_equal(gc, oc) and bits_equal(gf, of), (impl, scene, variant, nc, nf)
    assert ne.tolist() == [n * nc, n * (nc + nf) if nf else 0], (impl, scene, variant, nc, nf)


# ------------------------------------------------------------------------------------------------------------------------
# 2. empty grid
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("impl", list(IMPLS))
def test_empty_grid_composites_zero_density(impl, variant):
    _empty_grid_composites_zero_density(impl, "lego", variant)


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("scene", H256)
@pytest.mark.parametrize("impl", list(IMPLS))
def test_empty_grid_composites_zero_density_at_hidden_256(impl, scene, variant):
    _empty_grid_composites_zero_density(impl, scene, variant)


def _empty_grid_composites_zero_density(impl, scene, variant):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    archs, blobs, opts, rays, _, _ = _setup(scene, variant)
    grid = OccupancyGrid.empty(((-100.0,) * 3, (100.0,) * 3), 16)
    before = ops.launch_count()
    ne = torch.full((2,), -1, dtype=torch.int64, device="cuda")
    oc, of, _ = ops.render_fwd_grid(*archs, opts, blobs[0], blobs[1], rays, nb.SeededRandoms(1), grid,
                                    impl=IMPLS[impl], n_evaluated=ne)
    torch.cuda.synchronize()
    assert ne.tolist() == [0, 0]
    bg = 1.0 if VARIANTS[variant][2] else 0.0
    for out in (oc, of):
        assert torch.equal(out[:, :3], torch.full_like(out[:, :3], bg))
        assert torch.equal(out[:, 4], torch.zeros_like(out[:, 4])) and torch.equal(out[:, 5], torch.zeros_like(out[:, 5]))
        assert torch.isnan(out[:, 3]).all()  # 0 / 0, as the default kernel gives for acc = 0
    # two compaction launches' worth per pass and nothing else changes: 2 samplers, 2 x (3 compaction + MLP + composite)
    assert ops.launch_count() - before == 12


# ------------------------------------------------------------------------------------------------------------------------
# 3. the exact per-ray statement and the evaluated raw
# ------------------------------------------------------------------------------------------------------------------------
def _dense(raw, noise, std):
    pre = raw[..., 3]
    if std > 0:
        pre = pre + noise * torch.tensor(std, dtype=torch.float32, device=raw.device)
    return torch.relu(pre) > 0


GRIDS = ["rand10", "rand50", "rand90", "model"]


@pytest.mark.parametrize("grid_kind", GRIDS)
@pytest.mark.parametrize("variant", ["det", "perturb_noise"])
@pytest.mark.parametrize("scene", list(SCENES))
@pytest.mark.parametrize("impl", list(IMPLS))
def test_rays_without_skipped_density_are_bit_identical(impl, scene, variant, grid_kind):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    archs, blobs, opts, rays, models, enc = _setup(scene, variant)
    if grid_kind == "model":
        grid = _grid_model(scene, models, enc)
    else:
        grid = _grid_random(scene, int(grid_kind[4:]) / 100, seed=len(scene) + int(grid_kind[4:]))
    rng = nb.SeededRandoms(9, 4)
    (oc, of, ws), (gc, gf, gws), ne = _render_both(archs, blobs, opts, rays, grid, IMPLS[impl], rng)
    n, nc, ns = rays.shape[0], 64, 192
    lay = ops.render_workspace_layout(*archs, opts, n, False)
    z_c, z_f = ws_view(ws, lay, "z_coarse", n, nc, 1), ws_view(ws, lay, "z_fine", n, ns, 1)
    raw_c, raw_f = ws_view(ws, lay, "raw_coarse", n, nc, 4), ws_view(ws, lay, "raw_fine", n, ns, 4)
    std = opts.noise_std
    noise_c = ops.random_fill(rng, "noise_c", n, nc) if std > 0 else None
    noise_f = ops.random_fill(rng, "noise_f", n, ns) if std > 0 else None
    sk_c, sk_f = skipped_samples(grid, rays, z_c), skipped_samples(grid, rays, z_f)
    bad = (sk_c & _dense(raw_c, noise_c, std)).any(1) | (sk_f & _dense(raw_f, noise_f, std)).any(1)
    clean = ~bad
    ctx = (impl, scene, variant, grid_kind)
    report("rays with no skipped density / all", ctx, f"{int(clean.sum())} / {n}")
    report("evaluated fraction coarse, fine", ctx, (ne[0].item() / (n * nc), ne[1].item() / (n * ns)))
    assert int(clean.sum()) > 0, ctx
    for a, b in ((gc, oc), (gf, of)):
        assert bits_equal(a[clean], b[clean]), ctx
    assert ne[0].item() == int((~sk_c).sum())

    # every evaluated point's raw is the default raw at that point; skipped samples hold [0 0 0 -inf]
    g_zc, g_zf = ws_view(gws, lay, "z_coarse", n, nc, 1), ws_view(gws, lay, "z_fine", n, ns, 1)
    g_rc, g_rf = ws_view(gws, lay, "raw_coarse", n, nc, 4), ws_view(gws, lay, "raw_fine", n, ns, 4)
    assert bits_equal(g_zc, z_c)
    assert bits_equal(g_rc[~sk_c], raw_c[~sk_c])
    skip_raw = torch.tensor([0.0, 0.0, 0.0, -math.inf], device="cuda")
    assert torch.equal(g_rc[sk_c], skip_raw.expand(int(sk_c.sum()), 4))
    g_sk_f = skipped_samples(grid, rays, g_zf)
    same_z = g_zf.view(torch.int32) == z_f.view(torch.int32)
    ev = ~g_sk_f & same_z
    assert bits_equal(g_rf[ev], raw_f[ev])
    assert ne[1].item() == int((~g_sk_f).sum())
    # points whose depth moved: compare with the default kernel at the grid render's own depths
    moved = ~g_sk_f & ~same_z
    if moved.any():
        raw_at = ops.mlp_fwd(archs[1], blobs[1], rays, g_zf.contiguous(), impl=IMPLS[impl])
        assert bits_equal(g_rf[moved], raw_at[moved])


# ------------------------------------------------------------------------------------------------------------------------
# 4. compaction against a torch restatement
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1237, 64), (403, 192), (7, 15)])
def test_compaction_matches_torch_restatement_and_repeats(shape):
    from nerf_pytorch_b200 import ops

    n, s = shape
    _, _, _, rays, _, _ = _setup("lego")
    rays = rays[:n].contiguous()
    g = torch.Generator(device="cuda").manual_seed(n)
    z = torch.sort(2.0 + 4.0 * torch.rand(n, s, generator=g, device="cuda"), -1)[0]
    grid = _grid_random("lego", 0.3, seed=s, res=24)
    raw0 = torch.randn(n, s, 4, device="cuda")
    raw, m, blocks, nb_, ne = ops.grid_compact(grid, rays, z, raw0.clone())
    raw2, m2, blocks2, nb2, ne2 = ops.grid_compact(grid, rays, z, raw0.clone())
    torch.cuda.synchronize()
    keep, rows, want_blocks = compaction_reference(grid, rays, z)
    nb = nb_.item()
    assert nb == len(want_blocks) and ne.item() == int(keep.sum())
    assert m[:64 * nb].tolist() == rows
    assert [tuple(b) for b in blocks[:nb].tolist()] == want_blocks
    assert all(b - a + 1 <= 10 for a, b in want_blocks)
    assert torch.equal(raw[keep], raw0[keep])
    assert torch.equal(raw[~keep][:, :3], torch.zeros_like(raw[~keep][:, :3]))
    assert torch.isneginf(raw[~keep][:, 3]).all()
    assert torch.equal(m, m2) and torch.equal(blocks, blocks2) and nb2.item() == nb and torch.equal(raw, raw2)
    report("rows / evaluated", shape, (64 * nb, ne.item()))


# ------------------------------------------------------------------------------------------------------------------------
# 5. chunking
# ------------------------------------------------------------------------------------------------------------------------
def _image(scene, impl, chunk, grid=None, randoms=None, perturb=True, noise=0.5):
    import nerf_pytorch_b200 as nb
    from oracle import nerf_oracle as O

    _, H, W, focal, pose, no_ndc, near, far, l_xyz, *_ = SCENES[scene]
    mc, mf = M.scene_models(SCENES[scene])
    opts = O.make_options(no_ndc=no_ndc, near=near, far=far, num_coarse=64, num_fine=128, perturb=perturb,
                          radiance_field_noise_std=noise)
    return nb.render_image(H, W, focal, scene_pose(pose), mc, mf, opts, mode="validation",
                           encode_position_fn=nb.get_embedding_function(l_xyz),
                           encode_direction_fn=nb.get_embedding_function(4), rays_per_chunk=chunk, impl=impl,
                           randoms=randoms, grid=grid)


@pytest.mark.parametrize("impl", list(IMPLS))
def test_grid_render_image_is_chunking_invariant(impl):
    _grid_render_image_is_chunking_invariant(impl, "lego")


@pytest.mark.parametrize("scene", H256)
@pytest.mark.parametrize("impl", list(IMPLS))
def test_grid_render_image_is_chunking_invariant_at_hidden_256(impl, scene):
    _grid_render_image_is_chunking_invariant(impl, scene)


def _grid_render_image_is_chunking_invariant(impl, scene):
    import nerf_pytorch_b200 as nb

    grid = _grid_random(scene, 0.5, seed=3)
    rng = nb.SeededRandoms(21, 1)
    n = SCENES[scene][1] * SCENES[scene][2]
    whole = _image(scene, IMPLS[impl], n, grid, rng)
    for chunk in (1000, 333):
        part = _image(scene, IMPLS[impl], chunk, grid, rng)
        assert all(bits_equal(a, b) for a, b in zip(whole, part)), (scene, chunk)
    default = _image(scene, IMPLS[impl], n, None, rng)
    assert not all(bits_equal(a, b) for a, b in zip(whole, default)), scene  # the grid did skip density


# ------------------------------------------------------------------------------------------------------------------------
# 6. refusals
# ------------------------------------------------------------------------------------------------------------------------
def test_grid_refusals_fire_before_any_launch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops
    from nerf_pytorch_b200.occupancy import OccupancyGrid
    from oracle import nerf_oracle as O

    mc, mf = M.scene_models(SCENES["lego"])
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    kw = dict(encode_position_fn=epf, encode_direction_fn=edf)
    opts = O.make_options(num_coarse=64, num_fine=64)
    grid = OccupancyGrid.full(SCENES["lego"][-1], 16)
    rays = ops.gen_rays(scene_pose("spherical"), 16, 16, 20.0, None, "cuda")
    with torch.no_grad():  # pack both models once, so that nothing below is a first use
        nb.predict_and_render_radiance(rays, mc, mf, opts, grid=grid, **kw)
    torch.cuda.synchronize()
    before = ops.launch_count()
    ro = torch.randn(64, 3, device="cuda")
    with pytest.raises(NotImplementedError, match="inference"):
        nb.predict_and_render_radiance(rays, mc, mf, opts, grid=grid, **kw)
    with pytest.raises(NotImplementedError, match="inference"):
        nb.run_one_iter_of_nerf(16, 16, 20.0, mc, mf, ro, -ro, opts, grid=grid, **kw)
    with pytest.raises(NotImplementedError, match="inference"):
        nb.run_one_iter_of_nerf_from_pose(16, 16, 20.0, mc, mf, torch.eye(4), None, opts, grid=grid, **kw)
    with torch.no_grad():
        with pytest.raises(NotImplementedError, match="impl 0"):
            nb.predict_and_render_radiance(rays, mc, mf, opts, grid=grid, impl=ops.IMPL_SIMT, **kw)
        few = O.make_options(num_coarse=14, num_fine=0)
        with pytest.raises(NotImplementedError, match="fewer than 15 samples"):
            nb.predict_and_render_radiance(rays, mc, None, few, grid=grid, impl=ops.IMPL_TC, **kw)
        wide = nb.FlexibleNeRFModel(num_encoding_fn_xyz=11, include_input_xyz=False).cuda()
        with pytest.raises(NotImplementedError, match="wider than 64"):
            nb.predict_and_render_radiance(rays, wide, None, O.make_options(num_fine=0), grid=grid, impl=ops.IMPL_TC_FAST,
                                           encode_position_fn=nb.get_embedding_function(11, include_input=False),
                                           encode_direction_fn=edf)
        with pytest.raises(RuntimeError, match="is on cpu"):
            nb.predict_and_render_radiance(rays, mc, mf, opts, grid=grid.to("cpu"), **kw)
        with pytest.raises(RuntimeError, match="is on cpu"):
            nb.render_image(16, 16, 20.0, torch.eye(4), mc, mf, opts, grid=grid.to("cpu"), **kw)
        bad = OccupancyGrid.full(SCENES["lego"][-1], 16)
        bad.bits = bad.bits.to(torch.int64)
        with pytest.raises(RuntimeError, match="int32"):
            nb.predict_and_render_radiance(rays, mc, mf, opts, grid=bad, **kw)
        bad.bits = torch.zeros(7, dtype=torch.int32, device="cuda")
        with pytest.raises(RuntimeError, match="int32"):
            nb.render_image(16, 16, 20.0, torch.eye(4), mc, mf, opts, grid=bad, **kw)
        # 8x256 with L_dir 6: 39 direction channels, wider than the wgmma forward's 32
        ldir6 = [nb.FlexibleNeRFModel(num_layers=8, hidden_size=256, num_encoding_fn_xyz=10, num_encoding_fn_dir=6).cuda()
                 for _ in range(2)]
        kw6 = dict(encode_position_fn=epf, encode_direction_fn=nb.get_embedding_function(6))
        for impl in (None, ops.IMPL_TC, ops.IMPL_TC_FAST):
            with pytest.raises(NotImplementedError, match="32"):
                nb.predict_and_render_radiance(rays, *ldir6, opts, grid=grid, impl=impl, **kw6)
    assert ops.launch_count() == before
    with torch.no_grad(), pytest.raises(NotImplementedError, match="32"):  # after generating the image's rays
        nb.render_image(16, 16, 20.0, torch.eye(4), *ldir6, opts, grid=grid, **kw6)


# ------------------------------------------------------------------------------------------------------------------------
# 7. PSNR of model-built grids against the default render
# ------------------------------------------------------------------------------------------------------------------------
# grid render (from_models, 128^3) against the default render, dB, deterministic sampling.  Each bar is 3 dB under the
# lowest figure tools/grid_render_time.py measured on an H100 80GB HBM3 (700 W) over impl 1 / 3 and lego 400^2 / 800^2,
# fern 378 x 504 (first bracket); this test's smaller renders measured the second bracket (inf: identical images).
PSNR_BARS = {
    ("lego", "rgb_fine"): 71.9,    # [74.93; inf]
    ("lego", "rgb_coarse"): 65.0,  # [68.03; inf]
    ("fern", "rgb_fine"): 75.3,    # [78.39; 93.88]
    ("fern", "rgb_coarse"): 75.2,  # [78.24; inf]
}


@pytest.mark.parametrize("scene", ["lego", "fern"])
@pytest.mark.parametrize("impl", list(IMPLS))
def test_model_grid_render_psnr_against_default(impl, scene):
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    _, _, _, _, models, enc = _setup(scene)
    grid = OccupancyGrid.from_models(models, enc[0], SCENES[scene][-1], 128, encode_direction_fn=enc[1])
    report("occupied fraction", (scene,), grid.occupied_fraction)
    ref = _image(scene, IMPLS[impl], 4096, perturb=False, noise=0.0)
    got = _image(scene, IMPLS[impl], 4096, grid, perturb=False, noise=0.0)
    for out in ("rgb_fine", "rgb_coarse"):
        i = OUT_NAMES.index(out)
        p = psnr64(got[i], ref[i])
        report(f"PSNR dB grid vs default {out}", (impl, scene), p)
        assert p >= PSNR_BARS[(scene, out)], (impl, scene, out, p)
