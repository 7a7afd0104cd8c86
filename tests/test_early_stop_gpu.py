"""GPU: early ray termination in inference renders (ops.render_fwd_early_stop, render_image(early_stop=...)).
  1. t = 0 gives render_fwd's (no grid) and render_fwd_grid's outputs and n_evaluated bit for bit;
  2. per ray at t in {1e-4, 1e-2, 0.1}: evaluated raw is the default raw, the rest of the grid's samples from stop_sample
     on are [0 0 0 -inf], stop_sample is on a round boundary, the fp64 transmittance of the default raw is below t at the
     stop and not below it at every earlier boundary, unstopped rays and the coarse pass are bit-identical;
     1 and 2 also at the sample counts where the rounds change shape (COUNTS);
  3. the guarantee's output bounds, with their signs;
  4. determinism and chunking invariance;
  5. the shipped lego and fern weights at t = 1e-3, with and without a model-built grid;
  6. the refusals, before any launch.
Run with -s to print the measured figures."""
import math

import pytest
import torch

import mlp_checks as M
from helpers import OUT_NAMES, bits_equal, psnr64, scene_pose, transmittance64, ws_view
from mlp_checks import T_REL

pytestmark = pytest.mark.gpu

# (shipped weights or None, H, W, focal, pose, no_ndc, near, far, L_xyz, (coarse, fine) networks, bounds of a grid):
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
SKIP = torch.tensor([0.0, 0.0, 0.0, -math.inf])
# fp32 rounding allowance of the outputs (figures printed under -s; T_REL, the transmittance's, is mlp_checks').
# Measured on an H100 80GB HBM3 over every case below, no output moved against the guarantee's sign by more than 1.2e-7
OUT_ABS = 2e-6


def report(what, ctx, value):
    print(f"[early_stop] {what} {ctx}: {value}")


def _setup(scene, variant="det", n_fine=128, n_coarse=64):
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


def _grid(scene, kind, models=None, encoders=None):
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    bounds = SCENES[scene][-1]
    if kind is None:
        return None
    if kind == "full":
        return OccupancyGrid.full(bounds, 32)
    if kind == "model":
        return OccupancyGrid.from_models(models, encoders[0], bounds, 128, encode_direction_fn=encoders[1])
    g = torch.Generator(device="cuda").manual_seed(11)
    return OccupancyGrid.from_occupancy(bounds, torch.rand(32, 32, 32, generator=g, device="cuda") < 0.5)


def _reference(arch, arch_f, blobs, opts, rays, rng, grid, impl):
    """(out_c, out_f, workspace, n_evaluated) of the render early_stop is measured against."""
    from nerf_pytorch_b200 import ops

    if grid is None:
        oc, of, ws = ops.render_fwd(arch, arch_f, opts, blobs[0], blobs[1], rays, rng, training=False, impl=impl)
        return oc, of, ws, None
    ne = torch.zeros(2, dtype=torch.int64, device="cuda")
    oc, of, ws = ops.render_fwd_grid(arch, arch_f, opts, blobs[0], blobs[1], rays, rng, grid, impl=impl, n_evaluated=ne)
    return oc, of, ws, ne


# ------------------------------------------------------------------------------------------------------------------------
# 1. t = 0 is today's path
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid_kind", [None, "rand50", "full"])
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("impl", list(IMPLS))
def test_zero_threshold_is_the_default_render_bit_for_bit(impl, variant, grid_kind):
    _zero_threshold_is_the_default_render_bit_for_bit(impl, "lego", variant, grid_kind)


@pytest.mark.parametrize("grid_kind", [None, "rand50", "full"])
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("scene", H256)
@pytest.mark.parametrize("impl", list(IMPLS))
def test_zero_threshold_is_the_default_render_bit_for_bit_at_hidden_256(impl, scene, variant, grid_kind):
    _zero_threshold_is_the_default_render_bit_for_bit(impl, scene, variant, grid_kind)


def _zero_threshold_is_the_default_render_bit_for_bit(impl, scene, variant, grid_kind, nc=64, nf=128):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    ctx = (impl, scene, variant, grid_kind, nc, nf)
    (arch, arch_f), blobs, opts, rays, _, _ = _setup(scene, variant, nf, nc)
    grid = _grid(scene, grid_kind)
    rng = nb.SeededRandoms(5, 2)
    n = rays.shape[0]
    if nf:
        oc, of, _, ne_ref = _reference(arch, arch_f, blobs, opts, rays, rng, grid, IMPLS[impl])
        ec, ef, ne, stop = ops.render_fwd_early_stop(arch, arch_f, opts, blobs[0], blobs[1], rays, rng, grid, 0.0,
                                                     impl=IMPLS[impl], want_stop=True)
        assert bits_equal(ec, oc) and bits_equal(ef, of), ctx
        assert (stop == nc + nf).all(), ctx
        assert ne.tolist() == ([n * nc, n * (nc + nf)] if grid is None else ne_ref.tolist()), ctx

    # a coarse-only network: its one pass is the last
    perturb, noise, white = VARIANTS[variant]
    opts0 = ops.make_opts(nc, 0, perturb, False, white, noise)
    oc, _, _, ne_ref = _reference(arch, None, blobs, opts0, rays, rng, grid, IMPLS[impl])
    ec, ef, ne, stop = ops.render_fwd_early_stop(arch, None, opts0, blobs[0], None, rays, rng, grid, 0.0,
                                                 impl=IMPLS[impl], want_stop=True)
    assert ef is None and bits_equal(ec, oc), ctx
    assert (stop == nc).all(), ctx
    assert ne.tolist() == ([n * nc, 0] if grid is None else ne_ref.tolist()), ctx


# ------------------------------------------------------------------------------------------------------------------------
# 2, 3. per ray, and the output bounds
# ------------------------------------------------------------------------------------------------------------------------
_CACHE = {}


def _stopped_render(impl, scene, variant, grid_kind, t, nc=64, nf=128):
    """The default render and the early-stopping one; raw and z of the last pass (the fine pass, or the coarse pass
    when nf is 0) read from both workspaces."""
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    key = (impl, scene, variant, grid_kind, t, nc, nf)
    if key in _CACHE:
        return _CACHE[key]
    _CACHE.clear()
    archs, blobs, opts, rays, models, enc = _setup(scene, variant, nf, nc)
    if not nf:
        archs = (archs[0], None)
        blobs = [blobs[0], None]
    grid = _grid(scene, grid_kind, models, enc)
    rng = nb.SeededRandoms(9, 4)
    oc, of, ws, _ = _reference(*archs, blobs, opts, rays, rng, grid, IMPLS[impl])
    ec, ef, ne, stop = ops.render_fwd_early_stop(*archs, opts, blobs[0], blobs[1], rays, rng, grid, t,
                                                 impl=IMPLS[impl], want_stop=True)
    n, S, last = rays.shape[0], nc + nf, "fine" if nf else "coarse"
    lay = ops.render_workspace_layout(*archs, opts, n, False)
    es_ws = torch.empty(ops.render_early_stop_workspace_bytes(*archs, opts, n), dtype=torch.uint8, device="cuda")
    ops.render_fwd_early_stop(*archs, opts, blobs[0], blobs[1], rays, rng, grid, t, impl=IMPLS[impl],
                              workspace=es_ws)
    torch.cuda.synchronize()
    out = dict(opts=opts, rays=rays, rng=rng, ref=(oc, of), es=(ec, ef), ne=ne, stop=stop.long(), last=last,
               raw=ws_view(ws, lay, f"raw_{last}", n, S, 4), z=ws_view(ws, lay, f"z_{last}", n, S, 1),
               es_raw=ws_view(es_ws, lay, f"raw_{last}", n, S, 4), es_z=ws_view(es_ws, lay, f"z_{last}", n, S, 1))
    _CACHE[key] = out
    return out


PER_RAY = [(impl, scene, variant, grid_kind, t)
           for impl in IMPLS for t in (1e-4, 1e-2, 0.1)
           for scene, variant, grid_kind in (("lego", "det", None), ("lego", "perturb_noise", "rand50"),
                                             ("lego", "white_perturb", None), ("fern", "det", "model"),
                                             ("a2", "det", None), ("a2", "perturb_noise", "rand50"),
                                             ("a2", "white_perturb", "model"), ("mixed", "det", "rand50"),
                                             ("mixed_rev", "perturb_noise", None))]


@pytest.mark.parametrize("impl,scene,variant,grid_kind,t", PER_RAY)
def test_per_ray_contract(impl, scene, variant, grid_kind, t):
    _per_ray_contract(impl, scene, variant, grid_kind, t)


def _per_ray_contract(impl, scene, variant, grid_kind, t, nc=64, nf=128):
    from nerf_pytorch_b200 import ops

    r = _stopped_render(impl, scene, variant, grid_kind, t, nc, nf)
    ctx = (impl, scene, variant, grid_kind, t, nc, nf)
    K = ops.stop_round()
    raw, z, es_raw, stop = r["raw"], r["z"], r["es_raw"], r["stop"]
    n, S = z.shape
    i_last = 1 if nf else 0
    if nf:
        assert bits_equal(r["es"][0], r["ref"][0]), ctx  # the coarse pass and so the fine depths are untouched
    assert bits_equal(r["es_z"], z), ctx
    keep = raw[..., 3] != -math.inf  # the samples the grid keeps (all of them without a grid)
    j = torch.arange(S, device="cuda")[None, :]
    before = j < stop[:, None]
    want = torch.where((before | ~keep)[..., None], raw, SKIP.cuda().expand(n, S, 4))
    assert bits_equal(es_raw, want), ctx
    stopped = stop < S
    report("stopped rays / all", ctx, f"{int(stopped.sum())} / {n}")
    if scene == "a2" and t >= 1e-2 and S > K:
        assert stopped.any(), ctx  # the scaled weights turn rays opaque: the contract is not vacuous
    if S <= K:
        assert not stopped.any(), ctx  # one round: no ray has samples left after it
    assert (r["ne"][i_last] == (keep & before).sum()).item(), ctx
    assert bits_equal(r["es"][i_last][~stopped], r["ref"][i_last][~stopped]), ctx

    # round boundaries: the rank (1-based) of each kept sample among its ray's kept samples
    rank = torch.cumsum(keep.long(), 1)
    n_keep = rank[:, -1]
    ran = (keep & before).sum(1)
    assert ((ran[stopped] % K) == 0).all() and (ran[stopped] > 0).all() and (ran[stopped] < n_keep[stopped]).all(), ctx
    last_ran = torch.where(keep & before, j, -1).max(1).values
    assert (stop[stopped] == last_ran[stopped] + 1).all(), ctx

    noise = ops.random_fill(r["rng"], f"noise_{r['last'][0]}", n, S) if r["opts"].noise_std > 0 else None
    T = transmittance64(raw, z, r["rays"], noise, r["opts"].noise_std)
    # at the stop T < t; at every earlier boundary with samples left (and every boundary of an unstopped ray) T >= t
    if stopped.any():
        at_stop = T[stopped, stop[stopped]]
        report("max T64 / t at the stop", ctx, (at_stop / t).max().item())
        assert (at_stop < t * (1 + T_REL)).all(), ctx
    boundary = keep & (rank % K == 0) & (rank < n_keep[:, None]) & (j < stop[:, None] - 1)
    rows, cols = boundary.nonzero(as_tuple=True)
    if rows.numel():
        earlier = T[rows, cols + 1]
        report("min T64 / t at earlier boundaries", ctx, (earlier / t).min().item())
        assert (earlier >= t * (1 - T_REL)).all(), ctx


@pytest.mark.parametrize("impl,scene,variant,grid_kind,t", PER_RAY)
def test_output_bounds(impl, scene, variant, grid_kind, t):
    r = _stopped_render(impl, scene, variant, grid_kind, t)
    ctx = (impl, scene, variant, grid_kind, t)
    stopped = r["stop"] < r["z"].shape[1]
    o, e = r["ref"][1][stopped].double(), r["es"][1][stopped].double()
    if not stopped.any():
        return
    white = VARIANTS[variant][2]
    zmax = r["z"].max().item()
    d_rgb = (e[:, :3] - o[:, :3]) if white else (o[:, :3] - e[:, :3])
    d_acc, d_depth = o[:, 4] - e[:, 4], o[:, 5] - e[:, 5]
    report("rgb, acc, depth / zmax moves (min, max)", ctx,
           [(d.min().item(), d.max().item()) for d in (d_rgb, d_acc, d_depth / zmax)])
    assert (d_rgb >= -OUT_ABS).all() and (d_rgb <= t + OUT_ABS).all(), ctx
    assert (d_acc >= -OUT_ABS).all() and (d_acc <= t + OUT_ABS).all(), ctx
    assert (d_depth >= -OUT_ABS * zmax).all() and (d_depth <= (t + OUT_ABS) * zmax).all(), ctx
    # disp = 1 / (depth / acc) where acc is clear of 0: depth / acc moves by at most 2 t zmax / (acc - t)
    clear = o[:, 4] > 0.5
    if clear.any():
        ro, re = 1.0 / o[clear, 3], 1.0 / e[clear, 3]
        bound = 2 * t * zmax / (o[clear, 4] - t) + OUT_ABS * zmax
        assert ((ro - re).abs() <= bound).all(), ctx


# (n_coarse, n_fine) where the last pass's rounds of K = 32 change shape: one partial round (15 samples), a last round of
# one sample (33), exactly one round (15 + 17) and 32 rounds (15 + 1009).  With a grid, each compaction group of 10 rays
# holds 10 S rows, which no count here makes a multiple of the 64-row blocks.
COUNTS = [(15, 0), (33, 0), (15, 17), (15, 1009)]
COUNT_IDS = [f"{nc}+{nf}" for nc, nf in COUNTS]


@pytest.mark.parametrize("counts", COUNTS, ids=COUNT_IDS)
@pytest.mark.parametrize("grid_kind", [None, "rand50"])
@pytest.mark.parametrize("impl", list(IMPLS))
def test_zero_threshold_is_the_default_render_bit_for_bit_at_boundary_counts(impl, grid_kind, counts):
    _zero_threshold_is_the_default_render_bit_for_bit(impl, "lego", "perturb_noise", grid_kind, *counts)


@pytest.mark.parametrize("counts", COUNTS, ids=COUNT_IDS)
@pytest.mark.parametrize("scene,variant,grid_kind", [("a2", "perturb_noise", "rand50"), ("lego", "det", None)])
@pytest.mark.parametrize("impl", list(IMPLS))
def test_per_ray_contract_at_boundary_counts(impl, scene, variant, grid_kind, counts):
    _per_ray_contract(impl, scene, variant, grid_kind, 1e-2, *counts)


# ------------------------------------------------------------------------------------------------------------------------
# 4. determinism and chunking
# ------------------------------------------------------------------------------------------------------------------------
def _image(scene, impl, chunk, grid=None, randoms=None, early_stop=None, perturb=True, noise=0.5):
    import nerf_pytorch_b200 as nb
    from oracle import nerf_oracle as O

    _, H, W, focal, pose, no_ndc, near, far, l_xyz, *_ = SCENES[scene]
    mc, mf = M.scene_models(SCENES[scene])
    opts = O.make_options(no_ndc=no_ndc, near=near, far=far, num_coarse=64, num_fine=128, perturb=perturb,
                          radiance_field_noise_std=noise)
    return nb.render_image(H, W, focal, scene_pose(pose), mc, mf, opts, mode="validation",
                           encode_position_fn=nb.get_embedding_function(l_xyz),
                           encode_direction_fn=nb.get_embedding_function(4), rays_per_chunk=chunk, impl=impl,
                           randoms=randoms, grid=grid, early_stop=early_stop)


@pytest.mark.parametrize("grid_kind", [None, "rand50"])
@pytest.mark.parametrize("impl", list(IMPLS))
def test_render_image_is_deterministic_and_chunking_invariant(impl, grid_kind):
    _render_image_is_deterministic_and_chunking_invariant(impl, "lego", grid_kind)


@pytest.mark.parametrize("grid_kind", [None, "rand50"])
@pytest.mark.parametrize("scene", H256)
@pytest.mark.parametrize("impl", list(IMPLS))
def test_render_image_is_deterministic_and_chunking_invariant_at_hidden_256(impl, scene, grid_kind):
    _render_image_is_deterministic_and_chunking_invariant(impl, scene, grid_kind)


def _render_image_is_deterministic_and_chunking_invariant(impl, scene, grid_kind):
    import nerf_pytorch_b200 as nb

    grid = _grid(scene, grid_kind)
    rng = nb.SeededRandoms(21, 1)
    n = SCENES[scene][1] * SCENES[scene][2]
    whole = _image(scene, IMPLS[impl], n, grid, rng, 1e-2)
    again = _image(scene, IMPLS[impl], n, grid, rng, 1e-2)
    assert all(bits_equal(a, b) for a, b in zip(whole, again))
    for chunk in (1000, 333):
        part = _image(scene, IMPLS[impl], chunk, grid, rng, 1e-2)
        assert all(bits_equal(a, b) for a, b in zip(whole, part)), (scene, chunk)
    default = _image(scene, IMPLS[impl], n, grid, rng)
    assert not all(bits_equal(a, b) for a, b in zip(whole, default))  # some ray did stop
    assert bits_equal(whole[0], default[0])  # the coarse pass never stops


# ------------------------------------------------------------------------------------------------------------------------
# 5. shipped weights
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid_kind", [None, "model"])
@pytest.mark.parametrize("scene", ["lego", "fern"])
@pytest.mark.parametrize("impl", list(IMPLS))
def test_shipped_weights(impl, scene, grid_kind):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    (arch, _), blobs, opts, rays, models, enc = _setup(scene)
    grid = _grid(scene, grid_kind, models, enc)
    rng = nb.SeededRandoms(3, 0)
    full = _grid(scene, "full")
    ne_ref = torch.zeros(2, dtype=torch.int64, device="cuda")
    oc, of, _ = ops.render_fwd_grid(arch, arch, opts, blobs[0], blobs[1], rays, rng, grid if grid is not None else full,
                                    impl=IMPLS[impl], n_evaluated=ne_ref)
    ec, ef, ne, stop = ops.render_fwd_early_stop(arch, arch, opts, blobs[0], blobs[1], rays, rng, grid, 1e-3,
                                                 impl=IMPLS[impl], want_stop=True)
    ctx = (impl, scene, grid_kind)
    n = rays.shape[0]
    stopped = int((stop < 192).sum())
    p = psnr64(ef[:, :3], of[:, :3])
    report("stopped rays, fine rows early_stop / grid-only, PSNR dB", ctx,
           (f"{stopped} / {n}", f"{ne[1].item()} / {ne_ref[1].item()}", p))
    assert stopped > 0, ctx
    assert ne[1].item() < ne_ref[1].item(), ctx
    assert ne[0].item() == ne_ref[0].item() and bits_equal(ec, oc), ctx
    assert p >= 60.0, ctx


# ------------------------------------------------------------------------------------------------------------------------
# 6. refusals
# ------------------------------------------------------------------------------------------------------------------------
def test_early_stop_refusals_fire_before_any_launch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    (arch, _), blobs, opts, rays, (mc, mf), (epf, edf) = _setup("lego")
    kw = dict(encode_position_fn=epf, encode_direction_fn=edf)
    o = O.make_options(num_coarse=64, num_fine=64)
    with torch.no_grad():  # pack both models once, so that nothing below is a first use
        nb.predict_and_render_radiance(rays, mc, mf, o, early_stop=1e-3, **kw)
    grid = _grid("lego", "full")
    torch.cuda.synchronize()
    before = ops.launch_count()
    ro = torch.randn(64, 3, device="cuda")
    with pytest.raises(NotImplementedError, match="inference"):
        nb.predict_and_render_radiance(rays, mc, mf, o, early_stop=1e-3, **kw)
    with pytest.raises(NotImplementedError, match="inference"):
        nb.run_one_iter_of_nerf(16, 16, 20.0, mc, mf, ro, -ro, o, early_stop=1e-3, **kw)
    with pytest.raises(NotImplementedError, match="inference"):
        nb.run_one_iter_of_nerf_from_pose(16, 16, 20.0, mc, mf, torch.eye(4), None, o, early_stop=1e-3, **kw)
    with torch.no_grad():
        for bad in (1.0, -1e-3, float("nan"), "0.1", True):
            with pytest.raises(ValueError, match="early_stop"):
                nb.predict_and_render_radiance(rays, mc, mf, o, early_stop=bad, **kw)
        with pytest.raises(ValueError, match="early_stop"):
            nb.render_image(16, 16, 20.0, torch.eye(4), mc, mf, o, early_stop=2.0, **kw)
        for g in (None, grid):
            with pytest.raises(NotImplementedError, match="impl 0"):
                nb.predict_and_render_radiance(rays, mc, mf, o, grid=g, early_stop=0.1, impl=ops.IMPL_SIMT, **kw)
        few = O.make_options(num_coarse=14, num_fine=0)
        with pytest.raises(NotImplementedError, match="fewer than 15 samples"):
            nb.predict_and_render_radiance(rays, mc, None, few, early_stop=0.1, impl=ops.IMPL_TC, **kw)
        # the library's own refusals
        for t in (1.0, -0.5, float("nan")):
            with pytest.raises(RuntimeError, match="stop_transmittance"):
                ops.render_fwd_early_stop(arch, arch, opts, blobs[0], blobs[1], rays, {}, None, t)
        with pytest.raises(NotImplementedError, match="impl=0"):
            ops.render_fwd_early_stop(arch, arch, opts, blobs[0], blobs[1], rays, {}, grid, 0.1, impl=ops.IMPL_SIMT)
        # 8x256 with L_dir 6: 39 direction channels, wider than the wgmma forward's 32
        ldir6 = [nb.FlexibleNeRFModel(num_layers=8, hidden_size=256, num_encoding_fn_xyz=10, num_encoding_fn_dir=6).cuda()
                 for _ in range(2)]
        kw6 = dict(encode_position_fn=epf, encode_direction_fn=nb.get_embedding_function(6))
        for g in (None, grid):
            for impl in (None, ops.IMPL_TC, ops.IMPL_TC_FAST):
                with pytest.raises(NotImplementedError, match="32"):
                    nb.predict_and_render_radiance(rays, *ldir6, o, grid=g, early_stop=0.1, impl=impl, **kw6)
        a6 = ops.ArchSpec(num_layers=8, hidden=256, n_freq_xyz=10, n_freq_dir=6)
        blob6 = torch.zeros(a6.blob_floats(), device="cuda")
        for impl in (ops.IMPL_TC, ops.IMPL_TC_FAST):
            with pytest.raises(NotImplementedError, match="32"):
                ops.render_fwd_early_stop(a6, a6, opts, blob6, blob6, rays, {}, None, 0.1, impl=impl)
    assert ops.launch_count() == before
    with torch.no_grad(), pytest.raises(NotImplementedError, match="32"):  # after generating the image's rays
        nb.render_image(16, 16, 20.0, torch.eye(4), *ldir6, o, early_stop=0.1, **kw6)
