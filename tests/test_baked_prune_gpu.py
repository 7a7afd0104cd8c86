"""GPU: pruning baked fields (csrc/baked.cu baked_max_weight_kernel; nb.baked_brick_weights_rays, nb.baked_brick_weights,
nb.baked_transparent_bricks, nb.prune_baked, BakedFieldTrainer.prune; include/nerfb200.h "baked fields: pruning").

  1. peak weights against the per-brick amax of fp64 per-sample weights, each the difference of helpers.baked_render64's
     acc between copies of a ray cut just after the sample and just before it, its brick read from the colour of a
     probe field whose slots carry distinct colours: lego A0 at 256^3 over the grid of both networks, fern in NDC, and
     synthetic fields (rays along brick faces and through brick corners, a res that is not a multiple of 8, inactive
     bricks, rays that miss the box, axis-parallel rays, no view directions);
  2. exactness: on rays holding one sample inside the box each brick's peak is, bit for bit, the largest acc
     baked_render returns over the rays whose sample lies in it;
  3. determinism: one call, chunks of several sizes, a permuted ray order and a second run give the same bits;
  4. dropping transparent bricks leaves every render the same bits (all 8 output columns, NaNs as bits), with and
     without a white background and early stopping, from poses used nowhere else;
  5. dropping bricks with peak 0 leaves the measuring views' renders the same bits; tau = 1e-2 keeps held-out PSNR;
  6. a pruned field saves and loads, its tied gradient matches fp64 autograd, and trainer steps keep copies bit-equal;
  7. BakedFieldTrainer.prune keeps the kept rows of values, m and v and the step counter, shrinks the buffers, trains on,
     and prune-transparent-then-train reaches the held-out PSNR of train-unpruned.

Measured on an H100 80GB HBM3 at 700 W: the file runs in about 10 s; device memory allocated peaks at 8.3 GiB (the fp64
oracle over the cut lego rays)."""
import math

import pytest
import torch

from helpers import (LEGO_CAM, baked_render64, bake_scene, bits_equal, camera_rays, copies_bit_equal,
                     edge_rays, heldout_psnr, lattice_index, random_rays, ray_rows, scene_options, sphere_poses,
                     synthetic_field, targets)

pytestmark = pytest.mark.gpu

# peak weights against the fp64 oracle, absolute (weights lie in [0, 1]).  A weight is alpha times T, T a product of the
# ray's earlier q (fp32, up to ~900 factors for lego at 256^3), so its error grows with the samples before it: up to about
# n 2^-24 relative in the worst case, n = 900 giving 5.4e-5.  Measured on an H100 80GB HBM3 at 700 W: 4.5e-6 on the
# lego rays below (1.1e-5 over all 2304 rays of that view), at most 6.4e-7 on fern and the synthetic fields (tens to a
# hundred samples per ray)
PEAK_ABS = 3e-5
# the tied gradient of a pruned field against the fp64 sum over copies (test_baked_grad_gpu's bars)
SYN_REL = 1e-5
SAT_REL = 1e-4


def report(what, ctx, value):
    print(f"[baked-prune] {what} {ctx}: {value}")


_CACHE = {}


def _bake(kind, res, grid_res=None):
    """A fresh copy of helpers.bake_scene over the grid of both networks, each bake made once per file."""
    import nerf_pytorch_b200 as nb

    key = (kind, res, grid_res)
    if key not in _CACHE:
        _CACHE[key] = bake_scene(kind, res, grid_res, grid_from="both")
    f = _CACHE[key]
    return nb.BakedField(f.bounds, f.resolution, f.brick_map.clone(), f.bricks.clone(), f.values.clone(),
                         f.use_viewdirs)


Y0 = 0.28209479177387814


def _probe(field):
    """The field's bricks with sigma_raw 0.1 at every point and, in slot s, the red logit L_s = 8 (s + 1/2) / n - 4
    (green and blue 0): every sample in an active brick has alpha > 0, and its colour names its slot."""
    import nerf_pytorch_b200 as nb

    n = field.n_active
    v = torch.zeros_like(field.values)
    v[..., 0] = 0.1
    L = 8.0 * (torch.arange(n, device="cuda", dtype=torch.float64) + 0.5) / n - 4.0
    v[..., 1] = (L / Y0).float()[:, None]
    return nb.BakedField(field.bounds, field.resolution, field.brick_map, field.bricks, v, field.use_viewdirs)


def _slot_of(field, red, acc):
    """The slot a probe sample's colour red / acc names, -1 where acc is ~0 (no sample in an active brick; a probe
    sample there has weight >= 1e-4: alpha = 1 - exp(-0.1 delta) with delta half a cube, T >= 0.5 over these rays)."""
    hit = acc > 1e-9
    c = red / torch.where(hit, acc, 1.0)
    s = torch.floor((torch.log(c / (1.0 - c)) + 4.0) * field.n_active / 8.0)
    s = torch.where(hit, s, -1.0)
    assert bool(((s >= -1) & (s < field.n_active)).all())
    return s.long()


def _cut_rays(field, rays):
    """The rays with near moved a quarter step past the box's entry (an fp64 estimate of the slab interval, far from
    the fp32 one), so that a ray's interval starts at its near and sample k lies at t_k = near + (k + 1/2) dt; rays
    that miss the box are made empty.  Returns (rays, dt (fp32, the header's step), K (samples per ray, at most))."""
    lo = torch.tensor(field.bounds[0], dtype=torch.float64, device="cuda")
    hi = torch.tensor(field.bounds[1], dtype=torch.float64, device="cuda")
    o, d = rays[:, :3].double(), rays[:, 3:6].double()
    flat = d == 0
    inside = (o >= lo) & (o < hi)
    t0, t1 = (lo - o) / torch.where(flat, 1.0, d), (hi - o) / torch.where(flat, 1.0, d)
    entry = torch.where(flat, torch.where(inside, -math.inf, math.inf), torch.minimum(t0, t1)).amax(-1)
    exit_ = torch.where(flat, torch.where(inside, math.inf, -math.inf), torch.maximum(t0, t1)).amin(-1)
    h = ((torch.tensor(field.bounds[1], device="cuda") - torch.tensor(field.bounds[0], device="cuda"))
         / torch.tensor(field.resolution, device="cuda", dtype=torch.float32)).min()
    d32 = rays[:, 3:6]
    dt = (0.5 * h) / torch.sqrt((d32[:, 0] * d32[:, 0] + d32[:, 1] * d32[:, 1]) + d32[:, 2] * d32[:, 2])
    a = torch.maximum(rays[:, 6].double(), entry + 0.25 * dt.double())
    b = torch.minimum(rays[:, 7].double(), exit_)
    hits = a < b
    out = rays.clone()
    out[:, 6] = torch.where(hits, a.float(), rays[:, 6])
    out[:, 7] = torch.where(hits, rays[:, 7], out[:, 6])  # a ray that misses (or grazes) the box: far = near, empty
    K = int(torch.where(hits, torch.ceil((b - a) / dt.double()), 0.0).max().item()) + 1
    return out, dt, K


def _per_sample64(field, rays, max_samples=1 << 22):
    """fp64 weight and brick slot (-1 for a miss) of every sample k < K of ``rays`` (cut by _cut_rays), from
    helpers.baked_render64 alone: w_k is the difference of its acc between copies of the ray cut just after sample k
    (far = near + (k + 1) dt in fp32, between t_k and t_(k+1)) and just after sample k - 1, and the slot is read from
    the same difference of the probe field's render."""
    rays, dt, K = _cut_rays(field, rays)
    n = rays.shape[0]
    k = torch.arange(K, device="cuda", dtype=torch.float32)
    cut = rays[:, None].expand(n, K, rays.shape[1]).clone()
    cut[..., 7] = torch.minimum(rays[:, 7:8], rays[:, 6:7] + (k[None] + 1.0) * dt[:, None])
    cut = cut.reshape(n * K, -1)
    probe = _probe(field)
    acc, red, pacc = [], [], []
    step = max(1, max_samples // K)
    for s in range(0, cut.shape[0], step):
        c = cut[s:s + step].contiguous()
        acc.append(baked_render64(field, c, False)[1])
        rgb, a, *_ = baked_render64(probe, c, False)
        red.append(rgb[:, 0])
        pacc.append(a)
    diff = lambda x: torch.diff(torch.cat(x).view(n, K), dim=1, prepend=torch.zeros(n, 1, dtype=torch.float64,
                                                                                   device="cuda"))
    return rays, diff(acc), _slot_of(field, diff(red), diff(pacc))


def _oracle_peaks(field, rays):
    """The cut rays and the fp64 per-brick amax of their per-sample weights."""
    rays, w, slot = _per_sample64(field, rays)
    hit = slot >= 0
    assert bool((w[~hit].abs() <= 1e-12).all())  # a sample outside the active bricks has weight 0
    peaks = torch.zeros(field.n_active, dtype=torch.float64, device="cuda")
    peaks.scatter_reduce_(0, slot[hit], w[hit], reduce="amax")
    return rays, peaks


def _peak_check(field, rays, ctx):
    import nerf_pytorch_b200 as nb

    rays, want = _oracle_peaks(field, rays)
    got = nb.baked_brick_weights_rays(field, rays)
    err = (got.double() - want).abs().max().item()
    report("peak weight error (abs), bricks seen / active", ctx, (err, int((want > 0).sum()), field.n_active))
    assert torch.isfinite(got).all() and (got >= 0).all()
    assert (want > 0).any() and err <= PEAK_ABS, (ctx, err)
    return got


def _out_bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _render_rows(field, rays, white, stop):
    from nerf_pytorch_b200 import ops

    vals = field.values if field.n_active else field.values.new_zeros(1, 729, 32)
    return ops.baked_render(field.box(), field.brick_map, vals, field.use_viewdirs, rays, white, stop)


# ------------------------------------------------------------------------------------------------------------------------
# 1. peak weights against fp64
# ------------------------------------------------------------------------------------------------------------------------
def test_peak_weights_match_fp64_on_lego_both_network_grid():
    f = _bake("lego", 256, grid_res=128)
    rays = camera_rays("lego")[::23].contiguous()  # 101 rays of up to ~900 samples each
    rays[::11, 3:6] = -rays[::11, 3:6]  # rays that miss the box
    _peak_check(f, rays, "lego 256^3 both grids")


def test_peak_weights_match_fp64_on_fern_ndc():
    f = _bake("fern", (40, 36, 44), grid_res=32)
    _peak_check(f, camera_rays("fern")[::3].contiguous(), "fern ndc")


@pytest.mark.parametrize("case", ["edges", "res13", "inactive", "noview_inactive", "opaque"])
def test_peak_weights_match_fp64_on_synthetic_fields(case):
    if case == "edges":
        f = synthetic_field((24, 24, 24), seed=2)
    elif case == "res13":
        f = synthetic_field((13, 9, 17), seed=3)
    elif case == "inactive":
        f = synthetic_field((20, 17, 33), active=0.5, seed=4)
    elif case == "noview_inactive":
        f = synthetic_field((20, 17, 12), viewdirs=False, active=0.5, seed=5)
    else:
        f = synthetic_field((16, 16, 16), sigma=(8.0, 48.0), seed=1)
    rays = torch.cat([random_rays(1024, 10, f.use_viewdirs, misses=True), edge_rays(f, f.use_viewdirs)])
    _peak_check(f, rays, case)


# ------------------------------------------------------------------------------------------------------------------------
# 2. exactness on one-sample rays, 3. determinism
# ------------------------------------------------------------------------------------------------------------------------
def _one_sample_rays(field, n, seed):
    """Rays whose [near, far] holds exactly one sample, at a random point inside the box: near = 1 - dt / 2 and
    far = near + dt with dt the kernel's step (fp32), so t_0 = near + dt / 2 < far <= near + 3 dt / 2 = t_1."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    lo = torch.tensor(field.bounds[0], device="cuda")
    hi = torch.tensor(field.bounds[1], device="cuda")
    o = torch.randn(n, 3, generator=g, device="cuda")
    o = 3.0 * o / o.norm(dim=1, keepdim=True)
    p = lo + 0.02 * (hi - lo) + 0.96 * (hi - lo) * torch.rand(n, 3, generator=g, device="cuda")
    d = p - o
    res = torch.tensor(field.resolution, device="cuda", dtype=torch.float32)
    h = ((hi - lo) / res).min()
    dn = torch.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    dt = (0.5 * h) / dn
    near = 1.0 - 0.5 * dt
    return ray_rows(o, d, field.use_viewdirs, near, near + dt)


@pytest.mark.parametrize("kind", ["synthetic", "lego"])
def test_peak_is_the_largest_single_sample_acc_bit_for_bit(kind):
    import nerf_pytorch_b200 as nb

    f = synthetic_field((24, 24, 24), active=0.7, sigma=(-2.0, 6.0), seed=21) if kind == "synthetic" \
        else _bake("lego", (24, 20, 28), grid_res=32)
    rays = _one_sample_rays(f, 200_000, 22)
    rgb, pacc, *_ = baked_render64(_probe(f), rays, False)  # one sample: its colour names its slot
    s = _slot_of(f, rgb[:, 0], pacc)  # the ray's brick slot, -1 when its sample misses
    acc = _render_rows(f, rays, False, 0.0)[:, 4]
    assert bool((acc[s < 0] == 0).all())
    want = torch.zeros(f.n_active, dtype=torch.float32, device="cuda")
    want.scatter_reduce_(0, s[s >= 0], acc[s >= 0], reduce="amax")
    got = nb.baked_brick_weights_rays(f, rays)
    report("one-sample rays: bricks seen / active", kind, (int((got > 0).sum()), f.n_active))
    assert int((got > 0).sum()) >= (10 if kind == "lego" else f.n_active)  # lego: most of its bricks are empty
    assert bits_equal(got, want)


def test_peaks_are_the_same_bits_for_every_chunking_order_and_run():
    import nerf_pytorch_b200 as nb

    f = _bake("lego", (40, 36, 44), grid_res=32)
    rays = torch.cat([camera_rays("lego", p) for p in sphere_poses(6, offset=3.0)])
    one = nb.baked_brick_weights_rays(f, rays)
    assert int((one > 0).sum()) > 0
    for chunk in (997, 4096, 5000, rays.shape[0] - 1):
        out = torch.zeros(f.n_active, device="cuda")
        for s in range(0, rays.shape[0], chunk):
            nb.baked_brick_weights_rays(f, rays[s:s + chunk], out=out)
        assert bits_equal(out, one), chunk
    perm = torch.randperm(rays.shape[0], generator=torch.Generator().manual_seed(4)).cuda()
    assert bits_equal(nb.baked_brick_weights_rays(f, rays[perm].contiguous()), one)
    assert bits_equal(nb.baked_brick_weights_rays(f, rays), one)
    # baked_brick_weights over poses: the same as the rays of those poses, packed
    poses = sphere_poses(6, offset=3.0)
    H, W, focal = LEGO_CAM
    assert bits_equal(nb.baked_brick_weights(f, poses, H, W, focal, scene_options("lego")), one)
    assert bits_equal(nb.baked_brick_weights(f, poses.cuda(), H, W, focal, scene_options("lego")), one)


def test_nan_weight_is_recorded_as_inf_and_empty_field_launches_nothing():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    # sigma_raw = +inf everywhere and a ray from x = -1e6 whose steps dt (1 / 64) are below half an ulp of t (1 / 16):
    # delta = (t + dt) - t = 0, so alpha = 1 - exp(-(inf 0)) is NaN, w is NaN and T stays NaN after it.  The box is
    # offset so that no corner weight is 0 (0 inf would make the interpolated sigma_raw NaN, which sigma's fmaxf drops)
    f = synthetic_field((64, 16, 16), seed=9, box=((-1.01, -1.0, -1.0), (0.99, 1.0, 1.0)))
    f.values[..., 0] = float("inf")
    ray = ray_rows(torch.tensor([[-1.0e6, 0.1, 0.1]], device="cuda"), torch.tensor([[1.0, 0.0, 0.0]], device="cuda"),
                far=1.0e7)
    got = nb.baked_brick_weights_rays(f, ray)
    assert not torch.isnan(got).any()
    hit = got > 0
    assert int(hit.sum()) == 8 and bool((got[hit] == float("inf")).all()), got[hit]  # the ray's 8 bricks
    assert torch.isnan(_render_rows(f, ray, False, 0.0)[0, :3]).all()
    # a field without active bricks returns an empty tensor without a launch
    empty = nb.prune_baked(f, torch.zeros(f.n_active, dtype=torch.bool, device="cuda"))
    before = ops.launch_count()
    assert nb.baked_brick_weights_rays(empty, random_rays(64, 9, misses=True)).shape == (0,)
    assert nb.baked_brick_weights(empty, sphere_poses(2), 8, 8, 10.0, scene_options("lego")).shape == (0,)
    assert ops.launch_count() == before


# ------------------------------------------------------------------------------------------------------------------------
# 4. transparent prune, 5. tau = 0 prune
# ------------------------------------------------------------------------------------------------------------------------
def _renders_bit_equal(a, b, rays, ctx):
    for white in (False, True):
        for stop in (0.0, 1e-3, 0.5):
            ra, rb = _render_rows(a, rays, white, stop), _render_rows(b, rays, white, stop)
            assert _out_bits_equal(ra, rb), (ctx, white, stop)


def test_dropping_transparent_bricks_keeps_every_render_bit_for_bit():
    import nerf_pytorch_b200 as nb

    # lego over the grid of both networks; poses used nowhere else in this file
    f = _bake("lego", 256, grid_res=128)
    tr = nb.baked_transparent_bricks(f)
    p = nb.prune_baked(f, ~tr)
    report("lego 256^3 both grids: transparent bricks dropped / active", "", (int(tr.sum()), f.n_active))
    assert 0 < p.n_active < f.n_active
    poses = sphere_poses(3, radius=3.3, phis=(-60.0, 10.0, -5.0), offset=41.0)
    for i, pose in enumerate(poses):
        rays = camera_rays("lego", pose)
        _renders_bit_equal(f, p, rays, ("lego", i))
    # a synthetic field with planted transparent bricks (some of them -0, one with NaN in channels 28 .. 31)
    s = synthetic_field((24, 24, 16), active=0.8, sigma=(-3.0, 5.0), seed=31)
    planted = torch.arange(s.n_active, device="cuda") % 3 == 1
    s.values[planted, :, 0] = -s.values[planted, :, 0].abs()
    s.values[planted.nonzero()[0], :, 0] = -0.0
    s.values[planted.nonzero()[-1], :, 28:] = float("nan")
    tr = nb.baked_transparent_bricks(s)
    assert bool(tr[planted].all())
    q = nb.prune_baked(s, ~tr)
    assert q.n_active <= s.n_active - int(planted.sum())
    rays = torch.cat([random_rays(4096, 32, misses=True), edge_rays(s)])
    _renders_bit_equal(s, q, rays, "synthetic")


def test_dropping_unseen_bricks_keeps_the_measuring_renders_and_tau_keeps_psnr():
    import nerf_pytorch_b200 as nb

    f = _bake("lego", 256, grid_res=128)
    H, W, focal = LEGO_CAM
    opts = scene_options("lego")
    poses = sphere_poses(8, offset=13.0)
    w = nb.baked_brick_weights(f, poses, H, W, focal, opts)
    tr = nb.baked_transparent_bricks(f)
    p0 = nb.prune_baked(f, w > 0)
    unseen_opaque = int(((w == 0) & ~tr).sum())
    report("lego 256^3: active / transparent / unseen / unseen and not transparent", "",
           (f.n_active, int(tr.sum()), int((w == 0).sum()), unseen_opaque))
    assert unseen_opaque > 0  # interior bricks with density: never seen by these views
    for i, pose in enumerate(poses):
        rays = camera_rays("lego", pose)
        for stop in (0.0, 1e-3):
            assert _out_bits_equal(_render_rows(f, rays, False, stop), _render_rows(p0, rays, False, stop)), (i, stop)
    # tau = 1e-2 over 40 poses, held-out PSNR against the unpruned field
    train = sphere_poses(40, offset=7.0)
    held = sphere_poses(4, phis=(-20.0, -40.0), offset=29.0)
    w = nb.baked_brick_weights(f, train, H, W, focal, opts)
    p2 = nb.prune_baked(f, w > 1e-2)
    vals = []
    for pose in held:
        rays = camera_rays("lego", pose)
        a, b = _render_rows(f, rays, False, 0.0)[:, :3], _render_rows(p2, rays, False, 0.0)[:, :3]
        vals.append(-10.0 * math.log10(max(((a - b) ** 2).mean().item(), 1e-20)))
    psnr = sum(vals) / len(vals)
    report("lego 256^3 tau 1e-2: kept / active, held-out PSNR against unpruned", "", (p2.n_active, f.n_active, psnr))
    assert p2.n_active < p0.n_active
    assert psnr >= TAU_PSNR_BAR, psnr


# held-out PSNR of the tau = 1e-2 field against the unpruned one (lego A0 256^3, both grids, 40 poses); measured on an
# H100 80GB HBM3 at 700 W: 85.0 dB (1 777 of 11 149 bricks kept)
TAU_PSNR_BAR = 70.0


# ------------------------------------------------------------------------------------------------------------------------
# 6. a pruned field still works
# ------------------------------------------------------------------------------------------------------------------------
def test_pruned_field_saves_loads_and_differentiates(tmp_path):
    import nerf_pytorch_b200 as nb

    f = synthetic_field((20, 17, 33), active=0.5, seed=4)
    keep = torch.arange(f.n_active, device="cuda") % 2 == 0
    p = nb.prune_baked(f, keep)
    path = tmp_path / "pruned.pt"
    p.save(path)
    q = nb.BakedField.load(path)
    for x, y in ((p.brick_map, q.brick_map), (p.bricks, q.bricks), (p.values, q.values)):
        assert bits_equal(x, y)
    assert (q.bounds, q.resolution, q.use_viewdirs, q.n_active) == (p.bounds, p.resolution, p.use_viewdirs, p.n_active)
    # the tied gradient of render_baked_rays against the fp64 sum over copies of fp64 autograd
    idx = lattice_index(p)
    assert copies_bit_equal(p.values, idx)
    rays = torch.cat([random_rays(1024, 12, misses=True), edge_rays(p)])
    v64 = p.values.detach().double().requires_grad_()
    rgb64, *_ = baked_render64(nb.BakedField(p.bounds, p.resolution, p.brick_map, p.bricks, v64, True), rays, False)
    g = torch.randn(rays.shape[0], 3, generator=torch.Generator(device="cuda").manual_seed(3), device="cuda")
    (rgb64 * g.double()).sum().backward()
    flat = idx.reshape(-1)
    acc = torch.zeros(int(flat.max()) + 1, 32, dtype=torch.float64, device="cuda")
    acc.index_add_(0, flat, v64.grad.reshape(-1, 32))
    want = acc[flat].view(v64.shape)
    p.values.requires_grad_()
    rgb, *_ = nb.render_baked_rays(p, rays)
    (rgb * g).sum().backward()
    err = ((p.values.grad.double() - want).abs().max() / want.abs().max()).item()
    report("pruned field: tied gradient error", "", err)
    assert copies_bit_equal(p.values.grad, idx)
    assert err <= SYN_REL, err


# ------------------------------------------------------------------------------------------------------------------------
# 7. BakedFieldTrainer.prune
# ------------------------------------------------------------------------------------------------------------------------
def test_trainer_prune_keeps_rows_and_state_and_trains_on():
    import nerf_pytorch_b200 as nb

    f = _bake("lego", (40, 36, 44), grid_res=32)
    idx = lattice_index(f)
    poses = sphere_poses(6)
    imgs, opts = targets("lego", poses)
    t = nb.BakedFieldTrainer(f, imgs, poses.cuda(), LEGO_CAM[2], opts, rays_per_step=2048, seed=3)
    t.step(20)
    assert copies_bit_equal(f.values, idx)
    H, W, focal = LEGO_CAM
    keep = nb.baked_brick_weights(f, poses, H, W, focal, opts) > 0
    assert 0 < int(keep.sum()) < f.n_active
    kept = torch.nonzero(keep).reshape(-1)
    before = [x[kept].clone() for x in (f.values, t.m, t.v)]
    step, old_map = t.step_dev.clone(), f.brick_map.clone()
    field_obj = t.field
    t.prune(keep)
    assert t.field is field_obj and f.n_active == kept.numel()
    for a, b in zip(before, (f.values, t.m, t.v)):
        assert bits_equal(a, b)
    assert bits_equal(t.step_dev.view(torch.int32), step.view(torch.int32))
    for x in (f.values, t.m, t.v, t.d_values, t.d_tied):
        assert x.shape == (kept.numel(), 729, 32)
    assert bool((f.brick_map[f.bricks.long()] == torch.arange(f.n_active, device="cuda", dtype=torch.int32)).all())
    assert int((f.brick_map >= 0).sum()) == f.n_active and int((old_map >= 0).sum()) > f.n_active
    idx = lattice_index(f)
    assert copies_bit_equal(f.values, idx)
    for _ in range(10):
        loss = t.step(10)
        assert math.isfinite(loss.item())
    assert int(t.step_dev) == 120
    assert copies_bit_equal(f.values, idx)
    with pytest.raises(ValueError):
        t.prune(torch.zeros(f.n_active, dtype=torch.bool, device="cuda"))
    with pytest.raises(ValueError):
        t.prune(torch.ones(f.n_active, dtype=torch.bool))  # on the host


# held-out PSNR after FT_STEPS trainer steps, prune-transparent-then-train against train-unpruned (lego A0 256^3, both
# grids); measured on an H100 80GB HBM3 at 700 W: 30.85 dB both, equal to the last digit (2 154 of 11 149 bricks kept).  A
# transparent brick receives no gradient of its own (its sigma gate is closed and its weights are 0), so pruning it
# removes only +0 terms from the tie's sums.  The bar allows PRUNE_PSNR_MARGIN below train-unpruned.
FT_STEPS = 300
PRUNE_PSNR_MARGIN = 0.1


def test_prune_transparent_then_train_matches_train_unpruned():
    import nerf_pytorch_b200 as nb

    poses = sphere_poses(44)
    imgs, opts = targets("lego", poses)
    held = [5, 16, 27, 38]
    train = [i for i in range(44) if i not in held]
    psnr = {}
    for arm in ("unpruned", "transparent"):
        f = _bake("lego", 256, grid_res=128)
        t = nb.BakedFieldTrainer(f, imgs[train].contiguous(), poses[train].cuda(), LEGO_CAM[2], opts,
                                 rays_per_step=2048, seed=1)
        if arm == "transparent":
            t.prune(~nb.baked_transparent_bricks(f))
        t.step(FT_STEPS)
        psnr[arm] = (heldout_psnr(f, poses[held], imgs[held]), f.n_active)
        del t, f
        torch.cuda.empty_cache()
    report("held-out PSNR, n_active after 300 steps", "", psnr)
    assert psnr["transparent"][0] >= psnr["unpruned"][0] - PRUNE_PSNR_MARGIN, psnr
