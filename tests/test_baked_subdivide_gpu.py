"""GPU: subdividing baked fields and fitting them without a network (csrc/baked.cu baked_subdivide_kernel;
nb.subdivide_baked, BakedFieldTrainer.subdivide, nb.BakedField.full; include/nerfb200.h "baked fields: subdivision").

  1. bits: the child values equal a torch fp32 restatement of the header's rule bit for bit (NaN as a class where a
     NaN is summed), on sparse and dense synthetic fields, with and without view directions, at resolutions that are
     not multiples of 8 and anisotropic, with +-inf, NaN, -0 and subnormals planted; coincident points are the parent's
     bits, NaN payloads included;
  2. structure: the child's bricks are sorted, brick_map is their rank, the active set is the existing children of the
     active parents; the child's copies are bit-equal on bakes and synthetic fields;
  3. the same function: fp64 trilinear evaluation of parent and child at random points of active bricks agrees within
     the bound that fp32 rounding of the child values allows;
  4. scene bakes: the child's held-out PSNR against render_image is within a measured margin of the parent's;
  5. the trainer: subdivide gives subdivide_baked of the field, m and v bitwise, keeps step_dev, recounts P, trains on;
     prune, subdivide, step keeps every copy bit-equal;
  6. BakedField.full: values, identity maps, a render against helpers.baked_render64;
  7. a from-scratch fit on lego, 64^3 -> 128^3;
  8. a child past 2^31 floats (about 10 GB of device memory)."""
import pytest
import torch

from helpers import (LEGO_BOX, LEGO_CAM, OUT_ABS, baked_render64, bake_scene, bits_equal, camera_rays,
                     copies_bit_equal, heldout_psnr, lattice_index, psnr32, random_rays, sphere_poses,
                     synthetic_field, targets)

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def report(what, ctx, value):
    print(f"[baked-subdivide] {what} {ctx}: {value}")


def restated(parent, child_bricks, slots=None):
    """fp32 [n, 729, 32]: the header's child values of ``child_bricks`` (int32, the child box at twice the parent's
    resolution) restated in torch, each op its own fp32 kernel (no contraction, no flush to zero on the device)."""
    dev = parent.values.device
    res = [2 * r for r in parent.resolution]
    nbc = [-(-r // 8) for r in res]
    nbp = [-(-r // 8) for r in parent.resolution]
    cb = child_bricks.long() if slots is None else child_bricks.long()[slots]
    b = torch.stack([cb % nbc[0], cb // nbc[0] % nbc[1], cb // (nbc[0] * nbc[1])], -1)  # [n, 3]
    p = torch.arange(729, device=dev)
    l = torch.stack([p % 9, p // 9 % 9, p // 81], -1)
    q = torch.minimum(8 * b[:, None] + l[None], torch.tensor(res, device=dev))  # [n, 729, 3]
    pb = b // 2
    ps = parent.brick_map.long()[(pb[:, 2] * nbp[1] + pb[:, 1]) * nbp[0] + pb[:, 0]]
    assert bool((ps >= 0).all())
    s0 = (q >> 1) - 8 * pb[:, None]  # the parent brick's local point
    odd = (q & 1).bool()
    m = odd.sum(-1)
    w = torch.where(m == 1, 0.5, torch.where(m == 2, 0.25, 0.125)).float()[..., None]
    V = parent.values
    acc = torch.zeros(cb.numel(), 729, 32, device=dev)
    started = torch.zeros(cb.numel(), 729, 1, dtype=torch.bool, device=dev)
    copy = None
    for k in range(8):
        off = torch.tensor([k & 1, k >> 1 & 1, k >> 2], device=dev)
        present = ((off == 0) | odd).all(-1)[..., None]
        lp = torch.minimum(s0 + off, torch.tensor(8, device=dev))
        v = V[ps[:, None], (lp[..., 2] * 9 + lp[..., 1]) * 9 + lp[..., 0]]
        if k == 0:
            copy = v
        t = w * v
        acc = torch.where(present & started, acc + t, torch.where(present, t, acc))
        started = started | present
    out = torch.where((m == 0)[..., None], copy, acc)
    out[..., 28:] = 0.0
    return out


def same_bits_nan_class(a, b):
    ai, bi = a.contiguous().view(torch.int32), b.contiguous().view(torch.int32)
    return bool(((ai == bi) | (torch.isnan(a) & torch.isnan(b))).all())


def check_child(parent, child):
    """Structure, values and ties of ``child`` = subdivide_baked(parent)."""
    assert child.resolution == tuple(2 * r for r in parent.resolution) and child.bounds == parent.bounds
    assert child.use_viewdirs == parent.use_viewdirs and child.values.dtype == torch.float32
    nbp = [-(-r // 8) for r in parent.resolution]
    nbc = [-(-r // 8) for r in child.resolution]
    # the active set: every child brick whose parent is active, and nothing else
    cid = torch.arange(nbc[0] * nbc[1] * nbc[2], device="cuda")
    cx, cy, cz = cid % nbc[0], cid // nbc[0] % nbc[1], cid // (nbc[0] * nbc[1])
    want = cid[parent.brick_map.long()[((cz // 2) * nbp[1] + cy // 2) * nbp[0] + cx // 2] >= 0]
    assert torch.equal(child.bricks.long(), want)
    assert bool((child.bricks[1:] > child.bricks[:-1]).all())
    assert torch.equal(child.brick_map[child.bricks.long()], torch.arange(child.n_active, dtype=torch.int32,
                                                                          device="cuda"))
    assert int((child.brick_map >= 0).sum()) == child.n_active
    ref = restated(parent, child.bricks)
    assert same_bits_nan_class(child.values, ref)
    # coincident points are the parent's bits, NaN payloads included
    q = lattice_index(child)
    res = torch.tensor(child.resolution, device="cuda")
    qx, qy, qz = q % (res[0] + 1), q // (res[0] + 1) % (res[1] + 1), q // ((res[0] + 1) * (res[1] + 1))
    even = (qx % 2 == 0) & (qy % 2 == 0) & (qz % 2 == 0)
    assert bits_equal(child.values[even], ref[even])
    return ref


# ------------------------------------------------------------------------------------------------------------------------
# 1, 2. bits, structure and ties on synthetic fields
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("res,active,viewdirs", [((16, 16, 16), 1.0, True), ((16, 16, 16), 0.4, False),
                                                 ((20, 13, 37), 0.5, True), ((9, 8, 7), 1.0, True),
                                                 ((17, 33, 4), 0.7, False), ((3, 2, 12), 1.0, True)])
def test_child_bits_structure_and_ties_on_synthetic_fields(res, active, viewdirs):
    import nerf_pytorch_b200 as nb

    f = synthetic_field(res, viewdirs=viewdirs, active=active, seed=sum(res))
    c = nb.subdivide_baked(f)
    check_child(f, c)
    assert copies_bit_equal(c.values, lattice_index(c))


def test_special_values_planted():
    import nerf_pytorch_b200 as nb

    f = synthetic_field((20, 13, 37), active=0.8, seed=11)
    idx = lattice_index(f)
    payload = torch.tensor([0x7fc00123], dtype=torch.int32, device="cuda").view(torch.float32)
    specials = [float("inf"), -float("inf"), float("nan"), -0.0, 1e-40, -3e-42, 2.0 ** -126, 1.5e-45]
    g = torch.Generator(device="cuda").manual_seed(3)
    flat = idx.reshape(-1)
    vals = f.values.view(-1, 32)
    for i, s in enumerate(specials + [None] * 4):
        pts = torch.randint(0, int(flat.max()) + 1, (40,), generator=g, device="cuda")
        hit = torch.isin(flat, pts)
        ch = torch.randint(0, 28, (1,), generator=g, device="cuda").item()
        vals[hit, ch] = payload if s is None else s  # every copy of a point the same bits
    # whole neighbourhoods of subnormals, so that means of subnormals are formed too
    vals[(flat % 97) < 5, 3] = 1e-39
    vals[(flat % 89) < 5, 4] = -7e-41
    assert copies_bit_equal(f.values, idx)
    c = nb.subdivide_baked(f)
    check_child(f, c)
    assert copies_bit_equal(c.values, lattice_index(c))
    cv = c.values.view(-1, 32).contiguous().view(torch.int32)
    assert bool((cv == int(payload.view(torch.int32))).any())  # a NaN payload copied through
    assert bool(((c.values.abs() < 2.0 ** -126) & (c.values != 0)).any())  # subnormal means kept


def test_bits_and_ties_on_scene_bakes():
    import nerf_pytorch_b200 as nb

    for kind, res, grid in (("lego", (40, 36, 44), 32), ("fern", 48, 32), ("noview", 24, None)):
        f = bake_scene(kind, res, grid_res=grid)
        assert copies_bit_equal(f.values, lattice_index(f))
        c = nb.subdivide_baked(f)
        check_child(f, c)
        assert copies_bit_equal(c.values, lattice_index(c)), kind


def test_empty_field_gives_an_empty_child_without_a_launch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    f = synthetic_field((20, 13, 37), active=0.5, seed=2)
    e = nb.prune_baked(f, torch.zeros(f.n_active, dtype=torch.bool, device="cuda"))
    n0 = ops.launch_count()
    c = nb.subdivide_baked(e)
    assert ops.launch_count() == n0
    assert c.n_active == 0 and c.values.shape == (0, 729, 32) and c.resolution == (40, 26, 74)
    assert c.brick_map.numel() == 5 * 4 * 10 and bool((c.brick_map == -1).all())
    # the argument is untouched by a real subdivision
    snap = [x.clone() for x in (f.brick_map, f.bricks, f.values)]
    n0 = ops.launch_count()
    nb.subdivide_baked(f)
    assert ops.launch_count() == n0 + 1
    for a, b in zip(snap, (f.brick_map, f.bricks, f.values)):
        assert bits_equal(a, b)


# ------------------------------------------------------------------------------------------------------------------------
# 3. the same function
# ------------------------------------------------------------------------------------------------------------------------
def trilinear64(field, u):
    """fp64 channels 0 .. 27 of ``field`` at lattice coordinates u [n, 3] (cube i = floor(u), clamped to res - 1),
    each point inside an active brick."""
    res = torch.tensor(field.resolution, device="cuda")
    i = torch.minimum(u.floor().long(), res - 1)
    fr = u - i.double()
    nb_ = (res + 7) // 8
    b = i // 8
    slot = field.brick_map.long()[(b[:, 2] * nb_[1] + b[:, 1]) * nb_[0] + b[:, 0]]
    assert bool((slot >= 0).all())
    l = i % 8
    vals = field.values.double()
    v = torch.zeros(u.shape[0], 28, dtype=torch.float64, device="cuda")
    for k in range(8):
        off = torch.tensor([k & 1, k >> 1 & 1, k >> 2], device="cuda")
        lc = l + off
        w = torch.where(off.bool(), fr, 1 - fr).prod(-1)
        v += w[:, None] * vals[slot, (lc[:, 2] * 9 + lc[:, 1]) * 9 + lc[:, 0]][:, :28]
    return v


# |child(u) - parent(u)| <= 7 u M per channel: a child value is the fp32 sum of at most 8 exact terms w v whose
# magnitudes sum to at most M = max |parent value| of the channel (the weights sum to 1), so its rounding error is at
# most 7 u M (the sequential-sum bound (n - 1) u sum |t_i|); the child function at u is a convex combination of its 8
# corner values, so it is off the parent function by at most the same.  fp64 evaluation adds ~1e-15 M.
@pytest.mark.parametrize("kind", ["synthetic", "lego"])
def test_child_holds_the_parent_function(kind):
    import nerf_pytorch_b200 as nb

    f = synthetic_field((20, 13, 37), active=0.6, seed=5) if kind == "synthetic" else \
        bake_scene("lego", 64, grid_res=32)
    c = nb.subdivide_baked(f)
    g = torch.Generator(device="cuda").manual_seed(1)
    n = 200_000
    slot = torch.randint(0, f.n_active, (n,), generator=g, device="cuda")
    nb_ = [-(-r // 8) for r in f.resolution]
    br = f.bricks.long()[slot]
    b = torch.stack([br % nb_[0], br // nb_[0] % nb_[1], br // (nb_[0] * nb_[1])], -1)
    res = torch.tensor(f.resolution, device="cuda", dtype=torch.float64)
    u = torch.minimum(8 * b.double() + 8 * torch.rand(n, 3, generator=g, device="cuda", dtype=torch.float64), res)
    u[:n // 10] = u[:n // 10].floor()  # lattice points of the parent (floor: the point stays in its brick)
    u[n // 10:n // 5] = (2 * u[n // 10:n // 5]).floor() / 2  # new lattice points of the child
    pv, cv = trilinear64(f, u), trilinear64(c, 2 * u)
    M = f.values[..., :28].abs().reshape(-1, 28).amax(0).double()
    err = (cv - pv).abs()
    ratio = (err / (U * M)).amax(0)
    report("max |child - parent| / (u M) per channel", kind, [round(x, 3) for x in ratio.tolist()])
    assert bool((err <= 7 * U * M + 1e-14 * M).all()), ratio.max().item()


# ------------------------------------------------------------------------------------------------------------------------
# 4. scene bakes
# ------------------------------------------------------------------------------------------------------------------------
# held-out PSNR (dB) of the child against render_image minus the parent's.  The child renders the parent's continuous
# field at half the sample spacing.  Measured on an H100 80GB HBM3 at 700 W: lego 24.231 -> 24.187 dB (-0.044), fern
# 24.028 -> 24.033 dB (+0.005).  No training is involved, so the bits repeat; the bar allows 3x the lego loss.
CHILD_MARGIN = 0.15


def fern_psnr(field, poses, imgs):
    with torch.no_grad():
        return sum(psnr32(nb_render(field, camera_rays("fern", p)), im.reshape(-1, 3))
                   for p, im in zip(poses, imgs)) / len(poses)


def nb_render(field, rays):
    import nerf_pytorch_b200 as nb

    return nb.render_baked_rays(field, rays)[0]


@pytest.mark.parametrize("kind", ["lego", "fern"])
def test_child_psnr_on_scene_bakes(kind):
    import nerf_pytorch_b200 as nb

    if kind == "lego":
        poses = sphere_poses(44)[[5, 16, 27, 38]]
        imgs, _ = targets("lego", poses)
        f = bake_scene("lego", 128, grid_res=64, grid_from="both")
        ev = lambda x: heldout_psnr(x, poses, imgs)  # noqa: E731
    else:
        poses = torch.stack([torch.eye(4)] * 3)
        poses[1, 0, 3], poses[2, 1, 3] = 0.05, -0.05
        imgs, _ = targets("fern", poses)
        f = bake_scene("fern", 128, grid_res=64, grid_from="both")
        ev = lambda x: fern_psnr(x, poses, imgs)  # noqa: E731
    c = nb.subdivide_baked(f)
    pp, pc = ev(f), ev(c)
    report("held-out PSNR parent, child", kind, (round(pp, 3), round(pc, 3)))
    assert pc >= pp - CHILD_MARGIN, (pp, pc)


# ------------------------------------------------------------------------------------------------------------------------
# 5. the trainer
# ------------------------------------------------------------------------------------------------------------------------
def _full_mse(field, poses, imgs):
    import nerf_pytorch_b200 as nb

    with torch.no_grad():
        return sum(((nb.render_baked_rays(field, camera_rays("lego", p))[0] - im.reshape(-1, 3)) ** 2).mean().item()
                   for p, im in zip(poses, imgs)) / len(poses)


def test_trainer_subdivide():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    f = bake_scene("lego", (24, 20, 28), grid_res=32)
    poses = sphere_poses(6)
    imgs, opts = targets("lego", poses)
    t = nb.BakedFieldTrainer(f, imgs, poses.cuda(), LEGO_CAM[2], opts, rays_per_step=2048, seed=3, tv_sigma=1e-4,
                             sparsity=1e-4)
    t.step(10)
    parent = nb.BakedField(f.bounds, f.resolution, f.brick_map.clone(), f.bricks.clone(), f.values.clone(),
                           f.use_viewdirs)
    m, v = t.m.clone(), t.v.clone()
    step = t.step_dev.clone()
    t.subdivide()
    want = nb.subdivide_baked(parent)
    assert f.resolution == want.resolution and t._box.res[:] == list(want.resolution)
    for a, b in ((f.brick_map, want.brick_map), (f.bricks, want.bricks), (f.values, want.values)):
        assert bits_equal(a, b)
    for a, b in ((t.m, m), (t.v, v)):
        wb = nb.subdivide_baked(nb.BakedField(parent.bounds, parent.resolution, parent.brick_map, parent.bricks, b,
                                              True))
        assert bits_equal(a, wb.values)
    assert torch.equal(t.step_dev, step)
    assert t.d_values.shape == f.values.shape and t.d_tied.shape == f.values.shape
    assert int(t._count) == int(ops.baked_lattice_count(f.box(), f.brick_map, f.bricks))
    before = _full_mse(f, poses, imgs)
    t.step(60)
    after = _full_mse(f, poses, imgs)
    report("training-view mse before / after 60 steps at the child resolution", "", (before, after))
    assert after < before
    assert copies_bit_equal(f.values, lattice_index(f))


def test_prune_subdivide_step_keeps_copies_bit_equal():
    import nerf_pytorch_b200 as nb

    f = bake_scene("lego", (40, 40, 40))
    poses = sphere_poses(4)
    imgs, opts = targets("lego", poses)
    t = nb.BakedFieldTrainer(f, imgs, poses.cuda(), LEGO_CAM[2], opts, rays_per_step=1024, seed=5, tv_sigma=1e-4)
    t.step(3)
    keep = ~nb.baked_transparent_bricks(f)
    assert 0 < int(keep.sum()) < f.n_active
    t.prune(keep)
    t.subdivide()
    assert f.resolution == (80, 80, 80) and copies_bit_equal(f.values, lattice_index(f))
    t.step(10)
    assert copies_bit_equal(f.values, lattice_index(f))
    assert copies_bit_equal(t.m, lattice_index(f)) and copies_bit_equal(t.v, lattice_index(f))


# ------------------------------------------------------------------------------------------------------------------------
# 6. BakedField.full
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("viewdirs", [True, False])
def test_full_field(viewdirs):
    import nerf_pytorch_b200 as nb

    f = nb.BakedField.full(((-1.0,) * 3, (1.0,) * 3), (20, 13, 37), sigma_raw=0.7, use_viewdirs=viewdirs)
    n = 3 * 2 * 5
    assert f.values.is_cuda and f.n_active == n and f.dtype == torch.float32 and f.use_viewdirs == viewdirs
    ids = torch.arange(n, dtype=torch.int32, device="cuda")
    assert torch.equal(f.brick_map, ids) and torch.equal(f.bricks, ids)
    assert bool((f.values[..., 0] == 0.7).all()) and bool((f.values[..., 1:] == 0).all())
    rays = random_rays(512, seed=4, viewdirs=viewdirs, misses=True)
    rgb, disp, acc, depth = nb.render_baked_rays(f, rays)
    rgb64, acc64, depth64, _ = baked_render64(f, rays, False)
    assert (rgb.double() - rgb64).abs().max().item() < OUT_ABS
    assert (acc.double() - acc64).abs().max().item() < OUT_ABS
    assert (depth.double() - depth64).abs().max().item() < OUT_ABS * 6.0
    assert float(acc.max()) > 0.5 and bool((rgb[acc > 0] - 0.5 * acc[acc > 0, None]).abs().max() < 1e-5)


# ------------------------------------------------------------------------------------------------------------------------
# 7. a from-scratch fit
# ------------------------------------------------------------------------------------------------------------------------
# BakedField.full(LEGO_BOX, 64, sigma_raw 0.1), PIPE_STEPS trainer steps (2048 rays, 40 training views at 48 x 48,
# lr_sigma PIPE_LR_SIGMA, lr_sh PIPE_LR_SH), prune at peak weight > PIPE_TAU over the training views, subdivide to
# 128^3, PIPE_STEPS more.  Held-out PSNR against render_image at the 4 held-out poses of the fine-tuning tests.
PIPE_STEPS = 400
PIPE_LR_SIGMA, PIPE_LR_SH = 1.0, 3e-2
PIPE_TAU = 1e-3
# Measured on an H100 80GB HBM3 at 700 W: 23.18 dB at 64^3 (251 of 512 bricks kept), 23.40 dB at 128^3 (2 008 bricks),
# 0.7 s.  The backward's reductions run in hardware order, so runs differ in the last bits; the bar is 0.5 dB below.
PIPE_PSNR_MEASURED = 23.40
PIPE_PSNR_BAR = PIPE_PSNR_MEASURED - 0.5


def test_from_scratch_fit_on_lego():
    import time

    import nerf_pytorch_b200 as nb

    poses = sphere_poses(44)
    imgs, opts = targets("lego", poses)
    held = [5, 16, 27, 38]
    train = [i for i in range(44) if i not in held]
    tp = poses[train].cuda()
    t0 = time.perf_counter()
    f = nb.BakedField.full(LEGO_BOX, 64, sigma_raw=0.1)
    t = nb.BakedFieldTrainer(f, imgs[train].contiguous(), tp, LEGO_CAM[2], opts, lr_sigma=PIPE_LR_SIGMA,
                             lr_sh=PIPE_LR_SH, rays_per_step=2048, seed=1)
    t.step(PIPE_STEPS)
    first = heldout_psnr(f, poses[held], imgs[held])
    w = nb.baked_brick_weights(f, poses[train], LEGO_CAM[0], LEGO_CAM[1], LEGO_CAM[2], opts)
    t.prune(w > PIPE_TAU)
    n_pruned = f.n_active
    t.subdivide()
    t.step(PIPE_STEPS)
    final = heldout_psnr(f, poses[held], imgs[held])
    torch.cuda.synchronize()
    report("held-out PSNR 64^3, 128^3; bricks kept of 512 -> child; seconds", "",
           (round(first, 3), round(final, 3), n_pruned, f.n_active, round(time.perf_counter() - t0, 1)))
    assert final > first
    assert final >= PIPE_PSNR_BAR
    assert copies_bit_equal(f.values, lattice_index(f))


# ------------------------------------------------------------------------------------------------------------------------
# 8. a child past 2^31 floats
# ------------------------------------------------------------------------------------------------------------------------
def test_child_past_2_31_floats():
    """Allocates about 10 GB of device memory: a 256^3 parent on ~11 800 bricks (1.1 GB, plus a 2.2 GB lattice while it
    is built) and its child on ~94 000 (8.8 GB)."""
    import nerf_pytorch_b200 as nb

    f = synthetic_field((256, 256, 256), active=0.36, seed=9)
    c = nb.subdivide_baked(f)
    report("parent bricks, child bricks, child floats", "", (f.n_active, c.n_active, c.values.numel()))
    assert c.values.numel() > 2 ** 31
    first_past = (2 ** 31) // (729 * 32)
    slots = torch.tensor([0, first_past - 1, first_past, first_past + 1, c.n_active - 2, c.n_active - 1],
                         device="cuda")
    ref = restated(f, c.bricks, slots)
    assert same_bits_nan_class(c.values[slots], ref)
    del c
    torch.cuda.empty_cache()
