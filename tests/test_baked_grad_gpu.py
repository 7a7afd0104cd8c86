"""GPU: gradients and fine-tuning of baked fields (csrc/baked.cu baked_render_bwd_kernel / baked_tie_kernel,
csrc/sampling.cu baked_adam_dev_kernel; nb.render_baked_rays, nb.BakedFieldTrainer; include/nerfb200.h "baked fields:
gradients and fine-tuning").

  1. the kernel's untied gradient against fp64 autograd of helpers.baked_render64 on an fp64 leaf copy of the values:
     a loss sum g . (rgb, disp, acc, depth) with random g, and the MSE loss alone; lego A0 with and without a white
     background, the coarse-only network without view directions, fern in NDC, opaque synthetic fields (the suffix
     E - prefix), rays that miss the box, rays along brick faces and through brick corners, a res that is not a multiple
     of 8, a grid that leaves bricks inactive; every sample's sigma gate, restated from the kernel's fp32 interpolation,
     is the oracle's;
  2. the tie: the bake's copies are bit-equal; after baked_tie every copy's gradient is bit-equal and matches the fp64
     sum over copies of the oracle's gradient; after trainer steps and after torch.optim.Adam steps on
     render_baked_rays every copy of every lattice point is still bit-equal; the baked Adam is adam_step_dev bit for bit
     on each channel group;
  3. fine-tuning helps: lego A0 baked at 256^3, held-out PSNR against render_image rises; fern's loss falls;
  4. what should reproduce does: the same seed draws the same pixels and targets; two runs agree to fp32 rounding.

Measured on an H100 80GB HBM3 at 700 W: the file runs in about 22 s; device memory allocated peaks at 2.6 GiB through
the 256^3 lego fine-tuning test (the field and its four values-sized buffers)."""
import math

import pytest
import torch

from helpers import (FERN_CAM, LEGO_CAM, baked_render64, bake_scene, bits_equal, camera_rays, copies_bit_equal,
                     edge_rays, heldout_psnr, lattice_index, random_rays, sphere_poses, synthetic_field, targets)

pytestmark = pytest.mark.gpu

# the kernel's gradient against the fp64 oracle: max |d - d64| over a channel group divided by the group's max |d64|
# (sigma_raw: channel 0; coefficients: channels 1 .. 27), and the tied gradient against the fp64 sum over copies, the
# same way.  Measured on an H100 80GB HBM3 at 700 W:
#   SYN_REL, synthetic fields with sigma_raw up to 8: at most 5.5e-6 (sigma) and 2.4e-6 (coefficients);
#   SAT_REL, fields whose rays saturate: the baked networks at most 5.1e-5 (sigma, fern)
#   and 4.1e-5 (coefficients, the coarse-only network); the opaque synthetic field (sigma delta 0.5 .. 3) 3.3e-5 (sigma).
#   Once a ray saturates, S = E - prefix carries about one ulp of E per add where the true suffix is ~0, and the
#   largest sigma gradient of such a field is small (0.01 for the opaque field against 0.15 - 0.3 for the others): the
#   opaque field, where alpha never rounds to 1, shows that the approximation alone gives errors of this size.  On the
#   networks, alpha also rounds to 1 where sigma delta > ~17 (q = (1 - alpha) + 1e-10 keeps only the 1e-10), which the
#   fp64 oracle does not do.
SYN_REL = 1e-5
SAT_REL = 1e-4


def report(what, ctx, value):
    print(f"[baked-grad] {what} {ctx}: {value}")


def _sum_over_copies(x, idx):
    """x [n, 729, C] summed over every stored copy of each lattice point (fp64), returned at every copy."""
    C = x.shape[-1]
    flat = idx.reshape(-1)
    acc = torch.zeros(int(flat.max()) + 1, C, dtype=torch.float64, device=x.device)
    acc.index_add_(0, flat, x.reshape(-1, C).double())
    return acc[flat].view(x.shape)


def _gate_flips(field, rays):
    """Samples whose sigma gate (interpolated sigma_raw > 0) differs between the kernel's fp32 fmaf chain and fp64: the
    gate is the rendering's one discontinuity, and baked_render64 takes it from fp64.  The samples, cells and fractions
    are formed in fp32 as baked_render64 (and the header) form them; fmaf(w, a, v) is fp32(w a + v) with the exact
    product, formed in fp64."""
    f32 = torch.float32
    lo = torch.tensor(field.bounds[0], dtype=f32, device="cuda")
    hi = torch.tensor(field.bounds[1], dtype=f32, device="cuda")
    res = torch.tensor(field.resolution, device="cuda")
    o, d = rays[:, :3], rays[:, 3:6]
    t0, t1 = (lo - o) / d, (hi - o) / d
    flat = d == 0
    ta = torch.fmax(rays[:, 6], torch.where(flat, -math.inf, torch.fmin(t0, t1).nan_to_num(nan=-math.inf)).amax(-1))
    outside = (flat & ~((o >= lo) & (o < hi))).any(-1)
    tb = torch.where(outside, -math.inf, torch.fmin(rays[:, 7], torch.where(
        flat, math.inf, torch.fmax(t0, t1).nan_to_num(nan=math.inf)).amin(-1)))
    dn = torch.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    dt = (torch.tensor(0.5, dtype=f32, device="cuda") * ((hi - lo) / res.to(f32)).min()) / dn
    live = (ta < tb) & (dt > 0) & (dt < math.inf) & ((tb - ta) / dt < 16777216.0)
    K = int(torch.where(live, (tb - ta) / dt, 0.0).max().item()) + 2
    t = ta[:, None] + (torch.arange(K, device="cuda", dtype=f32) + 0.5)[None] * dt[:, None]
    valid = (t < tb[:, None]) & live[:, None]
    x = o[:, None] + d[:, None] * torch.where(valid, t, 0.0)[..., None]
    tc = (x - lo) * (res.to(f32) / (hi - lo))
    inside = ((tc >= 0) & (tc < res.to(f32))).all(-1) & valid
    i = torch.where(inside[..., None], tc, torch.zeros_like(tc)).to(torch.int64).clamp_max(res - 1)
    fr = tc - i.to(f32)
    nb_ = (res + 7) // 8
    b = i // 8
    slot = field.brick_map.long()[((b[..., 2] * nb_[1] + b[..., 1]) * nb_[0] + b[..., 0]).clamp(0, field.brick_map.numel() - 1)]
    hit = inside & (slot >= 0)
    l = i % 8
    s32 = torch.zeros(t.shape, dtype=f32, device="cuda")
    s64 = torch.zeros(t.shape, dtype=torch.float64, device="cuda")
    for c in range(8):
        off = torch.tensor([c & 1, c >> 1 & 1, c >> 2], device="cuda")
        wc = torch.where(off.bool(), fr, 1 - fr)
        w = (wc[..., 0] * wc[..., 1]) * wc[..., 2]
        lc = l + off
        a = field.values[slot.clamp_min(0), (lc[..., 2] * 9 + lc[..., 1]) * 9 + lc[..., 0], 0]
        s32 = (w.double() * a.double() + s32.double()).float()
        s64 = s64 + (1 - fr.double()).where(~off.bool(), fr.double()).prod(-1) * a.double()
    return int((hit & ((s32 > 0) != (s64 > 0))).sum())


def _grad_check(field, rays, white, loss, ctx, bar, seed=0):
    """The kernel's untied gradient and the fp64 oracle's; asserts the bars and returns (d, d64)."""
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    n = rays.shape[0]
    assert _gate_flips(field, rays) == 0, ctx  # the oracle's fp64 gate is the kernel's fp32 gate on every sample
    v64 = field.values.detach().double().requires_grad_()
    f64 = nb.BakedField(field.bounds, field.resolution, field.brick_map, field.bricks, v64, field.use_viewdirs)
    rgb, acc, depth, _ = baked_render64(f64, rays, white)
    out = ops.baked_render(field.box(), field.brick_map, field.values, field.use_viewdirs, rays, white)
    g = torch.Generator(device="cuda").manual_seed(seed)
    gout = torch.zeros(n, 8, device="cuda")
    if loss == "mse":
        target = torch.rand(n, 3, generator=g, device="cuda")
        alpha = torch.tensor(2.0 / (3.0 * n), dtype=torch.float32)
        gout[:, :3] = alpha.cuda() * (out[:, :3] - target)
        L = ((rgb - target.double()) ** 2).mean()
    else:
        gout[:, :6] = torch.randn(n, 6, generator=g, device="cuda")
        ok = out[:, 4] > 1e-3  # disp's gradient only where acc is well away from 0
        gout[~ok, 3] = 0.0
        okd = acc > 1e-3
        disp = 1.0 / torch.clamp(depth / torch.where(okd, acc, 1.0), min=1e-10)
        gd = gout.double()
        L = (gd[:, :3] * rgb).sum() + (gd[:, 3] * torch.where(okd, disp, 0.0)).sum() + (gd[:, 4] * acc).sum() \
            + (gd[:, 5] * depth).sum()
    L.backward()
    d64 = v64.grad
    d = torch.zeros_like(field.values)
    ops.baked_render_bwd(field.box(), field.brick_map, field.values, field.use_viewdirs, rays, white, out, gout, d)
    assert torch.isfinite(d).all() and (d[..., 28:] == 0).all()
    e_sig = ((d[..., 0].double() - d64[..., 0]).abs().max() / d64[..., 0].abs().max().clamp_min(1e-30)).item()
    e_coef = ((d[..., 1:28].double() - d64[..., 1:28]).abs().max() / d64[..., 1:28].abs().max().clamp_min(1e-30)).item()
    report("sigma / coefficient gradient error", ctx, (e_sig, e_coef, float(d64[..., 0].abs().max())))
    assert d64[..., 0].abs().max() > 0 and d64[..., 1:28].abs().max() > 0, ctx
    assert e_sig <= bar and e_coef <= bar, (ctx, e_sig, e_coef)
    return d, d64


# ------------------------------------------------------------------------------------------------------------------------
# 1. gradients against fp64
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("loss", ["dot", "mse"])
@pytest.mark.parametrize("kind,white", [("lego", False), ("lego", True), ("noview", False), ("fern", False)])
def test_gradient_matches_fp64_on_baked_networks(kind, white, loss):
    field = bake_scene(kind, (24, 20, 28))
    rays = camera_rays(kind, viewdirs=field.use_viewdirs)
    if kind == "lego":  # rays that miss the box: turned away from it
        rays[::7, 3:6] = -rays[::7, 3:6]
    _grad_check(field, rays, white, loss, (kind, white, loss), SAT_REL)


@pytest.mark.parametrize("case", ["opaque", "edges", "res13", "inactive", "noview_inactive"])
def test_gradient_matches_fp64_on_synthetic_fields(case):
    if case == "opaque":  # sigma delta in 0.5 .. 3: rays saturate within a few cubes, E - prefix cancels to the tail
        f = synthetic_field((16, 16, 16), sigma=(8.0, 48.0), seed=1)
    elif case == "edges":
        f = synthetic_field((24, 24, 24), seed=2)
    elif case == "res13":
        f = synthetic_field((13, 9, 17), seed=3)
    elif case == "inactive":
        f = synthetic_field((20, 17, 33), active=0.5, seed=4)
    else:
        f = synthetic_field((20, 17, 12), viewdirs=False, active=0.5, seed=5)
    rays = torch.cat([random_rays(1024, 10, f.use_viewdirs), edge_rays(f, f.use_viewdirs)])
    for white in (False, True):
        for loss in ("dot", "mse"):
            _grad_check(f, rays, white, loss, (case, white, loss), SAT_REL if case == "opaque" else SYN_REL)


def test_autograd_path_is_the_tied_kernel_gradient():
    """render_baked_rays' backward is baked_render_bwd then baked_tie; an empty field gets an empty gradient."""
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    f = synthetic_field((16, 12, 20), active=0.6, seed=6)
    rays = random_rays(512, 11)
    f.values.requires_grad_()
    rgb, disp, acc, depth = nb.render_baked_rays(f, rays, white_background=True)
    out = ops.baked_render(f.box(), f.brick_map, f.values.detach(), True, rays, True)
    assert bits_equal(rgb, out[:, :3]) and bits_equal(acc, out[:, 4]) and bits_equal(depth, out[:, 5])
    g = torch.randn(512, 3, device="cuda")
    (rgb * g).sum().backward()
    gout = torch.zeros(512, 8, device="cuda")
    gout[:, :3] = g
    d = torch.zeros_like(f.values)
    ops.baked_render_bwd(f.box(), f.brick_map, f.values.detach(), True, rays, True, out, gout, d)
    idx = lattice_index(f)
    assert copies_bit_equal(f.values.grad, idx)
    want = _sum_over_copies(d, idx)
    err = ((f.values.grad.double() - want).abs().max() / want.abs().max()).item()
    assert err <= SYN_REL, err
    empty = nb.BakedField(f.bounds, f.resolution, torch.full_like(f.brick_map, -1), f.bricks[:0],
                          torch.zeros(0, 729, 32, device="cuda", requires_grad=True), True)
    rgb, _, acc, _ = nb.render_baked_rays(empty, rays)
    assert (acc == 0).all() and (rgb == 0).all()
    rgb.sum().backward()
    assert empty.values.grad.shape == (0, 729, 32)


# ------------------------------------------------------------------------------------------------------------------------
# 2. the tie
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["lego", "res13", "inactive"])
def test_tie_gives_every_copy_the_fp64_sum_over_copies(kind):
    from nerf_pytorch_b200 import ops

    bar = SAT_REL if kind == "lego" else SYN_REL
    if kind == "lego":
        f = bake_scene("lego", (24, 20, 28), grid_res=32)
        rays = camera_rays("lego")
        assert 0 < f.n_active < f.brick_map.numel()
    else:
        f = synthetic_field((13, 9, 17), seed=3) if kind == "res13" else \
            synthetic_field((20, 17, 33), active=0.5, seed=4)
        rays = torch.cat([random_rays(1024, 12), edge_rays(f)])
    idx = lattice_index(f)
    assert copies_bit_equal(f.values, idx)  # the bake (and synthetic_field) write every copy the same bits
    d, d64 = _grad_check(f, rays, False, "dot", ("tie", kind), bar)
    tied = ops.baked_tie(f.box(), f.brick_map, f.bricks, d)
    assert copies_bit_equal(tied, idx) and (tied[..., 28:] == 0).all()
    want = _sum_over_copies(d64, idx)
    err = ((tied.double() - want).abs().max() / want.abs().max()).item()
    report("tied gradient error", kind, err)
    assert err <= bar, err
    assert not copies_bit_equal(d, idx)  # the untied gradient differs between copies: the tie did something


def test_baked_adam_is_adam_step_dev_per_channel_group():
    """baked_adam_step_dev gives sigma_raw the bits of adam_step_dev at lr_sigma and the coefficients those at lr_sh, at
    the same device step and schedule; channels 28 .. 31 of values, m and v are not touched."""
    from nerf_pytorch_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(8)
    vals, grad, m, v = (torch.randn(3, 729, 32, generator=g, device="cuda") for _ in range(4))
    v = v.abs()
    step = torch.full((1,), 1500, dtype=torch.int64, device="cuda")
    want = []
    for sl, lr in ((slice(0, 1), 0.7), (slice(1, 28), 0.02)):
        p, mm, vv = (x[..., sl].contiguous() for x in (vals, m, v))
        ops.adam_step_dev(p, grad[..., sl].contiguous(), mm, vv, step, lr, lr_decay=2.0, lr_decay_factor=0.1)
        want.append((p, mm, vv))
    before = [x.clone() for x in (vals, m, v)]
    ops.baked_adam_step_dev(vals, grad, m, v, step, 0.7, 0.02, lr_decay=2.0, lr_decay_factor=0.1)
    for i, x in enumerate((vals, m, v)):
        assert bits_equal(x[..., 0:1], want[0][i]) and bits_equal(x[..., 1:28], want[1][i]), i
        assert bits_equal(x[..., 28:], before[i][..., 28:]), i
    assert int(step) == 1500  # the counter is step_advance's to move


def test_copies_stay_bit_equal_under_the_trainer_and_torch_adam():
    import nerf_pytorch_b200 as nb

    f = bake_scene("lego", (24, 20, 28), grid_res=32)
    idx = lattice_index(f)
    poses = sphere_poses(6)
    imgs, opts = targets("lego", poses)
    t = nb.BakedFieldTrainer(f, imgs, poses.cuda(), LEGO_CAM[2], opts, rays_per_step=2048, seed=3)
    before = f.values.clone()
    t.step(20)
    assert not bits_equal(before, f.values) and copies_bit_equal(f.values, idx)
    assert bits_equal(before[..., 28:], f.values[..., 28:])
    # torch.optim.Adam on render_baked_rays
    g = bake_scene("lego", (24, 20, 28), grid_res=32)
    g.values.requires_grad_()
    opt = torch.optim.Adam([g.values], lr=1e-2)
    for i in range(20):
        rays = camera_rays("lego", poses[i % 6])
        rgb, *_ = nb.render_baked_rays(g, rays)
        loss = ((rgb - imgs[i % 6].reshape(-1, 3)) ** 2).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
    assert copies_bit_equal(g.values.detach(), idx)


# ------------------------------------------------------------------------------------------------------------------------
# 3. fine-tuning helps
# ------------------------------------------------------------------------------------------------------------------------
# held-out PSNR gain (dB) against render_image of lego A0 baked at 256^3 after FT_STEPS trainer steps at the default
# rates and 2048 rays per step, measured on an H100 80GB HBM3 at 700 W (29.71 -> 30.85 dB); the test asks for at least
# FT_GAIN_BAR, a margin of less than half the gain below it
FT_STEPS = 300
FT_GAIN_MEASURED = 1.13
FT_GAIN_BAR = 0.6


def test_fine_tuning_raises_heldout_psnr_on_lego():
    import nerf_pytorch_b200 as nb

    f = bake_scene("lego", 256, grid_res=128)
    poses = sphere_poses(44)
    imgs, opts = targets("lego", poses)
    train, held = list(range(0, 44)), [5, 16, 27, 38]
    train = [i for i in train if i not in held]
    p0 = heldout_psnr(f, poses[held], imgs[held])
    t = nb.BakedFieldTrainer(f, imgs[train].contiguous(), poses[train].cuda(), LEGO_CAM[2], opts, rays_per_step=2048, seed=1)
    first = t.step(1).item()
    losses = [t.step(1).item() for _ in range(9)]
    t.step(FT_STEPS - 20)
    last = [t.step(1).item() for _ in range(10)]
    p1 = heldout_psnr(f, poses[held], imgs[held])
    report("lego 256^3 held-out PSNR before / after, loss first / last, peak GiB", FT_STEPS,
           (p0, p1, first, sum(losses) / 9, sum(last) / 10, torch.cuda.max_memory_allocated() / 2 ** 30))
    assert sum(last) / 10 < 0.8 * (first + sum(losses)) / 10
    assert p1 - p0 >= FT_GAIN_BAR, (p0, p1)


def test_fine_tuning_lowers_the_loss_on_fern():
    import nerf_pytorch_b200 as nb

    f = bake_scene("fern", 256, grid_res=128)
    poses = []
    for i in range(8):
        p = torch.eye(4)
        p[0, 3], p[1, 3] = 0.03 * math.cos(i), 0.03 * math.sin(i)
        poses.append(p)
    poses = torch.stack(poses)
    imgs, opts = targets("fern", poses)
    t = nb.BakedFieldTrainer(f, imgs, poses.cuda(), FERN_CAM[2], opts, rays_per_step=2048, seed=2)
    first = sum(t.step(1).item() for _ in range(10)) / 10
    t.step(80)
    last = sum(t.step(1).item() for _ in range(10)) / 10
    report("fern loss first / last", 100, (first, last))
    assert last < 0.8 * first


# ------------------------------------------------------------------------------------------------------------------------
# 4. reproducibility
# ------------------------------------------------------------------------------------------------------------------------
def test_same_seed_same_pixels_and_runs_agree_to_rounding():
    import nerf_pytorch_b200 as nb

    poses = sphere_poses(6)
    imgs, opts = targets("lego", poses)
    runs = []
    for _ in range(2):
        f = bake_scene("lego", (24, 20, 28), grid_res=32)
        t = nb.BakedFieldTrainer(f, imgs, poses.cuda(), LEGO_CAM[2], opts, rays_per_step=1024, seed=5)
        loss = t.step(10).item()
        runs.append((f.values.clone(), t._ids.clone(), t._image.clone(), t._target.clone(), t._rays.clone(), loss))
    (a, ia, ma, ta, ra, la), (b, ib, mb, tb, rb, lb) = runs
    assert bits_equal(ia.view(torch.int32), ib.view(torch.int32)) and int(ma) == int(mb)
    assert bits_equal(ta, tb) and bits_equal(ra, rb)
    close = torch.isclose(a, b, rtol=1e-4, atol=1e-5).double().mean().item()
    report("fraction of values within 1e-4 between runs, losses", "", (close, la, lb))
    assert close >= 0.999 and abs(la - lb) <= 1e-3 * abs(la)
