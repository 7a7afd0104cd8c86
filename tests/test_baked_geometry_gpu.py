"""GPU: normal maps and point queries of baked fields (render_baked(normals=), render_baked_rays(normals=, ndc=),
nb.baked_raw, nb.baked_density_gradient; csrc/baked.cu baked_render_kernel<V, true, kNdc> and baked_query_kernel<V>;
include/nerfb200.h "baked fields: normal maps and point queries").

  1. exact on affine fields: the queried gradient is the slopes, every normal -a / |a| and the map acc (-a / |a|);
  2. against fp64: normal maps, raw values and gradients of random synthetic fields (with and without view directions,
     random, missing and edge rays, both backgrounds) against the fp64 restatement below;
  3. bit-equalities, for fp32, fp16 and 8-bit fields: the normals render's rows are baked_render's (with and without
     early_stop); fp16 / 8-bit normals, raw values and gradients are the float() field's; a transparent prune, rays that
     do not stop and chunking leave the normals the same bits;
  4. against the bake: at the lattice points of a power-of-two box, baked_raw's sigma_raw is the stored value and the
     bits mlp_fwd_pts (impl 1) gives there; points outside the box and in inactive bricks read 0;
  5. NDC: fern's world normal map against the fp64 J^T g oracle, and baked_density_gradient(ndc=) bit for bit the NDC
     query mapped by ndc_grad_to_world;
  6. quality: the mean angle between lego's baked normal map at 256^3 and render_image(normals=True)."""
import math

import pytest
import torch

from helpers import (FERN_CAM, LEGO_CAM, bake_scene, bits_equal, edge_rays, net_at, random_rays, scene_options,
                     scene_pose, shipped_models, sphere_poses, synthetic_field)

pytestmark = pytest.mark.gpu

F32_EPS = 2.0 ** -23


def report(what, ctx, value):
    print(f"[baked-geometry] {what} {ctx}: {value}")


# ------------------------------------------------------------------------------------------------------------------------
# the fp64 oracle: the cell rule in fp32 as the header states it, the gradient and the normal sums in fp64
# ------------------------------------------------------------------------------------------------------------------------
def _cells(field, x):
    """(hit, slot, l, f) of fp32 points x (..., 3) under the renderer's lookup: f the fp32 fractions, exact inputs of
    the fp64 sums."""
    f32 = torch.float32
    lo = torch.tensor(field.bounds[0], dtype=f32, device=x.device)
    hi = torch.tensor(field.bounds[1], dtype=f32, device=x.device)
    res = torch.tensor(field.resolution, device=x.device)
    tc = (x - lo) * (res.to(f32) / (hi - lo))
    inside = ((tc >= 0) & (tc < res.to(f32))).all(-1)
    i = torch.where(inside[..., None], tc, torch.zeros_like(tc)).to(torch.int64).clamp(0, None)
    i = torch.minimum(i, res - 1)
    fr = tc - i.to(f32)
    nb_ = (res + 7) // 8
    b = i // 8
    slot = field.brick_map.long()[((b[..., 2] * nb_[1] + b[..., 1]) * nb_[0] + b[..., 0]).clamp(0, field.brick_map.numel() - 1)]
    return inside & (slot >= 0), slot.clamp_min(0), i % 8, fr


def grad64(field, x, channels=1):
    """(v (..., channels), g (..., 3), cond (..., 3)) in fp64 at fp32 points x: the trilinear interp of the first
    ``channels`` channels, the gradient of channel 0 and, per axis, sum_k |coefficient_k v_k| scale_c (the size of the
    terms the fp32 sum cancels), all 0 for a miss."""
    hit, slot, l, fr = _cells(field, x)
    fr = fr.double()
    vals = field.float().values
    scale = (torch.tensor(field.resolution, dtype=torch.float32) /
             (torch.tensor(field.bounds[1], dtype=torch.float32) - torch.tensor(field.bounds[0], dtype=torch.float32))
             ).double().to(x.device)  # the cell rule's fp32 scale
    v = torch.zeros(*x.shape[:-1], channels, dtype=torch.float64, device=x.device)
    g = torch.zeros(*x.shape, dtype=torch.float64, device=x.device)
    cond = torch.zeros_like(g)
    for k in range(8):
        off = torch.tensor([k & 1, k >> 1 & 1, k >> 2], device=x.device)
        w1 = torch.where(off.bool(), fr, 1 - fr)  # per-axis weights
        lc = l + off
        idx = (lc[..., 2] * 9 + lc[..., 1]) * 9 + lc[..., 0]
        vk = torch.where(hit[..., None], vals[slot, idx][..., :channels].double(), 0.0)
        v += w1.prod(-1, keepdim=True) * vk
        for c in range(3):
            p = w1[..., [a for a in range(3) if a != c]].prod(-1)
            term = (p if (k >> c) & 1 else -p) * vk[..., 0]
            g[..., c] += term
            cond[..., c] += term.abs()
    return v, g * scale, cond * scale


def ndc_sw_sh(cam):
    H, W, focal = cam
    return -1.0 / (float(W) / (2.0 * float(torch.tensor(focal, dtype=torch.float32)))), \
        -1.0 / (float(H) / (2.0 * float(torch.tensor(focal, dtype=torch.float32))))


def to_world64(cam, q, g):
    """J^T(q) g in fp64 at NDC points q, with the NDC map's fp32 sw / sh."""
    sw, sh = (float(torch.tensor(s, dtype=torch.float32)) for s in ndc_sw_sh(cam))
    q = q.double()
    s = (q[..., 2] - 1) * 0.5
    t = q[..., 0] * g[..., 0] + q[..., 1] * g[..., 1]
    return torch.stack([s * sw * g[..., 0], s * sh * g[..., 1], s * (-t - (q[..., 2] - 1) * g[..., 2])], -1)


def normals64(field, rays, cam=None):
    """(normal map (R, 3), acc (R,), error bar (R,)) in fp64: the header's march with fp32 sample points and fp64
    weights, sum of w (-g / |g|) over the hit samples.  The bar of a ray is 3e-5 plus, per sample, w times the normal's
    possible error from the fp32 gradient's cancellation: min(2, 2 |dg| / |g|) with |dg| <= 16 eps cond (and the J^T
    map's own cancellation with a camera)."""
    f32 = torch.float32
    dev = rays.device
    lo = torch.tensor(field.bounds[0], dtype=f32, device=dev)
    hi = torch.tensor(field.bounds[1], dtype=f32, device=dev)
    res = torch.tensor(field.resolution, device=dev)
    o, d = rays[:, :3], rays[:, 3:6]
    t0, t1 = (lo - o) / d, (hi - o) / d
    flat = d == 0
    tmin = torch.where(flat, -math.inf, torch.fmin(t0, t1).nan_to_num(nan=-math.inf))
    tmax = torch.where(flat, math.inf, torch.fmax(t0, t1).nan_to_num(nan=math.inf))
    outside = (flat & ~((o >= lo) & (o < hi))).any(-1)
    ta = torch.fmax(rays[:, 6], tmin.amax(-1))
    tb = torch.where(outside, -math.inf, torch.fmin(rays[:, 7], tmax.amin(-1)))
    h = ((hi - lo) / res.to(f32)).min()
    dn = torch.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    dt = (torch.tensor(0.5, dtype=f32, device=dev) * h) / dn
    live = (ta < tb) & (dt > 0) & (dt < math.inf) & ((tb - ta) / dt < 16777216.0)
    K = int(torch.where(live, (tb - ta) / dt, 0.0).max().item()) + 2
    k = torch.arange(K, device=dev, dtype=f32) + 0.5
    t = ta[:, None] + k[None] * dt[:, None]
    valid = (t < tb[:, None]) & live[:, None]
    t = torch.where(valid, t, 0.0)
    x = o[:, None] + d[:, None] * t[..., None]
    hit = _cells(field, x)[0] & valid
    v, g, cond = grad64(field, x)
    sigma = torch.where(hit, v[..., 0], 0.0)
    alpha = 1 - torch.exp(-torch.relu(sigma) * (dt.double() * dn.double())[:, None])
    alpha = torch.where(valid, alpha, torch.zeros_like(alpha))
    q = 1 - alpha + 1e-10
    T = torch.cat([torch.ones_like(q[:, :1]), torch.cumprod(q, -1)[:, :-1]], -1)
    w = torch.where(hit, alpha * T, 0.0)
    dg = 16 * F32_EPS * cond
    if cam is not None:
        sw, sh = ndc_sw_sh(cam)
        xd = x.double()
        s = ((xd[..., 2] - 1) * 0.5).abs()
        dg = torch.stack([s * abs(sw) * dg[..., 0], s * abs(sh) * dg[..., 1],
                          s * (xd[..., 0].abs() * dg[..., 0] + xd[..., 1].abs() * dg[..., 1]
                               + (xd[..., 2] - 1).abs() * dg[..., 2])], -1)
        mag = s * (abs(sw) * g[..., 0].abs() + abs(sh) * g[..., 1].abs() + xd[..., 0].abs() * g[..., 0].abs()
                   + xd[..., 1].abs() * g[..., 1].abs() + (xd[..., 2] - 1).abs() * g[..., 2].abs())
        g = to_world64(cam, x, g)
        dg = dg + (8 * F32_EPS * mag)[..., None]
    norm = g.norm(dim=-1)
    n = torch.where((norm > 0)[..., None], -g / norm.clamp_min(1e-300)[..., None], 0.0)
    bound = torch.where(norm > 0, (2 * dg.norm(dim=-1) / norm.clamp_min(1e-300)).clamp(max=2.0), 2.0)
    N = (w[..., None] * n).sum(1)
    return N, w.sum(1), 3e-5 + (w * torch.where(hit, bound, 0.0)).sum(1)


def _rays(f, seed, n=1001):
    rays = torch.cat([random_rays(n, seed, f.use_viewdirs, misses=True), edge_rays(f, f.use_viewdirs)])
    assert rays.shape[0] % 4 != 0
    return rays


def _points(field, n, seed):
    """n random fp32 points in the field's box (a few outside it)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    lo = torch.tensor(field.bounds[0], device="cuda")
    hi = torch.tensor(field.bounds[1], device="cuda")
    u = torch.rand(n, 3, generator=g, device="cuda") * 1.1 - 0.05
    return (lo + (hi - lo) * u).contiguous()


FIELDS = {
    "res16": dict(res=(16, 16, 16), seed=1),
    "res24_20_28_half_noview": dict(res=(24, 20, 28), viewdirs=False, active=0.5, seed=2),
    "res13_9_17_third": dict(res=(13, 9, 17), active=0.3, seed=3),
}


def _synthetic(name):
    kw = dict(FIELDS[name])
    return synthetic_field(kw.pop("res"), **kw)


# ------------------------------------------------------------------------------------------------------------------------
# 1. affine fields
# ------------------------------------------------------------------------------------------------------------------------
SLOPES = (0.25, -0.5, 0.75)  # per lattice step


def _affine_field(res=16, bounds=((-1.0,) * 3, (1.0,) * 3)):
    """BakedField.full over a power-of-two box with sigma_raw = a . q + 9 at lattice index q (1 .. 25 at res 16)."""
    import nerf_pytorch_b200 as nb

    f = nb.BakedField.full(bounds, (res,) * 3, use_viewdirs=False)
    nb_ = -(-res // 8)
    br = f.bricks.long()
    b = torch.stack([br % nb_, br // nb_ % nb_, br // (nb_ * nb_)], -1)
    p = torch.arange(729, device="cuda")
    l = torch.stack([p % 9, p // 9 % 9, p // 81], -1)
    q = torch.minimum(b[:, None] * 8 + l[None], torch.tensor(res, device="cuda")).float()
    a = torch.tensor(SLOPES, device="cuda")
    f.values[..., 0] = (q * a).sum(-1) + 9.0  # small integers: exact in fp32
    return f


def test_affine_field_is_exact():
    import nerf_pytorch_b200 as nb

    f = _affine_field()
    scale = 16 / 2.0
    a = torch.tensor(SLOPES, dtype=torch.float64, device="cuda") * scale  # d sigma / dx in the box's units
    vmax = 25.0
    tol = 16 * F32_EPS * vmax * scale  # the fp32 sum's rounding, in ulps of the values it cancels
    pts = _points(f, 4096, 11)
    inside = ((pts > -1) & (pts < 1)).all(-1)
    sigma, grad = nb.baked_density_gradient(f, pts[inside])
    e = (grad.double() - a).abs().max().item()
    report("affine gradient error / bar", "", (e, tol))
    assert e <= tol
    n = -a / a.norm()
    assert ((-grad.double() / grad.double().norm(dim=-1, keepdim=True)) - n).abs().max().item() <= 1e-4
    # the normal map: every sample's normal is -a / |a|, so the map is acc (-a / |a|)
    rays = random_rays(2001, 12, viewdirs=False)
    with torch.no_grad():
        *_, acc, _, nrm = nb.render_baked_rays(f, rays, normals=True)
    assert bool((acc > 0.5).any())
    e = (nrm.double() - acc.double()[:, None] * n).abs().max().item()
    report("affine normal map error", "", e)
    assert e <= 1e-4  # fp32 rounding of the sums and of each sample's direction


# ------------------------------------------------------------------------------------------------------------------------
# 2. against fp64
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(FIELDS))
def test_normal_maps_match_fp64(name):
    import nerf_pytorch_b200 as nb

    f = _synthetic(name)
    rays = _rays(f, 5)
    N64, acc64, bar = normals64(f, rays)
    for white in (False, True):
        with torch.no_grad():
            out = nb.render_baked_rays(f, rays, white_background=white, normals=True)
        e = (out[4].double() - N64).abs().max(-1).values
        report("normal map error / median bar", (name, white), (e.max().item(), bar.median().item()))
        assert bool((e <= bar).all()), (name, white, (e - bar).max().item())
        assert bool((out[4].double().norm(dim=-1) <= out[2].double() + 1e-5).all())  # |N| <= acc
    assert (acc64 > 0.5).sum() > 50


@pytest.mark.parametrize("name", list(FIELDS))
def test_queries_match_fp64(name):
    import nerf_pytorch_b200 as nb

    f = _synthetic(name)
    pts = _points(f, 20000, 7)
    v64, g64, cond = grad64(f, pts, channels=28)
    # raw: sigma_raw and the logits against fp64, each within 16 ulps of the terms summed
    dirs = torch.nn.functional.normalize(torch.randn(pts.shape, device="cuda"), dim=-1) if f.use_viewdirs else None
    raw = nb.baked_raw(f, pts, dirs)
    hit = _cells(f, pts)[0]
    if f.use_viewdirs:
        X, Y, Z = dirs.double().unbind(-1)
        Ysh = torch.stack([torch.full_like(X, 0.28209479177387814), -0.4886025119029199 * Y, 0.4886025119029199 * Z,
                           -0.4886025119029199 * X, 1.0925484305920792 * X * Y, -1.0925484305920792 * Y * Z,
                           0.31539156525252005 * (2 * Z * Z - X * X - Y * Y), -1.0925484305920792 * X * Z,
                           0.5462742152960396 * (X * X - Y * Y)], -1)
    else:
        Ysh = torch.zeros(pts.shape[0], 9, dtype=torch.float64, device="cuda")
        Ysh[:, 0] = 0.28209479177387814
    coef = v64[:, 1:].view(-1, 3, 9)
    s64 = (coef * Ysh[:, None]).sum(-1)
    # bars: the interp's 8 fmaf within 16 ulps of the largest value; a logit sums 9 such coefficients times |Y_j| < 4
    vmax = f.float().values[..., :28].abs().amax((0, 1)).double()
    e_sigma = (raw[:, 3].double() - v64[:, 0]).abs()
    e_s = (raw[:, :3].double() - s64).abs()
    report("raw sigma / logit error", name, (e_sigma.max().item(), e_s.max().item()))
    assert bool((e_sigma <= 16 * F32_EPS * vmax[0]).all())
    assert bool((e_s <= 128 * F32_EPS * vmax[1:].max()).all())
    assert bool((raw[~hit] == 0).all())
    sigma, grad = nb.baked_density_gradient(f, pts)
    assert bits_equal(sigma, raw[:, 3])
    e = (grad.double() - g64).abs()
    report("gradient error / max bar", name, (e.max().item(), (16 * F32_EPS * cond).max().item()))
    assert bool((e <= 16 * F32_EPS * cond + 1e-30).all())
    assert bool((grad[~hit] == 0).all())


# ------------------------------------------------------------------------------------------------------------------------
# 3. bit-equalities
# ------------------------------------------------------------------------------------------------------------------------
def _bits(x):
    return x.contiguous().view(torch.int32).reshape(x.shape[0], -1)


def _formats(f):
    return {"fp32": f, "fp16": f.half(), "u8": f.quantize()}


@pytest.mark.parametrize("name", list(FIELDS))
def test_bit_equalities(name):
    import nerf_pytorch_b200 as nb

    base = _synthetic(name)
    rays = _rays(base, 8)
    pts = _points(base, 5000, 9)
    dirs = torch.nn.functional.normalize(torch.randn(pts.shape, device="cuda"), dim=-1) if base.use_viewdirs else None
    for fmt, f in _formats(base).items():
        w = f.float()
        with torch.no_grad():
            for white in (False, True):
                for stop in (None, 1e-3):
                    a = nb.render_baked_rays(f, rays, white_background=white, early_stop=stop, normals=True)
                    b = nb.render_baked_rays(f, rays, white_background=white, early_stop=stop)
                    for x, y in zip(a[:4], b):  # the normals render's rows are baked_render's
                        assert bits_equal(x, y), (name, fmt, white, stop)
                    c = nb.render_baked_rays(w, rays, white_background=white, early_stop=stop, normals=True)
                    assert bits_equal(a[4], c[4]), (name, fmt, white, stop)  # the float() field's normals
            # rays that do not stop: the normals of stop 0
            full = nb.render_baked_rays(f, rays, normals=True)
            stopped = nb.render_baked_rays(f, rays, early_stop=0.05, normals=True)
            same = torch.stack([(_bits(x) == _bits(y)).all(-1) for x, y in zip(full[:4], stopped[:4])]).all(0)
            report("rays that do not stop", (name, fmt), (int(same.sum()), rays.shape[0]))
            assert bits_equal(full[4][same], stopped[4][same]), (name, fmt)
            # chunks of rays
            parts = torch.cat([nb.render_baked_rays(f, rays[c:c + 333], normals=True)[4]
                               for c in range(0, rays.shape[0], 333)])
            assert bits_equal(parts, full[4]), (name, fmt)
            # a transparent prune
            p = nb.prune_baked(f, ~nb.baked_transparent_bricks(f))
            assert bits_equal(nb.render_baked_rays(p, rays, normals=True)[4], full[4]), (name, fmt)
        # queries: the float() field's bits
        assert bits_equal(nb.baked_raw(f, pts, dirs), nb.baked_raw(w, pts, dirs)), (name, fmt)
        for x, y in zip(nb.baked_density_gradient(f, pts), nb.baked_density_gradient(w, pts)):
            assert bits_equal(x, y), (name, fmt)


def test_render_baked_normals_keeps_the_image():
    import nerf_pytorch_b200 as nb

    f = bake_scene("lego", 64, 64)
    H, W, focal = LEGO_CAM
    opts = scene_options("lego")
    pose = scene_pose("spherical")
    for stop in (None, 1e-3):
        a = nb.render_baked(f, H, W, focal, pose, opts, early_stop=stop)
        b = nb.render_baked(f, H, W, focal, pose, opts, early_stop=stop, normals=True)
        c = nb.render_baked(f, H, W, focal, pose, opts, early_stop=stop, normals="world")
        assert len(b) == 4 and b[3].shape == (H, W, 3)
        for x, y in zip(a, b):
            assert bits_equal(x, y), stop
        assert bits_equal(b[3], c[3]), stop  # a Blender field: "world" is the field's frame
        assert nb.cast_to_normal_image(b[3]).shape == (H, W, 3)


# ------------------------------------------------------------------------------------------------------------------------
# 4. against the bake
# ------------------------------------------------------------------------------------------------------------------------
def _lattice_points(field, n, seed):
    """(points (n, 3) fp32, lattice indices q (n, 3)) of random lattice points below the upper faces."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    res = torch.tensor(field.resolution, device="cuda")
    q = (torch.rand(n, 3, generator=g, device="cuda") * res).long().clamp(max=res - 1)
    lo = torch.tensor(field.bounds[0], device="cuda")
    hi = torch.tensor(field.bounds[1], device="cuda")
    return (lo + q.float() * ((hi - lo) / res.float())).contiguous(), q


def _stored_sigma(field, q):
    """sigma_raw stored at lattice index q (n, 3) in its brick's copy, NaN where the brick is inactive."""
    res = torch.tensor(field.resolution, device="cuda")
    nb_ = (res + 7) // 8
    b, l = q // 8, q % 8
    slot = field.brick_map.long()[(b[:, 2] * nb_[1] + b[:, 1]) * nb_[0] + b[:, 0]]
    v = field.values[slot.clamp_min(0), (l[:, 2] * 9 + l[:, 1]) * 9 + l[:, 0], 0]
    return torch.where(slot >= 0, v, torch.nan), slot >= 0


def _lego_pow2():
    import nerf_pytorch_b200 as nb

    _, mf, epf, edf = shipped_models("lego")
    box = ((-2.0,) * 3, (2.0,) * 3)  # res 64: scale 16, every lattice point at fractions 0
    grid = nb.OccupancyGrid.from_models([mf], epf, box, 64, encode_direction_fn=edf)
    return nb.bake(mf, epf, edf, bounds=box, resolution=64, grid=grid), mf, epf, edf


@pytest.mark.parametrize("kind", ["noview", "lego_pow2"])
def test_lattice_points_read_the_bake(kind):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import mesh, train_utils

    if kind == "noview":
        f = bake_scene("noview", 64)
        torch.manual_seed(7)  # bake_scene's network
        m = nb.FlexibleNeRFModel(num_layers=4, hidden_size=128, skip_connect_every=4, num_encoding_fn_xyz=10,
                                 use_viewdirs=False).cuda()
        epf, edf = nb.get_embedding_function(10), None
    else:
        f, m, epf, edf = _lego_pow2()
    pts, q = _lattice_points(f, 20000, 3)
    stored, active = _stored_sigma(f, q)
    dirs = torch.nn.functional.normalize(torch.randn(pts.shape, device="cuda"), dim=-1) if f.use_viewdirs else None
    raw = nb.baked_raw(f, pts, dirs)
    report("lattice points in active / inactive bricks", kind, (int(active.sum()), int((~active).sum())))
    assert bool(active.any())
    assert bits_equal(raw[active, 3], stored[active]), kind
    assert bool((raw[~active] == 0).all()), kind
    arch = mesh._network(m, epf, edf)
    blob = train_utils._packed(m, arch)[1]
    net = net_at(arch, blob, pts[active], None if edf is None else torch.tensor([0.0, 0.0, 1.0], device="cuda"))
    assert bits_equal(raw[active, 3], net[:, 3]), kind
    # outside the box: zeros, gradient 0
    out = pts[:64] + torch.tensor(f.bounds[1], device="cuda") - torch.tensor(f.bounds[0], device="cuda")
    sigma, grad = nb.baked_density_gradient(f, out)
    assert bool((sigma == 0).all()) and bool((grad == 0).all())
    assert bool((nb.baked_raw(f, out, dirs[:64] if dirs is not None else None) == 0).all())


# ------------------------------------------------------------------------------------------------------------------------
# 5. NDC
# ------------------------------------------------------------------------------------------------------------------------
def test_ndc_world_normals_and_gradients():
    import importlib

    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    B = importlib.import_module("nerf_pytorch_b200.bake")  # the package's name bake is the function

    f = bake_scene("fern", 256)
    H, W, focal = FERN_CAM
    opts = scene_options("fern")
    pose = scene_pose("eye")
    img = nb.render_baked(f, H, W, focal, pose, opts, normals="world")
    rays = B._pose_rays(f, H, W, focal, pose, opts)
    N64, acc64, bar = normals64(f, rays, cam=FERN_CAM)
    e = (img[3].reshape(-1, 3).double() - N64).abs().max(-1).values
    report("fern world normal map error / median bar / pixels acc > 0.5", "",
           (e.max().item(), bar.median().item(), int((acc64 > 0.5).sum())))
    assert bool((e <= bar).all()), (e - bar).max().item()
    ndc_map = nb.render_baked(f, H, W, focal, pose, opts, normals=True)[3]
    assert not bits_equal(ndc_map, img[3])
    with torch.no_grad():  # the rays' form: ndc= gives the same world map
        assert bits_equal(nb.render_baked_rays(f, rays, normals=True, ndc=FERN_CAM)[4], img[3].reshape(-1, 3))
    # world points in front of the camera: N^-1 of points inside the NDC box
    q = _points(f, 8192, 4)
    q[:, 2] = q[:, 2].clamp(-0.99, 0.95)
    sw, sh = (float(torch.tensor(s, dtype=torch.float32)) for s in ndc_sw_sh(FERN_CAM))
    pz = 2.0 / (q[:, 2] - 1.0)
    p = torch.stack([q[:, 0] * pz / sw, q[:, 1] * pz / sh, pz], -1).contiguous()
    sigma, grad = nb.baked_density_gradient(f, p, ndc=FERN_CAM)
    cam = ops.ndc_struct(*FERN_CAM)
    qq = ops.ndc_from_world(cam, p)
    raw, g = ops.baked_query(f.box(), f.brick_map, f.values, False, qq)
    rows = torch.cat([raw[:, 3:], g], 1)
    ops.ndc_grad_to_world(cam, qq, rows, out=rows)
    assert bits_equal(sigma, rows[:, 0]) and bits_equal(grad, rows[:, 1:].contiguous())
    assert bool((grad != 0).any())


# ------------------------------------------------------------------------------------------------------------------------
# 6. quality against the network
# ------------------------------------------------------------------------------------------------------------------------
HELD = (5, 16, 27, 38)  # the held-out views of the fp16 and 8-bit quality tests
# mean angle (degrees) between the baked normal map of lego at 256^3 (grid of both networks, 128^3) and render_image's
# normal map, over the pixels with acc > 0.5 in both, at the 4 held-out 48 x 48 views: 15.77 (median 11.68, 2906 pixels),
# measured on an H100 80GB HBM3 at 700 W (DESIGN §4).  The baked map is the gradient of a trilinear field one cube wide,
# the network's that of its MLP.  The bar sits a little above the measured figure.
ANGLE_BAR_DEG = 17.0


def test_normal_angle_against_the_network():
    import nerf_pytorch_b200 as nb

    mc, mf, epf, edf = shipped_models("lego")
    f = bake_scene("lego", 256, 128, grid_from="both")
    H, W, focal = LEGO_CAM
    opts = scene_options("lego")
    angles, pixels = [], 0
    with torch.no_grad():
        for p in sphere_poses(44)[list(HELD)]:
            _, _, acc_b, nb_map = nb.render_baked(f, H, W, focal, p, opts, normals=True)
            net = nb.render_image(H, W, focal, p, mc, mf, opts, encode_position_fn=epf, encode_direction_fn=edf,
                                  impl=1, normals=True)
            acc_n, nn_map = net[5], net[6]
            m = (acc_b > 0.5) & (acc_n > 0.5)
            a = torch.nn.functional.normalize(nb_map[m].double(), dim=-1)
            b = torch.nn.functional.normalize(nn_map[m].double(), dim=-1)
            angles.append(torch.rad2deg(torch.acos((a * b).sum(-1).clamp(-1, 1))))
            pixels += int(m.sum())
    ang = torch.cat(angles)
    report("mean / median angle (deg) against render_image, pixels", f.n_active,
           (ang.mean().item(), ang.median().item(), pixels))
    assert pixels > 1000
    assert ang.mean().item() <= ANGLE_BAR_DEG
