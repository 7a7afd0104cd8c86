"""GPU: baked fields across the architecture table, on CTAs that run several tiles, and at the baked renderer's edge rays
(csrc/mlp_tc.cu bake_tc_kernel, csrc/baked.cu baked_render_kernel; include/nerfb200.h "baked fields").

  1. every architecture of mlp_checks.ALL_ARCHS (hidden 128) and H256_ARCHS (hidden 256) that ops.bake_refusal takes,
     weights "init" and "scaled", on a box with a partial brick on every axis under a random partial occupancy grid:
     sigma_raw and the logits hook at all 64 directions bit-equal mlp_fwd_pts(impl=1) at the mesh_sparse_points lattice
     points; sigma_raw and the logits at sampled points within TC_FWD_TOL of the fp64 oracle per column scale; the SH
     coefficients within COEF_REL of the fp64 projection; columns 28..31 zero; slots outside the window and logits rows
     past it untouched.  8x256_ldir6 (39 direction channels) is refused before any launch;
  2. persistent launches: more than twice as many tiles as multiprocessors, so that every CTA runs at least two tiles,
     with a ragged last tile and a non-zero first slot; two calls over disjoint slot windows give the bits of one call
     over their union, and a repeat gives the same bits;
  3. a large anisotropic lattice, (4096, 24, 9), baked on a few bricks at its far corner: the points are the lattice
     rule's and the bake is the network's there;
  4. the renderer on synthetic values (no network) against helpers.baked_render64: axis-parallel rays with +-0
     components from outside, inside and on the face, lattice and brick planes; rays through corners and along edges;
     origins inside with near 0; diagonal rays of at least 14 rounds; rays with d = 0, NaN or near >= far, which render
     empty.  Early stopping at t = 1e-2 keeps the per-ray contract of test_bake_gpu;
  5. the case lists reach what they are there for (several tiles per CTA, a ragged tile, wide and linear encodings,
     partial bricks, flat rays in the lower face plane).
Run with -s to print the measured figures beside their bars.  Measured on an H100 80GB HBM3 at 700 W: raw against fp64
at most 1.2e-5 of the column scale (10x256 "scaled"; bar TC_FWD_TOL 3e-5), coefficients 2.0e-6 (8x256 "scaled"; bar
COEF_REL 4e-6), the renderer 5.4e-6 (acc of the corner rays; bar OUT_ABS 1e-5).  The file runs in about 20 s with a peak
of 0.45 GiB of device memory allocated."""
import math

import numpy as np
import pytest
import torch

import mlp_checks as M
from helpers import COEF_REL, OUT_ABS, baked_render64, bits_equal, net_at
from mlp_checks import ALL_ARCHS, H256_ARCHS, STATES, TC_FWD_TOL

pytestmark = pytest.mark.gpu

ARCHS = list(ALL_ARCHS) + list(H256_ARCHS)
# a partial brick on every axis (20 = 2 x 8 + 4, 17 = 2 x 8 + 1, 33 = 4 x 8 + 1), spacings that are not powers of two
SWEEP_BOUNDS = ((-1.1, -0.9, -1.3), (0.9, 1.2, 1.0))
SWEEP_RES = (20, 17, 33)
# hidden-128 and hidden-256 networks with and without view directions for the persistent launches
PERSIST = ["8x128_widest", "4x128_noview", "8x256", "8x256_noview"]
PERSIST_BOUNDS = ((-1.0,) * 3, (1.0,) * 3)
PERSIST_RES = (72, 40, 48)  # 9 x 5 x 6 = 270 bricks
PERSIST_FIRST = 11
# a large anisotropic lattice: 512 x 3 x 2 bricks, the last ones partial on z
BIG_BOUNDS = ((-2.0, -0.5, -0.3), (2.5, 0.7, 0.4))
BIG_RES = (4096, 24, 9)
BIG_BRICKS = [(511, 2, 1), (510, 2, 1), (511, 1, 1), (511, 2, 0), (509, 0, 1)]
# the renderer's box: spacings 1/64, 1/32, 1/64 (h = 1/64), so that lattice and brick planes are exact in fp32
EDGE_BOUNDS = ((-1.0,) * 3, (1.0,) * 3)
EDGE_RES = (128, 64, 128)
STOP_T = 1e-2


def report(what, ctx, value):
    print(f"[bake sweep] {what} {ctx}: {value}")


def _rows(hidden):
    """Lattice points per CTA tile of the bake: 3 consumer warpgroups at hidden 128, one at 256."""
    return 192 if hidden == 128 else 64


def persist_count(hidden):
    """Bricks of a persistent launch: 2.5 x as many tiles as multiprocessors, rounded up to whole bricks."""
    return -(-5 * M.sms() * _rows(hidden) // (2 * 729))


def _setup(name, state):
    from nerf_pytorch_b200 import ops

    arch = M.spec(name)
    sd = M.arch_weights(arch, state)
    return arch, sd, ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))


def _sweep_grid():
    """A random partial occupancy grid over the sweep box: a few occupied cells of 16^3."""
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    g = torch.Generator().manual_seed(5)
    return OccupancyGrid.from_occupancy(SWEEP_BOUNDS, (torch.rand(16, 16, 16, generator=g) < 0.002).cuda())


def _network_bits(arch, blob, pts, got, logits, ctx):
    """sigma_raw (got[:, 0]) and the logits hook bit-equal mlp_fwd_pts(impl=1) at pts, every direction."""
    from nerf_pytorch_b200 import ops

    dirs, _ = ops.bake_basis()
    P = pts.shape[0]
    want_sigma = net_at(arch, blob, pts, dirs[0].cuda() if arch.use_viewdirs else None)[:, 3]
    assert bits_equal(got[:, 0], want_sigma), ctx
    if arch.use_viewdirs:
        for d in range(64):
            assert bits_equal(logits[:, d], net_at(arch, blob, pts, dirs[d].cuda())[:, :3]), ctx + (d,)
    else:
        raw = net_at(arch, blob, pts, None)
        assert bits_equal(logits, raw[:, None, :3].expand(P, 64, 3)), ctx


def _coef_error(arch, got, logits):
    """max |c - c64| / max |logit| of the point, c64 the fp64 projection of the kernel's own logits."""
    from nerf_pytorch_b200 import ops

    _, proj = ops.bake_basis()
    P = got.shape[0]
    if arch.use_viewdirs:
        coef64 = torch.einsum("jd,pdc->pcj", proj.double().cuda(), logits.double())
    else:
        coef64 = torch.zeros(P, 3, 9, dtype=torch.float64, device="cuda")
        coef64[:, :, 0] = logits[:, 0].double() / np.float32(0.28209479177387814)
    scale = logits.abs().amax(dim=(1, 2)).double()[:, None]
    return ((got[:, 1:28].double().view(P, 3, 9) - coef64).abs().view(P, 27) / scale.clamp_min(1e-30)).max().item()


# ------------------------------------------------------------------------------------------------------------------------
# 1. the architecture table
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("name", ARCHS)
def test_bake_across_the_architecture_table(name, state):
    from nerf_pytorch_b200 import ops

    arch, sd, blob = _setup(name, state)
    box = ops.grid_struct(SWEEP_BOUNDS, SWEEP_RES)
    brick_map, bricks, n = ops.mesh_sparse_bricks(box, _sweep_grid())
    n = int(n.item())
    ctx = (name, state)
    why = ops.bake_refusal(arch)
    if why is not None:
        assert name == "8x256_ldir6", (name, why)  # its 39 direction channels: the wgmma forward's refusal
        before = ops.launch_count()
        values = torch.full((n, 729, 32), float("nan"), device="cuda")
        with pytest.raises(NotImplementedError):
            ops.bake(arch, blob, box, bricks, 0, n, values)
        assert ops.launch_count() == before and torch.isnan(values).all()
        return
    assert 4 <= n < brick_map.numel(), n
    first, count = 1, n - 2
    P = count * 729
    values = torch.full((n, 729, 32), float("nan"), device="cuda")
    logits = torch.full((P + 500, 64, 3), float("nan"), device="cuda")
    ops.bake(arch, blob, box, bricks, first, count, values, logits)
    pts = torch.empty(P, 3, device="cuda")
    ops.mesh_sparse_points(box, bricks, first, count, False, pts)
    got = values[first:first + count].reshape(P, 32)
    _network_bits(arch, blob, pts, got, logits[:P], ctx)
    assert torch.isnan(logits[P:]).all(), ctx
    assert (got[:, 28:] == 0).all(), ctx
    untouched = torch.ones(n, dtype=torch.bool, device="cuda")
    untouched[first:first + count] = False
    assert torch.isnan(values[untouched]).all(), ctx

    # sigma_raw and the logits against the fp64 oracle at sampled points: rays o = p, d = 0, z = 0 give the points p
    g = torch.Generator().manual_seed(len(name))
    idx = torch.randperm(P, generator=g)[:3000].cuda()
    m = idx.numel()
    sd_dev = {k: v.cuda() for k, v in sd.items()}
    worst = 0.0
    for d in ((0, 21, 42, 63) if arch.use_viewdirs else (0,)):
        dirs, _ = ops.bake_basis()
        rays = torch.cat([pts[idx], torch.zeros(m, 3, device="cuda"), torch.zeros(m, 1, device="cuda"),
                          torch.ones(m, 1, device="cuda"), dirs[d].cuda().expand(m, 3)], -1)
        want = M.oracle(arch, sd_dev, rays if arch.use_viewdirs else rays[:, :8], torch.zeros(m, 1, device="cuda"))[0]
        have = torch.cat([logits[idx, d], got[idx, :1]], -1).double()
        scale = want.abs().amax(0)
        e = (have - want).abs().amax(0)
        worst = max(worst, (e / scale).max().item())
        assert (e <= TC_FWD_TOL * scale).all(), ctx + (d, e.tolist(), scale.tolist())
    err = _coef_error(arch, got, logits[:P])
    report(f"worst raw / column scale vs fp64 (bar TC_FWD_TOL {TC_FWD_TOL}), coefficient error / max |logit| "
           f"(bar COEF_REL {COEF_REL})", ctx + (count,), f"{worst:.3e}, {err:.3e}")
    assert err <= COEF_REL, ctx + (err,)


# ------------------------------------------------------------------------------------------------------------------------
# 2. persistent launches
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", PERSIST)
def test_persistent_bake_runs_several_tiles_per_cta(name):
    from nerf_pytorch_b200 import ops
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    arch, sd, blob = _setup(name, "scaled")
    box = ops.grid_struct(PERSIST_BOUNDS, PERSIST_RES)
    brick_map, bricks, n = ops.mesh_sparse_bricks(box, OccupancyGrid.full(PERSIST_BOUNDS, 8))
    n = int(n.item())
    first, count = PERSIST_FIRST, persist_count(arch.hidden)
    assert first + count <= n, (first, count, n)
    P = count * 729
    ctx = (name, count, -(-P // _rows(arch.hidden)), M.sms())

    def baked(f, c, into=None, logits=None):
        v = torch.full((n, 729, 32), float("nan"), device="cuda") if into is None else into
        return ops.bake(arch, blob, box, bricks, f, c, v, logits)

    logits = torch.empty(P, 64, 3, device="cuda")
    values = baked(first, count, logits=logits)
    pts = torch.empty(P, 3, device="cuda")
    ops.mesh_sparse_points(box, bricks, first, count, False, pts)
    got = values[first:first + count].reshape(P, 32)
    _network_bits(arch, blob, pts, got, logits, ctx)
    err = _coef_error(arch, got, logits)
    report(f"coefficient error / max |logit| (bar COEF_REL {COEF_REL}), (bricks, tiles, SMs)", ctx, f"{err:.3e}")
    assert err <= COEF_REL and (got[:, 28:] == 0).all(), ctx
    outside = torch.ones(n, dtype=torch.bool, device="cuda")
    outside[first:first + count] = False
    assert torch.isnan(values[outside]).all(), ctx
    # two disjoint windows, the first ending mid-tile, are the union's bits; a repeat is the same bits
    split = count // 3
    parts = baked(first, split)
    baked(first + split, count - split, into=parts)
    assert bits_equal(parts, values), ctx
    assert bits_equal(baked(first, count), values), ctx


# ------------------------------------------------------------------------------------------------------------------------
# 3. a large anisotropic lattice
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["8x128_widest", "8x256"])
def test_bake_on_a_large_anisotropic_lattice(name):
    from nerf_pytorch_b200 import ops

    arch, sd, blob = _setup(name, "scaled")
    box = ops.grid_struct(BIG_BOUNDS, BIG_RES)
    nb_ = [-(-r // 8) for r in BIG_RES]
    assert ops.mesh_sparse_brick_count(box) == nb_[0] * nb_[1] * nb_[2]
    ids = [(z * nb_[1] + y) * nb_[0] + x for x, y, z in BIG_BRICKS]
    bricks = torch.tensor(ids, dtype=torch.int32, device="cuda")
    count = len(ids)
    P = count * 729
    values = torch.full((count, 729, 32), float("nan"), device="cuda")
    logits = torch.empty(P, 64, 3, device="cuda")
    ops.bake(arch, blob, box, bricks, 0, count, values, logits)
    pts = torch.empty(P, 3, device="cuda")
    ops.mesh_sparse_points(box, bricks, 0, count, False, pts)
    # the lattice rule: p_c = lo_c + ((hi_c - lo_c) i_c) / res_c in fp32, i = 8 b + l clamped onto 0 .. res
    l = torch.arange(729, device="cuda")
    lc = torch.stack([l % 9, l // 9 % 9, l // 81], -1)
    bc = torch.tensor(BIG_BRICKS, device="cuda")
    res = torch.tensor(BIG_RES, device="cuda")
    i = torch.minimum(bc[:, None] * 8 + lc[None], res).reshape(P, 3).float()
    lo, hi = (torch.tensor(b, dtype=torch.float32, device="cuda") for b in BIG_BOUNDS)
    assert bits_equal(pts, lo + ((hi - lo) * i) / res.float()), name
    got = values.reshape(P, 32)
    _network_bits(arch, blob, pts, got, logits, (name,))
    assert _coef_error(arch, got, logits) <= COEF_REL and (got[:, 28:] == 0).all()


# ------------------------------------------------------------------------------------------------------------------------
# 4. the renderer's edge rays
# ------------------------------------------------------------------------------------------------------------------------
def _edge_field(use_viewdirs):
    """A synthetic field over the edge box: 30 % of the bricks active; sigma_raw (N(0, 1) + b) s with a per-brick offset
    b in [-2, 1) (mostly empty to mostly dense) and scale s from 0.1 to 1e3 (alpha from ~1e-3 to 1 per sample), so that
    rays range from transparent to opaque; coefficients N(0, 2^2); columns 28..31 zero."""
    import nerf_pytorch_b200 as nb

    g = torch.Generator().manual_seed(11)
    n_bricks = math.prod(-(-r // 8) for r in EDGE_RES)
    active = torch.rand(n_bricks, generator=g) < 0.3
    brick_map = torch.full((n_bricks,), -1, dtype=torch.int32)
    brick_map[active] = torch.arange(int(active.sum()), dtype=torch.int32)
    n = int(active.sum())
    values = torch.zeros(n, 729, 32)
    scale = 10.0 ** (torch.rand(n, 1, generator=g) * 4 - 1)
    offset = torch.rand(n, 1, generator=g) * 3 - 2
    values[:, :, 0] = (torch.randn(n, 729, generator=g) + offset) * scale
    values[:, :, 1:28] = torch.randn(n, 729, 27, generator=g) * 2
    bricks = torch.nonzero(active).reshape(-1).int()
    return nb.BakedField(EDGE_BOUNDS, EDGE_RES, brick_map.cuda(), bricks.cuda(), values.cuda(), use_viewdirs)


def edge_rays():
    """(rays [n, 11] fp32 on the CPU, kinds: list of n names).  Kinds: "empty" (d = 0, NaN components, near >= far),
    which must render nothing; else "flat_lo", a ray with some d_c = +-0 in the lower face plane of c (o_c = lo_c),
    "flat" the other axis-parallel rays, "corner", "edge", "inside" and "diagonal"."""
    f32 = np.float32
    g = np.random.default_rng(13)
    lo, hi = f32(-1.0), f32(1.0)
    spacing = [f32(2.0) / f32(r) for r in EDGE_RES]
    rows, kinds = [], []

    def add(o, d, near, far, kind, vd=None):
        d = np.asarray(d, dtype=f32)
        if vd is None:
            nrm = np.sqrt((d.astype(np.float64) ** 2).sum())
            vd = d / f32(nrm) if nrm > 0 and np.isfinite(nrm) else np.array([0, 0, 1], dtype=f32)
        o = np.asarray(o, dtype=f32)
        if kind != "empty" and ((d == 0) & (o == lo)).any():
            kind = "flat_lo"
        rows.append(np.concatenate([o, d, [f32(near), f32(far)], np.asarray(vd, dtype=f32)]))
        kinds.append(kind)

    # axis-parallel rays along axis a, the other two components +-0, at cross coordinates on planes of interest
    for a in range(3):
        k1, k2 = [c for c in range(3) if c != a]

        def cross(k):
            s = spacing[k]
            return [("lo", lo), ("hi", hi), ("below_lo", np.nextafter(lo, f32(-2))), ("below_hi", np.nextafter(hi, lo)),
                    ("lattice", lo + 5 * s), ("brick", lo + 8 * s), ("mid_brick", f32(0.0)), ("top_cube", hi - s),
                    ("random", f32(g.uniform(-0.95, 0.95)))]

        pairs = [(v, ("random", f32(g.uniform(-0.95, 0.95)))) for v in cross(k1)]
        pairs += [(("random", f32(g.uniform(-0.95, 0.95))), v) for v in cross(k2)]
        pairs += [(("lo", lo), ("lo", lo)), (("lo", lo), ("hi", hi)), (("hi", hi), ("lo", lo)), (("hi", hi), ("hi", hi))]
        for s in (1, -1):
            for start in ("outside", "inside", "lo", "hi"):
                for j, ((_, v1), (_, v2)) in enumerate(pairs):
                    mag = f32((1.0, 0.3, 2.5)[j % 3])
                    zero = f32(-0.0) if j % 2 else f32(0.0)
                    d = [zero, zero, zero]
                    d[a] = f32(s) * mag
                    o = [f32(0), f32(0), f32(0)]
                    o[k1], o[k2] = v1, v2
                    o[a] = {"outside": f32(-1.5 * s), "inside": f32(g.uniform(-0.9, 0.9)), "lo": lo, "hi": hi}[start]
                    add(o, d, 0.0, 4.0 / mag, "flat")
    # rays through the corners (the opposite corner too) and rays along the 12 edges
    for c in range(8):
        sgn = np.array([1 if c >> k & 1 else -1 for k in range(3)], dtype=f32)
        add(sgn + f32(0.5) * sgn, -sgn, 0.0, 5.0, "corner")
        side = np.array([1, -1, 0], dtype=f32) * sgn
        add(sgn + f32(0.25) * side, -side, 0.0, 2.0, "corner")  # grazing the corner in its z face plane
    for a in range(3):
        k1, k2 = [c for c in range(3) if c != a]
        for v1 in (lo, hi):
            for v2 in (lo, hi):
                o = [f32(0)] * 3
                o[k1], o[k2], o[a] = v1, v2, f32(-1.5)
                d = [f32(0)] * 3
                d[a] = f32(1)
                add(o, d, 0.0, 4.0, "edge")
    # origins inside the box, near 0
    for _ in range(96):
        d = g.standard_normal(3).astype(f32) * f32(g.uniform(0.3, 3.0))
        add(g.uniform(-1, 1, 3).astype(f32), d, 0.0, 3.0 / float(np.linalg.norm(d)), "inside")
    # diagonals through the box: about 443 samples, 14 rounds of 32
    for _ in range(24):
        sgn = g.choice([-1.0, 1.0], 3).astype(f32)
        d = (sgn + g.normal(0, 0.01, 3)).astype(f32)
        d /= f32(np.linalg.norm(d))
        add(-f32(1.25) * sgn + g.normal(0, 0.01, 3).astype(f32), d, 0.0, 6.0, "diagonal")
    # degenerate rays: no sample
    nan = f32(np.nan)
    add([0.1, 0.2, 0.3], [0, 0, 0], 0.0, 4.0, "empty")
    add([0.1, -0.2, 0.3], [-0.0, 0.0, -0.0], 0.0, 4.0, "empty")
    add([-1.0, -1.0, -1.0], [0, 0, 0], 0.0, 4.0, "empty")    # on the box's lower corner
    add([nan, 0.2, 0.3], [1, 0.5, 0.25], 0.0, 4.0, "empty")
    add([0.2, nan, -1.5], [0, 0, 1], 0.0, 4.0, "empty")         # NaN origin on a flat axis
    add([0.2, 0.1, -1.5], [0.1, nan, 1], 0.0, 4.0, "empty")
    add([-1.5, 0.1, 0.2], [1, 0, 0], 1.0, 1.0, "empty")         # near = far
    add([-1.5, 0.1, 0.2], [1, 0, 0], 3.0, 1.0, "empty")         # near > far
    add([-1.5, 0.1, 0.2], [1, 0.2, 0.1], 2.0, 0.5, "empty")
    add([0.3, -0.3, 0.3], [0.5, 0.5, -0.5], 0.0, 0.0, "empty")  # near = far = 0 inside the box
    return torch.from_numpy(np.stack(rows)), kinds


@pytest.mark.parametrize("white", [False, True])
@pytest.mark.parametrize("use_viewdirs", [True, False])
def test_renderer_at_edge_rays(use_viewdirs, white):
    from nerf_pytorch_b200 import ops

    field = _edge_field(use_viewdirs)
    rays, kinds = edge_rays()
    rays = (rays if use_viewdirs else rays[:, :8]).contiguous().cuda()
    kinds = np.array(kinds)
    ctx = (use_viewdirs, white)
    out = ops.baked_render(field.box(), field.brick_map, field.values, use_viewdirs, rays, white)
    assert torch.isfinite(out[:, [0, 1, 2, 4, 5]]).all() and (out[:, 6:] == 0).all(), ctx
    rgb, acc, depth, disp = baked_render64(field, rays, white)
    far = float(rays[:, 7].max())
    e_rgb = (out[:, :3].double() - rgb).abs().amax(-1)
    e_acc = (out[:, 4].double() - acc).abs()
    e_depth = (out[:, 5].double() - depth).abs() / far
    for kind in sorted(set(kinds)):
        sel = torch.from_numpy(kinds == kind).cuda()
        report(f"{kind}: rays, opaque, rgb / acc / depth error (bar OUT_ABS {OUT_ABS})", ctx,
               (int(sel.sum()), int((acc[sel] > 0.99).sum()), f"{e_rgb[sel].max().item():.2e}",
                f"{e_acc[sel].max().item():.2e}", f"{e_depth[sel].max().item():.2e}"))
    bad = (e_rgb > OUT_ABS) | (e_acc > OUT_ABS) | (e_depth > OUT_ABS)
    assert not bad.any(), ctx + ([(kinds[i], rays[i].tolist(), out[i].tolist(), acc[i].item())
                                  for i in bad.nonzero().reshape(-1)[:4].tolist()],)
    empty = acc == 0
    assert torch.isnan(out[empty, 3]).all(), ctx
    ok = acc > 1e-3
    assert torch.allclose(out[ok, 3].double(), disp[ok], rtol=1e-3), ctx
    # the degenerate rays: nothing, exactly
    deg = torch.from_numpy(kinds == "empty").cuda()
    bg = 1.0 if white else 0.0
    assert (out[deg, 4] == 0).all() and (out[deg, :3] == bg).all() and (out[deg, 5] == 0).all(), ctx
    assert torch.isnan(out[deg, 3]).all(), ctx
    # not vacuous: flat rays in a lower face plane that cross active bricks, opaque rays, long rays
    flat_lo = torch.from_numpy(kinds == "flat_lo").cuda()
    assert bool((out[flat_lo, 4] > 0).any()), ctx
    assert bool((acc > 0.99).any()) and bool(((acc > 0) & (acc < 0.5)).any()), ctx

    # early stopping: the per-ray contract against t = 0
    e = ops.baked_render(field.box(), field.brick_map, field.values, use_viewdirs, rays, white, STOP_T)
    same = (e == out).all(-1) | (((e[:, 3] != e[:, 3]) & (out[:, 3] != out[:, 3])) &
                                 (e[:, [0, 1, 2, 4, 5]] == out[:, [0, 1, 2, 4, 5]]).all(-1))
    stopped = ~same
    report("rays stopped at t = 1e-2", ctx, int(stopped.sum()))
    assert bool(stopped.any()) and bool(same.any()), ctx
    d = e[stopped] - out[stopped]
    lo_rgb, hi_rgb = (-1e-6, STOP_T + 1e-6) if white else (-STOP_T - 1e-6, 1e-6)
    assert ((d[:, :3] >= lo_rgb) & (d[:, :3] <= hi_rgb)).all(), ctx
    assert ((d[:, 4] <= 1e-6) & (d[:, 4] >= -STOP_T - 1e-6)).all(), ctx
    assert (out[stopped, 4] >= 1 - STOP_T - 1e-5).all(), ctx  # a ray stops only once it is nearly opaque
    assert (e[deg, 4] == 0).all() and torch.isnan(e[deg, 3]).all(), ctx


# ------------------------------------------------------------------------------------------------------------------------
# 5. what the case lists reach
# ------------------------------------------------------------------------------------------------------------------------
def test_the_case_lists_reach_the_bake_edges():
    """The persistent launches give every CTA two tiles or more at each hidden size with a ragged last tile; the sweep
    takes a direction encoding wider than 27 channels and linear xyz bands without the raw input, on a box with a partial
    brick on every axis; the edge rays include a flat ray in a lower face plane that the restatement renders."""
    from nerf_pytorch_b200 import ops

    for hidden in (128, 256):
        name = next(n for n in PERSIST if M.spec(n).hidden == hidden)
        count = persist_count(hidden)
        tiles = -(-count * 729 // _rows(hidden))
        report("bricks, tiles, SMs", (name,), (count, tiles, M.sms()))
        assert tiles >= 2 * M.sms() and (count * 729) % _rows(hidden) != 0 and PERSIST_FIRST > 0, (hidden, count)
    taken = [M.spec(n) for n in ARCHS if ops.bake_refusal(M.spec(n)) is None]
    assert any(a.use_viewdirs and a.dim_dir > 27 for a in taken)
    assert any(not a.include_input_xyz and not a.log_sampling_xyz for a in taken)
    assert {a.hidden for a in taken} == {128, 256} and any(not a.use_viewdirs for a in taken)
    assert all(r % 8 for r in SWEEP_RES)
    rays, kinds = edge_rays()
    d, o = rays[:, 3:6], rays[:, :3]
    lo = torch.tensor(EDGE_BOUNDS[0])
    flat_lo = ((d == 0) & (o == lo)).any(-1) & torch.tensor([k != "empty" for k in kinds])
    assert (flat_lo == torch.tensor([k == "flat_lo" for k in kinds])).all()
    field = _edge_field(True)
    _, acc, _, _ = baked_render64(field, rays.cuda(), False)
    assert bool((acc[flat_lo.cuda()] > 0).any())
    # every diagonal runs 14 rounds of 32 samples or more: (t_out - t_in) / dt samples, dt = 0.5 h / |d|
    diag = torch.tensor([k == "diagonal" for k in kinds])
    o64, d64 = o[diag].double(), d[diag].double()
    t0, t1 = (lo.double() - o64) / d64, (-lo.double() - o64) / d64
    t_in = torch.minimum(t0, t1).amax(-1).clamp_min(0.0)
    t_out = torch.maximum(t0, t1).amin(-1)
    h = min((b - a) / r for a, b, r in zip(*EDGE_BOUNDS, EDGE_RES))
    samples = (t_out - t_in) / (0.5 * h / d64.norm(dim=-1))
    report("diagonal samples (min)", (), samples.min().item())
    assert diag.any() and ((samples / 32).ceil() >= 14).all()
