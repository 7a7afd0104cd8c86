"""GPU: meshes of baked fields (csrc/baked.cu baked_mesh_dirs_kernel / baked_mesh_colors_kernel; nb.extract_baked_mesh;
include/nerfb200.h "baked fields: meshes").

  1. faces and vertices against the network's mesh: the lego bake at 256^3 against extract_mesh over the same grid,
     the fern bake in NDC, and a hidden-256 network at 48^3: faces and vertex ids bit-identical, vertices bit-identical
     on every edge whose endpoints both have sigma_raw >= 0, and every vertex the header's rule on the raw values;
  2. directions: on a field with every brick active, dirs are mesh_sparse_emit's view_dirs with halo = 1 bit for bit;
     on partly active fields dirs and normals equal a torch restatement that reads 0 where no active brick holds a point;
  3. colours: bit for bit a torch restatement of the two-corner fmaf chain, the SH and the sigmoid (fmaf(a, b, c) is
     fp32(a b + c) with the exact product formed in fp64), with and without view directions; on the lego bake, close
     to extract_mesh(colors=True)'s network colours;
  4. a sphere: closed, accurate, outward normals, uniform colour;
  5. pruning transparent bricks keeps the mesh and, where the gradient stencil keeps its copies, the attributes;
  6. an fp16 field meshes bit for bit like its widened field;
  7. a field fitted without a network meshes, is closed inside its active bricks and round-trips through save_ply;
  8. empty fields and levels give empty meshes; 9. launch counts."""
import math

import pytest
import torch

from helpers import (FERN_BOX, FERN_CAM, LEGO_BOX, LEGO_CAM, bits_equal, lattice_index, shipped_models, sphere_poses,
                     synthetic_field, targets)

pytestmark = pytest.mark.gpu

F32 = torch.float32


def report(what, ctx, value):
    print(f"[baked-mesh] {what} {ctx}: {value}")


# ---- torch restatements of the header's rules -------------------------------------------------------------------------
def mesh_keys(field, level):
    """(vertices, faces, edge keys) of mesh_sparse_count / _emit over the field's sigma_raw at halo 0."""
    from nerf_pytorch_b200 import ops

    sigma = field.values[..., 0].float().contiguous()
    box = field.box()
    totals, ws = ops.mesh_sparse_count(box, field.brick_map, field.bricks, field.n_active, sigma, False, level)
    n_v, n_f = (int(t) for t in totals.tolist())
    v, f, _, k = ops.mesh_sparse_emit(box, field.brick_map, field.bricks, field.n_active, sigma, False, level, ws, n_v,
                                      n_f, want_keys=True)
    return v, f, k


def canon_map(field):
    """int64 [lattice points]: the row (slot * 729 + point) of each lattice point's canonical copy, -1 where no active
    brick holds it.  The first copy in the tie's order is the lowest row (per axis either the bricks or the points
    differ, and activity depends on the brick alone)."""
    n = math.prod(r + 1 for r in field.resolution)
    idx = lattice_index(field).reshape(-1)
    canon = torch.full((n,), -1, dtype=torch.int64, device="cuda")
    canon.scatter_reduce_(0, idx, torch.arange(idx.numel(), device="cuda"), reduce="amin", include_self=False)
    return canon


def decode(field, keys):
    n0, n1 = field.resolution[0] + 1, field.resolution[1] + 1
    p = keys // 3
    return torch.stack([p % n0, p // n0 % n1, p // (n0 * n1)], -1), keys % 3


def lin(field, q):
    n0, n1 = field.resolution[0] + 1, field.resolution[1] + 1
    return (q[:, 2] * n1 + q[:, 1]) * n0 + q[:, 0]


def sigma_at(field, canon, q):
    c = canon[lin(field, q)]
    v = field.values.reshape(-1, 32)[c.clamp_min(0), 0].float()
    return torch.where(c >= 0, v, torch.zeros_like(v))


def ends(q, a):
    q1 = q.clone()
    q1[torch.arange(q.shape[0], device="cuda"), a] += 1
    return q1


def edge_t(field, canon, q, a, level):
    return (torch.tensor(level, dtype=F32, device="cuda") - sigma_at(field, canon, q)) / \
        (sigma_at(field, canon, ends(q, a)) - sigma_at(field, canon, q))


def lattice_grad(field, canon, q):
    lo = torch.tensor(field.bounds[0], dtype=F32, device="cuda")
    hi = torch.tensor(field.bounds[1], dtype=F32, device="cuda")
    res = torch.tensor(field.resolution, device="cuda")
    h = (hi - lo) / res.to(F32)
    g = []
    for c in range(3):
        ql, qh = q.clone(), q.clone()
        ql[:, c] = (q[:, c] - 1).clamp_min(0)
        qh[:, c] = torch.minimum(q[:, c] + 1, res[c])
        g.append((sigma_at(field, canon, qh) - sigma_at(field, canon, ql)) / (h[c] * (qh[:, c] - ql[:, c]).to(F32)))
    return torch.stack(g, -1)


def restated_dirs(field, keys, level):
    """(dirs, normals) of the header's rule."""
    canon = canon_map(field)
    q, a = decode(field, keys)
    t = edge_t(field, canon, q, a, level)
    g0, g1 = lattice_grad(field, canon, q), lattice_grad(field, canon, ends(q, a))
    g = g0 + t[:, None] * (g1 - g0)
    s = (g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1]) + g[:, 2] * g[:, 2]
    ok = ((s > 0) & (s < math.inf))[:, None]
    d = torch.where(ok, g / torch.sqrt(s)[:, None], torch.tensor([0.0, 0.0, 1.0], device="cuda"))
    return d, torch.where(ok, -d, torch.zeros_like(d))


def fmaf(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def sh_basis(d):
    def k(v):
        return torch.tensor(v, dtype=F32, device="cuda")

    x, y, z = d.unbind(-1)
    xx, yy, zz = x * x, y * y, z * z
    return [k(0.28209479177387814).expand_as(x), k(-0.4886025119029199) * y, k(0.4886025119029199) * z,
            k(-0.4886025119029199) * x, (k(1.0925484305920792) * x) * y, (k(-1.0925484305920792) * y) * z,
            k(0.31539156525252005) * ((k(2.0) * zz - xx) - yy), (k(-1.0925484305920792) * x) * z,
            k(0.5462742152960396) * (xx - yy)]


def restated_colors(field, keys, level, dirs):
    canon = canon_map(field)
    q, a = decode(field, keys)
    rows = field.values.reshape(-1, 32)
    v0 = rows[canon[lin(field, q)], :28].float()
    v1 = rows[canon[lin(field, ends(q, a))], :28].float()
    t = (torch.tensor(level, dtype=F32, device="cuda") - v0[:, 0]) / (v1[:, 0] - v0[:, 0])
    u = 1.0 - t
    v = fmaf(t[:, None], v1, fmaf(u[:, None], v0, torch.zeros_like(v0)))
    out = []
    for c in range(3):
        coef = v[:, 1 + 9 * c: 10 + 9 * c]
        if field.use_viewdirs:
            s = torch.zeros_like(t)
            for j, Y in enumerate(sh_basis(dirs)):
                s = fmaf(Y, coef[:, j], s)
        else:
            s = torch.tensor(0.28209479177387814, dtype=F32, device="cuda") * coef[:, 0]
        out.append(1.0 / (1.0 + torch.exp(-s)))
    return torch.stack(out, -1)


def restated_vertices(field, keys, level):
    """NDC / field-space vertices of the header's vertex rule on the raw sigma_raw."""
    canon = canon_map(field)
    q, a = decode(field, keys)
    t = edge_t(field, canon, q, a, level)
    lo = torch.tensor(field.bounds[0], dtype=F32, device="cuda")
    hi = torch.tensor(field.bounds[1], dtype=F32, device="cuda")
    res = torch.tensor(field.resolution, device="cuda").to(F32)
    p = lo + ((hi - lo) * q.to(F32)) / res
    p1 = lo + ((hi - lo) * ends(q, a).to(F32)) / res
    r = torch.arange(q.shape[0], device="cuda")
    x = p.clone()
    x[r, a] = p[r, a] + t * (p1[r, a] - p[r, a])
    return x


def both_nonneg(field, keys):
    canon = canon_map(field)
    q, a = decode(field, keys)
    return (sigma_at(field, canon, q) >= 0) & (sigma_at(field, canon, ends(q, a)) >= 0)


def positive_median(field):
    s = field.values[..., 0].float()
    return float(s[s > 0].median())


# ---- 1. faces and vertices against the network's mesh ------------------------------------------------------------------
def _against_network(model, epf, edf, box, res, grid, ndc=None):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import mesh, ops

    f = nb.bake(model, epf, edf, bounds=box, resolution=res, grid=grid)
    level = positive_median(f)
    with torch.no_grad():
        net, nkeys = mesh._extract_mesh(model, epf, box, res, level, edf, False, 1, None, False, grid, None,
                                        edge_keys=True, ndc=ndc)
    m = nb.extract_baked_mesh(f, level, ndc=ndc)
    _, _, keys = mesh_keys(f, level)
    assert m.faces.shape[0] > 0
    assert torch.equal(keys, nkeys) and torch.equal(m.faces, net.faces)
    same = both_nonneg(f, keys)
    assert bits_equal(m.vertices[same], net.vertices[same])
    x = restated_vertices(f, keys, level)
    if ndc is not None:
        x, _, _ = ops.ndc_mesh_to_world(ops.ndc_struct(*ndc), x, m.faces)
    assert bits_equal(m.vertices, x)
    return f, level, m, net, int((~same).sum())


def test_lego_faces_and_vertices_match_the_network_mesh():
    import nerf_pytorch_b200 as nb

    mc, mf, epf, edf = shipped_models("lego")
    grid = nb.OccupancyGrid.from_models([mf], epf, LEGO_BOX, 128, encode_direction_fn=edf)
    f, level, m, _, moved = _against_network(mf, epf, edf, LEGO_BOX, 256, grid)
    report("lego 256^3: level, vertices, faces, vertices on an edge with a negative end", "",
           (round(level, 3), m.vertices.shape[0], m.faces.shape[0], moved))


def test_fern_ndc_faces_and_vertices_match_the_network_mesh():
    import nerf_pytorch_b200 as nb

    mc, mf, epf, edf = shipped_models("fern")
    grid = nb.OccupancyGrid.from_models([mf], epf, FERN_BOX, 128, encode_direction_fn=edf)
    f, level, m, _, moved = _against_network(mf, epf, edf, FERN_BOX, 192, grid, ndc=FERN_CAM)
    report("fern 192^3 NDC: level, vertices, faces, moved", "", (round(level, 3), m.vertices.shape[0],
                                                               m.faces.shape[0], moved))


def test_hidden_256_faces_and_vertices_match_the_network_mesh():
    import nerf_pytorch_b200 as nb

    torch.manual_seed(11)
    model = nb.FlexibleNeRFModel(num_layers=8, hidden_size=256, skip_connect_every=4, num_encoding_fn_xyz=10,
                                 num_encoding_fn_dir=4).cuda()
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    box = ((-1.0,) * 3, (1.0,) * 3)
    _against_network(model, epf, edf, box, 48, nb.OccupancyGrid.full(box, 8))


# ---- 2. directions ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("res", [(24, 20, 17), (16, 16, 16)])
def test_dirs_on_a_fully_active_field_are_the_halo_view_dirs(res):
    from nerf_pytorch_b200 import ops

    f = synthetic_field(res, active=1.0, seed=3)
    level = 2.0
    v, faces, keys = mesh_keys(f, level)
    dirs, normals = ops.baked_mesh_dirs(f.box(), f.brick_map, f.values, level, keys, want_normals=True)
    # the halo layout: slot s, point l in 0 .. 10 per axis at lattice index 8 b + l - 1 clamped onto 0 .. res
    canon = canon_map(f)
    r = torch.tensor(res, device="cuda")
    nb_ = (r + 7) // 8
    br = f.bricks.long()
    b = torch.stack([br % nb_[0], br // nb_[0] % nb_[1], br // (nb_[0] * nb_[1])], -1)
    p = torch.arange(11 ** 3, device="cuda")
    l = torch.stack([p % 11, p // 11 % 11, p // 121], -1)
    q = torch.minimum((b[:, None] * 8 + l[None] - 1).clamp_min(0), r).reshape(-1, 3)
    halo = sigma_at(f, canon, q).contiguous()
    box = f.box()
    totals, ws = ops.mesh_sparse_count(box, f.brick_map, f.bricks, f.n_active, halo, True, level)
    n_v, n_f = (int(t) for t in totals.tolist())
    hv, hf, hd, hk = ops.mesh_sparse_emit(box, f.brick_map, f.bricks, f.n_active, halo, True, level, ws, n_v, n_f,
                                          want_dirs=True, want_keys=True)
    assert torch.equal(hk, keys) and torch.equal(hf, faces) and bits_equal(hv, v)
    assert bits_equal(dirs, hd)
    wd, wn = restated_dirs(f, keys, level)
    assert bits_equal(dirs, wd) and bits_equal(normals, wn)


@pytest.mark.parametrize("res,active,seed", [((24, 20, 17), 0.5, 4), ((40, 33, 9), 0.3, 5)])
def test_dirs_and_normals_on_partly_active_fields(res, active, seed):
    import nerf_pytorch_b200 as nb

    f = synthetic_field(res, active=active, seed=seed)
    level = 2.0
    m = nb.extract_baked_mesh(f, level, normals=True)
    _, _, keys = mesh_keys(f, level)
    from nerf_pytorch_b200 import ops

    dirs, _ = ops.baked_mesh_dirs(f.box(), f.brick_map, f.values, level, keys)
    wd, wn = restated_dirs(f, keys, level)
    assert bits_equal(dirs, wd) and bits_equal(m.normals, wn)
    assert m.vertices.shape[0] > 0


# ---- 3. colours -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("viewdirs", [True, False])
def test_colors_are_the_restated_rule(viewdirs):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    f = synthetic_field((24, 20, 17), active=0.6, viewdirs=viewdirs, seed=6)
    level = 1.5
    m = nb.extract_baked_mesh(f, level, colors=True, normals=True)
    _, _, keys = mesh_keys(f, level)
    dirs, _ = ops.baked_mesh_dirs(f.box(), f.brick_map, f.values, level, keys)
    assert bits_equal(m.colors, restated_colors(f, keys, level, dirs))
    assert m.colors.shape[0] > 0


# Mean absolute difference of the lego bake's vertex colours (256^3, level the median positive sigma_raw) from
# extract_mesh(colors=True)'s network colours over the same grid.  Measured on an H100 80GB HBM3 at 700 W: 0.0409 (the
# degree-2 SH fit of 64 directions against the network seen along its own lattice direction); the bar leaves 20 %.
LEGO_COLOR_MAD_BAR = 0.05


def test_lego_colors_close_to_the_network_colors():
    import nerf_pytorch_b200 as nb

    mc, mf, epf, edf = shipped_models("lego")
    grid = nb.OccupancyGrid.from_models([mf], epf, LEGO_BOX, 128, encode_direction_fn=edf)
    f = nb.bake(mf, epf, edf, bounds=LEGO_BOX, resolution=256, grid=grid)
    level = positive_median(f)
    m = nb.extract_baked_mesh(f, level, colors=True)
    with torch.no_grad():
        net = nb.extract_mesh(mf, epf, LEGO_BOX, 256, level, edf, colors=True, impl=1, grid=grid)
    assert torch.equal(m.faces, net.faces)
    mad = (m.colors - net.colors).abs().mean().item()
    report("lego 256^3 colour MAD against the network", "", round(mad, 5))
    assert mad < LEGO_COLOR_MAD_BAR


# ---- 4. a sphere ------------------------------------------------------------------------------------------------------
def _edge_counts(faces):
    e = torch.cat([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]]).long()
    e = torch.sort(e, 1).values
    _, counts = torch.unique(e[:, 0] * (int(faces.max()) + 1) + e[:, 1], return_counts=True)
    return e, counts


def test_sphere():
    import nerf_pytorch_b200 as nb

    res = 48
    f = synthetic_field((res,) * 3, active=1.0, seed=8)
    idx = lattice_index(f)
    n = res + 1
    i = torch.arange(n, device="cuda").to(F32)
    p = -1.0 + (2.0 * i) / res
    z, y, x = torch.meshgrid(p, p, p, indexing="ij")
    r = torch.sqrt(x * x + y * y + z * z).reshape(-1)
    c = torch.tensor([0.5, -1.0, 2.0], device="cuda")
    dense = torch.zeros(n ** 3, 32, device="cuda")
    dense[:, 0] = 100.0 * (0.6 - r)
    dense[:, 1:28].view(-1, 3, 9)[:, :, 0] = c
    f.values = dense[idx].contiguous()
    level = 10.0  # the sphere |x| = 0.5
    m = nb.extract_baked_mesh(f, level, colors=True, normals=True)
    V, F = m.vertices.shape[0], m.faces.shape[0]
    e, counts = _edge_counts(m.faces)
    assert bool((counts == 2).all())
    assert V - counts.numel() + F == 2
    rad = m.vertices.norm(dim=1)
    err = (rad - 0.5).abs().max().item()
    report("sphere 48^3: vertices, faces, max | |x| - 0.5 |", "", (V, F, err))
    assert err < 2e-3  # the chord of |x| over a cube side h = 1/24: h^2 / (8 * 0.45) ~ 5e-4
    assert bool(((m.normals * (m.vertices / rad[:, None])).sum(1) > 0.99).all())
    Y0 = torch.tensor(0.28209479177387814, dtype=F32, device="cuda")
    want = 1.0 / (1.0 + torch.exp(-(Y0 * c)))
    assert bits_equal(m.colors, want.expand(V, 3))


# ---- 5. transparent prune ---------------------------------------------------------------------------------------------
def test_transparent_prune_keeps_the_mesh():
    import nerf_pytorch_b200 as nb

    mc, mf, epf, edf = shipped_models("lego")
    grid = nb.OccupancyGrid.from_models([mf], epf, LEGO_BOX, 64, encode_direction_fn=edf)
    f = nb.bake(mf, epf, edf, bounds=LEGO_BOX, resolution=256, grid=grid)
    g = nb.prune_baked(f, ~nb.baked_transparent_bricks(f))
    for level in (0.0, positive_median(f)):
        a = nb.extract_baked_mesh(f, level, colors=True, normals=True)
        b = nb.extract_baked_mesh(g, level, colors=True, normals=True)
        assert bits_equal(a.vertices, b.vertices) and torch.equal(a.faces, b.faces)
        _, _, keys = mesh_keys(f, level)
        cf, cg = canon_map(f), canon_map(g)
        q, ax = decode(f, keys)
        kept = torch.ones(keys.numel(), dtype=torch.bool, device="cuda")
        res = torch.tensor(f.resolution, device="cuda")
        for e in (q, ends(q, ax)):
            for c in range(3):
                for s in (-1, 0, 1):
                    w = e.clone()
                    w[:, c] = (e[:, c] + s).clamp(min=0).minimum(res[c])
                    li = lin(f, w)
                    kept &= (cg[li] >= 0) == (cf[li] >= 0)
        assert bits_equal(a.normals[kept], b.normals[kept]) and bits_equal(a.colors[kept], b.colors[kept])
        report(f"transparent prune, level {level:.3f}: bricks kept, vertices, vertices whose stencil lost a copy", "",
               (g.n_active, f.n_active, keys.numel(), int((~kept).sum())))


# ---- 6. fp16 ----------------------------------------------------------------------------------------------------------
def test_half_field_meshes_like_its_widened_field():
    import nerf_pytorch_b200 as nb

    mc, mf, epf, edf = shipped_models("lego")
    grid = nb.OccupancyGrid.from_models([mf], epf, LEGO_BOX, 64, encode_direction_fn=edf)
    f = nb.bake(mf, epf, edf, bounds=LEGO_BOX, resolution=128, grid=grid)
    for field in (f, synthetic_field((24, 20, 17), active=0.6, seed=9)):
        h = field.half()
        level = positive_median(field)
        a = nb.extract_baked_mesh(h, level, colors=True, normals=True)
        b = nb.extract_baked_mesh(h.float(), level, colors=True, normals=True)
        assert a.vertices.shape[0] > 0
        for x, y in ((a.vertices, b.vertices), (a.faces, b.faces), (a.colors, b.colors), (a.normals, b.normals)):
            assert bits_equal(x, y)


# ---- 7. a field fitted without a network ------------------------------------------------------------------------------
def test_networkless_field(tmp_path):
    import nerf_pytorch_b200 as nb

    poses = sphere_poses(20)
    imgs, opts = targets("lego", poses)
    f = nb.BakedField.full(LEGO_BOX, 32, sigma_raw=0.1)
    t = nb.BakedFieldTrainer(f, imgs, poses.cuda(), LEGO_CAM[2], opts, lr_sigma=1.0, lr_sh=3e-2, rays_per_step=2048,
                             seed=2)
    t.step(200)
    w = nb.baked_brick_weights(f, poses, LEGO_CAM[0], LEGO_CAM[1], LEGO_CAM[2], opts)
    t.prune(w > 1e-3)
    t.subdivide()
    t.step(100)
    level = positive_median(f)
    m = nb.extract_baked_mesh(f, level, colors=True, normals=True)
    V, F = m.vertices.shape[0], m.faces.shape[0]
    assert V > 0 and F > 0
    # closed inside the active bricks: an edge in one face lies on a cube face next to a cube that is not marched, so
    # both its vertices' lattice edges touch such a cube
    e, counts = _edge_counts(m.faces)
    assert bool((counts <= 2).all())
    _, _, keys = mesh_keys(f, level)
    q, a = decode(f, keys)
    res = torch.tensor(f.resolution, device="cuda")
    nb_ = (res + 7) // 8
    outside = torch.zeros(V, dtype=torch.bool, device="cuda")
    r = torch.arange(V, device="cuda")
    for d in range(4):
        cube = q.clone()
        u, v = (a + 1) % 3, (a + 2) % 3
        cube[r, u] -= d & 1
        cube[r, v] -= d >> 1
        ok = ((cube >= 0) & (cube < res)).all(1)
        bc = cube.clamp_min(0) // 8
        slot = f.brick_map.long()[((bc[:, 2] * nb_[1] + bc[:, 1]) * nb_[0] + bc[:, 0]).clamp(0, f.brick_map.numel() - 1)]
        outside |= ~ok | (slot < 0)
    uniq = torch.unique(torch.sort(e, 1).values, dim=0, return_counts=True)
    boundary = uniq[0][uniq[1] == 1]
    assert bool(outside[boundary].all())
    report("networkless 64^3: bricks, vertices, faces, boundary edges", "", (f.n_active, V, F, boundary.shape[0]))
    path = tmp_path / "fit.ply"
    m.save_ply(path)
    with open(path, "rb") as fh:
        head = fh.read(1024).split(b"end_header")[0].decode()
    assert f"element vertex {V}" in head and f"element face {F}" in head
    assert path.stat().st_size == len(head) + len("end_header\n") + V * (12 + 12 + 3) + F * 13


# ---- 8. empty meshes; 9. launch counts --------------------------------------------------------------------------------
def test_empty_meshes_and_launch_counts():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    f = synthetic_field((24, 20, 17), active=0.6, seed=10)
    e = nb.prune_baked(f, torch.zeros(f.n_active, dtype=torch.bool, device="cuda"))
    before = ops.launch_count()
    m = nb.extract_baked_mesh(e, 1.0, colors=True, normals=True)
    assert ops.launch_count() == before
    assert m.vertices.shape == (0, 3) and m.faces.shape == (0, 3) and m.colors.shape == (0, 3)
    assert m.normals.shape == (0, 3)
    top = float(f.values[..., 0].max()) + 1.0
    before = ops.launch_count()
    m = nb.extract_baked_mesh(f, top, colors=True, normals=True)
    assert ops.launch_count() - before == 2  # classify and scan; nothing past the count
    assert m.vertices.shape == (0, 3) and m.faces.shape == (0, 3) and m.colors.shape == (0, 3)
    counts = {}
    for colors, normals in ((False, False), (False, True), (True, False), (True, True)):
        before = ops.launch_count()
        m = nb.extract_baked_mesh(f, 2.0, colors=colors, normals=normals)
        counts[(colors, normals)] = ops.launch_count() - before
        assert m.vertices.shape[0] > 0 and (m.colors is not None) == colors and (m.normals is not None) == normals
    assert counts == {(False, False): 3, (False, True): 4, (True, False): 5, (True, True): 5}
    g = synthetic_field((24, 20, 17), active=0.6, seed=10, viewdirs=False)
    before = ops.launch_count()
    nb.extract_baked_mesh(g, 2.0, colors=True)
    assert ops.launch_count() - before == 4  # no directions without view directions
