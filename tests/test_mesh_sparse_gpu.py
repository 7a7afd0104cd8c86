"""GPU: sparse mesh extraction over an occupancy grid's active bricks (csrc/mesh_sparse.cu, include/nerfb200.h
"sparse meshes").

The baseline is the library's dense path, which test_mesh_gpu.py pins to a numpy restatement.  Dense vertex ids follow
lattice-edge order, so each dense vertex's edge key q * 3 + a is the sorted list of sign changes; the sparse path
reports its keys, and a sparse mesh is compared with the dense one through them:
  - the same key set, bit-identical vertices (and view directions, colors, normals), and the same faces once mapped
    through the keys, restricted to the cubes of active bricks;
  - full grids on networks (A1 at init, lego A0, hidden 256) at several lattices, partial grids on analytic fields, and
    lego A0 with a grid from OccupancyGrid.from_models;
  - topology where the active region covers the surface, and open edges only on active / inactive brick faces where it
    does not; repeatability and independence of bricks_per_call; a 2048^3 lattice past the dense path's limit;
  - no refusal launches anything."""
import math

import numpy as np
import pytest
import torch

from helpers import LEGO_BOX, bits_equal, shipped_models

pytestmark = pytest.mark.gpu

BOX = ((-1.0,) * 3, (1.0,) * 3)


def report(what, ctx, value):
    print(f"[mesh_sparse] {what} {ctx}: {value}")


def _counts_table():
    import os
    import re

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    text = open(os.path.join(root, "nerf_pytorch_b200", "csrc", "mc_table.cuh")).read()
    return torch.tensor([int(v) for v in re.findall(r"-?\d+", re.search(r"kMcTriCount\[256\] = \{(.*?)\};", text,
                                                                          re.S).group(1))])


COUNTS = _counts_table()


def _dense_keys(vol, level):
    """Sorted int64 keys q * 3 + a of the crossing lattice edges of vol (n2, n1, n0): the dense vertex order."""
    n2, n1, n0 = vol.shape
    ins = vol > level
    q = torch.arange(n2 * n1 * n0, device=vol.device).view(n2, n1, n0)
    keys = [q[:, :, :-1][ins[:, :, :-1] != ins[:, :, 1:]] * 3,
            q[:, :-1, :][ins[:, :-1, :] != ins[:, 1:, :]] * 3 + 1,
            q[:-1][ins[:-1] != ins[1:]] * 3 + 2]
    return torch.sort(torch.cat(keys)).values


def _face_bricks(vol, level, B):
    """(F,) int64: the brick index of the cube of each dense face (faces run cube by cube, table counts each)."""
    n2, n1, n0 = vol.shape
    ins = (vol > level).to(torch.int64)
    case = torch.zeros(n2 - 1, n1 - 1, n0 - 1, dtype=torch.int64, device=vol.device)
    for c in range(8):
        dx, dy, dz = c & 1, c >> 1 & 1, c >> 2 & 1
        case |= ins[dz:n2 - 1 + dz, dy:n1 - 1 + dy, dx:n0 - 1 + dx] << c
    cnt = COUNTS.to(vol.device)[case.view(-1)]
    nb = [-(-(n - 1) // B) for n in (n0, n1, n2)]
    k = torch.arange(n2 - 1, device=vol.device) // B
    j = torch.arange(n1 - 1, device=vol.device) // B
    i = torch.arange(n0 - 1, device=vol.device) // B
    brick = ((k[:, None, None] * nb[1] + j[None, :, None]) * nb[0] + i[None, None, :]).reshape(-1)
    return torch.repeat_interleave(brick, cnt)


def _canon(faces):
    f = faces.cpu().numpy()
    return f[np.lexsort(f.T[::-1])] if f.size else f.reshape(0, 3)


def _assert_same(dense, sparse, skeys, dvol, level, brick_map=None, extras=()):
    """sparse (verts, faces) against dense (verts, faces) restricted to active bricks (all bricks without a map)."""
    from nerf_pytorch_b200 import ops

    dv, df = dense
    sv, sf = sparse
    dkeys = _dense_keys(dvol, level)
    assert dkeys.numel() == dv.shape[0]
    if brick_map is not None:
        keep = brick_map[_face_bricks(dvol, level, ops.mesh_brick())] >= 0
        df = df[keep]
    idx = torch.searchsorted(dkeys, skeys)
    assert bool((idx < dkeys.numel()).all()) and torch.equal(dkeys[idx.clamp(max=dkeys.numel() - 1)], skeys)
    assert torch.unique(skeys).numel() == skeys.numel()
    assert bits_equal(sv, dv[idx])
    for d, s in extras:
        assert bits_equal(s, d[idx])
    mapped = idx[sf.long()]
    assert np.array_equal(_canon(mapped), _canon(df.long()))
    used = torch.unique(df.long())
    assert torch.equal(torch.sort(idx).values, used)  # exactly the vertices the active cubes use
    return df.shape[0]


# ---- networks ---------------------------------------------------------------------------------------------------------
def _init_net(hidden, layers, skip):
    """A network at init, its sigma bias shifted so that raw sigma changes sign inside the box."""
    import nerf_pytorch_b200 as nb

    torch.manual_seed(11)
    m = nb.FlexibleNeRFModel(num_layers=layers, hidden_size=hidden, skip_connect_every=skip, num_encoding_fn_xyz=10,
                             num_encoding_fn_dir=4).cuda()
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    pts = (torch.rand(1 << 14, 3, device="cuda", generator=torch.Generator("cuda").manual_seed(3)) - 0.5) * 3.0
    with torch.no_grad():
        sigma, _ = nb.density_gradient(m, epf, pts)
        m.fc_alpha.bias -= sigma.median()
    return m, epf, edf


def _net(name):
    if name == "lego_a0":
        return shipped_models("lego")[1:]
    if name == "a1_init":
        return _init_net(128, 8, 3)
    return _init_net(256, 4, 4)


def _level_of(model, epf, edf, res):
    import nerf_pytorch_b200 as nb

    vol = nb.density_volume(model, epf, LEGO_BOX, res, encode_direction_fn=edf)
    return vol, float(vol[vol > 0].median()) if bool((vol > 0).any()) else 1.0


@pytest.mark.parametrize("net,res", [("a1_init", 64), ("lego_a0", 64), ("hidden256_init", 64), ("lego_a0", 128),
                                     ("a1_init", 128), ("lego_a0", 257), ("hidden256_init", 257),
                                     ("lego_a0", (72, 41, 97))])
def test_full_grid_equals_dense(net, res):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import mesh

    model, epf, edf = _net(net)
    vol, level = _level_of(model, epf, edf, res)
    if net == "lego_a0":
        level = 50.0
    dense = nb.extract_mesh(model, epf, LEGO_BOX, res, level, encode_direction_fn=edf, colors=True, normals=True)
    grid = nb.OccupancyGrid.full(LEGO_BOX, 16)
    sp, keys = mesh._extract_mesh(model, epf, LEGO_BOX, res, level, edf, True, None, None, True, grid, None,
                                  edge_keys=True)
    report(net, f"{res} vertices / faces", (sp.vertices.shape[0], sp.faces.shape[0]))
    assert sp.faces.shape[0] > 0
    _assert_same((dense.vertices, dense.faces), (sp.vertices, sp.faces), keys, vol, level,
                 extras=((dense.colors, sp.colors), (dense.normals, sp.normals)))
    assert sp.faces.shape[0] == dense.faces.shape[0]


# ---- analytic fields through the hooks ---------------------------------------------------------------------------------
def _field(kind, pts):
    x, y, z = (pts[:, c].double() for c in range(3))
    if kind == "sphere":
        f = 0.7 - torch.sqrt(x * x + y * y + z * z)
    elif kind == "torus":
        f = 0.25 - torch.sqrt((torch.sqrt(x * x + y * y) - 0.55) ** 2 + z * z)
    else:
        f = torch.maximum(0.3 - torch.sqrt((x - 0.45) ** 2 + y * y + z * z),
                          0.3 - torch.sqrt((x + 0.45) ** 2 + y * y + z * z))
    return f.float()


def _dense_field(kind, box, res):
    from nerf_pytorch_b200 import ops

    n0, n1, n2 = (r + 1 for r in res)
    pts = torch.empty(n0 * n1 * n2, 3, device="cuda")
    ops.mesh_lattice_points(box, 0, n2, pts)
    return _field(kind, pts).view(n2, n1, n0)


def _sparse_field(kind, box, grid, level, halo=True, bricks_per_call=None):
    """The sparse path on an analytic field: bricks, points, values, count, emit.  (verts, faces, dirs, keys, map)"""
    from nerf_pytorch_b200 import ops

    brick_map, bricks, n_dev = ops.mesh_sparse_bricks(box, grid)
    n = int(n_dev.item())
    per = (ops.mesh_brick() + 1 + 2 * halo) ** 3
    values = torch.empty(n * per, device="cuda")
    chunk = bricks_per_call or max(n, 1)
    pts = torch.empty(chunk * per, 3, device="cuda")
    for first in range(0, n, chunk):
        cnt = min(chunk, n - first)
        ops.mesh_sparse_points(box, bricks, first, cnt, halo, pts)
        values[first * per:(first + cnt) * per] = _field(kind, pts[:cnt * per])
    totals, ws = ops.mesh_sparse_count(box, brick_map, bricks, n, values, halo, level)
    nv, nf = totals.tolist()
    v, f, d, k = ops.mesh_sparse_emit(box, brick_map, bricks, n, values, halo, level, ws, nv, nf, want_dirs=halo,
                                      want_keys=True)
    return v, f, d, k, brick_map


def _random_grid(seed, frac, bounds=BOX, res=(11, 13, 9)):
    import nerf_pytorch_b200 as nb

    g = torch.Generator("cuda").manual_seed(seed)
    occ = torch.rand(res[2], res[1], res[0], generator=g, device="cuda") < frac
    return nb.OccupancyGrid.from_occupancy(bounds, occ)


def _halfspace_grid(x_max=0.1, res=16):
    """Cells whose centre has x < x_max occupied: the bricks past a plane are inactive, so the surface is cut there."""
    import nerf_pytorch_b200 as nb

    centre = -1 + (torch.arange(res, device="cuda").float() + 0.5) * 2 / res
    occ = (centre < x_max).view(1, 1, res).expand(res, res, res).contiguous()
    return nb.OccupancyGrid.from_occupancy(BOX, occ)


GRIDS = [("random", 0, 0.1), ("random", 1, 0.5), ("random", 2, 0.9), ("part_box", 3, 0.0), ("part_box", 4, 0.5),
         ("halfspace", 0, 0.5)]


@pytest.mark.parametrize("kind", ["sphere", "torus", "two_spheres"])
@pytest.mark.parametrize("grid_kind,seed,frac", GRIDS)
def test_partial_grid_equals_dense_restricted_to_active_bricks(kind, grid_kind, seed, frac):
    from nerf_pytorch_b200 import mesh, ops

    res = (70, 64, 53)
    box = ops.grid_struct(BOX, res)
    if grid_kind == "random":
        grid = _random_grid(seed, frac)
    elif grid_kind == "halfspace":
        grid = _halfspace_grid()
    else:  # a grid over part of the box: every brick with a corner outside it is active
        grid = _random_grid(seed, frac, ((-0.6, -1.3, -0.2), (0.9, 0.5, 1.4)), (6, 7, 5))
    dvol = _dense_field(kind, box, res)
    dv, df, dd = mesh._surface(dvol, box, 0.0, want_dirs=True)
    sv, sf, sd, keys, bmap = _sparse_field(kind, box, grid, 0.0)
    n = _assert_same((dv, df), (sv, sf), keys, dvol, 0.0, bmap, extras=((dd, sd),))
    report(kind, f"{grid_kind} {frac}: active bricks / faces kept / dense faces",
           (int((bmap >= 0).sum()), n, df.shape[0]))


def _edges(f):
    return np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])


@pytest.mark.parametrize("kind,chi", [("sphere", 2), ("torus", 0), ("two_spheres", 4)])
def test_topology(kind, chi):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    res = (64, 64, 64)
    box = ops.grid_struct(BOX, res)
    # the field's own occupancy at 16^3 cells, dilated: covers the surface and leaves most bricks inactive
    cells = torch.stack(torch.meshgrid(*(torch.arange(16, device="cuda") for _ in range(3)), indexing="ij"), -1)
    centres = (-1 + (cells.flip(-1).float() + 0.5) * 2 / 16).view(-1, 3)
    occ = (_field(kind, centres).abs() < 0.2).view(16, 16, 16)
    grid = nb.OccupancyGrid.from_occupancy(BOX, occ)
    v, f, _, _, bmap = _sparse_field(kind, box, grid, 0.0, halo=False)
    f = f.cpu().numpy()
    und = np.sort(_edges(f), 1)
    _, cu = np.unique(und, axis=0, return_counts=True)
    _, cd = np.unique(_edges(f), axis=0, return_counts=True)
    assert (cu == 2).all() and (cd == 1).all()
    n_e = np.unique(und, axis=0).shape[0]
    assert v.shape[0] - n_e + f.shape[0] == chi
    report(kind, "active bricks of all", (int((bmap >= 0).sum()), bmap.numel()))

    # a grid that cuts the surface: open edges lie on brick faces between active and inactive bricks
    grid = _halfspace_grid()
    v, f, _, keys, bmap = _sparse_field(kind, box, grid, 0.0, halo=False)
    f = f.cpu().numpy()
    und = np.sort(_edges(f), 1)
    u, c = np.unique(und, axis=0, return_counts=True)
    assert (c <= 2).all()
    once = u[c == 1]
    B = ops.mesh_brick()
    k = keys.cpu().numpy()
    q, a = k // 3, k % 3
    n0, n1 = res[0] + 1, res[1] + 1
    qc = np.stack((q % n0, (q // n0) % n1, q // (n0 * n1)), -1)
    nb_ = [-(-r // B) for r in res]
    act = (bmap >= 0).cpu().numpy()
    idx = lambda t: (t[2] * nb_[1] + t[1]) * nb_[0] + t[0]  # noqa: E731
    for e in once:
        # the segment lies on a cube face on a brick boundary plane (axis ax, plane b B) with an active brick on one
        # side and an inactive one on the other; along the other axes the cube's corner is the ends' smaller index
        ok = False
        for ax in range(3):
            if a[e[0]] == ax or a[e[1]] == ax or qc[e[0], ax] != qc[e[1], ax] or qc[e[0], ax] % B:
                continue
            b = qc[e[0], ax] // B
            if b == 0 or b == nb_[ax]:
                continue
            bc = [min(qc[e[0], c], qc[e[1], c]) // B for c in range(3)]
            lo_b, hi_b = list(bc), list(bc)
            lo_b[ax], hi_b[ax] = b - 1, b
            ok = ok or act[idx(lo_b)] != act[idx(hi_b)]
        assert ok, (qc[e[0]], a[e[0]], qc[e[1]], a[e[1]])
    report(kind, "open edges with a half-space grid", once.shape[0])
    assert once.shape[0] > 0


def test_repeatable_and_independent_of_bricks_per_call():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import mesh

    model, epf, edf = shipped_models("lego")[1:]
    grid = nb.OccupancyGrid.from_models([model], epf, LEGO_BOX, 64, encode_direction_fn=edf)
    outs = [mesh._extract_mesh(model, epf, LEGO_BOX, 96, 50.0, edf, True, None, None, False, grid, bpc,
                               edge_keys=True) for bpc in (None, None, 1, 7)]
    m0, k0 = outs[0]
    assert m0.faces.shape[0] > 0
    for m, k in outs[1:]:
        assert bits_equal(m.vertices, m0.vertices) and torch.equal(m.faces, m0.faces) and torch.equal(k, k0)
        assert bits_equal(m.colors, m0.colors)


@pytest.mark.parametrize("res", [256, 512])
def test_model_grid(res):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import mesh, ops

    model, epf, edf = shipped_models("lego")[1:]
    level = 50.0
    grid = nb.OccupancyGrid.from_models([model], epf, LEGO_BOX, 128, threshold=0.0, encode_direction_fn=edf)
    box = ops.grid_struct(LEGO_BOX, (res,) * 3)
    vol = nb.density_volume(model, epf, LEGO_BOX, res, encode_direction_fn=edf)
    brick_map, _, n_dev = ops.mesh_sparse_bricks(box, grid)
    fb = _face_bricks(vol, level, ops.mesh_brick())
    assert bool((brick_map[fb] >= 0).all()), "a dense face lies in a brick the grid calls empty"
    dense = nb.extract_mesh(model, epf, LEGO_BOX, res, level, encode_direction_fn=edf)
    sp, keys = mesh._extract_mesh(model, epf, LEGO_BOX, res, level, edf, False, None, None, False, grid, None,
                                  edge_keys=True)
    _assert_same((dense.vertices, dense.faces), (sp.vertices, sp.faces), keys, vol, level, brick_map)
    assert sp.faces.shape[0] == dense.faces.shape[0]
    n = int(n_dev.item())
    pts = n * (ops.mesh_brick() + 1) ** 3
    report(f"lego A0 {res}^3", "active bricks / points evaluated / (R + 1)^3 / ratio",
           (n, pts, (res + 1) ** 3, pts / (res + 1) ** 3))


def test_past_the_dense_limit():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import mesh, ops

    model, epf, edf = shipped_models("lego")[1:]
    res, level = 2048, 50.0
    grid = nb.OccupancyGrid.from_models([model], epf, LEGO_BOX, 128, threshold=0.0, encode_direction_fn=edf)
    box = ops.grid_struct(LEGO_BOX, (res,) * 3)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    sp, keys = mesh._extract_mesh(model, epf, LEGO_BOX, res, level, edf, False, None, None, False, grid, None,
                                  edge_keys=True)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    nv, nf = sp.vertices.shape[0], sp.faces.shape[0]
    _, _, n_dev = ops.mesh_sparse_bricks(box, grid)
    n = int(n_dev.item())
    B = ops.mesh_brick()
    per = (B + 1) ** 3
    chunk = min(n, mesh._SLAB_POINTS // per) * per
    rows = -(-chunk // 64) * 64
    # the documented memory: int32 map and list per brick, the brick scratch, per active brick its values and the
    # workspace, the MLP call's points (12 B), raw output (16 B) and relu (4 B) per row, and the outputs
    bound = (8 * ops.mesh_sparse_brick_count(box) + ops.mesh_sparse_scratch_bytes(box) + 4 * per * n
             + ops.mesh_sparse_workspace_bytes(box, n) + 32 * rows + 20 * nv + 12 * nf + (64 << 20))
    report("lego A0 2048^3", "active bricks / vertices / faces / peak bytes / bound / dense lattice points",
           (n, nv, nf, peak, bound, (res + 1) ** 3))
    assert nf > 0 and peak <= bound

    # every vertex (a seeded sample) is the header's vertex on its edge, from the network at the edge's two ends
    g = torch.Generator("cuda").manual_seed(5)
    pick = torch.randint(0, nv, (min(nv, 1 << 16),), generator=g, device="cuda")
    k = keys[pick]
    q, a = k // 3, k % 3
    n0 = res + 1
    i = torch.stack((q % n0, (q // n0) % n0, q // (n0 * n0)), -1)
    X = torch.from_numpy(np.float32(-1.5) + (np.float32(1.5) - np.float32(-1.5)) *
                         np.arange(n0, dtype=np.float32) / np.float32(res)).cuda()
    p0 = X[i]
    j = i + torch.nn.functional.one_hot(a, 3)
    p1 = X[j]
    both = torch.cat((p0, p1))
    pad = (-both.shape[0]) % 64
    both = torch.cat((both, both[:pad]))
    with torch.no_grad():
        raw = nb.run_network(model, both.view(-1, 64, 3),
                             torch.tensor([0.0, 0.0, 1.0], device="cuda").expand(both.shape[0] // 64, 3), 1 << 20,
                             epf, edf)
    sig = torch.relu(raw.reshape(-1, 4)[: 2 * k.numel(), 3])
    v0, v1 = sig[: k.numel()], sig[k.numel():]
    assert bool(((v0 > level) != (v1 > level)).all())
    t = (level - v0) / (v1 - v0)
    rows_ = torch.arange(k.numel(), device="cuda")
    want = p0.clone()
    want[rows_, a] = p0[rows_, a] + t * (p1[rows_, a] - p0[rows_, a])
    got = sp.vertices[pick]
    exact = (got.view(torch.int32) == want.view(torch.int32)).all(1).float().mean().item()
    report("lego A0 2048^3", "sampled vertices bit-identical to the vertex rule on run_network's sigma", exact)
    assert exact == 1.0

    # for seeded bricks holding vertices: the brick's faces are those of a dense extraction of its own 9^3 values.  A
    # face of the sparse mesh belongs to the brick when all three of its edges lie in the brick's cubes (the table puts
    # no triangle flat on a cube face, so a neighbour's triangle always has an edge outside); keys compare the two.
    skeys = keys[sp.faces.long()]  # (F, 3)
    sq, sa = skeys // 3, skeys % 3
    sqc = torch.stack((sq % n0, (sq // n0) % n0, sq // (n0 * n0)), -1)  # (F, 3, xyz)
    nb_ = res // B
    bricks = torch.unique(torch.clamp(i // B, max=nb_ - 1), dim=0)
    bricks = bricks[torch.randperm(bricks.shape[0], generator=g, device="cuda")[:16]]
    for bc in bricks.tolist():
        lo_i = torch.tensor(bc, device="cuda") * B
        idx = torch.arange(B + 1, device="cuda")
        kk, jj, ii = torch.meshgrid(idx + lo_i[2], idx + lo_i[1], idx + lo_i[0], indexing="ij")
        pts = torch.stack((X[ii], X[jj], X[kk]), -1).reshape(-1, 3)
        pad = (-pts.shape[0]) % 64
        rows = torch.cat((pts, pts[:pad])).view(-1, 64, 3)
        with torch.no_grad():
            raw = nb.run_network(model, rows, torch.tensor([0.0, 0.0, 1.0], device="cuda").expand(rows.shape[0], 3),
                                 1 << 20, epf, edf)
        vol = torch.relu(raw.reshape(-1, 4)[:pts.shape[0], 3]).view(B + 1, B + 1, B + 1).contiguous()
        local = nb.extract_mesh_from_volume(vol, ((-1.0,) * 3, (1.0,) * 3), level)
        lk = _dense_keys(vol, level)  # local keys, in the local mesh's vertex order
        lq, la = lk // 3, lk % 3
        m = B + 1
        gq = ((lq // (m * m) + lo_i[2]) * n0 + (lq // m) % m + lo_i[1]) * n0 + lq % m + lo_i[0]
        want_f = (gq * 3 + la)[local.faces.long()]
        rel = sqc - lo_i
        inside = ((rel >= 0) & (rel <= B)).all(-1) & (torch.gather(rel, 2, sa[..., None])[..., 0] < B)
        got_f = skeys[inside.all(-1)]
        assert np.array_equal(_canon(got_f), _canon(want_f)), bc
    report("lego A0 2048^3", "bricks whose faces equal a dense extraction of their own values", bricks.shape[0])


def test_refusals_launch_nothing():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    model, epf, edf = shipped_models("lego")[1:]
    full = nb.OccupancyGrid.full(LEGO_BOX, 8)
    bad_bits = nb.OccupancyGrid.full(LEGO_BOX, 8)
    bad_bits.bits = bad_bits.bits[:-1]
    torch.cuda.synchronize()
    before = ops.launch_count()
    cases = [
        (lambda: nb.extract_mesh(model, epf, LEGO_BOX, 32, grid="full"), ValueError),
        (lambda: nb.extract_mesh(model, epf, LEGO_BOX, 32, grid=full.bits), ValueError),
        (lambda: nb.extract_mesh(model, epf, LEGO_BOX, 32, grid=full.to("cpu")), NotImplementedError),
        (lambda: nb.extract_mesh(model, epf, LEGO_BOX, 32, grid=bad_bits), ValueError),
        (lambda: nb.extract_mesh(model, epf, LEGO_BOX, 32, grid=full, planes_per_slab=2), ValueError),
        (lambda: nb.extract_mesh(model, epf, LEGO_BOX, 32, grid=full, bricks_per_call=0), ValueError),
        (lambda: nb.extract_mesh(model, epf, LEGO_BOX, 4097, grid=full), ValueError),
        (lambda: nb.extract_mesh(model, epf, LEGO_BOX, 32, level=math.inf, grid=full), ValueError),
        (lambda: nb.extract_mesh(model, epf, LEGO_BOX, 32, grid=full, impl=7), NotImplementedError),
        (lambda: nb.extract_mesh(torch.nn.Linear(3, 4).cuda(), epf, LEGO_BOX, 32, grid=full), NotImplementedError),
    ]
    if torch.cuda.device_count() > 1:
        cases.append((lambda: nb.extract_mesh(model, epf, LEGO_BOX, 32, grid=full.to("cuda:1")), ValueError))
    for fn, err in cases:
        with pytest.raises(err):
            fn()
    torch.cuda.synchronize()
    assert ops.launch_count() == before
