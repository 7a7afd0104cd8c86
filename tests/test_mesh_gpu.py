"""GPU: marching cubes (csrc/mesh.cu) and nb.extract_mesh.

The oracle is restate() below: a numpy statement of the three kernels -- classify, scan, emit -- from the definitions in
include/nerfb200.h and the committed case table, in fp32 with numpy's correctly rounded operations.
  - restatement: faces identical and vertices (and view directions) bit-identical, on analytic and seeded random volumes;
  - topology: every undirected edge in exactly two faces and every directed edge in one when the surface stays inside
    the box; Euler characteristic 2 (sphere), 0 (torus), 4 (two spheres); no degenerate triangle;
  - geometry: the volume interpolated at each vertex is the level to fp32 rounding; a sphere's enclosed volume and its
    outward normals;
  - determinism and slab independence;
  - networks: lego A0 (shipped weights), A1 at init and a hidden-256 network: the volume is run_network's sigma bit for
    bit, the mesh is open only on the box's faces, and colors are run_network's at the vertices and view directions;
  - no refusal launches anything."""
import math
import os
import re

import numpy as np
import pytest
import torch

from helpers import LEGO_BOX, bits_equal, shipped_models

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BOX = ((-1.0,) * 3, (1.0,) * 3)


def report(what, ctx, value):
    print(f"[mesh] {what} {ctx}: {value}")


def _table():
    text = open(os.path.join(ROOT, "nerf_pytorch_b200", "csrc", "mc_table.cuh")).read()
    width = int(re.search(r"#define NERFB200_MC_MAX_TRIS (\d+)", text).group(1))
    counts = np.array([int(v) for v in re.findall(r"-?\d+", re.search(r"kMcTriCount\[256\] = \{(.*?)\};", text,
                                                                          re.S).group(1))])
    rows = re.findall(r"\{([^}]*)\}", re.search(r"kMcTris\[256\]\[\d+\] = \{(.*?)\n\};", text, re.S).group(1))
    tris = np.array([[int(v) for v in r.split(",")] for r in rows]).reshape(256, width, 3)
    return counts, tris


COUNTS, TRIS = _table()
# cube edge e: axis e >> 2, low corner offset (x, y, z) from the bits of e & 3 on the other two axes, lower axis first
EDGE_OFF = np.array([[0, m & 1, m >> 1] if a == 0 else ([m & 1, 0, m >> 1] if a == 1 else [m & 1, m >> 1, 0])
                     for a in range(3) for m in range(4)])


def _coords(lo, hi, res):
    """p_c(i) = lo + ((hi - lo) * i) / res in fp32, one array per axis."""
    return [np.float32(lo[c]) + (np.float32(hi[c]) - np.float32(lo[c])) * np.arange(res[c] + 1, dtype=np.float32)
            / np.float32(res[c]) for c in range(3)]


def _grad(vol, lo, hi):
    """(n2, n1, n0, 3) fp32: the header's per-axis central differences, one-sided at the lattice's faces."""
    out = np.empty(vol.shape + (3,), np.float32)
    for c in range(3):
        ax = 2 - c  # numpy axis of lattice axis c
        n = vol.shape[ax]
        i = np.arange(n)
        i_lo, i_hi = np.maximum(i - 1, 0), np.minimum(i + 1, n - 1)
        h = (np.float32(hi[c]) - np.float32(lo[c])) / np.float32(n - 1)
        num = np.take(vol, i_hi, axis=ax) - np.take(vol, i_lo, axis=ax)
        den = (h * (i_hi - i_lo).astype(np.float32)).astype(np.float32)
        shape = [1, 1, 1]
        shape[ax] = n
        out[..., c] = num / den.reshape(shape)
    return out


def restate(vol, bounds, level, want_dirs=False):
    """numpy marching cubes: (vertices (V, 3) fp32, faces (F, 3) int32, dirs (V, 3) fp32 | None, edge (V, 4) int:
    the lattice point (i, j, k) and axis of each vertex)."""
    vol = np.ascontiguousarray(vol, dtype=np.float32)
    lo, hi = bounds
    n2, n1, n0 = vol.shape
    res = (n0 - 1, n1 - 1, n2 - 1)
    lv = np.float32(level)
    inside = vol > lv
    # classify: each point's +x, +y, +z edges that cross
    cross = np.zeros(vol.shape + (3,), bool)
    cross[:, :, :-1, 0] = inside[:, :, :-1] != inside[:, :, 1:]
    cross[:, :-1, :, 1] = inside[:, :-1, :] != inside[:, 1:, :]
    cross[:-1, :, :, 2] = inside[:-1] != inside[1:]
    # scan: vertex ids in lattice-edge order
    flat = cross.reshape(-1)
    vid = np.where(flat, np.cumsum(flat) - 1, -1).reshape(cross.shape)
    nv = int(flat.sum())
    k, j, i, a = np.nonzero(cross)  # in id order
    step = np.eye(3, dtype=np.int64)[a]
    v0 = vol[k, j, i]
    v1 = vol[k + step[:, 2], j + step[:, 1], i + step[:, 0]]
    t = (lv - v0) / (v1 - v0)
    X = _coords(lo, hi, res)
    p0 = np.stack((X[0][i], X[1][j], X[2][k]), -1)
    p1 = np.stack((X[0][i + step[:, 0]], X[1][j + step[:, 1]], X[2][k + step[:, 2]]), -1)
    verts = p0.copy()
    rows = np.arange(nv)
    verts[rows, a] = p0[rows, a] + t * (p1[rows, a] - p0[rows, a])
    dirs = None
    if want_dirs:
        G = _grad(vol, lo, hi)
        g0 = G[k, j, i]
        g1 = G[k + step[:, 2], j + step[:, 1], i + step[:, 0]]
        g = g0 + t[:, None] * (g1 - g0)
        s = (g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1]) + g[:, 2] * g[:, 2]
        ok = (s > 0) & (s < np.inf)
        with np.errstate(invalid="ignore", divide="ignore"):
            dirs = np.where(ok[:, None], g / np.sqrt(s)[:, None], np.array([0, 0, 1], np.float32)).astype(np.float32)
    # emit faces: cube by cube in linear order, triangles in table order
    case = np.zeros((n2 - 1, n1 - 1, n0 - 1), np.int64)
    for c in range(8):
        dx, dy, dz = c & 1, c >> 1 & 1, c >> 2 & 1
        case |= inside[dz:n2 - 1 + dz, dy:n1 - 1 + dy, dx:n0 - 1 + dx].astype(np.int64) << c
    case = case.reshape(-1)
    cube = np.stack(np.unravel_index(np.arange(case.size), (n2 - 1, n1 - 1, n0 - 1)), -1)  # (k, j, i)
    keep = np.arange(TRIS.shape[1])[None, :] < COUNTS[case][:, None]
    edges = TRIS[case][keep]  # (F, 3) cube edge ids
    owner = np.repeat(cube, COUNTS[case], axis=0)
    off = EDGE_OFF[edges]  # (F, 3, xyz)
    faces = vid[owner[:, None, 0] + off[..., 2], owner[:, None, 1] + off[..., 1], owner[:, None, 2] + off[..., 0],
                edges >> 2]
    assert (faces >= 0).all()
    return verts.astype(np.float32), faces.astype(np.int32), dirs, np.stack((i, j, k, a), -1)


def _lattice(res=64, bounds=BOX):
    X = _coords(bounds[0], bounds[1], (res,) * 3)
    return np.meshgrid(X[0].astype(np.float64), X[1].astype(np.float64), X[2].astype(np.float64), indexing="xy")


def _field(kind, res=64):
    x, y, z = _lattice(res)
    x, y, z = (np.transpose(v, (2, 0, 1)) for v in (x, y, z))  # -> [k][j][i]
    if kind == "sphere":
        f = 0.7 - np.sqrt(x * x + y * y + z * z)
    elif kind == "torus":
        f = 0.25 - np.sqrt((np.sqrt(x * x + y * y) - 0.55) ** 2 + z * z)
    elif kind == "two_spheres":
        f = np.maximum(0.3 - np.sqrt((x - 0.45) ** 2 + y * y + z * z), 0.3 - np.sqrt((x + 0.45) ** 2 + y * y + z * z))
    else:  # seeded random: noise kept below the level near the box's faces
        seed = int(kind.split("_")[1])
        rng = np.random.default_rng(seed)
        f = rng.standard_normal(x.shape)
        f = np.where(np.maximum(np.maximum(abs(x), abs(y)), abs(z)) < 0.85, f, -1.0)
    return np.ascontiguousarray(f, dtype=np.float32)


def _gpu(vol, bounds, level, dirs=False):
    from nerf_pytorch_b200 import mesh, ops

    v = torch.from_numpy(vol).cuda()
    n2, n1, n0 = vol.shape
    box = ops.grid_struct(bounds, (n0 - 1, n1 - 1, n2 - 1))
    verts, faces, d = mesh._surface(v, box, float(level), want_dirs=dirs)
    return verts.cpu().numpy(), faces.cpu().numpy(), None if d is None else d.cpu().numpy()


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def _edges(faces):
    d = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    return d


def _closed_and_oriented(faces):
    d = _edges(faces)
    und = np.sort(d, 1)
    _, cu = np.unique(und, axis=0, return_counts=True)
    _, cd = np.unique(d, axis=0, return_counts=True)
    return bool((cu == 2).all() and (cd == 1).all())


def _euler(verts, faces):
    n_e = np.unique(np.sort(_edges(faces), 1), axis=0).shape[0]
    return verts.shape[0] - n_e + faces.shape[0]


VOLUMES = ["sphere", "torus", "two_spheres", "random_0", "random_1", "random_2"]


@pytest.mark.parametrize("kind", VOLUMES)
def test_mesh_matches_the_numpy_restatement(kind):
    level = 0.0 if not kind.startswith("random") else 0.3
    vol = _field(kind, 48 if kind.startswith("random") else 64)
    v, f, d = _gpu(vol, BOX, level, dirs=True)
    rv, rf, rd, _ = restate(vol, BOX, level, want_dirs=True)
    report("vertices / faces", kind, (v.shape[0], f.shape[0]))
    assert f.shape[0] > 0
    assert np.array_equal(f, rf)
    assert _same_bits(v, rv)
    assert _same_bits(d, rd)


@pytest.mark.parametrize("kind,chi", [("sphere", 2), ("torus", 0), ("two_spheres", 4), ("random_0", None),
                                      ("random_1", None), ("random_2", None)])
def test_topology(kind, chi):
    vol = _field(kind, 48 if kind.startswith("random") else 64)
    v, f, _ = _gpu(vol, BOX, 0.0 if chi is not None else 0.3)
    assert _closed_and_oriented(f), kind
    assert (f[:, 0] != f[:, 1]).all() and (f[:, 1] != f[:, 2]).all() and (f[:, 0] != f[:, 2]).all()
    assert np.unique(f).size == v.shape[0]  # every vertex is used
    if chi is not None:
        assert _euler(v, f) == chi, (kind, _euler(v, f))
    else:
        report("euler characteristic", kind, _euler(v, f))


@pytest.mark.parametrize("kind", ["sphere", "random_0"])
def test_vertices_lie_on_the_level(kind):
    level = 0.0 if kind == "sphere" else 0.3
    vol = _field(kind, 48)
    v, _, _ = _gpu(vol, BOX, level)
    _, _, _, e = restate(vol, BOX, level)
    i, j, k, a = e.T
    X = _coords(BOX[0], BOX[1], (48,) * 3)
    step = np.eye(3, dtype=np.int64)[a]
    p0 = np.stack((X[0][i], X[1][j], X[2][k]), -1).astype(np.float64)
    p1 = np.stack((X[0][i + step[:, 0]], X[1][j + step[:, 1]], X[2][k + step[:, 2]]), -1).astype(np.float64)
    rows = np.arange(v.shape[0])
    tt = (v[rows, a].astype(np.float64) - p0[rows, a]) / (p1[rows, a] - p0[rows, a])
    v0 = vol[k, j, i].astype(np.float64)
    v1 = vol[k + step[:, 2], j + step[:, 1], i + step[:, 0]].astype(np.float64)
    interp = v0 + tt * (v1 - v0)
    eps = np.finfo(np.float32).eps
    h = p1[rows, a] - p0[rows, a]
    tol = abs(v1 - v0) * (4 * eps * (abs(p0[rows, a]) + abs(p1[rows, a])) / h + 4 * eps) + 4 * eps * (
        abs(v0) + abs(v1) + abs(level))
    assert (abs(interp - level) <= tol).all(), float((abs(interp - level) / tol).max())


def test_sphere_volume_and_outward_normals():
    x, y, z = _lattice(128)
    x, y, z = (np.transpose(q, (2, 0, 1)) for q in (x, y, z))
    vol = np.ascontiguousarray(0.7 - np.sqrt(x * x + y * y + z * z), dtype=np.float32)
    v, f, _ = _gpu(vol, BOX, 0.0)
    p = v.astype(np.float64)[f]
    enclosed = np.einsum("ij,ij->i", p[:, 0], np.cross(p[:, 1], p[:, 2])).sum() / 6.0
    want = 4.0 / 3.0 * math.pi * 0.7 ** 3
    report("sphere volume", "r=0.7 @128^3", (enclosed, want))
    assert abs(enclosed - want) < 0.01 * want
    n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    assert (np.einsum("ij,ij->i", n, p.mean(1)) > 0).all()


def test_mesh_repeats_bit_for_bit():
    vol = _field("random_1", 48)
    a = _gpu(vol, BOX, 0.3, dirs=True)
    b = _gpu(vol, BOX, 0.3, dirs=True)
    assert all(_same_bits(x, y) if x.dtype == np.float32 else np.array_equal(x, y) for x, y in zip(a, b))


# ---- networks --------------------------------------------------------------------------------------------------------
def _init_net(hidden, layers, skip, res):
    """A network at init, its sigma bias shifted so that raw sigma changes sign inside the box (at init it may be
    negative everywhere, which leaves no surface)."""
    import nerf_pytorch_b200 as nb

    torch.manual_seed(11)
    m = nb.FlexibleNeRFModel(num_layers=layers, hidden_size=hidden, skip_connect_every=skip, num_encoding_fn_xyz=10,
                             num_encoding_fn_dir=4).cuda()
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    raw = _run_network_sigma(m, epf, edf, LEGO_BOX, res, relu=False)
    with torch.no_grad():
        m.fc_alpha.bias -= raw.median()
    return m, epf, edf


def _run_network_sigma(model, epf, edf, bounds, res, relu=True):
    """relu(sigma) of run_network at the lattice points (formed here in numpy), rows of 64 points, direction +z."""
    import nerf_pytorch_b200 as nb

    X = _coords(bounds[0], bounds[1], (res,) * 3)
    zz, yy, xx = np.meshgrid(X[2], X[1], X[0], indexing="ij")
    pts = torch.from_numpy(np.stack((xx, yy, zz), -1).reshape(-1, 3)).cuda()
    n = pts.shape[0]
    pad = (-n) % 64
    pts = torch.cat((pts, pts[:pad]))
    rows = pts.view(-1, 64, 3)
    ray = torch.tensor([0.0, 0.0, 1.0], device="cuda").expand(rows.shape[0], 3)
    with torch.no_grad():
        raw = nb.run_network(model, rows, ray, 1 << 20, epf, edf)
    sigma = raw.reshape(-1, 4)[:n, 3]
    return (torch.relu(sigma) if relu else sigma).view(res + 1, res + 1, res + 1)


def _open_edges_on_box_faces(v, f, bounds, res):
    d = np.sort(_edges(f), 1)
    u, c = np.unique(d, axis=0, return_counts=True)
    assert (c <= 2).all()
    once = u[c == 1]
    X = _coords(bounds[0], bounds[1], (res,) * 3)
    ends = [(X[ax][0], X[ax][-1]) for ax in range(3)]
    for e in once:
        a, b = v[e[0]], v[e[1]]
        assert any(a[ax] == b[ax] and a[ax] in ends[ax] for ax in range(3)), (a, b)
    return once.shape[0]


def test_lego_volume_is_run_networks_sigma_and_the_mesh_is_open_only_on_the_box():
    import nerf_pytorch_b200 as nb

    model, epf, edf = shipped_models("lego")[1:]
    res = 128
    vol = nb.density_volume(model, epf, LEGO_BOX, res, encode_direction_fn=edf)
    want = _run_network_sigma(model, epf, edf, LEGO_BOX, res)
    assert bits_equal(vol, want)
    level = min(50.0, 0.5 * float(vol.max()))
    report("lego A0 128^3", "max sigma / level", (float(vol.max()), level))
    m = nb.extract_mesh(model, epf, LEGO_BOX, res, level, encode_direction_fn=edf)
    v, f = m.vertices.cpu().numpy(), m.faces.cpu().numpy()
    rv, rf, _, _ = restate(vol.cpu().numpy(), LEGO_BOX, level)
    report("lego A0 128^3", "vertices / faces", (v.shape[0], f.shape[0]))
    assert f.shape[0] > 0 and np.array_equal(f, rf) and _same_bits(v, rv)
    report("lego A0 edges on one face", "", _open_edges_on_box_faces(v, f, LEGO_BOX, res))


def test_lego_colors_are_run_networks_at_the_vertices():
    import nerf_pytorch_b200 as nb

    model, epf, edf = shipped_models("lego")[1:]
    res, level = 64, 50.0
    m = nb.extract_mesh(model, epf, LEGO_BOX, res, level, encode_direction_fn=edf, colors=True)
    vol = nb.density_volume(model, epf, LEGO_BOX, res, encode_direction_fn=edf)
    rv, _, rd, _ = restate(vol.cpu().numpy(), LEGO_BOX, level, want_dirs=True)
    assert _same_bits(m.vertices.cpu().numpy(), rv)
    c = m.colors
    assert c.shape == m.vertices.shape and bool(((c >= 0) & (c <= 1)).all())
    with torch.no_grad():
        raw = nb.run_network(model, m.vertices[:, None, :], torch.from_numpy(rd).cuda(), 1 << 20, epf, edf)
    assert bits_equal(c, torch.sigmoid(raw[:, 0, :3]))


@pytest.mark.parametrize("net", ["a1_init", "hidden256_init"])
def test_other_networks_run_through_the_same_path(net):
    import nerf_pytorch_b200 as nb

    res = 48
    model, epf, edf = _init_net(128, 8, 3, res) if net == "a1_init" else _init_net(256, 4, 4, res)
    vol = nb.density_volume(model, epf, LEGO_BOX, res, encode_direction_fn=edf)
    assert bits_equal(vol, _run_network_sigma(model, epf, edf, LEGO_BOX, res))
    assert bool((vol > 0).any())
    level = float(vol[vol > 0].median())
    m = nb.extract_mesh(model, epf, LEGO_BOX, res, level, encode_direction_fn=edf, colors=True)
    rv, rf, _, _ = restate(vol.cpu().numpy(), LEGO_BOX, level)
    report(net, "vertices / faces", (rv.shape[0], rf.shape[0]))
    assert rf.shape[0] > 0 and np.array_equal(m.faces.cpu().numpy(), rf) and _same_bits(m.vertices.cpu().numpy(), rv)
    assert bool(((m.colors >= 0) & (m.colors <= 1)).all())


def test_volume_and_mesh_do_not_depend_on_the_slab_size():
    import nerf_pytorch_b200 as nb

    model, epf, edf = shipped_models("lego")[1:]
    res = 40
    vols = [nb.density_volume(model, epf, LEGO_BOX, res, encode_direction_fn=edf, planes_per_slab=s)
            for s in (None, 1, 7, 41)]
    assert all(bits_equal(vols[0], v) for v in vols[1:])
    meshes = [nb.extract_mesh(model, epf, LEGO_BOX, res, 50.0, encode_direction_fn=edf, planes_per_slab=s)
              for s in (None, 3)]
    assert bits_equal(meshes[0].vertices, meshes[1].vertices) and torch.equal(meshes[0].faces, meshes[1].faces)


def test_save_ply_round_trips(tmp_path):
    import nerf_pytorch_b200 as nb

    model, epf, edf = shipped_models("lego")[1:]
    m = nb.extract_mesh(model, epf, LEGO_BOX, 32, 50.0, encode_direction_fn=edf, colors=True)
    path = tmp_path / "lego.ply"
    m.save_ply(path)
    data = path.read_bytes()
    head, body = data.split(b"end_header\n", 1)
    nv, nf = m.vertices.shape[0], m.faces.shape[0]
    assert f"element vertex {nv}".encode() in head and f"element face {nf}".encode() in head
    vrec = np.frombuffer(body[: nv * 15], dtype=[("p", "<f4", (3,)), ("c", "u1", (3,))])
    frec = np.frombuffer(body[nv * 15:], dtype=[("n", "u1"), ("v", "<i4", (3,))])
    assert np.array_equal(vrec["p"], m.vertices.cpu().numpy()) and (frec["n"] == 3).all()
    assert np.array_equal(frec["v"], m.faces.cpu().numpy())


def test_refusals_launch_nothing():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    model, epf, edf = shipped_models("lego")[1:]
    before = ops.launch_count()
    cases = [
        (lambda: nb.extract_mesh(model, epf, LEGO_BOX, 1), ValueError),
        (lambda: nb.extract_mesh(model, epf, LEGO_BOX, 1290), ValueError),
        (lambda: nb.extract_mesh(model, epf, ((0, 0, 0), (1, 1, 0)), 8), ValueError),
        (lambda: nb.extract_mesh(model, epf, LEGO_BOX, 8, level=float("nan")), ValueError),
        (lambda: nb.extract_mesh(model, epf, LEGO_BOX, 8, impl=7), NotImplementedError),
        (lambda: nb.extract_mesh(torch.nn.Linear(3, 4).cuda(), epf, LEGO_BOX, 8), NotImplementedError),
        (lambda: nb.extract_mesh(model, lambda x: x * 2, LEGO_BOX, 8), NotImplementedError),
        (lambda: nb.extract_mesh_from_volume(torch.zeros(9, 9, 9), LEGO_BOX, 0.5), NotImplementedError),
        (lambda: nb.extract_mesh_from_volume(torch.zeros(9, 9, 9, device="cuda", dtype=torch.float64), LEGO_BOX, 0.5),
         ValueError),
        (lambda: nb.extract_mesh_from_volume(torch.zeros(2, 9, 9, device="cuda"), LEGO_BOX, 0.5), ValueError),
        (lambda: nb.extract_mesh_from_volume(torch.zeros(9, 9, 9, device="cuda"), LEGO_BOX, float("inf")), ValueError),
    ]
    for fn, err in cases:
        with pytest.raises(err):
            fn()
    torch.cuda.synchronize()
    assert ops.launch_count() == before
