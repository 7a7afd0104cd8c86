"""CPU: the marching-cubes case table and the mesh refusals that need no GPU.
  1. the committed table (csrc/mc_table.cuh, parsed here) against an independent statement of the face rule: on every
     face of every case the triangles' edges are exactly the rule's segments, in the rule's direction;
  2. every triangle lies on crossed edges only, and no triangle repeats an edge;
  3. each case's boundary closes into polygons, and each polygon's area vector points from its inside corners out;
  4. tools/gen_mc_table.py regenerates the committed header byte for byte;
  5. the C symbols are exported, and every refusal of the Python API fires before anything touches a device."""
import ctypes as C
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "nerf_pytorch_b200", "csrc", "mc_table.cuh")


def _table():
    text = open(HEADER).read()
    width = int(re.search(r"#define NERFB200_MC_MAX_TRIS (\d+)", text).group(1))
    counts_src = re.search(r"kMcTriCount\[256\] = \{(.*?)\};", text, re.S).group(1)
    counts = [int(v) for v in re.findall(r"-?\d+", counts_src)]
    tris_src = re.search(r"kMcTris\[256\]\[\d+\] = \{(.*?)\n\};", text, re.S).group(1)
    rows = re.findall(r"\{([^}]*)\}", tris_src)
    tris = [[int(v) for v in r.split(",")] for r in rows]
    assert len(counts) == 256 and len(tris) == 256 and all(len(r) == 3 * width for r in tris)
    out = []
    for case in range(256):
        r = tris[case]
        assert all(v == -1 for v in r[3 * counts[case]:])
        out.append([tuple(r[3 * t: 3 * t + 3]) for t in range(counts[case])])
    return out


def _corner(c):
    return np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1], dtype=np.float64)


def _edge_corners(e):
    a, m = e >> 2, e & 3
    u, v = [ax for ax in range(3) if ax != a]
    lo = ((m & 1) << u) | ((m >> 1) << v)
    return lo, lo | (1 << a)


def _faces():
    """(corners in cyclic order, outward normal) of the six cube faces."""
    out = []
    for axis in range(3):
        u, v = [ax for ax in range(3) if ax != axis]
        for side in (0, 1):
            b = side << axis
            n = np.zeros(3)
            n[axis] = 1.0 if side else -1.0
            out.append(([b, b | 1 << u, b | 1 << u | 1 << v, b | 1 << v], n))
    return out


def _edge(c0, c1):
    return next(e for e in range(12) if set(_edge_corners(e)) == {c0, c1})


def _mid(e):
    c0, c1 = _edge_corners(e)
    return (_corner(c0) + _corner(c1)) / 2


def _rule(case, ring):
    """The face rule, stated on its own: undirected segments {edge, edge} on one face.  Each corner both of whose face
    edges cross is cut off, except that on a face with two diagonal inside corners only the inside ones are; two
    adjacent inside corners give the segment between the two crossed edges."""
    ins = [bool(case >> c & 1) for c in ring]
    edges = [_edge(ring[i], ring[(i + 1) % 4]) for i in range(4)]
    crossed = [ins[i] != ins[(i + 1) % 4] for i in range(4)]
    if sum(crossed) == 0:
        return set()
    if sum(crossed) == 2 and sum(ins) == 2:
        return {frozenset(e for e, x in zip(edges, crossed) if x)}
    segs = set()
    for i in range(4):
        if crossed[i - 1] and crossed[i] and (sum(ins) != 2 or ins[i]):
            segs.add(frozenset((edges[i - 1], edges[i])))
    return segs


TABLE = _table()


def test_table_faces_carry_exactly_the_face_rule_segments():
    for case in range(256):
        tris = TABLE[case]
        directed = {(t[k], t[(k + 1) % 3]) for t in tris for k in range(3)}
        for ring, normal in _faces():
            on_face = [e for e in range(12) if set(_edge_corners(e)) <= set(ring)]
            got = {frozenset(d) for d in directed if d[0] in on_face and d[1] in on_face}
            assert got == _rule(case, ring), (case, ring)
            for a, b in directed:
                if a in on_face and b in on_face:
                    # seen from outside the cube, the surface is on the inner side of the face: the segment's direction
                    # crossed with the face's inward normal points from the inside corners to the outside ones
                    ins = [c for c in ring if case >> c & 1 and (c in _edge_corners(a) or c in _edge_corners(b))]
                    out = [c for c in ring if not case >> c & 1 and (c in _edge_corners(a) or c in _edge_corners(b))]
                    s = np.mean([_corner(c) for c in out], 0) - np.mean([_corner(c) for c in ins], 0)
                    assert np.dot(np.cross(s, _mid(b) - _mid(a)), -normal) > 0, (case, a, b)


def test_triangles_lie_on_crossed_edges_only():
    for case in range(256):
        crossed = {e for e in range(12) if (case >> _edge_corners(e)[0] & 1) != (case >> _edge_corners(e)[1] & 1)}
        used = {e for t in TABLE[case] for e in t}
        assert used == crossed, case
        for t in TABLE[case]:
            assert len(set(t)) == 3, (case, t)
        undirected = [frozenset((t[k], t[(k + 1) % 3])) for t in TABLE[case] for k in range(3)]
        assert all(undirected.count(u) <= 2 for u in undirected), case


def test_polygons_close_and_face_outward():
    for case in range(256):
        directed = [(t[k], t[(k + 1) % 3]) for t in TABLE[case] for k in range(3)]
        assert len(set(directed)) == len(directed), case  # consistently oriented inside the cube
        boundary = [d for d in directed if (d[1], d[0]) not in directed]
        outs, ins = {}, {}
        for a, b in boundary:
            outs[a] = outs.get(a, 0) + 1
            ins[b] = ins.get(b, 0) + 1
        assert outs == ins and all(v == 1 for v in outs.values()), case
        # each polygon (the triangles joined by shared edges) has an area vector that points from its inside corners
        # to its outside corners: summed over the polygon's cube edges, outside end minus inside end
        polys = []
        for t in TABLE[case]:
            hit = [p for p in polys if set(t) & p["edges"]]
            merged = {"edges": set(t), "tris": [t]}
            for p in hit:
                merged["edges"] |= p["edges"]
                merged["tris"] += p["tris"]
                polys.remove(p)
            polys.append(merged)
        for p in polys:
            area = sum(np.cross(_mid(t[1]) - _mid(t[0]), _mid(t[2]) - _mid(t[0])) for t in p["tris"])
            span = 0.0
            for e in p["edges"]:
                c0, c1 = _edge_corners(e)
                c_in, c_out = (c0, c1) if case >> c0 & 1 else (c1, c0)
                span += np.dot(area, _corner(c_out) - _corner(c_in))
            assert span > 0, (case, p)


def test_regenerating_the_table_gives_the_committed_header():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gen_mc_table.py"), "--check"], capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "up to date" in r.stdout
    largest, width = map(int, re.search(r"largest triangle count per case: (\d+) \(table width (\d+)\)",
                                        r.stdout).groups())
    assert largest <= width and max(len(t) for t in TABLE) == largest


def test_symbols_are_exported_and_queries_refuse_bad_boxes():
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    for name in ("nerfb200_mesh_count", "nerfb200_mesh_emit", "nerfb200_mesh_workspace_bytes",
                 "nerfb200_mesh_lattice_points"):
        assert name in _lib.SIGNATURES and hasattr(lib, name)
    ok = ops.grid_struct(((-1, -1, -1), (1, 1, 1)), (256, 256, 256))
    assert ops.mesh_workspace_bytes(ok) > 0
    for bad in ((((-1, -1, -1), (1, 1, 1)), (1290, 1290, 1290)),  # 1291^3 lattice points > 2^31
                (((0, 0, 0), (1, 1, 1)), (0, 4, 4)), (((0, 0, 0), (1, 0, 1)), (4, 4, 4))):
        assert lib.nerfb200_mesh_workspace_bytes(C.byref(ops.grid_struct(*bad))) == -1


def test_every_refusal_fires_before_any_launch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    model = nb.FlexibleNeRFModel()  # on the CPU
    epf = nb.get_embedding_function(6)
    before = ops.launch_count()
    box = ((-1.0,) * 3, (1.0,) * 3)
    for kw, err in ((dict(resolution=1), ValueError), (dict(resolution=1290), ValueError),
                    (dict(bounds=((0, 0, 0), (1, -1, 1))), ValueError),
                    (dict(bounds=((0, 0, math.nan), (1, 1, 1))), ValueError),
                    (dict(bounds=((0, 0, 0), (1, 1, math.inf))), ValueError),
                    (dict(level=math.nan), ValueError), (dict(level=math.inf), ValueError),
                    (dict(), NotImplementedError)):
        args = dict(bounds=box, resolution=8, level=1.0)
        args.update(kw)
        with pytest.raises(err):
            nb.extract_mesh(model, epf, **args)
    with pytest.raises(NotImplementedError, match="FlexibleNeRFModel"):
        nb.extract_mesh(torch.nn.Linear(3, 4), epf, box, 8)
    with pytest.raises(NotImplementedError, match="CUDA"):
        nb.extract_mesh_from_volume(torch.zeros(9, 9, 9), box, 0.5)
    assert ops.launch_count() == before
