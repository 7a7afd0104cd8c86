"""Derive the face-consistent marching-cubes case table and write nerf_pytorch_b200/csrc/mc_table.cuh.

Conventions (include/nerfb200.h "meshes"):
  corner c in 0..7 of a cube sits at offset (c & 1, (c >> 1) & 1, (c >> 2) & 1) in (x, y, z); a corner is inside when its
  value exceeds the level, and the case is the sum of (inside << c).
  edge e in 0..11 runs along axis a = e >> 2 from the corner whose other two coordinates are the bits of m = e & 3 (the
  lower axis first): axis x takes (y, z) = (m & 1, m >> 1), axis y takes (x, z), axis z takes (x, y).  It is the lattice
  edge along a owned by the lattice point at the cube's low corner plus that offset.

For every case, on each of the six cube faces the crossed edges are joined by one fixed rule that reads only that face's
four corner signs: one or three inside corners cut off the odd corner, two adjacent ones give the segment between the two
crossed (parallel) edges, and two diagonal inside corners (the ambiguous face) are kept apart, each cut off by its own
segment.  Each segment is directed so that the surface's normal, by the right-hand rule, points from inside to outside.
Every crossed edge then has one incoming and one outgoing segment, so the segments chain into closed polygons, which are
fan-triangulated.  The apex of the fan is the first vertex (lowest position in the chain started at the lowest edge id)
whose diagonals join no two vertices on a common cube face: a diagonal lying on a face would be drawn by the cube on the
other side of that face too.  Two cubes sharing a face see the same four corner signs, so they put the same segments on
it, in opposite directions: the mesh is closed and consistently oriented wherever the surface stays inside the lattice.

    python tools/gen_mc_table.py          # rewrite the header
    python tools/gen_mc_table.py --check  # exit 1 if the committed header differs
"""
from __future__ import annotations

import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "nerf_pytorch_b200", "csrc", "mc_table.cuh")
MAX_TRIS = 5  # the table's width in triangles; build() asserts every case fits


def corner_pos(c):
    return (c & 1, (c >> 1) & 1, (c >> 2) & 1)


def edge_corners(e):
    """The two corners of edge e, low end first."""
    a, m = e >> 2, e & 3
    others = [ax for ax in range(3) if ax != a]
    lo = ((m & 1) << others[0]) | ((m >> 1) << others[1])
    return lo, lo | (1 << a)


def edge_of(c0, c1):
    for e in range(12):
        if set(edge_corners(e)) == {c0, c1}:
            return e
    raise ValueError((c0, c1))


def edge_mid(e):
    c0, c1 = edge_corners(e)
    return tuple((p + q) / 2 for p, q in zip(corner_pos(c0), corner_pos(c1)))


# the six faces: (axis, side); corners in cyclic order around the face, and the outward normal
FACES = []
for axis in range(3):
    u, v = [ax for ax in range(3) if ax != axis]
    for side in (0, 1):
        base = side << axis
        ring = [base, base | (1 << u), base | (1 << u) | (1 << v), base | (1 << v)]
        normal = [0, 0, 0]
        normal[axis] = 1 if side else -1
        FACES.append((ring, tuple(normal)))


def _sub(p, q):
    return tuple(a - b for a, b in zip(p, q))


def _cross(p, q):
    return (p[1] * q[2] - p[2] * q[1], p[2] * q[0] - p[0] * q[2], p[0] * q[1] - p[1] * q[0])


def _dot(p, q):
    return sum(a * b for a, b in zip(p, q))


def face_segments(case, face):
    """The face rule: directed segments (edge_from, edge_to) on one face for one case."""
    ring, normal = face
    inside = [bool((case >> c) & 1) for c in ring]
    face_edges = [edge_of(ring[i], ring[(i + 1) % 4]) for i in range(4)]  # edge i joins ring[i], ring[i+1]
    crossed = [inside[i] != inside[(i + 1) % 4] for i in range(4)]
    n_in = sum(inside)
    segs = []  # (edge_a, edge_b, inside_point, outside_point)
    centre = tuple(sum(corner_pos(c)[k] for c in ring) / 4 for k in range(3))
    if n_in in (1, 3) or (n_in == 2 and inside[0] == inside[2]):
        # cut off every corner both of whose face edges are crossed: the odd corner of one or three inside, or each
        # inside corner of an ambiguous face
        for i in range(4):
            prev_e, next_e = face_edges[(i - 1) % 4], face_edges[i]
            if not (crossed[(i - 1) % 4] and crossed[i]):
                continue
            if n_in == 2 and not inside[i]:
                continue  # ambiguous face: the inside corners are the ones cut off, kept apart
            p = corner_pos(ring[i])
            ins, out = (p, centre) if inside[i] else (centre, p)
            segs.append((prev_e, next_e, ins, out))
    elif n_in == 2:
        idx = [i for i in range(4) if crossed[i]]
        ea, eb = face_edges[idx[0]], face_edges[idx[1]]
        ins = tuple(sum(corner_pos(ring[i])[k] for i in range(4) if inside[i]) / 2 for k in range(3))
        out = tuple(sum(corner_pos(ring[i])[k] for i in range(4) if not inside[i]) / 2 for k in range(3))
        segs.append((ea, eb, ins, out))
    directed = []
    inward = tuple(-x for x in normal)
    for ea, eb, ins, out in segs:
        d = _sub(edge_mid(eb), edge_mid(ea))
        s = _sub(out, ins)
        # the polygon lies to the left of its direction seen from its normal's side, and reaches into the cube
        sign = _dot(_cross(s, d), inward)
        assert sign != 0
        directed.append((ea, eb) if sign > 0 else (eb, ea))
    return directed


def polygons(case):
    nxt = {}
    for face in FACES:
        for a, b in face_segments(case, face):
            assert a not in nxt, (case, a)
            nxt[a] = b
    assert sorted(nxt) == sorted(set(nxt.values())), case
    polys, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        poly, e = [], start
        while e not in seen:
            seen.add(e)
            poly.append(e)
            e = nxt[e]
        assert e == start, case
        polys.append(poly)
    return polys


def share_face(e0, e1):
    c0, c1 = set(edge_corners(e0)), set(edge_corners(e1))
    return any(c0 <= set(ring) and c1 <= set(ring) for ring, _ in FACES)


def fan(poly):
    k = len(poly)
    for a in range(k):
        diagonals = [poly[(a + i) % k] for i in range(2, k - 1)]
        if all(not share_face(poly[a], d) for d in diagonals):
            return [(poly[a], poly[(a + i) % k], poly[(a + i + 1) % k]) for i in range(1, k - 1)]
    raise AssertionError(f"no fan apex without a face diagonal for polygon {poly}")


def build():
    """tri_count[256], tris[256] (lists of (e0, e1, e2)), polys[256]."""
    tris, polys = [], []
    for case in range(256):
        ps = polygons(case)
        polys.append(ps)
        tris.append([t for p in ps for t in fan(p)])
    widest = max(len(t) for t in tris)
    assert widest <= MAX_TRIS, f"a case needs {widest} triangles; the table holds {MAX_TRIS}"
    return [len(t) for t in tris], tris, polys


def render():
    counts, tris, _ = build()
    lines = [
        "// mc_table.cuh -- generated by tools/gen_mc_table.py; do not edit.",
        "// The face-consistent marching-cubes case table (corner, edge and case conventions in that script and in",
        "// include/nerfb200.h \"meshes\").  kMcTris[case] lists kMcTriCount[case] triangles as cube edge ids, three per",
        f"// triangle, counter-clockwise seen from outside; unused entries are -1.  Largest count: {max(counts)}.",
        "#pragma once",
        "",
        f"#define NERFB200_MC_MAX_TRIS {MAX_TRIS}",
        "",
        "__constant__ unsigned char kMcTriCount[256] = {",
    ]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(c) for c in counts[r:r + 32]) + ",")
    lines.append("};")
    lines.append("")
    lines.append(f"__constant__ signed char kMcTris[256][{3 * MAX_TRIS}] = {{")
    for case in range(256):
        flat = [e for t in tris[case] for e in t]
        flat += [-1] * (3 * MAX_TRIS - len(flat))
        lines.append("    {" + ", ".join(str(e) for e in flat) + f"}},  // {case}")
    lines.append("};")
    return "\n".join(lines) + "\n"


def main():
    text = render()
    counts, _, _ = build()
    print(f"largest triangle count per case: {max(counts)} (table width {MAX_TRIS})")
    if "--check" in sys.argv:
        with open(OUT) as f:
            same = f.read() == text
        print("mc_table.cuh is " + ("up to date" if same else "STALE"))
        sys.exit(0 if same else 1)
    with open(OUT, "w") as f:
        f.write(text)
    print(f"wrote {OUT}")


if __name__ == "__main__":
    main()
