"""Dev tool: dense against sparse nb.extract_mesh on one GPU, for the shipped lego A0 fine network
(tests/golden/weights_lego_lowres.npz) over the box [-1.5, 1.5]^3, level 50, with a grid from
OccupancyGrid.from_models (128^3 cells, threshold 0, the conservative default).  Per lattice (256^3, 512^3 and 1024^3
cubes for both paths, 2048^3 for the sparse path alone, which the dense path refuses):
  * dense:   "density" (nb.density_volume), "count" (ops.mesh_count: classify + scan), "emit" (ops.mesh_emit), and the
             whole extract_mesh call;
  * sparse:  "bricks" (ops.mesh_sparse_bricks), "query" (lattice points and the fused MLP over the active bricks),
             "count" (ops.mesh_sparse_count), "emit" (ops.mesh_sparse_emit), and the whole extract_mesh(grid=) call;
  * lattice points evaluated, active bricks, vertices and faces, and the peak device memory of each whole call
    (torch.cuda.max_memory_allocated above what was allocated before it).
The stages alternate round by round; each figure is the median over ROUNDS rounds of ITERS calls, with its range, from
CUDA events after warm-up.  The card's name, power limit and SM clocks are printed.

    python tools/mesh_sparse_time.py [--rounds 3] [--iters 1] [--res 256 512 1024] [--sparse-only 2048] [--json OUT]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import nerf_pytorch_b200 as nb  # noqa: E402
from nerf_pytorch_b200 import mesh, ops, train_utils  # noqa: E402
from mesh_time import BOX, LEVEL, lego_fine  # noqa: E402
from common import card  # noqa: E402
from run_network_time import compare  # noqa: E402


def peak_bytes(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    r = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del r
    return peak


def sparse_query(arch, blob, use, box, bricks, n_active, per_brick, chunk, pts):
    """The query stage of mesh._sparse_surface: values of the active bricks' lattice points."""
    values = torch.empty(n_active * per_brick, device=blob.device)
    for first in range(0, n_active, chunk):
        cnt = min(chunk, n_active - first)
        n = cnt * per_brick
        rows = -(-n // 64)
        ops.mesh_sparse_points(box, bricks, first, cnt, False, pts)
        dirs = torch.tensor([[0.0, 0.0, 1.0]], device=blob.device).expand(rows, 3) if arch.use_viewdirs else None
        raw = ops.mlp_fwd_pts(arch, blob, pts[:rows * 64].view(rows, 64, 3), dirs, impl=use)
        values[first * per_brick:first * per_brick + n].copy_(torch.relu(raw.view(-1, 4)[:n, 3]))
    return values


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=1)
    ap.add_argument("--res", type=int, nargs="+", default=[256, 512, 1024])
    ap.add_argument("--sparse-only", type=int, nargs="*", default=[2048])
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_sparse_time.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda")
    out = {"card (name, power limit, SM clock, max SM clock)": card(), "rounds": args.rounds, "iters": args.iters,
           "level": LEVEL, "brick": ops.mesh_brick()}
    print("card:", out["card (name, power limit, SM clock, max SM clock)"])
    model = lego_fine(dev)
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    arch = mesh._network(model, epf, edf)
    _, blob = train_utils._packed(model, arch)
    use = mesh._query_impl(arch, None)
    grid = nb.OccupancyGrid.from_models([model], epf, BOX, 128, threshold=0.0, encode_direction_fn=edf)
    out["grid occupied fraction"] = grid.occupied_fraction
    per_brick = (ops.mesh_brick() + 1) ** 3
    with torch.no_grad():
        for res in args.res + args.sparse_only:
            dense = res in args.res
            box = ops.grid_struct(BOX, (res,) * 3)
            n_pts = (res + 1) ** 3
            brick_map, bricks, n_dev = ops.mesh_sparse_bricks(box, grid)
            n_active = int(n_dev.item())
            chunk = max(1, min(n_active, mesh._SLAB_POINTS // per_brick))
            pts = torch.zeros(-(-chunk * per_brick // 64) * 64, 3, device=dev)
            values = sparse_query(arch, blob, use, box, bricks, n_active, per_brick, chunk, pts)
            totals, sws = ops.mesh_sparse_count(box, brick_map, bricks, n_active, values, False, LEVEL)
            s_v, s_f = (int(t) for t in totals.tolist())
            entry = {"lattice_points": n_pts, "active_bricks": n_active, "bricks": ops.mesh_sparse_brick_count(box),
                     "sparse_points_evaluated": n_active * per_brick, "sparse_vertices": s_v, "sparse_faces": s_f}
            fns = {
                "sp:bricks": lambda: ops.mesh_sparse_bricks(box, grid),
                "sp:query": lambda: sparse_query(arch, blob, use, box, bricks, n_active, per_brick, chunk, pts),
                "sp:count": lambda: ops.mesh_sparse_count(box, brick_map, bricks, n_active, values, False, LEVEL, sws),
                "sp:emit": lambda: ops.mesh_sparse_emit(box, brick_map, bricks, n_active, values, False, LEVEL, sws,
                                                        s_v, s_f),
                "sp:total": lambda: nb.extract_mesh(model, epf, BOX, res, LEVEL, encode_direction_fn=edf, grid=grid),
            }
            if dense:
                vol = nb.density_volume(model, epf, BOX, res, encode_direction_fn=edf)
                dtot, dws = ops.mesh_count(box, vol, LEVEL)
                d_v, d_f = (int(t) for t in dtot.tolist())
                entry.update({"dense_vertices": d_v, "dense_faces": d_f})
                fns.update({
                    "dn:density": lambda: nb.density_volume(model, epf, BOX, res, encode_direction_fn=edf),
                    "dn:count": lambda: ops.mesh_count(box, vol, LEVEL, dws),
                    "dn:emit": lambda: ops.mesh_emit(box, vol, LEVEL, dws, d_v, d_f),
                    "dn:total": lambda: nb.extract_mesh(model, epf, BOX, res, LEVEL, encode_direction_fn=edf),
                })
            print(f"{res}^3 cubes: {n_pts} lattice points, {n_active} of {entry['bricks']} bricks active, "
                  f"{entry['sparse_points_evaluated']} points evaluated ({entry['sparse_points_evaluated'] / n_pts:.3f} "
                  f"of the lattice), sparse {s_v} vertices / {s_f} faces"
                  + (f", dense {entry['dense_vertices']} / {entry['dense_faces']}" if dense else ""), flush=True)
            entry["times"] = compare(f"lego A0 fine {res}^3", fns, args.rounds, args.iters, n_pts)
            if dense:
                del vol, dws
            del values, sws, pts, brick_map, bricks
            torch.cuda.empty_cache()
            entry["peak_bytes_sparse"] = peak_bytes(
                lambda: nb.extract_mesh(model, epf, BOX, res, LEVEL, encode_direction_fn=edf, grid=grid))
            if dense:
                torch.cuda.empty_cache()
                entry["peak_bytes_dense"] = peak_bytes(
                    lambda: nb.extract_mesh(model, epf, BOX, res, LEVEL, encode_direction_fn=edf))
            print(f"{res}^3 peak device memory: sparse {entry['peak_bytes_sparse'] / 2 ** 20:.0f} MiB"
                  + (f", dense {entry['peak_bytes_dense'] / 2 ** 20:.0f} MiB" if dense else ""), flush=True)
            out[f"{res}^3"] = entry
            torch.cuda.empty_cache()
    print("card:", card())
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
