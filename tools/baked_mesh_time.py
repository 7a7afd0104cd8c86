"""Dev tool: meshes of baked fields (nb.extract_baked_mesh; csrc/baked.cu baked_mesh_dirs_kernel /
baked_mesh_colors_kernel over mesh_sparse_count / _emit) against meshes of the network (nb.extract_mesh over the same
grid) on the lego scene.

lego A0 (shipped weights) baked at 256^3 and 512^3 over OccupancyGrid.from_models (128^3) of both networks, unpruned and
transparent-pruned.  The level is the median positive sigma_raw of the 256^3 bake.  It reports, per field:

  baked     extract_baked_mesh without attributes and with colors and normals, ms;
  network   extract_mesh(model_fine, grid=the same grid) over the same lattice, impl 1, without and with colors, ms;
  mesh      vertices and faces of the baked mesh (the network's faces are the same at level >= 0);
  colour    mean absolute difference of the baked vertex colours from the network's.

In one process; the baked and network arms alternate in every round after a warm-up, CUDA events around whole calls
(each ends in its host read of the mesh totals), medians over ROUNDS rounds and their range.  The card's name, power
limit and SM clock are read in the same run.

    python tools/baked_mesh_time.py [--rounds 5] [--res 256 512] [--json OUT]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
from common import card, median, timed_once  # noqa: E402
import nerf_pytorch_b200 as nb  # noqa: E402
from helpers import LEGO_BOX, shipped_models  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--res", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    mc, mf, epf, edf = shipped_models("lego")
    grid = nb.OccupancyGrid.from_models([mc, mf], epf, LEGO_BOX, 128, encode_direction_fn=edf)
    rows, level = [], None
    for res in args.res:
        full = nb.bake(mf, epf, edf, bounds=LEGO_BOX, resolution=res, grid=grid)
        if level is None:
            s = full.values[..., 0]
            level = float(s[s > 0].median())
        for name, f in (("unpruned", full), ("transparent-pruned", nb.prune_baked(full, ~nb.baked_transparent_bricks(full)))):
            arms = {
                "baked": lambda: nb.extract_baked_mesh(f, level),
                "baked colors+normals": lambda: nb.extract_baked_mesh(f, level, colors=True, normals=True),
                "network": lambda: nb.extract_mesh(mf, epf, LEGO_BOX, res, level, edf, impl=1, grid=grid),
                "network colors": lambda: nb.extract_mesh(mf, epf, LEGO_BOX, res, level, edf, colors=True, impl=1,
                                                          grid=grid),
            }
            with torch.no_grad():
                for fn in arms.values():  # warm-up
                    fn()
                ms = {k: [] for k in arms}
                for _ in range(args.rounds):
                    for k, fn in arms.items():
                        ms[k].append(timed_once(fn)[0])
                m = nb.extract_baked_mesh(f, level, colors=True)
                net = nb.extract_mesh(mf, epf, LEGO_BOX, res, level, edf, colors=True, impl=1, grid=grid)
            row = dict(res=res, field=name, bricks=f.n_active, vertices=m.vertices.shape[0], faces=m.faces.shape[0],
                       same_faces=bool(torch.equal(m.faces, net.faces)),
                       color_mad=(m.colors - net.colors).abs().mean().item() if torch.equal(m.faces, net.faces) else None,
                       **{k: median(v) for k, v in ms.items()})
            rows.append(row)
            print(json.dumps(row), flush=True)
        del full
        torch.cuda.empty_cache()
    out = dict(card=card(), level=level, rows=rows)
    print(f"card: {out['card']}  level {level:.4f}")
    print(f"{'res':>5} {'field':>19} {'bricks':>7} {'vertices':>9} {'faces':>9} {'baked ms':>9} {'+attr ms':>9} "
          f"{'net ms':>9} {'net+col':>9} {'colour MAD':>10}")
    for r in rows:
        mad = f"{r['color_mad']:.4f}" if r["color_mad"] is not None else "-"
        print(f"{r['res']:>5} {r['field']:>19} {r['bricks']:>7} {r['vertices']:>9} {r['faces']:>9} "
              f"{r['baked']['ms']:>9.2f} {r['baked colors+normals']['ms']:>9.2f} {r['network']['ms']:>9.2f} "
              f"{r['network colors']['ms']:>9.2f} {mad:>10}")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
