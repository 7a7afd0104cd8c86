"""Dev tool: what the NDC -> world map costs a mesh extraction of a forward-facing scene, on one GPU.  The shipped fern
fine network (tests/golden/weights_fern_lowres.npz, A0 with 6 / 4 bands) over the NDC box [-1, 1] x [-1, 1] x
[-1, 0.95], at the level of the median positive density of a 64^3 lattice, with a grid from OccupancyGrid.from_models
(128^3 cells over the same box, threshold 0).  Per lattice (256^3 and 512^3 cubes by default):
  * "dn" / "dn:ndc": nb.extract_mesh dense, without and with ndc=(42, 56, 45.3);
  * "sp" / "sp:ndc": the same with grid=;
  * "map": ops.ndc_mesh_to_world alone on the dense mesh with its view directions (vertices, faces and directions).
Colors and normals are off, so the difference between a pair is the map itself.  The calls alternate round by round;
each figure is the median over ROUNDS rounds of ITERS calls, with its range, from CUDA events after warm-up.  The
card's name, power limit and SM clocks are printed.

    python tools/ndc_mesh_time.py [--rounds 5] [--iters 1] [--res 256 512] [--json OUT]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import nerf_pytorch_b200 as nb  # noqa: E402
from nerf_pytorch_b200 import ops  # noqa: E402
from run_network_time import card, compare  # noqa: E402

BOX = ((-1.0, -1.0, -1.0), (1.0, 1.0, 0.95))
HWF = (42, 56, 45.3)


def fern_fine(dev):
    import numpy as np

    z = np.load(os.path.join(ROOT, "tests", "golden", "weights_fern_lowres.npz"))
    sd = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("f.")}
    m = nb.FlexibleNeRFModel(num_layers=4, hidden_size=128, skip_connect_every=4, num_encoding_fn_xyz=6,
                             num_encoding_fn_dir=4)
    m.load_state_dict(sd)
    for p in m.parameters():
        p.requires_grad_(False)
    return m.to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=1)
    ap.add_argument("--res", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ndc_mesh_time.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda")
    out = {"card (name, power limit, SM clock, max SM clock)": card(), "rounds": args.rounds, "iters": args.iters,
           "box": BOX, "hwf": HWF}
    print("card:", out["card (name, power limit, SM clock, max SM clock)"])
    model = fern_fine(dev)
    epf, edf = nb.get_embedding_function(6), nb.get_embedding_function(4)
    with torch.no_grad():
        vol = nb.density_volume(model, epf, BOX, 64, encode_direction_fn=edf)
        level = float(vol[vol > 0].median())
        out["level"] = level
        grid = nb.OccupancyGrid.from_models([model], epf, BOX, 128, threshold=0.0, encode_direction_fn=edf)
        out["grid occupied fraction"] = grid.occupied_fraction
        cam = ops.ndc_struct(*HWF)
        for res in args.res:
            box = ops.grid_struct(BOX, (res,) * 3)
            vol = nb.density_volume(model, epf, BOX, res, encode_direction_fn=edf)
            totals, ws = ops.mesh_count(box, vol, level)
            n_v, n_f = (int(t) for t in totals.tolist())
            v, f, d = ops.mesh_emit(box, vol, level, ws, n_v, n_f, want_dirs=True)
            del vol, ws
            kw = dict(encode_direction_fn=edf)
            fns = {
                "dn": lambda: nb.extract_mesh(model, epf, BOX, res, level, **kw),
                "dn:ndc": lambda: nb.extract_mesh(model, epf, BOX, res, level, ndc=HWF, **kw),
                "sp": lambda: nb.extract_mesh(model, epf, BOX, res, level, grid=grid, **kw),
                "sp:ndc": lambda: nb.extract_mesh(model, epf, BOX, res, level, grid=grid, ndc=HWF, **kw),
                "map": lambda: ops.ndc_mesh_to_world(cam, v, f, d),
            }
            print(f"{res}^3 cubes: level {level:.3f}, {n_v} vertices, {n_f} faces", flush=True)
            out[f"{res}^3"] = {"vertices": n_v, "faces": n_f,
                               "times": compare(f"fern fine {res}^3", fns, args.rounds, args.iters, (res + 1) ** 3)}
            del v, f, d
            torch.cuda.empty_cache()
    print("card:", card())
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
