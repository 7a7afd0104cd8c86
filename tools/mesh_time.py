"""Dev tool: the cost of nb.extract_mesh on one GPU, stage by stage, for the shipped lego A0 fine network
(tests/golden/weights_lego_lowres.npz) over the box [-1.5, 1.5]^3 at 256^3 and 512^3 cubes, level 50:
  * density   nb.density_volume: the (R + 1)^3 lattice through the fused MLP (wgmma inference forward), slab by slab;
  * count     ops.mesh_count: classify + scan;
  * emit      ops.mesh_emit: vertices and faces (and, as "emit+dirs", with the view directions colors need);
  * colors    the colors query: sigmoid(rgb) at every vertex, one sample per row, so on the fp32 kernels;
  * eager     the eager-torch density query on the same lattice points (the reference's run_network in torch, in chunks
              of 2^20 points), the yardstick.
The contenders alternate round by round; each figure is the median over ROUNDS rounds of ITERS calls, with its range,
from CUDA events after warm-up.  Vertex and face counts, the card's name, power limit and SM clocks are printed.

    python tools/mesh_time.py [--rounds 5] [--iters 3] [--res 256 512] [--json OUT]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import nerf_pytorch_b200 as nb  # noqa: E402
from nerf_pytorch_b200 import mesh, ops, train_utils  # noqa: E402
from common import card  # noqa: E402
from run_network_time import EAGER_CHUNK, compare, eager_run_network  # noqa: E402

BOX = ((-1.5,) * 3, (1.5,) * 3)
LEVEL = 50.0


def lego_fine(dev):
    z = np.load(os.path.join(ROOT, "tests", "golden", "weights_lego_lowres.npz"))
    sd = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("f.")}
    m = nb.FlexibleNeRFModel(num_layers=4, hidden_size=128, skip_connect_every=4, num_encoding_fn_xyz=10,
                             num_encoding_fn_dir=4)
    m.load_state_dict(sd)
    return m.to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--res", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_time.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda")
    out = {"card (name, power limit, SM clock, max SM clock)": card(), "rounds": args.rounds, "iters": args.iters,
           "level": LEVEL}
    print("card:", out["card (name, power limit, SM clock, max SM clock)"])
    model = lego_fine(dev)
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    arch = mesh._network(model, epf, edf)
    _, blob = train_utils._packed(model, arch)
    color_impl = train_utils._auto_impl(arch, None, 1, 0, training=False)
    view = torch.tensor([[0.0, 0.0, 1.0]], device=dev)
    with torch.no_grad():
        for res in args.res:
            box = ops.grid_struct(BOX, (res,) * 3)
            vol = nb.density_volume(model, epf, BOX, res, encode_direction_fn=edf)
            totals, ws = ops.mesh_count(box, vol, LEVEL)
            n_v, n_f = (int(t) for t in totals.tolist())
            verts, _, dirs = ops.mesh_emit(box, vol, LEVEL, ws, n_v, n_f, want_dirs=True)
            pts = torch.empty((res + 1) ** 3, 3, device=dev)
            ops.mesh_lattice_points(box, 0, res + 1, pts)
            pts = pts.view(1, -1, 3)
            n_pts = (res + 1) ** 3
            print(f"{res}^3 cubes: {n_pts} lattice points, max sigma {float(vol.max()):.1f}, {n_v} vertices, "
                  f"{n_f} faces", flush=True)
            fns = {
                "density": lambda: nb.density_volume(model, epf, BOX, res, encode_direction_fn=edf),
                "count": lambda: ops.mesh_count(box, vol, LEVEL, ws),
                "emit": lambda: ops.mesh_emit(box, vol, LEVEL, ws, n_v, n_f),
                "emit+dirs": lambda: ops.mesh_emit(box, vol, LEVEL, ws, n_v, n_f, want_dirs=True),
                "colors": lambda: torch.sigmoid(ops.mlp_fwd_pts(arch, blob, verts.view(-1, 1, 3), dirs,
                                                                impl=color_impl)[..., :3]),
                "eager": lambda: eager_run_network(model, pts, view),
            }
            out[f"{res}^3"] = {"lattice_points": n_pts, "vertices": n_v, "faces": n_f,
                               "times": compare(f"lego A0 fine {res}^3", fns, args.rounds, args.iters, n_pts)}
            del vol, ws, pts, verts, dirs
            torch.cuda.empty_cache()
    print("card:", card())
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
