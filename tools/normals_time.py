"""Dev tool: the cost of the density gradient (nb.density_gradient / ops.density_grad) on one GPU.
  * points   A1 and A2 at init and the shipped lego A0 fine network on 2^20 .. 2^24 points uniform in [-1.5, 1.5]^3:
             density_grad (sigma + its gradient) against the wgmma inference forward alone (mlp_fwd_pts, impl 1, rows
             of 64 points) and against eager torch autograd of sigma w.r.t. the points (the model in torch on the same
             GPU, chunks of 2^20 points; at the smallest size only, it is slow);
  * mesh     nb.extract_mesh of lego A0 at 256^3 cubes, level 50, with and without normals=True.
The contenders alternate round by round; each figure is the median over ROUNDS rounds of ITERS calls, with its range,
from CUDA events after warm-up.  The card's name, power limit and SM clocks are printed.
    python tools/normals_time.py [--rounds 5] [--iters 3] [--log2 20 22 24] [--json OUT]"""
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
from mesh_time import lego_fine  # noqa: E402
from run_network_time import EAGER_CHUNK, card, compare, torch_encoding  # noqa: E402

BOX = ((-1.5,) * 3, (1.5,) * 3)


def init_model(layers, hidden, skip, dev):
    torch.manual_seed(5)
    return nb.FlexibleNeRFModel(num_layers=layers, hidden_size=hidden, skip_connect_every=skip, num_encoding_fn_xyz=10,
                                num_encoding_fn_dir=4).to(dev)


def eager_grad(model, pts):
    """sigma and d sigma / d x by torch autograd through the model and the encoding, in chunks."""
    out = []
    d = torch_encoding(torch.tensor([[0.0, 0.0, 1.0]], device=pts.device), 4)
    for i in range(0, pts.shape[0], EAGER_CHUNK):
        x = pts[i:i + EAGER_CHUNK].clone().requires_grad_()
        emb = torch.cat((torch_encoding(x, 10), d.expand(x.shape[0], -1)), -1)
        s = model(emb)[:, 3]
        g, = torch.autograd.grad(s.sum(), x)
        out.append(g)
    return torch.cat(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--log2", type=int, nargs="+", default=[20, 22, 24])
    ap.add_argument("--mesh-res", type=int, default=256)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("normals_time.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda")
    out = {"card (name, power limit, SM clock, max SM clock)": card(), "rounds": args.rounds, "iters": args.iters}
    print("card:", out["card (name, power limit, SM clock, max SM clock)"], flush=True)
    nets = {"A1 init": init_model(8, 128, 3, dev), "A2 init": init_model(8, 256, 4, dev), "lego A0": lego_fine(dev)}
    epf = nb.get_embedding_function(10)
    for name, model in nets.items():
        arch = mesh._network(model, epf, None)
        _, blob = train_utils._packed(model, arch)
        for lg in args.log2:
            n = 1 << lg
            g = torch.Generator(device=dev).manual_seed(lg)
            pts = torch.rand(n, 3, device=dev, generator=g) * 3.0 - 1.5
            rows = pts.view(-1, 64, 3)
            dirs = torch.tensor([[0.0, 0.0, 1.0]], device=dev).expand(rows.shape[0], 3) if arch.use_viewdirs else None
            fns = {"density_grad": lambda: ops.density_grad(arch, blob, pts),
                   "forward": lambda: ops.mlp_fwd_pts(arch, blob, rows, dirs, impl=ops.IMPL_TC)}
            if lg == min(args.log2):
                fns["eager autograd"] = lambda: eager_grad(model, pts)
            out[f"{name} 2^{lg}"] = compare(f"{name} 2^{lg} points", fns, args.rounds, args.iters, n)
            del pts, rows
            torch.cuda.empty_cache()
    model = nets["lego A0"]
    edf = nb.get_embedding_function(4)
    res = args.mesh_res
    with torch.no_grad():
        m = nb.extract_mesh(model, epf, BOX, res, 50.0, encode_direction_fn=edf, normals=True)
        n_v = m.vertices.shape[0]
        fns = {"extract_mesh": lambda: nb.extract_mesh(model, epf, BOX, res, 50.0, encode_direction_fn=edf),
               "extract_mesh normals": lambda: nb.extract_mesh(model, epf, BOX, res, 50.0, encode_direction_fn=edf,
                                                               normals=True)}
        out[f"lego A0 mesh {res}^3"] = {"vertices": n_v,
                                        "times": compare(f"lego A0 mesh {res}^3 ({n_v} vertices)", fns, args.rounds,
                                                         args.iters, n_v)}
    print("card:", card())
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
