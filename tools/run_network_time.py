"""Dev tool: throughput of run_network (the fused MLP at caller-given points) against the eager-torch equivalent, on one
GPU, in one process, alternating the contenders round by round, CUDA events after warm-up:
  * a density-grid query under torch.no_grad(): 256^3 points (1, 256^3, 3) with one view direction, for A0 and A1;
    impl 1 (wgmma), impl 3 (single-pass fp16 wgmma) and eager torch, i.e. models.FlexibleNeRFModel.forward on a torch
    positional encoding (the reference's run_network, nerf/train_utils.py:8-25, in chunks of EAGER_CHUNK points so that
    its activations fit);
  * a training-shaped call, 4096 rows x 64 samples: run_network forward + backward of a sum, impl 1 against eager torch.
Each figure is the median over ROUNDS rounds of ITERS calls, with its range.  The card's name, power limit and SM clocks
are printed beside the numbers.

    python tools/run_network_time.py [--rounds 5] [--iters 5] [--json OUT]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nerf_pytorch_b200 as nb  # noqa: E402
from nerf_pytorch_b200 import ops  # noqa: E402

ARCHS = {  # bench.py's architectures
    "A0": dict(num_layers=4, hidden_size=128, skip_connect_every=4),
    "A1": dict(num_layers=8, hidden_size=128, skip_connect_every=3),
}
GRID = 256
EAGER_CHUNK = 1 << 20


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True,
                           timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover - depends on the host
        q = f"nvidia-smi unavailable ({e})"
    return q or torch.cuda.get_device_name()


def timed(fn, iters):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def compare(name, fns, rounds, iters, points, warmup=2):
    """fns: {label: callable}, alternated; prints and returns median ms, points/s and the range over the rounds."""
    for _ in range(warmup):
        for f in fns.values():
            f()
    ms = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            ms[k].append(timed(f, iters))
    res = {}
    for k, v in ms.items():
        med = statistics.median(v)
        res[k] = {"median_ms": med, "min_ms": min(v), "max_ms": max(v), "points_per_s": points / (med * 1e-3)}
        print(f"{name:40s} {k:8s} {med:9.3f} ms (range {min(v):.3f} - {max(v):.3f})  "
              f"{res[k]['points_per_s'] / 1e6:9.1f} M points/s", flush=True)
    return res


def torch_encoding(x, L):
    """positional_encoding (nerf_helpers.py:113-157, log-sampled bands, input included) in torch ops."""
    parts = [x]
    for f in ops.frequency_bands(L, True).tolist():
        parts += [torch.sin(x * f), torch.cos(x * f)]
    return torch.cat(parts, -1)


def eager_run_network(model, pts, ray_batch):
    """The reference's run_network in torch: encode the points and their rows' view directions, run the model."""
    flat = pts.reshape(-1, 3)
    dirs = ray_batch[..., None, -3:].expand(pts.shape).reshape(-1, 3)
    out = []
    for i in range(0, flat.shape[0], EAGER_CHUNK):
        emb = torch.cat((torch_encoding(flat[i:i + EAGER_CHUNK], 10), torch_encoding(dirs[i:i + EAGER_CHUNK], 4)), -1)
        out.append(model(emb))
    return torch.cat(out, 0).reshape(pts.shape[:-1] + (4,))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("run_network_time.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda")
    out = {"card (name, power limit, SM clock, max SM clock)": card(), "rounds": args.rounds, "iters": args.iters}
    print("card:", out["card (name, power limit, SM clock, max SM clock)"])
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    t = torch.linspace(-1.5, 1.5, GRID, device=dev)
    grid = torch.stack(torch.meshgrid(t, t, t, indexing="ij"), -1).reshape(1, -1, 3)
    view = torch.tensor([[0.0, 0.0, 1.0]], device=dev)
    g = torch.Generator().manual_seed(0)
    n, s = 4096, 64
    o = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1) * 4.0
    d = -o / 4.0 + 0.25 * torch.randn(n, 3, generator=g)
    z = torch.sort(torch.rand(n, s, generator=g) * 4 + 2, -1).values
    pts = (o[:, None] + d[:, None] * z[..., None]).to(dev)
    rays = torch.cat([o, d, torch.full((n, 2), 2.0), d / d.norm(dim=-1, keepdim=True)], -1).to(dev)

    for a, kw in ARCHS.items():
        torch.manual_seed(1)
        model = nb.FlexibleNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4, **kw).to(dev)
        with torch.no_grad():
            fused = {f"impl{i}": (lambda i=i: nb.run_network(model, grid, view, EAGER_CHUNK, epf, edf, impl=i))
                     for i in (ops.IMPL_TC, ops.IMPL_TC_FAST)}
            out[f"{a} grid no_grad"] = compare(f"{a} density grid {GRID}^3, no_grad",
                                               {**fused, "eager": lambda: eager_run_network(model, grid, view)},
                                               args.rounds, args.iters, GRID ** 3)

        def train_step(fn):
            model.zero_grad(set_to_none=True)
            fn().sum().backward()

        out[f"{a} 4096x64 fwd+bwd"] = compare(
            f"{a} 4096 x 64 forward + backward",
            {"impl1": lambda: train_step(lambda: nb.run_network(model, pts, rays, 1024, epf, edf, impl=ops.IMPL_TC)),
             "eager": lambda: train_step(lambda: eager_run_network(model, pts, rays))},
            args.rounds, 4 * args.iters, n * s)
    print("card:", card())
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
