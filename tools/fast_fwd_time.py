"""Dev tool: the single-pass fp16 wgmma forward (impl 3) against the split-precision wgmma forward (impl 1), inference only.
In one process, alternating the two implementations, CUDA events after warm-up:
  * the fine-pass MLP forward alone (ops.mlp_fwd, 4096 rays x 192 samples) for A0, A1 and A2;
  * render_fwd with training = 0 on the same 4096 rays (64 + 128 samples);
  * one 800 x 800 render_image (A1, lego-like pose, deterministic sampling).
Each figure is the median over ROUNDS rounds of ITERS calls; the speed-up (impl 1 / impl 3) is given with its range over
the rounds.  The card's name, power limit and SM clocks are printed beside the numbers.

    python tools/fast_fwd_time.py [--rounds 3] [--iters 50] [--json OUT]"""
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
from oracle import nerf_oracle as O  # noqa: E402

ARCHS = {  # bench.py's architectures
    "A0": dict(num_layers=4, hidden=128, skip_every=4),
    "A1": dict(num_layers=8, hidden=128, skip_every=3),
    "A2": dict(num_layers=8, hidden=256, skip_every=4),
}
IMPLS = {"impl1": ops.IMPL_TC, "impl3": ops.IMPL_TC_FAST}


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


def compare(name, fns, rounds, iters, warmup=3):
    """fns: {impl label: callable}; alternates them, returns a result dict and prints one line."""
    for _ in range(warmup):
        for f in fns.values():
            f()
    ms = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            ms[k].append(timed(f, iters))
    speed = [a / b for a, b in zip(ms["impl1"], ms["impl3"])]
    res = {k: {"median_ms": statistics.median(v), "all_ms": v} for k, v in ms.items()}
    res["speedup"] = {"median": statistics.median(speed), "min": min(speed), "max": max(speed)}
    print(f"{name:34s} impl1 {res['impl1']['median_ms']:8.3f} ms   impl3 {res['impl3']['median_ms']:8.3f} ms   "
          f"speed-up {res['speedup']['median']:.2f}x (range {min(speed):.2f} - {max(speed):.2f})", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fast_fwd_time.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda")
    out = {"card (name, power limit, SM clock, max SM clock)": card(), "rounds": args.rounds, "iters": args.iters}
    print("card:", out["card (name, power limit, SM clock, max SM clock)"])
    n_rays, nc, nf = 4096, 64, 128
    g = torch.Generator().manual_seed(0)
    o = torch.nn.functional.normalize(torch.randn(n_rays, 3, generator=g), dim=-1) * 4.0
    d = -o / 4.0 + 0.25 * torch.randn(n_rays, 3, generator=g)
    rays = torch.cat([o, d, torch.full((n_rays, 1), 2.0), torch.full((n_rays, 1), 6.0),
                      d / d.norm(dim=-1, keepdim=True)], -1).to(dev).contiguous()
    z = torch.sort(torch.rand(n_rays, nc + nf, generator=g) * 4 + 2, -1).values.to(dev).contiguous()
    opts = ops.make_opts(nc, nf, False, False, False, 0.0)
    for a, kw in ARCHS.items():
        arch = ops.ArchSpec(n_freq_xyz=10, n_freq_dir=4, **kw)
        sd = O.init_flexible_nerf(arch.num_layers, arch.hidden, arch.skip_every, 10, 4,
                                  generator=torch.Generator().manual_seed(1))
        blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, dev))
        out[f"{a} fine-pass mlp_fwd"] = compare(
            f"{a} fine-pass mlp_fwd (4096 x 192)",
            {k: (lambda i=i: ops.mlp_fwd(arch, blob, rays, z, impl=i)) for k, i in IMPLS.items()}, args.rounds,
            args.iters)
        out[f"{a} render_fwd"] = compare(
            f"{a} render_fwd (4096 x (64 + 128))",
            {k: (lambda i=i: ops.render_fwd(arch, arch, opts, blob, blob, rays, {}, training=False, impl=i))
             for k, i in IMPLS.items()}, args.rounds, args.iters)

    # one 800 x 800 image, A1, deterministic sampling
    torch.manual_seed(0)
    mk = lambda: nb.FlexibleNeRFModel(num_layers=8, hidden_size=128, skip_connect_every=3, num_encoding_fn_xyz=10,
                                      num_encoding_fn_dir=4).to(dev)
    mc, mf = mk(), mk()
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    options = O.make_options(num_coarse=64, num_fine=128, perturb=False, radiance_field_noise_std=0.0)
    pose = O.pose_spherical(30.0, -30.0, 4.0)

    def image(i):
        return nb.render_image(800, 800, 1111.111, pose, mc, mf, options, encode_position_fn=epf,
                               encode_direction_fn=edf, rays_per_chunk=800 * 800, impl=i)

    out["A1 render_image 800x800"] = compare(
        "A1 render_image 800 x 800", {k: (lambda i=i: image(i)) for k, i in IMPLS.items()}, args.rounds,
        max(1, args.iters // 10), warmup=1)
    print("card:", card())
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
