"""Dev tool: time of one A1 config-2 training step (lego 400x400, 4096 rays, 64 + 128 samples, noise std 0.2, FusedAdam,
wgmma kernels) with the random inputs drawn by torch (the default) versus generated in-kernel from a seed
(``randoms=nb.SeededRandoms(seed, step)``).  The two arms alternate in one process; each round times STEPS steps with
CUDA events, and the median and range over the rounds are printed with the card's name and power limit.

    python tools/rng_step_time.py [--rounds 5] [--steps 50] [--json OUT]"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from common import card  # noqa: E402
import nerf_pytorch_b200 as nb  # noqa: E402
from nerf_pytorch_b200 import ops, parallel, train_utils  # noqa: E402
from oracle import nerf_oracle as O  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda")
    H = W = 400
    focal = 555.5555155968841
    nb.set_default_impl(ops.IMPL_TC)
    torch.manual_seed(0)
    mk = lambda: nb.FlexibleNeRFModel(num_layers=8, hidden_size=128, skip_connect_every=3, num_encoding_fn_xyz=10,
                                      num_encoding_fn_dir=4).to(dev)
    mc, mf = mk(), mk()
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    arch = train_utils._arch_of(mc, (10, True, True), (4, True, True))
    optim = parallel.FusedAdam([(mc, arch), (mf, arch)], lr=5e-3)
    options = O.make_options(num_coarse=64, num_fine=128, perturb=True, radiance_field_noise_std=0.2, chunksize=131072)
    pose = torch.tensor([[1.0, 0, 0, 0], [0, 1.0, 0, 0], [0, 0, 1.0, 4.0]])
    g = torch.Generator().manual_seed(0)
    pix = torch.randperm(H * W, generator=g)[:4096].to(dev)
    tgt = torch.rand(4096, 3, generator=g).to(dev)
    rays6 = ops.gen_rays(pose, H, W, focal, pix, dev, use_viewdirs=False, stride=6)
    ro, rd = rays6[:, :3].contiguous(), rays6[:, 3:].contiguous()
    it = [0]

    def step(seeded):
        r = nb.SeededRandoms(1234, it[0] % (1 << 30)) if seeded else None
        it[0] += 1
        out = nb.run_one_iter_of_nerf(H, W, focal, mc, mf, ro, rd, options, encode_position_fn=epf,
                                      encode_direction_fn=edf, randoms=r)
        loss = torch.nn.functional.mse_loss(out[0], tgt) + torch.nn.functional.mse_loss(out[3], tgt)
        optim.zero_grad()
        loss.backward()
        optim.step()

    def timed(seeded):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            step(seeded)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    for seeded in (False, True, False, True):  # warm-up of both arms
        for _ in range(5):
            step(seeded)
    ms = {"torch": [], "seeded": []}
    for _ in range(args.rounds):
        ms["torch"].append(timed(False))
        ms["seeded"].append(timed(True))
    res = {"card": card(), "workload": "A1, config 2 (4096 rays, 64 + 128 samples), wgmma kernels, FusedAdam",
           "steps_per_round": args.steps, "rounds": args.rounds}
    for k, v in ms.items():
        res[k] = {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v), "all_ms": v}
        print(f"{k:7s} step: median {statistics.median(v):.3f} ms (range {min(v):.3f} - {max(v):.3f}) over {args.rounds}"
              f" rounds of {args.steps} steps")
    d = res["seeded"]["median_ms"] - res["torch"]["median_ms"]
    res["seeded_minus_torch_ms"] = d
    print(f"card: {res['card']}")
    print(f"seeded - torch: {d:+.3f} ms per step")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
