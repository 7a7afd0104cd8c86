"""Dev tool: time of one training step driven three ways, at lego config-2 size (400 x 400 images, 64 + 128 samples,
noise std 0.2), impl 1, for A0 and A1 at 1024 rays (the pretrained configs' num_random_rays) and 4096 rays:

  eager     the reference loop's step: pose on the device, pixel draw (np.random.choice on the host, as
            train_nerf.py:213-226), run_one_iter_of_nerf_from_pose, mse_loss, backward, FusedAdam.step, loss.item()
  graph     CapturedTrainStep.step() (one CUDA graph launch) and loss.item() every step
  graph100  CapturedTrainStep.step(), the loss read every 100 steps

The arms alternate in one process, each on its own copy of the models; a round times STEPS steps with a host clock
around work that ends in a device synchronise.  Prints the median and range per arm and the card's name, power limit
and SM clock, read in the same run.

    python tools/graph_step_time.py [--rounds 5] [--steps 100] [--json OUT]"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from common import card  # noqa: E402
import nerf_pytorch_b200 as nb  # noqa: E402
from nerf_pytorch_b200 import parallel, train_utils  # noqa: E402
from oracle import nerf_oracle as O  # noqa: E402

ARCHS = {"A0": dict(num_layers=4, hidden_size=128, skip_connect_every=4),
         "A1": dict(num_layers=8, hidden_size=128, skip_connect_every=3)}
H = W = 400
FOCAL = 555.5555155968841
N_IMAGES = 20


def poses(n):
    import math

    out = []
    for i in range(n):
        th, ph = math.radians(360.0 * i / n), math.radians(-30.0)
        t = torch.tensor([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 4.0], [0, 0, 0, 1.0]])
        rp = torch.tensor([[1, 0, 0, 0], [0, math.cos(ph), -math.sin(ph), 0], [0, math.sin(ph), math.cos(ph), 0],
                           [0, 0, 0, 1.0]])
        rt = torch.tensor([[math.cos(th), 0, -math.sin(th), 0], [0, 1, 0, 0], [math.sin(th), 0, math.cos(th), 0],
                           [0, 0, 0, 1.0]])
        swap = torch.tensor([[-1, 0, 0, 0], [0, 0, 1, 0], [0, 1, 0, 0], [0, 0, 0, 1.0]])
        out.append(swap @ rt @ rp @ t)
    return torch.stack(out).float()


def workload(arch, n_rays, images, pose_table):
    options = O.make_options(num_coarse=64, num_fine=128, perturb=True, radiance_field_noise_std=0.2, chunksize=131072)
    options.nerf.train.num_random_rays = n_rays
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)

    def models():
        torch.manual_seed(0)
        mk = lambda: nb.FlexibleNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4, **ARCHS[arch]).cuda()
        mc, mf = mk(), mk()
        a = train_utils._arch_of(mc, (10, True, True), (4, True, True))
        return mc, mf, parallel.FusedAdam([(mc, a), (mf, a)], lr=5e-3, lr_decay=250, lr_decay_factor=0.1)

    mc, mf, opt = models()
    rng = np.random.default_rng(0)

    def eager(i):
        img = int(rng.integers(N_IMAGES))
        pose = pose_table[img]
        sel = torch.from_numpy(rng.choice(H * W, size=n_rays, replace=False)).cuda()
        out = nb.run_one_iter_of_nerf_from_pose(H, W, FOCAL, mc, mf, pose, sel, options, encode_position_fn=epf,
                                                encode_direction_fn=edf, impl=1)
        tgt = images[img].reshape(-1, 3)[sel]
        loss = torch.nn.functional.mse_loss(out[0], tgt) + torch.nn.functional.mse_loss(out[3], tgt)
        opt.zero_grad()
        loss.backward()
        opt.step()
        loss.item()

    gc, gf, gopt = models()
    cap = nb.CapturedTrainStep(gc, gf, epf, edf, options, gopt, 1234, (images, pose_table, FOCAL), impl=1)

    def graph(i):
        cap.step().item()

    def graph100(i):
        loss = cap.step()
        if i % 100 == 99:
            loss.item()

    return {"eager": eager, "graph": graph, "graph100": graph100}


def timed(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        fn(i)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("graph_step_time.py needs a CUDA device")
    g = torch.Generator().manual_seed(0)
    images = torch.rand(N_IMAGES, H, W, 3, generator=g).cuda()
    pose_table = poses(N_IMAGES).cuda()
    res = {"card_before": card(), "rounds": args.rounds, "steps_per_round": args.steps,
           "workload": "400 x 400 images, 64 + 128 samples, noise 0.2, impl 1, FusedAdam", "results": {}}
    for arch in ("A0", "A1"):
        for n in (1024, 4096):
            arms = workload(arch, n, images, pose_table)
            for fn in arms.values():  # warm-up
                timed(fn, 10)
            ms = {k: [] for k in arms}
            for _ in range(args.rounds):
                for k, fn in arms.items():
                    ms[k].append(timed(fn, args.steps))
            key = f"{arch} {n} rays"
            res["results"][key] = {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v),
                                       "all_ms": v} for k, v in ms.items()}
            line = ", ".join(f"{k} {statistics.median(v):.3f} ms ({min(v):.3f}-{max(v):.3f})" for k, v in ms.items())
            print(f"{key}: {line}", flush=True)
            del arms
            torch.cuda.empty_cache()
    res["card_after"] = card()
    print(f"card (name, power limit, SM clock, max SM clock): before {res['card_before']} / after {res['card_after']}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
