"""Dev tool: regularised fine-tuning of baked fields (nb.baked_regularizer, BakedFieldTrainer's tv_sigma / tv_sh /
sparsity; csrc/baked.cu baked_reg_kernel) on the lego scene.

  kernels  lego A0 (shipped fine weights) baked at 256^3 and 512^3 over OccupancyGrid.from_models of the fine network
           (128^3), unpruned and pruned to the non-transparent bricks: baked_regularizer (gradient only, as the trainer
           runs it), baked_tie for scale, and one whole trainer step at 4096 rays with and without the regulariser;
  sweep    held-out PSNR against render_image (64 + 128 samples, deterministic, impl 1) after 300 and 1000 steps at the
           default rates and 2048 rays per step, 40 training and 4 held-out poses on a sphere of radius 4, 48 x 48, at
           256^3: no regulariser, each weight alone over three values, and the best of each (where it beat no
           regulariser at 300 steps) together; the transparent-brick count and the field's TV after each run.
In one process, alternating the arms of the kernel table after a warm-up, CUDA events; medians over ROUNDS rounds (each
the mean of REPS launches) and their range.  The card's name, power limit and SM clock are read in the same run.

    python tools/baked_reg_time.py [--rounds 5] [--res 256 512] [--no-sweep] [--no-kernels] [--json OUT]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from baked_finetune_time import BOX, HELD, REPS, heldout_psnr, poses_and_targets, trainer  # noqa: E402
from common import card, median, timed_mean  # noqa: E402
from helpers import shipped_models  # noqa: E402

import nerf_pytorch_b200 as nb  # noqa: E402
from nerf_pytorch_b200 import ops  # noqa: E402

TIMED_REG = dict(tv_sigma=1e-5, tv_sh=1e-4, sparsity=1e-5)
SWEEP = {"tv_sigma": (1e-6, 1e-5, 1e-4), "tv_sh": (1e-5, 1e-4, 1e-3), "sparsity": (1e-5, 1e-4, 1e-3, 1e-2, 1e-1, 1.0)}


def kernel_table(field, poses, opts, rounds, label):
    box = field.box()
    count = ops.baked_lattice_count(box, field.brick_map, field.bricks)
    d = torch.zeros_like(field.values)
    tied = torch.empty_like(field.values)
    t = nb.BakedFieldTrainer(field, torch.rand(40, 64, 64, 3, device="cuda"), poses[:40].cuda(), 88.9, opts, seed=9,
                             **TIMED_REG)
    lam = tuple(TIMED_REG[k] for k in ("tv_sigma", "tv_sh", "sparsity"))

    def step(reg):
        t.reg = reg
        t.step(1)

    arms = {
        "baked_regularizer": lambda: ops.baked_regularizer(box, field.brick_map, field.bricks, field.values, count, *lam,
                                                           d=d),
        "baked_tie": lambda: ops.baked_tie(box, field.brick_map, field.bricks, d, tied),
        "trainer step 4096, no regulariser": lambda: step((0.0, 0.0, 0.0)),
        "trainer step 4096, regularised": lambda: step(lam),
    }
    for f in arms.values():
        f()
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, f in arms.items():
            ms[k].append(timed_mean(f, REPS))
    rows = []
    for k in arms:
        r = dict(field=label, n_active=field.n_active, P=int(count), arm=k, **median(ms[k]))
        rows.append(r)
        print(f"{label:24s} {k:36s} {r['ms']:9.3f} ms [{r['range'][0]:.3f}, {r['range'][1]:.3f}]", flush=True)
    del t, d, tied
    torch.cuda.empty_cache()
    return rows


def run(field, start, poses, imgs, opts, reg):
    field.values.copy_(start)
    t = trainer(field, poses, imgs, opts, **reg)
    out = dict(reg=reg)
    t.step(300)
    out["psnr_300"] = heldout_psnr(field, poses, imgs)
    out["transparent_300"] = int(nb.baked_transparent_bricks(field).sum())
    t.step(700)
    out["psnr_1000"] = heldout_psnr(field, poses, imgs)
    out["transparent_1000"] = int(nb.baked_transparent_bricks(field).sum())
    out["tv_1000"] = nb.baked_regularizer(field, tv_sigma=1.0, tv_sh=1.0).item()
    out["sparsity_1000"] = nb.baked_regularizer(field, sparsity=1.0).item()
    print(f"sweep {reg}: held-out PSNR {out['psnr_300']:.3f} / {out['psnr_1000']:.3f} dB after 300 / 1000 steps, "
          f"transparent bricks {out['transparent_300']} / {out['transparent_1000']} of {field.n_active}, "
          f"TV {out['tv_1000']:.4g}, sparsity {out['sparsity_1000']:.4g}", flush=True)
    del t
    return out


def sweep(field, poses, imgs, opts):
    start = field.values.clone()
    rows = [run(field, start, poses, imgs, opts, {})]
    plain = rows[0]["psnr_300"]
    best = {}
    for k, vals in SWEEP.items():
        for v in vals:
            r = run(field, start, poses, imgs, opts, {k: v})
            rows.append(r)
            if r["psnr_300"] > max(plain, best.get(k, (None, -1e9))[1]):
                best[k] = (v, r["psnr_300"])
    if best:
        rows.append(run(field, start, poses, imgs, opts, {k: v for k, (v, _) in best.items()}))
    field.values.copy_(start)
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--no-sweep", action="store_true")
    ap.add_argument("--no-kernels", action="store_true")
    ap.add_argument("--res", type=int, nargs="*", default=[256, 512])
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    mc, mf = shipped_models("lego")[:2]
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    grid = nb.OccupancyGrid.from_models([mf], epf, BOX, 128, encode_direction_fn=edf)
    poses, imgs, opts = poses_and_targets(mc, mf)
    out = dict(card=card(), held=HELD, kernels=[], sweep=[])
    for res in a.res:
        field = nb.bake(mf, epf, edf, bounds=BOX, resolution=res, grid=grid)
        print(f"{res}^3: {field.n_active} active bricks", flush=True)
        if not a.no_sweep and res == 256:
            out["sweep"] = sweep(field, poses, imgs, opts)
        if a.no_kernels:
            continue
        pruned = nb.prune_baked(field, ~nb.baked_transparent_bricks(field))
        out["kernels"] += kernel_table(field, poses, opts, a.rounds, f"{res}^3 unpruned")
        del field
        torch.cuda.empty_cache()
        out["kernels"] += kernel_table(pruned, poses, opts, a.rounds, f"{res}^3 transparent-pruned")
        del pruned
        torch.cuda.empty_cache()
    out["card_after"] = card()
    print("card after:", out["card_after"])
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
