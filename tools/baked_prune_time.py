"""Dev tool: pruning baked fields (nb.baked_transparent_bricks, nb.baked_brick_weights, nb.prune_baked; csrc/baked.cu
baked_max_weight_kernel) on the lego scene.

lego A0 (shipped weights) baked at 256^3 and 512^3 over OccupancyGrid.from_models (128^3) of both networks and of the
fine network alone.  Poses, views and the PSNR reference are tools/baked_finetune_time.py's: 40 training and 4 held-out
poses on a sphere of radius 4, 48 x 48, against render_image (64 + 128 samples, deterministic, impl 1).  Per criterion --
none, transparent bricks, and peak weight over the 40 training views > tau for tau = 0, 1e-3, 1e-2 -- it reports:

  bricks    active bricks and values GiB;
  weights   baked_brick_weights per 48 x 48 view (the 40 training views, once per round) and at 800 x 800;
  render    render_baked at 800 x 800, with and without early_stop = 1e-3;
  psnr      held-out PSNR against render_image before fine-tuning;
  trainer   BakedFieldTrainer step time (2048 rays) and the device memory the field and the trainer's buffers take;
  tuned     held-out PSNR after 300 trainer steps on the pruned field (criterion "none" is train-unpruned).

In one process; the weights and render arms alternate across criteria in every round after a warm-up, CUDA events,
medians over ROUNDS rounds (each the mean of REPS launches) and their range.  The trainers run one criterion after
another (at 512^3 the five do not fit on one card together).  The card's name, power limit and SM clock are read in
the same run.

    python tools/baked_prune_time.py [--rounds 3] [--res 256 512] [--json OUT]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import nerf_pytorch_b200 as nb  # noqa: E402
from oracle import nerf_oracle as O  # noqa: E402
from baked_finetune_time import BOX, FOCAL, H, HELD, heldout_psnr, poses_and_targets, trainer  # noqa: E402
from common import card, median, timed_mean  # noqa: E402
from helpers import shipped_models  # noqa: E402

BIG, BIG_FOCAL = 800, 1111.1
TAUS = (0.0, 1e-3, 1e-2)
STEPS = 300


def gib(field):
    return field.values.numel() * 4 / 2 ** 30


def criteria(field, poses, opts):
    train = torch.stack([poses[i] for i in range(44) if i not in HELD])
    w = nb.baked_brick_weights(field, train, H, H, FOCAL, opts)
    keeps = {"none": None, "transparent": ~nb.baked_transparent_bricks(field)}
    for tau in TAUS:
        keeps[f"w>{tau:g}"] = w > tau
    return train, keeps


def one_grid(mf, grid, grid_name, res, poses, imgs, opts, rounds):
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    base = nb.bake(mf, epf, edf, bounds=BOX, resolution=res, grid=grid)
    train, keeps = criteria(base, poses, opts)
    fields = {k: base if keep is None else nb.prune_baked(base, keep) for k, keep in keeps.items()}
    big_pose = O.pose_spherical(30.0, -30.0, 4.0)
    arms = {}
    for k, f in fields.items():
        arms[(k, "weights per 48x48 view")] = (lambda f=f: nb.baked_brick_weights(f, train, H, H, FOCAL, opts),
                                               len(train))
        arms[(k, "weights 800x800")] = (lambda f=f: nb.baked_brick_weights(f, big_pose[None], BIG, BIG, BIG_FOCAL,
                                                                           opts), 1)
        arms[(k, "render 800x800")] = (lambda f=f: nb.render_baked(f, BIG, BIG, BIG_FOCAL, big_pose, opts), 1)
        arms[(k, "render 800x800 early_stop 1e-3")] = (
            lambda f=f: nb.render_baked(f, BIG, BIG, BIG_FOCAL, big_pose, opts, early_stop=1e-3), 1)
    for fn, _ in arms.values():
        fn()
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, (fn, per) in arms.items():
            ms[k].append(timed_mean(fn, 3 if "48x48" in k[1] else 10) / per)
    rows = []
    for k, f in fields.items():
        r = dict(res=res, grid=grid_name, criterion=k, n_active=f.n_active, values_gib=gib(f),
                 psnr=heldout_psnr(f, poses, imgs))
        for (kk, arm), v in ms.items():
            if kk == k:
                r[arm] = median(v)
        rows.append(r)
    del arms
    # the trainers, one criterion after another: step time, memory, held-out PSNR after STEPS steps
    for r in rows:
        k = r["criterion"]
        f = fields[k]
        tuned = nb.BakedField(f.bounds, f.resolution, f.brick_map, f.bricks, f.values.clone(), f.use_viewdirs)
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        t = trainer(tuned, poses, imgs, opts, seed=1)
        t.step(5)
        step_ms = [timed_mean(lambda: t.step(1), 20) for _ in range(rounds)]
        t.step(max(0, STEPS - 5 - 20 * rounds))
        torch.cuda.synchronize()
        r["trainer step 2048"] = median(step_ms)
        r["finetune_gib"] = gib(f) + (torch.cuda.max_memory_allocated() - before) / 2 ** 30
        r["psnr_tuned"] = heldout_psnr(tuned, poses, imgs)
        del t, tuned
        torch.cuda.empty_cache()
        print(f"{res}^3 {grid_name:5s} {k:12s} bricks {r['n_active']:6d} values {r['values_gib']:6.2f} GiB | "
              f"weights/view {r['weights per 48x48 view']['ms']:7.3f} ms, 800^2 {r['weights 800x800']['ms']:7.2f} ms | "
              f"render {r['render 800x800']['ms']:7.2f} ms, early stop {r['render 800x800 early_stop 1e-3']['ms']:7.2f}"
              f" ms | PSNR {r['psnr']:.2f} dB | step {r['trainer step 2048']['ms']:7.3f} ms, fine-tune "
              f"{r['finetune_gib']:6.2f} GiB | PSNR after {STEPS} steps {r['psnr_tuned']:.2f} dB", flush=True)
    del fields, base
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--res", type=int, nargs="*", default=[256, 512])
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    mc, mf = shipped_models("lego")[:2]
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    grids = {"both": nb.OccupancyGrid.from_models([mc, mf], epf, BOX, 128, encode_direction_fn=edf),
             "fine": nb.OccupancyGrid.from_models([mf], epf, BOX, 128, encode_direction_fn=edf)}
    poses, imgs, opts = poses_and_targets(mc, mf)
    out = dict(card=card(), rows=[])
    for res in a.res:
        for name, grid in grids.items():
            out["rows"] += one_grid(mf, grid, name, res, poses, imgs, opts, a.rounds)
    out["card_after"] = card()
    print("card after:", out["card_after"])
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
