"""Dev tool: subdividing baked fields (nb.subdivide_baked, BakedFieldTrainer.subdivide; csrc/baked.cu
baked_subdivide_kernel) and fitting a field to images without a network, coarse to fine, on the lego scene.

Poses, views and the PSNR reference are tools/baked_finetune_time.py's: 4 held-out poses on a sphere of radius 4, 48 x
48, against render_image of the shipped lego A0 networks (64 + 128 samples, deterministic, impl 1).  Sections:

  subdivide  lego A0 baked at 128^3 and 256^3 over OccupancyGrid.from_models (128^3) of both networks, unpruned and
             transparent-pruned: the kernel alone (ops.baked_subdivide into a preallocated child, CUDA events, the mean
             of REPS launches; its write rate from shapes against 3.35 TB/s), subdivide_baked whole and its peak device
             memory, BakedFieldTrainer.subdivide whole and its peak; held-out PSNR of parent and child against
             render_image and of the child's render against the parent's.  The kernel arms alternate across fields in
             every round after a warm-up; medians over ROUNDS rounds and their range.
  pipeline   BakedField.full(box, 64) -> train -> prune at peak weight > tau over the training views -> subdivide ->
             ... -> 256^3 (and one run on to 512^3): per stage active bricks, values GiB, trainer step time, steps, wall
             time, peak device memory and held-out PSNR.  On the 40 training views at 48 x 48 (2048 rays per step) and
             on 100 views at 96 x 96 (4096 rays per step).
  sweep      the sigma / SH rates, then tau, the start sigma_raw and TV weights one at a time around the best rates,
             over 64^3 -> 128^3 on the 40 views.
  compare    bake at 256^3 (grid of both networks) + 300 trainer steps on the same views, against the pipeline.

The card's name, power limit and SM clock are read in the same run, before and after.

    python tools/baked_subdivide_time.py [--rounds 5] [--sections subdivide pipeline sweep compare] [--json OUT]"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import nerf_pytorch_b200 as nb  # noqa: E402
from nerf_pytorch_b200 import ops  # noqa: E402
from nerf_pytorch_b200.bake import _child_bricks  # noqa: E402
from oracle import nerf_oracle as O  # noqa: E402
from baked_finetune_time import BOX, FOCAL, H, HELD, heldout_psnr, poses_and_targets  # noqa: E402
from common import card, median, psnr, timed_mean, timed_once  # noqa: E402
from helpers import shipped_models  # noqa: E402

REPS = 10
HBM = 3.35e12  # B/s, the H100 SXM data sheet
# the pipeline's rates (the sweep's best pair on the 40 views), start, tau and schedule, as DESIGN §4 reports them
LR_SIGMA, LR_SH = 1.0, 3e-2
SIGMA0 = 0.1
TAU = 1e-3
STAGE_STEPS = 1000


def gib(field):
    return field.values.numel() * 4 / 2 ** 30


def mib_peak(before):
    return (torch.cuda.max_memory_allocated() - before) / 2 ** 20


def render_psnr(a, b, poses):
    """Mean PSNR of field a's held-out renders against field b's."""
    vals = []
    with torch.no_grad():
        for i in HELD:
            rays = ops.gen_rays(poses[i], H, H, FOCAL, None, "cuda", ndc=False, near=2.0, far=6.0, use_viewdirs=True)
            vals.append(psnr(nb.render_baked_rays(a, rays)[0], nb.render_baked_rays(b, rays)[0]))
    return sum(vals) / len(vals)


# ------------------------------------------------------------------------------------------------------------------------
def subdivide_section(mc, mf, poses, imgs, opts, rounds):
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    grid = nb.OccupancyGrid.from_models([mc, mf], epf, BOX, 128, encode_direction_fn=edf)
    train = [i for i in range(44) if i not in HELD]
    rows = []
    for res in (128, 256):
        base = nb.bake(mf, epf, edf, bounds=BOX, resolution=res, grid=grid)
        fields = {"unpruned": base, "transparent": nb.prune_baked(base, ~nb.baked_transparent_bricks(base))}
        # the kernel alone, alternating across the two fields
        prepared = {}
        for k, f in fields.items():
            bm, br = _child_bricks(f, tuple(2 * r for r in f.resolution))
            out = torch.empty(br.numel(), 729, 32, device="cuda")
            box = f.box()
            prepared[k] = (lambda box=box, f=f, br=br, out=out: ops.baked_subdivide(box, f.brick_map, f.values, br, out),
                           br.numel())
            del bm
        for fn, _ in prepared.values():
            fn()
        ms = {k: [] for k in prepared}
        for _ in range(rounds):
            for k, (fn, _) in prepared.items():
                ms[k].append(timed_mean(fn, REPS))
        for k, f in fields.items():
            n_child = prepared[k][1]
            written = n_child * 729 * 32 * 4
            kern = median(ms[k])
            r = dict(res=res, field=k, n_active=f.n_active, parent_gib=gib(f), n_child=n_child,
                     child_gib=written / 2 ** 30, kernel=kern, write_tbs=written / (kern["ms"] * 1e-3) / 1e12,
                     write_share=written / (kern["ms"] * 1e-3) / HBM)
            prepared[k] = None
            torch.cuda.empty_cache()
            torch.cuda.synchronize()
            before = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            whole, child = timed_once(lambda f=f: nb.subdivide_baked(f))
            r["subdivide_baked_ms"], r["subdivide_baked_peak_mib"] = whole, mib_peak(before)
            r["psnr_parent"] = heldout_psnr(f, poses, imgs)
            r["psnr_child"] = heldout_psnr(child, poses, imgs)
            r["psnr_child_vs_parent"] = render_psnr(child, f, poses)
            del child
            torch.cuda.empty_cache()
            # the trainer's subdivide: field, m and v through the kernel, the buffers reallocated, P recounted
            tuned = nb.BakedField(f.bounds, f.resolution, f.brick_map, f.bricks, f.values.clone(), f.use_viewdirs)
            t = nb.BakedFieldTrainer(tuned, imgs[train].contiguous(), poses[train].cuda(), FOCAL, opts,
                                     rays_per_step=2048, seed=1)
            t.step(5)
            torch.cuda.synchronize()
            before = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            r["trainer_subdivide_ms"] = timed_once(t.subdivide)[0]
            r["trainer_subdivide_peak_mib"] = mib_peak(before)
            r["trainer_gib_after"] = torch.cuda.memory_allocated() / 2 ** 30
            del t, tuned
            torch.cuda.empty_cache()
            rows.append(r)
            print(f"{res}^3 -> {2 * res}^3 {k:11s} bricks {f.n_active:6d} -> {n_child:6d} ({r['child_gib']:.2f} GiB) | "
                  f"kernel {kern['ms']:.3f} ms [{kern['range'][0]:.3f}, {kern['range'][1]:.3f}] "
                  f"{r['write_tbs']:.2f} TB/s written ({100 * r['write_share']:.0f} % of 3.35) | subdivide_baked "
                  f"{whole:.1f} ms peak {r['subdivide_baked_peak_mib']:.0f} MiB | trainer.subdivide "
                  f"{r['trainer_subdivide_ms']:.1f} ms peak {r['trainer_subdivide_peak_mib']:.0f} MiB | PSNR parent "
                  f"{r['psnr_parent']:.3f} child {r['psnr_child']:.3f} child-vs-parent {r['psnr_child_vs_parent']:.2f} dB",
                  flush=True)
        del fields, base, prepared
        torch.cuda.empty_cache()
    return rows


# ------------------------------------------------------------------------------------------------------------------------
def views(mc, mf, n, size, opts):
    """n training poses around the scene (4 elevations) and render_image's fine rgb at size x size, focal scaled."""
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    phis = (-15.0, -30.0, -45.0, -60.0)
    poses = torch.stack([O.pose_spherical(360.0 * i / n + 3.0 * (i % 4), phis[i % 4], 4.0) for i in range(n)])
    focal = FOCAL * size / H
    with torch.no_grad():
        imgs = torch.stack([nb.render_image(size, size, focal, p, mc, mf, opts, encode_position_fn=epf,
                                            encode_direction_fn=edf, impl=1)[3] for p in poses]).contiguous()
    return poses, imgs, focal


def pipeline(train_set, poses, imgs, opts, *, final=256, lr_sigma=LR_SIGMA, lr_sh=LR_SH, sigma0=SIGMA0, tau=TAU,
             steps=STAGE_STEPS, tv_sigma=0.0, tv_sh=0.0, rays=2048, quiet=False):
    """BakedField.full(BOX, 64) trained coarse to fine to ``final``; per-stage rows."""
    tposes, timgs, focal = train_set
    size = timgs.shape[1]
    field = nb.BakedField.full(BOX, 64, sigma_raw=sigma0)
    torch.cuda.synchronize()
    base_mem = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t = nb.BakedFieldTrainer(field, timgs, tposes.cuda(), focal, opts, lr_sigma=lr_sigma, lr_sh=lr_sh,
                             rays_per_step=rays, seed=1, tv_sigma=tv_sigma, tv_sh=tv_sh)
    rows = []
    res = 64
    while True:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        t.step(steps)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        step_ms = timed_mean(lambda: t.step(1), 20) if not quiet else wall * 1e3 / steps
        r = dict(res=res, n_active=field.n_active, values_gib=gib(field), steps=steps, wall_s=wall, step_ms=step_ms,
                 peak_gib=(torch.cuda.max_memory_allocated() - base_mem) / 2 ** 30,
                 psnr=heldout_psnr(field, poses, imgs), loss=float(t.loss))
        rows.append(r)
        if not quiet:
            print(f"  {res}^3 bricks {r['n_active']:6d} values {r['values_gib']:.3f} GiB | step {step_ms:.3f} ms x "
                  f"{steps} = {wall:.1f} s | peak {r['peak_gib']:.2f} GiB | held-out PSNR {r['psnr']:.3f} dB", flush=True)
        if res >= final:
            break
        w = nb.baked_brick_weights(field, tposes, size, size, focal, opts)
        keep = w > tau
        t.prune(keep)
        t.subdivide()
        res *= 2
    del t
    torch.cuda.empty_cache()
    return rows, field


def pipeline_section(mc, mf, poses, imgs, opts):
    out = {}
    sets = {"40 x 48^2": views(mc, mf, 40, 48, opts), "100 x 96^2": views(mc, mf, 100, 96, opts)}
    for name, s in sets.items():
        for final in (256, 512):
            rays = 2048 if s[1].shape[1] == 48 else 4096
            print(f"pipeline {name} to {final}^3 (lr_sigma {LR_SIGMA}, lr_sh {LR_SH}, sigma0 {SIGMA0}, tau {TAU}, "
                  f"{STAGE_STEPS} steps per stage, {rays} rays per step)", flush=True)
            out[f"{name} -> {final}"] = pipeline(s, poses, imgs, opts, final=final, rays=rays)[0]
    return out, sets


def sweep_section(train_set, poses, imgs, opts):
    res = {}

    def run(name, **kw):
        rows = pipeline(train_set, poses, imgs, opts, final=128, steps=500, quiet=True, **kw)[0]
        res[name] = [round(r["psnr"], 3) for r in rows] + [rows[-1]["n_active"]]
        print(f"  sweep {name}: held-out PSNR per stage {res[name][:-1]}, bricks {res[name][-1]}", flush=True)
        return rows[-1]["psnr"]

    best, best_rates = -1.0, (LR_SIGMA, LR_SH)
    for ls in (0.3, 1.0, 3.0):
        for lh in (1e-2, 3e-2, 1e-1):
            p = run(f"lr_sigma {ls} lr_sh {lh}", lr_sigma=ls, lr_sh=lh)
            if p > best:
                best, best_rates = p, (ls, lh)
    ls, lh = best_rates
    for tau in (0.0, 1e-2):
        run(f"best rates, tau {tau}", lr_sigma=ls, lr_sh=lh, tau=tau)
    for s0 in (0.01, 1.0):
        run(f"best rates, sigma0 {s0}", lr_sigma=ls, lr_sh=lh, sigma0=s0)
    for tvs, tvh in ((1e-5, 0.0), (0.0, 1e-4), (1e-4, 1e-3)):
        run(f"best rates, tv_sigma {tvs} tv_sh {tvh}", lr_sigma=ls, lr_sh=lh, tv_sigma=tvs, tv_sh=tvh)
    return dict(runs=res, best_rates=best_rates)


def compare_section(mc, mf, train_set, poses, imgs, opts, rays):
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    grid = nb.OccupancyGrid.from_models([mc, mf], epf, BOX, 128, encode_direction_fn=edf)
    f = nb.bake(mf, epf, edf, bounds=BOX, resolution=256, grid=grid)
    tposes, timgs, focal = train_set
    p0 = heldout_psnr(f, poses, imgs)
    t = nb.BakedFieldTrainer(f, timgs, tposes.cuda(), focal, opts, rays_per_step=rays, seed=1)
    t.step(300)
    r = dict(n_active=f.n_active, psnr_bake=p0, psnr_300=heldout_psnr(f, poses, imgs))
    del t, f
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--sections", nargs="*", default=["subdivide", "pipeline", "sweep", "compare"])
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    out = dict(card=card())
    print("card:", out["card"], flush=True)
    mc, mf = shipped_models("lego")[:2]
    poses, imgs, opts = poses_and_targets(mc, mf)
    if "subdivide" in a.sections:
        out["subdivide"] = subdivide_section(mc, mf, poses, imgs, opts, a.rounds)
    sets = None
    if "pipeline" in a.sections:
        out["pipeline"], sets = pipeline_section(mc, mf, poses, imgs, opts)
    if sets is None and ("sweep" in a.sections or "compare" in a.sections):
        sets = {"40 x 48^2": views(mc, mf, 40, 48, opts), "100 x 96^2": views(mc, mf, 100, 96, opts)}
    if "sweep" in a.sections:
        print("sweep over 64^3 -> 128^3, 500 steps per stage, 40 x 48^2 views", flush=True)
        out["sweep"] = sweep_section(sets["40 x 48^2"], poses, imgs, opts)
    if "compare" in a.sections:
        out["compare"] = {name: compare_section(mc, mf, s, poses, imgs, opts, 2048 if s[1].shape[1] == 48 else 4096)
                          for name, s in sets.items()}
        print("bake 256^3 + 300 steps:", out["compare"], flush=True)
    out["card_after"] = card()
    print("card after:", out["card_after"])
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
