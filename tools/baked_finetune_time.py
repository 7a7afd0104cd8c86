"""Dev tool: fine-tuning baked fields (nb.BakedFieldTrainer; csrc/baked.cu baked_render_bwd_kernel / baked_tie_kernel,
csrc/sampling.cu baked_adam_dev_kernel) on the lego scene.

  kernels  lego A0 (shipped fine weights) baked at 256^3 and 512^3 over OccupancyGrid.from_models of the fine network
           (128^3): baked_render and baked_render_bwd at 4096 and 65536 camera rays, baked_tie and baked_adam_step_dev
           over the whole field, and one whole trainer step at 4096 rays;
  psnr     held-out PSNR against render_image (64 + 128 samples, deterministic, impl 1) after 0 / 100 / 300 / 1000
           trainer steps at the default rates and 2048 rays per step: 40 training and 4 held-out poses on a sphere of
           radius 4, 48 x 48;
  sweep    (--sweep) held-out PSNR after 300 steps at 256^3 over a grid of lr_sigma x lr_sh.
In one process, alternating the arms of the kernel table after a warm-up, CUDA events; medians over ROUNDS rounds (each
the mean of REPS launches) and their range.  The card's name, power limit and SM clock are read in the same run.

    python tools/baked_finetune_time.py [--rounds 3] [--sweep] [--json OUT]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from common import card, median, psnr, timed_mean  # noqa: E402
from helpers import shipped_models  # noqa: E402
import nerf_pytorch_b200 as nb  # noqa: E402
from nerf_pytorch_b200 import ops  # noqa: E402
from oracle import nerf_oracle as O  # noqa: E402

BOX = ((-1.5,) * 3, (1.5,) * 3)
H, FOCAL = 48, 66.7
REPS = 10
HELD = (5, 16, 27, 38)


def poses_and_targets(mc, mf):
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    phis = (-30.0, -45.0, -15.0)
    poses = torch.stack([O.pose_spherical(360.0 * i / 44 + 7.0 * (i % 3), phis[i % 3], 4.0) for i in range(44)])
    opts = O.make_options(near=2.0, far=6.0, num_coarse=64, num_fine=128, perturb=False, radiance_field_noise_std=0.0)
    with torch.no_grad():
        imgs = torch.stack([nb.render_image(H, H, FOCAL, p, mc, mf, opts, encode_position_fn=epf,
                                            encode_direction_fn=edf, impl=1)[3] for p in poses]).contiguous()
    return poses, imgs, opts


def heldout_psnr(field, poses, imgs):
    vals = []
    with torch.no_grad():
        for i in HELD:
            rays = ops.gen_rays(poses[i], H, H, FOCAL, None, "cuda", ndc=False, near=2.0, far=6.0, use_viewdirs=True)
            vals.append(psnr(nb.render_baked_rays(field, rays)[0], imgs[i].reshape(-1, 3)))
    return sum(vals) / len(vals)


def trainer(field, poses, imgs, opts, **kw):
    train = [i for i in range(44) if i not in HELD]
    return nb.BakedFieldTrainer(field, imgs[train].contiguous(), poses[train].cuda(), FOCAL, opts, rays_per_step=2048,
                                **kw)


def kernel_table(field, poses, imgs, opts, rounds, res):
    box = field.box()
    big = ops.gen_rays(O.pose_spherical(30.0, -30.0, 4.0), 400, 400, 555.6, None, "cuda", ndc=False, near=2.0,
                       far=6.0, use_viewdirs=True)
    rays = {n: big[torch.randperm(big.shape[0], generator=torch.Generator().manual_seed(n))[:n].cuda()].contiguous()
            for n in (4096, 65536)}
    outs = {n: ops.baked_render(box, field.brick_map, field.values, True, r, False) for n, r in rays.items()}
    gouts = {n: torch.randn(n, 8, device="cuda") for n in rays}
    d = torch.zeros_like(field.values)
    tied = torch.empty_like(field.values)
    m, v = torch.zeros_like(field.values), torch.zeros_like(field.values)
    step = torch.zeros(1, dtype=torch.int64, device="cuda")
    # the step at 4096 rays: 64 x 64 images (random targets; the timing does not depend on them)
    t = nb.BakedFieldTrainer(field, torch.rand(40, 64, 64, 3, device="cuda"), poses[:40].cuda(), 88.9, opts, seed=9)
    arms = {}
    for n, r in rays.items():
        arms[f"baked_render {n}"] = lambda r=r, n=n: ops.baked_render(box, field.brick_map, field.values, True, r, False,
                                                                       out=outs[n])
        arms[f"baked_render_bwd {n}"] = lambda r=r, n=n: ops.baked_render_bwd(box, field.brick_map, field.values, True,
                                                                               r, False, outs[n], gouts[n], d)
    arms["baked_tie"] = lambda: ops.baked_tie(box, field.brick_map, field.bricks, d, tied)
    # zero rates: the Adam arm reads and writes the field as a step does without moving it
    arms["baked_adam_step_dev"] = lambda: ops.baked_adam_step_dev(field.values, tied, m, v, step, 0.0, 0.0)
    arms["trainer step 4096"] = lambda: t.step(1)
    for f in arms.values():
        f()
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, f in arms.items():
            ms[k].append(timed_mean(f, REPS))
    rows = []
    for k in arms:
        r = dict(res=res, arm=k, **median(ms[k]))
        rows.append(r)
        print(f"{res}^3 {k:24s} {r['ms']:9.3f} ms [{r['range'][0]:.3f}, {r['range'][1]:.3f}]", flush=True)
    del t, d, tied, m, v
    torch.cuda.empty_cache()
    return rows


def psnr_table(field, poses, imgs, opts, res):
    t = trainer(field, poses, imgs, opts)
    rows, done = [], 0
    for target in (0, 100, 300, 1000):
        if target > done:
            t.step(target - done)
        done = target
        p = heldout_psnr(field, poses, imgs)
        rows.append(dict(res=res, steps=target, psnr=p, loss=float(t.loss)))
        print(f"{res}^3 after {target:5d} steps: held-out PSNR {p:.2f} dB, last loss {float(t.loss):.3e}", flush=True)
    del t
    torch.cuda.empty_cache()
    return rows


def sweep(field, poses, imgs, opts):
    start = field.values.clone()
    rows = []
    for lr_sigma in (0.1, 1.0, 10.0):
        for lr_sh in (1e-3, 3e-3, 1e-2, 3e-2):
            field.values.copy_(start)
            t = trainer(field, poses, imgs, opts, lr_sigma=lr_sigma, lr_sh=lr_sh)
            t.step(300)
            p = heldout_psnr(field, poses, imgs)
            rows.append(dict(lr_sigma=lr_sigma, lr_sh=lr_sh, psnr=p))
            print(f"sweep lr_sigma {lr_sigma:g} lr_sh {lr_sh:g}: held-out PSNR after 300 steps {p:.2f} dB", flush=True)
            del t
    field.values.copy_(start)
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--res", type=int, nargs="*", default=[256, 512])
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    mc, mf = shipped_models("lego")[:2]
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    grid = nb.OccupancyGrid.from_models([mf], epf, BOX, 128, encode_direction_fn=edf)
    poses, imgs, opts = poses_and_targets(mc, mf)
    out = dict(card=card(), kernels=[], psnr=[], sweep=[])
    for res in a.res:
        field = nb.bake(mf, epf, edf, bounds=BOX, resolution=res, grid=grid)
        print(f"{res}^3: {field.n_active} active bricks, values {field.values.numel() * 4 / 2 ** 30:.2f} GiB", flush=True)
        if a.sweep and res == 256:
            out["sweep"] = sweep(field, poses, imgs, opts)
        out["kernels"] += kernel_table(field, poses, imgs, opts, a.rounds, res)
        field = nb.bake(mf, epf, edf, bounds=BOX, resolution=res, grid=grid)  # the timing's trainer moved the values
        torch.cuda.reset_peak_memory_stats()
        out["psnr"] += psnr_table(field, poses, imgs, opts, res)
        out[f"peak_gib_{res}"] = torch.cuda.max_memory_allocated() / 2 ** 30
        print(f"{res}^3 peak device memory allocated while fine-tuning: {out[f'peak_gib_{res}']:.2f} GiB", flush=True)
        del field
        torch.cuda.empty_cache()
    out["card_after"] = card()
    print("card after:", out["card_after"])
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
