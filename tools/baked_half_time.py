"""Dev tool: half-precision baked fields (nb.bake(dtype=torch.float16), BakedField.half; csrc/baked.cu
baked_render_kernel<__half>, csrc/mlp_tc.cu bake_tc_kernel<kH, __half>) against fp32 ones on the lego scene.

lego A0 (shipped weights) baked at 256^3 and 512^3 over OccupancyGrid.from_models (128^3) of both networks, unpruned and
transparent-pruned (the fp32 field's mask, which is the fp16 field's).  It reports:

  bake      nb.bake time and the peak device memory it adds, fp32 against dtype=torch.float16;
  bricks    active bricks and values GiB of each field;
  render    render_baked at 400 x 400 and 800 x 800, with and without early_stop = 1e-3, fp32 against fp16;
  psnr      mean over the 4 held-out views of tools/baked_finetune_time.py (48 x 48) of the fp16 render against the fp32
            render, and of each against render_image (64 + 128 samples, deterministic, impl 1).

In one process; the fp32 and fp16 arms alternate in every round after a warm-up, CUDA events, medians over ROUNDS rounds
(renders: each the mean of REPS launches) and their range.  The card's name, power limit and SM clock are read in the
same run.

    python tools/baked_half_time.py [--rounds 5] [--res 256 512] [--json OUT]"""
import argparse
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import nerf_pytorch_b200 as nb  # noqa: E402
from nerf_pytorch_b200 import ops  # noqa: E402
from oracle import nerf_oracle as O  # noqa: E402
from baked_finetune_time import BOX, FOCAL, H, HELD, heldout_psnr, poses_and_targets  # noqa: E402
from common import card, median, psnr, timed_mean, timed_once  # noqa: E402
from helpers import shipped_models  # noqa: E402

SIZES = {400: 555.6, 800: 1111.1}  # image side -> focal (the lego camera's field of view)
REPS = 10


def gib(field):
    return field.values.numel() * field.values.element_size() / 2 ** 30


def bake_arm(mf, grid, res, dtype):
    """(ms, added peak GiB, field) of one nb.bake."""
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ms, f = timed_once(lambda: nb.bake(mf, epf, edf, bounds=BOX, resolution=res, grid=grid, dtype=dtype))
    return ms, (torch.cuda.max_memory_allocated() - before) / 2 ** 30, f


def f16_vs_f32_psnr(h, f, poses):
    vals = []
    with torch.no_grad():
        for i in HELD:
            rays = ops.gen_rays(poses[i], H, H, FOCAL, None, "cuda", ndc=False, near=2.0, far=6.0, use_viewdirs=True)
            vals.append(psnr(nb.render_baked_rays(h, rays)[0], nb.render_baked_rays(f, rays)[0]))
    return sum(vals) / len(vals)


def one_res(mf, grid, res, poses, imgs, opts, rounds):
    rows = []
    bakes = {torch.float32: [], torch.float16: []}
    for dt in bakes:  # warm-up
        bake_arm(mf, grid, res, dt)
        torch.cuda.empty_cache()
    for _ in range(rounds):
        for dt in bakes:
            ms, peak, f = bake_arm(mf, grid, res, dt)
            bakes[dt].append((ms, peak))
            del f
            torch.cuda.empty_cache()
    f32 = nb.bake(mf, nb.get_embedding_function(10), nb.get_embedding_function(4), bounds=BOX, resolution=res, grid=grid)
    keep = ~nb.baked_transparent_bricks(f32)
    fields = {"none": (f32, f32.half())}
    fields["transparent"] = (nb.prune_baked(f32, keep), nb.prune_baked(fields["none"][1], keep))
    assert torch.equal(keep, ~nb.baked_transparent_bricks(fields["none"][1]))
    pose = O.pose_spherical(30.0, -30.0, 4.0)
    arms = {}
    for crit, pair in fields.items():
        for side, focal in SIZES.items():
            for stop in (None, 1e-3):
                for name, f in zip(("fp32", "fp16"), pair):
                    arms[(crit, side, stop, name)] = (lambda f=f, side=side, focal=focal, stop=stop:
                                                      nb.render_baked(f, side, side, focal, pose, opts, early_stop=stop))
    for fn in arms.values():
        fn()
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            ms[k].append(timed_mean(fn, REPS))
    bake_row = {("fp32" if dt == torch.float32 else "fp16"): dict(ms=median([b[0] for b in v]),
                                                                   peak_gib=max(b[1] for b in v))
                for dt, v in bakes.items()}
    print(f"{res}^3 bake: fp32 {bake_row['fp32']['ms']['ms']:8.1f} ms (peak +{bake_row['fp32']['peak_gib']:.2f} GiB), "
          f"fp16 {bake_row['fp16']['ms']['ms']:8.1f} ms (peak +{bake_row['fp16']['peak_gib']:.2f} GiB)", flush=True)
    # the fp16 field round-trips through save / load and renders as its widened copy, bit for bit
    f, h = fields["none"]
    with tempfile.TemporaryDirectory() as d:
        h.save(os.path.join(d, "f16.pt"))
        g = nb.BakedField.load(os.path.join(d, "f16.pt"))
    a = nb.render_baked(g, 800, 800, SIZES[800], pose, opts)
    b = nb.render_baked(h.float(), 800, 800, SIZES[800], pose, opts)
    same = all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in zip(a, b))
    print(f"{res}^3 save / load: dtype {g.dtype}, values {gib(g):.2f} GiB of the fp32 field's {gib(f):.2f}, 800^2 render "
          f"bit-equal to the widened field's: {same}", flush=True)
    assert same and g.dtype == torch.float16 and 2 * gib(g) == gib(f)
    del g, a, b
    for crit, (f, h) in fields.items():
        r = dict(res=res, criterion=crit, n_active=f.n_active, gib_fp32=gib(f), gib_fp16=gib(h),
                 psnr_f16_vs_f32=f16_vs_f32_psnr(h, f, poses), psnr_fp32=heldout_psnr(f, poses, imgs),
                 psnr_fp16=heldout_psnr(h, poses, imgs), bake=bake_row if crit == "none" else None, render={})
        for (c, side, stop, name), v in ms.items():
            if c == crit:
                r["render"][f"{side}x{side} early_stop {stop} {name}"] = median(v)
        rows.append(r)
        line = " | ".join(f"{side}^2{' es' if stop else ''} {r['render'][f'{side}x{side} early_stop {stop} fp32']['ms']:6.2f}"
                          f" / {r['render'][f'{side}x{side} early_stop {stop} fp16']['ms']:6.2f} ms"
                          for side in SIZES for stop in (None, 1e-3))
        print(f"{res}^3 {crit:11s} bricks {f.n_active:6d} values {r['gib_fp32']:5.2f} / {r['gib_fp16']:5.2f} GiB | "
              f"render fp32 / fp16: {line} | PSNR fp16 vs fp32 {r['psnr_f16_vs_f32']:.2f} dB, vs render_image "
              f"{r['psnr_fp32']:.3f} / {r['psnr_fp16']:.3f} dB", flush=True)
    del arms, fields, f32
    torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--res", type=int, nargs="*", default=[256, 512])
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    mc, mf = shipped_models("lego")[:2]
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    grid = nb.OccupancyGrid.from_models([mc, mf], epf, BOX, 128, encode_direction_fn=edf)
    poses, imgs, opts = poses_and_targets(mc, mf)
    out = dict(card=card(), rows=[])
    for res in a.res:
        out["rows"] += one_res(mf, grid, res, poses, imgs, opts, a.rounds)
    out["card_after"] = card()
    print("card after:", out["card_after"])
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
