"""Dev tool: normal maps and point queries of baked fields (render_baked(normals=), nb.baked_raw,
nb.baked_density_gradient; csrc/baked.cu baked_render_kernel<V, true, false>, baked_query_kernel<V>) on the lego
scene.

lego A0 (shipped weights) baked at 256^3 and 512^3 over OccupancyGrid.from_models (128^3) of both networks; the fp32
bake, its half() and its quantize().  For each field it reports:

  render   render_baked at 400 x 400 and 800 x 800 (the lego camera's field of view) with and without normals=True,
           CUDA events, and the normals render's extra time;
  query    ops.baked_query over 2^22 random points of the box, raw alone and raw with the gradient, in points/s;
  angle    the mean angle (degrees) between the baked normal map and render_image(normals=True) (64 + 128 samples,
           deterministic, impl 1) over the pixels with acc > 0.5 in both, at the 4 held-out 48 x 48 views of
           tools/baked_finetune_time.py.

In one process; the arms alternate in every round after a warm-up, medians over ROUNDS rounds (each figure the mean of
REPS launches) and their range.  The normals render's image is checked bit-equal to the render without normals.  The
card's name, power limit and SM clock are read in the same run.

    python tools/baked_normals_time.py [--rounds 5] [--res 256 512] [--json OUT]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import nerf_pytorch_b200 as nb  # noqa: E402
from nerf_pytorch_b200 import ops  # noqa: E402
from oracle import nerf_oracle as O  # noqa: E402
from baked_finetune_time import BOX, FOCAL, H, HELD, poses_and_targets  # noqa: E402
from common import card, median, timed_mean  # noqa: E402
from helpers import shipped_models  # noqa: E402

SIDES = {400: 555.6, 800: 1111.1}  # image side -> focal (the lego camera's field of view)
REPS = 10
N_POINTS = 1 << 22


def angle_deg(field, mc, mf, poses, opts):
    """Mean angle (degrees) between the field's normal map and render_image's over the pixels with acc > 0.5 in both."""
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    angles = []
    with torch.no_grad():
        for i in HELD:
            _, _, acc_b, nrm_b = nb.render_baked(field, H, H, FOCAL, poses[i], opts, normals=True)
            net = nb.render_image(H, H, FOCAL, poses[i], mc, mf, opts, encode_position_fn=epf,
                                  encode_direction_fn=edf, impl=1, normals=True)
            m = (acc_b > 0.5) & (net[5] > 0.5)
            a = torch.nn.functional.normalize(nrm_b[m].double(), dim=-1)
            b = torch.nn.functional.normalize(net[6][m].double(), dim=-1)
            angles.append(torch.rad2deg(torch.acos((a * b).sum(-1).clamp(-1, 1))))
    return torch.cat(angles).mean().item()


def one_res(mc, mf, grid, res, poses, opts, rounds):
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    f32 = nb.bake(mf, epf, edf, bounds=BOX, resolution=res, grid=grid)
    fields = {"fp32": f32, "fp16": f32.half(), "uint8": f32.quantize()}
    pose = O.pose_spherical(30.0, -30.0, 4.0)
    g = torch.Generator(device="cuda").manual_seed(0)
    pts = (torch.rand(N_POINTS, 3, generator=g, device="cuda") * 3.0 - 1.5).contiguous()
    dirs = torch.nn.functional.normalize(torch.randn(N_POINTS, 3, generator=g, device="cuda"), dim=-1).contiguous()
    arms = {}
    for name, f in fields.items():
        for side, focal in SIDES.items():
            for nrm in (False, True):
                arms[("render", name, side, nrm)] = \
                    lambda f=f, side=side, focal=focal, nrm=nrm: nb.render_baked(f, side, side, focal, pose, opts,
                                                                                 normals=nrm)
        for grad in (False, True):
            arms[("query", name, grad)] = lambda f=f, grad=grad: ops.baked_query(
                f.box(), f.brick_map, f.values, True, pts, dirs, True, grad, dequant=f.dequant)
    for fn in arms.values():
        fn()
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            ms[k].append(timed_mean(fn, REPS))
    same = all(torch.equal(x.view(torch.int32), y.view(torch.int32))
               for k in arms if k[0] == "render" and not k[3]
               for x, y in zip(arms[k](), arms[k[:3] + (True,)]()[:3]))
    print(f"{res}^3: every normals render's image bit-equal to the render without normals: {same}", flush=True)
    assert same
    rows = []
    for name, f in fields.items():
        r = dict(res=res, field=name, n_active=f.n_active, angle_deg=angle_deg(f, mc, mf, poses, opts))
        for side in SIDES:
            r[f"render{side}"] = median(ms[("render", name, side, False)])
            r[f"render{side}_normals"] = median(ms[("render", name, side, True)])
        for grad in (False, True):
            t = median(ms[("query", name, grad)])
            r["query_grad" if grad else "query_raw"] = dict(t, points_per_s=N_POINTS / (t["ms"] * 1e-3))
        rows.append(r)
        line = " | ".join(f"{side}^2 {r[f'render{side}']['ms']:6.2f} -> {r[f'render{side}_normals']['ms']:6.2f} ms "
                          f"(+{100 * (r[f'render{side}_normals']['ms'] / r[f'render{side}']['ms'] - 1):4.1f} %)"
                          for side in SIDES)
        print(f"{res}^3 {name:5s} bricks {f.n_active:6d} | render without -> with normals {line} | query raw "
              f"{r['query_raw']['points_per_s'] / 1e9:5.2f} G points/s, raw + grad "
              f"{r['query_grad']['points_per_s'] / 1e9:5.2f} G points/s | angle vs render_image "
              f"{r['angle_deg']:.2f} deg", flush=True)
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
    poses, _, opts = poses_and_targets(mc, mf)
    out = dict(card=card(), rows=[])
    for res in a.res:
        out["rows"] += one_res(mc, mf, grid, res, poses, opts, a.rounds)
    out["card_after"] = card()
    print("card after:", out["card_after"])
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
