"""Dev tool: 8-bit baked fields (BakedField.quantize; csrc/baked.cu baked_render_kernel<uint8_t>,
baked_max_weight_kernel<uint8_t>) against fp32 and fp16 ones on the lego scene.

lego A0 (shipped weights) baked at 256^3 and 512^3 over OccupancyGrid.from_models (128^3) of both networks; the fp32
bake, its half() and its quantize().  For each field it reports:

  bytes     the values' GiB;
  quantize  BakedField.quantize time from the fp32 field and from the fp16 field (the codes of its widened values);
  render    render_baked at 800 x 800 (the lego camera's field of view), CUDA events;
  weights   baked_brick_weights over that 800 x 800 view, CUDA events;
  psnr      mean over the 4 held-out views of tools/baked_finetune_time.py (48 x 48) of the render against the fp32
            field's and against render_image (64 + 128 samples, deterministic, impl 1); also for the quantised
            transparent-pruned fp32 field, with its sigma_raw scale against the unpruned field's.

In one process; the three arms alternate in every round after a warm-up, medians over ROUNDS rounds (each render and
weights figure the mean of REPS launches) and their range.  Every 8-bit render is checked bit-equal to the render of
its float() field.  The card's name, power limit and SM clock are read in the same run.

    python tools/baked_u8_time.py [--rounds 5] [--res 256 512] [--json OUT]"""
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
from baked_finetune_time import BOX, FOCAL, H, HELD, heldout_psnr, poses_and_targets  # noqa: E402
from common import card, median, psnr, timed_mean, timed_once  # noqa: E402
from helpers import shipped_models  # noqa: E402

SIDE, SIDE_FOCAL = 800, 1111.1  # image side and focal (the lego camera's field of view)
REPS = 10


def gib(field):
    return field.values.numel() * field.values.element_size() / 2 ** 30


def vs_fp32_psnr(g, f, poses):
    vals = []
    with torch.no_grad():
        for i in HELD:
            rays = ops.gen_rays(poses[i], H, H, FOCAL, None, "cuda", ndc=False, near=2.0, far=6.0, use_viewdirs=True)
            vals.append(psnr(nb.render_baked_rays(g, rays)[0], nb.render_baked_rays(f, rays)[0]))
    return sum(vals) / len(vals)


def one_res(mf, grid, res, poses, imgs, opts, rounds):
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    f32 = nb.bake(mf, epf, edf, bounds=BOX, resolution=res, grid=grid)
    f16 = f32.half()
    fields = {"fp32": f32, "fp16": f16, "uint8": f32.quantize()}
    # quantize() from fp32 and from fp16, alternating
    quant = {"fp32": [], "fp16": []}
    for src in quant:  # warm-up
        fields[src].quantize()
    for _ in range(rounds):
        for src in quant:
            ms, q = timed_once(fields[src].quantize)
            quant[src].append(ms)
            del q
    torch.cuda.empty_cache()
    pose = O.pose_spherical(30.0, -30.0, 4.0)
    posev = pose[None]
    arms = {}
    for name, f in fields.items():
        arms[("render", name)] = lambda f=f: nb.render_baked(f, SIDE, SIDE, SIDE_FOCAL, pose, opts)
        arms[("weights", name)] = lambda f=f: nb.baked_brick_weights(f, posev, SIDE, SIDE, SIDE_FOCAL, opts)
    for fn in arms.values():
        fn()
    ms = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            ms[k].append(timed_mean(fn, REPS))
    # an 8-bit field renders and weighs as its dequantised field, bit for bit
    q, w = fields["uint8"], fields["uint8"].float()
    same = all(torch.equal(x.view(torch.int32), y.view(torch.int32)) for x, y in
               zip(arms[("render", "uint8")](), nb.render_baked(w, SIDE, SIDE, SIDE_FOCAL, pose, opts)))
    same = same and torch.equal(arms[("weights", "uint8")]().view(torch.int32),
                                nb.baked_brick_weights(w, posev, SIDE, SIDE, SIDE_FOCAL, opts).view(torch.int32))
    print(f"{res}^3: 800^2 render and peak weights of the 8-bit field bit-equal to its float() field's: {same}",
          flush=True)
    assert same
    del w
    rows = []
    for name, f in fields.items():
        r = dict(res=res, field=name, n_active=f.n_active, gib=gib(f),
                 quantize=median(quant[name]) if name in quant else None,
                 render=median(ms[("render", name)]), weights=median(ms[("weights", name)]),
                 psnr_vs_fp32=vs_fp32_psnr(f, f32, poses) if name != "fp32" else None,
                 psnr_vs_render_image=heldout_psnr(f, poses, imgs),
                 scale_sigma=float(f.dequant[0, 0]) if f.dequant is not None else None)
        rows.append(r)
        qs = f"quantize {r['quantize']['ms']:7.1f} ms | " if r["quantize"] else ""
        vs = f"{r['psnr_vs_fp32']:6.2f}" if r["psnr_vs_fp32"] is not None else "     -"
        print(f"{res}^3 {name:5s} bricks {f.n_active:6d} values {r['gib']:5.2f} GiB | {qs}render 800^2 "
              f"{r['render']['ms']:6.2f} ms ({r['render']['range'][0]:.2f} .. {r['render']['range'][1]:.2f}) | "
              f"weights {r['weights']['ms']:6.2f} ms ({r['weights']['range'][0]:.2f} .. {r['weights']['range'][1]:.2f})"
              f" | PSNR vs fp32 {vs} dB, vs render_image {r['psnr_vs_render_image']:.3f} dB", flush=True)
    # the range of every channel spans the whole field; quantising the transparent-pruned field instead
    del arms, fields, f16, q
    torch.cuda.empty_cache()
    p = nb.prune_baked(f32, ~nb.baked_transparent_bricks(f32))
    pq = p.quantize()
    r = dict(res=res, field="uint8 of the transparent-pruned fp32 field", n_active=p.n_active, gib=gib(pq),
             psnr_vs_fp32=vs_fp32_psnr(pq, f32, poses), psnr_vs_render_image=heldout_psnr(pq, poses, imgs),
             scale_sigma=float(pq.dequant[0, 0]))
    rows.append(r)
    print(f"{res}^3 uint8 of the transparent-pruned field: bricks {p.n_active:6d} values {r['gib']:5.2f} GiB | sigma_raw "
          f"scale {r['scale_sigma']:.3f} (unpruned {rows[2]['scale_sigma']:.3f}) | PSNR vs fp32 {r['psnr_vs_fp32']:6.2f} "
          f"dB, vs render_image {r['psnr_vs_render_image']:.3f} dB", flush=True)
    del p, pq, f32
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
