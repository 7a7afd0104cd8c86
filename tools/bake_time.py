"""Dev tool: baked fields (nb.bake / nb.render_baked) on the lego scene.

  bake     lego A0 (shipped fine weights), A1 and A2 (at init) baked at 256^3 and 512^3 over the bricks of the lego
           grid (OccupancyGrid.from_models of the shipped pair, 128^3, so every architecture bakes the same bricks),
           against the same bake done as 64 mlp_fwd_pts(impl=1) calls plus a torch projection onto the SH basis;
           active bricks and bytes;
  render   render_baked of the lego A0 fields at 400 x 400 and 800 x 800 against render_image (64 + 128 samples,
           deterministic, one chunk) default, with the grid, and with grid + early_stop=1e-3, impl 1 and 3; PSNR of
           each against render_image's default fine output.
In one process, alternating the configurations of each table after a warm-up, CUDA events; medians over ROUNDS rounds
and their range.  The card's name, power limit and SM clock are read in the same run.

    python tools/bake_time.py [--rounds 3] [--json OUT]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from common import card, median, psnr, timed_once  # noqa: E402
from helpers import shipped_models  # noqa: E402
import nerf_pytorch_b200 as nb  # noqa: E402
from nerf_pytorch_b200 import mesh, ops, train_utils  # noqa: E402
from oracle import nerf_oracle as O  # noqa: E402

BOX = ((-1.5,) * 3, (1.5,) * 3)
ARCHS = {"A0": (4, 128, 4), "A1": (8, 128, 3), "A2": (8, 256, 4)}  # layers, hidden, skip


def bake_table(grid, rounds):
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    dirs, proj = ops.bake_basis()
    dirs, proj = dirs.cuda(), proj.cuda()
    rows = []
    for name, (layers, hidden, skip) in ARCHS.items():
        if name == "A0":
            m = shipped_models("lego")[1]
        else:
            torch.manual_seed(0)
            m = nb.FlexibleNeRFModel(num_layers=layers, hidden_size=hidden, skip_connect_every=skip,
                                      num_encoding_fn_xyz=10).cuda()
        arch = mesh._network(m, epf, edf)
        _, blob = train_utils._packed(m, arch)
        for res in (256, 512):
            box = ops.grid_struct(BOX, (res,) * 3)
            brick_map, bricks, n_dev = ops.mesh_sparse_bricks(box, grid)
            n = int(n_dev.item())
            P = n * 729
            values = torch.empty(n, 729, 32, device="cuda")
            rows_ = -(-P // 64)
            pts = torch.zeros(rows_ * 64, 3, device="cuda")
            ops.mesh_sparse_points(box, bricks, 0, n, False, pts)
            coef = torch.empty(P, 27, device="cuda")

            def fused():
                return ops.bake(arch, blob, box, bricks, 0, n, values)

            def unfused():
                coef.zero_()
                for d in range(64):
                    raw = ops.mlp_fwd_pts(arch, blob, pts.view(rows_, 64, 3), dirs[d].view(1, 3).expand(rows_, 3).contiguous(),
                                          impl=1).view(-1, 4)[:P]
                    coef.view(P, 3, 9).add_(raw[:, :3, None] * proj[None, None, :, d])
                return coef

            for _ in range(2):
                fused(), unfused()
            t_f, t_u = [], []
            for _ in range(rounds):
                t_f.append(timed_once(fused)[0])
                t_u.append(timed_once(unfused)[0])
            # the two agree up to the projection's summation order
            diff = (values.view(P, 32)[:, 1:28] - coef).abs().max().item()
            r = dict(arch=name, res=res, n_active=n, bricks=ops.mesh_sparse_brick_count(box), bytes=values.numel() * 4,
                     bake=median(t_f), unfused=median(t_u), max_coef_diff=diff)
            rows.append(r)
            print(f"bake {name} {res}^3: {n} of {r['bricks']} bricks, {r['bytes'] / 2 ** 30:.2f} GiB;  fused "
                  f"{r['bake']['ms']:9.2f} ms {r['bake']['range']}  64 x mlp_fwd_pts + projection {r['unfused']['ms']:9.2f} "
                  f"ms {r['unfused']['range']}  x{r['unfused']['ms'] / r['bake']['ms']:.1f}  max |coef diff| {diff:.2e}",
                  flush=True)
            del values, pts, coef
            torch.cuda.empty_cache()
    return rows


def render_table(mc, mf, grid, rounds):
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    pose = O.pose_spherical(30.0, -30.0, 4.0)
    fields = {res: nb.bake(mf, epf, edf, bounds=BOX, resolution=res, grid=grid) for res in (256, 512)}
    out = []
    for H, focal in ((400, 555.6), (800, 1111.1)):
        opts = O.make_options(near=2.0, far=6.0, num_coarse=64, num_fine=128, perturb=False,
                              radiance_field_noise_std=0.0, chunksize=H * H)

        def net(impl, g, t):
            def f():
                with torch.no_grad():
                    return nb.render_image(H, H, focal, pose, mc, mf, opts, encode_position_fn=epf,
                                           encode_direction_fn=edf, rays_per_chunk=H * H, impl=impl, grid=g,
                                           early_stop=t)[3]
            return f

        def baked(res):
            return lambda: nb.render_baked(fields[res], H, H, focal, pose, opts)[0]

        configs = {"baked256": baked(256), "baked512": baked(512)}
        for il, impl in (("impl1", 1), ("impl3", 3)):
            configs[f"default_{il}"] = net(impl, None, None)
            configs[f"grid_{il}"] = net(impl, grid, None)
            configs[f"grid+es1e-3_{il}"] = net(impl, grid, 1e-3)
        for _ in range(2):
            for f in configs.values():
                f()
        ms = {k: [] for k in configs}
        imgs = {}
        for _ in range(rounds):
            for k, f in configs.items():
                dt, imgs[k] = timed_once(f)
                ms[k].append(dt)
        for k in configs:
            r = dict(size=H, config=k, psnr=psnr(imgs[k], imgs["default_impl1"]), **median(ms[k]))
            out.append(r)
            print(f"render {H}x{H} {k:18s} {r['ms']:8.2f} ms [{r['range'][0]:.2f}, {r['range'][1]:.2f}]  PSNR vs default "
                  f"{r['psnr']:.2f} dB", flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    mc, mf = shipped_models("lego")[:2]
    grid = nb.OccupancyGrid.from_models([mc, mf], nb.get_embedding_function(10), BOX, 128,
                                        encode_direction_fn=nb.get_embedding_function(4))
    out = dict(card=card(), occupied_fraction=grid.occupied_fraction, bake=bake_table(grid, a.rounds),
               render=render_table(mc, mf, grid, a.rounds))
    out["card_after"] = card()
    print("card after:", out["card_after"])
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
