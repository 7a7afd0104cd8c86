"""Dev tool: render_image with an occupancy grid against the default render, inference only, impl 1 and impl 3.
Cases: the shipped lego A0 weights at 400 x 400 and 800 x 800, A1 at init (400 x 400), the shipped fern A0 weights in NDC
(378 x 504); 64 + 128 samples, deterministic sampling.  For each case and impl, in one process, alternating the two
paths, CUDA events after warm-up: the median render time over ROUNDS rounds and its range, the grid's build time
(OccupancyGrid.from_models, 128^3, 8 probes per cell), its occupied fraction, the fraction of samples evaluated per pass,
and the PSNR of the grid render against the default one.  The card's name, power limit and SM clock are printed beside.

    python tools/grid_render_time.py [--rounds 5] [--json OUT]"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from common import card, models, psnr, timed_once  # noqa: E402
import nerf_pytorch_b200 as nb  # noqa: E402
from nerf_pytorch_b200 import ops, train_utils  # noqa: E402
from oracle import nerf_oracle as O  # noqa: E402

# name: (weights or None, layers, skip, L_xyz, H, W, focal, ndc, near, far, bounds)
CASES = {
    "lego_A0_400": ("lego", 4, 4, 10, 400, 400, 555.6, False, 2.0, 6.0, ((-1.5,) * 3, (1.5,) * 3)),
    "lego_A0_800": ("lego", 4, 4, 10, 800, 800, 1111.1, False, 2.0, 6.0, ((-1.5,) * 3, (1.5,) * 3)),
    "A1_init_400": (None, 8, 3, 10, 400, 400, 555.6, False, 2.0, 6.0, ((-1.5,) * 3, (1.5,) * 3)),
    "fern_A0_ndc": ("fern", 4, 4, 6, 378, 504, 407.6, True, 0.0, 1.0, ((-1.2, -1.2, -1.0), (1.2, 1.2, 1.0))),
}
IMPLS = {"impl1": ops.IMPL_TC, "impl3": ops.IMPL_TC_FAST}


def run_case(name, rounds):
    weights, layers, skip, l_xyz, H, W, focal, ndc, near, far, bounds = CASES[name]
    mc, mf = models(weights, layers, skip, l_xyz)
    epf, edf = nb.get_embedding_function(l_xyz), nb.get_embedding_function(4)
    opts = O.make_options(no_ndc=not ndc, near=near, far=far, num_coarse=64, num_fine=128, perturb=False,
                          radiance_field_noise_std=0.0, chunksize=H * W)
    pose = torch.eye(4) if ndc else O.pose_spherical(30.0, -30.0, 4.0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    grid = nb.OccupancyGrid.from_models([mc, mf], epf, bounds, 128, encode_direction_fn=edf)
    torch.cuda.synchronize()
    build_ms = (time.perf_counter() - t0) * 1e3
    res = dict(case=name, grid_build_ms=build_ms, occupied_fraction=grid.occupied_fraction)

    # evaluated fraction per pass, on the whole image's rays in one call
    arch = train_utils._arch_of(mc, train_utils._probe_encoder(epf, None), train_utils._probe_encoder(edf, None))
    blobs = [train_utils._packed(m, arch)[1] for m in (mc, mf)]
    rays = ops.gen_rays(pose, H, W, focal, None, "cuda", ndc=ndc, near=near, far=far)
    ne = torch.zeros(2, dtype=torch.int64, device="cuda")
    ops.render_fwd_grid(arch, arch, ops.make_opts(64, 128, False, False, False, 0.0), blobs[0], blobs[1], rays, {},
                        grid, impl=ops.IMPL_TC, n_evaluated=ne)
    n = rays.shape[0]
    res["evaluated_fraction"] = dict(coarse=ne[0].item() / (n * 64), fine=ne[1].item() / (n * 192))

    def render(impl, g):
        with torch.no_grad():
            return nb.render_image(H, W, focal, pose, mc, mf, opts, mode="validation", encode_position_fn=epf,
                                   encode_direction_fn=edf, rays_per_chunk=H * W, impl=impl, grid=g)

    for label, impl in IMPLS.items():
        for _ in range(2):
            render(impl, None), render(impl, grid)
        ms = {"default": [], "grid": []}
        outs = {}
        for _ in range(rounds):
            for path, g in (("default", None), ("grid", grid)):
                t, outs[path] = timed_once(lambda: render(impl, g))
                ms[path].append(t)
        speed = [d / g for d, g in zip(ms["default"], ms["grid"])]
        res[label] = dict(
            default_ms=statistics.median(ms["default"]), default_range=(min(ms["default"]), max(ms["default"])),
            grid_ms=statistics.median(ms["grid"]), grid_range=(min(ms["grid"]), max(ms["grid"])),
            speedup=statistics.median(speed), speedup_range=(min(speed), max(speed)),
            psnr_fine=psnr(outs["grid"][3], outs["default"][3]), psnr_coarse=psnr(outs["grid"][0], outs["default"][0]))
        r = res[label]
        print(f"{name:12s} {label}: default {r['default_ms']:8.2f} ms  grid {r['grid_ms']:8.2f} ms  speed-up "
              f"{r['speedup']:.2f}x [{r['speedup_range'][0]:.2f}, {r['speedup_range'][1]:.2f}]  PSNR fine "
              f"{r['psnr_fine']:.2f} coarse {r['psnr_coarse']:.2f} dB", flush=True)
    print(f"{name:12s} grid build {build_ms:.1f} ms, occupied {res['occupied_fraction']:.4f}, evaluated coarse "
          f"{res['evaluated_fraction']['coarse']:.4f} fine {res['evaluated_fraction']['fine']:.4f}", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    out = dict(card=card(), cases=[run_case(c, a.rounds) for c in a.cases.split(",")])
    out["card_after"] = card()
    print("card after:", out["card_after"])
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
