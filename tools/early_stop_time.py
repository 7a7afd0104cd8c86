"""Dev tool: render_image with early ray termination (early_stop=t) against the default and the grid-only render,
inference only, impl 1 and impl 3.  Cases: the shipped lego A0 weights at 400 x 400 and 800 x 800, the shipped fern A0
weights in NDC (378 x 504), A1 at init (400 x 400: nothing is opaque, so no ray stops and the rounds are pure cost);
64 + 128 samples, deterministic sampling, one chunk per image.  Configurations: default, grid (OccupancyGrid.from_models,
128^3), grid + early_stop and early_stop alone at t in {1e-4, 1e-3, 1e-2}.  In one process, alternating the
configurations, CUDA events after warm-up: the median render time over ROUNDS rounds and its range; per configuration
the fine pass's evaluated rows, padding rows (64-row blocks the rounds filled minus rows) and the rounds that ran rows,
restated from stop_sample and the grid's kept samples; PSNR of the fine rgb against the default render.  The card's
name, power limit and SM clock are printed beside.

    python tools/early_stop_time.py [--rounds 5] [--json OUT]"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import nerf_pytorch_b200 as nb  # noqa: E402
from nerf_pytorch_b200 import ops, train_utils  # noqa: E402
from oracle import nerf_oracle as O  # noqa: E402

# name: (weights or None, layers, skip, L_xyz, H, W, focal, ndc, near, far, bounds)
CASES = {
    "lego_A0_400": ("lego", 4, 4, 10, 400, 400, 555.6, False, 2.0, 6.0, ((-1.5,) * 3, (1.5,) * 3)),
    "lego_A0_800": ("lego", 4, 4, 10, 800, 800, 1111.1, False, 2.0, 6.0, ((-1.5,) * 3, (1.5,) * 3)),
    "fern_A0_ndc": ("fern", 4, 4, 6, 378, 504, 407.6, True, 0.0, 1.0, ((-1.2, -1.2, -1.0), (1.2, 1.2, 1.0))),
    "A1_init_400": (None, 8, 3, 10, 400, 400, 555.6, False, 2.0, 6.0, ((-1.5,) * 3, (1.5,) * 3)),
}
IMPLS = {"impl1": ops.IMPL_TC, "impl3": ops.IMPL_TC_FAST}
THRESHOLDS = (1e-4, 1e-3, 1e-2)
GROUP = 10  # rays per compaction group (csrc/common.cuh kGridGroupRays)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True,
                           timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover - depends on the host
        q = f"nvidia-smi unavailable ({e})"
    return q or torch.cuda.get_device_name()


def models(weights, layers, skip, l_xyz):
    out = []
    torch.manual_seed(0)
    for i in range(2):
        m = nb.FlexibleNeRFModel(num_layers=layers, hidden_size=128, skip_connect_every=skip, num_encoding_fn_xyz=l_xyz,
                                 num_encoding_fn_dir=4)
        if weights:
            z = np.load(os.path.join(ROOT, "tests", "golden", f"weights_{weights}_lowres.npz"))
            pre = "cf"[i] + "."
            m.load_state_dict({k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith(pre)})
        out.append(m.cuda())
    return out


def timed(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def psnr(a, b):
    mse = (a.double() - b.double()).pow(2).mean().item()
    return math.inf if mse == 0 else -10.0 * math.log10(mse)


def round_stats(keep, stop, K):
    """(rows, padding rows, rounds with rows) of the fine pass's rounds, restated from the kept samples and stop_sample:
    round k gives each ray min(K, its run samples - k K) rows, each group of GROUP rays fills whole 64-row blocks."""
    S = keep.shape[1]
    j = torch.arange(S, device=keep.device)[None, :]
    ran = (keep & (j < stop[:, None])).sum(1)
    n = ran.shape[0]
    pad = (-n) % GROUP
    ran = torch.cat((ran, ran.new_zeros(pad))).view(-1, GROUP)
    rows = blocks = rounds = 0
    for k in range(-(-S // K)):
        per = (ran - k * K).clamp(0, K).sum(1)
        if per.sum() == 0:
            continue
        rounds += 1
        rows += int(per.sum())
        blocks += int(((per + 63) // 64).sum())
    return rows, 64 * blocks - rows, rounds


def run_case(name, rounds):
    weights, layers, skip, l_xyz, H, W, focal, ndc, near, far, bounds = CASES[name]
    mc, mf = models(weights, layers, skip, l_xyz)
    epf, edf = nb.get_embedding_function(l_xyz), nb.get_embedding_function(4)
    opts = O.make_options(no_ndc=not ndc, near=near, far=far, num_coarse=64, num_fine=128, perturb=False,
                          radiance_field_noise_std=0.0, chunksize=H * W)
    pose = torch.eye(4) if ndc else O.pose_spherical(30.0, -30.0, 4.0)
    grid = nb.OccupancyGrid.from_models([mc, mf], epf, bounds, 128, encode_direction_fn=edf)
    res = dict(case=name, occupied_fraction=grid.occupied_fraction)
    configs = [("default", None, None), ("grid", grid, None)]
    configs += [(f"grid+es{t:g}", grid, t) for t in THRESHOLDS] + [(f"es{t:g}", None, t) for t in THRESHOLDS]

    # rows, padding and rounds of each configuration's fine pass, on the whole image's rays in one call
    arch = train_utils._arch_of(mc, train_utils._probe_encoder(epf, None), train_utils._probe_encoder(edf, None))
    blobs = [train_utils._packed(m, arch)[1] for m in (mc, mf)]
    rays = ops.gen_rays(pose, H, W, focal, None, "cuda", ndc=ndc, near=near, far=far)
    ro = ops.make_opts(64, 128, False, False, False, 0.0)
    n = rays.shape[0]
    lay = ops.render_workspace_layout(arch, arch, ro, n, False)
    K = ops.stop_round()
    keeps = {}
    for g in (None, grid):
        if g is None:
            keeps[None] = torch.ones(n, 192, dtype=torch.bool, device="cuda")
            continue
        _, _, ws = ops.render_fwd_grid(arch, arch, ro, blobs[0], blobs[1], rays, {}, g, impl=ops.IMPL_TC)
        off = lay["raw_fine"] // 4
        keeps[id(g)] = ws.view(torch.float32)[off: off + n * 192 * 4].view(n, 192, 4)[..., 3] != -math.inf
        del ws
    stats = {}
    for label, g, t in configs:
        if t is None:
            keep = keeps[None] if g is None else keeps[id(g)]
            rows = int(keep.sum())
            stats[label] = dict(rows=rows, padding=None, rounds=None, stopped=0)
            continue
        _, _, ne, stop = ops.render_fwd_early_stop(arch, arch, ro, blobs[0], blobs[1], rays, {}, g, t,
                                                   impl=ops.IMPL_TC, want_stop=True)
        rows, padding, nr = round_stats(keeps[None] if g is None else keeps[id(g)], stop.long(), K)
        assert rows == ne[1].item(), (label, rows, ne.tolist())
        stats[label] = dict(rows=rows, padding=padding, rounds=nr, stopped=int((stop < 192).sum()))
    torch.cuda.empty_cache()

    def render(impl, g, t):
        with torch.no_grad():
            return nb.render_image(H, W, focal, pose, mc, mf, opts, mode="validation", encode_position_fn=epf,
                                   encode_direction_fn=edf, rays_per_chunk=H * W, impl=impl, grid=g, early_stop=t)

    for il, impl in IMPLS.items():
        for _ in range(2):
            for _, g, t in configs:
                render(impl, g, t)
        ms = {c[0]: [] for c in configs}
        outs = {}
        for _ in range(rounds):
            for label, g, t in configs:
                dt, outs[label] = timed(lambda: render(impl, g, t))
                ms[label].append(dt)
        res[il] = {}
        for label, _, _ in configs:
            m = ms[label]
            r = dict(ms=statistics.median(m), range=(min(m), max(m)),
                     psnr_fine=psnr(outs[label][3], outs["default"][3]), **stats[label])
            res[il][label] = r
            extra = "" if r["padding"] is None else f" padding {r['padding']:9d} rounds {r['rounds']} stopped " \
                                                    f"{r['stopped'] / n:.3f}"
            print(f"{name:12s} {il} {label:14s} {r['ms']:8.2f} ms [{r['range'][0]:.2f}, {r['range'][1]:.2f}]  fine rows "
                  f"{r['rows'] / (n * 192):.4f} of all{extra}  PSNR fine {r['psnr_fine']:.2f} dB", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    out = dict(card=card(), stop_round=ops.stop_round(), cases=[run_case(c, a.rounds) for c in a.cases.split(",")])
    out["card_after"] = card()
    print("card after:", out["card_after"])
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
