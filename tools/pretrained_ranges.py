"""How close the pretrained networks come to the fp16 x 2 split's range, on the CPU in fp64.

The wgmma kernels hold every A operand, and the training forward every stashed activation tile, as value / 16 split
into fp16 hi + lo: a value with |x| >= 16 x 65504 (1.05e6) does not fit.  For each of the seven pretrained scenes
(helpers.PRETRAINED_SCENES) and each network, this runs oracle.nerf_oracle's forward in fp64 at
  * rays: the points a training render samples, from ``--poses`` poses of the scene's ring (helpers.pretrained_poses),
    ``--rays`` random pixels each: 64 stratified coarse depths from seeded randoms, and the fine network at those plus
    the config's fine count drawn by inverse CDF (seeded u) of the fp64 coarse weights with seeded noise, as the
    library's render samples them;
  * box: ``--box`` uniform points of the scene's box (helpers.PRETRAINED_BOX) scaled by ``--box-scale``, random unit
    directions;
and prints, per network, the largest |value| of every split operand -- the encodings, layer1's output (no ReLU), each
layers_xyz output, fc_feat's output (the A operand of layers_dir.0) -- and of layers_dir.0's output (the stash tile the
backward reads for fc_rgb's weight gradient), with the number of points where any unit of that tensor reaches 1.05e6.

    python tools/pretrained_ranges.py [--scenes lego drums] [--poses 8] [--rays 512] [--box 65536]
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from helpers import PRETRAINED_BOX, PRETRAINED_SCENES, load_weights, pretrained_arch, pretrained_poses  # noqa: E402
from oracle import nerf_oracle as O  # noqa: E402

LIMIT = 16.0 * 65504.0
COLUMNS = ["enc", "layer1", "layers_xyz.0", "layers_xyz.1", "layers_xyz.2", "fc_feat", "layers_dir.0"]


def scene_rays(scene, poses, n_rays, seed):
    """fp32 ray rows (o, d, near, far, unit d) of n_rays random pixels of each pose, NDC for fern, as ops.gen_rays
    forms them (train_utils.py:143-168 through the oracle's helpers)."""
    *_, ndc, near, far, _, _, (H, W, focal) = PRETRAINED_SCENES[scene]
    g = torch.Generator().manual_seed(seed)
    rows = []
    for pose in poses:
        ro, rd = O.get_ray_bundle(H, W, focal, pose)
        pix = torch.randperm(H * W, generator=g)[:n_rays]
        ro, rd = ro.reshape(-1, 3)[pix], rd.reshape(-1, 3)[pix]
        vd = rd / rd.norm(dim=-1, keepdim=True)
        if ndc:
            ro, rd = O.ndc_rays(H, W, focal, 1.0, ro, rd)
        rows.append(torch.cat([ro, rd, torch.full_like(ro[:, :1], near), torch.full_like(ro[:, :1], far), vd], -1))
    return torch.cat(rows)


def encode(arch, pts, dirs):
    """fp64 [xyz encoding | direction encoding] of fp32 points and unit directions (x * 2^k is exact in fp64)."""
    parts = [O.positional_encoding(pts.double(), arch.n_freq_xyz), O.positional_encoding(dirs.double(), arch.n_freq_dir)]
    return torch.cat(parts, -1)


class Maxima:
    """Running max |value| and count of points past LIMIT per column."""

    def __init__(self):
        self.mx = {c: 0.0 for c in COLUMNS}
        self.over = {c: 0 for c in COLUMNS}
        self.points = 0

    def add(self, sd64, emb, dim_xyz):
        raw, acts = O.flexible_nerf_forward(sd64, emb, dim_xyz, return_acts=True)
        vals = {"enc": emb, "layer1": acts["h0"], "layers_xyz.0": acts["h1"], "layers_xyz.1": acts["h2"],
                "layers_xyz.2": acts["h3"], "fc_feat": acts["feat"], "layers_dir.0": acts["d"]}
        for c, v in vals.items():
            a = v.abs().amax(-1)
            self.mx[c] = max(self.mx[c], a.max().item())
            self.over[c] += int((a >= LIMIT).sum())
        self.points += emb.shape[0]
        return raw


def forward_in_chunks(stats, sd64, arch, pts, dirs, chunk=1 << 16):
    out = []
    for p0 in range(0, pts.shape[0], chunk):
        out.append(stats.add(sd64, encode(arch, pts[p0:p0 + chunk], dirs[p0:p0 + chunk]), arch.dim_xyz))
    return torch.cat(out)


def ray_maxima(scene, sds, rays, seed):
    """Maxima of the coarse and the fine network at the points a training render of `rays` samples."""
    arch = pretrained_arch(scene)
    _, nf, _, _, _, white, noise, _ = PRETRAINED_SCENES[scene]
    n, nc = rays.shape[0], 64
    g = torch.Generator().manual_seed(seed)
    t_rand, noise_c = torch.rand(n, nc, generator=g), torch.randn(n, nc, generator=g)
    u = torch.rand(n, nf, generator=g)
    z_c = O.stratified_z(rays[:, 6:7], rays[:, 7:8], nc, False, True, t_rand, torch.float32)
    sd_c, sd_f = ({k: v.double() for k, v in sd.items()} for sd in sds)
    stats = Maxima(), Maxima()

    def points(z):
        pts = (rays[:, None, :3] + rays[:, None, 3:6] * z[..., None]).reshape(-1, 3)
        return pts, rays[:, None, 8:11].expand(n, z.shape[1], 3).reshape(-1, 3)

    raw_c = forward_in_chunks(stats[0], sd_c, arch, *points(z_c)).view(n, nc, 4)
    _, _, _, w, _ = O.volume_render_radiance_field(raw_c, z_c.double(), rays[:, 3:6].double(), noise, white,
                                                   noise=noise_c.double())
    mids = 0.5 * (z_c[:, 1:] + z_c[:, :-1])
    z_s = O.sample_pdf(mids.double(), w[:, 1:-1], nf, u=u.double()).float()
    z_f = torch.sort(torch.cat([z_c, z_s], -1), -1).values
    forward_in_chunks(stats[1], sd_f, arch, *points(z_f))
    return stats


def box_maxima(scene, sds, n, scale, seed):
    arch = pretrained_arch(scene)
    lo, hi = (torch.tensor(b) * scale for b in PRETRAINED_BOX[scene])
    g = torch.Generator().manual_seed(seed)
    pts = lo + (hi - lo) * torch.rand(n, 3, generator=g)
    dirs = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    out = []
    for sd in sds:
        s = Maxima()
        forward_in_chunks(s, {k: v.double() for k, v in sd.items()}, arch, pts, dirs)
        out.append(s)
    return out


def table(title, rows):
    print(f"\n{title}: max |value| per split operand (points with a unit >= 1.05e6 in brackets where any)")
    print(f"{'network':18s} {'points':>9s} " + " ".join(f"{c:>17s}" for c in COLUMNS))
    for name, s in rows:
        cells = [f"{s.mx[c]:.3g}" + (f" [{s.over[c]}]" if s.over[c] else "") for c in COLUMNS]
        print(f"{name:18s} {s.points:9d} " + " ".join(f"{c:>17s}" for c in cells))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--scenes", nargs="*", default=sorted(PRETRAINED_SCENES))
    ap.add_argument("--poses", type=int, default=8)
    ap.add_argument("--rays", type=int, default=512, help="random pixels per pose")
    ap.add_argument("--box", type=int, default=1 << 16, help="uniform box points")
    ap.add_argument("--box-scale", type=float, default=1.0)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    rays_rows, box_rows = [], []
    for scene in a.scenes:
        sds = load_weights(f"{scene}_lowres")
        rays = scene_rays(scene, pretrained_poses(scene, a.poses), a.rays, a.seed)
        for tag, s in zip(("coarse", "fine"), ray_maxima(scene, sds, rays, a.seed + 1)):
            rays_rows.append((f"{scene} {tag}", s))
        for tag, s in zip(("coarse", "fine"), box_maxima(scene, sds, a.box, a.box_scale, a.seed + 2)):
            box_rows.append((f"{scene} {tag}", s))
        print(f"[{scene}] done", file=sys.stderr, flush=True)
    table(f"rays ({a.poses} poses x {a.rays} pixels, 64 coarse + the config's fine samples, seed {a.seed})", rays_rows)
    table(f"box points ({a.box} uniform in the scene's box x {a.box_scale:g})", box_rows)


if __name__ == "__main__":
    main()
