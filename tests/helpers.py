"""Shared test plumbing: golden-case loading, oracle drivers, error metrics.  (tests/ may use oracle/.)"""
from __future__ import annotations

import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from oracle import nerf_oracle as O  # noqa: E402

CASES = ["lego_a0_train", "lego_a0_det_white_val", "fern_a0_ndc", "a1_skip_lindisp", "a0_noview_coarse_only"]
OUT_NAMES = ["rgb_coarse", "disp_coarse", "acc_coarse", "rgb_fine", "disp_fine", "acc_fine"]


def load_weights(name):
    z = np.load(os.path.join(GOLD, f"weights_{name}.npz"))
    sd_c = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("c.")}
    sd_f = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("f.")}
    return sd_c, sd_f


class Case:
    def __init__(self, name):
        z = np.load(os.path.join(GOLD, name + ".npz"))
        self.name = name
        self.z = z
        self.H, self.W, self.focal = int(z["H"]), int(z["W"]), float(z["focal"])
        self.ro, self.rd = torch.from_numpy(z["ro"]), torch.from_numpy(z["rd"])
        self.target = torch.from_numpy(z["target"])
        self.enc_xyz = (int(z["enc_xyz"][0]), bool(z["enc_xyz"][1]), bool(z["enc_xyz"][2]))
        self.enc_dir = (int(z["enc_dir"][0]), bool(z["enc_dir"][1]), bool(z["enc_dir"][2]))
        self.use_viewdirs = bool(z["use_viewdirs"])
        self.mode = str(z["mode"])
        self.num_layers, self.hidden, self.skip = (int(v) for v in z["arch"])
        self.options = O.make_options(
            use_viewdirs=self.use_viewdirs, no_ndc=bool(z["no_ndc"]), near=float(z["near"]), far=float(z["far"]),
            num_coarse=int(z["num_coarse"]), num_fine=int(z["num_fine"]), perturb=bool(z["perturb"]),
            lindisp=bool(z["lindisp"]), white_background=bool(z["white_background"]),
            radiance_field_noise_std=float(z["noise_std"]))
        self.randoms = {k[4:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("rnd_")}
        self.outputs = [torch.from_numpy(z["out_" + n]) if ("out_" + n) in z.files else None for n in OUT_NAMES]
        self.loss = float(z["loss"])
        # weights
        if name.startswith("lego"):
            self.sd_c, self.sd_f = load_weights("lego_lowres")
        elif name.startswith("fern"):
            self.sd_c, self.sd_f = load_weights("fern_lowres")
        else:
            gen = torch.Generator().manual_seed(int(z["init_seed"]))
            kw = dict(num_layers=self.num_layers, hidden_size=self.hidden, skip_connect_every=self.skip,
                      num_encoding_fn_xyz=self.enc_xyz[0], num_encoding_fn_dir=self.enc_dir[0],
                      include_input_xyz=self.enc_xyz[1], include_input_dir=self.enc_dir[1],
                      use_viewdirs=self.use_viewdirs, generator=gen)
            self.sd_c = O.init_flexible_nerf(**kw)
            self.sd_f = O.init_flexible_nerf(**kw) if int(z["num_fine"]) > 0 else None
        if int(z["num_fine"]) == 0:
            self.sd_f = None

    def grad_digests(self, tag):
        pre = f"gd_{tag}_"
        return {k[len(pre):]: self.z[k] for k in self.z.files if k.startswith(pre)}

    def oracle(self, dtype=torch.float32, with_grad=False):
        """Run the oracle with the recorded randoms.  Returns (outputs6, loss, grads_c, grads_f)."""
        cast = lambda t: t.to(dtype) if t is not None else None
        sd_c = {k: v.to(dtype).clone().requires_grad_(with_grad) for k, v in self.sd_c.items()}
        sd_f = {k: v.to(dtype).clone().requires_grad_(with_grad) for k, v in self.sd_f.items()} if self.sd_f else None
        rnd = {k: v.to(dtype) for k, v in self.randoms.items()}
        out = O.run_one_iter_of_nerf(self.H, self.W, self.focal, sd_c, sd_f, cast(self.ro), cast(self.rd), self.options,
                                     mode=self.mode, enc_xyz=self.enc_xyz, enc_dir=self.enc_dir, randoms=rnd)
        loss = O.nerf_loss(tuple(x.reshape(-1, 3) if (x is not None and x.shape[-1] == 3 and x.dim() == 3) else x
                                 for x in out), cast(self.target))
        gc = gf = None
        if with_grad:
            loss.backward()
            gc = {k: v.grad for k, v in sd_c.items()}
            gf = {k: v.grad for k, v in sd_f.items()} if sd_f else None
        return out, loss, gc, gf

    def aux(self, dtype=torch.float32):
        """Stage-level intermediates of the oracle for this case (single chunk, train-mode options)."""
        rays = pack_rays(self, dtype)
        sd_c = {k: v.to(dtype) for k, v in self.sd_c.items()}
        sd_f = {k: v.to(dtype) for k, v in self.sd_f.items()} if self.sd_f else None
        rnd = {k: v.to(dtype) for k, v in self.randoms.items()}
        out, aux = O.predict_and_render_radiance(rays, sd_c, sd_f, self.options, mode="train", enc_xyz=self.enc_xyz,
                                                 enc_dir=self.enc_dir if self.use_viewdirs else None, randoms=rnd,
                                                 return_aux=True)
        return rays, out, aux


def pack_rays(case: Case, dtype=torch.float32):
    """The (N, 11 | 8) ray rows of train_utils.py:143-168, through the oracle's helpers."""
    ro, rd = case.ro.to(dtype), case.rd.to(dtype)
    vd = rd / rd.norm(p=2, dim=-1).unsqueeze(-1)
    vd = vd.reshape(-1, 3)
    if case.options.dataset.no_ndc is False:
        ro, rd = O.ndc_rays(case.H, case.W, case.focal, 1.0, ro, rd)
    ro, rd = ro.reshape(-1, 3), rd.reshape(-1, 3)
    near = case.options.dataset.near * torch.ones_like(rd[..., :1])
    far = case.options.dataset.far * torch.ones_like(rd[..., :1])
    rays = torch.cat((ro, rd, near, far), -1)
    if case.use_viewdirs:
        rays = torch.cat((rays, vd), -1)
    return rays.contiguous()


def arch_of(case: Case):
    """The ops.ArchSpec of a golden case's networks."""
    from nerf_pytorch_b200 import ops

    c = case
    return ops.ArchSpec(num_layers=c.num_layers, hidden=c.hidden, skip_every=c.skip, use_viewdirs=c.use_viewdirs,
                        n_freq_xyz=c.enc_xyz[0], n_freq_dir=c.enc_dir[0], include_input_xyz=c.enc_xyz[1],
                        include_input_dir=c.enc_dir[1], log_sampling_xyz=c.enc_xyz[2], log_sampling_dir=c.enc_dir[2])


def build_models(c: Case):
    """The golden case's coarse and fine FlexibleNeRFModels (fine None if it has none) on the GPU, and its encoders."""
    import nerf_pytorch_b200 as nb

    def mk(sd):
        m = nb.FlexibleNeRFModel(num_layers=c.num_layers, hidden_size=c.hidden, skip_connect_every=c.skip,
                                 num_encoding_fn_xyz=c.enc_xyz[0], num_encoding_fn_dir=c.enc_dir[0],
                                 include_input_xyz=c.enc_xyz[1], include_input_dir=c.enc_dir[1],
                                 use_viewdirs=c.use_viewdirs)
        m.load_state_dict(sd)
        return m.cuda()

    mc = mk(c.sd_c)
    mf = mk(c.sd_f) if c.sd_f is not None else None
    epf = nb.get_embedding_function(*c.enc_xyz)
    edf = nb.get_embedding_function(*c.enc_dir) if c.use_viewdirs else None
    return mc, mf, epf, edf


# ------------------------------------------------------------------------------------------------------------------------
# the shipped low-res networks and their scenes
# ------------------------------------------------------------------------------------------------------------------------
LEGO_BOX = ((-1.5,) * 3, (1.5,) * 3)
FERN_BOX = ((-1.2, -1.2, -1.0), (1.2, 1.2, 0.98))
# (H, W, focal): lego at pose_spherical(30, -30, 4), near 2, far 6; fern forward-facing at the identity in NDC, near 0,
# far 1
LEGO_CAM = (48, 48, 66.7)
FERN_CAM = (42, 56, 45.3)


def shipped_models(kind):
    """(coarse, fine, encode_position_fn, encode_direction_fn) of the shipped low-res "lego" or "fern" networks
    (golden/weights_<kind>_lowres.npz): A0, 4 x 128 skip 4, 10 (lego) or 6 (fern) position bands and 4 direction bands,
    the models on the GPU."""
    import nerf_pytorch_b200 as nb

    l_xyz = 10 if kind == "lego" else 6
    out = []
    for sd in load_weights(f"{kind}_lowres"):
        m = nb.FlexibleNeRFModel(num_layers=4, hidden_size=128, skip_connect_every=4, num_encoding_fn_xyz=l_xyz,
                                 num_encoding_fn_dir=4)
        m.load_state_dict(sd)
        out.append(m.cuda())
    return out[0], out[1], nb.get_embedding_function(l_xyz), nb.get_embedding_function(4)


def scene_pose(kind):
    """A scene's camera pose: "spherical" is pose_spherical(30, -30, 4), "eye" the identity."""
    return O.pose_spherical(30.0, -30.0, 4.0) if kind == "spherical" else torch.eye(4)


def scene_options(kind):
    """Reference options of a deterministic render_image of the shipped scene: 64 coarse and 128 fine samples."""
    ndc = kind == "fern"
    return O.make_options(no_ndc=not ndc, near=0.0 if ndc else 2.0, far=1.0 if ndc else 6.0, num_coarse=64,
                          num_fine=128, perturb=False, radiance_field_noise_std=0.0)


def camera_rays(kind, pose=None, viewdirs=True):
    """The ray rows of the scene's camera (LEGO_CAM, FERN_CAM) at ``pose``, by default the scene's own."""
    from nerf_pytorch_b200 import ops

    if kind == "fern":
        H, W, focal = FERN_CAM
        return ops.gen_rays(torch.eye(4) if pose is None else pose, H, W, focal, None, "cuda", ndc=True, near=0.0,
                            far=1.0, use_viewdirs=viewdirs)
    H, W, focal = LEGO_CAM
    pose = O.pose_spherical(30.0, -30.0, 4.0) if pose is None else pose
    return ops.gen_rays(pose, H, W, focal, None, "cuda", ndc=False, near=2.0, far=6.0, use_viewdirs=viewdirs)


def sphere_poses(n, radius=4.0, phis=(-30.0, -45.0, -15.0), offset=7.0):
    """n poses around the lego scene: azimuth 360 i / n + offset (i mod len(phis)), elevation phis[i mod len(phis)]."""
    return torch.stack([O.pose_spherical(360.0 * i / n + offset * (i % len(phis)), phis[i % len(phis)], radius)
                        for i in range(n)])


def targets(kind, poses):
    """(fine rgb images [n, H, W, 3] of render_image of the shipped networks at ``poses``, scene_options(kind))."""
    import nerf_pytorch_b200 as nb

    mc, mf, epf, edf = shipped_models(kind)
    H, W, focal = FERN_CAM if kind == "fern" else LEGO_CAM
    opts = scene_options(kind)
    with torch.no_grad():
        imgs = torch.stack([nb.render_image(H, W, focal, p, mc, mf, opts, encode_position_fn=epf,
                                            encode_direction_fn=edf, impl=1)[3] for p in poses])
    return imgs.contiguous(), opts


# The seven pretrained low-res scenes (golden/weights_<scene>_lowres.npz: oracle/make_golden.py writes lego and fern,
# oracle/make_pretrained.py the other five).  Every network is A0 by its tensors' shapes, whatever the scene's config
# says: 4 layers, hidden 128, skip 4, 4 direction bands, 10 position bands (fern 6).  Per scene: position bands, the
# config's fine samples per ray (64 coarse everywhere), NDC, near, far, white background, noise std of training and the
# camera (H, W, focal): the Blender scenes' half-resolution 400 x 400 camera, fern's 378 x 504 forward-facing one.
PRETRAINED_SCENES = {
    "chair": (10, 64, False, 2.0, 6.0, True, 0.2, (400, 400, 555.5555155968841)),
    "drums": (10, 64, False, 2.0, 6.0, True, 0.2, (400, 400, 555.5555155968841)),
    "fern": (6, 64, True, 0.0, 1.0, False, 1.0, (378, 504, 407.5658)),
    "hotdog": (10, 128, False, 2.0, 6.0, True, 0.2, (400, 400, 555.5555155968841)),
    "lego": (10, 64, False, 2.0, 6.0, True, 0.2, (400, 400, 555.5555155968841)),
    "materials": (10, 64, False, 2.0, 6.0, True, 0.2, (400, 400, 555.5555155968841)),
    "ship": (10, 128, False, 2.0, 6.0, True, 0.2, (400, 400, 555.5555155968841)),
}
# The boxes the scenes' geometry lies in: the Blender scenes' objects inside [-1.5, 1.5]^3, fern's NDC box (FERN_BOX).
PRETRAINED_BOX = {s: (FERN_BOX if s == "fern" else LEGO_BOX) for s in PRETRAINED_SCENES}


def pretrained_arch(scene):
    """The ops.ArchSpec of a pretrained scene's networks."""
    from nerf_pytorch_b200 import ops

    return ops.ArchSpec(num_layers=4, hidden=128, skip_every=4, n_freq_xyz=PRETRAINED_SCENES[scene][0], n_freq_dir=4)


def pretrained_poses(scene, n):
    """n camera poses of a pretrained scene: for the Blender scenes a ring of pose_spherical at radius 4.03 (the
    datasets' camera distance), azimuth 360 i / n + 7 (i mod 3), elevation -30, -45, -15 in turn; for fern the identity
    and n - 1 translations in the image plane by up to 0.1 (forward-facing captures move little)."""
    if scene != "fern":
        return sphere_poses(n, radius=4.03)
    out = []
    for i in range(n):
        p = torch.eye(4)
        if i:
            a = 2 * math.pi * (i - 1) / max(n - 1, 1)
            p[0, 3], p[1, 3] = 0.1 * math.cos(a), 0.1 * math.sin(a)
        out.append(p)
    return torch.stack(out)


def pretrained_options(scene, perturb=True):
    """Reference options of a pretrained scene's training step (perturbed, with its noise) or, perturb False, of its
    deterministic render."""
    _, nf, ndc, near, far, white, noise, _ = PRETRAINED_SCENES[scene]
    return O.make_options(no_ndc=not ndc, near=near, far=far, num_coarse=64, num_fine=nf, perturb=perturb,
                          radiance_field_noise_std=noise if perturb else 0.0, white_background=white)


def psnr32(a, b):
    """PSNR (dB) from the fp32 mean squared error, at most 120 dB (the error clamped at 1e-12)."""
    return -10.0 * math.log10(max(torch.mean((a - b) ** 2).item(), 1e-12))


def psnr64(a, b):
    """PSNR (dB) from the fp64 mean squared error; inf when a and b are equal."""
    mse = (a.double() - b.double()).pow(2).mean().item()
    return math.inf if mse == 0 else -10.0 * math.log10(mse)


def ws_view(ws, layout, name, n, s, cols):
    """The fp32 section ``name`` of a render workspace (ops.render_workspace_layout) as [n, s, cols], or [n, s] for one
    column."""
    off = layout[name] // 4
    t = ws.view(torch.float32)[off: off + n * s * cols]
    return t.view(n, s, cols) if cols > 1 else t.view(n, s)


def composite64(raw, z, dirs, noise_std=0.0, white_background=False, noise=None, raw64=None):
    """fp64 O.volume_render_radiance_field of the fp32 samples raw [.., S, 4], z [.., S], dirs [.., 3] with unit normals
    noise [.., S]: (rgb, disp, acc, weights, depth), differentiable with respect to raw64 (default raw.double()).

    The ReLU gate of sigma and the last sample's sigma are taken from the fp32 pre-activation
    fp32(raw + fp32(noise * std)) that the kernels and the reference round: the gate is the function's one
    discontinuity, and the last sample's alpha, 1 - exp(-sigma * 1e10 |d|), turns a rounding of a tiny sigma into an
    O(1) change.  Every other sigma is raw + noise * std in fp64.  disp is NaN where acc is 0, as in the reference, with
    a gradient that stays finite on the other rays.  Plain tensor ops: it runs on the device of its inputs."""
    if raw64 is None:
        raw64 = raw.double()
    pre32, pre64 = raw[..., 3], raw64[..., 3]
    if noise_std > 0.0:
        std32 = torch.tensor(noise_std, dtype=torch.float32, device=raw.device)
        nz32 = noise.float() * std32
        pre32 = pre32 + nz32
        pre64 = pre64 + noise.double() * float(std32)
    gate = pre32 > 0
    last = pre32[..., -1:].double() + (pre64[..., -1:] - pre64[..., -1:].detach())
    sigma = torch.where(gate, torch.cat((pre64[..., :-1], last), -1), 0.0)
    z64 = z.double()
    dists = torch.cat((z64[..., 1:] - z64[..., :-1], torch.full_like(z64[..., :1], 1e10)), -1)
    dists = dists * dirs.double().norm(p=2, dim=-1)[..., None]
    alpha = 1.0 - torch.exp(-sigma * dists)
    weights = alpha * O.cumprod_exclusive(1.0 - alpha + 1e-10)
    rgb = (weights[..., None] * torch.sigmoid(raw64[..., :3])).sum(-2)
    depth = (weights * z64).sum(-1)
    acc = weights.sum(-1)
    some = acc > 0
    disp = 1.0 / torch.clamp_min(depth / torch.where(some, acc, 1.0), 1e-10)
    disp = torch.where(some, disp, float("nan"))
    if white_background:
        rgb = rgb + (1.0 - acc[..., None])
    return rgb, disp, acc, weights, depth


def composite_grad64(raw, z, dirs, g, noise_std=0.0, white_background=False, noise=None):
    """fp64 d(sum(outputs * g)) / d(raw) of composite64: g [n][8] weighs rgb, disp (rays where g is 0 excluded) and acc,
    the render entry points' upstream layout.  raw: fp32 [n][S][4], or (fp32, fp64) to differentiate the fp64 values
    with the fp32 ones' gates."""
    r32, r64 = raw if isinstance(raw, tuple) else (raw, raw.double())
    r64 = r64.detach().clone().requires_grad_(True)
    rgb, disp, acc, _, _ = composite64(r32, z, dirs, noise_std, white_background, noise, raw64=r64)
    g = g.double()
    disp = torch.where(g[:, 3] != 0, disp, 0.0)
    loss = (rgb * g[:, :3]).sum() + (disp * g[:, 3]).sum() + (acc * g[:, 4]).sum()
    return torch.autograd.grad(loss, r64)[0]


def transmittance64(raw, z, rays, noise, std):
    """fp64 exclusive transmittance [n, S + 1] of fp32 raw [n, S, 4] at depths z [n, S] along rays [n, >= 6]:
    T[:, p] = prod over samples < p of 1 - alpha + 1e-10, with the sigma gate and the last sample's sigma taken from the
    fp32 pre-activation as the compositing rounds them (noise [n, S] times std, or std 0 and noise None)."""
    pre32, pre64 = raw[..., 3], raw[..., 3].double()
    if std > 0:
        std32 = torch.tensor(std, dtype=torch.float32, device=raw.device)
        pre32 = pre32 + noise * std32
        pre64 = pre64 + noise.double() * float(std32)
    sigma = torch.where(pre32 > 0, torch.cat((pre64[:, :-1], pre32[:, -1:].double()), 1), 0.0)
    z64 = z.double()
    dists = torch.cat((z64[:, 1:] - z64[:, :-1], torch.full_like(z64[:, :1], 1e10)), 1)
    dists = dists * rays[:, 3:6].double().norm(dim=1, keepdim=True)
    q = torch.exp(-sigma * dists) + 1e-10
    return torch.cat((torch.ones_like(q[:, :1]), torch.cumprod(q, 1)), 1)


def skipped_samples(grid, rays, z):
    """bool [n, S]: the samples at depths z [n, S] of rays [n, >= 6] that an occupancy grid skips, the fp32 points
    o + d z inside its box in a clear cell (OccupancyGrid.cell_of); points outside the box are always evaluated."""
    pts = rays[:, None, :3] + rays[:, None, 3:6] * z[..., None]
    cell = grid.cell_of(pts)
    occ = grid.occupancy().reshape(-1)
    return (cell >= 0) & ~occ[cell.clamp_min(0)]


def compaction_reference(grid, rays, z):
    """Torch restatement of one pass's sample compaction (nerfb200_grid_compact): (keep [n, S], map rows, blocks).  The
    kept points of each group of 10 rays, in (ray, sample) order, fill 64-row blocks from the group's first block; a
    group's last block is padded with -1; each block is (first ray, last ray) of its rows."""
    n, s = z.shape
    keep = ~skipped_samples(grid, rays, z)
    rows, blocks = [], []
    for g0 in range(0, n, 10):
        pts = (torch.nonzero(keep[g0:g0 + 10].reshape(-1)).reshape(-1) + g0 * s).tolist()
        for b0 in range(0, len(pts), 64):
            chunk = pts[b0:b0 + 64]
            blocks.append((chunk[0] // s, chunk[-1] // s))
            rows += chunk + [-1] * (64 - len(chunk))
    return keep, rows, blocks


# ------------------------------------------------------------------------------------------------------------------------
# baked fields (include/nerfb200.h "baked fields")
# ------------------------------------------------------------------------------------------------------------------------
# coefficients against the fp64 projection of the kernel's own logits: |c - c64| <= COEF_REL * max |logit| of the point.
# The fp32 fmaf chain over 64 terms; measured on an H100 80GB HBM3 at 700 W: at most 1.5e-6 (lego, fern), 2.0e-6 over the
# architecture table (test_bake_sweep_gpu, 8x256 "scaled").
COEF_REL = 4e-6
# the renderer against its fp64 restatement (absolute on rgb / acc, relative to far on depth); measured on an H100 80GB
# HBM3 at 700 W: rgb 1.1e-6, acc 1.6e-6, depth 1.1e-6 far on camera rays (test_bake_gpu); rgb 4.8e-6, acc 5.4e-6,
# depth 1.0e-6 far on the edge rays of test_bake_sweep_gpu (rays through two box corners, ~440 samples)
OUT_ABS = 1e-5


def net_at(arch, blob, pts, direction):
    """raw (P, 4) of mlp_fwd_pts(impl=1) at pts (P, 3), every point with `direction` (None without view directions)."""
    from nerf_pytorch_b200 import ops

    P = pts.shape[0]
    rows = -(-P // 64)
    pad = torch.cat([pts, pts[-1:].expand(rows * 64 - P, 3)]).contiguous()
    dirs = None if direction is None else direction.view(1, 3).expand(rows, 3).contiguous()
    return ops.mlp_fwd_pts(arch, blob, pad.view(rows, 64, 3), dirs, impl=1).view(-1, 4)[:P]


def baked_render64(field, rays, white):
    """fp64 restatement of the header's rendering of a baked field (nb.BakedField), gathering from its values; the
    interval, sample depths, points and cells are formed in fp32 as the header states.  (rgb, acc, depth, disp) per ray.
    The slab terms go through fmin / fmax as the kernel's fminf / fmaxf (a NaN term drops out); an axis with d = +-0
    leaves the interval as it is when lo <= o < hi and empties the ray otherwise.  A ray is live when t_a < t_b and dt is
    positive, finite and (t_b - t_a) / dt < 2^24."""
    f32 = torch.float32
    dev = rays.device
    lo = torch.tensor(field.bounds[0], dtype=f32, device=dev)
    hi = torch.tensor(field.bounds[1], dtype=f32, device=dev)
    res = torch.tensor(field.resolution, device=dev)
    o, d = rays[:, :3], rays[:, 3:6]
    t0, t1 = (lo - o) / d, (hi - o) / d
    flat = d == 0
    tmin = torch.where(flat, -math.inf, torch.fmin(t0, t1).nan_to_num(nan=-math.inf))
    tmax = torch.where(flat, math.inf, torch.fmax(t0, t1).nan_to_num(nan=math.inf))
    outside = (flat & ~((o >= lo) & (o < hi))).any(-1)
    ta = torch.fmax(rays[:, 6], tmin.amax(-1))
    tb = torch.where(outside, -math.inf, torch.fmin(rays[:, 7], tmax.amin(-1)))
    h = ((hi - lo) / res.to(f32)).min()
    dn = torch.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    dt = (torch.tensor(0.5, dtype=f32, device=dev) * h) / dn
    live = (ta < tb) & (dt > 0) & (dt < math.inf) & ((tb - ta) / dt < 16777216.0)
    K = int(torch.where(live, (tb - ta) / dt, 0.0).max().item()) + 2
    k = torch.arange(K, device=dev, dtype=f32) + 0.5
    t = ta[:, None] + k[None] * dt[:, None]
    valid = (t < tb[:, None]) & live[:, None]
    t = torch.where(valid, t, 0.0)
    x = o[:, None] + d[:, None] * t[..., None]
    scale = res.to(f32) / (hi - lo)
    tc = (x - lo) * scale
    inside = ((tc >= 0) & (tc < res.to(f32))).all(-1) & valid
    i = torch.where(inside[..., None], tc, torch.zeros_like(tc)).to(torch.int64).clamp_max(res - 1)
    fr = (tc - i.to(f32)).double()
    nb_ = (res + 7) // 8
    b = i // 8
    slot = field.brick_map.long()[((b[..., 2] * nb_[1] + b[..., 1]) * nb_[0] + b[..., 0]).clamp(0, field.brick_map.numel() - 1)]
    hit = inside & (slot >= 0)
    l = i % 8
    vals = field.values.double() if field.n_active else torch.zeros(1, 729, 32, dtype=torch.float64, device=dev)
    v = torch.zeros(*t.shape, 28, dtype=torch.float64, device=dev)
    for c in range(8):
        off = torch.tensor([c & 1, c >> 1 & 1, c >> 2], device=dev)
        lc = l + off
        w = torch.where(off.bool(), fr, 1 - fr).prod(-1)
        idx = (lc[..., 2] * 9 + lc[..., 1]) * 9 + lc[..., 0]
        w = torch.where(hit, w, 0.0)  # a miss's fractions may be NaN (a NaN origin)
        v += w[..., None] * vals[slot.clamp_min(0), idx][..., :28]
    sigma = torch.where(hit, v[..., 0], torch.zeros_like(v[..., 0]))
    coef = v[..., 1:].view(*t.shape, 3, 9)
    if field.use_viewdirs:
        vd = rays[:, 8:11].double()
        X, Y, Z = vd[:, 0], vd[:, 1], vd[:, 2]
        Ysh = torch.stack([torch.full_like(X, 0.28209479177387814), -0.4886025119029199 * Y, 0.4886025119029199 * Z,
                           -0.4886025119029199 * X, 1.0925484305920792 * X * Y, -1.0925484305920792 * Y * Z,
                           0.31539156525252005 * (2 * Z * Z - X * X - Y * Y), -1.0925484305920792 * X * Z,
                           0.5462742152960396 * (X * X - Y * Y)], -1)
        s = (coef * Ysh[:, None, None, :]).sum(-1)
    else:
        s = coef[..., 0] * 0.28209479177387814
    rgb = torch.where(hit[..., None], torch.sigmoid(s), torch.zeros_like(s))
    alpha = 1 - torch.exp(-torch.relu(sigma) * (dt.double() * dn.double())[:, None])
    alpha = torch.where(valid, alpha, torch.zeros_like(alpha))
    q = 1 - alpha + 1e-10
    T = torch.cat([torch.ones_like(q[:, :1]), torch.cumprod(q, -1)[:, :-1]], -1)
    w = alpha * T
    acc = w.sum(-1)
    depth = (w * t.double()).sum(-1)
    out_rgb = (w[..., None] * rgb).sum(1) + ((1 - acc)[:, None] if white else 0)
    return out_rgb, acc, depth, 1 / torch.clamp(depth / acc, min=1e-10)


def bake_scene(kind, res, grid_res=None, grid_from="fine"):
    """nb.bake of a scene's network over its box at ``res``.  "lego" and "fern" bake the shipped fine network (LEGO_BOX,
    FERN_BOX); "noview" a coarse-only network without view directions at torch's init under seed 7, over [-1, 1]^3.
    Bricks: every one with grid_res None, else those of OccupancyGrid.from_models at grid_res over the fine network
    (grid_from "fine") or over the coarse and fine networks ("both")."""
    import nerf_pytorch_b200 as nb

    if kind == "noview":
        torch.manual_seed(7)
        mc, mf = None, nb.FlexibleNeRFModel(num_layers=4, hidden_size=128, skip_connect_every=4, num_encoding_fn_xyz=10,
                                            use_viewdirs=False).cuda()
        epf, edf, box = nb.get_embedding_function(10), None, ((-1.0,) * 3, (1.0,) * 3)
    else:
        mc, mf, epf, edf = shipped_models(kind)
        box = FERN_BOX if kind == "fern" else LEGO_BOX
    nets = {"fine": [mf], "both": [mc, mf]}[grid_from]
    grid = nb.OccupancyGrid.full(box, 8) if grid_res is None else \
        nb.OccupancyGrid.from_models(nets, epf, box, grid_res, encode_direction_fn=edf)
    return nb.bake(mf, epf, edf, bounds=box, resolution=res, grid=grid)


def lattice_index(field):
    """int64 [n_active, 729]: the linear lattice index (x fastest over res + 1 points per axis) each stored value holds."""
    res = torch.tensor(field.resolution, device="cuda")
    nb_ = (res + 7) // 8
    br = field.bricks.long()
    b = torch.stack([br % nb_[0], br // nb_[0] % nb_[1], br // (nb_[0] * nb_[1])], -1)  # [n, 3]
    p = torch.arange(729, device="cuda")
    l = torch.stack([p % 9, p // 9 % 9, p // 81], -1)  # [729, 3]
    q = torch.minimum(b[:, None] * 8 + l[None], res)
    return (q[..., 2] * (res[1] + 1) + q[..., 1]) * (res[0] + 1) + q[..., 0]


def copies_bit_equal(x, idx):
    """Every copy of every lattice point (idx: lattice_index) holds the same bits in all 32 channels."""
    flat = idx.reshape(-1)
    bits = x.reshape(-1, 32).contiguous().view(torch.int32)
    first = torch.full((int(flat.max()) + 1,), -1, dtype=torch.int64, device=x.device)
    first.scatter_reduce_(0, flat, torch.arange(flat.numel(), device=x.device), reduce="amin", include_self=False)
    return bool((bits == bits[first[flat]]).all())


def synthetic_field(res, *, viewdirs=True, active=1.0, sigma=(-4.0, 8.0), seed=0, box=((-1.0,) * 3, (1.0,) * 3)):
    """A field with random values per lattice point (every copy of a point the same bits), on a random subset of
    bricks: sigma_raw uniform in ``sigma``, coefficients normal with std 0.7 (coefficients 1 .. 8 zero without view
    directions, as a bake writes them)."""
    import nerf_pytorch_b200 as nb

    g = torch.Generator(device="cuda").manual_seed(seed)
    nb_ = [-(-r // 8) for r in res]
    keep = torch.rand(nb_[0] * nb_[1] * nb_[2], generator=g, device="cuda") < active
    keep[0] = True
    brick_map = torch.where(keep, torch.cumsum(keep.int(), 0) - 1, -1).int()
    bricks = torch.nonzero(keep).reshape(-1).int()
    pts = (res[0] + 1) * (res[1] + 1) * (res[2] + 1)
    dense = torch.zeros(pts, 32, device="cuda")
    dense[:, 0] = sigma[0] + (sigma[1] - sigma[0]) * torch.rand(pts, generator=g, device="cuda")
    dense[:, 1:28] = 0.7 * torch.randn(pts, 27, generator=g, device="cuda")
    if not viewdirs:
        coef = dense[:, 1:28].reshape(pts, 3, 9).clone()
        coef[:, :, 1:] = 0
        dense[:, 1:28] = coef.reshape(pts, 27)
    f = nb.BakedField(box, res, brick_map, bricks, torch.empty(bricks.numel(), 729, 32, device="cuda"), viewdirs)
    f.values = dense[lattice_index(f)].contiguous()
    return f


def ray_rows(o, d, viewdirs=True, near=0.0, far=6.0):
    """Ray rows (o, d, near, far[, unit d]) on the GPU; near and far are numbers or per-ray tensors."""
    n = o.shape[0]
    near = torch.full((n, 1), near, device="cuda") if not torch.is_tensor(near) else near.view(n, 1)
    far = torch.full((n, 1), far, device="cuda") if not torch.is_tensor(far) else far.view(n, 1)
    cols = [o, d, near, far]
    if viewdirs:
        cols.append(d / d.norm(dim=1, keepdim=True))
    return torch.cat(cols, 1).contiguous()


def random_rays(n, seed, viewdirs=True, lo=-1.0, hi=1.0, misses=False):
    """Rays from a sphere of radius 3 towards random points of the box [lo, hi]^3, near 0, far 6; with ``misses`` every
    7th turned away from the box."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    o = torch.randn(n, 3, generator=g, device="cuda")
    o = 3.0 * o / o.norm(dim=1, keepdim=True)
    d = lo + (hi - lo) * torch.rand(n, 3, generator=g, device="cuda") - o
    if misses:
        d[::7] = -d[::7]
    return ray_rows(o, d, viewdirs)


def edge_rays(field, viewdirs=True):
    """Axis-parallel rays in brick-face planes (and on brick edges), and diagonals through brick corners."""
    lo = torch.tensor(field.bounds[0], device="cuda")
    hi = torch.tensor(field.bounds[1], device="cuda")
    res = torch.tensor(field.resolution, device="cuda", dtype=torch.float32)
    h = (hi - lo) / res
    o, d = [], []
    for a in range(3):  # along axis a, in the plane of the first brick face of axis b, at several offsets on axis c
        b, c = (a + 1) % 3, (a + 2) % 3
        for k in range(6):
            p = lo + (hi - lo) * 0.37
            p[b] = lo[b] + 8 * h[b] if res[b] > 8 else lo[b] + h[b]
            p[c] = lo[c] + (k / 5.0) * (hi[c] - lo[c]) * 0.99
            if k == 5:
                p[c] = lo[c] + 8 * h[c] if res[c] > 8 else lo[c]  # a brick edge
            p[a] = lo[a] - 1.0
            dd = torch.zeros(3, device="cuda")
            dd[a] = 1.0
            o.append(p.clone())
            d.append(dd)
    corner = lo + 8 * h * (res > 8)  # a brick corner point (or the box's lower corner)
    for s in ([1, 1, 1], [1, -1, 1], [-1, 1, 1], [1, 1, -1]):
        dd = torch.tensor(s, device="cuda", dtype=torch.float32)
        o.append(corner - 2.0 * dd)
        d.append(dd)
    return ray_rows(torch.stack(o), torch.stack(d), viewdirs)


def heldout_psnr(field, poses, imgs):
    """Mean psnr32 of the baked field's renders at lego-camera ``poses`` against ``imgs``."""
    import nerf_pytorch_b200 as nb

    with torch.no_grad():
        return sum(psnr32(nb.render_baked_rays(field, camera_rays("lego", p))[0], im.reshape(-1, 3))
                   for p, im in zip(poses, imgs)) / len(poses)


def axis_bricks(res, nb, c=None):
    """bool [res + 1, nb]: the bricks of lattice index q's copy list along one axis (include/nerfb200.h "baked fields:
    gradients and fine-tuning", Tie): {nb - 1} at q = res, {q / 8 - 1, q / 8} at a positive multiple of 8 below res, {q
    // 8} otherwise.  With ``c`` set (the edge axis) instead the one brick q // 8 for q < res and none at q = res."""
    q = np.arange(res + 1)
    m = np.zeros((res + 1, nb), dtype=bool)
    if c is not None:
        m[q[:-1], q[:-1] // 8] = True
        return m
    inner = q < res
    m[q[inner], q[inner] // 8] = True
    face = inner & (q > 0) & (q % 8 == 0)
    m[q[face], q[face] // 8 - 1] = True
    m[res, nb - 1] = True
    return m


def baked_lattice(res, active):
    """The regularisers' lattice (include/nerfb200.h "baked fields: regularisers") restated in numpy: (points, edges)
    with points bool [res_2 + 1, res_1 + 1, res_0 + 1] (the lattice points with a copy in an active brick) and edges a
    list over the axes c = 0, 1, 2 (x, y, z) of bool arrays of that shape, edges[c][q] for the edge (q, q + e_c): brick q_c
    // 8 along c and any brick of q's copy list along the other axes.  ``active`` is bool [nb_2, nb_1, nb_0]."""
    res = tuple(int(r) for r in res)
    nb = [-(-r // 8) for r in res]
    a = np.asarray(active).astype(np.int64)

    def spread(mx, my, mz):  # [qz, qy, qx] = any over bricks of mz[qz, bz] my[qy, by] mx[qx, bx] active[bz, by, bx]
        t = np.tensordot(a, mx.astype(np.int64), axes=([2], [1]))       # [bz, by, qx]
        t = np.tensordot(t, my.astype(np.int64), axes=([1], [1]))       # [bz, qx, qy]
        t = np.tensordot(t, mz.astype(np.int64), axes=([0], [1]))       # [qx, qy, qz]
        return t.transpose(2, 1, 0) > 0

    copies = [axis_bricks(res[c], nb[c]) for c in range(3)]
    points = spread(*copies)
    edges = []
    for c in range(3):
        m = list(copies)
        m[c] = axis_bricks(res[c], nb[c], c)
        edges.append(spread(*m))
    return points, edges


def bits_equal(a, b):
    """Same shape and the same bits (4-byte elements); two Nones are equal."""
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def err_stats(a: torch.Tensor, b: torch.Tensor):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    both_nan = torch.isnan(a) & torch.isnan(b)
    d = (a - b).abs()
    d[both_nan] = 0
    denom = b.abs().clamp_min(1e-30)
    return dict(max_abs=d.max().item(), max_rel=(d / denom)[b.abs() > 1e-3].max().item() if (b.abs() > 1e-3).any() else 0.0,
                nan_mismatch=int((torch.isnan(a) != torch.isnan(b)).sum()))


def frac_close(a, b, rtol, atol):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    ok = torch.isclose(a, b, rtol=rtol, atol=atol, equal_nan=True)
    return ok.double().mean().item()
