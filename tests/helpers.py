"""Shared test plumbing: golden-case loading, oracle drivers, error metrics.  (tests/ may use oracle/.)"""
from __future__ import annotations

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
