"""CPU oracle for the NeRF per-ray hot path  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A plain torch-CPU (fp32 or fp64) restatement of the reference algorithm
(krrish94/nerf-pytorch @ a14357d) behind ``run_one_iter_of_nerf`` /
``predict_and_render_radiance``.  Only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs may import this module; the
product package (``nerf_pytorch_b200``) never does.

Pinning status: the reference ships NO golden vectors or known-answer tests for this path
(SURVEY.md section 4), so the oracle is pinned against outputs of the reference itself:
``oracle/make_golden.py`` imports the unmodified reference from a checkout of it (two
``sys.modules`` shims, see that script), runs it on seeded inputs with the shipped
``pretrained/lego-lowres`` weights, asserts THIS restatement reproduces every output
bit-for-bit (same ATen ops in the same order, same RNG draw order), and commits the vectors
under ``tests/golden/``.  ``tests/test_oracle_golden.py`` re-checks the oracle against those
vectors on every run.

Every function cites the reference file:line (paths relative to the reference repository) it follows.
Differences from the reference are limited to:
  * randoms can be injected (``randoms=dict(t_rand=, noise_c=, u=, noise_f=)``); when absent
    they are drawn from the torch global RNG in the reference's order, so that a shared seed
    reproduces the reference exactly;
  * the MLP is functional (takes a ``state_dict``) and uses the *allocated* layer widths to
    decide where the skip concat happens, which repairs the ``self.linear_layers`` typo at
    nerf/models.py:243 without changing behaviour for any architecture the reference can
    actually run (SURVEY.md section 0.2);
  * optional extra outputs (weights, depth, z_vals, sample indices) for stage-level tests.
"""
from __future__ import annotations

import math
from types import SimpleNamespace
from typing import Dict, Optional

import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------------------
# Small helpers
# --------------------------------------------------------------------------------------
def make_options(
    *,
    use_viewdirs=True,
    no_ndc=True,
    near=2.0,
    far=6.0,
    chunksize=131072,
    num_coarse=64,
    num_fine=128,
    perturb=True,
    lindisp=False,
    white_background=False,
    radiance_field_noise_std=0.2,
    validation: Optional[dict] = None,
):
    """Build the attribute tree the reference reads (config/lego.yml:60-80 key names)."""
    train = SimpleNamespace(
        chunksize=chunksize,
        num_coarse=num_coarse,
        num_fine=num_fine,
        perturb=perturb,
        lindisp=lindisp,
        white_background=white_background,
        radiance_field_noise_std=radiance_field_noise_std,
    )
    val = SimpleNamespace(**{**vars(train), **(validation or {})})
    return SimpleNamespace(
        nerf=SimpleNamespace(use_viewdirs=use_viewdirs, train=train, validation=val),
        dataset=SimpleNamespace(no_ndc=no_ndc, near=near, far=far),
    )


def get_minibatches(inputs: torch.Tensor, chunksize: int = 1024 * 8):
    """nerf/nerf_helpers.py:20-25."""
    return [inputs[i : i + chunksize] for i in range(0, inputs.shape[0], chunksize)]


def meshgrid_xy(t1: torch.Tensor, t2: torch.Tensor):
    """nerf/nerf_helpers.py:28-40 (ij meshgrid, transposed)."""
    ii, jj = torch.meshgrid(t1, t2, indexing="ij")
    return ii.transpose(-1, -2), jj.transpose(-1, -2)


def get_ray_bundle(height: int, width: int, focal_length: float, tform_cam2world: torch.Tensor):
    """nerf/nerf_helpers.py:67-110.  Returns (H, W, 3) origins and (un-normalised) directions."""
    ii, jj = meshgrid_xy(
        torch.arange(width, dtype=tform_cam2world.dtype),
        torch.arange(height, dtype=tform_cam2world.dtype),
    )
    directions = torch.stack(
        [
            (ii - width * 0.5) / focal_length,
            -(jj - height * 0.5) / focal_length,
            -torch.ones_like(ii),
        ],
        dim=-1,
    )
    ray_directions = torch.sum(directions[..., None, :] * tform_cam2world[:3, :3], dim=-1)
    ray_origins = tform_cam2world[:3, -1].expand(ray_directions.shape)
    return ray_origins, ray_directions


def pose_spherical(theta: float, phi: float, radius: float) -> torch.Tensor:
    """nerf/load_blender.py:8-37 (numpy there; fp32 here as at load_blender.py:36-37 callers)."""
    import numpy as np

    t = np.eye(4, dtype=np.float32)
    t[2, 3] = radius
    p = phi / 180.0 * np.pi
    rp = np.eye(4, dtype=np.float32)
    rp[1, 1] = rp[2, 2] = np.cos(p)
    rp[1, 2] = -np.sin(p)
    rp[2, 1] = -rp[1, 2]
    th = theta / 180.0 * np.pi
    rt = np.eye(4, dtype=np.float32)
    rt[0, 0] = rt[2, 2] = np.cos(th)
    rt[0, 2] = -np.sin(th)
    rt[2, 0] = -rt[0, 2]
    c2w = rp @ t
    c2w = rt @ c2w
    c2w = np.array([[-1, 0, 0, 0], [0, 0, 1, 0], [0, 1, 0, 0], [0, 0, 0, 1]]) @ c2w
    return torch.from_numpy(c2w.astype(np.float32))


def ndc_rays(H, W, focal, near, rays_o, rays_d):
    """nerf/nerf_helpers.py:170-197."""
    t = -(near + rays_o[..., 2]) / rays_d[..., 2]
    rays_o = rays_o + t[..., None] * rays_d
    o0 = -1.0 / (W / (2.0 * focal)) * rays_o[..., 0] / rays_o[..., 2]
    o1 = -1.0 / (H / (2.0 * focal)) * rays_o[..., 1] / rays_o[..., 2]
    o2 = 1.0 + 2.0 * near / rays_o[..., 2]
    d0 = -1.0 / (W / (2.0 * focal)) * (rays_d[..., 0] / rays_d[..., 2] - rays_o[..., 0] / rays_o[..., 2])
    d1 = -1.0 / (H / (2.0 * focal)) * (rays_d[..., 1] / rays_d[..., 2] - rays_o[..., 1] / rays_o[..., 2])
    d2 = -2.0 * near / rays_o[..., 2]
    return torch.stack([o0, o1, o2], -1), torch.stack([d0, d1, d2], -1)


# --------------------------------------------------------------------------------------
# Encoding  (nerf/nerf_helpers.py:113-157)
# --------------------------------------------------------------------------------------
def positional_encoding(tensor, num_encoding_functions=6, include_input=True, log_sampling=True):
    encoding = [tensor] if include_input else []
    if log_sampling:
        frequency_bands = 2.0 ** torch.linspace(
            0.0, num_encoding_functions - 1, num_encoding_functions, dtype=tensor.dtype
        )
    else:
        frequency_bands = torch.linspace(
            2.0 ** 0.0, 2.0 ** (num_encoding_functions - 1), num_encoding_functions, dtype=tensor.dtype
        )
    for freq in frequency_bands:
        for func in [torch.sin, torch.cos]:
            encoding.append(func(tensor * freq))
    if len(encoding) == 1:
        return encoding[0]
    return torch.cat(encoding, dim=-1)


# --------------------------------------------------------------------------------------
# MLP  (nerf/models.py:185-256, FlexibleNeRFModel)
# --------------------------------------------------------------------------------------
def arch_from_state_dict(sd: Dict[str, torch.Tensor], dim_xyz: int, dim_dir: int) -> dict:
    """Recover (num_layers, hidden, wide-layer set) from the allocated shapes (models.py:207-230)."""
    hidden = sd["layer1.weight"].shape[0]
    n_xyz = len([k for k in sd if k.startswith("layers_xyz.") and k.endswith(".weight")])
    wide = [i for i in range(n_xyz) if sd[f"layers_xyz.{i}.weight"].shape[1] == hidden + dim_xyz]
    return dict(num_layers=n_xyz + 1, hidden=hidden, wide=wide, use_viewdirs=("fc_rgb.weight" in sd))


def flexible_nerf_forward(sd: Dict[str, torch.Tensor], x: torch.Tensor, dim_xyz: int, return_acts=False):
    """Functional FlexibleNeRFModel.forward (nerf/models.py:233-256).

    The skip concat ``cat((x, xyz))`` (models.py:245, hidden first) happens exactly for the
    layers ``__init__`` allocated wide (models.py:210-215) -- see module docstring.
    """
    use_viewdirs = "fc_rgb.weight" in sd
    hidden = sd["layer1.weight"].shape[0]
    xyz = x[..., :dim_xyz]
    view = x[..., dim_xyz:] if use_viewdirs else None
    acts = {}
    h = F.linear(xyz, sd["layer1.weight"], sd["layer1.bias"])  # models.py:238 (no activation)
    acts["h0"] = h
    i = 0
    while f"layers_xyz.{i}.weight" in sd:
        w = sd[f"layers_xyz.{i}.weight"]
        if w.shape[1] == hidden + dim_xyz:
            h = torch.cat((h, xyz), dim=-1)  # models.py:245
        h = F.relu(F.linear(h, w, sd[f"layers_xyz.{i}.bias"]))  # models.py:246
        acts[f"h{i + 1}"] = h
        i += 1
    if use_viewdirs:
        feat = F.relu(F.linear(h, sd["fc_feat.weight"], sd["fc_feat.bias"]))  # :248
        alpha = F.linear(h, sd["fc_alpha.weight"], sd["fc_alpha.bias"])  # :249
        d = torch.cat((feat, view), dim=-1)  # :250
        d = F.relu(F.linear(d, sd["layers_dir.0.weight"], sd["layers_dir.0.bias"]))  # :251-252
        rgb = F.linear(d, sd["fc_rgb.weight"], sd["fc_rgb.bias"])  # :253
        out = torch.cat((rgb, alpha), dim=-1)  # :254
        acts["feat"], acts["d"] = feat, d
    else:
        out = F.linear(h, sd["fc_out.weight"], sd["fc_out.bias"])  # :256
    return (out, acts) if return_acts else out


def init_flexible_nerf(
    num_layers=4,
    hidden_size=128,
    skip_connect_every=4,
    num_encoding_fn_xyz=6,
    num_encoding_fn_dir=4,
    include_input_xyz=True,
    include_input_dir=True,
    use_viewdirs=True,
    generator: Optional[torch.Generator] = None,
) -> Dict[str, torch.Tensor]:
    """State dict with the shapes ``FlexibleNeRFModel.__init__`` allocates (models.py:186-231) and
    ``nn.Linear``'s default init (kaiming_uniform(a=sqrt(5)) == U(+-1/sqrt(fan_in)) for W and b)."""
    dim_xyz = (3 if include_input_xyz else 0) + 2 * 3 * num_encoding_fn_xyz
    dim_dir = (3 if include_input_dir else 0) + 2 * 3 * num_encoding_fn_dir
    if not use_viewdirs:
        dim_dir = 0
    sd: Dict[str, torch.Tensor] = {}

    def lin(name, fin, fout):
        bound = 1.0 / math.sqrt(fin)
        sd[name + ".weight"] = (torch.rand(fout, fin, generator=generator) * 2 - 1) * bound
        sd[name + ".bias"] = (torch.rand(fout, generator=generator) * 2 - 1) * bound

    lin("layer1", dim_xyz, hidden_size)
    for i in range(num_layers - 1):
        if i % skip_connect_every == 0 and i > 0 and i != num_layers - 1:  # models.py:210
            lin(f"layers_xyz.{i}", dim_xyz + hidden_size, hidden_size)
        else:
            lin(f"layers_xyz.{i}", hidden_size, hidden_size)
    if use_viewdirs:
        lin("layers_dir.0", dim_dir + hidden_size, hidden_size // 2)
        lin("fc_alpha", hidden_size, 1)
        lin("fc_rgb", hidden_size // 2, 3)
        lin("fc_feat", hidden_size, hidden_size)
    else:
        lin("fc_out", hidden_size, 4)
    return sd


# --------------------------------------------------------------------------------------
# Volume rendering  (nerf/volume_rendering_utils.py:6-53, nerf/nerf_helpers.py:43-64)
# --------------------------------------------------------------------------------------
def cumprod_exclusive(tensor: torch.Tensor) -> torch.Tensor:
    cumprod = torch.cumprod(tensor, -1)
    cumprod = torch.roll(cumprod, 1, -1)
    cumprod[..., 0] = 1.0
    return cumprod


def volume_render_radiance_field(
    radiance_field,
    depth_values,
    ray_directions,
    radiance_field_noise_std=0.0,
    white_background=False,
    noise: Optional[torch.Tensor] = None,
):
    """``noise`` (optional) is the *unit* normal draw; the reference multiplies it by the std
    (volume_rendering_utils.py:29-37).  When None and std > 0 it is drawn here, like there."""
    one_e_10 = torch.tensor([1e10], dtype=ray_directions.dtype)
    dists = torch.cat(
        (depth_values[..., 1:] - depth_values[..., :-1], one_e_10.expand(depth_values[..., :1].shape)),
        dim=-1,
    )
    dists = dists * ray_directions[..., None, :].norm(p=2, dim=-1)
    rgb = torch.sigmoid(radiance_field[..., :3])
    nz = 0.0
    if radiance_field_noise_std > 0.0:
        if noise is None:
            noise = torch.randn(radiance_field[..., 3].shape, dtype=radiance_field.dtype)
        nz = noise * radiance_field_noise_std
    sigma_a = F.relu(radiance_field[..., 3] + nz)
    alpha = 1.0 - torch.exp(-sigma_a * dists)
    weights = alpha * cumprod_exclusive(1.0 - alpha + 1e-10)
    rgb_map = (weights[..., None] * rgb).sum(dim=-2)
    depth_map = (weights * depth_values).sum(dim=-1)
    acc_map = weights.sum(dim=-1)
    disp_map = 1.0 / torch.max(1e-10 * torch.ones_like(depth_map), depth_map / acc_map)
    if white_background:
        rgb_map = rgb_map + (1.0 - acc_map[..., None])
    return rgb_map, disp_map, acc_map, weights, depth_map


# --------------------------------------------------------------------------------------
# Hierarchical resampling  (nerf/nerf_helpers.py:260-302, sample_pdf_2)
# --------------------------------------------------------------------------------------
def sample_pdf(bins, weights, num_samples, det=False, u: Optional[torch.Tensor] = None, return_aux=False):
    """``torchsearchsorted.searchsorted(cdf, u, side="right")`` (third-party, unpinned --
    requirements.txt:9) has numpy semantics; ``torch.searchsorted(right=True)`` is the stand-in."""
    weights = weights + 1e-5
    pdf = weights / torch.sum(weights, dim=-1, keepdim=True)
    cdf = torch.cumsum(pdf, dim=-1)
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], dim=-1)
    if det:
        u = torch.linspace(0.0, 1.0, steps=num_samples, dtype=weights.dtype)
        u = u.expand(list(cdf.shape[:-1]) + [num_samples])
    elif u is None:
        u = torch.rand(list(cdf.shape[:-1]) + [num_samples], dtype=weights.dtype)
    u = u.contiguous()
    cdf = cdf.contiguous()
    inds = torch.searchsorted(cdf, u, right=True)
    below = torch.max(torch.zeros_like(inds - 1), inds - 1)
    above = torch.min((cdf.shape[-1] - 1) * torch.ones_like(inds), inds)
    inds_g = torch.stack((below, above), dim=-1)
    matched_shape = (inds_g.shape[0], inds_g.shape[1], cdf.shape[-1])
    cdf_g = torch.gather(cdf.unsqueeze(1).expand(matched_shape), 2, inds_g)
    bins_g = torch.gather(bins.unsqueeze(1).expand(matched_shape), 2, inds_g)
    denom = cdf_g[..., 1] - cdf_g[..., 0]
    denom = torch.where(denom < 1e-5, torch.ones_like(denom), denom)
    t = (u - cdf_g[..., 0]) / denom
    samples = bins_g[..., 0] + t * (bins_g[..., 1] - bins_g[..., 0])
    if return_aux:
        return samples, inds, cdf
    return samples


def sample_from_cdf(bins, cdf, u):
    """The tail of ``sample_pdf`` from a GIVEN cdf (the "bit-exact indices given the same cdf"
    contract of SURVEY.md section 7.3 item 4).  nerf/nerf_helpers.py:286-300."""
    inds = torch.searchsorted(cdf.contiguous(), u.contiguous(), right=True)
    below = torch.clamp(inds - 1, min=0)
    above = torch.clamp(inds, max=cdf.shape[-1] - 1)
    cb, ca = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
    bb, ba = torch.gather(bins, 1, below), torch.gather(bins, 1, above)
    denom = ca - cb
    denom = torch.where(denom < 1e-5, torch.ones_like(denom), denom)
    t = (u - cb) / denom
    return bb + t * (ba - bb), inds


# --------------------------------------------------------------------------------------
# Render driver  (nerf/train_utils.py)
# --------------------------------------------------------------------------------------
def stratified_z(near, far, num_coarse, lindisp, perturb, t_rand: Optional[torch.Tensor], dtype):
    """nerf/train_utils.py:45-65.  near/far: (N,1)."""
    num_rays = near.shape[0]
    t_vals = torch.linspace(0.0, 1.0, num_coarse, dtype=dtype)
    if not lindisp:
        z_vals = near * (1.0 - t_vals) + far * t_vals
    else:
        z_vals = 1.0 / (1.0 / near * (1.0 - t_vals) + 1.0 / far * t_vals)
    z_vals = z_vals.expand([num_rays, num_coarse])
    if perturb:
        mids = 0.5 * (z_vals[..., 1:] + z_vals[..., :-1])
        upper = torch.cat((mids, z_vals[..., -1:]), dim=-1)
        lower = torch.cat((z_vals[..., :1], mids), dim=-1)
        if t_rand is None:
            t_rand = torch.rand(z_vals.shape, dtype=dtype)
        z_vals = lower + (upper - lower) * t_rand
    return z_vals


def run_network(sd, pts, ray_batch, chunksize, enc_xyz, enc_dir):
    """nerf/train_utils.py:8-25.  ``enc_*`` = (L, include_input, log_sampling) or None."""
    pts_flat = pts.reshape((-1, pts.shape[-1]))
    embedded = positional_encoding(pts_flat, *enc_xyz)
    dim_xyz = embedded.shape[-1]
    if enc_dir is not None:
        viewdirs = ray_batch[..., None, -3:]
        input_dirs = viewdirs.expand(pts.shape)
        input_dirs_flat = input_dirs.reshape((-1, input_dirs.shape[-1]))
        embedded = torch.cat((embedded, positional_encoding(input_dirs_flat, *enc_dir)), dim=-1)
    preds = [flexible_nerf_forward(sd, b, dim_xyz) for b in get_minibatches(embedded, chunksize)]
    radiance_field = torch.cat(preds, dim=0)
    return radiance_field.reshape(list(pts.shape[:-1]) + [radiance_field.shape[-1]])


def predict_and_render_radiance(
    ray_batch,
    sd_coarse,
    sd_fine,
    options,
    mode="train",
    enc_xyz=(10, True, True),
    enc_dir=(4, True, True),
    randoms: Optional[dict] = None,
    return_aux=False,
):
    """nerf/train_utils.py:28-127.  RNG draw order (SURVEY.md section 5): t_rand -> noise_c -> u -> noise_f."""
    randoms = randoms or {}
    o = getattr(options.nerf, mode)
    ro, rd = ray_batch[..., :3], ray_batch[..., 3:6]
    bounds = ray_batch[..., 6:8].view((-1, 1, 2))
    near, far = bounds[..., 0], bounds[..., 1]
    z_vals = stratified_z(near, far, o.num_coarse, o.lindisp, o.perturb, randoms.get("t_rand"), ro.dtype)
    pts = ro[..., None, :] + rd[..., None, :] * z_vals[..., :, None]
    raw_c = run_network(sd_coarse, pts, ray_batch, o.chunksize, enc_xyz, enc_dir)
    rgb_c, disp_c, acc_c, weights, depth_c = volume_render_radiance_field(
        raw_c, z_vals, rd, o.radiance_field_noise_std, o.white_background, noise=randoms.get("noise_c")
    )
    aux = dict(z_coarse=z_vals, raw_coarse=raw_c, weights_coarse=weights, depth_coarse=depth_c)
    rgb_f = disp_f = acc_f = None
    if o.num_fine > 0:
        z_mid = 0.5 * (z_vals[..., 1:] + z_vals[..., :-1])
        z_samples, inds, cdf = sample_pdf(
            z_mid, weights[..., 1:-1], o.num_fine, det=(o.perturb == 0.0), u=randoms.get("u"), return_aux=True
        )
        z_samples = z_samples.detach()
        z_vals, _ = torch.sort(torch.cat((z_vals, z_samples), dim=-1), dim=-1)
        pts = ro[..., None, :] + rd[..., None, :] * z_vals[..., :, None]
        raw_f = run_network(sd_fine, pts, ray_batch, o.chunksize, enc_xyz, enc_dir)
        rgb_f, disp_f, acc_f, w_f, depth_f = volume_render_radiance_field(
            raw_f, z_vals, rd, o.radiance_field_noise_std, o.white_background, noise=randoms.get("noise_f")
        )
        aux.update(z_samples=z_samples, inds=inds, cdf=cdf, z_fine=z_vals, raw_fine=raw_f,
                   weights_fine=w_f, depth_fine=depth_f)
    out = (rgb_c, disp_c, acc_c, rgb_f, disp_f, acc_f)
    return (out, aux) if return_aux else out


def run_one_iter_of_nerf(
    height,
    width,
    focal_length,
    sd_coarse,
    sd_fine,
    ray_origins,
    ray_directions,
    options,
    mode="train",
    enc_xyz=(10, True, True),
    enc_dir=(4, True, True),
    randoms: Optional[dict] = None,
):
    """nerf/train_utils.py:130-202, including the quirk that ``mode`` is NOT forwarded to
    ``predict_and_render_radiance`` (train_utils.py:171-181): sampling always reads
    ``options.nerf.train``; only chunksize and the final reshape honour ``mode``."""
    viewdirs = None
    if options.nerf.use_viewdirs:
        viewdirs = ray_directions
        viewdirs = viewdirs / viewdirs.norm(p=2, dim=-1).unsqueeze(-1)
        viewdirs = viewdirs.view((-1, 3))
    restore_shapes = [ray_directions.shape, ray_directions.shape[:-1], ray_directions.shape[:-1]]
    if sd_fine:
        restore_shapes += restore_shapes
    if options.dataset.no_ndc is False:
        ro, rd = ndc_rays(height, width, focal_length, 1.0, ray_origins, ray_directions)
        ro, rd = ro.view((-1, 3)), rd.view((-1, 3))
    else:
        ro, rd = ray_origins.view((-1, 3)), ray_directions.view((-1, 3))
    near = options.dataset.near * torch.ones_like(rd[..., :1])
    far = options.dataset.far * torch.ones_like(rd[..., :1])
    rays = torch.cat((ro, rd, near, far), dim=-1)
    if options.nerf.use_viewdirs:
        rays = torch.cat((rays, viewdirs), dim=-1)
    batches = get_minibatches(rays, chunksize=getattr(options.nerf, mode).chunksize)
    if randoms is not None and len(batches) != 1:
        raise ValueError("injected randoms require a single ray chunk")
    pred = [
        predict_and_render_radiance(
            b, sd_coarse, sd_fine, options, enc_xyz=enc_xyz,
            enc_dir=enc_dir if options.nerf.use_viewdirs else None, randoms=randoms,
        )
        for b in batches
    ]
    imgs = list(zip(*pred))
    imgs = [torch.cat(im, dim=0) if im[0] is not None else None for im in imgs]
    if mode == "validation":
        imgs = [im.view(shape) if im is not None else None for (im, shape) in zip(imgs, restore_shapes)]
        if sd_fine:
            return tuple(imgs)
        return tuple(imgs + [None, None, None])
    return tuple(imgs)


def nerf_loss(out, target):
    """train_nerf.py:244-258: mse(rgb_coarse, target) + mse(rgb_fine, target)."""
    loss = F.mse_loss(out[0][..., :3], target[..., :3])
    if out[3] is not None:
        loss = loss + F.mse_loss(out[3][..., :3], target[..., :3])
    return loss
