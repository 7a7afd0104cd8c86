"""Normal maps of renders (include/nerfb200.h, "normal maps"; csrc/normals.cu and density_grad_tc_kernel) on the GPU:
  * with normals=True the six render outputs are bit for bit those of the same call without it: the default render,
    with an occupancy grid, with early stopping, and with both;
  * N against an fp64 restatement from the render's own workspace: the last pass's depths and raw outputs, the fp64
    compositing weights of that raw (with the seeded noise the render used), and grad sigma by fp64 autograd at o + d z,
    summed in sample order -- lego A0 (Blender), fern A0 (NDC), a coarse-only network, a seeded perturb + noise render;
  * |N| <= acc + eps, N = 0 exactly where acc = 0;
  * cast_to_normal_image, and the refusals (a call that would train, impl 0, impl 3) before any launch."""
import pytest
import torch

import mlp_checks as M
from helpers import bits_equal, composite64, load_weights
from oracle import nerf_oracle as O

pytestmark = pytest.mark.gpu

# (weights, H, W, focal, pose, no_ndc, near, far, L_xyz, bounds of a grid)
SCENES = {
    "lego": ("lego_lowres", 48, 48, 66.7, "spherical", True, 2.0, 6.0, 10, ((-1.5,) * 3, (1.5,) * 3)),
    "fern": ("fern_lowres", 42, 56, 45.3, "eye", False, 0.0, 1.0, 6, ((-1.2, -1.2, -1.0), (1.2, 1.2, 1.0))),
}
# |N - N64| per ray against the conditioning of its samples: a gradient error of G_ERR times the pass's largest |grad|
# (test_density_grad_gpu bounds it by 2e-5 off ReLU ties) turns a sample's unit normal by at most 2 G_ERR max|g| / |g_i|
# (and never by more than 2), times its weight.  Samples where |grad| nearly vanishes are where N is ill-conditioned:
# A sample with a ReLU tie may turn its normal by up to 2 (times its weight).  Measured on an H100 80GB HBM3 at 700 W,
# the unconditioned worst is 1.1e-6 (lego), 6.8e-3 (fern, lego with noise).
G_ERR = 1e-4
N_FLOOR = 1e-5
ACC_EPS = 1e-5


def report(what, ctx, value):
    print(f"measured {what} {ctx}: {value}")


def _models(scene):
    import nerf_pytorch_b200 as nb

    weights, *_, l_xyz, _ = SCENES[scene]
    out = []
    for sd in load_weights(weights):
        m = nb.FlexibleNeRFModel(num_layers=4, hidden_size=128, skip_connect_every=4, num_encoding_fn_xyz=l_xyz,
                                 num_encoding_fn_dir=4)
        m.load_state_dict(sd)
        out.append(m.cuda())
    return out


def _pose(kind):
    return O.pose_spherical(30.0, -30.0, 4.0) if kind == "spherical" else torch.eye(4)


def _options(scene, perturb=False, noise=0.0, num_fine=128):
    _, H, W, focal, pose, no_ndc, near, far, *_ = SCENES[scene]
    return O.make_options(no_ndc=no_ndc, near=near, far=far, num_coarse=64, num_fine=num_fine, perturb=perturb,
                          radiance_field_noise_std=noise)


def _grid(scene, models, encoders):
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    return OccupancyGrid.from_models(models, encoders[0], SCENES[scene][-1], 128, encode_direction_fn=encoders[1])


def _image(scene, normals, grid=None, early_stop=None, randoms=None, perturb=False, noise=0.0):
    import nerf_pytorch_b200 as nb

    _, H, W, focal, pose, _, _, _, l_xyz, _ = SCENES[scene]
    mc, mf = _models(scene)
    return nb.render_image(H, W, focal, _pose(pose), mc, mf, _options(scene, perturb, noise), mode="validation",
                           encode_position_fn=nb.get_embedding_function(l_xyz),
                           encode_direction_fn=nb.get_embedding_function(4), impl=1, grid=grid,
                           early_stop=early_stop, randoms=randoms, normals=normals)


@pytest.mark.parametrize("variant", ["default", "grid", "early_stop", "grid+early_stop"])
def test_six_outputs_are_those_of_the_render_without_normals(variant):
    import nerf_pytorch_b200 as nb

    grid = None
    if "grid" in variant:
        mc, mf = _models("lego")
        grid = _grid("lego", [mc, mf], (nb.get_embedding_function(10), nb.get_embedding_function(4)))
    stop = 1e-3 if "early_stop" in variant else None
    rng = nb.SeededRandoms(5, 2)
    plain = _image("lego", False, grid, stop, rng, perturb=True, noise=0.2)
    with_n = _image("lego", True, grid, stop, rng, perturb=True, noise=0.2)
    assert len(plain) == 6 and len(with_n) == 7
    assert all(bits_equal(a, b) for a, b in zip(plain, with_n[:6])), variant
    n, acc = with_n[6], with_n[5]
    assert n.shape == (48, 48, 3) and torch.isfinite(n).all()
    norm = n.norm(dim=-1)
    report("max |N| - acc", variant, f"{(norm - acc).max().item():.3e}")
    assert (norm <= acc + ACC_EPS).all()
    assert (n[acc == 0] == 0).all()
    img = nb.cast_to_normal_image(n)
    assert img.dtype == torch.uint8 and img.shape == n.shape


def _render(scene, perturb, noise, coarse_only, seed):
    """(arch of the last pass, its state dict, rays, z, raw, noise of the last pass or None, noise_std, normals, acc)
    of one render_fwd_normals call, read back from its workspace."""
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops, train_utils

    _, H, W, focal, pose, no_ndc, near, far, l_xyz, _ = SCENES[scene]
    mc, mf = _models(scene)
    sd_last = load_weights(SCENES[scene][0])[0 if coarse_only else 1]
    epf, edf = nb.get_embedding_function(l_xyz), nb.get_embedding_function(4)
    arch = train_utils._arch_of(mc, train_utils._probe_encoder(epf, None), train_utils._probe_encoder(edf, None))
    blobs = [train_utils._packed(m, arch)[1] for m in (mc, mf)]
    nf = 0 if coarse_only else 128
    opts = ops.make_opts(64, nf, perturb, False, False, noise)
    rays = ops.gen_rays(_pose(pose), H, W, focal, None, "cuda", ndc=not no_ndc, near=near, far=far)
    rng = nb.SeededRandoms(seed, 0)
    arch_f = None if coarse_only else arch
    with torch.no_grad():
        out_c, out_f, normals, ws = ops.render_fwd_normals(arch, arch_f, opts, blobs[0], blobs[1] if nf else None, rays,
                                                           rng, None, None, impl=1)
    n, s = rays.shape[0], 64 + nf
    lay = ops.render_workspace_layout(arch, arch_f, opts, n, False)
    zname, rname = ("z_coarse", "raw_coarse") if coarse_only else ("z_fine", "raw_fine")
    f = ws.view(torch.float32)
    z = f[lay[zname] // 4: lay[zname] // 4 + n * s].view(n, s)
    raw = f[lay[rname] // 4: lay[rname] // 4 + n * s * 4].view(n, s, 4)
    nz = ops.random_fill(rng, "noise_c" if coarse_only else "noise_f", n, s) if noise > 0 else None
    acc = (out_c if coarse_only else out_f)[:, 4]
    return arch, sd_last, rays, z.clone(), raw.clone(), nz, noise, normals, acc


def _ties(sd64, xyz, hidden):
    """Points with a ReLU tie: a layers_xyz unit within mlp_checks.STASH_TOL of its layer's largest activation (over
    this batch) from zero in fp64, where the kernel's decision may be the other one."""
    h = torch.nn.functional.linear(xyz, sd64["layer1.weight"], sd64["layer1.bias"])
    tie = torch.zeros(xyz.shape[0], dtype=torch.bool, device=xyz.device)
    i = 0
    while f"layers_xyz.{i}.weight" in sd64:
        w = sd64[f"layers_xyz.{i}.weight"]
        if w.shape[1] != hidden:
            h = torch.cat((h, xyz), -1)
        pre = torch.nn.functional.linear(h, w, sd64[f"layers_xyz.{i}.bias"])
        tie |= (pre.abs() <= M.STASH_TOL * pre.max().clamp_min(0.0)).any(-1)
        h = torch.relu(pre)
        i += 1
    return tie


def _grad64(arch, sd, pts):
    """fp64 autograd of sigma w.r.t. the points, the bands' fp32 arguments as values (test_density_grad_gpu), and
    the points with a ReLU tie."""
    sd64 = {k: v.double().cuda() for k, v in sd.items()}
    out, ties = [], []
    d = torch.tensor([0.0, 0.0, 1.0], device="cuda")
    for p0 in range(0, pts.shape[0], 1 << 17):
        x32 = pts[p0:p0 + (1 << 17)]
        x64 = x32.double().requires_grad_()
        parts = [x64]
        for k in range(arch.n_freq_xyz):
            f = 2.0 ** k  # log-sampled bands: 2^k, exact in fp32
            a = x64 * f + ((x32 * f).double() - x64.detach() * f)
            parts += [torch.sin(a), torch.cos(a)]
        emb = torch.cat(parts + [M.embed(d.expand(x32.shape[0], 3), arch.n_freq_dir, True, True)], -1)
        raw = O.flexible_nerf_forward(sd64, emb, arch.dim_xyz)
        g, = torch.autograd.grad(raw[:, 3].sum(), x64)
        out.append(g)
        with torch.no_grad():
            ties.append(_ties(sd64, torch.cat(parts, -1).detach(), arch.hidden))
    return torch.cat(out), torch.cat(ties)


@pytest.mark.parametrize("scene,perturb,noise,coarse_only", [
    ("lego", False, 0.0, False), ("fern", False, 0.0, False), ("lego", False, 0.0, True), ("lego", True, 0.2, False)])
def test_normals_match_an_fp64_restatement(scene, perturb, noise, coarse_only):
    ctx = (scene, perturb, noise, coarse_only)
    arch, sd, rays, z, raw, nz, std, normals, acc = _render(scene, perturb, noise, coarse_only, seed=3)
    assert arch.log_sampling_xyz and arch.include_input_xyz
    pts = (rays[:, None, :3] + rays[:, None, 3:6] * z[..., None]).reshape(-1, 3)
    _, _, _, w64, _ = composite64(raw, z, rays[:, 3:6], noise_std=std, noise=nz)
    w64 = w64.reshape(-1)
    live = w64 != 0
    g = torch.zeros(pts.shape[0], 3, dtype=torch.float64, device="cuda")
    tie = torch.zeros(pts.shape[0], dtype=torch.bool, device="cuda")
    g[live], tie[live] = _grad64(arch, sd, pts[live].contiguous())
    mag = g.norm(dim=-1, keepdim=True)
    nrm64 = torch.where(mag > 0, -g / mag, torch.zeros_like(g))
    terms = (w64[:, None] * nrm64).view(rays.shape[0], -1, 3)
    N64 = torch.zeros(rays.shape[0], 3, dtype=torch.float64, device="cuda")
    for j in range(terms.shape[1]):  # in sample order
        N64 += terms[:, j]
    err = (normals.double() - N64).abs().max(-1).values
    gmax = mag.max()
    turn = torch.clamp(2 * G_ERR * gmax / mag.squeeze(-1).clamp_min(1e-300), max=2.0)
    turn[tie] = 2.0  # a ReLU tie may turn its sample's normal anywhere
    bound = (w64 * turn).view(rays.shape[0], -1).sum(-1) + N_FLOOR
    report("max |N - N64|", ctx, f"{err.max().item():.3e}, max err / bound {(err / bound).max().item():.3f} (rays "
                                 f"{rays.shape[0]}, live samples {int(live.sum())}, tie samples {int(tie.sum())})")
    assert (err <= bound).all(), ctx
    assert (normals.norm(dim=-1) <= acc + ACC_EPS).all(), ctx
    assert (normals[acc == 0] == 0).all(), ctx


def test_normals_refusals_fire_before_any_launch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    mc, mf = _models("lego")
    kw = dict(encode_position_fn=nb.get_embedding_function(10), encode_direction_fn=nb.get_embedding_function(4))
    o = _options("lego", num_fine=64)
    rays = ops.gen_rays(torch.eye(4), 8, 8, 10.0, None, "cuda", ndc=False, near=2.0, far=6.0)
    with torch.no_grad():  # pack both models once, so that nothing below is a first use
        nb.predict_and_render_radiance(rays, mc, mf, o, normals=True, **kw)
    torch.cuda.synchronize()
    before = ops.launch_count()
    with pytest.raises(NotImplementedError, match="inference"):
        nb.predict_and_render_radiance(rays, mc, mf, o, normals=True, **kw)
    with pytest.raises(NotImplementedError, match="inference"):
        nb.run_one_iter_of_nerf(8, 8, 10.0, mc, mf, rays[:, :3], rays[:, 3:6], o, normals=True, **kw)
    with torch.no_grad():
        for bad in (ops.IMPL_SIMT, ops.IMPL_TC_FAST):
            with pytest.raises(NotImplementedError, match="impl"):
                nb.predict_and_render_radiance(rays, mc, mf, o, normals=True, impl=bad, **kw)
            with pytest.raises(NotImplementedError, match="impl=1"):
                ops.render_fwd_normals(ops.ArchSpec(num_layers=4, hidden=128, skip_every=4, n_freq_xyz=10,
                                                    n_freq_dir=4), None, ops.make_opts(64, 0, False, False, False, 0.0),
                                       torch.zeros(1, device="cuda"), None, rays, {}, impl=bad)
    assert ops.launch_count() == before
