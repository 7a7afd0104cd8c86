"""GPU: the host-side pieces that sit in the timed step next to the per-ray kernels -- ray generation / packing
(csrc/raygen.cu), the flat-parameter fused Adam with the reference's LR schedule, the full-image renderer -- each
against the oracle / torch on the same inputs."""
import math

import pytest
import torch

from helpers import CASES, Case, arch_of, build_models, pack_rays
from oracle import nerf_oracle as O

pytestmark = pytest.mark.gpu


def _ulp_close(a, b, ulps=2):
    a, b = a.double().cpu(), b.double().cpu()
    tol = ulps * 2.0 ** -23 * b.abs().clamp_min(1e-30)
    return bool(((a - b).abs() <= tol).all())


@pytest.mark.parametrize("name", CASES)
def test_pack_rays_matches_reference_packing(name):
    """[o d near far viewdir] rows (train_utils.py:143-168, incl. the NDC case) from one kernel == the oracle's torch ops."""
    from nerf_pytorch_b200 import ops

    c = Case(name)
    want = pack_rays(c)                      # oracle helpers on CPU
    got = ops.pack_rays(c.ro.reshape(-1, 3).cuda(), c.rd.reshape(-1, 3).cuda(), c.H, c.W, c.focal,
                        c.options.dataset.no_ndc is False, c.options.dataset.near, c.options.dataset.far, c.use_viewdirs)
    assert got.shape == want.shape
    exact = (got.cpu() == want).float().mean().item()
    assert exact > 0.999, exact              # bit-identical almost everywhere ...
    assert _ulp_close(got, want, ulps=2)     # ... and never more than 2 ulp away (3-term sums / the norm)


@pytest.mark.parametrize("ndc", [False, True])
def test_gen_rays_from_pose_matches_get_ray_bundle(ndc):
    from nerf_pytorch_b200 import ops
    import nerf_pytorch_b200 as nb

    H, W, focal = 37, 52, 41.5
    pose = O.pose_spherical(30.0, -30.0, 4.0) if not ndc else torch.eye(4)
    ro, rd = O.get_ray_bundle(H, W, focal, pose)
    # get_ray_bundle mirror: every pixel, (H, W, 3) x 2
    g_ro, g_rd = nb.get_ray_bundle(H, W, focal, pose)
    assert torch.equal(g_ro.cpu(), ro) and _ulp_close(g_rd, rd, ulps=1)
    assert (g_rd.cpu() == rd).float().mean().item() > 0.999
    # selected pixels straight into packed rows
    g = torch.Generator().manual_seed(0)
    pix = torch.randperm(H * W, generator=g)[:500]
    vd = rd / rd.norm(p=2, dim=-1).unsqueeze(-1)
    ro_s, rd_s = ro.reshape(-1, 3)[pix], rd.reshape(-1, 3)[pix]
    if ndc:
        ro_s, rd_s = O.ndc_rays(H, W, focal, 1.0, ro_s, rd_s)
    want = torch.cat([ro_s, rd_s, torch.full((500, 1), 0.25), torch.full((500, 1), 3.5), vd.reshape(-1, 3)[pix]], -1)
    got = ops.gen_rays(pose, H, W, focal, pix.cuda(), "cuda", ndc=ndc, near=0.25, far=3.5, use_viewdirs=True)
    assert _ulp_close(got, want, ulps=2), (got.cpu() - want).abs().max()
    if ndc:  # the ndc_rays mirror
        n_ro, n_rd = nb.ndc_rays(H, W, focal, 1.0, ro.cuda(), rd.cuda())
        w_ro, w_rd = O.ndc_rays(H, W, focal, 1.0, ro, rd)
        assert _ulp_close(n_ro, w_ro, ulps=2) and _ulp_close(n_rd, w_rd, ulps=2)


def test_fused_adam_matches_torch_adam_with_reference_lr_schedule():
    """parallel.FusedAdam (nerfb200_adam_step over the flat buffers of flatten_parameters) against torch.optim.Adam driven
    the way train_nerf.py:136-141,261-270 drives it (LR updated AFTER each step), 15 steps, fast decay."""
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import parallel, train_utils

    torch.manual_seed(3)
    kw = dict(num_layers=8, hidden_size=128, skip_connect_every=3, num_encoding_fn_xyz=10, num_encoding_fn_dir=4)
    ours, ref = nb.FlexibleNeRFModel(**kw).cuda(), nb.FlexibleNeRFModel(**kw).cuda()
    ref.load_state_dict(ours.state_dict())
    arch = train_utils._arch_of(ours, (10, True, True), (4, True, True))
    sd_before = {k: v.clone() for k, v in ours.state_dict().items()}
    lr0, decay_k, factor = 5e-3, 0.004, 0.1          # lr_decay * 1000 = 4 steps per decade: the schedule really moves
    opt = parallel.FusedAdam([(ours, arch)], lr=lr0, lr_decay=decay_k, lr_decay_factor=factor)
    # flatten_parameters: same names / values, parameters are views of ONE buffer in the library's order
    assert all(torch.equal(sd_before[k], v) for k, v in ours.state_dict().items())
    flat = opt.items[0]["flat"]
    params = train_utils._ordered_params(ours, arch)
    assert params[0].data_ptr() == flat.data_ptr() and sum(p.numel() for p in params) == flat.numel()
    assert train_utils._flat_view_if_contiguous(params) is flat
    topt = torch.optim.Adam(ref.parameters(), lr=lr0)
    names = [n for n, _ in ours.named_parameters()]
    g = torch.Generator(device="cuda").manual_seed(5)
    for i in range(15):
        grads = {n: torch.randn(p.shape, generator=g, device="cuda") * (0.1 + i) for n, p in ours.named_parameters()}
        for n, p in ours.named_parameters():
            p.grad = grads[n].clone()
        for n, p in ref.named_parameters():
            p.grad = grads[n].clone()
        assert math.isclose(opt.current_lr(), topt.param_groups[0]["lr"], rel_tol=1e-12), i
        opt.step()
        topt.step()
        lr_new = lr0 * (factor ** (i / (decay_k * 1000.0)))   # train_nerf.py:264-270, after the step
        for pg in topt.param_groups:
            pg["lr"] = lr_new
    for n in names:
        a, b = dict(ours.named_parameters())[n], dict(ref.named_parameters())[n]
        assert torch.allclose(a, b, rtol=2e-5, atol=2e-7), (n, (a - b).abs().max().item())
    assert getattr(ours, "_nerfb200_epoch", 0) == 15   # the packed-weight cache is invalidated on every step


def test_training_trajectory_through_fused_adam_matches_oracle():
    """The whole timed step of bench.py (render, loss, backward, FusedAdam on the flat buffers) against the oracle + torch
    Adam with identical injected randoms: same loss trajectory."""
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import parallel, train_utils

    torch.set_num_threads(8)
    c = Case("lego_a0_train")
    n, nc, nf, iters = 96, 64, 64, 10
    opts = O.make_options(num_coarse=nc, num_fine=nf, perturb=True, radiance_field_noise_std=0.2)
    gi = torch.Generator().manual_seed(5)
    sd0c = O.init_flexible_nerf(4, 128, 4, 10, 4, generator=gi)
    sd0f = O.init_flexible_nerf(4, 128, 4, 10, 4, generator=gi)
    g = torch.Generator().manual_seed(9)
    rnds = [dict(t_rand=torch.rand(n, nc, generator=g), noise_c=torch.randn(n, nc, generator=g),
                 u=torch.rand(n, nf, generator=g), noise_f=torch.randn(n, nc + nf, generator=g)) for _ in range(iters)]
    tgt = torch.rand(n, 3, generator=g)
    sc = {k: v.clone().requires_grad_(True) for k, v in sd0c.items()}
    sf = {k: v.clone().requires_grad_(True) for k, v in sd0f.items()}
    topt = torch.optim.Adam(list(sc.values()) + list(sf.values()), lr=5e-3)
    ref_losses = []
    for r in rnds:
        out = O.run_one_iter_of_nerf(c.H, c.W, c.focal, sc, sf, c.ro, c.rd, opts, randoms=r)
        loss = O.nerf_loss(out, tgt)
        topt.zero_grad(); loss.backward(); topt.step()
        ref_losses.append(loss.item())

    def mk(sd):
        m = nb.FlexibleNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4)
        m.load_state_dict(sd)
        return m.cuda()
    mc, mf = mk(sd0c), mk(sd0f)
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    arch = train_utils._arch_of(mc, (10, True, True), (4, True, True))
    opt = parallel.FusedAdam([(mc, arch), (mf, arch)], lr=5e-3)
    losses = []
    for r in rnds:
        out = nb.run_one_iter_of_nerf(c.H, c.W, c.focal, mc, mf, c.ro.cuda(), c.rd.cuda(), opts,
                                      encode_position_fn=epf, encode_direction_fn=edf,
                                      randoms={k: v.cuda() for k, v in r.items()})
        loss = torch.nn.functional.mse_loss(out[0], tgt.cuda()) + torch.nn.functional.mse_loss(out[3], tgt.cuda())
        opt.zero_grad(); loss.backward(); opt.step()
        losses.append(loss.item())
    rel = [abs(a - b) / abs(b) for a, b in zip(losses, ref_losses)]
    assert max(rel[:4]) < 2e-3, (losses[:4], ref_losses[:4])
    assert max(rel) < 5e-2, (losses, ref_losses)
    assert losses[-1] < 0.7 * losses[0]


def test_render_image_matches_run_one_iter_validation():
    """eval_utils.render_image (rays generated on the device from the pose, chunked forward) == run_one_iter_of_nerf in
    validation mode on get_ray_bundle's rays; uint8 conversions of eval_nerf.py:23-36."""
    import nerf_pytorch_b200 as nb

    c = Case("lego_a0_det_white_val")        # deterministic sampler, white background
    mc, mf, epf, edf = build_models(c)
    H, W, focal = 24, 32, 44.0
    pose = O.pose_spherical(20.0, -35.0, 4.0)
    ro, rd = nb.get_ray_bundle(H, W, focal, pose)
    with torch.no_grad():
        want = nb.run_one_iter_of_nerf(H, W, focal, mc, mf, ro, rd, c.options, mode="validation",
                                       encode_position_fn=epf, encode_direction_fn=edf)
    got = nb.render_image(H, W, focal, pose, mc, mf, c.options, mode="validation", encode_position_fn=epf,
                          encode_direction_fn=edf, rays_per_chunk=300)
    for a, b in zip(got, want):
        assert a.shape == b.shape
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-6, equal_nan=True)
    img = nb.cast_to_image(got[3])
    assert img.dtype == torch.uint8 and img.shape == (H, W, 3)
    assert torch.equal(img, (got[3] * 255).clamp(0, 255).to(torch.uint8))
    dimg = nb.cast_to_disparity_image(got[4])
    assert dimg.dtype == torch.uint8 and dimg.shape == (H, W)


def test_tc_out_of_range_activations_are_visible_not_clamped():
    """The fp16 x 2 operands cover |activation| < 1.05e6 (value / 16 in fp16): beyond that the wgmma forward produces
    inf / NaN (non-saturating conversions) instead of silently clamping -- and stays exact below."""
    from nerf_pytorch_b200 import ops

    c = Case("lego_a0_train")
    rays, _, aux = c.aux()
    arch = arch_of(c)
    z = aux["z_fine"].cuda().contiguous()
    flat = ops.flatten_state_dict(arch, c.sd_f, "cuda")
    for scale, expect_finite in ((1.0, True), (40.0, False)):
        f2 = flat.clone()
        for name, w_off, b_off, fin, fout in arch.flat_layout():
            if name == "layer1":                     # blow up the first layer's output: activations * scale
                f2[w_off:w_off + fin * fout] *= scale
                f2[b_off:b_off + fout] *= scale
        blob = ops.pack_weights(arch, f2)
        r1 = ops.mlp_fwd(arch, blob, rays.cuda(), z, impl=ops.IMPL_TC)
        r0 = ops.mlp_fwd(arch, blob, rays.cuda(), z, impl=ops.IMPL_SIMT)
        assert torch.isfinite(r0).all()
        if expect_finite:
            assert torch.isfinite(r1).all()
        else:
            bad = ~torch.isfinite(r1)
            # wherever the result is finite it is still right; where the range was exceeded it is inf / NaN, never a
            # plausible-looking clamped number
            ok = ~bad
            s = r0.abs().max().item()
            assert bad.any()
            if ok.any():
                assert (r1[ok] - r0[ok]).abs().max().item() <= 1e-4 * s
