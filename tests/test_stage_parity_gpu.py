"""GPU: every CUDA stage against the oracle on the golden cases' own intermediates.

Tolerances (fp32 path): the kernels perform the same IEEE operations as the reference wherever the
reference's op order is defined (sampling, mid-points, lerp: bit-exact expected), and fp32 FMA
dot products / libm-grade sin, cos, exp elsewhere: relative 1e-4 per north_star, with the absolute
floor stated per test."""
import pytest
import torch

from helpers import CASES, Case, err_stats, frac_close

pytestmark = pytest.mark.gpu


def _arch(c: Case):
    from nerf_pytorch_b200 import ops

    return ops.ArchSpec(num_layers=c.num_layers, hidden=c.hidden, skip_every=c.skip, use_viewdirs=c.use_viewdirs,
                        n_freq_xyz=c.enc_xyz[0], n_freq_dir=c.enc_dir[0], include_input_xyz=c.enc_xyz[1],
                        include_input_dir=c.enc_dir[1], log_sampling_xyz=c.enc_xyz[2], log_sampling_dir=c.enc_dir[2])


@pytest.mark.parametrize("name", CASES)
def test_sample_coarse_in_kernel_grid_bit_exact(name):
    from nerf_pytorch_b200 import ops

    c = Case(name)
    rays, _, aux = c.aux()
    o = c.options.nerf.train
    t_rand = c.randoms["t_rand"].cuda() if o.perturb else None
    z = ops.sample_coarse(rays.cuda(), t_rand, o.num_coarse, o.perturb, o.lindisp)
    assert torch.equal(z.cpu(), aux["z_coarse"]), err_stats(z, aux["z_coarse"])


@pytest.mark.parametrize("L,include,log_sampling", [(10, True, True), (4, True, True), (6, False, False), (0, True, True)])
def test_encode(L, include, log_sampling):
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    g = torch.Generator().manual_seed(1)
    x = (torch.rand(1000, 3, generator=g) * 2 - 1) * 6.0  # |x| <= 6: arguments up to 2^9 * 6 rad
    want = O.positional_encoding(x.double(), L, include, log_sampling)
    arch = ops.ArchSpec(n_freq_xyz=L, include_input_xyz=include, log_sampling_xyz=log_sampling)
    got = ops.encode(arch, 0, x.cuda())
    assert got.shape == want.shape
    # sin/cos of an fp32-rounded argument: the fp64 oracle sees the same rounded argument only if
    # x*f is exact (log sampling: powers of two).  Otherwise compare with the fp32 oracle.
    if not log_sampling:
        want = O.positional_encoding(x, L, include, log_sampling).double()
    assert (got.double().cpu() - want).abs().max() < 2e-6


@pytest.mark.parametrize("name", CASES)
def test_mlp_forward(name):
    from nerf_pytorch_b200 import ops

    c = Case(name)
    rays, _, aux = c.aux()
    _, _, aux64 = c.aux(torch.float64)
    arch = _arch(c)
    for tag, sd in (("coarse", c.sd_c), ("fine", c.sd_f)):
        if sd is None:
            continue
        blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))
        # evaluate OUR mlp at the ORACLE's fp32 depths (stage isolation)
        z = aux["z_" + tag].cuda().contiguous()
        raw = ops.mlp_fwd(arch, blob, rays.cuda(), z).cpu()
        want32, want64 = aux["raw_" + tag], aux64["raw_" + tag]
        # the fp64 oracle ran on fp64-propagated depths for the fine pass; use fp32 oracle as the
        # primary target and fp64-vs-fp32 spread as the yardstick of what fp32 can resolve
        scale = want32.abs().max().item()
        e = (raw.double() - want32.double()).abs().max().item()
        assert e <= 1e-4 * scale + 1e-5, (tag, e, scale)
        assert frac_close(raw, want32, rtol=1e-4, atol=1e-5 * max(1.0, scale)) > 0.999, tag


@pytest.mark.parametrize("name", CASES)
def test_composite_forward_and_weights(name):
    from nerf_pytorch_b200 import ops

    c = Case(name)
    rays, out, aux = c.aux()
    o = c.options.nerf.train
    for tag, k0 in (("coarse", 0), ("fine", 3)):
        if ("raw_" + tag) not in aux:
            continue
        raw, z = aux["raw_" + tag].cuda().contiguous(), aux["z_" + tag].cuda().contiguous()
        noise = c.randoms.get("noise_c" if tag == "coarse" else "noise_f")
        noise = noise.cuda() if noise is not None else None
        res, w = ops.composite_fwd(raw, z, rays.cuda(), noise, o.radiance_field_noise_std, o.white_background)
        res, w = res.cpu(), w.cpu()
        assert torch.allclose(res[:, :3], out[k0], rtol=1e-4, atol=2e-6), err_stats(res[:, :3], out[k0])
        assert torch.allclose(res[:, 4], out[k0 + 2], rtol=1e-4, atol=2e-6)
        assert torch.allclose(w, aux["weights_" + tag], rtol=1e-4, atol=1e-6)
        assert torch.allclose(res[:, 5], aux["depth_" + tag], rtol=1e-4, atol=1e-5)
        # disp = 1/max(1e-10, depth/acc): NaN on empty rays in the reference too; compare where acc is resolvable
        acc = out[k0 + 2]
        m = acc > 1e-3
        assert torch.isnan(res[:, 3]).eq(torch.isnan(out[k0 + 1])).all()
        assert torch.allclose(res[:, 3][m], out[k0 + 1][m], rtol=2e-4, atol=1e-6)


@pytest.mark.parametrize("name", ["lego_a0_train", "fern_a0_ndc", "a1_skip_lindisp"])
def test_sample_pdf_indices_exact_given_cdf_and_values(name):
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    c = Case(name)
    _, _, aux = c.aux()
    o = c.options.nerf.train
    zc, wc = aux["z_coarse"].cuda().contiguous(), aux["weights_coarse"].cuda().contiguous()
    u = c.randoms["u"].cuda().contiguous()
    # (1) given the oracle's own cdf: indices are integer-exact and samples bit-exact
    z_fine, zs, inds, cdf = ops.sample_pdf_merge(zc, wc, u, o.num_fine, cdf_in=aux["cdf"].cuda().contiguous(), want_aux=True)
    assert torch.equal(inds.cpu().long(), aux["inds"])
    assert torch.equal(zs.cpu(), aux["z_samples"])
    assert torch.equal(z_fine.cpu(), aux["z_fine"])
    # (2) computing the cdf in-kernel: cdf within 1 ulp-ish, indices may flip only where u sits on a cdf edge
    z_fine2, zs2, inds2, cdf2 = ops.sample_pdf_merge(zc, wc, u, o.num_fine, want_aux=True)
    # torch's CPU `sum` (vectorised fp32) and the kernel's fp64-accumulated sum differ by <= 1 ulp, so the
    # cdf agrees to a few ulp; an index can flip only where u sits on a cdf edge, and -- because of the
    # reference's `denom < 1e-5 -> 1` rule (nerf_helpers.py:296) -- a flip across an (almost) empty bin
    # moves the sample by up to one bin width.  Everywhere else the samples agree to fp32 resolution.
    assert (cdf2.cpu() - aux["cdf"]).abs().max() < 1e-6
    same = inds2.cpu().long() == aux["inds"]
    assert (~same).sum().item() <= max(2, inds2.numel() // 2000), (~same).sum().item()
    # the `denom < 1e-5 -> 1` switch itself is a discontinuity: a bin whose cdf step is within an ulp of
    # 1e-5 lands on either side of it, which also moves a sample by up to one bin width at EQUAL index.
    # So: (almost) all samples agree to fp32 resolution, none differs by more than a bin.
    d = (zs2.cpu() - aux["z_samples"]).abs()
    assert (d > 1e-4).double().mean().item() < 2e-3, (d > 1e-4).double().mean().item()
    bin_w = (aux["z_coarse"][:, 1:] - aux["z_coarse"][:, :-1]).max().item()
    assert d.max() <= 1.01 * bin_w
    assert (z_fine2[:, 1:] >= z_fine2[:, :-1]).all()


def test_sample_pdf_in_kernel_det_linspace():
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    c = Case("lego_a0_det_white_val")
    _, _, aux = c.aux()
    o = c.options.nerf.train
    zc, wc = aux["z_coarse"].cuda().contiguous(), aux["weights_coarse"].cuda().contiguous()
    z_fine, zs, inds, cdf = ops.sample_pdf_merge(zc, wc, None, o.num_fine, cdf_in=aux["cdf"].cuda().contiguous(),
                                                 want_aux=True)
    assert torch.equal(inds.cpu().long(), aux["inds"])  # includes u = 1.0 -> index len(cdf)
    assert torch.equal(z_fine.cpu(), aux["z_fine"])


@pytest.mark.parametrize("white", [False, True])
def test_composite_backward_matches_autograd(white):
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    g = torch.Generator().manual_seed(3)
    n, s = 37, 77
    raw = torch.randn(n, s, 4, generator=g) * 2
    z = torch.sort(torch.rand(n, s, generator=g) * 4 + 2, -1).values
    rays = torch.randn(n, 11, generator=g)
    noise = torch.randn(n, s, generator=g)
    g_out = torch.zeros(n, 8)
    g_out[:, :5] = torch.randn(n, 5, generator=g)
    raw64 = raw.double().requires_grad_(True)
    rgb, disp, acc, w, depth = O.volume_render_radiance_field(raw64, z.double(), rays[:, 3:6].double(), 0.3, white,
                                                              noise=noise.double())
    loss = (rgb * g_out[:, :3].double()).sum() + (disp * g_out[:, 3].double()).sum() + (acc * g_out[:, 4].double()).sum()
    loss.backward()
    got = ops.composite_bwd(raw.cuda(), z.cuda(), rays.cuda(), noise.cuda(), g_out.cuda(), 0.3, white).cpu()
    want = raw64.grad
    scale = want.abs().max().item()
    assert (got.double() - want).abs().max().item() <= 2e-4 * scale, err_stats(got, want)


@pytest.mark.parametrize("name", ["lego_a0_train", "a1_skip_lindisp", "a0_noview_coarse_only"])
def test_mlp_backward_matches_autograd(name):
    """d(sum(raw * G))/d(params) through the CUDA dgrad/wgrad kernels vs torch autograd of the oracle MLP."""
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    c = Case(name)
    rays, _, aux = c.aux()
    arch = _arch(c)
    sd = c.sd_c
    z = aux["z_coarse"]
    gen = torch.Generator().manual_seed(11)
    G = torch.randn(z.shape[0], z.shape[1], 4, generator=gen)
    # oracle (fp64 autograd)
    sd64 = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    # the points are formed in fp32 exactly like the reference does (train_utils.py:67) and only then
    # promoted: an fp64 `o + d*z` is a different input (2^9 * 6e-8 * |x| rad at the top frequency)
    pts = (rays[:, None, :3] + rays[:, None, 3:6] * z[..., None]).double()
    raw64 = O.run_network(sd64, pts, rays.double(), 1 << 20, c.enc_xyz, c.enc_dir if c.use_viewdirs else None)
    (raw64 * G.double()).sum().backward()
    # ours
    flat = ops.flatten_state_dict(arch, sd, "cuda")
    blob = ops.pack_weights(arch, flat)
    raw, stash = ops.mlp_fwd(arch, blob, rays.cuda(), z.cuda().contiguous(), want_stash=True)
    flat_grad, _ = ops.mlp_bwd(arch, blob, rays.cuda(), z.cuda().contiguous(), G.cuda().contiguous(), stash)
    flat_grad = flat_grad.cpu()
    for lname, w_off, b_off, fin, fout in arch.flat_layout():
        gw = flat_grad[w_off:w_off + fin * fout].view(fout, fin)
        gb = flat_grad[b_off:b_off + fout]
        for got, want, what in ((gw, sd64[lname + ".weight"].grad, "weight"), (gb, sd64[lname + ".bias"].grad, "bias")):
            scale = want.abs().max().item() + 1e-30
            e = (got.double() - want).abs().max().item()
            assert e <= 2e-4 * scale, (lname, what, e, scale)
