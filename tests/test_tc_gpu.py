"""GPU: the wgmma kernels against the oracle (fp64 where the comparison is a gradient) and the fp32 CUDA-core kernels.

The three-term fp16x2 splits (x = hi + lo 2^-11, x_hi*w_hi + x_lo*w_hi + x_hi*w_lo, fp32 accumulate) keep ~22 bits of
every product, so the bar is the fp32 path's: the MEASURED error is ~5e-6 of the tensor's scale on the shipped
checkpoints; the asserts below are written against that (with headroom for the sum over 128..320 terms), far inside the
1e-4 relative of north_star, and the worst element is bounded, not just a quantile."""
import pytest
import torch

from helpers import Case, arch_of, build_models, frac_close
from mlp_checks import (StashLayout, as_state_dict, check_blocks, mask_words, oracle, read_layer, relu_ties,
                        tensor_blocks)

pytestmark = pytest.mark.gpu

TC_CASES = ["lego_a0_train", "fern_a0_ndc", "a1_skip_lindisp", "a0_noview_coarse_only"]
TC_TRAIN_CASES = ["lego_a0_train", "fern_a0_ndc", "a1_skip_lindisp"]  # the fused backward needs the view-dependent heads


@pytest.mark.parametrize("name", TC_CASES)
def test_tc_forward_matches_simt_and_oracle(name):
    from nerf_pytorch_b200 import ops

    c = Case(name)
    rays, _, aux = c.aux()
    arch = arch_of(c)
    layers = StashLayout(arch).layers
    for tag, sd in (("coarse", c.sd_c), ("fine", c.sd_f)):
        if sd is None:
            continue
        blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))
        z = aux["z_" + tag].cuda().contiguous()
        raw0, st0 = ops.mlp_fwd(arch, blob, rays.cuda(), z, impl=ops.IMPL_SIMT, want_stash=True)
        raw1, st1 = ops.mlp_fwd(arch, blob, rays.cuda(), z, impl=ops.IMPL_TC, want_stash=True)
        torch.cuda.synchronize()
        want = aux["raw_" + tag]
        scale = want.abs().max().item()
        e_tc = (raw1.cpu().double() - want.double()).abs().max().item()
        e_simt = (raw0.cpu().double() - want.double()).abs().max().item()
        # worst element: 3e-5 of the output scale (measured ~5e-6; the fp32 reference itself is ~2e-6 from fp64)
        assert e_tc <= 3e-5 * scale + 1e-6, (tag, e_tc, e_simt, scale)
        assert frac_close(raw1.cpu(), want, rtol=1e-4, atol=1e-5 * max(1.0, scale)) > 0.9999, tag
        # the stash the backward consumes: every layer's activation tile decodes to the fp32 kernel's activations
        P = z.numel()
        for lname, n, cum in layers:
            a0 = read_layer(st0, P, cum, n, "fp32")
            a1 = read_layer(st1, P, cum, n, "wgmma")
            s = a0.abs().max().item()
            assert (a1 - a0).abs().max().item() <= 3e-5 * s + 1e-7, (tag, lname, (a1 - a0).abs().max().item(), s)


@pytest.mark.parametrize("viewdirs", [True, False])
def test_tc_forward_hidden_256_matches_oracle_and_fp32_kernel(viewdirs):
    """pretrained/*/config.yml as written (8 x 256, skip 4): the wgmma inference forward (one tile in flight, N = 256 MMAs)
    against the fp64 oracle MLP and the fp32 CUDA-core kernel, ragged tile tail included."""
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    arch = ops.ArchSpec(num_layers=8, hidden=256, skip_every=4, n_freq_xyz=10, n_freq_dir=4, use_viewdirs=viewdirs)
    g = torch.Generator().manual_seed(3)
    sd = O.init_flexible_nerf(8, 256, 4, 10, 4, use_viewdirs=viewdirs, generator=g)
    n, s_ = 37, 52   # 1924 points: 15 full tiles + a ragged one, tiles straddle rays
    d = torch.randn(n, 3, generator=g)
    rays = torch.cat([torch.randn(n, 3, generator=g) * 0.3, d, torch.full((n, 1), 2.0), torch.full((n, 1), 6.0),
                      d / d.norm(dim=-1, keepdim=True)], -1)
    rays = (rays if viewdirs else rays[:, :8]).contiguous()
    z = torch.sort(torch.rand(n, s_, generator=g) * 4 + 2, -1).values.contiguous()
    blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))
    raw0 = ops.mlp_fwd(arch, blob, rays.cuda(), z.cuda(), impl=ops.IMPL_SIMT)
    raw1 = ops.mlp_fwd(arch, blob, rays.cuda(), z.cuda(), impl=ops.IMPL_TC)
    torch.cuda.synchronize()
    want = oracle(arch, sd, rays, z)[0].view(n, s_, 4)
    scale = want.abs().max().item()
    e_tc = (raw1.cpu().double() - want).abs().max().item()
    e_simt = (raw0.cpu().double() - want).abs().max().item()
    assert e_tc <= 3e-5 * scale + 1e-6, (e_tc, e_simt, scale)
    assert e_simt <= 3e-5 * scale, (e_tc, e_simt, scale)   # the fp32 kernels measure <= 3.3e-6 (test_simt_hidden256_gpu)
    assert torch.isfinite(raw1).all()


def test_hidden_256_renders_on_wgmma_in_inference_and_trains_on_fp32_kernels():
    """The automatic implementation choice for the shipped-checkpoint architecture (8 x 256): torch.no_grad() renders go
    through the wgmma forward and agree with the fp32 CUDA-core path; a training step silently uses the fp32 kernels."""
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops, train_utils
    from oracle import nerf_oracle as O

    torch.manual_seed(0)
    kw = dict(num_layers=8, hidden_size=256, skip_connect_every=4, num_encoding_fn_xyz=10, num_encoding_fn_dir=4)
    mc, mf = nb.FlexibleNeRFModel(**kw).cuda(), nb.FlexibleNeRFModel(**kw).cuda()
    epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
    arch = train_utils._arch_of(mc, (10, True, True), (4, True, True))
    assert train_utils._auto_impl(arch, arch, 64, 64, training=False) == ops.IMPL_TC
    assert train_utils._auto_impl(arch, arch, 64, 64, training=True) == ops.IMPL_SIMT
    n = 300
    d = torch.randn(n, 3, device="cuda")
    ro, rd = torch.randn(n, 3, device="cuda") * 0.2 + torch.tensor([0.0, 0.0, 4.0], device="cuda"), -d.abs() * 0.3 - torch.tensor([0, 0, 1.0], device="cuda")
    det = O.make_options(num_coarse=64, num_fine=64, perturb=False, radiance_field_noise_std=0.0)
    with torch.no_grad():
        out_tc = nb.run_one_iter_of_nerf(100, 100, 120.0, mc, mf, ro, rd, det, mode="validation", encode_position_fn=epf,
                                         encode_direction_fn=edf)
        out_32 = nb.run_one_iter_of_nerf(100, 100, 120.0, mc, mf, ro, rd, det, mode="validation", encode_position_fn=epf,
                                         encode_direction_fn=edf, impl=ops.IMPL_SIMT)
    for i, (a, b) in enumerate(zip(out_tc, out_32)):   # (rgb, disp, acc) of the coarse and of the fine pass
        if i % 3 != 1:   # rgb and acc: the same render to fp32 round-off of the MLP outputs
            assert torch.isfinite(a).all()
            # coarse pass: fp32 round-off; fine pass: the resampler sits on the coarse weights, a 1e-7 difference there can move
            # a sample across a bin edge (the same sensitivity the reference has between its own fp32 and fp64 runs)
            tol = 2e-5 if i < 3 else 5e-4
            assert (a - b).abs().max().item() <= tol * max(1.0, b.abs().max().item()), (i, (a - b).abs().max().item())
            assert (a - b).abs().mean().item() <= 2e-6, (i, (a - b).abs().mean().item())
        else:            # disp = 1 / (depth / acc) is NaN on an empty ray (reference quirk) and ill-conditioned on a nearly
            acc = out_32[i + 1]   # empty one: compared where the ray has hit something
            hit = acc > 1e-2
            assert (torch.isnan(a) == torch.isnan(b)).all()
            assert (a[hit] - b[hit]).abs().max().item() <= 1e-3 * b[hit].abs().max().item(), (i, (a[hit] - b[hit]).abs().max().item())
    # training: no wgmma backward for hidden 256 -> the fp32 kernels, chosen by the library, gradients arrive
    tr = O.make_options(num_coarse=32, num_fine=32, perturb=True, radiance_field_noise_std=0.2)
    out = nb.run_one_iter_of_nerf(100, 100, 120.0, mc, mf, ro[:64], rd[:64], tr, mode="train", encode_position_fn=epf,
                                  encode_direction_fn=edf)
    (out[0].sum() + out[3].sum()).backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in list(mc.parameters()) + list(mf.parameters()))


def test_tc_ragged_tail_and_sizes():
    """Tiles that straddle rays / a ragged last tile / 1 ray: same results as the fp32 kernel."""
    from nerf_pytorch_b200 import ops

    c = Case("lego_a0_train")
    arch = arch_of(c)
    blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, c.sd_f, "cuda"))
    g = torch.Generator().manual_seed(5)
    for n, s in ((1, 64), (3, 192), (7, 50), (33, 17), (129, 100)):
        d = torch.randn(n, 3, generator=g)
        rays = torch.cat([torch.randn(n, 3, generator=g) * 0.1 + torch.tensor([0.0, -2.0, 3.0]), d,
                          torch.full((n, 1), 2.0), torch.full((n, 1), 6.0), d / d.norm(dim=-1, keepdim=True)], -1).cuda()
        z = torch.sort(torch.rand(n, s, generator=g) * 4 + 2, -1).values.cuda().contiguous()
        r0 = ops.mlp_fwd(arch, blob, rays.contiguous(), z, impl=ops.IMPL_SIMT)
        r1 = ops.mlp_fwd(arch, blob, rays.contiguous(), z, impl=ops.IMPL_TC)
        scale = r0.abs().max().item()
        assert (r1 - r0).abs().max().item() <= 3e-5 * scale + 1e-6, (n, s, (r1 - r0).abs().max().item(), scale)


@pytest.mark.parametrize("name", TC_TRAIN_CASES)
def test_tc_backward_matches_fp64_oracle(name):
    """The fused wgmma backward (data-gradient chain + every weight gradient in one kernel) against fp64 autograd of
    the oracle MLP, directly: every weight / bias gradient tensor within 1e-4 of its own scale (worst element)."""
    from nerf_pytorch_b200 import ops

    c = Case(name)
    rays, _, aux = c.aux()
    arch = arch_of(c)
    for tag, sd in (("coarse", c.sd_c), ("fine", c.sd_f)):
        if sd is None:
            continue
        z = aux["z_" + tag]
        gen = torch.Generator().manual_seed(11)
        G = torch.randn(z.shape[0], z.shape[1], 4, generator=gen)
        # realistic upstream gradients span decades across the samples of a ray (compositing weights): scale the rows
        G = G * torch.exp(torch.randn(z.shape[0], z.shape[1], 1, generator=gen) * 3.0)
        _, acts, _, want = oracle(arch, sd, rays, z, G)
        blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))
        zc, Gc = z.cuda().contiguous(), G.cuda().contiguous()
        _, stash = ops.mlp_fwd(arch, blob, rays.cuda(), zc, impl=ops.IMPL_TC, want_stash=True)
        # ReLU ties: a unit whose pre-activation is within rounding of zero gets relu'() = 0 or 1 depending on the
        # arithmetic (fp64 oracle / fp32 reference / split-precision forward) -- a genuine discontinuity of the
        # function, not a property of the backward.  Count the forward's disagreements with the fp64 oracle, check
        # each is such a tie, then give the backward the oracle's masks so the comparison below measures the
        # backward's arithmetic alone.  Every disagreement sits within 2e-5 of the layer's scale of zero.
        n_ties = relu_ties(arch, stash, z.numel(), acts, "wgmma", 2e-5, (name, tag), adopt=True)
        g1, _ = ops.mlp_bwd(arch, blob, rays.cuda(), zc, Gc, stash, impl=ops.IMPL_TC)
        torch.cuda.synchronize()
        check_blocks(arch, g1, want, tensor_blocks(arch), 2e-5, (name, tag, f"{n_ties} relu ties patched"), None)


def test_tc_backward_ragged_sizes():
    """Point counts that are not multiples of the 128-point tile, tiles that straddle many rays, a single ray: the fused
    wgmma backward vs the fp32 CUDA-core kernels."""
    from nerf_pytorch_b200 import ops

    for case in ("lego_a0_train", "a1_skip_lindisp"):
        c = Case(case)
        arch = arch_of(c)
        blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, c.sd_f, "cuda"))
        g = torch.Generator().manual_seed(7)
        for n, s in ((1, 16), (7, 50), (33, 17), (5, 37), (129, 100)):
            d = torch.randn(n, 3, generator=g)
            rays = torch.cat([torch.randn(n, 3, generator=g) * 0.1 + torch.tensor([0.0, -2.0, 3.0]), d,
                              torch.full((n, 1), 2.0), torch.full((n, 1), 6.0), d / d.norm(dim=-1, keepdim=True)],
                             -1).cuda().contiguous()
            z = torch.sort(torch.rand(n, s, generator=g) * 4 + 2, -1).values.cuda().contiguous()
            G = torch.randn(n, s, 4, generator=g).cuda()
            _, st0 = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_SIMT, want_stash=True)
            _, st1 = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC, want_stash=True)
            # same ReLU decisions for both (see test_tc_backward_matches_fp64_oracle): copy the fp32 kernel's masks
            for li in range(1, len(StashLayout(arch).layers)):
                mask_words(arch, st1, n * s, li, "wgmma").copy_(mask_words(arch, st0, n * s, li, "fp32"))
            g0, _ = ops.mlp_bwd(arch, blob, rays, z, G, st0, impl=ops.IMPL_SIMT)
            g1, _ = ops.mlp_bwd(arch, blob, rays, z, G, st1, impl=ops.IMPL_TC)
            check_blocks(arch, g1, as_state_dict(arch, g0), tensor_blocks(arch), 3e-5, (case, n, s), None)


def test_tc_backward_accumulates_and_repeats():
    """flat_grad is accumulated into (+=), and two calls give bit-identical gradients: the CTAs add into a fixed-point
    gradient blob, whose integer sums do not depend on the order of the adds."""
    from nerf_pytorch_b200 import ops

    c = Case("a1_skip_lindisp")
    rays, _, aux = c.aux()
    arch = arch_of(c)
    blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, c.sd_c, "cuda"))
    z = aux["z_coarse"].cuda().contiguous()
    G = torch.randn(z.shape[0], z.shape[1], 4, generator=torch.Generator().manual_seed(3)).cuda()
    _, stash = ops.mlp_fwd(arch, blob, rays.cuda(), z, impl=ops.IMPL_TC, want_stash=True)
    g1, _ = ops.mlp_bwd(arch, blob, rays.cuda(), z, G, stash, impl=ops.IMPL_TC)
    g2, _ = ops.mlp_bwd(arch, blob, rays.cuda(), z, G, stash, impl=ops.IMPL_TC)
    scale = g1.abs().max().item()
    assert scale > 0 and torch.equal(g1, g2)


def test_tc_unsupported_configs_are_refused():
    from nerf_pytorch_b200 import ops

    arch = ops.ArchSpec(num_layers=8, hidden=256, skip_every=4, n_freq_xyz=10)
    blob = ops.pack_weights(arch, torch.zeros(arch.flat_param_count(), device="cuda"))
    rays = torch.zeros(4, 11, device="cuda")
    z = torch.ones(4, 64, device="cuda")
    with pytest.raises(NotImplementedError):   # hidden 256: no activation stash / fused backward on wgmma ...
        ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC, want_stash=True)
    ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC)   # ... but the inference forward runs
    assert not ops.impl_supported(arch, 64, ops.IMPL_TC)
    assert ops.impl_supported(arch, 64, ops.IMPL_TC_FWD)
    assert ops.impl_supported(arch, 64, ops.IMPL_SIMT)
    # the fused backward rides the heads' weight gradients on layers_dir[0]: no view directions -> CUDA cores
    assert not ops.impl_supported(ops.ArchSpec(use_viewdirs=False), 64, ops.IMPL_TC)
    assert ops.impl_supported(ops.ArchSpec(num_layers=8, hidden=128, skip_every=3, n_freq_xyz=10), 64, ops.IMPL_TC)
    # the stage-level halves do not exist on wgmma
    a0 = ops.ArchSpec()
    with pytest.raises(NotImplementedError):
        ops.mlp_dgrad(a0, blob, torch.zeros(4, 64, 4, device="cuda"), torch.zeros(8, device="cuda"), impl=ops.IMPL_TC)


@pytest.mark.parametrize("name", ["lego_a0_train", "a1_skip_lindisp"])
def test_tc_end_to_end_against_reference_golden(name):
    import nerf_pytorch_b200 as nb

    c = Case(name)
    mc, mf, epf, edf = build_models(c)
    rnd = {k: v.cuda() for k, v in c.randoms.items()}
    with torch.no_grad():
        out = nb.run_one_iter_of_nerf(c.H, c.W, c.focal, mc, mf, c.ro.cuda(), c.rd.cuda(), c.options, mode=c.mode,
                                      encode_position_fn=epf, encode_direction_fn=edf, randoms=rnd, impl=1)
    for k in (0, 2, 3, 5):
        assert frac_close(out[k].cpu(), c.outputs[k], rtol=1e-4, atol=2e-5) > 0.97, k
