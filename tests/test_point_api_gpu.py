"""GPU: run_network and volume_render_radiance_field, the drop-ins for the reference's per-sample pipeline
(nerf/train_utils.py:8-25, nerf/volume_rendering_utils.py:6-53) on caller-given points and depths.

  1. composed on the render path's own samples they give the render path's bits, outputs and gradients;
  2. run_network at points off any ray against the fp64 oracle MLP, forward and per-block parameter gradients;
  3. the view direction is read in place from the last three columns of any row layout;
  4. volume_render_radiance_field against the fp64 oracle, all five outputs and their gradients;
  5. a density-grid query without rows stays on the wgmma kernels;
  6. with gradient sync on, the backward leaves the reduction to FusedAdam.step."""
import math

import pytest
import torch

from helpers import Case, bits_equal, build_models, composite64
from mlp_checks import (ALL_ARCHS, BLOCK_TOL, COMP_GRAD_TOL, COMP_TOL, H256_ARCHS, SHAPES, SIMT128_ARCHS, SIMT_FWD_TOL,
                        TC_ARCHS, TC_FWD_TOL, _floors, _split_floors, arch_weights, check_blocks, oracle, report, spec,
                        tc_blocks, upstream)

pytestmark = pytest.mark.gpu

FAST_TOL = 2e-2         # the single-pass forward against fp64 (test_tc_fast_gpu.py FAST_TOL)
REF32_FACTOR = 4.0      # trained compositing regime, each output alone: x the fp32 reference's own error [2.0]


def _nb():
    import nerf_pytorch_b200 as nb

    return nb


def _model(arch, sd):
    nb = _nb()
    m = nb.FlexibleNeRFModel(num_layers=arch.num_layers, hidden_size=arch.hidden, skip_connect_every=arch.skip_every,
                             num_encoding_fn_xyz=arch.n_freq_xyz, num_encoding_fn_dir=arch.n_freq_dir,
                             include_input_xyz=arch.include_input_xyz, include_input_dir=arch.include_input_dir,
                             use_viewdirs=arch.use_viewdirs)
    m.load_state_dict(sd)
    epf = nb.get_embedding_function(arch.n_freq_xyz, arch.include_input_xyz, arch.log_sampling_xyz)
    edf = (nb.get_embedding_function(arch.n_freq_dir, arch.include_input_dir, arch.log_sampling_dir)
           if arch.use_viewdirs else None)
    return m.cuda(), epf, edf


def _flat_grad(arch, model):
    from nerf_pytorch_b200 import ops

    return ops.flatten_state_dict(arch, {k: p.grad for k, p in model.named_parameters()}, "cpu")


# ------------------------------------------------------------------------------------------------------------------------
# 1. the render path's samples through the two drop-ins: the render path's bits
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("noise_std", [0.0, 0.3])
@pytest.mark.parametrize("impl", [0, 1, 3])
@pytest.mark.parametrize("case_name", ["lego_a0_train", "a1_skip_lindisp"])  # A0 with the lego weights, A1 at init
def test_composed_drop_ins_give_the_render_paths_bits(case_name, impl, noise_std):
    from oracle import nerf_oracle as O
    from nerf_pytorch_b200 import ops

    nb = _nb()
    c = Case(case_name)
    mc, _, epf, edf = build_models(c)
    nc = 64
    opts = O.make_options(use_viewdirs=c.use_viewdirs, no_ndc=True, near=2.0, far=6.0, num_coarse=nc, num_fine=0,
                          perturb=False, radiance_field_noise_std=noise_std)
    ro, rd = c.ro.reshape(-1, 3).cuda(), c.rd.reshape(-1, 3).cuda()
    rays = ops.pack_rays(ro, rd, c.H, c.W, c.focal, False, 2.0, 6.0, c.use_viewdirs)
    n = rays.shape[0]
    noise = torch.randn(n, nc, generator=torch.Generator().manual_seed(11)).cuda()
    rnd = {"noise_c": noise} if noise_std > 0 else {}
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(12)).cuda()
    train = impl != ops.IMPL_TC_FAST
    ctx = (case_name, impl, noise_std)

    def loss_of(rgb, acc):
        return torch.nn.functional.mse_loss(rgb, target) + 0.1 * acc.mean()

    with torch.set_grad_enabled(train):
        want = nb.predict_and_render_radiance(rays, mc, None, opts, encode_position_fn=epf, encode_direction_fn=edf,
                                              randoms=rnd, impl=impl)
        if train:
            loss_of(want[0], want[2]).backward()
            g_want = {k: p.grad.clone() for k, p in mc.named_parameters()}
            mc.zero_grad()
        z = ops.sample_coarse(rays, None, nc, False, False)
        pts = rays[:, None, :3] + rays[:, None, 3:6] * z[..., None]  # pts = ro + rd * z: one mul, one add
        raw = nb.run_network(mc, pts, rays, 1024, epf, edf if c.use_viewdirs else None, impl=impl)
        rgb, disp, acc, weights, depth = nb.volume_render_radiance_field(raw, z, rays[:, 3:6], noise_std, False,
                                                                         noise=noise)
        for name, a, b in (("rgb", rgb, want[0]), ("disp", disp, want[1]), ("acc", acc, want[2])):
            assert bits_equal(a, b), ctx + (name,)
        if not train:
            return
        loss_of(rgb, acc).backward()
    for k, p in mc.named_parameters():
        if impl == ops.IMPL_TC:  # fixed-point sums: the same bits
            assert torch.equal(p.grad, g_want[k]), ctx + (k,)
        else:                    # fp32 atomics: the summation order differs
            e = (p.grad - g_want[k]).abs().max().item()
            assert e <= 1e-6 * g_want[k].abs().max().item(), ctx + (k, e)


# ------------------------------------------------------------------------------------------------------------------------
# 2. run_network at points off any ray against fp64
# ------------------------------------------------------------------------------------------------------------------------
def _box_points(arch, lead, s, seed):
    """pts (*lead, s, 3) uniform in [-1.5, 1.5]^3, unit view directions (*lead, 11) rows (last three columns), and the
    same samples as one-point "rays" [pts, 0, 0, 0, 2, 6, dir] with z = 0 for mlp_checks' oracle (pts + 0 * 0 = pts)."""
    g = torch.Generator().manual_seed(seed)
    n = math.prod(lead)
    pts = torch.rand(n, s, 3, generator=g) * 3.0 - 1.5
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1)
    ray_batch = torch.cat([torch.randn(n, 8, generator=g), d], -1)
    per_point = torch.cat([pts.reshape(-1, 3), torch.zeros(n * s, 3), torch.full((n * s, 1), 2.0),
                           torch.full((n * s, 1), 6.0), d[:, None, :].expand(n, s, 3).reshape(-1, 3)], -1)
    if not arch.use_viewdirs:
        per_point = per_point[:, :8]
    return (pts.reshape(*lead, s, 3), ray_batch.reshape(*lead, 11), per_point.contiguous(), torch.zeros(n * s, 1))


FWD_SHAPES = [((n,), s) for n, s in SHAPES] + [((1,), 100000), ((2, 3, 4), 16)]
# hidden 128 on both kernel families, hidden-128 encodings that only the fp32 kernels take, hidden 256
NAMES = ([f"h128_{k}" for k in ALL_ARCHS] + [f"h128_{k}" for k in SIMT128_ARCHS if k not in ALL_ARCHS]
         + [f"h256_{k}" for k in H256_ARCHS])


@pytest.mark.parametrize("shape", FWD_SHAPES, ids=lambda s: "x".join(map(str, s[0] + (s[1],))))
@pytest.mark.parametrize("name", NAMES)
def test_run_network_forward_matches_fp64_at_points_off_any_ray(name, shape):
    from nerf_pytorch_b200 import ops

    nb = _nb()
    arch = spec(name.split("_", 1)[1])
    sd = arch_weights(arch, "init")
    lead, s = shape
    pts, ray_batch, per_point, z0 = _box_points(arch, lead, s, seed=21)
    want = oracle(arch, sd, per_point, z0)[0]
    scale = want.abs().amax(0)
    model, epf, edf = _model(arch, sd)
    impls = [(ops.IMPL_SIMT, SIMT_FWD_TOL)]
    if ops.impl_supported(arch, s, ops.IMPL_TC_FWD):
        impls += [(ops.IMPL_TC, TC_FWD_TOL), (ops.IMPL_TC_FAST, FAST_TOL)]
    with torch.no_grad():
        for impl, tol in impls:
            raw = nb.run_network(model, pts.cuda(), ray_batch.cuda(), 4096, epf, edf, impl=impl)
            assert raw.shape == pts.shape[:-1] + (4,) and raw.dtype == torch.float32
            e = ((raw.reshape(-1, 4).double().cpu() - want).abs().amax(0) / scale).max().item()
            report(f"run_network forward impl={impl}", (name, shape), e)
            assert e <= tol, (name, shape, impl, e)


# each architecture on the kernels that train it
GRAD_CASES = ([(f"h128_{k}", 1) for k in TC_ARCHS] + [(f"h128_{k}", 0) for k in SIMT128_ARCHS]
              + [(f"h256_{k}", 0) for k in H256_ARCHS])


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("name, impl", GRAD_CASES)
def test_run_network_parameter_gradients_match_fp64_per_block(name, impl, shape):
    nb = _nb()
    arch = spec(name.split("_", 1)[1])
    sd = arch_weights(arch, "init")
    n, s = shape
    pts, ray_batch, per_point, z0 = _box_points(arch, (n,), s, seed=31)
    G = upstream(n * s, 1, seed=32).reshape(n, s, 4)
    _, acts, dpre, want = oracle(arch, sd, per_point, z0, G)
    model, epf, edf = _model(arch, sd)
    raw = nb.run_network(model, pts.cuda(), ray_batch.cuda(), 4096, epf, edf, impl=impl)
    (raw * G.cuda()).sum().backward()
    got = _flat_grad(arch, model)
    split = _split_floors(arch, G, acts, dpre, per_point, z0) if impl == 1 else None
    check_blocks(arch, got, want, tc_blocks(arch), BLOCK_TOL, (name, impl, shape), "run_network gradient blocks",
                 _floors(arch, n * s, split))


# ------------------------------------------------------------------------------------------------------------------------
# 3. view directions in place from any row layout
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", [0, 1])
def test_view_directions_are_read_from_the_last_three_columns_of_any_rows(impl):
    nb = _nb()
    arch = spec("8x128_widest")
    model, epf, edf = _model(arch, arch_weights(arch, "init"))
    g = torch.Generator().manual_seed(41)
    n, s = 37, 33
    pts = (torch.rand(n, s, 3, generator=g) * 3 - 1.5).cuda()
    d = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1).cuda()
    wide = torch.cat([torch.randn(n, 5, generator=g).cuda(), d, torch.randn(n, 4, generator=g).cuda()], -1)
    layouts = {"3": d.clone(), "11": torch.cat([torch.randn(n, 8).cuda(), d], -1),
               "14": torch.cat([torch.randn(n, 11).cuda(), d], -1), "slice": wide[:, 2:8]}
    assert not layouts["slice"].is_contiguous()
    G = torch.randn(n, s, 4, generator=g).cuda()
    outs, grads = {}, {}
    for k, rb in layouts.items():
        model.zero_grad()
        raw = nb.run_network(model, pts, rb, 1024, epf, edf, impl=impl)
        (raw * G).sum().backward()
        outs[k], grads[k] = raw.detach(), _flat_grad(arch, model)
    for k in layouts:
        assert bits_equal(outs[k], outs["3"]), k
        if impl == 1:
            assert torch.equal(grads[k], grads["3"]), k


# ------------------------------------------------------------------------------------------------------------------------
# 4. volume_render_radiance_field against fp64
# ------------------------------------------------------------------------------------------------------------------------
def _comp_inputs(n, s, seed, empty_rays=0):
    g = torch.Generator().manual_seed(seed)
    raw = torch.randn(n, s, 4, generator=g) * 2
    raw[:, 0, 3] = raw[:, 0, 3].abs() + 2.0  # every ray holds some density (else its disp is NaN)
    if empty_rays:
        raw[:empty_rays, :, 3] = -50.0  # no density: acc = 0, disp NaN as in the reference
    z = torch.sort(torch.rand(n, s, generator=g) * 4 + 2, -1).values
    dirs = torch.randn(n, 3, generator=g)
    noise = torch.randn(n, s, generator=g)
    return raw, z, dirs, noise


def _trained_inputs(n, s, seed):
    """Samples as a trained network makes them (raw sigma at 1e2 .. 1e4, surfaces, merged depths clustering there):
    sigma * delta log-uniform over 1e-3 .. 1e3; a run of six samples at sigma * delta = 1e3 where the ray has room
    (alpha rounds to 1 in fp32 and q to 1e-10, so T passes through the fp32 subnormals to 0); exact duplicate depths
    (delta = 0); a last sample (delta = 1e10) with a tiny positive sigma, sigma * 1e10 |d| in 1e-2 .. 3, and no noise
    so that it stays so.  The first sample's sigma is at least 3, so that no ray is empty."""
    g = torch.Generator().manual_seed(seed)
    z = torch.sort(torch.rand(n, s, generator=g) * 4 + 2, -1).values
    if s >= 3:  # z[j + 1] = z[j] for some j >= 1, from the old values: z stays sorted
        z[:, 2:] = torch.where(torch.rand(n, s - 2, generator=g) < 0.05, z[:, 1:-1], z[:, 2:])
    if s >= 4:
        z[:, s // 2] = z[:, s // 2 - 1]
    dirs = torch.randn(n, 3, generator=g)
    dnorm = dirs.norm(dim=-1, keepdim=True)
    x = 10.0 ** (torch.rand(n, s, generator=g) * 6 - 3)
    if s >= 10:
        k = torch.randint(1, s - 7, (n, 1), generator=g)
        j = torch.arange(s)[None]
        x = torch.where((j >= k) & (j < k + 6), 1e3, x)
    sigma = x[:, :-1] / ((z[:, 1:] - z[:, :-1]) * dnorm).clamp_min(1e-6)  # delta = 0: alpha is 0 whatever sigma
    sigma[:, 0] = sigma[:, 0].clamp_min(3.0)
    last = 10.0 ** (torch.rand(n, 1, generator=g) * 2.5 - 2) / (1e10 * dnorm)
    raw = torch.randn(n, s, 4, generator=g) * 2
    raw[..., 3] = torch.cat((sigma, last), -1)
    noise = torch.randn(n, s, generator=g)
    noise[:, -1] = 0.0
    return raw, z, dirs, noise


# "random": raw ~ 2 N(0, 1); "trained": the saturated regime of _trained_inputs, also at 199 samples (not a multiple of
# the warp's 32 lanes).  The random regime keeps its original test ids.  The kernels' lane L owns samples [L C, (L + 1) C)
# with C = ceil(S / 32): 1 and 31 samples leave lanes idle, 33 gives lane 16 a single sample and 1023 leaves lane 31 one
# short of 32.
COMP_REGIMES = ([("random", s) for s in (2, 64, 192, 1024, 1, 31, 33, 1023)] +
                [("trained", s) for s in (2, 64, 192, 199, 1024, 31, 33, 1023)])
COMP_IDS = [str(s) if r == "random" else f"{r}-{s}" for r, s in COMP_REGIMES]


@pytest.mark.parametrize("regime, s", COMP_REGIMES, ids=COMP_IDS)
@pytest.mark.parametrize("white", [False, True])
@pytest.mark.parametrize("noise_std", [0.0, 0.3])
def test_volume_render_outputs_and_gradients_match_fp64(regime, s, white, noise_std):
    from oracle import nerf_oracle as O

    nb = _nb()
    n = 37
    raw, z, dirs, noise = (_comp_inputs if regime == "random" else _trained_inputs)(n, s, seed=51 + s)
    raw64 = raw.double().requires_grad_(True)
    want = composite64(raw, z, dirs, noise_std, white, noise, raw64=raw64)
    raw_c = raw.cuda().requires_grad_(True)
    got = nb.volume_render_radiance_field(raw_c, z.cuda(), dirs.cuda(), noise_std, white, noise=noise.cuda())
    ctx = (regime, s, white, noise_std)
    names = ("rgb", "disp", "acc", "weights", "depth")
    for name, a, b in zip(names, got, want):
        assert a.shape == b.shape and a.dtype == torch.float32, ctx + (name,)
        e = (a.double().cpu() - b.detach()).abs().max().item()
        report(f"volume_render {name}", ctx, e / b.abs().max().item())
        assert e <= COMP_TOL * b.abs().max().item(), ctx + (name, e)
    gen = torch.Generator().manual_seed(52)
    ups = [torch.randn(b.shape, generator=gen, dtype=torch.float64) for b in want]
    sum(((b * u).sum() for b, u in zip(want, ups))).backward()
    sum(((a * u.float().cuda()).sum() for a, u in zip(got, ups))).backward()
    scale = raw64.grad.abs().max().item()
    e = (raw_c.grad.double().cpu() - raw64.grad).abs().max().item()
    report("volume_render d_raw", ctx, e / scale)
    assert e <= COMP_GRAD_TOL * scale, ctx + (e, scale)
    # each output alone, the two the render backward never took (weights and depth) included.  In the trained regime the
    # gradient of acc alone is cancellation: on an opaque ray acc = 1 - T_end is flat in every sigma (d acc / d sigma_i
    # ~ T_end ~ 0) while the terms that cancel are ~T_i, so no fp32 evaluation resolves it; there the bar adds
    # REF32_FACTOR x the error of the fp32 reference itself (O.volume_render_radiance_field in fp32 autograd, 1.5e2 ..
    # 5.5e2 x the gradient's scale; the kernel's is at most 2.0 x the reference's, on an H100 80GB HBM3 at 700 W).
    for i, name in enumerate(names):
        raw64.grad = raw_c.grad = None
        w64 = composite64(raw, z, dirs, noise_std, white, noise, raw64=raw64)
        wc = nb.volume_render_radiance_field(raw_c, z.cuda(), dirs.cuda(), noise_std, white, noise=noise.cuda())
        (w64[i] * ups[i]).sum().backward()
        (wc[i] * ups[i].float().cuda()).sum().backward()
        scale = raw64.grad.abs().max().item()
        e = (raw_c.grad.double().cpu() - raw64.grad).abs().max().item()
        e_ref = 0.0
        if regime == "trained":
            r32 = raw.clone().requires_grad_(True)
            w32 = O.volume_render_radiance_field(r32, z, dirs, noise_std, white, noise=noise)
            (w32[i] * ups[i].float()).sum().backward()
            e_ref = (r32.grad.double() - raw64.grad).abs().max().item()
            report(f"volume_render d_raw of {name} alone / (bar + fp32 reference's error)", ctx,
                   e / (COMP_GRAD_TOL * scale + REF32_FACTOR * e_ref))
        assert e <= COMP_GRAD_TOL * scale + REF32_FACTOR * e_ref, ctx + (name, e, scale, e_ref)


def test_volume_render_empty_rays_give_the_references_nan_disparity():
    from oracle import nerf_oracle as O

    nb = _nb()
    raw, z, dirs, _ = _comp_inputs(16, 64, seed=61, empty_rays=5)
    want = O.volume_render_radiance_field(raw.double(), z.double(), dirs.double())
    got = nb.volume_render_radiance_field(raw.cuda(), z.cuda(), dirs.cuda())
    assert torch.equal(torch.isnan(got[1]).cpu(), torch.isnan(want[1]))
    assert torch.isnan(got[1][:5]).all() and (got[2][:5] == 0).all()


def test_volume_render_default_noise_is_the_references_torch_randn_draw():
    nb = _nb()
    raw, z, dirs, _ = _comp_inputs(33, 64, seed=71)
    raw, z, dirs = raw.cuda(), z.cuda(), dirs.cuda()
    torch.manual_seed(5)
    drawn = nb.volume_render_radiance_field(raw, z, dirs, 0.5, True)
    torch.manual_seed(5)
    noise = torch.randn(raw[..., 3].shape, dtype=raw.dtype, device=raw.device)
    injected = nb.volume_render_radiance_field(raw, z, dirs, 0.5, True, noise=noise)
    for a, b in zip(drawn, injected):
        assert bits_equal(a, b)


def test_volume_render_any_leading_shape():
    nb = _nb()
    raw, z, dirs, noise = _comp_inputs(24, 32, seed=81)
    flat = nb.volume_render_radiance_field(raw.cuda(), z.cuda(), dirs.cuda(), 0.2, False, noise=noise.cuda())
    shaped = nb.volume_render_radiance_field(raw.view(2, 3, 4, 32, 4).cuda(), z.view(2, 3, 4, 32).cuda(),
                                             dirs.view(2, 3, 4, 3).cuda(), 0.2, False,
                                             noise=noise.view(2, 3, 4, 32).cuda())
    for a, b in zip(flat, shaped):
        assert b.shape[:3] == (2, 3, 4) and bits_equal(a, b.reshape(a.shape))


# ------------------------------------------------------------------------------------------------------------------------
# 5. density grid
# ------------------------------------------------------------------------------------------------------------------------
def test_density_grid_query_without_rows_stays_on_the_wgmma_kernels():
    nb = _nb()
    c = Case("lego_a0_train")
    mc, _, epf, edf = build_models(c)
    t = torch.linspace(-1.5, 1.5, 128, device="cuda")
    grid = torch.stack(torch.meshgrid(t, t, t, indexing="ij"), -1).reshape(1, -1, 3)
    view = torch.tensor([[0.0, 0.0, 1.0]], device="cuda")
    with torch.no_grad():
        auto = nb.run_network(mc, grid, view, 65536, epf, edf)
        tc = nb.run_network(mc, grid, view, 65536, epf, edf, impl=1)
        simt = nb.run_network(mc, grid, view, 65536, epf, edf, impl=0)
    assert auto.shape == (1, 128 ** 3, 4)
    assert bits_equal(auto, tc)
    assert not bits_equal(tc, simt)  # the two families round differently: the check above can tell them apart


# ------------------------------------------------------------------------------------------------------------------------
# 6. gradient sync
# ------------------------------------------------------------------------------------------------------------------------
def test_run_network_backward_leaves_the_reduction_to_fused_adam(tmp_path):
    import torch.distributed as dist
    from nerf_pytorch_b200 import parallel, train_utils

    nb = _nb()
    dist.init_process_group("gloo", store=dist.FileStore(str(tmp_path / "store"), 1), rank=0, world_size=1)
    try:
        parallel.enable_gradient_sync()
        c = Case("lego_a0_train")
        mc, _, epf, edf = build_models(c)
        opt = parallel.FusedAdam([(mc, train_utils._arch_of(mc, c.enc_xyz, c.enc_dir))])
        pts = torch.rand(8, 32, 3, device="cuda")
        rays = torch.randn(8, 11, device="cuda")
        nb.run_network(mc, pts, rays, 1024, epf, edf).square().sum().backward()
        assert train_utils._PENDING_SYNC
        before = [p.detach().clone() for p in mc.parameters()]
        opt.step()
        assert not train_utils._PENDING_SYNC
        assert any(not torch.equal(a, p) for a, p in zip(before, mc.parameters()))
    finally:
        parallel.disable_gradient_sync()
        dist.destroy_process_group()
