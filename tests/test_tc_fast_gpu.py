"""GPU: the single-pass fp16 wgmma forward (impl 3, ops.IMPL_TC_FAST), the inference-only forward that issues one
fp16(w) x fp16(activation / 16) product per k-step with fp32 accumulation instead of impl 1's three-term split.
  1. raw outputs against fp64 and against an fp64 oracle that rounds each gemm layer's weights and its input / 16 to
     fp16 as the kernel does, over the hidden-128 and hidden-256 architectures of mlp_checks.py;
  2. PSNR of whole renders of the shipped lego and fern checkpoints, fast against impl 1;
  3. bit-identical repeats, chunkings and seeded renders;
  4. the refusals: anything that trains, and every configuration the wgmma inference forward refuses;
  5. out-of-range operands give inf / NaN, not a finite wrong value.

Bars: each is below 10x the worst figure measured on an H100 over every parameter set (figures beside the constants);
the PSNR bars are 3 dB under the H100 figure.  Run with -s to print the measured figures."""
import pytest
import torch

from helpers import OUT_NAMES, bits_equal, psnr64, scene_pose, shipped_models
from mlp_checks import (ALL_ARCHS, H256_ARCHS, SHAPES, STATES, TC_FWD_TOL, arch_weights, encodings, oracle, points,
                        report, sms_shape, spec)

pytestmark = pytest.mark.gpu

# Worst raw element per output column as a fraction of the column's scale.  Measured on an H100 80GB HBM3, worst over
# all parameter sets and both weight states, in brackets.
FAST_TOL = 2e-2        # against fp64 [6.7e-3]
EMU_WORST = 1e-2       # against the fp16-rounding oracle, every point [4.2e-3]
# fp16 rounding-tie flips: the kernel rounds its fp32 activation, the oracle its fp64 one, to fp16; where the two sit on
# either side of a rounding boundary the operand differs by one fp16 ulp (2^-11 of it), and everything downstream
# moves.  The fp32 accumulation differs from fp64 by ~1e-7 of an activation, so each of the ~10^3 operands per point
# flips with probability ~1e-4..1e-3: a point without a flip agrees with the oracle to EMU_TOL, and the test allows
# at most FLIP_FRAC[state] of the points beyond it.  The scaled weights (activations up to 1e4, deeper networks) flip
# most often.
EMU_TOL = 1e-4
FLIP_FRAC = {"init": 0.35, "scaled": 0.8}  # fraction of points beyond EMU_TOL [0.20, 0.60 (9 of 15 points)]

# every architecture of mlp_checks the wgmma inference forward takes (8x256_ldir6's 39 direction channels are > 32)
ARCHS = [f"h128_{k}" for k in ALL_ARCHS] + [f"h256_{k}" for k in H256_ARCHS if k != "8x256_ldir6"]
FWD_SHAPES = SHAPES + [("sms+1", 128)]  # the last: more tiles than SMs, so one CTA runs two


def _f16(x):
    """fp64 -> fp16 -> fp64: one rounding to nearest even, inf beyond the fp16 range (as the kernel's conversions)."""
    return x.half().double()


def _oracle_fp16(arch, sd, rays, z):
    """fp64 raw [P][4] of the network with every gemm layer computing fp16(input / 16) * 16 @ fp16(W)^T + b: the
    single-pass kernel's operands.  The heads (fc_alpha, fc_rgb, fc_out) and the direction-encoding columns of
    layers_dir.0 take fp64 inputs and weights, as the kernel's fp32 register dot products and per-ray bias do."""
    H = arch.hidden
    sd = {k: v.double() for k, v in sd.items()}
    xyz, view = encodings(arch, rays, z)  # of the fp32 points, as the kernel forms them

    def gemm(x, w):
        return (_f16(x / 16) * 16) @ _f16(w).T

    def layer(x, name):
        return gemm(x, sd[name + ".weight"]) + sd[name + ".bias"]

    def head(x, name):
        return x @ sd[name + ".weight"].T + sd[name + ".bias"]

    h = layer(xyz, "layer1")
    for i in range(arch.num_layers - 1):
        name = f"layers_xyz.{i}"
        if sd[name + ".weight"].shape[1] == H + arch.dim_xyz:
            h = torch.cat((h, xyz), -1)
        h = torch.relu(layer(h, name))
    if not arch.use_viewdirs:
        return head(h, "fc_out")
    feat = torch.relu(layer(h, "fc_feat"))
    w = sd["layers_dir.0.weight"]
    d = torch.relu(gemm(feat, w[:, :H]) + view @ w[:, H:].T + sd["layers_dir.0.bias"])
    return torch.cat((head(d, "fc_rgb"), head(h, "fc_alpha")), -1)


# ------------------------------------------------------------------------------------------------------------------------
# 1. forward against fp64 and against the fp16-rounding oracle
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("shape", FWD_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("name", ARCHS)
def test_fast_forward_matches_fp64_and_fp16_oracle(name, shape, state):
    from nerf_pytorch_b200 import ops

    arch = spec(name.split("_", 1)[1])
    sd = arch_weights(arch, state)
    rays, z = points(arch, *sms_shape(shape), seed=1)
    blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))
    ctx = (name, state, tuple(z.shape))
    assert ops.impl_supported(arch, z.shape[1], ops.IMPL_TC_FAST)
    fast = ops.mlp_fwd(arch, blob, rays.cuda(), z.cuda(), impl=ops.IMPL_TC_FAST)
    tc = ops.mlp_fwd(arch, blob, rays.cuda(), z.cuda(), impl=ops.IMPL_TC)
    torch.cuda.synchronize()
    got = fast.reshape(-1, 4).double().cpu()
    assert torch.isfinite(got).all(), ctx

    want = oracle(arch, sd, rays, z)[0]
    scale = want.abs().amax(0)
    e64 = ((got - want).abs().amax(0) / scale).max().item()
    report("fast vs fp64", ctx, e64)
    assert e64 <= FAST_TOL, ctx + (e64,)

    emu = _oracle_fp16(arch, sd, rays, z)
    rel = ((got - emu).abs() / scale).amax(1)  # per point, worst column
    flipped = rel > EMU_TOL
    n_flip = int(flipped.sum())
    worst_rest = rel[~flipped].max().item() if n_flip < rel.numel() else 0.0
    report("fast vs fp16 oracle: worst unflipped point", ctx, worst_rest)
    report("fast vs fp16 oracle: fraction of points beyond EMU_TOL", ctx, n_flip / rel.numel())
    report("fast vs fp16 oracle: worst point", ctx, rel.max().item())
    assert n_flip <= FLIP_FRAC[state] * rel.numel(), ctx + (n_flip, rel.numel())
    assert rel.max().item() <= EMU_WORST, ctx + (rel.max().item(),)

    # the single-pass kernel ran: its output is NOT within impl 1's parity bar
    e_tc = ((tc.reshape(-1, 4).double().cpu() - got).abs().amax(0) / scale).max().item()
    report("fast vs impl 1", ctx, e_tc)
    if state == "scaled":
        assert e_tc > TC_FWD_TOL, ctx + (e_tc,)


# ------------------------------------------------------------------------------------------------------------------------
# 2. PSNR of whole renders of the shipped checkpoints
# ------------------------------------------------------------------------------------------------------------------------
# fast against impl 1 on the same rays, dB; each bar 3 dB under the H100 figure in brackets.
PSNR_BARS = {
    ("lego", "rgb_fine"): 46.9,    # [49.92; max abs 0.34, 0.47 % of pixels off by more than 1/255]
    ("lego", "rgb_coarse"): 55.0,  # [58.03; max abs 0.046, 0.76 %]
    ("fern", "rgb_fine"): 62.4,    # [65.48; max abs 0.020, 0.34 %]
    ("fern", "rgb_coarse"): 71.2,  # [74.20; max abs 0.0037, 0 %]
}
# (H, W, focal, pose, no_ndc, near, far) of the shipped scenes: lego at pose_spherical(30, -30, 4); fern forward-facing
# in NDC
VIEWS = {
    "lego": (100, 100, 138.89, "spherical", True, 2.0, 6.0),
    "fern": (63, 84, 67.9, "eye", False, 0.0, 1.0),
}


def _render(view, impl, perturb=False, noise=0.0, chunk=None, randoms=None):
    """render_image of a shipped A0 checkpoint.  The options set train and validation alike, so the render is the same
    whether train_utils.COMPAT_MODE_QUIRK sends it to options.nerf.train (the reference's behaviour) or not."""
    import nerf_pytorch_b200 as nb
    from oracle import nerf_oracle as O

    H, W, focal, pose, no_ndc, near, far = VIEWS[view]
    mc, mf, epf, edf = shipped_models(view)
    opts = O.make_options(no_ndc=no_ndc, near=near, far=far, num_coarse=64, num_fine=128, perturb=perturb,
                          radiance_field_noise_std=noise)
    return nb.render_image(H, W, focal, scene_pose(pose), mc, mf, opts, mode="validation", encode_position_fn=epf,
                           encode_direction_fn=edf, rays_per_chunk=chunk or H * W, impl=impl, randoms=randoms)


@pytest.mark.parametrize("view", list(VIEWS))
def test_fast_render_psnr_against_impl1(view):
    from nerf_pytorch_b200 import ops

    ref = _render(view, ops.IMPL_TC)
    fast = _render(view, ops.IMPL_TC_FAST)
    torch.cuda.synchronize()
    for out in ("rgb_fine", "rgb_coarse"):
        i = OUT_NAMES.index(out)
        a, b = fast[i], ref[i]
        assert torch.isfinite(a).all(), (view, out)
        p = psnr64(a, b)
        d = (a - b).abs()
        report(f"PSNR dB fast vs impl 1 {out}", (view,), p)
        report(f"max abs fast vs impl 1 {out}", (view,), d.max().item())
        report(f"fraction of pixels off by > 1/255 {out}", (view,), (d.amax(-1) > 1 / 255).double().mean().item())
        assert p >= PSNR_BARS[(view, out)], (view, out, p)
    assert PSNR_BARS[("lego", "rgb_fine")] >= 45.0


# ------------------------------------------------------------------------------------------------------------------------
# 3. determinism and chunking
# ------------------------------------------------------------------------------------------------------------------------
def _same_bits(x, y):
    return all(bits_equal(a, b) for a, b in zip(x, y))


def test_fast_render_is_bit_reproducible_and_chunking_invariant():
    """Two identical fast renders, a 4096-ray chunking and a whole-image chunk give the same bits; so does a seeded
    render with perturb and noise on, whatever the chunking."""
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    first = _render("lego", ops.IMPL_TC_FAST)
    again = _render("lego", ops.IMPL_TC_FAST)
    chunked = _render("lego", ops.IMPL_TC_FAST, chunk=4096)
    assert _same_bits(first, again)
    assert _same_bits(first, chunked)

    rng = nb.SeededRandoms(11, 3)
    s_whole = _render("lego", ops.IMPL_TC_FAST, perturb=True, noise=0.5, randoms=rng)
    s_chunk = _render("lego", ops.IMPL_TC_FAST, perturb=True, noise=0.5, chunk=4096, randoms=rng)
    s_again = _render("lego", ops.IMPL_TC_FAST, perturb=True, noise=0.5, randoms=rng)
    assert _same_bits(s_whole, s_chunk) and _same_bits(s_whole, s_again)
    assert not torch.equal(s_whole[3], first[3])  # the seeded jitter and noise did act


# ------------------------------------------------------------------------------------------------------------------------
# 4. refusals
# ------------------------------------------------------------------------------------------------------------------------
def test_training_with_the_fast_forward_raises_before_any_launch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    mc, mf, epf, edf = shipped_models("lego")
    opts = O.make_options(num_coarse=64, num_fine=64)
    g = torch.Generator().manual_seed(3)
    ro = torch.nn.functional.normalize(torch.randn(256, 3, generator=g), dim=-1).cuda() * 4.0
    rd = -ro / 4.0
    kw = dict(encode_position_fn=epf, encode_direction_fn=edf)
    torch.cuda.synchronize()
    before = ops.launch_count()
    with pytest.raises(NotImplementedError, match="inference"):
        nb.run_one_iter_of_nerf(100, 100, 120.0, mc, mf, ro, rd, opts, impl=ops.IMPL_TC_FAST, **kw)
    with pytest.raises(NotImplementedError, match="inference"):
        nb.run_one_iter_of_nerf_from_pose(100, 100, 120.0, mc, mf, torch.eye(4), None, opts, impl=ops.IMPL_TC_FAST,
                                          **kw)
    assert ops.launch_count() == before
    with torch.no_grad():  # the same call without training renders
        out = nb.run_one_iter_of_nerf(100, 100, 120.0, mc, mf, ro, rd, opts, impl=ops.IMPL_TC_FAST, **kw)
    assert ops.launch_count() > before and torch.isfinite(out[3]).all()


def test_library_refuses_the_fast_forward_wherever_it_would_train():
    """mlp_fwd with a stash, render_fwd(training=True), render_bwd, mlp_bwd, mlp_dgrad and mlp_wgrad with impl 3 raise
    NotImplementedError naming inference; an impl 1 forward is bit-identical before and after the refusals."""
    from nerf_pytorch_b200 import ops

    arch = ops.ArchSpec(num_layers=4, hidden=128, n_freq_xyz=10)
    sd = arch_weights(arch, "init")
    blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))
    rays, z = points(arch, 64, 64, seed=2)
    rays, z = rays.cuda(), z.cuda()
    before = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC)
    _, stash = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC, want_stash=True)
    d_raw = torch.ones(64, 64, 4, device="cuda")
    opts = ops.make_opts(64, 64, False, False, False, 0.0)
    with pytest.raises(NotImplementedError, match="inference"):
        ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC_FAST, want_stash=True)
    with pytest.raises(NotImplementedError, match="inference"):
        ops.render_fwd(arch, arch, opts, blob, blob, rays, {}, training=True, impl=ops.IMPL_TC_FAST)
    _, _, ws = ops.render_fwd(arch, arch, opts, blob, blob, rays, {}, training=True, impl=ops.IMPL_TC)
    g = torch.zeros(64, 8, device="cuda")
    fg = torch.zeros(arch.flat_param_count(), device="cuda")
    with pytest.raises(NotImplementedError, match="inference"):
        ops.render_bwd(arch, arch, opts, blob, blob, rays, {}, g, g, ws, fg, fg.clone(), impl=ops.IMPL_TC_FAST)
    with pytest.raises(NotImplementedError, match="inference"):
        ops.mlp_bwd(arch, blob, rays, z, d_raw, stash, impl=ops.IMPL_TC_FAST)
    with pytest.raises(NotImplementedError, match="inference"):
        ops.mlp_dgrad(arch, blob, d_raw, stash, impl=ops.IMPL_TC_FAST)
    with pytest.raises(NotImplementedError, match="inference"):
        ops.mlp_wgrad(arch, rays, z, d_raw, stash, stash, impl=ops.IMPL_TC_FAST)
    after = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC)
    torch.cuda.synchronize()
    assert torch.equal(before, after)


def test_fast_forward_is_refused_where_the_wgmma_inference_forward_is():
    """14 samples per ray and an xyz encoding 72 wide (L_xyz 11 without input): impl_supported says no for 2 and 3
    alike, and mlp_fwd refuses impl 3 for the reason it refuses impl 1.  The shared-memory depth limit of the forward
    is not reachable within the 16 layers the library accepts (test_tc_fast_host_cpu.py sweeps the query)."""
    from nerf_pytorch_b200 import ops

    arch = ops.ArchSpec(num_layers=4, hidden=128, n_freq_xyz=6)
    blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, arch_weights(arch, "init"), "cuda"))
    rays, z = points(arch, 9, 14, seed=12)
    rays, z = rays.cuda(), z.cuda()
    wide = ops.ArchSpec(num_layers=4, hidden=128, n_freq_xyz=11, include_input_xyz=False)
    blob_w = ops.pack_weights(wide, torch.zeros(wide.flat_param_count(), device="cuda"))
    z64 = points(wide, 9, 64, seed=13)[1].cuda()
    before = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_SIMT)
    for a, b, zz, reason in ((arch, blob, z, "fewer than 15 samples"), (wide, blob_w, z64, "wider than 64")):
        assert not ops.impl_supported(a, zz.shape[1], ops.IMPL_TC_FWD)
        assert not ops.impl_supported(a, zz.shape[1], ops.IMPL_TC_FAST)
        msgs = []
        for impl in (ops.IMPL_TC, ops.IMPL_TC_FAST):
            with pytest.raises(NotImplementedError, match=reason) as err:
                ops.mlp_fwd(a, b, rays, zz, impl=impl)
            msgs.append(str(err.value).split("): ", 1)[1])
        assert msgs[0] == msgs[1], msgs
    after = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_SIMT)
    torch.cuda.synchronize()
    assert torch.equal(before, after)


# ------------------------------------------------------------------------------------------------------------------------
# 5. range
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("what", ["activation", "weight"])
def test_fast_out_of_range_operands_are_visible_not_clamped(what):
    """|activation| >= 1.05e6 (value / 16 beyond fp16) or |weight| >= 32 (the hs = fp16(w) 2^11 copy overflows) turns
    the output into inf / NaN; the unmodified network and a weight of 31 give finite outputs."""
    from nerf_pytorch_b200 import ops

    arch = ops.ArchSpec(num_layers=4, hidden=128, n_freq_xyz=10)
    sd = arch_weights(arch, "init")
    rays, z = points(arch, 64, 64, seed=5)
    rays, z = rays.cuda(), z.cuda()
    flat = ops.flatten_state_dict(arch, sd, "cuda")
    layout = {name: (w_off, b_off, fin, fout) for name, w_off, b_off, fin, fout in arch.flat_layout()}
    w_off, b_off, fin, fout = layout["layer1" if what == "activation" else "layers_xyz.0"]
    for bad in (False, True):
        f2 = flat.clone()
        if what == "activation" and bad:  # layer1's biases at 2e6 (they stay fp32): its output beyond 1.05e6
            f2[b_off:b_off + fout] = 2e6
        if what == "weight":  # one weight of layers_xyz.0 at 31 (in range) or 33
            f2[w_off] = 33.0 if bad else 31.0
        raw = ops.mlp_fwd(arch, ops.pack_weights(arch, f2), rays, z, impl=ops.IMPL_TC_FAST)
        torch.cuda.synchronize()
        if bad:
            assert not torch.isfinite(raw).all(), what
        else:
            assert torch.isfinite(raw).all(), what
