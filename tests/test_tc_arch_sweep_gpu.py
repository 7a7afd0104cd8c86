"""GPU: the wgmma forward and fused backward at hidden 128, across the architectures and sample counts they accept,
against fp64 autograd of the oracle MLP, block by block.

Every hidden-128 model trains on these kernels by default (train_utils._auto_impl), so every architecture family that
bwd_tc_supported accepts gets its own job table (make_bwd_plan), gradient-blob layout (blob_map) and unpack mapping.  The
sweep reaches what the golden cases do not:
  * 1 layer (the heads and fc_feat read layer1's output, which has no ReLU), 16 layers (18 gemm layers), up to four wide
    (skip) layers, a wide layer every 1, 2, 3, 4 or 5 layers;
  * xyz-encoding operand tiles 16 wide (3 and 9 channels) and 64 wide (60 and 63 channels), linear bands without the raw
    input, direction encodings of 3, 9, 15, 24 and 27 channels;
  * 15 samples per ray, where one 128-point tile spans 10 rays: every ray slot of the backward's indicator tile, s_encd
    and s_sums (and of the forward's per-ray view bias);
  * persistent CTAs that run several tiles: one CTA with two tiles (sms + 1 rays x 128), about four per CTA (8 sms rays
    x 64) and tiles inside one ray (3 x 1024, the renderer's largest sample count).
Checks, each printed with -s:
  1. forward, stash-writing and inference: raw outputs per column, every layer's stashed activation tile, the xyz-encoding
     tile (padding included) and the ReLU mask words;
  2. fused backward: every block it produces separately (tc_blocks), against that block's own scale, with the fp32
     CUDA-core backward through the same check as the control;
  3. accumulation into a non-zero flat_grad and bit-identical repeats where CTAs add several tiles;
  4. the sample-count and encoding-width limits of the wgmma path;
  5. one training step through run_one_iter_of_nerf that picks the wgmma kernels, against fp64 autograd.
Two more architectures get the forward checks: L_dir 5 without input (30 direction channels: the wgmma forward takes it,
the fused backward does not, and test_simt_mlp_gpu.py checks its training backward on the fp32 kernels) and a model
without view directions, whose training backward runs on the fp32 kernels and is checked here with those.

The oracle and its inputs are those of mlp_checks.py (fp32 points and band products, fp64 from there on);
weights are the seeded reference init ("init") and the same with every gemm layer scaled until max |raw| ~ 3e3
("scaled"), inside the fp16x2 split's range (|weight| < 32, |activation| < 1.05e6).

Fixed-point floor: the fused backward adds every tile's weight-gradient block, and every CTA's bias and direction-
encoding sums, into 64-bit fixed point at 2^-32 (mlp_tc_bwd.cu, to_fix); each add rounds by up to 2^-33 whatever the
size of the gradient.  Every bar below carries that term explicitly, n_adds * 2^-33, next to the part relative to scale.

Bars: each is below 10x the worst figure measured on an H100 over every parameter set (figures beside the constants)."""
import pytest
import torch

from mlp_checks import (ALL_ARCHS, FIX_LSB, FWD_ONLY_ARCHS, SHAPES, STATES, TC_ARCHS as ARCHS,
                        TC_FWD_TOL as FWD_TOL, StashLayout, _floors, _in_blob_range, _split_floors, as_state_dict,
                        check_blocks, encodings, oracle, random_previous, read_layer, relu_ties, report, setup, spec,
                        tc_blocks, training_step_vs_oracle, upstream)

pytestmark = pytest.mark.gpu

# Worst element as a fraction of the compared block's scale.  Measured on an H100 80GB HBM3, worst over all parameter
# sets and both weight states, in brackets.
STASH_TOL = 2e-5     # stashed activation and encoding tiles, per layer; also how far from zero a ReLU tie may sit [9.8e-6]
BLOCK_TOL = 3e-5     # parameter gradients, per block: wgmma [1.3e-5], fp32 kernels [5.2e-6]
ACCUM_TOL = 2e-6     # accumulated minus previous contents vs the gradient, per block [2.5e-7]
FP32_TIE_TOL = 1e-5  # how far from zero an fp32 ReLU tie may sit: test_simt_mlp_gpu.py's STASH_TOL [1.4e-6]

# tiles inside one ray; one CTA with two tiles; ~four tiles per CTA ("sms": the device's multiprocessor count)
MULTI_ARCHS = ["6x128_skip1", "16x128_skip5"]
MULTI_SHAPES = [(3, 1024), ("sms+1", 128), ("8sms", 64)]


def _ids(case):
    name, (n, s) = case
    return f"{name}-{n}x{s}"


FWD_CASES = [(a, s) for a in ALL_ARCHS for s in SHAPES] + [(a, s) for a in MULTI_ARCHS for s in MULTI_SHAPES]
BWD_CASES = [(a, s) for a in [*ARCHS, "4x128_noview"] for s in SHAPES] + [(a, s) for a in MULTI_ARCHS
                                                                         for s in MULTI_SHAPES]


# ------------------------------------------------------------------------------------------------------------------------
# 1. forward: raw outputs, stash tiles, mask words; stash-writing and inference instances
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("case", FWD_CASES, ids=_ids)
def test_tc_forward_and_stash_match_fp64(case, state):
    """mlp_fwd_tc_kernel<true, 128> (training, writes the stash) and <false, 128> (inference) against fp64: raw outputs
    per output column, every gemm layer's activation tile and the xyz-encoding tile decoded from the stash, the ReLU
    mask words; the two instances share the epilogue arithmetic and give the same raw bits."""
    from nerf_pytorch_b200 import ops

    name, shape = case
    arch, sd, rays, z, blob = setup(name, state, shape, seed=1)
    ctx = (name, state, tuple(z.shape))
    assert ops.impl_supported(arch, z.shape[1], ops.IMPL_TC_FWD)
    raw, stash = ops.mlp_fwd(arch, blob, rays.cuda(), z.cuda(), impl=ops.IMPL_TC, want_stash=True)
    raw_inf = ops.mlp_fwd(arch, blob, rays.cuda(), z.cuda(), impl=ops.IMPL_TC)
    torch.cuda.synchronize()
    want, acts, _, _ = oracle(arch, sd, rays, z)
    P = z.numel()
    scale = want.abs().amax(0)
    for what, r in (("train", raw), ("inference", raw_inf)):
        e = (r.reshape(-1, 4).double().cpu() - want).abs().amax(0)
        report(f"forward raw ({what})", ctx, (e / scale).max().item())
        assert (e <= FWD_TOL * scale).all(), ctx + (what, e.tolist(), scale.tolist())
    assert torch.equal(raw, raw_inf), ctx

    lay = StashLayout(arch)
    # the xyz-encoding tile (the B operand of the encoding jobs): real channels against fp64, padding exactly zero
    emb = encodings(arch, rays, z)[0]
    tile = read_layer(stash, P, lay.cum_total, lay.enc_w, "wgmma").cpu()
    assert (tile[:, arch.dim_xyz:] == 0).all(), ctx
    ee = (tile[:, :arch.dim_xyz] - emb).abs().max().item() / emb.abs().max().item()
    worst = ee
    assert ee <= STASH_TOL, ctx + ("xyz encoding", ee)
    for li, (lname, n, cum) in enumerate(lay.layers):
        a = read_layer(stash, P, cum, n, "wgmma").cpu()
        s = acts[li].abs().max().item()
        ea = (a - acts[li]).abs().max().item() / s
        assert ea <= STASH_TOL, ctx + (lname, ea)
        worst = max(worst, ea)
    report("forward stash", ctx, worst)
    report("relu ties", ctx, relu_ties(arch, stash, P, acts, "wgmma", STASH_TOL, ctx, adopt=False))


# ------------------------------------------------------------------------------------------------------------------------
# 2. fused backward, block by block; the fp32 kernels as the control
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("case", BWD_CASES, ids=_ids)
def test_tc_backward_blocks_match_fp64(case, state):
    """ops.mlp_bwd on wgmma (mlp_bwd_tc_kernel + unpack_grad_kernel) given the oracle's ReLU decisions: every block of
    tc_blocks against fp64 autograd, each against its own scale.  The fp32 CUDA-core backward, given the same tie
    handling, goes through the same check.  4x128_noview trains on the fp32 kernels and is checked with those alone."""
    from nerf_pytorch_b200 import ops

    name, shape = case
    arch, sd, rays, z, blob = setup(name, state, shape, seed=4)
    n, s = z.shape
    P = n * s
    ctx = (name, state, (n, s))
    G, acts, dpre, want = _in_blob_range(arch, sd, rays, z, upstream(n, s, seed=5))
    rays_c, z_c, G_c = rays.cuda(), z.cuda(), G.cuda().contiguous()
    on_tc = ops.impl_supported(arch, s, ops.IMPL_TC)
    assert on_tc == (name in ARCHS), ctx
    if on_tc:
        _, stash = ops.mlp_fwd(arch, blob, rays_c, z_c, impl=ops.IMPL_TC, want_stash=True)
        report("relu ties", ctx + ("wgmma",), relu_ties(arch, stash, P, acts, "wgmma", STASH_TOL, ctx + ("wgmma",),
                                                        adopt=True))
        g, _ = ops.mlp_bwd(arch, blob, rays_c, z_c, G_c, stash, impl=ops.IMPL_TC)
        torch.cuda.synchronize()
        check_blocks(arch, g, want, tc_blocks(arch), BLOCK_TOL, ctx, "wgmma backward blocks",
                     _floors(arch, P, _split_floors(arch, G, acts, dpre, rays, z)))
    _, stash32 = ops.mlp_fwd(arch, blob, rays_c, z_c, impl=ops.IMPL_SIMT, want_stash=True)
    report("relu ties", ctx + ("fp32",), relu_ties(arch, stash32, P, acts, "fp32", FP32_TIE_TOL, ctx + ("fp32",),
                                                   adopt=True))
    g32, _ = ops.mlp_bwd(arch, blob, rays_c, z_c, G_c, stash32, impl=ops.IMPL_SIMT)
    torch.cuda.synchronize()
    check_blocks(arch, g32, want, tc_blocks(arch), BLOCK_TOL, ctx, "fp32 backward blocks", _floors(arch, P))


# ------------------------------------------------------------------------------------------------------------------------
# 3. accumulation and bit-identical repeats where CTAs run several tiles
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", MULTI_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("name", MULTI_ARCHS)
def test_tc_backward_accumulates_and_repeats_over_many_tiles(name, state, shape):
    """mlp_bwd adds into a non-zero flat_grad (result - previous contents = the gradient, per block), and two runs give
    the same bits: the CTAs' fixed-point adds are integer sums, whatever their order and however many tiles a CTA runs."""
    from nerf_pytorch_b200 import ops

    arch, sd, rays, z, blob = setup(name, state, shape, seed=6)
    n, s = z.shape
    ctx = (name, state, (n, s))
    G = _in_blob_range(arch, sd, rays, z, upstream(n, s, seed=7))[0].cuda().contiguous()
    rays, z = rays.cuda(), z.cuda()
    _, stash = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC, want_stash=True)
    g1, _ = ops.mlp_bwd(arch, blob, rays, z, G, stash, impl=ops.IMPL_TC)
    g2, _ = ops.mlp_bwd(arch, blob, rays, z, G, stash, impl=ops.IMPL_TC)
    prev = random_previous(arch, g1, tc_blocks(arch), seed=8)
    g3, _ = ops.mlp_bwd(arch, blob, rays, z, G, stash, impl=ops.IMPL_TC, flat_grad=prev.cuda())
    torch.cuda.synchronize()
    assert torch.equal(g1, g2), ctx
    check_blocks(arch, g3.cpu() - prev, as_state_dict(arch, g1.cpu()), tc_blocks(arch), ACCUM_TOL, ctx,
                 "wgmma accumulate", _floors(arch, n * s))


# ------------------------------------------------------------------------------------------------------------------------
# 4. the limits of the wgmma path
# ------------------------------------------------------------------------------------------------------------------------
def test_tc_sample_count_and_encoding_width_limits():
    """15 samples per ray is the smallest count the wgmma kernels take (ceil(128 / 15) + 1 = 10 rays per tile, the
    ray-slot limit); 14 is refused with a message naming 15, and the automatic choice falls back to the fp32 kernels.
    An xyz encoding wider than 64 padded (L_xyz 11 without input: 66 -> 72) is refused the same way."""
    from nerf_pytorch_b200 import ops, train_utils

    for name in ARCHS:
        arch = spec(name)
        for impl in (ops.IMPL_TC, ops.IMPL_TC_FWD):
            assert ops.impl_supported(arch, 15, impl) and not ops.impl_supported(arch, 14, impl), (name, impl)
        for training in (True, False):
            assert train_utils._auto_impl(arch, arch, 15, 49, training=training) == ops.IMPL_TC, name
            assert train_utils._auto_impl(arch, arch, 14, 49, training=training) == ops.IMPL_SIMT, name
    for name in FWD_ONLY_ARCHS:  # the wgmma forward, the fp32 backward
        arch = spec(name)
        assert ops.impl_supported(arch, 15, ops.IMPL_TC_FWD) and not ops.impl_supported(arch, 15, ops.IMPL_TC), name
        assert train_utils._auto_impl(arch, arch, 64, 64, training=True) == ops.IMPL_SIMT, name
        assert train_utils._auto_impl(arch, arch, 64, 64, training=False) == ops.IMPL_TC, name
    assert spec("8x128_ldir5_noinput").dim_dir == 30

    arch, _, rays, z, blob = setup("4x128_l1_skip2", "init", (9, 14), seed=12)
    rays, z = rays.cuda(), z.cuda()
    before = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_SIMT)
    for want_stash in (False, True):
        with pytest.raises(NotImplementedError, match="fewer than 15 samples"):
            ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC, want_stash=want_stash)

    wide = ops.ArchSpec(num_layers=4, hidden=128, n_freq_xyz=11, include_input_xyz=False)
    assert wide.dim_xyz == 66
    for impl in (ops.IMPL_TC, ops.IMPL_TC_FWD):
        assert not ops.impl_supported(wide, 64, impl)
    for training in (True, False):
        assert train_utils._auto_impl(wide, wide, 64, 64, training=training) == ops.IMPL_SIMT
    blob_w = ops.pack_weights(wide, torch.zeros(wide.flat_param_count(), device="cuda"))
    z64 = torch.sort(torch.rand(9, 64, generator=torch.Generator().manual_seed(13)) * 4 + 2, -1).values.cuda()
    with pytest.raises(NotImplementedError, match="wider than 64"):
        ops.mlp_fwd(wide, blob_w, rays, z64, impl=ops.IMPL_TC)
    after = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_SIMT)  # the library works after the refusals
    torch.cuda.synchronize()
    assert torch.equal(before, after)


# ------------------------------------------------------------------------------------------------------------------------
# 5. one training step end to end on the wgmma kernels
# ------------------------------------------------------------------------------------------------------------------------
# As in test_simt_mlp_gpu: the step forms depths and points in fp32, so the coarse network's worst element is
# bounded in units of the fp32 reference's own distance from fp64, per tensor, and the fine network (whose samples the
# resampler places from the coarse weights) by relative L2.  At loss scale the fixed-point floor is not negligible, so it
# is added to both bars.  Measured on an H100 80GB HBM3 in brackets.
E2E_REL_L2 = 8e-6            # whole-network relative L2 of the gradients [1.0e-6]
E2E_COARSE_VS_REF32 = 2.0    # worst element per coarse tensor / (the fp32 oracle's worst there + floor / this bar) [1.22]
E2E_LOSS_TOL = 1e-6          # relative [1.4e-7]


@pytest.mark.parametrize("name", ["4x128_l1_skip2", "16x128_skip5"])
def test_tc_training_step_matches_fp64_oracle(name, monkeypatch):
    """Coarse and fine networks of a swept architecture, 96 rays x (15 + 49) samples, perturb and noise std 0.2 with
    injected randoms, through run_one_iter_of_nerf(mode="train"): the library picks the wgmma kernels, and the loss and
    every parameter gradient of both networks match fp64 autograd of the oracle."""
    from nerf_pytorch_b200 import ops

    used = training_step_vs_oracle(monkeypatch, spec(name), 20, 15, 49, (name,), E2E_REL_L2, E2E_COARSE_VS_REF32,
                                   E2E_LOSS_TOL, fix_lsb=FIX_LSB)
    assert used and all(i == ops.IMPL_TC for i in used), used
