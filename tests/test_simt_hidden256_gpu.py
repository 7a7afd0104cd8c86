"""GPU: the fp32 CUDA-core MLP kernels at hidden 256 against fp64 autograd of the oracle MLP.

Five of the reference's seven pretrained configurations are 8 x 256 with skip 4, and that architecture trains on these
kernels (the wgmma backward is hidden 128 only).  At hidden 256 they are separate instantiations: a 16-row weight chunk,
two output-row and two input-column blocks per layer in the weight-gradient item list, a 256-input head gradient and a
forward shared-memory footprint close to the 227 KB limit.  Every stage is compared here with fp64, block by block:
  * forward: raw outputs, every layer's stashed activation and its ReLU mask words;
  * data gradient: every layer's pre-activation gradient in the gradient stash;
  * weight gradient: every output-row x input-column block, every bias block and every head, each against its own scale;
  * accumulation into a non-zero flat_grad and run-to-run agreement, in both grid regimes of the wgrad kernel;
  * the widest direction encoding that fits shared memory, and the refusal of the next one;
  * one training step end to end through run_one_iter_of_nerf.
Every kernel test runs two weight states: the reference's default init, and the same weights with every gemm layer scaled
so that the raw outputs reach ~3e3 (the shipped lego weights reach 1e4), which exercises fp32's dynamic range.

The oracle and its inputs are those of mlp_checks.py.

Bars: each is below 10x the worst error measured on an H100 over every parameter set (figures beside the constants).
Run with -s to print the measured figures."""
import pytest
import torch

from mlp_checks import (H256_ARCHS, STATES, StashLayout, as_state_dict, check_blocks, mask_words, oracle, pack_mask,
                        random_previous, read_layer, relu_ties, report, setup, spec, training_step_vs_oracle, upstream)

pytestmark = pytest.mark.gpu

# Worst element as a fraction of the compared tensor's scale.  Measured on an H100 80GB HBM3, worst over all parameter
# sets and both weight states, in brackets; each bar is below 10x its measurement.
FWD_TOL = 3e-5       # raw outputs, per output column [3.3e-6]
STASH_TOL = 1e-5     # stashed activations, per layer; also how far from zero a ReLU tie may sit [1.4e-6]
DGRAD_TOL = 8e-6     # pre-activation gradients, per layer [9.7e-7]
WGRAD_TOL = 2.5e-5   # weight / bias gradients, per block [2.9e-6]
REPEAT_TOL = 3e-6    # two runs of the weight-gradient kernel (fp32 atomics: summation order differs), per block [3.8e-7]
ACCUM_TOL = 1.5e-5   # accumulated minus previous contents vs the gradient, per block [1.7e-6]

# 1 ray; ragged last tiles and tiles that straddle rays; the pretrained fine pass (64 + 64 samples)
FWD_SHAPES = [(1, 16), (7, 50), (33, 17), (129, 100), (64, 128)]
BWD_SHAPES = [(1, 16), (33, 17), (64, 128)]


def _check_forward(arch, raw, stash, want, acts, ctx):
    """raw per output column and every layer's stashed activation against fp64, worst element; mask words exact."""
    P = want.shape[0]
    got = raw.reshape(-1, 4).double().cpu()
    scale = want.abs().amax(0)
    e = (got - want).abs().amax(0)
    report("forward raw", ctx, (e / scale).max().item())
    assert (e <= FWD_TOL * scale).all(), ctx + ("raw", e.tolist(), scale.tolist())
    for li, (lname, n, cum) in enumerate(StashLayout(arch).layers):
        a = read_layer(stash, P, cum, n, "fp32")
        s = acts[li].abs().max().item()
        ea = (a.cpu() - acts[li]).abs().max().item()
        report("forward stash", ctx + (lname,), ea / s)
        assert ea <= STASH_TOL * s, ctx + (lname, ea, s)
        # the mask words are the ReLU decisions of the stashed fp32 activations, bit for bit
        assert torch.equal(mask_words(arch, stash, P, li, "fp32"), pack_mask(a > 0)), ctx + (lname,)


def _blocks(arch):
    """(label, key, rows, cols) of every block the weight-gradient kernel reduces separately: output rows 0-127 / 128-255,
    input columns 0-127 / 128-255 of the hidden part, the encoding columns, the bias per row block, and each head."""
    out = []
    for name, _, _, fin, fout in arch.flat_layout():
        if fout < 64:  # fc_alpha / fc_rgb / fc_out
            out += [(name + ".weight", name + ".weight", slice(None), slice(None)),
                    (name + ".bias", name + ".bias", slice(None), None)]
            continue
        k_h = 0 if name == "layer1" else arch.hidden
        for r0 in range(0, fout, 128):
            rows = slice(r0, r0 + 128)
            for c0 in range(0, k_h, 128):
                out.append((f"{name}.weight[{r0}:+128, {c0}:+128]", name + ".weight", rows, slice(c0, c0 + 128)))
            if fin > k_h:
                out.append((f"{name}.weight[{r0}:+128, enc]", name + ".weight", rows, slice(k_h, fin)))
            out.append((f"{name}.bias[{r0}:+128]", name + ".bias", rows, None))
    return out


# ------------------------------------------------------------------------------------------------------------------------
# 1. forward and stash
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", FWD_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("name", list(H256_ARCHS))
def test_forward_and_stash_match_fp64(name, state, shape):
    """Raw outputs, every layer's stashed activation and the ReLU mask words of the fp32 forward
    (mlp_fwd_simt_kernel<4>) against the fp64 oracle."""
    from nerf_pytorch_b200 import ops

    arch, sd, rays, z, blob = setup(name, state, shape, seed=1)
    raw, stash = ops.mlp_fwd(arch, blob, rays.cuda(), z.cuda(), impl=ops.IMPL_SIMT, want_stash=True)
    torch.cuda.synchronize()
    want, acts, _, _ = oracle(arch, sd, rays, z)
    _check_forward(arch, raw, stash, want, acts, (name, state, shape))


# ------------------------------------------------------------------------------------------------------------------------
# 2. data-gradient stash
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", BWD_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("name", list(H256_ARCHS))
def test_dgrad_stash_matches_fp64(name, state, shape):
    """ops.mlp_dgrad alone (mlp_bwd_dgrad_kernel<4>, head terms folded in by `finish`): every layer's pre-activation
    gradient in the gradient stash against fp64 autograd, worst element per layer."""
    from nerf_pytorch_b200 import ops

    arch, sd, rays, z, blob = setup(name, state, shape, seed=2)
    G = upstream(*shape, seed=3)
    _, stash = ops.mlp_fwd(arch, blob, rays.cuda(), z.cuda(), impl=ops.IMPL_SIMT, want_stash=True)
    _, acts, dpre, _ = oracle(arch, sd, rays, z, G)
    P = z.numel()
    ctx = (name, state, shape)
    report("relu ties", ctx, relu_ties(arch, stash, P, acts, "fp32", STASH_TOL, ctx, adopt=True))
    gstash = ops.mlp_dgrad(arch, blob, G.cuda().contiguous(), stash, impl=ops.IMPL_SIMT)
    torch.cuda.synchronize()
    worst = 0.0
    for li, (lname, n, cum) in enumerate(StashLayout(arch).layers):
        got = read_layer(gstash, P, cum, n, "fp32").cpu()
        s = dpre[li].abs().max().item()
        e = (got - dpre[li]).abs().max().item()
        assert s > 0 and e <= DGRAD_TOL * s, ctx + (lname, e, s)
        worst = max(worst, e / s)
    report("dgrad", ctx, worst)


# ------------------------------------------------------------------------------------------------------------------------
# 3. weight and bias gradients, per block
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", BWD_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("name", list(H256_ARCHS))
def test_weight_gradients_per_block_match_fp64(name, state, shape):
    """ops.mlp_bwd on the CUDA cores: every block the weight-gradient kernel reduces separately (row blocks, hidden
    column blocks, encoding columns, biases, heads) against fp64 autograd, each against its own scale."""
    from nerf_pytorch_b200 import ops

    arch, sd, rays, z, blob = setup(name, state, shape, seed=4)
    G = upstream(*shape, seed=5)
    _, stash = ops.mlp_fwd(arch, blob, rays.cuda(), z.cuda(), impl=ops.IMPL_SIMT, want_stash=True)
    _, acts, _, want = oracle(arch, sd, rays, z, G)
    ctx = (name, state, shape)
    report("relu ties", ctx, relu_ties(arch, stash, z.numel(), acts, "fp32", STASH_TOL, ctx, adopt=True))
    g, _ = ops.mlp_bwd(arch, blob, rays.cuda(), z.cuda(), G.cuda().contiguous(), stash, impl=ops.IMPL_SIMT)
    torch.cuda.synchronize()
    check_blocks(arch, g, want, _blocks(arch), WGRAD_TOL, ctx, "wgrad")


# ------------------------------------------------------------------------------------------------------------------------
# 4. accumulation and repeat runs
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1, 16), (7, 50), (64, 128)], ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("state", STATES)
def test_wgrad_accumulates_and_repeats(state, shape):
    """ops.mlp_wgrad adds into flat_grad, and two runs agree to fp32 summation-order noise (the kernel flushes with
    atomics, so not bit for bit).  1 x 16 and 7 x 50: the grid split is capped by the number of 32-point stages;
    64 x 128: many CTAs share each item."""
    from nerf_pytorch_b200 import ops

    arch, sd, rays, z, blob = setup("8x256", state, shape, seed=6)
    G = upstream(*shape, seed=7).cuda().contiguous()
    rays, z = rays.cuda(), z.cuda()
    _, stash = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_SIMT, want_stash=True)
    gstash = ops.mlp_dgrad(arch, blob, G, stash, impl=ops.IMPL_SIMT)
    g1 = ops.mlp_wgrad(arch, rays, z, G, stash, gstash, impl=ops.IMPL_SIMT)
    g2 = ops.mlp_wgrad(arch, rays, z, G, stash, gstash, impl=ops.IMPL_SIMT)
    prev = random_previous(arch, g1, _blocks(arch), seed=8)
    g3 = ops.mlp_wgrad(arch, rays, z, G, stash, gstash, impl=ops.IMPL_SIMT, flat_grad=prev.cuda())
    torch.cuda.synchronize()
    ctx = (state, shape)
    check_blocks(arch, g2, as_state_dict(arch, g1), _blocks(arch), REPEAT_TOL, ctx, "wgrad repeat")
    check_blocks(arch, g3.cpu() - prev, as_state_dict(arch, g1), _blocks(arch), ACCUM_TOL, ctx, "wgrad accumulate")


# ------------------------------------------------------------------------------------------------------------------------
# 5. shared-memory boundary of the hidden-256 forward
# ------------------------------------------------------------------------------------------------------------------------
def _fwd_smem_bytes(arch):
    """fwd_smem_layout (mlp_simt.cu) restated: activation, xyz / direction encoding tiles (rows padded by 4 floats),
    two 16-row weight chunks, head weights and biases."""
    pad8 = lambda x: (x + 7) & ~7  # noqa: E731
    H = arch.hidden
    floats = (128 * (H + 4) + 128 * (pad8(arch.dim_xyz) + 4) + 128 * (pad8(arch.dim_dir) + 4) + 2 * 16 * H + 5 * H + 16)
    return 4 * floats


def test_widest_direction_encoding_that_fits_shared_memory():
    """8 x 256 with L_xyz 10 needs 4 * (43792 + 128 * (64 + dim_dir_pad)) bytes of shared memory in the fp32 forward.
    L_dir 6 (40 columns, 228 416 B) fits 227 KB and is checked against fp64 with the other architectures above;
    L_dir 7 (48 columns, 232 512 B) is refused with NotImplementedError and leaves the library working.  The wgmma
    forward takes at most 32 direction channels, so the accepted case renders on the fp32 kernels in inference too."""
    from nerf_pytorch_b200 import ops, train_utils

    fits = spec("8x256_ldir6")
    wider = ops.ArchSpec(num_layers=8, hidden=256, skip_every=4, n_freq_xyz=10, n_freq_dir=7)
    assert _fwd_smem_bytes(ops.ArchSpec(num_layers=8, hidden=256, skip_every=4, n_freq_xyz=10)) == 224320
    assert _fwd_smem_bytes(fits) == 228416 <= 227 * 1024 < _fwd_smem_bytes(wider) == 232512
    assert train_utils._auto_impl(fits, fits, 64, 64, training=False) == ops.IMPL_SIMT
    assert train_utils._auto_impl(fits, fits, 64, 64, training=True) == ops.IMPL_SIMT

    _, sd, rays, z, blob = setup("8x256_ldir6", "init", (33, 17), seed=9)
    rays, z = rays.cuda(), z.cuda()
    before = ops.mlp_fwd(fits, blob, rays, z, impl=ops.IMPL_SIMT)
    blob7 = ops.pack_weights(wider, torch.zeros(wider.flat_param_count(), device="cuda"))
    with pytest.raises(NotImplementedError, match="shared memory"):
        ops.mlp_fwd(wider, blob7, rays, z, impl=ops.IMPL_SIMT)
    after = ops.mlp_fwd(fits, blob, rays, z, impl=ops.IMPL_SIMT)
    torch.cuda.synchronize()
    assert torch.equal(before, after)


# ------------------------------------------------------------------------------------------------------------------------
# 6. one training step end to end
# ------------------------------------------------------------------------------------------------------------------------
# The step's depths and points are formed in fp32 (bit for bit as the fp32 reference forms them), and an encoding
# channel sin(2^9 x) moves by ~1e-4 for a one-ulp change of x, so the fp32 reference itself is up to ~1e-2 of scale
# (worst element) from fp64 here.  The coarse network's worst element is therefore bounded in units of the fp32
# reference's own distance from fp64, per tensor.  Measured on an H100 80GB HBM3 in brackets.
E2E_REL_L2 = 2e-3       # whole-network relative L2 of the gradients [2.1e-4]
E2E_COARSE_VS_REF32 = 2.0   # worst element per coarse tensor / the fp32 oracle's worst element there [1.002]
E2E_LOSS_TOL = 5e-5     # relative [5.4e-6]


@pytest.mark.parametrize("white", [False, True])
def test_training_step_matches_fp64_oracle(white, monkeypatch):
    """8 x 256 coarse and fine networks, 96 rays x (64 + 64) samples, perturb and noise std 0.2 with injected randoms,
    through run_one_iter_of_nerf(mode="train"): the library picks the fp32 kernels, and the loss and every parameter
    gradient of both networks match fp64 autograd of the oracle."""
    from nerf_pytorch_b200 import ops

    used = training_step_vs_oracle(monkeypatch, spec("8x256"), 10 + int(white), 64, 64, (white,), E2E_REL_L2,
                                   E2E_COARSE_VS_REF32, E2E_LOSS_TOL, white=white)
    assert used and all(i == ops.IMPL_SIMT for i in used), used
