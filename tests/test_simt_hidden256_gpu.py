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

The oracle is O.flexible_nerf_forward in fp64, fed the encoding run_network builds, with the points formed in fp32 as the
reference forms them (train_utils.py:67).  Its sin / cos arguments are the fp32 products x * f the reference evaluates
(nerf_helpers.py:149-151), promoted to fp64: for log-sampled bands that is exactly run_network's fp64 encoding (x * 2^k
is exact), for linear bands it removes the rounding of x * f that an fp64 run would not do.

Bars: each is below 10x the worst error measured on an H100 over every parameter set (figures beside the constants).
Run with -s to print the measured figures."""
import functools

import pytest
import torch

from test_tc_gpu import decode_simt_stash_layer, gemm_layers, pack_mask

pytestmark = pytest.mark.gpu

# Worst element as a fraction of the compared tensor's scale.  Measured on an H100 80GB HBM3, worst over all parameter
# sets and both weight states, in brackets; each bar is below 10x its measurement.
FWD_TOL = 3e-5       # raw outputs, per output column [3.3e-6]
STASH_TOL = 1e-5     # stashed activations, per layer; also how far from zero a ReLU tie may sit [1.4e-6]
DGRAD_TOL = 8e-6     # pre-activation gradients, per layer [9.7e-7]
WGRAD_TOL = 2.5e-5   # weight / bias gradients, per block [2.9e-6]
REPEAT_TOL = 3e-6    # two runs of the weight-gradient kernel (fp32 atomics: summation order differs), per block [3.8e-7]
ACCUM_TOL = 1.5e-5   # accumulated minus previous contents vs the gradient, per block [1.7e-6]

ARCHS = {
    "8x256": dict(num_layers=8, n_freq_xyz=10, n_freq_dir=4),
    "8x256_noview": dict(num_layers=8, n_freq_xyz=10, n_freq_dir=4, use_viewdirs=False),
    "8x256_lxyz6": dict(num_layers=8, n_freq_xyz=6, n_freq_dir=4),     # skip layer K = 256 + 40: a partial 16-row chunk
    "8x256_noinput_linear": dict(num_layers=8, n_freq_xyz=10, n_freq_dir=4, include_input_xyz=False,
                                 log_sampling_xyz=False, log_sampling_dir=False),
    "10x256": dict(num_layers=10, n_freq_xyz=10, n_freq_dir=4),          # two wide layers (layers_xyz.4 and .8)
    "8x256_ldir6": dict(num_layers=8, n_freq_xyz=10, n_freq_dir=6),     # the widest encodings the forward's smem fits
}
STATES = ["init", "scaled"]
# 1 ray; ragged last tiles and tiles that straddle rays; the pretrained fine pass (64 + 64 samples)
FWD_SHAPES = [(1, 16), (7, 50), (33, 17), (129, 100), (64, 128)]
BWD_SHAPES = [(1, 16), (33, 17), (64, 128)]


def _spec(name):
    from nerf_pytorch_b200 import ops

    return ops.ArchSpec(hidden=256, skip_every=4, **ARCHS[name])


def _points(arch, n, s, seed):
    """Lego-like rays: origins on a sphere of radius 4 looking at the centre, near 2, far 6, sorted random depths."""
    g = torch.Generator().manual_seed(seed)
    o = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1) * 4.0
    d = -o / 4.0 + 0.25 * torch.randn(n, 3, generator=g)
    rays = torch.cat([o, d, torch.full((n, 1), 2.0), torch.full((n, 1), 6.0), d / d.norm(dim=-1, keepdim=True)], -1)
    z = torch.sort(torch.rand(n, s, generator=g) * 4 + 2, -1).values
    return (rays if arch.use_viewdirs else rays[:, :8]).contiguous(), z.contiguous()


def _upstream(n, s, seed):
    """d(loss)/d(raw) whose rows span several decades, as compositing weights make them."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, s, 4, generator=g) * torch.exp(torch.randn(n, s, 1, generator=g) * 3.0)


def _embed(x, L, include, log_sampling):
    from nerf_pytorch_b200 import ops

    parts = [x.double()] if include else []
    for f in ops.frequency_bands(L, log_sampling):
        a = (x * f).double()  # the fp32 argument, as the reference evaluates `tensor * freq` before sin / cos
        parts += [torch.sin(a), torch.cos(a)]
    return torch.cat(parts, -1)


def _oracle(arch, sd, rays, z, G=None):
    """fp64: raw [P][4], every gemm layer's activation in the library's order and, given G, the gradients of
    sum(raw * G) with respect to every layer's pre-activation and every parameter."""
    from oracle import nerf_oracle as O

    n, s = z.shape
    sd64 = {k: v.double().requires_grad_(G is not None) for k, v in sd.items()}
    pts = (rays[:, None, :3] + rays[:, None, 3:6] * z[..., None]).reshape(-1, 3)  # fp32, as train_utils.py:67
    emb = _embed(pts, arch.n_freq_xyz, arch.include_input_xyz, arch.log_sampling_xyz)
    if arch.use_viewdirs:
        vd = rays[:, None, 8:11].expand(n, s, 3).reshape(-1, 3)
        emb = torch.cat((emb, _embed(vd, arch.n_freq_dir, arch.include_input_dir, arch.log_sampling_dir)), -1)
    raw, a = O.flexible_nerf_forward(sd64, emb, arch.dim_xyz, return_acts=True)
    acts = [a[f"h{i}"] for i in range(arch.num_layers)] + ([a["feat"], a["d"]] if arch.use_viewdirs else [])
    if G is None:
        return raw, acts, None, None
    keys = list(sd64)
    grads = torch.autograd.grad((raw * G.reshape(-1, 4).double()).sum(), acts + [sd64[k] for k in keys])
    # relu'(pre) = (act > 0); layer1 has no activation (models.py:238)
    dpre = [g if li == 0 else g * (x > 0) for li, (g, x) in enumerate(zip(grads, acts))]
    return raw.detach(), [x.detach() for x in acts], dpre, dict(zip(keys, grads[len(acts):]))


def _scaled(sd, c):
    return {k: v * c if v.shape[0] >= 64 else v for k, v in sd.items()}  # gemm layers only, not the heads


def _weights(name, state):
    return arch_weights(_spec(name), state)


@functools.lru_cache(maxsize=None)
def arch_weights(arch, state):
    """Seeded reference init of `arch` (an ops.ArchSpec); "scaled": every gemm layer's weight and bias times one factor
    c, found by bisection so that max |raw| over a probe batch is ~3e3."""
    from oracle import nerf_oracle as O

    sd = O.init_flexible_nerf(arch.num_layers, arch.hidden, arch.skip_every, arch.n_freq_xyz, arch.n_freq_dir,
                              include_input_xyz=arch.include_input_xyz, include_input_dir=arch.include_input_dir,
                              use_viewdirs=arch.use_viewdirs, generator=torch.Generator().manual_seed(2024))
    if state == "init":
        return sd
    rays, z = _points(arch, 16, 64, seed=99)
    lo, hi = 1.0, 16.0
    for _ in range(24):
        c = (lo * hi) ** 0.5
        if _oracle(arch, _scaled(sd, c), rays, z)[0].abs().max().item() < 3e3:
            lo = c
        else:
            hi = c
    return _scaled(sd, lo)


def _setup(name, state, shape, seed):
    from nerf_pytorch_b200 import ops

    arch = _spec(name)
    sd = _weights(name, state)
    rays, z = _points(arch, *shape, seed=seed)
    blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))
    return arch, sd, rays, z, blob


def _report(what, ctx, value):
    print(f"measured {what} {ctx}: {value:.3e}")


def _mask_words(arch, stash, P, li, layers, cum_total):
    """The ReLU mask words the fp32 forward writes for gemm layer `li`: int32 [P][n/32], bit j of word w = column 32w+j."""
    mask_base = cum_total + ((arch.dim_xyz + 15) & ~15) + ((arch.dim_dir + 7) & ~7)
    start = P * (mask_base + sum(n // 32 for _, n, _ in layers[:li]))
    n = layers[li][1]
    return stash.view(torch.int32)[start:start + P * (n // 32)].view(P, n // 32)


def _write_simt_stash_layer(stash, P, cum_n, n, val):
    """Inverse of decode_simt_stash_layer: store val [P][n] with the stash's row swizzle."""
    x = stash[P * cum_n: P * (cum_n + n)].view(P, n // 32, 8, 4)
    pt = torch.arange(P, device=stash.device) & 7
    idx = torch.arange(8, device=stash.device)[None, :] ^ pt[:, None]
    x.scatter_(2, idx[:, None, :, None].expand(P, n // 32, 8, 4), val.float().view(P, n // 32, 8, 4))


def _check_forward(arch, raw, stash, want, acts, ctx):
    """raw per output column and every layer's stashed activation against fp64, worst element; mask words exact."""
    P = want.shape[0]
    got = raw.reshape(-1, 4).double().cpu()
    scale = want.abs().amax(0)
    e = (got - want).abs().amax(0)
    _report("forward raw", ctx, (e / scale).max().item())
    assert (e <= FWD_TOL * scale).all(), ctx + ("raw", e.tolist(), scale.tolist())
    layers, cum_total = gemm_layers(arch)
    for li, (lname, n, cum) in enumerate(layers):
        a = decode_simt_stash_layer(stash, P, cum, n)
        s = acts[li].abs().max().item()
        ea = (a.cpu() - acts[li]).abs().max().item()
        _report("forward stash", ctx + (lname,), ea / s)
        assert ea <= STASH_TOL * s, ctx + (lname, ea, s)
        # the mask words are the ReLU decisions of the stashed fp32 activations, bit for bit
        assert torch.equal(_mask_words(arch, stash, P, li, layers, cum_total), pack_mask(a > 0)), ctx + (lname,)


def _adopt_oracle_relu(arch, stash, P, acts, ctx):
    """ReLU ties: a unit whose pre-activation is within rounding of zero is on (fp32) and off (fp64) or the reverse, a
    discontinuity of the function, not an error of the backward.  The fp32 data-gradient kernel takes its ReLU decision
    from the stashed activation (mlp_simt.cu, finish: a > 0), so count the disagreements, check that each sits within
    rounding of zero, and overwrite those stash entries with the oracle's value.  Returns the number of ties."""
    layers, cum_total = gemm_layers(arch)
    n_ties = 0
    for li, (lname, n, cum) in enumerate(layers):
        if li == 0:
            continue  # layer1 has no ReLU
        a32 = decode_simt_stash_layer(stash, P, cum, n)
        a64 = acts[li].to(a32.device)
        flip = (a32 > 0) != (a64 > 0)
        k = int(flip.sum())
        if k:
            assert (a32 - a64)[flip].abs().max().item() <= STASH_TOL * a64.abs().max().item(), ctx + (lname,)
            _write_simt_stash_layer(stash, P, cum, n, torch.where(flip, a64, a32))
        n_ties += k
    _report("relu ties", ctx, n_ties)
    assert n_ties <= 1e-5 * P * cum_total + 2, ctx + (n_ties,)
    return n_ties


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


def _as_sd(arch, flat):
    """Views of a flat parameter / gradient vector under the reference's state_dict names."""
    out = {}
    for name, w_off, b_off, fin, fout in arch.flat_layout():
        out[name + ".weight"] = flat[w_off:w_off + fin * fout].view(fout, fin)
        out[name + ".bias"] = flat[b_off:b_off + fout]
    return out


def _block(t, rows, cols):
    return t[rows] if cols is None else t[rows, cols]


def _check_blocks(arch, got_flat, want_sd, tol, ctx, what):
    got_sd = _as_sd(arch, got_flat.double().cpu())
    worst = 0.0
    for label, key, rows, cols in _blocks(arch):
        got, want = _block(got_sd[key], rows, cols), _block(want_sd[key].double().cpu(), rows, cols)
        scale = want.abs().max().item()
        e = (got - want).abs().max().item()
        assert scale > 0 and e <= tol * scale, ctx + (label, e, scale)
        worst = max(worst, e / scale)
    _report(what, ctx, worst)


# ------------------------------------------------------------------------------------------------------------------------
# 1. forward and stash
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", FWD_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("name", list(ARCHS))
def test_forward_and_stash_match_fp64(name, state, shape):
    """Raw outputs, every layer's stashed activation and the ReLU mask words of the fp32 forward
    (mlp_fwd_simt_kernel<4>) against the fp64 oracle."""
    from nerf_pytorch_b200 import ops

    arch, sd, rays, z, blob = _setup(name, state, shape, seed=1)
    raw, stash = ops.mlp_fwd(arch, blob, rays.cuda(), z.cuda(), impl=ops.IMPL_SIMT, want_stash=True)
    torch.cuda.synchronize()
    want, acts, _, _ = _oracle(arch, sd, rays, z)
    _check_forward(arch, raw, stash, want, acts, (name, state, shape))


# ------------------------------------------------------------------------------------------------------------------------
# 2. data-gradient stash
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", BWD_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("name", list(ARCHS))
def test_dgrad_stash_matches_fp64(name, state, shape):
    """ops.mlp_dgrad alone (mlp_bwd_dgrad_kernel<4>, head terms folded in by `finish`): every layer's pre-activation
    gradient in the gradient stash against fp64 autograd, worst element per layer."""
    from nerf_pytorch_b200 import ops

    arch, sd, rays, z, blob = _setup(name, state, shape, seed=2)
    G = _upstream(*shape, seed=3)
    _, stash = ops.mlp_fwd(arch, blob, rays.cuda(), z.cuda(), impl=ops.IMPL_SIMT, want_stash=True)
    _, acts, dpre, _ = _oracle(arch, sd, rays, z, G)
    P = z.numel()
    ctx = (name, state, shape)
    _adopt_oracle_relu(arch, stash, P, acts, ctx)
    gstash = ops.mlp_dgrad(arch, blob, G.cuda().contiguous(), stash, impl=ops.IMPL_SIMT)
    torch.cuda.synchronize()
    worst = 0.0
    for li, (lname, n, cum) in enumerate(gemm_layers(arch)[0]):
        got = decode_simt_stash_layer(gstash, P, cum, n).cpu()
        s = dpre[li].abs().max().item()
        e = (got - dpre[li]).abs().max().item()
        assert s > 0 and e <= DGRAD_TOL * s, ctx + (lname, e, s)
        worst = max(worst, e / s)
    _report("dgrad", ctx, worst)


# ------------------------------------------------------------------------------------------------------------------------
# 3. weight and bias gradients, per block
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", BWD_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("name", list(ARCHS))
def test_weight_gradients_per_block_match_fp64(name, state, shape):
    """ops.mlp_bwd on the CUDA cores: every block the weight-gradient kernel reduces separately (row blocks, hidden
    column blocks, encoding columns, biases, heads) against fp64 autograd, each against its own scale."""
    from nerf_pytorch_b200 import ops

    arch, sd, rays, z, blob = _setup(name, state, shape, seed=4)
    G = _upstream(*shape, seed=5)
    _, stash = ops.mlp_fwd(arch, blob, rays.cuda(), z.cuda(), impl=ops.IMPL_SIMT, want_stash=True)
    _, acts, _, want = _oracle(arch, sd, rays, z, G)
    ctx = (name, state, shape)
    _adopt_oracle_relu(arch, stash, z.numel(), acts, ctx)
    g, _ = ops.mlp_bwd(arch, blob, rays.cuda(), z.cuda(), G.cuda().contiguous(), stash, impl=ops.IMPL_SIMT)
    torch.cuda.synchronize()
    _check_blocks(arch, g, want, WGRAD_TOL, ctx, "wgrad")


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

    arch, sd, rays, z, blob = _setup("8x256", state, shape, seed=6)
    G = _upstream(*shape, seed=7).cuda().contiguous()
    rays, z = rays.cuda(), z.cuda()
    _, stash = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_SIMT, want_stash=True)
    gstash = ops.mlp_dgrad(arch, blob, G, stash, impl=ops.IMPL_SIMT)
    g1 = ops.mlp_wgrad(arch, rays, z, G, stash, gstash, impl=ops.IMPL_SIMT)
    g2 = ops.mlp_wgrad(arch, rays, z, G, stash, gstash, impl=ops.IMPL_SIMT)
    # previous contents: random, with every block at the scale of that block's gradient
    gen = torch.Generator().manual_seed(8)
    prev = torch.zeros_like(g1, device="cpu")
    prev_sd, g1_sd = _as_sd(arch, prev), _as_sd(arch, g1.cpu())
    for _, key, rows, cols in _blocks(arch):
        b = _block(prev_sd[key], rows, cols)
        b.copy_(torch.randn(b.shape, generator=gen) * _block(g1_sd[key], rows, cols).abs().max())
    g3 = ops.mlp_wgrad(arch, rays, z, G, stash, gstash, impl=ops.IMPL_SIMT, flat_grad=prev.cuda())
    torch.cuda.synchronize()
    ctx = (state, shape)
    _check_blocks(arch, g2, _as_sd(arch, g1), REPEAT_TOL, ctx, "wgrad repeat")
    _check_blocks(arch, g3.cpu() - prev, _as_sd(arch, g1), ACCUM_TOL, ctx, "wgrad accumulate")


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

    fits = _spec("8x256_ldir6")
    wider = ops.ArchSpec(num_layers=8, hidden=256, skip_every=4, n_freq_xyz=10, n_freq_dir=7)
    assert _fwd_smem_bytes(ops.ArchSpec(num_layers=8, hidden=256, skip_every=4, n_freq_xyz=10)) == 224320
    assert _fwd_smem_bytes(fits) == 228416 <= 227 * 1024 < _fwd_smem_bytes(wider) == 232512
    assert train_utils._auto_impl(fits, fits, 64, 64, training=False) == ops.IMPL_SIMT
    assert train_utils._auto_impl(fits, fits, 64, 64, training=True) == ops.IMPL_SIMT

    _, sd, rays, z, blob = _setup("8x256_ldir6", "init", (33, 17), seed=9)
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
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    used = []
    render_fwd, render_bwd = ops.render_fwd, ops.render_bwd
    monkeypatch.setattr(ops, "render_fwd", lambda *a, **k: used.append(k["impl"]) or render_fwd(*a, **k))
    monkeypatch.setattr(ops, "render_bwd", lambda *a, **k: used.append(k["impl"]) or render_bwd(*a, **k))

    g = torch.Generator().manual_seed(10 + int(white))
    kw = dict(num_layers=8, hidden_size=256, skip_connect_every=4, num_encoding_fn_xyz=10, num_encoding_fn_dir=4)
    sds = [O.init_flexible_nerf(8, 256, 4, 10, 4, generator=g) for _ in range(2)]
    models = []
    for sd in sds:
        m = nb.FlexibleNeRFModel(**kw)
        m.load_state_dict(sd)
        models.append(m.cuda())
    n, nc, nf = 96, 64, 64
    ro = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1) * 4.0
    rd = -ro / 4.0 + 0.25 * torch.randn(n, 3, generator=g)
    rnd = dict(t_rand=torch.rand(n, nc, generator=g), noise_c=torch.randn(n, nc, generator=g),
               u=torch.rand(n, nf, generator=g), noise_f=torch.randn(n, nc + nf, generator=g))
    target = torch.rand(n, 3, generator=g)
    opts = O.make_options(num_coarse=nc, num_fine=nf, perturb=True, radiance_field_noise_std=0.2, white_background=white)

    out = nb.run_one_iter_of_nerf(100, 100, 120.0, models[0], models[1], ro.cuda(), rd.cuda(), opts, mode="train",
                                  encode_position_fn=nb.get_embedding_function(10),
                                  encode_direction_fn=nb.get_embedding_function(4),
                                  randoms={k: v.cuda() for k, v in rnd.items()})
    tgt = target.cuda()
    loss = torch.nn.functional.mse_loss(out[0], tgt) + torch.nn.functional.mse_loss(out[3], tgt)
    loss.backward()
    torch.cuda.synchronize()
    assert used and all(i == ops.IMPL_SIMT for i in used), used

    def oracle(dtype):
        sd_ = [{k: v.detach().to(dtype).clone().requires_grad_(True) for k, v in sd.items()} for sd in sds]
        out_ = O.run_one_iter_of_nerf(100, 100, 120.0, sd_[0], sd_[1], ro.to(dtype), rd.to(dtype), opts, mode="train",
                                      randoms={k: v.to(dtype) for k, v in rnd.items()})
        loss_ = O.nerf_loss(out_, target.to(dtype))
        loss_.backward()
        return loss_.item(), [{k: v.grad.double() for k, v in s.items()} for s in sd_]

    loss64, g64 = oracle(torch.float64)
    _, g32 = oracle(torch.float32)
    e_loss = abs(loss.item() - loss64) / abs(loss64)
    _report("e2e loss", (white,), e_loss)
    assert e_loss <= E2E_LOSS_TOL, (loss.item(), loss64)
    for i, (tag, model) in enumerate((("coarse", models[0]), ("fine", models[1]))):
        num = den = 0.0
        for k, p in model.named_parameters():
            got, w = p.grad.double().cpu(), g64[i][k]
            num += (got - w).pow(2).sum().item()
            den += w.pow(2).sum().item()
            if tag == "coarse":
                e, s = (got - w).abs().max().item(), w.abs().max().item()
                e_ref = max((g32[i][k] - w).abs().max().item(), 1e-6 * s)
                _report("e2e coarse worst / fp32 oracle's", (white, k), e / e_ref)
                assert e <= E2E_COARSE_VS_REF32 * e_ref, (white, k, e, e_ref, s)
        rel = (num / den) ** 0.5
        _report("e2e rel L2", (white, tag), rel)
        assert rel <= E2E_REL_L2, (white, tag, rel)
