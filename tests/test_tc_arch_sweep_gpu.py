"""GPU: the wgmma forward and fused backward at hidden 128, across the architectures and sample counts they accept,
against fp64 autograd of the oracle MLP, block by block.

Every hidden-128 model trains on these kernels by default (train_utils._auto_impl), so every architecture family that
bwd_tc_supported accepts gets its own job table (bwd_jobs), gradient-blob layout (blob_map) and unpack mapping.  The
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
  2. fused backward: every block it produces separately (_tc_blocks), against that block's own scale, with the fp32
     CUDA-core backward through the same check as the control;
  3. accumulation into a non-zero flat_grad and bit-identical repeats where CTAs add several tiles;
  4. the sample-count and encoding-width limits of the wgmma path;
  5. one training step through run_one_iter_of_nerf that picks the wgmma kernels, against fp64 autograd.
Two more architectures get the forward checks: L_dir 5 without input (30 direction channels: the wgmma forward takes it,
the fused backward does not) and a model without view directions, whose training backward runs on the fp32 kernels and
is checked here with those.

The oracle and its inputs are those of test_simt_hidden256_gpu.py (fp32 points and band products, fp64 from there on);
weights are the seeded reference init ("init") and the same with every gemm layer scaled until max |raw| ~ 3e3
("scaled"), inside the fp16x2 split's range (|weight| < 32, |activation| < 1.05e6).

Fixed-point floor: the fused backward adds every tile's weight-gradient block, and every CTA's bias and direction-
encoding sums, into 64-bit fixed point at 2^-32 (mlp_tc_bwd.cu, to_fix); each add rounds by up to 2^-33 whatever the
size of the gradient.  Every bar below carries that term explicitly, n_adds * 2^-33, next to the part relative to scale.

Bars: each is below 10x the worst figure measured on an H100 over every parameter set (figures beside the constants)."""
import pytest
import torch

from test_simt_hidden256_gpu import (_adopt_oracle_relu, _as_sd, _block, _embed, _oracle, _points, _report, _upstream,
                                     arch_weights)
from test_tc_gpu import decode_tc_stash_layer, gemm_layers, pack_mask, tc_mask_view

pytestmark = pytest.mark.gpu

# Worst element as a fraction of the compared block's scale.  Measured on an H100 80GB HBM3, worst over all parameter
# sets and both weight states, in brackets.
FWD_TOL = 3e-5       # raw outputs, per output column; stash-writing and inference forward [1.1e-5]
STASH_TOL = 2e-5     # stashed activation and encoding tiles, per layer; also how far from zero a ReLU tie may sit [9.8e-6]
BLOCK_TOL = 3e-5     # parameter gradients, per block: wgmma [1.3e-5], fp32 kernels [5.2e-6]
ACCUM_TOL = 2e-6     # accumulated minus previous contents vs the gradient, per block [2.5e-7]
FIX_LSB = 2.0 ** -33  # rounding of one add into the fixed-point gradient blob (resolution 2^-32)
# Resolution of the fp16x2 split below fp16's normal range (tc_common.cuh split_f16x2): hi and lo are subnormal there,
# so x = hi + lo 2^-11 is resolved to 2^-36 absolutely.  The fused backward splits G (and d_raw) at the tile's scale,
# max |d_raw| of the tile -> [4, 8), so a G element is resolved to 2^-36 / 4 = 2^-38 of the tile's max |d_raw|, however
# small it is; the stash holds activation / 16, resolved to 2^-36 * 16 = 2^-32 absolutely.
G_SPLIT_LSB = 2.0 ** -38
ACT_SPLIT_LSB = 2.0 ** -32
BLOB_MAX = 2.0 ** 28  # the gradient blob holds sums below 2^31 (mlp_tc_bwd.cu); the checks keep every gradient below this

# hidden 128; the fused backward takes all of these
ARCHS = {
    "1x128": dict(num_layers=1, skip_every=4, n_freq_xyz=10, n_freq_dir=4),
    "4x128_l0": dict(num_layers=4, skip_every=4, n_freq_xyz=0, n_freq_dir=0),
    "4x128_l1_skip2": dict(num_layers=4, skip_every=2, n_freq_xyz=1, n_freq_dir=1),
    "6x128_skip1": dict(num_layers=6, skip_every=1, n_freq_xyz=6, n_freq_dir=2),
    "8x128_noinput_linear": dict(num_layers=8, skip_every=3, n_freq_xyz=10, n_freq_dir=4, include_input_xyz=False,
                                 include_input_dir=False, log_sampling_xyz=False, log_sampling_dir=False),
    "8x128_widest": dict(num_layers=8, skip_every=4, n_freq_xyz=10, n_freq_dir=4),
    "16x128_skip5": dict(num_layers=16, skip_every=5, n_freq_xyz=6, n_freq_dir=4),
}
# the wgmma forward only: their training backward runs on the fp32 kernels
FWD_ONLY_ARCHS = {
    "8x128_ldir5_noinput": dict(num_layers=8, skip_every=4, n_freq_xyz=10, n_freq_dir=5, include_input_dir=False),
    "4x128_noview": dict(num_layers=4, skip_every=4, n_freq_xyz=5, log_sampling_xyz=False, use_viewdirs=False),
}
ALL_ARCHS = {**ARCHS, **FWD_ONLY_ARCHS}
STATES = ["init", "scaled"]
# one ray at the smallest accepted count; tiles spanning 10 rays; ragged tiles
SHAPES = [(1, 15), (37, 15), (33, 17)]
# tiles inside one ray; one CTA with two tiles; ~four tiles per CTA ("sms": the device's multiprocessor count)
MULTI_ARCHS = ["6x128_skip1", "16x128_skip5"]
MULTI_SHAPES = [(3, 1024), ("sms+1", 128), ("8sms", 64)]


def _ids(case):
    name, (n, s) = case
    return f"{name}-{n}x{s}"


FWD_CASES = [(a, s) for a in ALL_ARCHS for s in SHAPES] + [(a, s) for a in MULTI_ARCHS for s in MULTI_SHAPES]
BWD_CASES = [(a, s) for a in [*ARCHS, "4x128_noview"] for s in SHAPES] + [(a, s) for a in MULTI_ARCHS
                                                                         for s in MULTI_SHAPES]


def _spec(name):
    from nerf_pytorch_b200 import ops

    return ops.ArchSpec(hidden=128, **ALL_ARCHS[name])


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _shape(shape):
    n, s = shape
    if n == "sms+1":
        n = _sms() + 1
    elif n == "8sms":
        n = 8 * _sms()
    return n, s


def _setup(name, state, shape, seed):
    from nerf_pytorch_b200 import ops

    arch = _spec(name)
    sd = arch_weights(arch, state)
    rays, z = _points(arch, *_shape(shape), seed=seed)
    blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))
    return arch, sd, rays, z, blob


def _tc_blocks(arch):
    """(label, key, rows, cols, per_cta) of every block the fused backward produces on its own path, from the rules of
    bwd_jobs / blob_map (mlp_tc_bwd.cu):
      * gemm layer with hidden inputs: the kind-0 job on the hidden columns; warpgroup w owns output rows [64 w, +64);
      * layer1 and every wide layer: the xyz-encoding job (B = the encoding tile), per row half;
      * layers_dir.0: its direction-encoding columns come from the per-ray sums x s_encd (s_dacc -> blob region xd);
      * every gemm layer's bias: the indicator product summed in s_bgrad (region xb), per row half;
      * fc_alpha / fc_rgb weights: the kind-1 jobs (region xh), A = the source layer's activation tile, whose feature
        rows [64 w, +64) warpgroup w handles; their biases: G-tile rows 64..67 of the indicator product (region xb).
    per_cta: the block reaches the blob once per CTA (biases, direction encodings), else once per tile.  Without view
    directions (fp32 kernels only) fc_out is listed like a head."""
    out = []
    for name, _, _, fin, fout in arch.flat_layout():
        if fout < 64:  # heads
            for c0 in range(0, fin, 64):
                out.append((f"{name}.weight[:, {c0}:+64]", name + ".weight", slice(None), slice(c0, c0 + 64), False))
            out.append((name + ".bias", name + ".bias", slice(None), None, True))
            continue
        k_h = 0 if name == "layer1" else arch.hidden
        for r0 in range(0, fout, 64):
            rows = slice(r0, r0 + 64)
            if k_h:
                out.append((f"{name}.weight[{r0}:+64, hidden]", name + ".weight", rows, slice(0, k_h), False))
            if fin > k_h:
                if name == "layers_dir.0":
                    out.append((f"{name}.weight[{r0}:+64, dir enc]", name + ".weight", rows, slice(k_h, fin), True))
                else:
                    out.append((f"{name}.weight[{r0}:+64, xyz enc]", name + ".weight", rows, slice(k_h, fin), False))
            out.append((f"{name}.bias[{r0}:+64]", name + ".bias", rows, None, True))
    return out


def _check_blocks(arch, got_flat, want_sd, n_points, tol, ctx, what, split_floors=None):
    """Every _tc_blocks block within tol of its own scale plus the fixed-point floor (n_adds * 2^-33) and, for the wgmma
    kernels, the split's resolution floor of that block (_split_floors).  Reports the worst e / (scale + floors / tol),
    the figure the bar `tol` applies to."""
    n_tiles = -(-n_points // 128)
    n_ctas = min(n_tiles, _sms())
    got_sd = _as_sd(arch, got_flat.double().cpu())
    worst = 0.0
    for label, key, rows, cols, per_cta in _tc_blocks(arch):
        got, want = _block(got_sd[key], rows, cols), _block(want_sd[key].double().cpu(), rows, cols)
        scale = want.abs().max().item()
        e = (got - want).abs().max().item()
        floor = (n_ctas if per_cta else n_tiles) * FIX_LSB + (split_floors or {}).get(label, 0.0)
        assert scale > 0 and e <= tol * scale + floor, ctx + (what, label, e, scale, floor)
        worst = max(worst, e / (scale + floor / tol))
    _report(what, ctx, worst)


def _in_blob_range(arch, sd, rays, z, G):
    """fp64 oracle of sum(raw * G), with G scaled by a power of two (exact on both sides) if needed so that every
    parameter gradient stays below BLOB_MAX.  Returns (G, acts, dpre, grads)."""
    _, acts, dpre, want = _oracle(arch, sd, rays, z, G)
    m = max(v.abs().max().item() for v in want.values())
    if m > BLOB_MAX:
        c = 2.0 ** -int(torch.tensor(m / BLOB_MAX).log2().ceil().item())
        G, dpre, want = G * c, [x * c for x in dpre], {k: v * c for k, v in want.items()}
    return G, acts, dpre, want


def _split_floors(arch, G, acts, dpre, rays, z):
    """label -> the wgmma backward's resolution floor of that block, from the split's absolute resolution:
        sum_p G_SPLIT_LSB * D(p) * max |X[p]|  +  ACT_SPLIT_LSB * max |G[p]|
    over the points p, with D(p) the max |d_raw| of p's tile, X the block's input columns (activations, encodings, or 1
    for the indicator sums) and G the block's output rows of the pre-activation gradient (d_raw for the heads).  It
    matters where G is many decades below d_raw: the deep layers of an initialised network, whose gradient vanishes."""
    P = z.numel()
    d_raw = G.reshape(-1, 4).double().abs()
    D = torch.nn.functional.pad(d_raw.amax(1), (0, -P % 128)).view(-1, 128).amax(1).repeat_interleave(128)[:P]
    pts = (rays[:, None, :3] + rays[:, None, 3:6] * z[..., None]).reshape(-1, 3)
    x_enc = _embed(pts, arch.n_freq_xyz, arch.include_input_xyz, arch.log_sampling_xyz).abs().amax(1)
    x_dir = None
    if arch.use_viewdirs:
        vd = rays[:, None, 8:11].expand(*z.shape, 3).reshape(-1, 3)
        x_dir = _embed(vd, arch.n_freq_dir, arch.include_input_dir, arch.log_sampling_dir).abs().amax(1)
    index = {lname: li for li, (lname, _, _) in enumerate(gemm_layers(arch)[0])}
    heads = {"fc_alpha": (arch.num_layers - 1, [3]), "fc_rgb": (len(acts) - 1, [0, 1, 2]),
             "fc_out": (arch.num_layers - 1, [0, 1, 2, 3])}
    out = {}
    for label, key, rows, cols, _ in _tc_blocks(arch):
        lname, kind = key.rsplit(".", 1)
        g = 0.0
        if lname in heads:
            src, outs = heads[lname]
            x = 1.0 if kind == "bias" else acts[src][:, cols].abs().amax(1)
            if kind == "weight":
                g = d_raw[:, outs].amax(1)
        elif kind == "bias":
            x = 1.0
        elif "dir enc" in label:
            x = x_dir  # per-ray sums (indicator) x the fp32 direction encoding: no activation split
        else:
            x = x_enc if "xyz enc" in label else acts[index[lname] - 1].abs().amax(1)
            g = dpre[index[lname]][:, rows].abs().amax(1)
        out[label] = (G_SPLIT_LSB * (D * x).sum() + ACT_SPLIT_LSB * torch.as_tensor(g).sum()).item()
    return out


def _tc_relu_ties(arch, stash, P, acts, ctx, adopt):
    """The wgmma forward's ReLU mask words against act64 > 0.  Every disagreement must be a tie: a unit whose fp64
    activation is within STASH_TOL of the layer's scale of zero; their number is bounded.  With `adopt`, the words are
    overwritten with the oracle's decisions, so that the backward is measured on its own arithmetic."""
    layers, cum_total = gemm_layers(arch)
    shifts = torch.arange(32, device=stash.device, dtype=torch.int32)
    n_ties = 0
    for li, (lname, n, _) in enumerate(layers):
        if li == 0:
            continue  # layer1 has no ReLU; the backward does not read its words
        words = tc_mask_view(arch, stash, P, li, layers, cum_total)
        a64 = acts[li].to(stash.device)
        want = pack_mask(a64 > 0)
        flip = (((words ^ want).unsqueeze(-1) >> shifts) & 1).view(P, n).bool()
        k = int(flip.sum())
        if k:
            assert a64[flip].abs().max().item() <= STASH_TOL * a64.abs().max().item(), ctx + (lname,)
        if adopt:
            words.copy_(want)
        n_ties += k
    _report("relu ties", ctx, n_ties)
    assert n_ties <= 1e-5 * P * cum_total + 2, ctx + (n_ties,)


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
    arch, sd, rays, z, blob = _setup(name, state, shape, seed=1)
    ctx = (name, state, tuple(z.shape))
    assert ops.impl_supported(arch, z.shape[1], ops.IMPL_TC_FWD)
    raw, stash = ops.mlp_fwd(arch, blob, rays.cuda(), z.cuda(), impl=ops.IMPL_TC, want_stash=True)
    raw_inf = ops.mlp_fwd(arch, blob, rays.cuda(), z.cuda(), impl=ops.IMPL_TC)
    torch.cuda.synchronize()
    want, acts, _, _ = _oracle(arch, sd, rays, z)
    P = z.numel()
    scale = want.abs().amax(0)
    for what, r in (("train", raw), ("inference", raw_inf)):
        e = (r.reshape(-1, 4).double().cpu() - want).abs().amax(0)
        _report(f"forward raw ({what})", ctx, (e / scale).max().item())
        assert (e <= FWD_TOL * scale).all(), ctx + (what, e.tolist(), scale.tolist())
    assert torch.equal(raw, raw_inf), ctx

    layers, cum_total = gemm_layers(arch)
    # the xyz-encoding tile (the B operand of the encoding jobs): real channels against fp64, padding exactly zero
    enc_w = (arch.dim_xyz + 15) & ~15
    pts = (rays[:, None, :3] + rays[:, None, 3:6] * z[..., None]).reshape(-1, 3)
    emb = _embed(pts, arch.n_freq_xyz, arch.include_input_xyz, arch.log_sampling_xyz)
    tile = decode_tc_stash_layer(stash, P, cum_total, enc_w).cpu()
    assert (tile[:, arch.dim_xyz:] == 0).all(), ctx
    ee = (tile[:, :arch.dim_xyz] - emb).abs().max().item() / emb.abs().max().item()
    worst = ee
    assert ee <= STASH_TOL, ctx + ("xyz encoding", ee)
    for li, (lname, n, cum) in enumerate(layers):
        a = decode_tc_stash_layer(stash, P, cum, n).cpu()
        s = acts[li].abs().max().item()
        ea = (a - acts[li]).abs().max().item() / s
        assert ea <= STASH_TOL, ctx + (lname, ea)
        worst = max(worst, ea)
    _report("forward stash", ctx, worst)
    _tc_relu_ties(arch, stash, P, acts, ctx, adopt=False)


# ------------------------------------------------------------------------------------------------------------------------
# 2. fused backward, block by block; the fp32 kernels as the control
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("case", BWD_CASES, ids=_ids)
def test_tc_backward_blocks_match_fp64(case, state):
    """ops.mlp_bwd on wgmma (mlp_bwd_tc_kernel + unpack_grad_kernel) given the oracle's ReLU decisions: every block of
    _tc_blocks against fp64 autograd, each against its own scale.  The fp32 CUDA-core backward, given the same tie
    handling, goes through the same check.  4x128_noview trains on the fp32 kernels and is checked with those alone."""
    from nerf_pytorch_b200 import ops

    name, shape = case
    arch, sd, rays, z, blob = _setup(name, state, shape, seed=4)
    n, s = z.shape
    P = n * s
    ctx = (name, state, (n, s))
    G, acts, dpre, want = _in_blob_range(arch, sd, rays, z, _upstream(n, s, seed=5))
    rays_c, z_c, G_c = rays.cuda(), z.cuda(), G.cuda().contiguous()
    on_tc = ops.impl_supported(arch, s, ops.IMPL_TC)
    assert on_tc == (name in ARCHS), ctx
    if on_tc:
        _, stash = ops.mlp_fwd(arch, blob, rays_c, z_c, impl=ops.IMPL_TC, want_stash=True)
        _tc_relu_ties(arch, stash, P, acts, ctx + ("wgmma",), adopt=True)
        g, _ = ops.mlp_bwd(arch, blob, rays_c, z_c, G_c, stash, impl=ops.IMPL_TC)
        torch.cuda.synchronize()
        _check_blocks(arch, g, want, P, BLOCK_TOL, ctx, "wgmma backward blocks",
                      _split_floors(arch, G, acts, dpre, rays, z))
    _, stash32 = ops.mlp_fwd(arch, blob, rays_c, z_c, impl=ops.IMPL_SIMT, want_stash=True)
    _adopt_oracle_relu(arch, stash32, P, acts, ctx + ("fp32",))
    g32, _ = ops.mlp_bwd(arch, blob, rays_c, z_c, G_c, stash32, impl=ops.IMPL_SIMT)
    torch.cuda.synchronize()
    _check_blocks(arch, g32, want, P, BLOCK_TOL, ctx, "fp32 backward blocks")


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

    arch, sd, rays, z, blob = _setup(name, state, shape, seed=6)
    n, s = z.shape
    ctx = (name, state, (n, s))
    G = _in_blob_range(arch, sd, rays, z, _upstream(n, s, seed=7))[0].cuda().contiguous()
    rays, z = rays.cuda(), z.cuda()
    _, stash = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC, want_stash=True)
    g1, _ = ops.mlp_bwd(arch, blob, rays, z, G, stash, impl=ops.IMPL_TC)
    g2, _ = ops.mlp_bwd(arch, blob, rays, z, G, stash, impl=ops.IMPL_TC)
    # previous contents: random, every block at the scale of that block's gradient
    gen = torch.Generator().manual_seed(8)
    prev = torch.zeros(g1.shape)
    prev_sd, g1_sd = _as_sd(arch, prev), _as_sd(arch, g1.cpu())
    for _, key, rows, cols, _ in _tc_blocks(arch):
        b = _block(prev_sd[key], rows, cols)
        b.copy_(torch.randn(b.shape, generator=gen) * _block(g1_sd[key], rows, cols).abs().max())
    g3, _ = ops.mlp_bwd(arch, blob, rays, z, G, stash, impl=ops.IMPL_TC, flat_grad=prev.cuda())
    torch.cuda.synchronize()
    assert torch.equal(g1, g2), ctx
    _check_blocks(arch, g3.cpu() - prev, _as_sd(arch, g1.cpu()), n * s, ACCUM_TOL, ctx, "wgmma accumulate")


# ------------------------------------------------------------------------------------------------------------------------
# 4. the limits of the wgmma path
# ------------------------------------------------------------------------------------------------------------------------
def test_tc_sample_count_and_encoding_width_limits():
    """15 samples per ray is the smallest count the wgmma kernels take (ceil(128 / 15) + 1 = 10 rays per tile, the
    ray-slot limit); 14 is refused with a message naming 15, and the automatic choice falls back to the fp32 kernels.
    An xyz encoding wider than 64 padded (L_xyz 11 without input: 66 -> 72) is refused the same way."""
    from nerf_pytorch_b200 import ops, train_utils

    for name in ARCHS:
        arch = _spec(name)
        for impl in (ops.IMPL_TC, ops.IMPL_TC_FWD):
            assert ops.impl_supported(arch, 15, impl) and not ops.impl_supported(arch, 14, impl), (name, impl)
        for training in (True, False):
            assert train_utils._auto_impl(arch, arch, 15, 49, training=training) == ops.IMPL_TC, name
            assert train_utils._auto_impl(arch, arch, 14, 49, training=training) == ops.IMPL_SIMT, name
    for name in FWD_ONLY_ARCHS:  # the wgmma forward, the fp32 backward
        arch = _spec(name)
        assert ops.impl_supported(arch, 15, ops.IMPL_TC_FWD) and not ops.impl_supported(arch, 15, ops.IMPL_TC), name
        assert train_utils._auto_impl(arch, arch, 64, 64, training=True) == ops.IMPL_SIMT, name
        assert train_utils._auto_impl(arch, arch, 64, 64, training=False) == ops.IMPL_TC, name
    assert _spec("8x128_ldir5_noinput").dim_dir == 30

    arch, _, rays, z, blob = _setup("4x128_l1_skip2", "init", (9, 14), seed=12)
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
# As in test_simt_hidden256_gpu: the step forms depths and points in fp32, so the coarse network's worst element is
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
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    used = []
    render_fwd, render_bwd = ops.render_fwd, ops.render_bwd
    monkeypatch.setattr(ops, "render_fwd", lambda *a, **k: used.append(k["impl"]) or render_fwd(*a, **k))
    monkeypatch.setattr(ops, "render_bwd", lambda *a, **k: used.append(k["impl"]) or render_bwd(*a, **k))

    arch = _spec(name)
    g = torch.Generator().manual_seed(20)
    sds = [O.init_flexible_nerf(arch.num_layers, 128, arch.skip_every, arch.n_freq_xyz, arch.n_freq_dir, generator=g)
           for _ in range(2)]
    models = []
    for sd in sds:
        m = nb.FlexibleNeRFModel(num_layers=arch.num_layers, hidden_size=128, skip_connect_every=arch.skip_every,
                                 num_encoding_fn_xyz=arch.n_freq_xyz, num_encoding_fn_dir=arch.n_freq_dir)
        m.load_state_dict(sd)
        models.append(m.cuda())
    n, nc, nf = 96, 15, 49
    ro = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1) * 4.0
    rd = -ro / 4.0 + 0.25 * torch.randn(n, 3, generator=g)
    rnd = dict(t_rand=torch.rand(n, nc, generator=g), noise_c=torch.randn(n, nc, generator=g),
               u=torch.rand(n, nf, generator=g), noise_f=torch.randn(n, nc + nf, generator=g))
    target = torch.rand(n, 3, generator=g)
    opts = O.make_options(num_coarse=nc, num_fine=nf, perturb=True, radiance_field_noise_std=0.2)
    enc_xyz, enc_dir = (arch.n_freq_xyz, True, True), (arch.n_freq_dir, True, True)

    out = nb.run_one_iter_of_nerf(100, 100, 120.0, models[0], models[1], ro.cuda(), rd.cuda(), opts, mode="train",
                                  encode_position_fn=nb.get_embedding_function(*enc_xyz),
                                  encode_direction_fn=nb.get_embedding_function(*enc_dir),
                                  randoms={k: v.cuda() for k, v in rnd.items()})
    tgt = target.cuda()
    loss = torch.nn.functional.mse_loss(out[0], tgt) + torch.nn.functional.mse_loss(out[3], tgt)
    loss.backward()
    torch.cuda.synchronize()
    assert used and all(i == ops.IMPL_TC for i in used), used

    def oracle(dtype):
        sd_ = [{k: v.detach().to(dtype).clone().requires_grad_(True) for k, v in sd.items()} for sd in sds]
        out_ = O.run_one_iter_of_nerf(100, 100, 120.0, sd_[0], sd_[1], ro.to(dtype), rd.to(dtype), opts, mode="train",
                                      enc_xyz=enc_xyz, enc_dir=enc_dir, randoms={k: v.to(dtype) for k, v in rnd.items()})
        loss_ = O.nerf_loss(out_, target.to(dtype))
        loss_.backward()
        return loss_.item(), [{k: v.grad.double() for k, v in s.items()} for s in sd_]

    loss64, g64 = oracle(torch.float64)
    _, g32 = oracle(torch.float32)
    e_loss = abs(loss.item() - loss64) / abs(loss64)
    _report("e2e loss", (name,), e_loss)
    assert e_loss <= E2E_LOSS_TOL, (loss.item(), loss64)
    for i, (tag, model, samples) in enumerate((("coarse", models[0], nc), ("fine", models[1], nc + nf))):
        floor = -(-n * samples // 128) * FIX_LSB  # one fixed-point add per tile at most, per element
        num = den = 0.0
        count = 0
        for k, p in model.named_parameters():
            got, w = p.grad.double().cpu(), g64[i][k]
            num += (got - w).pow(2).sum().item()
            den += w.pow(2).sum().item()
            count += w.numel()
            if tag == "coarse":
                e, s = (got - w).abs().max().item(), w.abs().max().item()
                e_ref = max((g32[i][k] - w).abs().max().item(), 1e-6 * s)
                _report("e2e coarse worst / (fp32 oracle's + floor / bar)", (name, k),
                        e / (e_ref + floor / E2E_COARSE_VS_REF32))
                assert e <= E2E_COARSE_VS_REF32 * e_ref + floor, (name, k, e, e_ref, s)
        rel = (num / den) ** 0.5
        _report("e2e rel L2", (name, tag), rel)
        assert rel <= E2E_REL_L2 + count ** 0.5 * floor / den ** 0.5, (name, tag, rel)
