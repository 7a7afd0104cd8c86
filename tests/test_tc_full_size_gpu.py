"""GPU: the wgmma forward and fused backward at the training batch against fp64, every point, every block and single
tiles.

The bench step (A1, 4096 rays x (64 + 128) samples) gives the fine pass 6144 tiles of 128 points, so each persistent
CTA runs 46 or 47 of them on a 132-SM H100, and its 4.1 GB stash lies mostly beyond 2^31 bytes.  The sweep
(test_tc_arch_sweep_gpu.py) stops at about four tiles per CTA; what only shows after many tiles per CTA -- a stale or
early-overwritten activation tile, an mbarrier phase that drifts, the one-job-ahead stash load crossing into the next
tile or past a CTA's last, the partial last wave -- is checked here, with the oracle of mlp_checks.py run on the device
in chunks of whole tiles (oracle_tiles):
  1. forward, stash-writing and inference: raw outputs per column at every point, every stashed activation tile and the
     xyz-encoding tile, the ReLU ties; a failure names the worst tile and the CTA that ran it;
  2. backward on the oracle's ReLU decisions, every block of tc_blocks, with the fp32 kernels as the control, under
     the upstream gradient of an MSE loss through the compositing of those samples, scaled by a power of two (exact)
     so that max |d_raw| lies in [4, 8): the distribution training produces, clear of the absolute fixed-point floor;
  3. single-tile probes: d_raw zero but on one tile (the first, either side of the first wave's end, CTA 0's 47th,
     the last CTA's 46th, the last and the ragged partial one), against the oracle on that tile's points alone, so a
     tile lost, repeated or swapped shows undiluted;
  4. exact cases at full size: zero d_raw gives exact zeros and leaves a non-zero flat_grad's bits alone, and two runs
     give the same bits;
  5. run_network on a 128^3 density grid, one row of 16384 tiles, forward and parameter gradients.
Tile counts and probe tiles follow the device's multiprocessor count (sms()).

Bars are the sweep's: errors are relative to each block's or column's scale, and a per-tile error does not grow with the
tile count.  The whole file runs in about 25 s on an H100 and holds at most 8.1 GiB of device memory (the A1 fine
pass's fp32 stash and gradient stash; every case frees its stashes and the oracle's chunks before the next)."""
import math
import time

import pytest
import torch

from helpers import load_weights
from mlp_checks import (BLOCK_TOL, FP32_TIE_TOL, SIMT_FWD_TOL, STASH_TOL, TC_FWD_TOL, StashLayout, _adopt_masks,
                        _floors, _split_floors, arch_weights, blob_range_factor, check_blocks, encodings, oracle,
                        oracle_tiles, pack_mask, points, random_previous, read_layer, relu_ties, report, sms, tc_blocks,
                        upstream)

pytestmark = pytest.mark.gpu

# Worst element as a fraction of the compared scale: the bars of test_tc_arch_sweep_gpu.py (TC_FWD_TOL, BLOCK_TOL,
# SIMT_FWD_TOL, all 3e-5, and STASH_TOL, 2e-5, for stashed activation and encoding tiles too, from mlp_checks), the worst
# figure over this file's cases in brackets, measured on an H100 80GB HBM3 at a 700 W power limit and 1980 MHz SM clock.
# wgmma forward raw [2.8e-5, A0 fern]: its pretrained weights far outside their scene; stashed tiles [1.1e-5, A0 fern];
# parameter gradients per block: wgmma [6.3e-6, a probe], fp32 kernels [4.1e-6, A2]; the fp32 kernels' raw [7.8e-7].
ORACLE_PIN = 1e-12   # the device oracle against the CPU oracle, relative to each tensor's scale [2.4e-15]

NETS = {  # ops.ArchSpec arguments
    "A1": dict(num_layers=8, hidden=128, skip_every=3, n_freq_xyz=10, n_freq_dir=4),   # bench A1, config/lego.yml
    "A0": dict(num_layers=4, hidden=128, skip_every=4, n_freq_xyz=10, n_freq_dir=4),   # the pretrained lego network
    "A0_fern": dict(num_layers=4, hidden=128, skip_every=4, n_freq_xyz=6, n_freq_dir=4),  # config 4's network
    "A2": dict(num_layers=8, hidden=256, skip_every=4, n_freq_xyz=10, n_freq_dir=4),   # hidden 256: the fp32 kernels
}
FINE, COARSE = (4096, 192), (4096, 64)
RAGGED = "ragged"  # 46 sms + 1 tiles of A1 at an odd sample count, the last one partial


@pytest.fixture(autouse=True)
def _free_and_measure():
    """Every case starts from an empty cache and prints its peak device memory and time."""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB, {time.perf_counter() - t:.1f} s")
    torch.cuda.empty_cache()


def _net(name, weights):
    """ArchSpec and state_dict: "init" / "scaled" (mlp_checks.arch_weights) or a pretrained fine network."""
    from nerf_pytorch_b200 import ops

    arch = ops.ArchSpec(**NETS[name])
    if weights in ("lego", "fern"):
        return arch, load_weights(weights + "_lowres")[1]
    return arch, arch_weights(arch, weights)


def _shape(shape):
    """(rays, samples); RAGGED: 46 sms + 1 tiles at 199 samples per ray, the last tile partial."""
    if shape != RAGGED:
        return shape
    tiles = 46 * sms() + 1
    n = (tiles - 1) * 128 // 199 + 1
    assert (tiles - 1) * 128 < n * 199 < tiles * 128, (n, tiles)
    return n, 199


def _where(tile, n_tiles):
    grid = min(n_tiles, sms())
    return f"tile {tile} of {n_tiles}: CTA {tile % grid}'s tile {tile // grid}"


def _per_tile(e, n_tiles):
    """Per-point figures [P] -> the worst of every 128-point tile [n_tiles]."""
    return torch.nn.functional.pad(e, (0, n_tiles * 128 - e.numel())).view(n_tiles, 128).amax(1)


def _to_4_8(G):
    """G times the power of two that puts max |G| in [4, 8) (exact)."""
    return G * 2.0 ** (3 - math.frexp(G.abs().max().item())[1])


def _setup(name, weights, shape, seed):
    """arch, weights, rays and depths on the device, the packed weights."""
    from nerf_pytorch_b200 import ops

    arch, sd = _net(name, weights)
    rays, z = points(arch, *_shape(shape), seed=seed)
    blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))
    return arch, sd, rays.cuda(), z.cuda(), blob


def _compositing_upstream(raw, rays, z, seed):
    """d(loss)/d(raw) of the MSE of the composited colour against seeded targets, scaled to max |d_raw| in [4, 8)."""
    import nerf_pytorch_b200 as nb

    target = torch.rand(z.shape[0], 3, generator=torch.Generator().manual_seed(seed)).cuda()
    r = raw.detach().requires_grad_(True)
    rgb = nb.volume_render_radiance_field(r, z, rays[:, 3:6], 0.0, False)[0]
    G, = torch.autograd.grad(torch.nn.functional.mse_loss(rgb, target), r)
    return _to_4_8(G).contiguous()


# ------------------------------------------------------------------------------------------------------------------------
# 0. the device oracle is the CPU oracle
# ------------------------------------------------------------------------------------------------------------------------
def test_device_oracle_in_tile_chunks_matches_the_cpu_oracle():
    """oracle_tiles on the device, in chunks of 3 tiles over 5 rays x 199 samples (a partial last tile), against
    mlp_checks.oracle on the CPU in one piece: raw, ReLU decisions, max |activation|, every parameter gradient and the
    split floors to 1e-12 of scale; a tile range gives the same rows."""
    arch, sd = _net("A1", "scaled")
    rays, z = points(arch, 5, 199, seed=3)
    G = upstream(5, 199, seed=4)
    raw, acts, dpre, want = oracle(arch, sd, rays, z, G)
    split = _split_floors(arch, G, acts, dpre, rays, z)
    dev = oracle_tiles(arch, sd, rays.cuda(), z.cuda(), G.cuda(), chunk_tiles=3)

    def rel(a, b):
        return (a.cpu() - b).abs().max().item() / b.abs().max().item()

    worst = rel(dev.raw, raw)
    for li, a in enumerate(acts):
        assert torch.equal(dev.masks[li].cpu(), pack_mask(a > 0)), li
        worst = max(worst, abs(dev.act_max[li] - a.abs().max().item()) / a.abs().max().item())
    for k, v in want.items():
        worst = max(worst, rel(dev.grads[k], v))
    for label, v in split.items():
        worst = max(worst, abs(dev.split[label] - v) / v)
    report("device oracle vs CPU oracle", ("A1", "scaled"), worst)
    assert worst <= ORACLE_PIN
    part = oracle_tiles(arch, sd, rays.cuda(), z.cuda(), tiles=(3, 8), chunk_tiles=2)
    assert part.raw.shape == (5 * 199 - 384, 4) and rel(part.raw, dev.raw[384:].cpu()) <= ORACLE_PIN


# ------------------------------------------------------------------------------------------------------------------------
# 1-2. every point forward, every block backward
# ------------------------------------------------------------------------------------------------------------------------
def _check_forward(arch, sd, rays, z, blob, ref, ctx):
    """Stash-writing and inference raw outputs per column against ref.raw (the same bits); every stashed activation
    tile and the xyz-encoding tile; the ReLU ties.  Returns the stash."""
    from nerf_pytorch_b200 import ops

    P = z.numel()
    n_tiles = -(-P // 128)
    raw, stash = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC, want_stash=True)
    raw_inf = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC)
    assert torch.equal(raw, raw_inf), ctx
    del raw_inf
    scale = ref.raw.abs().amax(0)
    tiles = _per_tile(((raw.reshape(-1, 4).double() - ref.raw).abs() / scale).amax(1), n_tiles)
    t = int(tiles.argmax())
    report("full-size forward raw", ctx, tiles[t].item())
    assert tiles[t] <= TC_FWD_TOL, ctx + (_where(t, n_tiles), tiles[t].item())

    lay = StashLayout(arch)
    err = torch.zeros(len(lay.layers) + 1, n_tiles, dtype=torch.float64, device=z.device)  # absolute, per tile
    enc_max, ties = [0.0], [0]

    def visit(p0, p1, rays_c, z_c, acts):
        t0, t1 = p0 // 128, -(-p1 // 128)
        xyz = encodings(arch, rays_c, z_c)[0]
        enc = read_layer(stash, P, lay.cum_total, lay.enc_w, "wgmma", (p0, p1))
        assert (enc[:, arch.dim_xyz:] == 0).all(), ctx + ("xyz encoding padding", p0)
        err[-1, t0:t1] = _per_tile((enc[:, :arch.dim_xyz] - xyz).abs().amax(1), t1 - t0)
        enc_max[0] = max(enc_max[0], xyz.abs().max().item())
        for li, (_, n, cum) in enumerate(lay.layers):
            a = read_layer(stash, P, cum, n, "wgmma", (p0, p1))
            err[li, t0:t1] = _per_tile((a - acts[li]).abs().amax(1), t1 - t0)
        ties[0] += relu_ties(arch, stash, P, acts, "wgmma", STASH_TOL, ctx + (p0,), adopt=False, rows=(p0, p1),
                             scales=ref.act_max)

    oracle_tiles(arch, sd, rays, z, visit=visit)
    rel = err / torch.tensor(ref.act_max + enc_max, dtype=torch.float64, device=z.device)[:, None]
    worst = rel.amax(0)
    t = int(worst.argmax())
    report("full-size forward stash", ctx, worst[t].item())
    names = [lname for lname, _, _ in lay.layers] + ["xyz encoding"]
    assert worst[t] <= STASH_TOL, ctx + (_where(t, n_tiles), names[int(rel[:, t].argmax())], worst[t].item())
    report("full-size relu ties", ctx, ties[0])
    assert ties[0] <= 1e-5 * P * lay.cum_total + 2, ctx + (ties[0],)
    return stash


def _check_backward_fp32(arch, sd, rays, z, blob, G, ref, ctx):
    """The fp32 kernels' backward with the oracle's ReLU decisions (ties adopted chunk by chunk), every block."""
    from nerf_pytorch_b200 import ops

    P = z.numel()
    _, stash32 = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_SIMT, want_stash=True)
    ties = [0]

    def visit(p0, p1, rays_c, z_c, acts):
        ties[0] += relu_ties(arch, stash32, P, acts, "fp32", FP32_TIE_TOL, ctx + ("fp32", p0), adopt=True,
                             rows=(p0, p1), scales=ref.act_max)

    oracle_tiles(arch, sd, rays, z, visit=visit)
    report("full-size relu ties", ctx + ("fp32",), ties[0])
    g32, _ = ops.mlp_bwd(arch, blob, rays, z, G, stash32, impl=ops.IMPL_SIMT)
    del stash32
    check_blocks(arch, g32, ref.grads, tc_blocks(arch), BLOCK_TOL, ctx, "full-size fp32 backward blocks",
                 _floors(arch, P))


def _oracle_with_upstream(arch, sd, rays, z, raw, seed):
    """The compositing upstream gradient of raw (brought into the blob's range if needed, exact) and the oracle with
    it."""
    G = _compositing_upstream(raw, rays, z, seed)
    ref = oracle_tiles(arch, sd, rays, z, G)
    c = blob_range_factor(ref.grads)
    if c != 1.0:
        G = G * c
        ref.grads = {k: v * c for k, v in ref.grads.items()}
        ref.split = {k: v * c for k, v in ref.split.items()}
    return G, ref


CASES = [("A1", "init", FINE), ("A1", "scaled", FINE), ("A1", "init", COARSE), ("A1", "scaled", COARSE),
         ("A0", "lego", FINE), ("A0_fern", "fern", FINE), ("A1", "init", RAGGED)]


@pytest.mark.parametrize("name, weights, shape", CASES, ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple)
                         else str(v))
def test_full_size_forward_and_backward_match_fp64(name, weights, shape):
    """mlp_fwd (both wgmma instances) and mlp_bwd on wgmma at every point and every block of a training batch against
    the fp64 oracle, the fp32 kernels' backward through the same block check."""
    from nerf_pytorch_b200 import ops

    arch, sd, rays, z, blob = _setup(name, weights, shape, seed=1)
    P = z.numel()
    ctx = (name, weights, tuple(z.shape))
    assert ops.impl_supported(arch, z.shape[1], ops.IMPL_TC), ctx
    raw = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC)
    G, ref = _oracle_with_upstream(arch, sd, rays, z, raw, seed=2)
    del raw
    report("full-size max |d_raw|", ctx, G.abs().max().item())
    stash = _check_forward(arch, sd, rays, z, blob, ref, ctx)
    _adopt_masks(arch, stash, P, ref.masks)
    g, _ = ops.mlp_bwd(arch, blob, rays, z, G, stash, impl=ops.IMPL_TC)
    del stash
    check_blocks(arch, g, ref.grads, tc_blocks(arch), BLOCK_TOL, ctx, "full-size wgmma backward blocks",
                 _floors(arch, P, ref.split))
    _check_backward_fp32(arch, sd, rays, z, blob, G, ref, ctx)


def test_full_size_hidden256_backward_on_the_fp32_kernels_matches_fp64():
    """A2 (8x256 skip 4), the hidden-256 training path, on the fp32 kernels at 4096 x 64: raw outputs at every point,
    every block of the backward (4096 x 192 would put fp32 stash and gradient stash at ~20 GB)."""
    from nerf_pytorch_b200 import ops

    arch, sd, rays, z, blob = _setup("A2", "init", COARSE, seed=5)
    ctx = ("A2", "init", tuple(z.shape))
    assert not ops.impl_supported(arch, z.shape[1], ops.IMPL_TC), ctx
    raw = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_SIMT)
    G, ref = _oracle_with_upstream(arch, sd, rays, z, raw, seed=6)
    e = ((raw.reshape(-1, 4).double() - ref.raw).abs() / ref.raw.abs().amax(0)).max().item()
    del raw
    report("full-size fp32 forward raw", ctx, e)
    assert e <= SIMT_FWD_TOL, ctx
    _check_backward_fp32(arch, sd, rays, z, blob, G, ref, ctx)


# ------------------------------------------------------------------------------------------------------------------------
# 3. single-tile probes
# ------------------------------------------------------------------------------------------------------------------------
def _probe_tiles(n_tiles):
    """The first tile; the last of the first wave and the first of the second; CTA 0's 47th tile; the last CTA's 46th;
    the last tile (in the ragged case also CTA 0's 47th, and partial)."""
    m = sms()
    return sorted(t for t in {0, m - 1, m, 46 * m, m - 1 + 45 * m, n_tiles - 1} if t < n_tiles)


@pytest.mark.parametrize("name, weights, shape", [("A1", "init", FINE), ("A1", "scaled", FINE), ("A1", "init", RAGGED)],
                         ids=lambda v: "x".join(map(str, v)) if isinstance(v, tuple) else str(v))
def test_single_tile_probes_match_fp64_per_block(name, weights, shape):
    """d_raw zero except on one tile, through the fused backward over the whole batch's stash with the oracle's ReLU
    decisions, against the oracle on that tile's points alone.  The tile's d_raw is mlp_checks.upstream's, rows spanning
    several decades, scaled to [4, 8): behind an opaque sample the compositing gradient is exactly zero, so at "scaled"
    weights most tiles of a ray would have nothing to probe."""
    from nerf_pytorch_b200 import ops

    arch, sd, rays, z, blob = _setup(name, weights, shape, seed=1)
    P = z.numel()
    n_tiles = -(-P // 128)
    _, stash = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC, want_stash=True)
    G = upstream(*z.shape, seed=2).cuda()
    _adopt_masks(arch, stash, P, oracle_tiles(arch, sd, rays, z).masks)
    for t in _probe_tiles(n_tiles):
        ctx = (name, weights, tuple(z.shape), _where(t, n_tiles))
        rows = slice(128 * t, min(128 * t + 128, P))
        Gt = torch.zeros_like(G)
        Gt.view(-1, 4)[rows] = G.view(-1, 4)[rows]
        Gt = _to_4_8(Gt)
        ref = oracle_tiles(arch, sd, rays, z, Gt, tiles=(t, t + 1))
        g, _ = ops.mlp_bwd(arch, blob, rays, z, Gt, stash, impl=ops.IMPL_TC)
        check_blocks(arch, g, ref.grads, tc_blocks(arch), BLOCK_TOL, ctx, "probe wgmma backward blocks",
                     _floors(arch, rows.stop - rows.start, ref.split))


# ------------------------------------------------------------------------------------------------------------------------
# 4. exact cases at full size
# ------------------------------------------------------------------------------------------------------------------------
def test_full_size_zero_upstream_and_repeats_are_exact():
    """A1 at 4096 x 192 on wgmma: zero d_raw gives a flat gradient of exact zeros and leaves a non-zero flat_grad's bits
    unchanged; two runs on the compositing gradient give the same bits."""
    from nerf_pytorch_b200 import ops

    arch, sd, rays, z, blob = _setup("A1", "init", FINE, seed=1)
    raw, stash = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC, want_stash=True)
    G = _compositing_upstream(raw, rays, z, seed=2)
    zero = torch.zeros_like(G)
    g0, _ = ops.mlp_bwd(arch, blob, rays, z, zero, stash, impl=ops.IMPL_TC)
    assert (g0.view(torch.int32) == 0).all()
    g1, _ = ops.mlp_bwd(arch, blob, rays, z, G, stash, impl=ops.IMPL_TC)
    g2, _ = ops.mlp_bwd(arch, blob, rays, z, G, stash, impl=ops.IMPL_TC)
    assert torch.equal(g1.view(torch.int32), g2.view(torch.int32))
    prev = random_previous(arch, g1, tc_blocks(arch), seed=3).cuda()
    g3, _ = ops.mlp_bwd(arch, blob, rays, z, zero, stash, impl=ops.IMPL_TC, flat_grad=prev.clone())
    assert torch.equal(g3.view(torch.int32), prev.view(torch.int32))


# ------------------------------------------------------------------------------------------------------------------------
# 5. a density grid through run_network
# ------------------------------------------------------------------------------------------------------------------------
def test_density_grid_run_network_matches_fp64():
    """run_network (impl 1) on the pretrained lego A0 coarse network over 1 x 128^3 points with one view direction: one
    row of 16384 tiles through the per-ray sums and the per-CTA direction-encoding sums.  The forward per point and
    column against fp64; the parameter gradients of sum(raw * u) are those of mlp_bwd_pts on the same stash, bit for
    bit, and with the oracle's ReLU decisions adopted in that stash they match fp64 per block.  u weights density and
    colour alike: with density alone the colour branch (fc_feat, layers_dir.0 with its direction-encoding sums, fc_rgb)
    would get an exact zero gradient and check nothing.  (With u of random sign the gradient sums cancel to ~sqrt(P)
    points' worth, so a single ReLU tie's point would show in every block.)"""
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    arch = ops.ArchSpec(**NETS["A0"])
    sd = load_weights("lego_lowres")[0]
    model = nb.FlexibleNeRFModel(num_layers=4, hidden_size=128, skip_connect_every=4, num_encoding_fn_xyz=10,
                                 num_encoding_fn_dir=4)
    model.load_state_dict(sd)
    model.cuda()
    t = torch.linspace(-1.5, 1.5, 128, device="cuda")
    grid = torch.stack(torch.meshgrid(t, t, t, indexing="ij"), -1).reshape(1, -1, 3)
    view = torch.tensor([[0.0, 0.0, 1.0]], device="cuda")
    P = grid.shape[1]
    n_tiles = P // 128
    u = torch.randn(1, P, 4, generator=torch.Generator().manual_seed(7)).cuda()
    raw = nb.run_network(model, grid, view, 65536, nb.get_embedding_function(10), nb.get_embedding_function(4), impl=1)
    (raw * u).sum().backward()
    got = ops.flatten_state_dict(arch, {k: p.grad for k, p in model.named_parameters()}, "cuda")
    G = u
    blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))
    raw_ops, stash = ops.mlp_fwd_pts(arch, blob, grid, view, impl=ops.IMPL_TC, want_stash=True)
    assert torch.equal(raw_ops, raw.detach())
    assert torch.equal(ops.mlp_bwd_pts(arch, blob, view, G, stash, impl=ops.IMPL_TC), got)

    # every point a ray [pts, d = 0, near, far, view direction] at z = 0: pts + 0 * 0 = pts
    rays = torch.cat([grid[0], torch.zeros(P, 3, device="cuda"), torch.full((P, 1), 2.0, device="cuda"),
                      torch.full((P, 1), 6.0, device="cuda"), view.expand(P, 3)], -1)
    z0 = torch.zeros(P, 1, device="cuda")
    ref = oracle_tiles(arch, sd, rays, z0, G.view(P, 1, 4))
    assert blob_range_factor(ref.grads) == 1.0
    ctx = ("A0 lego", "density grid", P)
    tiles = _per_tile(((raw_ops.reshape(-1, 4).double() - ref.raw).abs() / ref.raw.abs().amax(0)).amax(1), n_tiles)
    k = int(tiles.argmax())
    report("density grid forward raw", ctx, tiles[k].item())
    assert tiles[k] <= TC_FWD_TOL, ctx + (_where(k, n_tiles), tiles[k].item())
    ties = [0]

    def visit(p0, p1, rays_c, z_c, acts):
        ties[0] += relu_ties(arch, stash, P, acts, "wgmma", STASH_TOL, ctx + (p0,), adopt=True, rows=(p0, p1),
                             scales=ref.act_max)

    oracle_tiles(arch, sd, rays, z0, visit=visit)
    report("density grid relu ties", ctx, ties[0])
    assert ties[0] <= 1e-5 * P * StashLayout(arch).cum_total + 2, ctx + (ties[0],)
    g = ops.mlp_bwd_pts(arch, blob, view, G, stash, impl=ops.IMPL_TC)
    check_blocks(arch, g, ref.grads, tc_blocks(arch), BLOCK_TOL, ctx, "density grid backward blocks",
                 _floors(arch, P, ref.split))
