"""GPU: the hidden-128 wgmma forward where a CTA tile (192 points, three 64-row blocks, one per consumer warpgroup) and a
stash tile (128 points, two blocks) are different things.

Block b of a batch holds points [64 b, 64 b + 64); CTA tile b / 3 computes it and it is half b & 1 of stash tile b >> 1, so
every second stash tile has its two halves written by two different CTAs.  The sizes here put the end of the batch at
every place the two tilings can disagree about:
  * P = 64 k - 1, 64 k, 64 k + 1 for k = 1, 3 and 6: the last CTA tile has one, two or three live blocks, the last block
    is full or holds one or 63 points, and the last stash tile has one half past P (filled from the last point, as the
    backward reads whole tiles) or, beyond it, a block of the CTA tile that has no stash tile at all and must write nothing;
  * fewer than 64 points; exactly one CTA tile (1 x 192, also the longest run inside one ray) ;
  * 15 samples per ray: 10 rays per block, every ray slot of the per-ray view bias;
  * one and two blocks more than three per multiprocessor, whole and ragged: the last round of the persistent CTAs runs
    one CTA with one or two live warpgroups while its others walk the weight ring without work.
Checks: raw of the stash-writing, inference and point-source (run_network) forwards against fp64 and equal bit for bit;
the single-pass forward (impl 3) at its own bar; every stash tile (activations, encoding tile, mask words) against fp64
through the shared stash reader, rows up to P; then the fused backward on that stash against fp64 autograd, block by
block, which it can only pass if both kernels agree on where each block's rows are."""
import pytest
import torch

from mlp_checks import (STASH_TOL, TC_FWD_TOL as FWD_TOL, BLOCK_TOL, StashLayout, _floors, _in_blob_range,
                        _split_floors, check_blocks, encodings, oracle, read_layer, relu_ties, report, setup, sms,
                        tc_blocks, upstream)

pytestmark = pytest.mark.gpu

FAST_TOL = 2e-2  # impl 3 against fp64, per column of raw (tests/test_tc_fast_gpu.py measures 6.7e-3 at worst)

ARCHS = ["8x128_noinput_linear", "4x128_l1_skip2"]  # A1's shape (skip 3, 64-wide encoding tile); a 16-wide encoding tile
# (rays, samples); "3sms+1" = three blocks per multiprocessor and one more
SHAPES = [(1, 15), (1, 63), (1, 64), (1, 65), (1, 191), (1, 192), (1, 193), (1, 383), (3, 128), (7, 55), (37, 15),
          ("3sms+1", 64), ("3sms+2", 64), ("3sms+1", 63), ("6sms+2", 33)]
BWD_SHAPES = [(1, 65), (1, 193), (7, 55), (37, 15), ("3sms+1", 63), ("6sms+2", 33)]


def _shape(shape):
    n, s = shape
    if isinstance(n, str):
        k, extra = n.split("sms+")
        n = int(k) * sms() + int(extra)
    return n, s


def _id(shape):
    return f"{shape[0]}x{shape[1]}"


@pytest.mark.parametrize("shape", SHAPES, ids=_id)
@pytest.mark.parametrize("name", ARCHS)
def test_forward_raw_and_stash_tiles_match_fp64(name, shape):
    from nerf_pytorch_b200 import ops

    arch, sd, rays, z, blob = setup(name, "init", _shape(shape), seed=31)
    n, s = z.shape
    P = n * s
    ctx = (name, (n, s))
    rays_c, z_c = rays.cuda(), z.cuda()
    raw, stash = ops.mlp_fwd(arch, blob, rays_c, z_c, impl=ops.IMPL_TC, want_stash=True)
    raw_inf = ops.mlp_fwd(arch, blob, rays_c, z_c, impl=ops.IMPL_TC)
    raw_fast = ops.mlp_fwd(arch, blob, rays_c, z_c, impl=ops.IMPL_TC_FAST)
    # the same points as run_network's caller would form them: o + d z in fp32, two roundings
    pts = (rays_c[:, None, :3] + rays_c[:, None, 3:6] * z_c[..., None]).contiguous()
    raw_pts, stash_pts = ops.mlp_fwd_pts(arch, blob, pts, rays_c[:, 8:11], impl=ops.IMPL_TC, want_stash=True)
    torch.cuda.synchronize()
    want, acts, _, _ = oracle(arch, sd, rays, z)
    scale = want.abs().amax(0)
    for what, r, tol in (("train", raw, FWD_TOL), ("inference", raw_inf, FWD_TOL), ("single pass", raw_fast, FAST_TOL)):
        e = (r.reshape(-1, 4).double().cpu() - want).abs().amax(0)
        report(f"forward raw ({what})", ctx, (e / scale).max().item())
        assert (e <= tol * scale).all(), ctx + (what, e.tolist(), scale.tolist())
    assert torch.equal(raw, raw_inf), ctx
    assert torch.equal(raw, raw_pts), ctx

    lay = StashLayout(arch)
    emb = encodings(arch, rays, z)[0]
    worst = 0.0
    for st in (stash, stash_pts):
        tile = read_layer(st, P, lay.cum_total, lay.enc_w, "wgmma").cpu()
        assert (tile[:, arch.dim_xyz:] == 0).all(), ctx
        ee = (tile[:, :arch.dim_xyz] - emb).abs().max().item() / emb.abs().max().item()
        assert ee <= STASH_TOL, ctx + ("xyz encoding", ee)
        worst = max(worst, ee)
        for li, (lname, width, cum) in enumerate(lay.layers):
            a = read_layer(st, P, cum, width, "wgmma").cpu()
            ea = (a - acts[li]).abs().max().item() / acts[li].abs().max().item()
            assert ea <= STASH_TOL, ctx + (lname, ea)
            worst = max(worst, ea)
        relu_ties(arch, st, P, acts, "wgmma", STASH_TOL, ctx, adopt=False)
    report("forward stash", ctx, worst)


@pytest.mark.parametrize("shape", BWD_SHAPES, ids=_id)
@pytest.mark.parametrize("name", ARCHS)
def test_backward_reads_the_stash_the_forward_wrote(name, shape):
    from nerf_pytorch_b200 import ops

    arch, sd, rays, z, blob = setup(name, "init", _shape(shape), seed=33)
    n, s = z.shape
    P = n * s
    ctx = (name, (n, s))
    G, acts, dpre, want = _in_blob_range(arch, sd, rays, z, upstream(n, s, seed=34))
    rays_c, z_c, G_c = rays.cuda(), z.cuda(), G.cuda().contiguous()
    _, stash = ops.mlp_fwd(arch, blob, rays_c, z_c, impl=ops.IMPL_TC, want_stash=True)
    relu_ties(arch, stash, P, acts, "wgmma", STASH_TOL, ctx, adopt=True)
    g, _ = ops.mlp_bwd(arch, blob, rays_c, z_c, G_c, stash, impl=ops.IMPL_TC)
    torch.cuda.synchronize()
    assert torch.isfinite(g).all(), ctx
    check_blocks(arch, g, want, tc_blocks(arch), BLOCK_TOL, ctx, "wgmma backward blocks",
                 _floors(arch, P, _split_floors(arch, G, acts, dpre, rays, z)))
