"""GPU: occupancy-grid, early-stopping and normal-map renders across every architecture the wgmma inference forward
takes.  These renders run the MLP over a row map (mlp_fwd_tc_kernel<false, kH, kFast, false, /*kMap=*/true>, launched by
launch_mlp_fwd_tc_map): the live block count comes from device memory, each 64-row block's rays from blocks[], and the
per-ray view bias is built for up to 10 rays per block.  Normal maps add the density gradient with its point count read
from device memory (density_grad_tc_kernel).

The architectures are mlp_checks.ALL_ARCHS at hidden 128 and H256_ARCHS at hidden 256 (one consumer warpgroup, 64-row
CTA tiles) but 8x256_ldir6, whose 39 direction channels the wgmma forward refuses; weights "init" and "scaled"; impl 1
and impl 3.  Small lego-camera renders, (rays, n_coarse, n_fine) from one ray at 15 coarse-only samples (the fewest the
wgmma path takes) to 20 x (64 + 960) (1024 samples, the most the renderer takes, 32 early-stop rounds); the ray counts
leave a partial last 10-ray group.  Grids: full, empty, random 10 % and 50 % at 32^3, and a box whose outside (always
evaluated) holds the first and last sample of every ray.

Per case, from the workspaces (ops.render_workspace_layout):
  1. a skipped sample's raw is exactly [0 0 0 -inf]; every other sample's raw is bit for bit the unmapped forward's
     (ops.mlp_fwd, same impl) at that point (include/nerfb200.h: a row's MLP result does not depend on its block);
     n_evaluated is the torch restatement's count (helpers.compaction_reference); impl 1: the evaluated raw against the
     fp64 oracle per column, within TC_FWD_TOL;
  2. early stopping at t = 0 is render_fwd_grid bit for bit; at t = 1e-2 on "scaled" weights, the per-ray contract:
     evaluated raw is the grid render's raw, stops fall on round boundaries, stop_sample is consistent, the fp64
     transmittance is below t at the stop and not below it at any earlier boundary (within T_REL);
  3. the sweep reaches the map's edges: a block holding rows of all 10 rays of its group (every viewb / encd slot),
     hidden-128 block counts at each residue mod 3 (the CTA tile is 3 blocks), an early-stop round without blocks;
  4. normal maps, on every architecture ops.density_grad_refusal accepts: the six outputs are those of the same render
     without normals, bit for bit; N against mlp_checks.normals64 (G_ERR, N_FLOOR); |N| <= acc + ACC_EPS, N = 0 where
     acc = 0.
Run with -s to print the measured figures beside their bars."""
import math

import pytest
import torch

import mlp_checks as M
from helpers import bits_equal, compaction_reference, transmittance64, ws_view
from mlp_checks import ACC_EPS, ALL_ARCHS, H256_ARCHS, STATES, T_REL, TC_FWD_TOL

pytestmark = pytest.mark.gpu

ARCHS = list(ALL_ARCHS) + [a for a in H256_ARCHS if a != "8x256_ldir6"]
IMPLS = {"impl1": 1, "impl3": 3}
SHAPES = [(1, 15, 0), (37, 15, 17), (41, 64, 128), (20, 64, 960)]  # (rays, n_coarse, n_fine)
GRIDS = ["full", "empty", "rand10", "rand50", "box"]
BOUNDS = ((-1.5,) * 3, (1.5,) * 3)
# every sample lies in [2, 6] along rays from radius 4 whose direction has unit component towards the centre, so the
# first and last sample of every ray are at least 2 from the centre: outside this box
BOX = ((-1.0,) * 3, (1.0,) * 3)
STOP_T = 1e-2
# their "scaled" weights leave sigma at or below zero along nearly every ray here, so no ray stops; the contract's other
# half (no stop where the transmittance is at or above t) still runs on them
NO_STOPS = ["6x128_skip1", "16x128_skip5"]
SKIP = torch.tensor([0.0, 0.0, 0.0, -math.inf])


def report(what, ctx, value):
    print(f"[map sweep] {what} {ctx}: {value}")


def _rays(arch, n, seed):
    """n rays of a 16 x 16 lego camera (near 2, far 6), a seeded choice of pixels; 8 columns without view directions."""
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    rays = ops.gen_rays(O.pose_spherical(30.0, -30.0, 4.0), 16, 16, 20.0, None, "cuda", near=2.0, far=6.0)
    pick = torch.randperm(256, generator=torch.Generator().manual_seed(seed))[:n].cuda()
    rays = rays[pick]
    return (rays if arch.use_viewdirs else rays[:, :8]).contiguous()


def _grid(kind):
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    g = torch.Generator(device="cuda").manual_seed(len(kind))
    if kind == "full":
        return OccupancyGrid.full(BOUNDS, 32)
    if kind == "empty":
        return OccupancyGrid.from_occupancy(BOUNDS, torch.zeros(32, 32, 32, dtype=torch.bool, device="cuda"))
    if kind == "box":
        return OccupancyGrid.from_occupancy(BOX, torch.rand(16, 16, 16, generator=g, device="cuda") < 0.3)
    return OccupancyGrid.from_occupancy(BOUNDS, torch.rand(32, 32, 32, generator=g, device="cuda") < int(kind[4:]) / 100)


def _setup(name, state):
    from nerf_pytorch_b200 import ops

    arch = M.spec(name)
    sd = M.arch_weights(arch, state)
    return arch, sd, ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))


def _passes(arch, blob, shape):
    """(arch_f, blob_f, opts, [(pass name, samples)]) of a shape: the same network in both passes."""
    from nerf_pytorch_b200 import ops

    n, nc, nf = shape
    opts = ops.make_opts(nc, nf, False, False, False, 0.0)
    passes = [("coarse", nc)] + ([("fine", nc + nf)] if nf else [])
    return (arch if nf else None), (blob if nf else None), opts, passes


class Edges:
    """What the compaction restatements of a run reach."""

    def __init__(self):
        self.full_group = False   # a block with rows of all 10 rays of its group
        self.residues = set()     # hidden 128: block counts mod 3 (live counts only)
        self.empty_round = False  # an early-stop round with no rows

    def blocks(self, arch, blocks, n_rays):
        self.full_group |= any(b - a + 1 == 10 for a, b in blocks)
        assert all(b - a + 1 <= 10 and a // 10 == b // 10 and b < n_rays for a, b in blocks)
        if arch.hidden == 128 and blocks:
            self.residues.add(len(blocks) % 3)

    def rounds(self, ran, S):
        K = _stop_round()
        n_rounds = -(-S // K)
        self.empty_round |= int(ran.max()) <= (n_rounds - 1) * K


def _stop_round():
    from nerf_pytorch_b200 import ops

    return ops.stop_round()


# ------------------------------------------------------------------------------------------------------------------------
# 1, 2. grid and early-stopping renders
# ------------------------------------------------------------------------------------------------------------------------
def _grid_case(arch, sd, blob, shape, kind, impl, edges, worst, stop_check):
    """One grid render and its early-stopping renders at t = 0 and, with stop_check, at STOP_T: checks 1 and 2.
    Records what the restated compactions reach in `edges` and the measured figures in `worst`."""
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    n = shape[0]
    rays = _rays(arch, n, seed=sum(shape))
    arch_f, blob_f, opts, passes = _passes(arch, blob, shape)
    grid = _grid(kind)
    rng = nb.SeededRandoms(3, 1)
    ctx = (M.arch_name(arch), shape, kind, impl)
    ne = torch.zeros(2, dtype=torch.int64, device="cuda")
    gc, gf, gws = ops.render_fwd_grid(arch, arch_f, opts, blob, blob_f, rays, rng, grid, impl=impl, n_evaluated=ne)
    lay = ops.render_workspace_layout(arch, arch_f, opts, n, False)
    keeps, zs, raws = [], [], []
    for i, (pname, s) in enumerate(passes):
        z = ws_view(gws, lay, f"z_{pname}", n, s, 1).clone()
        raw = ws_view(gws, lay, f"raw_{pname}", n, s, 4).clone()
        keep, _, blocks = compaction_reference(grid, rays, z)
        edges.blocks(arch, blocks, n)
        skip = ~keep
        assert torch.equal(raw[skip], SKIP.cuda().expand(int(skip.sum()), 4)), ctx + (pname,)
        assert ne[i].item() == int(keep.sum()), ctx + (pname, ne.tolist(), int(keep.sum()))
        ref = ops.mlp_fwd(arch, blob, rays, z, impl=impl)
        bad = (raw.view(torch.int32) != ref.view(torch.int32)).any(-1) & keep
        assert not bad.any(), ctx + (pname, "rows (ray, sample) differing from the unmapped forward",
                                     bad.nonzero()[:8].tolist())
        if impl == 1 and keep.any():
            want = M.oracle_tiles(arch, sd, rays, z).raw.view(n, s, 4)
            scale = want.abs().amax((0, 1))
            e = (raw[keep].double() - want[keep]).abs().amax(0)
            worst["raw"] = max(worst["raw"], (e / scale).max().item())
            assert (e <= TC_FWD_TOL * scale).all(), ctx + (pname, e.tolist(), scale.tolist())
        keeps.append(keep)
        zs.append(z)
        raws.append(raw)

    # early stopping at t = 0: the grid render bit for bit
    ec, ef, ne0, stop0 = ops.render_fwd_early_stop(arch, arch_f, opts, blob, blob_f, rays, rng, grid, 0.0, impl=impl,
                                                   want_stop=True)
    S = passes[-1][1]
    assert bits_equal(ec, gc) and bits_equal(ef, gf), ctx
    assert ne0.tolist() == ne.tolist() and (stop0 == S).all(), ctx
    edges.rounds(keeps[-1].sum(1), S)
    if not stop_check:
        return

    # at STOP_T: the per-ray contract on the last pass
    es_ws = torch.empty(ops.render_early_stop_workspace_bytes(arch, arch_f, opts, n), dtype=torch.uint8, device="cuda")
    ec, ef, ne_s, stop = ops.render_fwd_early_stop(arch, arch_f, opts, blob, blob_f, rays, rng, grid, STOP_T,
                                                   impl=impl, want_stop=True, workspace=es_ws)
    torch.cuda.synchronize()
    last, lname = (ef, gf) if arch_f is not None else (ec, gc), passes[-1][0]
    es_z, es_raw = ws_view(es_ws, lay, f"z_{lname}", n, S, 1), ws_view(es_ws, lay, f"raw_{lname}", n, S, 4)
    keep, z, raw = keeps[-1], zs[-1], raws[-1]
    stop = stop.long()
    assert bits_equal(es_z, z), ctx
    if arch_f is not None:
        assert bits_equal(ec, gc), ctx  # the coarse pass never stops
    K = ops.stop_round()
    j = torch.arange(S, device="cuda")[None, :]
    before = j < stop[:, None]
    want = torch.where((before | ~keep)[..., None], raw, SKIP.cuda().expand(n, S, 4))
    assert bits_equal(es_raw, want), ctx
    stopped = stop < S
    assert bits_equal(last[0][~stopped], last[1][~stopped]), ctx
    assert ne_s[len(passes) - 1].item() == int((keep & before).sum()), ctx
    rank = torch.cumsum(keep.long(), 1)
    n_keep = rank[:, -1]
    ran = (keep & before).sum(1)
    edges.rounds(ran, S)
    assert ((ran[stopped] % K) == 0).all() and (ran[stopped] > 0).all() and (ran[stopped] < n_keep[stopped]).all(), ctx
    last_ran = torch.where(keep & before, j, -1).max(1).values
    assert (stop[stopped] == last_ran[stopped] + 1).all(), ctx
    T = transmittance64(raw, z, rays, None, 0.0)
    if stopped.any():
        worst["stops"] += int(stopped.sum())
        at_stop = T[stopped, stop[stopped]]
        worst["T_stop"] = max(worst["T_stop"], (at_stop / STOP_T).max().item())
        assert (at_stop < STOP_T * (1 + T_REL)).all(), ctx
    boundary = keep & (rank % K == 0) & (rank < n_keep[:, None]) & (j < stop[:, None] - 1)
    rows, cols = boundary.nonzero(as_tuple=True)
    if rows.numel():
        earlier = T[rows, cols + 1]
        worst["T_earlier"] = min(worst["T_earlier"], (earlier / STOP_T).min().item())
        assert (earlier >= STOP_T * (1 - T_REL)).all(), ctx


@pytest.mark.parametrize("impl", list(IMPLS))
@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("name", ARCHS)
def test_grid_and_early_stop_renders_over_the_row_map(name, state, impl):
    arch, sd, blob = _setup(name, state)
    worst = dict(raw=0.0, T_stop=0.0, T_earlier=math.inf, stops=0)
    edges = Edges()
    for shape in SHAPES:
        for kind in GRIDS:
            _grid_case(arch, sd, blob, shape, kind, IMPLS[impl], edges, worst, state == "scaled")
    ctx = (name, state, impl)
    if IMPLS[impl] == 1:
        report(f"worst raw / column scale vs fp64 (bar TC_FWD_TOL {TC_FWD_TOL})", ctx, f"{worst['raw']:.3e}")
    if state == "scaled":
        report(f"stopped rays, max T64 / t at the stop, min at earlier boundaries (bar T_REL {T_REL})", ctx,
               (worst["stops"], worst["T_stop"], worst["T_earlier"]))
        assert (worst["stops"] > 0) == (name not in NO_STOPS), ctx  # the contract is not vacuous


# ------------------------------------------------------------------------------------------------------------------------
# 3. the edges the case list reaches
# ------------------------------------------------------------------------------------------------------------------------
def test_the_case_list_reaches_the_row_map_edges():
    """The compaction restatements of the sweep's shapes and grids, on a hidden-128 network, reach: a block with rows of
    all 10 rays of its group, block counts at each residue mod 3, and an early-stop round without rows.  A change of the
    case list that loses one of them fails here."""
    worst = dict(raw=0.0, T_stop=0.0, T_earlier=math.inf, stops=0)
    edges = Edges()
    arch, sd, blob = _setup("8x128_widest", "scaled")
    for shape in SHAPES:
        for kind in GRIDS:
            _grid_case(arch, sd, blob, shape, kind, 3, edges, worst, True)
    report("block with all 10 rays of its group, residues mod 3, empty round", (),
           (edges.full_group, sorted(edges.residues), edges.empty_round))
    assert edges.full_group and edges.residues == {0, 1, 2} and edges.empty_round
    assert worst["stops"] > 0


# ------------------------------------------------------------------------------------------------------------------------
# 4. normal maps
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("state", STATES)
@pytest.mark.parametrize("name", ARCHS)
def test_normal_maps_over_the_row_map(name, state):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    arch, sd, blob = _setup(name, state)
    why = ops.density_grad_refusal(arch)
    if why is not None:  # the library's refusal, before any launch
        before = ops.launch_count()
        rays = _rays(arch, 37, seed=1)
        with pytest.raises(NotImplementedError):
            ops.render_fwd_normals(arch, arch, ops.make_opts(15, 17, False, False, False, 0.0), blob, blob, rays, {})
        assert ops.launch_count() == before and "too deep" in why, why
        return
    worst = 0.0
    for shape in SHAPES[1:3]:
        n = shape[0]
        rays = _rays(arch, n, seed=sum(shape))
        arch_f, blob_f, opts, passes = _passes(arch, blob, shape)
        lname, S = passes[-1]
        for kind, stop in ((None, None), ("rand50", STOP_T), ("box", None), (None, STOP_T)):
            ctx = (name, state, shape, kind, stop)
            grid = _grid(kind) if kind else None
            rng = nb.SeededRandoms(5, 2)
            with torch.no_grad():
                oc, of, N, ws = ops.render_fwd_normals(arch, arch_f, opts, blob, blob_f, rays, rng, grid, stop, impl=1)
                if stop is not None:
                    pc, pf, _ = ops.render_fwd_early_stop(arch, arch_f, opts, blob, blob_f, rays, rng, grid, stop, impl=1)
                elif grid is not None:
                    pc, pf, _ = ops.render_fwd_grid(arch, arch_f, opts, blob, blob_f, rays, rng, grid, impl=1)
                else:
                    pc, pf, _ = ops.render_fwd(arch, arch_f, opts, blob, blob_f, rays, rng, training=False, impl=1)
            torch.cuda.synchronize()
            assert bits_equal(oc[:, :6], pc[:, :6]) and bits_equal(of[:, :6], pf[:, :6]), ctx
            lay = ops.render_workspace_layout(arch, arch_f, opts, n, False)
            z, raw = ws_view(ws, lay, f"z_{lname}", n, S, 1), ws_view(ws, lay, f"raw_{lname}", n, S, 4)
            N64, bound, _, _ = M.normals64(arch, sd, rays, z, raw)
            err = (N.double() - N64).abs().max(-1).values
            worst = max(worst, (err / bound).max().item())
            assert (err <= bound).all(), ctx + (err.max().item(),)
            acc = (of if arch_f is not None else oc)[:, 4]
            assert (N.norm(dim=-1) <= acc + ACC_EPS).all(), ctx
            assert (N[acc == 0] == 0).all(), ctx
    report("max |N - N64| / bound (G_ERR, N_FLOOR)", (name, state), f"{worst:.3f}")
