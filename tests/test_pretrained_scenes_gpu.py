"""GPU: every kernel path on the seven pretrained low-res networks (chair, drums, fern, hotdog, lego, materials, ship;
coarse and fine) against fp64, at the points their own scenes' renders sample.

Trained networks reach activations that default or scaled init weights never do, and those magnitudes are where the
fp16 x 2 split of the wgmma kernels could run out of range (|value| >= 16 x 65504 = 1.05e6).  Every scene is A0 by its
weights' shapes (helpers.PRETRAINED_SCENES), so all of them run the default wgmma path.  Per scene, on rays of several
poses of its own camera ring (helpers.pretrained_poses):
  1. training step (impl 1 and impl 0, 4096 rays, the config's sample counts, perturb and noise): d_raw against fp64
     autograd of the compositing, then every parameter block of both networks against the fp64 oracle at the kernel's
     own d_raw with its ReLU decisions adopted, at the training loss's scale and at max |d_raw| in [4, 8); the heads
     (fc_rgb, fc_alpha) and layers_dir.0 are reported on their own;
  2. the stash tiles (impl 1): every stashed activation read back against fp64, and every layer's fp64 maximum inside
     the split's range -- a failure names the layer that left it;
  3. the inference forward on impl 1, 0 and 3, at the render's points and at uniform points of the scene's box;
  4. compositing of both passes (rgb, disp, acc, depth, weights) against helpers.composite64 of the kernel's raw;
  5. the density gradient at box points against fp64 autograd;
  6. a 128^3 bake, fp32 and fp16, against the network.
The bars are the suite's own (mlp_checks and the files named beside the others).  Worst over this file's cases, measured
on an H100 80GB HBM3 at a 700 W power limit and 1980 MHz SM clock, where the file runs in 47 s: parameter blocks, figure
/ (scale + floor / bar), 5.6e-6 (fc_alpha, materials coarse), fc_rgb 2.4e-6, layers_dir.0 3.5e-6, trunk and fc_feat
5.4e-6; d_raw 1.8e-6; compositing outputs 1.8e-6, disp 2.3e-3 of its bar; stash tiles 6.9e-6 of the layer's scale;
raw per column impl 1 2.0e-5, impl 0 1.2e-5, impl 3 1.1e-2 (all fern fine); density gradient 2.2e-6 off ReLU ties
(2.5e-2 at them); bake coefficients 2.2e-6.  The largest activation is drums coarse's layers_dir.0 output, 0.26 of the split's range."""
import math

import pytest
import torch

from helpers import (COEF_REL, PRETRAINED_BOX, PRETRAINED_SCENES, bits_equal, composite64, composite_grad64,
                     load_weights, net_at, pretrained_arch, pretrained_poses)
from mlp_checks import (BLOCK_TOL, COMP_GRAD_TOL, COMP_TOL, FP32_TIE_TOL, SIMT_FWD_TOL, STASH_TOL, TC_FWD_TOL,
                        StashLayout, _floors, blob_range_factor, check_blocks, oracle, oracle_tiles, read_layer,
                        relu_ties, report, sigma_grad64, tc_blocks)

pytestmark = pytest.mark.gpu

SCENES = sorted(PRETRAINED_SCENES)
NETS = ["coarse", "fine"]
POSES = 4
N_RAYS = 4096
SPLIT_MAX = 16.0 * 65504.0  # value / 16 must stay an fp16 number (csrc/tc_common.cuh, kActScale)
# The single-pass fp16 forward (impl 3) per column against fp64 (test_tc_fast_gpu.py FAST_TOL).
FAST_TOL = 2e-2
# The density gradient against fp64 relative to the batch's max |grad|, off ReLU ties, and at a tie
# (test_density_grad_gpu.py GRAD_TOL, TIE_GRAD_TOL).
GRAD_TOL = 2e-5
TIE_GRAD_TOL = 0.2
DISP_K = 4.0  # disp's bar on rays with small acc (test_render_full_size_gpu.py _check_compositing)


@pytest.fixture(autouse=True)
def _free():
    torch.cuda.empty_cache()
    yield
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------------
# set-up
# ------------------------------------------------------------------------------------------------------------------------
class Scene:
    """A pretrained scene's networks (state dicts and packed blobs), options and N_RAYS rays: N_RAYS / POSES random
    pixels of each of POSES poses."""

    def __init__(self, scene, perturb=True):
        from nerf_pytorch_b200 import ops

        self.name = scene
        _, self.nf, ndc, near, far, self.white, noise, (H, W, focal) = PRETRAINED_SCENES[scene]
        self.noise = noise if perturb else 0.0
        self.perturb = perturb
        self.nc, self.n = 64, N_RAYS
        self.ns = self.nc + self.nf
        self.arch = pretrained_arch(scene)
        self.sds = load_weights(f"{scene}_lowres")
        self.blobs = [ops.pack_weights(self.arch, ops.flatten_state_dict(self.arch, sd, "cuda")) for sd in self.sds]
        self.opts = ops.make_opts(self.nc, self.nf, perturb, False, self.white, self.noise)
        g = torch.Generator().manual_seed(17)
        rows = []
        for pose in pretrained_poses(scene, POSES):
            pix = torch.randperm(H * W, generator=g)[:N_RAYS // POSES]
            rows.append(ops.gen_rays(pose, H, W, focal, pix.cuda(), "cuda", ndc=ndc, near=near, far=far))
        self.rays = torch.cat(rows).contiguous()
        self.target = torch.rand(self.n, 3, generator=g).cuda()
        self.rnd = {}
        if perturb:
            rnd = dict(t_rand=torch.rand(self.n, self.nc, generator=g),
                       noise_c=torch.randn(self.n, self.nc, generator=g), u=torch.rand(self.n, self.nf, generator=g),
                       noise_f=torch.randn(self.n, self.ns, generator=g))
            self.rnd = {k: v.cuda() for k, v in rnd.items()}
        self.ops = ops

    def forward(self, impl, training):
        """render_fwd: (out_c, out_f, workspace bytes, layout)."""
        out_c, out_f, ws = self.ops.render_fwd(self.arch, self.arch, self.opts, *self.blobs, self.rays, self.rnd,
                                               training=training, impl=impl)
        return out_c, out_f, ws, self.ops.render_workspace_layout(self.arch, self.arch, self.opts, self.n, training)

    def section(self, ws, lay, name, count):
        return ws[lay[name]: lay[name] + 4 * count].view(torch.float32)

    def passes(self, ws, lay):
        """Per network (coarse, fine): z [n][S], raw [n][S][4], stash (training workspaces) or None, noise or None."""
        n, out = self.n, []
        for tag, S, stash_from, stash_to in (("coarse", self.nc, "stash_coarse", "stash_fine"),
                                             ("fine", self.ns, "stash_fine", "gstash")):
            z = self.section(ws, lay, f"z_{tag}", n * S).view(n, S)
            raw = self.section(ws, lay, f"raw_{tag}", n * S * 4).view(n, S, 4)
            stash = ws[lay[stash_from]:lay[stash_to]].view(torch.float32) if stash_to in lay else None
            out.append((z, raw, stash, self.rnd.get(f"noise_{tag[0]}")))
        return out


def _to_4_8(d_raw):
    """The power of two that puts max |d_raw| in [4, 8)."""
    return 2.0 ** (3 - math.frexp(d_raw.abs().max().item())[1])


def _block_groups(arch):
    """tc_blocks split into the heads, layers_dir.0 and the trunk, each reported on its own."""
    groups = {"fc_rgb": [], "fc_alpha": [], "layers_dir.0": [], "trunk and fc_feat": []}
    for b in tc_blocks(arch):
        key = b[1].rsplit(".", 1)[0]
        groups[key if key in groups else "trunk and fc_feat"].append(b)
    return groups


# ------------------------------------------------------------------------------------------------------------------------
# 4. compositing
# ------------------------------------------------------------------------------------------------------------------------
def _check_compositing(sc, out, weights, raw, z, noise, ctx):
    """rgb, acc, depth (and weights) at COMP_TOL of their scale against composite64 of our raw and z; disp NaN exactly
    where acc is 0 and elsewhere within test_render_full_size_gpu.py's derived bar."""
    S = z.shape[1]
    rgb, disp, acc, w, depth = (t.detach() for t in composite64(raw, z, sc.rays[:, 3:6], sc.noise, sc.white, noise))
    worst = 0.0
    for name, a, b in (("rgb", out[:, :3], rgb), ("acc", out[:, 4], acc), ("depth", out[:, 5], depth),
                       ("weights", weights, w)):
        if a is None:
            continue
        e = (a.double() - b).abs().max().item() / b.abs().max().item()
        worst = max(worst, e)
        assert e <= COMP_TOL, ctx + (name, e)
    report("compositing outputs", ctx, worst)
    d32 = out[:, 3].double()
    empty = out[:, 4] == 0
    assert torch.equal(torch.isnan(d32), empty), ctx + ("disp NaN where acc > 0 or finite where acc == 0",)
    ok = ~empty
    r64 = depth[ok] / acc[ok]
    span = (z[ok, -1] - z[ok, 0]).double()
    bar = d32[ok] * disp[ok] * (COMP_TOL * r64 + DISP_K * S * 2.0 ** -24 * span / acc[ok])
    e = (d32[ok] - disp[ok]).abs()
    report("disp / its bar", ctx, (e / bar).max().item())
    assert (e <= bar).all(), ctx + ("disp", (e / bar).max().item())


# ------------------------------------------------------------------------------------------------------------------------
# 1, 2, 4. the training step
# ------------------------------------------------------------------------------------------------------------------------
def _check_net(sc, impl, which, ws, lay, z, raw, stash, noise, g_pair, ctx):
    """One network's backward (render_bwd parts=1 fine, 2 coarse) against fp64, its stash (impl 1) and its range."""
    parts = 2 if which == 0 else 1
    arch, sd = sc.arch, sc.sds[which]
    S = z.shape[1]
    P = sc.n * S
    family = "wgmma" if impl == 1 else "fp32"
    lay_s = StashLayout(arch)

    def run(gs):
        flats = [torch.zeros(arch.flat_param_count(), device="cuda") for _ in range(2)]
        sc.ops.render_bwd(arch, arch, sc.opts, *sc.blobs, sc.rays, sc.rnd, *gs, ws, *flats, impl=impl, parts=parts)
        return flats[which], sc.section(ws, lay, "d_raw", P * 4).view(sc.n, S, 4).clone()

    _, d_raw = run(g_pair)
    want = composite_grad64(raw, z, sc.rays[:, 3:6], g_pair[which], sc.noise, sc.white, noise)
    e = (d_raw.double() - want).abs().max().item() / want.abs().max().item()
    report("d_raw", ctx, e)
    assert e <= COMP_GRAD_TOL, ctx + ("d_raw", e)

    stash_err = [0.0] * len(lay_s.layers)
    ties = [0]

    def visit(p0, p1, rays_c, z_c, acts):
        if impl == 1:  # the tiles as the backward reads them, before any ReLU decision is adopted
            for li, (_, n, cum) in enumerate(lay_s.layers):
                a = read_layer(stash, P, cum, n, family, (p0, p1))
                stash_err[li] = max(stash_err[li], (a - acts[li]).abs().max().item())
        ties[0] += relu_ties(arch, stash, P, acts, family, STASH_TOL if impl == 1 else FP32_TIE_TOL, ctx + (p0,),
                             adopt=True, rows=(p0, p1))

    ref = oracle_tiles(arch, sd, sc.rays, z, d_raw, visit=visit)
    report("relu ties", ctx, ties[0])

    # 2. range: every stashed layer (and so every split operand) inside the split's range, margin reported per layer
    for li, (lname, _, _) in enumerate(lay_s.layers):
        report(f"max |{lname}| / 1.05e6", ctx, ref.act_max[li] / SPLIT_MAX)
        assert ref.act_max[li] < SPLIT_MAX, ctx + (f"{lname} reaches {ref.act_max[li]:.4g}, past the fp16 x 2 split's "
                                                   f"range {SPLIT_MAX:.4g}: its stash tile cannot hold it",)
        if impl == 1:
            rel = stash_err[li] / ref.act_max[li]
            report(f"stash {lname}", ctx, rel)
            assert rel <= STASH_TOL, ctx + ("stash", lname, rel)

    # 3. the training forward's raw, per column
    tol = TC_FWD_TOL if impl == 1 else SIMT_FWD_TOL
    col = ((raw.reshape(-1, 4).double() - ref.raw).abs() / ref.raw.abs().amax(0)).amax(0)
    report("raw per column", ctx, col.max().item())
    assert (col <= tol).all(), ctx + ("raw", col.tolist())

    # 1. parameter gradients per block, the heads and layers_dir.0 on their own, at the loss's scale and scaled
    assert blob_range_factor(ref.grads) == 1.0, ctx
    split = ref.split if impl == 1 else None
    flat, _ = run(g_pair)
    floors = _floors(arch, P, split)
    for group, blocks in _block_groups(arch).items():
        check_blocks(arch, flat, ref.grads, blocks, BLOCK_TOL, ctx + ("loss scale", group), f"blocks {group}", floors)
    c = _to_4_8(d_raw)
    c *= blob_range_factor({k: v * c for k, v in ref.grads.items()})
    flat, _ = run(tuple(None if g is None else g * c for g in g_pair))
    floors = _floors(arch, P, {k: v * c for k, v in split.items()} if split else None)
    for group, blocks in _block_groups(arch).items():
        check_blocks(arch, flat, {k: v * c for k, v in ref.grads.items()}, blocks, BLOCK_TOL,
                     ctx + ("max |d_raw| in [4, 8)", group), f"blocks {group}", floors)


@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("scene", SCENES)
def test_training_step_matches_fp64(scene, impl):
    sc = Scene(scene)
    ctx = (scene, f"impl {impl}")
    out_c, out_f, ws, lay = sc.forward(impl, training=True)
    passes = sc.passes(ws, lay)
    if impl == 1:  # the inference forward computes the same bits
        inf_c, inf_f, ws_i, lay_i = sc.forward(impl, training=False)
        for (z, raw, _, _), (z_i, raw_i, _, _) in zip(passes, sc.passes(ws_i, lay_i)):
            assert bits_equal(z, z_i) and bits_equal(raw, raw_i), ctx + ("training=False",)
        assert bits_equal(inf_c, out_c) and bits_equal(inf_f, out_f), ctx + ("training=False",)
        del ws_i
    w_c = sc.section(ws, lay, "weights_coarse", sc.n * sc.nc).view(sc.n, sc.nc)
    for tag, out, (z, raw, _, noise), w in (("coarse", out_c, passes[0], w_c), ("fine", out_f, passes[1], None)):
        _check_compositing(sc, out, w, raw, z, noise, ctx + (tag, "compositing"))

    oc, of = out_c.detach().clone().requires_grad_(True), out_f.detach().clone().requires_grad_(True)
    loss = torch.nn.functional.mse_loss(oc[:, :3], sc.target) + torch.nn.functional.mse_loss(of[:, :3], sc.target)
    g_pair = tuple(g.contiguous() for g in torch.autograd.grad(loss, (oc, of)))
    # the fine network first: parts=1 leaves the coarse pass's workspace as it was
    for which, tag in ((1, "fine"), (0, "coarse")):
        z, raw, stash, noise = passes[which]
        _check_net(sc, impl, which, ws, lay, z, raw, stash, noise, g_pair, ctx + (tag,))


# ------------------------------------------------------------------------------------------------------------------------
# 3. the inference forward on every impl, at the render's points and at box points
# ------------------------------------------------------------------------------------------------------------------------
def _box_points(scene, n, seed):
    lo, hi = (torch.tensor(b) for b in PRETRAINED_BOX[scene])
    g = torch.Generator().manual_seed(seed)
    pts = lo + (hi - lo) * torch.rand(n, 3, generator=g)
    dirs = torch.nn.functional.normalize(torch.randn(n // 64, 3, generator=g), dim=-1)
    return pts.cuda(), dirs.cuda()


def _check_columns(raw, ref, tol, ctx):
    col = ((raw.reshape(-1, 4).double() - ref).abs() / ref.abs().amax(0)).amax(0)
    report("raw per column", ctx, col.max().item())
    assert (col <= tol).all(), ctx + (col.tolist(),)


@pytest.mark.parametrize("net", NETS)
@pytest.mark.parametrize("scene", SCENES)
def test_inference_forward_matches_fp64(scene, net):
    from nerf_pytorch_b200 import ops

    sc = Scene(scene, perturb=False)
    which = NETS.index(net)
    arch, sd, blob = sc.arch, sc.sds[which], sc.blobs[which]
    _, _, ws, lay = sc.forward(1, training=False)
    z, _, _, _ = sc.passes(ws, lay)[which]
    z = z.clone()
    del ws
    ref = oracle_tiles(arch, sd, sc.rays, z).raw
    pts, dirs = _box_points(scene, 1 << 16, seed=3)
    # each box point as a ray of one sample at depth 0 with its row's direction: the oracle's point o + d 0 is o
    d_pt = dirs.repeat_interleave(64, 0)
    box_rays = torch.cat([pts, d_pt, torch.zeros_like(pts[:, :2]), d_pt], 1)
    ref_box = oracle(arch, {k: v.cuda() for k, v in sd.items()}, box_rays, torch.zeros_like(pts[:, :1]))[0]
    for impl, tol in ((ops.IMPL_TC, TC_FWD_TOL), (ops.IMPL_SIMT, SIMT_FWD_TOL), (ops.IMPL_TC_FAST, FAST_TOL)):
        ctx = (scene, net, f"impl {impl}")
        _check_columns(ops.mlp_fwd(arch, blob, sc.rays, z, impl=impl), ref, tol, ctx + ("rays",))
        _check_columns(ops.mlp_fwd_pts(arch, blob, pts.view(-1, 64, 3), dirs, impl=impl), ref_box, tol,
                       ctx + ("box",))


# ------------------------------------------------------------------------------------------------------------------------
# 5. density gradient
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("net", NETS)
@pytest.mark.parametrize("scene", SCENES)
def test_density_gradient_matches_fp64(scene, net):
    from nerf_pytorch_b200 import ops

    arch = pretrained_arch(scene)
    sd = load_weights(f"{scene}_lowres")[NETS.index(net)]
    blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))
    pts, _ = _box_points(scene, 1 << 16, seed=7)
    out = ops.density_grad(arch, blob, pts)
    up = torch.tensor([0.0, 0.0, 1.0], device="cuda")
    assert bits_equal(out[:, 0].contiguous(), net_at(arch, blob, pts, up)[:, 3].contiguous()), (scene, net, "sigma")
    g64, tie = sigma_grad64(arch, sd, pts)
    scale = g64.norm(dim=-1).max().item()
    err = (out[:, 1:].double() - g64).abs().amax(-1) / scale
    worst = err[~tie].max().item()
    worst_tie = err[tie].max().item() if tie.any() else 0.0
    report("density gradient / batch scale", (scene, net), worst)
    report(f"density gradient / batch scale at the {int(tie.sum())} ReLU-tie points", (scene, net), worst_tie)
    assert torch.isfinite(out).all(), (scene, net)
    assert worst <= GRAD_TOL, (scene, net, worst)
    assert worst_tie <= TIE_GRAD_TOL, (scene, net, worst_tie)


# ------------------------------------------------------------------------------------------------------------------------
# 6. bake
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("net", NETS)
@pytest.mark.parametrize("scene", SCENES)
def test_bake_matches_the_network(scene, net):
    """ops.bake over every brick of the scene's box at 128^3: sigma and the 64 direction logits are the wgmma forward's
    bits, the SH coefficients within COEF_REL of the fp64 projection of those logits; the fp16 bake is the fp32 bake
    under the conversion rule, bit for bit."""
    from nerf_pytorch_b200 import ops
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    arch = pretrained_arch(scene)
    sd = load_weights(f"{scene}_lowres")[NETS.index(net)]
    blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))
    box = PRETRAINED_BOX[scene]
    g = ops.grid_struct(box, (128,) * 3)
    _, bricks, n = ops.mesh_sparse_bricks(g, OccupancyGrid.full(box, 8))
    n = int(n.item())
    P = n * 729
    values = torch.empty(n, 729, 32, device="cuda")
    logits = torch.empty(P, 64, 3, device="cuda")
    ops.bake(arch, blob, g, bricks, 0, n, values, logits)
    half = ops.bake(arch, blob, g, bricks, 0, n, torch.empty(n, 729, 32, dtype=torch.float16, device="cuda"))
    v = values.view(P, 32)
    assert bits_equal(half.view(torch.int16), torch.where(values.isfinite(), values.clamp(-65504, 65504),
                                                          values).half().view(torch.int16)), (scene, net, "fp16")
    pts = ops.mesh_sparse_points(g, bricks, 0, n, False, torch.empty(P, 3, device="cuda"))
    dirs, proj = ops.bake_basis()
    assert bits_equal(v[:, 0].contiguous(), net_at(arch, blob, pts, dirs[0].cuda())[:, 3].contiguous()), (scene, net)
    coef64 = torch.zeros(P, 3, 9, dtype=torch.float64, device="cuda")
    proj = proj.double().cuda()
    for d in range(64):
        raw = net_at(arch, blob, pts, dirs[d].cuda())[:, :3]
        assert bits_equal(logits[:, d].contiguous(), raw.contiguous()), (scene, net, d)
        coef64 += proj[:, d][None, None, :] * raw.double()[:, :, None]
    scale = logits.abs().amax(dim=(1, 2)).double()[:, None]
    err = ((v[:, 1:28].double().view(P, 3, 9) - coef64).abs().view(P, 27) / scale.clamp_min(1e-30)).max().item()
    report("bake coefficient error / max |logit|", (scene, net), err)
    assert err <= COEF_REL, (scene, net, err)
    assert (v[:, 28:] == 0).all()
