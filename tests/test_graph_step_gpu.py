"""GPU: CapturedTrainStep, a whole training step as one CUDA graph (pixel draw, rays, render, loss, backward, Adam with
the step count on the device), against the existing eager path and against itself replayed."""
import copy
import math

import numpy as np
import pytest
import torch

from helpers import bits_equal
from oracle import nerf_oracle as O

pytestmark = pytest.mark.gpu

SEED = 1234
ARCHS = {"A0": dict(num_layers=4, hidden_size=128, skip_connect_every=4),
         "A1": dict(num_layers=8, hidden_size=128, skip_connect_every=3)}


def _pose(theta, phi, r=4.0):
    th, ph = math.radians(theta), math.radians(phi)
    t = torch.tensor([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, r], [0, 0, 0, 1.0]])
    rp = torch.tensor([[1, 0, 0, 0], [0, math.cos(ph), -math.sin(ph), 0], [0, math.sin(ph), math.cos(ph), 0], [0, 0, 0, 1.0]])
    rt = torch.tensor([[math.cos(th), 0, -math.sin(th), 0], [0, 1, 0, 0], [math.sin(th), 0, math.cos(th), 0], [0, 0, 0, 1.0]])
    swap = torch.tensor([[-1, 0, 0, 0], [0, 0, 1, 0], [0, 1, 0, 0], [0, 0, 0, 1.0]])
    return swap @ rt @ rp @ t


class Scene:
    """Four posed images of H x W, a model pair (or a coarse model alone) with its FusedAdam, and the options."""

    def __init__(self, arch="A0", fine=True, ndc=False, n=256, H=24, W=32, init_seed=0):
        import nerf_pytorch_b200 as nb
        from nerf_pytorch_b200 import parallel, train_utils

        self.H, self.W, self.focal, self.n = H, W, 30.0, n
        lxyz = 6 if ndc else 10
        g = torch.Generator().manual_seed(7)
        self.images = torch.rand(4, H, W, 3, generator=g).cuda()
        if ndc:
            poses = [torch.eye(4) for _ in range(4)]
            for i, p in enumerate(poses):
                p[:3, 3] = torch.tensor([0.05 * i, -0.03 * i, 0.02 * i])
        else:
            poses = [_pose(30.0 + 40 * i, -30.0 + 5 * i) for i in range(4)]
        self.poses = torch.stack(poses).float().cuda()
        self.options = O.make_options(no_ndc=not ndc, near=0.0 if ndc else 2.0, far=1.0 if ndc else 6.0, num_coarse=64,
                                      num_fine=64 if fine else 0, perturb=True,
                                      radiance_field_noise_std=1.0 if ndc else 0.2, chunksize=8192)
        self.options.nerf.train.num_random_rays = n
        torch.manual_seed(init_seed)
        mk = lambda: nb.FlexibleNeRFModel(num_encoding_fn_xyz=lxyz, num_encoding_fn_dir=4, **ARCHS[arch]).cuda()
        self.mc = mk()
        self.mf = mk() if fine else None
        self.epf, self.edf = nb.get_embedding_function(lxyz), nb.get_embedding_function(4)
        a = train_utils._arch_of(self.mc, (lxyz, True, True), (4, True, True))
        self.opt = parallel.FusedAdam([(m, a) for m in (self.mc, self.mf) if m is not None], lr=5e-3, lr_decay=250,
                                      lr_decay_factor=0.1)

    def clone(self):
        """The same scene with its own copy of the models and a fresh optimizer in the same state."""
        from nerf_pytorch_b200 import parallel

        c = copy.copy(self)
        c.mc = copy.deepcopy(self.mc)
        c.mf = copy.deepcopy(self.mf) if self.mf is not None else None
        c.opt = parallel.FusedAdam([(m, it["arch"]) for m, it in zip((c.mc, c.mf), self.opt.items)],
                                   lr=5e-3, lr_decay=250, lr_decay_factor=0.1)
        for mine, theirs in zip(c.opt.items, self.opt.items):
            mine["flat"].copy_(theirs["flat"]); mine["m"].copy_(theirs["m"]); mine["v"].copy_(theirs["v"])
        c.opt.step_count = self.opt.step_count
        return c

    def captured(self, source=None, **kw):
        import nerf_pytorch_b200 as nb

        src = source if source is not None else (self.images, self.poses, self.focal)
        return nb.CapturedTrainStep(self.mc, self.mf, self.epf, self.edf, self.options, self.opt, SEED, src, **kw)

    def state(self):
        return [(it["flat"].clone(), it["m"].clone(), it["v"].clone()) for it in self.opt.items]


def _eager_step(sc, k, image, pix, impl, pool=None):
    """The existing path: run_one_iter_of_nerf[_from_pose] with SeededRandoms(SEED, k), torch mse_loss, backward,
    FusedAdam.step.  Returns (loss, target, flat gradient)."""
    import nerf_pytorch_b200 as nb

    F = torch.nn.functional
    if pool is None:
        out = nb.run_one_iter_of_nerf_from_pose(sc.H, sc.W, sc.focal, sc.mc, sc.mf, sc.poses[image], pix, sc.options,
                                                encode_position_fn=sc.epf, encode_direction_fn=sc.edf,
                                                randoms=nb.SeededRandoms(SEED, k), impl=impl)
        tgt = sc.images[image].reshape(-1, 3)[pix]
    else:
        sel = pool.offsets[image] + pix
        out = nb.run_one_iter_of_nerf(sc.H, sc.W, sc.focal, sc.mc, sc.mf, pool.ray_origins[sel],
                                      pool.ray_directions[sel], sc.options, encode_position_fn=sc.epf,
                                      encode_direction_fn=sc.edf, randoms=nb.SeededRandoms(SEED, k), impl=impl)
        tgt = pool.targets[sel]
    loss = F.mse_loss(out[0], tgt)
    if sc.mf is not None:
        loss = loss + F.mse_loss(out[3], tgt)
    sc.opt.zero_grad()
    loss.backward()
    grad = torch.cat([p.grad.reshape(-1) for it in sc.opt.items for p in it["params"]])
    sc.opt.step()
    return loss.detach(), tgt, grad


def _make_pool(sc, tmp_path):
    from nerf_pytorch_b200 import CachedRayPool, ops

    paths = []
    for i in range(sc.poses.shape[0]):
        r = ops.gen_rays(sc.poses[i], sc.H, sc.W, sc.focal, None, "cuda", use_viewdirs=False, stride=6).cpu()
        d = {"height": sc.H, "width": sc.W, "focal_length": sc.focal,
             "ray_bundle": torch.stack([r[:, :3], r[:, 3:]]).reshape(2, sc.H, sc.W, 3),
             "target": sc.images[i].cpu()}
        p = tmp_path / f"{i:03d}.data"
        torch.save(d, p)
        paths.append(str(p))
    return CachedRayPool(paths, device="cuda")


CASES = {  # name: (arch, impl, fine, ndc, source)
    "A0-impl1": ("A0", 1, True, False, "images"),
    "A1-impl1": ("A1", 1, True, False, "images"),
    "A0-impl0": ("A0", 0, True, False, "images"),
    "A1-impl0": ("A1", 0, True, False, "images"),
    "fern-ndc-noise1": ("A0", 1, True, True, "images"),
    "coarse-only": ("A0", 1, False, False, "images"),
    "pool": ("A0", 1, True, False, "pool"),
}


@pytest.mark.parametrize("case", list(CASES))
def test_eager_step_equals_existing_path(case, tmp_path):
    arch, impl, fine, ndc, source = CASES[case]
    a = Scene(arch, fine=fine, ndc=ndc)
    b = a.clone()
    pool = _make_pool(a, tmp_path) if source == "pool" else None
    step = a.captured(pool, impl=impl, capture=False)
    worst = 0.0
    for k in range(5):
        if impl == 0:
            # impl 0 sums its weight gradients with float atomics, equal only up to their order of addition, and the
            # trajectories drift apart: each step is compared from the same starting state
            for mine, theirs in zip(b.opt.items, a.opt.items):
                for key in ("flat", "m", "v"):
                    mine[key].copy_(theirs[key])
        loss = step.step()
        image, pix = int(step.image.item()), step.pixel_ids.clone()
        ref_loss, ref_tgt, ref_grad = _eager_step(b, k, image, pix, impl, pool)
        assert a.opt.step_count == b.opt.step_count == k + 1
        assert bits_equal(step.target, ref_tgt)
        worst = max(worst, abs(loss.item() - ref_loss.item()) / ref_loss.item())
        if impl == 1:
            assert bits_equal(step.flat_grad, ref_grad), (case, k)
            for (p, m, v), (rp, rm, rv) in zip(a.state(), b.state()):
                assert bits_equal(p, rp) and bits_equal(m, rm) and bits_equal(v, rv), (case, k)
        else:
            # Adam turns an order-of-addition difference into up to 2 lr on a gradient near zero whose sign it flips
            assert (step.flat_grad - ref_grad).norm() <= 1e-5 * ref_grad.norm(), (case, k)
            for (p, _, _), (rp, _, _) in zip(a.state(), b.state()):
                assert (p - rp).norm() <= 1e-3 * rp.norm(), (case, k)
    # the loss: an fp64 sum rounded once against torch's fp32 tree sum
    assert worst < (2e-6 if impl == 1 else 1e-4), worst
    print(f"{case}: largest relative loss difference to torch's mse_loss {worst:.2e}")


def test_graph_replays_equal_eager_steps():
    a = Scene("A1")
    b = a.clone()
    graph, eager = a.captured(impl=1), b.captured(impl=1, capture=False)
    assert a.opt.step_count == 0 and bits_equal(a.state()[0][0], b.state()[0][0])  # capture left the state as it was
    la = [graph.step() for _ in range(20)]
    lb = [eager.step() for _ in range(20)]
    for x, y in zip(la, lb):
        assert bits_equal(x, y)
    for (p, m, v), (rp, rm, rv) in zip(a.state(), b.state()):
        assert bits_equal(p, rp) and bits_equal(m, rm) and bits_equal(v, rv)
    assert a.opt.step_count == b.opt.step_count == 20
    assert int(graph.step_dev.item()) == 20


def test_replays_do_no_host_work():
    from nerf_pytorch_b200 import ops

    sc = Scene("A0")
    step = sc.captured(impl=1)
    step.step()
    torch.cuda.synchronize()
    before = ops.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        losses = [step.step() for _ in range(10)]
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert ops.launch_count() == before
    assert all(math.isfinite(x.item()) for x in losses)


def test_resume_continues_the_run():
    a = Scene("A0")
    b = a.clone()
    straight = a.captured(impl=1)
    for _ in range(5):
        straight.step()
    first = b.captured(impl=1, capture=False)
    for _ in range(3):
        first.step()
    second = b.captured(impl=1)  # built on the optimizer at step 3
    for _ in range(2):
        second.step()
    for (p, m, v), (rp, rm, rv) in zip(a.state(), b.state()):
        assert bits_equal(p, rp) and bits_equal(m, rm) and bits_equal(v, rv)


# ------------------------------------------------------------------------------------------------
# the kernels on their own
# ------------------------------------------------------------------------------------------------
_MASK = (1 << 32) - 1


def _philox(c, k0, k1):
    c = list(c)
    for i in range(10):
        if i:
            k0, k1 = (k0 + 0x9E3779B9) & _MASK, (k1 + 0xBB67AE85) & _MASK
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k0, p1 & _MASK, (p0 >> 32) ^ c[3] ^ k1, p0 & _MASK]
    return c


def _draw_reference(seed, step, n_images, n_pixels, n):
    """The draw restated in Python integers (csrc/common.cuh, step.cu)."""
    k0, k1 = seed & _MASK, seed >> 32
    keys = []
    for q in range((n_pixels + 1) // 2):
        w = _philox((q, step & _MASK, 0, 0x80000000), k0, k1)
        keys += [(w[0] << 32 | w[1], 2 * q), (w[2] << 32 | w[3], 2 * q + 1)]
    ids = [p for _, p in sorted(keys[:n_pixels])[:n]]
    w = _philox((0, step & _MASK, 1, 0x80000000), k0, k1)
    return ((w[0] << 32 | w[1]) * n_images) >> 64, ids


def _draw(seed, step, n_images, n_pixels, n):
    from nerf_pytorch_b200 import ops

    s = torch.tensor([step], dtype=torch.int64, device="cuda")
    image, ids = ops.draw_pixels(seed, s, n_images, n_pixels, n)
    return int(image.item()), ids.cpu()


@pytest.mark.parametrize("n_pixels,n", [(5003, 300), (1073, 1073), (20000, 20000), (160000, 4096)])
def test_draw_is_exact_distinct_and_deterministic(n_pixels, n):
    image, ids = _draw(SEED, 17, 7, n_pixels, n)
    assert ids.unique().numel() == n and int(ids.min()) >= 0 and int(ids.max()) < n_pixels
    if n == n_pixels:
        assert torch.equal(ids.sort().values, torch.arange(n_pixels))
    again = _draw(SEED, 17, 7, n_pixels, n)
    assert image == again[0] and torch.equal(ids, again[1])
    if n_pixels <= 20000:
        ref_image, ref_ids = _draw_reference(SEED, 17, 7, n_pixels, n)
        assert image == ref_image and ids.tolist() == ref_ids
    assert not torch.equal(ids, _draw(SEED, 18, 7, n_pixels, n)[1])
    assert not torch.equal(ids, _draw(SEED + 1, 17, 7, n_pixels, n)[1])


def test_draw_frequencies_pass_chi_square():
    from scipy.stats import chisquare

    from nerf_pytorch_b200 import ops

    n_images, n_pixels, n, steps = 5, 64, 8, 4000
    s = torch.zeros(1, dtype=torch.int64, device="cuda")
    ws = torch.empty(ops.draw_workspace_bytes(n_pixels), dtype=torch.uint8, device="cuda")
    images, ids = [], []
    for k in range(steps):
        s.fill_(k)
        im, px = ops.draw_pixels(SEED, s, n_images, n_pixels, n, workspace=ws)
        images.append(im)
        ids.append(px)
    images, ids = torch.cat(images).cpu(), torch.cat(ids).cpu()
    assert chisquare(torch.bincount(images, minlength=n_images).numpy()).pvalue > 1e-4
    assert chisquare(torch.bincount(ids, minlength=n_pixels).numpy()).pvalue > 1e-4
    first = ids.view(steps, n)[:, 0]  # the order within a draw is random too
    assert chisquare(torch.bincount(first, minlength=n_pixels).numpy()).pvalue > 1e-4


@pytest.mark.parametrize("ndc", [False, True])
@pytest.mark.parametrize("rows", [3, 4])
def test_rays_from_a_device_pose_table_equal_gen_rays(ndc, rows):
    from nerf_pytorch_b200 import ops

    poses = torch.stack([_pose(20.0 * i, -30.0) for i in range(3)]).float().cuda()[:, :rows].contiguous()
    pix = torch.randperm(40 * 50, generator=torch.Generator().manual_seed(3))[:500].cuda()
    for i in range(3):
        image = torch.tensor([i], dtype=torch.int64, device="cuda")
        for vd in (False, True):
            got = ops.gen_rays_posed(poses, image, 40, 50, 41.5, pix, ndc=ndc, near=0.0, far=1.0, use_viewdirs=vd)
            ref = ops.gen_rays(poses[i], 40, 50, 41.5, pix, "cuda", ndc=ndc, near=0.0, far=1.0, use_viewdirs=vd)
            assert bits_equal(got, ref)


@pytest.mark.parametrize("fine", [True, False])
def test_loss_gradients_are_autograds_bits(fine):
    from nerf_pytorch_b200 import ops

    F = torch.nn.functional
    g = torch.Generator(device="cuda").manual_seed(5)
    n = 3000
    out_c = torch.rand(n, 8, device="cuda", generator=g).requires_grad_(True)
    out_f = torch.rand(n, 8, device="cuda", generator=g).requires_grad_(True) if fine else None
    t = torch.rand(n, 3, device="cuda", generator=g)
    loss = F.mse_loss(out_c[:, :3], t) + (F.mse_loss(out_f[:, :3], t) if fine else 0.0)
    loss.backward()
    got, g_c, g_f = ops.mse_loss(out_c.detach(), out_f.detach() if fine else None, t)
    assert bits_equal(g_c, out_c.grad)
    assert bits_equal(g_f, out_f.grad if fine else None)
    assert abs(got.item() - loss.item()) <= 2e-6 * loss.item()


def test_device_schedule_equals_fused_adam_lr():
    from nerf_pytorch_b200 import ops, parallel, train_utils
    import nerf_pytorch_b200 as nb

    m = nb.FlexibleNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4).cuda()
    opt = parallel.FusedAdam([(m, train_utils._arch_of(m, (10, True, True), (4, True, True)))], lr=5e-4,
                             lr_decay=250, lr_decay_factor=0.1)
    done = torch.arange(0, 300000, dtype=torch.int64)
    got = ops.lr_schedule(done.cuda(), opt.lr0, opt.lr_decay, opt.lr_decay_factor).cpu().numpy()
    ref = np.empty(done.numel(), dtype=np.float32)
    for d in range(done.numel()):
        opt.step_count = d
        ref[d] = opt.current_lr()
    assert np.array_equal(got.view(np.int32), ref.view(np.int32))
    const = ops.lr_schedule(done[:10].cuda(), 5e-3, None).cpu()
    assert torch.equal(const, torch.full((10,), 5e-3, dtype=torch.float32))
