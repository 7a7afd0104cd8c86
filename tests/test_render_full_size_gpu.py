"""GPU: the whole render step at training size against fp64, stage by stage, from the render workspace.

Each case runs ops.render_fwd(training=True) once on 4096 rays (or its own count) and reads the workspace's sections through
ops.render_workspace_layout.  Every stage is checked on this library's own previous stage, so that one stage's rounding
never shows as another's error:
  z_coarse     O.stratified_z in fp32 on the CPU with the same t_rand: bit for bit;
  raw          mlp_checks.oracle_tiles (fp64 on the device) at our z, per column; a failure names ray, tile and CTA;
  compositing  helpers.composite64 of our raw and z with the same noise: weights_coarse and every output of both passes;
  resampling   sample_pdf_merge on the workspace's weights_coarse gives its z_fine; its cdf against the fp64 cdf; given
               that cdf, indices and samples are O.sample_from_cdf's in fp32; z_fine is sort(cat(z_coarse, samples));
  backward     render_bwd(parts=1), then parts=2: d_raw against fp64 autograd of composite64; the parameter gradients
               against the oracle at our d_raw with its ReLU decisions adopted into the stash, per block; at the training
               loss's own scale (the fixed-point floor in the bar) and with the upstream scaled by the power of two that
               puts max |d_raw| in [4, 8), where the bars are test_tc_full_size_gpu.py's;
  whole chain  the parameter gradients against the oracle at fp64 d_raw (compositing of the oracle's raw).
The upstream gradient is the training loss, MSE of rgb_coarse and rgb_fine against seeded targets; one variant adds seeded
terms on disp and acc, which no training loss reaches.  On impl 1 the checks also tie the stages to what training runs:
parts=3 gives the bits of parts=1 then parts=2, run_one_iter_of_nerf_from_pose's autograd the same gradient bits, and
render_fwd(training=False) the same z / raw / output bits; the bench step's seeded randoms, ray indices straddling 2^32,
give the bits of the same step fed ops.random_fill's tensors.

Bars: the figures in brackets are the worst over this file's cases, measured on an H100 80GB HBM3 at a 700 W power
limit and 1980 MHz SM clock.  There the whole file runs in 20 s (4.4 s for the longest case) and holds at most 19.5 GiB
of device memory: the impl-1 bench step, whose seeded run takes a second 9.3 GiB workspace while the first is alive
(the impl-0 bench step holds 10.2 GiB).  The 8 x 128 network with 16 xyz bands, which only the fp32 kernels take, adds
3.3 s and holds 10.6 GiB.  The cases at the sample counts where the kernels change shape ("nc2" .. "nc1024") add 9.3 s
together (1.6 s for the longest, nc1023_nf1) and hold at most 4.8 GiB (nc683_nf1)."""
import math
import time

import pytest
import torch

from helpers import bits_equal, composite64, composite_grad64, load_weights
from mlp_checks import (BLOCK_TOL, COMP_GRAD_TOL, COMP_TOL, FP32_TIE_TOL, SIMT_FWD_TOL, STASH_TOL, TC_FWD_TOL,
                        as_state_dict, blob_range_factor, check_blocks, oracle_tiles, relu_ties, report, sms,
                        tc_blocks, _floors)
from oracle import nerf_oracle as O

pytestmark = pytest.mark.gpu

# The stages' own bars are those of mlp_checks (TC_FWD_TOL, SIMT_FWD_TOL, BLOCK_TOL, COMP_TOL, COMP_GRAD_TOL).  Measured:
# raw per column [2.1e-5, fern]; compositing outputs [2.8e-6, deterministic lego, fine]; disp [7.9e-3 of its bar];
# d_raw [1.5e-6; 1.0e-5 with the disp and acc terms]; parameter gradient blocks, figure / (scale + floor / bar) [5.4e-6
# at the loss's scale, fern; 3.1e-6 at max |d_raw| in [4, 8)].  At the loss's own scale the fixed-point floor is up to
# 99.98 % of a block's bar (every case's smallest block: 93 % to 99.98 %).  At the boundary sample counts: compositing
# outputs [9.5e-6, 1024 samples]; d_raw [9.1e-6, 1024 samples]; disp [1.9e-2 of its bar, 4 + 1]; raw [2.0e-6].
CDF_ULPS = 3         # in-kernel cdf against the fp64 cdf of the same weights, in units of 2^-24 [2.02]
DISP_K = 4.0         # disp's bar on rays with small acc, a derived bound (see _check_compositing)
# Parameter gradients against the oracle at fp64 d_raw (the compositing of the oracle's raw), per block, relative to its
# scale plus the floors: our d_raw carries the MLP forward's rounding through compositing, which the pretrained
# networks' sigma up to 1e4 amplifies [2.3e-2, deterministic lego, fine; A1 at init 3.8e-4].
CHAIN_TOL = 5e-2

NETS = {  # ops.ArchSpec arguments
    "A1": dict(num_layers=8, hidden=128, skip_every=3, n_freq_xyz=10, n_freq_dir=4),   # bench A1, config/lego.yml
    "A0": dict(num_layers=4, hidden=128, skip_every=4, n_freq_xyz=10, n_freq_dir=4),   # the pretrained lego network
    "A0_fern": dict(num_layers=4, hidden=128, skip_every=4, n_freq_xyz=6, n_freq_dir=4),  # config 4's network
    "A0_noview": dict(num_layers=4, hidden=128, skip_every=4, n_freq_xyz=10, n_freq_dir=4, use_viewdirs=False,
                      log_sampling_xyz=False, log_sampling_dir=False),
    # 99 xyz channels: the wgmma kernels refuse it, so it renders and trains on the fp32 kernels
    "wide_enc": dict(num_layers=8, hidden=128, skip_every=4, n_freq_xyz=16, n_freq_dir=6),
}
CONFIGS = {  # bench.py's: lego 400 x 400 and the fern-like NDC camera
    2: dict(H=400, W=400, focal=555.5555155968841, near=2.0, far=6.0, ndc=False),
    4: dict(H=378, W=504, focal=407.5658, near=0.0, far=1.0, ndc=True),
}
CASES = {
    "bench_step": dict(net="A1", weights="init", config=2, nc=64, nf=128, perturb=True, noise=0.2, variants=True),
    "lego": dict(net="A0", weights="lego", config=2, nc=64, nf=128, perturb=True, noise=0.2),
    "fern_ndc": dict(net="A0_fern", weights="fern", config=4, nc=64, nf=128, perturb=True, noise=1.0),
    "odd_counts": dict(net="A1", weights="init", config=2, nc=48, nf=80, perturb=True, noise=0.2, lindisp=True,
                       white=True),
    "deterministic": dict(net="A0", weights="lego", config=2, nc=64, nf=128, perturb=False, noise=0.0),
    # no view directions: the fused backward needs the fc_rgb / fc_alpha heads, so this network trains on impl 0
    "coarse_only": dict(net="A0_noview", weights="init", config=2, nc=64, nf=0, perturb=True, noise=0.2),
    "wide_encodings": dict(net="wide_enc", weights="init", config=2, nc=64, nf=128, perturb=True, noise=0.2),
    # The sample counts where the per-ray kernels and the wgmma tiling change shape (test_sample_counts_gpu.py lists the
    # kernels' boundaries).  Each ray count is a multiple of neither 4 (the per-ray kernels' warps per CTA) nor 10 (rays
    # per compaction group), and each pass's points end partway through a 128-point tile (no S = 1024 count can) and
    # partway through the last wave of CTAs on 132 SMs.
    "nc2": dict(net="A1", weights="init", config=2, nc=2, nf=0, perturb=True, noise=0.2, rays=4095),
    # the smallest hierarchical step: four coarse samples, two interior weights, one fine sample
    "nc4_nf1": dict(net="A1", weights="init", config=2, nc=4, nf=1, perturb=True, noise=0.2, white=True, rays=4095),
    # 14 samples: the wgmma kernels refuse it (test_wgmma_refuses_fewer_than_15_samples_before_any_launch)
    "nc14": dict(net="A1", weights="init", config=2, nc=14, nf=0, perturb=True, noise=0.2, rays=4095),
    # the smallest pass the wgmma kernels take: 10 rays per 128-point tile
    "nc15_nf1": dict(net="A1", weights="init", config=2, nc=15, nf=1, perturb=True, noise=0.2, rays=4095),
    # 31 interior weights; a fine pass of 64 samples, so the composite kernels' lanes hold two samples each
    "nc33_nf31": dict(net="A1", weights="init", config=2, nc=33, nf=31, perturb=True, noise=0.2, lindisp=True,
                      rays=4097),
    # 129 fine samples: the resampling sort pads to 256
    "nc64_nf65": dict(net="A1", weights="init", config=2, nc=64, nf=65, perturb=False, noise=0.0, white=True,
                      rays=2047),
    # resampling's shared memory passes 48 KiB and takes the opt-in
    "nc683_nf1": dict(net="A1", weights="init", config=2, nc=683, nf=1, perturb=True, noise=0.2, rays=399),
    # the largest coarse pass with a fine pass, whose 1024 samples fill every lane's 32
    "nc1023_nf1": dict(net="A0", weights="init", config=2, nc=1023, nf=1, perturb=True, noise=0.2, rays=399),
    # 1024 samples in one pass: the composite backward's shared memory is exactly 48 KiB
    "nc1024": dict(net="A0", weights="init", config=2, nc=1024, nf=0, perturb=True, noise=0.2, white=True, rays=399),
}
RUNS = [("bench_step", 1), ("bench_step", 0), ("lego", 1), ("fern_ndc", 1), ("odd_counts", 1), ("deterministic", 1),
        ("coarse_only", 0), ("wide_encodings", 0),
        ("nc2", 0), ("nc4_nf1", 0), ("nc14", 0), ("nc15_nf1", 1), ("nc15_nf1", 0), ("nc33_nf31", 1), ("nc64_nf65", 1),
        ("nc683_nf1", 1), ("nc1023_nf1", 1), ("nc1024", 1), ("nc1024", 0)]
N_RAYS = 4096  # a case's rays unless it sets "rays"


def _n_rays(cfg):
    return cfg.get("rays", N_RAYS)


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


# ------------------------------------------------------------------------------------------------------------------------
# set-up
# ------------------------------------------------------------------------------------------------------------------------
def _nets(cfg):
    """(arch, state_dict) of the coarse and the fine network (None, None without a fine pass)."""
    from nerf_pytorch_b200 import ops

    arch = ops.ArchSpec(**NETS[cfg["net"]])
    if cfg["weights"] in ("lego", "fern"):
        sd_c, sd_f = load_weights(cfg["weights"] + "_lowres")
    else:
        g = torch.Generator().manual_seed(2024)
        sd_c, sd_f = (O.init_flexible_nerf(arch.num_layers, arch.hidden, arch.skip_every, arch.n_freq_xyz,
                                           arch.n_freq_dir, include_input_xyz=arch.include_input_xyz,
                                           include_input_dir=arch.include_input_dir, use_viewdirs=arch.use_viewdirs,
                                           generator=g) for _ in range(2))
    if cfg["nf"] == 0:
        return (arch, sd_c), (None, None)
    return (arch, sd_c), (arch, sd_f)


def _camera(cfg):
    """Pose, pixel ids (a randperm pick, as bench.py) and the seeded targets of the batch."""
    cam = CONFIGS[cfg["config"]]
    g = torch.Generator().manual_seed(17)
    n = _n_rays(cfg)
    pix = torch.randperm(cam["H"] * cam["W"], generator=g)[:n].contiguous()
    target = torch.rand(n, 3, generator=g)
    pose = torch.eye(4) if cam["ndc"] else O.pose_spherical(30.0, -30.0, 4.0)
    return cam, pose, pix, target


def _randoms(cfg, seed):
    """The random tensors the options use, torch-drawn (CPU generator) and moved to the device."""
    n, nc, nf = _n_rays(cfg), cfg["nc"], cfg["nf"]
    g = torch.Generator().manual_seed(seed)
    rnd = {}
    if cfg["perturb"]:
        rnd["t_rand"] = torch.rand(n, nc, generator=g)
    if cfg["noise"] > 0:
        rnd["noise_c"] = torch.randn(n, nc, generator=g)
    if nf and cfg["perturb"]:
        rnd["u"] = torch.rand(n, nf, generator=g)
    if nf and cfg["noise"] > 0:
        rnd["noise_f"] = torch.randn(n, nc + nf, generator=g)
    return {k: v.cuda() for k, v in rnd.items()}


def _seeded_tensors(cfg, rng):
    """ops.random_fill's tensors of `rng` for the streams the options use."""
    from nerf_pytorch_b200 import ops

    nc, nf = cfg["nc"], cfg["nf"]
    per_ray = {"t_rand": nc, "noise_c": nc, "u": nf, "noise_f": nc + nf}
    used = {"t_rand": cfg["perturb"], "noise_c": cfg["noise"] > 0, "u": nf and cfg["perturb"],
            "noise_f": nf and cfg["noise"] > 0}
    return {k: ops.random_fill(rng, k, _n_rays(cfg), per_ray[k]) for k in per_ray if used[k]}


class Workspace:
    """Views of a render workspace's sections (byte offsets of ops.render_workspace_layout; fp32 but the stashes)."""

    def __init__(self, ws, lay, n, nc, ns):
        def f32(name, count):
            return ws[lay[name]: lay[name] + 4 * count].view(torch.float32)

        self.ws = ws
        self.z_c, self.raw_c, self.w_c = f32("z_coarse", n * nc).view(n, nc), \
            f32("raw_coarse", n * nc * 4).view(n, nc, 4), f32("weights_coarse", n * nc).view(n, nc)
        self.z_f = f32("z_fine", n * ns).view(n, ns) if ns else None
        self.raw_f = f32("raw_fine", n * ns * 4).view(n, ns, 4) if ns else None
        if "stash_coarse" in lay and lay["gstash"] > lay["stash_coarse"]:
            self.stash_c = ws[lay["stash_coarse"]:lay["stash_fine"]].view(torch.float32)
            self.stash_f = ws[lay["stash_fine"]:lay["gstash"]].view(torch.float32) if ns else None

        self.d_raw = lambda S: f32("d_raw", n * S * 4).view(n, S, 4)


def _where(p, S, n_tiles, impl):
    """Ray and sample of point p; on the wgmma kernels its 128-point tile and the persistent CTA that ran it."""
    at = f"ray {p // S} sample {p % S}"
    if impl != 1:
        return at
    t = p // 128
    grid = min(n_tiles, sms())
    return f"{at}: tile {t} of {n_tiles}, CTA {t % grid}'s tile {t // grid}"


def _to_4_8(d_raw):
    """The power of two that puts max |d_raw| in [4, 8)."""
    return 2.0 ** (3 - math.frexp(d_raw.abs().max().item())[1])


def _state_dict_of(flat, arch):
    return {k: v.double().cpu() for k, v in as_state_dict(arch, flat).items()}


# ------------------------------------------------------------------------------------------------------------------------
# stage checks
# ------------------------------------------------------------------------------------------------------------------------
def _check_raw(raw, ref_raw, S, impl, ctx):
    """Our raw [n][S][4] against the oracle's per column, relative to the column's scale."""
    P = ref_raw.shape[0]
    tol = TC_FWD_TOL if impl == 1 else SIMT_FWD_TOL
    e = (raw.reshape(-1, 4).double() - ref_raw).abs() / ref_raw.abs().amax(0)
    worst = e.amax(1)
    p = int(worst.argmax())
    report("raw per column", ctx, worst[p].item())
    assert worst[p] <= tol, ctx + (_where(p, S, -(-P // 128), impl), "column", int(e[p].argmax()), worst[p].item())


def _check_compositing(out, weights, raw, z, rays, noise, cfg, ctx):
    """out [n][8] = [rgb disp acc depth ..] (and weights [n][S]) against composite64 of our raw and z.  rgb, acc, depth,
    weights at COMP_TOL of their scale.  disp is NaN exactly where our acc is 0; there every fp32 alpha is 0, so each
    fp64 alpha is below ~2^-24 and the fp64 acc below S 2^-24.  Elsewhere disp = 1 / r with r = depth / acc, so
    |disp - disp64| = |r - r64| disp disp64, and
        |r - r64| <= COMP_TOL r64 + DISP_K S 2^-24 (z_last - z_first) / acc64:
    every fp32 alpha is off by up to 2^-24 absolutely (1 - exp(-x) rounds at 1), which moves the weighted mean of z by
    at most that sum times the ray's depth span, over acc."""
    S = z.shape[1]
    rgb, disp, acc, w, depth = (t.detach() for t in composite64(raw, z, rays[:, 3:6], cfg["noise"], cfg.get("white",
                                                                False), noise))
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
    if empty.any():
        assert acc[empty].max().item() <= S * 2.0 ** -24, ctx + ("fp64 acc of an empty ray", acc[empty].max().item())
    ok = ~empty
    r64 = depth[ok] / acc[ok]
    span = (z[ok, -1] - z[ok, 0]).double()
    bar = d32[ok] * disp[ok] * (COMP_TOL * r64 + DISP_K * S * 2.0 ** -24 * span / acc[ok])
    e = (d32[ok] - disp[ok]).abs()
    report("disp / its bar", ctx + (int(empty.sum()), "empty rays"), (e / bar).max().item())
    assert (e <= bar).all(), ctx + ("disp", (e / bar).max().item())


def _check_resampling(ws, rnd, cfg, ctx):
    """(a) sample_pdf_merge on the workspace's weights_coarse gives its z_fine; (b) its cdf against the fp64 cdf of
    those weights; (c) given that cdf, indices and samples are O.sample_from_cdf's in fp32 on the CPU; (d) z_fine is
    sort(cat(z_coarse, samples))."""
    from nerf_pytorch_b200 import ops

    nc, nf = cfg["nc"], cfg["nf"]
    u = rnd.get("u")
    z_fine, zs, inds, cdf = ops.sample_pdf_merge(ws.z_c, ws.w_c, u, nf, want_aux=True)
    assert bits_equal(z_fine, ws.z_f), ctx + ("z_fine",)
    w = ws.w_c[:, 1:-1].double() + 1e-5
    cdf64 = torch.nn.functional.pad(torch.cumsum(w / w.sum(-1, keepdim=True), -1), (1, 0))
    ulps = (cdf.double() - cdf64).abs().max().item() / 2.0 ** -24
    report("cdf against fp64 (2^-24 units)", ctx, ulps)
    assert ulps <= CDF_ULPS, ctx + ("cdf", ulps)
    _, zs_in, inds_in, _ = ops.sample_pdf_merge(ws.z_c, ws.w_c, u, nf, cdf_in=cdf, want_aux=True)
    z_c = ws.z_c.cpu()
    bins = 0.5 * (z_c[:, 1:] + z_c[:, :-1])
    u_cpu = u.cpu() if u is not None else torch.linspace(0.0, 1.0, nf).expand(_n_rays(cfg), nf).contiguous()
    want_zs, want_inds = O.sample_from_cdf(bins, cdf.cpu(), u_cpu)
    assert torch.equal(inds_in.cpu().long(), want_inds), ctx + ("indices given the cdf",)
    assert bits_equal(zs_in.cpu(), want_zs) and bits_equal(zs_in, zs), ctx + ("samples given the cdf",)
    assert bits_equal(torch.sort(torch.cat((ws.z_c, zs), -1), -1).values, ws.z_f), ctx + ("merge",)


def _composite_grad64(raw, z, rays, noise, g, cfg):
    """helpers.composite_grad64 with the case's noise and background."""
    return composite_grad64(raw, z, rays[:, 3:6], g, cfg["noise"], cfg.get("white", False), noise)


def _floor_share(arch, want, floors, tol):
    """The largest share of a block's bar (tol x scale + floor) that its absolute floor accounts for, and its block."""
    share, where = 0.0, None
    for label, key, rows, cols, _ in tc_blocks(arch):
        b = want[key].double().cpu()
        b = b[rows] if cols is None else b[rows, cols]
        s = floors[label] / (tol * b.abs().max().item() + floors[label])
        if s > share:
            share, where = s, label
    return share, where


# ------------------------------------------------------------------------------------------------------------------------
# the test
# ------------------------------------------------------------------------------------------------------------------------
class Step:
    """One case's networks, rays, randoms, forward and upstream gradient."""

    def __init__(self, name, impl):
        import nerf_pytorch_b200 as nb
        from nerf_pytorch_b200 import ops

        self.name, self.impl = name, impl
        self.cfg = cfg = CASES[name]
        (self.arch_c, self.sd_c), (self.arch_f, self.sd_f) = _nets(cfg)
        self.cam, self.pose, self.pix, target = _camera(cfg)
        cam = self.cam
        self.rays = ops.gen_rays(self.pose, cam["H"], cam["W"], cam["focal"], self.pix.cuda(), "cuda", ndc=cam["ndc"],
                                 near=cam["near"], far=cam["far"], use_viewdirs=self.arch_c.use_viewdirs)
        self.nc, self.nf, self.n = cfg["nc"], cfg["nf"], _n_rays(cfg)
        self.ns = self.nc + self.nf if self.nf else 0
        self.opts = ops.make_opts(self.nc, self.nf, cfg["perturb"], cfg.get("lindisp", False), cfg.get("white", False),
                                  cfg["noise"])
        self.blob_c = ops.pack_weights(self.arch_c, ops.flatten_state_dict(self.arch_c, self.sd_c, "cuda"))
        self.blob_f = (ops.pack_weights(self.arch_f, ops.flatten_state_dict(self.arch_f, self.sd_f, "cuda"))
                       if self.nf else None)
        self.target = target.cuda()
        self.nb, self.ops = nb, ops

    def forward(self, randoms, training=True, zeroed=False):
        """render_fwd; zeroed: into a zero-filled workspace, so that two of them compare byte for byte."""
        arch_f = self.arch_f if self.nf else None
        ws = None
        if zeroed:
            need = self.ops.render_workspace_bytes(self.arch_c, arch_f, self.opts, self.n, training)
            ws = torch.zeros(need, dtype=torch.uint8, device="cuda")
        out_c, out_f, ws = self.ops.render_fwd(self.arch_c, self.arch_f, self.opts, self.blob_c, self.blob_f, self.rays,
                                               randoms, training=training, impl=self.impl, workspace=ws)
        lay = self.ops.render_workspace_layout(self.arch_c, arch_f, self.opts, self.n, training)
        return out_c, out_f, Workspace(ws, lay, self.n, self.nc, self.ns)

    def backward(self, randoms, ws, g_c, g_f, parts):
        """render_bwd into zeroed flat gradients; returns (flat_c, flat_f)."""
        fc = torch.zeros(self.arch_c.flat_param_count(), device="cuda")
        ff = torch.zeros(self.arch_f.flat_param_count(), device="cuda") if self.nf else None
        self.ops.render_bwd(self.arch_c, self.arch_f, self.opts, self.blob_c, self.blob_f, self.rays, randoms, g_c, g_f,
                            ws.ws, fc, ff, impl=self.impl, parts=parts)
        return fc, ff

    def loss_upstream(self, out_c, out_f):
        """d(loss)/d(out_c), d(loss)/d(out_f) of MSE(rgb_coarse) + MSE(rgb_fine), through torch autograd as training."""
        oc = out_c.detach().clone().requires_grad_(True)
        leaves = [oc]
        loss = torch.nn.functional.mse_loss(oc[:, :3], self.target)
        if self.nf:
            of = out_f.detach().clone().requires_grad_(True)
            leaves.append(of)
            loss = loss + torch.nn.functional.mse_loss(of[:, :3], self.target)
        grads = torch.autograd.grad(loss, leaves)
        return grads[0].contiguous(), (grads[1].contiguous() if self.nf else None)


def _check_part(step, tag, arch, sd, ws, z, raw, stash, noise, out_g, rnd, ctx):
    """One network's backward (tag "fine": parts=1, "coarse": parts=2) at the training loss's scale, then scaled to
    max |d_raw| in [4, 8), then (out_g["extra"]) with seeded disp / acc terms; and the whole chain.  out_g: the
    upstream gradients {"loss": (g_c, g_f), "extra": (g_c, g_f) or None}.  Returns the training-scale flat gradient
    (ReLU decisions of our own forward) for the checks against training."""
    parts, which = (1, 1) if tag == "fine" else (2, 0)
    impl = step.impl
    S = z.shape[1]
    P = step.n * S
    ctx = ctx + (tag,)
    family = "wgmma" if impl == 1 else "fp32"

    def run(g_pair):
        flat = step.backward(rnd, ws, *g_pair, parts=parts)[which]
        return flat, ws.d_raw(S).clone()

    g_loss = out_g["loss"]
    flat_train, d_raw = run(g_loss)
    want = _composite_grad64(raw, z, step.rays, noise, g_loss[which], step.cfg)
    e = (d_raw.double() - want).abs().max().item() / want.abs().max().item()
    report("d_raw", ctx, e)
    assert e <= COMP_GRAD_TOL, ctx + ("d_raw", e)

    # the oracle at our d_raw, its ReLU decisions adopted into the stash chunk by chunk
    ties = [0]

    def visit(p0, p1, rays_c, z_c, acts):
        ties[0] += relu_ties(arch, stash, P, acts, family, STASH_TOL if impl == 1 else FP32_TIE_TOL, ctx + (p0,),
                             adopt=True, rows=(p0, p1))

    ref = oracle_tiles(arch, sd, step.rays, z, d_raw, visit=visit)
    report("relu ties", ctx, ties[0])
    _check_raw(raw, ref.raw, S, impl, ctx)
    assert blob_range_factor(ref.grads) == 1.0, ctx
    split = ref.split if impl == 1 else None
    floors = _floors(arch, P, split)
    flat, _ = run(g_loss)
    check_blocks(arch, flat, ref.grads, tc_blocks(arch), BLOCK_TOL, ctx + ("loss scale",), "parameter gradient blocks",
                 floors)
    share, label = _floor_share(arch, ref.grads, floors, BLOCK_TOL)
    report(f"floor's largest share of a block's bar at the loss scale ({label})", ctx, share)

    c = _to_4_8(d_raw)
    c *= blob_range_factor({k: v * c for k, v in ref.grads.items()})
    flat, d_scaled = run(tuple(None if g is None else g * c for g in g_loss))
    # compositing is linear in its upstream, but products that underflow fp32 (T behind the opaque samples of the
    # pretrained networks, then divided by q = 1e-10 or multiplied by the last delta, 1e10) round differently at the two
    # scales: the two agree to 2^-40 of max |d_raw|, below the 2^-38 to which the fused backward resolves G
    e = (d_scaled - d_raw * c).abs().max().item()
    assert e <= 2.0 ** -40 * d_scaled.abs().max().item(), ctx + ("compositing is linear in its upstream", e)
    check_blocks(arch, flat, {k: v * c for k, v in ref.grads.items()}, tc_blocks(arch), BLOCK_TOL,
                 ctx + ("scaled", c), "parameter gradient blocks, max |d_raw| in [4, 8)",
                 _floors(arch, P, {k: v * c for k, v in split.items()} if split else None))

    # the whole chain: compositing of the oracle's raw in fp64 -> the oracle MLP, against training's gradient
    raw_o = ref.raw.view(step.n, S, 4)
    d64 = _composite_grad64((raw_o.float(), raw_o), z, step.rays, noise, g_loss[which], step.cfg)
    chain = oracle_tiles(arch, sd, step.rays, z, d64)
    check_blocks(arch, flat_train, chain.grads, tc_blocks(arch), CHAIN_TOL, ctx + ("whole chain",),
                 "whole chain blocks", _floors(arch, P, chain.split if impl == 1 else None))
    del ref, chain, raw_o, d64

    if out_g.get("extra") is not None:
        g_x = out_g["extra"]
        _, d_x = run(g_x)
        want = _composite_grad64(raw, z, step.rays, noise, g_x[which], step.cfg)
        e = (d_x.double() - want).abs().max().item() / want.abs().max().item()
        report("d_raw with disp and acc terms", ctx, e)
        assert e <= COMP_GRAD_TOL, ctx + ("d_raw with disp and acc terms", e)
        ref = oracle_tiles(arch, sd, step.rays, z, d_x)
        c = _to_4_8(d_x)
        c *= blob_range_factor({k: v * c for k, v in ref.grads.items()})
        flat, _ = run(tuple(None if g is None else g * c for g in g_x))
        check_blocks(arch, flat, {k: v * c for k, v in ref.grads.items()}, tc_blocks(arch), BLOCK_TOL,
                     ctx + ("disp and acc terms", c), "parameter gradient blocks with disp and acc terms",
                     _floors(arch, P, {k: v * c for k, v in ref.split.items()} if impl == 1 else None))
    return flat_train


def _check_against_training(step, rnd, g_c, g_f, fc, ff, ctx):
    """parts=3 on a fresh forward gives the bits of parts=1 then parts=2 (impl 0: within BLOCK_TOL, its fp32 weight
    gradients use atomics); on impl 1, run_one_iter_of_nerf_from_pose's autograd with the same randoms and upstream
    gives the same gradient bits."""
    _, _, ws = step.forward(rnd)
    fc3, ff3 = step.backward(rnd, ws, g_c, g_f, parts=3)
    del ws
    for arch, a, b in ((step.arch_c, fc3, fc), (step.arch_f, ff3, ff)):
        if arch is None:
            continue
        if step.impl == 1:
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), ctx + ("parts=3",)
        else:
            check_blocks(arch, a, _state_dict_of(b, arch), tc_blocks(arch), BLOCK_TOL, ctx + ("parts=3",), None)
    if step.impl != 1:
        return
    nb, ops = step.nb, step.ops
    cam, arch = step.cam, step.arch_c
    models = [None, None]
    for i, sd in enumerate((step.sd_c, step.sd_f)):
        if sd is None:
            continue
        m = nb.FlexibleNeRFModel(num_layers=arch.num_layers, hidden_size=arch.hidden, skip_connect_every=arch.skip_every,
                                 num_encoding_fn_xyz=arch.n_freq_xyz, num_encoding_fn_dir=arch.n_freq_dir)
        m.load_state_dict(sd)
        models[i] = m.cuda()
    cfg = step.cfg
    options = O.make_options(no_ndc=not cam["ndc"], near=cam["near"], far=cam["far"], num_coarse=step.nc,
                             num_fine=step.nf, perturb=cfg["perturb"], lindisp=cfg.get("lindisp", False),
                             white_background=cfg.get("white", False), radiance_field_noise_std=cfg["noise"])
    out = nb.run_one_iter_of_nerf_from_pose(cam["H"], cam["W"], cam["focal"], models[0], models[1], step.pose,
                                            step.pix.cuda(), options, mode="train",
                                            encode_position_fn=nb.get_embedding_function(arch.n_freq_xyz),
                                            encode_direction_fn=nb.get_embedding_function(arch.n_freq_dir),
                                            randoms=rnd, impl=1)
    loss = torch.nn.functional.mse_loss(out[0], step.target)
    if step.nf:
        loss = loss + torch.nn.functional.mse_loss(out[3], step.target)
    loss.backward()
    for m, flat in zip(models, (fc, ff)):
        if m is None:
            continue
        got = ops.flatten_state_dict(arch, {k: p.grad for k, p in m.named_parameters()}, "cuda")
        assert torch.equal(got.view(torch.int32), flat.view(torch.int32)), ctx + ("run_one_iter_of_nerf_from_pose",)


@pytest.mark.parametrize("name, impl", RUNS, ids=[f"{n}-impl{i}" for n, i in RUNS])
def test_render_step_matches_fp64_stage_by_stage(name, impl):
    from nerf_pytorch_b200 import ops

    step = Step(name, impl)
    cfg, nc, nf, ns = step.cfg, step.nc, step.nf, step.ns
    ctx = (name, f"impl {impl}")
    if cfg.get("variants") and impl == 1:
        # seeded randoms, the 4096 rays' global indices straddling 2^32, against ops.random_fill's tensors
        rng = ops.SeededRandoms(seed=0x5EED, step=3, ray_offset=2 ** 32 - step.n // 2)
        rnd = _seeded_tensors(cfg, rng)
    else:
        rnd = _randoms(cfg, seed=5)
    out_c, out_f, ws = step.forward(rnd, zeroed=True)
    g_c, g_f = step.loss_upstream(out_c, out_f)

    # the inference forward computes the same bits
    inf_c, inf_f, ws_inf = step.forward(rnd, training=False)
    for what, a, b in (("z_coarse", ws_inf.z_c, ws.z_c), ("raw_coarse", ws_inf.raw_c, ws.raw_c),
                       ("weights_coarse", ws_inf.w_c, ws.w_c), ("z_fine", ws_inf.z_f, ws.z_f),
                       ("raw_fine", ws_inf.raw_f, ws.raw_f), ("out_coarse", inf_c, out_c), ("out_fine", inf_f, out_f)):
        assert bits_equal(a, b), ctx + ("training=False", what)
    del ws_inf, inf_c, inf_f

    if cfg.get("variants") and impl == 1:
        out_sc, out_sf, ws_s = step.forward(rng, zeroed=True)
        for what in ("z_c", "raw_c", "w_c", "z_f", "raw_f", "stash_c", "stash_f"):
            assert bits_equal(getattr(ws_s, what), getattr(ws, what)), ctx + ("seeded", what)
        assert bits_equal(out_sc, out_c) and bits_equal(out_sf, out_f), ctx + ("seeded outputs",)
        seeded = step.backward(rng, ws_s, g_c, g_f, parts=3)
        del ws_s

    # z_coarse: the fp32 CPU oracle with the same t_rand, bit for bit
    rays_cpu = step.rays.cpu()
    want = O.stratified_z(rays_cpu[:, 6:7], rays_cpu[:, 7:8], nc, cfg.get("lindisp", False), cfg["perturb"],
                          rnd["t_rand"].cpu() if cfg["perturb"] else None, torch.float32)
    assert bits_equal(ws.z_c.cpu(), want.contiguous()), ctx + ("z_coarse",)

    # compositing of both passes on our raw and z; resampling on our weights
    _check_compositing(out_c, ws.w_c, ws.raw_c, ws.z_c, step.rays, rnd.get("noise_c"), cfg, ctx + ("coarse",))
    if nf:
        _check_compositing(out_f, None, ws.raw_f, ws.z_f, step.rays, rnd.get("noise_f"), cfg, ctx + ("fine",))
        _check_resampling(ws, rnd, cfg, ctx)

    # upstream gradients: the training loss; with disp (zero where it is NaN) and acc terms added
    out_g = {"loss": (g_c, g_f), "extra": None}
    if cfg.get("variants") and impl == 1:
        gen = torch.Generator().manual_seed(23)
        extra = []
        for g, out in ((g_c, out_c), (g_f, out_f)):
            g = g.clone()
            scale = g[:, :3].abs().max().item()
            g[:, 3] = torch.where(torch.isnan(out[:, 3]), 0.0, torch.randn(step.n, generator=gen).cuda() * scale)
            g[:, 4] = torch.randn(step.n, generator=gen).cuda() * scale
            extra.append(g.contiguous())
        out_g["extra"] = tuple(extra)

    # part by part against fp64; each returns its gradient as training computes it, before any ReLU decision is adopted
    ff = None
    if nf:
        ff = _check_part(step, "fine", step.arch_f, step.sd_f, ws, ws.z_f, ws.raw_f, ws.stash_f, rnd.get("noise_f"),
                         out_g, rnd, ctx)
    fc = _check_part(step, "coarse", step.arch_c, step.sd_c, ws, ws.z_c, ws.raw_c, ws.stash_c, rnd.get("noise_c"),
                     out_g, rnd, ctx)
    del ws
    torch.cuda.empty_cache()

    if cfg.get("variants") and impl == 1:
        for a, b in zip(seeded, (fc, ff)):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), ctx + ("seeded gradients",)
    _check_against_training(step, rnd, g_c, g_f, fc, ff, ctx)


def test_wgmma_refuses_fewer_than_15_samples_before_any_launch():
    """A 14-sample pass needs 11 rays in a 128-point tile, one more than the wgmma kernels hold: render_fwd (training or
    not) and render_bwd on impl 1 refuse it before launching anything; impl 0 runs the same step (RUNS "nc14")."""
    from nerf_pytorch_b200 import ops

    step = Step("nc14", 1)
    rnd = _randoms(step.cfg, seed=5)
    n = step.n
    ws = torch.zeros(ops.render_workspace_bytes(step.arch_c, None, step.opts, n, True), dtype=torch.uint8,
                     device="cuda")
    g = torch.zeros(n, 8, device="cuda")
    flat = torch.zeros(step.arch_c.flat_param_count(), device="cuda")
    torch.cuda.synchronize()
    before = ops.launch_count()
    for training in (True, False):
        with pytest.raises(NotImplementedError, match="fewer than 15 samples"):
            step.forward(rnd, training=training)
    with pytest.raises(NotImplementedError, match="fewer than 15 samples"):
        ops.render_bwd(step.arch_c, None, step.opts, step.blob_c, None, step.rays, rnd, g, None, ws, flat, None,
                       impl=1, parts=3)
    assert ops.launch_count() == before
