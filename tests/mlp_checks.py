"""Shared machinery of the MLP-kernel tests (not a test module): parameter tables, the fp64 oracle MLP, the forward
stash's layout, the ReLU-tie rule, per-block gradient comparisons with the wgmma backward's absolute floors, the oracle
in chunks of whole tiles on the device for training-size batches, and one training step against the oracle.

The oracle is O.flexible_nerf_forward in fp64, fed the encoding run_network builds, with the points formed in fp32 as the
reference forms them (train_utils.py:67).  Its sin / cos arguments are the fp32 products x * f the reference evaluates
(nerf_helpers.py:149-151), promoted to fp64: for log-sampled bands that is exactly run_network's fp64 encoding (x * 2^k
is exact), for linear bands it removes the rounding of x * f that an fp64 run would not do."""
import functools
import types

import torch

from oracle import nerf_oracle as O

# hidden 256, skip 4: the pretrained configurations' family, trained on the fp32 kernels
H256_ARCHS = {
    "8x256": dict(num_layers=8, n_freq_xyz=10, n_freq_dir=4),
    "8x256_noview": dict(num_layers=8, n_freq_xyz=10, n_freq_dir=4, use_viewdirs=False),
    "8x256_lxyz6": dict(num_layers=8, n_freq_xyz=6, n_freq_dir=4),     # skip layer K = 256 + 40: a partial 16-row chunk
    "8x256_noinput_linear": dict(num_layers=8, n_freq_xyz=10, n_freq_dir=4, include_input_xyz=False,
                                 log_sampling_xyz=False, log_sampling_dir=False),
    "10x256": dict(num_layers=10, n_freq_xyz=10, n_freq_dir=4),          # two wide layers (layers_xyz.4 and .8)
    "8x256_ldir6": dict(num_layers=8, n_freq_xyz=10, n_freq_dir=6),     # the widest encodings the forward's smem fits
}
# hidden 128; the fused wgmma backward takes all of these
TC_ARCHS = {
    "1x128": dict(num_layers=1, skip_every=4, n_freq_xyz=10, n_freq_dir=4),
    "4x128_l0": dict(num_layers=4, skip_every=4, n_freq_xyz=0, n_freq_dir=0),
    "4x128_l1_skip2": dict(num_layers=4, skip_every=2, n_freq_xyz=1, n_freq_dir=1),
    "6x128_skip1": dict(num_layers=6, skip_every=1, n_freq_xyz=6, n_freq_dir=2),
    "8x128_noinput_linear": dict(num_layers=8, skip_every=3, n_freq_xyz=10, n_freq_dir=4, include_input_xyz=False,
                                 include_input_dir=False, log_sampling_xyz=False, log_sampling_dir=False),
    "8x128_widest": dict(num_layers=8, skip_every=4, n_freq_xyz=10, n_freq_dir=4),
    "16x128_skip5": dict(num_layers=16, skip_every=5, n_freq_xyz=6, n_freq_dir=4),
}
# hidden 128, the wgmma forward only: their training backward runs on the fp32 kernels
FWD_ONLY_ARCHS = {
    "8x128_ldir5_noinput": dict(num_layers=8, skip_every=4, n_freq_xyz=10, n_freq_dir=5, include_input_dir=False),
    "4x128_noview": dict(num_layers=4, skip_every=4, n_freq_xyz=5, log_sampling_xyz=False, use_viewdirs=False),
}
ALL_ARCHS = {**TC_ARCHS, **FWD_ONLY_ARCHS}
# hidden 128 that the wgmma training path refuses (encodings wider than 64 xyz / 32 direction channels, or a direction
# encoding wider than 28 in the fused backward): all of them train, and all but the last also render, on the fp32
# kernels.  The comments give xyz / direction channels and the wgrad_block<RN, RK> instances their encoding items reach.
SIMT128_ARCHS = {
    # the widest encodings (NERFB200_MAX_FREQS bands each) and the largest fp32 forward smem, 213 568 B: (8, 7), (4, 7)
    "8x128_lxyz16_ldir16": dict(num_layers=8, skip_every=4, n_freq_xyz=16, n_freq_dir=16),
    "6x128_lxyz13_ldir5_skip2": dict(num_layers=6, skip_every=2, n_freq_xyz=13, n_freq_dir=5),  # 81 / 33: (8, 6), (4, 3)
    "4x128_lxyz11_noinput_ldir8": dict(num_layers=4, skip_every=4, n_freq_xyz=11, n_freq_dir=8,
                                       include_input_xyz=False),                                # 66 / 51: (8, 5), (4, 4)
    # linear bands, not powers of two, so the fp32 product x * f rounds: 75 / 81, (8, 5), (4, 6)
    "10x128_lin12_ldir13": dict(num_layers=10, skip_every=4, n_freq_xyz=12, n_freq_dir=13, log_sampling_xyz=False,
                                log_sampling_dir=False),
    "3x128_ldir11_skip1": dict(num_layers=3, skip_every=1, n_freq_xyz=6, n_freq_dir=11),       # 39 / 69: (8, 3), (4, 5)
    # fc_out reads layer1's output, which has no ReLU; layer1 has no hidden columns: 99 / -, (8, 7)
    "1x128_lxyz16_noview": dict(num_layers=1, skip_every=4, n_freq_xyz=16, use_viewdirs=False),
    # the wgmma forward takes it, the fused backward does not: 63 / 30, (8, 4), (4, 2)
    "8x128_ldir5_noinput": FWD_ONLY_ARCHS["8x128_ldir5_noinput"],
}
# every architecture the fp32-kernel checks run (test_simt_mlp_gpu.py)
SIMT_NAMES = [*H256_ARCHS, *SIMT128_ARCHS]
STATES = ["init", "scaled"]
# one ray at the smallest sample count the wgmma kernels accept; tiles spanning 10 rays; ragged tiles
SHAPES = [(1, 15), (37, 15), (33, 17)]

# Worst raw element per output column as a fraction of the column's scale, wgmma forward (stash-writing and inference)
# against fp64.  Measured on an H100 80GB HBM3, worst over all parameter sets and both weight states [1.1e-5].
TC_FWD_TOL = 3e-5
# The fp32 kernels' raw outputs per column (test_simt_mlp_gpu.py FWD_TOL) [7.8e-7, test_tc_full_size_gpu.py].
SIMT_FWD_TOL = 3e-5
# Parameter gradients per block, relative to the block's scale (test_tc_arch_sweep_gpu.py BLOCK_TOL): at training size
# wgmma [6.3e-6, a probe], fp32 kernels [4.1e-6, A2] (test_tc_full_size_gpu.py, H100 80GB HBM3, 700 W, 1980 MHz).
BLOCK_TOL = 3e-5
# How far from zero a ReLU tie may sit, relative to the layer's scale: the wgmma stash [1.1e-5, A0 fern], and the fp32
# kernels' (test_tc_arch_sweep_gpu.py FP32_TIE_TOL).
STASH_TOL = 2e-5
FP32_TIE_TOL = 1e-5
# Compositing against fp64 (helpers.composite64): every output relative to its scale, and d_raw relative to its scale
# (test_stage_parity_gpu.py).
COMP_TOL = 1e-4
COMP_GRAD_TOL = 2e-4
# Early ray termination (helpers.transmittance64): how far the fp64 transmittance of the default raw may sit on the wrong
# side of the threshold t, relative to t.  Measured on an H100 80GB HBM3 over test_early_stop_gpu.py's cases: at most
# 0.99934 t at a stop and at least 1.00004 t at every earlier boundary.
T_REL = 2e-3
# Normal maps against normals64: |N - N64| per ray against the conditioning of its samples.  A gradient error of G_ERR
# times the pass's largest |grad| (test_density_grad_gpu bounds it by 2e-5 off ReLU ties) turns a sample's unit normal by
# at most 2 G_ERR max|g| / |g_i| (and never by more than 2), times its weight.  Samples where |grad| nearly vanishes are
# where N is ill-conditioned; a sample with a ReLU tie may turn its normal by up to 2 (times its weight).  Measured on an
# H100 80GB HBM3 at 700 W, the unconditioned worst is 1.1e-6 (lego), 6.8e-3 (fern, lego with noise).  ACC_EPS: |N| <= acc
# + ACC_EPS.
G_ERR = 1e-4
N_FLOOR = 1e-5
ACC_EPS = 1e-5


# Scenes of the render tests (test_occupancy_gpu, test_early_stop_gpu, test_normals_render_gpu): (shipped weights or
# None, H, W, focal, pose, no_ndc, near, far, L_xyz, (coarse, fine) networks, bounds of a grid).  A network is (layers,
# hidden, skip, weights): "shipped" (the scene's coarse / fine pair), "init" (torch's init under seed 7, in order) or
# ("scaled", seed) (arch_weights: max |raw| ~ 3e3, so rays turn opaque and early stopping fires).  These run the
# pretrained architecture, 8 x 256 skip 4 (A2), in the last pass, the first or both, on the lego camera; their grid box
# leaves the image's outer rays outside it.
_BOX = ((-0.7,) * 3, (0.7,) * 3)
H256_SCENES = {
    "a2": (None, 40, 40, 55.0, "spherical", True, 2.0, 6.0, 10, ((8, 256, 4, ("scaled", 1)), (8, 256, 4, ("scaled", 2))),
           _BOX),
    "mixed": (None, 40, 40, 55.0, "spherical", True, 2.0, 6.0, 10,
              ((8, 128, 3, ("scaled", 3)), (8, 256, 4, ("scaled", 2))), _BOX),
    "mixed_rev": (None, 40, 40, 55.0, "spherical", True, 2.0, 6.0, 10,
                  ((8, 256, 4, ("scaled", 1)), (8, 128, 3, ("scaled", 5))), _BOX),
}


def scene_models(scene):
    """The (coarse, fine) FlexibleNeRFModels of a scene row (H256_SCENES' format) on the GPU; "shipped" networks are
    helpers.shipped_models'."""
    import nerf_pytorch_b200 as nb
    from helpers import shipped_models
    from nerf_pytorch_b200 import ops

    weights, *_, l_xyz, nets, _ = scene
    shipped = shipped_models(weights.removesuffix("_lowres")) if weights else None
    if any(state == "init" for *_, state in nets):
        torch.manual_seed(7)
    out = []
    for i, (layers, hidden, skip, state) in enumerate(nets):
        if state == "shipped":
            out.append(shipped[i])
            continue
        m = nb.FlexibleNeRFModel(num_layers=layers, hidden_size=hidden, skip_connect_every=skip,
                                 num_encoding_fn_xyz=l_xyz, num_encoding_fn_dir=4)
        if state != "init":
            arch = ops.ArchSpec(num_layers=layers, hidden=hidden, skip_every=skip, n_freq_xyz=l_xyz, n_freq_dir=4)
            m.load_state_dict(arch_weights(arch, *state))
        out.append(m.cuda())
    return out


def spec(name):
    """The ops.ArchSpec of a table entry: H256_ARCHS at hidden 256 / skip 4, ALL_ARCHS and SIMT128_ARCHS at hidden
    128."""
    from nerf_pytorch_b200 import ops

    if name in H256_ARCHS:
        return ops.ArchSpec(hidden=256, skip_every=4, **H256_ARCHS[name])
    return ops.ArchSpec(hidden=128, **(ALL_ARCHS[name] if name in ALL_ARCHS else SIMT128_ARCHS[name]))


def arch_name(arch):
    """The table name of an ops.ArchSpec (its repr if it is in no table)."""
    return next((k for k in [*H256_ARCHS, *ALL_ARCHS, *SIMT128_ARCHS] if spec(k) == arch), repr(arch))


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def sms_shape(shape):
    """(rays, samples) with a ray count of "sms+1" or "8sms" resolved against the device's multiprocessor count."""
    n, s = shape
    if n == "sms+1":
        n = sms() + 1
    elif n == "8sms":
        n = 8 * sms()
    return n, s


def points(arch, n, s, seed):
    """Lego-like rays: origins on a sphere of radius 4 looking at the centre, near 2, far 6, sorted random depths."""
    g = torch.Generator().manual_seed(seed)
    o = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1) * 4.0
    d = -o / 4.0 + 0.25 * torch.randn(n, 3, generator=g)
    rays = torch.cat([o, d, torch.full((n, 1), 2.0), torch.full((n, 1), 6.0), d / d.norm(dim=-1, keepdim=True)], -1)
    z = torch.sort(torch.rand(n, s, generator=g) * 4 + 2, -1).values
    return (rays if arch.use_viewdirs else rays[:, :8]).contiguous(), z.contiguous()


def upstream(n, s, seed):
    """d(loss)/d(raw) whose rows span several decades, as compositing weights make them."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, s, 4, generator=g) * torch.exp(torch.randn(n, s, 1, generator=g) * 3.0)


def embed(x, L, include, log_sampling):
    from nerf_pytorch_b200 import ops

    parts = [x.double()] if include else []
    for f in ops.frequency_bands(L, log_sampling):
        a = (x * f).double()  # the fp32 argument, as the reference evaluates `tensor * freq` before sin / cos
        parts += [torch.sin(a), torch.cos(a)]
    return torch.cat(parts, -1)


def encodings(arch, rays, z):
    """fp64 xyz encoding [P][dim_xyz] of the fp32 points o + d z (train_utils.py:67), and the direction encoding
    [P][dim_dir] of each point's ray (None without view directions)."""
    pts = (rays[:, None, :3] + rays[:, None, 3:6] * z[..., None]).reshape(-1, 3)
    xyz = embed(pts, arch.n_freq_xyz, arch.include_input_xyz, arch.log_sampling_xyz)
    if not arch.use_viewdirs:
        return xyz, None
    vd = rays[:, None, 8:11].expand(*z.shape, 3).reshape(-1, 3)
    return xyz, embed(vd, arch.n_freq_dir, arch.include_input_dir, arch.log_sampling_dir)


def oracle(arch, sd, rays, z, G=None):
    """fp64: raw [P][4], every gemm layer's activation in the library's order and, given G, the gradients of
    sum(raw * G) with respect to every layer's pre-activation and every parameter."""
    sd64 = {k: v.double().requires_grad_(G is not None) for k, v in sd.items()}
    xyz, view = encodings(arch, rays, z)
    emb = xyz if view is None else torch.cat((xyz, view), -1)
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


@functools.lru_cache(maxsize=None)
def arch_weights(arch, state, seed=2024):
    """Reference init of `arch` (an ops.ArchSpec) seeded with `seed`; "scaled": every gemm layer's weight and bias times
    one factor c, found by bisection so that max |raw| over a probe batch is ~3e3."""
    sd = O.init_flexible_nerf(arch.num_layers, arch.hidden, arch.skip_every, arch.n_freq_xyz, arch.n_freq_dir,
                              include_input_xyz=arch.include_input_xyz, include_input_dir=arch.include_input_dir,
                              use_viewdirs=arch.use_viewdirs, generator=torch.Generator().manual_seed(seed))
    if state == "init":
        return sd
    rays, z = points(arch, 16, 64, seed=99)
    lo, hi = 1.0, 16.0
    for _ in range(24):
        c = (lo * hi) ** 0.5
        if oracle(arch, _scaled(sd, c), rays, z)[0].abs().max().item() < 3e3:
            lo = c
        else:
            hi = c
    return _scaled(sd, lo)


def setup(name, state, shape, seed):
    """arch, weights, rays and depths (CPU) and the packed weights (GPU) of one parameter set."""
    from nerf_pytorch_b200 import ops

    arch = spec(name)
    sd = arch_weights(arch, state)
    rays, z = points(arch, *sms_shape(shape), seed=seed)
    blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))
    return arch, sd, rays, z, blob


def report(what, ctx, value):
    print(f"measured {what} {ctx}: {value:.3e}")


# ------------------------------------------------------------------------------------------------------------------------
# the forward stash
# ------------------------------------------------------------------------------------------------------------------------
class StashLayout:
    """Sections of a forward stash, in 4-byte columns of P rows (fp32 kernels) or P_pad rows (wgmma, P rounded up to the
    128-point tile): every gemm layer's activations, `layers` = [(name, n, cum)] in the library's order (heads
    skipped); the xyz-encoding tile at column cum_total, enc_w wide; the direction encoding padded to 8; then the ReLU
    mask words from mask_base, n / 32 columns per gemm layer, layer li's at mask_base + mask_cum[li]."""

    def __init__(self, arch):
        self.layers, cum = [], 0
        for name, _, _, _, fout in arch.flat_layout():
            if fout >= 64:
                self.layers.append((name, fout, cum))
                cum += fout
        self.cum_total = cum
        self.enc_w = (arch.dim_xyz + 15) & ~15
        self.mask_base = cum + self.enc_w + ((arch.dim_dir + 7) & ~7)
        self.mask_cum = [sum(n // 32 for _, n, _ in self.layers[:li]) for li in range(len(self.layers))]


def _rows(n_points, family):
    return (n_points + 127) // 128 * 128 if family == "wgmma" else n_points


def read_layer(stash, n_points, cum, n, family, rows=None):
    """Columns [cum, cum + n) of a stash as fp64 [n_points][n], or of the points rows = (p0, p1) alone (for "wgmma"
    p0 a multiple of 128).  "wgmma": operand tiles (csrc/tc_common.cuh "Operand tiles"), fp16 hi + lo 2^-11 of
    value / 16; "fp32": fp32 rows with 16-byte chunks XOR-swizzled by (point & 7) inside each 128-byte segment
    (csrc/common.cuh swz_col)."""
    p0, p1 = rows or (0, n_points)
    if family == "wgmma":
        assert p0 % 128 == 0, p0
        t0, t1 = p0 // 128, (p1 + 127) // 128
        base = 2 * _rows(n_points, family) * cum
        raw = stash.view(torch.int16)[base + 256 * n * t0: base + 256 * n * t1]  # 2 x 128 x n halves per tile
        t = raw.view(t1 - t0, 2, 16, n // 8, 8, 8).view(torch.float16).double()  # [tile][hi|lo][pb][fb][p%8][f%8]
        val = (t[:, 0] + t[:, 1] / 2048.0) * 16.0
        return val.permute(0, 1, 3, 2, 4).reshape((t1 - t0) * 128, n)[:p1 - p0]
    x = stash[n_points * cum + p0 * n: n_points * cum + p1 * n].view(p1 - p0, n // 32, 8, 4)
    pt = torch.arange(p0, p1, device=stash.device) & 7
    q = torch.arange(8, device=stash.device)
    idx = (q[None, :] ^ pt[:, None])                                   # stored position of logical chunk q
    return torch.gather(x, 2, idx[:, None, :, None].expand(p1 - p0, n // 32, 8, 4)).reshape(p1 - p0, n).double()


def write_simt_layer(stash, P, cum, n, val, rows=None):
    """Inverse of read_layer(..., "fp32"): store val [P][n] (or [p1 - p0][n], rows = (p0, p1)) with the stash's row
    swizzle."""
    p0, p1 = rows or (0, P)
    x = stash[P * cum + p0 * n: P * cum + p1 * n].view(p1 - p0, n // 32, 8, 4)
    pt = torch.arange(p0, p1, device=stash.device) & 7
    idx = torch.arange(8, device=stash.device)[None, :] ^ pt[:, None]
    x.scatter_(2, idx[:, None, :, None].expand(p1 - p0, n // 32, 8, 4), val.float().view(p1 - p0, n // 32, 8, 4))


def mask_words(arch, stash, n_points, li, family, rows=None):
    """The ReLU mask words of gemm layer `li` in a forward stash: an int32 view [P][n/32] (or of the points
    rows = (p0, p1) alone), bit j of word w = column 32 w + j."""
    lay = StashLayout(arch)
    n = lay.layers[li][1]
    start = _rows(n_points, family) * (lay.mask_base + lay.mask_cum[li])
    p0, p1 = rows or (0, n_points)
    return stash.view(torch.int32)[start:start + n_points * (n // 32)].view(n_points, n // 32)[p0:p1]


def pack_mask(act):
    """bool [P][n] -> int32 words [P][n/32], bit j of word w = column 32 w + j."""
    P, n = act.shape
    b = act.view(P, n // 32, 32).to(torch.int64)
    w = (b << torch.arange(32, device=act.device, dtype=torch.int64)).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def relu_ties(arch, stash, P, acts, family, tol, ctx, adopt, rows=None, scales=None):
    """ReLU ties: a unit whose pre-activation is within rounding of zero is on in the kernel and off in fp64 or the
    reverse, a discontinuity of the function, not an error of the kernel.  Counts the forward's disagreements with the
    fp64 activations `acts`, checks that each is such a tie and that their number is bounded, and with `adopt` gives the
    stash the oracle's decisions so that a backward run on it is measured on its own arithmetic.  Returns the count.
      * "fp32": the data-gradient kernel takes its decision from the stashed activation (mlp_simt.cu, finish: a > 0); a
        tie is |a32 - a64| <= tol * scale, and adopting overwrites the activation with a64;
      * "wgmma": the backward reads the mask words; a tie is |a64| <= tol * scale, and adopting overwrites the words.
    rows = (p0, p1): `acts` are those points' alone (for "wgmma" p0 a multiple of 128), and the count is bounded for
    them; scales: every layer's scale (the whole run's max |activation|) instead of that of `acts`."""
    lay = StashLayout(arch)
    shifts = torch.arange(32, device=stash.device, dtype=torch.int32)
    n_pts = rows[1] - rows[0] if rows else P
    n_ties = 0
    for li, (lname, n, cum) in enumerate(lay.layers):
        if li == 0:
            continue  # layer1 has no ReLU (models.py:238); the backward does not read its decisions
        a64 = acts[li].to(stash.device)
        if family == "wgmma":
            words = mask_words(arch, stash, P, li, family, rows)
            want = pack_mask(a64 > 0)
            flip = (((words ^ want).unsqueeze(-1) >> shifts) & 1).view(n_pts, n).bool()
            off = a64
        else:
            a32 = read_layer(stash, P, cum, n, family, rows)
            flip = (a32 > 0) != (a64 > 0)
            off = a32 - a64
        k = int(flip.sum())
        if k:
            scale = scales[li] if scales else a64.abs().max().item()
            assert off[flip].abs().max().item() <= tol * scale, ctx + (lname,)
        if adopt and family == "wgmma":
            words.copy_(want)
        elif adopt and k:
            write_simt_layer(stash, P, cum, n, torch.where(flip, a64, a32), rows)
        n_ties += k
    assert n_ties <= 1e-5 * n_pts * lay.cum_total + 2, ctx + (n_ties,)
    return n_ties


def _adopt_masks(arch, stash, P, masks):
    """Give a wgmma stash the oracle's ReLU decisions (layer1 has no ReLU; the backward does not read its words)."""
    for li in range(1, len(StashLayout(arch).layers)):
        mask_words(arch, stash, P, li, "wgmma").copy_(masks[li])


# ------------------------------------------------------------------------------------------------------------------------
# gradients
# ------------------------------------------------------------------------------------------------------------------------
def as_state_dict(arch, flat):
    """Views of a flat parameter / gradient vector under the reference's state_dict names."""
    out = {}
    for name, w_off, b_off, fin, fout in arch.flat_layout():
        out[name + ".weight"] = flat[w_off:w_off + fin * fout].view(fout, fin)
        out[name + ".bias"] = flat[b_off:b_off + fout]
    return out


def block(t, rows, cols):
    return t[rows] if cols is None else t[rows, cols]


def tensor_blocks(arch):
    """(label, key, rows, cols) of every parameter tensor, whole."""
    out = []
    for name, _, _, _, _ in arch.flat_layout():
        out += [(name + ".weight", name + ".weight", slice(None), slice(None)),
                (name + ".bias", name + ".bias", slice(None), None)]
    return out


def tc_blocks(arch):
    """(label, key, rows, cols, per_cta) of every block the fused backward produces on its own path, from the rules of
    make_bwd_plan / blob_map (mlp_tc_bwd.cu):
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


def check_blocks(arch, got, want, blocks, tol, ctx, what, floors=None):
    """Every block (label, key, rows, cols, ...) of the flat gradient `got` within tol of the same block of the
    state_dict `want`, relative to that block's own scale, plus an absolute floor per label if given.  Reports the
    worst e / (scale + floor / tol), the figure the bar `tol` applies to, under `what` (None: no report)."""
    got_sd = as_state_dict(arch, got.double().cpu())
    worst = 0.0
    for label, key, rows, cols, *_ in blocks:
        g, w = block(got_sd[key], rows, cols), block(want[key].double().cpu(), rows, cols)
        scale = w.abs().max().item()
        e = (g - w).abs().max().item()
        floor = floors[label] if floors else 0.0
        assert scale > 0 and e <= tol * scale + floor, ctx + (what, label, e, scale, floor)
        worst = max(worst, e / (scale + floor / tol))
    if what:
        report(what, ctx, worst)


def random_previous(arch, g, blocks, seed):
    """flat_grad's previous contents for an accumulation test (CPU): random, every block at the scale of that block of
    the gradient g."""
    gen = torch.Generator().manual_seed(seed)
    prev = torch.zeros(g.shape)
    prev_sd, g_sd = as_state_dict(arch, prev), as_state_dict(arch, g.cpu())
    for _, key, rows, cols, *_ in blocks:
        b = block(prev_sd[key], rows, cols)
        b.copy_(torch.randn(b.shape, generator=gen) * block(g_sd[key], rows, cols).abs().max())
    return prev


# ------------------------------------------------------------------------------------------------------------------------
# the wgmma backward's absolute floors
# ------------------------------------------------------------------------------------------------------------------------
FIX_LSB = 2.0 ** -33  # rounding of one add into the fixed-point gradient blob (resolution 2^-32)
# Resolution of the fp16x2 split below fp16's normal range (tc_common.cuh split_f16x2): hi and lo are subnormal there,
# so x = hi + lo 2^-11 is resolved to 2^-36 absolutely.  The fused backward splits G (and d_raw) at the tile's scale,
# max |d_raw| of the tile -> [4, 8), so a G element is resolved to 2^-36 / 4 = 2^-38 of the tile's max |d_raw|, however
# small it is; the stash holds activation / 16, resolved to 2^-36 * 16 = 2^-32 absolutely.
G_SPLIT_LSB = 2.0 ** -38
ACT_SPLIT_LSB = 2.0 ** -32
BLOB_MAX = 2.0 ** 28  # the gradient blob holds sums below 2^31 (mlp_tc_bwd.cu); the checks keep every gradient below this


def _floors(arch, n_points, split_floors=None):
    """label -> the floor of every tc_blocks block: the fixed-point rounding n_adds * 2^-33 plus, for the wgmma kernels,
    the split's resolution floor of that block (_split_floors)."""
    n_tiles = -(-n_points // 128)
    n_ctas = min(n_tiles, sms())
    return {label: (n_ctas if per_cta else n_tiles) * FIX_LSB + (split_floors or {}).get(label, 0.0)
            for label, _, _, _, per_cta in tc_blocks(arch)}


def blob_range_factor(grads):
    """The power of two (1 or below) that brings every parameter gradient below BLOB_MAX."""
    m = max(v.abs().max().item() for v in grads.values())
    return 2.0 ** -int(torch.tensor(m / BLOB_MAX).log2().ceil().item()) if m > BLOB_MAX else 1.0


def _in_blob_range(arch, sd, rays, z, G):
    """fp64 oracle of sum(raw * G), with G scaled by a power of two (exact on both sides) if needed so that every
    parameter gradient stays below BLOB_MAX.  Returns (G, acts, dpre, grads)."""
    _, acts, dpre, want = oracle(arch, sd, rays, z, G)
    c = blob_range_factor(want)
    if c != 1.0:
        G, dpre, want = G * c, [x * c for x in dpre], {k: v * c for k, v in want.items()}
    return G, acts, dpre, want


def _split_floors(arch, G, acts, dpre, rays, z, into=None):
    """label -> the wgmma backward's resolution floor of that block, from the split's absolute resolution:
        sum_p G_SPLIT_LSB * D(p) * max |X[p]|  +  ACT_SPLIT_LSB * max |G[p]|
    over the points p, with D(p) the max |d_raw| of p's tile, X the block's input columns (activations, encodings, or 1
    for the indicator sums) and G the block's output rows of the pre-activation gradient (d_raw for the heads).  It
    matters where G is many decades below d_raw: the deep layers of an initialised network, whose gradient vanishes.
    A sum over points: given `into` (a previous result), the sums of these points, whole 128-point tiles from a tile's
    first point, are added to it, so that a run can be accumulated chunk by chunk."""
    P = z.numel()
    d_raw = G.reshape(-1, 4).double().abs()
    D = torch.nn.functional.pad(d_raw.amax(1), (0, -P % 128)).view(-1, 128).amax(1).repeat_interleave(128)[:P]
    xyz, view = encodings(arch, rays, z)
    x_enc = xyz.abs().amax(1)
    x_dir = None if view is None else view.abs().amax(1)
    index = {lname: li for li, (lname, _, _) in enumerate(StashLayout(arch).layers)}
    heads = {"fc_alpha": (arch.num_layers - 1, [3]), "fc_rgb": (len(acts) - 1, [0, 1, 2]),
             "fc_out": (arch.num_layers - 1, [0, 1, 2, 3])}
    out = {}
    for label, key, rows, cols, _ in tc_blocks(arch):
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
    if into is not None:
        out = {label: into[label] + v for label, v in out.items()}
    return out


# ------------------------------------------------------------------------------------------------------------------------
# the oracle at training size: chunks of whole tiles on the device
# ------------------------------------------------------------------------------------------------------------------------
def oracle_tiles(arch, sd, rays, z, G=None, tiles=None, chunk_tiles=128, visit=None):
    """The oracle over the points of (rays [n][C], z [n][S]), 128-point tile by tile in chunks of chunk_tiles on the
    device of z, or over tiles = (t0, t1) of them alone: a run at training size decodes to tens of GB in fp64 at once.
    Returns a namespace with, for the points covered,
      raw      fp64 [points][4];
      masks    per gemm layer, the fp64 ReLU decisions as pack_mask words [points][n / 32];
      act_max  per gemm layer, max |activation|;
    and given G [n][S][4] (the upstream gradient of every point), the sums over the chunks of
      grads    every parameter gradient of sum(raw * G) (a state_dict, fp64);
      split    _split_floors of those points.
    visit(p0, p1, rays_c, z_c, acts) sees each chunk: points [p0, p1), one row per point of rays and z, and their fp64
    activations."""
    dev = z.device
    n_rays, S = z.shape
    P = n_rays * S
    t0, t1 = tiles or (0, (P + 127) // 128)
    sd_d = {k: v.to(dev) for k, v in sd.items()}
    lay = StashLayout(arch)
    first = t0 * 128
    n_pts = min(t1 * 128, P) - first
    out = types.SimpleNamespace(raw=torch.empty(n_pts, 4, dtype=torch.float64, device=dev),
                                masks=[torch.empty(n_pts, n // 32, dtype=torch.int32, device=dev)
                                       for _, n, _ in lay.layers],
                                act_max=[0.0] * len(lay.layers), grads=None, split=None)
    for c0 in range(t0, t1, chunk_tiles):
        p0, p1 = c0 * 128, min(min(c0 + chunk_tiles, t1) * 128, P)
        idx = torch.arange(p0, p1, device=dev)
        rays_c, z_c = rays[idx // S], z.reshape(-1)[p0:p1, None]
        G_c = None if G is None else G.reshape(-1, 4)[p0:p1]
        raw, acts, dpre, grads = oracle(arch, sd_d, rays_c, z_c, G_c)
        out.raw[p0 - first:p1 - first] = raw.detach()
        for li, a in enumerate(acts):
            out.masks[li][p0 - first:p1 - first] = pack_mask(a > 0)
            out.act_max[li] = max(out.act_max[li], a.abs().max().item())
        if G is not None:
            out.grads = grads if out.grads is None else {k: out.grads[k] + v for k, v in grads.items()}
            out.split = _split_floors(arch, G_c, acts, dpre, rays_c, z_c, into=out.split)
        if visit is not None:
            visit(p0, p1, rays_c, z_c, acts)
        del raw, acts, dpre, grads
    return out


# ------------------------------------------------------------------------------------------------------------------------
# density gradients and normal maps
# ------------------------------------------------------------------------------------------------------------------------
def relu_tie_points(sd64, xyz, hidden):
    """Points with a ReLU tie: a layers_xyz unit within STASH_TOL of its layer's largest activation (over this batch)
    from zero in fp64, where the kernel's decision may be the other one.  xyz: the fp64 xyz encoding [P][dim_xyz]."""
    h = torch.nn.functional.linear(xyz, sd64["layer1.weight"], sd64["layer1.bias"])
    tie = torch.zeros(xyz.shape[0], dtype=torch.bool, device=xyz.device)
    i = 0
    while f"layers_xyz.{i}.weight" in sd64:
        w = sd64[f"layers_xyz.{i}.weight"]
        if w.shape[1] != hidden:
            h = torch.cat((h, xyz), -1)
        pre = torch.nn.functional.linear(h, w, sd64[f"layers_xyz.{i}.bias"])
        tie |= (pre.abs() <= STASH_TOL * pre.max().clamp_min(0.0)).any(-1)
        h = torch.relu(pre)
        i += 1
    return tie


def sigma_grad64(arch, sd, pts):
    """fp64 autograd of sigma (raw column 3, the fc_alpha output or fc_out's fourth) with respect to the fp32 points
    pts [P][3], and the points with a ReLU tie (relu_tie_points).  The bands' arguments are the fp32 products x * f as
    values (as embed forms them) with the derivative f, for log-sampled and linear bands, with or without the raw input;
    sigma does not depend on the view direction, which is +z."""
    from nerf_pytorch_b200 import ops

    sd64 = {k: v.double().to(pts.device) for k, v in sd.items()}
    bands = ops.frequency_bands(arch.n_freq_xyz, arch.log_sampling_xyz).tolist()
    d = torch.tensor([0.0, 0.0, 1.0], device=pts.device)
    out, ties = [], []
    for p0 in range(0, pts.shape[0], 1 << 17):
        x32 = pts[p0:p0 + (1 << 17)]
        x64 = x32.double().requires_grad_()
        parts = [x64] if arch.include_input_xyz else []
        for f in bands:
            a = x64 * f + ((x32 * f).double() - x64.detach() * f)
            parts += [torch.sin(a), torch.cos(a)]
        xyz = torch.cat(parts, -1)
        emb = xyz
        if arch.use_viewdirs:
            view = embed(d.expand(x32.shape[0], 3), arch.n_freq_dir, arch.include_input_dir, arch.log_sampling_dir)
            emb = torch.cat((xyz, view), -1)
        raw = O.flexible_nerf_forward(sd64, emb, arch.dim_xyz)
        g, = torch.autograd.grad(raw[:, 3].sum(), x64)
        out.append(g)
        with torch.no_grad():
            ties.append(relu_tie_points(sd64, xyz.detach(), arch.hidden))
    return torch.cat(out), torch.cat(ties)


def normals64(arch, sd, rays, z, raw, noise_std=0.0, noise=None):
    """fp64 restatement of a render's normal map from its last pass: depths z [n][S] and raw [n][S][4] read from the
    render's workspace, the fp64 compositing weights of that raw (helpers.composite64, with the noise the render used),
    and the outward unit normal -grad sigma / |grad sigma| by sigma_grad64 at o + d z, summed in sample order.
    Returns (N64 [n][3], bound [n], live samples, tie samples): bound is the allowance on |N - N64| per ray, the sum of
    its samples' weights times how far each may turn (G_ERR relative to the pass's largest |grad|, 2 at a ReLU tie),
    plus N_FLOOR."""
    from helpers import composite64

    pts = (rays[:, None, :3] + rays[:, None, 3:6] * z[..., None]).reshape(-1, 3)
    _, _, _, w64, _ = composite64(raw, z, rays[:, 3:6], noise_std=noise_std, noise=noise)
    w64 = w64.reshape(-1)
    live = w64 != 0
    g = torch.zeros(pts.shape[0], 3, dtype=torch.float64, device=pts.device)
    tie = torch.zeros(pts.shape[0], dtype=torch.bool, device=pts.device)
    if live.any():
        g[live], tie[live] = sigma_grad64(arch, sd, pts[live].contiguous())
    mag = g.norm(dim=-1, keepdim=True)
    nrm64 = torch.where(mag > 0, -g / mag, torch.zeros_like(g))
    terms = (w64[:, None] * nrm64).view(rays.shape[0], -1, 3)
    N64 = torch.zeros(rays.shape[0], 3, dtype=torch.float64, device=pts.device)
    for j in range(terms.shape[1]):  # in sample order
        N64 += terms[:, j]
    turn = torch.clamp(2 * G_ERR * mag.max() / mag.squeeze(-1).clamp_min(1e-300), max=2.0)
    turn[tie] = 2.0  # a ReLU tie may turn its sample's normal anywhere
    bound = (w64 * turn).view(rays.shape[0], -1).sum(-1) + N_FLOOR
    return N64, bound, int(live.sum()), int(tie.sum())


# ------------------------------------------------------------------------------------------------------------------------
# one training step end to end
# ------------------------------------------------------------------------------------------------------------------------
def step_inputs(arch, seed, n_coarse, n_fine):
    """Seeded coarse and fine weights of `arch` and 96 lego-like rays with their injected randoms and targets."""
    g = torch.Generator().manual_seed(seed)
    sds = [O.init_flexible_nerf(arch.num_layers, arch.hidden, arch.skip_every, arch.n_freq_xyz, arch.n_freq_dir,
                                generator=g) for _ in range(2)]
    n = 96
    ro = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1) * 4.0
    rd = -ro / 4.0 + 0.25 * torch.randn(n, 3, generator=g)
    rnd = dict(t_rand=torch.rand(n, n_coarse, generator=g), noise_c=torch.randn(n, n_coarse, generator=g),
               u=torch.rand(n, n_fine, generator=g), noise_f=torch.randn(n, n_coarse + n_fine, generator=g))
    target = torch.rand(n, 3, generator=g)
    return sds, ro, rd, rnd, target


def training_step_vs_oracle(monkeypatch, arch, seed, n_coarse, n_fine, ctx, rel_l2, coarse_vs_ref32, loss_tol,
                            fix_lsb=0.0, white=False):
    """Coarse and fine networks of `arch` (step_inputs), perturb and noise std 0.2 with injected randoms, through
    run_one_iter_of_nerf(mode="train"), against fp64 autograd of the oracle: the loss within loss_tol relative; every
    coarse tensor's worst element within coarse_vs_ref32 x the fp32 oracle's worst there; each network's relative L2
    within rel_l2.  fix_lsb: the rounding of one fixed-point gradient add, added to both bars once per 128-point tile.
    Returns the impl of every render_fwd / render_bwd call the step made."""
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    used = []
    render_fwd, render_bwd = ops.render_fwd, ops.render_bwd
    monkeypatch.setattr(ops, "render_fwd", lambda *a, **k: used.append(k["impl"]) or render_fwd(*a, **k))
    monkeypatch.setattr(ops, "render_bwd", lambda *a, **k: used.append(k["impl"]) or render_bwd(*a, **k))

    sds, ro, rd, rnd, target = step_inputs(arch, seed, n_coarse, n_fine)
    models = []
    for sd in sds:
        m = nb.FlexibleNeRFModel(num_layers=arch.num_layers, hidden_size=arch.hidden,
                                 skip_connect_every=arch.skip_every, num_encoding_fn_xyz=arch.n_freq_xyz,
                                 num_encoding_fn_dir=arch.n_freq_dir)
        m.load_state_dict(sd)
        models.append(m.cuda())
    opts = O.make_options(num_coarse=n_coarse, num_fine=n_fine, perturb=True, radiance_field_noise_std=0.2,
                          white_background=white)
    enc_xyz, enc_dir = (arch.n_freq_xyz, True, True), (arch.n_freq_dir, True, True)

    out = nb.run_one_iter_of_nerf(100, 100, 120.0, models[0], models[1], ro.cuda(), rd.cuda(), opts, mode="train",
                                  encode_position_fn=nb.get_embedding_function(*enc_xyz),
                                  encode_direction_fn=nb.get_embedding_function(*enc_dir),
                                  randoms={k: v.cuda() for k, v in rnd.items()})
    tgt = target.cuda()
    loss = torch.nn.functional.mse_loss(out[0], tgt) + torch.nn.functional.mse_loss(out[3], tgt)
    loss.backward()
    torch.cuda.synchronize()

    def run_oracle(dtype):
        sd_ = [{k: v.detach().to(dtype).clone().requires_grad_(True) for k, v in sd.items()} for sd in sds]
        out_ = O.run_one_iter_of_nerf(100, 100, 120.0, sd_[0], sd_[1], ro.to(dtype), rd.to(dtype), opts, mode="train",
                                      enc_xyz=enc_xyz, enc_dir=enc_dir,
                                      randoms={k: v.to(dtype) for k, v in rnd.items()})
        loss_ = O.nerf_loss(out_, target.to(dtype))
        loss_.backward()
        return loss_.item(), [{k: v.grad.double() for k, v in s.items()} for s in sd_]

    loss64, g64 = run_oracle(torch.float64)
    _, g32 = run_oracle(torch.float32)
    e_loss = abs(loss.item() - loss64) / abs(loss64)
    report("e2e loss", ctx, e_loss)
    assert e_loss <= loss_tol, (loss.item(), loss64)
    label = "e2e coarse worst / (fp32 oracle's + floor / bar)" if fix_lsb else "e2e coarse worst / fp32 oracle's"
    n = ro.shape[0]
    nets = (("coarse", models[0], n_coarse), ("fine", models[1], n_coarse + n_fine))
    for i, (tag, model, samples) in enumerate(nets):
        floor = -(-n * samples // 128) * fix_lsb  # one fixed-point add per tile at most, per element
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
                report(label, ctx + (k,), e / (e_ref + floor / coarse_vs_ref32))
                assert e <= coarse_vs_ref32 * e_ref + floor, ctx + (k, e, e_ref, s)
        rel = (num / den) ** 0.5
        report("e2e rel L2", ctx + (tag,), rel)
        assert rel <= rel_l2 + count ** 0.5 * floor / den ** 0.5, ctx + (tag, rel)
    return used
