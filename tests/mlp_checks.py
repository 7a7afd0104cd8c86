"""Shared machinery of the MLP-kernel tests (not a test module): parameter tables, the fp64 oracle MLP, the forward
stash's layout, the ReLU-tie rule, per-block gradient comparisons and one training step against the oracle.

The oracle is O.flexible_nerf_forward in fp64, fed the encoding run_network builds, with the points formed in fp32 as the
reference forms them (train_utils.py:67).  Its sin / cos arguments are the fp32 products x * f the reference evaluates
(nerf_helpers.py:149-151), promoted to fp64: for log-sampled bands that is exactly run_network's fp64 encoding (x * 2^k
is exact), for linear bands it removes the rounding of x * f that an fp64 run would not do."""
import functools

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
STATES = ["init", "scaled"]
# one ray at the smallest sample count the wgmma kernels accept; tiles spanning 10 rays; ragged tiles
SHAPES = [(1, 15), (37, 15), (33, 17)]

# Worst raw element per output column as a fraction of the column's scale, wgmma forward (stash-writing and inference)
# against fp64.  Measured on an H100 80GB HBM3, worst over all parameter sets and both weight states [1.1e-5].
TC_FWD_TOL = 3e-5


def spec(name):
    """The ops.ArchSpec of a table entry: H256_ARCHS at hidden 256 / skip 4, ALL_ARCHS at hidden 128."""
    from nerf_pytorch_b200 import ops

    if name in H256_ARCHS:
        return ops.ArchSpec(hidden=256, skip_every=4, **H256_ARCHS[name])
    return ops.ArchSpec(hidden=128, **ALL_ARCHS[name])


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
def arch_weights(arch, state):
    """Seeded reference init of `arch` (an ops.ArchSpec); "scaled": every gemm layer's weight and bias times one factor
    c, found by bisection so that max |raw| over a probe batch is ~3e3."""
    sd = O.init_flexible_nerf(arch.num_layers, arch.hidden, arch.skip_every, arch.n_freq_xyz, arch.n_freq_dir,
                              include_input_xyz=arch.include_input_xyz, include_input_dir=arch.include_input_dir,
                              use_viewdirs=arch.use_viewdirs, generator=torch.Generator().manual_seed(2024))
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


def read_layer(stash, n_points, cum, n, family):
    """Columns [cum, cum + n) of a stash as fp64 [n_points][n].  "wgmma": operand tiles (csrc/tc_common.cuh "Operand
    tiles"), fp16 hi + lo 2^-11 of value / 16; "fp32": fp32 rows with 16-byte chunks XOR-swizzled by (point & 7) inside
    each 128-byte segment (csrc/common.cuh swz_col)."""
    if family == "wgmma":
        tiles = (n_points + 127) // 128
        p_pad = tiles * 128
        raw = stash.view(torch.int16)[2 * p_pad * cum: 2 * p_pad * (cum + n)]
        t = raw.view(tiles, 2, 16, n // 8, 8, 8).view(torch.float16).double()  # [tile][hi|lo][pb][fb][p%8][f%8]
        val = (t[:, 0] + t[:, 1] / 2048.0) * 16.0
        return val.permute(0, 1, 3, 2, 4).reshape(p_pad, n)[:n_points]
    x = stash[n_points * cum: n_points * (cum + n)].view(n_points, n // 32, 8, 4)
    pt = torch.arange(n_points, device=stash.device) & 7
    q = torch.arange(8, device=stash.device)
    idx = (q[None, :] ^ pt[:, None])                                   # stored position of logical chunk q
    return torch.gather(x, 2, idx[:, None, :, None].expand(n_points, n // 32, 8, 4)).reshape(n_points, n).double()


def write_simt_layer(stash, P, cum, n, val):
    """Inverse of read_layer(..., "fp32"): store val [P][n] with the stash's row swizzle."""
    x = stash[P * cum: P * (cum + n)].view(P, n // 32, 8, 4)
    pt = torch.arange(P, device=stash.device) & 7
    idx = torch.arange(8, device=stash.device)[None, :] ^ pt[:, None]
    x.scatter_(2, idx[:, None, :, None].expand(P, n // 32, 8, 4), val.float().view(P, n // 32, 8, 4))


def mask_words(arch, stash, n_points, li, family):
    """The ReLU mask words of gemm layer `li` in a forward stash: an int32 view [P][n/32], bit j of word w = column
    32 w + j."""
    lay = StashLayout(arch)
    n = lay.layers[li][1]
    start = _rows(n_points, family) * (lay.mask_base + lay.mask_cum[li])
    return stash.view(torch.int32)[start:start + n_points * (n // 32)].view(n_points, n // 32)


def pack_mask(act):
    """bool [P][n] -> int32 words [P][n/32], bit j of word w = column 32 w + j."""
    P, n = act.shape
    b = act.view(P, n // 32, 32).to(torch.int64)
    w = (b << torch.arange(32, device=act.device, dtype=torch.int64)).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def relu_ties(arch, stash, P, acts, family, tol, ctx, adopt):
    """ReLU ties: a unit whose pre-activation is within rounding of zero is on in the kernel and off in fp64 or the
    reverse, a discontinuity of the function, not an error of the kernel.  Counts the forward's disagreements with the
    fp64 activations `acts`, checks that each is such a tie and that their number is bounded, and with `adopt` gives the
    stash the oracle's decisions so that a backward run on it is measured on its own arithmetic.  Returns the count.
      * "fp32": the data-gradient kernel takes its decision from the stashed activation (mlp_simt.cu, finish: a > 0); a
        tie is |a32 - a64| <= tol * scale, and adopting overwrites the activation with a64;
      * "wgmma": the backward reads the mask words; a tie is |a64| <= tol * scale, and adopting overwrites the words."""
    lay = StashLayout(arch)
    shifts = torch.arange(32, device=stash.device, dtype=torch.int32)
    n_ties = 0
    for li, (lname, n, cum) in enumerate(lay.layers):
        if li == 0:
            continue  # layer1 has no ReLU (models.py:238); the backward does not read its decisions
        a64 = acts[li].to(stash.device)
        if family == "wgmma":
            words = mask_words(arch, stash, P, li, family)
            want = pack_mask(a64 > 0)
            flip = (((words ^ want).unsqueeze(-1) >> shifts) & 1).view(P, n).bool()
            off = a64
        else:
            a32 = read_layer(stash, P, cum, n, family)
            flip = (a32 > 0) != (a64 > 0)
            off = a32 - a64
        k = int(flip.sum())
        if k:
            assert off[flip].abs().max().item() <= tol * a64.abs().max().item(), ctx + (lname,)
        if adopt and family == "wgmma":
            words.copy_(want)
        elif adopt and k:
            write_simt_layer(stash, P, cum, n, torch.where(flip, a64, a32))
        n_ties += k
    assert n_ties <= 1e-5 * P * lay.cum_total + 2, ctx + (n_ties,)
    return n_ties


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
