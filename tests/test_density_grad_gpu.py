"""The density gradient (include/nerfb200.h, "density gradient"; csrc/mlp_tc.cu density_grad_tc_kernel) on the GPU.

  * sigma_raw is bit for bit what the wgmma forward (mlp_fwd_pts, impl 1) writes at the same points;
  * the gradient against fp64 autograd of the oracle MLP and the positional encoding w.r.t. the points, per component
    relative to the batch's largest |grad|, over hidden-128 sweep architectures, A0, A1, A2 (hidden 256), the shipped
    lego and fern weights, init and x3e3-output weights, and point counts 1 .. 2 M;
  * ReLU ties -- a unit whose fp64 pre-activation sits within rounding of zero, where the kernel's on-chip decision may
    differ from fp64's -- are found from the fp64 pre-activations with mlp_checks' tie rule, asserted rare, and bounded
    apart from the main bar;
  * an operand past the fp16 range gives inf / NaN, not a clamped value;
  * mesh vertex normals: -grad / |grad| of the kernel at the vertices, against fp64, and outward (they agree with the
    area-weighted normals of the adjacent faces)."""
import numpy as np
import pytest
import torch

import mlp_checks as M
from helpers import bits_equal, load_weights
from oracle import nerf_oracle as O

pytestmark = pytest.mark.gpu

# Worst gradient component over non-tie points, relative to the batch's max |grad| (fp64), over every case below:
# measured on an H100 80GB HBM3 at 700 W [6.6e-6, 16x128_skip5 scaled; 2e-6 typical at hidden 128, 4e-6 at 256].
GRAD_TOL = 2e-5
# ReLU ties (a trunk unit within mlp_checks.STASH_TOL of its layer's scale from zero in fp64): at most TIE_UNIT_FRAC of
# the batch's units [measured up to 1.4e-4, 63 points], and a point with one is within TIE_GRAD_TOL of the batch scale
# [measured up to 0.11, 2 M points] (a unit switched on or off moves the gradient by that unit's share).  With hundreds
# of units per point, a few percent of the points hold one.
TIE_UNIT_FRAC = 5e-4
TIE_GRAD_TOL = 0.2
# Unit vertex normals against fp64 at vertices whose |grad| is at least NORMAL_MIN of the mesh's median [1.4e-5].
NORMAL_TOL = 1e-4
NORMAL_MIN = 0.05
# lego A0 mesh at 128^3: fraction of vertices whose normal points the way of their faces' area-weighted normal
# [0.874].  The analytic gradient sees detail finer than the lattice spacing (10 bands reach wavelengths of 0.012, the
# lattice steps 0.023), which the faces, interpolated from the lattice, do not.
ORIENT_FRAC = 0.85


def report(what, ctx, value):
    print(f"measured {what} {ctx}: {value}")


def _embed(x64, x32, L, include, log_sampling):
    """Positional encoding in fp64 with the fp32 arguments x * f the kernel and the reference use as values, and d/dx
    = f (the rounding of x * f has no derivative).  The bands as the reference builds them (nerf_helpers.py:131-147),
    derived here rather than taken from the package under test."""
    bands = (2.0 ** torch.linspace(0.0, L - 1, L, dtype=torch.float32) if log_sampling
             else torch.linspace(2.0 ** 0.0, 2.0 ** (L - 1), L, dtype=torch.float32)) if L else torch.zeros(0)
    parts = [x64] if include else []
    for f in bands:
        a32 = (x32 * f).double()
        a = x64 * float(f) + (a32 - x64.detach() * float(f))
        parts += [torch.sin(a), torch.cos(a)]
    return torch.cat(parts, -1)


def _pre_activations(sd64, xyz, hidden):
    """The fp64 pre-activations of the trunk's ReLU layers (layers_xyz)."""
    h = torch.nn.functional.linear(xyz, sd64["layer1.weight"], sd64["layer1.bias"])
    pres, i = [], 0
    while f"layers_xyz.{i}.weight" in sd64:
        w = sd64[f"layers_xyz.{i}.weight"]
        if w.shape[1] != hidden:
            h = torch.cat((h, xyz), -1)
        pre = torch.nn.functional.linear(h, w, sd64[f"layers_xyz.{i}.bias"])
        pres.append(pre)
        h = torch.relu(pre)
        i += 1
    return pres


def oracle(arch, sd, pts, chunk=1 << 17):
    """fp64 (sigma_raw, grad, tie) at fp32 points (P, 3) on the device: tie[p] = some ReLU unit of the trunk is within
    mlp_checks.STASH_TOL of its layer's scale (over the whole batch) from zero."""
    sd64 = {k: v.double().to(pts.device) for k, v in sd.items()}
    sig, grad, pres_max, pres, n_units = [], [], None, [], 0
    for p0 in range(0, pts.shape[0], chunk):
        x32 = pts[p0:p0 + chunk]
        x64 = x32.double().requires_grad_()
        xyz = _embed(x64, x32, arch.n_freq_xyz, arch.include_input_xyz, arch.log_sampling_xyz)
        emb = xyz
        if arch.use_viewdirs:
            d = torch.tensor([0.0, 0.0, 1.0], device=pts.device).expand(x32.shape[0], 3)
            emb = torch.cat((xyz, M.embed(d, arch.n_freq_dir, arch.include_input_dir, arch.log_sampling_dir)), -1)
        raw = O.flexible_nerf_forward(sd64, emb, arch.dim_xyz)
        g, = torch.autograd.grad(raw[:, 3].sum(), x64)
        sig.append(raw[:, 3].detach())
        grad.append(g)
        with torch.no_grad():
            pre = _pre_activations(sd64, xyz.detach(), arch.hidden)
        mx = [q.max().clamp_min(0.0) for q in pre]  # the layer's scale: its largest activation
        pres_max = mx if pres_max is None else [torch.maximum(a, b) for a, b in zip(pres_max, mx)]
        pres.append([q.abs() for q in pre])
        n_units += sum(q.numel() for q in pre)
    tie = torch.zeros(pts.shape[0], dtype=torch.bool, device=pts.device)
    tie_units = 0
    for ci, pr in enumerate(pres):
        for q, s in zip(pr, pres_max):
            near = q <= M.STASH_TOL * s
            tie_units += int(near.sum())
            tie[ci * chunk:ci * chunk + q.shape[0]] |= near.any(-1)
    return torch.cat(sig), torch.cat(grad), tie, tie_units / max(n_units, 1)


def forward_sigma(arch, blob, pts):
    """raw sigma of the wgmma inference forward (mlp_fwd_pts, impl 1) at pts (P, 3): rows of 64 samples."""
    from nerf_pytorch_b200 import ops

    n = pts.shape[0]
    pad = (-n) % 64
    rows = torch.cat((pts, pts[:1].expand(pad, 3))).view(-1, 64, 3).contiguous()
    dirs = torch.tensor([[0.0, 0.0, 1.0]], device=pts.device).expand(rows.shape[0], 3) if arch.use_viewdirs else None
    return ops.mlp_fwd_pts(arch, blob, rows, dirs, impl=ops.IMPL_TC).view(-1, 4)[:n, 3]


def uniform_points(n, seed, lo=-1.5, hi=1.5):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(n, 3, generator=g) * (hi - lo) + lo).cuda()


def check(arch, sd, pts, ctx):
    """The kernel at pts against the forward (sigma bits) and fp64 (grad); returns (worst, tie fraction)."""
    from nerf_pytorch_b200 import ops

    blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))
    out = ops.density_grad(arch, blob, pts)
    assert bits_equal(out[:, 0], forward_sigma(arch, blob, pts)), ctx
    _, g64, tie, unit_frac = oracle(arch, sd, pts)
    scale = g64.norm(dim=-1).max().item()
    err = (out[:, 1:].double() - g64).abs().max(-1).values / scale
    assert torch.isfinite(out).all(), ctx
    frac = tie.float().mean().item()
    worst = err[~tie].max().item() if (~tie).any() else 0.0
    worst_tie = err[tie].max().item() if tie.any() else 0.0
    report("grad err / batch scale", ctx, f"{worst:.3e} (tie units {unit_frac:.2e}, tie points {frac:.4f}, worst tie "
                                          f"{worst_tie:.3e}, scale {scale:.3e})")
    assert worst <= GRAD_TOL, (ctx, worst)
    assert unit_frac <= TIE_UNIT_FRAC, (ctx, unit_frac)
    assert worst_tie <= TIE_GRAD_TOL, (ctx, worst_tie)
    return worst, frac


# A0 / A1 at 128, A2 at 256, and the mlp_checks sweep: skip every 1 .. 5, linear bands, no view directions, 1 layer,
# no frequency bands
ARCHS = ["A0", "A1", "A2", "1x128", "4x128_l0", "4x128_l1_skip2", "6x128_skip1", "8x128_noinput_linear",
         "16x128_skip5", "4x128_noview", "8x256_noview", "8x256_noinput_linear"]


def spec(name):
    from nerf_pytorch_b200 import ops

    if name == "A0":
        return ops.ArchSpec(num_layers=4, hidden=128, skip_every=4, n_freq_xyz=10, n_freq_dir=4)
    if name == "A1":
        return ops.ArchSpec(num_layers=8, hidden=128, skip_every=3, n_freq_xyz=10, n_freq_dir=4)
    if name == "A2":
        return ops.ArchSpec(num_layers=8, hidden=256, skip_every=4, n_freq_xyz=10, n_freq_dir=4)
    return M.spec(name)


def _ragged_multiwave():
    # several full waves of CTA tiles over every SM plus a partial tile (two 64-row blocks per tile at hidden 128)
    return 3 * M.sms() * 128 + 77


@pytest.mark.parametrize("state", ["init", "scaled"])
@pytest.mark.parametrize("name", ARCHS)
def test_grad_matches_fp64_across_architectures(name, state):
    arch = spec(name)
    check(arch, M.arch_weights(arch, state), uniform_points(4099, seed=3), (name, state))


@pytest.mark.parametrize("n", [1, 63, 64, 65, "waves"])
@pytest.mark.parametrize("name", ["A1", "A2"])
def test_point_counts(name, n):
    arch = spec(name)
    n = _ragged_multiwave() if n == "waves" else n
    check(arch, M.arch_weights(arch, "init"), uniform_points(n, seed=5 + n), (name, n))


def _shipped(which):
    """A0 with the encoding widths of the shipped weights (lego: 10 / 4 bands, fern: 6 / 4)."""
    from nerf_pytorch_b200 import ops

    _, sd_f = load_weights(which)
    lx = (sd_f["layer1.weight"].shape[1] - 3) // 6
    ld = (sd_f["layers_dir.0.weight"].shape[1] - 128 - 3) // 6
    return ops.ArchSpec(num_layers=4, hidden=128, skip_every=4, n_freq_xyz=lx, n_freq_dir=ld), sd_f


@pytest.mark.parametrize("which,lo,hi", [("lego_lowres", -1.5, 1.5), ("fern_lowres", -1.0, 1.0)])
def test_shipped_weights(which, lo, hi):
    arch, sd = _shipped(which)
    check(arch, sd, uniform_points(65536, seed=7, lo=lo, hi=hi), (which,))


def test_two_million_points():
    arch = spec("A1")
    check(arch, M.arch_weights(arch, "scaled"), uniform_points(1 << 21, seed=11), ("A1", "2M"))


def test_out_of_range_operands_are_not_clamped():
    """sigma head weights past 16 x 65504: the seed of the reverse chain leaves the fp16 range, so every gradient is
    inf / NaN; sigma itself (an fp32 head) keeps the forward's bits."""
    from nerf_pytorch_b200 import ops

    arch = spec("A0")
    sd = dict(M.arch_weights(arch, "init"))
    sd["fc_alpha.weight"] = sd["fc_alpha.weight"].sign() * 2e6
    blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))
    pts = uniform_points(1000, seed=13)
    out = ops.density_grad(arch, blob, pts)
    assert bits_equal(out[:, 0], forward_sigma(arch, blob, pts))
    assert not torch.isfinite(out[:, 1:]).all(-1).any()


# ---- the public API and mesh normals ---------------------------------------------------------------------------------
def _lego():
    import nerf_pytorch_b200 as nb

    _, sd_f = load_weights("lego_lowres")
    m = nb.FlexibleNeRFModel(num_layers=4, hidden_size=128, skip_connect_every=4, num_encoding_fn_xyz=10,
                             num_encoding_fn_dir=4)
    m.load_state_dict(sd_f)
    return m.cuda(), nb.get_embedding_function(10), nb.get_embedding_function(4), sd_f


def test_density_gradient_api_is_the_kernel_and_keeps_shapes():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    model, epf, _, sd = _lego()
    arch, _ = _shipped("lego_lowres")
    pts = uniform_points(2 * 3 * 50, seed=17).view(2, 3, 50, 3)
    with torch.no_grad():
        sigma, grad = nb.density_gradient(model, epf, pts)
    assert sigma.shape == (2, 3, 50) and grad.shape == (2, 3, 50, 3)
    blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))
    out = ops.density_grad(arch, blob, pts.reshape(-1, 3).contiguous())
    assert bits_equal(sigma.reshape(-1), out[:, 0]) and bits_equal(grad.reshape(-1, 3), out[:, 1:])
    with pytest.raises(NotImplementedError, match="inference only"):
        nb.density_gradient(model, epf, pts)  # autograd on, parameters require grad
    with torch.no_grad():
        for bad in (ops.IMPL_SIMT, ops.IMPL_TC_FAST):
            n0 = ops.launch_count()
            with pytest.raises(NotImplementedError, match="impl=1"):
                nb.density_gradient(model, epf, pts, impl=bad)
            assert ops.launch_count() == n0


def test_mesh_vertex_normals():
    import nerf_pytorch_b200 as nb

    model, epf, edf, sd = _lego()
    arch, _ = _shipped("lego_lowres")
    box = ((-1.5,) * 3, (1.5,) * 3)
    with torch.no_grad():
        plain = nb.extract_mesh(model, epf, box, 128, 50.0, encode_direction_fn=edf)
        m = nb.extract_mesh(model, epf, box, 128, 50.0, encode_direction_fn=edf, normals=True)
    assert plain.normals is None and bits_equal(plain.vertices, m.vertices) and torch.equal(plain.faces, m.faces)
    v, f, n = m.vertices, m.faces.long(), m.normals
    assert n.shape == v.shape and v.shape[0] > 0
    # against fp64 at the vertices
    _, g64, tie, _ = oracle(arch, sd, v)
    mag = g64.norm(dim=-1)
    n64 = -g64 / mag[:, None]
    keep = (mag >= NORMAL_MIN * mag.median()) & ~tie
    err = (n.double() - n64).abs().max(-1).values[keep].max().item()
    report("lego A0 128^3 vertex normals", "max |n - n64|", f"{err:.3e} over {int(keep.sum())} / {v.shape[0]}")
    assert err <= NORMAL_TOL
    assert torch.allclose(n.norm(dim=-1)[mag > 0], torch.ones_like(mag[mag > 0]).float(), atol=1e-5)
    # outward: agree with the area-weighted normals of the adjacent faces (counter-clockwise seen from outside)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    fn = torch.linalg.cross(b - a, c - a)  # twice the area times the unit normal
    acc = torch.zeros_like(v)
    for k in range(3):
        acc.index_add_(0, f[:, k], fn)
    agree = ((acc * n).sum(-1) > 0).float().mean().item()
    report("lego A0 128^3 vertex normals", "fraction agreeing with face normals", f"{agree:.4f}")
    assert agree >= ORIENT_FRAC


def test_ply_with_normals(tmp_path):
    import nerf_pytorch_b200 as nb

    model, epf, edf, _ = _lego()
    with torch.no_grad():
        m = nb.extract_mesh(model, epf, ((-1.5,) * 3, (1.5,) * 3), 64, 50.0, encode_direction_fn=edf, normals=True)
    path = tmp_path / "lego_n.ply"
    m.save_ply(path)
    data = path.read_bytes()
    head, body = data.split(b"end_header\n", 1)
    assert b"property float nx\nproperty float ny\nproperty float nz\n" in head
    V = m.vertices.shape[0]
    rec = np.frombuffer(body[:V * 24], dtype="<f4").reshape(V, 6)
    assert np.array_equal(rec[:, :3], m.vertices.cpu().numpy()) and np.array_equal(rec[:, 3:], m.normals.cpu().numpy())
