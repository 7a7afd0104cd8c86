"""World-space geometry of forward-facing (NDC) scenes on the GPU (include/nerfb200.h "NDC scenes"; csrc/ndc.cu), on the
shipped fern network and on A1 at init:
  * the map kernels (N, N^-1 with the face swap and the view directions, J^T) bit for bit against a torch fp32
    restatement of the header's op order;
  * density_gradient(ndc=) against fp64 autograd of the oracle MLP composed with N at world points in the frustum, per
    component relative to the batch's largest |grad|; sigma_raw with the bits of the wgmma forward at N(p);
  * extract_mesh(ndc=) at 128^3 and 256^3: N^-1 of the NDC mesh's vertices, its faces with two ids swapped, colors of
    the network at the NDC vertices seen along the world directions, normals against fp64, and the faces' orientation;
  * the sparse path over an NDC occupancy grid against the dense world mesh on the active bricks;
  * normals="world": on fern, sum of w_i n_i formed in fp32 from the render's weights and the world gradients at its
    samples; on lego, bit for bit normals=True; the six other outputs bit for bit those of the render without normals."""
import os
import re

import numpy as np
import pytest
import torch

import mlp_checks as M
from helpers import bits_equal, shipped_models
from oracle import nerf_oracle as O

pytestmark = pytest.mark.gpu

# the fern scene of the shipped weights, as tests/test_normals_render_gpu.py renders it
H, W, FOCAL = 42, 56, 45.3
# an NDC box inside the frustum, short of the far plane at z = 1
BOX = ((-1.0, -1.0, -1.0), (1.0, 1.0, 0.95))
# Bars as tests/test_density_grad_gpu.py: worst non-tie component relative to the batch's largest |grad|, and ReLU
# ties.  Measured on an H100 80GB HBM3 at 700 W: 1.7e-6 (fern), 2.3e-6 (A1 at init); ties 1.0e-3, 4.7e-3.
GRAD_TOL = 2e-5
TIE_GRAD_TOL = 0.2
# Unit world vertex normals against fp64 at vertices whose |grad| is at least NORMAL_MIN of the mesh's median
# [1.3e-5 .. 1.5e-5].
NORMAL_TOL = 1e-4
NORMAL_MIN = 0.05
# Orientation of the world faces of non-negligible area (test_world_mesh): the share counter-clockwise seen from
# outside, "outside" being the side opposite the vertices' lattice-gradient view directions [fern 0.99527 at 128^3,
# 0.99837 at 256^3; A1 at init 0.96532], and the share whose orientation sign is that of the NDC face [1.000000,
# 1.000000; 0.999999].  A1 at init puts 10 bands on a 128^3 lattice over a box of side 2: its shortest wavelength
# (0.012) is below the lattice step (0.016), so its faces and lattice gradients disagree more.
ORIENT_FRAC = {"fern": 0.99, "a1_init": 0.95}
SAME_SIGN_FRAC = 0.9999


def report(what, ctx, value):
    print(f"measured {what} {ctx}: {value}")


def _cam():
    from nerf_pytorch_b200 import ops

    return ops.ndc_struct(H, W, FOCAL)


def _swh():
    """sw, sh as fp32 values: -1 / (W / (2 f)) in double with the fp32 focal, rounded once."""
    f = float(np.float32(FOCAL))
    return float(np.float32(-1.0 / (float(W) / (2.0 * f)))), float(np.float32(-1.0 / (float(H) / (2.0 * f))))


# ---- the header's op order in torch fp32 (every torch elementwise op on CUDA rounds once) -----------------------------
def t_forward(p):
    sw, sh = (torch.tensor(v, dtype=torch.float32, device=p.device) for v in _swh())
    return torch.stack([(sw * p[:, 0]) / p[:, 2], (sh * p[:, 1]) / p[:, 2], 1.0 + 2.0 / p[:, 2]], -1)


def t_inverse(q):
    sw, sh = (torch.tensor(v, dtype=torch.float32, device=q.device) for v in _swh())
    pz = 2.0 / (q[:, 2] - 1.0)
    return torch.stack([(q[:, 0] * pz) / sw, (q[:, 1] * pz) / sh, pz], -1)


def t_grad(q, g):
    sw, sh = (torch.tensor(v, dtype=torch.float32, device=q.device) for v in _swh())
    qz1 = q[:, 2] - 1.0
    s = qz1 * 0.5
    t = q[:, 0] * g[:, 0] + q[:, 1] * g[:, 1]
    return torch.stack([s * (sw * g[:, 0]), s * (sh * g[:, 1]), s * (-t - qz1 * g[:, 2])], -1)


def t_unit(v):
    sq = v * v
    ln = (sq[:, 0] + sq[:, 1]) + sq[:, 2]
    ok = (ln > 0) & (ln < float("inf"))
    d = v / torch.sqrt(ln)[:, None]
    z = torch.tensor([0.0, 0.0, 1.0], device=v.device).expand_as(v)
    return torch.where(ok[:, None], d, z)


def jt64(q, g):
    sw, sh = _swh()
    q = q.double()
    s = (q[:, 2] - 1.0) * 0.5
    return torch.stack([s * sw * g[:, 0], s * sh * g[:, 1],
                        s * (-(q[:, 0] * g[:, 0] + q[:, 1] * g[:, 1]) - (q[:, 2] - 1.0) * g[:, 2])], -1)


# ---- networks ---------------------------------------------------------------------------------------------------------
def _net(name):
    """(model, encode_position_fn, encode_direction_fn, state dict, arch)."""
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    if name == "fern":
        _, m, epf, edf = shipped_models("fern")
        arch = ops.ArchSpec(num_layers=4, hidden=128, skip_every=4, n_freq_xyz=6, n_freq_dir=4)
    else:
        torch.manual_seed(11)  # A1 at init, its sigma bias shifted so that raw sigma changes sign inside the box
        m = nb.FlexibleNeRFModel(num_layers=8, hidden_size=128, skip_connect_every=3, num_encoding_fn_xyz=10,
                                 num_encoding_fn_dir=4).cuda()
        epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
        lo, hi = torch.tensor(BOX[0]), torch.tensor(BOX[1])
        pts = (torch.rand(1 << 14, 3, generator=torch.Generator().manual_seed(3)) * (hi - lo) + lo).cuda()
        with torch.no_grad():
            sigma, _ = nb.density_gradient(m, epf, pts)
            m.fc_alpha.bias -= sigma.median()
        arch = ops.ArchSpec(num_layers=8, hidden=128, skip_every=3, n_freq_xyz=10, n_freq_dir=4)
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    return m, epf, edf, sd, arch


def _level(model, epf, edf):
    import nerf_pytorch_b200 as nb

    vol = nb.density_volume(model, epf, BOX, 64, encode_direction_fn=edf)
    return float(vol[vol > 0].median())


def oracle(arch, sd, x32, q32, to_q):
    """fp64 autograd of raw sigma w.r.t. the leaf x (fp32 points x32, mapped to the NDC point by to_q in fp64; q32 the
    fp32 NDC point the kernel encodes, whose rounded band arguments are taken as values), and the points with a ReLU
    tie (a trunk unit within mlp_checks.STASH_TOL of its layer's largest activation from zero)."""
    sd64 = {k: v.double().cuda() for k, v in sd.items()}
    grads, ties = [], []
    d = torch.tensor([0.0, 0.0, 1.0], device="cuda")
    for p0 in range(0, x32.shape[0], 1 << 16):
        x64 = x32[p0:p0 + (1 << 16)].double().requires_grad_()
        qq = q32[p0:p0 + (1 << 16)]
        q64 = to_q(x64)
        parts = [q64]
        for k in range(arch.n_freq_xyz):
            f = 2.0 ** k  # log-sampled bands: 2^k, exact in fp32
            a = q64 * f + ((qq * f).double() - q64.detach() * f)
            parts += [torch.sin(a), torch.cos(a)]
        xyz = torch.cat(parts, -1)
        emb = torch.cat((xyz, M.embed(d.expand(qq.shape[0], 3), arch.n_freq_dir, True, True)), -1)
        raw = O.flexible_nerf_forward(sd64, emb, arch.dim_xyz)
        g, = torch.autograd.grad(raw[:, 3].sum(), x64)
        grads.append(g)
        with torch.no_grad():
            xyz = xyz.detach()
            h = torch.nn.functional.linear(xyz, sd64["layer1.weight"], sd64["layer1.bias"])
            tie = torch.zeros(xyz.shape[0], dtype=torch.bool, device="cuda")
            i = 0
            while f"layers_xyz.{i}.weight" in sd64:
                w = sd64[f"layers_xyz.{i}.weight"]
                if w.shape[1] != arch.hidden:
                    h = torch.cat((h, xyz), -1)
                pre = torch.nn.functional.linear(h, w, sd64[f"layers_xyz.{i}.bias"])
                tie |= (pre.abs() <= M.STASH_TOL * pre.max().clamp_min(0.0)).any(-1)
                h = torch.relu(pre)
                i += 1
            ties.append(tie)
    return torch.cat(grads), torch.cat(ties)


def _n64(x64):
    sw, sh = _swh()
    return torch.stack([sw * x64[:, 0] / x64[:, 2], sh * x64[:, 1] / x64[:, 2], 1.0 + 2.0 / x64[:, 2]], -1)


def _inv64(q):
    """N^-1 in fp64."""
    sw, sh = _swh()
    pz = 2.0 / (q[:, 2] - 1.0)
    return torch.stack([q[:, 0] * pz / sw, q[:, 1] * pz / sh, pz], -1)


def forward_sigma(arch, blob, q):
    """raw sigma of the wgmma inference forward (mlp_fwd_pts, impl 1) at q (P, 3): rows of 64 samples."""
    from nerf_pytorch_b200 import ops

    n = q.shape[0]
    rows = torch.cat((q, q[:1].expand((-n) % 64, 3))).view(-1, 64, 3).contiguous()
    dirs = torch.tensor([[0.0, 0.0, 1.0]], device=q.device).expand(rows.shape[0], 3)
    return ops.mlp_fwd_pts(arch, blob, rows, dirs, impl=ops.IMPL_TC).view(-1, 4)[:n, 3]


def _frustum(n, seed):
    """World points (fp32, z < 0) whose NDC images fill BOX."""
    g = torch.Generator().manual_seed(seed)
    lo, hi = torch.tensor(BOX[0], dtype=torch.float64), torch.tensor(BOX[1], dtype=torch.float64)
    q = torch.rand(n, 3, generator=g, dtype=torch.float64) * (hi - lo) + lo
    sw, sh = _swh()
    pz = 2.0 / (q[:, 2] - 1.0)
    return torch.stack([q[:, 0] * pz / sw, q[:, 1] * pz / sh, pz], -1).float().cuda()


# ---- the map kernels --------------------------------------------------------------------------------------------------
def test_map_kernels_are_the_headers_op_order():
    from nerf_pytorch_b200 import ops

    cam = _cam()
    p = _frustum(200003, 1)
    q = ops.ndc_from_world(cam, p)
    assert bits_equal(q, t_forward(p))
    g = torch.randn(q.shape[0], 4, generator=torch.Generator("cuda").manual_seed(2), device="cuda")
    g[:7, 1:] = 0.0
    out = ops.ndc_grad_to_world(cam, q, g)
    assert bits_equal(out[:, 0], g[:, 0]) and bits_equal(out[:, 1:], t_grad(q, g[:, 1:]))
    inplace = g.clone()
    ops.ndc_grad_to_world(cam, q, inplace, out=inplace)
    assert bits_equal(inplace, out)
    # a mesh: more faces than vertices, and the reverse
    for nv, nf in ((1000, 2503), (3001, 17)):
        v = q[:nv].contiguous()
        f = torch.randint(0, nv, (nf, 3), dtype=torch.int32, device="cuda",
                          generator=torch.Generator("cuda").manual_seed(nf))
        d = t_unit(torch.randn(nv, 3, device="cuda", generator=torch.Generator("cuda").manual_seed(nv)))
        d[:5] = torch.tensor([0.0, 0.0, 1.0], device="cuda")  # the view directions' own fallback
        wv, wf, wd = ops.ndc_mesh_to_world(cam, v, f, d)
        assert bits_equal(wv, t_inverse(v))
        assert torch.equal(wf, f[:, [0, 2, 1]])
        assert bits_equal(wd, t_unit(t_grad(v, d)))
        wv2, wf2, wd2 = ops.ndc_mesh_to_world(cam, v, f)
        assert bits_equal(wv2, wv) and torch.equal(wf2, wf) and wd2 is None
    # round trip: N^-1(N(p)) within a few ulp of p
    back = t_inverse(q)
    rel = ((back - p).abs() / p.abs().clamp_min(1e-30)).max().item()
    report("N^-1(N(p)) relative error", "", f"{rel:.2e}")
    assert rel < 1e-5


# ---- density_gradient(ndc=) -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["fern", "a1_init"])
def test_density_gradient_in_world_space(name):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import train_utils

    model, epf, edf, sd, arch = _net(name)
    p = _frustum(65536, 7)
    with torch.no_grad():
        sigma, grad = nb.density_gradient(model, epf, p, ndc=(H, W, FOCAL))
        s2, g2 = nb.density_gradient(model, epf, p.view(256, 256, 3), ndc=(H, W, FOCAL))
    assert bits_equal(s2.reshape(-1), sigma) and bits_equal(g2.reshape(-1, 3), grad)
    q = t_forward(p)
    a = train_utils._arch_of(model, train_utils._probe_encoder(epf, None), train_utils._probe_encoder(edf, None))
    assert a == arch
    _, blob = train_utils._packed(model, a)
    assert bits_equal(sigma, forward_sigma(a, blob, q))
    g64, tie = oracle(arch, sd, p, q, _n64)
    scale = g64.norm(dim=-1).max().item()
    err = (grad.double() - g64).abs().max(-1).values / scale
    worst = err[~tie].max().item()
    worst_tie = err[tie].max().item() if tie.any() else 0.0
    report("world grad err / batch scale", name, f"{worst:.3e} (tie points {tie.float().mean().item():.4f}, worst tie "
                                                 f"{worst_tie:.3e}, scale {scale:.3e})")
    assert torch.isfinite(grad).all()
    assert worst <= GRAD_TOL and worst_tie <= TIE_GRAD_TOL
    # J^T of the plain NDC gradient at N(p), in fp32: the same bits
    with torch.no_grad():
        _, gq = nb.density_gradient(model, epf, q)
    assert bits_equal(grad, t_grad(q, gq))


# ---- extract_mesh(ndc=) -----------------------------------------------------------------------------------------------
def _ndc_dirs(model, epf, edf, res, level):
    """The NDC mesh's own vertices, faces and view directions, through the library's dense path."""
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    vol = nb.density_volume(model, epf, BOX, res, encode_direction_fn=edf)
    box = ops.grid_struct(BOX, (res,) * 3)
    totals, ws = ops.mesh_count(box, vol, level)
    n_v, n_f = (int(t) for t in totals.tolist())
    v, f, d = ops.mesh_emit(box, vol, level, ws, n_v, n_f, want_dirs=True)
    return vol, v, f, d


@pytest.mark.parametrize("name,res", [("fern", 128), ("fern", 256), ("a1_init", 128)])
def test_world_mesh(name, res):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops, train_utils

    model, epf, edf, sd, arch = _net(name)
    level = _level(model, epf, edf)
    with torch.no_grad():
        ndc_mesh = nb.extract_mesh(model, epf, BOX, res, level, encode_direction_fn=edf)
        wm = nb.extract_mesh(model, epf, BOX, res, level, encode_direction_fn=edf, colors=True, normals=True,
                             ndc=(H, W, FOCAL))
        _, v, f, d = _ndc_dirs(model, epf, edf, res, level)
    report(name, f"{res}^3 level / vertices / faces", (level, v.shape[0], f.shape[0]))
    assert f.shape[0] > 100
    assert bits_equal(v, ndc_mesh.vertices) and torch.equal(f, ndc_mesh.faces)
    # vertices, faces
    assert bits_equal(wm.vertices, t_inverse(v))
    assert torch.equal(wm.faces, f[:, [0, 2, 1]])
    assert (wm.vertices[:, 2] < 0).all()
    # colors: the network at the NDC vertex, seen along the world view direction
    wd = t_unit(t_grad(v, d))
    a = train_utils._arch_of(model, train_utils._probe_encoder(epf, None), train_utils._probe_encoder(edf, None))
    _, blob = train_utils._packed(model, a)
    with torch.no_grad():
        raw = ops.mlp_fwd_pts(a, blob, v.view(-1, 1, 3), wd, impl=train_utils._auto_impl(a, None, 1, 0, False))
    assert bits_equal(wm.colors, torch.sigmoid(raw.view(-1, 4)[:, :3]))
    # normals: -J^T g / |J^T g| against fp64
    gq64, tie = oracle(arch, sd, v, v, lambda x: x)
    g64 = jt64(v, gq64)
    mag = g64.norm(dim=-1)
    n64 = -g64 / mag[:, None]
    keep = (mag >= NORMAL_MIN * mag.median()) & ~tie
    err = (wm.normals.double() - n64).abs().max(-1).values[keep].max().item()
    report(f"{name} {res}^3 world vertex normals", "max |n - n64|", f"{err:.3e} over {int(keep.sum())} / {v.shape[0]}")
    assert err <= NORMAL_TOL
    # orientation, without a metric: the sign of det[b - a, c - a, x_out - a] over a face's world vertices and the world
    # image x_out of its NDC centroid stepped outward (against the vertices' mean NDC view direction) by a quarter
    # cell.  A projective map scales such a determinant by det J over a product of four negative denominators, so the
    # swap must restore, face by face, the sign the NDC mesh has; and that sign says the face is counter-clockwise seen
    # from outside.  Faces of non-negligible area only (in NDC, against the lattice cell).
    fl, fq = wm.faces.long(), f.long()
    h = min((hi - lo) / res for lo, hi in zip(*BOX))
    vq, dq = v.double(), d.double()
    cen = (vq[fq[:, 0]] + vq[fq[:, 1]] + vq[fq[:, 2]]) / 3
    dm = dq[fq[:, 0]] + dq[fq[:, 1]] + dq[fq[:, 2]]
    x_out_q = cen - 0.25 * h * dm / dm.norm(dim=-1, keepdim=True)
    nq = torch.linalg.cross(vq[fq[:, 1]] - vq[fq[:, 0]], vq[fq[:, 2]] - vq[fq[:, 0]])
    big = (nq.norm(dim=-1) / 2 >= 1e-2 * h * h) & (dm.norm(dim=-1) > 0)
    side_q = (nq * (x_out_q - vq[fq[:, 0]])).sum(-1)
    wv = wm.vertices.double()
    nw = torch.linalg.cross(wv[fl[:, 1]] - wv[fl[:, 0]], wv[fl[:, 2]] - wv[fl[:, 0]])
    side_w = (nw * (_inv64(x_out_q) - wv[fl[:, 0]])).sum(-1)
    same = ((side_w > 0) == (side_q > 0))[big].float().mean().item()
    outward = (side_w > 0)[big].float().mean().item()
    report(f"{name} {res}^3 world faces", "share outward / share with the NDC face's sign",
           f"{outward:.5f} / {same:.6f} over {int(big.sum())} / {fl.shape[0]}")
    assert int(big.sum()) > 0.5 * fl.shape[0]
    assert same >= SAME_SIGN_FRAC
    assert outward >= ORIENT_FRAC[name]


# ---- the sparse path over an NDC occupancy grid -----------------------------------------------------------------------
def _counts_table():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    text = open(os.path.join(root, "nerf_pytorch_b200", "csrc", "mc_table.cuh")).read()
    return torch.tensor([int(v) for v in re.findall(r"-?\d+", re.search(r"kMcTriCount\[256\] = \{(.*?)\};", text,
                                                                          re.S).group(1))])


def _dense_keys(vol, level):
    """Sorted keys q * 3 + a of the crossing lattice edges: the dense vertex order."""
    n2, n1, n0 = vol.shape
    ins = vol > level
    q = torch.arange(n2 * n1 * n0, device=vol.device).view(n2, n1, n0)
    keys = [q[:, :, :-1][ins[:, :, :-1] != ins[:, :, 1:]] * 3,
            q[:, :-1, :][ins[:, :-1, :] != ins[:, 1:, :]] * 3 + 1,
            q[:-1][ins[:-1] != ins[1:]] * 3 + 2]
    return torch.sort(torch.cat(keys)).values


def _face_bricks(vol, level, B):
    """The brick of the cube of each dense face (faces run cube by cube, the table's count each)."""
    n2, n1, n0 = vol.shape
    ins = (vol > level).to(torch.int64)
    case = torch.zeros(n2 - 1, n1 - 1, n0 - 1, dtype=torch.int64, device=vol.device)
    for c in range(8):
        dx, dy, dz = c & 1, c >> 1 & 1, c >> 2 & 1
        case |= ins[dz:n2 - 1 + dz, dy:n1 - 1 + dy, dx:n0 - 1 + dx] << c
    cnt = _counts_table().to(vol.device)[case.view(-1)]
    nb_ = [-(-(n - 1) // B) for n in (n0, n1, n2)]
    k = torch.arange(n2 - 1, device=vol.device) // B
    j = torch.arange(n1 - 1, device=vol.device) // B
    i = torch.arange(n0 - 1, device=vol.device) // B
    brick = ((k[:, None, None] * nb_[1] + j[None, :, None]) * nb_[0] + i[None, None, :]).reshape(-1)
    return torch.repeat_interleave(brick, cnt)


def _canon(faces):
    f = faces.cpu().numpy()
    return f[np.lexsort(f.T[::-1])] if f.size else f.reshape(0, 3)


def test_sparse_world_mesh_is_the_dense_one_on_active_bricks():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import mesh, ops

    model, epf, edf, _, _ = _net("fern")
    level = _level(model, epf, edf)
    res = 256
    grid = nb.OccupancyGrid.from_models([model], epf, BOX, 128, threshold=0.0, encode_direction_fn=edf)
    with torch.no_grad():
        dense = nb.extract_mesh(model, epf, BOX, res, level, encode_direction_fn=edf, colors=True, normals=True,
                                ndc=(H, W, FOCAL))
        sp, skeys = mesh._extract_mesh(model, epf, BOX, res, level, edf, True, None, None, True, grid, None,
                                       edge_keys=True, ndc=(H, W, FOCAL))
        vol = nb.density_volume(model, epf, BOX, res, encode_direction_fn=edf)
    brick_map, _, n_dev = ops.mesh_sparse_bricks(ops.grid_struct(BOX, (res,) * 3), grid)
    dkeys = _dense_keys(vol, level)
    assert dkeys.numel() == dense.vertices.shape[0]
    keep = brick_map[_face_bricks(vol, level, ops.mesh_brick())] >= 0
    df = dense.faces[keep]
    idx = torch.searchsorted(dkeys, skeys)
    assert bool((idx < dkeys.numel()).all()) and torch.equal(dkeys[idx.clamp(max=dkeys.numel() - 1)], skeys)
    for a, b in ((dense.vertices, sp.vertices), (dense.colors, sp.colors), (dense.normals, sp.normals)):
        assert bits_equal(b, a[idx])
    assert np.array_equal(_canon(idx[sp.faces.long()]), _canon(df.long()))
    report("fern 256^3 sparse world mesh", "active bricks / faces / dense faces",
           (int(n_dev.item()), sp.faces.shape[0], dense.faces.shape[0]))
    assert sp.faces.shape[0] > 0


# ---- normal maps ------------------------------------------------------------------------------------------------------
def test_world_normal_map_of_a_fern_render():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops, train_utils

    mc, mf, epf, edf = shipped_models("fern")
    opts_o = O.make_options(no_ndc=False, near=0.0, far=1.0, num_coarse=64, num_fine=128, perturb=False,
                            radiance_field_noise_std=0.0)
    kw = dict(mode="validation", encode_position_fn=epf, encode_direction_fn=edf, impl=1)
    with torch.no_grad():
        plain = nb.render_image(H, W, FOCAL, torch.eye(4), mc, mf, opts_o, **kw)
        ndc_n = nb.render_image(H, W, FOCAL, torch.eye(4), mc, mf, opts_o, normals=True, **kw)
        world = nb.render_image(H, W, FOCAL, torch.eye(4), mc, mf, opts_o, normals="world", **kw)
    assert len(world) == 7 and all(bits_equal(a, b) for a, b in zip(plain, world[:6]))
    # the same render through the ops layer, read back from its workspace
    arch = train_utils._arch_of(mc, train_utils._probe_encoder(epf, None), train_utils._probe_encoder(edf, None))
    blobs = [train_utils._packed(m, arch)[1] for m in (mc, mf)]
    opts = ops.make_opts(64, 128, False, False, False, 0.0)
    rays = ops.gen_rays(torch.eye(4), H, W, FOCAL, None, "cuda", ndc=True, near=0.0, far=1.0)
    with torch.no_grad():
        out_c, out_f, normals, ws = ops.render_fwd_normals(arch, arch, opts, blobs[0], blobs[1], rays, {}, impl=1,
                                                           ndc=_cam())
    assert bits_equal(normals, world[6].view(-1, 3)) and bits_equal(out_f[:, :3], world[3].view(-1, 3))
    n, s = rays.shape[0], 192
    lay = ops.render_workspace_layout(arch, arch, opts, n, False)
    f = ws.view(torch.float32)
    z = f[lay["z_fine"] // 4: lay["z_fine"] // 4 + n * s].view(n, s).clone()
    raw = f[lay["raw_fine"] // 4: lay["raw_fine"] // 4 + n * s * 4].view(n, s, 4).clone()
    _, w = ops.composite_fwd(raw, z, rays, None, 0.0, False)
    pts = rays[:, None, :3] + rays[:, None, 3:6] * z[..., None]
    live = w != 0
    with torch.no_grad():
        _, gq = nb.density_gradient(mf, epf, pts[live].contiguous())
    g = t_grad(pts[live], gq)
    ln = torch.sqrt((g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1]) + g[:, 2] * g[:, 2])
    unit = torch.where(ln[:, None] != 0, -(g / ln[:, None]), torch.zeros_like(g))
    terms = torch.zeros(n, s, 3, device="cuda")
    terms[live] = w[live][:, None] * unit
    N = torch.zeros(n, 3, device="cuda")
    for j in range(s):  # in sample order, fp32; skipped samples add +0
        N = N + terms[:, j]
    diff = (N - normals).abs().max().item()
    report("fern world normal map", "max |N - sum w n| (fp32 restatement)", f"{diff:.3e}, bit-identical "
                                                                          f"{bits_equal(N, normals)}")
    assert diff <= 1e-6
    # world normals differ from the NDC ones, and point toward the camera (+z) where the scene is opaque
    acc = out_f[:, 4]
    solid = acc > 0.5
    report("fern world normal map", "share of opaque rays with N_z > 0", f"{(normals[solid, 2] > 0).float().mean():.4f}")
    assert not bits_equal(world[6], ndc_n[6])
    assert (normals.norm(dim=-1) <= acc + 1e-5).all()


def test_world_normal_map_of_a_blender_render_is_normals_true():
    import nerf_pytorch_b200 as nb

    mc, mf, epf, edf = shipped_models("lego")
    opts = O.make_options(no_ndc=True, near=2.0, far=6.0, num_coarse=64, num_fine=128, perturb=True,
                          radiance_field_noise_std=0.2)
    kw = dict(mode="validation", encode_position_fn=epf, encode_direction_fn=edf, impl=1,
              randoms=nb.SeededRandoms(5, 2))
    pose = O.pose_spherical(30.0, -30.0, 4.0)
    with torch.no_grad():
        a = nb.render_image(48, 48, 66.7, pose, mc, mf, opts, normals=True, **kw)
        b = nb.render_image(48, 48, 66.7, pose, mc, mf, opts, normals="world", **kw)
    assert len(a) == len(b) == 7 and all(bits_equal(x, y) for x, y in zip(a, b))
