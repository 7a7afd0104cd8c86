"""GPU: 8-bit baked fields (BakedField.quantize / float; csrc/baked.cu baked_render_kernel<uint8_t>,
baked_max_weight_kernel<uint8_t>, baked_mesh_dirs_kernel<uint8_t> and baked_mesh_colors_kernel<uint8_t>;
include/nerfb200.h "baked fields: 8-bit values").

  0. BakedField.quantize on a CUDA field gives the codes and dequant bits of the same field quantised on the CPU and of a
     numpy restatement of the rule (synthetic fields, lego and fern bakes, an fp16 bake), and float() agrees;
  1. an 8-bit field renders bit for bit like its dequantised fp32 field: synthetic fields with and without view
     directions, non-cubic resolutions, several active fractions, rays that miss the box and edge rays, white
     background, early_stop 0 and 1e-3, ray counts that are not a multiple of 4; render_baked of the lego, fern and
     no-view-direction bakes (quantised from fp16, as a user ships them) at their test poses;
  2. the 8-bit renders against helpers.baked_render64 of the dequantised field, at test_bake_gpu's bars;
  3. peak weights bit-equal to the dequantised field's, in one call, in chunks through out= and over whole views; pruning at w > 0 and
     at transparency keeps the measuring rays' renders the same bits;
  4. meshes (faces, vertices, normals, colours, and in NDC) bit-equal to the dequantised field's;
  5. quality on lego 256^3 at the 4 held-out 48 x 48 views of the fp16 quality test;
  6. the trainer, the regulariser, subdivision and a differentiable render refuse an 8-bit field before any launch."""
import numpy as np
import pytest
import torch

from helpers import (FERN_CAM, LEGO_CAM, OUT_ABS, baked_render64, bake_scene, bits_equal, camera_rays, edge_rays, psnr64,
                     random_rays, scene_options, scene_pose, sphere_poses, synthetic_field, targets)

pytestmark = pytest.mark.gpu


def report(what, ctx, value):
    print(f"[baked-u8] {what} {ctx}: {value}")


FIELDS = {
    "res16": dict(res=(16, 16, 16), seed=1),
    "res24_20_28_half_noview": dict(res=(24, 20, 28), viewdirs=False, active=0.5, seed=2),
    "res13_9_17_third": dict(res=(13, 9, 17), active=0.3, seed=3),
    "wide_sigma": dict(res=(20, 17, 12), sigma=(-300.0, 900.0), active=0.7, seed=4),
}


def _synthetic(name):
    kw = dict(FIELDS[name])
    return synthetic_field(kw.pop("res"), **kw)


def _rays(f, seed, n=1001):
    rays = torch.cat([random_rays(n, seed, f.use_viewdirs, misses=True), edge_rays(f, f.use_viewdirs)])
    assert rays.shape[0] % 4 != 0
    return rays


def _rule_numpy(v):
    """(codes uint8 [.., 32], scale [28], offset [28]) of fp32 values ``v`` (a CPU tensor): the header's rule restated in
    numpy fp32, every division correctly rounded."""
    x = v.numpy().astype(np.float32)
    flat = x[..., :28].reshape(-1, 28)
    lo = np.minimum(np.float32(0), flat.min(0))
    hi = np.maximum(np.float32(0), flat.max(0))
    s = (hi - lo) / np.float32(255)
    s = np.where(s == 0, np.float32(1), s).astype(np.float32)
    z = np.clip(np.rint(-lo / s), 0, 255).astype(np.float32)
    z = np.where(z == 0, np.float32(0), z)  # the integer 0 as +0
    o = -(z * s)
    q = np.zeros(x.shape, dtype=np.uint8)
    q[..., :28] = np.clip(np.rint((x[..., :28] - o) / s), 0, 255).astype(np.uint8)
    return q, s, o


def _on_cpu(f):
    import nerf_pytorch_b200 as nb

    return nb.BakedField(f.bounds, f.resolution, f.brick_map.cpu(), f.bricks.cpu(), f.values.cpu(), f.use_viewdirs)


# ------------------------------------------------------------------------------------------------------------------------
# 0. quantize() on the GPU is the rule: the same codes and dequant bits as on the CPU and as numpy
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(FIELDS) + ["lego_bake", "lego_bake_fp16", "fern_bake"])
def test_cuda_quantize_is_the_rule(name):
    if name in FIELDS:
        f = _synthetic(name)
    else:
        f = bake_scene(name.split("_")[0], 96, 64)
        if name.endswith("fp16"):
            f = f.half()
    q = f.quantize(chunk=7)
    c = _on_cpu(f).quantize()
    assert q.values.is_cuda and q.dequant.is_cuda
    assert torch.equal(q.dequant.cpu().view(torch.int32), c.dequant.view(torch.int32)), name
    assert torch.equal(q.values.cpu(), c.values), name
    codes, s, o = _rule_numpy(f.values.cpu().float())
    assert np.array_equal(q.dequant[0].cpu().numpy().view(np.int32), s.view(np.int32)), name
    assert np.array_equal(q.dequant[1].cpu().numpy().view(np.int32), o.view(np.int32)), name
    assert np.array_equal(q.values.cpu().numpy(), codes), name
    # and float() on the GPU is the CPU's dequantisation
    assert torch.equal(q.float().values.cpu().view(torch.int32), c.float().values.view(torch.int32)), name


# ------------------------------------------------------------------------------------------------------------------------
# 1-3 on synthetic fields
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(FIELDS))
def test_renders_are_the_dequantised_fields_bit_for_bit(name):
    import nerf_pytorch_b200 as nb

    q = _synthetic(name).quantize()
    w = q.float()
    assert q.dtype == torch.uint8 and w.dtype == torch.float32 and q.dequant.is_cuda
    for n in (1001, 3):
        rays = _rays(q, 5, n)
        for white in (False, True):
            for stop in (None, 1e-3):
                with torch.no_grad():
                    a = nb.render_baked_rays(q, rays, white_background=white, early_stop=stop)
                    b = nb.render_baked_rays(w, rays, white_background=white, early_stop=stop)
                for x, y in zip(a, b):
                    assert bits_equal(x, y), (name, n, white, stop)


@pytest.mark.parametrize("name", list(FIELDS))
def test_renders_match_fp64(name):
    from nerf_pytorch_b200 import ops

    q = _synthetic(name).quantize()
    rays = _rays(q, 6)
    for white in (False, True):
        out = ops.baked_render(q.box(), q.brick_map, q.values, q.use_viewdirs, rays, white, dequant=q.dequant)
        rgb, acc, depth, _ = baked_render64(q.float(), rays, white)
        far = float(rays[:, 7].max())
        e = ((out[:, :3].double() - rgb).abs().max().item(), (out[:, 4].double() - acc).abs().max().item(),
             (out[:, 5].double() - depth).abs().max().item() / far)
        report("rgb / acc / depth error against fp64", (name, white), e)
        assert max(e) <= OUT_ABS, (name, white, e)


@pytest.mark.parametrize("name", list(FIELDS))
def test_peak_weights_and_pruning(name):
    import nerf_pytorch_b200 as nb

    q = _synthetic(name).quantize()
    w = q.float()
    rays = _rays(q, 7)
    one = nb.baked_brick_weights_rays(q, rays)
    assert bits_equal(one, nb.baked_brick_weights_rays(w, rays))
    acc = torch.zeros(q.n_active, device="cuda")
    for c in range(0, rays.shape[0], 333):
        nb.baked_brick_weights_rays(q, rays[c:c + 333], out=acc)
    assert bits_equal(acc, one)
    with torch.no_grad():
        base = nb.render_baked_rays(q, rays)
        for k, keep in {"w>0": one > 0, "transparent": ~nb.baked_transparent_bricks(q)}.items():
            p = nb.prune_baked(q, keep)
            assert p.dtype == torch.uint8 and p.dequant is q.dequant
            report("bricks kept", (name, k), (p.n_active, q.n_active))
            for x, y in zip(nb.render_baked_rays(p, rays), base):
                assert bits_equal(x, y), (name, k)
    assert torch.equal(nb.baked_transparent_bricks(q), nb.baked_transparent_bricks(w))


# ------------------------------------------------------------------------------------------------------------------------
# 1-3 on the scenes' bakes
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["lego", "fern", "noview"])
def test_scene_bakes_render_bit_for_bit_and_match_fp64(kind):
    import nerf_pytorch_b200 as nb

    f = bake_scene(kind, 64, 64)
    q = f.half().quantize()  # the shipping path: an fp16 bake quantised
    assert torch.equal(q.values, f.half().float().quantize().values)
    w = q.float()
    H, W, focal = FERN_CAM if kind == "fern" else LEGO_CAM
    pose = scene_pose("eye" if kind == "fern" else "spherical")
    opts = scene_options("fern" if kind == "fern" else "lego")
    opts.nerf.use_viewdirs = f.use_viewdirs
    for stop in (None, 1e-3):
        a = nb.render_baked(q, H, W, focal, pose, opts, early_stop=stop)
        b = nb.render_baked(w, H, W, focal, pose, opts, early_stop=stop)
        for x, y in zip(a, b):
            assert bits_equal(x, y), (kind, stop)
    rays = camera_rays("fern" if kind == "fern" else "lego", pose, viewdirs=f.use_viewdirs)
    with torch.no_grad():
        out = nb.render_baked_rays(q, rays)
    rgb, acc, depth, _ = baked_render64(w, rays, False)
    e = (out[0].double() - rgb).abs().max().item()
    report("rgb error against fp64", kind, e)
    assert e <= OUT_ABS
    report("PSNR 8-bit vs fp32 field at 64^3", kind, psnr64(a[0], nb.render_baked(f, H, W, focal, pose, opts)[0]))
    # peak weights over whole views (the pose form), bit-equal to the dequantised field's
    shifted = pose.clone()
    shifted[:3, 3] += 0.05
    poses = torch.stack([pose, shifted])
    pw = nb.baked_brick_weights(q, poses, H, W, focal, opts)
    assert bool((pw > 0).any()) and bits_equal(pw, nb.baked_brick_weights(w, poses, H, W, focal, opts)), kind


# ------------------------------------------------------------------------------------------------------------------------
# 4. meshes
# ------------------------------------------------------------------------------------------------------------------------
def _level(field):
    """The median of the field's positive sigma_raw: a level with plenty of crossings."""
    s = field.float().values[..., 0]
    return float(s[s > 0].median())


def _meshes_equal(a, b):
    return all(bits_equal(x, y) for x, y in ((a.vertices, b.vertices), (a.faces, b.faces), (a.colors, b.colors),
                                             (a.normals, b.normals)))


def test_meshes_are_the_dequantised_fields_meshes():
    import nerf_pytorch_b200 as nb

    fields = {"lego128": bake_scene("lego", 128, 64).half().quantize(),
              "synthetic": synthetic_field((24, 20, 17), active=0.6, seed=9).quantize(),
              "noview": synthetic_field((16, 16, 16), viewdirs=False, seed=10).quantize()}
    for name, q in fields.items():
        level = _level(q)
        w = q.float()
        for colors, normals in ((True, True), (True, False), (False, True), (False, False)):
            a = nb.extract_baked_mesh(q, level, colors=colors, normals=normals)
            b = nb.extract_baked_mesh(w, level, colors=colors, normals=normals)
            assert a.vertices.shape[0] > 0 and _meshes_equal(a, b), (name, colors, normals)
        report("mesh vertices / faces", name, (a.vertices.shape[0], a.faces.shape[0]))
        # a transparent prune keeps the faces and vertices
        p = nb.prune_baked(q, ~nb.baked_transparent_bricks(q))
        m, n = nb.extract_baked_mesh(p, level), nb.extract_baked_mesh(q, level)
        assert bits_equal(m.vertices, n.vertices) and bits_equal(m.faces, n.faces), name


def test_ndc_mesh_is_the_dequantised_fields_mesh():
    import nerf_pytorch_b200 as nb

    q = bake_scene("fern", 96, 64).half().quantize()
    level = _level(q)
    a = nb.extract_baked_mesh(q, level, colors=True, normals=True, ndc=FERN_CAM)
    b = nb.extract_baked_mesh(q.float(), level, colors=True, normals=True, ndc=FERN_CAM)
    assert a.vertices.shape[0] > 0 and _meshes_equal(a, b)


# ------------------------------------------------------------------------------------------------------------------------
# 5. quality
# ------------------------------------------------------------------------------------------------------------------------
HELD = (5, 16, 27, 38)  # the held-out views of tools/baked_finetune_time.py and of the fp16 quality test
# mean PSNR (dB) over HELD on lego 256^3 (grid of both networks, 128^3), measured on an H100 80GB HBM3 at 700 W (DESIGN
# §4): the 8-bit render against the fp32 render 19.04 dB; against render_image 18.62 dB for the 8-bit field and
# 29.71 dB for the fp32 one (a loss of 11.1 dB).  One linear range per channel spans the whole field, and empty space
# stores sigma_raw and coefficients in the thousands (scales 38.4 and 23.2 for sigma_raw and coefficient 0), so a step
# of the code is wider than the densities and logits that shape the surface.  The bars sit a little below.
PSNR_U8_VS_F32_BAR = 18.5
PSNR_LOSS_BAR = 11.6


def test_quality_on_lego_256():
    import nerf_pytorch_b200 as nb

    poses = sphere_poses(44)[list(HELD)]
    imgs, _ = targets("lego", poses)
    f = bake_scene("lego", 256, 128, grid_from="both")
    q = f.quantize()
    vs32, ref8, ref32 = [], [], []
    with torch.no_grad():
        for p, im in zip(poses, imgs):
            rays = camera_rays("lego", p)
            a, b = nb.render_baked_rays(q, rays)[0], nb.render_baked_rays(f, rays)[0]
            vs32.append(psnr64(a, b))
            ref8.append(psnr64(a, im.reshape(-1, 3)))
            ref32.append(psnr64(b, im.reshape(-1, 3)))
    vs32, ref8, ref32 = (sum(x) / len(x) for x in (vs32, ref8, ref32))
    report("PSNR 8-bit vs fp32 / 8-bit vs render_image / fp32 vs render_image", f.n_active, (vs32, ref8, ref32))
    report("scales of sigma_raw and the first coefficient", "", q.dequant[0, :2].tolist())
    assert vs32 >= PSNR_U8_VS_F32_BAR
    assert ref8 >= ref32 - PSNR_LOSS_BAR


# ------------------------------------------------------------------------------------------------------------------------
# 6. refusals
# ------------------------------------------------------------------------------------------------------------------------
def test_fine_tuning_paths_refuse_an_8bit_field_before_any_launch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    q = synthetic_field((16, 16, 16), seed=8).quantize()
    imgs = torch.zeros(2, 8, 8, 3, device="cuda")
    poses = torch.eye(4, device="cuda").expand(2, 4, 4).contiguous()
    opts = scene_options("lego")
    rays = random_rays(8, 1)
    torch.cuda.synchronize()
    before, mem = ops.launch_count(), torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match=r"float\(\)"):
        nb.BakedFieldTrainer(q, imgs, poses, 10.0, opts)
    with pytest.raises(ValueError, match=r"float\(\)"):
        nb.baked_regularizer(q, tv_sigma=1.0)
    with pytest.raises(ValueError, match=r"float\(\)"):
        nb.subdivide_baked(q)
    with pytest.raises(ValueError, match="no gradient"):  # grad mode
        nb.render_baked_rays(q, rays)
    with pytest.raises(ValueError, match=r"float\(\)"):
        q.half()
    with pytest.raises(ValueError, match=r"float\(\)"):
        q.quantize()
    bad = nb.BakedField(q.bounds, q.resolution, q.brick_map, q.bricks, q.values, q.use_viewdirs)  # no dequant
    with torch.no_grad(), pytest.raises(ValueError, match="dequant"):
        nb.render_baked_rays(bad, rays)
    assert ops.launch_count() == before and torch.cuda.memory_allocated() == mem
