"""GPU: half-precision baked fields (nb.bake(dtype=torch.float16), BakedField.half / float; csrc/mlp_tc.cu
bake_tc_kernel<kH, __half>, csrc/baked.cu baked_render_kernel<__half> and baked_max_weight_kernel<__half>;
include/nerfb200.h "baked fields: half precision").

  1. the fp16 bake is the fp32 bake under the conversion rule, bit for bit (NaN as a class): lego A0, A1 and A2 at init,
     a coarse-only network without view directions, fern in NDC; 1 brick and a count that ends mid-tile, at first > 0;
     and nb.bake(dtype=torch.float16) against nb.bake().half();
  2. an fp16 field renders bit for bit like its widened fp32 copy: synthetic fields with and without view directions,
     non-cubic resolutions, several active fractions, saturated and +-inf corners, rays that miss the box and edge rays,
     white background, early_stop 0 and 1e-3, ray counts that are not a multiple of 4; render_baked of the lego and fern
     bakes at their test poses;
  3. the fp16 renders against helpers.baked_render64 of the widened field, at test_bake_gpu's bars;
  4. peak weights bit-equal to the widened field's, in one call and in chunks through out=; pruning at w > 0 and at
     transparency keeps the measuring rays' fp16 renders the same bits;
  5. quality on lego 256^3 at the 4 held-out 48 x 48 views: PSNR against the fp32 render, and against render_image
     within a bar of the fp32 field's;
  6. the trainer, the regulariser and a differentiable render refuse an fp16 field before any launch."""
import pytest
import torch

from helpers import (FERN_CAM, LEGO_CAM, OUT_ABS, baked_render64, bake_scene, bits_equal, edge_rays, psnr64,
                     random_rays, scene_options, scene_pose, camera_rays, sphere_poses, synthetic_field, targets)

pytestmark = pytest.mark.gpu


def report(what, ctx, value):
    print(f"[baked-half] {what} {ctx}: {value}")


def rule(x):
    """The header's conversion rule in torch."""
    return torch.where(x.isfinite(), x.clamp(-65504, 65504), x).half()


def half_bits_equal(a, b):
    """fp16 tensors of one shape with the same bits, NaN compared as a class."""
    if a.shape != b.shape or a.dtype != torch.float16 or b.dtype != torch.float16:
        return False
    na, nb_ = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb_) and torch.equal(a.view(torch.int16)[~na], b.view(torch.int16)[~nb_])


# ------------------------------------------------------------------------------------------------------------------------
# 1. the bake
# ------------------------------------------------------------------------------------------------------------------------
def _model(kind):
    """(model, encode_position_fn, encode_direction_fn or None, box): the shipped scenes' fine network, or "a1", "a2"
    and "noview" (coarse-only, no view directions) at torch's init under seed 7."""
    import nerf_pytorch_b200 as nb
    from helpers import FERN_BOX, LEGO_BOX, shipped_models

    if kind in ("lego", "fern"):
        _, m, epf, edf = shipped_models(kind)
        return m, epf, edf, LEGO_BOX if kind == "lego" else FERN_BOX
    torch.manual_seed(7)
    if kind == "a1":
        m = nb.FlexibleNeRFModel(num_layers=8, hidden_size=128, skip_connect_every=3, num_encoding_fn_xyz=10)
    elif kind == "a2":
        m = nb.FlexibleNeRFModel(num_layers=8, hidden_size=256, skip_connect_every=4, num_encoding_fn_xyz=10)
    else:
        m = nb.FlexibleNeRFModel(num_layers=4, hidden_size=128, skip_connect_every=4, num_encoding_fn_xyz=10,
                                 use_viewdirs=False)
    m = m.cuda()
    return m, nb.get_embedding_function(10), nb.get_embedding_function(4) if m.use_viewdirs else None, \
        ((-1.0,) * 3, (1.0,) * 3)


@pytest.mark.parametrize("count", [1, 3])
@pytest.mark.parametrize("kind", ["lego", "a1", "a2", "noview", "fern"])
def test_fp16_bake_is_the_fp32_bake_under_the_rule(kind, count):
    from nerf_pytorch_b200 import mesh, ops, train_utils
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    m, epf, edf, box = _model(kind)
    arch = mesh._network(m, epf, edf)
    blob = train_utils._packed(m, arch)[1]
    g = ops.grid_struct(box, (24, 24, 24))
    _, bricks, n = ops.mesh_sparse_bricks(g, OccupancyGrid.full(box, 8))
    n, first = int(n.item()), 5
    v32 = torch.full((n, 729, 32), float("nan"), device="cuda")
    v16 = torch.full((n, 729, 32), 7.0, dtype=torch.float16, device="cuda")
    ops.bake(arch, blob, g, bricks, first, count, v32)
    ops.bake(arch, blob, g, bricks, first, count, v16)
    s = slice(first, first + count)
    assert half_bits_equal(v16[s], rule(v32[s])), kind
    assert (v16[s][..., 28:].view(torch.int16) == 0).all()
    untouched = torch.ones(n, dtype=torch.bool, device="cuda")
    untouched[s] = False
    assert (v16[untouched] == 7.0).all()


@pytest.mark.parametrize("case", ["saturating", "non_finite"])
def test_fp16_bake_saturates_and_keeps_infinities_in_the_kernel(case):
    """The shipped lego network with its heads (fc_alpha, fc_rgb: fp32 in the bake) scaled so that sigma_raw, the
    logits and the SH coefficients pass 65504, and with +inf / -inf head biases so that values are +-inf and NaN: the
    fp16 bake is still the fp32 bake under the rule, bit for bit (NaN as a class), so the kernel's store saturates
    finite values and keeps the non-finite ones."""
    from nerf_pytorch_b200 import mesh, ops, train_utils
    from nerf_pytorch_b200.occupancy import OccupancyGrid

    m, epf, edf, box = _model("lego")
    with torch.no_grad():
        for head in (m.fc_alpha, m.fc_rgb):
            head.weight.mul_(3e5)
            head.bias.mul_(3e5)
        if case == "non_finite":
            m.fc_alpha.bias.fill_(float("inf"))
            m.fc_rgb.bias[1] = float("-inf")
    arch = mesh._network(m, epf, edf)
    blob = train_utils._packed(m, arch)[1]
    g = ops.grid_struct(box, (24, 24, 24))
    _, bricks, n = ops.mesh_sparse_bricks(g, OccupancyGrid.full(box, 8))
    n, first, count = int(n.item()), 2, 5
    v32 = torch.full((n, 729, 32), float("nan"), device="cuda")
    v16 = torch.full((n, 729, 32), 7.0, dtype=torch.float16, device="cuda")
    ops.bake(arch, blob, g, bricks, first, count, v32)
    ops.bake(arch, blob, g, bricks, first, count, v16)
    s = slice(first, first + count)
    x, y = v32[s][..., :28], v16[s][..., :28]
    big = x.isfinite() & (x.abs() > 65504)
    report("fp32 values beyond 65504 / +-inf / NaN", case,
           (int(big.sum()), int(x.isinf().sum()), int(x.isnan().sum())))
    assert bool(big.any()) and bool((y[big].abs() == 65504).all())
    if case == "non_finite":
        assert bool((x == float("inf")).any()) and bool((x == float("-inf")).any()) and bool(x.isnan().any())
    assert half_bits_equal(v16[s], rule(v32[s])), case
    assert not bool(y[x.isfinite()].isinf().any())


def test_nb_bake_fp16_is_bake_half():
    import nerf_pytorch_b200 as nb

    m, epf, edf, box = _model("lego")
    grid = nb.OccupancyGrid.from_models([m], epf, box, 32, encode_direction_fn=edf)
    f32 = nb.bake(m, epf, edf, bounds=box, resolution=40, grid=grid)
    f16 = nb.bake(m, epf, edf, bounds=box, resolution=40, grid=grid, dtype=torch.float16)
    assert f16.dtype == torch.float16 and f16.n_active == f32.n_active > 0
    assert bits_equal(f16.brick_map, f32.brick_map) and bits_equal(f16.bricks, f32.bricks)
    assert half_bits_equal(f16.values, f32.half().values)


# ------------------------------------------------------------------------------------------------------------------------
# 2-4. renders, fp64 and peak weights on synthetic fields
# ------------------------------------------------------------------------------------------------------------------------
FIELDS = {
    "res16": dict(res=(16, 16, 16), seed=1),
    "res24_20_28_half_noview": dict(res=(24, 20, 28), viewdirs=False, active=0.5, seed=2),
    "res13_9_17_third": dict(res=(13, 9, 17), active=0.3, seed=3),
    "saturated": dict(res=(16, 16, 16), sigma=(-1e5, 1e5), seed=4),
    "infinite": dict(res=(20, 17, 12), active=0.7, seed=5),
}


def _synthetic(name):
    kw = dict(FIELDS[name])
    f = synthetic_field(kw.pop("res"), **kw)
    g = torch.Generator(device="cuda").manual_seed(11)
    if name == "saturated":  # coefficients beyond the fp16 range too
        big = torch.rand(f.values.shape[:2], generator=g, device="cuda") < 0.05
        f.values[..., 1:28][big] *= 2e5
    if name == "infinite":  # +-inf sigma_raw and coefficients at a few stored points
        pick = torch.rand(f.values.shape[:2], generator=g, device="cuda")
        f.values[..., 0][pick < 0.002] = float("inf")
        f.values[..., 0][(pick >= 0.002) & (pick < 0.004)] = float("-inf")
        f.values[..., 5][(pick >= 0.004) & (pick < 0.005)] = float("inf")
    return f


def _rays(f, seed, n=1001):
    rays = torch.cat([random_rays(n, seed, f.use_viewdirs, misses=True), edge_rays(f, f.use_viewdirs)])
    assert rays.shape[0] % 4 != 0
    return rays


@pytest.mark.parametrize("name", list(FIELDS))
def test_fp16_renders_are_the_widened_fields_bit_for_bit(name):
    import nerf_pytorch_b200 as nb

    f = _synthetic(name)
    h = f.half()
    w = h.float()
    assert h.dtype == torch.float16 and w.dtype == torch.float32
    if name == "saturated":
        assert bool((h.values.abs() == 65504).any()) and not bool(h.values.isinf().any())
    if name == "infinite":
        assert bool((h.values == float("inf")).any()) and bool((h.values == float("-inf")).any())
    for n in (1001, 3):
        rays = _rays(f, 5, n)
        for white in (False, True):
            for stop in (None, 1e-3):
                with torch.no_grad():
                    a = nb.render_baked_rays(h, rays, white_background=white, early_stop=stop)
                    b = nb.render_baked_rays(w, rays, white_background=white, early_stop=stop)
                for x, y in zip(a, b):
                    assert bits_equal(x, y), (name, n, white, stop)


@pytest.mark.parametrize("name", ["res16", "res24_20_28_half_noview", "res13_9_17_third"])
def test_fp16_renders_match_fp64(name):
    from nerf_pytorch_b200 import ops

    h = _synthetic(name).half()
    rays = _rays(h, 6)
    for white in (False, True):
        out = ops.baked_render(h.box(), h.brick_map, h.values, h.use_viewdirs, rays, white)
        rgb, acc, depth, _ = baked_render64(h.float(), rays, white)
        far = float(rays[:, 7].max())
        e = ((out[:, :3].double() - rgb).abs().max().item(), (out[:, 4].double() - acc).abs().max().item(),
             (out[:, 5].double() - depth).abs().max().item() / far)
        report("rgb / acc / depth error against fp64", (name, white), e)
        assert max(e) <= OUT_ABS, (name, white, e)


@pytest.mark.parametrize("name", list(FIELDS))
def test_fp16_peak_weights_and_pruning(name):
    import nerf_pytorch_b200 as nb

    h = _synthetic(name).half()
    w = h.float()
    rays = _rays(h, 7)
    one = nb.baked_brick_weights_rays(h, rays)
    assert bits_equal(one, nb.baked_brick_weights_rays(w, rays))
    acc = torch.zeros(h.n_active, device="cuda")
    for c in range(0, rays.shape[0], 333):
        nb.baked_brick_weights_rays(h, rays[c:c + 333], out=acc)
    assert bits_equal(acc, one)
    with torch.no_grad():
        base = nb.render_baked_rays(h, rays)
        keeps = {"w>0": one > 0}
        if name != "infinite":  # the transparency rule holds for finite fields
            keeps["transparent"] = ~nb.baked_transparent_bricks(h)
        for k, keep in keeps.items():
            p = nb.prune_baked(h, keep)
            assert p.dtype == torch.float16
            report("bricks kept", (name, k), (p.n_active, h.n_active))
            for x, y in zip(nb.render_baked_rays(p, rays), base):
                assert bits_equal(x, y), (name, k)


# ------------------------------------------------------------------------------------------------------------------------
# 2-3 on the scenes' bakes
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["lego", "fern"])
def test_scene_bakes_render_bit_for_bit_and_match_fp64(kind):
    import nerf_pytorch_b200 as nb

    f = bake_scene(kind, 64, 64)
    h = f.half()
    w = h.float()
    H, W, focal = LEGO_CAM if kind == "lego" else FERN_CAM
    pose = scene_pose("spherical" if kind == "lego" else "eye")
    opts = scene_options(kind)
    for stop in (None, 1e-3):
        a = nb.render_baked(h, H, W, focal, pose, opts, early_stop=stop)
        b = nb.render_baked(w, H, W, focal, pose, opts, early_stop=stop)
        for x, y in zip(a, b):
            assert bits_equal(x, y), (kind, stop)
    rays = camera_rays(kind, pose)
    with torch.no_grad():
        rgb32 = nb.render_baked_rays(h, rays)
    rgb, acc, depth, _ = baked_render64(w, rays, False)
    e = (rgb32[0].double() - rgb).abs().max().item()
    report("rgb error against fp64", kind, e)
    assert e <= OUT_ABS
    report("PSNR fp16 vs fp32 field at 64^3", kind, psnr64(nb.render_baked(h, H, W, focal, pose, opts)[0],
                                                           nb.render_baked(f, H, W, focal, pose, opts)[0]))


# ------------------------------------------------------------------------------------------------------------------------
# 5. quality
# ------------------------------------------------------------------------------------------------------------------------
HELD = (5, 16, 27, 38)  # the held-out views of tools/baked_finetune_time.py
# mean PSNR (dB) over HELD on lego 256^3 (grid of both networks, 128^3), measured on an H100 80GB HBM3 at 700 W (DESIGN
# §4): the fp16 render against the fp32 render 100.91 dB; against render_image 29.712117 dB for the fp16 field and
# 29.712124 dB for the fp32 one (a loss of 6e-6 dB).  The bars sit a few dB and a few hundredths of a dB below.
PSNR_F16_VS_F32_BAR = 97.0
PSNR_LOSS_BAR = 0.02


def test_quality_on_lego_256():
    import nerf_pytorch_b200 as nb

    poses = sphere_poses(44)[list(HELD)]
    imgs, _ = targets("lego", poses)
    f = bake_scene("lego", 256, 128, grid_from="both")
    h = f.half()
    H, W, focal = LEGO_CAM
    vs32, ref16, ref32 = [], [], []
    with torch.no_grad():
        for p, im in zip(poses, imgs):
            rays = camera_rays("lego", p)
            a, b = nb.render_baked_rays(h, rays)[0], nb.render_baked_rays(f, rays)[0]
            vs32.append(psnr64(a, b))
            ref16.append(psnr64(a, im.reshape(-1, 3)))
            ref32.append(psnr64(b, im.reshape(-1, 3)))
    vs32, ref16, ref32 = (sum(x) / len(x) for x in (vs32, ref16, ref32))
    report("PSNR fp16 vs fp32 / fp16 vs render_image / fp32 vs render_image", f.n_active, (vs32, ref16, ref32))
    assert vs32 >= PSNR_F16_VS_F32_BAR
    assert ref16 >= ref32 - PSNR_LOSS_BAR


# ------------------------------------------------------------------------------------------------------------------------
# 6. refusals
# ------------------------------------------------------------------------------------------------------------------------
def test_fine_tuning_paths_refuse_an_fp16_field_before_any_launch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    h = synthetic_field((16, 16, 16), seed=8).half()
    imgs = torch.zeros(2, 8, 8, 3, device="cuda")
    poses = torch.eye(4, device="cuda").expand(2, 4, 4).contiguous()
    opts = scene_options("lego")
    rays = random_rays(8, 1)
    torch.cuda.synchronize()
    before, mem = ops.launch_count(), torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match=r"float\(\)"):
        nb.BakedFieldTrainer(h, imgs, poses, 10.0, opts)
    with pytest.raises(ValueError, match=r"float\(\)"):
        nb.baked_regularizer(h, tv_sigma=1.0)
    h.values.requires_grad_(True)
    with pytest.raises(ValueError, match="no gradient"):
        nb.render_baked_rays(h, rays)
    with torch.no_grad(), pytest.raises(ValueError, match="no gradient"):
        nb.render_baked_rays(h, rays)
    h.values.requires_grad_(False)
    with pytest.raises(ValueError, match="no gradient"):  # grad mode: the refusal fp16 fields met before this change
        nb.render_baked_rays(h, rays)
    assert ops.launch_count() == before and torch.cuda.memory_allocated() == mem
