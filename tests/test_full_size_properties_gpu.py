"""GPU: BASELINE.json's full-size configurations through size-independent properties (the oracle is too slow at
these sizes): sortedness / containment of the merged depths, compositing invariants, bit-determinism, ray-chunk
invariance, agreement of the two kernel families (fp32 CUDA cores vs wgmma split precision) forward and backward."""
import math

import pytest
import torch

from helpers import load_weights
from oracle import nerf_oracle as O

pytestmark = pytest.mark.gpu


def _setup(n_rays, H=400, W=400, focal=555.5555, L_xyz=10, ndc=False, arch=(4, 128, 4), weights="lego", seed=0, **opt):
    import nerf_pytorch_b200 as nb

    torch.manual_seed(seed)
    if ndc:
        pose = torch.eye(4)
    else:
        pose = O.pose_spherical(30.0, -30.0, 4.0)
    ro, rd = O.get_ray_bundle(H, W, focal, pose)
    idx = torch.randperm(H * W)[:n_rays]
    ro, rd = ro.reshape(-1, 3)[idx].cuda().contiguous(), rd.reshape(-1, 3)[idx].cuda().contiguous()
    mk = lambda: nb.FlexibleNeRFModel(num_layers=arch[0], hidden_size=arch[1], skip_connect_every=arch[2],
                                      num_encoding_fn_xyz=L_xyz, num_encoding_fn_dir=4).cuda()
    mc, mf = mk(), mk()
    if weights:
        sd_c, sd_f = load_weights(weights + "_lowres")
        mc.load_state_dict(sd_c); mf.load_state_dict(sd_f)
    options = O.make_options(no_ndc=not ndc, **opt)
    epf, edf = nb.get_embedding_function(L_xyz), nb.get_embedding_function(4)
    return nb, mc, mf, ro, rd, options, epf, edf, (H, W, focal)


def _randoms(n, nc, nf, seed=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return dict(t_rand=torch.rand(n, nc, device="cuda", generator=g), noise_c=torch.randn(n, nc, device="cuda", generator=g),
                u=torch.rand(n, nf, device="cuda", generator=g), noise_f=torch.randn(n, nc + nf, device="cuda", generator=g))


@pytest.mark.parametrize("n_rays,res", [(4096, 400), (8192, 800)])   # BASELINE configs 2 and 3
def test_lego_full_size_invariants_determinism_and_chunking(n_rays, res):
    nb, mc, mf, ro, rd, options, epf, edf, (H, W, f) = _setup(
        n_rays, H=res, W=res, focal=555.5555 * res / 400, num_coarse=64, num_fine=128, perturb=True,
        radiance_field_noise_std=0.2, near=2.0, far=6.0)
    rnd = _randoms(n_rays, 64, 128)
    run = lambda **kw: nb.run_one_iter_of_nerf(H, W, f, mc, mf, ro, rd, options, encode_position_fn=epf,
                                               encode_direction_fn=edf, **kw)
    with torch.no_grad():
        a = run(randoms=rnd)
        b = run(randoms=rnd)
        for x, y in zip(a, b):   # bit-deterministic
            assert torch.equal(torch.nan_to_num(x, nan=-1.0), torch.nan_to_num(y, nan=-1.0))
        rgb_c, disp_c, acc_c, rgb_f, disp_f, acc_f = a
        assert rgb_f.shape == (n_rays, 3) and acc_f.shape == (n_rays,)
        for rgb, acc in ((rgb_c, acc_c), (rgb_f, acc_f)):
            assert torch.isfinite(rgb).all() and torch.isfinite(acc).all()
            assert (acc >= 0).all() and (acc <= 1 + 1e-4).all()          # weights are a sub-probability measure
            assert (rgb >= -1e-6).all() and (rgb <= 1 + 1e-4).all()      # convex combination of sigmoids
        ok = ~torch.isnan(disp_f)
        assert (disp_f[ok] > 0).all()
        # ray-chunk invariance: rays are independent, so two chunks of half the rays give the same rows bit for bit
        h = n_rays // 2
        first = nb.run_one_iter_of_nerf(H, W, f, mc, mf, ro[:h], rd[:h], options, encode_position_fn=epf,
                                        encode_direction_fn=edf, randoms={k: v[:h].contiguous() for k, v in rnd.items()})
        assert torch.equal(torch.nan_to_num(first[3], nan=-1.0), torch.nan_to_num(rgb_f[:h], nan=-1.0))


def test_merged_depths_sorted_and_contain_coarse_at_full_size():
    from nerf_pytorch_b200 import ops

    n, nc, nf = 4096, 64, 128
    g = torch.Generator(device="cuda").manual_seed(3)
    zc = torch.sort(torch.rand(n, nc, device="cuda", generator=g) * 4 + 2, -1).values.contiguous()
    w = torch.rand(n, nc, device="cuda", generator=g) ** 8
    u = torch.rand(n, nf, device="cuda", generator=g)
    z_fine, zs, inds, cdf = ops.sample_pdf_merge(zc, w.contiguous(), u, nf, want_aux=True)
    assert (z_fine[:, 1:] >= z_fine[:, :-1]).all()
    assert (inds >= 1).all() and (inds <= nc - 1).all()                 # searchsorted(right) on a cdf starting at 0
    assert (cdf[:, 1:] >= cdf[:, :-1]).all() and (cdf[:, 0] == 0).all() and (cdf[:, -1] - 1).abs().max() < 1e-5
    mids = 0.5 * (zc[:, 1:] + zc[:, :-1])
    assert (zs >= mids[:, :1] - 1e-6).all() and (zs <= mids[:, -1:] + 1e-6).all()
    # multiset identity: sort(cat(z_coarse, z_samples)) == z_fine
    ref = torch.sort(torch.cat([zc, zs], -1), -1).values
    assert torch.equal(ref, z_fine)


def test_fern_ndc_full_size_runs_and_kernel_families_agree():            # BASELINE config 4
    nb, mc, mf, ro, rd, options, epf, edf, (H, W, f) = _setup(
        4096, H=378, W=504, focal=407.5658, L_xyz=6, ndc=True, weights="fern", num_coarse=64, num_fine=128,
        perturb=True, radiance_field_noise_std=1.0, near=0.0, far=1.0)
    rnd = _randoms(4096, 64, 128, seed=5)
    with torch.no_grad():
        o0 = nb.run_one_iter_of_nerf(H, W, f, mc, mf, ro, rd, options, encode_position_fn=epf, encode_direction_fn=edf,
                                     randoms=rnd, impl=0)
        o1 = nb.run_one_iter_of_nerf(H, W, f, mc, mf, ro, rd, options, encode_position_fn=epf, encode_direction_fn=edf,
                                     randoms=rnd, impl=1)
    for k in (0, 2, 3, 5):
        assert torch.isfinite(o0[k]).all()
        close = torch.isclose(o1[k], o0[k], rtol=1e-4, atol=2e-5).float().mean().item()
        assert close > 0.97, (k, close)


def test_kernel_families_agree_on_gradients_at_full_size():
    """One train step at the bench size (A1 = config/lego.yml as written): wgmma vs fp32 kernels."""
    nb, mc, mf, ro, rd, options, epf, edf, (H, W, f) = _setup(
        4096, arch=(8, 128, 3), weights=None, num_coarse=64, num_fine=128, perturb=True, radiance_field_noise_std=0.2)
    rnd = _randoms(4096, 64, 128, seed=9)
    tgt = torch.rand(4096, 3, device="cuda")
    grads = []
    for impl in (0, 1):
        mc.zero_grad(); mf.zero_grad()
        out = nb.run_one_iter_of_nerf(H, W, f, mc, mf, ro, rd, options, encode_position_fn=epf, encode_direction_fn=edf,
                                      randoms=rnd, impl=impl)
        loss = torch.nn.functional.mse_loss(out[0], tgt) + torch.nn.functional.mse_loss(out[3], tgt)
        loss.backward()
        grads.append((loss.item(), torch.cat([p.grad.reshape(-1) for p in list(mc.parameters()) + list(mf.parameters())])))
    assert abs(grads[0][0] - grads[1][0]) < 1e-5 * abs(grads[0][0]) + 1e-7
    rel = ((grads[0][1] - grads[1][1]).norm() / grads[0][1].norm()).item()
    assert rel < 2e-3, rel


def test_config5_sized_batch_single_gpu():
    """32768 rays (the 8-GPU global batch of BASELINE config 5) in one call on one GPU: chunked by chunksize."""
    nb, mc, mf, ro, rd, options, epf, edf, (H, W, f) = _setup(
        32768, H=800, W=800, focal=1111.111, num_coarse=64, num_fine=128, perturb=True, radiance_field_noise_std=0.2,
        chunksize=8192)
    with torch.no_grad():
        out = nb.run_one_iter_of_nerf(H, W, f, mc, mf, ro, rd, options, encode_position_fn=epf, encode_direction_fn=edf)
    assert out[3].shape == (32768, 3) and torch.isfinite(out[3]).all()
