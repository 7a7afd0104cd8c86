"""CPU: the oracle reproduces the committed golden vectors (generated from the UNMODIFIED reference by
oracle/make_golden.py, which asserts bit equality at generation time).

Same torch build -> bit-exact; the tolerance below only absorbs a different CPU vector ISA on the
box that runs the tests (torch's sin/exp kernels are ISA-dispatched)."""
import numpy as np
import pytest
import torch

from helpers import CASES, Case, OUT_NAMES


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_outputs(name):
    torch.set_num_threads(1)
    c = Case(name)
    out, loss, _, _ = c.oracle()
    for n, got, want in zip(OUT_NAMES, out, c.outputs):
        assert (got is None) == (want is None), n
        if want is None:
            continue
        assert got.shape == want.shape, n
        assert torch.allclose(got, want, rtol=1e-4, atol=1e-5, equal_nan=True), (n, (got - want).abs().max())
    assert abs(loss.item() - c.loss) <= 1e-5 * max(1.0, abs(c.loss))


@pytest.mark.parametrize("name", ["lego_a0_train", "a1_skip_lindisp", "a0_noview_coarse_only"])
def test_oracle_matches_reference_gradients(name):
    torch.set_num_threads(1)
    c = Case(name)
    _, _, gc, gf = c.oracle(with_grad=True)
    for tag, grads in (("c", gc), ("f", gf)):
        if grads is None:
            continue
        dig = c.grad_digests(tag)
        assert set(dig) == set(grads), (sorted(dig), sorted(grads))
        for k, g in grads.items():
            f = g.double().flatten()
            got = np.array([f.sum().item(), f.abs().sum().item(), (f * f).sum().item()] + f[:5].tolist())
            want = dig[k]
            scale = max(1e-12, np.abs(want[1]))
            assert np.allclose(got[:3], want[:3], rtol=1e-3, atol=1e-6 * scale), (k, got[:3], want[:3])


def test_oracle_rng_order_matches_reference():
    """Seeded (non-injected) run draws t_rand -> noise_c -> u -> noise_f like the reference."""
    from oracle import nerf_oracle as O

    c = Case("lego_a0_train")
    torch.manual_seed(int(c.z["seed"]))
    out = O.run_one_iter_of_nerf(c.H, c.W, c.focal, c.sd_c, c.sd_f, c.ro, c.rd, c.options, mode=c.mode,
                                 enc_xyz=c.enc_xyz, enc_dir=c.enc_dir)
    assert torch.allclose(out[3], c.outputs[3], rtol=1e-4, atol=1e-5, equal_nan=True)


def test_tiny_nerf_oracle_matches_reference_outputs_and_gradients():
    """BASELINE.json configs[0] (tiny_nerf.py, CPU-only): oracle/tiny_oracle.py against the vectors the unmodified reference
    produced (oracle/make_golden_tiny.py asserted bit equality when it wrote them): image, loss and the six gradients."""
    import os

    from helpers import GOLD
    from oracle import tiny_oracle as T

    torch.set_num_threads(1)
    z = np.load(os.path.join(GOLD, "tiny_nerf.npz"))
    sd = {k[2:]: torch.from_numpy(z[k]).requires_grad_(True) for k in z.files if k.startswith("w.")}
    out = T.run_one_iter_of_tinynerf(int(z["H"]), int(z["W"]), float(z["focal"]), torch.from_numpy(z["pose"]), float(z["near"]),
                                     float(z["far"]), int(z["S"]), int(z["L"]), int(z["chunk"]), sd, rand=torch.from_numpy(z["rand"]))
    want = torch.from_numpy(z["rgb"])
    assert out.shape == want.shape == (32, 32, 3)      # 1024 rays, 64 samples each
    assert torch.allclose(out, want, rtol=1e-4, atol=1e-5), (out - want).abs().max()
    loss = torch.nn.functional.mse_loss(out, torch.from_numpy(z["target"]))
    assert abs(loss.item() - float(z["loss"])) <= 1e-5
    loss.backward()
    for k, p in sd.items():
        f = p.grad.double().flatten()
        got = np.array([f.sum().item(), f.abs().sum().item(), (f * f).sum().item()] + f[:5].tolist())
        assert np.allclose(got, z["g." + k], rtol=1e-3, atol=1e-7), (k, got, z["g." + k])
    # the jittered grid: depth = linspace + U[0,1) * (far - near) / S, NOT clamped to its cell (tiny_nerf.py:47-56)
    _, depth = T.compute_query_points_from_rays(torch.zeros(4, 3), torch.ones(4, 3), 2.0, 6.0, 64, rand=torch.ones(4, 64) * 0.999)
    assert depth.shape == (4, 64) and float(depth[0, 0]) > 2.0 and float(depth[0, -1]) > 6.0


@pytest.mark.parametrize("scene", ["chair", "drums", "fern", "hotdog", "lego", "materials", "ship"])
def test_pretrained_fixtures_load_with_a0_shapes(scene):
    """Every pretrained scene's coarse and fine state dicts load with the shapes of A0 (4 x 128, skip 4, 4 direction
    bands, 10 position bands or fern's 6), finite, into the oracle's functional forward and into FlexibleNeRFModel."""
    from helpers import PRETRAINED_SCENES, load_weights, pretrained_arch
    from oracle import nerf_oracle as O
    import nerf_pytorch_b200 as nb

    assert sorted(PRETRAINED_SCENES) == ["chair", "drums", "fern", "hotdog", "lego", "materials", "ship"]
    arch = pretrained_arch(scene)
    for sd in load_weights(f"{scene}_lowres"):
        want = O.init_flexible_nerf(4, 128, 4, arch.n_freq_xyz, 4)
        assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in want.items()}
        assert all(v.dtype == torch.float32 and bool(torch.isfinite(v).all()) for v in sd.values())
        assert O.arch_from_state_dict(sd, arch.dim_xyz, arch.dim_dir) == dict(num_layers=4, hidden=128, wide=[],
                                                                               use_viewdirs=True)
        m = nb.FlexibleNeRFModel(num_layers=4, hidden_size=128, skip_connect_every=4,
                                 num_encoding_fn_xyz=arch.n_freq_xyz, num_encoding_fn_dir=4)
        m.load_state_dict(sd)
