"""CPU (no GPU needed): the C-ABI library loads and exports every symbol include/nerfb200.h declares,
its host-side planning functions answer correctly, and the Python host logic (encoder probing,
model introspection, sharding) behaves.  No compute kernels are launched here."""
import ctypes as C
import math
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_and_binding_match_the_v101_header():
    from nerf_pytorch_b200 import _lib

    hdr = open(os.path.join(ROOT, "include", "nerfb200.h")).read()
    declared = sorted(set(re.findall(r"\b(nerfb200_[a-z0-9_]+)\s*\(", hdr)))
    assert len(declared) >= 20
    lib = C.CDLL(_lib.LIB_PATH)
    missing = [n for n in declared if not hasattr(lib, n)]
    assert not missing, missing
    # and the ctypes table binds exactly the declared set
    assert sorted(_lib.SIGNATURES) == declared
    assert _lib.load().nerfb200_version() == 101


def test_flat_layout_matches_reference_state_dict_shapes():
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    for kw, n_params in ((dict(num_layers=4, hidden=128, skip_every=4), 84548),
                         (dict(num_layers=8, hidden=128, skip_every=3), 166724),
                         (dict(num_layers=8, hidden=256, skip_every=4), 595844)):   # SURVEY.md section 0.1 / 6
        arch = ops.ArchSpec(n_freq_xyz=10, n_freq_dir=4, **kw)
        assert arch.flat_param_count() == n_params
        sd = O.init_flexible_nerf(kw["num_layers"], kw["hidden"], kw["skip_every"], 10, 4)
        off = 0
        for name, w_off, b_off, fin, fout in arch.flat_layout():
            assert tuple(sd[name + ".weight"].shape) == (fout, fin), name
            assert w_off == off and b_off == off + fin * fout
            off = b_off + fout
        assert off == n_params
        assert set(n + s for n in arch.slot_names() for s in (".weight", ".bias")) == set(sd)


def test_tc_gradient_blocks_partition_the_flat_gradient():
    """The blocks the wgmma architecture sweep compares one by one (tests/mlp_checks.py, tc_blocks) cover
    every element of every swept architecture's flat gradient exactly once, so no element goes unchecked; the xyz-
    encoding blocks sit on layer1 and the wide layers the skip rule allocates, and the direction-encoding block has the
    width of the direction encoding (at most 28 columns in the fused backward)."""
    import re

    from nerf_pytorch_b200 import ops
    from mlp_checks import ALL_ARCHS, TC_ARCHS, as_state_dict, block, spec, tc_blocks

    for name in ALL_ARCHS:
        arch = spec(name)
        assert ops.impl_supported(arch, 15, ops.IMPL_TC) == (name in TC_ARCHS), name
        hits = torch.zeros(arch.flat_param_count(), dtype=torch.int32)
        sd = as_state_dict(arch, hits)
        blocks = tc_blocks(arch)
        for _, key, rows, cols, _ in blocks:
            block(sd[key], rows, cols).add_(1)
        assert (hits == 1).all(), (name, int((hits == 0).sum()), int((hits > 1).sum()))
        wide = {f"layers_xyz.{i}" for i in range(arch.num_layers - 1) if i % arch.skip_every == 0 and i > 0}
        enc = {re.sub(r"\.weight.*", "", b[0]) for b in blocks if "xyz enc" in b[0]}
        assert enc == {"layer1"} | wide, name
        dirs = [b for b in blocks if "dir enc" in b[0]]
        if arch.use_viewdirs:
            assert len(dirs) == 1 and sd[dirs[0][1]][dirs[0][2], dirs[0][3]].shape == (64, arch.dim_dir), name
            assert arch.dim_dir <= 28 or name not in TC_ARCHS, name
        else:
            assert not dirs, name


def test_unsupported_architectures_are_rejected_not_approximated():
    from nerf_pytorch_b200 import ops

    with pytest.raises(NotImplementedError):
        ops.ArchSpec(hidden=96).flat_param_count()
    with pytest.raises(NotImplementedError):
        ops.ArchSpec(num_layers=40).blob_floats()
    with pytest.raises(NotImplementedError):
        ops.ArchSpec(n_freq_xyz=17).c_struct()


def test_frequency_bands_follow_reference():
    from nerf_pytorch_b200 import ops

    assert ops.frequency_bands(10, True).tolist() == [2.0 ** i for i in range(10)]
    assert torch.equal(ops.frequency_bands(5, False), torch.linspace(1.0, 16.0, 5))


def test_encoder_probe_identifies_reference_lambdas():
    from nerf_pytorch_b200 import train_utils
    from nerf_pytorch_b200.nerf_helpers import get_embedding_function
    from oracle import nerf_oracle as O

    for L, inc, log in ((10, True, True), (4, True, True), (6, False, True), (5, True, False), (0, True, True)):
        fn = lambda x, L=L, inc=inc, log=log: O.positional_encoding(x, L, inc, log)  # noqa: E731
        got = train_utils._probe_encoder(fn, None)
        if L == 0:
            assert got[0] == 0 and got[1] is True
        else:
            assert got == (L, inc, log), (got, (L, inc, log))
    assert train_utils._probe_encoder(get_embedding_function(7, False, True), None) == (7, False, True)
    with pytest.raises(NotImplementedError):
        train_utils._probe_encoder(lambda x: torch.tanh(x), None)


def test_encoder_probe_is_memoised_and_invalidate_bumps_the_cache_epoch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import train_utils
    from oracle import nerf_oracle as O

    calls = []

    def enc(x):
        calls.append(1)
        return O.positional_encoding(x, 10, True, True)

    assert train_utils._probe_encoder(enc, None) == (10, True, True)
    n = len(calls)
    for _ in range(5):   # every chunk of every iteration asks again: no further evaluations of the user's callable
        assert train_utils._probe_encoder(enc, None) == (10, True, True)
    assert len(calls) == n
    m = nb.FlexibleNeRFModel()
    e0 = getattr(m, "_nerfb200_epoch", 0)
    nb.invalidate(m)
    assert m._nerfb200_epoch == e0 + 1 and m not in train_utils._CACHE


def test_model_introspection_and_state_dict_compat():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import train_utils
    from oracle import nerf_oracle as O

    m = nb.FlexibleNeRFModel(num_layers=8, hidden_size=128, skip_connect_every=3, num_encoding_fn_xyz=10)
    sd = O.init_flexible_nerf(8, 128, 3, 10, 4)
    m.load_state_dict(sd)  # same keys/shapes as the reference class
    arch = train_utils._arch_of(m, (10, True, True), (4, True, True))
    assert (arch.num_layers, arch.hidden, arch.skip_every) == (8, 128, 3)
    x = torch.randn(5, 63 + 27)
    assert torch.allclose(m(x), O.flexible_nerf_forward(sd, x, 63), atol=1e-6)
    with pytest.raises(NotImplementedError):
        train_utils._arch_of(torch.nn.Linear(3, 3), (10, True, True), (4, True, True))
    with pytest.raises(RuntimeError):
        train_utils._arch_of(m, (6, True, True), (4, True, True))  # encoder / layer1 width mismatch


def test_product_path_refuses_cpu_tensors():
    import nerf_pytorch_b200 as nb
    from oracle import nerf_oracle as O

    m = nb.FlexibleNeRFModel(num_encoding_fn_xyz=10)
    rays = torch.zeros(4, 11)
    with pytest.raises(NotImplementedError):
        nb.predict_and_render_radiance(rays, m, m, O.make_options(), encode_position_fn=nb.get_embedding_function(10),
                                       encode_direction_fn=nb.get_embedding_function(4))


def test_shard_bounds_partition():
    from nerf_pytorch_b200.parallel import shard_bounds

    for n, w in ((32768, 8), (4096, 1), (10, 3), (7, 8)):
        spans = [shard_bounds(n, r, w) for r in range(w)]
        assert spans[0][0] == 0 and spans[-1][1] == n
        assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
        assert max(h - l for l, h in spans) - min(h - l for l, h in spans) <= 1


def test_fp16x2_split_precision_model():
    """CPU model of the operand split the wgmma chain kernels use (csrc/tc_common.cuh split_f16x2):
    hi = fp16(x) saturating, lo = fp16((x - hi) * 2^11); x ~= hi + lo * 2^-11.  Pins the documented claims: ~22
    significant bits over 6.1e-5 <= |x| < 65504 (1.5e-11 absolute below), and a three-term product sum (hi*hi + 2^-11 (lo*hi + hi*lo), fp32
    accumulation) that stays far inside the 1e-4 parity bar where a plain fp16 or tf32 product does not."""
    import torch

    def split(x):
        hi = x.clamp(-65504.0, 65504.0).to(torch.float16)
        lo = ((x - hi.float()) * 2048.0).clamp(-65504.0, 65504.0).to(torch.float16)
        return hi.float(), lo.float()

    g = torch.Generator().manual_seed(0)
    # magnitudes log-uniform over the claimed range, both signs
    mag = torch.exp(torch.empty(200000).uniform_(math.log(1e-7), math.log(6e4), generator=g))
    x = mag * torch.where(torch.rand(200000, generator=g) < 0.5, -1.0, 1.0)
    hi, lo = split(x)
    err = ((hi.double() + lo.double() / 2048.0) - x.double()).abs()
    normal = x.abs() >= 6.2e-5  # hi is a normal fp16 number
    assert (err[normal] / x.double().abs()[normal]).max().item() < 2.0 ** -20
    assert err[~normal].max().item() < 2e-11
    # the unscaled residual would be subnormal below 0.125 and lose that precision
    lo_plain = (x - hi).to(torch.float16).float()
    small = x.abs() < 1e-3
    rel_plain = ((hi.double() + lo_plain.double()) - x.double()).abs() / x.double().abs()
    assert rel_plain[small].max().item() > 2.0 ** -16

    # a 128-wide layer: activations ~ ReLU outputs, weights ~ trained-NeRF scale
    a = torch.randn(512, 128, generator=g).clamp_min(0) * 3.0
    w = torch.randn(128, 128, generator=g) * 0.2
    ref = a.double() @ w.double().t()
    ah, al = split(a)
    wh, wl = split(w)
    got = ah @ wh.t() + (al @ wh.t() + ah @ wl.t()) / 2048.0
    scale = ref.abs().max().item()
    assert (got.double() - ref).abs().max().item() <= 2e-6 * scale
    single = a.to(torch.float16).float() @ w.to(torch.float16).float().t()
    assert (single.double() - ref).abs().max().item() > 1e-4 * scale  # why one fp16 term is not enough

    # dgrad rows run in their own power-of-two scale: max-abs of the row lands in [1, 2), exactly invertible
    d = torch.randn(1000, 4, generator=g) * torch.exp(torch.empty(1000, 1).uniform_(-40, 10, generator=g))
    m = d.abs().amax(dim=1)
    e = (m.view(torch.int32) >> 23) & 0xFF
    sc = ((254 - e) << 23).view(torch.float32)
    scaled = d * sc[:, None]
    smax = scaled.abs().amax(dim=1)
    assert bool(((smax >= 1.0) & (smax < 2.0)).all())
    assert torch.equal(scaled * (e << 23).view(torch.float32)[:, None], d)


def test_cached_dataset_pool_reads_the_reference_cache_format(tmp_path):
    """cache_dataset.py:104-135 files (one torch.save dict per image) -> one resident pool; sample() = the reference's
    two-stage draw (train_nerf.py:175-193): one image, n distinct rays of it, targets cut to rgb."""
    import nerf_pytorch_b200 as nb

    g = torch.Generator().manual_seed(0)
    os.makedirs(tmp_path / "train"), os.makedirs(tmp_path / "val")
    imgs = []
    for i, (shape, tch) in enumerate((((2, 50, 3), 3), ((2, 6, 8, 3), 4))):   # sampled-ray and whole-image variants, rgb / rgba
        rb = torch.randn(*shape, generator=g)
        tgt = torch.rand(*shape[1:-1], tch, generator=g)
        torch.save({"height": 6, "width": 8, "focal_length": 11.5, "ray_bundle": rb, "target": tgt}, tmp_path / "train" / f"{i:04d}.data")
        imgs.append((rb, tgt))
    torch.save({"height": 6, "width": 8, "focal_length": 11.5, "ray_origins": torch.randn(6, 8, 3), "ray_directions": torch.randn(6, 8, 3),
                "target": torch.rand(6, 8, 4)}, tmp_path / "val" / "0007.data")
    pool = nb.CachedRayPool.from_dir(str(tmp_path), device="cpu")
    assert pool.num_images == 2 and len(pool) == 50 + 48
    seen = set()
    for _ in range(20):
        h, w, f, ro, rd, tg = pool.sample(16, generator=g)
        assert (h, w, f) == (6, 8, 11.5) and ro.shape == rd.shape == tg.shape == (16, 3)
        # the 16 rows are distinct rows of ONE cached image, with that image's directions and rgb targets
        hit = None
        for k, (rb, tgt) in enumerate(imgs):
            o_all, d_all, t_all = rb[0].reshape(-1, 3), rb[1].reshape(-1, 3), tgt[..., :3].reshape(-1, 3)
            idx = [(o_all == r).all(-1).nonzero() for r in ro]
            if all(len(j) == 1 for j in idx):
                j = torch.cat(idx).flatten()
                assert len(set(j.tolist())) == 16 and torch.equal(d_all[j], rd) and torch.equal(t_all[j], tg)
                hit = k
        assert hit is not None
        seen.add(hit)
    assert seen == {0, 1}
    with pytest.raises(ValueError):
        while True:
            pool.sample(49, generator=g)   # the 48-ray image cannot give 49 distinct rays (np.random.choice(replace=False) raises too)
    ro, rd, tg = pool.sample_global(200, generator=g)
    assert ro.shape == (200, 3)
    val = nb.CachedValidationSet.from_dir(str(tmp_path), device="cpu")
    h, w, f, ro, rd, tg = val.choice(generator=g)
    assert len(val) == 1 and ro.shape == (6, 8, 3) and tg.shape == (6, 8, 4)
