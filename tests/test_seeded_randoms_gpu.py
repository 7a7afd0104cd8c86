"""Seeded in-kernel random numbers (ops.SeededRandoms, nerfb200_rng_t).

The stream is checked against a numpy restatement of Philox4x32-10 (itself pinned to Random123's known-answer vectors,
CPU), then the render path is checked to consume exactly that stream: a seeded step equals a step fed the same numbers
as tensors, bit for bit, and a ray's result does not depend on how the batch is chunked or sharded."""
import copy
import math

import numpy as np
import pytest
import torch

from helpers import Case, OUT_NAMES

# ------------------------------------------------------------------------------------------------
# numpy restatement of the stream (csrc/common.cuh)
# ------------------------------------------------------------------------------------------------
_MASK = np.uint64(0xFFFFFFFF)
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on uint32 values held in uint64 arrays; returns the four output words (uint64 arrays)."""
    c = [np.asarray(x, dtype=np.uint64) & _MASK for x in (c0, c1, c2, c3)]
    k0, k1 = np.uint64(k0), np.uint64(k1)
    for i in range(10):
        if i:
            k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
        p0, p1 = _M0 * c[0], _M1 * c[2]  # 32 x 32 -> 64 bits, exact in uint64
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & _MASK]
    return c


def stream_words(seed, step, stream, ray_offset, n_rays, per_ray):
    """uint64 [n_rays, ceil(per_ray / 4) * 4] words of one stream: counter (sample / 4, stream + 4 step, ray lo, ray hi)."""
    nb = (per_ray + 3) // 4
    ray = np.arange(n_rays, dtype=np.uint64)[:, None] + np.uint64(ray_offset)
    blk = np.arange(nb, dtype=np.uint64)[None, :]
    ray, blk = np.broadcast_arrays(ray, blk)
    w = philox4x32_10(blk, np.uint64(stream + 4 * step), ray & _MASK, ray >> np.uint64(32), seed & 0xFFFFFFFF, seed >> 32)
    return np.stack(w, axis=-1).reshape(n_rays, nb * 4)


def stream_values(seed, step, stream, ray_offset, n_rays, per_ray):
    """Uniforms (streams 0, 2: float32, exact) or normals (streams 1, 3: float64 Box-Muller) of one stream."""
    w = stream_words(seed, step, stream, ray_offset, n_rays, per_ray)
    if stream in (0, 2):
        return ((w >> np.uint64(8)).astype(np.float64) * 2.0 ** -24).astype(np.float32)[:, :per_ray]
    a, b = w[:, 0::2], w[:, 1::2]  # pairs (w0, w1), (w2, w3), ...
    u1 = ((a >> np.uint64(8)).astype(np.float64) + 1.0) * 2.0 ** -24
    u2 = (b >> np.uint64(8)).astype(np.float64) * 2.0 ** -24
    r = np.sqrt(-2.0 * np.log(u1))
    out = np.empty(w.shape, dtype=np.float64)
    out[:, 0::2] = r * np.cos(2.0 * np.pi * u2)
    out[:, 1::2] = r * np.sin(2.0 * np.pi * u2)
    return out[:, :per_ray]


def test_philox_restatement_matches_random123_known_answers():
    # Random123 kat_vectors, philox4x32 10 rounds (confirmed with ATen's at::Philox4_32)
    assert [int(x) for x in philox4x32_10(0, 0, 0, 0, 0, 0)] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    f = 0xFFFFFFFF
    assert [int(x) for x in philox4x32_10(f, f, f, f, f, f)] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    got = philox4x32_10(0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344, 0xA4093822, 0x299F31D0)
    assert [int(x) for x in got] == [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]


def test_seeded_randoms_value_type():
    from nerf_pytorch_b200 import SeededRandoms

    r = SeededRandoms(2 ** 64 - 1, 2 ** 30 - 1, 5)
    assert r.shifted(7) == SeededRandoms(2 ** 64 - 1, 2 ** 30 - 1, 12)
    assert hash(r) == hash(SeededRandoms(2 ** 64 - 1, 2 ** 30 - 1, 5))
    c = r.c_struct()
    assert (c.seed, c.step, c.ray_offset) == (2 ** 64 - 1, 2 ** 30 - 1, 5)
    for bad in (dict(seed=-1), dict(seed=2 ** 64), dict(seed=0, step=2 ** 30), dict(seed=0, ray_offset=-1)):
        with pytest.raises(ValueError):
            SeededRandoms(**bad)


# ------------------------------------------------------------------------------------------------
# GPU: the stream itself
# ------------------------------------------------------------------------------------------------
gpu = pytest.mark.gpu


def _fill(rng, stream, n, per_ray):
    from nerf_pytorch_b200 import ops

    return ops.random_fill(rng, stream, n, per_ray, device="cuda")


@gpu
@pytest.mark.parametrize("stream", [0, 1, 2, 3])
def test_random_fill_equals_the_numpy_restatement(stream):
    from nerf_pytorch_b200 import SeededRandoms

    # a ray range that crosses 2^32 (the counter's high ray word), 13 samples (a partial last block)
    for seed, step, off, n, per in ((0, 0, 0, 64, 13), (0x0123456789ABCDEF, 12345, 2 ** 32 - 40, 96, 13),
                                    (2 ** 64 - 1, 2 ** 30 - 1, 7, 33, 192)):
        got = _fill(SeededRandoms(seed, step, off), stream, n, per).cpu().numpy()
        want = stream_values(seed, step, stream, off, n, per)
        if stream in (0, 2):
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (seed, step, off)
        else:
            err = np.abs(got.astype(np.float64) - want)
            print(f"stream {stream} seed {seed:#x}: max |device - float64| = {err.max():.3g}")
            # fp64 Box-Muller rounded once: within one fp32 ulp of the float64 restatement (measured: half an ulp)
            assert err.max() <= 1e-6 and (err <= np.spacing(np.abs(want).astype(np.float32))).all(), err.max()


@gpu
def test_stream_statistics():
    from scipy import stats

    from nerf_pytorch_b200 import SeededRandoms

    n_rays, per = 32768, 128  # 4 194 304 draws per stream
    rng = SeededRandoms(20261015, 3, 1000)
    u = {s: _fill(rng, s, n_rays, per).double() for s in range(4)}
    n = n_rays * per
    for s in (0, 2):
        assert u[s].min().item() >= 0.0 and u[s].max().item() < 1.0
        p = stats.kstest(u[s].flatten().cpu().numpy(), "uniform").pvalue
        assert p > 1e-3, (s, p)
    for s in (1, 3):
        p = stats.kstest(u[s].flatten().cpu().numpy(), "norm").pvalue
        assert p > 1e-3, (s, p)
        m, v = u[s].mean().item(), u[s].var().item()
        assert abs(m) < 5 / math.sqrt(n) and abs(v - 1) < 5 * math.sqrt(2 / n), (m, v)

    def corr(a, b):
        a, b = a.flatten() - a.mean(), b.flatten() - b.mean()
        return ((a * b).sum() / (a.norm() * b.norm())).item()

    bar = 3 / math.sqrt(n)
    pairs = {f"streams {a}/{b}": (u[a], u[b]) for a, b in ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))}
    # adjacent rays: row r against row r + 1 (ray_offset + 1), and adjacent steps
    nxt = {s: _fill(rng.shifted(1), s, n_rays, per).double() for s in (0, 1)}
    pairs.update({f"ray+1 stream {s}": (u[s], nxt[s]) for s in (0, 1)})
    step1 = SeededRandoms(rng.seed, rng.step + 1, rng.ray_offset)
    pairs.update({f"step+1 stream {s}": (u[s], _fill(step1, s, n_rays, per).double()) for s in (0, 1)})
    # adjacent samples of one ray (the cos / sin halves of one Box-Muller pair for the normals)
    pairs.update({f"sample+1 stream {s}": (u[s][:, :-1], u[s][:, 1:]) for s in (0, 1)})
    for name, (a, b) in pairs.items():
        c = corr(a, b)
        assert abs(c) < bar, (name, c, bar)
    # the shifted stream is the same stream: ray r of offset k + 1 is ray r + 1 of offset k
    assert torch.equal(nxt[0][:-1], u[0][1:])


@gpu
def test_every_key_component_changes_the_words():
    from nerf_pytorch_b200 import SeededRandoms

    base = SeededRandoms(99, 5, 4096)
    ref = _fill(base, 0, 2048, 64)
    for other in (SeededRandoms(100, 5, 4096), SeededRandoms(99 + 2 ** 32, 5, 4096), SeededRandoms(99, 6, 4096),
                  SeededRandoms(99, 5, 4097), SeededRandoms(99, 5, 4096 + 2 ** 32)):
        same = (_fill(other, 0, 2048, 64) == ref).double().mean().item()
        assert same < 1e-3, (other, same)
    assert not torch.equal(_fill(base, 2, 2048, 64), ref)  # stream id


# ------------------------------------------------------------------------------------------------
# GPU: the render path consumes exactly that stream
# ------------------------------------------------------------------------------------------------
def _models(c: Case):
    import nerf_pytorch_b200 as nb

    def mk(sd):
        m = nb.FlexibleNeRFModel(num_layers=c.num_layers, hidden_size=c.hidden, skip_connect_every=c.skip,
                                 num_encoding_fn_xyz=c.enc_xyz[0], num_encoding_fn_dir=c.enc_dir[0],
                                 include_input_xyz=c.enc_xyz[1], include_input_dir=c.enc_dir[1],
                                 use_viewdirs=c.use_viewdirs)
        m.load_state_dict(sd)
        return m.cuda()

    mc = mk(c.sd_c)
    mf = mk(c.sd_f) if c.sd_f is not None else None
    epf = nb.get_embedding_function(*c.enc_xyz)
    edf = nb.get_embedding_function(*c.enc_dir) if c.use_viewdirs else None
    return mc, mf, epf, edf


def _tensors_of(rng, n, opts_train, fine):
    nc, nf = int(opts_train.num_coarse), int(opts_train.num_fine)
    d = dict(t_rand=_fill(rng, "t_rand", n, nc), noise_c=_fill(rng, "noise_c", n, nc))
    if fine:
        d.update(u=_fill(rng, "u", n, nf), noise_f=_fill(rng, "noise_f", n, nc + nf))
    return d


def _step(c, mc, mf, epf, edf, options, randoms, impl, tgt=None, grad=True):
    import nerf_pytorch_b200 as nb

    for m in (mc, mf):
        if m is not None:
            m.zero_grad(set_to_none=True)
    out = nb.run_one_iter_of_nerf(c.H, c.W, c.focal, mc, mf, c.ro.cuda(), c.rd.cuda(), options, mode=c.mode,
                                  encode_position_fn=epf, encode_direction_fn=edf, randoms=randoms, impl=impl)
    loss = None
    if grad:
        tgt = c.target.cuda() if tgt is None else tgt
        loss = torch.nn.functional.mse_loss(out[0].reshape(-1, 3), tgt)
        if out[3] is not None:
            loss = loss + torch.nn.functional.mse_loss(out[3].reshape(-1, 3), tgt)
        loss.backward()
    grads = [p.grad.clone() for m in (mc, mf) if m is not None for p in m.parameters()]
    return [o.detach().clone() if o is not None else None for o in out], loss, grads


def _bits_equal(a, b):
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# (golden case, overrides of options.nerf.train): A0 lego weights, A1 at init, NDC, coarse-only
EXACT_CASES = {
    "perturb_noise": ("lego_a0_train", {}),
    "perturb_no_noise": ("lego_a0_train", dict(radiance_field_noise_std=0.0)),
    "det_noise": ("lego_a0_train", dict(perturb=False)),
    "det_white_val": ("lego_a0_det_white_val", {}),
    "ndc_fern": ("fern_a0_ndc", {}),
    "a1_lindisp_white": ("a1_skip_lindisp", {}),
    "coarse_only": ("lego_a0_train", dict(num_fine=0)),
    "coarse_only_noview": ("a0_noview_coarse_only", dict(radiance_field_noise_std=0.5)),
}
# the wgmma backward needs the view-dependent heads: the model without them trains on the fp32 kernels only
EXACT_PARAMS = [(k, i) for k in EXACT_CASES for i in (0, 1) if not (k == "coarse_only_noview" and i == 1)]


@gpu
@pytest.mark.parametrize("key,impl", EXACT_PARAMS, ids=[f"{k}-{'tc' if i else 'simt'}" for k, i in EXACT_PARAMS])
def test_seeded_step_equals_injected_tensors_bit_for_bit(key, impl):
    from nerf_pytorch_b200 import SeededRandoms

    name, over = EXACT_CASES[key]
    c = Case(name)
    options = copy.deepcopy(c.options)
    for k, v in over.items():
        setattr(options.nerf.train, k, v)
    mc, mf, epf, edf = _models(c)
    if options.nerf.train.num_fine == 0:
        mf = None
    rng = SeededRandoms(0xC0FFEE, 17, 0)
    n = c.ro.reshape(-1, 3).shape[0]
    out_s, loss_s, g_s = _step(c, mc, mf, epf, edf, options, rng, impl)
    tens = _tensors_of(rng, n, options.nerf.train, mf is not None)
    out_d, loss_d, g_d = _step(c, mc, mf, epf, edf, options, tens, impl)
    for nm, a, b in zip(OUT_NAMES, out_s, out_d):
        assert _bits_equal(a, b), (key, nm)
    assert _bits_equal(loss_s, loss_d), (loss_s.item(), loss_d.item())
    if impl == 1:
        # the wgmma backward sums its gradients in fixed point: the same inputs give the same bits
        for i, (a, b) in enumerate(zip(g_s, g_d)):
            assert _bits_equal(a, b), (key, i)
    else:
        # the fp32 CUDA-core weight-gradient kernel flushes its partial sums with float atomics, so two runs on the same
        # inputs already differ in summation order: compare against that run-to-run spread
        _, _, g_d2 = _step(c, mc, mf, epf, edf, options, tens, impl)
        for i, (a, b, b2) in enumerate(zip(g_s, g_d, g_d2)):
            scale = b.abs().max().item() + 1e-30
            d_sd, d_dd = (a - b).abs().max().item() / scale, (b2 - b).abs().max().item() / scale
            assert d_sd <= max(4 * d_dd, 1e-6), (key, i, d_sd, d_dd)


def _pose_rays(n, seed=0, H=100, W=100, focal=120.0):
    from nerf_pytorch_b200 import ops

    pose = torch.tensor([[1.0, 0, 0, 0], [0, 1.0, 0, 0], [0, 0, 1.0, 4.0], [0, 0, 0, 1.0]])
    g = torch.Generator().manual_seed(seed)
    pix = torch.randperm(H * W, generator=g)[:n].cuda()
    rays6 = ops.gen_rays(pose, H, W, focal, pix, torch.device("cuda"), use_viewdirs=False, stride=6)
    return pose, rays6[:, :3].contiguous(), rays6[:, 3:].contiguous(), torch.rand(n, 3, generator=g).cuda()


def _a1_models(seed=0):
    import nerf_pytorch_b200 as nb
    from oracle import nerf_oracle as O

    gen = torch.Generator().manual_seed(seed)
    mods = []
    for _ in range(2):
        m = nb.FlexibleNeRFModel(num_layers=8, hidden_size=128, skip_connect_every=3, num_encoding_fn_xyz=10,
                                 num_encoding_fn_dir=4)
        m.load_state_dict(O.init_flexible_nerf(8, 128, 3, 10, 4, generator=gen))
        mods.append(m.cuda())
    return mods[0], mods[1], nb.get_embedding_function(10), nb.get_embedding_function(4)


def _lego_models():
    return _models(Case("lego_a0_train"))[:4]


@gpu
@pytest.mark.parametrize("impl", [0, 1], ids=["simt", "tc"])
def test_chunking_and_sharding_do_not_change_a_ray(impl):
    import nerf_pytorch_b200 as nb
    from oracle import nerf_oracle as O

    n, k = 1000, 389
    _, ro, rd, tgt = _pose_rays(n)
    mc, mf, epf, edf = _lego_models()
    rng = nb.SeededRandoms(424242, 9, 0)

    def run(ro_, rd_, tgt_, chunk, r):
        opts = O.make_options(chunksize=chunk, radiance_field_noise_std=0.2)
        for m in (mc, mf):
            m.zero_grad(set_to_none=True)
        out = nb.run_one_iter_of_nerf(100, 100, 120.0, mc, mf, ro_, rd_, opts, encode_position_fn=epf,
                                      encode_direction_fn=edf, randoms=r, impl=impl)
        loss = (torch.nn.functional.mse_loss(out[0], tgt_, reduction="sum") +
                torch.nn.functional.mse_loss(out[3], tgt_, reduction="sum"))
        loss.backward()
        return [o.detach().clone() for o in out], [p.grad.clone() for m in (mc, mf) for p in m.parameters()]

    whole, g_whole = run(ro, rd, tgt, n, rng)
    thirds, g_thirds = run(ro, rd, tgt, n // 3, rng)  # 333, 333, 333, 1: ragged
    a, g_a = run(ro[:k], rd[:k], tgt[:k], n, rng)
    b, g_b = run(ro[k:], rd[k:], tgt[k:], n, rng.shifted(k))
    shards = [torch.cat([x, y]) for x, y in zip(a, b)]
    for nm, w, t, s in zip(OUT_NAMES, whole, thirds, shards):
        assert _bits_equal(w, t), ("chunked", nm)
        assert _bits_equal(w, s), ("sharded", nm)
    # gradients: the chunks' sums are added in fp32 afterwards, so they agree to that rounding (measured on an H100:
    # 5.6e-7 of the tensor's max on the fp32 kernels, 1.6e-7 on the wgmma kernels)
    worst = 0.0
    for gw, gt, ga, gb in zip(g_whole, g_thirds, g_a, g_b):
        scale = gw.abs().max().item() + 1e-30
        worst = max(worst, (gt - gw).abs().max().item() / scale, (ga + gb - gw).abs().max().item() / scale)
    print(f"impl {impl}: worst chunked / sharded gradient difference {worst:.3g} of the tensor's max")
    assert worst < 3e-6, worst


@gpu
def test_seeded_full_image_render_is_reproducible_across_chunk_sizes():
    import nerf_pytorch_b200 as nb
    from oracle import nerf_oracle as O

    pose = torch.tensor([[1.0, 0, 0, 0], [0, 1.0, 0, 0], [0, 0, 1.0, 4.0]])
    mc, mf, epf, edf = _lego_models()
    opts = O.make_options(perturb=True, radiance_field_noise_std=0.2)
    rng = nb.SeededRandoms(7, 0)

    def render(chunk, r):
        return nb.render_image(100, 100, 120.0, pose, mc, mf, opts, encode_position_fn=epf, encode_direction_fn=edf,
                               rays_per_chunk=chunk, randoms=r)

    first = render(4096, rng)
    again = render(4096, rng)
    other = render(1500, rng)
    for nm, a, b, c in zip(OUT_NAMES, first, again, other):
        assert _bits_equal(a, b), ("twice", nm)
        assert _bits_equal(a, c), ("chunk size", nm)
    # a different step renders different jitter
    assert not torch.equal(render(4096, nb.SeededRandoms(7, 1))[3], first[3])
    with pytest.raises(TypeError):
        render(4096, {"t_rand": None})


@gpu
def test_seeded_step_leaves_torch_generators_alone_and_saves_no_noise():
    import nerf_pytorch_b200 as nb

    c = Case("lego_a0_train")
    mc, mf, epf, edf = _models(c)
    n = c.ro.shape[0]
    nc, nf = c.options.nerf.train.num_coarse, c.options.nerf.train.num_fine
    saved = []

    def pack(t):
        saved.append(tuple(t.shape))
        return t

    torch.cuda.synchronize()
    cuda_state, cpu_state = torch.cuda.get_rng_state(), torch.get_rng_state()
    with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
        _step(c, mc, mf, epf, edf, c.options, nb.SeededRandoms(1, 2), None)
    torch.cuda.synchronize()
    assert torch.equal(torch.cuda.get_rng_state(), cuda_state)
    assert torch.equal(torch.get_rng_state(), cpu_state)
    noise_shapes = {(n, nc), (n, nc + nf)}
    assert saved and not noise_shapes & set(saved), saved
    # the torch-drawn path does keep them (the hook sees what the render saves) and advances the generator
    saved.clear()
    with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
        _step(c, mc, mf, epf, edf, c.options, None, None)
    assert noise_shapes <= set(saved), saved
    assert not torch.equal(torch.cuda.get_rng_state(), cuda_state)


@gpu
@pytest.mark.parametrize("impl", [0, 1], ids=["simt", "tc"])
def test_seeded_render_bwd_reads_no_noise_tensor(impl):
    """The C entry points directly: render_fwd + render_bwd given a SeededRandoms against the same calls fed the
    random_fill tensors.  The seeded backward regenerates the noise for the sigma ReLU gate."""
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops, train_utils

    c = Case("fern_a0_ndc")  # noise std 1.0: many gates flip
    mc, mf, epf, edf = _models(c)
    o = c.options.nerf.train
    arch = train_utils._arch_of(mc, c.enc_xyz, c.enc_dir)
    _, blob_c = train_utils._packed(mc, arch)
    _, blob_f = train_utils._packed(mf, arch)
    rays = ops.pack_rays(c.ro.cuda().contiguous(), c.rd.cuda().contiguous(), c.H, c.W, c.focal,
                         c.options.dataset.no_ndc is False, c.options.dataset.near, c.options.dataset.far, True)
    n, nc, nf = rays.shape[0], o.num_coarse, o.num_fine
    opts = ops.make_opts(nc, nf, o.perturb, o.lindisp, o.white_background, o.radiance_field_noise_std)
    rng = nb.SeededRandoms(31337, 4, 10 ** 6)
    r = _tensors_of(rng, n, o, True)
    g = torch.Generator().manual_seed(3)
    g_c, g_f = torch.randn(n, 8, generator=g).cuda(), torch.randn(n, 8, generator=g).cuda()
    nfl = arch.flat_param_count()

    out_s = ops.render_fwd(arch, arch, opts, blob_c, blob_f, rays, rng, training=True, impl=impl)
    fg_s = torch.zeros(2 * nfl, device="cuda")
    ops.render_bwd(arch, arch, opts, blob_c, blob_f, rays, rng, g_c, g_f, out_s[2], fg_s[:nfl], fg_s[nfl:], impl=impl)
    out_d = ops.render_fwd(arch, arch, opts, blob_c, blob_f, rays, r, training=True, impl=impl)
    fg_d = torch.zeros(2 * nfl, device="cuda")
    ops.render_bwd(arch, arch, opts, blob_c, blob_f, rays, r, g_c, g_f, out_d[2], fg_d[:nfl], fg_d[nfl:], impl=impl)
    assert _bits_equal(out_s[0], out_d[0]) and _bits_equal(out_s[1], out_d[1])
    if impl == 1:
        assert _bits_equal(fg_s, fg_d)
    else:  # float atomics in the fp32 weight-gradient flush (see the step test)
        torch.testing.assert_close(fg_s, fg_d, rtol=1e-5, atol=1e-6 * fg_d.abs().max().item())


@gpu
def test_library_refuses_out_of_range_rng():
    import ctypes as C

    from nerf_pytorch_b200 import _lib

    lib = _lib.load()
    out = torch.empty(4, 4, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for rng in (_lib.Rng(0, 2 ** 30, 0), _lib.Rng(0, 0, -1)):
        assert lib.nerfb200_random_fill(C.byref(rng), 0, 4, 4, C.c_void_p(out.data_ptr()), stream) == _lib.ERR_INVALID
    assert lib.nerfb200_random_fill(C.byref(_lib.Rng(0, 0, 0)), 4, 4, 4, C.c_void_p(out.data_ptr()), stream) == \
        _lib.ERR_INVALID
    assert lib.nerfb200_random_fill(C.byref(_lib.Rng(0, 2 ** 30 - 1, 0)), 3, 4, 4, C.c_void_p(out.data_ptr()), stream) == \
        _lib.OK


@gpu
def test_render_entry_points_refuse_rng_with_tensors_and_out_of_range_rng():
    """render_fwd / render_bwd take the randoms from an rng or from tensors, never both, and check the rng."""
    import ctypes as C

    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    arch = ops.ArchSpec()
    nc, nf, n = 64, 64, 128
    opts = ops.make_opts(nc, nf, True, False, False, 1.0)
    nfl = arch.flat_param_count()
    blob = ops.pack_weights(arch, torch.zeros(nfl, device="cuda"))
    rays = torch.rand(n, 11, device="cuda")
    rays[:, 6], rays[:, 7] = 2.0, 6.0
    ws = torch.empty(ops.render_workspace_bytes(arch, arch, opts, n, True), dtype=torch.uint8, device="cuda")
    out = torch.empty(2, n, 8, device="cuda")
    g = torch.zeros(n, 8, device="cuda")
    fg = torch.zeros(2 * nfl, device="cuda")
    rnd = torch.rand(n, nc + nf, device="cuda")  # large enough for any of the four inputs
    p = lambda t: C.c_void_p(t.data_ptr())
    a, o = C.byref(arch.c_struct()), C.byref(opts)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def fwd(rng, tensors):
        return lib.nerfb200_render_fwd(a, a, o, p(blob), p(blob), p(rays), 11, n, rng, *tensors, p(out[0]), p(out[1]),
                                       p(ws), 1, ops.IMPL_SIMT, stream)

    def bwd(rng, tensors):
        return lib.nerfb200_render_bwd(a, a, o, p(blob), p(blob), p(rays), 11, n, rng, *tensors, p(g), p(g), p(ws),
                                       p(fg[:nfl]), p(fg[nfl:]), ops.IMPL_SIMT, 3, stream)

    def one_tensor(k, count):
        return [p(rnd) if i == k else None for i in range(count)]

    rng = C.byref(_lib.Rng(5, 6, 7))
    assert fwd(rng, [None] * 4) == _lib.OK and bwd(rng, [None] * 2) == _lib.OK
    for k in range(4):
        assert fwd(rng, one_tensor(k, 4)) == _lib.ERR_INVALID, k
        assert b"random tensor" in lib.nerfb200_last_error()
    for k in range(2):
        assert bwd(rng, one_tensor(k, 2)) == _lib.ERR_INVALID, k
        assert b"random tensor" in lib.nerfb200_last_error()
    for bad in (_lib.Rng(0, 2 ** 30, 0), _lib.Rng(0, 0, -1)):
        assert fwd(C.byref(bad), [None] * 4) == _lib.ERR_INVALID
        assert bwd(C.byref(bad), [None] * 2) == _lib.ERR_INVALID
    torch.cuda.synchronize()


@gpu
def test_sample_coarse_grid_is_torch_linspace_at_every_sample_count():
    """The stratified grid is built in the kernel: with near 0, far 1 and no jitter, z = 0 * (1 - t) + 1 * t = t exactly,
    so z must be torch's CUDA linspace bit for bit at every n_coarse the library accepts."""
    from nerf_pytorch_b200 import ops

    rays = torch.zeros(3, 8, device="cuda")
    rays[:, 7] = 1.0
    for nc in range(2, 1025):
        z = ops.sample_coarse(rays, None, nc, False, False)
        want = torch.linspace(0.0, 1.0, nc, device="cuda").expand(3, nc)
        assert _bits_equal(z, want), nc


@gpu
def test_sample_pdf_det_u_is_torch_linspace_at_every_fine_count():
    """u = None resamples at the det=True linspace built in the kernel: the same bits as feeding torch's CUDA linspace
    to every ray, at every n_fine the library accepts for n_coarse 64."""
    from nerf_pytorch_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(11)
    n, nc = 8, 64
    zc = torch.sort(torch.rand(n, nc, device="cuda", generator=g) * 4 + 2, -1).values.contiguous()
    w = (torch.rand(n, nc, device="cuda", generator=g) ** 4).contiguous()
    for nf in range(1, 1024 - nc + 1):
        got = ops.sample_pdf_merge(zc, w, None, nf, want_aux=True)
        u = torch.linspace(0.0, 1.0, nf, device="cuda").expand(n, nf).contiguous()
        want = ops.sample_pdf_merge(zc, w, u, nf, want_aux=True)
        for a, b in zip(got, want):
            assert _bits_equal(a, b), nf


@gpu
def test_seeded_fused_adam_training_is_bit_reproducible():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import parallel, train_utils
    from oracle import nerf_oracle as O

    _, ro, rd, tgt = _pose_rays(1024, seed=5)
    opts = O.make_options(radiance_field_noise_std=0.2)

    def train():
        mc, mf, epf, edf = _a1_models(seed=1)
        arch = train_utils._arch_of(mc, (10, True, True), (4, True, True))
        optim = parallel.FusedAdam([(mc, arch), (mf, arch)], lr=5e-3)
        losses = []
        for i in range(10):
            out = nb.run_one_iter_of_nerf(100, 100, 120.0, mc, mf, ro, rd, opts, encode_position_fn=epf,
                                          encode_direction_fn=edf, randoms=nb.SeededRandoms(2026, i))
            loss = torch.nn.functional.mse_loss(out[0], tgt) + torch.nn.functional.mse_loss(out[3], tgt)
            optim.zero_grad()
            loss.backward()
            optim.step()
            losses.append(loss.detach())
        return torch.stack(losses), torch.cat([it["flat"] for it in optim.items])

    l1, p1 = train()
    l2, p2 = train()
    print("seeded losses:", [round(x, 6) for x in l1.tolist()])
    assert _bits_equal(l1, l2) and _bits_equal(p1, p2)
    assert l1[-1].item() < l1[0].item()
