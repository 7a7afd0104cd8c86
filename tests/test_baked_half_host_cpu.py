"""Host: half-precision baked fields (include/nerfb200.h "baked fields: half precision").  The three fp16 entry points'
ABI and refusals, the fp32 -> fp16 conversion rule of BakedField.half against numpy, the exact widening of
BakedField.float, pruning and save / load of an fp16 field, and the Python refusals.  No GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

BOX = ((-1.0,) * 3, (1.0,) * 3)


def test_signatures_of_the_fp16_entry_points():
    from nerf_pytorch_b200 import _lib

    AP, GP, P = C.POINTER(_lib.Arch), C.POINTER(_lib.Grid), C.c_void_p
    I32, I64, F32 = C.c_int32, C.c_int64, C.c_float
    assert _lib.SIGNATURES["nerfb200_bake_f16"] == (I32, [AP, P, GP, P, I64, I64, P, P, P])
    assert _lib.SIGNATURES["nerfb200_baked_render_f16"] == (I32, [GP, P, P, I32, P, I32, I64, I32, F32, P, P])
    assert _lib.SIGNATURES["nerfb200_baked_max_weights_f16"] == (I32, [GP, P, P, I32, P, I32, I64, P, P])
    lib = _lib.load()
    for name in ("nerfb200_bake_f16", "nerfb200_baked_render_f16", "nerfb200_baked_max_weights_f16"):
        assert hasattr(lib, name)
    # their fp32 twins keep their signatures
    assert _lib.SIGNATURES["nerfb200_bake"] == _lib.SIGNATURES["nerfb200_bake_f16"]
    assert _lib.SIGNATURES["nerfb200_baked_render"] == _lib.SIGNATURES["nerfb200_baked_render_f16"]
    assert _lib.SIGNATURES["nerfb200_baked_max_weights"] == _lib.SIGNATURES["nerfb200_baked_max_weights_f16"]


def test_fp16_entry_points_refuse_before_any_launch():
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    before = ops.launch_count()
    box = ops.grid_struct(BOX, (16, 16, 16))
    bad_box = ops.grid_struct(((1.0,) * 3, (-1.0,) * 3), (16, 16, 16))
    arch = ops.ArchSpec().c_struct()
    fake, odd = C.c_void_p(256), C.c_void_p(256 + 8)  # 16-B aligned and not
    nan = float("nan")
    bake = lib.nerfb200_bake_f16
    for args in ((None, box, fake, 0, 1, fake), (fake, box, None, 0, 1, fake), (fake, box, fake, 0, 1, None),
                 (fake, box, fake, 0, 9, fake), (fake, box, fake, -1, 1, fake), (fake, box, fake, 0, 0, fake),
                 (fake, box, fake, 7, 2, fake), (fake, bad_box, fake, 0, 1, fake), (fake, box, fake, 0, 1, odd)):
        blob, b, bricks, first, count, values = args
        assert bake(C.byref(arch), blob, C.byref(b), bricks, first, count, values, None, None) == _lib.ERR_INVALID, args
    wide = ops.ArchSpec(n_freq_xyz=16).c_struct()
    assert bake(C.byref(wide), fake, C.byref(box), fake, 0, 1, fake, None, None) == _lib.ERR_UNSUPPORTED
    r = lib.nerfb200_baked_render_f16
    for vd, stride, n, t, bm, vals, rays, out, b in (
            (1, 8, 4, 0.0, fake, fake, fake, fake, box),       # stride too short with view directions
            (0, 7, 4, 0.0, fake, fake, fake, fake, box),       # and without
            (0, 8, 4, 1.0, fake, fake, fake, fake, box),       # t outside [0, 1)
            (0, 8, 4, -0.1, fake, fake, fake, fake, box),
            (0, 8, 4, nan, fake, fake, fake, fake, box),
            (0, 8, 0, 0.0, fake, fake, fake, fake, box),       # no ray
            (0, 8, 4, 0.0, None, fake, fake, fake, box),       # null pointers
            (0, 8, 4, 0.0, fake, None, fake, fake, box),
            (0, 8, 4, 0.0, fake, fake, None, fake, box),
            (0, 8, 4, 0.0, fake, fake, fake, None, box),
            (0, 8, 4, 0.0, fake, fake, fake, fake, bad_box),   # invalid box
            (0, 8, 4, 0.0, fake, odd, fake, fake, box)):       # values not 16-B aligned
        assert r(C.byref(b), bm, vals, vd, rays, stride, n, 0, t, out, None) == _lib.ERR_INVALID, (vd, stride, n, t)
    w = lib.nerfb200_baked_max_weights_f16
    for vd, stride, n, bm, vals, rays, mw, b in (
            (1, 8, 4, fake, fake, fake, fake, box), (0, 7, 4, fake, fake, fake, fake, box),
            (0, 8, 0, fake, fake, fake, fake, box), (0, 8, 4, None, fake, fake, fake, box),
            (0, 8, 4, fake, None, fake, fake, box), (0, 8, 4, fake, fake, None, fake, box),
            (0, 8, 4, fake, fake, fake, None, box), (0, 8, 4, fake, fake, fake, fake, bad_box),
            (0, 8, 4, fake, odd, fake, fake, box)):
        assert w(C.byref(b), bm, vals, vd, rays, stride, n, mw, None) == _lib.ERR_INVALID, (vd, stride, n)
    assert "16-B aligned" in lib.nerfb200_last_error().decode()
    assert ops.launch_count() == before


# ------------------------------------------------------------------------------------------------------------------------
# the conversion rule on a CPU field
# ------------------------------------------------------------------------------------------------------------------------
# finite values around the fp16 range, the fp16 subnormals and fp32 subnormals, and the non-finite ones
EDGES = [0.0, -0.0, 1.0, -1.0, 1.0 / 3.0, 65504.0, -65504.0, 65505.0, 65519.99, -65519.99, 65520.0, -65520.0, 65536.0,
         1e6, -1e30, 3.4e38, -3.4e38, 2.0 ** -14, 2.0 ** -24, -2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -26, 1.5 * 2.0 ** -24,
         2.5 * 2.0 ** -24, 6e-8, -6e-8, 1e-8, 1e-40, -1e-40, 2049.0, 2051.0, float("inf"), float("-inf"), float("nan")]


def _field(values, bricks=None):
    import nerf_pytorch_b200 as nb

    n = values.shape[0]
    bricks = torch.arange(n, dtype=torch.int32) if bricks is None else bricks
    brick_map = torch.full((8,), -1, dtype=torch.int32)
    brick_map[bricks.long()] = torch.arange(n, dtype=torch.int32)
    return nb.BakedField(BOX, (16, 16, 16), brick_map, bricks, values, True)


def _edge_values(seed=0):
    """fp32 [3, 729, 32]: random values over a wide range with EDGES spread over channels 0 .. 27, channels 28 .. 31 0."""
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(3, 729, 32, generator=g) * torch.exp(8 * torch.randn(3, 729, 32, generator=g))
    e = torch.tensor(EDGES, dtype=torch.float32)
    flat = v[..., :28].reshape(-1)
    idx = torch.randperm(flat.numel(), generator=g)[:40 * e.numel()]
    flat[idx] = e.repeat(40)
    v[..., :28] = flat.view(3, 729, 28)
    v[..., 28:] = 0
    return v


def _rule_numpy(x):
    """The header's rule restated in numpy (numpy's own fp16 rounding)."""
    x = x.numpy()
    with np.errstate(over="ignore", invalid="ignore"):
        return np.where(np.isfinite(x), np.clip(x, -65504, 65504), x).astype(np.float16)


def test_half_applies_the_conversion_rule():
    v = _edge_values()
    f = _field(v)
    h = f.half(chunk=2)  # a chunk that does not divide n_active
    assert h.dtype == torch.float16 and f.dtype == torch.float32
    assert h.brick_map is f.brick_map and h.bricks is f.bricks and h.values.shape == v.shape
    got = h.values.view(torch.int16).numpy()
    want = _rule_numpy(v)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(h.values.float().numpy()), nan)  # NaN stays NaN (payload unspecified)
    assert np.array_equal(got[~nan], want.view(np.int16)[~nan])
    # and the torch restatement of the header gives the same bits
    t = torch.where(v.isfinite(), v.clamp(-65504, 65504), v).half()
    assert torch.equal(t.view(torch.int16)[~torch.from_numpy(nan)], h.values.view(torch.int16)[~torch.from_numpy(nan)])


def test_saturation_infinities_and_subnormals():
    x = torch.tensor(EDGES, dtype=torch.float32)
    v = torch.zeros(1, 729, 32)
    v[0, :x.numel(), 0] = x
    h = _field(v).half().values[0, :x.numel(), 0]
    bits = h.view(torch.int16)
    for val, b, w in zip(EDGES, bits.tolist(), h.float().tolist()):
        if val != val:
            assert w != w
        elif abs(val) == float("inf"):
            assert w == val
        elif abs(val) > 65504:  # saturates, whether round-to-nearest would give 65504 (below 65520) or inf
            assert w == (65504.0 if val > 0 else -65504.0) and (b & 0x7FFF) == 0x7BFF, val
        else:
            assert abs(w) < float("inf")
    sub = {2.0 ** -24: 2.0 ** -24, 2.0 ** -25: 0.0, 3 * 2.0 ** -26: 2.0 ** -24, 1.5 * 2.0 ** -24: 2 * 2.0 ** -24,
           2.5 * 2.0 ** -24: 2 * 2.0 ** -24, 1e-40: 0.0, 2051.0: 2052.0, 2049.0: 2048.0}  # ties to even
    for val, want in sub.items():
        assert h.float()[EDGES.index(val)].item() == want, val
    # signed zeros survive: -1e-40 and -0 round to -0
    assert bits[EDGES.index(-1e-40)].item() == -32768 and bits[1].item() == -32768  # EDGES[1] is -0.0
    assert not torch.isinf(h[[i for i, e in enumerate(EDGES) if abs(e) < float("inf")]]).any()


def test_channels_28_to_31_stay_zero_and_float_is_exact():
    v = _edge_values(1)
    h = _field(v).half()
    assert (h.values[..., 28:].view(torch.int16) == 0).all()
    w = h.float()
    assert w.dtype == torch.float32 and w.brick_map is h.brick_map and w.bricks is h.bricks
    want = h.values.numpy().astype(np.float32)  # numpy's exact widening
    assert np.array_equal(w.values.numpy().view(np.int32)[~np.isnan(want)], want.view(np.int32)[~np.isnan(want)])
    assert np.array_equal(np.isnan(w.values.numpy()), np.isnan(want))
    again = w.half()
    assert torch.equal(again.values.view(torch.int16), h.values.view(torch.int16))  # half().float().half() is a fixed point
    f = _field(v)
    assert f.float().values is f.values  # an fp32 field's own tensor, as torch's .float()


def test_repr_counts_the_element_size():
    f = _field(torch.zeros(20, 729, 32), torch.zeros(20, dtype=torch.int32))
    assert "1.8 MiB," in repr(f) and "0.9 MiB fp16," in repr(f.half())


def test_prune_and_transparency_keep_the_dtype():
    import nerf_pytorch_b200 as nb

    v = torch.randn(3, 729, 32)
    v[..., 28:] = 0
    v[0, :, 0] = -torch.rand(729)      # transparent
    v[1, :, 0] = -torch.rand(729)
    v[1, 5, 3] = float("inf")           # not transparent: a non-finite coefficient
    v[2, :, 0] = -1e6                   # transparent, saturates to -65504
    h = _field(v).half()
    mask = nb.baked_transparent_bricks(h)
    assert torch.equal(mask, nb.baked_transparent_bricks(h.float())) and mask.tolist() == [True, False, True]
    p = nb.prune_baked(h, ~mask)
    assert p.dtype == torch.float16 and p.n_active == 1
    assert torch.equal(p.values.view(torch.int16), h.values[1:2].view(torch.int16))
    assert p.brick_map.tolist() == [-1, 0, -1, -1, -1, -1, -1, -1]


def test_save_and_load_keep_dtype_and_bits(tmp_path):
    import nerf_pytorch_b200 as nb

    h = _field(_edge_values(2)).half()
    h.save(tmp_path / "f.pt")
    g = nb.BakedField.load(tmp_path / "f.pt", device="cpu")
    assert g.dtype == torch.float16 and torch.equal(g.values.view(torch.int16), h.values.view(torch.int16))
    assert torch.equal(g.brick_map, h.brick_map) and torch.equal(g.bricks, h.bricks)


def test_python_refusals_precede_any_launch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    before = ops.launch_count()
    m = nb.FlexibleNeRFModel()
    epf = nb.get_embedding_function(6)
    for dt in (torch.bfloat16, torch.float64, torch.int16, "float16"):
        with pytest.raises(ValueError, match="dtype"):
            nb.bake(m, epf, bounds=BOX, resolution=16, grid=None, dtype=dt)
    for chunk in (0, -3):
        with pytest.raises(ValueError, match="chunk"):
            _field(torch.zeros(1, 729, 32)).half(chunk=chunk)
    h = _field(torch.zeros(1, 729, 32)).half()
    with pytest.raises(ValueError, match=r"float\(\)"):
        nb.baked_regularizer(h, tv_sigma=1.0)
    opts = O.make_options()
    imgs, poses = torch.zeros(2, 8, 8, 3), torch.zeros(2, 4, 4)
    with pytest.raises(ValueError, match=r"float\(\)"):
        nb.BakedFieldTrainer(h, imgs, poses, 10.0, opts)
    h.values.requires_grad_(True)
    with pytest.raises(ValueError):
        nb.render_baked_rays(h, torch.zeros(4, 11))
    with torch.no_grad():
        with pytest.raises(ValueError):  # CPU values
            nb.render_baked_rays(_field(torch.zeros(1, 729, 32)).half(), torch.zeros(4, 11))
    # the dispatch refuses any other dtype before reaching a pointer
    box = ops.grid_struct(BOX, (16, 16, 16))
    bm = torch.zeros(8, dtype=torch.int32)
    for dt in (torch.bfloat16, torch.float64):
        with pytest.raises(ValueError, match="fp32 or fp16"):
            ops.baked_render(box, bm, torch.zeros(1, 729, 32, dtype=dt), True, torch.zeros(4, 11), False)
        with pytest.raises(ValueError, match="fp32 or fp16"):
            ops.baked_max_weights(box, bm, torch.zeros(1, 729, 32, dtype=dt), True, torch.zeros(4, 11), torch.zeros(1))
    assert ops.launch_count() == before
