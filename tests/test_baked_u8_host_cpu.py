"""Host: 8-bit baked fields (include/nerfb200.h "baked fields: 8-bit values").  The quantisation rule of
BakedField.quantize and the dequantisation of BakedField.float against a numpy restatement, the properties the rule
promises (exact zero, sigma_raw <= 0 kept <= 0, bit-equal copies), pruning, transparency, repr and save / load of an
8-bit field, the four uint8 entry points' ABI and refusals, and the Python refusals.  No GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

BOX = ((-1.0,) * 3, (1.0,) * 3)


def _field(values, bricks=None, res=(16, 16, 16), viewdirs=True):
    import nerf_pytorch_b200 as nb

    n = values.shape[0]
    nbk = [-(-r // 8) for r in res]
    bricks = torch.arange(n, dtype=torch.int32) if bricks is None else bricks
    brick_map = torch.full((nbk[0] * nbk[1] * nbk[2],), -1, dtype=torch.int32)
    brick_map[bricks.long()] = torch.arange(n, dtype=torch.int32)
    return nb.BakedField(BOX, res, brick_map, bricks, values, viewdirs)


def _values(seed=0, n=3):
    """fp32 [n, 729, 32]: channel 0 in [-4, 8] (sigma_raw), channel 1 all positive, channel 2 all negative, channel 3
    constant 0, channel 4 constant 2.5, channels 5 .. 27 normal over several magnitudes, channels 28 .. 31 zero; a few
    exact zeros and negative zeros."""
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(n, 729, 32, generator=g) * torch.exp(3 * torch.randn(1, 1, 32, generator=g))
    v[..., 0] = -4 + 12 * torch.rand(n, 729, generator=g)
    v[..., 1] = 0.5 + torch.rand(n, 729, generator=g)
    v[..., 2] = -0.5 - torch.rand(n, 729, generator=g)
    v[..., 3] = 0.0
    v[..., 4] = 2.5
    v[..., 28:] = 0
    v[0, :7, 5:28] = 0.0
    v[1, :7, 5:28] = -0.0
    return v


def _rule_numpy(v):
    """(codes uint8 [.., 32], scale [28], offset [28]): the header's rule restated in numpy fp32."""
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


def _dequant_numpy(q, s, o):
    out = np.zeros(q.shape, dtype=np.float32)
    out[..., :28] = (q[..., :28].astype(np.float32) * s).astype(np.float32) + o
    return out


def _bits(x):
    return np.asarray(x, dtype=np.float32).view(np.int32)


# ------------------------------------------------------------------------------------------------------------------------
# the rule on CPU fields
# ------------------------------------------------------------------------------------------------------------------------
def test_quantize_applies_the_rule():
    v = _values()
    f = _field(v)
    q = f.quantize(chunk=2)  # a chunk that does not divide n_active
    assert q.dtype == torch.uint8 and f.dtype == torch.float32 and f.dequant is None
    assert q.brick_map is f.brick_map and q.bricks is f.bricks and q.values.shape == v.shape
    assert q.dequant.dtype == torch.float32 and q.dequant.shape == (2, 28)
    codes, s, o = _rule_numpy(v)
    assert np.array_equal(_bits(q.dequant[0]), _bits(s)) and np.array_equal(_bits(q.dequant[1]), _bits(o))
    assert np.array_equal(q.values.numpy(), codes)
    assert (q.values[..., 28:] == 0).all()
    # the chunking does not matter
    assert torch.equal(f.quantize().values, q.values) and torch.equal(f.quantize(chunk=1).dequant, q.dequant)


def test_float_dequantises_exactly():
    q = _field(_values(1)).quantize()
    w = q.float()
    assert w.dtype == torch.float32 and w.dequant is None and w.brick_map is q.brick_map and w.bricks is q.bricks
    want = _dequant_numpy(q.values.numpy(), q.dequant[0].numpy(), q.dequant[1].numpy())
    assert np.array_equal(_bits(w.values), _bits(want))
    # torch's restatement of the header gives the same bits, and the chunking does not matter
    t = q.values[..., :28].float() * q.dequant[0] + q.dequant[1]
    assert torch.equal(w.values[..., :28].view(torch.int32), t.view(torch.int32))
    assert torch.equal(q.float(chunk=2).values.view(torch.int32), w.values.view(torch.int32))
    assert (w.values[..., 28:].view(torch.int32) == 0).all()
    # the dequantised values lie within half a step of the originals (plus rounding)
    v = _values(1)
    err = (w.values[..., :28] - v[..., :28]).abs() / q.dequant[0]
    assert float(err.max()) <= 0.5 + 1e-3


def test_saturation_at_codes_0_and_255_and_the_zero_point():
    v = _values(2)
    q = _field(v).quantize()
    codes, s, o = q.values.long(), q.dequant[0], q.dequant[1]
    z = torch.round(-(o / s))
    # sigma_raw spans [-4, 8]: its minimum takes code 0 and its maximum code 255
    assert int(codes[..., 0].min()) == 0 and int(codes[..., 0].max()) == 255
    # the all-positive channel: lo = 0, zero point 0, offset -0, its maximum at code 255; the all-negative one: hi = 0
    # (0 is in the range though no value reaches it), zero point 255, its minimum at code 0 and every value below z
    assert float(z[1]) == 0 and int(codes[..., 1].max()) == 255 and int(codes[..., 1].min()) > 0
    assert float(z[2]) == 255 and int(codes[..., 2].min()) == 0 and int(codes[..., 2].max()) < 255
    # the constant-0 channel: scale 1, zero point +0 so offset -0, every code 0, dequantised +0
    assert float(s[3]) == 1.0 and int(codes[..., 3].max()) == 0 and int(o[3:4].view(torch.int32)) == -2 ** 31
    w = q.float().values
    assert (w[..., 3].view(torch.int32) == 0).all()
    # the constant 2.5 channel: lo = 0, scale 2.5 / 255, every code 255
    assert float(s[4]) == float(np.float32(2.5) / np.float32(255)) and bool((codes[..., 4] == 255).all())
    # every channel's extremes land on the clamp's bounds or inside them, never wrapped
    assert bool((w[..., 1:3] * torch.tensor([1.0, -1.0]) >= 0).all())


def test_zero_is_exact_and_sigma_raw_at_most_0_stays_at_most_0():
    v = _values(3)
    q = _field(v).quantize()
    w = q.float().values
    zero = v[..., :28] == 0  # +0 and -0
    assert bool(zero.any())
    assert (w[..., :28][zero].view(torch.int32) == 0).all()  # +0 exactly
    s, o = q.dequant
    z = torch.round(-(o / s)).long()
    assert torch.equal(q.values[..., :28][zero].long(), z.expand(*zero.shape)[zero])
    nonpos = v[..., 0] <= 0
    assert bool(nonpos.any()) and bool((w[..., 0][nonpos] <= 0).all())
    assert bool((q.values[..., 0][nonpos].long() <= z[0]).all())


def test_fp16_field_quantizes_as_its_widened_field():
    f = _field(_values(4)).half()
    a, b = f.quantize(), f.float().quantize()
    assert torch.equal(a.values, b.values) and torch.equal(a.dequant.view(torch.int32), b.dequant.view(torch.int32))


def _lattice_index(field):
    """int64 [n_active, 729]: the linear lattice index each stored value holds (tests/helpers.lattice_index on CPU)."""
    res = torch.tensor(field.resolution)
    nbk = (res + 7) // 8
    br = field.bricks.long()
    b = torch.stack([br % nbk[0], br // nbk[0] % nbk[1], br // (nbk[0] * nbk[1])], -1)
    p = torch.arange(729)
    l = torch.stack([p % 9, p // 9 % 9, p // 81], -1)
    qi = torch.minimum(b[:, None] * 8 + l[None], res)
    return (qi[..., 2] * (res[1] + 1) + qi[..., 1]) * (res[0] + 1) + qi[..., 0]


def test_copies_stay_bit_equal():
    from helpers import copies_bit_equal

    res = (20, 17, 12)
    nbk = [-(-r // 8) for r in res]
    bricks = torch.tensor([0, 1, 2, 4, 5, 7, 9, 10, 11, 17], dtype=torch.int32)
    assert int(bricks.max()) < nbk[0] * nbk[1] * nbk[2]
    f = _field(torch.zeros(bricks.numel(), 729, 32), bricks, res)
    idx = _lattice_index(f)
    g = torch.Generator().manual_seed(5)
    dense = torch.randn(int(idx.max()) + 1, 32, generator=g) * 3
    dense[:, 28:] = 0
    f.values = dense[idx].contiguous()
    assert copies_bit_equal(f.values, idx)
    q = f.quantize(chunk=3)
    assert copies_bit_equal(q.values.float(), idx)  # one code per fp32 element: every channel's code compared
    assert copies_bit_equal(q.float().values, idx)


# ------------------------------------------------------------------------------------------------------------------------
# pruning, transparency, repr, save / load
# ------------------------------------------------------------------------------------------------------------------------
def test_prune_and_transparency_on_an_8bit_field():
    import nerf_pytorch_b200 as nb

    v = _values(6)
    v[0, :, 0] = -torch.rand(729)  # transparent
    v[2, :, 0] = -3.0              # transparent
    v[2, 17, 0] = 0.0
    q = _field(v).quantize()
    mask = nb.baked_transparent_bricks(q)
    assert mask.tolist() == [True, False, True]
    assert torch.equal(mask, nb.baked_transparent_bricks(q.float()))
    p = nb.prune_baked(q, ~mask)
    assert p.dtype == torch.uint8 and p.n_active == 1 and p.dequant is q.dequant
    assert torch.equal(p.values, q.values[1:2])
    assert p.brick_map.tolist() == [-1, 0, -1, -1, -1, -1, -1, -1]


def test_repr_marks_the_field_8bit():
    f = _field(torch.zeros(20, 729, 32), torch.zeros(20, dtype=torch.int32))
    assert "1.8 MiB," in repr(f) and "0.4 MiB 8-bit," in repr(f.quantize())


def test_save_and_load_keep_the_codes_and_dequant(tmp_path):
    import nerf_pytorch_b200 as nb

    q = _field(_values(7)).quantize()
    q.save(tmp_path / "q.pt")
    g = nb.BakedField.load(tmp_path / "q.pt", device="cpu")
    assert g.dtype == torch.uint8 and torch.equal(g.values, q.values)
    assert torch.equal(g.dequant.view(torch.int32), q.dequant.view(torch.int32))
    assert torch.equal(g.brick_map, q.brick_map) and torch.equal(g.bricks, q.bricks)
    # an fp32 field saves dequant None
    f = _field(_values(7))
    f.save(tmp_path / "f.pt")
    assert nb.BakedField.load(tmp_path / "f.pt", device="cpu").dequant is None
    # a file written before 8-bit fields (no "dequant" key) still loads
    torch.save({"bounds": f.bounds, "resolution": f.resolution, "brick_map": f.brick_map, "bricks": f.bricks,
                "values": f.values.half(), "use_viewdirs": True}, tmp_path / "old.pt")
    old = nb.BakedField.load(tmp_path / "old.pt", device="cpu")
    assert old.dequant is None and old.dtype == torch.float16 and torch.equal(old.values, f.values.half())


# ------------------------------------------------------------------------------------------------------------------------
# the C ABI
# ------------------------------------------------------------------------------------------------------------------------
def test_signatures_of_the_uint8_entry_points():
    from nerf_pytorch_b200 import _lib

    GP, P = C.POINTER(_lib.Grid), C.c_void_p
    I32, I64, F32 = C.c_int32, C.c_int64, C.c_float
    sig = _lib.SIGNATURES
    assert sig["nerfb200_baked_render_u8"] == (I32, [GP, P, P, P, I32, P, I32, I64, I32, F32, P, P])
    assert sig["nerfb200_baked_max_weights_u8"] == (I32, [GP, P, P, P, I32, P, I32, I64, P, P])
    assert sig["nerfb200_baked_mesh_dirs_u8"] == (I32, [GP, P, P, P, F32, P, I64, P, P, P])
    assert sig["nerfb200_baked_mesh_colors_u8"] == (I32, [GP, P, P, P, I32, F32, P, P, I64, P, P])
    lib = _lib.load()
    for name in ("render", "max_weights", "mesh_dirs", "mesh_colors"):
        assert hasattr(lib, f"nerfb200_baked_{name}_u8")
        # the fp32 twin's arguments with dequant after values
        twin = sig[f"nerfb200_baked_{name}"][1]
        assert sig[f"nerfb200_baked_{name}_u8"][1] == twin[:3] + [P] + twin[3:]


def test_uint8_entry_points_refuse_before_any_launch():
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    before = ops.launch_count()
    box = ops.grid_struct(BOX, (16, 16, 16))
    bad_box = ops.grid_struct(((1.0,) * 3, (-1.0,) * 3), (16, 16, 16))
    fake, odd = C.c_void_p(256), C.c_void_p(256 + 8)  # 16-B aligned and not
    nan = float("nan")
    r = lib.nerfb200_baked_render_u8
    for vd, stride, n, t, bm, vals, dq, rays, out, b in (
            (1, 8, 4, 0.0, fake, fake, fake, fake, fake, box),       # stride too short with view directions
            (0, 7, 4, 0.0, fake, fake, fake, fake, fake, box),       # and without
            (0, 8, 4, 1.0, fake, fake, fake, fake, fake, box),       # t outside [0, 1)
            (0, 8, 4, nan, fake, fake, fake, fake, fake, box),
            (0, 8, 0, 0.0, fake, fake, fake, fake, fake, box),       # no ray
            (0, 8, 4, 0.0, None, fake, fake, fake, fake, box),       # null pointers
            (0, 8, 4, 0.0, fake, None, fake, fake, fake, box),
            (0, 8, 4, 0.0, fake, fake, fake, None, fake, box),
            (0, 8, 4, 0.0, fake, fake, fake, fake, None, box),
            (0, 8, 4, 0.0, fake, fake, fake, fake, fake, bad_box),   # invalid box
            (0, 8, 4, 0.0, fake, odd, fake, fake, fake, box),        # codes not 16-B aligned
            (0, 8, 4, 0.0, fake, fake, None, fake, fake, box)):      # no dequant
        assert r(C.byref(b), bm, vals, dq, vd, rays, stride, n, 0, t, out, None) == _lib.ERR_INVALID, (vd, stride, n)
    assert "dequant" in lib.nerfb200_last_error().decode()
    w = lib.nerfb200_baked_max_weights_u8
    for vd, stride, n, bm, vals, dq, rays, mw, b in (
            (1, 8, 4, fake, fake, fake, fake, fake, box), (0, 7, 4, fake, fake, fake, fake, fake, box),
            (0, 8, 0, fake, fake, fake, fake, fake, box), (0, 8, 4, None, fake, fake, fake, fake, box),
            (0, 8, 4, fake, None, fake, fake, fake, box), (0, 8, 4, fake, fake, fake, None, fake, box),
            (0, 8, 4, fake, fake, fake, fake, None, box), (0, 8, 4, fake, fake, fake, fake, fake, bad_box),
            (0, 8, 4, fake, odd, fake, fake, fake, box), (0, 8, 4, fake, fake, None, fake, fake, box)):
        assert w(C.byref(b), bm, vals, dq, vd, rays, stride, n, mw, None) == _lib.ERR_INVALID, (vd, stride, n)
    d = lib.nerfb200_baked_mesh_dirs_u8
    for bm, vals, dq, level, keys, n, dirs, b in (
            (None, fake, fake, 1.0, fake, 4, fake, box), (fake, None, fake, 1.0, fake, 4, fake, box),
            (fake, fake, fake, 1.0, None, 4, fake, box), (fake, fake, fake, 1.0, fake, 4, None, box),
            (fake, fake, fake, 1.0, fake, -1, fake, box), (fake, fake, fake, nan, fake, 4, fake, box),
            (fake, fake, fake, float("inf"), fake, 4, fake, box), (fake, fake, fake, 1.0, fake, 4, fake, bad_box),
            (fake, odd, fake, 1.0, fake, 4, fake, box), (fake, fake, None, 1.0, fake, 4, fake, box)):
        assert d(C.byref(b), bm, vals, dq, level, keys, n, dirs, None, None) == _lib.ERR_INVALID, (level, n)
    c = lib.nerfb200_baked_mesh_colors_u8
    for bm, vals, dq, vd, level, keys, dirs, n, cols, b in (
            (None, fake, fake, 0, 1.0, fake, None, 4, fake, box), (fake, None, fake, 0, 1.0, fake, None, 4, fake, box),
            (fake, fake, fake, 0, 1.0, None, None, 4, fake, box), (fake, fake, fake, 0, 1.0, fake, None, 4, None, box),
            (fake, fake, fake, 1, 1.0, fake, None, 4, fake, box),  # view directions without dirs
            (fake, fake, fake, 0, 1.0, fake, None, -1, fake, box), (fake, fake, fake, 0, nan, fake, None, 4, fake, box),
            (fake, fake, fake, 0, 1.0, fake, None, 4, fake, bad_box), (fake, odd, fake, 0, 1.0, fake, None, 4, fake, box),
            (fake, fake, None, 0, 1.0, fake, None, 4, fake, box)):
        assert c(C.byref(b), bm, vals, dq, vd, level, keys, dirs, n, cols, None) == _lib.ERR_INVALID, (vd, level, n)
    assert ops.launch_count() == before


# ------------------------------------------------------------------------------------------------------------------------
# Python refusals
# ------------------------------------------------------------------------------------------------------------------------
def test_python_refusals_precede_any_launch():
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops
    from oracle import nerf_oracle as O

    before = ops.launch_count()
    q = _field(_values(8)).quantize()
    with pytest.raises(ValueError, match=r"float\(\)"):
        q.half()
    with pytest.raises(ValueError, match=r"float\(\)"):
        q.quantize()
    for chunk in (0, -3):
        with pytest.raises(ValueError, match="chunk"):
            _field(_values(8)).quantize(chunk=chunk)
        with pytest.raises(ValueError, match="chunk"):
            q.float(chunk=chunk)
    for bad in (float("nan"), float("inf"), float("-inf")):
        v = _values(8)
        v[1, 100, 17] = bad
        with pytest.raises(ValueError, match="finite"):
            _field(v).quantize()
    v = _values(8)  # a range that overflows fp32
    v[0, 0, 6], v[0, 1, 6] = 3e38, -3e38
    with pytest.raises(ValueError, match="fp32"):
        _field(v).quantize()
    v = _values(8)  # non-finite values in channels 28 .. 31 are never read
    v[..., 30] = float("nan")
    assert torch.equal(_field(v).quantize().values, _field(_values(8)).quantize().values)
    # fine-tuning, the regulariser and subdivision name float()
    opts = O.make_options()
    imgs, poses = torch.zeros(2, 8, 8, 3), torch.zeros(2, 4, 4)
    with pytest.raises(ValueError, match=r"float\(\)"):
        nb.BakedFieldTrainer(q, imgs, poses, 10.0, opts)
    with pytest.raises(ValueError, match=r"float\(\)"):
        nb.baked_regularizer(q, tv_sigma=1.0)
    with pytest.raises(ValueError, match=r"float\(\)"):
        nb.subdivide_baked(q)
    # a CPU field has no render (the grad-mode refusal is pinned on the GPU); bake writes no codes
    with pytest.raises(ValueError):
        nb.render_baked_rays(q, torch.zeros(4, 11))
    box = ops.grid_struct(BOX, (16, 16, 16))
    with pytest.raises(ValueError, match="quantise"):
        ops.bake(ops.ArchSpec(), torch.zeros(4), box, torch.zeros(1, dtype=torch.int32), 0, 1,
                 torch.zeros(1, 729, 32, dtype=torch.uint8))
    # the dispatch wants uint8 codes' dequant: missing, of the wrong shape or dtype
    bm = torch.zeros(8, dtype=torch.int32)
    codes = torch.zeros(1, 729, 32, dtype=torch.uint8)
    for dq in (None, torch.zeros(28), torch.zeros(2, 28, dtype=torch.float64), torch.zeros(2, 32)):
        with pytest.raises(ValueError, match="dequant"):
            ops.baked_render(box, bm, codes, True, torch.zeros(4, 11), False, dequant=dq)
        with pytest.raises(ValueError, match="dequant"):
            ops.baked_max_weights(box, bm, codes, True, torch.zeros(4, 11), torch.zeros(1), dequant=dq)
        with pytest.raises(ValueError, match="dequant"):
            ops.baked_mesh_dirs(box, bm, codes, 1.0, torch.zeros(4, dtype=torch.int64), dequant=dq)
        with pytest.raises(ValueError, match="dequant"):
            ops.baked_mesh_colors(box, bm, codes, False, 1.0, torch.zeros(4, dtype=torch.int64), dequant=dq)
    for dt in (torch.bfloat16, torch.float64, torch.int8):
        with pytest.raises(ValueError, match="fp32 or fp16"):
            ops.baked_render(box, bm, torch.zeros(1, 729, 32, dtype=dt), True, torch.zeros(4, 11), False)
    assert ops.launch_count() == before
