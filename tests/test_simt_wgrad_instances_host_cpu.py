"""CPU: the fp32 kernel tests reach every instance of the weight-gradient kernel's register tile.

mlp_bwd_wgrad_kernel (mlp_simt.cu) runs one item of wg_decode's list (wgrad_items.cuh) per blockIdx.y and picks one of
14 wgrad_block<RN, RK> instances from the item's shape: RN = 8 for blocks of more than 64 output rows, else 4; RK =
kblk / 16 for 2..7, and the default case, 8, for every other value (kblk 128 of the hidden columns, and encodings of at
most 16 columns).  Which instances a model reaches depends only on its layer shapes, so a table of architectures can
silently stop reaching one.  This restates the item rule and the switch and asserts that the architectures
test_simt_mlp_gpu.py checks against fp64 (mlp_checks.SIMT_NAMES) reach all 14, and that every hidden-128 entry among
them is one the wgmma training path refuses, so that the fp32 kernels are what trains it."""
import pytest

from mlp_checks import H256_ARCHS, SIMT128_ARCHS, SIMT_NAMES, spec

ALL_INSTANCES = {(rn, rk) for rn in (4, 8) for rk in range(2, 9)}


def wgrad_items(arch):
    """wg_decode restated: (nblk, kblk) of every gemm-layer item, in order.  A layer of n outputs, k_h hidden inputs and
    enc_real encoding inputs has ceil(n / 128) row blocks, each with ceil(k_h / 128) hidden-column items of up to 128
    columns and, if enc_real > 0, one encoding item of enc_real padded to 16 columns."""
    items = []
    for name, _, _, fin, fout in arch.flat_layout():
        if fout < 64:  # fc_alpha / fc_rgb / fc_out: head items, reduced by wgrad_head
            continue
        k_h = 0 if name == "layer1" else arch.hidden
        enc_real = fin - k_h
        for n0 in range(0, fout, 128):
            nblk = min(128, fout - n0)
            items += [(nblk, min(128, k_h - k0)) for k0 in range(0, k_h, 128)]
            if enc_real > 0:
                items.append((nblk, (enc_real + 15) & ~15))
    return items


def instance(nblk, kblk):
    """The NB_WG switch of mlp_bwd_wgrad_kernel: (RN, RK) of an item."""
    rk = kblk // 16
    return (8 if nblk > 64 else 4, rk if 2 <= rk <= 7 else 8)


def instances(name):
    return {instance(*it) for it in wgrad_items(spec(name))}


def test_restated_items_of_known_architectures():
    """The rule on two architectures worked by hand.  8 x 256: layer1 (2 row blocks x the 63-column encoding), six
    narrow layers (2 x 2 hidden items), one wide layer (2 x 3), fc_feat (2 x 2), layers_dir.0 (128 rows: 2 hidden items
    and the 27-column direction encoding) = 39 gemm items.  8 x 128 with 16 / 16 bands: 99 columns pad to 112 (RK 7) for
    layer1, the wide layer and the 64-row layers_dir.0."""
    items = wgrad_items(spec("8x256"))
    assert len(items) == 39
    assert {instance(*it) for it in items} == {(8, 8), (8, 4), (8, 2)}
    items = wgrad_items(spec("8x128_lxyz16_ldir16"))
    assert items == [(128, 112)] + [(128, 128)] * 4 + [(128, 128), (128, 112)] + [(128, 128)] * 3 + [(64, 128),
                                                                                                      (64, 112)]
    assert {instance(*it) for it in items} == {(8, 7), (8, 8), (4, 8), (4, 7)}
    assert instance(128, 16) == instance(128, 128) == (8, 8)  # kblk 16: rk 1 takes the default case


def test_fp32_test_tables_reach_every_wgrad_instance():
    reached = {}
    for name in SIMT_NAMES:
        for inst in instances(name):
            reached.setdefault(inst, []).append(name)
    missing = ALL_INSTANCES - set(reached)
    assert not missing, sorted(missing)


def test_hidden256_table_alone_misses_the_wide_encoding_instances():
    """Why SIMT128_ARCHS exists: at hidden 256 every block has 128 rows and the encodings are at most 63 columns, so the
    hidden-256 table reaches 4 of the 14 instances."""
    reached = set().union(*(instances(name) for name in H256_ARCHS))
    assert reached == {(8, 2), (8, 3), (8, 4), (8, 8)}


@pytest.mark.parametrize("name", list(SIMT128_ARCHS))
def test_hidden128_table_trains_on_the_fp32_kernels(name):
    """impl 0 takes every SIMT128_ARCHS entry and the wgmma training path (impl 1) refuses it, so run_one_iter_of_nerf
    trains it on the kernels test_simt_mlp_gpu.py checks."""
    from nerf_pytorch_b200 import ops, train_utils

    arch = spec(name)
    assert arch.hidden == 128
    assert ops.impl_supported(arch, 64, ops.IMPL_SIMT), ops.impl_refusal(arch, 64, ops.IMPL_SIMT)
    assert not ops.impl_supported(arch, 64, ops.IMPL_TC)
    assert train_utils._auto_impl(arch, arch, 64, 64, training=True) == ops.IMPL_SIMT
