"""CPU: the library's answers about which impl codes it runs, from the plan alone.  0 is the fp32 CUDA-core family,
1 wgmma, 3 the single-pass fp16 forward; 2 asks impl_supported for the wgmma forward alone; every other code is
refused."""
import ctypes as C

import pytest


def test_fp32_support_query_refuses_a_forward_that_exceeds_shared_memory():
    """8 x 256 with L_dir 7 needs 232 512 B of shared memory in the fp32 forward, which refuses it; L_dir 6 fits."""
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    fits = ops.ArchSpec(num_layers=8, hidden=256, n_freq_xyz=10, n_freq_dir=6)
    wider = ops.ArchSpec(num_layers=8, hidden=256, n_freq_xyz=10, n_freq_dir=7)
    assert lib.nerfb200_impl_supported(C.byref(fits.c_struct()), 64, ops.IMPL_SIMT) == _lib.OK
    assert lib.nerfb200_impl_supported(C.byref(wider.c_struct()), 64, ops.IMPL_SIMT) == _lib.ERR_UNSUPPORTED
    why = lib.nerfb200_last_error().decode()
    assert "impl=0" in why and "shared memory" in why, why


def test_hidden128_widest_encodings_run_on_the_fp32_kernels_only():
    """8 x 128 with 16 xyz and 16 direction bands (NERFB200_MAX_FREQS, 99 channels each): the fp32 forward fits it
    (213 568 B of shared memory), and every wgmma code refuses encodings wider than 64 xyz / 32 direction channels."""
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    arch = ops.ArchSpec(num_layers=8, hidden=128, n_freq_xyz=16, n_freq_dir=16)
    assert lib.nerfb200_impl_supported(C.byref(arch.c_struct()), 64, ops.IMPL_SIMT) == _lib.OK
    for impl in (1, 2, 3):
        assert lib.nerfb200_impl_supported(C.byref(arch.c_struct()), 64, impl) == _lib.ERR_UNSUPPORTED, impl
        why = lib.nerfb200_last_error().decode()
        assert f"impl={1 if impl == 2 else impl}" in why and "encodings wider than 64" in why, (impl, why)


@pytest.mark.parametrize("impl", [2, 4, -1])
def test_backward_scratch_query_refuses_codes_that_have_no_backward(impl):
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    a = C.byref(ops.ArchSpec().c_struct())
    assert lib.nerfb200_bwd_scratch_floats(a, 4096, ops.IMPL_SIMT) == ops.stash_floats(ops.ArchSpec(), 4096)
    assert lib.nerfb200_bwd_scratch_floats(a, 4096, impl) == -1
    assert f"unknown impl {impl}" in lib.nerfb200_last_error().decode()


@pytest.mark.parametrize("impl", [-1, 4, 7])
def test_support_query_calls_codes_outside_0_to_3_invalid(impl):
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    for n_samples in (15, 64):
        assert lib.nerfb200_impl_supported(C.byref(ops.ArchSpec().c_struct()), n_samples, impl) == _lib.ERR_INVALID
        assert f"unknown impl {impl}" in lib.nerfb200_last_error().decode()
    assert not ops.impl_supported(ops.ArchSpec(), 64, impl)
