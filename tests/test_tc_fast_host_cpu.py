"""CPU: where the single-pass fp16 wgmma forward (impl 3, ops.IMPL_TC_FAST) is accepted and where it is refused.  These
answers come from the library's plan alone, so they need no GPU."""
import ctypes as C

import pytest
import torch


def _supported_with_reason(arch, n_samples, impl):
    from nerf_pytorch_b200 import _lib

    lib = _lib.load()
    rc = lib.nerfb200_impl_supported(C.byref(arch.c_struct()), n_samples, impl)
    return rc, lib.nerfb200_last_error().decode() if rc else ""


def test_fast_forward_is_accepted_exactly_where_the_wgmma_inference_forward_is():
    """impl_supported(arch, n, 3) == impl_supported(arch, n, 2) over hidden 128 / 256, 1..16 layers, every xyz band count,
    with and without view directions, at 14 (refused), 15 and 64 samples; a refusal gives the same reason."""
    from nerf_pytorch_b200 import ops

    assert ops.IMPL_TC_FAST == 3
    n_refused = 0
    for hidden in (128, 256):
        for layers in (1, 4, 8, 16):
            for fx in range(0, 17, 2):
                for fd, viewdirs in ((4, True), (6, True), (0, False)):
                    arch = ops.ArchSpec(num_layers=layers, hidden=hidden, use_viewdirs=viewdirs, n_freq_xyz=fx,
                                        n_freq_dir=fd)
                    for s in (14, 15, 64):
                        rc2, why2 = _supported_with_reason(arch, s, ops.IMPL_TC_FWD)
                        rc3, why3 = _supported_with_reason(arch, s, ops.IMPL_TC_FAST)
                        assert rc2 == rc3, (arch, s)
                        if rc2:
                            n_refused += 1
                            assert why2.split(": ", 1)[1] == why3.split(": ", 1)[1], (why2, why3)
                            assert "impl=3" in why3
    assert n_refused > 0


def test_auto_choice_never_picks_the_fast_forward():
    from nerf_pytorch_b200 import ops, train_utils

    for hidden in (128, 256):
        arch = ops.ArchSpec(num_layers=8, hidden=hidden, n_freq_xyz=10)
        for training in (True, False):
            assert train_utils._auto_impl(arch, arch, 64, 128, training=training) != ops.IMPL_TC_FAST


def test_backward_scratch_query_refuses_the_fast_forward():
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    arch = ops.ArchSpec()
    assert lib.nerfb200_bwd_scratch_floats(C.byref(arch.c_struct()), 4096, ops.IMPL_TC) > 0
    assert lib.nerfb200_bwd_scratch_floats(C.byref(arch.c_struct()), 4096, ops.IMPL_TC_FAST) == -1
    assert "inference only" in lib.nerfb200_last_error().decode()


def test_training_call_with_the_fast_forward_raises_before_touching_the_rays():
    """A call that would train (grad enabled, parameters that require grad) with impl 3 raises NotImplementedError naming
    inference, whether impl 3 came as the argument or as the default; the check precedes any device work, so CPU
    tensors reach it."""
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops, train_utils
    from oracle import nerf_oracle as O

    mc, mf = nb.FlexibleNeRFModel(), nb.FlexibleNeRFModel()
    opts = O.make_options()
    ro, rd = torch.zeros(4, 3), torch.ones(4, 3)
    epf, edf = nb.get_embedding_function(6), nb.get_embedding_function(4)
    with pytest.raises(NotImplementedError, match="inference"):
        nb.run_one_iter_of_nerf(8, 8, 10.0, mc, mf, ro, rd, opts, encode_position_fn=epf, encode_direction_fn=edf,
                                impl=ops.IMPL_TC_FAST)
    with pytest.raises(NotImplementedError, match="inference"):
        nb.run_one_iter_of_nerf_from_pose(8, 8, 10.0, mc, mf, torch.eye(4), None, opts, encode_position_fn=epf,
                                          encode_direction_fn=edf, impl=ops.IMPL_TC_FAST)
    with pytest.raises(NotImplementedError, match="inference"):
        nb.predict_and_render_radiance(torch.zeros(4, 11), mc, mf, opts, encode_position_fn=epf,
                                       encode_direction_fn=edf, impl=ops.IMPL_TC_FAST)
    saved = train_utils.DEFAULT_IMPL
    try:
        train_utils.set_default_impl(ops.IMPL_TC_FAST)
        with pytest.raises(NotImplementedError, match="inference"):
            nb.run_one_iter_of_nerf(8, 8, 10.0, mc, mf, ro, rd, opts, encode_position_fn=epf,
                                    encode_direction_fn=edf)
    finally:
        train_utils.set_default_impl(saved)
    # not training: the refusal does not apply (the CPU tensors are then refused for what they are)
    with torch.no_grad(), pytest.raises(NotImplementedError, match="CUDA"):
        nb.run_one_iter_of_nerf(8, 8, 10.0, mc, mf, ro, rd, opts, encode_position_fn=epf, encode_direction_fn=edf,
                                impl=ops.IMPL_TC_FAST)
