"""CPU: the early-stopping render's C ABI and Python refusals that need no GPU.
  1. the header's entry points are exported and the round constant is the header's;
  2. the library refuses impl 0, a threshold outside [0, 1) or NaN, an invalid grid and a grid without bits (or bits
     without a grid) from fake device pointers, before any launch;
  3. its workspace holds render_fwd's inference sections first;
  4. the Python keyword refuses training calls and bad thresholds before it touches the rays."""
import ctypes as C
import math

import pytest
import torch

import nerf_pytorch_b200 as nb
from nerf_pytorch_b200 import _lib, ops

_FAKE = C.c_void_p(1 << 20)  # never dereferenced: every call below is refused on the host


def _call(t=0.01, impl=1, grid=None, bits=None, n_fine=64, arch=None):
    lib = _lib.load()
    a = (arch or ops.ArchSpec(num_layers=4, hidden=128, n_freq_xyz=10)).c_struct()
    opts = ops.make_opts(64, n_fine, False, False, False, 0.0)
    return lib.nerfb200_render_fwd_early_stop(C.byref(a), C.byref(a), C.byref(opts), _FAKE, _FAKE, _FAKE, 11, 100, None,
                                              None, None, None, None, C.byref(grid) if grid is not None else None, bits,
                                              t, _FAKE, _FAKE, _FAKE, impl, None, None, None)


def test_entry_points_are_exported():
    lib = _lib.load()
    for name in ("nerfb200_render_fwd_early_stop", "nerfb200_render_early_stop_workspace_bytes",
                 "nerfb200_render_early_stop_round"):
        assert callable(getattr(lib, name))
    assert ops.stop_round() == 32
    assert callable(ops.render_fwd_early_stop)


@pytest.mark.parametrize("t", [1.0, 1.5, -1e-6, math.nan, math.inf])
def test_threshold_outside_the_unit_interval_is_invalid(t):
    before = ops.launch_count()
    assert _call(t=t) == _lib.ERR_INVALID
    assert "stop_transmittance" in _lib.load().nerfb200_last_error().decode()
    assert ops.launch_count() == before


def test_impl0_and_grid_mismatches_are_refused():
    before = ops.launch_count()
    lib = _lib.load()
    assert _call(impl=0) == _lib.ERR_UNSUPPORTED
    assert "impl=0" in lib.nerfb200_last_error().decode()
    assert _call(impl=2) == _lib.ERR_INVALID
    grid = ops.grid_struct(((-1.0,) * 3, (1.0,) * 3), (8, 8, 8))
    assert _call(grid=grid, bits=None) == _lib.ERR_INVALID
    assert _call(grid=None, bits=_FAKE) == _lib.ERR_INVALID
    bad = ops.grid_struct(((-1.0,) * 3, (1.0,) * 3), (0, 8, 8))
    assert _call(grid=bad, bits=_FAKE) == _lib.ERR_INVALID
    assert "invalid grid" in lib.nerfb200_last_error().decode()
    # an architecture the wgmma inference forward refuses: its reason
    assert _call(n_fine=0, impl=3, arch=ops.ArchSpec(num_layers=4, hidden=128, n_freq_xyz=11, include_input_xyz=False)) \
        == _lib.ERR_UNSUPPORTED
    assert ops.launch_count() == before


def test_workspace_extends_the_inference_workspace():
    a = ops.ArchSpec(num_layers=4, hidden=128, n_freq_xyz=10)
    for nf in (0, 128):
        opts = ops.make_opts(64, nf, False, False, False, 0.0)
        es = ops.render_early_stop_workspace_bytes(a, a if nf else None, opts, 1000)
        assert es > ops.render_workspace_bytes(a, a if nf else None, opts, 1000, False)
    lib = _lib.load()
    opts = ops.make_opts(64, 128, False, False, False, 0.0)
    assert lib.nerfb200_render_early_stop_workspace_bytes(C.byref(a.c_struct()), None, C.byref(opts), 0) == -1


def test_python_refusals_precede_the_rays():
    m = nb.FlexibleNeRFModel(num_layers=2, hidden_size=128, num_encoding_fn_xyz=2, num_encoding_fn_dir=1)
    from nerf_pytorch_b200 import train_utils

    with pytest.raises(NotImplementedError, match="inference"):
        train_utils.check_early_stop_call(0.01, m)
    with torch.no_grad():
        train_utils.check_early_stop_call(0.0, m)
        for bad in (1.0, -0.1, math.nan, None, "0.1", True):
            with pytest.raises(ValueError, match="early_stop"):
                train_utils.check_early_stop_call(bad, m)
    # a training call raises before the rays are looked at (CPU tensors reach the check)
    rays = torch.zeros(4, 11)
    with pytest.raises(NotImplementedError, match="inference"):
        nb.predict_and_render_radiance(rays, m, None, None, early_stop=0.01)
