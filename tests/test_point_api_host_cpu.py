"""CPU: run_network and volume_render_radiance_field refuse what they cannot do before anything is launched, and the
library's caller-given-point entry points refuse malformed arguments from the plan alone."""
import ctypes as C

import pytest
import torch

import nerf_pytorch_b200 as nb
from nerf_pytorch_b200 import _lib, ops


def _model(use_viewdirs=True):
    return nb.FlexibleNeRFModel(num_layers=2, hidden_size=128, num_encoding_fn_xyz=2, num_encoding_fn_dir=1,
                                use_viewdirs=use_viewdirs)


EPF, EDF = nb.get_embedding_function(2), nb.get_embedding_function(1)


class _CudaLike:
    """A stand-in for a CUDA tensor (this machine may have no GPU): the refusals below must fire on shapes and flags
    before any device work, so nothing else of it is used."""

    def __init__(self, t, requires_grad=False):
        self._t = t
        self.requires_grad = requires_grad
        self.is_cuda = True
        self.shape = t.shape
        self.dtype = t.dtype

    def dim(self):
        return self._t.dim()

    def numel(self):
        return self._t.numel()

    def __getitem__(self, k):
        return _CudaLike(self._t[k])


def _no_launch(monkeypatch):
    before = ops.launch_count()

    def boom(*a, **k):
        raise AssertionError("launched")

    for name in ("pack_weights", "mlp_fwd_pts", "mlp_bwd_pts", "volume_render_fwd", "volume_render_bwd"):
        monkeypatch.setattr(ops, name, boom)
    return before


def test_both_functions_are_exported():
    assert callable(nb.run_network) and "run_network" in nb.__all__
    assert callable(nb.volume_render_radiance_field) and "volume_render_radiance_field" in nb.__all__


def test_run_network_refuses_cpu_tensors():
    with pytest.raises(NotImplementedError, match="CUDA"):
        nb.run_network(_model(), torch.zeros(2, 16, 3), torch.zeros(2, 11), 1024, EPF, EDF)


@pytest.mark.parametrize("shape", [(2, 16, 2), (2, 16, 4)])
def test_run_network_refuses_points_that_are_not_3d(monkeypatch, shape):
    before = _no_launch(monkeypatch)
    with pytest.raises(ValueError, match=r"\(\.\.\., 3\)"):
        nb.run_network(_model(), _CudaLike(torch.zeros(shape)), _CudaLike(torch.zeros(2, 11)), 1024, EPF, EDF)
    assert ops.launch_count() == before


@pytest.mark.parametrize("rays", [(3, 11), (2, 5, 11), (2, 2)])
def test_run_network_refuses_a_ray_batch_of_another_leading_shape(monkeypatch, rays):
    before = _no_launch(monkeypatch)
    with pytest.raises(ValueError, match="does not match"):
        nb.run_network(_model(), _CudaLike(torch.zeros(2, 16, 3)), _CudaLike(torch.zeros(rays)), 1024, EPF, EDF)
    assert ops.launch_count() == before


def test_run_network_refuses_a_view_dependent_model_without_embeddirs_fn(monkeypatch):
    before = _no_launch(monkeypatch)
    with pytest.raises(RuntimeError, match="view directions"):
        nb.run_network(_model(), _CudaLike(torch.zeros(2, 16, 3)), _CudaLike(torch.zeros(2, 11)), 1024, EPF, None)
    assert ops.launch_count() == before


def test_run_network_refuses_points_that_require_grad(monkeypatch):
    before = _no_launch(monkeypatch)
    pts = _CudaLike(torch.zeros(2, 16, 3), requires_grad=True)
    with pytest.raises(NotImplementedError, match="points"):
        nb.run_network(_model(), pts, _CudaLike(torch.zeros(2, 11)), 1024, EPF, EDF)
    assert ops.launch_count() == before


def test_run_network_refuses_the_single_pass_forward_while_training(monkeypatch):
    before = _no_launch(monkeypatch)
    with pytest.raises(NotImplementedError, match="inference"):
        nb.run_network(_model(), _CudaLike(torch.zeros(2, 16, 3)), _CudaLike(torch.zeros(2, 11)), 1024, EPF, EDF,
                       impl=ops.IMPL_TC_FAST)
    assert ops.launch_count() == before


def test_run_network_refuses_other_modules(monkeypatch):
    before = _no_launch(monkeypatch)
    with pytest.raises(NotImplementedError, match="FlexibleNeRFModel"):
        nb.run_network(torch.nn.Linear(3, 4), _CudaLike(torch.zeros(2, 16, 3)), _CudaLike(torch.zeros(2, 11)), 1024,
                       EPF, None)
    assert ops.launch_count() == before


def test_volume_render_refuses_cpu_tensors():
    with pytest.raises(NotImplementedError, match="CUDA"):
        nb.volume_render_radiance_field(torch.zeros(2, 8, 4), torch.zeros(2, 8), torch.zeros(2, 3))


@pytest.mark.parametrize("which", ["depth_values", "ray_directions"])
def test_volume_render_refuses_inputs_that_require_grad(monkeypatch, which):
    before = _no_launch(monkeypatch)
    args = dict(radiance_field=_CudaLike(torch.zeros(2, 8, 4)), depth_values=_CudaLike(torch.zeros(2, 8)),
                ray_directions=_CudaLike(torch.zeros(2, 3)))
    args[which].requires_grad = True
    with pytest.raises(NotImplementedError, match=which):
        nb.volume_render_radiance_field(args["radiance_field"], args["depth_values"], args["ray_directions"])
    assert ops.launch_count() == before


@pytest.mark.parametrize("shapes", [((2, 8, 4), (2, 7), (2, 3)), ((2, 8, 3), (2, 8), (2, 3)), ((2, 8, 4), (2, 8), (3, 3))])
def test_volume_render_refuses_mismatched_shapes(monkeypatch, shapes):
    before = _no_launch(monkeypatch)
    rf, z, d = (_CudaLike(torch.zeros(s)) for s in shapes)
    with pytest.raises(ValueError, match="radiance_field"):
        nb.volume_render_radiance_field(rf, z, d)
    assert ops.launch_count() == before


def test_volume_render_refuses_more_than_1024_samples(monkeypatch):
    before = _no_launch(monkeypatch)
    with pytest.raises(NotImplementedError, match="1025 samples"):
        nb.volume_render_radiance_field(_CudaLike(torch.zeros(2, 1025, 4)), _CudaLike(torch.zeros(2, 1025)),
                                        _CudaLike(torch.zeros(2, 3)))
    assert ops.launch_count() == before


# ---- the C ABI: refusals decided before any device pointer is touched --------------------------------------------------
_FAKE = C.c_void_p(16)  # never dereferenced: every call below is refused first


def test_point_forward_wants_directions_exactly_when_the_model_has_them():
    lib = _lib.load()
    for arch, dirs in ((ops.ArchSpec(), None), (ops.ArchSpec(use_viewdirs=False), _FAKE)):
        rc = lib.nerfb200_mlp_fwd_pts(C.byref(arch.c_struct()), _FAKE, _FAKE, dirs, 3, 4, 64, _FAKE, None,
                                      ops.IMPL_TC, None)
        assert rc == _lib.ERR_INVALID
        assert "dirs must be given iff" in lib.nerfb200_last_error().decode()


@pytest.mark.parametrize("impl", [4, 7, -1])
def test_point_forward_calls_unknown_impl_codes_invalid(impl):
    lib = _lib.load()
    rc = lib.nerfb200_mlp_fwd_pts(C.byref(ops.ArchSpec().c_struct()), _FAKE, _FAKE, _FAKE, 3, 4, 64, _FAKE, None, impl,
                                  None)
    assert rc == _lib.ERR_INVALID and f"unknown impl {impl}" in lib.nerfb200_last_error().decode()


def test_point_forward_refuses_the_single_pass_forward_with_a_stash():
    lib = _lib.load()
    rc = lib.nerfb200_mlp_fwd_pts(C.byref(ops.ArchSpec().c_struct()), _FAKE, _FAKE, _FAKE, 3, 4, 64, _FAKE, _FAKE,
                                  ops.IMPL_TC_FAST, None)
    assert rc == _lib.ERR_UNSUPPORTED and "inference only" in lib.nerfb200_last_error().decode()


def test_point_backward_refuses_what_the_render_backward_refuses():
    lib = _lib.load()
    a = ops.ArchSpec(use_viewdirs=False)
    rc = lib.nerfb200_mlp_bwd_pts(C.byref(a.c_struct()), _FAKE, None, 0, 4, 64, _FAKE, _FAKE, _FAKE, _FAKE,
                                  ops.IMPL_TC, None)
    assert rc == _lib.ERR_UNSUPPORTED and "view-dependent" in lib.nerfb200_last_error().decode()
    rc = lib.nerfb200_mlp_bwd_pts(C.byref(ops.ArchSpec().c_struct()), _FAKE, _FAKE, 3, 4, 8, _FAKE, _FAKE, _FAKE,
                                  _FAKE, ops.IMPL_TC, None)
    assert rc == _lib.ERR_UNSUPPORTED and "15 samples" in lib.nerfb200_last_error().decode()


@pytest.mark.parametrize("n_samples, stride", [(0, 3), (1025, 3), (64, -1)])
def test_volume_render_entry_points_refuse_bad_sizes(n_samples, stride):
    lib = _lib.load()
    assert lib.nerfb200_volume_render_fwd(_FAKE, _FAKE, _FAKE, stride, None, 4, n_samples, 0.0, 0, _FAKE, None,
                                          None) == _lib.ERR_INVALID
    assert lib.nerfb200_volume_render_bwd(_FAKE, _FAKE, _FAKE, stride, None, _FAKE, None, 4, n_samples, 0.0, 0, _FAKE,
                                          None) == _lib.ERR_INVALID
