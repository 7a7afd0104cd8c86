"""The density field of a trained FlexibleNeRFModel probed at caller-given points: raw sigma and its gradient with
respect to the point, from one fused kernel (csrc/mlp_tc.cu, density_grad_tc_kernel; the rule is in
include/nerfb200.h, "density gradient").  The outward surface normal of a level set of sigma is -grad / |grad|."""
from __future__ import annotations

from typing import Optional

import torch

from . import ops


def _checked_points(pts) -> torch.Tensor:
    if not isinstance(pts, torch.Tensor):
        raise TypeError(f"nerfb200: pts must be a tensor, got {type(pts).__name__}")
    if pts.dtype != torch.float32 or pts.dim() < 1 or pts.shape[-1] != 3:
        raise ValueError(f"nerfb200: pts must be an fp32 tensor of shape (..., 3), got {pts.dtype}{list(pts.shape)}")
    if not pts.is_cuda:
        raise NotImplementedError("nerfb200: pts must be a CUDA tensor (there is no CPU path)")
    return pts


def refusal(arch: ops.ArchSpec, impl: Optional[int]) -> int:
    """The impl the density gradient runs ``arch`` on (None: 1, the only one), or NotImplementedError with the
    library's reason."""
    use = ops.IMPL_TC if impl is None else int(impl)
    why = ops.density_grad_refusal(arch, use)
    if why is not None:
        raise NotImplementedError(f"nerfb200 density_gradient: {why}")
    return use


def density_grad_points(arch: ops.ArchSpec, blob: torch.Tensor, pts: torch.Tensor, impl: int):
    """(sigma_raw (P,), grad (P, 3)) at flat points (P, 3) that passed the refusals; P may be 0."""
    if pts.shape[0] == 0:
        return pts.new_zeros(0), pts.new_zeros(0, 3)
    if pts.device != blob.device:
        raise RuntimeError(f"nerfb200: the points are on {pts.device}, the network on {blob.device}")
    with torch.no_grad():
        out = ops.density_grad(arch, blob, pts.contiguous(), impl)
    return out[:, 0], out[:, 1:]


def density_gradient(model, encode_position_fn, pts: torch.Tensor, *, impl: Optional[int] = None):
    """Raw sigma (before the ReLU) of ``model`` and its gradient w.r.t. the points, at ``pts`` (..., 3) fp32 CUDA:
    returns ``(sigma_raw (...), grad (..., 3))``.

    The gradient is taken in the coordinates the network encodes (world space for Blender scenes, NDC for LLFF), by
    the exact chain rule through the trunk and the positional encoding on the wgmma tensor cores (impl 1, the only
    one); sigma_raw has the bits the wgmma forward (``run_network`` on impl 1) gives at the same point.  Sigma reads no
    view direction, so none is needed.  Inference only: a call with autograd on and parameters that require grad is
    refused, as are CPU tensors and architectures or impls the kernel does not run (NotImplementedError), all before
    any launch."""
    from . import train_utils
    from .mesh import _network

    params = list(model.parameters()) if hasattr(model, "parameters") else []
    if train_utils._trains(params):
        raise NotImplementedError("nerfb200: density_gradient is inference only (no backward); call it under "
                                  "torch.no_grad() or on parameters that do not require grad")
    pts = _checked_points(pts)
    arch = _network(model, encode_position_fn, None)
    use = refusal(arch, impl)
    _, blob = train_utils._packed(model, arch)
    sigma, grad = density_grad_points(arch, blob, pts.reshape(-1, 3), use)
    return sigma.reshape(pts.shape[:-1]), grad.reshape(pts.shape)
