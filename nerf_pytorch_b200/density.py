"""The density field of a trained FlexibleNeRFModel probed at caller-given points: raw sigma and its gradient with
respect to the point, from one fused kernel (csrc/mlp_tc.cu, density_grad_tc_kernel; the rule is in
include/nerfb200.h, "density gradient").  The outward surface normal of a level set of sigma is -grad / |grad|.
For a forward-facing (NDC) scene the points and gradients can be taken in world space through the NDC map
(csrc/ndc.cu, include/nerfb200.h "NDC scenes")."""
from __future__ import annotations

import math
import numbers
from typing import Optional

import torch

from . import ops


def ndc_camera(ndc) -> ops.Ndc:
    """The NDC map of ``ndc = (H, W, focal)``, the image size and focal length an LLFF scene's rays were generated
    with; ValueError for anything else."""
    try:
        h, w, f = ndc
    except (TypeError, ValueError):
        raise ValueError(f"nerfb200: ndc must be (H, W, focal), got {ndc!r}") from None
    ints = all(isinstance(v, numbers.Integral) and not isinstance(v, bool) and 0 < v < 2 ** 31 for v in (h, w))
    if not ints or not isinstance(f, numbers.Real) or isinstance(f, bool) or not (math.isfinite(f) and f > 0):
        raise ValueError(f"nerfb200: ndc must be (H, W, focal) with H, W positive ints and a finite focal > 0, got "
                         f"{ndc!r}")
    return ops.ndc_struct(h, w, f)


def _checked_points(pts, world_ndc: bool = False) -> torch.Tensor:
    if not isinstance(pts, torch.Tensor):
        raise TypeError(f"nerfb200: pts must be a tensor, got {type(pts).__name__}")
    if pts.dtype != torch.float32 or pts.dim() < 1 or pts.shape[-1] != 3:
        raise ValueError(f"nerfb200: pts must be an fp32 tensor of shape (..., 3), got {pts.dtype}{list(pts.shape)}")
    if world_ndc and not bool((pts[..., 2] < 0).all()):
        raise ValueError("nerfb200: with ndc=, pts are world points in front of the camera: every z must be < 0")
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


def ndc_density_grad_points(arch: ops.ArchSpec, blob: torch.Tensor, q: torch.Tensor, impl: int, cam: ops.Ndc):
    """(sigma_raw (P,), world grad J^T(q) g (P, 3)) at flat NDC points q (P, 3) that passed the refusals."""
    if q.shape[0] == 0:
        return q.new_zeros(0), q.new_zeros(0, 3)
    if q.device != blob.device:
        raise RuntimeError(f"nerfb200: the points are on {q.device}, the network on {blob.device}")
    q = q.contiguous()
    with torch.no_grad():
        out = ops.density_grad(arch, blob, q, impl)
        ops.ndc_grad_to_world(cam, q, out, out=out)
    return out[:, 0], out[:, 1:]


def density_gradient(model, encode_position_fn, pts: torch.Tensor, *, impl: Optional[int] = None, ndc=None):
    """Raw sigma (before the ReLU) of ``model`` and its gradient w.r.t. the points, at ``pts`` (..., 3) fp32 CUDA:
    returns ``(sigma_raw (...), grad (..., 3))``.

    The gradient is taken in the coordinates the network encodes (world space for Blender scenes, NDC for LLFF), by
    the exact chain rule through the trunk and the positional encoding on the wgmma tensor cores (impl 1, the only
    one); sigma_raw has the bits the wgmma forward (``run_network`` on impl 1) gives at the same point.  Sigma reads no
    view direction, so none is needed.  Inference only: a call with autograd on and parameters that require grad is
    refused, as are CPU tensors and architectures or impls the kernel does not run (NotImplementedError), all before
    any launch.

    ``ndc=(H, W, focal)`` takes a forward-facing scene's ``pts`` in world space (every z < 0, in front of the camera;
    ValueError otherwise): sigma_raw is that of the network at the NDC point N(p) its rays encode (the bits
    ``run_network`` gives there on impl 1), and grad is the world gradient J^T grad_q (include/nerfb200.h "NDC
    scenes")."""
    from . import train_utils
    from .mesh import _network

    cam = ndc_camera(ndc) if ndc is not None else None
    params = list(model.parameters()) if hasattr(model, "parameters") else []
    if train_utils._trains(params):
        raise NotImplementedError("nerfb200: density_gradient is inference only (no backward); call it under "
                                  "torch.no_grad() or on parameters that do not require grad")
    pts = _checked_points(pts, world_ndc=cam is not None)
    arch = _network(model, encode_position_fn, None)
    use = refusal(arch, impl)
    _, blob = train_utils._packed(model, arch)
    if cam is None:
        sigma, grad = density_grad_points(arch, blob, pts.reshape(-1, 3), use)
    else:
        if pts.device != blob.device:
            raise RuntimeError(f"nerfb200: the points are on {pts.device}, the network on {blob.device}")
        q = ops.ndc_from_world(cam, pts.reshape(-1, 3).contiguous())
        sigma, grad = ndc_density_grad_points(arch, blob, q, use, cam)
    return sigma.reshape(pts.shape[:-1]), grad.reshape(pts.shape)
