"""Drop-in replacement for the reference's nerf/volume_rendering_utils.py:

    volume_render_radiance_field    nerf/volume_rendering_utils.py:6-53

Same positional signature and 5-tuple result, compositing caller-given samples on the render path's kernels
(csrc/composite.cu), differentiable w.r.t. ``radiance_field`` through all five outputs."""
from __future__ import annotations

import math
from typing import Optional

import torch

from . import ops


class _VolumeRender(torch.autograd.Function):
    @staticmethod
    def forward(ctx, raw, z, dirs, noise, noise_std, white_bkgd):
        out, weights = ops.volume_render_fwd(raw, z, dirs, noise, noise_std, white_bkgd)
        ctx.save_for_backward(raw, z, dirs, noise)
        ctx.cfg = (noise_std, white_bkgd)
        ctx.set_materialize_grads(False)
        return out, weights

    @staticmethod
    def backward(ctx, g_out, g_weights):
        raw, z, dirs, noise = ctx.saved_tensors
        noise_std, white_bkgd = ctx.cfg
        if g_out is None:
            g_out = torch.zeros(z.shape[0], 8, dtype=torch.float32, device=z.device)
        d_raw = ops.volume_render_bwd(raw, z, dirs, noise, g_out.contiguous(),
                                      None if g_weights is None else g_weights.contiguous(), noise_std, white_bkgd)
        return (d_raw,) + (None,) * 5


def volume_render_radiance_field(radiance_field, depth_values, ray_directions, radiance_field_noise_std=0.0,
                                 white_background=False, *, noise: Optional[torch.Tensor] = None):
    """``radiance_field`` (*B, S, 4), ``depth_values`` (*B, S), ``ray_directions`` (*B, 3), 1 <= S <= 1024, all on a
    CUDA device.  Returns ``(rgb_map, disp_map, acc_map, weights, depth_map)`` as the reference does (fp32).

    With ``radiance_field_noise_std > 0`` the sigma noise is ``torch.randn(radiance_field[..., 3].shape)`` drawn here
    as the reference draws it, times the std; ``noise`` (keyword-only) injects those unit normals instead.  The same
    noise is used by the backward.  No gradient w.r.t. ``depth_values`` or ``ray_directions``."""
    if not (radiance_field.is_cuda and depth_values.is_cuda and ray_directions.is_cuda):
        raise NotImplementedError("nerfb200: compositing inputs must be on a CUDA device (there is no CPU path)")
    if torch.is_grad_enabled() and (depth_values.requires_grad or ray_directions.requires_grad):
        raise NotImplementedError("nerfb200: volume_render_radiance_field gives no gradient w.r.t. depth_values or "
                                  "ray_directions; detach them")
    lead, S = tuple(depth_values.shape[:-1]), depth_values.shape[-1] if depth_values.dim() else 0
    if (depth_values.dim() < 1 or tuple(radiance_field.shape) != lead + (S, 4)
            or tuple(ray_directions.shape) != lead + (3,)):
        raise ValueError(f"nerfb200: need radiance_field (*B, S, 4), depth_values (*B, S), ray_directions (*B, 3); got "
                         f"{tuple(radiance_field.shape)}, {tuple(depth_values.shape)}, {tuple(ray_directions.shape)}")
    if not 1 <= S <= 1024:
        raise NotImplementedError(f"nerfb200: {S} samples per ray (the compositing kernels take 1..1024)")
    n = math.prod(lead)
    noise_std = float(radiance_field_noise_std)
    nz = None
    if noise_std > 0.0:
        if noise is None:
            noise = torch.randn(radiance_field[..., 3].shape, dtype=radiance_field.dtype, device=radiance_field.device)
        nz = noise.detach().to(device=depth_values.device, dtype=torch.float32).reshape(n, S).contiguous()
    raw = radiance_field.float().reshape(n, S, 4).contiguous()
    z = depth_values.detach().float().reshape(n, S).contiguous()
    dirs = ray_directions.detach().float().reshape(n, 3)
    if dirs.stride(1) != 1:
        dirs = dirs.contiguous()
    out, weights = _VolumeRender.apply(raw, z, dirs, nz, noise_std, bool(white_background))
    return (out[:, :3].reshape(lead + (3,)), out[:, 3].reshape(lead), out[:, 4].reshape(lead),
            weights.reshape(lead + (S,)), out[:, 5].reshape(lead))
