"""Full-image rendering on the fused path (the reference's render loops: eval_nerf.py:156-190, the validation block of
train_nerf.py:287-371).

``render_image`` generates the rays of EVERY pixel on the device from the pose (csrc/raygen.cu: no (H, W, 3) ray
tensors built by a chain of torch ops, view directions / NDC / near / far packed in the same kernel), renders them in
chunks under ``torch.no_grad()`` through ``predict_and_render_radiance`` and returns the reference's 6-tuple in image
shape.  ``cast_to_image`` / ``cast_to_disparity_image`` reproduce eval_nerf.py:23-36 on the device (uint8 tensors)."""
from __future__ import annotations

from typing import Optional

import torch

from . import ops, train_utils
from .ops import SeededRandoms


def render_image(height, width, focal_length, tform_cam2world, model_coarse, model_fine, options, mode="validation",
                 encode_position_fn=None, encode_direction_fn=None, *, rays_per_chunk: Optional[int] = None,
                 device=None, impl: Optional[int] = None, randoms: Optional[SeededRandoms] = None, grid=None,
                 early_stop: Optional[float] = None, normals=False):
    """One pose -> (rgb_coarse (H,W,3), disp_coarse (H,W), acc_coarse (H,W), rgb_fine, disp_fine, acc_fine).

    Like the reference, the per-chunk sampler options come from ``options.nerf.train`` unless
    ``train_utils.COMPAT_MODE_QUIRK`` is switched off (the reference forgets to forward ``mode``, train_utils.py:171-181);
    the chunk size comes from ``options.nerf.<mode>.chunksize`` (``rays_per_chunk`` overrides it: the fused kernels
    need no small chunks, an H100's 80 GB of HBM hold a whole 800 x 800 image's intermediates).

    ``randoms``: a ``SeededRandoms`` makes a render with ``perturb`` or noise on reproducible: pixel ``j * width + i`` is
    ray ``ray_offset + j * width + i`` of the seeded stream whatever the chunk size.  Default: torch draws per chunk.

    ``impl=ops.IMPL_TC_FAST`` renders with the single-pass fp16 wgmma forward (INTEGRATION.md, "Optional fast paths"):
    fewer MMAs, fp16 operands, judged by PSNR against the default path rather than by parity with it.

    ``grid``: an ``OccupancyGrid`` (INTEGRATION.md, "Optional fast paths"): samples in its empty cells skip the MLP and
    get zero density; impl 1 or 3 only.  Every other sample, and so every ray none of whose skipped samples had density,
    is computed bit for bit as without the grid.

    ``early_stop``: a transmittance threshold t in [0, 1) (INTEGRATION.md, "Optional fast paths"; combines with
    ``grid``): the fine pass stops a ray once its transmittance falls below t.  A ray that never stops is bit for bit
    the render without it; one that stops moves its rgb and acc by at most t.

    ``normals=True`` (impl 1, inference; combines with ``grid`` and ``early_stop``) returns a seventh output, the normal
    map (H, W, 3) of the last pass: the compositing weights times the outward unit normals -grad sigma / |grad sigma| at
    its samples, summed per ray and not renormalised (include/nerfb200.h "normal maps"); ``cast_to_normal_image``
    turns it into uint8.  The six other outputs are exactly those of the call without it.  ``normals="world"`` gives
    the normal map in world space: for an NDC scene (``options.dataset.no_ndc`` false) the gradient at each sample is
    mapped by the Jacobian of this call's NDC map (``height``, ``width``, ``focal_length``) before it is normalised
    and weighted (include/nerfb200.h "NDC scenes"); for a Blender scene it is exactly ``normals=True``."""
    normals = train_utils.normals_mode(normals)
    ndc = (height, width, focal_length) if normals == "world" else None
    if ndc is not None:
        train_utils._world_ndc(normals, options, ndc)  # a malformed camera is refused before any launch
    if randoms is not None and not isinstance(randoms, SeededRandoms):
        raise TypeError("render_image: randoms must be a SeededRandoms (tensors cannot span several chunks)")
    if device is None:
        device = next(model_coarse.parameters()).device
    use_viewdirs = bool(options.nerf.use_viewdirs)
    if grid is not None:
        with torch.no_grad():
            train_utils.check_grid_call(grid, device, model_coarse, model_fine)
    if early_stop is not None:
        with torch.no_grad():
            train_utils.check_early_stop_call(early_stop, model_coarse, model_fine)
    with torch.no_grad():
        rays = ops.gen_rays(tform_cam2world, height, width, focal_length, None, device,
                            ndc=options.dataset.no_ndc is False, near=options.dataset.near, far=options.dataset.far,
                            use_viewdirs=use_viewdirs)
        n = rays.shape[0]
        chunk = int(rays_per_chunk or getattr(options.nerf, mode).chunksize)
        inner_mode = "train" if train_utils.COMPAT_MODE_QUIRK else mode
        parts = [train_utils.predict_and_render_radiance(
            rays[i:i + chunk], model_coarse, model_fine, options, mode=inner_mode,
            encode_position_fn=encode_position_fn,
            encode_direction_fn=encode_direction_fn if use_viewdirs else None, impl=impl, grid=grid,
            early_stop=early_stop, normals=normals, randoms=randoms.shifted(i) if randoms is not None else None,
            _ndc=ndc)
            for i in range(0, n, chunk)]
    cols = [torch.cat(c, 0) if c[0] is not None else None for c in zip(*parts)]
    shapes = [(height, width, 3), (height, width), (height, width)] * 2 + [(height, width, 3)]
    return tuple(c.view(s) if c is not None else None for c, s in zip(cols, shapes))


def cast_to_image(rgb: torch.Tensor) -> torch.Tensor:
    """eval_nerf.py:23-30: (H, W, 3) floats in [0, 1] -> uint8 (H, W, 3) the way ToPILImage does it (x * 255, truncated)."""
    return rgb[..., :3].mul(255).clamp(0, 255).to(torch.uint8)


def cast_to_normal_image(normals: torch.Tensor) -> torch.Tensor:
    """A normal map (..., 3) with components in [-1, 1] -> uint8 (..., 3): (N * 0.5 + 0.5) * 255, converted as
    ``cast_to_image`` converts."""
    img = (normals.detach() * 0.5 + 0.5) * 255
    return img.clamp(0, 255).to(torch.uint8)


def cast_to_disparity_image(disp: torch.Tensor) -> torch.Tensor:
    """eval_nerf.py:33-36: min-max normalised disparity as uint8.  Rays that hit nothing have NaN disparity in the
    reference (0 / 0, volume_rendering_utils.py:48); they are excluded from the min / max and drawn as 0 here."""
    finite = torch.isfinite(disp)
    d = torch.where(finite, disp, torch.zeros_like(disp))
    if finite.any():
        lo, hi = disp[finite].min(), disp[finite].max()
        d = (d - lo) / (hi - lo).clamp_min(1e-30)
    return (d.clamp(0, 1) * 255).masked_fill(~finite, 0).to(torch.uint8)
