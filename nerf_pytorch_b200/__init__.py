"""nerf_pytorch_b200 -- an H100-native (sm_90a) per-ray render/train path that drops in behind
krrish94/nerf-pytorch's ``run_one_iter_of_nerf`` / ``predict_and_render_radiance``.

Host side: Python/PyTorch (device memory, streams, torch.distributed).  Everything per ray runs in
``libnerfb200.so`` (hand-written CUDA behind the C ABI of include/nerfb200.h).  The names exported
here mirror ``from nerf import ...`` of the reference for the hot path."""
from .models import FlexibleNeRFModel
from .nerf_helpers import (Embedder, get_embedding_function, get_minibatches, get_ray_bundle, img2mse,
                           meshgrid_xy, mse2psnr, ndc_rays, positional_encoding, sample_pdf)
from .train_utils import (invalidate, predict_and_render_radiance, run_network, run_one_iter_of_nerf,
                          run_one_iter_of_nerf_from_pose, set_default_impl)
from .volume_rendering_utils import volume_render_radiance_field
from .eval_utils import cast_to_disparity_image, cast_to_image, cast_to_normal_image, render_image
from .cache_pool import CachedRayPool, CachedValidationSet
from .ops import SeededRandoms
from .graph_step import CapturedTrainStep
from .occupancy import OccupancyGrid
from .mesh import Mesh, density_volume, extract_mesh, extract_mesh_from_volume
from .density import density_gradient
from .bake import (BakedField, BakedFieldTrainer, bake, baked_brick_weights, baked_brick_weights_rays,
                   baked_density_gradient, baked_raw, baked_regularizer, baked_transparent_bricks, extract_baked_mesh,
                   prune_baked, render_baked, render_baked_rays, subdivide_baked)
from . import ops, parallel

__all__ = [
    "FlexibleNeRFModel", "Embedder", "get_embedding_function", "get_minibatches", "get_ray_bundle", "img2mse",
    "meshgrid_xy", "mse2psnr", "ndc_rays", "positional_encoding", "sample_pdf", "predict_and_render_radiance",
    "run_network", "volume_render_radiance_field",
    "run_one_iter_of_nerf", "run_one_iter_of_nerf_from_pose", "set_default_impl", "invalidate", "render_image", "cast_to_image", "cast_to_disparity_image", "cast_to_normal_image", "CachedRayPool", "CachedValidationSet", "SeededRandoms", "CapturedTrainStep", "OccupancyGrid", "Mesh",
    "density_volume", "extract_mesh", "extract_mesh_from_volume", "density_gradient", "BakedField", "bake", "render_baked",
    "render_baked_rays", "BakedFieldTrainer", "baked_brick_weights", "baked_brick_weights_rays",
    "baked_transparent_bricks", "prune_baked", "baked_regularizer", "subdivide_baked", "extract_baked_mesh",
    "baked_density_gradient", "baked_raw",
    "ops",
    "parallel",
]
