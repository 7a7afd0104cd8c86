"""ctypes binding of libnerfb200.so (C ABI declared in include/nerfb200.h).

The product path has NO fallback: if the shared library is missing or a call fails, a
RuntimeError is raised (never a silent PyTorch / CPU path)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libnerfb200.so")

MAX_FREQS = 16

OK, ERR_INVALID, ERR_UNSUPPORTED, ERR_CUDA = 0, -1, -2, -3


class Arch(C.Structure):
    """nerfb200_arch_t"""

    _fields_ = [
        ("num_layers", C.c_int32),
        ("hidden", C.c_int32),
        ("skip_every", C.c_int32),
        ("use_viewdirs", C.c_int32),
        ("n_freq_xyz", C.c_int32),
        ("n_freq_dir", C.c_int32),
        ("include_input_xyz", C.c_int32),
        ("include_input_dir", C.c_int32),
        ("freq_xyz", C.c_float * MAX_FREQS),
        ("freq_dir", C.c_float * MAX_FREQS),
    ]


class RenderOpts(C.Structure):
    """nerfb200_render_opts_t"""

    _fields_ = [
        ("n_coarse", C.c_int32),
        ("n_fine", C.c_int32),
        ("perturb", C.c_int32),
        ("lindisp", C.c_int32),
        ("white_bkgd", C.c_int32),
        ("noise_std", C.c_float),
    ]


class Rng(C.Structure):
    """nerfb200_rng_t"""

    _fields_ = [
        ("seed", C.c_uint64),
        ("step", C.c_uint64),
        ("ray_offset", C.c_int64),
    ]


class Ndc(C.Structure):
    """nerfb200_ndc_t: the camera of a forward-facing scene's NDC map (include/nerfb200.h "NDC scenes")"""

    _fields_ = [
        ("height", C.c_int32),
        ("width", C.c_int32),
        ("focal", C.c_float),
    ]


class Grid(C.Structure):
    """nerfb200_grid_t: the box [lo, hi) and its cells per axis (the bit order is in include/nerfb200.h)"""

    _fields_ = [
        ("lo", C.c_float * 3),
        ("hi", C.c_float * 3),
        ("res", C.c_int32 * 3),
    ]


P = C.c_void_p
I32, I64, F32, F64, U64 = C.c_int32, C.c_int64, C.c_float, C.c_double, C.c_uint64
AP, OP, RP, GP, NP = C.POINTER(Arch), C.POINTER(RenderOpts), C.POINTER(Rng), C.POINTER(Grid), C.POINTER(Ndc)

# name -> (restype, argtypes); mirrors include/nerfb200.h one-to-one
SIGNATURES = {
    "nerfb200_version": (I32, []),
    "nerfb200_last_error": (C.c_char_p, []),
    "nerfb200_launch_count": (I64, []),
    "nerfb200_bwd_bytes_per_point": (I64, [AP]),
    "nerfb200_impl_supported": (I32, [AP, I32, I32]),
    "nerfb200_num_linear": (I64, [AP]),
    "nerfb200_flat_param_count": (I64, [AP]),
    "nerfb200_blob_floats": (I64, [AP]),
    "nerfb200_flat_layout": (I32, [AP, I32, C.POINTER(I64), C.POINTER(I64), C.POINTER(I32), C.POINTER(I32)]),
    "nerfb200_pack_weights": (I32, [AP, P, P, P]),
    "nerfb200_sample_coarse": (I32, [P, I32, I64, P, I32, I32, I32, P, P]),
    "nerfb200_gen_rays": (I32, [C.POINTER(F32), I32, I32, F32, P, I64, I32, F32, F32, I32, I32, P, P]),
    "nerfb200_pack_rays": (I32, [P, P, I64, I32, I32, F32, I32, F32, F32, I32, I32, P, P]),
    "nerfb200_encode": (I32, [AP, I32, P, I64, P, P]),
    "nerfb200_stash_floats": (I64, [AP, I64]),
    "nerfb200_mlp_fwd": (I32, [AP, P, P, I32, P, I64, I32, P, P, I32, P]),
    "nerfb200_composite_fwd": (I32, [P, P, P, I32, P, I64, I32, F32, I32, P, P, P]),
    "nerfb200_composite_bwd": (I32, [P, P, P, I32, P, P, I64, I32, F32, I32, P, P]),
    "nerfb200_sample_pdf_merge": (I32, [P, P, P, P, I64, I32, I32, P, P, P, P, P]),
    "nerfb200_bwd_scratch_floats": (I64, [AP, I64, I32]),
    "nerfb200_mlp_bwd": (I32, [AP, P, P, I32, P, I64, I32, P, P, P, P, I32, P]),
    "nerfb200_mlp_dgrad": (I32, [AP, P, P, P, P, I64, I32, P]),
    "nerfb200_mlp_wgrad": (I32, [AP, P, I32, P, I64, I32, P, P, P, P, I32, P]),
    "nerfb200_mlp_fwd_pts": (I32, [AP, P, P, P, I32, I64, I32, P, P, I32, P]),
    "nerfb200_mlp_bwd_pts": (I32, [AP, P, P, I32, I64, I32, P, P, P, P, I32, P]),
    "nerfb200_volume_render_fwd": (I32, [P, P, P, I32, P, I64, I32, F32, I32, P, P, P]),
    "nerfb200_volume_render_bwd": (I32, [P, P, P, I32, P, P, P, I64, I32, F32, I32, P, P]),
    "nerfb200_render_workspace_bytes": (I64, [AP, AP, OP, I64, I32]),
    "nerfb200_render_workspace_layout": (I32, [AP, AP, OP, I64, I32, C.POINTER(I64)]),
    "nerfb200_render_fwd": (I32, [AP, AP, OP, P, P, P, I32, I64, RP, P, P, P, P, P, P, P, I32, I32, P]),
    "nerfb200_render_bwd": (I32, [AP, AP, OP, P, P, P, I32, I64, RP, P, P, P, P, P, P, P, I32, I32, P]),
    "nerfb200_random_fill": (I32, [RP, I32, I64, I32, P, P]),
    "nerfb200_adam_step": (I32, [P, P, P, P, I64, I32, F32, F32, F32, F32, F32, P]),
    "nerfb200_random_fill_dev": (I32, [RP, P, I32, I64, I32, P, P]),
    "nerfb200_draw_workspace_bytes": (I64, [I64]),
    "nerfb200_draw_pixels": (I32, [U64, P, I32, I64, I64, P, P, P, P]),
    "nerfb200_gen_rays_posed": (I32, [P, I32, P, I32, I32, F32, P, I64, I32, F32, F32, I32, I32, P, P]),
    "nerfb200_gather_rows": (I32, [P, I64, P, P, I64, P, P]),
    "nerfb200_mse_loss": (I32, [P, P, P, I64, P, P, P, P]),
    "nerfb200_lr_schedule": (I32, [P, I64, F64, F64, F64, P, P]),
    "nerfb200_adam_step_dev": (I32, [P, P, P, P, I64, P, F64, F64, F64, F32, F32, F32, F32, P]),
    "nerfb200_step_advance": (I32, [P, P]),
    "nerfb200_grid_words": (I64, [GP]),
    "nerfb200_grid_locate": (I32, [GP, C.POINTER(F32), I64, C.POINTER(I64)]),
    "nerfb200_grid_max_blocks": (I64, [I64, I32]),
    "nerfb200_grid_scratch_ints": (I64, [I64, I32]),
    "nerfb200_grid_compact": (I32, [GP, P, P, I32, P, I64, I32, P, P, P, P, P, P, P]),
    "nerfb200_render_grid_workspace_bytes": (I64, [AP, AP, OP, I64]),
    "nerfb200_render_fwd_grid": (I32, [AP, AP, OP, P, P, P, I32, I64, RP, P, P, P, P, GP, P, P, P, P, I32, P, P]),
    "nerfb200_render_early_stop_round": (I32, []),
    "nerfb200_render_early_stop_workspace_bytes": (I64, [AP, AP, OP, I64]),
    "nerfb200_render_fwd_early_stop": (I32, [AP, AP, OP, P, P, P, I32, I64, RP, P, P, P, P, GP, P, F32, P, P, P, I32, P,
                                             P, P]),
    "nerfb200_mesh_workspace_bytes": (I64, [GP]),
    "nerfb200_mesh_lattice_points": (I32, [GP, I32, I32, P, P]),
    "nerfb200_mesh_count": (I32, [GP, P, F32, P, P, P]),
    "nerfb200_mesh_emit": (I32, [GP, P, F32, P, I64, I64, P, P, P, P]),
    "nerfb200_mesh_brick": (I32, []),
    "nerfb200_mesh_sparse_brick_count": (I64, [GP]),
    "nerfb200_mesh_sparse_scratch_bytes": (I64, [GP]),
    "nerfb200_mesh_sparse_workspace_bytes": (I64, [GP, I64]),
    "nerfb200_mesh_sparse_bricks": (I32, [GP, GP, P, P, P, P, P, P]),
    "nerfb200_mesh_sparse_bricks_host": (I32, [GP, GP, P, P]),
    "nerfb200_mesh_sparse_points": (I32, [GP, P, I64, I64, I32, P, P]),
    "nerfb200_mesh_sparse_count": (I32, [GP, P, P, I64, P, I32, F32, P, P, P]),
    "nerfb200_mesh_sparse_emit": (I32, [GP, P, P, I64, P, I32, F32, P, I64, I64, P, P, P, P, P]),
    "nerfb200_density_grad_supported": (I32, [AP, I32]),
    "nerfb200_density_grad": (I32, [AP, P, P, I64, P, I32, P]),
    "nerfb200_render_normals_workspace_bytes": (I64, [AP, AP, OP, I64]),
    "nerfb200_render_fwd_normals": (I32, [AP, AP, OP, P, P, P, I32, I64, RP, P, P, P, P, GP, P, F32, P, P, P, P, I32, P]),
    "nerfb200_ndc_mesh_to_world": (I32, [NP, P, P, P, I64, I64, P, P, P, P]),
    "nerfb200_ndc_from_world": (I32, [NP, P, I64, P, P]),
    "nerfb200_ndc_grad_to_world": (I32, [NP, P, P, I64, P, P]),
    "nerfb200_render_fwd_normals_ndc": (I32, [AP, AP, OP, P, P, P, I32, I64, RP, P, P, P, P, GP, P, F32, NP, P, P, P, P,
                                              I32, P]),
}

_lib = None


def build_library(verbose: bool = False) -> str:
    """Compile csrc/*.cu into libnerfb200.so for sm_90a (nvcc cross-compiles without a GPU)."""
    cmd = ["make", "-C", os.path.join(_HERE, "csrc"), "-j8"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("building libnerfb200.so failed:\n" + r.stdout[-4000:] + r.stderr[-4000:])
    if verbose:
        print(r.stdout[-2000:])
    return LIB_PATH


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C nerf_pytorch_b200/csrc`). There is no fallback path."
        )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here = header/library mismatch
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc != OK:
        msg = load().nerfb200_last_error().decode(errors="replace")
        kind = {ERR_INVALID: "invalid argument", ERR_UNSUPPORTED: "unsupported configuration", ERR_CUDA: "CUDA error"}.get(rc, "error")
        if rc == ERR_UNSUPPORTED:
            raise NotImplementedError(f"nerfb200 {what}: {kind}: {msg}")
        raise RuntimeError(f"nerfb200 {what}: {kind}: {msg}")
