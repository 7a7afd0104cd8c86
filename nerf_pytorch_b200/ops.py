"""Torch-tensor wrappers over the C ABI (include/nerfb200.h): device memory, streams, nothing else.

Every function checks that its tensors are CUDA / fp32 / contiguous, allocates the outputs with
``torch.empty`` and launches on ``torch.cuda.current_stream()``.  No math happens in Python."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from functools import lru_cache
from typing import Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import Arch, Grid, Ndc, RenderOpts, Rng

IMPL_SIMT = 0  # fp32 CUDA cores
IMPL_TC = 1    # wgmma tensor cores (fp16x2 three-term splits, fp32 accumulation)
IMPL_TC_FWD = 2  # query only (impl_supported): the wgmma forward alone (inference), which also runs hidden 256
# inference only: single-pass fp16 wgmma forward (one fp16(w) x fp16(activation / 16) product per k-step, fp32
# accumulation); ~3x fewer MMAs than IMPL_TC at ~11 significant bits per operand.  Renders, never trains; never chosen
# automatically.  Accepted exactly where IMPL_TC_FWD is.
IMPL_TC_FAST = 3


def _ptr(t: Optional[torch.Tensor]):
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("nerfb200: tensor is not on a CUDA device (there is no CPU path)")
    if t.dtype not in (torch.float32, torch.int32, torch.int64, torch.uint8):
        raise RuntimeError(f"nerfb200: unsupported dtype {t.dtype}")
    if not t.is_contiguous():
        raise RuntimeError("nerfb200: tensor must be contiguous")
    return C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def launch_count() -> int:
    """Kernels launched by libnerfb200.so in this process so far."""
    return int(_lib.load().nerfb200_launch_count())


def frequency_bands(n: int, log_sampling: bool) -> torch.Tensor:
    """The bands exactly as the reference builds them (nerf/nerf_helpers.py:131-147), fp32, on CPU."""
    if n == 0:
        return torch.zeros(0)
    if log_sampling:
        return 2.0 ** torch.linspace(0.0, n - 1, n, dtype=torch.float32)
    return torch.linspace(2.0 ** 0.0, 2.0 ** (n - 1), n, dtype=torch.float32)


@dataclass(frozen=True)
class ArchSpec:
    """Hashable description of one FlexibleNeRFModel + its encoders (-> nerfb200_arch_t)."""

    num_layers: int = 4
    hidden: int = 128
    skip_every: int = 4
    use_viewdirs: bool = True
    n_freq_xyz: int = 6
    n_freq_dir: int = 4
    include_input_xyz: bool = True
    include_input_dir: bool = True
    log_sampling_xyz: bool = True
    log_sampling_dir: bool = True

    @property
    def dim_xyz(self):
        return (3 if self.include_input_xyz else 0) + 6 * self.n_freq_xyz

    @property
    def dim_dir(self):
        return ((3 if self.include_input_dir else 0) + 6 * self.n_freq_dir) if self.use_viewdirs else 0

    @lru_cache(maxsize=None)
    def c_struct(self) -> Arch:
        a = Arch()
        a.num_layers, a.hidden, a.skip_every = self.num_layers, self.hidden, self.skip_every
        a.use_viewdirs = int(self.use_viewdirs)
        a.n_freq_xyz, a.n_freq_dir = self.n_freq_xyz, self.n_freq_dir
        a.include_input_xyz, a.include_input_dir = int(self.include_input_xyz), int(self.include_input_dir)
        if self.n_freq_xyz > _lib.MAX_FREQS or self.n_freq_dir > _lib.MAX_FREQS:
            raise NotImplementedError("nerfb200: more than 16 encoding frequencies")
        for i, f in enumerate(frequency_bands(self.n_freq_xyz, self.log_sampling_xyz).tolist()):
            a.freq_xyz[i] = f
        for i, f in enumerate(frequency_bands(self.n_freq_dir, self.log_sampling_dir).tolist()):
            a.freq_dir[i] = f
        return a

    # ---- flat parameter vector layout -------------------------------------------------------
    def slot_names(self) -> Sequence[str]:
        """Reference state_dict prefixes in the canonical slot order of include/nerfb200.h."""
        names = ["layer1"] + [f"layers_xyz.{i}" for i in range(self.num_layers - 1)]
        if self.use_viewdirs:
            names += ["fc_feat", "fc_alpha", "layers_dir.0", "fc_rgb"]
        else:
            names += ["fc_out"]
        return names

    @lru_cache(maxsize=None)
    def flat_layout(self):
        """[(name, w_off, b_off, in, out)] from the library (single source of truth)."""
        lib = _lib.load()
        a = self.c_struct()
        out = []
        for slot, name in enumerate(self.slot_names()):
            w, b, i, o = C.c_int64(), C.c_int64(), C.c_int32(), C.c_int32()
            _lib.check(lib.nerfb200_flat_layout(C.byref(a), slot, C.byref(w), C.byref(b), C.byref(i), C.byref(o)),
                       "flat_layout")
            out.append((name, w.value, b.value, i.value, o.value))
        return out

    @lru_cache(maxsize=None)
    def flat_param_count(self) -> int:
        n = _lib.load().nerfb200_flat_param_count(C.byref(self.c_struct()))
        if n < 0:
            _lib.check(_lib.ERR_UNSUPPORTED, "flat_param_count")
        return n

    @lru_cache(maxsize=None)
    def blob_floats(self) -> int:
        n = _lib.load().nerfb200_blob_floats(C.byref(self.c_struct()))
        if n < 0:
            _lib.check(_lib.ERR_UNSUPPORTED, "blob_floats")
        return n


@dataclass(frozen=True)
class SeededRandoms:
    """The render path's random inputs generated in-kernel from a counter-based stream (include/nerfb200.h,
    ``nerfb200_rng_t``): every number is a pure function of (seed, step, stream, global ray index, sample), so a ray gets
    the same numbers however the batch is chunked or sharded.  ``ray_offset`` is the global index of the first ray
    passed; give each optimisation step its own ``step`` (< 2^30)."""

    seed: int
    step: int = 0
    ray_offset: int = 0

    def __post_init__(self):
        if not 0 <= int(self.seed) < 2 ** 64:
            raise ValueError("SeededRandoms: seed must be in [0, 2^64)")
        if not 0 <= int(self.step) < 2 ** 30:
            raise ValueError("SeededRandoms: step must be in [0, 2^30)")
        if int(self.ray_offset) < 0:
            raise ValueError("SeededRandoms: ray_offset must be >= 0")

    def shifted(self, n_rays: int) -> "SeededRandoms":
        """The same stream for the rays that start ``n_rays`` further on (a later chunk or shard)."""
        return SeededRandoms(self.seed, self.step, self.ray_offset + int(n_rays))

    def c_struct(self) -> Rng:
        return Rng(int(self.seed), int(self.step), int(self.ray_offset))


RAND_STREAMS = {"t_rand": 0, "noise_c": 1, "u": 2, "noise_f": 3}


def random_fill(rng: SeededRandoms, stream, n_rays: int, per_ray: int, device=None) -> torch.Tensor:
    """Stream ``stream`` (a name of RAND_STREAMS or its id) of ``rng`` for ``n_rays`` rays from ``rng.ray_offset`` on:
    (n_rays, per_ray) fp32, uniforms in [0, 1) for t_rand / u, unit normals for noise_c / noise_f.  These are exactly
    the numbers the seeded render kernels consume."""
    lib = _lib.load()
    sid = RAND_STREAMS[stream] if isinstance(stream, str) else int(stream)
    out = torch.empty(int(n_rays), int(per_ray), dtype=torch.float32,
                      device=device if device is not None else torch.cuda.current_device())
    _lib.check(lib.nerfb200_random_fill(C.byref(rng.c_struct()), sid, int(n_rays), int(per_ray), _ptr(out), _stream()),
               "random_fill")
    return out


def make_opts(n_coarse, n_fine, perturb, lindisp, white_bkgd, noise_std) -> RenderOpts:
    o = RenderOpts()
    o.n_coarse, o.n_fine = int(n_coarse), int(n_fine)
    o.perturb, o.lindisp, o.white_bkgd = int(bool(perturb)), int(bool(lindisp)), int(bool(white_bkgd))
    o.noise_std = float(noise_std)
    return o


# ------------------------------------------------------------------------------------------------
# parameters
# ------------------------------------------------------------------------------------------------
def flatten_state_dict(arch: ArchSpec, sd, device) -> torch.Tensor:
    """state_dict (reference key names) -> flat fp32 vector in canonical order."""
    parts = []
    for name, _, _, fin, fout in arch.flat_layout():
        w, b = sd[name + ".weight"], sd[name + ".bias"]
        if tuple(w.shape) != (fout, fin) or tuple(b.shape) != (fout,):
            raise RuntimeError(f"nerfb200: {name} has shape {tuple(w.shape)}, expected {(fout, fin)}")
        parts += [w.reshape(-1), b.reshape(-1)]
    return torch.cat([p.to(device=device, dtype=torch.float32) for p in parts]).contiguous()


def pack_weights(arch: ArchSpec, flat: torch.Tensor, blob: Optional[torch.Tensor] = None) -> torch.Tensor:
    lib = _lib.load()
    if flat.numel() != arch.flat_param_count():
        raise RuntimeError("nerfb200: flat parameter vector has the wrong length")
    if blob is None:
        blob = torch.empty(arch.blob_floats(), dtype=torch.float32, device=flat.device)
    _lib.check(lib.nerfb200_pack_weights(C.byref(arch.c_struct()), _ptr(flat), _ptr(blob), _stream()), "pack_weights")
    return blob


# ------------------------------------------------------------------------------------------------
# stage-level ops (test hooks + building blocks)
# ------------------------------------------------------------------------------------------------
def sample_coarse(rays, t_rand, n_coarse, perturb, lindisp):
    lib = _lib.load()
    n = rays.shape[0]
    z = torch.empty(n, n_coarse, dtype=torch.float32, device=rays.device)
    _lib.check(lib.nerfb200_sample_coarse(_ptr(rays), rays.shape[1], n, _ptr(t_rand) if perturb else None, n_coarse,
                                          int(bool(perturb)), int(bool(lindisp)), _ptr(z), _stream()),
               "sample_coarse")
    return z


def gen_rays(c2w, height, width, focal, pixel_ids, device, ndc=False, near=0.0, far=1.0, use_viewdirs=True, stride=None):
    """Rays of the given pixels (int64 ids j * W + i on `device`, or None for the whole image) of a pinhole camera with
    camera-to-world matrix ``c2w`` (anything convertible to 12+ host floats: the top 3 x 4 block is used)."""
    lib = _lib.load()
    m = torch.as_tensor(c2w, dtype=torch.float32, device="cpu").reshape(-1, 4)[:3].contiguous().reshape(-1)
    c12 = (C.c_float * 12)(*m.tolist())
    n = int(pixel_ids.numel()) if pixel_ids is not None else int(height) * int(width)
    if stride is None:
        stride = 11 if use_viewdirs else 8
    out = torch.empty(n, stride, dtype=torch.float32, device=device)
    _lib.check(lib.nerfb200_gen_rays(c12, int(height), int(width), float(focal), _ptr(pixel_ids), n, int(bool(ndc)),
                                     float(near), float(far), int(bool(use_viewdirs) and stride == 11), stride, _ptr(out),
                                     _stream()), "gen_rays")
    return out


def pack_rays(ro, rd, height, width, focal, ndc, near, far, use_viewdirs, stride=None):
    """[o d near far (viewdir)] rows from caller-supplied origins / directions (train_utils.py:143-168);
    stride 6 returns [o d] only (ndc_rays)."""
    lib = _lib.load()
    n = ro.shape[0]
    if stride is None:
        stride = 11 if use_viewdirs else 8
    out = torch.empty(n, stride, dtype=torch.float32, device=ro.device)
    _lib.check(lib.nerfb200_pack_rays(_ptr(ro), _ptr(rd), n, int(height), int(width), float(focal), int(bool(ndc)),
                                      float(near), float(far), int(bool(use_viewdirs)), stride, _ptr(out), _stream()),
               "pack_rays")
    return out


def encode(arch: ArchSpec, which: int, x: torch.Tensor) -> torch.Tensor:
    lib = _lib.load()
    n = x.shape[0]
    dim = arch.dim_dir if which else arch.dim_xyz
    out = torch.empty(n, dim, dtype=torch.float32, device=x.device)
    _lib.check(lib.nerfb200_encode(C.byref(arch.c_struct()), which, _ptr(x), n, _ptr(out), _stream()), "encode")
    return out


def stash_floats(arch: ArchSpec, n_points: int) -> int:
    return _lib.load().nerfb200_stash_floats(C.byref(arch.c_struct()), n_points)


def mlp_fwd(arch: ArchSpec, blob, rays, z, impl=IMPL_SIMT, want_stash=False):
    lib = _lib.load()
    n, s = z.shape
    raw = torch.empty(n, s, 4, dtype=torch.float32, device=z.device)
    stash = torch.empty(stash_floats(arch, n * s), dtype=torch.float32, device=z.device) if want_stash else None
    _lib.check(lib.nerfb200_mlp_fwd(C.byref(arch.c_struct()), _ptr(blob), _ptr(rays), rays.shape[1], _ptr(z), n, s,
                                    _ptr(raw), _ptr(stash), impl, _stream()), "mlp_fwd")
    return (raw, stash) if want_stash else raw


def impl_supported(arch: ArchSpec, n_samples: int, impl: int) -> bool:
    """Can `impl` run this architecture forward and backward (the library decides, not Python)?"""
    return _lib.load().nerfb200_impl_supported(C.byref(arch.c_struct()), int(n_samples), int(impl)) == _lib.OK


def impl_refusal(arch: ArchSpec, n_samples: int, impl: int) -> Optional[str]:
    """None when ``impl_supported(arch, n_samples, impl)``, else the library's reason."""
    lib = _lib.load()
    if lib.nerfb200_impl_supported(C.byref(arch.c_struct()), int(n_samples), int(impl)) == _lib.OK:
        return None
    return lib.nerfb200_last_error().decode(errors="replace")


def mlp_bwd(arch: ArchSpec, blob, rays, z, d_raw, stash, impl=IMPL_SIMT, flat_grad=None):
    """Parameter gradients, accumulated into ``flat_grad`` (a fresh zero vector when None).  Returns (flat_grad,
    scratch): scratch is the gradient stash for impl 0, the gradient blob for impl 1."""
    lib = _lib.load()
    n, s = z.shape
    n_scratch = lib.nerfb200_bwd_scratch_floats(C.byref(arch.c_struct()), n * s, impl)
    if n_scratch < 0:
        _lib.check(_lib.ERR_UNSUPPORTED, "mlp_bwd")  # the library's refusal, e.g. impl 3, which does not train
    gstash = torch.empty(n_scratch, dtype=torch.float32, device=z.device)
    if flat_grad is None:
        flat_grad = torch.zeros(arch.flat_param_count(), dtype=torch.float32, device=z.device)
    _lib.check(lib.nerfb200_mlp_bwd(C.byref(arch.c_struct()), _ptr(blob), _ptr(rays), rays.shape[1], _ptr(z), n, s,
                                    _ptr(d_raw), _ptr(stash), _ptr(gstash), _ptr(flat_grad), impl, _stream()),
               "mlp_bwd")
    return flat_grad, gstash


def mlp_dgrad(arch: ArchSpec, blob, d_raw, stash, impl=IMPL_SIMT, gstash=None):
    """First half of mlp_bwd: the pre-activation gradients of every layer (the gradient stash)."""
    lib = _lib.load()
    if gstash is None:
        gstash = torch.empty_like(stash)
    _lib.check(lib.nerfb200_mlp_dgrad(C.byref(arch.c_struct()), _ptr(blob), _ptr(d_raw), _ptr(stash), _ptr(gstash),
                                      d_raw.numel() // 4, impl, _stream()), "mlp_dgrad")
    return gstash


def mlp_wgrad(arch: ArchSpec, rays, z, d_raw, stash, gstash, impl=IMPL_SIMT, flat_grad=None):
    """Second half of mlp_bwd: dW = dY^T X over all points, accumulated into ``flat_grad``."""
    lib = _lib.load()
    n, s = z.shape
    if flat_grad is None:
        flat_grad = torch.zeros(arch.flat_param_count(), dtype=torch.float32, device=z.device)
    _lib.check(lib.nerfb200_mlp_wgrad(C.byref(arch.c_struct()), _ptr(rays), rays.shape[1], _ptr(z), n, s, _ptr(d_raw),
                                      _ptr(stash), _ptr(gstash), _ptr(flat_grad), impl, _stream()), "mlp_wgrad")
    return flat_grad


def _rows_ptr(dirs: Optional[torch.Tensor]):
    """(pointer, row stride) of an (n, 3) fp32 CUDA tensor whose rows may be any distance apart (a column slice of
    wider rows, or stride 0 for one shared row), or (None, 0)."""
    if dirs is None:
        return None, 0
    if not dirs.is_cuda or dirs.dtype != torch.float32:
        raise RuntimeError("nerfb200: view directions must be an fp32 CUDA tensor")
    if dirs.dim() != 2 or dirs.shape[1] != 3 or dirs.stride(1) != 1 or not 0 <= dirs.stride(0) < 2 ** 31:
        raise RuntimeError(f"nerfb200: view directions must be (n, 3) rows of unit column stride, got shape "
                           f"{tuple(dirs.shape)} strides {dirs.stride()}")
    return C.c_void_p(dirs.data_ptr()), dirs.stride(0)


def mlp_fwd_pts(arch: ArchSpec, blob, pts, dirs, impl=IMPL_SIMT, want_stash=False):
    """The MLP at caller-given points ``pts`` (n_rays, n_samples, 3); ``dirs`` (n_rays, 3) gives each row's view
    direction (None without view directions) and may be a strided view.  Returns raw (n_rays, n_samples, 4)[, stash]."""
    lib = _lib.load()
    n, s, _ = pts.shape
    raw = torch.empty(n, s, 4, dtype=torch.float32, device=pts.device)
    stash = torch.empty(stash_floats(arch, n * s), dtype=torch.float32, device=pts.device) if want_stash else None
    dptr, dstride = _rows_ptr(dirs)
    _lib.check(lib.nerfb200_mlp_fwd_pts(C.byref(arch.c_struct()), _ptr(blob), _ptr(pts), dptr, dstride, n, s, _ptr(raw),
                                        _ptr(stash), impl, _stream()), "mlp_fwd_pts")
    return (raw, stash) if want_stash else raw


def density_grad_refusal(arch: ArchSpec, impl: int = IMPL_TC) -> Optional[str]:
    """None when ``density_grad`` runs ``arch`` with ``impl``, else the library's reason (no device is touched)."""
    lib = _lib.load()
    if lib.nerfb200_density_grad_supported(C.byref(arch.c_struct()), int(impl)) == _lib.OK:
        return None
    return lib.nerfb200_last_error().decode(errors="replace")


def density_grad(arch: ArchSpec, blob, pts, impl=IMPL_TC):
    """(P, 4) = (sigma_raw, d sigma_raw / dx, dy, dz) at ``pts`` (P, 3), P >= 1 (include/nerfb200.h, "density
    gradient")."""
    lib = _lib.load()
    if pts.dim() != 2 or pts.shape[1] != 3:
        raise RuntimeError(f"nerfb200: density_grad takes points (P, 3), got {tuple(pts.shape)}")
    out = torch.empty(pts.shape[0], 4, dtype=torch.float32, device=pts.device)
    _lib.check(lib.nerfb200_density_grad(C.byref(arch.c_struct()), _ptr(blob), _ptr(pts), pts.shape[0], _ptr(out),
                                         int(impl), _stream()), "density_grad")
    return out


def mlp_bwd_pts(arch: ArchSpec, blob, dirs, d_raw, stash, impl=IMPL_SIMT, flat_grad=None):
    """Backward of ``mlp_fwd_pts`` w.r.t. the parameters, accumulated into ``flat_grad`` (a fresh zero vector when
    None); ``d_raw`` (n_rays, n_samples, 4).  Returns flat_grad."""
    lib = _lib.load()
    n, s, _ = d_raw.shape
    n_scratch = lib.nerfb200_bwd_scratch_floats(C.byref(arch.c_struct()), n * s, impl)
    if n_scratch < 0:
        _lib.check(_lib.ERR_UNSUPPORTED, "mlp_bwd_pts")
    gstash = torch.empty(n_scratch, dtype=torch.float32, device=d_raw.device)
    if flat_grad is None:
        flat_grad = torch.zeros(arch.flat_param_count(), dtype=torch.float32, device=d_raw.device)
    dptr, dstride = _rows_ptr(dirs)
    _lib.check(lib.nerfb200_mlp_bwd_pts(C.byref(arch.c_struct()), _ptr(blob), dptr, dstride, n, s, _ptr(d_raw),
                                        _ptr(stash), _ptr(gstash), _ptr(flat_grad), impl, _stream()), "mlp_bwd_pts")
    return flat_grad


def volume_render_fwd(raw, z, dirs, noise, noise_std, white_bkgd):
    """Compositing of caller-given samples: raw (n, s, 4), z (n, s), dirs (n, 3) rows (strided allowed), noise unit
    normals (n, s) or None.  Returns (out[n, 8] = [r g b disp acc depth 0 0], weights[n, s])."""
    lib = _lib.load()
    n, s = z.shape
    out = torch.empty(n, 8, dtype=torch.float32, device=z.device)
    w = torch.empty(n, s, dtype=torch.float32, device=z.device)
    dptr, dstride = _rows_ptr(dirs)
    _lib.check(lib.nerfb200_volume_render_fwd(_ptr(raw), _ptr(z), dptr, dstride, _ptr(noise), n, s, float(noise_std),
                                              int(bool(white_bkgd)), _ptr(out), _ptr(w), _stream()), "volume_render_fwd")
    return out, w


def volume_render_bwd(raw, z, dirs, noise, g_out, g_weights, noise_std, white_bkgd):
    """d_raw (n, s, 4) from the upstream gradients of every output: g_out (n, 8) incl. the depth slot, g_weights (n, s)
    or None."""
    lib = _lib.load()
    n, s = z.shape
    d_raw = torch.empty(n, s, 4, dtype=torch.float32, device=z.device)
    dptr, dstride = _rows_ptr(dirs)
    _lib.check(lib.nerfb200_volume_render_bwd(_ptr(raw), _ptr(z), dptr, dstride, _ptr(noise), _ptr(g_out),
                                              _ptr(g_weights), n, s, float(noise_std), int(bool(white_bkgd)),
                                              _ptr(d_raw), _stream()), "volume_render_bwd")
    return d_raw


def bwd_bytes_per_point(arch: ArchSpec) -> int:
    """HBM bytes the wgmma backward reads per point (activation tiles of its weight-gradient jobs, masks, d_raw)."""
    return int(_lib.load().nerfb200_bwd_bytes_per_point(C.byref(arch.c_struct())))


def composite_fwd(raw, z, rays, noise, noise_std, white_bkgd, want_weights=True):
    lib = _lib.load()
    n, s = z.shape
    out = torch.empty(n, 8, dtype=torch.float32, device=z.device)
    w = torch.empty(n, s, dtype=torch.float32, device=z.device) if want_weights else None
    _lib.check(lib.nerfb200_composite_fwd(_ptr(raw), _ptr(z), _ptr(rays), rays.shape[1], _ptr(noise), n, s,
                                          float(noise_std), int(bool(white_bkgd)), _ptr(out), _ptr(w), _stream()),
               "composite_fwd")
    return out, w


def composite_bwd(raw, z, rays, noise, g_out, noise_std, white_bkgd):
    lib = _lib.load()
    n, s = z.shape
    d_raw = torch.empty(n, s, 4, dtype=torch.float32, device=z.device)
    _lib.check(lib.nerfb200_composite_bwd(_ptr(raw), _ptr(z), _ptr(rays), rays.shape[1], _ptr(noise), _ptr(g_out), n,
                                          s, float(noise_std), int(bool(white_bkgd)), _ptr(d_raw), _stream()),
               "composite_bwd")
    return d_raw


def sample_pdf_merge(z_coarse, weights_coarse, u, n_fine, cdf_in=None, want_aux=False):
    """u: (n_rays, n_fine), or None for the det=True linspace (built in the kernel)."""
    lib = _lib.load()
    n, nc = z_coarse.shape
    if u is not None and tuple(u.shape) != (n, n_fine):
        raise ValueError(f"nerfb200 sample_pdf_merge: u has shape {tuple(u.shape)}, expected {(n, n_fine)}")
    dev = z_coarse.device
    z_fine = torch.empty(n, nc + n_fine, dtype=torch.float32, device=dev)
    zs = torch.empty(n, n_fine, dtype=torch.float32, device=dev) if want_aux else None
    inds = torch.empty(n, n_fine, dtype=torch.int32, device=dev) if want_aux else None
    cdf = torch.empty(n, nc - 1, dtype=torch.float32, device=dev) if want_aux else None
    _lib.check(lib.nerfb200_sample_pdf_merge(_ptr(z_coarse), _ptr(weights_coarse), _ptr(u), _ptr(cdf_in), n, nc, n_fine,
                                             _ptr(z_fine), _ptr(zs), _ptr(inds), _ptr(cdf), _stream()),
               "sample_pdf_merge")
    return (z_fine, zs, inds, cdf) if want_aux else z_fine


def adam_step(p, g, m, v, step, lr, beta1=0.9, beta2=0.999, eps=1e-8, grad_scale=1.0):
    lib = _lib.load()
    _lib.check(lib.nerfb200_adam_step(_ptr(p), _ptr(g), _ptr(m), _ptr(v), p.numel(), int(step), float(lr), float(beta1),
                                      float(beta2), float(eps), float(grad_scale), _stream()), "adam_step")


# ------------------------------------------------------------------------------------------------
# a training step whose step count lives on the device (include/nerfb200.h: every value that changes from one step to
# the next is read from ``step_dev``, an int64 CUDA tensor of one element holding the steps done before this one)
# ------------------------------------------------------------------------------------------------
def random_fill_dev(seed: int, step_dev, stream, n_rays: int, per_ray: int, ray_offset: int = 0, out=None):
    """``random_fill(SeededRandoms(seed, step, ray_offset), ...)`` with step = ``step_dev`` read when the kernel runs."""
    sid = RAND_STREAMS[stream] if isinstance(stream, str) else int(stream)
    if out is None:
        out = torch.empty(int(n_rays), int(per_ray), dtype=torch.float32, device=step_dev.device)
    _lib.check(_lib.load().nerfb200_random_fill_dev(C.byref(SeededRandoms(seed, 0, ray_offset).c_struct()),
                                                    _ptr(step_dev), sid, int(n_rays), int(per_ray), _ptr(out),
                                                    _stream()), "random_fill_dev")
    return out


def draw_workspace_bytes(n_pixels: int) -> int:
    n = _lib.load().nerfb200_draw_workspace_bytes(int(n_pixels))
    if n < 0:
        _lib.check(_lib.ERR_INVALID, f"draw_workspace_bytes (n_pixels {n_pixels})")
    return n


def draw_pixels(seed: int, step_dev, n_images: int, n_pixels: int, n: int, image=None, ids=None, workspace=None):
    """One image index out of ``n_images`` and ``n`` distinct pixel ids out of ``n_pixels`` from (seed, step): returns
    (image int64[1], ids int64[n]), both on the device."""
    dev = step_dev.device
    if image is None:
        image = torch.empty(1, dtype=torch.int64, device=dev)
    if ids is None:
        ids = torch.empty(int(n), dtype=torch.int64, device=dev)
    if workspace is None:
        workspace = torch.empty(draw_workspace_bytes(n_pixels), dtype=torch.uint8, device=dev)
    _lib.check(_lib.load().nerfb200_draw_pixels(int(seed), _ptr(step_dev), int(n_images), int(n_pixels), int(n),
                                                _ptr(image), _ptr(ids), _ptr(workspace), _stream()), "draw_pixels")
    return image, ids


def gen_rays_posed(poses, image, height, width, focal, pixel_ids, ndc=False, near=0.0, far=1.0, use_viewdirs=True,
                   out=None):
    """``gen_rays`` of the pose ``poses[image]`` of a device table (n_images, 3 | 4, 4), ``image`` an int64[1] tensor."""
    stride = 11 if use_viewdirs else 8
    if out is None:
        out = torch.empty(pixel_ids.numel(), stride, dtype=torch.float32, device=pixel_ids.device)
    _lib.check(_lib.load().nerfb200_gen_rays_posed(_ptr(poses), int(poses.shape[1]), _ptr(image), int(height),
                                                   int(width), float(focal), _ptr(pixel_ids), pixel_ids.numel(),
                                                   int(bool(ndc)), float(near), float(far), int(bool(use_viewdirs)),
                                                   stride, _ptr(out), _stream()), "gen_rays_posed")
    return out


def gather_rows(src, rows_per_image: int, image, ids, out=None):
    """Rows ``image * rows_per_image + ids`` of ``src`` (rows of 3 floats): (n, 3)."""
    if out is None:
        out = torch.empty(ids.numel(), 3, dtype=torch.float32, device=ids.device)
    _lib.check(_lib.load().nerfb200_gather_rows(_ptr(src), int(rows_per_image), _ptr(image), _ptr(ids), ids.numel(),
                                                _ptr(out), _stream()), "gather_rows")
    return out


def mse_loss(out_c, out_f, target, loss=None, g_c=None, g_f=None):
    """mse(out_c[:, :3], target) (+ the same of out_f) into a 0-dim tensor, and the (n, 8) upstream gradients of
    ``render_bwd``.  Returns (loss, g_c, g_f)."""
    n = out_c.shape[0]
    dev = out_c.device
    if loss is None:
        loss = torch.empty((), dtype=torch.float32, device=dev)
    if g_c is None:
        g_c = torch.empty(n, 8, dtype=torch.float32, device=dev)
    if out_f is not None and g_f is None:
        g_f = torch.empty(n, 8, dtype=torch.float32, device=dev)
    _lib.check(_lib.load().nerfb200_mse_loss(_ptr(out_c), _ptr(out_f), _ptr(target), n, _ptr(loss), _ptr(g_c),
                                             _ptr(g_f), _stream()), "mse_loss")
    return loss, g_c, g_f


def _schedule(lr0, lr_decay, lr_decay_factor):
    return float(lr0), (0.0 if lr_decay is None else float(lr_decay)), float(lr_decay_factor)


def lr_schedule(done, lr0, lr_decay=None, lr_decay_factor=0.1):
    """The fp32 rate ``parallel.FusedAdam`` uses after ``done`` (int64 CUDA tensor) steps, computed on the device."""
    out = torch.empty(done.numel(), dtype=torch.float32, device=done.device)
    _lib.check(_lib.load().nerfb200_lr_schedule(_ptr(done), done.numel(), *_schedule(lr0, lr_decay, lr_decay_factor),
                                                _ptr(out), _stream()), "lr_schedule")
    return out


def adam_step_dev(p, g, m, v, step_dev, lr0, lr_decay=None, lr_decay_factor=0.1, beta1=0.9, beta2=0.999, eps=1e-8,
                  grad_scale=1.0):
    """``adam_step`` of step ``step_dev + 1`` at the scheduled rate, both read on the device."""
    _lib.check(_lib.load().nerfb200_adam_step_dev(_ptr(p), _ptr(g), _ptr(m), _ptr(v), p.numel(), _ptr(step_dev),
                                                  *_schedule(lr0, lr_decay, lr_decay_factor), float(beta1),
                                                  float(beta2), float(eps), float(grad_scale), _stream()),
               "adam_step_dev")


def step_advance(step_dev):
    _lib.check(_lib.load().nerfb200_step_advance(_ptr(step_dev), _stream()), "step_advance")


# ------------------------------------------------------------------------------------------------
# whole path
# ------------------------------------------------------------------------------------------------
WS_SECTIONS = ("z_coarse", "raw_coarse", "weights_coarse", "z_fine", "raw_fine", "stash_coarse", "stash_fine",
               "gstash", "d_raw")


def _archs(arch_c, arch_f):
    """The C arguments of a coarse and an optional fine ArchSpec."""
    return C.byref(arch_c.c_struct()), (C.byref(arch_f.c_struct()) if arch_f is not None else None)


def _render_bytes(query, arch_c, arch_f, opts: RenderOpts, n_rays: int, *rest) -> int:
    """The workspace bytes nerfb200_<query> returns; its -1 raises NotImplementedError."""
    n = getattr(_lib.load(), "nerfb200_" + query)(*_archs(arch_c, arch_f), C.byref(opts), n_rays, *rest)
    if n < 0:
        _lib.check(_lib.ERR_UNSUPPORTED, query)
    return n


def render_workspace_bytes(arch_c, arch_f, opts: RenderOpts, n_rays: int, training: bool) -> int:
    return _render_bytes("render_workspace_bytes", arch_c, arch_f, opts, n_rays, int(training))


def render_workspace_layout(arch_c, arch_f, opts: RenderOpts, n_rays: int, training: bool) -> dict:
    offs = (C.c_int64 * 9)()
    _lib.check(_lib.load().nerfb200_render_workspace_layout(*_archs(arch_c, arch_f), C.byref(opts), n_rays,
                                                            int(training), offs), "workspace_layout")
    return dict(zip(WS_SECTIONS, list(offs)))


def _random_args(randoms):
    """The C arguments (rng, t_rand, noise_c, u, noise_f) of a render call.  ``randoms`` is a ``SeededRandoms`` (the
    kernels generate all four inputs) or a dict of tensors keyed by RAND_STREAMS (a missing key: not supplied)."""
    if isinstance(randoms, SeededRandoms):
        return (C.byref(randoms.c_struct()), None, None, None, None)
    return (None,) + tuple(_ptr(randoms.get(k)) for k in RAND_STREAMS)


def _render_call(query, arch_c, arch_f, opts: RenderOpts, blob_c, blob_f, rays, randoms, grid, workspace, *rest):
    """What the forward render calls share.  Returns (args, grid_args, out_c, out_f, workspace): the leading C
    arguments (the arch pair, options, blobs, rays and random inputs), the optional grid's (descriptor, bits) checked
    to be on the rays' device, the outputs, and ``workspace`` when it holds nerfb200_<query>'s bytes, else a new one."""
    n, dev = rays.shape[0], rays.device
    fine = opts.n_fine > 0
    af = arch_f if fine else None
    grid_args = (None, None)
    if grid is not None:
        g, bits = _grid_args(grid)
        if bits.device != dev:
            raise RuntimeError(f"nerfb200: the grid is on {bits.device}, the rays on {dev}")
        grid_args = (C.byref(g), _ptr(bits))
    need = _render_bytes(query, arch_c, af, opts, n, *rest)
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, dtype=torch.uint8, device=dev)
    out_c = torch.empty(n, 8, dtype=torch.float32, device=dev)
    out_f = torch.empty(n, 8, dtype=torch.float32, device=dev) if fine else None
    args = (*_archs(arch_c, af), C.byref(opts), _ptr(blob_c), _ptr(blob_f) if fine else None, _ptr(rays),
            rays.shape[1], n, *_random_args(randoms))
    return args, grid_args, out_c, out_f, workspace


def render_fwd(arch_c, arch_f, opts: RenderOpts, blob_c, blob_f, rays, randoms, training: bool, impl: int = IMPL_SIMT,
               workspace: Optional[torch.Tensor] = None):
    """One ray chunk through the whole path.  Returns (out_coarse[N,8], out_fine[N,8] | None, workspace)."""
    args, _, out_c, out_f, workspace = _render_call("render_workspace_bytes", arch_c, arch_f, opts, blob_c, blob_f,
                                                    rays, randoms, None, workspace, int(training))
    _lib.check(_lib.load().nerfb200_render_fwd(*args, _ptr(out_c), _ptr(out_f), _ptr(workspace), int(training), impl,
                                               _stream()), "render_fwd")
    return out_c, out_f, workspace


def render_bwd(arch_c, arch_f, opts: RenderOpts, blob_c, blob_f, rays, randoms, g_c, g_f, workspace, flat_grad_c,
               flat_grad_f, impl: int = IMPL_SIMT, parts: int = 3):
    """Backward of a ``render_fwd`` workspace, given the same ``randoms`` (only the noise is needed again: a
    ``SeededRandoms`` regenerates it in-kernel, a dict supplies the tensors)."""
    fine = opts.n_fine > 0
    rng, _, noise_c, _, noise_f = _random_args(randoms)
    _lib.check(_lib.load().nerfb200_render_bwd(*_archs(arch_c, arch_f if fine else None), C.byref(opts), _ptr(blob_c),
                                               _ptr(blob_f) if fine else None, _ptr(rays), rays.shape[1],
                                               rays.shape[0], rng, noise_c, noise_f, _ptr(g_c),
                                               _ptr(g_f) if fine else None, _ptr(workspace), _ptr(flat_grad_c),
                                               _ptr(flat_grad_f) if fine else None, impl, int(parts), _stream()),
               "render_bwd")


# ------------------------------------------------------------------------------------------------
# occupancy grid (include/nerfb200.h "occupancy grid"; nerf_pytorch_b200/occupancy.py builds the grids)
# ------------------------------------------------------------------------------------------------
def grid_struct(bounds, resolution) -> Grid:
    """nerfb200_grid_t of ``bounds`` ((lo_x, lo_y, lo_z), (hi_x, hi_y, hi_z)) and ``resolution`` (three ints)."""
    g = Grid()
    (lo, hi), res = bounds, resolution
    for c in range(3):
        g.lo[c], g.hi[c], g.res[c] = float(lo[c]), float(hi[c]), int(res[c])
    return g


def grid_words(g: Grid) -> int:
    n = _lib.load().nerfb200_grid_words(C.byref(g))
    if n < 0:
        _lib.check(_lib.ERR_INVALID, "grid_words")
    return int(n)


def grid_locate(g: Grid, xyz: torch.Tensor) -> torch.Tensor:
    """The library's host restatement of the cell rule: int64 cell index of each (n, 3) CPU point, -1 outside."""
    x = xyz.detach().to(device="cpu", dtype=torch.float32).contiguous()
    out = torch.empty(x.shape[0], dtype=torch.int64)
    _lib.check(_lib.load().nerfb200_grid_locate(C.byref(g), C.cast(x.data_ptr(), C.POINTER(C.c_float)), x.shape[0],
                                                C.cast(out.data_ptr(), C.POINTER(C.c_int64))), "grid_locate")
    return out


def _grid_args(grid):
    """(descriptor, bits) of an OccupancyGrid-like object: ``.c_struct()`` and ``.bits`` (int32 words on the device)."""
    bits = grid.bits
    if not bits.is_cuda or bits.dtype != torch.int32 or bits.dim() != 1 or not bits.is_contiguous():
        raise RuntimeError("nerfb200: the grid's bits must be a contiguous 1-d int32 CUDA tensor")
    g = grid.c_struct()
    if bits.numel() != grid_words(g):
        raise RuntimeError(f"nerfb200: the grid's bits hold {bits.numel()} words, its resolution needs {grid_words(g)}")
    return g, bits


def grid_compact(grid, rays, z, raw=None):
    """Sample compaction of one pass (nerfb200_grid_compact): writes [0 0 0 -inf] into ``raw`` (n, s, 4) at every
    skipped sample and returns (raw, map int32[rows], blocks int32[max_blocks, 2], n_blocks int32[1],
    n_evaluated int64[1]); rows past 64 * n_blocks are not written."""
    lib = _lib.load()
    g, bits = _grid_args(grid)
    n, s = z.shape
    dev = z.device
    if raw is None:
        raw = torch.zeros(n, s, 4, dtype=torch.float32, device=dev)
    mb = lib.nerfb200_grid_max_blocks(n, s)
    if mb < 0:
        _lib.check(_lib.ERR_INVALID, "grid_max_blocks")
    m = torch.full((mb * 64,), -2, dtype=torch.int32, device=dev)
    blocks = torch.full((mb, 2), -2, dtype=torch.int32, device=dev)
    nb = torch.empty(1, dtype=torch.int32, device=dev)
    ne = torch.empty(1, dtype=torch.int64, device=dev)
    scratch = torch.empty(lib.nerfb200_grid_scratch_ints(n, s), dtype=torch.int32, device=dev)
    _lib.check(lib.nerfb200_grid_compact(C.byref(g), _ptr(bits), _ptr(rays), rays.shape[1], _ptr(z), n, s, _ptr(raw),
                                         _ptr(m), _ptr(blocks), _ptr(nb), _ptr(ne), _ptr(scratch), _stream()),
               "grid_compact")
    return raw, m, blocks, nb, ne


def render_grid_workspace_bytes(arch_c, arch_f, opts: RenderOpts, n_rays: int) -> int:
    return _render_bytes("render_grid_workspace_bytes", arch_c, arch_f, opts, n_rays)


def render_fwd_grid(arch_c, arch_f, opts: RenderOpts, blob_c, blob_f, rays, randoms, grid, impl: int = IMPL_TC,
                    workspace: Optional[torch.Tensor] = None, n_evaluated: Optional[torch.Tensor] = None):
    """``render_fwd`` for inference with an occupancy grid (impl 1 or 3).  ``n_evaluated``: an int64 CUDA tensor of 2
    receiving the evaluated samples of the coarse and fine pass, or None.  Returns (out_coarse, out_fine | None,
    workspace); the workspace's first sections are laid out as ``render_workspace_layout(..., training=False)``."""
    args, grid_args, out_c, out_f, workspace = _render_call("render_grid_workspace_bytes", arch_c, arch_f, opts,
                                                            blob_c, blob_f, rays, randoms, grid, workspace)
    if n_evaluated is not None and (n_evaluated.dtype != torch.int64 or n_evaluated.numel() < 2):
        raise RuntimeError("nerfb200: n_evaluated must be an int64 tensor of 2 elements")
    _lib.check(_lib.load().nerfb200_render_fwd_grid(*args, *grid_args, _ptr(out_c), _ptr(out_f), _ptr(workspace),
                                                    int(impl), _ptr(n_evaluated), _stream()), "render_fwd_grid")
    return out_c, out_f, workspace


# ------------------------------------------------------------------------------------------------
# early ray termination (include/nerfb200.h "early ray termination")
# ------------------------------------------------------------------------------------------------
def stop_round() -> int:
    """K: the evaluated samples per ray each round of an early-stopping pass runs (NERFB200_STOP_ROUND)."""
    return int(_lib.load().nerfb200_render_early_stop_round())


def render_early_stop_workspace_bytes(arch_c, arch_f, opts: RenderOpts, n_rays: int) -> int:
    return _render_bytes("render_early_stop_workspace_bytes", arch_c, arch_f, opts, n_rays)


def render_fwd_normals(arch_c, arch_f, opts: RenderOpts, blob_c, blob_f, rays, randoms, grid=None,
                       stop: Optional[float] = None, impl: int = IMPL_TC, ndc: Optional[Ndc] = None):
    """Inference ``render_fwd`` (with an occupancy ``grid`` and / or early stopping at ``stop`` when given) that also
    returns the normal map of the last pass (include/nerfb200.h, "normal maps").  ``ndc`` (an ``ndc_struct``) makes it
    the world-space normal map of an NDC render of that camera ("NDC scenes").  Returns (out_coarse, out_fine | None,
    normals[N, 3], workspace); the workspace's first sections are laid out as ``render_workspace_layout(...,
    training=False)``."""
    args, grid_args, out_c, out_f, workspace = _render_call("render_normals_workspace_bytes", arch_c, arch_f, opts,
                                                            blob_c, blob_f, rays, randoms, grid, None)
    normals = torch.empty(rays.shape[0], 3, dtype=torch.float32, device=rays.device)
    lib = _lib.load()
    head = (*args, *grid_args, -1.0 if stop is None else float(stop))
    tail = (_ptr(out_c), _ptr(out_f), _ptr(normals), _ptr(workspace), int(impl), _stream())
    if ndc is None:
        _lib.check(lib.nerfb200_render_fwd_normals(*head, *tail), "render_fwd_normals")
    else:
        _lib.check(lib.nerfb200_render_fwd_normals_ndc(*head, C.byref(ndc), *tail), "render_fwd_normals_ndc")
    return out_c, out_f, normals, workspace


def render_fwd_early_stop(arch_c, arch_f, opts: RenderOpts, blob_c, blob_f, rays, randoms, grid, stop,
                          impl: int = IMPL_TC, want_stop: bool = False, workspace: Optional[torch.Tensor] = None):
    """``render_fwd`` for inference (impl 1 or 3) whose last pass stops each ray once its transmittance falls below
    ``stop`` (0 <= stop < 1), with an occupancy ``grid`` or None.  Returns (out_coarse, out_fine | None, n_evaluated
    int64[2]) and, with ``want_stop``, the int32 ``stop_sample`` of every ray (the header's definition).  A given
    ``workspace`` large enough is used; its first sections are laid out as ``render_workspace_layout(...,
    training=False)``."""
    args, grid_args, out_c, out_f, workspace = _render_call("render_early_stop_workspace_bytes", arch_c, arch_f,
                                                            opts, blob_c, blob_f, rays, randoms, grid, workspace)
    n, dev = rays.shape[0], rays.device
    n_evaluated = torch.zeros(2, dtype=torch.int64, device=dev)
    stop_sample = torch.empty(n, dtype=torch.int32, device=dev) if want_stop else None
    _lib.check(_lib.load().nerfb200_render_fwd_early_stop(*args, *grid_args, float(stop), _ptr(out_c), _ptr(out_f),
                                                          _ptr(workspace), int(impl), _ptr(n_evaluated),
                                                          _ptr(stop_sample), _stream()), "render_fwd_early_stop")
    if want_stop:
        return out_c, out_f, n_evaluated, stop_sample
    return out_c, out_f, n_evaluated


# ------------------------------------------------------------------------------------------------
# meshes (include/nerfb200.h "meshes"; nerf_pytorch_b200/mesh.py is the public interface).  The box is a Grid read as
# res cubes per axis, its lattice the (res + 1) points per axis at the cube corners.
# ------------------------------------------------------------------------------------------------
def mesh_workspace_bytes(box: Grid) -> int:
    n = _lib.load().nerfb200_mesh_workspace_bytes(C.byref(box))
    if n < 0:
        _lib.check(_lib.ERR_INVALID, "mesh_workspace_bytes")
    return int(n)


def mesh_lattice_points(box: Grid, z0: int, nz: int, out: torch.Tensor) -> torch.Tensor:
    """The lattice points of planes z0 .. z0 + nz - 1 into the first nz * (res_y + 1) * (res_x + 1) rows of ``out``
    (fp32 CUDA, (rows, 3) or anything of that many floats)."""
    _lib.check(_lib.load().nerfb200_mesh_lattice_points(C.byref(box), int(z0), int(nz), _ptr(out), _stream()),
               "mesh_lattice_points")
    return out


def mesh_count(box: Grid, volume: torch.Tensor, level: float, workspace: Optional[torch.Tensor] = None):
    """Classify and scan: returns (totals int64[2] = [vertices, faces] on the device, workspace)."""
    need = mesh_workspace_bytes(box)
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, dtype=torch.uint8, device=volume.device)
    totals = torch.empty(2, dtype=torch.int64, device=volume.device)
    _lib.check(_lib.load().nerfb200_mesh_count(C.byref(box), _ptr(volume), float(level), _ptr(workspace), _ptr(totals),
                                               _stream()), "mesh_count")
    return totals, workspace


def mesh_emit(box: Grid, volume: torch.Tensor, level: float, workspace: torch.Tensor, n_vertices: int, n_faces: int,
              want_dirs: bool = False):
    """Vertices (V, 3) fp32, faces (F, 3) int32 and, with ``want_dirs``, each vertex's view direction (V, 3)."""
    dev = volume.device
    verts = torch.empty(n_vertices, 3, dtype=torch.float32, device=dev)
    faces = torch.empty(n_faces, 3, dtype=torch.int32, device=dev)
    dirs = torch.empty(n_vertices, 3, dtype=torch.float32, device=dev) if want_dirs else None
    _lib.check(_lib.load().nerfb200_mesh_emit(C.byref(box), _ptr(volume), float(level), _ptr(workspace),
                                              int(n_vertices), int(n_faces), _ptr(verts) if n_vertices else None,
                                              _ptr(faces) if n_faces else None,
                                              _ptr(dirs) if want_dirs and n_vertices else None, _stream()),
               "mesh_emit")
    return verts, faces, dirs


# ------------------------------------------------------------------------------------------------
# sparse meshes (include/nerfb200.h "sparse meshes"): marching cubes over the bricks an occupancy grid calls occupied
# ------------------------------------------------------------------------------------------------
def mesh_brick() -> int:
    """Cubes per brick axis (NERFB200_MESH_BRICK)."""
    return int(_lib.load().nerfb200_mesh_brick())


def mesh_sparse_brick_count(box: Grid) -> int:
    n = _lib.load().nerfb200_mesh_sparse_brick_count(C.byref(box))
    if n < 0:
        _lib.check(_lib.ERR_INVALID, "mesh_sparse_brick_count")
    return int(n)


def mesh_sparse_workspace_bytes(box: Grid, n_active: int) -> int:
    n = _lib.load().nerfb200_mesh_sparse_workspace_bytes(C.byref(box), int(n_active))
    if n < 0:
        _lib.check(_lib.ERR_INVALID, "mesh_sparse_workspace_bytes")
    return int(n)


def mesh_sparse_scratch_bytes(box: Grid) -> int:
    n = _lib.load().nerfb200_mesh_sparse_scratch_bytes(C.byref(box))
    if n < 0:
        _lib.check(_lib.ERR_INVALID, "mesh_sparse_scratch_bytes")
    return int(n)


def mesh_sparse_bricks(box: Grid, grid):
    """The activity test of an OccupancyGrid-like ``grid`` over the box's bricks: (brick_map int32[bricks] = slot or
    -1, bricks int32[bricks] whose first n_active entries are the active bricks in order, n_active int64[1] on the
    device)."""
    lib = _lib.load()
    g, bits = _grid_args(grid)
    n = mesh_sparse_brick_count(box)
    dev = bits.device
    brick_map = torch.empty(n, dtype=torch.int32, device=dev)
    bricks = torch.empty(n, dtype=torch.int32, device=dev)
    n_active = torch.empty(1, dtype=torch.int64, device=dev)
    scratch = torch.empty(mesh_sparse_scratch_bytes(box), dtype=torch.uint8, device=dev)
    _lib.check(lib.nerfb200_mesh_sparse_bricks(C.byref(box), C.byref(g), _ptr(bits), _ptr(brick_map), _ptr(bricks),
                                               _ptr(n_active), _ptr(scratch), _stream()), "mesh_sparse_bricks")
    return brick_map, bricks, n_active


def mesh_sparse_bricks_host(box: Grid, grid: Grid, bits: torch.Tensor) -> torch.Tensor:
    """The library's host statement of the activity test: bool[bricks] from int32 grid words on the CPU."""
    b = bits.detach().to(device="cpu", dtype=torch.int32).contiguous()
    out = torch.empty(mesh_sparse_brick_count(box), dtype=torch.uint8)
    _lib.check(_lib.load().nerfb200_mesh_sparse_bricks_host(C.byref(box), C.byref(grid), C.c_void_p(b.data_ptr()),
                                                            C.c_void_p(out.data_ptr())), "mesh_sparse_bricks_host")
    return out.bool()


def mesh_sparse_points(box: Grid, bricks: torch.Tensor, first: int, count: int, halo: bool, out: torch.Tensor):
    """The lattice points of active slots first .. first + count - 1, brick-major (with the one-point halo when
    ``halo``), into the first count * P rows of ``out`` (fp32 CUDA, P = (B + 1 + 2 halo)^3)."""
    _lib.check(_lib.load().nerfb200_mesh_sparse_points(C.byref(box), _ptr(bricks), int(first), int(count), int(halo),
                                                       _ptr(out), _stream()), "mesh_sparse_points")
    return out


def mesh_sparse_count(box: Grid, brick_map, bricks, n_active: int, values, halo: bool, level: float,
                      workspace: Optional[torch.Tensor] = None):
    """Classify and scan over the active bricks' values: (totals int64[2] on the device, workspace)."""
    need = mesh_sparse_workspace_bytes(box, n_active)
    dev = brick_map.device
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(max(need, 1), dtype=torch.uint8, device=dev)
    totals = torch.empty(2, dtype=torch.int64, device=dev)
    _lib.check(_lib.load().nerfb200_mesh_sparse_count(C.byref(box), _ptr(brick_map), _ptr(bricks), int(n_active),
                                                      _ptr(values), int(halo), float(level), _ptr(workspace),
                                                      _ptr(totals), _stream()), "mesh_sparse_count")
    return totals, workspace


def mesh_sparse_emit(box: Grid, brick_map, bricks, n_active: int, values, halo: bool, level: float, workspace,
                     n_vertices: int, n_faces: int, want_dirs: bool = False, want_keys: bool = False):
    """Vertices (V, 3) fp32, faces (F, 3) int32, view directions (V, 3) with ``want_dirs`` (needs the halo) and the
    lattice edge key q * 3 + a of each vertex, int64 (V,), with ``want_keys``."""
    dev = brick_map.device
    verts = torch.empty(n_vertices, 3, dtype=torch.float32, device=dev)
    faces = torch.empty(n_faces, 3, dtype=torch.int32, device=dev)
    dirs = torch.empty(n_vertices, 3, dtype=torch.float32, device=dev) if want_dirs else None
    keys = torch.empty(n_vertices, dtype=torch.int64, device=dev) if want_keys else None
    nv = n_vertices > 0
    _lib.check(_lib.load().nerfb200_mesh_sparse_emit(
        C.byref(box), _ptr(brick_map), _ptr(bricks), int(n_active), _ptr(values), int(halo), float(level),
        _ptr(workspace), int(n_vertices), int(n_faces), _ptr(verts) if nv else None, _ptr(faces) if n_faces else None,
        _ptr(dirs) if want_dirs and nv else None, _ptr(keys) if want_keys and nv else None, _stream()),
        "mesh_sparse_emit")
    return verts, faces, dirs, keys


# ------------------------------------------------------------------------------------------------
# NDC scenes (include/nerfb200.h "NDC scenes"): the map N of ndc_rays between world space and the NDC points a
# forward-facing scene's MLP encodes, and its Jacobian
# ------------------------------------------------------------------------------------------------
def ndc_struct(height: int, width: int, focal: float) -> Ndc:
    """The nerfb200_ndc_t of an image of ``height`` x ``width`` pixels and focal length ``focal`` (the call's H, W,
    focal: the NDC map of its rays)."""
    return Ndc(int(height), int(width), float(focal))


def ndc_mesh_to_world(ndc: Ndc, vertices, faces, view_dirs=None):
    """A mesh extracted in NDC, in world space: (N^-1 of each vertex (V, 3), faces (F, 3) with their last two ids
    swapped, and with ``view_dirs`` each one's unit world direction J^T d, else None).  New tensors; the inputs are
    kept."""
    nv, nf = vertices.shape[0], faces.shape[0]
    wv, wf = torch.empty_like(vertices), torch.empty_like(faces)
    wd = torch.empty_like(view_dirs) if view_dirs is not None else None
    _lib.check(_lib.load().nerfb200_ndc_mesh_to_world(
        C.byref(ndc), _ptr(vertices) if nv else None, _ptr(faces) if nf else None,
        _ptr(view_dirs) if view_dirs is not None and nv else None, nv, nf, _ptr(wv) if nv else None,
        _ptr(wf) if nf else None, _ptr(wd) if wd is not None and nv else None, _stream()), "ndc_mesh_to_world")
    return wv, wf, wd


def ndc_from_world(ndc: Ndc, pts) -> torch.Tensor:
    """q = N(p) for world points ``pts`` (P, 3)."""
    q = torch.empty_like(pts)
    _lib.check(_lib.load().nerfb200_ndc_from_world(C.byref(ndc), _ptr(pts) if pts.shape[0] else None, pts.shape[0],
                                                   _ptr(q) if pts.shape[0] else None, _stream()), "ndc_from_world")
    return q


def ndc_grad_to_world(ndc: Ndc, q, rows, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """(sigma, J^T(q) g) of ``density_grad`` rows (P, 4) = (sigma, g) at NDC points ``q`` (P, 3); ``out`` may be
    ``rows``."""
    out = torch.empty_like(rows) if out is None else out
    n = q.shape[0]
    _lib.check(_lib.load().nerfb200_ndc_grad_to_world(C.byref(ndc), _ptr(q) if n else None, _ptr(rows) if n else None,
                                                      n, _ptr(out) if n else None, _stream()), "ndc_grad_to_world")
    return out


# ------------------------------------------------------------------------------------------------
# baked fields (include/nerfb200.h "baked fields"): density and SH colour coefficients on the bricks of a lattice
# ------------------------------------------------------------------------------------------------
def bake_dirs() -> int:
    """Directions a bake evaluates the colour at (NERFB200_BAKE_DIRS)."""
    return 64


def bake_basis() -> Tuple[torch.Tensor, torch.Tensor]:
    """The library's bake directions (64, 3) and SH projection M (9, 64), fp32 CPU tensors."""
    dirs = torch.empty(bake_dirs(), 3, dtype=torch.float32)
    proj = torch.empty(9, bake_dirs(), dtype=torch.float32)
    f = C.POINTER(C.c_float)
    _lib.check(_lib.load().nerfb200_bake_basis(C.cast(dirs.data_ptr(), f), C.cast(proj.data_ptr(), f)), "bake_basis")
    return dirs, proj


def bake_refusal(arch: ArchSpec) -> Optional[str]:
    """None when ``bake`` runs ``arch``, else the library's reason (no device is touched)."""
    lib = _lib.load()
    if lib.nerfb200_bake_supported(C.byref(arch.c_struct())) == _lib.OK:
        return None
    return lib.nerfb200_last_error().decode(errors="replace")


def _baked_values(values, what, dequant=None):
    """(entry point suffix, the values' leading arguments) of baked ``values``: "" and (pointer,) for fp32, "_f16" and
    (pointer,) for fp16 (include/nerfb200.h "baked fields: half precision"), "_u8" and (codes, ``dequant``) for uint8
    codes, whose ``dequant`` must be their fp32 (2, 28) table on the same device (include/nerfb200.h "baked fields:
    8-bit values"); any other dtype is refused."""
    if values.dtype == torch.float32:
        return "", (_ptr(values),)
    if values.dtype == torch.float16:
        return "_f16", (_ptr(values.view(torch.uint8)),)  # _ptr takes no fp16; the pointer is the same
    if values.dtype == torch.uint8:
        if not (isinstance(dequant, torch.Tensor) and dequant.dtype == torch.float32 and dequant.shape == (2, 28)
                and dequant.device == values.device):
            raise ValueError(f"nerfb200 {what}: uint8 baked values need their dequant, an fp32 (2, 28) tensor on "
                             f"{values.device}")
        return "_u8", (_ptr(values), _ptr(dequant))
    raise ValueError(f"nerfb200 {what}: baked values must be fp32 or fp16, or uint8 with their dequant, got "
                     f"{values.dtype}")


def bake(arch: ArchSpec, blob, box: Grid, bricks, first: int, count: int, values, logits=None):
    """The values of slots first .. first + count - 1 into ``values`` (n_active, 729, 32), fp32 or fp16 (the conversion
    rule at the store); ``logits`` (count * 729, 64, 3) fp32 or None receives the network's rgb logits at the 64
    directions (a test hook)."""
    if values.dtype == torch.uint8:
        raise ValueError("nerfb200 bake: a bake writes fp32 or fp16 values; quantise the baked field afterwards")
    sfx, (pv,) = _baked_values(values, "bake")
    _lib.check(getattr(_lib.load(), "nerfb200_bake" + sfx)(C.byref(arch.c_struct()), _ptr(blob), C.byref(box),
                                                           _ptr(bricks), int(first), int(count), pv, _ptr(logits),
                                                           _stream()), "bake" + sfx)
    return values


def baked_render(box: Grid, brick_map, values, use_viewdirs: bool, rays, white_background: bool,
                 stop_transmittance: float = 0.0, out=None, dequant=None) -> torch.Tensor:
    """Rows (n, 8) = [r g b disp acc depth 0 0] of the packed ``rays`` through a baked field whose ``values`` are fp32
    or fp16, or uint8 codes with their ``dequant`` table."""
    sfx, pv = _baked_values(values, "baked_render", dequant)
    n = rays.shape[0]
    out = torch.empty(n, 8, dtype=torch.float32, device=rays.device) if out is None else out
    _lib.check(getattr(_lib.load(), "nerfb200_baked_render" + sfx)(
        C.byref(box), _ptr(brick_map), *pv, int(bool(use_viewdirs)), _ptr(rays), rays.shape[1], n,
        int(bool(white_background)), float(stop_transmittance), _ptr(out), _stream()), "baked_render" + sfx)
    return out


def baked_render_normals(box: Grid, brick_map, values, use_viewdirs: bool, rays, white_background: bool,
                         stop_transmittance: float = 0.0, ndc: Optional[Ndc] = None, dequant=None):
    """(rows (n, 8) bit for bit ``baked_render``'s, normal map (n, 3)) of the packed ``rays`` through a baked field
    (include/nerfb200.h "baked fields: normal maps and point queries"): the sum of w (-g / |g|) in sample order, g the
    gradient of the trilinear sigma_raw, in the field's frame, or with ``ndc`` (``ndc_struct`` of the rays' camera)
    mapped to world space by J^T first."""
    sfx, pv = _baked_values(values, "baked_render_normals", dequant)
    n = rays.shape[0]
    out = torch.empty(n, 8, dtype=torch.float32, device=rays.device)
    normals = torch.empty(n, 3, dtype=torch.float32, device=rays.device)
    _lib.check(getattr(_lib.load(), "nerfb200_baked_render_normals" + sfx)(
        C.byref(box), _ptr(brick_map), *pv, int(bool(use_viewdirs)), _ptr(rays), rays.shape[1], n,
        int(bool(white_background)), float(stop_transmittance), None if ndc is None else C.byref(ndc), _ptr(out),
        _ptr(normals), _stream()), "baked_render_normals" + sfx)
    return out, normals


def baked_query(box: Grid, brick_map, values, use_viewdirs: bool, pts, dirs=None, want_raw: bool = True,
                want_grad: bool = True, dequant=None):
    """(raw (P, 4) or None, grad (P, 3) or None) of a baked field at the field-frame points ``pts`` (P, 3)
    (include/nerfb200.h "baked fields: normal maps and point queries"): raw = (s_r, s_g, s_b, sigma_raw) with the
    logits seen along ``dirs`` (P, 3, read with view directions only) and grad the gradient of the trilinear
    sigma_raw."""
    sfx, pv = _baked_values(values, "baked_query", dequant)
    n = pts.shape[0]
    raw = torch.empty(n, 4, dtype=torch.float32, device=pts.device) if want_raw else None
    grad = torch.empty(n, 3, dtype=torch.float32, device=pts.device) if want_grad else None
    _lib.check(getattr(_lib.load(), "nerfb200_baked_query" + sfx)(
        C.byref(box), _ptr(brick_map), *pv, int(bool(use_viewdirs)), _ptr(pts), _ptr(dirs), n, _ptr(raw), _ptr(grad),
        _stream()), "baked_query" + sfx)
    return raw, grad


def baked_render_bwd(box: Grid, brick_map, values, use_viewdirs: bool, rays, white_background: bool, out, g_out,
                     d_values):
    """Adds into ``d_values`` (the layout of ``values``) the gradient of ``baked_render`` (stop 0) whose rows were
    ``out``, given upstream gradient rows ``g_out`` (n, 8).  Untied: see ``baked_tie``."""
    _lib.check(_lib.load().nerfb200_baked_render_bwd(C.byref(box), _ptr(brick_map), _ptr(values),
                                                     int(bool(use_viewdirs)), _ptr(rays), rays.shape[1], rays.shape[0],
                                                     int(bool(white_background)), _ptr(out), _ptr(g_out),
                                                     _ptr(d_values), _stream()), "baked_render_bwd")
    return d_values


def baked_tie(box: Grid, brick_map, bricks, d_values, d_tied=None):
    """Every stored copy of a lattice point receives the sum over all its copies of ``d_values``: (n_active, 729, 32)."""
    if d_tied is None:
        d_tied = torch.empty_like(d_values)
    _lib.check(_lib.load().nerfb200_baked_tie(C.byref(box), _ptr(brick_map), _ptr(bricks), d_values.shape[0],
                                              _ptr(d_values), _ptr(d_tied), _stream()), "baked_tie")
    return d_tied


def baked_max_weights(box: Grid, brick_map, values, use_viewdirs: bool, rays, max_w, dequant=None):
    """Max-accumulates into ``max_w`` fp32[n_active] each brick slot's largest rendering weight over the packed
    ``rays`` (``baked_render``'s weights at stop 0; a NaN weight as +inf).  Zero ``max_w`` once before the first
    chunk.  ``values`` fp32 or fp16, or uint8 codes with their ``dequant`` table."""
    sfx, pv = _baked_values(values, "baked_max_weights", dequant)
    _lib.check(getattr(_lib.load(), "nerfb200_baked_max_weights" + sfx)(
        C.byref(box), _ptr(brick_map), *pv, int(bool(use_viewdirs)), _ptr(rays), rays.shape[1], rays.shape[0],
        _ptr(max_w), _stream()), "baked_max_weights" + sfx)
    return max_w


def baked_lattice_count(box: Grid, brick_map, bricks, count=None):
    """int64[1] on the device: P, the lattice points with a copy in an active brick (include/nerfb200.h "baked fields:
    regularisers").  ``bricks`` is int32[n_active]."""
    if count is None:
        count = torch.empty(1, dtype=torch.int64, device=bricks.device)
    _lib.check(_lib.load().nerfb200_baked_lattice_count(C.byref(box), _ptr(brick_map), _ptr(bricks), bricks.shape[0],
                                                        _ptr(count), _stream()), "baked_lattice_count")
    return count


def baked_regularizer(box: Grid, brick_map, bricks, values, count, tv_sigma, tv_sh, sparsity, d=None, partials=None):
    """Adds the regularisers' gradient into ``d`` (the layout of ``values``; None: not formed) and writes their fp64
    per-slot value partials into ``partials`` (fp64[n_active]; None: not formed), P read from ``count``
    (``baked_lattice_count``) on the device."""
    if partials is not None and partials.dtype != torch.float64:
        raise RuntimeError("nerfb200: baked_regularizer partials must be fp64")
    pp = None if partials is None else _ptr(partials.view(torch.int64))  # _ptr takes no fp64; the bits are the same
    _lib.check(_lib.load().nerfb200_baked_regularizer(C.byref(box), _ptr(brick_map), _ptr(bricks), values.shape[0],
                                                      _ptr(values), _ptr(count), float(tv_sigma), float(tv_sh),
                                                      float(sparsity), _ptr(d), pp, _stream()), "baked_regularizer")
    return d, partials


def baked_adam_step_dev(values, g, m, v, step_dev, lr_sigma, lr_sh, lr_decay=None, lr_decay_factor=0.1, beta1=0.9,
                        beta2=0.999, eps=1e-8):
    """``adam_step_dev`` over baked values: sigma_raw at ``lr_sigma``, the SH coefficients at ``lr_sh``."""
    _, decay, factor = _schedule(0.0, lr_decay, lr_decay_factor)
    _lib.check(_lib.load().nerfb200_baked_adam_step_dev(_ptr(values), _ptr(g), _ptr(m), _ptr(v), values.shape[0],
                                                        _ptr(step_dev), float(lr_sigma), float(lr_sh), decay, factor,
                                                        float(beta1), float(beta2), float(eps), _stream()),
               "baked_adam_step_dev")


def baked_subdivide(box: Grid, brick_map, values, child_bricks, child_values):
    """Writes into ``child_values`` (n_child, 729, 32) fp32 the field on the box at twice ``box``'s resolution whose
    active bricks are ``child_bricks`` int32[n_child] (the children of the parent's active bricks, ascending), from the
    parent's fp32 ``values`` (include/nerfb200.h "baked fields: subdivision")."""
    _lib.check(_lib.load().nerfb200_baked_subdivide(C.byref(box), _ptr(brick_map), values.shape[0], _ptr(values),
                                                    _ptr(child_bricks), child_bricks.shape[0], _ptr(child_values),
                                                    _stream()), "baked_subdivide")
    return child_values


def baked_mesh_dirs(box: Grid, brick_map, values, level: float, edge_keys, want_normals: bool = False, dequant=None):
    """(dirs (V, 3), normals (V, 3) or None) of the vertices whose lattice edges are ``edge_keys`` int64 (V,) on a baked
    field's fp32 or fp16 ``values``, or uint8 codes with their ``dequant`` table (include/nerfb200.h "baked fields:
    meshes"): the view direction -n and the outward normal n (0 where the direction fell back)."""
    sfx, pv = _baked_values(values, "baked_mesh_dirs", dequant)
    n = edge_keys.shape[0]
    dirs = torch.empty(n, 3, dtype=torch.float32, device=edge_keys.device)
    normals = torch.empty(n, 3, dtype=torch.float32, device=edge_keys.device) if want_normals else None
    _lib.check(getattr(_lib.load(), "nerfb200_baked_mesh_dirs" + sfx)(
        C.byref(box), _ptr(brick_map), *pv, float(level), _ptr(edge_keys), n, _ptr(dirs), _ptr(normals), _stream()),
        "baked_mesh_dirs" + sfx)
    return dirs, normals


def baked_mesh_colors(box: Grid, brick_map, values, use_viewdirs: bool, level: float, edge_keys, dirs=None,
                      dequant=None):
    """colors (V, 3) of the vertices whose lattice edges are ``edge_keys`` int64 (V,) on a baked field's fp32 or fp16
    ``values``, or uint8 codes with their ``dequant`` table, seen along ``dirs`` (V, 3) with view directions
    (include/nerfb200.h "baked fields: meshes")."""
    sfx, pv = _baked_values(values, "baked_mesh_colors", dequant)
    n = edge_keys.shape[0]
    colors = torch.empty(n, 3, dtype=torch.float32, device=edge_keys.device)
    _lib.check(getattr(_lib.load(), "nerfb200_baked_mesh_colors" + sfx)(
        C.byref(box), _ptr(brick_map), *pv, int(bool(use_viewdirs)), float(level), _ptr(edge_keys), _ptr(dirs), n,
        _ptr(colors), _stream()), "baked_mesh_colors" + sfx)
    return colors
