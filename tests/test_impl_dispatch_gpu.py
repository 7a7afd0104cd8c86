"""GPU: impl codes the library does not run, and networks it refuses, stop a call before its first launch.  Every call
gets real device tensors, so a refusal that regressed would run on valid memory and fail an assertion here."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

N_RAYS, N_SAMPLES = 16, 32


def _blob(arch, seed):
    from nerf_pytorch_b200 import ops

    g = torch.Generator().manual_seed(seed)
    return ops.pack_weights(arch, ((torch.rand(arch.flat_param_count(), generator=g) - 0.5) * 0.2).cuda())


def _rays(n, seed):
    """Origins on a sphere of radius 4 looking at the centre, near 2, far 6, with view directions."""
    g = torch.Generator().manual_seed(seed)
    o = torch.nn.functional.normalize(torch.randn(n, 3, generator=g), dim=-1) * 4.0
    d = -o / 4.0 + 0.25 * torch.randn(n, 3, generator=g)
    rays = torch.cat([o, d, torch.full((n, 1), 2.0), torch.full((n, 1), 6.0), d / d.norm(dim=-1, keepdim=True)], -1)
    return rays.cuda().contiguous()


def _render_fwd(arch_c, arch_f, opts, blob_c, blob_f, rays, out_c, out_f, workspace, training, impl):
    """nerfb200_render_fwd into the caller's outputs (ops.render_fwd allocates its own)."""
    from nerf_pytorch_b200 import _lib, ops

    return _lib.load().nerfb200_render_fwd(
        C.byref(arch_c.c_struct()), C.byref(arch_f.c_struct()), C.byref(opts), ops._ptr(blob_c), ops._ptr(blob_f),
        ops._ptr(rays), rays.shape[1], rays.shape[0], None, None, None, None, None, ops._ptr(out_c), ops._ptr(out_f),
        ops._ptr(workspace), int(training), impl, ops._stream())


@pytest.mark.parametrize("impl", [2, 4, -1])
def test_unknown_impl_is_refused_by_every_entry_point_before_any_launch(impl):
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    arch = ops.ArchSpec(num_layers=4, hidden=128, n_freq_xyz=10)
    blob = _blob(arch, 1)
    rays = _rays(N_RAYS, 2)
    z = torch.sort(torch.rand(N_RAYS, N_SAMPLES, generator=torch.Generator().manual_seed(3)) * 4 + 2, -1).values.cuda()
    raw, stash = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_SIMT, want_stash=True)
    d_raw = torch.ones(N_RAYS, N_SAMPLES, 4, device="cuda")
    gstash = torch.empty_like(stash)
    flat_grad = torch.zeros(arch.flat_param_count(), device="cuda")
    opts = ops.make_opts(16, 16, False, False, False, 0.0)
    _, _, ws = ops.render_fwd(arch, arch, opts, blob, blob, rays, {}, training=True, impl=ops.IMPL_SIMT)
    g = torch.zeros(N_RAYS, 8, device="cuda")
    torch.cuda.synchronize()
    before = ops.launch_count()

    for want_stash in (False, True):
        with pytest.raises(RuntimeError, match=f"mlp_fwd: unknown impl {impl}"):
            ops.mlp_fwd(arch, blob, rays, z, impl=impl, want_stash=want_stash)
    # ops.mlp_bwd stops at the scratch query (test_impl_dispatch_host_cpu.py), so the entry point is called directly
    rc = lib.nerfb200_mlp_bwd(C.byref(arch.c_struct()), ops._ptr(blob), ops._ptr(rays), rays.shape[1], ops._ptr(z),
                              N_RAYS, N_SAMPLES, ops._ptr(d_raw), ops._ptr(stash), ops._ptr(gstash),
                              ops._ptr(flat_grad), impl, ops._stream())
    assert rc == _lib.ERR_INVALID and f"mlp_bwd: unknown impl {impl}" in lib.nerfb200_last_error().decode()
    with pytest.raises(RuntimeError, match=f"mlp_dgrad: unknown impl {impl}"):
        ops.mlp_dgrad(arch, blob, d_raw, stash, impl=impl, gstash=gstash)
    with pytest.raises(RuntimeError, match=f"mlp_wgrad: unknown impl {impl}"):
        ops.mlp_wgrad(arch, rays, z, d_raw, stash, gstash, impl=impl, flat_grad=flat_grad)
    for training in (False, True):
        with pytest.raises(RuntimeError, match=f"render_fwd: unknown impl {impl}"):
            ops.render_fwd(arch, arch, opts, blob, blob, rays, {}, training=training, impl=impl)
    with pytest.raises(RuntimeError, match=f"render_bwd: unknown impl {impl}"):
        ops.render_bwd(arch, arch, opts, blob, blob, rays, {}, g, g, ws, flat_grad, flat_grad.clone(), impl=impl)
    assert ops.launch_count() == before
    torch.cuda.synchronize()
    assert not flat_grad.any()


def test_render_fwd_checks_the_fine_network_before_the_coarse_pass():
    """impl 1 with a coarse network it takes and a fine one whose xyz encoding is 72 wide (L_xyz 11 without input,
    more than 64): the call is refused with nothing launched and out_coarse as it was.  The same call with the coarse
    network in both places renders."""
    from nerf_pytorch_b200 import _lib, ops

    lib = _lib.load()
    coarse = ops.ArchSpec(num_layers=4, hidden=128, n_freq_xyz=10)
    wide = ops.ArchSpec(num_layers=4, hidden=128, n_freq_xyz=11, include_input_xyz=False)
    assert ops.impl_supported(coarse, 16, ops.IMPL_TC_FWD) and not ops.impl_supported(wide, 32, ops.IMPL_TC_FWD)
    blob_c, blob_w = _blob(coarse, 4), _blob(wide, 5)
    rays = _rays(N_RAYS, 6)
    opts = ops.make_opts(16, 16, False, False, False, 0.0)
    ws = torch.empty(max(ops.render_workspace_bytes(coarse, f, opts, N_RAYS, False) for f in (coarse, wide)),
                     dtype=torch.uint8, device="cuda")
    out_c = torch.full((N_RAYS, 8), 12345.0, device="cuda")
    out_f = torch.full((N_RAYS, 8), 12345.0, device="cuda")
    torch.cuda.synchronize()
    before = ops.launch_count()
    rc = _render_fwd(coarse, wide, opts, blob_c, blob_w, rays, out_c, out_f, ws, False, ops.IMPL_TC)
    assert rc == _lib.ERR_UNSUPPORTED
    assert "wider than 64" in lib.nerfb200_last_error().decode()
    assert ops.launch_count() == before
    torch.cuda.synchronize()
    assert (out_c == 12345.0).all() and (out_f == 12345.0).all()

    assert _render_fwd(coarse, coarse, opts, blob_c, blob_c, rays, out_c, out_f, ws, False, ops.IMPL_TC) == _lib.OK
    torch.cuda.synchronize()
    assert ops.launch_count() > before and (out_c != 12345.0).all() and (out_f != 12345.0).all()


def test_render_bwd_checks_the_coarse_network_before_the_fine_part():
    """A coarse network with 30 direction channels (L_dir 5 without input) trains through the wgmma forward (at most
    32) but not the fused backward (at most 28): render_bwd(parts = 3), whose fine part runs first, is refused with
    nothing launched and flat_grad_f as it was.  The fine part alone (parts = 1) runs."""
    from nerf_pytorch_b200 import ops

    coarse = ops.ArchSpec(num_layers=8, hidden=128, n_freq_xyz=10, n_freq_dir=5, include_input_dir=False)
    fine = ops.ArchSpec(num_layers=4, hidden=128, n_freq_xyz=10)
    assert coarse.dim_dir == 30 and ops.impl_supported(fine, 32, ops.IMPL_TC)
    blob_c, blob_f = _blob(coarse, 7), _blob(fine, 8)
    rays = _rays(N_RAYS, 9)
    opts = ops.make_opts(16, 16, False, False, False, 0.0)
    _, _, ws = ops.render_fwd(coarse, fine, opts, blob_c, blob_f, rays, {}, training=True, impl=ops.IMPL_TC)
    g = torch.ones(N_RAYS, 8, device="cuda")
    flat_grad_c = torch.full((coarse.flat_param_count(),), 12345.0, device="cuda")
    flat_grad_f = torch.full((fine.flat_param_count(),), 12345.0, device="cuda")
    torch.cuda.synchronize()
    before = ops.launch_count()
    with pytest.raises(NotImplementedError, match="render_bwd impl=1 \\(wgmma\\): direction encodings wider than 28"):
        ops.render_bwd(coarse, fine, opts, blob_c, blob_f, rays, {}, g, g, ws, flat_grad_c, flat_grad_f,
                       impl=ops.IMPL_TC)
    assert ops.launch_count() == before
    torch.cuda.synchronize()
    assert (flat_grad_c == 12345.0).all() and (flat_grad_f == 12345.0).all()

    flat_grad_f.zero_()
    ops.render_bwd(coarse, fine, opts, blob_c, blob_f, rays, {}, g, g, ws, flat_grad_c, flat_grad_f, impl=ops.IMPL_TC,
                   parts=1)
    torch.cuda.synchronize()
    assert ops.launch_count() > before and flat_grad_f.any() and (flat_grad_c == 12345.0).all()
