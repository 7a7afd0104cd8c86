"""Dev tool: per-tensor error of the wgmma fused backward (and the CUDA-core one) against fp64 autograd of the oracle
MLP, on golden cases and on ragged synthetic sizes.    python tools/bwd_diag.py"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import Case  # noqa: E402
from test_stage_parity_gpu import _arch  # noqa: E402
from test_tc_gpu import oracle_mlp_grads  # noqa: E402
from nerf_pytorch_b200 import ops  # noqa: E402


def report(tag, arch, flat, want):
    worst = []
    for lname, w_off, b_off, fin, fout in arch.flat_layout():
        for off, cnt, what, shape in ((w_off, fin * fout, "weight", (fout, fin)), (b_off, fout, "bias", (fout,))):
            got = flat[off:off + cnt].view(shape).double().cpu()
            w = want[lname + "." + what].double().cpu()
            s = w.abs().max().item() + 1e-30
            d = (got - w).abs()
            e = d.max().item() / s
            worst.append((e, lname + "." + what))
            if e > 5e-5:
                idx = d.argmax().item()
                r, c = (idx // shape[1], idx % shape[1]) if len(shape) == 2 else (idx, 0)
                print(f"   {tag} {lname}.{what}: rel {e:.2e} at ({r},{c}) got {got.flatten()[idx]:.6g} want {w.flatten()[idx]:.6g}; "
                      f"rows>1e-4: {(d.reshape(shape[0], -1).max(1).values / s > 1e-4).nonzero().flatten().tolist()[:12]}")
    worst.sort(reverse=True)
    print(f" {tag}: worst {worst[0][0]:.2e} ({worst[0][1]}), median {worst[len(worst) // 2][0]:.2e}")


for case in ("lego_a0_train", "a1_skip_lindisp"):
    c = Case(case)
    arch = _arch(c)
    sd = c.sd_f
    blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, "cuda"))
    g = torch.Generator().manual_seed(7)
    for n, s in ((1, 16), (7, 50), (33, 17), (5, 37), (129, 100), (64, 192)):
        d = torch.randn(n, 3, generator=g)
        rays = torch.cat([torch.randn(n, 3, generator=g) * 0.1 + torch.tensor([0.0, -2.0, 3.0]), d,
                          torch.full((n, 1), 2.0), torch.full((n, 1), 6.0), d / d.norm(dim=-1, keepdim=True)], -1)
        z = torch.sort(torch.rand(n, s, generator=g) * 4 + 2, -1).values
        G = torch.randn(n, s, 4, generator=g)
        want = oracle_mlp_grads(c, sd, rays, z, G)
        rc, zc, Gc = rays.cuda().contiguous(), z.cuda().contiguous(), G.cuda().contiguous()
        print(case, n, s)
        for impl, tag in ((ops.IMPL_SIMT, "simt"), (ops.IMPL_TC, "tc  ")):
            _, st = ops.mlp_fwd(arch, blob, rc, zc, impl=impl, want_stash=True)
            for rep in range(2 if impl == ops.IMPL_TC else 1):
                fg, _ = ops.mlp_bwd(arch, blob, rc, zc, Gc, st, impl=impl)
                torch.cuda.synchronize()
                report(tag + str(rep), arch, fg, want)
