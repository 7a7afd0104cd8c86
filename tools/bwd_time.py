"""Dev tool: CUDA-event time of the fused wgmma backward alone (fine-pass size, A1)."""
import os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from nerf_pytorch_b200 import ops  # noqa: E402
arch = ops.ArchSpec(num_layers=8, hidden=128, skip_every=3, n_freq_xyz=10)
torch.manual_seed(0)
flat = (torch.rand(arch.flat_param_count(), device="cuda") - 0.5) * 0.2
blob = ops.pack_weights(arch, flat)
n, s = 4096, 192
d = torch.randn(n, 3, device="cuda")
rays = torch.cat([torch.randn(n, 3, device="cuda") * 0.1, d, torch.full((n, 1), 2.0, device="cuda"),
                  torch.full((n, 1), 6.0, device="cuda"), d / d.norm(dim=-1, keepdim=True)], -1).contiguous()
z = torch.sort(torch.rand(n, s, device="cuda") * 4 + 2, -1).values.contiguous()
raw, stash = ops.mlp_fwd(arch, blob, rays, z, impl=1, want_stash=True)
G = torch.randn_like(raw)
for _ in range(3):
    ops.mlp_bwd(arch, blob, rays, z, G, stash, impl=1)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
torch.cuda.synchronize(); e0.record()
for _ in range(10):
    ops.mlp_bwd(arch, blob, rays, z, G, stash, impl=1)
e1.record(); torch.cuda.synchronize()
print(f"mlp_bwd (fused wgmma, 4096 x 192 points, A1): {e0.elapsed_time(e1) / 10:.3f} ms")
