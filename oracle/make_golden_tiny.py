"""Generate tests/golden/tiny_nerf.npz from the UNMODIFIED reference's tiny_nerf.py  --  TEST INFRASTRUCTURE.

BASELINE.json configs[0] ("tiny_nerf.py lego 100x100, 1024 rays, 64 coarse samples, CPU-only"): one forward + backward of
`run_one_iter_of_tinynerf` (tiny_nerf.py:109-155) on a 32 x 32 image (= 1024 rays) with 64 samples per ray, L = 10,
pose_spherical(30, -30, 4), seeded `VeryTinyNerfModel`; then the same through oracle/tiny_oracle.py, from the same seed and
with the recorded random tensor injected, ASSERTING bit equality of the image, the loss and every gradient.
Needs NERF_PYTORCH_REFERENCE like oracle/make_golden.py: ``NERF_PYTORCH_REFERENCE=... python oracle/make_golden_tiny.py``."""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from oracle import nerf_oracle as O  # noqa: E402
from oracle import tiny_oracle as T  # noqa: E402
from oracle.make_golden import GOLD, REF, RecordRNG, grad_digest, import_reference  # noqa: E402


def import_tiny():
    nerf = import_reference()
    for name in ("matplotlib", "matplotlib.pyplot"):     # tiny_nerf.py:4 imports pyplot for its progress plots only
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.path.insert(0, REF)
    import tiny_nerf  # noqa

    return nerf, tiny_nerf


def main():
    torch.set_num_threads(1)
    nerf, tiny = import_tiny()
    H = W = 32
    focal, near, far, S, L, chunk = 44.0, 2.0, 6.0, 64, 10, 16384
    pose = O.pose_spherical(30.0, -30.0, 4.0)
    g = torch.Generator().manual_seed(7)
    sd = T.init_very_tiny_nerf(128, L, generator=g)
    target = torch.rand(H, W, 3, generator=g)

    model = tiny.VeryTinyNerfModel(num_encoding_functions=L)
    model.load_state_dict(sd)
    torch.manual_seed(11)
    with RecordRNG() as rec:
        ref = tiny.run_one_iter_of_tinynerf(H, W, focal, pose, near, far, S, nerf.positional_encoding, nerf.get_minibatches,
                                            chunk, model, L)
    loss_ref = torch.nn.functional.mse_loss(ref, target)
    loss_ref.backward()
    assert len(rec.rand) == 1 and not rec.randn
    rand = rec.rand[0]

    def oracle(rand_in, seed):
        leaves = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
        if seed is not None:
            torch.manual_seed(seed)
        out = T.run_one_iter_of_tinynerf(H, W, focal, pose, near, far, S, L, chunk, leaves, rand=rand_in)
        loss = torch.nn.functional.mse_loss(out, target)
        loss.backward()
        return out, loss, leaves

    for tag, (out, loss, leaves) in (("same seed", oracle(None, 11)), ("injected randoms", oracle(rand, None))):
        assert torch.equal(out, ref), (tag, (out - ref).abs().max())
        assert torch.equal(loss, loss_ref), tag
        for k, p in model.named_parameters():
            assert torch.equal(leaves[k].grad, p.grad), (tag, k)
    print(f"tiny_nerf: reference == oracle bit for bit (image, loss {loss_ref.item():.6f}, {len(sd)} gradients), both RNG modes")

    arrs = {"H": H, "W": W, "focal": focal, "near": near, "far": far, "S": S, "L": L, "chunk": chunk, "pose": pose.numpy(),
            "target": target.numpy(), "rand": rand.numpy(), "rgb": ref.detach().numpy(), "loss": loss_ref.item()}
    for k, v in sd.items():
        arrs["w." + k] = v.numpy()
    for k, p in model.named_parameters():
        arrs["g." + k] = grad_digest(p.grad)
    os.makedirs(GOLD, exist_ok=True)
    np.savez_compressed(os.path.join(GOLD, "tiny_nerf.npz"), **arrs)
    print("wrote", os.path.join(GOLD, "tiny_nerf.npz"))


if __name__ == "__main__":
    main()
