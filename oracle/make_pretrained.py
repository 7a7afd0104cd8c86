"""Write tests/golden/weights_<scene>_lowres.npz for the pretrained low-res scenes that make_golden.py does not write
(chair, drums, hotdog, materials, ship)  --  TEST INFRASTRUCTURE.

Needs a checkout of the unmodified krrish94/nerf-pytorch, named by the environment variable NERF_PYTORCH_REFERENCE:
``NERF_PYTORCH_REFERENCE=/path/to/nerf-pytorch python oracle/make_pretrained.py``.  Only the checkpoints' coarse and fine
state dicts are read (fp32, reference key names, "c." / "f." prefixed as make_golden.py writes lego and fern).  Every
network must be A0 by its tensors' shapes (4 layers, hidden 128, skip 4, 10 position bands, 4 direction bands, view
directions on), whatever its config.yml says; the script refuses anything else.
"""
from __future__ import annotations

import glob
import os

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("NERF_PYTORCH_REFERENCE", "")
GOLD = os.path.join(REPO, "tests", "golden")
SCENES = ["chair", "drums", "hotdog", "materials", "ship"]

# reference key -> shape of the A0 network with 10 position and 4 direction bands (63 and 27 encoding channels)
A0_SHAPES = {"layer1.weight": (128, 63), "layer1.bias": (128,),
             **{f"layers_xyz.{i}.{p}": s for i in range(3) for p, s in (("weight", (128, 128)), ("bias", (128,)))},
             "fc_feat.weight": (128, 128), "fc_feat.bias": (128,), "fc_alpha.weight": (1, 128), "fc_alpha.bias": (1,),
             "layers_dir.0.weight": (64, 128 + 27), "layers_dir.0.bias": (64,), "fc_rgb.weight": (3, 64),
             "fc_rgb.bias": (3,)}


def main():
    if not os.path.isdir(os.path.join(REF, "pretrained")):
        raise SystemExit("set NERF_PYTORCH_REFERENCE to a checkout of the unmodified krrish94/nerf-pytorch")
    for scene in SCENES:
        ckpt, = glob.glob(os.path.join(REF, "pretrained", f"{scene}-lowres", "checkpoint*.ckpt"))
        ck = torch.load(ckpt, map_location="cpu", weights_only=False)
        out = {}
        for tag, key in (("c", "model_coarse_state_dict"), ("f", "model_fine_state_dict")):
            sd = ck[key]
            shapes = {k: tuple(v.shape) for k, v in sd.items()}
            if shapes != A0_SHAPES:
                raise SystemExit(f"{scene} {key}: not A0 with 10 / 4 bands: {shapes}")
            out.update({f"{tag}.{k}": v.float().numpy() for k, v in sd.items()})
        path = os.path.join(GOLD, f"weights_{scene}_lowres.npz")
        np.savez(path, **out)
        print(f"[pretrained] {scene}: {os.path.basename(ckpt)} -> {os.path.relpath(path, REPO)}")


if __name__ == "__main__":
    main()
