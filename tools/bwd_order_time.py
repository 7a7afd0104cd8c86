"""Dev tool: the fused wgmma backward of this build against another build of the library (for instance the parent
commit's, `make -C nerf_pytorch_b200/csrc` in a checkout of it), both loaded with ctypes in one process and alternated,
CUDA events after warm-up:
  * ops.mlp_bwd (impl 1) at the fine-pass (4096 x 192) and coarse-pass (4096 x 64) sizes for A1 and the fine-pass size
    for A0, on the stash of a training forward and a random d_raw;
  * one render_bwd at training size: 4096 rays, 64 + 128 samples, A1, on a render_fwd(training=True) workspace.
Each figure is the median over ROUNDS rounds of ITERS calls with the range over the rounds; the gradients of the two
builds are asserted byte-identical.  The card's name, power limit and SM clocks are printed beside the numbers.

    python tools/bwd_order_time.py --other PATH/libnerfb200.so [--rounds 5] [--iters 20] [--json OUT]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from common import card  # noqa: E402
from fwd_wg_time import compare, open_build  # noqa: E402
from nerf_pytorch_b200 import _lib, ops  # noqa: E402
from oracle import nerf_oracle as O  # noqa: E402

ARCHS = {"A0": dict(num_layers=4, hidden=128, skip_every=4), "A1": dict(num_layers=8, hidden=128, skip_every=3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", required=True, help="path of the library to time this build against")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bwd_order_time.py measures on the GPU; no CUDA device found")
    if not os.path.exists(args.other):
        raise SystemExit(f"{args.other} is missing")
    dev = torch.device("cuda")
    builds = {"this": _lib.load(), "other": open_build(args.other)}
    out = {"card (name, power limit, SM clock, max SM clock)": card(), "rounds": args.rounds, "iters": args.iters}
    print("card:", out["card (name, power limit, SM clock, max SM clock)"])
    n_rays, nc, nf = 4096, 64, 128
    g = torch.Generator().manual_seed(0)
    o = torch.nn.functional.normalize(torch.randn(n_rays, 3, generator=g), dim=-1) * 4.0
    d = -o / 4.0 + 0.25 * torch.randn(n_rays, 3, generator=g)
    rays = torch.cat([o, d, torch.full((n_rays, 1), 2.0), torch.full((n_rays, 1), 6.0),
                      d / d.norm(dim=-1, keepdim=True)], -1).to(dev).contiguous()
    zs = {"fine": torch.sort(torch.rand(n_rays, nc + nf, generator=g) * 4 + 2, -1).values.to(dev).contiguous(),
          "coarse": torch.sort(torch.rand(n_rays, nc, generator=g) * 4 + 2, -1).values.to(dev).contiguous()}
    for a, passes in (("A1", ("fine", "coarse")), ("A0", ("fine",))):
        arch = ops.ArchSpec(n_freq_xyz=10, n_freq_dir=4, **ARCHS[a])
        sd = O.init_flexible_nerf(arch.num_layers, arch.hidden, arch.skip_every, 10, 4,
                                  generator=torch.Generator().manual_seed(1))
        blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, dev))
        for pname in passes:
            z = zs[pname]
            _, stash = ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC, want_stash=True)
            d_raw = torch.randn(*z.shape, 4, generator=g).to(dev)
            what = f"{a} {pname}-pass mlp_bwd {tuple(z.shape)}"
            out[what] = compare(what, builds,
                                lambda: (ops.mlp_bwd(arch, blob, rays, z, d_raw, stash, impl=ops.IMPL_TC)[0],),
                                args.rounds, args.iters)
            del stash
        if a == "A1":
            opts = ops.make_opts(nc, nf, False, False, False, 0.0)
            _, _, ws = ops.render_fwd(arch, arch, opts, blob, blob, rays, {}, training=True, impl=ops.IMPL_TC)
            g_c = torch.randn(n_rays, 8, generator=g).to(dev)
            g_f = torch.randn(n_rays, 8, generator=g).to(dev)
            fg_c = torch.zeros(arch.flat_param_count(), device=dev)
            fg_f = torch.zeros_like(fg_c)

            def render_bwd():  # render_bwd adds into the flat gradients: zeroed before every call
                fg_c.zero_()
                fg_f.zero_()
                ops.render_bwd(arch, arch, opts, blob, blob, rays, {}, g_c, g_f, ws, fg_c, fg_f, impl=ops.IMPL_TC)
                return fg_c, fg_f

            out["A1 render_bwd"] = compare("A1 render_bwd 4096 x (64 + 128)", builds, render_bwd, args.rounds,
                                           args.iters)
            del ws
    _lib._lib = builds["this"]
    print("card:", card())
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
