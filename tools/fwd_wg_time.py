"""Dev tool: the hidden-128 wgmma forward with three consumer warpgroups (192-point CTA tiles, the default build) against
the same library built with two (128-point tiles, `make -C nerf_pytorch_b200/csrc wg2` -> libnerfb200_fwd_wg2.so).
Both files are loaded with ctypes in one process and alternated, CUDA events after warm-up:
  * ops.mlp_fwd at the fine-pass (4096 x 192) and coarse-pass (4096 x 64) sizes for A0 and A1: inference, stash-writing
    (the training forward) and the single-pass forward (impl 3);
  * one render_fwd(training=True) on 4096 rays (64 + 128 samples), A1.
Each figure is the median over ROUNDS rounds of ITERS calls with the range over the rounds; raw and the stash of the
builds are asserted byte-identical.  The card's name, power limit and SM clocks are printed beside the numbers.

    python tools/fwd_wg_time.py [--rounds 5] [--iters 30] [--extra NAME=PATH ...] [--json OUT]"""
import argparse
import ctypes
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from common import card, timed_mean  # noqa: E402
from nerf_pytorch_b200 import _lib, ops  # noqa: E402
from oracle import nerf_oracle as O  # noqa: E402

ARCHS = {"A0": dict(num_layers=4, hidden=128, skip_every=4), "A1": dict(num_layers=8, hidden=128, skip_every=3)}
WG2_PATH = os.path.join(os.path.dirname(_lib.LIB_PATH), "libnerfb200_fwd_wg2.so")


def open_build(path):
    """A second copy of the library, bound like _lib.load() binds the default one."""
    if not os.path.exists(path):
        raise SystemExit(f"{path} is missing (the two-warpgroup build: make -C nerf_pytorch_b200/csrc wg2)")
    lib = ctypes.CDLL(path)
    for name, (res, args) in _lib.SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    return lib


def compare(name, builds, fn, rounds, iters, warmup=3, reset=None):
    """fn() runs under each build in turn (ops looks the library up on every call); its tensors must be the same bytes.
    reset() clears caller-owned outputs before a build's first call, so that bytes nobody writes compare equal."""
    outs = {}
    for k, lib in builds.items():
        _lib._lib = lib
        if reset:
            reset()
        for _ in range(warmup):
            r = fn()
        torch.cuda.synchronize()
        outs[k] = [t.clone() for t in r]
    first = next(iter(outs))
    for k, ts in outs.items():
        for a, b in zip(outs[first], ts):
            assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), f"{name}: {k} differs from {first}"
    del outs, r
    torch.cuda.empty_cache()
    ms = {k: [] for k in builds}
    for _ in range(rounds):
        for k, lib in builds.items():
            _lib._lib = lib
            ms[k].append(timed_mean(fn, iters))
    res = {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)} for k, v in ms.items()}
    print(f"{name:42s} " + "   ".join(f"{k} {r['median_ms']:7.3f} ms ({r['min_ms']:.3f} - {r['max_ms']:.3f})"
                                      for k, r in res.items()), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--extra", action="append", default=[], help="NAME=PATH of a further build to time alongside")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fwd_wg_time.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda")
    builds = {"wg3": _lib.load(), "wg2": open_build(WG2_PATH)}
    for e in args.extra:
        k, path = e.split("=", 1)
        builds[k] = open_build(path)
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
    opts = ops.make_opts(nc, nf, False, False, False, 0.0)
    for a, kw in ARCHS.items():
        arch = ops.ArchSpec(n_freq_xyz=10, n_freq_dir=4, **kw)
        sd = O.init_flexible_nerf(arch.num_layers, arch.hidden, arch.skip_every, 10, 4,
                                  generator=torch.Generator().manual_seed(1))
        blob = ops.pack_weights(arch, ops.flatten_state_dict(arch, sd, dev))
        for pname, z in zs.items():
            what = f"{a} {pname}-pass mlp_fwd {tuple(z.shape)}"
            out[what + " inference"] = compare(what + " inference", builds,
                                               lambda: (ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC),),
                                               args.rounds, args.iters)
            raw = torch.empty(*z.shape, 4, device=dev)
            stash = torch.empty(ops.stash_floats(arch, z.numel()), device=dev)

            def train():  # ops.mlp_fwd(want_stash=True) into a stash this tool owns
                _lib.check(_lib.load().nerfb200_mlp_fwd(ctypes.byref(arch.c_struct()), ops._ptr(blob), ops._ptr(rays),
                                                        rays.shape[1], ops._ptr(z), z.shape[0], z.shape[1],
                                                        ops._ptr(raw), ops._ptr(stash), ops.IMPL_TC, ops._stream()),
                           "mlp_fwd")
                return raw, stash

            out[what + " training"] = compare(what + " training", builds, train, args.rounds, args.iters,
                                              reset=lambda: (raw.zero_(), stash.zero_()))
            del raw, stash
            out[what + " impl 3"] = compare(what + " impl 3", builds,
                                            lambda: (ops.mlp_fwd(arch, blob, rays, z, impl=ops.IMPL_TC_FAST),),
                                            args.rounds, args.iters)
        if a == "A1":
            ws = [None]

            def render():
                oc, of, ws[0] = ops.render_fwd(arch, arch, opts, blob, blob, rays, {}, training=True, impl=ops.IMPL_TC,
                                               workspace=ws[0])
                return oc, of

            out["A1 render_fwd training"] = compare("A1 render_fwd(training=True) 4096 x (64 + 128)", builds, render,
                                                    args.rounds, args.iters)
    _lib._lib = builds["wg3"]
    print("card:", card())
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
