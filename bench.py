#!/usr/bin/env python
"""bench.py -- rays/s of the NeRF per-ray hot path on synthetic lego-shaped input.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--arch A1|A0|A2] [--config 2|3|4]
                    [--dump-outputs DIR]

Workload (BASELINE.json configs[1]; SURVEY.md section 8d): config/lego.yml as written -- 8x128
FlexibleNeRFModel with skip every 3 (coarse + fine), L_xyz 10, L_dir 4 -- 400x400 lego-like camera
(pose_spherical(30,-30,4), focal 555.5555), 4096 random rays per GPU, 64 coarse + 128 fine samples,
near 2 / far 6, perturb on, noise std 0.2, default-init weights under seed 0, random targets.

A "step" is one pass of the hot path over one batch: run_one_iter_of_nerf (forward), the coarse+fine
MSE loss, backward, the single gradient all-reduce (N > 1) and the fused Adam update.  `value` is
whole-job rays/s with the batch already resident in HBM; `e2e` is the same step driven from pinned
HOST buffers (H2D of origins/directions/targets and D2H of the loss inside the timed region).
`fwd_only` (extra key) is the inference path (torch.no_grad) on the same batch.

--config selects the BASELINE.json workload: 2 (default) = lego 400x400, 4096 rays; 3 = lego 800x800, 8192 rays;
4 = LLFF-like fern (378x504, NDC rays, L_xyz 6, noise std 1.0), 4096 rays.  (Config 5 = config 3's shape at --gpus 8.)

--dump-outputs DIR writes what the last timed training step computed, as float32 .npy files: the six render outputs
of run_one_iter_of_nerf, the loss, and per network the flat gradient and the parameters after the Adam update.  All
inputs are seeded, so two builds run with the same arguments can be compared output for output.

--impl reference times the reference's CPU implementation of the same step (the oracle port: the same
ATen ops in the same order as the unmodified reference, all host threads) on the SAME batch size (falls back to a
stated fraction of it only when a step would take longer than 20 s).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

ARCHS = {
    "A0": dict(num_layers=4, hidden_size=128, skip_connect_every=4),   # what the reference CLI actually builds
    "A1": dict(num_layers=8, hidden_size=128, skip_connect_every=3),   # config/lego.yml as written
    "A2": dict(num_layers=8, hidden_size=256, skip_connect_every=4),   # pretrained/*/config.yml as written
}
MACS_PER_POINT = {"A0": 83840, "A1": 165504, "A2": 593408}  # SURVEY.md section 8(d), weights only
NC, NF = 64, 128
# BASELINE.json configs[1..3] (SURVEY.md section 8d): name, H, W, focal, rays per GPU, near, far, ndc, noise std, L_xyz
CONFIGS = {
    2: dict(name="config/lego.yml 400x400", H=400, W=400, focal=555.5555155968841, rays=4096, near=2.0, far=6.0, ndc=False,
            noise=0.2, L_xyz=10),
    3: dict(name="config/lego.yml 800x800 full-res", H=800, W=800, focal=1111.1110311937682, rays=8192, near=2.0, far=6.0,
            ndc=False, noise=0.2, L_xyz=10),
    4: dict(name="config/llff.yml fern-like (NDC rays)", H=378, W=504, focal=407.5658, rays=4096, near=0.0, far=1.0, ndc=True,
            noise=1.0, L_xyz=6),
}
CFG = CONFIGS[2]          # set in main()
RAYS_PER_GPU = 4096       # set in main()


def camera_pose(ndc):
    """Blender-like: pose_spherical(theta 30, phi -30, radius 4) (nerf/load_blender.py:32-37 composes
    translate_z(r), rot_phi, rot_theta and an axis swap); LLFF-like: a forward-facing camera at the origin."""
    import math

    if ndc:
        return torch.eye(4)
    th, ph, r = math.radians(30.0), math.radians(-30.0), 4.0
    t = torch.tensor([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, r], [0, 0, 0, 1.0]])
    rp = torch.tensor([[1, 0, 0, 0], [0, math.cos(ph), -math.sin(ph), 0], [0, math.sin(ph), math.cos(ph), 0], [0, 0, 0, 1.0]])
    rt = torch.tensor([[math.cos(th), 0, -math.sin(th), 0], [0, 1, 0, 0], [math.sin(th), 0, math.cos(th), 0], [0, 0, 0, 1.0]])
    swap = torch.tensor([[-1, 0, 0, 0], [0, 0, 1, 0], [0, 1, 0, 0], [0, 0, 0, 1.0]])
    return swap @ rt @ rp @ t


def synthetic_batch(n, seed):
    """Pixel ids (randperm pick over the image, train_nerf.py:213-226) and random targets, on the host."""
    g = torch.Generator().manual_seed(seed)
    pix = torch.randperm(CFG["H"] * CFG["W"], generator=g)[:n].contiguous()
    tgt = torch.rand(n, 3, generator=g)
    return pix, tgt


def make_options():
    """The option tree run_one_iter_of_nerf reads (config/lego.yml:34-38,136-147 / fern.yml), as plain namespaces."""
    from types import SimpleNamespace as NS

    o = NS(num_coarse=NC, num_fine=NF, perturb=True, lindisp=False, white_background=False,
           radiance_field_noise_std=CFG["noise"], chunksize=131072, num_random_rays=RAYS_PER_GPU)
    return NS(nerf=NS(use_viewdirs=True, train=o, validation=o),
              dataset=NS(no_ndc=not CFG["ndc"], near=CFG["near"], far=CFG["far"]))


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        self.idx, self.rows, self.proc = gpu_index, [], None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "100", "-i", str(self.idx)], stdout=subprocess.PIPE, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons, power = [], [], set(), []
        for r in self.rows:
            try:
                sm.append(float(r[1])); mx.append(float(r[2])); power.append(float(r[3]))
            except Exception:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "power_w_max": max(power) if power else None, "samples": len(sm), "reasons": sorted(reasons)}


def measured_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d, "measured bf16 cuBLAS burst (MEASURED_PEAKS.json)"
    # NVIDIA's H100 SXM data sheet (700 W card): HBM3 bandwidth and dense BF16 / FP16 tensor rate
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}, "H100 SXM data sheet, dense BF16/FP16 (not measured)"


# ------------------------------------------------------------------------------------------------
# reference arm / CPU baseline: the oracle port timed on the host cores
# ------------------------------------------------------------------------------------------------
def best_cpu_threads(arch):
    """The reference is timed with the thread count that serves IT best: torch's intra-op pool does not scale
    to 100+ threads on these small ops (measured: 128 threads are ~20x slower than 16), so probe a few."""
    cores = os.cpu_count() or 1
    cands = sorted({c for c in (8, 16, 32, 64, cores) if c <= cores})
    best, best_t = cands[0], float("inf")
    for c in cands:
        t = cpu_train_steps(arch, 128, steps=1, warmup=1, threads=c)[0]
        if t < best_t:
            best, best_t = c, t
        if t > 3 * best_t:
            break
    return best


def cpu_train_steps(arch, n_rays, steps, warmup, threads=None, device="cpu"):
    """fwd + loss + backward + Adam of the reference algorithm (oracle/nerf_oracle.py: the reference's ATen ops in the
    reference's order) on the host cores -- or, device="cuda", as eager PyTorch on the GPU, the "same code,
    device=cuda" yardstick of SURVEY.md section 8(d).  Returns s/step list."""
    from oracle import nerf_oracle as O

    if threads:
        torch.set_num_threads(threads)
    kw = ARCHS[arch]
    gen = torch.Generator().manual_seed(0)
    mk = lambda: {k: v.to(device).requires_grad_(True) for k, v in O.init_flexible_nerf(
        kw["num_layers"], kw["hidden_size"], kw["skip_connect_every"], CFG["L_xyz"], 4, generator=gen).items()}
    sd_c, sd_f = mk(), mk()
    opt = torch.optim.Adam(list(sd_c.values()) + list(sd_f.values()), lr=5e-3)
    pix, tgt = synthetic_batch(n_rays, seed=0)
    ro, rd = O.get_ray_bundle(CFG["H"], CFG["W"], CFG["focal"], camera_pose(CFG["ndc"]))
    ro, rd = ro.reshape(-1, 3)[pix].contiguous().to(device), rd.reshape(-1, 3)[pix].contiguous().to(device)
    tgt = tgt.to(device)
    options = O.make_options(num_coarse=NC, num_fine=NF, perturb=True, radiance_field_noise_std=CFG["noise"],
                             near=CFG["near"], far=CFG["far"], no_ndc=not CFG["ndc"], chunksize=131072)
    times = []
    import contextlib
    # the port creates its helper tensors (t_vals, noise, frequency bands) with device-less factory calls like the
    # reference does; on the GPU they follow torch's default-device context, as under the reference's own `.to(device)` flow
    ctx = (lambda: torch.device(device)) if device != "cpu" else contextlib.nullcontext
    for i in range(warmup + steps):
        if device != "cpu":
            torch.cuda.synchronize()
        t0 = time.perf_counter()
        with ctx():
            out = O.run_one_iter_of_nerf(CFG["H"], CFG["W"], CFG["focal"], sd_c, sd_f, ro, rd, options,
                                         enc_xyz=(CFG["L_xyz"], True, True), enc_dir=(4, True, True))
        loss = O.nerf_loss(out, tgt)
        opt.zero_grad()
        loss.backward()
        opt.step()
        if device != "cpu":
            torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if i >= warmup:
            times.append(dt)
    return times


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return  # rank 0 alone runs the CPU arm
    threads = best_cpu_threads(args.arch)
    n_sample = RAYS_PER_GPU
    probe = cpu_train_steps(args.arch, 512, steps=1, warmup=1, threads=threads)[0]
    if probe * (RAYS_PER_GPU / 512) > 20.0:      # a step of the full batch would exceed 20 s: bounded sample instead
        n_sample = max(512, int(RAYS_PER_GPU * 20.0 / (probe * (RAYS_PER_GPU / 512))) // 256 * 256)
    times = cpu_train_steps(args.arch, n_sample, args.steps, args.warmup, threads=threads)
    ms = 1e3 * sum(times) / len(times)
    value = n_sample / (ms / 1e3)
    sample = (f"{n_sample} of the {RAYS_PER_GPU} rays per step (same sampler/model/loss/Adam), {args.steps} steps; "
              f"thread count = best of a probe over 8..{os.cpu_count()} host threads")
    line = {
        "impl": "reference", "metric": "rays/sec (4096 rays, 64c+128f samples), train step", "value": value,
        "unit": "rays/s", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": dict(workload_config(args, 1), reference_rays_per_step=n_sample),
        "cpu_baseline": {"value": value, "unit": "rays/s", "cores": torch.get_num_threads(), "kind": "port",
                         "sample": sample},
        "e2e": {"value": value, "unit": "rays/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line))


def workload_config(args, world):
    kw = ARCHS[args.arch]
    return {
        "workload": f"{CFG['name']}, {RAYS_PER_GPU} rays/GPU x {world} GPU, {NC}c+{NF}f hierarchical, "
                    f"FlexibleNeRFModel {kw['num_layers']}x{kw['hidden_size']} skip {kw['skip_connect_every']} ({args.arch}), "
                    "train step = fwd + mse(coarse)+mse(fine) + bwd + grad all-reduce + Adam",
        "rays_per_gpu": RAYS_PER_GPU, "global_rays": RAYS_PER_GPU * world, "n_coarse": NC, "n_fine": NF,
        "parallelism": f"ray-sharded dp{world}, one flat-gradient all-reduce per step",
        "cache": "no L2 flush: every step streams its activation stash (GBs, >> 50 MB L2) through HBM; "
                 "weights/rays are L2-resident as in real training",
    }


# ------------------------------------------------------------------------------------------------
# our arm
# ------------------------------------------------------------------------------------------------
def run_ours(args):
    import torch.distributed as dist

    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops, parallel, train_utils

    rank, local, world = parallel.init_distributed()
    if not torch.cuda.is_available():
        raise RuntimeError("bench.py (impl ours) needs a GPU: the product path has no CPU fallback")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    impl = {"simt": ops.IMPL_SIMT, "tc": ops.IMPL_TC}[args.kernels]
    if args.arch == "A2":
        # hidden 256: training on the fp32 CUDA-core kernels, inference (`fwd_only`) on the wgmma forward -- the library's
        # automatic choice; the per-kernel roofline below probes the fp32 kernels
        impl, args.kernels = ops.IMPL_SIMT, "simt (training), tc (inference forward)"
        nb.set_default_impl(None)
    else:
        nb.set_default_impl(impl)
    parallel.enable_gradient_sync()

    kw = ARCHS[args.arch]
    Lx = CFG["L_xyz"]
    H, W, FOCAL = CFG["H"], CFG["W"], CFG["focal"]
    torch.manual_seed(0)
    mk = lambda: nb.FlexibleNeRFModel(num_encoding_fn_xyz=Lx, num_encoding_fn_dir=4, **kw).to(dev)
    mc, mf = mk(), mk()   # same seed on every rank -> identical replicas
    epf, edf = nb.get_embedding_function(Lx, True, True), nb.get_embedding_function(4, True, True)
    arch = train_utils._arch_of(mc, (Lx, True, True), (4, True, True))
    optim = parallel.FusedAdam([(mc, arch), (mf, arch)], lr=5e-3, lr_decay=250, lr_decay_factor=0.1)
    options = make_options()
    pose = camera_pose(CFG["ndc"])

    # this rank's shard of the global batch (weak scaling: RAYS_PER_GPU rays per GPU): pixel ids + targets
    pix_h, tgt_h = synthetic_batch(RAYS_PER_GPU * world, seed=0)
    lo, hi = parallel.shard_bounds(RAYS_PER_GPU * world, rank, world)
    pix_h, tgt_h = pix_h[lo:hi].contiguous().pin_memory(), tgt_h[lo:hi].contiguous().pin_memory()
    tgt = tgt_h.to(dev)
    # HBM-resident variant: origins / directions of the batch as the reference API takes them
    rays6 = ops.gen_rays(pose, H, W, FOCAL, pix_h.to(dev), dev, use_viewdirs=False, stride=6)
    ro, rd = rays6[:, :3].contiguous(), rays6[:, 3:].contiguous()
    torch.manual_seed(1234 + rank)  # per-rank sampling noise
    losses = []

    def finish(out, tgt_):
        loss = torch.nn.functional.mse_loss(out[0], tgt_) + torch.nn.functional.mse_loss(out[3], tgt_)
        optim.zero_grad()
        loss.backward()       # grads of both nets land in one flat buffer; one all-reduce (two overlapped halves) when world > 1
        optim.step()          # fused Adam over the flat parameter buffers
        return loss

    last = {}

    def step(ro_, rd_, tgt_):
        out = nb.run_one_iter_of_nerf(H, W, FOCAL, mc, mf, ro_, rd_, options, mode="train",
                                      encode_position_fn=epf, encode_direction_fn=edf)
        last["out"] = out
        return finish(out, tgt_)

    loss_host = torch.empty((), dtype=torch.float32).pin_memory()

    def step_e2e():
        # everything a training iteration needs from the host: the sampled pixel ids and their target colours; the rays
        # are generated on the device from (pose, pixel ids)
        a, c = pix_h.to(dev, non_blocking=True), tgt_h.to(dev, non_blocking=True)
        out = nb.run_one_iter_of_nerf_from_pose(H, W, FOCAL, mc, mf, pose, a, options, mode="train",
                                                encode_position_fn=epf, encode_direction_fn=edf)
        loss = finish(out, c)
        loss_host.copy_(loss.detach(), non_blocking=True)

    def fwd_only():
        with torch.no_grad():
            return nb.run_one_iter_of_nerf(H, W, FOCAL, mc, mf, ro, rd, options, mode="train",
                                           encode_position_fn=epf, encode_direction_fn=edf)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn, steps):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)   # max over ranks
        return ms.item()

    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()   # nvidia-smi needs a few hundred ms for its first sample: start before the warm-up
    for _ in range(max(args.warmup, 3)):
        losses.append(step(ro, rd, tgt).detach())
    torch.cuda.synchronize()
    if rank == 0:
        time.sleep(0.3)
        sampler.rows.clear()  # keep only samples taken from here on (timed region)
    l0 = ops.launch_count()
    total_ms = timed(lambda: losses.append(step(ro, rd, tgt).detach()), args.steps)
    launches = (ops.launch_count() - l0) // args.steps
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last["out"], losses[-1], optim)
    ms_per_step = total_ms / args.steps
    value = RAYS_PER_GPU * world / (ms_per_step / 1e3)

    for _ in range(3):
        step_e2e()
    e2e_ms = timed(step_e2e, args.steps) / args.steps
    for _ in range(3):
        fwd_only()
    fwd_ms = timed(fwd_only, args.steps) / args.steps
    clocks = sampler.stop() if rank == 0 else None   # sampled across the three timed loops (train, e2e, forward)

    # ---- roofline of the dominant kernels, timed alone with CUDA events on this stream ----
    roof = roof_bwd = None
    if rank == 0:
        peaks, peak_kind = measured_peaks()
        blob = ops.pack_weights(arch, optim.items[1]["flat"])
        rays = ops.pack_rays(ro, rd, H, W, FOCAL, CFG["ndc"], CFG["near"], CFG["far"], True)
        span = CFG["far"] - CFG["near"]
        z = torch.sort(torch.rand(RAYS_PER_GPU, NC + NF, device=dev) * span + CFG["near"] + 1e-3, -1).values.contiguous()
        n_wide = 1 + sum(1 for i in range(kw["num_layers"] - 1) if i % kw["skip_connect_every"] == 0 and 0 < i != kw["num_layers"] - 1)
        macs = MACS_PER_POINT[args.arch] - n_wide * (63 - (6 * Lx + 3)) * kw["hidden_size"]   # the table is for L_xyz = 10
        flops_fwd = 2.0 * macs * RAYS_PER_GPU * (NC + NF)

        def t_alone(fn, n=10):
            for _ in range(3):
                fn()
            return timed(fn, n) / n if world == 1 else None

        if world == 1:
            t = t_alone(lambda: ops.mlp_fwd(arch, blob, rays, z, impl=impl))
            ach = flops_fwd / (t * 1e-3) / 1e12
            roof = {"kernel": f"mlp_fwd_{args.kernels.split()[0]} (fine pass, {RAYS_PER_GPU}x{NC + NF} points)", "bound": "tensor",
                    "achieved": ach, "peak": peaks["bf16_tflops"], "peak_source": peak_kind,
                    "unit": "TFLOP/s", "frac": ach / peaks["bf16_tflops"], "ms": t, "algorithmic_flops": flops_fwd}
            raw, stash = ops.mlp_fwd(arch, blob, rays, z, impl=impl, want_stash=True)
            roof["ms_training_forward"] = t_alone(lambda: ops.mlp_fwd(arch, blob, rays, z, impl=impl, want_stash=True), n=5)
            G = torch.randn_like(raw)
            tb = t_alone(lambda: ops.mlp_bwd(arch, blob, rays, z, G, stash, impl=impl))
            achb = 2 * flops_fwd / (tb * 1e-3) / 1e12
            roof_bwd = {"kernel": "mlp_bwd (dgrad + wgrad kernels, fine pass)", "bound": "tensor", "achieved": achb,
                        "peak": peaks["bf16_tflops"], "unit": "TFLOP/s", "frac": achb / peaks["bf16_tflops"], "ms": tb}
            if impl == ops.IMPL_TC:
                # one fused kernel (data-gradient chain + all weight gradients): tensor-bound; its HBM side is the
                # activation tiles it streams back (algorithmic bytes from the library)
                bbytes = float(ops.bwd_bytes_per_point(arch)) * RAYS_PER_GPU * (NC + NF)
                roof_bwd["kernel"] = "mlp_bwd_tc (fused dgrad + wgrad, fine pass)"
                roof_bwd["peak_source"] = peak_kind
                roof_bwd["algorithmic_flops"] = 2 * flops_fwd
                roof_bwd["hbm"] = {"algorithmic_bytes": bbytes, "achieved": bbytes / (tb * 1e-3) / 1e9,
                                   "peak": peaks["hbm_gbs"], "unit": "GB/s",
                                   "frac": bbytes / (tb * 1e-3) / 1e9 / peaks["hbm_gbs"]}
            else:
                # the two CUDA-core backward kernels apart (stage-level entry points of the C ABI)
                gst = ops.mlp_dgrad(arch, blob, G, stash, impl=impl)
                fg = torch.zeros(arch.flat_param_count(), dtype=torch.float32, device=dev)
                roof_bwd["dgrad_ms"] = t_alone(lambda: ops.mlp_dgrad(arch, blob, G, stash, impl=impl, gstash=gst))
                roof_bwd["wgrad_ms"] = t_alone(lambda: ops.mlp_wgrad(arch, rays, z, G, stash, gst, impl=impl, flat_grad=fg))
                del gst, fg
            del stash, raw, G

    # ---- CPU baseline beside it (rank 0, N = 1 only): bounded sample of the same step ----
    cpu = eager = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        n_sample = 1024
        times = cpu_train_steps(args.arch, n_sample, steps=3, warmup=1, threads=best_cpu_threads(args.arch))
        v = n_sample / (sum(times) / len(times))
        cpu = {"value": v, "unit": "rays/s", "cores": torch.get_num_threads(), "kind": "port",
               "sample": f"{n_sample} of the {RAYS_PER_GPU} rays per step, 3 timed steps after 1 warm-up (oracle port of "
                         f"the reference ops, torch CPU; thread count = best of a probe over 8..{os.cpu_count()} host threads)"}
        # the same port as eager PyTorch on this GPU ("same code, device=cuda", SURVEY.md section 8d): the honest
        # PyTorch-ops yardstick next to the CPU figure
        try:
            times = cpu_train_steps(args.arch, RAYS_PER_GPU, steps=5, warmup=2, device=dev)
            ms_e = 1e3 * sum(times) / len(times)
            eager = {"value": RAYS_PER_GPU / (ms_e / 1e3), "unit": "rays/s", "ms_per_step": ms_e,
                     "what": "oracle port of the reference's torch ops run eagerly on this GPU, full batch, fp32 "
                             "(torch.backends.cuda.matmul.allow_tf32 off), wall clock around synchronised steps"}
        except Exception as e:  # pragma: no cover
            eager = {"unavailable": repr(e)[:200]}

    loss_first = float(losses[0]) if losses else None
    loss_last = float(losses[-1]) if losses else None
    if rank == 0 and losses:
        import math
        # a wrong optimizer update or stale packed weights would show here: the loss must be finite and must have gone down
        # from the random-init value over the warm-up + timed steps (random targets: it converges towards 2 * var = 1/6)
        assert math.isfinite(loss_first) and math.isfinite(loss_last), (loss_first, loss_last)
        assert loss_last < loss_first, (loss_first, loss_last)

    if rank == 0:
        line = {
            "metric": f"rays/sec ({RAYS_PER_GPU} rays, 64c+128f samples), train step", "value": value, "unit": "rays/s",
            "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": ms_per_step,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": workload_config(args, world), "kernels": args.kernels,
            "e2e": {"value": RAYS_PER_GPU * world / (e2e_ms / 1e3), "unit": "rays/s", "ms_per_step": e2e_ms,
                    "h2d_bytes_per_step": RAYS_PER_GPU * (8 + 3 * 4), "d2h_bytes_per_step": 4,
                    "api": "run_one_iter_of_nerf_from_pose: pixel ids + targets from pinned host memory, rays generated on the device"},
            "fwd_only": {"value": RAYS_PER_GPU * world / (fwd_ms / 1e3), "unit": "rays/s", "ms_per_step": fwd_ms},
            "gpu_launches": int(launches), "clocks": clocks,
            # `roofline` = the kernel with the largest share of the step: the fused backward (tensor-bound)
            "roofline": roof_bwd or roof, "roofline_fwd": roof, "roofline_bwd": roof_bwd,
            "cpu_baseline": cpu, "torch_eager_gpu": eager,
            "loss": {"first_step": loss_first, "last_step": loss_last, "steps": len(losses),
                     "check": "finite and lower than at the first step (asserted)"},
        }
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


def dump_outputs(path, out, loss, optim):
    """The last timed step's results as float32 .npy files (a few MB for the default workloads)."""
    import numpy as np

    os.makedirs(path, exist_ok=True)
    names = ("rgb_coarse", "disp_coarse", "acc_coarse", "rgb_fine", "disp_fine", "acc_fine")
    arrays = {n: t for n, t in zip(names, out) if t is not None}
    arrays["loss"] = loss.reshape(1)
    for net, it in zip(("coarse", "fine"), optim.items):
        arrays[f"grad_{net}"] = torch.cat([p.grad.reshape(-1) for p in it["params"]])
        arrays[f"params_{net}"] = it["flat"]
    for n, t in arrays.items():
        np.save(os.path.join(path, n + ".npy"), t.detach().float().cpu().numpy())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--arch", default="A1", choices=list(ARCHS))
    ap.add_argument("--kernels", default=os.environ.get("NERFB200_KERNELS", "tc"), choices=["simt", "tc"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--config", type=int, default=2, choices=sorted(CONFIGS))
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the last timed step's outputs, gradients and updated parameters as .npy files to DIR")
    args = ap.parse_args()
    global CFG, RAYS_PER_GPU
    CFG = CONFIGS[args.config]
    RAYS_PER_GPU = CFG["rays"]
    if args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
