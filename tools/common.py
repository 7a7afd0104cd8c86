"""Shared pieces of the timing tools: the card line printed beside every figure, CUDA-event timers, PSNR, the median
summary of a list of timings and the networks of the render scenes.  Importing it puts the repository root and tests/
(for helpers.shipped_models and helpers.load_weights) on sys.path."""
import math
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def card():
    """The current GPU's name, power limit, SM clock and max SM clock as nvidia-smi reports them (the device name when
    nvidia-smi is unavailable)."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True,
                           timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover - depends on the host
        q = f"nvidia-smi unavailable ({e})"
    return q or torch.cuda.get_device_name()


def timed_once(fn):
    """(ms, fn()): one call timed with CUDA events."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def timed_mean(fn, iters):
    """Mean ms per call of ``iters`` back-to-back calls, timed with CUDA events."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def psnr(a, b):
    """PSNR (dB) from the fp64 mean squared error; inf when a and b are equal."""
    mse = (a.double() - b.double()).pow(2).mean().item()
    return math.inf if mse == 0 else -10.0 * math.log10(mse)


def median(ms):
    return dict(ms=statistics.median(ms), range=(min(ms), max(ms)))


def models(weights, layers, skip, l_xyz):
    """(coarse, fine) FlexibleNeRFModels (hidden 128) on the GPU, at torch's init under seed 0, holding the shipped
    low-res ``weights`` ("lego", "fern") unless that is None."""
    import nerf_pytorch_b200 as nb
    from helpers import load_weights

    torch.manual_seed(0)
    out = []
    for sd in (load_weights(f"{weights}_lowres") if weights else (None, None)):
        m = nb.FlexibleNeRFModel(num_layers=layers, hidden_size=128, skip_connect_every=skip, num_encoding_fn_xyz=l_xyz,
                                 num_encoding_fn_dir=4)
        if sd is not None:
            m.load_state_dict(sd)
        out.append(m.cuda())
    return out
