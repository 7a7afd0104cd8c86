"""GPU: the per-ray kernels around the MLP at every sample count the render entry points accept (2 <= n_coarse,
n_coarse + n_fine <= 1024, n_coarse >= 4 with a fine pass), against CPU fp32 and fp64 oracles.

Each kernel changes shape with the count.  The boundaries, and the counts that reach them:
  sample_coarse_kernel (one thread per sample)
    - linspace01's two halves (q < n / 2 counts up from 0, the rest down from 1): every n_coarse in 2..1024;
    - perturb's one-sided strata at i = 0 and i = n_coarse - 1, and lindisp: each on and off at every count;
    - lindisp at NDC bounds, near 0: 1 / near = inf makes the last depth inf * 0 = NaN, and its stratum NaN; a ray
      with near == far.
  sample_pdf_merge_kernel (one warp per ray, 4 warps per CTA, 4 (npow2 + 3 n_coarse) floats of shared memory)
    - shared memory over 48 KiB, which needs the cudaFuncSetAttribute opt-in: (683, 1) and every n_coarse above it;
      (682, 2) is the largest request below it; (1023, 1) the largest of all;
    - the bitonic sort's +inf padding to npow2: n_coarse + n_fine = 2^k (none) and 2^k + 1 (npow2 doubles), by every
      n_fine at n_coarse in {4, 15, 33, 34, 683} and n_fine = 1024 - n_coarse (npow2 = 1024, unpadded) at every
      n_coarse;
    - the lanes' strided loops over n_coarse - 2 weights and n_coarse - 1 bins: 31, 32 at n_coarse 33, 34 (and every
      n_coarse in 4..1023); over n_fine samples: every n_fine at the five n_coarse above;
    - the sequential fp64 cdf scan on lane 0 over up to 1021 weights: every n_coarse;
    - the search (side="right"): u = 0, u equal to a cdf entry, u = 1 (the det linspace's last), one-hot weights whose
      empty bins fall under denom < 1e-5, all-zero weights (a uniform pdf), mass only on the first or the last interior
      sample; n_coarse = 1020 with n_fine 1..4.
  composite_fwd_kernel / composite_bwd_kernel<false> (the render path's instances; one warp per ray, lane L owns
  samples [L C, (L + 1) C) with C = ceil(S / 32))
    - S <= 32: one sample per lane and 32 - S lanes idle; S = 33: C = 2, lane 16 holds one sample, 17..31 idle;
      S = 1024: 32 samples in every lane: every S in 1..1024, each with one of the four (noise std 0 / 1, white
      background or not) in turn, and all four at the counts where the chunks change shape (LANE_COUNTS);
    - the backward's 48 S bytes of dynamic shared memory, exactly 48 KiB at S = 1024 (no opt-in needed);
    - near-opaque rays where q reaches 1e-10 and T underflows to 0; empty rays (acc 0, disp NaN).
Every kernel runs on 37 rays (the last of 10 CTAs has one warp of four busy), and on their first 1 and 5 (resampling:
with the seeded u): a ray's results depend on its own inputs only, so the short batches must give the long batch's
bits.

Oracles and bars:
  sample_coarse      O.stratified_z in fp32 on the CPU with the same t_rand, bit for bit (NaN where it is NaN): torch's
                     CPU linspace and linspace01 are the same symmetric FMA formula, and every other step is one IEEE
                     operation, which the kernel writes with _rn intrinsics.
  sample_pdf_merge   given the kernel's own cdf (cdf_in), indices, samples and z_fine are O.sample_from_cdf's and
                     the sort of cat(z_coarse, samples) on the CPU exactly, and the in-kernel cdf gives the same
                     bits.  The in-kernel cdf against the fp64 cdf of the same fp32 weights: CDF_ULPS.
  compositing        helpers.composite64 of the same fp32 inputs (fp64, on the device): rgb, acc, depth and weights
                     within COMP_TOL of their scale; disp is fp32 1 / max(1e-10, depth / acc) of the kernel's own depth
                     and acc, bit for bit, so NaN exactly where acc is 0, which is exactly where the fp64 acc is 0;
                     d_raw against fp64 autograd of composite64 (helpers.composite_grad64) within COMP_GRAD_TOL of its
                     scale.
Measured on an H100 80GB HBM3 at a 700 W power limit and 1980 MHz SM clock: the file runs in 58 s (resampling 32 s,
compositing 18 s, sample_coarse 8 s); compositing outputs [4.3e-6 of their scale] and d_raw [4.2e-6] against COMP_TOL
and COMP_GRAD_TOL; the cdf's worst figure beside CDF_ULPS."""
import time

import numpy as np
import pytest
import torch

from helpers import bits_equal, composite64, composite_grad64
from mlp_checks import COMP_GRAD_TOL, COMP_TOL
from oracle import nerf_oracle as O

pytestmark = pytest.mark.gpu

# In-kernel cdf against the fp64 cdf c of the same fp32 weights w, in units of u = 2^-24 [2.12].  The kernel
# forms a_j = fp32(w_j + 1e-5), the total A = fp32(sum a_j) (an fp64 sum, rounded once), p_j = fp32(a_j / A) and
# cdf_k = fp32(sum_{j<k} p_j) (an fp64 scan, rounded per entry); its fp64 sums add below 2^-40 u.
#   - w + 1e-5 rounds each term by a relative 2^-24, and 1e-5f differs from 1e-5 by a relative 2^-28.6: 1.05 u in all.
#     Perturbing the terms before and after k by +-e moves c_k = X / (X + Y) by at most 2 e c_k (1 - c_k).
#   - The total's rounding scales every p_j by 1 + b, |b| <= u; each p_j's own rounding moves it by u p_j, at most u c_k
#     summed over j < k because the pdf sums to 1: together 2 u c_k.
#   - The entry's final rounding: half an ulp, u / 2 below 1 and u at or above 1 (a cdf entry of 1 + 2^-23).
# 2.1 u c (1 - c) + 2 u c peaks at 2.001 u (c = 0.976); an entry that rounds at or above 1 has c >= 1 - 2.001 u, where the
# first term vanishes and the final rounding is u: at most 3 u in every case, whatever the count.
CDF_ULPS = 3

N_RAYS = 37
PREFIXES = (1, 5)  # the shorter batches, the first rays of the 37


def report(what, value):
    print(f"measured {what}: {value}")


def _bits_or_nan_equal(a, b):
    """Same shape, NaN at the same places and the same bits elsewhere (a NaN's payload is the platform's own)."""
    if a.shape != b.shape:
        return False
    na, nb_ = torch.isnan(a), torch.isnan(b)
    if not torch.equal(na, nb_):
        return False
    return torch.equal(torch.where(na, 0.0, a).view(torch.int32), torch.where(nb_, 0.0, b).view(torch.int32))


def _prefixes_agree(run, full):
    """run(k) on the first k rays gives the first k rows of every tensor of full (the 37-ray run), for k in PREFIXES."""
    for k in PREFIXES:
        for a, b in zip(run(k), full):
            if b is not None and not bits_equal(a, b[:k]):
                return False
    return True


# ------------------------------------------------------------------------------------------------------------------------
# sample_coarse
# ------------------------------------------------------------------------------------------------------------------------
def _coarse_rays():
    """37 ray rows [o d near far]: lego bounds (2, 6) and NDC bounds (0, 1) alternating, ray 3 with near == far."""
    g = torch.Generator().manual_seed(1)
    rays = torch.randn(N_RAYS, 8, generator=g)
    rays[0::2, 6], rays[0::2, 7] = 2.0, 6.0
    rays[1::2, 6], rays[1::2, 7] = 0.0, 1.0
    rays[3, 6] = rays[3, 7] = 3.7
    return rays


def test_sample_coarse_matches_the_fp32_oracle_bit_for_bit_at_every_count():
    from nerf_pytorch_b200 import ops

    t0 = time.perf_counter()
    rays = _coarse_rays()
    rays_d = rays.cuda()
    g = torch.Generator().manual_seed(2)
    nan_counts = 0
    for nc in range(2, 1025):
        t_rand = torch.rand(N_RAYS, nc, generator=g)
        t_d = t_rand.cuda()
        for perturb in (False, True):
            for lindisp in (False, True):
                ctx = (nc, perturb, lindisp)
                z = ops.sample_coarse(rays_d, t_d, nc, perturb, lindisp)
                want = O.stratified_z(rays[:, 6:7], rays[:, 7:8], nc, lindisp, perturb, t_rand if perturb else None,
                                      torch.float32).contiguous()
                z_cpu = z.cpu()
                assert _bits_or_nan_equal(z_cpu, want), ctx + (int((z_cpu != want).sum()),)
                nan_counts += int(torch.isnan(z_cpu).sum())
                assert _prefixes_agree(lambda k: (ops.sample_coarse(rays_d[:k], t_d[:k], nc, perturb, lindisp),),
                                       (z,)), ctx
    assert nan_counts > 0  # lindisp at near 0 reached its NaN
    report("sample_coarse, s", round(time.perf_counter() - t0, 1))


# ------------------------------------------------------------------------------------------------------------------------
# sample_pdf_merge
# ------------------------------------------------------------------------------------------------------------------------
PDF_PAIRS = sorted({(nc, 1) for nc in range(4, 1024)} | {(nc, 1024 - nc) for nc in range(4, 1024)}
                   | {(nc, nf) for nc in (4, 15, 33, 34, 683) for nf in range(1, 1025 - nc)}
                   | {(1020, nf) for nf in range(1, 5)} | {(682, 2)})


def _pdf_inputs(nc, g):
    """z_coarse [37, nc] sorted in [2, 6) and weights [37, nc] (only 1 .. nc - 2 are read): ray 0 rand^4, 1 all zero,
    2 one-hot, 3 mass on the first interior sample only, 4 on the last only; then uniform, rand^40 and rand^4 rows.
    The end weights, which the kernel must ignore, are random on every ray."""
    z = torch.sort(torch.rand(N_RAYS, nc, generator=g) * 4 + 2, -1).values
    w = torch.rand(N_RAYS, nc, generator=g)
    inner = w[:, 1:-1]
    inner[0] = inner[0] ** 4
    inner[1:5] = 0.0
    inner[2, int(torch.randint(0, nc - 2, (1,), generator=g))] = 1.0
    inner[3, 0] = 0.7
    inner[4, -1] = 0.7
    inner[5::3] = 0.5
    inner[6::3] = inner[6::3] ** 40
    inner[7::3] = inner[7::3] ** 4
    return z, w


def _seeded_u(cdf, nf, g):
    """Uniforms [37, nf], with u = 0 on the even rays and a cdf entry of the ray on the odd ones (one of each on every
    ray when nf > 1), which searchsorted(side="right") must place after it."""
    u = torch.rand(N_RAYS, nf, generator=g)
    r = torch.arange(N_RAYS)
    for i in range(min(nf, 2)):
        entry = cdf[r, (7 * r + 3 * i) % cdf.shape[1]]
        u[r, (r + i) % nf] = torch.where((r + i) % 2 == 0, 0.0, entry)
    return u


def _mismatch(a, b):
    """A device bool: a and b differ in some bit."""
    return (a.contiguous().view(torch.int32) != b.contiguous().view(torch.int32)).any()


def test_sample_pdf_merge_matches_the_oracles_at_every_count():
    """Per n_coarse one draw of z and weights serves every n_fine paired with it; the fp32 oracle takes all those
    n_fine's u at once (each u is searched on its own), and each z_fine is checked against its own sort."""
    from nerf_pytorch_b200 import ops

    t0 = time.perf_counter()
    g = torch.Generator().manual_seed(3)
    by_nc = {}
    for nc, nf in PDF_PAIRS:
        by_nc.setdefault(nc, []).append(nf)
    worst = 0.0
    for nc, nfs in by_nc.items():
        z, w = _pdf_inputs(nc, g)
        z_d, w_d = z.cuda(), w.cuda()
        bins = 0.5 * (z[:, 1:] + z[:, :-1])
        w64 = w[:, 1:-1].double() + 1e-5
        cdf64 = torch.nn.functional.pad(torch.cumsum(w64 / w64.sum(-1, keepdim=True), -1), (1, 0))
        cdf_d = ops.sample_pdf_merge(z_d, w_d, None, nfs[0], want_aux=True)[3]
        cdf = cdf_d.cpu()
        ulps = (cdf.double() - cdf64).abs().max().item() / 2.0 ** -24
        worst = max(worst, ulps)
        assert ulps <= CDF_ULPS, (nc, "cdf in 2^-24 units", ulps)
        for seeded in (False, True):
            us = [_seeded_u(cdf, nf, g) if seeded else torch.linspace(0.0, 1.0, nf).expand(N_RAYS, nf) for nf in nfs]
            outs, flags = [], []
            for nf, u in zip(nfs, us):
                u_d = u.cuda() if seeded else None
                got = ops.sample_pdf_merge(z_d, w_d, u_d, nf, want_aux=True)
                given = ops.sample_pdf_merge(z_d, w_d, u_d, nf, cdf_in=cdf_d, want_aux=True)
                outs.append(given[:3])
                # in-kernel: the same cdf, so the same bits; the 1- and 5-ray batches: the 37-ray batch's first rays
                flags += [_mismatch(a, b) for a, b in zip(got, (*given[:3], cdf_d))]
                for k in PREFIXES if seeded else ():
                    short = ops.sample_pdf_merge(z_d[:k], w_d[:k], u_d[:k], nf, want_aux=True)
                    flags += [_mismatch(a, b[:k]) for a, b in zip(short, got)]
            flags = torch.stack(flags).view(len(nfs), -1).cpu()
            for nf, f in zip(nfs, flags):
                assert not f.any(), (nc, nf, seeded, "in-kernel cdf (4), then seeded: 1 and 5 rays (4 each)", f.tolist())
            # given the kernel's own cdf: indices and samples are the fp32 oracle's, z_fine the sort of the merge
            want_zs, want_inds = O.sample_from_cdf(bins, cdf, torch.cat(us, 1))
            z_fine = torch.cat([o[0] for o in outs], 1).cpu()
            zs = torch.cat([o[1] for o in outs], 1).cpu()
            inds = torch.cat([o[2] for o in outs], 1).cpu()
            ctx = (nc, nfs[0], nfs[-1], "seeded u" if seeded else "det u")
            assert torch.equal(inds.long(), want_inds), ctx + ("indices given the cdf",)
            assert bits_equal(zs, want_zs.contiguous()), ctx + ("samples given the cdf",)
            q0 = p0 = 0
            for nf in nfs:
                want_zf = np.sort(np.concatenate((z.numpy(), want_zs[:, q0:q0 + nf].numpy()), 1), 1)
                assert bits_equal(z_fine[:, p0:p0 + nc + nf], torch.from_numpy(want_zf)), ctx + (nf, "z_fine")
                q0, p0 = q0 + nf, p0 + nc + nf
    report("in-kernel cdf against fp64, 2^-24 units", worst)
    report("sample_pdf_merge, s", round(time.perf_counter() - t0, 1))


# ------------------------------------------------------------------------------------------------------------------------
# compositing
# ------------------------------------------------------------------------------------------------------------------------
EMPTY = 2  # the empty ray: no density after any noise
OPAQUE = torch.arange(N_RAYS) % 2 == 1  # near-opaque rays; the others (but EMPTY) hold random raw


def _composite_inputs(s, g):
    """raw [37, s, 4], z [37, s] sorted in [2, 6), rays [37, 11] (directions N(0, 1)), unit noise [37, s], upstream
    g_out [37, 8].  Random rays: raw ~ 2 N(0, 1) with the first sigma at least 2.  Near-opaque rays: sigma
    log-uniform over 1e2 .. 1e4 (so a sample's sigma delta |d| is ~1 .. 1e2: alpha rounds to 1 and q to 1e-10, and T
    passes through the fp32 subnormals to 0).  The empty ray has sigma -50.  g_out's depth slot and padding, which the
    render path's backward ignores, are random too; its disp weight is 0 on the empty ray, whose disp is NaN."""
    raw = torch.randn(N_RAYS, s, 4, generator=g) * 2
    raw[:, 0, 3] = raw[:, 0, 3].abs() + 2.0
    raw[OPAQUE, :, 3] = 10.0 ** (2 + 2 * torch.rand(int(OPAQUE.sum()), s, generator=g))
    raw[EMPTY, :, 3] = -50.0
    z = torch.sort(torch.rand(N_RAYS, s, generator=g) * 4 + 2, -1).values
    rays = torch.randn(N_RAYS, 11, generator=g)
    noise = torch.randn(N_RAYS, s, generator=g)
    g_out = torch.randn(N_RAYS, 8, generator=g)
    g_out[EMPTY, 3] = 0.0
    return raw, z, rays, noise, g_out


# (noise_std, white background): all four at the counts where the lanes' chunks change shape, one in turn elsewhere
OPTIONS = [(0.0, False), (1.0, False), (0.0, True), (1.0, True)]
LANE_COUNTS = {1, 2, 31, 32, 33, 63, 64, 65, 992, 993, 1023, 1024}


def test_compositing_matches_fp64_at_every_count():
    from nerf_pytorch_b200 import ops

    t0 = time.perf_counter()
    g = torch.Generator().manual_seed(4)
    opaque = OPAQUE.cuda()
    worst = {"outputs": 0.0, "d_raw": 0.0}
    names = ("rgb", "acc", "depth", "weights", "d_raw")
    for s in range(1, 1025):
        raw, z, rays, noise, g_out = (t.cuda() for t in _composite_inputs(s, g))
        dirs = rays[:, 3:6]
        for std, white in (OPTIONS if s in LANE_COUNTS else OPTIONS[s % 4:s % 4 + 1]):
            ctx = (s, std, white)
            out, w = ops.composite_fwd(raw, z, rays, noise, std, white)
            d_raw = ops.composite_bwd(raw, z, rays, noise, g_out, std, white)
            rgb, _, acc, w64, depth = composite64(raw, z, dirs, std, white, noise)
            d64 = composite_grad64(raw, z, dirs, g_out, std, white, noise)
            # one transfer per case: the errors relative to scale, then the exact checks as 0 / 1
            errs = [(a.double() - b).abs().max() / b.abs().max()
                    for a, b in ((out[:, :3], rgb), (out[:, 4], acc), (out[:, 5], depth), (w, w64), (d_raw, d64))]
            ratio = out[:, 5] / out[:, 4]
            disp = torch.where(torch.isnan(ratio), ratio, 1.0 / torch.clamp_min(ratio, 1e-10))
            nan = torch.isnan(out[:, 3])
            exact = [(nan != torch.isnan(disp)).any() | _mismatch(torch.where(nan, 0.0, out[:, 3]),
                                                                       torch.where(nan, 0.0, disp)),
                     (nan != (acc == 0)).any() | ~nan[EMPTY],
                     ~(w[opaque, -1] == 0).any() if s >= 64 else torch.zeros((), dtype=torch.bool, device="cuda")]
            for k in PREFIXES:
                short = (*ops.composite_fwd(raw[:k], z[:k], rays[:k], noise[:k], std, white),
                         ops.composite_bwd(raw[:k], z[:k], rays[:k], noise[:k], g_out[:k], std, white))
                exact += [_mismatch(a, b[:k]) for a, b in zip(short, (out, w, d_raw))]
            e = torch.stack(errs).cpu().tolist()
            bad = torch.stack([torch.as_tensor(x, device="cuda") for x in exact]).cpu().tolist()
            worst["outputs"] = max(worst["outputs"], *e[:4])
            worst["d_raw"] = max(worst["d_raw"], e[4])
            for name, x in zip(names, e):
                assert x <= (COMP_GRAD_TOL if name == "d_raw" else COMP_TOL), ctx + (name, x)
            assert not bad[0], ctx + ("disp is not fp32 1 / max(1e-10, depth / acc) of the kernel's outputs",)
            assert not bad[1], ctx + ("disp NaN where the fp64 acc is not 0, or finite on the empty ray",)
            assert not bad[2], ctx + ("no near-opaque ray's T underflowed",)
            assert not any(bad[3:]), ctx + ("1 and 5 rays (out, weights, d_raw each) against 37", bad[3:])
    report("compositing outputs / d_raw against fp64, relative to scale", worst)
    report("compositing, s", round(time.perf_counter() - t0, 1))
