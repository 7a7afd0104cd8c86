"""Generate tests/golden/*.npz from the UNMODIFIED reference  --  TEST INFRASTRUCTURE.

Needs a checkout of the unmodified krrish94/nerf-pytorch, named by the environment variable NERF_PYTORCH_REFERENCE:
``NERF_PYTORCH_REFERENCE=/path/to/nerf-pytorch python oracle/make_golden.py``.  The tests only read what it wrote.

What it does, per case:
  1. imports krrish94/nerf-pytorch from that checkout with two ``sys.modules`` shims
     (``imageio`` is only used by the dataset loaders; ``torchsearchsorted`` -- an unpinned
     third-party wheel, requirements.txt:9 -- is replaced by ``torch.searchsorted`` which has
     the same numpy ``side="right"`` semantics);
  2. runs the reference ``run_one_iter_of_nerf`` (and loss.backward()) on seeded inputs while
     recording the tensors ``torch.rand`` / ``torch.randn`` hand out;
  3. runs oracle/nerf_oracle.py twice -- once from the same seed (must reproduce the reference
     bit-for-bit: same RNG order) and once with the recorded randoms injected -- and ASSERTS
     bit equality of all six outputs, the loss and every parameter gradient;
  4. writes inputs, randoms, outputs and gradient digests to tests/golden/<case>.npz.
"""
from __future__ import annotations

import os
import sys
import types

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from oracle import nerf_oracle as O  # noqa: E402

REF = os.environ.get("NERF_PYTORCH_REFERENCE", "")
GOLD = os.path.join(REPO, "tests", "golden")


def import_reference():
    sys.modules.setdefault("imageio", types.ModuleType("imageio"))
    ts = types.ModuleType("torchsearchsorted")
    ts.searchsorted = lambda a, v, out=None, side="left": torch.searchsorted(a, v, right=(side == "right"))
    sys.modules["torchsearchsorted"] = ts
    if not os.path.isdir(REF):
        raise SystemExit("set NERF_PYTORCH_REFERENCE to a checkout of the unmodified krrish94/nerf-pytorch")
    sys.path.insert(0, REF)
    import nerf  # noqa

    return nerf


class RecordRNG:
    """Interpose torch.rand / torch.randn, keep what they return (call order = SURVEY section 5)."""

    def __enter__(self):
        self.rand, self.randn = [], []
        self._r, self._n = torch.rand, torch.randn

        def rand(*a, **k):
            t = self._r(*a, **k)
            self.rand.append(t.clone())
            return t

        def randn(*a, **k):
            t = self._n(*a, **k)
            self.randn.append(t.clone())
            return t

        torch.rand, torch.randn = rand, randn
        return self

    def __exit__(self, *exc):
        torch.rand, torch.randn = self._r, self._n


def make_ref_model(nerf, sd, arch, enc_xyz, enc_dir, use_viewdirs):
    """Reference FlexibleNeRFModel; for archs with a live skip, a subclass that overrides only the
    broken predicate in forward (models.py:240-244) -- SURVEY.md section 8(c) 'oracle repairs'."""
    base = nerf.FlexibleNeRFModel

    class Repaired(base):
        def forward(self, x):
            if self.use_viewdirs:
                xyz, view = x[..., : self.dim_xyz], x[..., self.dim_xyz:]
            else:
                xyz = x[..., : self.dim_xyz]
            x = self.layer1(xyz)
            for i in range(len(self.layers_xyz)):
                if self.layers_xyz[i].in_features != self.layers_xyz[i].out_features:
                    x = torch.cat((x, xyz), dim=-1)
                x = self.relu(self.layers_xyz[i](x))
            if self.use_viewdirs:
                feat = self.relu(self.fc_feat(x))
                alpha = self.fc_alpha(x)
                x = torch.cat((feat, view), dim=-1)
                for l in self.layers_dir:
                    x = self.relu(l(x))
                rgb = self.fc_rgb(x)
                return torch.cat((rgb, alpha), dim=-1)
            return self.fc_out(x)

    needs_repair = any(
        i % arch["skip"] == 0 and i > 0 for i in range(arch["num_layers"] - 1)
    )
    cls = Repaired if needs_repair else base
    m = cls(
        num_layers=arch["num_layers"], hidden_size=arch["hidden"], skip_connect_every=arch["skip"],
        num_encoding_fn_xyz=enc_xyz[0], num_encoding_fn_dir=enc_dir[0],
        include_input_xyz=enc_xyz[1], include_input_dir=enc_dir[1], use_viewdirs=use_viewdirs,
    )
    m.load_state_dict(sd)
    return m


def grad_digest(g: torch.Tensor) -> np.ndarray:
    f = g.detach().double().flatten()
    return np.array([f.sum().item(), f.abs().sum().item(), (f * f).sum().item()] + f[:5].tolist(), dtype=np.float64)


def run_case(nerf, name, *, sd_c, sd_f, arch, enc_xyz, enc_dir, use_viewdirs, options, H, W, focal,
             ro, rd, target, seed, mode="train"):
    epf = nerf.get_embedding_function(*enc_xyz)
    edf = nerf.get_embedding_function(*enc_dir) if use_viewdirs else None
    mc = make_ref_model(nerf, sd_c, arch, enc_xyz, enc_dir, use_viewdirs)
    mf = make_ref_model(nerf, sd_f, arch, enc_xyz, enc_dir, use_viewdirs) if sd_f is not None else None

    # -- the reference
    torch.manual_seed(seed)
    with RecordRNG() as rec:
        ref = nerf.run_one_iter_of_nerf(H, W, focal, mc, mf, ro, rd, options, mode=mode,
                                        encode_position_fn=epf, encode_direction_fn=edf)
    loss = torch.nn.functional.mse_loss(ref[0].reshape(-1, 3), target)
    if ref[3] is not None:
        loss = loss + torch.nn.functional.mse_loss(ref[3].reshape(-1, 3), target)
    loss.backward()

    o = options.nerf.train  # quirk: sampling options always come from .train
    randoms, ri, ni = {}, 0, 0
    if o.perturb:
        randoms["t_rand"] = rec.rand[ri]; ri += 1
    if o.radiance_field_noise_std > 0:
        randoms["noise_c"] = rec.randn[ni]; ni += 1
    if o.num_fine > 0 and o.perturb:
        randoms["u"] = rec.rand[ri]; ri += 1
    if o.num_fine > 0 and o.radiance_field_noise_std > 0:
        randoms["noise_f"] = rec.randn[ni]; ni += 1
    assert ri == len(rec.rand) and ni == len(rec.randn), (ri, len(rec.rand), ni, len(rec.randn))

    # -- the oracle, (a) from the same seed, (b) with injected randoms
    def leaf(sd):
        return {k: v.clone().requires_grad_(True) for k, v in sd.items()} if sd is not None else None

    for label, rnd in (("seeded", None), ("injected", randoms)):
        pc, pf = leaf(sd_c), leaf(sd_f)
        torch.manual_seed(seed)
        out = O.run_one_iter_of_nerf(H, W, focal, pc, pf, ro, rd, options, mode=mode, enc_xyz=enc_xyz,
                                     enc_dir=enc_dir, randoms=rnd)
        for k, (a, b) in enumerate(zip(ref, out)):
            assert (a is None) == (b is None), (name, label, k)
            if a is not None:
                assert a.shape == b.shape, (name, label, k, a.shape, b.shape)
                assert torch.equal(torch.nan_to_num(a, nan=-7.0), torch.nan_to_num(b, nan=-7.0)), (name, label, k)
        ol = O.nerf_loss(tuple(x.reshape(-1, *x.shape[-1:]) if (x is not None and x.dim() == 3) else x for x in out), target)
        assert torch.equal(ol, loss), (name, label, ol.item(), loss.item())
        ol.backward()
        for m, p in ((mc, pc), (mf, pf)):
            if m is None:
                continue
            for k, v in m.named_parameters():
                assert torch.equal(v.grad, p[k].grad), (name, label, k, (v.grad - p[k].grad).abs().max())
    print(f"[golden] {name}: oracle == reference bit-for-bit (outputs, loss, {sum(1 for _ in mc.parameters())} grads/net)")

    save = dict(
        H=np.int64(H), W=np.int64(W), focal=np.float64(focal), seed=np.int64(seed),
        ro=ro.numpy(), rd=rd.numpy(), target=target.numpy(), loss=np.float32(loss.item()),
        enc_xyz=np.array(enc_xyz, dtype=np.int64), enc_dir=np.array(enc_dir, dtype=np.int64),
        use_viewdirs=np.int64(use_viewdirs), no_ndc=np.int64(options.dataset.no_ndc),
        near=np.float64(options.dataset.near), far=np.float64(options.dataset.far),
        num_coarse=np.int64(o.num_coarse), num_fine=np.int64(o.num_fine), perturb=np.int64(bool(o.perturb)),
        lindisp=np.int64(o.lindisp), white_background=np.int64(o.white_background),
        noise_std=np.float64(o.radiance_field_noise_std), mode=np.array(mode),
        arch=np.array([arch["num_layers"], arch["hidden"], arch["skip"]], dtype=np.int64),
    )
    for k, v in randoms.items():
        save["rnd_" + k] = v.numpy()
    names = ["rgb_coarse", "disp_coarse", "acc_coarse", "rgb_fine", "disp_fine", "acc_fine"]
    for n, t in zip(names, ref):
        if t is not None:
            save["out_" + n] = t.detach().numpy()
    for tag, m in (("c", mc), ("f", mf)):
        if m is None:
            continue
        for k, v in m.named_parameters():
            save[f"gd_{tag}_{k}"] = grad_digest(v.grad)
    return save


def lego_rays(nerf, n, H=400, W=400, focal=555.5555155968841, seed=0):
    pose = torch.from_numpy(nerf.load_blender.pose_spherical(30.0, -30.0, 4.0).astype(np.float32))
    ro, rd = nerf.get_ray_bundle(H, W, focal, pose)
    # oracle helpers pinned against the reference too
    assert torch.equal(pose, O.pose_spherical(30.0, -30.0, 4.0))
    ro2, rd2 = O.get_ray_bundle(H, W, focal, pose)
    assert torch.equal(ro, ro2) and torch.equal(rd, rd2)
    g = torch.Generator().manual_seed(seed)
    # bias the selection towards the object (image centre) so that rays actually hit density
    idx = torch.randperm(H * W, generator=g)[: 4 * n]
    yy, xx = idx // W, idx % W
    keep = ((yy - H / 2).abs() < H * 0.3) & ((xx - W / 2).abs() < W * 0.3)
    idx = torch.cat([idx[keep], idx[~keep]])[:n]
    return ro.reshape(-1, 3)[idx].contiguous(), rd.reshape(-1, 3)[idx].contiguous(), g


def main():
    nerf = import_reference()
    os.makedirs(GOLD, exist_ok=True)
    torch.set_num_threads(1)  # fixed reduction order for the bit-for-bit assertions

    lego = torch.load(f"{REF}/pretrained/lego-lowres/checkpoint199999.ckpt", map_location="cpu", weights_only=False)
    fern = torch.load(f"{REF}/pretrained/fern-lowres/checkpoint249999.ckpt", map_location="cpu", weights_only=False)
    A0 = dict(num_layers=4, hidden=128, skip=4)
    A1 = dict(num_layers=8, hidden=128, skip=3)

    # pretrained weights travel as fixtures (fp32, reference key names)
    np.savez(os.path.join(GOLD, "weights_lego_lowres.npz"),
             **{f"c.{k}": v.numpy() for k, v in lego["model_coarse_state_dict"].items()},
             **{f"f.{k}": v.numpy() for k, v in lego["model_fine_state_dict"].items()})
    np.savez(os.path.join(GOLD, "weights_fern_lowres.npz"),
             **{f"c.{k}": v.numpy() for k, v in fern["model_coarse_state_dict"].items()},
             **{f"f.{k}": v.numpy() for k, v in fern["model_fine_state_dict"].items()})

    N = 96
    ro, rd, g = lego_rays(nerf, N)
    target = torch.rand(N, 3, generator=g)
    cases = {}

    # 1. lego A0, training sampler (config/lego.yml with num_fine 64 -> 128, BASELINE config 2)
    cases["lego_a0_train"] = run_case(
        nerf, "lego_a0_train", sd_c=lego["model_coarse_state_dict"], sd_f=lego["model_fine_state_dict"], arch=A0,
        enc_xyz=(10, True, True), enc_dir=(4, True, True), use_viewdirs=True,
        options=O.make_options(num_coarse=64, num_fine=128, perturb=True, radiance_field_noise_std=0.2),
        H=400, W=400, focal=555.5555155968841, ro=ro, rd=rd, target=target, seed=1234)

    # 2. deterministic sampler, white background, no noise, validation reshape (ro/rd as an image patch)
    Hp, Wp = 8, 12
    cases["lego_a0_det_white_val"] = run_case(
        nerf, "lego_a0_det_white_val", sd_c=lego["model_coarse_state_dict"], sd_f=lego["model_fine_state_dict"],
        arch=A0, enc_xyz=(10, True, True), enc_dir=(4, True, True), use_viewdirs=True,
        options=O.make_options(num_coarse=64, num_fine=64, perturb=False, radiance_field_noise_std=0.0,
                               white_background=True),
        H=400, W=400, focal=555.5555155968841, ro=ro.view(Hp, Wp, 3), rd=rd.view(Hp, Wp, 3), target=target,
        seed=7, mode="validation")

    # 3. fern A0: NDC rays, L_xyz = 6, near 0 / far 1, noise std 1.0 (config/fern.yml), BASELINE config 4
    H, W, focal = 378, 504, 407.5658
    pose = torch.eye(4)[:3, :4].clone()
    fro, frd = nerf.get_ray_bundle(H, W, focal, torch.eye(4))
    gi = torch.Generator().manual_seed(3)
    idx = torch.randperm(H * W, generator=gi)[:N]
    fro, frd = fro.reshape(-1, 3)[idx].contiguous(), frd.reshape(-1, 3)[idx].contiguous()
    cases["fern_a0_ndc"] = run_case(
        nerf, "fern_a0_ndc", sd_c=fern["model_coarse_state_dict"], sd_f=fern["model_fine_state_dict"], arch=A0,
        enc_xyz=(6, True, True), enc_dir=(4, True, True), use_viewdirs=True,
        options=O.make_options(no_ndc=False, near=0.0, far=1.0, num_coarse=64, num_fine=128, perturb=True,
                               radiance_field_noise_std=1.0),
        H=H, W=W, focal=focal, ro=fro, rd=frd, target=target, seed=99)

    # 4. A1 = config/lego.yml as written (8x128, skip 3), default init, lindisp, coarse+fine of odd sizes
    gen = torch.Generator().manual_seed(2024)
    sd1c = O.init_flexible_nerf(8, 128, 3, 10, 4, generator=gen)
    sd1f = O.init_flexible_nerf(8, 128, 3, 10, 4, generator=gen)
    cases["a1_skip_lindisp"] = run_case(
        nerf, "a1_skip_lindisp", sd_c=sd1c, sd_f=sd1f, arch=A1, enc_xyz=(10, True, True), enc_dir=(4, True, True),
        use_viewdirs=True,
        options=O.make_options(near=0.5, far=6.0, num_coarse=48, num_fine=80, perturb=True, lindisp=True,
                               radiance_field_noise_std=0.2, white_background=True),
        H=400, W=400, focal=555.5555155968841, ro=ro, rd=rd, target=target, seed=5)
    cases["a1_skip_lindisp"]["init_seed"] = np.int64(2024)

    # 5. no view directions (fc_out head), linear frequency sampling, no include_input, coarse only
    gen = torch.Generator().manual_seed(77)
    sd2 = O.init_flexible_nerf(4, 128, 4, 5, 4, include_input_xyz=False, use_viewdirs=False, generator=gen)
    cases["a0_noview_coarse_only"] = run_case(
        nerf, "a0_noview_coarse_only", sd_c=sd2, sd_f=None, arch=A0, enc_xyz=(5, False, False),
        enc_dir=(4, True, True), use_viewdirs=False,
        options=O.make_options(use_viewdirs=False, num_coarse=64, num_fine=0, perturb=True,
                               radiance_field_noise_std=0.0),
        H=400, W=400, focal=555.5555155968841, ro=ro, rd=rd, target=target, seed=11)
    cases["a0_noview_coarse_only"]["init_seed"] = np.int64(77)

    for name, save in cases.items():
        np.savez_compressed(os.path.join(GOLD, name + ".npz"), **save)
    print("[golden] wrote", sorted(os.listdir(GOLD)))


if __name__ == "__main__":
    main()
