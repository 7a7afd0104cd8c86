"""lego PSNR after equal iterations at scale: this library (CUDA, FusedAdam) vs the reference algorithm run as eager PyTorch
on the same GPU (oracle port, the reference's ATen ops in the reference's order), several sampling-noise seeds each.

No dataset is on disk (SURVEY.md section 0.5), so the images come from a TEACHER: the shipped pretrained lego-lowres fine
network rendered through this library's deterministic forward (perturb off, noise 0) at 400 x 400 from 8 spherical poses
(load_blender.py:32-37).  Students: config/lego.yml as written (A1 = 8 x 128, skip every 3, coarse + fine, 64 + 128 samples,
perturb on, noise std 0.2, Adam 5e-3 with the reference's exponential decay), started from the SAME initial weights and
fed the SAME ray batches in the same order; every run draws its own sampling noise, like two runs of the reference would.
PSNR is measured on 8192 held-out rays with the deterministic sampler.  Writes psnr_out/psnr_scale.json.

    PSNR_ITERS=5000 PSNR_BATCH=1024 PSNR_SEEDS=3 python tools/psnr_scale.py
"""
import json, math, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
from helpers import load_weights
from oracle import nerf_oracle as O
import nerf_pytorch_b200 as nb
from nerf_pytorch_b200 import parallel, train_utils

ITERS = int(os.environ.get("PSNR_ITERS", "5000"))
BATCH = int(os.environ.get("PSNR_BATCH", "1024"))
SEEDS = int(os.environ.get("PSNR_SEEDS", "3"))
EVAL_EVERY = int(os.environ.get("PSNR_EVAL", "500"))
H = W = int(os.environ.get("PSNR_RES", "400"))
FOCAL = 0.5 * W / math.tan(0.5 * 0.6911112070083618)
ARCH = dict(num_layers=8, hidden_size=128, skip_connect_every=3)
dev = torch.device("cuda", 0)
torch.cuda.set_device(0)


def model_from(sd, **kw):
    m = nb.FlexibleNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4, **kw)
    m.load_state_dict(sd)
    return m.to(dev)


# ---- teacher images (this library's deterministic forward over the pretrained lego-lowres networks) ----
sd_tc, sd_tf = load_weights("lego_lowres")
tc_, tf_ = model_from(sd_tc), model_from(sd_tf)
epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
det = O.make_options(num_coarse=64, num_fine=128, perturb=False, radiance_field_noise_std=0.0, white_background=False)
g = torch.Generator().manual_seed(0)
ros, rds, tgts = [], [], []
for th in range(0, 360, 45):
    pose = O.pose_spherical(float(th), -30.0, 4.0)
    ro, rd = O.get_ray_bundle(H, W, FOCAL, pose)
    with torch.no_grad():
        out = nb.run_one_iter_of_nerf(H, W, FOCAL, tc_, tf_, ro.reshape(-1, 3).to(dev), rd.reshape(-1, 3).to(dev), det,
                                      encode_position_fn=epf, encode_direction_fn=edf)
    ros.append(ro.reshape(-1, 3)); rds.append(rd.reshape(-1, 3)); tgts.append(out[3].cpu())
ro_all, rd_all, tg_all = torch.cat(ros).to(dev), torch.cat(rds).to(dev), torch.cat(tgts).to(dev)
perm = torch.randperm(ro_all.shape[0], generator=g).to(dev)
hold, pool = perm[:8192], perm[8192:]
print(f"teacher set: {ro_all.shape[0]} rays, mean rgb {tg_all.mean().item():.3f}", flush=True)

train_opt = O.make_options(num_coarse=64, num_fine=128, perturb=True, radiance_field_noise_std=0.2)  # config/lego.yml
gi = torch.Generator().manual_seed(1)
sd0c = O.init_flexible_nerf(ARCH["num_layers"], ARCH["hidden_size"], ARCH["skip_connect_every"], 10, 4, generator=gi)
sd0f = O.init_flexible_nerf(ARCH["num_layers"], ARCH["hidden_size"], ARCH["skip_connect_every"], 10, 4, generator=gi)
pick = torch.randint(0, pool.shape[0], (ITERS, BATCH), generator=g).to(dev)
LR0, DECAY, FACTOR = 5e-3, 250, 0.1     # config/lego.yml; train_nerf.py:261-270: lr = lr0 * factor ** (i / (decay * 1000))


def psnr(rgb):
    return -10 * math.log10(torch.nn.functional.mse_loss(rgb, tg_all[hold]).item())


def train_ours(seed):
    torch.manual_seed(seed)
    mc, mf = model_from(sd0c, **ARCH), model_from(sd0f, **ARCH)
    arch = train_utils._arch_of(mc, (10, True, True), (4, True, True))
    opt = parallel.FusedAdam([(mc, arch), (mf, arch)], lr=LR0, lr_decay=DECAY, lr_decay_factor=FACTOR)
    curve = []
    for i in range(ITERS):
        idx = pool[pick[i]]
        out = nb.run_one_iter_of_nerf(H, W, FOCAL, mc, mf, ro_all[idx], rd_all[idx], train_opt, mode="train",
                                      encode_position_fn=epf, encode_direction_fn=edf)
        tgt = tg_all[idx]
        loss = torch.nn.functional.mse_loss(out[0], tgt) + torch.nn.functional.mse_loss(out[3], tgt)
        opt.zero_grad(); loss.backward(); opt.step()
        if (i + 1) % EVAL_EVERY == 0:
            with torch.no_grad():
                o = nb.run_one_iter_of_nerf(H, W, FOCAL, mc, mf, ro_all[hold], rd_all[hold], det, mode="validation",
                                            encode_position_fn=epf, encode_direction_fn=edf)
            curve.append((i + 1, psnr(o[3].reshape(-1, 3))))
    return curve


def train_reference_eager(seed):
    """The oracle port (reference ops, reference order) as eager PyTorch on the GPU; torch.optim.Adam with the reference's
    post-step learning-rate update."""
    torch.manual_seed(seed)
    sc = {k: v.clone().to(dev).requires_grad_(True) for k, v in sd0c.items()}
    sf = {k: v.clone().to(dev).requires_grad_(True) for k, v in sd0f.items()}
    opt = torch.optim.Adam(list(sc.values()) + list(sf.values()), lr=LR0)
    curve = []
    for i in range(ITERS):
        idx = pool[pick[i]]
        with torch.device(dev):
            out = O.run_one_iter_of_nerf(H, W, FOCAL, sc, sf, ro_all[idx], rd_all[idx], train_opt)
        loss = O.nerf_loss(out, tg_all[idx])
        opt.zero_grad(); loss.backward(); opt.step()
        for pg in opt.param_groups:
            pg["lr"] = LR0 * (FACTOR ** (i / (DECAY * 1000)))
        if (i + 1) % EVAL_EVERY == 0:
            with torch.no_grad(), torch.device(dev):
                o = O.run_one_iter_of_nerf(H, W, FOCAL, sc, sf, ro_all[hold], rd_all[hold], det)
            curve.append((i + 1, psnr(o[3].reshape(-1, 3))))
    return curve


res = {"iters": ITERS, "batch_rays": BATCH, "arch": "A1 8x128 skip 3 (config/lego.yml as written)", "samples": "64c+128f",
       "teacher": f"pretrained/lego-lowres networks rendered at {H}x{W} from 8 spherical poses (64c+128f, deterministic)",
       "holdout_rays": int(hold.shape[0]), "ours": [], "reference_eager_gpu": []}
for s in range(SEEDS):
    torch.cuda.synchronize(); t0 = time.time()
    c = train_ours(100 + s)
    torch.cuda.synchronize(); dt = time.time() - t0
    res["ours"].append({"seed": 100 + s, "curve": c, "seconds": dt})
    print("ours", 100 + s, c[-1], f"{dt:.1f}s", flush=True)
REF_BUDGET = float(os.environ.get("PSNR_REF_BUDGET_S", "1e9"))   # wall-clock guard for the slow arm (GPU-minute budget)
ref_spent = 0.0
for s in range(int(os.environ.get("PSNR_REF_SEEDS", str(SEEDS)))):
    if s > 0 and ref_spent * (s + 1) / s > REF_BUDGET:
        print(f"reference arm: budget of {REF_BUDGET:.0f} s reached after {s} seed(s)", flush=True)
        break
    torch.cuda.synchronize(); t0 = time.time()
    c = train_reference_eager(200 + s)
    torch.cuda.synchronize(); dt = time.time() - t0
    ref_spent += dt
    res["reference_eager_gpu"].append({"seed": 200 + s, "curve": c, "seconds": dt})
    print("reference (eager GPU)", 200 + s, c[-1], f"{dt:.1f}s", flush=True)
fo = [r["curve"][-1][1] for r in res["ours"]]
fr = [r["curve"][-1][1] for r in res["reference_eager_gpu"]]
res["final_psnr_ours"] = fo
res["final_psnr_reference"] = fr
if fo and fr:
    res["final_gap_db_mean"] = sum(fo) / len(fo) - sum(fr) / len(fr)
    res["speedup_vs_eager_gpu"] = (sum(r["seconds"] for r in res["reference_eager_gpu"]) / len(fr)) / (sum(r["seconds"] for r in res["ours"]) / len(fo))
os.makedirs(os.path.join(ROOT, "psnr_out"), exist_ok=True)
json.dump(res, open(os.path.join(ROOT, "psnr_out", "psnr_scale.json"), "w"), indent=1)
print(json.dumps({k: v for k, v in res.items() if k not in ("ours", "reference_eager_gpu")}))
