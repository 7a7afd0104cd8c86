"""lego PSNR after equal iterations: reference algorithm (oracle port, torch CPU) vs this library (CUDA).

No dataset is on disk (SURVEY.md section 0.5), so the images come from a TEACHER: the shipped pretrained
lego-lowres fine network rendered through this library's deterministic forward (perturb off, noise 0) on
rays of spherical poses (load_blender.py:32-37).  Both students are 4x128 FlexibleNeRFModels (the architecture
the reference CLI actually trains, SURVEY section 0.1) started from the SAME initial weights and fed the SAME
ray batches in the same order; each draws its own sampling noise, like two runs of the reference would.
PSNR is measured on held-out rays with the deterministic sampler.  Writes psnr_out/psnr_equivalence.json.
"""
import json, math, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
from helpers import load_weights
from oracle import nerf_oracle as O
import nerf_pytorch_b200 as nb

ITERS = int(os.environ.get("PSNR_ITERS", "300"))
BATCH = int(os.environ.get("PSNR_BATCH", "1024"))
EVAL_EVERY = int(os.environ.get("PSNR_EVAL", "50"))
THREADS = int(os.environ.get("PSNR_THREADS", "32"))
H = W = 100
FOCAL = 0.5 * W / math.tan(0.5 * 0.6911112070083618)
dev = "cuda"
torch.set_num_threads(THREADS)

def model_from(sd):
    m = nb.FlexibleNeRFModel(num_encoding_fn_xyz=10, num_encoding_fn_dir=4); m.load_state_dict(sd); return m.to(dev)

# ---- teacher images ----
sd_tc, sd_tf = load_weights("lego_lowres")
tc_, tf_ = model_from(sd_tc), model_from(sd_tf)
epf, edf = nb.get_embedding_function(10), nb.get_embedding_function(4)
det = O.make_options(num_coarse=64, num_fine=64, perturb=False, radiance_field_noise_std=0.0, white_background=False)
g = torch.Generator().manual_seed(0)
ros, rds, tgts = [], [], []
for th in range(0, 360, 45):
    pose = O.pose_spherical(float(th), -30.0, 4.0)
    ro, rd = O.get_ray_bundle(H, W, FOCAL, pose)
    with torch.no_grad():
        out = nb.run_one_iter_of_nerf(H, W, FOCAL, tc_, tf_, ro.reshape(-1, 3).to(dev), rd.reshape(-1, 3).to(dev), det,
                                      encode_position_fn=epf, encode_direction_fn=edf)
    ros.append(ro.reshape(-1, 3)); rds.append(rd.reshape(-1, 3)); tgts.append(out[3].cpu())
ro_all, rd_all, tg_all = torch.cat(ros), torch.cat(rds), torch.cat(tgts)
perm = torch.randperm(ro_all.shape[0], generator=g)
hold = perm[:4096]; pool = perm[4096:]
print(f"teacher set: {ro_all.shape[0]} rays, mean rgb {tg_all.mean().item():.3f}", flush=True)

train_opt = O.make_options(num_coarse=64, num_fine=64, perturb=True, radiance_field_noise_std=0.2)  # config/lego.yml
gi = torch.Generator().manual_seed(1)
sd0c = O.init_flexible_nerf(4, 128, 4, 10, 4, generator=gi)
sd0f = O.init_flexible_nerf(4, 128, 4, 10, 4, generator=gi)
batches = [pool[torch.randint(0, pool.shape[0], (BATCH,), generator=g)] for _ in range(ITERS)]
lr_at = lambda i: 5e-3 * (0.1 ** (i / (250 * 1000)))   # train_nerf.py:264-270

def psnr_ours(mc, mf):
    with torch.no_grad():
        out = nb.run_one_iter_of_nerf(H, W, FOCAL, mc, mf, ro_all[hold].to(dev), rd_all[hold].to(dev), det,
                                      encode_position_fn=epf, encode_direction_fn=edf)
    return -10 * math.log10(torch.nn.functional.mse_loss(out[3].cpu(), tg_all[hold]).item())

def psnr_oracle(sc, sf):
    with torch.no_grad():
        out = O.run_one_iter_of_nerf(H, W, FOCAL, sc, sf, ro_all[hold], rd_all[hold], det)
    return -10 * math.log10(torch.nn.functional.mse_loss(out[3], tg_all[hold]).item())

# ---- ours (CUDA): several sampling-noise seeds give the run-to-run band ----
def train_ours(seed):
    torch.manual_seed(seed)
    mc, mf = model_from(sd0c), model_from(sd0f)
    opt = torch.optim.Adam(list(mc.parameters()) + list(mf.parameters()), lr=5e-3)
    curve = []
    for i, idx in enumerate(batches):
        out = nb.run_one_iter_of_nerf(H, W, FOCAL, mc, mf, ro_all[idx].to(dev), rd_all[idx].to(dev), train_opt,
                                      encode_position_fn=epf, encode_direction_fn=edf)
        tgt = tg_all[idx].to(dev)
        loss = torch.nn.functional.mse_loss(out[0], tgt) + torch.nn.functional.mse_loss(out[3], tgt)
        opt.zero_grad(); loss.backward(); opt.step()
        for pg in opt.param_groups: pg["lr"] = lr_at(i)
        if (i + 1) % EVAL_EVERY == 0:
            curve.append((i + 1, psnr_ours(mc, mf)))
    return curve

t0 = time.time()
curves_ours = [train_ours(100 + s) for s in range(int(os.environ.get("PSNR_SEEDS", "6")))]
torch.cuda.synchronize(); t_ours = (time.time() - t0) / len(curves_ours)
curve_ours = curves_ours[0]
finals = [c[-1][1] for c in curves_ours]
print("ours finals:", finals, f"{t_ours:.1f}s/run", flush=True)

# ---- reference algorithm (oracle, CPU) ----
torch.manual_seed(200)
sc = {k: v.clone().requires_grad_(True) for k, v in sd0c.items()}
sf = {k: v.clone().requires_grad_(True) for k, v in sd0f.items()}
opt = torch.optim.Adam(list(sc.values()) + list(sf.values()), lr=5e-3)
curve_ref, t0 = [], time.time()
for i, idx in enumerate(batches):
    out = O.run_one_iter_of_nerf(H, W, FOCAL, sc, sf, ro_all[idx], rd_all[idx], train_opt)
    loss = O.nerf_loss(out, tg_all[idx])
    opt.zero_grad(); loss.backward(); opt.step()
    for pg in opt.param_groups: pg["lr"] = lr_at(i)
    if (i + 1) % EVAL_EVERY == 0:
        curve_ref.append((i + 1, psnr_oracle(sc, sf)))
        print("ref", curve_ref[-1], f"{time.time()-t0:.0f}s", flush=True)
t_ref = time.time() - t0
res = {"iters": ITERS, "batch_rays": BATCH, "arch": "A0 4x128 (as the reference CLI trains)", "samples": "64c+64f",
       "teacher": "pretrained/lego-lowres fine net rendered at 100x100 from 8 spherical poses",
       "psnr_ours": curve_ours, "psnr_reference_cpu": curve_ref, "seconds_ours": t_ours, "seconds_reference_cpu": t_ref,
       "cpu_threads": THREADS, "psnr_ours_final_all_seeds": finals,
       "final_gap_db_vs_mean": sum(finals) / len(finals) - curve_ref[-1][1]}
os.makedirs(os.path.join(ROOT, "psnr_out"), exist_ok=True)
json.dump(res, open(os.path.join(ROOT, "psnr_out", "psnr_equivalence.json"), "w"), indent=1)
print(json.dumps(res))
