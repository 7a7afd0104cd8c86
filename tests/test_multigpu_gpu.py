"""GPU, 2 ranks over NCCL (skipped on a 1-GPU box): the ray-sharded step gives every rank the gradient of the
GLOBAL batch -- one all-reduce of the flat gradient buffer inside the render backward (SURVEY.md section 8e)."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, ret):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    import torch.distributed as dist
    from helpers import Case, build_models
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import parallel

    parallel.init_distributed()
    c = Case("a0_noview_coarse_only")
    n = c.ro.shape[0]

    def grads(rows, sync):
        (parallel.enable_gradient_sync if sync else parallel.disable_gradient_sync)()
        mc, _, epf, edf = build_models(c)
        rnd = {k: v[rows].cuda() for k, v in c.randoms.items()}
        out = nb.run_one_iter_of_nerf(c.H, c.W, c.focal, mc, None, c.ro[rows].cuda(), c.rd[rows].cuda(), c.options,
                                      encode_position_fn=epf, encode_direction_fn=edf, randoms=rnd)
        torch.nn.functional.mse_loss(out[0], c.target[rows].cuda()).backward()
        return torch.cat([p.grad.reshape(-1) for p in mc.parameters()])

    lo, hi = parallel.shard_bounds(n, rank, world)
    g_shard = grads(slice(lo, hi), sync=True)        # all-reduced inside backward
    g_full = grads(slice(0, n), sync=False)          # single-GPU global batch
    rel = ((g_shard - g_full).norm() / g_full.norm()).item()

    # coarse + fine networks: the fine half of the all-reduce is issued before the coarse backward runs
    c2 = Case("lego_a0_train")
    n2 = c2.ro.shape[0]

    def grads2(rows, sync):
        (parallel.enable_gradient_sync if sync else parallel.disable_gradient_sync)()
        mc, mf, epf, edf = build_models(c2)
        rnd = {k: v[rows].cuda() for k, v in c2.randoms.items()}
        out = nb.run_one_iter_of_nerf(c2.H, c2.W, c2.focal, mc, mf, c2.ro[rows].cuda(), c2.rd[rows].cuda(), c2.options,
                                      encode_position_fn=epf, encode_direction_fn=edf, randoms=rnd)
        tgt = c2.target[rows].cuda()
        (torch.nn.functional.mse_loss(out[0], tgt) + torch.nn.functional.mse_loss(out[3], tgt)).backward()
        return torch.cat([p.grad.reshape(-1) for p in list(mc.parameters()) + list(mf.parameters())])

    lo2, hi2 = parallel.shard_bounds(n2, rank, world)
    g2_shard = grads2(slice(lo2, hi2), sync=True)
    g2_full = grads2(slice(0, n2), sync=False)
    rel2 = ((g2_shard - g2_full).norm() / g2_full.norm()).item()
    ret[rank] = max(rel, rel2)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_allreduced_gradient_equals_global_batch():
    import torch.multiprocessing as mp

    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, 29600 + os.getpid() % 1000, ret), nprocs=2, join=True)
    assert all(v < 1e-4 for v in ret.values()), dict(ret)
