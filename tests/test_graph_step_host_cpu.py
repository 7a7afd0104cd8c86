"""CPU (no GPU needed): CapturedTrainStep refuses what it cannot capture before it launches anything."""
import pytest
import torch

from oracle import nerf_oracle as O


def _setup(n=64, chunksize=8192, fine=True):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import parallel, train_utils

    torch.manual_seed(0)
    mk = lambda: nb.FlexibleNeRFModel(num_layers=4, hidden_size=128, skip_connect_every=4, num_encoding_fn_xyz=10,
                                      num_encoding_fn_dir=4)
    mc, mf = mk(), (mk() if fine else None)
    arch = train_utils._arch_of(mc, (10, True, True), (4, True, True))
    opt = parallel.FusedAdam([(m, arch) for m in (mc, mf) if m is not None], lr=5e-3, lr_decay=250)
    options = O.make_options(num_coarse=64, num_fine=64 if fine else 0, chunksize=chunksize)
    options.nerf.train.num_random_rays = n
    source = (torch.rand(2, 8, 10, 3), torch.eye(4).repeat(2, 1, 1), 12.0)
    return dict(model_coarse=mc, model_fine=mf, encode_position_fn=nb.get_embedding_function(10),
                encode_direction_fn=nb.get_embedding_function(4), options=options, optimizer=opt, seed=1,
                source=source)


def _refused(exc, match, **change):
    import nerf_pytorch_b200 as nb
    from nerf_pytorch_b200 import ops

    kw = _setup(**{k: change.pop(k) for k in ("n", "chunksize") if k in change})
    kw.update(change)
    before = ops.launch_count()
    with pytest.raises(exc, match=match):
        nb.CapturedTrainStep(**kw)
    assert ops.launch_count() == before


def test_refuses_cpu_tensors():
    _refused(NotImplementedError, "CUDA tensor")


def test_refuses_impl_3_and_unknown_impls():
    _refused(NotImplementedError, "inference only", impl=3)
    _refused(ValueError, "impl must be", impl=2)


def test_refuses_more_rays_than_one_chunk():
    _refused(ValueError, "one chunk", n=64, chunksize=32)


def test_refuses_gradient_sync():
    from nerf_pytorch_b200 import train_utils

    train_utils._GRAD_SYNC = (None, 2)
    try:
        _refused(NotImplementedError, "gradient sync")
    finally:
        train_utils._GRAD_SYNC = None


def test_refuses_more_rays_than_pixels():
    _refused(ValueError, "cannot draw 81 distinct", n=81)


def test_refuses_a_pool_of_unlike_images(tmp_path):
    from nerf_pytorch_b200 import CachedRayPool

    paths = []
    for i, (h, w) in enumerate(((4, 5), (4, 6))):
        d = {"height": h, "width": w, "focal_length": 5.0, "ray_bundle": torch.rand(2, h, w, 3),
             "target": torch.rand(h, w, 3)}
        torch.save(d, tmp_path / f"{i}.data")
        paths.append(str(tmp_path / f"{i}.data"))
    _refused(ValueError, "differ", n=8, source=CachedRayPool(paths, device="cpu"))


def test_refuses_a_schedule_that_disagrees_with_the_options():
    from types import SimpleNamespace as NS

    kw = _setup()
    kw["options"].optimizer = NS(lr=1e-3)
    kw["options"].scheduler = NS(lr_decay=250, lr_decay_factor=0.1)
    import nerf_pytorch_b200 as nb

    with pytest.raises(ValueError, match="disagrees"):
        nb.CapturedTrainStep(**kw)
